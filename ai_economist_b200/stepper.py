"""Thin Python driver over the C-ABI: allocates the device buffers (PyTorch-owned), binds them, uploads host
reset snapshots and launches steps.  Plumbing only — all compute is in the CUDA library."""
import ctypes as C
import numbers

import numpy as np

from . import _abi


def bf16_bits_to_float32(a):
    """float32 values of raw bfloat16 bits (uint16): exact, every bfloat16 is a float32."""
    return (np.asarray(a).astype(np.uint32) << 16).view(np.float32)


def buf_kind_numpy(buf):
    """"f32" / "bf16" for a C-contiguous float32 / uint16 (raw bfloat16 bits) numpy array, else None."""
    if isinstance(buf, np.ndarray) and buf.flags["C_CONTIGUOUS"]:
        return {np.dtype(np.float32): "f32", np.dtype(np.uint16): "bf16"}.get(buf.dtype)
    return None


def buf_kind_torch(torch, device, buf):
    """"f32" / "bf16" for a contiguous float32 / bfloat16 tensor on `device`, else None."""
    if isinstance(buf, torch.Tensor) and buf.device == device and buf.is_contiguous():
        return {torch.float32: "f32", torch.bfloat16: "bf16"}.get(buf.dtype)
    return None


def float_kind_numpy(buf):
    """"f32" / "f64" for a C-contiguous float32 / float64 numpy array, else None."""
    if isinstance(buf, np.ndarray) and buf.flags["C_CONTIGUOUS"]:
        return {np.dtype(np.float32): "f32", np.dtype(np.float64): "f64"}.get(buf.dtype)
    return None


def float_kind_torch(torch, device, buf):
    """"f32" / "f64" for a contiguous float32 / float64 tensor on `device`, else None."""
    if isinstance(buf, torch.Tensor) and buf.device == device and buf.is_contiguous():
        return {torch.float32: "f32", torch.float64: "f64"}.get(buf.dtype)
    return None


def is_i32_numpy(buf):
    return isinstance(buf, np.ndarray) and buf.flags["C_CONTIGUOUS"] and buf.dtype == np.int32


def is_i32_torch(torch, device, buf):
    return isinstance(buf, torch.Tensor) and buf.device == device and buf.is_contiguous() and buf.dtype == torch.int32


_EVALUATE_ACTIONS = None


def evaluate_actions_function():
    """The torch.autograd.Function of evaluate_actions (built on first use: torch is imported lazily)."""
    global _EVALUATE_ACTIONS
    if _EVALUATE_ACTIONS is not None:
        return _EVALUATE_ACTIONS
    import torch
    from torch.autograd.function import once_differentiable

    class EvaluateActions(torch.autograd.Function):
        """(log_prob_agent, log_prob_planner, entropy_agent, entropy_planner) of stored actions, differentiable with
        respect to both logits tensors: the backward is one launch of the library's backward kernel on the current
        stream, which recomputes the softmax from the saved logits and masks."""

        @staticmethod
        def forward(ctx, stepper, logits_agent, logits_planner, actions_agent, actions_planner, mask_agent, mask_planner):
            ctx.set_materialize_grads(False)   # an unused output's gradient stays None: a NULL upstream (zero)
            ctx.stepper = stepper
            ctx.save_for_backward(logits_agent, logits_planner, actions_agent, actions_planner, mask_agent, mask_planner)
            return stepper.evaluate_policy(logits_agent, logits_planner, (actions_agent, actions_planner),
                                           (mask_agent, mask_planner))

        @staticmethod
        @once_differentiable
        def backward(ctx, g_lp_a, g_lp_p, g_h_a, g_h_p):
            la, lp, aa, ap, ma, mp = ctx.saved_tensors
            c = lambda g: None if g is None else g.to(torch.float32).contiguous()
            ga, gp = ctx.stepper.evaluate_policy_backward(la, lp, (aa, ap), (ma, mp), (c(g_lp_a), c(g_lp_p)),
                                                          (c(g_h_a), c(g_h_p)))
            return None, ga, gp, None, None, None, None

    _EVALUATE_ACTIONS = EvaluateActions
    return _EVALUATE_ACTIONS


class PolicySampler:
    """sample_policy() of a stepper: a policy's actions drawn on the device from its logits under the env's current
    masks (aie_sample_policy / aie_covid_sample_policy).  The stepper provides _policy_fn (the ABI entry point),
    _policy_shapes() -> (agent logits, planner logits or None, agent log-probs, planner log-probs or None) and
    _buf_kind(buf) ("f32" | "bf16" | None: not a contiguous float buffer of this backend's device)."""

    def sample_policy(self, logits_agent, logits_planner=None, seed=0, greedy=False, out=None):
        """Overwrite the action buffers with one draw per mask segment (greedy=True: the masked argmax) and return
        (log_prob_agent, log_prob_planner): float32 buffers shaped like the action buffers (log_prob_planner is None
        without planner actions).  They are the stepper's own, reused by every call, unless `out` = (log_prob_agent,
        log_prob_planner) names the caller's (either may be None).  Asynchronous on the stream.  Logits: contiguous
        float32 or bfloat16 (raw uint16 bits on numpy backends), both of the same dtype, on the stepper's device;
        anything else is a ValueError before the library is called."""
        sa, sp, sla, slp = self._policy_shapes()
        kind = self._buf_kind(logits_agent)
        if kind is None or tuple(logits_agent.shape) != sa:
            raise ValueError("logits_agent must be a contiguous float32 or bfloat16 %s tensor on the env's device" % (sa,))
        if sp is not None:
            if logits_planner is None:
                raise ValueError("logits_planner is required: this config has planner actions")
            if self._buf_kind(logits_planner) != kind or tuple(logits_planner.shape) != sp:
                raise ValueError("logits_planner must be a contiguous %s tensor of shape %s on the env's device (the dtype "
                                 "of logits_agent)" % ("float32" if kind == "f32" else "bfloat16", sp))
        lp_a, lp_p = (None, None) if out is None else out
        if getattr(self, "_policy_lp", None) is None:
            self._policy_lp = {}
        if lp_a is None:
            lp_a = self._policy_lp.get("a")
            if lp_a is None:
                lp_a = self._policy_lp["a"] = self._alloc(sla, "f32")
        elif self._buf_kind(lp_a) != "f32" or tuple(lp_a.shape) != sla:
            raise ValueError("out[0] must be a contiguous float32 %s tensor on the env's device" % (sla,))
        if slp is None:
            lp_p = None
        elif lp_p is None:
            lp_p = self._policy_lp.get("p")
            if lp_p is None:
                lp_p = self._policy_lp["p"] = self._alloc(slp, "f32")
        elif self._buf_kind(lp_p) != "f32" or tuple(lp_p.shape) != slp:
            raise ValueError("out[1] must be a contiguous float32 %s tensor on the env's device" % (slp,))
        p = _abi.AiePolicyLogits()
        p.agent = self._ptr(logits_agent)
        p.planner = self._ptr(logits_planner) if sp is not None else None
        p.logits_dtype = _abi.OBS_BF16 if kind == "bf16" else _abi.OBS_F32
        p.greedy = 1 if greedy else 0
        p.log_prob_agent = self._ptr(lp_a)
        p.log_prob_planner = self._ptr(lp_p) if lp_p is not None else None
        self._check(self._policy_fn(self._h, C.byref(p), C.c_uint64(int(seed)), self._stream()))
        return lp_a, lp_p

    # -- captured rollouts (aie_rollout_capture_begin ... / aie_covid_rollout_capture_begin ...) ----------------------
    # The stepper provides _capture_prefix ("aie" | "aie_covid"); the four calls keep rollout_slot in step with the
    # library's cursor.  A stepper that can record CUDA graphs sets supports_rollout_capture.
    supports_rollout_capture = False

    def _capture_fn(self, name):
        return getattr(self.lib, "%s_rollout_%s" % (self._capture_prefix, name))

    def rollout_capture_begin(self):
        """Start recording the bound rollout (slot 0): until rollout_capture_end() only step() and sample_policy() run."""
        self._check(self._capture_fn("capture_begin")(self._h, self._stream()))
        self._capturing = True

    def rollout_capture_end(self):
        """Stop recording: the library's host state and the cursor are as they were at rollout_capture_begin()."""
        self._capturing = False
        self._check(self._capture_fn("capture_end")(self._h))
        self.rollout_slot = 0

    def rollout_replay_begin(self):
        """Before a replay (cursor 0): the current call counter into the device counter, on the stream."""
        self._check(self._capture_fn("replay_begin")(self._h, self._stream()))

    def rollout_replay_end(self):
        """After a replay: the library's host state advanced by what the captured calls did; the cursor at T."""
        self._check(self._capture_fn("replay_end")(self._h))
        self.rollout_slot = self.rollout.T

    def _refused_in_capture(self, rc):
        """A call the library refused because a rollout is being recorded (only the step and the policy sampler run)."""
        if rc == _abi.AIE_ESTATE and getattr(self, "_capturing", False):
            raise ValueError("not available while a rollout is being captured (capture_rollout's act may call "
                             "sample_actions only): %s" % self.lib.aie_last_error().decode())

    # -- evaluation of stored actions (aie_evaluate_policy / aie_covid_evaluate_policy and their backward) -----------
    def _eval_args(self, logits_agent, logits_planner, actions, masks, grads=()):
        """Validate the inputs of an evaluation; returns (aie_policy_eval with the inputs set, leading shape, row
        count, planner?, logits kind, output row shapes).  Raises ValueError before the library is called."""
        sa, sp, sla, slp = self._policy_shapes()
        ra, rp, rla = sa[1:], None if sp is None else sp[1:], sla[1:]
        rlp = None if slp is None else slp[1:]
        rma, rmp = self._mask_rows()
        kind = self._buf_kind(logits_agent)
        shape = tuple(getattr(logits_agent, "shape", ()))
        if kind is None or len(shape) < len(ra) or shape[len(shape) - len(ra):] != ra:
            raise ValueError("logits_agent must be a contiguous float32 or bfloat16 [*B, %s] tensor on the env's device"
                             % ", ".join(map(str, ra)))
        lead = shape[:len(shape) - len(ra)]
        tname = "float32" if kind == "f32" else "bfloat16"
        if not isinstance(actions, (tuple, list)) or len(actions) != 2:
            raise ValueError("actions must be (actions_agent, actions_planner)")
        if not isinstance(masks, (tuple, list)) or len(masks) != 2:
            raise ValueError("masks must be (mask_agent, mask_planner)")
        mkind = self._buf_kind(masks[0])
        if mkind is None or tuple(masks[0].shape) != lead + rma:
            raise ValueError("mask_agent must be a contiguous float32 or bfloat16 %s tensor on the env's device"
                             % (lead + rma,))
        if not self._is_i32(actions[0]) or tuple(actions[0].shape) != lead + rla:
            raise ValueError("actions_agent must be a contiguous int32 %s tensor on the env's device" % (lead + rla,))
        planner = sp is not None
        if planner:
            if logits_planner is None or self._buf_kind(logits_planner) != kind or tuple(logits_planner.shape) != lead + rp:
                raise ValueError("logits_planner must be a contiguous %s %s tensor on the env's device (the dtype of "
                                 "logits_agent): this config has planner actions" % (tname, lead + rp))
            if masks[1] is None or self._buf_kind(masks[1]) != mkind or tuple(masks[1].shape) != lead + rmp:
                raise ValueError("mask_planner must be a contiguous %s tensor of the dtype of mask_agent on the env's "
                                 "device" % (lead + rmp,))
            if not self._is_i32(actions[1]) or tuple(actions[1].shape) != lead + rlp:
                raise ValueError("actions_planner must be a contiguous int32 %s tensor on the env's device" % (lead + rlp,))
        for name, (ga, gp) in grads:
            if ga is not None and (self._buf_kind(ga) != "f32" or tuple(ga.shape) != lead + rla):
                raise ValueError("%s[0] must be None or a contiguous float32 %s tensor on the env's device" % (name, lead + rla))
            if planner and gp is not None and (self._buf_kind(gp) != "f32" or tuple(gp.shape) != lead + rlp):
                raise ValueError("%s[1] must be None or a contiguous float32 %s tensor on the env's device" % (name, lead + rlp))
        p = _abi.AiePolicyEval()
        p.logits_agent, p.mask_agent, p.actions_agent = self._ptr(logits_agent), self._ptr(masks[0]), self._ptr(actions[0])
        if planner:
            p.logits_planner, p.mask_planner, p.actions_planner = (self._ptr(logits_planner), self._ptr(masks[1]),
                                                                   self._ptr(actions[1]))
        p.logits_dtype = _abi.OBS_BF16 if kind == "bf16" else _abi.OBS_F32
        p.mask_dtype = _abi.OBS_BF16 if mkind == "bf16" else _abi.OBS_F32
        n = int(np.prod(lead, dtype=np.int64)) if lead else 1
        return p, lead, n, planner, kind, (ra, rp, rla, rlp)

    def evaluate_policy(self, logits_agent, logits_planner, actions, masks):
        """Log-probabilities and entropies of stored actions under the masks they were drawn with, per mask segment:
        (log_prob_agent, log_prob_planner, entropy_agent, entropy_planner), new float32 buffers shaped like the actions
        (the planner entries are None without planner actions).  Logits: [*B, <the sampler's logits row>], float32 or
        bfloat16 (raw uint16 bits on numpy backends), both of one dtype; masks = (mask_agent, mask_planner) as the
        env wrote them ([*B, <mask row>], float32 or bfloat16); actions = (actions_agent, actions_planner), int32
        [*B, <action row>].  *B is any leading shape (a minibatch of stored steps).  Asynchronous on the stream; no
        state of the env is read or changed.  Anything else is a ValueError before the library is called."""
        p, lead, n, planner, _, (_, _, rla, rlp) = self._eval_args(logits_agent, logits_planner, actions, masks)
        lp_a, h_a = self._eval_out(lead + rla, "f32"), self._eval_out(lead + rla, "f32")
        lp_p, h_p = (self._eval_out(lead + rlp, "f32"), self._eval_out(lead + rlp, "f32")) if planner else (None, None)
        p.log_prob_agent, p.entropy_agent = self._ptr(lp_a), self._ptr(h_a)
        if planner:
            p.log_prob_planner, p.entropy_planner = self._ptr(lp_p), self._ptr(h_p)
        self._check(self._eval_fns[0](self._h, C.byref(p), C.c_int64(n), self._stream()))
        return lp_a, lp_p, h_a, h_p

    def evaluate_policy_backward(self, logits_agent, logits_planner, actions, masks, grad_log_prob=(None, None),
                                 grad_entropy=(None, None)):
        """The gradient of sum(g_lp * log_prob + g_H * entropy) with respect to (logits_agent, logits_planner) for
        the inputs of evaluate_policy; grad_log_prob and grad_entropy = (agent, planner) float32 tensors shaped like
        the actions, None for zero.  Returns new tensors of the logits' shape and dtype (None for the planner without
        planner actions).  Asynchronous on the stream."""
        p, lead, n, planner, kind, (ra, rp, _, _) = self._eval_args(
            logits_agent, logits_planner, actions, masks, (("grad_log_prob", grad_log_prob), ("grad_entropy", grad_entropy)))
        ga = self._eval_out(lead + ra, kind)
        gp = self._eval_out(lead + rp, kind) if planner else None
        ptr = lambda x: None if x is None else self._ptr(x)
        p.grad_log_prob_agent, p.grad_entropy_agent, p.grad_logits_agent = ptr(grad_log_prob[0]), ptr(grad_entropy[0]), ptr(ga)
        if planner:
            p.grad_log_prob_planner, p.grad_entropy_planner = ptr(grad_log_prob[1]), ptr(grad_entropy[1])
            p.grad_logits_planner = ptr(gp)
        self._check(self._eval_fns[1](self._h, C.byref(p), C.c_int64(n), self._stream()))
        return ga, gp

    def evaluate_actions(self, logits_agent, logits_planner, actions, masks):
        """evaluate_policy, differentiable with respect to both logits tensors when they are torch tensors (through
        evaluate_actions_function()); numpy backends call evaluate_policy directly."""
        if isinstance(logits_agent, np.ndarray):
            return self.evaluate_policy(logits_agent, logits_planner, actions, masks)
        planner = self._policy_shapes()[1] is not None
        if not isinstance(actions, (tuple, list)) or len(actions) != 2:
            raise ValueError("actions must be (actions_agent, actions_planner)")
        if not isinstance(masks, (tuple, list)) or len(masks) != 2:
            raise ValueError("masks must be (mask_agent, mask_planner)")
        return evaluate_actions_function().apply(self, logits_agent, logits_planner if planner else None, actions[0],
                                                 actions[1] if planner else None, masks[0], masks[1] if planner else None)

    # -- advantages of a stored rollout (aie_compute_advantages / aie_covid_compute_advantages) -----------------------
    @staticmethod
    def _discount_pair(x, name, planner):
        """(agent, planner) of a gamma or lambda given as a float or a pair; each a float in [0, 1]."""
        pair = tuple(x) if isinstance(x, (tuple, list)) else (x, x)
        if len(pair) != 2:
            raise ValueError("%s must be a float or an (agents, planner) pair" % name)
        out = []
        for k, v in enumerate(pair):
            if k == 1 and not planner:
                out.append(0.0)
                continue
            if isinstance(v, bool) or not isinstance(v, numbers.Real):
                raise ValueError("%s must be a float or an (agents, planner) pair of floats" % name)
            if not 0.0 <= float(v) <= 1.0:   # NaN fails both comparisons
                raise ValueError("%s must lie in [0, 1], got %r" % (name, v))
            out.append(float(v))
        return out

    def compute_advantages(self, rewards, values, dones, last_values, final_values=None, *, gamma, lam=1.0,
                           per_episode_end=False):
        """Generalised advantage estimates and value targets of a stored rollout of T steps, bootstrapped at episode
        ends: (adv_agent, adv_planner, ret_agent, ret_planner), new float32 buffers shaped like the rewards.  rewards =
        (agent [T, E, A], planner [T, E]), float32 or float64 each; values = (agent, planner), float32 like the
        rewards; dones int32 [T, E]; last_values = (agent [E, A], planner [E]), float32; final_values None (an episode
        end is terminal) or (agent, planner) like values, read only where dones is set.  gamma, lam: floats in
        [0, 1], or (agents, planner) pairs.  Every planner entry may be None together (no planner outputs).  The
        recursion and its float64 rounding are spelled out in include/aie_b200.h.  Asynchronous on the stream; no
        state of the env is read or changed.  Anything else is a ValueError before the library is called."""
        sa = self._policy_shapes()[0]
        E, A = sa[0], sa[1]
        if not isinstance(rewards, (tuple, list)) and tuple(getattr(rewards, "shape", ())[1:]) == (E, A + 1):
            # a rollout's rewards as the env stores them, [T, E, A + 1] (agents, then the planner): split, one copy each
            rewards = (self._contiguous(rewards[..., :A]), self._contiguous(rewards[..., A]))
        pairs = dict(rewards=rewards, values=values, last_values=last_values)
        if final_values is not None:
            pairs["final_values"] = final_values
        for name, x in pairs.items():
            if not isinstance(x, (tuple, list)) or len(x) != 2:
                raise ValueError("%s must be an (agent, planner) pair" % name)
        planner = rewards[1] is not None
        if any((x[1] is not None) != planner for x in pairs.values()):
            raise ValueError("the planner entries of rewards, values, last_values and final_values must be all given "
                             "or all None")
        shape_a = tuple(getattr(rewards[0], "shape", ()))
        if len(shape_a) != 3 or shape_a[1:] != (E, A):
            raise ValueError("rewards[0] must be a [T, %d, %d] tensor" % (E, A))
        T = shape_a[0]
        if T > 0x7FFFFFFF:
            raise ValueError("T must fit in int32")
        rows = ((T, E, A), (T, E))
        # final values [T, E, ...] (the row of each done step), or with per_episode_end=True [K, E, ...], K >= 1 (the row
        # of each done step's episode-end ordinal in its column: a bound rollout's final slots, aie_compute_advantages_k)
        K = None
        if per_episode_end:
            if final_values is None:
                raise ValueError("per_episode_end=True needs final_values [K, E, ...]")
            fs = tuple(getattr(final_values[0], "shape", ()))
            if len(fs) != 3 or fs[1:] != (E, A) or fs[0] < 1:
                raise ValueError("final_values[0] must be a [K, %d, %d] tensor, K >= 1, with per_episode_end=True" % (E, A))
            K = fs[0]
        frows = ((K or T, E, A), (K or T, E))
        rk = []
        for k, who in enumerate(("agent", "planner")[:2 if planner else 1]):
            kind = self._float_kind(rewards[k])
            if kind is None or tuple(rewards[k].shape) != rows[k]:
                raise ValueError("rewards[%d] (%s) must be a contiguous float32 or float64 %s tensor on the env's device"
                                 % (k, who, rows[k]))
            rk.append(kind)
            for name, want in (("values", rows[k]), ("last_values", rows[k][1:]), ("final_values", frows[k])):
                if name in pairs and (self._float_kind(pairs[name][k]) != "f32" or tuple(pairs[name][k].shape) != want):
                    raise ValueError("%s[%d] (%s) must be a contiguous float32 %s tensor on the env's device"
                                     % (name, k, who, want))
        if not self._is_i32(dones) or tuple(dones.shape) != (T, E):
            raise ValueError("dones must be a contiguous int32 %s tensor on the env's device" % ((T, E),))
        g, l = self._discount_pair(gamma, "gamma", planner), self._discount_pair(lam, "lam", planner)
        q = _abi.AieAdvantageArgs()
        q.rewards_agent, q.values_agent, q.last_values_agent = self._ptr(rewards[0]), self._ptr(values[0]), self._ptr(last_values[0])
        q.rewards_agent_dtype = _abi.REWARD_F64 if rk[0] == "f64" else _abi.REWARD_F32
        q.dones = self._ptr(dones)
        q.gamma_agent, q.gamma_planner, q.lambda_agent, q.lambda_planner = g[0], g[1], l[0], l[1]
        adv_a, ret_a = self._eval_out(rows[0], "f32"), self._eval_out(rows[0], "f32")
        q.adv_agent, q.ret_agent = self._ptr(adv_a), self._ptr(ret_a)
        adv_p = ret_p = None
        if planner:
            q.rewards_planner, q.values_planner = self._ptr(rewards[1]), self._ptr(values[1])
            q.last_values_planner = self._ptr(last_values[1])
            q.rewards_planner_dtype = _abi.REWARD_F64 if rk[1] == "f64" else _abi.REWARD_F32
            adv_p, ret_p = self._eval_out(rows[1], "f32"), self._eval_out(rows[1], "f32")
            q.adv_planner, q.ret_planner = self._ptr(adv_p), self._ptr(ret_p)
        if final_values is not None:
            q.final_values_agent = self._ptr(final_values[0])
            if planner:
                q.final_values_planner = self._ptr(final_values[1])
        if K is not None:
            self._check(self._adv_k_fn(self._h, C.byref(q), C.c_int32(T), C.c_int32(K), self._stream()))
        else:
            self._check(self._adv_fn(self._h, C.byref(q), C.c_int32(T), self._stream()))
        return adv_a, adv_p, ret_a, ret_p

    @staticmethod
    def _contiguous(x):
        return x.contiguous() if hasattr(x, "contiguous") else np.ascontiguousarray(x)

    def _mask_rows(self):
        """(agent mask row, planner mask row or None): the logits' rows (COVID-19 overrides: its agent mask is transposed)."""
        sa, sp, _, _ = self._policy_shapes()
        return sa[1:], None if sp is None else sp[1:]

    def _eval_out(self, shape, kind):
        return np.empty(shape, {"f32": np.float32, "bf16": np.uint16}[kind])

    def _is_i32(self, buf):
        return is_i32_numpy(buf)

    def _float_kind(self, buf):
        return float_kind_numpy(buf)

    def _buf_kind(self, buf):
        return buf_kind_numpy(buf)


class Rollout:
    """The device tensors of a rollout of T steps stored in place (aie_bind_rollout), allocated by the stepper.

    buf[name]: every observation / mask tensor [T + 1, E, ...] (slot t: the observation step t's action is taken from,
    slot T: the one after the last step), "actions_agent" / "actions_planner" [T, E, ...], "reward" [T, E, A + 1] and
    "done" [T, E] (step t's), and with final_obs "final_<name>" [K, E, ...], K = ceil(T / episode_length): row (k, e) the
    observation of the state in which replica e's k-th episode end within the rollout ended."""

    def __init__(self, T, K, buf, obs_names, final_obs):
        self.T, self.K, self.buf = T, K, buf
        self.obs_names = tuple(obs_names)
        self.has_final_obs = final_obs

    @property
    def obs_tensors(self):
        return {k: self.buf[k] for k in self.obs_names}

    @property
    def final_obs_tensors(self):
        return {k: self.buf["final_" + k] for k in self.obs_names} if self.has_final_obs else None


class BatchStepper(PolicySampler):
    """Backend-agnostic part (buffer bookkeeping + ABI calls).  Subclasses supply allocation.

    Reference counterpart: FoundationEnvWrapper (ai_economist/foundation/env_wrapper.py:84-418), which owns
    the WarpDrive data manager / function manager for the COVID env.
    """

    # "bf16": bfloat16 observations (spec["obs_dtype"] == "bfloat16"); numpy backends hold their raw bits
    _DTYPES = {"u8": np.uint8, "i16": np.int16, "i32": np.int32, "f32": np.float32, "f64": np.float64, "bf16": np.uint16}

    def __init__(self, spec, n_envs, lib, device_index=0, auto_reset=True, event_envs=0):
        self.spec = dict(spec)
        self.n_envs = int(n_envs)
        self.lib = lib
        self.cfg = _abi.config_from_spec(spec, auto_reset=auto_reset)
        h = C.c_void_p()
        self._check(lib.aie_create(C.byref(self.cfg), self.n_envs, int(device_index), C.byref(h)))
        self._h = h
        self.dims = _abi.AieDims()
        self._check(lib.aie_get_dims(self._h, C.byref(self.dims)))
        d, E, A = self.dims, self.n_envs, spec["n_agents"]
        H, W = spec["height"], spec["width"]
        full = bool(spec.get("full_observability", 0))   # agents see the whole map: [M, H, W] / [2, H, W] per agent
        none = bool(spec.get("scenario_kind", 0) == 1)   # one-step-economy: no spatial observations (zero-size tensors)
        assert d.agent_map_elems == (0 if none else d.n_map_channels * H * W if full else (d.n_map_channels + 1) * d.window ** 2)
        fo = "bf16" if self.cfg.obs_dtype == _abi.OBS_BF16 else "f32"   # the float observation / mask tensors
        shapes = {
            "state": ("u8", (E, d.state_bytes)), "state0": ("u8", (E, d.state_bytes)),
            "actions_agent": ("i32", (E, A, d.n_act_agent)),
            "actions_planner": ("i32", (E, max(1, d.n_act_planner))),
            "obs_agent_map": (fo, (E, A, 0) if none else (E, A, d.n_map_channels, H, W) if full else
                              (E, A, d.n_map_channels + 1, d.window, d.window)),
            "obs_agent_idx": ("i16", (E, A, 0) if none else (E, A, 2, H, W) if full else (E, A, 2, d.window, d.window)),
            "obs_agent_flat": (fo, (E, A, d.flat_agent)),
            "mask_agent": (fo, (E, A, d.mask_agent)),
            "obs_planner_map": (fo, (E, d.n_map_channels, H, W)),
            "obs_planner_idx": ("i16", (E, 2, H, W)),
            "obs_planner_flat": (fo, (E, d.flat_planner)),
            "obs_planner_agents": (fo, (E, A, d.flat_planner_agent)),
            "mask_planner": (fo, (E, d.mask_planner)),
            "obs_time": (fo, (E,)),
            "reward": ("f64", (E, A + 1)),
            "done": ("i32", (E,)),
        }
        if auto_reset:  # end-of-episode record snapshots (previous_episode_metrics)
            shapes["episode_final"] = ("u8", (E, d.state_bytes))
        if not spec["planner_gets_spatial_info"]:
            del shapes["obs_planner_map"], shapes["obs_planner_idx"]
        # spec["final_obs"]: final_<name> twins of the observation / mask buffers, written by step() for the replicas
        # whose episode the auto-reset ended (aie_observe_final)
        self.final_obs = bool(spec.get("final_obs", False))
        if self.final_obs and not auto_reset:
            raise ValueError("final_obs needs auto_reset: without it the observations of the ending step are the final ones")
        if self.final_obs:
            shapes.update({"final_" + k: shapes[k] for k in _abi.OBS_NAMES if k in shapes})
        # per-step event log of the first event_envs replicas (dense logs): capacity = every agent builds, gathers both
        # resources and every resting order trades
        self.event_envs = max(0, min(int(event_envs), E))
        K = int(spec.get("max_num_orders", 0) or 0) if "ContinuousDoubleAuction" in spec["components"] else 0
        self.event_cap = int(min(1024, 3 * A + 2 * A * K + 8))
        if self.event_envs:
            shapes["events"] = ("i32", (self.event_envs, self.event_cap + 1, 8))
        self.buf = {k: self._alloc(shape, dt) for k, (dt, shape) in shapes.items()}
        self._shapes = shapes
        self.rollout = None   # the bound Rollout (bind_rollout), and its slot cursor
        self.rollout_slot = 0
        self._bf16 = {k for k, (dt, _) in shapes.items() if dt == "bf16"}
        bufs = _abi.AieBuffers()
        for name in _abi._BUF_NAMES:
            ok = name in self.buf and int(np.prod(self.buf[name].shape)) > 0   # zero-size tensors have no storage
            setattr(bufs, name, self._ptr(self.buf[name]) if ok else None)
        bufs.events = self._ptr(self.buf["events"]) if self.event_envs else None
        bufs.event_envs, bufs.event_cap = self.event_envs, self.event_cap
        self._check(lib.aie_bind_buffers(self._h, C.byref(bufs)))
        self._fields = {}
        self._final_out = self._final_bufs = None
        if self.final_obs:   # the default destination of observe_final, built once (step() launches into it every step)
            self._final_out = {k: self.buf["final_" + k] for k in _abi.OBS_NAMES if k in self.buf}
            self._final_bufs = self._obs_buffers(self._final_out)

    # -- to be provided by subclasses ------------------------------------------------------------------
    def _alloc(self, shape, dt):
        raise NotImplementedError

    def _ptr(self, buf):
        raise NotImplementedError

    def _stream(self):
        return None

    def _empty(self, shape, dt):
        """An output buffer whose contents are about to be overwritten (default: the zeroed allocation)."""
        return self._alloc(shape, dt)

    def to_numpy(self, buf):
        raise NotImplementedError

    # --------------------------------------------------------------------------------------------------
    def _check(self, rc):
        if rc != _abi.AIE_OK:
            self._refused_in_capture(rc)
            raise _abi.AieError("aie error %d: %s" % (rc, self.lib.aie_last_error().decode()))

    _capture_prefix = "aie"

    def close(self):
        if getattr(self, "_h", None):
            self.lib.aie_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def flat_layout(self, which):
        """[(key, offset, size)] of the fields concatenated into a flat vector (base_env.py:562-589);
        which: "agent" | "planner" | "planner_agent"."""
        idx = {"agent": 0, "planner": 1, "planner_agent": 2}[which]
        n = self.lib.aie_get_flat_layout(self._h, idx, None, 0)
        if n < 0:
            self._check(n)
        arr = (_abi.AieFlatField * max(1, n))()
        self.lib.aie_get_flat_layout(self._h, idx, arr, n)
        return [(arr[i].key.decode(), int(arr[i].offset), int(arr[i].size)) for i in range(n)]

    def metric_layout(self):
        """[(key, is_int)] of the episode-metrics table's columns: the reference's env.metrics keys for this config in
        their dict order (aie_get_metric_layout)."""
        if getattr(self, "_metric_layout", None) is None:
            n = self.lib.aie_get_metric_layout(self._h, None, 0)
            if n < 0:
                self._check(n)
            arr = (_abi.AieMetricKey * max(1, n))()
            self.lib.aie_get_metric_layout(self._h, arr, n)
            self._metric_layout = [(arr[i].key.decode(), bool(arr[i].is_int)) for i in range(n)]
        return list(self._metric_layout)

    def episode_metrics(self, final=False, out=None):
        """env.metrics of every replica as a float64 table [n_envs, K] in metric_layout() order, computed on the device by
        one kernel launch, asynchronous on the stream (aie_episode_metrics).  final=True: the metrics of each replica's
        last finished episode (needs auto_reset; rows of replicas that have finished none are NaN).  out: an optional
        preallocated contiguous float64 [n_envs, K] buffer on the same device."""
        K = len(self.metric_layout())
        if out is None:
            out = self._empty((self.n_envs, K), "f64")
        elif tuple(out.shape) != (self.n_envs, K) or not self._is_f64_contiguous(out):
            raise _abi.AieError("episode_metrics: out must be a contiguous float64 [%d, %d] buffer" % (self.n_envs, K))
        self._check(self.lib.aie_episode_metrics(self._h, 1 if final else 0, self._ptr(out), self._stream()))
        return out

    def _is_f64_contiguous(self, buf):
        return isinstance(buf, np.ndarray) and buf.dtype == np.float64 and buf.flags["C_CONTIGUOUS"]

    def _host_state(self, host_state, keep):
        """aie_host_state over the numpy arrays of host_state (kept alive in `keep`)."""
        def arr(key, dt, required=True):
            v = host_state.get(key)
            if v is None:
                assert not required, key
                return None
            a = np.ascontiguousarray(v, dtype=dt)
            keep.append(a)
            return a.ctypes.data_as(C.c_void_p)

        hs = _abi.AieHostState()
        hs.n = int(np.asarray(host_state["loc"]).shape[0])
        for key, dt, req in [("stone", np.uint8, True), ("wood", np.uint8, True), ("stone_src", np.uint8, True),
                             ("wood_src", np.uint8, True), ("water", np.uint8, False), ("loc", np.int16, True),
                             ("coin", np.float64, True), ("inv_stone", np.int32, False), ("inv_wood", np.int32, False),
                             ("build_payment", np.float64, True), ("build_skill", np.float64, True),
                             ("bonus_gather_prob", np.float64, True), ("mt_key", np.uint32, True),
                             ("mt_pos", np.int32, True), ("completions", np.int32, False),
                             ("gauss_has", np.int32, False), ("gauss_val", np.float64, False),
                             ("split_skill", np.float64, False)]:
            setattr(hs, key, arr(key, dt, req))
        return hs

    def load_state(self, host_state, env_lo=0):
        """host_state: dict of numpy arrays with a leading env axis (see aie_host_state in the header)."""
        keep = []
        hs = self._host_state(host_state, keep)
        self._check(self.lib.aie_load_state(self._h, C.byref(hs), int(env_lo), self._stream()))

    def reset_envs(self, template=None, streams=None, env_lo=0, n=None):
        """Explicit reset of replicas [env_lo, env_lo + n) on the device (aie_reset_envs; configs with reset_mode == 1):
        the records come out as load_state leaves them for the host reset of the same streams.  template: None (each
        replica restarts from its own state0) or a host reset snapshot of ONE replica (load_state's dict, leading axis 1).
        streams: None (each record's stream continues) or a dict of numpy arrays with a leading axis n: mt_key, mt_pos
        and, where the config needs them, gauss_has / gauss_val, split_skill.  Asynchronous on the stream when neither is
        given."""
        n = self.n_envs - int(env_lo) if n is None else int(n)
        keep = []
        tmpl = C.byref(self._host_state(template, keep)) if template is not None else None
        rs = None
        if streams is not None:
            s = _abi.AieResetStreams()
            for key, dt in [("mt_key", np.uint32), ("mt_pos", np.int32), ("gauss_has", np.int32), ("gauss_val", np.float64),
                            ("split_skill", np.float64)]:
                if streams.get(key) is not None:
                    a = np.ascontiguousarray(streams[key], dtype=dt)
                    keep.append(a)
                    setattr(s, key, a.ctypes.data_as(C.c_void_p))
            rs = C.byref(s)
        self._check(self.lib.aie_reset_envs(self._h, tmpl, rs, int(env_lo), n, self._stream()))

    def step(self):
        """Advance every env by one timestep from the bound action buffers (asynchronous on the stream); with final_obs,
        then write the final observations of the episodes that ended into the final_<name> buffers.  With a rollout
        bound: from the actions of slot s into slot s (rewards, done) and s + 1 (observations), the final observations
        into the rollout's final slots, then s advances."""
        self._check(self.lib.aie_step(self._h, self._stream()))
        if self.rollout is not None:
            self.rollout_slot += 1
        elif self.final_obs:
            self.observe_final()

    # -- rollouts stored in place (aie_bind_rollout) ---------------------------------------------------------------
    def bind_rollout(self, T, final_obs=False):
        """Allocate and bind a rollout of T steps (a Rollout), with final slots [K, E, ...] when final_obs."""
        if isinstance(T, bool) or not isinstance(T, numbers.Integral) or T < 1:
            raise ValueError("T must be a positive int")
        if self.rollout is not None:
            raise ValueError("a rollout is already bound: unbind_rollout() first")
        T = int(T)
        K = -(-T // int(self.spec["episode_length"]))
        sh = self._shapes
        names = [k for k in _abi.OBS_NAMES if k in sh]
        buf = {k: self._alloc((T + 1,) + sh[k][1], sh[k][0]) for k in names}
        for k in ("actions_agent", "actions_planner", "reward", "done"):
            buf[k] = self._alloc((T,) + sh[k][1], sh[k][0])
        if final_obs:
            buf.update({"final_" + k: self._alloc((K,) + sh[k][1], sh[k][0]) for k in names})
        r = _abi.AieRollout()
        r.T = T
        r.obs = self._obs_buffers({k: buf[k] for k in names})
        if final_obs:
            r.final_obs = self._obs_buffers({k: buf["final_" + k] for k in names})
        r.actions_agent, r.reward, r.done = self._ptr(buf["actions_agent"]), self._ptr(buf["reward"]), self._ptr(buf["done"])
        r.actions_planner = self._ptr(buf["actions_planner"]) if self.dims.n_act_planner else None
        self._check(self.lib.aie_bind_rollout(self._h, C.byref(r)))
        self.rollout, self.rollout_slot = Rollout(T, K, buf, names, bool(final_obs)), 0
        return self.rollout

    def restart_rollout(self):
        """Next rollout: the observations of slot T move to slot 0 (one device copy per tensor), s = 0."""
        self._check(self.lib.aie_rollout_restart(self._h, self._stream()))
        self.rollout_slot = 0

    def unbind_rollout(self):
        self._check(self.lib.aie_bind_rollout(self._h, None))
        self.rollout, self.rollout_slot = None, 0

    def observe(self):
        self._check(self.lib.aie_observe(self._h, self._stream()))

    def observe_final(self, out=None):
        """Observations / masks of the state each episode that ended in the latest step ended in (its episode_final
        record), into row e of every replica e whose done flag is set; other rows are left as they are (aie_observe_final,
        one launch, asynchronous on the stream; needs auto_reset).  out: None (the final_<name> buffers) or a dict
        name -> buffer for every observation / mask buffer of the stepper (same shape and dtype, contiguous), e.g. a
        trainer's rollout slot.  Returns the dict written to."""
        if out is None:
            if not self.final_obs:
                raise _abi.AieError("observe_final: no final_<name> buffers (final_obs is off); pass out=")
            out, o = self._final_out, self._final_bufs
        else:
            for k in _abi.OBS_NAMES:
                if k not in self.buf:
                    continue
                if k not in out:
                    raise _abi.AieError("observe_final: out has no %s buffer" % k)
                if not self._same_layout(out[k], self.buf[k]):
                    raise _abi.AieError("observe_final: out[%r] must be a contiguous %s %s buffer on the stepper's device"
                                        % (k, self.buf[k].dtype, tuple(self.buf[k].shape)))
            o = self._obs_buffers(out)
        self._check(self.lib.aie_observe_final(self._h, C.byref(o), self._stream()))
        return out

    def _obs_buffers(self, out):
        """aie_obs_buffers over the buffers of `out` (zero-size tensors have no storage: NULL)."""
        o = _abi.AieObsBuffers()
        for k in _abi.OBS_NAMES:
            if k in self.buf and int(np.prod(self.buf[k].shape)) > 0:
                setattr(o, k, self._ptr(out[k]))
        return o

    def _same_layout(self, buf, like):
        return (isinstance(buf, np.ndarray) and buf.dtype == like.dtype and buf.shape == like.shape
                and buf.flags["C_CONTIGUOUS"])

    def step_dynamics(self):
        self._check(self.lib.aie_step_dynamics(self._h, self._stream()))

    def sample_random_actions(self, seed=0):
        """Device-side random policy: one uniformly random unmasked action per agent/subspace."""
        self._check(self.lib.aie_sample_random_actions(self._h, C.c_uint64(int(seed)), self._stream()))

    def set_fused_policy(self, seed):
        """seed != 0: every following step() also draws the NEXT step's uniformly random unmasked actions into the action
        buffers inside the observation pass (no sampler launch per step); 0 turns it off (aie_set_fused_policy)."""
        self._check(self.lib.aie_set_fused_policy(self._h, C.c_uint64(int(seed)), self._stream()))

    @property
    def _policy_fn(self):
        return self.lib.aie_sample_policy

    @property
    def _eval_fns(self):
        return self.lib.aie_evaluate_policy, self.lib.aie_evaluate_policy_backward

    @property
    def _adv_fn(self):
        return self.lib.aie_compute_advantages

    @property
    def _adv_k_fn(self):
        return self.lib.aie_compute_advantages_k

    def _policy_shapes(self):
        d, E, A = self.dims, self.n_envs, self.spec["n_agents"]
        has_p = d.n_act_planner > 0
        return ((E, A, d.mask_agent), (E, d.mask_planner) if has_p else None, (E, A, d.n_act_agent),
                (E, d.n_act_planner) if has_p else None)

    def step_host(self, actions_agent, actions_planner, out_ptrs, compact=False, n_threads=0):
        """End-to-end step with HOST buffers (aie_step_host).  out_ptrs: dict name -> host pointer / None.
        compact=True: same bytes in the host tensors, bit- / byte-packed over PCIe (aie_step_host_compact)."""
        o = _abi.AieHostOut()
        for name in _abi._OUT_NAMES:
            setattr(o, name, out_ptrs.get(name))
        if compact:
            self._check(self.lib.aie_step_host_compact(self._h, actions_agent, actions_planner, C.byref(o),
                                                       int(n_threads), self._stream()))
        else:
            self._check(self.lib.aie_step_host(self._h, actions_agent, actions_planner, C.byref(o), self._stream()))

    def host_timing(self):
        """Host-clock breakdown (ms) of the last compacted step_host call (aie_get_host_timing)."""
        out = (C.c_double * 16)()
        self.lib.aie_get_host_timing(self._h, out, 16)
        k = ["enqueued", "first_slice", "last_slice", "expanded", "slices", "threads", "d2h_bytes", "before_transfer",
             "wait_sum", "busy_sum", "first_slice_dev", "last_slice_dev", "expand_only", "overflow_envs", "chunks", "staging_node"]
        return dict(zip(k, list(out)))

    def compact_bytes_per_env(self):
        return int(self.lib.aie_compact_bytes_per_env(self._h))

    def launch_count(self):
        return int(self.lib.aie_launch_count(self._h))

    def get_counters(self):
        """The library's host-side counters of this handle (aie_get_counters) as a dict of ints."""
        c = _abi.AieCounters()
        self._check(self.lib.aie_get_counters(self._h, C.byref(c)))
        return {k: int(getattr(c, k)) for k, _ in _abi.AieCounters._fields_ if k != "reserved"}

    def set_counters(self, counters):
        """Write the counters of get_counters() back (aie_set_counters); marks the records as loaded."""
        c = _abi.AieCounters(**{k: int(v) for k, v in counters.items()})
        self._check(self.lib.aie_set_counters(self._h, C.byref(c)))

    def field(self, name):
        if name not in self._fields:
            f = _abi.AieField()
            self._check(self.lib.aie_get_field(self._h, name.encode(), C.byref(f)))
            self._fields[name] = f
        return self._fields[name]

    def read_state(self, e, final=False):
        """Readback of env e in the test oracle's layout (dict of numpy arrays + 'books').  final=True reads the
        end-of-episode snapshot of the env's last finished episode instead (auto-reset only; no order books)."""
        A, H, W = self.spec["n_agents"], self.spec["height"], self.spec["width"]
        P = self.spec["max_bid_ask"] + 1 if "ContinuousDoubleAuction" in self.spec["components"] else 1
        B = max(1, self.spec["n_brackets"])
        cap = A * max(1, self.spec["max_num_orders"])
        out = dict(
            cell=np.zeros((H, W), np.uint8), owner=np.zeros((H, W), np.int8), loc=np.zeros((A, 2), np.int16),
            coin=np.zeros(A), esc_coin=np.zeros(A), labor=np.zeros(A),
            inv=np.zeros((A, 2), np.int32), esc=np.zeros((A, 2), np.int32),
            n_orders=np.zeros((2, A), np.int32), bid_hist=np.zeros((2, A, P), np.int32),
            ask_hist=np.zeros((2, A, P), np.int32), price_hist=np.zeros((2, A, P)),
            tax_pos=np.zeros(1, np.int32), rate_idx=np.zeros(B, np.int32),
            last_coin=np.zeros(A), last_income=np.zeros(A), last_marg=np.zeros(A),
            mt_key=np.zeros(624, np.uint32), mt_pos=np.zeros(1, np.int32), t=np.zeros(1, np.int32),
            completions=np.zeros(1, np.int32),
            book_rows=np.zeros((2, 2, cap, 3), np.int32), book_count=np.zeros((2, 2), np.int32),
            stats=np.zeros(self.dims.n_stats), util_prev=np.zeros(A + 1), auto_warmup=np.zeros(1, np.int32),
        )
        d = _abi.AieStateDump()
        for k in _abi._DUMP_PTRS + _abi._DUMP_PTRS2:
            setattr(d, k, out[k].ctypes.data_as(C.c_void_p))
        d.book_cap = cap
        fn = self.lib.aie_read_episode_final if final else self.lib.aie_read_state
        self._check(fn(self._h, int(e), C.byref(d)))
        out["books"] = {(c, s): out["book_rows"][c, s, :out["book_count"][c, s]].copy()
                        for c in (0, 1) for s in (0, 1)}
        if hasattr(self, "state_view"):   # skills / payments (one-step-economy: SimpleLabor skill / cumulative production)
            for k in ("build_payment", "build_skill"):
                out[k] = np.asarray(self.to_numpy(self.state_view(k, final=final)[e]), np.float64).copy()
        return out

    def read_events(self, e):
        """Events of replica e's last step (dense logs): list of int rows [kind, ...] (include/aie_b200.h)."""
        blk = self.to_numpy(self.buf["events"][e])
        n, dropped = int(blk[0, 0]), int(blk[0, 2])
        if dropped:
            raise _abi.AieError("event log overflow: %d events dropped (capacity %d)" % (dropped, self.event_cap))
        return [tuple(int(v) for v in blk[1 + i]) for i in range(n)]

    def obs_to_numpy(self, name, e=None):
        """Host copy of output buffer `name` (of env e), bfloat16 observations upcast to float32 (exact)."""
        a = self.to_numpy(self.buf[name] if e is None else self.buf[name][e])
        return bf16_bits_to_float32(a) if name in self._bf16 and np.asarray(a).dtype == np.uint16 else a

    def read_obs(self, e):
        """Host copy of env e's outputs in the oracle's obs layout (tests); float observations as float32."""
        g = lambda k: self.obs_to_numpy(k, e) if k in self.buf else None
        out = dict(a_map=g("obs_agent_map"), a_idx=g("obs_agent_idx"), a_flat=g("obs_agent_flat"),
                   a_mask=g("mask_agent"), p_flat=g("obs_planner_flat"), p_agents=g("obs_planner_agents"),
                   p_mask=g("mask_planner"), time=np.atleast_1d(g("obs_time")), rew=g("reward"),
                   done=np.atleast_1d(g("done")))
        if "obs_planner_map" in self.buf:
            out["p_map"], out["p_idx"] = g("obs_planner_map"), g("obs_planner_idx")
        return out


class CudaStepper(BatchStepper):
    """The product path: torch-owned CUDA tensors, kernels launched on torch's current stream."""

    _TORCH = None
    supports_rollout_capture = True

    def __init__(self, spec, n_envs, device="cuda:0", auto_reset=True, lib_path=None, event_envs=0):
        import torch

        if not torch.cuda.is_available():
            raise _abi.AieError("no CUDA device visible: ai_economist_b200 has no CPU fallback")
        self.torch = torch
        self.device = torch.device(device)
        if self.device.type != "cuda":
            raise _abi.AieError("device must be a CUDA device, got %s" % device)
        idx = self.device.index if self.device.index is not None else torch.cuda.current_device()
        self.device = torch.device("cuda", idx)
        lib = _abi.load_library(lib_path)
        with torch.cuda.device(self.device):
            super().__init__(spec, n_envs, lib, device_index=idx, auto_reset=auto_reset, event_envs=event_envs)

    def _torch_dtype(self, dt):
        t = self.torch
        return {"u8": t.uint8, "i16": t.int16, "i32": t.int32, "f32": t.float32, "f64": t.float64, "bf16": t.bfloat16}[dt]

    def _alloc(self, shape, dt):
        return self.torch.zeros(shape, dtype=self._torch_dtype(dt), device=self.device)

    def _empty(self, shape, dt):
        return self.torch.empty(shape, dtype=self._torch_dtype(dt), device=self.device)

    def _is_f64_contiguous(self, buf):
        t = self.torch
        return isinstance(buf, t.Tensor) and buf.dtype == t.float64 and buf.is_contiguous() and buf.device == self.device

    def _same_layout(self, buf, like):
        t = self.torch
        return (isinstance(buf, t.Tensor) and buf.dtype == like.dtype and buf.shape == like.shape and buf.is_contiguous()
                and buf.device == self.device)

    def _is_i32(self, buf):
        return is_i32_torch(self.torch, self.device, buf)

    def _float_kind(self, buf):
        return float_kind_torch(self.torch, self.device, buf)

    def _eval_out(self, shape, kind):
        return self._empty(shape, kind)

    def _buf_kind(self, buf):
        return buf_kind_torch(self.torch, self.device, buf)

    def _ptr(self, buf):
        return C.c_void_p(buf.data_ptr())

    def _stream(self):
        return C.c_void_p(self.torch.cuda.current_stream(self.device).cuda_stream)

    def to_numpy(self, buf):
        if buf.dtype == self.torch.bfloat16:   # numpy has no bfloat16: float32 holds every value exactly
            buf = buf.float()
        return buf.detach().cpu().numpy()

    def state_view(self, name, final=False):
        """Strided struct-of-arrays view [E, ...] of one state field inside the packed records (final=True: inside the
        end-of-episode snapshots of the last finished episode, auto-reset only)."""
        t = self.torch
        f = self.field(name)
        shape = [f.shape[i] for i in range(f.ndim)]
        n = int(np.prod(shape)) if shape else 1
        dt = {(1, 0, 0): t.uint8, (1, 0, 1): t.int8, (2, 0, 1): t.int16, (4, 0, 1): t.int32, (4, 0, 0): t.int32,
              (8, 1, 1): t.float64}[(f.elem_bytes, f.is_float, f.is_signed)]
        raw = self.buf["episode_final" if final else "state"][:, f.offset:f.offset + n * f.elem_bytes]
        return raw.view(dt).view([self.n_envs] + shape) if shape else raw.view(dt)[:, 0]
