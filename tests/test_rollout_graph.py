"""A bound rollout recorded once as a CUDA graph and replayed: `env.capture_rollout(act)` / `RolloutGraph.replay()`
(aie_rollout_capture_begin / _end, aie_rollout_replay_begin / _end and their COVID-19 twins).

Contract: from the same state, a replay leaves every output the eager loop `for t: act(t, slot t); env.step(...)` leaves,
byte for byte (slots, final slots, rewards, done, log-probabilities, rate observations, records, metric accumulators,
counters, state_dict()), wherever the rollout's episode ends fall, with eager rollouts run between replays.

The CPU tests run the host emulation of the device source (tests/emu): there a capture executes as it goes, so the
capture pair followed by an empty replay pair is one eager rollout run through the capturable variants (the
device-counter policy sampler, the COVID-19 step that finds its final row on the device) and the replay's host
bookkeeping; its bytes must be the eager loop's.  The `-m gpu` tests record and replay real CUDA graphs.
"""
import numpy as np
import pytest
import torch

from ai_economist_b200 import _abi
from ai_economist_b200.stepper import bf16_bits_to_float32
from tests.emu.emu_stepper import emu_lib
from tests.test_checkpoint import _cfg, _covid, _make_gtb, _np, _same

AIE_EINVAL, AIE_ESTATE = -1, -3   # include/aie_b200.h
RATE = "VaccinationCampaign-next_vaccination_rate"


# ------------------------------------------------------------------------------------------------ helpers
def _on(env, a):
    buf = env.stepper.buf["done"]
    return a if isinstance(buf, np.ndarray) else torch.as_tensor(a, device=buf.device)


class Heads:
    """A deterministic stand-in for a policy: logits from each slot's observations by element-wise torch ops and fixed
    reductions (no library whose algorithm may change between an eager call and a captured one), log-probabilities into
    per-slot rows of the caller's buffers.  On the emulation the torch ops run on the CPU over the numpy buffers."""

    def __init__(self, env, T, seed=4242, covid=False):
        sa, sp, na, npl = env.stepper._policy_shapes()
        self.covid, self.seed, self.env = covid, seed, env
        self.host = isinstance(env.stepper.buf["done"], np.ndarray)
        dev = "cpu" if self.host else env.stepper.buf["done"].device
        g = np.random.RandomState(11)
        w = lambda n: torch.as_tensor(g.standard_normal(n).astype(np.float32), device=dev)
        self.wa, self.ba = w(sa[-1]), w(sa[-1])
        self.wp, self.bp = (w(sp[-1]), w(sp[-1])) if sp is not None else (None, None)
        z = lambda sh: _on(env, np.zeros((T,) + sh, np.float32))
        self.lp_a, self.lp_p = z(na), (z(npl) if npl is not None else None)

    def _f32(self, x):
        if not self.host:
            return x.float()
        return torch.from_numpy(bf16_bits_to_float32(x) if x.dtype == np.uint16 else x.astype(np.float32))

    def logits(self, obs):
        if self.covid:
            xa = self._f32(obs["obs_agent_state"]).sum(1)                   # [E, S]
            xp = self._f32(obs["obs_scalars"]).sum(1, keepdim=True)         # [E, 1]
        else:
            xa = self._f32(obs["obs_agent_flat"]).sum(-1)                   # [E, A]
            xp = self._f32(obs["obs_planner_flat"]).sum(-1, keepdim=True)   # [E, 1]
        la = (torch.tanh(xa[..., None] * 1e-3 * self.wa + self.ba) * 3.0).contiguous()
        lp = (torch.tanh(xp * 1e-3 * self.wp + self.bp) * 3.0).contiguous() if self.wp is not None else None
        if self.host:
            return la.numpy(), (lp.numpy() if lp is not None else None)
        return la, lp

    def __call__(self, t, obs):
        la, lp = self.logits(obs)
        self.env.sample_actions(la, lp, seed=self.seed,
                                out=(self.lp_a[t], self.lp_p[t] if self.lp_p is not None else None))


def _bufs(env):
    """Every buffer a rollout leaves: the stepper's own and the rollout's."""
    out = {"st_" + k: v for k, v in env.stepper.buf.items()}
    out.update({"ro_" + k: v for k, v in env.rollout.buf.items()})
    return out


def compare(A, B, ha, hb, label):
    ba, bb = _bufs(A), _bufs(B)
    assert set(ba) == set(bb)
    for k in ba:
        _same(ba[k], bb[k], "%s: %s" % (label, k))
    _same(ha.lp_a, hb.lp_a, "%s: log_prob_agent" % label)
    if ha.lp_p is not None:
        _same(ha.lp_p, hb.lp_p, "%s: log_prob_planner" % label)
    assert A.stepper.rollout_slot == B.stepper.rollout_slot, label
    if hasattr(A, "_rate_tab") and A._rate_tab is not None:
        for g in ("a", "p"):
            _same(A.obs[g][RATE], B.obs[g][RATE], "%s: rate %s" % (label, g))
    covid = hasattr(A, "_rate_tab")
    if not covid or A._episode_metrics:
        _same(A.metrics_tensor(), B.metrics_tensor(), "%s: metrics_tensor" % label)
        if A.stepper.has_previous_episode() if covid else "episode_final" in A.stepper.buf:
            _same(A.previous_episode_metrics_tensor(), B.previous_episode_metrics_tensor(), "%s: previous" % label)


def compare_at_slot0(A, B, label):
    """Counters and state_dict(), read at slot 0 (after restart_rollout)."""
    assert A.stepper.get_counters() == B.stepper.get_counters(), label
    sa, sb = A.state_dict(), B.state_dict()
    assert sa["counters"] == sb["counters"], label
    assert set(sa["buffers"]) == set(sb["buffers"]), label
    for k in sa["buffers"]:
        _same(sa["buffers"][k], sb["buffers"][k], "%s: state_dict %s" % (label, k))


def eager(env, heads, T):
    for t in range(T):
        heads(t, env.rollout.obs_slots[t])
        env.step(env.action_buffers)


def emulated_capture_and_replay(env, heads, T):
    """The capture pair executes on the emulation: capture (T steps through the capturable variants), which leaves the
    host state as it was, then an (empty) replay pair applies what the capture recorded."""
    st = env.stepper
    c0 = st.get_counters()
    st.rollout_capture_begin()
    try:
        eager(env, heads, T)
        with pytest.raises(ValueError, match="being captured"):   # only the step and the policy sampler run
            st.sample_random_actions(seed=3)
    finally:
        st.rollout_capture_end()
    env._aim_rollout()
    assert st.rollout_slot == 0 and st.get_counters() == c0
    st.rollout_replay_begin()
    st.rollout_replay_end()
    env._aim_rollout()
    assert st.rollout_slot == T


def run_twins(A, B, T, rounds, covid, mode, label, interleave=(2,)):
    """A runs the eager loop every round; B the capture (mode "emu": the emulated pair; "gpu": capture_rollout once, at
    the start of the first round not in `interleave`, then replay()), except in the rounds `interleave`, where it runs
    the eager loop too.  Returns the ends seen."""
    for env in (A, B):
        env.bind_rollout(T, final_obs=True)
        env.reset()
    ha, hb = Heads(A, T, covid=covid), Heads(B, T, covid=covid)
    graph, ends = None, set()
    for rnd in range(rounds):
        if rnd:
            for env in (A, B):
                env.restart_rollout()
            compare_at_slot0(A, B, "%s round %d: at slot 0" % (label, rnd))
        if mode == "gpu" and graph is None and rnd not in interleave:
            la, lp = hb.logits(B.rollout.obs_slots[0])   # the policy gives the same logits eagerly and under capture
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                cla, clp = hb.logits(B.rollout.obs_slots[0])
            g.replay()
            _same(la, cla, "policy logits under capture")
            if lp is not None:
                _same(lp, clp, "policy planner logits under capture")
            graph = B.capture_rollout(hb)
            assert B.stepper.rollout_slot == 0
            compare_at_slot0(A, B, "%s: after capture" % label)
        eager(A, ha, T)
        if rnd in interleave:
            eager(B, hb, T)
        elif mode == "emu":
            emulated_capture_and_replay(B, hb, T)
        else:
            graph.replay()
        compare(A, B, ha, hb, "%s round %d" % (label, rnd))
        d = _np(A.rollout.buf["done"])
        ends.update(int(t) for t in np.nonzero(d.any(1))[0])
    for env in (A, B):
        env.restart_rollout()
    compare_at_slot0(A, B, "%s: end" % label)
    return ends


# ------------------------------------------------------------------------------------------------ CPU: emulation
@pytest.mark.parametrize("obs_dtype", [None, torch.bfloat16])
def test_emulated_capture_gtb_matches_eager(obs_dtype):
    """Episode length 10, T = 7: over seven rounds the ends fall on every slot."""
    name, kw = _cfg("c1_tutorial", episode_length=10)
    A, B = (_make_gtb(name, kw, 3, 1000, final_obs=True, obs_dtype=obs_dtype) for _ in range(2))
    ends = run_twins(A, B, 7, 10, False, "emu", "gtb", interleave=(3,))
    assert ends == set(range(7))


def test_emulated_capture_gtb_multi_action_and_tax():
    name, kw = _cfg("tax_us_federal", episode_length=6)
    A, B = (_make_gtb(name, kw, 2, 1000, final_obs=True) for _ in range(2))
    assert run_twins(A, B, 4, 4, False, "emu", "tax_us_federal", interleave=(1,))


@pytest.mark.parametrize("obs_dtype", [None, torch.bfloat16])
def test_emulated_capture_covid_matches_eager(obs_dtype):
    """Episode length 12, T = 5: the ends fall on slots 1, 3, 0, 2, 4 of rounds 2, 4, 7, 9, 11 (round 5, eager on both
    twins, has none)."""
    A, B = (_covid(3, 1, episode_length=12, episode_metrics=True, final_obs=True, obs_dtype=obs_dtype)
            for _ in range(2))
    ends = run_twins(A, B, 5, 12, True, "emu", "covid", interleave=(5,))
    assert ends == set(range(5))


def _emu_gtb_handle():
    name, kw = _cfg("c1_tutorial", episode_length=10)
    return _make_gtb(name, kw, 2, 1000, final_obs=True)


def test_abi_errors():
    """Wrong slot, no capture, nothing bound, double begin; null handles; calls refused inside the pair."""
    L = emu_lib()
    for env, pre in ((_emu_gtb_handle(), "aie"), (_covid(2, 1, final_obs=True), "aie_covid")):
        st = env.stepper
        h = st._h
        f = lambda n: getattr(L, "%s_rollout_%s" % (pre, n))
        for n in ("capture_begin", "replay_begin"):
            assert f(n)(None, None) == AIE_EINVAL
        for n in ("capture_end", "replay_end"):
            assert f(n)(None) == AIE_EINVAL
        env.reset()
        assert f("capture_begin")(h, None) == AIE_ESTATE and b"no rollout bound" in L.aie_last_error()
        env.bind_rollout(3, final_obs=True)
        env.reset()
        assert f("capture_end")(h) == AIE_ESTATE and b"no capture in progress" in L.aie_last_error()
        assert f("replay_begin")(h, None) == AIE_ESTATE and b"nothing captured" in L.aie_last_error()
        assert f("replay_end")(h) == AIE_ESTATE
        env.step(env.action_buffers)
        assert f("capture_begin")(h, None) == AIE_ESTATE and b"slot 0" in L.aie_last_error()
        env.step(env.action_buffers)
        env.step(env.action_buffers)
        env.restart_rollout()
        assert f("capture_begin")(h, None) == 0
        assert f("capture_begin")(h, None) == AIE_ESTATE and b"already in progress" in L.aie_last_error()
        rs = L.aie_rollout_restart if pre == "aie" else L.aie_covid_rollout_restart
        assert rs(h, None) == AIE_ESTATE and b"being captured" in L.aie_last_error()
        assert f("replay_begin")(h, None) == AIE_ESTATE and b"in progress" in L.aie_last_error()
        assert f("capture_end")(h) == 0
        assert f("replay_begin")(h, None) == 0 and f("replay_end")(h) == 0
        env.step(env.action_buffers)
        assert f("replay_begin")(h, None) == AIE_ESTATE and b"slot 0" in L.aie_last_error()
        env.unbind_rollout()   # unbinding drops the capture
        env.bind_rollout(3, final_obs=True)
        assert f("replay_begin")(h, None) == AIE_ESTATE and b"nothing captured" in L.aie_last_error()


def test_python_refusals_on_cpu():
    """capture_rollout without the CUDA stepper, under the Saez tax model and through the reference API; the emulated
    pair refuses the random sampler with ValueError."""
    env = _emu_gtb_handle()
    env.bind_rollout(3, final_obs=True)
    env.reset()
    with pytest.raises(NotImplementedError, match="cannot capture"):
        env.capture_rollout(lambda t, o: None)
    cv = _covid(2, 1, final_obs=True)
    cv.bind_rollout(3, final_obs=True)
    cv.reset()
    with pytest.raises(NotImplementedError, match="cannot capture"):
        cv.capture_rollout(lambda t, o: None)
    name, kw = _cfg("saez_reset", episode_length=10)
    sz = _make_gtb(name, kw, 2, 1000)
    with pytest.raises(ValueError, match="Saez"):
        sz.capture_rollout(lambda t, o: None)
    from ai_economist_b200.adapters import ReferenceApiEnv
    with pytest.raises(ValueError, match="reference API"):
        ReferenceApiEnv(env).capture_rollout(lambda t, o: None)
    st = env.stepper
    st.rollout_capture_begin()
    try:
        for call in (lambda: st.sample_random_actions(seed=1), lambda: st.observe(), lambda: st.get_counters()):
            with pytest.raises(ValueError, match="being captured"):
                call()
    finally:
        st.rollout_capture_end()
    env.step(env.action_buffers)   # the env works on after the pair


# ------------------------------------------------------------------------------------------------ GPU: real graphs
GPU_GTB = {
    # (config, overrides, n_envs, T, rounds); episode length 10 and T = 7: the ends move over the slots
    "c1": ("c1_tutorial", dict(episode_length=10), 37, 7, 7),
    "c3_tax": ("c3_short_period", dict(episode_length=10), 19, 7, 6),
    "multi_action": ("tax_us_federal", dict(episode_length=10), 23, 7, 6),
    "c5_small": ("c5_small", dict(episode_length=10), 13, 7, 5),
    "c2_workload": ("c1_tutorial", dict(episode_length=10), 8192, 7, 5),
}


@pytest.mark.gpu
@pytest.mark.parametrize("case", sorted(GPU_GTB))
def test_gpu_replay_matches_eager_gtb(case):
    cfg, over, E, T, rounds = GPU_GTB[case]
    name, kw = _cfg(cfg, **over)
    A, B = (_make_gtb(name, kw, E, 1000, cuda=True, final_obs=True) for _ in range(2))
    ends = run_twins(A, B, T, rounds, False, "gpu", case, interleave=(3,))
    assert len(ends) >= 3


GPU_COVID = {
    # (n_envs, obs_dtype, episode length, T, rounds, eager rounds of B); episode length 60, T = 16: the ends fall on
    # slots 11 and 7 of rounds 3 and 7.  Episode length 7, T = 10 (K = 2), captured in round 1, mid-episode: later
    # rollouts end on slots whose count of earlier ends differs from the captured rollout's (round 3: slot 4, first end)
    "f32_odd": (37, None, 60, 16, 8, (5,)),
    "bf16_odd": (53, torch.bfloat16, 60, 16, 8, (5,)),
    "c4_workload": (4096, None, 60, 16, 8, (5,)),
    "f32_two_final_rows": (29, None, 7, 10, 8, (0, 5)),
}


@pytest.mark.gpu
@pytest.mark.parametrize("case", sorted(GPU_COVID))
def test_gpu_replay_matches_eager_covid(case):
    E, obs_dtype, L, T, rounds, interleave = GPU_COVID[case]
    A, B = (_covid(E, 1, cuda=True, episode_length=L, episode_metrics=True, final_obs=True, obs_dtype=obs_dtype)
            for _ in range(2))
    ends = run_twins(A, B, T, rounds, True, "gpu", case, interleave=interleave)
    assert len(ends) >= 2


@pytest.mark.gpu
def test_gpu_foreign_capture_is_refused():
    """A plain torch.cuda.graph around the eager loop raises instead of recording; the env works on eagerly after."""
    name, kw = _cfg("c1_tutorial", episode_length=10)
    for env in (_make_gtb(name, kw, 5, 1000, cuda=True, final_obs=True),
                _covid(5, 1, cuda=True, episode_length=12, final_obs=True)):
        r = env.bind_rollout(3, final_obs=True)
        env.reset()
        h = Heads(env, 3, covid=not hasattr(env, "_saez"))
        for body in (lambda: h(0, r.obs_slots[0]), lambda: env.step(env.action_buffers)):
            g = torch.cuda.CUDAGraph()
            with pytest.raises(_abi.AieError, match="being captured into a CUDA graph"):
                with torch.cuda.graph(g):
                    body()
        assert env.stepper.rollout_slot == 0
        eager(env, h, 3)
        assert env.stepper.rollout_slot == 3


@pytest.mark.gpu
def test_gpu_refusals_and_invalidation():
    name, kw = _cfg("c1_tutorial", episode_length=10)
    env = _make_gtb(name, kw, 5, 1000, cuda=True, final_obs=True)
    env.bind_rollout(3, final_obs=True)
    env.reset()
    h = Heads(env, 3)
    refused = {
        "step": lambda: env.step(env.action_buffers), "reset": lambda: env.reset(),
        "evaluate_actions": lambda: env.evaluate_actions(*h.logits(env.rollout.obs_slots[0]), env.action_buffers,
                                                         (env.obs_tensors["mask_agent"], env.obs_tensors["mask_planner"])),
        "metrics": lambda: env.metrics_tensor(), "state_dict": lambda: env.state_dict(),
        "random sampler": lambda: env.stepper.sample_random_actions(seed=1),
    }
    c0 = env.stepper.get_counters()
    for what, call in refused.items():
        def act(t, obs, call=call):
            h(t, obs)
            call()
        with pytest.raises(ValueError):
            env.capture_rollout(act)
        assert env.stepper.rollout_slot == 0 and env.stepper.get_counters() == c0, what
    g = env.capture_rollout(h)
    g.replay()
    with pytest.raises(ValueError, match="slot 0"):
        g.replay()
    env.restart_rollout()
    sd = env.state_dict()
    env.load_state_dict(sd)
    with pytest.raises(ValueError, match="no longer matches"):
        g.replay()
    g = env.capture_rollout(h)
    env.unbind_rollout()
    env.bind_rollout(3, final_obs=True)
    with pytest.raises(ValueError, match="no longer matches"):
        g.replay()
    g = env.capture_rollout(h)
    env.step(env.action_buffers)
    with pytest.raises(_abi.AieError):
        env.reset()   # mid-rollout: refused, and the graph with it
    with pytest.raises(ValueError, match="no longer matches"):
        g.replay()
