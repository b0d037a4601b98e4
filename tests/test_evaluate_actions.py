"""Evaluation of stored actions (env.evaluate_actions / aie_evaluate_policy / aie_covid_evaluate_policy and their
backward): log-probabilities, entropies and their gradient with respect to the logits, per mask segment, under the
masks the actions were drawn with.

The restatement below is the contract of include/aie_b200.h in float64 torch: the masked log-softmax, its entropy and
their autograd gradients, with the edge cases (nothing open, a NaN / +inf open logit or no finite one, a closed or
out-of-range action) spelled out.  Log-probabilities and entropies must lie within one float32 ulp of it (1e-12
absolute near 0), gradients within one ulp of their dtype plus 1e-12 times the upstream magnitudes; closed entries
get exactly 0.  Log-probabilities must also equal the sampler's bit for bit."""
import ctypes as C

import numpy as np
import pytest
import torch

from ai_economist_b200 import _abi
from tests.test_policy_sampler import (EXACT_CFGS, as_f32, covid_env, covid_shapes, emu_covid, emu_env, gtb_kwargs,
                                       gtb_segments, logit_shapes, random_logits, to_bf16_bits)

AIE_EINVAL = -1


# ---------------------------------------------------------------------------------------------- float64 restatement
def ref_segment(open_, logits, a):
    """(lp, H, d lp / d logits, d H / d logits) of one segment in float64 under the contract (numpy)."""
    o = np.asarray(open_, bool)
    l = np.asarray(logits, np.float32).astype(np.float64)
    n = len(l)
    zero = np.zeros(n)
    if not o.any():
        return 0.0, 0.0, zero, zero
    lo = l[o]
    if np.isnan(lo).any() or (lo == np.inf).any() or not np.isfinite(lo).any():
        nan = np.where(o, np.nan, 0.0)
        return float("nan"), float("nan"), nan, nan
    x = torch.tensor(np.where(o, l, 0.0), dtype=torch.float64, requires_grad=True)
    logp = torch.log_softmax(x.masked_fill(~torch.as_tensor(o), float("-inf")), 0)
    p = logp.exp()
    H = -(p * torch.where(p > 0, logp, torch.zeros_like(logp))).sum()
    g_h = torch.autograd.grad(H, x, retain_graph=True)[0].numpy()
    if not (0 <= a < n and o[a]):
        return float("nan"), float(H), np.where(o, np.nan, 0.0), g_h
    g_lp = torch.autograd.grad(logp[a], x)[0].numpy()
    return float(logp[a]), float(H), g_lp, g_h


def close_f32(got, ref):
    """Within one float32 ulp of the float64 value, 1e-12 absolute near 0; NaN where it is NaN."""
    if np.isnan(ref):
        return bool(np.isnan(got))
    return abs(float(got) - ref) <= max(float(np.spacing(np.float32(abs(ref)))), 1e-12)


def close_grad(got, ref, scale, bf16):
    """Gradient entries: one ulp of the output dtype plus 1e-12 * scale (NaN where the reference is NaN, exactly 0
    where it is exactly 0 with no upstream term: the closed entries)."""
    got = np.asarray(got, np.float64)
    nan = np.isnan(ref)
    if not np.array_equal(np.isnan(got), nan):
        return False
    ulp = np.spacing(np.abs(ref[~nan]).astype(np.float32)).astype(np.float64) * (2.0 ** 16 if bf16 else 1.0)
    return bool(np.all(np.abs(got[~nan] - ref[~nan]) <= ulp + 1e-12 * scale))


# ---------------------------------------------------------------------------------------------- segment walks
def gtb_walk(spec, dims):
    """[(who, unit, slot, offset, length)] of one row's segments."""
    return [(w, u, s, o, n) for w, u, s, o, n, _ in gtb_segments(spec, dims)]


def seg_views_gtb(spec, dims, la, lp, ma, mp, aa, ap, r):
    """(open, logits, action, (who, unit, slot, offset, length)) of every segment of flat row r (float32 numpy)."""
    for who, unit, slot, off, ln in gtb_walk(spec, dims):
        if who == "a":
            yield ma[r, unit, off:off + ln] != 0, la[r, unit, off:off + ln], int(aa[r, unit, slot]), (who, unit, slot, off, ln)
        else:
            yield mp[r, off:off + ln] != 0, lp[r, off:off + ln], int(ap[r, slot]), (who, unit, slot, off, ln)


def seg_views_covid(la, lp, ma, mp, aa, ap, r):
    for s in range(la.shape[1]):
        yield ma[r, :, s] != 0, la[r, s], int(aa[r, s]), ("a", s, None, None, None)
    yield mp[r] != 0, lp[r], int(ap[r]), ("p", 0, None, None, None)


def flat(x, lead):
    return None if x is None else np.asarray(x).reshape((int(np.prod(lead)),) + np.asarray(x).shape[len(lead):])


def check_all(views, lead, out, grads=None, ups=None, bf16=False):
    """Every segment against the restatement.  views(r) -> segment views of flat row r; out = (lp_a, lp_p, H_a, H_p);
    grads = (g_a, g_p) for upstream ups = (glp_a, glp_p, gh_a, gh_p) (None: zero).  Returns the segments checked and
    counts of the planted edge kinds seen."""
    lp_a, lp_p, h_a, h_p = [flat(x, lead) for x in out]
    kinds = dict(closed=0, bad=0, bad_action=0, ninf_open=0)
    n = 0
    for r in range(int(np.prod(lead))):
        for o, l, a, (who, unit, slot, off, ln) in views(r):
            rlp, rh, glp, gh = ref_segment(o, l, a)
            if who == "a":
                idx = (r, unit) if slot is None else (r, unit, slot)
                got_lp, got_h = lp_a[idx], h_a[idx]
            else:
                idx = (r,) if slot is None else (r, slot)
                got_lp, got_h = lp_p[idx], h_p[idx]
            assert close_f32(got_lp, rlp), (who, r, unit, slot, float(got_lp), rlp)
            assert close_f32(got_h, rh), (who, r, unit, slot, float(got_h), rh)
            lf = np.asarray(l, np.float32)
            kinds["closed"] += int(not o.any())
            kinds["bad"] += int(o.any() and np.isnan(rh))
            kinds["bad_action"] += int(not np.isnan(rh) and o.any() and np.isnan(rlp))
            kinds["ninf_open"] += int(bool((o & (lf == -np.inf)).any()))
            if grads is not None:
                u = [flat(x, lead) for x in ups]
                ulp_, uh = (u[0], u[2]) if who == "a" else (u[1], u[3])
                cl = 0.0 if ulp_ is None else float(ulp_[idx])
                ch = 0.0 if uh is None else float(uh[idx])
                with np.errstate(invalid="ignore"):
                    ref = cl * glp + ch * gh if (cl or ch) else np.where(np.isnan(glp) | np.isnan(gh), np.nan, 0.0)
                if np.isnan(rlp) and not np.isnan(rh):   # a bad action: NaN at the open entries whatever the upstream
                    ref = np.where(o, np.nan, 0.0)
                g = flat(grads[0], lead) if who == "a" else flat(grads[1], lead)
                if slot is None:   # COVID-19
                    got = g[r, unit] if who == "a" else g[r]
                elif who == "a":
                    got = g[r, unit, off:off + ln]
                else:
                    got = g[r, off:off + ln]
                got = as_f32(np.ascontiguousarray(got))
                assert close_grad(got, ref, abs(cl) + abs(ch), bf16), (who, r, unit, slot, got, ref)
                assert np.all(got[~o] == 0.0)
            n += 1
    return n, kinds


# ---------------------------------------------------------------------------------------------- rollouts (emulation)
def gtb_rollout(cfg, obs_dtype, E, T, seed=11, bf16_logits=False):
    """T steps of sample_actions + step on an emulated env: stacked [T, E, ...] logits, masks (raw buffers), actions
    and the sampler's log-probabilities."""
    env = emu_env(cfg, n_envs=E, obs_dtype=obs_dtype)
    st = env.stepper
    sa, sp = logit_shapes(env)
    rng = np.random.RandomState(seed)
    rec = {k: [] for k in ("la", "lp", "ma", "mp", "aa", "ap", "lpa", "lpp")}
    for t in range(T):
        la = random_logits(rng, sa)
        lp = random_logits(rng, sp) if sp else None
        if bf16_logits:
            la, lp = to_bf16_bits(la), (None if lp is None else to_bf16_bits(lp))
        rec["ma"].append(st.buf["mask_agent"].copy())
        rec["mp"].append(st.buf["mask_planner"].copy())
        lpa, lpp = env.sample_actions(la, lp, seed=seed, greedy=(t % 2 == 1))
        rec["la"].append(la)
        rec["lp"].append(lp)
        rec["aa"].append(st.buf["actions_agent"].copy())
        rec["ap"].append(st.buf["actions_planner"].copy())
        rec["lpa"].append(lpa.copy())
        rec["lpp"].append(None if lpp is None else lpp.copy())
        env.step(env.action_buffers)
    out = {k: (None if v[0] is None else np.stack(v)) for k, v in rec.items()}
    return env, out


def covid_rollout(E, T, seed=13, bf16_logits=False):
    env = emu_covid(E)
    st = env.stepper
    sa, sp = covid_shapes(env)
    rng = np.random.RandomState(seed)
    rec = {k: [] for k in ("la", "lp", "ma", "mp", "aa", "ap", "lpa", "lpp")}
    for t in range(T):
        la, lp = random_logits(rng, sa), random_logits(rng, sp)
        if bf16_logits:
            la, lp = to_bf16_bits(la), to_bf16_bits(lp)
        rec["ma"].append(st.buf["mask_agent"].copy())
        rec["mp"].append(st.buf["mask_planner"].copy())
        lpa, lpp = env.sample_actions(la, lp, seed=seed, greedy=(t % 2 == 1))
        rec["la"].append(la)
        rec["lp"].append(lp)
        rec["aa"].append(st.buf["actions_agent"].copy())
        rec["ap"].append(st.buf["actions_planner"].copy())
        rec["lpa"].append(lpa.copy())
        rec["lpp"].append(lpp.copy())
        for _ in range(9):   # the stringency cooldown closes and reopens agent entries
            env.step(env.action_buffers)
    return env, {k: np.stack(v) for k, v in rec.items()}


def nan_of(x):
    """A NaN of x's storage (float32, or bfloat16 bits)."""
    return np.uint16(0x7FC0) if x.dtype == np.uint16 else np.float32(np.nan)


def value_of(x, v):
    return to_bf16_bits(np.float32(v)) if x.dtype == np.uint16 else np.float32(v)


def plant_gtb(env, R):
    """Edge cases in known segments of flat rows 0..5 (R: flat views of the rollout): nothing open, a NaN open logit,
    +inf at an open entry, every logit -inf, a closed action, an action outside [0, n)."""
    segs = gtb_walk(env.spec, env.stepper.dims)
    who, unit, slot, off, ln = segs[0]
    sl = slice(off, off + ln)
    R["ma"][0, unit, sl] = 0
    o1 = np.nonzero(R["ma"][1, unit, sl] != 0)[0]   # the NO-OP is always open
    R["la"][1, unit, off + o1[-1]] = nan_of(R["la"])
    R["ma"][2, unit, off] = value_of(R["ma"], 1.0)
    R["la"][2, unit, off] = value_of(R["la"], np.inf)
    R["la"][3, unit, sl] = value_of(R["la"], -np.inf)
    closed = np.nonzero(R["ma"][4, unit, sl] == 0)[0]
    R["aa"][4, unit, slot] = int(closed[0]) if len(closed) else ln
    R["aa"][5, unit, slot] = -1 if ln % 2 else ln


def plant_covid(R):
    S = R["la"].shape[1]
    R["ma"][0, :, 3] = 0
    R["la"][1, 4, 0] = nan_of(R["la"])          # the NO-OP is always open
    R["la"][2, 5, :] = value_of(R["la"], -np.inf)
    R["aa"][3, 6] = R["la"].shape[2]            # outside [0, n)
    closed = np.nonzero(R["ma"][4, :, 7] == 0)[0]
    R["aa"][4, 7] = int(closed[0]) if len(closed) else -1
    R["ap"][5] = -3
    assert S > 7


def run_eval(st, R, lead):
    sh = lambda k: None if R[k] is None else np.ascontiguousarray(R[k].reshape(lead + R[k].shape[1:]))
    return st.evaluate_policy(sh("la"), sh("lp"), (sh("aa"), sh("ap")), (sh("ma"), sh("mp")))


def flat_rollout(out):
    """The [T, E, ...] rollout as [T*E, ...] rows (copies)."""
    return {k: (None if v is None else np.ascontiguousarray(v.reshape((-1,) + v.shape[2:]))) for k, v in out.items()}


CPU_CFGS = [(c, d) for c, d in EXACT_CFGS] + [("covid", None)]


@pytest.mark.parametrize("bf16_logits", [False, True], ids=["f32_logits", "bf16_logits"])
@pytest.mark.parametrize("cfg,obs_dtype", CPU_CFGS, ids=lambda v: str(v).replace("torch.", ""))
def test_emulated_forward_and_backward_match_the_restatement(cfg, obs_dtype, bf16_logits):
    """Random logits from a short rollout with edge cases planted in known segments: (T, E) rows forward, a gathered
    (N,) minibatch (N != n_envs) forward and backward for g_lp only, g_H only and both."""
    big = cfg in ("c5_small", "one_step")
    E, T = (3, 3) if big else (4, 3)
    if cfg == "covid":
        env, out = covid_rollout(3, 3, bf16_logits=bf16_logits)
    else:
        env, out = gtb_rollout(cfg, obs_dtype, E, T, bf16_logits=bf16_logits)
    st = env.stepper
    T, E = out["la"].shape[:2]
    R = flat_rollout(out)
    (plant_covid if cfg == "covid" else lambda r: plant_gtb(env, r))(R)
    R32 = {k: as_f32(v) for k, v in R.items()}
    if cfg == "covid":
        views = lambda r, D=R32: seg_views_covid(D["la"], D["lp"], D["ma"], D["mp"], D["aa"], D["ap"], r)
    else:
        views = lambda r, D=R32: seg_views_gtb(env.spec, st.dims, D["la"], D["lp"], D["ma"], D["mp"], D["aa"], D["ap"], r)
    res = run_eval(st, R, (T, E))
    assert res[0].shape[:2] == (T, E) and res[0].dtype == np.float32
    n, kinds = check_all(views, (T, E), res)
    assert n > 0 and kinds["closed"] >= 1 and kinds["bad"] >= 2 and kinds["bad_action"] >= 1 and kinds["ninf_open"] >= 1
    # a gathered minibatch: the planted rows and a few others, N != n_envs
    idx = np.array([0, 1, 2, 3, 4, 5, T * E - 1, 7])
    G = {k: (None if v is None else np.ascontiguousarray(v[idx])) for k, v in R.items()}
    G32 = {k: as_f32(v) for k, v in G.items()}
    N = len(idx)
    assert N != E
    gres = run_eval(st, G, (N,))
    for x, y in zip(gres, res):
        if x is not None:
            assert x.tobytes() == flat(y, (T, E))[idx].tobytes()
    if cfg == "covid":
        gviews = lambda r: seg_views_covid(G32["la"], G32["lp"], G32["ma"], G32["mp"], G32["aa"], G32["ap"], r)
    else:
        gviews = lambda r: seg_views_gtb(env.spec, st.dims, G32["la"], G32["lp"], G32["ma"], G32["mp"], G32["aa"], G32["ap"], r)
    rng = np.random.RandomState(2)
    planner = gres[1] is not None
    up = lambda like: None if like is None else rng.standard_normal(like.shape).astype(np.float32)
    for mode in ("lp", "h", "both"):
        glp = (up(gres[0]), up(gres[1])) if mode in ("lp", "both") else (None, None)
        gh = (up(gres[2]), up(gres[3])) if mode in ("h", "both") else (None, None)
        ga, gp = st.evaluate_policy_backward(G["la"], G["lp"], (G["aa"], G["ap"]), (G["ma"], G["mp"]), glp, gh)
        assert ga.shape == G["la"].shape and ga.dtype == G["la"].dtype
        assert (gp is None) == (not planner)
        check_all(gviews, (N,), gres, grads=(ga, gp), ups=(glp[0], glp[1], gh[0], gh[1]), bf16=bf16_logits)


@pytest.mark.parametrize("cfg,obs_dtype", CPU_CFGS, ids=lambda v: str(v).replace("torch.", ""))
def test_emulated_log_probs_are_the_samplers_bit_for_bit(cfg, obs_dtype):
    """The sampler's logits, the masks at that moment and the drawn actions give back its log-probabilities exactly,
    for stochastic and greedy draws and both logits dtypes."""
    for bf16 in (False, True):
        if cfg == "covid":
            env, out = covid_rollout(3, 4, seed=21, bf16_logits=bf16)
        else:
            env, out = gtb_rollout(cfg, obs_dtype, 3, 4, seed=21, bf16_logits=bf16)
        lead = out["la"].shape[:2]
        res = env.evaluate_actions(out["la"], out["lp"], (out["aa"], out["ap"]), (out["ma"], out["mp"]))
        assert res[0].tobytes() == out["lpa"].tobytes()
        if out["lpp"] is not None:
            assert res[1].tobytes() == out["lpp"].tobytes()
        assert res[0].shape == lead + out["aa"].shape[2:]


def test_emulated_bf16_gradient_is_the_rounded_float64():
    """bfloat16 gradients are the round-to-nearest-even of the float64 value: the float32 call's gradient (itself
    within one float32 ulp) rounds to the same bfloat16 except at a float32 tie neighbourhood, which must be rare."""
    env, out = gtb_rollout("tax_us_federal", None, 4, 2, bf16_logits=True)
    R = flat_rollout(out)
    st = env.stepper
    g16 = st.evaluate_policy_backward(R["la"], R["lp"], (R["aa"], R["ap"]), (R["ma"], R["mp"]),
                                      (np.ones(R["aa"].shape, np.float32), None), (None, None))[0]
    g32 = st.evaluate_policy_backward(as_f32(R["la"]), as_f32(R["lp"]), (R["aa"], R["ap"]), (R["ma"], R["mp"]),
                                      (np.ones(R["aa"].shape, np.float32), None), (None, None))[0]
    assert g16.dtype == np.uint16
    rounded = to_bf16_bits(g32)
    nan = np.isnan(g32)
    assert np.array_equal(np.isnan(as_f32(g16)), nan) and nan.any()
    assert np.mean(rounded[~nan] != g16[~nan]) < 1e-3


def test_emulated_value_errors_and_empty_batches():
    env = emu_env("c3_reset", n_envs=2)
    st = env.stepper
    _, out = gtb_rollout("c3_reset", None, 2, 2)
    R = flat_rollout(out)
    la, lp, aa, ap, ma, mp = (R[k] for k in ("la", "lp", "aa", "ap", "ma", "mp"))
    good = dict(la=la, lp=lp, acts=(aa, ap), masks=(ma, mp))
    bad = [
        dict(la=la[:, :-1]),                                        # row shape
        dict(la=la.astype(np.float64)),                             # dtype
        dict(la=np.asfortranarray(la)),                             # contiguity
        dict(lp=None),                                              # planner actions need planner logits
        dict(lp=to_bf16_bits(lp)),                                  # logits dtypes differ
        dict(lp=lp[:-1]),                                           # leading shapes differ
        dict(acts=(aa.astype(np.int64), ap)),                       # action dtype
        dict(acts=(aa, None)),                                      # planner actions missing
        dict(acts=aa),                                              # not a pair
        dict(masks=(ma[:, :, :-1].copy(), mp)),                     # mask shape
        dict(masks=(ma, to_bf16_bits(mp))),                         # mask dtypes differ
        dict(masks=(ma.astype(np.int32), mp)),                      # mask dtype
    ]
    for b in bad:
        kw = dict(good)
        kw.update(b)
        with pytest.raises(ValueError):
            env.evaluate_actions(kw["la"], kw["lp"], kw["acts"], kw["masks"])
        with pytest.raises(ValueError):
            st.evaluate_policy_backward(kw["la"], kw["lp"], kw["acts"], kw["masks"])
    with pytest.raises(ValueError):   # upstream gradients shaped like the actions, float32
        st.evaluate_policy_backward(la, lp, (aa, ap), (ma, mp), (np.ones(aa.shape, np.float64), None))
    with pytest.raises(ValueError):
        st.evaluate_policy_backward(la, lp, (aa, ap), (ma, mp), (None, None), (None, np.ones((1, 1), np.float32)))
    # zero rows: empty outputs, no error
    z = lambda x: np.ascontiguousarray(x[:0])
    res = env.evaluate_actions(z(la), z(lp), (z(aa), z(ap)), (z(ma), z(mp)))
    assert res[0].shape == (0,) + aa.shape[1:] and res[1].shape == (0,) + ap.shape[1:]
    g = st.evaluate_policy_backward(z(la), z(lp), (z(aa), z(ap)), (z(ma), z(mp)))
    assert g[0].shape == (0,) + la.shape[1:]
    # no planner actions: planner inputs are ignored, planner outputs are None
    env1, out1 = gtb_rollout("c1_tutorial", None, 2, 1)
    R1 = flat_rollout(out1)
    res = env1.evaluate_actions(R1["la"], "ignored", (R1["aa"], None), (R1["ma"], None))
    assert res[1] is None and res[3] is None
    assert env1.stepper.evaluate_policy_backward(R1["la"], None, (R1["aa"], None), (R1["ma"], None))[1] is None
    # COVID-19: the agent mask is transposed against the logits
    cenv, cout = covid_rollout(2, 1)
    CR = flat_rollout(cout)
    with pytest.raises(ValueError):
        cenv.evaluate_actions(CR["la"], CR["lp"], (CR["aa"], CR["ap"]),
                              (np.ascontiguousarray(CR["ma"].transpose(0, 2, 1)), CR["mp"]))
    with pytest.raises(ValueError):
        cenv.evaluate_actions(CR["la"], CR["lp"], (CR["aa"], CR["ap"][:, None].copy()), (CR["ma"], CR["mp"]))


def _eval_struct(la, lp, ma, mp, aa, ap, outs, grads=None, bwd=False):
    q = _abi.AiePolicyEval()
    q.logits_agent, q.logits_planner = la.ctypes.data, (None if lp is None else lp.ctypes.data)
    q.mask_agent, q.mask_planner = ma.ctypes.data, (None if mp is None else mp.ctypes.data)
    q.actions_agent, q.actions_planner = aa.ctypes.data, (None if ap is None else ap.ctypes.data)
    q.logits_dtype = q.mask_dtype = _abi.OBS_F32
    q.log_prob_agent, q.log_prob_planner, q.entropy_agent, q.entropy_planner = [x.ctypes.data for x in outs]
    if bwd:
        q.grad_logits_agent, q.grad_logits_planner = grads[0].ctypes.data, grads[1].ctypes.data
    return q


@pytest.mark.parametrize("scenario", ["gtb", "covid"])
def test_abi_errors(scenario):
    """Every AIE_EINVAL case of both directions, a row count of 0, and no bound buffers or loaded state needed."""
    from tests.emu.emu_stepper import emu_lib
    lib = emu_lib()
    if scenario == "gtb":
        _, out = gtb_rollout("c3_reset", None, 2, 1)
        from ai_economist_b200 import foundation
        from tests.emu.emu_stepper import emu_factory
        kw = gtb_kwargs("c3_reset")
        name = kw.pop("scenario_name")
        fresh = foundation.make_env_instance(name, n_envs=2, seeds=[0, 1], stepper_factory=emu_factory, **kw)   # no reset
        h, fwd, bwd = fresh.stepper._h, lib.aie_evaluate_policy, lib.aie_evaluate_policy_backward
    else:
        cenv, out = covid_rollout(2, 1)
        h, fwd, bwd = cenv.stepper._h, lib.aie_covid_evaluate_policy, lib.aie_covid_evaluate_policy_backward
    R = flat_rollout(out)
    la, lp, ma, mp, aa, ap = (R[k] for k in ("la", "lp", "ma", "mp", "aa", "ap"))
    N = la.shape[0]
    outs = [np.zeros(aa.shape, np.float32), np.zeros(ap.shape, np.float32), np.zeros(aa.shape, np.float32),
            np.zeros(ap.shape, np.float32)]
    grads = [np.zeros(la.shape, np.float32), np.zeros(lp.shape, np.float32)]

    def call(fn, n=N, bwd_=False, **over):
        q = _eval_struct(la, lp, ma, mp, aa, ap, outs, grads, bwd=bwd_)
        for k, v in over.items():
            setattr(q, k, v)
        return fn(h, C.byref(q), C.c_int64(n), None)

    assert call(fwd) == 0 and call(bwd, bwd_=True) == 0
    assert fwd(h, None, C.c_int64(N), None) == AIE_EINVAL
    assert fwd(None, C.byref(_eval_struct(la, lp, ma, mp, aa, ap, outs)), C.c_int64(N), None) == AIE_EINVAL
    for fn, b in ((fwd, False), (bwd, True)):
        assert call(fn, n=-1, bwd_=b) == AIE_EINVAL
        assert call(fn, bwd_=b, logits_dtype=5) == AIE_EINVAL
        assert call(fn, bwd_=b, mask_dtype=-1) == AIE_EINVAL
        for k in ("logits_agent", "mask_agent", "actions_agent", "logits_planner", "mask_planner", "actions_planner"):
            assert call(fn, bwd_=b, **{k: None}) == AIE_EINVAL, k
        assert call(fn, bwd_=b, logits_agent=la.ctypes.data + 2) == AIE_EINVAL
        assert call(fn, bwd_=b, mask_planner=mp.ctypes.data + 1) == AIE_EINVAL
        assert call(fn, bwd_=b, actions_agent=aa.ctypes.data + 2) == AIE_EINVAL
        assert call(fn, n=0, bwd_=b, logits_agent=None, mask_agent=None) == 0      # zero rows: a no-op
    for k in ("log_prob_agent", "entropy_agent", "log_prob_planner", "entropy_planner"):
        assert call(fwd, **{k: None}) == AIE_EINVAL, k
    assert call(fwd, log_prob_agent=outs[0].ctypes.data + 2) == AIE_EINVAL
    for k in ("grad_logits_agent", "grad_logits_planner"):
        assert call(bwd, bwd_=True, **{k: None}) == AIE_EINVAL, k
    assert call(bwd, bwd_=True, grad_logits_agent=grads[0].ctypes.data + 2) == AIE_EINVAL
    up = np.ones(aa.shape, np.float32)
    assert call(bwd, bwd_=True, grad_log_prob_agent=up.ctypes.data + 1) == AIE_EINVAL
    assert call(bwd, bwd_=True, grad_log_prob_agent=up.ctypes.data) == 0
    assert call(bwd, logits_dtype=_abi.OBS_BF16, bwd_=True, grad_logits_agent=grads[0].ctypes.data + 2) == 0   # 2-byte alignment
    # the forward's outputs are not needed by the backward, nor the backward's by the forward
    assert call(bwd, bwd_=True, log_prob_agent=None, entropy_agent=None, log_prob_planner=None, entropy_planner=None) == 0
    assert call(fwd, grad_logits_agent=None, grad_logits_planner=None) == 0


def test_no_counter_moves_and_no_env_state_is_touched():
    """Evaluation leaves the env alone: the sampler's next draws and the launch count are those of an env that never
    evaluated."""
    e1, e2 = emu_env("c3_reset", n_envs=2), emu_env("c3_reset", n_envs=2)
    sa, sp = logit_shapes(e1)
    rng = np.random.RandomState(3)
    la, lp = random_logits(rng, sa), random_logits(rng, sp)
    ma, mp = e1.stepper.buf["mask_agent"].copy(), e1.stepper.buf["mask_planner"].copy()
    e1.sample_actions(la, lp, seed=4)
    e2.sample_actions(la, lp, seed=4)
    aa, ap = e1.stepper.buf["actions_agent"].copy(), e1.stepper.buf["actions_planner"].copy()
    n0 = e1.stepper.launch_count()
    e1.evaluate_actions(la, lp, (aa, ap), (ma, mp))
    e1.stepper.evaluate_policy_backward(la, lp, (aa, ap), (ma, mp), (np.ones(aa.shape, np.float32), None))
    assert e1.stepper.launch_count() == n0
    r1 = e1.sample_actions(la, lp, seed=4)
    r2 = e2.sample_actions(la, lp, seed=4)
    assert r1[0].tobytes() == r2[0].tobytes() and r1[1].tobytes() == r2[1].tobytes()


# ---------------------------------------------------------------------------------------------- GPU
def _gpu_logits(shape, dt, g):
    x = torch.randn(shape, device="cuda:0", generator=g) * 3
    x[torch.rand(shape, device="cuda:0", generator=g) < 0.1] = float("-inf")
    return x.to(dt)


def _gtb_rollout_cuda(cfg, E, T, ldt, obs_dtype=None):
    """T steps of sample_actions + step at full size, staggered episodes: stacked [T, E, ...] device tensors."""
    from ai_economist_b200 import foundation, workloads
    kw = dict(workloads.BASELINE_CONFIGS[cfg])
    name = kw.pop("scenario_name")
    if cfg == "c5_full":
        kw["device_reset"] = "snapshot"
    env = foundation.make_env_instance(name, n_envs=E, device="cuda:0", seeds=list(range(E)), obs_dtype=obs_dtype, **kw)
    env.reset()
    st = env.stepper
    Tep = int(env.episode_length)
    st.state_view("t").copy_((torch.arange(E, device="cuda:0", dtype=torch.int64) * Tep // E).to(torch.int32))
    sa, sp = logit_shapes(env)
    g = torch.Generator(device="cuda:0").manual_seed(5)
    rec = {k: [] for k in ("la", "lp", "ma", "mp", "aa", "ap", "lpa", "lpp")}
    for t in range(T):
        la = _gpu_logits(sa, ldt, g)
        lp = _gpu_logits(sp, ldt, g) if sp else None
        rec["ma"].append(st.buf["mask_agent"].clone())
        rec["mp"].append(st.buf["mask_planner"].clone())
        lpa, lpp = env.sample_actions(la, lp, seed=17, greedy=(t == T - 1))
        rec["la"].append(la)
        rec["lp"].append(lp)
        rec["aa"].append(st.buf["actions_agent"].clone())
        rec["ap"].append(st.buf["actions_planner"].clone())
        rec["lpa"].append(lpa.clone())
        rec["lpp"].append(None if lpp is None else lpp.clone())
        env.step(env.action_buffers)
    return env, {k: (None if v[0] is None else torch.stack(v)) for k, v in rec.items()}


def _covid_rollout_cuda(E, T, ldt):
    env = covid_env(E)
    st = env.stepper
    Tep = int(env.episode_length)
    st.buf["hdr"][:, 0] = (torch.arange(E, device="cuda:0") * Tep // E).to(torch.int32)
    sa, sp = covid_shapes(env)
    g = torch.Generator(device="cuda:0").manual_seed(6)
    rec = {k: [] for k in ("la", "lp", "ma", "mp", "aa", "ap", "lpa", "lpp")}
    for t in range(T):
        la, lp = _gpu_logits(sa, ldt, g), _gpu_logits(sp, ldt, g)
        rec["ma"].append(st.buf["mask_agent"].clone())
        rec["mp"].append(st.buf["mask_planner"].clone())
        lpa, lpp = env.sample_actions(la, lp, seed=19, greedy=(t == T - 1))
        rec["la"].append(la)
        rec["lp"].append(lp)
        rec["aa"].append(st.buf["actions_agent"].clone())
        rec["ap"].append(st.buf["actions_planner"].clone())
        rec["lpa"].append(lpa.clone())
        rec["lpp"].append(lpp.clone())
        env.step(env.action_buffers)
    return env, {k: torch.stack(v) for k, v in rec.items()}


def _np(x):
    """numpy form of a device tensor: float32 / int32, or the raw bits of bfloat16."""
    if x is None:
        return None
    x = x.detach()
    return x.view(torch.int16).cpu().numpy().view(np.uint16) if x.dtype == torch.bfloat16 else x.cpu().numpy()


GPU_CFGS = [("c1_tutorial", 8192), ("c3_paper_tax", 8192), ("c5_full", 2048), ("covid", 4096)]


@pytest.mark.gpu
@pytest.mark.parametrize("ldt", [torch.float32, torch.bfloat16], ids=["f32_logits", "bf16_logits"])
@pytest.mark.parametrize("cfg,E", GPU_CFGS, ids=[c for c, _ in GPU_CFGS])
def test_cuda_full_size(cfg, E, ldt):
    """Full size, a T x E batch of rollout rows with masks stored from real steps: the sampler's log-probabilities bit
    for bit; sampled rows against the restatement, forward and backward; autograd equals the stepper-level backward;
    a gathered contiguous minibatch gives the same rows as the full batch."""
    T = 3
    if cfg == "covid":
        env, R = _covid_rollout_cuda(E, T, ldt)
    else:
        env, R = _gtb_rollout_cuda(cfg, E, T, ldt)
    st = env.stepper
    planner = R["lp"] is not None
    # 1. the sampler's log-probabilities, bit for bit
    res = env.evaluate_actions(R["la"], R["lp"], (R["aa"], R["ap"]), (R["ma"], R["mp"]))
    assert torch.equal(res[0].view(torch.int32), R["lpa"].view(torch.int32))
    if planner:
        assert torch.equal(res[1].view(torch.int32), R["lpp"].view(torch.int32))
    # 2. sampled rows against the restatement (forward, then backward with both upstream terms)
    flatR = {k: (None if v is None else v.reshape((T * E,) + v.shape[2:])) for k, v in R.items()}
    pick = torch.tensor(np.r_[0:4, E:E + 2, T * E // 2:T * E // 2 + 2, T * E - 4:T * E], device="cuda:0")
    G = {k: (None if v is None else v.index_select(0, pick).contiguous()) for k, v in flatR.items()}
    N = len(pick)
    gres = st.evaluate_policy(G["la"], G["lp"], (G["aa"], G["ap"]), (G["ma"], G["mp"]))
    full = [None if x is None else x.reshape((T * E,) + x.shape[2:]).index_select(0, pick) for x in res]
    for x, y in zip(gres, full):   # 4. a gathered minibatch gives the same rows
        assert (x is None and y is None) or torch.equal(x.view(torch.int32), y.view(torch.int32))
    gen = torch.Generator(device="cuda:0").manual_seed(9)
    up = lambda like: None if like is None else torch.randn(like.shape, device="cuda:0", generator=gen)
    glp, gh = (up(gres[0]), up(gres[1])), (up(gres[2]), up(gres[3]))
    ga, gp = st.evaluate_policy_backward(G["la"], G["lp"], (G["aa"], G["ap"]), (G["ma"], G["mp"]), glp, gh)
    G32 = {k: as_f32(_np(v)) for k, v in G.items()}
    if cfg == "covid":
        views = lambda r: seg_views_covid(G32["la"], G32["lp"], G32["ma"], G32["mp"], G32["aa"], G32["ap"], r)
    else:
        views = lambda r: seg_views_gtb(env.spec, st.dims, G32["la"], G32["lp"], G32["ma"], G32["mp"], G32["aa"],
                                        G32["ap"], r)
    n, _ = check_all(views, (N,), [_np(x) for x in gres], grads=(_np(ga), _np(gp)),
                     ups=[_np(x) for x in (glp[0], glp[1], gh[0], gh[1])], bf16=(ldt == torch.bfloat16))
    assert n > 0
    # 3. through autograd: the stepper-level backward's gradients, on the full batch
    la = R["la"].detach().clone().requires_grad_(True)
    lp = R["lp"].detach().clone().requires_grad_(True) if planner else None
    lpa, lpp, ha, hp = env.evaluate_actions(la, lp, (R["aa"], R["ap"]), (R["ma"], R["mp"]))
    loss = lpa.nan_to_num(0.0).sum() + 0.01 * ha.nan_to_num(0.0).sum()
    if planner:
        loss = loss + lpp.nan_to_num(0.0).sum() + 0.01 * hp.nan_to_num(0.0).sum()
    loss.backward()
    ones = lambda x: None if x is None else torch.where(torch.isnan(x), 0.0, 1.0).contiguous()
    hund = lambda x: None if x is None else torch.where(torch.isnan(x), 0.0, 0.01).contiguous()
    ra, rp = st.evaluate_policy_backward(R["la"], R["lp"], (R["aa"], R["ap"]), (R["ma"], R["mp"]),
                                         (ones(lpa), ones(lpp)), (hund(ha), hund(hp)))
    assert la.grad.dtype == ldt and torch.equal(la.grad.view(torch.int16 if ldt == torch.bfloat16 else torch.int32),
                                                ra.view(torch.int16 if ldt == torch.bfloat16 else torch.int32))
    if planner:
        assert torch.equal(lp.grad.view(ra.dtype == torch.bfloat16 and torch.int16 or torch.int32),
                           rp.view(ra.dtype == torch.bfloat16 and torch.int16 or torch.int32))


@pytest.mark.gpu
def test_cuda_matches_the_emulation():
    """The CUDA kernels and the host build of the same source on the same rows: log-probabilities and entropies within
    one float32 ulp, gradients within one ulp, in both launch shapes' configs (c3: one warp per row, c5: per unit)."""
    from ai_economist_b200 import foundation, workloads
    from tests.emu.emu_stepper import emu_factory
    for cfg, E in (("c3_paper_tax", 512), ("c5_full", 256)):
        env, R = _gtb_rollout_cuda(cfg, E, 2, torch.float32)
        kw = dict(workloads.BASELINE_CONFIGS[cfg])
        name = kw.pop("scenario_name")
        twin = foundation.make_env_instance(name, n_envs=2, seeds=[0, 1], stepper_factory=emu_factory, **kw)
        n = 16
        F = {k: (None if v is None else v.reshape((-1,) + v.shape[2:])[:n].contiguous()) for k, v in R.items()}
        Fn = {k: _np(v) for k, v in F.items()}
        a = env.stepper.evaluate_policy(F["la"], F["lp"], (F["aa"], F["ap"]), (F["ma"], F["mp"]))
        b = twin.stepper.evaluate_policy(Fn["la"], Fn["lp"], (Fn["aa"], Fn["ap"]), (Fn["ma"], Fn["mp"]))
        for x, y in zip(a, b):
            if x is not None:
                assert torch.equal(x.view(torch.int32).cpu(), torch.from_numpy(y).view(torch.int32)) or \
                    np.all((np.abs(_np(x) - y) <= np.spacing(np.abs(y))) | (np.isnan(y) & np.isnan(_np(x))))
        ones = np.ones(Fn["aa"].shape, np.float32)
        ga = env.stepper.evaluate_policy_backward(F["la"], F["lp"], (F["aa"], F["ap"]), (F["ma"], F["mp"]),
                                                  (torch.from_numpy(ones).cuda(), None))[0]
        gb = twin.stepper.evaluate_policy_backward(Fn["la"], Fn["lp"], (Fn["aa"], Fn["ap"]), (Fn["ma"], Fn["mp"]),
                                                   (ones, None))[0]
        ga = _np(ga)
        assert np.all((np.abs(ga - gb) <= np.spacing(np.abs(gb)) + 1e-12) | (np.isnan(gb) & np.isnan(ga)))
        del env
        torch.cuda.empty_cache()
