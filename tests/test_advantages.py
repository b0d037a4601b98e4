"""Advantages and value targets of a stored rollout (env.compute_advantages / aie_compute_advantages /
aie_covid_compute_advantages): generalised advantage estimation over the agents' [T, E, A] and the planner's [T, E]
columns, bootstrapped at episode ends from the values of the final observations.

`gae_ref` below restates the recursion of include/aie_b200.h in numpy float64 (every operation rounded, no fused
multiply-add, gl = gamma * lam computed once, np.where for the selects).  The host build of the device source and the
CUDA kernel must give its float32 bits exactly, NaN positions included; a NaN's payload is not part of the contract."""
import ctypes as C

import numpy as np
import pytest
import torch

from ai_economist_b200 import _abi
from tests import batch_utils as bu
from tests.test_policy_sampler import covid_env, emu_covid, emu_env

AIE_EINVAL = -1


# ---------------------------------------------------------------------------------------------- numpy restatement
def gae_ref(R, V, D, LV, F, gamma, lam, f64=False):
    """(adv, ret) float32 of one group: R [T, E(, A)] float32 / float64, V and F (or None) float32 like R, D int32 [T, E],
    LV float32 [E(, A)].  f64=True also returns the float64 advantages."""
    T = R.shape[0]
    D = np.broadcast_to((D != 0).reshape(D.shape + (1,) * (R.ndim - 2)), R.shape)
    R64, V64 = R.astype(np.float64), V.astype(np.float64)
    gamma, gl = np.float64(gamma), np.float64(gamma) * np.float64(lam)
    adv, ret = np.empty(R.shape, np.float32), np.empty(R.shape, np.float32)
    a64 = np.empty(R.shape, np.float64)
    a = np.zeros(R.shape[1:])
    vnext = LV.astype(np.float64)
    with np.errstate(invalid="ignore", over="ignore"):
        for t in range(T - 1, -1, -1):
            d = D[t]
            f = F[t].astype(np.float64) if F is not None else np.zeros(R.shape[1:])
            nv = np.where(d, f, vnext)
            delta = (R64[t] + gamma * nv) - V64[t]
            a = delta if t == T - 1 else np.where(d, delta, delta + gl * a)
            a64[t] = a
            adv[t] = a.astype(np.float32)
            ret[t] = (a + V64[t]).astype(np.float32)
            vnext = V64[t]
    return (adv, ret, a64) if f64 else (adv, ret)


def same_bits(got, ref):
    """float32 arrays equal bit for bit, NaN where the reference is NaN (any payload)."""
    got, ref = np.asarray(got, np.float32), np.asarray(ref, np.float32)
    nan = np.isnan(ref)
    return (got.shape == ref.shape and np.array_equal(np.isnan(got), nan)
            and np.array_equal(got[~nan].view(np.uint32), ref[~nan].view(np.uint32)))


def ref_all(inp, gamma, lam):
    """(adv_a, adv_p, ret_a, ret_p) of the restatement for an input dict (planner entries may be None)."""
    pair = lambda x: tuple(x) if isinstance(x, (tuple, list)) else (x, x)
    g, l = pair(gamma), pair(lam)
    fa, fp = inp["final"] if inp["final"] is not None else (None, None)
    aa, ra = gae_ref(inp["r"][0], inp["v"][0], inp["d"], inp["lv"][0], fa, g[0], l[0])
    if inp["r"][1] is None:
        return aa, None, ra, None
    ap, rp = gae_ref(inp["r"][1], inp["v"][1], inp["d"], inp["lv"][1], fp, g[1], l[1])
    return aa, ap, ra, rp


def check_outputs(out, ref):
    for k, (x, y) in enumerate(zip(out, ref)):
        if y is None:
            assert x is None
        else:
            assert same_bits(x, y), "output %d" % k


# ---------------------------------------------------------------------------------------------- inputs
def random_inputs(rng, T, E, A, r_dtypes, final=True, planner=True, done_mode="random"):
    """Random rewards, values, dones and final values; done_mode plants the episode ends: "random", "first" (t = 0),
    "last" (t = T - 1), "consecutive" (two steps in a row), "all" (every step) or "none"."""
    f32 = lambda *s: (rng.standard_normal(s) * 2).astype(np.float32)
    r = (rng.standard_normal((T, E, A)).astype(r_dtypes[0]), rng.standard_normal((T, E)).astype(r_dtypes[1]))
    d = {"random": (rng.random_sample((T, E)) < 0.15), "none": np.zeros((T, E), bool),
         "all": np.ones((T, E), bool)}.get(done_mode)
    if d is None:
        d = np.zeros((T, E), bool)
        if done_mode == "first":
            d[0] = True
        elif done_mode == "last":
            d[T - 1] = True
        elif done_mode == "consecutive":
            d[T // 2, ::2] = d[min(T // 2 + 1, T - 1), ::2] = True
            d[0, 1::2] = True
    inp = dict(r=r, v=(f32(T, E, A), f32(T, E)), d=d.astype(np.int32), lv=(f32(E, A), f32(E)),
               final=(f32(T, E, A), f32(T, E)) if final else None)
    if not planner:
        inp["r"], inp["v"], inp["lv"] = (r[0], None), (inp["v"][0], None), (inp["lv"][0], None)
        if final:
            inp["final"] = (inp["final"][0], None)
    return inp


def call(env, inp, gamma, lam):
    return env.compute_advantages(inp["r"], inp["v"], inp["d"], inp["lv"], inp["final"], gamma=gamma, lam=lam)


_ENVS = {}


def cpu_env(kind):
    """Emulated envs of the shapes the tests use: c1 (E = 3, A = 4) and COVID-19 (E = 2, A = 51)."""
    if kind not in _ENVS:
        _ENVS[kind] = emu_env("c1_reset", n_envs=3) if kind == "c1" else emu_covid(2)
    return _ENVS[kind]


def env_shape(env):
    sa = env.stepper._policy_shapes()[0]
    return sa[0], sa[1]


# ---------------------------------------------------------------------------------------------- CPU: exactness
@pytest.mark.parametrize("scenario", ["c1", "covid"])
@pytest.mark.parametrize("T", [1, 2, 7, 64])
def test_emulated_matches_the_restatement_bit_for_bit(scenario, T):
    """Both reward dtypes per group, scalar and paired gamma / lambda, final values given and None, planner entries
    given and None, every planted done pattern."""
    env = cpu_env(scenario)
    E, A = env_shape(env)
    rng = np.random.RandomState(T)
    cases = [((np.float64, np.float64), 0.998, 0.98, True, True, "random"),
             ((np.float32, np.float64), (0.99, 0.9), (0.95, 1.0), False, True, "random"),
             ((np.float32, np.float32), 0.98, 1.0, True, False, "first"),
             ((np.float64, np.float32), (1.0, 0.5), 0.0, True, True, "last"),
             ((np.float64, np.float64), 0.9, (0.7, 0.3), True, True, "consecutive"),
             ((np.float32, np.float64), 0.97, 0.9, True, True, "all"),
             ((np.float64, np.float64), 0.0, 1.0, False, True, "none"),
             ((np.float64, np.float64), 1.0, 1.0, True, True, "none")]
    for dt, g, l, final, planner, mode in cases:
        inp = random_inputs(rng, T, E, A, dt, final=final, planner=planner, done_mode=mode)
        out = call(env, inp, g, l)
        assert out[0].dtype == np.float32 and out[0].shape == (T, E, A)
        assert (out[1] is None) == (not planner)
        check_outputs(out, ref_all(inp, g, l))


@pytest.mark.parametrize("scenario", ["c1", "covid"])
def test_emulated_nan_rules(scenario):
    """NaN in final values where done is 0 never reaches the outputs; a NaN value reaches exactly the restatement's
    cells (its own step and the earlier steps of its chain, up to the previous cut)."""
    env = cpu_env(scenario)
    E, A = env_shape(env)
    T = 12
    rng = np.random.RandomState(5)
    inp = random_inputs(rng, T, E, A, (np.float64, np.float64))
    d = inp["d"]
    d[:] = 0
    d[3, 0] = d[8, 0] = 1
    fa, fp = inp["final"]
    fa[d == 0] = np.nan          # every row the contract does not read
    fp[d == 0] = np.nan
    out = call(env, inp, 0.99, 0.95)
    assert not any(np.isnan(x).any() for x in out)
    check_outputs(out, ref_all(inp, 0.99, 0.95))
    va, vp = inp["v"]
    va[6, 0, 1] = np.nan
    vp[10, 1] = np.nan
    out = call(env, inp, 0.99, 0.95)
    ref = ref_all(inp, 0.99, 0.95)
    check_outputs(out, ref)
    nan_a = np.isnan(ref[0])
    # replica 0, agent 1: V[6] is NaN -> steps 6 and 5 (nv = V[6]) and back to the cut at t = 3 (step 3 is cut: done)
    assert np.array_equal(np.nonzero(nan_a[:, 0, 1])[0], [4, 5, 6])
    assert nan_a.sum() == 3
    assert np.array_equal(np.nonzero(np.isnan(ref[1])[:, 1])[0], np.arange(0, 11))


def test_restatement_is_gae():
    """The recursion is Σ_k (γλ)^k δ_{t+k} summed inside each episode segment (within 1e-12), and with λ = 1, zero
    values and no final values its returns are WarpDrive's discounted reward-to-go."""
    rng = np.random.RandomState(0)
    T, E = 40, 6
    for gamma, lam, final in ((0.998, 0.98, True), (0.9, 0.5, False), (1.0, 1.0, True), (0.98, 0.0, True)):
        inp = random_inputs(rng, T, E, 1, (np.float64, np.float64), final=final)
        R, V, D, LV = inp["r"][1], inp["v"][1], inp["d"] != 0, inp["lv"][1]
        F = inp["final"][1] if final else None
        _, _, a64 = gae_ref(R, V, inp["d"], LV, F, gamma, lam, f64=True)
        for e in range(E):
            delta = np.empty(T)
            for t in range(T):
                nv = (float(F[t, e]) if F is not None else 0.0) if D[t, e] else (float(LV[e]) if t == T - 1 else float(V[t + 1, e]))
                delta[t] = float(R[t, e]) + gamma * nv - float(V[t, e])
            for t in range(T):
                end = t
                while not D[end, e] and end < T - 1:
                    end += 1
                want = sum((gamma * lam) ** k * delta[t + k] for k in range(end - t + 1))
                assert abs(a64[t, e] - want) <= 1e-12 * max(1.0, abs(want)), (gamma, lam, t, e)
    # WarpDrive's trainer: returns[t] = r[t] + gamma * (1 - done[t]) * returns[t + 1], returns[T - 1] = r[T - 1]
    inp = random_inputs(rng, T, E, 1, (np.float64, np.float32), final=False)
    R, D = inp["r"][1], inp["d"]
    z = np.zeros((T, E), np.float32)
    _, ret = gae_ref(R, z, D, np.zeros(E, np.float32), None, 0.98, 1.0)
    wd = np.zeros((T, E))
    wd[T - 1] = R[T - 1]
    for t in range(T - 2, -1, -1):
        wd[t] = R[t] + 0.98 * (1 - D[t]) * wd[t + 1]
    assert np.allclose(ret.astype(np.float64), wd, rtol=1e-6, atol=0)   # float32 outputs of the float64 recursion
    _, _, a64 = gae_ref(R, z, D, np.zeros(E, np.float32), None, 0.98, 1.0, f64=True)
    assert np.allclose(a64, wd, rtol=1e-12, atol=1e-12)


def test_emulated_rollout_bootstraps_from_the_final_observation():
    """A Foundation rollout under the auto-reset with final_obs=True, staggered episodes, random actions and a fixed
    linear value function of the flat observations: at every done step the advantage is r + γ·V(final_obs) − V(s)."""
    E, T, gamma, lam = 3, 70, 0.99, 0.95
    env = emu_env("c3_reset", n_envs=E, auto_reset=True, final_obs=True)
    st = env.stepper
    A = env.n_agents
    Tep = env.episode_length
    st.state_view("t")[...] = (np.arange(E) * Tep // E).astype(np.int32)
    st.observe()
    sp = env.spec
    seg_a, seg_p = bu.segments(sp, "a"), bu.segments(sp, "p")
    rng = np.random.RandomState(3)
    fa = st.obs_to_numpy("obs_agent_flat").shape[-1]
    fp = st.obs_to_numpy("obs_planner_flat").shape[-1]
    wa, wp = rng.standard_normal(fa) * 0.01, rng.standard_normal(fp) * 0.01
    val_a = lambda x: (x.astype(np.float64) @ wa).astype(np.float32)
    val_p = lambda x: (x.astype(np.float64) @ wp).astype(np.float32)
    rec = {k: [] for k in ("ra", "rp", "va", "vp", "fa", "fp", "d")}
    for t in range(T):
        rec["va"].append(val_a(st.obs_to_numpy("obs_agent_flat")))
        rec["vp"].append(val_p(st.obs_to_numpy("obs_planner_flat")))
        aa = bu.sample_from_masks(st.obs_to_numpy("mask_agent"), seg_a, rng)
        ap = bu.sample_from_masks(st.obs_to_numpy("mask_planner"), seg_p, rng) if seg_p else None
        env.step((aa, ap))
        rew = st.to_numpy(st.buf["reward"])
        rec["ra"].append(rew[:, :A].copy())
        rec["rp"].append(rew[:, A].copy())
        rec["d"].append(st.to_numpy(st.buf["done"]).copy())
        rec["fa"].append(val_a(st.obs_to_numpy("final_obs_agent_flat")))   # the whole tensor, unspecified rows included
        rec["fp"].append(val_p(st.obs_to_numpy("final_obs_planner_flat")))
    lva, lvp = val_a(st.obs_to_numpy("obs_agent_flat")), val_p(st.obs_to_numpy("obs_planner_flat"))
    R = {k: np.ascontiguousarray(np.stack(v)) for k, v in rec.items()}
    assert R["ra"].dtype == np.float64 and R["d"].sum() >= E and R["d"][:-1].any()
    inp = dict(r=(R["ra"], R["rp"]), v=(R["va"], R["vp"]), d=R["d"], lv=(lva, lvp), final=(R["fa"], R["fp"]))
    out = call(env, inp, gamma, lam)
    check_outputs(out, ref_all(inp, gamma, lam))
    for t, e in zip(*np.nonzero(R["d"])):
        want_a = np.float32((R["ra"][t, e] + gamma * R["fa"][t, e].astype(np.float64)) - R["va"][t, e].astype(np.float64))
        want_p = np.float32((R["rp"][t, e] + gamma * np.float64(R["fp"][t, e])) - np.float64(R["vp"][t, e]))
        assert same_bits(out[0][t, e], want_a) and same_bits(out[1][t, e], want_p), (t, e)
    # without final values the episode end is terminal
    inp["final"] = None
    out = call(env, inp, gamma, lam)
    for t, e in zip(*np.nonzero(R["d"])):
        assert same_bits(out[0][t, e], np.float32(R["ra"][t, e] - R["va"][t, e].astype(np.float64)))


# ---------------------------------------------------------------------------------------------- CPU: errors, side effects
def test_emulated_value_errors():
    env = cpu_env("c1")
    E, A = env_shape(env)
    T = 4
    inp = random_inputs(np.random.RandomState(1), T, E, A, (np.float64, np.float64))
    ok = dict(r=inp["r"], v=inp["v"], d=inp["d"], lv=inp["lv"], final=inp["final"], gamma=0.99, lam=0.95)
    ra, rp = inp["r"]
    va, vp = inp["v"]
    bad = [
        dict(r=ra),                                                 # not a pair
        dict(r=(ra[:, :, :-1].copy(), rp)),                         # agent shape
        dict(r=(ra[:, :-1].copy(), rp)),                            # E
        dict(r=(ra.astype(np.float16), rp)),                        # reward dtype
        dict(r=(np.asfortranarray(ra), rp)),                        # contiguity
        dict(r=(ra, rp[:-1].copy())),                               # planner T
        dict(r=(ra, rp.astype(np.int32))),                          # planner dtype
        dict(v=(va.astype(np.float64), vp)),                        # values are float32
        dict(v=(va, vp[:, :-1].copy())),                            # values shape
        dict(v=(va, None)),                                         # planner entries all or none
        dict(lv=(inp["lv"][0][:-1].copy(), inp["lv"][1])),          # last values shape
        dict(lv=(inp["lv"][0], inp["lv"][1].astype(np.float64))),   # last values dtype
        dict(final=(inp["final"][0], None)),                        # final values: planner entry missing
        dict(final=(inp["final"][0][:-1].copy(), inp["final"][1])),   # final values shape
        dict(final=inp["final"][0]),                                # not a pair
        dict(d=inp["d"].astype(np.int64)),                          # dones dtype
        dict(d=inp["d"][:-1].copy()),                               # dones shape
        dict(gamma=1.5), dict(gamma=-0.1), dict(gamma=float("nan")), dict(lam=float("inf")),
        dict(gamma=(0.9, None)), dict(gamma=(0.9, 0.9, 0.9)), dict(lam="0.9"), dict(gamma=True),
    ]
    for b in bad:
        kw = dict(ok)
        kw.update(b)
        with pytest.raises(ValueError):
            env.compute_advantages(kw["r"], kw["v"], kw["d"], kw["lv"], kw["final"], gamma=kw["gamma"], lam=kw["lam"])
    # T = 0: empty outputs
    z = lambda x: None if x is None else np.ascontiguousarray(x[:0])
    out = env.compute_advantages((z(ra), z(rp)), (z(va), z(vp)), z(inp["d"]), inp["lv"], gamma=0.9)
    assert out[0].shape == (0, E, A) and out[1].shape == (0, E)
    # no planner: a planner gamma of None is fine, planner outputs are None
    out = env.compute_advantages((ra, None), (va, None), inp["d"], (inp["lv"][0], None), gamma=(0.9, None), lam=1.0)
    assert out[1] is None and out[3] is None


def _args(inp, gamma=0.99, lam=0.95, outs=None):
    q = _abi.AieAdvantageArgs()
    q.rewards_agent, q.rewards_planner = inp["r"][0].ctypes.data, inp["r"][1].ctypes.data
    q.rewards_agent_dtype = q.rewards_planner_dtype = _abi.REWARD_F64
    q.values_agent, q.values_planner = inp["v"][0].ctypes.data, inp["v"][1].ctypes.data
    q.dones = inp["d"].ctypes.data
    q.last_values_agent, q.last_values_planner = inp["lv"][0].ctypes.data, inp["lv"][1].ctypes.data
    q.final_values_agent, q.final_values_planner = inp["final"][0].ctypes.data, inp["final"][1].ctypes.data
    q.gamma_agent = q.gamma_planner = gamma
    q.lambda_agent = q.lambda_planner = lam
    q.adv_agent, q.adv_planner, q.ret_agent, q.ret_planner = [x.ctypes.data for x in outs]
    return q


@pytest.mark.parametrize("scenario", ["gtb", "covid"])
def test_abi_errors(scenario):
    """Every AIE_EINVAL case, T = 0, and no bound buffers or loaded state needed."""
    from tests.emu.emu_stepper import emu_lib
    lib = emu_lib()
    if scenario == "gtb":
        from ai_economist_b200 import foundation
        from tests.emu.emu_stepper import emu_factory
        from tests.test_policy_sampler import gtb_kwargs
        kw = gtb_kwargs("c1_reset")
        name = kw.pop("scenario_name")
        fresh = foundation.make_env_instance(name, n_envs=3, seeds=[0, 1, 2], stepper_factory=emu_factory, **kw)   # no reset
        h, fn, (E, A) = fresh.stepper._h, lib.aie_compute_advantages, env_shape(fresh)
    else:
        env = cpu_env("covid")
        h, fn, (E, A) = env.stepper._h, lib.aie_covid_compute_advantages, env_shape(env)
    T = 5
    inp = random_inputs(np.random.RandomState(2), T, E, A, (np.float64, np.float64))
    outs = [np.zeros((T, E, A), np.float32), np.zeros((T, E), np.float32), np.zeros((T, E, A), np.float32),
            np.zeros((T, E), np.float32)]

    def run(t=T, **over):
        q = _args(inp, outs=outs)
        for k, v in over.items():
            setattr(q, k, v)
        return fn(h, C.byref(q), C.c_int32(t), None)

    assert run() == 0
    ref = ref_all(inp, 0.99, 0.95)
    check_outputs(outs, ref)
    assert fn(h, None, C.c_int32(T), None) == AIE_EINVAL
    assert fn(None, C.byref(_args(inp, outs=outs)), C.c_int32(T), None) == AIE_EINVAL
    assert run(t=-1) == AIE_EINVAL
    assert run(rewards_agent_dtype=2) == AIE_EINVAL and run(rewards_planner_dtype=-1) == AIE_EINVAL
    for k in ("gamma_agent", "gamma_planner", "lambda_agent", "lambda_planner"):
        for v in (float("nan"), -1e-300, 1.0000000000000002, float("inf")):
            assert run(**{k: v}) == AIE_EINVAL, (k, v)
    for k in ("rewards_agent", "values_agent", "values_planner", "dones", "last_values_agent", "last_values_planner",
              "adv_agent", "adv_planner", "ret_agent", "ret_planner"):
        assert run(**{k: None}) == AIE_EINVAL, k
    for k, x in (("rewards_agent", inp["r"][0]), ("rewards_planner", inp["r"][1]), ("values_agent", inp["v"][0]),
                 ("dones", inp["d"]), ("last_values_planner", inp["lv"][1]), ("final_values_agent", inp["final"][0]),
                 ("adv_planner", outs[1]), ("ret_agent", outs[2])):
        assert run(**{k: x.ctypes.data + 2}) == AIE_EINVAL, k
    assert run(rewards_agent=inp["r"][0].ctypes.data + 4) == AIE_EINVAL            # float64: 8-byte alignment
    f32 = inp["r"][0].astype(np.float32)
    assert run(rewards_agent=f32.ctypes.data + 4, rewards_agent_dtype=_abi.REWARD_F32, t=1) == 0   # float32: 4 bytes
    # T = 0: a no-op with no pointer read; the pointer checks and the planner group
    outs[0][...] = 7.0
    assert run(t=0, rewards_agent=None, values_agent=None, adv_agent=None) == 0
    assert np.all(outs[0] == 7.0)
    # no planner group: its entries are ignored, gamma included; final values are optional per group
    outs[1][...] = 7.0
    assert run(rewards_planner=None, values_planner=None, adv_planner=None, gamma_planner=float("nan")) == 0
    assert np.all(outs[1] == 7.0)
    assert run(final_values_agent=None, final_values_planner=None) == 0


def test_no_counter_moves_and_no_env_state_is_touched():
    """compute_advantages reads only its arguments: every env buffer and the launch count are byte-identical after it."""
    env = emu_env("c3_reset", n_envs=2, auto_reset=True, final_obs=True)
    env.step(None)
    st = env.stepper
    E, A = env_shape(env)
    before = {k: np.asarray(v).tobytes() for k, v in st.buf.items()}
    n0 = st.launch_count()
    inp = random_inputs(np.random.RandomState(4), 9, E, A, (np.float64, np.float64))
    call(env, inp, 0.99, 0.95)
    assert st.launch_count() == n0
    assert {k: np.asarray(v).tobytes() for k, v in st.buf.items()} == before
    cenv = cpu_env("covid")
    cst = cenv.stepper
    before = {k: np.asarray(v).tobytes() for k, v in cst.buf.items()}
    n0 = cst.launch_count()
    E, A = env_shape(cenv)
    call(cenv, random_inputs(np.random.RandomState(5), 9, E, A, (np.float32, np.float64)), 0.98, 1.0)
    assert cst.launch_count() == n0 and {k: np.asarray(v).tobytes() for k, v in cst.buf.items()} == before


# ---------------------------------------------------------------------------------------------- GPU
def _cuda_gtb(cfg, E):
    from ai_economist_b200 import foundation, workloads
    kw = dict(workloads.BASELINE_CONFIGS[cfg])
    name = kw.pop("scenario_name")
    if cfg == "c5_full":
        kw["device_reset"] = "snapshot"
    env = foundation.make_env_instance(name, n_envs=E, device="cuda:0", seeds=list(range(E)), **kw)
    env.reset()
    Tep = int(env.episode_length)
    env.stepper.state_view("t").copy_((torch.arange(E, device="cuda:0", dtype=torch.int64) * Tep // E).to(torch.int32))
    return env


def _cuda_rollout(env, T, covid):
    """T steps of sample_actions + step from random logits: stacked rewards [T, E, A] / [T, E] and dones [T, E]."""
    st = env.stepper
    E, A = env_shape(env)
    if covid:
        Tep = int(env.episode_length)
        st.buf["hdr"][:, 0] = (torch.arange(E, device="cuda:0") * Tep // E).to(torch.int32)
    sa, sp, _, _ = st._policy_shapes()
    g = torch.Generator(device="cuda:0").manual_seed(7)
    ra, rp, d = [], [], []
    for t in range(T):
        la = torch.randn(sa, device="cuda:0", generator=g)
        lp = torch.randn(sp, device="cuda:0", generator=g) if sp is not None else None
        env.sample_actions(la, lp, seed=11)
        env.step(env.action_buffers)
        if covid:
            ra.append(env.rew["a"].clone())
            rp.append(env.rew["p"].clone())
        else:
            ra.append(st.buf["reward"][:, :A].contiguous())
            rp.append(st.buf["reward"][:, A].contiguous())
        d.append(env.done["__all__"].clone())
    return torch.stack(ra), torch.stack(rp), torch.stack(d)


GPU_CASES = [("c1_tutorial", 8192, 200), ("c3_paper_tax", 8192, 200), ("c5_full", 2048, 150), ("covid", 4096, 90),
             ("covid", 4096, 540)]


@pytest.mark.gpu
@pytest.mark.parametrize("cfg,E,T", GPU_CASES, ids=["%s-E%d-T%d" % c for c in GPU_CASES])
def test_cuda_full_size_matches_the_restatement_and_the_host_build(cfg, E, T):
    """Rewards and dones of a real staggered rollout, random values and final values (NaN planted in rows where done is
    0, and in one value): bit for bit the restatement over every column, and the host build on a slice of replicas."""
    covid = cfg == "covid"
    env = covid_env(E) if covid else _cuda_gtb(cfg, E)
    ra, rp, d = _cuda_rollout(env, T, covid)
    assert bool(d.any()) and bool(d[:-1].any())
    E_, A = env_shape(env)
    assert E_ == E
    g = torch.Generator(device="cuda:0").manual_seed(13)
    rnd = lambda *s: torch.randn(s, device="cuda:0", generator=g)
    va, vp, lva, lvp = rnd(T, E, A), rnd(T, E), rnd(E, A), rnd(E)
    fa, fp = rnd(T, E, A), rnd(T, E)
    fa[(d == 0)] = float("nan")
    fp[(d == 0)] = float("nan")
    va[T // 2, 3, 0] = float("nan")
    rf = (ra, rp)
    np_ = lambda x: x.cpu().numpy()
    inp = dict(r=tuple(np_(x) for x in rf), v=(np_(va), np_(vp)), d=np_(d), lv=(np_(lva), np_(lvp)),
               final=(np_(fa), np_(fp)))
    for gamma, lam, final in ((0.998, 0.98, True), ((0.98, 0.99), (1.0, 0.9), False)):
        out = env.compute_advantages(rf, (va, vp), d, (lva, lvp), (fa, fp) if final else None, gamma=gamma, lam=lam)
        torch.cuda.synchronize()
        assert out[0].dtype == torch.float32 and out[0].shape == (T, E, A) and out[1].shape == (T, E)
        i = dict(inp, final=inp["final"] if final else None)
        ref = ref_all(i, gamma, lam)
        got = [np_(x) for x in out]
        check_outputs(got, ref)
        assert np.isnan(ref[0]).any() and not np.isnan(ref[1]).any()
    # the host build of the same source on the first replicas (the columns of a replica depend on nothing else)
    n = 2
    if covid:
        twin = emu_covid(n)
    else:
        from ai_economist_b200 import foundation, workloads
        from tests.emu.emu_stepper import emu_factory
        kw = dict(workloads.BASELINE_CONFIGS[cfg])
        name = kw.pop("scenario_name")
        twin = foundation.make_env_instance(name, n_envs=n, seeds=[0, 1], stepper_factory=emu_factory, **kw)
    assert env_shape(twin) == (n, A)
    head = lambda x: np.ascontiguousarray(x[:, :n])
    j = dict(r=tuple(head(x) for x in inp["r"]), v=tuple(head(x) for x in inp["v"]), d=head(inp["d"]),
             lv=tuple(np.ascontiguousarray(x[:n]) for x in inp["lv"]), final=tuple(head(x) for x in inp["final"]))
    host = call(twin, j, 0.998, 0.98)
    dev = env.compute_advantages(rf, (va, vp), d, (lva, lvp), (fa, fp), gamma=0.998, lam=0.98)
    for x, y in zip(host, dev):
        assert same_bits(x, np_(y)[:, :n])
    del env
    torch.cuda.empty_cache()


@pytest.mark.gpu
def test_cuda_is_asynchronous_on_the_current_stream_and_touches_nothing():
    """On a side stream the outputs are ordered after the inputs' producers; the env's buffers and counters stay put."""
    env = _cuda_gtb("c1_tutorial", 512)
    st = env.stepper
    E, A = env_shape(env)
    T = 33
    inp = random_inputs(np.random.RandomState(8), T, E, A, (np.float64, np.float64))
    dev = lambda x: None if x is None else torch.as_tensor(x, device="cuda:0")
    raw = lambda v: v.reshape(-1).view(torch.uint8).cpu()
    before = {k: raw(v) for k, v in st.buf.items()}
    n0 = st.launch_count()
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        out = env.compute_advantages(tuple(dev(x) for x in inp["r"]), tuple(dev(x) for x in inp["v"]), dev(inp["d"]),
                                     tuple(dev(x) for x in inp["lv"]), tuple(dev(x) for x in inp["final"]),
                                     gamma=0.99, lam=0.95)
    s.synchronize()
    check_outputs([x.cpu().numpy() for x in out], ref_all(inp, 0.99, 0.95))
    assert st.launch_count() == n0
    for k, v in st.buf.items():
        assert torch.equal(raw(v), before[k]), k
