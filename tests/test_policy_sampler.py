"""The policy sampler (env.sample_actions / aie_sample_policy / aie_covid_sample_policy): a policy's actions drawn on the
device from its logits under the env's current masks, with their log-probabilities.

The numpy restatement below is the contract of include/aie_b200.h: the stream (splitmix64 keys per env and segment, a
53-bit uniform), the float64 inverse CDF and the log-probability.  Actions must equal it exactly, except where u * Z lies
within 1e-12 * Z of a boundary of the cumulative sum (the accumulation order moves it by ~1e-16): such draws are counted
and must not occur at these sizes.  Log-probabilities must lie within one float32 ulp of the float64 log-softmax."""
import ctypes as C
import json
import os

import numpy as np
import pytest
import torch

from ai_economist_b200 import _abi, foundation, workloads
from oracle.configs import CONFIGS

EXCLUDE = 1e-12
U64 = 0xFFFFFFFFFFFFFFFF
ONE_STEP = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden_one_step", "isoelastic_31_seed1001.npz")
AIE_EINVAL, AIE_ESTATE = -1, -3


# ---------------------------------------------------------------------------------------------- numpy restatement
def mix64(x):
    """splitmix64 finaliser on Python ints (mod 2^64)."""
    x = (x + 0x9E3779B97F4A7C15) & U64
    x = ((x ^ (x >> 30)) * 0xBF58476D1CE4E5B9) & U64
    x = ((x ^ (x >> 27)) * 0x94D049BB133111EB) & U64
    return x ^ (x >> 31)


def call_stream(seed, call):
    """s of an env's call-th (1-based) sample_actions call."""
    return mix64(seed) ^ mix64(call)


def env_key(s, e):
    return mix64(s ^ mix64(e))


def uniform(key):
    return float(mix64(key & U64) >> 11) * 2.0 ** -53


def draw(open_, logits, u, greedy):
    """(action, float64 log-probability, near-boundary flag) of one segment under the contract."""
    open_ = np.asarray(open_, bool)
    l = np.asarray(logits, np.float32)
    if not open_.any():
        return 0, 0.0, False
    lo = l[open_]
    if np.isnan(lo).any() or (lo == np.inf).any() or not np.isfinite(lo).any():
        return int(np.argmax(open_)), float("nan"), False
    m = float(lo[np.isfinite(lo)].max())
    with np.errstate(invalid="ignore"):
        w = np.where(open_, np.exp(l.astype(np.float64) - m), 0.0)
    c = np.cumsum(w)
    Z = c[-1]
    near = False
    if greedy:
        a = int(np.argmax(open_ & (l == np.float32(m))))
    else:
        t = u * Z
        cand = np.nonzero((w > 0) & (t < c))[0]
        a = int(cand[0]) if len(cand) else int(np.nonzero(w > 0)[0][-1])
        near = bool(np.any(np.abs(t - c[w > 0]) < EXCLUDE * Z))
    return a, (float(l[a]) - m) - float(np.log(Z)), near


def log_softmax_ref(open_, logits, a):
    """float64 torch.log_softmax over the open entries of the segment, at a."""
    t = torch.as_tensor(np.asarray(logits, np.float32).astype(np.float64))
    t = t.masked_fill(~torch.as_tensor(np.asarray(open_, bool)), float("-inf"))
    return float(torch.log_softmax(t, 0)[a])


def gtb_segments(spec, dims):
    """[(who, unit, slot, offset, length, key offset)] of every mask segment of an env (who: "a" | "p"): a single-action
    agent's whole mask row, each subspace of a multi-action agent, each planner bracket (or the single index)."""
    out = []
    seg_a = workloads.mask_segments(spec, "a") if spec["multi_action_agents"] else [dims.mask_agent]
    for a in range(spec["n_agents"]):
        off = 0
        for si, n in enumerate(seg_a):
            out.append(("a", a, si, off, n, 0x100 * a + (si + 1 if spec["multi_action_agents"] else 0)))
            off += n
    n_p = dims.n_act_planner
    for b in range(n_p):
        ln = dims.mask_planner // n_p
        out.append(("p", 0, b, b * ln, ln, 0x10000 + b))
    return out


def check_segment(o, l, u, greedy, got, got_lp):
    """One segment against the restatement; returns 1 when the draw is excluded (near a boundary)."""
    a, ref_lp, near = draw(o, l, u, greedy)
    if near:
        return 1
    assert int(got) == a, (int(got), a)
    assert bool(o[a]) or not o.any()
    if not o.any():
        assert got_lp == 0.0
    elif np.isnan(ref_lp):
        assert np.isnan(got_lp)
    else:
        ref = log_softmax_ref(o, l, a)
        assert abs(float(got_lp) - ref) <= float(np.spacing(np.float32(abs(ref)))), (float(got_lp), ref)
    return 0


def as_f32(x):
    return None if x is None else (bits_to_f32(x) if x.dtype == np.uint16 else np.asarray(x, np.float32))


def check_gtb_call(spec, dims, la, lp, seed, call, greedy, acts_a, acts_p, mask_a, mask_p, lpa, lpp, envs=None):
    """Every segment of every env of one call (numpy inputs; row i is replica envs[i], default i); returns (draws,
    excluded draws)."""
    la32, lp32 = as_f32(la), as_f32(lp)
    s = call_stream(seed, call)
    n = near = 0
    for e in range(la32.shape[0]):
        k = env_key(s, e if envs is None else int(envs[e]))
        for who, unit, slot, off, ln, ko in gtb_segments(spec, dims):
            if who == "a":
                args = (mask_a[e, unit, off:off + ln] != 0, la32[e, unit, off:off + ln], uniform(k + ko), greedy,
                        acts_a[e, unit, slot], lpa[e, unit, slot])
            else:
                args = (mask_p[e, off:off + ln] != 0, lp32[e, off:off + ln], uniform(k + ko), greedy,
                        acts_p[e, slot], lpp[e, slot])
            near += check_segment(*args)
            n += 1
    return n, near


def check_covid_call(la, lp, seed, call, greedy, acts_a, acts_p, mask_a, mask_p, lpa, lpp, envs=None):
    la32, lp32 = as_f32(la), as_f32(lp)
    s = call_stream(seed, call)
    n = near = 0
    for e in range(la32.shape[0]):
        k = env_key(s, e if envs is None else int(envs[e]))
        for a in range(la32.shape[1]):
            near += check_segment(mask_a[e, :, a] != 0, la32[e, a], uniform(k + 0x100 * a), greedy, acts_a[e, a], lpa[e, a])
        near += check_segment(mask_p[e] != 0, lp32[e], uniform(k ^ 0xABCDEF), greedy, acts_p[e], lpp[e])
        n += la32.shape[1] + 1
    return n, near


def bits_to_f32(a):
    return (np.asarray(a).astype(np.uint32) << 16).view(np.float32)


def to_bf16_bits(a):
    return torch.as_tensor(np.asarray(a, np.float32)).bfloat16().view(torch.int16).numpy().view(np.uint16)


def random_logits(rng, shape, p_ninf=0.1, scale=3.0):
    l = (rng.standard_normal(shape) * scale).astype(np.float32)
    l[rng.random_sample(shape) < p_ninf] = -np.inf
    return l


# ---------------------------------------------------------------------------------------------- fixtures
def gtb_kwargs(cfg):
    if cfg == "one_step":   # one-step-economy: 31 agents x 101 labor levels, 7 planner brackets x 22 rates
        kw = dict(json.loads(str(np.load(ONE_STEP)["meta_json"]))["reference_kwargs"])
        kw["components"] = [tuple(c) for c in kw["components"]]
        return kw
    return dict(CONFIGS[cfg])


def make_env(cfg, n_envs, factory=None, obs_dtype=None, **over):
    kw = gtb_kwargs(cfg)
    kw.update(over)
    name = kw.pop("scenario_name")
    dev = dict(stepper_factory=factory) if factory else dict(device="cuda:0")
    env = foundation.make_env_instance(name, n_envs=n_envs, seeds=list(range(n_envs)), obs_dtype=obs_dtype, **dev, **kw)
    env.reset()
    return env


def emu_env(cfg, n_envs=4, obs_dtype=None, **over):
    from tests.emu.emu_stepper import emu_factory
    return make_env(cfg, n_envs, emu_factory, obs_dtype, **over)


def logit_shapes(env):
    d, E, A = env.stepper.dims, env.n_envs, env.n_agents
    return (E, A, d.mask_agent), ((E, d.mask_planner) if d.n_act_planner else None)


def outputs(st):
    """(agent actions, planner actions, agent mask, planner mask) as numpy (masks as float32)."""
    return (st.to_numpy(st.buf["actions_agent"]).copy(), st.to_numpy(st.buf["actions_planner"]).copy(),
            st.obs_to_numpy("mask_agent").copy(), st.obs_to_numpy("mask_planner").copy())


def np_(st, x):
    return None if x is None else st.to_numpy(x).copy()


# ---------------------------------------------------------------------------------------------- CPU (emulation)
EXACT_CFGS = [("c1_tutorial", None), ("tax_us_federal", None), ("c3_reset", None), ("tax_single_planner", None),
              ("c5_small", None), ("one_step", None), ("tax_us_federal", torch.bfloat16)]


@pytest.mark.parametrize("greedy", [False, True])
@pytest.mark.parametrize("cfg,obs_dtype", EXACT_CFGS, ids=lambda v: str(v).replace("torch.", ""))
def test_emulated_actions_and_log_probs_match_the_restatement(cfg, obs_dtype, greedy):
    env = emu_env(cfg, n_envs=3 if cfg in ("c5_small", "one_step") else 4, obs_dtype=obs_dtype)
    st, rng, seed = env.stepper, np.random.RandomState(7), 1234
    sa, sp = logit_shapes(env)
    total = near = 0
    for call in range(1, 5):   # a few steps: the masks change between calls
        la = random_logits(rng, sa)
        lp = random_logits(rng, sp) if sp else None
        _, _, mask_a, mask_p = outputs(st)
        lpa, lpp = env.sample_actions(la, lp, seed=seed, greedy=greedy)
        aa, ap, _, _ = outputs(st)
        n, k = check_gtb_call(env.spec, st.dims, la, lp, seed, call, greedy, aa, ap, mask_a, mask_p,
                              np_(st, lpa), np_(st, lpp))
        total, near = total + n, near + k
        env.step(env.action_buffers)
    assert total > 0 and near == 0


@pytest.mark.parametrize("cfg", ["tax_us_federal", "c5_small", "one_step"])
def test_emulated_bf16_logits_give_the_float32_call_on_their_values(cfg):
    """bfloat16 logits: byte-identical actions and log-probabilities to a float32 call on logits.bfloat16().float()."""
    e1, e2 = emu_env(cfg, n_envs=3), emu_env(cfg, n_envs=3)
    rng = np.random.RandomState(3)
    sa, sp = logit_shapes(e1)
    for _ in range(3):
        la = to_bf16_bits(random_logits(rng, sa))
        lp = to_bf16_bits(random_logits(rng, sp)) if sp else None
        r1 = [np_(e1.stepper, x) for x in e1.sample_actions(la, lp, seed=5)]
        r2 = [np_(e2.stepper, x) for x in e2.sample_actions(bits_to_f32(la), as_f32(lp), seed=5)]
        for x, y in zip(r1, r2):
            assert (x is None and y is None) or x.tobytes() == y.tobytes()
        assert outputs(e1.stepper)[0].tobytes() == outputs(e2.stepper)[0].tobytes()
        assert outputs(e1.stepper)[1].tobytes() == outputs(e2.stepper)[1].tobytes()
        e1.step(e1.action_buffers)
        e2.step(e2.action_buffers)


def test_emulated_edge_segments():
    """All-closed, NaN / +inf / all -inf segments, -inf entries never drawn, greedy = masked argmax; every action open."""
    env = emu_env("c1_tutorial", n_envs=4)
    st = env.stepper
    sa, _ = logit_shapes(env)
    ma = st.buf["mask_agent"]
    rng = np.random.RandomState(0)
    ma[0, 0, :] = 0.0                              # env 0 agent 0: nothing open
    la = random_logits(rng, sa, p_ninf=0.0)
    open1 = np.nonzero(ma[1, 0])[0]
    la[1, 0, open1[-1]] = np.nan                   # env 1 agent 0: a NaN open logit
    la[1, 1, 0] = np.inf                           # env 1 agent 1: +inf at the NO-OP (always open)
    la[2, 0, :] = -np.inf                          # env 2 agent 0: every logit -inf
    open3 = np.nonzero(ma[3, 0])[0]
    la[3, 0, open3[1:]] = -np.inf                  # env 3 agent 0: one finite open entry -> always drawn
    la[1, 0, :open1[-1]][ma[1, 0, :open1[-1]] == 0] = np.nan   # NaN at closed entries is ignored elsewhere
    for call in range(1, 30):
        lpa, _ = env.sample_actions(la, None, seed=9)
        aa = st.to_numpy(st.buf["actions_agent"])[..., 0]
        lp = st.to_numpy(lpa)[..., 0]
        assert aa[0, 0] == 0 and lp[0, 0] == 0.0
        assert aa[1, 0] == open1[0] and np.isnan(lp[1, 0])
        assert aa[1, 1] == np.nonzero(ma[1, 1])[0][0] and np.isnan(lp[1, 1])
        assert aa[2, 0] == np.nonzero(ma[2, 0])[0][0] and np.isnan(lp[2, 0])
        assert aa[3, 0] == open3[0] and lp[3, 0] == 0.0
        for e in range(4):
            for a in range(env.n_agents):
                if ma[e, a].any():
                    assert ma[e, a, aa[e, a]] == 1.0
                    assert not (e == 3 and a == 0) or aa[e, a] == open3[0]
    la2 = random_logits(rng, sa, p_ninf=0.3)
    env.sample_actions(la2, None, seed=1, greedy=True)
    aa = st.to_numpy(st.buf["actions_agent"])[..., 0]
    for e in range(1, 4):
        for a in range(env.n_agents):
            o = ma[e, a] != 0
            if o.any() and np.isfinite(la2[e, a][o]).any():
                assert aa[e, a] == int(np.argmax(np.where(o, la2[e, a], -np.inf)))


def test_emulated_draws_follow_the_softmax():
    """Fixed masks and logits, 24 000 calls: per-entry frequencies pass a chi-square test against the masked softmax,
    and closed or -inf entries are never drawn."""
    from scipy import stats
    env = emu_env("c1_tutorial", n_envs=2)
    st = env.stepper
    sa, _ = logit_shapes(env)
    rng = np.random.RandomState(42)
    la = (rng.standard_normal(sa) * 0.7).astype(np.float32)
    ma = st.obs_to_numpy("mask_agent")
    ninf = np.nonzero(ma[0, 1])[0][-1]
    la[0, 1, ninf] = -np.inf
    counts = np.zeros(sa, np.int64)
    n_calls = 24000
    for _ in range(n_calls):
        env.sample_actions(la, None, seed=2024)
        aa = st.buf["actions_agent"][..., 0]
        for e in range(sa[0]):
            counts[e, np.arange(sa[1]), aa[e]] += 1
    assert counts[0, 1, ninf] == 0
    for e in range(sa[0]):
        for a in range(sa[1]):
            o = (ma[e, a] != 0) & np.isfinite(la[e, a])
            assert counts[e, a][~o].sum() == 0
            if o.sum() < 2:
                continue
            p = np.exp(la[e, a][o].astype(np.float64) - la[e, a][o].max())
            p /= p.sum()
            assert stats.chisquare(counts[e, a][o], p * n_calls).pvalue > 1e-4


def _rollout(seed, steps=14, obs_dtype=None):
    """sample_actions then step(env.action_buffers), 14 steps of 25-step episodes started at t = 0, 8, 16: the bytes of
    every step's actions, masks, rewards, done flags, flat observations and log-probabilities, and the episode ends seen."""
    env = emu_env("c1_reset", n_envs=3, obs_dtype=obs_dtype)
    st = env.stepper
    st.state_view("t")[...] = np.array([0, 8, 16], np.int32)
    sa, _ = logit_shapes(env)
    rng = np.random.RandomState(seed)
    out, ends = [], 0
    for _ in range(steps):
        la = random_logits(rng, sa)
        if obs_dtype is not None:
            la = to_bf16_bits(la)
        lpa, _ = env.sample_actions(la, None, seed=seed)
        env.step(env.action_buffers)
        out += [st.to_numpy(st.buf[k]).tobytes() for k in ("actions_agent", "mask_agent", "reward", "done", "obs_agent_flat")]
        out.append(st.to_numpy(lpa).tobytes())
        ends += int(st.to_numpy(st.buf["done"]).sum())
    return out, ends


@pytest.mark.parametrize("obs_dtype", [None, torch.bfloat16], ids=["float32", "bfloat16"])
def test_emulated_rollouts_are_deterministic_across_episode_ends(obs_dtype):
    r1, ends = _rollout(77, obs_dtype=obs_dtype)
    r2, _ = _rollout(77, obs_dtype=obs_dtype)
    assert ends >= 1 and r1 == r2
    r3, _ = _rollout(78, obs_dtype=obs_dtype)
    assert r1 != r3


def test_emulated_call_counter_is_separate_from_the_random_sampler():
    e1, e2 = emu_env("c3_reset", n_envs=2), emu_env("c3_reset", n_envs=2)
    sa, sp = logit_shapes(e1)
    rng = np.random.RandomState(1)
    la, lp = random_logits(rng, sa), random_logits(rng, sp)
    e2.stepper.sample_random_actions(seed=3)   # does not move the policy sampler's counter
    r1 = [np_(e1.stepper, x) for x in e1.sample_actions(la, lp, seed=8)]
    r2 = [np_(e2.stepper, x) for x in e2.sample_actions(la, lp, seed=8)]
    assert all(x.tobytes() == y.tobytes() for x, y in zip(r1, r2))
    assert outputs(e1.stepper)[0].tobytes() == outputs(e2.stepper)[0].tobytes()
    r3 = [np_(e1.stepper, x) for x in e1.sample_actions(la, lp, seed=8)]   # second call: a new stream
    assert r3[0].tobytes() != r1[0].tobytes()


def test_emulated_out_destinations_and_value_errors():
    env = emu_env("c3_reset", n_envs=2)
    st = env.stepper
    sa, sp = logit_shapes(env)
    d = st.dims
    rng = np.random.RandomState(4)
    la, lp = random_logits(rng, sa), random_logits(rng, sp)
    own_a, own_p = env.sample_actions(la, lp, seed=1)
    again = env.sample_actions(la, lp, seed=1)
    assert again[0] is own_a and again[1] is own_p            # library-owned buffers are reused
    assert own_a.shape == (2, env.n_agents, d.n_act_agent) and own_p.shape == (2, d.n_act_planner)
    oa, op = np.full(own_a.shape, 7, np.float32), np.full(own_p.shape, 7, np.float32)
    ga, gp = env.sample_actions(la, lp, seed=1, out=(oa, op))
    assert ga is oa and gp is op and not (oa == 7).any() and not (op == 7).any()
    ga, gp = env.sample_actions(la, lp, seed=1, out=(None, op))
    assert ga is own_a and gp is op
    bad = [
        dict(logits_agent=la[:, :-1]),                                     # shape
        dict(logits_agent=la.astype(np.float64)),                          # dtype
        dict(logits_agent=np.asfortranarray(la)),                          # contiguity
        dict(logits_planner=None),                                         # planner actions need planner logits
        dict(logits_planner=to_bf16_bits(lp)),                             # dtypes differ
        dict(out=(np.zeros(own_a.shape, np.float64), None)),
        dict(out=(None, np.zeros((2, 1), np.float32))),
    ]
    for b in bad:
        kw = dict(logits_agent=la, logits_planner=lp, out=None)
        kw.update(b)
        with pytest.raises(ValueError):
            env.sample_actions(kw["logits_agent"], kw["logits_planner"], seed=1, out=kw["out"])
    # no planner actions: planner logits are ignored, log_prob_planner is None
    env1 = emu_env("c1_tutorial", n_envs=2)
    sa1, sp1 = logit_shapes(env1)
    assert sp1 is None and env1.sample_actions(random_logits(rng, sa1), "ignored", seed=2)[1] is None


def test_abi_errors():
    from tests.emu.emu_stepper import emu_factory, emu_lib
    lib = emu_lib()
    kw = gtb_kwargs("c3_reset")
    name = kw.pop("scenario_name")
    env = foundation.make_env_instance(name, n_envs=2, seeds=[0, 1], stepper_factory=emu_factory, **kw)
    st = env.stepper
    sa, sp = logit_shapes(env)
    la, lp = np.zeros(sa, np.float32), np.zeros(sp, np.float32)
    lpa = np.zeros(st.buf["actions_agent"].shape, np.float32)

    def p(**over):
        q = _abi.AiePolicyLogits()
        q.agent, q.planner = la.ctypes.data, lp.ctypes.data
        q.logits_dtype, q.greedy = _abi.OBS_F32, 0
        q.log_prob_agent = lpa.ctypes.data
        for k, v in over.items():
            setattr(q, k, v)
        return C.byref(q)

    call = lambda q: lib.aie_sample_policy(st._h, q, C.c_uint64(1), None)
    assert call(p()) == AIE_ESTATE                         # nothing loaded yet
    env.reset()
    assert call(p()) == 0
    assert call(None) == AIE_EINVAL
    assert call(p(agent=None)) == AIE_EINVAL
    assert call(p(planner=None)) == AIE_EINVAL
    assert call(p(logits_dtype=7)) == AIE_EINVAL
    assert call(p(greedy=2)) == AIE_EINVAL
    assert call(p(agent=la.ctypes.data + 2)) == AIE_EINVAL
    assert call(p(agent=la.ctypes.data + 2, logits_dtype=_abi.OBS_BF16)) == 0   # bfloat16: 2-byte alignment
    assert call(p(agent=la.ctypes.data + 1, logits_dtype=_abi.OBS_BF16)) == AIE_EINVAL
    assert call(p(log_prob_agent=lpa.ctypes.data + 2)) == AIE_EINVAL
    assert call(p(log_prob_agent=None)) == 0
    assert lib.aie_sample_policy(None, p(), C.c_uint64(1), None) == AIE_EINVAL


# ---------------------------------------------------------------------------------------------- COVID-19
def covid_env(n_envs, factory=None):
    from oracle.gen_golden_covid import COVID_KWARGS, reference_config
    cfg = reference_config(COVID_KWARGS)
    name = cfg.pop("scenario_name")
    dev = dict(stepper_factory=factory) if factory else dict(device="cuda:0")
    env = foundation.make_env_instance(name, n_envs=n_envs, auto_reset=True, **dev, **cfg)
    env.reset()
    return env


def emu_covid(n_envs=3):
    from tests.emu.emu_stepper import EmuCovidStepper
    return covid_env(n_envs, lambda params, n, ar: EmuCovidStepper(params, n, ar))


def covid_shapes(env):
    st = env.stepper
    return ((env.n_envs, env.n_agents, 1 + st.p["num_stringency_levels"]), (env.n_envs, 1 + st.p["num_subsidy_levels"]))


@pytest.mark.parametrize("greedy", [False, True])
@pytest.mark.parametrize("bf16", [False, True])
def test_emulated_covid_matches_the_restatement(greedy, bf16):
    env = emu_covid()
    st = env.stepper
    sa, sp = covid_shapes(env)
    rng = np.random.RandomState(5)
    total = near = 0
    for call in range(1, 5):
        la, lp = random_logits(rng, sa), random_logits(rng, sp)
        if call == 2:
            la[0, 3] = -np.inf
            lp[1, 2] = np.nan
        if bf16:
            la, lp = to_bf16_bits(la), to_bf16_bits(lp)
        mask_a, mask_p = st.to_numpy(st.buf["mask_agent"]).copy(), st.to_numpy(st.buf["mask_planner"]).copy()
        lpa, lpp = env.sample_actions(la, lp, seed=31, greedy=greedy)
        aa, ap = st.to_numpy(st.buf["actions_agent"]), st.to_numpy(st.buf["actions_planner"])
        n, k = check_covid_call(la, lp, 31, call, greedy, aa, ap, mask_a, mask_p, st.to_numpy(lpa), st.to_numpy(lpp))
        total, near = total + n, near + k
        for _ in range(30):   # the stringency cooldown closes and reopens entries of the agent masks
            env.step(env.action_buffers)
    assert total > 0 and near == 0


def test_emulated_covid_errors():
    from tests.emu.emu_stepper import emu_lib
    env = emu_covid(2)
    sa, sp = covid_shapes(env)
    la, lp = np.zeros(sa, np.float32), np.zeros(sp, np.float32)
    with pytest.raises(ValueError):
        env.sample_actions(la, None, seed=1)
    with pytest.raises(ValueError):
        env.sample_actions(la.transpose(0, 2, 1).copy(), lp, seed=1)
    with pytest.raises(ValueError):
        env.sample_actions(la, lp, seed=1, out=(np.zeros((2, 51), np.float64), None))
    a, p = env.sample_actions(la, lp, seed=1)
    assert a.shape == (2, 51) and p.shape == (2,)
    lib = emu_lib()
    q = _abi.AiePolicyLogits()
    q.agent, q.planner, q.logits_dtype = la.ctypes.data, None, _abi.OBS_F32
    assert lib.aie_covid_sample_policy(env.stepper._h, C.byref(q), C.c_uint64(1), None) == AIE_EINVAL
    q.planner, q.greedy = lp.ctypes.data, 3
    assert lib.aie_covid_sample_policy(env.stepper._h, C.byref(q), C.c_uint64(1), None) == AIE_EINVAL
    q.greedy = 1
    assert lib.aie_covid_sample_policy(env.stepper._h, C.byref(q), C.c_uint64(1), None) == 0


# ---------------------------------------------------------------------------------------------- GPU
def _stagger(env):
    """Episode phases as in bench.py: replica e starts at t = e * T / E."""
    st, E, T = env.stepper, env.n_envs, int(env.episode_length)
    st.state_view("t").copy_((torch.arange(E, device="cuda:0", dtype=torch.int64) * T // E).to(torch.int32))


def _np_logits(x):
    """numpy form of a device logits tensor: float32, or the raw bits of bfloat16."""
    if x is None:
        return None
    return x.view(torch.int16).cpu().numpy().view(np.uint16) if x.dtype == torch.bfloat16 else x.cpu().numpy()


def _np_mask(st, name, n):
    """The first n rows of a device mask in the emulation's storage (float32, or bfloat16 bits)."""
    x = st.buf[name][:n]
    return _np_logits(x) if x.dtype == torch.bfloat16 else x.cpu().numpy()


def _close_lp(a, b):
    """Log-probabilities equal within one float32 ulp (NaN where the other is NaN)."""
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    return bool(np.all((np.abs(a - b) <= np.spacing(np.abs(a))) | (np.isnan(a) & np.isnan(b))))


def _gpu_logits(shape, dt, g):
    x = torch.randn(shape, device="cuda:0", generator=g) * 3
    x[torch.rand(shape, device="cuda:0", generator=g) < 0.1] = float("-inf")
    return x.to(dt)


GPU_CFGS = [("c1_tutorial", 8192), ("c3_paper_tax", 8192), ("c5_full", 2048)]
MODES = [(torch.float32, False), (torch.bfloat16, False), (torch.float32, True), (torch.bfloat16, True)]


def _gtb_cuda(cfg, E, obs_dtype):
    kw = dict(workloads.BASELINE_CONFIGS[cfg])
    name = kw.pop("scenario_name")
    if cfg == "c5_full":
        kw["device_reset"] = "snapshot"
    env = foundation.make_env_instance(name, n_envs=E, device="cuda:0", seeds=list(range(E)), obs_dtype=obs_dtype, **kw)
    env.reset()
    _stagger(env)
    env.stepper.set_fused_policy(5)   # a few random steps: masks of different phases
    for _ in range(3):
        env.step(env.action_buffers)
    env.stepper.set_fused_policy(0)
    return env, name, kw


@pytest.mark.gpu
@pytest.mark.parametrize("obs_dtype", [None, torch.bfloat16], ids=["f32_masks", "bf16_masks"])
@pytest.mark.parametrize("cfg,E", GPU_CFGS, ids=[c for c, _ in GPU_CFGS])
def test_cuda_full_size_matches_restatement_and_emulation(cfg, E, obs_dtype):
    """Full size, staggered episodes, float32 and bfloat16 logits, stochastic and greedy: actions byte-identical to the
    numpy restatement (a sample of replicas, under the exclusion rule) and to the emulation run on the same masks and
    logits (the first replicas); log-probabilities within one float32 ulp of both."""
    from tests.emu.emu_stepper import emu_factory
    env, name, kw = _gtb_cuda(cfg, E, obs_dtype)
    st = env.stepper
    sa, sp = logit_shapes(env)
    n_emu = 8 if cfg == "c5_full" else 64
    twin = foundation.make_env_instance(name, n_envs=n_emu, stepper_factory=emu_factory, seeds=list(range(n_emu)),
                                        obs_dtype=obs_dtype, **kw)
    twin.reset()
    tst = twin.stepper
    g = torch.Generator(device="cuda:0").manual_seed(0)
    pick = np.r_[0:8, E // 2:E // 2 + 4, E - 8:E]
    total = near = 0
    for call, (ldt, greedy) in enumerate(MODES, start=1):
        la = _gpu_logits(sa, ldt, g)
        lp = _gpu_logits(sp, ldt, g) if sp else None
        mask_a, mask_p = st.obs_to_numpy("mask_agent"), st.obs_to_numpy("mask_planner")
        lpa, lpp = env.sample_actions(la, lp, seed=99, greedy=greedy)
        aa, ap = st.to_numpy(st.buf["actions_agent"]), st.to_numpy(st.buf["actions_planner"])
        lpa_n = st.to_numpy(lpa)
        lpp_n = st.to_numpy(lpp) if lpp is not None else None
        la_n, lp_n = _np_logits(la), _np_logits(lp)
        n, k = check_gtb_call(env.spec, st.dims, la_n[pick], None if lp_n is None else lp_n[pick], 99, call,
                              greedy, aa[pick], ap[pick], mask_a[pick], mask_p[pick], lpa_n[pick],
                              None if lpp_n is None else lpp_n[pick], envs=pick)
        total, near = total + n, near + k
        # the emulation on the same masks and logits, same call index
        tst.buf["mask_agent"][...] = _np_mask(st, "mask_agent", n_emu)
        tst.buf["mask_planner"][...] = _np_mask(st, "mask_planner", n_emu)
        ta, tp = twin.sample_actions(la_n[:n_emu], None if lp_n is None else lp_n[:n_emu], seed=99, greedy=greedy)
        assert tst.buf["actions_agent"].tobytes() == aa[:n_emu].tobytes()
        assert _close_lp(ta, lpa_n[:n_emu])
        if sp:
            assert tst.buf["actions_planner"].tobytes() == ap[:n_emu].tobytes()
            assert _close_lp(tp, lpp_n[:n_emu])
        env.step(env.action_buffers)
    assert total > 0 and near == 0


def _cuda_calls(env, sa, sp, n=3):
    """The outputs of n calls with fixed logits (stochastic), one step after each."""
    st, out = env.stepper, []
    g = torch.Generator(device="cuda:0").manual_seed(1)
    for _ in range(n):
        la = _gpu_logits(sa, torch.float32, g)
        lp = _gpu_logits(sp, torch.float32, g) if sp else None
        lpa, lpp = env.sample_actions(la, lp, seed=7)
        out += [st.to_numpy(st.buf["actions_agent"]).tobytes(), st.to_numpy(st.buf["actions_planner"]).tobytes(),
                st.to_numpy(lpa).tobytes(), b"" if lpp is None else st.to_numpy(lpp).tobytes()]
        env.step(env.action_buffers)
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("cfg,E", [("c1_tutorial", 8192), ("c3_paper_tax", 8192)])
def test_cuda_same_calls_give_the_same_bytes(cfg, E):
    runs = []
    for _ in range(2):
        env, _, _ = _gtb_cuda(cfg, E, None)
        sa, sp = logit_shapes(env)
        runs.append(_cuda_calls(env, sa, sp))
        del env
        torch.cuda.empty_cache()
    assert runs[0] == runs[1]


@pytest.mark.gpu
def test_cuda_covid_full_size():
    """COVID-19 at 4 096 replicas, staggered, both logits dtypes, stochastic and greedy: restatement (sampled replicas),
    emulation (first replicas) and a second identical run."""
    from tests.emu.emu_stepper import EmuCovidStepper
    E, n_emu = 4096, 16

    def staggered():
        env = covid_env(E)
        T = int(env.episode_length)
        env.stepper.buf["hdr"][:, 0] = (torch.arange(E, device="cuda:0") * T // E).to(torch.int32)
        for _ in range(3):
            env.stepper.sample_random_actions(seed=3)
            env.step(env.action_buffers)
        return env

    env = staggered()
    st = env.stepper
    twin = emu_covid(n_emu)
    tst = twin.stepper
    sa, sp = covid_shapes(env)
    g = torch.Generator(device="cuda:0").manual_seed(2)
    pick = np.r_[0:8, E - 8:E]
    total = near = 0
    record = []
    for call, (ldt, greedy) in enumerate(MODES, start=1):
        la, lp = _gpu_logits(sa, ldt, g), _gpu_logits(sp, ldt, g)
        mask_a, mask_p = st.to_numpy(st.buf["mask_agent"]), st.to_numpy(st.buf["mask_planner"])
        lpa, lpp = env.sample_actions(la, lp, seed=41, greedy=greedy)
        aa, ap = st.to_numpy(st.buf["actions_agent"]), st.to_numpy(st.buf["actions_planner"])
        lpa_n, lpp_n = st.to_numpy(lpa), st.to_numpy(lpp)
        record += [aa.tobytes(), ap.tobytes(), lpa_n.tobytes(), lpp_n.tobytes()]
        la_n, lp_n = _np_logits(la), _np_logits(lp)
        n, k = check_covid_call(la_n[pick], lp_n[pick], 41, call, greedy, aa[pick], ap[pick], mask_a[pick], mask_p[pick],
                                lpa_n[pick], lpp_n[pick], envs=pick)
        total, near = total + n, near + k
        tst.buf["mask_agent"][...] = mask_a[:n_emu]
        tst.buf["mask_planner"][...] = mask_p[:n_emu]
        ta, tp = twin.sample_actions(la_n[:n_emu], lp_n[:n_emu], seed=41, greedy=greedy)
        assert tst.buf["actions_agent"].tobytes() == aa[:n_emu].tobytes()
        assert tst.buf["actions_planner"].tobytes() == ap[:n_emu].tobytes()
        assert _close_lp(ta, lpa_n[:n_emu]) and _close_lp(tp, lpp_n[:n_emu])
        env.step(env.action_buffers)
    assert total > 0 and near == 0
    del env
    torch.cuda.empty_cache()
    env2 = staggered()
    g = torch.Generator(device="cuda:0").manual_seed(2)
    again = []
    for ldt, greedy in MODES:
        la, lp = _gpu_logits(sa, ldt, g), _gpu_logits(sp, ldt, g)
        lpa, lpp = env2.sample_actions(la, lp, seed=41, greedy=greedy)
        st2 = env2.stepper
        again += [st2.to_numpy(st2.buf["actions_agent"]).tobytes(), st2.to_numpy(st2.buf["actions_planner"]).tobytes(),
                  st2.to_numpy(lpa).tobytes(), st2.to_numpy(lpp).tobytes()]
        env2.step(env2.action_buffers)
    assert again == record
