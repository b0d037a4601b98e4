"""The COVID-19 step kernel across its parameter space, its episode ends and its batch sizes.

Fixtures: tests/golden/covid_variants/<name>.npz, recorded from the unmodified reference by
`python oracle/gen_golden_covid.py --variant <name> --check` for each entry of its VARIANTS table.  Each trace runs
across two episode ends: the step that ends an episode carries that step's rewards and `done`, and the observation
of the fresh episode (what the auto-reset returns).

CPU: the numpy oracle and the device source compiled for the host (tests/emu) step through every trace, the traced
replica inside a batch; the change list is held to the history window's changes at every step; the random policy is
uniform over the open entries.
GPU: the CUDA kernel against every trace (traced replicas at the ends and the middle of a batch of 257), against the
oracle and the emulation on batches across two auto-resets, with the change list overflowing, at full size across
the episode ends the benchmark crosses, and its random policy against the emulation's.

Tolerance as tests/test_covid.py: float32 fields <= 1e-6 relative (atol 1e-9); masks, `done` and integers exact.  One
exception: the rewards of an eta whose x ** (1 - eta) takes no fast path (see REW_ATOL_GENERAL_POW).
"""
import json

import numpy as np
import pytest

from ai_economist_b200.foundation.covid19 import build_covid_params
from oracle.covid_oracle import CovidOracleEnv
from oracle.gen_golden_covid import COVID_KWARGS, VARIANTS, variant_kwargs, variant_path

OBS_KEYS = ["agent_state", "postsubsidy", "lagged", "policy_ind", "scalars", "mask_a", "mask_p"]
ST_KEYS = ["susceptible", "infected", "deaths", "unemployed", "stringency", "subsidy"]   # the traces' st_* series
FLOAT_STATE = ["susceptible", "infected", "recovered", "deaths", "vaccinated", "unemployed", "subsidy", "postsubsidy"]
RTOL, ATOL = 1e-6, 1e-9
NAMES = sorted(VARIANTS)
OUT_BUFS = ["obs_agent_state", "obs_postsubsidy", "obs_lagged_stringency", "obs_policy_indicators", "obs_scalars",
            "mask_agent", "mask_planner", "reward_agent", "reward_planner", "done", "state", "ints", "hdr"]
INT_BUFS = ["ints", "hdr", "ring", "changes", "mask_agent", "mask_planner", "done"]     # equal bit for bit across backends
LIST_CAP, LIST_DAY0 = 32, 1 << 20                                                     # aie_covid_core.cuh
# numpy's float32 power (its AVX-512 routine on x86), glibc's powf (the emulation) and CUDA's powf are each within 1 ulp
# of the correctly rounded power and differ from it, and from each other, for about one argument in five (measured on
# 2e6 arguments in [0.1, 3] for the exponents -2 and -0.5, on an H100 80GB HBM3).  The min-max normalisation of the agent
# reward turns that ulp of a power up to 0.1 ** -2 = 100 into an absolute error of up to 9.5e-7 on these traces (planner
# rewards: none).  Observations are not affected.
REW_ATOL_GENERAL_POW = 2e-6


def rew_atol(p):
    return ATOL if float(1 - np.float32(p["crra_eta"])) in (-1.0, 2.0, 0.5, 1.0, 0.0) else REW_ATOL_GENERAL_POW


def load(name):
    z = np.load(variant_path(name))
    meta = json.loads(str(z["meta_json"]))
    return z, meta, build_covid_params(**meta["kwargs"])


# ---------------------------------------------------------------------------------------------------- helpers
def snapshot(s, extra=()):
    return {k: s.to_numpy(s.buf[k]) for k in OUT_BUFS + [k for k in extra if k in s.buf]}


def obs_of(snap, e):
    return dict(agent_state=snap["obs_agent_state"][e], postsubsidy=snap["obs_postsubsidy"][e],
                lagged=snap["obs_lagged_stringency"][e], policy_ind=snap["obs_policy_indicators"][e],
                scalars=snap["obs_scalars"][e], mask_a=snap["mask_agent"][e], mask_p=snap["mask_planner"][e],
                rew_a=snap["reward_agent"][e], rew_p=np.float64(snap["reward_planner"][e]), done=np.int32(snap["done"][e]))


def state_of(snap, e):
    st, ints, hdr = snap["state"][e], snap["ints"][e], snap["hdr"][e]
    names = ["susceptible", "infected", "recovered", "deaths", "vaccinated", "unemployed", "stringency", "subsidy", "postsubsidy"]
    out = {n: st[i] for i, n in enumerate(names)}
    out.update(t=int(hdr[0]), subsidy_level=int(hdr[1]), cooldown_until=ints[0], vaccines_available=ints[1], episodes=int(hdr[3]))
    return out


def random_actions(rng, snap):
    """uniform over each state's / the planner's unmasked actions"""
    ma, mp = snap["mask_agent"], snap["mask_planner"]
    aa = np.argmax(ma * (rng.random_sample(ma.shape) + 1e-3), axis=1).astype(np.int32)
    ap = np.argmax(mp * (rng.random_sample(mp.shape) + 1e-3), axis=1).astype(np.int32)
    return aa, ap


def set_actions(s, aa, ap):
    ba, bp = s.buf["actions_agent"], s.buf["actions_planner"]
    if isinstance(ba, np.ndarray):
        ba[...] = aa; bp[...] = ap
    else:
        import torch
        ba.copy_(torch.from_numpy(np.ascontiguousarray(aa))); bp.copy_(torch.from_numpy(np.ascontiguousarray(ap)))


def episode_clock(z, n):
    """(t within the episode, auto-resets so far) of every step 0..n of a trace"""
    t_ep, eps = [0], [0]
    for i in range(1, n + 1):
        d = int(z["done"][i - 1])
        t_ep.append(0 if d else t_ep[-1] + 1)
        eps.append(eps[-1] + d)
    return t_ep, eps


def check_obs(want, got, label, rewards=True, ratol=ATOL):
    for k in OBS_KEYS:
        assert np.allclose(want[k], got[k], rtol=RTOL, atol=ATOL), "%s: %s" % (label, k)
    assert np.array_equal(want["mask_a"], got["mask_a"]) and np.array_equal(want["mask_p"], got["mask_p"]), label
    if rewards:
        assert np.allclose(want["rew_a"], got["rew_a"], rtol=RTOL, atol=ratol), "%s: rew_a" % label
        assert np.isclose(float(want["rew_p"]), float(got["rew_p"]), rtol=RTOL, atol=ratol), "%s: rew_p" % label
        assert int(want["done"]) == int(got["done"]), "%s: done" % label


def trace_obs(z, t):
    o = {k: z[k][t] for k in OBS_KEYS}
    if t:
        o.update(rew_a=z["rew_a"][t - 1], rew_p=z["rew_p"][t - 1], done=z["done"][t - 1])
    return o


def check_trace_step(z, clock, t, obs, st, label, ratol=ATOL):
    check_obs(trace_obs(z, t), obs, "%s step %d" % (label, t), rewards=t > 0, ratol=ratol)
    for k in ST_KEYS:
        assert np.allclose(z["st_" + k][t], st[k], rtol=RTOL, atol=ATOL), "%s step %d: state %s" % (label, t, k)
    assert np.array_equal(z["st_stringency"][t], st["stringency"]), "%s step %d" % (label, t)
    assert (st["t"], st["episodes"]) == (clock[0][t], clock[1][t]), "%s step %d: (t, episodes)" % (label, t)


def check_oracle_state(want, got, label):
    for k in FLOAT_STATE:
        assert np.allclose(want[k], got[k], rtol=RTOL, atol=ATOL), "%s: state %s" % (label, k)
    assert np.array_equal(want["stringency"], got["stringency"]), label
    for k in ["cooldown_until", "vaccines_available"]:
        assert np.array_equal(np.asarray(want[k], np.int64), np.asarray(got[k], np.int64)), "%s: %s" % (label, k)
    for k in ["t", "episodes", "subsidy_level"]:
        assert int(want[k]) == int(got[k]), "%s: %s" % (label, k)


def window_changes(ring_e, head, L):
    """[(index, change)] per state of the logical history window (oldest first), as the scan finds them"""
    L1 = L + 1
    win = ring_e[:, (head + np.arange(L1)) % L1].astype(np.int64)
    d = np.diff(win, axis=1)
    return [[(int(k), int(d[a, k])) for k in np.nonzero(d[a])[0]] for a in range(win.shape[0])]


def decoded_list(chg_e, t, L):
    """(count, [(index, change)] oldest first) per state of one replica's persistent change list"""
    chg_e = chg_e.view(np.uint32)
    out = []
    for a in range(chg_e.shape[1]):
        hd = int(chg_e[0, a])
        lhead, cnt = hd & 0xFF, (hd >> 8) & 0xFF
        entries = []
        for i in range(cnt if cnt != 255 else 0):
            en = int(chg_e[1 + (lhead + i) % LIST_CAP, a])
            tc, d = (en & 0xFFFFFF) - LIST_DAY0, (en >> 24) - 128
            entries.append((L - 1 - (t - tc), d))
        out.append((cnt, entries))
    return out


def check_change_lists(snap, L, label):
    """every list that has not overflowed holds exactly the window's changes; an overflowed one has more than it can"""
    for e in range(snap["hdr"].shape[0]):
        t, head = int(snap["hdr"][e, 0]), int(snap["hdr"][e, 2])
        want = window_changes(snap["ring"][e], head, L)
        for a, (cnt, got) in enumerate(decoded_list(snap["changes"][e], t, L)):
            if cnt == 255:
                assert len(want[a]) > LIST_CAP or t > 0, "%s e=%d state %d: overflowed at reset with %d changes" % (label, e, a, len(want[a]))
            else:
                assert got == want[a], "%s e=%d state %d t=%d: list %s, window %s" % (label, e, a, t, got[:4], want[a][:4])


def replay_trace(s, z, meta, traced, seed, label, check_lists=False):
    """the replicas in `traced` step the trace's actions, every other one seeded random unmasked actions"""
    n, L = meta["n_steps"], s.p["filter_len"]
    clock = episode_clock(z, n)
    rng = np.random.RandomState(seed)
    extra = ("ring", "changes") if check_lists else ()
    for t in range(n + 1):
        snap = snapshot(s, extra)
        for e in traced:
            check_trace_step(z, clock, t, obs_of(snap, e), state_of(snap, e), "%s e=%d" % (label, e), rew_atol(s.p))
        if check_lists:
            check_change_lists(snap, L, "%s step %d" % (label, t))
        if t == n:
            break
        aa, ap = random_actions(rng, snap)
        aa[traced] = z["act_a"][t]
        ap[traced] = z["act_p"][t]
        set_actions(s, aa, ap)
        s.step()
    assert clock[1][n] == 2


def ulp_distance(a, b):
    a, b = np.asarray(a), np.asarray(b)
    it = {4: np.int32, 8: np.int64}[a.dtype.itemsize]
    ia, ib = a.view(it).astype(np.int64), b.view(it).astype(np.int64)
    sign = np.int64(-1) << (8 * a.dtype.itemsize - 1)
    ia = np.where(ia < 0, sign - ia, ia)   # two's-complement order of the float values
    ib = np.where(ib < 0, sign - ib, ib)
    return int(np.abs(ia - ib).max()) if ia.size else 0


# ---------------------------------------------------------------------------------------------------- CPU
def test_variant_traces_cover_what_they_are_for():
    """the fixtures are the table's variants, end two episodes, and reach the code they were chosen for"""
    etas = set()
    for name in NAMES:
        z, meta, p = load(name)
        kw, seed = variant_kwargs(name)
        assert meta["kwargs"] == kw and meta["seed"] == seed, name
        T, n = kw["episode_length"], meta["n_steps"]
        assert n > 2 * T and list(np.nonzero(z["done"])[0]) == [T - 1, 2 * T - 1], name
        for t in (T, 2 * T):   # the reset observation is the first observation of an episode
            for k in OBS_KEYS + ["st_" + k for k in ST_KEYS]:
                assert np.array_equal(z[k][t], z[k][0]), (name, t, k)
        assert z["mask_p"].shape[1] == 1 + kw["num_subsidy_levels"]
        assert (z["mask_p"][:, 1:] == 1).any() and ((z["mask_p"][:, 1:] == 0).any() == (kw["subsidy_interval"] > 1)), name
        assert (z["mask_a"][:, 1:] == 1).any() and ((z["mask_a"][:, 1:] == 0).any() == (kw["action_cooldown_period"] > 1)), name
        etas.add(float(kw["economic_reward_crra_eta"]))
    assert {0.5, 1.5, 2.0, 3.0} <= etas                            # sqrt, reciprocal and general powf exponents
    assert {2, 21, 41} <= {1 + VARIANTS[n][1].get("num_subsidy_levels", COVID_KWARGS["num_subsidy_levels"]) for n in NAMES}
    assert min(build_covid_params(**variant_kwargs(n)[0])["time_when_vaccine_delivery_begins"] for n in NAMES) < 0


@pytest.mark.parametrize("name", NAMES)
def test_oracle_follows_variant_trace(name):
    z, meta, p = load(name)
    env = CovidOracleEnv(p, auto_reset=True)
    clock = episode_clock(z, meta["n_steps"])
    for t in range(meta["n_steps"] + 1):
        if t:
            env.step(z["act_a"][t - 1].astype(np.int32), np.int32(z["act_p"][t - 1]))
        check_trace_step(z, clock, t, env.obs(), env.state(), "oracle")


@pytest.mark.parametrize("name", NAMES)
@pytest.mark.parametrize("change_list", [False, True], ids=["scan", "change_list"])
def test_emulation_follows_variant_trace(change_list, name):
    """the traced replica in the middle of 3; with the change list, each list is the window's changes at every step"""
    from tests.emu.emu_stepper import EmuCovidStepper
    z, meta, p = load(name)
    s = EmuCovidStepper(p, 3, auto_reset=True, change_list=change_list)
    s.reset()
    replay_trace(s, z, meta, [1], 7, "emu", check_lists=change_list)


def random_policy_counts(s, seeds):
    """per-state counts of the drawn stringency levels [S, 1 + levels] and of the planner's [1 + sub_levels]"""
    na, npl = 1 + s.p["num_stringency_levels"], 1 + s.p["num_subsidy_levels"]
    ca, cp, draws = np.zeros((s.p["n_states"], na), np.int64), np.zeros(npl, np.int64), []
    for seed in seeds:
        s.sample_random_actions(seed=seed)
        aa, ap = s.to_numpy(s.buf["actions_agent"]), s.to_numpy(s.buf["actions_planner"])
        for a in range(aa.shape[1]):
            ca[a] += np.bincount(aa[:, a], minlength=na)
        cp += np.bincount(ap, minlength=npl)
        draws.append(aa)
    return ca, cp, draws


def check_uniform(ca, cp, draws):
    from scipy.stats import chisquare
    for a in range(ca.shape[0]):
        assert chisquare(ca[a]).pvalue > 1e-4, (a, ca[a])
    assert chisquare(cp).pvalue > 1e-4, cp
    for i, aa in enumerate(draws):
        assert not (aa[1:] == aa[:-1]).all(axis=1).any(), "two neighbouring replicas drew the same actions"
        if i:
            assert not (aa == draws[i - 1]).all(axis=1).any(), "a replica drew the same actions for consecutive seeds"


def check_closed_never_drawn(s):
    ma, mp = s.to_numpy(s.buf["mask_agent"]), s.to_numpy(s.buf["mask_planner"])
    aa, ap = s.to_numpy(s.buf["actions_agent"]), s.to_numpy(s.buf["actions_planner"])
    assert np.all(np.take_along_axis(ma, aa[:, None, :], axis=1) == 1.0)
    assert np.all(np.take_along_axis(mp, ap[:, None], axis=1) == 1.0)
    return (ma[:, 1] == 0).any(), (mp[:, 1] == 0).any()


def test_emulated_random_policy_is_uniform_over_open_entries():
    from tests.emu.emu_stepper import EmuCovidStepper
    p = build_covid_params(**dict(COVID_KWARGS, episode_length=40, action_cooldown_period=7, subsidy_interval=5))
    s = EmuCovidStepper(p, 512, auto_reset=True)
    s.reset()                                   # every entry open at t = 0
    check_uniform(*random_policy_counts(s, range(500, 516)))
    closed_a = closed_p = False
    for t in range(12):
        s.sample_random_actions(seed=40 + t)
        ca, cp = check_closed_never_drawn(s)
        closed_a |= ca; closed_p |= cp
        s.step()
    assert closed_a and closed_p


# ---------------------------------------------------------------------------------------------------- GPU
@pytest.mark.gpu
@pytest.mark.parametrize("name", NAMES)
@pytest.mark.parametrize("change_list", [False, True], ids=["scan", "change_list"])
def test_cuda_follows_variant_trace(change_list, name):
    """replicas 0, E/2 and E-1 of E = 257 step the trace's actions, the others seeded random ones"""
    from ai_economist_b200.covid_stepper import CudaCovidStepper
    z, meta, p = load(name)
    E = 257
    s = CudaCovidStepper(p, E, auto_reset=True, change_list=change_list)
    s.reset()
    replay_trace(s, z, meta, [0, E // 2, E - 1], 17, "cuda", check_lists=change_list)


@pytest.mark.gpu
@pytest.mark.parametrize("name", NAMES)
def test_cuda_batch_matches_oracle_and_emulation_across_auto_resets(name):
    """64 replicas, distinct random actions, two auto-resets: every replica at every step against the numpy oracle
    (outputs and state) and against the emulation of the same source (integer buffers exact, floats to tolerance)"""
    from ai_economist_b200.covid_stepper import CudaCovidStepper
    from tests.emu.emu_stepper import EmuCovidStepper
    _, meta, p = load(name)
    E, T = 64, p["episode_length"]
    cuda = {cl: CudaCovidStepper(p, E, auto_reset=True, change_list=cl) for cl in (False, True)}
    emu = {cl: EmuCovidStepper(p, E, auto_reset=True, change_list=cl) for cl in (False, True)}
    orc = [CovidOracleEnv(p, auto_reset=True) for _ in range(E)]
    for s in list(cuda.values()) + list(emu.values()):
        s.reset()
    rng = np.random.RandomState(101)
    ulp_emu, ulp_orc = {}, {}
    for t in range(2 * T + 6):
        for cl in (False, True):
            got, want = snapshot(cuda[cl], ("ring", "changes")), snapshot(emu[cl], ("ring", "changes"))
            for k in got:
                if k in INT_BUFS:
                    assert np.array_equal(got[k], want[k]), (t, cl, k)
                else:
                    assert np.allclose(want[k], got[k], rtol=RTOL, atol=rew_atol(p) if k.startswith("reward") else ATOL), (t, cl, k)
                    ulp_emu[k] = max(ulp_emu.get(k, 0), ulp_distance(want[k], got[k]))
            for e in range(E):
                ro, rs = orc[e].obs(), orc[e].state()
                go = obs_of(got, e)
                check_obs(ro, go, "oracle t=%d e=%d change_list=%s" % (t, e, cl), rewards=t > 0, ratol=rew_atol(p))
                check_oracle_state(rs, state_of(got, e), "oracle t=%d e=%d" % (t, e))
                for k in OBS_KEYS[:5] + (["rew_a", "rew_p"] if t else []):
                    ulp_orc[k] = max(ulp_orc.get(k, 0), ulp_distance(np.asarray(ro[k]).astype(np.asarray(go[k]).dtype), go[k]))
        aa, ap = random_actions(rng, got)
        for s in list(cuda.values()) + list(emu.values()):
            set_actions(s, aa, ap)
            s.step()
        for e in range(E):
            orc[e].step(aa[e], ap[e])
    assert all(o.episodes == 2 for o in orc)
    print("\n[%s] largest ulp distance, CUDA vs emulation: %s" % (name, json.dumps(ulp_emu, sort_keys=True)))
    print("[%s] largest ulp distance, CUDA vs numpy oracle: %s" % (name, json.dumps(ulp_orc, sort_keys=True)))


@pytest.mark.gpu
def test_cuda_change_list_overflows_and_resets_like_the_scan():
    """1-day cooldowns: the 32-entry lists overflow during the first episode, the outputs follow the scan's at every step,
    and the auto-reset rebuilds every list from its initial window (the count recomputed here from the real-world
    stringency history)"""
    from ai_economist_b200.covid_stepper import CudaCovidStepper
    kw, _ = variant_kwargs("cooldown1_len60")
    p = build_covid_params(**kw)
    E, T, L, steps = 64, p["episode_length"], p["filter_len"], 95
    scan = CudaCovidStepper(p, E, auto_reset=True, change_list=False)
    lst = CudaCovidStepper(p, E, auto_reset=True, change_list=True)
    scan.reset(); lst.reset()
    hist = np.asarray(p["init"]["stringency_history"], np.int64)        # [L + 1, S], oldest first
    n0 = (np.diff(hist, axis=0) != 0).sum(axis=0)
    want_cnt = np.where(n0 > LIST_CAP, 255, n0)
    assert (want_cnt < 255).all()
    want_lists = window_changes(hist.T, 0, L)
    rng = np.random.RandomState(3)
    overflowed = False
    for t in range(steps + 1):
        a, b = snapshot(scan, ("ring",)), snapshot(lst, ("ring", "changes"))
        for k in a:
            if k in INT_BUFS:
                assert np.array_equal(a[k], b[k]), (t, k)
            else:
                assert np.allclose(a[k], b[k], rtol=RTOL, atol=ATOL), (t, k)
        hd = b["changes"][:, 0, :].view(np.uint32)
        counts = (hd >> 8) & 0xFF
        if 0 < t < T:
            overflowed |= bool((counts == 255).any())
        if t in (0, T):   # a fresh episode: every list is its initial window's
            assert (b["hdr"][:, 0] == 0).all() and (b["hdr"][:, 3] == (t // T)).all()
            assert (counts == want_cnt[None]).all() and ((hd & 0xFF) == 0).all(), t
            for e in range(E):
                assert [l for _, l in decoded_list(b["changes"][e], 0, L)] == want_lists, (t, e)
        check_change_lists(b, L, "step %d" % t)
        if t == steps:
            break
        aa, ap = random_actions(rng, b)
        for s in (scan, lst):
            set_actions(s, aa, ap)
            s.step()
    assert overflowed


@pytest.mark.gpu
def test_cuda_full_size_across_episode_ends():
    """4 096 replicas, episodes of 40 steps, 100 steps of the device random policy: a sample of replicas replayed through
    the oracle with the device's actions at every step, every replica's observations at both episode ends equal to a
    fresh reset's bytes, two episodes counted everywhere, a second run bit-identical"""
    import torch
    from ai_economist_b200.covid_stepper import CudaCovidStepper
    p = build_covid_params(**dict(COVID_KWARGS, episode_length=40))
    E, T, steps = 4096, 40, 100
    sample = [0, 1, 63, 64, 1000, 2047, 2048, 3333, 4094, 4095]
    obs_bufs = OUT_BUFS[:7]
    fresh = CudaCovidStepper(p, 1, auto_reset=True)
    fresh.reset()
    idx = torch.tensor(sample, device=fresh.device)

    def run(check):
        s = CudaCovidStepper(p, E, auto_reset=True)
        s.reset()
        envs = {e: CovidOracleEnv(p, auto_reset=True) for e in sample}
        record = []
        for t in range(1, steps + 1):
            s.sample_random_actions(seed=900 + t)
            record += [s.buf["actions_agent"].clone(), s.buf["actions_planner"].clone()]
            s.step()
            record += [s.buf["reward_agent"].clone(), s.buf["reward_planner"].clone()]
            if not check:
                continue
            aa, ap = s.to_numpy(s.buf["actions_agent"][idx]), s.to_numpy(s.buf["actions_planner"][idx])
            sub = {k: s.to_numpy(s.buf[k][idx]) for k in OUT_BUFS}
            for i, e in enumerate(sample):
                envs[e].step(aa[i], ap[i])
                check_obs(envs[e].obs(), obs_of(sub, i), "t=%d e=%d" % (t, e))
                check_oracle_state(envs[e].state(), state_of(sub, i), "t=%d e=%d" % (t, e))
            if t % T == 0:
                assert bool((s.buf["done"] == 1).all()) and bool((s.buf["hdr"][:, 0] == 0).all()), t
                for k in obs_bufs:
                    assert torch.equal(s.buf[k], fresh.buf[k].expand_as(s.buf[k])), (t, k)
        assert bool((s.buf["hdr"][:, 3] == 2).all()) and bool((s.buf["hdr"][:, 0] == steps - 2 * T).all())
        return s, record

    s1, r1 = run(True)
    s2, r2 = run(False)
    assert all(torch.equal(x, y) for x, y in zip(r1, r2))
    for k in s1.buf:
        assert torch.equal(s1.buf[k], s2.buf[k]), k


@pytest.mark.gpu
def test_cuda_random_policy_draws_the_emulation_s_integers():
    """same seeds, same masks: the device draws the integers the emulation draws, and never a closed entry"""
    from ai_economist_b200.covid_stepper import CudaCovidStepper
    from tests.emu.emu_stepper import EmuCovidStepper
    p = build_covid_params(**dict(COVID_KWARGS, episode_length=40, action_cooldown_period=7, subsidy_interval=5))
    E = 256
    cuda, emu = CudaCovidStepper(p, E, auto_reset=True), EmuCovidStepper(p, E, auto_reset=True)
    cuda.reset(); emu.reset()
    closed_a = closed_p = False
    for t in range(24):
        for s in (cuda, emu):
            s.sample_random_actions(seed=300 + t)
        for k in ["actions_agent", "actions_planner", "mask_agent", "mask_planner"]:
            assert np.array_equal(cuda.to_numpy(cuda.buf[k]), emu.to_numpy(emu.buf[k])), (t, k)
        ca, cp = check_closed_never_drawn(cuda)
        closed_a |= ca; closed_p |= cp
        cuda.step(); emu.step()
    assert closed_a and closed_p


@pytest.mark.gpu
def test_cuda_random_policy_is_uniform_over_open_entries():
    """4 096 replicas x 32 seeds at t = 0 (every entry open): chi-square per state and for the planner"""
    from ai_economist_b200.covid_stepper import CudaCovidStepper
    p = build_covid_params(**dict(COVID_KWARGS, episode_length=40))
    s = CudaCovidStepper(p, 4096, auto_reset=True)
    s.reset()
    check_uniform(*random_policy_counts(s, range(700, 732)))
