"""Episode metrics of the COVID-19 scenario (aie_covid_bind_metrics / aie_covid_episode_metrics,
make_env_instance("CovidAndEconomySimulation", ..., episode_metrics=True)).

The contract:
1. Bit for bit between CUDA, the host build of the device source and the numpy restatement in oracle/covid_metrics_oracle.py
   (covid_metric_accumulators + covid_metrics_row over the float32 records the device stored), at every t and every
   episode end.  One exception: under a CRRA exponent without a fast path (economic_reward_crra_eta not 2 or 0.5) the
   step's float32 powf is the C library's (host build) or CUDA's, and numpy's float32 power may differ from either in
   the last place, so the economic-index columns are held to RESTATE_POWF_RTOL there.
2. Against the reference's scenario_metrics() (tests/golden/covid_metrics/, oracle/gen_golden_covid_metrics.py), one
   bound per column group, from the step kernel's 1e-6 relative agreement with the reference's state (tests/test_covid.py):
   - totals (infected / recovered / deaths, millions): int32 casts of float32 state, so 1e-6 relative plus one person;
   - time aggregates (means, totals over t; usa/ unemployment, subsidy, productivity): 1e-6 relative per summand, plus
     the reference's float32 pairwise sums and float32 results (about (log2 T + 1) * 2^-24): 2e-6 relative;
   - end-state USA sums (usa/vaccinated, usa/deaths): 1e-6 relative plus a float32 sum of 51 values: 2e-6 relative;
   - index sums: the per-step reward tolerance (1e-6 relative) plus one float32 rounding per step in each of the two
     running sums: (1e-6 + T * 2^-24) relative, 1e-7 absolute.
3. Nothing else changes: with the option on, every buffer the step writes is byte-identical to an env without it.
"""
import ctypes as C
import glob
import json
import os

import numpy as np
import pytest

from ai_economist_b200 import _abi, foundation
from ai_economist_b200.foundation.covid19 import build_covid_params
from ai_economist_b200.workloads import COVID_KWARGS
from oracle.covid_metrics_oracle import covid_metric_accumulators, covid_metrics_row

AIE_EINVAL, AIE_ESTATE = -1, -3
HERE = os.path.dirname(os.path.abspath(__file__))
FIXTURES = sorted(glob.glob(os.path.join(HERE, "golden", "covid_metrics", "*.npz")))
RESTATE_POWF_RTOL = 1e-5
BOUND_REL = {"totals": 1e-6, "time": 2e-6, "usa_end": 2e-6}


def emu(params, n, auto_reset=True, **kw):
    """The COVID-19 stepper over the host build of the device source (numpy buffers)."""
    from ai_economist_b200.covid_stepper import CovidStepperBase
    from tests.emu.emu_stepper import emu_lib

    class _Emu(CovidStepperBase):
        def _alloc(self, shape, dt):
            return np.zeros(shape, dtype=self._DT[dt])

        def _ptr(self, buf):
            return buf.ctypes.data_as(C.c_void_p)

        def to_numpy(self, buf):
            return np.array(buf)

    return _Emu(params, n, emu_lib(), auto_reset=auto_reset, **kw)


def group(key):
    field = key.split("/", 1)[1]
    if "millions" in field:
        return "totals"
    if "index" in field:
        return "index"
    if key.startswith("usa/") and ("vaccinated" in field or "deaths" in field):
        return "usa_end"
    return "time"


def restated(p, records):
    sums, index = covid_metric_accumulators(p, records)
    return covid_metrics_row(p, records[-1][1:5], sums, index)


def check_restated(p, keys, got, want, where):
    """got == want bit for bit, but for the economic-index columns of a powf CRRA exponent (module docstring)."""
    fast = float(1 - np.float32(p["crra_eta"])) in (-1.0, 2.0, 0.5, 1.0, 0.0)
    for i, k in enumerate(keys):
        if not fast and k.endswith("economic_index_at_end_of_episode"):
            assert abs(got[i] - want[i]) <= RESTATE_POWF_RTOL * abs(want[i]), (where, k, got[i], want[i])
        else:
            assert got[i] == want[i], (where, k, got[i], want[i])


@pytest.mark.parametrize("path", FIXTURES, ids=[os.path.splitext(os.path.basename(f))[0] for f in FIXTURES])
def test_fixture_matches_restatement_and_reference(path):
    """Replays a recorded trace's actions on the host build: every recorded point's row equals the restatement, lies
    within the per-group bounds of the reference's scenario_metrics(), and previous_episode_metrics keeps the last
    episode end's row until the next one."""
    fx = np.load(path)
    meta = json.loads(str(fx["meta_json"]))
    p = build_covid_params(**meta["kwargs"])
    T = p["episode_length"]
    tr = np.load(os.path.join(os.path.dirname(HERE), meta["trace"]))
    env = emu(p, 1, episode_metrics=True)
    twin = emu(p, 1, auto_reset=False)   # its records, including the state an episode ended in
    env.reset(); twin.reset()
    keys = [k for k, _ in env.metric_layout()]
    assert keys == fx["keys"].tolist() and len(keys) == 8 * 51 + 7
    records = [twin.to_numpy(twin.buf["state"][0])]
    points = {int(n): (bool(end), v) for n, end, v in zip(fx["n"], fx["end"], fx["values"])}
    worst, last_end = {}, None
    for n in range(1, meta["n_steps"] + 1):
        for st in (env, twin):
            st.buf["actions_agent"][...] = tr["act_a"][n - 1]
            st.buf["actions_planner"][...] = tr["act_p"][n - 1]
            st.step()
        records.append(twin.to_numpy(twin.buf["state"][0]))
        if n in points:
            end, ref = points[n]
            row = env.episode_metrics(final=end)[0]
            check_restated(p, keys, row, restated(p, records), (n, end))
            for i, k in enumerate(keys):
                g, d = group(k), abs(row[i] - ref[i])
                if g == "totals":
                    bound = BOUND_REL[g] * abs(ref[i]) + 1e-6 * (1 + 1e-9)
                elif g == "index":
                    bound = (1e-6 + T * 2.0 ** -24) * abs(ref[i]) + 1e-7
                else:
                    bound = BOUND_REL[g] * abs(ref[i])
                assert d <= bound, (n, k, row[i], ref[i])
                worst[g] = max(worst.get(g, 0.0), d / max(abs(ref[i]), 1e-300))
            if end:
                last_end = row.copy()
            elif last_end is not None:   # the previous episode's row holds until the next end
                assert np.array_equal(env.episode_metrics(final=True)[0], last_end)
        if n % T == 0:
            twin.reset()
            records = [twin.to_numpy(twin.buf["state"][0])]
    print(os.path.basename(path), "largest relative error vs the reference:",
          {g: "%.2e" % v for g, v in sorted(worst.items())})


def _next_actions(seed):
    rng = np.random.RandomState(seed)

    def nxt(st):
        ma, mp = st.obs_to_numpy("mask_agent"), st.obs_to_numpy("mask_planner")
        aa = np.argmax(ma * (rng.random_sample(ma.shape) + 1e-3), axis=1).astype(np.int32)
        ap = np.argmax(mp * (rng.random_sample(mp.shape) + 1e-3), axis=1).astype(np.int32)
        return aa, ap
    return nxt


def _same(x, y):
    if isinstance(x, np.ndarray):
        return x.shape == y.shape and x.tobytes() == y.tobytes()
    import torch
    return x.shape == y.shape and torch.equal(x.reshape(-1).view(torch.uint8), y.reshape(-1).view(torch.uint8))


def _twins(make, p, E, steps, final_obs, obs_dtype, rollout_T, nxt):
    """An env with episode metrics and one without, the same actions: every buffer byte-identical after every step."""
    on = make(p, E, final_obs=final_obs, obs_dtype=obs_dtype, episode_metrics=True)
    off = make(p, E, final_obs=final_obs, obs_dtype=obs_dtype)
    if rollout_T:
        ron, roff = on.bind_rollout(rollout_T, final_obs=final_obs), off.bind_rollout(rollout_T, final_obs=final_obs)
    on.reset(); off.reset()
    for s in range(steps):
        if rollout_T and on.rollout_slot == rollout_T:
            on.restart_rollout(); off.restart_rollout()
        if rollout_T:   # the samplers write into slot s of each rollout
            a_on, a_off = ron.buf["actions_agent"][on.rollout_slot], roff.buf["actions_agent"][off.rollout_slot]
            p_on, p_off = ron.buf["actions_planner"][on.rollout_slot], roff.buf["actions_planner"][off.rollout_slot]
            off.sample_random_actions(1000 + s); on.sample_random_actions(1000 + s)
            assert _same(a_on, a_off) and _same(p_on, p_off)
        else:
            aa, ap = nxt(off)
            for st in (on, off):
                st.buf["actions_agent"][...] = aa if isinstance(st.buf["actions_agent"], np.ndarray) else \
                    st.torch.as_tensor(aa, device=st.device)
                st.buf["actions_planner"][...] = ap if isinstance(st.buf["actions_planner"], np.ndarray) else \
                    st.torch.as_tensor(ap, device=st.device)
        on.step(); off.step()
        for k in off.buf:
            assert _same(on.buf[k], off.buf[k]), (s, k)
    if rollout_T:
        for k in roff.buf:
            assert _same(ron.buf[k], roff.buf[k]), k
    assert on.has_previous_episode()
    return on


TWIN_CASES = [(fo, dt, rt) for fo in (False, True) for dt in (None, "bfloat16") for rt in (0, 10, 30)]


@pytest.mark.parametrize("final_obs,obs_dtype,rollout_T", TWIN_CASES,
                         ids=["final%d-%s-rollout%d" % (fo, dt or "float32", rt) for fo, dt, rt in TWIN_CASES])
def test_emulated_twins_are_byte_identical(final_obs, obs_dtype, rollout_T):
    """rollout_T 10 holds one episode end per rollout (K = 1), 30 two or three (K >= 2)."""
    p = build_covid_params(**dict(COVID_KWARGS, episode_length=12))
    _twins(emu, p, 3, 40, final_obs, obs_dtype, rollout_T, _next_actions(7))


def test_emulated_launch_counts():
    p = build_covid_params(**dict(COVID_KWARGS, episode_length=6))
    on, off = emu(p, 2, episode_metrics=True, final_obs=True), emu(p, 2, final_obs=True)
    for st in (on, off):
        st.reset()
        for s in range(8):
            st.sample_random_actions(s)
            st.step()
    assert on.launch_count() == off.launch_count()
    n = on.launch_count()
    on.episode_metrics()
    assert on.launch_count() == n + 1
    on.episode_metrics(final=True)
    assert on.launch_count() == n + 2


def _metric_struct(st, **over):
    m = _abi.AieCovidMetricBuffers()
    for name in ("sums", "prev_sums", "index", "prev_index", "prev_end"):
        setattr(m, name, st._ptr(st.buf["metric_" + name]))
    m.us_population = 3.3e8
    for k, v in over.items():
        setattr(m, k, v)
    return m


def test_emulated_abi_errors():
    p = build_covid_params(**dict(COVID_KWARGS, episode_length=5))
    st = emu(p, 2, episode_metrics=True)
    L, h = st.lib, st._h
    out = np.zeros((2, 8 * 51 + 7), np.float64)
    optr = out.ctypes.data_as(C.c_void_p)
    # before the reset that starts the accumulation
    assert L.aie_covid_episode_metrics(h, 0, optr, None) == AIE_ESTATE
    st.reset()
    assert L.aie_covid_episode_metrics(h, 1, optr, None) == AIE_ESTATE   # no episode has ended yet
    assert L.aie_covid_episode_metrics(h, 0, optr, None) == 0
    assert L.aie_covid_episode_metrics(h, 2, optr, None) == AIE_EINVAL
    assert L.aie_covid_episode_metrics(h, 0, None, None) == AIE_EINVAL
    raw = np.zeros(8 * out.size + 8, np.uint8)
    assert L.aie_covid_episode_metrics(h, 0, C.c_void_p(raw.ctypes.data + 4), None) == AIE_EINVAL
    assert L.aie_covid_episode_metrics(None, 0, optr, None) == AIE_EINVAL
    # binding: NULL / misaligned / bad population, and not while a rollout is bound
    assert L.aie_covid_bind_metrics(h, C.byref(_metric_struct(st, sums=None))) == AIE_EINVAL
    assert L.aie_covid_bind_metrics(h, C.byref(_metric_struct(st, prev_end=C.c_void_p(raw.ctypes.data + 2)))) == AIE_EINVAL
    assert L.aie_covid_bind_metrics(h, C.byref(_metric_struct(st, sums=C.c_void_p(raw.ctypes.data + 4)))) == AIE_EINVAL
    assert L.aie_covid_bind_metrics(h, C.byref(_metric_struct(st, us_population=0.0))) == AIE_EINVAL
    st.bind_rollout(4)
    assert L.aie_covid_bind_metrics(h, C.byref(_metric_struct(st))) == AIE_ESTATE
    assert L.aie_covid_bind_metrics(h, None) == AIE_ESTATE
    st.unbind_rollout()
    for s in range(5):
        st.step()
    assert L.aie_covid_episode_metrics(h, 1, optr, None) == 0
    # unbinding: the metrics calls refuse, the step runs the plain kernels
    assert L.aie_covid_bind_metrics(h, None) == 0
    assert L.aie_covid_episode_metrics(h, 0, optr, None) == AIE_ESTATE
    st.step()
    # rebinding: previous metrics need a new episode end, current ones a reset
    assert L.aie_covid_bind_metrics(h, C.byref(_metric_struct(st))) == 0
    assert L.aie_covid_episode_metrics(h, 0, optr, None) == AIE_ESTATE
    st.reset()
    assert L.aie_covid_episode_metrics(h, 1, optr, None) == AIE_ESTATE
    # layout
    assert L.aie_covid_get_metric_layout(h, None, 0) == 8 * 51 + 7
    assert L.aie_covid_get_metric_layout(None, None, 0) == AIE_EINVAL
    # an env without metric buffers
    plain = emu(p, 1)
    plain.reset()
    assert plain.lib.aie_covid_episode_metrics(plain._h, 0, optr, None) == AIE_ESTATE


def _env(n_envs=3, episode_length=8, **kw):
    def factory(params, n, auto_reset, **fkw):
        return emu(params, n, auto_reset=auto_reset, **fkw)
    return foundation.make_env_instance(
        "CovidAndEconomySimulation",
        components=[("ControlUSStateOpenCloseStatus", {"action_cooldown_period": 2}), ("FederalGovernmentSubsidy", {}),
                    ("VaccinationCampaign", {"observe_rate": True})],
        episode_length=episode_length, n_envs=n_envs, stepper_factory=factory, **kw)


def test_env_surface_and_rows_as_dicts():
    env = _env(episode_metrics=True, final_obs=True)
    env.reset()
    keys = env.metric_keys
    assert len(keys) == 415 and keys[0] == "Alabama/infected (millions)" and keys[-1] == "usa/economic_index_at_end_of_episode"
    assert env.previous_episode_metrics is None
    for s in range(11):
        env.step()
    m = env.metrics_tensor()
    assert m.shape == (3, 415) and m.dtype == np.float64
    dicts = env.metrics_rows_as_dicts(m)
    assert [list(d) for d in dicts] == [keys] * 3
    assert all(np.array_equal(np.array(list(d.values())), m[e]) for e, d in enumerate(dicts))
    assert env.metrics == dicts[0] and env.metrics_of(2) == dicts[2]
    pm = env.previous_episode_metrics_tensor()
    assert env.previous_episode_metrics_of(1) == env.metrics_rows_as_dicts(pm)[1]
    assert env.metrics_rows_as_dicts(pm, envs=[2])[0] == env.previous_episode_metrics_of(2)
    out = np.full((3, 415), -1.0)
    assert env.metrics_tensor(out=out) is out and np.array_equal(out, m)
    with pytest.raises(_abi.AieError):
        env.metrics_tensor(out=np.zeros((3, 414)))


def test_keyword_checks():
    env = _env()
    env.reset()
    for call in (lambda: env.metrics, lambda: env.metrics_tensor(), lambda: env.previous_episode_metrics,
                 lambda: env.metric_keys, lambda: env.previous_episode_metrics_tensor()):
        with pytest.raises(ValueError, match="episode_metrics"):
            call()

    def plain_factory(params, n, auto_reset, **kw):
        kw.pop("episode_metrics", None)
        return emu(params, n, auto_reset=auto_reset, **kw)
    with pytest.raises(NotImplementedError, match="episode_metrics"):
        foundation.make_env_instance(
            "CovidAndEconomySimulation",
            components=[("ControlUSStateOpenCloseStatus", {}), ("FederalGovernmentSubsidy", {}), ("VaccinationCampaign", {})],
            episode_length=8, n_envs=1, stepper_factory=plain_factory, episode_metrics=True)


# ------------------------------------------------------------------------------------------------ GPU
def _cuda(params, n, **kw):
    from ai_economist_b200.covid_stepper import CudaCovidStepper
    return CudaCovidStepper(params, n, **kw)


@pytest.mark.gpu
def test_cuda_rows_equal_the_host_build_and_the_restatement():
    """4 096 replicas over two 540-step episodes under random masked actions.  Every CUDA row of a sample of 64
    replicas equals the host build's (the same actions) bit for bit, and 8 of them the restatement over the CUDA
    records, at mid-episode points and at both episode ends."""
    import torch
    E, T = 4096, 540
    p = build_covid_params(**dict(COVID_KWARGS, episode_length=T))
    g = _cuda(p, E, episode_metrics=True)
    pick = np.linspace(0, E - 1, 64).astype(np.int64)
    h = emu(p, len(pick), episode_metrics=True)
    twin = _cuda(p, E, auto_reset=False)   # the CUDA records, with the state each episode ended in
    g.reset(); h.reset(); twin.reset()
    keys = [k for k, _ in g.metric_layout()]
    sel = torch.as_tensor(pick[:8], device=g.device)
    recs = [[r] for r in twin.to_numpy(twin.buf["state"][sel])]
    checked = 0
    for n in range(1, 2 * T + 1):
        g.sample_random_actions(n)
        aa, ap = g.buf["actions_agent"], g.buf["actions_planner"]
        twin.buf["actions_agent"].copy_(aa); twin.buf["actions_planner"].copy_(ap)
        h.buf["actions_agent"][...] = aa.cpu().numpy()[pick]
        h.buf["actions_planner"][...] = ap.cpu().numpy()[pick]
        g.step(); h.step(); twin.step()
        st = twin.to_numpy(twin.buf["state"][sel])
        for i in range(len(sel)):
            recs[i].append(st[i])
        if n % 90 == 0 or n % T == 0:
            end = n % T == 0
            got = g.episode_metrics(final=end).cpu().numpy()
            assert np.array_equal(got[pick], h.episode_metrics(final=end)), n
            for i, e in enumerate(pick[:8]):
                check_restated(p, keys, got[e], restated(p, recs[i]), (n, int(e)))
            checked += 1
        if n % T == 0:
            twin.reset()
            recs = [[r] for r in twin.to_numpy(twin.buf["state"][sel])]
    torch.cuda.synchronize()
    assert checked == 12


@pytest.mark.gpu
@pytest.mark.parametrize("E,final_obs,obs_dtype,rollout_T", [(4096, False, None, 0), (4096, True, None, 0),
                                                             (4096, True, "bfloat16", 0), (512, True, None, 600),
                                                             (512, False, "bfloat16", 300)],
                         ids=["plain", "final", "final-bf16", "final-rollout600", "bf16-rollout300"])
def test_cuda_twins_are_byte_identical(E, final_obs, obs_dtype, rollout_T):
    """Full 540-step episodes: one episode end and 20 steps into the next."""
    p = build_covid_params(**dict(COVID_KWARGS, episode_length=540))
    calls = [0]

    def nxt(st):
        calls[0] += 1
        st.sample_random_actions(calls[0])
        return st.buf["actions_agent"].cpu().numpy(), st.buf["actions_planner"].cpu().numpy()
    _twins(_cuda, p, E, 560, final_obs, obs_dtype, rollout_T, nxt)
