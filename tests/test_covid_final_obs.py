"""Final observations of the COVID-19 scenario (aie_covid_step_final, CovidBatchedEnv(final_obs=True)).

Every COVID-19 episode ends on its time limit, and the auto-reset replaces the state it ended in within the same step.
With final_obs the step kernel observes that state once more, into the final_<name> buffers, before it resets.

CPU (the host build of the device source): the reference's last-step observations; byte-for-byte twins against an
env without the auto-reset across two episode ends; the ABI errors; the Python surface; a rollout's advantages
bootstrapped from env.final_obs.  GPU: the same twins and rollout at full size, and the CUDA final rows against the
host build's.
"""
import ctypes as C

import numpy as np
import pytest

from ai_economist_b200 import _abi, foundation
from ai_economist_b200.foundation.covid19 import build_covid_params
from ai_economist_b200.workloads import COVID_KWARGS, covid_reference_config
from tests.test_advantages import gae_ref, same_bits
from tests.test_covid import ATOL, OBS_KEYS, RTOL, VARIANTS, load

AIE_EINVAL, AIE_ESTATE = -1, -3
STATE_BUFS = ["state", "ints", "hdr", "ring", "changes", "reward_agent", "reward_planner", "done"] + _abi.COVID_OBS_NAMES
RATE = "VaccinationCampaign-next_vaccination_rate"


def emu(params, n, auto_reset, final_obs=False, change_list=True):
    """The COVID-19 stepper over the host emulation of the device source (numpy buffers), with final_obs."""
    from ai_economist_b200.covid_stepper import CovidStepperBase
    from tests.emu.emu_stepper import emu_lib

    class _Emu(CovidStepperBase):
        def _alloc(self, shape, dt):
            return np.zeros(shape, dtype=self._DT[dt])

        def _ptr(self, buf):
            return buf.ctypes.data_as(C.c_void_p)

        def to_numpy(self, buf):
            return np.array(buf)

    return _Emu(params, n, emu_lib(), auto_reset=auto_reset, change_list=change_list, final_obs=final_obs)


def final_rows(st, e):
    """Row e of the final buffers, keyed like read_obs."""
    g = lambda k: st.to_numpy(st.buf["final_" + k][e])
    return dict(agent_state=g("obs_agent_state"), postsubsidy=g("obs_postsubsidy"), lagged=g("obs_lagged_stringency"),
                policy_ind=g("obs_policy_indicators"), scalars=g("obs_scalars"), mask_a=g("mask_agent"),
                mask_p=g("mask_planner"))


def same(x, y):
    """Byte-for-byte equality of two buffers (numpy, or torch compared on their device)."""
    if isinstance(x, np.ndarray):
        return x.shape == y.shape and x.tobytes() == y.tobytes()
    import torch
    return x.shape == y.shape and torch.equal(x.reshape(-1).view(torch.uint8), y.reshape(-1).view(torch.uint8))


def snap(st, prefix=""):
    """Copies of the seven observation / mask buffers (prefix "final_": their final twins)."""
    cp = lambda x: x.copy() if isinstance(x, np.ndarray) else x.clone()
    return {k: cp(st.buf[prefix + k]) for k in _abi.COVID_OBS_NAMES}


def same_obs(x, y):
    return all(same(x[k], y[k]) for k in _abi.COVID_OBS_NAMES)


def random_masked_actions(st, rng):
    ma, mp = st.to_numpy(st.buf["mask_agent"]), st.to_numpy(st.buf["mask_planner"])
    aa = np.argmax(ma * (rng.random_sample(ma.shape) + 1e-3), axis=1).astype(np.int32)
    ap = np.argmax(mp * (rng.random_sample(mp.shape) + 1e-3), axis=1).astype(np.int32)
    return aa, ap


def set_actions(st, aa, ap):
    st.buf["actions_agent"][...] = aa
    st.buf["actions_planner"][...] = ap


# ------------------------------------------------------------------------------------------------ 1. reference traces
@pytest.mark.parametrize("name", VARIANTS)
@pytest.mark.parametrize("change_list", [False, True], ids=["scan", "change_list"])
def test_emulated_final_rows_match_the_reference_last_step(change_list, name):
    z, meta, p = load(name)
    n = meta["n_steps"]
    assert n == p["episode_length"]   # the trace ends on its episode's last step
    s = emu(p, 2, True, final_obs=True, change_list=change_list)
    s.reset()
    first = {k: v.copy() for k, v in s.read_obs(1).items()}
    for t in range(n):
        s.buf["actions_agent"][1] = z["act_a"][t].astype(np.int32)
        s.buf["actions_planner"][1] = np.int32(z["act_p"][t])
        s.step()
    fin = final_rows(s, 1)
    for k in OBS_KEYS:
        assert np.allclose(z[k][n], fin[k], rtol=RTOL, atol=ATOL), k
    assert np.array_equal(z["mask_a"][n], fin["mask_a"]) and np.array_equal(z["mask_p"][n], fin["mask_p"])
    live = s.read_obs(1)
    assert int(live["done"]) == 1
    for k in OBS_KEYS:
        assert live[k].tobytes() == first[k].tobytes(), k


# ------------------------------------------------------------------------------------------------ 2. twins
def _twins(make, params, E, episodes, next_actions, sentinel):
    """Steps F (auto-reset + final_obs), A (auto-reset) and N (no auto-reset; re-created and reset for each episode)
    with the same actions over `episodes` episodes and checks, at every step: F's buffers equal A's byte for byte; on
    an ending step F's final rows equal N's observations byte for byte; on every other step F's sentinel-filled final
    rows are untouched."""
    T = params["episode_length"]
    F, A = make(params, E, True, final_obs=True), make(params, E, True)
    F.reset(); A.reset()

    def fill():
        for k in _abi.COVID_OBS_NAMES:
            F.buf["final_" + k][...] = float(sentinel)
        return snap(F, "final_")
    untouched = fill()
    for ep in range(episodes):
        N = make(params, E, False)
        N.reset()
        for t in range(T):
            aa, ap = next_actions(F)
            for st in (F, A, N):
                set_actions(st, aa, ap)
                st.step()
            for k in (k for k in STATE_BUFS if k in F.buf):   # "changes" only with the change list
                assert same(F.buf[k], A.buf[k]), (ep, t, k)
            done = F.to_numpy(F.buf["done"])
            if t < T - 1:
                assert not done.any()
                assert same_obs(snap(F, "final_"), untouched), (ep, t)
            else:
                assert (done == 1).all() and (N.to_numpy(N.buf["done"]) == 1).all()
                assert same_obs(snap(F, "final_"), snap(N)), ep
                untouched = fill()
        N.close()


@pytest.mark.parametrize("change_list", [False, True], ids=["scan", "change_list"])
def test_emulated_twins_across_two_episode_ends(change_list):
    p = build_covid_params(**dict(COVID_KWARGS, episode_length=50))
    rng = np.random.RandomState(7)
    make = lambda params, n, ar, final_obs=False: emu(params, n, ar, final_obs=final_obs, change_list=change_list)
    _twins(make, p, 3, 2, lambda st: random_masked_actions(st, rng), np.float32(-7.25))


# ------------------------------------------------------------------------------------------------ 3. ABI errors
def _final_struct(bufs):
    fb = _abi.AieCovidObsBuffers()
    for k in _abi.COVID_OBS_NAMES:
        setattr(fb, k, bufs[k].ctypes.data)
    return fb


def test_emulated_abi_errors_and_launch_count():
    from tests.emu.emu_stepper import emu_lib
    L = emu_lib()
    p = build_covid_params(**dict(COVID_KWARGS, episode_length=20))
    s = emu(p, 2, True, final_obs=True)
    own = {k: np.zeros(s.buf[k].shape, np.float32) for k in _abi.COVID_OBS_NAMES}
    fb = _final_struct(own)
    call = lambda h, out: L.aie_covid_step_final(h, C.byref(out) if out is not None else None, None)
    # bound, not reset yet
    assert call(s._h, fb) == AIE_ESTATE and b"reset first" in L.aie_last_error()
    s.reset()
    n0 = s.launch_count()
    assert call(None, fb) == AIE_EINVAL
    assert call(s._h, None) == AIE_EINVAL
    raw = np.zeros(64, np.uint8)
    odd = raw[1:].ctypes.data   # not 4-byte aligned
    for k in _abi.COVID_OBS_NAMES:
        for bad, msg in ((None, b"NULL"), (odd, b"aligned")):
            b = _final_struct(own)
            setattr(b, k, bad)
            assert call(s._h, b) == AIE_EINVAL and msg in L.aie_last_error(), (k, bad)
    assert s.launch_count() == n0
    for i in range(3):
        assert call(s._h, fb) == 0
        assert s.launch_count() == n0 + i + 1
    # auto_reset off: the step's own observations are the final ones
    n = emu(p, 2, False)
    n.reset()
    assert call(n._h, fb) == AIE_ESTATE and b"auto_reset" in L.aie_last_error()
    # created, no buffers bound
    from ai_economist_b200.covid_stepper import covid_config_from_params
    cfg, keep = covid_config_from_params(p, True)
    h = C.c_void_p()
    assert L.aie_covid_create(C.byref(cfg), 2, 0, C.byref(h)) == 0
    try:
        assert call(h, fb) == AIE_ESTATE
        assert L.aie_covid_launch_count(h) == 0
    finally:
        L.aie_covid_destroy(h)


# ------------------------------------------------------------------------------------------------ 4. Python surface
def _env(final_obs=True, auto_reset=True, episode_length=40, n_envs=3, observe_rate=True):
    kw = dict(COVID_KWARGS, episode_length=episode_length, start_date="2020-12-01", delivery_interval=7,
              vaccine_delivery_start_date="2020-12-15")
    cfg = covid_reference_config(kw)
    if observe_rate:
        for c in cfg["components"]:
            if "VaccinationCampaign" in c:
                c["VaccinationCampaign"]["observe_rate"] = True
    factory = lambda params, n, ar, final_obs=False: emu(params, n, ar, final_obs=final_obs)
    return foundation.make_env_instance(cfg.pop("scenario_name"), n_envs=n_envs, auto_reset=auto_reset,
                                        final_obs=final_obs, stepper_factory=factory, **cfg)


def test_env_final_obs_mirrors_env_obs():
    env = _env()
    st = env.stepper
    assert env.final_obs is not None and set(env.final_obs) == {"a", "p"}
    for g in ("a", "p"):
        assert set(env.final_obs[g]) == set(env.obs[g]) and RATE in env.final_obs[g]
    assert env.final_obs["a"]["world-agent_state"] is st.buf["final_obs_agent_state"]
    assert env.final_obs["p"]["action_mask"] is st.buf["final_mask_planner"]
    env.reset()
    T = env.episode_length
    tab = env._rate_tab
    assert tab.shape == (T + 1,) and tab[T] > 0
    for t in range(T):
        env.step(None)
        fin = env.final_obs
        if t < T - 1:
            assert not fin["p"][RATE].any() and not fin["a"][RATE].any()
            continue
        assert (env.done["__all__"] == 1).all()
        assert np.allclose(fin["p"]["time"], 1.0)   # t = T under observation scaling
        assert np.array_equal(fin["p"][RATE], np.full(env.n_envs, tab[T], np.float32))
        assert np.array_equal(fin["a"][RATE], np.full((env.n_envs, env.n_agents), tab[T], np.float32))
        # the live rate is that of the new episode's first step
        assert np.array_equal(env.obs["p"][RATE], np.full(env.n_envs, tab[0], np.float32))
    # rows of replicas whose episode did not end keep their rate
    env.step(None)
    assert np.array_equal(env.final_obs["p"][RATE], np.full(env.n_envs, tab[T], np.float32))


def test_keyword_checks():
    """final_obs=True without the auto-reset is a ValueError for both envs; the COVID-19 env accepts the option, unless
    its stepper_factory makes a stepper without final observations."""
    from tests.emu.emu_stepper import emu_factory
    from tests.test_obs_bf16 import _cfg
    name, kw = _cfg("c1_tutorial", episode_length=5)
    with pytest.raises(ValueError, match="auto_reset"):
        foundation.make_env_instance(name, n_envs=1, seeds=[1], stepper_factory=emu_factory, auto_reset=False,
                                     final_obs=True, **kw)
    with pytest.raises(ValueError, match="auto_reset"):
        _env(auto_reset=False)
    assert _env(n_envs=1).final_obs is not None
    cfg = covid_reference_config(dict(COVID_KWARGS, episode_length=20))
    with pytest.raises(NotImplementedError):
        foundation.make_env_instance(cfg.pop("scenario_name"), n_envs=2, auto_reset=True, final_obs=True,
                                     stepper_factory=lambda params, n, ar, **k: emu(params, n, ar), **cfg)


def test_final_obs_needs_auto_reset_and_defaults_off():
    with pytest.raises(ValueError):
        _env(auto_reset=False)
    with pytest.raises(ValueError):
        emu(build_covid_params(**dict(COVID_KWARGS, episode_length=20)), 2, False, final_obs=True)
    env = _env(final_obs=False)
    assert env.final_obs is None and "final_obs_scalars" not in env.stepper.buf
    # a three-argument stepper factory keeps working while the option is off
    cfg = covid_reference_config(dict(COVID_KWARGS, episode_length=20))
    env = foundation.make_env_instance(cfg.pop("scenario_name"), n_envs=2, auto_reset=True,
                                       stepper_factory=lambda params, n, ar: emu(params, n, ar), **cfg)
    assert env.final_obs is None


# ------------------------------------------------------------------------------------------------ 5. advantages
def value_fns(S, seed=11):
    """A fixed linear value function of the observation: state s from its 9 own features and the 4 scalars, the planner
    from all of them; float64 products rounded to float32."""
    rng = np.random.RandomState(seed)
    wa, wp = rng.standard_normal(13) * 0.1, rng.standard_normal(9 * S + 4) * 0.01

    def feats(o):   # o: name -> [E, ...] numpy
        per = np.concatenate([o["obs_agent_state"], o["obs_postsubsidy"][:, None], o["obs_lagged_stringency"][:, None],
                              o["obs_policy_indicators"][:, None]], axis=1)   # [E, 9, S]
        return per.astype(np.float64), o["obs_scalars"].astype(np.float64)

    def va(o):
        per, sc = feats(o)
        return (np.einsum("efs,f->es", per, wa[:9]) + (sc @ wa[9:])[:, None]).astype(np.float32)

    def vp(o):
        per, sc = feats(o)
        return (np.concatenate([per.reshape(len(sc), -1), sc], axis=1) @ wp).astype(np.float32)
    return va, vp


def host_obs(st, prefix=""):
    return {k: st.to_numpy(st.buf[prefix + k]) for k in _abi.COVID_OBS_NAMES}


def _rollout(F, N, T_roll, next_actions, skip=0):
    """Steps F and N together; records a rollout of T_roll steps after `skip` unrecorded steps.  F's values of its
    final rows are stored at every step; the restatement bootstraps from V of N's observation at the done steps."""
    S = F.p["n_states"]
    va, vp = value_fns(S)
    rec = {k: [] for k in ("ra", "rp", "va", "vp", "fa", "fp", "na", "np", "d")}
    n_alive = True
    for t in range(skip + T_roll):
        if t >= skip:
            o = host_obs(F)
            rec["va"].append(va(o)); rec["vp"].append(vp(o))
        aa, ap = next_actions(F)
        for st in ((F, N) if n_alive else (F,)):
            set_actions(st, aa, ap)
            st.step()
        d = F.to_numpy(F.buf["done"]).copy()
        if t >= skip:
            fo = host_obs(F, "final_")
            rec["fa"].append(va(fo)); rec["fp"].append(vp(fo))
            if d.any():
                no = host_obs(N)
                rec["na"].append(va(no)); rec["np"].append(vp(no))
            else:
                rec["na"].append(np.zeros_like(rec["fa"][-1])); rec["np"].append(np.zeros_like(rec["fp"][-1]))
            rec["ra"].append(F.to_numpy(F.buf["reward_agent"]).copy())
            rec["rp"].append(F.to_numpy(F.buf["reward_planner"]).copy())
            rec["d"].append(d)
        if d.any():
            n_alive = False
    o = host_obs(F)
    R = {k: np.ascontiguousarray(np.stack(v)) for k, v in rec.items()}
    return R, (va(o), vp(o))


def _check_advantages(env_adv, R, lv, gamma, lam, to_dev):
    assert R["d"].any() and R["d"].sum() == R["d"].shape[1]   # one episode end per replica inside the rollout
    out = env_adv(tuple(map(to_dev, (R["ra"], R["rp"]))), tuple(map(to_dev, (R["va"], R["vp"]))), to_dev(R["d"]),
                  tuple(map(to_dev, lv)), tuple(map(to_dev, (R["fa"], R["fp"]))), gamma=gamma, lam=lam)
    out = [np.asarray(x.cpu() if hasattr(x, "cpu") else x) for x in out]
    aa, ra = gae_ref(R["ra"], R["va"], R["d"], lv[0], R["na"], gamma, lam)
    ap, rp = gae_ref(R["rp"], R["vp"], R["d"], lv[1], R["np"], gamma, lam)
    for got, want in zip(out, (aa, ap, ra, rp)):
        assert same_bits(got, want)


def test_emulated_advantages_bootstrap_from_final_obs():
    T = 50
    env = _env(episode_length=T, observe_rate=False)
    env.reset()
    F = env.stepper
    N = emu(F.p, env.n_envs, False)
    N.reset()
    rng = np.random.RandomState(5)
    R, lv = _rollout(F, N, 70, lambda st: random_masked_actions(st, rng))
    assert R["d"][T - 1].all()
    _check_advantages(env.compute_advantages, R, lv, 0.99, 0.95, lambda x: x)


# ------------------------------------------------------------------------------------------------ GPU
def _cuda(params, n, ar, final_obs=False):
    from ai_economist_b200.covid_stepper import CudaCovidStepper
    return CudaCovidStepper(params, n, auto_reset=ar, final_obs=final_obs)


def _cuda_sampler(seed):
    calls = [0]

    def nxt(st):
        calls[0] += 1
        st.sample_random_actions(seed + calls[0])
        return st.buf["actions_agent"].clone(), st.buf["actions_planner"].clone()
    return nxt


@pytest.mark.gpu
@pytest.mark.parametrize("E,T,episodes", [(4096, 540, 1), (4096, 60, 2)], ids=["full_episode", "len60_two_ends"])
def test_cuda_twins(E, T, episodes):
    p = build_covid_params(**dict(COVID_KWARGS, episode_length=T))
    _twins(_cuda, p, E, episodes, _cuda_sampler(100), np.float32(-7.25))


@pytest.mark.gpu
def test_cuda_advantages_bootstrap_from_final_obs():
    import torch
    E, T = 4096, 540
    p = build_covid_params(**dict(COVID_KWARGS, episode_length=T))
    F, N = _cuda(p, E, True, final_obs=True), _cuda(p, E, False)
    F.reset(); N.reset()
    R, lv = _rollout(F, N, 60, _cuda_sampler(300), skip=T - 40)
    assert R["d"][39].all()
    _check_advantages(F.compute_advantages, R, lv, 0.99, 0.95, lambda x: torch.as_tensor(x, device=F.device))


@pytest.mark.gpu
def test_cuda_final_rows_equal_the_emulation():
    import torch
    E, T = 64, 60
    p = build_covid_params(**dict(COVID_KWARGS, episode_length=T))
    g, h = _cuda(p, E, True, final_obs=True), emu(p, E, True, final_obs=True)
    g.reset(); h.reset()
    nxt = _cuda_sampler(500)
    ends = 0
    for t in range(2 * T):
        aa, ap = nxt(g)
        g.step()
        set_actions(h, aa.cpu().numpy(), ap.cpu().numpy())
        h.step()
        if g.to_numpy(g.buf["done"]).any():
            ends += 1
            host = lambda o: {k: v.cpu().numpy() for k, v in o.items()}
            assert same_obs(host(snap(g, "final_")), snap(h, "final_")), t
            assert same_obs(host(snap(g)), snap(h)), t
    torch.cuda.synchronize()
    assert ends == 2
