"""bfloat16 observations of the COVID-19 scenario (aie_covid_config.obs_dtype, make_env_instance(..., obs_dtype=...)).

Contract: each of the seven observation / mask tensors (and their final_ twins) holds the round-to-nearest-even bfloat16
of what a float32 twin writes, bit for bit torch's `.to(torch.bfloat16)`; every other buffer, and the actions and
log-probabilities of both samplers, are byte-identical to the twin's.

CPU (the host build of the device source): float32 / bfloat16 twins across two episode ends over the configs of the
three golden traces and two variant traces, with the auto-reset, change list and final observations on and off; the
rate observation under observe_rate; evaluate_actions on stored bfloat16 masks; advantages fed from a bfloat16
final_obs rollout; the ABI checks; the WarpDrive-style wrapper's spaces.  GPU: CUDA twins at 4 096 replicas, CUDA
bfloat16 against the host build's, and the policy sampler on a bfloat16 env.
"""
import ctypes as C

import numpy as np
import pytest
import torch

from ai_economist_b200 import _abi, foundation
from ai_economist_b200.foundation.covid19 import build_covid_params
from ai_economist_b200.workloads import COVID_KWARGS, covid_reference_config
from tests.test_covid import VARIANTS, load
from tests.test_covid_variants import load as load_variant

AIE_EINVAL, AIE_ESTATE = -1, -3
OTHER_BUFS = ["state", "ints", "hdr", "ring", "changes", "actions_agent", "actions_planner", "reward_agent",
              "reward_planner", "done"]
RATE = "VaccinationCampaign-next_vaccination_rate"
TRACE_CONFIGS = [("golden", n) for n in VARIANTS] + [("variant", "eta05_cooldown7_interval1"),
                                                      ("variant", "late_start_window_drops")]


def emu(params, n, auto_reset, final_obs=False, change_list=True, obs_dtype=None):
    """The COVID-19 stepper over the host emulation of the device source (numpy buffers; bfloat16 as raw bits)."""
    from ai_economist_b200.covid_stepper import CovidStepperBase
    from tests.emu.emu_stepper import emu_lib

    class _Emu(CovidStepperBase):
        def _alloc(self, shape, dt):
            return np.zeros(shape, dtype=self._DT[dt])

        def _ptr(self, buf):
            return buf.ctypes.data_as(C.c_void_p)

        def to_numpy(self, buf):
            return np.array(buf)

    return _Emu(params, n, emu_lib(), auto_reset=auto_reset, change_list=change_list, final_obs=final_obs,
                obs_dtype=obs_dtype)


def rne_bits(x):
    """torch's round-to-nearest-even bfloat16 of float32 x, as int16 bits (numpy in -> numpy out, torch -> torch)."""
    if isinstance(x, np.ndarray):
        return torch.from_numpy(np.ascontiguousarray(x)).to(torch.bfloat16).view(torch.int16).numpy()
    return x.to(torch.bfloat16).view(torch.int16)


def bits(x):
    """int16 bits of a bfloat16 buffer (raw uint16 on numpy backends, torch.bfloat16 on CUDA)."""
    return x.view(np.int16) if isinstance(x, np.ndarray) else x.view(torch.int16)


def same(x, y):
    if isinstance(x, np.ndarray):
        return x.shape == y.shape and x.dtype == y.dtype and x.tobytes() == y.tobytes()
    return x.shape == y.shape and x.dtype == y.dtype and torch.equal(x.reshape(-1).view(torch.uint8),
                                                                     y.reshape(-1).view(torch.uint8))


def check_twins(f, b, label):
    """b (bfloat16) against its float32 twin f: observation buffers (and final_ twins) are the RNE of f's, the rest
    byte-identical."""
    for k in _abi.COVID_OBS_NAMES:
        for name in (k, "final_" + k):
            if name not in f.buf:
                continue
            assert b.buf[name].dtype in (np.uint16, torch.bfloat16), name
            want, got = rne_bits(f.buf[name]), bits(b.buf[name])
            assert same(want, got), (label, name)
    for k in OTHER_BUFS:
        if k in f.buf:
            assert same(f.buf[k], b.buf[k]), (label, k)


def random_logits(rng, st, bf16):
    """Random logits of the policy sampler's shapes, float32 or bfloat16 (raw bits on numpy backends)."""
    sa, sp, _, _ = st._policy_shapes()
    la, lp = rng.standard_normal(sa).astype(np.float32) * 2, rng.standard_normal(sp).astype(np.float32) * 2
    if bf16:
        la, lp = rne_bits(la).view(np.uint16), rne_bits(lp).view(np.uint16)
    if isinstance(st.buf["state"], np.ndarray):
        return la, lp
    return tuple(torch.as_tensor(x.view(np.int16) if bf16 else x, device=st.device).view(torch.bfloat16 if bf16 else torch.float32)
                 for x in (la, lp))


def drive_twins(f, b, steps, seed, reset_at=None):
    """Steps twins f (float32) and b (bfloat16) for `steps` steps, the actions alternating between the random sampler,
    the policy sampler on float32 logits and on bfloat16 logits; checks the actions, log-probabilities and buffers
    after every step.  reset_at: steps after which both are reset (twins without the auto-reset)."""
    rng = np.random.RandomState(seed)
    f.reset(); b.reset()
    check_twins(f, b, "reset")
    ends = 0
    for t in range(steps):
        mode = t % 3
        if mode == 0:
            f.sample_random_actions(seed + t); b.sample_random_actions(seed + t)
        else:
            la, lp = random_logits(rng, f, bf16=mode == 2)
            lfa, lfp = f.sample_policy(la, lp, seed=seed + t)
            lba, lbp = b.sample_policy(la, lp, seed=seed + t)
            assert same(lfa, lba) and same(lfp, lbp), t
        assert same(f.buf["actions_agent"], b.buf["actions_agent"]) and same(f.buf["actions_planner"], b.buf["actions_planner"]), t
        f.step(); b.step()
        check_twins(f, b, t)
        ends += int(f.to_numpy(f.buf["done"]).any())
        if reset_at and (t + 1) % reset_at == 0:
            f.reset(); b.reset()
            check_twins(f, b, ("reset", t))
    return ends


def trace_params(kind, name):
    return (load(name) if kind == "golden" else load_variant(name))[2]


# (auto_reset, final_obs, change_list): each option on and off at least once
MODES = [(True, True, True), (True, False, False), (False, False, True), (True, True, False)]


@pytest.mark.parametrize("mode", MODES, ids=["autoreset_final_list", "autoreset_scan", "noreset_list", "autoreset_final_scan"])
@pytest.mark.parametrize("kind,name", TRACE_CONFIGS, ids=[n.replace(".npz", "") for _, n in TRACE_CONFIGS])
def test_emulated_twins_across_two_episode_ends(kind, name, mode):
    auto_reset, final_obs, change_list = mode
    p = trace_params(kind, name)
    T = p["episode_length"]
    mk = lambda dt: emu(p, 2, auto_reset, final_obs=final_obs, change_list=change_list, obs_dtype=dt)
    f, b = mk(None), mk(torch.bfloat16)
    assert f.obs_dtype == "float32" and b.obs_dtype == "bfloat16"
    ends = drive_twins(f, b, 2 * T, 17, reset_at=None if auto_reset else T)
    assert ends == 2
    # read_obs hands out exact float32
    for k, v in b.read_obs(1).items():
        if v.dtype == np.float32 and k not in ("rew_a",):
            assert v.tobytes() == torch.from_numpy(f.read_obs(1)[k]).to(torch.bfloat16).float().numpy().tobytes(), k


# ------------------------------------------------------------------------------------------------ rate observation
def _cfg(episode_length=540, observe_rate=True, early_vaccines=True):
    """early_vaccines: deliveries begin at t = 14 (else the workload's dates: at t = 296)."""
    kw = dict(COVID_KWARGS, episode_length=episode_length)
    if early_vaccines:
        kw.update(start_date="2020-12-01", delivery_interval=7, vaccine_delivery_start_date="2020-12-15")
    cfg = covid_reference_config(kw)
    if observe_rate:
        for c in cfg["components"]:
            if "VaccinationCampaign" in c:
                c["VaccinationCampaign"]["observe_rate"] = True
    return cfg


def _env(obs_dtype=None, final_obs=True, n_envs=2, episode_length=540, observe_rate=True, early_vaccines=True):
    cfg = _cfg(episode_length, observe_rate, early_vaccines)
    factory = lambda params, n, ar, **k: emu(params, n, ar, **k)
    return foundation.make_env_instance(cfg.pop("scenario_name"), n_envs=n_envs, auto_reset=True,
                                        final_obs=final_obs, obs_dtype=obs_dtype, stepper_factory=factory, **cfg)


def test_rate_observation_at_every_timestep():
    """next_vaccination_rate of a bfloat16 env is the RNE of its float32 twin's at every t of a 540-step episode, the
    final rows included.  The bfloat16 time scalar alone cannot give it: t / 540 rounded to bfloat16 maps distinct
    timesteps onto one value: with deliveries from t = 296 on, t = 296 reads as 295, before the rate switches on."""
    f, b = _env(None, early_vaccines=False), _env(torch.bfloat16, early_vaccines=False)
    f.reset(); b.reset()
    T = f.episode_length
    scalar_t, true_t = [], []
    for t in range(T + 1):
        for g in ("a", "p"):
            assert same(rne_bits(f.obs[g][RATE]), bits(b.obs[g][RATE])), (t, g)
            assert same(rne_bits(f.final_obs[g][RATE]), bits(b.final_obs[g][RATE])), (t, g)
            assert b.obs[g][RATE].dtype == np.uint16 and f.obs[g][RATE].dtype == np.float32
        sc = b.stepper.obs_to_numpy("obs_scalars")[:, 0].astype(np.float64) * float(b.params["time_scale"])
        scalar_t.append(np.rint(sc).astype(np.int64)); true_t.append(b.stepper.buf["hdr"][:, 0].copy())
        if t < T:
            f.step(None); b.step(None)
    assert (f.done["__all__"] == 1).all()
    tab = f._rate_tab
    assert len(set(tab.tolist())) == 2   # the rate switches on inside the episode
    # the scalar-based lookup the float32 env uses would read the wrong timestep (and rate) under bfloat16
    scalar_t, true_t = np.array(scalar_t), np.array(true_t)
    assert (scalar_t != true_t).any()
    assert (tab[np.minimum(scalar_t, T)] != tab[true_t]).any()


def test_env_surface_and_stepper_factory_checks():
    env = _env(torch.bfloat16)
    assert env.obs["a"]["world-agent_state"].dtype == np.uint16
    assert env.final_obs["p"]["action_mask"] is env.stepper.buf["final_mask_planner"]
    assert env.rew["p"].dtype == np.float64 and env.rew["a"].dtype == np.float32
    assert _env("bfloat16").stepper.obs_dtype == "bfloat16"
    assert _env(torch.float32).stepper.obs_dtype == "float32"
    with pytest.raises(ValueError):
        _env("float16")
    # a factory whose stepper ignores obs_dtype is refused; a three-argument factory still serves float32
    cfg = _cfg(20, False)
    with pytest.raises(NotImplementedError, match="obs_dtype"):
        foundation.make_env_instance(cfg.pop("scenario_name"), n_envs=2, obs_dtype=torch.bfloat16,
                                     stepper_factory=lambda params, n, ar, **k: emu(params, n, ar), **cfg)
    cfg = _cfg(20, False)
    env = foundation.make_env_instance(cfg.pop("scenario_name"), n_envs=2,
                                       stepper_factory=lambda params, n, ar: emu(params, n, ar), **cfg)
    assert env.obs["a"]["action_mask"].dtype == np.float32


def test_warpdrive_wrapper_spaces_are_float32_over_bfloat16_tensors():
    from ai_economist_b200.adapters import WarpDriveStyleEnvWrapper
    env = _env(torch.bfloat16, final_obs=False)
    w = WarpDriveStyleEnvWrapper(env)
    for who in ("0", "p"):
        for k, sp in w.env.observation_space[who].spaces.items():
            assert np.dtype(sp.dtype) == np.float32, (who, k)
    assert w.tensor("observations_a_world-agent_state") is env.stepper.buf["obs_agent_state"]
    assert w.tensor("observations_a_world-agent_state").dtype == np.uint16


# ------------------------------------------------------------------------------------------------ training loop
def test_evaluate_actions_on_stored_bfloat16_masks():
    f, b = _env(None, final_obs=False), _env(torch.bfloat16, final_obs=False)
    f.reset(); b.reset()
    rng = np.random.RandomState(3)
    store = {k: [] for k in ("mfa", "mfp", "mba", "mbp", "aa", "ap")}
    for t in range(40):
        for env, ka, kp in ((f, "mfa", "mfp"), (b, "mba", "mbp")):
            store[ka].append(env.obs["a"]["action_mask"].copy()); store[kp].append(env.obs["p"]["action_mask"].copy())
        f.stepper.sample_random_actions(t); b.stepper.sample_random_actions(t)
        store["aa"].append(f.stepper.buf["actions_agent"].copy()); store["ap"].append(f.stepper.buf["actions_planner"].copy())
        f.step(f.action_buffers); b.step(b.action_buffers)
    S = {k: np.ascontiguousarray(np.stack(v)) for k, v in store.items()}
    la = rng.standard_normal(S["aa"].shape + (f.stepper.p["num_stringency_levels"] + 1,)).astype(np.float32)
    lp = rng.standard_normal(S["mfp"].shape).astype(np.float32)
    for logits in ((la, lp), (rne_bits(la).view(np.uint16), rne_bits(lp).view(np.uint16))):
        of = f.evaluate_actions(*logits, (S["aa"], S["ap"]), (S["mfa"], S["mfp"]))
        ob = b.evaluate_actions(*logits, (S["aa"], S["ap"]), (S["mba"], S["mbp"]))
        for x, y in zip(of, ob):
            assert same(x, y)


def test_advantages_from_a_bfloat16_final_obs_rollout():
    from tests.test_covid_final_obs import value_fns
    T = 30
    env = _env(torch.bfloat16, final_obs=True, n_envs=3, episode_length=T, observe_rate=False)
    env.reset()
    st = env.stepper
    va, vp = value_fns(env.n_agents)
    obs = lambda prefix: {k: st.obs_to_numpy(prefix + k) for k in _abi.COVID_OBS_NAMES}
    R = {k: [] for k in ("ra", "rp", "va", "vp", "fa", "fp", "d")}
    for t in range(T + 10):
        o = obs("")
        R["va"].append(va(o)); R["vp"].append(vp(o))
        st.sample_random_actions(t)
        env.step(env.action_buffers)
        fo = obs("final_")
        R["fa"].append(va(fo)); R["fp"].append(vp(fo))
        R["ra"].append(env.rew["a"].copy()); R["rp"].append(env.rew["p"].copy()); R["d"].append(env.done["__all__"].copy())
    R = {k: np.ascontiguousarray(np.stack(v)) for k, v in R.items()}
    assert R["d"][T - 1].all() and R["d"].sum() == env.n_envs
    o = obs("")
    adv_a, adv_p, ret_a, ret_p = env.compute_advantages((R["ra"], R["rp"]), (R["va"], R["vp"]), R["d"], (va(o), vp(o)),
                                                        (R["fa"], R["fp"]), gamma=0.99, lam=0.95)
    assert adv_a.shape == R["va"].shape and adv_p.shape == R["vp"].shape
    assert np.isfinite(adv_a).all() and np.isfinite(ret_p).all()


# ------------------------------------------------------------------------------------------------ ABI
def _config(p, obs_dtype):
    from ai_economist_b200.covid_stepper import covid_config_from_params
    cfg, keep = covid_config_from_params(p, True, obs_dtype)
    return cfg, keep


def test_abi_obs_dtype_and_version_checks():
    from tests.emu.emu_stepper import emu_lib
    L = emu_lib()
    p = build_covid_params(**dict(COVID_KWARGS, episode_length=20))
    assert L.aie_abi_version() == 6 == _abi.ABI_VERSION
    cfg, keep = _config(p, torch.bfloat16)
    assert cfg.obs_dtype == _abi.OBS_BF16
    h = C.c_void_p()
    for bad in (2, -1):
        cfg.obs_dtype = bad
        assert L.aie_covid_create(C.byref(cfg), 2, 0, C.byref(h)) == AIE_EINVAL and b"obs_dtype" in L.aie_last_error()
    cfg.obs_dtype = _abi.OBS_BF16
    cfg.abi_version = 5   # a config laid out for ABI 5 (without obs_dtype)
    assert L.aie_covid_create(C.byref(cfg), 2, 0, C.byref(h)) == AIE_EINVAL and b"abi_version" in L.aie_last_error()
    cfg.abi_version = _abi.ABI_VERSION
    assert L.aie_covid_create(C.byref(cfg), 2, 0, C.byref(h)) == 0
    L.aie_covid_destroy(h)


def test_abi_step_final_alignment_and_launch_counts():
    from tests.emu.emu_stepper import emu_lib
    L = emu_lib()
    p = build_covid_params(**dict(COVID_KWARGS, episode_length=20))
    f = emu(p, 2, True, final_obs=True)
    b = emu(p, 2, True, final_obs=True, obs_dtype="bfloat16")
    f.reset(); b.reset()
    n0 = b.launch_count()
    assert n0 == f.launch_count() == 1
    raw = np.zeros(4096, np.uint8)
    base = (-raw.ctypes.data) % 16
    two = raw[base + 2:].ctypes.data   # 2-byte but not 4-byte aligned
    odd = raw[base + 1:].ctypes.data
    call = lambda st, out: L.aie_covid_step_final(st._h, C.byref(out), None)
    for k in _abi.COVID_OBS_NAMES:
        fb = _abi.AieCovidObsBuffers()
        for j in _abi.COVID_OBS_NAMES:
            setattr(fb, j, b.buf["final_" + j].ctypes.data)
        setattr(fb, k, odd)
        assert call(b, fb) == AIE_EINVAL and b"2-byte aligned" in L.aie_last_error(), k
        setattr(fb, k, two)   # 2-byte aligned: accepted (the scratch holds every tensor of these 2 replicas)
        assert call(b, fb) == 0, k
    assert b.launch_count() == n0 + len(_abi.COVID_OBS_NAMES)
    ffb = _abi.AieCovidObsBuffers()
    for j in _abi.COVID_OBS_NAMES:
        setattr(ffb, j, f.buf["final_" + j].ctypes.data)
    setattr(ffb, "obs_scalars", two)
    assert call(f, ffb) == AIE_EINVAL and b"4-byte aligned" in L.aie_last_error()
    # every entry point is one launch, as for the float32 env
    for st in (f, b):
        st.sample_random_actions(1)
        st.step()
        st.sample_policy(*random_logits(np.random.RandomState(0), st, False), seed=1)
        st.sample_policy(*random_logits(np.random.RandomState(0), st, True), seed=1)
        st.reset()
    assert b.launch_count() - (n0 + len(_abi.COVID_OBS_NAMES)) == f.launch_count() - n0 == 5


# ------------------------------------------------------------------------------------------------ GPU
def _cuda(params, n, ar, final_obs=False, obs_dtype=None):
    from ai_economist_b200.covid_stepper import CudaCovidStepper
    return CudaCovidStepper(params, n, auto_reset=ar, final_obs=final_obs, obs_dtype=obs_dtype)


@pytest.mark.gpu
@pytest.mark.parametrize("E,T,episodes", [(4096, 540, 1), (4096, 60, 2)], ids=["full_episode", "len60_two_ends"])
def test_cuda_twins(E, T, episodes):
    p = build_covid_params(**dict(COVID_KWARGS, episode_length=T))
    f, b = _cuda(p, E, True, final_obs=True), _cuda(p, E, True, final_obs=True, obs_dtype=torch.bfloat16)
    assert b.buf["obs_agent_state"].dtype == torch.bfloat16 and b.buf["final_mask_agent"].dtype == torch.bfloat16
    ends = drive_twins(f, b, episodes * T, 100)
    torch.cuda.synchronize()
    assert ends == episodes


@pytest.mark.gpu
def test_cuda_bfloat16_equals_the_emulation():
    E, T = 64, 60
    p = build_covid_params(**dict(COVID_KWARGS, episode_length=T))
    g, h = _cuda(p, E, True, final_obs=True, obs_dtype="bfloat16"), emu(p, E, True, final_obs=True, obs_dtype="bfloat16")
    g.reset(); h.reset()
    host = lambda x: x.view(torch.int16).cpu().numpy().view(np.uint16) if x.dtype == torch.bfloat16 else x.cpu().numpy()
    ends = 0
    for t in range(2 * T):
        g.sample_random_actions(500 + t)
        h.buf["actions_agent"][...] = host(g.buf["actions_agent"]); h.buf["actions_planner"][...] = host(g.buf["actions_planner"])
        g.step(); h.step()
        for k in h.buf:
            assert same(host(g.buf[k]), h.buf[k]), (t, k)
        ends += int(h.buf["done"].any())
    assert ends == 2


@pytest.mark.gpu
def test_cuda_policy_sampler_on_a_bfloat16_env():
    E, T = 1024, 90
    p = build_covid_params(**dict(COVID_KWARGS, episode_length=T))
    f, b = _cuda(p, E, True), _cuda(p, E, True, obs_dtype=torch.bfloat16)
    f.reset(); b.reset()
    rng = np.random.RandomState(9)
    for t in range(T + 5):
        la, lp = random_logits(rng, f, bf16=t % 2 == 1)
        for greedy in (False, True):
            of = f.sample_policy(la, lp, seed=t, greedy=greedy)
            ob = b.sample_policy(la, lp, seed=t, greedy=greedy)
            assert same(of[0], ob[0]) and same(of[1], ob[1]), t
            assert same(f.buf["actions_agent"], b.buf["actions_agent"]), t
            assert same(f.buf["actions_planner"], b.buf["actions_planner"]), t
        f.step(); b.step()
        check_twins(f, b, t)
    torch.cuda.synchronize()
