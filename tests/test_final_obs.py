"""Final observations of the episodes the auto-reset ends (`make_env_instance(..., final_obs=True)`).

Contract: after a step, row e of every final_<name> buffer of a replica whose done flag is set holds, byte for byte, what
the step's own observation pass would have written for that replica without the auto-reset (the observation of the state
its episode ended in); rows of the other replicas are left untouched, and nothing else the env computes changes.  The CPU
tests run through the host emulation of the device source (tests/emu), the `-m gpu` tests through the CUDA kernels.
A split record (AIE_SPLIT=1) keeps its price history in global memory, and only the device's auto-reset copies it into
the episode_final snapshot (the emulation's copies the resident part and the statistics), so split records are compared
on the GPU: against the no-auto-reset twin, and against the emulation's pass over the device's records.
"""
import ctypes as C

import numpy as np
import pytest
import torch

from ai_economist_b200 import _abi, foundation
from tests import batch_utils as bu
from tests import golden_utils as gu
from tests.test_obs_bf16 import _bits16, _bytes, _cfg, rne_bits

OBS = _abi.OBS_NAMES
BF16_KEYS = ("obs_agent_map", "obs_agent_flat", "mask_agent", "obs_planner_map", "obs_planner_flat",
             "obs_planner_agents", "mask_planner", "obs_time")


def _make(name, kw, E, factory, seeds, **extra):
    dev = dict(stepper_factory=factory) if factory is not None else dict(device="cuda:0")
    return foundation.make_env_instance(name, n_envs=E, seeds=seeds, **dev, **extra, **kw)


def _row(buf, e):
    return _bytes(buf[e:e + 1])


def _stagger(env, E):
    T = env.episode_length
    v = env.stepper.state_view("t")
    start = (np.arange(E, dtype=np.int64) * T // E).astype(np.int32)
    if isinstance(v, np.ndarray):
        v[...] = start
    else:
        v.copy_(torch.as_tensor(start, device=v.device))


def run_final_twins(name, kw, E, factory, obs_dtype=None, steps=None, seed0=500):
    """F (auto-reset, final_obs) and N (auto_reset=False) from the same seeds, staggered the same way, stepped with the
    same host-drawn actions; at the step where replica e first reports done, F's final rows equal N's output rows."""
    seeds = [seed0 + 7 * e for e in range(E)]
    F = _make(name, kw, E, factory, seeds, auto_reset=True, final_obs=True, obs_dtype=obs_dtype)
    N = _make(name, kw, E, factory, seeds, auto_reset=False, obs_dtype=obs_dtype)
    sf, sn = F.stepper, N.stepper
    assert set(sf.buf) == set(sn.buf) | {"episode_final"} | {"final_" + k for k in OBS if k in sn.buf}
    for env in (F, N):
        env.reset()
        _stagger(env, E)
        env.stepper.observe()
    sp = F.spec
    seg_a, seg_p = bu.segments(sp, "a"), bu.segments(sp, "p")
    rng = np.random.RandomState(11)
    T = F.episode_length
    ended = np.zeros(E, bool)
    for t in range(1, (steps or T + 1) + 1):
        aa = bu.sample_from_masks(sf.obs_to_numpy("mask_agent"), seg_a, rng)
        ap = bu.sample_from_masks(sf.obs_to_numpy("mask_planner"), seg_p, rng) if seg_p else None
        F.step((aa, ap))
        N.step((aa, ap))
        done_f, done_n = sf.to_numpy(sf.buf["done"]), sn.to_numpy(sn.buf["done"])
        for e in np.nonzero(~ended)[0]:
            assert done_f[e] == done_n[e], "t=%d replica %d: done" % (t, e)
            assert np.array_equal(_row(sf.buf["reward"], e), _row(sn.buf["reward"], e)), "t=%d replica %d: reward" % (t, e)
            if done_f[e]:
                for k in OBS:
                    if k in sn.buf:
                        assert np.array_equal(_row(sf.buf["final_" + k], e), _row(sn.buf[k], e)), \
                            "t=%d replica %d: final_%s" % (t, e, k)
                ended[e] = True
    assert ended.all(), "every replica ends an episode"
    return F, N


# ---- CPU: the reference's last-step observations --------------------------------------------------------------------
ENDING_TRACES = ["c1_tutorial_seed1001", "c3_short_period_seed1001", "c5_small_seed1001", "full_obs_tax_seed1001",
                 "multi_zone_seed1001", "quadrant_seed1001", "ref_unit_test_seed1001", "split_layout_seed1001",
                 "tax_single_planner_seed1001", "tax_us_federal_seed1001", "uniform_halfwidth_seed1001"]


def _final_obs_of(st, e):
    """read_obs(e) over the final_<name> buffers."""
    g = lambda k: st.obs_to_numpy("final_" + k, e) if "final_" + k in st.buf else None
    out = dict(a_map=g("obs_agent_map"), a_idx=g("obs_agent_idx"), a_flat=g("obs_agent_flat"), a_mask=g("mask_agent"),
               p_flat=g("obs_planner_flat"), p_agents=g("obs_planner_agents"), p_mask=g("mask_planner"),
               time=np.atleast_1d(g("obs_time")))
    if "final_obs_planner_map" in st.buf:
        out["p_map"], out["p_idx"] = g("obs_planner_map"), g("obs_planner_idx")
    return out


def _replay_to_end(path, obs_dtype):
    from tests.emu.emu_stepper import EmuStepper
    from tests.stepper_adapters import GoldenStepperAdapter
    z, meta, init = gu.load_fixture(path)
    spec = dict(meta["spec"], final_obs=True, obs_dtype=obs_dtype)
    ad = GoldenStepperAdapter(EmuStepper(spec, 1, auto_reset=True), init)
    n = int(meta["n_steps"])
    assert n == spec["episode_length"] and int(z["step_done"][n]) == 1
    for t in range(1, n + 1):
        ap = z["act_p"][t - 1].astype(np.int32)
        ad.step(z["act_a"][t - 1].astype(np.int32), ap if ap.size else None)
    return z, ad.s, n


@pytest.mark.parametrize("trace", ENDING_TRACES)
def test_final_obs_of_the_last_step_match_reference_trace(trace):
    """Each trace ends on its episode's last step: with auto-reset the reference's last-step observations become the
    final observations, at the trace's tolerances; reward and done are the trace's."""
    path = [p for p in gu.golden_files() if p.endswith("/" + trace + ".npz")][0]
    z, st, n = _replay_to_end(path, "float32")
    o, full_idx = _final_obs_of(st, 0), {int(t): i for i, t in enumerate(z["full_steps"])}[n]
    sp = bool(st.spec["planner_gets_spatial_info"])
    assert int(st.to_numpy(st.buf["done"])[0]) == 1
    assert np.allclose(z["step_rew"][n], st.to_numpy(st.buf["reward"])[0], rtol=gu.RTOL, atol=gu.ATOL_F64)
    assert int(st.to_numpy(st.state_view("t"))[0]) == 0, "the live record has been auto-reset"
    for k in gu.EXACT_OBS:
        if "step_%s_crc" % k in z.files and (sp or k not in ("p_map", "p_idx")):
            assert gu.crc(o[k]) == int(z["step_%s_crc" % k][n]), k
        if "full_" + k in z.files and (sp or k not in ("p_map", "p_idx")):
            ref = z["full_" + k][full_idx]
            assert np.array_equal(ref.astype(o[k].dtype), np.asarray(o[k]).reshape(ref.shape)), k
    for k in gu.FLOAT_OBS:
        ref = z["full_" + k][full_idx]
        assert np.allclose(ref, np.asarray(o[k]).reshape(ref.shape), rtol=gu.RTOL, atol=gu.ATOL_F32), k


@pytest.mark.parametrize("trace", ["c3_short_period_seed1001", "full_obs_tax_seed1001", "multi_zone_seed1001",
                                   "tax_single_planner_seed1001"])
def test_bf16_final_obs_are_the_rounded_float32_final_obs(trace):
    path = [p for p in gu.golden_files() if p.endswith("/" + trace + ".npz")][0]
    _, s32, _ = _replay_to_end(path, "float32")
    _, s16, _ = _replay_to_end(path, "bfloat16")
    for k in OBS:
        if "final_" + k not in s32.buf:
            continue
        a, b = s32.buf["final_" + k], s16.buf["final_" + k]
        if k in BF16_KEYS:
            assert np.array_equal(rne_bits(a), _bits16(b)), k
        else:
            assert np.array_equal(_bytes(a), _bytes(b)), k


# ---- CPU: F / N twins through the emulation ----------------------------------------------------------------------
TWIN_CASES = [
    ("c1_tutorial", {}),                                    # fixed layout
    ("c3_short_period", {}),                                # c3-like tax
    ("saez_reset", {}),                                     # Saez (host estimator)
    ("split_layout", {}),
    ("uniform_halfwidth", {}), ("quadrant", {}), ("multi_zone", {}),
    ("one_step", {}),
    ("c1_tutorial", dict(multi_action_mode_agents=True)),
    ("tax_single_planner", {}),                             # single-action planner
    ("full_obs_tax", {}),
    ("c1_tutorial", dict(planner_gets_spatial_info=False)),
]


def _twin_cfg(cfg, over):
    over = dict(over)
    if cfg != "one_step":
        over.setdefault("episode_length", 7)
    return _cfg(cfg, **over)


@pytest.mark.parametrize("obs_dtype", ["float32", "bfloat16"])
@pytest.mark.parametrize("cfg,over", TWIN_CASES, ids=["%s-%s" % (c, "_".join(sorted(o)) or "plain") for c, o in TWIN_CASES])
def test_emulated_final_obs_equal_the_no_auto_reset_twin(cfg, over, obs_dtype):
    from tests.emu.emu_stepper import emu_factory
    name, kw = _twin_cfg(cfg, over)
    run_final_twins(name, kw, 3, emu_factory, obs_dtype=obs_dtype)


@pytest.mark.parametrize("nt", [32, 128])
@pytest.mark.parametrize("obs_dtype", ["float32", "bfloat16"])
@pytest.mark.parametrize("cfg", ["c3_short_period", "full_obs_tax", "c5_small"])
def test_emulated_final_obs_thread_walks(cfg, obs_dtype, nt, monkeypatch):
    from tests.emu.emu_stepper import emu_factory
    monkeypatch.setenv("AIE_EMU_NT", str(nt))
    name, kw = _cfg(cfg, episode_length=5)
    run_final_twins(name, kw, 2, emu_factory, obs_dtype=obs_dtype)


@pytest.mark.parametrize("view", [dict(flatten_observations=False, flatten_masks=False),
                                  dict(collate_agent_step_and_reset_data=True), {}], ids=["named", "collated", "flat"])
def test_final_obs_views_mirror_obs(view):
    """env.final_obs has env.obs's keys and views, over the final tensors; final_obs_tensors mirrors obs_tensors."""
    from tests.emu.emu_stepper import emu_factory
    name, kw = _cfg("c3_short_period", episode_length=4, **view)
    env = _make(name, kw, 2, emu_factory, [3, 4], auto_reset=True, final_obs=True)
    env.reset()
    st = env.stepper
    assert set(env.final_obs_tensors) == set(env.obs_tensors)
    for k, v in env.final_obs_tensors.items():
        assert v is st.buf["final_" + k] and v.shape == env.obs_tensors[k].shape and v.dtype == env.obs_tensors[k].dtype

    def walk(a, b, path=""):
        assert type(a) is type(b), path
        if isinstance(a, dict):
            assert list(a) == list(b), path
            for k in a:
                walk(a[k], b[k], path + "/" + k)
        else:
            assert a.shape == b.shape and a.dtype == b.dtype, path
            assert np.shares_memory(a, b) is False, path

    walk(env.obs, env.final_obs)
    for _ in range(4):
        env.step()
    assert st.to_numpy(st.buf["done"]).all()
    # the views slice the final tensors
    assert np.shares_memory(env.final_obs["p"]["time"], env.final_obs_tensors["obs_time"])


# ---- CPU: rows the pass must not touch --------------------------------------------------------------------------
def _fill(st, byte):
    for k in OBS:
        if "final_" + k in st.buf:
            st.buf["final_" + k].view(np.uint8)[...] = byte


def test_untouched_rows_keep_their_contents_and_reset_leaves_them_alone():
    from tests.emu.emu_stepper import emu_factory
    name, kw = _cfg("c3_short_period", episode_length=6)
    E = 4
    env = _make(name, kw, E, emu_factory, [20 + e for e in range(E)], auto_reset=True, final_obs=True)
    env.reset()
    st = env.stepper
    st.state_view("t")[...] = np.array([5, 2, 5, 0], np.int32)   # replicas 0 and 2 end with the next step
    _fill(st, 0xA5)
    env.step()
    assert st.to_numpy(st.buf["done"]).tolist() == [1, 0, 1, 0]
    for k in OBS:
        if "final_" + k not in st.buf:
            continue
        b = st.buf["final_" + k]
        for e in (1, 3):
            assert (_row(b, e) == 0xA5).all(), "final_%s row %d" % (k, e)
        if b[0].size:
            assert not (_row(b, 0) == 0xA5).all(), "final_%s row 0 written" % k
    snap = {k: np.array(st.buf["final_" + k]) for k in OBS if "final_" + k in st.buf}
    n0 = st.launch_count()
    env.reset()
    assert st.launch_count() > n0
    for k, v in snap.items():
        assert np.array_equal(_bytes(st.buf["final_" + k]), _bytes(v)), k


def test_option_off_adds_no_buffers_launches_or_changes():
    """final_obs off: no final buffers and one launch per step; on: one more launch per step, and every other buffer,
    including the fused policy's actions, byte-identical to the option-off env."""
    from tests.emu.emu_stepper import emu_factory
    name, kw = _cfg("c3_short_period", episode_length=5)
    seeds = [40, 41, 42]
    off = _make(name, kw, 3, emu_factory, seeds, auto_reset=True)
    on = _make(name, kw, 3, emu_factory, seeds, auto_reset=True, final_obs=True)
    assert not any(k.startswith("final_") for k in off.stepper.buf) and off.final_obs is None
    assert off.spec["final_obs"] is False and on.spec["final_obs"] is True
    for env in (off, on):
        env.reset()
        _stagger(env, 3)
        env.stepper.set_fused_policy(99)
    for t in range(12):
        counts = []
        for env in (off, on):
            n0 = env.stepper.launch_count()
            env.step(env.action_buffers)
            counts.append(env.stepper.launch_count() - n0)
        assert counts == [1, 2], counts
        for k in off.stepper.buf:
            assert np.array_equal(_bytes(off.stepper.buf[k]), _bytes(on.stepper.buf[k])), "t=%d %s" % (t, k)


def test_keyword_checks():
    from ai_economist_b200 import workloads as wl
    from tests.emu.emu_stepper import emu_factory
    name, kw = _cfg("c1_tutorial", episode_length=5)
    with pytest.raises(ValueError, match="auto_reset"):
        _make(name, kw, 1, emu_factory, [1], auto_reset=False, final_obs=True)
    cfg = wl.covid_reference_config()
    cname = cfg.pop("scenario_name")
    with pytest.raises(NotImplementedError):
        foundation.make_env_instance(cname, n_envs=1, stepper_factory=lambda *a, **k: None, final_obs=True, **cfg)


def test_observe_final_into_other_destinations():
    """observe_final(out=...) writes a caller's buffers (a rollout slot), the same bytes as the final buffers."""
    from tests.emu.emu_stepper import emu_factory
    name, kw = _cfg("full_obs_tax", episode_length=3)
    env = _make(name, kw, 2, emu_factory, [5, 6], auto_reset=True, final_obs=True)
    env.reset()
    st = env.stepper
    for _ in range(3):
        env.step()
    slot = {k: np.zeros_like(st.buf[k]) for k in OBS if k in st.buf}
    assert st.observe_final(out=slot) is slot
    for k, v in slot.items():
        assert np.array_equal(_bytes(v), _bytes(st.buf["final_" + k])), k
    bad = dict(slot, obs_agent_flat=slot["obs_agent_flat"][:, :, :-1])
    with pytest.raises(_abi.AieError, match="obs_agent_flat"):
        st.observe_final(out=bad)
    missing = {k: v for k, v in slot.items() if k != "mask_planner"}
    with pytest.raises(_abi.AieError, match="mask_planner"):
        st.observe_final(out=missing)
    plain = _make(name, kw, 2, emu_factory, [5, 6], auto_reset=True)
    plain.reset()
    with pytest.raises(_abi.AieError, match="final_obs is off"):
        plain.stepper.observe_final()


# ---- CPU: C-ABI --------------------------------------------------------------------------------------------------
def test_abi_errors():
    from tests.emu.emu_stepper import EmuStepper, emu_factory, emu_lib
    L = emu_lib()
    name, kw = _cfg("c3_short_period", episode_length=5)
    env = _make(name, kw, 2, emu_factory, [1, 2], auto_reset=True, final_obs=True)
    st = env.stepper

    def obs_bufs(**over):
        o = _abi.AieObsBuffers()
        for k in OBS:
            if k in st.buf:
                setattr(o, k, st._ptr(st.buf["final_" + k]))
        for k, v in over.items():
            setattr(o, k, v)
        return o

    def call(h, o):
        return L.aie_observe_final(h, o if o is None else C.byref(o), None)

    assert call(st._h, obs_bufs()) == -3 and b"load state" in L.aie_last_error()   # AIE_ESTATE: nothing loaded
    env.reset()
    assert call(st._h, None) == -1 and b"null argument" in L.aie_last_error()     # AIE_EINVAL
    assert call(st._h, obs_bufs(mask_agent=None)) == -1 and b"required buffer is NULL" in L.aie_last_error()
    assert call(st._h, obs_bufs(obs_planner_map=None)) == -1                       # planner_gets_spatial_info
    misaligned = st.buf["final_obs_agent_flat"].ctypes.data + 2
    assert call(st._h, obs_bufs(obs_agent_flat=misaligned)) == -1 and b"aligned" in L.aie_last_error()
    misaligned_idx = st.buf["final_obs_agent_idx"].ctypes.data + 1
    assert call(st._h, obs_bufs(obs_agent_idx=misaligned_idx)) == -1
    assert call(st._h, obs_bufs()) == 0
    # bound but without episode_final records: auto-reset off
    n = EmuStepper(dict(env.spec, final_obs=False), 2, auto_reset=False)
    n.load_state(env.host_reset_arrays())
    assert call(n._h, obs_bufs()) == -3 and b"episode_final" in L.aie_last_error()
    # not bound at all
    h = C.c_void_p()
    cfg = _abi.config_from_spec(env.spec)
    assert L.aie_create(C.byref(cfg), 2, 0, C.byref(h)) == 0
    assert call(h, obs_bufs()) == -3 and b"bind buffers" in L.aie_last_error()
    L.aie_destroy(h)


# ---- CPU: compiled code --------------------------------------------------------------------------------------------
def test_new_kernels_are_compiled_for_both_element_types():
    import subprocess
    from tests import test_step_kernel_footprint as fp
    lib = fp.build_library()
    names = subprocess.run([fp._tool("cuobjdump"), "-symbols", lib], check=True, capture_output=True, text=True).stdout
    for k in ("aie_observe_final_kernel", "aie_observe_final_bf16_kernel"):
        for ext in ("Lb0E", "Lb1E"):
            assert ("%d%s%s" % (len(k), k, "I" + ext)) in names, (k, ext)


# ---- GPU ----------------------------------------------------------------------------------------------------------
def _gpu_twins(cfg_name, E, obs_dtype, steps_extra=7, knob_cfg=None):
    name, kw = bu.product_kwargs(cfg_name) if knob_cfg is None else _cfg(cfg_name, episode_length=9)
    if cfg_name == "c5_full":
        kw["device_reset"] = "snapshot"
    seeds = [2000 + e for e in range(E)]
    F = _make(name, kw, E, None, seeds, auto_reset=True, final_obs=True, obs_dtype=obs_dtype)
    N = _make(name, kw, E, None, seeds, auto_reset=False, obs_dtype=obs_dtype)
    T = F.episode_length
    for env in (F, N):
        env.reset()
        _stagger(env, E)
        env.stepper.observe()
        env.stepper.set_fused_policy(4321)
    sf, sn = F.stepper, N.stepper
    keys = [k for k in OBS if k in sn.buf and sn.buf[k].numel()]
    ended = torch.zeros(E, dtype=torch.bool, device="cuda:0")
    for t in range(T + steps_extra):
        sf.step()
        sn.step()
        live = ~ended
        assert torch.equal(sf.buf["done"][live], sn.buf["done"][live]), "t=%d done" % t
        assert torch.equal(sf.buf["reward"][live], sn.buf["reward"][live]), "t=%d reward" % t
        now = live & (sf.buf["done"] != 0)
        if bool(now.any()):
            for k in keys:
                a, b = sf.buf["final_" + k][now], sn.buf[k][now]
                assert torch.equal(a.view(torch.uint8) if a.dtype != torch.uint8 else a,
                                   b.view(torch.uint8) if b.dtype != torch.uint8 else b), "t=%d final_%s" % (t, k)
        ended |= now
    assert bool(ended.all()), "every replica ends an episode within T + 7 steps"
    return F, N, name, kw


def _check_against_emulation(F, name, kw, obs_dtype):
    """The rows of the replicas that finished in the latest step against the emulation's pass over the same records."""
    from tests.emu.emu_stepper import emu_factory
    sf = F.stepper
    done = torch.nonzero(sf.buf["done"]).flatten().tolist()
    assert done, "a replica finished in the last step"
    k = len(done)
    emu = _make(name, kw, k, emu_factory, [1 + i for i in range(k)], auto_reset=True, final_obs=True, obs_dtype=obs_dtype)
    emu.reset()
    se = emu.stepper
    se.buf["episode_final"][...] = sf.buf["episode_final"][done].cpu().numpy()
    se.buf["done"][...] = 1
    se.observe_final()
    for key in OBS:
        if key not in se.buf or not se.buf[key].size:
            continue
        a, b = sf.buf["final_" + key][done], se.buf["final_" + key]
        if key in BF16_KEYS and obs_dtype == "bfloat16":
            a32, b32 = a.float().cpu().numpy(), (b.astype(np.uint32) << 16).view(np.float32)
        else:
            a32, b32 = a.cpu().numpy(), b
        if key in ("obs_agent_flat", "obs_planner_flat", "obs_planner_agents"):   # float32 sums may differ in the last bit
            tol = 1e-2 if obs_dtype == "bfloat16" else 1e-6
            assert np.allclose(a32, b32, rtol=tol, atol=1e-6), key
        else:
            assert np.array_equal(a32, b32), key


@pytest.mark.gpu
@pytest.mark.parametrize("obs_dtype", ["float32", "bfloat16"])
@pytest.mark.parametrize("cfg,E", [("c1_tutorial", 8192), ("c3_paper_tax", 8192), ("c5_full", 2048)], ids=["c2", "c3", "c5"])
def test_cuda_full_size_final_obs_equal_the_no_auto_reset_twin(cfg, E, obs_dtype):
    F, _, name, kw = _gpu_twins(cfg, E, obs_dtype)
    _check_against_emulation(F, name, kw, obs_dtype)


@pytest.mark.gpu
@pytest.mark.parametrize("knob,value,cfg", [("AIE_MW", "4", "c3_short_period"), ("AIE_MW", "1", "c5_small"),
                                            ("AIE_SPLIT", "1", "c5_small"), ("AIE_SPLIT", "0", "c5_small"),
                                            ("AIE_STEP_WPB", "2", "c3_short_period"), ("AIE_STEP_WPB", "1", "c1_tutorial")])
def test_cuda_final_obs_under_launch_knobs(knob, value, cfg, monkeypatch):
    """Every launch shape gives the default launch's final rows (and those equal the no-auto-reset twin's)."""
    default, _, _, _ = _gpu_twins(cfg, 37, "float32", knob_cfg=True)
    monkeypatch.setenv(knob, value)
    knobbed, _, name, kw = _gpu_twins(cfg, 37, "float32", knob_cfg=True)
    _check_against_emulation(knobbed, name, kw, "float32")
    for k in OBS:
        if "final_" + k in default.stepper.buf:
            assert torch.equal(default.stepper.buf["final_" + k], knobbed.stepper.buf["final_" + k]), k
