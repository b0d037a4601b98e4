"""bfloat16 observations and masks (`make_env_instance(..., obs_dtype=torch.bfloat16)`).

Contract: the eight float observation / mask tensors are bfloat16 with unchanged shapes, each element the
round-to-nearest-even bfloat16 of the float32 a default env writes for the same state (what `t.to(torch.bfloat16)` gives,
bit for bit); every other buffer (index planes, reward, done, state, state0, episode_final, events, actions drawn by the
fused policy and by the sampler) and every numpy stream is byte-identical to a float32 twin with the same seeds and
actions.  The CPU tests run twins through the host emulation of the device source (tests/emu), the `-m gpu` tests through
the CUDA kernels.
"""
import ctypes as C
import os
import subprocess
import textwrap

import numpy as np
import pytest
import torch

from ai_economist_b200 import _abi, foundation
from ai_economist_b200.stepper import bf16_bits_to_float32
from oracle import configs
from tests import batch_utils as bu

BF16_KEYS = ("obs_agent_map", "obs_agent_flat", "mask_agent", "obs_planner_map", "obs_planner_flat",
             "obs_planner_agents", "mask_planner", "obs_time")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

ONE_STEP_KW = dict(components=[("SimpleLabor", dict(mask_first_step=True, payment_max_skill_multiplier=3)),
                               ("PeriodicBracketTax", dict(bracket_spacing="us-federal", period=2, tax_model="model_wrapper",
                                                           rate_disc=0.05))],
                   n_agents=6, world_size=[1, 1], episode_length=3, planner_reward_type="coin_eq_times_productivity",
                   agent_reward_type="isoelastic_coin_minus_labor", labor_cost=0.02)


def _cfg(cfg, **over):
    if cfg == "one_step":
        return "one-step-economy", dict(ONE_STEP_KW, **over)
    kw = dict(configs.CONFIGS[cfg])
    name = kw.pop("scenario_name")
    kw["components"] = [tuple(c) for c in kw["components"]]
    kw.update(over)
    return name, kw


def _bits16(buf):
    """Raw bits of a bfloat16 buffer (torch.bfloat16 on CUDA, uint16 on numpy backends)."""
    if isinstance(buf, np.ndarray):
        return np.ascontiguousarray(buf).view(np.uint16)
    return buf.contiguous().view(torch.int16).cpu().numpy().view(np.uint16)


def _bytes(buf):
    if isinstance(buf, np.ndarray):
        return np.ascontiguousarray(buf).view(np.uint8).reshape(-1)
    return buf.contiguous().cpu().numpy().view(np.uint8).reshape(-1)


def rne_bits(a):
    """torch's float32 -> bfloat16 conversion, as raw bits."""
    t = torch.from_numpy(np.ascontiguousarray(a, np.float32)).to(torch.bfloat16)
    return t.view(torch.int16).numpy().view(np.uint16)


def check_twins(f32, b16, label):
    sf, sb = f32.stepper, b16.stepper
    assert set(sf.buf) == set(sb.buf)
    for k in sf.buf:
        if k in BF16_KEYS:
            want = rne_bits(sf.to_numpy(sf.buf[k]))
            got = _bits16(sb.buf[k])
            assert tuple(sb.buf[k].shape) == tuple(sf.buf[k].shape), "%s: shape of %s" % (label, k)
            bad = np.argwhere(want.reshape(-1) != got.reshape(-1))
            assert not len(bad), "%s: %s differs from float32 -> bfloat16 at %s" % (label, k, bad[:3].ravel().tolist())
        else:
            assert np.array_equal(_bytes(sf.buf[k]), _bytes(sb.buf[k])), "%s: %s not byte-identical" % (label, k)


def _make(name, kw, E, factory, auto_reset, obs_dtype, seeds):
    extra = dict(stepper_factory=factory) if factory is not None else dict(device="cuda:0")
    return foundation.make_env_instance(name, n_envs=E, auto_reset=auto_reset, seeds=seeds, obs_dtype=obs_dtype,
                                        **extra, **kw)


def run_twins(name, kw, E, steps, auto_reset, policy, factory=None, seed0=300):
    seeds = [seed0 + 11 * e for e in range(E)]
    f32 = _make(name, kw, E, factory, auto_reset, None, seeds)
    b16 = _make(name, kw, E, factory, auto_reset, torch.bfloat16, seeds)
    assert b16.spec["obs_dtype"] == "bfloat16" and f32.spec["obs_dtype"] == "float32"
    for env in (f32, b16):
        env.reset()
    check_twins(f32, b16, "reset")
    sp = f32.spec
    seg_a, seg_p = bu.segments(sp, "a"), bu.segments(sp, "p")
    rng = np.random.RandomState(5)
    if policy == "fused":
        for env in (f32, b16):
            env.stepper.set_fused_policy(77)
        check_twins(f32, b16, "fused policy armed")
    T = f32.episode_length
    for t in range(1, steps + 1):
        acts = None   # "fused" / "sampler": the actions already in the action buffers
        if policy == "sampler":
            for env in (f32, b16):
                env.stepper.sample_random_actions(seed=t)
            check_twins(f32, b16, "sampler t=%d" % t)
        elif policy == "host":
            st = f32.stepper
            aa = bu.sample_from_masks(st.to_numpy(st.buf["mask_agent"]), seg_a, rng)
            ap = bu.sample_from_masks(st.to_numpy(st.buf["mask_planner"]), seg_p, rng) if seg_p else None
            acts = (aa, ap)
        for env in (f32, b16):
            env.step(env.action_buffers if acts is None else acts)
        check_twins(f32, b16, "t=%d" % t)
        if not auto_reset and t % T == 0:
            for env in (f32, b16):
                env.reset()
            check_twins(f32, b16, "reset after t=%d" % t)
    for e in range(E):   # the host-side numpy streams
        a, b = f32.stream_state(e), b16.stream_state(e)
        assert np.array_equal(a[1], b[1]) and a[2:] == b[2:], "stream of replica %d" % e
    return f32, b16


# ---- CPU: host emulation twins ------------------------------------------------------------------------------------
EMU_CASES = [
    ("c1_tutorial", {}, "host"),                                   # reset_mode 0: host reset + snapshot auto-reset
    ("c1_tutorial", dict(planner_gets_spatial_info=False), "sampler"),
    ("c1_tutorial", dict(device_reset="snapshot"), "fused"),
    ("c3_short_period", {}, "fused"),
    ("c3_reset", {}, "host"),                                      # device reset (reset_mode 1)
    ("full_obs_tax", {}, "host"),
    ("tax_single_planner", {}, "sampler"),
    ("us_federal_annealed_reset", {}, "fused"),
    ("saez_reset", {}, "host"),                                    # Saez hybrid: host estimator, re-observe
    ("multi_zone", {}, "host"),
    ("c5_small", {}, "fused"),
    ("one_step", {}, "sampler"),
    ("c1_tutorial", dict(flatten_observations=False, flatten_masks=False), "host"),
    ("c1_tutorial", dict(collate_agent_step_and_reset_data=True), "fused"),
]


@pytest.mark.parametrize("auto_reset", [True, False], ids=["auto_reset", "explicit_reset"])
@pytest.mark.parametrize("cfg,over,policy", EMU_CASES,
                         ids=["%s-%s-%s" % (c, "_".join(sorted(o)) or "plain", p) for c, o, p in EMU_CASES])
def test_emulated_bf16_twin_matches_float32(cfg, over, policy, auto_reset):
    from tests.emu.emu_stepper import emu_factory
    over = dict(over)
    if cfg != "one_step":
        over.setdefault("episode_length", 6)
    name, kw = _cfg(cfg, **over)
    E = 2 if cfg == "c5_small" else 3
    T = kw["episode_length"]
    f32, b16 = run_twins(name, kw, E, 2 * T + 1, auto_reset, policy, factory=emu_factory)
    if not kw.get("flatten_observations", True) or kw.get("collate_agent_step_and_reset_data"):
        # the named-field / collated views are slices of the bfloat16 buffers
        assert b16.obs["p"]["time"].dtype == np.uint16
    # host copies are float32, equal to the float32 twin's rounded values
    for e in range(E):
        of, ob = f32.stepper.read_obs(e), b16.stepper.read_obs(e)
        for k in ("a_flat", "a_mask", "p_flat", "p_mask", "time"):
            assert ob[k].dtype == np.float32
            assert np.array_equal(ob[k], bf16_bits_to_float32(rne_bits(of[k])))


@pytest.mark.parametrize("nt", [32, 128])
@pytest.mark.parametrize("cfg", ["c3_short_period", "full_obs_tax", "c5_small"])
def test_emulated_bf16_thread_walks(cfg, nt, monkeypatch):
    """The phases walked with the device's thread counts: run heads and tails move with the element size."""
    from tests.emu.emu_stepper import emu_factory
    monkeypatch.setenv("AIE_EMU_NT", str(nt))
    name, kw = _cfg(cfg, episode_length=4)
    run_twins(name, kw, 2, 9, True, "fused", factory=emu_factory)


def test_reference_api_and_wrappers_hand_out_float32():
    from ai_economist_b200.adapters import MultiAgentDictEnv, ReferenceApiEnv, WarpDriveStyleEnvWrapper
    from tests.emu.emu_stepper import emu_factory
    name, kw = _cfg("c1_tutorial", episode_length=6)
    f32 = _make(name, kw, 2, emu_factory, True, None, [3, 4])
    b16 = _make(name, kw, 2, emu_factory, True, "bfloat16", [3, 4])
    of, ob = ReferenceApiEnv(f32, 1).reset(), ReferenceApiEnv(b16, 1).reset()
    for k in ("flat", "action_mask", "world-map"):
        assert ob["0"][k].dtype == np.float32
        assert np.array_equal(ob["0"][k], bf16_bits_to_float32(rne_bits(of["0"][k])))
    assert MultiAgentDictEnv(b16, 0).observation_space["flat"].dtype == np.float32
    w = WarpDriveStyleEnvWrapper(b16)
    assert b16.observation_space["0"]["world-map"].dtype == np.float32
    assert w.tensor("observations_a_flat") is b16.stepper.buf["obs_agent_flat"]


# ---- CPU: the host build's rounding helper --------------------------------------------------------------------------
_RNE_SRC = textwrap.dedent("""
    #define AIE_EMU 1
    #include <string.h>
    #include "ai_economist_b200/csrc/aie_core.cuh"
    extern "C" void rne(const float *x, unsigned short *out, long n) {
        for (long i = 0; i < n; i++) out[i] = (unsigned short)aie::bf16_rn(x[i]);
    }
    extern "C" void rne2(const float *x, unsigned *out, long n) {
        for (long i = 0; i < n; i++) out[i] = aie::bf16x2_rn(x[2 * i], x[2 * i + 1]);
    }
""")


def test_host_rounding_equals_torch(tmp_path):
    src, lib = tmp_path / "rne.cpp", tmp_path / "librne.so"
    src.write_text(_RNE_SRC)
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-I", ROOT, "-o", str(lib), str(src)])
    L = C.CDLL(str(lib))
    rng = np.random.RandomState(0)
    u = [np.arange(0, 1 << 20, dtype=np.uint32) << 12,                       # a sweep of exponents / upper mantissas
         rng.randint(0, 1 << 32, size=1 << 20, dtype=np.uint64).astype(np.uint32),   # random patterns
         (np.arange(1 << 16, dtype=np.uint32) << 16) | 0x8000,               # exact ties (round to even both ways)
         (np.arange(1 << 16, dtype=np.uint32) << 16) | 0x7FFF, (np.arange(1 << 16, dtype=np.uint32) << 16) | 0x8001,
         np.arange(0, 1 << 16, dtype=np.uint32) * 61,                        # subnormals
         np.array([0x7F7F7FFF, 0x7F7F8000, 0x7F7FFFFF, 0xFF7F8000, 0x7F7F0000, 0x7F800000, 0xFF800000], np.uint32),
         np.float32([0.0, -0.0, 1.0, -1.0, 0.5, 3.0, 1e-3]).view(np.uint32)]
    bits = np.concatenate(u)
    bits = bits[(bits & 0x7FFFFFFF) <= 0x7F800000]   # NaN payloads aside
    x = np.ascontiguousarray(bits.view(np.float32))
    out = np.zeros(x.size, np.uint16)
    L.rne(x.ctypes.data_as(C.c_void_p), out.ctypes.data_as(C.c_void_p), C.c_long(x.size))
    want = rne_bits(x)
    assert np.array_equal(out, want), x[out != want][:5]
    n2 = x.size // 2
    out2 = np.zeros(n2, np.uint32)
    L.rne2(x.ctypes.data_as(C.c_void_p), out2.ctypes.data_as(C.c_void_p), C.c_long(n2))
    assert np.array_equal(out2.view(np.uint16), want[:2 * n2])


# ---- CPU: C-ABI -------------------------------------------------------------------------------------------------
def test_abi_rejects_unknown_obs_dtype_and_host_steps():
    from tests.emu.emu_stepper import emu_factory, emu_lib
    L = emu_lib()
    name, kw = _cfg("c1_tutorial", episode_length=6)
    env = _make(name, kw, 2, emu_factory, True, "bfloat16", [1, 2])
    cfg = _abi.config_from_spec(env.spec)
    assert cfg.obs_dtype == _abi.OBS_BF16
    cfg.obs_dtype = 2
    h = C.c_void_p()
    assert L.aie_create(C.byref(cfg), 2, 0, C.byref(h)) == -1   # AIE_EINVAL
    assert b"obs_dtype" in L.aie_last_error()
    env.reset()
    st = env.stepper
    acts = np.zeros(st.buf["actions_agent"].shape, np.int32)
    for compact in (False, True):
        with pytest.raises(_abi.AieError, match="float32 observations only"):
            st.step_host(acts.ctypes.data_as(C.c_void_p), None, {}, compact=compact)
    # the algorithmic byte count uses the element size
    f32 = _make(name, kw, 2, emu_factory, True, None, [1, 2])
    d32, d16 = f32.stepper.dims, st.dims
    A = d32.n_agents
    n_float = A * (d32.agent_map_elems + d32.flat_agent + d32.mask_agent + d32.flat_planner_agent) + \
        d32.flat_planner + d32.mask_planner + 1 + d32.n_map_channels * d32.height * d32.width
    assert d32.algorithmic_bytes_per_env_step - d16.algorithmic_bytes_per_env_step == 2 * n_float


def test_bad_obs_dtype_and_covid_rejects_bfloat16():
    from ai_economist_b200 import workloads as wl
    name, kw = _cfg("c1_tutorial")
    with pytest.raises(ValueError):
        foundation.make_env_instance(name, n_envs=1, stepper_factory=lambda *a, **k: None, obs_dtype=torch.float16, **kw)
    cfg = wl.covid_reference_config()
    cname = cfg.pop("scenario_name")
    with pytest.raises(NotImplementedError):
        foundation.make_env_instance(cname, n_envs=1, stepper_factory=lambda *a, **k: None, obs_dtype=torch.bfloat16, **cfg)


# ---- CPU: footprint of the new kernels ---------------------------------------------------------------------------
C2_BF16 = "_ZN3aie20aie_step_bf16_kernelILi4ELb0ELi7EEEvNS_6DevCfgENS_7DevBufsEii"
C3_BF16 = "_ZN3aie20aie_step_bf16_kernelILi3ELb0ELi15EEEvNS_6DevCfgENS_7DevBufsEii"


@pytest.mark.parametrize("kernel,ref,regs", [(C2_BF16, "C2_KERNEL", 64), (C3_BF16, "C3_KERNEL", 80)], ids=["c2", "c3"])
def test_bf16_step_kernels_within_float32_budgets(kernel, ref, regs):
    """The bfloat16 step kernels stay inside the budgets of their float32 twins."""
    from tests import test_step_kernel_footprint as fp
    lib = fp.build_library()
    import tempfile
    with tempfile.TemporaryDirectory() as tmp:
        subprocess.run([fp._tool("cuobjdump"), "-xelf", "all", lib], cwd=tmp, check=True, capture_output=True)
        dis = "".join(subprocess.run([fp._tool("nvdisasm"), "-c", os.path.join(tmp, f)], check=True, capture_output=True,
                                     text=True).stdout for f in os.listdir(tmp) if f.endswith(".cubin"))
    r = getattr(fp, ref)
    hot, local, total, slots = fp.section_stats(dis, kernel)
    assert hot <= fp.HOT_INSTR_BUDGET[r] and local <= fp.HOT_LOCAL_BUDGET[r] and slots <= fp.HOT_SLOT_BUDGET[r], \
        (hot, local, slots)
    assert 16 * total <= fp.SECTION_BYTES_BUDGET[r], total
    import re
    out = subprocess.run([fp._tool("cuobjdump"), "-res-usage", lib], check=True, capture_output=True, text=True).stdout
    m = re.search(r"Function " + re.escape(kernel) + r":\s*\n\s*REG:(\d+) STACK:(\d+)", out)
    assert m and int(m.group(1)) <= regs and int(m.group(2)) <= fp.STACK_BUDGET[r], m and m.groups()


# ---- GPU: CUDA twins ------------------------------------------------------------------------------------------------
def _gpu_check(f32, b16, label):
    """Every element on the device: the bfloat16 tensors against the float32 twin's conversion, the rest by bytes."""
    sf, sb = f32.stepper.buf, b16.stepper.buf
    for k in sf:
        a, b = sf[k], sb[k]
        if k in BF16_KEYS:
            ok = torch.equal(a.to(torch.bfloat16).view(torch.int16), b.view(torch.int16))
        else:
            ok = torch.equal(a.view(torch.uint8) if a.dim() else a, b.view(torch.uint8) if b.dim() else b)
        assert ok, "%s: %s" % (label, k)


def _gpu_twins(cfg_name, table, E, episodes, knobs=None, over=None):
    name, kw = (bu.product_kwargs(cfg_name) if table is None else _cfg(cfg_name))
    kw = dict(kw, **(over or {}))
    if cfg_name == "c5_full":
        kw["device_reset"] = "snapshot"
    seeds = [1000 + e for e in range(E)]
    f32 = foundation.make_env_instance(name, n_envs=E, device="cuda:0", seeds=seeds, auto_reset=True, **kw)
    b16 = foundation.make_env_instance(name, n_envs=E, device="cuda:0", seeds=seeds, auto_reset=True,
                                       obs_dtype=torch.bfloat16, **kw)
    T = f32.episode_length
    for env in (f32, b16):
        env.reset()
        env.stepper.state_view("t").copy_((torch.arange(E, device="cuda:0", dtype=torch.int64) * T // E).to(torch.int32))
        env.stepper.set_fused_policy(4321)
    _gpu_check(f32, b16, "reset")
    for t in range(episodes * T):
        f32.stepper.step()
        b16.stepper.step()
        _gpu_check(f32, b16, "t=%d" % t)
    torch.cuda.synchronize()
    return f32, b16


@pytest.mark.gpu
@pytest.mark.parametrize("cfg,E", [("c1_tutorial", 8192), ("c3_paper_tax", 8192), ("c5_full", 2048)], ids=["c2", "c3", "c5"])
def test_cuda_bf16_twins_two_staggered_episodes(cfg, E):
    _gpu_twins(cfg, None, E, 2)


@pytest.mark.gpu
@pytest.mark.parametrize("knob,value,cfg", [("AIE_STEP_MINB", "3", "c3_short_period"), ("AIE_STEP_MINB", "4", "c3_short_period"),
                                            ("AIE_STEP_WPB", "2", "c3_short_period"), ("AIE_PHASE_SYNC", "1", "c3_short_period"),
                                            ("AIE_MW", "4", "c3_short_period"), ("AIE_MW", "1", "c5_small"),
                                            ("AIE_SPLIT", "1", "c5_small"), ("AIE_SPLIT", "0", "c5_small")])
def test_cuda_bf16_twins_under_launch_knobs(knob, value, cfg, monkeypatch):
    monkeypatch.setenv(knob, value)
    f32, b16 = _gpu_twins(cfg, configs.CONFIGS, 37, 2, over=dict(episode_length=9))
    for env in (f32, b16):   # the stand-alone observation pass and the sampler
        env.stepper.set_fused_policy(0)
        env.stepper.observe()
        env.stepper.sample_random_actions(seed=9)
    _gpu_check(f32, b16, "observe + sampler")


@pytest.mark.gpu
@pytest.mark.parametrize("cfg", ["c3_reset", "full_obs_tax", "tax_single_planner"])
def test_cuda_bf16_equals_emulation(cfg):
    from tests.emu.emu_stepper import emu_factory
    name, kw = _cfg(cfg, episode_length=5)
    seeds = [70 + e for e in range(6)]
    cuda = _make(name, kw, 6, None, True, torch.bfloat16, seeds)
    emu = _make(name, kw, 6, emu_factory, True, torch.bfloat16, seeds)
    seg_a, seg_p = bu.segments(cuda.spec, "a"), bu.segments(cuda.spec, "p")
    rng = np.random.RandomState(3)
    for env in (cuda, emu):
        env.reset()
    for t in range(12):
        se = emu.stepper
        aa = bu.sample_from_masks(se.obs_to_numpy("mask_agent"), seg_a, rng)
        ap = bu.sample_from_masks(se.obs_to_numpy("mask_planner"), seg_p, rng) if seg_p else None
        cuda.step((aa, ap))
        emu.step((aa, ap))
        torch.cuda.synchronize()
        for k in BF16_KEYS + ("obs_agent_idx", "done"):
            if k in se.buf and int(np.prod(se.buf[k].shape)):
                a = _bits16(cuda.stepper.buf[k]) if k in BF16_KEYS else cuda.stepper.to_numpy(cuda.stepper.buf[k])
                b = _bits16(se.buf[k]) if k in BF16_KEYS else se.to_numpy(se.buf[k])
                if k in ("obs_agent_flat", "obs_planner_flat", "obs_planner_agents"):   # float32 sums may differ in the last bit
                    assert np.allclose(bf16_bits_to_float32(a), bf16_bits_to_float32(b), rtol=1e-2, atol=1e-6), "t=%d %s" % (t, k)
                else:
                    assert np.array_equal(a, b), "t=%d %s" % (t, k)
