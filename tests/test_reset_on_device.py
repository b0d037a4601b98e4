"""Explicit env.reset() on the device (aie_reset_envs) for configs whose auto-reset is reference-exact (reset_mode == 1).

Twin envs with identical seeds: one resets through env.reset() (one launch re-draws every replica on the device), the
other through the host path it replaces - the scenario's host_reset per replica, packed and uploaded by
load_host_state, with the bookkeeping reset() did before (streams synced from the device, completions, the carried
energy warm-up integrator, the Saez state).  After every reset the records (state and state0), every observation and
mask tensor, reward, done and every replica's numpy stream must be byte-identical.
"""
import os
import sys

import numpy as np
import pytest

from ai_economist_b200 import _abi, foundation
from ai_economist_b200 import workloads as wl
from oracle.configs import CONFIGS

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools"))


def _kwargs(cfg, **over):
    kw = dict(cfg)
    kw.update(over)
    name = kw.pop("scenario_name")
    kw["components"] = [tuple(c) for c in kw["components"]]
    seed = kw.pop("seed", None)
    return name, kw, seed


def _make(cfg, E, factory, auto_reset=False, dense=None, **over):
    name, kw, ctor_seed = _kwargs(cfg, **over)
    extra = dict(stepper_factory=factory) if factory else dict(device="cuda:0")
    if ctor_seed is not None:   # a constructor seed (split_layout's skill tables): distinct per replica
        kw["seeds"] = [ctor_seed + 7 * e for e in range(E)]
    return foundation.make_env_instance(name, n_envs=E, auto_reset=auto_reset, dense_log_frequency=dense, **kw, **extra)


def _host_reset(env, seed_state=None):
    """What reset() ran before the device path: the per-replica host reset, packed and uploaded."""
    st = env.stepper
    if env._loaded and env._rs is not None:
        env._completions = env.completions()
        env._sync_streams_from_device()
    if seed_state is not None:
        env._rs[0].set_state(env._np_state(seed_state))
    saez_n = env._saez.before_host_reset() if env._saez is not None else None
    warm = st.to_numpy(st.state_view("auto_warmup")).copy() if env._loaded else None
    env.load_host_state(env.host_reset_arrays())
    if warm is not None and warm.any():
        v = st.state_view("auto_warmup")
        if isinstance(v, np.ndarray):
            v[...] = warm
        else:
            import torch
            v.copy_(torch.as_tensor(warm, device=v.device, dtype=v.dtype))
    if env._saez is not None:
        env._saez.after_host_reset(saez_n)


def _compare(dev, host, label):
    sd, sh = dev.stepper, host.stepper
    assert sorted(sd.buf) == sorted(sh.buf)
    for k in sd.buf:
        if k.startswith("actions_"):
            continue
        a, b = sd.to_numpy(sd.buf[k]), sh.to_numpy(sh.buf[k])
        if not np.array_equal(a.view(np.uint8), b.view(np.uint8)):
            bad = np.nonzero((a.view(np.uint8) != b.view(np.uint8)).reshape(a.shape[0], -1).any(axis=1))[0]
            raise AssertionError("%s: %s differs in replicas %s" % (label, k, bad.tolist()))
    for e in range(dev.n_envs):
        s1, s2 = dev.stream_state(e), host.stream_state(e)
        assert s1[0] == s2[0] and np.array_equal(s1[1], s2[1]) and s1[2:] == s2[2:], "%s: stream of replica %d" % (label, e)


def _random_steps(dev, host, n, rng):
    """n steps of the same mask-respecting random actions on both envs."""
    seg_a, seg_p = wl.mask_segments(dev.spec, "a"), wl.mask_segments(dev.spec, "p")
    sd = dev.stepper
    for _ in range(n):
        acts = wl.sample_from_masks(sd.to_numpy(sd.buf["mask_agent"]), seg_a, rng)
        pa = wl.sample_from_masks(sd.to_numpy(sd.buf["mask_planner"]), seg_p, rng) if seg_p else None
        dev.step((acts, pa) if pa is not None else acts)
        host.step((acts, pa) if pa is not None else acts)


def _twin(cfg, factory, E=5, seeds=None, rounds=None, auto_reset=False, **over):
    """First reset, then further explicit resets after random steps: rounds lists the steps before each of them (the
    default ends one episode exactly, waiting for its reset, and leaves the next unfinished)."""
    dev = _make(cfg, E, factory, auto_reset=auto_reset, **over)
    host = _make(cfg, E, factory, auto_reset=auto_reset, **over)
    assert dev.spec["reset_mode"] == 1
    seeds = seeds or [1000 + 37 * e for e in range(E)]
    dev.seed(seeds)
    host.seed(seeds)
    dev.reset()
    _host_reset(host)
    _compare(dev, host, "first reset")
    T = dev.episode_length
    rng = np.random.RandomState(sum(seeds))
    for r, n in enumerate(rounds if rounds is not None else [T, min(3, T - 1)]):
        _random_steps(dev, host, n, rng)
        dev.reset()
        _host_reset(host)
        _compare(dev, host, "reset %d after %d steps" % (r + 2, n))
    return dev, host


# ---------------------------------------------------------------------------------------------- CPU, emulated device
def _emu():
    from tests.emu.emu_stepper import emu_factory
    return emu_factory


def _uniform(**kw):
    base = dict(CONFIGS["quadrant"])
    base.update(scenario_name="uniform/simple_wood_and_stone", checker_source_blocks=False)
    base.update(kw)
    return base


def _short(cfg, T=10):
    return dict(cfg, episode_length=T)


NAMED = {
    "c1": _short(CONFIGS["c1_reset"]),
    "c3_tax": _short(CONFIGS["c3_reset"]),
    "us_federal_annealed": _short(CONFIGS["us_federal_annealed_reset"]),
    "split_layout": _short(CONFIGS["split_layout"]),
    "lognormal": _short(CONFIGS["lognormal_reset"]),
    "uniform_halfwidth": _short(CONFIGS["uniform_halfwidth"], 8),
    "checkered_uniform": _uniform(checker_source_blocks=True, episode_length=8),
    "quadrant": _short(CONFIGS["quadrant"], 8),
    "multi_zone": _short(CONFIGS["multi_zone"], 8),
    "saez": _short(CONFIGS["saez_reset"], 12),
    "saez_annealed": _short(CONFIGS["saez_annealed_reset"], 12),
    "energy_auto": dict(_short(CONFIGS["c3_reset"]), energy_warmup_method="auto", energy_warmup_constant=3),
    "full_observability": _short(CONFIGS["full_obs_tax"]),
    "multi_action_agents": dict(_short(CONFIGS["c1_reset"]), multi_action_mode_agents=True),
    "single_action_planner": _short(CONFIGS["tax_single_planner"]),
}


@pytest.mark.parametrize("which", sorted(NAMED))
def test_emulated_device_reset_matches_host_reset(which):
    _twin(NAMED[which], _emu())


def test_emulated_device_reset_fixed_four_across_auto_resets():
    """fixed_four (c1) with auto-reset on: explicit resets between auto-reset episodes, episode_final untouched."""
    _twin(_short(CONFIGS["c1_reset"], 6), _emu(), auto_reset=True, rounds=[13, 4])


def test_emulated_device_reset_energy_warmup_is_carried():
    dev, host = _twin(NAMED["energy_auto"], _emu(), rounds=[10, 10])
    assert dev.stepper.to_numpy(dev.stepper.state_view("auto_warmup")).any(), "the warm-up integrator never moved"


def test_emulated_device_reset_split_record(monkeypatch):
    monkeypatch.setenv("AIE_SPLIT", "1")   # c5-small with its price history and order slots in global memory
    dev, _ = _twin(_short(CONFIGS["c5_small"], 5), _emu(), E=2, rounds=[5])
    assert dev.stepper.dims.state_bytes > 24 * 1024


def test_emulated_device_reset_large_record():
    """A record of more than 100 KB (deep order book, many agents): split on its own, four warps per env."""
    cfg = _uniform(n_agents=64, world_size=[24, 24], episode_length=4,
                   components=[("Build", dict(skill_dist="pareto", payment_max_skill_multiplier=3)),
                               ("ContinuousDoubleAuction", dict(max_num_orders=100, max_bid_ask=31)),
                               ("Gather", dict(skill_dist="pareto"))])
    dev, _ = _twin(cfg, _emu(), E=2, rounds=[4])
    assert dev.stepper.dims.state_bytes > 100 * 1024


def test_emulated_device_reset_mw4_record():
    dev, _ = _twin(_short(CONFIGS["c5_small"], 5), _emu(), E=2, rounds=[5])
    assert dev.stepper.dims.state_bytes > 24 * 1024


def _fuzz_cases(kind, n):
    import fuzz_device_reset_vs_reference as fz
    gen = {"layout": fz.random_config, "dynamic": fz.random_dynamic_config, "saez": fz.random_saez_config}[kind]
    rng = np.random.RandomState({"layout": 11, "dynamic": 12, "saez": 13}[kind])
    out = []
    for _ in range(n):
        cfg = gen(rng)
        cfg["episode_length"] = min(cfg["episode_length"], 12)
        out.append(cfg)
    return out


@pytest.mark.parametrize("kind", ["layout", "dynamic", "saez"])
@pytest.mark.parametrize("i", range(20))
def test_emulated_device_reset_fuzzed_configs(kind, i):
    cfg = _fuzz_cases(kind, 20)[i]
    _twin(cfg, _emu(), E=3, rounds=[cfg["episode_length"], 2])


def test_emulated_reset_seed_state_moves_one_stream():
    """The reference API's reset(seed_state): replica 0 restarts from the given stream, the others continue theirs."""
    cfg = NAMED["quadrant"]
    ss = np.random.RandomState(4242).get_state()
    dev, host = _make(cfg, 3, _emu()), _make(cfg, 3, _emu())
    for env in (dev, host):
        env.seed([9, 10, 11])
    dev.reset(seed_state=ss)   # the first reset takes it too
    _host_reset(host, seed_state=ss)
    _compare(dev, host, "first reset(seed_state)")
    _random_steps(dev, host, 5, np.random.RandomState(3))
    ss = np.random.RandomState(4243).get_state()
    dev.reset(seed_state=ss)
    _host_reset(host, seed_state=ss)
    _compare(dev, host, "reset(seed_state)")


def test_emulated_second_reset_does_no_host_work(monkeypatch):
    """auto_reset off, no Saez, no dense log: a second env.reset() runs no host reset and reads nothing of size n_envs
    back; it is two launches (the reset kernel and the observation pass)."""
    E = 5
    dev = _make(NAMED["multi_zone"], E, _emu())
    dev.seed(77)
    dev.reset()
    dev.step()
    st = dev.stepper

    def no_host_reset(*a, **k):
        raise AssertionError("host_reset called")
    monkeypatch.setattr(dev.scenario, "host_reset", no_host_reset)
    real = st.to_numpy

    def small_reads_only(buf):
        a = real(buf)
        assert a.ndim == 0 or a.shape[0] < E, "a read of size n_envs: %s" % (a.shape,)
        return a
    monkeypatch.setattr(st, "to_numpy", small_reads_only)
    n0 = st.launch_count()
    dev.reset()
    assert st.launch_count() - n0 == 2


def test_emulated_reset_envs_abi_errors():
    import ctypes as C
    from tests.emu.emu_stepper import emu_lib
    lib = emu_lib()
    dev = _make(NAMED["c1"], 2, _emu())
    h = dev.stepper._h
    assert lib.aie_reset_envs(None, None, None, 0, 1, None) == -1
    assert lib.aie_reset_envs(h, None, None, 0, 2, None) == -3          # nothing loaded, no template
    dev.seed(5)
    dev.reset()
    assert lib.aie_reset_envs(h, None, None, 0, 2, None) == 0
    for lo, n in [(-1, 1), (0, 0), (1, 2), (0, 3)]:
        assert lib.aie_reset_envs(h, None, None, lo, n, None) == -1, (lo, n)
    s = _abi.AieResetStreams()   # streams without arrays
    assert lib.aie_reset_envs(h, None, C.byref(s), 0, 2, None) == -1
    tmpl = _abi.AieHostState()
    tmpl.n = 2
    assert lib.aie_reset_envs(h, C.byref(tmpl), None, 0, 2, None) == -1
    snap = _make(CONFIGS["saez_reset"], 2, _emu(), device_reset="snapshot")   # reset_mode 0
    assert snap.spec["reset_mode"] == 0
    assert lib.aie_reset_envs(snap.stepper._h, None, None, 0, 2, None) == -1


# ---------------------------------------------------------------------------------------------- GPU (CUDA kernels)
# CUDA's exp / log / pow can differ from the host libm's in the last place: the float64 fields computed with them are
# compared to 1e-12 relative - the Pareto / lognormal skills, the cached second Gaussian variate of the polar method
# (gauss_state, where the config has one) and, against the emulation, whose finish_reset_env runs on the host, the
# utilities - and float32 outputs that show them to 1e-6; every other byte (maps, placements, streams, counters) exactly.
SKILL_FIELDS = ("build_payment", "build_skill", "bonus_gather_prob", "gauss_state")


def _compare_large(dev, other, label, libm_fields=SKILL_FIELDS):
    """Record / output bytes of every replica (the streams are inside the records); stream_state of a few replicas."""
    sd, so = dev.stepper, other.stepper
    skill = []
    for f in libm_fields:
        try:
            fd = sd.field(f)
        except _abi.AieError:   # no such section in this config (gauss_state)
            continue
        skill.append((fd.offset, fd.offset + 8 * int(np.prod([fd.shape[i] for i in range(fd.ndim)]))))
    for k in sd.buf:
        if k.startswith("actions_") or k not in so.buf:
            continue
        a, b = sd.to_numpy(sd.buf[k]), so.to_numpy(so.buf[k])
        if k in ("state", "state0", "episode_final"):
            for lo, hi in skill:
                x, y = a[:, lo:hi].copy().view(np.float64), b[:, lo:hi].copy().view(np.float64)
                assert np.allclose(x, y, rtol=1e-12, atol=0), "%s: %s skills" % (label, k)
                a[:, lo:hi] = b[:, lo:hi]
        elif a.dtype == np.float32 and not np.array_equal(a, b):
            assert np.allclose(a, b, rtol=1e-6, atol=0), "%s: %s" % (label, k)
            continue
        diff = (a.view(np.uint8) != b.view(np.uint8)).reshape(a.shape[0], -1).any(axis=1)
        assert not diff.any(), "%s: %s differs in replicas %s" % (label, k, np.nonzero(diff)[0][:10].tolist())
    for e in (0, dev.n_envs // 2, dev.n_envs - 1):
        s1, s2 = dev.stream_state(e), other.stream_state(e)
        assert np.array_equal(s1[1], s2[1]) and s1[2:4] == s2[2:4], "%s: stream of replica %d" % (label, e)
        assert np.isclose(s1[4], s2[4], rtol=1e-12, atol=0), "%s: cached Gaussian of replica %d" % (label, e)


def _gpu_twin(cfg_name, E, steps):
    from tests.batch_utils import product_kwargs
    name, kw = product_kwargs(cfg_name)
    cfg = dict(kw, scenario_name=name)
    dev, host = _make(cfg, E, None), _make(cfg, E, None)
    assert dev.spec["reset_mode"] == 1
    for env in (dev, host):
        env.seed(1000)
    dev.reset()
    _host_reset(host)
    _compare_large(dev, host, "first reset")
    _random_steps(dev, host, steps, np.random.RandomState(5))
    dev.reset()
    _host_reset(host)
    _compare_large(dev, host, "second reset after %d steps" % steps)


@pytest.mark.gpu
@pytest.mark.parametrize("cfg_name", ["c1_tutorial", "c3_paper_tax"])
def test_cuda_device_reset_matches_host_reset_full_size(cfg_name):
    """c2 (the c1 tutorial config at 8 192 replicas) and c3 at 8 192 replicas."""
    _gpu_twin(cfg_name, 8192, 3)


@pytest.mark.gpu
def test_cuda_device_reset_matches_host_reset_c5_size():
    """c5's record (64x64, 64 agents, four warps per env) with 128 replicas against the host path."""
    _gpu_twin("c5_full", 128, 3)


@pytest.mark.gpu
def test_cuda_device_reset_matches_emulation_c5_full():
    """All 2 048 c5 replicas: the CUDA reset kernel against the emulation's records for the same streams, for the first
    reset (template + uploaded streams) and a second one (state0 + the records' own streams)."""
    from tests.batch_utils import product_kwargs
    name, kw = product_kwargs("c5_full")
    cfg = dict(kw, scenario_name=name)
    E = 2048
    dev, emu = _make(cfg, E, None), _make(cfg, E, _emu())
    for env in (dev, emu):
        env.seed(2000)
    for label in ("first reset", "second reset"):
        dev.reset()
        emu.reset()
        _compare_large(dev, emu, label, libm_fields=SKILL_FIELDS + ("util_prev",))
