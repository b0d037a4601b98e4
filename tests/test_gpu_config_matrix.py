"""The CUDA reset, staging and compact-transfer paths on the configs the host emulation is held to.

The 1-lane host emulation (tests/emu) is held to the host paths and the oracle over a wide set of configs; the GPU runs
the warp-level code (32 lanes, bulk copies, ballots, __popc / __fns offsets, several envs per CTA) that the emulation
does not.  This module runs the cross product, reusing the emulation's harnesses:

A. env.reset() on the device (aie_reset_envs: the reset and finish-reset kernels) against the host reset, for every named
   config, the special records and the 60 fuzzed configs of tests/test_reset_on_device.py, plus dynamic layouts wider
   than a warp (W or H of 33 .. 63) - the lane-strided generator loops take more than one pass there.  Each batch leaves
   the last CTA of its launch shape (envs per CTA, read from the AIE_VERBOSE lines of aie_create) partial.
B. The four branches of the observation pass's staging plan (tests/test_staging_plan.py) on CUDA against the oracle,
   every replica, and across two auto-resets against the emulation's records.
C. aie_step_host_compact (tests/test_compact_transfer.py) on more layouts, on the emulation and on CUDA: the device
   branches of pack_bits / pack_sparse_u8, the uint16 open-order counts of c5, the work-item sizes and the overflow path.

Libm-derived values (the Pareto / lognormal skills, the cached Gaussian, utilities and rewards, and against the
emulation the coin a skill-dependent build payment went into) are held to 1e-12; every other byte of the records and
outputs must match.
"""
import re

import numpy as np
import pytest

from ai_economist_b200 import foundation
from oracle import configs
from oracle.configs import CONFIGS
from oracle.oracle import OracleBatch
from tests import batch_utils as bu
from tests import test_reset_on_device as rd
from tests.test_compact_transfer import _check
from tests.test_staging_plan import CASES as STAGING, placement


def _emu():
    from tests.emu.emu_stepper import emu_factory
    return emu_factory


def _created(monkeypatch, capfd, make, environ=()):
    """make() under AIE_VERBOSE (and the knobs in environ): (its result, aie_create's host line, the CUDA backend's
    launch-shape line or None for the emulation)."""
    for k, v in dict(environ).items():
        monkeypatch.setenv(k, v)
    monkeypatch.setenv("AIE_VERBOSE", "1")
    capfd.readouterr()
    out = make()
    err = capfd.readouterr().err.splitlines()
    monkeypatch.delenv("AIE_VERBOSE")
    host = [ln for ln in err if ln.startswith("[aie] A ")]
    backend = [ln for ln in err if ln.startswith("[aie] record ")]
    assert len(host) == 1 and len(backend) <= 1, err
    return out, host[0], backend[0] if backend else None


def _partial_batch(cfg, monkeypatch, capfd, environ=(), **over):
    """A batch size whose last CTA is partial in the launch shape this config gets on the device: two CTAs, the second
    one env short (envs per CTA from the backend's AIE_VERBOSE line; with mw > 1 warps per env a CTA holds one env)."""
    _, host, backend = _created(monkeypatch, capfd, lambda: rd._make(cfg, 1, None, **over), environ)
    assert backend, host
    wpb = int(re.search(r"(\d+) envs/CTA", backend).group(1))
    mw = int(re.search(r" mw (\d+),", host).group(1))
    assert wpb == 1 or mw == 1, (host, backend)
    E = 2 * wpb - 1 if wpb > 1 else 3
    assert wpb == 1 or E % wpb, E
    return E


def _gpu_twin(cfg, monkeypatch, capfd, environ=(), **kw):
    E = _partial_batch(cfg, monkeypatch, capfd, environ)   # the knobs in environ stay set for the twins
    return rd._twin(cfg, None, E=E, compare=rd._compare_large, **kw)


# ---------------------------------------------------------------------------------- A. device reset vs host reset
def _wide(fam, H, W, A, **kw):
    cfg = dict(scenario_name=fam + "/simple_wood_and_stone",
               components=[("Build", dict(skill_dist="pareto", payment_max_skill_multiplier=3)),
                           ("ContinuousDoubleAuction", dict(max_num_orders=5)),
                           ("Gather", dict(skill_dist="lognormal"))],
               n_agents=A, world_size=[H, W], episode_length=8, starting_agent_coin=10,
               multi_action_mode_agents=False, multi_action_mode_planner=True, flatten_observations=True,
               flatten_masks=True, starting_wood_coverage=0.1, starting_stone_coverage=0.08, wood_clumpiness=0.35,
               stone_clumpiness=0.5, gradient_steepness=4, checker_source_blocks=False, wood_regen_weight=0.05,
               stone_regen_weight=0.5)
    cfg.update(kw)
    return cfg


# dynamic layouts wider than a warp: HW / 32 is not an integer, rows straddle lanes, conv7_same reads across row ends
WIDE = {
    "uniform_33x45": _wide("uniform", 33, 45, 5),
    "quadrant_37x37_checkered": _wide("quadrant", 37, 37, 8, checker_source_blocks=True),
    "uniform_20x63_40_agents": _wide("uniform", 20, 63, 40),   # more agents than lanes: two passes of the agent loops
    "multi_zone_45x33": _wide("multi_zone", 45, 33, 6, num_partitions_row=3, num_partitions_col=3, num_wood_zones=2,
                              num_stone_zones=2, num_wood_and_stone_zones=1),
}


@pytest.mark.gpu
@pytest.mark.parametrize("which", sorted(rd.NAMED))
def test_cuda_device_reset_matches_host_reset_on_named_config(which, monkeypatch, capfd):
    _gpu_twin(rd.NAMED[which], monkeypatch, capfd)


@pytest.mark.gpu
@pytest.mark.parametrize("which", sorted(WIDE))
def test_cuda_device_reset_matches_host_reset_on_wide_dynamic_layout(which, monkeypatch, capfd):
    _gpu_twin(WIDE[which], monkeypatch, capfd)


@pytest.mark.gpu
def test_cuda_device_reset_fixed_four_across_auto_resets(monkeypatch, capfd):
    _gpu_twin(rd._short(CONFIGS["c1_reset"], 6), monkeypatch, capfd, auto_reset=True, rounds=[13, 4])


@pytest.mark.gpu
def test_cuda_device_reset_energy_warmup_is_carried(monkeypatch, capfd):
    dev, _ = _gpu_twin(rd.NAMED["energy_auto"], monkeypatch, capfd, rounds=[10, 10])
    assert dev.stepper.to_numpy(dev.stepper.state_view("auto_warmup")).any(), "the warm-up integrator never moved"


@pytest.mark.gpu
def test_cuda_device_reset_split_record(monkeypatch, capfd):
    dev, _ = _gpu_twin(rd._short(CONFIGS["c5_small"], 5), monkeypatch, capfd, {"AIE_SPLIT": "1"}, rounds=[5, 2])
    assert dev.stepper.dims.state_bytes > 24 * 1024


@pytest.mark.gpu
def test_cuda_device_reset_large_record(monkeypatch, capfd):
    cfg = rd._uniform(n_agents=64, world_size=[24, 24], episode_length=4,
                      components=[("Build", dict(skill_dist="pareto", payment_max_skill_multiplier=3)),
                                  ("ContinuousDoubleAuction", dict(max_num_orders=100, max_bid_ask=31)),
                                  ("Gather", dict(skill_dist="pareto"))])
    dev, _ = _gpu_twin(cfg, monkeypatch, capfd, rounds=[4, 2])
    assert dev.stepper.dims.state_bytes > 100 * 1024


@pytest.mark.gpu
def test_cuda_device_reset_mw4_record(monkeypatch, capfd):
    dev, _ = _gpu_twin(rd._short(CONFIGS["c5_small"], 5), monkeypatch, capfd, rounds=[5, 2])
    assert dev.stepper.dims.state_bytes > 24 * 1024


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["layout", "dynamic", "saez"])
@pytest.mark.parametrize("i", range(20))
def test_cuda_device_reset_fuzzed_configs(kind, i, monkeypatch, capfd):
    cfg = rd._fuzz_cases(kind, 20)[i]
    _gpu_twin(cfg, monkeypatch, capfd, rounds=[cfg["episode_length"], 2])


# ------------------------------------------------------------------------------ B. staging branches vs the oracle
E_STAGING = 37


def _staging_kwargs(branch, T=None):
    kw = dict(STAGING[branch][0])
    kw.pop("seed", None)
    if T is not None:
        kw["episode_length"] = T
    name = kw.pop("scenario_name")
    kw["components"] = [tuple(c) for c in kw["components"]]
    return name, kw


@pytest.mark.gpu
@pytest.mark.parametrize("branch", sorted(STAGING))
def test_cuda_staging_branch_matches_oracle(branch, monkeypatch, capfd):
    name, kw = _staging_kwargs(branch)
    env, line, _ = _created(monkeypatch, capfd, lambda: foundation.make_env_instance(
        name, n_envs=E_STAGING, device="cuda:0", auto_reset=False, seed=2024, **kw), STAGING[branch][1])
    got, mw = placement(line)
    assert branch in got, (branch, line)
    if branch == "split_record":
        assert mw == 4
    host = env.host_reset_arrays()
    env.load_host_state(host)   # the stand-alone observation pass
    orc = OracleBatch(env.spec, E_STAGING)
    for e in range(E_STAGING):
        orc.load_env(e, {k: v[e] for k, v in host.items()})
        bu.compare_env(orc, env.stepper, e, "reset", spatial=bool(env.spec["planner_gets_spatial_info"]))
    bu.run_pair(env, orc, 40, np.random.RandomState(31), check_every=10)


@pytest.mark.gpu
@pytest.mark.parametrize("branch", sorted(STAGING))
def test_cuda_staging_branch_across_auto_resets_equals_emulation(branch, monkeypatch, capfd):
    """Two episode ends inside the run (auto-reset in the step kernel, then the observation pass on the new records):
    the CUDA records and outputs against the emulation's, byte for byte but for the libm-derived values."""
    T = 8
    name, kw = _staging_kwargs(branch, T)
    seeds = [7000 + 11 * e for e in range(E_STAGING)]
    envs = []
    for factory in (None, _emu()):
        extra = dict(stepper_factory=factory) if factory else dict(device="cuda:0")
        env, line, _ = _created(monkeypatch, capfd, lambda: foundation.make_env_instance(
            name, n_envs=E_STAGING, auto_reset=True, seed=2024, **kw, **extra), STAGING[branch][1])
        assert branch in placement(line)[0], (branch, line)
        env.seed(seeds)
        env.reset()
        envs.append(env)
    cuda, emu = envs
    # a house pays the builder its Pareto-skill payment: from then on coin carries that payment's last-place difference
    libm = dict(libm_fields=rd.SKILL_FIELDS + ("util_prev", "coin"), libm_bufs=("reward",))
    rd._compare_large(cuda, emu, "reset", **libm)
    seg_a, seg_p = bu.segments(cuda.spec, "a"), bu.segments(cuda.spec, "p")
    rng = np.random.RandomState(17)
    sc = cuda.stepper
    for t in range(1, 2 * T + 2):
        aa = bu.sample_from_masks(sc.to_numpy(sc.buf["mask_agent"]), seg_a, rng)
        ap = bu.sample_from_masks(sc.to_numpy(sc.buf["mask_planner"]), seg_p, rng) if seg_p else None
        cuda.step((aa, ap))
        emu.step((aa, ap))
        if t % T in (0, 1) or t == T // 2:   # the step that resets, the one after, one mid-episode
            rd._compare_large(cuda, emu, "t=%d" % t, **libm)
    assert int(sc.to_numpy(sc.state_view("completions")).min()) == 2


# ------------------------------------------------------------------------------------------ C. compact transfer
# layouts beyond tests/test_compact_transfer.py: c5-small's open-order counts need uint16 ((A - 1) * K = 1 550 > 255) and
# its four-warp records step in two chunks; Gather only; no auction; no spatial planner; dynamic multi-zone layouts; Saez;
# split layout; the redistribution component; a wide price range
COMPACT = ["c5_small", "cda_wide_prices", "gather_only_unscaled", "multi_zone", "saez_reset", "split_layout",
           "tax_period_one", "wealth_redistribution", "wide_window_no_cda"]


@pytest.mark.parametrize("cfg", COMPACT)
def test_emulated_compact_transfer_on_more_layouts(cfg):
    _check(cfg, 5, factory=_emu())


def test_compact_record_carries_c5_open_order_counts_as_uint16():
    """(A - 1) * K > 255: every open-order count of the agents' flat vectors takes two bytes in the compact record.  With
    K = 8 (31 * 8 = 248) the same layout takes one byte per count; the records differ by exactly A * n_counts bytes."""
    def record(K):
        kw = dict(CONFIGS["c5_small"])
        name = kw.pop("scenario_name")
        kw.pop("seed", None)
        kw["components"] = [(c, dict(a, max_num_orders=K) if c == "ContinuousDoubleAuction" else a)
                            for c, a in kw["components"]]
        env = foundation.make_env_instance(name, n_envs=1, stepper_factory=_emu(), **kw)
        counts = sum(n for key, _, n in env.stepper.flat_layout("agent") if "-available_" in key or "-my_" in key)
        return env.stepper.compact_bytes_per_env(), counts, env.n_agents
    wide, counts, A = record(50)
    narrow, counts8, _ = record(8)
    assert A == 32 and counts == counts8 == 8 * 11   # (bids, asks) x (available, own) x (Stone, Wood) x 11 price levels
    assert wide - narrow == A * counts


_GPU_COMPACT = [(cfg, n) for cfg in COMPACT for n in (1, 17, 300)] + [("c5_full", 1), ("c5_full", 17)]


@pytest.mark.gpu
@pytest.mark.parametrize("cfg,n_envs", _GPU_COMPACT)
def test_cuda_compact_transfer_on_more_layouts(cfg, n_envs):
    _check(cfg, n_envs, device="cuda:0")


@pytest.mark.gpu
@pytest.mark.parametrize("item_envs", [8, 64])
@pytest.mark.parametrize("cfg", ["c5_small", "multi_zone"])
def test_cuda_compact_transfer_work_item_sizes(cfg, item_envs, monkeypatch):
    monkeypatch.setenv("AIE_E2E_ITEM_ENVS", str(item_envs))
    _check(cfg, 300, device="cuda:0", threads=(0, 3))


@pytest.mark.gpu
@pytest.mark.parametrize("cfg", ["c5_small", "multi_zone"])
def test_cuda_compact_transfer_overflow_on_more_layouts(cfg, monkeypatch):
    """Index-plane capacities forced down to 4 entries: every env takes the direct-fetch path, multi_zone's spatial
    planner index plane (p_idx) included."""
    assert configs.CONFIGS[cfg].get("planner_gets_spatial_info", True)
    monkeypatch.setenv("AIE_COMPACT_TINY_CAPS", "1")
    _check(cfg, 64, device="cuda:0", threads=(4,))
