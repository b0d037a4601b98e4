"""Seeded, bounded subsets of the randomised configuration fuzzers in tools/fuzz_*.py as collected test cases.

The fuzzers draw configurations from the whole supported option space (scenario families, component subsets and orders,
both action modes, tax models incl. annealing, WealthRedistribution, view radius, full observability, regen halfwidths,
social welfare functions, skill distributions).  Unbounded runs are a tool (`python tools/fuzz_*.py N SEED`); here every fuzzer contributes N_CASES configurations drawn from a fixed seed, one test case each:

  * emu vs oracle            CPU, always            the device source (1-lane emulation) against the C oracle
  * cuda vs oracle           -m gpu                 the same configurations on the CUDA build (through the C-ABI)
  * oracle vs reference      -m reference           the C oracle against the live imported reference
  * device reset vs ref.     -m reference           reference-exact auto-reset across 4 episodes against env.reset()
  * reference API vs ref.    -m reference           ReferenceApiEnv against the reference: obs, rewards, metrics, dense logs
  * dynamic layouts vs ref.  -m reference           uniform / quadrant: device-side layout generation at every auto-reset
  * one-step-economy vs ref. -m reference           SimpleLabor + one-step-economy incl. finished-episode metrics
  * Saez hybrid vs reference -m reference           the Saez tax model (device / host), with and without tax annealing
  * COVID vs reference       -m reference           COVID device code (scan and change list) under parameter variants

`-m reference` cases run against the live reference where a checkout is present, and against what it returned there
(tests/golden/reference_tapes/, oracle/ref_tape.py) everywhere else.
"""
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))

import fuzz_emu_vs_oracle as fz  # noqa: E402
from oracle.ref_tape import taped  # noqa: E402

N_CASES = 20


def _configs(seed, n=N_CASES, draw=None):
    rng = np.random.RandomState(seed)
    return [(draw or fz.random_config)(rng) for _ in range(n)]


def _skip_unsupported(fn, *a, **k):
    """Configurations the product rejects loudly or that the reference itself cannot build
    (layout coverage asserts) are skipped, like the tools do."""
    try:
        fn(*a, **k)
    except (NotImplementedError, TimeoutError) as ex:
        pytest.skip("unsupported / unbuildable configuration: %r" % (ex,))


EMU_CASES = _configs(20260923)


@pytest.mark.parametrize("i", range(N_CASES))
def test_fuzz_emulated_device_code_matches_oracle(i):
    name, kw = EMU_CASES[i]
    _skip_unsupported(fz.run_one, name, kw, seed=1 + i, steps=60)


@pytest.mark.gpu
@pytest.mark.parametrize("i", range(N_CASES))
def test_fuzz_cuda_matches_oracle(i):
    """GPU twin of the case above: same configurations, the CUDA build through the C-ABI (incl. the EXT kernels)."""
    from ai_economist_b200 import foundation
    from oracle.oracle import OracleBatch
    from tests import batch_utils as bu

    name, kw = EMU_CASES[i]
    E = 3
    env = foundation.make_env_instance(name, n_envs=E, device="cuda:0", auto_reset=False, seed=1 + i, **kw)
    host = env.host_reset_arrays()
    env.load_host_state(host)
    orc = OracleBatch(env.spec, E)
    for e in range(E):
        orc.load_env(e, {k: v[e] for k, v in host.items()})
    for e in range(E):
        bu.compare_env(orc, env.stepper, e, "reset", spatial=bool(env.spec["planner_gets_spatial_info"]))
    bu.run_pair(env, orc, min(60, kw["episode_length"]), np.random.RandomState(1 + i), check_every=15)


@pytest.mark.reference
@pytest.mark.parametrize("i", range(N_CASES))
@taped
def test_fuzz_oracle_matches_live_reference(i):
    from oracle import configs
    from oracle.validate_vs_reference import run

    name, kw = _configs(5)[i]
    configs.CONFIGS["_fuzz"] = dict(kw, scenario_name=name)
    try:
        ok = run("_fuzz", 100 + i, min(60, kw["episode_length"]), verbose=False)
    except (AssertionError, NotImplementedError, TimeoutError) as ex:   # the reference refusing its own configuration
        pytest.skip("reference / harness refused the configuration: %r" % (ex,))
    assert ok


@pytest.mark.reference
@pytest.mark.parametrize("i", range(N_CASES))
@taped
def test_fuzz_device_reset_matches_live_reference(i):
    import fuzz_device_reset_vs_reference as fr

    cfg = _configs(0, draw=fr.random_config)[i]
    fr.run_one(cfg, seed=500 + i, episodes=3)


@pytest.mark.reference
@pytest.mark.parametrize("i", range(N_CASES))
@taped
def test_fuzz_dynamic_layout_device_reset_matches_live_reference(i):
    """uniform / quadrant: the device generates a new clumped layout at every auto-reset (rand thinning, randn + convolve2d
    growth, coverage retries, checkering, water lines) and must land on the reference's maps, placements and stream."""
    import fuzz_device_reset_vs_reference as fr

    cfg = _configs(11, draw=fr.random_dynamic_config)[i]
    try:
        fr.run_one(cfg, seed=600 + i, episodes=3)
    except TimeoutError as ex:   # the reference's own placement loop giving up on a crowded map
        pytest.skip(repr(ex))


@pytest.mark.reference
@pytest.mark.parametrize("i", range(10))
@taped
def test_fuzz_multi_zone_device_reset_matches_live_reference(i, monkeypatch):
    """multi_zone: np.random.shuffle of the region -> zone-type vector on the device before every layout."""
    import fuzz_device_reset_vs_reference as fr

    monkeypatch.setattr(fr, "FAMILIES", ["multi_zone"])
    cfg = _configs(21, n=10, draw=fr.random_dynamic_config)[i]
    try:
        fr.run_one(cfg, seed=650 + i, episodes=3)
    except (TimeoutError, AssertionError) as ex:
        if isinstance(ex, AssertionError) and "coverage" not in str(ex) and "World" not in str(ex):
            raise
        pytest.skip(repr(ex))   # the reference refusing its own configuration


@pytest.mark.reference
@pytest.mark.parametrize("i", range(10))
@taped
def test_fuzz_saez_hybrid_matches_live_reference(i):
    """PeriodicBracketTax(tax_model="saez"): warm-up draws on the device, buffer / regression / formula on the host, rates in
    force and observed across resets - random bracket layouts, weights, fixed elasticities, rate bounds, with and without a
    tax_annealing_schedule, over enough episodes to run the formula for two of them."""
    import fuzz_device_reset_vs_reference as fr

    cfg = _configs(31, n=10, draw=fr.random_saez_config)[i]
    fr.run_one(cfg, seed=800 + i, episodes=fr.saez_episodes(cfg))


@pytest.mark.reference
@pytest.mark.parametrize("i", range(N_CASES))
@taped
def test_fuzz_reference_api_matches_live_reference(i):
    import fuzz_reference_api_vs_reference as fa

    name, kw = _configs(0)[i]
    _skip_unsupported(fa.run_one, name, kw, seed=700 + i)


@pytest.mark.reference
@pytest.mark.parametrize("i", range(N_CASES))
@taped
def test_fuzz_one_step_economy_matches_live_reference(i):
    """SimpleLabor + one-step-economy (components/simple_labor.py, scenarios/one_step_economy): observations, masks, rewards,
    numpy stream and finished-episode metrics across auto-resets, random reward types / tax settings / populations."""
    import fuzz_one_step_vs_reference as fo

    cfg = _configs(3, draw=fo.random_config)[i]
    fo.run_one(cfg, seed=300 + i, episodes=3)


@pytest.mark.reference
@pytest.mark.parametrize("i", range(8))
@taped
def test_fuzz_covid_matches_live_reference(i):
    import fuzz_covid_vs_reference as fc

    kw = _configs(0, n=8, draw=fc.random_kwargs)[i]
    fc.run_one(kw, 900 + i)
