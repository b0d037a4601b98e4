"""CPU: the C oracle against the reference on seeds and lengths other than the golden traces', with the full observations
compared at every step: against traces recorded from the unmodified reference (tests/golden/live/, written by
oracle/gen_golden.py), and in addition against the live imported reference wherever a reference checkout is present."""
import os

import pytest

from oracle import ref_harness as rh
from tests import golden_utils as gu
from tests.test_oracle_golden import OracleStepper

LIVE_DIR = os.path.join(gu.GOLDEN_DIR, "live")


@pytest.mark.parametrize("cfg,seed,steps", [
    ("c1_tutorial", 31, 150), ("c3_short_period", 32, 120), ("c5_small", 33, 40), ("ref_unit_test", 34, 60),
])
def test_oracle_tracks_live_reference(cfg, seed, steps):
    assert gu.replay(os.path.join(LIVE_DIR, "%s_seed%d.npz" % (cfg, seed)), OracleStepper) == steps
    if rh.reference_available():
        from oracle.validate_vs_reference import run
        assert run(cfg, seed, steps, verbose=False)
