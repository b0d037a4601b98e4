"""The observation pass's staging plan (aie_host.h: build_devcfg, `place`) against the oracle, one config per branch.

The pass stages its buffers on top of the dead parts of the env's shared-memory region.  The early buffers (used before
the record's write-back has been read) go into the MT19937 key image, then into the step scratch, or - when one of them
fits in neither - all into extra memory behind the region.  The late buffers follow the early ones in the key image and
run on into extra memory; when early buffers sit in the step scratch and the late block does not fit in front of them,
the whole late block moves behind the region.  A split record keeps its price history and order slots in global memory.

The host emulation runs the kernels on an image of that region (0xFF wherever the kernel has not loaded or written
anything), so a wrong offset in the plan shows up here as a NaN / -1 in the outputs.  Each case asserts which branch its
config takes (read from the AIE_VERBOSE line of aie_create) and steps the emulation against the C oracle.
"""
import re

import numpy as np
import pytest

from ai_economist_b200 import foundation
from oracle.configs import CONFIGS
from oracle.oracle import OracleBatch
from tests import batch_utils as bu

_UNIFORM = dict(multi_action_mode_agents=False, multi_action_mode_planner=True, flatten_observations=True,
                flatten_masks=True, starting_agent_coin=10, starting_wood_coverage=0.1, starting_stone_coverage=0.1)


def _uniform(A, S, max_bid_ask, K):
    return dict(scenario_name="uniform/simple_wood_and_stone",
                components=[("Build", {}), ("ContinuousDoubleAuction", dict(max_num_orders=K, max_bid_ask=max_bid_ask)),
                            ("Gather", {})],
                n_agents=A, world_size=[S, S], episode_length=100, **_UNIFORM)


# branch -> (config, environment of aie_create)
CASES = {
    # 10 agents on 40x40: the location map fills most of the key image, three early buffers go to the step scratch
    "early_in_scratch": (CONFIGS["c3_paper_tax"], {}),
    # 6 agents on 40x40, one order slot: early buffers in the step scratch, and the small record leaves too little room
    # in front of them for the late block
    "shifted_late_block": (_uniform(6, 40, 10, 1), {}),
    # 3 agents on 44x44: the location map fits neither the key image nor the step scratch (one warp per env)
    "early_in_extra": (_uniform(3, 44, 10, 1), {}),
    # c5-small under AIE_SPLIT=1: four warps per env, price history and order slots in global memory
    "split_record": (CONFIGS["c5_small"], {"AIE_SPLIT": "1"}),
}


def placement(line):
    """The staging branches one AIE_VERBOSE line of aie_create reports."""
    m = re.search(r"record (\d+) B \(resident (\d+), obs prefix \d+, mt @(\d+), price_hist @\d+\), step scratch (\d+), "
                  r"obs extra (\d+) \(alias mt (\d)\).* mw (\d+),.*; ob:((?: -?\d+)+)", line)
    assert m, line
    rec, res, mt, scr, extra, alias, mw = (int(v) for v in m.groups()[:7])
    ob = [int(v) for v in m.group(8).split()]
    early, late = ob[:6], ob[6:10]   # OB_NET_HIST .. OB_LOCMAP; OB_WC, OB_WI, OB_PL, OB_BITS (aie_layout.h)
    got = set()
    if alias:
        assert all(mt <= o < mt + 2496 or res <= o < res + scr for o in early), line
        if any(res <= o < res + scr for o in early):
            got.add("early_in_scratch")
            if min(late) == res + scr:
                got.add("shifted_late_block")
    else:
        assert extra > 0 and all(o >= res + scr for o in early), line
        got.add("early_in_extra")
    if res < rec:
        got.add("split_record")
    return got, mw


@pytest.mark.parametrize("branch", sorted(CASES))
def test_emulated_staging_branch_matches_oracle(branch, monkeypatch, capfd):
    from tests.emu.emu_stepper import emu_factory
    cfg, environ = CASES[branch]
    for k, v in environ.items():
        monkeypatch.setenv(k, v)
    monkeypatch.setenv("AIE_VERBOSE", "1")
    kw = dict(cfg)
    name = kw.pop("scenario_name")
    kw["components"] = [tuple(c) for c in kw["components"]]
    E = 2 if branch == "split_record" else 3
    capfd.readouterr()
    env = foundation.make_env_instance(name, n_envs=E, stepper_factory=emu_factory, auto_reset=False, seed=2024, **kw)
    lines = [ln for ln in capfd.readouterr().err.splitlines() if ln.startswith("[aie] A ")]
    assert len(lines) == 1, lines
    got, mw = placement(lines[0])
    assert branch in got, (branch, lines[0])
    if branch == "split_record":
        assert mw == 4
    host = env.host_reset_arrays()
    env.load_host_state(host)   # the stand-alone observation pass
    orc = OracleBatch(env.spec, E)
    for e in range(E):
        orc.load_env(e, {k: v[e] for k, v in host.items()})
        bu.compare_env(orc, env.stepper, e, "reset", spatial=bool(env.spec["planner_gets_spatial_info"]))
    bu.run_pair(env, orc, 30, np.random.RandomState(31), check_every=10)
