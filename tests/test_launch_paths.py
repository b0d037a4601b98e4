"""-m gpu: every launch path of the step computes the same bytes.

The launch shape of the step kernel is chosen from the device's shared memory (envs per CTA, register variant), and
tuning overrides change it: AIE_STEP_WPB, AIE_STEP_MINB, AIE_MW, AIE_SPLIT, AIE_PHASE_SYNC.  The caller may also step
the dynamics and the observation pass as two launches (aie_step_dynamics + aie_observe) instead of the fused aie_step.
All of these run the same source with the same arithmetic, so each variant must reproduce the default launch bit for
bit: the state records and every output buffer, at every step, across auto-resets.  A variant that changes the record
layout (AIE_SPLIT) is compared field by field.  The batch of 37 envs leaves the last CTA partial for every envs-per-CTA
count but one.

Also here: the stand-alone observation pass right after a fused step reproduces the fused pass's outputs (the one-warp
kernel compiles the pass for its component set, aie_observe for every component kind), and the fused random policy
draws the same actions on the GPU as in the host emulation.
"""
import numpy as np
import pytest

from ai_economist_b200 import foundation
from oracle.configs import CONFIGS
from tests import batch_utils as bu
from tests.test_staging_plan import CASES as STAGING

pytestmark = pytest.mark.gpu

E = 37
T = 10        # episode length: two auto-resets inside the run
STEPS = 25
KNOBS = ("AIE_STEP_WPB", "AIE_STEP_MINB", "AIE_MW", "AIE_SPLIT", "AIE_PHASE_SYNC")
ONE_WARP = {"minb3": {"AIE_STEP_MINB": "3"}, "minb4": {"AIE_STEP_MINB": "4"}, "wpb1": {"AIE_STEP_WPB": "1"},
            "wpb3": {"AIE_STEP_WPB": "3"}, "phase_sync": {"AIE_PHASE_SYNC": "1"}, "dynamics_then_observe": {}}
# config -> variants; one config per instantiation of the step kernel and per staging branch
CASES = {
    "c1_tutorial": dict(ONE_WARP, mw4={"AIE_MW": "4"}),                 # <MINB, false, CS_GTB>
    "c3_paper_tax": dict(ONE_WARP, mw4={"AIE_MW": "4"}),                # <MINB, false, CS_GTB_TAX>
    "wealth_redistribution": dict(ONE_WARP),                            # <MINB, false, CS_ALL>
    "tax_single_planner": dict(ONE_WARP),                               # <MINB, true, CS_ALL> (EXT)
    "saez_reset": dict(ONE_WARP),                                       # Saez section read by the observation pass
    "uniform_reset": dict(ONE_WARP),                                    # reset_mode 1: device reset inside the kernel
    "c5_small": {"split": {"AIE_SPLIT": "1"}, "dynamics_then_observe": {}},   # four warps per env
    "shifted_late_block": dict(ONE_WARP),                               # staging branches (tests/test_staging_plan.py)
    "early_in_extra": dict(ONE_WARP),
}
# named state fields compared where the record layout differs (aie_host.h: lookup_field)
FIELDS = ["t", "tax_pos", "completions", "auto_warmup", "mt_pos", "episodes", "stats", "saez_n", "saez_rates",
          "saez_avg_rates", "saez_obs_rates", "util_prev", "gauss_state", "coin", "esc_coin", "labor", "build_payment",
          "build_skill", "bonus_gather_prob", "last_coin", "last_income", "last_marg", "price_hist", "inv", "esc", "loc",
          "n_orders", "bid_hist", "ask_hist", "rate_idx", "cell", "owner", "orders", "mt_key"]


def _kwargs(cfg):
    kw = dict(STAGING[cfg][0] if cfg in STAGING else CONFIGS[cfg])
    name = kw.pop("scenario_name")
    kw["components"] = [tuple(c) for c in kw["components"]]
    kw["episode_length"] = T
    kw.pop("seed", None)
    return name, kw


def _make(cfg, environ, monkeypatch, factory=None, n_envs=E):
    for k in KNOBS:
        monkeypatch.delenv(k, raising=False)
    for k, v in environ.items():
        monkeypatch.setenv(k, v)
    name, kw = _kwargs(cfg)
    dev = dict(stepper_factory=factory) if factory else dict(device="cuda:0")
    env = foundation.make_env_instance(name, n_envs=n_envs, auto_reset=True, **kw, **dev)
    for k in environ:   # the knobs are read when the handle is created
        monkeypatch.delenv(k)
    env.seed([7000 + 11 * e for e in range(n_envs)])
    env.reset()
    return env


def _bytes(st, buf):
    return np.ascontiguousarray(st.to_numpy(buf)).view(np.uint8)


def _fields(st):
    out = {}
    for k in FIELDS:
        try:
            out[k] = np.ascontiguousarray(st.to_numpy(st.state_view(k))).view(np.uint8)
        except Exception:   # not part of this config's record
            continue
    return out


def _compare(base, other, label, by_field):
    sb, so = base.stepper, other.stepper
    for k in sorted(sb.buf):
        if k.startswith("actions") or (by_field and k in ("state", "state0", "episode_final")):
            continue
        a, b = _bytes(sb, sb.buf[k]), _bytes(so, so.buf[k])
        if not np.array_equal(a, b):
            bad = np.argwhere(a.reshape(E, -1) != b.reshape(E, -1))[:1].tolist()
            raise AssertionError("%s: %s differs (first [env, byte] %s)" % (label, k, bad))
    if by_field:
        fa, fb = _fields(sb), _fields(so)
        assert fa.keys() == fb.keys(), label
        for k in fa:
            assert np.array_equal(fa[k], fb[k]), "%s: state field %s differs" % (label, k)


@pytest.mark.parametrize("cfg", sorted(CASES))
def test_every_launch_path_gives_the_bytes_of_the_default_launch(cfg, monkeypatch):
    base = _make(cfg, {}, monkeypatch)
    variants = {}
    for v, environ in sorted(CASES[cfg].items()):
        env = _make(cfg, environ, monkeypatch)
        if v == "dynamics_then_observe":
            st = env.stepper
            st.step = lambda st=st: (st.step_dynamics(), st.observe())
        variants[v] = env
        _compare(base, env, "%s/%s after reset" % (cfg, v), by_field="AIE_SPLIT" in environ)
    sb = base.stepper
    seg_a, seg_p = bu.segments(base.spec, "a"), bu.segments(base.spec, "p")
    rng = np.random.RandomState(3)
    outs = [k for k in sb.buf if k.startswith(("obs_", "mask_"))]
    for t in range(1, STEPS + 1):
        aa = bu.sample_from_masks(sb.to_numpy(sb.buf["mask_agent"]), seg_a, rng)
        ap = bu.sample_from_masks(sb.to_numpy(sb.buf["mask_planner"]), seg_p, rng) if seg_p else None
        for env in [base] + list(variants.values()):
            env.step((aa, ap))
        for v, env in variants.items():
            _compare(base, env, "%s/%s t=%d" % (cfg, v, t), by_field="AIE_SPLIT" in CASES[cfg][v])
        fused = {k: _bytes(sb, sb.buf[k]) for k in outs}
        sb.observe()   # stand-alone pass over the same records
        for k in outs:
            assert np.array_equal(fused[k], _bytes(sb, sb.buf[k])), "%s t=%d: aie_observe changed %s" % (cfg, t, k)
    assert int(sb.to_numpy(sb.state_view("completions")).min()) == 2


def _bits(a):
    a = np.ascontiguousarray(a)
    return a.view(np.dtype("u%d" % a.dtype.itemsize)) if a.dtype.kind in "iu" else a


@pytest.mark.parametrize("cfg", ["c1_tutorial", "c3_paper_tax", "c5_small"])
def test_cuda_fused_policy_equals_emulation(cfg, monkeypatch):
    """The path bench.py times: the observation pass draws the next step's actions (aie_set_fused_policy).  The draw is
    integer-only on the mask limits, so the actions must agree exactly; the state too, floats to the tolerances of
    tests/test_cuda_vs_emulation.py."""
    from tests.emu.emu_stepper import emu_factory
    cuda, emu = _make(cfg, {}, monkeypatch, n_envs=8), _make(cfg, {}, monkeypatch, emu_factory, n_envs=8)
    sc, se = cuda.stepper, emu.stepper
    for st in (sc, se):
        st.set_fused_policy(4242)
    for t in range(1, 3 * T + 1):
        for k in ("actions_agent", "actions_planner"):
            assert np.array_equal(sc.to_numpy(sc.buf[k]), se.to_numpy(se.buf[k])), "t=%d: %s" % (t, k)
        cuda.step(cuda.action_buffers)
        emu.step(emu.action_buffers)
        for k in ("cell", "owner", "loc", "inv", "esc", "n_orders", "bid_hist", "ask_hist", "mt_key", "mt_pos", "t",
                  "completions"):
            a, b = _bits(sc.to_numpy(sc.state_view(k))), _bits(se.to_numpy(se.state_view(k)))
            assert np.array_equal(a, b), "t=%d: state %s" % (t, k)
        for k in ("coin", "esc_coin", "labor", "price_hist"):
            assert np.allclose(sc.to_numpy(sc.state_view(k)), se.to_numpy(se.state_view(k)), rtol=1e-9, atol=1e-12), (t, k)
        for k in ("mask_agent", "mask_planner", "obs_agent_idx", "obs_agent_map"):
            assert np.array_equal(sc.to_numpy(sc.buf[k]), se.to_numpy(se.buf[k])), "t=%d: %s" % (t, k)
        for k in ("obs_agent_flat", "obs_planner_flat", "reward"):
            assert np.allclose(sc.to_numpy(sc.buf[k]), se.to_numpy(se.buf[k]), rtol=1e-6, atol=1e-7), "t=%d: %s" % (t, k)
    assert int(sc.to_numpy(sc.state_view("completions")).min()) >= 2
