"""The batched episode metrics (aie_episode_metrics, env.metrics_tensor / previous_episode_metrics_tensor): one kernel
launch computes env.metrics of every replica on the device.  Each row must be what the per-replica path
(metrics_of / previous_episode_metrics_of, i.e. foundation/metrics.py on one record) returns, in the same key order.

The kernel sums in numpy's order (pairwise summation, the Gini's A x A differences as one np.sum, sort + cumsum), so
the rows are bit-equal to metrics_from_state.  The one documented exception is labor/weighted_cost under an energy
warm-up: 1 - exp(-x / c) uses the platform's exp (CUDA, or libm in the emulation), which can differ from numpy's in the
last place; it is held to 1e-12 relative.

CPU: the 1-lane emulation of the device source through the same C-ABI.  GPU: the CUDA kernel."""
import ctypes as C
import glob
import json
import math
import os

import numpy as np
import pytest

from ai_economist_b200 import _abi, foundation
from ai_economist_b200.foundation.metrics import metrics_from_state
from tests import golden_utils as gu
from tests import metrics_utils as mu
from tests.stepper_adapters import GoldenStepperAdapter

NOT_BIT_EQUAL = {"labor/weighted_cost": 1e-12}
GOLDEN_RESET = sorted(glob.glob(os.path.join(mu.HERE, "golden_metrics_reset", "*.json")))


def assert_same_metrics(got, want, label):
    """got / want: metrics dicts.  Same keys in the same order; ints exact (and int), NaN where want is NaN, floats
    bit-equal except the documented keys."""
    assert list(got) == list(want), "%s: key order differs" % label
    for k, w in want.items():
        g = got[k]
        if isinstance(w, int):
            assert type(g) is int and g == w, "%s: %s = %r, want %r" % (label, k, g, w)
        elif math.isnan(w):
            assert isinstance(g, float) and math.isnan(g), "%s: %s = %r, want NaN" % (label, k, g)
        elif k in NOT_BIT_EQUAL:
            assert abs(g - w) <= NOT_BIT_EQUAL[k] * abs(w), "%s: %s = %r, want %r" % (label, k, g, w)
        else:
            assert g == w, "%s: %s = %r, want %r (not bit-equal)" % (label, k, g, w)


def rows_as_dicts(stepper, rows):
    a = rows.detach().cpu().numpy() if hasattr(rows, "detach") else np.asarray(rows)
    lay = stepper.metric_layout()
    return [None if np.isnan(r).all() else {k: (int(v) if i else float(v)) for (k, i), v in zip(lay, r.tolist())}
            for r in a]


# ---------------------------------------------------------------------------------------------------------------------
# 1 / 5: golden traces
def _replay_golden(path, make_stepper):
    ref = json.load(open(path))
    z, meta, init = gu.load_fixture(os.path.join(mu.HERE, "golden", ref["fixture"]))
    spec = meta["spec"]
    st = make_stepper(spec)
    ad = GoldenStepperAdapter(st, init)
    want = dict(zip(ref["steps"], ref["metrics"]))
    checked = 0
    for t in range(1, int(meta["n_steps"]) + 1):
        ap = z["act_p"][t - 1].astype(np.int32)
        ad.step(z["act_a"][t - 1].astype(np.int32), ap if ap.size else None)
        if t in want:
            label = "%s t=%d" % (ref["fixture"], t)
            row = rows_as_dicts(st, st.episode_metrics())[0]
            mu.compare_metrics(want[t], row, label)
            assert_same_metrics(row, metrics_from_state(spec, ad.state()), label)
            checked += 1
    assert checked >= 3


@pytest.mark.parametrize("path", mu.metric_files(), ids=lambda p: p.split("/")[-1])
def test_emulated_metrics_rows_match_reference_and_per_replica_path(path):
    from tests.emu.emu_stepper import EmuStepper
    _replay_golden(path, lambda spec: EmuStepper(spec, 1))


def _replay_golden_reset(path, factory):
    """Multi-episode traces: previous_episode_metrics_tensor() row of replica 1 after each auto-reset == the reference's
    previous_episode_metrics, and == previous_episode_metrics_of(1)."""
    ref = json.load(open(path))
    want = dict(zip(ref["steps"], ref["metrics"]))
    z, meta, init = gu.load_fixture(path.replace("golden_metrics_reset", "golden_reset").replace(".json", ".npz"))
    kw = dict(meta["reference_kwargs"])
    name = kw.pop("scenario_name")
    kw["components"] = [tuple(c) for c in kw["components"]]
    if "seed" in kw:
        kw["seeds"] = [kw.pop("seed")] * 2
    extra = dict(stepper_factory=factory) if factory else dict(device="cuda:0")
    env = foundation.make_env_instance(name, n_envs=2, auto_reset=True, **kw, **extra)
    env.seed([meta["seed"], meta["seed"]])
    env.reset()
    assert env.metrics_rows_as_dicts(env.previous_episode_metrics_tensor()) == [None, None]
    seen = 0
    for t in range(1, int(meta["n_steps"]) + 1):
        acts = {str(i): np.repeat(z["act_a"][t - 1][i][None], 2, axis=0) for i in range(env.n_agents)}
        if z["act_p"].shape[1]:
            acts["p"] = np.repeat(z["act_p"][t - 1][None], 2, axis=0)
        env.step(acts)
        cur = env.metrics_rows_as_dicts(env.metrics_tensor())
        assert_same_metrics(cur[1], env.metrics_of(1), "current t=%d" % t)
        if t in want:
            prev = env.metrics_rows_as_dicts(env.previous_episode_metrics_tensor())
            mu.compare_metrics(want[t], prev[1], "episode ending at t=%d" % t)
            assert_same_metrics(prev[1], env.previous_episode_metrics_of(1), "episode ending at t=%d" % t)
            seen += 1
    assert seen >= 2


@pytest.mark.parametrize("path", GOLDEN_RESET, ids=lambda p: os.path.basename(p))
def test_emulated_previous_episode_rows_match_reference_across_episodes(path):
    from tests.emu.emu_stepper import emu_factory
    _replay_golden_reset(path, emu_factory)


# ---------------------------------------------------------------------------------------------------------------------
# 2 / 3: many replicas, auto-reset, configurations the golden traces do not cover
_LAYOUT = dict(env_layout_file="quadrant_25x25_20each_30clump.txt", world_size=[25, 25], starting_agent_coin=5,
               fixed_four_skill_and_loc=False)
_GTB = [("Build", dict(skill_dist="pareto", payment_max_skill_multiplier=3)),
        ("ContinuousDoubleAuction", dict(max_num_orders=3, order_duration=7)), ("Gather", dict(skill_dist="pareto"))]
_LFF = "layout_from_file/simple_wood_and_stone"


def _tax(**kw):
    return ("PeriodicBracketTax", dict(dict(bracket_spacing="us-federal", period=5), **kw))


def _one_step_config():
    z = np.load(os.path.join(mu.HERE, "golden_one_step", "paper_like_seed1001.npz"))
    kw = dict(json.loads(str(z["meta_json"]))["reference_kwargs"])
    kw["components"] = [tuple(c) for c in kw["components"]]
    return kw.pop("scenario_name"), kw


EXPLICIT = {
    "sorted_gini_32_agents": (_LFF, dict(_LAYOUT, components=_GTB + [_tax()], n_agents=32)),
    "welfare_inv_income_coin": (_LFF, dict(_LAYOUT, components=_GTB + [_tax()], n_agents=5,
                                           planner_reward_type="inv_income_weighted_coin_endowments")),
    "welfare_inv_income_utility": (_LFF, dict(_LAYOUT, components=_GTB, n_agents=6,
                                              planner_reward_type="inv_income_weighted_utility")),
    # usd_scaling 1e6: every cutoff truncates to 0, so all brackets pool under the key "000"
    "duplicate_bracket_keys": (_LFF, dict(_LAYOUT, components=_GTB + [_tax(usd_scaling=1e6)], n_agents=4)),
    "disable_taxes": (_LFF, dict(_LAYOUT, components=_GTB + [_tax(disable_taxes=True)], n_agents=4)),
    "saez": (_LFF, dict(_LAYOUT, components=_GTB + [_tax(tax_model="saez", usd_scaling=10000.0)], n_agents=10)),
    "saez_annealed": (_LFF, dict(_LAYOUT, components=_GTB + [_tax(tax_model="saez", usd_scaling=10000.0,
                                                                   tax_annealing_schedule=[-2, 0.15])], n_agents=10)),
    "one_step_economy": _one_step_config(),
    "gather_only": (_LFF, dict(_LAYOUT, components=[("Gather", {})], n_agents=3)),
    "warmup_decay": (_LFF, dict(_LAYOUT, components=_GTB, n_agents=4, energy_warmup_constant=3,
                                energy_warmup_method="decay")),
    "warmup_auto": (_LFF, dict(_LAYOUT, components=_GTB, n_agents=4, energy_warmup_constant=3,
                               energy_warmup_method="auto")),
}


def _fuzz_configs(n=20, seed=20261016):
    from tools.fuzz_emu_vs_oracle import random_config
    rng = np.random.RandomState(seed)
    return {"random_%d" % i: random_config(rng) for i in range(n)}


CONFIGS = dict(EXPLICIT, **_fuzz_configs())
E, T = 8, 12


def _check_all_rows(env, label):
    cur = env.metrics_rows_as_dicts(env.metrics_tensor())
    for e in range(env.n_envs):
        assert_same_metrics(cur[e], env.metrics_of(e), "%s current e=%d" % (label, e))
    if "episode_final" not in env.stepper.buf:
        with pytest.raises(_abi.AieError, match="episode_final"):
            env.previous_episode_metrics_tensor()
        return
    prev = env.metrics_rows_as_dicts(env.previous_episode_metrics_tensor())
    for e in range(env.n_envs):
        want = env.previous_episode_metrics_of(e)
        if want is None:
            assert prev[e] is None, "%s previous e=%d: a row for a replica that has finished no episode" % (label, e)
        else:
            assert_same_metrics(prev[e], want, "%s previous e=%d" % (label, e))


def _run(name, kw, factory, auto_reset=True, n_envs=E, steps=None):
    kw = dict(kw, episode_length=T if name != "one-step-economy" else kw.get("episode_length", 1))
    kw.pop("seed", None)
    extra = dict(stepper_factory=factory) if factory else dict(device="cuda:0")
    env = foundation.make_env_instance(name, n_envs=n_envs, auto_reset=auto_reset, seeds=[101 + 7 * e for e in range(n_envs)],
                                       **kw, **extra)
    env.reset()
    assert env.metric_keys == list(env.metrics_of(0))
    T_ = env.episode_length
    n = steps if steps is not None else T_ + T_ // 2 + 1   # across one episode boundary (auto-reset)
    for t in range(n):
        env.stepper.sample_random_actions(seed=1 + t)
        env.step(env.action_buffers)
        if t in (0, T_ - 1, n - 1):
            _check_all_rows(env, "%s t=%d" % (name, t + 1))
    return env


@pytest.mark.parametrize("which", sorted(CONFIGS))
def test_emulated_metrics_rows_match_per_replica_path(which):
    from tests.emu.emu_stepper import emu_factory
    name, kw = CONFIGS[which]
    _run(name, kw, emu_factory)


@pytest.mark.parametrize("which", ["warmup_decay", "warmup_auto"])
def test_emulated_finished_episode_waiting_for_reset_counts_like_metrics_of(which):
    """auto_reset off, every replica at t == episode_length: labor/weighted_cost counts the finished episode (metrics_of's
    completions + 1), and there are no end-of-episode records to read."""
    from tests.emu.emu_stepper import emu_factory
    name, kw = CONFIGS[which]
    env = _run(name, kw, emu_factory, auto_reset=False, steps=T)
    t = env.stepper.to_numpy(env.stepper.state_view("t"))
    assert (t >= T).all()
    row = env.metrics_rows_as_dicts(env.metrics_tensor())[0]
    assert row["labor/weighted_cost"] == pytest.approx(env.metrics_of(0)["labor/weighted_cost"], rel=1e-12)
    if which == "warmup_decay":   # "decay" anneals by the completion count ("auto" by the integrator, which no reset moves)
        assert row["labor/weighted_cost"] != env.metrics_of(0, _count_finished=False)["labor/weighted_cost"]


# ---------------------------------------------------------------------------------------------------------------------
# 4: the C-ABI's errors
def test_metrics_abi_errors():
    from ai_economist_b200.workloads import product_kwargs
    from tests.emu.emu_stepper import EmuStepper, emu_lib
    name, kw = product_kwargs("c1_tutorial")
    spec = foundation.make_env_instance(name, n_envs=2, auto_reset=False, stepper_factory=lambda *a, **k: None, **kw).spec
    lib = emu_lib()
    st = EmuStepper(spec, 2, auto_reset=False)
    K = len(st.metric_layout())
    out = np.zeros((2, K))
    p = out.ctypes.data_as(C.c_void_p)
    assert lib.aie_episode_metrics(st._h, 0, None, None) == -1                   # NULL out: AIE_EINVAL
    assert lib.aie_episode_metrics(st._h, 2, p, None) == -1                      # unknown source: AIE_EINVAL
    assert lib.aie_episode_metrics(st._h, -1, p, None) == -1
    assert lib.aie_episode_metrics(st._h, 1, p, None) == -3                      # no episode_final: AIE_ESTATE
    assert lib.aie_last_error().decode() == "aie_episode_metrics: no episode_final buffer bound"
    assert lib.aie_episode_metrics(st._h, 0, p, None) == 0
    # before aie_bind_buffers
    cfg, h = _abi.config_from_spec(spec, auto_reset=True), C.c_void_p()
    assert lib.aie_create(C.byref(cfg), 2, 0, C.byref(h)) == 0
    try:
        assert lib.aie_episode_metrics(h, 0, p, None) == -3
        assert "not bound" in lib.aie_last_error().decode()
        # cap smaller than K: returns K, writes only cap entries
        arr = (_abi.AieMetricKey * K)()
        for i in range(K):
            arr[i].key, arr[i].is_int = b"untouched", 7
        assert lib.aie_get_metric_layout(h, arr, 3) == K
        assert [arr[i].key.decode() for i in range(3)] == list(st.metric_layout()[i][0] for i in range(3))
        assert all(arr[i].key == b"untouched" and arr[i].is_int == 7 for i in range(3, K))
        assert lib.aie_get_metric_layout(h, None, 0) == K
        assert lib.aie_get_metric_layout(h, None, 5) == -1                       # cap > 0 with a NULL array
    finally:
        lib.aie_destroy(h)
    with pytest.raises(_abi.AieError, match="contiguous float64"):
        st.episode_metrics(out=np.zeros((2, K), np.float32))


def test_emulated_metrics_count_one_launch_and_fill_a_given_buffer():
    from tests.emu.emu_stepper import emu_factory
    name, kw = EXPLICIT["saez"]
    env = _run(name, kw, emu_factory, steps=3)
    st = env.stepper
    out = np.full((env.n_envs, len(env.metric_keys)), -1.0)
    n0 = st.launch_count()
    assert env.metrics_tensor(out=out) is out and st.launch_count() == n0 + 1
    col = env.metric_keys.index("PeriodicTax/saez/estimated_elasticity")
    assert np.array_equal(out[:, col], np.asarray(env._saez.batch.elas_tm1, np.float64))


# ---------------------------------------------------------------------------------------------------------------------
# GPU
@pytest.mark.gpu
@pytest.mark.parametrize("path", mu.metric_files(), ids=lambda p: p.split("/")[-1])
def test_cuda_metrics_rows_match_reference_and_per_replica_path(path):
    from ai_economist_b200.stepper import CudaStepper
    _replay_golden(path, lambda spec: CudaStepper(spec, 1, auto_reset=False))


@pytest.mark.gpu
@pytest.mark.parametrize("path", GOLDEN_RESET, ids=lambda p: os.path.basename(p))
def test_cuda_previous_episode_rows_match_reference_across_episodes(path):
    _replay_golden_reset(path, None)


@pytest.mark.gpu
@pytest.mark.parametrize("which", ["sorted_gini_32_agents", "duplicate_bracket_keys", "saez_annealed", "one_step_economy",
                                   "welfare_inv_income_utility", "warmup_auto"])
def test_cuda_metrics_rows_match_per_replica_path(which):
    name, kw = CONFIGS[which]
    _run(name, kw, None)


@pytest.mark.gpu
@pytest.mark.parametrize("workload,n_envs", [("c1_tutorial", 8192), ("c3_paper_tax", 8192), ("c5_full", 2048)],
                         ids=["c2", "c3", "c5"])
def test_cuda_full_size_staggered_rows_match_per_replica_path_and_emulation(workload, n_envs):
    """The benchmark's workloads at full size, episodes staggered (replica e starts at t = e*T/E), run for more than one
    episode length.  A fixed sample of replicas (plus every replica whose episode ended in the last step) against the
    per-replica path; every row against the host emulation's metrics kernel run on the same records."""
    import torch
    from ai_economist_b200.workloads import product_kwargs
    from tests.emu.emu_stepper import EmuStepper
    name, kw = product_kwargs(workload)
    env = foundation.make_env_instance(name, n_envs=n_envs, device="cuda:0", seeds=list(range(1000, 1000 + n_envs)),
                                       auto_reset=True, **kw)
    env.reset()
    st, T = env.stepper, env.episode_length
    st.state_view("t").copy_((torch.arange(n_envs, device="cuda:0", dtype=torch.int64) * T // n_envs).to(torch.int32))
    st.set_fused_policy(4321)
    for _ in range(T + 7):
        st.step()
    n0 = st.launch_count()
    cur, prev = env.metrics_tensor(), env.previous_episode_metrics_tensor()
    assert st.launch_count() == n0 + 2
    done = torch.nonzero(st.buf["done"]).flatten().tolist()
    assert done, "no replica finished in the last step"
    sample = sorted(set(np.random.RandomState(0).choice(n_envs, 256, replace=False).tolist()) | set(done))
    cur_d, prev_d = env.metrics_rows_as_dicts(cur, sample), env.metrics_rows_as_dicts(prev, sample)
    for i, e in enumerate(sample):
        assert_same_metrics(cur_d[i], env.metrics_of(e), "%s current e=%d" % (workload, e))
        want = env.previous_episode_metrics_of(e)
        assert want is not None, "every replica has finished an episode after T + 7 steps"
        assert_same_metrics(prev_d[i], want, "%s previous e=%d" % (workload, e))
    # the emulation's metrics kernel on the same records, in chunks
    cur_h, prev_h = cur.cpu().numpy(), prev.cpu().numpy()
    rec, fin = st.buf["state"].cpu().numpy(), st.buf["episode_final"].cpu().numpy()
    chunk = 512
    emu = EmuStepper(env.spec, chunk, auto_reset=True)
    for lo in range(0, n_envs, chunk):
        emu.buf["state"][...] = rec[lo:lo + chunk]
        emu.buf["episode_final"][...] = fin[lo:lo + chunk]
        for got, final in ((cur_h, False), (prev_h, True)):
            want = emu.episode_metrics(final=final)
            close = np.isclose(got[lo:lo + chunk], want, rtol=1e-12, atol=0.0, equal_nan=True)
            assert close.all(), "%s rows %d..: device and emulation differ in %s" % (
                workload, lo, sorted({env.metric_keys[j] for j in np.nonzero(~close)[1]})[:5])
