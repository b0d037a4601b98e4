"""GPU: the CUDA product, called through the C-ABI, against (1) the golden traces recorded from the
unmodified reference and (2) the C oracle on identical seeds + action sequences.

Tolerances (BASELINE.json north_star): bit-exact for grid / inventory / index / mask / RNG state; <= 1e-6
relative for coin / labor / utility / reward floats (atol 1e-9 on float64 state, 1e-7 on float32 observations).
"""
import numpy as np
import pytest

from tests import batch_utils as bu
from tests import golden_utils as gu
from tests.stepper_adapters import GoldenStepperAdapter

pytestmark = pytest.mark.gpu


def _cuda_stepper(spec, n_envs, auto_reset=False):
    from ai_economist_b200.stepper import CudaStepper
    return CudaStepper(spec, n_envs, device="cuda:0", auto_reset=auto_reset)


def _make_env(cfg_name, n_envs, seed, **extra):
    from ai_economist_b200 import foundation
    name, kw = bu.product_kwargs(cfg_name)
    kw.pop("seed", None)   # split_layout carries a constructor seed for its golden trace
    kw.update(extra)
    if "stepper_factory" not in kw:
        kw["device"] = "cuda:0"
    return foundation.make_env_instance(name, n_envs=n_envs, seed=seed, **kw)


def _load_both(env):
    from oracle.oracle import OracleBatch
    host = env.host_reset_arrays()
    env.load_host_state(host)
    orc = OracleBatch(env.spec, env.n_envs)
    for e in range(env.n_envs):
        orc.load_env(e, {k: v[e] for k, v in host.items()})
    return orc, host


@pytest.mark.parametrize("path", gu.golden_files(), ids=lambda p: p.split("/")[-1])
def test_cuda_matches_reference_golden_trace(path):
    def make(spec, init):
        return GoldenStepperAdapter(_cuda_stepper(spec, 3), init, env_index=1)  # env 1 of 3: exercises indexing

    assert gu.replay(path, make) >= 50


@pytest.mark.parametrize("cfg,E,steps,every", [
    ("c1_tutorial", 96, 400, 50),       # c2 shape: 4 agents, 25x25, single-action
    ("c3_paper_tax", 48, 320, 40),      # 10 agents 40x40 + PeriodicBracketTax (3 tax days)
    ("c3_short_period", 32, 200, 25),   # tax annealing, random placement, short order duration
    ("tax_us_federal", 32, 120, 20),    # multi-action agents, fixed schedule
    ("c5_small", 8, 150, 25),           # 32 agents, multi-action, K=50 book, sorted-gini branch
    ("c5_full", 6, 40, 20),             # BASELINE config 5 shape: 64 agents, 64x64, K=50 (2 agents per lane)
    ("wealth_redistribution", 32, 200, 25),  # WealthRedistribution as the last component, 9 agents (numpy pairwise sum)
    ("tax_single_planner", 32, 150, 25),  # single-action planner: one index over [NO-OP] ++ B x R rates
    ("uniform_halfwidth", 32, 150, 25),   # regen_halfwidth 1 / 2: window-count respawn thresholds
    ("quadrant", 16, 120, 30),            # uniform family with water lines, lognormal skills
    ("multi_zone", 16, 120, 30),
    ("split_layout", 4, 120, 30),         # (the 100000-row skill table per replica keeps this one small)
    ("full_obs_tax", 24, 100, 25),        # full_observability: whole-map agent observations
])
def test_cuda_batch_matches_oracle(cfg, E, steps, every):
    env = _make_env(cfg, E, seed=4000, auto_reset=False)
    orc, _ = _load_both(env)
    for e in range(E):
        bu.compare_env(orc, env.stepper, e, "reset", spatial=bool(env.spec["planner_gets_spatial_info"]))
    bu.run_pair(env, orc, steps, np.random.RandomState(123), check_every=every)


def test_cuda_full_size_c2_against_oracle_and_invariants():
    """BASELINE config 2 at full size (8192 env replicas on one GPU), 60 steps: every env is compared with the
    oracle on a cheap digest (state bytes that must be bit-exact), a sample of envs array-for-array, and
    size-independent invariants are checked on the whole batch."""
    import torch
    E = 8192
    env = _make_env("c1_tutorial", E, seed=1000, auto_reset=False)
    orc, host = _load_both(env)
    rng = np.random.RandomState(7)
    bu.run_pair(env, orc, 60, rng, check_every=60, check_envs=list(range(0, E, 257)))
    st = env.stepper
    loc = st.state_view("loc").cpu().numpy()
    inv = st.state_view("inv").cpu().numpy()
    esc = st.state_view("esc").cpu().numpy()
    n_orders = st.state_view("n_orders").cpu().numpy().astype(np.int64)
    bid_hist = st.state_view("bid_hist").cpu().numpy().astype(np.int64)
    ask_hist = st.state_view("ask_hist").cpu().numpy().astype(np.int64)
    mt_pos = st.state_view("mt_pos").cpu().numpy()
    for e in range(E):  # oracle digest for every env
        s = orc.state(e)
        assert np.array_equal(s["loc"], loc[e]) and np.array_equal(s["inv"], inv[e]), e
        assert int(s["mt_pos"][0]) == int(mt_pos[e]), e
    print("c2 full size, max relative float error over all replicas:", _batch_wide_float_error(env, orc, E))
    # invariants: order counts equal histogram mass; escrowed units equal open asks; agents on distinct cells
    assert np.array_equal(n_orders, bid_hist.sum(-1) + ask_hist.sum(-1))
    assert np.array_equal(esc.transpose(0, 2, 1), ask_hist.sum(-1))
    flat = loc[..., 0].astype(np.int64) * 25 + loc[..., 1]
    assert all(len(set(row)) == 4 for row in flat)
    assert (inv >= 0).all() and (esc >= 0).all()
    # determinism: a second run from the same snapshot gives bit-identical state records
    first = st.buf["state"].clone()
    env.stepper.load_state(host)
    rng = np.random.RandomState(7)
    from oracle.oracle import OracleBatch
    orc2 = OracleBatch(env.spec, 1)  # only used to advance the action RNG identically
    seg_a = bu.segments(env.spec, "a")
    for t in range(60):
        aa = bu.sample_from_masks(st.to_numpy(st.buf["mask_agent"]), seg_a, rng)
        env.step((aa, None))
    torch.cuda.synchronize()
    assert torch.equal(first, st.buf["state"])


@pytest.mark.parametrize("cfg,E,steps", [("c3_paper_tax", 8192, 30), ("c5_full", 2048, 12)],
                         ids=["c3_full_size", "c5_full_size"])
def test_cuda_full_size_c3_c5_against_oracle_and_invariants(cfg, E, steps):
    """BASELINE configs 3 and 5 at their per-GPU sizes (8 192 replicas of 10 agents on 40x40 with taxes; 2 048 replicas of
    64 agents on 64x64 with a 50-deep book): every replica digest-compared with the oracle, a sample array-for-array, and
    the size-independent invariants on the whole batch."""
    env = _make_env(cfg, E, seed=2000, auto_reset=False)
    if cfg == "c5_full":
        # the clumped 64x64 layout generator costs ~0.2 s per replica on the host: 64 distinct layouts / placements are
        # tiled over the batch and every replica gets its own numpy stream, so the trajectories diverge from step 1
        from oracle.oracle import OracleBatch
        small = _make_env(cfg, 64, seed=2000, auto_reset=False, stepper_factory=lambda *a, **k: None)
        h64 = small.host_reset_arrays()
        host = {k: np.concatenate([np.asarray(v)] * (E // 64)) for k, v in h64.items()}
        host["mt_key"] = np.stack([np.random.RandomState(70000 + e).get_state()[1] for e in range(E)]).astype(np.uint32)
        host["mt_pos"] = np.full(E, 624, np.int32)
        env.load_host_state(host)
        orc = OracleBatch(env.spec, E)
        for e in range(E):
            orc.load_env(e, {k: v[e] for k, v in host.items()})
    else:
        orc, host = _load_both(env)
    A, (H, W) = env.n_agents, env.world_size
    bu.run_pair(env, orc, steps, np.random.RandomState(3), check_every=steps, check_envs=list(range(0, E, 509)))
    st = env.stepper
    loc = st.state_view("loc").cpu().numpy()
    inv = st.state_view("inv").cpu().numpy()
    esc = st.state_view("esc").cpu().numpy()
    coin = st.state_view("coin").cpu().numpy()
    n_orders = st.state_view("n_orders").cpu().numpy().astype(np.int64)
    bid_hist = st.state_view("bid_hist").cpu().numpy().astype(np.int64)
    ask_hist = st.state_view("ask_hist").cpu().numpy().astype(np.int64)
    mt_pos = st.state_view("mt_pos").cpu().numpy()
    for e in range(E):  # oracle digest for every replica
        s = orc.state(e)
        assert np.array_equal(s["loc"], loc[e]) and np.array_equal(s["inv"], inv[e]), e
        assert int(s["mt_pos"][0]) == int(mt_pos[e]), e
    print(cfg, "full size, max relative float error over all replicas:", _batch_wide_float_error(env, orc, E))
    assert np.array_equal(n_orders, bid_hist.sum(-1) + ask_hist.sum(-1))          # order counts = histogram mass
    assert np.array_equal(esc.transpose(0, 2, 1), ask_hist.sum(-1))               # escrowed units = open asks
    assert n_orders.max() <= env.spec["max_num_orders"]
    flat = loc[..., 0].astype(np.int64) * W + loc[..., 1]
    assert all(len(set(row)) == A for row in flat)                                # agents on distinct cells
    assert (loc >= 0).all() and (loc[..., 0] < H).all() and (loc[..., 1] < W).all()
    assert (inv >= 0).all() and (esc >= 0).all() and (coin > -1e-9).all()



def _batch_wide_float_error(env, orc, E, rtol=1e-6):
    """Max relative error of the float64 state (coin, escrowed coin, labor) and of the last step's rewards over EVERY
    replica of the batch against the oracle - the north star's "within 1e-6 relative for coin/utility floats"."""
    st = env.stepper
    dev = {k: st.state_view(k).cpu().numpy() for k in ("coin", "esc_coin", "labor")}
    rew = st.to_numpy(st.buf["reward"])
    worst = {}
    for e in range(E):
        s, o = orc.state(e), orc.obs(e)
        for k, got in list((k, dev[k][e]) for k in dev) + [("rew", rew[e])]:
            want = np.asarray(o["rew"] if k == "rew" else s[k], np.float64).reshape(np.asarray(got).shape)
            err = float(np.max(np.abs(want - got) / np.maximum(np.abs(want), 1.0)))   # relative, absolute below 1
            worst[k] = max(worst.get(k, 0.0), err)
    assert all(v <= rtol for v in worst.values()), worst
    return worst


def test_auto_reset_restores_snapshot_and_continues_stream():
    """auto_reset=1: an env that reaches episode_length is restored from its load-time snapshot inside the same
    step (WarpDrive save_copy_and_apply_at_reset semantics); the numpy-legacy stream carries on."""
    from oracle.oracle import OracleBatch
    E, T = 16, 12
    env = _make_env("c1_tutorial", E, seed=77, auto_reset=True, episode_length=T, device_reset="snapshot")
    orc, host = _load_both(env)
    rng = np.random.RandomState(5)
    bu.run_pair(env, orc, T - 1, rng, check_every=T - 1)
    # terminal step: rewards/done come from the finished episode, state+obs are those of the fresh episode
    st = env.stepper
    seg_a = bu.segments(env.spec, "a")
    aa = bu.sample_from_masks(st.to_numpy(st.buf["mask_agent"]), seg_a, rng)
    env.step((aa, None))
    orc.step(aa, None)
    done = st.to_numpy(st.buf["done"])
    assert done.all()
    rew = st.to_numpy(st.buf["reward"])
    fresh = OracleBatch(env.spec, E)
    for e in range(E):
        o = orc.obs(e)
        assert np.allclose(o["rew"], rew[e], rtol=1e-6, atol=1e-9)
        s_end = orc.state(e)
        snap = {k: v[e] for k, v in host.items()}
        snap["mt_key"], snap["mt_pos"] = s_end["mt_key"], int(s_end["mt_pos"][0])
        snap["completions"] = 1
        fresh.load_env(e, snap)
        ps = st.read_state(e)
        assert int(ps["t"][0]) == 0 and int(ps["completions"][0]) == 1
    for e in range(E):
        bu.compare_env(fresh, st, e, "after auto-reset", skip=("rew", "done"))  # those belong to the finished episode
    bu.run_pair(env, fresh, 5, rng, check_every=5)  # and the new episode keeps tracking the oracle


def test_public_api_reset_step_shapes_on_device():
    import torch
    env = _make_env("c1_tutorial", 5, seed=3)
    obs = env.reset()
    assert obs["0"]["world-map"].shape == (5, 7, 11, 11) and obs["0"]["world-map"].is_cuda
    assert obs["p"]["world-map"].shape == (5, 6, 25, 25)
    assert obs["0"]["action_mask"].shape == (5, 50) and obs["p"]["action_mask"].shape == (5, 1)
    o2, rew, done, info = env.step({"0": torch.full((5,), 46, dtype=torch.int32)})
    assert rew["p"].shape == (5,) and done["__all__"].shape == (5,)
    assert float(obs["0"]["time"][0]) == pytest.approx(1 / 1000)
    coin = env.stepper.state_view("coin")
    assert coin.shape == (5, 4) and torch.all(coin == 10.0)
