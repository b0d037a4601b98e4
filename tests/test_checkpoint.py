"""Checkpoints of a batched env: `env.state_dict()` / `env.load_state_dict(sd)` (aie_get_counters / aie_set_counters and
their COVID-19 twins), and `MultiAgentDictEnv.save_game_object` / `load_game_object`.

Twin contract: env A steps k steps and takes its state_dict; env B, made with the same configuration but other seeds,
loads it after a torch.save / torch.load round trip; then both take the same m steps with the same actions (the policy
sampler under one seed, the random sampler, or the fused random policy) and after every step every buffer matches byte
for byte (final observations on the rows whose done flag is set), as do the metrics, the dense logs and the samplers'
draws and log-probabilities.  The CPU tests run the host emulation of the device source (tests/emu), the `-m gpu` tests
the CUDA kernels at workload sizes.
"""
import ctypes as C

import numpy as np
import pytest
import torch

from ai_economist_b200 import _abi, foundation
from ai_economist_b200.adapters import MultiAgentDictEnv
from oracle import configs
from tests.emu.emu_stepper import emu_factory, emu_lib
from tests.test_covid_metrics import emu as covid_emu

RATE = "VaccinationCampaign-next_vaccination_rate"
AIE_EINVAL = -1   # include/aie_b200.h


# ------------------------------------------------------------------------------------------------ helpers
def _cfg(cfg, **over):
    kw = dict(configs.CONFIGS[cfg] if cfg in configs.CONFIGS else configs.EDGE_CONFIGS[cfg])
    name = kw.pop("scenario_name")
    kw["components"] = [tuple(c) for c in kw["components"]]
    kw.update(over)
    return name, kw


def _tax(kw, **tax_over):
    """kw with its PeriodicBracketTax's kwargs updated."""
    comps = []
    for n, ckw in kw["components"]:
        comps.append((n, dict(ckw, **tax_over) if n == "PeriodicBracketTax" else ckw))
    return dict(kw, components=comps)


ONE_STEP_KW = dict(components=[("SimpleLabor", dict(mask_first_step=True, payment_max_skill_multiplier=3)),
                               ("PeriodicBracketTax", dict(bracket_spacing="us-federal", period=2, tax_model="model_wrapper",
                                                           rate_disc=0.05))],
                   n_agents=6, world_size=[1, 1], episode_length=3, planner_reward_type="coin_eq_times_productivity",
                   agent_reward_type="isoelastic_coin_minus_labor", labor_cost=0.02)


def _make_gtb(name, kw, E, seed0, cuda=False, **extra):
    dev = dict(device="cuda:0") if cuda else dict(stepper_factory=emu_factory)
    kw = dict(kw)
    kw.pop("seed", None)
    return foundation.make_env_instance(name, n_envs=E, seeds=[seed0 + 13 * e for e in range(E)], **dev, **extra, **kw)


def _bytes(x):
    return np.ascontiguousarray(x).view(np.uint8).reshape(-1)


def _same(a, b, what):
    assert tuple(a.shape) == tuple(b.shape) and a.dtype == b.dtype, what
    if isinstance(a, np.ndarray):
        assert np.array_equal(_bytes(a), _bytes(b)), what
    else:   # on the device: the rollout tensors at workload sizes are gigabytes
        u = lambda x: x.detach().contiguous().view(torch.uint8)
        assert torch.equal(u(a), u(b)), what


def _rows(x, mask):
    return x[mask] if isinstance(x, np.ndarray) else x[torch.as_tensor(mask, device=x.device)]


def _np(x):
    return x if isinstance(x, np.ndarray) else x.detach().cpu().numpy()


def _save_load(sd, tmp_path):
    p = tmp_path / "env.pt"
    torch.save(sd, p)
    return torch.load(p, weights_only=False)


def compare_gtb(A, B, label):
    """Every buffer of the two envs' steppers (final observations on done rows only), the rollout slots when bound,
    the metrics, completions, dense logs and library counters."""
    sa, sb = A.stepper, B.stepper
    assert set(sa.buf) == set(sb.buf)
    done = _np(sa.buf["done"]) != 0
    for k in sa.buf:
        if k.startswith("final_"):
            _same(_rows(sa.buf[k], done), _rows(sb.buf[k], done), "%s: %s (done rows)" % (label, k))
        else:
            _same(sa.buf[k], sb.buf[k], "%s: %s" % (label, k))
    if A.rollout is not None:
        for k in A.rollout.buf:
            _same(A.rollout.buf[k], B.rollout.buf[k], "%s: rollout %s" % (label, k))
    assert sa.get_counters() == sb.get_counters(), label
    assert np.array_equal(A.completions(), B.completions()), label
    assert repr(A.metrics) == repr(B.metrics), label
    assert repr(A.previous_episode_metrics) == repr(B.previous_episode_metrics), label
    _same(A.metrics_tensor(), B.metrics_tensor(), "%s: metrics_tensor" % label)
    if "episode_final" in sa.buf:
        _same(A.previous_episode_metrics_tensor(), B.previous_episode_metrics_tensor(), "%s: previous metrics" % label)
    assert repr(A.dense_log) == repr(B.dense_log), label
    assert repr(A.previous_episode_dense_log) == repr(B.previous_episode_dense_log), label


def _logits(env, rng):
    sa, sp, _, _ = env.stepper._policy_shapes()
    la = rng.standard_normal(sa).astype(np.float32)
    lp = rng.standard_normal(sp).astype(np.float32) if sp is not None else None
    buf = env.stepper.buf["done"]
    if not isinstance(buf, np.ndarray):
        la = torch.as_tensor(la, device=buf.device)
        lp = torch.as_tensor(lp, device=buf.device) if lp is not None else None
    return la, lp


def _act(envs, t, rng, mode):
    """The same actions for every env of `envs` at step t: the policy sampler (one logits draw, one seed), the random
    sampler, both in turn, or nothing (the fused random policy already wrote them).  Returns the log-probabilities."""
    if mode == "fused":
        return None
    if mode == "mixed" and t % 3 == 2:
        for env in envs:
            env.stepper.sample_random_actions(seed=91)
        return None
    la, lp = _logits(envs[0], rng)
    out = [env.sample_actions(la, lp, seed=4242) for env in envs]
    for o in out[1:]:
        for x, y in zip(out[0], o):
            if x is not None:
                _same(x, y, "step %d: log-probabilities" % t)
    return out


def run_gtb_twins(name, kw, E, k, m, tmp_path, mode="mixed", cuda=False, reset_after=True, **extra):
    A = _make_gtb(name, kw, E, 1000, cuda=cuda, **extra)
    B = _make_gtb(name, kw, E, 7000, cuda=cuda, **extra)
    A.reset()
    if mode == "fused":
        A.stepper.set_fused_policy(77)
    rng = np.random.RandomState(5)
    for t in range(k):
        _act([A], t, rng, mode)
        A.step(A.action_buffers)
    sd = _save_load(A.state_dict(), tmp_path)
    B.load_state_dict(sd)
    compare_gtb(A, B, "after load")
    ends = 0
    for t in range(m):
        _act([A, B], t, rng, mode)
        A.step(A.action_buffers)
        B.step(B.action_buffers)
        ends += int(_np(A.done["__all__"]).sum())
        compare_gtb(A, B, "step %d after load" % t)
    if reset_after:   # an explicit reset continues every replica's stream, the completion counts and the Saez state
        A.reset()
        B.reset()
        compare_gtb(A, B, "reset after load")
        _act([A, B], 0, rng, "policy")
        A.step(A.action_buffers)
        B.step(B.action_buffers)
        compare_gtb(A, B, "step after reset")
    return A, B, ends


# ------------------------------------------------------------------------------------------------ 1. twins (emulation)
TWINS = {
    # layout_from_file with the planner-driven (model_wrapper) tax: an episode end at 30, tax periods of 10
    "model_wrapper": lambda: _cfg("c3_reset", episode_length=30),
    "us_federal_annealed": lambda: _cfg("us_federal_annealed_reset"),
    "fixed_rates_annealed": lambda: (lambda n, kw: (n, _tax(dict(kw, episode_length=20), tax_annealing_schedule=[-2, 0.25])))(
        *_cfg("eta_high_fixed_rates")),
    "energy_auto": lambda: _cfg("c1_reset", energy_warmup_method="auto", energy_warmup_constant=10),
    "energy_decay": lambda: _cfg("c1_reset", energy_warmup_method="decay", energy_warmup_constant=10),
    "uniform": lambda: _cfg("uniform_reset"),
    "quadrant": lambda: _cfg("quadrant_reset"),
    "multi_zone": lambda: _cfg("multi_zone_reset"),
    "split_layout": lambda: _cfg("split_reset"),
    "lognormal": lambda: _cfg("lognormal_reset"),
    "one_step": lambda: ("one-step-economy", dict(ONE_STEP_KW)),
}


@pytest.mark.parametrize("case", sorted(TWINS))
def test_twins_resume_bit_for_bit(case, tmp_path):
    name, kw = TWINS[case]()
    T = kw["episode_length"]
    k = T + T // 2 + 1 if T > 3 else 4   # past one episode end; m spans the next one
    _, _, ends = run_gtb_twins(name, kw, 3, k, T + 2, tmp_path, final_obs=True)
    assert ends >= 3


@pytest.mark.parametrize("case", ["bf16_final_dense", "fused"])
def test_twins_bfloat16_final_obs_dense_log_and_fused_policy(case, tmp_path):
    name, kw = _cfg("c3_reset", episode_length=24)
    if case == "bf16_final_dense":
        A, B, ends = run_gtb_twins(name, kw, 2, 30, 26, tmp_path, obs_dtype=torch.bfloat16, final_obs=True,
                                   dense_log_frequency=1)
        assert B.previous_episode_dense_log["states"] and B.dense_log["actions"]
    else:
        A, B, ends = run_gtb_twins(name, kw, 2, 17, 26, tmp_path, mode="fused", final_obs=True)
        assert A.stepper.get_counters()["fused_policy_on"] == 1
    assert ends >= 2


@pytest.mark.parametrize("E,annealed", [(2, False), (2, True), (65, False)])
def test_twins_saez_estimator_resumes(E, annealed, tmp_path):
    """SaezLoop (<= 64 replicas) and SaezBatch (> 64): the checkpoint is taken once the 500-sample buffers are full and
    the formula has set rates, so the smoothed elasticities, running averages and ring positions all matter."""
    name, kw = _cfg("saez_annealed_reset" if annealed else "saez_reset", episode_length=30)
    kw = _tax(kw, period=1)   # 10 samples per step: the buffers fill in 50 steps
    A, B, ends = run_gtb_twins(name, kw, E, 56, 10, tmp_path, final_obs=True)
    st = B._saez.state_dict()
    assert st["kind"] == ("batch" if E > 64 else "loop")
    assert ends == E
    assert all(v is not None for v in B._saez.elas_at_episode_end)


def test_twins_bound_rollout_saved_at_slot_zero(tmp_path):
    """Save at slot 0 of a bound rollout (after restart_rollout), load into a bound env: the stored slots of the next
    two rollouts match."""
    name, kw = _cfg("c1_reset")
    E, T = 3, 10
    A = _make_gtb(name, kw, E, 1000, final_obs=True)
    B = _make_gtb(name, kw, E, 7000, final_obs=True)
    ra, rb = A.bind_rollout(T, final_obs=True), B.bind_rollout(T, final_obs=True)
    A.reset()
    rng = np.random.RandomState(3)
    for t in range(T):
        _act([A], t, rng, "mixed")
        A.step(A.action_buffers)
    A.restart_rollout()
    B.load_state_dict(_save_load(A.state_dict(), tmp_path))
    for k in ra.obs_names:
        _same(ra.buf[k][0], rb.buf[k][0], "slot 0 of %s" % k)
    for rnd in range(2):
        if rnd:
            A.restart_rollout()
            B.restart_rollout()
        for t in range(T):
            _act([A, B], t, rng, "mixed")
            A.step(A.action_buffers)
            B.step(B.action_buffers)
        for k in ra.buf:
            if not k.startswith("final_"):
                _same(ra.buf[k], rb.buf[k], "round %d: rollout %s" % (rnd, k))
        for kk in range(ra.K):   # final slot kk of the replicas that ended kk + 1 times or more
            hit = _np(ra.buf["done"]).sum(0) > kk
            for k in ra.obs_names:
                _same(_rows(ra.buf["final_" + k][kk], hit), _rows(rb.buf["final_" + k][kk], hit), "final %s" % k)
        assert repr(A.metrics) == repr(B.metrics)


# ------------------------------------------------------------------------------------------------ 2. COVID-19 twins
def _covid(E, seed_unused, cuda=False, **kw):
    from ai_economist_b200.workloads import COVID_KWARGS, covid_reference_config
    cfg = covid_reference_config(dict(COVID_KWARGS, episode_length=kw.pop("episode_length", 12),
                                      start_date="2020-12-01", delivery_interval=7,
                                      vaccine_delivery_start_date="2020-12-05"))
    for c in cfg["components"]:
        if "VaccinationCampaign" in c:
            c["VaccinationCampaign"]["observe_rate"] = True
    dev = dict(device="cuda:0") if cuda else dict(stepper_factory=lambda p, n, ar, **fkw: covid_emu(p, n, auto_reset=ar, **fkw))
    return foundation.make_env_instance(cfg.pop("scenario_name"), n_envs=E, **dev, **cfg, **kw)


def compare_covid(A, B, label):
    sa, sb = A.stepper, B.stepper
    assert set(sa.buf) == set(sb.buf)
    for k in sa.buf:
        _same(sa.buf[k], sb.buf[k], "%s: %s" % (label, k))   # every replica ends on the same step: final rows all equal
    if A.rollout is not None:
        for k in A.rollout.buf:
            _same(A.rollout.buf[k], B.rollout.buf[k], "%s: rollout %s" % (label, k))
    for g in ("a", "p"):
        _same(A.obs[g][RATE], B.obs[g][RATE], "%s: rate %s" % (label, g))
        if A.final_obs is not None:
            _same(A.final_obs[g][RATE], B.final_obs[g][RATE], "%s: final rate %s" % (label, g))
    assert sa.get_counters() == sb.get_counters(), label
    if A._episode_metrics:
        _same(A.metrics_tensor(), B.metrics_tensor(), "%s: metrics_tensor" % label)
        assert repr(A.previous_episode_metrics) == repr(B.previous_episode_metrics), label
        if sa.has_previous_episode():
            _same(A.previous_episode_metrics_tensor(), B.previous_episode_metrics_tensor(), "%s: previous" % label)


def run_covid_twins(E, k, m, tmp_path, cuda=False, **kw):
    A, B = _covid(E, 1, cuda=cuda, **kw), _covid(E, 2, cuda=cuda, **kw)
    A.reset()
    rng = np.random.RandomState(9)

    def act(envs, t):
        if t % 4 == 3:
            for env in envs:
                env.stepper.sample_random_actions(seed=33)
            return
        sa, sp, _, _ = envs[0].stepper._policy_shapes()
        la, lp = rng.standard_normal(sa).astype(np.float32), rng.standard_normal(sp).astype(np.float32)
        if cuda:
            la, lp = torch.as_tensor(la, device="cuda:0"), torch.as_tensor(lp, device="cuda:0")
        out = [env.sample_actions(la, lp, seed=808) for env in envs]
        for o in out[1:]:
            for x, y in zip(out[0], o):
                _same(x, y, "step %d: log-probabilities" % t)

    for t in range(k):
        act([A], t)
        A.step(A.action_buffers)
    B.load_state_dict(_save_load(A.state_dict(), tmp_path))
    compare_covid(A, B, "after load")
    for t in range(m):
        act([A, B], t)
        A.step(A.action_buffers)
        B.step(B.action_buffers)
        compare_covid(A, B, "step %d after load" % t)
    return A, B


@pytest.mark.parametrize("obs_dtype", [None, torch.bfloat16])
def test_covid_twins_resume_bit_for_bit(obs_dtype, tmp_path):
    A, B = run_covid_twins(3, 17, 15, tmp_path, episode_metrics=True, final_obs=True, obs_dtype=obs_dtype)
    assert B.previous_episode_metrics is not None and B.stepper.get_counters()["policy_calls"] > 0


def test_covid_twins_bound_rollout_at_slot_zero(tmp_path):
    E, T = 2, 8
    A, B = _covid(E, 1, episode_length=6, final_obs=True), _covid(E, 2, episode_length=6, final_obs=True)
    ra, rb = A.bind_rollout(T, final_obs=True), B.bind_rollout(T, final_obs=True)
    A.reset()
    for t in range(T):
        A.stepper.sample_random_actions(seed=5)
        A.step(A.action_buffers)
    A.restart_rollout()
    B.load_state_dict(_save_load(A.state_dict(), tmp_path))
    for rnd in range(2):
        if rnd:
            A.restart_rollout()
            B.restart_rollout()
        for t in range(T):
            for env in (A, B):
                env.stepper.sample_random_actions(seed=5)
                env.step(env.action_buffers)
        for k in ra.buf:
            _same(ra.buf[k], rb.buf[k], "round %d: rollout %s" % (rnd, k))


# ------------------------------------------------------------------------------------------------ 3. refusals
def test_refusals_name_the_field(tmp_path):
    name, kw = _cfg("c1_reset")
    A = _make_gtb(name, kw, 2, 1000)
    with pytest.raises(ValueError, match="first reset"):
        A.state_dict()
    A.reset()
    A.step(None)
    sd = A.state_dict()
    for other, field in [(_make_gtb(name, kw, 3, 1000), "n_envs"),
                         (_make_gtb(name, kw, 2, 1000, obs_dtype=torch.bfloat16), "obs_dtype"),
                         (_make_gtb(name, dict(kw, episode_length=26), 2, 1000), "spec"),
                         (_make_gtb(name, kw, 2, 1000, final_obs=True), "final_obs"),
                         (_make_gtb(name, kw, 2, 1000, auto_reset=False), "auto_reset"),
                         (_make_gtb(name, kw, 2, 1000, dense_log_frequency=2), "dense_log"),
                         (_make_gtb(*_cfg("uniform_reset"), 2, 1000), "scenario")]:
        with pytest.raises(ValueError, match=field):
            other.load_state_dict(sd)
    for key, val, field in [("format_version", 99, "format_version"), ("config", dict(sd["config"], abi_version=5),
                                                                        "abi_version")]:
        with pytest.raises(ValueError, match=field):
            _make_gtb(name, kw, 2, 1000).load_state_dict(dict(sd, **{key: val}))
    cv = _covid(2, 1, episode_metrics=True)
    cv.reset()
    csd = cv.state_dict()
    with pytest.raises(ValueError, match="episode_metrics"):
        _covid(2, 1).load_state_dict(csd)
    with pytest.raises(ValueError, match="n_envs"):
        _covid(3, 1, episode_metrics=True).load_state_dict(csd)
    with pytest.raises(ValueError, match="first reset"):
        _covid(2, 1).state_dict()


def test_refusals_mid_rollout():
    name, kw = _cfg("c1_reset")
    A, B = _make_gtb(name, kw, 2, 1000), _make_gtb(name, kw, 2, 7000)
    A.reset()
    sd = A.state_dict()
    A.bind_rollout(4)
    B.bind_rollout(4)
    B.reset()
    for env in (A, B):
        env.step(None)
    with pytest.raises(ValueError, match="slot 0"):
        A.state_dict()
    with pytest.raises(ValueError, match="slot 0"):
        B.load_state_dict(sd)
    # the library refuses as well
    for fn in (A.stepper.get_counters, lambda: A.stepper.set_counters(sd["counters"])):
        with pytest.raises(_abi.AieError, match="aie error -3"):
            fn()
    cv = _covid(2, 1)
    cv.bind_rollout(3)
    cv.reset()
    cv.step(None)
    with pytest.raises(ValueError, match="slot 0"):
        cv.state_dict()
    with pytest.raises(_abi.AieError, match="aie error -3"):
        cv.stepper.get_counters()


def test_counter_calls_with_null_give_einval():
    L = emu_lib()
    name, kw = _cfg("c1_reset")
    env = _make_gtb(name, kw, 2, 1000)
    h = env.stepper._h
    c = _abi.AieCounters()
    assert L.aie_get_counters(None, C.byref(c)) == AIE_EINVAL
    assert L.aie_get_counters(h, None) == AIE_EINVAL
    assert L.aie_set_counters(None, C.byref(c)) == AIE_EINVAL
    assert L.aie_set_counters(h, None) == AIE_EINVAL
    c.fused_policy_key, c.fused_policy_on = 5, 0   # on / off must agree with the key
    assert L.aie_set_counters(h, C.byref(c)) == AIE_EINVAL
    cv = _covid(2, 1)
    cc = _abi.AieCovidCounters()
    assert L.aie_covid_get_counters(None, C.byref(cc)) == AIE_EINVAL
    assert L.aie_covid_get_counters(cv.stepper._h, None) == AIE_EINVAL
    assert L.aie_covid_set_counters(None, C.byref(cc)) == AIE_EINVAL
    assert L.aie_covid_set_counters(cv.stepper._h, None) == AIE_EINVAL
    cc.t = -1
    assert L.aie_covid_set_counters(cv.stepper._h, C.byref(cc)) == AIE_EINVAL


# ------------------------------------------------------------------------------------------------ 4. adapter
def test_multi_agent_dict_env_save_and_load_game_object(tmp_path):
    name, kw = _cfg("c1_reset")
    A = MultiAgentDictEnv(_make_gtb(name, kw, 2, 1000), e=1)
    B = MultiAgentDictEnv(_make_gtb(name, kw, 2, 7000), e=1)
    rng = np.random.RandomState(2)
    for _ in range(30):
        A.step({str(i): int(rng.randint(0, 5)) for i in range(4)})
    A.save_game_object(str(tmp_path))
    B.load_game_object(str(tmp_path))
    for t in range(30):
        acts = {str(i): int(rng.randint(0, 5)) for i in range(4)}
        oa, ra, da, _ = A.step(acts)
        ob, rb, db, _ = B.step(acts)
        assert repr(ra) == repr(rb) and da == db
        for ag in oa:
            for key in oa[ag]:
                assert np.array_equal(np.asarray(oa[ag][key]), np.asarray(ob[ag][key])), (t, ag, key)
    assert repr(A.summary) == repr(B.summary)


# ------------------------------------------------------------------------------------------------ 5. GPU twins
def _gpu_rollout_twins(name, kw, E, T, tmp_path, final=True, **extra):
    """Two rollouts of T steps on A, save at slot 0, two more rollouts on A and on B (loaded), with the policy sampler
    and compute_advantages over each: every slot, every advantage and every record match."""
    A = _make_gtb(name, kw, E, 1000, cuda=True, final_obs=final, **extra)
    B = _make_gtb(name, kw, E, 7000, cuda=True, final_obs=final, **extra)
    ra, rb = A.bind_rollout(T, final_obs=final), B.bind_rollout(T, final_obs=final)
    A.reset()
    g = torch.Generator(device="cuda:0").manual_seed(1)
    sa, sp, _, _ = A.stepper._policy_shapes()

    def rollout(envs, rnd):
        for env in envs:
            if rnd:
                env.restart_rollout()
        for t in range(T):
            la = torch.randn(sa, device="cuda:0", generator=g)
            lp = torch.randn(sp, device="cuda:0", generator=g) if sp is not None else None
            out = [env.sample_actions(la, lp, seed=17) for env in envs]
            for o in out[1:]:
                for x, y in zip(out[0], o):
                    if x is not None:
                        _same(x, y, "round %d step %d: log-probabilities" % (rnd, t))
            for env in envs:
                env.step(env.action_buffers)
        advs = []
        for env in envs:
            r = env.rollout
            A_ = env.n_agents
            v = (torch.zeros((T, E, A_), device="cuda:0"), torch.zeros((T, E), device="cuda:0"))
            lv = (torch.zeros((E, A_), device="cuda:0"), torch.zeros(E, device="cuda:0"))
            fv = (torch.ones((r.K, E, A_), device="cuda:0"), torch.ones((r.K, E), device="cuda:0")) if final else None
            advs.append(env.compute_advantages(r.buf["reward"], v, r.buf["done"], lv, fv, gamma=0.99, lam=0.95,
                                               per_episode_end=final))
        for o in advs[1:]:
            for x, y in zip(advs[0], o):
                _same(x, y, "round %d: advantages" % rnd)

    for rnd in range(2):
        rollout([A], rnd)
    A.restart_rollout()
    B.load_state_dict(_save_load(A.state_dict(), tmp_path))
    for rnd in range(2):
        rollout([A, B], rnd + 1 if rnd else 0)
        for k in ra.buf:
            if not k.startswith("final_"):
                _same(ra.buf[k], rb.buf[k], "round %d: rollout %s" % (rnd, k))
        for kk in range(ra.K if final else 0):
            hit = (ra.buf["done"].sum(0) > kk).cpu().numpy()
            for k in ra.obs_names:
                _same(_rows(ra.buf["final_" + k][kk], hit), _rows(rb.buf["final_" + k][kk], hit), "final %s" % k)
        for k in ("state", "state0", "episode_final"):
            _same(A.stepper.buf[k], B.stepper.buf[k], "round %d: %s" % (rnd, k))
        _same(A.metrics_tensor(), B.metrics_tensor(), "round %d: metrics_tensor" % rnd)
    for env in (A, B):   # the counters are read at slot 0
        env.restart_rollout()
    assert A.stepper.get_counters() == B.stepper.get_counters()


GPU_CASES = {
    # (config, overrides, n_envs, rollout length)
    # episodes end at steps 20 and 40 (c5: every 10 steps) of the 32 steps after the save at step 16
    "c2": ("c1_tutorial", dict(episode_length=20), 8192, 8),
    "c3": ("c3_paper_tax", dict(episode_length=20), 8192, 8),
    "c5_snapshot": ("c5_full", dict(episode_length=10, device_reset="snapshot"), 2048, 8),
}


@pytest.mark.gpu
@pytest.mark.parametrize("case", sorted(GPU_CASES))
def test_gpu_twins_at_workload_sizes(case, tmp_path):
    cfg, over, E, T = GPU_CASES[case]
    name, kw = _cfg(cfg, **over)
    _gpu_rollout_twins(name, kw, E, T, tmp_path)


@pytest.mark.gpu
def test_gpu_twins_saez_batch(tmp_path):
    name, kw = _cfg("saez_annealed_reset", episode_length=30)
    kw = _tax(kw, period=1)
    A, B, ends = run_gtb_twins(name, kw, 128, 56, 10, tmp_path, cuda=True, final_obs=True)
    assert B._saez.state_dict()["kind"] == "batch" and ends == 128


@pytest.mark.gpu
def test_gpu_twins_gtb_plain_steps(tmp_path):
    """Without a rollout: final observations, the random sampler and an explicit reset after the load (c3-like)."""
    name, kw = _cfg("c3_reset", episode_length=30)
    run_gtb_twins(name, kw, 1024, 40, 32, tmp_path, cuda=True, final_obs=True)


@pytest.mark.gpu
def test_gpu_covid_twins_c4(tmp_path):
    """c4 at 4 096 replicas: two rollouts each side of the save, with metrics, final observations and bfloat16."""
    E, T = 4096, 10
    for obs_dtype in (None, torch.bfloat16):
        A = _covid(E, 1, cuda=True, episode_length=15, episode_metrics=True, final_obs=True, obs_dtype=obs_dtype)
        B = _covid(E, 2, cuda=True, episode_length=15, episode_metrics=True, final_obs=True, obs_dtype=obs_dtype)
        ra, rb = A.bind_rollout(T, final_obs=True), B.bind_rollout(T, final_obs=True)
        A.reset()
        g = torch.Generator(device="cuda:0").manual_seed(3)
        sa, sp, _, _ = A.stepper._policy_shapes()

        def rollout(envs, rnd):
            for env in envs:
                if rnd:
                    env.restart_rollout()
            for t in range(T):
                la, lp = torch.randn(sa, device="cuda:0", generator=g), torch.randn(sp, device="cuda:0", generator=g)
                out = [env.sample_actions(la, lp, seed=29) for env in envs]
                for o in out[1:]:
                    for x, y in zip(out[0], o):
                        _same(x, y, "log-probabilities")
                for env in envs:
                    env.step(env.action_buffers)
            advs = []
            for env in envs:
                r, S = env.rollout, env.n_agents
                v = (torch.zeros((T, E, S), device="cuda:0"), torch.zeros((T, E), device="cuda:0"))
                lv = (torch.zeros((E, S), device="cuda:0"), torch.zeros(E, device="cuda:0"))
                fv = (torch.ones((r.K, E, S), device="cuda:0"), torch.ones((r.K, E), device="cuda:0"))
                advs.append(env.compute_advantages((r.buf["reward_agent"], r.buf["reward_planner"]), v, r.buf["done"],
                                                   lv, fv, gamma=0.99, lam=0.95, per_episode_end=True))
            for o in advs[1:]:
                for x, y in zip(advs[0], o):
                    _same(x, y, "advantages")

        for rnd in range(2):
            rollout([A], rnd)
        A.restart_rollout()
        B.load_state_dict(_save_load(A.state_dict(), tmp_path))
        for rnd in range(2):
            rollout([A, B], 1 if rnd else 0)
            for k in ra.buf:
                _same(ra.buf[k], rb.buf[k], "round %d: rollout %s" % (rnd, k))
        for env in (A, B):   # the counters are read at slot 0
            env.restart_rollout()
        compare_covid(A, B, "after two rollouts")
