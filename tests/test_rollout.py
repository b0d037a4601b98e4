"""Rollouts stored in place (`env.bind_rollout(T, final_obs=...)`, aie_bind_rollout / aie_rollout_restart /
aie_compute_advantages_k).

Contract: a bound env writes, slot by slot, exactly the bytes a twin running the copy loop of INTEGRATION §7 copies out
of its own buffers after every step (observations and masks into slot t before step t and slot T after the last one,
actions and log-probabilities of the samplers, rewards and done), and final slot (k, e) holds the twin's env.final_obs
row e at the step that ended replica e's k-th episode of the rollout.  Advantages from the bound rollout's [K, ...]
final values have the bits of today's call over the twin's [T, ...] buffers.  The CPU tests run the host emulation of
the device source (tests/emu), the `-m gpu` tests the CUDA kernels.
"""
import ctypes as C

import numpy as np
import pytest
import torch

from ai_economist_b200 import _abi, foundation
from tests.test_advantages import gae_ref, same_bits
from tests.test_final_obs import _stagger
from tests.test_obs_bf16 import _cfg

OBS = _abi.OBS_NAMES


def _make(name, kw, E, factory, obs_dtype, **extra):
    dev = dict(stepper_factory=factory) if factory is not None else dict(device="cuda:0")
    seeds = [300 + 11 * e for e in range(E)]
    return foundation.make_env_instance(name, n_envs=E, seeds=seeds, obs_dtype=obs_dtype, final_obs=True, **dev,
                                        **extra, **kw)


def _np(x):
    return x if isinstance(x, np.ndarray) else x.detach().cpu().numpy()


def _snap(x):
    """A copy of a buffer on its own backend (the copy loop's torch.clone on CUDA)."""
    return np.array(x) if isinstance(x, np.ndarray) else x.clone()


def _same(a, b):
    """Byte-for-byte equality of two buffers of one backend."""
    if isinstance(a, np.ndarray):
        return np.array_equal(np.ascontiguousarray(a).view(np.uint8), np.ascontiguousarray(b).view(np.uint8))
    return a.shape == b.shape and torch.equal(a.contiguous().view(torch.uint8), b.contiguous().view(torch.uint8))


def _like(env, a):
    """a host array on the env's backend (numpy for the emulation, CUDA tensors otherwise)."""
    buf = env.stepper.buf["done"]
    return a if isinstance(buf, np.ndarray) else torch.as_tensor(a, device=buf.device)


def _start(env, E):
    env.reset()
    _stagger(env, E)
    env.stepper.observe()


def run_rollout_twins(name, kw, E, factory, obs_dtype, T, rounds, gamma=0.97, lam=0.9):
    """B binds a rollout of T steps with final slots; Y copies its outputs after every step (INTEGRATION §7).  Both draw
    actions with the policy sampler from the same logits.  Returns the number of episode ends seen."""
    B, Y = _make(name, kw, E, factory, obs_dtype), _make(name, kw, E, factory, obs_dtype)
    r = B.bind_rollout(T, final_obs=True)
    assert r.K == -(-T // B.episode_length)
    for env in (B, Y):
        _start(env, E)
    sa, sp, na, npl = B.stepper._policy_shapes()
    rng = np.random.RandomState(7)
    lp_a = np.zeros((T,) + na, np.float32)
    lp_p = np.zeros((T,) + npl, np.float32) if npl else None
    lp_b = (_like(B, lp_a.copy()), _like(B, lp_p.copy()) if npl else None)
    ends = 0
    for rnd in range(rounds):
        if rnd:
            B.restart_rollout()
            for k in OBS:
                if k in r.buf:
                    assert _same(r.buf[k][0], last_obs[k]), "round %d: slot 0 of %s" % (rnd, k)
        copies = {k: [] for k in list(OBS) + ["actions_agent", "actions_planner", "reward", "done", "lp_a", "lp_p"]}
        finals = []   # (t, e, {name: row bytes}) of the twin's final observations
        for t in range(T):
            assert B.stepper.rollout_slot == t
            for k in OBS:
                if k in r.buf:
                    assert B.obs_tensors[k] is r.obs_slots[t][k]
                    copies[k].append(_snap(Y.obs_tensors[k]))
            la = rng.standard_normal(sa).astype(np.float32)
            lpl = rng.standard_normal(sp).astype(np.float32) if sp else None
            ob = B.sample_actions(_like(B, la), _like(B, lpl) if sp else None, seed=5 + rnd,
                                  out=(lp_b[0][t], lp_b[1][t] if npl else None))
            oy = Y.sample_actions(_like(Y, la), _like(Y, lpl) if sp else None, seed=5 + rnd)
            copies["lp_a"].append(_np(oy[0]).copy())
            if npl:
                copies["lp_p"].append(_np(oy[1]).copy())
            ya, yp = Y.action_buffers
            copies["actions_agent"].append(_snap(ya))
            copies["actions_planner"].append(_snap(yp))
            B.step(B.action_buffers)
            Y.step(Y.action_buffers)
            assert B.done is r.done[t] and B.rew is r.rew[t]
            copies["reward"].append(_snap(Y.stepper.buf["reward"]))
            done = _np(Y.stepper.buf["done"]).copy()
            copies["done"].append(done)
            for e in np.nonzero(done)[0]:
                finals.append((t, e, {k: _snap(Y.stepper.buf["final_" + k][e:e + 1]) for k in OBS if k in r.buf}))
        last_obs = {k: _snap(Y.obs_tensors[k]) for k in OBS if k in r.buf}
        for k in OBS:
            if k in r.buf:
                for t in range(T):
                    assert _same(r.buf[k][t], copies[k][t]), "round %d slot %d: %s" % (rnd, t, k)
                assert _same(r.buf[k][T], last_obs[k]), "round %d slot T: %s" % (rnd, k)
        for k in ("actions_agent", "actions_planner", "reward"):
            if k == "actions_planner" and not npl:
                continue
            for t in range(T):
                assert _same(r.buf[k][t], copies[k][t]), "round %d slot %d: %s" % (rnd, t, k)
        assert np.array_equal(_np(r.buf["done"]), np.stack(copies["done"]))
        assert np.array_equal(_np(lp_b[0]).view(np.uint32), np.stack(copies["lp_a"]).view(np.uint32))
        if npl:
            assert np.array_equal(_np(lp_b[1]).view(np.uint32), np.stack(copies["lp_p"]).view(np.uint32))
        D = np.stack(copies["done"])
        for t, e, rows in finals:
            k = int(D[:t, e].sum())
            assert k < r.K
            for name_, row in rows.items():
                assert _same(r.buf["final_" + name_][k][e:e + 1], row), \
                    "round %d: final slot (%d, %d) of %s (step %d)" % (rnd, k, e, name_, t)
        ends += len(finals)
        check_advantages(B, Y, r, D, copies, rng, gamma, lam)
    return ends


def check_advantages(B, Y, r, D, copies, rng, gamma, lam):
    """compute_advantages over the bound rollout ([T, E, A+1] rewards, [K, ...] final values) against today's call on
    the twin's [T, ...] buffers and the float64 numpy restatement."""
    T, K = r.T, r.K
    E, A = B.n_envs, B.n_agents
    R = np.stack([_np(x) for x in copies["reward"]])
    V = (rng.standard_normal((T, E, A)).astype(np.float32), rng.standard_normal((T, E)).astype(np.float32))
    LV = (rng.standard_normal((E, A)).astype(np.float32), rng.standard_normal(E).astype(np.float32))
    FK = (rng.standard_normal((K, E, A)).astype(np.float32), rng.standard_normal((K, E)).astype(np.float32))
    FT = (np.full((T, E, A), np.nan, np.float32), np.full((T, E), np.nan, np.float32))   # unread rows: NaN
    for e in range(E):
        for k, t in enumerate(np.nonzero(D[:, e])[0]):
            FT[0][t, e], FT[1][t, e] = FK[0][k, e], FK[1][k, e]
    gB = lambda x: tuple(_like(B, a) for a in x)
    out_b = B.compute_advantages(r.buf["reward"], gB(V), r.buf["done"], gB(LV), gB(FK), gamma=gamma, lam=lam,
                                 per_episode_end=True)
    Rp = (np.ascontiguousarray(R[..., :A]), np.ascontiguousarray(R[..., A]))
    gY = lambda x: tuple(_like(Y, a) for a in x)
    out_y = Y.compute_advantages(gY(Rp), gY(V), _like(Y, np.ascontiguousarray(D)), gY(LV), gY(FT), gamma=gamma, lam=lam)
    for x, y in zip(out_b, out_y):
        assert same_bits(_np(x), _np(y))
    for g in range(2):
        adv, ret = gae_ref(Rp[g], V[g], D, LV[g], FT[g], gamma, lam)
        assert same_bits(_np(out_b[g]), adv) and same_bits(_np(out_b[2 + g]), ret)


CASES = [("c1_tutorial", dict(planner_gets_spatial_info=False)),   # c1-size map, spatial agents
         ("c3_short_period", {}),                                  # c3-like tax config
         ("c5_small", {})]                                         # multi-action agents


@pytest.mark.parametrize("obs_dtype", ["float32", "bfloat16"])
@pytest.mark.parametrize("T,rounds", [(5, 3), (16, 2)])   # K = 1 and K = 3 at episode_length 7
@pytest.mark.parametrize("cfg,over", CASES, ids=[c for c, _ in CASES])
def test_emulated_rollout_equals_the_copy_loop(cfg, over, T, rounds, obs_dtype):
    from tests.emu.emu_stepper import emu_factory
    name, kw = _cfg(cfg, episode_length=7, **over)
    assert run_rollout_twins(name, kw, 3, emu_factory, obs_dtype, T, rounds) >= 2 * 3


def _emu_env(final_obs=True, **extra):
    from tests.emu.emu_stepper import emu_factory
    name, kw = _cfg("c3_short_period", episode_length=7)
    return foundation.make_env_instance(name, n_envs=2, seeds=[1, 2], stepper_factory=emu_factory, final_obs=final_obs,
                                        **extra, **kw)


def _rollout_struct(st, r, **over):
    q = _abi.AieRollout()
    q.T = r.T
    q.obs = st._obs_buffers({k: r.buf[k] for k in r.obs_names})
    q.actions_agent, q.reward, q.done = st._ptr(r.buf["actions_agent"]), st._ptr(r.buf["reward"]), st._ptr(r.buf["done"])
    q.actions_planner = st._ptr(r.buf["actions_planner"]) if st.dims.n_act_planner else None
    if r.has_final_obs:
        q.final_obs = st._obs_buffers({k: r.buf["final_" + k] for k in r.obs_names})
    for k, v in over.items():
        setattr(q, k, v)
    return q


def test_emulated_abi_errors_and_launch_counts():
    env = _emu_env()
    env.reset()
    st, lib = env.stepper, env.stepper.lib
    r = env.bind_rollout(3, final_obs=True)
    lib.aie_bind_rollout(st._h, None)
    addr = lambda b: b.ctypes.data
    # EINVAL: zero T, a NULL required pointer, misaligned pointers, final slots partly given
    assert lib.aie_bind_rollout(st._h, C.byref(_rollout_struct(st, r, T=0))) == -1
    assert lib.aie_bind_rollout(st._h, C.byref(_rollout_struct(st, r, done=None))) == -1
    assert lib.aie_bind_rollout(st._h, C.byref(_rollout_struct(st, r, reward=addr(r.buf["reward"]) + 4))) == -1
    assert lib.aie_bind_rollout(st._h, C.byref(_rollout_struct(st, r, done=addr(r.buf["done"]) + 2))) == -1
    q = _rollout_struct(st, r)
    q.final_obs.obs_time = None
    assert lib.aie_bind_rollout(st._h, C.byref(q)) == -1
    q = _rollout_struct(st, r)
    q.obs.mask_agent = addr(r.buf["mask_agent"]) + 1
    assert lib.aie_bind_rollout(st._h, C.byref(q)) == -1
    assert lib.aie_compute_advantages_k(st._h, None, 3, 1, None) == -1
    # back to the stepper's own binding
    assert lib.aie_bind_rollout(st._h, C.byref(_rollout_struct(st, r))) == 0
    st.rollout_slot = 0
    n0 = st.launch_count()
    assert lib.aie_rollout_restart(st._h, None) == -3        # s != T
    assert lib.aie_set_fused_policy(st._h, 9, None) == -3
    assert lib.aie_step_dynamics(st._h, None) == -3
    assert lib.aie_observe_final(st._h, C.byref(st._final_bufs), None) == -3
    assert lib.aie_step_host(st._h, addr(r.buf["actions_agent"]), addr(r.buf["actions_planner"]),
                             C.byref(_abi.AieHostOut()), None) == -3
    assert lib.aie_bind_buffers(st._h, C.byref(_abi.AieBuffers())) == -3
    assert st.launch_count() == n0
    for t in range(3):
        st.sample_random_actions(t + 1)
        assert st.launch_count() == n0 + 1
        st.step()   # the step, then the final pass: two launches, as aie_step + aie_observe_final
        assert st.launch_count() == n0 + 3
        n0 += 3
        if t == 0:
            assert lib.aie_load_state(st._h, None, 0, None) == -1   # argument checks first
            with pytest.raises(_abi.AieError):
                env.reset()                                                  # resets only at slot 0
    assert lib.aie_step(st._h, None) == -3                          # s == T
    assert lib.aie_sample_random_actions(st._h, 1, None) == -3
    assert st.rollout_slot == 3
    st.restart_rollout()
    assert st.launch_count() == n0                                           # copies only
    env.reset()                                                              # allowed at slot 0
    # final slots need auto_reset and an episode_final buffer
    env2 = _emu_env(final_obs=False, auto_reset=False)
    st2 = env2.stepper
    with pytest.raises(ValueError):
        env2.bind_rollout(2, final_obs=True)
    r2 = st2.bind_rollout(2)
    st2.unbind_rollout()
    q = _rollout_struct(st2, r2)
    q.final_obs = _rollout_struct(st, r).final_obs
    assert st2.lib.aie_bind_rollout(st2._h, C.byref(q)) == -3
    # the fused random policy refuses the binding
    env3 = _emu_env()
    env3.reset()
    env3.stepper.set_fused_policy(3)
    with pytest.raises(_abi.AieError):
        env3.bind_rollout(2)


def test_emulated_unbound_env_is_unchanged():
    """An env that binds, runs and unbinds a rollout steps on exactly as one that never bound: same bytes, same
    launches per step."""
    A_, B_ = _emu_env(), _emu_env()
    for env in (A_, B_):
        env.reset()
    r = B_.bind_rollout(2, final_obs=True)
    B_.step(None)
    B_.step(None)
    B_.unbind_rollout()
    assert B_.obs_tensors["mask_agent"] is B_.stepper.buf["mask_agent"]
    A_.step(None)
    A_.step(None)
    for env in (A_, B_):
        env.stepper.observe()
    for t in range(9):
        n = [env.stepper.launch_count() for env in (A_, B_)]
        for env in (A_, B_):
            env.stepper.sample_random_actions(t + 40)
            env.step(env.action_buffers)
        assert [env.stepper.launch_count() for env in (A_, B_)] == [n[0] + 3, n[1] + 3]
        for k in list(OBS) + ["reward", "done"] + ["final_" + k for k in OBS]:
            if k in A_.stepper.buf:
                assert _same(A_.stepper.buf[k], B_.stepper.buf[k]), (t, k)
    assert r.buf["done"].shape == (2, 2)


def test_refusals():
    with pytest.raises(ValueError):
        _emu_env(dense_log_frequency=1).bind_rollout(2)

    def factory(spec, n_envs, auto_reset, **kw):
        from tests.emu.emu_stepper import EmuStepper

        class NoRollout(EmuStepper):
            bind_rollout = property(lambda self: (_ for _ in ()).throw(AttributeError("bind_rollout")))
        return NoRollout(spec, n_envs, auto_reset=auto_reset)

    name, kw = _cfg("c3_short_period", episode_length=7)
    env = foundation.make_env_instance(name, n_envs=2, seeds=[1, 2], stepper_factory=factory, **kw)
    with pytest.raises(NotImplementedError):
        env.bind_rollout(2)
    from ai_economist_b200.adapters import ReferenceApiEnv
    with pytest.raises(NotImplementedError):
        ReferenceApiEnv(_emu_env()).bind_rollout(2)


def test_emulated_saez_twin():
    """The Saez model's host estimator reads the state records, so a bound Saez env steps as its copy-loop twin."""
    from tests.emu.emu_stepper import emu_factory
    name, kw = _cfg("saez_reset", episode_length=7)
    assert run_rollout_twins(name, kw, 2, emu_factory, "float32", 8, 2) >= 2


# ---- GPU -----------------------------------------------------------------------------------------------------------
# c2 and c3 at bench size with 3-step episodes (K = 2 in a 4-step rollout); c5 keeps its 150-step episodes, so its
# rollout is 160 steps (K = 2) over 128 replicas, the size whose 161 observation slots and twin copies fit the card.
GPU_CASES = [("c1_tutorial", 8192, 4, 3), ("c3_paper_tax", 8192, 4, 3), ("c5_full", 128, 160, None)]


@pytest.mark.gpu
@pytest.mark.parametrize("cfg,E,T,ep", GPU_CASES, ids=["c2", "c3", "c5"])
def test_cuda_rollout_equals_the_copy_loop_at_bench_size(cfg, E, T, ep):
    name, kw = _cfg(cfg)
    if ep:
        kw["episode_length"] = ep
    assert run_rollout_twins(name, kw, E, None, "float32", T, 2) >= E


@pytest.mark.gpu
@pytest.mark.parametrize("obs_dtype", ["float32", "bfloat16"])
def test_cuda_covid_rollout_equals_the_copy_loop_at_bench_size(obs_dtype):
    """c4 size (4 096 replicas), 60-step episodes: a 130-step rollout crosses three episode ends (K = 3)."""
    assert run_covid_twins(4096, 60, obs_dtype, 130, 2, cuda=True) >= 4


@pytest.mark.gpu
def test_cuda_rollout_bf16_and_emulation_slots():
    """bfloat16 twins on CUDA, and CUDA's slots against the emulation's, byte for byte."""
    from tests.emu.emu_stepper import emu_factory
    name, kw = _cfg("c3_short_period", episode_length=7)
    assert run_rollout_twins(name, kw, 64, None, "bfloat16", 16, 2) >= 64
    envs = [_make(name, kw, 16, f, "float32") for f in (None, emu_factory)]
    rs = [env.bind_rollout(16, final_obs=True) for env in envs]
    for env in envs:
        _start(env, 16)
    for t in range(16):
        for env in envs:
            env.stepper.sample_random_actions(t + 1)
            env.step(env.action_buffers)
    torch.cuda.synchronize()
    for k, v in rs[1].buf.items():
        assert np.array_equal(np.ascontiguousarray(_np(rs[0].buf[k])).view(np.uint8), np.ascontiguousarray(v).view(np.uint8)), k


# ---- COVID-19 -------------------------------------------------------------------------------------------------------
COVID_OBS = _abi.COVID_OBS_NAMES


def _covid(E, episode_length, obs_dtype, cuda=False, observe_rate=True):
    from ai_economist_b200.workloads import COVID_KWARGS, covid_reference_config
    kw = dict(COVID_KWARGS, episode_length=episode_length, start_date="2020-12-01", delivery_interval=7,
              vaccine_delivery_start_date="2020-12-15")
    cfg = covid_reference_config(kw)
    if observe_rate:
        for c in cfg["components"]:
            if "VaccinationCampaign" in c:
                c["VaccinationCampaign"]["observe_rate"] = True
    dev = dict(device="cuda:0")
    if not cuda:
        from tests.test_covid_obs_bf16 import emu
        dev = dict(stepper_factory=lambda p, n, ar, final_obs=False, obs_dtype=None:
                   emu(p, n, ar, final_obs=final_obs, obs_dtype=obs_dtype))
    return foundation.make_env_instance(cfg.pop("scenario_name"), n_envs=E, auto_reset=True, final_obs=True,
                                        obs_dtype=obs_dtype, **dev, **cfg)


def run_covid_twins(E, episode_length, obs_dtype, T, rounds, cuda=False, gamma=0.97, lam=0.9):
    """The COVID-19 twins: B binds a rollout with final slots, Y runs the copy loop.  Also checks that every replica
    ends on the same step and that the final slot k is the episodes counter of hdr minus its value at the rollout's
    start.  Returns the number of episode ends (steps) seen."""
    B, Y = _covid(E, episode_length, obs_dtype, cuda), _covid(E, episode_length, obs_dtype, cuda)
    r = B.bind_rollout(T, final_obs=True)
    for env in (B, Y):
        env.reset()
    RATE = "VaccinationCampaign-next_vaccination_rate"
    sa, sp, na, npl = B.stepper._policy_shapes()
    rng = np.random.RandomState(3)
    lp = (_like(B, np.zeros((T,) + na, np.float32)), _like(B, np.zeros((T,) + npl, np.float32)))
    ends = 0
    for rnd in range(rounds):
        if rnd:
            B.restart_rollout()
            for k in COVID_OBS:
                assert _same(r.buf[k][0], last[k]), "round %d: slot 0 of %s" % (rnd, k)
        ep0 = _np(B.stepper.buf["hdr"])[:, 3].copy()
        copies = {k: [] for k in list(COVID_OBS) + ["a", "p", "ra", "rp", "done", "lpa", "lpp", "rate_a", "rate_p"]}
        finals = []
        for t in range(T):
            assert B.obs is r.obs[t]
            for k in COVID_OBS:
                copies[k].append(_snap(Y.stepper.buf[k]))
            copies["rate_a"].append(_snap(Y.obs["a"][RATE]))
            copies["rate_p"].append(_snap(Y.obs["p"][RATE]))
            la, lpl = rng.standard_normal(sa).astype(np.float32), rng.standard_normal(sp).astype(np.float32)
            B.sample_actions(_like(B, la), _like(B, lpl), seed=9 + rnd, out=(lp[0][t], lp[1][t]))
            oy = Y.sample_actions(_like(Y, la), _like(Y, lpl), seed=9 + rnd)
            copies["lpa"].append(_np(oy[0]).copy())
            copies["lpp"].append(_np(oy[1]).copy())
            copies["a"].append(_snap(Y.action_buffers[0]))
            copies["p"].append(_snap(Y.action_buffers[1]))
            B.step(B.action_buffers)
            Y.step(Y.action_buffers)
            copies["ra"].append(_snap(Y.rew["a"]))
            copies["rp"].append(_snap(Y.rew["p"]))
            done = _np(Y.done["__all__"]).copy()
            copies["done"].append(done)
            ep = _np(B.stepper.buf["hdr"])[:, 3]
            assert done.all() or not done.any(), "every replica ends on the same step"
            if done.any():
                k = int(ep[0] - ep0[0]) - 1
                assert (ep - ep0 == k + 1).all()
                finals.append((k, {n: _snap(Y.stepper.buf["final_" + n]) for n in COVID_OBS},
                               (_snap(Y.final_obs["a"][RATE]), _snap(Y.final_obs["p"][RATE]))))
        last = {k: _snap(Y.stepper.buf[k]) for k in COVID_OBS}
        for k in COVID_OBS:
            for t in range(T):
                assert _same(r.buf[k][t], copies[k][t]), "round %d slot %d: %s" % (rnd, t, k)
            assert _same(r.buf[k][T], last[k]), k
        assert _same(r.buf["rate_agent"][T], _snap(Y.obs["a"][RATE])) and _same(r.buf["rate_planner"][T], _snap(Y.obs["p"][RATE]))
        for t in range(T):
            for mine, theirs in (("actions_agent", "a"), ("actions_planner", "p"), ("reward_agent", "ra"),
                                 ("reward_planner", "rp"), ("rate_agent", "rate_a"), ("rate_planner", "rate_p")):
                assert _same(r.buf[mine][t], copies[theirs][t]), "round %d slot %d: %s" % (rnd, t, mine)
        D = np.stack(copies["done"])
        assert np.array_equal(_np(r.buf["done"]), D)
        assert np.array_equal(_np(lp[0]).view(np.uint32), np.stack(copies["lpa"]).view(np.uint32))
        assert np.array_equal(_np(lp[1]).view(np.uint32), np.stack(copies["lpp"]).view(np.uint32))
        for k, rows, (fra, frp) in finals:
            assert k < r.K
            for n, row in rows.items():
                assert _same(r.buf["final_" + n][k], row), "round %d final slot %d: %s" % (rnd, k, n)
            assert _same(r.buf["final_rate_agent"][k], fra) and _same(r.buf["final_rate_planner"][k], frp)
        ends += len(finals)
        # advantages: the stored rewards and [K, ...] final values against the copy loop's [T, ...] call
        S = B.n_agents
        V = (rng.standard_normal((T, E, S)).astype(np.float32), rng.standard_normal((T, E)).astype(np.float32))
        LV = (rng.standard_normal((E, S)).astype(np.float32), rng.standard_normal(E).astype(np.float32))
        FK = (rng.standard_normal((r.K, E, S)).astype(np.float32), rng.standard_normal((r.K, E)).astype(np.float32))
        FT = (np.full((T, E, S), np.nan, np.float32), np.full((T, E), np.nan, np.float32))
        for k, t in enumerate(np.nonzero(D[:, 0])[0]):
            FT[0][t], FT[1][t] = FK[0][k], FK[1][k]
        g = lambda env, x: tuple(_like(env, a) for a in x)
        out_b = B.compute_advantages((r.buf["reward_agent"], r.buf["reward_planner"]), g(B, V), r.buf["done"], g(B, LV),
                                     g(B, FK), gamma=gamma, lam=lam, per_episode_end=True)
        R = (np.stack([_np(x) for x in copies["ra"]]), np.stack([_np(x) for x in copies["rp"]]))
        out_y = Y.compute_advantages(g(Y, R), g(Y, V), _like(Y, D), g(Y, LV), g(Y, FT), gamma=gamma, lam=lam)
        for x, y in zip(out_b, out_y):
            assert same_bits(_np(x), _np(y))
        for gi in range(2):
            adv, ret = gae_ref(R[gi], V[gi], D, LV[gi], FT[gi], gamma, lam)
            assert same_bits(_np(out_b[gi]), adv) and same_bits(_np(out_b[2 + gi]), ret)
    return ends


@pytest.mark.parametrize("obs_dtype", ["float32", "bfloat16"])
@pytest.mark.parametrize("T,rounds", [(5, 4), (16, 2)])   # K = 1 and K = 3 at episode_length 7
def test_emulated_covid_rollout_equals_the_copy_loop(T, rounds, obs_dtype):
    assert run_covid_twins(2, 7, obs_dtype, T, rounds) >= 2


def test_emulated_covid_abi_errors_and_launch_counts():
    env = _covid(2, 7, "float32")
    env.reset()
    st, lib = env.stepper, env.stepper.lib
    r = env.bind_rollout(3, final_obs=True)
    q = _abi.AieCovidRollout()
    assert lib.aie_covid_bind_rollout(st._h, C.byref(q)) == -1          # T = 0
    q.T = 3
    assert lib.aie_covid_bind_rollout(st._h, C.byref(q)) == -1          # NULL buffers
    assert lib.aie_covid_compute_advantages_k(st._h, None, 3, 0, None) == -1
    assert lib.aie_covid_step_final(st._h, C.byref(st._final_bufs), None) == -3
    assert lib.aie_covid_bind_buffers(st._h, C.byref(_abi.AieCovidBuffers())) == -3
    assert lib.aie_covid_rollout_restart(st._h, None) == -3             # s != T
    n0 = lib.aie_covid_launch_count(st._h)
    for t in range(3):
        st.sample_random_actions(t + 1)
        env.step(env.action_buffers)
        assert lib.aie_covid_launch_count(st._h) == n0 + 2 * (t + 1)    # one launch per call
        if t == 0:
            with pytest.raises(_abi.AieError):
                env.reset()
    assert lib.aie_covid_step(st._h, None) == -3
    assert lib.aie_covid_sample_random_actions(st._h, 1, None) == -3
    env.restart_rollout()
    assert lib.aie_covid_launch_count(st._h) == n0 + 6
    env.unbind_rollout()
    assert env.obs["a"]["world-agent_state"] is st.buf["obs_agent_state"]
    from tests.test_covid_obs_bf16 import emu
    no_reset = emu(env.params, 2, False)
    with pytest.raises(_abi.AieError):   # final slots need the auto-reset
        no_reset.bind_rollout(2, final_obs=True)


def test_per_episode_end_keeps_shape_mistakes_loud():
    env = _emu_env()
    env.reset()
    E, A = 2, env.n_agents
    z = lambda *s: np.zeros(s, np.float32)
    r = np.zeros((4, E, A + 1)), np.zeros((4, E), np.int32)
    args = (r[0], (z(4, E, A), z(4, E)), r[1], (z(E, A), z(E)))
    with pytest.raises(ValueError):   # [K, ...] final values without the keyword
        env.compute_advantages(*args, (z(2, E, A), z(2, E)), gamma=0.9)
    env.compute_advantages(*args, (z(2, E, A), z(2, E)), gamma=0.9, per_episode_end=True)
    with pytest.raises(ValueError):
        env.compute_advantages(*args, None, gamma=0.9, per_episode_end=True)
