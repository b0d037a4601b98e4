"""Device-side reset with reference semantics (SURVEY §8f row 1).

Multi-episode golden traces (tests/golden_reset/, recorded from the unmodified reference with env.reset() between
episodes — the reference keeps drawing from the same global numpy stream) are replayed through the public API with
auto_reset on: when an env finishes, the step kernel restores maps / inventories / books from the snapshot and then
re-draws placement, skills and the fixed_four assignment from the env's own MT19937 stream on the device.  Rewards
and done of the terminal step belong to the finished episode; state and observations to the fresh one.
"""
import glob
import os

import numpy as np
import pytest

from ai_economist_b200 import foundation
from tests import golden_utils as gu

FILES = sorted(glob.glob(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden_reset", "*.npz")))


def _env(meta, factory):
    kw = dict(meta["reference_kwargs"])
    name = kw.pop("scenario_name")
    kw["components"] = [tuple(c) for c in kw["components"]]
    if "seed" in kw:   # a constructor seed (split_layout's skill table): both replicas like the reference's single env
        kw["seeds"] = [kw.pop("seed")] * 2
    extra = dict(stepper_factory=factory) if factory else dict(device="cuda:0")
    return foundation.make_env_instance(name, n_envs=2, auto_reset=True, **kw, **extra)


def _replay(path, factory):
    z, meta, init = gu.load_fixture(path)
    env = _env(meta, factory)
    assert env.spec["reset_mode"] == 1
    env.seed([meta["seed"], meta["seed"]])     # both replicas identical: checks env indexing too
    env.reset()
    s = env.stepper
    full = {int(t): i for i, t in enumerate(z["full_steps"])}
    A = env.n_agents
    n_done = 0
    gu.check_step(z, 0, s.read_obs(1), s.read_state(1), full.get(0), "reset-trace")
    for t in range(1, int(meta["n_steps"]) + 1):
        acts = {str(i): np.repeat(z["act_a"][t - 1][i][None], 2, axis=0) for i in range(A)}
        if z["act_p"].shape[1]:
            acts["p"] = np.repeat(z["act_p"][t - 1][None], 2, axis=0)
        env.step(acts)
        st = s.read_state(1)
        gu.check_step(z, t, s.read_obs(1), st, full.get(t), "reset-trace", books=st["books"])
        n_done += int(z["step_done"][t])
    assert n_done >= 2, "the trace must cross at least two episode boundaries"
    assert int(s.read_state(1)["completions"][0]) == n_done


@pytest.mark.parametrize("path", FILES, ids=lambda p: os.path.basename(p))
def test_emulated_device_reset_matches_reference_across_episodes(path):
    from tests.emu.emu_stepper import emu_factory
    _replay(path, emu_factory)


@pytest.mark.gpu
@pytest.mark.parametrize("path", FILES, ids=lambda p: os.path.basename(p))
def test_cuda_device_reset_matches_reference_across_episodes(path):
    _replay(path, None)


def _replay_previous_episode_metrics(path, factory):
    """env.previous_episode_metrics after each auto-reset == the reference's after its env.reset()."""
    import json
    from tests.metrics_utils import compare_metrics
    ref = json.load(open(path.replace("golden_reset", "golden_metrics_reset").replace(".npz", ".json")))
    want = dict(zip(ref["steps"], ref["metrics"]))
    z, meta, init = gu.load_fixture(path)
    env = _env(meta, factory)
    env.seed([meta["seed"], meta["seed"]])
    env.reset()
    assert env.previous_episode_metrics_of(1) is None
    A, seen = env.n_agents, 0
    for t in range(1, int(meta["n_steps"]) + 1):
        acts = {str(i): np.repeat(z["act_a"][t - 1][i][None], 2, axis=0) for i in range(A)}
        if z["act_p"].shape[1]:
            acts["p"] = np.repeat(z["act_p"][t - 1][None], 2, axis=0)
        env.step(acts)
        if t in want:
            compare_metrics(want[t], env.previous_episode_metrics_of(1), "episode ending at t=%d" % t)
            seen += 1
    assert seen >= 2


@pytest.mark.parametrize("path", FILES, ids=lambda p: os.path.basename(p))
def test_emulated_previous_episode_metrics_match_reference(path):
    from tests.emu.emu_stepper import emu_factory
    _replay_previous_episode_metrics(path, emu_factory)


@pytest.mark.gpu
@pytest.mark.parametrize("path", FILES, ids=lambda p: os.path.basename(p))
def test_cuda_previous_episode_metrics_match_reference(path):
    _replay_previous_episode_metrics(path, None)


EXPLICIT = ["saez_reset", "saez_annealed_reset", "c3_reset", "c1_reset", "lognormal_reset", "us_federal_annealed"]


def _replay_explicit_host_resets(which, factory):
    """auto_reset off: env.reset() between episodes goes through the host reset path.  It has to carry the Saez
    estimator's persistent state (sample counter, rates in force / observed) across the repacked records, and the
    completed-episode count that drives the tax-annealing and energy-warm-up schedules (c3_reset; base_env.py:1021-1025
    increments it on the step that ends the episode).  Every reset ends in the stand-alone observation pass, which has to
    stage the Saez section the curr_rates / marginal_rate observations read."""
    path = [p for p in FILES if which in p][0]
    z, meta, init = gu.load_fixture(path)
    kw = dict(meta["reference_kwargs"])
    name = kw.pop("scenario_name")
    kw["components"] = [tuple(c) for c in kw["components"]]
    extra = dict(stepper_factory=factory) if factory else dict(device="cuda:0")
    env = foundation.make_env_instance(name, n_envs=1, auto_reset=False, **kw, **extra)
    env.seed([meta["seed"]])
    env.reset()
    s = env.stepper
    full = {int(t): i for i, t in enumerate(z["full_steps"])}
    A = env.n_agents
    for t in range(1, int(meta["n_steps"]) + 1):
        acts = {str(i): z["act_a"][t - 1][i][None] for i in range(A)}
        if z["act_p"].shape[1]:
            acts["p"] = z["act_p"][t - 1][None]
        env.step(acts)
        last = s.read_obs(0)
        if int(z["step_done"][t]):
            env.reset()
        st, ob = s.read_state(0), s.read_obs(0)
        ob["rew"], ob["done"] = last["rew"], last["done"]   # reward / done belong to the step, not to the reset
        gu.check_step(z, t, ob, st, full.get(t), "host-reset-trace", books=st["books"])


@pytest.mark.parametrize("which", EXPLICIT)
def test_emulated_explicit_host_resets_match_reference(which):
    from tests.emu.emu_stepper import emu_factory
    _replay_explicit_host_resets(which, emu_factory)


@pytest.mark.gpu
@pytest.mark.parametrize("which", EXPLICIT)
def test_cuda_explicit_host_resets_match_reference(which):
    _replay_explicit_host_resets(which, None)
