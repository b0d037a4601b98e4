"""RL-framework adapters over BatchedFoundationEnv (SURVEY 8f row 4).  Plumbing only: they rename / re-shape the
tensors the step kernel already wrote, without copies on the batched path.

* `WarpDriveStyleEnvWrapper` mirrors FoundationEnvWrapper (ai_economist/foundation/env_wrapper.py:84-418): spaces on
  the env (:139-172), `reset_all_envs()` / `step_all_envs()`, and the reserved array names WarpDrive trainers look up
  (`observations_*`, `actions_*`, `rewards_*`, `_done_`, `_timestep_`; covid19_env.py:700-722, 1002-1040) served as
  zero-copy views of the device tensors.
* `MultiAgentDictEnv` mirrors the RLlib wrapper (tutorials/rllib/env_wrapper.py:50-211) for ONE replica: nested
  per-agent dicts of numpy arrays in, reference action dict out.  One device->host copy per step; meant for
  evaluation / debugging - a learner should consume the batched tensors.
"""
import numpy as np

_BIG_NUMBER = 1e20

try:  # gym / gymnasium when present; tiny stand-ins otherwise (neither is part of this image)
    from gymnasium import spaces as _spaces  # noqa: F401
    Box, Discrete, MultiDiscrete, Dict = _spaces.Box, _spaces.Discrete, _spaces.MultiDiscrete, _spaces.Dict
except Exception:  # pragma: no cover - depends on the image
    class Box:
        def __init__(self, low, high, shape, dtype):
            self.low, self.high, self.shape, self.dtype = float(low), float(high), tuple(shape), np.dtype(dtype)

        def contains(self, x):
            x = np.asarray(x)
            return x.shape == self.shape and bool(np.all(x >= self.low)) and bool(np.all(x <= self.high))

        def __repr__(self):
            return "Box(%g, %g, %s, %s)" % (self.low, self.high, self.shape, self.dtype)

    class Discrete:
        def __init__(self, n):
            self.n, self.dtype, self.shape = int(n), np.dtype(np.int64), ()

        def contains(self, x):
            return 0 <= int(x) < self.n

        def __repr__(self):
            return "Discrete(%d)" % self.n

    class MultiDiscrete:
        def __init__(self, nvec):
            self.nvec = np.asarray(nvec, np.int64)
            self.dtype, self.shape = np.dtype(np.int64), self.nvec.shape

        def contains(self, x):
            x = np.asarray(x)
            return x.shape == self.nvec.shape and bool(np.all(x >= 0)) and bool(np.all(x < self.nvec))

        def __repr__(self):
            return "MultiDiscrete(%s)" % self.nvec.tolist()

    class Dict(dict):
        @property
        def spaces(self):
            return self


def _space_of(shape, dtype):
    """The Box the reference builds for an observation array (tutorials/rllib/env_wrapper.py:117-140): symmetric
    bounds, halved until representable in the dtype."""
    dtype = np.dtype(dtype)
    x = float(_BIG_NUMBER)
    if dtype.kind in "iu":
        x = float(min(x, np.iinfo(dtype).max))
    while not np.isfinite(np.array(x, dtype=dtype)) or np.array(x, dtype=dtype) <= 0:
        x = x // 2
    return Box(low=-x, high=x, shape=tuple(shape), dtype=dtype)


def _action_space(agent):
    sp = agent.action_spaces
    return MultiDiscrete(sp) if agent.multi_action_mode else Discrete(int(sp))


class WarpDriveStyleEnvWrapper:
    """FoundationEnvWrapper for the batched env: `env` is a BatchedFoundationEnv (or make_env_instance kwargs)."""

    def __init__(self, env_obj=None, **make_env_kwargs):
        if env_obj is None:
            from . import foundation
            env_obj = foundation.make_env_instance(**make_env_kwargs)
        self.env = env_obj
        self.n_envs = env_obj.n_envs
        self.n_agents = env_obj.num_agents            # mobile agents + planner (env_wrapper.py:133)
        self.episode_length = env_obj.episode_length
        self.name = env_obj.name
        self.use_cuda = True
        self.reset_on_host = True
        A = env_obj.n_agents
        b = env_obj.stepper.buf
        if hasattr(env_obj, "params"):   # the COVID-19 scenario: the env the reference's wrapper was written for
            self._init_covid(env_obj, A, b)
            return
        # ---- spaces (env_wrapper.py:139-172): per agent id, from the per-replica slice of each tensor ----
        self.env.observation_space = Dict({k: Dict({kk: _space_of(tuple(v.shape[1:]), self._np_dtype(v))
                                                    for kk, v in d.items()}) for k, d in env_obj.obs.items()})
        self.env.action_space = {str(i): _action_space(env_obj.get_agent(i)) for i in range(A)}
        self.env.action_space["p"] = _action_space(env_obj.get_agent("p"))
        assert set(self.env.observation_space.keys()) == set(self.env.action_space.keys())
        # ---- reserved array names -> zero-copy views [E, ...] ----
        d = {"_done_": b["done"], "actions_a": b["actions_agent"], "actions_p": b["actions_planner"],
             "rewards_a": b["reward"][:, :A], "rewards_p": b["reward"][:, A]}
        if hasattr(env_obj.stepper, "state_view"):
            d["_timestep_"] = env_obj.stepper.state_view("t")
        names = {"obs_agent_map": "a_world-map", "obs_agent_idx": "a_world-idx_map", "obs_agent_flat": "a_flat",
                 "mask_agent": "a_action_mask", "obs_planner_map": "p_world-map", "obs_planner_idx": "p_world-idx_map",
                 "obs_planner_flat": "p_flat", "mask_planner": "p_action_mask", "obs_time": "a_time",
                 "obs_planner_agents": "p_agents"}
        for k, n in names.items():
            if k in b:
                d["observations_" + n] = b[k]
        d["observations_p_time"] = b["obs_time"]
        self.data = d

    def _init_covid(self, env_obj, A, b):
        """CovidAndEconomySimulation (collated "a" / "p" observations, single-action agents and planner): per-state
        observation spaces as the reference builds them by un-collating "a" (env_wrapper.py:139-150), Discrete action
        spaces, and the reserved array names of covid19_env.py:700-722, 1002-1040 as views of the device tensors."""
        p = env_obj.params
        per_agent = Dict({k: _space_of(tuple(v.shape[1:-1]), self._np_dtype(v)) for k, v in env_obj.obs["a"].items()})
        spaces = {str(i): per_agent for i in range(A)}
        spaces["p"] = Dict({k: _space_of(tuple(v.shape[1:]), self._np_dtype(v)) for k, v in env_obj.obs["p"].items()})
        self.env.observation_space = Dict(spaces)
        self.env.action_space = {str(i): Discrete(1 + int(p["num_stringency_levels"])) for i in range(A)}
        self.env.action_space["p"] = Discrete(1 + int(p["num_subsidy_levels"]))
        assert set(self.env.observation_space.keys()) == set(self.env.action_space.keys())
        d = {"_done_": b["done"], "_timestep_": b["hdr"][:, 0], "actions_a": b["actions_agent"], "actions_p": b["actions_planner"],
             "rewards_a": b["reward_agent"], "rewards_p": b["reward_planner"]}
        for who in ("a", "p"):
            for k, v in env_obj.obs[who].items():
                d["observations_%s_%s" % (who, k)] = v
        self.data = d

    @staticmethod
    def _np_dtype(v):
        """numpy dtype of a tensor's Box: bfloat16 observations (raw uint16 bits on numpy backends) get float32 spaces."""
        if isinstance(v, np.ndarray):
            return np.dtype(np.float32) if v.dtype == np.uint16 else v.dtype
        name = str(v.dtype).replace("torch.", "")
        return np.dtype(np.float32 if name == "bfloat16" else name)

    def tensor(self, name):
        """Device tensor registered under a WarpDrive-style name (cuda_data_manager.device_data(name))."""
        return self.data[name]

    def reset_all_envs(self):
        """Host reset of every replica (first reset; later episodes reset on the device inside step)."""
        obs = self.env.reset()
        self.reset_on_host = False
        return obs

    def reset_only_done_envs(self):
        """With auto_reset the step kernel already restarted finished replicas (env_wrapper.py:335-337)."""
        return {}

    def step_all_envs(self, actions=None):
        """actions=None: step from whatever a policy wrote into actions_a / actions_p (the WarpDrive convention)."""
        return self.env.step(self.env.action_buffers if actions is None else actions)

    step = step_all_envs
    reset = reset_all_envs


class MultiAgentDictEnv:
    """RLlib-style view of replica `e`: reset()/step(action_dict) with nested numpy dicts."""

    def __init__(self, env_obj, e=0):
        self.env, self.e = env_obj, int(e)
        self.sample_agent_idx = "0"
        self._ensure_loaded()
        obs, _, _ = env_obj.reference_view(self.e)
        mk = lambda d: Dict({k: _space_of(np.asarray(v).shape if np.ndim(v) else (1,), np.asarray(v).dtype)
                             for k, v in d.items()})
        self.observation_space, self.observation_space_pl = mk(obs["0"]), mk(obs["p"])
        self.action_space = _action_space(env_obj.get_agent(0))
        self.action_space_pl = _action_space(env_obj.get_agent("p"))

    def _ensure_loaded(self):
        if not getattr(self.env, "_loaded", False):
            self.env.reset()

    @property
    def n_agents(self):
        return self.env.n_agents

    @property
    def summary(self):
        m = self.env.previous_episode_metrics_of(self.e)
        if m is None:
            return {}
        m["completions"] = int(self.env.stepper.read_state(self.e)["completions"][0])
        return m

    def reset(self):
        self.env.reset()
        return self.env.reference_view(self.e)[0]

    # ---- checkpoints (tutorials/rllib/env_wrapper.py:155-165, pickle_file): the whole batched env, every replica ----
    pickle_file = "game_object.pt"

    def save_game_object(self, save_dir):
        """Write env.state_dict() to save_dir/game_object.pt (torch.save)."""
        import os

        import torch
        assert os.path.isdir(save_dir)
        torch.save(self.env.state_dict(), os.path.join(save_dir, self.pickle_file))

    def load_game_object(self, save_dir):
        """Load save_dir/game_object.pt into the wrapped env (load_state_dict), which must have the configuration of the
        env it was saved from."""
        import os

        import torch
        assert os.path.isdir(save_dir)
        # the dict holds numpy arrays and plain Python values next to tensors: not a weights-only file
        self.env.load_state_dict(torch.load(os.path.join(save_dir, self.pickle_file), weights_only=False))

    def step(self, action_dict):
        """action_dict: {agent id: int | list} for this replica; the other replicas take NO-OPs."""
        st = self.env.stepper
        ba, bp = st.buf["actions_agent"], st.buf["actions_planner"]
        ba[...] = 0
        bp[...] = 0
        for k, v in action_dict.items():
            row = np.atleast_1d(np.asarray(v, np.int32))
            if str(k) == "p":
                if st.dims.n_act_planner:
                    bp[self.e] = self.env._as_buf(row, bp, (st.dims.n_act_planner,))
            else:
                ba[self.e, int(k)] = self.env._as_buf(row, ba, (st.dims.n_act_agent,))
        self.env.step(self.env.action_buffers)
        obs, rew, done = self.env.reference_view(self.e)
        return obs, rew, done, {k: {} for k in obs}


class ReferenceApiEnv:
    """One replica behind the reference's exact single-env interface (base/base_env.py:852-1032), so that code written
    against ai_economist.foundation - the tutorials' `sample_random_actions(env, obs)` / `play_random_episode(env)`
    loops, tutorials/utils/plotting.py - runs unchanged:

        env = foundation.make_env_instance(**env_config, reference_api=True)     # or AIE_REFERENCE_API=1
        obs = env.reset()                              # nested dicts of numpy arrays / floats, keyed "0".."n-1", "p"
        obs, rew, done, info = env.step({"0": 3, "1": [0, 2, ...], "p": [...]})

    Observation layout follows flatten_observations / flatten_masks / collate_agent_step_and_reset_data like the
    reference.  Everything else (get_agent, episode_length, world, metrics, dense logs, seed ...) is the wrapped
    BatchedFoundationEnv's.  One device->host copy per step: an evaluation / debugging surface, not the training path.
    One difference is inherent: the env draws from its OWN numpy-legacy stream, not from the process-global
    np.random, so caller code that samples from np.random between steps no longer perturbs the env's draws.
    """

    def __init__(self, env_obj, e=0):
        object.__setattr__(self, "_env", env_obj)
        object.__setattr__(self, "_e", int(e))

    def __getattr__(self, name):           # get_agent, n_agents, episode_length, world, metrics, dense logs, seed ...
        return getattr(self._env, name)

    def bind_rollout(self, T, final_obs=False):
        raise NotImplementedError("the reference API steps one replica through host copies; bind rollouts on the "
                                  "batched env (reference_api=False)")

    def capture_rollout(self, act):
        raise ValueError("the reference API steps one replica through host copies; capture rollouts on the batched env "
                         "(reference_api=False)")

    @property
    def _completions(self):                # int, like the reference's (tutorials/rllib/env_wrapper.py:176 reads it)
        return int(self._env.completions()[self._e])

    # ---- output conversion -------------------------------------------------------------------------------
    def _np(self, v):
        """numpy copy of an output tensor; bfloat16 observations as float32 (raw uint16 bits on numpy backends)."""
        from .stepper import bf16_bits_to_float32
        st = self._env.stepper
        a = st.to_numpy(v) if not isinstance(v, np.ndarray) else v
        return bf16_bits_to_float32(a) if np.asarray(a).dtype == np.uint16 else a

    def _one(self, v):
        """The replica's slice of a batched value: arrays stay arrays, per-env scalars become Python floats."""
        if isinstance(v, dict):
            return {k: self._one(x) for k, x in v.items()}
        a = np.asarray(self._np(v))[self._e]
        return float(a) if a.ndim == 0 else np.array(a)

    def _outputs(self):
        env, e = self._env, self._e
        if env._flatten_observations and env._flatten_masks and not env.collate_agent_step_and_reset_data:
            obs, rew, done = env.reference_view(e)          # one readback through aie_read-style debug copies
            return obs, rew, done
        obs = {}
        for idx, d in env.obs.items():
            o = {}
            for k, v in d.items():
                if k == "time":
                    t = np.asarray(self._np(v))[e]
                    o[k] = np.array(t, np.float64).reshape(-1) if np.ndim(t) else [float(t)]
                else:
                    o[k] = self._one(v)
            obs[idx] = o
        rew = {k: (self._one(v) if k != "a" else [float(x) for x in np.asarray(self._np(v))[e]])
               for k, v in env.rew.items()}
        done = {"__all__": bool(int(np.asarray(self._np(env.done["__all__"]))[e]))}
        return obs, rew, done

    # ---- replay logs (base_env.py:358-360, 444-471, 980-982) -----------------------------------------------
    @property
    def replay_log(self):
        """The current (possibly incomplete) replay log: {"reset": {"seed_state"}, "step": [{"actions", "seed_state"}]}."""
        return self.__dict__.get("_replay", {"reset": dict(seed_state=None), "step": []})

    @property
    def previous_episode_replay_log(self):
        """Replay log of the last completed episode: `env.reset(**log["reset"])` then `env.step(**s)` for every s in
        log["step"] reproduces it exactly (logs recorded by the reference itself replay here too)."""
        return self.__dict__.get("_last_replay", {"reset": dict(seed_state=None), "step": []})

    # ---- the Gym-style surface ---------------------------------------------------------------------------
    def reset(self, seed_state=None, force_dense_logging=False):
        env, e = self._env, self._e
        mine = env._np_state(seed_state) if seed_state is not None else env.stream_state(e)
        # like the reference (base_env.py:899): the log holds the stream state the reset cycle starts from
        object.__setattr__(self, "_replay", {"reset": dict(seed_state=mine), "step": []})
        if seed_state is not None and env.n_envs > 1:   # only this replica's stream moves
            seed_state = [mine if i == e else env.stream_state(i) for i in range(env.n_envs)]
        env.reset(seed_state=seed_state, force_dense_logging=force_dense_logging)
        return self._outputs()[0]

    def step(self, actions=None, seed_state=None):
        """actions: {agent idx (int or str): int | sequence of ints} (BaseAgent.parse_actions, base_agent.py:407-438);
        missing agents take NO-OPs, like the reference."""
        env, e = self._env, self._e
        st = env.stepper
        if seed_state is not None:
            env.set_stream_state(seed_state, e)
        if "_replay" in self.__dict__:
            self._replay["step"].append(dict(actions=actions, seed_state=env.stream_state(e)))
        ba, bp = st.buf["actions_agent"], st.buf["actions_planner"]
        ba[e] = 0
        bp[e] = 0
        for k, v in (actions or {}).items():
            if isinstance(v, dict):   # {subspace name: index}
                ag = env.get_agent(k)
                unknown = set(v) - set(ag._action_names)
                assert not unknown, "unknown action subspace(s) %s" % sorted(unknown)
                if ag.multi_action_mode:
                    # one entry per named subspace, the others stay NO-OP (set_component_action per name,
                    # base_agent.py:367-383; the reference's own dict branch only covers single-action agents)
                    v = [int(v.get(name, 0)) for name in ag._action_names]
                else:         # single-action agents (base_agent.py:419-427): at most one named sub-action
                    assert len(v) <= 1
                    g, lo = 0, 1
                    for name in ag._action_names:
                        if name in v and int(v[name]) > 0:
                            g = lo + int(v[name]) - 1
                        lo += int(ag.action_dim[name])
                    v = g
            row = np.atleast_1d(np.asarray(v)).astype(np.int32)
            if str(k) == "p":
                if st.dims.n_act_planner:
                    bp[e] = env._as_buf(row, bp, (st.dims.n_act_planner,))
            elif str(k) == "a":       # collated: [n_agents] or [n_agents, n_act]
                ba[e] = env._as_buf(row, ba, tuple(ba.shape[1:]))
            else:
                ba[e, int(k)] = env._as_buf(row, ba, (st.dims.n_act_agent,))
        env.step(env.action_buffers)
        obs, rew, done = self._outputs()
        if done["__all__"] and "_replay" in self.__dict__:
            object.__setattr__(self, "_last_replay", self._replay)   # _finalize_logs (base_env.py:763-765)
        return obs, rew, done, {k: {} for k in obs} if "a" not in obs else \
            {"a": {str(i): {} for i in range(env.n_agents)}, "p": {}}
