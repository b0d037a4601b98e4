"""BatchedFoundationEnv — the Gym-style reset/step surface of the reference's BaseEnvironment
(base/base_env.py:24-1120), over E env replicas that live on one GPU.

Differences from the reference API (all additive):
  * new kwargs `n_envs`, `device`, `seeds`, `auto_reset`, `device_reset`, `obs_dtype` (torch.float32, the default, or
    torch.bfloat16: the float observation / mask tensors are written as bfloat16 by the step kernel itself),
    `final_obs` (with auto_reset: `env.final_obs` holds the observations of the state each episode that ended in the
    latest step ended in, for bootstrapping the value of a truncated episode);
  * observations / rewards / done are persistent device tensors with a leading env axis, keyed exactly like
    the reference's dicts ("0".."n-1", "p"; "world-map", "world-idx_map", "flat", "action_mask", "time", "p<i>");
  * `reference_view(e)` re-creates the reference's nested numpy dict for one env (tests / debugging).
"""
import ctypes as C

import numpy as np

from .agents import agent_registry
from . import rollout_graph as _rg
from .components import component_registry
from .entities import endogenous_registry, landmark_registry, resource_registry


class _MapsView:
    """Read-only mirror of world.maps for one env replica (reference: base/world.py:13-329)."""
    _BITS = {"Stone": 1, "Wood": 2, "StoneSourceBlock": 4, "WoodSourceBlock": 8, "Water": 16, "House": 32}

    def __init__(self, env, e):
        self._env, self._e = env, e

    def keys(self):
        ks = ["Stone", "Wood", "House"] + (["Water"] if self._env._spec["has_water"] else [])
        return ks + ["StoneSourceBlock", "WoodSourceBlock"]

    def get(self, name, owner=False):
        st = self._env._stepper.read_state(self._e)
        if owner:
            assert name == "House"
            return st["owner"].astype(np.int16)
        return ((st["cell"] & self._BITS[name]) > 0).astype(np.float64)

    @property
    def state(self):
        return np.stack([self.get(k) for k in self.keys()]).astype(np.float32)


class _WorldView:
    def __init__(self, env, e=0):
        self._env, self._e = env, e
        self.maps = _MapsView(env, e)
        self.world_size = list(env.world_size)
        self.n_agents = env.n_agents

    @property
    def agents(self):
        return self._env._agents

    @property
    def planner(self):
        return self._env._planner

    @property
    def timestep(self):
        return int(self._env._stepper.read_state(self._e)["t"][0])


class BatchedFoundationEnv:
    def __init__(self, scenario_cls, components=None, n_agents=None, world_size=None, episode_length=1000,
                 multi_action_mode_agents=False, multi_action_mode_planner=True, flatten_observations=True,
                 flatten_masks=True, allow_observation_scaling=True, dense_log_frequency=None,
                 world_dense_log_frequency=50, collate_agent_step_and_reset_data=False, seed=None,
                 n_envs=1, device="cuda:0", seeds=None, auto_reset=True, stepper_factory=None, device_reset=None,
                 obs_dtype=None, final_obs=False, **scenario_kwargs):
        # ---- base_env.py:178-366 argument checks ----
        if final_obs and not auto_reset:
            raise ValueError("final_obs=True needs auto_reset=True: without the auto-reset, env.obs after the step that "
                             "ends an episode already is its final observation")
        assert isinstance(world_size, (tuple, list)) and len(world_size) == 2
        self.world_size = list(world_size)
        assert isinstance(n_agents, int) and n_agents >= 2
        self.n_agents = n_agents
        self.num_agents = n_agents + 1
        assert isinstance(components, (tuple, list))
        self._episode_length = int(episode_length)
        assert self._episode_length >= 1
        self.multi_action_mode_agents = bool(multi_action_mode_agents)
        self.multi_action_mode_planner = bool(multi_action_mode_planner)
        # flatten_observations / flatten_masks = False (base_env.py:260-270): the named fields are handed out as slices
        # of the flat tensors (aie_get_flat_layout), the per-subspace masks as slices of the flat masks - no copy
        self._flatten_observations = bool(flatten_observations)
        self._flatten_masks = bool(flatten_masks)
        self.collate_agent_step_and_reset_data = bool(collate_agent_step_and_reset_data)
        self._allow_observation_scaling = bool(allow_observation_scaling)
        self.n_envs = int(n_envs)
        assert self.n_envs >= 1

        # ---- entities + components (base_env.py:289-346) ----
        ents = {"resources": ["Coin"], "landmarks": [], "endogenous": ["Labor"]}

        def register(names):
            for n in names:
                for reg, key in ((resource_registry, "resources"), (landmark_registry, "landmarks"),
                                 (endogenous_registry, "endogenous")):
                    if reg.has(n):
                        if n not in ents[key]:
                            ents[key].append(n)
                        break
                else:
                    raise KeyError("Unknown entity: {}".format(n))

        register(scenario_cls.required_entities)
        specs = []
        for spec in components:
            if isinstance(spec, (tuple, list)):
                assert len(spec) == 2 and isinstance(spec[0], str) and isinstance(spec[1], dict)
                cname, ckw = spec
            else:
                assert isinstance(spec, dict) and len(spec) == 1
                cname, ckw = list(spec.items())[0]
            ccls = component_registry.get(cname)
            register(ccls.required_entities)
            specs.append((ccls, ckw))
        self._entities = ents
        self._components = [ccls(self.n_agents, self._episode_length, inventory_scale=self.inv_scale, **ckw)
                            for ccls, ckw in specs]
        self._components_dict = {c.name: c for c in self._components}
        self._shorthand_lookup = {c.shorthand: c for c in self._components}
        if len(self._components_dict) != len(self._components):
            raise ValueError("duplicate component")

        mobile, planner = agent_registry.get("BasicMobileAgent"), agent_registry.get("BasicPlanner")
        self._agents = [mobile(i, self.multi_action_mode_agents) for i in range(self.n_agents)]
        self._planner = planner(self.multi_action_mode_planner)
        for ag in self._agents + [self._planner]:
            ag._register(self._components)
            ag._env = self
        self._agent_lookup = {str(a.idx): a for a in self.all_agents}

        # base_env.py:286-287: a `seed` kwarg seeds the stream before anything is built, so scenario constructors that
        # draw (split_layout's skill table, multi_zone's first zone shuffle) consume the seeded stream
        self._rs = None
        self._seeds = None
        if seeds is not None:
            self.seed(seeds)
        elif seed is not None:
            self.seed(seed)
        self.scenario = scenario_cls(self, **scenario_kwargs)
        self.name = scenario_cls.name

        # ---- flat numeric spec handed to the C-ABI ----
        spec = dict(components=[c.name for c in self._components], n_agents=self.n_agents,
                    height=self.world_size[0], width=self.world_size[1], episode_length=self._episode_length,
                    multi_action_agents=int(self.multi_action_mode_agents),
                    single_action_planner=int(not self.multi_action_mode_planner),
                    allow_observation_scaling=int(self._allow_observation_scaling),
                    build_payment=10.0, build_labor=10.0, move_labor=1.0, collect_labor=1.0,
                    max_bid_ask=10, order_duration=50, max_num_orders=50, order_labor=0.25,
                    tax_model=0, disable_taxes=0, period=100, n_brackets=0, n_disc_rates=0, bracket_cutoffs=[],
                    disc_rates=[], fixed_rates=[], tax_annealing=0, annealing_warmup=0.0, annealing_slope=0.0,
                    rate_max=1.0)
        spec.update(self.scenario.scenario_spec_fields())
        for c in self._components:
            spec.update(c.spec_fields())
        if device_reset is not None:  # "reference" (default where supported) | "snapshot" (WarpDrive-style restore)
            assert device_reset in ("reference", "snapshot")
            if device_reset == "snapshot":
                spec["reset_mode"] = 0
            else:
                assert spec.get("reset_mode", 0) == 1, "reference-exact device reset is not available for this config"
        from .._abi import obs_dtype_name
        spec["obs_dtype"] = obs_dtype_name(obs_dtype)   # "float32" | "bfloat16"
        spec["final_obs"] = bool(final_obs)
        self._spec = spec

        # ---- dense logging (base_env.py:273-283): replica 0, every dense_log_frequency-th episode ----
        self._create_dense_log_every = None if dense_log_frequency is None else int(dense_log_frequency)
        assert self._create_dense_log_every is None or self._create_dense_log_every >= 1
        self._world_dense_log_frequency = int(world_dense_log_frequency)
        assert self._world_dense_log_frequency >= 1
        self._dense_logger = None
        self._rollout = None   # bind_rollout
        self._dense_log = {"world": [], "states": [], "actions": [], "rewards": []}
        self._last_ep_dense_log = dict(self._dense_log)
        self._auto_reset = bool(auto_reset)
        event_envs = 0 if self._create_dense_log_every is None else 1

        if stepper_factory is None:
            from ..stepper import CudaStepper
            self._stepper = CudaStepper(spec, self.n_envs, device=device, auto_reset=auto_reset, event_envs=event_envs)
        else:
            try:
                self._stepper = stepper_factory(spec, self.n_envs, auto_reset, event_envs=event_envs)
            except TypeError:
                self._stepper = stepper_factory(spec, self.n_envs, auto_reset)
        self._loaded = False
        self._completions = np.zeros(self.n_envs, np.int64)
        if self._stepper is not None:  # stepper_factory may return None: host-side reset/spec only (CPU oracle legs)
            self._build_views()
        # Saez tax model: the estimator half lives on the host (foundation/saez.py)
        self._saez = None
        tax = self._components_dict.get("PeriodicBracketTax")
        if tax is not None and tax.tax_model == "saez" and self._stepper is not None:
            from .saez import SaezHost
            self._saez = SaezHost(self, tax)

    # ------------------------------------------------------------------ properties (base_env.py:385-437)
    @property
    def episode_length(self):
        return int(self._episode_length)

    @property
    def inv_scale(self):
        return 0.01 if self._allow_observation_scaling else 1

    @property
    def resources(self):
        return sorted(self._entities["resources"])

    @property
    def landmarks(self):
        return sorted(self._entities["landmarks"])

    @property
    def endogenous(self):
        return sorted(self._entities["endogenous"])

    @property
    def all_agents(self):
        return self._agents + [self._planner]

    @property
    def components(self):
        return self._components

    @property
    def world(self):
        return _WorldView(self, 0)

    def world_of(self, e):
        return _WorldView(self, e)

    @property
    def spec(self):
        return dict(self._spec)

    @property
    def stepper(self):
        return self._stepper

    def get_component(self, name):
        if name in self._components_dict:
            return self._components_dict[name]
        if name in self._shorthand_lookup:
            return self._shorthand_lookup[name]
        raise KeyError("No component with name or shorthand name {} found; registered components are:\n\t{}".format(
            name, "\n\t".join(self._components_dict)))

    def get_agent(self, agent_idx):
        agent = self._agent_lookup.get(str(agent_idx))
        if agent is None:
            raise ValueError("No agent with associated index {}".format(agent_idx))
        return agent

    # ------------------------------------------------------------------ seeding (base_env.py:481-494)
    def seed(self, seed):
        """int -> env e is seeded with seed + e (n_envs == 1 reproduces the reference's global seeding);
        a sequence gives each env its own seed."""
        if isinstance(seed, (int, float)):
            seed = int(seed)
            assert seed > 0
            seeds = [seed + e for e in range(self.n_envs)]
        else:
            seeds = [int(s) for s in seed]
            assert len(seeds) == self.n_envs
        self._seeds = seeds
        self._rs = [np.random.RandomState(s) for s in seeds]

    # ------------------------------------------------------------------ reset / step
    def _has_gauss_state(self):
        """numpy's legacy Gaussian cache is part of the record when the device reset draws Gaussians (lognormal skills,
        dynamic layouts): the host stream and the record's copy are kept in step."""
        sp = self._spec
        return sp.get("reset_mode", 0) == 1 and (2 in (sp.get("build_skill_dist", 0), sp.get("gather_skill_dist", 0))
                                                 or bool(sp.get("dyn_layout", 0)))

    def _sync_streams_from_device(self):
        """The device advanced each env's numpy-legacy stream while stepping; continue from there
        (the reference's reset() keeps drawing from the same global stream, base_env.py:896-911)."""
        st = self._stepper
        key = st.to_numpy(st.state_view("mt_key")) if hasattr(st, "state_view") else None
        pos = st.to_numpy(st.state_view("mt_pos")) if hasattr(st, "state_view") else None
        gauss = None
        if key is not None and self._has_gauss_state():
            gauss = st.to_numpy(st.state_view("gauss_state"))   # the device reset may have consumed / refilled the cache
        for e, rs in enumerate(self._rs):
            if key is None:
                d = st.read_state(e)
                k, p = d["mt_key"], int(d["mt_pos"][0])
            else:
                k, p = key[e], int(pos[e])
            s = rs.get_state()
            has_g, val_g = (s[3], s[4]) if gauss is None else (int(gauss[e][1] != 0.0), float(gauss[e][0]))
            rs.set_state((s[0], np.asarray(k, np.uint32), p, has_g, val_g))

    def load_host_state(self, host_state, env_lo=0):
        """Upload host reset snapshots (the arrays `host_reset_arrays()` returns, or a caller's own states in the same
        layout) for replicas [env_lo, env_lo + n) and mark the env ready to step - the public form of what `reset()`
        does after running the host reset (aie_load_state)."""
        self._stepper.load_state(host_state, env_lo=env_lo)
        self._loaded = True
        return self.obs

    def host_reset_arrays(self):
        """Run the reference-faithful host reset for every env; returns the aie_host_state arrays."""
        if self._rs is None:
            self._rs = [np.random.RandomState() for _ in range(self.n_envs)]
        per = []
        for e in range(self.n_envs):
            rs = self._rs[e]
            st = self.scenario.host_reset(rs, e)
            key = rs.get_state()
            st["mt_key"], st["mt_pos"] = np.asarray(key[1], np.uint32), int(key[2])
            st["gauss_has"], st["gauss_val"] = int(key[3]), float(key[4])   # legacy Gaussian cache (lognormal skills)
            st["completions"] = int(self._completions[e])
            per.append(st)
        out = {k: np.stack([np.asarray(p[k]) for p in per]) for k in per[0]}
        return out

    @staticmethod
    def _np_state(seed_state):
        """The 5-tuple np.random.set_state() expects (base_env.py:873-883)."""
        assert isinstance(seed_state, (tuple, list)) and len(seed_state) == 5
        return (str(seed_state[0]), np.array(seed_state[1], dtype=np.uint32), int(seed_state[2]), int(seed_state[3]),
                float(seed_state[4]))

    def stream_state(self, e=0):
        """np.random.get_state() of replica e's stream as it stands now (on the device once the env is loaded)."""
        if self._rs is None:
            self._rs = [np.random.RandomState() for _ in range(self.n_envs)]
        if self._loaded and hasattr(self._stepper, "state_view"):   # only this replica's 2.5 KB key
            st = self._stepper
            key = st.to_numpy(st.state_view("mt_key")[e])
            pos = int(st.to_numpy(st.state_view("mt_pos")[e]))
            s = self._rs[e].get_state()
            has_g, val_g = s[3], s[4]
            if self._has_gauss_state():
                g = st.to_numpy(st.state_view("gauss_state")[e])
                has_g, val_g = int(g[1] != 0.0), float(g[0])
            self._rs[e].set_state((s[0], np.asarray(key, np.uint32), pos, has_g, val_g))
        elif self._loaded:
            self._sync_streams_from_device()
        return self._rs[e].get_state()

    def set_stream_state(self, seed_state, e=0):
        """np.random.set_state(seed_state) for replica e: host stream and, once loaded, the key inside its record."""
        ss = self._np_state(seed_state)
        if self._rs is None:
            self._rs = [np.random.RandomState() for _ in range(self.n_envs)]
        self._rs[e].set_state(ss)
        if self._loaded:
            st = self._stepper
            for name, val in (("mt_key", ss[1].astype(np.int64)), ("mt_pos", ss[2])):
                v = st.state_view(name)
                if isinstance(v, np.ndarray):
                    v[e] = val
                else:
                    import torch
                    v[e] = torch.as_tensor(val, device=v.device).to(v.dtype)
            if self._has_gauss_state():
                g = st.state_view("gauss_state")
                vals = np.array([ss[4], float(ss[3])])
                if isinstance(g, np.ndarray):
                    g[e] = vals
                else:
                    import torch
                    g[e] = torch.as_tensor(vals, device=g.device, dtype=g.dtype)

    def reset(self, seed_state=None, force_dense_logging=False):
        """seed_state: optional numpy stream state(s) to start the reset from (base_env.py:873-884) - one 5-tuple (every
        replica when n_envs == 1, else replica 0) or a list with one 5-tuple per replica."""
        _rg.refuse_in_act(self, "reset")
        if self._rollout is not None and self._stepper.rollout_slot != 0:
            _rg.invalidate(self)   # refused below: the graph's rollout was left mid-way
        if self._loaded and "episode_final" not in self._stepper.buf and self._episode_finished(0):
            # base_env.py:763-765, 1022-1025: _finalize_logs stores the metrics only on the step that ENDS an episode, so
            # resetting an unfinished episode (or resetting twice) leaves previous_episode_metrics untouched
            self._last_ep_metrics_host = self.metrics_of(0, _count_finished=False)
        if self._spec.get("reset_mode", 0) == 1 and hasattr(self._stepper, "reset_envs"):
            return self._reset_on_device(seed_state, force_dense_logging)
        if self._loaded and self._rs is not None:
            self._completions = self.completions()
            self._sync_streams_from_device()
        if seed_state is not None:
            if self._rs is None:
                self._rs = [np.random.RandomState() for _ in range(self.n_envs)]
            per_env = seed_state if (isinstance(seed_state, (tuple, list)) and len(seed_state) == self.n_envs
                                     and isinstance(seed_state[0], (tuple, list))) else [seed_state]
            for e, ss in enumerate(per_env):
                self._rs[e].set_state(self._np_state(ss))
        saez_n = self._saez.before_host_reset() if self._saez is not None else None
        # the "auto" energy warm-up integrator survives resets in the reference (layout_from_file.py:153, 557: only the
        # constructor zeroes it); a host reset repacks the records, so carry it over
        warm = None
        if self._loaded and hasattr(self._stepper, "state_view"):
            warm = self._stepper.to_numpy(self._stepper.state_view("auto_warmup")).copy()
        self._stepper.load_state(self.host_reset_arrays())
        if warm is not None and warm.any():
            v = self._stepper.state_view("auto_warmup")
            if isinstance(v, np.ndarray):
                v[...] = warm
            else:
                import torch
                v.copy_(torch.as_tensor(warm, device=v.device, dtype=v.dtype))
        self._loaded = True
        if self._saez is not None:
            self._saez.after_host_reset(saez_n)
        self._start_dense_log(force_dense_logging, int(self._completions[0]))
        return self.obs

    def _reset_on_device(self, seed_state, force_dense_logging):
        """reset() of a config whose auto-reset is reference-exact: one launch re-draws every replica on the device from
        its own stream (aie_reset_envs) and leaves what the host reset of the same streams would.  Once loaded, nothing of
        size n_envs crosses PCIe (Saez and dense logs aside): the streams, the completion counts and the energy warm-up
        integrators stay in the records, as they do across an auto-reset."""
        if seed_state is not None:
            if self._rs is None:
                self._rs = [np.random.RandomState() for _ in range(self.n_envs)]
            per_env = seed_state if (isinstance(seed_state, (tuple, list)) and len(seed_state) == self.n_envs
                                     and isinstance(seed_state[0], (tuple, list))) else [seed_state]
            for e, ss in enumerate(per_env):
                self.set_stream_state(ss, e)   # once loaded, this also installs the stream in replica e's record
        saez_n = self._saez.before_host_reset() if self._saez is not None else None
        if self._loaded:
            self._stepper.reset_envs()
        else:
            streams = self._host_streams()
            self._stepper.reset_envs(template=self._reset_template(), streams=streams)
            self._loaded = True
        if self._saez is not None:
            self._saez.after_host_reset(saez_n)
        completions0 = 0
        if force_dense_logging or self._create_dense_log_every is not None:
            st = self._stepper
            completions0 = int(st.to_numpy(st.state_view("completions")[0:1])[0])
        self._start_dense_log(force_dense_logging, completions0)
        return self.obs

    def _host_streams(self):
        """Every replica's host stream (after the constructor's draws) in aie_reset_streams' layout."""
        if self._rs is None:
            self._rs = [np.random.RandomState() for _ in range(self.n_envs)]
        states = [rs.get_state() for rs in self._rs]
        out = dict(mt_key=np.stack([np.asarray(s[1], np.uint32) for s in states]),
                   mt_pos=np.array([s[2] for s in states], np.int32),
                   gauss_has=np.array([s[3] for s in states], np.int32),
                   gauss_val=np.array([s[4] for s in states], np.float64))
        out.update(self.scenario.device_reset_tables())
        return out

    def _reset_template(self):
        """The host reset of replica 0 on a copy of its stream, as a one-replica snapshot: the parts of a starting
        record that do not depend on the stream (maps of a fixed layout, coin, water) for every replica; the device
        re-draws the rest."""
        rs = np.random.RandomState()
        rs.set_state(self._rs[0].get_state())
        st = self.scenario.host_reset(rs, 0)
        key = rs.get_state()
        st["mt_key"], st["mt_pos"] = np.asarray(key[1], np.uint32), int(key[2])
        st["gauss_has"], st["gauss_val"] = int(key[3]), float(key[4])
        st["completions"] = int(self._completions[0])
        return {k: np.asarray(v)[None] for k, v in st.items()}

    def _episode_finished(self, e):
        st = self._stepper
        if not hasattr(st, "state_view"):
            return True
        return int(st.to_numpy(st.state_view("t")[e:e + 1])[0]) >= self._episode_length

    def completions(self):
        """Completed episodes per replica (BaseEnvironment._completions, base_env.py:1021-1025: incremented on the step
        that ends an episode).  The device counts an episode when it auto-resets it; a finished episode still waiting
        for an explicit reset() (auto_reset off) is added here."""
        st = self._stepper
        if not self._loaded or not hasattr(st, "state_view"):
            return self._completions
        done_waiting = st.to_numpy(st.state_view("t")).astype(np.int64) >= self._episode_length
        return st.to_numpy(st.state_view("completions")).astype(np.int64) + done_waiting

    # ------------------------------------------------------------------ dense logs (base_env.py:440-452, 763-814)
    @property
    def dense_log(self):
        """The contents of the current (potentially incomplete) dense log of replica 0."""
        return self._dense_logger.log if self._dense_logger is not None else self._dense_log

    @property
    def previous_episode_dense_log(self):
        return self._last_ep_dense_log

    def _start_dense_log(self, force, completions):
        every = self._create_dense_log_every
        on = bool(force) or (every is not None and completions % every == 0)
        if on and getattr(self._stepper, "event_envs", 0) < 1:
            raise RuntimeError("dense logging needs dense_log_frequency to be set at construction (event buffer)")
        from .dense_log import DenseLogger
        self._dense_logger = DenseLogger(self, 0, self._world_dense_log_frequency) if on else None
        self._dense_log = {"world": [], "states": [], "actions": [], "rewards": []}

    def _write_actions(self, actions):
        st = self._stepper
        buf_a, buf_p = self.action_buffers
        if actions is None:
            buf_a[...] = 0
            buf_p[...] = 0
            return
        if isinstance(actions, dict):
            buf_a[...] = 0
            buf_p[...] = 0
            for k, v in actions.items():
                k = str(k)
                if k == "p":
                    if st.dims.n_act_planner:
                        buf_p[...] = self._as_buf(v, buf_p, (self.n_envs, st.dims.n_act_planner))
                else:
                    i = int(k)
                    buf_a[:, i, :] = self._as_buf(v, buf_a, (self.n_envs, st.dims.n_act_agent))
            return
        a, p = actions if isinstance(actions, (tuple, list)) and len(actions) == 2 else (actions, None)
        if a is not buf_a:
            buf_a[...] = self._as_buf(a, buf_a, tuple(buf_a.shape))
        if p is not None and p is not buf_p and st.dims.n_act_planner:
            buf_p[...] = self._as_buf(p, buf_p, tuple(buf_p.shape))

    @staticmethod
    def _as_buf(v, like, shape):
        if isinstance(like, np.ndarray):
            return np.asarray(v, dtype=like.dtype).reshape(shape)
        import torch
        if isinstance(v, torch.Tensor):
            return v.to(device=like.device, dtype=like.dtype).reshape(shape)
        return torch.as_tensor(np.asarray(v, dtype=np.int32), device=like.device).reshape(shape)

    def step(self, actions=None, seed_state=None):
        """actions: None (all NO-OP) | reference-style dict {agent_idx: action(s)} with a leading env axis |
        tensor [E, A, n_act] | (agent_actions, planner_actions).  Writing straight into
        `env.action_buffers` and calling step(env.action_buffers) avoids any copy."""
        _rg.refuse_in_act(self, "step")
        assert self._loaded, "call reset() first"
        self._write_actions(actions)
        lg = self._dense_logger
        if lg is not None:
            st = self._stepper
            lg.before_step(st.to_numpy(st.buf["actions_agent"][0]), st.to_numpy(st.buf["actions_planner"][0])
                           if st.dims.n_act_planner else None)
        self._stepper.step()
        if self._rollout is not None:
            self._aim_rollout()
        if self._saez is not None:
            self._saez.after_step()
        if lg is not None:
            st = self._stepper
            ended = bool(int(st.to_numpy(st.buf["done"][0])))
            post = st.read_state(0, final=True) if (ended and self._auto_reset) else st.read_state(0)
            lg.after_step(st.to_numpy(st.buf["reward"][0]), post)
            if ended:  # _finalize_logs; under auto-reset the next episode of replica 0 has already begun
                self._last_ep_dense_log = lg.finalize(post)
                self._dense_logger = None
                if self._auto_reset:
                    self._start_dense_log(False, int(st.read_state(0)["completions"][0]))
        return self.obs, self.rew, self.done, self.info

    @property
    def action_buffers(self):
        if self._rollout is not None:
            return self._rollout.actions[min(self._stepper.rollout_slot, self._rollout.T - 1)]
        return self._stepper.buf["actions_agent"], self._stepper.buf["actions_planner"]

    # ------------------------------------------------------------------ rollouts stored in place
    def bind_rollout(self, T, final_obs=False):
        """Store the next rollouts of T steps in place: returns a rollout object whose device tensors the kernels write
        directly (include/aie_b200.h, aie_bind_rollout), so the loop copies nothing per step.

        rollout.buf: every observation / mask tensor [T + 1, E, ...] (slot t: the observation step t's action is taken
        from, slot T: the one after the last step), actions_agent / actions_planner [T, E, ...], reward [T, E, A + 1],
        done [T, E]; with final_obs (needs auto_reset) final_<name> [K, E, ...], K = ceil(T / episode_length), row
        (k, e) the observation of the state in which replica e's k-th episode end within the rollout ended.
        rollout.obs[t] / rollout.final_obs[k] are the named views env.obs / env.final_obs build, rollout.rew[t] /
        rollout.done[t] / rollout.actions[t] those of env.rew, env.done and env.action_buffers, all built here once.

        While bound, with the slot cursor s (0 here and after restart_rollout()): env.obs / env.obs_tensors and
        env.action_buffers show slot s (sample_actions writes there), env.rew / env.done the latest step's slot s - 1
        (slot 0 before the first step), and step() advances s.  env.final_obs / env.final_obs_tensors are not written
        while a rollout is bound (they keep what they held): the final observations go to rollout.final_obs.  reset() is allowed only at s == 0 and writes the first
        observations into slot 0.  After T steps call restart_rollout(), which carries slot T into slot 0.
        unbind_rollout() returns to the env's own buffers.  Dense logging (it reads replica 0's bound action, reward
        and done buffers) is refused with a ValueError, a stepper_factory whose stepper cannot bind rollouts with
        NotImplementedError."""
        _rg.refuse_in_act(self, "bind_rollout")
        _rg.invalidate(self)
        st = self._stepper
        if not hasattr(st, "bind_rollout"):
            raise NotImplementedError("this env's stepper cannot bind rollouts")
        if self._create_dense_log_every is not None or self._dense_logger is not None:
            raise ValueError("bind_rollout: dense logging reads the env's own action, reward and done buffers; "
                             "construct the env without dense_log_frequency")
        if final_obs and not self._auto_reset:
            raise ValueError("final_obs=True needs auto_reset=True")
        if self._rollout is not None:
            raise ValueError("a rollout is already bound: unbind_rollout() first")
        r = st.bind_rollout(T, final_obs=final_obs)
        b, A = r.buf, self.n_agents
        slot = lambda t: {k: b[k][t] for k in r.obs_names}
        r.obs = [self._obs_views(slot(t)) for t in range(r.T + 1)]
        r.obs_slots = [slot(t) for t in range(r.T + 1)]
        r.final_obs = [self._obs_views({k: b["final_" + k][k_] for k in r.obs_names}) for k_ in range(r.K)] \
            if final_obs else None
        r.actions = [(b["actions_agent"][t], b["actions_planner"][t]) for t in range(r.T)]
        if self.collate_agent_step_and_reset_data:
            r.rew = [{"a": b["reward"][t][:, :A], "p": b["reward"][t][:, A]} for t in range(r.T)]
        else:
            r.rew = [dict({str(i): b["reward"][t][:, i] for i in range(A)}, p=b["reward"][t][:, A]) for t in range(r.T)]
        r.done = [{"__all__": b["done"][t]} for t in range(r.T)]
        self._rollout = r
        self._aim_rollout()
        return r

    def restart_rollout(self):
        """Start the next rollout in the bound tensors (after its T steps): slot T's observations move to slot 0."""
        _rg.refuse_in_act(self, "restart_rollout")
        if self._rollout is None:
            raise ValueError("no rollout bound")
        self._stepper.restart_rollout()
        self._aim_rollout()

    def capture_rollout(self, act):
        """Record the bound rollout's T steps once as a CUDA graph and return a RolloutGraph whose replay() runs them
        again: for t in range(T), act(t, rollout.obs_slots[t]) then step(env.action_buffers).

        act: the policy's part of a step, torch ops on the env's device plus at most sample_actions (any other env call
        inside it is a ValueError).  It must not synchronise with the host or branch on device values, and its outputs
        should go to tensors that outlive the capture (e.g. per-slot rows of the trainer's buffers).  Needs a bound
        rollout at slot 0 after reset(), and the CUDA stepper (NotImplementedError otherwise).  Before recording, act
        runs once at slot 0 as torch's warm-up; the sampler's draws and the slot's actions it wrote are given back.
        Recording executes nothing: the env's counters, cursor and buffers are as they were before the call.

        replay() needs cursor 0 (after reset() or restart_rollout()) and leaves it at T, with every output what the
        eager loop leaves from the same state, byte for byte, when act is bit-reproducible under capture: the policy
        sampler reads its call count on the device, so draws differ from replay to replay as they do eagerly; the seed
        passed to sample_actions is fixed at capture.  Tensors are read by address, so in-place updates of the policy's
        weights are seen.  Eager rollouts may run between replays.  Unbinding or re-binding the rollout,
        load_state_dict() and reset() attempted mid-rollout invalidate the graph (replay() raises ValueError), as does
        capturing again.  Refused with ValueError under the Saez tax model, whose host-side estimator runs after every
        step.  The launch count includes the warm-up's launches."""
        if self._saez is not None:
            raise ValueError("capture_rollout: the Saez tax model runs its estimator on the host after every step")
        return _rg.capture_rollout(self, act)

    def unbind_rollout(self):
        """Back to the env's own buffers (env.obs, env.rew, ... as before bind_rollout)."""
        _rg.refuse_in_act(self, "unbind_rollout")
        _rg.invalidate(self)
        if self._rollout is None:
            return
        self._stepper.unbind_rollout()
        self._rollout = None
        self._build_views()

    @property
    def rollout(self):
        """The bound rollout object, or None."""
        return self._rollout

    def _aim_rollout(self):
        r, s = self._rollout, self._stepper.rollout_slot
        self.obs, self.obs_tensors = r.obs[s], r.obs_slots[s]
        self.rew, self.done = r.rew[max(s - 1, 0)], r.done[max(s - 1, 0)]

    def sample_actions(self, logits_agent, logits_planner=None, *, seed, greedy=False, out=None):
        """A policy's actions, drawn on the device into `action_buffers` (then step(env.action_buffers) consumes them).

        One categorical per mask segment of every replica: the whole mask row of a single-action agent, each subspace of
        a multi-action agent (with its own NO-OP), each planner bracket (or the single-action planner's one index), from
        the softmax of the logits restricted to the open entries of the current masks (env.obs_tensors["mask_*"]).
        logits_agent: [E, A, Na] laid out like mask_agent; logits_planner: [E, Np] like mask_planner, required when the
        config has planner actions (ignored otherwise).  Contiguous float32 or bfloat16 (the same for both) on the env's
        device, whatever obs_dtype is.  greedy=True: the masked argmax (evaluation).  The draws are a function of
        (seed, number of earlier sample_actions calls, replica, agent, segment).  Returns (log_prob_agent [E, A, n_act],
        log_prob_planner [E, n_act_p] or None), float32: buffers of the env reused by the next call, or the caller's
        `out` = (log_prob_agent, log_prob_planner) tensors (e.g. a rollout slot; either may be None).  Asynchronous."""
        return self._stepper.sample_policy(logits_agent, logits_planner, seed=seed, greedy=greedy, out=out)

    def evaluate_actions(self, logits_agent, logits_planner, actions, masks):
        """Log-probabilities and entropies of stored actions under the masks they were drawn with, for the update pass:
        (log_prob_agent, log_prob_planner, entropy_agent, entropy_planner), float32, shaped like the actions (the
        planner entries are None without planner actions).

        The segments are sample_actions's, and so is the arithmetic: a log-probability is bit for bit what
        sample_actions returned for the same logits, masks and action.  logits_agent: [*B, A, Na], logits_planner:
        [*B, Np] (ignored without planner actions), one dtype, float32 or bfloat16; masks = (mask_agent [*B, A, Na],
        mask_planner [*B, Np]) as the env wrote them (obs_tensors["mask_*"] at sampling time), float32 or bfloat16;
        actions = (actions_agent [*B, A, n_act], actions_planner [*B, n_act_p]), int32.  *B is any leading shape,
        e.g. a minibatch of stored rollout steps; every tensor contiguous on the env's device.  Differentiable with
        respect to both logits tensors: the backward is one device launch that recomputes the softmax.  A segment
        with nothing open gives 0 and 0 (gradient 0); a NaN or +inf open logit, no finite open logit, or a stored
        action that is closed gives NaN (see include/aie_b200.h).  Asynchronous; the env's state is not touched."""
        _rg.refuse_in_act(self, "evaluate_actions")
        return self._stepper.evaluate_actions(logits_agent, logits_planner, actions, masks)

    def compute_advantages(self, rewards, values, dones, last_values, final_values=None, *, gamma, lam=1.0,
                           per_episode_end=False):
        """Advantages and value targets of a stored rollout of T steps (generalised advantage estimation), bootstrapped
        at episode ends: (adv_agent [T, E, A], adv_planner [T, E], ret_agent, ret_planner), float32, one device launch.

        rewards = (agent [T, E, A], planner [T, E]) as the env wrote them after each step (rew["a"] / rew["p"] with
        collated data), float32 or float64; values = (agent, planner), float32, the value of the observation each
        step's action was taken from; dones = int32 [T, E], done["__all__"] after each step; last_values = (agent
        [E, A], planner [E]), float32, the value of the observation after the last step.  Every episode here ends on its
        time limit, and the auto-reset hands back the next episode's observation at the step that ends one, so the
        target of a done step should bootstrap from the value of that step's env.final_obs: pass those values as
        final_values = (agent, planner) shaped like values (rows where dones is 0 are never read, so the value net's
        output over the whole final_obs tensor will do).  final_values=None treats an episode end as terminal.  gamma,
        lam: floats in [0, 1] or (agents, planner) pairs.  The planner entries may be None together (a trainer without
        a planner policy; its outputs are then None).  Computed in float64 exactly as include/aie_b200.h spells out.
        Every tensor contiguous on the env's device; asynchronous on the current stream; the env's state is not touched.

        A bound rollout's storage is taken as it is: rewards = rollout.buf["reward"] [T, E, A + 1] (split here with one
        copy per group), dones = rollout.buf["done"], and with per_episode_end=True final_values [K, E, A] / [K, E], the
        values of the final slots: a done step reads the row of its episode-end ordinal in its replica (0 for the first)."""
        _rg.refuse_in_act(self, "compute_advantages")
        return self._stepper.compute_advantages(rewards, values, dones, last_values, final_values, gamma=gamma, lam=lam,
                                                per_episode_end=per_episode_end)

    # ------------------------------------------------------------------ checkpoints
    def _checkpoint_config(self):
        """What a checkpoint must have been taken from to load into this env (load_state_dict checks each field)."""
        from .._abi import ABI_VERSION
        return dict(scenario=self.name, n_envs=self.n_envs, obs_dtype=self._spec["obs_dtype"], auto_reset=self._auto_reset,
                    final_obs=self._spec["final_obs"],
                    dense_log=[self._create_dense_log_every, self._world_dense_log_frequency], abi_version=ABI_VERSION,
                    spec=self._spec)

    def _checkpoint_buffers(self):
        """name -> the buffer a checkpoint holds: the records, the event log, and the action / reward / done tensors
        env.action_buffers / env.rew / env.done show (slot 0 of a bound rollout)."""
        st = self._stepper
        out = {k: st.buf[k] for k in ("state", "state0", "episode_final", "events") if k in st.buf}
        out["actions_agent"], out["actions_planner"] = self.action_buffers
        if self._rollout is None:
            out["reward"], out["done"] = st.buf["reward"], st.buf["done"]
        else:
            out["reward"], out["done"] = self._rollout.buf["reward"][0], self._rollout.buf["done"][0]
        if self._saez is not None:
            # the host writes a new tax period's rates into the records after the step that observed the old ones, so the
            # stand-alone pass would show the agents' marginal rates under the new rates: keep the step's observations
            out.update(self.obs_tensors)
        return out

    def state_dict(self):
        """The whole state of the batched env between steps, for resuming a run bit for bit: a dict of tensors (copies
        on the env's device), numpy arrays and plain Python values that torch.save can write.  It holds every replica's
        state record, its auto-reset snapshot and end-of-episode record, the action / reward / done buffers, the
        library's sampler counters and fused-policy key, the completion counts, the Saez estimator, the dense log being
        recorded and the host-side tables drawn at construction.  Observations are not stored (except under the Saez
        tax model): load_state_dict() re-derives them from the records.  Allowed after the first reset(); with a rollout
        bound only at slot 0 (ValueError otherwise)."""
        _rg.refuse_in_act(self, "state_dict")
        from . import checkpoint as ck
        if not self._loaded:
            raise ValueError("state_dict: nothing to save before the first reset()")
        ck.refuse_mid_rollout(self, "state_dict")
        if not hasattr(self._stepper, "get_counters"):
            raise NotImplementedError("this env's stepper keeps no checkpointable counters")
        buffers = {k: ck.snapshot(v) for k, v in self._checkpoint_buffers().items()}
        rs = self._rs if self._rs is not None else []
        host = dict(completions=self._completions.copy(), last_ep_metrics=getattr(self, "_last_ep_metrics_host", None),
                    gauss_has=np.array([s.get_state()[3] for s in rs], np.int64),
                    gauss_val=np.array([s.get_state()[4] for s in rs], np.float64),
                    dense_log=self._dense_log, last_ep_dense_log=self._last_ep_dense_log, dense_logger=None,
                    saez=self._saez.state_dict() if self._saez is not None else None)
        lg = self._dense_logger
        if lg is not None:
            host["dense_logger"] = dict(log=lg.log, comp=lg.comp, paid_prev=lg._paid_prev, static=lg._static)
        # host tables drawn from the seeded streams at construction (a resumed env is made with other seeds)
        if hasattr(self.scenario, "_split_ranked_skill"):
            host["split_ranked_skill"] = self.scenario._split_ranked_skill
        labor = self._components_dict.get("SimpleLabor")
        if labor is not None:
            host["labor_skills"] = labor.skills
        return dict(format_version=ck.FORMAT_VERSION, config=ck.plain(self._checkpoint_config()), buffers=buffers,
                    counters=self._stepper.get_counters(), host=ck.host_copy(host))

    def load_state_dict(self, sd):
        """Load a state_dict() taken from an env of the same configuration (scenario, numeric spec, n_envs, obs_dtype,
        auto_reset, final_obs, dense-log settings, ABI and format version: ValueError naming the field otherwise) into
        this env's own buffers, then re-derive the observations (and, with final_obs and no rollout bound, the final
        observations of the replicas whose done flag is set) with the stand-alone observation pass.  Returns env.obs.
        From here on every call returns what
        it would have returned in the env the dict was taken from.  Allowed on a new env before any reset(), and between
        steps; with a rollout bound only at slot 0 (the observations go into slot 0)."""
        _rg.refuse_in_act(self, "load_state_dict")
        _rg.invalidate(self)
        from . import checkpoint as ck
        ck.check_config(sd, self._checkpoint_config())
        ck.refuse_mid_rollout(self, "load_state_dict")
        st = self._stepper
        mine = self._checkpoint_buffers()
        if set(sd["buffers"]) != set(mine):
            raise ValueError("load_state_dict: the checkpoint holds buffers %s, this env %s"
                             % (sorted(sd["buffers"]), sorted(mine)))
        for k, dst in mine.items():
            ck.copy_into(dst, sd["buffers"][k], k)
        host = ck.host_copy(sd["host"])
        counters = dict(sd["counters"])
        # the stand-alone pass would draw the fused random policy's next actions over the restored ones: run it with the
        # policy off, then restore the key
        st.set_counters(dict(counters, fused_policy_key=0, fused_policy_on=0))
        if self._saez is None:
            st.observe()
        if self._rollout is None and getattr(st, "final_obs", False):
            st.observe_final()
        st.set_counters(counters)
        self._loaded = True
        self._completions = np.asarray(host["completions"], np.int64).copy()
        if host["last_ep_metrics"] is not None:
            self._last_ep_metrics_host = host["last_ep_metrics"]
        elif hasattr(self, "_last_ep_metrics_host"):
            del self._last_ep_metrics_host
        if self._rs is None:
            self._rs = [np.random.RandomState() for _ in range(self.n_envs)]
        for rs, has, val in zip(self._rs, host["gauss_has"], host["gauss_val"]):
            s = rs.get_state()   # the key and position are the record's (synchronised before every host use)
            rs.set_state((s[0], s[1], s[2], int(has), float(val)))
        if "split_ranked_skill" in host:
            self.scenario._split_ranked_skill = np.asarray(host["split_ranked_skill"], np.float64)
        if "labor_skills" in host:
            self._components_dict["SimpleLabor"].skills = np.asarray(host["labor_skills"])
        if self._saez is not None:
            self._saez.load_state_dict(host["saez"])
        self._dense_log, self._last_ep_dense_log = host["dense_log"], host["last_ep_dense_log"]
        self._dense_logger = None
        if host["dense_logger"] is not None:
            from .dense_log import DenseLogger
            lg = self._dense_logger = DenseLogger(self, 0, self._world_dense_log_frequency)
            d = host["dense_logger"]
            lg.log, lg.comp, lg._paid_prev, lg._static = d["log"], d["comp"], d["paid_prev"], d["static"]
        return self.obs

    # ------------------------------------------------------------------ outputs
    @staticmethod
    def _named_fields(flat, layout):
        """{key: slice of the flat vector} (scalars lose the trailing axis), base_env.py:562-612 undone."""
        return {k: (flat[..., off] if n == 1 else flat[..., off:off + n]) for k, off, n in layout if k != "time"}

    def _mask_dict(self, agent, flat_mask):
        """{subspace name: slice of the flat mask} (base_env.py:706-756 with flatten_masks=False)."""
        out, off = {}, 0 if agent.multi_action_mode else 1
        for name in agent._action_names:
            k = int(agent.action_dim[name])
            if agent.multi_action_mode:
                out[name] = flat_mask[..., off + 1:off + k]   # the subspace's own NO-OP leads its slice
            else:
                out[name] = flat_mask[..., off:off + k]
            off += k
        # quirk kept: a PeriodicBracketTax with a fixed schedule falls back to BaseComponent.generate_masks, which
        # hands every agent type an EMPTY mask for its 0 actions (base_component.py:303-317, redistribution.py:1100-1102)
        tax = self._components_dict.get("PeriodicBracketTax")
        if tax is not None and tax.tax_model != "model_wrapper" and not tax.disable_taxes:
            out[tax.name] = flat_mask[..., 0:0]
        return out

    def _build_views(self):
        b = self._stepper.buf
        A = self.n_agents
        self.obs_tensors = {k: b[k] for k in b if k.startswith("obs_") or k.startswith("mask_")}
        self.obs = self._obs_views(b)
        self.rew = {str(i): b["reward"][:, i] for i in range(A)}
        self.rew["p"] = b["reward"][:, A]
        self.done = {"__all__": b["done"]}
        self.info = {k: {} for k in self.obs}
        if self.collate_agent_step_and_reset_data:
            self.rew = {"a": b["reward"][:, :A], "p": b["reward"][:, A]}
            self.info = {"a": {str(i): {} for i in range(A)}, "p": {}}
        # final_obs=True: env.final_obs / env.final_obs_tensors mirror env.obs / env.obs_tensors over the final_<name>
        # buffers.  After a step, row e of a replica with done["__all__"][e] == 1 holds the observation of the state its
        # episode ended in (env.obs already shows the next episode's first); the other rows are unspecified (they keep
        # whatever an earlier episode end wrote).  reset() does not touch them.  None when final_obs is off.
        self.final_obs_tensors = self.final_obs = None
        if getattr(self._stepper, "final_obs", False):
            self.final_obs_tensors = {k: b["final_" + k] for k in self.obs_tensors}
            self.final_obs = self._obs_views(self.final_obs_tensors)

    def _obs_views(self, b):
        """The nested observation dict (keys and views as the reference's step returns them) over the observation / mask
        buffers `b` (name -> tensor): the live ones, or their final_<name> twins."""
        A = self.n_agents
        flat_o, flat_m = self._flatten_observations, self._flatten_masks
        if not flat_o:
            st = self._stepper
            lay_a, lay_p, lay_pa = st.flat_layout("agent"), st.flat_layout("planner"), st.flat_layout("planner_agent")
        obs = {}
        spatial = int(self._spec.get("scenario_kind", 0)) != 1   # the one-step-economy has no spatial observations at all
        for i in range(A):
            obs[str(i)] = {"time": b["obs_time"]}
            if spatial:
                obs[str(i)].update({"world-map": b["obs_agent_map"][:, i], "world-idx_map": b["obs_agent_idx"][:, i]})
            if flat_o:
                obs[str(i)]["flat"] = b["obs_agent_flat"][:, i]
            else:
                obs[str(i)].update(self._named_fields(b["obs_agent_flat"][:, i], lay_a))
            obs[str(i)]["action_mask"] = b["mask_agent"][:, i] if flat_m else \
                self._mask_dict(self._agents[i], b["mask_agent"][:, i])
        p = {"time": b["obs_time"]}
        if flat_o:
            p["flat"] = b["obs_planner_flat"]
        else:
            p.update(self._named_fields(b["obs_planner_flat"], lay_p))
        p["action_mask"] = b["mask_planner"] if flat_m else self._mask_dict(self._planner, b["mask_planner"])
        if "obs_planner_map" in b:
            p["world-map"], p["world-idx_map"] = b["obs_planner_map"], b["obs_planner_idx"]
        for i in range(A if self._stepper.dims.flat_planner_agent else 0):   # (no p<i> with full observability and no tax)
            p["p%d" % i] = b["obs_planner_agents"][:, i] if flat_o else \
                self._named_fields(b["obs_planner_agents"][:, i], lay_pa)
        obs["p"] = p
        if self.collate_agent_step_and_reset_data:
            # base_env.py:816-850: the agents' entries are stacked under "a" with the agent axis LAST
            # ([E, ..., A]); these are strided views of the same [E, A, ...] device tensors, no copy
            def last(t):
                return t.movedim(1, -1) if hasattr(t, "movedim") else np.moveaxis(t, 1, -1)
            time_a = b["obs_time"].reshape(self.n_envs, 1)
            time_a = time_a.expand(self.n_envs, A) if hasattr(time_a, "expand") else np.broadcast_to(time_a, (self.n_envs, A))
            if not (flat_o and flat_m):
                raise NotImplementedError("collate_agent_step_and_reset_data needs flattened observations and masks")
            obs = {"a": {"flat": last(b["obs_agent_flat"]), "time": time_a, "action_mask": last(b["mask_agent"])},
                   "p": obs["p"]}
            if spatial:
                obs["a"].update({"world-map": last(b["obs_agent_map"]), "world-idx_map": last(b["obs_agent_idx"])})
        return obs

    def reference_view(self, e=0):
        """(obs, rew, done) of env e as nested numpy dicts in the reference's layout."""
        o = self._stepper.read_obs(e)
        A = self.n_agents
        obs = {}
        spatial = int(self._spec.get("scenario_kind", 0)) != 1
        for i in range(A):
            obs[str(i)] = {"flat": o["a_flat"][i], "time": o["time"].astype(np.float64), "action_mask": o["a_mask"][i]}
            if spatial:
                obs[str(i)].update({"world-map": o["a_map"][i], "world-idx_map": o["a_idx"][i]})
        obs["p"] = {"flat": o["p_flat"], "time": o["time"].astype(np.float64), "action_mask": o["p_mask"]}
        if "p_map" in o:
            obs["p"]["world-map"], obs["p"]["world-idx_map"] = o["p_map"], o["p_idx"]
        for i in range(A if o["p_agents"].shape[-1] else 0):
            obs["p"]["p%d" % i] = o["p_agents"][i]
        rew = {str(i): float(o["rew"][i]) for i in range(A)}
        rew["p"] = float(o["rew"][A])
        return obs, rew, {"__all__": bool(o["done"][0])}

    def _agent_state(self, idx, e):
        d = self._stepper.read_state(e)
        if idx == "p":
            return dict(inventory={r: 0 for r in self.resources}, escrow={r: 0 for r in self.resources}, endogenous={})
        i = int(idx)
        return dict(loc=[int(d["loc"][i, 0]), int(d["loc"][i, 1])],
                    inventory={"Coin": float(d["coin"][i]), "Stone": int(d["inv"][i, 0]), "Wood": int(d["inv"][i, 1])},
                    escrow={"Coin": float(d["esc_coin"][i]), "Stone": int(d["esc"][i, 0]), "Wood": int(d["esc"][i, 1])},
                    endogenous={"Labor": float(d["labor"][i])})

    @property
    def metrics(self):
        """The combined scenario + component metrics of env 0 (BaseEnvironment.metrics, base_env.py:421-432)."""
        _rg.refuse_in_act(self, "metrics")
        return self.metrics_of(0)

    def metrics_of(self, e, _count_finished=True):
        """`env.metrics` of replica e: layout_from_file.py:595-650 + every component's get_metrics(), computed from the
        replica's state record (the event logs are device-side running sums, see foundation/metrics.py)."""
        _rg.refuse_in_act(self, "metrics_of")
        from .metrics import metrics_from_state
        st = self._stepper.read_state(e)
        if _count_finished and int(np.asarray(st["t"]).reshape(-1)[0]) >= self._episode_length:
            # a finished episode waiting for its reset(): the reference has already counted it (base_env.py:1021-1025),
            # which shows in the completion-driven labor/weighted_cost
            st = dict(st)
            st["completions"] = np.asarray(st["completions"]) + 1
        return metrics_from_state(self._spec, st,
                                  saez_elasticity=self._saez.est[e].elas_tm1 if self._saez is not None else None)

    @property
    def previous_episode_metrics(self):
        """Metrics of the episode env 0 finished last (base_env.py:414-418); None before the first auto-reset."""
        _rg.refuse_in_act(self, "previous_episode_metrics")
        return self.previous_episode_metrics_of(0)

    def previous_episode_metrics_of(self, e):
        _rg.refuse_in_act(self, "previous_episode_metrics_of")
        from .metrics import metrics_from_state
        st = self._stepper
        if "episode_final" not in st.buf:   # no auto-reset: what the last explicit reset() stored (replica 0 only)
            return getattr(self, "_last_ep_metrics_host", None) if e == 0 else None
        fin = st.read_state(e, final=True)
        if int(fin["t"][0]) == 0:   # nothing recorded yet
            return None
        return metrics_from_state(self._spec, fin, saez_elasticity=self._saez.elas_at_episode_end[e]
                                  if self._saez is not None else None)

    # ------------------------------------------------------------------ batched metrics (one launch for every replica)
    @property
    def metric_keys(self):
        """Column order of metrics_tensor() / previous_episode_metrics_tensor(): the keys of metrics_of(e), in order."""
        return [k for k, _ in self._stepper.metric_layout()]

    def metrics_tensor(self, out=None):
        """`env.metrics` of every replica as one float64 tensor [n_envs, K] on the device (columns: metric_keys), computed
        by one kernel launch with no synchronisation and no host copy; row e equals metrics_of(e).  A training loop reads
        the curves it logs (productivity, equality, trades, tax rates) without stalling the stream, e.g.
        `env.metrics_tensor()[:, env.metric_keys.index("social/productivity")].mean()`.  out: an optional preallocated
        contiguous float64 [n_envs, K] tensor."""
        _rg.refuse_in_act(self, "metrics_tensor")
        m = self._stepper.episode_metrics(final=False, out=out)
        if self._saez is not None:
            self._fill_saez_elasticity(m, np.asarray(self._saez.batch.elas_tm1, np.float64))
        return m

    def previous_episode_metrics_tensor(self, out=None):
        """previous_episode_metrics of every replica as one float64 tensor [n_envs, K] (columns: metric_keys): the
        metrics of the episode each replica finished last, NaN in every column for a replica that has finished none.
        Needs auto_reset (the end-of-episode records); without it the library's AieError is raised.  Training-loop idiom,
        the metrics of the episodes that ended in this step with no synchronisation until the caller reduces them:
            m = env.previous_episode_metrics_tensor(); logged = m[env.done["__all__"].bool()]"""
        _rg.refuse_in_act(self, "previous_episode_metrics_tensor")
        m = self._stepper.episode_metrics(final=True, out=out)
        if self._saez is not None:
            ends = self._saez.elas_at_episode_end
            self._fill_saez_elasticity(m, np.array([np.nan if v is None else v for v in ends], np.float64), keep_nan_rows=True)
        return m

    def _fill_saez_elasticity(self, m, values, keep_nan_rows=False):
        """The Saez estimator runs on the host: its elasticity column is filled with one host-to-device copy of E doubles.
        keep_nan_rows: rows the device wrote as all NaN (no finished episode) stay NaN."""
        keys = self.metric_keys
        col = keys.index("PeriodicTax/saez/estimated_elasticity")
        if isinstance(m, np.ndarray):
            m[:, col] = np.where(np.isnan(m[:, 0]), np.nan, values) if keep_nan_rows else values
            return
        import torch
        v = torch.as_tensor(values).to(m.device)
        m[:, col] = torch.where(torch.isnan(m[:, 0]), m[:, col], v) if keep_nan_rows else v

    def metrics_rows_as_dicts(self, rows, envs=None):
        """Rows of metrics_tensor() / previous_episode_metrics_tensor() ([n, K], tensor or array) back as the dicts
        metrics_of(e) / previous_episode_metrics_of(e) return: same key order, ints as int, NaN as float("nan"); a row
        that is NaN in every column (no finished episode yet) becomes None.  envs: the row indices to convert (default:
        all).  Copies the rows to the host, i.e. synchronises with the stream that produced them."""
        a = rows.detach().cpu().numpy() if hasattr(rows, "detach") else np.asarray(rows)
        a = np.asarray(a, np.float64).reshape(-1, a.shape[-1])
        layout = self._stepper.metric_layout()
        out = []
        for e in (range(a.shape[0]) if envs is None else envs):
            r = a[int(e)]
            if np.isnan(r).all():
                out.append(None)
                continue
            out.append({k: (int(v) if is_int else float(v)) for (k, is_int), v in zip(layout, r.tolist())})
        return out
