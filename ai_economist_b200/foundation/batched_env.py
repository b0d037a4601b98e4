"""BatchedFoundationEnv — the Gym-style reset/step surface of the reference's BaseEnvironment
(base/base_env.py:24-1120), over E env replicas that live on one GPU.

Differences from the reference API (all additive):
  * new kwargs `n_envs`, `device`, `seeds`, `auto_reset`, `device_reset`;
  * observations / rewards / done are persistent device tensors with a leading env axis, keyed exactly like
    the reference's dicts ("0".."n-1", "p"; "world-map", "world-idx_map", "flat", "action_mask", "time", "p<i>");
  * `reference_view(e)` re-creates the reference's nested numpy dict for one env (tests / debugging).
"""
import ctypes as C

import numpy as np

from .agents import agent_registry
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
                 **scenario_kwargs):
        # ---- base_env.py:178-366 argument checks ----
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
        self._spec = spec

        # ---- dense logging (base_env.py:273-283): replica 0, every dense_log_frequency-th episode ----
        self._create_dense_log_every = None if dense_log_frequency is None else int(dense_log_frequency)
        assert self._create_dense_log_every is None or self._create_dense_log_every >= 1
        self._world_dense_log_frequency = int(world_dense_log_frequency)
        assert self._world_dense_log_frequency >= 1
        self._dense_logger = None
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
        if self._loaded and "episode_final" not in self._stepper.buf and self._episode_finished(0):
            # base_env.py:763-765, 1022-1025: _finalize_logs stores the metrics only on the step that ENDS an episode, so
            # resetting an unfinished episode (or resetting twice) leaves previous_episode_metrics untouched
            self._last_ep_metrics_host = self.metrics_of(0, _count_finished=False)
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
        buf_a, buf_p = st.buf["actions_agent"], st.buf["actions_planner"]
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
        assert self._loaded, "call reset() first"
        self._write_actions(actions)
        lg = self._dense_logger
        if lg is not None:
            st = self._stepper
            lg.before_step(st.to_numpy(st.buf["actions_agent"][0]), st.to_numpy(st.buf["actions_planner"][0])
                           if st.dims.n_act_planner else None)
        self._stepper.step()
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
        return self._stepper.buf["actions_agent"], self._stepper.buf["actions_planner"]

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
        self.rew = {str(i): b["reward"][:, i] for i in range(A)}
        self.rew["p"] = b["reward"][:, A]
        self.done = {"__all__": b["done"]}
        self.info = {k: {} for k in obs}
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
            self.rew = {"a": b["reward"][:, :A], "p": b["reward"][:, A]}
            self.info = {"a": {str(i): {} for i in range(A)}, "p": {}}
        self.obs = obs

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
        return self.metrics_of(0)

    def metrics_of(self, e, _count_finished=True):
        """`env.metrics` of replica e: layout_from_file.py:595-650 + every component's get_metrics(), computed from the
        replica's state record (the event logs are device-side running sums, see foundation/metrics.py)."""
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
        return self.previous_episode_metrics_of(0)

    def previous_episode_metrics_of(self, e):
        from .metrics import metrics_from_state
        st = self._stepper
        if "episode_final" not in st.buf:   # no auto-reset: what the last explicit reset() stored (replica 0 only)
            return getattr(self, "_last_ep_metrics_host", None) if e == 0 else None
        fin = st.read_state(e, final=True)
        if int(fin["t"][0]) == 0:   # nothing recorded yet
            return None
        return metrics_from_state(self._spec, fin, saez_elasticity=self._saez.elas_at_episode_end[e]
                                  if self._saez is not None else None)
