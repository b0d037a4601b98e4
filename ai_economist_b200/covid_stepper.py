"""Python driver of the COVID-19 scenario kernels (plumbing: buffers + ABI calls)."""
import ctypes as C
import numbers

import numpy as np

from . import _abi
from .stepper import PolicySampler, Rollout, bf16_bits_to_float32, buf_kind_torch, float_kind_torch, is_i32_torch

F32, I32 = np.float32, np.int32


def covid_config_from_params(p, auto_reset=True, obs_dtype=None):
    """p: dict from foundation.covid19.build_covid_params; obs_dtype: the observations' element type (torch.float32 /
    torch.bfloat16 or their names, None: float32).  Returns (AieCovidConfig, keep-alive list)."""
    cfg = _abi.AieCovidConfig()
    keep = []

    def arr(v, dt):
        a = np.ascontiguousarray(np.asarray(v), dtype=dt)
        keep.append(a)
        return a.ctypes.data_as(C.c_void_p)

    cfg.abi_version = _abi.ABI_VERSION
    cfg.n_states = p["n_states"]
    cfg.episode_length = p["episode_length"]
    cfg.num_stringency_levels = p["num_stringency_levels"]
    cfg.action_cooldown_period = p["action_cooldown_period"]
    cfg.subsidy_interval = p["subsidy_interval"]
    cfg.num_subsidy_levels = p["num_subsidy_levels"]
    cfg.time_when_vaccine_delivery_begins = p["time_when_vaccine_delivery_begins"]
    cfg.delivery_interval = p["delivery_interval"]
    cfg.t_first_delivery = p["t_first_delivery"]
    cfg.beta_delay = p["beta_delay"]
    cfg.filter_len = p["filter_len"]
    cfg.num_filters = p["num_filters"]
    cfg.start_date_index = p["start_date_index"]
    cfg.rw_policy_days = int(p["rw_policy"].shape[0])
    cfg.value_of_life = int(p["value_of_life"])
    cfg.auto_reset = int(bool(auto_reset))
    cfg.obs_dtype = {"float32": _abi.OBS_F32, "bfloat16": _abi.OBS_BF16}[_abi.obs_dtype_name(obs_dtype)]
    for dst, src in [("gamma", "gamma"), ("death_rate", "death_rate"),
                     ("infection_too_sick_to_work_rate", "infection_too_sick_to_work_rate"),
                     ("pop_between_age_18_65", "pop_between_age_18_65"), ("risk_free_interest_rate", "risk_free_interest_rate"),
                     ("crra_eta", "crra_eta"), ("planner_health_norm", "planner_health_norm"),
                     ("planner_economic_norm", "planner_economic_norm"),
                     ("min_planner_health", "min_marginal_planner_health_index"),
                     ("max_planner_health", "max_marginal_planner_health_index"),
                     ("min_planner_econ", "min_marginal_planner_economic_index"),
                     ("max_planner_econ", "max_marginal_planner_economic_index"),
                     ("w_planner_health", "w_planner_health"), ("w_planner_econ", "w_planner_econ")]:
        setattr(cfg, dst, float(F32(p[src])))
    cfg.reward_normalization_factor = float(p["reward_normalization_factor"])
    cfg.time_scale = float(p["time_scale"])
    cfg.population = arr(p["population"], I32)
    cfg.num_vaccines_per_delivery = arr(p["num_vaccines_per_delivery"], I32)
    for dst, src in [("beta_slopes", "beta_slopes"), ("beta_intercepts", "beta_intercepts"),
                     ("unemployment_bias", "unemployment_bias"), ("maximum_productivity", "maximum_productivity"),
                     ("agents_health_norm", "agents_health_norm"), ("agents_economic_norm", "agents_economic_norm"),
                     ("min_agent_health", "min_marginal_agent_health_index"), ("max_agent_health", "max_marginal_agent_health_index"),
                     ("min_agent_econ", "min_marginal_agent_economic_index"), ("max_agent_econ", "max_marginal_agent_economic_index"),
                     ("w_agent_health", "w_agent_health"), ("w_agent_econ", "w_agent_econ"),
                     ("conv_weights", "conv_weights"), ("conv_filters", "conv_filters")]:
        setattr(cfg, dst, arr(p[src], F32))
    cfg.daily_production_per_worker = arr(np.array([p["daily_production_per_worker"]]), F32)
    cfg.max_daily_subsidy_per_state = arr(p["max_daily_subsidy_per_state"], np.float64)
    cfg.rw_policy = arr(p["rw_policy"], np.int8)
    ini = p["init"]
    init_state = np.stack([np.asarray(ini[k], F32) for k in ["susceptible", "infected", "recovered", "deaths", "vaccinated", "unemployed"]])
    cfg.init_state = arr(init_state, F32)
    return cfg, keep


class CovidStepperBase(PolicySampler):
    # "bf16": the observation / mask buffers of a bfloat16 env; numpy backends hold their raw bits
    _DT = {"f32": np.float32, "f64": np.float64, "i32": np.int32, "i8": np.int8, "bf16": np.uint16}

    def __init__(self, params, n_envs, lib, device_index=0, auto_reset=True, change_list=None, final_obs=False,
                 obs_dtype=None, episode_metrics=False):
        # obs_dtype: element type of the seven observation / mask buffers (and their final_ twins), float32 (default)
        # or bfloat16, each element the round-to-nearest-even of the float32 a float32 env writes.
        self.obs_dtype = _abi.obs_dtype_name(obs_dtype)
        # final_obs: keep final_<name> twins of the seven observation / mask buffers; step() then writes into row e the
        # observations of the state replica e's episode ended in, when that step ends it (done == 1).  Needs auto_reset.
        if final_obs and not auto_reset:
            raise ValueError("final_obs=True needs auto_reset=True: without the auto-reset, the observations after the step "
                             "that ends an episode already are its final ones")
        self.final_obs = bool(final_obs)
        # change_list: keep a persistent per-state list of stringency changes (O(changes) unemployment response instead
        # of a history scan, whose cost grows with the episode).  Default ON; AIE_COVID_CHANGE_LIST=0 selects the scan.
        if change_list is None:
            import os
            change_list = os.environ.get("AIE_COVID_CHANGE_LIST", "1") not in ("", "0")
        self.change_list = bool(change_list)
        self.p = params
        self.n_envs = int(n_envs)
        self.lib = lib
        cfg, self._keep = covid_config_from_params(params, auto_reset, self.obs_dtype)
        h = C.c_void_p()
        self._check(lib.aie_covid_create(C.byref(cfg), self.n_envs, int(device_index), C.byref(h)))
        self._h = h
        E, S, L = self.n_envs, params["n_states"], params["filter_len"]
        fo = "bf16" if self.obs_dtype == "bfloat16" else "f32"   # the observation / mask tensors
        shapes = {
            "state": ("f32", (E, 9, S)), "ints": ("i32", (E, 2, S)), "hdr": ("i32", (E, 4)), "ring": ("i8", (E, S, (L + 1 + 15) // 16 * 16)),
            "actions_agent": ("i32", (E, S)), "actions_planner": ("i32", (E,)),
            "obs_agent_state": (fo, (E, 6, S)), "obs_postsubsidy": (fo, (E, S)),
            "obs_lagged_stringency": (fo, (E, S)), "obs_policy_indicators": (fo, (E, S)),
            "obs_scalars": (fo, (E, 4)), "mask_agent": (fo, (E, 1 + params["num_stringency_levels"], S)),
            "mask_planner": (fo, (E, 1 + params["num_subsidy_levels"])), "reward_agent": ("f32", (E, S)),
            "reward_planner": ("f64", (E,)), "done": ("i32", (E,)),
        }
        if self.change_list:
            shapes["changes"] = ("i32", (E, 33, S))
        self.buf = {k: self._alloc(shape, dt) for k, (dt, shape) in shapes.items()}
        self._shapes = shapes
        self.rollout = None   # the bound Rollout (bind_rollout), and its slot cursor
        self.rollout_slot = 0
        bufs = _abi.AieCovidBuffers()
        for name in _abi._COVID_BUF_NAMES:
            setattr(bufs, name, self._ptr(self.buf[name]))
        bufs.changes = self._ptr(self.buf["changes"]) if self.change_list else None
        self._check(lib.aie_covid_bind_buffers(self._h, C.byref(bufs)))
        if self.final_obs:
            self._final_bufs = _abi.AieCovidObsBuffers()
            for name in _abi.COVID_OBS_NAMES:
                self.buf["final_" + name] = self._alloc(shapes[name][1], shapes[name][0])
                setattr(self._final_bufs, name, self._ptr(self.buf["final_" + name]))
        # episode_metrics: keep the episode-metric accumulators (aie_covid_bind_metrics); the step kernels add to them
        # and episode_metrics() turns them into scenario_metrics() rows.  Bound before the first reset, which zeroes them.
        self.episode_metrics_on = bool(episode_metrics)
        self._auto_reset, self._t, self._ended = bool(auto_reset), 0, False   # host mirror of the lock-step timestep
        if self.episode_metrics_on:
            m = _abi.AieCovidMetricBuffers()
            for name, dt, shape in [("sums", "f64", (E, 4, S)), ("prev_sums", "f64", (E, 4, S)),
                                    ("index", "f32", (E, 2, S + 1)), ("prev_index", "f32", (E, 2, S + 1)),
                                    ("prev_end", "f32", (E, 4, S))]:
                self.buf["metric_" + name] = self._alloc(shape, dt)
                setattr(m, name, self._ptr(self.buf["metric_" + name]))
            m.us_population = float(params["us_population"])
            self._check(lib.aie_covid_bind_metrics(self._h, C.byref(m)))

    def _check(self, rc):
        if rc != _abi.AIE_OK:
            self._refused_in_capture(rc)
            raise _abi.AieError("aie error %d: %s" % (rc, self.lib.aie_last_error().decode()))

    # captured rollouts (PolicySampler.rollout_capture_begin ...): this driver's mirror of the lock-step timestep is put
    # back at the end of a capture and advanced by T steps after a replay, as the library's own
    _capture_prefix = "aie_covid"

    def rollout_capture_begin(self):
        super().rollout_capture_begin()
        self._capture_host = (self._t, self._ended)

    def rollout_capture_end(self):
        super().rollout_capture_end()
        self._t, self._ended = self._capture_host

    def rollout_replay_end(self):
        super().rollout_replay_end()
        for _ in range(self.rollout.T):
            self._stepped()

    def _stream(self):
        return None

    def close(self):
        if getattr(self, "_h", None):
            self.lib.aie_covid_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def reset(self):
        self._check(self.lib.aie_covid_reset(self._h, self._stream()))
        self._t = 0

    def _stepped(self):
        self._t += 1
        if self._auto_reset and self._t >= int(self.p["episode_length"]):
            self._t, self._ended = 0, True

    def has_previous_episode(self):
        """Whether an episode has ended under the auto-reset (every replica ends on the same step)."""
        return self._ended

    def step(self):
        if self.rollout is not None:   # slot s -> s + 1; the final observations go to the rollout's final slots
            self._check(self.lib.aie_covid_step(self._h, self._stream()))
            self.rollout_slot += 1
        elif self.final_obs:
            self._check(self.lib.aie_covid_step_final(self._h, C.byref(self._final_bufs), self._stream()))
        else:
            self._check(self.lib.aie_covid_step(self._h, self._stream()))
        self._stepped()

    # -- rollouts stored in place (aie_covid_bind_rollout) -----------------------------------------------------------
    def bind_rollout(self, T, final_obs=False):
        """Allocate and bind a rollout of T steps (a Rollout), with final slots [K, E, ...] when final_obs."""
        if isinstance(T, bool) or not isinstance(T, numbers.Integral) or T < 1:
            raise ValueError("T must be a positive int")
        if self.rollout is not None:
            raise ValueError("a rollout is already bound: unbind_rollout() first")
        T = int(T)
        K = -(-T // int(self.p["episode_length"]))
        sh, names = self._shapes, list(_abi.COVID_OBS_NAMES)
        buf = {k: self._alloc((T + 1,) + sh[k][1], sh[k][0]) for k in names}
        for k in ("actions_agent", "actions_planner", "reward_agent", "reward_planner", "done"):
            buf[k] = self._alloc((T,) + sh[k][1], sh[k][0])
        r = _abi.AieCovidRollout()
        r.T = T
        for k in names:
            setattr(r.obs, k, self._ptr(buf[k]))
        if final_obs:
            for k in names:
                buf["final_" + k] = self._alloc((K,) + sh[k][1], sh[k][0])
                setattr(r.final_obs, k, self._ptr(buf["final_" + k]))
        for k in ("actions_agent", "actions_planner", "reward_agent", "reward_planner", "done"):
            setattr(r, k, self._ptr(buf[k]))
        self._check(self.lib.aie_covid_bind_rollout(self._h, C.byref(r)))
        self.rollout, self.rollout_slot = Rollout(T, K, buf, names, bool(final_obs)), 0
        return self.rollout

    def restart_rollout(self):
        self._check(self.lib.aie_covid_rollout_restart(self._h, self._stream()))
        self.rollout_slot = 0

    def unbind_rollout(self):
        self._check(self.lib.aie_covid_bind_rollout(self._h, None))
        self.rollout, self.rollout_slot = None, 0

    def sample_random_actions(self, seed=0):
        self._check(self.lib.aie_covid_sample_random_actions(self._h, C.c_uint64(int(seed)), self._stream()))

    # sample_policy (PolicySampler): agent logits [E, S, 1 + levels] (action axis last; the mask is [E, 1 + levels, S]),
    # planner logits [E, 1 + subsidy levels]; log-probabilities [E, S] and [E]
    @property
    def _policy_fn(self):
        return self.lib.aie_covid_sample_policy

    def _policy_shapes(self):
        E, S = self.n_envs, self.p["n_states"]
        return ((E, S, 1 + self.p["num_stringency_levels"]), (E, 1 + self.p["num_subsidy_levels"]), (E, S), (E,))

    @property
    def _eval_fns(self):
        return self.lib.aie_covid_evaluate_policy, self.lib.aie_covid_evaluate_policy_backward

    @property
    def _adv_fn(self):
        return self.lib.aie_covid_compute_advantages

    @property
    def _adv_k_fn(self):
        return self.lib.aie_covid_compute_advantages_k

    def _mask_rows(self):   # evaluate_policy: the agent mask is [*B, 1 + levels, S], transposed against the logits
        S, L = self.p["n_states"], self.p["num_stringency_levels"]
        return (1 + L, S), (1 + self.p["num_subsidy_levels"],)

    def launch_count(self):
        return int(self.lib.aie_covid_launch_count(self._h))

    def get_counters(self):
        """The library's host-side counters of this handle (aie_covid_get_counters) and this driver's mirror of the
        lock-step timestep, as a dict of ints."""
        c = _abi.AieCovidCounters()
        self._check(self.lib.aie_covid_get_counters(self._h, C.byref(c)))
        out = {k: int(getattr(c, k)) for k, _ in _abi.AieCovidCounters._fields_}
        out.update(host_t=int(self._t), host_ended=int(self._ended))
        return out

    def set_counters(self, counters):
        """Write the counters of get_counters() back (aie_covid_set_counters); marks the buffers as reset."""
        c = _abi.AieCovidCounters(**{k: int(counters[k]) for k, _ in _abi.AieCovidCounters._fields_})
        self._check(self.lib.aie_covid_set_counters(self._h, C.byref(c)))
        self._t, self._ended = int(counters["host_t"]), bool(counters["host_ended"])

    # -- episode metrics (aie_covid_bind_metrics / aie_covid_episode_metrics) -------------------------------------------
    def metric_layout(self):
        """[(key, is_int)] of the metric columns: "<state name>/<field>" for each state, then "usa/<field>" (the
        reference's scenario_metrics() keys in its dict order); no column is an int."""
        if getattr(self, "_metric_layout", None) is None:
            n = self.lib.aie_covid_get_metric_layout(self._h, None, 0)
            if n < 0:
                self._check(n)
            arr = (_abi.AieCovidMetricColumn * n)()
            self.lib.aie_covid_get_metric_layout(self._h, arr, n)
            names = self.p["state_names"]
            self._metric_layout = [("%s/%s" % ("usa" if arr[i].state < 0 else names[arr[i].state], arr[i].field.decode()),
                                    False) for i in range(n)]
        return list(self._metric_layout)

    def episode_metrics(self, final=False, out=None):
        """scenario_metrics() of every replica as float64 [n_envs, K] in metric_layout() order, one launch, asynchronous
        (aie_covid_episode_metrics).  final=True: of the episode each replica finished last.  out: an optional contiguous
        float64 [n_envs, K] buffer of this stepper's kind."""
        K = len(self.metric_layout())
        if out is None:
            out = self._alloc((self.n_envs, K), "f64")
        elif self._float_kind(out) != "f64" or tuple(out.shape) != (self.n_envs, K):
            raise _abi.AieError("episode_metrics: out must be a contiguous float64 [%d, %d] buffer" % (self.n_envs, K))
        self._check(self.lib.aie_covid_episode_metrics(self._h, 1 if final else 0, self._ptr(out), self._stream()))
        return out

    def obs_to_numpy(self, name, e=None):
        """Host copy of buffer `name` (of env e), bfloat16 observations as float32 (exact: every bfloat16 is a float32)."""
        a = self.to_numpy(self.buf[name] if e is None else self.buf[name][e])
        return bf16_bits_to_float32(a) if np.asarray(a).dtype == np.uint16 else a

    def read_obs(self, e):
        """Host copy of env e's outputs in oracle/covid_oracle.py's layout (observations as float32)."""
        g = lambda k: self.obs_to_numpy(k, e)
        return dict(agent_state=g("obs_agent_state"), postsubsidy=g("obs_postsubsidy"), lagged=g("obs_lagged_stringency"),
                    policy_ind=g("obs_policy_indicators"), scalars=g("obs_scalars"), mask_a=g("mask_agent"),
                    mask_p=g("mask_planner"), rew_a=g("reward_agent"), rew_p=np.float64(g("reward_planner")),
                    done=np.int32(g("done")))

    def read_state(self, e):
        st, ints, hdr = self.to_numpy(self.buf["state"][e]), self.to_numpy(self.buf["ints"][e]), self.to_numpy(self.buf["hdr"][e])
        names = ["susceptible", "infected", "recovered", "deaths", "vaccinated", "unemployed", "stringency", "subsidy", "postsubsidy"]
        out = {n: st[i] for i, n in enumerate(names)}
        out.update(t=int(hdr[0]), subsidy_level=int(hdr[1]), cooldown_until=ints[0], vaccines_available=ints[1], episodes=int(hdr[3]))
        return out


class CudaCovidStepper(CovidStepperBase):
    supports_rollout_capture = True

    def __init__(self, params, n_envs, device="cuda:0", auto_reset=True, lib_path=None, change_list=None, final_obs=False,
                 obs_dtype=None, episode_metrics=False):
        import torch

        if not torch.cuda.is_available():
            raise _abi.AieError("no CUDA device visible: ai_economist_b200 has no CPU fallback")
        self.torch = torch
        self.device = torch.device(device)
        idx = self.device.index if self.device.index is not None else torch.cuda.current_device()
        self.device = torch.device("cuda", idx)
        lib = _abi.load_library(lib_path)
        with torch.cuda.device(self.device):
            super().__init__(params, n_envs, lib, device_index=idx, auto_reset=auto_reset, change_list=change_list,
                             final_obs=final_obs, obs_dtype=obs_dtype, episode_metrics=episode_metrics)

    def _alloc(self, shape, dt):
        t = self.torch
        m = {"i8": t.int8, "i32": t.int32, "f32": t.float32, "f64": t.float64, "bf16": t.bfloat16}
        return t.zeros(shape, dtype=m[dt], device=self.device)

    def _buf_kind(self, buf):
        return buf_kind_torch(self.torch, self.device, buf)

    def _is_i32(self, buf):
        return is_i32_torch(self.torch, self.device, buf)

    def _float_kind(self, buf):
        return float_kind_torch(self.torch, self.device, buf)

    def _eval_out(self, shape, kind):
        t = self.torch
        return t.empty(shape, dtype={"f32": t.float32, "bf16": t.bfloat16}[kind], device=self.device)

    def _ptr(self, buf):
        return C.c_void_p(buf.data_ptr())

    def _stream(self):
        return C.c_void_p(self.torch.cuda.current_stream(self.device).cuda_stream)

    def to_numpy(self, buf):
        if buf.dtype == self.torch.bfloat16:   # numpy has no bfloat16: float32 holds every value exactly
            buf = buf.float()
        return buf.detach().cpu().numpy()
