"""Python driver of the COVID-19 scenario kernels (plumbing: buffers + ABI calls)."""
import ctypes as C

import numpy as np

from . import _abi

F32, I32 = np.float32, np.int32


def covid_config_from_params(p, auto_reset=True):
    """p: dict from foundation.covid19.build_covid_params.  Returns (AieCovidConfig, keep-alive list)."""
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


class CovidStepperBase:
    _DT = {"f32": np.float32, "f64": np.float64, "i32": np.int32, "i8": np.int8}

    def __init__(self, params, n_envs, lib, device_index=0, auto_reset=True, change_list=None):
        # change_list: keep a persistent per-state list of stringency changes (O(changes) unemployment response instead
        # of a history scan, whose cost grows with the episode).  Default ON; AIE_COVID_CHANGE_LIST=0 selects the scan.
        if change_list is None:
            import os
            change_list = os.environ.get("AIE_COVID_CHANGE_LIST", "1") not in ("", "0")
        self.change_list = bool(change_list)
        self.p = params
        self.n_envs = int(n_envs)
        self.lib = lib
        cfg, self._keep = covid_config_from_params(params, auto_reset)
        h = C.c_void_p()
        self._check(lib.aie_covid_create(C.byref(cfg), self.n_envs, int(device_index), C.byref(h)))
        self._h = h
        E, S, L = self.n_envs, params["n_states"], params["filter_len"]
        shapes = {
            "state": ("f32", (E, 9, S)), "ints": ("i32", (E, 2, S)), "hdr": ("i32", (E, 4)), "ring": ("i8", (E, S, (L + 1 + 15) // 16 * 16)),
            "actions_agent": ("i32", (E, S)), "actions_planner": ("i32", (E,)),
            "obs_agent_state": ("f32", (E, 6, S)), "obs_postsubsidy": ("f32", (E, S)),
            "obs_lagged_stringency": ("f32", (E, S)), "obs_policy_indicators": ("f32", (E, S)),
            "obs_scalars": ("f32", (E, 4)), "mask_agent": ("f32", (E, 1 + params["num_stringency_levels"], S)),
            "mask_planner": ("f32", (E, 1 + params["num_subsidy_levels"])), "reward_agent": ("f32", (E, S)),
            "reward_planner": ("f64", (E,)), "done": ("i32", (E,)),
        }
        if self.change_list:
            shapes["changes"] = ("i32", (E, 33, S))
        self.buf = {k: self._alloc(shape, dt) for k, (dt, shape) in shapes.items()}
        bufs = _abi.AieCovidBuffers()
        for name in _abi._COVID_BUF_NAMES:
            setattr(bufs, name, self._ptr(self.buf[name]))
        bufs.changes = self._ptr(self.buf["changes"]) if self.change_list else None
        self._check(lib.aie_covid_bind_buffers(self._h, C.byref(bufs)))

    def _check(self, rc):
        if rc != _abi.AIE_OK:
            raise _abi.AieError("aie error %d: %s" % (rc, self.lib.aie_last_error().decode()))

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

    def step(self):
        self._check(self.lib.aie_covid_step(self._h, self._stream()))

    def sample_random_actions(self, seed=0):
        self._check(self.lib.aie_covid_sample_random_actions(self._h, C.c_uint64(int(seed)), self._stream()))

    def launch_count(self):
        return int(self.lib.aie_covid_launch_count(self._h))

    def read_obs(self, e):
        """Host copy of env e's outputs in oracle/covid_oracle.py's layout."""
        g = lambda k: self.to_numpy(self.buf[k][e])
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
    def __init__(self, params, n_envs, device="cuda:0", auto_reset=True, lib_path=None, change_list=None):
        import torch

        if not torch.cuda.is_available():
            raise _abi.AieError("no CUDA device visible: ai_economist_b200 has no CPU fallback")
        self.torch = torch
        self.device = torch.device(device)
        idx = self.device.index if self.device.index is not None else torch.cuda.current_device()
        self.device = torch.device("cuda", idx)
        lib = _abi.load_library(lib_path)
        with torch.cuda.device(self.device):
            super().__init__(params, n_envs, lib, device_index=idx, auto_reset=auto_reset, change_list=change_list)

    def _alloc(self, shape, dt):
        t = self.torch
        m = {"i8": t.int8, "i32": t.int32, "f32": t.float32, "f64": t.float64}
        return t.zeros(shape, dtype=m[dt], device=self.device)

    def _ptr(self, buf):
        return C.c_void_p(buf.data_ptr())

    def _stream(self):
        return C.c_void_p(self.torch.cuda.current_stream(self.device).cuda_stream)

    def to_numpy(self, buf):
        return buf.detach().cpu().numpy()
