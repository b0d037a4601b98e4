"""ctypes mirror of include/aie_b200.h (the C-ABI of the CUDA library).  No compute happens here."""
import ctypes as C

import numpy as np
import os

ABI_VERSION = 6
MAX_COMPONENTS, MAX_BRACKETS, MAX_RATES = 8, 16, 64
AIE_OK = 0
AIE_ESTATE = -3   # a call out of order (include/aie_b200.h)
OBS_F32, OBS_BF16 = 0, 1   # aie_config.obs_dtype, aie_covid_config.obs_dtype
REWARD_F32, REWARD_F64 = 0, 1   # aie_advantage_args.rewards_*_dtype

COMPONENT_KIND = {"Build": 0, "ContinuousDoubleAuction": 1, "Gather": 2, "PeriodicBracketTax": 3,
                  "WealthRedistribution": 4, "SimpleLabor": 5}

CSRC_DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), "csrc")
DEFAULT_LIB = os.path.join(CSRC_DIR, "libaie_b200.so")


class AieConfig(C.Structure):
    _fields_ = [
        ("abi_version", C.c_int32),
        ("n_agents", C.c_int32), ("height", C.c_int32), ("width", C.c_int32), ("episode_length", C.c_int32),
        ("multi_action_agents", C.c_int32), ("n_components", C.c_int32),
        ("components", C.c_int32 * MAX_COMPONENTS),
        ("has_water", C.c_int32), ("obs_range", C.c_int32), ("planner_gets_spatial_info", C.c_int32),
        ("allow_observation_scaling", C.c_int32),
        ("regen_weight", C.c_double * 2),
        ("isoelastic_eta", C.c_double), ("energy_cost", C.c_double), ("energy_warmup_constant", C.c_double),
        ("energy_warmup_auto", C.c_int32), ("planner_reward_type", C.c_int32),
        ("mixing_weight_gini_vs_coin", C.c_double),
        ("build_payment", C.c_double), ("build_labor", C.c_double),
        ("move_labor", C.c_double), ("collect_labor", C.c_double),
        ("max_bid_ask", C.c_int32), ("order_duration", C.c_int32), ("max_num_orders", C.c_int32),
        ("order_labor", C.c_double),
        ("tax_model", C.c_int32), ("disable_taxes", C.c_int32), ("period", C.c_int32),
        ("n_brackets", C.c_int32), ("n_disc_rates", C.c_int32),
        ("bracket_cutoffs", C.c_double * MAX_BRACKETS), ("disc_rates", C.c_double * MAX_RATES),
        ("fixed_rates", C.c_double * MAX_BRACKETS),
        ("tax_annealing", C.c_int32), ("annealing_warmup", C.c_double), ("annealing_slope", C.c_double),
        ("rate_max", C.c_double), ("rate_min", C.c_double),
        ("auto_reset", C.c_int32),
        ("reset_mode", C.c_int32), ("build_skill_dist", C.c_int32), ("gather_skill_dist", C.c_int32),
        ("payment_max_skill_multiplier", C.c_int32), ("fixed_four", C.c_int32),
        ("ranked_locs", (C.c_int16 * 2) * 64), ("avg_ranked_skill", C.c_double * 64),
        ("single_action_planner", C.c_int32), ("regen_halfwidth", C.c_int32 * 2),
        ("full_observability", C.c_int32),
        ("split_layout", C.c_int32), ("split_water_row", C.c_int32), ("split_top_ranks", C.c_uint64),
        ("dyn_layout", C.c_int32), ("dyn_checker", C.c_int32), ("dyn_coverage", C.c_double * 2), ("dyn_clump", C.c_double * 2),
        ("dyn_prob", C.c_void_p),
        ("scenario_kind", C.c_int32), ("agent_reward_type", C.c_int32), ("labor_exponent", C.c_double), ("labor_cost", C.c_double),
        ("mz_partitions", C.c_int32 * 2), ("mz_zones", C.c_int32 * 3),
        ("labor_mask_first_step", C.c_int32), ("labor_skill_scale", C.c_double),
        ("obs_dtype", C.c_int32),
    ]


class AieDims(C.Structure):
    _fields_ = [(n, C.c_int32) for n in [
        "n_envs", "n_agents", "height", "width", "n_map_channels", "window", "flat_agent", "flat_planner",
        "flat_planner_agent", "mask_agent", "mask_planner", "n_act_agent", "n_act_planner", "state_bytes",
        "algorithmic_bytes_per_env_step", "n_stats", "stats_trade", "stats_tax", "agent_map_elems",
        "agent_idx_elems"]]


_BUF_NAMES = ["state", "state0", "actions_agent", "actions_planner", "obs_agent_map", "obs_agent_idx",
              "obs_agent_flat", "mask_agent", "obs_planner_map", "obs_planner_idx", "obs_planner_flat",
              "obs_planner_agents", "mask_planner", "obs_time", "reward", "done", "episode_final"]


class AieBuffers(C.Structure):
    _fields_ = [(n, C.c_void_p) for n in _BUF_NAMES] + [("events", C.c_void_p), ("event_envs", C.c_int32),
                                                        ("event_cap", C.c_int32)]


class AieHostState(C.Structure):
    _fields_ = [("n", C.c_int32)] + [(n, C.c_void_p) for n in [
        "stone", "wood", "stone_src", "wood_src", "water", "loc", "coin", "inv_stone", "inv_wood",
        "build_payment", "build_skill", "bonus_gather_prob", "mt_key", "mt_pos", "completions", "gauss_has", "gauss_val", "split_skill"]]


class AieResetStreams(C.Structure):
    _fields_ = [(n, C.c_void_p) for n in ["mt_key", "mt_pos", "gauss_has", "gauss_val", "split_skill"]]


_DUMP_PTRS = ["cell", "owner", "loc", "coin", "esc_coin", "labor", "inv", "esc", "n_orders", "bid_hist", "ask_hist",
              "price_hist", "tax_pos", "rate_idx", "last_coin", "last_income", "last_marg", "mt_key", "mt_pos", "t",
              "completions", "book_rows", "book_count"]
_DUMP_PTRS2 = ["stats", "util_prev", "auto_warmup"]  # after book_cap (ABI 2)


class AieStateDump(C.Structure):
    _fields_ = ([(n, C.c_void_p) for n in _DUMP_PTRS] + [("book_cap", C.c_int32)] +
                [(n, C.c_void_p) for n in _DUMP_PTRS2])


class AieFlatField(C.Structure):
    _fields_ = [("key", C.c_char * 64), ("offset", C.c_int32), ("size", C.c_int32)]


class AieMetricKey(C.Structure):
    _fields_ = [("key", C.c_char * 64), ("is_int", C.c_int32)]


class AieField(C.Structure):
    _fields_ = [("offset", C.c_int32), ("elem_bytes", C.c_int32), ("is_float", C.c_int32),
                ("is_signed", C.c_int32), ("ndim", C.c_int32), ("shape", C.c_int32 * 4)]


_OUT_NAMES = ["obs_agent_map", "obs_agent_idx", "obs_agent_flat", "mask_agent", "obs_planner_map", "obs_planner_idx",
              "obs_planner_flat", "obs_planner_agents", "mask_planner", "obs_time", "reward", "done"]


class AieHostOut(C.Structure):
    _fields_ = [(n, C.c_void_p) for n in _OUT_NAMES]


OBS_NAMES = _OUT_NAMES[:10]   # the observation / mask tensors (aie_obs_buffers)


class AieObsBuffers(C.Structure):
    _fields_ = [(n, C.c_void_p) for n in OBS_NAMES]


class AieRollout(C.Structure):
    """aie_rollout: the device tensors of a rollout stored in place (aie_bind_rollout)."""
    _fields_ = [("T", C.c_int32), ("obs", AieObsBuffers), ("actions_agent", C.c_void_p), ("actions_planner", C.c_void_p),
                ("reward", C.c_void_p), ("done", C.c_void_p), ("final_obs", AieObsBuffers)]


class AiePolicyLogits(C.Structure):
    _fields_ = [("agent", C.c_void_p), ("planner", C.c_void_p), ("logits_dtype", C.c_int32), ("greedy", C.c_int32),
                ("log_prob_agent", C.c_void_p), ("log_prob_planner", C.c_void_p)]


class AiePolicyEval(C.Structure):
    _fields_ = ([(n, C.c_void_p) for n in ["logits_agent", "logits_planner", "mask_agent", "mask_planner",
                                           "actions_agent", "actions_planner"]]
                + [("logits_dtype", C.c_int32), ("mask_dtype", C.c_int32)]
                + [(n, C.c_void_p) for n in ["log_prob_agent", "log_prob_planner", "entropy_agent", "entropy_planner",
                                             "grad_log_prob_agent", "grad_log_prob_planner", "grad_entropy_agent",
                                             "grad_entropy_planner", "grad_logits_agent", "grad_logits_planner"]])


class AieAdvantageArgs(C.Structure):
    _fields_ = ([("rewards_agent", C.c_void_p), ("rewards_planner", C.c_void_p), ("rewards_agent_dtype", C.c_int32),
                 ("rewards_planner_dtype", C.c_int32)]
                + [(n, C.c_void_p) for n in ["values_agent", "values_planner", "dones", "last_values_agent",
                                             "last_values_planner", "final_values_agent", "final_values_planner"]]
                + [(n, C.c_double) for n in ["gamma_agent", "gamma_planner", "lambda_agent", "lambda_planner"]]
                + [(n, C.c_void_p) for n in ["adv_agent", "adv_planner", "ret_agent", "ret_planner"]])


class AieCovidConfig(C.Structure):
    _fields_ = ([(n, C.c_int32) for n in [
        "abi_version", "n_states", "episode_length", "num_stringency_levels", "action_cooldown_period",
        "subsidy_interval", "num_subsidy_levels", "time_when_vaccine_delivery_begins", "delivery_interval",
        "t_first_delivery", "beta_delay", "filter_len", "num_filters", "start_date_index", "rw_policy_days",
        "value_of_life", "auto_reset"]]
        + [(n, C.c_float) for n in [
            "gamma", "death_rate", "infection_too_sick_to_work_rate", "pop_between_age_18_65",
            "risk_free_interest_rate", "crra_eta", "planner_health_norm", "planner_economic_norm",
            "min_planner_health", "max_planner_health", "min_planner_econ", "max_planner_econ", "w_planner_health",
            "w_planner_econ"]]
        + [("reward_normalization_factor", C.c_double), ("time_scale", C.c_double)]
        + [(n, C.c_void_p) for n in [
            "population", "num_vaccines_per_delivery", "beta_slopes", "beta_intercepts", "unemployment_bias",
            "daily_production_per_worker", "maximum_productivity", "agents_health_norm", "agents_economic_norm",
            "min_agent_health", "max_agent_health", "min_agent_econ", "max_agent_econ", "w_agent_health",
            "w_agent_econ", "conv_weights", "conv_filters", "max_daily_subsidy_per_state", "rw_policy",
            "init_state"]]
        + [("obs_dtype", C.c_int32)])


_COVID_BUF_NAMES = ["state", "ints", "hdr", "ring", "actions_agent", "actions_planner", "obs_agent_state",
                    "obs_postsubsidy", "obs_lagged_stringency", "obs_policy_indicators", "obs_scalars", "mask_agent",
                    "mask_planner", "reward_agent", "reward_planner", "done"]


class AieCovidBuffers(C.Structure):
    _fields_ = [(n, C.c_void_p) for n in _COVID_BUF_NAMES] + [("changes", C.c_void_p)]


COVID_OBS_NAMES = _COVID_BUF_NAMES[6:13]   # the observation / mask tensors (aie_covid_obs_buffers)


class AieCovidObsBuffers(C.Structure):
    _fields_ = [(n, C.c_void_p) for n in COVID_OBS_NAMES]


class AieCovidMetricBuffers(C.Structure):
    """aie_covid_metric_buffers: the episode-metric accumulators of a COVID-19 env (aie_covid_bind_metrics)."""
    _fields_ = [("sums", C.c_void_p), ("prev_sums", C.c_void_p), ("index", C.c_void_p), ("prev_index", C.c_void_p),
                ("prev_end", C.c_void_p), ("us_population", C.c_double)]


class AieCovidMetricColumn(C.Structure):
    _fields_ = [("state", C.c_int32), ("field", C.c_char * 60)]


class AieCounters(C.Structure):
    """aie_counters: the host-side counters of a handle (aie_get_counters / aie_set_counters)."""
    _fields_ = [("sample_calls", C.c_uint64), ("policy_calls", C.c_uint64), ("fused_policy_key", C.c_uint64),
                ("fused_policy_on", C.c_int32), ("reserved", C.c_int32)]


class AieCovidCounters(C.Structure):
    """aie_covid_counters: the host-side counters of a COVID-19 handle (aie_covid_get_counters / _set_counters)."""
    _fields_ = [("sample_calls", C.c_uint64), ("policy_calls", C.c_uint64), ("t", C.c_int32),
                ("previous_episode", C.c_int32)]


class AieCovidRollout(C.Structure):
    """aie_covid_rollout: the device tensors of a COVID-19 rollout stored in place (aie_covid_bind_rollout)."""
    _fields_ = [("T", C.c_int32), ("obs", AieCovidObsBuffers), ("actions_agent", C.c_void_p),
                ("actions_planner", C.c_void_p), ("reward_agent", C.c_void_p), ("reward_planner", C.c_void_p),
                ("done", C.c_void_p), ("final_obs", AieCovidObsBuffers)]


class AieError(RuntimeError):
    pass


def load_library(path=None):
    """Open the C-ABI shared library and declare every prototype in include/aie_b200.h."""
    path = path or os.environ.get("AIE_LIB_PATH") or DEFAULT_LIB  # AIE_LIB_PATH: alternative CUDA build (tuning)
    if not os.path.exists(path):
        raise AieError(
            "CUDA extension %s not found. Build it first: `python -c \"import __graft_entry__ as g; g.build()\"` "
            "(nvcc, sm_90a). There is no CPU fallback." % path)
    L = C.CDLL(path)
    P = C.c_void_p
    L.aie_last_error.restype = C.c_char_p
    L.aie_abi_version.restype = C.c_int
    L.aie_create.argtypes = [C.POINTER(AieConfig), C.c_int32, C.c_int32, C.POINTER(P)]
    L.aie_destroy.argtypes = [P]
    L.aie_get_dims.argtypes = [P, C.POINTER(AieDims)]
    L.aie_get_field.argtypes = [P, C.c_char_p, C.POINTER(AieField)]
    L.aie_get_flat_layout.argtypes = [P, C.c_int32, C.POINTER(AieFlatField), C.c_int32]
    L.aie_get_flat_layout.restype = C.c_int
    L.aie_bind_buffers.argtypes = [P, C.POINTER(AieBuffers)]
    L.aie_load_state.argtypes = [P, C.POINTER(AieHostState), C.c_int32, P]
    L.aie_reset_envs.argtypes = [P, C.POINTER(AieHostState), C.POINTER(AieResetStreams), C.c_int32, C.c_int32, P]
    L.aie_reset_envs.restype = C.c_int
    L.aie_step.argtypes = [P, P]
    L.aie_observe.argtypes = [P, P]
    L.aie_observe_final.argtypes = [P, C.POINTER(AieObsBuffers), P]
    L.aie_observe_final.restype = C.c_int
    L.aie_step_dynamics.argtypes = [P, P]
    L.aie_sample_random_actions.argtypes = [P, C.c_uint64, P]
    L.aie_set_fused_policy.argtypes = [P, C.c_uint64, P]
    L.aie_sample_policy.argtypes = [P, C.POINTER(AiePolicyLogits), C.c_uint64, P]
    L.aie_sample_policy.restype = C.c_int
    L.aie_covid_sample_policy.argtypes = [P, C.POINTER(AiePolicyLogits), C.c_uint64, P]
    L.aie_covid_sample_policy.restype = C.c_int
    for fn in ["aie_evaluate_policy", "aie_evaluate_policy_backward", "aie_covid_evaluate_policy",
               "aie_covid_evaluate_policy_backward"]:
        getattr(L, fn).argtypes = [P, C.POINTER(AiePolicyEval), C.c_int64, P]
        getattr(L, fn).restype = C.c_int
    for fn in ["aie_compute_advantages", "aie_covid_compute_advantages"]:
        getattr(L, fn).argtypes = [P, C.POINTER(AieAdvantageArgs), C.c_int32, P]
        getattr(L, fn).restype = C.c_int
    L.aie_compute_advantages_k.argtypes = [P, C.POINTER(AieAdvantageArgs), C.c_int32, C.c_int32, P]
    L.aie_compute_advantages_k.restype = C.c_int
    L.aie_bind_rollout.argtypes = [P, C.POINTER(AieRollout)]
    L.aie_bind_rollout.restype = C.c_int
    L.aie_rollout_restart.argtypes = [P, P]
    L.aie_rollout_restart.restype = C.c_int
    L.aie_covid_compute_advantages_k.argtypes = [P, C.POINTER(AieAdvantageArgs), C.c_int32, C.c_int32, P]
    L.aie_covid_compute_advantages_k.restype = C.c_int
    L.aie_covid_bind_rollout.argtypes = [P, C.POINTER(AieCovidRollout)]
    L.aie_covid_bind_rollout.restype = C.c_int
    L.aie_covid_rollout_restart.argtypes = [P, P]
    L.aie_covid_rollout_restart.restype = C.c_int
    L.aie_covid_bind_metrics.argtypes = [P, C.POINTER(AieCovidMetricBuffers)]
    L.aie_covid_bind_metrics.restype = C.c_int
    L.aie_covid_get_metric_layout.argtypes = [P, C.POINTER(AieCovidMetricColumn), C.c_int32]
    L.aie_covid_get_metric_layout.restype = C.c_int
    L.aie_covid_episode_metrics.argtypes = [P, C.c_int32, P, P]
    L.aie_covid_episode_metrics.restype = C.c_int
    L.aie_step_host.argtypes = [P, P, P, C.POINTER(AieHostOut), P]
    L.aie_step_host_compact.argtypes = [P, P, P, C.POINTER(AieHostOut), C.c_int32, P]
    L.aie_step_host_compact.restype = C.c_int
    L.aie_compact_bytes_per_env.argtypes = [P]
    L.aie_compact_bytes_per_env.restype = C.c_int32
    L.aie_get_host_timing.argtypes = [P, C.POINTER(C.c_double), C.c_int32]
    L.aie_get_host_timing.restype = C.c_int
    L.aie_read_state.argtypes = [P, C.c_int32, C.POINTER(AieStateDump)]
    L.aie_read_episode_final.argtypes = [P, C.c_int32, C.POINTER(AieStateDump)]
    L.aie_read_episode_final.restype = C.c_int
    L.aie_get_metric_layout.argtypes = [P, C.POINTER(AieMetricKey), C.c_int32]
    L.aie_get_metric_layout.restype = C.c_int
    L.aie_episode_metrics.argtypes = [P, C.c_int32, P, P]
    L.aie_episode_metrics.restype = C.c_int
    L.aie_launch_count.argtypes = [P]
    L.aie_covid_create.argtypes = [C.POINTER(AieCovidConfig), C.c_int32, C.c_int32, C.POINTER(P)]
    L.aie_covid_destroy.argtypes = [P]
    L.aie_covid_bind_buffers.argtypes = [P, C.POINTER(AieCovidBuffers)]
    L.aie_covid_reset.argtypes = [P, P]
    L.aie_covid_step.argtypes = [P, P]
    L.aie_covid_step_final.argtypes = [P, C.POINTER(AieCovidObsBuffers), P]
    L.aie_covid_sample_random_actions.argtypes = [P, C.c_uint64, P]
    L.aie_covid_launch_count.argtypes = [P]
    L.aie_covid_launch_count.restype = C.c_int64
    for fn in ["aie_covid_create", "aie_covid_destroy", "aie_covid_bind_buffers", "aie_covid_reset", "aie_covid_step",
               "aie_covid_step_final", "aie_covid_sample_random_actions"]:
        getattr(L, fn).restype = C.c_int
    L.aie_launch_count.restype = C.c_int64
    for fn in ["aie_create", "aie_destroy", "aie_get_dims", "aie_get_field", "aie_bind_buffers", "aie_load_state",
               "aie_step", "aie_observe", "aie_step_host", "aie_step_host_compact", "aie_compact_bytes_per_env", "aie_read_state", "aie_step_dynamics",
               "aie_sample_random_actions", "aie_set_fused_policy"]:
        getattr(L, fn).restype = C.c_int
    for fn, st in (("aie_get_counters", AieCounters), ("aie_set_counters", AieCounters),
                   ("aie_covid_get_counters", AieCovidCounters), ("aie_covid_set_counters", AieCovidCounters)):
        getattr(L, fn).argtypes = [P, C.POINTER(st)]
        getattr(L, fn).restype = C.c_int
    for fam in ("aie", "aie_covid"):   # captured rollouts
        for fn, args in (("rollout_capture_begin", [P, P]), ("rollout_capture_end", [P]),
                         ("rollout_replay_begin", [P, P]), ("rollout_replay_end", [P])):
            getattr(L, "%s_%s" % (fam, fn)).argtypes = args
            getattr(L, "%s_%s" % (fam, fn)).restype = C.c_int
    if L.aie_abi_version() != ABI_VERSION:
        raise AieError("ABI version mismatch between %s and the Python binding" % path)
    return L


EXPORTED_SYMBOLS = ["aie_create", "aie_destroy", "aie_get_dims", "aie_get_field", "aie_get_flat_layout", "aie_bind_buffers",
                    "aie_load_state", "aie_reset_envs", "aie_step", "aie_step_dynamics", "aie_observe", "aie_observe_final", "aie_sample_random_actions",
                    "aie_set_fused_policy", "aie_sample_policy", "aie_evaluate_policy", "aie_evaluate_policy_backward", "aie_compute_advantages", "aie_compute_advantages_k", "aie_bind_rollout", "aie_rollout_restart", "aie_step_host", "aie_step_host_compact", "aie_compact_bytes_per_env", "aie_get_host_timing", "aie_read_state", "aie_read_episode_final",
                    "aie_get_metric_layout", "aie_episode_metrics", "aie_launch_count", "aie_last_error", "aie_abi_version",
                    "aie_get_counters", "aie_set_counters", "aie_covid_get_counters", "aie_covid_set_counters",
                    "aie_covid_create", "aie_covid_destroy", "aie_covid_bind_buffers", "aie_covid_reset", "aie_covid_step",
                    "aie_covid_step_final", "aie_covid_sample_random_actions", "aie_covid_sample_policy", "aie_covid_evaluate_policy",
                    "aie_covid_evaluate_policy_backward", "aie_covid_compute_advantages", "aie_covid_launch_count",
                    "aie_covid_bind_rollout", "aie_covid_rollout_restart", "aie_covid_compute_advantages_k",
                    "aie_covid_bind_metrics", "aie_covid_get_metric_layout", "aie_covid_episode_metrics",
                    "aie_rollout_capture_begin", "aie_rollout_capture_end", "aie_rollout_replay_begin", "aie_rollout_replay_end",
                    "aie_covid_rollout_capture_begin", "aie_covid_rollout_capture_end", "aie_covid_rollout_replay_begin",
                    "aie_covid_rollout_replay_end"]


def obs_dtype_name(obs_dtype):
    """"float32" or "bfloat16" for an obs_dtype kwarg: torch.float32 / torch.bfloat16, their names, or None (float32)."""
    name = "float32" if obs_dtype is None else str(obs_dtype).replace("torch.", "")
    if name not in ("float32", "bfloat16"):
        raise ValueError("obs_dtype must be torch.float32 or torch.bfloat16, got %r" % (obs_dtype,))
    return name


def config_from_spec(spec, auto_reset=True):
    """spec: the flat numeric env description produced by foundation.spec.EnvSpec.to_dict()."""
    cfg = AieConfig()
    cfg.abi_version = ABI_VERSION
    for k in ["n_agents", "height", "width", "episode_length", "multi_action_agents", "has_water", "obs_range",
              "planner_gets_spatial_info", "allow_observation_scaling", "isoelastic_eta", "energy_cost",
              "energy_warmup_constant", "energy_warmup_auto", "planner_reward_type", "mixing_weight_gini_vs_coin",
              "build_payment", "build_labor", "move_labor", "collect_labor", "max_bid_ask", "order_duration",
              "max_num_orders", "order_labor", "tax_model", "disable_taxes", "period", "n_brackets", "n_disc_rates",
              "tax_annealing", "annealing_warmup", "annealing_slope", "rate_max"]:
        setattr(cfg, k, spec[k])
    cfg.rate_min = float(spec.get("rate_min", 0.0))
    comps = [COMPONENT_KIND[c] for c in spec["components"]]
    cfg.n_components = len(comps)
    for i, c in enumerate(comps):
        cfg.components[i] = c
    cfg.regen_weight[0], cfg.regen_weight[1] = spec["regen_weight"]
    for i, v in enumerate(spec["bracket_cutoffs"]):
        cfg.bracket_cutoffs[i] = v
    for i, v in enumerate(spec["disc_rates"]):
        cfg.disc_rates[i] = v
    for i, v in enumerate(spec["fixed_rates"]):
        cfg.fixed_rates[i] = v
    cfg.auto_reset = int(bool(auto_reset))
    cfg.reset_mode = int(spec.get("reset_mode", 0))
    cfg.build_skill_dist = int(spec.get("build_skill_dist", 0))
    cfg.gather_skill_dist = int(spec.get("gather_skill_dist", 0))
    cfg.payment_max_skill_multiplier = int(spec.get("payment_max_skill_multiplier", 1))
    cfg.fixed_four = int(spec.get("fixed_four", 0))
    for i, rc in enumerate(spec.get("ranked_locs", [])):
        cfg.ranked_locs[i][0], cfg.ranked_locs[i][1] = int(rc[0]), int(rc[1])
    for i, v in enumerate(spec.get("avg_ranked_skill", [])):
        cfg.avg_ranked_skill[i] = float(v)
    cfg.single_action_planner = int(spec.get("single_action_planner", 0))
    cfg.regen_halfwidth[0], cfg.regen_halfwidth[1] = [int(v) for v in spec.get("regen_halfwidth", [0, 0])]
    cfg.full_observability = int(spec.get("full_observability", 0))
    cfg.split_layout = int(spec.get("split_layout", 0))
    cfg.split_water_row = int(spec.get("split_water_row", 0))
    cfg.split_top_ranks = int(spec.get("split_top_ranks", 0))
    cfg.scenario_kind = int(spec.get("scenario_kind", 0))
    cfg.agent_reward_type = int(spec.get("agent_reward_type", 0))
    cfg.labor_exponent = float(spec.get("labor_exponent", 2.0))
    cfg.labor_cost = float(spec.get("labor_cost", 1.0))
    cfg.labor_mask_first_step = int(spec.get("labor_mask_first_step", 1))
    cfg.labor_skill_scale = float(spec.get("labor_skill_scale", 1.0))
    cfg.obs_dtype = {"float32": OBS_F32, "bfloat16": OBS_BF16}[spec.get("obs_dtype", "float32")]
    cfg.dyn_layout = int(spec.get("dyn_layout", 0)) if cfg.reset_mode == 1 else 0
    if cfg.dyn_layout:
        cfg.dyn_checker = int(spec.get("dyn_checker", 0))
        cfg.dyn_coverage[0], cfg.dyn_coverage[1] = [float(v) for v in spec["dyn_coverage"]]
        cfg.dyn_clump[0], cfg.dyn_clump[1] = [float(v) for v in spec["dyn_clump"]]
        if cfg.dyn_layout == 3:   # MultiZone: the maps follow from the per-reset zone shuffle
            cfg.mz_partitions[0], cfg.mz_partitions[1] = [int(v) for v in spec["mz_partitions"]]
            for i, v in enumerate(spec["mz_zones"]):
                cfg.mz_zones[i] = int(v)
        else:
            prob = np.ascontiguousarray(np.asarray(spec["dyn_prob"], np.float64))
            assert prob.shape == (2, spec["height"], spec["width"]), "dyn_prob must be float64 [2][height][width]"
            cfg._dyn_prob_keep = prob    # aie_create copies it; kept alive until then
            cfg.dyn_prob = prob.ctypes.data
    return cfg
