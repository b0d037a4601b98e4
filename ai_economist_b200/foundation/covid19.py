"""COVID-19 and economy scenario (BASELINE config 4): host-side mirror.

reference: scenarios/covid19/covid19_env.py (CovidAndEconomyEnvironment), components/covid19_components.py
(ControlUSStateOpenCloseStatus, FederalGovernmentSubsidy, VaccinationCampaign).

`build_covid_params` resolves the scenario + component kwargs and the fitted-parameter / real-world data files
into plain arrays: everything the per-timestep path needs.  The derived constants (daily production per
worker, maximum productivity, reward norms and weightages) follow the reference constructor expression by
expression, including its float32 / int32 / float64 dtypes (covid19_env.py:96-385, 1517-1625), because the
step arithmetic downstream is dtype-sensitive.
"""
import json
import os
from datetime import datetime

import numpy as np

from .._abi import COVID_OBS_NAMES
from . import rollout_graph as _rg

DATA_DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), "covid19_data")
F32, I32 = np.float32, np.int32


def _softplus(x, beta=1, threshold=20):  # covid19_env.py:1398-1406
    return 1 / beta * np.log(1 + np.exp(beta * x)) * (beta * x <= threshold) + x * (beta * x > threshold)


def build_covid_params(episode_length=540, start_date="2020-03-22", pop_between_age_18_65=0.6,
                       infection_too_sick_to_work_rate=0.1, risk_free_interest_rate=0.03,
                       economic_reward_crra_eta=2, health_priority_scaling_agents=1,
                       health_priority_scaling_planner=1, reward_normalization_factor=1,
                       path_to_data_and_fitted_params="", action_cooldown_period=28, n_stringency_levels=10,
                       subsidy_interval=90, num_subsidy_levels=20, max_annual_subsidy_per_person=20000,
                       daily_vaccines_per_million_people=4500, delivery_interval=1,
                       vaccine_delivery_start_date="2020-12-22", allow_observation_scaling=True):
    path = path_to_data_and_fitted_params or DATA_DIR
    rw = dict(np.load(os.path.join(path, "real_world_data.npz")))
    mc = json.load(open(os.path.join(path, "model_constants.json")))
    fp = json.load(open(os.path.join(path, "fitted_params.json")))
    p = {}
    date_format = mc["DATE_FORMAT"]
    pop = I32(mc["US_STATE_POPULATION"])
    us_pop = I32(mc["US_POPULATION"])
    S = len(pop)
    p["n_states"] = S
    p["episode_length"] = int(episode_length)
    # episode metrics (scenario_metrics, covid19_env.py:1613-1687): state names of the keys, the usa/ rates' divisor
    p["state_names"] = [mc["US_STATE_IDX_TO_STATE_NAME"][str(a)] for a in range(S)]
    p["us_population"] = int(us_pop)
    p["population"] = pop
    p["num_stringency_levels"] = int(mc["NUM_STRINGENCY_LEVELS"])
    assert int(n_stringency_levels) == p["num_stringency_levels"], \
        "For the given model fit, the number of stringency levels must be {}".format(p["num_stringency_levels"])
    p["death_rate"] = F32(mc["SIR_MORTALITY"])
    p["gamma"] = F32(mc["SIR_GAMMA"])
    gdp_per_capita = F32(mc["GDP_PER_CAPITA"])
    policy_start = datetime.strptime(fp["POLICY_START_DATE"], date_format)
    start = datetime.strptime(start_date, date_format)
    assert start >= policy_start
    sdi = (start - policy_start).days
    assert 0 <= sdi < len(rw["policy"])
    p["start_date_index"] = sdi
    p["value_of_life"] = I32(fp["VALUE_OF_LIFE"])
    p["beta_delay"] = int(fp["BETA_DELAY"])
    p["beta_slopes"] = np.array(fp["BETA_SLOPES"], dtype=F32)
    p["beta_intercepts"] = np.array(fp["BETA_INTERCEPTS"], dtype=F32)
    for k in ["MIN_MARGINAL_AGENT_HEALTH_INDEX", "MAX_MARGINAL_AGENT_HEALTH_INDEX",
              "MIN_MARGINAL_AGENT_ECONOMIC_INDEX", "MAX_MARGINAL_AGENT_ECONOMIC_INDEX"]:
        p[k.lower()] = np.array(fp[k], dtype=F32)
    for k in ["MIN_MARGINAL_PLANNER_HEALTH_INDEX", "MAX_MARGINAL_PLANNER_HEALTH_INDEX",
              "MIN_MARGINAL_PLANNER_ECONOMIC_INDEX", "MAX_MARGINAL_PLANNER_ECONOMIC_INDEX"]:
        p[k.lower()] = F32(fp[k])
    inferred_w_agent = np.array(fp["INFERRED_WEIGHTAGE_ON_AGENT_HEALTH_INDEX"], dtype=F32)
    inferred_w_planner = F32(fp["INFERRED_WEIGHTAGE_ON_PLANNER_HEALTH_INDEX"])
    L = int(fp["FILTER_LEN"])
    p["filter_len"] = L
    conv_lambdas = np.array(fp["CONV_LAMBDAS"], dtype=F32)
    F = len(conv_lambdas)
    p["num_filters"] = F
    p["unemployment_bias"] = np.array(fp["UNEMPLOYMENT_BIAS"], dtype=F32)
    gw = np.array(fp["GROUPED_CONVOLUTIONAL_FILTER_WEIGHTS"], dtype=F32)
    p["conv_weights"] = gw.reshape(S, F)                                      # float32 [S, F]
    f_ts = np.tile(np.flip(np.arange(L), (0,))[None, None], (1, F, 1)).astype(F32)
    p["conv_filters"] = np.exp(-f_ts / conv_lambdas[None, :, None])[0]        # float32 [F, L]
    p["risk_free_interest_rate"] = F32(risk_free_interest_rate)
    # unemployment at closure policy "all ones" (timestep 0: zero stringency deltas), covid19_env.py:260-262, 1407-1441
    delta0 = np.zeros((L, S))
    w_x = delta0[None].transpose(2, 0, 1) * np.repeat(p["conv_weights"][:, :, None], L, axis=-1)
    excess = _softplus(np.sum(w_x * p["conv_filters"][None], axis=(1, 2)), beta=1)
    unemployed_level_1 = (excess + p["unemployment_bias"]) * pop / 100
    workforce = (us_pop * pop_between_age_18_65 - np.sum(unemployed_level_1)).astype(I32)
    workers_per_capita = (workforce / us_pop).astype(F32)
    gdp_per_worker = (gdp_per_capita / workers_per_capita).astype(F32)
    p["daily_production_per_worker"] = (gdp_per_worker / 365).astype(F32)
    p["infection_too_sick_to_work_rate"] = F32(infection_too_sick_to_work_rate)
    p["pop_between_age_18_65"] = F32(pop_between_age_18_65)
    # economy_step with nobody sick, dead (covid19_env.py:283-292, 1444-1475)
    zero = np.zeros(S, dtype=I32)
    incapacitated = (p["infection_too_sick_to_work_rate"] * zero) + zero
    cant_work = (incapacitated * p["pop_between_age_18_65"]) + unemployed_level_1
    can_work = np.maximum(0, pop * p["pop_between_age_18_65"] - cant_work)
    p["maximum_productivity"] = (can_work * p["daily_production_per_worker"]).astype(F32)
    p["crra_eta"] = F32(economic_reward_crra_eta)
    p["agents_health_norm"] = p["maximum_productivity"] * 365
    p["planner_health_norm"] = np.sum(p["agents_health_norm"])
    p["agents_economic_norm"] = p["maximum_productivity"] * 365
    p["planner_economic_norm"] = np.sum(p["agents_economic_norm"])

    def scale(h, alphas):  # covid19_env.py:312-321
        z = alphas / (1 - alphas)
        sz = h * z
        return sz / (1 + sz)

    p["w_agent_health"] = scale(health_priority_scaling_agents, inferred_w_agent)
    p["w_agent_econ"] = 1 - p["w_agent_health"]
    p["w_planner_health"] = scale(health_priority_scaling_planner, inferred_w_planner)
    p["w_planner_econ"] = 1 - p["w_planner_health"]
    p["reward_normalization_factor"] = reward_normalization_factor
    # components
    p["action_cooldown_period"] = int(action_cooldown_period)
    p["subsidy_interval"] = int(subsidy_interval)
    p["num_subsidy_levels"] = int(num_subsidy_levels)
    p["max_daily_subsidy_per_state"] = pop * float(max_annual_subsidy_per_person) / 365   # float64 [S]
    vstart = datetime.strptime(vaccine_delivery_start_date, "%Y-%m-%d")
    p["time_when_vaccine_delivery_begins"] = (vstart - start).days
    p["delivery_interval"] = int(delivery_interval)
    daily_vaccines = (pop / 1e6) * int(daily_vaccines_per_million_people)
    p["num_vaccines_per_delivery"] = np.array(np.floor(int(delivery_interval) * daily_vaccines), dtype=I32)
    t_first = int(p["time_when_vaccine_delivery_begins"])
    while t_first % p["delivery_interval"] != 0:
        t_first += 1
    p["t_first_delivery"] = t_first
    p["time_scale"] = float(episode_length) if allow_observation_scaling else 1.0
    # real-world series used at reset and for lagged stringency before the episode has enough history
    p["rw_policy"] = np.asarray(rw["policy"])                  # int64 [D, S]
    # initial state (covid19_env.py:1175-1215)
    p["init"] = dict(
        susceptible=rw["susceptible"][sdi], infected=rw["infected"][sdi], recovered=rw["recovered"][sdi],
        deaths=rw["recovered"][sdi] * p["death_rate"], unemployed=rw["unemployed"][sdi], vaccinated=rw["vaccinated"][sdi],
        stringency=rw["policy"][sdi],
        stringency_history=np.pad(rw["policy"][: sdi + 1], [(L, 0), (0, 0)], constant_values=1)[-(L + 1):],
    )
    return p


# ---------------------------------------------------------------------------------------------------------
# Registry entries + the batched env (Gym-style surface of CovidAndEconomyEnvironment)
# ---------------------------------------------------------------------------------------------------------
from .components import BaseComponent, component_registry  # noqa: E402
from .scenarios import BaseScenario, scenario_registry  # noqa: E402


@component_registry.add
class ControlUSStateOpenCloseStatus(BaseComponent):
    """reference: components/covid19_components.py:43-96"""
    name = "ControlUSStateOpenCloseStatus"
    agent_subclasses = ["BasicMobileAgent"]

    def __init__(self, *a, n_stringency_levels=10, action_cooldown_period=28, **k):
        super().__init__(*a, **k)
        self.n_stringency_levels = int(n_stringency_levels)
        assert self.n_stringency_levels >= 2
        self.action_cooldown_period = action_cooldown_period

    def get_n_actions(self, agent_cls_name):
        return self.n_stringency_levels if agent_cls_name == "BasicMobileAgent" else None

    def spec_fields(self):
        return dict(n_stringency_levels=self.n_stringency_levels, action_cooldown_period=self.action_cooldown_period)


@component_registry.add
class FederalGovernmentSubsidy(BaseComponent):
    """reference: components/covid19_components.py:241-314"""
    name = "FederalGovernmentSubsidy"
    agent_subclasses = ["BasicPlanner"]

    def __init__(self, *a, subsidy_interval=90, num_subsidy_levels=20, max_annual_subsidy_per_person=20000, **k):
        super().__init__(*a, **k)
        self.subsidy_interval = int(subsidy_interval)
        assert self.subsidy_interval >= 1
        self.num_subsidy_levels = int(num_subsidy_levels)
        assert self.num_subsidy_levels >= 1
        self.max_annual_subsidy_per_person = float(max_annual_subsidy_per_person)
        assert self.max_annual_subsidy_per_person >= 0

    def get_n_actions(self, agent_cls_name):
        return self.num_subsidy_levels if agent_cls_name == "BasicPlanner" else None

    def spec_fields(self):
        return dict(subsidy_interval=self.subsidy_interval, num_subsidy_levels=self.num_subsidy_levels,
                    max_annual_subsidy_per_person=self.max_annual_subsidy_per_person)


@component_registry.add
class VaccinationCampaign(BaseComponent):
    """reference: components/covid19_components.py:465-560 (passive component)"""
    name = "VaccinationCampaign"
    agent_subclasses = ["BasicMobileAgent"]

    def __init__(self, *a, daily_vaccines_per_million_people=4500, delivery_interval=1,
                 vaccine_delivery_start_date="2020-12-22", observe_rate=False, **k):
        super().__init__(*a, **k)
        self.daily_vaccines_per_million_people = int(daily_vaccines_per_million_people)
        assert 0 <= self.daily_vaccines_per_million_people <= 1e6
        self.delivery_interval = int(delivery_interval)
        assert 1 <= self.delivery_interval <= 5000
        self.vaccine_delivery_start_date = vaccine_delivery_start_date
        self.observe_rate = bool(observe_rate)   # adds the `next_vaccination_rate` observation (covid19_components.py:659-661)

    def spec_fields(self):
        return dict(daily_vaccines_per_million_people=self.daily_vaccines_per_million_people,
                    delivery_interval=self.delivery_interval, vaccine_delivery_start_date=self.vaccine_delivery_start_date)


class CovidBatchedEnv:
    """reset()/step() over E replicas of the COVID-19 + economy simulation on one GPU.

    Observations come collated exactly like the reference's mandatory `collate_agent_step_and_reset_data=True`
    layout: obs["a"][key] has the agent (US state) axis last, obs["p"][key] is the planner's; every tensor has
    a leading env axis.  Values are float32 (the reference's own CUDA path also uses float32 placeholders), or with
    obs_dtype=torch.bfloat16 bfloat16: every observation and mask element is the round-to-nearest-even bfloat16 of the
    float32 value, written by the step kernel itself (rewards, done and actions are unchanged).
    """

    def __init__(self, components=None, n_agents=51, world_size=(1, 1), episode_length=540,
                 multi_action_mode_agents=False, multi_action_mode_planner=False, flatten_observations=False,
                 flatten_masks=True, collate_agent_step_and_reset_data=True, allow_observation_scaling=True,
                 use_real_world_data=False, use_real_world_policies=False, n_envs=1, device="cuda:0", auto_reset=True,
                 stepper_factory=None, seed=None, seeds=None, dense_log_frequency=None, world_dense_log_frequency=50,
                 obs_dtype=None, final_obs=False, episode_metrics=False, **scenario_kwargs):
        from .._abi import obs_dtype_name
        self._obs_dtype = obs_dtype_name(obs_dtype)
        if final_obs and not auto_reset:
            raise ValueError("final_obs=True needs auto_reset=True: without the auto-reset, env.obs after the step that "
                             "ends an episode already is its final observation")
        assert collate_agent_step_and_reset_data, \
            "The env. config 'collate_agent_step_and_reset_data' should be set to True."
        if use_real_world_data or use_real_world_policies:
            raise NotImplementedError("replaying real-world data/policies is a host-side mode outside the GPU hot path")
        if multi_action_mode_agents or multi_action_mode_planner or not flatten_masks:
            raise NotImplementedError("the COVID path uses single-action agents/planner and flattened masks")
        kw = dict(episode_length=episode_length, allow_observation_scaling=allow_observation_scaling)
        self._components = []
        for spec in components or []:
            cname, ckw = (spec if isinstance(spec, (tuple, list)) else list(spec.items())[0])
            comp = component_registry.get(cname)(n_agents, episode_length, **ckw)
            self._components.append(comp)
            kw.update(comp.spec_fields())
        names = [c.name for c in self._components]
        assert names == ["ControlUSStateOpenCloseStatus", "FederalGovernmentSubsidy", "VaccinationCampaign"], \
            "the GPU path implements the reference's three COVID components in their canonical order"
        for k in ["start_date", "pop_between_age_18_65", "infection_too_sick_to_work_rate", "risk_free_interest_rate",
                  "economic_reward_crra_eta", "health_priority_scaling_agents", "health_priority_scaling_planner",
                  "reward_normalization_factor", "path_to_data_and_fitted_params"]:
            if k in scenario_kwargs:
                kw[k] = scenario_kwargs.pop(k)
        assert not scenario_kwargs, "unknown kwargs: %s" % list(scenario_kwargs)
        self.params = build_covid_params(**kw)
        assert n_agents == self.params["n_states"], \
            "n_agents should be set to the number of US states, i.e., {}.".format(self.params["n_states"])
        self.name = "CovidAndEconomySimulation"
        self.n_agents, self.n_envs = n_agents, int(n_envs)
        self.num_agents = n_agents + 1
        self.world_size = list(world_size)
        self._episode_length = int(episode_length)
        if stepper_factory is None:
            from ..covid_stepper import CudaCovidStepper
            self._stepper = CudaCovidStepper(self.params, self.n_envs, device=device, auto_reset=auto_reset,
                                             final_obs=bool(final_obs), obs_dtype=self._obs_dtype,
                                             episode_metrics=bool(episode_metrics))
        else:
            # a factory gets final_obs / obs_dtype only when they differ from the defaults, so a three-argument
            # factory keeps working for a default env
            kw = {}
            if final_obs:
                kw["final_obs"] = True
            if self._obs_dtype != "float32":
                kw["obs_dtype"] = self._obs_dtype
            if episode_metrics:
                kw["episode_metrics"] = True
            self._stepper = stepper_factory(self.params, self.n_envs, auto_reset, **kw)
            if episode_metrics and not getattr(self._stepper, "episode_metrics_on", False):
                raise NotImplementedError("episode_metrics=True: the stepper made by stepper_factory keeps no episode-metric "
                                          "accumulators (it needs aie_covid_bind_metrics buffers)")
            if final_obs and not getattr(self._stepper, "final_obs", False):
                raise NotImplementedError("final_obs=True: the stepper made by stepper_factory does not write final "
                                          "observations (it needs final_<name> buffers and a final-observation step)")
            if getattr(self._stepper, "obs_dtype", "float32") != self._obs_dtype:
                raise NotImplementedError("obs_dtype=%s: the stepper made by stepper_factory writes %s observations"
                                          % (self._obs_dtype, getattr(self._stepper, "obs_dtype", "float32")))
        self._final_obs = bool(final_obs)
        self._episode_metrics = bool(episode_metrics)
        self._loaded = False
        self._rollout = None   # bind_rollout
        self._build_views()
        self._build_rate_observation()

    @property
    def episode_length(self):
        return self._episode_length

    @property
    def components(self):
        return self._components

    @property
    def stepper(self):
        return self._stepper

    def seed(self, seed):  # the scenario is deterministic
        return None

    @property
    def action_buffers(self):
        """(agent actions [E, S], planner actions [E]): write in place and call step(env.action_buffers) for zero copies.
        With a rollout bound: slot s of its actions."""
        if self._rollout is not None:
            return self._rollout.actions[min(self._stepper.rollout_slot, self._rollout.T - 1)]
        return self._stepper.buf["actions_agent"], self._stepper.buf["actions_planner"]

    # ------------------------------------------------------------------ rollouts stored in place
    def bind_rollout(self, T, final_obs=False):
        """Store the next rollouts of T steps in place (the contract of BatchedFoundationEnv.bind_rollout): rollout.buf
        holds the seven observation / mask tensors [T + 1, E, ...], actions_agent [T, E, 51], actions_planner [T, E],
        reward_agent [T, E, 51] float32, reward_planner [T, E] float64, done [T, E], and with final_obs (needs auto_reset)
        final_<name> [K, E, ...], K = ceil(T / episode_length), written by the step kernel on the step that ends an
        episode (every replica ends on the same step).  Under VaccinationCampaign(observe_rate=True) also
        rate_agent [T + 1, E, 51] / rate_planner [T + 1, E] and final_rate_agent / final_rate_planner [K, ...]: the
        next_vaccination_rate of each slot, from the same table lookup as env.obs.  rollout.obs[t] / rollout.final_obs[k]
        are env.obs-style views, rollout.rew[t] / rollout.done[t] / rollout.actions[t] those of env.rew, env.done and
        env.action_buffers.  While bound, env.obs and env.action_buffers show slot s, env.rew / env.done the latest
        step's slot, step() advances s and reset() is allowed only at s == 0; env.final_obs is not written.  After T
        steps, restart_rollout() carries slot T into slot 0.  A stepper_factory whose stepper cannot bind rollouts is
        refused with NotImplementedError."""
        _rg.refuse_in_act(self, "bind_rollout")
        _rg.invalidate(self)
        st = self._stepper
        if not hasattr(st, "bind_rollout"):
            raise NotImplementedError("this env's stepper cannot bind rollouts")
        if self._rollout is not None:
            raise ValueError("a rollout is already bound: unbind_rollout() first")
        r = st.bind_rollout(T, final_obs=final_obs)
        b = r.buf
        slot = lambda t: {k: b[k][t] for k in r.obs_names}
        r.obs_slots = [slot(t) for t in range(r.T + 1)]
        r.obs = [self._obs_views(r.obs_slots[t], "") for t in range(r.T + 1)]
        r.final_obs = [self._obs_views({k: b["final_" + k][k_] for k in r.obs_names}, "") for k_ in range(r.K)] \
            if final_obs else None
        r.actions = [(b["actions_agent"][t], b["actions_planner"][t]) for t in range(r.T)]
        r.rew = [{"a": b["reward_agent"][t], "p": b["reward_planner"][t]} for t in range(r.T)]
        r.done = [{"__all__": b["done"][t]} for t in range(r.T)]
        if self._rate_tab is not None:
            E, S = self.n_envs, self.n_agents
            zeros = (lambda sh: np.zeros(sh, self._rate_a.dtype)) if isinstance(self._rate_a, np.ndarray) else \
                (lambda sh: self._rate_a.new_zeros(sh))
            b["rate_agent"], b["rate_planner"] = zeros((r.T + 1, E, S)), zeros((r.T + 1, E))
            for t in range(r.T + 1):
                r.obs[t]["a"]["VaccinationCampaign-next_vaccination_rate"] = b["rate_agent"][t]
                r.obs[t]["p"]["VaccinationCampaign-next_vaccination_rate"] = b["rate_planner"][t]
            if final_obs:
                b["final_rate_agent"], b["final_rate_planner"] = zeros((r.K, E, S)), zeros((r.K, E))
                for k in range(r.K):
                    r.final_obs[k]["a"]["VaccinationCampaign-next_vaccination_rate"] = b["final_rate_agent"][k]
                    r.final_obs[k]["p"]["VaccinationCampaign-next_vaccination_rate"] = b["final_rate_planner"][k]
        self._home_rate = (self._rate_a, self._rate_p) if self._rate_tab is not None else None
        self._rollout = r
        self._aim_rollout()
        if self._loaded:
            self._refresh_rate_observation()
        return r

    def restart_rollout(self):
        """Start the next rollout in the bound tensors (after its T steps): slot T moves to slot 0."""
        _rg.refuse_in_act(self, "restart_rollout")
        if self._rollout is None:
            raise ValueError("no rollout bound")
        self._stepper.restart_rollout()
        r = self._rollout
        if self._rate_tab is not None:
            r.buf["rate_agent"][0][...] = r.buf["rate_agent"][r.T]
            r.buf["rate_planner"][0][...] = r.buf["rate_planner"][r.T]
        self._aim_rollout()

    def capture_rollout(self, act):
        """Record the bound rollout's T steps once as a CUDA graph (the contract of
        BatchedFoundationEnv.capture_rollout).  The step finds the final-slot row of an episode end on the device, and
        under VaccinationCampaign(observe_rate=True) the rate lookups are device-side torch ops of each slot, recorded
        with the step."""
        return _rg.capture_rollout(self, act)

    def unbind_rollout(self):
        _rg.refuse_in_act(self, "unbind_rollout")
        _rg.invalidate(self)
        if self._rollout is None:
            return
        self._stepper.unbind_rollout()
        self._rollout = None
        if self._home_rate is not None:
            self._rate_a, self._rate_p = self._home_rate
        self._build_views()
        if self._rate_tab is not None:
            self.obs["a"]["VaccinationCampaign-next_vaccination_rate"] = self._rate_a
            self.obs["p"]["VaccinationCampaign-next_vaccination_rate"] = self._rate_p
            if self.final_obs is not None:
                self.final_obs["a"]["VaccinationCampaign-next_vaccination_rate"] = self._final_rate_a
                self.final_obs["p"]["VaccinationCampaign-next_vaccination_rate"] = self._final_rate_p

    @property
    def rollout(self):
        return self._rollout

    def _aim_rollout(self):
        r, s = self._rollout, self._stepper.rollout_slot
        self.obs = r.obs[s]
        self.rew, self.done = r.rew[max(s - 1, 0)], r.done[max(s - 1, 0)]
        if self._rate_tab is not None:
            self._rate_a, self._rate_p = r.buf["rate_agent"][s], r.buf["rate_planner"][s]

    def sample_actions(self, logits_agent, logits_planner=None, *, seed, greedy=False, out=None):
        """A policy's actions, drawn on the device into `action_buffers` from the softmax of its logits restricted to the
        open entries of the current masks (greedy=True: the masked argmax).  logits_agent: [E, 51, 1 + stringency levels]
        (action axis last; obs["a"]["action_mask"] is [E, 1 + levels, 51]); logits_planner: [E, 1 + subsidy levels];
        contiguous float32 or bfloat16 on the env's device.  Returns (log_prob_agent [E, 51], log_prob_planner [E]),
        float32: buffers of the env reused by the next call, or the caller's `out` tensors.  Asynchronous."""
        return self._stepper.sample_policy(logits_agent, logits_planner, seed=seed, greedy=greedy, out=out)

    def evaluate_actions(self, logits_agent, logits_planner, actions, masks):
        """Log-probabilities and entropies of stored actions (the contract of BatchedFoundationEnv.evaluate_actions):
        logits_agent [*B, 51, 1 + stringency levels], logits_planner [*B, 1 + subsidy levels]; masks = (mask_agent
        [*B, 1 + levels, 51] as obs["a"]["action_mask"], mask_planner [*B, 1 + subsidy levels]); actions =
        (actions_agent [*B, 51], actions_planner [*B]), int32.  Returns (log_prob_agent [*B, 51], log_prob_planner
        [*B], entropy_agent [*B, 51], entropy_planner [*B]), differentiable with respect to both logits tensors."""
        _rg.refuse_in_act(self, "evaluate_actions")
        return self._stepper.evaluate_actions(logits_agent, logits_planner, actions, masks)

    def compute_advantages(self, rewards, values, dones, last_values, final_values=None, *, gamma, lam=1.0,
                           per_episode_end=False):
        """Advantages and value targets of a stored rollout (the contract of BatchedFoundationEnv.compute_advantages),
        A = 51 states: rewards = (rew["a"] [T, E, 51] float32, rew["p"] [T, E] float64) stacked over the steps, values
        = (agent, planner) float32 of the same shapes, dones int32 [T, E], last_values = ([E, 51], [E]).  Every episode
        ends on its time limit, so it is truncated: final_values = the values of env.final_obs stored at each step
        (env created with final_obs=True) bootstraps it; final_values=None treats an episode end as terminal.  A bound
        rollout: (rollout.buf["reward_agent"], rollout.buf["reward_planner"]), rollout.buf["done"] and, with
        per_episode_end=True, the values of its [K, ...] final slots."""
        _rg.refuse_in_act(self, "compute_advantages")
        return self._stepper.compute_advantages(rewards, values, dones, last_values, final_values, gamma=gamma, lam=lam,
                                                per_episode_end=per_episode_end)

    # ------------------------------------------------------------------ episode metrics (episode_metrics=True)
    # scenario_metrics() (covid19_env.py:1613-1687) of every replica, from accumulators the step kernel keeps on the
    # device: float64 time sums of the stored float32 series, float32 index sums as the reference keeps them.  A row is
    # one launch away from metrics_tensor(); the dict forms copy it to the host.  Every replica ends its episodes on the
    # same step, so previous_episode_metrics exists for all of them or for none.
    def _need_metrics(self):
        if not self._episode_metrics:
            raise ValueError("episode metrics need make_env_instance(\"CovidAndEconomySimulation\", ..., "
                             "episode_metrics=True)")
        assert self._loaded, "call reset() first"

    @property
    def metric_keys(self):
        """Column order of metrics_tensor() / previous_episode_metrics_tensor(): the reference's scenario_metrics() keys,
        eight per state ("<state name>/<field>") then seven "usa/<field>", K = 8 * 51 + 7 = 415."""
        self._need_metrics()
        return [k for k, _ in self._stepper.metric_layout()]

    def metrics_tensor(self, out=None):
        """scenario_metrics() of every replica's running episode as one float64 tensor [n_envs, K] on the device (columns:
        metric_keys), one kernel launch, no synchronisation.  Mid-episode the time means divide by episode_length, as the
        reference's zero-padded global_state does.  out: an optional contiguous float64 [n_envs, K] tensor."""
        _rg.refuse_in_act(self, "metrics_tensor")
        self._need_metrics()
        return self._stepper.episode_metrics(final=False, out=out)

    def previous_episode_metrics_tensor(self, out=None):
        """scenario_metrics() of the episode every replica finished last, float64 [n_envs, K] on the device, one launch.
        Before any episode has ended the library's AieError is raised (previous_episode_metrics is None then)."""
        _rg.refuse_in_act(self, "previous_episode_metrics_tensor")
        self._need_metrics()
        return self._stepper.episode_metrics(final=True, out=out)

    def metrics_rows_as_dicts(self, rows, envs=None):
        """Rows of metrics_tensor() / previous_episode_metrics_tensor() ([n, K], tensor or array) as the dicts
        metrics_of(e) returns, in metric_keys order (floats).  envs: the row indices (default: all).  Copies to the host."""
        self._need_metrics()
        a = rows.detach().cpu().numpy() if hasattr(rows, "detach") else np.asarray(rows)
        a = np.asarray(a, np.float64).reshape(-1, a.shape[-1])
        keys = self.metric_keys
        return [dict(zip(keys, a[int(e)].tolist())) for e in (range(a.shape[0]) if envs is None else envs)]

    @property
    def metrics(self):
        """scenario_metrics() of replica 0's running episode (BaseEnvironment.metrics)."""
        _rg.refuse_in_act(self, "metrics")
        return self.metrics_of(0)

    def metrics_of(self, e):
        _rg.refuse_in_act(self, "metrics_of")
        return self.metrics_rows_as_dicts(self.metrics_tensor(), envs=[e])[0]

    @property
    def previous_episode_metrics(self):
        """scenario_metrics() of the episode replica 0 finished last; None before any has ended."""
        _rg.refuse_in_act(self, "previous_episode_metrics")
        return self.previous_episode_metrics_of(0)

    def previous_episode_metrics_of(self, e):
        _rg.refuse_in_act(self, "previous_episode_metrics_of")
        self._need_metrics()
        if not self._stepper.has_previous_episode():
            return None
        return self.metrics_rows_as_dicts(self.previous_episode_metrics_tensor(), envs=[e])[0]

    def _build_views(self):
        b = self._stepper.buf
        self.obs = self._obs_views(b, "")
        # final_obs=True: env.final_obs mirrors env.obs over the final_<name> buffers.  After a step, row e of a replica
        # with done["__all__"][e] == 1 holds the observation of the state its episode ended in (env.obs already shows the
        # next episode's first); the other rows keep whatever an earlier episode end wrote.  reset() does not touch them.
        self.final_obs = self._obs_views(b, "final_") if self._final_obs else None
        self.rew = {"a": b["reward_agent"], "p": b["reward_planner"]}
        self.done = {"__all__": b["done"]}
        self.info = {"a": {}, "p": {}}

    def _obs_views(self, b, prefix):
        """The collated "a" / "p" observation dict over the observation / mask buffers b[prefix + name]."""
        g = lambda k: b[prefix + k]
        S = self.n_agents
        sc = g("obs_scalars")
        exp = (lambda v: v[:, None].expand(-1, S)) if hasattr(sc, "expand") else (lambda v: np.repeat(v[:, None], S, axis=1))
        return {
            "a": {"world-agent_state": g("obs_agent_state"), "world-agent_postsubsidy_productivity": g("obs_postsubsidy"),
                  "world-lagged_stringency_level": g("obs_lagged_stringency"), "time": exp(sc[:, 0]),
                  "ControlUSStateOpenCloseStatus-agent_policy_indicators": g("obs_policy_indicators"),
                  "FederalGovernmentSubsidy-t_until_next_subsidy": exp(sc[:, 1]),
                  "FederalGovernmentSubsidy-current_subsidy_level": exp(sc[:, 2]),
                  "VaccinationCampaign-t_until_next_vaccines": exp(sc[:, 3]), "action_mask": g("mask_agent")},
            "p": {"world-agent_state": g("obs_agent_state"), "world-agent_postsubsidy_productivity": g("obs_postsubsidy"),
                  "world-lagged_stringency_level": g("obs_lagged_stringency"), "time": sc[:, 0:1],
                  "ControlUSStateOpenCloseStatus-agent_policy_indicators": g("obs_policy_indicators"),
                  "FederalGovernmentSubsidy-t_until_next_subsidy": sc[:, 1],
                  "FederalGovernmentSubsidy-current_subsidy_level": sc[:, 2],
                  "VaccinationCampaign-t_until_next_vaccines": sc[:, 3], "action_mask": g("mask_planner")},
        }

    def _build_rate_observation(self):
        """VaccinationCampaign(observe_rate=True) (covid19_components.py:629-661): the vaccination rate of the NEXT timestep, 0
        until deliveries have begun.  It depends on the timestep alone, so it is a table lookup by the replica's timestep after
        every step / reset (the reference's own CUDA path does not emit it; no kernel involved).  The table and the rate
        tensors have the observations' element type: under bfloat16 each entry is the round-to-nearest-even of the
        float32 rate (raw bits on numpy backends, as the stepper's observation buffers)."""
        vac = self._components[2]
        self._rate_tab = None
        if not vac.observe_rate:
            return
        T, t_first = self._episode_length, int(self.params["t_first_delivery"])
        rate = np.float32(vac.daily_vaccines_per_million_people / 1e6)
        tab = np.array([np.float32(0.0) if t + 1 <= t_first else rate for t in range(T + 1)], np.float32)
        sc = self._stepper.buf["obs_scalars"]
        E, S = self.n_envs, self.n_agents
        if isinstance(sc, np.ndarray):
            if sc.dtype == np.uint16:   # raw bfloat16 bits, rounded to nearest even (the rates are finite)
                u = tab.view(np.uint32)
                tab = ((u + np.uint32(0x7FFF) + ((u >> 16) & np.uint32(1))) >> 16).astype(np.uint16)
            self._rate_tab, self._rate_a, self._rate_p = tab, np.zeros((E, S), tab.dtype), np.zeros(E, tab.dtype)
        else:
            import torch
            self._rate_tab = torch.as_tensor(tab, device=sc.device).to(sc.dtype)
            self._rate_a, self._rate_p = torch.zeros((E, S), dtype=sc.dtype, device=sc.device), torch.zeros(E, dtype=sc.dtype, device=sc.device)
        self.obs["a"]["VaccinationCampaign-next_vaccination_rate"] = self._rate_a
        self.obs["p"]["VaccinationCampaign-next_vaccination_rate"] = self._rate_p
        if self.final_obs is not None:
            if isinstance(sc, np.ndarray):
                self._final_rate_a, self._final_rate_p = np.zeros_like(self._rate_a), np.zeros_like(self._rate_p)
            else:
                self._final_rate_a, self._final_rate_p = torch.zeros_like(self._rate_a), torch.zeros_like(self._rate_p)
            self.final_obs["a"]["VaccinationCampaign-next_vaccination_rate"] = self._final_rate_a
            self.final_obs["p"]["VaccinationCampaign-next_vaccination_rate"] = self._final_rate_p

    def _timesteps(self):
        """Each replica's timestep: from the float32 time scalar t / time_scale, which holds it exactly, or under bfloat16
        observations from hdr[:, 0] (a bfloat16 t / 540 spans one to two timesteps)."""
        b = self._stepper.buf
        sc = b["obs_scalars"] if self._rollout is None else self._rollout.obs_slots[self._stepper.rollout_slot]["obs_scalars"]
        scale = float(self.params["time_scale"])
        if isinstance(sc, np.ndarray):
            return b["hdr"][:, 0] if sc.dtype == np.uint16 else np.rint(sc[:, 0].astype(np.float64) * scale).astype(np.int64)
        import torch
        return b["hdr"][:, 0].long() if sc.dtype == torch.bfloat16 else torch.round(sc[:, 0].double() * scale).long()

    def _refresh_rate_observation(self, stepped=False):
        """The table's rates at each replica's timestep.  The final rows are those of episodes that ended on their time
        limit, so their rate is the table's last entry (t = episode_length)."""
        if self._rate_tab is None:
            return
        b = self._stepper.buf
        rate = self._rate_tab[self._timesteps()]
        if isinstance(rate, np.ndarray):
            self._rate_p[...] = rate
            self._rate_a[...] = self._rate_p[:, None]
        else:
            self._rate_p.copy_(rate)
            self._rate_a.copy_(self._rate_p[:, None].expand_as(self._rate_a))
        if stepped and self._rollout is not None:
            r, s = self._rollout, self._stepper.rollout_slot
            if r.final_obs is not None and s >= 1:
                # the rows of the episodes this step ended, at their final slot k (the episode ends before it in the rollout)
                done, last = r.buf["done"][s - 1] != 0, self._rate_tab[self._episode_length]
                before = r.buf["done"][:s - 1].sum(0) if s > 1 else done * 0
                fa, fp = r.buf["final_rate_agent"], r.buf["final_rate_planner"]
                for k in range(r.K):
                    m = done & (before == k)
                    if isinstance(m, np.ndarray):
                        fp[k][...] = np.where(m, last, fp[k])
                        fa[k][...] = np.where(m[:, None], last, fa[k])
                    else:
                        import torch
                        fp[k].copy_(torch.where(m, last, fp[k]))
                        fa[k].copy_(torch.where(m[:, None], last, fa[k]))
        elif stepped and self.final_obs is not None:
            # only the rows of the episodes this step ended
            done = b["done"] != 0
            last = self._rate_tab[self._episode_length]
            if isinstance(done, np.ndarray):
                self._final_rate_p[...] = np.where(done, last, self._final_rate_p)
                self._final_rate_a[...] = np.where(done[:, None], last, self._final_rate_a)
            else:
                import torch
                self._final_rate_p.copy_(torch.where(done, last, self._final_rate_p))
                self._final_rate_a.copy_(torch.where(done[:, None], last, self._final_rate_a))

    # ------------------------------------------------------------------ checkpoints
    def _checkpoint_config(self):
        from .._abi import ABI_VERSION
        return dict(scenario=self.name, n_envs=self.n_envs, obs_dtype=self._obs_dtype,
                    auto_reset=getattr(self._stepper, "_auto_reset", None), final_obs=self._final_obs,
                    episode_metrics=self._episode_metrics, observe_rate=self._rate_tab is not None,
                    abi_version=ABI_VERSION, spec=self.params)

    def _checkpoint_buffers(self):
        """name -> the buffer a checkpoint holds: the simulation state, the observations, masks, rewards, done and
        actions env.obs / env.rew / env.done / env.action_buffers show (slot 0 of a bound rollout), the final
        observations, the rate observations and the episode-metric accumulators."""
        st, r = self._stepper, self._rollout
        out = {k: st.buf[k] for k in ("state", "ints", "hdr", "ring", "changes") if k in st.buf}
        obs = st.buf if r is None else r.obs_slots[0]
        out.update({k: obs[k] for k in COVID_OBS_NAMES})
        out["actions_agent"], out["actions_planner"] = self.action_buffers
        src = st.buf if r is None else {k: r.buf[k][0] for k in ("reward_agent", "reward_planner", "done")}
        out.update({k: src[k] for k in ("reward_agent", "reward_planner", "done")})
        out.update({k: v for k, v in st.buf.items() if k.startswith("final_") or k.startswith("metric_")})
        if self._rate_tab is not None:
            out["rate_agent"], out["rate_planner"] = self._rate_a, self._rate_p
            if self._final_obs:
                out["final_rate_agent"], out["final_rate_planner"] = self._final_rate_a, self._final_rate_p
        return out

    def state_dict(self):
        """The whole state of the batched env between steps (the contract of BatchedFoundationEnv.state_dict): the
        simulation buffers, observations, rewards, actions, final observations and metric accumulators (copies on the
        env's device), the library's sampler counters and the lock-step timestep.  Allowed after the first reset();
        with a rollout bound only at slot 0 (ValueError otherwise)."""
        _rg.refuse_in_act(self, "state_dict")
        from . import checkpoint as ck
        if not self._loaded:
            raise ValueError("state_dict: nothing to save before the first reset()")
        ck.refuse_mid_rollout(self, "state_dict")
        if not hasattr(self._stepper, "get_counters"):
            raise NotImplementedError("this env's stepper keeps no checkpointable counters")
        return dict(format_version=ck.FORMAT_VERSION, config=ck.plain(self._checkpoint_config()),
                    buffers={k: ck.snapshot(v) for k, v in self._checkpoint_buffers().items()},
                    counters=self._stepper.get_counters())

    def load_state_dict(self, sd):
        """Load a state_dict() taken from an env of the same configuration (ValueError naming the field that differs)
        into this env's own buffers; with a rollout bound only at slot 0, whose observations it writes.  Allowed on a
        new env before any reset()."""
        _rg.refuse_in_act(self, "load_state_dict")
        _rg.invalidate(self)
        from . import checkpoint as ck
        ck.check_config(sd, self._checkpoint_config())
        ck.refuse_mid_rollout(self, "load_state_dict")
        mine = self._checkpoint_buffers()
        if set(sd["buffers"]) != set(mine):
            raise ValueError("load_state_dict: the checkpoint holds buffers %s, this env %s"
                             % (sorted(sd["buffers"]), sorted(mine)))
        for k, dst in mine.items():
            ck.copy_into(dst, sd["buffers"][k], k)
        self._stepper.set_counters(sd["counters"])
        self._loaded = True
        return self.obs

    def reset(self):
        _rg.refuse_in_act(self, "reset")
        if self._rollout is not None and self._stepper.rollout_slot != 0:
            _rg.invalidate(self)   # refused below: the graph's rollout was left mid-way
        self._stepper.reset()
        self._loaded = True
        if self._rollout is not None:
            self._aim_rollout()
        self._refresh_rate_observation()
        return self.obs

    def step(self, actions=None):
        """actions: None | {"a": int tensor [E, 51], "p": int tensor [E]} | (agent_actions, planner_actions)."""
        _rg.refuse_in_act(self, "step")
        assert self._loaded, "call reset() first"
        ba, bp = self.action_buffers
        if actions is None:
            ba[...] = 0
            bp[...] = 0
        else:
            a, p = (actions.get("a"), actions.get("p")) if isinstance(actions, dict) else actions
            for buf, v in ((ba, a), (bp, p)):
                if v is None:
                    buf[...] = 0
                elif v is not buf:
                    if isinstance(buf, np.ndarray):
                        buf[...] = np.asarray(v, dtype=buf.dtype).reshape(buf.shape)
                    else:
                        import torch
                        buf[...] = torch.as_tensor(np.asarray(v) if not isinstance(v, torch.Tensor) else v,
                                                   device=buf.device).to(buf.dtype).reshape(buf.shape)
        self._stepper.step()
        if self._rollout is not None:
            self._aim_rollout()
        self._refresh_rate_observation(stepped=True)
        return self.obs, self.rew, self.done, self.info


@scenario_registry.add
class CovidAndEconomySimulation(BaseScenario):
    """Registry entry; make_env_instance routes this name to CovidBatchedEnv."""
    name = "CovidAndEconomySimulation"
    env_class = CovidBatchedEnv
