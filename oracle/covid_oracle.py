"""TEST INFRASTRUCTURE ONLY — numpy restatement of the reference's COVID-19 + economy step (BASELINE config 4).

Follows, per env replica, the Python (CPU) path of
    ControlUSStateOpenCloseStatus.component_step   components/covid19_components.py:145-221
    FederalGovernmentSubsidy.component_step        components/covid19_components.py:361-443
    VaccinationCampaign.component_step             components/covid19_components.py:593-627
    CovidAndEconomyEnvironment.scenario_step       scenarios/covid19/covid19_env.py:650-917
      sir_step :1477-1515, unemployment_step :1374-1441, economy_step :1444-1475
    generate_observations :919-993 (+ component observations / masks), compute_reward :995-1173
with numpy arrays of the reference's own dtypes, so numpy's type promotion reproduces the reference's mixed
float32 / int32 / float64 arithmetic.  State is held as plain arrays (no agent dicts).  The derived constants
come from ai_economist_b200.foundation.covid19.build_covid_params (checked bit-for-bit against the reference
constructor in tests/test_covid.py).

Parity status: PINNED by tests/golden/covid_*.npz (recorded from the unmodified reference, oracle/gen_golden_covid.py).
Only tests/, bench.py's CPU legs and __graft_entry__.smoke() may import this module.
"""
import numpy as np

F32, I32 = np.float32, np.int32


def _softplus(x, beta=1, threshold=20):
    return 1 / beta * np.log(1 + np.exp(beta * x)) * (beta * x <= threshold) + x * (beta * x > threshold)


class CovidOracleEnv:
    def __init__(self, params, auto_reset=False):
        # auto_reset: a step that ends the episode resets the env, as the product's auto-reset does: the observations are
        # the fresh episode's, the rewards and `done` those of the step that ended the finished one
        self.p = params
        self.auto_reset = auto_reset
        self.episodes = 0
        self.reset()

    def reset(self):
        p = self.p
        T, S = p["episode_length"], p["n_states"]
        ini = p["init"]
        self.t = 0
        z = lambda: np.zeros((T + 1, S), dtype=F32)
        self.gs = {k: z() for k in ["Susceptible", "Infected", "Recovered", "Deaths", "Unemployed", "Vaccinated",
                                    "Stringency Level", "Subsidy", "Postsubsidy Productivity"]}
        for k, src in [("Susceptible", "susceptible"), ("Infected", "infected"), ("Recovered", "recovered"),
                       ("Deaths", "deaths"), ("Unemployed", "unemployed"), ("Vaccinated", "vaccinated"),
                       ("Stringency Level", "stringency")]:
            self.gs[k][0] = ini[src]
        self.hist = np.array(ini["stringency_history"])          # [L+1, S]
        self.cooldown_until = np.zeros(S, dtype=np.int64)        # additional_reset_steps: world.timestep == 0
        self.subsidy_level = I32(0)
        self.vaccines_available = np.zeros(S, dtype=np.int64)
        self.rew_a = np.zeros(S, dtype=F32)
        self.rew_p = 0.0
        self.done = 0

    # ------------------------------------------------------------------ step
    def step(self, act_a, act_p):
        p, gs = self.p, self.gs
        S = p["n_states"]
        self.t += 1
        t = self.t
        act_a = np.asarray(act_a).reshape(S)
        # ControlUSStateOpenCloseStatus (per-agent scalar arithmetic in the reference)
        for a in range(S):
            action = int(act_a[a])
            gs["Stringency Level"][t, a] = gs["Stringency Level"][t - 1, a] * (action == 0) + action
            if t == self.cooldown_until[a] + 1:
                self.cooldown_until[a] += 1 if action == 0 else p["action_cooldown_period"]
        # FederalGovernmentSubsidy
        if (t - 1) % p["subsidy_interval"] == 0:
            subsidy_level = int(act_p)
        else:
            subsidy_level = self.subsidy_level
        self.subsidy_level = np.array(subsidy_level).astype(I32)
        gs["Subsidy"][t] = (subsidy_level / p["num_subsidy_levels"]) * p["max_daily_subsidy_per_state"]
        # VaccinationCampaign
        if t >= p["time_when_vaccine_delivery_begins"] and (t % p["delivery_interval"]) == 0:
            self.vaccines_available = self.vaccines_available + p["num_vaccines_per_delivery"]
        # scenario_step
        bd, sdi = p["beta_delay"], p["start_date_index"]
        if t - bd < 0:
            tmk = np.ones(S) if sdi + t - bd < 0 else p["rw_policy"][sdi + t - bd, :]
        else:
            tmk = gs["Stringency Level"][t - bd]
        tmk = tmk.astype(I32)
        S_tm1, I_tm1, R_tm1, V_tm1 = (gs[k][t - 1] for k in ("Susceptible", "Infected", "Recovered", "Vaccinated"))
        vacc_avail = np.zeros(S, dtype=I32)
        vacc_avail[:] = self.vaccines_available
        self.vaccines_available = np.zeros(S, dtype=np.int64)
        dS, dI, dR, dV = self._sir(S_tm1, I_tm1, tmk, vacc_avail)
        S_t = np.maximum(S_tm1 + dS, 0)
        I_t = np.maximum(I_tm1 + dI, 0)
        R_t = np.maximum(R_tm1 + dR, 0)
        V_t = np.maximum(V_tm1 + dV, 0)
        D_t = p["death_rate"] * (R_t - V_t)
        gs["Susceptible"][t], gs["Infected"][t], gs["Recovered"][t] = S_t, I_t, R_t
        gs["Deaths"][t], gs["Vaccinated"][t] = D_t, V_t
        unemployed = self._unemployment(gs["Stringency Level"][t])
        gs["Unemployed"][t] = unemployed
        productivity = self._economy(I_t, D_t, unemployed)
        gs["Postsubsidy Productivity"][t] = productivity + gs["Subsidy"][t]
        self._reward()
        self.done = int(t >= p["episode_length"])
        if self.auto_reset and self.done:
            rew_a, rew_p = self.rew_a, self.rew_p
            self.reset()
            self.rew_a, self.rew_p, self.done = rew_a, rew_p, 1
            self.episodes += 1
        return self.obs()

    def _sir(self, S_tm1, I_tm1, tmk, vacc_avail):
        p = self.p
        S = p["n_states"]
        intercepts = p["beta_intercepts"] * 1
        slopes = p["beta_slopes"] * 1
        beta_i = (intercepts + slopes * tmk).astype(F32)
        frac_vacc = np.minimum(np.ones(S, dtype=I32), vacc_avail / (S_tm1 + 1e-10)).astype(F32)
        vaccinated = np.minimum(vacc_avail, S_tm1)
        si_over_n = (S_tm1 / p["population"]) * I_tm1
        dS = (-beta_i * si_over_n * (1 - frac_vacc) - vaccinated).astype(F32)
        dR = (p["gamma"] * I_tm1 + vaccinated).astype(F32)
        dI = -dS - dR
        return dS, dI, dR, vaccinated.astype(F32)

    def _unemployment(self, current):
        p = self.p
        L = p["filter_len"]
        self.hist = np.concatenate((self.hist[1:], current.reshape(1, -1)))
        delta = (self.hist[1:] - self.hist[:-1]) * 1
        x = delta[None].transpose(2, 0, 1)
        weighted = x * np.repeat(p["conv_weights"][:, :, None], L, axis=-1)
        excess = _softplus(np.sum(weighted * p["conv_filters"][None], axis=(1, 2)), beta=1)
        return (excess + p["unemployment_bias"]) * p["population"] / 100

    def _economy(self, infected, deaths, unemployed):
        p = self.p
        incapacitated = (p["infection_too_sick_to_work_rate"] * infected) + deaths
        cant_work = (incapacitated * p["pop_between_age_18_65"]) + unemployed
        can_work = np.maximum(0, p["population"] * p["pop_between_age_18_65"] - cant_work)
        return (can_work * p["daily_production_per_worker"]).astype(F32)

    def _reward(self):
        p, gs, t = self.p, self.gs, self.t
        eta = p["crra_eta"]

        def crra(x):
            ax = 365 * x
            axc = np.clip(ax, 0.1, 3)
            return (1 + (axc ** (1 - eta) - 1) / (1 - eta)) / 365

        def mm(x, lo, hi):
            return (x - lo) / (hi - lo + 1e-10)

        def wavg(wh, h, we, e):
            return (wh * h + we * e) / (wh + we)

        md = gs["Deaths"][t] - gs["Deaths"][t - 1]
        subsidy, post = gs["Subsidy"][t], gs["Postsubsidy Productivity"][t]
        h = (-md.astype(F32) * p["value_of_life"] / p["agents_health_norm"]).astype(F32)
        e = crra(post / p["agents_economic_norm"]).astype(F32)
        h = mm(h, p["min_marginal_agent_health_index"], p["max_marginal_agent_health_index"]).astype(F32)
        e = mm(e, p["min_marginal_agent_economic_index"], p["max_marginal_agent_economic_index"]).astype(F32)
        self.rew_a = wavg(p["w_agent_health"], h, p["w_agent_econ"], e) / p["reward_normalization_factor"]
        ph = -np.sum(md).astype(F32) * p["value_of_life"] / p["planner_health_norm"]
        cost = (1 + p["risk_free_interest_rate"]) * np.sum(subsidy)
        pe = crra((np.sum(post) - cost) / p["planner_economic_norm"])
        ph = mm(ph, p["min_marginal_planner_health_index"], p["max_marginal_planner_health_index"])
        pe = mm(pe, p["min_marginal_planner_economic_index"], p["max_marginal_planner_economic_index"])
        self.rew_p = wavg(p["w_planner_health"], ph, p["w_planner_econ"], pe) / p["reward_normalization_factor"]

    # ------------------------------------------------------------------ observations / masks
    def obs(self):
        """Arrays in the product's output layout (float32)."""
        p, gs, t = self.p, self.gs, self.t
        S = p["n_states"]
        feats = np.vstack([gs[k][t] for k in ["Susceptible", "Infected", "Recovered", "Deaths", "Vaccinated", "Unemployed"]])
        agent_state = feats / p["population"][None]
        post = gs["Postsubsidy Productivity"][t] / p["maximum_productivity"]
        t_beta = t - p["beta_delay"] + 1
        lag = p["rw_policy"][p["start_date_index"] + t_beta] if t_beta < 0 else gs["Stringency Level"][t_beta]
        lag = lag / p["num_stringency_levels"]
        policy_ind = gs["Stringency Level"][t] / p["num_stringency_levels"]
        t_until_sub = (p["subsidy_interval"] - t % p["subsidy_interval"]) / p["subsidy_interval"]
        sub_level = self.subsidy_level / p["num_subsidy_levels"]
        nxt = t + 1
        if nxt <= p["t_first_delivery"]:
            t_vac = np.minimum(1, (p["t_first_delivery"] - nxt) / p["delivery_interval"])
        else:
            t_vac = p["delivery_interval"] - nxt % p["delivery_interval"]
        t_vac = t_vac / p["delivery_interval"]
        mask_a = np.zeros((1 + p["num_stringency_levels"], S), dtype=F32)
        mask_a[0] = 1
        mask_a[1:, :] = (t >= self.cooldown_until)[None].astype(F32)
        mask_p = np.zeros(1 + p["num_subsidy_levels"], dtype=F32)
        mask_p[0] = 1
        mask_p[1:] = 1.0 if t % p["subsidy_interval"] == 0 else 0.0
        return dict(
            agent_state=agent_state.astype(F32), postsubsidy=np.asarray(post, F32), lagged=np.asarray(lag, F32),
            policy_ind=np.asarray(policy_ind, F32),
            scalars=np.array([t / p["time_scale"], t_until_sub, sub_level, t_vac], F32),
            mask_a=mask_a, mask_p=mask_p, rew_a=np.asarray(self.rew_a, F32), rew_p=np.float64(self.rew_p),
            done=np.int32(self.done))

    def state(self):
        gs, t = self.gs, self.t
        return dict(t=t, susceptible=gs["Susceptible"][t], infected=gs["Infected"][t], recovered=gs["Recovered"][t],
                    deaths=gs["Deaths"][t], vaccinated=gs["Vaccinated"][t], unemployed=gs["Unemployed"][t],
                    stringency=gs["Stringency Level"][t], subsidy=gs["Subsidy"][t],
                    postsubsidy=gs["Postsubsidy Productivity"][t], cooldown_until=self.cooldown_until.copy(),
                    subsidy_level=int(self.subsidy_level), vaccines_available=self.vaccines_available.copy(),
                    episodes=self.episodes)


class CovidOracleBatch:
    def __init__(self, params, n_envs, auto_reset=False):
        self.envs = [CovidOracleEnv(params, auto_reset) for _ in range(n_envs)]

    def step(self, act_a, act_p):
        for e, env in enumerate(self.envs):
            env.step(act_a[e], act_p[e])

    def obs(self, e):
        return self.envs[e].obs()

    def state(self, e):
        return self.envs[e].state()
