// TEST / BASELINE INFRASTRUCTURE - not part of the product, never loaded by ai_economist_b200/.
//
// Host-side launcher for the REFERENCE's own COVID-19 CUDA kernels, so that they can be run and timed on the same
// GPU as aie_covid_step_kernel (BASELINE.md config 4: the reference's CUDA kernels as an additional bar where they can be
// built).  The kernels are NOT copied: this file #includes the reference's build unit where it lies in a
// reference checkout at compile time (REF_COVID_BUILD_CU, passed by oracle/build_ref_covid.py), and the output goes to
// oracle/_ref/ (git-ignored).  What is written here is only the launch sequence, which in the reference lives in
// Python on top of WarpDrive / PyCUDA (not a dependency of this project):
//   components/covid19_components.py:145-172, 355-383, 587-608   component_step() GPU branches, in component order
//   scenarios/covid19/covid19_env.py:650-705                      scenario_step() GPU branch (includes observations)
//   scenarios/covid19/covid19_env.py:995-1040                     compute_reward() GPU branch
// with the reference's launch geometry: grid = (num_envs), block = (n_agents incl. the planner) (env_wrapper.py /
// WarpDrive CUDAFunctionManager).
#include <assert.h>
#include <cuda_runtime.h>
#include <stdint.h>

#ifndef REF_COVID_BUILD_CU
#error "compile with -DREF_COVID_BUILD_CU=\"/root/reference/.../covid19_build.cu\" (oracle/build_ref_covid.py)"
#endif
#include REF_COVID_BUILD_CU

// Everything the five kernels take, by the data-dictionary names of the reference (covid19_env.py:388-636,
// covid19_components.py:110-136, 327-352, 562-584).  Device pointers unless noted.
struct RefCovidArgs {
    // time-dependent state [E, T+1, S]
    float *susceptible, *infected, *recovered, *deaths, *vaccinated, *unemployed, *subsidy, *productivity,
        *postsubsidy_productivity;
    int *stringency_level, *subsidy_level;
    // per-env scratch / state
    float *beta, *incapacitated, *cant_work, *num_people_that_can_work;   // [E, S]
    int *delta_stringency_level;                                           // [E, L, S]
    float *signal;                                                         // [E, S, F, L]
    int *action_in_cooldown_until, *num_vaccines_available_t;              // [E, S]
    int *timestep, *done;                                                  // [E]
    // constants
    const int *default_agent_action_mask, *no_op_agent_action_mask;        // [NS + 1]
    const int *default_planner_action_mask, *no_op_planner_action_mask;    // [NL + 1]
    const float *max_daily_subsidy_per_state;                              // [S]
    const int *num_vaccines_per_delivery, *us_state_population;            // [S]
    const int *real_world_stringency_policy_history;                       // [beta_delay - 1, S]
    const float *beta_slopes, *beta_intercepts;                            // [S]
    const float *grouped_convolutional_filter_weights;                     // [S, F]
    const float *unemp_conv_filters;                                       // [F, L]
    const float *unemployment_bias, *maximum_productivity;                 // [S]
    const float *min_marginal_agent_health_index, *max_marginal_agent_health_index,
        *min_marginal_agent_economic_index, *max_marginal_agent_economic_index;   // [S]
    const float *weightage_on_marginal_agent_health_index, *weightage_on_marginal_agent_economic_index;   // [S]
    const float *agents_health_norm, *agents_economic_norm;                // [S]
    // actions in, observations / rewards out
    int *actions_a, *actions_p;                                            // [E, S], [E]
    float *obs_a_policy_indicators, *obs_a_action_mask, *obs_p_policy_indicators;   // [E,S], [E,NS+1,S], [E,S]
    float *obs_a_t_until_next_subsidy, *obs_a_current_subsidy_level, *obs_p_t_until_next_subsidy,
        *obs_p_current_subsidy_level, *obs_p_action_mask;                  // [E,S] x2, [E] x2, [E, NL+1]
    float *obs_a_t_until_next_vaccines, *obs_p_t_until_next_vaccines;      // [E,S], [E]
    float *obs_a_agent_state, *obs_a_postsubsidy, *obs_a_lagged, *obs_a_time;   // [E,6,S], [E,S], [E,S], [E,S]
    float *obs_p_agent_state, *obs_p_postsubsidy, *obs_p_lagged, *obs_p_time;   // [E,6,S], [E,S], [E,S], [E]
    float *rewards_a, *rewards_p;                                          // [E,S], [E]
    // scalars
    int action_cooldown_period, num_stringency_levels, subsidy_interval, num_subsidy_levels, delivery_interval,
        time_when_vaccine_delivery_begins, beta_delay, filter_len, num_filters, num_days_in_an_year, value_of_life,
        n_agents /* S + 1 */, episode_length, n_envs;
    float gamma, death_rate, infection_too_sick_to_work_rate, population_between_age_18_65,
        daily_production_per_worker, risk_free_interest_rate, economic_reward_crra_eta,
        min_marginal_planner_health_index, max_marginal_planner_health_index, min_marginal_planner_economic_index,
        max_marginal_planner_economic_index, weightage_on_marginal_planner_health_index,
        weightage_on_marginal_planner_economic_index, planner_health_norm, planner_economic_norm;
};

extern "C" int ref_covid_args_size() { return (int)sizeof(RefCovidArgs); }

// One env.step() of the reference's GPU path: five launches.  Returns the CUDA error code of the last launch check.
extern "C" int ref_covid_step(const RefCovidArgs *a, void *stream) {
    cudaStream_t st = (cudaStream_t)stream;
    const dim3 grid(a->n_envs), block(a->n_agents);
    CudaControlUSStateOpenCloseStatusStep<<<grid, block, 0, st>>>(
        a->stringency_level, a->action_cooldown_period, a->action_in_cooldown_until, a->default_agent_action_mask,
        a->no_op_agent_action_mask, a->num_stringency_levels, a->actions_a, a->obs_a_policy_indicators,
        a->obs_a_action_mask, a->obs_p_policy_indicators, a->timestep, a->n_agents, a->episode_length);
    CudaFederalGovernmentSubsidyStep<<<grid, block, 0, st>>>(
        a->subsidy_level, a->subsidy, a->subsidy_interval, a->num_subsidy_levels, a->max_daily_subsidy_per_state,
        a->default_planner_action_mask, a->no_op_planner_action_mask, a->actions_p, a->obs_a_t_until_next_subsidy,
        a->obs_a_current_subsidy_level, a->obs_p_t_until_next_subsidy, a->obs_p_current_subsidy_level,
        a->obs_p_action_mask, a->timestep, a->n_agents, a->episode_length);
    CudaVaccinationCampaignStep<<<grid, block, 0, st>>>(
        (int *)a->vaccinated /* declared int*, unused by the kernel */, a->num_vaccines_per_delivery,
        a->num_vaccines_available_t, a->delivery_interval, a->time_when_vaccine_delivery_begins,
        a->obs_a_t_until_next_vaccines, a->obs_p_t_until_next_vaccines, a->timestep, a->n_agents, a->episode_length);
    CudaCovidAndEconomySimulationStep<<<grid, block, 0, st>>>(
        a->susceptible, a->infected, a->recovered, a->deaths, a->vaccinated, a->unemployed, a->subsidy, a->productivity,
        a->stringency_level, a->num_stringency_levels, a->postsubsidy_productivity, a->num_vaccines_available_t,
        a->real_world_stringency_policy_history, a->beta_delay, a->beta_slopes, a->beta_intercepts, a->beta, a->gamma,
        a->death_rate, a->incapacitated, a->cant_work, a->num_people_that_can_work, a->us_state_population,
        a->infection_too_sick_to_work_rate, a->population_between_age_18_65, a->filter_len, a->num_filters,
        a->delta_stringency_level, a->grouped_convolutional_filter_weights, a->unemp_conv_filters, a->unemployment_bias,
        a->signal, a->daily_production_per_worker, a->maximum_productivity, a->obs_a_agent_state, a->obs_a_postsubsidy,
        a->obs_a_lagged, a->obs_a_time, a->obs_p_agent_state, a->obs_p_postsubsidy, a->obs_p_lagged, a->obs_p_time,
        a->timestep, a->n_agents, a->episode_length);
    CudaComputeReward<<<grid, block, 0, st>>>(
        a->rewards_a, a->rewards_p, a->num_days_in_an_year, a->value_of_life, a->risk_free_interest_rate,
        a->economic_reward_crra_eta, a->min_marginal_agent_health_index, a->max_marginal_agent_health_index,
        a->min_marginal_agent_economic_index, a->max_marginal_agent_economic_index,
        a->min_marginal_planner_health_index, a->max_marginal_planner_health_index,
        a->min_marginal_planner_economic_index, a->max_marginal_planner_economic_index,
        a->weightage_on_marginal_agent_health_index, a->weightage_on_marginal_agent_economic_index,
        a->weightage_on_marginal_planner_health_index, a->weightage_on_marginal_planner_economic_index,
        a->agents_health_norm, a->agents_economic_norm, a->planner_health_norm, a->planner_economic_norm, a->deaths,
        a->subsidy, a->postsubsidy_productivity, a->done, a->timestep, a->n_agents, a->episode_length);
    return (int)cudaGetLastError();
}
