/*
 * aie_b200.h — C-ABI of the H100-native (sm_90a) batched Foundation environment stepper.
 *
 * Drop-in boundary for the reference's per-timestep hot path
 *   BaseEnvironment.step()                     ai_economist/foundation/base/base_env.py:929-1032
 * of the gather-trade-build family (Build, ContinuousDoubleAuction, Gather,
 * PeriodicBracketTax + resource regeneration + observation/mask/reward generation),
 * batched over E independent env replicas.  Plain pointers and sizes only; PyTorch (or any
 * other allocator) owns every device buffer, the library owns only its handle.
 *
 * The reference's own GPU plugin convention this replaces (WarpDrive, COVID path only):
 *   FoundationEnvWrapper.__init__ / reset_all_envs / step_all_envs
 *                                              ai_economist/foundation/env_wrapper.py:84-418
 *   data pushed once via get_data_dictionary() -> CUDADataManager.push_data_to_device
 *                                              env_wrapper.py:281-332
 *   kernels looked up by name Cuda<Component>Step / Cuda<Scenario>Step / CudaComputeReward
 *                                              env_wrapper.py:230-252
 * There is no return code or error channel in that convention (device asserts only); here every
 * entry point returns 0 on success or a negative AIE_E* code and aie_last_error() describes it.
 *
 * Threading: one handle per device; calls on a handle must be serialised by the caller.  All
 * device work is enqueued on the caller-supplied CUDA stream and is asynchronous unless stated.
 */
#ifndef AIE_B200_H
#define AIE_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define AIE_ABI_VERSION 4

#define AIE_MAX_COMPONENTS 8
#define AIE_MAX_BRACKETS 16
#define AIE_MAX_RATES 64
#define AIE_MAX_AGENTS 64      /* mobile agents per env */
#define AIE_MAX_PRICE_LEVELS 32 /* max_bid_ask + 1 */

/* error codes */
#define AIE_OK 0
#define AIE_EINVAL (-1)   /* bad argument / unsupported configuration */
#define AIE_ECUDA (-2)    /* CUDA runtime error (message in aie_last_error) */
#define AIE_ESTATE (-3)   /* call out of order (e.g. step before buffers are bound) */
#define AIE_ENOMEM (-4)

/* Component kinds, in the order the reference's registry names them:
 *   Build                    components/build.py:16
 *   ContinuousDoubleAuction  components/continuous_double_auction.py:17
 *   Gather                   components/move.py:16
 *   PeriodicBracketTax       components/redistribution.py:78 */
enum { AIE_COMP_BUILD = 0, AIE_COMP_CDA = 1, AIE_COMP_GATHER = 2, AIE_COMP_TAX = 3,
       AIE_COMP_WEALTH = 4 /* WealthRedistribution, components/redistribution.py:21-75 */,
       AIE_COMP_SIMPLE_LABOR = 5 /* SimpleLabor, components/simple_labor.py:16-134 (one-step-economy scenario only) */ };
/* tax_model (redistribution.py:160-166): planner-driven discretised rates, or a fixed schedule
 * ("us-federal-single-filer-2018-scaled" / "fixed-bracket-rates", rates supplied by the host). */
enum { AIE_TAX_MODEL_WRAPPER = 0, AIE_TAX_FIXED_RATES = 1,
       AIE_TAX_SAEZ = 2 /* redistribution.py:437-823, device/host hybrid: the estimator runs on the host once per tax
                           period and writes the bracket rates into the "saez_rates" field of the state record; until
                           the income buffer holds 500 samples the device draws uniform random rates from the env's
                           own stream exactly as the reference does (:444-457) */ };
/* planner_reward_type (layout_from_file.py:153, scenarios/utils/rewards.py:84-133) */
enum { AIE_SWF_COIN_EQ_TIMES_PROD = 0, AIE_SWF_INV_INCOME_COIN = 1, AIE_SWF_INV_INCOME_UTIL = 2 };

/* Static configuration of one batch of identical env replicas.  Field meaning and defaults are
 * the reference constructor kwargs (base_env.py:178-193, layout_from_file.py:68-85,
 * dynamic_layout.py:80-106, build.py:41-49, move.py:41-48, continuous_double_auction.py:42-50,
 * redistribution.py:137-155), already resolved to numbers by the host-side mirror. */
typedef struct aie_config {
    int32_t abi_version;            /* = AIE_ABI_VERSION */
    int32_t n_agents, height, width, episode_length;
    int32_t multi_action_agents;    /* multi_action_mode_agents */
    int32_t n_components;
    int32_t components[AIE_MAX_COMPONENTS]; /* AIE_COMP_*, in the env's component-list order */
    /* scenario */
    int32_t has_water;              /* Water landmark registered (6 map channels, else 5) */
    int32_t obs_range;              /* mobile_agent_observation_range (w) */
    int32_t planner_gets_spatial_info;
    int32_t allow_observation_scaling;
    double regen_weight[2];         /* resource_regen_prob / {stone,wood}_regen_weight: [Stone, Wood] */
    double isoelastic_eta, energy_cost, energy_warmup_constant;
    int32_t energy_warmup_auto;     /* energy_warmup_method == "auto" */
    int32_t planner_reward_type;    /* AIE_SWF_* */
    double mixing_weight_gini_vs_coin;
    /* Build */
    double build_payment, build_labor;
    /* Gather */
    double move_labor, collect_labor;
    /* ContinuousDoubleAuction */
    int32_t max_bid_ask, order_duration, max_num_orders;
    double order_labor;
    /* PeriodicBracketTax */
    int32_t tax_model, disable_taxes, period, n_brackets, n_disc_rates;
    double bracket_cutoffs[AIE_MAX_BRACKETS];
    double disc_rates[AIE_MAX_RATES];
    double fixed_rates[AIE_MAX_BRACKETS];
    int32_t tax_annealing;          /* tax_annealing_schedule is not None */
    double annealing_warmup, annealing_slope, rate_max;
    double rate_min;                /* lower end of the random Saez warm-up rates (redistribution.py:452-456) */
    /* batching (new; no reference equivalent) */
    int32_t auto_reset;             /* 1: an env that reaches episode_length is restored from its load-time
                                       snapshot inside the same step (WarpDrive save_copy_and_apply_at_reset
                                       semantics, env_wrapper.py:299-337); its numpy-legacy RNG stream continues */
    /* Device-side reset with reference semantics (used by auto_reset when reset_mode == 1): re-draws, from the
     * env's own numpy stream, what LayoutFromFile's reset draws - random placement
     * (layout_from_file.py:336-370), Build / Gather skills (build.py:224-254, move.py:193-210) and the
     * fixed_four_skill_and_loc assignment (layout_from_file.py:580-586) - instead of re-using the snapshot's. */
    int32_t reset_mode;             /* 0: restore the load-time snapshot; 1: reference-exact layout_from_file reset */
    int32_t build_skill_dist, gather_skill_dist;  /* 0 "none", 1 "pareto", 2 "lognormal" (numpy legacy_gauss incl. its
                                                     cached second variate, which lives in the state record) */
    int32_t payment_max_skill_multiplier;
    int32_t fixed_four;             /* fixed_four_skill_and_loc */
    int16_t ranked_locs[AIE_MAX_AGENTS][2];       /* start cell of the i-th skill-ranked slot */
    double avg_ranked_skill[AIE_MAX_AGENTS];      /* build payment of the i-th skill-ranked slot */
    /* ABI 3 */
    int32_t single_action_planner;  /* multi_action_mode_planner == False (base_env.py:259): the planner sends ONE index
                                       into [NO-OP] ++ bracket 0's rates ++ bracket 1's rates ... (single_action_map,
                                       base_agent.py:109-114) and its flattened mask is 1 + n_brackets * n_disc_rates long */
    int32_t regen_halfwidth[2];     /* {stone,wood}_regen_halfwidth, [Stone, Wood], 0..3 (dynamic_layout.py:150-153):
                                       a source cell respawns with probability convolve2d(source map, regen_weight /
                                       d^2 * ones(d, d))[cell], d = 1 + 2 * halfwidth (dynamic_layout.py:446-461) */
    int32_t full_observability;     /* layout_from_file.py:465-472 / dynamic_layout.py:526-533: every mobile agent's
                                       "world-map" is the whole map [M, H, W] (no window, no "inside" plane), its
                                       "world-idx_map" [2, H, W] with the agent's own index recoded to 1; the loc-row /
                                       loc-col scalars and the scenario's share of the planner's p<i> vectors are absent */
    /* split_layout/simple_wood_and_stone, device-side reset (layout_from_file.py:766-790): after the layout_from_file
     * reset, a random order hands out the rank-averaged skills (aie_host_state.split_skill, one table per replica) and
     * re-places everybody - the agents at the ranks in split_top_ranks above split_water_row, the others below */
    int32_t split_layout, split_water_row;
    uint64_t split_top_ranks;       /* bit i: the i-th agent of the random order starts above the water row */
    /* ABI 4.  Device-side reset of the dynamic-layout scenarios (uniform/..., quadrant/...): with reset_mode == 1 an
     * auto-reset also re-draws the clumped source layout from the env's own numpy stream exactly as
     * Uniform.reset_starting_layout does (scenarios/simple_wood_and_stone/dynamic_layout.py:313-392: np.random.rand
     * noise thinned by 0.9 until the clumped coverage is reached, then repeated growth by a random 7x7 kernel convolved
     * - scipy.signal.convolve2d, 'same' - with the candidate map plus Gaussian noise; up to 100 attempts until both
     * coverages are within 1.4x of their targets), then places the agents in a random order (:418-429). */
    int32_t dyn_layout;             /* 0: layout fixed at load time; 1: Uniform generator; 2: Quadrant (generator, then
                                       resources cleared on the two water lines, dynamic_layout.py:992-1030); 3: MultiZone
                                       (the region -> zone-type vector is re-shuffled from the env's stream before every
                                       layout, np.random.shuffle, and the probability maps follow from it, :778-872;
                                       dyn_prob is not used) */
    int32_t dyn_checker;            /* checker_source_blocks: sources only on cells with (row + col) odd (:387-392) */
    double dyn_coverage[2];         /* target coverage [Wood, Stone] (doubled when checkered, :181-186) */
    double dyn_clump[2];            /* 1 - clip(clumpiness, 0, 0.99), [Wood, Stone] */
    const double *dyn_prob;         /* HOST pointer: source probability maps float64 [2][height][width] (Wood, Stone),
                                       copied by aie_create (source_prob_maps, :289-308 / :960-990) */
    /* The "one-step-economy" scenario (scenarios/one_step_economy/one_step_economy.py:15-336) with SimpleLabor
     * (+ PeriodicBracketTax): no world map and no spatial observations (the map tensors have zero elements and may be
     * NULL in aie_buffers), agents choose 0..100 hours of labor once, utilities are coin minus a labor cost.
     * State reuse: aie_host_state.build_skill carries the SimpleLabor skill, build_payment the cumulative production. */
    int32_t scenario_kind;          /* 0: gather-trade-build family; 1: one-step-economy */
    int32_t agent_reward_type;      /* one-step-economy: 0 "isoelastic_coin_minus_labor", 1 "coin_minus_labor_cost" (:283-301) */
    double labor_exponent, labor_cost;      /* rewards.py:46-70 */
    int32_t mz_partitions[2];       /* MultiZone: num_partitions_row, num_partitions_col (at most 128 regions) */
    int32_t mz_zones[3];            /* MultiZone: number of Wood, Stone and WoodStone zones */
    int32_t labor_mask_first_step;  /* SimpleLabor mask_first_step: every labor action masked in the reset observation */
    double labor_skill_scale;       /* SimpleLabor payment_max_skill_multiplier: the skill observation is skill / this */
} aie_config;

/* Sizes the caller needs to allocate the device buffers. */
typedef struct aie_dims {
    int32_t n_envs, n_agents, height, width;
    int32_t n_map_channels;   /* M */
    int32_t window;           /* 2w+1 */
    int32_t flat_agent;       /* F_a : length of each agent's "flat" vector */
    int32_t flat_planner;     /* F_p */
    int32_t flat_planner_agent; /* length of each p<i> vector */
    int32_t mask_agent;       /* flattened agent action mask length */
    int32_t mask_planner;
    int32_t n_act_agent;      /* ints per agent per step (1 single-action, #subspaces multi-action) */
    int32_t n_act_planner;    /* ints per env per step for the planner (n_brackets, 1 for a single-action planner, or 0) */
    int32_t state_bytes;      /* bytes per env of the packed state record (multiple of 16) */
    int32_t algorithmic_bytes_per_env_step; /* SURVEY 8(d): obs+mask+rew/done out + actions in + 2*state */
    /* episode statistics ("stats" field of the state record, float64[n_stats], zero at reset): the accumulators
     * behind the reference's component get_metrics() (build.py:198-222, continuous_double_auction.py:585-641,
     * redistribution.py:1141-1186).  Layout: [0] executed trades; [1 + a] houses built by agent a;
     * [stats_trade + ((a*2 + commodity)*2 + side)*2 + k] side 0 = as seller / 1 = as buyer, k 0 = count / 1 = sum
     * of trade prices; from stats_tax (-1 without PeriodicBracketTax): periods enacted, total collected, sum of
     * effective rates, sum of bracket rates over periods [16], bracket occupancy [16], sum of max(0, income)
     * over tax days [A], sum of tax paid [A]. */
    int32_t n_stats, stats_trade, stats_tax;
    /* ABI 3: elements per agent of obs_agent_map / obs_agent_idx: (M+1)*win*win and 2*win*win, or M*H*W and 2*H*W
     * with full_observability */
    int32_t agent_map_elems, agent_idx_elems;
} aie_dims;

/* Raw device pointers.  All tensors are contiguous, env-major.
 *   state, state0 : uint8  [E, state_bytes]           packed per-env state records (see DESIGN.md)
 *   actions_agent : int32  [E, A, n_act_agent]        reference action encoding (base_agent.py:407-438)
 *   actions_planner: int32 [E, n_act_planner]         may be NULL when n_act_planner == 0
 *   obs_*         : what the reference's step returns per agent key (base_env.py:614-704),
 *                   stacked over envs:  "world-map", "world-idx_map", "flat", "action_mask", "time",
 *                   and for the planner "p<i>" vectors stacked as [E, A, flat_planner_agent]
 *   reward        : float64 [E, A+1]                  agents then planner (layout_from_file.py:519-559)
 *   done          : int32 [E]                         done["__all__"] (base_env.py:1012) */
typedef struct aie_buffers {
    void *state, *state0;
    const int32_t *actions_agent, *actions_planner;
    float *obs_agent_map;       /* [E, A, M+1, win, win]  ([E, A, M, H, W] with full_observability) */
    int16_t *obs_agent_idx;     /* [E, A, 2, win, win]    ([E, A, 2, H, W]) */
    float *obs_agent_flat;      /* [E, A, F_a] */
    float *mask_agent;          /* [E, A, mask_agent] */
    float *obs_planner_map;     /* [E, M, H, W]   (ignored unless planner_gets_spatial_info) */
    int16_t *obs_planner_idx;   /* [E, 2, H, W] */
    float *obs_planner_flat;    /* [E, F_p] */
    float *obs_planner_agents;  /* [E, A, flat_planner_agent]  (may be NULL when flat_planner_agent == 0) */
    float *mask_planner;        /* [E, mask_planner] */
    float *obs_time;            /* [E] */
    double *reward;             /* [E, A+1] */
    int32_t *done;              /* [E] */
    void *episode_final;        /* optional (may be NULL): uint8 [E, state_bytes]; with auto_reset, the state record
                                   of an env as it stood at the end of its last finished episode, i.e. what
                                   BaseEnvironment.previous_episode_metrics is computed from (base_env.py:414-418) */
    int32_t *events;            /* optional (may be NULL): int32 [event_envs, event_cap + 1, 8], the per-step event log of
                                   the first event_envs replicas, rewritten by every step - the source of the components'
                                   dense logs (build.py:150-159, move.py:140-151, continuous_double_auction.py:293-316).
                                   Row 0 of a replica's block = {count, t, dropped, 0...}; then `count` rows
                                   {1 BUILD, agent, row, col} | {2 GATHER, agent, resource, n, row, col} |
                                   {3 TRADE, seller, buyer, commodity, ask, bid, ask_lifetime, bid_lifetime} */
    int32_t event_envs, event_cap;
} aie_buffers;

/* Host-side post-reset snapshot of n envs (struct of arrays, env-major), i.e. what the reference holds
 * after reset_starting_layout / reset_agent_states / component resets / additional_reset_steps
 * (base_env.py:899-911).  Maps are 0/1 bytes [n, H, W]. */
typedef struct aie_host_state {
    int32_t n;
    const uint8_t *stone, *wood, *stone_src, *wood_src, *water; /* water may be NULL */
    const int16_t *loc;                 /* [n, A, 2] (row, col) */
    const double *coin;                 /* [n, A] starting coin */
    const int32_t *inv_stone, *inv_wood;/* [n, A] (may be NULL -> 0) */
    const double *build_payment, *build_skill, *bonus_gather_prob; /* [n, A] */
    const uint32_t *mt_key;             /* [n, 624] numpy MT19937 key (np.random.get_state()[1]) */
    const int32_t *mt_pos;              /* [n] */
    const int32_t *completions;         /* [n] (may be NULL -> 0) */
    /* ABI 3, optional: the legacy Gaussian cache of the numpy stream (np.random.get_state()[3:5]); only read by configs
     * with a lognormal skill distribution, whose device-side reset continues that stream */
    const int32_t *gauss_has;           /* [n] has_gauss */
    const double *gauss_val;            /* [n] cached_gaussian */
    const double *split_skill;          /* [n, A] optional: split_layout's rank -> build payment table of each replica */
} aie_host_state;

/* Debug / test readback of one env (host arrays, any pointer may be NULL).  Layout mirrors the
 * test oracle's state dump so parity tests compare array-for-array. */
typedef struct aie_state_dump {
    uint8_t *cell;        /* [H*W] bit0 Stone bit1 Wood bit2 StoneSrc bit3 WoodSrc bit4 Water bit5 House */
    int8_t *owner;        /* [H*W] house owner, -1 none */
    int16_t *loc;         /* [A,2] */
    double *coin, *esc_coin, *labor;      /* [A] */
    int32_t *inv, *esc;   /* [A,2] Stone, Wood */
    int32_t *n_orders;    /* [2,A] */
    int32_t *bid_hist, *ask_hist; /* [2,A,P] */
    double *price_hist;   /* [2,A,P] */
    int32_t *tax_pos;     /* [1] */
    int32_t *rate_idx;    /* [B] */
    double *last_coin, *last_income, *last_marg; /* [A] */
    uint32_t *mt_key;     /* [624] */
    int32_t *mt_pos, *t, *completions; /* [1] */
    int32_t *book_rows;   /* [2 commodities][2 sides][book_cap][3] = (agent, price, lifetime), sorted the way
                             the reference stores its lists (continuous_double_auction.py:246-253, 349-350) */
    int32_t *book_count;  /* [2][2] */
    int32_t book_cap;     /* capacity (rows) per (commodity, side) of book_rows */
    double *stats;        /* [n_stats] episode statistics (aie_dims) */
    double *util_prev;    /* [A+1] curr_optimization_metric of agents then planner (layout_from_file.py:160-163) */
    int32_t *auto_warmup; /* [1] _auto_warmup_integrator */
} aie_state_dump;

/* A named view into the packed state record, for host frameworks that want struct-of-arrays
 * tensors [E, ...] (strided views over `state`). */
typedef struct aie_field {
    int32_t offset;       /* bytes from the start of an env record */
    int32_t elem_bytes;   /* 1, 2, 4 or 8 */
    int32_t is_float;     /* 1 float, 0 integer */
    int32_t is_signed;
    int32_t ndim;
    int32_t shape[4];
} aie_field;

typedef struct aie_env aie_env;

/* Host outputs for aie_step_host (any pointer may be NULL = do not copy that tensor back). */
typedef struct aie_host_out {
    float *obs_agent_map; int16_t *obs_agent_idx; float *obs_agent_flat; float *mask_agent;
    float *obs_planner_map; int16_t *obs_planner_idx; float *obs_planner_flat; float *obs_planner_agents;
    float *mask_planner; float *obs_time; double *reward; int32_t *done;
} aie_host_out;

/* Lifecycle ------------------------------------------------------------------------------------ */

/* Replaces: Scenario construction through foundation.make_env_instance (foundation/__init__.py:16-18,
 * base_env.py:178-366) for the device-resident part of the env.  `device` is the CUDA ordinal. */
int aie_create(const aie_config *cfg, int32_t n_envs, int32_t device, aie_env **out);
int aie_destroy(aie_env *env);
int aie_get_dims(const aie_env *env, aie_dims *out);
/* name: "t", "coin", "esc_coin", "labor", "inv", "esc", "loc", "cell", "owner", "n_orders", "bid_hist",
 * "ask_hist", "price_hist", "tax_pos", "rate_idx", "last_coin", "last_income", "last_marg",
 * "build_payment", "build_skill", "bonus_gather_prob", "mt_key", "mt_pos", "completions", "orders" */
int aie_get_field(const aie_env *env, const char *name, aie_field *out);

/* ABI 3.  The named fields behind a "flat" vector, in concatenation order, i.e. what BaseEnvironment._build_packager
 * records (base_env.py:562-589: every scalar / 1-D observation, sorted by key "<Component>-<obs>" / "world-<obs>" /
 * "time").  With it a caller rebuilds the flatten_observations=False dictionaries as slices of the flat tensors.
 * which: 0 = each agent's "flat", 1 = the planner's "flat", 2 = the planner's per-agent "p<i>" vectors.
 * Fills at most cap entries; returns the number of fields (or a negative AIE_E* code). */
typedef struct aie_flat_field { char key[64]; int32_t offset, size; } aie_flat_field;
int aie_get_flat_layout(const aie_env *env, int32_t which, aie_flat_field *out, int32_t cap);

/* Replaces: CUDADataManager.push_data_to_device + placeholders (env_wrapper.py:297-332). */
int aie_bind_buffers(aie_env *env, const aie_buffers *bufs);

/* Replaces: env.reset() host->device push (env_wrapper.py:281-332).  Packs envs [env_lo, env_lo+hs->n)
 * into `state`, saves the same records into `state0` (auto-reset snapshot), finishes the reset on the
 * device (tax last_coin, utility metric_0; layout_from_file.py:588-593, redistribution.py:1106-1139) and
 * writes their first observations/masks.  Synchronous. */
int aie_load_state(aie_env *env, const aie_host_state *hs, int32_t env_lo, void *stream);

/* Replaces: FoundationEnvWrapper.step_all_envs (env_wrapper.py:355-377) == BaseEnvironment.step
 * (base_env.py:929-1032) for every env: reads actions_*, advances `state`, writes obs/masks/reward/done. */
int aie_step(aie_env *env, void *stream);

/* The two halves of aie_step, separately launchable (profiling / custom pipelines):
 * aie_step_dynamics = components + scenario_step + rewards + done (base_env.py:1000-1005, 1011-1012);
 * aie_observe       = observations + masks from the current state (base_env.py:614-756). */
int aie_step_dynamics(aie_env *env, void *stream);
int aie_observe(aie_env *env, void *stream);

/* Random policy on the device: writes into the bound action buffers one uniformly random *unmasked* action
 * per agent (per subspace in multi-action mode) and per planner bracket, from the current mask tensors.
 * Replaces: BaseAgent.get_random_action / populate_random_actions (base/base_agent.py:365-405) and the
 * tutorial's mask-aware random sampler (tutorials/economic_simulation_basic.ipynb, cell 18).  The stream is a
 * counter-based hash of (seed, call index, env, agent, subspace); it is not the env's numpy stream. */
int aie_sample_random_actions(aie_env *env, uint64_t seed, void *stream);

/* The same random policy fused into the step: with a non-zero seed every following aie_step / aie_observe also writes
 * the NEXT step's uniformly random unmasked actions into the bound action buffers, drawn by the observation pass from
 * the mask limits it has just computed (no mask read-back, no sampler launch per step).  The call itself samples once
 * from the current masks so that the very next aie_step has actions.  seed == 0 turns it off.  Rollout loops with a
 * random policy (the benchmark's "random actions", tutorials/economic_simulation_basic.ipynb cell 18) call this once
 * and then only aie_step. */
int aie_set_fused_policy(aie_env *env, uint64_t seed, void *stream);

/* End-to-end variant with HOST buffers: copies the actions host->device, steps, copies every non-NULL
 * output device->host, and synchronises the stream.  Buffers should be pinned for full PCIe rate. */
int aie_step_host(aie_env *env, const int32_t *actions_agent_host, const int32_t *actions_planner_host,
                  const aie_host_out *out, void *stream);

/* ABI 3.  Same contract as aie_step_host - the caller's host tensors receive exactly the same bytes - with a compacted
 * device->host transfer: the 0/1-valued float planes (maps, masks) cross PCIe as bits, the int16 index planes as a bitmap of
 * their non-zero cells plus byte values, the agents' flat vectors de-duplicated by entry class.  The batch steps in a few
 * launches over env ranges; after each, a pack kernel rewrites that chunk's outputs into a library-owned compact device
 * buffer and the records go down in slices on a library-owned copy stream into a pinned staging buffer while the next chunk
 * steps; n_threads host threads (<= 0: half the hardware threads; at most 128) expand each slice as it lands into the
 * caller's tensors (a transfer format: no simulation work runs on the host).  c2: 2.7 KB instead of 36 KB per env-step over
 * PCIe.  Synchronous; ordered on `stream` like aie_step_host. */
int aie_step_host_compact(aie_env *env, const int32_t *actions_agent, const int32_t *actions_planner,
                          const aie_host_out *out, int32_t n_threads, void *stream);
/* bytes one env contributes to the compacted transfer (0 on error) */
int32_t aie_compact_bytes_per_env(const aie_env *env);
/* Host-clock breakdown of the last aie_step_host_compact call, milliseconds from the start of its transfer phase:
 * [0] copies enqueued, [1] first transfer slice on the host, [2] last slice on the host, [3] expansion finished,
 * [4] number of slices, [5] host threads used, [6] bytes moved device->host, [7] time before the transfer phase (action
 * upload + launches enqueued), [8] time the threads spent waiting for their slice and [9] expanding (summed over threads),
 * [10] / [11] device-clock arrival of the first / last slice since the call's first enqueue, [12] the expansion alone
 * (only with AIE_E2E_REPEAT_EXPAND=n in the environment), [13] envs whose index planes were fetched directly, [14] number of
 * step chunks (the batch steps in up to AIE_E2E_CHUNKS launches, default 4, or 2 for large records, so that the first slices go down while the rest
 * of the batch still steps), [15] NUMA node of the library's pinned staging buffer (-1: plain cudaHostAlloc).  Returns the number of words defined (diagnostics for tuning). */
#define AIE_HOST_TIMING_WORDS 16
int aie_get_host_timing(const aie_env *env, double *out, int32_t cap);

/* Test/debug readback of env `e` (synchronous). */
int aie_read_state(aie_env *env, int32_t e, const aie_state_dump *out);
/* Same readback from the episode_final snapshot of env e (the record as it stood when its last finished episode
 * ended, before the auto-reset): the input of previous_episode_metrics (base_env.py:414-418).  Order books are
 * not part of the snapshot (book_rows / book_count are ignored).  AIE_ESTATE when no episode_final buffer is bound. */
int aie_read_episode_final(aie_env *env, int32_t env_index, const aie_state_dump *out);

/* Number of kernels the library has launched on this handle since creation (for bench "gpu_launches"). */
int64_t aie_launch_count(const aie_env *env);

/* ================================================================================================
 * COVID-19 + economy scenario (BASELINE config 4)
 *
 * Replaces the reference's WarpDrive kernels for this scenario, which are launched one after the other by
 * FoundationEnvWrapper.step_all_envs (ai_economist/foundation/env_wrapper.py:355-377):
 *   CudaControlUSStateOpenCloseStatusStep   components/covid19_components_step.cu:10-113
 *   CudaFederalGovernmentSubsidyStep        components/covid19_components_step.cu:115-209
 *   CudaVaccinationCampaignStep             components/covid19_components_step.cu:211-262
 *   CudaCovidAndEconomySimulationStep       scenarios/covid19/covid19_env_step.cu:274-476
 *   CudaComputeReward                       scenarios/covid19/covid19_env_step.cu:480-619
 * by ONE fused kernel per step that follows the *Python* path's arithmetic (covid19_env.py:650-1173,
 * covid19_components.py:145-627), including its mixed float32 / int32 / float64 promotions.
 * All fitted parameters are resolved on the host (ai_economist_b200/foundation/covid19.py) and copied into
 * library-owned device memory at creation.
 * ================================================================================================ */
typedef struct aie_covid_config {
    int32_t abi_version;
    int32_t n_states;            /* 51 */
    int32_t episode_length, num_stringency_levels, action_cooldown_period;
    int32_t subsidy_interval, num_subsidy_levels;
    int32_t time_when_vaccine_delivery_begins, delivery_interval, t_first_delivery;
    int32_t beta_delay, filter_len, num_filters, start_date_index, rw_policy_days;
    int32_t value_of_life;
    int32_t auto_reset;
    float gamma, death_rate, infection_too_sick_to_work_rate, pop_between_age_18_65, risk_free_interest_rate, crra_eta;
    float planner_health_norm, planner_economic_norm;
    float min_planner_health, max_planner_health, min_planner_econ, max_planner_econ, w_planner_health, w_planner_econ;
    double reward_normalization_factor, time_scale;
    /* host arrays, copied at creation ([S] unless noted) */
    const int32_t *population, *num_vaccines_per_delivery;
    const float *beta_slopes, *beta_intercepts, *unemployment_bias, *daily_production_per_worker /* [1] */,
        *maximum_productivity, *agents_health_norm, *agents_economic_norm, *min_agent_health, *max_agent_health,
        *min_agent_econ, *max_agent_econ, *w_agent_health, *w_agent_econ;
    const float *conv_weights;      /* [S, F] */
    const float *conv_filters;      /* [F, L] exp(-(L-1-k)/lambda_f) evaluated in float32 as the reference does */
    const double *max_daily_subsidy_per_state;
    const int8_t *rw_policy;        /* [rw_policy_days, S] real-world stringency (initial history, lag before t = beta_delay) */
    const float *init_state;        /* [6, S] Susceptible, Infected, Recovered, Deaths, Vaccinated, Unemployed at t = 0 */
} aie_covid_config;

/* Device buffers (contiguous, env-major).  state: float32 [E, 9, S] = S, I, R, D, V, U, stringency, subsidy,
 * postsubsidy productivity at the current timestep; ints: int32 [E, 2, S] = cooldown_until, vaccines_available;
 * hdr: int32 [E, 4] = t, subsidy_level, ring_head, episodes; ring: int8 [E, S, ROW] stringency history, time-minor
 * (ROW = filter_len + 1 rounded up to a multiple of 16 bytes; logical entry k sits at column (ring_head + k) mod (L+1)).
 * Observations are the reference's collated "a"/"p" fields (covid19_env.py:919-993 + components), float32. */
typedef struct aie_covid_buffers {
    float *state; int32_t *ints; int32_t *hdr; int8_t *ring;
    const int32_t *actions_agent;   /* [E, S] stringency action 0..num_stringency_levels (0 = NO-OP) */
    const int32_t *actions_planner; /* [E]    subsidy level action 0..num_subsidy_levels */
    float *obs_agent_state;         /* [E, 6, S]  world-agent_state */
    float *obs_postsubsidy;         /* [E, S]     world-agent_postsubsidy_productivity */
    float *obs_lagged_stringency;   /* [E, S]     world-lagged_stringency_level */
    float *obs_policy_indicators;   /* [E, S]     ControlUSStateOpenCloseStatus-agent_policy_indicators */
    float *obs_scalars;             /* [E, 4]     time, t_until_next_subsidy, current_subsidy_level, t_until_next_vaccines */
    float *mask_agent;              /* [E, 1+levels, S] */
    float *mask_planner;            /* [E, 1+num_subsidy_levels] */
    float *reward_agent;            /* [E, S] */
    double *reward_planner;         /* [E] */
    int32_t *done;                  /* [E] */
    uint32_t *changes;              /* optional (may be NULL), ABI 3: uint32 [E, 33, S] scratch state owned by the kernels -
                                       per-state list of the stringency changes inside the filter window, so that the
                                       unemployment response costs O(changes) instead of a scan of the filter_len-day
                                       history (covid19_env.py:1374-1441) per state and step */
} aie_covid_buffers;

typedef struct aie_covid_env aie_covid_env;

int aie_covid_create(const aie_covid_config *cfg, int32_t n_envs, int32_t device, aie_covid_env **out);
int aie_covid_destroy(aie_covid_env *env);
int aie_covid_bind_buffers(aie_covid_env *env, const aie_covid_buffers *bufs);
/* env.reset() for every replica (covid19_env.py:1175-1290 is deterministic): state, history, first observations. */
int aie_covid_reset(aie_covid_env *env, void *stream);
/* One env.step() for every replica: 3 component steps + scenario step + observations + rewards + done. */
int aie_covid_step(aie_covid_env *env, void *stream);
/* Random policy on the device (uniform over the unmasked actions of the current masks); see aie_sample_random_actions. */
int aie_covid_sample_random_actions(aie_covid_env *env, uint64_t seed, void *stream);
int64_t aie_covid_launch_count(const aie_covid_env *env);

const char *aie_last_error(void);
int aie_abi_version(void);

#ifdef __cplusplus
}
#endif
#endif /* AIE_B200_H */
