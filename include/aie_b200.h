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

#define AIE_ABI_VERSION 6

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
    /* ABI 5.  Element type of the float observation / mask tensors (obs_agent_map, obs_agent_flat, mask_agent,
     * obs_planner_map, obs_planner_flat, obs_planner_agents, mask_planner, obs_time): AIE_OBS_F32 (default), or
     * AIE_OBS_BF16 - every element is the round-to-nearest-even bfloat16 of the float32 the default writes, converted in
     * the observation pass (half the bytes, no extra pass).  Index planes, rewards, done, state and actions are unchanged.
     * aie_step_host / aie_step_host_compact take float32 configs only (AIE_EINVAL otherwise). */
    int32_t obs_dtype;
} aie_config;
enum { AIE_OBS_F32 = 0, AIE_OBS_BF16 = 1 };

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
    int32_t algorithmic_bytes_per_env_step; /* SURVEY 8(d): obs+mask+rew/done out + actions in + 2*state (observation
                                               bytes at the config's obs_dtype) */
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
 *                   and for the planner "p<i>" vectors stacked as [E, A, flat_planner_agent].
 *                   With aie_config::obs_dtype == AIE_OBS_BF16 the float* observation / mask pointers below point to
 *                   bfloat16 storage (2 bytes per element, same shapes)
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

/* Explicit reset on the device (configs with reset_mode == 1): env.reset() of replicas [env_lo, env_lo + n) without a
 * host reset per replica.  One launch re-draws, from each replica's own numpy stream and in the reference's order, what
 * the auto-reset re-draws (layout, placement, skills, fixed_four / split_layout assignment), then one launch writes the
 * first observations.  Each record comes out as aie_load_state leaves it for the host reset of the same stream (byte
 * for byte, except that the device's exp / log can move Pareto / lognormal skills and the cached Gaussian in the last place): t 0, episodes 0, Saez section and counter zero (the caller's Saez estimator restores them), reward and done
 * zero, state0 the same record; the live record additionally carries auto_warmup over.  episode_final and the event
 * log are not touched.
 *   tmpl:    NULL: every replica restarts from its own state0 (the record its last reset produced).  Else one host reset
 *            snapshot (n == 1): its maps, coin and inventories become every replica's starting record (everything
 *            random in it is re-drawn); its completions count seeds replicas that have never been loaded.
 *   streams: NULL: each record's stream continues.  Else the streams of the n replicas (arrays indexed from 0).
 * Counters: once the env is loaded, completions = the record's count + 1 if its episode has ended and waits for this
 * reset (t >= episode_length), auto_warmup carried over; before that, from tmpl.  Asynchronous on `stream`, except that
 * a call with tmpl or streams uploads them through a staging buffer of its own and synchronises.  AIE_EINVAL for a reset_mode 0 config, a bad range
 * or a missing array; AIE_ESTATE before aie_bind_buffers, or without tmpl and streams before anything was loaded. */
typedef struct aie_reset_streams {
    const uint32_t *mt_key;             /* [n, 624] numpy MT19937 key */
    const int32_t *mt_pos;              /* [n] */
    const int32_t *gauss_has;           /* [n] legacy Gaussian cache: required for lognormal skills and dynamic layouts */
    const double *gauss_val;            /* [n] */
    const double *split_skill;          /* [n, A] split_layout's rank -> build payment table (required there) */
} aie_reset_streams;
int aie_reset_envs(aie_env *env, const aie_host_state *tmpl, const aie_reset_streams *streams, int32_t env_lo, int32_t n,
                   void *stream);

/* Replaces: FoundationEnvWrapper.step_all_envs (env_wrapper.py:355-377) == BaseEnvironment.step
 * (base_env.py:929-1032) for every env: reads actions_*, advances `state`, writes obs/masks/reward/done. */
int aie_step(aie_env *env, void *stream);

/* The two halves of aie_step, separately launchable (profiling / custom pipelines):
 * aie_step_dynamics = components + scenario_step + rewards + done (base_env.py:1000-1005, 1011-1012);
 * aie_observe       = observations + masks from the current state (base_env.py:614-756). */
int aie_step_dynamics(aie_env *env, void *stream);
int aie_observe(aie_env *env, void *stream);

/* The ten observation / mask tensors of aie_buffers, with the same shapes and element types (the float pointers point to
 * bfloat16 storage when obs_dtype == AIE_OBS_BF16); the same pointers are required as by aie_bind_buffers. */
typedef struct aie_obs_buffers {
    float *obs_agent_map; int16_t *obs_agent_idx; float *obs_agent_flat; float *mask_agent;
    float *obs_planner_map; int16_t *obs_planner_idx; float *obs_planner_flat; float *obs_planner_agents;
    float *mask_planner; float *obs_time;
} aie_obs_buffers;

/* ABI 5.  Final observations of the episodes the auto-reset ended: for every env whose done flag is non-zero after the
 * latest aie_step, writes the observations / masks of its episode_final record (the state its episode ended in, which
 * the step's own outputs no longer show: they belong to the new episode) into row e of `out`; every other row is left
 * untouched.  What a trainer bootstraps a truncated episode's value from (gymnasium's final_obs).  One launch,
 * asynchronous on `stream`; draws no actions, even with the fused policy on.  AIE_EINVAL for a NULL out, a missing
 * required pointer or a pointer not aligned to its element size; AIE_ESTATE before buffers are bound and state is
 * loaded, or without episode_final records (no episode_final buffer bound, or auto_reset off). */
int aie_observe_final(aie_env *env, const aie_obs_buffers *out, void *stream);

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

/* A policy's logits, laid out like the masks with the action axis last, and where the log-probabilities go. */
typedef struct aie_policy_logits {
    const void *agent;        /* DEVICE [E, A, Na] (the mask_agent layout, each multi-action subspace with its own NO-OP) */
    const void *planner;      /* DEVICE [E, Np] (the mask_planner layout), or NULL when the config has no planner actions */
    int32_t logits_dtype;     /* AIE_OBS_F32 | AIE_OBS_BF16 (independent of the config's obs_dtype) */
    int32_t greedy;           /* 0: draw from the softmax; 1: the open entry with the largest logit (lowest index on ties) */
    float *log_prob_agent;    /* DEVICE [E, A, n_act_a] or NULL */
    float *log_prob_planner;  /* DEVICE [E, n_act_p] or NULL */
} aie_policy_logits;

/* ABI 5.  A policy's actions on the device: for every env, agent (every subspace in multi-action mode) and planner
 * bracket (or the single-action planner's one index), one draw from the softmax of the segment's logits restricted to
 * the open entries of the CURRENT mask buffers (what the latest reset / step / observe wrote), into the bound action
 * buffers (whatever was there is overwritten, the fused random policy's draw included); the log-probability of each
 * action into the optional log_prob tensors.  One launch, asynchronous on `stream`.
 *   Stream: s = host_mix64(seed) ^ host_mix64(n), n = 1, 2, .. counting this env's aie_sample_policy calls (its own
 *   counter: aie_sample_random_actions does not move it); env key k = mix64(s ^ mix64(env)) (mix64: the splitmix64
 *   finaliser); segment key k + 0x100 * agent (single-action agents), k + 0x100 * agent + subspace + 1 (multi-action),
 *   k + 0x10000 + bracket (planner brackets; bracket 0 for the single-action planner); u = (mix64(segment key) >> 11) * 2^-53.
 *   Draw (float64): m = the largest open logit, w_j = exp((double)l_j - m) for open j (0 for closed), Z = sum w_j; the
 *   action is the smallest j with w_j > 0 and u * Z < w_0 + .. + w_j, else (rounding) the last j with w_j > 0.
 *   greedy = 1: the first open j with l_j == m.  Log-probability: (float)(((double)l_a - m) - log(Z)).
 *   A segment with no open entry: action 0, log-probability 0.  An open logit that is NaN or +inf, or no finite open
 *   logit: the first open entry, log-probability NaN.  Open entries at -inf are never drawn.
 * AIE_EINVAL for a NULL p or agent logits, missing planner logits when the config has planner actions, an unknown
 * logits_dtype, greedy not 0 or 1, or a pointer not aligned to its element size; AIE_ESTATE before buffers are bound
 * and state is loaded. */
int aie_sample_policy(aie_env *env, const aie_policy_logits *p, uint64_t seed, void *stream);

/* Stored actions of a policy and the masks they were drawn under, for the update pass: N rows, each laid out like one
 * env's logits, masks and actions (a PPO minibatch of rollout steps, any N).  DEVICE pointers; "planner" entries are
 * NULL / ignored when the config has no planner actions. */
typedef struct aie_policy_eval {
    const void *logits_agent;             /* [N, A, Na] (the layout of aie_policy_logits::agent); COVID-19 [N, S, 1 + levels] */
    const void *logits_planner;           /* [N, Np]; COVID-19 [N, 1 + subsidy levels] */
    const void *mask_agent;               /* [N, A, Na] as the env wrote mask_agent; COVID-19 [N, 1 + levels, S] */
    const void *mask_planner;             /* [N, Np]; COVID-19 [N, 1 + subsidy levels] */
    const int32_t *actions_agent;         /* [N, A, n_act_a]; COVID-19 [N, S] */
    const int32_t *actions_planner;       /* [N, n_act_p]; COVID-19 [N] */
    int32_t logits_dtype;                 /* AIE_OBS_F32 | AIE_OBS_BF16: both logits tensors and both gradients */
    int32_t mask_dtype;                   /* AIE_OBS_F32 | AIE_OBS_BF16: both masks */
    float *log_prob_agent, *log_prob_planner;    /* forward outputs, shaped like the actions */
    float *entropy_agent, *entropy_planner;      /* forward outputs, shaped like the actions */
    const float *grad_log_prob_agent, *grad_log_prob_planner;   /* backward: upstream gradients, NULL = zero */
    const float *grad_entropy_agent, *grad_entropy_planner;     /* backward: upstream gradients, NULL = zero */
    void *grad_logits_agent, *grad_logits_planner;              /* backward outputs: the logits' layout and dtype */
} aie_policy_eval;

/* ABI 5.  Log-probabilities and entropies of stored actions: per row and mask segment (the sampler's segments: a
 * single-action agent's whole row, each multi-action subspace with its own NO-OP, each planner bracket or the
 * single-action planner's one index), with m = the largest open logit, w_j = exp((double)l_j - m) for open j,
 * Z = sum w_j (accumulated in aie_sample_policy's order), p_j = w_j / Z, a = the stored action, in float64 and rounded once:
 *   log_prob = (float)(((double)l_a - m) - log(Z))   - bit for bit what aie_sample_policy returned for the same logits,
 *                                                      masks and action on the same backend;
 *   entropy  = (float)(log(Z) - sum_j p_j ((double)l_j - m)).
 * A segment with no open entry: 0 and 0.  An open logit that is NaN or +inf, or no finite open logit: NaN and NaN.
 * An action that is closed or outside [0, n): log_prob NaN, the entropy as usual.
 * One launch, asynchronous on `stream`; N = 0 is a no-op.  It reads no env record and needs no bound buffers or loaded
 * state (only the config), and moves no counter of the env.  AIE_EINVAL for a NULL p, a negative N, an unknown
 * logits_dtype or mask_dtype, and (N > 0) a NULL required pointer (the logits, masks, actions and outputs of the agents,
 * and of the planner when the config has planner actions) or a pointer not aligned to its element size. */
int aie_evaluate_policy(aie_env *env, const aie_policy_eval *p, int64_t n_rows, void *stream);
/* ABI 5.  The gradient of sum(g_lp * log_prob + g_H * entropy) with respect to the logits (the backward of
 * aie_evaluate_policy; m and Z recomputed from the logits), into grad_logits_*, every entry written: for open j
 *   g_lp ([j = a] - p_j) - g_H p_j (((double)l_j - m - log(Z)) + H)   (H the float64 entropy; an open entry with
 *                                                                     p_j = 0 has no g_H term),
 * 0 for closed entries.  A segment with no open entry: 0.  An open logit that is NaN or +inf, no finite open logit, or
 * a stored action that is closed or outside [0, n): NaN at the open entries, 0 at the closed ones.  bfloat16 gradients
 * are the round-to-nearest-even of the float64 value.  The outputs of aie_evaluate_policy are neither read nor needed
 * (log_prob_* / entropy_* may be NULL); grad_logits_* are required instead.  Errors as aie_evaluate_policy. */
int aie_evaluate_policy_backward(aie_env *env, const aie_policy_eval *p, int64_t n_rows, void *stream);

/* A stored rollout of T steps of the E replicas, for advantages and value targets: two groups of columns, the agents'
 * ([T, E, A]: COVID-19 A = S states) and the planner's ([T, E]).  DEVICE pointers, contiguous. */
enum { AIE_REWARD_F32 = 0, AIE_REWARD_F64 = 1 };
typedef struct aie_advantage_args {
    const void *rewards_agent;                /* [T, E, A], as the env wrote its rewards after each step */
    const void *rewards_planner;              /* [T, E], or NULL: no planner group (its other entries are then ignored) */
    int32_t rewards_agent_dtype;              /* AIE_REWARD_F32 | AIE_REWARD_F64 */
    int32_t rewards_planner_dtype;
    const float *values_agent, *values_planner;             /* [T, E, A], [T, E]: the value of the observation each
                                                               step's action was taken from */
    const int32_t *dones;                                    /* [T, E]: done["__all__"] after each step */
    const float *last_values_agent, *last_values_planner;   /* [E, A], [E]: the value of the observation after step T-1 */
    const float *final_values_agent, *final_values_planner; /* like values (the value of final_obs after each step), or
                                                               NULL: an episode end is terminal */
    double gamma_agent, gamma_planner;        /* each in [0, 1] */
    double lambda_agent, lambda_planner;      /* each in [0, 1] */
    float *adv_agent, *adv_planner;           /* outputs, like the rewards */
    float *ret_agent, *ret_planner;           /* outputs, like the rewards */
} aie_advantage_args;

/* ABI 5.  Generalised advantage estimation over a stored rollout, bootstrapped at episode ends.  For every column (agent
 * (e, a) or planner e) of a group with discount gamma and lambda lam, in float64 with every operation rounded (no fused
 * multiply-add), gl = gamma * lam computed once, R the rewards, V the values, F the final values, LV the last values:
 *   for t = T-1 .. 0:
 *       d     = dones[t, e] != 0
 *       nv    = d ? (F given ? F[t] : 0) : (t == T-1 ? LV : V[t+1])
 *       delta = (R[t] + gamma * nv) - V[t]
 *       A     = (d || t == T-1) ? delta : delta + gl * A_next        (the chain is cut, not multiplied by 0)
 *       adv[t] = (float)A;  ret[t] = (float)(A + V[t])
 * Under the auto-reset the step that ends an episode returns that episode's reward and done but the next episode's
 * observation, and every episode ends on its time limit (truncated, not terminal): the target at a done step bootstraps
 * from the value of that step's final observation (env.final_obs), which F supplies.  F is read only where d holds, so it
 * may be the value net's output over the whole final-observation tensor, unspecified rows included; without F an episode
 * end is treated as terminal.  A NaN propagates backwards through its chain up to the previous cut.  The CUDA kernel
 * and a host build of the same source give the same bits.  One launch, asynchronous on `stream`; T = 0 is a no-op.  It
 * reads no env record, needs no bound buffers or loaded state (only E and A), and moves no counter of the env.
 * AIE_EINVAL for a NULL args, a negative T, an unknown reward dtype, a gamma or lambda that is NaN or outside [0, 1],
 * and (T > 0) a NULL required pointer (every pointer of a group but its final values) or a pointer not aligned to its
 * element size. */
int aie_compute_advantages(aie_env *env, const aie_advantage_args *args, int32_t T, void *stream);

/* Rollouts stored in place.  A rollout of T steps of the E replicas is a set of caller-owned DEVICE tensors, contiguous,
 * slot-major: slot t of a tensor is the [E, ...] block of the bound buffer of the same name (aie_buffers), at
 * t * (bytes of that block).  K = ceil(T / episode_length). */
typedef struct aie_rollout {
    int32_t T;                    /* slots of the step outputs, >= 1 */
    aie_obs_buffers obs;          /* [T + 1, E, ...] each: slot t the observation step t's action is taken from, slot T the
                                     observation after the last step (the bootstrap input).  NULL exactly where
                                     aie_bind_buffers allows NULL */
    int32_t *actions_agent;       /* [T, E, A, n_act_agent] */
    int32_t *actions_planner;     /* [T, E, n_act_planner]; NULL when n_act_planner == 0 */
    double *reward;               /* [T, E, A + 1] */
    int32_t *done;                /* [T, E] */
    aie_obs_buffers final_obs;    /* optional: every member NULL (no final slots), or [K, E, ...] each: row (k, e) the
                                     observation of the state in which replica e's k-th episode end within this rollout
                                     ended (k counts from 0).  Needs auto_reset and an episode_final buffer */
} aie_rollout;

/* ABI 6 (additive).  Binds a rollout: from here on the library keeps a slot cursor s (0 after this call) and
 *   - aie_sample_random_actions / aie_sample_policy read the masks of slot s and write the actions into slot s;
 *   - aie_step reads the actions of slot s, writes the observations and masks into slot s + 1 and the rewards and done
 *     into slot s; with final slots it then writes the final observation of every episode it ended into row
 *     (k, e) of final_obs, k = the number of done flags of replica e in slots 0 .. s - 1 (a replica ends at most K times
 *     in T steps, since every episode lasts episode_length steps; a k >= K is not written); then s advances.  With final
 *     slots that is two launches (the step, then the final pass: the same count as aie_step + aie_observe_final today),
 *     without them one;
 *   - aie_observe writes the observations of the current state into slot s;
 *   - aie_load_state / aie_reset_envs write the first observations into slot 0, and are allowed only at s == 0.
 * AIE_ESTATE while a rollout is bound: aie_step, the samplers at s == T; aie_load_state / aie_reset_envs at s != 0;
 * aie_set_fused_policy (its draws would overwrite the stored actions), aie_step_dynamics, aie_observe_final (the final
 * slots replace it), aie_step_host, aie_step_host_compact and aie_bind_buffers.  s advances once the step launch succeeds (the state
 * has then moved on), even if the final pass after it fails; any other call that fails leaves s where it was.
 * r == NULL unbinds: every pointer returns to the buffers of aie_bind_buffers, so a caller that never binds a rollout sees
 * no change.  No launch; no device work.  AIE_EINVAL for T < 1, a NULL required pointer, a pointer not aligned to its
 * element size, or final slots partly given; AIE_ESTATE before aie_bind_buffers, with the fused random policy on, or
 * final slots without auto_reset and an episode_final buffer. */
int aie_bind_rollout(aie_env *env, const aie_rollout *r);
/* Starts the next rollout of the bound tensors: copies the observations of slot T into slot 0 (one device copy per
 * tensor), sets s = 0 and so restarts the episode-end count k.  Asynchronous on `stream`; no launch.  AIE_ESTATE without
 * a bound rollout or before its T steps are done (s != T). */
int aie_rollout_restart(aie_env *env, void *stream);
/* The advantages of aie_compute_advantages over a bound rollout's final slots: final_values_* are [K, E, A] / [K, E]
 * (the value of final_obs row (k, e)), and a done step reads the row of its episode-end ordinal within the column
 * (0 for the first done flag of replica e in 0 .. T-1); an ordinal >= K reads NaN.  Every other input, the recursion,
 * its rounding and its NaN behaviour are aie_compute_advantages's, so the result has the same bits as that call over
 * [T, E, ...] final values holding row (k, e) at the k-th done step of replica e.  One launch.  AIE_EINVAL as
 * aie_compute_advantages, and for K < 1. */
int aie_compute_advantages_k(aie_env *env, const aie_advantage_args *args, int32_t T, int32_t K, void *stream);

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

/* Episode metrics of every replica in one launch (aie_metrics_kernel: one warp per env reads its record in global
 * memory and writes one row).  Each row is BaseEnvironment.metrics (base_env.py:421-432) of that replica, i.e. what
 * foundation/metrics.py computes from one record, summed in numpy's order.
 *
 * The reference's env.metrics keys for this config, in column order; is_int marks keys whose reference value is an
 * int (n_builds, total_builds, n_sales, n_trades, warmup_integrator, one-step "endow/p/Coin").  Fills at most cap
 * entries, returns K (or a negative AIE_E* code), like aie_get_flat_layout. */
typedef struct aie_metric_key { char key[64]; int32_t is_int; } aie_metric_key;
int aie_get_metric_layout(const aie_env *env, aie_metric_key *out, int32_t cap);
/* source 0: the current records (env.metrics of every replica; a replica at t >= episode_length counts its finished
 * episode, like the reference before its reset); 1: the episode_final records (previous_episode_metrics; a replica that
 * has finished no episode yet gets a row of NaN).  out: DEVICE float64 [n_envs, K].  Asynchronous on `stream`: no
 * synchronisation, no host copy.  Trade averages without trades are NaN; the Saez model's estimated_elasticity column
 * is written NaN (the estimator runs on the host).  AIE_EINVAL for a NULL out or an unknown source, AIE_ESTATE before
 * aie_bind_buffers or, for source 1, without an episode_final buffer. */
int aie_episode_metrics(aie_env *env, int32_t source, double *out, void *stream);

/* Number of kernels the library has launched on this handle since creation (for bench "gpu_launches"). */
int64_t aie_launch_count(const aie_env *env);

/* ABI 6 (additive).  The counters the library keeps on the host for a handle, beyond what the caller's buffers hold:
 * with them and every record of state / state0 / episode_final, a checkpoint of an env resumes bit for bit. */
typedef struct aie_counters {
    uint64_t sample_calls;       /* aie_sample_random_actions calls, aie_set_fused_policy's own draw included */
    uint64_t policy_calls;       /* aie_sample_policy calls (the policy sampler's stream counter n) */
    uint64_t fused_policy_key;   /* the fused random policy's key, host_mix64(seed) | 1; 0 when it is off */
    int32_t fused_policy_on;     /* 1: the fused random policy is on (fused_policy_key != 0), 0: off */
    int32_t reserved;            /* 0 */
} aie_counters;
/* Reads the counters into *out.  aie_set_counters writes them back and marks the env loaded: the caller has written
 * every record of state and state0 (and episode_final) itself, from an env of the same configuration, so aie_step and
 * aie_observe may follow without aie_load_state.  Neither call launches anything; the launch count is diagnostic and
 * is neither read nor written.  AIE_EINVAL for a NULL env or counters, and (set) fused_policy_on not 0 or 1, or not
 * matching fused_policy_key != 0; AIE_ESTATE before aie_bind_buffers, while a rollout is bound at s != 0, and (set) a
 * fused policy that is on while a rollout is bound. */
int aie_get_counters(aie_env *env, aie_counters *out);
int aie_set_counters(aie_env *env, const aie_counters *in);

/* ABI 6 (additive).  A bound rollout recorded once as a CUDA graph and replayed (torch.cuda.graph, cudaStreamBeginCapture).
 * A replay repeats the launches' arguments as they were at capture, so nothing a launch takes from the host may change
 * between replays.  The gather-trade-build step takes only the slot's pointers (fixed per slot) and the final pass
 * finds its row from the stored done flags on the device; what remains is the policy sampler's key, which counts calls
 * on the host.  Between aie_rollout_capture_begin and aie_rollout_capture_end, aie_sample_policy launches
 * aie_sample_policy_counter_kernel, whose key is host_mix64(seed) ^ host_mix64(base + i + 1): base is read on the device
 * from the handle's call counter, i is the call's ordinal since capture_begin, baked into the launch.  That is the key
 * of call base + i + 1 of an eager loop, so a replay draws what the same calls made eagerly from the same state would.
 *
 * aie_rollout_capture_begin: needs a bound rollout at slot 0.  Allocates the handle's device counter (16 bytes, once,
 * before any capture is opened: nothing may allocate inside one), writes policy_calls into it on `stream`, saves the
 * host state (slot cursor, policy_calls, launch count) and switches aie_sample_policy to the variant above.  Between it
 * and aie_rollout_capture_end only aie_step and aie_sample_policy are allowed (every other entry point of the handle is
 * AIE_ESTATE); the caller opens and closes the stream capture inside the pair.  aie_rollout_capture_end records what the
 * captured calls did (steps, sampler calls, launches) and puts the saved host state back: nothing was executed.
 * aie_rollout_replay_begin: needs slot 0 and a capture in the bound rollout (aie_bind_rollout, bind or unbind, drops
 * it); writes the current policy_calls into the device counter with one launch on `stream`, which the caller then
 * replays the graph on.  aie_rollout_replay_end applies the recorded deltas: s = the captured steps (T), policy_calls
 * += the captured sampler calls, the launch count += the captured launches.  Eager rollouts may run between replays.
 *
 * A capture opened without the pair is refused rather than recorded wrong: aie_step, aie_sample_policy,
 * aie_sample_random_actions, aie_set_fused_policy, aie_reset_envs, aie_load_state, aie_rollout_restart and the pair's
 * own calls return AIE_ESTATE when their stream is being captured outside capture_begin / capture_end (the check is one
 * cudaStreamIsCapturing query; uncaptured calls are unchanged).
 * AIE_EINVAL for a NULL env; AIE_ESTATE as above, for a second capture_begin before capture_end, capture_end without
 * capture_begin, and replay_end without replay_begin; AIE_ENOMEM if the counter cannot be allocated. */
int aie_rollout_capture_begin(aie_env *env, void *stream);
int aie_rollout_capture_end(aie_env *env);
int aie_rollout_replay_begin(aie_env *env, void *stream);
int aie_rollout_replay_end(aie_env *env);

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
    /* ABI 6.  Element type of the seven observation / mask tensors, obs_agent_state .. mask_planner, of aie_covid_buffers
     * and of aie_covid_obs_buffers: AIE_OBS_F32 (default), or AIE_OBS_BF16 - every element is the round-to-nearest-even
     * bfloat16 of the float32 the default writes (a value computed in float64 is rounded to float32 first, then to
     * bfloat16), converted by the kernels that write it (same launches, half the bytes).  State, ints, hdr, ring,
     * changes, rewards, done and actions are unchanged; the masks are 0 / 1, so both samplers draw the same actions.
     * Any other value: AIE_EINVAL at aie_covid_create. */
    int32_t obs_dtype;
} aie_covid_config;

/* Device buffers (contiguous, env-major).  state: float32 [E, 9, S] = S, I, R, D, V, U, stringency, subsidy,
 * postsubsidy productivity at the current timestep; ints: int32 [E, 2, S] = cooldown_until, vaccines_available;
 * hdr: int32 [E, 4] = t, subsidy_level, ring_head, episodes; ring: int8 [E, S, ROW] stringency history, time-minor
 * (ROW = filter_len + 1 rounded up to a multiple of 16 bytes; logical entry k sits at column (ring_head + k) mod (L+1)).
 * Observations are the reference's collated "a"/"p" fields (covid19_env.py:919-993 + components), float32; with
 * aie_covid_config::obs_dtype == AIE_OBS_BF16 the seven float* observation / mask pointers point to bfloat16 storage
 * (2 bytes per element, same shapes). */
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

/* The seven observation / mask tensors of aie_covid_buffers, with the same shapes and element type (float32, or
 * bfloat16 storage under AIE_OBS_BF16). */
typedef struct aie_covid_obs_buffers {
    float *obs_agent_state, *obs_postsubsidy, *obs_lagged_stringency, *obs_policy_indicators, *obs_scalars,
          *mask_agent, *mask_planner;
} aie_covid_obs_buffers;

/* ABI 5.  aie_covid_step, and in the same launch the final observations of the episodes it ends: for every env whose
 * done flag this step sets, row e of `final_out` receives what aie_covid_step writes for that env with auto_reset off
 * (the observations and masks of the state its episode ended in; the bound tensors already show the next episode's
 * first).  Rows of the other envs are left untouched.  What a trainer bootstraps a truncated episode's value from.
 * One launch, asynchronous on `stream`.  AIE_EINVAL for a NULL env or final_out, a NULL member or a member not aligned
 * to its element (4 bytes, 2 under AIE_OBS_BF16); AIE_ESTATE before buffers are bound and the env has been reset, or
 * with auto_reset off. */
int aie_covid_step_final(aie_covid_env *env, const aie_covid_obs_buffers *final_out, void *stream);
/* Random policy on the device (uniform over the unmasked actions of the current masks); see aie_sample_random_actions. */
int aie_covid_sample_random_actions(aie_covid_env *env, uint64_t seed, void *stream);
/* A policy's actions on the device (the contract of aie_sample_policy): agent logits [E, S, 1 + levels] (action axis
 * last; the mask they are read against is mask_agent [E, 1 + levels, S]), planner logits [E, 1 + subsidy levels]
 * (required); log-probabilities [E, S] and [E].  Keys as the random policy's: env key k = cv_mix64(s ^ cv_mix64(env))
 * with s = host_mix64(seed) ^ host_mix64(n), n counting this env's aie_covid_sample_policy calls; state a draws with
 * k + 0x100 * a, the planner with k ^ 0xabcdef.  AIE_EINVAL also when 1 + subsidy levels > 160. */
int aie_covid_sample_policy(aie_covid_env *env, const aie_policy_logits *p, uint64_t seed, void *stream);
/* Log-probabilities, entropies and their gradient for stored actions (the contract of aie_evaluate_policy /
 * aie_evaluate_policy_backward): agent logits [N, S, 1 + levels] read against masks [N, 1 + levels, S], planner logits
 * and masks [N, 1 + subsidy levels] (required), actions [N, S] and [N]; outputs shaped like the actions.
 * AIE_EINVAL also when 1 + subsidy levels > 160. */
int aie_covid_evaluate_policy(aie_covid_env *env, const aie_policy_eval *p, int64_t n_rows, void *stream);
int aie_covid_evaluate_policy_backward(aie_covid_env *env, const aie_policy_eval *p, int64_t n_rows, void *stream);
/* Advantages and value targets of a stored rollout (the contract of aie_compute_advantages), A = S states. */
int aie_covid_compute_advantages(aie_covid_env *env, const aie_advantage_args *args, int32_t T, void *stream);
int64_t aie_covid_launch_count(const aie_covid_env *env);

/* A COVID-19 rollout stored in place (the contract of aie_rollout, with this scenario's tensors); K = ceil(T /
 * episode_length). */
typedef struct aie_covid_rollout {
    int32_t T;                    /* >= 1 */
    aie_covid_obs_buffers obs;    /* [T + 1, E, ...] each (slot t: the observation step t's action is taken from) */
    int32_t *actions_agent;       /* [T, E, S] */
    int32_t *actions_planner;     /* [T, E] */
    float *reward_agent;          /* [T, E, S] */
    double *reward_planner;       /* [T, E] */
    int32_t *done;                /* [T, E] */
    aie_covid_obs_buffers final_obs;   /* optional (every member NULL: none): [K, E, ...] each, row (k, e) the observation of
                                          the state in which replica e's k-th episode end within the rollout ended */
} aie_covid_rollout;
/* ABI 6 (additive).  aie_bind_rollout for the COVID-19 scenario: while bound, the samplers read the masks of slot s and
 * write the actions into slot s; aie_covid_step reads the actions of slot s, writes the observations into slot s + 1 and
 * the rewards and done into slot s, and on the step that ends an episode writes its final observations into row (k, e)
 * of final_obs in the same launch (aie_covid_step_final's kernel with its destination moved to row k); then s advances.
 * Every replica ends on the same step: aie_covid_reset starts them all at t = 0 and they step in lock-step, so k is one
 * host-side count (the episode ends this rollout has seen; hdr[:, 3], the episodes counter, grows by one on each) and
 * the step kernels are unchanged.  A caller that writes hdr's t itself breaks the lock-step and must not bind final
 * slots.  aie_covid_reset writes into slot 0 and is allowed only at s == 0.  AIE_ESTATE while bound: aie_covid_step and
 * the samplers at s == T, aie_covid_reset at s != 0, aie_covid_step_final and aie_covid_bind_buffers.  r == NULL
 * unbinds.  No launch.  AIE_EINVAL for T < 1, a NULL required pointer, a pointer not aligned to its element, or final
 * slots partly given; AIE_ESTATE before aie_covid_bind_buffers, or final slots without auto_reset. */
int aie_covid_bind_rollout(aie_covid_env *env, const aie_covid_rollout *r);
/* aie_rollout_restart for the COVID-19 scenario. */
int aie_covid_rollout_restart(aie_covid_env *env, void *stream);
/* aie_compute_advantages_k for the COVID-19 scenario, A = S states. */
int aie_covid_compute_advantages_k(aie_covid_env *env, const aie_advantage_args *args, int32_t T, int32_t K, void *stream);

/* ABI 6 (additive).  Episode metrics of the COVID-19 scenario: CovidAndEconomySimulation.scenario_metrics()
 * (covid19_env.py:1613-1687) of every replica, from accumulators the step kernel keeps in caller-owned DEVICE buffers.
 * Two blocks per replica, "current" (the running episode) and "previous" (the episode it finished last):
 *   sums / prev_sums    float64 [E, 4, S]: sums over t = 1..t of the float32 Unemployed, Stringency Level,
 *                       Postsubsidy Productivity and Subsidy the step stores, in step order
 *   index / prev_index  float32 [E, 2, S + 1]: Health Index then Economic Index, of each state then the planner, each
 *                       the float32 running sum of the step's marginal index (covid19_env.py:1124-1125, 1160-1161)
 *   prev_end            float32 [E, 4, S]: I, R, D, V of the state the previous episode ended in
 *   us_population       the divisor of the usa/ rates (model_constants.json US_POPULATION)
 * While bound, every step kernel adds to the current block (the same launches as without, in kernel variants that also
 * accumulate); the step that ends an episode under the auto-reset copies it, with the end state, to the previous block
 * and zeroes it, before the reset.  aie_covid_reset zeroes the current block, and accumulation counts from there: bind,
 * then reset.  m == NULL unbinds.  No launch.  AIE_EINVAL for a NULL pointer, a pointer not aligned to its element or
 * us_population <= 0; AIE_ESTATE before aie_covid_bind_buffers or while a rollout is bound. */
typedef struct aie_covid_metric_buffers {
    double *sums, *prev_sums;
    float *index, *prev_index, *prev_end;
    double us_population;
} aie_covid_metric_buffers;
int aie_covid_bind_metrics(aie_covid_env *env, const aie_covid_metric_buffers *m);
/* The columns of aie_covid_episode_metrics, in the reference's dict order: for each state s = 0..S-1 the eight fields
 * "infected (millions)", "recovered (millions)", "deaths (millions)", "mean_unemployment_rate (%)",
 * "mean_open_close_stringency_level", "total_productivity (billion $)", "health_index_at_end_of_episode",
 * "economic_index_at_end_of_episode" (state = s; the key is "<state name>/<field>"), then seven with state = -1 (key
 * "usa/<field>").  The library holds no state names.  Fills at most cap entries, returns K = 8 S + 7 (or a negative
 * AIE_E* code). */
typedef struct aie_covid_metric_column { int32_t state; char field[60]; } aie_covid_metric_column;
int aie_covid_get_metric_layout(const aie_covid_env *env, aie_covid_metric_column *out, int32_t cap);
/* One launch (aie_covid_metrics_kernel: one CTA per replica, one thread per state) writes float64 [n_envs, K] to the
 * DEVICE buffer out.  source 0: the current block and the live state (env.metrics mid-episode: the time means divide by
 * episode_length, as the reference's zero-padded global_state does); 1: the previous block (previous_episode_metrics).
 * Each value is float64 arithmetic in a fixed order (USA sums over the states in index order).  Asynchronous on
 * `stream`.  AIE_EINVAL for a NULL or misaligned out or an unknown source; AIE_ESTATE without bound metric buffers,
 * before aie_covid_reset has run since they were bound, or for source 1 before an episode has ended since then. */
int aie_covid_episode_metrics(aie_covid_env *env, int32_t source, double *out, void *stream);

/* ABI 6 (additive).  The host-side counters of a COVID-19 handle (the contract of aie_get_counters / aie_set_counters):
 * with them and the caller's buffers (state, ints, hdr, ring, changes, and the metric accumulators when bound) a
 * checkpoint resumes bit for bit.  aie_covid_set_counters marks the env reset (the caller has written its buffers),
 * with its metric accumulators live when they are bound.  AIE_EINVAL for a NULL env or counters, and (set) t < 0 or
 * previous_episode not 0 or 1; AIE_ESTATE before aie_covid_bind_buffers or while a rollout is bound at s != 0. */
typedef struct aie_covid_counters {
    uint64_t sample_calls;       /* aie_covid_sample_random_actions calls */
    uint64_t policy_calls;       /* aie_covid_sample_policy calls */
    int32_t t;                   /* the replicas' lock-step timestep */
    int32_t previous_episode;    /* 1: an episode has ended since the metric buffers were bound (source 1 is valid) */
} aie_covid_counters;
int aie_covid_get_counters(aie_covid_env *env, aie_covid_counters *out);
int aie_covid_set_counters(aie_covid_env *env, const aie_covid_counters *in);

/* ABI 6 (additive).  A captured rollout of the COVID-19 scenario: the contract of aie_rollout_capture_begin and its three
 * companions, with aie_covid_step and aie_covid_sample_policy the calls allowed inside the pair (aie_covid_sample_policy
 * launches aie_covid_sample_policy_counter_kernel, keyed as the gather-trade-build one).  The eager step picks the final
 * row k and the kernel from the host's lock-step timestep; inside the pair, with final slots bound, every step launches
 * aie_covid_step_slot_kernel instead, which finds the step that ends an episode from the record's own t and the row k
 * from the replica's done flags in slots 0 .. s - 1 of the rollout (the ordinal the gather-trade-build final pass uses).
 * capture_begin also saves the timestep, the episode-end count of the rollout and the previous-episode flag, and
 * capture_end puts them back; aie_covid_rollout_replay_end advances them as T eager steps would (every replica ends an
 * episode on the same step).  Refused on a capture opened without the pair: aie_covid_step, aie_covid_step_final,
 * aie_covid_sample_policy, aie_covid_sample_random_actions, aie_covid_reset, aie_covid_rollout_restart. */
int aie_covid_rollout_capture_begin(aie_covid_env *env, void *stream);
int aie_covid_rollout_capture_end(aie_covid_env *env);
int aie_covid_rollout_replay_begin(aie_covid_env *env, void *stream);
int aie_covid_rollout_replay_end(aie_covid_env *env);

const char *aie_last_error(void);
int aie_abi_version(void);

#ifdef __cplusplus
}
#endif
#endif /* AIE_B200_H */
