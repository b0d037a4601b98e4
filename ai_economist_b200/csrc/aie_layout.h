// aie_layout.h — device-side configuration (DevCfg) and the packed per-env state record layout.
//
// One env replica = one contiguous, 16-byte aligned record in HBM ("state" tensor, uint8 [E, rec_bytes]).
// Inside a record the state is struct-of-arrays indexed [agent, ...]; across envs the records are
// env-major, so every per-field tensor the north star names is a strided view [E, A, ...] over `state`
// (aie_get_field).  The step kernel moves a whole record HBM -> shared memory with one TMA bulk copy
// (cp.async.bulk), works on it in shared memory, and bulk-copies it back; the observe kernel bulk-loads
// only the prefix [0, obs_prefix_bytes) (everything except the order slots and the MT19937 key).
//
// Reference state this replaces: Maps (base/world.py:13-329), BaseAgent.state (base/base_agent.py:62),
// ContinuousDoubleAuction book/histograms (continuous_double_auction.py:79-99), PeriodicBracketTax
// trackers (redistribution.py:319-330), scenario utility trackers (layout_from_file.py:160-163) and the
// numpy global MT19937 state (base_env.py:481-494).
#pragma once
#include <stdint.h>

namespace aie {

// cell bitfield (1 byte per map cell); max_health == 1 for every entity in the supported configs
enum : uint8_t {
    CELL_STONE = 1u << 0, CELL_WOOD = 1u << 1, CELL_STONE_SRC = 1u << 2, CELL_WOOD_SRC = 1u << 3,
    CELL_WATER = 1u << 4, CELL_HOUSE = 1u << 5
};

// header words (int32) at the start of a record
enum { HDR_T = 0, HDR_TAX_POS = 1, HDR_COMPLETIONS = 2, HDR_AUTO_WARMUP = 3, HDR_MT_POS = 4,
       HDR_ERR = 5, HDR_EPISODES = 6, HDR_SAEZ_N = 7 /* (income, rate) samples seen so far, survives resets */,
       HDR_WORDS = 8 };

// Episode statistics ("stats" section of the record, float64, zeroed at reset): what the reference's component
// get_metrics() need beyond the live state (build.py:198-222, continuous_double_auction.py:585-641,
// redistribution.py:1141-1186).  Counts are stored as doubles (exact below 2^53).
//   [ST_N_TRADES]                                   executed trades
//   [ST_BUILDS + a]                                 houses built by agent a
//   [st_trade + (((a*2 + c)*2 + side)*2 + k)]       side 0 = as seller, 1 = as buyer; k 0 = count, 1 = sum of prices
//   [st_tax + ST_TAX_*]  (only with PeriodicBracketTax) periods enacted, total collected, sum of effective rates,
//                        sum of each bracket's rate over periods [16], bracket occupancy [16],
//                        then per agent: sum of max(0, income) over tax days [A], sum of tax paid [A]
enum { ST_N_TRADES = 0, ST_BUILDS = 1 };
enum { ST_TAX_PERIODS = 0, ST_TAX_COLLECTED = 1, ST_TAX_EFF_SUM = 2, ST_TAX_SCHED = 3, ST_TAX_OCC = 19, ST_TAX_AGENT = 35 };

// per-step event rows (int32[8]); row 0 of an env's block is the header {count, t, dropped, 0...}
//   EV_BUILD  {kind, agent, row, col}
//   EV_GATHER {kind, agent, resource (0 Stone, 1 Wood), n, row, col}
//   EV_TRADE  {kind, seller, buyer, commodity, ask, bid, ask_lifetime, bid_lifetime}
enum { EV_BUILD = 1, EV_GATHER = 2, EV_TRADE = 3 };

enum { COMP_BUILD = 0, COMP_CDA = 1, COMP_GATHER = 2, COMP_TAX = 3, COMP_WEALTH = 4, COMP_LABOR = 5, COMP_KINDS = 6 };
enum { SUB_BUILD = 0, SUB_BUY = 1, SUB_SELL = 2, SUB_GATHER = 3, SUB_LABOR = 4 };

// Observation "programs" (built once on the host from the reference's sorted-key flattening, base_env.py:562-612).
// flat entry  = kind << 13 | payload:
//   FK_SHARED  payload = index into the per-env shared float staging array (SH_*, then sh_full: full bid/ask counts)
//   FK_AGENT   payload = index of one of the agent's scalar observations (AS_*)
//   FK_MY      payload = i = (side * 2 + commodity) * P + price level (side 0 bids, 1 asks): the agent's own open orders there,
//              read from the record's uint8 histograms at hoff[i] + agent * P (hoff: table built on the host)
//   FK_AVAIL   same i: everybody else's open orders = full count (shared staging at sh_full + i) - own
// mask entry  = slot << 8 | idx; the mask value is (idx < limit[agent][slot])
// mask segment = count << 8 | slot: `count` consecutive mask entries of one slot with idx 0 .. count-1 (random policy)
enum { FK_SHARED = 0, FK_AGENT = 1, FK_MY = 2, FK_AVAIL = 3 };
// observation staging buffers (see ObsScratch in aie_obs.cuh); offsets DevCfg::ob[] / ob_emu[]
enum { OB_NET_HIST = 0, OB_SHF, OB_SC_A, OB_LIM, OB_PSH, OB_LOCMAP, OB_WC, OB_WI, OB_PL, OB_BITS, OB_VALS, OB_COUNT };
enum { AS_LOC_ROW = 0, AS_LOC_COL, AS_INV_COIN, AS_INV_STONE, AS_INV_WOOD, AS_BUILD_PAYMENT, AS_BUILD_SKILL, AS_BONUS,
       AS_TAX_MARG, AS_TAX_LAST_INCOME, AS_TAX_LAST_MARG, AS_LABOR_SKILL /* one-step-economy */, AS_COUNT = 12 };
enum { SH_ZERO = 0, SH_TIME = 1, SH_MARKET_RATE = 2, SH_ONE_PROD = 2, SH_ONE_EQ = 3 /* one-step-economy (no auction): planner scalars */, SH_TAX_IS_TAX_DAY = 4, SH_TAX_IS_FIRST = 5, SH_TAX_PHASE = 6,
       SH_PRICE_HIST = 8 /* [2][P], then curr_rates [16], then sorted last incomes [A] */ };
enum { MS_ONE = 0, MS_BUILD, MS_BUY0, MS_BUY1, MS_SELL0, MS_SELL1, MS_G0, MS_G1, MS_G2, MS_G3, MS_LABOR, MS_COUNT = 12 };

#define AIE_FLAT_ENTRY(kind, payload) ((uint16_t)(((kind) << 13) | (payload)))
#define AIE_FLAT_KIND(e) ((e) >> 13)
#define AIE_FLAT_PAYLOAD(e) ((e) & 0x1FFF)
#define AIE_MASK_ENTRY(slot, idx) ((uint16_t)(((slot) << 8) | (idx)))

constexpr int MAX_FLAT = 448;
constexpr int MAX_MASK = 160;
constexpr uint32_t ORDER_EMPTY = 0xFFFFFFFFu;  // order slot: birth << 8 | price << 1 | side(0 bid, 1 ask)

struct DevCfg {
    int32_t A, H, W, HW, T, multi_action, n_comp;
    int32_t comp[8];
    int32_t has[8];
    int32_t has_water, M, w, win, planner_spatial, obs_scaling;
    uint64_t regen_thresh[2];  // ceil(regen_weight * 2^53): u < weight  <=>  53-bit integer draw < thresh
    double eta, energy_cost, warm_const;
    int32_t warm_auto, swf;
    double mix;
    double build_payment, build_labor, move_labor, collect_labor, order_labor;
    int32_t P, D, K;
    uint32_t K_magic;  // floor(2^32 / K) + 1, or 0 when K == 1
    int32_t tax_model, disable_taxes, period, B, R;
    double cutoffs[16], disc_rates[64], fixed_rates[16];
    int32_t tax_annealing;
    double ann_warm, ann_slope, rate_max, ann_full, rate_min;
    int32_t auto_reset;
    int32_t reset_mode, build_skill_dist, gather_skill_dist, pmsm, fixed_four;
    int16_t ranked_locs[64][2];
    double avg_ranked_skill[64];
    // action subspaces in registration order (base_agent.py:97-169)
    int32_t n_sub;
    int32_t sub_kind[8], sub_c[8], sub_n[8], sub_lo[8];
    int32_t n_act_a, n_act_p, planner_acts;
    // output dims
    int32_t Fa, Fp, Fpa, Na, Np;
    // record layout (byte offsets)
    int32_t off_coin, off_esc_coin, off_labor, off_bpay, off_bskill, off_bonus, off_last_coin, off_last_income,
        off_last_marg, off_util_prev, off_price_hist, off_inv, off_esc, off_loc, off_n_orders, off_bid_hist,
        off_ask_hist, off_rate_idx, off_cell, off_owner, off_orders, off_mt, off_stats, off_saez;
    int32_t keep_bytes;  // [off_mt, off_mt + keep_bytes): what a reset never touches (MT key, then the Saez rates)
    int32_t n_stats, st_trade, st_tax;  // stats section: doubles, sub-offsets (st_tax < 0: no tax component)
    int32_t obs_prefix_bytes, rec_bytes;
    // Large envs (deep order books, many agents) keep the two big, sparsely touched sections - price history and
    // order slots, laid out last - in HBM/L2 and stage only [0, resident_bytes) in shared memory (split != 0).
    int32_t split, resident_bytes;
    // The observation pass runs after the record has been written back.  Its staging buffers live, where they fit, on top
    // of DEAD parts of the record's shared-memory image: the MT19937 key (dead from the start of the pass: obs_alias_mt
    // != 0 makes the kernel write the key back as its own first bulk group) and, once the scalars are staged, the price
    // history / order slots (kernel waits for the whole write-back to have been read first).  What does not fit goes to
    // obs_extra_bytes of additional shared memory per env.  The value staging of the flat vectors (OB_VALS) shares its bytes
    // with the window / plane buffers (OB_WC, OB_WI, OB_PL, OB_BITS): the flat runs are finished before those are first used.  ob[]: byte offsets from the env's shared-memory region
    // (the suite's host emulation, tests/emu, stages on an image of that region too).  ob_emu[]: offsets inside a separate
    // scratch allocation of obs_scratch_bytes, for a host emulation that keeps the staging apart from a live record; no
    // kernel reads them.
    int32_t obs_alias_mt, obs_extra_bytes;
    int32_t ob[OB_COUNT], ob_emu[OB_COUNT];
    int32_t ob_chunk;       // agents whose windows are staged / streamed together
    int32_t fl_chunk;       // agents whose flat vectors / masks / p<i> rows are staged (OB_VALS) and copied out together
    int32_t vals_off[4];    // float offsets inside OB_VALS of the four staged runs: agent flat rows, agent mask rows, p<i> rows, planner flat
    int32_t wc_stride;      // bytes per agent of the window-cell staging (window cells rounded up to 8)
    int32_t pl_stride_a, pl_stride_p;   // bytes per plane-local bitmap: one agent window / the whole map
    // mw: warps cooperating on one env in the step / observe kernels (1: one warp per env, several envs per CTA;
    // 4: one CTA per env for large records - warp 0 runs the dynamics, all four stream the observations)
    int32_t mw;
    // step-kernel scratch (per env, shared memory, behind the record image); separate observation scratch (ob_emu[])
    int32_t step_scratch_bytes, obs_scratch_bytes;
    int32_t n_envs;
    int32_t sh_curr_rates, sh_last_incomes, sh_full, sh_count;  // offsets / size of the shared float staging array
    int32_t tab_p, tab_pa, tab_m, tab_n;               // offsets (u16 words) into the program table, total words (even)
    int32_t tab_hoff, tab_seg, tab_lut;                // more tables in the same array: histogram offsets [4P], mask segments, nibble -> float4 table (16-byte aligned)
    int32_t tab_cslot;                                 // [Fa] (behind tab_n, not staged): index of agent-flat entry j inside its class (shared / agent scalar / order count), for the compacted transfer
    int32_t cf_n_sh, cf_n_ag, cf_n_cnt;                // entries per class of the agents' flat vector
    int32_t seg_lo[10];                                // mask segments of action subspace si: [seg_lo[si], seg_lo[si + 1]) (single-action agents: si = 0 covers everything)
    uint32_t HW_magic, ww_magic, Fa_magic, Fpa_magic, Na_magic;  // floor(2^32 / n) + 1: run index -> (row, column)
    uint32_t wcu_magic;     // floor(2^32 / (wc_stride / 8)) + 1: (agent, 8-cell unit) pairs of a chunk
    uint32_t win_magic; int32_t win_dr32, win_dc32;  // window walk: lane / win, and the (row, col) step of 32 cells
    // single-action planner (multi_action_mode_planner=False): act_p is one index into [NO-OP] ++ B x R rates
    int32_t planner_single;
    int32_t ext;  // planner_single or a regen halfwidth is set: the host launches the EXT instantiations of the kernels
    // regen_halfwidth > 0 (cold path): threshold by the number n of source cells in the d x d window of the cell,
    // regen_tab[c][n] = ceil(p_n * 2^53) with p_n the running float64 sum of n copies of regen_weight / d^2
    int32_t regen_hw[2];
    uint64_t regen_tab[2][50];
    // full_observability: agents get the whole map; a_map_elems / a_idx_elems = elements per agent of the two tensors
    int32_t full_obs, a_map_elems, a_idx_elems;
    // lognormal skills on the device reset: numpy's legacy_gauss cache {cached value, has_gauss as 0.0 / 1.0}, f64[2], in the
    // part of the record a reset keeps (0: no such section)
    int32_t off_gauss;
    // split_layout device reset: per-replica rank -> build payment table f64[A] in the kept part of the record
    int32_t split_layout, split_water_row, off_split_skill;
    uint64_t split_top_ranks;
    // one-step-economy (aie_config::scenario_kind == 1): no map, SimpleLabor, coin-minus-labor-cost utilities
    int32_t one_step, agent_reward_type, labor_mask_first, no_spatial;
    double labor_exponent, labor_cost, labor_skill_scale;
    // dynamic-layout scenarios: device-side layout generation at reset (see aie_config::dyn_layout)
    int32_t dyn_layout, dyn_checker;
    double dyn_cov[2], dyn_clump[2];   // [Wood, Stone]
    int32_t mz_rows, mz_cols, mz_psr, mz_psc, mz_zones[3];   // MultiZone: partitions, partition size in cells, zones per type
};

// raw device pointers (mirrors aie_buffers)
struct DevBufs {
    uint8_t *state, *state0, *final;  // final: optional end-of-episode record snapshots (auto-reset)
    const int32_t *act_a, *act_p;
    float *a_map; int16_t *a_idx; float *a_flat; float *a_mask;
    float *p_map; int16_t *p_idx; float *p_flat; float *p_agents; float *p_mask;
    float *time_obs; double *rew; int32_t *done;
    // observation / mask programs in device memory (library-owned, written once at aie_create): indexed by the
    // thread-varying flat position, which would serialise on the constant bank if read from the kernel params
    const uint16_t *tab;
    // optional per-step event log of the first event_envs replicas (dense logs): int32 [event_envs][event_cap + 1][8]
    int32_t *events; int32_t event_envs, event_cap;
    // dynamic layouts (library-owned): source probability maps f64 [2][HW] and one f64 [HW] work map per env
    const double *dyn_prob; double *dyn_work;
    // non-zero (aie_set_fused_policy): the observation pass also draws the NEXT step's uniformly random unmasked actions
    // into the action buffers, from the mask limits it has just staged - instead of a separate sampler launch per step
    uint64_t policy_seed;
};
// compact program table: [agent flat (Fa) | planner flat (Fp) | p<i> flat (Fpa) | agent mask (Na)], offsets in DevCfg
// then: histogram offsets u16 [4P <= 128], mask segments u16 [<= 64], nibble -> float4 table (64 floats = 128 u16)
constexpr int TAB_WORDS = 2 * MAX_FLAT + 16 + MAX_MASK + 128 + 64 + 128 + 16 + MAX_FLAT;
struct Tables { uint16_t w[TAB_WORDS]; };

}  // namespace aie
