// aie_core.cuh — per-env dynamics ("step") and observation ("observe") bodies.
//
// Compiled two ways:
//   * nvcc, sm_90a: NL = 32 lanes.  One warp owns one env replica whose state record lives in shared
//     memory.  Order-dependent sections (agent loops in np.random.permutation order, auction matching) run
//     as warp-uniform code — every lane evaluates the same control flow from shared memory, lane 0 commits
//     the writes — so warp collectives (MT19937 twist, redux/ballot scans of the order book) can be called
//     from anywhere inside them.  Embarrassingly parallel sections (order creation/expiry, price-history
//     decay, regeneration over the grid, taxes, utilities) stride agents/cells across lanes.
//   * g++ with -DAIE_EMU (tests/emu only): NL = 1, collectives degenerate to identities.  This is a logic
//     check of the same source on the build container, which has no GPU.  It is never built into or loaded
//     by the product library.
//
// Reference semantics restated here (paths relative to ai_economist/foundation/):
//   Build.component_step                      components/build.py:112-161
//   ContinuousDoubleAuction.component_step    components/continuous_double_auction.py:440-489 (+168-406)
//   Gather.component_step                     components/move.py:93-153
//   PeriodicBracketTax.component_step         components/redistribution.py:945-972 (+419-434, 837-915)
//   LayoutFromFile.scenario_step              scenarios/simple_wood_and_stone/layout_from_file.py:372-410
//   compute_reward / optimization metrics     layout_from_file.py:269-318, 519-559; scenarios/utils/*.py
//   generate_observations / masks             layout_from_file.py:412-517; base/base_env.py:562-756;
//                                             build.py:163-193; move.py:155-188;
//                                             continuous_double_auction.py:491-580; redistribution.py:974-1104
//   numpy legacy RandomState stream           numpy/random/src/mt19937/mt19937.c, legacy-distributions.c
#pragma once
#include <math.h>
#include <stdint.h>
#include <string.h>

#include "aie_layout.h"
#if defined(__CUDACC__) && !defined(AIE_EMU)
#include <cuda_bf16.h>
#endif

#if defined(__CUDACC__) && !defined(AIE_EMU)
#define AIE_DEV __device__ __forceinline__
#define AIE_DEV_MEMBER __device__ __forceinline__
#define AIE_DEV_NOINLINE __device__ __noinline__
#define AIE_ON_DEVICE 1
#else
#define AIE_DEV static inline
#define AIE_DEV_MEMBER inline
#define AIE_DEV_NOINLINE static
#define AIE_ON_DEVICE 0
#endif

#ifndef AIE_TWIST_UNROLL
#define AIE_TWIST_UNROLL 8
#endif
#define AIE_PRAGMA_(x) _Pragma(#x)
#define AIE_UNROLL(n) AIE_PRAGMA_(unroll n)

namespace aie {

#if AIE_ON_DEVICE
constexpr int NL = 32;
AIE_DEV void wsync() { __syncwarp(); }
AIE_DEV uint32_t wmax(uint32_t v) { return __reduce_max_sync(0xffffffffu, v); }
AIE_DEV uint32_t wballot(bool p) { return __ballot_sync(0xffffffffu, p); }
AIE_DEV uint32_t wshfl(uint32_t v, int src) { return __shfl_sync(0xffffffffu, v, src); }
AIE_DEV bool wany(bool p) { return __any_sync(0xffffffffu, p); }
AIE_DEV double wsum(double v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
AIE_DEV int first_lane(uint32_t m) { return __ffs(m) - 1; }
// The calling thread's lane, read afresh from %laneid (volatile: never merged with an earlier read).  A lane index kept
// live through the whole step is the value the 64-register variant spills first; re-reading it at the start of each
// component / observation phase keeps its live ranges short.  `lane` is the value the caller holds (host emulation).
AIE_DEV int relane(int) { int l; asm volatile("mov.u32 %0, %%laneid;" : "=r"(l)); return l; }
AIE_DEV int __popc_u32(uint32_t m) { return __popc(m); }
AIE_DEV uint32_t fshr(uint32_t lo, uint32_t hi, int sh) { return __funnelshift_r(lo, hi, sh); }  // sh in [0, 31]
AIE_DEV uint32_t prmt(uint32_t a, uint32_t b, uint32_t sel) { return __byte_perm(a, b, sel); }
#else
#ifndef AIE_EMU_NL
#define AIE_EMU_NL 1   // tests/emu/planes_check.cpp sets 32 to walk the per-lane store loops lane by lane (no collectives there)
#endif
constexpr int NL = AIE_EMU_NL;
AIE_DEV void wsync() {}
AIE_DEV uint32_t wmax(uint32_t v) { return v; }
AIE_DEV uint32_t wballot(bool p) { return p ? 1u : 0u; }
AIE_DEV uint32_t wshfl(uint32_t v, int) { return v; }
AIE_DEV bool wany(bool p) { return p; }
AIE_DEV double wsum(double v) { return v; }
AIE_DEV int first_lane(uint32_t m) { return m ? 0 : -1; }
AIE_DEV int relane(int lane) { return lane; }
AIE_DEV int __popc_u32(uint32_t m) { return __builtin_popcount(m); }
AIE_DEV uint32_t fshr(uint32_t lo, uint32_t hi, int sh) { return sh ? (lo >> sh) | (hi << (32 - sh)) : lo; }
AIE_DEV uint32_t prmt(uint32_t a, uint32_t b, uint32_t sel) {
    const uint64_t v = ((uint64_t)b << 32) | a;
    uint32_t r = 0;
    for (int i = 0; i < 4; i++) r |= (uint32_t)((v >> (8 * ((sel >> (4 * i)) & 7))) & 0xFFu) << (8 * i);
    return r;
}
#endif

// ------------------------------------------------------------------------------------------------
// Views into a state record
// ------------------------------------------------------------------------------------------------
struct Env {
    int32_t *hdr;
    double *coin, *esc_coin, *labor, *bpay, *bskill, *bonus, *last_coin, *last_income, *last_marg, *util_prev,
        *price_hist, *stats, *gauss, *split_skill, *saez;  // gauss: numpy legacy_gauss cache {value, has}; saez (Saez model only): [16] bracket rates, [16] running average, [16] observed rates
    int32_t *inv, *esc;  // [A][2]
    int16_t *loc;        // [A][2]
    uint8_t *n_orders, *bid_hist, *ask_hist, *rate_idx, *cell;
    int8_t *owner;
    uint32_t *orders, *mt;
    int32_t *ev; int32_t ev_cap;  // this env's event block for the current step, or nullptr (no dense log)
};

// rec: the resident image of the record (shared memory on the device); grec: the record in global memory, used for
// the price-history / order-slot sections when the config is split (large envs).  In emulation rec == grec.
AIE_DEV Env env_view(uint8_t *rec, uint8_t *grec, const DevCfg &c) {
    Env e;
    e.ev = nullptr; e.ev_cap = 0;
    uint8_t *big = c.split ? grec : rec;
    e.hdr = (int32_t *)rec;
    e.coin = (double *)(rec + c.off_coin);
    e.saez = (double *)(rec + c.off_saez);
    e.gauss = (double *)(rec + c.off_gauss);
    e.split_skill = (double *)(rec + c.off_split_skill);
    e.stats = (double *)(big + c.off_stats);  // resident unless the config is split
    e.esc_coin = (double *)(rec + c.off_esc_coin);
    e.labor = (double *)(rec + c.off_labor);
    e.bpay = (double *)(rec + c.off_bpay);
    e.bskill = (double *)(rec + c.off_bskill);
    e.bonus = (double *)(rec + c.off_bonus);
    e.last_coin = (double *)(rec + c.off_last_coin);
    e.last_income = (double *)(rec + c.off_last_income);
    e.last_marg = (double *)(rec + c.off_last_marg);
    e.util_prev = (double *)(rec + c.off_util_prev);
    e.price_hist = (double *)(big + c.off_price_hist);
    e.inv = (int32_t *)(rec + c.off_inv);
    e.esc = (int32_t *)(rec + c.off_esc);
    e.loc = (int16_t *)(rec + c.off_loc);
    e.n_orders = rec + c.off_n_orders;
    e.bid_hist = rec + c.off_bid_hist;
    e.ask_hist = rec + c.off_ask_hist;
    e.rate_idx = rec + c.off_rate_idx;
    e.cell = rec + c.off_cell;
    e.owner = (int8_t *)(rec + c.off_owner);
    e.orders = (uint32_t *)(big + c.off_orders);
    e.mt = (uint32_t *)(rec + c.off_mt);
    return e;
}

// Component sets the step body can be compiled for (bit k: component kind k is handled).  The one-warp step kernel is
// instantiated per set and the host launches the smallest set that holds the config's components, so a config without
// taxes does not carry the tax code inside its hot loops.
constexpr int CS_GTB = (1 << COMP_BUILD) | (1 << COMP_CDA) | (1 << COMP_GATHER);   // gather-trade-build
constexpr int CS_GTB_TAX = CS_GTB | (1 << COMP_TAX);
constexpr int CS_ALL = (1 << COMP_KINDS) - 1;
inline int step_comp_set(const DevCfg &c) {
    int m = 0;
    for (int i = 0; i < c.n_comp; i++) m |= 1 << c.comp[i];
    return (m & ~CS_GTB) == 0 ? CS_GTB : (m & ~CS_GTB_TAX) == 0 ? CS_GTB_TAX : CS_ALL;
}

// Append one event row (called by the committing lane only).  Rows beyond the capacity are counted as dropped.
// Only the dense-log replicas have an event block: the row writer is kept out of line.
AIE_DEV_NOINLINE void emit_event_row(int32_t *ev, int cap, int kind, int a0, int a1, int a2, int a3, int a4, int a5, int a6) {
    const int n = ev[0];
    if (n >= cap) { ev[2] += 1; return; }
    int32_t *row = ev + 8 * (n + 1);
    row[0] = kind; row[1] = a0; row[2] = a1; row[3] = a2; row[4] = a3; row[5] = a4; row[6] = a5; row[7] = a6;
    ev[0] = n + 1;
}
AIE_DEV void emit_event(const Env &e, int kind, int a0, int a1 = 0, int a2 = 0, int a3 = 0, int a4 = 0, int a5 = 0, int a6 = 0) {
    if (e.ev) emit_event_row(e.ev, e.ev_cap, kind, a0, a1, a2, a3, a4, a5, a6);
}

// per-env scratch of the step body (shared memory on the device)
struct StepScratch {
    uint8_t *act_build, *act_move, *act_buy, *act_sell;  // [A], [A], [2][A], [2][A]
    uint8_t *act_tax;                                    // [16]
    uint8_t *perm;                                       // [A]
    double *tmp;                                         // [2A + 4]
    uint32_t *book;                                      // [4][A] per-agent best bid/ask key + slot (matching)
};
AIE_DEV StepScratch step_scratch_view(uint8_t *p, const DevCfg &c) {
    StepScratch s;
    s.tmp = (double *)p;  p += 8 * (2 * c.A + 4);
    s.book = (uint32_t *)p;  p += 16 * c.A;
    s.act_build = p;      p += c.A;
    s.act_move = p;       p += c.A;
    s.act_buy = p;        p += 2 * c.A;
    s.act_sell = p;       p += 2 * c.A;
    s.perm = p;           p += c.A;
    s.act_tax = p;
    return s;
}

// ------------------------------------------------------------------------------------------------
// numpy legacy MT19937 stream (bit-exact): mt19937_gen / mt19937_next / next_double / random_interval
// ------------------------------------------------------------------------------------------------
AIE_DEV uint32_t mt_temper(uint32_t y) {
    y ^= (y >> 11);
    y ^= (y << 7) & 0x9d2c5680u;
    y ^= (y << 15) & 0xefc60000u;
    y ^= (y >> 18);
    return y;
}

// One phase of the in-place twist: key[k] = key[k + MOFF] ^ f(key[k], key[k+1]) for k in [BASE, BASE+N).
// Every lane first computes all of its outputs from the old values, then the warp syncs, then stores, so
// reads of key[k+1] never see this phase's writes.
template <int BASE, int N, int MOFF>
AIE_DEV void mt_twist_phase(uint32_t *mt, int lane) {
    constexpr int PER = (N + NL - 1) / NL;
    uint32_t v[PER];
#if AIE_ON_DEVICE
    AIE_UNROLL(AIE_TWIST_UNROLL)
#endif
    for (int j = 0; j < PER; j++) {
        int k = BASE + lane + j * NL;
        if (k < BASE + N) {
            uint32_t y = (mt[k] & 0x80000000u) | (mt[k + 1] & 0x7fffffffu);
            v[j] = mt[k + MOFF] ^ (y >> 1) ^ ((y & 1u) ? 0x9908b0dfu : 0u);
        }
    }
    wsync();
#if AIE_ON_DEVICE
    AIE_UNROLL(AIE_TWIST_UNROLL)
#endif
    for (int j = 0; j < PER; j++) {
        int k = BASE + lane + j * NL;
        if (k < BASE + N) mt[k] = v[j];
    }
    wsync();
}

// Warp-collective regeneration of the 624-word key.  Dependencies: new[0,227) <- old; new[227,454) <-
// new[0,227); new[454,623) <- new[227,396); new[623] <- new[396], new[0].
// Not inlined: rng_next() is called from a dozen places and each inlined copy of the twist is ~700 instructions;
// a single copy keeps the kernel inside the instruction cache.
#if AIE_ON_DEVICE
// Device version: the same recurrence in chunks of 128 words, four consecutive words per lane (one 16-byte load of the
// old values, one 16-byte store).  Any split into chunks of at most 227 words keeps the dependencies of the in-place
// twist: word k takes key[k + 397] (still old: it lies in a later chunk) for k < 227 and key[k - 227] (already new: it
// lies in an earlier chunk) otherwise, and every chunk reads all its inputs before it stores.  Word 623 wraps around to
// the new key[0] and is done last by one lane.
__device__ __forceinline__ uint32_t mt_mix(uint32_t a, uint32_t b, uint32_t src) {
    const uint32_t y = (a & 0x80000000u) | (b & 0x7fffffffu);
    return src ^ (y >> 1) ^ ((0u - (y & 1u)) & 0x9908b0dfu);
}
template <int BASE>
__device__ __forceinline__ void mt_twist_chunk(uint32_t *mt, int lane) {
    const int k0 = BASE + 4 * lane;
    const bool act = k0 < 623;
    uint32_t v[4] = {0u, 0u, 0u, 0u};
    if (act) {
        const uint4 x = *reinterpret_cast<const uint4 *>(mt + k0);
        const uint32_t xs[5] = {x.x, x.y, x.z, x.w, mt[k0 + 4 < 624 ? k0 + 4 : 623]};
#pragma unroll
        for (int j = 0; j < 4; j++) {
            const int k = k0 + j;
            const int src = (BASE + 127 < 227) ? k + 397 : (BASE >= 227 ? k - 227 : (k < 227 ? k + 397 : k - 227));
            v[j] = mt_mix(xs[j], xs[j + 1], mt[src < 624 ? src : 623]);
        }
    }
    __syncwarp();
    if (act) {
        if (k0 + 4 <= 623) *reinterpret_cast<uint4 *>(mt + k0) = make_uint4(v[0], v[1], v[2], v[3]);
        else { for (int j = 0; j < 4; j++) if (k0 + j < 623) mt[k0 + j] = v[j]; }
    }
    __syncwarp();
}
AIE_DEV_NOINLINE void mt_twist(uint32_t *mt, int lane) {
    __syncwarp();
    mt_twist_chunk<0>(mt, lane);
    mt_twist_chunk<128>(mt, lane);
    mt_twist_chunk<256>(mt, lane);
    mt_twist_chunk<384>(mt, lane);
    mt_twist_chunk<512>(mt, lane);
    if (lane == 0) mt[623] = mt_mix(mt[623], mt[0], mt[396]);
    __syncwarp();
}
#else
AIE_DEV_NOINLINE void mt_twist(uint32_t *mt, int lane) {
    wsync();
    mt_twist_phase<0, 227, 397>(mt, lane);
    mt_twist_phase<227, 227, -227>(mt, lane);
    mt_twist_phase<454, 169, -227>(mt, lane);
    if (lane == 0) {
        uint32_t y = (mt[623] & 0x80000000u) | (mt[0] & 0x7fffffffu);
        mt[623] = mt[396] ^ (y >> 1) ^ ((y & 1u) ? 0x9908b0dfu : 0u);
    }
    wsync();
}
#endif

struct Rng {
    uint32_t *mt;
    int pos;   // warp-uniform
    int lane;
};

AIE_DEV uint32_t rng_next(Rng &r) {  // warp-uniform call
    if (r.pos == 624) { mt_twist(r.mt, r.lane); r.pos = 0; }
    return mt_temper(r.mt[r.pos++]);
}
AIE_DEV double rng_double(Rng &r) {  // np.random.rand()
    int32_t a = (int32_t)(rng_next(r) >> 5);
    int32_t b = (int32_t)(rng_next(r) >> 6);
    return (a * 67108864.0 + b) / 9007199254740992.0;
}
AIE_DEV uint32_t rng_interval(Rng &r, uint32_t max) {  // legacy random_interval, 32-bit path
    if (max == 0) return 0;
    uint32_t mask = max, v;
    mask |= mask >> 1; mask |= mask >> 2; mask |= mask >> 4; mask |= mask >> 8; mask |= mask >> 16;
    while ((v = (rng_next(r) & mask)) > max) {}
    return v;
}
// np.random.permutation(A) into scratch perm[] (world.get_random_order_agents, base/world.py:418-422)
AIE_DEV void rng_permutation(Rng &r, uint8_t *perm, int A) {
    for (int a = r.lane; a < A; a += NL) perm[a] = (uint8_t)a;
    wsync();
    for (int i = A - 1; i >= 1; i--) {
        int j = (int)rng_interval(r, (uint32_t)i);
        if (r.lane == 0) { uint8_t t = perm[j]; perm[j] = perm[i]; perm[i] = t; }
        wsync();
    }
}

// ------------------------------------------------------------------------------------------------
// Actions  (BaseAgent.parse_actions, base/base_agent.py:407-438)
// ------------------------------------------------------------------------------------------------
// EXT (here and below): compile the rarely used options in - single-action planner, regen_halfwidth > 0.  The kernels
// are instantiated both ways and the host picks by config (DevCfg::ext), so the default configurations run exactly
// the instruction stream that was profiled without those options.
template <bool EXT = false>
AIE_DEV void decode_actions(const DevCfg &c, const StepScratch &s, const int32_t *act_a, const int32_t *act_p,
                            int lane, const uint16_t *tab = nullptr) {
    for (int a = lane; a < c.A; a += NL) {
        uint8_t build = 0, move = 0, buy0 = 0, buy1 = 0, sell0 = 0, sell1 = 0;
        int g = (!c.multi_action && act_a) ? act_a[a] : 0;
        if (tab && !c.multi_action) {
            // single-action agents: the mask program already maps the flat action index to (subspace, level)
            if (g > 0 && g < c.Na) {
                const uint32_t en = tab[c.tab_m + g], slot = en >> 8, idx = en & 255u;
                if (slot == MS_BUILD) build = 1;
                else if (slot == MS_BUY0) buy0 = (uint8_t)(idx + 1);
                else if (slot == MS_BUY1) buy1 = (uint8_t)(idx + 1);
                else if (slot == MS_SELL0) sell0 = (uint8_t)(idx + 1);
                else if (slot == MS_SELL1) sell1 = (uint8_t)(idx + 1);
                else if (EXT && slot == MS_LABOR) move = (uint8_t)(idx + 1);   // hours of labor travel in the Gather slot
                else if (slot >= MS_G0) move = (uint8_t)(slot - MS_G0 + 1);
            }
        } else
        for (int si = 0; si < c.n_sub; si++) {
            int v;
            if (c.multi_action) v = act_a ? act_a[a * c.n_sub + si] : 0;
            else v = (g >= c.sub_lo[si] && g < c.sub_lo[si] + c.sub_n[si]) ? g - c.sub_lo[si] + 1 : 0;
            if (v < 0 || v > c.sub_n[si]) v = 0;  // out-of-range input is treated as NO-OP
            int kind = c.sub_kind[si];
            if (kind == SUB_BUILD) build = (uint8_t)v;
            else if (kind == SUB_GATHER || kind == SUB_LABOR) move = (uint8_t)v;
            else if (kind == SUB_BUY) { if (c.sub_c[si] == 0) buy0 = (uint8_t)v; else buy1 = (uint8_t)v; }
            else { if (c.sub_c[si] == 0) sell0 = (uint8_t)v; else sell1 = (uint8_t)v; }
        }
        s.act_build[a] = build; s.act_move[a] = move;
        s.act_buy[a] = buy0; s.act_buy[c.A + a] = buy1;
        s.act_sell[a] = sell0; s.act_sell[c.A + a] = sell1;
    }
    for (int b = lane; b < 16; b += NL) {
        int v;
        if (EXT && c.planner_single) {  // single_action_map (base_agent.py:109-114): bracket (g-1) / R, sub-action (g-1) % R + 1
            const int g = act_p ? act_p[0] - 1 : -1;
            v = (g >= 0 && g < c.B * c.R && g / c.R == b) ? g % c.R + 1 : 0;
        } else {
            v = (act_p && b < c.n_act_p) ? act_p[b] : 0;
        }
        if (v < 0 || v > c.R) v = 0;
        s.act_tax[b] = (uint8_t)v;
    }
    wsync();
}

// ------------------------------------------------------------------------------------------------
// Build  (components/build.py:70-83, 112-161)
// ------------------------------------------------------------------------------------------------
AIE_DEV bool can_build(const DevCfg &c, const Env &e, int a) {
    int k = e.loc[2 * a] * c.W + e.loc[2 * a + 1];
    // needs 1 Wood + 1 Stone; the cell must hold no resource and no landmark (House, Water, source block)
    return e.inv[2 * a] >= 1 && e.inv[2 * a + 1] >= 1 && e.cell[k] == 0;
}

AIE_DEV void build_step(const DevCfg &c, Env &e, const StepScratch &s, Rng &r) {
    rng_permutation(r, s.perm, c.A);
    for (int i = 0; i < c.A; i++) {
        int a = s.perm[i];
        const bool do_build = s.act_build[a] == 1 && can_build(c, e, a);
        wsync();  // every lane has evaluated the predicate before lane 0 changes the state it reads
        if (do_build) {
            if (r.lane == 0) {
                int k = e.loc[2 * a] * c.W + e.loc[2 * a + 1];
                e.inv[2 * a] -= 1;
                e.inv[2 * a + 1] -= 1;
                e.cell[k] |= CELL_HOUSE;
                e.owner[k] = (int8_t)a;
                e.coin[a] += e.bpay[a];
                e.labor[a] += c.build_labor;
                e.stats[ST_BUILDS + a] += 1.0;
                emit_event(e, EV_BUILD, a, e.loc[2 * a], e.loc[2 * a + 1]);
            }
        }
        wsync();
    }
}

// ------------------------------------------------------------------------------------------------
// ContinuousDoubleAuction  (components/continuous_double_auction.py)
// ------------------------------------------------------------------------------------------------
// i / K without a run-time division (K_magic = floor(2^32 / K) + 1, exact for i < 2^32 / K; K == 1 -> magic 0)
AIE_DEV int div_K(const DevCfg &c, int i) {
#if AIE_ON_DEVICE
    return c.K_magic ? (int)__umulhi((uint32_t)i, c.K_magic) : i;
#else
    return c.K_magic ? (int)(((uint64_t)(uint32_t)i * c.K_magic) >> 32) : i;
#endif
}

AIE_DEV uint32_t order_pack(int birth, int price, int side) { return ((uint32_t)birth << 8) | ((uint32_t)price << 1) | (uint32_t)side; }
AIE_DEV int order_birth(uint32_t o) { return (int)(o >> 8); }
AIE_DEV int order_price(uint32_t o) { return (int)((o >> 1) & 127u); }
AIE_DEV int order_side(uint32_t o) { return (int)(o & 1u); }

// BIG: the order slots live in global memory (split record).  Scans then avoid early exits and are unrolled so
// that ~10 independent loads are in flight per lane instead of one L2 round trip per slot.
template <bool BIG>
AIE_DEV void order_insert(uint32_t *slots, int K, uint32_t o) {
    if (!BIG) {
        for (int k = 0; k < K; k++)
            if (slots[k] == ORDER_EMPTY) { slots[k] = o; return; }
        return;
    }
    int pos = K;
#if AIE_ON_DEVICE
    AIE_UNROLL(10)
#endif
    for (int k = 0; k < K; k++)
        if (slots[k] == ORDER_EMPTY && k < pos) pos = k;
    if (pos < K) slots[pos] = o;
}

// :440-489 first half — price-history decay and order creation (create_bid :168-198, create_ask :200-229).
// Each agent only touches its own state, so agents run lane-parallel; agent-index order of the reference's
// loop survives as the final tie-break of the matching key.
template <bool BIG>
AIE_DEV void cda_create(const DevCfg &c, Env &e, const StepScratch &s, int t, int lane) {
    const int A = c.A, P = c.P, K = c.K;
#if AIE_ON_DEVICE
    AIE_UNROLL(4)
#endif
    for (int i = lane; i < 2 * A * P; i += NL) e.price_hist[i] *= 0.995;  // independent of order creation
    for (int a = lane; a < A; a += NL) {
        for (int cc = 0; cc < 2; cc++) {
            uint32_t *slots = e.orders + (cc * A + a) * K;
            int kb = s.act_buy[cc * A + a];
            if (kb != 0) {
                int price = kb - 1;
                if (e.n_orders[cc * A + a] < K && e.coin[a] >= (double)price) {
                    order_insert<BIG>(slots, K, order_pack(t, price, 0));
                    e.bid_hist[(cc * A + a) * P + price] += 1;
                    e.n_orders[cc * A + a] += 1;
                    e.coin[a] -= (double)price;
                    e.esc_coin[a] += (double)price;
                    e.labor[a] += c.order_labor;
                }
            }
            int ks = s.act_sell[cc * A + a];
            if (ks != 0) {
                int price = ks - 1;
                if (e.n_orders[cc * A + a] < K && e.inv[2 * a + cc] > 0) {
                    order_insert<BIG>(slots, K, order_pack(t, price, 1));
                    e.ask_hist[(cc * A + a) * P + price] += 1;
                    e.n_orders[cc * A + a] += 1;
                    e.inv[2 * a + cc] -= 1;
                    e.esc[2 * a + cc] += 1;
                    e.labor[a] += c.order_labor;
                }
            }
        }
    }
    wsync();
}

// match_orders :231-350.  The reference stable-sorts bids by (price desc, lifetime desc) and asks by
// (price asc, lifetime desc); ties keep creation order, i.e. agent index ascending.  Here every order maps to a
// packed key (price | lifetime | 255 - agent) with the same total order.  Each agent's best bid and best ask
// (key + slot) are found once per step; the restart-from-top loop then only reduces over agents (redux.max),
// and after a trade just the two agents involved rescan their own K slots.  Same buyer-level `possible_match`
// bookkeeping as the reference.
AIE_DEV uint32_t bid_key(int t, uint32_t o, int a) {
    return ((uint32_t)(order_price(o) + 1) << 20) | ((uint32_t)(t - order_birth(o)) << 8) | (uint32_t)(255 - a);
}
AIE_DEV uint32_t ask_key(int t, int P, uint32_t o, int a) {
    return ((uint32_t)(P - order_price(o)) << 20) | ((uint32_t)(t - order_birth(o)) << 8) | (uint32_t)(255 - a);
}
// best order of one side for agent a, scanned by the whole warp over its K slots; lane 0 stores it
AIE_DEV void refresh_best(const DevCfg &c, const uint32_t *slots, int a, int side, int t, uint32_t *best_key,
                          uint32_t *best_slot, int lane) {
    uint32_t bk = 0, bs = 0;
    for (int k = lane; k < c.K; k += NL) {
        const uint32_t o = slots[a * c.K + k];
        if (o != ORDER_EMPTY && order_side(o) == side) {
            const uint32_t key = side == 0 ? bid_key(t, o, a) : ask_key(t, c.P, o, a);
            if (key > bk) { bk = key; bs = (uint32_t)(a * c.K + k); }
        }
    }
    const uint32_t m = wmax(bk);
    bs = wshfl(bs, first_lane(wballot(bk == m)));
    wsync();
    if (lane == 0) { best_key[a] = m; best_slot[a] = bs; }
}

template <bool BIG>
AIE_DEV void cda_match(const DevCfg &c, Env &e, const StepScratch &s, int t, int lane) {
    const int A = c.A, P = c.P, K = c.K, n = A * K;
    uint32_t *bb_key = s.book, *bb_slot = s.book + A, *ba_key = s.book + 2 * A, *ba_slot = s.book + 3 * A;
    for (int cc = 0; cc < 2; cc++) {
        uint32_t *slots = e.orders + cc * n;
        // one pass over the book: lane-per-agent scan of its K slots
        for (int a = lane; a < A; a += NL) {
            uint32_t bk = 0, bs = 0, ak = 0, as = 0;
#if AIE_ON_DEVICE
            AIE_UNROLL(BIG ? 10 : 1)
#endif
            for (int k = 0; k < K; k++) {
                const uint32_t o = slots[a * K + k];
                if (o == ORDER_EMPTY) continue;
                if (order_side(o) == 0) { const uint32_t key = bid_key(t, o, a); if (key > bk) { bk = key; bs = (uint32_t)(a * K + k); } }
                else { const uint32_t key = ask_key(t, P, o, a); if (key > ak) { ak = key; as = (uint32_t)(a * K + k); } }
            }
            bb_key[a] = bk; bb_slot[a] = bs; ba_key[a] = ak; ba_slot[a] = as;
        }
        wsync();
        uint64_t possible = (A >= 64) ? ~0ull : ((1ull << A) - 1ull);
        for (;;) {
            // first bid whose buyer is still possible
            uint32_t bk = 0;
            for (int a = lane; a < A; a += NL)
                if (((possible >> a) & 1ull) && bb_key[a] > bk) bk = bb_key[a];
            const uint32_t bmax = wmax(bk);
            if (bmax == 0) break;  // idx_bid ran off the list: keep_checking = False
            const int buyer = 255 - (int)(bmax & 255u);
            const int bprice = (int)(bmax >> 20) - 1;
            const int blife = (int)((bmax >> 8) & 4095u);
            // first ask whose seller is not the buyer
            uint32_t ak = 0, ak_any = 0;
            for (int a = lane; a < A; a += NL) {
                if (ba_key[a] > ak_any) ak_any = ba_key[a];
                if (a != buyer && ba_key[a] > ak) ak = ba_key[a];
            }
            // Shortcut with the same outcome as marking the remaining buyers impossible one by one: the best remaining
            // bid is below the cheapest ask of the whole book (or there is no ask at all), so no remaining buyer can trade.
            const uint32_t amax_any = wmax(ak_any);
            if (amax_any == 0 || bprice < P - (int)(amax_any >> 20)) break;
            const uint32_t amax = wmax(ak);
            if (amax == 0) { possible &= ~(1ull << buyer); if (!possible) break; continue; }
            const int seller = 255 - (int)(amax & 255u);
            const int aprice = P - (int)(amax >> 20);
            const int alife = (int)((amax >> 8) & 4095u);
            if (bprice < aprice) { possible &= ~(1ull << buyer); if (!possible) break; continue; }
            // trade: price of whichever order came first (:297-304)
            const int price = (blife <= alife) ? aprice : bprice;
            const uint32_t bi = bb_slot[buyer], ai = ba_slot[seller];
            wsync();  // all lanes have read the bests lane 0 is about to invalidate
            if (lane == 0) {
                slots[bi] = ORDER_EMPTY;
                slots[ai] = ORDER_EMPTY;
                e.bid_hist[(cc * A + buyer) * P + bprice] -= 1;
                e.ask_hist[(cc * A + seller) * P + aprice] -= 1;
                e.n_orders[cc * A + seller] -= 1;
                e.n_orders[cc * A + buyer] -= 1;
                e.price_hist[(cc * A + seller) * P + price] += 1.0;
                e.esc[2 * seller + cc] -= 1;
                e.inv[2 * buyer + cc] += 1;
                e.esc_coin[buyer] -= (double)bprice;
                e.coin[seller] += (double)price;
                e.coin[buyer] += (double)(bprice - price);
                e.stats[ST_N_TRADES] += 1.0;
                double *ts = e.stats + c.st_trade + ((seller * 2 + cc) * 2 + 0) * 2;
                double *tb = e.stats + c.st_trade + ((buyer * 2 + cc) * 2 + 1) * 2;
                ts[0] += 1.0; ts[1] += (double)price; tb[0] += 1.0; tb[1] += (double)price;
                emit_event(e, EV_TRADE, seller, buyer, cc, aprice, bprice, alife, blife);
            }
            wsync();
            refresh_best(c, slots, buyer, 0, t, bb_key, bb_slot, lane);
            refresh_best(c, slots, seller, 1, t, ba_key, ba_slot, lane);
            wsync();
        }
        wsync();
    }
}

// remove_expired_orders :352-406.  lifetime after the increment is t - birth + 1; expired iff > D.
template <bool BIG>
AIE_DEV void cda_expire(const DevCfg &c, Env &e, int t, int lane) {
    const int A = c.A, P = c.P, K = c.K;
    for (int a = lane; a < A; a += NL) {
        for (int cc = 0; cc < 2; cc++) {
            uint32_t *slots = e.orders + (cc * A + a) * K;
            // an agent creates at most one bid and one ask per commodity per step, so at most one of each
            // expires here; they touch different state (coin vs. the commodity), so one pass is order-safe
#if AIE_ON_DEVICE
            AIE_UNROLL(BIG ? 10 : 1)
#endif
            for (int k = 0; k < K; k++) {
                uint32_t o = slots[k];
                if (o == ORDER_EMPTY || t - order_birth(o) < c.D) continue;
                int price = order_price(o);
                if (order_side(o) == 0) {
                    e.esc_coin[a] -= (double)price;
                    e.coin[a] += (double)price;
                    e.bid_hist[(cc * A + a) * P + price] -= 1;
                } else {
                    e.esc[2 * a + cc] -= 1;
                    e.inv[2 * a + cc] += 1;
                    e.ask_hist[(cc * A + a) * P + price] -= 1;
                }
                e.n_orders[cc * A + a] -= 1;
                slots[k] = ORDER_EMPTY;
            }
        }
    }
    wsync();
}

// ------------------------------------------------------------------------------------------------
// Gather  (components/move.py:93-153; world.py:150-173, 284-288, 424-460, 481-483)
// ------------------------------------------------------------------------------------------------
AIE_DEV void gather_step(const DevCfg &c, Env &e, const StepScratch &s, Rng &r) {
    const int A = c.A, W = c.W, H = c.H, lane = r.lane;
    rng_permutation(r, s.perm, A);
    for (int i = 0; i < A; i++) {
        int a = s.perm[i], action = s.act_move[a];
        int row = e.loc[2 * a], col = e.loc[2 * a + 1], nr = row, nc = col;
        if (action != 0) {
            int tr = row + (action == 3 ? -1 : (action == 4 ? 1 : 0));
            int tc = col + (action == 1 ? -1 : (action == 2 ? 1 : 0));
            bool ok = tr >= 0 && tr < H && tc >= 0 && tc < W;
            if (ok) {
                int k = tr * W + tc;
                uint8_t cb = e.cell[k];
                int8_t ow = e.owner[k];
                ok = !(cb & CELL_WATER) && (ow < 0 || ow == a);  // Maps.accessibility
            }
            bool occ = false;  // Maps.unoccupied: is any agent standing on the target cell?
            if (ok)
                for (int a2 = lane; a2 < A; a2 += NL) occ |= (e.loc[2 * a2] == tr && e.loc[2 * a2 + 1] == tc);
            occ = wany(occ);
            if (ok && !occ) {
                nr = tr; nc = tc;
                wsync();
                if (lane == 0) {
                    e.loc[2 * a] = (int16_t)nr; e.loc[2 * a + 1] = (int16_t)nc;
                    e.labor[a] += c.move_labor;
                }
            }
        }
        // harvest at the (possibly unchanged) location — also on NO-OP.  Resource order Stone, Wood.
        int k = nr * W + nc;
        uint8_t cb = e.cell[k];
        for (int cc = 0; cc < 2; cc++) {
            if (cb & (1u << cc)) {
                double u = rng_double(r);  // drawn even when bonus_gather_prob == 0
                int n_gathered = 1 + (u < e.bonus[a] ? 1 : 0);
                wsync();
                if (lane == 0) {
                    e.inv[2 * a + cc] += n_gathered;
                    e.cell[k] = (uint8_t)(e.cell[k] & ~(1u << cc));
                    e.labor[a] += c.collect_labor;
                    emit_event(e, EV_GATHER, a, cc, n_gathered, nr, nc);
                }
            }
        }
        wsync();
    }
}

// ------------------------------------------------------------------------------------------------
// PeriodicBracketTax  (components/redistribution.py)
// ------------------------------------------------------------------------------------------------
// curr_rate_max (:390-394): rate_max, or under a tax_annealing_schedule (fixed schedules and the Saez model; behind EXT) the
// annealed maximum of this episode (components/utils.py:10-57, refreshed whenever the completion count changes).
// Quirk kept: the limit is refreshed in generate_masks, which runs AFTER the observations of a reset are built
// (base_env.py:614-704), so the reset observation (t == 0) still shows the previous episode's limit.
template <bool EXT = false>
AIE_DEV double tax_rate_cap(const DevCfg &c, const Env &e) {
    if (EXT && c.tax_annealing && c.tax_model != 0) {
        int done_eps = e.hdr[HDR_COMPLETIONS];
        if (e.hdr[HDR_T] == 0 && done_eps > 0) done_eps -= 1;
        const double vis = fmax(0.0, fmin(1.0, c.ann_slope * ((double)done_eps - c.ann_warm)));
        return vis * c.rate_max;
    }
    return c.rate_max;
}
template <bool EXT = false>
AIE_DEV double tax_rate(const DevCfg &c, const Env &e, int b) {  // curr_marginal_rates :381-405
    if (c.tax_model == 2) return fmin(e.saez[b], tax_rate_cap<EXT>(c, e));  // Saez: np.minimum(curr_bracket_tax_rates, curr_rate_max)
    if (EXT && c.tax_model == 1 && c.tax_annealing) return fmin(c.fixed_rates[b], tax_rate_cap<EXT>(c, e));  // np.minimum(schedule, curr_rate_max)
    return c.tax_model == 0 ? c.disc_rates[e.rate_idx[b]] : c.fixed_rates[b];
}
template <bool EXT = false>
AIE_DEV double tax_rate_observed(const DevCfg &c, const Env &e, int b) {  // _curr_rates_obs (:960, :1123)
    return c.tax_model == 2 ? fmin(e.saez[32 + b], tax_rate_cap<EXT>(c, e)) : tax_rate<EXT>(c, e, b);
}
AIE_DEV int tax_income_bin(const DevCfg &c, double income) {  // :828-835 (bracket index; negative income -> 0)
    int arg = 0;
    for (int b = c.B - 1; b >= 0; b--) {
        double hi = (b + 1 < c.B) ? c.cutoffs[b + 1] : INFINITY;
        if (income >= c.cutoffs[b] && income < hi) arg = b;
    }
    return arg;
}
template <bool EXT = false>
AIE_DEV double tax_marginal_rate(const DevCfg &c, const Env &e, double income) {  // :837-844
    if (income < 0) return 0.0;
    return tax_rate<EXT>(c, e, tax_income_bin(c, income));
}
template <bool EXT = false>
AIE_DEV double tax_due(const DevCfg &c, const Env &e, double income) {  // :846-851
    double sum = 0.0;
    for (int b = 0; b < c.B; b++) {
        double size = ((b + 1 < c.B) ? c.cutoffs[b + 1] : INFINITY) - c.cutoffs[b];
        double past = fmax(0.0, income - c.cutoffs[b]);
        sum += tax_rate<EXT>(c, e, b) * fmin(size, past);
    }
    return sum;
}

template <bool EXT = false>
AIE_DEV void tax_step(const DevCfg &c, Env &e, const StepScratch &s, Rng &r, int lane) {  // :945-972
    const int A = c.A;
    int pos = e.hdr[HDR_TAX_POS];
    if (pos == 1 && c.tax_model == 2 && e.hdr[HDR_SAEZ_N] < 500) {
        // Saez warm-up (:444-457): until 500 (income, rate) samples exist the period's rates are
        // np.random.uniform(rate_min, curr_rate_max, n_brackets) from the env's stream; afterwards the host estimator has
        // already written this period's rates into the record.
        const double cap = tax_rate_cap<EXT>(c, e);
        for (int b = 0; b < c.B; b++) {
            const double u = rng_double(r);
            if (lane == 0) e.saez[b] = c.rate_min + (cap - c.rate_min) * u;
        }
        wsync();
    }
    if (pos == 1 && c.tax_model == 2) {  // _curr_rates_obs = curr_marginal_rates (:960): this period's rates
        for (int b = lane; b < 16; b += NL) e.saez[32 + b] = e.saez[b];
        wsync();
    }
    if (pos == 1 && c.tax_model == 0 && !c.disable_taxes) {  // set_new_period_rates_model :419-434
        for (int b = lane; b < c.B; b += NL) {
            int act = s.act_tax[b];
            if (act != 0) e.rate_idx[b] = (uint8_t)(act - 1);
        }
        wsync();
    }
    if (pos >= c.period) {  // enact_taxes :853-915
        for (int a = lane; a < A; a += NL) {
            double income = (e.coin[a] + e.esc_coin[a]) - e.last_coin[a];
            double due = tax_due<EXT>(c, e, income);
            double paid = fmin(e.coin[a], due);  // never touches escrow
            e.last_marg[a] = tax_marginal_rate<EXT>(c, e, income);
            e.last_income[a] = income;
            e.coin[a] -= paid;
            s.tmp[a] = paid;
            s.tmp[A + a] = paid / fmax(0.000001, income);  // effective rate (:880)
            double *ta = e.stats + c.st_tax + ST_TAX_AGENT;
            ta[a] += fmax(0.0, income); ta[A + a] += paid;
        }
        wsync();
        double net = 0.0;
        for (int a = 0; a < A; a++) net += s.tmp[a];  // sequential, agent order (uniform)
        if (lane == 0) {  // episode statistics (:862-897): schedule, occupancy, effective rates, revenue
            double *st = e.stats + c.st_tax;
            st[ST_TAX_PERIODS] += 1.0;
            if (c.tax_model == 2 && e.hdr[HDR_SAEZ_N] < (1 << 30)) e.hdr[HDR_SAEZ_N] += A;  // _update_saez_buffer :535-544
            st[ST_TAX_COLLECTED] += net;
            for (int b = 0; b < c.B; b++) st[ST_TAX_SCHED + b] += tax_rate<EXT>(c, e, b);
            for (int a = 0; a < A; a++) {
                st[ST_TAX_EFF_SUM] += s.tmp[A + a];
                st[ST_TAX_OCC + tax_income_bin(c, e.last_income[a])] += 1.0;
            }
        }
        double lump = net / A;
        for (int a = lane; a < A; a += NL) {
            e.coin[a] += lump;
            e.last_coin[a] = e.coin[a] + e.esc_coin[a];
        }
        pos = 0;
    }
    pos += 1;
    wsync();
    if (lane == 0) e.hdr[HDR_TAX_POS] = pos;
    wsync();
}

// ------------------------------------------------------------------------------------------------
// Resource regeneration (layout_from_file.py:372-410): for resource in [Wood, Stone], one uniform per cell
// in row-major order; an empty source cell respawns iff u < regen_weight.  The whole 2*H*W-word run of the
// stream is consumed; only empty source cells temper/compare their two words.
// ------------------------------------------------------------------------------------------------
// regen_halfwidth > 0 (dynamic_layout.py:446-461): the respawn probability of source cell k is the box-filtered
// source map (health = max(resource, source) = source for max_health 1), i.e. a function of the number of source
// cells in its d x d window.  Cold: only evaluated for empty source cells of configs that set a halfwidth.
AIE_DEV_NOINLINE uint64_t regen_window_thresh(const DevCfg &c, const Env &e, int cc, int k) {
    const int hw = c.regen_hw[cc], r0 = k / c.W, c0 = k - r0 * c.W;
    const uint8_t src_bit = (uint8_t)(4u << cc);
    int n = 0;
    for (int r = r0 - hw; r <= r0 + hw; r++) {
        if (r < 0 || r >= c.H) continue;
        for (int q = c0 - hw; q <= c0 + hw; q++)
            if (q >= 0 && q < c.W && (e.cell[r * c.W + q] & src_bit)) n++;
    }
    return c.regen_tab[cc][n];
}

template <bool EXT>
AIE_DEV void regen_resource(const DevCfg &c, Env &e, int cc, Rng &r) {
    const int HW = c.HW, lane = r.lane;
    const uint8_t res_bit = (uint8_t)(1u << cc), src_bit = (uint8_t)(4u << cc);
    const uint64_t thresh = c.regen_thresh[cc];
    int w = 0;                 // words of this run consumed so far (warp-uniform)
    const int total = 2 * HW;
    uint32_t pend_a = 0;       // first word of a cell that straddles a key regeneration
    while (w < total) {
        if (r.pos == 624) { mt_twist(r.mt, lane); r.pos = 0; }
        int n = 624 - r.pos;
        if (n > total - w) n = total - w;
        int w_end = w + n;
        const int base = r.pos - w;  // key index of run word j is base + j
        if (w & 1) {                 // finish the straddling cell with its second word
            int k = w >> 1;
            if (lane == 0) {
                uint8_t cb = e.cell[k];
                if ((cb & src_bit) && !(cb & res_bit)) {
                    uint64_t v = ((uint64_t)(pend_a >> 5) << 26) | (uint64_t)(mt_temper(e.mt[base + w]) >> 6);
                    if (v < ((EXT && c.regen_hw[cc]) ? regen_window_thresh(c, e, cc, k) : thresh)) e.cell[k] = cb | res_bit;
                }
            }
        }
        wsync();  // lane 0's straddle fix-up is visible before the group loads below touch the same word
        int k_lo = (w + 1) >> 1, k_hi = w_end >> 1;  // cells with both words inside this segment
        // 4 cells per lane per iteration: one 32-bit load finds the (rare) empty source cells of a group
        const uint32_t *cell32 = (const uint32_t *)e.cell;
        for (int g = (k_lo >> 2) + lane; 4 * g < k_hi; g += NL) {
            const uint32_t wv = cell32[g];
            uint32_t cand = ((wv >> (2 + cc)) & ~(wv >> cc)) & 0x01010101u;  // byte LSB: source set, resource clear
            while (cand) {
#if AIE_ON_DEVICE
                const int j = (__ffs(cand) - 1) >> 3;
#else
                const int j = (__builtin_ffs(cand) - 1) >> 3;
#endif
                cand &= cand - 1;
                const int k = 4 * g + j;
                if (k < k_lo || k >= k_hi) continue;
                uint64_t v = ((uint64_t)(mt_temper(e.mt[base + 2 * k]) >> 5) << 26) |
                             (uint64_t)(mt_temper(e.mt[base + 2 * k + 1]) >> 6);
                if (v < ((EXT && c.regen_hw[cc]) ? regen_window_thresh(c, e, cc, k) : thresh)) e.cell[k] = (uint8_t)(e.cell[k] | res_bit);
            }
        }
        if (w_end & 1) pend_a = mt_temper(e.mt[base + w_end - 1]);
        wsync();
        r.pos += n;
        w = w_end;
    }
}

// ------------------------------------------------------------------------------------------------
// Utilities / rewards (layout_from_file.py:249-318, 519-559; rewards.py:12-48, 84-133;
// social_metrics.py:10-46)
// ------------------------------------------------------------------------------------------------
AIE_DEV double energy_weight(const DevCfg &c, const Env &e) {
    if (c.warm_const <= 0.0) return 1.0;
    double n = c.warm_auto ? (double)e.hdr[HDR_AUTO_WARMUP] : (double)e.hdr[HDR_COMPLETIONS];
    return 1.0 - exp(-n / c.warm_const);
}

// Gini coefficient of the endowments x_a = coin[a] + esc_coin[a], sort-based branch (A >= 30): rank each endowment,
// scatter to sorted order (tmp[A]), then cumulative sums.  Warp-collective.  Inlined: large populations (c5) take it
// every step.
AIE_DEV double gini_sorted(const double *coin, const double *esc_coin, double *tmp, int A, int lane) {
    for (int i = lane; i < A; i += NL) {
        double xi = coin[i] + esc_coin[i];
        int rank = 0;
        for (int j = 0; j < A; j++) {
            double xj = coin[j] + esc_coin[j];
            rank += (xj < xi || (xj == xi && j < i)) ? 1 : 0;
        }
        tmp[rank] = xi;
    }
    wsync();
    double tot = 0.0, cum = 0.0, acc = 0.0;
    for (int i = 0; i < A; i++) tot += tmp[i];
    for (int i = 0; i < A; i++) { cum += tmp[i]; acc += cum / (tot + 1e-10); }
    return 1.0 - (2.0 / (A + 1)) * acc;
}
// inv_income_weighted_coin_endowments (swf 1) / inv_income_weighted_utility (swf 2): weights 1 / max(x_a, 1), normalised.
// Out of line: the benchmarked configurations use the default welfare function (coin_eq_times_productivity).
AIE_DEV_NOINLINE double inv_income_weighted(const double *coin, const double *esc_coin, const double *util, int A, int swf) {
    double wsum_ = 0.0, acc = 0.0;
    for (int a = 0; a < A; a++) wsum_ += 1.0 / fmax(coin[a] + esc_coin[a], 1.0);
    for (int a = 0; a < A; a++) {
        double x = coin[a] + esc_coin[a];
        double wgt = (1.0 / fmax(x, 1.0)) / wsum_;
        acc += (swf == 1 ? x : util[a]) * wgt;
    }
    return acc;
}

// Writes util[0..A] (agents, then planner) into `out` (scratch or record).  Warp-collective.
AIE_DEV void current_metrics(const DevCfg &c, const Env &e, double *out, double *tmp, int lane) {
    const int A = c.A;
    const double coef = energy_weight(c, e) * c.energy_cost;
    for (int a = lane; a < A; a += NL) {
        double x = e.coin[a] + e.esc_coin[a];
        // eta == 0: x ** 1.0 is x exactly in IEEE arithmetic (numpy / libm); the device pow() is not guaranteed to return
        // it, and with energy_warmup_method "auto" a last-place difference can flip `mean reward > 0` when linear utilities
        // cancel exactly (found by the CUDA-vs-oracle configuration fuzz)
        double util_c = (c.eta == 1.0) ? log(fmax(1.0, x)) : ((c.eta == 0.0 ? x : pow(x, 1.0 - c.eta)) - 1.0) / (1.0 - c.eta);
        out[a] = util_c - e.labor[a] * coef;
    }
    wsync();
    double planner;
    if (c.swf == 0) {  // coin_eq_times_productivity
        double total = 0.0;
        for (int a = 0; a < A; a++) total += e.coin[a] + e.esc_coin[a];  // uniform, agent order
        double gini;
        if (A < 30) {
            double part = 0.0;
            for (int i = lane; i < A; i += NL) {
                double xi = e.coin[i] + e.esc_coin[i];
                for (int j = 0; j < A; j++) part += fabs(xi - (e.coin[j] + e.esc_coin[j]));
            }
            double diff = wsum(part);
            gini = (diff / (2 * A * total + 1e-10)) / ((A - 1) / (double)A);
        } else {
            gini = gini_sorted(e.coin, e.esc_coin, tmp, A, lane);
        }
        double eqw = 1.0 - c.mix;
        planner = (eqw * (1.0 - gini) + (1.0 - eqw)) * (total / A);
    } else {
        planner = inv_income_weighted(e.coin, e.esc_coin, out, A, c.swf);
    }
    wsync();
    if (lane == 0) out[A] = planner;
    wsync();
}

// numpy's pairwise_sum for n <= 128 (numpy/core/src/umath/loops_utils.h.src): plain loop below 8 elements,
// otherwise 8 interleaved accumulators combined as a tree plus a sequential tail.  Warp-uniform.
AIE_DEV double np_pairwise_sum(const double *a, int n) {
    if (n < 8) {
        double res = 0.0;
        for (int i = 0; i < n; i++) res += a[i];
        return res;
    }
    double r[8];
    for (int j = 0; j < 8; j++) r[j] = a[j];
    int i;
    for (i = 8; i < n - (n % 8); i += 8)
        for (int j = 0; j < 8; j++) r[j] += a[i + j];
    double res = ((r[0] + r[1]) + (r[2] + r[3])) + ((r[4] + r[5]) + (r[6] + r[7]));
    for (; i < n; i++) res += a[i];
    return res;
}

// ------------------------------------------------------------------------------------------------
// WealthRedistribution (components/redistribution.py:52-68): every step all agents end up with the same total coin;
// escrowed coin stays where it is, so inventory coin becomes (sum of inventory + escrow) / A - own escrow.
// ------------------------------------------------------------------------------------------------
AIE_DEV void wealth_step(const DevCfg &c, Env &e, const StepScratch &s, int lane) {
    const int A = c.A;
    for (int a = lane; a < A; a += NL) s.tmp[a] = e.coin[a] + e.esc_coin[a];
    wsync();
    const double target = np_pairwise_sum(s.tmp, A) / A;  // np.sum(ic + ec) / n_agents
    wsync();
    for (int a = lane; a < A; a += NL) e.coin[a] = target - e.esc_coin[a];
    wsync();
}

// ------------------------------------------------------------------------------------------------
// SimpleLabor (components/simple_labor.py:100-126): action h in 1..100 sets the agent's labor to h hours and pays
// h * skill into its coin and its cumulative production.  The random order only consumes the permutation draw.
// Record reuse: skill lives in the build_skill field, production in build_payment.
// ------------------------------------------------------------------------------------------------
AIE_DEV void labor_step(const DevCfg &c, Env &e, const StepScratch &s, Rng &r) {
    rng_permutation(r, s.perm, c.A);
    for (int a = r.lane; a < c.A; a += NL) {
        const int h = s.act_move[a];
        if (h >= 1 && h <= 100) {
            const double payoff = h * e.bskill[a];
            e.labor[a] = (double)h;
            e.bpay[a] += payoff;
            e.coin[a] += payoff;
        }
    }
    wsync();
}

// one-step-economy utilities (one_step_economy.py:264-336; rewards.py:12-70, 84-133): agents coin minus a labor cost,
// planner a social welfare function over them (weights from the pre-tax incomes = production)
AIE_DEV void one_step_metrics(const DevCfg &c, const Env &e, double *out, double *tmp, int lane) {
    const int A = c.A;
    // coin_eq_times_productivity only looks at the coin endowments: take the planner's value from the family's own routine
    // (both Gini forms), then replace the agents' utilities
    double planner = 0.0;
    if (c.swf == 0) { current_metrics(c, e, out, tmp, lane); planner = out[A]; wsync(); }
    for (int a = lane; a < A; a += NL) {
        const double x = e.coin[a] + e.esc_coin[a], l = e.labor[a];
        double u;
        if (c.agent_reward_type == 1) {   // coin_minus_labor_cost: x - l ** exponent * coefficient
            const double lp = c.labor_exponent == 2.0 ? l * l : pow(l, c.labor_exponent);
            u = x - lp * c.labor_cost;
        } else {                          // isoelastic_coin_minus_labor (no energy warm-up here)
            const double uc = (c.eta == 1.0) ? log(fmax(1.0, x)) : ((c.eta == 0.0 ? x : pow(x, 1.0 - c.eta)) - 1.0) / (1.0 - c.eta);
            u = uc - l * c.labor_cost;
        }
        out[a] = u;
    }
    wsync();
    if (c.swf != 0) {   // inv_income_weighted_utility(coin_endowments = pretax incomes, utilities)
        double wsum_ = 0.0, acc = 0.0;
        for (int a = 0; a < A; a++) wsum_ += 1.0 / fmax(e.bpay[a], 1.0);
        for (int a = 0; a < A; a++) acc += out[a] * ((1.0 / fmax(e.bpay[a], 1.0)) / wsum_);
        planner = acc;
    }
    wsync();
    if (lane == 0) out[A] = planner;
    wsync();
}

template <bool EXT = false>
AIE_DEV void compute_reward(const DevCfg &c, Env &e, const StepScratch &s, double *rew_out, int lane) {
    const int A = c.A;
    double *cur = s.tmp;  // [A+1] new metrics; the second half of tmp is sort / staging scratch
    if (EXT && c.one_step) one_step_metrics(c, e, cur, cur + (A + 2), lane);
    else current_metrics(c, e, cur, cur + (A + 2), lane);
    double *rw_s = cur + (A + 2);  // rewards staged so the mean can be formed in numpy's summation order
    for (int a = lane; a <= A; a += NL) {
        double rw = cur[a] - e.util_prev[a];
        if (rew_out) rew_out[a] = rw;
        rw_s[a] = rw;
    }
    wsync();
    const double avg = np_pairwise_sum(rw_s, A) / A;  // np.mean([...]) (layout_from_file.py:552)
    for (int a = lane; a <= A; a += NL) e.util_prev[a] = cur[a];
    if (lane == 0 && avg > 0) e.hdr[HDR_AUTO_WARMUP] += 1;
    wsync();
}

// ------------------------------------------------------------------------------------------------
// One env.step() (base/base_env.py:929-1032) without the observation pass.  CS: the component kinds compiled in
// (a superset of the config's, see step_comp_set).
// ------------------------------------------------------------------------------------------------
template <bool BIG, bool EXT = false, int CS = CS_ALL>
AIE_DEV void step_env(const DevCfg &c, uint8_t *rec, uint8_t *grec, uint8_t *scratch, const int32_t *act_a,
                      const int32_t *act_p, double *rew_out, int32_t *done_out, int lane, bool decoded = false,
                      int32_t *events = nullptr, int event_cap = 0, const uint16_t *tab = nullptr) {
    Env e = env_view(rec, grec, c);
    StepScratch s = step_scratch_view(scratch, c);
    if (events) {  // dense-log replicas: this step's event block starts empty
        e.ev = events; e.ev_cap = event_cap;
        if (lane == 0) { events[0] = 0; events[1] = e.hdr[HDR_T] + 1; events[2] = 0; }
    }
    if (!decoded) decode_actions<EXT>(c, s, act_a, act_p, lane, tab);  // the CUDA kernel decodes while the record is in flight
    Rng r; r.mt = e.mt; r.pos = e.hdr[HDR_MT_POS]; r.lane = lane;
    const int t = e.hdr[HDR_T] + 1;
    wsync();
    if (lane == 0) e.hdr[HDR_T] = t;
    for (int i = 0; i < c.n_comp; i++) {
        lane = relane(lane); r.lane = lane;
        switch (c.comp[i]) {
            case COMP_BUILD: if (CS & (1 << COMP_BUILD)) build_step(c, e, s, r); break;
            case COMP_CDA:
                if (CS & (1 << COMP_CDA)) { cda_create<BIG>(c, e, s, t, lane); cda_match<BIG>(c, e, s, t, lane); cda_expire<BIG>(c, e, t, lane); }
                break;
            case COMP_GATHER: if (CS & (1 << COMP_GATHER)) gather_step(c, e, s, r); break;
            case COMP_TAX: if (CS & (1 << COMP_TAX)) tax_step<EXT>(c, e, s, r, lane); break;
            case COMP_WEALTH: if (CS & (1 << COMP_WEALTH)) wealth_step(c, e, s, lane); break;
            case COMP_LABOR: if (EXT && (CS & (1 << COMP_LABOR))) labor_step(c, e, s, r); break;
        }
    }
#if AIE_ON_DEVICE
#pragma unroll 1
#endif
    for (int ri = 0; ri < 2; ri++) {  // Wood, then Stone (one inlined copy); the one-step-economy has no map: scenario_step() is empty
        lane = relane(lane); r.lane = lane;
        if (!(EXT && c.one_step)) regen_resource<EXT>(c, e, 1 - ri, r);
    }
    lane = relane(lane);
    compute_reward<EXT>(c, e, s, rew_out, lane);
    lane = relane(lane);
    if (lane == 0) {
        e.hdr[HDR_MT_POS] = r.pos;
        if (done_out) *done_out = (t >= c.T) ? 1 : 0;
    }
    wsync();
}

// Finish a host reset on the device: tax trackers + metric_0 (redistribution.py:1106-1139,
// layout_from_file.py:588-593).  The host packer has already zeroed books, escrow, labor.
// Reset-only code is kept out of line: inlined it would triple the step kernel's code for a once-per-episode path.
AIE_DEV_NOINLINE void finish_reset_env(const DevCfg &c, uint8_t *rec, uint8_t *grec, uint8_t *scratch, int lane) {
    Env e = env_view(rec, grec, c);
    StepScratch s = step_scratch_view(scratch, c);
    for (int a = lane; a < c.A; a += NL) {
        e.last_coin[a] = e.coin[a] + e.esc_coin[a];
        e.last_income[a] = 0.0;
        e.last_marg[a] = 0.0;
    }
    // Saez: the reference caches the rate observation BEFORE it resets curr_bracket_tax_rates to the running average
    // (:1123 vs :1138-1139): the reset observation's curr_rates are the previous episode's last rates while the agents'
    // marginal_rate observation already uses the running average.
    if (c.has[COMP_TAX] && c.tax_model == 2)
        for (int b = lane; b < 16; b += NL) { e.saez[32 + b] = e.saez[b]; e.saez[b] = e.saez[16 + b]; }
    wsync();
    if (c.one_step) one_step_metrics(c, e, e.util_prev, s.tmp, lane);
    else current_metrics(c, e, e.util_prev, s.tmp, lane);
    wsync();
}

// Device-side reset draws with reference semantics (reset_mode == 1; layout_from_file scenarios).  The maps,
// inventories, books and trackers have already been restored from the load-time snapshot; this re-draws, from the
// env's own numpy stream and in the reference's order, the random placement (layout_from_file.py:336-370),
// the component skills (build.py:224-254, move.py:193-210) and the fixed_four assignment (:580-586).
AIE_DEV double rng_pareto(Rng &r, double a) {  // numpy legacy_pareto: exp(-log(1 - U) / a) - 1
    const double e = -log(1.0 - rng_double(r));
    return exp(e / a) - 1.0;
}
// numpy's legacy_gauss (legacy-distributions.c): polar Box-Muller; the second variate of a pair is cached in the stream
// state (here: the record's gauss section) and returned by the next call - across components, resets and episodes.
AIE_DEV double rng_gauss(Rng &r, double *g) {   // warp-uniform call
    if (g[1] != 0.0) {
        const double cached = g[0];
        wsync();
        if (r.lane == 0) { g[0] = 0.0; g[1] = 0.0; }
        wsync();
        return cached;
    }
    double x1, x2, r2;
    do {
        x1 = 2.0 * rng_double(r) - 1.0;
        x2 = 2.0 * rng_double(r) - 1.0;
        r2 = x1 * x1 + x2 * x2;
    } while (r2 >= 1.0 || r2 == 0.0);
    const double f = sqrt(-2.0 * log(r2) / r2);
    wsync();
    if (r.lane == 0) { g[0] = f * x1; g[1] = 1.0; }
    wsync();
    return f * x2;
}
AIE_DEV double rng_lognormal(Rng &r, double *g, double mean, double sigma) { return exp(mean + sigma * rng_gauss(r, g)); }


// ------------------------------------------------------------------------------------------------
// Dynamic layouts at reset (aie_config::dyn_layout): Uniform.reset_starting_layout, dynamic_layout.py:313-392
// ------------------------------------------------------------------------------------------------
// n uniform doubles (np.random.rand: random_sample) into out[0 .. n), drawn lane-parallel: double i is key words 2i, 2i + 1
// of the run.  A double straddling a key regeneration is finished by the sequential path.
AIE_DEV void rng_fill_double(Rng &r, double *out, int n) {
    int i = 0;
    while (i < n) {
        if (r.pos == 624) { mt_twist(r.mt, r.lane); r.pos = 0; }
        const int avail = (624 - r.pos) >> 1;
        if (avail == 0) {
            const double v = rng_double(r);
            if (r.lane == 0) out[i] = v;
            i++;
            continue;
        }
        const int m = avail < n - i ? avail : n - i;
        for (int j = r.lane; j < m; j += NL) {
            const int32_t a = (int32_t)(mt_temper(r.mt[r.pos + 2 * j]) >> 5), b = (int32_t)(mt_temper(r.mt[r.pos + 2 * j + 1]) >> 6);
            out[i + j] = (a * 67108864.0 + b) / 9007199254740992.0;
        }
        wsync();
        r.pos += 2 * m; i += m;
    }
}
AIE_DEV int kth_set_bit(uint32_t m, int k) {   // position of the k-th (1-based) set bit of m
#if AIE_ON_DEVICE
    return (int)__fns(m, 0, k);
#else
    for (int i = 0; i < 32; i++) if ((m >> i) & 1u) { if (--k == 0) return i; }
    return -1;
#endif
}
// n standard normals (np.random.randn: legacy_gauss) into out[0 .. n).  The polar method draws trial pairs of uniforms
// until one falls inside the unit circle and then yields TWO normals - f * x2 at once, f * x1 cached for the next call.
// Every trial consumes exactly four key words whether it is accepted or not, so trials are evaluated lane-parallel and
// the accepted ones numbered by a ballot; the stream stops right after the trial that supplies the last normal needed.
// g: the cache {value, has} in the record (shared with every other Gaussian draw of the env).
AIE_DEV void rng_fill_gauss(Rng &r, double *g, double *out, int n) {
    const int lane = r.lane;
    int i = 0;
    const bool has_cached = n > 0 && g[1] != 0.0;
    const double cached = g[0];
    wsync();   // every lane has read the cache before any lane (this call's last accepted trial) refills it
    if (has_cached) {
        if (lane == 0) { out[0] = cached; g[0] = 0.0; g[1] = 0.0; }
        wsync();
        i = 1;
    }
    while (i < n) {
        const int need = (n - i + 1) >> 1;   // accepted pairs still needed
        if (r.pos == 624) { mt_twist(r.mt, lane); r.pos = 0; }
        const int avail = (624 - r.pos) >> 2;
        if (avail == 0) {   // a trial straddling a key regeneration: sequential
            const double x1 = 2.0 * rng_double(r) - 1.0, x2 = 2.0 * rng_double(r) - 1.0, r2 = x1 * x1 + x2 * x2;
            if (!(r2 >= 1.0 || r2 == 0.0)) {
                const double f = sqrt(-2.0 * log(r2) / r2);
                wsync();
                if (lane == 0) {
                    out[i] = f * x2;
                    if (i + 1 < n) out[i + 1] = f * x1; else { g[0] = f * x1; g[1] = 1.0; }
                }
                wsync();
                i += 2;
            }
            continue;
        }
        const int nb = avail < NL ? avail : NL;
        bool acc = false;
        double x1 = 0.0, x2 = 0.0, r2 = 1.0;
        if (lane < nb) {
            const uint32_t *w = r.mt + r.pos + 4 * lane;
            const int32_t a1 = (int32_t)(mt_temper(w[0]) >> 5), b1 = (int32_t)(mt_temper(w[1]) >> 6);
            const int32_t a2 = (int32_t)(mt_temper(w[2]) >> 5), b2 = (int32_t)(mt_temper(w[3]) >> 6);
            x1 = 2.0 * ((a1 * 67108864.0 + b1) / 9007199254740992.0) - 1.0;
            x2 = 2.0 * ((a2 * 67108864.0 + b2) / 9007199254740992.0) - 1.0;
            r2 = x1 * x1 + x2 * x2;
            acc = !(r2 >= 1.0 || r2 == 0.0);
        }
        const uint32_t m = wballot(acc);
        const int cnt = __popc_u32(m);
        int use_pairs = cnt, used_trials = nb;
        if (cnt >= need) { use_pairs = need; used_trials = kth_set_bit(m, need) + 1; }
        if (acc) {
            const int rank = __popc_u32(m & ((1u << lane) - 1u));
            if (rank < use_pairs) {
                const double f = sqrt(-2.0 * log(r2) / r2);
                const int idx = i + 2 * rank;
                out[idx] = f * x2;
                if (idx + 1 < n) out[idx + 1] = f * x1; else { g[0] = f * x1; g[1] = 1.0; }
            }
        }
        wsync();
        r.pos += 4 * used_trials; i += 2 * use_pairs;
    }
}

// One output of scipy.signal.convolve2d(x, kernel, "same") for a 7 x 7 kernel of zeros and ones (bit j * 7 + k of
// `kern`): out[m, n] = sum_{j, k} x[m - j + 3, n - k + 3] * kernel[j, k], zero outside the map.  The float64 sum is
// accumulated in the order of scipy's C loop (verified bit for bit against scipy 1.18 on random inputs, see
// tests/test_dynamic_layout.py): kernel rows in ascending order; inside a row the first four taps as one expression
// ((t0 + t1) + t2) + t3 added to the accumulator, then taps 4, 5, 6 one by one.
AIE_DEV double conv7_same(const double *x, int H, int W, int m, int n, uint64_t kern) {
    double acc = 0.0;
    for (int j = 0; j < 7; j++) {
        const int rr = m - j + 3;
        double t[7];
        for (int k = 0; k < 7; k++) {
            const int cc = n - k + 3;
            const bool in = (unsigned)rr < (unsigned)H && (unsigned)cc < (unsigned)W && ((kern >> (j * 7 + k)) & 1ull);
            t[k] = in ? x[rr * W + cc] : 0.0;
        }
        acc += ((t[0] + t[1]) + t[2]) + t[3];
        acc += t[4]; acc += t[5]; acc += t[6];
    }
    return acc;
}

constexpr uint8_t CELL_CAND = 0x80;   // scratch bit of the cell byte while a layout is being generated

// Clumped random source placement.  prob: float64 [2][HW] (Wood, Stone); work: this env's float64 [HW] scratch map.
// Leaves the Wood / Stone resource and source bits of e.cell set; water and house bits are not touched.
AIE_DEV void gen_layout(const DevCfg &c, Env &e, Rng &r, const double *prob, double *work) {
    const int HW = c.HW, H = c.H, W = c.W, lane = r.lane;
    const uint8_t res_bits[2] = {(uint8_t)(CELL_WOOD | CELL_WOOD_SRC), (uint8_t)(CELL_STONE | CELL_STONE_SRC)};
    auto count_cand = [&]() {
        int n = 0;
        for (int k = lane; k < HW; k += NL) n += (e.cell[k] & CELL_CAND) ? 1 : 0;
        return (double)wsum((double)n) / (double)HW;   // np.mean of a boolean map
    };
    // MultiZone (dynamic_layout.py:778-872): np.random.shuffle of the region -> zone-type vector (Wood 0, Stone 1, WoodStone 2,
    // none 255), then probability (1 / share of the world inside the resource's zones) * Wood coverage inside them, 0 outside
    uint8_t *grid = reinterpret_cast<uint8_t *>(work + HW);
    double mz_val[2] = {0.0, 0.0};
    auto in_zone = [&](int ri, int k) {
        const int m = k / W, n = k - m * W;
        const uint8_t z = grid[(m / c.mz_psr) * c.mz_cols + (n / c.mz_psc)];
        return z == 2 || z == (uint8_t)ri;   // ri 0 = Wood, 1 = Stone
    };
    if (c.dyn_layout == 3) {
        const int nreg = c.mz_rows * c.mz_cols;
        if (lane == 0) {
            int at = 0;
            for (int z = 0; z < 3; z++) for (int q = 0; q < c.mz_zones[z]; q++) grid[at++] = (uint8_t)z;
            while (at < nreg) grid[at++] = 255;
        }
        wsync();
        for (int i = nreg - 1; i >= 1; i--) {   // legacy shuffle: swap x[i] with x[random_interval(i)]
            const int j = (int)rng_interval(r, (uint32_t)i);
            if (lane == 0) { const uint8_t t = grid[j]; grid[j] = grid[i]; grid[i] = t; }
            wsync();
        }
        for (int ri = 0; ri < 2; ri++) {
            int cnt = 0;
            for (int k = lane; k < HW; k += NL) cnt += in_zone(ri, k) ? 1 : 0;
            const double mean = wsum((double)cnt) / (double)HW;
            mz_val[ri] = (1.0 / mean) * c.dyn_cov[0];   // sic: both maps are scaled by the Wood coverage (:860-863)
        }
    }
    for (int attempt = 0; attempt < 100; attempt++) {
        for (int k = lane; k < HW; k += NL) e.cell[k] &= (uint8_t)~(res_bits[0] | res_bits[1] | CELL_CAND);   // maps.clear()
        wsync();
        double mean_res[2];
        for (int ri = 0; ri < 2; ri++) {   // Wood, then Stone on what Wood left empty
            const double clump = c.dyn_clump[ri], cover = c.dyn_cov[ri];
            const double *sp = prob + (size_t)ri * HW;
            auto threshold_pass = [&](bool decay) {
                for (int k = lane; k < HW; k += NL) {
                    double v = work[k];
                    if (decay) { v *= 0.9; work[k] = v; }
                    const uint8_t cb = e.cell[k];
                    const bool empty = !(cb & (res_bits[0] | res_bits[1]));
                    const double spk = c.dyn_layout == 3 ? (in_zone(ri, k) ? mz_val[ri] : 0.0) : sp[k];
                    e.cell[k] = (uint8_t)((cb & ~CELL_CAND) | ((v < spk * 0.1 * clump && empty) ? CELL_CAND : 0));
                }
                wsync();
            };
            rng_fill_double(r, work, HW);
            threshold_pass(false);
            double mean = count_cand();
            for (int tries = 0; mean < cover * clump;) {
                threshold_pass(true);
                mean = count_cand();
                if (++tries > 200) break;
            }
            for (int grow = 0; mean < cover && grow < 100000; grow++) {
                // kernel = np.random.randn(7, 7) > 0
                rng_fill_gauss(r, e.gauss, work, 49);
                wsync();
                uint64_t kern = 0;
                for (int q = 0; q < 49; q++) kern |= (uint64_t)(work[q] > 0.0 ? 1 : 0) << q;
                wsync();
                // x = candidate + 0.2 * np.random.randn(H, W) - 0.25
                rng_fill_gauss(r, e.gauss, work, HW);
                wsync();
                for (int k = lane; k < HW; k += NL) work[k] = (((e.cell[k] & CELL_CAND) ? 1.0 : 0.0) + 0.2 * work[k]) - 0.25;
                wsync();
                // candidate = max(convolve2d(x, kernel, "same") > 0, candidate) * empty
                for (int k = lane; k < HW; k += NL) {
                    const uint8_t cb = e.cell[k];
                    if (cb & (CELL_CAND | res_bits[0] | res_bits[1])) continue;   // already a candidate, or not empty
                    const int m = k / W, n = k - m * W;
                    if (conv7_same(work, H, W, m, n, kern) > 0.0) e.cell[k] = (uint8_t)(cb | CELL_CAND);
                }
                wsync();
                mean = count_cand();
            }
            mean_res[ri] = mean;
            for (int k = lane; k < HW; k += NL) {   // world.maps.set(resource, ...), set(resource + "SourceBlock", ...)
                const uint8_t cb = e.cell[k];
                if (cb & CELL_CAND) e.cell[k] = (uint8_t)((cb & ~CELL_CAND) | res_bits[ri]);
            }
            wsync();
        }
        bool happy = true;   // both coverages within 1.4x of their targets, else start over
        for (int ri = 0; ri < 2; ri++) {
            const double q = mean_res[ri] / c.dyn_cov[ri];
            if (!((1.0 / (1.0 + 0.4)) <= q && q <= (1.0 + 0.4))) happy = false;
        }
        if (happy) break;
    }
    if (c.dyn_checker || c.dyn_layout == 2) {
        const int col_line = H / 2, row_line = W / 2;   // Quadrant: state[:, height // 2] = 0; state[width // 2, :] = 0
        for (int k = lane; k < HW; k += NL) {
            const int m = k / W, n = k - m * W;
            const bool drop = (c.dyn_checker && ((m + n) & 1) == 0) || (c.dyn_layout == 2 && (n == col_line || m == row_line));
            if (drop) e.cell[k] &= (uint8_t)~(res_bits[0] | res_bits[1]);
        }
        wsync();
    }
}

template <bool EXT>
AIE_DEV void device_reset_draws(const DevCfg &c, Env &e, const StepScratch &s, Rng &r, const double *dyn_prob, double *dyn_work) {
    const int A = c.A, lane = r.lane;
    const bool dyn = c.dyn_layout != 0;   // (not behind EXT: the whole reset is one out-of-line call, cold code)
    if (dyn) {   // dynamic_layout.py:313-392, then reset_agent_states places the agents in a random order (:418-429)
        gen_layout(c, e, r, dyn_prob, dyn_work);
        rng_permutation(r, s.perm, A);
        for (int a = lane; a < A; a += NL) { e.loc[2 * a] = -1; e.loc[2 * a + 1] = -1; }
        wsync();
    }
    for (int i = 0; i < A; i++) {  // np.random.randint(0, H), randint(0, W) until the cell is free and not water
        const int a = dyn ? s.perm[i] : i;
        int row = 0, col = 0;
        for (int tries = 0; tries <= 201; tries++) {
            row = (int)rng_interval(r, (uint32_t)(c.H - 1));
            col = (int)rng_interval(r, (uint32_t)(c.W - 1));
            bool blocked = (e.cell[row * c.W + col] & CELL_WATER) != 0;
            if (dyn) { for (int a2 = 0; a2 < A && !blocked; a2++) blocked = e.loc[2 * a2] == row && e.loc[2 * a2 + 1] == col; }
            else { for (int a2 = 0; a2 < a && !blocked; a2++) blocked = e.loc[2 * a2] == row && e.loc[2 * a2 + 1] == col; }
            if (!blocked) break;
        }
        wsync();
        if (lane == 0) { e.loc[2 * a] = (int16_t)row; e.loc[2 * a + 1] = (int16_t)col; }
        wsync();
    }
    for (int i = 0; i < c.n_comp; i++) {  // component.reset() in list order
        if (c.comp[i] == COMP_BUILD) {
            for (int a = 0; a < A; a++) {
                double skill = 1.0, rate = 1.0;
                if (c.build_skill_dist == 1) {
                    skill = rng_pareto(r, 4.0);
                    rate = fmin((double)c.pmsm, (double)(c.pmsm - 1) * skill + 1.0);
                } else if (EXT && c.build_skill_dist == 2) {   // build.py:243-245
                    skill = rng_lognormal(r, e.gauss, -1.0, 0.5);
                    rate = fmin((double)c.pmsm, (double)(c.pmsm - 1) * skill + 1.0);
                }
                if (lane == 0) { e.bpay[a] = rate * c.build_payment; e.bskill[a] = skill; }
            }
        } else if (c.comp[i] == COMP_GATHER) {
            for (int a = 0; a < A; a++) {
                double bonus = 0.0;
                if (c.gather_skill_dist == 1) bonus = fmin(2.0, rng_pareto(r, 3.0)) / 2.0;
                else if (EXT && c.gather_skill_dist == 2) bonus = fmin(2.0, rng_lognormal(r, e.gauss, -2.022, 0.938)) / 2.0;  // move.py:204-205
                if (lane == 0) e.bonus[a] = bonus;
            }
        }
    }
    wsync();
    if (EXT && c.split_layout) {
        // SplitLayout.additional_reset_steps (layout_from_file.py:766-790): everybody is taken off the map; a random order
        // hands out the rank-averaged payments and re-places the agents, the chosen ranks above the water row
        rng_permutation(r, s.perm, A);
        for (int a = lane; a < A; a += NL) { e.loc[2 * a] = -1; e.loc[2 * a + 1] = -1; }
        wsync();
        for (int i = 0; i < A; i++) {
            const int a = s.perm[i];
            const bool top = (c.split_top_ranks >> i) & 1ull;
            const int r_min = top ? 0 : c.split_water_row + 1, r_max = top ? c.split_water_row : c.H;
            int row = 0, col = 0;
            for (int tries = 0; tries <= 201; tries++) {
                row = r_min + (int)rng_interval(r, (uint32_t)(r_max - r_min - 1));
                col = (int)rng_interval(r, (uint32_t)(c.W - 1));
                bool blocked = (e.cell[row * c.W + col] & CELL_WATER) != 0;
                for (int a2 = 0; a2 < A && !blocked; a2++) blocked = e.loc[2 * a2] == row && e.loc[2 * a2 + 1] == col;
                if (!blocked) break;
            }
            wsync();
            if (lane == 0) { e.loc[2 * a] = (int16_t)row; e.loc[2 * a + 1] = (int16_t)col; e.bpay[a] = e.split_skill[i]; }
            wsync();
        }
    }
    if (c.fixed_four) {
        rng_permutation(r, s.perm, A);
        for (int i = lane; i < A; i += NL) {
            const int a = s.perm[i];
            e.loc[2 * a] = c.ranked_locs[i][0]; e.loc[2 * a + 1] = c.ranked_locs[i][1];
            e.bpay[a] = c.avg_ranked_skill[i];
        }
    }
    wsync();
}

// What the step kernel does when an env finishes with auto_reset on and reset_mode == 1, after the snapshot restore.
template <bool EXT = false>
AIE_DEV_NOINLINE void device_reset_env(const DevCfg &c, uint8_t *rec, uint8_t *grec, uint8_t *scratch, int lane,
                                       const double *dyn_prob = nullptr, double *dyn_work = nullptr) {
    Env e = env_view(rec, grec, c);
    StepScratch s = step_scratch_view(scratch, c);
    Rng r; r.mt = e.mt; r.pos = e.hdr[HDR_MT_POS]; r.lane = lane;
    wsync();
    device_reset_draws<EXT>(c, e, s, r, dyn_prob, dyn_work);
    if (lane == 0) e.hdr[HDR_MT_POS] = r.pos;
    wsync();
}

// Explicit reset (aie_reset_envs), after env i's record image [0, off_mt) (and the big sections) has been restored from
// the template or state0 and, without new streams, the kept section [off_mt, off_mt + keep_bytes) loaded from the current
// record: the header and kept section a host reset packs (aie_host.h: pack_record) - counters zero but completions, the
// stream installed, the Saez section zeroed (the caller's Saez estimator writes its persistent state back afterwards).
AIE_DEV void reset_install_stream(const DevCfg &c, const ResetSrc &s, int i, uint8_t *rec, int32_t completions,
                                  int32_t mt_pos, int lane) {
    if (s.mt_key) {
        uint32_t *kept = (uint32_t *)(rec + c.off_mt);
        for (int k = lane; k < c.keep_bytes / 4; k += NL) kept[k] = 0u;
        wsync();
        for (int k = lane; k < 624; k += NL) kept[k] = s.mt_key[(size_t)i * 624 + k];
        if (c.off_gauss && lane == 0) {
            double *g = (double *)(rec + c.off_gauss);
            g[0] = s.gauss[2 * (size_t)i]; g[1] = s.gauss[2 * (size_t)i + 1];
        }
        if (c.off_split_skill)
            for (int a = lane; a < c.A; a += NL) ((double *)(rec + c.off_split_skill))[a] = s.split_skill[(size_t)i * c.A + a];
    } else if (c.off_saez) {
        for (int k = lane; k < 48; k += NL) ((double *)(rec + c.off_saez))[k] = 0.0;
    }
    if (lane == 0) {
        int32_t *hdr = (int32_t *)rec;
        for (int w = 0; w < HDR_WORDS; w++) hdr[w] = 0;
        hdr[HDR_TAX_POS] = 1; hdr[HDR_COMPLETIONS] = completions; hdr[HDR_MT_POS] = mt_pos;
    }
    wsync();
}

}  // namespace aie

#include "aie_obs.cuh"   // observations + masks (the other half of the fused step kernel)

namespace aie {

// ------------------------------------------------------------------------------------------------
// Random policy (bench / testing utility): uniform over the unmasked entries of one mask segment.
// ------------------------------------------------------------------------------------------------
AIE_DEV uint64_t mix64(uint64_t x) {  // splitmix64 finaliser
    x += 0x9e3779b97f4a7c15ull;
    x = (x ^ (x >> 30)) * 0xbf58476d1ce4e5b9ull;
    x = (x ^ (x >> 27)) * 0x94d049bb133111ebull;
    return x ^ (x >> 31);
}
// The policy sampler's stream key of a call inside a captured rollout (aie_rollout_capture_begin): seed_mix =
// host_mix64(seed), *base = the handle's policy_calls when the replay began (written on the stream by
// aie_rollout_replay_begin), ord = the call's ordinal since the capture began.  Call n of an eager loop has the key
// host_mix64(seed) ^ host_mix64(n), so a replay draws what the same calls made eagerly would.
AIE_DEV uint64_t policy_call_key(uint64_t seed_mix, const uint64_t *base, uint64_t ord) {
    return seed_mix ^ mix64(*base + ord + 1);
}
// Uniform choice among the set entries of mask[0..n) by one warp: ballots count the open entries, a hashed
// rank picks one, and the lane holding it is found with popcounts.  Returns the same value on every lane.
// (masks are 0 / 1: any non-zero element is open; MT: float or bf16_t)
AIE_DEV bool mask_open(float v) { return v != 0.0f; }
AIE_DEV bool mask_open(bf16_t v) { return (v.bits & 0x7FFFu) != 0u; }
template <typename MT>
AIE_DEV int sample_segment_warp(const MT *mask, int n, uint64_t key, int lane) {
#if AIE_ON_DEVICE
    // one pass: the segment (at most MAX_MASK = 160 entries) becomes five ballot words held in registers
    uint32_t w[5];
    int total = 0;
#pragma unroll
    for (int ch = 0; ch < 5; ch++) {
        const int j = ch * NL + lane;
        w[ch] = wballot(j < n && mask_open(mask[j]));
        total += __popc(w[ch]);
    }
    if (total == 0) return 0;
    int r = (int)((uint32_t)(mix64(key) >> 32) % (uint32_t)total);
#pragma unroll
    for (int ch = 0; ch < 5; ch++) {
        const int cnt = __popc(w[ch]);
        if (r < cnt) return ch * NL + (int)__fns(w[ch], 0, r + 1);  // position of the (r+1)-th open entry
        r -= cnt;
    }
    return 0;
#else
    int total = 0;
    for (int base = 0; base < n; base += NL) {
        const int j = base + lane;
        total += __popc_u32(wballot(j < n && mask_open(mask[j])));
    }
    if (total == 0) return 0;
    int r = (int)((uint32_t)(mix64(key) >> 32) % (uint32_t)total);
    for (int base = 0; base < n; base += NL) {
        const int j = base + lane;
        const uint32_t m = wballot(j < n && mask_open(mask[j]));
        const int cnt = __popc_u32(m);
        if (r < cnt) {
            uint32_t mm = m;
            for (int i = 0; i < r; i++) mm &= mm - 1;  // drop the r lowest set bits
            return base + first_lane(mm);
        }
        r -= cnt;
    }
    return 0;
#endif
}

// One unit of an env's random policy: unit u < A = agent u (one draw per subspace), unit A + b = planner bracket b.
// Units are independent, so the kernel gives each its own warp.
template <bool EXT = false, typename MT = float>
AIE_DEV void sample_actions_unit(const DevCfg &c, const MT *a_mask, const MT *p_mask, int32_t *act_a,
                                 int32_t *act_p, uint64_t key, int u, int lane) {
    if (u < c.A) {
        const int a = u;
        const MT *m = a_mask + (size_t)a * c.Na;
        if (!c.multi_action) {
            const int v = sample_segment_warp(m, c.Na, key + 0x100 * a, lane);
            if (lane == 0) act_a[a] = v;
        } else {
            int off = 0;
            for (int si = 0; si < c.n_sub; si++) {
                const int v = sample_segment_warp(m + off, c.sub_n[si] + 1, key + 0x100 * a + si + 1, lane);
                if (lane == 0) act_a[a * c.n_sub + si] = v;
                off += c.sub_n[si] + 1;
            }
        }
    } else if (EXT && c.planner_single) {
        if (u == c.A) {
            const int v = sample_segment_warp(p_mask, c.Np, key + 0x10000, lane);
            if (lane == 0) act_p[0] = v;
        }
    } else if (c.planner_acts) {
        const int b = u - c.A;
        const int v = sample_segment_warp(p_mask + (size_t)b * (1 + c.R), 1 + c.R, key + 0x10000 + b, lane);
        if (lane == 0) act_p[b] = v;
    }
}
// One env: every agent (and planner bracket) draws one uniformly random unmasked action per subspace.
template <bool EXT = false, typename MT = float>
AIE_DEV void sample_actions_env(const DevCfg &c, const MT *a_mask, const MT *p_mask, int32_t *act_a,
                                int32_t *act_p, uint64_t key, int lane) {
    const int units = c.A + (c.planner_acts ? c.B : 0);
    for (int u = 0; u < units; u++) sample_actions_unit<EXT, MT>(c, a_mask, p_mask, act_a, act_p, key, u, lane);
}

// ------------------------------------------------------------------------------------------------
// Policy sampler (aie_sample_policy): one categorical draw per mask segment from the softmax of the caller's logits
// restricted to the open entries.  Random stream: u = (mix64(k) >> 11) * 2^-53 per segment, k the key the random
// sampler hashes for that segment (sample_actions_unit; the per-env key comes from a call counter of its own).  Draw:
// m = largest open logit, w_j = exp((double)l_j - m) for open j (0 otherwise), Z = sum w; the action is the smallest
// j with w_j > 0 and u * Z < w_0 + .. + w_j (float64), else the last j with w_j > 0 (rounding).  greedy: the first
// open j with l_j == m.  log-prob = (float)(((double)l_a - m) - log(Z)).  No open entry: action 0, log-prob 0; an open
// logit that is NaN or +inf, or no finite open logit: the first open entry, log-prob NaN.
// ------------------------------------------------------------------------------------------------
AIE_DEV float logit_value(float v) { return v; }
AIE_DEV float logit_value(bf16_t v) {
#if AIE_ON_DEVICE
    return __uint_as_float((uint32_t)v.bits << 16);
#else
    const uint32_t u = (uint32_t)v.bits << 16;
    float f;
    memcpy(&f, &u, 4);
    return f;
#endif
}
AIE_DEV double policy_uniform(uint64_t key) { return (double)(mix64(key) >> 11) * 0x1.0p-53; }

// The open entries, m and Z of one segment: mask[j * ms] (ms: element stride of the mask; 1 except for the COVID
// agents' [levels][S] masks) and logit[j], j < n <= MAX_MASK.  Shared by the sampler (policy_segment_warp) and the
// evaluation (policy_segment_eval), so both sum Z in one order: on the device a float64 inclusive warp scan per chunk of
// 32 entries (entry j on lane j % 32 of chunk j / 32) with the chunks' totals added in turn, in the host build a serial
// sum.  Two steps, so that a caller leaves on the edge cases before the scan: policy_segment_open returns 0: no open
// entry; 1: an open logit is NaN or +inf, or no open logit is finite; 2: policy_segment_z then sets mx and Z.
struct PolicySeg {
    float mx;          // the largest open logit (m = (double)mx)
    double Z;          // sum over open j of exp((double)l_j - m)
#if AIE_ON_DEVICE
    float lv[5];       // this lane's entry of each chunk: its logit when open, else -inf
    uint32_t om[5];    // open entries, one ballot per chunk
    double w[5];       // this lane's w of each chunk (chunks past n: unset)
    double cum[5];     // inclusive prefix of w over the segment, this lane's entry of each chunk (chunks past n: 0)
    uint32_t pos[5];   // entries with w > 0
#else
    int first;         // the first open entry
#endif
};
template <typename MT, typename LT>
AIE_DEV int policy_segment_open(const MT *mask, int ms, const LT *logit, int n, int lane, PolicySeg &s) {
#if AIE_ON_DEVICE
    uint32_t bad = 0, fin = 0, any = 0;
    float mx = -INFINITY;
#pragma unroll
    for (int ch = 0; ch < 5; ch++) {
        const int j = ch * NL + lane;
        const bool o = j < n && mask_open(mask[(size_t)j * ms]);
        const float v = o ? logit_value(logit[j]) : -INFINITY;
        s.lv[ch] = v;
        s.om[ch] = wballot(o);
        any |= s.om[ch];
        bad |= wballot(o && !(v < INFINITY));          // NaN or +inf
        fin |= wballot(o && v > -INFINITY && v < INFINITY);
        mx = fmaxf(mx, v);
    }
    s.mx = mx;   // this lane's part (policy_segment_z reduces it)
    return !any ? 0 : (bad || !fin) ? 1 : 2;
#else
    (void)lane;
    int first = -1;
    bool bad = false, fin = false;
    float mx = -INFINITY;
    for (int j = 0; j < n; j++) {
        if (!mask_open(mask[(size_t)j * ms])) continue;
        const float v = logit_value(logit[j]);
        if (first < 0) first = j;
        if (!(v < INFINITY)) bad = true;
        else if (v > -INFINITY) { fin = true; mx = v > mx ? v : mx; }
    }
    s.first = first;
    s.mx = mx;
    return first < 0 ? 0 : (bad || !fin) ? 1 : 2;
#endif
}
template <typename MT, typename LT>
AIE_DEV void policy_segment_z(const MT *mask, int ms, const LT *logit, int n, int lane, PolicySeg &s) {
#if AIE_ON_DEVICE
    (void)mask; (void)ms; (void)logit;
    float mx = s.mx;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    s.mx = mx;
    const double m = (double)mx;
    double carry = 0.0;
#pragma unroll
    for (int ch = 0; ch < 5; ch++) {
        s.cum[ch] = 0.0; s.pos[ch] = 0u;
        if (ch * NL < n) {   // warp-uniform
            const double w = ((s.om[ch] >> lane) & 1u) ? exp((double)s.lv[ch] - m) : 0.0;
            s.w[ch] = w;
            s.pos[ch] = wballot(w > 0.0);
            double t = w;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const double u = __shfl_up_sync(0xffffffffu, t, o);
                if (lane >= o) t += u;
            }
            s.cum[ch] = carry + t;
            carry = __shfl_sync(0xffffffffu, s.cum[ch], 31);
        }
    }
    s.Z = carry;
#else
    (void)lane;
    const double m = (double)s.mx;
    double Z = 0.0;
    for (int j = 0; j < n; j++)
        if (mask_open(mask[(size_t)j * ms])) Z += exp((double)logit_value(logit[j]) - m);
    s.Z = Z;
#endif
}

// One segment of the sampler (the layout of policy_segment_open).  Returns the action on every lane and writes the
// log-probability to *lp on every lane.  Device: one warp; the crossing of u * Z is found by ballots over the prefix.
template <typename MT, typename LT>
AIE_DEV int policy_segment_warp(const MT *mask, int ms, const LT *logit, int n, uint64_t key, int greedy, int lane, float *lp) {
    PolicySeg s;
    const int st = policy_segment_open(mask, ms, logit, n, lane, s);
    if (st == 0) { *lp = 0.0f; return 0; }
#if AIE_ON_DEVICE
    if (st == 1) {
        *lp = __int_as_float(0x7fc00000);
#pragma unroll
        for (int ch = 0; ch < 5; ch++)
            if (s.om[ch]) return ch * NL + first_lane(s.om[ch]);
        return 0;
    }
    policy_segment_z(mask, ms, logit, n, lane, s);
    const float mx = s.mx;
    const double m = (double)mx, Z = s.Z;
    int a = -1;
    if (greedy) {
#pragma unroll
        for (int ch = 0; ch < 5; ch++) {
            const uint32_t hit = wballot(((s.om[ch] >> lane) & 1u) && s.lv[ch] == mx);
            if (a < 0 && hit) a = ch * NL + first_lane(hit);
        }
    } else {
        const double t = policy_uniform(key) * Z;
#pragma unroll
        for (int ch = 0; ch < 5; ch++) {
            const uint32_t hit = wballot(((s.pos[ch] >> lane) & 1u) && t < s.cum[ch]);
            if (a < 0 && hit) a = ch * NL + first_lane(hit);
        }
        if (a < 0) {
#pragma unroll
            for (int ch = 0; ch < 5; ch++)
                if (s.pos[ch]) a = ch * NL + 31 - __clz(s.pos[ch]);
        }
    }
    const double la = greedy ? m : (double)logit_value(logit[a]);
    *lp = (float)((la - m) - log(Z));
    return a;
#else
    if (st == 1) { *lp = NAN; return s.first; }
    policy_segment_z(mask, ms, logit, n, lane, s);
    const float mx = s.mx;
    const double m = (double)mx, Z = s.Z;
    int a = -1;
    if (greedy) {
        for (int j = 0; j < n && a < 0; j++)
            if (mask_open(mask[(size_t)j * ms]) && logit_value(logit[j]) == mx) a = j;
    } else {
        const double t = policy_uniform(key) * Z;
        double cum = 0.0;
        int last = -1;
        for (int j = 0; j < n && a < 0; j++) {
            if (!mask_open(mask[(size_t)j * ms])) continue;
            const double w = exp((double)logit_value(logit[j]) - m);
            cum += w;
            if (w > 0.0) { last = j; if (t < cum) a = j; }
        }
        if (a < 0) a = last;
    }
    *lp = (float)(((double)logit_value(logit[a]) - m) - log(Z));
    return a;
#endif
}

// Where aie_sample_policy reads and writes (device pointers; the log-probabilities are optional)
struct PolicyBufs {
    const void *a_logit, *p_logit;   // [E][A][Na], [E][Np]: float or bf16_t (the kernel's LT)
    float *lp_a, *lp_p;              // [E][A][n_act_a], [E][n_act_p] or null
    int32_t greedy;
};

// One unit of the policy sampler, laid out and keyed like sample_actions_unit (unit u < A: agent u, one draw per
// subspace; unit A + b: planner bracket b, or the single-action planner's one index).
template <bool EXT, typename MT, typename LT>
AIE_DEV void policy_actions_unit(const DevCfg &c, const MT *a_mask, const MT *p_mask, const LT *a_logit, const LT *p_logit,
                                 int32_t *act_a, int32_t *act_p, float *lp_a, float *lp_p, uint64_t key, int greedy, int u,
                                 int lane) {
    float lp;
    if (u < c.A) {
        const int a = u;
        const MT *m = a_mask + (size_t)a * c.Na;
        const LT *l = a_logit + (size_t)a * c.Na;
        if (!c.multi_action) {
            const int v = policy_segment_warp(m, 1, l, c.Na, key + 0x100 * a, greedy, lane, &lp);
            if (lane == 0) { act_a[a] = v; if (lp_a) lp_a[a] = lp; }
        } else {
            int off = 0;
            for (int si = 0; si < c.n_sub; si++) {
                const int v = policy_segment_warp(m + off, 1, l + off, c.sub_n[si] + 1, key + 0x100 * a + si + 1, greedy, lane, &lp);
                if (lane == 0) { act_a[a * c.n_sub + si] = v; if (lp_a) lp_a[a * c.n_sub + si] = lp; }
                off += c.sub_n[si] + 1;
            }
        }
    } else if (EXT && c.planner_single) {
        if (u == c.A) {
            const int v = policy_segment_warp(p_mask, 1, p_logit, c.Np, key + 0x10000, greedy, lane, &lp);
            if (lane == 0) { act_p[0] = v; if (lp_p) lp_p[0] = lp; }
        }
    } else if (c.planner_acts) {
        const int b = u - c.A;
        const size_t off = (size_t)b * (1 + c.R);
        const int v = policy_segment_warp(p_mask + off, 1, p_logit + off, 1 + c.R, key + 0x10000 + b, greedy, lane, &lp);
        if (lane == 0) { act_p[b] = v; if (lp_p) lp_p[b] = lp; }
    }
}
// Env e's pointers, and every unit of it (u < 0) or unit u only.  key: mix64(s ^ mix64(e)), s the call's stream.
template <bool EXT, typename MT, typename LT>
AIE_DEV void policy_actions_env(const DevCfg &c, const DevBufs &b, const PolicyBufs &p, int e, uint64_t key, int u, int lane) {
    const MT *am = (const MT *)b.a_mask + (size_t)e * c.A * c.Na, *pm = (const MT *)b.p_mask + (size_t)e * c.Np;
    const LT *al = (const LT *)p.a_logit + (size_t)e * c.A * c.Na;
    const LT *pl = c.n_act_p ? (const LT *)p.p_logit + (size_t)e * c.Np : nullptr;
    int32_t *aa = const_cast<int32_t *>(b.act_a) + (size_t)e * c.A * c.n_act_a;
    int32_t *ap = c.n_act_p ? const_cast<int32_t *>(b.act_p) + (size_t)e * c.n_act_p : nullptr;
    float *la = p.lp_a ? p.lp_a + (size_t)e * c.A * c.n_act_a : nullptr;
    float *lq = (p.lp_p && c.n_act_p) ? p.lp_p + (size_t)e * c.n_act_p : nullptr;
    if (u >= 0) { policy_actions_unit<EXT>(c, am, pm, al, pl, aa, ap, la, lq, key, p.greedy, u, lane); return; }
    const int units = c.A + (c.planner_acts ? c.B : 0);
    for (int v = 0; v < units; v++) policy_actions_unit<EXT>(c, am, pm, al, pl, aa, ap, la, lq, key, p.greedy, v, lane);
}

// ------------------------------------------------------------------------------------------------
// Evaluation of stored actions (aie_evaluate_policy, aie_evaluate_policy_backward): per mask segment, the
// log-probability of the stored action a and the entropy of the softmax of the logits restricted to the open entries,
// and the gradient of g_lp * lp + g_H * H with respect to the logits.  m and Z are policy_segment_open / _z's, the
// sampler's own, so lp is bit for bit what the sampler returned for (logits, masks, a).  In float64, rounded once:
//   lp = (float)(((double)l_a - m) - log Z),  H = (float)(log Z - sum_j p_j (l_j - m)),  p_j = w_j / Z;
//   gradient of open j: g_lp ([j = a] - p_j) - g_H p_j ((l_j - m - log Z) + H), closed j: 0.
// No open entry: lp = H = 0, gradient 0.  An open logit NaN or +inf, or none finite: lp = H = NaN, the open entries'
// gradient NaN.  a closed or outside [0, n): lp = NaN, the open entries' gradient NaN, H as usual (a is read, never
// the mask or logit outside the segment).  An open entry with w_j = 0 (at -inf) has p_j = 0: no entropy term.
// The backward recomputes m and Z from the logits; nothing of the forward is stored.
// ------------------------------------------------------------------------------------------------
// round-to-nearest-even bfloat16 bits of a float64 value without double rounding: to float32 rounded to odd (toward
// zero, the last bit set when inexact), then to nearest even (NaN -> a quiet NaN)
AIE_DEV uint16_t bf16_from_double(double x) {
    if (x != x) return 0x7FC0u;
    const float f = (float)x;
    uint32_t u;
#if AIE_ON_DEVICE
    u = __float_as_uint(f);
#else
    memcpy(&u, &f, 4);
#endif
    if ((double)f != x) {
        if (fabs((double)f) > fabs(x)) u -= 1u;   // one step toward zero (from +-inf on overflow: +-FLT_MAX)
        u |= 1u;
    }
    return (uint16_t)((u + 0x7FFFu + ((u >> 16) & 1u)) >> 16);
}
AIE_DEV void put_grad(float *p, double g) { *p = (float)g; }
AIE_DEV void put_grad(bf16_t *p, double g) { p->bits = bf16_from_double(g); }

// One segment (the layout of policy_segment_open), the stored action at *act.  Forward (BWD false): lp and H to *lp,
// *h from lane 0.  Backward: g_lp = *glp and g_H = *gh (null: 0), the gradient of entries j < n to grad[j].
template <bool BWD, typename MT, typename LT>
AIE_DEV void policy_segment_eval(const MT *mask, int ms, const LT *logit, int n, const int32_t *act, const float *glp,
                                 const float *gh, float *lp, float *h, LT *grad, int lane) {
    PolicySeg s;
    const int st = policy_segment_open(mask, ms, logit, n, lane, s);
    if (st == 2) policy_segment_z(mask, ms, logit, n, lane, s);
    const int a = *act;
    const bool ok = a >= 0 && a < n && mask_open(mask[(size_t)a * ms]);
    double m = 0.0, Z = 1.0, lz = 0.0, H = 0.0;
    if (st == 2) {
        m = (double)s.mx;
        Z = s.Z;
        lz = log(Z);
        double e = 0.0;   // sum over open j of w_j (l_j - m)
#if AIE_ON_DEVICE
#pragma unroll
        for (int ch = 0; ch < 5; ch++)
            if (ch * NL < n && s.w[ch] > 0.0) e += s.w[ch] * ((double)s.lv[ch] - m);
        e = wsum(e);
#else
        for (int j = 0; j < n; j++) {
            if (!mask_open(mask[(size_t)j * ms])) continue;
            const double d = (double)logit_value(logit[j]) - m, w = exp(d);
            if (w > 0.0) e += w * d;
        }
#endif
        H = lz - e / Z;
    }
    if (!BWD) {
        if (lane == 0) {
            if (st == 2) {
                *lp = ok ? (float)(((double)logit_value(logit[a]) - m) - lz) : NAN;
                *h = (float)H;
            } else {
                *lp = *h = st ? NAN : 0.0f;
            }
        }
        return;
    }
    const double g_lp = glp ? (double)*glp : 0.0, g_h = gh ? (double)*gh : 0.0;
    const bool nan_open = st == 1 || (st == 2 && !ok);
#if AIE_ON_DEVICE
#pragma unroll
    for (int ch = 0; ch < 5; ch++) {
        const int j = ch * NL + lane;
        if (j < n) {
            double g = 0.0;
            if ((s.om[ch] >> lane) & 1u) {
                if (nan_open) {
                    g = NAN;
                } else {
                    const double p = s.w[ch] / Z;
                    g = g_lp * ((j == a ? 1.0 : 0.0) - p);
                    if (p > 0.0) g -= g_h * p * ((((double)s.lv[ch] - m) - lz) + H);
                }
            }
            put_grad(grad + j, g);
        }
    }
#else
    for (int j = 0; j < n; j++) {
        double g = 0.0;
        if (mask_open(mask[(size_t)j * ms])) {
            if (nan_open) {
                g = NAN;
            } else {
                const double d = (double)logit_value(logit[j]) - m, p = exp(d) / Z;
                g = g_lp * ((j == a ? 1.0 : 0.0) - p);
                if (p > 0.0) g -= g_h * p * ((d - lz) + H);
            }
        }
        put_grad(grad + j, g);
    }
#endif
}

// Where aie_evaluate_policy reads and writes (device pointers; rows of the leading batch, N of them, at r * row size)
struct PolicyEvalBufs {
    const void *a_logit, *p_logit;              // [N][A][Na], [N][Np] (COVID-19: [N][S][1 + levels], [N][1 + sub levels]): LT
    const void *a_mask, *p_mask;                // the mask layouts (COVID-19 agents: [N][1 + levels][S]): MT
    const int32_t *act_a, *act_p;               // [N][A][n_act_a], [N][n_act_p] (COVID-19: [N][S], [N])
    float *lp_a, *lp_p, *h_a, *h_p;             // forward: log-probabilities and entropies, shaped like the actions
    const float *glp_a, *glp_p, *gh_a, *gh_p;   // backward: their upstream gradients, or null (zero)
    void *g_a, *g_p;                            // backward: the gradient with respect to the logits (LT, their layout)
};
// One segment of row r, slot k of its actions, entries at off of its logits and masks (ms: the masks' stride).
template <bool BWD, typename MT, typename LT>
AIE_DEV void policy_eval_slot(const MT *mask, int ms, const void *logit, int n, size_t off, const int32_t *act,
                              const float *glp, const float *gh, float *lp, float *h, void *grad, size_t k, int lane) {
    policy_segment_eval<BWD>(mask, ms, (const LT *)logit + off, n, act + k, BWD && glp ? glp + k : nullptr,
                             BWD && gh ? gh + k : nullptr, BWD ? nullptr : lp + k, BWD ? nullptr : h + k,
                             BWD ? (LT *)grad + off : nullptr, lane);
}
// One unit of row r: u < A is agent u (every subspace in multi-action mode), u = A + b planner slot b (a bracket, or
// the single-action planner's one index).
template <bool BWD, typename MT, typename LT>
AIE_DEV void policy_eval_unit(const DevCfg &c, const PolicyEvalBufs &p, long long r, int u, int lane) {
    if (u < c.A) {
        const size_t row = ((size_t)r * c.A + u) * c.Na, slot = ((size_t)r * c.A + u) * c.n_act_a;
        int off = 0;
        for (int si = 0; si < c.n_act_a; si++) {
            const int n = c.multi_action ? c.sub_n[si] + 1 : c.Na;
            policy_eval_slot<BWD, MT, LT>((const MT *)p.a_mask + row + off, 1, p.a_logit, n, row + off, p.act_a, p.glp_a,
                                          p.gh_a, p.lp_a, p.h_a, p.g_a, slot + si, lane);
            off += n;
        }
    } else {
        const int b = u - c.A, n = c.planner_single ? c.Np : 1 + c.R;
        const size_t off = (size_t)r * c.Np + (size_t)b * n;
        policy_eval_slot<BWD, MT, LT>((const MT *)p.p_mask + off, 1, p.p_logit, n, off, p.act_p, p.glp_p, p.gh_p, p.lp_p,
                                      p.h_p, p.g_p, (size_t)r * c.n_act_p + b, lane);
    }
}
// Row r: every unit (u < 0) or unit u only; units = A + n_act_p.
template <bool BWD, typename MT, typename LT>
AIE_DEV void policy_eval_row(const DevCfg &c, const PolicyEvalBufs &p, long long r, int u, int lane) {
    if (u >= 0) { policy_eval_unit<BWD, MT, LT>(c, p, r, u, lane); return; }
    const int units = c.A + c.n_act_p;
    for (int v = 0; v < units; v++) policy_eval_unit<BWD, MT, LT>(c, p, r, v, lane);
}

// Where aie_compute_advantages reads and writes: group g = 0 the agents' columns ([T][E * A]), g = 1 the planner's ([T][E]).
struct AdvantageBufs {
    const void *r[2];                 // rewards, float or double (the kernel's template arguments)
    const float *v[2], *lv[2], *fv[2];   // values [T][n], last values [n], final values [T][n] or null
    const int32_t *done;              // [T][E]
    float *adv[2], *ret[2];           // [T][n]
    double gamma[2], gl[2];           // gl = gamma * lambda
    long long n[2];                   // columns: E * A, E (0: no planner group)
    int per_env[2];                   // columns per env: A, 1
};
// Timesteps per chunk of a column's loads: the loads of the next chunk are issued before the current one is computed,
// and they do not depend on the carry, so a column keeps 2 * AIE_GAE_K timesteps of loads in flight.
#ifndef AIE_GAE_K
#define AIE_GAE_K 8
#endif
#if AIE_ON_DEVICE
#define AIE_GAE_UNROLL AIE_UNROLL(AIE_GAE_K)
#else
#define AIE_GAE_UNROLL
#endif
// The dones of the chunk ending at row hi - 1 (rows hi - AIE_GAE_K .. hi - 1 read backwards; rows < 0 are 0).
AIE_DEV void gae_load_done(int32_t *d, const int32_t *done, long long E, long long e, int hi) {
    AIE_GAE_UNROLL
    for (int k = 0; k < AIE_GAE_K; k++) {
        const int t = hi - 1 - k;
        d[k] = t >= 0 ? done[(long long)t * E + e] : 0;
    }
}
// Rewards, values and (where the done holds) final values of the same chunk.
template <typename RT>
AIE_DEV void gae_load_vals(RT *r, float *v, float *f, const int32_t *d, const RT *R, const float *V, const float *F,
                           long long n, long long col, int hi) {
    AIE_GAE_UNROLL
    for (int k = 0; k < AIE_GAE_K; k++) {
        const int t = hi - 1 - k;
        const long long i = (long long)t * n + col;
        r[k] = t >= 0 ? R[i] : (RT)0;
        v[k] = t >= 0 ? V[i] : 0.f;
        f[k] = (t >= 0 && F && d[k]) ? F[i] : 0.f;
    }
}
// One column of group g over T steps (the recursion of aie_compute_advantages, include/aie_b200.h).  The carry is
// only A and the value of the next row; the dones run one chunk ahead of the other loads so that the final values of
// a chunk can be fetched as soon as its rewards and values are.
// KF (aie_compute_advantages_k): the final values are [nk][n], row = the done's episode-end ordinal in the column: the
// column's done count is taken first, and a done step reads its row when the recursion reaches it (an ordinal >= nk
// reads NaN).
template <typename RT, bool KF = false>
AIE_DEV void gae_column(const AdvantageBufs &b, int g, long long E, long long col, int T, int nk = 0) {
    constexpr int K = AIE_GAE_K;
    const long long n = b.n[g], e = col / b.per_env[g];
    const RT *R = (const RT *)b.r[g];
    const float *V = b.v[g], *F = KF ? nullptr : b.fv[g];
    const float *FK = KF ? b.fv[g] : nullptr;
    int ord = 0;   // KF: done steps of the column not yet reached by the backward recursion
    if constexpr (KF) {
        if (FK)
            for (int t = 0; t < T; t++) ord += b.done[(long long)t * E + e] != 0;
    }
    const double gamma = b.gamma[g], gl = b.gl[g];
    int32_t dn[K], dnn[K];
    RT rn[K];
    float vn[K], fn[K];
    gae_load_done(dn, b.done, E, e, T);
    gae_load_vals<RT>(rn, vn, fn, dn, R, V, F, n, col, T);
    gae_load_done(dnn, b.done, E, e, T - K);
    float vnext = b.lv[g][col];
    double a = 0.0;
    for (int hi = T; hi > 0; hi -= K) {
        int32_t d[K];
        RT r[K];
        float v[K], f[K];
        AIE_GAE_UNROLL
        for (int k = 0; k < K; k++) { d[k] = dn[k]; r[k] = rn[k]; v[k] = vn[k]; f[k] = fn[k]; dn[k] = dnn[k]; }
        if (hi - K > 0) {
            gae_load_vals<RT>(rn, vn, fn, dn, R, V, F, n, col, hi - K);
            gae_load_done(dnn, b.done, E, e, hi - 2 * K);
        }
        AIE_GAE_UNROLL
        for (int k = 0; k < K; k++) {
            const int t = hi - 1 - k;
            if (t < 0) break;
            const bool dk = d[k] != 0;
            double fk = (double)f[k];
            if constexpr (KF) {
                if (dk && FK) { --ord; fk = ord < nk ? (double)FK[(long long)ord * n + col] : (double)NAN; }
            }
            const double nv = dk ? fk : (double)vnext;
            const double delta = ((double)r[k] + gamma * nv) - (double)v[k];
            a = (dk || t == T - 1) ? delta : delta + gl * a;
            const long long i = (long long)t * n + col;
            b.adv[g][i] = (float)a;
            b.ret[g][i] = (float)(a + (double)v[k]);
            vnext = v[k];
        }
    }
}

}  // namespace aie
