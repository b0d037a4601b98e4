// aie_metrics.cuh — env.metrics of one replica from its state record (aie_metrics_kernel, aie_episode_metrics).
//
// One warp per env reads the record in global memory (the current one or its end-of-episode snapshot) and writes one row
// of the caller's [E, K] float64 table.  The columns are an op program built on the host (aie_host.h:
// build_metric_layout); this file only evaluates it.  The values are what foundation/metrics.py computes from the same
// record, and every reduction follows numpy's summation order so that the rows are bit-equal to it:
//   np.sum / np.mean of a contiguous float64 run   pairwise summation, blocks of 128 (np_pairwise_sum), longer runs split
//                                                  at n / 2 rounded down to a multiple of 8 (np_sum_staged)
//   gini, A < 30                                   one np.sum over the A x A absolute differences, row-major
//   gini, A >= 30                                  np.sort, a sequential np.cumsum, pairwise sums
// The one exception is labor/weighted_cost under an energy warm-up: 1 - exp(-x / c) uses the platform's exp, which can
// differ from numpy's in the last place.
// Compiled by nvcc (sm_90a, NL = 32: aie_metrics_kernel in aie_abi.cu) and by the host emulation (tests/emu, NL = 1:
// metrics_env_host below, called by aie_episode_metrics in place of the kernel launch).
#pragma once
#include <string.h>

#include "aie_core.cuh"

namespace aie {

constexpr int MET_BLOCK = 128;       // numpy's pairwise-summation block (PW_BLOCKSIZE)
constexpr int MET_MAX_AGENTS = 64;   // = AIE_MAX_AGENTS
// per-warp staging (doubles): endowments [64], weights [64], scratch [64], one summation block [128]
constexpr int MET_WARP_DOUBLES = 3 * MET_MAX_AGENTS + MET_BLOCK;

#if AIE_ON_DEVICE
AIE_DEV double met_nan() { return __longlong_as_double(0x7ff8000000000000ll); }
#else
AIE_DEV double met_nan() { return NAN; }
#endif

// numpy's pairwise sum of the n elements f(lo) .. f(lo + n - 1): runs above one block split as numpy splits them, each
// block is staged in blk[] by the lanes and summed by np_pairwise_sum (warp-uniform).  D bounds the recursion
// (n <= 128 * 2^D).
template <int D, class F>
AIE_DEV double np_sum_staged(const F &f, double *blk, int lo, int n, int lane) {
    if constexpr (D > 0) {
        if (n > MET_BLOCK) {
            int n2 = n / 2;
            n2 -= n2 % 8;
            const double left = np_sum_staged<D - 1>(f, blk, lo, n2, lane);
            return left + np_sum_staged<D - 1>(f, blk, lo + n2, n - n2, lane);
        }
    }
    for (int k = lane; k < n; k += NL) blk[k] = f(lo + k);
    wsync();
    const double r = np_pairwise_sum(blk, n);
    wsync();
    return r;
}

// scenarios/utils/social_metrics.py:10-46 in numpy's order (foundation/metrics.py: gini).  x[A] staged; sum_x = np.sum(x).
AIE_DEV double np_gini(const double *x, double sum_x, double *tmp, double *blk, int A, int lane) {
    if (A < 30) {
        const double diff = np_sum_staged<4>([&](int k) { const int i = k / A; return fabs(x[i] - x[k - i * A]); }, blk, 0, A * A, lane);
        const double norm = (double)(2 * A) * sum_x;
        return (diff / (norm + 1e-10)) / ((A - 1) / (double)A);
    }
    for (int i = lane; i < A; i += NL) {   // np.sort: rank, ties by index (equal values are interchangeable)
        int rank = 0;
        for (int j = 0; j < A; j++) rank += (x[j] < x[i] || (x[j] == x[i] && j < i)) ? 1 : 0;
        tmp[rank] = x[i];
    }
    wsync();
    const double tot = np_pairwise_sum(tmp, A) + 1e-10;
    if (lane == 0) {   // np.cumsum(s) / (np.sum(s) + 1e-10)
        double cum = 0.0;
        for (int i = 0; i < A; i++) { cum += tmp[i]; blk[i] = cum / tot; }
    }
    wsync();
    const double acc = np_pairwise_sum(blk, A);
    wsync();
    return 1.0 - (2.0 / (A + 1)) * acc;
}

// One row: rec = the env's record in global memory; source 0 = current record, 1 = end-of-episode snapshot.
// sm: MET_WARP_DOUBLES of this warp's shared memory.  Warp-collective.
AIE_DEV void metrics_env(const DevCfg &c, const uint8_t *rec, const uint32_t *prog, int K, int source, double *row,
                         double *sm, int lane) {
    const int A = c.A;
    const int32_t *hdr = (const int32_t *)rec;
    if (source == 1 && hdr[HDR_T] == 0) {   // no finished episode recorded yet (previous_episode_metrics is None)
        for (int j = lane; j < K; j += NL) row[j] = met_nan();
        return;
    }
    const double *coin = (const double *)(rec + c.off_coin), *esc_coin = (const double *)(rec + c.off_esc_coin);
    const double *labor = (const double *)(rec + c.off_labor), *util = (const double *)(rec + c.off_util_prev);
    const double *bpay = (const double *)(rec + c.off_bpay), *stats = (const double *)(rec + c.off_stats);
    const int32_t *inv = (const int32_t *)(rec + c.off_inv), *esc = (const int32_t *)(rec + c.off_esc);
    double *x = sm, *w = sm + MET_MAX_AGENTS, *tmp = sm + 2 * MET_MAX_AGENTS, *blk = sm + 3 * MET_MAX_AGENTS;

    for (int a = lane; a < A; a += NL) x[a] = coin[a] + esc_coin[a];   // total_endowment("Coin")
    wsync();
    const double sum_x = np_pairwise_sum(x, A);
    const double gini = np_gini(x, sum_x, tmp, blk, A, lane);
    // inverse-income weights 1 / max(v, 1) normalised by their sum (v: endowments; one-step-economy: production)
    const double *wv = c.one_step ? bpay : x;
    for (int a = lane; a < A; a += NL) w[a] = 1.0 / fmax(wv[a], 1.0);
    wsync();
    const double wtot = np_pairwise_sum(w, A);
    for (int a = lane; a < A; a += NL) {
        const double wa = w[a] / wtot;
        tmp[a] = x[a] * wa;
        blk[a] = util[a] * wa;
    }
    wsync();
    const double inv_w_coin = np_pairwise_sum(tmp, A), inv_w_util = np_pairwise_sum(blk, A);
    double houses = 0.0;
    if (c.has[COMP_BUILD]) {
        const uint8_t *cell = rec + c.off_cell;
        int n = 0;
        for (int k = lane; k < c.HW; k += NL) n += (cell[k] & CELL_HOUSE) ? 1 : 0;
        houses = wsum((double)n);
    }
    int poorest = 0, richest = 0;   // first index of np.argmin / np.argmax
    for (int a = 1; a < A; a++) {
        if (x[a] < x[poorest]) poorest = a;
        if (x[a] > x[richest]) richest = a;
    }
    // a finished episode still waiting for its reset has been counted by the reference (base_env.py:1021-1025)
    const int completions = hdr[HDR_COMPLETIONS] + ((source == 0 && hdr[HDR_T] >= c.T) ? 1 : 0);
    double ew = 1.0;   // layout_from_file.py:249-267
    if (c.warm_const > 0.0) ew = 1.0 - exp((double)(-(c.warm_auto ? hdr[HDR_AUTO_WARMUP] : completions)) / c.warm_const);
    const double *tax = stats + (c.st_tax >= 0 ? c.st_tax : 0);
    const double periods = tax[ST_TAX_PERIODS];
    const double n_obs = c.st_tax >= 0 ? fmax(1.0, np_pairwise_sum(tax + ST_TAX_OCC, 16)) : 1.0;

    for (int j = lane; j < K; j += NL) {
        const uint32_t op = prog[j] >> 24, arg = prog[j] & 0xFFFFFFu;
        double v = 0.0;
        switch (op) {
            case MT_PRODUCTIVITY: v = sum_x; break;
            case MT_EQUALITY: v = 1.0 - gini; break;
            case MT_COIN_EQ_PROD: v = (1.0 - gini) * (sum_x / A); break;
            case MT_INV_W_COIN: v = inv_w_coin; break;
            case MT_INV_W_UTIL: v = inv_w_util; break;
            case MT_MEAN_COIN: v = sum_x / A; break;
            case MT_MEAN_LABOR: v = np_pairwise_sum(labor, A) / A; break;
            case MT_MEAN_UTIL: v = np_pairwise_sum(util, A) / A; break;
            case MT_COIN: v = x[arg]; break;
            case MT_INV: v = (double)(inv[arg] + esc[arg]); break;
            case MT_LABOR: v = labor[arg]; break;
            case MT_UTIL: v = util[arg]; break;
            case MT_WEIGHTED_COST: v = c.energy_cost * ew; break;
            case MT_WARMUP_INT: v = (double)hdr[HDR_AUTO_WARMUP]; break;
            case MT_N_BUILDS: v = stats[ST_BUILDS + arg]; break;
            case MT_TOTAL_BUILDS: v = houses; break;
            case MT_TRADE_AVG: v = stats[arg] == 0.0 ? met_nan() : stats[arg + 1] / stats[arg]; break;
            case MT_TRADE_N: v = stats[arg]; break;
            case MT_N_TRADES: v = stats[ST_N_TRADES]; break;
            case MT_BRACKET_RATE:
            case MT_BRACKET_OCC: {   // Python's sum() over the pooled brackets, in bracket order
                const double *src = tax + (op == MT_BRACKET_RATE ? ST_TAX_SCHED : ST_TAX_OCC);
                double s = 0.0;
                int nb = 0;
                for (int b = 0; b < 16; b++)
                    if ((arg >> b) & 1u) { s += src[b]; nb++; }
                if (op == MT_BRACKET_OCC) v = s / n_obs;
                else v = periods != 0.0 ? s / (periods * nb) : met_nan();
                break;
            }
            case MT_EFF_RATE: v = periods != 0.0 ? tax[ST_TAX_EFF_SUM] / (periods * A) : met_nan(); break;
            case MT_COLLECTED: v = tax[ST_TAX_COLLECTED]; break;
            case MT_TAX_POOREST: v = tax[ST_TAX_AGENT + A + poorest] / fmax(0.001, tax[ST_TAX_AGENT + poorest]); break;
            case MT_TAX_RICHEST: v = tax[ST_TAX_AGENT + A + richest] / fmax(0.001, tax[ST_TAX_AGENT + richest]); break;
            case MT_ZERO: v = 0.0; break;
            default: v = met_nan(); break;   // MT_NAN: filled by the caller
        }
        row[j] = v;
    }
}

#if !AIE_ON_DEVICE
// The same launch for a host build of the device source (the suite's 1-lane emulation, tests/emu): every env in turn, its
// warp's shared-memory staging filled with 0xFF (NaN) first, so that a read of staging the body never wrote shows.
static inline void metrics_env_host(const DevCfg &c, const uint8_t *recs, const uint32_t *prog, int K, int source, double *out) {
    double sm[MET_WARP_DOUBLES];
    for (int e = 0; e < c.n_envs; e++) {
        memset(sm, 0xFF, sizeof(sm));
        metrics_env(c, recs + (size_t)e * c.rec_bytes, prog, K, source, out + (size_t)e * K, sm, 0);
    }
}
#endif

}  // namespace aie
