// aie_covid_core.cuh — COVID-19 + economy scenario: one fused per-env step (device body).
//
// One CTA per env replica, one thread per US state (51) on the device; serial in the 1-lane host emulation
// used by the CPU tests (-DAIE_EMU).  Follows the reference's *Python* path operation by operation, including
// the places where numpy promotes float32 (x) int32 to float64 — annotated with "f64:" below:
//   ControlUSStateOpenCloseStatus.component_step   components/covid19_components.py:180-221
//   FederalGovernmentSubsidy.component_step        components/covid19_components.py:421-443
//   VaccinationCampaign.component_step             components/covid19_components.py:615-627
//   scenario_step / sir_step / unemployment_step / economy_step   scenarios/covid19/covid19_env.py:727-917,
//                                                                 1477-1515, 1374-1441, 1444-1475
//   generate_observations (+ component obs, masks) covid19_env.py:919-993; covid19_components.py:97-108, 223-238,
//                                                  316-325, 445-462, 629-663
//   compute_reward                                 covid19_env.py:1047-1173
#pragma once
#include <math.h>
#include <stdint.h>

#include "aie_core.cuh"   // policy_segment_warp, PolicyBufs

#if defined(__CUDACC__) && !defined(AIE_EMU)
#define CV_DEV __device__ __forceinline__
#define CV_ON_DEVICE 1
#else
#define CV_DEV static inline
#define CV_ON_DEVICE 0
#endif

namespace aie {

struct CovidCfg {
    int32_t S, T, levels, cooldown, sub_interval, sub_levels, vac_begin, vac_interval, t_first_delivery;
    int32_t beta_delay, L, F, sdi, rw_days, value_of_life, auto_reset, n_envs;
    float gamma, death_rate, sick_rate, p1865, rfr, crra_eta;
    float planner_health_norm, planner_econ_norm, min_ph, max_ph, min_pe, max_pe, w_ph, w_pe;
    double reward_norm, time_scale;
    // device copies of the fitted parameters
    const int32_t *pop, *vac_per_delivery;
    const float *beta_slopes, *beta_intercepts, *unemp_bias, *max_prod, *health_norm, *econ_norm, *min_ah, *max_ah,
        *min_ae, *max_ae, *w_ah, *w_ae, *conv_w, *conv_filt, *init_state;
    float dppw;
    const double *max_daily_subsidy;
    const int8_t *rw_policy;
};

struct CovidBufs {
    float *state; int32_t *ints; int32_t *hdr; int8_t *ring;
    const int32_t *act_a, *act_p;
    float *o_state, *o_post, *o_lag, *o_pol, *o_scal, *mask_a, *mask_p, *rew_a;
    double *rew_p;
    int32_t *done;
    // optional persistent per-state list of the stringency changes inside the history window (NULL: scan the history):
    // uint32 [E][CV_LIST_CAP + 1][S], entry-major so that an env's S threads read coalesced.  Row 0 = head | count << 8
    // (count 255: the list overflowed, this state scans its history again); rows 1.. = ring of
    // (day the newer value was appended + 2^20) | (change + 128) << 24, oldest first.
    uint32_t *chg;
};
constexpr int CV_LIST_CAP = 32;
constexpr uint32_t CV_LIST_DAY0 = 1u << 20;

enum { CVS_S = 0, CVS_I, CVS_R, CVS_D, CVS_V, CVS_U, CVS_STRG, CVS_SUBSIDY, CVS_POST, CVS_FIELDS = 9 };
enum { CVH_T = 0, CVH_SUBSIDY_LEVEL, CVH_RING_HEAD, CVH_EPISODES };

// Episode-metric accumulators (aie_covid_bind_metrics), caller-owned, two blocks per replica:
//   sums  float64 [E][CVM_SUMS][S]: sums over t = 1..t of the float32 Unemployed, Stringency Level, Postsubsidy
//         Productivity and Subsidy the step stores (the reference's global_state[...][1:] time aggregates)
//   index float32 [E][2][S + 1]: Health Index, Economic Index of each state, then the planner's, summed as the reference
//         sums them (covid19_env.py:1124-1125, 1160-1161)
//   end   float32 [E][4][S] (previous block only): I, R, D, V of the state the episode ended in
// The current block is zeroed by aie_covid_reset and by the step that ends an episode, after copying it to the previous.
enum { CVM_U = 0, CVM_STRG, CVM_POST, CVM_SUBSIDY, CVM_SUMS = 4 };
constexpr int CVM_PER_STATE = 8, CVM_USA = 7;   // metric columns: 8 per state, then 7 for the USA
struct CovidStats {
    double *sums, *prev_sums;
    float *index, *prev_index, *prev_end;
    double us_pop;
};

#if CV_ON_DEVICE
CV_DEV void cv_bsync() { __syncthreads(); }
#else
CV_DEV void cv_bsync() {}
#endif

// numpy's float32 pairwise sum for n < 128: 8 interleaved accumulators, tree-combined, sequential tail
CV_DEV float np_sum_f32(const float *a, int n) {
    if (n < 8) { float r = 0.f; for (int i = 0; i < n; i++) r += a[i]; return r; }
    float r[8];
    for (int j = 0; j < 8; j++) r[j] = a[j];
    int i;
    for (i = 8; i < n - (n % 8); i += 8)
        for (int j = 0; j < 8; j++) r[j] += a[i + j];
    float res = ((r[0] + r[1]) + (r[2] + r[3])) + ((r[4] + r[5]) + (r[6] + r[7]));
    for (; i < n; i++) res += a[i];
    return res;
}

// x ** (1 - eta) as numpy evaluates it for float32 (scalar-exponent fast paths: reciprocal, square, sqrt)
CV_DEV float cv_pow(float x, float e) {
    if (e == -1.0f) return 1.0f / x;
    if (e == 2.0f) return x * x;
    if (e == 0.5f) return sqrtf(x);
    if (e == 1.0f) return x;
    if (e == 0.0f) return 1.0f;
    return powf(x, e);
}
CV_DEV float cv_crra(float x, float eta) {  // covid19_env.py:1053-1058 (float32 throughout)
    float ax = 365.0f * x;
    float axc = fminf(fmaxf(ax, 0.1f), 3.0f);
    float one_m = 1.0f - eta;
    float annual = 1.0f + (cv_pow(axc, one_m) - 1.0f) / one_m;
    return annual / 365.0f;
}
CV_DEV float cv_minmax(float x, float lo, float hi) { return (x - lo) / ((hi - lo) + 1e-10f); }

// Stringency history: int8 [S][ROW] per env, time-minor (ROW = L+1 rounded up to 16 bytes) so that one state's
// history is contiguous and can be scanned with 16-byte loads.  Logical index k (0 = oldest) lives at physical
// column (head + k) mod (L+1).
struct alignas(16) cv_b16 { int8_t b[16]; };
CV_DEV int cv_ring_row(int L1) { return (L1 + 15) & ~15; }
CV_DEV int8_t cv_ring_at(const int8_t *ring, int head, int k, int L1, int S, int a) {
    int p = head + k;
    if (p >= L1) p -= L1;
    return ring[(size_t)a * cv_ring_row(L1) + p];
}

// Observations + masks of the current state (used after a step and after a reset).  OT: the element type of the seven
// observation / mask tensors (float, or bf16_t under AIE_OBS_BF16): every value is computed as for float32 output and
// rounded float32 -> bfloat16 on the way out (put_out), so a float64 intermediate is rounded to float32 first.
template <typename OT = float>
CV_DEV void covid_observe(const CovidCfg &c, const float *st, const int32_t *ints, const int32_t *hdr, const int8_t *ring,
                          int head, int e, const CovidBufs &b, int tid, int nthr) {
    // Each value is computed before its destination address, the order of the float32 assignments this replaced.
    const int S = c.S, L1 = c.L + 1, t = hdr[CVH_T];
    for (int a = tid; a < S; a += nthr) {
        const double pop = (double)c.pop[a];
        for (int k = 0; k < 6; k++) {  // f64: float32 state / int32 population
            const float v = (float)((double)st[k * S + a] / pop);
            put_out((OT *)b.o_state + ((size_t)e * 6 + k) * S + a, v);
        }
        const float post = st[CVS_POST * S + a] / c.max_prod[a];
        put_out((OT *)b.o_post + (size_t)e * S + a, post);
        const float lag = (float)cv_ring_at(ring, head, c.L - c.beta_delay + 1, L1, S, a);
        const float lag_v = lag / (float)c.levels;
        put_out((OT *)b.o_lag + (size_t)e * S + a, lag_v);
        const float pol = st[CVS_STRG * S + a] / (float)c.levels;
        put_out((OT *)b.o_pol + (size_t)e * S + a, pol);
        const float open = (t >= ints[a]) ? 1.0f : 0.0f;  // cooldown_until
        OT *m = (OT *)b.mask_a + (size_t)e * (1 + c.levels) * S;
        put_out(m + a, 1.0f);
        for (int l = 1; l <= c.levels; l++) put_out(m + (size_t)l * S + a, open);
    }
    for (int j = tid; j <= c.sub_levels; j += nthr) {
        const float v = (j == 0 || (t % c.sub_interval) == 0) ? 1.0f : 0.0f;
        put_out((OT *)b.mask_p + (size_t)e * (1 + c.sub_levels) + j, v);
    }
    if (tid == 0) {
        OT *sc = (OT *)b.o_scal + (size_t)e * 4;
        const float s0 = (float)((double)t / c.time_scale);
        put_out(sc + 0, s0);
        const float s1 = (float)((double)(c.sub_interval - t % c.sub_interval) / (double)c.sub_interval);
        put_out(sc + 1, s1);
        const float s2 = (float)((double)hdr[CVH_SUBSIDY_LEVEL] / (double)c.sub_levels);
        put_out(sc + 2, s2);
        const int nxt = t + 1;
        double tv;
        if (nxt <= c.t_first_delivery) tv = fmin(1.0, (double)(c.t_first_delivery - nxt) / (double)c.vac_interval);
        else tv = (double)(c.vac_interval - nxt % c.vac_interval);
        const float s3 = (float)(tv / (double)c.vac_interval);
        put_out(sc + 3, s3);
    }
}

// env.reset(): covid19_env.py:1175-1290 (deterministic: initial series from the real-world data at start_date)
template <typename OT = float>
CV_DEV void covid_reset_env(const CovidCfg &c, int e, const CovidBufs &b, int tid, int nthr, bool keep_outputs) {
    const int S = c.S, L1 = c.L + 1;
    float *st = b.state + (size_t)e * CVS_FIELDS * S;
    int32_t *ints = b.ints + (size_t)e * 2 * S;
    int32_t *hdr = b.hdr + (size_t)e * 4;
    int8_t *ring = b.ring + (size_t)e * cv_ring_row(L1) * S;
    for (int a = tid; a < S; a += nthr) {
        for (int k = 0; k < 6; k++) st[k * S + a] = c.init_state[k * S + a];
        st[CVS_STRG * S + a] = (float)c.rw_policy[(size_t)c.sdi * S + a];
        st[CVS_SUBSIDY * S + a] = 0.0f;
        st[CVS_POST * S + a] = 0.0f;
        ints[a] = 0; ints[S + a] = 0;
        // stringency history = real-world policy up to the start date, padded with 1 before the data begins
        for (int k = 0; k < L1; k++) {
            const int day = c.sdi - c.L + k;
            ring[(size_t)a * cv_ring_row(L1) + k] = day < 0 ? (int8_t)1 : c.rw_policy[(size_t)day * S + a];
        }
        if (!keep_outputs) b.rew_a[(size_t)e * S + a] = 0.0f;
        if (b.chg) {  // the changes already inside the initial window; pair (k, k + 1) reaches index k - t at step t
            uint32_t *col = b.chg + (size_t)e * (CV_LIST_CAP + 1) * S + a;
            const int8_t *row = ring + (size_t)a * cv_ring_row(L1);
            int cnt = 0;
            for (int k = 0; k < c.L && cnt != 255; k++) {
                const int d = (int)row[k + 1] - (int)row[k];
                if (d == 0) continue;
                if (cnt == CV_LIST_CAP) { cnt = 255; break; }
                col[(size_t)(1 + cnt) * S] = (uint32_t)((int)CV_LIST_DAY0 + k - (c.L - 1)) | ((uint32_t)(d + 128) << 24);
                cnt++;
            }
            col[0] = (uint32_t)cnt << 8;
        }
    }
    cv_bsync();
    if (tid == 0) {
        const int episodes = hdr[CVH_EPISODES];
        hdr[CVH_T] = 0; hdr[CVH_SUBSIDY_LEVEL] = 0; hdr[CVH_RING_HEAD] = 0;
        hdr[CVH_EPISODES] = keep_outputs ? episodes + 1 : 0;
        if (!keep_outputs) { b.rew_p[e] = 0.0; b.done[e] = 0; }
    }
    cv_bsync();
    covid_observe<OT>(c, st, ints, hdr, ring, 0, e, b, tid, nthr);
}

// red: scratch float [3][S] (shared memory on the device)
// acc += sum over the listed changes (k, d), in list order, of d * w_f * filter_f[k] for f = 0..F-1 (f64 like the reference)
CV_DEV double cv_accumulate_changes(const CovidCfg &c, const uint32_t *lst, int n, const double *wf, double acc) {
    for (int i = 0; i < n; i++) {
        const int k = (int)(lst[i] & 0xFFFFu), d = (int)(lst[i] >> 16) - 128;
#if CV_ON_DEVICE
#pragma unroll
#endif
        for (int f = 0; f < 8; f++)   // F <= 8 (checked at creation); unrolled so wf[] stays in registers
            if (f < c.F) acc += ((double)d * wf[f]) * (double)c.conv_filt[f * c.L + k];
    }
    return acc;
}

// chg: scratch uint32 [nthr][CV_CHG_CAP] (shared memory on the device): per-state list of the stringency changes in
// the history window
constexpr int CV_CHG_CAP = 32;
// FINAL: on the step that ends an episode under the auto-reset, first write the observations / masks of the state the
// episode ended in into row e of fin's seven observation / mask tensors (fin: b with those pointers replaced), then
// reset.  Unused without FINAL.  OT: the element type of the observation / mask tensors (covid_observe).
// STATS: add this step's values to the current block of *ms (CovidStats); on the step that ends an episode under the
// auto-reset, write the sums with this step's values to the previous block, with the end state, and zero the current
// one.  Each state's thread owns its columns and thread 0 the planner's, so no reduction across states.  ms is unused
// without STATS.
// SLOT (a step of a captured rollout, aie_rollout_capture_begin): fin's pointers are at row 0 of a bound rollout's final
// slots and done0 at slot 0 of its done flags; the step that ends an episode (known from the record's own t) writes its
// final observations into row (k, e), k = the replica's done flags in slots 0 .. s - 1, when k < nk.  Nothing here
// depends on a host-side timestep or episode count, so a replay at any point of the episode writes the right row.
template <bool FINAL, typename OT = float, bool STATS = false, bool SLOT = false>
CV_DEV void covid_step_env(const CovidCfg &c, int e, const CovidBufs &b, const CovidBufs &fin, float *red, uint32_t *chg,
                           int tid, int nthr, const CovidStats *ms = nullptr, const int32_t *done0 = nullptr, int s = 0,
                           int nk = 0) {
    const int S = c.S, L = c.L, L1 = c.L + 1, F = c.F;
    float *st = b.state + (size_t)e * CVS_FIELDS * S;
    int32_t *ints = b.ints + (size_t)e * 2 * S;
    int32_t *hdr = b.hdr + (size_t)e * 4;
    int8_t *ring = b.ring + (size_t)e * cv_ring_row(L1) * S;
    const int t = hdr[CVH_T] + 1;
    const int head = hdr[CVH_RING_HEAD];                  // physical row of the oldest history entry
    const int new_head = head + 1 == L1 ? 0 : head + 1;
    // FederalGovernmentSubsidy: the level changes on the first day of each interval (covid19_components.py:421-433)
    const int act_p = b.act_p ? b.act_p[e] : 0;
    int level = hdr[CVH_SUBSIDY_LEVEL];
    if ((t - 1) % c.sub_interval == 0) level = (act_p < 0 || act_p > c.sub_levels) ? 0 : act_p;
    const double level_frac = (double)level / (double)c.sub_levels;
    const bool vac_day = t >= c.vac_begin && (t % c.vac_interval) == 0;
    float *red_md = red, *red_sub = red + S, *red_post = red + 2 * S;
    cv_bsync();  // every thread has read the header before thread 0 rewrites it below
    for (int a = tid; a < S; a += nthr) {
        // ControlUSStateOpenCloseStatus (covid19_components.py:180-221)
        int action = b.act_a[(size_t)e * S + a];
        if (action < 0 || action > c.levels) action = 0;
        const float strg_prev = st[CVS_STRG * S + a];   // == the newest history entry
        const float strg = strg_prev * (action == 0 ? 1.0f : 0.0f) + (float)action;
        st[CVS_STRG * S + a] = strg;
        if (t == ints[a] + 1) ints[a] += (action == 0) ? 1 : c.cooldown;
        // subsidy for this state (f64 product stored into the float32 series)
        const float subsidy = (float)(level_frac * c.max_daily_subsidy[a]);
        st[CVS_SUBSIDY * S + a] = subsidy;
        // VaccinationCampaign (covid19_components.py:615-627): deliveries accumulate, scenario_step consumes them
        int vacc = ints[S + a] + (vac_day ? c.vac_per_delivery[a] : 0);
        ints[S + a] = 0;
        // stringency history: drop the oldest entry, append today's level (covid19_env.py:1412-1420)
        ring[(size_t)a * cv_ring_row(L1) + head] = (int8_t)strg;
        // ---- sir_step (covid19_env.py:1477-1515) ----
        const double tmk = (double)(int)cv_ring_at(ring, new_head, L - c.beta_delay, L1, S, a);
        const float beta_i = (float)((double)c.beta_intercepts[a] + (double)c.beta_slopes[a] * tmk);  // f64: f32 * int32
        const float S_tm1 = st[CVS_S * S + a], I_tm1 = st[CVS_I * S + a], R_tm1 = st[CVS_R * S + a], V_tm1 = st[CVS_V * S + a];
        const float D_tm1 = st[CVS_D * S + a];
        const float frac_vacc = (float)fmin(1.0, (double)vacc / (double)(S_tm1 + 1e-10f));           // f64: int32 / f32
        const double vaccinated = fmin((double)vacc, (double)S_tm1);
        const double si_over_n = ((double)S_tm1 / (double)c.pop[a]) * (double)I_tm1;                  // f64: f32 / int32
        const float dS = (float)(((double)(-beta_i) * si_over_n) * (double)(1.0f - frac_vacc) - vaccinated);
        const float dR = (float)((double)(c.gamma * I_tm1) + vaccinated);
        const float dI = -dS - dR;
        const float dV = (float)vaccinated;
        const float S_t = fmaxf(S_tm1 + dS, 0.0f), I_t = fmaxf(I_tm1 + dI, 0.0f), R_t = fmaxf(R_tm1 + dR, 0.0f);
        const float V_t = fmaxf(V_tm1 + dV, 0.0f);
        const float D_t = c.death_rate * (R_t - V_t);
        // ---- unemployment_step (covid19_env.py:1374-1441): discounted sum of past stringency changes (f64) ----
        // The row is scanned in PHYSICAL order with 16-byte loads; the pair (p, p+1 mod L1) is the stringency change
        // at logical index k = (p - new_head) mod L1, and k == L is the seam between newest and oldest (skipped).
        double acc = 0.0;
        bool scan = true;
        if (b.chg) {
            // Persistent change list: a change appended on day tc sits at window index L - 1 - (t - tc); entries leave
            // at the front when that index drops below 0.  Same (index, change) pairs as the scan finds, accumulated
            // oldest first.  O(changes) instead of O(filter_len) per state and step.
            uint32_t *col = b.chg + (size_t)e * (CV_LIST_CAP + 1) * S + a;
            const uint32_t hd = col[0];
            int lhead = (int)(hd & 0xFFu), cnt = (int)((hd >> 8) & 0xFFu);
            if (cnt != 255) {
                const int d_new = (int)strg - (int)strg_prev;
                if (d_new != 0) {
                    if (cnt == CV_LIST_CAP) cnt = 255;
                    else {
                        int slot = lhead + cnt; if (slot >= CV_LIST_CAP) slot -= CV_LIST_CAP;
                        col[(size_t)(1 + slot) * S] = (CV_LIST_DAY0 + (uint32_t)t) | ((uint32_t)(d_new + 128) << 24);
                        cnt++;
                    }
                }
            }
            if (cnt != 255) {
                uint32_t *my_chg = chg + (size_t)tid * CV_CHG_CAP;
                double wf[8];
                for (int f = 0; f < 8; f++) wf[f] = f < F ? (double)c.conv_w[a * F + f] : 0.0;
                int n_chg = 0, drop = 0;
                for (int i = 0; i < cnt; i++) {
                    int slot = lhead + i; if (slot >= CV_LIST_CAP) slot -= CV_LIST_CAP;
                    const uint32_t en = col[(size_t)(1 + slot) * S];
                    const int tc = (int)(en & 0xFFFFFFu) - (int)CV_LIST_DAY0, d = (int)(en >> 24) - 128;
                    const int k = L - 1 - (t - tc);
                    if (k < 0) { drop++; continue; }   // (oldest first: only leading entries can have left the window)
                    my_chg[n_chg++] = (uint32_t)k | ((uint32_t)(d + 128) << 16);
                }
                acc = cv_accumulate_changes(c, my_chg, n_chg, wf, 0.0);
                lhead += drop; if (lhead >= CV_LIST_CAP) lhead -= CV_LIST_CAP;
                cnt -= drop;
                scan = false;
            }
            col[0] = (uint32_t)lhead | ((uint32_t)cnt << 8);
        }
        if (scan) {
            const int8_t *row = ring + (size_t)a * cv_ring_row(L1);
            int prev = row[L1 - 1];                       // predecessor of physical column 0
            uint32_t *my_chg = chg + (size_t)tid * CV_CHG_CAP;
            int n_chg = 0;
            double wf[8];                                 // this state's filter weights (F <= 8), widened once
            for (int f = 0; f < 8; f++) wf[f] = f < F ? (double)c.conv_w[a * F + f] : 0.0;
#if CV_ON_DEVICE
            int4 nxt = *(const int4 *)row;                // software pipeline: the next 16 columns are always in flight
#endif
            for (int p0 = 0; p0 < L1; p0 += 16) {
#if CV_ON_DEVICE
                union { int4 v; int8_t b[16]; uint32_t w32[4]; } ld;
                ld.v = nxt;
                if (p0 + 16 < L1) nxt = *(const int4 *)(row + p0 + 16);   // rows are padded to 16 bytes (LDG.128)
#else
                cv_b16 ld = *(const cv_b16 *)(row + p0);
#endif
                const int8_t *chunk = ld.b;
                // Stringency changes are rare (an action every cooldown period at most): a 4-column word that equals
                // itself shifted by one column (with the previous column shifted in) holds no change and is skipped.
#if CV_ON_DEVICE
#pragma unroll
#endif
                for (int wj = 0; wj < 4; wj++) {
                    const int pw = p0 + 4 * wj;
                    if (pw >= L1) break;
#if CV_ON_DEVICE
                    const uint32_t w = ld.w32[wj];
#else
                    const uint32_t w = (uint32_t)(uint8_t)chunk[4 * wj] | ((uint32_t)(uint8_t)chunk[4 * wj + 1] << 8) |
                                       ((uint32_t)(uint8_t)chunk[4 * wj + 2] << 16) | ((uint32_t)(uint8_t)chunk[4 * wj + 3] << 24);
#endif
                    if (pw + 4 <= L1 && w == ((w << 8) | (uint32_t)(uint8_t)prev)) { prev = (int)(int8_t)(w >> 24); continue; }
                    for (int j = 4 * wj; j < 4 * wj + 4; j++) {
                        const int p = p0 + j;
                        if (p >= L1) break;
                        const int cur = chunk[j];
                        const int d = cur - prev;             // change between physical columns p-1 and p
                        prev = cur;
                        if (d != 0) {
                            int k = (p - 1) - new_head;       // logical index of the older element of the pair
                            if (k < 0) k += L1;
                            if (k < L) {
                                // Changes are first collected (in scan order) and accumulated afterwards: the states of a
                                // warp change on different days, and accumulating inside the scan would run the body once
                                // per distinct day of the whole warp instead of once per change of the busiest state.
                                if (n_chg == CV_CHG_CAP) { acc = cv_accumulate_changes(c, my_chg, n_chg, wf, acc); n_chg = 0; }
                                my_chg[n_chg++] = (uint32_t)k | ((uint32_t)(d + 128) << 16);
                            }
                        }
                    }
                }
            }
            acc = cv_accumulate_changes(c, my_chg, n_chg, wf, acc);
        }
        const double excess = (acc <= 20.0) ? log(1.0 + exp(acc)) : acc;  // softplus, beta = 1, threshold = 20
        const double unemployed = (excess + (double)c.unemp_bias[a]) * (double)c.pop[a] / 100.0;
        // ---- economy_step (covid19_env.py:1444-1475) ----
        const float incapacitated = (c.sick_rate * I_t) + D_t;
        const double cant_work = (double)(incapacitated * c.p1865) + unemployed;
        const double can_work = fmax(0.0, (double)c.pop[a] * (double)c.p1865 - cant_work);           // f64: int32 * f32
        const float productivity = (float)(can_work * (double)c.dppw);
        const float post = productivity + subsidy;
        st[CVS_S * S + a] = S_t; st[CVS_I * S + a] = I_t; st[CVS_R * S + a] = R_t; st[CVS_D * S + a] = D_t;
        st[CVS_V * S + a] = V_t; st[CVS_U * S + a] = (float)unemployed; st[CVS_POST * S + a] = post;
        // ---- agent reward (covid19_env.py:1083-1130) ----
        const float md = D_t - D_tm1;
        float h = (float)(((double)(-md) * (double)c.value_of_life) / (double)c.health_norm[a]);      // f64: f32 * int32
        float ec = cv_crra(post / c.econ_norm[a], c.crra_eta);
        h = cv_minmax(h, c.min_ah[a], c.max_ah[a]);
        ec = cv_minmax(ec, c.min_ae[a], c.max_ae[a]);
        const float wh = c.w_ah[a], we = c.w_ae[a];
            b.rew_a[(size_t)e * S + a] = (((wh * h) + (we * ec)) / (wh + we)) / (float)c.reward_norm;
        red_md[a] = md; red_sub[a] = subsidy; red_post[a] = post;
        if (STATS) {
            double *cs = ms->sums + (size_t)e * CVM_SUMS * S + a;
            float *ci = ms->index + (size_t)e * 2 * (S + 1) + a;
            const double su = cs[CVM_U * S] + (double)(float)unemployed, sg = cs[CVM_STRG * S] + (double)strg;
            const double sp = cs[CVM_POST * S] + (double)post, ss = cs[CVM_SUBSIDY * S] + (double)subsidy;
            const float ih = ci[0] + h, ie = ci[S + 1] + ec;
            if (c.auto_reset && t >= c.T) {
                double *ps = ms->prev_sums + (size_t)e * CVM_SUMS * S + a;
                float *pi = ms->prev_index + (size_t)e * 2 * (S + 1) + a, *pe = ms->prev_end + (size_t)e * 4 * S + a;
                ps[CVM_U * S] = su; ps[CVM_STRG * S] = sg; ps[CVM_POST * S] = sp; ps[CVM_SUBSIDY * S] = ss;
                pi[0] = ih; pi[S + 1] = ie;
                pe[0] = I_t; pe[S] = R_t; pe[2 * S] = D_t; pe[3 * S] = V_t;
                cs[CVM_U * S] = 0.0; cs[CVM_STRG * S] = 0.0; cs[CVM_POST * S] = 0.0; cs[CVM_SUBSIDY * S] = 0.0;
                ci[0] = 0.0f; ci[S + 1] = 0.0f;
            } else {
                cs[CVM_U * S] = su; cs[CVM_STRG * S] = sg; cs[CVM_POST * S] = sp; cs[CVM_SUBSIDY * S] = ss;
                ci[0] = ih; ci[S + 1] = ie;
            }
        }
    }
    cv_bsync();
    if (tid == 0) {
        // ---- planner reward (covid19_env.py:1132-1171) ----
        const float sum_md = np_sum_f32(red_md, S), sum_sub = np_sum_f32(red_sub, S), sum_post = np_sum_f32(red_post, S);
        double ph = ((double)(-sum_md) * (double)c.value_of_life) / (double)c.planner_health_norm;   // f64: f32 * int32 scalars
        const float cost = (1.0f + c.rfr) * sum_sub;
        float pe = cv_crra((sum_post - cost) / c.planner_econ_norm, c.crra_eta);
        ph = (ph - (double)c.min_ph) / (double)((c.max_ph - c.min_ph) + 1e-10f);
        pe = cv_minmax(pe, c.min_pe, c.max_pe);
        const double num = (double)c.w_ph * ph + (double)(c.w_pe * pe);
        b.rew_p[e] = (num / (double)(c.w_ph + c.w_pe)) / c.reward_norm;
        if (STATS) {   // the planner's float32 indices; ph is float64 there (covid19_env.py:1160-1161)
            float *ci = ms->index + (size_t)e * 2 * (S + 1);
            const float ih = (float)((double)ci[S] + ph), ie = ci[2 * S + 1] + pe;
            if (c.auto_reset && t >= c.T) {
                float *pi = ms->prev_index + (size_t)e * 2 * (S + 1);
                pi[S] = ih; pi[2 * S + 1] = ie;
                ci[S] = 0.0f; ci[2 * S + 1] = 0.0f;
            } else {
                ci[S] = ih; ci[2 * S + 1] = ie;
            }
        }
        b.done[e] = t >= c.T ? 1 : 0;
        hdr[CVH_T] = t; hdr[CVH_SUBSIDY_LEVEL] = level; hdr[CVH_RING_HEAD] = new_head;
    }
    cv_bsync();
    if (SLOT) {
        const bool end = c.auto_reset && t >= c.T;   // uniform across the CTA: t is the replica's
        int k = 0;
        if (end) {
#if CV_ON_DEVICE
            for (int t0 = 0; t0 < s; t0 += nthr) {
                const int u = t0 + tid;
                k += __syncthreads_count(u < s && done0[(size_t)u * c.n_envs + e] != 0);
            }
#else
            for (int u = 0; u < s; u++) k += done0[(size_t)u * c.n_envs + e] != 0;
#endif
        }
        if (end && k < nk) {
            covid_observe<OT>(c, st, ints, hdr, ring, new_head, k * c.n_envs + e, fin, tid, nthr);
            cv_bsync();   // the reset below overwrites what the final pass reads
        }
        if (end) covid_reset_env<OT>(c, e, b, tid, nthr, true);
        else covid_observe<OT>(c, st, ints, hdr, ring, new_head, e, b, tid, nthr);
    } else if (FINAL) {
        // One observation pass whose destination is chosen per step: a second inlined pass for the ending step made
        // the ordinary steps of this kernel 7.7 % slower on an H100 (the code ptxas makes of the whole body); this form
        // leaves them unchanged (DESIGN §6).
        const bool end = c.auto_reset && t >= c.T;
        covid_observe<OT>(c, st, ints, hdr, ring, new_head, e, end ? fin : b, tid, nthr);
        if (end) {
            cv_bsync();   // once per episode: the reset below overwrites what the final pass reads
            covid_reset_env<OT>(c, e, b, tid, nthr, true);
        }
    } else if (c.auto_reset && t >= c.T) covid_reset_env<OT>(c, e, b, tid, nthr, true);
    else covid_observe<OT>(c, st, ints, hdr, ring, new_head, e, b, tid, nthr);
}
// The step without final observations (aie_covid_step).
CV_DEV void covid_step_env(const CovidCfg &c, int e, const CovidBufs &b, float *red, uint32_t *chg, int tid, int nthr) {
    covid_step_env<false>(c, e, b, b, red, chg, tid, nthr);
}

// aie_covid_reset with metrics bound: the current block starts from zero.
CV_DEV void covid_zero_stats(const CovidCfg &c, int e, const CovidStats &ms, int tid, int nthr) {
    const int S = c.S;
    for (int i = tid; i < CVM_SUMS * S; i += nthr) ms.sums[(size_t)e * CVM_SUMS * S + i] = 0.0;
    for (int i = tid; i < 2 * (S + 1); i += nthr) ms.index[(size_t)e * 2 * (S + 1) + i] = 0.0f;
}

// One row of aie_covid_episode_metrics: CovidAndEconomySimulation.scenario_metrics() (covid19_env.py:1613-1687) from an
// end state `end` (float32 [4][S]: I, R, D, V), the time sums `sums` ([CVM_SUMS][S]) and the indices `index`
// ([2][S + 1]).  Columns: 8 per state (CVM_PER_STATE), then the 7 USA columns.  Means over time divide by
// episode_length (the reference's global_state rows 1..episode_length, zero after t).  Every value is one float64
// expression in a fixed order; the USA sums run over the states in index order on thread 0.
CV_DEV void covid_metrics_row(const CovidCfg &c, const float *end, const double *sums, const float *index, double us_pop,
                              double *row, int tid, int nthr) {
    const int S = c.S;
    const double T = (double)c.T;
    for (int a = tid; a < S; a += nthr) {
        double *r = row + (size_t)a * CVM_PER_STATE;
        r[0] = (double)(int32_t)end[a] / 1e6;           // Total Infected / Recovered / Deaths: int32 casts
        r[1] = (double)(int32_t)end[S + a] / 1e6;
        r[2] = (double)(int32_t)end[2 * S + a] / 1e6;
        r[3] = ((sums[CVM_U * S + a] / T) / (double)c.pop[a]) * 100.0;
        r[4] = sums[CVM_STRG * S + a] / T;
        r[5] = sums[CVM_POST * S + a] / 1e9;
        r[6] = (double)index[a];
        r[7] = (double)index[S + 1 + a];
    }
    if (tid == 0) {
        double v = 0.0, d = 0.0, u = 0.0, sub = 0.0, post = 0.0;
        for (int a = 0; a < S; a++) {
            v += (double)end[3 * S + a]; d += (double)end[2 * S + a];
            u += sums[CVM_U * S + a]; sub += sums[CVM_SUBSIDY * S + a]; post += sums[CVM_POST * S + a];
        }
        double *r = row + (size_t)S * CVM_PER_STATE;
        r[0] = (v / us_pop) * 100.0;
        r[1] = d / 1e3;
        r[2] = ((u / us_pop) / T) * 100.0;
        r[3] = sub / 1e12;
        r[4] = post / 1e12;
        r[5] = (double)index[S];
        r[6] = (double)index[2 * S + 1];
    }
}
// source 0: the current block and the live state of replica e; 1: the previous block and its end state
CV_DEV void covid_metrics_env(const CovidCfg &c, int e, const CovidBufs &b, const CovidStats &ms, int source, double *out,
                              int tid, int nthr) {
    const int S = c.S;
    const size_t K = (size_t)S * CVM_PER_STATE + CVM_USA;
    const float *end = source ? ms.prev_end + (size_t)e * 4 * S : b.state + (size_t)e * CVS_FIELDS * S + CVS_I * S;
    const double *sums = (source ? ms.prev_sums : ms.sums) + (size_t)e * CVM_SUMS * S;
    const float *index = (source ? ms.prev_index : ms.index) + (size_t)e * 2 * (S + 1);
    covid_metrics_row(c, end, sums, index, ms.us_pop, out + (size_t)e * K, tid, nthr);
}

// Random policy: uniform over the unmasked actions (NO-OP is always open).
CV_DEV uint64_t cv_mix64(uint64_t x) {
    x += 0x9e3779b97f4a7c15ull;
    x = (x ^ (x >> 30)) * 0xbf58476d1ce4e5b9ull;
    x = (x ^ (x >> 27)) * 0x94d049bb133111ebull;
    return x ^ (x >> 31);
}
// MT: the element type of the masks (float, or bf16_t under AIE_OBS_BF16).
template <typename MT = float>
CV_DEV void covid_sample_env(const CovidCfg &c, int e, const CovidBufs &b, uint64_t key, int tid, int nthr) {
    const int S = c.S;
    int32_t *act_a = const_cast<int32_t *>(b.act_a) + (size_t)e * S;
    for (int a = tid; a < S; a += nthr) {
        const bool open = mask_open(((const MT *)b.mask_a)[((size_t)e * (1 + c.levels) + 1) * S + a]);
        const uint32_t r = (uint32_t)(cv_mix64(key + 0x100 * (uint64_t)a) >> 32);
        act_a[a] = open ? (int32_t)(r % (uint32_t)(1 + c.levels)) : 0;
    }
    if (tid == 0) {
        const bool open = mask_open(((const MT *)b.mask_p)[(size_t)e * (1 + c.sub_levels) + 1]);
        const uint32_t r = (uint32_t)(cv_mix64(key ^ 0xabcdefull) >> 32);
        const_cast<int32_t *>(b.act_p)[e] = open ? (int32_t)(r % (uint32_t)(1 + c.sub_levels)) : 0;
    }
}

// Policy sampler (aie_covid_sample_policy, policy_segment_warp in aie_core.cuh): unit u < S draws state u's stringency
// level from its logits [E][S][1 + levels] under the mask column mask_a[e][.][u]; unit S draws the planner's subsidy
// level from [E][1 + sub_levels].  Keys as covid_sample_env: key + 0x100 * u for a state, key ^ 0xabcdef for the planner.
// LT: the logits' element type; MT: the masks' (float, or bf16_t under AIE_OBS_BF16).
template <typename LT, typename MT = float>
CV_DEV void covid_policy_unit(const CovidCfg &c, int e, const CovidBufs &b, const PolicyBufs &p, uint64_t key, int u, int lane) {
    float lp;
    if (u < c.S) {
        const int n = 1 + c.levels;
        const size_t i = (size_t)e * c.S + u;
        const int v = policy_segment_warp((const MT *)b.mask_a + (size_t)e * n * c.S + u, c.S, (const LT *)p.a_logit + i * n, n,
                                          key + 0x100 * (uint64_t)u, p.greedy, lane, &lp);
        if (lane == 0) { const_cast<int32_t *>(b.act_a)[i] = v; if (p.lp_a) p.lp_a[i] = lp; }
    } else {
        const int n = 1 + c.sub_levels;
        const int v = policy_segment_warp((const MT *)b.mask_p + (size_t)e * n, 1, (const LT *)p.p_logit + (size_t)e * n, n,
                                          key ^ 0xabcdefull, p.greedy, lane, &lp);
        if (lane == 0) { const_cast<int32_t *>(b.act_p)[e] = v; if (p.lp_p) p.lp_p[e] = lp; }
    }
}

// Evaluation of stored actions (aie_covid_evaluate_policy, policy_segment_eval in aie_core.cuh): unit u < S is state u
// of row r, its logits [N][S][1 + levels] read against the mask column mask_a[r][.][u]; unit S is the planner, logits
// [N][1 + sub_levels].  Actions [N][S] and [N].
template <bool BWD, typename MT, typename LT>
CV_DEV void covid_policy_eval_unit(const CovidCfg &c, const PolicyEvalBufs &p, long long r, int u, int lane) {
    if (u < c.S) {
        const int n = 1 + c.levels;
        const size_t i = (size_t)r * c.S + u;
        policy_eval_slot<BWD, MT, LT>((const MT *)p.a_mask + (size_t)r * n * c.S + u, c.S, p.a_logit, n, i * n, p.act_a,
                                      p.glp_a, p.gh_a, p.lp_a, p.h_a, p.g_a, i, lane);
    } else {
        const int n = 1 + c.sub_levels;
        policy_eval_slot<BWD, MT, LT>((const MT *)p.p_mask + (size_t)r * n, 1, p.p_logit, n, (size_t)r * n, p.act_p,
                                      p.glp_p, p.gh_p, p.lp_p, p.h_p, p.g_p, (size_t)r, lane);
    }
}

}  // namespace aie
