// TEST INFRASTRUCTURE ONLY — host emulation of the device source with a 1-lane "warp".
//
// The build container has no GPU, so CPU tests compile ai_economist_b200/csrc/aie_core.cuh with g++
// (-DAIE_EMU, NL = 1: warp collectives become identities) behind the very same C-ABI implementation
// (aie_abi.inl) and check it against the golden traces and the C oracle.  This validates the algorithmic
// content of the kernels (not their warp synchronisation, which the `-m gpu` tests and compute-sanitizer
// cover on the GPU).  The product never builds, ships or loads this file: ai_economist_b200/_lib.py only
// opens libaie_b200.so (CUDA) and raises if it is missing.
#define AIE_EMU 1
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include <new>
#include <vector>

#include "../../ai_economist_b200/csrc/aie_core.cuh"
#include "../../ai_economist_b200/csrc/aie_covid_core.cuh"
#include "../../ai_economist_b200/csrc/aie_host.h"
#include "../../ai_economist_b200/csrc/aie_compact.cuh"

struct aie_env;
struct aie_covid_env;
namespace aie { namespace be {
struct State { std::vector<uint8_t> scratch; std::vector<uint16_t> tab; std::vector<uint8_t> compact_dev, compact_host; int nt = 1; };
struct DevScope { explicit DevScope(int) {} bool ok() const { return true; } };
int check_device(int device);
int init(aie_env *);
void destroy(aie_env *);
int upload(aie_env *, void *dst, const void *src, size_t n, void *stream);
int download(aie_env *, void *dst, const void *src, size_t n, void *stream);
int dev_copy(aie_env *, void *dst, const void *src, size_t n, void *stream);
int sync(aie_env *, void *stream);
int sync_all(aie_env *);
int launch_finish_reset(aie_env *, int lo, int n, void *stream);
int launch_step(aie_env *, int emit_obs, void *stream);
int launch_step_range(aie_env *, int emit_obs, int lo, int hi, void *stream);
int launch_observe(aie_env *, int lo, int n, void *stream);
int launch_sample(aie_env *, uint64_t seed, void *stream);
int compact_buffers(aie_env *, size_t bytes, uint8_t **dev, uint8_t **host);
int staging_node(aie_env *);
int launch_pack_range(aie_env *, const CompactLayout &L, uint8_t *dev, int lo, int hi, void *stream);
int chunk_ready(aie_env *, void *stream);
int copies_done(aie_env *, void *stream);
int download_slice(aie_env *, int k, void *host, const void *dev, size_t n, void *stream);
int wait_slice(aie_env *, int k);
double slice_device_ms(aie_env *, int k);
int mark_call_start(aie_env *, void *stream);
void *const_upload(const void *host, size_t bytes);
void *dev_alloc(size_t bytes);
void const_free(void *dev);
int covid_launch_reset(aie_covid_env *, void *stream);
int covid_launch_step(aie_covid_env *, void *stream);
int covid_launch_sample(aie_covid_env *, uint64_t key, void *stream);
} }

#include "../../ai_economist_b200/csrc/aie_abi.inl"
#include "../../ai_economist_b200/csrc/aie_covid_abi.inl"

namespace aie { namespace be {
int check_device(int) { return AIE_OK; }
int init(aie_env *env) {
    env->be.scratch.assign((size_t)env->cfg.step_scratch_bytes + env->cfg.obs_scratch_bytes + 64, 0);
    // threads per env in the observation pass: 1 for the logic tests; AIE_EMU_NT=32 / 128 walks the phases with the
    // device's thread counts, one thread index after the other (thread-layout check of the writers)
    env->be.nt = 1;
    if (const char *v = getenv("AIE_EMU_NT")) { const int n = atoi(v); if (n >= 1 && n <= 1024) env->be.nt = n; }
    env->bufs.tab = env->tables.w;
    return AIE_OK;
}
void destroy(aie_env *) {}
int compact_buffers(aie_env *env, size_t bytes, uint8_t **dev, uint8_t **host) {
    if (env->be.compact_dev.size() < bytes) { env->be.compact_dev.assign(bytes, 0); env->be.compact_host.assign(bytes, 0); }
    *dev = env->be.compact_dev.data(); *host = env->be.compact_host.data();
    return AIE_OK;
}
int download_slice(aie_env *, int, void *host, const void *dev, size_t n, void *) { memcpy(host, dev, n); return AIE_OK; }
int wait_slice(aie_env *, int) { return AIE_OK; }
double slice_device_ms(aie_env *, int) { return -1.0; }
int mark_call_start(aie_env *, void *) { return AIE_OK; }
int staging_node(aie_env *) { return -1; }
int chunk_ready(aie_env *, void *) { return AIE_OK; }
int copies_done(aie_env *, void *) { return AIE_OK; }
int launch_pack_range(aie_env *env, const CompactLayout &L, uint8_t *dev, int lo, int hi, void *) {
    for (int e = lo; e < hi; e++) pack_env(env->cfg, env->bufs, L, (size_t)e, dev + (size_t)e * L.bytes, 0);
    return AIE_OK;
}
int upload(aie_env *, void *dst, const void *src, size_t n, void *) { if (dst != src) memcpy(dst, src, n); return AIE_OK; }
int download(aie_env *, void *dst, const void *src, size_t n, void *) { if (dst != src) memcpy(dst, src, n); return AIE_OK; }
int dev_copy(aie_env *, void *dst, const void *src, size_t n, void *) { memcpy(dst, src, n); return AIE_OK; }
int sync(aie_env *, void *) { return AIE_OK; }
int sync_all(aie_env *) { return AIE_OK; }

int launch_finish_reset(aie_env *env, int lo, int n, void *) {
    const DevCfg &c = env->cfg;
    for (int e = lo; e < lo + n; e++) {
        finish_reset_env(c, env->bufs.state + (size_t)e * c.rec_bytes, env->bufs.state + (size_t)e * c.rec_bytes,
                         env->be.scratch.data(), 0);
        env->bufs.done[e] = 0;
        for (int a = 0; a <= c.A; a++) env->bufs.rew[(size_t)e * (c.A + 1) + a] = 0.0;
    }
    env->launches++;
    return AIE_OK;
}
int launch_observe(aie_env *env, int lo, int n, void *);
int launch_step(aie_env *env, int emit_obs, void *) { return launch_step_range(env, emit_obs, 0, env->n_envs, nullptr); }
int launch_step_range(aie_env *env, int emit_obs, int lo, int hi, void *) {
    const DevCfg &c = env->cfg;
    const DevBufs &b = env->bufs;
    for (int e = lo; e < hi; e++) {
        uint8_t *rec = b.state + (size_t)e * c.rec_bytes;
        int32_t *events = (b.events && e < b.event_envs) ? b.events + (size_t)e * 8 * (b.event_cap + 1) : nullptr;
        const int32_t *aa = b.act_a + (size_t)e * c.A * c.n_act_a;
        const int32_t *ap = (b.act_p && c.n_act_p) ? b.act_p + (size_t)e * c.n_act_p : nullptr;
        // same dispatch as the CUDA launcher: the EXT instantiations only for configs that set one of the rare options
#define AIE_EMU_STEP(BIG, EXT) step_env<BIG, EXT>(c, rec, rec, env->be.scratch.data(), aa, ap, b.rew + (size_t)e * (c.A + 1), \
                                                  b.done + e, 0, false, events, b.event_cap, b.tab)
        if (c.ext) { if (c.split) AIE_EMU_STEP(true, true); else AIE_EMU_STEP(false, true); }
        else { if (c.split) AIE_EMU_STEP(true, false); else AIE_EMU_STEP(false, false); }
#undef AIE_EMU_STEP
        int32_t *hdr = (int32_t *)rec;
        if (c.auto_reset && hdr[HDR_T] >= c.T) {  // same sequence as aie_step_kernel
            int32_t completions = hdr[HDR_COMPLETIONS] + 1, warm = hdr[HDR_AUTO_WARMUP], mt_pos = hdr[HDR_MT_POS],
                    episodes = hdr[HDR_EPISODES] + 1, saez_n = hdr[HDR_SAEZ_N];
            if (b.final) memcpy(b.final + (size_t)e * c.rec_bytes, rec, c.rec_bytes);
            memcpy(rec, b.state0 + (size_t)e * c.rec_bytes, c.off_mt);
            memcpy(rec + c.off_price_hist, b.state0 + (size_t)e * c.rec_bytes + c.off_price_hist, c.rec_bytes - c.off_price_hist);
            hdr[HDR_COMPLETIONS] = completions; hdr[HDR_AUTO_WARMUP] = warm; hdr[HDR_MT_POS] = mt_pos;
            hdr[HDR_EPISODES] = episodes; hdr[HDR_SAEZ_N] = saez_n;
            if (c.reset_mode == 1) {
                double *work = b.dyn_work ? b.dyn_work + (size_t)e * (c.HW + 16) : nullptr;
                if (c.ext) device_reset_env<true>(c, rec, rec, env->be.scratch.data(), 0, b.dyn_prob, work);
                else device_reset_env<false>(c, rec, rec, env->be.scratch.data(), 0, b.dyn_prob, work);
            }
            finish_reset_env(c, rec, rec, env->be.scratch.data(), 0);
        }
    }
    env->launches++;
    if (emit_obs) { launch_observe(env, lo, hi - lo, nullptr); env->launches--; }
    return AIE_OK;
}
int launch_observe(aie_env *env, int lo, int n, void *) {
    const DevCfg &c = env->cfg;
    const DevBufs &b = env->bufs;
    for (int env_i = lo; env_i < lo + n; env_i++) {
        size_t e = env_i;
        ObsOut o; o.b = &b; o.c = &c; o.env = e;
        uint8_t *stage = env->be.scratch.data() + ((c.step_scratch_bytes + 15) & ~15);
        if (c.ext) observe_env<true>(c, b.state + e * c.rec_bytes, b.state + e * c.rec_bytes, stage, c.ob_emu, o, b.tab, SeqExec{env->be.nt});
        else observe_env<false>(c, b.state + e * c.rec_bytes, b.state + e * c.rec_bytes, stage, c.ob_emu, o, b.tab, SeqExec{env->be.nt});
    }
    env->launches++;
    return AIE_OK;
}
int launch_sample(aie_env *env, uint64_t seed, void *) {
    const DevCfg &c = env->cfg;
    const DevBufs &b = env->bufs;
    const uint64_t s = host_mix64(seed) ^ host_mix64(++env->sample_calls);
    for (int e = 0; e < env->n_envs; e++)
        if (c.ext)
            sample_actions_env<true>(c, b.a_mask + (size_t)e * c.A * c.Na, b.p_mask + (size_t)e * c.Np,
                           const_cast<int32_t *>(b.act_a) + (size_t)e * c.A * c.n_act_a,
                           c.n_act_p ? const_cast<int32_t *>(b.act_p) + (size_t)e * c.n_act_p : nullptr,
                           mix64(s ^ mix64((uint64_t)e)), 0);
        else
            sample_actions_env<false>(c, b.a_mask + (size_t)e * c.A * c.Na, b.p_mask + (size_t)e * c.Np,
                           const_cast<int32_t *>(b.act_a) + (size_t)e * c.A * c.n_act_a,
                           c.n_act_p ? const_cast<int32_t *>(b.act_p) + (size_t)e * c.n_act_p : nullptr,
                           mix64(s ^ mix64((uint64_t)e)), 0);
    env->launches++;
    return AIE_OK;
}
void *const_upload(const void *host, size_t bytes) { void *d = malloc(bytes ? bytes : 1); if (d) memcpy(d, host, bytes); return d; }
void *dev_alloc(size_t bytes) { return calloc(bytes ? bytes : 1, 1); }
void const_free(void *dev) { free(dev); }
int covid_launch_reset(aie_covid_env *env, void *) {
    for (int e = 0; e < env->n_envs; e++) covid_reset_env(env->cfg, e, env->bufs, 0, 1, false);
    env->launches++;
    return AIE_OK;
}
int covid_launch_sample(aie_covid_env *env, uint64_t key, void *) {
    for (int e = 0; e < env->n_envs; e++) covid_sample_env(env->cfg, e, env->bufs, cv_mix64(key ^ cv_mix64((uint64_t)e)), 0, 1);
    env->launches++;
    return AIE_OK;
}
int covid_launch_step(aie_covid_env *env, void *) {
    std::vector<float> red(3 * 64);
    std::vector<uint32_t> chg(64 * CV_CHG_CAP);
    for (int e = 0; e < env->n_envs; e++) covid_step_env(env->cfg, e, env->bufs, red.data(), chg.data(), 0, 1);
    env->launches++;
    return AIE_OK;
}
} }
