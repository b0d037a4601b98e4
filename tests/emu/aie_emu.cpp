// TEST INFRASTRUCTURE ONLY — host emulation of the device source with a 1-lane "warp".
//
// CPU tests compile ai_economist_b200/csrc/aie_core.cuh with g++ (-DAIE_EMU, NL = 1: warp collectives become
// identities) behind the very same C-ABI implementation (aie_abi.inl) and check it against the golden traces and the
// C oracle.  This validates the algorithmic content of the kernels and their shared-memory staging: every launch
// works on a per-env image of the region the kernel would own (record image | step scratch | observation extra),
// filled with 0xFF except for what the kernel bulk-loads, with the write-backs at the latest point the kernel allows
// and the observation staging (DevCfg::ob) aliasing the dead parts of the image as on the device.  A read of bytes the
// kernel never loaded or has already reused sees NaN / -1.  Warp synchronisation and the bulk-copy engine themselves
// are covered by the `-m gpu` tests only.  The product never builds, ships or loads this file:
// ai_economist_b200/_lib.py only opens libaie_b200.so (CUDA) and raises if it is missing.
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
// img: one env's shared-memory region as the kernels lay it out (record image | step scratch | observation extra)
struct State { std::vector<uint8_t> img; std::vector<uint16_t> tab; std::vector<uint8_t> compact_dev, compact_host; int nt = 1; };
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
    // exactly the per-env share of the kernel's shared memory (aie_abi.cu: warp_region): ASan sees reads past it
    env->be.img.assign((size_t)env->cfg.resident_bytes + env->cfg.step_scratch_bytes + env->cfg.obs_extra_bytes, 0xFF);
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

// Executor of the observation pass: runs a phase for every thread index of the group in turn (phases only read what
// earlier phases wrote).  record_stored() is where the fused kernel waits for the record's write-back to have read
// shared memory (DevExec<NT, true>): the emulation writes the record back there, the latest moment the device allows,
// and poisons the part of the image the pass may reuse from then on.  The stand-alone pass stores nothing.
struct EmuExec {
    int n;
    const DevCfg *c;
    uint8_t *img, *grec;
    bool fused;
    int nt() const { return n; }
    template <class F> void operator()(F f) const { for (int t = 0; t < n; t++) f(t); }
    void record_stored() const {
        if (!fused) return;
        const int mt_end = c->off_mt + 4 * 624;
        if (c->obs_alias_mt) {   // the key went out as its own group before the pass
            memcpy(grec, img, c->off_mt);
            memcpy(grec + mt_end, img + mt_end, c->resident_bytes - mt_end);
            memset(img + mt_end, 0xFF, c->resident_bytes - mt_end);
        } else {
            memcpy(grec, img, c->resident_bytes);
            memset(img + c->off_mt, 0xFF, c->resident_bytes - c->off_mt);
        }
    }
};

static uint8_t *fresh_image(aie_env *env) {
    memset(env->be.img.data(), 0xFF, env->be.img.size());
    return env->be.img.data();
}

int launch_finish_reset(aie_env *env, int lo, int n, void *) {   // aie_finish_reset_kernel
    const DevCfg &c = env->cfg;
    for (int e = lo; e < lo + n; e++) {
        uint8_t *grec = env->bufs.state + (size_t)e * c.rec_bytes, *img = fresh_image(env);
        memcpy(img, grec, c.resident_bytes);
        finish_reset_env(c, img, grec, img + c.resident_bytes, 0);
        env->bufs.done[e] = 0;
        for (int a = 0; a <= c.A; a++) env->bufs.rew[(size_t)e * (c.A + 1) + a] = 0.0;
        memcpy(grec, img, c.resident_bytes);
    }
    env->launches++;
    return AIE_OK;
}

// auto_reset_env (aie_abi.cu) on the image: restore everything but the RNG stream from the load-time snapshot
template <bool EXT>
static void emu_auto_reset(aie_env *env, int e, uint8_t *img, uint8_t *grec) {
    const DevCfg &c = env->cfg;
    const DevBufs &b = env->bufs;
    int32_t *hdr = (int32_t *)img;
    const int32_t completions = hdr[HDR_COMPLETIONS] + 1, warm = hdr[HDR_AUTO_WARMUP], mt_pos = hdr[HDR_MT_POS],
                  episodes = hdr[HDR_EPISODES] + 1, saez_n = hdr[HDR_SAEZ_N];
    const uint8_t *snap = b.state0 + (size_t)e * c.rec_bytes;
    const size_t tail = (size_t)(c.rec_bytes - c.off_price_hist);
    if (b.final) {   // the resident record as it stands; a split record's statistics and price history (which the final
                     // observation pass reads) come from global memory
        memcpy(b.final + (size_t)e * c.rec_bytes, img, c.resident_bytes);
        if (c.split) {
            memcpy(b.final + (size_t)e * c.rec_bytes + c.off_stats, grec + c.off_stats, 16 * ((8 * (size_t)c.n_stats + 15) / 16));
            memcpy(b.final + (size_t)e * c.rec_bytes + c.off_price_hist, grec + c.off_price_hist, 16 * ((size_t)(c.off_orders - c.off_price_hist) / 16));
        }
    }
    memcpy(img, snap, c.off_mt);
    memcpy((c.split ? grec : img) + c.off_price_hist, snap + c.off_price_hist, tail);
    hdr[HDR_COMPLETIONS] = completions; hdr[HDR_AUTO_WARMUP] = warm; hdr[HDR_MT_POS] = mt_pos;
    hdr[HDR_EPISODES] = episodes; hdr[HDR_SAEZ_N] = saez_n;
    uint8_t *scratch = img + c.resident_bytes;
    if (c.reset_mode == 1)
        device_reset_env<EXT>(c, img, grec, scratch, 0, b.dyn_prob, b.dyn_work ? b.dyn_work + (size_t)e * (c.HW + 16) : nullptr);
    finish_reset_env(c, img, grec, scratch, 0);
}

// One env through warp_step + the fused observation pass (aie_step_kernel / aie_step_mw_kernel), on the image.
// OCS: the component set of the observation pass (the one-warp kernel passes its own, the four-warp kernel CS_ALL).
template <bool BIG, bool EXT, int CS, int OCS>
static void emu_step_env(aie_env *env, int e, int emit_obs) {
    const DevCfg &c = env->cfg;
    const DevBufs &b = env->bufs;
    uint8_t *grec = b.state + (size_t)e * c.rec_bytes, *img = fresh_image(env);
    memcpy(img, grec, c.resident_bytes);   // the bulk load
    int32_t *events = (b.events && e < b.event_envs) ? b.events + (size_t)e * 8 * (b.event_cap + 1) : nullptr;
    const int32_t *aa = b.act_a + (size_t)e * c.A * c.n_act_a;
    const int32_t *ap = (b.act_p && c.n_act_p) ? b.act_p + (size_t)e * c.n_act_p : nullptr;
    step_env<BIG, EXT, CS>(c, img, grec, img + c.resident_bytes, aa, ap, b.rew + (size_t)e * (c.A + 1), b.done + e, 0, false,
                           events, b.event_cap, b.tab);
    if (c.auto_reset && ((const int32_t *)img)[HDR_T] >= c.T) emu_auto_reset<EXT>(env, e, img, grec);
    if (!emit_obs) { memcpy(grec, img, c.resident_bytes); return; }
    const int mt_end = c.off_mt + 4 * 624;
    if (c.obs_alias_mt) {   // the key's own bulk group has been read: its image is staging memory from here on
        memcpy(grec + c.off_mt, img + c.off_mt, 4 * 624);
        memset(img + c.off_mt, 0xFF, mt_end - c.off_mt);
    }
    memset(img + c.resident_bytes, 0xFF, c.step_scratch_bytes);   // the step scratch is dead
    ObsOut o; o.b = &b; o.c = &c; o.env = (size_t)e;
    observe_env<EXT, OCS>(c, img, grec, img, c.ob, o, b.tab, EmuExec{env->be.nt, &c, img, grec, true});
}

int launch_observe(aie_env *env, int lo, int n, void *);
int launch_step(aie_env *env, int emit_obs, void *) { return launch_step_range(env, emit_obs, 0, env->n_envs, nullptr); }
int launch_step_range(aie_env *env, int emit_obs, int lo, int hi, void *) {
    const DevCfg &c = env->cfg;
    // the instantiations the CUDA launcher picks: four warps per env -> <BIG = split, EXT> with every component kind;
    // one warp per env -> <false, EXT, step_comp_set> (EXT configs: every component kind)
    void (*one)(aie_env *, int, int);
    if (c.mw > 1) {
        if (c.ext) one = c.split ? emu_step_env<true, true, CS_ALL, CS_ALL> : emu_step_env<false, true, CS_ALL, CS_ALL>;
        else one = c.split ? emu_step_env<true, false, CS_ALL, CS_ALL> : emu_step_env<false, false, CS_ALL, CS_ALL>;
    } else if (c.ext) one = emu_step_env<false, true, CS_ALL, CS_ALL>;
    else {
        const int cs = step_comp_set(c);
        one = cs == CS_GTB ? emu_step_env<false, false, CS_GTB, CS_GTB>
            : cs == CS_GTB_TAX ? emu_step_env<false, false, CS_GTB_TAX, CS_GTB_TAX> : emu_step_env<false, false, CS_ALL, CS_ALL>;
    }
    for (int e = lo; e < hi; e++) one(env, e, emit_obs);
    env->launches++;
    return AIE_OK;
}
// aie_observe_kernel / aie_observe_mw_kernel: the image holds only what load_obs_prefix bulk-loads
int launch_observe(aie_env *env, int lo, int n, void *) {
    const DevCfg &c = env->cfg;
    const DevBufs &b = env->bufs;
    for (int e = lo; e < lo + n; e++) {
        uint8_t *grec = b.state + (size_t)e * c.rec_bytes, *img = fresh_image(env);
        memcpy(img, grec, c.obs_prefix_bytes);
        if (!c.split) memcpy(img + c.off_price_hist, grec + c.off_price_hist, c.off_orders - c.off_price_hist);
        if (c.off_saez) memcpy(img + c.off_saez, grec + c.off_saez, 8 * 48);
        ObsOut o; o.b = &b; o.c = &c; o.env = (size_t)e;
        const EmuExec ex{env->be.nt, &c, img, grec, false};
        if (c.ext) observe_env<true>(c, img, grec, img, c.ob, o, b.tab, ex);
        else observe_env<false>(c, img, grec, img, c.ob, o, b.tab, ex);
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
