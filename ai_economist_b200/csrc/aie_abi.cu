// aie_abi.cu — CUDA backend of the C-ABI (the product).  sm_90a only; there is no CPU path.
//
// Kernels (see DESIGN.md for the roofline of each):
//   aie_step_kernel        one warp per env replica.  The env's packed state record is staged HBM -> shared
//                          memory with one TMA bulk copy (cp.async.bulk + mbarrier), advanced one timestep in
//                          shared memory (aie_core.cuh: step_env), and written back with one bulk copy.
//   aie_observe_kernel     one CTA per env replica.  Bulk-loads the observable prefix of the record and streams
//                          out every observation / mask tensor with coalesced stores (the HBM-bound part).
//   aie_finish_reset_kernel  one warp per env: tax trackers + utility metric_0 after a host reset upload.
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>

#include <new>

#include "aie_core.cuh"
#include "aie_covid_core.cuh"
#include "aie_host.h"
#include "aie_compact.cuh"

struct aie_env;
struct aie_covid_env;

namespace aie {
namespace be {
constexpr int AIE_MAX_SLICES_BE = 16;   // = AIE_MAX_SLICES (aie_compact_host.h)
struct State {
    int step_wpb;        // warps (envs) per CTA of the step kernel
    int step_minb;       // register-allocation variant of the step kernel (3 or 4 CTAs per SM)
    int step_cs;         // component set the step kernel is instantiated for (step_comp_set)
    int phase_sync;      // 2 (AIE_PHASE_SYNC set): the warps of a CTA enter the fused observation pass together; else 0
    size_t step_smem;    // dynamic shared memory per CTA
    int obs_threads;
    size_t obs_smem;
    uint16_t *tab_dev;   // observation programs (device copy)
    uint8_t *compact_dev = nullptr, *compact_host = nullptr;   // aie_step_host_compact: device + pinned host staging
    size_t compact_bytes = 0, compact_host_bytes = 0;
    int compact_host_node = -1;   // >= 0: staging pages bound to that NUMA node (mmap + mbind + cudaHostRegister)
    cudaEvent_t slice_ev[AIE_MAX_SLICES_BE] = {};   // one per transfer slice of the compacted D2H copy
    cudaStream_t copy_st = nullptr;   // aie_step_host_compact: the slices go down on this stream while later chunks still step
    cudaEvent_t chunk_ev = nullptr, tail_ev = nullptr;   // caller's stream -> copy stream (a chunk is packed), and back (all slices down)
    cudaEvent_t call_ev = nullptr;   // recorded when a host-buffer step starts enqueueing (timing reference of the slices)
};
// Makes `device` current for the lifetime of the object and restores the caller's device afterwards, so a handle
// created for cuda:1 works while cuda:0 is current (streams passed in must belong to the handle's device).
struct DevScope {
    int prev = -1; bool ok_ = true;
    explicit DevScope(int device) {
        if (cudaGetDevice(&prev) != cudaSuccess) { prev = -1; cudaGetLastError(); }
        if (prev == device) { prev = -1; return; }
        ok_ = cudaSetDevice(device) == cudaSuccess;
        if (!ok_) cudaGetLastError();
    }
    ~DevScope() { if (prev >= 0) cudaSetDevice(prev); }
    bool ok() const { return ok_; }
};
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
}  // namespace be
}  // namespace aie

#include "aie_abi.inl"
#include "aie_covid_abi.inl"

namespace aie {

// compacted D2H transfer (aie_compact.cuh): one warp rewrites one env's outputs as a compact record
__global__ void __launch_bounds__(256) aie_pack_kernel(const __grid_constant__ DevCfg c, const DevBufs b, const CompactLayout L,
                                                       uint8_t *dst, int env_lo) {
    const size_t env = (size_t)env_lo + ((blockIdx.x * (size_t)blockDim.x + threadIdx.x) >> 5);   // c.n_envs = end of the range
    if (env >= (size_t)c.n_envs) return;
    pack_env(c, b, L, env, dst + env * (size_t)L.bytes, threadIdx.x & 31);
}

static_assert(sizeof(DevCfg) <= 4000, "DevCfg is passed by value as a __grid_constant__ kernel parameter");

// ---- TMA bulk-copy / mbarrier primitives (PTX ISA: cp.async.bulk, mbarrier) -----------------------------
__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t *bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t *bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t *bar, uint32_t phase) {
    uint32_t ok;
    do {
        asm volatile(
            "{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
            : "=r"(ok) : "r"(smem_u32(bar)), "r"(phase) : "memory");
    } while (!ok);
}
__device__ __forceinline__ void bulk_g2s(void *smem_dst, const void *gmem_src, uint32_t bytes, uint64_t *bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"(smem_u32(smem_dst)), "l"(gmem_src), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void bulk_s2g_part(void *gmem_dst, const void *smem_src, uint32_t bytes) {
    asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;"
                 ::"l"(gmem_dst), "r"(smem_u32(smem_src)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
__device__ __forceinline__ void bulk_s2g(void *gmem_dst, const void *smem_src, uint32_t bytes) {
    bulk_s2g_part(gmem_dst, smem_src, bytes);
    bulk_commit();
}
__device__ __forceinline__ void bulk_wait_read() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }
__device__ __forceinline__ void bulk_wait_read_oldest() { asm volatile("cp.async.bulk.wait_group.read 1;" ::: "memory"); }
__device__ __forceinline__ void fence_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// shared-memory carve-up: [mbarriers | block-shared observation programs | per-warp (record | scratch | obs scratch)]
__device__ __forceinline__ int tab_smem_bytes(const DevCfg &c) { return (2 * c.tab_n + 15) & ~15; }
__device__ __forceinline__ uint8_t *warp_region(uint8_t *smem, int wpb, int warp, const DevCfg &c) {
    return smem + ((8 * wpb + 15) & ~15) + tab_smem_bytes(c) +
           (size_t)warp * (c.resident_bytes + c.step_scratch_bytes + c.obs_extra_bytes);
}
// The programs are indexed by the lane-varying flat position; reading them from global memory costs an L2 round
// trip per access here because the L1 carve-out is almost entirely shared memory.  One cooperative copy per CTA.
__device__ __forceinline__ const uint16_t *stage_tables(uint8_t *smem, int wpb, const DevCfg &c, const DevBufs &b) {
    uint32_t *dst = (uint32_t *)(smem + ((8 * wpb + 15) & ~15));
    const uint32_t *src = (const uint32_t *)b.tab;
    for (int i = threadIdx.x; i < c.tab_n / 2; i += blockDim.x) dst[i] = src[i];
    __syncthreads();
    return (const uint16_t *)dst;
}

__device__ __forceinline__ ObsOut obs_out_for(const DevCfg &c, const DevBufs &b, int env) {
    ObsOut o; o.b = &b; o.c = &c; o.env = (size_t)env;
    return o;
}

// Executor of the observation pass on the device (aie_obs.cuh): thread `tid` of the NT threads that own one env runs
// the phase body, then the group's barrier.  FUSED: the pass runs behind the record's write-back in the step kernel.
template <int NT, bool FUSED>
struct DevExec {
    int tid;
    __device__ __forceinline__ int nt() const { return NT; }
    __device__ __forceinline__ void sync() const { if (NT == 32) __syncwarp(); else __syncthreads(); }
    // one warp per env: the phase gets the lane re-read from %laneid, so no lane index stays live across phases
    template <class F> __device__ __forceinline__ void operator()(F f) const { f(NT == 32 ? relane(tid) : tid); sync(); }
    // the record image's tail (price history, order slots) is about to be reused as staging memory
    __device__ __forceinline__ void record_stored() const {
        if (FUSED) { if (tid == 0) bulk_wait_read(); sync(); }
    }
};

// Auto-reset (WarpDrive save_copy_and_apply_at_reset semantics): restore everything but the RNG stream from the
// load-time snapshot; the episode counters and the numpy stream carry on.  Once per episode: kept out of line so that
// the step's hot text does not carry it.
template <bool EXT>
__device__ __noinline__ void auto_reset_env(const DevCfg &c, const DevBufs &b, int env, uint8_t *rec, uint64_t *bar, int lane) {
    uint8_t *scratch = rec + c.resident_bytes;
    uint8_t *grec = b.state + (size_t)env * c.rec_bytes;
    int32_t *hdr = (int32_t *)rec;
    const int32_t completions = hdr[HDR_COMPLETIONS] + 1, warm = hdr[HDR_AUTO_WARMUP], mt_pos = hdr[HDR_MT_POS],
                  episodes = hdr[HDR_EPISODES] + 1, saez_n = hdr[HDR_SAEZ_N];
    const uint8_t *snap = b.state0 + (size_t)env * c.rec_bytes;
    const uint32_t tail = (uint32_t)(c.rec_bytes - c.off_price_hist);  // price history + order slots
    fence_async_smem();
    __syncwarp();
    if (b.final && lane == 0) {  // end-of-episode snapshot (previous_episode_metrics): the resident record as it stands
        bulk_s2g(b.final + (size_t)env * c.rec_bytes, rec, (uint32_t)c.resident_bytes);
        bulk_wait_read();
    }
    if (b.final && c.split) {  // the statistics of a split record live in global memory
        const uint4 *src = (const uint4 *)(grec + c.off_stats);
        uint4 *dst = (uint4 *)(b.final + (size_t)env * c.rec_bytes + c.off_stats);
        for (int i = lane; i < (8 * c.n_stats + 15) / 16; i += 32) dst[i] = src[i];
    }
    __syncwarp();
    if (lane == 0) {
        mbar_expect_tx(bar, (uint32_t)c.off_mt + (c.split ? 0u : tail));
        bulk_g2s(rec, snap, (uint32_t)c.off_mt, bar);
        if (!c.split) bulk_g2s(rec + c.off_price_hist, snap + c.off_price_hist, tail, bar);
    }
    if (c.split) {  // the big sections live in global memory: copy them back from the snapshot with plain stores
        const uint4 *src = (const uint4 *)(snap + c.off_price_hist);
        uint4 *dst = (uint4 *)(grec + c.off_price_hist);
        for (uint32_t i = lane; i < tail / 16; i += 32) dst[i] = src[i];
    }
    __syncwarp();
    mbar_wait(bar, 1);
    if (lane == 0) {
        hdr[HDR_COMPLETIONS] = completions; hdr[HDR_AUTO_WARMUP] = warm; hdr[HDR_MT_POS] = mt_pos;
        hdr[HDR_EPISODES] = episodes; hdr[HDR_SAEZ_N] = saez_n;
    }
    __syncwarp();
    if (c.reset_mode == 1)   // reference-exact layout (dynamic scenarios) / placement / skills
        device_reset_env<EXT>(c, rec, grec, scratch, lane, b.dyn_prob, b.dyn_work ? b.dyn_work + (size_t)env * (c.HW + 16) : nullptr);
    finish_reset_env(c, rec, grec, scratch, lane);  // metric_0 under the new completions count
}

// One warp: bulk-load env's record, advance it one timestep (auto-reset included), start the write-back.  On return the
// record image is final; with obs_alias_mt the MT19937 key went out as its own first group and has been read already.
// CS: the component kinds compiled into the step body (step_comp_set).
template <bool BIG, bool EXT, int CS = CS_ALL>
__device__ __forceinline__ void warp_step(const DevCfg &c, const DevBufs &b, int env, uint8_t *rec, uint64_t *bar,
                                          const uint16_t *tab, int lane) {
    uint8_t *scratch = rec + c.resident_bytes;
    uint8_t *grec = b.state + (size_t)env * c.rec_bytes;
    if (lane == 0) {
        mbar_init(bar, 1);
        mbar_expect_tx(bar, (uint32_t)c.resident_bytes);
        bulk_g2s(rec, grec, (uint32_t)c.resident_bytes, bar);
    }
    __syncwarp();
    // the actions are decoded into the scratch area while the bulk load of the record is in flight
    const int32_t *act_a = b.act_a + (size_t)env * c.A * c.n_act_a;
    const int32_t *act_p = (b.act_p && c.n_act_p) ? b.act_p + (size_t)env * c.n_act_p : nullptr;
    decode_actions<EXT>(c, step_scratch_view(scratch, c), act_a, act_p, lane, tab);
    mbar_wait(bar, 0);

    int32_t *events = (b.events && env < b.event_envs) ? b.events + (size_t)env * 8 * (b.event_cap + 1) : nullptr;
    step_env<BIG, EXT, CS>(c, rec, grec, scratch, act_a, act_p, b.rew + (size_t)env * (c.A + 1), b.done + env, lane, true,
                           events, b.event_cap);
    lane = relane(lane);
    if (c.auto_reset && ((const int32_t *)rec)[HDR_T] >= c.T) auto_reset_env<EXT>(c, b, env, rec, bar, lane);

    fence_async_smem();  // generic-proxy writes to the record -> visible to the bulk (async-proxy) store
    __syncwarp();
    // Observations / masks of the post-step state stream out of the same shared-memory record while the bulk store
    // drains (both only read the record).  When observation staging aliases the MT19937 key image, the key goes out as
    // its own (first) bulk group and only that group must have finished READING shared memory before the pass starts;
    // the pass itself waits for the rest before it reuses the record's tail (DevExec::record_stored).
    if (lane == 0) {
        if (c.obs_alias_mt) {
            const uint32_t mt_end = (uint32_t)c.off_mt + 4u * 624u;
            bulk_s2g(grec + c.off_mt, rec + c.off_mt, 4u * 624u);
            bulk_s2g_part(grec, rec, (uint32_t)c.off_mt);
            if ((uint32_t)c.resident_bytes > mt_end) bulk_s2g_part(grec + mt_end, rec + mt_end, (uint32_t)c.resident_bytes - mt_end);
            bulk_commit();
            bulk_wait_read_oldest();
        } else {
            bulk_s2g(grec, rec, (uint32_t)c.resident_bytes);
        }
    }
    __syncwarp();
}

// ---------------------------------------------------------------------------------------------------------
// One warp per env, up to 8 envs per CTA.  MINB = minimum resident CTAs per SM the register allocation targets
// (occupancy vs. registers per thread); CS = the component kinds compiled in (step_comp_set).
template <int MINB, bool EXT, int CS>
__global__ void __launch_bounds__(256, MINB) aie_step_kernel(const __grid_constant__ DevCfg c, const __grid_constant__ DevBufs b,
                                                              const int emit_obs, const int env_lo) {
    extern __shared__ __align__(128) uint8_t smem[];
    const int wpb = blockDim.x >> 5, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int env = env_lo + blockIdx.x * wpb + warp;   // the launch covers envs [env_lo, c.n_envs)
    const uint16_t *tab = stage_tables(smem, wpb, c, b);
    const bool phase_sync = emit_obs & 2;   // tuning aid (AIE_PHASE_SYNC): all warps of a CTA enter the observation pass together
    if (env >= c.n_envs && !phase_sync) return;  // from here on warps are independent: no block-wide barrier below
    uint64_t *bar = (uint64_t *)smem + warp;
    uint8_t *rec = warp_region(smem, wpb, warp, c);
    if (env < c.n_envs) warp_step<false, EXT, CS>(c, b, env, rec, bar, tab, lane);
    if (phase_sync) { __syncthreads(); if (env >= c.n_envs) return; }
    if (emit_obs & 1) observe_env<EXT, CS>(c, rec, b.state + (size_t)env * c.rec_bytes, rec, c.ob, obs_out_for(c, b, env), tab, DevExec<32, true>{lane});
    else if (lane == 0) bulk_wait_read();
}

// Large records: one CTA of four warps per env.  Warp 0 runs the (serial) dynamics; all four stream the observations.
template <bool BIG, bool EXT = false>
__global__ void __launch_bounds__(128, 4) aie_step_mw_kernel(const __grid_constant__ DevCfg c, const __grid_constant__ DevBufs b,
                                                             const int emit_obs, const int env_lo) {
    extern __shared__ __align__(128) uint8_t smem[];
    const int env = env_lo + blockIdx.x;
    const uint16_t *tab = stage_tables(smem, 1, c, b);
    uint8_t *rec = warp_region(smem, 1, 0, c);
    if (threadIdx.x < 32) warp_step<BIG, EXT>(c, b, env, rec, (uint64_t *)smem, tab, threadIdx.x);
    __syncthreads();
    if (emit_obs) observe_env<EXT>(c, rec, b.state + (size_t)env * c.rec_bytes, rec, c.ob, obs_out_for(c, b, env), tab, DevExec<128, true>{(int)threadIdx.x});
    else if (threadIdx.x == 0) bulk_wait_read();
}

__global__ void __launch_bounds__(256) aie_finish_reset_kernel(const __grid_constant__ DevCfg c, const DevBufs b,
                                                               int lo, int n) {
    extern __shared__ __align__(128) uint8_t smem[];
    const int wpb = blockDim.x >> 5, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int i = blockIdx.x * wpb + warp;
    if (i >= n) return;
    const int env = lo + i;
    uint64_t *bar = (uint64_t *)smem + warp;
    uint8_t *rec = warp_region(smem, wpb, warp, c);
    uint8_t *grec = b.state + (size_t)env * c.rec_bytes;
    if (lane == 0) {
        mbar_init(bar, 1);
        mbar_expect_tx(bar, (uint32_t)c.resident_bytes);
        bulk_g2s(rec, grec, (uint32_t)c.resident_bytes, bar);
    }
    __syncwarp();
    mbar_wait(bar, 0);
    finish_reset_env(c, rec, grec, rec + c.resident_bytes, lane);
    if (lane == 0) { b.done[env] = 0; }
    for (int a = lane; a <= c.A; a += 32) b.rew[(size_t)env * (c.A + 1) + a] = 0.0;
    fence_async_smem();
    __syncwarp();
    if (lane == 0) {
        bulk_s2g(grec, rec, (uint32_t)c.resident_bytes);
        bulk_wait_read();
    }
}

// Stand-alone observation pass (after a reset upload, or when the caller steps dynamics separately): bulk-loads only
// what observe_env reads.  One warp per env, or (MW) one CTA of four warps per env.
// observe_env reads the record's prefix [0, obs_prefix_bytes) and, outside it, only in phase A (before any staging
// buffer that may overlap them is written):
//   - the price history [off_price_hist, off_orders) (the auction's price_history / market_rate; in global memory when split);
//   - the Saez section [off_saez, off_saez + 384) (tax_rate_observed: curr_rates, tax_marginal_rate: marginal_rate).
// A field added to a phase-A read outside the prefix has to be added here (the emulation stages the same list).
__device__ __forceinline__ void load_obs_prefix(const DevCfg &c, uint8_t *rec, const uint8_t *grec, uint64_t *bar) {
    const uint32_t ph = (uint32_t)(c.off_orders - c.off_price_hist);
    const uint32_t saez = c.off_saez ? 8u * 48u : 0u;
    mbar_init(bar, 1);
    mbar_expect_tx(bar, (uint32_t)c.obs_prefix_bytes + (c.split ? 0u : ph) + saez);
    bulk_g2s(rec, grec, (uint32_t)c.obs_prefix_bytes, bar);
    if (!c.split) bulk_g2s(rec + c.off_price_hist, grec + c.off_price_hist, ph, bar);
    if (saez) bulk_g2s(rec + c.off_saez, grec + c.off_saez, saez, bar);
}
template <bool EXT>
__global__ void __launch_bounds__(256) aie_observe_kernel(const __grid_constant__ DevCfg c, const __grid_constant__ DevBufs b, int lo, int n) {
    extern __shared__ __align__(128) uint8_t smem[];
    const int wpb = blockDim.x >> 5, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int i = blockIdx.x * wpb + warp;
    const uint16_t *tab = stage_tables(smem, wpb, c, b);
    if (i >= n) return;
    const int env = lo + i;
    uint64_t *bar = (uint64_t *)smem + warp;
    uint8_t *rec = warp_region(smem, wpb, warp, c);
    uint8_t *grec = b.state + (size_t)env * c.rec_bytes;
    if (lane == 0) load_obs_prefix(c, rec, grec, bar);
    __syncwarp();
    mbar_wait(bar, 0);
    observe_env<EXT>(c, rec, grec, rec, c.ob, obs_out_for(c, b, env), tab, DevExec<32, false>{lane});
}
template <bool EXT>
__global__ void __launch_bounds__(128, 4) aie_observe_mw_kernel(const __grid_constant__ DevCfg c, const __grid_constant__ DevBufs b, int lo, int n) {
    extern __shared__ __align__(128) uint8_t smem[];
    const int env = lo + blockIdx.x;
    const uint16_t *tab = stage_tables(smem, 1, c, b);
    uint64_t *bar = (uint64_t *)smem;
    uint8_t *rec = warp_region(smem, 1, 0, c);
    uint8_t *grec = b.state + (size_t)env * c.rec_bytes;
    if (threadIdx.x == 0) load_obs_prefix(c, rec, grec, bar);
    __syncthreads();
    mbar_wait(bar, 0);
    observe_env<EXT>(c, rec, grec, rec, c.ob, obs_out_for(c, b, env), tab, DevExec<128, false>{(int)threadIdx.x});
}

// per_unit == 0: one warp per env (fastest for few agents: c2 15.2 us vs 17.5 us);  per_unit == 1: one warp per
// (env, agent | planner bracket) - many agents x subspaces make the per-env chain long (c5: 64 agents x 6 subspaces).
template <bool EXT>
__global__ void __launch_bounds__(256) aie_sample_kernel(const __grid_constant__ DevCfg c, const DevBufs b, uint64_t seed,
                                                         int per_unit) {
    const long long wid = (long long)((blockIdx.x * (size_t)blockDim.x + threadIdx.x) >> 5);
    const int lane = threadIdx.x & 31;
    const int units = per_unit ? c.A + (c.planner_acts ? c.B : 0) : 1;
    const int env = (int)(wid / units), u = (int)(wid - (long long)env * units);
    if (env >= c.n_envs) return;
    const float *am = b.a_mask + (size_t)env * c.A * c.Na, *pm = b.p_mask + (size_t)env * c.Np;
    int32_t *aa = const_cast<int32_t *>(b.act_a) + (size_t)env * c.A * c.n_act_a;
    int32_t *ap = c.n_act_p ? const_cast<int32_t *>(b.act_p) + (size_t)env * c.n_act_p : nullptr;
    const uint64_t key = mix64(seed ^ mix64((uint64_t)env));
    if (per_unit) sample_actions_unit<EXT>(c, am, pm, aa, ap, key, u, lane);
    else sample_actions_env<EXT>(c, am, pm, aa, ap, key, lane);
}

// ---------------------------------------------------------------------------------------------------------
namespace be {

static int cuda_fail(cudaError_t e, const char *what) {
    return fail(AIE_ECUDA, std::string(what) + ": " + cudaGetErrorString(e));
}
#define AIE_CUDA(call, what) do { cudaError_t e_ = (call); if (e_ != cudaSuccess) return cuda_fail(e_, what); } while (0)

int check_device(int device) {
    int ndev = 0;
    cudaError_t e = cudaGetDeviceCount(&ndev);
    if (e != cudaSuccess || ndev == 0)
        return fail(AIE_ECUDA, std::string("no CUDA device: this library has no CPU fallback (") +
                                   (e == cudaSuccess ? "device count 0" : cudaGetErrorString(e)) + ")");
    if (device < 0 || device >= ndev) return fail(AIE_EINVAL, "device ordinal out of range");
    int major = 0, minor = 0;
    AIE_CUDA(cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, device), "cudaDeviceGetAttribute");
    AIE_CUDA(cudaDeviceGetAttribute(&minor, cudaDevAttrComputeCapabilityMinor, device), "cudaDeviceGetAttribute");
    // sm_90a code runs on compute capability 9.0 and nothing else (arch-specific targets are not forward compatible)
    if (major != 9 || minor != 0) return fail(AIE_ECUDA, "this build targets sm_90a (Hopper H100) only");
    return AIE_OK;
}

int init(aie_env *env) {
    {
        const int rc = check_device(env->device);
        if (rc != AIE_OK) return rc;
    }
    AIE_CUDA(cudaSetDevice(env->device), "cudaSetDevice");
    cudaDeviceProp prop;
    AIE_CUDA(cudaGetDeviceProperties(&prop, env->device), "cudaGetDeviceProperties");
    const DevCfg &c = env->cfg;
    const size_t max_smem = prop.sharedMemPerBlockOptin;
    const size_t per_env = (size_t)c.resident_bytes + c.step_scratch_bytes + c.obs_extra_bytes;
    // envs (warps) per CTA: the count in 1..8 that keeps the most warps resident per SM (shared memory is the limit;
    // at most 32 warps = 4 CTAs x 8 with the 64-register variant); ties go to the larger CTA.  AIE_STEP_WPB overrides.
    const size_t tabs = (2 * (size_t)c.tab_n + 15) & ~(size_t)15;
    auto cta_smem = [&](int w) { return align16(8 * w) + tabs + (size_t)w * per_env; };
    int wpb = 0, best_warps = 0;
    for (int w = (c.mw > 1 ? 1 : 8); w >= 1; w--) {   // mw > 1: one env per CTA, c.mw warps
        if (cta_smem(w) > max_smem) continue;
        int ctas = (int)(prop.sharedMemPerMultiprocessor / (cta_smem(w) + 1024));
        if (ctas * w > 32) ctas = 32 / w;
        if (ctas * w > best_warps) { best_warps = ctas * w; wpb = w; }
    }
    if (wpb == 0) return fail(AIE_EINVAL, "env state record does not fit in shared memory");
    if (const char *ov = getenv("AIE_STEP_WPB")) { int v = atoi(ov); if (c.mw == 1 && v >= 1 && v <= 8 && cta_smem(v) <= max_smem) wpb = v; }
    env->be.step_wpb = wpb;
    env->be.step_smem = cta_smem(wpb);
    env->be.obs_threads = wpb * 32;
    env->be.obs_smem = env->be.step_smem;
    // Register budget: the 64-register variant (launch bounds 256 x 4) when more than 24 warps can be resident (c2: 32
    // warps per SM), otherwise the 80-register variant (c3: 20 warps).  Override: AIE_STEP_MINB=3|4.  Measured on an
    // H100 80GB HBM3 (700 W), one 300-step run per setting, step kernel: c2 248 us with 64 registers vs 305 us with 80;
    // c3 511 us with 80 vs 539 us with 64.  Envs per CTA stay at the search above: c2 at 4 per CTA took 248 us, as at
    // 8.  c3 at 2 per CTA, alternated five times with 8 on an H100 80GB HBM3 (400 W), took 0.4870 ms / step (range
    // 0.4854-0.4871) vs 0.4879 (0.4863-0.4883), while its step kernel timed alone took 532 us vs 502 us: no clear gain.
    const size_t smem_sm = prop.sharedMemPerMultiprocessor;
    int fit = (int)(smem_sm / (env->be.step_smem + 1024));
    const int resident_warps = (fit * wpb > 32) ? 32 : fit * wpb;
    env->be.step_minb = resident_warps > 24 ? 4 : 3;
    if (const char *ov = getenv("AIE_STEP_MINB")) { int v = atoi(ov); if (v == 3 || v == 4) env->be.step_minb = v; }
    env->be.step_cs = step_comp_set(c);
    env->be.phase_sync = getenv("AIE_PHASE_SYNC") ? 2 : 0;   // tuning aid, one-warp kernel only
    if (getenv("AIE_VERBOSE"))
        fprintf(stderr, "[aie] record %d B (resident %d, obs prefix %d), step scratch %d (alias mt %d), per env %zu B, "
                        "%d envs/CTA, %zu B smem/CTA, register variant %d, %d CTAs/SM fit\n", c.rec_bytes, c.resident_bytes, c.obs_prefix_bytes,
                c.step_scratch_bytes, c.obs_alias_mt, per_env, wpb, env->be.step_smem, env->be.step_minb, fit);
    // The attribute belongs to the function (per device, process-wide), not to this handle: a second env with a smaller
    // record must not lower it under the first one, so every kernel is simply opted in to the device maximum.
    const int sm = (int)max_smem;
#define AIE_OPT_IN(k) AIE_CUDA(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, sm), "smem attr")
    AIE_OPT_IN((aie_step_kernel<3, false, CS_GTB>)); AIE_OPT_IN((aie_step_kernel<4, false, CS_GTB>));
    AIE_OPT_IN((aie_step_kernel<3, false, CS_GTB_TAX>)); AIE_OPT_IN((aie_step_kernel<4, false, CS_GTB_TAX>));
    AIE_OPT_IN((aie_step_kernel<3, false, CS_ALL>)); AIE_OPT_IN((aie_step_kernel<4, false, CS_ALL>));
    AIE_OPT_IN((aie_step_kernel<3, true, CS_ALL>)); AIE_OPT_IN((aie_step_kernel<4, true, CS_ALL>));
    AIE_OPT_IN((aie_step_mw_kernel<false, false>)); AIE_OPT_IN((aie_step_mw_kernel<false, true>));
    AIE_OPT_IN((aie_step_mw_kernel<true, false>)); AIE_OPT_IN((aie_step_mw_kernel<true, true>));
    AIE_OPT_IN(aie_finish_reset_kernel);
    AIE_OPT_IN(aie_observe_kernel<false>); AIE_OPT_IN(aie_observe_kernel<true>);
    AIE_OPT_IN(aie_observe_mw_kernel<false>); AIE_OPT_IN(aie_observe_mw_kernel<true>);
#undef AIE_OPT_IN
    {
        AIE_CUDA(cudaMalloc((void **)&env->be.tab_dev, sizeof(Tables)), "cudaMalloc tables");
        AIE_CUDA(cudaMemcpy(env->be.tab_dev, env->tables.w, sizeof(Tables), cudaMemcpyHostToDevice), "upload tables");
        env->bufs.tab = env->be.tab_dev;
    }
    return AIE_OK;
}
static void free_compact_host(aie_env *env);
void destroy(aie_env *env) {
    if (env->be.tab_dev) cudaFree(env->be.tab_dev);
    if (env->be.copy_st) cudaStreamDestroy(env->be.copy_st);
    if (env->be.chunk_ev) cudaEventDestroy(env->be.chunk_ev);
    if (env->be.tail_ev) cudaEventDestroy(env->be.tail_ev);
    if (env->be.compact_dev) cudaFree(env->be.compact_dev);
    free_compact_host(env);
    for (cudaEvent_t &ev : env->be.slice_ev) if (ev) cudaEventDestroy(ev);
    if (env->be.call_ev) cudaEventDestroy(env->be.call_ev);
}
int download_slice(aie_env *env, int k, void *host, const void *dev, size_t n, void *stream) {
    if (k < 0 || k >= AIE_MAX_SLICES_BE) return fail(AIE_EINVAL, "transfer slice index");
    if (!env->be.slice_ev[k]) AIE_CUDA(cudaEventCreate(&env->be.slice_ev[k]), "cudaEventCreate");
    cudaStream_t cs = env->be.copy_st ? env->be.copy_st : (cudaStream_t)stream;   // after chunk_ready: the copy stream
    AIE_CUDA(cudaMemcpyAsync(host, dev, n, cudaMemcpyDeviceToHost, cs), "D2H slice");
    AIE_CUDA(cudaEventRecord(env->be.slice_ev[k], cs), "cudaEventRecord");
    return AIE_OK;
}
int wait_slice(aie_env *env, int k) { return cudaEventSynchronize(env->be.slice_ev[k]) == cudaSuccess ? AIE_OK : AIE_ECUDA; }
int mark_call_start(aie_env *env, void *stream) {
    if (!env->be.call_ev) AIE_CUDA(cudaEventCreate(&env->be.call_ev), "cudaEventCreate");
    AIE_CUDA(cudaEventRecord(env->be.call_ev, (cudaStream_t)stream), "cudaEventRecord");
    return AIE_OK;
}
double slice_device_ms(aie_env *env, int k) {
    float ms = -1.0f;
    if (!env->be.call_ev || k < 0 || k >= AIE_MAX_SLICES_BE || !env->be.slice_ev[k]) return -1.0;
    if (cudaEventElapsedTime(&ms, env->be.call_ev, env->be.slice_ev[k]) != cudaSuccess) { cudaGetLastError(); return -1.0; }
    return (double)ms;
}
static void free_compact_host(aie_env *env) {
    if (!env->be.compact_host) return;
    if (env->be.compact_host_node >= 0) { cudaHostUnregister(env->be.compact_host); free_on_node(env->be.compact_host, env->be.compact_host_bytes); }
    else cudaFreeHost(env->be.compact_host);
    env->be.compact_host = nullptr; env->be.compact_host_node = -1;
}
int compact_buffers(aie_env *env, size_t bytes, uint8_t **dev, uint8_t **host) {
    if (env->be.compact_bytes < bytes) {
        if (env->be.compact_dev) cudaFree(env->be.compact_dev);
        free_compact_host(env);
        env->be.compact_dev = nullptr; env->be.compact_bytes = 0;
        AIE_CUDA(cudaMalloc((void **)&env->be.compact_dev, bytes), "cudaMalloc compact buffer");
        // AIE_E2E_STAGING_NODE: -1 (default) plain cudaHostAlloc, k >= 0 pages bound to NUMA node k, -2 the node the GPU
        // hangs off.  The staging traffic is a small part of the expansion's, so the plain allocation is the default and
        // placement stays a tuning aid.
        int node = -1;
        if (const char *v = getenv("AIE_E2E_STAGING_NODE")) node = atoi(v);
        if (node == -2) {
            char bus[64] = {0};
            node = (numa_node_count() > 1 && cudaDeviceGetPCIBusId(bus, (int)sizeof(bus), env->device) == cudaSuccess) ? pci_numa_node(bus) : -1;
            cudaGetLastError();
        }
        if (node >= 0) {
            const size_t rounded = (bytes + 4095) & ~(size_t)4095;
            void *p = alloc_on_node(rounded, node);
            if (p && cudaHostRegister(p, rounded, cudaHostRegisterDefault) == cudaSuccess) {
                env->be.compact_host = (uint8_t *)p; env->be.compact_host_node = node; env->be.compact_host_bytes = rounded;
            } else { cudaGetLastError(); free_on_node(p, rounded); }
        }
        if (!env->be.compact_host) {
            AIE_CUDA(cudaHostAlloc((void **)&env->be.compact_host, bytes, cudaHostAllocDefault), "cudaHostAlloc compact buffer");
            env->be.compact_host_node = -1;
        }
        env->be.compact_bytes = bytes;
    }
    *dev = env->be.compact_dev; *host = env->be.compact_host;
    return AIE_OK;
}
int staging_node(aie_env *env) { return env->be.compact_host_node; }
int launch_pack_range(aie_env *env, const CompactLayout &L, uint8_t *dev, int lo, int hi, void *stream) {
    if (lo < 0 || hi > env->n_envs || hi <= lo) return fail(AIE_EINVAL, "launch_pack_range: env range");
    const long long warps = hi - lo;
    DevCfg ranged;
    const DevCfg *cp = &env->cfg;
    if (hi != env->n_envs) { ranged = env->cfg; ranged.n_envs = hi; cp = &ranged; }
    aie_pack_kernel<<<(unsigned)((warps + 7) / 8), 256, 0, (cudaStream_t)stream>>>(*cp, env->bufs, L, dev, lo);
    AIE_CUDA(cudaGetLastError(), "aie_pack_kernel launch");
    env->launches++;
    return AIE_OK;
}
// The compact records of everything enqueued on `stream` so far may go down: later download_slice calls (copy stream) wait for it.
int chunk_ready(aie_env *env, void *stream) {
    if (!env->be.copy_st) AIE_CUDA(cudaStreamCreateWithFlags(&env->be.copy_st, cudaStreamNonBlocking), "cudaStreamCreate");
    if (!env->be.chunk_ev) AIE_CUDA(cudaEventCreateWithFlags(&env->be.chunk_ev, cudaEventDisableTiming), "cudaEventCreate");
    AIE_CUDA(cudaEventRecord(env->be.chunk_ev, (cudaStream_t)stream), "cudaEventRecord");
    AIE_CUDA(cudaStreamWaitEvent(env->be.copy_st, env->be.chunk_ev, 0), "cudaStreamWaitEvent");
    return AIE_OK;
}
// `stream` continues only after every slice enqueued so far has arrived (stream-order semantics of the call are the caller's stream's).
int copies_done(aie_env *env, void *stream) {
    if (!env->be.copy_st) return AIE_OK;
    if (!env->be.tail_ev) AIE_CUDA(cudaEventCreateWithFlags(&env->be.tail_ev, cudaEventDisableTiming), "cudaEventCreate");
    AIE_CUDA(cudaEventRecord(env->be.tail_ev, env->be.copy_st), "cudaEventRecord");
    AIE_CUDA(cudaStreamWaitEvent((cudaStream_t)stream, env->be.tail_ev, 0), "cudaStreamWaitEvent");
    return AIE_OK;
}

int upload(aie_env *, void *dst, const void *src, size_t n, void *stream) {
    AIE_CUDA(cudaMemcpyAsync(dst, src, n, cudaMemcpyHostToDevice, (cudaStream_t)stream), "H2D copy");
    return AIE_OK;
}
int download(aie_env *, void *dst, const void *src, size_t n, void *stream) {
    AIE_CUDA(cudaMemcpyAsync(dst, src, n, cudaMemcpyDeviceToHost, (cudaStream_t)stream), "D2H copy");
    return AIE_OK;
}
int dev_copy(aie_env *, void *dst, const void *src, size_t n, void *stream) {
    AIE_CUDA(cudaMemcpyAsync(dst, src, n, cudaMemcpyDeviceToDevice, (cudaStream_t)stream), "D2D copy");
    return AIE_OK;
}
int sync(aie_env *, void *stream) {
    AIE_CUDA(cudaStreamSynchronize((cudaStream_t)stream), "stream sync");
    return AIE_OK;
}
int sync_all(aie_env *) {
    AIE_CUDA(cudaDeviceSynchronize(), "device sync");
    return AIE_OK;
}
int launch_finish_reset(aie_env *env, int lo, int n, void *stream) {
    const int wpb = env->be.step_wpb;
    aie_finish_reset_kernel<<<(n + wpb - 1) / wpb, wpb * 32, env->be.step_smem, (cudaStream_t)stream>>>(env->cfg, env->bufs, lo, n);
    AIE_CUDA(cudaGetLastError(), "aie_finish_reset_kernel launch");
    env->launches++;
    return AIE_OK;
}
int launch_step(aie_env *env, int emit_obs, void *stream) { return launch_step_range(env, emit_obs, 0, env->n_envs, stream); }
// One launch over envs [lo, hi): the kernels take the range as (env_lo, cfg.n_envs = hi); env replicas never interact.
int launch_step_range(aie_env *env, int emit_obs, int lo, int hi, void *stream) {
    const int wpb = env->be.step_wpb, n = hi - lo;
    cudaStream_t st = (cudaStream_t)stream;
    const size_t sm = env->be.step_smem;
    if (lo < 0 || hi > env->n_envs || n <= 0) return fail(AIE_EINVAL, "launch_step_range: env range");
    if (env->cfg.mw == 1) emit_obs = (emit_obs ? 1 : 0) | env->be.phase_sync;
    DevCfg ranged;
    const DevCfg *cp = &env->cfg;
    if (hi != env->n_envs) { ranged = env->cfg; ranged.n_envs = hi; cp = &ranged; }
    const DevCfg &cfg = *cp;
    if (env->cfg.mw > 1) {   // large records: one CTA of four warps per env
        const dim3 grid(n), block(32 * env->cfg.mw);
        if (env->cfg.ext) {
            if (env->cfg.split) aie_step_mw_kernel<true, true><<<grid, block, sm, st>>>(cfg, env->bufs, emit_obs, lo);
            else aie_step_mw_kernel<false, true><<<grid, block, sm, st>>>(cfg, env->bufs, emit_obs, lo);
        } else if (env->cfg.split) aie_step_mw_kernel<true, false><<<grid, block, sm, st>>>(cfg, env->bufs, emit_obs, lo);
        else aie_step_mw_kernel<false, false><<<grid, block, sm, st>>>(cfg, env->bufs, emit_obs, lo);
    } else {
        const dim3 grid((n + wpb - 1) / wpb), block(wpb * 32);
        const bool m4 = env->be.step_minb == 4;
#define AIE_STEP(EXT, CS) (m4 ? aie_step_kernel<4, EXT, CS><<<grid, block, sm, st>>>(cfg, env->bufs, emit_obs, lo) \
                              : aie_step_kernel<3, EXT, CS><<<grid, block, sm, st>>>(cfg, env->bufs, emit_obs, lo))
        // EXT: rarely used options compiled in (single-action planner, regen halfwidth), with every component kind
        if (env->cfg.ext) AIE_STEP(true, CS_ALL);
        else if (env->be.step_cs == CS_GTB) AIE_STEP(false, CS_GTB);
        else if (env->be.step_cs == CS_GTB_TAX) AIE_STEP(false, CS_GTB_TAX);
        else AIE_STEP(false, CS_ALL);
#undef AIE_STEP
    }
    AIE_CUDA(cudaGetLastError(), "aie_step_kernel launch");
    env->launches++;
    return AIE_OK;
}
int launch_observe(aie_env *env, int lo, int n, void *stream) {
    const int wpb = env->be.step_wpb;
    cudaStream_t st = (cudaStream_t)stream;
    if (env->cfg.mw > 1) {
        if (env->cfg.ext) aie_observe_mw_kernel<true><<<n, 32 * env->cfg.mw, env->be.obs_smem, st>>>(env->cfg, env->bufs, lo, n);
        else aie_observe_mw_kernel<false><<<n, 32 * env->cfg.mw, env->be.obs_smem, st>>>(env->cfg, env->bufs, lo, n);
    } else if (env->cfg.ext) aie_observe_kernel<true><<<(n + wpb - 1) / wpb, wpb * 32, env->be.obs_smem, st>>>(env->cfg, env->bufs, lo, n);
    else aie_observe_kernel<false><<<(n + wpb - 1) / wpb, wpb * 32, env->be.obs_smem, st>>>(env->cfg, env->bufs, lo, n);
    AIE_CUDA(cudaGetLastError(), "aie_observe_kernel launch");
    env->launches++;
    return AIE_OK;
}

int launch_sample(aie_env *env, uint64_t seed, void *stream) {
    const DevCfg &c = env->cfg;
    (void)c;
    const int units = env->cfg.A + (env->cfg.planner_acts ? env->cfg.B : 0);
    const int per_unit = (env->cfg.A * (env->cfg.multi_action ? env->cfg.n_sub : 1) >= 64) ? 1 : 0;
    const long long warps = (long long)env->n_envs * (per_unit ? units : 1);
    const uint64_t sd = host_mix64(seed) ^ host_mix64(++env->sample_calls);
    if (env->cfg.ext) aie_sample_kernel<true><<<(unsigned)((warps + 7) / 8), 256, 0, (cudaStream_t)stream>>>(env->cfg, env->bufs, sd, per_unit);
    else aie_sample_kernel<false><<<(unsigned)((warps + 7) / 8), 256, 0, (cudaStream_t)stream>>>(env->cfg, env->bufs, sd, per_unit);
    AIE_CUDA(cudaGetLastError(), "aie_sample_kernel launch");
    env->launches++;
    return AIE_OK;
}

}  // namespace be

// ---------------------------------------------------------------------------------------------------------
// COVID-19 scenario: one CTA per env replica, one thread per US state; a single fused kernel per step.
__global__ void __launch_bounds__(64) aie_covid_step_kernel(const __grid_constant__ CovidCfg c, const CovidBufs b) {
    __shared__ float red[3 * 64];
    __shared__ uint32_t chg[64 * CV_CHG_CAP];
    covid_step_env(c, blockIdx.x, b, red, chg, threadIdx.x, blockDim.x);
}
__global__ void __launch_bounds__(64) aie_covid_reset_kernel(const __grid_constant__ CovidCfg c, const CovidBufs b) {
    covid_reset_env(c, blockIdx.x, b, threadIdx.x, blockDim.x, false);
}

__global__ void __launch_bounds__(64) aie_covid_sample_kernel(const __grid_constant__ CovidCfg c, const CovidBufs b, uint64_t key) {
    covid_sample_env(c, blockIdx.x, b, cv_mix64(key ^ cv_mix64(blockIdx.x)), threadIdx.x, blockDim.x);
}

namespace be {
void *const_upload(const void *host, size_t bytes) {
    void *d = nullptr;
    if (cudaMalloc(&d, bytes) != cudaSuccess) return nullptr;
    if (cudaMemcpy(d, host, bytes, cudaMemcpyHostToDevice) != cudaSuccess) { cudaFree(d); return nullptr; }
    return d;
}
void *dev_alloc(size_t bytes) {
    void *d = nullptr;
    if (cudaMalloc(&d, bytes) != cudaSuccess) { cudaGetLastError(); return nullptr; }
    if (cudaMemset(d, 0, bytes) != cudaSuccess) { cudaFree(d); return nullptr; }
    return d;
}
void const_free(void *dev) { cudaFree(dev); }
int covid_launch_reset(aie_covid_env *env, void *stream) {
    aie_covid_reset_kernel<<<env->n_envs, 64, 0, (cudaStream_t)stream>>>(env->cfg, env->bufs);
    AIE_CUDA(cudaGetLastError(), "aie_covid_reset_kernel launch");
    env->launches++;
    return AIE_OK;
}
int covid_launch_sample(aie_covid_env *env, uint64_t key, void *stream) {
    aie_covid_sample_kernel<<<env->n_envs, 64, 0, (cudaStream_t)stream>>>(env->cfg, env->bufs, key);
    AIE_CUDA(cudaGetLastError(), "aie_covid_sample_kernel launch");
    env->launches++;
    return AIE_OK;
}
int covid_launch_step(aie_covid_env *env, void *stream) {
    aie_covid_step_kernel<<<env->n_envs, 64, 0, (cudaStream_t)stream>>>(env->cfg, env->bufs);
    AIE_CUDA(cudaGetLastError(), "aie_covid_step_kernel launch");
    env->launches++;
    return AIE_OK;
}
}  // namespace be
}  // namespace aie
