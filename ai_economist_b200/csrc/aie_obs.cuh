// aie_obs.cuh — observation + mask generation for one env replica (the larger half of the fused step kernel).
//
// Reference semantics restated here (paths relative to ai_economist/foundation/):
//   generate_observations / masks      scenarios/simple_wood_and_stone/layout_from_file.py:412-517;
//                                      base/base_env.py:562-756; components/build.py:163-193; move.py:155-188;
//                                      continuous_double_auction.py:491-580; redistribution.py:974-1104
//
// Shape of the pass.  NT threads cooperate on one env (NT = 32: one warp per env; NT = 128: a CTA per env for large
// records).  The pass is a sequence of PHASES; inside a phase every thread works on its own slice (stride NT) and only
// reads what earlier phases wrote, so the only synchronisation is one barrier between phases.  The phases are handed to
// an executor: on the device it runs the phase body for this thread and then the barrier; the host emulation runs the
// body for every thread index in turn (NT = 1 for the logic tests, NT = 32 / 128 for the lane-layout test).
//
// The spatial tensors are 0/1-valued float32 bit planes of one byte per cell ("world-map": per plane one bit of the
// cell byte).  They are produced in three steps that keep the per-element instruction count low:
//   1. transpose: 8 cell bytes -> 8 plane bytes (one 8x8 bit-matrix transpose per 8 cells, all planes at once),
//      written to plane-local bitmaps;
//   2. concat: the planes of a tensor slice are concatenated into ONE bit string whose bit b is element head + b of the
//      output run (head = the <= 3 floats before the first 16-byte boundary), 32 bits per thread per iteration;
//   3. stream: every 16-byte group of the run is lut[nibble] - one shared-memory word, a shift, a 16-entry float4 table
//      lookup and one 16-byte store per thread per iteration, front to back in address order.
// Index planes stream as bytes -> int16, flat vectors / masks as table-driven gathers, each as ONE run per tensor slice.
#pragma once

namespace aie {

// ---- executors ---------------------------------------------------------------------------------------------------
// host: runs a phase for every thread index of the group, one after the other (phases only read earlier phases' data)
struct SeqExec {
    int n;
    AIE_DEV_MEMBER int nt() const { return n; }
    template <class F> AIE_DEV_MEMBER void operator()(F f) const { for (int t = 0; t < n; t++) f(t); }
    AIE_DEV_MEMBER void record_stored() const {}
};

// ---- small output runs -------------------------------------------------------------------------------------------
struct RunSplit { int head, nq, tail0; };
AIE_DEV RunSplit run_split(const void *dst, int n, int elem_log2) {
    const int per = 16 >> elem_log2;  // elements per 16-byte group
    RunSplit r;
    r.head = (int)((per - (((uintptr_t)dst >> elem_log2) & (per - 1))) & (per - 1));
    if (r.head > n) r.head = n;
    r.nq = (n - r.head) / per;
    r.tail0 = r.head + r.nq * per;
    return r;
}
AIE_DEV void store4(float *p, float v0, float v1, float v2, float v3) {
#if AIE_ON_DEVICE
    *reinterpret_cast<float4 *>(p) = make_float4(v0, v1, v2, v3);
#else
    p[0] = v0; p[1] = v1; p[2] = v2; p[3] = v3;
#endif
}
AIE_DEV void store8(int16_t *p, uint32_t w0, uint32_t w1, uint32_t w2, uint32_t w3) {  // 8 int16, little endian
#if AIE_ON_DEVICE
    *reinterpret_cast<uint4 *>(p) = make_uint4(w0, w1, w2, w3);
#else
    const uint32_t w[4] = {w0, w1, w2, w3};
    for (int j = 0; j < 8; j++) p[j] = (int16_t)((w[j >> 1] >> (16 * (j & 1))) & 0xFFFFu);
#endif
}
AIE_DEV uint32_t div_magic(uint32_t x, uint32_t magic) {  // floor(x / n), magic = floor(2^32 / n) + 1, x * n < 2^32
#if AIE_ON_DEVICE
    return magic ? __umulhi(x, magic) : x;  // magic == 0 <=> n == 1
#else
    return magic ? (uint32_t)(((uint64_t)x * magic) >> 32) : x;
#endif
}
// the (at most per-1 + per-1) elements outside the whole 16-byte groups of a run: one scalar store per thread
template <typename T, typename F>
AIE_DEV void store_edges(T *dst, const RunSplit &r, int n, int tid, int NT, F value_at) {
    const int ne = r.head + (n - r.tail0);
    for (int j = tid; j < ne; j += NT) { const int i = j < r.head ? j : r.tail0 + (j - r.head); dst[i] = (T)value_at(i); }
}
template <typename F>
AIE_DEV void store_run_f32(float *dst, int n, int tid, int NT, F value_at) {
    const RunSplit r = run_split(dst, n, 2);
    store_edges(dst, r, n, tid, NT, value_at);
#if AIE_ON_DEVICE
    AIE_UNROLL(1)
#endif
    for (int g = tid; g < r.nq; g += NT) {
        const int i0 = r.head + 4 * g;
        store4(dst + i0, value_at(i0), value_at(i0 + 1), value_at(i0 + 2), value_at(i0 + 3));
    }
}
// rows x n matrix, contiguous: dst[row * n + i] = value_at(row, i), written as ONE run (n_magic = floor(2^32 / n) + 1)
template <typename F>
AIE_DEV void store_rows_f32(float *dst, int rows, int n, uint32_t n_magic, int tid, int NT, F value_at) {
    const int total = rows * n;
    auto flat_value = [&](int x) { const int row = (int)div_magic((uint32_t)x, n_magic); return value_at(row, x - row * n); };
    if (n < 4) { for (int x = tid; x < total; x += NT) dst[x] = flat_value(x); return; }
    const RunSplit r = run_split(dst, total, 2);
    store_edges(dst, r, total, tid, NT, flat_value);
#if AIE_ON_DEVICE
    AIE_UNROLL(1)
#endif
    for (int g = tid; g < r.nq; g += NT) {
        const int x0 = r.head + 4 * g;
        const int row = (int)div_magic((uint32_t)x0, n_magic), i = x0 - row * n;
        float v[4];
        for (int j = 0; j < 4; j++) { const bool nx = i + j >= n; v[j] = value_at(nx ? row + 1 : row, nx ? i + j - n : i + j); }
        store4(dst + x0, v[0], v[1], v[2], v[3]);
    }
}
// dst[i] = code(bytes[i]) widened to int16, code = identity (OWNER == false) or the house-owner encoding of an
// int8 owner byte (-1 -> 0, a -> a + 2; layout_from_file.py:438-440) applied four bytes at a time.
// `bytes` is 4-byte aligned and readable up to 12 bytes past n.
template <bool OWNER>
AIE_DEV uint32_t idx_code4(uint32_t v) {
    if (!OWNER) return v;
    const uint32_t none = (v >> 7) & 0x01010101u;                 // 1 in every byte that held -1
    return ((v & 0x7F7F7F7Fu) + 0x02020202u) & ~(none * 0xFFu);   // owner indices are < 64: no carry between bytes
}
template <bool OWNER>
AIE_DEV void store_bytes_i16(int16_t *dst, int n, const uint8_t *bytes, int tid, int NT) {
    const RunSplit r = run_split(dst, n, 1);
    store_edges(dst, r, n, tid, NT, [&](int i) { return (int)(idx_code4<OWNER>(bytes[i]) & 0xFFu); });
    const uint32_t *wd = reinterpret_cast<const uint32_t *>(bytes) + (r.head >> 2);
    const int sh = 8 * (r.head & 3);
    int16_t *q = dst + r.head;
#if AIE_ON_DEVICE
    AIE_UNROLL(1)
#endif
    for (int g = tid; g < r.nq; g += NT) {
        const uint32_t w0 = wd[2 * g], w1 = wd[2 * g + 1], w2 = wd[2 * g + 2];
        const uint32_t lo = idx_code4<OWNER>(fshr(w0, w1, sh)), hi = idx_code4<OWNER>(fshr(w1, w2, sh));
        store8(q + 8 * g, prmt(lo, 0u, 0x4140u), prmt(lo, 0u, 0x4342u), prmt(hi, 0u, 0x4140u), prmt(hi, 0u, 0x4342u));
    }
}

// ---- staged runs ---------------------------------------------------------------------------------------------------
// Small float tensors (flat vectors, masks) are first written element by element into shared memory, laid out exactly like
// the output run and shifted so that the 16-byte groups of the destination are 16-byte groups of the staging area
// (element x of the run at vals[a + x], a = the destination's offset inside its 16-byte group, in floats); a second phase
// copies the run out front to back, whole groups as float4 and the <= 3 elements at either end one by one.
AIE_DEV int run_align(const float *dst) { return (int)(((uintptr_t)dst >> 2) & 3); }
AIE_DEV void copy_run_f32(float *dst, int total, const float *vals, int tid, int NT) {
    const int a = run_align(dst);
    float *g0 = dst - a;
    const int ng = (a + total + 3) >> 2;
#if AIE_ON_DEVICE
    AIE_UNROLL(1)
#endif
    for (int k = tid; k < ng; k += NT) {
        const int lo = 4 * k - a;   // run index of the group's first float
        if (lo >= 0 && lo + 4 <= total) {
#if AIE_ON_DEVICE
            *reinterpret_cast<float4 *>(g0 + 4 * k) = *reinterpret_cast<const float4 *>(vals + 4 * k);
#else
            for (int j = 0; j < 4; j++) g0[4 * k + j] = vals[4 * k + j];
#endif
        } else {
            for (int j = 0; j < 4; j++) if (lo + j >= 0 && lo + j < total) g0[4 * k + j] = vals[4 * k + j];
        }
    }
}

// ---- bit planes ----------------------------------------------------------------------------------------------------
// 8x8 bit-matrix transpose of 8 bytes held little-endian in (lo, hi): afterwards byte k holds bit k of the 8 input bytes
// (bit j of output byte k = bit k of input byte j).
AIE_DEV void transpose8(uint32_t &lo, uint32_t &hi) {
    uint64_t x = ((uint64_t)hi << 32) | lo, t;
    t = (x ^ (x >> 7)) & 0x00AA00AA00AA00AAull;  x ^= t ^ (t << 7);
    t = (x ^ (x >> 14)) & 0x0000CCCC0000CCCCull; x ^= t ^ (t << 14);
    t = (x ^ (x >> 28)) & 0x00000000F0F0F0F0ull; x ^= t ^ (t << 28);
    lo = (uint32_t)x; hi = (uint32_t)(x >> 32);
}
// cells[0 .. n) (one byte per cell, 8-byte aligned, readable up to the next multiple of 8) -> np plane-local bitmaps:
// plane m holds bit psh[m] of every cell, planes[m * stride + (i >> 3)] bit (i & 7) = cell i.
AIE_DEV void planes_from_cells(const uint8_t *cells, int n, uint8_t *planes, int stride, int np, const uint8_t *psh,
                               int tid, int NT) {
    const uint32_t *c32 = reinterpret_cast<const uint32_t *>(cells);
    const uint32_t s0 = reinterpret_cast<const uint32_t *>(psh)[0], s1 = reinterpret_cast<const uint32_t *>(psh)[1];
    for (int u = tid; 8 * u < n; u += NT) {
        uint32_t lo = c32[2 * u], hi = c32[2 * u + 1];
        transpose8(lo, hi);
        uint8_t *q = planes + u;
        for (int m = 0; m < np; m++) { q[0] = (uint8_t)prmt(lo, hi, ((m < 4 ? s0 : s1) >> (8 * (m & 3))) & 7u); q += stride; }
    }
}
// the same for `count` cell arrays `cell_stride` bytes apart (cell_stride = 8 * units: a multiple of 8), array k's planes at
// planes + k * np * stride: ONE loop over all (array, unit) pairs, units_magic = floor(2^32 / units) + 1
AIE_DEV void planes_from_cells_multi(const uint8_t *cells, int units, uint32_t units_magic, int count, uint8_t *planes, int stride,
                                     int np, const uint8_t *psh, int tid, int NT) {
    const uint32_t *c32 = reinterpret_cast<const uint32_t *>(cells);
    const uint32_t s0 = reinterpret_cast<const uint32_t *>(psh)[0], s1 = reinterpret_cast<const uint32_t *>(psh)[1];
    const int total = count * units, blk = np * stride;
    for (int t = tid; t < total; t += NT) {
        const int k = (int)div_magic((uint32_t)t, units_magic), u = t - k * units;
        uint32_t lo = c32[2 * t], hi = c32[2 * t + 1];   // arrays are contiguous: unit t of the concatenation
        transpose8(lo, hi);
        uint8_t *q = planes + k * blk + u;
        for (int m = 0; m < np; m++) { q[0] = (uint8_t)prmt(lo, hi, ((m < 4 ? s0 : s1) >> (8 * (m & 3))) & 7u); q += stride; }
    }
}
// 32 bits of a plane-local bitmap starting at bit i (the word after the last one of the bitmap must be readable)
AIE_DEV uint32_t take32(const uint8_t *plane, int i) {
    const uint32_t *p = reinterpret_cast<const uint32_t *>(plane);
    return fshr(p[i >> 5], p[(i >> 5) + 1], i & 31);
}
// element x of the run (x in [0, nplanes * n)): plane x / n, bit x % n
AIE_DEV float plane_value(const uint8_t *planes, int stride, int n, uint32_t n_magic, int x) {
    const int p = (int)div_magic((uint32_t)x, n_magic), i = x - p * n;
    return (float)((planes[p * stride + (i >> 3)] >> (i & 7)) & 1u);
}
// bits[J] bit k = element head + 32 J + k of the run made of `nplanes` planes of n bits each (plane-local bitmaps at
// `planes`, `stride` bytes apart), for J in [0, nwords)
AIE_DEV void concat_planes(uint32_t *bits, int nwords, int head, const uint8_t *planes, int stride, int nplanes, int n,
                           uint32_t n_magic, int tid, int NT) {
    if (n >= 32) {   // a word of the string spans at most two planes
        for (int J = tid; J < nwords; J += NT) {
            const int x = head + 32 * J;
            const int p = (int)div_magic((uint32_t)x, n_magic), i = x - p * n, rem = n - i;
            uint32_t w = 0;
            if (p < nplanes) {
                w = take32(planes + p * stride, i);
                if (rem < 32) {
                    w &= (1u << rem) - 1u;
                    if (p + 1 < nplanes) w |= reinterpret_cast<const uint32_t *>(planes + (p + 1) * stride)[0] << rem;
                }
            }
            bits[J] = w;
        }
        return;
    }
    for (int J = tid; J < nwords; J += NT) {
        const int x = head + 32 * J;
        int p = (int)div_magic((uint32_t)x, n_magic), i = x - p * n, filled = 0;
        uint32_t w = 0;
        while (filled < 32 && p < nplanes) {
            int take = n - i;
            if (take > 32 - filled) take = 32 - filled;
            uint32_t v = take32(planes + p * stride, i);
            if (take < 32) v &= (1u << take) - 1u;
            w |= v << filled;
            filled += take; p++; i = 0;
        }
        bits[J] = w;
    }
}
// the run dst[0 .. total) = the concatenated planes as 0.0f / 1.0f: 16-byte groups from the bit string, edges one by one.
// Thread tid owns groups tid, tid + NT, ...: group g is nibble (g & 1) of byte g >> 1 of the string, so with NT even the
// thread's nibble position is fixed and its byte index advances by NT / 2 per group; four groups per iteration.
AIE_DEV void stream_bits_f32(float *dst, int total, const uint32_t *bits, const float *lut, const uint8_t *planes, int stride,
                             int n, uint32_t n_magic, int tid, int NT) {
    const RunSplit r = run_split(dst, total, 2);
    store_edges(dst, r, total, tid, NT, [&](int x) { return plane_value(planes, stride, n, n_magic, x); });
    float *q = dst + r.head + 4 * tid;
    if (NT & 1) {   // (host emulation with one thread)
        for (int g = tid; g < r.nq; g += NT) {
            const uint32_t nib = (bits[g >> 3] >> (4 * (g & 7))) & 15u;
            store4(q, lut[4 * nib], lut[4 * nib + 1], lut[4 * nib + 2], lut[4 * nib + 3]);
            q += 4 * NT;
        }
        return;
    }
    const uint8_t *b8 = reinterpret_cast<const uint8_t *>(bits) + (tid >> 1);
    const int sh = 4 * (tid & 1), hb = NT >> 1;
    int g = tid;
#if AIE_ON_DEVICE
    const float4 *lut4 = reinterpret_cast<const float4 *>(lut);
    float4 *q4 = reinterpret_cast<float4 *>(q);
    AIE_UNROLL(1)
    for (; g + 3 * NT < r.nq; g += 4 * NT) {
        const uint32_t v0 = b8[0], v1 = b8[hb], v2 = b8[2 * hb], v3 = b8[3 * hb];
        q4[0] = lut4[(v0 >> sh) & 15u]; q4[NT] = lut4[(v1 >> sh) & 15u];
        q4[2 * NT] = lut4[(v2 >> sh) & 15u]; q4[3 * NT] = lut4[(v3 >> sh) & 15u];
        b8 += 4 * hb; q4 += 4 * NT;
    }
    AIE_UNROLL(1)
    for (; g < r.nq; g += NT) { q4[0] = lut4[((uint32_t)b8[0] >> sh) & 15u]; b8 += hb; q4 += NT; }
#else
    for (; g < r.nq; g += NT) {
        const uint32_t nib = ((uint32_t)b8[0] >> sh) & 15u;
        store4(q, lut[4 * nib], lut[4 * nib + 1], lut[4 * nib + 2], lut[4 * nib + 3]);
        b8 += hb; q += 4 * NT;
    }
#endif
}
// how many words of bit string a run at `dst` needs (whole 16-byte groups only)
AIE_DEV int bits_words_for(const float *dst, int total, int *head) {
    const RunSplit r = run_split(dst, total, 2);
    *head = r.head;
    return (4 * r.nq + 31) >> 5;
}

// ---- staging -------------------------------------------------------------------------------------------------------
struct ObsScratch {
    double *net_hist;     // [2][P] summed price history (fp64, for the market rate); [2P] = annealed tax limit
    float *shf;           // [sh_count] shared float staging (SH_*): scalars + price history + rates + incomes + full counts
    float *sc_a;          // [A][AS_COUNT] per-agent scalar observations
    uint8_t *lim;         // [A][MS_COUNT] mask limits: mask[j] = idx_j < lim[slot_j]
    uint8_t *psh;         // [8] map plane -> bit index of the cell byte (maps.state order); plane M = bit 6 ("inside the world")
    uint8_t *locmap;      // [HW]  0 none, a+2
    uint8_t *wc;          // [chunk][wc_stride] window cells of a chunk of agents: cell bits | 0x40 inside
    uint8_t *wi;          // [chunk][2][ww] owner code, agent-location code (the int16 index planes as bytes)
    uint8_t *pl;          // plane-local bitmaps (agent chunk: [chunk][M+1] planes of ww bits; planner: [M] planes of HW bits)
    uint32_t *bits;       // concatenated bit string of the run being streamed
    float *vals;          // staged runs of the flat vectors / masks (shares its bytes with wc / wi / pl / bits)
};
// base: the env's shared-memory region (offsets c.ob[] may alias dead parts of the record image; the suite's host
// emulation passes its image of that region), or a separate scratch allocation (c.ob_emu[])
AIE_DEV ObsScratch obs_scratch_view(uint8_t *base, const int32_t *ob) {
    ObsScratch s;
    s.net_hist = (double *)(base + ob[OB_NET_HIST]);
    s.shf = (float *)(base + ob[OB_SHF]);
    s.sc_a = (float *)(base + ob[OB_SC_A]);
    s.lim = base + ob[OB_LIM];
    s.psh = base + ob[OB_PSH];
    s.locmap = base + ob[OB_LOCMAP];
    s.wc = base + ob[OB_WC];
    s.wi = base + ob[OB_WI];
    s.pl = base + ob[OB_PL];
    s.bits = (uint32_t *)(base + ob[OB_BITS]);
    s.vals = (float *)(base + ob[OB_VALS]);
    return s;
}

// Output slices of one env, computed where they are used (keeping ten 64-bit pointers live through the pass would
// spill under the register budget).
struct ObsOut {
    const DevBufs *b; const DevCfg *c; size_t env;
    AIE_DEV_MEMBER float *a_map() const { return b->a_map + env * c->A * c->a_map_elems; }
    AIE_DEV_MEMBER int16_t *a_idx() const { return b->a_idx + env * c->A * c->a_idx_elems; }
    AIE_DEV_MEMBER float *a_flat() const { return b->a_flat + env * c->A * c->Fa; }
    AIE_DEV_MEMBER float *a_mask() const { return b->a_mask + env * c->A * c->Na; }
    AIE_DEV_MEMBER float *p_map() const { return b->p_map + env * c->M * c->HW; }
    AIE_DEV_MEMBER int16_t *p_idx() const { return b->p_idx + env * 2 * c->HW; }
    AIE_DEV_MEMBER float *p_flat() const { return b->p_flat + env * c->Fp; }
    AIE_DEV_MEMBER float *p_agents() const { return b->p_agents + env * c->A * c->Fpa; }
    AIE_DEV_MEMBER float *p_mask() const { return b->p_mask + env * c->Np; }
    AIE_DEV_MEMBER float *time_obs() const { return b->time_obs + env; }
};

// One element of a "flat" vector (program entry -> value).  FK_SHARED: the per-env shared float staging; FK_AGENT: agent
// a's scalars; FK_MY / FK_AVAIL: agent a's own / everybody else's open orders at one (side, commodity, price level),
// straight from the uint8 histograms of the record (continuous_double_auction.py:515-542).
AIE_DEV float flat_value(const float *shf, const float *sc, const uint8_t *hist, const uint16_t *hoff, int aP, int sh_full,
                         uint32_t entry) {
    const uint32_t kind = AIE_FLAT_KIND(entry), p = AIE_FLAT_PAYLOAD(entry);
    if (kind == FK_SHARED) return shf[p];
    if (kind == FK_AGENT) return sc[p];
    const float mine = (float)hist[hoff[p] + aP];
    return kind == FK_MY ? mine : shf[sh_full + p] - mine;
}

// Random policy fused into the pass (DevBufs::policy_seed != 0): the next step's action of one agent / planner bracket,
// uniform over its open actions, computed by ONE thread from the mask limits (no mask read-back, no extra launch).
AIE_DEV uint64_t obs_mix64(uint64_t x) {  // splitmix64 finaliser
    x += 0x9e3779b97f4a7c15ull;
    x = (x ^ (x >> 30)) * 0xbf58476d1ce4e5b9ull;
    x = (x ^ (x >> 27)) * 0x94d049bb133111ebull;
    return x ^ (x >> 31);
}
// The flattened action mask is a list of SEGMENTS (slot, count): entry idx of a segment is open iff idx < lim[slot], so
// the open entries of a segment are its first min(lim[slot], count).  Uniform choice among the open entries of segments
// [s0, s1): returns the position inside that slice of the mask (= the action value; position 0 is the NO-OP).
AIE_DEV int policy_pick(const uint16_t *seg, int s0, int s1, const uint8_t *lim, uint64_t key) {
    int total = 0;
    for (int k = s0; k < s1; k++) { const int cnt = seg[k] >> 8, l = lim[seg[k] & 255u]; total += l < cnt ? l : cnt; }
    if (total == 0) return 0;
    int r = (int)((uint32_t)(obs_mix64(key) >> 32) % (uint32_t)total), j = 0;
    for (int k = s0; k < s1; k++) {
        const int cnt = seg[k] >> 8, l = lim[seg[k] & 255u], open = l < cnt ? l : cnt;
        if (r < open) return j + r;
        r -= open; j += cnt;
    }
    return 0;
}

// CS: the component kinds compiled in (see step_env)
template <bool EXT, int CS = CS_ALL, class Exec>
AIE_DEV void observe_env(const DevCfg &c, uint8_t *rec, uint8_t *grec, uint8_t *stage_base, const int32_t *ob, const ObsOut &o,
                         const uint16_t *tab, const Exec &ex) {
    const Env e = env_view(rec, grec, c);
    const ObsScratch s = obs_scratch_view(stage_base, ob);
    const int NT = ex.nt();
    const int A = c.A, H = c.H, W = c.W, HW = c.HW, P = c.P, M = c.M, win = c.win, w = c.w, ww = win * win;
    const double inv_scale = c.obs_scaling ? 0.01 : 1.0;
    const float *lut = reinterpret_cast<const float *>(tab + c.tab_lut);
    const uint16_t *hoff = tab + c.tab_hoff;

    // ---- phase A: stage every scalar the flat vectors / masks need (float, final values) -------------
    ex([&](int tid) {
        const double time_v = (double)e.hdr[HDR_T] / (c.obs_scaling ? (double)c.T : 1.0);
        for (int k = tid; k < (HW + 3) / 4; k += NT) ((uint32_t *)s.locmap)[k] = 0u;
        for (int m = tid; m < 8; m += NT) {  // maps.state channel order: Stone, Wood, House, [Water], StoneSrc, WoodSrc
            const int b3 = c.has_water ? 4 : 2, b4 = c.has_water ? 2 : 3;   // bit indices: Water 4, StoneSrc 2, WoodSrc 3
            const int bit = m == 0 ? 0 : m == 1 ? 1 : m == 2 ? 5 : m == 3 ? b3 : m == 4 ? b4 : 3;
            s.psh[m] = (uint8_t)(m == M ? 6 : (m < M ? bit : 7));          // plane M: "inside"; unused planes: bit 7 (never set)
        }
        if (c.has[COMP_CDA]) {  // continuous_double_auction.py:491-542
            for (int i = tid; i < 2 * P; i += NT) {  // i = cc * P + p; sums over agents in index order
                int cc = i / P, p = i - cc * P;
                double acc = 0.0; int fa = 0, fb = 0;
                for (int a = 0; a < A; a++) {
                    acc += e.price_hist[(cc * A + a) * P + p];
                    fa += e.ask_hist[(cc * A + a) * P + p];
                    fb += e.bid_hist[(cc * A + a) * P + p];
                }
                s.net_hist[i] = acc; s.shf[c.sh_full + i] = (float)fb; s.shf[c.sh_full + 2 * P + i] = (float)fa;
                s.shf[SH_PRICE_HIST + i] = (float)(acc * inv_scale);
            }
        }
        if ((CS & (1 << COMP_TAX)) && c.has[COMP_TAX]) {  // redistribution.py:974-1023
            const int pos = e.hdr[HDR_TAX_POS];
            if (tid == 0) {
                s.shf[SH_TAX_IS_TAX_DAY] = pos >= c.period ? 1.0f : 0.0f;
                s.shf[SH_TAX_IS_FIRST] = pos == 1 ? 1.0f : 0.0f;
                s.shf[SH_TAX_PHASE] = (float)((double)pos / c.period);
                // components/utils.py:10-57: current annealed |rate| limit for the planner mask
                double vis = fmax(0.0, fmin(1.0, c.ann_slope * ((double)e.hdr[HDR_COMPLETIONS] - c.ann_warm)));
                s.net_hist[2 * P] = vis * c.ann_full;
            }
            for (int b = tid; b < c.B; b += NT) s.shf[c.sh_curr_rates + b] = (float)tax_rate_observed<EXT>(c, e, b);
            for (int a = tid; a < A; a += NT) {
                s.sc_a[a * AS_COUNT + AS_TAX_MARG] = (float)tax_marginal_rate<EXT>(c, e, (e.coin[a] + e.esc_coin[a]) - e.last_coin[a]);
                const double v = e.last_income[a] / c.period;  // ascending rank -> sorted position (:908-911)
                int rank = 0;
                for (int j = 0; j < A; j++) {
                    double vj = e.last_income[j] / c.period;
                    rank += (vj < v || (vj == v && j < a)) ? 1 : 0;
                }
                s.shf[c.sh_last_incomes + rank] = (float)v;
                s.sc_a[a * AS_COUNT + AS_TAX_LAST_INCOME] = (float)v;
                s.sc_a[a * AS_COUNT + AS_TAX_LAST_MARG] = (float)e.last_marg[a];
            }
        }
        if (tid == 0) { s.shf[SH_ZERO] = 0.0f; s.shf[SH_TIME] = (float)time_v; o.time_obs()[0] = (float)time_v; }
    });
    ex([&](int tid) {
        for (int a = tid; a < A; a += NT) {
            const int row = (EXT && c.no_spatial) ? 0 : e.loc[2 * a], col = (EXT && c.no_spatial) ? 0 : e.loc[2 * a + 1];
            if (!(EXT && c.no_spatial)) s.locmap[row * W + col] = (uint8_t)(a + 2);
            float *sc = s.sc_a + a * AS_COUNT;
            if (EXT && c.one_step) sc[AS_LABOR_SKILL] = (float)(e.bskill[a] / c.labor_skill_scale);   // simple_labor.py:128-134
            sc[AS_LOC_ROW] = (float)((double)row / H);
            sc[AS_LOC_COL] = (float)((double)col / W);
            sc[AS_INV_COIN] = (float)(e.coin[a] * inv_scale);
            sc[AS_INV_STONE] = (float)(e.inv[2 * a] * inv_scale);
            sc[AS_INV_WOOD] = (float)(e.inv[2 * a + 1] * inv_scale);
            sc[AS_BUILD_PAYMENT] = (float)(e.bpay[a] / c.build_payment);
            sc[AS_BUILD_SKILL] = (float)e.bskill[a];
            sc[AS_BONUS] = (float)e.bonus[a];
        }
        if (EXT && c.one_step && tid == 0) {   // one_step_economy.py:146-158: equality and per-capita productivity / 1000
            double total = 0.0, diff = 0.0;
            for (int a = 0; a < A; a++) total += e.coin[a] + e.esc_coin[a];
            double eq;
            if (A < 30) {
                for (int i = 0; i < A; i++) for (int j = 0; j < A; j++) diff += fabs((e.coin[i] + e.esc_coin[i]) - (e.coin[j] + e.esc_coin[j]));
                eq = 1.0 - (diff / (2 * A * total + 1e-10)) / ((A - 1) / (double)A);
            } else {   // social_metrics.py: sorted form for larger populations
                double acc = 0.0;
                // O(A^2) without scratch: sum over sorted position k of cumsum_k = sum_i x_i * (number of positions >= rank_i)
                for (int i = 0; i < A; i++) {
                    const double xi = e.coin[i] + e.esc_coin[i];
                    int rank = 0;
                    for (int j = 0; j < A; j++) { const double xj = e.coin[j] + e.esc_coin[j]; rank += (xj < xi || (xj == xi && j < i)) ? 1 : 0; }
                    acc += xi * (double)(A - rank);
                }
                eq = (2.0 / (A + 1)) * (acc / (total + 1e-10));   // 1 - gini
            }
            s.shf[SH_ONE_PROD] = (float)(total / A / 1000.0);
            s.shf[SH_ONE_EQ] = (float)eq;
        }
        if (c.has[COMP_CDA])
            for (int cc = tid; cc < 2; cc += NT) {  // market_rate (:504-513)
                double dot = 0.0, tot = 0.0;
                for (int p = 0; p < P; p++) { dot += p * s.net_hist[cc * P + p]; tot += s.net_hist[cc * P + p]; }
                s.shf[SH_MARKET_RATE + cc] = (float)(dot / fmax(0.001, tot));
            }
    });
    ex([&](int tid) {
        for (int a = tid; a < A; a += NT) {  // mask limits (build.py:180-193, move.py:167-188, cda :544-580)
            uint8_t *lim = s.lim + a * MS_COUNT;
            lim[MS_ONE] = 1;
            if (EXT && c.one_step) {   // simple_labor.py:93-98: everything masked in the reset observation, open afterwards
                lim[MS_LABOR] = (uint8_t)((c.labor_mask_first && e.hdr[HDR_T] == 0) ? 0 : 100);
                continue;
            }
            lim[MS_BUILD] = can_build(c, e, a) ? 1 : 0;
            const int row = e.loc[2 * a], col = e.loc[2 * a + 1];
            const int roff[4] = {0, 0, -1, 1}, coff[4] = {-1, 1, 0, 0};
            for (int d = 0; d < 4; d++) {
                int r2 = row + roff[d], c2 = col + coff[d];
                bool ok = r2 >= 0 && r2 < H && c2 >= 0 && c2 < W;
                if (ok) {
                    int k = r2 * W + c2;
                    int8_t ow = e.owner[k];
                    ok = s.locmap[k] == 0 && !(e.cell[k] & CELL_WATER) && (ow < 0 || ow == a);
                }
                lim[MS_G0 + d] = ok ? 1 : 0;
            }
            lim[MS_BUY0] = lim[MS_BUY1] = lim[MS_SELL0] = lim[MS_SELL1] = 0;
            if (c.has[COMP_CDA]) {
                // Buy_c[p] = (n_orders < K) and (p <= Coin)  <=>  p < min(P, floor(Coin) + 1)
                const double coin = e.coin[a];
                const int can_pay = coin >= (double)P ? P : (int)floor(coin) + 1;
                for (int cc = 0; cc < 2; cc++) {
                    const bool open = e.n_orders[cc * A + a] < c.K;
                    lim[MS_BUY0 + cc] = (uint8_t)(open ? can_pay : 0);
                    lim[MS_SELL0 + cc] = (uint8_t)((open && e.inv[2 * a + cc] > 0) ? P : 0);
                }
            }
        }
    });
    // From here on the pass no longer reads the price history / order slots of the record image, and its own staging may
    // live on top of them: the record's write-back must have finished reading shared memory first.
    ex.record_stored();

    // ---- phase B: the planner's flat vector (staged; copied out with the first agent chunk below), planner mask, policy ----
    ex([&](int tid) {
        {
            const uint16_t *tp = tab + c.tab_p;
            float *v = s.vals + c.vals_off[3] + run_align(o.p_flat());
            for (int j = tid; j < c.Fp; j += NT) v[j] = flat_value(s.shf, s.shf, e.bid_hist, hoff, 0, c.sh_full, tp[j]);
        }
        if (c.planner_acts) {  // redistribution.py:1025-1104, multi-action planner: per bracket [1] ++ rates
            const bool first_day = e.hdr[HDR_TAX_POS] == 1;
            const int per = 1 + c.R;
            for (int x = tid; x < c.B * per; x += NT) {
                const int b = x / per, rr = x - b * per;
                bool open = rr == 0 || first_day;
                if (open && rr != 0 && c.tax_annealing) open = fabs(c.disc_rates[rr - 1]) <= s.net_hist[2 * P];
                // single-action planner: one leading NO-OP, then every bracket's R rates (base_agent.py:452-459)
                const int at = (EXT && c.planner_single) ? (rr == 0 ? 0 : b * c.R + rr) : x;
                o.p_mask()[at] = open ? 1.0f : 0.0f;
            }
        } else if (tid == 0) {
            o.p_mask()[0] = 1.0f;
        }
        if (o.b->policy_seed) {   // the next step's random actions, from the limits / conditions the masks were written from
            const uint64_t key0 = obs_mix64(o.b->policy_seed ^ obs_mix64((uint64_t)o.env)) + ((uint64_t)(uint32_t)e.hdr[HDR_T] << 20) +
                                  ((uint64_t)(uint32_t)e.hdr[HDR_EPISODES] << 44);
            const uint16_t *seg = tab + c.tab_seg;
            int32_t *aa = const_cast<int32_t *>(o.b->act_a) + o.env * (size_t)(A * c.n_act_a);
            const int per_a = c.n_act_a;
            for (int u = tid; u < A * per_a; u += NT) {   // one thread per (agent, action subspace)
                const int a = u / per_a, si = u - a * per_a;
                aa[u] = policy_pick(seg, c.seg_lo[si], c.seg_lo[si + 1], s.lim + a * MS_COUNT,
                                    key0 + 0x100 * a + (c.multi_action ? si + 1 : 0));
            }
            if (c.planner_acts && o.b->act_p) {
                int32_t *ap = const_cast<int32_t *>(o.b->act_p) + o.env * (size_t)c.n_act_p;
                const bool first_day = e.hdr[HDR_TAX_POS] == 1;
                const double limit = s.net_hist[2 * P];
                auto n_open = [&]() {   // open rates of one bracket (the same for every bracket): NO-OP + allowed rates
                    int n = 0;
                    if (first_day) for (int rr = 1; rr <= c.R; rr++) n += (!c.tax_annealing || fabs(c.disc_rates[rr - 1]) <= limit) ? 1 : 0;
                    return n;
                };
                auto kth_open = [&](int k) {   // k-th open rate index (1-based rate number), k in [0, n_open)
                    for (int rr = 1; rr <= c.R; rr++)
                        if (!c.tax_annealing || fabs(c.disc_rates[rr - 1]) <= limit) { if (k == 0) return rr; k--; }
                    return 0;
                };
                if (EXT && c.planner_single) {
                    if (tid == 0) {
                        const int no = n_open(), total = 1 + c.B * no;
                        const int r = (int)((uint32_t)(obs_mix64(key0 + 0x10000) >> 32) % (uint32_t)total);
                        ap[0] = r == 0 ? 0 : ((r - 1) / no) * c.R + kth_open((r - 1) % no);
                    }
                } else {
                    for (int b = tid; b < c.B; b += NT) {
                        const int total = 1 + n_open();
                        const int r = (int)((uint32_t)(obs_mix64(key0 + 0x10000 + b) >> 32) % (uint32_t)total);
                        ap[b] = r == 0 ? 0 : kth_open(r - 1);
                    }
                }
            }
        }
    });

    // ---- flat vectors / masks of the agents (base_env.py:562-612, base_agent.py:440-460), fl_chunk agents at a time:
    // phase 1 stages the chunk's rows of the three tensors as runs, phase 2 copies them out
    for (int a0 = 0; a0 < A; a0 += c.fl_chunk) {
        const int na = (A - a0 < c.fl_chunk) ? A - a0 : c.fl_chunk;
        float *d_flat = o.a_flat() + (size_t)a0 * c.Fa, *d_mask = o.a_mask() + (size_t)a0 * c.Na, *d_pa = o.p_agents() + (size_t)a0 * c.Fpa;
        ex([&](int tid) {
            const float *shf = s.shf;
            const uint8_t *hist = e.bid_hist;
            const int sh_full = c.sh_full;
            {   // agents' flat vectors: sorted-key concatenation
                float *v = s.vals + c.vals_off[0] + run_align(d_flat);
                const int n = c.Fa, total = na * n;
                for (int x = tid; x < total; x += NT) {
                    const int al = (int)div_magic((uint32_t)x, c.Fa_magic), j = x - al * n, a = a0 + al;
                    v[x] = flat_value(shf, s.sc_a + a * AS_COUNT, hist, hoff, a * P, sh_full, tab[j]);
                }
            }
            {   // action masks: entry (slot, idx) is open iff idx < limit[agent][slot]
                float *v = s.vals + c.vals_off[1] + run_align(d_mask);
                const uint16_t *mt = tab + c.tab_m;
                const int n = c.Na, total = na * n;
                for (int x = tid; x < total; x += NT) {
                    const int al = (int)div_magic((uint32_t)x, c.Na_magic), j = x - al * n;
                    const uint32_t en = mt[j];
                    v[x] = ((en & 255u) < s.lim[(a0 + al) * MS_COUNT + (en >> 8)]) ? 1.0f : 0.0f;
                }
            }
            if (!EXT || c.Fpa > 0) {   // the planner's per-agent vectors p<i>
                float *v = s.vals + c.vals_off[2] + run_align(d_pa);
                const uint16_t *tpa = tab + c.tab_pa;
                const int n = c.Fpa, total = na * n;
                for (int x = tid; x < total; x += NT) {
                    const int al = (int)div_magic((uint32_t)x, c.Fpa_magic), j = x - al * n, a = a0 + al;
                    v[x] = flat_value(shf, s.sc_a + a * AS_COUNT, hist, hoff, a * P, sh_full, tpa[j]);
                }
            }
        });
        ex([&](int tid) {
            copy_run_f32(d_flat, na * c.Fa, s.vals + c.vals_off[0], tid, NT);
            copy_run_f32(d_mask, na * c.Na, s.vals + c.vals_off[1], tid, NT);
            if (!EXT || c.Fpa > 0) copy_run_f32(d_pa, na * c.Fpa, s.vals + c.vals_off[2], tid, NT);
            if (a0 == 0) copy_run_f32(o.p_flat(), c.Fp, s.vals + c.vals_off[3], tid, NT);
        });
    }

    if (EXT && c.no_spatial) return;   // one-step-economy: nothing spatial

    // ---- phase C: the planner's spatial tensors: M bit planes of the whole map + the two index planes -----------------
    const int psp = c.pl_stride_p;   // bytes per whole-map plane bitmap
    if (c.planner_spatial || (EXT && c.full_obs)) {
        ex([&](int tid) { planes_from_cells(e.cell, HW, s.pl, psp, M, s.psh, tid, NT); });
    }
    if (c.planner_spatial) {
        int head = 0;
        const int nwords = bits_words_for(o.p_map(), M * HW, &head);
        ex([&](int tid) {
            concat_planes(s.bits, nwords, head, s.pl, psp, M, HW, c.HW_magic, tid, NT);
            store_bytes_i16<true>(o.p_idx(), HW, (const uint8_t *)e.owner, tid, NT);
            store_bytes_i16<false>(o.p_idx() + HW, HW, s.locmap, tid, NT);
        });
        ex([&](int tid) { stream_bits_f32(o.p_map(), M * HW, s.bits, lut, s.pl, psp, HW, c.HW_magic, tid, NT); });
    }
    if (EXT && c.full_obs) {
        // full_observability (layout_from_file.py:465-472): every agent gets the whole map - the same M bit planes as
        // the planner - and the two index planes with its own index recoded to 1 (staged as bytes per agent)
        const int HW4 = (HW + 3) & ~3;
        uint8_t *so = s.wi, *sl = s.wi + HW4;
        for (int a = 0; a < A; a++) {
            float *am = o.b->a_map + (o.env * A + a) * (size_t)c.a_map_elems;
            int16_t *ai = o.b->a_idx + (o.env * A + a) * (size_t)c.a_idx_elems;
            int head = 0;
            const int nwords = bits_words_for(am, M * HW, &head);
            ex([&](int tid) {
                concat_planes(s.bits, nwords, head, s.pl, psp, M, HW, c.HW_magic, tid, NT);
                for (int k = tid; k < HW; k += NT) {
                    const int ow = e.owner[k], vl = s.locmap[k];
                    so[k] = (uint8_t)(ow < 0 ? 0 : (ow == a ? 1 : ow + 2));
                    sl[k] = (uint8_t)(vl == a + 2 ? 1 : vl);
                }
            });
            ex([&](int tid) {
                stream_bits_f32(am, M * HW, s.bits, lut, s.pl, psp, HW, c.HW_magic, tid, NT);
                store_bytes_i16<false>(ai, HW, so, tid, NT);
                store_bytes_i16<false>(ai + HW, HW, sl, tid, NT);
            });
        }
        return;
    }

    // ---- phase D: agent windows (layout_from_file.py:468-515), a chunk of agents at a time ----------------------------
    // per chunk: the window cells of its agents are staged as bytes (cell bits | inside flag, owner code, location code),
    // transposed into plane-local bitmaps, concatenated, and streamed as ONE run of chunk x (M+1) x ww floats; the index
    // planes of the chunk stream as one run of chunk x 2 x ww int16.
    const int psa = c.pl_stride_a, wcs = c.wc_stride, np1 = M + 1;
    for (int a0 = 0; a0 < A; a0 += c.ob_chunk) {
        const int na = (A - a0 < c.ob_chunk) ? A - a0 : c.ob_chunk;
        float *am = o.a_map() + (size_t)a0 * np1 * ww;
        int head = 0;
        const int nwords = bits_words_for(am, na * np1 * ww, &head);
        ex([&](int tid) {
            const int total = na * ww;
            for (int t = tid; t < total; t += NT) {   // one (agent, window cell) pair per thread and iteration
                const int al = (int)div_magic((uint32_t)t, c.ww_magic), q = t - al * ww, a = a0 + al;
                const int dr = (int)div_magic((uint32_t)q, c.win_magic), dc = q - dr * win;
                const int r2 = e.loc[2 * a] - w + dr, c2 = e.loc[2 * a + 1] - w + dc;
                uint32_t cb = 0; int vo = 0, vl = 0;
                if ((unsigned)r2 < (unsigned)H && (unsigned)c2 < (unsigned)W) {
                    const int k = r2 * W + c2;
                    cb = e.cell[k] | 0x40u;
                    const int ow = e.owner[k];
                    vo = ow < 0 ? 0 : (ow == a ? 1 : ow + 2);
                    vl = s.locmap[k];
                    if (vl == a + 2) vl = 1;
                }
                s.wc[al * wcs + q] = (uint8_t)cb;
                uint8_t *wi = s.wi + al * 2 * ww + q;
                wi[0] = (uint8_t)vo; wi[ww] = (uint8_t)vl;
            }
        });
        ex([&](int tid) {
            planes_from_cells_multi(s.wc, wcs >> 3, c.wcu_magic, na, s.pl, psa, np1, s.psh, tid, NT);
            store_bytes_i16<false>(o.a_idx() + (size_t)a0 * 2 * ww, na * 2 * ww, s.wi, tid, NT);
        });
        ex([&](int tid) { concat_planes(s.bits, nwords, head, s.pl, psa, na * np1, ww, c.ww_magic, tid, NT); });
        ex([&](int tid) { stream_bits_f32(am, na * np1 * ww, s.bits, lut, s.pl, psa, ww, c.ww_magic, tid, NT); });
    }
}

}  // namespace aie
