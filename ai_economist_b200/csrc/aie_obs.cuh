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
//
// Output element type OT.  The float tensors (maps, flat vectors, masks, time) are float32 (OT = float), or bfloat16
// (OT = bf16_t, aie_config::obs_dtype == AIE_OBS_BF16): every value is computed in float32 as for float32 output and
// rounded to nearest even on the way out, 8 elements per 16-byte group instead of 4.
#pragma once

namespace aie {

// ---- bfloat16 output ---------------------------------------------------------------------------------------------
struct bf16_t { uint16_t bits; };   // bfloat16 storage
// round-to-nearest-even bfloat16 bits of v (what torch's float32 -> bfloat16 conversion gives; NaN -> a quiet NaN)
AIE_DEV uint32_t bf16_rn(float v) {
#if AIE_ON_DEVICE
    return __bfloat16_as_ushort(__float2bfloat16_rn(v));
#else
    uint32_t u;
    memcpy(&u, &v, 4);
    if ((u & 0x7FFFFFFFu) > 0x7F800000u) return 0x7FC0u;
    return (u + 0x7FFFu + ((u >> 16) & 1u)) >> 16;
#endif
}
AIE_DEV uint32_t bf16x2_rn(float lo, float hi) {   // two values, lo in the low half (the lower address)
#if AIE_ON_DEVICE
    uint32_t r;
    asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(hi), "f"(lo));
    return r;
#else
    return bf16_rn(lo) | (bf16_rn(hi) << 16);
#endif
}
AIE_DEV void put_out(float *p, float v) { *p = v; }
AIE_DEV void put_out(bf16_t *p, float v) { p->bits = (uint16_t)bf16_rn(v); }

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
// The 16-byte output stores are streaming stores (st.global.cs, evict-first): the outputs are written once per step and
// are several times the size of L2, so kept at normal priority they would push the env records (read and written back
// by the next step) out of L2.
AIE_DEV void store4(float *p, float v0, float v1, float v2, float v3) {
#if AIE_ON_DEVICE
    __stcs(reinterpret_cast<float4 *>(p), make_float4(v0, v1, v2, v3));
#else
    p[0] = v0; p[1] = v1; p[2] = v2; p[3] = v3;
#endif
}
AIE_DEV void store8(int16_t *p, uint32_t w0, uint32_t w1, uint32_t w2, uint32_t w3) {  // 8 int16, little endian
#if AIE_ON_DEVICE
    __stcs(reinterpret_cast<uint4 *>(p), make_uint4(w0, w1, w2, w3));
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
AIE_DEV void store_edges(bf16_t *dst, const RunSplit &r, int n, int tid, int NT, F value_at) {   // (<= 7 + 7 elements)
    const int ne = r.head + (n - r.tail0);
    for (int j = tid; j < ne; j += NT) { const int i = j < r.head ? j : r.tail0 + (j - r.head); put_out(dst + i, value_at(i)); }
}
// rows x n matrix, contiguous: dst[row * n + i] = value_at(row, i), written as ONE run (n_magic = floor(2^32 / n) + 1; not
// read when rows == 1).  Thread tid owns the 16-byte groups tid, tid + NT, ... of the destination: it computes the group's
// values in registers, one after the other through a single value_at site (the small code matters more than the three
// moves per value), and stores them as one float4, or one by one for the <= 2 groups at the ends of the run.
template <typename F>
AIE_DEV void store_rows_f32(float *dst, int rows, int n, uint32_t n_magic, int tid, int NT, F value_at) {
    const int total = rows * n;
    const int a = (int)(((uintptr_t)dst >> 2) & 3);   // floats in front of the run inside its first 16-byte group
    const int ng = (a + total + 3) >> 2;
#if AIE_ON_DEVICE
    AIE_UNROLL(1)
#endif
    for (int k = tid; k < ng; k += NT) {
        const int x0 = 4 * k - a;   // run index of the group's first float (negative in the first group when a > 0)
        const int xs = x0 > 0 ? x0 : 0;
        int row = rows > 1 ? (int)div_magic((uint32_t)xs, n_magic) : 0, i = xs - row * n;
        float v0 = 0.0f, v1 = 0.0f, v2 = 0.0f, v3 = 0.0f;
#if AIE_ON_DEVICE
        AIE_UNROLL(1)
#endif
        for (int x = x0; x < x0 + 4; x++) {
            float v = 0.0f;
            if (x >= 0 && x < total) { v = value_at(row, i); if (++i == n) { i = 0; row++; } }
            v0 = v1; v1 = v2; v2 = v3; v3 = v;
        }
        float *q = dst + x0;
        if (x0 >= 0 && x0 + 4 <= total) {
            store4(q, v0, v1, v2, v3);
        } else {
            if (x0 >= 0 && x0 < total) q[0] = v0;
            if (x0 + 1 >= 0 && x0 + 1 < total) q[1] = v1;
            if (x0 + 2 >= 0 && x0 + 2 < total) q[2] = v2;
            if (x0 + 3 < total) q[3] = v3;
        }
    }
}
// The same for bfloat16 output: eight values per 16-byte group, rounded in pairs into four words (one value_at site).
template <typename F>
AIE_DEV void store_rows_bf16(bf16_t *dst, int rows, int n, uint32_t n_magic, int tid, int NT, F value_at) {
    const int total = rows * n;
    const int a = (int)(((uintptr_t)dst >> 1) & 7);   // elements in front of the run inside its first 16-byte group
    const int ng = (a + total + 7) >> 3;
#if AIE_ON_DEVICE
    AIE_UNROLL(1)
#endif
    for (int k = tid; k < ng; k += NT) {
        const int x0 = 8 * k - a;
        const int xs = x0 > 0 ? x0 : 0;
        int row = rows > 1 ? (int)div_magic((uint32_t)xs, n_magic) : 0, i = xs - row * n;
        uint32_t w0 = 0u, w1 = 0u, w2 = 0u, w3 = 0u;
        float lo = 0.0f;
#if AIE_ON_DEVICE
        AIE_UNROLL(1)
#endif
        for (int x = x0; x < x0 + 8; x++) {
            float v = 0.0f;
            if (x >= 0 && x < total) { v = value_at(row, i); if (++i == n) { i = 0; row++; } }
            if (((x - x0) & 1) == 0) { lo = v; } else { w0 = w1; w1 = w2; w2 = w3; w3 = bf16x2_rn(lo, v); }
        }
        bf16_t *q = dst + x0;
        if (x0 >= 0 && x0 + 8 <= total) {
            store8(reinterpret_cast<int16_t *>(q), w0, w1, w2, w3);
        } else {
#if AIE_ON_DEVICE
            AIE_UNROLL(1)
#endif
            for (int j = 0; j < 8; j++) {   // element j is the low half of w0 after j shifts
                if (x0 + j >= 0 && x0 + j < total) q[j].bits = (uint16_t)w0;
                w0 = fshr(w0, w1, 16); w1 = fshr(w1, w2, 16); w2 = fshr(w2, w3, 16); w3 >>= 16;
            }
        }
    }
}
template <typename F>
AIE_DEV void store_rows(float *dst, int rows, int n, uint32_t n_magic, int tid, int NT, F value_at) {
    store_rows_f32(dst, rows, n, n_magic, tid, NT, value_at);
}
template <typename F>
AIE_DEV void store_rows(bf16_t *dst, int rows, int n, uint32_t n_magic, int tid, int NT, F value_at) {
    store_rows_bf16(dst, rows, n, n_magic, tid, NT, value_at);
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
        __stcs(q4, lut4[(v0 >> sh) & 15u]); __stcs(q4 + NT, lut4[(v1 >> sh) & 15u]);
        __stcs(q4 + 2 * NT, lut4[(v2 >> sh) & 15u]); __stcs(q4 + 3 * NT, lut4[(v3 >> sh) & 15u]);
        b8 += 4 * hb; q4 += 4 * NT;
    }
    AIE_UNROLL(1)
    for (; g < r.nq; g += NT) { __stcs(q4, lut4[((uint32_t)b8[0] >> sh) & 15u]); b8 += hb; q4 += NT; }
#else
    for (; g < r.nq; g += NT) {
        const uint32_t nib = ((uint32_t)b8[0] >> sh) & 15u;
        store4(q, lut[4 * nib], lut[4 * nib + 1], lut[4 * nib + 2], lut[4 * nib + 3]);
        b8 += hb; q += 4 * NT;
    }
#endif
}
// bfloat16 output: group g of the run is byte g of the bit string, two lut entries of four bf16 (8 bytes) each;
// lut8[2 * k], lut8[2 * k + 1] = the words of nibble k (bit j of the nibble -> element j).  Thread tid owns groups tid,
// tid + NT, ...: its byte index advances by NT per group; four groups per iteration.
AIE_DEV void stream_bits_bf16(bf16_t *dst, int total, const uint32_t *bits, const uint32_t *lut8, const uint8_t *planes,
                              int stride, int n, uint32_t n_magic, int tid, int NT) {
    const RunSplit r = run_split(dst, total, 1);
    store_edges(dst, r, total, tid, NT, [&](int x) { return plane_value(planes, stride, n, n_magic, x); });
    const uint8_t *b8 = reinterpret_cast<const uint8_t *>(bits) + tid;
    int g = tid;
#if AIE_ON_DEVICE
    const uint2 *lut2 = reinterpret_cast<const uint2 *>(lut8);
    uint4 *q4 = reinterpret_cast<uint4 *>(dst + r.head) + tid;
    auto group = [&](uint32_t v) {
        const uint2 lo = lut2[v & 15u], hi = lut2[v >> 4];
        return make_uint4(lo.x, lo.y, hi.x, hi.y);
    };
    AIE_UNROLL(1)
    for (; g + 3 * NT < r.nq; g += 4 * NT) {
        const uint32_t v0 = b8[0], v1 = b8[NT], v2 = b8[2 * NT], v3 = b8[3 * NT];
        __stcs(q4, group(v0)); __stcs(q4 + NT, group(v1));
        __stcs(q4 + 2 * NT, group(v2)); __stcs(q4 + 3 * NT, group(v3));
        b8 += 4 * NT; q4 += 4 * NT;
    }
    AIE_UNROLL(1)
    for (; g < r.nq; g += NT) { __stcs(q4, group(b8[0])); b8 += NT; q4 += NT; }
#else
    int16_t *q = reinterpret_cast<int16_t *>(dst + r.head) + 8 * tid;
    for (; g < r.nq; g += NT) {
        const uint32_t lo = b8[0] & 15u, hi = b8[0] >> 4;
        store8(q, lut8[2 * lo], lut8[2 * lo + 1], lut8[2 * hi], lut8[2 * hi + 1]);
        b8 += NT; q += 8 * NT;
    }
#endif
}
AIE_DEV void stream_bits(float *dst, int total, const uint32_t *bits, const uint16_t *lut, const uint8_t *planes, int stride,
                         int n, uint32_t n_magic, int tid, int NT) {
    stream_bits_f32(dst, total, bits, reinterpret_cast<const float *>(lut), planes, stride, n, n_magic, tid, NT);
}
AIE_DEV void stream_bits(bf16_t *dst, int total, const uint32_t *bits, const uint16_t *lut, const uint8_t *planes, int stride,
                         int n, uint32_t n_magic, int tid, int NT) {
    stream_bits_bf16(dst, total, bits, reinterpret_cast<const uint32_t *>(lut), planes, stride, n, n_magic, tid, NT);
}
// how many words of bit string a run at `dst` needs (whole 16-byte groups only)
AIE_DEV int bits_words_for(const float *dst, int total, int *head) {
    const RunSplit r = run_split(dst, total, 2);
    *head = r.head;
    return (4 * r.nq + 31) >> 5;
}
AIE_DEV int bits_words_for(const bf16_t *dst, int total, int *head) {
    const RunSplit r = run_split(dst, total, 1);
    *head = r.head;
    return (8 * r.nq + 31) >> 5;
}

// ---- staging -------------------------------------------------------------------------------------------------------
struct ObsScratch {
    double *net_hist;     // [2][P] summed price history (fp64, for the market rate); [2P] = annealed tax limit
    float *shf;           // [sh_count] shared float staging (SH_*): scalars + price history + rates + incomes + full counts
    float *sc_a;          // [A][AS_COUNT] per-agent scalar observations
    uint8_t *lim;         // [A][MS_COUNT] mask limits: mask[j] = idx_j < lim[slot_j]
    uint8_t *psh;         // [8] map plane -> bit index of the cell byte (maps.state order); plane M = bit 6 ("inside the world")
    uint8_t *locmap;      // [HW]  0 none, a+2
    uint8_t *wi;          // [chunk][2][ww] owner code, agent-location code (the int16 index planes as bytes)
    uint8_t *pl;          // plane-local bitmaps (agent chunk: [chunk][M+1] planes of ww bits; planner: [M] planes of HW bits)
    uint32_t *bits;       // concatenated bit string of the run being streamed
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
    s.wi = base + ob[OB_WI];
    s.pl = base + ob[OB_PL];
    s.bits = (uint32_t *)(base + ob[OB_BITS]);
    return s;
}

// Output slices of one env, computed where they are used (keeping ten 64-bit pointers live through the pass would
// spill under the register budget).  OT: the element type of the float tensors (their buffers hold OT when bfloat16).
struct ObsOut {
    const DevBufs *b; const DevCfg *c; size_t env;
    template <typename OT = float> AIE_DEV_MEMBER OT *a_map() const { return (OT *)b->a_map + env * c->A * c->a_map_elems; }
    AIE_DEV_MEMBER int16_t *a_idx() const { return b->a_idx + env * c->A * c->a_idx_elems; }
    template <typename OT = float> AIE_DEV_MEMBER OT *a_flat() const { return (OT *)b->a_flat + env * c->A * c->Fa; }
    template <typename OT = float> AIE_DEV_MEMBER OT *a_mask() const { return (OT *)b->a_mask + env * c->A * c->Na; }
    template <typename OT = float> AIE_DEV_MEMBER OT *p_map() const { return (OT *)b->p_map + env * c->M * c->HW; }
    AIE_DEV_MEMBER int16_t *p_idx() const { return b->p_idx + env * 2 * c->HW; }
    template <typename OT = float> AIE_DEV_MEMBER OT *p_flat() const { return (OT *)b->p_flat + env * c->Fp; }
    template <typename OT = float> AIE_DEV_MEMBER OT *p_agents() const { return (OT *)b->p_agents + env * c->A * c->Fpa; }
    template <typename OT = float> AIE_DEV_MEMBER OT *p_mask() const { return (OT *)b->p_mask + env * c->Np; }
    template <typename OT = float> AIE_DEV_MEMBER OT *time_obs() const { return (OT *)b->time_obs + env; }
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

// CS: the component kinds compiled in (see step_env); OT: the output element type of the float tensors (float, bf16_t).
template <bool EXT, int CS = CS_ALL, typename OT = float, class Exec>
AIE_DEV void observe_env(const DevCfg &c, uint8_t *rec, uint8_t *grec, uint8_t *stage_base, const int32_t *ob, const ObsOut &o,
                         const uint16_t *tab, const Exec &ex) {
#if !AIE_ON_DEVICE
    // host build of the device source: one entry for both element types, picked from the config as the CUDA launchers
    // pick the bfloat16 kernels
    if (sizeof(OT) == 4 && c.obs_bf16) { observe_env<EXT, CS, bf16_t>(c, rec, grec, stage_base, ob, o, tab, ex); return; }
#endif
    const Env e = env_view(rec, grec, c);
    const ObsScratch s = obs_scratch_view(stage_base, ob);
    const int NT = ex.nt();
    const int A = c.A, H = c.H, W = c.W, HW = c.HW, P = c.P, M = c.M, win = c.win, w = c.w, ww = win * win;
    const double inv_scale = c.obs_scaling ? 0.01 : 1.0;
    const uint16_t *lut = tab + c.tab_lut;   // nibble -> 4 elements of OT (float4 / four bf16)
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
        if (tid == 0) { s.shf[SH_ZERO] = 0.0f; s.shf[SH_TIME] = (float)time_v; put_out(o.time_obs<OT>(), (float)time_v); }
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

    // ---- phase B: the flat vectors and masks (base_env.py:562-612, base_agent.py:440-460), the policy ----------------
    // Every flat / mask tensor is ONE run written straight from the staged scalars / limits: the four values of a 16-byte
    // group are computed in registers and stored together (store_rows).
    ex([&](int tid) {
        const float *shf = s.shf;
        const uint8_t *hist = e.bid_hist;
        const int sh_full = c.sh_full;
        {   // the planner's flat vector
            const uint16_t *tp = tab + c.tab_p;
            store_rows(o.p_flat<OT>(), 1, c.Fp, 0u, tid, NT, [&](int, int j) { return flat_value(shf, shf, hist, hoff, 0, sh_full, tp[j]); });
        }
        // agents' flat vectors: sorted-key concatenation
        store_rows(o.a_flat<OT>(), A, c.Fa, c.Fa_magic, tid, NT, [&](int a, int j) {
            return flat_value(shf, s.sc_a + a * AS_COUNT, hist, hoff, a * P, sh_full, tab[j]);
        });
        {   // action masks: entry (slot, idx) is open iff idx < limit[agent][slot]
            const uint16_t *mt = tab + c.tab_m;
            store_rows(o.a_mask<OT>(), A, c.Na, c.Na_magic, tid, NT, [&](int a, int j) {
                const uint32_t en = mt[j];
                return ((en & 255u) < s.lim[a * MS_COUNT + (en >> 8)]) ? 1.0f : 0.0f;
            });
        }
        if (!EXT || c.Fpa > 0) {   // the planner's per-agent vectors p<i>
            const uint16_t *tpa = tab + c.tab_pa;
            store_rows(o.p_agents<OT>(), A, c.Fpa, c.Fpa_magic, tid, NT, [&](int a, int j) {
                return flat_value(shf, s.sc_a + a * AS_COUNT, hist, hoff, a * P, sh_full, tpa[j]);
            });
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
                put_out(o.p_mask<OT>() + at, open ? 1.0f : 0.0f);
            }
        } else if (tid == 0) {
            put_out(o.p_mask<OT>(), 1.0f);
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

    if (EXT && c.no_spatial) return;   // one-step-economy: nothing spatial

    // ---- phase C: the planner's spatial tensors: M bit planes of the whole map + the two index planes -----------------
    const int psp = c.pl_stride_p;   // bytes per whole-map plane bitmap
    if (c.planner_spatial || (EXT && c.full_obs)) {
        ex([&](int tid) { planes_from_cells(e.cell, HW, s.pl, psp, M, s.psh, tid, NT); });
    }
    if (c.planner_spatial) {
        int head = 0;
        const int nwords = bits_words_for(o.p_map<OT>(), M * HW, &head);
        ex([&](int tid) {
            concat_planes(s.bits, nwords, head, s.pl, psp, M, HW, c.HW_magic, tid, NT);
            store_bytes_i16<true>(o.p_idx(), HW, (const uint8_t *)e.owner, tid, NT);
            store_bytes_i16<false>(o.p_idx() + HW, HW, s.locmap, tid, NT);
        });
        ex([&](int tid) { stream_bits(o.p_map<OT>(), M * HW, s.bits, lut, s.pl, psp, HW, c.HW_magic, tid, NT); });
    }
    if (EXT && c.full_obs) {
        // full_observability (layout_from_file.py:465-472): every agent gets the whole map - the same M bit planes as
        // the planner - and the two index planes with its own index recoded to 1 (staged as bytes per agent)
        const int HW4 = (HW + 3) & ~3;
        uint8_t *so = s.wi, *sl = s.wi + HW4;
        for (int a = 0; a < A; a++) {
            OT *am = (OT *)o.b->a_map + (o.env * A + a) * (size_t)c.a_map_elems;
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
                stream_bits(am, M * HW, s.bits, lut, s.pl, psp, HW, c.HW_magic, tid, NT);
                store_bytes_i16<false>(ai, HW, so, tid, NT);
                store_bytes_i16<false>(ai + HW, HW, sl, tid, NT);
            });
        }
        return;
    }

    // ---- phase D: agent windows (layout_from_file.py:468-515), a chunk of agents at a time ----------------------------
    // per chunk: a thread takes 8 consecutive window cells of one agent (an 8-cell unit), builds their cell bytes (cell bits
    // | inside flag) in registers and transposes them straight into the plane-local bitmaps, staging the owner / location
    // codes as bytes; the bitmaps are then concatenated and streamed as ONE run of chunk x (M+1) x ww floats, the index
    // planes of the chunk as one run of chunk x 2 x ww int16.
    const int psa = c.pl_stride_a, units = (ww + 7) >> 3, np1 = M + 1;
    for (int a0 = 0; a0 < A; a0 += c.ob_chunk) {
        const int na = (A - a0 < c.ob_chunk) ? A - a0 : c.ob_chunk;
        OT *am = o.a_map<OT>() + (size_t)a0 * np1 * ww;
        int head = 0;
        const int nwords = bits_words_for(am, na * np1 * ww, &head);
        ex([&](int tid) {
            const uint32_t s0 = reinterpret_cast<const uint32_t *>(s.psh)[0], s1 = reinterpret_cast<const uint32_t *>(s.psh)[1];
            const int total = na * units;
            for (int t = tid; t < total; t += NT) {   // one (agent, 8-cell unit) pair per thread and iteration
                const int al = (int)div_magic((uint32_t)t, c.wcu_magic), u = t - al * units, a = a0 + al, q0 = 8 * u;
                int dr = (int)div_magic((uint32_t)q0, c.win_magic), dc = q0 - dr * win;
                const int r0 = e.loc[2 * a] - w, c0 = e.loc[2 * a + 1] - w;
                uint8_t *wi = s.wi + al * 2 * ww;
                uint32_t lo = 0u, hi = 0u;   // the unit's cell bytes, shifted in from the top (cells past ww are 0)
#if AIE_ON_DEVICE
                AIE_UNROLL(1)
#endif
                for (int q = q0; q < q0 + 8; q++) {
                    uint32_t cb = 0;
                    if (q < ww) {
                        const int r2 = r0 + dr, c2 = c0 + dc;
                        int vo = 0, vl = 0;
                        if ((unsigned)r2 < (unsigned)H && (unsigned)c2 < (unsigned)W) {
                            const int k = r2 * W + c2;
                            cb = e.cell[k] | 0x40u;
                            const int ow = e.owner[k];
                            vo = ow < 0 ? 0 : (ow == a ? 1 : ow + 2);
                            vl = s.locmap[k];
                            if (vl == a + 2) vl = 1;
                        }
                        wi[q] = (uint8_t)vo; wi[ww + q] = (uint8_t)vl;
                        if (++dc == win) { dc = 0; dr++; }
                    }
                    lo = fshr(lo, hi, 8); hi = fshr(hi, cb, 8);
                }
                transpose8(lo, hi);
                uint8_t *pq = s.pl + al * np1 * psa + u;
                for (int m = 0; m < np1; m++) { pq[0] = (uint8_t)prmt(lo, hi, ((m < 4 ? s0 : s1) >> (8 * (m & 3))) & 7u); pq += psa; }
            }
        });
        ex([&](int tid) {
            store_bytes_i16<false>(o.a_idx() + (size_t)a0 * 2 * ww, na * 2 * ww, s.wi, tid, NT);
            concat_planes(s.bits, nwords, head, s.pl, psa, na * np1, ww, c.ww_magic, tid, NT);
        });
        ex([&](int tid) { stream_bits(am, na * np1 * ww, s.bits, lut, s.pl, psa, ww, c.ww_magic, tid, NT); });
    }
}

}  // namespace aie
