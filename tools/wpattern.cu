// wpattern.cu — micro-benchmark: how fast can one warp per env stream its observation planes to HBM on H100,
// depending on the store pattern?  (Experiment behind DESIGN.md "observation write-out".)
//
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o /tmp/wpattern tools/wpattern.cu && /tmp/wpattern
//
// Every pattern writes the same bytes: per env a "planner map" of 6 planes x 625 floats followed by 4 "agent
// windows" of 7 planes x 121 floats (28552 B), 8192 envs, 8 warps per CTA, 4 CTAs per SM (shared-memory limited,
// like the step kernel).
#include <cstdio>
#include <cstdlib>
#include <cuda_runtime.h>

constexpr int HW = 625, M = 6, WW = 121, AM = 7, A = 4;
constexpr int ENV_FLOATS = M * HW + A * AM * WW;  // 7138

__device__ __forceinline__ float val(int x, int salt) { return ((x * 2654435761u + salt) >> 31) ? 1.0f : 0.0f; }

// spin: `work` dependent integer ops, result folded into the value so it is not dead code
__device__ __forceinline__ int spin(int x, int work) {
    for (int i = 0; i < work; i++) x = x * 1664525 + 1013904223;
    return x;
}

template <int PAT>
__global__ void __launch_bounds__(256, 4) kern(float *out, int n_env, int stride, int work) {
    extern __shared__ float sm[];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int env = blockIdx.x * 8 + warp;
    if (env >= n_env) return;
    float *base = out + (size_t)env * stride;
    if (PAT == 0) {  // contiguous 16-byte stores over the whole env slice (stride must be a multiple of 4 floats)
        float4 *b4 = (float4 *)base;
        for (int i = lane; i < ENV_FLOATS / 4; i += 32) {
            int s = spin(i, work);
            b4[i] = make_float4(val(i, s), val(i + 1, s), val(i + 2, s), val(i + 3, s));
        }
    } else if (PAT == 1) {  // cell-major: one cell fans out to all planes (current kernel)
        for (int k = lane; k < HW; k += 32) {
            int s = spin(k, work);
#pragma unroll
            for (int m = 0; m < M; m++) base[m * HW + k] = val(k, s + m);
        }
        for (int a = 0; a < A; a++) {
            float *am = base + M * HW + a * AM * WW;
            for (int q = lane; q < WW; q += 32) {
                int s = spin(q, work);
#pragma unroll
                for (int m = 0; m < AM; m++) am[m * WW + q] = val(q, s + m);
            }
        }
    } else if (PAT == 2) {  // plane-major scalar stores: the env slice is written front to back
        for (int i = lane; i < ENV_FLOATS; i += 32) {
            int s = spin(i, work / 6);
            base[i] = val(i, s);
        }
    } else if (PAT == 3) {  // front to back, 16-byte stores with a scalar head/tail (any 4-byte alignment)
        const int mis = (int)(((size_t)base >> 2) & 3);  // floats past a 16-byte boundary
        const int head = (4 - mis) & 3;
        if (lane < head) base[lane] = val(lane, 1);
        float4 *b4 = (float4 *)(base + head);
        const int n4 = (ENV_FLOATS - head) / 4;
        for (int i = lane; i < n4; i += 32) {
            int s = spin(i, work);
            int f = head + 4 * i;
            b4[i] = make_float4(val(f, s), val(f + 1, s), val(f + 2, s), val(f + 3, s));
        }
        const int done = head + 4 * n4;
        if (lane < ENV_FLOATS - done) base[done + lane] = val(done + lane, 1);
    } else if (PAT == 4) {  // cell-major, but 4 cells per lane: 16-byte stores per plane where alignment allows (8-byte here)
        for (int k = 2 * lane; k < HW - 1; k += 64) {
            int s = spin(k, work);
#pragma unroll
            for (int m = 0; m < M; m++) {
                float *p = base + m * HW + k;
                if ((((size_t)p) & 7) == 0) *(float2 *)p = make_float2(val(k, s + m), val(k + 1, s + m));
                else { p[0] = val(k, s + m); p[1] = val(k + 1, s + m); }
            }
        }
        if (lane < M) base[lane * HW + HW - 1] = 1.0f;
        for (int i = M * HW + lane; i < ENV_FLOATS; i += 32) base[i] = val(i, 3);
    }
}

template <int PAT>
float run(float *buf, int n_env, int stride, int work, int reps) {
    cudaFuncSetAttribute(kern<PAT>, cudaFuncAttributeMaxDynamicSharedMemorySize, 46 * 1024);
    cudaEvent_t s, e;
    cudaEventCreate(&s); cudaEventCreate(&e);
    const int grid = (n_env + 7) / 8;
    for (int i = 0; i < 3; i++) kern<PAT><<<grid, 256, 46 * 1024>>>(buf, n_env, stride, work);
    cudaEventRecord(s);
    for (int i = 0; i < reps; i++) kern<PAT><<<grid, 256, 46 * 1024>>>(buf, n_env, stride, work);
    cudaEventRecord(e);
    cudaEventSynchronize(e);
    float ms; cudaEventElapsedTime(&ms, s, e);
    cudaError_t err = cudaGetLastError();
    if (err != cudaSuccess) printf("CUDA error %s\n", cudaGetErrorString(err));
    return ms / reps;
}

int main() {
    const int n_env = 8192, reps = 20;
    float *buf;
    const size_t cap = (size_t)n_env * 8192 * sizeof(float);
    cudaMalloc(&buf, cap);
    const char *names[] = {"contig16B", "cell-major(cur)", "front-to-back 4B", "front-to-back 16B+peel", "cell-major 8B"};
    for (int work : {0, 40, 160}) {
        for (int stride : {ENV_FLOATS, 7140, 7168}) {
            printf("work=%d stride=%d floats (%d B/env, %.0f MB)\n", work, stride, ENV_FLOATS * 4, n_env * ENV_FLOATS * 4 / 1e6);
            float t[5] = {0, 0, 0, 0, 0};
            if (stride % 4 == 0) t[0] = run<0>(buf, n_env, stride, work, reps);
            t[1] = run<1>(buf, n_env, stride, work, reps);
            t[2] = run<2>(buf, n_env, stride, work, reps);
            t[3] = run<3>(buf, n_env, stride, work, reps);
            t[4] = run<4>(buf, n_env, stride, work, reps);
            for (int p = 0; p < 5; p++)
                if (t[p] > 0) printf("  %-26s %8.1f us  %7.0f GB/s\n", names[p], t[p] * 1e3, n_env * (double)ENV_FLOATS * 4 / t[p] / 1e6);
        }
    }
    return 0;
}
