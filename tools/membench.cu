// membench.cu — isolates the streaming patterns of the fast join kernels (which loads/stores reach HBM speed?).
// Build: nvcc -O3 -gencode arch=compute_90a,code=sm_90a -o membench tools/membench.cu
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#define CK(x) do { cudaError_t e = (x); if (e != cudaSuccess) { printf("CUDA error %s at %d\n", cudaGetErrorString(e), __LINE__); exit(1); } } while (0)
__device__ __forceinline__ uint64_t mix(uint64_t x) { x += 0x9E3779B97F4A7C15ULL; x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ULL; x = (x ^ (x >> 27)) * 0x94D049BB133111EBULL; return x ^ (x >> 31); }

template <int MODE>  // 0 plain, 1 .cs both, 2 .cs loads only, 3 .cs stores only
__global__ void k_copy(const int4 *__restrict__ a, int4 *__restrict__ b, size_t n) {
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        int4 v = (MODE == 1 || MODE == 2) ? __ldcs(a + i) : a[i];
        if (MODE == 1 || MODE == 3) __stcs(b + i, v); else b[i] = v;
    }
}
// AoS rows in -> 6 SoA columns out (8,4,4,8,4,4 B), RPT rows per thread in flight
template <int MODE, int RPT>
__global__ void k_soa(const int4 *__restrict__ in, long long *c0, int *c1, int *c2, long long *c3, int *c4, int *c5, size_t n, size_t shift) {
    size_t tile = (size_t)blockDim.x * RPT;
    for (size_t t0 = blockIdx.x * tile; t0 < n; t0 += (size_t)gridDim.x * tile) {
        int4 v[RPT];
#pragma unroll
        for (int k = 0; k < RPT; k++) { size_t r = t0 + k * blockDim.x + threadIdx.x; v[k] = r < n ? (MODE ? __ldcs(in + r) : in[r]) : make_int4(0, 0, 0, 0); }
#pragma unroll
        for (int k = 0; k < RPT; k++) {
            size_t r = t0 + k * blockDim.x + threadIdx.x; if (r >= n) continue;
            size_t p = r + shift;
            long long key = ((long long)v[k].y << 32) | (unsigned)v[k].x;
            if (MODE) { __stcs(c0 + p, key); __stcs(c1 + p, v[k].z); __stcs(c2 + p, v[k].w); __stcs(c3 + p, key); __stcs(c4 + p, v[k].z ^ 1); __stcs(c5 + p, v[k].w ^ 1); }
            else { c0[p] = key; c1[p] = v[k].z; c2[p] = v[k].w; c3[p] = key; c4[p] = v[k].z ^ 1; c5[p] = v[k].w ^ 1; }
        }
    }
}
// 3 SoA columns in -> AoS 16 B rows out, in order (no scatter)
template <int MODE, int RPT>
__global__ void k_aos(const long long *c0, const int *c1, const int *c2, int4 *out, size_t n) {
    size_t tile = (size_t)blockDim.x * RPT;
    for (size_t t0 = blockIdx.x * tile; t0 < n; t0 += (size_t)gridDim.x * tile) {
        long long a[RPT]; int b[RPT], c[RPT];
#pragma unroll
        for (int k = 0; k < RPT; k++) { size_t r = t0 + k * blockDim.x + threadIdx.x; bool ok = r < n; a[k] = ok ? (MODE ? __ldcs(c0 + r) : c0[r]) : 0; b[k] = ok ? (MODE ? __ldcs(c1 + r) : c1[r]) : 0; c[k] = ok ? (MODE ? __ldcs(c2 + r) : c2[r]) : 0; }
#pragma unroll
        for (int k = 0; k < RPT; k++) { size_t r = t0 + k * blockDim.x + threadIdx.x; if (r >= n) continue; int4 v = make_int4((int)a[k], (int)(a[k] >> 32), b[k], c[k]); if (MODE) __stcs(out + r, v); else out[r] = v; }
    }
}
// scatter: like k_fj_scatter_sm's flush.  One 1024-thread block per SM walks its rows in tiles of T rows; a tile is
// cut into P runs in partition order (run p is tile rows [bound(p), bound(p+1)), bound(p) = p * T / P), and run p of
// the block's t-th tile goes to partition p's region, behind the same run of every earlier tile.  n is a multiple of
// gridDim.x * T, so every row is read once and written once (a bijection), 16 bytes each way.
__global__ void __launch_bounds__(1024, 1) k_runs(const int4 *__restrict__ in, int4 *out, size_t n, int P, int T) {
    const size_t ntiles = n / T, tpb = ntiles / gridDim.x;
    for (size_t t = 0; t < tpb; t++) {
        const size_t tile = blockIdx.x * tpb + t, t0 = tile * T;
        for (int i = threadIdx.x; i < T; i += blockDim.x) {
            const int p = (int)(((long long)(i + 1) * P - 1) / T);
            const size_t lo = (size_t)p * T / P, len = (size_t)(p + 1) * T / P - lo;
            __stcs(out + lo * ntiles + tile * len + (i - lo), __ldcs(in + t0 + i));
        }
    }
}
template <typename F> static float timeit(F f) { cudaEvent_t a, b; cudaEventCreate(&a); cudaEventCreate(&b); f(); CK(cudaDeviceSynchronize()); float best = 1e30f; for (int i = 0; i < 3; i++) { cudaEventRecord(a); f(); cudaEventRecord(b); CK(cudaEventSynchronize(b)); float ms; cudaEventElapsedTime(&ms, a, b); if (ms < best) best = ms; } return best; }
int main() {
    int sms; cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0);
    size_t n = (size_t)1 << 28;
    int4 *in, *out; CK(cudaMalloc(&in, n * 16)); CK(cudaMalloc(&out, n * 32 + 4096)); CK(cudaMemset(in, 1, n * 16));
    long long *c0 = (long long *)out, *c3 = c0 + n + 64; int *c1 = (int *)(c3 + n + 64), *c2 = c1 + n + 64, *c4 = c2 + n + 64, *c5 = c4 + n + 64;
    int g = sms * 8;
    printf("copy plain (16 B in, 16 B out): %.1f GB/s\n", n * 32.0 / timeit([&] { k_copy<0><<<g, 256>>>(in, out, n); }) / 1e6);
    printf("copy .cs ld+st  : %.1f GB/s\n", n * 32.0 / timeit([&] { k_copy<1><<<g, 256>>>(in, out, n); }) / 1e6);
    printf("copy .cs ld     : %.1f GB/s\n", n * 32.0 / timeit([&] { k_copy<2><<<g, 256>>>(in, out, n); }) / 1e6);
    printf("copy .cs st     : %.1f GB/s\n", n * 32.0 / timeit([&] { k_copy<3><<<g, 256>>>(in, out, n); }) / 1e6);
    for (int sh = 0; sh <= 3; sh += 3) {
        printf("AoS->6 SoA plain RPT4 shift %d: %.1f GB/s\n", sh, n * 48.0 / timeit([&] { k_soa<0, 4><<<sms * 6, 256>>>(in, c0, c1, c2, c3, c4, c5, n, sh); }) / 1e6);
        printf("AoS->6 SoA .cs   RPT4 shift %d: %.1f GB/s\n", sh, n * 48.0 / timeit([&] { k_soa<1, 4><<<sms * 6, 256>>>(in, c0, c1, c2, c3, c4, c5, n, sh); }) / 1e6);
        printf("AoS->6 SoA .cs   RPT8 shift %d: %.1f GB/s\n", sh, n * 48.0 / timeit([&] { k_soa<1, 8><<<sms * 4, 256>>>(in, c0, c1, c2, c3, c4, c5, n, sh); }) / 1e6);
    }
    printf("3 SoA->AoS plain RPT8: %.1f GB/s\n", n * 32.0 / timeit([&] { k_aos<0, 8><<<sms * 4, 256>>>(c0, c1, c2, in, n); }) / 1e6);
    printf("3 SoA->AoS .cs   RPT8: %.1f GB/s\n", n * 32.0 / timeit([&] { k_aos<1, 8><<<sms * 4, 256>>>(c0, c1, c2, in, n); }) / 1e6);
    CK(cudaMemset(in, 1, n * 16));
    // (P, T): runs of T / P rows; the last line is C2's probe scatter (287 partitions, 6144-row tiles, 16-byte rows)
    const int geo[][2] = {{256, 2048}, {256, 5376}, {256, 16384}, {96, 768}, {96, 2016}, {96, 6144}, {287, 6027}, {287, 6314},
                          {287, 4592}, {287, 9184}, {287, 6144}};
    for (auto &pt : geo) {
        const int P = pt[0], T = pt[1];
        const size_t m = n / ((size_t)sms * T) * sms * T;
        float ms = timeit([&] { k_runs<<<sms, 1024>>>(in, out, m, P, T); });
        printf("scatter runs P=%3d T=%5d (%.1f rows/run): %.3f ms -> %.1f GB/s (every row read and written once)\n", P, T,
               (double)T / P, ms, m * 32.0 / ms / 1e6);
    }
    return 0;
}
