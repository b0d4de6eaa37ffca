// Generic int32 inclusive scan (tile sums -> one-CTA scan of the tile sums -> apply), shared by
// the device shuffle (shuffle.cu) and the data-preparation passes (prepare.cu).
//   off[k] = x[0] + ... + x[k]  for k < n;  tsum: int32[ceil(n / SC_TILE)] scratch.
// An exclusive scan with the total at the end is the same call with off + 1 and off[0] = 0.
#pragma once

#include <stdint.h>

namespace {

constexpr int SC_TILE = 4096, SC_THREADS = 256, SC_ITEMS = 16;

__global__ void __launch_bounds__(SC_THREADS)
scan_tilesum_kernel(const int32_t* __restrict__ x, int64_t n, int32_t* tsum) {
    __shared__ int sh[SC_THREADS / 32];
    const int64_t base = static_cast<int64_t>(blockIdx.x) * SC_TILE;
    int s = 0;
#pragma unroll
    for (int r = 0; r < SC_ITEMS; ++r) {
        const int64_t k = base + r * SC_THREADS + threadIdx.x;
        if (k < n) s += x[k];
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = s;
    __syncthreads();
    if (threadIdx.x == 0) {
        int t = 0;
        for (int w = 0; w < SC_THREADS / 32; ++w) t += sh[w];
        tsum[blockIdx.x] = t;
    }
}

__global__ void __launch_bounds__(1024) scan_tiles_kernel(int32_t* tsum, int ntiles) {
    __shared__ int shw[32];
    const int per = (ntiles + 1023) / 1024;
    const int lo = threadIdx.x * per, hi = min(lo + per, ntiles);
    int s = 0;
    for (int k = lo; k < hi; ++k) s += tsum[k];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    int inc = s;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const int a = __shfl_up_sync(0xffffffffu, inc, o);
        if (lane >= o) inc += a;
    }
    if (lane == 31) shw[warp] = inc;
    __syncthreads();
    int pre = inc - s;
    for (int w = 0; w < warp; ++w) pre += shw[w];
    for (int k = lo; k < hi; ++k) { const int c = tsum[k]; tsum[k] = pre; pre += c; }
}

__global__ void __launch_bounds__(SC_THREADS)
scan_apply_kernel(const int32_t* __restrict__ x, int64_t n, const int32_t* __restrict__ tsum,
                  int32_t* __restrict__ off) {
    __shared__ int sh[SC_THREADS / 32];
    const int64_t first = static_cast<int64_t>(blockIdx.x) * SC_TILE + threadIdx.x * SC_ITEMS;
    int c[SC_ITEMS];
    int s = 0;
#pragma unroll
    for (int r = 0; r < SC_ITEMS; ++r) { c[r] = first + r < n ? x[first + r] : 0; s += c[r]; }
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    int inc = s;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const int a = __shfl_up_sync(0xffffffffu, inc, o);
        if (lane >= o) inc += a;
    }
    if (lane == 31) sh[warp] = inc;
    __syncthreads();
    int pre = tsum[blockIdx.x] + inc - s;
    for (int w = 0; w < warp; ++w) pre += sh[w];
#pragma unroll
    for (int r = 0; r < SC_ITEMS; ++r) {
        pre += c[r];
        if (first + r < n) off[first + r] = pre;         // inclusive: one past the segment's last slot
    }
}

inline int scan_tiles_for(int64_t n) { return static_cast<int>((n + SC_TILE - 1) / SC_TILE); }

}  // namespace
