// Shared device/host helpers for the spotlight_b200 kernels (sm_90a).
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include <type_traits>

#include "../../include/spotlight_b200.h"

void slb_set_error(const char* fmt, ...);
int slb_sms();

#define SLB_REQUIRE(cond, ...)                 \
    do {                                       \
        if (!(cond)) {                         \
            slb_set_error(__VA_ARGS__);        \
            return SLB_EINVAL;                 \
        }                                      \
    } while (0)

#define SLB_LAUNCH_CHECK(name)                                                   \
    do {                                                                         \
        cudaError_t e__ = cudaGetLastError();                                    \
        if (e__ != cudaSuccess) {                                                \
            slb_set_error("%s: launch failed: %s", name, cudaGetErrorString(e__)); \
            return SLB_ECUDA;                                                    \
        }                                                                        \
    } while (0)

static inline size_t slb_align_up(size_t x, size_t a) { return (x + a - 1) / a * a; }

// Grid of `want` blocks, at least one and at most per_sm per SM.
static inline int slb_grid(int64_t want, int per_sm) {
    const int64_t cap = static_cast<int64_t>(slb_sms()) * per_sm;
    const int64_t g = want < cap ? want : cap;
    return g < 1 ? 1 : static_cast<int>(g);
}

// Lanes per row of width D: one 128-bit piece per lane, a power of two, at most a warp.
static inline int lpr_for_dim(int D) {
    const int l = D / 4;
    int p = 1;
    while (p < l && p < 32) p <<= 1;
    return p;
}

// Calls f(std::integral_constant<int, L>{}) for the lane count L == lpr, L a power of two from
// FIRST to 32 (any other lpr gets 32): a launch site names its kernel once, for every L.
template <int FIRST = 1, typename F>
void with_lpr(int lpr, F&& f) {
    if constexpr (FIRST == 32) f(std::integral_constant<int, 32>{});
    else if (lpr == FIRST) f(std::integral_constant<int, FIRST>{});
    else with_lpr<2 * FIRST>(lpr, f);
}

// f(std::true_type{}) or f(std::false_type{}): a run-time flag as a compile-time kernel parameter.
template <typename F>
void with_bool(bool b, F&& f) {
    if (b) f(std::true_type{});
    else f(std::false_type{});
}

// Carves sub-buffers out of a caller-owned workspace (256 B aligned).
struct WsCarver {
    char* base;
    size_t off;
    explicit WsCarver(void* p) : base(static_cast<char*>(p)), off(0) {}
    template <typename T>
    T* take(size_t count) {
        off = slb_align_up(off, 256);
        T* p = base ? reinterpret_cast<T*>(base + off) : nullptr;
        off += count * sizeof(T);
        return p;
    }
    size_t bytes() const { return slb_align_up(off, 256); }
};

#ifdef __CUDACC__

__device__ __forceinline__ float4 ldg4(const float* p) {
    return __ldg(reinterpret_cast<const float4*>(p));
}
__device__ __forceinline__ float4 ld4(const float* p) {
    return *reinterpret_cast<const float4*>(p);
}
__device__ __forceinline__ void st4(float* p, float4 v) { *reinterpret_cast<float4*>(p) = v; }

__device__ __forceinline__ float dot4(float4 a, float4 b) {
    return a.x * b.x + a.y * b.y + a.z * b.z + a.w * b.w;
}
__device__ __forceinline__ void fma4(float4& acc, float g, float4 v) {
    acc.x = fmaf(g, v.x, acc.x);
    acc.y = fmaf(g, v.y, acc.y);
    acc.z = fmaf(g, v.z, acc.z);
    acc.w = fmaf(g, v.w, acc.w);
}

// Sum over the LPR consecutive lanes of a group (LPR power of two <= 32);
// every lane of the group gets the result.  `mask` names exactly the lanes
// that execute this call.
template <int LPR>
__device__ __forceinline__ float group_sum(float v, unsigned mask) {
#pragma unroll
    for (int o = LPR / 2; o > 0; o >>= 1) v += __shfl_xor_sync(mask, v, o);
    return v;
}

__device__ __forceinline__ unsigned group_mask(int lpr) {
    const int lane = threadIdx.x & 31;
    const unsigned m = lpr == 32 ? 0xffffffffu : ((1u << lpr) - 1u);
    return m << (lane & ~(lpr - 1));
}

__device__ __forceinline__ float sigmoidf_(float x) { return 1.0f / (1.0f + expf(-x)); }

// Block-wide sum; result valid in thread 0.  Fixed reduction tree -> deterministic.
template <int THREADS>
__device__ __forceinline__ float block_sum(float v, float* smem /* THREADS/32 floats */) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
    const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
    if (l == 0) smem[w] = v;
    __syncthreads();
    if (w == 0) {
        v = l < THREADS / 32 ? smem[l] : 0.f;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
    }
    return v;
}

// Deterministic grid-wide sum without float atomics: every block stores its block_sum of v in
// partial[blockIdx.x] and takes a ticket; the last block to arrive sums the partials, then (EXTRA)
// extra[0..n_extra), lane-strided in a fixed order, and folds the warp with a fixed shuffle tree.
// Returns true in that block's thread 0, with the sum in `total`.  The caller writes the result
// and, if it reuses the ticket, resets it.  sh_red (THREADS / 32 floats) and is_last are the
// caller's shared memory, so that they keep their place in its layout.  EXTRA is a compile-time
// switch because the compiler keeps the second loop even for a constant n_extra == 0.
template <int THREADS, bool EXTRA = false>
__device__ __forceinline__ bool grid_fold(float v, float* sh_red, bool& is_last, float* partial, int32_t* ticket,
                                          float& total, const float* extra = nullptr, int n_extra = 0) {
    const float bsum = block_sum<THREADS>(v, sh_red);
    if (threadIdx.x == 0) {
        partial[blockIdx.x] = bsum;
        __threadfence();
        is_last = atomicAdd(ticket, 1) == static_cast<int>(gridDim.x) - 1;
    }
    __syncthreads();
    bool first = false;
    if (is_last && threadIdx.x < 32) {
        __threadfence();
        float t = 0.f;
        for (int k = threadIdx.x; k < static_cast<int>(gridDim.x); k += 32)
            t += *reinterpret_cast<volatile float*>(partial + k);
        if (EXTRA)
            for (int k = threadIdx.x; k < n_extra; k += 32)
                t += *reinterpret_cast<const volatile float*>(extra + k);
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) t += __shfl_down_sync(0xffffffffu, t, o);
        total = t;
        first = threadIdx.x == 0;
    }
    return first;
}

// d loss_b / d pos and d loss_b / d neg (unscaled by 1/B), and the loss term, of one pair of
// scores: bpr, pointwise, or hinge (adaptive hinge on its selected negative).
__device__ __forceinline__ void pair_loss(int loss, float p, float n, float& per, float& gp, float& gn) {
    if (loss == SLB_LOSS_BPR) {
        const float s = sigmoidf_(p - n);
        per = 1.0f - s;
        gp = -s * (1.0f - s);
        gn = -gp;
    } else if (loss == SLB_LOSS_POINTWISE) {
        const float sp = sigmoidf_(p), sn = sigmoidf_(n);
        per = (1.0f - sp) + sn;
        gp = -sp * (1.0f - sp);
        gn = sn * (1.0f - sn);
    } else {
        const float z = n - p + 1.0f;
        per = fmaxf(z, 0.0f);
        const float act = z >= 0.0f ? 1.0f : 0.0f;  // clamp backward passes at the boundary
        gp = -act;
        gn = act;
    }
}

// MurmurHash3_x86_32 of the 4 little-endian bytes of a 32-bit key
// (sklearn.utils.murmurhash3_32 on an int32 array; spotlight/layers.py:183).
__device__ __forceinline__ uint32_t murmur3_32(uint32_t k, uint32_t seed) {
    k *= 0xcc9e2d51u;
    k = (k << 15) | (k >> 17);
    k *= 0x1b873593u;
    uint32_t h = seed ^ k;
    h = (h << 13) | (h >> 19);
    h = h * 5u + 0xe6546b64u;
    h ^= 4u;
    h ^= h >> 16;
    h *= 0x85ebca6bu;
    h ^= h >> 13;
    h *= 0xc2b2ae35u;
    h ^= h >> 16;
    return h;
}

// BloomEmbedding row: int32(hash) floor-mod rows, 0 for the padding id
// (spotlight/layers.py:183-186).
__device__ __forceinline__ int64_t bloom_row(int64_t id, uint32_t seed, int64_t rows,
                                             int64_t padding_idx) {
    if (id == padding_idx) return 0;
    const int64_t h = static_cast<int32_t>(murmur3_32(static_cast<uint32_t>(id), seed));
    int64_t m = h % rows;
    if (m < 0) m += rows;
    return m;
}

// ---- row-wise optimizers shared by the MF and sequence kernels --------------------------------
// Adagrad step  w -= lr * g / (sqrt(s) + eps)  with MUFU-based sqrt and division (rsqrt 2 ulp,
// fast divide 2 ulp: ~5e-7 relative, far inside the 1e-5 parity budget; the IEEE sqrtf +
// division pair costs ~20 instructions per element and made the update kernels issue-bound).
__device__ __forceinline__ float adagrad_delta(float lr, float g, float s, float eps) {
    const float root = s > 0.f ? s * rsqrtf(s) : 0.f;
    return __fdividef(lr * g, root + eps);
}

struct OptV2 { int32_t opt; float lr, wd, eps; };

__device__ __forceinline__ void row_update(const OptV2& o, float4& w, float4& s, const float4& g0) {
    float gv[4] = {g0.x + o.wd * w.x, g0.y + o.wd * w.y, g0.z + o.wd * w.z, g0.w + o.wd * w.w};
    float wv[4] = {w.x, w.y, w.z, w.w};
    if (o.opt == SLB_OPT_SGD) {
#pragma unroll
        for (int q = 0; q < 4; ++q) wv[q] -= o.lr * gv[q];
    } else {
        float sv[4] = {s.x, s.y, s.z, s.w};
#pragma unroll
        for (int q = 0; q < 4; ++q) {
            sv[q] += gv[q] * gv[q];
            wv[q] -= adagrad_delta(o.lr, gv[q], sv[q], o.eps);
        }
        s = make_float4(sv[0], sv[1], sv[2], sv[3]);
    }
    w = make_float4(wv[0], wv[1], wv[2], wv[3]);
}

__device__ __forceinline__ void bias_update(const OptV2& o, float* bw, float* bs, float g) {
    const float gb = g + o.wd * *bw;
    if (o.opt == SLB_OPT_SGD) {
        *bw -= o.lr * gb;
    } else {
        const float sv = *bs + gb * gb;
        *bs = sv;
        *bw -= adagrad_delta(o.lr, gb, sv, o.eps);
    }
}

// ---- row-wise lazy-exact Adam shared by the MF (mf_adam.cuh) and sequence kernels -------------
// Per-step scalars (computed by the host in double, as torch does):
//   sched[2t] = lr / (1 - beta1^t)      sched[2t+1] = sqrt(1 - beta2^t)
struct AdamDev {
    float beta1, beta2, omb1, omb2, eps, wd;
    const float* sched;       // [2 * (t_max + 1)]
    int32_t t;                // this step (1-based)
};

// one Adam step on one element (torch/optim/adam.py, _single_tensor_adam / foreach form)
__device__ __forceinline__ void adam_elem(const AdamDev& o, float ss, float bc2s, float g, float& w, float& m, float& v) {
    g += o.wd * w;
    m += (g - m) * o.omb1;                       // exp_avg.lerp_(grad, 1 - beta1)
    v = v * o.beta2 + o.omb2 * g * g;            // mul_(beta2).addcmul_(grad, grad, 1 - beta2)
    const float denom = sqrtf(v) / bc2s + o.eps;
    w -= ss * (m / denom);                                  // addcdiv_(exp_avg, denom, value=-step_size)
}

// replay steps (from, to] with zero data gradient
__device__ __forceinline__ void adam_catch_up(const AdamDev& o, int from, int to, float4& w, float4& m, float4& v) {
    // a row that was never touched has m = v = 0: without weight decay nothing moves
    if (from >= to) return;
    if (o.wd == 0.f && m.x == 0.f && m.y == 0.f && m.z == 0.f && m.w == 0.f &&
        v.x == 0.f && v.y == 0.f && v.z == 0.f && v.w == 0.f) return;
    for (int s = from + 1; s <= to; ++s) {
        const float ss = __ldg(o.sched + 2 * s), bc = __ldg(o.sched + 2 * s + 1);
        adam_elem(o, ss, bc, 0.f, w.x, m.x, v.x);
        adam_elem(o, ss, bc, 0.f, w.y, m.y, v.y);
        adam_elem(o, ss, bc, 0.f, w.z, m.z, v.z);
        adam_elem(o, ss, bc, 0.f, w.w, m.w, v.w);
    }
}

__device__ __forceinline__ void adam_catch_up1(const AdamDev& o, int from, int to, float& w, float& m, float& v) {
    if (from >= to || (o.wd == 0.f && m == 0.f && v == 0.f)) return;
    for (int s = from + 1; s <= to; ++s)
        adam_elem(o, __ldg(o.sched + 2 * s), __ldg(o.sched + 2 * s + 1), 0.f, w, m, v);
}

#endif  // __CUDACC__
