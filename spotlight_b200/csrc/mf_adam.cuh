// Row-wise LAZY-EXACT Adam for the embedding tables.
//
// The reference's default optimizer is dense torch.optim.Adam
// (spotlight/factorization/implicit.py:143-148): every row of every table is rewritten
// every minibatch -- rows without a gradient still move, because their first moment decays
// geometrically.  That sweep is O(table) per step.  Here a row is brought up to date only
// when it is touched: the steps it missed (gradient 0, or weight_decay * w) are replayed for
// it element by element -- the same recurrence torch runs, in the same order -- and then the
// real step is applied.  `last[row]` remembers the step a row is current for; adam_flush
// replays the pending steps of every row (end of fit(), before parameters are read).  The
// result equals dense Adam up to fp32 rounding of identical formulas; the cost per step is
// O(touched rows x steps missed), never more arithmetic than the dense sweep did.
//
// Per-step scalars (computed by the host in double, as torch does):
//   sched[2t] = lr / (1 - beta1^t)      sched[2t+1] = sqrt(1 - beta2^t)
#pragma once

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

// Before the forward pass of step t every row the minibatch references must be current through
// step t-1 (dense Adam moved it at every step it missed, and the scores must see that).  One
// lane group per reference (user / positive item / negative item); atomicMax on last[row] elects
// exactly one group per distinct row to replay its pending steps; the others find it current.
template <int LPR>
__global__ void __launch_bounds__(MF_THREADS)
mf_adam_prepass_kernel(MfDev a, AdamDev o, float* vWu, float* vWi, float* vbu, float* vbi, int32_t* last_u, int32_t* last_i) {
    constexpr int GROUPS = MF_THREADS / LPR;
    const int gl = threadIdx.x & (LPR - 1);
    const int gib = threadIdx.x / LPR;
    const unsigned gmask = group_mask(LPR);
    const int D = a.D;
    const int64_t nneg = a.negs ? a.B * a.n_neg : 0;       // rating losses have no negatives
    const int64_t total = 2 * a.B + nneg;
    const int upto = o.t - 1;
    if (upto <= 0) return;
    for (int64_t r = static_cast<int64_t>(blockIdx.x) * GROUPS + gib; r < total; r += static_cast<int64_t>(gridDim.x) * GROUPS) {
        const bool isA = r < a.B;
        const int64_t row = isA ? a.users[r] : (r < 2 * a.B ? a.items[r - a.B] : a.negs[r - 2 * a.B]);
        if (row < 0 || row >= (isA ? a.U : a.I)) continue;                // the forward flags bad ids
        int old = 0;
        if (gl == 0) old = atomicMax((isA ? last_u : last_i) + row, upto);
        old = __shfl_sync(gmask, old, (threadIdx.x & 31) & ~(LPR - 1));
        if (old >= upto) continue;
        float* W = (isA ? a.Wu : a.Wi) + row * D;
        float* M = (isA ? a.sWu : a.sWi) + row * D;
        float* V = (isA ? vWu : vWi) + row * D;
        for (int c = gl * 4; c < D; c += LPR * 4) {
            float4 w = ld4(W + c), m = ld4(M + c), v = ld4(V + c);
            adam_catch_up(o, old, upto, w, m, v);
            st4(W + c, w); st4(M + c, m); st4(V + c, v);
        }
        if (gl == 0) {
            float* bw = (isA ? a.bu : a.bi) + row;
            float* bm = (isA ? a.sbu : a.sbi) + row;
            float* bv = (isA ? vbu : vbi) + row;
            float w = *bw, m = *bm, v = *bv;
            adam_catch_up1(o, old, upto, w, m, v);
            *bw = w; *bm = m; *bv = v;
        }
    }
}

// Adam on the touched rows, from the compact gradients of the step (rows ascending in
// urows / irows, gradient row k in gWu / gWi, bias gradient in gbu / gbi).
template <int LPR>
__global__ void __launch_bounds__(MF_THREADS)
mf_adam_apply_kernel(MfDev a, AdamDev o, float* vWu, float* vWi, float* vbu, float* vbi, int32_t* last_u, int32_t* last_i) {
    constexpr int GROUPS = MF_THREADS / LPR;
    const int gl = threadIdx.x & (LPR - 1);
    const int gib = threadIdx.x / LPR;
    const int D = a.D;
    const int nseg = a.seg.totals[0];
    const int nsegA = a.seg.totals[2];
    const float ss = o.sched[2 * o.t], bc = o.sched[2 * o.t + 1];
    for (int64_t s = static_cast<int64_t>(blockIdx.x) * GROUPS + gib; s < nseg; s += static_cast<int64_t>(gridDim.x) * GROUPS) {
        const bool isA = s < nsegA;
        const int64_t k = isA ? s : s - nsegA;
        const int64_t row = isA ? a.urows[k] : a.irows[k];
        if (row < 0) continue;
        float* W = (isA ? a.Wu : a.Wi) + row * D;
        float* M = (isA ? a.sWu : a.sWi) + row * D;
        float* V = (isA ? vWu : vWi) + row * D;
        const float* G = (isA ? a.gWu : a.gWi) + k * D;
        int32_t* lastp = (isA ? last_u : last_i) + row;
        const int last = *lastp;
        for (int c = gl * 4; c < D; c += LPR * 4) {
            float4 w = ld4(W + c), m = ld4(M + c), v = ld4(V + c);
            const float4 g = ld4(G + c);
            adam_catch_up(o, last, o.t - 1, w, m, v);
            adam_elem(o, ss, bc, g.x, w.x, m.x, v.x);
            adam_elem(o, ss, bc, g.y, w.y, m.y, v.y);
            adam_elem(o, ss, bc, g.z, w.z, m.z, v.z);
            adam_elem(o, ss, bc, g.w, w.w, m.w, v.w);
            st4(W + c, w); st4(M + c, m); st4(V + c, v);
        }
        __syncwarp(group_mask(LPR));          // every lane has read `last` before it moves
        if (gl == 0) {
            float* bw = (isA ? a.bu : a.bi) + row;
            float* bm = (isA ? a.sbu : a.sbi) + row;
            float* bv = (isA ? vbu : vbi) + row;
            float w = *bw, m = *bm, v = *bv;
            adam_catch_up1(o, last, o.t - 1, w, m, v);
            adam_elem(o, ss, bc, (isA ? a.gbu : a.gbi)[k], w, m, v);
            *bw = w; *bm = m; *bv = v;
            *lastp = o.t;
        }
    }
}

// Replays the pending steps of every row up to and including step o.t (no data gradient).
template <int LPR>
__global__ void __launch_bounds__(MF_THREADS)
adam_flush_kernel(float* W, float* M, float* V, float* bw, float* bm, float* bv, int32_t* last, int64_t rows, int D,
                  AdamDev o) {
    constexpr int GROUPS = MF_THREADS / LPR;
    const int gl = threadIdx.x & (LPR - 1);
    const int gib = threadIdx.x / LPR;
    for (int64_t row = static_cast<int64_t>(blockIdx.x) * GROUPS + gib; row < rows; row += static_cast<int64_t>(gridDim.x) * GROUPS) {
        const int lastv = last[row];
        if (lastv >= o.t) continue;
        for (int c = gl * 4; c < D; c += LPR * 4) {
            float4 w = ld4(W + row * D + c), m = ld4(M + row * D + c), v = ld4(V + row * D + c);
            adam_catch_up(o, lastv, o.t, w, m, v);
            st4(W + row * D + c, w); st4(M + row * D + c, m); st4(V + row * D + c, v);
        }
        __syncwarp(group_mask(LPR));
        if (gl == 0) {
            float w = bw[row], m = bm[row], v = bv[row];
            adam_catch_up1(o, lastv, o.t, w, m, v);
            bw[row] = w; bm[row] = m; bv[row] = v;
            last[row] = o.t;
        }
    }
}
