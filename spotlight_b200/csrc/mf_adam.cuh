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
// The element recurrence and the catch-up (AdamDev, adam_elem, adam_catch_up) are in common.cuh.
#pragma once

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

// Users-only mode (opt_users_only: the item table is a row cache whose owners keep the item rows'
// Adam state).  The prepass catches up the user rows the minibatch references only.
template <int LPR>
__global__ void __launch_bounds__(MF_THREADS)
mf_adam_users_prepass_kernel(MfDev a, AdamDev o, float* vWu, float* vbu, int32_t* last_u) {
    constexpr int GROUPS = MF_THREADS / LPR;
    const int gl = threadIdx.x & (LPR - 1);
    const int gib = threadIdx.x / LPR;
    const unsigned gmask = group_mask(LPR);
    const int D = a.D;
    const int upto = o.t - 1;
    if (upto <= 0) return;
    for (int64_t r = static_cast<int64_t>(blockIdx.x) * GROUPS + gib; r < a.B; r += static_cast<int64_t>(gridDim.x) * GROUPS) {
        const int64_t row = a.users[r];
        if (row < 0 || row >= a.U) continue;                               // the forward flags bad ids
        int old = 0;
        if (gl == 0) old = atomicMax(last_u + row, upto);
        old = __shfl_sync(gmask, old, (threadIdx.x & 31) & ~(LPR - 1));
        if (old >= upto) continue;
        float* W = a.Wu + row * D;
        float* M = a.sWu + row * D;
        float* V = vWu + row * D;
        for (int c = gl * 4; c < D; c += LPR * 4) {
            float4 w = ld4(W + c), m = ld4(M + c), v = ld4(V + c);
            adam_catch_up(o, old, upto, w, m, v);
            st4(W + c, w); st4(M + c, m); st4(V + c, v);
        }
        if (gl == 0) {
            float w = a.bu[row], m = a.sbu[row], v = vbu[row];
            adam_catch_up1(o, old, upto, w, m, v);
            a.bu[row] = w; a.sbu[row] = m; vbu[row] = v;
        }
    }
}

// Users-only mode: step t on the user rows with a gradient term, in place, after the item kernels
// (mf_bwd_*_kernel<.., 1>) have read the rows at t - 1.  One lane group per user segment sums the
// row's gradient from the step's terms in ascending term order, as mf_bwd_tile_kernel does, and
// applies Adam to it straight away: O(batch), no gradient row materialised, no sweep of the shard.
template <int LPR>
__global__ void __launch_bounds__(MF_THREADS)
mf_adam_users_kernel(MfDev a, AdamDev o, float* vWu, float* vbu, int32_t* last_u) {
    constexpr int GROUPS = MF_THREADS / LPR;
    constexpr int CAP = seg_sort_cap(LPR);
    __shared__ int32_t sh_all[GROUPS * 2 * CAP];
    const int gl = threadIdx.x & (LPR - 1);
    const int gib = threadIdx.x / LPR;
    const unsigned gmask = group_mask(LPR);
    int32_t* sh = sh_all + gib * 2 * CAP;
    const int D = a.D;
    const int nsegA = a.seg.totals[2];
    const float ss = o.sched[2 * o.t], bc = o.sched[2 * o.t + 1];
    for (int s = blockIdx.x * GROUPS + gib; s < nsegA; s += gridDim.x * GROUPS) {
        const int start = a.seg.seg_start[s];
        const int len = a.seg.seg_start[s + 1] - start;
        const int64_t row = a.seg.seg_row[s];
        float* W = a.Wu + row * D;
        float* M = a.sWu + row * D;
        float* V = vWu + row * D;
        const int last = last_u[row];
        float bacc = 0.f;
        for (int c0 = 0; c0 < D; c0 += LPR * 4) {
            const int c = c0 + gl * 4;
            float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
            float b2 = 0.f;
            // hot rows (len > CAP) were sorted in place by seg_sort_long_kernel
            seg_visit_sorted<LPR>(a.seg.members, start, len, gl, gmask, sh, [&](int32_t t) {
                const float g = a.t_g[t];
                if (c < D) fma4(acc, g, ldg4(a.Wi + static_cast<int64_t>(a.t_b[t]) * D + c));
                b2 += g;
            }, true);
            if (c0 == 0) bacc = b2;
            if (c < D) {
                float4 w = ld4(W + c), m = ld4(M + c), v = ld4(V + c);
                adam_catch_up(o, last, o.t - 1, w, m, v);
                adam_elem(o, ss, bc, acc.x, w.x, m.x, v.x);
                adam_elem(o, ss, bc, acc.y, w.y, m.y, v.y);
                adam_elem(o, ss, bc, acc.z, w.z, m.z, v.z);
                adam_elem(o, ss, bc, acc.w, w.w, m.w, v.w);
                st4(W + c, w); st4(M + c, m); st4(V + c, v);
            }
        }
        __syncwarp(gmask);                    // every lane has read `last` before it moves
        if (gl == 0) {
            float w = a.bu[row], m = a.sbu[row], v = vbu[row];
            adam_catch_up1(o, last, o.t - 1, w, m, v);
            adam_elem(o, ss, bc, bacc, w, m, v);
            a.bu[row] = w; a.sbu[row] = m; vbu[row] = v;
            last_u[row] = o.t;
        }
    }
}

// Dense Adam step o.t on a table pair (W [rows, D], bias [rows]) sharing `last`: every row first
// replays its pending steps through o.t - 1 (nothing when it is current), then takes step o.t with
// its gradient row G [rows, D] / gb [rows].  A zero gradient row is a real step, as in dense
// torch.optim.Adam.  Any D >= 1: one lane group of LPR lanes per row, one element per lane at a time.
template <int LPR>
__global__ void __launch_bounds__(MF_THREADS)
adam_dense_kernel(float* W, float* M, float* V, float* bw, float* bm, float* bv, int32_t* last, const float* G,
                  const float* gb, int64_t rows, int D, AdamDev o) {
    constexpr int GROUPS = MF_THREADS / LPR;
    const int gl = threadIdx.x & (LPR - 1);
    const int gib = threadIdx.x / LPR;
    const float ss = o.sched[2 * o.t], bc = o.sched[2 * o.t + 1];
    for (int64_t row = static_cast<int64_t>(blockIdx.x) * GROUPS + gib; row < rows; row += static_cast<int64_t>(gridDim.x) * GROUPS) {
        const int lastv = last[row];
        for (int c = gl; c < D; c += LPR) {
            const int64_t e = row * D + c;
            float w = W[e], m = M[e], v = V[e];
            adam_catch_up1(o, lastv, o.t - 1, w, m, v);
            adam_elem(o, ss, bc, G[e], w, m, v);
            W[e] = w; M[e] = m; V[e] = v;
        }
        __syncwarp(group_mask(LPR));          // every lane has read `last` before it moves
        if (gl == 0) {
            float w = bw[row], m = bm[row], v = bv[row];
            adam_catch_up1(o, lastv, o.t - 1, w, m, v);
            adam_elem(o, ss, bc, gb[row], w, m, v);
            bw[row] = w; bm[row] = m; bv[row] = v;
            last[row] = o.t;
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

// The same for one table with its own `last` and any width D >= 1 (a hashed table, an id-indexed
// (rows, 1) bias): one lane group of LPR lanes per row, one element per lane at a time.
template <int LPR>
__global__ void __launch_bounds__(MF_THREADS)
adam_flush_table_kernel(float* W, float* M, float* V, int32_t* last, int64_t rows, int D, AdamDev o) {
    constexpr int GROUPS = MF_THREADS / LPR;
    const int gl = threadIdx.x & (LPR - 1);
    const int gib = threadIdx.x / LPR;
    for (int64_t row = static_cast<int64_t>(blockIdx.x) * GROUPS + gib; row < rows; row += static_cast<int64_t>(gridDim.x) * GROUPS) {
        const int lastv = last[row];
        if (lastv >= o.t) continue;
        for (int c = gl; c < D; c += LPR) {
            const int64_t e = row * D + c;
            float w = W[e], m = M[e], v = V[e];
            adam_catch_up1(o, lastv, o.t, w, m, v);
            W[e] = w; M[e] = m; V[e] = v;
        }
        __syncwarp(group_mask(LPR));          // every lane has read `last` before it moves
        if (gl == 0) last[row] = o.t;
    }
}
