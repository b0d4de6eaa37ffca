// Planned two-kernel training step (pointwise / bpr / hinge with a fused row-wise optimizer).
//
// The gradient of a minibatch depends on its ids only through *which* interactions share a
// row.  That grouping is integer work on ids that are known before the step runs (the epoch's
// shuffle and negative draw are done), so it is split off as a PLAN that can run ahead of the
// floating-point kernels, on a second stream, double-buffered:
//
//   plan (ids only)   count rows -> scan -> fill member records -> sort each member list
//                     user segment s : rows of {b, i_b, j_b}  (interactions of one user)
//                     item segment s : rows of {t, useg}      (terms 2b / 2b+1 on one item row,
//                                                              with the user segment of b)
//   mf_user_kernel    ONE pass over the touched user rows: load U[u] once, score every
//                     interaction of that user against its two item rows (item table is L2
//                     resident), loss, d loss / d score, accumulate dU, stash the old row for
//                     the item side, apply the optimizer in place.  Forward and the user half
//                     of the backward are the same kernel: the user row is read once per step
//                     instead of once per interaction and again in the backward.
//   mf_item_kernel    one pass over the touched item rows: sum g * U_old[u] over the row's
//                     terms in ascending term order (from the stash, mostly L2 hits), apply
//                     the optimizer in place.
//
// Replaces, for this route, mf_fwd_tile + seg scan + fill + bwd<items> + bwd<users> + apply
// (10 launches, user rows gathered twice) of the first-generation step; semantics identical:
// spotlight/factorization/implicit.py:229-243 with a row-wise SGD / Adagrad optimizer.
// Deterministic: no float atomics, every row has one writer that sums in ascending
// interaction order.
//
// Rating losses (regression / poisson / logistic, spotlight/factorization/explicit.py:223-234) run
// the same step in ONE-TERM mode: no negative, one item member per interaction with term id b
// (instead of 2b / 2b+1), and the user record's j slot carries the rating's bits, so the user
// kernel scores one item row per interaction with no extra dependent load.
#pragma once

struct __align__(16) URec { int32_t b, i, j, pad; };     // one-term mode: j = the rating's bits
struct __align__(8) IRec { int32_t t, useg; };

struct PlanDev {
    SegIndex seg;          // cnt / off / sid / status / totals / seg_row / seg_start / long_list
    URec* mu;              // [B]   user-side member records (segment order)
    IRec* mi;              // [2B]  item-side member records
    URec* mu_tmp;          // [B]   scratch of the hot-row sort
    IRec* mi_tmp;          // [2B]
    uint32_t* bits;        // [SEG_LONG_CTAS][2 * words] bitmap + prefix of the hot-row sort
    int64_t words;
    int32_t* err;
    int64_t B, U, I;
    const int64_t* users; const int64_t* items; const int64_t* negs;
    const float* ratings;  // one-term mode (rating losses): [B], negs == nullptr
};

struct StepV2 {
    float* t_g;            // [2B] d loss / d score of term t (already / B); [B] in one-term mode
    float* stash;          // [B][D] old user rows, by user segment
    float* partial;        // [MF_MAX_GRID] loss partials of mf_user_kernel
    float* partial_long;   // [SEG_LONG_CTAS * 4] loss partials of the hot-row kernel
    int32_t* done;
};

// ------------------------------------------------------------------ plan kernels

__global__ void __launch_bounds__(256) plan_count_kernel(PlanDev p) {
    const int64_t nth = static_cast<int64_t>(gridDim.x) * blockDim.x;
    if (blockIdx.x == 0 && threadIdx.x == 0) p.seg.totals[3] = 0;
    for (int64_t b = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; b < p.B; b += nth) {
        const int64_t u = p.users[b], i = p.items[b], j = p.negs ? p.negs[b] : 0;
        if (u < 0 || u >= p.U || i < 0 || i >= p.I || j < 0 || j >= p.I) { atomicExch(p.err, 1); continue; }
        atomicAdd(p.seg.cnt + u, 1);
        atomicAdd(p.seg.cnt + p.U + i, 1);
        if (p.negs) atomicAdd(p.seg.cnt + p.U + j, 1);
    }
}

__global__ void __launch_bounds__(256) plan_fill_kernel(PlanDev p) {
    const int64_t nth = static_cast<int64_t>(gridDim.x) * blockDim.x;
    const int ubase = p.seg.seg_start[p.seg.totals[2]];     // user-side members come first
    for (int64_t b = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; b < p.B; b += nth) {
        const int64_t u = p.users[b], i = p.items[b], j = p.negs ? p.negs[b] : 0;
        if (u < 0 || u >= p.U || i < 0 || i >= p.I || j < 0 || j >= p.I) continue;
        const int su = p.seg.off[u] + atomicSub(p.seg.cnt + u, 1) - 1;
        URec r;
        r.b = static_cast<int32_t>(b); r.i = static_cast<int32_t>(i); r.pad = 0;
        r.j = p.negs ? static_cast<int32_t>(j) : __float_as_int(p.ratings[b]);
        p.mu[su] = r;
        const int useg = p.seg.sid[u];
        const int si = p.seg.off[p.U + i] + atomicSub(p.seg.cnt + p.U + i, 1) - 1 - ubase;
        if (!p.negs) {                                      // one-term mode: term b
            IRec a; a.t = static_cast<int32_t>(b); a.useg = useg;
            p.mi[si] = a;
            continue;
        }
        const int sj = p.seg.off[p.U + j] + atomicSub(p.seg.cnt + p.U + j, 1) - 1 - ubase;
        IRec a; a.t = static_cast<int32_t>(2 * b); a.useg = useg;
        IRec c; c.t = static_cast<int32_t>(2 * b + 1); c.useg = useg;
        p.mi[si] = a;
        p.mi[sj] = c;
    }
}

__device__ __forceinline__ int rec_key(const URec& r) { return r.b; }
__device__ __forceinline__ int rec_key(const IRec& r) { return r.t; }

constexpr int PLAN_SORT_SMALL = 16;

__device__ __forceinline__ URec rec_shfl_xor(const URec& r, int j) {
    URec o;
    o.b = __shfl_xor_sync(0xffffffffu, r.b, j); o.i = __shfl_xor_sync(0xffffffffu, r.i, j);
    o.j = __shfl_xor_sync(0xffffffffu, r.j, j); o.pad = 0;
    return o;
}
__device__ __forceinline__ IRec rec_shfl_xor(const IRec& r, int j) {
    IRec o;
    o.t = __shfl_xor_sync(0xffffffffu, r.t, j); o.useg = __shfl_xor_sync(0xffffffffu, r.useg, j);
    return o;
}
__device__ __forceinline__ void rec_set_key(URec& r, int k) { r.b = k; r.i = 0; r.j = 0; r.pad = 0; }
__device__ __forceinline__ void rec_set_key(IRec& r, int k) { r.t = k; r.useg = 0; }

// Sorts each member list of a 32-segment tile ascending by key (the fill placed members in
// atomic order).  Lists of two: one compare-exchange by the owning lane.  Lists of 3..16: a
// 16-wide bitonic network over half a warp, one record per lane, two lists per pass.  Lists
// up to `cap`: ranked by counting by the whole warp.  Hot rows (> cap): plan_sort_long_kernel.
// `len` is 0 for the lanes whose segment belongs to the other table.
template <typename Rec>
__device__ __forceinline__ void plan_sort_tile(Rec* base, int start, int len, int cap, Rec* tmp_base) {
    const int lane = threadIdx.x & 31;
    if (len == 2) {
        const Rec x = base[start], y = base[start + 1];
        if (rec_key(x) > rec_key(y)) { base[start] = y; base[start + 1] = x; }
    }
    unsigned net = __ballot_sync(0xffffffffu, len > 2 && len <= PLAN_SORT_SMALL);
    const int half = lane >> 4, lid = lane & 15;
    while (net) {
        const int s0 = __ffs(net) - 1;
        net &= net - 1;
        int s1 = -1;
        if (net) { s1 = __ffs(net) - 1; net &= net - 1; }
        const int mine = half == 0 ? s0 : s1;
        const int m_start = __shfl_sync(0xffffffffu, start, mine < 0 ? 0 : mine);
        const int t_len = __shfl_sync(0xffffffffu, len, mine < 0 ? 0 : mine);     // every lane takes part
        const int m_len = mine < 0 ? 0 : t_len;
        Rec v;
        if (lid < m_len) v = base[m_start + lid];
        else rec_set_key(v, 0x7fffffff);
#pragma unroll
        for (int k = 2; k <= 16; k <<= 1) {
#pragma unroll
            for (int j = k >> 1; j > 0; j >>= 1) {
                const Rec o = rec_shfl_xor(v, j);
                const bool keep_min = ((lid & j) == 0) == ((lid & k) == 0);
                const bool other_smaller = rec_key(o) < rec_key(v);
                if (keep_min == other_smaller) v = o;
            }
        }
        if (lid < m_len) base[m_start + lid] = v;
    }
    // medium lists: the warp ranks one list at a time
    unsigned med = __ballot_sync(0xffffffffu, len > PLAN_SORT_SMALL && len <= cap);
    while (med) {
        const int src = __ffs(med) - 1;
        med &= med - 1;
        const int s_start = __shfl_sync(0xffffffffu, start, src);
        const int s_len = __shfl_sync(0xffffffffu, len, src);
        for (int i = lane; i < s_len; i += 32) {
            const Rec x = base[s_start + i];
            int r = 0;
            for (int m = 0; m < s_len; ++m) r += rec_key(base[s_start + m]) < rec_key(x);
            tmp_base[s_start + r] = x;
        }
        __syncwarp();
        for (int i = lane; i < s_len; i += 32) base[s_start + i] = tmp_base[s_start + i];
        __syncwarp();
    }
}

__global__ void __launch_bounds__(128) plan_sort_kernel(PlanDev p, int cap) {
    const int nseg = p.seg.totals[0], nsegA = p.seg.totals[2];
    const int ubase = p.seg.seg_start[nsegA];
    const int lane = threadIdx.x & 31;
    const int ntiles = (nseg + 31) / 32;
    for (int tile = blockIdx.x * 4 + (threadIdx.x >> 5); tile < ntiles; tile += gridDim.x * 4) {
        const int s = tile * 32 + lane;
        int start = 0, len = 0;
        if (s < nseg) { start = p.seg.seg_start[s]; len = p.seg.seg_start[s + 1] - start; }
        // a tile may straddle the user / item boundary: two passes with the other half masked
        plan_sort_tile<URec>(p.mu, start, (s < nsegA) ? len : 0, cap, p.mu_tmp);
        plan_sort_tile<IRec>(p.mi, start - ubase, (s >= nsegA && s < nseg) ? len : 0, cap, p.mi_tmp);
    }
}

// Hot rows: keys are distinct and < nbits, so the rank of a record is the number of set bits
// below its key in a bitmap of the list (bitmap -> per-word prefix popcount -> rank).
template <typename Rec>
__device__ void plan_sort_long_one(Rec* base, Rec* tmp, int start, int len, uint32_t* bits, uint32_t* pre,
                                   int W, uint32_t* sh_scan) {
    const int per = (W + 255) / 256;
    for (int w = threadIdx.x; w < W; w += 256) bits[w] = 0u;
    __syncthreads();
    for (int i = threadIdx.x; i < len; i += 256) {
        const int t = rec_key(base[start + i]);
        atomicOr(bits + (t >> 5), 1u << (t & 31));
    }
    __syncthreads();
    const int lo = threadIdx.x * per, hi = lo + per < W ? lo + per : W;
    uint32_t sum = 0;
    for (int w = lo; w < hi; ++w) sum += __popc(bits[w]);
    sh_scan[threadIdx.x] = sum;
    __syncthreads();
    for (int o = 1; o < 256; o <<= 1) {
        const uint32_t v = threadIdx.x >= o ? sh_scan[threadIdx.x - o] : 0u;
        __syncthreads();
        sh_scan[threadIdx.x] += v;
        __syncthreads();
    }
    uint32_t run = sh_scan[threadIdx.x] - sum;
    for (int w = lo; w < hi; ++w) { pre[w] = run; run += __popc(bits[w]); }
    __syncthreads();
    for (int i = threadIdx.x; i < len; i += 256) {
        const Rec x = base[start + i];
        const int t = rec_key(x);
        const uint32_t r = pre[t >> 5] + __popc(bits[t >> 5] & ((1u << (t & 31)) - 1u));
        tmp[start + r] = x;
    }
    __syncthreads();
    for (int i = threadIdx.x; i < len; i += 256) base[start + i] = tmp[start + i];
    __syncthreads();
}

// The scan appends hot segments to long_list in atomic order, which varies from run to run.
// One CTA puts the list in ascending segment order (segment ids are distinct and < nseg: set
// their bits, then each thread enumerates its own run of words after an exclusive prefix of
// the popcounts), so every hot row lands on the same CTA of the long kernels in every run and
// mf_user_kernel folds the hot-row loss partials in a fixed order.  Uses the first bitmap of
// p.bits (2 * words >= ceil(3B / 32) words), which plan_sort_long_kernel only touches later.
__global__ void __launch_bounds__(256) plan_order_long_kernel(PlanDev p) {
    __shared__ uint32_t sh_scan[256];
    const int nlong = p.seg.totals[3];
    if (nlong < 2) return;                        // block-uniform
    uint32_t* bits = p.bits;
    const int W = (p.seg.totals[0] + 31) / 32;
    const int per = (W + 255) / 256;
    for (int w = threadIdx.x; w < W; w += 256) bits[w] = 0u;
    __syncthreads();
    for (int i = threadIdx.x; i < nlong; i += 256) {
        const int s = p.seg.long_list[i];
        atomicOr(bits + (s >> 5), 1u << (s & 31));
    }
    __syncthreads();
    const int lo = threadIdx.x * per, hi = lo + per < W ? lo + per : W;
    uint32_t sum = 0;
    for (int w = lo; w < hi; ++w) sum += __popc(bits[w]);
    sh_scan[threadIdx.x] = sum;
    __syncthreads();
    for (int o = 1; o < 256; o <<= 1) {
        const uint32_t v = threadIdx.x >= o ? sh_scan[threadIdx.x - o] : 0u;
        __syncthreads();
        sh_scan[threadIdx.x] += v;
        __syncthreads();
    }
    uint32_t run = sh_scan[threadIdx.x] - sum;
    for (int w = lo; w < hi; ++w) {
        for (uint32_t m = bits[w]; m; m &= m - 1u) p.seg.long_list[run++] = w * 32 + __ffs(m) - 1;
    }
}

__global__ void __launch_bounds__(256) plan_sort_long_kernel(PlanDev p) {
    __shared__ uint32_t sh_scan[256];
    const int nlong = p.seg.totals[3];
    const int nsegA = p.seg.totals[2];
    const int ubase = p.seg.seg_start[nsegA];
    uint32_t* bits = p.bits + static_cast<size_t>(blockIdx.x) * 2 * p.words;
    uint32_t* pre = bits + p.words;
    for (int li = blockIdx.x; li < nlong; li += gridDim.x) {
        const int s = p.seg.long_list[li];
        const int start = p.seg.seg_start[s];
        const int len = p.seg.seg_start[s + 1] - start;
        if (s < nsegA) plan_sort_long_one<URec>(p.mu, p.mu_tmp, start, len, bits, pre, static_cast<int>((p.B + 31) / 32), sh_scan);
        else plan_sort_long_one<IRec>(p.mi, p.mi_tmp, start - ubase, len, bits, pre, static_cast<int>((2 * p.B + 31) / 32), sh_scan);
    }
}

// ------------------------------------------------------------------ optimizer

// ------------------------------------------------------------------ user side (forward + dU + update)

#ifndef V2_UMINB
#define V2_UMINB 8
#endif
#ifndef V2_UMINB2
#define V2_UMINB2 6
#endif
#ifndef V2_UVPL
#define V2_UVPL 2
#endif
#ifndef V2_UPF
#define V2_UPF 0
#endif

// A lane holds VPL 128-bit pieces of a row: columns gl*4 + v*LPR*4 (every load of a group covers
// whole 128-byte lines).  VPL = 2 halves the lanes per row, so a warp iteration carries twice the
// segments -- twice the bytes in flight per warp, one shuffle level less per reduction.
template <int VPL>
struct RowV { float4 v[VPL]; };

template <int LPR, int VPL>
__device__ __forceinline__ RowV<VPL> row_ldg(const float* row, int gl) {
    RowV<VPL> r;
#pragma unroll
    for (int q = 0; q < VPL; ++q) r.v[q] = ldg4(row + gl * 4 + q * LPR * 4);
    return r;
}
template <int LPR, int VPL>
__device__ __forceinline__ RowV<VPL> row_ldcs(const float* row, int gl) {
    RowV<VPL> r;
#pragma unroll
    for (int q = 0; q < VPL; ++q) r.v[q] = __ldcs(reinterpret_cast<const float4*>(row + gl * 4 + q * LPR * 4));
    return r;
}
template <int VPL>
__device__ __forceinline__ RowV<VPL> row_zero() {
    RowV<VPL> r;
#pragma unroll
    for (int q = 0; q < VPL; ++q) r.v[q] = make_float4(0.f, 0.f, 0.f, 0.f);
    return r;
}

// One interaction of a user segment: two dots, loss, d loss / d score, gradient accumulation.
// FULL: the whole warp is converged on this call (every group runs it), so the group reductions
// shuffle under the constant full mask -- plain SHFL.BFLY, no per-shuffle WARPSYNC / MATCH
// sequence that a run-time group mask compiles to.
template <int LPR, int VPL, int LOSS, bool FULL>
__device__ __forceinline__ void user_member(const RowV<VPL>& w, float ub, const RowV<VPL>& qi, const RowV<VPL>& qj,
                                            float bi_, float bj_, int b, float invB, unsigned gmask, int gl,
                                            float* t_g, RowV<VPL>& acc, float& bacc, bool& nz, float& lsum) {
    if constexpr (LOSS >= SLB_LOSS_REGRESSION) {
        // one-term mode: bj_ is the rating, qj is not used
        float dp = 0.f;
#pragma unroll
        for (int q = 0; q < VPL; ++q) dp += dot4(w.v[q], qi.v[q]);
        dp = group_sum<LPR>(dp, FULL ? 0xffffffffu : gmask);
        float per, g;
        rating_loss(LOSS, dp + ub + bi_, bj_, per, g);
        g *= invB;
        if (gl == 0) {
            lsum += per;
            t_g[b] = g;
        }
#pragma unroll
        for (int q = 0; q < VPL; ++q) fma4(acc.v[q], g, qi.v[q]);
        bacc += g;
        nz = nz || g != 0.f;
        return;
    }
    float dp = 0.f, dn = 0.f;
#pragma unroll
    for (int q = 0; q < VPL; ++q) { dp += dot4(w.v[q], qi.v[q]); dn += dot4(w.v[q], qj.v[q]); }
    dp = group_sum<LPR>(dp, FULL ? 0xffffffffu : gmask);
    dn = group_sum<LPR>(dn, FULL ? 0xffffffffu : gmask);
    float per, gp, gn;
    pair_loss(LOSS, dp + ub + bi_, dn + ub + bj_, per, gp, gn);
    gp *= invB; gn *= invB;
    if (gl == 0) {
        lsum += per;
        *reinterpret_cast<float2*>(t_g + 2 * static_cast<int64_t>(b)) = make_float2(gp, gn);
    }
#pragma unroll
    for (int q = 0; q < VPL; ++q) { fma4(acc.v[q], gp, qi.v[q]); fma4(acc.v[q], gn, qj.v[q]); }
    bacc += gp + gn;
    nz = nz || gp != 0.f || gn != 0.f;
}

// Stash the pre-update row for the item side, apply the optimizer in place.  The weight and
// state rows stream through (evict-first loads / stores): they are touched once per step,
// while the stash is re-read by mf_item_kernel and the item table by every other segment.
template <int LPR, int VPL>
__device__ __forceinline__ void user_finish(const MfDev& a, const OptV2& o, float* stash_row, float* wrow, float* srow,
                                            RowV<VPL> w, RowV<VPL> s, const RowV<VPL>& acc, float bacc, bool nz,
                                            int row, int gl) {
#pragma unroll
    for (int q = 0; q < VPL; ++q) st4(stash_row + gl * 4 + q * LPR * 4, w.v[q]);
    if (nz) {                                        // all-zero gradients leave the row untouched
#pragma unroll
        for (int q = 0; q < VPL; ++q) {
            row_update(o, w.v[q], s.v[q], acc.v[q]);
            __stcs(reinterpret_cast<float4*>(wrow + gl * 4 + q * LPR * 4), w.v[q]);
            if (srow) __stcs(reinterpret_cast<float4*>(srow + gl * 4 + q * LPR * 4), s.v[q]);
        }
        if (gl == 0) bias_update(o, a.bu + row, a.sbu ? a.sbu + row : nullptr, bacc);
    }
}

template <int LPR, int VPL, int LOSS, int TI>
__global__ void __launch_bounds__(MF_TILE_THREADS, (VPL == 1 ? V2_UMINB : V2_UMINB2)) mf_user_kernel(MfDev a, PlanDev p, StepV2 v, int n_long_partials) {
    constexpr int D = LPR * 4 * VPL;
    constexpr int GPW = 32 / LPR;
    constexpr int WARPS = MF_TILE_THREADS / 32;
    constexpr bool RATING = LOSS >= SLB_LOSS_REGRESSION;    // one-term mode: j carries the rating
    __shared__ float sh_red[WARPS];
    __shared__ int sh_inv[WARPS][32];
    __shared__ bool is_last;
    const int lane = threadIdx.x & 31;
    const int warp = threadIdx.x >> 5;
    const int gl = lane & (LPR - 1);
    const int grp = lane / LPR;
    const unsigned gmask = group_mask(LPR);
    const unsigned below = (1u << lane) - 1u;
    const float invB = 1.0f / static_cast<float>(a.NB);
    const OptV2 o = {a.opt, a.lr, a.wd, a.eps};
    const int nsegA = p.seg.totals[2];
    const int ntiles = (nsegA + TI - 1) / TI;
    const int wstride = gridDim.x * WARPS;
    const int cap = p.seg.long_cap;
    const bool adagrad = a.opt == SLB_OPT_ADAGRAD;
    float lsum = 0.f;

    for (int tile = blockIdx.x * WARPS + warp; tile < ntiles; tile += wstride) {
        const int sidx = tile * TI + lane;
        const bool valid = lane < TI && sidx < nsegA;
        int start = 0, len = 0, row = 0;
        int4 r0 = make_int4(0, 0, 0, 0), r1 = r0;
        if (valid) {
            start = p.seg.seg_start[sidx];
            len = p.seg.seg_start[sidx + 1] - start;
            row = p.seg.seg_row[sidx];
            r0 = __ldg(reinterpret_cast<const int4*>(p.mu + start));
            if (len == 2) r1 = __ldg(reinterpret_cast<const int4*>(p.mu + start + 1));
#if V2_UPF
            // experiment: ask L2 for this segment's weight / state rows a whole tile ahead
            pf_row_l2(a.Wu + static_cast<int64_t>(row) * D, D);
            if (adagrad) pf_row_l2(a.sWu + static_cast<int64_t>(row) * D, D);
#endif
        }
        // Order the tile's segments by length class (1, 2, longer, none) so that a whole warp
        // iteration runs one specialised, unpredicated code path: three quarters of the user
        // rows of a uniform batch have one interaction, a fifth have two.
        const unsigned m1 = __ballot_sync(0xffffffffu, len == 1);
        const unsigned m2 = __ballot_sync(0xffffffffu, len == 2);
        const unsigned m3 = __ballot_sync(0xffffffffu, len > 2);
        const int n1 = __popc(m1), n2 = __popc(m2), n3 = __popc(m3);
        int pos;
        if (len == 1) pos = __popc(m1 & below);
        else if (len == 2) pos = n1 + __popc(m2 & below);
        else if (len > 2) pos = n1 + n2 + __popc(m3 & below);
        else pos = n1 + n2 + n3 + __popc(~(m1 | m2 | m3) & below);
        __syncwarp();
        sh_inv[warp][pos] = lane;
        __syncwarp();
        const int nvalid = n1 + n2 + n3;

        for (int q0 = 0; q0 < nvalid; q0 += GPW) {
            const int q = q0 + grp;
            const int src = sh_inv[warp][q & 31];
            const int s_len = __shfl_sync(0xffffffffu, len, src);
            const int s_row = __shfl_sync(0xffffffffu, row, src);
            const int b0 = __shfl_sync(0xffffffffu, r0.x, src);
            const int i0 = __shfl_sync(0xffffffffu, r0.y, src);
            const int j0 = __shfl_sync(0xffffffffu, r0.z, src);
            const int s = tile * TI + src;
            float* wrow = a.Wu + static_cast<int64_t>(s_row) * D;
            float* srow = adagrad ? a.sWu + static_cast<int64_t>(s_row) * D : nullptr;
            float* stash_row = v.stash + static_cast<int64_t>(s) * D;
            RowV<VPL> acc = row_zero<VPL>();
            float bacc = 0.f;
            bool nz = false;
            if (q0 + GPW <= n1) {
                // ---- every group of the warp: one interaction
                const RowV<VPL> w = row_ldcs<LPR, VPL>(wrow, gl);
                RowV<VPL> st_ = row_zero<VPL>();
                if (adagrad) st_ = row_ldcs<LPR, VPL>(srow, gl);
                const RowV<VPL> qi = row_ldg<LPR, VPL>(a.Wi + static_cast<int64_t>(i0) * D, gl);
                const RowV<VPL> qj = RATING ? row_zero<VPL>() : row_ldg<LPR, VPL>(a.Wi + static_cast<int64_t>(j0) * D, gl);
                const float ub = a.bu[s_row], bi_ = __ldg(a.bi + i0);
                const float bj_ = RATING ? __int_as_float(j0) : __ldg(a.bi + j0);
                user_member<LPR, VPL, LOSS, true>(w, ub, qi, qj, bi_, bj_, b0, invB, gmask, gl, v.t_g, acc, bacc, nz, lsum);
                user_finish<LPR, VPL>(a, o, stash_row, wrow, srow, w, st_, acc, bacc, nz, s_row, gl);
            } else if (q0 >= n1 && q0 + GPW <= n1 + n2) {
                // ---- every group of the warp: two interactions
                const int b1 = __shfl_sync(0xffffffffu, r1.x, src);
                const int i1 = __shfl_sync(0xffffffffu, r1.y, src);
                const int j1 = __shfl_sync(0xffffffffu, r1.z, src);
                const RowV<VPL> w = row_ldcs<LPR, VPL>(wrow, gl);
                RowV<VPL> st_ = row_zero<VPL>();
                if (adagrad) st_ = row_ldcs<LPR, VPL>(srow, gl);
                const RowV<VPL> qi0 = row_ldg<LPR, VPL>(a.Wi + static_cast<int64_t>(i0) * D, gl);
                const RowV<VPL> qj0 = RATING ? row_zero<VPL>() : row_ldg<LPR, VPL>(a.Wi + static_cast<int64_t>(j0) * D, gl);
                const float ub = a.bu[s_row];
                const float bi0 = __ldg(a.bi + i0), bi1 = __ldg(a.bi + i1);
                const float bj0 = RATING ? __int_as_float(j0) : __ldg(a.bi + j0);
                const float bj1 = RATING ? __int_as_float(j1) : __ldg(a.bi + j1);
                user_member<LPR, VPL, LOSS, true>(w, ub, qi0, qj0, bi0, bj0, b0, invB, gmask, gl, v.t_g, acc, bacc, nz, lsum);
                const RowV<VPL> qi1 = row_ldg<LPR, VPL>(a.Wi + static_cast<int64_t>(i1) * D, gl);
                const RowV<VPL> qj1 = RATING ? row_zero<VPL>() : row_ldg<LPR, VPL>(a.Wi + static_cast<int64_t>(j1) * D, gl);
                user_member<LPR, VPL, LOSS, true>(w, ub, qi1, qj1, bi1, bj1, b1, invB, gmask, gl, v.t_g, acc, bacc, nz, lsum);
                user_finish<LPR, VPL>(a, o, stash_row, wrow, srow, w, st_, acc, bacc, nz, s_row, gl);
            } else {
                // ---- mixed iteration (class boundaries, lists of 3+): group-divergent generic path
                const int s_start = __shfl_sync(0xffffffffu, start, src);
                if (q >= nvalid || s_len > cap) continue;         // idle group / hot row (mf_user_long_kernel)
                const RowV<VPL> w = row_ldcs<LPR, VPL>(wrow, gl);
                RowV<VPL> st_ = row_zero<VPL>();
                if (adagrad) st_ = row_ldcs<LPR, VPL>(srow, gl);
                const float ub = a.bu[s_row];
                for (int k = 0; k < s_len; ++k) {
                    // every lane of the group reads the same (sorted) record: one broadcast transaction
                    const int4 r = __ldg(reinterpret_cast<const int4*>(p.mu + s_start + k));
                    const RowV<VPL> qi = row_ldg<LPR, VPL>(a.Wi + static_cast<int64_t>(r.y) * D, gl);
                    const RowV<VPL> qj = RATING ? row_zero<VPL>() : row_ldg<LPR, VPL>(a.Wi + static_cast<int64_t>(r.z) * D, gl);
                    const float bj_ = RATING ? __int_as_float(r.z) : __ldg(a.bi + r.z);
                    user_member<LPR, VPL, LOSS, false>(w, ub, qi, qj, __ldg(a.bi + r.y), bj_, r.x, invB, gmask,
                                                       gl, v.t_g, acc, bacc, nz, lsum);
                }
                user_finish<LPR, VPL>(a, o, stash_row, wrow, srow, w, st_, acc, bacc, nz, s_row, gl);
            }
        }
    }

    // deterministic loss reduction: fixed tree per block, fixed order over blocks (+ hot-row partials)
    const float bsum = block_sum<MF_TILE_THREADS>(lsum, sh_red);
    if (threadIdx.x == 0) {
        v.partial[blockIdx.x] = bsum;
        __threadfence();
        is_last = atomicAdd(v.done, 1) == static_cast<int>(gridDim.x) - 1;
    }
    __syncthreads();
    if (is_last && threadIdx.x < 32) {
        __threadfence();
        float t = 0.f;
        for (int k = threadIdx.x; k < static_cast<int>(gridDim.x); k += 32)
            t += *reinterpret_cast<volatile float*>(v.partial + k);
        for (int k = threadIdx.x; k < n_long_partials; k += 32)
            t += *reinterpret_cast<volatile float*>(v.partial_long + k);
#pragma unroll
        for (int off = 16; off > 0; off >>= 1) t += __shfl_down_sync(0xffffffffu, t, off);
        if (threadIdx.x == 0) { *a.loss_out = t * invB; *v.done = 0; }
    }
}

// Hot user rows (more interactions in this batch than the tile kernel's cap): one CTA per row,
// each lane group scores a contiguous chunk of the sorted member list, chunk partials are
// combined in chunk order.  Runs before mf_user_kernel (its loss partials are folded there).
template <int LPR, int LOSS>
__global__ void __launch_bounds__(256) mf_user_long_kernel(MfDev a, PlanDev p, StepV2 v) {
    constexpr int D = LPR * 4;
    constexpr int GROUPS = 256 / LPR;
    constexpr int PS = D + 4;
    extern __shared__ float sh_part[];            // [GROUPS][D + 4]
    __shared__ float sh_red[8];
    const int gl = threadIdx.x & (LPR - 1);
    const int gq = threadIdx.x / LPR;
    const int c = gl * 4;
    const unsigned gmask = group_mask(LPR);
    const float invB = 1.0f / static_cast<float>(a.NB);
    const OptV2 o = {a.opt, a.lr, a.wd, a.eps};
    const int nlong = p.seg.totals[3];
    const int nsegA = p.seg.totals[2];
    float lsum = 0.f;
    for (int li = blockIdx.x; li < nlong; li += gridDim.x) {
        const int s = p.seg.long_list[li];
        if (s >= nsegA) continue;                 // block-uniform
        const int start = p.seg.seg_start[s];
        const int len = p.seg.seg_start[s + 1] - start;
        const int row = p.seg.seg_row[s];
        float* wrow = a.Wu + static_cast<int64_t>(row) * D + c;
        const float4 w4 = ld4(wrow);
        const float ub = a.bu[row];
        const int chunk = (len + GROUPS - 1) / GROUPS;
        const int lo = min(gq * chunk, len), hi = min(lo + chunk, len);
        float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
        float bacc = 0.f, nzf = 0.f;
        for (int k = lo; k < hi; ++k) {
            const int4 r0 = __ldg(reinterpret_cast<const int4*>(p.mu + start + k));
            const float4 a0 = ldg4(a.Wi + static_cast<int64_t>(r0.y) * D + c);
            if constexpr (LOSS >= SLB_LOSS_REGRESSION) {              // one-term mode: r0.z = rating bits
                const float dp = group_sum<LPR>(dot4(w4, a0), gmask);
                float per, g;
                rating_loss(LOSS, dp + ub + __ldg(a.bi + r0.y), __int_as_float(r0.z), per, g);
                g *= invB;
                if (gl == 0) {
                    lsum += per;
                    v.t_g[r0.x] = g;
                }
                fma4(acc, g, a0);
                bacc += g;
                if (g != 0.f) nzf = 1.f;
                continue;
            }
            const float4 b0 = ldg4(a.Wi + static_cast<int64_t>(r0.z) * D + c);
            const float dp = group_sum<LPR>(dot4(w4, a0), gmask);
            const float dn = group_sum<LPR>(dot4(w4, b0), gmask);
            float per, gp, gn;
            pair_loss(LOSS, dp + ub + __ldg(a.bi + r0.y), dn + ub + __ldg(a.bi + r0.z), per, gp, gn);
            gp *= invB; gn *= invB;
            if (gl == 0) {
                lsum += per;
                *reinterpret_cast<float2*>(v.t_g + 2 * static_cast<int64_t>(r0.x)) = make_float2(gp, gn);
            }
            fma4(acc, gp, a0);
            fma4(acc, gn, b0);
            bacc += gp + gn;
            if (gp != 0.f || gn != 0.f) nzf = 1.f;
        }
        st4(sh_part + gq * PS + c, acc);
        if (gl == 0) { sh_part[gq * PS + D] = bacc; sh_part[gq * PS + D + 1] = nzf; }
        __syncthreads();
        if (gq == 0) {
            float4 tot = make_float4(0.f, 0.f, 0.f, 0.f);
            float bt = 0.f, nzt = 0.f;
            for (int q = 0; q < GROUPS; ++q) {
                const float4 x = ld4(sh_part + q * PS + c);
                tot.x += x.x; tot.y += x.y; tot.z += x.z; tot.w += x.w;
                bt += sh_part[q * PS + D];
                nzt += sh_part[q * PS + D + 1];
            }
            st4(v.stash + static_cast<int64_t>(s) * D + c, w4);
            if (nzt != 0.f) {
                float4 wn = w4, s4 = make_float4(0.f, 0.f, 0.f, 0.f);
                float* srow = a.opt == SLB_OPT_ADAGRAD ? a.sWu + static_cast<int64_t>(row) * D + c : nullptr;
                if (srow) s4 = ld4(srow);
                row_update(o, wn, s4, tot);
                st4(wrow, wn);
                if (srow) st4(srow, s4);
                if (gl == 0) bias_update(o, a.bu + row, a.sbu ? a.sbu + row : nullptr, bt);
            }
        }
        __syncthreads();
    }
    const float bsum = block_sum<256>(lsum, sh_red);
    if (threadIdx.x == 0) v.partial_long[blockIdx.x] = bsum;
}

// ------------------------------------------------------------------ item side (dQ + update)

#ifndef V2_IFAST
#define V2_IFAST 4
#endif
#ifndef V2_IMINB
#define V2_IMINB 6
#endif
#ifndef V2_ICHUNK
#define V2_ICHUNK 8
#endif

template <int LPR, int TI>
__global__ void __launch_bounds__(MF_TILE_THREADS, V2_IMINB) mf_item_kernel(MfDev a, PlanDev p, StepV2 v) {
    constexpr int D = LPR * 4;
    constexpr int GPW = 32 / LPR;
    constexpr int ITERS = TI / GPW > 0 ? TI / GPW : 1;
    constexpr int WARPS = MF_TILE_THREADS / 32;
    constexpr int CAP = seg_sort_cap(LPR);
    __shared__ int32_t sh_all[WARPS * GPW * 2 * CAP];
    const int lane = threadIdx.x & 31;
    const int gl = lane & (LPR - 1);
    const int grp = lane / LPR;
    const int c = gl * 4;
    const unsigned gmask = group_mask(LPR);
    int32_t* sh = sh_all + ((threadIdx.x >> 5) * GPW + grp) * 2 * CAP;
    const OptV2 o = {a.opt, a.lr, a.wd, a.eps};
    const int nseg = p.seg.totals[0];
    const int nsegA = p.seg.totals[2];
    const int ubase = p.seg.seg_start[nsegA];
    const int ntiles = (nseg - nsegA + TI - 1) / TI;
    const int wstride = gridDim.x * WARPS;
    const float* __restrict__ t_g = v.t_g;

    for (int tile = blockIdx.x * WARPS + (threadIdx.x >> 5); tile < ntiles; tile += wstride) {
        const int sidx = nsegA + tile * TI + lane;
        const bool valid = lane < TI && sidx < nseg;
        int start = 0, len = 0, row = 0;
        int pu[V2_IFAST] = {};
        float pg[V2_IFAST] = {};
        if (valid) {
            start = p.seg.seg_start[sidx] - ubase;
            len = p.seg.seg_start[sidx + 1] - ubase - start;
            row = p.seg.seg_row[sidx] - static_cast<int>(a.U);
            if (len <= V2_IFAST) {
#pragma unroll
                for (int k = 0; k < V2_IFAST; ++k)
                    if (k < len) {
                        const int2 r = __ldg(reinterpret_cast<const int2*>(p.mi + start + k));
                        pu[k] = r.y;
                        pg[k] = t_g[r.x];
                    }
            }
        }
        for (int it = 0; it < ITERS; ++it) {
            const int src = it * GPW + grp;
            const int s_len = __shfl_sync(0xffffffffu, len, src & 31);
            const int s_row = __shfl_sync(0xffffffffu, row, src & 31);
            const int s_start = __shfl_sync(0xffffffffu, start, src & 31);
            int su[V2_IFAST];
            float sg[V2_IFAST];
#pragma unroll
            for (int k = 0; k < V2_IFAST; ++k) {
                su[k] = __shfl_sync(0xffffffffu, pu[k], src & 31);
                sg[k] = __shfl_sync(0xffffffffu, pg[k], src & 31);
            }
            const int s = nsegA + tile * TI + src;
            if (src >= TI || s >= nseg) continue;             // group-uniform
            if (s_len > CAP) continue;                        // hot row: mf_item_long_kernel
            float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
            float bacc = 0.f;
            bool nz = false;
            if (s_len <= V2_IFAST) {
                float4 x[V2_IFAST];
#pragma unroll
                for (int k = 0; k < V2_IFAST; ++k)
                    if (k < s_len) x[k] = ld4(v.stash + static_cast<int64_t>(su[k]) * D + c);
#pragma unroll
                for (int k = 0; k < V2_IFAST; ++k)
                    if (k < s_len) { fma4(acc, sg[k], x[k]); bacc += sg[k]; nz = nz || sg[k] != 0.f; }
            } else {
                float* lg = reinterpret_cast<float*>(sh);
                int32_t* lu = sh + CAP;
                for (int i = gl; i < s_len; i += LPR) {
                    const int2 r = __ldg(reinterpret_cast<const int2*>(p.mi + s_start + i));
                    lg[i] = t_g[r.x];
                    lu[i] = r.y;
                    pf_row_l2(v.stash + static_cast<int64_t>(r.y) * D, D);      // the walk below then runs at L2 latency
                }
                __syncwarp(gmask);
                int i = 0;
                for (; i + V2_ICHUNK <= s_len; i += V2_ICHUNK) {
                    float4 x[V2_ICHUNK];
#pragma unroll
                    for (int k = 0; k < V2_ICHUNK; ++k) x[k] = ld4(v.stash + static_cast<int64_t>(lu[i + k]) * D + c);
#pragma unroll
                    for (int k = 0; k < V2_ICHUNK; ++k) { fma4(acc, lg[i + k], x[k]); bacc += lg[i + k]; nz = nz || lg[i + k] != 0.f; }
                }
                for (; i < s_len; ++i) {
                    fma4(acc, lg[i], ld4(v.stash + static_cast<int64_t>(lu[i]) * D + c));
                    bacc += lg[i];
                    nz = nz || lg[i] != 0.f;
                }
                __syncwarp(gmask);                            // scratch is reused by the next segment
            }
            if (a.dWi) {
                // item rows owned elsewhere (multi-GPU): hand the gradient out, dense, caller-zeroed
                st4(a.dWi + static_cast<int64_t>(s_row) * D + c, acc);
                if (gl == 0) a.dbi[s_row] = bacc;
            } else if (nz) {
                float* wrow = a.Wi + static_cast<int64_t>(s_row) * D + c;
                float* srow = a.opt == SLB_OPT_ADAGRAD ? a.sWi + static_cast<int64_t>(s_row) * D + c : nullptr;
                float4 w4 = ld4(wrow);
                float4 s4 = make_float4(0.f, 0.f, 0.f, 0.f);
                if (srow) s4 = ld4(srow);
                row_update(o, w4, s4, acc);
                st4(wrow, w4);
                if (srow) st4(srow, s4);
                if (gl == 0) bias_update(o, a.bi + s_row, a.sbi ? a.sbi + s_row : nullptr, bacc);
            }
        }
    }
}

template <int LPR>
__global__ void __launch_bounds__(256) mf_item_long_kernel(MfDev a, PlanDev p, StepV2 v) {
    constexpr int D = LPR * 4;
    constexpr int GROUPS = 256 / LPR;
    constexpr int PS = D + 4;
    extern __shared__ float sh_part[];            // [GROUPS][D + 4]
    const int gl = threadIdx.x & (LPR - 1);
    const int gq = threadIdx.x / LPR;
    const int c = gl * 4;
    const OptV2 o = {a.opt, a.lr, a.wd, a.eps};
    const int nlong = p.seg.totals[3];
    const int nsegA = p.seg.totals[2];
    const int ubase = p.seg.seg_start[nsegA];
    for (int li = blockIdx.x; li < nlong; li += gridDim.x) {
        const int s = p.seg.long_list[li];
        if (s < nsegA) continue;                  // block-uniform
        const int start = p.seg.seg_start[s] - ubase;
        const int len = p.seg.seg_start[s + 1] - ubase - start;
        const int row = p.seg.seg_row[s] - static_cast<int>(a.U);
        const int chunk = (len + GROUPS - 1) / GROUPS;
        const int lo = min(gq * chunk, len), hi = min(lo + chunk, len);
        float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
        float bacc = 0.f, nzf = 0.f;
        int i = lo;
        for (; i + 4 <= hi; i += 4) {
            int2 r[4]; float g[4]; float4 x[4];
#pragma unroll
            for (int k = 0; k < 4; ++k) r[k] = __ldg(reinterpret_cast<const int2*>(p.mi + start + i + k));
#pragma unroll
            for (int k = 0; k < 4; ++k) { g[k] = v.t_g[r[k].x]; x[k] = ld4(v.stash + static_cast<int64_t>(r[k].y) * D + c); }
#pragma unroll
            for (int k = 0; k < 4; ++k) { fma4(acc, g[k], x[k]); bacc += g[k]; if (g[k] != 0.f) nzf = 1.f; }
        }
        for (; i < hi; ++i) {
            const int2 r = __ldg(reinterpret_cast<const int2*>(p.mi + start + i));
            const float g = v.t_g[r.x];
            fma4(acc, g, ld4(v.stash + static_cast<int64_t>(r.y) * D + c));
            bacc += g;
            if (g != 0.f) nzf = 1.f;
        }
        st4(sh_part + gq * PS + c, acc);
        if (gl == 0) { sh_part[gq * PS + D] = bacc; sh_part[gq * PS + D + 1] = nzf; }
        __syncthreads();
        if (gq == 0) {
            float4 tot = make_float4(0.f, 0.f, 0.f, 0.f);
            float bt = 0.f, nzt = 0.f;
            for (int q = 0; q < GROUPS; ++q) {
                const float4 x = ld4(sh_part + q * PS + c);
                tot.x += x.x; tot.y += x.y; tot.z += x.z; tot.w += x.w;
                bt += sh_part[q * PS + D];
                nzt += sh_part[q * PS + D + 1];
            }
            if (a.dWi) {
                st4(a.dWi + static_cast<int64_t>(row) * D + c, tot);
                if (gl == 0) a.dbi[row] = bt;
            } else if (nzt != 0.f) {
                float* wrow = a.Wi + static_cast<int64_t>(row) * D + c;
                float* srow = a.opt == SLB_OPT_ADAGRAD ? a.sWi + static_cast<int64_t>(row) * D + c : nullptr;
                float4 w4 = ld4(wrow), s4 = make_float4(0.f, 0.f, 0.f, 0.f);
                if (srow) s4 = ld4(srow);
                row_update(o, w4, s4, tot);
                st4(wrow, w4);
                if (srow) st4(srow, s4);
                if (gl == 0) bias_update(o, a.bi + row, a.sbi ? a.sbi + row : nullptr, bt);
            }
        }
        __syncthreads();
    }
}
