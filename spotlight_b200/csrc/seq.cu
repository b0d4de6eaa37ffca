// Sequence-model training step for sm_90a: PoolNet and CNNNet.
//
// Replaces the loop body of ImplicitSequenceModel.fit
// (spotlight/sequence/implicit.py:230-255): user_representation
// (PoolNet spotlight/sequence/representations.py:91-114, CNNNet :385-422),
// the target/negative scoring (:136-144, :444-453), the masked loss
// (spotlight/losses.py) and loss.backward().
//
// Data layout: every activation is time-major (B, T, D) fp32 so a position is
// one contiguous row (the reference's (B, D, T, 1) conv layout is only a view
// for cuDNN).  Representation entry t has seen items < t; T = S + 1.
//
// Kernels
//   seq_mask_kernel      sum of the mask (seq != 0), id range check
//   pool_rep_kernel      causal prefix mean; one CTA per sequence, 8 warps split
//                        the time axis (two-level scan through shared memory)
//   conv_gemm_kernel     causal dilated conv as a shifted-row GEMM on the tensor cores
//                        (mma.sync TF32, 3xTF32 split for fp32-level accuracy, 64x64x16
//                        tiles): forward (+bias, act, residual) and input-gradient modes;
//                        at D = 128 tc_conv_gemm_kernel / tc_conv_dw_kernel (wgmma, seq_tc.cuh)
//   conv_dw_kernel       weight gradient, split over positions + fixed-order reduce
//   seq_score_kernel     one lane group per position: dots, loss, d loss/d r,
//                        target-role contribution rows, row counts
//   pool_bwd_kernel      exclusive suffix sums of d r / (count + 1)
//   seq_fill / seq_reduce  deterministic segmented scatter into dE, dbias
//   lstm_fwd / lstm_bwd  LSTMNet recurrence and its BPTT on thread-block clusters (seq_lstm.cuh);
//                        the LSTM's projections and weight gradients are k = 1 conv GEMMs
//   mix_score_kernel     MixtureLSTMNet head (seq_mix.cuh): softmax-weighted taste scores and their
//                        gradients into the 2M projection blocks; the projection is 2M k = 1 conv GEMMs
//
// Hashed item table (BloomEmbedding, item_hashes > 0): seq_gather_hashed_kernel sums each
// position's H hashed rows once into Xs (B, S, D) -- the X0 of CNN / LSTM / mixture -- and the pool,
// score and mixture kernels read the input and target rows from it by position (template row
// source); negatives are summed from their hashed rows where they are scored.  The backward keys
// every term once per hash onto table rows and once onto its id's bias, in one segment index over
// the two key spaces; hot rows go through seg_sort_long_kernel.
#include <stdlib.h>

#include "segindex.cuh"

namespace {

constexpr int SQ_THREADS = 256;
constexpr int SQ_MAX_GRID = 132 * 8;
constexpr int MAX_LAYERS = 8;

struct SeqDev {
    int64_t B; int S; int T;          // T = S + 1
    int64_t I; int D;
    const int64_t* seqs; const int64_t* negs;
    int loss; int n_neg;
    const float* E; const float* bias;
    float* rep;        // (B, T, D) final representation
    float* dR;         // (B, T, D)
    float* C;          // (2*B*S, D) contribution rows: [0,BS) seq role, [BS,2BS) neg role
    int32_t* keys;     // (2*B*S) row id or -1
    float* gs;         // (2*B*S) score grads (bias grads)
    int32_t* hdr;      // [0] done, [1] err, [2] mask count
    const int32_t* norm;   // optional global mask count (multi-GPU)
    float* partial;
    float* loss_out; float* pos_out; float* neg_out;
    float* dE; float* dbias;
    // fused row-wise optimizer (0 = gradients written to dE / dbias)
    int32_t opt; float lr, wd, eps; float* sE; float* sbias;
    SegIndex seg;
    // MixtureLSTMNet head: M mixtures, P = 2M blocks of (B, T, D) (components, then mixture
    // vectors); mix_score_kernel overwrites P with d loss / d P
    int M; float* P;
    // hashed item table (H > 0): E holds Mrows rows, an item is the sum of its H rows (item4);
    // Xs (B, S, D) holds the summed rows of the sequence positions, read by position
    int H; int64_t Mrows; uint32_t seeds[24];
    const float* Xs;
    // lazy-exact Adam (SLB_OPT_ADAM): sE / sbias hold exp_avg, vE / vbias exp_avg_sq; lastE / lastb
    // the step a table row / bias is current for (a plain table's bias shares lastE)
    AdamDev ad; float* vE; float* vbias; int32_t* lastE; int32_t* lastb;
};

// Row source of the item reads: a plain table by id, or the hashed sum of the H rows of the
// id in hash order (BloomEmbedding, layers.py:132-244; the padding id maps to row 0).
template <bool HASHED>
__device__ __forceinline__ float4 item4(const SeqDev& a, int64_t id, int c) {
    if (!HASHED) return ldg4(a.E + id * a.D + c);
    float4 s = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
    for (int k = 0; k < 24; ++k) {          // static seed indices: the seeds stay in the parameter bank
        if (k < a.H) {
            const float4 v = ldg4(a.E + bloom_row(id, a.seeds[k], a.Mrows, 0) * a.D + c);
            s.x += v.x; s.y += v.y; s.z += v.z; s.w += v.w;
        }
    }
    return s;
}

// ---------------------------------------------------------------- mask count
__global__ void __launch_bounds__(256)
seq_mask_kernel(const int64_t* __restrict__ seqs, const int64_t* __restrict__ negs, int64_t n,
                int64_t n_negs, int64_t I, int32_t* hdr) {
    __shared__ int sh[8];
    int c = 0;
    bool bad = false;
    const int64_t nth = static_cast<int64_t>(gridDim.x) * blockDim.x;
    for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += nth) {
        const int64_t v = seqs[i];
        c += v != 0;
        bad |= v < 0 || v >= I;
    }
    if (negs)
        for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n_negs; i += nth) {
            const int64_t v = negs[i];
            bad |= v < 0 || v >= I;
        }
    if (bad) atomicExch(hdr + 1, 1);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) c += __shfl_down_sync(0xffffffffu, c, o);
    if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = c;
    __syncthreads();
    if (threadIdx.x == 0) {
        int s = 0;
        for (int k = 0; k < 8; ++k) s += sh[k];
        if (s) atomicAdd(hdr + 2, s);      // integer: order-independent
    }
}

__device__ __forceinline__ int64_t clamp_id(int64_t v, int64_t I) { return v < 0 || v >= I ? 0 : v; }

// Input row of position (b, t): E[seq] of a plain table, or (BYPOS) row b * S + t of the
// materialised (B, S, D) rows of a hashed one.
template <bool BYPOS>
__device__ __forceinline__ const float* in_row(const float* E, const int64_t* sq, int64_t b, int t, int S, int D,
                                               int64_t I) {
    return BYPOS ? E + (b * S + t) * D : E + clamp_id(sq[t], I) * D;
}

// ------------------------------------------------------------------ PoolNet
// r_t = sum_{s<t} e_s / (sum_{s<t} [e_s != 0] + 1)      representations.py:91-114
// One CTA per sequence; warp w owns time chunk [w*ch, (w+1)*ch).
template <int NCH, bool BYPOS>
__global__ void __launch_bounds__(SQ_THREADS)
pool_rep_kernel(const float* __restrict__ E, const int64_t* __restrict__ seqs, int S, int D,
                int64_t I, float* __restrict__ rep) {
    extern __shared__ float sh[];            // [8][D] sums, [8][D] counts
    const int b = blockIdx.x;
    const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int ch = (S + 7) / 8;
    const int lo = min(w * ch, S), hi = min(lo + ch, S);
    const int64_t* sq = seqs + static_cast<int64_t>(b) * S;
    float4 sum[NCH], cnt[NCH];
#pragma unroll
    for (int q = 0; q < NCH; ++q) { sum[q] = make_float4(0, 0, 0, 0); cnt[q] = make_float4(0, 0, 0, 0); }
    for (int t = lo; t < hi; ++t) {
        const float* row = in_row<BYPOS>(E, sq, b, t, S, D, I);
#pragma unroll
        for (int q = 0; q < NCH; ++q) {
            const int c = lane * 4 + q * 128;
            if (c < D) {
                const float4 e = ldg4(row + c);
                sum[q].x += e.x; sum[q].y += e.y; sum[q].z += e.z; sum[q].w += e.w;
                cnt[q].x += e.x != 0.f; cnt[q].y += e.y != 0.f; cnt[q].z += e.z != 0.f; cnt[q].w += e.w != 0.f;
            }
        }
    }
#pragma unroll
    for (int q = 0; q < NCH; ++q) {
        const int c = lane * 4 + q * 128;
        if (c < D) { st4(sh + w * D + c, sum[q]); st4(sh + (8 + w) * D + c, cnt[q]); }
    }
    __syncthreads();
    float4 P[NCH], Cn[NCH];
#pragma unroll
    for (int q = 0; q < NCH; ++q) {
        P[q] = make_float4(0, 0, 0, 0); Cn[q] = make_float4(0, 0, 0, 0);
        const int c = lane * 4 + q * 128;
        if (c < D)
            for (int w2 = 0; w2 < w; ++w2) {
                const float4 a = ld4(sh + w2 * D + c), k = ld4(sh + (8 + w2) * D + c);
                P[q].x += a.x; P[q].y += a.y; P[q].z += a.z; P[q].w += a.w;
                Cn[q].x += k.x; Cn[q].y += k.y; Cn[q].z += k.z; Cn[q].w += k.w;
            }
    }
    float* out = rep + static_cast<int64_t>(b) * (S + 1) * D;
    for (int t = lo; t < hi; ++t) {
        const float* row = in_row<BYPOS>(E, sq, b, t, S, D, I);
#pragma unroll
        for (int q = 0; q < NCH; ++q) {
            const int c = lane * 4 + q * 128;
            if (c < D) {
                st4(out + static_cast<int64_t>(t) * D + c,
                    make_float4(P[q].x / (Cn[q].x + 1.f), P[q].y / (Cn[q].y + 1.f),
                                P[q].z / (Cn[q].z + 1.f), P[q].w / (Cn[q].w + 1.f)));
                const float4 e = ldg4(row + c);
                P[q].x += e.x; P[q].y += e.y; P[q].z += e.z; P[q].w += e.w;
                Cn[q].x += e.x != 0.f; Cn[q].y += e.y != 0.f; Cn[q].z += e.z != 0.f; Cn[q].w += e.w != 0.f;
            }
        }
    }
    if (w == 7) {   // final representation (all items seen); chunk 7 ends at S
#pragma unroll
        for (int q = 0; q < NCH; ++q) {
            const int c = lane * 4 + q * 128;
            if (c < D)
                st4(out + static_cast<int64_t>(S) * D + c,
                    make_float4(P[q].x / (Cn[q].x + 1.f), P[q].y / (Cn[q].y + 1.f),
                                P[q].z / (Cn[q].z + 1.f), P[q].w / (Cn[q].w + 1.f)));
        }
    }
}

// d e_s (input role) = sum_{t>s} dR_t / (c_t + 1), added onto the seq-role
// contribution rows C[b, s].   Same chunking as the forward.
template <int NCH, bool BYPOS>
__global__ void __launch_bounds__(SQ_THREADS)
pool_bwd_kernel(const float* __restrict__ E, const int64_t* __restrict__ seqs, int S, int D,
                int64_t I, const float* __restrict__ dR, float* __restrict__ C) {
    extern __shared__ float sh[];            // [8][D] counts, [8][D] dP totals
    const int b = blockIdx.x;
    const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int ch = (S + 7) / 8;
    const int lo = min(w * ch, S), hi = min(lo + ch, S);
    const int64_t* sq = seqs + static_cast<int64_t>(b) * S;
    const float* dr = dR + static_cast<int64_t>(b) * (S + 1) * D;
    float* cb = C + static_cast<int64_t>(b) * S * D;
    float4 cnt[NCH];
#pragma unroll
    for (int q = 0; q < NCH; ++q) cnt[q] = make_float4(0, 0, 0, 0);
    for (int t = lo; t < hi; ++t) {
        const float* row = in_row<BYPOS>(E, sq, b, t, S, D, I);
#pragma unroll
        for (int q = 0; q < NCH; ++q) {
            const int c = lane * 4 + q * 128;
            if (c < D) {
                const float4 e = ldg4(row + c);
                cnt[q].x += e.x != 0.f; cnt[q].y += e.y != 0.f; cnt[q].z += e.z != 0.f; cnt[q].w += e.w != 0.f;
            }
        }
    }
#pragma unroll
    for (int q = 0; q < NCH; ++q) {
        const int c = lane * 4 + q * 128;
        if (c < D) st4(sh + w * D + c, cnt[q]);
    }
    __syncthreads();
    // count before position `hi` = counts of chunks <= w
    float4 cend[NCH];
#pragma unroll
    for (int q = 0; q < NCH; ++q) {
        cend[q] = make_float4(0, 0, 0, 0);
        const int c = lane * 4 + q * 128;
        if (c < D)
            for (int w2 = 0; w2 <= w; ++w2) {
                const float4 k = ld4(sh + w2 * D + c);
                cend[q].x += k.x; cend[q].y += k.y; cend[q].z += k.z; cend[q].w += k.w;
            }
    }
    for (int pass = 0; pass < 2; ++pass) {
        float4 sfx[NCH], cc[NCH];
#pragma unroll
        for (int q = 0; q < NCH; ++q) {
            cc[q] = cend[q];
            sfx[q] = make_float4(0, 0, 0, 0);
            const int c = lane * 4 + q * 128;
            if (pass == 1 && c < D)
                for (int w2 = w + 1; w2 < 8; ++w2) {
                    const float4 k = ld4(sh + (8 + w2) * D + c);
                    sfx[q].x += k.x; sfx[q].y += k.y; sfx[q].z += k.z; sfx[q].w += k.w;
                }
        }
        for (int t = hi - 1; t >= lo; --t) {
            const float* row = in_row<BYPOS>(E, sq, b, t, S, D, I);
#pragma unroll
            for (int q = 0; q < NCH; ++q) {
                const int c = lane * 4 + q * 128;
                if (c < D) {
                    const float4 e = ldg4(row + c);
                    // c_t = c_{t+1} - [e_t != 0]
                    cc[q].x -= e.x != 0.f; cc[q].y -= e.y != 0.f; cc[q].z -= e.z != 0.f; cc[q].w -= e.w != 0.f;
                    const float4 g = ld4(dr + static_cast<int64_t>(t) * D + c);
                    if (pass == 1) {
                        float4 o = ld4(cb + static_cast<int64_t>(t) * D + c);
                        o.x += sfx[q].x; o.y += sfx[q].y; o.z += sfx[q].z; o.w += sfx[q].w;
                        st4(cb + static_cast<int64_t>(t) * D + c, o);
                    }
                    sfx[q].x += g.x / (cc[q].x + 1.f); sfx[q].y += g.y / (cc[q].y + 1.f);
                    sfx[q].z += g.z / (cc[q].z + 1.f); sfx[q].w += g.w / (cc[q].w + 1.f);
                }
            }
        }
        if (pass == 0) {
#pragma unroll
            for (int q = 0; q < NCH; ++q) {
                const int c = lane * 4 + q * 128;
                if (c < D) st4(sh + (8 + w) * D + c, sfx[q]);
            }
            __syncthreads();
        }
    }
}

// ------------------------------------------------------------------ scoring
// representations.py:136-144 / 444-453 + the masked loss + d loss / d r.
// Masked loss of the step: the grid's loss sum (grid_fold: fixed order, no float atomics) over
// msum positions.
__device__ __forceinline__ void seq_loss_fold(const SeqDev& a, float lsum, float msum) {
    __shared__ float sh_red[SQ_THREADS / 32];
    __shared__ bool is_last;
    float t;
    if (grid_fold<SQ_THREADS>(lsum, sh_red, is_last, a.partial, a.hdr, t)) *a.loss_out = t / msum;
}

// Backward keys of one position's terms.  Plain table: the seq-role term pidx and the credited
// negative's term BS + pidx are keyed by item id (row 0 frozen).  Hashed table (H > 0), one
// segment index over two key spaces: [0, Mrows) table rows, term m = t * H + k for hash k of
// term t's id (a key on the frozen row 0 dropped); [Mrows, Mrows + I) bias ids, term 2 * BS * H + t,
// keyed as the plain table keys its rows.
template <bool HASHED>
__device__ __forceinline__ void seq_keys(const SeqDev& a, int64_t BS, int64_t pidx, int64_t id, int64_t nid,
                                         float gn) {
    const bool ks = id != 0, kn = nid != 0 && gn != 0.f;
    if (!HASHED) {
        a.keys[pidx] = ks ? static_cast<int32_t>(id) : -1;
        a.keys[BS + pidx] = kn ? static_cast<int32_t>(nid) : -1;
        if (ks) atomicAdd(a.seg.cnt + id, 1);
        if (kn) atomicAdd(a.seg.cnt + nid, 1);
        return;
    }
    const int H = a.H;
#pragma unroll
    for (int k = 0; k < 24; ++k) {          // static seed indices, as item4
        if (k < H) {
            const int64_t rs = bloom_row(id, a.seeds[k], a.Mrows, 0);
            const int64_t rn = kn ? bloom_row(nid, a.seeds[k], a.Mrows, 0) : 0;
            a.keys[pidx * H + k] = rs != 0 ? static_cast<int32_t>(rs) : -1;
            a.keys[(BS + pidx) * H + k] = rn != 0 ? static_cast<int32_t>(rn) : -1;
            if (rs != 0) atomicAdd(a.seg.cnt + rs, 1);
            if (rn != 0) atomicAdd(a.seg.cnt + rn, 1);
        }
    }
    const int64_t TH = 2 * BS * H;
    a.keys[TH + pidx] = ks ? static_cast<int32_t>(a.Mrows + id) : -1;
    a.keys[TH + BS + pidx] = kn ? static_cast<int32_t>(a.Mrows + nid) : -1;
    if (ks) atomicAdd(a.seg.cnt + a.Mrows + id, 1);
    if (kn) atomicAdd(a.seg.cnt + a.Mrows + nid, 1);
}

template <int LPR, bool HASHED>
__global__ void __launch_bounds__(SQ_THREADS) seq_score_kernel(SeqDev a) {
    constexpr int GROUPS = SQ_THREADS / LPR;
    if (HASHED && blockIdx.x == 0 && threadIdx.x == 0) a.seg.totals[3] = 0;   // hot-row list of this step
    const int gl = threadIdx.x & (LPR - 1);
    const unsigned gmask = group_mask(LPR);
    const int D = a.D, S = a.S, T = a.T;
    const int64_t BS = a.B * S, BT = a.B * T;
    const float msum = static_cast<float>(a.norm ? *a.norm : a.hdr[2]);
    const float inv = 1.0f / msum;
    const int64_t gid = static_cast<int64_t>(blockIdx.x) * GROUPS + threadIdx.x / LPR;
    const int64_t gstride = static_cast<int64_t>(gridDim.x) * GROUPS;
    const int64_t iters = (BT + gstride - 1) / gstride;
    float lsum = 0.f;
    for (int64_t it = 0; it < iters; ++it) {
        const int64_t m = gid + it * gstride;
        const bool valid = m < BT;
        const int64_t mm = valid ? m : 0;
        const int64_t b = mm / T;
        const int t = static_cast<int>(mm - b * T);
        float* drow = a.dR + mm * D;
        if (t == S) {                               // final step is not trained on
            if (valid) for (int c = gl * 4; c < D; c += LPR * 4) st4(drow + c, make_float4(0, 0, 0, 0));
            continue;                               // group-uniform
        }
        const int64_t pidx = b * S + t;
        const int64_t id = clamp_id(a.seqs[pidx], a.I);
        const float* r = a.rep + mm * D;
        // the target is the input item of position t: its summed row is Xs[b, t] on a hashed table
        const float* et = HASHED ? a.Xs + pidx * D : a.E + id * D;
        float dp = 0.f;
        for (int c = gl * 4; c < D; c += LPR * 4) dp += dot4(ld4(r + c), ldg4(et + c));
        const float p = group_sum<LPR>(dp, gmask) + __ldg(a.bias + id);
        float nbest = -INFINITY;
        int64_t nid = 0;
        for (int k = 0; k < a.n_neg; ++k) {
            const int64_t nidx = (static_cast<int64_t>(k) * a.B + b) * S + t;   // implicit.py:281-286
            const int64_t j = clamp_id(a.negs[nidx], a.I);
            const float* en = a.E + j * D;
            float dn = 0.f;
            for (int c = gl * 4; c < D; c += LPR * 4)
                dn += dot4(ld4(r + c), HASHED ? item4<true>(a, j, c) : ldg4(en + c));
            const float nk = group_sum<LPR>(dn, gmask) + __ldg(a.bias + j);
            if (valid && gl == 0 && a.neg_out) a.neg_out[nidx] = nk;
            if (k == 0 || nk > nbest) { nbest = nk; nid = j; }
        }
        float per, gp, gn;
        pair_loss(a.loss, p, nbest, per, gp, gn);
        const float mk = id != 0 ? 1.0f : 0.0f;      // mask = seq != PADDING_IDX
        lsum += (valid && gl == 0) ? per * mk : 0.f;
        gp *= mk * inv; gn *= mk * inv;
        if (!valid) continue;                        // no shuffles below
        const float* en = a.E + nid * D;
        float* cs = a.C + pidx * D;
        float* cn = a.C + (BS + pidx) * D;
        for (int c = gl * 4; c < D; c += LPR * 4) {
            const float4 rv = ld4(r + c), ev = ldg4(et + c), nv = HASHED ? item4<true>(a, nid, c) : ldg4(en + c);
            st4(drow + c, make_float4(gp * ev.x + gn * nv.x, gp * ev.y + gn * nv.y,
                                      gp * ev.z + gn * nv.z, gp * ev.w + gn * nv.w));
            st4(cs + c, make_float4(gp * rv.x, gp * rv.y, gp * rv.z, gp * rv.w));
            st4(cn + c, make_float4(gn * rv.x, gn * rv.y, gn * rv.z, gn * rv.w));
        }
        if (gl == 0) {
            if (a.pos_out) a.pos_out[pidx] = p;
            // rows of the padding id are frozen (padding_idx=0): drop their terms
            seq_keys<HASHED>(a, BS, pidx, id, nid, gn);
            a.gs[pidx] = gp; a.gs[BS + pidx] = gn;
        }
    }
    seq_loss_fold(a, lsum, msum);
}

__global__ void __launch_bounds__(256) seq_fill_kernel(SeqDev a) {
    seg_rearm(a.seg);
    const int64_t T2 = 2 * a.B * a.S * (a.H + 1);      // keys of the step (plain: H = 0)
    const int64_t nth = static_cast<int64_t>(gridDim.x) * blockDim.x;
    for (int64_t t = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; t < T2; t += nth) {
        const int32_t k = a.keys[t];
        if (k >= 0) seg_place(a.seg, k, static_cast<int32_t>(t));
    }
}

// One lane group per touched row: sums the row's contribution rows C[t] and score gradients
// gs[t] in ascending term order, then writes dE / dbias, or applies the fused optimizer.
// The fused optimizer updates a row (embedding and bias together) when any of its terms has
// a non-zero score gradient or its summed embedding gradient is non-zero -- the MF rule
// (mf_v2.cuh user_member / user_finish) extended by the input role, whose gradient reaches a
// row through later positions' scores.  With weight decay an updated row is decayed in every
// element, including those whose gradient is zero.
// Hashed table (H > 0): a table-row segment sums C[m / H] over its terms m (a row named by two
// hashes of one id takes the term twice) and owns no bias; a bias segment (row >= Mrows) sums
// gs[m - 2 BS H] and, fused, updates the bias of id row - Mrows when one of its terms has a
// non-zero score gradient (the MF Bloom rule).  Hot rows were pre-sorted by seg_sort_long_kernel.
template <int LPR, bool HASHED>
__global__ void __launch_bounds__(SQ_THREADS) seq_reduce_kernel(SeqDev a) {
    constexpr int GROUPS = SQ_THREADS / LPR;
    constexpr int CAP = seg_sort_cap(LPR);
    constexpr int NCH = LPR == 32 ? 4 : 1;   // float4 chunks per lane: D <= LPR * 4 below 128, <= 512
    __shared__ int32_t sh_sort[GROUPS * 2 * CAP];
    const int gl = threadIdx.x & (LPR - 1);
    const int gib = threadIdx.x / LPR;
    const unsigned gmask = group_mask(LPR);
    int32_t* sh = sh_sort + gib * 2 * CAP;
    const int D = a.D;
    const int H = HASHED ? a.H : 0;
    const int64_t TH = 2 * a.B * a.S * H;    // first bias term of a hashed step
    const int nseg = a.seg.totals[0];
    for (int64_t s = static_cast<int64_t>(blockIdx.x) * GROUPS + gib; s < nseg;
         s += static_cast<int64_t>(gridDim.x) * GROUPS) {
        const int start = a.seg.seg_start[s];
        const int len = a.seg.seg_start[s + 1] - start;
        const int64_t row = a.seg.seg_row[s];
        const bool bseg = H > 0 && row >= a.Mrows;    // a bias segment of a hashed step (group-uniform)
        float4 acc[NCH];
#pragma unroll
        for (int q = 0; q < NCH; ++q) acc[q] = make_float4(0, 0, 0, 0);
        float bacc = 0.f;
        bool nz = false;                     // a term with a non-zero score gradient (group-uniform)
        seg_visit_sorted<LPR>(a.seg.members, start, len, gl, gmask, sh, [&](int32_t m) {
            const int64_t t = H == 0 ? m : (bseg ? m - TH : m / H);
            if (!bseg) {
                const float* src = a.C + t * D;
#pragma unroll
                for (int q = 0; q < NCH; ++q) {
                    const int c = gl * 4 + q * LPR * 4;
                    if (c < D) {
                        const float4 v = ld4(src + c);
                        acc[q].x += v.x; acc[q].y += v.y; acc[q].z += v.z; acc[q].w += v.w;
                    }
                }
            }
            const float g = a.gs[t];
            bacc += g;
            nz = nz || g != 0.f;
        }, HASHED);
        if (bseg) {
            if (gl == 0) {
                if (a.opt == SLB_OPT_NONE) {
                    a.dbias[row - a.Mrows] = bacc;
                } else if (nz) {
                    const OptV2 o = {a.opt, a.lr, a.wd, a.eps};
                    bias_update(o, const_cast<float*>(a.bias) + (row - a.Mrows),
                                a.opt == SLB_OPT_ADAGRAD ? a.sbias + (row - a.Mrows) : nullptr, bacc);
                }
            }
            continue;
        }
        if (a.opt == SLB_OPT_NONE) {
#pragma unroll
            for (int q = 0; q < NCH; ++q) {
                const int c = gl * 4 + q * LPR * 4;
                if (c < D) st4(a.dE + row * D + c, acc[q]);
            }
            if (gl == 0 && H == 0) a.dbias[row] = bacc;
            continue;
        }
#pragma unroll
        for (int q = 0; q < NCH; ++q)
            nz = nz || acc[q].x != 0.f || acc[q].y != 0.f || acc[q].z != 0.f || acc[q].w != 0.f;
        if (!__any_sync(gmask, nz)) continue;   // group-uniform
        // row-wise optimizer applied in place: this is the last kernel of the step, every
        // gradient that reads E has been formed
        const OptV2 o = {a.opt, a.lr, a.wd, a.eps};
#pragma unroll
        for (int q = 0; q < NCH; ++q) {
            const int c = gl * 4 + q * LPR * 4;
            if (c < D) {
                float* wrow = const_cast<float*>(a.E) + row * D + c;
                float* srow = a.opt == SLB_OPT_ADAGRAD ? a.sE + row * D + c : nullptr;
                float4 w4 = ld4(wrow), s4 = make_float4(0.f, 0.f, 0.f, 0.f);
                if (srow) s4 = ld4(srow);
                row_update(o, w4, s4, acc[q]);
                st4(wrow, w4);
                if (srow) st4(srow, s4);
            }
        }
        if (gl == 0 && H == 0)
            bias_update(o, const_cast<float*>(a.bias) + row, a.opt == SLB_OPT_ADAGRAD ? a.sbias + row : nullptr, bacc);
    }
}

// Lazy-exact Adam (SLB_OPT_ADAM) in place of seq_reduce_kernel's optimizers: the segment sum is
// the same; the summed gradient of a row takes the real step t and the row's last becomes t.
// seq_adam_prepass_kernel has made every keyed row current through t - 1.  A row whose terms are all
// zero is skipped: a gradient-free step equals the catch-up it gets when next referenced or
// flushed, so this stays dense Adam, weight decay included.  (A kernel of its own, so that the
// SGD / Adagrad / gradient instantiations of seq_reduce_kernel keep their code.)
template <int LPR, bool HASHED>
__global__ void __launch_bounds__(SQ_THREADS) seq_reduce_adam_kernel(SeqDev a) {
    constexpr int GROUPS = SQ_THREADS / LPR;
    constexpr int CAP = seg_sort_cap(LPR);
    constexpr int NCH = LPR == 32 ? 4 : 1;
    __shared__ int32_t sh_sort[GROUPS * 2 * CAP];
    const int gl = threadIdx.x & (LPR - 1);
    const int gib = threadIdx.x / LPR;
    const unsigned gmask = group_mask(LPR);
    int32_t* sh = sh_sort + gib * 2 * CAP;
    const int D = a.D;
    const int H = HASHED ? a.H : 0;
    const int64_t TH = 2 * a.B * a.S * H;
    const int nseg = a.seg.totals[0];
    const AdamDev o = a.ad;
    for (int64_t s = static_cast<int64_t>(blockIdx.x) * GROUPS + gib; s < nseg;
         s += static_cast<int64_t>(gridDim.x) * GROUPS) {
        const int start = a.seg.seg_start[s];
        const int len = a.seg.seg_start[s + 1] - start;
        const int64_t row = a.seg.seg_row[s];
        const bool bseg = H > 0 && row >= a.Mrows;
        float4 acc[NCH];
#pragma unroll
        for (int q = 0; q < NCH; ++q) acc[q] = make_float4(0, 0, 0, 0);
        float bacc = 0.f;
        bool nz = false;
        seg_visit_sorted<LPR>(a.seg.members, start, len, gl, gmask, sh, [&](int32_t m) {
            const int64_t t = H == 0 ? m : (bseg ? m - TH : m / H);
            if (!bseg) {
                const float* src = a.C + t * D;
#pragma unroll
                for (int q = 0; q < NCH; ++q) {
                    const int c = gl * 4 + q * LPR * 4;
                    if (c < D) {
                        const float4 v = ld4(src + c);
                        acc[q].x += v.x; acc[q].y += v.y; acc[q].z += v.z; acc[q].w += v.w;
                    }
                }
            }
            const float g = a.gs[t];
            bacc += g;
            nz = nz || g != 0.f;
        }, HASHED);
        // the bias of a plain row (shares the row's last), or of a hashed bias segment (its own)
        const int64_t bid = bseg ? row - a.Mrows : row;
        float ss, bc;                         // this step's scalars, loaded where they are used
        if (!bseg) {
#pragma unroll
            for (int q = 0; q < NCH; ++q)
                nz = nz || acc[q].x != 0.f || acc[q].y != 0.f || acc[q].z != 0.f || acc[q].w != 0.f;
            if (!__any_sync(gmask, nz)) continue;   // group-uniform
            ss = __ldg(o.sched + 2 * o.t); bc = __ldg(o.sched + 2 * o.t + 1);
#pragma unroll
            for (int q = 0; q < NCH; ++q) {
                const int c = gl * 4 + q * LPR * 4;
                if (c < D) {
                    float* W = const_cast<float*>(a.E) + row * D + c;
                    float4 w = ld4(W), m = ld4(a.sE + row * D + c), v = ld4(a.vE + row * D + c);
                    adam_elem(o, ss, bc, acc[q].x, w.x, m.x, v.x);
                    adam_elem(o, ss, bc, acc[q].y, w.y, m.y, v.y);
                    adam_elem(o, ss, bc, acc[q].z, w.z, m.z, v.z);
                    adam_elem(o, ss, bc, acc[q].w, w.w, m.w, v.w);
                    st4(W, w); st4(a.sE + row * D + c, m); st4(a.vE + row * D + c, v);
                }
            }
            if (gl == 0) a.lastE[row] = o.t;
        } else if (!nz) {
            continue;
        } else {
            ss = __ldg(o.sched + 2 * o.t); bc = __ldg(o.sched + 2 * o.t + 1);
        }
        if (gl == 0 && (H == 0 || bseg)) {
            float* bw = const_cast<float*>(a.bias) + bid;
            float w = *bw, m = a.sbias[bid], v = a.vbias[bid];
            adam_elem(o, ss, bc, bacc, w, m, v);
            *bw = w; a.sbias[bid] = m; a.vbias[bid] = v;
            if (bseg) a.lastb[bid] = o.t;
        }
    }
}

// Lazy-exact Adam, before anything in step t reads E: every row the minibatch references is
// brought current through step t - 1 (dense Adam moved it at every step it missed, and the
// representation and the scores must see that).  References: each sequence position (its item is
// both an input and a target) and each negative; on a hashed table each of the id's H rows (work
// slot k < H) and the id's bias (slot H).  The padding id is caught up like any other: dense Adam
// with weight decay moves its row, whose gradient is zero.  atomicMax on last elects one lane group
// per distinct row, as mf_adam_prepass_kernel does.
template <int LPR, bool HASHED>
__global__ void __launch_bounds__(SQ_THREADS) seq_adam_prepass_kernel(SeqDev a) {
    constexpr int GROUPS = SQ_THREADS / LPR;
    __shared__ uint32_t sh_seeds[24];
    if (HASHED && threadIdx.x == 0) {
#pragma unroll
        for (int k = 0; k < 24; ++k) sh_seeds[k] = a.seeds[k];   // static indices: the seeds stay in the parameter bank
    }
    if (HASHED) __syncthreads();
    const int gl = threadIdx.x & (LPR - 1);
    const unsigned gmask = group_mask(LPR);
    const int D = a.D;
    const int upto = a.ad.t - 1;
    const int64_t BS = a.B * a.S;
    const int slots = HASHED ? a.H + 1 : 1;
    const int64_t total = BS * (1 + a.n_neg) * slots;
    for (int64_t w = static_cast<int64_t>(blockIdx.x) * GROUPS + threadIdx.x / LPR; w < total;
         w += static_cast<int64_t>(gridDim.x) * GROUPS) {
        const int64_t r = HASHED ? w / slots : w;
        const int k = HASHED ? static_cast<int>(w - r * slots) : 0;
        const int64_t id = clamp_id(r < BS ? a.seqs[r] : a.negs[r - BS], a.I);   // seq_mask_kernel flags bad ids
        const bool bslot = HASHED && k == a.H;                                   // group-uniform
        const int64_t row = (HASHED && !bslot) ? bloom_row(id, sh_seeds[k], a.Mrows, 0) : id;
        int32_t* last = (bslot ? a.lastb : a.lastE) + row;
        int old = 0;
        if (gl == 0) old = atomicMax(last, upto);
        old = __shfl_sync(gmask, old, (threadIdx.x & 31) & ~(LPR - 1));
        if (old >= upto) continue;
        if (!bslot) {
            float* W = const_cast<float*>(a.E) + row * D;
            float* M = a.sE + row * D;
            float* V = a.vE + row * D;
            for (int c = gl * 4; c < D; c += LPR * 4) {
                float4 wv = ld4(W + c), m = ld4(M + c), v = ld4(V + c);
                adam_catch_up(a.ad, old, upto, wv, m, v);
                st4(W + c, wv); st4(M + c, m); st4(V + c, v);
            }
        }
        if (gl == 0 && (!HASHED || bslot)) {    // the bias: with its row (plain) or in its own slot
            float* bw = const_cast<float*>(a.bias) + id;
            float wb = *bw, m = a.sbias[id], v = a.vbias[id];
            adam_catch_up1(a.ad, old, upto, wb, m, v);
            *bw = wb; a.sbias[id] = m; a.vbias[id] = v;
        }
    }
}

// ------------------------------------------------------------------ CNNNet
// Causal dilated convolution as a shifted-row GEMM:
//   Out[(b,t), n] = epi( sum_{j<k} sum_{c<D} In[b, t + shift_j, c] * Wm[j][c][n] )
// rows outside [0, Tin) read as zero (the reference's left zero padding,
// representations.py:394-400, 414).
constexpr int GM = 64, GN = 64, GK = 16;

struct ConvGemm {
    const float* In; int Tin;
    float* Out; int Tout;
    const float* Wm;              // [k][D][D]
    int k; int shift[16];
    int64_t B; int D;
    int mode;                     // 0 forward, 1 input gradient
    // forward epilogue; nonlin 0 tanh, 1 relu, 2 identity (a bias-only projection)
    const float* bias; int nonlin; float* Aout;     // activation (pre-residual), nullable
    const float* Res; int res_T; int res_shift;     // Res[b, t + res_shift] added when in range
    // input-gradient epilogue: Out = acc + Res[...]; accumulate != 0 -> Out += ...
    int accumulate;
};

// Tensor-core inner product with fp32-level accuracy: mma.sync m16n8k8 TF32 with the
// 3xTF32 error-compensated split (a = a_hi + a_lo, b = b_hi + b_lo; the product keeps
// a_lo*b_hi + a_hi*b_lo + a_hi*b_hi), accumulating in fp32.  Relative error ~2^-21,
// inside the 1e-5 parity budget that plain TF32 (2^-11) would miss (SURVEY hard part 4).
// Tiles live in shared memory as As[k][row] / Bs[k][col] with a 72-float stride so the
// fragment loads (k = lane%4, row/col = lane/4) are bank-conflict free.
constexpr int TS = 72;      // padded tile stride

__device__ __forceinline__ uint32_t tf32_hi(float x) {
    uint32_t r;
    asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(x));
    return r;
}
__device__ __forceinline__ void split_tf32(float x, uint32_t& hi, uint32_t& lo) {
    hi = tf32_hi(x);
    lo = tf32_hi(x - __uint_as_float(hi));
}
__device__ __forceinline__ void mma_tf32(float (&c)[4], const uint32_t (&a)[4], const uint32_t (&b)[2]) {
    asm volatile("mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                 : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b[0]), "r"(b[1]));
}

// One GK = 16 deep chunk for a warp's 16 x 32 output tile (4 n-subtiles of 8).
__device__ __forceinline__ void warp_mma_chunk(const float (*As)[TS], const float (*Bs)[TS], int wm, int wn,
                                               int lane, float (&acc)[4][4]) {
    const int gq = lane >> 2, tq = lane & 3;
#pragma unroll
    for (int k8 = 0; k8 < GK; k8 += 8) {
        uint32_t ah[4], al[4];
        split_tf32(As[k8 + tq][wm * 16 + gq], ah[0], al[0]);
        split_tf32(As[k8 + tq][wm * 16 + gq + 8], ah[1], al[1]);
        split_tf32(As[k8 + tq + 4][wm * 16 + gq], ah[2], al[2]);
        split_tf32(As[k8 + tq + 4][wm * 16 + gq + 8], ah[3], al[3]);
#pragma unroll
        for (int ns = 0; ns < 4; ++ns) {
            uint32_t bh[2], bl[2];
            split_tf32(Bs[k8 + tq][wn * 32 + ns * 8 + gq], bh[0], bl[0]);
            split_tf32(Bs[k8 + tq + 4][wn * 32 + ns * 8 + gq], bh[1], bl[1]);
            mma_tf32(acc[ns], al, bh);
            mma_tf32(acc[ns], ah, bl);
            mma_tf32(acc[ns], ah, bh);
        }
    }
}

__device__ __forceinline__ float conv_act(float v, int nonlin) {
    return nonlin == 0 ? tanhf(v) : (nonlin == 1 ? fmaxf(v, 0.f) : v);
}

__global__ void __launch_bounds__(256) conv_gemm_kernel(ConvGemm g) {
    __shared__ float As[GK][TS];
    __shared__ float Bs[GK][TS];
    const int tid = threadIdx.x;
    const int lane = tid & 31, warp = tid >> 5;
    const int wm = warp & 3, wn = warp >> 2;
    const int64_t M = g.B * g.Tout;
    const int64_t m0 = static_cast<int64_t>(blockIdx.x) * GM;
    const int n0 = blockIdx.y * GN;
    const int D = g.D;
    float acc[4][4] = {};
    // A-tile load mapping: row ar (0..63), 4 consecutive channels at ac
    const int ar = tid >> 2, ac = (tid & 3) * 4;
    const int64_t am = m0 + ar;
    const int64_t ab = am < M ? am / g.Tout : 0;
    const int at = am < M ? static_cast<int>(am - ab * g.Tout) : 0;
    // B-tile load mapping
    const int bk = tid >> 4, bn = (tid & 15) * 4;
    for (int j = 0; j < g.k; ++j) {
        const int q = at + g.shift[j];
        const bool rowok = am < M && q >= 0 && q < g.Tin;
        const float* arow = g.In + (ab * g.Tin + (rowok ? q : 0)) * D;
        const float* wj = g.Wm + static_cast<int64_t>(j) * D * D;
        for (int c0 = 0; c0 < D; c0 += GK) {
            float4 av = make_float4(0, 0, 0, 0);
            if (rowok && c0 + ac < D) av = ld4(arow + c0 + ac);
            float4 bv = make_float4(0, 0, 0, 0);
            if (c0 + bk < D && n0 + bn < D) bv = ldg4(wj + static_cast<int64_t>(c0 + bk) * D + n0 + bn);
            __syncthreads();
            As[ac][ar] = av.x; As[ac + 1][ar] = av.y; As[ac + 2][ar] = av.z; As[ac + 3][ar] = av.w;
            *reinterpret_cast<float4*>(&Bs[bk][bn]) = bv;
            __syncthreads();
            warp_mma_chunk(As, Bs, wm, wn, lane, acc);
        }
    }
    // epilogue: thread owns rows (wm*16 + gq, +8), column pairs (wn*32 + ns*8 + 2*tq, +1)
    const int gq = lane >> 2, tq = lane & 3;
#pragma unroll
    for (int half = 0; half < 2; ++half) {
        const int64_t m = m0 + wm * 16 + gq + half * 8;
        if (m >= M) continue;
        const int64_t b = m / g.Tout;
        const int t = static_cast<int>(m - b * g.Tout);
        const int rt = t + g.res_shift;
        const bool resok = g.Res && rt >= 0 && rt < g.res_T;
#pragma unroll
        for (int ns = 0; ns < 4; ++ns) {
            const int n = n0 + wn * 32 + ns * 8 + 2 * tq;
            if (n >= D) continue;
            float v0 = acc[ns][half * 2], v1 = acc[ns][half * 2 + 1];
            float2 res = make_float2(0.f, 0.f);
            if (resok) res = *reinterpret_cast<const float2*>(g.Res + (b * g.res_T + rt) * D + n);
            if (g.mode == 0) {
                const float2 bb = *reinterpret_cast<const float2*>(g.bias + n);
                v0 = conv_act(v0 + bb.x, g.nonlin);
                v1 = conv_act(v1 + bb.y, g.nonlin);
                if (g.Aout) *reinterpret_cast<float2*>(g.Aout + m * D + n) = make_float2(v0, v1);
            }
            float2 o = make_float2(v0 + res.x, v1 + res.y);
            if (g.accumulate) {
                const float2 old = *reinterpret_cast<const float2*>(g.Out + m * D + n);
                o.x += old.x; o.y += old.y;
            }
            *reinterpret_cast<float2*>(g.Out + m * D + n) = o;
        }
    }
}

// dZ = dY * act'(A)
__global__ void __launch_bounds__(256)
conv_dz_kernel(const float* __restrict__ dY, const float* __restrict__ A, int64_t n4, int nonlin,
               float* __restrict__ dZ) {
    const int64_t nth = static_cast<int64_t>(gridDim.x) * blockDim.x;
    for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n4; i += nth) {
        const float4 g = ld4(dY + 4 * i), a = ld4(A + 4 * i);
        float4 o;
        if (nonlin == 0) {
            o = make_float4(g.x * (1.f - a.x * a.x), g.y * (1.f - a.y * a.y),
                            g.z * (1.f - a.z * a.z), g.w * (1.f - a.w * a.w));
        } else {
            o = make_float4(a.x > 0.f ? g.x : 0.f, a.y > 0.f ? g.y : 0.f,
                            a.z > 0.f ? g.z : 0.f, a.w > 0.f ? g.w : 0.f);
        }
        st4(dZ + 4 * i, o);
    }
}

// Weight gradient partials: part[split][j][i][o] = sum_{m in slab} In[b, t + shift_j, i] * dZ[m, o]
struct ConvDw {
    const float* In; int Tin;
    const float* dZ; int Tout;
    int k; int shift[16];
    int64_t B; int D;
    int64_t slab;                 // positions per split
    float* part;                  // [splits][k][D][D]
    float* bpart;                 // [splits][D]
};

}  // namespace
#include "seq_tc.cuh"
#include "seq_lstm.cuh"
#include "seq_mix.cuh"
namespace {

__global__ void __launch_bounds__(256) conv_dw_kernel(ConvDw g) {
    __shared__ float As[GK][TS];   // [pos][i]
    __shared__ float Bs[GK][TS];   // [pos][o]
    const int tid = threadIdx.x;
    const int lane = tid & 31, warp = tid >> 5;
    const int wm = warp & 3, wn = warp >> 2;
    const int D = g.D;
    const int tiles_n = (D + GN - 1) / GN;
    const int i0 = (blockIdx.x / tiles_n) * GM, o0 = (blockIdx.x % tiles_n) * GN;
    const int j = blockIdx.y;
    const int64_t split = blockIdx.z;
    const int64_t M = g.B * g.Tout;
    const int64_t mlo = split * g.slab, mhi = mlo + g.slab < M ? mlo + g.slab : M;
    float acc[4][4] = {};
    float bacc = 0.f;             // column sums of dZ (bias grad), by the i0 == 0, j == 0 tiles
    const int lk = tid >> 4, lc = (tid & 15) * 4;
    for (int64_t mb = mlo; mb < mhi; mb += GK) {
        const int64_t m = mb + lk;
        float4 av = make_float4(0, 0, 0, 0), bv = make_float4(0, 0, 0, 0);
        if (m < mhi) {
            const int64_t b = m / g.Tout;
            const int t = static_cast<int>(m - b * g.Tout);
            const int q = t + g.shift[j];
            if (q >= 0 && q < g.Tin && i0 + lc < D) av = ld4(g.In + (b * g.Tin + q) * D + i0 + lc);
            if (o0 + lc < D) bv = ld4(g.dZ + m * D + o0 + lc);
        }
        __syncthreads();
        *reinterpret_cast<float4*>(&As[lk][lc]) = av;
        *reinterpret_cast<float4*>(&Bs[lk][lc]) = bv;
        __syncthreads();
        warp_mma_chunk(As, Bs, wm, wn, lane, acc);
        if (i0 == 0 && j == 0 && tid < GN) {
#pragma unroll
            for (int kk = 0; kk < GK; ++kk) bacc += Bs[kk][tid];
        }
    }
    float* out = g.part + ((split * g.k + j) * D) * D;
    const int gq = lane >> 2, tq = lane & 3;
#pragma unroll
    for (int half = 0; half < 2; ++half) {
        const int i = i0 + wm * 16 + gq + half * 8;
        if (i >= D) continue;
#pragma unroll
        for (int ns = 0; ns < 4; ++ns) {
            const int o = o0 + wn * 32 + ns * 8 + 2 * tq;
            if (o < D)
                *reinterpret_cast<float2*>(out + static_cast<int64_t>(i) * D + o) =
                    make_float2(acc[ns][half * 2], acc[ns][half * 2 + 1]);
        }
    }
    if (i0 == 0 && j == 0 && tid < GN && o0 + tid < D) g.bpart[split * D + o0 + tid] = bacc;
}

// dW[o][i][j] = sum_split part[split][j][i][o] (fixed order); db likewise.
__global__ void __launch_bounds__(256)
conv_dw_reduce_kernel(const float* __restrict__ part, const float* __restrict__ bpart, int splits,
                      int k, int D, float* __restrict__ dW, float* __restrict__ db) {
    const int64_t n = static_cast<int64_t>(k) * D * D;
    const int64_t nth = static_cast<int64_t>(gridDim.x) * blockDim.x;
    for (int64_t e = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; e < n + D; e += nth) {
        float s = 0.f;
        if (e < n) {
            for (int sp = 0; sp < splits; ++sp) s += part[sp * n + e];
            const int j = static_cast<int>(e / (static_cast<int64_t>(D) * D));
            const int64_t rem = e - static_cast<int64_t>(j) * D * D;
            const int i = static_cast<int>(rem / D), o = static_cast<int>(rem - static_cast<int64_t>(i) * D);
            dW[(static_cast<int64_t>(o) * D + i) * k + j] = s;
        } else {
            const int o = static_cast<int>(e - n);
            for (int sp = 0; sp < splits; ++sp) s += bpart[sp * D + o];
            db[o] = s;
        }
    }
}

// Wf[j][i][o] = W[o][i][j] ; Wb[j][o][i] = W[o][i][j]
__global__ void __launch_bounds__(256)
conv_wt_kernel(const float* __restrict__ W, int k, int D, float* __restrict__ Wf, float* __restrict__ Wb) {
    const int64_t n = static_cast<int64_t>(k) * D * D;
    const int64_t nth = static_cast<int64_t>(gridDim.x) * blockDim.x;
    for (int64_t e = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; e < n; e += nth) {
        const int o = static_cast<int>(e / (static_cast<int64_t>(D) * k));
        const int64_t rem = e - static_cast<int64_t>(o) * D * k;
        const int i = static_cast<int>(rem / k), j = static_cast<int>(rem - static_cast<int64_t>(i) * k);
        const float v = W[e];
        Wf[(static_cast<int64_t>(j) * D + i) * D + o] = v;
        if (Wb) Wb[(static_cast<int64_t>(j) * D + o) * D + i] = v;
    }
}

// X0[b, t, :] = E[seq[b, t]]
template <int LPR>
__global__ void __launch_bounds__(SQ_THREADS)
seq_gather_kernel(const float* __restrict__ E, const int64_t* __restrict__ seqs, int64_t n, int D,
                  int64_t I, float* __restrict__ X) {
    constexpr int GROUPS = SQ_THREADS / LPR;
    const int gl = threadIdx.x & (LPR - 1);
    for (int64_t p = static_cast<int64_t>(blockIdx.x) * GROUPS + threadIdx.x / LPR; p < n;
         p += static_cast<int64_t>(gridDim.x) * GROUPS) {
        const float* row = E + clamp_id(seqs[p], I) * D;
        for (int c = gl * 4; c < D; c += LPR * 4) st4(X + p * D + c, ldg4(row + c));
    }
}

// Xs[b, t, :] = sum_k E[bloom(seq[b, t], k)]: a hashed table's input rows, summed once per step
// and then read by position (the representation's X0 and the target rows of the scores).
template <int LPR>
__global__ void __launch_bounds__(SQ_THREADS) seq_gather_hashed_kernel(SeqDev a, float* __restrict__ X) {
    constexpr int GROUPS = SQ_THREADS / LPR;
    const int gl = threadIdx.x & (LPR - 1);
    const int D = a.D;
    const int64_t n = a.B * a.S;
    for (int64_t p = static_cast<int64_t>(blockIdx.x) * GROUPS + threadIdx.x / LPR; p < n;
         p += static_cast<int64_t>(gridDim.x) * GROUPS) {
        const int64_t id = clamp_id(a.seqs[p], a.I);
        for (int c = gl * 4; c < D; c += LPR * 4) st4(X + p * D + c, item4<true>(a, id, c));
    }
}

// ------------------------------------------------------------------ host side
struct SeqLayout {
    int32_t* hdr; float* partial; SegIndex seg;
    float* rep_pool;                     // PoolNet: (B,T,D)
    float* X0;                           // CNN: (B,S,D)
    float* A[MAX_LAYERS]; float* Y[MAX_LAYERS];
    float* Wf[MAX_LAYERS]; float* Wb[MAX_LAYERS];
    float* dR; float* dZ; float* dYa; float* dYb;
    float* C; int32_t* keys; float* gs;
    float* part; float* bpart; int splits; int64_t slab;
    float* G; float* Cs; float* WT;      // LSTM: (4,B,T,D) gates, (B,T,D) cells, 4 x (D,D) W_ih^T blocks
    float* P; float* WTm;                // mixture: (2M,B,T,D) projection (d loss / d P in training),
                                         // 2M x (D,D) transposed projection blocks
    size_t bytes;
};

// The weight-gradient split counts follow the device's SM count: the fixed-order reduction
// over splits is deterministic on one GPU model, but its summation order (and so the last
// bits of dW) can differ between models with different SM counts.
int dw_splits(int64_t M, int D, int k) {
    const int tiles = ((D + GM - 1) / GM) * ((D + GN - 1) / GN) * k;
    int s = (2 * slb_sms() + tiles - 1) / tiles;
    if (s < 1) s = 1;
    if (s > 128) s = 128;
    const int64_t maxs = (M + GK - 1) / GK;
    if (s > maxs) s = static_cast<int>(maxs);
    return s;
}

// wgmma path: D == 128 exactly (one 128 x 128 tile spans all channels)
bool use_tc(int D) {
    static const bool disabled = getenv("SLB_NO_WGMMA") != nullptr;
    return !disabled && D == 128;
}

int dw_splits_tc(int64_t M, int k) {
    int s = (2 * slb_sms() + k - 1) / k;
    const int64_t maxs = (M + tc::KC - 1) / tc::KC;
    if (s > maxs) s = static_cast<int>(maxs);
    return s < 1 ? 1 : s;
}

template <typename K>
int tc_configure(K kernel) {
    return cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, tc::SMEM_BYTES) == cudaSuccess ? 0 : -1;
}

SeqLayout seq_layout(void* base, const slb_seq_step_args* x, bool training) {
    WsCarver ws(base);
    SeqLayout l = {};
    const int64_t B = x->batch, S = x->seq_len, T = S + 1, D = x->dim;
    const int L = x->n_layers;
    const int64_t H = x->item_hashes;
    // zero-at-rest region first (offsets depend on the key space only: num_items, plus item_rows
    // on a hashed table)
    l.hdr = ws.take<int32_t>(16);
    l.seg = seg_index_carve(ws, H ? x->item_rows + x->num_items : x->num_items, training ? 2 * B * S * (H + 1) : 1);
    l.partial = ws.take<float>(SQ_MAX_GRID);
    if (H && !x->lstm_w_ih && L == 0) l.X0 = ws.take<float>(B * S * D);   // PoolNet's summed input rows
    if (x->lstm_w_ih) {
        l.rep_pool = ws.take<float>(B * T * D);          // h_t
        l.X0 = ws.take<float>(B * S * D);
        l.G = ws.take<float>(4 * B * T * D);
        l.Cs = ws.take<float>(B * T * D);
        l.WT = ws.take<float>(4 * D * D);
        if (x->mix_w) {
            const int64_t J = 2 * static_cast<int64_t>(x->num_mixtures);
            l.P = ws.take<float>(J * B * T * D);
            l.WTm = ws.take<float>(J * D * D);
        }
        if (training) {                                  // k = 1 weight gradients over B * T positions
            l.splits = use_tc(static_cast<int>(D)) ? dw_splits_tc(B * T, 1) : dw_splits(B * T, static_cast<int>(D), 1);
            l.part = ws.take<float>(static_cast<size_t>(l.splits) * D * D);
            l.bpart = ws.take<float>(static_cast<size_t>(l.splits) * D);
        }
    } else if (L == 0) {
        l.rep_pool = ws.take<float>(B * T * D);
    } else {
        l.X0 = ws.take<float>(B * S * D);
        int kmax = 1;
        for (int i = 0; i < L; ++i) {
            const int k = x->kernel_width[i];
            kmax = k > kmax ? k : kmax;
            l.A[i] = ws.take<float>(B * T * D);
            l.Y[i] = x->residual ? ws.take<float>(B * T * D) : l.A[i];
            l.Wf[i] = ws.take<float>(static_cast<size_t>(k) * D * D);
            l.Wb[i] = (training || use_tc(static_cast<int>(D))) ? ws.take<float>(static_cast<size_t>(k) * D * D) : nullptr;
        }
        if (training) {
            l.dZ = ws.take<float>(B * T * D);
            l.dYa = ws.take<float>(B * T * D);
            l.dYb = ws.take<float>(B * T * D);
            size_t part_elems = 0;
            for (int i = 0; i < L; ++i) {
                const int sp = use_tc(static_cast<int>(D)) ? dw_splits_tc(B * T, x->kernel_width[i])
                                                           : dw_splits(B * T, static_cast<int>(D), x->kernel_width[i]);
                l.splits = sp > l.splits ? sp : l.splits;
                const size_t e = static_cast<size_t>(sp) * x->kernel_width[i] * D * D;
                part_elems = e > part_elems ? e : part_elems;
            }
            l.part = ws.take<float>(part_elems);
            l.bpart = ws.take<float>(static_cast<size_t>(l.splits) * D);
        }
    }
    if (training) {
        l.dR = ws.take<float>(B * T * D);
        l.C = ws.take<float>(2 * B * S * D);
        l.keys = ws.take<int32_t>(2 * B * S * (H + 1));
        l.gs = ws.take<float>(2 * B * S);
    }
    l.bytes = ws.bytes();
    return l;
}

int64_t seq_hashed_terms(const slb_seq_step_args* x) {
    return 2 * x->batch * static_cast<int64_t>(x->seq_len) * (x->item_hashes + 1);
}

int seq_validate(const slb_seq_step_args* x, bool training) {
    SLB_REQUIRE(x != nullptr, "seq: null args");
    SLB_REQUIRE(x->batch > 0 && x->seq_len > 0, "seq: empty batch");
    SLB_REQUIRE(x->dim >= 4 && x->dim % 4 == 0 && x->dim <= 512, "seq: dim must be a multiple of 4 in [4, 512] (got %d)", x->dim);
    SLB_REQUIRE(x->num_items > 0 && x->num_items < (1ll << 31) - SEG_SCAN_TILE, "seq: bad num_items");
    SLB_REQUIRE(x->seqs && x->E, "seq: null pointer");
    SLB_REQUIRE(x->n_layers >= 0 && x->n_layers <= MAX_LAYERS, "seq: at most %d conv layers", MAX_LAYERS);
    SLB_REQUIRE(x->batch * (x->seq_len + 1) * 2 < (1ll << 31), "seq: batch * seq_len too large");
    if (x->n_layers > 0) {
        SLB_REQUIRE(x->kernel_width && x->dilation && x->conv_w && x->conv_b, "seq: conv descriptors missing");
        for (int i = 0; i < x->n_layers; ++i)
            SLB_REQUIRE(x->kernel_width[i] >= 1 && x->kernel_width[i] <= 16 && x->dilation[i] >= 1,
                        "seq: kernel_width must be in [1,16], dilation >= 1");
        SLB_REQUIRE(x->nonlinearity == 0 || x->nonlinearity == 1, "seq: nonlinearity must be tanh(0) or relu(1)");
    }
    if (x->lstm_w_ih) {
        SLB_REQUIRE(x->n_layers == 0, "seq: the LSTM representation takes no conv layers");
        SLB_REQUIRE(x->dim <= 256, "seq: the fused LSTM supports dim <= 256 (got %d)", x->dim);
        SLB_REQUIRE(x->lstm_w_hh && x->lstm_b_ih && x->lstm_b_hh, "seq: LSTM parameters missing");
        if (training)
            SLB_REQUIRE(x->dlstm_w_ih && x->dlstm_w_hh && x->dlstm_b_ih && x->dlstm_b_hh, "seq: LSTM grads missing");
    }
    if (x->mix_w) {
        SLB_REQUIRE(x->lstm_w_ih != nullptr, "seq: the mixture head needs the LSTM parameters");
        SLB_REQUIRE(x->num_mixtures >= 1 && x->num_mixtures <= mix::MAX_M,
                    "seq: num_mixtures must be in [1, %d] (got %d)", mix::MAX_M, x->num_mixtures);
        SLB_REQUIRE(x->mix_b != nullptr, "seq: mixture projection bias missing");
        if (training) SLB_REQUIRE(x->dmix_w && x->dmix_b, "seq: mixture projection grads missing");
    }
    SLB_REQUIRE(x->item_hashes >= 0 && x->item_hashes <= 24, "seq: item_hashes must be in [0, 24] (got %d)", x->item_hashes);
    if (x->item_hashes > 0) {
        SLB_REQUIRE(x->item_rows > 0 && x->item_rows + x->num_items < (1ll << 31) - SEG_SCAN_TILE,
                    "seq: hashed table needs 0 < item_rows, item_rows + num_items < 2^31 - %d", SEG_SCAN_TILE);
        SLB_REQUIRE(x->item_padding_idx == 0, "seq: a hashed item table's padding_idx must be 0 (PADDING_IDX)");
        if (training)
            SLB_REQUIRE(seq_hashed_terms(x) < (1ll << 31),
                        "seq: 2 * batch * seq_len * (item_hashes + 1) = %lld gradient terms, must stay below 2^31",
                        static_cast<long long>(seq_hashed_terms(x)));
    }
    if (training) {
        SLB_REQUIRE(x->negs && x->bias && x->loss_out, "seq: null pointer");
        SLB_REQUIRE(x->opt != SLB_OPT_NONE || (x->dE && x->dbias), "seq: dE / dbias needed without a fused optimizer");
        SLB_REQUIRE(x->opt == SLB_OPT_NONE || x->opt == SLB_OPT_SGD || (x->opt == SLB_OPT_ADAGRAD && x->state_E && x->state_bias) ||
                    x->opt == SLB_OPT_ADAM,
                    "seq: fused optimizer is SGD, Adagrad with state_E / state_bias, or Adam");
        if (x->opt == SLB_OPT_ADAM)
            SLB_REQUIRE(x->state_E && x->state_bias && x->state2_E && x->state2_bias && x->last_E &&
                        (x->item_hashes == 0 || x->last_bias) && x->adam_sched && x->adam_step >= 1 &&
                        x->adam_step < (1ll << 31),
                        "seq: fused Adam needs exp_avg / exp_avg_sq / last (last_bias on a hashed table), "
                        "the schedule and 1 <= adam_step < 2^31");
        SLB_REQUIRE(x->loss >= 0 && x->loss <= 3, "seq: bad loss kind");
        SLB_REQUIRE(x->n_neg >= 1 && (x->loss == SLB_LOSS_ADAPTIVE_HINGE || x->n_neg == 1), "seq: bad n_neg");
        if (x->n_layers > 0) SLB_REQUIRE(x->dconv_w && x->dconv_b, "seq: conv grads missing");
    }
    SLB_REQUIRE(x->workspace != nullptr, "seq: null workspace");
    return SLB_OK;
}

int sq_grid(int64_t groups_needed) { return min(slb_grid(groups_needed, 8), SQ_MAX_GRID); }

#define SQ_DISPATCH_NCH_T(D, KERNEL, BYPOS, grid, smem, stream, ...)                     \
    if ((D) <= 128) KERNEL<1, BYPOS><<<grid, SQ_THREADS, smem, stream>>>(__VA_ARGS__);   \
    else if ((D) <= 256) KERNEL<2, BYPOS><<<grid, SQ_THREADS, smem, stream>>>(__VA_ARGS__); \
    else KERNEL<4, BYPOS><<<grid, SQ_THREADS, smem, stream>>>(__VA_ARGS__);

#define SQ_DISPATCH_NCH(D, KERNEL, bypos, grid, smem, stream, ...)                       \
    if (bypos) { SQ_DISPATCH_NCH_T(D, KERNEL, true, grid, smem, stream, __VA_ARGS__) }   \
    else { SQ_DISPATCH_NCH_T(D, KERNEL, false, grid, smem, stream, __VA_ARGS__) }

// The item-table part of the device arguments: E, its shape and, on a hashed table, the hashes.
SeqDev seq_dev_table(const slb_seq_step_args* x) {
    SeqDev a = {};
    a.B = x->batch; a.S = x->seq_len; a.T = x->seq_len + 1; a.I = x->num_items; a.D = x->dim;
    a.seqs = x->seqs; a.E = x->E;
    a.H = x->item_hashes;
    a.Mrows = a.H ? x->item_rows : x->num_items;
    for (int k = 0; k < 24; ++k) a.seeds[k] = x->item_seeds[k];
    return a;
}

// X0 = the input rows of every position: E[seq], or the hashed sums
int launch_gather(const slb_seq_step_args* x, const SeqLayout& l, cudaStream_t st) {
    const int64_t n = x->batch * x->seq_len;
    const int lpr = lpr_for_dim(x->dim);
    const int grid = sq_grid((n + SQ_THREADS / lpr - 1) / (SQ_THREADS / lpr));
    if (x->item_hashes) {
        const SeqDev a = seq_dev_table(x);
        with_lpr(lpr, [&](auto L) { seq_gather_hashed_kernel<L><<<grid, SQ_THREADS, 0, st>>>(a, l.X0); });
        SLB_LAUNCH_CHECK("seq_gather_hashed_kernel");
    } else {
        with_lpr(lpr, [&](auto L) {
            seq_gather_kernel<L><<<grid, SQ_THREADS, 0, st>>>(x->E, x->seqs, n, x->dim, x->num_items, l.X0);
        });
        SLB_LAUNCH_CHECK("seq_gather_kernel");
    }
    return SLB_OK;
}

void conv_shifts(const slb_seq_step_args* x, int layer, int* shift, int* Tin) {
    const int k = x->kernel_width[layer], d = x->dilation[layer];
    const int rf = k + (k - 1) * (d - 1);
    const int pad = layer == 0 ? rf : rf - 1;       // representations.py:394-400 vs :414
    for (int j = 0; j < k; ++j) shift[j] = j * d - pad;
    *Tin = layer == 0 ? x->seq_len : x->seq_len + 1;
}

// One shifted-row conv GEMM (forward or input gradient): wgmma at D = 128 with W_nc ([j][n][c],
// the contraction index contiguous), mma.sync otherwise with W_cn ([j][c][n]).
int launch_conv_gemm(ConvGemm g, const float* W_nc, const float* W_cn, cudaStream_t st, const char* name) {
    const int64_t rows = g.B * g.Tout;
    if (use_tc(g.D)) {
        g.Wm = W_nc;
        if (tc_configure(tc::tc_conv_gemm_kernel) != 0) { slb_set_error("seq: cannot configure wgmma kernel"); return SLB_ECUDA; }
        tc::tc_conv_gemm_kernel<<<static_cast<unsigned>((rows + tc::TM - 1) / tc::TM), 128, tc::SMEM_BYTES, st>>>(g);
    } else {
        g.Wm = W_cn;
        dim3 grid(static_cast<unsigned>((rows + GM - 1) / GM), static_cast<unsigned>((g.D + GN - 1) / GN));
        conv_gemm_kernel<<<grid, 256, 0, st>>>(g);
    }
    SLB_LAUNCH_CHECK(name);
    return SLB_OK;
}

// One conv weight gradient: split over position slabs into w.part / w.bpart, then the
// fixed-order reduce into dW (D, D, k) and db (D).
int launch_conv_dw(ConvDw w, float* dW, float* db, cudaStream_t st) {
    const int64_t M = w.B * w.Tout;
    const bool tcp = use_tc(w.D);
    const int splits = tcp ? dw_splits_tc(M, w.k) : dw_splits(M, w.D, w.k);
    const int slab_q = tcp ? tc::KC : GK;
    w.slab = ((M + splits - 1) / splits + slab_q - 1) / slab_q * slab_q;
    if (tcp) {
        if (tc_configure(tc::tc_conv_dw_kernel) != 0) { slb_set_error("seq: cannot configure wgmma kernel"); return SLB_ECUDA; }
        dim3 wg(static_cast<unsigned>(w.k), static_cast<unsigned>(splits));
        tc::tc_conv_dw_kernel<<<wg, 128, tc::SMEM_BYTES, st>>>(w);
        SLB_LAUNCH_CHECK("tc_conv_dw_kernel");
    } else {
        dim3 wg(static_cast<unsigned>(((w.D + GM - 1) / GM) * ((w.D + GN - 1) / GN)), static_cast<unsigned>(w.k),
                static_cast<unsigned>(splits));
        conv_dw_kernel<<<wg, 256, 0, st>>>(w);
        SLB_LAUNCH_CHECK("conv_dw_kernel");
    }
    conv_dw_reduce_kernel<<<sq_grid((static_cast<int64_t>(w.k) * w.D * w.D + w.D + 255) / 256), 256, 0, st>>>(
        w.part, w.bpart, splits, w.k, w.D, dW, db);
    SLB_LAUNCH_CHECK("conv_dw_reduce_kernel");
    return SLB_OK;
}

// ------------------------------------------------------------------ LSTMNet host side
// Cluster size c of the recurrence kernels: W_hh (16 D^2 bytes) is split over c CTAs' shared memory.
int lstm_cluster_size(int D) { return D <= 64 ? 1 : (D <= 128 ? 4 : 8); }

lstm::LstmDev lstm_dev(const slb_seq_step_args* x, const SeqLayout& l, float* H) {
    lstm::LstmDev a = {};
    const int D = x->dim, c = lstm_cluster_size(D);
    a.B = x->batch; a.T = x->seq_len + 1; a.D = D;
    a.U = (D + c - 1) / c;
    const int nb = lstm::THREADS / a.U;              // one (sequence, unit) item per thread
    a.NB = nb > 32 ? 32 : nb;                        // U <= 64, so NB >= 4
    a.ntiles = static_cast<int>((a.B + a.NB - 1) / a.NB);
    a.w_hh = x->lstm_w_hh; a.b_ih = x->lstm_b_ih; a.b_hh = x->lstm_b_hh;
    a.G = l.G; a.Cs = l.Cs; a.H = H; a.dR = l.dR;
    return a;
}

// Launches a recurrence kernel on clusters of lstm_cluster_size(D) CTAs: as many clusters as
// can be resident at once, each walking the sequence tiles.  Refuses to launch when not even
// one cluster can be scheduled.
int lstm_launch(void (*kernel)(lstm::LstmDev), const lstm::LstmDev& a, size_t smem_floats, cudaStream_t st,
                const char* name) {
    const int c = lstm_cluster_size(a.D);
    const size_t smem = smem_floats * sizeof(float);
    SLB_REQUIRE(a.NB >= 1 && a.U * a.NB <= lstm::THREADS, "%s: a tile needs one thread per item", name);
    if (cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem)) != cudaSuccess) {
        cudaGetLastError();
        slb_set_error("%s: cannot configure %zu B of shared memory", name, smem);
        return SLB_ECUDA;
    }
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = c;
    attr[0].val.clusterDim.y = 1;
    attr[0].val.clusterDim.z = 1;
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(static_cast<unsigned>(c * a.ntiles));
    cfg.blockDim = dim3(lstm::THREADS);
    cfg.dynamicSmemBytes = smem;
    cfg.stream = st;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    int active = 0;
    if (cudaOccupancyMaxActiveClusters(&active, kernel, &cfg) != cudaSuccess || active < 1) {
        cudaGetLastError();
        slb_set_error("%s: a cluster of %d CTAs with %zu B of shared memory each cannot be scheduled", name, c, smem);
        return SLB_ECUDA;
    }
    cfg.gridDim = dim3(static_cast<unsigned>(c * (active < a.ntiles ? active : a.ntiles)));
    if (cudaLaunchKernelEx(&cfg, kernel, a) != cudaSuccess) {
        slb_set_error("%s: launch failed: %s", name, cudaGetErrorString(cudaGetLastError()));
        return SLB_ECUDA;
    }
    return SLB_OK;
}

// h_t for t = 0..S into H: gather, four projection GEMMs into G, the recurrence
int run_lstm_forward(const slb_seq_step_args* x, const SeqLayout& l, float* H, cudaStream_t st) {
    const int64_t B = x->batch;
    const int S = x->seq_len, T = S + 1, D = x->dim;
    const int64_t BTD = B * T * D, DD = static_cast<int64_t>(D) * D;
    const int grc = launch_gather(x, l, st);
    if (grc != SLB_OK) return grc;
    for (int g = 0; g < 4; ++g) {
        conv_wt_kernel<<<sq_grid((DD + 255) / 256), 256, 0, st>>>(x->lstm_w_ih + g * DD, 1, D, l.WT + g * DD, nullptr);
        SLB_LAUNCH_CHECK("conv_wt_kernel(lstm)");
        // x_t = E[seq_{t-1}], x_0 = 0: the layer-0 shift of -1 (representations.py:213-224)
        ConvGemm p = {};
        p.In = l.X0; p.Tin = S; p.Out = l.G + g * BTD; p.Tout = T; p.k = 1; p.shift[0] = -1;
        p.B = B; p.D = D; p.mode = 1;                     // pure GEMM: no bias, no activation
        const int rc = launch_conv_gemm(p, x->lstm_w_ih + g * DD, l.WT + g * DD, st, "conv_gemm(lstm projection)");
        if (rc != SLB_OK) return rc;
    }
    const lstm::LstmDev a = lstm_dev(x, l, H);
    return lstm_launch(lstm::lstm_fwd_kernel, a, lstm::fwd_smem_floats(D, a.U, a.NB), st, "lstm_fwd_kernel");
}

// BPTT from dR, then per gate block: dW_ih, dW_hh (+ both bias gradients) and the input
// gradient accumulated into the seq-role contribution rows C[b, s] (x_{s+1} = e_s).
int run_lstm_backward(const slb_seq_step_args* x, const SeqLayout& l, cudaStream_t st) {
    const int64_t B = x->batch;
    const int S = x->seq_len, T = S + 1, D = x->dim;
    const int64_t BTD = B * T * D, DD = static_cast<int64_t>(D) * D;
    const lstm::LstmDev a = lstm_dev(x, l, l.rep_pool);
    int rc = lstm_launch(lstm::lstm_bwd_kernel, a, lstm::bwd_smem_floats(D, a.U, a.NB), st, "lstm_bwd_kernel");
    if (rc != SLB_OK) return rc;
    for (int g = 0; g < 4; ++g) {
        ConvDw w = {};                                    // a_t reads x_t = X0[t - 1] and h_{t-1}
        w.dZ = l.G + g * BTD; w.Tout = T; w.k = 1; w.shift[0] = -1; w.B = B; w.D = D;
        w.part = l.part; w.bpart = l.bpart;
        w.In = l.X0; w.Tin = S;
        rc = launch_conv_dw(w, x->dlstm_w_ih + g * DD, x->dlstm_b_ih + g * D, st);
        if (rc != SLB_OK) return rc;
        w.In = l.rep_pool; w.Tin = T;
        rc = launch_conv_dw(w, x->dlstm_w_hh + g * DD, x->dlstm_b_hh + g * D, st);
        if (rc != SLB_OK) return rc;
        ConvGemm d = {};                                  // d e_s = d x_{s+1}
        d.In = l.G + g * BTD; d.Tin = T; d.Out = l.C; d.Tout = S; d.k = 1; d.shift[0] = 1;
        d.B = B; d.D = D; d.mode = 1; d.accumulate = 1;
        rc = launch_conv_gemm(d, l.WT + g * DD, x->lstm_w_ih + g * DD, st, "conv_gemm(lstm dx)");
        if (rc != SLB_OK) return rc;
    }
    return SLB_OK;
}

// ------------------------------------------------------------------ MixtureLSTMNet host side
// P_j = W_p[j] h + b_p[j] for the 2M projection blocks (representations.py:549-553): shift-0
// k = 1 conv GEMMs over the LSTM's h_t with the identity epilogue.
int run_mix_forward(const slb_seq_step_args* x, const SeqLayout& l, cudaStream_t st) {
    const int64_t B = x->batch;
    const int T = x->seq_len + 1, D = x->dim;
    const int64_t BTD = B * T * D, DD = static_cast<int64_t>(D) * D;
    for (int j = 0; j < 2 * x->num_mixtures; ++j) {
        conv_wt_kernel<<<sq_grid((DD + 255) / 256), 256, 0, st>>>(x->mix_w + j * DD, 1, D, l.WTm + j * DD, nullptr);
        SLB_LAUNCH_CHECK("conv_wt_kernel(mixture)");
        ConvGemm p = {};
        p.In = l.rep_pool; p.Tin = T; p.Out = l.P + j * BTD; p.Tout = T; p.k = 1; p.shift[0] = 0;
        p.B = B; p.D = D; p.mode = 0; p.bias = x->mix_b + j * D; p.nonlin = 2;
        const int rc = launch_conv_gemm(p, x->mix_w + j * DD, l.WTm + j * DD, st, "conv_gemm(mixture projection)");
        if (rc != SLB_OK) return rc;
    }
    return SLB_OK;
}

// From dP (in place of P): per block dW_p[j], db_p[j] and dh = sum_j W_p[j]^T dP_j into dR,
// accumulated in block order.
int run_mix_backward(const slb_seq_step_args* x, const SeqLayout& l, cudaStream_t st) {
    const int64_t B = x->batch;
    const int T = x->seq_len + 1, D = x->dim;
    const int64_t BTD = B * T * D, DD = static_cast<int64_t>(D) * D;
    for (int j = 0; j < 2 * x->num_mixtures; ++j) {
        ConvDw w = {};
        w.In = l.rep_pool; w.Tin = T; w.dZ = l.P + j * BTD; w.Tout = T; w.k = 1; w.shift[0] = 0;
        w.B = B; w.D = D; w.part = l.part; w.bpart = l.bpart;
        int rc = launch_conv_dw(w, x->dmix_w + j * DD, x->dmix_b + j * D, st);
        if (rc != SLB_OK) return rc;
        ConvGemm d = {};
        d.In = l.P + j * BTD; d.Tin = T; d.Out = l.dR; d.Tout = T; d.k = 1; d.shift[0] = 0;
        d.B = B; d.D = D; d.mode = 1; d.accumulate = j > 0;
        rc = launch_conv_gemm(d, l.WTm + j * DD, x->mix_w + j * DD, st, "conv_gemm(mixture dh)");
        if (rc != SLB_OK) return rc;
    }
    return SLB_OK;
}

// representation forward; returns pointer to the (B,T,D) result inside the workspace
int run_representation(const slb_seq_step_args* x, const SeqLayout& l, float* rep_dst, cudaStream_t st,
                       float** rep_out) {
    const int64_t B = x->batch;
    const int S = x->seq_len, T = S + 1, D = x->dim;
    if (x->lstm_w_ih && x->mix_w) {
        int rc = run_lstm_forward(x, l, l.rep_pool, st);     // h_t stays for the projection's backward
        if (rc == SLB_OK) rc = run_mix_forward(x, l, st);
        if (rc == SLB_OK && rep_dst) {
            const int J = 2 * x->num_mixtures;
            mix::mix_rep_kernel<<<sq_grid((B * T * J * D / 4 + 255) / 256), 256, 0, st>>>(l.P, B * T, D, J, rep_dst);
            SLB_LAUNCH_CHECK("mix_rep_kernel");
        }
        *rep_out = l.rep_pool;
        return rc;
    }
    if (x->lstm_w_ih) {
        float* H = rep_dst ? rep_dst : l.rep_pool;
        const int rc = run_lstm_forward(x, l, H, st);
        *rep_out = H;
        return rc;
    }
    if (x->n_layers == 0) {
        float* rep = rep_dst ? rep_dst : l.rep_pool;
        const size_t smem = static_cast<size_t>(16) * D * sizeof(float);
        const bool hashed = x->item_hashes != 0;
        if (hashed) {
            const int grc = launch_gather(x, l, st);
            if (grc != SLB_OK) return grc;
        }
        SQ_DISPATCH_NCH(D, pool_rep_kernel, hashed, static_cast<unsigned>(B), smem, st, hashed ? l.X0 : x->E,
                        x->seqs, S, D, x->num_items, rep);
        SLB_LAUNCH_CHECK("pool_rep_kernel");
        *rep_out = rep;
        return SLB_OK;
    }
    const int grc = launch_gather(x, l, st);
    if (grc != SLB_OK) return grc;
    for (int i = 0; i < x->n_layers; ++i) {
        const int k = x->kernel_width[i];
        conv_wt_kernel<<<sq_grid((static_cast<int64_t>(k) * D * D + 255) / 256), 256, 0, st>>>(
            x->conv_w[i], k, D, l.Wf[i], l.Wb[i]);
        SLB_LAUNCH_CHECK("conv_wt_kernel");
        ConvGemm g = {};
        conv_shifts(x, i, g.shift, &g.Tin);
        g.In = i == 0 ? l.X0 : l.Y[i - 1];
        const bool last = i == x->n_layers - 1;
        float* yout = (last && rep_dst) ? rep_dst : l.Y[i];
        g.Out = yout; g.Tout = T; g.Wm = l.Wf[i]; g.k = k; g.B = B; g.D = D; g.mode = 0;
        g.bias = x->conv_b[i]; g.nonlin = x->nonlinearity; g.Aout = l.A[i];
        if (x->residual) {
            g.Res = g.In; g.res_T = g.Tin; g.res_shift = i == 0 ? -1 : 0;   // representations.py:404-407, 419-420
        }
        if (!x->residual && !(last && rep_dst)) g.Out = l.A[i];
        if (use_tc(D)) SLB_REQUIRE(l.Wb[i] != nullptr, "seq: wgmma forward needs the [k][out][in] weight copy");
        // Wb = [j][n = out][c = in], Wf = [j][c = in][n = out]
        const int rc = launch_conv_gemm(g, l.Wb[i], l.Wf[i], st, "conv_gemm(fwd)");
        if (rc != SLB_OK) return rc;
        *rep_out = g.Out;
    }
    return SLB_OK;
}

}  // namespace

extern "C" {

size_t slb_seq_step_workspace_bytes(const slb_seq_step_args* x) {
    if (!x || x->batch <= 0 || x->seq_len <= 0 || x->dim <= 0) return 0;
    if (x->n_layers > 0 && !x->kernel_width) return 0;
    if (x->mix_w && (x->num_mixtures < 1 || x->num_mixtures > mix::MAX_M)) return 0;
    if (x->item_hashes > 0 && seq_hashed_terms(x) >= (1ll << 31)) return 0;      // the step rejects it
    return seq_layout(nullptr, x, x->negs != nullptr || x->loss_out != nullptr).bytes;
}

int slb_seq_representation(const slb_seq_step_args* x, float* rep_out, slb_stream_t stream) {
    int rc = seq_validate(x, false);
    if (rc != SLB_OK) return rc;
    SLB_REQUIRE(rep_out != nullptr, "seq_representation: null output");
    SeqLayout l = seq_layout(x->workspace, x, x->negs != nullptr || x->loss_out != nullptr);
    if (x->workspace_bytes < l.bytes) { slb_set_error("seq_representation: workspace too small"); return SLB_ENOSPC; }
    float* rep = nullptr;
    return run_representation(x, l, rep_out, static_cast<cudaStream_t>(stream), &rep);
}

int slb_seq_train_step(const slb_seq_step_args* x, slb_stream_t stream) {
    int rc = seq_validate(x, true);
    if (rc != SLB_OK) return rc;
    SeqLayout l = seq_layout(x->workspace, x, true);
    if (x->workspace_bytes < l.bytes) {
        slb_set_error("seq_train_step: workspace too small (%zu < %zu)", x->workspace_bytes, l.bytes);
        return SLB_ENOSPC;
    }
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const int64_t B = x->batch;
    const int S = x->seq_len, T = S + 1, D = x->dim;
    const int lpr = lpr_for_dim(D);
    const int groups = SQ_THREADS / lpr;
    if (cudaMemsetAsync(l.hdr, 0, 16 * sizeof(int32_t), st) != cudaSuccess) {
        slb_set_error("seq_train_step: memset failed");
        return SLB_ECUDA;
    }
    seq_mask_kernel<<<sq_grid((B * S + 255) / 256), 256, 0, st>>>(
        x->seqs, x->negs, B * S, static_cast<int64_t>(x->n_neg) * B * S, x->num_items, l.hdr);
    SLB_LAUNCH_CHECK("seq_mask_kernel");

    const bool hashed = x->item_hashes != 0;
    SeqDev a = seq_dev_table(x);
    a.negs = x->negs; a.loss = x->loss; a.n_neg = x->n_neg; a.Xs = l.X0;
    a.bias = x->bias;
    const bool adam = x->opt == SLB_OPT_ADAM;
    if (adam) {
        a.ad = {x->beta1, x->beta2, x->one_minus_beta1, x->one_minus_beta2, x->eps, x->weight_decay, x->adam_sched,
                static_cast<int32_t>(x->adam_step)};
        a.sE = x->state_E; a.sbias = x->state_bias; a.vE = x->state2_E; a.vbias = x->state2_bias;
        a.lastE = x->last_E; a.lastb = hashed ? x->last_bias : x->last_E;
        if (x->adam_step > 1) {
            const int64_t work = B * S * (1 + x->n_neg) * (hashed ? x->item_hashes + 1 : 1);
            with_bool(hashed, [&](auto H) {
                with_lpr(lpr, [&](auto L) {
                    seq_adam_prepass_kernel<L, H><<<sq_grid((work + groups - 1) / groups), SQ_THREADS, 0, st>>>(a);
                });
            });
            SLB_LAUNCH_CHECK("seq_adam_prepass_kernel");
        }
    }
    float* rep = nullptr;
    rc = run_representation(x, l, nullptr, st, &rep);
    if (rc != SLB_OK) return rc;
    a.rep = rep; a.dR = l.dR; a.C = l.C; a.keys = l.keys; a.gs = l.gs;
    a.hdr = l.hdr; a.partial = l.partial; a.norm = x->norm_count;
    a.loss_out = x->loss_out; a.pos_out = x->pos_out; a.neg_out = x->neg_out;
    a.dE = x->dE; a.dbias = x->dbias; a.seg = l.seg;
    // hashed rows are hot at small item_rows: sort their member lists with seg_sort_long_kernel
    if (hashed) a.seg.long_cap = seg_sort_cap(lpr);
    a.opt = x->opt; a.lr = x->lr; a.wd = x->weight_decay; a.eps = x->eps;
    if (!adam) { a.sE = x->state_E; a.sbias = x->state_bias; }
    const int score_grid = sq_grid((B * T + groups - 1) / groups);
    if (x->mix_w) {
        a.M = x->num_mixtures; a.P = l.P;
        with_bool(hashed, [&](auto H) {
            with_lpr(lpr, [&](auto L) { mix::mix_score_kernel<L, H><<<score_grid, SQ_THREADS, 0, st>>>(a); });
        });
        SLB_LAUNCH_CHECK("mix_score_kernel");
        rc = run_mix_backward(x, l, st);
        if (rc != SLB_OK) return rc;
    } else {
        with_bool(hashed, [&](auto H) {
            with_lpr(lpr, [&](auto L) { seq_score_kernel<L, H><<<score_grid, SQ_THREADS, 0, st>>>(a); });
        });
        SLB_LAUNCH_CHECK("seq_score_kernel");
    }

    if (x->lstm_w_ih) {
        rc = run_lstm_backward(x, l, st);
        if (rc != SLB_OK) return rc;
    } else if (x->n_layers == 0) {
        const size_t smem = static_cast<size_t>(16) * D * sizeof(float);
        SQ_DISPATCH_NCH(D, pool_bwd_kernel, hashed, static_cast<unsigned>(B), smem, st, hashed ? l.X0 : x->E,
                        x->seqs, S, D, x->num_items, l.dR, l.C);
        SLB_LAUNCH_CHECK("pool_bwd_kernel");
    } else {
        const float* dY = l.dR;
        float* ping = l.dYa;
        float* pong = l.dYb;
        const int64_t n4 = B * T * D / 4;
        for (int i = x->n_layers - 1; i >= 0; --i) {
            const int k = x->kernel_width[i];
            conv_dz_kernel<<<sq_grid((n4 + 255) / 256), 256, 0, st>>>(dY, l.A[i], n4, x->nonlinearity, l.dZ);
            SLB_LAUNCH_CHECK("conv_dz_kernel");
            ConvDw w = {};
            conv_shifts(x, i, w.shift, &w.Tin);
            w.In = i == 0 ? l.X0 : l.Y[i - 1];
            w.dZ = l.dZ; w.Tout = T; w.k = k; w.B = B; w.D = D;
            w.part = l.part; w.bpart = l.bpart;
            rc = launch_conv_dw(w, x->dconv_w[i], x->dconv_b[i], st);
            if (rc != SLB_OK) return rc;
            // input gradient: shifted GEMM over dZ with the transposed weights
            ConvGemm g = {};
            int fshift[16], Tin;
            conv_shifts(x, i, fshift, &Tin);
            for (int j = 0; j < k; ++j) g.shift[j] = -fshift[j];
            g.In = l.dZ; g.Tin = T; g.Tout = Tin; g.k = k; g.B = B; g.D = D; g.mode = 1;
            if (x->residual) { g.Res = dY; g.res_T = T; g.res_shift = i == 0 ? 1 : 0; }
            if (i == 0) { g.Out = l.C; g.accumulate = 1; }      // seq-role rows C[b, s] += d e_s
            else { g.Out = ping; }
            // Wf = [j][n = in][c = out], Wb = [j][c = out][n = in]
            rc = launch_conv_gemm(g, l.Wf[i], l.Wb[i], st, "conv_gemm(dx)");
            if (rc != SLB_OK) return rc;
            if (i > 0) { dY = ping; float* tmp = ping; ping = pong; pong = tmp; }
        }
    }
    seg_scan_launch(a.seg, a.seg.Rpad, st);
    SLB_LAUNCH_CHECK("seg_scan_kernel");
    const int64_t nkeys = 2 * B * S * (a.H + 1);
    seq_fill_kernel<<<sq_grid((nkeys + 255) / 256), 256, 0, st>>>(a);
    SLB_LAUNCH_CHECK("seq_fill_kernel");
    if (hashed) {
        seg_sort_long_kernel<<<SEG_LONG_CTAS, 256, 0, st>>>(a.seg);     // no-op unless hot rows exist
        SLB_LAUNCH_CHECK("seg_sort_long_kernel");
    }
    const int reduce_grid = sq_grid((nkeys + groups - 1) / groups);
    with_bool(hashed, [&](auto H) {
        with_lpr(lpr, [&](auto L) {
            if (adam) seq_reduce_adam_kernel<L, H><<<reduce_grid, SQ_THREADS, 0, st>>>(a);
            else seq_reduce_kernel<L, H><<<reduce_grid, SQ_THREADS, 0, st>>>(a);
        });
    });
    SLB_LAUNCH_CHECK("seq_reduce_kernel");
    return SLB_OK;
}

}  // extern "C"
