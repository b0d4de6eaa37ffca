// MixtureLSTMNet head (representations.py:517-596) for the sequence step.  Included by seq.cu
// after the LSTM.  The net is the LSTM of seq_lstm.cuh, a k = 1 projection of h_t to 2M blocks
// of D channels (2M shift-0 conv GEMMs with the identity epilogue, bias included), and a
// mixture-of-tastes score for every item e with bias beta:
//
//   c_m = P[m], v_m = P[M + m]  (m < M)        components and mixture vectors of a position
//   a_m = v_m . e,  w = softmax(a),  z_m = c_m . e,  s = beta + sum_m w_m z_m
//
// and, with g = d loss / d s (masked, normalised),
//
//   dc_m = g w_m e,  dv_m = g w_m (z_m - s_bar) e,  de = g sum_m w_m (c_m + (z_m - s_bar) v_m).
//
// mix_score_kernel mirrors seq_score_kernel's bookkeeping: one lane group per position, the
// loss of pair_loss folded by seq_loss_fold, pos_out / neg_out, the contribution rows C (now
// de of the target and of the credited negative), keys, gs and the row counts.  Instead of
// d loss / d r it writes d loss / d P over P in place: each position's group reads its own 2M
// rows before it overwrites them.  The row t = S is zeroed (the final step is not trained on).
#pragma once

namespace mix {

constexpr int MAX_M = 8;         // logits and scores of a position stay in registers

// Scores one item row against the position whose 2M rows start at p (row j at p + j * BTD):
// returns beta + s_bar and leaves the softmax weights w, the taste scores z and s_bar.  e(c) is
// the row's float4 at channel c (the row source: a table row, or a hashed item's summed rows).
template <int LPR, typename Row>
__device__ __forceinline__ float mix_item(const float* p, int64_t BTD, int M, int D, Row e,
                                          float beta, int gl, unsigned gmask, float (&w)[MAX_M], float (&z)[MAX_M],
                                          float& sbar) {
    float av[MAX_M];
#pragma unroll
    for (int m = 0; m < MAX_M; ++m) { av[m] = 0.f; z[m] = 0.f; }
    for (int c = gl * 4; c < D; c += LPR * 4) {
        const float4 ev = e(c);
#pragma unroll
        for (int m = 0; m < MAX_M; ++m)
            if (m < M) {
                z[m] += dot4(ld4(p + m * BTD + c), ev);
                av[m] += dot4(ld4(p + (M + m) * BTD + c), ev);
            }
    }
    float amax = -INFINITY;
#pragma unroll
    for (int m = 0; m < MAX_M; ++m)
        if (m < M) {
            z[m] = group_sum<LPR>(z[m], gmask);
            av[m] = group_sum<LPR>(av[m], gmask);
            amax = fmaxf(amax, av[m]);
        }
    float den = 0.f;                                  // softmax with max subtraction, as F.softmax
#pragma unroll
    for (int m = 0; m < MAX_M; ++m) {
        w[m] = m < M ? expf(av[m] - amax) : 0.f;
        den += w[m];
    }
    sbar = 0.f;
#pragma unroll
    for (int m = 0; m < MAX_M; ++m) {
        w[m] = w[m] / den;
        sbar += w[m] * z[m];                          // z = 0 beyond M
    }
    return beta + sbar;
}

template <int LPR, bool HASHED>
__global__ void __launch_bounds__(SQ_THREADS) mix_score_kernel(SeqDev a) {
    constexpr int GROUPS = SQ_THREADS / LPR;
    if (HASHED && blockIdx.x == 0 && threadIdx.x == 0) a.seg.totals[3] = 0;   // hot-row list of this step
    const int gl = threadIdx.x & (LPR - 1);
    const unsigned gmask = group_mask(LPR);
    const int D = a.D, S = a.S, T = a.T, M = a.M;
    const int64_t BS = a.B * S, BT = a.B * T, BTD = BT * D;
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
        float* prow = a.P + mm * D;                   // row j of the position: prow + j * BTD
        if (t == S) {                                 // final step is not trained on
            if (valid)
                for (int j = 0; j < 2 * M; ++j)
                    for (int c = gl * 4; c < D; c += LPR * 4) st4(prow + j * BTD + c, make_float4(0, 0, 0, 0));
            continue;                                 // group-uniform
        }
        const int64_t pidx = b * S + t;
        const int64_t id = clamp_id(a.seqs[pidx], a.I);
        // the target is the input item of position t: its summed row is Xs[b, t] on a hashed table
        const float* et = HASHED ? a.Xs + pidx * D : a.E + id * D;
        float wt[MAX_M], zt[MAX_M], st;
        const float p = mix_item<LPR>(prow, BTD, M, D, [&](int c) { return ldg4(et + c); }, __ldg(a.bias + id), gl,
                                      gmask, wt, zt, st);
        float nbest = -INFINITY, sn = 0.f;
        float wn[MAX_M], zn[MAX_M];
        int64_t nid = 0;
        for (int k = 0; k < a.n_neg; ++k) {
            const int64_t nidx = (static_cast<int64_t>(k) * a.B + b) * S + t;   // implicit.py:281-286
            const int64_t j = clamp_id(a.negs[nidx], a.I);
            float wk[MAX_M], zk[MAX_M], sk;
            const float nk = mix_item<LPR>(prow, BTD, M, D, [&](int c) { return item4<HASHED>(a, j, c); },
                                           __ldg(a.bias + j), gl, gmask, wk, zk, sk);
            if (valid && gl == 0 && a.neg_out) a.neg_out[nidx] = nk;
            if (k == 0 || nk > nbest) {               // the first of bit-identical maxima
                nbest = nk; nid = j; sn = sk;
#pragma unroll
                for (int q = 0; q < MAX_M; ++q) { wn[q] = wk[q]; zn[q] = zk[q]; }
            }
        }
        float per, gp, gn;
        pair_loss(a.loss, p, nbest, per, gp, gn);
        const float mk = id != 0 ? 1.0f : 0.0f;       // mask = seq != PADDING_IDX
        lsum += (valid && gl == 0) ? per * mk : 0.f;
        gp *= mk * inv; gn *= mk * inv;
        if (!valid) continue;                         // no shuffles below
        float* cs = a.C + pidx * D;
        float* cn = a.C + (BS + pidx) * D;
        for (int c = gl * 4; c < D; c += LPR * 4) {
            const float4 ev = ldg4(et + c), nv = item4<HASHED>(a, nid, c);
            float4 dt = make_float4(0, 0, 0, 0), dn = make_float4(0, 0, 0, 0);
#pragma unroll
            for (int q = 0; q < MAX_M; ++q)
                if (q < M) {
                    float* pc = prow + q * BTD + c;
                    float* pv = prow + (M + q) * BTD + c;
                    const float4 cv = ld4(pc), vv = ld4(pv);
                    const float ct = gp * wt[q], ut = ct * (zt[q] - st);
                    const float cq = gn * wn[q], uq = cq * (zn[q] - sn);
                    fma4(dt, ct, cv); fma4(dt, ut, vv);
                    fma4(dn, cq, cv); fma4(dn, uq, vv);
                    st4(pc, make_float4(ct * ev.x + cq * nv.x, ct * ev.y + cq * nv.y,
                                        ct * ev.z + cq * nv.z, ct * ev.w + cq * nv.w));
                    st4(pv, make_float4(ut * ev.x + uq * nv.x, ut * ev.y + uq * nv.y,
                                        ut * ev.z + uq * nv.z, ut * ev.w + uq * nv.w));
                }
            st4(cs + c, dt);
            st4(cn + c, dn);
        }
        if (gl == 0) {
            if (a.pos_out) a.pos_out[pidx] = p;
            a.gs[pidx] = gp; a.gs[BS + pidx] = gn;
            // rows of the padding id are frozen (padding_idx=0): drop their terms
            seq_keys<HASHED>(a, BS, pidx, id, nid, gn);
        }
    }
    seq_loss_fold(a, lsum, msum);
}

// rep[b, t, j * D + d] = P_j[b, t, d]: the (B, T, 2MD) time-major representation (the reference's
// (B, 2M, D, T) view, transposed)
__global__ void __launch_bounds__(256)
mix_rep_kernel(const float* __restrict__ P, int64_t BT, int D, int J, float* __restrict__ rep) {
    const int64_t JD = static_cast<int64_t>(J) * D;
    const int64_t n4 = BT * JD / 4;
    const int64_t nth = static_cast<int64_t>(gridDim.x) * blockDim.x;
    for (int64_t e = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; e < n4; e += nth) {
        const int64_t q = 4 * e;
        const int64_t row = q / JD;
        const int64_t rem = q - row * JD;
        const int j = static_cast<int>(rem / D);
        const int d = static_cast<int>(rem - static_cast<int64_t>(j) * D);
        st4(rep + q, ld4(P + (j * BT + row) * D + d));
    }
}

}  // namespace mix
