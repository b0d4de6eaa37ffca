// LSTMNet recurrence (representations.py:147-258) for the sequence step.  Included by seq.cu
// after the conv GEMMs, which carry the rest of the layer: the input projection
// W_ih x_t (four k = 1 shifted-row GEMMs, one per gate block, shift -1 so x_0 = 0), the
// weight gradients dW_ih / dW_hh and the input gradient.  What is left is sequential:
//
//   a_t = Gx_t + b_ih + b_hh + W_hh h_{t-1}          (4D rows, gate order i, f, g, o)
//   c_t = f * c_{t-1} + i * g,  h_t = o * tanh(c_t),  h_{-1} = c_{-1} = 0
//
// and its backpropagation through time.  Padding is not masked inside the recurrence.
//
// Both kernels run on a thread-block cluster of c CTAs that owns a tile of NB sequences.
// CTA r owns hidden units [r*U, r*U + nu) and their four gate rows of W_hh, which stay in
// its shared memory for the whole launch (16 U D bytes: 64 KB at D = 64, c = 1; 64 KB at
// D = 128, c = 4; 128 KB at D = 256, c = 8).  The clusters are persistent: each walks the
// sequence tiles with a stride of the cluster count, and a tail tile is masked, never
// skipped, so every CTA passes every cluster barrier.
//
//   lstm_fwd_kernel  per step, one item = (sequence, own unit): the four gate dots with
//                    h_{t-1}, the activations and the cell update; h_t is pushed into the
//                    h buffer of every CTA of the cluster (distributed shared memory,
//                    double-buffered) and a cluster barrier ends the step.  Writes h_t to
//                    the (B, T, D) representation, c_t, and the gate activations in place
//                    of Gx.
//   lstm_bwd_kernel  reverse time.  dh_t = dR_t + W_hh^T dgates_{t+1}: every CTA forms the
//                    partial product of its own gate rows for all D units, and the owner of
//                    a unit sums the c partials in rank order.  The gate derivatives
//                    overwrite the activations (gate-major dgates (4, B, T, D)).
// Arithmetic is fp32 FMA with expf / tanhf; there are no atomics, every sum has a fixed order.
#pragma once

#include <cooperative_groups.h>

namespace lstm {

namespace cg = cooperative_groups;

constexpr int THREADS = 256;

struct LstmDev {
    int64_t B; int T; int D;
    int U; int NB; int ntiles;    // units per CTA, sequences per tile (U * NB <= THREADS), tiles
    const float* w_hh;            // (4D, D)
    const float* b_ih; const float* b_hh;
    float* G;                     // (4, B, T, D): W_ih x_t in, gate activations out (fwd);
                                  // activations in, gate derivatives out (bwd)
    float* Cs;                    // (B, T, D) c_t
    float* H;                     // (B, T, D) h_t
    const float* dR;              // (B, T, D) d loss / d h_t from the scoring (bwd)
};

// shared-memory floats of each kernel (host and device)
__host__ __device__ inline size_t fwd_smem_floats(int D, int U, int NB) {
    return static_cast<size_t>(4) * U * D + 4 * U + 2 * static_cast<size_t>(NB) * (D + 4);
}
__host__ __device__ inline size_t bwd_smem_floats(int D, int U, int NB) {
    return static_cast<size_t>(4) * U * D + 4 * static_cast<size_t>(NB) * U + 2 * static_cast<size_t>(NB) * D;
}

// Thread tid owns the item (sequence s = tid / U of the tile, unit j = tid % U) for the whole
// tile, so c_{t-1} (fwd) and dc_{t+1} f_{t+1} (bwd) stay in registers, and the item's global
// inputs of the next step are loaded before the cluster barrier that ends the current one.
__global__ void __launch_bounds__(THREADS) lstm_fwd_kernel(LstmDev a) {
    cg::cluster_group cluster = cg::this_cluster();
    extern __shared__ __align__(16) float lsm[];
    const int D = a.D, U = a.U, NB = a.NB, T = a.T;
    const int HS = D + 4;                                 // h row stride (16 B aligned, staggers banks)
    const int c = static_cast<int>(cluster.num_blocks());
    const int r = static_cast<int>(cluster.block_rank());
    const int u0 = r * U;
    const int nu = min(U, D - u0);
    const int tid = threadIdx.x;
    const int64_t BTD = a.B * T * D;
    float4* W4 = reinterpret_cast<float4*>(lsm);          // [D][U]: W4[k*U + j] = W_hh[g*D + u0 + j][k], g = 0..3
    float4* bs4 = W4 + static_cast<size_t>(U) * D;        // [U] b_ih + b_hh
    float* hbuf = reinterpret_cast<float*>(bs4 + U);      // [2][NB][HS]

    for (int e = tid; e < U * D; e += THREADS) {
        const int j = e % U, k = e / U;
        float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
        if (j < nu) {
            const float* w = a.w_hh + static_cast<int64_t>(u0 + j) * D + k;
            v = make_float4(w[0], w[static_cast<int64_t>(D) * D], w[2 * static_cast<int64_t>(D) * D],
                            w[3 * static_cast<int64_t>(D) * D]);
        }
        W4[e] = v;
    }
    for (int j = tid; j < U; j += THREADS) {
        float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
        if (j < nu) {
            const int u = u0 + j;
            v = make_float4(a.b_ih[u] + a.b_hh[u], a.b_ih[D + u] + a.b_hh[D + u],
                            a.b_ih[2 * D + u] + a.b_hh[2 * D + u], a.b_ih[3 * D + u] + a.b_hh[3 * D + u]);
        }
        bs4[j] = v;
    }
    const int j = tid % U, s = tid / U;
    const int u = u0 + j;
    const int ncl = static_cast<int>(gridDim.x) / c;
    for (int tile = static_cast<int>(blockIdx.x) / c; tile < a.ntiles; tile += ncl) {
        const int64_t b = static_cast<int64_t>(tile) * NB + s;
        const bool live = s < NB && j < nu && b < a.B;   // masked items compute nothing
        const int64_t p0 = (b * T) * D + u;               // position t is p0 + t * D
        for (int e = tid; e < NB * HS; e += THREADS) hbuf[e] = 0.f;      // h_{-1} (buffer 0)
        float cprev = 0.f;
        float4 gx = make_float4(0.f, 0.f, 0.f, 0.f);
        if (live) gx = make_float4(a.G[p0], a.G[p0 + BTD], a.G[p0 + 2 * BTD], a.G[p0 + 3 * BTD]);
        cluster.sync();              // the previous tile's last pushes have landed; h_{-1} is zero
        for (int t = 0; t < T; ++t) {
            const float* hcur = hbuf + (t & 1) * NB * HS;
            const int nxt = ((t + 1) & 1) * NB * HS;
            const int64_t p = p0 + static_cast<int64_t>(t) * D;
            if (live) {
                const float* hr = hcur + s * HS;
                float4 acc = bs4[j];
                for (int k = 0; k < D; k += 4) {
                    const float4 h4 = ld4(hr + k);
                    fma4(acc, h4.x, W4[(k + 0) * U + j]);
                    fma4(acc, h4.y, W4[(k + 1) * U + j]);
                    fma4(acc, h4.z, W4[(k + 2) * U + j]);
                    fma4(acc, h4.w, W4[(k + 3) * U + j]);
                }
                const float gi = sigmoidf_(acc.x + gx.x);
                const float gf = sigmoidf_(acc.y + gx.y);
                const float gg = tanhf(acc.z + gx.z);
                const float go = sigmoidf_(acc.w + gx.w);
                const float cc = gf * cprev + gi * gg;
                const float h = go * tanhf(cc);
                cprev = cc;
                float* gp = a.G + p;
                gp[0] = gi; gp[BTD] = gf; gp[2 * BTD] = gg; gp[3 * BTD] = go;
                a.Cs[p] = cc;
                a.H[p] = h;
                for (int q = 0; q < c; ++q) cluster.map_shared_rank(hbuf, q)[nxt + s * HS + u] = h;
                if (t + 1 < T) gx = make_float4(gp[D], gp[BTD + D], gp[2 * BTD + D], gp[3 * BTD + D]);
            }
            cluster.sync();          // h_t complete in every CTA; h_{t-1} may be overwritten
        }
    }
}

__global__ void __launch_bounds__(THREADS) lstm_bwd_kernel(LstmDev a) {
    cg::cluster_group cluster = cg::this_cluster();
    extern __shared__ __align__(16) float lsm[];
    const int D = a.D, U = a.U, NB = a.NB, T = a.T;
    const int c = static_cast<int>(cluster.num_blocks());
    const int r = static_cast<int>(cluster.block_rank());
    const int u0 = r * U;
    const int nu = min(U, D - u0);
    const int tid = threadIdx.x;
    const int64_t BTD = a.B * T * D;
    float4* W4 = reinterpret_cast<float4*>(lsm);          // [U][D]: W4[j*D + k] = W_hh[g*D + u0 + j][k], g = 0..3
    float4* dg4 = W4 + static_cast<size_t>(U) * D;        // [NB][U] dgates_t of the own units
    float* pbuf = reinterpret_cast<float*>(dg4 + NB * U); // [2][NB][D] partial W_hh^T dgates (own rows)

    for (int e = tid; e < U * D; e += THREADS) {
        const int j = e / D, k = e % D;
        float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
        if (j < nu) {
            const float* w = a.w_hh + static_cast<int64_t>(u0 + j) * D + k;
            v = make_float4(w[0], w[static_cast<int64_t>(D) * D], w[2 * static_cast<int64_t>(D) * D],
                            w[3 * static_cast<int64_t>(D) * D]);
        }
        W4[e] = v;
    }
    const int j = tid % U, s = tid / U;
    const int u = u0 + j;
    const int ncl = static_cast<int>(gridDim.x) / c;
    for (int tile = static_cast<int>(blockIdx.x) / c; tile < a.ntiles; tile += ncl) {
        const int64_t b = static_cast<int64_t>(tile) * NB + s;
        const bool live = s < NB && j < nu && b < a.B;
        const int64_t p0 = (b * T) * D + u;
        if (s < NB) dg4[tid] = make_float4(0.f, 0.f, 0.f, 0.f);   // masked items stay zero
        float dcf = 0.f;                                  // dc_{t+1} * f_{t+1}
        // inputs of step T - 1: d loss / d h, the gate activations, c_t and c_{t-1}
        float dr = 0.f, cc = 0.f, cprev = 0.f;
        float4 act = make_float4(0.f, 0.f, 0.f, 0.f);
        if (live) {
            const int64_t p = p0 + static_cast<int64_t>(T - 1) * D;
            dr = a.dR[p];
            act = make_float4(a.G[p], a.G[p + BTD], a.G[p + 2 * BTD], a.G[p + 3 * BTD]);
            cc = a.Cs[p];
            cprev = T > 1 ? a.Cs[p - D] : 0.f;
        }
        cluster.sync();              // no CTA still reads the previous tile's partials
        for (int t = T - 1; t >= 0; --t) {
            const int pin = ((t + 1) & 1) * NB * D;          // partials of dgates_{t+1}
            if (live) {
                const int64_t p = p0 + static_cast<int64_t>(t) * D;
                float dh = dr;
                if (t + 1 < T)
                    for (int q = 0; q < c; ++q) dh += cluster.map_shared_rank(pbuf, q)[pin + s * D + u];
                const float gi = act.x, gf = act.y, gg = act.z, go = act.w;
                const float tc = tanhf(cc);
                const float dc = dh * go * (1.f - tc * tc) + dcf;
                const float4 d = make_float4(dc * gg * gi * (1.f - gi), dc * cprev * gf * (1.f - gf),
                                             dc * gi * (1.f - gg * gg), dh * tc * go * (1.f - go));
                dcf = dc * gf;
                float* gp = a.G + p;
                gp[0] = d.x; gp[BTD] = d.y; gp[2 * BTD] = d.z; gp[3 * BTD] = d.w;
                dg4[tid] = d;
                if (t > 0) {                                 // step t - 1's inputs, in flight below
                    dr = a.dR[p - D];
                    act = make_float4(gp[-D], gp[BTD - D], gp[2 * BTD - D], gp[3 * BTD - D]);
                    cc = cprev;
                    cprev = t > 1 ? a.Cs[p - 2 * D] : 0.f;
                }
            }
            __syncthreads();
            if (t > 0) {                                     // dgates_0 feeds no earlier step
                float* pout = pbuf + (t & 1) * NB * D;
                for (int it = tid; it < D * NB; it += THREADS) {
                    const int k = it % D, sq = it / D;
                    const float4* dgs = dg4 + sq * U;
                    float acc = 0.f;
                    for (int jj = 0; jj < U; ++jj) {
                        const float4 w = W4[jj * D + k], dv = dgs[jj];
                        acc = fmaf(w.x, dv.x, acc);
                        acc = fmaf(w.y, dv.y, acc);
                        acc = fmaf(w.z, dv.z, acc);
                        acc = fmaf(w.w, dv.w, acc);
                    }
                    pout[it] = acc;
                }
            }
            cluster.sync();          // partials of dgates_t visible to the cluster
        }
    }
}

}  // namespace lstm
