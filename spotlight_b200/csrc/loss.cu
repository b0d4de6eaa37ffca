// Standalone implicit-feedback losses (generic / custom-representation path).
// Replaces spotlight/losses.py:18-166: pointwise, bpr, hinge, adaptive hinge,
// each with the optional mask (masked mean = sum(loss*mask)/mask.sum()).
#include "common.cuh"

namespace {

constexpr int L_THREADS = 256;
constexpr int L_MAX_GRID = 132 * 8;

__device__ __forceinline__ float pick_neg(int loss, const float* __restrict__ neg, int64_t i,
                                          int64_t n, int n_neg, int& kstar) {
    kstar = 0;
    if (loss != SLB_LOSS_ADAPTIVE_HINGE) return neg[i];
    float best = neg[i];
    for (int k = 1; k < n_neg; ++k) {
        const float v = neg[static_cast<int64_t>(k) * n + i];
        if (v > best) { best = v; kstar = k; }   // first arg-max (torch.max on CPU)
    }
    return best;
}

// partial[2*b] = sum loss*m, partial[2*b+1] = sum m ; last block folds them in
// a fixed order into sums[0..1] and writes loss_out.
__global__ void __launch_bounds__(L_THREADS)
loss_reduce_kernel(int loss, const float* __restrict__ pos, const float* __restrict__ neg,
                   const uint8_t* __restrict__ mask, int64_t n, int n_neg, float* partial,
                   int32_t* done, float* sums, float* loss_out) {
    __shared__ float red[L_THREADS / 32];
    __shared__ bool is_last;
    float ls = 0.f, ms = 0.f;
    for (int64_t i = static_cast<int64_t>(blockIdx.x) * L_THREADS + threadIdx.x; i < n;
         i += static_cast<int64_t>(gridDim.x) * L_THREADS) {
        int ks;
        const float nv = pick_neg(loss, neg, i, n, n_neg, ks);
        float per, gp, gn;
        pair_loss(loss, pos[i], nv, per, gp, gn);
        const float m = mask ? (mask[i] ? 1.0f : 0.0f) : 1.0f;
        ls += per * m; ms += m;
    }
    const float bl = block_sum<L_THREADS>(ls, red);
    __syncthreads();
    const float bm = block_sum<L_THREADS>(ms, red);
    if (threadIdx.x == 0) {
        partial[2 * blockIdx.x] = bl;
        partial[2 * blockIdx.x + 1] = bm;
        __threadfence();
        is_last = atomicAdd(done, 1) == static_cast<int>(gridDim.x) - 1;
    }
    __syncthreads();
    if (is_last && threadIdx.x < 32) {
        __threadfence();
        float a = 0.f, b = 0.f;
        for (int k = threadIdx.x; k < static_cast<int>(gridDim.x); k += 32) {
            a += *reinterpret_cast<volatile float*>(partial + 2 * k);
            b += *reinterpret_cast<volatile float*>(partial + 2 * k + 1);
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            a += __shfl_down_sync(0xffffffffu, a, o);
            b += __shfl_down_sync(0xffffffffu, b, o);
        }
        if (threadIdx.x == 0) { sums[0] = a; sums[1] = b; *loss_out = a / b; *done = 0; }
    }
}

__global__ void __launch_bounds__(L_THREADS)
loss_grad_kernel(int loss, const float* __restrict__ pos, const float* __restrict__ neg,
                 const uint8_t* __restrict__ mask, int64_t n, int n_neg, const float* sums,
                 float* __restrict__ gpos, float* __restrict__ gneg) {
    const float inv = 1.0f / sums[1];
    for (int64_t i = static_cast<int64_t>(blockIdx.x) * L_THREADS + threadIdx.x; i < n;
         i += static_cast<int64_t>(gridDim.x) * L_THREADS) {
        int ks;
        const float nv = pick_neg(loss, neg, i, n, n_neg, ks);
        float per, gp, gn;
        pair_loss(loss, pos[i], nv, per, gp, gn);
        const float w = (mask ? (mask[i] ? 1.0f : 0.0f) : 1.0f) * inv;
        gpos[i] = gp * w;
        if (loss == SLB_LOSS_ADAPTIVE_HINGE) {
            for (int k = 0; k < n_neg; ++k) gneg[static_cast<int64_t>(k) * n + i] = k == ks ? gn * w : 0.f;
        } else {
            gneg[i] = gn * w;
        }
    }
}

// Rating losses on the prediction the caller hands in (poisson: already exp(score)),
// spotlight/losses.py:188-244.  d = d per / d pred.
__device__ __forceinline__ void rating_elem(int loss, float p, float r, float& per, float& d) {
    if (loss == SLB_LOSS_REGRESSION) {
        const float e = r - p;
        per = e * e; d = -2.0f * e;
    } else if (loss == SLB_LOSS_POISSON) {
        per = p - r * logf(p); d = 1.0f - r / p;
    } else {
        const float t = fminf(fmaxf(r, 0.0f), 1.0f);       // (-1, 1) targets -> (0, 1), losses.py:240
        per = fmaxf(p, 0.0f) - p * t + log1pf(expf(-fabsf(p)));
        d = sigmoidf_(p) - t;
    }
}

// One pass: per-element gradients (the divisor n is known up front) and the block partials;
// the last block folds the partials in a fixed order.
__global__ void __launch_bounds__(L_THREADS)
rating_loss_kernel(int loss, const float* __restrict__ pred, const float* __restrict__ ratings, int64_t n,
                   float* partial, int32_t* done, float* loss_out, float* __restrict__ grad) {
    __shared__ float red[L_THREADS / 32];
    __shared__ bool is_last;
    const float inv = 1.0f / static_cast<float>(n);
    float ls = 0.f;
    for (int64_t i = static_cast<int64_t>(blockIdx.x) * L_THREADS + threadIdx.x; i < n;
         i += static_cast<int64_t>(gridDim.x) * L_THREADS) {
        float per, d;
        rating_elem(loss, pred[i], ratings[i], per, d);
        ls += per;
        if (grad) grad[i] = d * inv;
    }
    float a;
    if (grid_fold<L_THREADS>(ls, red, is_last, partial, done, a)) { *loss_out = a * inv; *done = 0; }
}

}  // namespace

extern "C" {

size_t slb_loss_workspace_bytes(int64_t n) {
    (void)n;
    WsCarver ws(nullptr);
    ws.take<int32_t>(8);
    ws.take<float>(8);
    ws.take<float>(2 * L_MAX_GRID);
    return ws.bytes();
}

int slb_pairwise_loss(int32_t loss, const float* pos, const float* neg, const uint8_t* mask,
                      int64_t n, int32_t n_neg, float* loss_out, float* gpos, float* gneg,
                      void* workspace, size_t workspace_bytes, slb_stream_t stream) {
    SLB_REQUIRE(loss >= 0 && loss <= 3, "pairwise_loss: bad loss kind %d", loss);
    SLB_REQUIRE(pos && neg && loss_out && workspace, "pairwise_loss: null pointer");
    SLB_REQUIRE(n > 0 && n_neg >= 1, "pairwise_loss: bad sizes");
    SLB_REQUIRE((gpos == nullptr) == (gneg == nullptr), "pairwise_loss: gpos and gneg go together");
    if (workspace_bytes < slb_loss_workspace_bytes(n)) {
        slb_set_error("pairwise_loss: workspace too small");
        return SLB_ENOSPC;
    }
    WsCarver ws(workspace);
    int32_t* done = ws.take<int32_t>(8);
    float* sums = ws.take<float>(8);
    float* partial = ws.take<float>(2 * L_MAX_GRID);
    int64_t want = (n + L_THREADS - 1) / L_THREADS;
    const int grid = min(slb_grid(want, 8), L_MAX_GRID);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    loss_reduce_kernel<<<grid, L_THREADS, 0, st>>>(loss, pos, neg, mask, n, n_neg, partial, done, sums, loss_out);
    SLB_LAUNCH_CHECK("loss_reduce_kernel");
    if (gpos) {
        loss_grad_kernel<<<grid, L_THREADS, 0, st>>>(loss, pos, neg, mask, n, n_neg, sums, gpos, gneg);
        SLB_LAUNCH_CHECK("loss_grad_kernel");
    }
    return SLB_OK;
}

int slb_rating_loss(int32_t loss, const float* pred, const float* ratings, int64_t n,
                    float* loss_out, float* grad, void* workspace, size_t workspace_bytes,
                    slb_stream_t stream) {
    SLB_REQUIRE(loss >= SLB_LOSS_REGRESSION && loss <= SLB_LOSS_LOGISTIC, "rating_loss: bad loss kind %d", loss);
    SLB_REQUIRE(pred && ratings && loss_out && workspace, "rating_loss: null pointer");
    SLB_REQUIRE(n > 0, "rating_loss: n must be > 0");
    if (workspace_bytes < slb_loss_workspace_bytes(n)) {
        slb_set_error("rating_loss: workspace too small");
        return SLB_ENOSPC;
    }
    WsCarver ws(workspace);
    int32_t* done = ws.take<int32_t>(8);
    ws.take<float>(8);
    float* partial = ws.take<float>(2 * L_MAX_GRID);
    const int64_t want = (n + L_THREADS - 1) / L_THREADS;
    const int grid = min(slb_grid(want, 8), L_MAX_GRID);
    rating_loss_kernel<<<grid, L_THREADS, 0, static_cast<cudaStream_t>(stream)>>>(loss, pred, ratings, n, partial,
                                                                                  done, loss_out, grad);
    SLB_LAUNCH_CHECK("rating_loss_kernel");
    return SLB_OK;
}

}  // extern "C"
