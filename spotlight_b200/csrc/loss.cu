// Standalone implicit-feedback losses (generic / custom-representation path).
// Replaces spotlight/losses.py:18-166: pointwise, bpr, hinge, adaptive hinge,
// each with the optional mask (masked mean = sum(loss*mask)/mask.sum()).
#include "common.cuh"

namespace {

constexpr int L_THREADS = 256;
constexpr int L_MAX_GRID = 132 * 8;

__device__ __forceinline__ void elem_loss(int loss, float p, float n, float& per, float& gp, float& gn) {
    if (loss == SLB_LOSS_BPR) {
        const float s = sigmoidf_(p - n);
        per = 1.0f - s; gp = -s * (1.0f - s); gn = -gp;
    } else if (loss == SLB_LOSS_POINTWISE) {
        const float sp = sigmoidf_(p), sn = sigmoidf_(n);
        per = (1.0f - sp) + sn; gp = -sp * (1.0f - sp); gn = sn * (1.0f - sn);
    } else {
        const float z = n - p + 1.0f;
        per = fmaxf(z, 0.0f);
        const float act = z >= 0.0f ? 1.0f : 0.0f;
        gp = -act; gn = act;
    }
}

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
        elem_loss(loss, pos[i], nv, per, gp, gn);
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
        elem_loss(loss, pos[i], nv, per, gp, gn);
        const float w = (mask ? (mask[i] ? 1.0f : 0.0f) : 1.0f) * inv;
        gpos[i] = gp * w;
        if (loss == SLB_LOSS_ADAPTIVE_HINGE) {
            for (int k = 0; k < n_neg; ++k) gneg[static_cast<int64_t>(k) * n + i] = k == ks ? gn * w : 0.f;
        } else {
            gneg[i] = gn * w;
        }
    }
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
    const int64_t cap = static_cast<int64_t>(slb_sms()) * 8 < L_MAX_GRID ? static_cast<int64_t>(slb_sms()) * 8 : L_MAX_GRID;
    const int grid = static_cast<int>(want < cap ? want : cap);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    loss_reduce_kernel<<<grid, L_THREADS, 0, st>>>(loss, pos, neg, mask, n, n_neg, partial, done, sums, loss_out);
    SLB_LAUNCH_CHECK("loss_reduce_kernel");
    if (gpos) {
        loss_grad_kernel<<<grid, L_THREADS, 0, st>>>(loss, pos, neg, mask, n, n_neg, sums, gpos, gneg);
        SLB_LAUNCH_CHECK("loss_grad_kernel");
    }
    return SLB_OK;
}

}  // extern "C"
