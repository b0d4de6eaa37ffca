// f3 evaluation scoring for the mixture-of-tastes head (MixtureLSTMNet): every sequence of a block
// against every item in one launch, FP32 FMA throughout, never writing the 2M per-pair dot products.
//
// The block is a GEMM with a per-pair epilogue: the rows (r, j) of reps, viewed as a
// (n_rows * 2M, D) matrix, times the item rows; the 2M products of one (sequence, item) pair are
// then reduced by the softmax head.  A CTA covers SEQS sequences x ITEMS items.  Each thread owns
// TR sequences x TI items and keeps their TR * 2M * TI dot products in registers; the rep and item
// tiles are staged through shared memory KC columns of D at a time, double-buffered with
// cp.async so the next chunk's copies run under the current chunk's FMAs.
//
// Determinism: every dot product is one fmaf chain over d = 0 .. D-1 in order (columns past D in
// the last chunk are zero and add +0), and the epilogue is the same straight-line code for every
// pair, so scores[r, i] depends only on reps[r], items[i] and item_bias[i] -- not on n_rows,
// n_items or where the pair falls in a tile.
#include "common.cuh"

namespace {

constexpr int MIX_THREADS = 256;   // 16 x 16: tx along items, ty along sequences
constexpr int MIX_KC = 16;         // columns of D per shared-memory stage
constexpr int MIX_PAD = 4;         // keeps float4 reads aligned, halves the transposed-store conflicts

template <int M>
struct MixTile {
    static constexpr int TR = M == 1 ? 4 : (M == 2 ? 2 : 1);   // sequences per thread
    static constexpr int ROWS = TR * 2 * M;                   // rep rows per thread
    static constexpr int TI = ROWS <= 8 ? 8 : 4;              // items per thread: <= 64 accumulators
    static constexpr int SEQS = 16 * TR;
    static constexpr int ITEMS = 16 * TI;
    static constexpr int A_ROWS = SEQS * 2 * M;               // rep rows per CTA
    static constexpr int A_LD = A_ROWS + MIX_PAD;
    static constexpr int B_LD = ITEMS + MIX_PAD;
    static constexpr int A_ELEMS = A_ROWS * MIX_KC;            // per stage
    static constexpr int B_ELEMS = ITEMS * MIX_KC;
    static_assert(ROWS % 2 == 0 && ROWS * TI <= 64, "thread tile");
};

// Copies element e of a (rows, KC) stage whose first row is `row0` of a (n, D) matrix into
// sm[k][row] (transposed, so a thread's rows or items at one k are adjacent), asynchronously and
// zero-filled past the matrix.
__device__ __forceinline__ void mix_copy(float* sm, int ld, const float* __restrict__ src, int64_t row0, int64_t n,
                                         int dim, int k0, int e) {
    const int row = e / MIX_KC, k = e % MIX_KC;
    const bool in = row0 + row < n && k0 + k < dim;
    const float* g = in ? src + (row0 + row) * dim + k0 + k : src;
    const unsigned dst = static_cast<unsigned>(__cvta_generic_to_shared(sm + k * ld + row));
    asm volatile("cp.async.ca.shared.global [%0], [%1], 4, %2;\n" ::"r"(dst), "l"(g), "r"(in ? 4 : 0));
}

template <int M>
__global__ void __launch_bounds__(MIX_THREADS, 2)
mixture_scores_kernel(const float* __restrict__ reps, int64_t n_rows, int dim, const float* __restrict__ items,
                      const float* __restrict__ item_bias, int64_t n_items, int64_t row_tiles,
                      float* __restrict__ scores) {
    using T = MixTile<M>;
    __shared__ __align__(16) float As[2][MIX_KC * T::A_LD];
    __shared__ __align__(16) float Bs[2][MIX_KC * T::B_LD];

    // consecutive CTAs share an item tile, so it is read from HBM once and the rest hit L2
    const int64_t tile = blockIdx.x;
    const int64_t seq0 = (tile % row_tiles) * T::SEQS;
    const int64_t item0 = (tile / row_tiles) * T::ITEMS;
    const int64_t a_row0 = seq0 * 2 * M;
    const int64_t a_rows = n_rows * 2 * M;
    const int tid = threadIdx.x;
    const int tx = tid % 16, ty = tid / 16;

    float acc[T::ROWS][T::TI];
#pragma unroll
    for (int r = 0; r < T::ROWS; ++r)
#pragma unroll
        for (int u = 0; u < T::TI; ++u) acc[r][u] = 0.f;

    auto fetch = [&](int c) {
        const int k0 = c * MIX_KC;
#pragma unroll
        for (int e = tid; e < T::A_ELEMS; e += MIX_THREADS)
            mix_copy(As[c & 1], T::A_LD, reps, a_row0, a_rows, dim, k0, e);
#pragma unroll
        for (int e = tid; e < T::B_ELEMS; e += MIX_THREADS)
            mix_copy(Bs[c & 1], T::B_LD, items, item0, n_items, dim, k0, e);
        asm volatile("cp.async.commit_group;\n" ::);
    };

    const int chunks = (dim + MIX_KC - 1) / MIX_KC;
    fetch(0);
    for (int c = 0; c < chunks; ++c) {
        if (c + 1 < chunks) {
            fetch(c + 1);
            asm volatile("cp.async.wait_group 1;\n" ::);
        } else {
            asm volatile("cp.async.wait_group 0;\n" ::);
        }
        __syncthreads();
        const float* as = As[c & 1] + ty * T::ROWS;
        const float* bs = Bs[c & 1] + tx * 4;
#pragma unroll
        for (int k = 0; k < MIX_KC; ++k) {
            float a[T::ROWS], b[T::TI];
            if constexpr (T::ROWS % 4 == 0) {
#pragma unroll
                for (int r = 0; r < T::ROWS; r += 4) {
                    const float4 x = *reinterpret_cast<const float4*>(as + k * T::A_LD + r);
                    a[r] = x.x;
                    a[r + 1] = x.y;
                    a[r + 2] = x.z;
                    a[r + 3] = x.w;
                }
            } else {
#pragma unroll
                for (int r = 0; r < T::ROWS; r += 2) {
                    const float2 x = *reinterpret_cast<const float2*>(as + k * T::A_LD + r);
                    a[r] = x.x;
                    a[r + 1] = x.y;
                }
            }
#pragma unroll
            for (int h = 0; h < T::TI / 4; ++h) {
                const float4 x = *reinterpret_cast<const float4*>(bs + k * T::B_LD + 64 * h);
                b[4 * h] = x.x;
                b[4 * h + 1] = x.y;
                b[4 * h + 2] = x.z;
                b[4 * h + 3] = x.w;
            }
#pragma unroll
            for (int r = 0; r < T::ROWS; ++r)
#pragma unroll
                for (int u = 0; u < T::TI; ++u) acc[r][u] = fmaf(a[r], b[u], acc[r][u]);
        }
        __syncthreads();   // the next iteration's copies overwrite this stage
    }

    // epilogue: w = softmax_m(v_m . e), score = beta + sum_m w_m (c_m . e), four items per store
#pragma unroll
    for (int t = 0; t < T::TR; ++t) {
        const int64_t r = seq0 + ty * T::TR + t;
        if (r >= n_rows) continue;
#pragma unroll
        for (int h = 0; h < T::TI / 4; ++h) {
            const int64_t i0 = item0 + 64 * h + tx * 4;
            float s[4];
#pragma unroll
            for (int q = 0; q < 4; ++q) {
                const int u = 4 * h + q;
                float mx = acc[t * 2 * M + M][u];
#pragma unroll
                for (int m = 1; m < M; ++m) mx = fmaxf(mx, acc[t * 2 * M + M + m][u]);
                float w[M];
                float sum = 0.f;
#pragma unroll
                for (int m = 0; m < M; ++m) {
                    w[m] = expf(acc[t * 2 * M + M + m][u] - mx);
                    sum += w[m];
                }
                float sbar = 0.f;
#pragma unroll
                for (int m = 0; m < M; ++m) sbar = fmaf(w[m] / sum, acc[t * 2 * M + m][u], sbar);
                const int64_t i = i0 + q;
                s[q] = i < n_items ? __ldg(item_bias + i) + sbar : 0.f;
            }
            float* dst = scores + r * n_items + i0;
            if (i0 + 3 < n_items && (n_items & 3) == 0) {
                *reinterpret_cast<float4*>(dst) = make_float4(s[0], s[1], s[2], s[3]);
            } else {
#pragma unroll
                for (int q = 0; q < 4; ++q)
                    if (i0 + q < n_items) dst[q] = s[q];
            }
        }
    }
}

template <int M>
int launch_mixture_scores(const float* reps, int64_t n_rows, int dim, const float* items, const float* item_bias,
                          int64_t n_items, float* scores, cudaStream_t stream) {
    using T = MixTile<M>;
    const int64_t row_tiles = (n_rows + T::SEQS - 1) / T::SEQS;
    const int64_t item_tiles = (n_items + T::ITEMS - 1) / T::ITEMS;
    SLB_REQUIRE(row_tiles <= INT32_MAX / item_tiles, "mixture_scores: %lld x %lld tiles exceed one grid",
                static_cast<long long>(row_tiles), static_cast<long long>(item_tiles));
    mixture_scores_kernel<M><<<static_cast<unsigned>(row_tiles * item_tiles), MIX_THREADS, 0, stream>>>(
        reps, n_rows, dim, items, item_bias, n_items, row_tiles, scores);
    SLB_LAUNCH_CHECK("mixture_scores_kernel");
    return SLB_OK;
}

bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

}  // namespace

extern "C" {

int slb_mixture_scores(const float* reps, int64_t n_rows, int32_t num_mixtures, int32_t dim, const float* items,
                       const float* item_bias, int64_t n_items, float* scores, slb_stream_t stream) {
    SLB_REQUIRE(reps && items && item_bias && scores, "mixture_scores: null pointer");
    SLB_REQUIRE(n_rows > 0 && n_items > 0, "mixture_scores: n_rows = %lld, n_items = %lld must be positive",
                static_cast<long long>(n_rows), static_cast<long long>(n_items));
    SLB_REQUIRE(num_mixtures >= 1 && num_mixtures <= 8, "mixture_scores: num_mixtures = %d not in 1..8",
                num_mixtures);
    SLB_REQUIRE(dim > 0 && dim % 4 == 0, "mixture_scores: dim = %d must be a positive multiple of 4", dim);
    SLB_REQUIRE(aligned16(reps) && aligned16(items) && aligned16(scores),
                "mixture_scores: reps, items and scores must be 16-byte aligned");
    const cudaStream_t st = static_cast<cudaStream_t>(stream);
    switch (num_mixtures) {
        case 1: return launch_mixture_scores<1>(reps, n_rows, dim, items, item_bias, n_items, scores, st);
        case 2: return launch_mixture_scores<2>(reps, n_rows, dim, items, item_bias, n_items, scores, st);
        case 3: return launch_mixture_scores<3>(reps, n_rows, dim, items, item_bias, n_items, scores, st);
        case 4: return launch_mixture_scores<4>(reps, n_rows, dim, items, item_bias, n_items, scores, st);
        case 5: return launch_mixture_scores<5>(reps, n_rows, dim, items, item_bias, n_items, scores, st);
        case 6: return launch_mixture_scores<6>(reps, n_rows, dim, items, item_bias, n_items, scores, st);
        case 7: return launch_mixture_scores<7>(reps, n_rows, dim, items, item_bias, n_items, scores, st);
        default: return launch_mixture_scores<8>(reps, n_rows, dim, items, item_bias, n_items, scores, st);
    }
}

}  // extern "C"
