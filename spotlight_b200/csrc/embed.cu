// Embedding gathers and their deterministic backward for sm_90a.
//
// Replaces ScaledEmbedding / ZeroEmbedding / BloomEmbedding forward
// (spotlight/layers.py:23-56, 206-244: nn.Embedding lookup; Bloom = index_select
// of the pre-hashed (N, H) table + H-row gather + sum(1)) and
// aten::embedding_dense_backward.  Bloom hashes are computed in registers
// (murmur3 of the id, layers.py:178-204) instead of reading the reference's
// 8*H bytes/id hash table.
#include <cfloat>

#include "segindex.cuh"

namespace {

constexpr int EMB_THREADS = 256;
constexpr int MAX_HASH = 24;  // len(SEEDS), layers.py:13-20

struct HashSpec {
    int32_t H;            // 0 = plain lookup
    int64_t padding_idx;
    uint32_t seeds[MAX_HASH];
};

__device__ __forceinline__ int64_t term_row(const HashSpec& hs, const int64_t* __restrict__ ids,
                                            int64_t t, int64_t rows) {
    if (hs.H == 0) return ids[t];
    return bloom_row(ids[t / hs.H], hs.seeds[t % hs.H], rows, hs.padding_idx);
}

template <int LPR, bool VEC4>
__global__ void __launch_bounds__(EMB_THREADS)
emb_fwd_kernel(const float* __restrict__ W, int64_t rows, int D, const int64_t* __restrict__ ids,
               int64_t n, HashSpec hs, float* __restrict__ out, int32_t* err) {
    constexpr int GROUPS = EMB_THREADS / LPR;
    const int gl = threadIdx.x & (LPR - 1);
    const int fan = hs.H == 0 ? 1 : hs.H;
    for (int64_t b = static_cast<int64_t>(blockIdx.x) * GROUPS + threadIdx.x / LPR; b < n;
         b += static_cast<int64_t>(gridDim.x) * GROUPS) {
        constexpr int STEP = VEC4 ? 4 : 1;
        for (int c = gl * STEP; c < D; c += LPR * STEP) {
            float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
            for (int k = 0; k < fan; ++k) {
                int64_t r = term_row(hs, ids, b * fan + k, rows);
                if (r < 0 || r >= rows) { if (err) atomicExch(err, 1); r = 0; }
                if (VEC4) {
                    const float4 v = ldg4(W + r * D + c);
                    acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w;
                } else {
                    acc.x += __ldg(W + r * D + c);
                }
            }
            if (VEC4) st4(out + b * D + c, acc); else out[b * D + c] = acc.x;
        }
    }
}

__global__ void bloom_rows_kernel(const int64_t* __restrict__ ids, int64_t n, HashSpec hs,
                                  int64_t rows, int64_t* __restrict__ out) {
    const int64_t T = n * hs.H;
    for (int64_t t = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; t < T;
         t += static_cast<int64_t>(gridDim.x) * blockDim.x)
        out[t] = term_row(hs, ids, t, rows);
}

__global__ void __launch_bounds__(256)
emb_count_kernel(const int64_t* __restrict__ ids, int64_t T, HashSpec hs, int64_t rows,
                 int32_t* __restrict__ keys, SegIndex seg, int32_t* err) {
    for (int64_t t = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; t < T;
         t += static_cast<int64_t>(gridDim.x) * blockDim.x) {
        int64_t r = term_row(hs, ids, t, rows);
        if (r < 0 || r >= rows) { atomicExch(err, 1); r = 0; }
        keys[t] = static_cast<int32_t>(r);
        atomicAdd(seg.cnt + r, 1);
    }
}

__global__ void __launch_bounds__(256)
emb_fill_kernel(const int32_t* __restrict__ keys, int64_t T, SegIndex seg) {
    seg_rearm(seg);
    for (int64_t t = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; t < T;
         t += static_cast<int64_t>(gridDim.x) * blockDim.x)
        seg_place(seg, keys[t], static_cast<int32_t>(t));
}

template <int LPR, bool VEC4>
__global__ void __launch_bounds__(EMB_THREADS)
emb_bwd_kernel(const float* __restrict__ dout, int D, int fan, SegIndex seg, int64_t frozen_row,
               float* __restrict__ dW) {
    constexpr int GROUPS = EMB_THREADS / LPR;
    constexpr int CAP = seg_sort_cap(LPR);
    __shared__ int32_t sh_sort[GROUPS * 2 * CAP];
    const int gl = threadIdx.x & (LPR - 1);
    const int gib = threadIdx.x / LPR;
    const unsigned gmask = group_mask(LPR);
    int32_t* sh = sh_sort + gib * 2 * CAP;
    const int nseg = seg.totals[0];
    constexpr int STEP = VEC4 ? 4 : 1;
    for (int64_t s = static_cast<int64_t>(blockIdx.x) * GROUPS + gib; s < nseg;
         s += static_cast<int64_t>(gridDim.x) * GROUPS) {
        const int start = seg.seg_start[s];
        const int len = seg.seg_start[s + 1] - start;
        const int64_t row = seg.seg_row[s];
        if (row == frozen_row) continue;
        for (int c0 = 0; c0 < D; c0 += LPR * STEP) {
            const int c = c0 + gl * STEP;
            float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
            seg_visit_sorted<LPR>(seg.members, start, len, gl, gmask, sh, [&](int32_t t) {
                const float* src = dout + static_cast<int64_t>(t / fan) * D;
                if (c < D) {
                    if (VEC4) {
                        const float4 v = ldg4(src + c);
                        acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w;
                    } else {
                        acc.x += __ldg(src + c);
                    }
                }
            });
            if (c < D) { if (VEC4) st4(dW + row * D + c, acc); else dW[row * D + c] = acc.x; }
        }
    }
}

int pow2_lanes(int n) {
    int p = 1;
    while (p < n && p < 32) p <<= 1;
    return p;
}

int make_hash(HashSpec& hs, int32_t H, const uint32_t* seeds, int64_t padding_idx) {
    SLB_REQUIRE(H >= 0 && H <= MAX_HASH, "hash_count must be in [0, %d]", MAX_HASH);
    SLB_REQUIRE(H == 0 || seeds != nullptr, "hash seeds missing");
    hs.H = H;
    hs.padding_idx = padding_idx;
    for (int k = 0; k < MAX_HASH; ++k) hs.seeds[k] = k < H ? seeds[k] : 0u;
    return SLB_OK;
}

struct EmbLayout { int32_t* flags; int32_t* keys; SegIndex seg; size_t bytes; };

EmbLayout emb_layout(void* base, int64_t T, int64_t rows) {
    WsCarver ws(base);
    EmbLayout l;
    l.flags = ws.take<int32_t>(8);
    l.seg = seg_index_carve(ws, rows, T);
    l.keys = ws.take<int32_t>(T);
    l.bytes = ws.bytes();
    return l;
}

}  // namespace

extern "C" {

int slb_embedding_forward(const float* W, int64_t rows, int32_t dim, const int64_t* ids, int64_t n,
                          int32_t hash_count, const uint32_t* seeds, int64_t padding_idx,
                          float* out, slb_stream_t stream) {
    SLB_REQUIRE(rows > 0 && dim > 0, "embedding_forward: bad table shape");
    if (n <= 0) return SLB_OK;          // an empty lookup: its tensors may have no storage
    SLB_REQUIRE(W && ids && out, "embedding_forward: null pointer");
    HashSpec hs;
    const int rc = make_hash(hs, hash_count, seeds, padding_idx);
    if (rc != SLB_OK) return rc;
    const bool vec4 = dim % 4 == 0;
    const int lpr = pow2_lanes(vec4 ? dim / 4 : dim);
    const int grid = slb_grid((n + EMB_THREADS / lpr - 1) / (EMB_THREADS / lpr), 8);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    with_bool(vec4, [&](auto V) {
        with_lpr(lpr, [&](auto L) {
            emb_fwd_kernel<L, V><<<grid, EMB_THREADS, 0, st>>>(W, rows, dim, ids, n, hs, out, nullptr);
        });
    });
    SLB_LAUNCH_CHECK("emb_fwd_kernel");
    return SLB_OK;
}

int slb_bloom_rows(const int64_t* ids, int64_t n, int32_t hash_count, const uint32_t* seeds,
                   int64_t rows, int64_t padding_idx, int64_t* rows_out, slb_stream_t stream) {
    SLB_REQUIRE(hash_count > 0 && rows > 0, "bloom_rows: bad arguments");
    if (n <= 0) return SLB_OK;
    SLB_REQUIRE(ids && rows_out, "bloom_rows: null pointer");
    HashSpec hs;
    const int rc = make_hash(hs, hash_count, seeds, padding_idx);
    if (rc != SLB_OK) return rc;
    bloom_rows_kernel<<<slb_grid((n * hash_count + 255) / 256, 8), 256, 0, static_cast<cudaStream_t>(stream)>>>(
        ids, n, hs, rows, rows_out);
    SLB_LAUNCH_CHECK("bloom_rows_kernel");
    return SLB_OK;
}

size_t slb_embedding_backward_workspace_bytes(int64_t n_terms, int64_t rows) {
    return emb_layout(nullptr, n_terms, rows).bytes;
}

int slb_embedding_backward(const float* dout, const int64_t* ids, int64_t n, int32_t hash_count,
                           const uint32_t* seeds, int64_t rows, int32_t dim, int64_t frozen_row,
                           float* dW, void* workspace, size_t workspace_bytes, slb_stream_t stream) {
    SLB_REQUIRE(rows > 0 && dim > 0, "embedding_backward: bad table shape");
    if (n <= 0) return SLB_OK;          // nothing to scatter: dW stays as the caller zeroed it
    SLB_REQUIRE(dout && ids && dW && workspace, "embedding_backward: null pointer");
    HashSpec hs;
    const int rc = make_hash(hs, hash_count, seeds, -1);
    if (rc != SLB_OK) return rc;
    hs.padding_idx = frozen_row;   // Bloom: padding id hashes to row 0 (layers.py:184)
    const int fan = hash_count == 0 ? 1 : hash_count;
    const int64_t T = n * fan;
    SLB_REQUIRE(T < (1ll << 31) && rows < (1ll << 31) - SEG_SCAN_TILE, "embedding_backward: too large");
    EmbLayout l = emb_layout(workspace, T, rows);
    if (workspace_bytes < l.bytes) {
        slb_set_error("embedding_backward: workspace too small (%zu < %zu)", workspace_bytes, l.bytes);
        return SLB_ENOSPC;
    }
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const int g1 = slb_grid((T + 255) / 256, 8);
    emb_count_kernel<<<g1, 256, 0, st>>>(ids, T, hs, rows, l.keys, l.seg, l.flags + 4);
    SLB_LAUNCH_CHECK("emb_count_kernel");
    seg_scan_launch(l.seg, rows, st);
    SLB_LAUNCH_CHECK("seg_scan_kernel");
    emb_fill_kernel<<<g1, 256, 0, st>>>(l.keys, T, l.seg);
    SLB_LAUNCH_CHECK("emb_fill_kernel");
    const bool vec4 = dim % 4 == 0;
    const int lpr = pow2_lanes(vec4 ? dim / 4 : dim);
    const int grid = slb_grid((T + EMB_THREADS / lpr - 1) / (EMB_THREADS / lpr), 8);
    // Bloom: the inner table is ScaledEmbedding(M, D, padding_idx=padding_idx)
    // (layers.py:162-164), so the same index is frozen in the compressed table
    with_bool(vec4, [&](auto V) {
        with_lpr(lpr, [&](auto L) { emb_bwd_kernel<L, V><<<grid, EMB_THREADS, 0, st>>>(dout, dim, fan, l.seg, frozen_row, dW); });
    });
    SLB_LAUNCH_CHECK("emb_bwd_kernel");
    return SLB_OK;
}

// f3 evaluation scoring: average rank (scipy.stats.rankdata of the NEGATED scores, as
// spotlight/evaluation.py:49 uses it) of selected items within their user's score row:
//   rank = 1 + #(scores > s) + 0.5 * (#(scores == s) - 1).
// One warp per (row, item) pair; the row is L2 resident between the pairs of one user.
static __global__ void __launch_bounds__(256)
rank_pairs_kernel(const float* __restrict__ scores, int64_t n_items, const int64_t* __restrict__ pair_row,
                  const int64_t* __restrict__ pair_item, int64_t n_pairs, float* __restrict__ ranks) {
    const int lane = threadIdx.x & 31;
    const int64_t warp = (static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
    const int64_t nwarps = (static_cast<int64_t>(gridDim.x) * blockDim.x) >> 5;
    for (int64_t p = warp; p < n_pairs; p += nwarps) {
        const float* row = scores + pair_row[p] * n_items;
        const float s = row[pair_item[p]];
        int gt = 0, eq = 0;
        for (int64_t k = lane; k < n_items; k += 32) {
            const float v = __ldg(row + k);
            gt += v > s;
            eq += v == s;
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            gt += __shfl_xor_sync(0xffffffffu, gt, o);
            eq += __shfl_xor_sync(0xffffffffu, eq, o);
        }
        if (lane == 0) ranks[p] = 1.0f + static_cast<float>(gt) + 0.5f * static_cast<float>(eq - 1);
    }
}

int slb_rank_pairs(const float* scores, int64_t n_rows, int64_t n_items, const int64_t* pair_row,
                   const int64_t* pair_item, int64_t n_pairs, float* ranks, slb_stream_t stream) {
    if (n_pairs <= 0) return SLB_OK;
    SLB_REQUIRE(scores && pair_row && pair_item && ranks && n_rows > 0 && n_items > 0, "rank_pairs: bad arguments");
    const int64_t want = (n_pairs * 32 + 255) / 256;
    const int grid = static_cast<int>(want < static_cast<int64_t>(slb_sms()) * 16 ? want : static_cast<int64_t>(slb_sms()) * 16);
    rank_pairs_kernel<<<grid, 256, 0, static_cast<cudaStream_t>(stream)>>>(scores, n_items, pair_row, pair_item, n_pairs, ranks);
    SLB_LAUNCH_CHECK("rank_pairs_kernel");
    return SLB_OK;
}

}  // extern "C"

// f3 evaluation ranking in one pass per row: for every target of a row, the average rank
// (rank_pairs_kernel's, bit for bit) and the stable position (where the target lands in
// argsort(-row, kind='stable')), from #(row > s), #(row == s) and #(row == s, item < target).
// One CTA per row.  The row's targets are staged in shared memory sorted by (score desc, id asc);
// each row element is binary-searched against them once and drops +1/-1 boundaries into integer
// histograms whose prefix sums are every target's three counts.  Integer counts only, so the
// result does not depend on the order the elements are visited in.  A row with more than
// RT_CAP targets is handled in chunks of RT_CAP and re-read once per chunk.  NaN compares as
// neither greater nor equal, as in rank_pairs_kernel.
//
// The kernel is written once over an output policy.  RankFinal (slb_rank_targets) reads each
// target's score from its row and writes the average rank and stable position; RankCounts
// (slb_rank_counts) ranks against a block of the columns [col_offset, col_offset + n_cols) of the
// full row, takes the targets' scores from the caller (a target may lie outside the block) and
// writes the three counts, which add up across disjoint column ranges.
namespace {

constexpr int RT_THREADS = 256;
constexpr int RT_CAP = 1024;
constexpr int RT_WARPS = RT_THREADS / 32;

// f(v, i) for every element of row[0, n): scalar head up to 16-byte alignment, float4 body,
// scalar tail (a row of a [rows, n] block is 16-byte aligned only when n % 4 == 0)
template <class F>
__device__ __forceinline__ void rt_stream_row(const float* __restrict__ row, int64_t n, F&& f) {
    const int64_t mis = static_cast<int64_t>((reinterpret_cast<uintptr_t>(row) >> 2) & 3);
    const int64_t head = min(n, (4 - mis) & 3);
    for (int64_t i = threadIdx.x; i < head; i += RT_THREADS) f(__ldg(row + i), i);
    const int64_t nv = (n - head) >> 2;
    const float4* row4 = reinterpret_cast<const float4*>(row + head);
    for (int64_t q = threadIdx.x; q < nv; q += RT_THREADS) {
        const float4 v = __ldg(row4 + q);
        const int64_t i = head + 4 * q;
        f(v.x, i); f(v.y, i + 1); f(v.z, i + 2); f(v.w, i + 3);
    }
    for (int64_t i = head + 4 * nv + threadIdx.x; i < n; i += RT_THREADS) f(__ldg(row + i), i);
}

// (score desc, id asc), NaN scores last
__device__ __forceinline__ bool rt_before(float ka, int32_t ia, float kb, int32_t ib) {
    const bool na = isnan(ka), nb = isnan(kb);
    if (na != nb) return nb;
    if (!na && ka != kb) return ka > kb;
    return ia < ib;
}

// block-wide exclusive prefix sum of three ints (all threads must call)
__device__ __forceinline__ void rt_exclusive_scan3(int v[3], int (*warp_tot)[RT_WARPS]) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    int inc[3] = {v[0], v[1], v[2]};
#pragma unroll
    for (int o = 1; o < 32; o <<= 1)
#pragma unroll
        for (int k = 0; k < 3; ++k) {
            const int u = __shfl_up_sync(0xffffffffu, inc[k], o);
            if (lane >= o) inc[k] += u;
        }
    if (lane == 31)
        for (int k = 0; k < 3; ++k) warp_tot[k][warp] = inc[k];
    __syncthreads();
    for (int k = 0; k < 3; ++k) {
        int before = inc[k] - v[k];
        for (int w = 0; w < warp; ++w) before += warp_tot[k][w];
        v[k] = before;
    }
    __syncthreads();
}

__device__ __forceinline__ void rt_write(int64_t p, int gt, int eq, int eq_before, float* __restrict__ avg_rank,
                                         int64_t* __restrict__ position) {
    if (avg_rank) avg_rank[p] = 1.0f + static_cast<float>(gt) + 0.5f * static_cast<float>(eq - 1);
    if (position) position[p] = static_cast<int64_t>(gt) + eq_before;
}

// the whole row: the target's score is its own element, the counts become rank and position
struct RankFinal {
    float* avg_rank;
    int64_t* position;
    static constexpr int64_t col0 = 0;
    __device__ __forceinline__ float key(const float* row, int64_t, int64_t t) const { return row[t]; }
    __device__ __forceinline__ void write(int64_t p, int gt, int eq, int eq_before) const {
        rt_write(p, gt, eq, eq_before, avg_rank, position);
    }
};

// one column range of the row: scores supplied per target, the counts written as they are
struct RankCounts {
    const float* target_scores;
    int64_t col0;                                 // global id of the block's first column
    int32_t* gt;
    int32_t* eq;
    int32_t* eq_before;
    __device__ __forceinline__ float key(const float*, int64_t p, int64_t) const { return target_scores[p]; }
    __device__ __forceinline__ void write(int64_t p, int g, int e, int b) const {
        gt[p] = g; eq[p] = e; eq_before[p] = b;
    }
};

template <class Out>
__global__ void __launch_bounds__(RT_THREADS)
rank_targets_kernel(const float* __restrict__ scores, int64_t n_rows, int64_t n_items,
                    const int64_t* __restrict__ row_ptr, const int64_t* __restrict__ targets, Out out) {
    __shared__ float key[RT_CAP];
    __shared__ int32_t id[RT_CAP];
    __shared__ int16_t slot[RT_CAP];              // index of the sorted entry within its chunk
    __shared__ int32_t hist[3][RT_CAP + 1];       // boundaries of the greater / equal / equal-before ranges
    __shared__ int warp_tot[3][RT_WARPS];

    for (int64_t r = blockIdx.x; r < n_rows; r += gridDim.x) {
        const float* row = scores + r * n_items;
        const int64_t t0 = row_ptr[r], t1 = row_ptr[r + 1];
        if (t1 - t0 == 1) {
            // one target (sequence_mrr_score): plain compares and a block reduction
            const int64_t t = targets[t0];
            const float s = out.key(row, t0, t);
            int c[3] = {0, 0, 0};
            rt_stream_row(row, n_items, [&](float v, int64_t i) {
                c[0] += v > s;
                c[1] += v == s;
                c[2] += (v == s) & (out.col0 + i < t);
            });
            int tot[3] = {c[0], c[1], c[2]};
            rt_exclusive_scan3(c, warp_tot);
            if (threadIdx.x == RT_THREADS - 1)
                out.write(t0, c[0] + tot[0], c[1] + tot[1], c[2] + tot[2]);
            continue;
        }
        for (int64_t c0 = t0; c0 < t1; c0 += RT_CAP) {
            const int m = static_cast<int>(min(static_cast<int64_t>(RT_CAP), t1 - c0));
            int P = 1;
            while (P < m) P <<= 1;
            for (int j = threadIdx.x; j < P; j += RT_THREADS) {
                if (j < m) {
                    const int64_t t = targets[c0 + j];
                    id[j] = static_cast<int32_t>(t);
                    key[j] = out.key(row, c0 + j, t);
                } else {
                    id[j] = INT32_MAX;
                    key[j] = __int_as_float(0x7fffffff);
                }
                slot[j] = static_cast<int16_t>(j);
            }
            for (int j = threadIdx.x; j <= m; j += RT_THREADS) hist[0][j] = hist[1][j] = hist[2][j] = 0;
            __syncthreads();
            // bitonic sort of the P staged entries
            for (int k = 2; k <= P; k <<= 1)
                for (int h = k >> 1; h > 0; h >>= 1) {
                    for (int i = threadIdx.x; i < P; i += RT_THREADS) {
                        const int l = i ^ h;
                        if (l <= i) continue;
                        const bool swap = (i & k) == 0 ? rt_before(key[l], id[l], key[i], id[i])
                                                       : rt_before(key[i], id[i], key[l], id[l]);
                        if (swap) {
                            const float tk = key[i]; key[i] = key[l]; key[l] = tk;
                            const int32_t ti = id[i]; id[i] = id[l]; id[l] = ti;
                            const int16_t ts = slot[i]; slot[i] = slot[l]; slot[l] = ts;
                        }
                    }
                    __syncthreads();
                }
            int nv = 0;                                   // non-NaN targets, sorted first
            for (int j0 = 0; j0 < P; j0 += RT_THREADS) {
                const int j = j0 + threadIdx.x;
                nv += __syncthreads_count(j < P && !isnan(key[j]));
            }
            if (nv > 0)
                rt_stream_row(row, n_items, [&](float v, int64_t i) {
                    if (isnan(v)) return;
                    // a = #(targets with key >= v): v is greater than the targets [a, nv)
                    int lo = 0, hi = nv;
                    while (lo < hi) { const int mid = (lo + hi) >> 1; if (key[mid] >= v) lo = mid + 1; else hi = mid; }
                    const int a = lo;
                    if (a < nv) atomicAdd(&hist[0][a], 1);
                    if (a == 0 || key[a - 1] != v) return;
                    // b = #(targets with key > v): v equals the targets [b, a)
                    lo = 0; hi = a - 1;
                    while (lo < hi) { const int mid = (lo + hi) >> 1; if (key[mid] > v) lo = mid + 1; else hi = mid; }
                    const int b = lo;
                    atomicAdd(&hist[1][b], 1);
                    atomicSub(&hist[1][a], 1);
                    // within [b, a) the ids ascend: v precedes the targets with id > its global id gi
                    hi = a;
                    const int64_t gi = out.col0 + i;
                    while (lo < hi) { const int mid = (lo + hi) >> 1; if (id[mid] <= gi) lo = mid + 1; else hi = mid; }
                    if (lo < a) {
                        atomicAdd(&hist[2][lo], 1);
                        atomicSub(&hist[2][a], 1);
                    }
                });
            __syncthreads();
            // inclusive prefix sums over [0, nv): thread x owns a contiguous run of entries
            const int L = (nv + RT_THREADS - 1) / RT_THREADS;
            const int beg = min(nv, static_cast<int>(threadIdx.x) * L), end = min(nv, beg + L);
            int run[3] = {0, 0, 0};
            for (int x = beg; x < end; ++x)
                for (int k = 0; k < 3; ++k) run[k] += hist[k][x];
            rt_exclusive_scan3(run, warp_tot);
            for (int x = beg; x < end; ++x) {
                for (int k = 0; k < 3; ++k) run[k] += hist[k][x];
                out.write(c0 + slot[x], run[0], run[1], run[2]);
            }
            for (int x = nv + threadIdx.x; x < m; x += RT_THREADS) out.write(c0 + slot[x], 0, 0, 0);
            __syncthreads();
        }
    }
}

// The shard-local step between scoring and counting in the sharded sequence scorers: one CTA per
// row of the block [n_rows, n_cols] (the global items [col0, col0 + n_cols)) first writes -FLT_MAX
// over the row's excluded items that fall in the block (repeated ids write the same value), then,
// once those writes are visible to the CTA, reads every target's score when the target is in the
// block and 0 otherwise, so that summing the ranks' target_scores gives each target's score.
constexpr int MT_THREADS = 128;

__global__ void __launch_bounds__(MT_THREADS)
shard_mask_targets_kernel(float* scores, int64_t n_rows, int64_t n_cols, int64_t col0,
                          const int64_t* __restrict__ excluded, int64_t n_excl,
                          const int64_t* __restrict__ row_ptr, const int64_t* __restrict__ targets,
                          float* __restrict__ target_scores) {
    for (int64_t r = blockIdx.x; r < n_rows; r += gridDim.x) {
        float* row = scores + r * n_cols;
        for (int64_t j = threadIdx.x; j < n_excl; j += MT_THREADS) {
            const int64_t c = __ldg(excluded + r * n_excl + j) - col0;
            if (c >= 0 && c < n_cols) row[c] = -FLT_MAX;
        }
        __syncthreads();
        const int64_t t1 = __ldg(row_ptr + r + 1);
        for (int64_t p = __ldg(row_ptr + r) + threadIdx.x; p < t1; p += MT_THREADS) {
            const int64_t c = __ldg(targets + p) - col0;
            target_scores[p] = (c >= 0 && c < n_cols) ? row[c] : 0.f;
        }
    }
}

}  // namespace

extern "C" {

int slb_rank_targets(const float* scores, int64_t n_rows, int64_t n_items, const int64_t* row_ptr,
                     const int64_t* targets, int64_t n_targets, float* avg_rank, int64_t* position,
                     slb_stream_t stream) {
    if (n_targets <= 0 || n_rows <= 0) return SLB_OK;
    SLB_REQUIRE(scores && row_ptr && targets && n_items > 0 && n_items <= INT32_MAX,
                "rank_targets: bad arguments");
    if (!avg_rank && !position) return SLB_OK;
    const int64_t cap = static_cast<int64_t>(slb_sms()) * 8;
    const int grid = static_cast<int>(n_rows < cap ? n_rows : cap);
    rank_targets_kernel<<<grid, RT_THREADS, 0, static_cast<cudaStream_t>(stream)>>>(
        scores, n_rows, n_items, row_ptr, targets, RankFinal{avg_rank, position});
    SLB_LAUNCH_CHECK("rank_targets_kernel");
    return SLB_OK;
}

int slb_rank_counts(const float* scores, int64_t n_rows, int64_t n_cols, int64_t col_offset,
                    const int64_t* row_ptr, const int64_t* targets, const float* target_scores,
                    int64_t n_targets, int32_t* gt, int32_t* eq, int32_t* eq_before, slb_stream_t stream) {
    if (n_targets <= 0 || n_rows <= 0) return SLB_OK;
    SLB_REQUIRE(row_ptr && targets && target_scores && gt && eq && eq_before, "rank_counts: null pointer");
    SLB_REQUIRE(n_cols >= 0 && n_cols <= INT32_MAX && col_offset >= 0 && col_offset <= INT32_MAX - n_cols,
                "rank_counts: columns [%lld, %lld + %lld) outside [0, INT32_MAX]", static_cast<long long>(col_offset),
                static_cast<long long>(col_offset), static_cast<long long>(n_cols));
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    if (n_cols == 0) {                  // an empty item range: nothing ranks above or beside any target
        int32_t* outs[3] = {gt, eq, eq_before};
        for (int32_t* c : outs) {
            const cudaError_t e = cudaMemsetAsync(c, 0, sizeof(int32_t) * n_targets, st);
            if (e != cudaSuccess) {
                slb_set_error("rank_counts: %s", cudaGetErrorString(e));
                return SLB_ECUDA;
            }
        }
        return SLB_OK;
    }
    SLB_REQUIRE(scores, "rank_counts: null pointer");
    const int64_t cap = static_cast<int64_t>(slb_sms()) * 8;
    const int grid = static_cast<int>(n_rows < cap ? n_rows : cap);
    rank_targets_kernel<<<grid, RT_THREADS, 0, st>>>(scores, n_rows, n_cols, row_ptr, targets,
                                                     RankCounts{target_scores, col_offset, gt, eq, eq_before});
    SLB_LAUNCH_CHECK("rank_targets_kernel");
    return SLB_OK;
}

int slb_shard_mask_targets(float* scores, int64_t n_rows, int64_t n_cols, int64_t col_offset,
                           const int64_t* excluded, int64_t n_excluded_per_row, const int64_t* row_ptr,
                           const int64_t* targets, float* target_scores, slb_stream_t stream) {
    SLB_REQUIRE(n_rows >= 0 && n_excluded_per_row >= 0, "shard_mask_targets: n_rows = %lld, excluded per row = %lld",
                static_cast<long long>(n_rows), static_cast<long long>(n_excluded_per_row));
    SLB_REQUIRE(n_cols >= 0 && n_cols <= INT32_MAX && col_offset >= 0 && col_offset <= INT32_MAX - n_cols,
                "shard_mask_targets: columns [%lld, %lld + %lld) outside [0, INT32_MAX]",
                static_cast<long long>(col_offset), static_cast<long long>(col_offset), static_cast<long long>(n_cols));
    if (n_rows == 0) return SLB_OK;
    SLB_REQUIRE(row_ptr && targets && target_scores && (scores || n_cols == 0) && (excluded || n_excluded_per_row == 0),
                "shard_mask_targets: null pointer");
    const int64_t cap = static_cast<int64_t>(slb_sms()) * 8;
    const int grid = static_cast<int>(n_rows < cap ? n_rows : cap);
    shard_mask_targets_kernel<<<grid, MT_THREADS, 0, static_cast<cudaStream_t>(stream)>>>(
        scores, n_rows, n_cols, col_offset, excluded, n_excluded_per_row, row_ptr, targets, target_scores);
    SLB_LAUNCH_CHECK("shard_mask_targets_kernel");
    return SLB_OK;
}

}  // extern "C"
