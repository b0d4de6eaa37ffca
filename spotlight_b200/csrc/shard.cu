// Per-batch index bucketing for range-sharded embedding rows (SURVEY §8e).
//
// The reference has no multi-GPU path; this is the routing step of the new
// design: the distinct item ids a rank needs this step, in ascending order, are
// automatically grouped by owner (owner = id / chunk), so one counting pass over
// the row space + the segment scan yields the request lists for the all-to-all,
// and `inverse` remaps the batch onto the received row cache.
#include "segindex.cuh"

namespace {

__global__ void __launch_bounds__(256)
uq_count_kernel(const int64_t* __restrict__ ids, int64_t n, int64_t rows, SegIndex seg, int32_t* err) {
    const int64_t nth = static_cast<int64_t>(gridDim.x) * blockDim.x;
    for (int64_t t = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; t < n; t += nth) {
        int64_t r = ids[t];
        if (r < 0 || r >= rows) { atomicExch(err, 1); r = 0; }
        atomicAdd(seg.cnt + r, 1);
    }
}

// segment s <-> distinct id seg_row[s]; off[] is reused as the id -> position map
__global__ void __launch_bounds__(256)
uq_emit_kernel(SegIndex seg, int64_t chunk, int nparts, int64_t* __restrict__ uniq, int64_t* counts_out) {
    const int nseg = seg.totals[0];
    const int64_t nth = static_cast<int64_t>(gridDim.x) * blockDim.x;
    for (int64_t s = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; s < nseg; s += nth) {
        const int row = seg.seg_row[s];
        uniq[s] = row;
        seg.off[row] = static_cast<int32_t>(s);
        seg.cnt[row] = 0;                       // restore the zero-at-rest invariant
        // first position owned by each rank: boundary between consecutive distinct ids
        const int64_t own = row / chunk;
        const int64_t prev_own = s == 0 ? -1 : seg.seg_row[s - 1] / chunk;
        for (int64_t p = prev_own + 1; p <= own; ++p) counts_out[p] = s;
        if (s == nseg - 1)
            for (int64_t p = own + 1; p <= nparts; ++p) counts_out[p] = nseg;
    }
    if (blockIdx.x == 0 && threadIdx.x == 0) {
        counts_out[nparts + 1] = nseg;
        if (nseg == 0) for (int p = 0; p <= nparts; ++p) counts_out[p] = 0;
    }
}

__global__ void __launch_bounds__(256)
uq_inverse_kernel(const int64_t* __restrict__ ids, int64_t n, int64_t rows, SegIndex seg,
                  int64_t* __restrict__ inverse) {
    const int64_t nth = static_cast<int64_t>(gridDim.x) * blockDim.x;
    for (int64_t t = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; t < n; t += nth) {
        int64_t r = ids[t];
        if (r < 0 || r >= rows) r = 0;
        inverse[t] = seg.off[r];
    }
}

// users_out[k] = users[pos[k]] - user_lo, items_out[k] = items[pos[k]],
// negs_out[k*n + q] = negs[(pos[k] - neg_base)*n + q]: this rank's members of one global minibatch
__global__ void __launch_bounds__(256)
shard_gather_batch_kernel(const int64_t* __restrict__ pos, int64_t m, const int64_t* __restrict__ users,
                          const int64_t* __restrict__ items, const int64_t* __restrict__ negs, int64_t neg_base,
                          int n_neg, int64_t user_lo, int64_t* __restrict__ users_out,
                          int64_t* __restrict__ items_out, int64_t* __restrict__ negs_out) {
    const int64_t nth = static_cast<int64_t>(gridDim.x) * blockDim.x;
    for (int64_t k = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; k < m; k += nth) {
        const int64_t p = pos[k];
        users_out[k] = users[p] - user_lo;
        items_out[k] = items[p];
        for (int q = 0; q < n_neg; ++q) negs_out[k * n_neg + q] = negs[(p - neg_base) * n_neg + q];
    }
}

// torch.optim.Adagrad (lr_decay 0) on a dense shard; zero gradients leave the element unchanged,
// so this equals the row-wise update of the touched rows
__global__ void __launch_bounds__(256)
adagrad_dense_kernel(float* __restrict__ W, float* __restrict__ S, const float* __restrict__ G, int64_t n,
                     float lr, float eps) {
    const int64_t nth = static_cast<int64_t>(gridDim.x) * blockDim.x;
    for (int64_t k = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; k < n; k += nth) {
        const float g = G[k];
        if (g != 0.f) {
            const float sv = S[k] + g * g;
            S[k] = sv;
            W[k] -= lr * g / (sqrtf(sv) + eps);
        }
    }
}

// ---- owner update of the received gradient rows (slb_shard_rows_adagrad, slb_shard_rows_adam) ----
// local_ids entries outside [0, rows) are padding slots: neither counted nor placed.
__global__ void __launch_bounds__(256)
rows_count_kernel(const int64_t* __restrict__ ids, int64_t R, int64_t rows, SegIndex seg) {
    if (blockIdx.x == 0 && threadIdx.x == 0) seg.totals[3] = 0;     // hot-row list of this call
    const int64_t nth = static_cast<int64_t>(gridDim.x) * blockDim.x;
    for (int64_t t = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; t < R; t += nth) {
        const int64_t r = ids[t];
        if (r >= 0 && r < rows) atomicAdd(seg.cnt + r, 1);
    }
}

__global__ void __launch_bounds__(256)
rows_fill_kernel(const int64_t* __restrict__ ids, int64_t R, int64_t rows, SegIndex seg) {
    const int64_t nth = static_cast<int64_t>(gridDim.x) * blockDim.x;
    for (int64_t t = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; t < R; t += nth) {
        const int64_t r = ids[t];
        if (r >= 0 && r < rows) seg_place(seg, r, static_cast<int32_t>(t));
    }
}

// One group of LPR lanes per distinct row: the row's contributions in ascending position (= peer
// rank) order, then the shared row-wise Adagrad step on the row and its bias.  Hot rows (longer
// than the group's sort capacity: padding-heavy exchanges) were pre-sorted by seg_sort_long_kernel.
template <int LPR, bool VEC4>
__global__ void __launch_bounds__(256, 4)
rows_adagrad_kernel(const float* __restrict__ g_rows, const float* __restrict__ g_bias, int D, SegIndex seg,
                    OptV2 o, float* __restrict__ W, float* __restrict__ S, float* __restrict__ b,
                    float* __restrict__ sb) {
    constexpr int GROUPS = 256 / LPR;
    constexpr int CAP = seg_sort_cap(LPR);
    constexpr int STEP = VEC4 ? 4 : 1;
    __shared__ int32_t sh_sort[GROUPS * 2 * CAP];
    const int gl = threadIdx.x & (LPR - 1);
    const int gib = threadIdx.x / LPR;
    const unsigned gmask = group_mask(LPR);
    int32_t* sh = sh_sort + gib * 2 * CAP;
    const int nseg = seg.totals[0];
    for (int64_t s = static_cast<int64_t>(blockIdx.x) * GROUPS + gib; s < nseg;
         s += static_cast<int64_t>(gridDim.x) * GROUPS) {
        const int start = seg.seg_start[s];
        const int len = seg.seg_start[s + 1] - start;
        const int64_t row = seg.seg_row[s];
        float gb = 0.f;
        for (int c0 = 0; c0 < D; c0 += LPR * STEP) {
            const int c = c0 + gl * STEP;
            float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
            seg_visit_sorted<LPR>(seg.members, start, len, gl, gmask, sh, [&](int32_t t) {
                const float* src = g_rows + static_cast<int64_t>(t) * D;
                if (c0 == 0) gb += __ldg(g_bias + t);
                if (c < D) {
                    if (VEC4) {
                        const float4 v = ldg4(src + c);
                        acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w;
                    } else {
                        acc.x += __ldg(src + c);
                    }
                }
            }, true);
            if (c < D) {
                float* w = W + row * D + c;
                float* st = S + row * D + c;
                if (VEC4) {
                    float4 w4 = ld4(w), s4 = ld4(st);
                    row_update(o, w4, s4, acc);
                    st4(w, w4);
                    st4(st, s4);
                } else {
                    bias_update(o, w, st, acc.x);
                }
            }
        }
        if (gl == 0) bias_update(o, b + row, sb + row, gb);
    }
}

// Lazy-exact Adam, before the owner gathers the requested rows of step t: every requested row and
// its bias are brought current through step t - 1 (dense Adam moved them at every step they
// missed, and the peers' forward must see that).  A row can be requested by several peers, so
// atomicMax on last[row] elects one lane group per distinct row, as mf_adam_prepass_kernel does;
// the others find it current and read nothing.  A kernel of its own ahead of the gather: a gather
// fused into it would let a losing group read a row the elected group is still writing.
template <int LPR, bool VEC4>
__global__ void __launch_bounds__(256)
rows_adam_catch_up_kernel(const int64_t* __restrict__ ids, int64_t R, int64_t rows, int D, AdamDev o,
                          float* __restrict__ W, float* __restrict__ M, float* __restrict__ V, float* __restrict__ b,
                          float* __restrict__ bm, float* __restrict__ bv, int32_t* __restrict__ last) {
    constexpr int GROUPS = 256 / LPR;
    constexpr int STEP = VEC4 ? 4 : 1;
    const int gl = threadIdx.x & (LPR - 1);
    const unsigned gmask = group_mask(LPR);
    const int upto = o.t - 1;
    for (int64_t k = static_cast<int64_t>(blockIdx.x) * GROUPS + threadIdx.x / LPR; k < R;
         k += static_cast<int64_t>(gridDim.x) * GROUPS) {
        const int64_t row = ids[k];
        if (row < 0 || row >= rows) continue;                 // padding slot (group-uniform)
        int old = 0;
        if (gl == 0) old = atomicMax(last + row, upto);
        old = __shfl_sync(gmask, old, (threadIdx.x & 31) & ~(LPR - 1));
        if (old >= upto) continue;
        for (int c = gl * STEP; c < D; c += LPR * STEP) {
            const int64_t e = row * D + c;
            if (VEC4) {
                float4 w = ld4(W + e), m = ld4(M + e), v = ld4(V + e);
                adam_catch_up(o, old, upto, w, m, v);
                st4(W + e, w); st4(M + e, m); st4(V + e, v);
            } else {
                float w = W[e], m = M[e], v = V[e];
                adam_catch_up1(o, old, upto, w, m, v);
                W[e] = w; M[e] = m; V[e] = v;
            }
        }
        if (gl == 0) {
            float w = b[row], m = bm[row], v = bv[row];
            adam_catch_up1(o, old, upto, w, m, v);
            b[row] = w; bm[row] = m; bv[row] = v;
        }
    }
}

// Adam step t on each distinct received row: the segment sum of rows_adagrad_kernel (rank order, no
// float atomics), then the step on the row and its bias, which share last[row] (= t afterwards).
// Every received row takes the step, also one whose summed gradient is zero: that step is exactly
// the catch-up the row would get later.  A row not yet current through t - 1 (an apply without the
// catch-up ahead of it) is caught up first, as mf_adam_apply_kernel does.  (A kernel of its own, so
// that rows_adagrad_kernel keeps its code.)
template <int LPR, bool VEC4>
__global__ void __launch_bounds__(256, 4)
rows_adam_kernel(const float* __restrict__ g_rows, const float* __restrict__ g_bias, int D, SegIndex seg, AdamDev o,
                 float* __restrict__ W, float* __restrict__ M, float* __restrict__ V, float* __restrict__ b,
                 float* __restrict__ bm, float* __restrict__ bv, int32_t* __restrict__ last) {
    constexpr int GROUPS = 256 / LPR;
    constexpr int CAP = seg_sort_cap(LPR);
    constexpr int STEP = VEC4 ? 4 : 1;
    __shared__ int32_t sh_sort[GROUPS * 2 * CAP];
    const int gl = threadIdx.x & (LPR - 1);
    const int gib = threadIdx.x / LPR;
    const unsigned gmask = group_mask(LPR);
    int32_t* sh = sh_sort + gib * 2 * CAP;
    const int nseg = seg.totals[0];
    const float ss = __ldg(o.sched + 2 * o.t), bc = __ldg(o.sched + 2 * o.t + 1);
    for (int64_t s = static_cast<int64_t>(blockIdx.x) * GROUPS + gib; s < nseg;
         s += static_cast<int64_t>(gridDim.x) * GROUPS) {
        const int start = seg.seg_start[s];
        const int len = seg.seg_start[s + 1] - start;
        const int64_t row = seg.seg_row[s];
        const int lastv = last[row];
        float gb = 0.f;
        for (int c0 = 0; c0 < D; c0 += LPR * STEP) {
            const int c = c0 + gl * STEP;
            float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
            seg_visit_sorted<LPR>(seg.members, start, len, gl, gmask, sh, [&](int32_t t) {
                const float* src = g_rows + static_cast<int64_t>(t) * D;
                if (c0 == 0) gb += __ldg(g_bias + t);
                if (c < D) {
                    if (VEC4) {
                        const float4 v = ldg4(src + c);
                        acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w;
                    } else {
                        acc.x += __ldg(src + c);
                    }
                }
            }, true);
            if (c < D) {
                const int64_t e = row * D + c;
                if (VEC4) {
                    float4 w = ld4(W + e), m = ld4(M + e), v = ld4(V + e);
                    adam_catch_up(o, lastv, o.t - 1, w, m, v);
                    adam_elem(o, ss, bc, acc.x, w.x, m.x, v.x);
                    adam_elem(o, ss, bc, acc.y, w.y, m.y, v.y);
                    adam_elem(o, ss, bc, acc.z, w.z, m.z, v.z);
                    adam_elem(o, ss, bc, acc.w, w.w, m.w, v.w);
                    st4(W + e, w); st4(M + e, m); st4(V + e, v);
                } else {
                    float w = W[e], m = M[e], v = V[e];
                    adam_catch_up1(o, lastv, o.t - 1, w, m, v);
                    adam_elem(o, ss, bc, acc.x, w, m, v);
                    W[e] = w; M[e] = m; V[e] = v;
                }
            }
        }
        __syncwarp(gmask);                    // every lane has read last[row] before it moves
        if (gl == 0) {
            float w = b[row], m = bm[row], v = bv[row];
            adam_catch_up1(o, lastv, o.t - 1, w, m, v);
            adam_elem(o, ss, bc, gb, w, m, v);
            b[row] = w; bm[row] = m; bv[row] = v;
            last[row] = o.t;
        }
    }
}

struct RowsLayout { SegIndex seg; size_t bytes; };

RowsLayout rows_layout(void* base, int64_t R, int64_t rows) {
    WsCarver ws(base);
    RowsLayout l;
    l.seg = seg_index_carve(ws, rows, R);
    l.bytes = ws.bytes();
    return l;
}

bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }

// The segment index of the received rows (distinct shard rows ascending, each with its positions
// in local_ids), shared by both owner updates; hot rows (more than seg_sort_cap(lpr) positions) are
// pre-sorted.
int rows_index(const int64_t* local_ids, int64_t R, int64_t rows, int lpr, RowsLayout& l, cudaStream_t st) {
    l.seg.long_cap = seg_sort_cap(lpr);
    const int g1 = slb_grid((R + 255) / 256, 8);
    rows_count_kernel<<<g1, 256, 0, st>>>(local_ids, R, rows, l.seg);
    SLB_LAUNCH_CHECK("rows_count_kernel");
    seg_scan_launch(l.seg, rows, st);
    SLB_LAUNCH_CHECK("seg_scan_kernel");
    rows_fill_kernel<<<g1, 256, 0, st>>>(local_ids, R, rows, l.seg);
    SLB_LAUNCH_CHECK("rows_fill_kernel");
    seg_sort_long_kernel<<<SEG_LONG_CTAS, 256, 0, st>>>(l.seg);     // no-op unless hot rows exist
    SLB_LAUNCH_CHECK("seg_sort_long_kernel");
    return SLB_OK;
}

struct UqLayout { int32_t* flags; SegIndex seg; size_t bytes; };

UqLayout uq_layout(void* base, int64_t n, int64_t rows) {
    WsCarver ws(base);
    UqLayout l;
    l.flags = ws.take<int32_t>(8);
    l.seg = seg_index_carve(ws, rows, n < rows ? n : rows);
    l.bytes = ws.bytes();
    return l;
}

}  // namespace

extern "C" {

size_t slb_unique_workspace_bytes(int64_t n, int64_t rows) { return uq_layout(nullptr, n, rows).bytes; }

int slb_unique_bucket(const int64_t* ids, int64_t n, int64_t rows, int64_t chunk, int32_t nparts,
                      int64_t* uniq, int64_t* inverse, int64_t* counts_out, void* workspace,
                      size_t workspace_bytes, slb_stream_t stream) {
    SLB_REQUIRE(ids && uniq && inverse && counts_out && workspace, "unique_bucket: null pointer");
    SLB_REQUIRE(n > 0 && rows > 0 && chunk > 0 && nparts >= 1, "unique_bucket: bad sizes");
    SLB_REQUIRE(chunk * nparts >= rows, "unique_bucket: chunk * nparts must cover the row space");
    SLB_REQUIRE(rows < (1ll << 31) - SEG_SCAN_TILE && n < (1ll << 31), "unique_bucket: too large");
    UqLayout l = uq_layout(workspace, n, rows);
    if (workspace_bytes < l.bytes) {
        slb_set_error("unique_bucket: workspace too small (%zu < %zu)", workspace_bytes, l.bytes);
        return SLB_ENOSPC;
    }
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const int sms = slb_sms();
    int g = static_cast<int>((n + 255) / 256);
    if (g > sms * 8) g = sms * 8;
    uq_count_kernel<<<g, 256, 0, st>>>(ids, n, rows, l.seg, l.flags + 4);
    SLB_LAUNCH_CHECK("uq_count_kernel");
    seg_scan_launch(l.seg, l.seg.Rpad, st);
    SLB_LAUNCH_CHECK("seg_scan_kernel");
    uq_emit_kernel<<<g, 256, 0, st>>>(l.seg, chunk, nparts, uniq, counts_out);
    SLB_LAUNCH_CHECK("uq_emit_kernel");
    uq_inverse_kernel<<<g, 256, 0, st>>>(ids, n, rows, l.seg, inverse);
    SLB_LAUNCH_CHECK("uq_inverse_kernel");
    return SLB_OK;
}

int slb_shard_gather_batch(const int64_t* pos, int64_t m, const int64_t* users, const int64_t* items,
                           const int64_t* negs, int64_t neg_base, int32_t n_neg, int64_t user_lo,
                           int64_t* users_out, int64_t* items_out, int64_t* negs_out, slb_stream_t stream) {
    if (m <= 0) return SLB_OK;
    SLB_REQUIRE(pos && users && items && negs && users_out && items_out && negs_out && n_neg >= 1,
                "shard_gather_batch: bad arguments");
    int g = static_cast<int>((m + 255) / 256);
    if (g > slb_sms() * 8) g = slb_sms() * 8;
    shard_gather_batch_kernel<<<g, 256, 0, static_cast<cudaStream_t>(stream)>>>(pos, m, users, items, negs, neg_base,
                                                                               n_neg, user_lo, users_out, items_out, negs_out);
    SLB_LAUNCH_CHECK("shard_gather_batch_kernel");
    return SLB_OK;
}

int slb_adagrad_dense(float* W, float* state, const float* grad, int64_t n, float lr, float eps,
                      slb_stream_t stream) {
    if (n <= 0) return SLB_OK;
    SLB_REQUIRE(W && state && grad, "adagrad_dense: null pointer");
    int g = static_cast<int>((n + 255) / 256);
    if (g > slb_sms() * 16) g = slb_sms() * 16;
    adagrad_dense_kernel<<<g, 256, 0, static_cast<cudaStream_t>(stream)>>>(W, state, grad, n, lr, eps);
    SLB_LAUNCH_CHECK("adagrad_dense_kernel");
    return SLB_OK;
}

size_t slb_shard_rows_workspace_bytes(int64_t R, int64_t rows) {
    return rows_layout(nullptr, R > 0 ? R : 0, rows > 0 ? rows : 1).bytes;
}

int slb_shard_rows_adagrad(const int64_t* local_ids, const float* g_rows, const float* g_bias, int64_t R,
                           float* W, float* state_W, float* b, float* state_b, int64_t rows, int32_t dim,
                           float lr, float eps, void* workspace, size_t workspace_bytes, slb_stream_t stream) {
    SLB_REQUIRE(R >= 0 && rows >= 0 && dim >= 1, "shard_rows_adagrad: bad sizes");
    if (R == 0) return SLB_OK;          // nothing arrived: the received tensors may have no storage
    SLB_REQUIRE(local_ids && g_rows && g_bias && W && state_W && b && state_b && workspace,
                "shard_rows_adagrad: null pointer");
    SLB_REQUIRE(rows >= 1, "shard_rows_adagrad: rows arrived for an empty shard");
    SLB_REQUIRE(R < (1ll << 31) && rows < (1ll << 31) - SEG_SCAN_TILE && dim < (1 << 28),
                "shard_rows_adagrad: too large");
    RowsLayout l = rows_layout(workspace, R, rows);
    if (workspace_bytes < l.bytes) {
        slb_set_error("shard_rows_adagrad: workspace too small (%zu < %zu)", workspace_bytes, l.bytes);
        return SLB_ENOSPC;
    }
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const bool vec4 = dim % 4 == 0 && aligned16(g_rows) && aligned16(W) && aligned16(state_W);
    // lanes per row: one float4 (or one float) per lane, a power of two up to a warp
    const int lpr = lpr_for_dim(vec4 ? dim : 4 * dim);
    const int rc = rows_index(local_ids, R, rows, lpr, l, st);
    if (rc != SLB_OK) return rc;
    const OptV2 o = {SLB_OPT_ADAGRAD, lr, 0.f, eps};
    const int grid = slb_grid((R + 256 / lpr - 1) / (256 / lpr), 8);
    with_bool(vec4, [&](auto V) {
        with_lpr(lpr, [&](auto L) {
            rows_adagrad_kernel<L, V><<<grid, 256, 0, st>>>(g_rows, g_bias, dim, l.seg, o, W, state_W, b, state_b);
        });
    });
    SLB_LAUNCH_CHECK("rows_adagrad_kernel");
    return SLB_OK;
}

int slb_shard_rows_adam_catch_up(const int64_t* local_ids, int64_t R, float* W, float* exp_avg, float* exp_avg_sq,
                                 float* b, float* b_avg, float* b_avg_sq, int32_t* last, int64_t rows, int32_t dim,
                                 const float* sched, int64_t step, float beta1, float beta2, float one_minus_beta1,
                                 float one_minus_beta2, float eps, float weight_decay, slb_stream_t stream) {
    SLB_REQUIRE(R >= 0 && rows >= 0 && dim >= 1 && step >= 1 && step < (1ll << 31),
                "shard_rows_adam_catch_up: bad sizes");
    if (R == 0) return SLB_OK;
    SLB_REQUIRE(local_ids && W && exp_avg && exp_avg_sq && b && b_avg && b_avg_sq && last && sched,
                "shard_rows_adam_catch_up: null pointer");
    SLB_REQUIRE(rows >= 1, "shard_rows_adam_catch_up: rows requested from an empty shard");
    SLB_REQUIRE(R < (1ll << 31) && rows < (1ll << 31) && dim < (1 << 28), "shard_rows_adam_catch_up: too large");
    if (step == 1) return SLB_OK;       // nothing pending before the first step
    const AdamDev o = {beta1, beta2, one_minus_beta1, one_minus_beta2, eps, weight_decay, sched,
                       static_cast<int32_t>(step)};
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const bool vec4 = dim % 4 == 0 && aligned16(W) && aligned16(exp_avg) && aligned16(exp_avg_sq);
    const int lpr = lpr_for_dim(vec4 ? dim : 4 * dim);
    const int grid = slb_grid((R + 256 / lpr - 1) / (256 / lpr), 8);
    with_bool(vec4, [&](auto V) {
        with_lpr(lpr, [&](auto L) {
            rows_adam_catch_up_kernel<L, V><<<grid, 256, 0, st>>>(local_ids, R, rows, dim, o, W, exp_avg, exp_avg_sq,
                                                                 b, b_avg, b_avg_sq, last);
        });
    });
    SLB_LAUNCH_CHECK("rows_adam_catch_up_kernel");
    return SLB_OK;
}

int slb_shard_rows_adam(const int64_t* local_ids, const float* g_rows, const float* g_bias, int64_t R, float* W,
                        float* exp_avg, float* exp_avg_sq, float* b, float* b_avg, float* b_avg_sq, int32_t* last,
                        int64_t rows, int32_t dim, const float* sched, int64_t step, float beta1, float beta2,
                        float one_minus_beta1, float one_minus_beta2, float eps, float weight_decay, void* workspace,
                        size_t workspace_bytes, slb_stream_t stream) {
    SLB_REQUIRE(R >= 0 && rows >= 0 && dim >= 1 && step >= 1 && step < (1ll << 31), "shard_rows_adam: bad sizes");
    if (R == 0) return SLB_OK;          // nothing arrived: the received tensors may have no storage
    SLB_REQUIRE(local_ids && g_rows && g_bias && W && exp_avg && exp_avg_sq && b && b_avg && b_avg_sq && last &&
                sched && workspace, "shard_rows_adam: null pointer");
    SLB_REQUIRE(rows >= 1, "shard_rows_adam: rows arrived for an empty shard");
    SLB_REQUIRE(R < (1ll << 31) && rows < (1ll << 31) - SEG_SCAN_TILE && dim < (1 << 28),
                "shard_rows_adam: too large");
    RowsLayout l = rows_layout(workspace, R, rows);
    if (workspace_bytes < l.bytes) {
        slb_set_error("shard_rows_adam: workspace too small (%zu < %zu)", workspace_bytes, l.bytes);
        return SLB_ENOSPC;
    }
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const bool vec4 = dim % 4 == 0 && aligned16(g_rows) && aligned16(W) && aligned16(exp_avg) &&
                      aligned16(exp_avg_sq);
    const int lpr = lpr_for_dim(vec4 ? dim : 4 * dim);
    const int rc = rows_index(local_ids, R, rows, lpr, l, st);
    if (rc != SLB_OK) return rc;
    const AdamDev o = {beta1, beta2, one_minus_beta1, one_minus_beta2, eps, weight_decay, sched,
                       static_cast<int32_t>(step)};
    const int grid = slb_grid((R + 256 / lpr - 1) / (256 / lpr), 8);
    with_bool(vec4, [&](auto V) {
        with_lpr(lpr, [&](auto L) {
            rows_adam_kernel<L, V><<<grid, 256, 0, st>>>(g_rows, g_bias, dim, l.seg, o, W, exp_avg, exp_avg_sq, b,
                                                        b_avg, b_avg_sq, last);
        });
    });
    SLB_LAUNCH_CHECK("rows_adam_kernel");
    return SLB_OK;
}

}  // extern "C"
