// Data preparation on the device, in front of fit():
//   - the stable (user, timestamp) order of Interactions.to_sequence
//     (spotlight/interactions.py:233-238, np.lexsort) as an LSD radix sort of the original index,
//     the per-user window counts and the left-padded window rows (interactions.py:240-262);
//   - the stable train/test partition of user_based_train_test_split
//     (spotlight/cross_validation.py:143-174).
//
// Every ordering step is one stable partition pass: per-tile digit histograms, an exclusive
// scan over (digit, tile), and a scatter that ranks each element among the equal digits before
// it in index order (warp match + per-warp running counts).  Integer-only, no atomics whose
// order matters, so the outputs are deterministic and equal to the host code's.
#include "common.cuh"
#include "scan.cuh"

namespace {

constexpr int PT_THREADS = 256, PT_WARPS = PT_THREADS / 32, PT_ROUNDS = 8;
constexpr int PT_TILE = PT_WARPS * PT_ROUNDS * 32;        // elements per tile; warp w owns a 256-run

// ---- digit functors: digit of the element whose payload (original position) is src ---------
struct RadixDigit {           // 8-bit digit of (key - kmin)
    const uint64_t* key;
    uint64_t kmin;
    int shift;
    __device__ __forceinline__ int operator()(int32_t src) const {
        return static_cast<int>(((key[src] - kmin) >> shift) & 0xFFu);
    }
};

struct SplitDigit {           // 1 = test: mask[murmur3_32(uid, seed) % 100]
    const int32_t* uid;
    uint32_t seed;
    uint64_t mask_lo, mask_hi;
    __device__ __forceinline__ int operator()(int32_t src) const {
        const uint32_t r = murmur3_32(static_cast<uint32_t>(uid[src]), seed) % 100u;
        return static_cast<int>((r < 64 ? mask_lo >> r : mask_hi >> (r - 64)) & 1u);
    }
};

struct HeadDigit {            // 1 where sorted position i starts a new user
    const uint64_t* ukey;
    const int32_t* order;
    __device__ __forceinline__ int operator()(int32_t i) const {
        return i == 0 || ukey[order[i]] != ukey[order[i - 1]];
    }
};

// hist[d * ntiles + tile] = elements of the tile with digit d
template <int RADIX, class F>
__global__ void __launch_bounds__(PT_THREADS)
pt_count_kernel(F f, const int32_t* __restrict__ idx, int32_t n, int ntiles, int32_t* __restrict__ hist) {
    __shared__ int cnt[RADIX];
    for (int d = threadIdx.x; d < RADIX; d += PT_THREADS) cnt[d] = 0;
    __syncthreads();
    const int64_t base = static_cast<int64_t>(blockIdx.x) * PT_TILE;
    for (int k = threadIdx.x; k < PT_TILE; k += PT_THREADS) {
        const int64_t i = base + k;
        if (i < n) atomicAdd(&cnt[f(idx ? idx[i] : static_cast<int32_t>(i))], 1);
    }
    __syncthreads();
    for (int d = threadIdx.x; d < RADIX; d += PT_THREADS) hist[static_cast<int64_t>(d) * ntiles + blockIdx.x] = cnt[d];
}

// out[off[d, tile] + (equal digits before it in the tile)] = payload: a stable scatter
template <int RADIX, class F>
__global__ void __launch_bounds__(PT_THREADS)
pt_scatter_kernel(F f, const int32_t* __restrict__ idx, int32_t n, int ntiles, const int32_t* __restrict__ off,
                  int32_t* __restrict__ out) {
    __shared__ int wbase[PT_WARPS][RADIX];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (int k = threadIdx.x; k < PT_WARPS * RADIX; k += PT_THREADS) (&wbase[0][0])[k] = 0;
    __syncthreads();
    const int64_t first = static_cast<int64_t>(blockIdx.x) * PT_TILE + warp * (PT_ROUNDS * 32);
    const unsigned lt = (1u << lane) - 1u;
    int dig[PT_ROUNDS];
    int32_t pay[PT_ROUNDS];
    // pass 1: per-warp digit counts (the warp's rounds run in index order)
#pragma unroll
    for (int r = 0; r < PT_ROUNDS; ++r) {
        const int64_t i = first + r * 32 + lane;
        pay[r] = i < n ? (idx ? idx[i] : static_cast<int32_t>(i)) : 0;
        dig[r] = i < n ? f(pay[r]) : RADIX;
        const unsigned peers = __match_any_sync(0xffffffffu, dig[r]);
        if (dig[r] < RADIX && (peers & lt) == 0) wbase[warp][dig[r]] += __popc(peers);
        __syncwarp();
    }
    __syncthreads();
    // warp bases: the tile's global offset plus the counts of the warps before
    for (int d = threadIdx.x; d < RADIX; d += PT_THREADS) {
        int s = off[static_cast<int64_t>(d) * ntiles + blockIdx.x];
#pragma unroll
        for (int w = 0; w < PT_WARPS; ++w) {
            const int c = wbase[w][d];
            wbase[w][d] = s;
            s += c;
        }
    }
    __syncthreads();
    // pass 2: rank within the round, write, advance the warp's base
#pragma unroll
    for (int r = 0; r < PT_ROUNDS; ++r) {
        const unsigned peers = __match_any_sync(0xffffffffu, dig[r]);
        const bool valid = dig[r] < RADIX;
        if (valid) out[wbase[warp][dig[r]] + __popc(peers & lt)] = pay[r];
        __syncwarp();
        if (valid && (peers & lt) == 0) wbase[warp][dig[r]] += __popc(peers);
        __syncwarp();
    }
}

struct PtLayout {
    int ntiles;
    int32_t *hist, *off, *tsum, *tmp;
    size_t bytes;
};

// hist[RADIX * ntiles], off[RADIX * ntiles + 1] (exclusive scan, total last), tsum (tile sums of
// a scan of up to max(RADIX * ntiles, n) values), and `extra` int32 for the caller
PtLayout pt_layout(void* ws, int64_t n, int radix, int64_t extra) {
    PtLayout l;
    WsCarver c(ws);
    l.ntiles = static_cast<int>((n + PT_TILE - 1) / PT_TILE);
    const int64_t m = static_cast<int64_t>(radix) * l.ntiles;
    l.hist = c.take<int32_t>(m);
    l.off = c.take<int32_t>(m + 1);
    l.tsum = c.take<int32_t>(scan_tiles_for(m > n ? m : n) + 1);
    l.tmp = c.take<int32_t>(extra);
    l.bytes = c.bytes();
    return l;
}

// exclusive scan of x[0..m) into off[0..m], off[m] = total
int excl_scan(const int32_t* x, int64_t m, int32_t* off, int32_t* tsum, cudaStream_t st) {
    if (cudaMemsetAsync(off, 0, sizeof(int32_t), st) != cudaSuccess) {
        slb_set_error("prepare: memset failed");
        return SLB_ECUDA;
    }
    if (m == 0) return SLB_OK;
    const int nt = scan_tiles_for(m);
    scan_tilesum_kernel<<<nt, SC_THREADS, 0, st>>>(x, m, tsum);
    scan_tiles_kernel<<<1, 1024, 0, st>>>(tsum, nt);
    scan_apply_kernel<<<nt, SC_THREADS, 0, st>>>(x, m, tsum, off + 1);
    SLB_LAUNCH_CHECK("scan kernels");
    return SLB_OK;
}

// One stable pass: out = the payloads (idx[i], or i when idx is null) ordered by digit, ties in
// index order.  bucket1 (optional, device int32): where digit 1 starts in out.
template <int RADIX, class F>
int pt_pass(F f, const int32_t* idx, int32_t n, int32_t* out, const PtLayout& l, int32_t* bucket1,
            cudaStream_t st) {
    pt_count_kernel<RADIX><<<l.ntiles, PT_THREADS, 0, st>>>(f, idx, n, l.ntiles, l.hist);
    SLB_LAUNCH_CHECK("pt_count_kernel");
    const int rc = excl_scan(l.hist, static_cast<int64_t>(RADIX) * l.ntiles, l.off, l.tsum, st);
    if (rc != SLB_OK) return rc;
    pt_scatter_kernel<RADIX><<<l.ntiles, PT_THREADS, 0, st>>>(f, idx, n, l.ntiles, l.off, out);
    SLB_LAUNCH_CHECK("pt_scatter_kernel");
    if (bucket1 && cudaMemcpyAsync(bucket1, l.off + l.ntiles, sizeof(int32_t), cudaMemcpyDeviceToDevice,
                                   st) != cudaSuccess) {
        slb_set_error("prepare: copy failed");
        return SLB_ECUDA;
    }
    return SLB_OK;
}

unsigned pr_grid(int64_t n, int threads) {
    const int64_t want = (n + threads - 1) / threads;
    const int64_t cap = static_cast<int64_t>(slb_sms()) * 16;
    return static_cast<unsigned>(want < 1 ? 1 : (want < cap ? want : cap));
}

__device__ __forceinline__ int64_t load_id(const void* p, int bytes, int64_t i) {
    return bytes == 8 ? static_cast<const int64_t*>(p)[i] : static_cast<const int32_t*>(p)[i];
}

// ---- order-preserving unsigned keys -----------------------------------------------------------
// ints: flip the sign bit of the int64 value.  floats (float32 widens exactly): the IEEE flip,
// with -0.0 folded onto +0.0 and every NaN on the largest key, as np.lexsort orders them.
__device__ __forceinline__ uint64_t int_key(int64_t v) {
    return static_cast<uint64_t>(v) ^ (uint64_t(1) << 63);
}
__device__ __forceinline__ uint64_t float_key(double v) {
    if (v != v) return ~uint64_t(0);
    if (v == 0.0) return uint64_t(1) << 63;
    const uint64_t b = static_cast<uint64_t>(__double_as_longlong(v));
    return (b >> 63) ? ~b : (b | (uint64_t(1) << 63));
}

__device__ __forceinline__ void minmax_warp(uint64_t& lo, uint64_t& hi) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const uint64_t a = __shfl_xor_sync(0xffffffffu, lo, o), b = __shfl_xor_sync(0xffffffffu, hi, o);
        lo = a < lo ? a : lo;
        hi = b > hi ? b : hi;
    }
}

__global__ void range_init_kernel(uint64_t* range) {
    range[0] = range[2] = ~uint64_t(0);
    range[1] = range[3] = 0;
}

__global__ void __launch_bounds__(256)
sort_keys_kernel(const void* __restrict__ users, int user_bytes, const void* __restrict__ ts, int ts_kind,
                 int64_t n, uint64_t* __restrict__ ukey, uint64_t* __restrict__ tkey, uint64_t* range) {
    uint64_t ulo = ~uint64_t(0), uhi = 0, tlo = ~uint64_t(0), thi = 0;
    for (int64_t i = blockIdx.x * int64_t(blockDim.x) + threadIdx.x; i < n; i += int64_t(gridDim.x) * blockDim.x) {
        const uint64_t u = int_key(load_id(users, user_bytes, i));
        uint64_t t;
        switch (ts_kind) {
            case SLB_TS_INT32: t = int_key(static_cast<const int32_t*>(ts)[i]); break;
            case SLB_TS_INT64: t = int_key(static_cast<const int64_t*>(ts)[i]); break;
            case SLB_TS_FLOAT32: t = float_key(static_cast<const float*>(ts)[i]); break;
            default: t = float_key(static_cast<const double*>(ts)[i]); break;
        }
        ukey[i] = u;
        tkey[i] = t;
        ulo = u < ulo ? u : ulo;
        uhi = u > uhi ? u : uhi;
        tlo = t < tlo ? t : tlo;
        thi = t > thi ? t : thi;
    }
    minmax_warp(ulo, uhi);
    minmax_warp(tlo, thi);
    if ((threadIdx.x & 31) == 0) {            // min / max: the result does not depend on the order
        atomicMin(reinterpret_cast<unsigned long long*>(range + 0), ulo);
        atomicMax(reinterpret_cast<unsigned long long*>(range + 1), uhi);
        atomicMin(reinterpret_cast<unsigned long long*>(range + 2), tlo);
        atomicMax(reinterpret_cast<unsigned long long*>(range + 3), thi);
    }
}

__global__ void iota_kernel(int32_t* out, int32_t n) {
    for (int64_t i = blockIdx.x * int64_t(blockDim.x) + threadIdx.x; i < n; i += int64_t(gridDim.x) * blockDim.x)
        out[i] = static_cast<int32_t>(i);
}

// ---- windows -----------------------------------------------------------------------------------
// heads[n0 .. n) are the first sorted positions of the users (ascending).
// For user k: c interactions, w = ceil(c / step) windows, of which the `kept` newest survive the
// min_sequence_length filter (need < 0: no filter).
__global__ void __launch_bounds__(256)
window_counts_kernel(const int32_t* __restrict__ heads, const int32_t* __restrict__ n0p, int32_t n, int64_t step,
                     int64_t need, int32_t* __restrict__ starts, int32_t* __restrict__ kept,
                     int32_t* __restrict__ num_users) {
    const int32_t n0 = *n0p, U = n - n0;
    for (int64_t k = blockIdx.x * int64_t(blockDim.x) + threadIdx.x; k <= n; k += int64_t(gridDim.x) * blockDim.x) {
        if (k == 0) *num_users = U;
        if (k < U) {
            const int64_t s = heads[n0 + k], c = (k + 1 < U ? heads[n0 + k + 1] : n) - s;
            const int64_t w = (c + step - 1) / step;
            int64_t keep = w;
            if (need >= 0) keep = c >= need ? min(w, (c - need) / step + 1) : 0;
            starts[k] = static_cast<int32_t>(s);
            kept[k] = static_cast<int32_t>(keep);
        } else {
            if (k == U) starts[k] = n;
            if (k < n) kept[k] = 0;
        }
    }
}

// One warp per output row: row r of user k (row_offs[k] <= r < row_offs[k + 1]) is the user's
// window rank = r - row_offs[k], ending (exclusive) at c - rank * step and left-padded with 0.
__global__ void __launch_bounds__(256)
sequence_emit_kernel(const int32_t* __restrict__ order, const void* __restrict__ users, int user_bytes,
                     const void* __restrict__ items, int item_bytes, const int32_t* __restrict__ starts,
                     const int32_t* __restrict__ row_offs, int32_t U, int64_t rows, int32_t L, int64_t step,
                     int32_t* __restrict__ seqs, int32_t* __restrict__ seq_users) {
    const int lane = threadIdx.x & 31;
    const int64_t r = (blockIdx.x * int64_t(blockDim.x) + threadIdx.x) >> 5;
    if (r >= rows) return;
    int lo = 0, hi = U - 1;                   // last k with row_offs[k] <= r
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (row_offs[mid] <= r) lo = mid; else hi = mid - 1;
    }
    const int64_t s = starts[lo], c = starts[lo + 1] - s;
    const int64_t end = c - (r - row_offs[lo]) * step;
    int32_t* row = seqs + r * L;
    for (int j = lane; j < L; j += 32) {
        const int64_t src = end - L + j;
        row[j] = src >= 0 ? static_cast<int32_t>(load_id(items, item_bytes, order[s + src])) : 0;
    }
    if (lane == 0) seq_users[r] = static_cast<int32_t>(load_id(users, user_bytes, order[s]));
}

template <typename I, typename T>
__global__ void __launch_bounds__(256)
gather_kernel(const I* __restrict__ index, int64_t n, const T* __restrict__ src, T* __restrict__ dst) {
    for (int64_t i = blockIdx.x * int64_t(blockDim.x) + threadIdx.x; i < n; i += int64_t(gridDim.x) * blockDim.x)
        dst[i] = src[index[i]];
}

template <typename I>
void gather_launch(const void* index, int64_t n, const void* src, int elem_bytes, void* dst, cudaStream_t st) {
    const I* ix = static_cast<const I*>(index);
    if (elem_bytes == 8)
        gather_kernel<<<pr_grid(n, 256), 256, 0, st>>>(ix, n, static_cast<const int64_t*>(src), static_cast<int64_t*>(dst));
    else
        gather_kernel<<<pr_grid(n, 256), 256, 0, st>>>(ix, n, static_cast<const int32_t*>(src), static_cast<int32_t*>(dst));
}

constexpr int64_t PR_MAX_N = (int64_t(1) << 31) - 1;

}  // namespace

extern "C" {

int slb_sort_keys(const void* users, int32_t user_bytes, const void* timestamps, int32_t ts_kind, int64_t n,
                  uint64_t* ukey, uint64_t* tkey, uint64_t* range, slb_stream_t stream) {
    SLB_REQUIRE(n >= 1 && n <= PR_MAX_N, "sort_keys: n must be in [1, 2^31)");
    SLB_REQUIRE(users && timestamps && ukey && tkey && range, "sort_keys: null pointer");
    SLB_REQUIRE(user_bytes == 4 || user_bytes == 8, "sort_keys: user ids must be int32 or int64");
    SLB_REQUIRE(ts_kind >= SLB_TS_INT32 && ts_kind <= SLB_TS_FLOAT64, "sort_keys: bad timestamp kind");
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    range_init_kernel<<<1, 1, 0, st>>>(range);
    sort_keys_kernel<<<pr_grid(n, 256), 256, 0, st>>>(users, user_bytes, timestamps, ts_kind, n, ukey, tkey, range);
    SLB_LAUNCH_CHECK("sort_keys_kernel");
    return SLB_OK;
}

size_t slb_radix_order_workspace_bytes(int64_t n) {
    if (n < 0 || n > PR_MAX_N) return 0;
    return pt_layout(nullptr, n, 256, n).bytes;
}

int slb_radix_order(const uint64_t* ukey, uint64_t umin, int32_t ubits, const uint64_t* tkey, uint64_t tmin,
                    int32_t tbits, int64_t n, int32_t* order, void* workspace, size_t workspace_bytes,
                    slb_stream_t stream) {
    SLB_REQUIRE(n >= 1 && n <= PR_MAX_N, "radix_order: n must be in [1, 2^31)");
    SLB_REQUIRE(order && workspace, "radix_order: null pointer");
    SLB_REQUIRE(ubits >= 0 && ubits <= 64 && tbits >= 0 && tbits <= 64, "radix_order: key bits must be in [0, 64]");
    SLB_REQUIRE((ukey || !ubits) && (tkey || !tbits), "radix_order: null key");
    PtLayout l = pt_layout(workspace, n, 256, n);
    if (l.bytes > workspace_bytes) {
        slb_set_error("radix_order: workspace too small");
        return SLB_ENOSPC;
    }
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const int tpass = (tbits + 7) / 8, passes = tpass + (ubits + 7) / 8;
    if (passes == 0) {
        iota_kernel<<<pr_grid(n, 256), 256, 0, st>>>(order, static_cast<int32_t>(n));
        SLB_LAUNCH_CHECK("iota_kernel");
        return SLB_OK;
    }
    // timestamp digits first, then user digits (LSD); the last pass lands in `order`
    const int32_t* in = nullptr;
    for (int p = 0; p < passes; ++p) {
        int32_t* out = ((passes - 1 - p) & 1) ? l.tmp : order;
        const RadixDigit f = p < tpass ? RadixDigit{tkey, tmin, 8 * p} : RadixDigit{ukey, umin, 8 * (p - tpass)};
        const int rc = pt_pass<256>(f, in, static_cast<int32_t>(n), out, l, nullptr, st);
        if (rc != SLB_OK) return rc;
        in = out;
    }
    return SLB_OK;
}

size_t slb_sequence_windows_workspace_bytes(int64_t n) {
    if (n < 0 || n > PR_MAX_N) return 0;
    return pt_layout(nullptr, n, 2, 2 * n + 1).bytes;
}

int slb_sequence_windows(const int32_t* order, const uint64_t* ukey, int64_t n, int64_t step, int64_t need,
                         int32_t* starts, int32_t* row_offs, int32_t* num_users, void* workspace,
                         size_t workspace_bytes, slb_stream_t stream) {
    SLB_REQUIRE(n >= 1 && n <= PR_MAX_N, "sequence_windows: n must be in [1, 2^31)");
    SLB_REQUIRE(order && ukey && starts && row_offs && num_users && workspace, "sequence_windows: null pointer");
    SLB_REQUIRE(step >= 1, "sequence_windows: step_size must be >= 1");
    PtLayout l = pt_layout(workspace, n, 2, 2 * n + 1);
    if (l.bytes > workspace_bytes) {
        slb_set_error("sequence_windows: workspace too small");
        return SLB_ENOSPC;
    }
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    int32_t* heads = l.tmp;                   // n: the non-heads, then the users' first positions
    int32_t* n0 = l.tmp + n;                  // where the heads start
    int32_t* kept = l.tmp + n + 1;            // n: kept windows per user, 0 past the last user
    const int32_t nn = static_cast<int32_t>(n);
    int rc = pt_pass<2>(HeadDigit{ukey, order}, nullptr, nn, heads, l, n0, st);
    if (rc != SLB_OK) return rc;
    window_counts_kernel<<<pr_grid(n + 1, 256), 256, 0, st>>>(heads, n0, nn, step, need, starts, kept, num_users);
    SLB_LAUNCH_CHECK("window_counts_kernel");
    return excl_scan(kept, n, row_offs, l.tsum, st);     // row_offs[n] = rows
}

int slb_sequence_emit(const int32_t* order, const void* users, int32_t user_bytes, const void* items,
                      int32_t item_bytes, const int32_t* starts, const int32_t* row_offs, int64_t num_users,
                      int64_t rows, int32_t max_len, int64_t step, int32_t* sequences, int32_t* sequence_users,
                      slb_stream_t stream) {
    SLB_REQUIRE(rows >= 0 && num_users >= 1 && num_users <= PR_MAX_N, "sequence_emit: bad sizes");
    if (rows == 0) return SLB_OK;
    SLB_REQUIRE(order && users && items && starts && row_offs && sequences && sequence_users,
                "sequence_emit: null pointer");
    SLB_REQUIRE(user_bytes == 4 || user_bytes == 8, "sequence_emit: user ids must be int32 or int64");
    SLB_REQUIRE(item_bytes == 4 || item_bytes == 8, "sequence_emit: item ids must be int32 or int64");
    SLB_REQUIRE(max_len >= 1 && step >= 1, "sequence_emit: max_len and step must be >= 1");
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const int64_t blocks = (rows + 7) / 8;
    SLB_REQUIRE(blocks < (int64_t(1) << 31), "sequence_emit: too many rows");
    sequence_emit_kernel<<<static_cast<unsigned>(blocks), 256, 0, st>>>(
        order, users, user_bytes, items, item_bytes, starts, row_offs, static_cast<int32_t>(num_users), rows,
        max_len, step, sequences, sequence_users);
    SLB_LAUNCH_CHECK("sequence_emit_kernel");
    return SLB_OK;
}

size_t slb_user_split_workspace_bytes(int64_t n) {
    if (n < 0 || n > PR_MAX_N) return 0;
    return pt_layout(nullptr, n, 2, 0).bytes;
}

int slb_user_split_order(const int32_t* user_ids, int64_t n, uint32_t seed, uint64_t mask_lo, uint64_t mask_hi,
                         int32_t* order, int32_t* num_train, void* workspace, size_t workspace_bytes,
                         slb_stream_t stream) {
    SLB_REQUIRE(n >= 1 && n <= PR_MAX_N, "user_split_order: n must be in [1, 2^31)");
    SLB_REQUIRE(user_ids && order && num_train && workspace, "user_split_order: null pointer");
    PtLayout l = pt_layout(workspace, n, 2, 0);
    if (l.bytes > workspace_bytes) {
        slb_set_error("user_split_order: workspace too small");
        return SLB_ENOSPC;
    }
    return pt_pass<2>(SplitDigit{user_ids, seed, mask_lo, mask_hi}, nullptr, static_cast<int32_t>(n), order, l,
                      num_train, static_cast<cudaStream_t>(stream));
}

int slb_gather_elements(const void* index, int32_t index_bytes, int64_t n, const void* src, int32_t elem_bytes,
                        void* dst, slb_stream_t stream) {
    SLB_REQUIRE(n >= 0, "gather_elements: n must be >= 0");
    if (n == 0) return SLB_OK;
    SLB_REQUIRE(index && src && dst, "gather_elements: null pointer");
    SLB_REQUIRE(index_bytes == 4 || index_bytes == 8, "gather_elements: index must be int32 or int64");
    SLB_REQUIRE(elem_bytes == 4 || elem_bytes == 8, "gather_elements: elements must be 4 or 8 bytes");
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    if (index_bytes == 8)
        gather_launch<int64_t>(index, n, src, elem_bytes, dst, st);
    else
        gather_launch<int32_t>(index, n, src, elem_bytes, dst, st);
    SLB_LAUNCH_CHECK("gather_kernel");
    return SLB_OK;
}

}  // extern "C"
