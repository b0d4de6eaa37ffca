// Device-side, NumPy-bit-exact RandomState.shuffle(arange(n))  --  replaces the
// epoch permutation of spotlight/torch_utils.py:46-47 (called from
// factorization/implicit.py:212-214 and sequence/implicit.py:220), which the
// reference (and round-1's host path, csrc/host_shuffle.cpp) runs as n dependent
// swaps on one host thread.
//
// numpy's legacy shuffle is   for i = n-1 .. 1:  j = rk_interval(i);  swap(x[i], x[j])
// with rk_interval(i) = first stream word w, masked to bit_length(i) bits, that is <= i.
// Both halves look sequential; neither is.
//
// A. Draws.  Word t of the stream is consumed by step i_t = n-1-A(t), A(t) = number of
//    words accepted before t, and is accepted iff (w_t & mask(i_t)) <= i_t.  The
//    recursion is forward-determined, so its solution is the unique fixed point of
//    "flags from A -> A = exclusive prefix sum of flags", and any iteration that stops
//    changing has found it.  The dependence is weak: a wrong A only matters for words
//    whose masked value lies between the assumed and the true bound, a fraction
//    ~ error / mask.  Two nested fixed points: a CTA resolves its 2048-word tile
//    *exactly* given the tile's start count (threads are exact over their own 8 words
//    and iterate on the 256 thread bases), and the global rounds iterate only on the
//    tile start counts (count kernel over tiles whose start moved -> one-CTA scan),
//    starting from the expected acceptance curve.  Convergence is checked, not assumed.
//
// B. Swaps.  Step i is the last writer of position i, so order[i] = the value held by
//    position j_i just before step i.  With T(p) = steps targeting position p in
//    ascending order, that value was deposited by the next-larger member of T(j_i)
//    ("parent"), which moved V(parent) = the value position `parent` held before its own
//    step, and V(x) = V(m(x)) with m(x) = the smallest step > x targeting position x,
//    or x itself when no step does (arange start).  parent / m come from grouping the
//    steps by target (integer-atomic histogram -> scan -> unordered fill -> per-target
//    sort, as the gradient segment index), then every position chases its short m-chain
//    (expected O(1), O(log n) w.h.p.).
#include "common.cuh"
#include "scan.cuh"

namespace {

constexpr int SH_T = 2048;          // stream words per tile
constexpr int SH_THREADS = 256;
constexpr int SH_WPT = 8;           // words per thread
constexpr int F_CONV = 0, F_TOTAL = 1, F_ROUNDS = 2;

__device__ __forceinline__ uint32_t sh_temper(uint32_t y) {
    y ^= y >> 11;
    y ^= (y << 7) & 0x9d2c5680u;
    y ^= (y << 15) & 0xefc60000u;
    y ^= y >> 18;
    return y;
}

__device__ __forceinline__ uint32_t sh_mask(int32_t i) {      // i >= 1
    return 0xffffffffu >> __clz(static_cast<uint32_t>(i));
}

// Block-wide exclusive prefix of one int per thread (SH_THREADS threads); also the total.
__device__ __forceinline__ int sh_block_excl(int v, int& total, int* sh /* 8 ints */) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    int inc = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const int a = __shfl_up_sync(0xffffffffu, inc, o);
        if (lane >= o) inc += a;
    }
    __syncthreads();                       // previous readers of sh are done
    if (lane == 31) sh[warp] = inc;
    __syncthreads();
    int wpre = 0, tot = 0;
#pragma unroll
    for (int w = 0; w < SH_THREADS / 32; ++w) {
        const int s = sh[w];
        if (w < warp) wpre += s;
        tot += s;
    }
    total = tot;
    return wpre + inc - v;
}

// Exact acceptance flags of one tile given i0 = the bound of its first word
// (i0 = n-1-start; may be <= 0 past the end of the shuffle).  Returns this thread's
// flag bits; base = accepted words of the tile before this thread's first word.
__device__ __forceinline__ uint32_t sh_tile_resolve(const uint32_t (&v)[SH_WPT], int nvalid, int32_t i0,
                                                    int& base, int& total, int* sh) {
    // initial thread bases from the expected acceptance rate at i0
    float p = 0.f;
    if (i0 >= 1) p = (static_cast<float>(i0) + 1.f) / (static_cast<float>(sh_mask(i0)) + 1.f);
    base = static_cast<int>(p * static_cast<float>(threadIdx.x * SH_WPT));
    uint32_t fl;
    for (;;) {
        int c = base;
        fl = 0;
#pragma unroll
        for (int k = 0; k < SH_WPT; ++k) {
            const int32_t i = i0 - c;
            const bool a = k < nvalid && i >= 1 && (v[k] & sh_mask(i)) <= static_cast<uint32_t>(i);
            fl |= static_cast<uint32_t>(a) << k;
            c += a;
        }
        const int nb = sh_block_excl(c - base, total, sh);
        const int changed = nb != base;
        base = nb;
        if (!__syncthreads_or(changed)) break;
    }
    return fl;
}

__device__ __forceinline__ int sh_load(const uint32_t* __restrict__ blocks, int64_t w0, int64_t W,
                                       int tile, uint32_t (&v)[SH_WPT]) {
    const int64_t first = static_cast<int64_t>(tile) * SH_T + threadIdx.x * SH_WPT;
    int nvalid = 0;
#pragma unroll
    for (int k = 0; k < SH_WPT; ++k) {
        v[k] = 0;
        if (first + k < W) { v[k] = sh_temper(__ldg(blocks + w0 + first + k)); nvalid = k + 1; }
    }
    return nvalid;
}

// Expected number of accepted words before stream word t (per mask epoch the bound
// decays as (i+1) = (hi+1) exp(-(t-t0)/M)).
__global__ void shuf_init_kernel(int32_t* start, int32_t* prev, int ntiles, int32_t n, int32_t* flags) {
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k == 0) { flags[F_CONV] = 0; flags[F_TOTAL] = 0; flags[F_ROUNDS] = 0; }
    if (k >= ntiles) return;
    const double t = static_cast<double>(k) * SH_T;
    double t0 = 0.0, res = static_cast<double>(n - 1);
    int64_t hi = n - 1;
    while (hi >= 1) {
        const double M = static_cast<double>(static_cast<int64_t>(sh_mask(static_cast<int32_t>(hi))) + 1);
        const int64_t lo = static_cast<int64_t>(M) / 2;          // epoch covers i in [lo, hi]
        const double t1 = t0 + M * log((hi + 1.0) / static_cast<double>(lo));
        if (t < t1) { res = n - (hi + 1.0) * exp(-(t - t0) / M); break; }
        t0 = t1;
        hi = lo - 1;
    }
    res = fmin(fmax(res, 0.0), static_cast<double>(n - 1));
    start[k] = static_cast<int32_t>(res);
    prev[k] = -1;
}

__global__ void __launch_bounds__(SH_THREADS)
shuf_count_kernel(const uint32_t* __restrict__ blocks, int64_t w0, int64_t W, int32_t n,
                  const int32_t* __restrict__ start, int32_t* prev, int32_t* cnt, const int32_t* flags) {
    __shared__ int sh[SH_THREADS / 32];
    if (flags[F_CONV]) return;
    const int tile = blockIdx.x;
    const int32_t st = start[tile];
    if (st == prev[tile]) return;                 // same start as last time: count stands
    uint32_t v[SH_WPT];
    const int nvalid = sh_load(blocks, w0, W, tile, v);
    int base, total;
    sh_tile_resolve(v, nvalid, n - 1 - st, base, total, sh);
    if (threadIdx.x == 0) { cnt[tile] = total; prev[tile] = st; }
}

// One CTA: start[] <- exclusive prefix of cnt[]; converged when nothing moved.
__global__ void __launch_bounds__(1024)
shuf_scan_kernel(const int32_t* __restrict__ cnt, int32_t* start, int ntiles, int32_t* flags) {
    __shared__ int64_t shw[32];
    if (flags[F_CONV]) return;
    const int per = (ntiles + 1023) / 1024;
    const int lo = threadIdx.x * per, hi = min(lo + per, ntiles);
    int64_t s = 0;
    for (int k = lo; k < hi; ++k) s += cnt[k];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    int64_t inc = s;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const int64_t a = __shfl_up_sync(0xffffffffu, inc, o);
        if (lane >= o) inc += a;
    }
    if (lane == 31) shw[warp] = inc;
    __syncthreads();
    int64_t pre = inc - s, tot = 0;
    for (int w = 0; w < 32; ++w) { if (w < warp) pre += shw[w]; tot += shw[w]; }
    int moved = 0;
    for (int k = lo; k < hi; ++k) {
        const int32_t nv = static_cast<int32_t>(min(pre, static_cast<int64_t>(0x7fffffff)));
        if (start[k] != nv) { start[k] = nv; moved = 1; }
        pre += cnt[k];
    }
    moved = __syncthreads_or(moved);
    if (threadIdx.x == 0) {
        flags[F_CONV] = !moved;
        flags[F_TOTAL] = static_cast<int32_t>(min(tot, static_cast<int64_t>(0x7fffffff)));
        flags[F_ROUNDS] += 1;
    }
}

// With exact starts: j[i] for every step, the end of the consumed stream, and the verdict.
__global__ void __launch_bounds__(SH_THREADS)
shuf_emit_kernel(const uint32_t* __restrict__ blocks, int64_t w0, int64_t W, int32_t n,
                 const int32_t* __restrict__ start, int32_t* __restrict__ jv, int64_t* cursor,
                 const int32_t* flags) {
    __shared__ int sh[SH_THREADS / 32];
    const int tile = blockIdx.x;
    if (tile == 0 && threadIdx.x == 0) {
        jv[0] = 0;
        cursor[1] = flags[F_TOTAL];
        cursor[2] = flags[F_CONV];
        cursor[3] = flags[F_ROUNDS];
        if (n <= 1) cursor[0] = w0;
    }
    if (!flags[F_CONV]) return;
    const int32_t st = start[tile];
    if (st >= n - 1) return;                      // shuffle finished before this tile
    uint32_t v[SH_WPT];
    const int nvalid = sh_load(blocks, w0, W, tile, v);
    int base, total;
    const uint32_t fl = sh_tile_resolve(v, nvalid, n - 1 - st, base, total, sh);
    int c = st + base;
#pragma unroll
    for (int k = 0; k < SH_WPT; ++k) {
        if ((fl >> k) & 1u) {
            const int32_t i = n - 1 - c;
            jv[i] = static_cast<int32_t>(v[k] & sh_mask(i));
            if (i == 1) cursor[0] = w0 + static_cast<int64_t>(tile) * SH_T + threadIdx.x * SH_WPT + k + 1;
            ++c;
        }
    }
}

// ---- stage B ------------------------------------------------------------------------
__device__ __forceinline__ bool shuf_ok(const int32_t* flags, int32_t n) {
    return flags[F_CONV] && flags[F_TOTAL] >= n - 1;       // else j[] is incomplete: leave `order` alone
}

__global__ void shuf_hist_kernel(const int32_t* __restrict__ jv, int32_t n, int32_t* cnt, const int32_t* flags) {
    if (!shuf_ok(flags, n)) return;
    const int64_t stride = static_cast<int64_t>(gridDim.x) * blockDim.x;
    for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += stride)
        atomicAdd(cnt + jv[i], 1);
}

// cur[v] enters as the end offset of v's segment and leaves as its start offset.
__global__ void shuf_fill_kernel(const int32_t* __restrict__ jv, int32_t n, int32_t* cur,
                                 int32_t* members, const int32_t* flags) {
    if (!shuf_ok(flags, n)) return;
    const int64_t stride = static_cast<int64_t>(gridDim.x) * blockDim.x;
    for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += stride)
        members[atomicSub(cur + jv[i], 1) - 1] = static_cast<int32_t>(i);
}

// Per target position v: sort its steps ascending, link each to the next one (parent),
// and record m(v) = the smallest step > v that targets v.
__global__ void shuf_link_kernel(int32_t n, const int32_t* __restrict__ off, int32_t* members,
                                 int32_t* __restrict__ parent, int32_t* __restrict__ mlink,
                                 const int32_t* flags) {
    if (!shuf_ok(flags, n)) return;
    const int64_t stride = static_cast<int64_t>(gridDim.x) * blockDim.x;
    for (int64_t v = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; v < n; v += stride) {
        const int32_t s = off[v], e = off[v + 1];
        const int len = e - s;
        if (len == 0) { mlink[v] = -1; continue; }
        if (len == 1) {
            const int32_t a = members[s];
            parent[a] = -1;
            mlink[v] = a > v ? a : -1;
            continue;
        }
        for (int x = s + 1; x < e; ++x) {           // insertion sort (lengths ~ Poisson(1), max ~ ln n)
            const int32_t key = members[x];
            int y = x - 1;
            while (y >= s && members[y] > key) { members[y + 1] = members[y]; --y; }
            members[y + 1] = key;
        }
        int32_t a = members[s];
        const int32_t a0 = a, a1 = members[s + 1];
        for (int x = s + 1; x < e; ++x) { const int32_t b = members[x]; parent[a] = b; a = b; }
        parent[a] = -1;
        mlink[v] = a0 > v ? a0 : a1;
    }
}

__global__ void shuf_final_kernel(int32_t n, const int32_t* __restrict__ jv,
                                  const int32_t* __restrict__ parent, const int32_t* __restrict__ mlink,
                                  int64_t* __restrict__ order, const int32_t* flags) {
    if (!shuf_ok(flags, n)) return;
    const int64_t stride = static_cast<int64_t>(gridDim.x) * blockDim.x;
    for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += stride) {
        int32_t x = parent[i];
        if (x < 0) { order[i] = jv[i]; continue; }
        for (;;) {
            const int32_t y = __ldg(mlink + x);
            if (y < 0) break;
            x = y;
        }
        order[i] = x;
    }
}

// users_out[i] = users[order[i]], items_out[i] = items[order[i]] (ids widened to int64):
// the two fancy-index gathers of torch_utils.shuffle (torch_utils.py:49-52) in one pass.
template <typename T>
__global__ void permute_ids_kernel(const int64_t* __restrict__ order, int64_t n, const T* __restrict__ a,
                                   const T* __restrict__ b, int64_t* __restrict__ oa,
                                   int64_t* __restrict__ ob) {
    const int64_t stride = static_cast<int64_t>(gridDim.x) * blockDim.x;
    for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += stride) {
        const int64_t o = order[i];
        if (o < 0 || o >= n) { oa[i] = -1; if (b) ob[i] = -1; continue; }     // caught by the id range flags
        oa[i] = static_cast<int64_t>(__ldg(a + o));
        if (b) ob[i] = static_cast<int64_t>(__ldg(b + o));
    }
}

struct ShufLayout {
    int32_t *start, *prev, *cntT, *flags, *jv, *cnt, *off, *members, *parent, *mlink, *tsum;
    int ntiles, nscan;
    size_t bytes;
};

ShufLayout shuf_layout(void* ws, int64_t n, int64_t nwords) {
    ShufLayout l;
    WsCarver c(ws);
    l.ntiles = static_cast<int>((nwords + SH_T - 1) / SH_T);
    l.nscan = static_cast<int>((n + 1 + SC_TILE - 1) / SC_TILE);
    l.flags = c.take<int32_t>(8);
    l.start = c.take<int32_t>(l.ntiles);
    l.prev = c.take<int32_t>(l.ntiles);
    l.cntT = c.take<int32_t>(l.ntiles);
    l.jv = c.take<int32_t>(n);
    l.cnt = c.take<int32_t>(n + 1);
    l.off = c.take<int32_t>(n + 1);
    l.members = c.take<int32_t>(n);
    l.parent = c.take<int32_t>(n);
    l.mlink = c.take<int32_t>(n);
    l.tsum = c.take<int32_t>(l.nscan + 1);
    l.bytes = c.bytes();
    return l;
}

unsigned grid_for(int64_t n, int threads) {
    const int64_t want = (n + threads - 1) / threads;
    const int64_t cap = static_cast<int64_t>(slb_sms()) * 16;
    return static_cast<unsigned>(want < 1 ? 1 : (want < cap ? want : cap));
}

}  // namespace

extern "C" {

size_t slb_shuffle_workspace_bytes(int64_t n, int64_t nwords) {
    if (n < 0 || nwords < 0) return 0;
    return shuf_layout(nullptr, n, nwords).bytes;
}

int slb_shuffle_order(const uint32_t* blocks, int64_t nwords, int64_t* cursor, int64_t first_word,
                      int64_t n, int32_t rounds, int32_t resume, int64_t* order, void* workspace,
                      size_t workspace_bytes, slb_stream_t stream) {
    SLB_REQUIRE(blocks && cursor && order && workspace, "shuffle_order: null pointer");
    SLB_REQUIRE(n >= 1 && n <= (int64_t(1) << 29), "shuffle_order: n must be in [1, 2^29]");
    SLB_REQUIRE(first_word >= 0 && first_word < nwords, "shuffle_order: first_word out of range");
    SLB_REQUIRE(nwords - first_word < (int64_t(1) << 31), "shuffle_order: stream too long");
    SLB_REQUIRE(rounds >= 1, "shuffle_order: rounds must be >= 1");
    const int64_t W = nwords - first_word;
    ShufLayout l = shuf_layout(workspace, n, W);
    if (l.bytes > workspace_bytes) {
        slb_set_error("shuffle_order: workspace too small");
        return SLB_ENOSPC;
    }
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const int32_t n32 = static_cast<int32_t>(n);
    const int nt = l.ntiles > 0 ? l.ntiles : 1;
    if (!resume) {
        shuf_init_kernel<<<(nt + 255) / 256, 256, 0, st>>>(l.start, l.prev, l.ntiles, n32, l.flags);
        SLB_LAUNCH_CHECK("shuf_init_kernel");
    }
    if (l.ntiles > 0) {
        for (int r = 0; r < rounds; ++r) {
            shuf_count_kernel<<<l.ntiles, SH_THREADS, 0, st>>>(blocks, first_word, W, n32, l.start, l.prev,
                                                              l.cntT, l.flags);
            shuf_scan_kernel<<<1, 1024, 0, st>>>(l.cntT, l.start, l.ntiles, l.flags);
        }
        SLB_LAUNCH_CHECK("shuf_count/scan_kernel");
    }
    shuf_emit_kernel<<<nt, SH_THREADS, 0, st>>>(blocks, first_word, W, n32, l.start, l.jv, cursor, l.flags);
    SLB_LAUNCH_CHECK("shuf_emit_kernel");
    // stage B runs only when the draw converged and produced all n-1 swaps (device-side
    // guard); the caller reads cursor[1..2] and extends the stream / adds rounds otherwise
    if (cudaMemsetAsync(l.cnt, 0, sizeof(int32_t) * (n + 1), st) != cudaSuccess) {
        slb_set_error("shuffle_order: memset failed");
        return SLB_ECUDA;
    }
    shuf_hist_kernel<<<grid_for(n, 256), 256, 0, st>>>(l.jv, n32, l.cnt, l.flags);
    scan_tilesum_kernel<<<l.nscan, SC_THREADS, 0, st>>>(l.cnt, n + 1, l.tsum);
    scan_tiles_kernel<<<1, 1024, 0, st>>>(l.tsum, l.nscan);
    scan_apply_kernel<<<l.nscan, SC_THREADS, 0, st>>>(l.cnt, n + 1, l.tsum, l.off);
    shuf_fill_kernel<<<grid_for(n, 256), 256, 0, st>>>(l.jv, n32, l.off, l.members, l.flags);
    shuf_link_kernel<<<grid_for(n, 256), 256, 0, st>>>(n32, l.off, l.members, l.parent, l.mlink, l.flags);
    shuf_final_kernel<<<grid_for(n, 256), 256, 0, st>>>(n32, l.jv, l.parent, l.mlink, order, l.flags);
    SLB_LAUNCH_CHECK("shuffle stage B");
    return SLB_OK;
}

int slb_permute_ids(const int64_t* order, int64_t n, const void* users, const void* items,
                    int32_t elem_bytes, int64_t* users_out, int64_t* items_out, slb_stream_t stream) {
    SLB_REQUIRE(n >= 0, "permute_ids: n must be >= 0");
    if (n == 0) return SLB_OK;
    SLB_REQUIRE(order && users && users_out, "permute_ids: null pointer");
    SLB_REQUIRE((items == nullptr) == (items_out == nullptr), "permute_ids: items / items_out mismatch");
    SLB_REQUIRE(elem_bytes == 4 || elem_bytes == 8, "permute_ids: elem_bytes must be 4 or 8");
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    if (elem_bytes == 4)
        permute_ids_kernel<int32_t><<<grid_for(n, 256), 256, 0, st>>>(
            order, n, static_cast<const int32_t*>(users), static_cast<const int32_t*>(items), users_out, items_out);
    else
        permute_ids_kernel<int64_t><<<grid_for(n, 256), 256, 0, st>>>(
            order, n, static_cast<const int64_t*>(users), static_cast<const int64_t*>(items), users_out, items_out);
    SLB_LAUNCH_CHECK("permute_ids_kernel");
    return SLB_OK;
}

}  // extern "C"
