// Warpgroup tensor-core (wgmma, sm_90a) path of the CNNNet causal convolution for
// D = 128 -- BASELINE configs[4].  Included by seq.cu after ConvGemm / ConvDw.
//
// The conv is a dense contraction (SURVEY §8a row Q2): per layer
//   forward / input-gradient : Out[(b,t), n] = sum_{j<k} sum_c In[b, t + shift_j, c] * W_j[n][c]
//   weight gradient          : dW_j[i][o]    = sum_{(b,t)} In[b, t + shift_j, i] * dZ[(b,t), o]
// Both run as 128 x 128 output tiles computed by one warpgroup (128 threads): two
// wgmma.mma_async m64n128k8 tf32 per K step (rows 0..63 and 64..127), fp32
// accumulators in registers (2 x 64 per thread).  fp32-level accuracy (the 1e-5
// parity budget) comes from the 3xTF32 split: every operand chunk is staged twice
// in shared memory (hi = tf32(x), lo = tf32(x - hi)) and each K step issues
// lo*hi + hi*lo + hi*hi into the same accumulator.
//
// Operands are staged by the CUDA cores (the split has to touch every element
// anyway) straight into the no-swizzle canonical K-major layout of the shared
// memory matrix descriptors: 8 rows x 16 B core matrices, element (r, k) at
//   (r/8)*SBO + (k/4)*LBO + (r%8)*16 + (k%4)*4,  LBO = 128, SBO = 1024
// (tf32 wgmma takes K-major operands only).  The weight gradient contracts over
// positions, which are the *outer* index of its operands in memory; its staging
// transposes 4 x 4 register blocks so it can use the same K-major layout.
// The pipeline is single stage (stage -> fence -> wgmma -> wait); the weight
// gradient's bias column sums run while the MMAs of a chunk are in flight.
#pragma once

namespace tc {

constexpr int TM = 128;          // tile rows (positions / in-channels)
constexpr int TN = 128;          // tile cols (= D)
constexpr int KC = 32;           // K elements staged per chunk (4 MMA k-steps of 8)
constexpr int TILE_BYTES = TM * KC * 4;          // 16 KB per staged operand copy
constexpr int SMEM_BYTES = 4 * TILE_BYTES;       // A_hi, A_lo, B_hi, B_lo
constexpr uint32_t LBO = 128;                    // next core matrix along K
constexpr uint32_t SBO = 1024;                   // next 8-row group
constexpr uint32_t HALF_BYTES = 8 * SBO;         // rows 64..127 of a staged operand
constexpr uint32_t KSTEP_BYTES = 2 * LBO;        // 8 tf32 of K = two core matrices

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
    return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
// generic-proxy stores to shared memory become visible to the wgmma (async proxy) reads
__device__ __forceinline__ void fence_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_wait_all() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }

// shared-memory matrix descriptor (sm_90): start address, LBO and SBO in 16-byte
// units, base offset 0, no swizzle
__device__ __forceinline__ uint64_t make_desc(uint32_t smem_addr) {
    return static_cast<uint64_t>((smem_addr >> 4) & 0x3fffu) |
           (static_cast<uint64_t>((LBO >> 4) & 0x3fffu) << 16) |
           (static_cast<uint64_t>((SBO >> 4) & 0x3fffu) << 32);
}

// d (64 x 128 fp32, wgmma accumulator fragment) += A (64 x 8 tf32) * B (8 x 128 tf32)
__device__ __forceinline__ void wgmma_tf32(float (&d)[64], uint64_t adesc, uint64_t bdesc) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "setp.ne.b32 p, %66, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
        "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
        "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
        "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
        "%64, %65, p, 1, 1;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
          "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
          "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
          "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
          "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
          "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
          "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
          "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "l"(adesc), "l"(bdesc), "r"(1)
        : "memory");
}

__device__ __forceinline__ void split4(float4 x, uint4& hi, uint4& lo) {
    split_tf32(x.x, hi.x, lo.x); split_tf32(x.y, hi.y, lo.y);
    split_tf32(x.z, hi.z, lo.z); split_tf32(x.w, hi.w, lo.w);
}

// 2 halves x 3 x (KC / 8) MMAs for one staged chunk, committed as one group and waited for
__device__ __forceinline__ void mma_chunk(float (&acc)[2][64], const uint8_t* A_hi, const uint8_t* A_lo,
                                          const uint8_t* B_hi, const uint8_t* B_lo) {
    const uint32_t ah0 = smem_u32(A_hi), al0 = smem_u32(A_lo), bh0 = smem_u32(B_hi), bl0 = smem_u32(B_lo);
    wgmma_fence();
#pragma unroll
    for (int s = 0; s < KC / 8; ++s) {
        const uint32_t o = s * KSTEP_BYTES;
        const uint64_t bh = make_desc(bh0 + o), bl = make_desc(bl0 + o);
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const uint64_t ah = make_desc(ah0 + h * HALF_BYTES + o), al = make_desc(al0 + h * HALF_BYTES + o);
            wgmma_tf32(acc[h], al, bh);
            wgmma_tf32(acc[h], ah, bl);
            wgmma_tf32(acc[h], ah, bh);
        }
    }
    wgmma_commit();
}

// Accumulator fragment of m64nNk8: warp w of the warpgroup holds rows 16w .. 16w+15 of
// each 64-row half; acc[h][4i + 2r + c] is row 64h + 16w + 8r + lane/4, column
// 8i + 2(lane%4) + c.
__device__ __forceinline__ int frag_row(int h, int r) {
    return h * 64 + (threadIdx.x >> 5) * 16 + r * 8 + ((threadIdx.x & 31) >> 2);
}
__device__ __forceinline__ int frag_col(int i) { return i * 8 + 2 * (threadIdx.x & 3); }

// ---------------------------------------------------------------------------
// forward / input-gradient:  K-major operands.  g.Wm is [k][n][c] (row n holds the
// contraction index contiguously): Wb for the forward, Wf for the input gradient.
// ---------------------------------------------------------------------------
__global__ void __launch_bounds__(128) tc_conv_gemm_kernel(ConvGemm g) {
    extern __shared__ __align__(128) uint8_t tc_smem[];
    uint8_t* A_hi = tc_smem;
    uint8_t* A_lo = tc_smem + TILE_BYTES;
    uint8_t* B_hi = tc_smem + 2 * TILE_BYTES;
    uint8_t* B_lo = tc_smem + 3 * TILE_BYTES;
    const int tid = threadIdx.x;
    const int D = g.D;                                   // == 128
    const int64_t M = g.B * g.Tout;
    const int64_t m0 = static_cast<int64_t>(blockIdx.x) * TM;
    const int64_t ms = m0 + tid;                         // the A row this thread stages
    const int64_t bs = ms < M ? ms / g.Tout : 0;
    const int ts = ms < M ? static_cast<int>(ms - bs * g.Tout) : 0;

    float acc[2][64];
#pragma unroll
    for (int h = 0; h < 2; ++h)
#pragma unroll
        for (int i = 0; i < 64; ++i) acc[h][i] = 0.f;

    const uint32_t off = (tid >> 3) * SBO + (tid & 7) * 16;          // (r/8)*SBO + (r%8)*16
    for (int j = 0; j < g.k; ++j) {
        const int q = ts + g.shift[j];
        const bool rowok = ms < M && q >= 0 && q < g.Tin;
        const float* arow = g.In + (bs * g.Tin + (rowok ? q : 0)) * D;
        const float* brow = g.Wm + (static_cast<int64_t>(j) * D + tid) * D;     // row n = tid
        for (int c0 = 0; c0 < D; c0 += KC) {
#pragma unroll
            for (int c = 0; c < KC / 4; ++c) {
                float4 av = make_float4(0, 0, 0, 0);
                if (rowok) av = ld4(arow + c0 + 4 * c);
                const float4 bv = ldg4(brow + c0 + 4 * c);
                uint4 h, l;
                split4(av, h, l);
                *reinterpret_cast<uint4*>(A_hi + off + c * LBO) = h;
                *reinterpret_cast<uint4*>(A_lo + off + c * LBO) = l;
                split4(bv, h, l);
                *reinterpret_cast<uint4*>(B_hi + off + c * LBO) = h;
                *reinterpret_cast<uint4*>(B_lo + off + c * LBO) = l;
            }
            fence_async_smem();
            __syncthreads();
            mma_chunk(acc, A_hi, A_lo, B_hi, B_lo);
            wgmma_wait_all();
            __syncthreads();                 // every warp's MMAs done: operands may be overwritten
        }
    }

    // epilogue: 4 output rows per thread, 16 column pairs each
#pragma unroll
    for (int h = 0; h < 2; ++h) {
#pragma unroll
        for (int r = 0; r < 2; ++r) {
            const int64_t m = m0 + frag_row(h, r);
            if (m >= M) continue;
            const int64_t b = m / g.Tout;
            const int t = static_cast<int>(m - b * g.Tout);
            const int rt = t + g.res_shift;
            const bool resok = g.Res && rt >= 0 && rt < g.res_T;
#pragma unroll
            for (int i = 0; i < TN / 8; ++i) {
                const int n = frag_col(i);
                float v0 = acc[h][4 * i + 2 * r], v1 = acc[h][4 * i + 2 * r + 1];
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
}

// ---------------------------------------------------------------------------
// weight gradient (positions are the contraction index):
//   A[row = i][k = pos] = In[b, t + shift_j, i],  B[row = o][k = pos] = dZ[pos, o]
// grid = (k taps, splits); every CTA owns the whole 128 x 128 (i, o) tile of one tap.
// ---------------------------------------------------------------------------
__global__ void __launch_bounds__(128) tc_conv_dw_kernel(ConvDw g) {
    extern __shared__ __align__(128) uint8_t tc_smem[];
    uint8_t* A_hi = tc_smem;
    uint8_t* A_lo = tc_smem + TILE_BYTES;
    uint8_t* B_hi = tc_smem + 2 * TILE_BYTES;
    uint8_t* B_lo = tc_smem + 3 * TILE_BYTES;
    const int tid = threadIdx.x;
    const int D = g.D;                                   // == 128
    const int j = blockIdx.x;
    const int64_t split = blockIdx.y;
    const int64_t M = g.B * g.Tout;
    const int64_t mlo = split * g.slab, mhi = mlo + g.slab < M ? mlo + g.slab : M;

    float acc[2][64];
#pragma unroll
    for (int h = 0; h < 2; ++h)
#pragma unroll
        for (int i = 0; i < 64; ++i) acc[h][i] = 0.f;

    // staging: both operands are brought into the K-major canonical layout (rows =
    // channel, k = position) by a 4 x 4 register transpose: a unit is 4 positions x 4
    // channels; thread handles units (pg = u / 32, cg = u % 32) for u = tid, tid + 128.
    float bacc = 0.f;                                    // bias gradient: column sums of dZ (tap 0 only)
    for (int64_t mb = mlo; mb < mhi; mb += KC) {
#pragma unroll
        for (int uu = 0; uu < 2; ++uu) {
            const int u = tid + uu * 128;
            const int pg = u >> 5, cg = u & 31;
            float4 a4[4], b4[4];
#pragma unroll
            for (int pp = 0; pp < 4; ++pp) {
                const int64_t mm = mb + pg * 4 + pp;
                const bool ok = mm < mhi;
                const int64_t bb = ok ? mm / g.Tout : 0;
                const int t = ok ? static_cast<int>(mm - bb * g.Tout) : 0;
                const int q = t + g.shift[j];
                a4[pp] = make_float4(0, 0, 0, 0);
                b4[pp] = make_float4(0, 0, 0, 0);
                if (ok && q >= 0 && q < g.Tin) a4[pp] = ld4(g.In + (bb * g.Tin + q) * D + cg * 4);
                if (ok) b4[pp] = ld4(g.dZ + mm * D + cg * 4);
            }
            // channel i = 4*cg + q owns the 16-byte chunk holding positions 4*pg .. 4*pg+3
            const float ar[4][4] = {{a4[0].x, a4[1].x, a4[2].x, a4[3].x}, {a4[0].y, a4[1].y, a4[2].y, a4[3].y},
                                    {a4[0].z, a4[1].z, a4[2].z, a4[3].z}, {a4[0].w, a4[1].w, a4[2].w, a4[3].w}};
            const float br[4][4] = {{b4[0].x, b4[1].x, b4[2].x, b4[3].x}, {b4[0].y, b4[1].y, b4[2].y, b4[3].y},
                                    {b4[0].z, b4[1].z, b4[2].z, b4[3].z}, {b4[0].w, b4[1].w, b4[2].w, b4[3].w}};
#pragma unroll
            for (int qd = 0; qd < 4; ++qd) {
                const int row = cg * 4 + qd;
                const uint32_t o = (row >> 3) * SBO + pg * LBO + (row & 7) * 16;
                uint4 h, l;
                split4(make_float4(ar[qd][0], ar[qd][1], ar[qd][2], ar[qd][3]), h, l);
                *reinterpret_cast<uint4*>(A_hi + o) = h;
                *reinterpret_cast<uint4*>(A_lo + o) = l;
                split4(make_float4(br[qd][0], br[qd][1], br[qd][2], br[qd][3]), h, l);
                *reinterpret_cast<uint4*>(B_hi + o) = h;
                *reinterpret_cast<uint4*>(B_lo + o) = l;
            }
        }
        fence_async_smem();
        __syncthreads();
        mma_chunk(acc, A_hi, A_lo, B_hi, B_lo);
        if (j == 0) {                                     // db[o = tid]: fixed order over the chunk
            for (int pp = 0; pp < KC; ++pp) {
                const int64_t m2 = mb + pp;
                if (m2 < mhi) bacc += g.dZ[m2 * D + tid];
            }
        }
        wgmma_wait_all();
        __syncthreads();
    }
    float* out = g.part + ((split * g.k + j) * D) * D;   // [i][o]
#pragma unroll
    for (int h = 0; h < 2; ++h)
#pragma unroll
        for (int r = 0; r < 2; ++r) {
            const int64_t i = frag_row(h, r);
#pragma unroll
            for (int c = 0; c < TN / 8; ++c)
                *reinterpret_cast<float2*>(out + i * D + frag_col(c)) =
                    make_float2(acc[h][4 * c + 2 * r], acc[h][4 * c + 2 * r + 1]);
        }
    if (j == 0) g.bpart[split * D + tid] = bacc;
}

}  // namespace tc
