// The GEMMs of the backward pass on Hopper tensor cores (wgmma), bf16x3, sm_90a: what ggnn_set_backward_precision(GGNN_PREC_BF16X3)
// selects.  Each kernel has exactly the contract of the FFMA kernel it stands in for (ggnn_bwd.cuh), so the host swaps one launch for the
// other:
//   gemm_nt_tc_kernel<ACC>      C[M,N] (+)= sum_s A_s[M,K] . B_s[N,K]^T            (= gemm_nt_kernel: data gradients)
//   gemm_tn_tc_atomic_kernel    C_s[K,N] += A_s^T . B over the rows of a split      (= gemm_tn_atomic_kernel: weight gradients, atomics)
//   gemm_tn_tc_split_kernel     ... stored into the split's own slab                 (= gemm_tn_split_kernel, then split_reduce_kernel)
//
// fp32 accuracy as in the forward (DESIGN 2.1): every fp32 operand is split on its way from global to shared memory into x = hi + lo
// (two bf16, tc::split8) and each product is issued as the three MMAs  Ah.Bh + Ah.Bl + Al.Bh  into fp32 accumulators.  No pre-split weight
// cache: the split happens per launch, so there is nothing to rebuild after ggnn_set_weights.  Tails (M, N, K, and the rows of a split) are
// zero in both parts; the bias that rides with a weight-gradient launch is summed from the fp32 values of B, not by an MMA.
//
// Shared memory: operand tiles in the canonical K-major no-swizzle layout of ggnn_fwd_tc.cuh,
//   byte(row, k) = part*PART + (k/8)*RS + row*16 + (k%8)*2      (RS = 16 * rows of the tile; LBO = RS, SBO = 128)
// double-buffered through registers like the FFMA kernels: the next slab's global loads are issued before the MMAs of the current one,
// split and stored into the other buffer while the MMAs run.
//
// Determinism: gemm_nt_tc_kernel has no split-K (one CTA owns an output tile over the whole sum, segments and K in order), so d h0 is
// bit-identical run to run and on any SM count; the split kernel's partials depend on (shape, split) only.
#pragma once
#include <cuda_bf16.h>

#include "ggnn_bwd.cuh"
#include "ggnn_fwd_tc.cuh"
#include "ggnn_wgmma.cuh"

namespace ggnn {
namespace bwd_tc {

// 8 consecutive fp32 of row `row` from column k (zero outside rows < rows, columns < cols; cols % 4 == 0, 16-byte aligned rows)
__device__ __forceinline__ void load_row8(const float* __restrict__ base, int ld, int row, int rows, int k, int cols, float (&v)[8]) {
    float4 a = make_float4(0.f, 0.f, 0.f, 0.f), b = a;
    if (row < rows) {
        const float* p = base + (size_t)row * ld + k;
        if (k + 4 <= cols) a = *reinterpret_cast<const float4*>(p);
        if (k + 8 <= cols) b = *reinterpret_cast<const float4*>(p + 4);
    }
    v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
}
// column `col` of 8 consecutive rows from row m (zero outside rows < me, columns < cols): one warp reads 32 consecutive columns per row
__device__ __forceinline__ void load_col8(const float* __restrict__ base, int ld, int m, int me, int col, int cols, float (&v)[8]) {
#pragma unroll
    for (int i = 0; i < 8; ++i) v[i] = (m + i < me && col < cols) ? base[(size_t)(m + i) * ld + col] : 0.f;
}
__device__ __forceinline__ void store_split8(uint8_t* p, uint32_t part_b, const float (&v)[8]) {
    uint4 hi, lo;
    tc::split8(v, hi, lo);
    *reinterpret_cast<uint4*>(p) = hi;
    *reinterpret_cast<uint4*>(p + part_b) = lo;
}

// ---------------------------------------------------------------- data gradients: C[M,N] (+)= sum_s A_s[M,K] . B_s[N,K]^T
// 128x128 output tile, two warpgroups (rows 0..63 / 64..127, all 128 columns: m64n128k16), K in slabs of 16 (one K-step).  Thread t loads
// row t%128 of the A and B tiles, k-group t/128 of the slab.  Arguments, alignment and ACC as gemm_nt_kernel (ggnn_bwd.cuh).
constexpr int NT_TC_BM = 128, NT_TC_BN = 128, NT_TC_THREADS = 256;
constexpr uint32_t NT_TC_RS = 128 * 16;                      // k-group stride of both tiles (128 rows)
constexpr uint32_t NT_TC_PART = 2 * NT_TC_RS;                // one part of a 16-wide slab
constexpr uint32_t NT_TC_STAGE = 4 * NT_TC_PART;             // A hi | A lo | B hi | B lo
template <bool ACC>
__global__ void __launch_bounds__(NT_TC_THREADS, 2) gemm_nt_tc_kernel(const float* __restrict__ A, int lda, int a_stride, const float* __restrict__ B,
                                                                     int ldb, int b_stride, int nseg, float* __restrict__ C, int ldc, int M, int N, int K) {
    __shared__ __align__(128) uint8_t sm[2][NT_TC_STAGE];
    const int tid = threadIdx.x, wgi = tid >> 7, lr = tid & 127, lkc = tid >> 7;
    const int m0 = blockIdx.y * NT_TC_BM, n0 = blockIdx.x * NT_TC_BN;
    const int kslabs = (K + 15) / 16, nit = nseg * kslabs;
    float acc[64];
#pragma unroll
    for (int i = 0; i < 64; ++i) acc[i] = 0.f;
    float ra[8], rb[8];
    auto load_global = [&](int it) {
        const int sg = it / kslabs, k = (it - sg * kslabs) * 16 + lkc * 8;
        load_row8(A + (size_t)sg * a_stride, lda, m0 + lr, M, k, K, ra);
        load_row8(B + (size_t)sg * b_stride, ldb, n0 + lr, N, k, K, rb);
    };
    auto store_shared = [&](int buf) {
        uint8_t* s = sm[buf] + lkc * NT_TC_RS + lr * 16;
        store_split8(s, NT_TC_PART, ra);
        store_split8(s + 2 * NT_TC_PART, NT_TC_PART, rb);
    };
    if (nit > 0) {
        load_global(0);
        store_shared(0);
    }
    tc::fence_async_smem();
    __syncthreads();
    for (int it = 0; it < nit; ++it) {
        const int buf = it & 1;
        if (it + 1 < nit) load_global(it + 1);
        const uint32_t s = tc::smem_u32(sm[buf]);
        const uint32_t a = s + (uint32_t)wgi * 64u * 16u, b = s + 2u * NT_TC_PART;
        const uint64_t ah = wg::make_desc(a, NT_TC_RS, 128), bh = wg::make_desc(b, NT_TC_RS, 128);
        wg::fence();
        wg::Mma<128>::run(acc, ah, bh);
        wg::Mma<128>::run(acc, ah, wg::make_desc(b + NT_TC_PART, NT_TC_RS, 128));
        wg::Mma<128>::run(acc, wg::make_desc(a + NT_TC_PART, NT_TC_RS, 128), bh);
        wg::commit();
        if (it + 1 < nit) store_shared(buf ^ 1);   // the other buffer: its MMAs completed before the last barrier
        wg::wait_all();
        tc::fence_async_smem();
        __syncthreads();
    }
    const int w = (tid & 127) >> 5, lane = tid & 31;
    const int r0 = m0 + wgi * 64 + w * 16 + (lane >> 2);
#pragma unroll
    for (int j = 0; j < 16; ++j) {
        const int c = n0 + 8 * j + 2 * (lane & 3);
        if (c >= N) continue;   // N % 4 == 0: c < N implies c + 1 < N
#pragma unroll
        for (int hr = 0; hr < 2; ++hr) {
            const int r = r0 + 8 * hr;
            if (r >= M) continue;
            float2* p = reinterpret_cast<float2*>(C + (size_t)r * ldc + c);
            float2 v = make_float2(acc[4 * j + 2 * hr], acc[4 * j + 2 * hr + 1]);
            if (ACC) { const float2 o = *p; v.x += o.x; v.y += o.y; }
            *p = v;
        }
    }
}

// ---------------------------------------------------------------- weight gradients: C_s[K,N] += A_s^T . B over the rows of a split
// The output tile is bwd::TN_TILE x bwd::TN_TILE (the tile tn_split sizes its grid and workspace by): one warpgroup, m64n64k16, rows of the
// split in slabs of 32 (two K-steps of the MMA, whose reduction dimension is the node rows).  Both operands are transposed on the way to
// shared memory: thread t loads column t%64 of the A_s and B tiles, 8 rows at a time (row groups t/64 and t/64 + 2 of the slab), so that
// each thread stores one 16-byte k-group row of each part.  Arguments as gemm_tn_tile (ggnn_bwd.cuh) with a_vec = 1; bias_out is summed in
// fp32 from the loaded B values: each thread adds its rows in order, the two row halves are added at the end.
constexpr int TN_TC_THREADS = 128, TN_TC_ROWS = 32;
static_assert(bwd::TN_TILE == 64, "the weight-gradient MMAs are m64n64");
constexpr uint32_t TN_TC_RS = 64 * 16;                       // k-group stride of both tiles (64 rows)
constexpr uint32_t TN_TC_PART = (TN_TC_ROWS / 8) * TN_TC_RS; // one part of a 32-row slab
constexpr uint32_t TN_TC_STAGE = 4 * TN_TC_PART;             // A hi | A lo | B hi | B lo
template <bool SPLIT>
__device__ __forceinline__ void gemm_tn_tc_tile(const bwd::SegList& segs, int kblocks, const float* __restrict__ B, int ldb, float* __restrict__ C,
                                                int ldc, size_t c_stride, float* __restrict__ bias_out, int M, int N, int K, int rows_per_split) {
    __shared__ __align__(128) uint8_t sm[2][TN_TC_STAGE];
    __shared__ float s_bias[2][64];
    const int tid = threadIdx.x, col = tid & 63, mg = tid >> 6;
    const int sg = blockIdx.y / kblocks;
    const int k0 = (blockIdx.y - sg * kblocks) * bwd::TN_TILE, n0 = blockIdx.x * bwd::TN_TILE;
    const float* __restrict__ A = segs.p[sg];
    const int lda = segs.ld[sg];
    const int mb = blockIdx.z * rows_per_split, me = min(M, mb + rows_per_split);
    const bool do_bias = bias_out != nullptr && blockIdx.y == 0;
    float acc[32];
#pragma unroll
    for (int i = 0; i < 32; ++i) acc[i] = 0.f;
    float bsum = 0.f;
    float ra[2][8], rb[2][8];
    auto load_global = [&](int m) {
#pragma unroll
        for (int g = 0; g < 2; ++g) {
            load_col8(A, lda, m + (mg + 2 * g) * 8, me, k0 + col, K, ra[g]);
            load_col8(B, ldb, m + (mg + 2 * g) * 8, me, n0 + col, N, rb[g]);
        }
    };
    auto store_shared = [&](int buf) {
#pragma unroll
        for (int g = 0; g < 2; ++g) {
            uint8_t* s = sm[buf] + (mg + 2 * g) * TN_TC_RS + col * 16;
            store_split8(s, TN_TC_PART, ra[g]);
            store_split8(s + 2 * TN_TC_PART, TN_TC_PART, rb[g]);
        }
    };
    auto add_bias = [&]() {
#pragma unroll
        for (int g = 0; g < 2; ++g)
#pragma unroll
            for (int i = 0; i < 8; ++i) bsum += rb[g][i];
    };
    const int nit = (me - mb + TN_TC_ROWS - 1) / TN_TC_ROWS;
    if (nit > 0) {
        load_global(mb);
        if (do_bias) add_bias();
        store_shared(0);
    }
    tc::fence_async_smem();
    __syncthreads();
    for (int it = 0; it < nit; ++it) {
        const int buf = it & 1;
        if (it + 1 < nit) load_global(mb + (it + 1) * TN_TC_ROWS);
        const uint32_t s = tc::smem_u32(sm[buf]);
        wg::fence();
#pragma unroll
        for (int h = 0; h < TN_TC_ROWS / 16; ++h) {
            const uint32_t a = s + (uint32_t)h * 2u * TN_TC_RS, b = a + 2u * TN_TC_PART;
            const uint64_t ah = wg::make_desc(a, TN_TC_RS, 128), bh = wg::make_desc(b, TN_TC_RS, 128);
            wg::Mma<64>::run(acc, ah, bh);
            wg::Mma<64>::run(acc, ah, wg::make_desc(b + TN_TC_PART, TN_TC_RS, 128));
            wg::Mma<64>::run(acc, wg::make_desc(a + TN_TC_PART, TN_TC_RS, 128), bh);
        }
        wg::commit();
        if (it + 1 < nit) {
            if (do_bias) add_bias();
            store_shared(buf ^ 1);
        }
        wg::wait_all();
        tc::fence_async_smem();
        __syncthreads();
    }
    float* Cs = C + (size_t)sg * c_stride;
    const int w = tid >> 5, lane = tid & 31;
    const int kr0 = k0 + w * 16 + (lane >> 2);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        const int n = n0 + 8 * j + 2 * (lane & 3);
        if (n >= N) continue;
#pragma unroll
        for (int hr = 0; hr < 2; ++hr) {
            const int k = kr0 + 8 * hr;
            if (k >= K) continue;
            const float2 v = make_float2(acc[4 * j + 2 * hr], acc[4 * j + 2 * hr + 1]);
            float2* p = reinterpret_cast<float2*>(Cs + (size_t)k * ldc + n);
            if (SPLIT) *p = v;
            else atomicAdd(p, v);
        }
    }
    if (do_bias) {
        s_bias[mg][col] = bsum;
        __syncthreads();
        if (tid < 64 && n0 + tid < N) {
            const float v = s_bias[0][tid] + s_bias[1][tid];
            if (SPLIT) bias_out[n0 + tid] = v;
            else atomicAdd(bias_out + n0 + tid, v);
        }
    }
}
__global__ void __launch_bounds__(TN_TC_THREADS) gemm_tn_tc_atomic_kernel(bwd::SegList segs, int kblocks, const float* __restrict__ B, int ldb,
                                                                          float* __restrict__ C, int ldc, size_t c_stride, float* __restrict__ bias_out,
                                                                          int M, int N, int K, int rows_per_split) {
    gemm_tn_tc_tile<false>(segs, kblocks, B, ldb, C, ldc, c_stride, bias_out, M, N, K, rows_per_split);
}
// the partial layout of gemm_tn_split_kernel: part[z][s][K][N], bias_part[z][N]
__global__ void __launch_bounds__(TN_TC_THREADS) gemm_tn_tc_split_kernel(bwd::SegList segs, int kblocks, const float* __restrict__ B, int ldb,
                                                                         float* __restrict__ part, float* __restrict__ bias_part, int M, int N, int K,
                                                                         int rows_per_split) {
    const size_t per = (size_t)K * N;
    gemm_tn_tc_tile<true>(segs, kblocks, B, ldb, part + (size_t)blockIdx.z * (gridDim.y / kblocks) * per, N, per,
                          bias_part ? bias_part + (size_t)blockIdx.z * N : nullptr, M, N, K, rows_per_split);
}

}  // namespace bwd_tc
}  // namespace ggnn
