// Dense adjacency on the device (ggnn_prepare_graph_dense_device, ggnn_set_message_weights, ggnn_backward_weighted): the dense model's
// [b, T, v, v] matrix A as an fp32 device buffer, A[g, t, i, j] the weight of the type-t message from node j to node i of graph g, the
// batch's rows g*v + i.  Per timestep, with step input state h:
//   X_t[g*v+i] = sum_j A[g,t,i,j] h[g*v+j]                                     (j ascending, fmaf from +0)
//   agg        = sum_t X_t W_t + sum_t rowsum(A[g,t,i,:]) b_t                  (the row sums: ImageView::indeg)
//   dA[g,t,i,j] += <P_t[g*v+i], h[g*v+j]> + <dx'[g*v+i], b_t>,   P = dx' . W_t^T
// The kernels here form X (forward, and the backward's At), its transpose product G_t[g*v+j] = sum_i A[g,t,i,j] dx'[g*v+i] (the backward's
// Gt), the row sums, and dA.  Every output element is written by one thread, and the sums run in a fixed order without atomics, so every
// result repeats bit for bit.
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>

#include "ggnn_fwd_stream.cuh"

namespace ggnn {
namespace dadj {

constexpr int BI = 32;    // output rows of a block (rows of one graph)
constexpr int BK = 64;    // output columns of a block
constexpr int JC = 32;    // summation indices staged in shared memory per pass (a graph larger than this is tiled over j)
constexpr int THREADS = 256;

// One (graph, type, 32-row, 64-column) output tile per loop iteration of a block; thread (r = tid / 8, c = tid % 8) owns row r and the 8
// columns 8c .. 8c + 7.  TRANS = false: out row i = sum_j A[g,t,i,j] x[g*v+j]; TRANS = true: out row j = sum_i A[g,t,i,j] x[g*v+i].  The sum
// runs over the summation index ascending, one fmaf per term from +0, in passes of JC indices that keep the order.
// IN_CHUNK: x is the streaming plan's chunk-major fp32 state (DP columns, see ggnn_fwd_stream.cuh), else row-major [V][D].
// OUT_IMG: the result goes to the streaming plan's virtual-row image `img` (row g*v+i of type t is virtual row (g*v+i)*T + t, DP columns,
// those from D on zero, split to bf16 hi/lo), else to `out` [V][T*D] row-major fp32 (row, type t at columns t*D ..).
template <bool TRANS, bool IN_CHUNK, bool OUT_IMG>
__global__ void __launch_bounds__(THREADS) dense_apply_kernel(const float* __restrict__ A, const float* __restrict__ x, float* __restrict__ out,
                                                              uint8_t* __restrict__ img, int b, int v, int T, int D, int DP) {
    __shared__ float sA[BI][JC + 1];
    __shared__ __align__(16) float sX[JC][BK];
    const int tid = threadIdx.x, r = tid >> 3, c = tid & 7;
    const int ncols = OUT_IMG ? DP : D;
    const int rtiles = (v + BI - 1) / BI, ctiles = (ncols + BK - 1) / BK;
    const int64_t nblk = (int64_t)b * T * rtiles * ctiles;
    const int NKC = DP >> 3, NKS = DP >> 4;
    for (int64_t blk = blockIdx.x; blk < nblk; blk += gridDim.x) {
        const int ct = (int)(blk % ctiles);
        int64_t rest = blk / ctiles;
        const int rt = (int)(rest % rtiles);
        rest /= rtiles;
        const int t = (int)(rest % T), g = (int)(rest / T);
        const int o0 = rt * BI, k0 = ct * BK;
        const float* Ag = A + ((size_t)g * T + t) * (size_t)v * v;
        const size_t grow0 = (size_t)g * v;
        float acc[8];
#pragma unroll
        for (int q = 0; q < 8; ++q) acc[q] = 0.0f;
        for (int j0 = 0; j0 < v; j0 += JC) {
            const int jn = min(JC, v - j0);
            __syncthreads();   // the previous pass (or tile) is done reading the shared tiles
            // the lane walks the matrix row (coalesced): TRANS, output rows = matrix columns; else summation indices = matrix columns
            static_assert(BI == 32 && JC == 32 && THREADS % 32 == 0, "one warp per 32-wide matrix row segment");
#pragma unroll 1
            for (int w = tid >> 5; w < 32; w += THREADS / 32) {
                const int lane = tid & 31, ro = TRANS ? lane : w, jj = TRANS ? w : lane;
                float a = 0.0f;
                if (o0 + ro < v && jj < jn) a = TRANS ? Ag[(size_t)(j0 + jj) * v + o0 + ro] : Ag[(size_t)(o0 + ro) * v + j0 + jj];
                sA[ro][jj] = a;
            }
            for (int e = tid; e < JC * (BK / 4); e += THREADS) {
                const int jj = e / (BK / 4), k = k0 + (e % (BK / 4)) * 4;
                float4 val = make_float4(0.f, 0.f, 0.f, 0.f);
                if (jj < jn && k < D) {
                    const size_t row = grow0 + j0 + jj;
                    if (IN_CHUNK)
                        val = __ldcg(reinterpret_cast<const float4*>(x + ts::chunk_off(NKC, (int)(row >> 7), k >> 3, (int)(row & 127)) + (k & 4)));
                    else
                        val = __ldg(reinterpret_cast<const float4*>(x + row * D + k));
                }
                *reinterpret_cast<float4*>(&sX[jj][(e % (BK / 4)) * 4]) = val;
            }
            __syncthreads();
            for (int jj = 0; jj < jn; ++jj) {
                const float a = sA[r][jj];
                const float4 x0 = *reinterpret_cast<const float4*>(&sX[jj][c * 8]), x1 = *reinterpret_cast<const float4*>(&sX[jj][c * 8 + 4]);
                acc[0] = fmaf(a, x0.x, acc[0]); acc[1] = fmaf(a, x0.y, acc[1]); acc[2] = fmaf(a, x0.z, acc[2]); acc[3] = fmaf(a, x0.w, acc[3]);
                acc[4] = fmaf(a, x1.x, acc[4]); acc[5] = fmaf(a, x1.y, acc[5]); acc[6] = fmaf(a, x1.z, acc[6]); acc[7] = fmaf(a, x1.w, acc[7]);
            }
        }
        const int orow = o0 + r, col = k0 + c * 8;
        if (orow < v && col < ncols) {
            const size_t grow = grow0 + orow;
            if (OUT_IMG) {
                const size_t vid = grow * T + t;
                ts::img_store_chunk(img, NKS, (int)(vid >> 7), (int)(vid & 127), col, acc);   // columns from D on are zero (sX was)
            } else {
                float* o = out + (grow * T + t) * D + col;
                *reinterpret_cast<float4*>(o) = make_float4(acc[0], acc[1], acc[2], acc[3]);
                if (col + 4 < D) *reinterpret_cast<float4*>(o + 4) = make_float4(acc[4], acc[5], acc[6], acc[7]);
            }
        }
    }
}

// rowsum[(g*v+i)*T + t] = sum_j A[g,t,i,j]: fp32 adds in column order from +0, one thread per (graph, type, row).  The edge bias's scale
// (agg += rowsum . b_t), read as the batch's in-degree table.
__global__ void __launch_bounds__(256) dense_row_sums_kernel(const float* __restrict__ A, float* __restrict__ rowsum, int b, int v, int T) {
    const int64_t n = (int64_t)b * T * v;
    for (int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; k < n; k += (int64_t)gridDim.x * blockDim.x) {
        const int i = (int)(k % v);
        const int64_t gt = k / v;
        const int t = (int)(gt % T), g = (int)(gt / T);
        const float* row = A + (size_t)k * v;
        float s = 0.0f;
        for (int j = 0; j < v; ++j) s += row[j];
        rowsum[((size_t)g * v + i) * T + t] = s;
    }
}

// One timestep's adjacency gradient:  dA[g,t,i,j] += <P[g*v+i, t*D ..], h[g*v+j]> + <dx'[g*v+i], b_t>  (the second term only with `bias`),
// P = dx' . W_t^T [V][T*D], h the step's input state and dx' the gradient of its aggregated messages, all row-major.  One (graph, type,
// 32 x 32) tile of dA per loop iteration of a block; thread (i = tid / 8, jq = tid % 8) owns row i and columns 4 jq .. 4 jq + 3.  Both dot
// products run over the hidden columns ascending, one fmaf per term from +0; every entry has one writer, so dA repeats bit for bit.
__global__ void __launch_bounds__(THREADS) dense_adj_grad_kernel(const float* __restrict__ P, const float* __restrict__ h, const float* __restrict__ dx,
                                                                 const float* __restrict__ bias, float* __restrict__ dA, int b, int v, int T, int D) {
    constexpr int KC = 32;
    __shared__ float sP[BI][KC + 1];
    __shared__ float sH[BI][KC + 1];
    __shared__ float sD[BI][KC + 1];
    __shared__ float sB[KC];
    const int tid = threadIdx.x, i = tid >> 3, jq = tid & 7;
    const int rtiles = (v + BI - 1) / BI;
    const int64_t nblk = (int64_t)b * T * rtiles * rtiles;
    const size_t TD = (size_t)T * D;
    for (int64_t blk = blockIdx.x; blk < nblk; blk += gridDim.x) {
        const int jt = (int)(blk % rtiles);
        int64_t rest = blk / rtiles;
        const int it = (int)(rest % rtiles);
        rest /= rtiles;
        const int t = (int)(rest % T), g = (int)(rest / T);
        const int i0 = it * BI, j0 = jt * BI;
        const size_t grow0 = (size_t)g * v;
        float acc[4] = {0.0f, 0.0f, 0.0f, 0.0f}, bacc = 0.0f;
        for (int k0 = 0; k0 < D; k0 += KC) {
            const int kn = min(KC, D - k0);
            __syncthreads();
            for (int e = tid; e < BI * KC; e += THREADS) {
                const int rr = e / KC, kk = e % KC;
                const bool kin = kk < kn;
                sP[rr][kk] = kin && i0 + rr < v ? P[(grow0 + i0 + rr) * TD + (size_t)t * D + k0 + kk] : 0.0f;
                sH[rr][kk] = kin && j0 + rr < v ? h[(grow0 + j0 + rr) * D + k0 + kk] : 0.0f;
                if (bias) sD[rr][kk] = kin && i0 + rr < v ? dx[(grow0 + i0 + rr) * D + k0 + kk] : 0.0f;
            }
            if (bias && tid < KC) sB[tid] = tid < kn ? bias[(size_t)t * D + k0 + tid] : 0.0f;
            __syncthreads();
            for (int kk = 0; kk < kn; ++kk) {
                const float p = sP[i][kk];
#pragma unroll
                for (int q = 0; q < 4; ++q) acc[q] = fmaf(p, sH[jq * 4 + q][kk], acc[q]);
                if (bias) bacc = fmaf(sD[i][kk], sB[kk], bacc);
            }
        }
        if (i0 + i < v) {
            float* o = dA + (((size_t)g * T + t) * v + i0 + i) * (size_t)v;
#pragma unroll
            for (int q = 0; q < 4; ++q) {
                const int j = j0 + jq * 4 + q;
                if (j < v) o[j] += bias ? acc[q] + bacc : acc[q];
            }
        }
    }
}

}  // namespace dadj
}  // namespace ggnn
