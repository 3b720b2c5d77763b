// Sparse GCN propagation (Kipf & Welling; chem_tensorflow_gcn.py:59-82), sm_90a.  Per layer l:
//   S  = A . H        S[i] += w * H[j] over the nonzeros (i, j, w) of the batch, per row in list order (the stable target-sorted CSR
//                     keeps it: the serial order of TF's CPU sparse_tensor_dense_matmul functor as we recall it from TF's source)
//   H' = S . W_l (+ b_l),  then relu and state dropout on every layer but the last (the last layer is linear)
//
// Two kernels:
//   gcn_wgmma_kernel  hidden <= 128, bf16x3 / bf16 precision.  One CTA per tile of <= 128 rows.  LOCAL: the tile is a union of whole
//                     connected components, all layers run in one launch and H stays in shared memory between layers.  GLOBAL: one launch
//                     per layer, the gather reads the previous layer's fp32 state from global memory (a component larger than a tile).
//                     Warp roles and operand layouts follow ggnn_fwd_tc.cuh: four worker warpgroups, warpgroup w owns rows 64*(w%2) .. +64 and
//                     columns NH*(w/2) .. +NH (NH = DP/2) of S . W; S is split into bf16 hi/lo in the canonical no-swizzle K-major layout.
//                     The pre-split, pre-tiled W_l (tc::ggnn_tile_weights_kernel) streams through the tile kernels' weight ring
//                     (tc::RingWriter / tc::RingReader, tc::gemm_narrow); a timeout sets the engine's error flag (ggnn_sync_check).
//   gcn_fp32_kernel   fp32 precision, and hidden sizes above 128 without ggnn_gcn_config.wide_hidden: per layer, 32 rows per CTA,
//                     weighted CSR gather into shared memory, FFMA GEMM with W_l from L1/L2, same epilogue.
//   gcn_gather_image_kernel  hidden sizes above 128 on bf16x3 / bf16 with wide_hidden: S = A . H into the streaming operand image, which the
//                     TMA-fed ts::ggnn_stream_kernel multiplies by W_l (EPI_GCN: the same epilogue); two launches per layer.
// The backward pass (ggnn_engine.cu) reuses ggnn_bwd.cuh; only the relu / dropout gradient below is GCN-specific, and on a
// message-weighted batch the source-row pass that also forms the adjacency weights' gradient (gcn_source_grad_kernel).
#pragma once
#include "ggnn_common.cuh"
#include "ggnn_fwd_stream.cuh"
#include "ggnn_fwd_tc.cuh"
#include "ggnn_wgmma.cuh"

namespace ggnn {
namespace gcn {

constexpr int NTHREADS = tc::NUM_WORKERS + 32;   // the tile kernels' four worker warpgroups + one producer warp (no spills at 96 registers)
constexpr int MAX_STAGES = 8;
constexpr int KGS = 2048;              // A-operand k-group stride: 128 rows x 16 bytes
constexpr int F32_ROWS = 32;           // rows per CTA of the fp32 kernel
constexpr int F32_THREADS = 256;

struct GcnParams {
    int V, D, DP, L;
    int nparts;                        // 3: bf16x3, 1: bf16
    int nstages;                       // weight ring depth (slots of two K-step stages)
    int save;                          // LOCAL: write every layer's output to global memory (backward, ggnn_layer_state)
    const int* tile_start;             // [ntiles + 1]
    const int* row_ptr;                // [V + 1] target (output row) CSR
    const int* csr_src;                // [nnz]   input column of every slot
    const float* slot_w;               // [nnz]   weight of every slot
    const float* state[MAX_LAYERS + 1];   // [0] = h0, [L] = result
    float* state_w[MAX_LAYERS + 1];
    const uint8_t* w_tiled[MAX_LAYERS];   // pre-split, pre-tiled W_l: DP/16 stages of 64*DP bytes
    const float* bias[MAX_LAYERS];        // [D] or nullptr
    const float* kernel[MAX_LAYERS];      // fp32 W_l [D, D] (fp32 kernel)
    int g_layer;                       // GLOBAL mode / fp32 kernel: the layer of this launch
    float drop_keep;
    unsigned long long drop_seed;
    int* error_flag;
};

// bias, relu and state dropout of one output element (row, col < D) of layer l
__device__ __forceinline__ float epilogue(float v, const GcnParams& p, int l, int row, int col) {
    if (p.bias[l]) v += __ldg(p.bias[l] + col);
    if (l < p.L - 1) {
        v = fmaxf(v, 0.0f);
        if (p.drop_keep < 1.0f) v = dropout_apply(v, p.drop_seed, l, p.V, p.D, row, col, p.drop_keep);
    }
    return v;
}

// ------------------------------------------------------------------------------------------------ tensor cores
// X3: bf16x3 (p.nparts == 3), else one bf16 MMA per product; DP = 2*NH
template <bool LOCAL, int NH, bool X3>
__global__ void __launch_bounds__(NTHREADS, 1) gcn_wgmma_kernel(const __grid_constant__ GcnParams p) {
    using namespace tc;
    constexpr int NF = NH / 2;   // accumulator floats per thread (m64 x NH fragment)
    constexpr int NJ = NH / 8;   // 8-column blocks of a fragment
    extern __shared__ __align__(1024) uint8_t smem[];
    __shared__ __align__(8) uint64_t bar_full[MAX_STAGES];
    __shared__ __align__(8) uint64_t bar_empty[MAX_STAGES];
    __shared__ int s_abort;

    constexpr int DP = 2 * NH;
    constexpr int NKC = DP >> 3, NKS = DP >> 4;
    constexpr uint32_t PART_B = (uint32_t)DP * KGS / 8u;
    constexpr uint32_t OPB = 2u * PART_B;
    constexpr uint32_t STAGE_B = (uint32_t)DP * 64u;
    const int D = p.D;
    uint8_t* opS = smem;
    uint8_t* ring = opS + OPB;
    float* sH = reinterpret_cast<float*>(ring + (size_t)p.nstages * 2 * STAGE_B);   // LOCAL: [128][DP] fp32 node states of the tile

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int row0 = p.tile_start[blockIdx.x];
    const int rows = p.tile_start[blockIdx.x + 1] - row0;
    const int nst = p.nstages;
    if (tid == 0) {
        s_abort = 0;
        ring_init(bar_full, bar_empty, MAX_STAGES);
    }
    __syncthreads();
    volatile int* abortp = &s_abort;
    const int l_begin = LOCAL ? 0 : p.g_layer;
    const int l_end = LOCAL ? p.L : p.g_layer + 1;

    if (warp < WARP_PROD) {
        // ============================================================ WORKERS
        const int row = (warp & 3) * 32 + lane, cg = warp >> 2;   // gather view: one row, column chunks cg, cg + 4, ...
        constexpr int NCG = NUM_WORKERS / 128;
        const int wgi = warp >> 2, mh = wgi & 1, nh = wgi >> 1;   // fragment view
        const int fr0 = mh * 64 + (warp & 3) * 16 + (lane >> 2);
        const int fc0 = nh * NH + (lane & 3) * 2;
        bool ok = true;
        RingReader rd{bar_full, bar_empty, abortp, smem_u32(ring), (uint32_t)nst};
        const uint32_t a_row = (uint32_t)mh * 64u * 16u;

        if (LOCAL) {   // the tile's input states -> shared memory (padding columns zero)
            for (int idx = tid; idx < rows * NKC; idx += NUM_WORKERS) {
                const int r = idx / NKC, kc = idx - r * NKC;
                float v[8];
                load8_guarded(p.state[0] + (size_t)(row0 + r) * D, kc * 8, D, v);
                float* d = sH + (size_t)r * DP + kc * 8;
                *reinterpret_cast<float4*>(d) = make_float4(v[0], v[1], v[2], v[3]);
                *reinterpret_cast<float4*>(d + 4) = make_float4(v[4], v[5], v[6], v[7]);
            }
            workers_sync(abortp, ok);
        }
        for (int l = l_begin; l < l_end && ok; ++l) {
            // ---- S = A . H for the tile's rows -> operand tile (hi / lo); rows beyond the tile are zero
            {
                int beg = 0, end = 0;
                if (row < rows) { beg = __ldg(p.row_ptr + row0 + row); end = __ldg(p.row_ptr + row0 + row + 1); }
                const float* gin = p.state[l];
                for (int kc = cg; kc < NKC; kc += NCG) {
                    float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
                    for (int m = beg; m < end; ++m) {
                        const int s = __ldg(p.csr_src + m);
                        const float w = __ldg(p.slot_w + m);
                        float x[8];
                        if (LOCAL) lds8(sH + (size_t)(s - row0) * DP + kc * 8, x);
                        else load8_guarded_cg(gin + (size_t)s * D, kc * 8, D, x);
#pragma unroll
                        for (int j = 0; j < 8; ++j) acc[j] = fmaf(w, x[j], acc[j]);
                    }
                    store_operand_chunk(opS, KGS, PART_B, kc, row, acc);
                }
            }
            fence_async_smem();
            workers_sync(abortp, ok);
            // ---- S . W_l on wgmma
            float acc[NF];
#pragma unroll
            for (int i = 0; i < NF; ++i) acc[i] = 0.f;
            gemm_narrow<NH, DP, X3, (uint32_t)KGS>(rd, acc, smem_u32(opS), a_row, nh * NH, lane);
            // ---- epilogue: bias, relu, dropout; the state goes back to the tile (LOCAL) and to global memory
            const bool to_smem = LOCAL && l + 1 < l_end;
            const bool to_global = !LOCAL || l + 1 == l_end || p.save;
            float* gout = p.state_w[l + 1];
#pragma unroll
            for (int j = 0; j < NJ; ++j)
#pragma unroll
                for (int hr = 0; hr < 2; ++hr) {
                    const int r = fr0 + 8 * hr, c = fc0 + 8 * j;
                    if (r >= rows) continue;
                    float v0 = 0.f, v1 = 0.f;
                    if (c < D) {
                        v0 = epilogue(acc[4 * j + 2 * hr], p, l, row0 + r, c);
                        v1 = epilogue(acc[4 * j + 2 * hr + 1], p, l, row0 + r, c + 1);
                        if (to_global) st2(gout + (size_t)(row0 + r) * D + c, v0, v1);
                    }
                    if (to_smem) st2(sH + (size_t)r * DP + c, v0, v1);
                }
            workers_sync(abortp, ok);   // the next layer's gather reads the new states and overwrites the operand tile
        }
        if (!ok && tid == 0) atomicExch(p.error_flag, 1);
    } else if (lane == 0) {
        // ============================================================ WEIGHT PRODUCER: W_l of every layer
        RingWriter wr{bar_full, bar_empty, abortp, ring, (uint32_t)nst, STAGE_B};
        for (int l = l_begin; l < l_end && wr.ok; ++l) wr.push(p.w_tiled[l], NKS);
        if (!wr.ok) atomicExch(p.error_flag, 3);
    }
    __syncthreads();
}

// ------------------------------------------------------------------------------------------------ fp32 CUDA cores
// One layer: CTA = 32 output rows, 8 warps.  Gather: warp w sums rows 4w .. 4w+3 (lanes over float4 columns).  GEMM: a thread owns 4 rows
// x 4 columns per item, W_l rows are read as float4 through L1.
__global__ void __launch_bounds__(F32_THREADS) gcn_fp32_kernel(const __grid_constant__ GcnParams p) {
    extern __shared__ __align__(16) float sS[];   // [32][D]
    const int D = p.D, l = p.g_layer, D4 = D >> 2;
    const int row0 = blockIdx.x * F32_ROWS;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const float* __restrict__ in = p.state[l];
    for (int rr = 0; rr < 4; ++rr) {
        const int r = warp * 4 + rr, v = row0 + r;
        int beg = 0, end = 0;
        if (v < p.V) { beg = __ldg(p.row_ptr + v); end = __ldg(p.row_ptr + v + 1); }
        for (int c4 = lane; c4 < D4; c4 += 32) {
            float4 s = make_float4(0.f, 0.f, 0.f, 0.f);
            for (int m = beg; m < end; ++m) {
                const float w = __ldg(p.slot_w + m);
                const float4 x = __ldcg(reinterpret_cast<const float4*>(in + (size_t)__ldg(p.csr_src + m) * D) + c4);
                s.x = fmaf(w, x.x, s.x); s.y = fmaf(w, x.y, s.y); s.z = fmaf(w, x.z, s.z); s.w = fmaf(w, x.w, s.w);
            }
            *reinterpret_cast<float4*>(sS + (size_t)r * D + 4 * c4) = s;
        }
    }
    __syncthreads();
    const float* __restrict__ W = p.kernel[l];
    float* out = p.state_w[l + 1];
    for (int it = threadIdx.x; it < (F32_ROWS / 4) * D4; it += F32_THREADS) {
        const int rq = it / D4, cq = it - rq * D4;
        float acc[4][4] = {{0.f}};
        const float* s0 = sS + (size_t)(rq * 4) * D;
        for (int k = 0; k < D; ++k) {
            const float4 w = __ldg(reinterpret_cast<const float4*>(W + (size_t)k * D) + cq);
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                const float a = s0[(size_t)i * D + k];
                acc[i][0] = fmaf(a, w.x, acc[i][0]); acc[i][1] = fmaf(a, w.y, acc[i][1]);
                acc[i][2] = fmaf(a, w.z, acc[i][2]); acc[i][3] = fmaf(a, w.w, acc[i][3]);
            }
        }
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const int v = row0 + rq * 4 + i;
            if (v >= p.V) continue;
            const int c = cq * 4;
            float4 o;
            o.x = epilogue(acc[i][0], p, l, v, c); o.y = epilogue(acc[i][1], p, l, v, c + 1);
            o.z = epilogue(acc[i][2], p, l, v, c + 2); o.w = epilogue(acc[i][3], p, l, v, c + 3);
            *reinterpret_cast<float4*>(out + (size_t)v * D + c) = o;
        }
    }
}

// ------------------------------------------------------------------------------------------------ streaming plan: the gather
// S = A . H of one layer, straight into the tile-major bf16 hi/lo operand image of ggnn_fwd_stream.cuh (ts::img_store_chunk), from the
// layer input's row-major fp32 state.  The arithmetic of gcn_wgmma_kernel's gather: per (row, 8 columns), acc = fmaf(w, x, acc) from 0 over
// the row's target-CSR slots in list order.  Rows V .. ntiles*128 and columns D .. DP are written as zeros; no read leaves the V x D state.
// A warp covers 4 rows x 8 column chunks, so each message it reads is 256 contiguous bytes of a row and each image store 64 contiguous
// bytes of a k-group.
__global__ void __launch_bounds__(256) gcn_gather_image_kernel(const int* __restrict__ row_ptr, const int* __restrict__ csr_src,
                                                               const float* __restrict__ slot_w, const float* __restrict__ h,
                                                               uint8_t* __restrict__ img, int V, int D, int DP, int ntiles) {
    const int NKC = DP >> 3, NKS = DP >> 4, ncg = (NKC + 7) >> 3;
    const long long nwarps = (long long)ntiles * (ts::TILE_M / 4) * ncg;
    const long long w = (blockIdx.x * (long long)blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (w >= nwarps) return;
    const int rg = (int)(w / ncg), cg = (int)(w - (long long)rg * ncg);
    const int row = rg * 4 + (lane & 3), kc = cg * 8 + (lane >> 2);
    if (kc >= NKC) return;
    float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    if (row < V) {
        const int beg = __ldg(row_ptr + row), end = __ldg(row_ptr + row + 1);
        for (int m = beg; m < end; ++m) {
            const int s = __ldg(csr_src + m);
            const float wm = __ldg(slot_w + m);
            float x[8];
            tc::load8_guarded_cg(h + (size_t)s * D, kc * 8, D, x);
#pragma unroll
            for (int j = 0; j < 8; ++j) acc[j] = fmaf(wm, x[j], acc[j]);
        }
    }
    ts::img_store_chunk(img, NKS, row >> 7, row & 127, kc * 8, acc);
}

// ------------------------------------------------------------------------------------------------ backward helper
// gradient through relu and state dropout of a hidden layer, from the layer's saved output y = relu(pre) * mask / keep:
// y > 0 exactly where the unit was kept and active, so  d pre = y > 0 ? dy / keep : 0  (no mask regeneration needed)
__global__ void gcn_relu_dropout_grad_kernel(const float* __restrict__ dy, const float* __restrict__ y, float* __restrict__ dpre, float inv_keep,
                                             long long n) {
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
        dpre[i] = y[i] > 0.0f ? dy[i] * inv_keep : 0.0f;
}

// ------------------------------------------------------------------------------------------------ message-weighted batches: d w
// One layer's source-row pass of the backward on a message-weighted batch (ggnn_gcn_backward_weighted), over the source-keyed CSR
// (trow [V+1], ttgt / tslot / tslotw [nnz]): for every source row j and each of its entries e (target i = ttgt[e]), in order,
//   dH[j]               = sum_e tslotw[e] * dS[i]     per element fmaf(w, x, acc) from 0: csr_gather_all_kernel's arithmetic, bit for bit
//   dw_slot[tslot[e]]  += <dS[i], H[j]>               the entry's term of d w = sum_l <dS_l[i], H_l[j]>
// dS[i] is read once for both.  One warp per source row; lane c owns the float4 column chunks c, c + 32, ... (CHUNKS of them, so
// D <= 128 * CHUNKS), H[j] stays in registers.  The lanes' partial dots are added by a fixed butterfly and lane 0 adds the sum into the
// entry's target slot, which no other entry shares: no atomics, the same bits on every call.  WANT_DH = false (layer 0 without d h0) forms
// d w alone.  D is a multiple of 4; rows are 16-byte aligned.
template <int CHUNKS, bool WANT_DH>
__global__ void __launch_bounds__(256) gcn_source_grad_kernel(const int* __restrict__ trow, const int* __restrict__ ttgt,
                                                              const int* __restrict__ tslot, const float* __restrict__ tslotw,
                                                              const float* __restrict__ dS, const float* __restrict__ H, float* __restrict__ dH,
                                                              float* __restrict__ dw_slot, int V, int D) {
    const int j = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (j >= V) return;
    const int D4 = D >> 2;
    float4 h[CHUNKS], acc[CHUNKS];
#pragma unroll
    for (int c = 0; c < CHUNKS; ++c) {
        const int c4 = lane + 32 * c;
        h[c] = c4 < D4 ? reinterpret_cast<const float4*>(H + (size_t)j * D)[c4] : make_float4(0.f, 0.f, 0.f, 0.f);
        acc[c] = make_float4(0.f, 0.f, 0.f, 0.f);
    }
    const int beg = trow[j], end = trow[j + 1];
    for (int e = beg; e < end; ++e) {
        const float a = tslotw[e];
        const float4* row = reinterpret_cast<const float4*>(dS + (size_t)ttgt[e] * D);
        float s = 0.f;
#pragma unroll
        for (int c = 0; c < CHUNKS; ++c) {
            const int c4 = lane + 32 * c;
            if (c4 < D4) {
                const float4 x = row[c4];
                if (WANT_DH) {
                    acc[c].x = fmaf(a, x.x, acc[c].x); acc[c].y = fmaf(a, x.y, acc[c].y);
                    acc[c].z = fmaf(a, x.z, acc[c].z); acc[c].w = fmaf(a, x.w, acc[c].w);
                }
                s = fmaf(x.x, h[c].x, s); s = fmaf(x.y, h[c].y, s); s = fmaf(x.z, h[c].z, s); s = fmaf(x.w, h[c].w, s);
            }
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
        if (lane == 0) dw_slot[tslot[e]] += s;
    }
    if (WANT_DH) {
#pragma unroll
        for (int c = 0; c < CHUNKS; ++c) {
            const int c4 = lane + 32 * c;
            if (c4 < D4) reinterpret_cast<float4*>(dH + (size_t)j * D)[c4] = acc[c];
        }
    }
}

}  // namespace gcn
}  // namespace ggnn
