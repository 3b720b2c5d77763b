// Fused GGNN propagation, fp32 FFMA path (sm_90a).
//
// One CTA owns one tile of MT = 8*RG consecutive node rows.  In LOCAL mode the tile is a union of whole
// connected components (the batch is a disjoint union of small graphs, sparse:279-280), so EVERY layer and
// timestep of compute_final_node_representations (sparse:131-216) runs inside this one launch with the
// node states resident in shared memory: per step
//     for each edge type t present in the tile:  A_t[row] = sum_{msgs (src->row) of type t} h[src]   (gather :161 + segment_sum :198)
//                                                agg     += A_t . W[l][t]                            (matmul :163, summed over types)
//     agg += indeg . B[l]  (:202-204);  agg /= (sum indeg + 1e-7)  (:206-209)
//     GRU: [r|u] = sigmoid([res..., agg, h] . K_g + b_g);  c = act([res..., agg, r*h] . K_c + b_c);  h = u*h + (1-u)*c   (:215, TF-1.3 GRUCell)
//     CudnnCompatibleGRUCell (:105-108): same gates;  c = tanh([res..., agg] . K_in + b_in + r*(h . K_hid + b_hid))
//     RNN: h = act([res..., agg, h] . K + b)                                                         (BasicRNNCell)
// (sum-then-transform is algebraically identical to the reference's transform-then-sum and needs V*T*D*D
// instead of M*D*D MACs only where a (target,type) pair exists; types absent from a tile are skipped.)
// In GLOBAL mode (a component larger than a tile, e.g. one 10k-node graph) the same kernel runs ONE step per
// launch, gathering source rows from the previous step's state in global memory (L2 resident).
//
// GEMMs: warp = 8 rows x (32*NB strided columns); A operand broadcast from shared memory (LDS.128), the weight
// operand streamed global->shared with cp.async in KC-row double-buffered stages, accumulators in registers.
#pragma once
#include "ggnn_common.cuh"

namespace ggnn {

struct ASeg {
    const float* ptr;  // shared tile base ([MT][lda]) or global state base ([V][lda])
    int lda;
    int k;             // K extent of the segment (multiple of 4)
    int is_global;
};

// acc[j][r] += sum_k A[8*rg + r][k] * B[k][col0 + cbase + 32*j]
template <int NB, int RG, int CS>
__device__ __forceinline__ void gemm_accumulate(float (&acc)[NB][8], const ASeg* segs, int nseg,
                                                const float* __restrict__ gB, int ldb, int col0, int ncols,
                                                float* sB, float* sStage, int row0, int rows) {
    constexpr int PW = 32 * NB * CS;
    constexpr int MT = RG * 8;
    constexpr int NT = RG * CS * 32;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int rg = warp % RG, cs = warp / RG;
    const int cbase = cs * 32 * NB + lane;
    const bool active = (rg * 8 < rows) && (cs * 32 * NB < ncols);
    const int nvec = ncols >> 2;

    int nchunks = 0;
    for (int s = 0; s < nseg; ++s) nchunks += (segs[s].k + KC - 1) / KC;

    auto issue = [&](int buf, int s, int k0, int krow) {
        const ASeg sg = segs[s];
        const int kc = min(KC, sg.k - k0);
        for (int idx = tid; idx < kc * nvec; idx += NT) {
            const int k = idx / nvec, c = (idx - k * nvec) << 2;
            cp_async16(&sB[(buf * KC + k) * PW + c], &gB[(size_t)(krow + k) * ldb + col0 + c]);
        }
        if (sg.is_global) {
            const int kv = kc >> 2;
            for (int idx = tid; idx < rows * kv; idx += NT) {
                const int r = idx / kv, c = (idx - r * kv) << 2;
                cp_async16(&sStage[(buf * MT + r) * KC + c], &sg.ptr[(size_t)(row0 + r) * sg.lda + k0 + c]);
            }
        }
        cp_async_commit();
    };

    int is = 0, ik = 0, ikrow = 0;  // issue cursor: segment, k offset in segment, global K row
    int cseg = 0, ck = 0;           // compute cursor
    issue(0, is, ik, ikrow);
    {
        const int kc = min(KC, segs[is].k - ik);
        ikrow += kc; ik += kc;
        if (ik >= segs[is].k) { ++is; ik = 0; }
    }
    for (int c = 0; c < nchunks; ++c) {
        if (c + 1 < nchunks) {
            issue((c + 1) & 1, is, ik, ikrow);
            const int kc = min(KC, segs[is].k - ik);
            ikrow += kc; ik += kc;
            if (ik >= segs[is].k) { ++is; ik = 0; }
            cp_async_wait<1>();
        } else {
            cp_async_wait<0>();
        }
        __syncthreads();
        const ASeg sg = segs[cseg];
        const int kc = min(KC, sg.k - ck);
        if (active) {
            const float* A;
            int lda;
            if (sg.is_global) { A = sStage + ((c & 1) * MT + rg * 8) * KC; lda = KC; }
            else              { A = sg.ptr + (size_t)(rg * 8) * sg.lda + ck; lda = sg.lda; }
            const float* Bc = sB + (c & 1) * KC * PW + cbase;
#pragma unroll 1
            for (int kk = 0; kk < kc; kk += 4) {
                float4 a[8];
#pragma unroll
                for (int r = 0; r < 8; ++r) a[r] = *reinterpret_cast<const float4*>(A + r * lda + kk);
#pragma unroll
                for (int q = 0; q < 4; ++q) {
                    float b[NB];
#pragma unroll
                    for (int j = 0; j < NB; ++j) b[j] = Bc[(kk + q) * PW + 32 * j];
#pragma unroll
                    for (int j = 0; j < NB; ++j) {
#pragma unroll
                        for (int r = 0; r < 8; ++r) {
                            const float av = q == 0 ? a[r].x : q == 1 ? a[r].y : q == 2 ? a[r].z : a[r].w;
                            acc[j][r] = fmaf(av, b[j], acc[j][r]);
                        }
                    }
                }
            }
        }
        __syncthreads();
        ck += kc;
        if (ck >= sg.k) { ++cseg; ck = 0; }
    }
}

template <int NB>
__device__ __forceinline__ void zero_acc(float (&acc)[NB][8]) {
#pragma unroll
    for (int j = 0; j < NB; ++j)
#pragma unroll
        for (int r = 0; r < 8; ++r) acc[j][r] = 0.0f;
}

template <int RG, int CS, int NB1, int NB2, bool LOCAL, int MINB>
__global__ void __launch_bounds__(RG * CS * 32, MINB) ggnn_fwd_ffma_kernel(const __grid_constant__ FwdParams p) {
    constexpr int MT = RG * 8;
    constexpr int NT = RG * CS * 32;
    constexpr int NWARP = NT / 32;
    constexpr int PW1 = 32 * NB1 * CS;
    constexpr int PW2 = 32 * NB2 * CS;
    constexpr int PWMAX = PW2 > PW1 ? PW2 : PW1;
    extern __shared__ __align__(16) float smem[];
    const int D = p.D, T = p.T;
    const int D4 = D >> 2;
    float* sH = smem;
    float* sX = sH + MT * D;
    float* sA = sX + MT * D;
    float* sU = sA + MT * D;
    float* sB = sU + MT * D;                // [2][KC][PWMAX]
    float* sStage = sB + 2 * KC * PWMAX;    // [2][MT][KC]
    float* sBias = sStage + 2 * MT * KC;    // [T][D]

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int rg = warp % RG, cs = warp / RG;
    const int tile = blockIdx.x;
    const int row0 = p.tile_start[tile];
    const int rows = p.tile_start[tile + 1] - row0;
    const unsigned tmask = p.tile_mask[tile];
    const size_t VD = (size_t)p.V * D;

    // ---- load the tile's node states (zero the padding rows of every tile buffer)
    {
        const float* hin = LOCAL ? p.state[0] : p.g_in;
        for (int idx = tid; idx < MT * D4; idx += NT) {
            const int r = idx / D4, c = (idx - r * D4) << 2;
            float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
            if (r < rows) v = *reinterpret_cast<const float4*>(hin + (size_t)(row0 + r) * D + c);
            *reinterpret_cast<float4*>(sH + r * D + c) = v;
            const float4 z = make_float4(0.f, 0.f, 0.f, 0.f);
            *reinterpret_cast<float4*>(sX + r * D + c) = z;
            *reinterpret_cast<float4*>(sA + r * D + c) = z;
            *reinterpret_cast<float4*>(sU + r * D + c) = z;
        }
    }
    __syncthreads();

    const int l_begin = LOCAL ? 0 : p.g_layer;
    const int l_end = LOCAL ? p.L : p.g_layer + 1;
    for (int l = l_begin; l < l_end; ++l) {
        const LayerDev& ly = p.layer[l];
        if (p.use_bias) {
            for (int idx = tid; idx < T * D; idx += NT) sBias[idx] = ly.edge_b[idx];
        }
        const int s_begin = LOCAL ? 0 : p.g_step;
        const int s_end = LOCAL ? ly.steps : p.g_step + 1;
        for (int s = s_begin; s < s_end; ++s) {
            const size_t save_off = (size_t)(p.step_base[l] + s) * VD;
            if (p.save) {
                for (int idx = tid; idx < rows * D4; idx += NT) {
                    const int r = idx / D4, c = (idx - r * D4) << 2;
                    *reinterpret_cast<float4*>(p.save_buf.h_in + save_off + (size_t)(row0 + r) * D + c) =
                        *reinterpret_cast<const float4*>(sH + r * D + c);
                }
            }
            // ------------------------------------------------ message phase: agg = sum_t A_t . W_t
            float acc1[NB1][8];
            zero_acc<NB1>(acc1);
            float* att = nullptr;
            if (p.use_att) {
                // ---- propagation attention (sparse:170-196): a softmax over ALL incoming messages of a node (every edge type), score =
                // <h[source], h[target]> * edge_type_attention_weight[type].  One warp per target row; the rows v*T .. v*T+T-1 of the
                // target-keyed CSR are contiguous, so a node's messages are one slot range.  att[slot] ends up holding the probability.
                att = p.att + (size_t)(p.step_base[l] + s) * p.att_stride;
                for (int r = warp; r < rows; r += NWARP) {
                    const int v = row0 + r;
                    const float* hv = LOCAL ? (sH + (size_t)r * D) : (p.g_in + (size_t)v * D);
                    const int mbeg = p.row_ptr[(size_t)v * T], mend = p.row_ptr[(size_t)(v + 1) * T];
                    float mx = -INFINITY;
                    for (int t = 0; t < T; ++t) {
                        const float aw = ly.att_w[t];
                        const int beg = p.row_ptr[(size_t)v * T + t], end = p.row_ptr[(size_t)v * T + t + 1];
                        for (int m = beg; m < end; ++m) {
                            const int src = p.csr_src[m];
                            const float* hp = LOCAL ? (sH + (size_t)(src - row0) * D) : (p.g_in + (size_t)src * D);
                            float dot = 0.f;
                            for (int c4 = lane; c4 < D4; c4 += 32) {
                                const float4 a = *reinterpret_cast<const float4*>(hp + (c4 << 2));
                                const float4 b = *reinterpret_cast<const float4*>(hv + (c4 << 2));
                                dot += a.x * b.x + a.y * b.y + a.z * b.z + a.w * b.w;
                            }
#pragma unroll
                            for (int o = 16; o > 0; o >>= 1) dot += __shfl_xor_sync(0xffffffffu, dot, o);
                            const float sc = dot * aw;
                            if (lane == 0) att[m] = sc;
                            mx = fmaxf(mx, sc);
                        }
                    }
                    __syncwarp();
                    float sum = 0.f;
                    for (int m = mbeg + lane; m < mend; m += 32) {
                        const float ex = expf(att[m] - mx);
                        att[m] = ex;
                        sum += ex;
                    }
#pragma unroll
                    for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
                    const float den = sum + 1e-7f;   // SMALL_NUMBER, sparse:194
                    for (int m = mbeg + lane; m < mend; m += 32) att[m] = att[m] / den;
                    __syncwarp();
                }
                // the same warp gathers the same rows below, so __syncwarp is all the ordering the att[] values need
            }
            // per-slot message weights: the attention probabilities, or the entries of a weighted dense adjacency
            const float* msg_w = att ? att : p.slot_w;
            for (int t = 0; t < T; ++t) {
                if (!((tmask >> t) & 1u)) continue;
                // A_t rows: sum of the source states of the row's incoming type-t messages (CSR order = message order)
                for (int r = warp; r < rows; r += NWARP) {
                    const int v = row0 + r;
                    const int beg = p.row_ptr[(size_t)v * T + t], end = p.row_ptr[(size_t)v * T + t + 1];
                    for (int c4 = lane; c4 < D4; c4 += 32) {
                        float4 sum = make_float4(0.f, 0.f, 0.f, 0.f);
                        if (msg_w) {   // weighted messages (attention: sparse:196; a weighted adjacency: dense:110-112)
                            for (int m = beg; m < end; ++m) {
                                const int src = p.csr_src[m];
                                const float a = msg_w[m];
                                const float* hp = LOCAL ? (sH + (size_t)(src - row0) * D) : (p.g_in + (size_t)src * D);
                                const float4 hv = *reinterpret_cast<const float4*>(hp + (c4 << 2));
                                sum.x = fmaf(a, hv.x, sum.x); sum.y = fmaf(a, hv.y, sum.y);
                                sum.z = fmaf(a, hv.z, sum.z); sum.w = fmaf(a, hv.w, sum.w);
                            }
                        } else
                        for (int m = beg; m < end; ++m) {
                            const int src = p.csr_src[m];
                            const float* hp = LOCAL ? (sH + (size_t)(src - row0) * D) : (p.g_in + (size_t)src * D);
                            const float4 hv = *reinterpret_cast<const float4*>(hp + (c4 << 2));
                            sum.x += hv.x; sum.y += hv.y; sum.z += hv.z; sum.w += hv.w;
                        }
                        *reinterpret_cast<float4*>(sA + r * D + (c4 << 2)) = sum;
                    }
                }
                __syncthreads();
                ASeg seg{sA, D, D, 0};
                gemm_accumulate<NB1, RG, CS>(acc1, &seg, 1, ly.edge_w + (size_t)t * D * D, D, 0, D, sB, sStage, row0, rows);
            }
            // epilogue: + indeg . B  (sparse:202-204), / (deg + 1e-7) (sparse:206-209)  -> sX
#pragma unroll
            for (int j = 0; j < NB1; ++j) {
                const int col = cs * 32 * NB1 + lane + 32 * j;
                if (col < D) {
#pragma unroll
                    for (int r = 0; r < 8; ++r) {
                        const int row = rg * 8 + r;
                        if (row < rows) {
                            float v = acc1[j][r];
                            if (p.use_bias) {
                                for (int t = 0; t < T; ++t) v = fmaf(p.indeg[(size_t)(row0 + row) * T + t], sBias[t * D + col], v);
                            }
                            if (p.use_avg) v = v / p.denom[row0 + row];
                            sX[row * D + col] = v;
                            if (p.save) p.save_buf.agg[save_off + (size_t)(row0 + row) * D + col] = v;
                        }
                    }
                }
            }
            __syncthreads();

            // ------------------------------------------------ cell
            ASeg segs[MAX_RES + 2];
            int nseg = 0;
            for (int i = 0; i < ly.nres; ++i) segs[nseg++] = ASeg{p.state[ly.res[i]], D, D, 1};
            segs[nseg++] = ASeg{sX, D, D, 0};
            segs[nseg++] = ASeg{sH, D, D, 0};

            if (p.cell == CELL_GRU || p.cell == CELL_CUDNN_GRU) {
                // CudnnCompatibleGRUCell (tf.contrib.cudnn_rnn, sparse:105-108): same gates, but the reset gate multiplies the recurrent
                // projection AFTER the matmul:  c = tanh(x . K_in + b_in + r * (h . K_hid + b_hid)),  K_in / K_hid = the first Din / last D rows of cand_k
                const bool cudnn = p.cell == CELL_CUDNN_GRU;
                const int N2 = 2 * D;
                for (int col0 = 0; col0 < N2; col0 += PW2) {
                    const int ncols = min(PW2, N2 - col0);
                    float acc2[NB2][8];
                    zero_acc<NB2>(acc2);
                    gemm_accumulate<NB2, RG, CS>(acc2, segs, nseg, ly.gate_k, N2, col0, ncols, sB, sStage, row0, rows);
#pragma unroll
                    for (int j = 0; j < NB2; ++j) {
                        const int cl = cs * 32 * NB2 + lane + 32 * j;
                        if (cl < ncols) {
                            const int g = col0 + cl;
                            const float bg = ly.gate_b[g];
#pragma unroll
                            for (int r = 0; r < 8; ++r) {
                                const int row = rg * 8 + r;
                                if (row < rows) {
                                    const float sg = sigmoidf_acc(acc2[j][r] + bg);
                                    if (g < D) {
                                        sA[row * D + g] = cudnn ? sg : sg * sH[row * D + g];  // r*h, the candidate's recurrent operand (cudnn: r itself)
                                        if (p.save) p.save_buf.r[save_off + (size_t)(row0 + row) * D + g] = sg;
                                    } else {
                                        sU[row * D + (g - D)] = sg;
                                        if (p.save) p.save_buf.u[save_off + (size_t)(row0 + row) * D + (g - D)] = sg;
                                    }
                                }
                            }
                        }
                    }
                }
                __syncthreads();
                if (cudnn) {
                    // q = h . K_hid + b_hid (kept for the backward pass);  sA <- r * q.  The thread that wrote sA[row][col] = r in the gate
                    // epilogue is not this one (different column mapping) -- the __syncthreads above orders the two.
                    ASeg hseg{sH, D, D, 0};
                    zero_acc<NB1>(acc1);
                    gemm_accumulate<NB1, RG, CS>(acc1, &hseg, 1, ly.cand_k + (size_t)D * (ly.nres + 1) * D, D, 0, D, sB, sStage, row0, rows);
#pragma unroll
                    for (int j = 0; j < NB1; ++j) {
                        const int col = cs * 32 * NB1 + lane + 32 * j;
                        if (col < D) {
                            const float bh = ly.cand_hb[col];
#pragma unroll
                            for (int r = 0; r < 8; ++r) {
                                const int row = rg * 8 + r;
                                if (row < rows) {
                                    const float q = acc1[j][r] + bh;
                                    sA[row * D + col] *= q;
                                    if (p.save) p.save_buf.q[save_off + (size_t)(row0 + row) * D + col] = q;
                                }
                            }
                        }
                    }
                    // the same thread reads sA[row][col] again in the candidate epilogue below (same mapping): no barrier needed for it
                } else {
                    segs[nseg - 1] = ASeg{sA, D, D, 0};
                }
                zero_acc<NB1>(acc1);
                gemm_accumulate<NB1, RG, CS>(acc1, segs, cudnn ? nseg - 1 : nseg, ly.cand_k, D, 0, D, sB, sStage, row0, rows);
#pragma unroll
                for (int j = 0; j < NB1; ++j) {
                    const int col = cs * 32 * NB1 + lane + 32 * j;
                    if (col < D) {
                        const float bc = ly.cand_b[col];
#pragma unroll
                        for (int r = 0; r < 8; ++r) {
                            const int row = rg * 8 + r;
                            if (row < rows) {
                                float pre = acc1[j][r] + bc;
                                if (cudnn) pre += sA[row * D + col];
                                const float c = activate(pre, p.act);
                                const float u = sU[row * D + col];
                                const float h = sH[row * D + col];
                                float hn = u * h + (1.0f - u) * c;
                                if (p.drop_keep < 1.0f) hn = dropout_apply(hn, p.drop_seed, p.step_base[l] + s, p.V, D, row0 + row, col, p.drop_keep);
                                sH[row * D + col] = hn;
                                if (p.save) p.save_buf.c[save_off + (size_t)(row0 + row) * D + col] = c;
                            }
                        }
                    }
                }
                __syncthreads();
            } else {
                zero_acc<NB1>(acc1);
                gemm_accumulate<NB1, RG, CS>(acc1, segs, nseg, ly.cand_k, D, 0, D, sB, sStage, row0, rows);
#pragma unroll
                for (int j = 0; j < NB1; ++j) {
                    const int col = cs * 32 * NB1 + lane + 32 * j;
                    if (col < D) {
                        const float bc = ly.cand_b[col];
#pragma unroll
                        for (int r = 0; r < 8; ++r) {
                            const int row = rg * 8 + r;
                            if (row < rows) {
                                float hn = activate(acc1[j][r] + bc, p.act);
                                if (p.drop_keep < 1.0f) hn = dropout_apply(hn, p.drop_seed, p.step_base[l] + s, p.V, D, row0 + row, col, p.drop_keep);
                                sA[row * D + col] = hn;
                            }
                        }
                    }
                }
                __syncthreads();
                float* tmp = sH; sH = sA; sA = tmp;  // new state lives in the former scratch tile
            }
        }  // steps
        // ---- layer output -> node_states_per_layer[l+1] (LOCAL) / step output (GLOBAL)
        float* outp = LOCAL ? p.state_w[l + 1] : p.g_out;
        for (int idx = tid; idx < rows * D4; idx += NT) {
            const int r = idx / D4, c = (idx - r * D4) << 2;
            *reinterpret_cast<float4*>(outp + (size_t)(row0 + r) * D + c) = *reinterpret_cast<const float4*>(sH + r * D + c);
        }
        __syncthreads();
    }
}

}  // namespace ggnn
