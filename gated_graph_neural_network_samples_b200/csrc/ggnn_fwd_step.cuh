// Per-timestep fp32 propagation (sm_90a), the fp32 path of hidden sizes above 256: precision fp32, propagation attention and
// CudnnCompatibleGRUCell there.  The fused fp32 tile kernel (ggnn_fwd_ffma.cuh) keeps four MT x D fp32 tiles in shared memory, which no
// longer fit an SM at D = 512, so here one timestep is a short sequence of launches over the whole batch, each with the tile kernel's
// arithmetic (fp32 FFMA, the same summation orders):
//   [attention]  alpha[slot] = softmax over the messages into v of <h[src], h[v]> * a_t      (step::attention_kernel, one warp per node)
//   gather       A[v, t*D..] = sum over the type-t messages into v of (alpha or slot weight) * h[src]  (bwd::csr_gather_all_kernel)
//   messages     agg = sum_t A_t . W_t                                    (bwd::gemm_nt_kernel over the transposed W_t, one launch)
//                agg = (agg + indeg . B) / denom                          (step::agg_epilogue_kernel)
//   GRU gates    [r|u] = sigmoid([res.. | agg | h] . K_g + b_g)          (gemm_nt + step::gate_epilogue_kernel; writes r*h)
//   [cudnn]      q = h . K_hid                                            (gemm_nt; + b_hid in the update)
//   candidate    c = act([res.. | agg | r*h] . K_c + b_c),  h' = u*h + (1-u)*c, state dropout  (gemm_nt + step::update_kernel)
//   RNN          h' = act([res.. | agg | h] . K + b)
// The cell input row [res.. | agg | h] is one [V, D*(R+2)] array, so that every GEMM is a single gemm_nt launch.  No atomics: the forward is
// bit-identical from run to run.  The saved activations are those of the tile kernel, in its layout.
#pragma once
#include "ggnn_common.cuh"

namespace ggnn {
namespace step {

// dst[b][c][r] = src[b][r][c] for `rows` x `cols` matrices, batch b = blockIdx.z; 32 x 32 tiles, 32 x 8 threads
__global__ void __launch_bounds__(256) transpose_kernel(const float* __restrict__ src, float* __restrict__ dst, int rows, int cols) {
    __shared__ float tile[32][33];
    const size_t off = (size_t)blockIdx.z * rows * cols;
    const int c0 = blockIdx.x * 32, r0 = blockIdx.y * 32;
    for (int i = threadIdx.y; i < 32; i += 8) {
        const int r = r0 + i, c = c0 + threadIdx.x;
        if (r < rows && c < cols) tile[i][threadIdx.x] = src[off + (size_t)r * cols + c];
    }
    __syncthreads();
    for (int i = threadIdx.y; i < 32; i += 8) {
        const int c = c0 + i, r = r0 + threadIdx.x;
        if (r < rows && c < cols) dst[off + (size_t)c * rows + r] = tile[threadIdx.x][i];
    }
}

// Propagation attention (sparse:170-196), the pre-pass of the tile kernel on its own: one warp per target row; the rows v*T .. v*T+T-1 of
// the target-keyed CSR are contiguous, so a node's messages are one slot range.  att[slot] ends up holding the probability.
__global__ void __launch_bounds__(256) attention_kernel(const int* __restrict__ row_ptr, const int* __restrict__ csr_src, const float* __restrict__ h,
                                                        const float* __restrict__ att_w, float* __restrict__ att, int V, int D, int T) {
    const int v = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (v >= V) return;
    const int D4 = D >> 2;
    const float* hv = h + (size_t)v * D;
    const int mbeg = row_ptr[(size_t)v * T], mend = row_ptr[(size_t)(v + 1) * T];
    float mx = -INFINITY;
    for (int t = 0; t < T; ++t) {
        const float aw = att_w[t];
        const int beg = row_ptr[(size_t)v * T + t], end = row_ptr[(size_t)v * T + t + 1];
        for (int m = beg; m < end; ++m) {
            const float* hp = h + (size_t)csr_src[m] * D;
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
}

// The message epilogue, in place in the cell input row X [V, ldx]: X[v, xoff + c] = (sum_t A_t W_t + sum_t indeg[v,t] B[t,c]) / denom[v]
// (sparse:202-209; bias / denom null when unused); also copies the step's input state h into X[v, hoff..] and saves agg and h_in.
__global__ void agg_epilogue_kernel(float* __restrict__ X, int ldx, int xoff, int hoff, const float* __restrict__ h, const float* __restrict__ bias,
                                    const float* __restrict__ indeg, const float* __restrict__ denom, float* __restrict__ sv_agg,
                                    float* __restrict__ sv_h, long long n, int D, int T) {
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        const long long row = i / D;
        const int col = (int)(i - row * D);
        float* x = X + row * ldx;
        float v = x[xoff + col];
        if (bias)
            for (int t = 0; t < T; ++t) v = fmaf(indeg[row * T + t], bias[(size_t)t * D + col], v);
        if (denom) v = v / denom[row];
        x[xoff + col] = v;
        const float hh = h[i];
        x[hoff + col] = hh;
        if (sv_agg) { sv_agg[i] = v; sv_h[i] = hh; }
    }
}

// The GRU gates: G [V, 2D] pre-activations -> [r | u] = sigmoid(G + b_g) in place; X[v, roff + c] = r*h, the candidate's recurrent operand
// (null for CudnnCompatibleGRUCell, whose reset gate multiplies the recurrent projection in update_kernel).
__global__ void gate_epilogue_kernel(float* __restrict__ G, const float* __restrict__ bias, const float* __restrict__ h, float* __restrict__ X, int ldx,
                                     int roff, float* __restrict__ sv_r, float* __restrict__ sv_u, long long n, int D) {
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        const long long row = i / D;
        const int col = (int)(i - row * D);
        float* g = G + row * 2 * D;
        const float r = sigmoidf_acc(g[col] + bias[col]), u = sigmoidf_acc(g[D + col] + bias[D + col]);
        g[col] = r;
        g[D + col] = u;
        if (X) X[row * ldx + roff + col] = r * h[i];
        if (sv_r) { sv_r[i] = r; sv_u[i] = u; }
    }
}

// The candidate epilogue and the state update.  C = the candidate GEMM, G = [r | u] (null for the RNN cell), Q = h . K_hid (Cudnn-
// CompatibleGRUCell only: c = tanh(C + b_in + r*(Q + b_hid)), q saved).  State dropout with the counter hash at global step gstep.
__global__ void update_kernel(const float* __restrict__ C, const float* __restrict__ bias, const float* __restrict__ G, const float* __restrict__ Q,
                              const float* __restrict__ qbias, const float* __restrict__ h, float* __restrict__ h_out, float* __restrict__ sv_c,
                              float* __restrict__ sv_q, int act, float keep, unsigned long long seed, int gstep, int V, long long n, int D) {
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        const long long row = i / D;
        const int col = (int)(i - row * D);
        float pre = C[i] + bias[col];
        float hn;
        if (G) {
            if (Q) {
                const float q = Q[i] + qbias[col];
                pre += G[row * 2 * D + col] * q;
                if (sv_q) sv_q[i] = q;
            }
            const float c = activate(pre, act);
            const float u = G[row * 2 * D + D + col];
            hn = u * h[i] + (1.0f - u) * c;
            if (sv_c) sv_c[i] = c;
        } else {
            hn = activate(pre, act);
        }
        if (keep < 1.0f) hn = dropout_apply(hn, seed, gstep, V, D, (int)row, col, keep);
        h_out[i] = hn;
    }
}

}  // namespace step
}  // namespace ggnn
