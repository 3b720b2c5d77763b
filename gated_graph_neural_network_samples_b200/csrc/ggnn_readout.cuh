// Gated regression readout (sparse:220-231, dense:119-129) for one task, fused:
//   val[v]  = sigmoid([h_T[v] | h_0[v]] . w_gate + b_gate) * (h_T[v] . w_trans + b_trans) * mask[v]
//   out[g]  = sum of val over the nodes of graph g          (tf.unsorted_segment_sum / masked reduce_sum)
// The reference's readout MLPs have no hidden layers (chem_tensorflow.py:153-157), so each is one affine map to a scalar.
// Forward: one warp per node computes val[v] (every node row read once, float4), then one thread per graph adds its nodes in
// order (the serial order of TF's CPU segment sum, deterministic); node lists not grouped by graph take an atomicAdd stage (in deterministic
// mode, the same per-graph order through a by-graph permutation).  Backward: one warp per node recomputes the two dot products, writes d h_T,
// accumulates the weight gradients in registers and reduces them per block.
#pragma once
#include "ggnn_common.cuh"
#include "ggnn_bwd.cuh"

namespace ggnn {
namespace readout {

// The backward kernels hold DPL columns per lane (column lane + 32 j): instances DPL = 8 for D <= 256 and DPL = 16 for 256 < D <= 512.
constexpr int MAX_D_PER_LANE = 16;

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

struct Weights {
    const float* w_gate;    // [2D]  rows of the [2D,1] kernel: first D act on h_T, last D on h_0
    const float* b_gate;    // [1]
    const float* w_trans;   // [D]
    const float* b_trans;   // [1]
};

__device__ __forceinline__ void node_dots(const float* __restrict__ hT, const float* __restrict__ h0, const Weights& w, int D, int lane,
                                          float& gate_pre, float& trans_pre) {
    float g = 0.f, t = 0.f;
    for (int d = lane; d < D; d += 32) {
        const float a = hT[d];
        g = fmaf(a, w.w_gate[d], g);
        g = fmaf(h0[d], w.w_gate[D + d], g);
        t = fmaf(a, w.w_trans[d], t);
    }
    gate_pre = warp_sum(g) + w.b_gate[0];
    trans_pre = warp_sum(t) + w.b_trans[0];
}

// stage 1: one warp per node -> val[v]   (fully parallel; the node rows are read exactly once, 16 bytes per lane)
__global__ void __launch_bounds__(256) readout_node_kernel(const float* __restrict__ h_last, const float* __restrict__ h0, Weights w,
                                                           const float* __restrict__ mask, float* __restrict__ val, int V, int D) {
    const int v = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (v >= V) return;
    const float4* hT = reinterpret_cast<const float4*>(h_last + (size_t)v * D);
    const float4* hz = reinterpret_cast<const float4*>(h0 + (size_t)v * D);
    const float4* wa = reinterpret_cast<const float4*>(w.w_gate);
    const float4* wb = reinterpret_cast<const float4*>(w.w_gate + D);
    const float4* wt = reinterpret_cast<const float4*>(w.w_trans);
    float g = 0.f, t = 0.f;
    for (int q = lane; q < (D >> 2); q += 32) {
        const float4 a = hT[q], z = hz[q], ga = wa[q], gb = wb[q], tt = wt[q];
        g += a.x * ga.x + a.y * ga.y + a.z * ga.z + a.w * ga.w + z.x * gb.x + z.y * gb.y + z.z * gb.z + z.w * gb.w;
        t += a.x * tt.x + a.y * tt.y + a.z * tt.z + a.w * tt.w;
    }
    g = warp_sum(g) + w.b_gate[0];
    t = warp_sum(t) + w.b_trans[0];
    float r = sigmoidf_acc(g) * t;
    if (mask) r *= mask[v];
    if (lane == 0) val[v] = r;
}
// stage 2, graphs grouped: graph g owns nodes [graph_start[g], graph_start[g+1]); summed in node order (deterministic, the order of
// TF's CPU unsorted_segment_sum)
__global__ void __launch_bounds__(128) readout_sum_grouped_kernel(const float* __restrict__ val, const int* __restrict__ graph_start,
                                                                  float* __restrict__ out, int G) {
    const int g = blockIdx.x * 128 + threadIdx.x;
    if (g >= G) return;
    float acc = 0.f;
    for (int v = graph_start[g]; v < graph_start[g + 1]; ++v) acc += val[v];
    out[g] = acc;
}
// stage 2, arbitrary graph_of[v]: out must be zeroed by the caller
__global__ void __launch_bounds__(256) readout_sum_atomic_kernel(const float* __restrict__ val, const int* __restrict__ graph_of,
                                                                 float* __restrict__ out, int V) {
    const int v = blockIdx.x * 256 + threadIdx.x;
    if (v < V) atomicAdd(out + graph_of[v], val[v]);
}

// stage 2 of an ungrouped graph_of[v] in deterministic mode: graph g owns positions [graph_start[g], graph_start[g+1]) of the stable by-graph
// permutation `perm` (node index order inside a graph), summed in that order -- the grouped kernel's order, through one indirection
__global__ void __launch_bounds__(128) readout_sum_permuted_kernel(const float* __restrict__ val, const int* __restrict__ graph_start,
                                                                   const int* __restrict__ perm, float* __restrict__ out, int G) {
    const int g = blockIdx.x * 128 + threadIdx.x;
    if (g >= G) return;
    float acc = 0.f;
    for (int i = graph_start[g]; i < graph_start[g + 1]; ++i) acc += val[perm[i]];
    out[g] = acc;
}

// d_out[G] -> d_h_last[V,D] (written), d_w_gate[2D] / d_b_gate[1] / d_w_trans[D] / d_b_trans[1].
// ORDERED = false accumulates them with shared, then global atomics per block.  ORDERED = true (ggnn_set_deterministic): each warp stores its
// sums to its own shared row, the block adds the rows in warp order and stores its partial [d_w_gate | d_w_trans | d_b_gate | d_b_trans]
// ([3D+2]) to part[blockIdx.x]; readout_bwd_reduce_kernel adds the blocks.  The grid must then not depend on the GPU (the grid-stride loop
// gives every warp its nodes by gridDim).
// A warp's row of sums: [d_w_gate(h_T part) | d_w_gate(h_0 part) | d_w_trans] for d < 32*DPL, then the two biases
template <int DPL>
__host__ __device__ constexpr int ro_row() { return 3 * 32 * DPL + 2; }
// Shared memory of the ordered instance: 8 warp rows, over the 48 KiB of static shared memory at DPL = 16 (dynamic there)
template <int DPL>
__host__ __device__ constexpr size_t ro_ordered_smem() { return 8 * ro_row<DPL>() * sizeof(float); }
constexpr int RO_ORDERED_BLOCKS = 512;
template <int DPL, bool ORDERED>
__device__ __forceinline__ void readout_bwd(const float* __restrict__ h_last, const float* __restrict__ h0, const Weights& w,
                                            const int* __restrict__ graph_of, const float* __restrict__ mask, const float* __restrict__ d_out,
                                            float* __restrict__ d_h_last, float* __restrict__ d_w_gate, float* __restrict__ d_b_gate,
                                            float* __restrict__ d_w_trans, float* __restrict__ d_b_trans, float* __restrict__ part, int V, int D) {
    constexpr int RO_ROW = ro_row<DPL>(), W = 32 * DPL;
    constexpr bool DYN = ORDERED && ro_ordered_smem<DPL>() > 48 * 1024;
    __shared__ float red_static[DYN ? 1 : (ORDERED ? 8 * RO_ROW : RO_ROW)];
    extern __shared__ float red_dynamic[];
    float* red = DYN ? red_dynamic : red_static;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (!ORDERED) {
        for (int i = threadIdx.x; i < RO_ROW; i += 256) red[i] = 0.f;
        __syncthreads();
    }
    float gw_a[DPL], gw_b[DPL], tw[DPL];
#pragma unroll
    for (int j = 0; j < DPL; ++j) gw_a[j] = gw_b[j] = tw[j] = 0.f;
    float gb = 0.f, tb = 0.f;
    for (int v = blockIdx.x * 8 + warp; v < V; v += gridDim.x * 8) {
        const float* hT = h_last + (size_t)v * D;
        const float* hz = h0 + (size_t)v * D;
        float gp, tp;
        node_dots(hT, hz, w, D, lane, gp, tp);
        const float go = d_out[graph_of[v]] * (mask ? mask[v] : 1.0f);
        const float g = sigmoidf_acc(gp);
        const float dgp = go * tp * g * (1.0f - g);   // d gate pre-activation
        const float dt = go * g;                      // d transform output
#pragma unroll
        for (int j = 0; j < DPL; ++j) {
            const int d = lane + 32 * j;
            if (d < D) {
                const float a = hT[d];
                d_h_last[(size_t)v * D + d] = fmaf(dgp, w.w_gate[d], dt * w.w_trans[d]);
                gw_a[j] = fmaf(dgp, a, gw_a[j]);
                gw_b[j] = fmaf(dgp, hz[d], gw_b[j]);
                tw[j] = fmaf(dt, a, tw[j]);
            }
        }
        gb += dgp; tb += dt;
    }
    if (ORDERED) {
        float* row = red + warp * RO_ROW;
#pragma unroll
        for (int j = 0; j < DPL; ++j) {
            const int d = lane + 32 * j;
            if (d < D) { row[d] = gw_a[j]; row[W + d] = gw_b[j]; row[2 * W + d] = tw[j]; }
        }
        if (lane == 0) { row[3 * W] = gb; row[3 * W + 1] = tb; }
        __syncthreads();
        float* out = part + (size_t)blockIdx.x * (3 * D + 2);
        for (int c = threadIdx.x; c < 3 * D + 2; c += 256) {
            // column c of the partial: [0, 2D) d_w_gate, [2D, 3D) d_w_trans, 3D d_b_gate, 3D+1 d_b_trans
            const int src = c < D ? c : c < 2 * D ? W + c - D : c < 3 * D ? 2 * W + c - 2 * D : 3 * W + c - 3 * D;
            float a = red[src];
            for (int q = 1; q < 8; ++q) a += red[q * RO_ROW + src];
            out[c] = a;
        }
        return;
    }
#pragma unroll
    for (int j = 0; j < DPL; ++j) {
        const int d = lane + 32 * j;
        if (d < D) { atomicAdd(&red[d], gw_a[j]); atomicAdd(&red[W + d], gw_b[j]); atomicAdd(&red[2 * W + d], tw[j]); }
    }
    if (lane == 0) { atomicAdd(&red[3 * W], gb); atomicAdd(&red[3 * W + 1], tb); }
    __syncthreads();
    for (int d = threadIdx.x; d < D; d += 256) {
        if (d_w_gate) { atomicAdd(d_w_gate + d, red[d]); atomicAdd(d_w_gate + D + d, red[W + d]); }
        if (d_w_trans) atomicAdd(d_w_trans + d, red[2 * W + d]);
    }
    if (threadIdx.x == 0) {
        if (d_b_gate) atomicAdd(d_b_gate, red[3 * W]);
        if (d_b_trans) atomicAdd(d_b_trans, red[3 * W + 1]);
    }
}
template <int DPL>
__global__ void __launch_bounds__(256) readout_bwd_kernel(const float* __restrict__ h_last, const float* __restrict__ h0, Weights w,
                                                          const int* __restrict__ graph_of, const float* __restrict__ mask,
                                                          const float* __restrict__ d_out, float* __restrict__ d_h_last,
                                                          float* __restrict__ d_w_gate, float* __restrict__ d_b_gate,
                                                          float* __restrict__ d_w_trans, float* __restrict__ d_b_trans, int V, int D) {
    readout_bwd<DPL, false>(h_last, h0, w, graph_of, mask, d_out, d_h_last, d_w_gate, d_b_gate, d_w_trans, d_b_trans, nullptr, V, D);
}
// part: [gridDim.x][3D+2] block partials, reduced by readout_bwd_reduce_kernel; launched with ro_ordered_smem<16>() bytes of dynamic shared
// memory at DPL = 16
template <int DPL>
__global__ void __launch_bounds__(256) readout_bwd_ordered_kernel(const float* __restrict__ h_last, const float* __restrict__ h0, Weights w,
                                                                  const int* __restrict__ graph_of, const float* __restrict__ mask,
                                                                  const float* __restrict__ d_out, float* __restrict__ d_h_last,
                                                                  float* __restrict__ part, int V, int D) {
    readout_bwd<DPL, true>(h_last, h0, w, graph_of, mask, d_out, d_h_last, nullptr, nullptr, nullptr, nullptr, part, V, D);
}
// one block per column of the [blocks][3D+2] partials: the blocks added in a fixed order (ggnn::bwd::ordered_column_sum), then once into the
// caller's gradient (any of the four may be NULL)
__global__ void __launch_bounds__(256) readout_bwd_reduce_kernel(const float* __restrict__ part, int blocks, int D, float* __restrict__ d_w_gate,
                                                                 float* __restrict__ d_b_gate, float* __restrict__ d_w_trans,
                                                                 float* __restrict__ d_b_trans) {
    __shared__ float s_red[256];
    const int c = blockIdx.x;
    float* dst = c < 2 * D ? (d_w_gate ? d_w_gate + c : nullptr) : c < 3 * D ? (d_w_trans ? d_w_trans + c - 2 * D : nullptr)
                                                                              : c == 3 * D ? d_b_gate : d_b_trans;
    if (!dst) return;
    const float a = bwd::ordered_column_sum(part, blocks, 3 * D + 2, c, s_red);
    if (threadIdx.x == 0) *dst += a;
}

// Masked regression loss of one task (chem_tensorflow.py:161-166): diff = (computed - target) * mask,
//   loss = sum 0.5*diff^2 / (sum mask + 1e-7),  accuracy (= MAE) = sum |diff| / (sum mask + 1e-7).
// One block per task; every thread adds a strided slice in index order and the block reduces in a fixed tree: run-to-run identical.
// out[task] = loss, out[num_tasks + task] = accuracy.
__global__ void __launch_bounds__(256) masked_loss_kernel(const float* __restrict__ computed, const float* __restrict__ target_values,
                                                          const float* __restrict__ target_mask, float* __restrict__ out, int G, int num_tasks) {
    __shared__ float s_sq[256], s_abs[256], s_cnt[256];
    const int task = blockIdx.x, tid = threadIdx.x;
    const float* c = computed + (size_t)task * G;
    const float* tv = target_values + (size_t)task * G;
    const float* tm = target_mask + (size_t)task * G;
    float sq = 0.f, ab = 0.f, cnt = 0.f;
    for (int g = tid; g < G; g += 256) {
        const float m = tm[g], d = (c[g] - tv[g]) * m;
        sq += 0.5f * d * d; ab += fabsf(d); cnt += m;
    }
    s_sq[tid] = sq; s_abs[tid] = ab; s_cnt[tid] = cnt;
    __syncthreads();
    for (int o = 128; o > 0; o >>= 1) {
        if (tid < o) { s_sq[tid] += s_sq[tid + o]; s_abs[tid] += s_abs[tid + o]; s_cnt[tid] += s_cnt[tid + o]; }
        __syncthreads();
    }
    if (tid == 0) {
        const float num = s_cnt[0] + 1e-7f;   // SMALL_NUMBER, utils.py:8
        out[task] = s_sq[0] / num;
        out[num_tasks + task] = s_abs[0] / num;
    }
}

}  // namespace readout
}  // namespace ggnn
