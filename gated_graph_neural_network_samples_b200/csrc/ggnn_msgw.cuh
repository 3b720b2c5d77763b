// Message weights of the sparse GGNN model (ggnn_prepare_graph_sparse_weighted, ggnn_set_message_weights, ggnn_backward_weighted):
//   incoming[v] = ( sum_t (sum_{m into v, type t} w_m h[s_m]) W_t  +  sum_t indeg[v,t] b_t ) / denom[v]
// The forward kernels read the weights as slot weights (ImageView::slotw / tslotw); these kernels put them there and form their gradient.
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>

namespace ggnn {
namespace msgw {

// slotw[k] = w[msg[k]] for every target-CSR slot k and, with the source-keyed CSR, tslotw[j] = w[msg[tslot[j]]] (the weight of the target
// slot that source entry j is): the caller's [M] weights in type-major message order, scattered into the image's two weight sections.
__global__ void __launch_bounds__(256) scatter_message_weights_kernel(const float* __restrict__ w, const int* __restrict__ msg,
                                                                      const int* __restrict__ tslot, float* __restrict__ slotw,
                                                                      float* __restrict__ tslotw, int64_t M) {
    for (int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; k < M; k += (int64_t)gridDim.x * blockDim.x) {
        slotw[k] = w[msg[k]];
        if (tslotw) tslotw[k] = w[msg[tslot[k]]];
    }
}

// One timestep's weight gradient:  dw_slot[k] += <P[v, t*D ..], h[src[k]]>  for every target-CSR slot k of target v and type t, where
// P = dx' . W_t^T ([V, T*D]) and h is the step's input state.  One warp per target; each slot has one owner and the lanes' partial dot
// products are added by a fixed butterfly, so the sums do not depend on scheduling (no atomics).  D is a multiple of 4; P and h rows are
// 16-byte aligned.
__global__ void __launch_bounds__(256) message_weight_grad_kernel(const int* __restrict__ row_ptr, const int* __restrict__ csr_src,
                                                                  const float* __restrict__ P, const float* __restrict__ h,
                                                                  float* __restrict__ dw_slot, int V, int D, int T) {
    const int v = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (v >= V) return;
    const int D4 = D >> 2;
    for (int t = 0; t < T; ++t) {
        const int beg = row_ptr[(size_t)v * T + t], end = row_ptr[(size_t)v * T + t + 1];
        if (beg == end) continue;
        const float4* Pv = reinterpret_cast<const float4*>(P + ((size_t)v * T + t) * D);
        for (int m = beg; m < end; ++m) {
            const float4* hs = reinterpret_cast<const float4*>(h + (size_t)csr_src[m] * D);
            float s = 0.f;
            for (int c = lane; c < D4; c += 32) {
                const float4 p = Pv[c], x = hs[c];
                s = fmaf(p.x, x.x, s); s = fmaf(p.y, x.y, s); s = fmaf(p.z, x.z, s); s = fmaf(p.w, x.w, s);
            }
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
            if (lane == 0) dw_slot[m] += s;
        }
    }
}

// The end of a backward call: d_w[msg[k]] += dw_slot[k].  msg is a permutation of the messages, so every entry has one writer.
__global__ void __launch_bounds__(256) add_slot_grads_kernel(const int* __restrict__ msg, const float* __restrict__ dw_slot, float* __restrict__ d_w,
                                                             int64_t M) {
    for (int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; k < M; k += (int64_t)gridDim.x * blockDim.x) d_w[msg[k]] += dw_slot[k];
}

}  // namespace msgw
}  // namespace ggnn
