// Shared device-side definitions of the GGNN propagation engine (sm_90a).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace ggnn {

constexpr int MAX_LAYERS = 16;
constexpr int MAX_RES = 4;     // residual inputs per layer
constexpr int KC = 16;         // K rows of a weight operand per shared-memory stage (FFMA path)

enum { CELL_GRU = 0, CELL_RNN = 1, CELL_CUDNN_GRU = 2 };
enum { ACT_TANH = 0, ACT_RELU = 1 };

struct LayerDev {
    const float* edge_w;   // [T][D][D]
    const float* edge_b;   // [T][D] or nullptr
    const float* gate_k;   // [(Din+D)][2D]
    const float* gate_b;   // [2D]
    const float* cand_k;   // [(Din+D)][D]   (RNN: the only kernel)
    const float* cand_b;   // [D]
    const float* att_w;    // [T] edge_type_attention_weights or nullptr (sparse:94-96)
    const float* cand_hb;  // [D] hidden-projection bias of CudnnCompatibleGRUCell (sparse:105-108) or nullptr
    int steps;
    int nres;
    int res[MAX_RES];      // indices into node_states_per_layer
};

// The sections of a batch's graph image as typed pointers into one copy of it: the host image the builder fills, the device image the
// engine reads, or the device image the dataset kernels write.  The engine's image_view() makes it from the plan's layout; a section the
// plan does not carry is null.
struct ImageView {
    int *row_ptr, *src, *msg;                  // target CSR: rows target*T+type, the source and message id of every slot
    float *indeg, *denom;
    int* tile_start;
    unsigned* tile_mask;
    int *trow, *ttgt, *tslot;                  // source-keyed CSR (save_for_backward); tslot: attention only
    int *pair, *vptr, *vsrc, *tvp, *vinfo;     // streaming plan
    int* vslot;                                // weighted streaming plan: first target-CSR slot of every virtual row
    float *slotw, *tslotw;                     // weighted batches: per-slot weights in target-CSR / source-CSR order
};

// Per-(layer,step) activations kept for the backward pass; each [V][D] (device), index = global step.
struct SaveDev {
    float* h_in;   // state entering the step
    float* agg;    // aggregated incoming messages after bias/mean (the cell's message input)
    float* r;      // reset gate   (GRU)
    float* u;      // update gate  (GRU)
    float* c;      // candidate    (GRU) -- for RNN the new state itself is enough
    float* q;      // CudnnCompatibleGRUCell only: h . K_hid + b_hid, the recurrent projection BEFORE the reset gate
};

struct FwdParams {
    int V, D, T, L;
    int use_bias, use_avg, cell, act;
    int save;                 // keep activations for backward
    const int* tile_start;    // [ntiles+1] first node of each tile
    const unsigned* tile_mask;// [ntiles] bit t set iff some node of the tile has an incoming type-t message
    const int* row_ptr;       // [V*T+1] CSR rows keyed target*T+type (stable in message order)
    const int* csr_src;       // [M] source node of each CSR slot
    const float* slot_w;      // [M] weight of each CSR slot (weighted dense adjacency), or nullptr
    const float* indeg;       // [V][T] num_incoming_edges_per_type
    const float* denom;       // [V] fp32(sum_t indeg) + 1e-7f
    const float* state[MAX_LAYERS + 1];   // node_states_per_layer: [0]=h0 ... [L]=result (read side)
    float* state_w[MAX_LAYERS + 1];       // write side ([0] unused)
    LayerDev layer[MAX_LAYERS];
    SaveDev save_buf;         // base pointers; step s lives at +s*V*D
    int step_base[MAX_LAYERS];// global step index of (layer,0)
    // global (one step per launch) mode
    int g_layer, g_step;
    const float* g_in;
    float* g_out;
    // propagation attention (sparse:170-196): per-message softmax weight, indexed by target-CSR slot; step gs lives at att + gs*att_stride
    int use_att;
    float* att;
    size_t att_stride;
    // DropoutWrapper(state_keep_prob) (sparse:113-114,216 / dense:89): off when drop_keep >= 1
    float drop_keep;
    unsigned long long drop_seed;
};

// State-dropout mask: a counter-based hash (splitmix64 finaliser) of (seed, global step, node, column), so the forward
// kernels, the backward pass and the test oracle regenerate the same mask without storing it.  TF's own generator cannot
// be reproduced; what is kept is DropoutWrapper's arithmetic: kept values are DIVIDED by keep_prob, dropped ones are 0.
__host__ __device__ __forceinline__ bool dropout_keeps(unsigned long long seed, int gstep, int V, int D, int row, int col, float keep) {
    unsigned long long x = ((unsigned long long)gstep * (unsigned long long)V + (unsigned long long)row) * (unsigned long long)D + (unsigned long long)col;
    x += (seed + 1ull) * 0x9E3779B97F4A7C15ull;
    x ^= x >> 30; x *= 0xBF58476D1CE4E5B9ull;
    x ^= x >> 27; x *= 0x94D049BB133111EBull;
    x ^= x >> 31;
    return (float)(x >> 40) * (1.0f / 16777216.0f) < keep;
}
__host__ __device__ __forceinline__ float dropout_apply(float v, unsigned long long seed, int gstep, int V, int D, int row, int col, float keep) {
    return dropout_keeps(seed, gstep, V, D, row, col, keep) ? v / keep : 0.0f;
}

__device__ __forceinline__ void cp_async16(void* smem_dst, const void* gmem_src) {
    unsigned s = (unsigned)__cvta_generic_to_shared(smem_dst);
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;\n" ::"r"(s), "l"(gmem_src));
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;\n" ::); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;\n" ::"n"(N)); }

__device__ __forceinline__ float sigmoidf_acc(float v) { return 1.0f / (1.0f + expf(-v)); }
__device__ __forceinline__ float activate(float v, int act) { return act == ACT_TANH ? tanhf(v) : fmaxf(v, 0.0f); }

}  // namespace ggnn
