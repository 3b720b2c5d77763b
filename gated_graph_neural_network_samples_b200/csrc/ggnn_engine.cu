// Host side of the GGNN propagation engine + the C ABI declared in include/ggnn_b200.h.
//
// Mirrors the two ChemModel hooks of the reference for this path:
//   ggnn_create / ggnn_set_weights            <- prepare_specific_graph_model        (sparse:63-115, dense:68-91)
//   ggnn_set_graph_* + ggnn_forward           <- compute_final_node_representations  (sparse:117-218, dense:93-117)
// Host work per batch: validate indices, stable counting sort of the type-major message list by
// (target, type) -> CSR, find where the batch can be cut between connected components, pack tiles.
#include <cuda_runtime.h>

#include <algorithm>
#include <array>
#include <chrono>
#ifdef _OPENMP
#include <omp.h>
#include <sched.h>
#endif
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <type_traits>
#include <vector>

#include "../../include/ggnn_b200.h"
#include "ggnn_common.cuh"
#include "ggnn_bwd.cuh"
#include "ggnn_bwd_tc.cuh"
#include "ggnn_readout.cuh"
#include "ggnn_fwd_ffma.cuh"
#include "ggnn_fwd_tc.cuh"
#include "ggnn_fwd_stream.cuh"
#include "ggnn_fwd_step.cuh"
#include "ggnn_gcn.cuh"
#include "ggnn_dataset.cuh"
#include "ggnn_msgw.cuh"
#include "ggnn_dense_adj.cuh"
#include "ggnn_tc_smem.h"

using namespace ggnn;

namespace {

std::string g_create_error;

struct DevBuf {
    void* ptr = nullptr;
    size_t cap = 0;
    cudaError_t reserve(size_t bytes) {
        if (bytes <= cap) return cudaSuccess;
        if (ptr) cudaFree(ptr);
        ptr = nullptr; cap = 0;
        size_t want = bytes + bytes / 4 + 256;
        cudaError_t e = cudaMalloc(&ptr, want);
        if (e == cudaSuccess) cap = want;
        return e;
    }
    void release() { if (ptr) cudaFree(ptr); ptr = nullptr; cap = 0; }
};

struct HostPinned {
    void* ptr = nullptr;
    size_t cap = 0;
    cudaError_t reserve(size_t bytes) {
        if (bytes <= cap) return cudaSuccess;
        if (ptr) cudaFreeHost(ptr);
        ptr = nullptr; cap = 0;
        size_t want = bytes + bytes / 4 + 256;
        cudaError_t e = cudaMallocHost(&ptr, want);
        if (e == cudaSuccess) cap = want;
        return e;
    }
    void release() { if (ptr) cudaFreeHost(ptr); ptr = nullptr; cap = 0; }
};

// A host image that one cudaMemcpyAsync uploads: pinned memory, or plain memory for host-only builds, which make no CUDA call.
struct StagedImage {
    bool use_cuda = true;
    char* ptr = nullptr;
    HostPinned pinned;
    std::vector<char> plain;
    cudaEvent_t uploaded = nullptr;   // recorded after the last upload: begin() waits for it before the image is overwritten

    cudaError_t begin(size_t bytes) {
        if (!use_cuda) {
            if (plain.size() < bytes) plain.resize(bytes + bytes / 4 + 256);
            ptr = plain.data();
            return cudaSuccess;
        }
        if (uploaded) {
            cudaError_t st = cudaEventSynchronize(uploaded);
            if (st != cudaSuccess) return st;
        }
        cudaError_t st = pinned.reserve(bytes);
        ptr = (char*)pinned.ptr;
        return st;
    }
    cudaError_t upload(void* dev, size_t bytes, cudaStream_t stream) {
        cudaError_t st = cudaMemcpyAsync(dev, ptr, bytes, cudaMemcpyHostToDevice, stream);
        if (st != cudaSuccess) return st;
        if (!use_cuda) return cudaStreamSynchronize(stream);   // a pageable image must be consumed before the caller may reuse it
        if (!uploaded && (st = cudaEventCreateWithFlags(&uploaded, cudaEventDisableTiming)) != cudaSuccess) return st;
        return cudaEventRecord(uploaded, stream);
    }
    void release() {
        if (uploaded) { cudaEventSynchronize(uploaded); cudaEventDestroy(uploaded); uploaded = nullptr; }
        pinned.release();
    }
};

inline size_t align_up(size_t x, size_t a) { return (x + a - 1) / a * a; }

// which model an engine or a prepared graph was created for: ggnn_create / ggnn_gcn_create
enum { MODEL_GGNN = 0, MODEL_GCN = 1 };

// The text of the last error of an engine or a prepared graph (ggnn_last_error / ggnn_prepared_graph_error).
struct ErrorText {
    std::string err;

    int fail(int code, const char* fmt, ...) {
        char buf[512];
        va_list ap;
        va_start(ap, fmt);
        vsnprintf(buf, sizeof buf, fmt, ap);
        va_end(ap);
        err = buf;
        return code;
    }
};

// What ggnn_create / ggnn_gcn_create fix for the engine's lifetime (a host-only prepare call takes it from a config).
struct ModelShape {
    int model = MODEL_GGNN;
    int D = 0, T = 0, L = 0;
    int DP = 0;         // hidden size padded to a multiple of 16 (tensor-core path)
    int steps[MAX_LAYERS] = {0};
    int nres[MAX_LAYERS] = {0};
    int res[MAX_LAYERS][MAX_RES] = {{0}};
    int step_base[MAX_LAYERS] = {0};
    int total_steps = 0;
    int use_bias = 0, use_avg = 0, cell = 0, act = 0, precision = 0, device = 0;
    int use_att = 0;    // use_propagation_attention (sparse:170-196): on the fp32 kernels, or on the streaming wgmma kernels when the
                        // precision is not fp32 (GGNN_ATT_TENSOR_CORES)
    int cudnn_tc = 0;   // GGNN_CELL_CUDNN_GRU_TENSOR_CORES: cell is CELL_CUDNN_GRU and keeps the configured precision (the streaming plan)
    int wide_hidden = 0;   // GCN, ggnn_gcn_config.wide_hidden: hidden sizes up to 512, on the streaming plan above 128 on bf16x3 / bf16
    int num_sms = 132;
    size_t max_smem = 0;
};

// The shared memory per block of a model shape made without a device (host-only prepare calls, datasets and tile plans): an H100's
// opt-in maximum.
constexpr size_t HOST_MAX_SMEM = 227 * 1024;

// What build_plan and the image builders derive from one batch: the tile plan and the layout of the graph image.
struct BatchPlan {
    bool weighted = false;   // every message has a weight (GCN, weighted dense adjacency): the image carries the slot weights
    int V = 0;
    int64_t M = 0;
    int variant = 0;  // 0: RG=8,CS=1 (64-row tiles)   1: RG=4,CS=2 (32-row tiles)
    int nb1 = 0;
    bool local = false;
    int ntiles = 0;
    int max_span = 0;
    int max_tile_msgs = 0;   // largest number of messages whose target lies in one tile
    int max_tile_types = 0;  // largest number of edge types present in one tile
    std::string plan_text;
    // streaming tensor-core plan (ggnn_fwd_stream.cuh): D > 128, or forced with GGNN_TC_STREAM=1
    bool stream = false;
    int ts_nc[2] = {0, 0}, ts_nblk[2] = {0, 0};      // [0]: DP-wide outputs (agg, candidate)  [1]: the 2*DP-wide gate output
    int ts_nv = 0;                                   // number of virtual rows of the current batch
    bool stepwise = false;   // fp32 above hidden 256 (ggnn_fwd_step.cuh): a few launches over the whole batch per timestep
    int tc_row_budget = 128, tc_kgs = 2048;   // tensor-core plan: no tile has more rows than the budget; <= 64 selects compact operand tiles
    // the graph image: row_ptr | csr_src | csr_msg | indeg | denom | tile_start | tile_mask | ...
    size_t off_row_ptr = 0, off_src = 0, off_msg = 0, off_indeg = 0, off_denom = 0, off_tiles = 0, off_mask = 0;
    size_t off_trow = 0, off_ttgt = 0;   // source-keyed CSR (rows source*T+type -> targets), built when save_for_backward is on
    bool has_transpose = false;
    size_t off_tslot = 0;            // source-keyed CSR entry -> target-CSR slot (attention backward)
    size_t off_pair = 0, off_vptr = 0, off_vsrc = 0, off_tvp = 0, off_vinfo = 0;   // streaming plan: (target,type) -> source table, virtual rows (pairs with several messages)
    size_t off_vslot = 0;   // weighted streaming plan: the first target-CSR slot of every virtual row (its weights are slot_w[vslot[vid] + m])
    bool all_virtual = false;   // attention on the streaming plan: every (target, type) pair with messages is a virtual row, weighted by the
                                // step's attention probabilities through vslot (the image has vslot and no slot weights); a message-weighted
                                // batch likewise, weighted by its slot weights, so that the plan does not depend on their values
    bool msg_weighted = false;  // ggnn_prepare_graph_sparse_weighted / ggnn_prepare_graph_gcn_message_weighted: weighted, its slot weights
                                // zero in the image until ggnn_set_message_weights writes them on the device; the image carries the
                                // source-keyed CSR's slot map (tslot) with save_for_backward
    size_t off_slotw = 0, off_tslotw = 0;   // weighted: per-slot adjacency weights in target-CSR order / source-CSR order (with the transpose)
    // ggnn_prepare_graph_dense_device (also msg_weighted): the [b, T, v, v] adjacency is set on the device (ggnn_set_message_weights), its row
    // sums become the in-degree section.  The image lists no messages (its CSR sections are empty) and M counts the matrix's b*T*v*v
    // entries; on the streaming plan every (row, type) pair is virtual row row*T + type, written by the dense aggregation kernel
    // (ggnn_dense_adj.cuh) before every gather launch
    bool dense_device = false;
    int dense_b = 0, dense_v = 0;
    // (offset, bytes) of the image's bytes no section builder writes: alignment gaps and the one-element room of empty sections.  The host
    // builder zeroes them (the device dataset zeroes its whole image), so that an image is one function of its batch, whatever the
    // staging memory held before
    std::vector<std::pair<size_t, size_t>> pads;
};

// The weights in the pre-split, pre-tiled bf16 layout of one tensor-core kernel family, with each layer's offsets.  The tiles are rebuilt
// when the weights changed since they were made (ggnn_set_weights / ggnn_gcn_set_weights bump the engine's weights generation) or when
// the layout changed, and at no other time.
struct WeightTiles {
    DevBuf buf;
    size_t off_edge[MAX_LAYERS] = {0}, off_gate[MAX_LAYERS] = {0}, off_cand[MAX_LAYERS] = {0};
    size_t off_hproj[MAX_LAYERS] = {0};   // streaming layout, CudnnCompatibleGRUCell: the hidden projection K_hid (the last D rows of cand_kernel)
    uint64_t gen = 0;     // the weights generation the tiles were made from (0: none)
    size_t bytes = 0;     // the layout they were made for: its size and, for the streaming layout, its N-block widths
    int nc[2] = {0, 0};

    // Makes room for a layout of `size` bytes and N-block widths n0 / n1.  `retile` says whether the tiles are not those of weights
    // generation `want` in that layout; the caller then makes them and sets `gen`.
    cudaError_t reserve(size_t size, int n0, int n1, uint64_t want, bool& retile) {
        retile = gen != want || bytes != size || nc[0] != n0 || nc[1] != n1;
        if (retile) { gen = 0; bytes = size; nc[0] = n0; nc[1] = n1; }
        return buf.reserve(size);
    }
};

}  // namespace

struct ggnn_engine : ModelShape, BatchPlan, ErrorText {
    bool weights_set = false;
    uint64_t weights_gen = 0;   // bumped by every successful ggnn_set_weights / ggnn_gcn_set_weights
    ggnn_layer_weights w[MAX_LAYERS];
    ggnn_gcn_layer_weights gcn_w[MAX_LAYERS] = {};
    bool graph_set = false;
    bool msg_weights_set = false;   // a message-weighted batch: ggnn_set_message_weights ran since its upload
    DevBuf dense_adj;               // a dense-device batch: the engine's copy of its [b, T, v, v] adjacency (ggnn_set_message_weights)

    // device memory
    DevBuf graph_buf;   // the graph image of the current batch
    size_t graph_bytes = 0;
    DevBuf ds_table;    // the batch table of a dataset batch (ggnn_set_graph_dataset): tile starts and per-graph offsets
    ImageView gd;       // the view of graph_buf every driver reads, made by every graph upload (bind_graph)
    // readout (gated_regression): node -> graph map of the current batch
    DevBuf ro_buf; StagedImage ro_stage;
    int ro_V = -1, ro_G = 0; bool ro_grouped = false, ro_has_mask = false;
    size_t ro_off_graph_of = 0, ro_off_start = 0, ro_off_mask = 0, ro_off_val = 0;
    size_t ro_off_perm = 0;   // ungrouped lists: the stable by-graph node permutation (graph g owns perm[start[g] .. start[g+1]))
    DevBuf ro_ws;             // deterministic readout backward: per-block partials of the weight gradients
    DevBuf ro_kval;           // ggnn_readout_predict: the per-node gated values of every task [K][V]
    bool ro_from_dataset = false;          // the map came with a dataset batch, whose graphs' dataset indices are ...
    const int* ro_dataset_slots = nullptr;  // ... this device table [G] (in ds_table)
    DevBuf state_buf;   // intermediate layer states (L-1) + 2 ping-pong step buffers, each [V][D]
    DevBuf save_bufs;   // 5 (CudnnCompatibleGRUCell: 6) x total_steps x [V][D]
    DevBuf io_buf;      // h0 / h_out staging for ggnn_forward_host
    DevBuf bwd_buf;     // backward scratch
    WeightTiles tc_tiles;   // the weights tiled for the tile-local wgmma kernel (GGNN) or the GCN wgmma kernel
    WeightTiles ts_tiles;   // ... and for the streaming kernel
    WeightTiles step_wt;    // ... and the transposed fp32 copies of the per-timestep fp32 path
    DevBuf step_buf;        // the per-timestep fp32 path's scratch: gathered messages, cell input row, gates, candidate
    DevBuf tc_respre;   // residual pre-products [ntiles][128][3*DP]
    DevBuf err_flag;    // device int written by kernels on a barrier timeout
    // the state buffers of the last forward on the current graph; fwd_valid is cleared by every graph upload.  Without save_for_backward
    // the fused GCN kernel keeps the layers between h0 and h_out on chip: layers_written says whether state_buf holds them.
    const float* last_h0 = nullptr;
    float* last_out = nullptr;
    bool fwd_valid = false, layers_written = false;
    bool save = false;
    bool saved_valid = false;   // the saved activations are those of the last forward, with the current weights
    bool det = false;           // ggnn_set_deterministic: fixed-order weight-gradient and readout sums
    int bwd_precision = GGNN_PREC_FP32;   // ggnn_set_backward_precision: the GEMMs of the backward on FFMA or on bf16x3 wgmma
    DevBuf ts_images;                                // the streaming plan's operand images and chunk-major states
    DevBuf ts_virt;                                  // the operand image of the streaming plan's virtual rows
    DevBuf att_buf;                  // attention probabilities per target-CSR slot ([steps][M] when saving for backward, else [M])
    float drop_keep = 1.0f; unsigned long long drop_seed = 0;          // state dropout for the next forward
    float saved_drop_keep = 1.0f; unsigned long long saved_drop_seed = 0; // ... and what the saved forward used
    int last_launches = 0;
    struct ggnn_prepared_graph* own_prep = nullptr;   // the prepared graph ggnn_set_graph_* build and upload from (reused every batch)
};

// The host half of ggnn_set_graph_*: the model shape goes in, the batch plan and the packed image (CSR, in-degrees, tiles, streaming
// tables, the slot weights of a weighted batch) come out; nothing here touches the device but the pinned image.  Built by a producer thread,
// uploaded by the engine's thread (ggnn_set_graph_prepared) -- the ThreadedIterator overlap of the reference's training loop
// (chem_tensorflow.py:225, utils.py:16-36).
struct ggnn_prepared_graph : ErrorText {
    ModelShape shape;
    bool save = false;   // whether the image carries the source-keyed CSR of the backward pass
    BatchPlan plan;
    StagedImage image;
    size_t bytes = 0;
    bool valid = false;
    std::vector<int> h_counts, h_diff, h_cursor;   // host scratch of the sparse-graph builder, kept between batches
};

#define CU_TRY(e, call)                                                                           \
    do {                                                                                          \
        cudaError_t _st = (call);                                                                 \
        if (_st != cudaSuccess) return (e)->fail(GGNN_ECUDA, "%s failed: %s", #call, cudaGetErrorString(_st)); \
    } while (0)

// ------------------------------------------------------------------------------------------ the engine's device buffers of a batch
// Elements of one [V][D] state array (at least one row).
static size_t state_elems(const ggnn_engine* e) { return (size_t)std::max(e->V, 1) * e->D; }

// node_states_per_layer of the forward that read h0 and wrote h_out: [0] is h0 (only ever read), [L] is h_out, the layers between live at
// the front of state_buf.
static float* layer_state(const ggnn_engine* e, int l, const float* h0, float* h_out) {
    if (l == 0) return const_cast<float*>(h0);
    if (l == e->L) return h_out;
    return (float*)e->state_buf.ptr + (size_t)(l - 1) * state_elems(e);
}

// The state pointers of a kernel's parameters (FwdParams, TcParams, GcnParams): read side [0..L], write side [1..L].
template <class Params>
static void set_layer_states(const ggnn_engine* e, Params& p, const float* h0, float* h_out) {
    p.state[0] = h0;
    for (int l = 1; l <= e->L; ++l) p.state[l] = p.state_w[l] = layer_state(e, l, h0, h_out);
}

// The GLOBAL plans' ping-pong temporaries (i = 0, 1) of a layer's inner timesteps: the two [V][D] slots of state_buf behind the layers.
static float* step_temp(const ggnn_engine* e, int i) { return (float*)e->state_buf.ptr + (size_t)(e->L - 1 + i) * state_elems(e); }

// The activations global step `gs` saves for the backward pass, each [V][D]: save_bufs holds 5 (CudnnCompatibleGRUCell: 6) arrays of
// total_steps steps.  All null when save_for_backward is off.
static SaveDev saved_step(const ggnn_engine* e, int gs) {
    SaveDev s;
    memset(&s, 0, sizeof s);
    if (!e->save) return s;
    const size_t per = state_elems(e) * (size_t)std::max(e->total_steps, 1);
    float* b = (float*)e->save_bufs.ptr + (size_t)gs * state_elems(e);
    s.h_in = b; s.agg = b + per; s.r = b + 2 * per; s.u = b + 3 * per; s.c = b + 4 * per;
    s.q = e->cell == CELL_CUDNN_GRU ? b + 5 * per : nullptr;
    return s;
}

// The fields the parameters of the fp32 and the tile-local wgmma kernels share (FwdParams, tc::TcParams); the rest is zero.
template <class Params>
static void fill_common_params(const ggnn_engine* e, Params& p, const float* h0, float* h_out) {
    memset(&p, 0, sizeof p);
    p.V = e->V; p.D = e->D; p.T = e->T; p.L = e->L;
    p.use_bias = e->use_bias; p.use_avg = e->use_avg; p.cell = e->cell; p.act = e->act;
    p.save = e->save ? 1 : 0;
    p.drop_keep = e->drop_keep; p.drop_seed = e->drop_seed;
    const ImageView& gd = e->gd;
    p.tile_start = gd.tile_start; p.tile_mask = gd.tile_mask; p.row_ptr = gd.row_ptr; p.csr_src = gd.src;
    p.slot_w = gd.slotw; p.indeg = gd.indeg; p.denom = gd.denom;
    set_layer_states(e, p, h0, h_out);
    p.save_buf = saved_step(e, 0);   // the kernels index it by global step
    for (int l = 0; l < e->L; ++l) {
        p.layer[l].steps = e->steps[l]; p.layer[l].nres = e->nres[l];
        for (int i = 0; i < MAX_RES; ++i) p.layer[l].res[i] = e->res[l][i];
        p.step_base[l] = e->step_base[l];
    }
}

// Runs a forward kernel of the fp32 or the tile-local wgmma family: `launch(p)` launches it once.  A LOCAL plan runs every layer and
// timestep in one launch.  A GLOBAL plan launches once per timestep: a layer's inner timesteps ping-pong between the two step temporaries
// and its last one writes the layer's state; a layer without timesteps aliases its input (sparse:152).
template <class Params, class Launch>
static int launch_steps(ggnn_engine* e, Params& p, cudaStream_t st, Launch launch) {
    if (e->local) {
        launch(p);
        ++e->last_launches;
        return GGNN_OK;
    }
    const size_t vd_bytes = (size_t)e->V * e->D * sizeof(float);
    for (int l = 0; l < e->L; ++l) {
        const float* in = p.state[l];
        if (e->steps[l] == 0) {
            CU_TRY(e, cudaMemcpyAsync(p.state_w[l + 1], in, vd_bytes, cudaMemcpyDeviceToDevice, st));
            continue;
        }
        for (int s = 0; s < e->steps[l]; ++s) {
            float* out = (s == e->steps[l] - 1) ? p.state_w[l + 1] : step_temp(e, s & 1);
            p.g_layer = l; p.g_step = s; p.g_in = in; p.g_out = out;
            launch(p);
            ++e->last_launches;
            in = out;
        }
    }
    return GGNN_OK;
}

// Everything the engine knows about the previous batch beyond its buffers: the graph, the last forward and its saved activations, and the
// readout's node -> graph map.  Called first by every graph upload, so a failed upload leaves no batch behind either.
static void forget_batch(ggnn_engine* e) {
    e->graph_set = false; e->saved_valid = false; e->msg_weights_set = false;
    e->last_h0 = nullptr; e->last_out = nullptr; e->fwd_valid = false; e->layers_written = false;
    e->ro_V = -1;
}

static int no_graph(ggnn_engine* e) {
    return e->fail(GGNN_ESTATE, "no graph set (%s)", e->model == MODEL_GCN ? "ggnn_set_graph_gcn / ggnn_set_graph_prepared" : "ggnn_set_graph_sparse/dense");
}

// The gradient pointers of a layer; the weight-gradient kernels update them with 16-byte vector atomics.
static std::array<const void*, 8> grad_pointers(const ggnn_layer_grads& g) {
    return {g.edge_weights, g.edge_biases, g.gate_kernel, g.gate_bias, g.cand_kernel, g.cand_bias, g.edge_type_attention_weights, g.cand_hidden_bias};
}
static std::array<const void*, 8> grad_pointers(const ggnn_gcn_layer_grads& g) { return {g.kernel, g.bias}; }

// The checks both backward calls start with.  `fn` names the call, `graph_call` the call that builds the source-keyed CSR.
template <class Grads>
static int begin_backward(ggnn_engine* e, const char* fn, const char* graph_call, const float* d_h_out, const Grads* grads, int num_layers,
                          const float* d_h0) {
    if (!e->graph_set || !e->weights_set) return e->fail(GGNN_ESTATE, "no graph / weights set");
    if (!e->saved_valid) return e->fail(GGNN_ESTATE, "%s needs a preceding ggnn_forward with save_for_backward enabled", fn);
    if (!e->has_transpose) return e->fail(GGNN_ESTATE, "enable save_for_backward BEFORE %s (the source-keyed CSR is built there)", graph_call);
    if (!grads || num_layers != e->L || (!d_h_out && e->V > 0)) return e->fail(GGNN_EINVAL, "bad backward arguments");
    for (int l = 0; l < e->L; ++l)
        for (const void* q : grad_pointers(grads[l]))
            if ((uintptr_t)q & 15) return e->fail(GGNN_EINVAL, "layer %d: gradient pointers must be 16-byte aligned", l);
    if (((uintptr_t)d_h_out & 15) || ((uintptr_t)d_h0 & 15)) return e->fail(GGNN_EINVAL, "d_h_out / d_h0 must be 16-byte aligned");
    CU_TRY(e, cudaSetDevice(e->device));
    e->last_launches = 0;
    return GGNN_OK;
}

// The device side of the host-buffer calls: h0 and h_out in two 256-byte-aligned slots at the front of io_buf, `scratch_bytes` more
// behind them.  Enqueues the upload of the `bytes` of h0.
struct IoSlots {
    float* in;
    float* out;
    char* scratch;
};
static int stage_io(ggnn_engine* e, const float* h0_host, size_t bytes, size_t scratch_bytes, cudaStream_t st, IoSlots& io) {
    CU_TRY(e, cudaSetDevice(e->device));
    const size_t slot = align_up(std::max<size_t>(bytes, 16), 256);
    CU_TRY(e, e->io_buf.reserve(2 * slot + scratch_bytes));
    char* b = (char*)e->io_buf.ptr;
    io = IoSlots{(float*)b, (float*)(b + slot), b + 2 * slot};
    if (bytes) CU_TRY(e, cudaMemcpyAsync(io.in, h0_host, bytes, cudaMemcpyHostToDevice, st));
    return GGNN_OK;
}

// The calls of the other model refuse a GGNN / GCN engine.
static int wrong_model(ErrorText* t, const char* fn, int have, int want) {
    return t->fail(GGNN_ESTATE, "%s is a %s call; this engine was created with %s", fn, want == MODEL_GCN ? "GCN" : "GGNN",
                   have == MODEL_GCN ? "ggnn_gcn_create" : "ggnn_create");
}
#define GGNN_REQUIRE_MODEL(e, m)                                                  \
    do {                                                                          \
        if ((e)->model != (m)) return wrong_model((e), __func__, (e)->model, (m)); \
    } while (0)

// ------------------------------------------------------------------------------------------ kernel table
namespace {

typedef void (*FwdKernel)(const FwdParams);

template <int RG, int CS, int NB1, bool LOCAL>
FwdKernel fwd_kernel_ptr() {
    constexpr int NB2 = (2 * NB1 > 8) ? 8 : 2 * NB1;
    constexpr int MINB = (CS == 2 && NB1 <= 2) ? 2 : 1;
    return ggnn_fwd_ffma_kernel<RG, CS, NB1, NB2, LOCAL, MINB>;
}

FwdKernel pick_fwd_kernel(int variant, int nb1, bool local) {
    if (variant == 0) {
        if (nb1 == 1) return local ? fwd_kernel_ptr<8, 1, 1, true>() : fwd_kernel_ptr<8, 1, 1, false>();
        if (nb1 == 2) return local ? fwd_kernel_ptr<8, 1, 2, true>() : fwd_kernel_ptr<8, 1, 2, false>();
        if (nb1 == 4) return local ? fwd_kernel_ptr<8, 1, 4, true>() : fwd_kernel_ptr<8, 1, 4, false>();
    } else {
        if (nb1 == 1) return local ? fwd_kernel_ptr<4, 2, 1, true>() : fwd_kernel_ptr<4, 2, 1, false>();
        if (nb1 == 2) return local ? fwd_kernel_ptr<4, 2, 2, true>() : fwd_kernel_ptr<4, 2, 2, false>();
        if (nb1 == 4) return local ? fwd_kernel_ptr<4, 2, 4, true>() : fwd_kernel_ptr<4, 2, 4, false>();
    }
    return nullptr;
}

int variant_mt(int variant) { return variant == 0 ? 64 : 32; }
int variant_cs(int variant) { return variant == 0 ? 1 : 2; }

int pick_nb1(int variant, int D) {
    const int per = 32 * variant_cs(variant);
    int nb = (D + per - 1) / per;
    if (nb <= 1) return 1;
    if (nb <= 2) return 2;
    if (nb <= 4) return 4;
    return 0;
}

size_t fwd_smem_bytes(int variant, int nb1, int D, int T) {
    const int MT = variant_mt(variant), CS = variant_cs(variant);
    const int nb2 = std::min(8, 2 * nb1);
    const int pw = 32 * nb2 * CS;
    return sizeof(float) * ((size_t)4 * MT * D + (size_t)2 * KC * pw + (size_t)2 * MT * KC + (size_t)T * D);
}

// Launches per timestep of the per-timestep fp32 path: gather, message GEMM, its epilogue, the candidate GEMM and the update; the attention
// pre-pass; the gate GEMM and its epilogue (GRU cells); the recurrent projection (CudnnCompatibleGRUCell).
int stepwise_launches(const ModelShape& s) {
    return 5 + (s.use_att ? 1 : 0) + (s.cell != CELL_RNN ? 2 : 0) + (s.cell == CELL_CUDNN_GRU ? 1 : 0);
}

// Tiles of whole components: a tile closes before the component that would take it past `budget` rows.
void pack_components(const std::vector<int>& cuts, int V, int budget, std::vector<int>& tile_start) {
    tile_start.assign(1, 0);
    int cur = 0;
    for (size_t i = 1; i < cuts.size(); ++i)
        if (cuts[i] - cur > budget) { tile_start.push_back(cuts[i - 1]); cur = cuts[i - 1]; }
    if (V > cur) tile_start.push_back(V);
}

// Tiles of `rows` rows each, whatever the components.
void fixed_tiles(int V, int rows, std::vector<int>& tile_start) {
    tile_start.assign(1, 0);
    for (int r = rows; r < V; r += rows) tile_start.push_back(r);
    if (V > 0) tile_start.push_back(V);
}

// Whole-component tiles of up to 128 rows = two wgmma M = 64 halves, but a small batch then occupies only V/128 SMs and every tile
// sees every edge type.  When the batch cannot fill the chip, shrink the row budget to the smallest multiple of 8 that still fits all
// tiles in one wave: more SMs, and fewer edge-type blocks per tile (absent types are skipped).  Returns the budget.
int pack_to_fill_chip(const std::vector<int>& cuts, int V, int max_span, int num_sms, std::vector<int>& tile_start) {
    pack_components(cuts, V, tc::TILE_M, tile_start);
    if ((int)tile_start.size() - 1 < num_sms) {
        std::vector<int> trial;
        for (int b = std::max(32, (max_span + 7) / 8 * 8); b < tc::TILE_M; b += 8) {
            pack_components(cuts, V, b, trial);
            if ((int)trial.size() - 1 <= num_sms) { tile_start = trial; return b; }
        }
    }
    return tc::TILE_M;
}

// Whether a GCN runs on the streaming plan: hidden sizes above 128 on the tensor-core precisions, when its config asked for wide_hidden (else
// those sizes run the fp32 kernel, up to 256).
bool gcn_streams(const ModelShape& s) { return s.wide_hidden && s.precision != GGNN_PREC_FP32 && s.DP > 128; }

// The tile plan of a batch of V nodes: which kernel, and the tiles.  `cuts` are the sorted node indices where the batch may be split
// between connected components (cuts.front() == 0, cuts.back() == V); `weighted`: every message has a weight; `stream_weighted`: a weighted
// batch may take the streaming plan above hidden 128 on the tensor-core precisions (the ..._dense_weighted entries), else it is refused
// there.  Starts `p` afresh; the image builders fill in the rest.
int build_plan(const ModelShape& s, int V, bool weighted, const std::vector<int>& cuts, BatchPlan& p, std::vector<int>& tile_start,
               std::string& err, bool stream_weighted = false, bool msg_weighted = false) {
    p = BatchPlan();
    p.V = V;
    p.weighted = weighted;
    p.msg_weighted = msg_weighted;
    int max_span = 0;
    for (size_t i = 1; i < cuts.size(); ++i) max_span = std::max(max_span, cuts[i] - cuts[i - 1]);
    p.max_span = max_span;
    const char* fg = getenv("GGNN_FORCE_GLOBAL");
    const bool force_global = fg && fg[0] == '1';
    const char* prec = s.precision == GGNN_PREC_BF16X3 ? "bf16x3" : "bf16";
    char buf[256];
    if (s.model == MODEL_GCN && gcn_streams(s)) {
        // streaming plan (wide_hidden, hidden > 128, bf16x3 / bf16): fixed 128-row tiles, per layer a weighted gather into the operand
        // image and one TMA-fed streaming GEMM launch of N blocks of MMA_N columns.  No pair tables: the gather reads the target CSR.
        p.variant = 4;
        fixed_tiles(V, ts::TILE_M, tile_start);
        p.ntiles = (int)tile_start.size() - 1;
        p.ts_nblk[0] = (s.DP + ts::MMA_N - 1) / ts::MMA_N;
        p.ts_nc[0] = ts::MMA_N;
        snprintf(buf, sizeof buf, "gcn-stream-%s (2 launches per layer: weighted gather, GEMM) tiles=%d DP=%d N-blocks=%dx%d", prec, p.ntiles,
                 s.DP, p.ts_nblk[0], p.ts_nc[0]);
    } else if (s.model == MODEL_GCN) {
        // wgmma path (hidden <= 128, bf16x3 / bf16): LOCAL when every connected component fits a 128-row tile -- tiles are unions of whole
        // components, shrunk like the GGNN plan when the batch cannot fill the chip -- else GLOBAL with fixed 128-row tiles.  fp32 path:
        // fixed 32-row blocks, one launch per layer.
        p.variant = 4;
        const bool tcore = s.precision != GGNN_PREC_FP32 && s.DP <= 128;
        p.local = tcore && max_span <= tc::TILE_M && !force_global;
        p.tc_row_budget = tcore ? tc::TILE_M : gcn::F32_ROWS;
        if (p.local) p.tc_row_budget = pack_to_fill_chip(cuts, V, max_span, s.num_sms, tile_start);
        else fixed_tiles(V, p.tc_row_budget, tile_start);
        p.ntiles = (int)tile_start.size() - 1;
        if (tcore)
            snprintf(buf, sizeof buf, "gcn-wgmma-%s %s tiles=%d rows/tile<=%d DP=%d max_component=%d", prec,
                     p.local ? "LOCAL(all layers fused, 1 launch)" : "GLOBAL(1 launch per layer)", p.ntiles, p.tc_row_budget, s.DP, max_span);
        else
            snprintf(buf, sizeof buf, "gcn-fp32-ffma GLOBAL(weighted gather + FFMA GEMM, 1 launch per layer) blocks=%d rows/block=%d D=%d", p.ntiles,
                     gcn::F32_ROWS, s.D);
    } else if (s.precision != GGNN_PREC_FP32) {
        const char* fs = getenv("GGNN_TC_STREAM");
        // a component larger than a tile cannot use the tile-local fused kernel: the streaming plan beats one launch per timestep of that
        // kernel (cfg5 on an H100: 0.77 vs 0.94 ms), so it is the default there; GGNN_TC_STREAM=0/1 and GGNN_FORCE_GLOBAL=1 override.
        // A weighted batch streams only above hidden 128, where the tile kernel cannot run, and only when its caller asked for it; up to 128 it
        // keeps the tile kernel's plans (GLOBAL for a component over 128 rows), on which every pair is gathered with its weights and none
        // becomes a virtual row.
        const bool big_component = max_span > tc::TILE_M && !weighted && !force_global && !(fs && fs[0] == '0');
        // attention and CudnnCompatibleGRUCell (GGNN_CELL_CUDNN_GRU_TENSOR_CORES: the tile kernel has no candidate for it) always stream
        const bool cudnn = s.cell == CELL_CUDNN_GRU;
        if (s.DP > 128 || big_component || (fs && fs[0] == '1' && !weighted) || s.use_att || cudnn) {
            // streaming plan: fixed 128-row tiles (the gather reads the previous state from L2, so tiles need not respect components),
            // one launch per GEMM of a timestep; N blocks sized so that small batches still spread over the chip
            if (weighted && !stream_weighted) {
                err = "hidden_size > 128 on the tensor-core path needs unweighted messages here (a weighted dense adjacency runs on GGNN_PREC_FP32, "
                      "or on the streaming wgmma kernels through ggnn_set_graph_dense_weighted / ggnn_prepare_graph_dense_weighted)";
                return GGNN_EUNSUPPORTED;
            }
            p.stream = true; p.variant = 3;
            p.all_virtual = s.use_att != 0 || msg_weighted;   // (attention runs on the streaming plan at every hidden size)
            fixed_tiles(V, ts::TILE_M, tile_start);
            p.ntiles = (int)tile_start.size() - 1;
            for (int i = 0; i < 2; ++i) {
                const int width = (i + 1) * s.DP;
                // one wgmma accumulator of MMA_N columns per CTA (the MMA warpgroup holds both 64-row halves in registers)
                p.ts_nblk[i] = (width + ts::MMA_N - 1) / ts::MMA_N;
                p.ts_nc[i] = ts::MMA_N;
            }
            const char* steps = s.use_att ? (cudnn ? "+attention+cudnn-gru(5 launches per step: attention, gather-GEMM, gate GEMM, hidden-projection "
                                                     "GEMM, candidate GEMM)"
                                                   : "+attention(4 launches per step: attention, gather-GEMM, gate GEMM, candidate GEMM)")
                                          : (cudnn ? "+cudnn-gru(4 launches per step: gather-GEMM, gate GEMM, hidden-projection GEMM, candidate GEMM)"
                                                   : "(3 launches per step: gather-GEMM, gate GEMM, candidate GEMM)");
            int len = snprintf(buf, sizeof buf, "wgmma-%s STREAM%s tiles=%d DP=%d N-blocks agg/cand=%dx%d gate=%dx%d", prec, steps, p.ntiles, s.DP,
                               p.ts_nblk[0], p.ts_nc[0], p.ts_nblk[1], p.ts_nc[1]);
            if (s.DP <= 128) snprintf(buf + len, sizeof buf - len, " max_component=%d", max_span);   // (not computed for hidden sizes > 128: fixed tiles)
        } else {
            p.variant = 2;
            p.local = max_span <= tc::TILE_M && !force_global;
            int budget = tc::TILE_M;
            if (p.local) budget = pack_to_fill_chip(cuts, V, max_span, s.num_sms, tile_start);
            else fixed_tiles(V, tc::TILE_M, tile_start);
            p.ntiles = (int)tile_start.size() - 1;
            p.tc_row_budget = budget;
            // compact operand tiles when no tile exceeds 64 rows (k-group stride 1024 instead of 2048): half the operand bytes, a ~3x deeper ring
            p.tc_kgs = p.tc_row_budget <= 64 ? 1024 : 2048;
            snprintf(buf, sizeof buf, "wgmma-%s %s tiles=%d rows/tile<=%d%s DP=%d max_component=%d", prec,
                     p.local ? "LOCAL(all layers+steps fused, 1 launch)" : "GLOBAL(1 launch per step)", p.ntiles, budget,
                     p.tc_kgs == 1024 ? " (compact 64-row operand tiles)" : "", s.DP, max_span);
        }
    } else if (s.D > 256) {
        // the fp32 tile kernel holds four MT x D tiles in shared memory and at most 256 columns in its register blocking: above hidden 256
        // each timestep runs as a few launches over the whole batch.  Tiles play no part; fixed 128-row ones only split the host build.
        p.stepwise = true;
        fixed_tiles(V, ts::TILE_M, tile_start);
        p.ntiles = (int)tile_start.size() - 1;
        snprintf(buf, sizeof buf, "fp32-stepwise%s%s (%d launches per step) V=%d D=%d T=%d", s.use_att ? "+attention" : "",
                 s.cell == CELL_CUDNN_GRU ? "+cudnn-gru" : "", stepwise_launches(s), V, s.D, s.T);
    } else {
        const int D = s.D;
        const bool a_ok = pick_nb1(0, D) > 0 && fwd_smem_bytes(0, pick_nb1(0, D), D, s.T) <= s.max_smem;
        const bool b_ok = pick_nb1(1, D) > 0 && fwd_smem_bytes(1, pick_nb1(1, D), D, s.T) <= s.max_smem;
        if (!a_ok && !b_ok) {
            snprintf(buf, sizeof buf, "hidden_size=%d does not fit any fp32 tile variant", D);
            err = buf;
            return GGNN_EUNSUPPORTED;
        }
        const char* force = getenv("GGNN_FFMA_VARIANT");
        const bool a_local = a_ok && max_span <= 64, b_local = b_ok && max_span <= 32;
        if (force && (force[0] == '0' || force[0] == '1') && ((force[0] == '0') ? a_ok : b_ok)) {
            p.variant = force[0] - '0';
            p.local = p.variant == 0 ? a_local : b_local;
        } else if (b_local && (!a_local || (long)V <= (long)32 * s.num_sms * 2)) {
            p.variant = 1; p.local = true;
        } else if (a_local) {
            p.variant = 0; p.local = true;
        } else {
            p.variant = a_ok ? 0 : 1; p.local = false;
        }
        if (force_global) p.local = false;
        p.nb1 = pick_nb1(p.variant, D);
        const int MT = variant_mt(p.variant);
        if (p.local) pack_components(cuts, V, MT, tile_start);
        else fixed_tiles(V, MT, tile_start);
        p.ntiles = (int)tile_start.size() - 1;
        snprintf(buf, sizeof buf, "fp32-ffma%s%s %s tiles=%d rows/tile<=%d warps=8 colsplit=%d nb1=%d max_component=%d smem=%zuB", s.use_att ? "+attention" : "",
                 s.cell == CELL_CUDNN_GRU ? "+cudnn-gru" : "",
                 p.local ? "LOCAL(all layers+steps fused, 1 launch)" : "GLOBAL(1 launch per step)", p.ntiles, MT,
                 variant_cs(p.variant), p.nb1, max_span, fwd_smem_bytes(p.variant, p.nb1, D, s.T));
    }
    p.plan_text = buf;
    return GGNN_OK;
}

// The cut points of a batch: node boundaries no edge crosses.  The boundary before node i is crossed iff max_{j < i} reach[j] >= i, where
// reach[j] is the farthest node an edge whose lower end is node j touches.  Without `reach`, the batch is one component.
void find_cuts(const int* reach, int V, std::vector<int>& cuts) {
    cuts.assign(1, 0);
    if (reach) {
        int far = 0;
        for (int i = 1; i < V; ++i) {
            far = std::max(far, reach[i - 1]);
            if (far < i) cuts.push_back(i);
        }
    }
    if (V > 0) cuts.push_back(V);
}

}  // namespace

// ------------------------------------------------------------------------------------------ backward (host orchestration)
// The weight-gradient launch  C_s[K,N] += A_s^T . B  for every segment s (C_s = C + s*c_stride), bias[n] += sum_m B[m,n], shared by the
// GGNN and the GCN backward.  Where the split policy lives:
//  - atomic (the default): ~4 CTAs of 64 threads per SM, >= 64 rows per split (every split costs K*N atomics per segment), the splits add
//    into C with float atomics; a bias-only request sums 512-row blocks with atomics.
//  - deterministic (ggnn_set_deterministic): the split count and boundaries depend on (M, N, K, nseg) only -- the same target of
//    DET_TARGET_CTAS CTAs whatever the GPU -- and every split stores its partial into `ws`; split_reduce_kernel adds them in split order and
//    adds the sum into C (and bias) once.  A bias-only request: 512-row splits, the same reduction.
struct TnSplit {
    int splits = 1, rows = 0;   // number of row splits, rows per split (a multiple of GEMM_BK)
    size_t ws_floats = 0;       // deterministic: floats of the partials, [splits][nseg][K][N] + [splits][N]
};
constexpr int DET_TARGET_CTAS = 512;
constexpr int COLSUM_ROWS = 512;
static TnSplit tn_split(int target_ctas, bool has_C, bool has_bias, int M, int N, int K, int nseg) {
    using ggnn::bwd::TN_TILE;
    TnSplit p;
    if (has_C) {
        const int kblocks = (K + TN_TILE - 1) / TN_TILE;
        const int tiles = ((N + TN_TILE - 1) / TN_TILE) * nseg * kblocks;
        const int want = std::max(1, (target_ctas + tiles - 1) / tiles);
        const int splits = std::max(1, std::min(want, (M + 63) / 64));
        p.rows = ((M + splits - 1) / splits + ggnn::bwd::GEMM_BK - 1) / ggnn::bwd::GEMM_BK * ggnn::bwd::GEMM_BK;
        p.splits = (M + p.rows - 1) / p.rows;
        p.ws_floats = (size_t)p.splits * nseg * K * N;
    } else {
        p.rows = COLSUM_ROWS;
        p.splits = (M + COLSUM_ROWS - 1) / COLSUM_ROWS;
    }
    if (has_bias) p.ws_floats += (size_t)p.splits * N;
    return p;
}
// Floats of deterministic workspace a gemm_tn call of this shape needs (0 when the engine is not in deterministic mode).
static size_t gemm_tn_workspace(const ggnn_engine* e, bool has_C, bool has_bias, int M, int N, int K, int nseg) {
    return e->det && (has_C || has_bias) ? tn_split(DET_TARGET_CTAS, has_C, has_bias, M, N, K, nseg).ws_floats : 0;
}
// `ws` holds `ws_cap` floats; a deterministic call whose partials would not fit launches nothing and fails (the caller sizes the workspace
// from every shape it launches, gemm_tn_workspace, so this is a guard against a sizing mistake, never a silent overflow).
static int gemm_tn(ggnn_engine* e, cudaStream_t st, float* ws, size_t ws_cap, const ggnn::bwd::SegList& segs, int nseg, bool a_vec, const float* B,
                   int ldb, float* C, int ldc, size_t c_stride, float* bias, int M, int N, int K) {
    using namespace ggnn::bwd;
    if (!C && !bias) return GGNN_OK;
    const int kblocks = (K + TN_TILE - 1) / TN_TILE;
    const dim3 tiles((N + TN_TILE - 1) / TN_TILE, nseg * kblocks);
    // bf16x3 backward: the tensor-core kernels take every vector-loaded A (the edge-bias gradient's in-degree table stays on FFMA)
    const bool tcore = e->bwd_precision == GGNN_PREC_BF16X3 && a_vec;
    if (!e->det) {
        if (C) {
            const TnSplit p = tn_split(4 * e->num_sms, true, false, M, N, K, nseg);
            const dim3 grid(tiles.x, tiles.y, p.splits);
            if (tcore)
                ggnn::bwd_tc::gemm_tn_tc_atomic_kernel<<<grid, ggnn::bwd_tc::TN_TC_THREADS, 0, st>>>(segs, kblocks, B, ldb, C, ldc, c_stride, bias,
                                                                                                      M, N, K, p.rows);
            else
                gemm_tn_atomic_kernel<<<grid, 64, 0, st>>>(segs, kblocks, a_vec ? 1 : 0, B, ldb, C, ldc, c_stride, bias, M, N, K, p.rows);
        } else {
            colsum_atomic_kernel<<<dim3((N + 255) / 256, (M + COLSUM_ROWS - 1) / COLSUM_ROWS), 256, 0, st>>>(B, ldb, nullptr, 0, bias, M, N,
                                                                                                              COLSUM_ROWS);
        }
        ++e->last_launches;
        return GGNN_OK;
    }
    const TnSplit p = tn_split(DET_TARGET_CTAS, C != nullptr, bias != nullptr, M, N, K, nseg);
    if (p.ws_floats > ws_cap)
        return e->fail(GGNN_ESTATE, "internal: the deterministic workspace holds %zu floats, a weight-gradient launch (M %d, N %d, K %d, %d segments) "
                                    "needs %zu", ws_cap, M, N, K, nseg, p.ws_floats);
    float* bias_part = bias ? ws + (C ? (size_t)p.splits * nseg * K * N : 0) : nullptr;
    const dim3 grid(tiles.x, tiles.y, p.splits);
    if (C && tcore)
        ggnn::bwd_tc::gemm_tn_tc_split_kernel<<<grid, ggnn::bwd_tc::TN_TC_THREADS, 0, st>>>(segs, kblocks, B, ldb, ws, bias_part, M, N, K, p.rows);
    else if (C) gemm_tn_split_kernel<<<grid, 64, 0, st>>>(segs, kblocks, a_vec ? 1 : 0, B, ldb, ws, bias_part, M, N, K, p.rows);
    else colsum_split_kernel<<<dim3((N + 255) / 256, p.splits), 256, 0, st>>>(B, ldb, bias_part, M, N, p.rows);
    const size_t work = (C ? (size_t)nseg * K * N / 4 : 0) + (bias ? N : 0);
    split_reduce_kernel<<<(int)std::min<size_t>((work + 255) / 256, 4096), 256, 0, st>>>(ws, bias_part, p.splits, nseg, K, N, C, ldc, c_stride, bias);
    e->last_launches += 2;
    return GGNN_OK;
}
// The data-gradient launch  C[M,N] (+)= sum_s A_s[M,K] . B_s[N,K]^T  of the GGNN and the GCN backward: gemm_nt_kernel (FFMA), or its bf16x3
// wgmma twin when the engine's backward precision says so.  One CTA per output tile over the whole sum either way (no split-K).
static void gemm_nt(ggnn_engine* e, cudaStream_t st, bool acc, const float* A, int lda, int a_stride, const float* B, int ldb, int b_stride, int nseg,
                    float* C, int ldc, int M, int N, int K) {
    using namespace ggnn::bwd;
    using namespace ggnn::bwd_tc;
    if (e->bwd_precision == GGNN_PREC_BF16X3) {
        const dim3 grid((N + NT_TC_BN - 1) / NT_TC_BN, (M + NT_TC_BM - 1) / NT_TC_BM);
        if (acc) gemm_nt_tc_kernel<true><<<grid, NT_TC_THREADS, 0, st>>>(A, lda, a_stride, B, ldb, b_stride, nseg, C, ldc, M, N, K);
        else gemm_nt_tc_kernel<false><<<grid, NT_TC_THREADS, 0, st>>>(A, lda, a_stride, B, ldb, b_stride, nseg, C, ldc, M, N, K);
    } else {
        const dim3 grid((N + NT_BN - 1) / NT_BN, (M + NT_BM - 1) / NT_BM);
        if (acc) gemm_nt_kernel<true><<<grid, 128, 0, st>>>(A, lda, a_stride, B, ldb, b_stride, nseg, C, ldc, M, N, K);
        else gemm_nt_kernel<false><<<grid, 128, 0, st>>>(A, lda, a_stride, B, ldb, b_stride, nseg, C, ldc, M, N, K);
    }
    ++e->last_launches;
}

// The dense-device kernels (ggnn_dense_adj.cuh) over the current batch's b graphs of v rows: X = A.x (trans: A^T.x) from the row-major
// [V][D] `x` into `out` [V][T*D] fp32 or, with `img`, from the chunk-major `x` into the streaming plan's virtual-row image; and dA += the
// step's adjacency gradient.  Grid-stride blocks over the (graph, type, tile) list, at most 2^20 of them.  The callers count the launches.
static void dense_apply_launch(ggnn_engine* e, cudaStream_t st, bool trans, const float* A, const float* x, float* out, uint8_t* img) {
    using namespace ggnn::dadj;
    const int64_t rt = (e->dense_v + BI - 1) / BI, ct = ((img ? e->DP : e->D) + BK - 1) / BK;
    const int grid = (int)std::max<int64_t>(1, std::min<int64_t>((int64_t)e->dense_b * e->T * rt * ct, 1 << 20));
    const int b = e->dense_b, v = e->dense_v, T = e->T, D = e->D, DP = e->DP;
    if (img) dense_apply_kernel<false, true, true><<<grid, THREADS, 0, st>>>(A, x, nullptr, img, b, v, T, D, DP);
    else if (trans) dense_apply_kernel<true, false, false><<<grid, THREADS, 0, st>>>(A, x, out, nullptr, b, v, T, D, DP);
    else dense_apply_kernel<false, false, false><<<grid, THREADS, 0, st>>>(A, x, out, nullptr, b, v, T, D, DP);
}
static void dense_adj_launch(ggnn_engine* e, cudaStream_t st, const float* P, const float* h, const float* dx, const float* bias, float* dA) {
    using namespace ggnn::dadj;
    const int64_t rt = (e->dense_v + BI - 1) / BI;
    const int grid = (int)std::max<int64_t>(1, std::min<int64_t>((int64_t)e->dense_b * e->T * rt * rt, 1 << 20));
    dense_adj_grad_kernel<<<grid, THREADS, 0, st>>>(P, h, dx, bias, dA, e->dense_b, e->dense_v, e->T, e->D);
}

// The gradient fields of layer l the model has, with their sizes in floats, in ggnn_layer_grads order (a field the model lacks: size 0).
static std::array<size_t, 8> layer_grad_floats(const ggnn_engine* e, int l) {
    const size_t D = e->D, T = e->T, rows = D * (2 + e->nres[l]);   // [res.. | x | h] rows of the cell kernels
    const bool gates = e->cell != CELL_RNN;
    return {T * D * D, e->use_bias ? T * D : 0, gates ? rows * 2 * D : 0, gates ? 2 * D : 0, rows * D, D, e->use_att ? T : 0,
            e->cell == CELL_CUDNN_GRU ? D : 0};
}
static float** grad_field(ggnn_layer_grads& g, int i) {
    float** f[8] = {&g.edge_weights, &g.edge_biases, &g.gate_kernel, &g.gate_bias, &g.cand_kernel, &g.cand_bias, &g.edge_type_attention_weights,
                    &g.cand_hidden_bias};
    return f[i];
}

// d_dw (DEVICE [M] or null): the message weights' gradient, accumulated into (message-weighted batches only); on a dense-device batch the
// adjacency's gradient [b, T, v, v] (d_dA below), added into step by step.
static int ggnn_backward_impl(ggnn_engine* e, const float* d_h_out, const ggnn_layer_grads* grads, int32_t num_layers,
                              float* d_h0, float* d_dw, ggnn_stream_t stream) {
    using namespace ggnn::bwd;
    if (int rc = begin_backward(e, "ggnn_backward", "ggnn_set_graph_sparse", d_h_out, grads, num_layers, d_h0)) return rc;
    float* const d_dA = e->dense_device ? d_dw : nullptr;
    if (e->dense_device) d_dw = nullptr;
    cudaStream_t st = (cudaStream_t)stream;
    const int V = e->V, D = e->D, T = e->T, L = e->L;
    if (V == 0) return GGNN_OK;
    const size_t vd = (size_t)V * D;
    int maxres = 0;
    for (int l = 0; l < L; ++l) maxres = std::max(maxres, e->nres[l]);
    const int ldx_max = D * (maxres + 2);
    // ---- scratch
    size_t off = 0;
    auto take = [&](size_t floats) { size_t o = off; off = align_up(off + floats * sizeof(float), 256); return o; };
    const size_t o_dstate = take(vd * (L + 1)), o_dha = take(vd), o_dhb = take(vd), o_dpc = take(vd), o_dpg = take(2 * vd);
    const size_t o_dxc = take((size_t)V * ldx_max), o_dxg = take((size_t)V * ldx_max), o_rh = take(vd), o_dxp = take(vd), o_at = take(vd * T), o_gt = take(vd * T);
    // P = dx' . W^T: attention's softmax backward and the message weights' gradient (dw_slot: its per-slot sums over the steps)
    const size_t o_pall = take(e->use_att || d_dw || d_dA ? vd * T : 0), o_dsa = take(e->use_att ? (size_t)std::max<int64_t>(e->M, 1) : 0);
    const size_t o_dws = take(d_dw ? (size_t)std::max<int64_t>(e->M, 1) : 0);
    // deterministic mode: room for the partials of every weight-gradient launch below (the need is not monotone in the segment count --
    // fewer segments get more splits -- so every launched shape is sized), and the attention's per-block d a_t
    const int nodes_blocks = (V + 7) / 8;
    size_t ws_floats = 0;
    if (e->det) {
        auto need = [&](bool has_C, int N, int K, int nseg) { ws_floats = std::max(ws_floats, gemm_tn_workspace(e, has_C, true, V, N, K, nseg)); };
        for (int l = 0; l < L; ++l) {
            const int R = e->nres[l];
            need(true, D, D, R + 2);         // candidate kernel (GRU, RNN), [res.. | x | r*h or h]
            need(true, 2 * D, D, R + 2);     // gate kernel
            if (e->cell == CELL_CUDNN_GRU) { need(true, D, D, R + 1); need(true, D, D, 1); }   // input and hidden projections
        }
        need(true, D, T, 1);                 // edge biases (indeg^T . dx'), no bias partial: sized with one, which is larger
        for (int t0 = 0; t0 < T; t0 += MAX_SEGS) need(true, D, D, std::min(MAX_SEGS, T - t0));   // edge-weight chunks
        need(false, D, D, 1);                // bias-only requests
        need(false, 2 * D, D, 1);
        if (e->use_att) ws_floats = std::max(ws_floats, (size_t)nodes_blocks * T);
    }
    const size_t o_ws = take(ws_floats);
    // deterministic mode: a layer's weight gradients are summed over its timesteps in zeroed buffers, then added to the caller's once
    size_t gsum_floats = 0;
    if (e->det)
        for (int l = 0; l < L; ++l) {
            size_t f = 0;
            for (size_t x : layer_grad_floats(e, l)) f += align_up(x, 64);
            gsum_floats = std::max(gsum_floats, f);
        }
    const size_t o_gsum = take(gsum_floats);
    const size_t o_ptrs = off; off += 256;
    CU_TRY(e, e->bwd_buf.reserve(off));
    char* bb = (char*)e->bwd_buf.ptr;
    float* dstate = (float*)(bb + o_dstate);
    float *dha = (float*)(bb + o_dha), *dhb = (float*)(bb + o_dhb), *dpc = (float*)(bb + o_dpc), *dpg = (float*)(bb + o_dpg);
    float *dxc = (float*)(bb + o_dxc), *dxg = (float*)(bb + o_dxg), *rh = (float*)(bb + o_rh), *dxp = (float*)(bb + o_dxp);
    float *At = (float*)(bb + o_at), *Gt = (float*)(bb + o_gt), *Pall = (float*)(bb + o_pall), *dsa = (float*)(bb + o_dsa);
    float** d_ptrs = (float**)(bb + o_ptrs);
    float* ws = (float*)(bb + o_ws);
    float* dw_slot = (float*)(bb + o_dws);
    if (d_dw && e->M > 0) CU_TRY(e, cudaMemsetAsync(dw_slot, 0, sizeof(float) * (size_t)e->M, st));
    CU_TRY(e, cudaMemsetAsync(dstate, 0, vd * L * sizeof(float), st));
    CU_TRY(e, cudaMemcpyAsync(dstate + vd * L, d_h_out, vd * sizeof(float), cudaMemcpyDeviceToDevice, st));
    // forward values of node_states_per_layer
    std::vector<const float*> fstate(L + 1);
    for (int l = 0; l <= L; ++l) fstate[l] = layer_state(e, l, e->last_h0, e->last_out);
    const ImageView& gd = e->gd;
    const long long n = (long long)vd;
    const int eb = (int)std::min<long long>((n + 255) / 256, 4096);
    auto gemm_nt = [&](bool acc, const float* A, int lda, int a_stride, const float* B, int ldb, int b_stride, int nseg, float* C, int ldc,
                       int M, int N, int K) { ::gemm_nt(e, st, acc, A, lda, a_stride, B, ldb, b_stride, nseg, C, ldc, M, N, K); };
    // C_s[K,N] += A_s^T . B for every segment (C_s = C + s*c_stride), bias[n] += sum_m B[m,n]
    int ws_rc = GGNN_OK;   // the first failure of a weight-gradient launch (none launches after it)
    auto gemm_tn = [&](const SegList& segs, int nseg, bool a_vec, const float* B, int ldb, float* C, int ldc, size_t c_stride, float* bias, int M,
                       int N, int K) {
        if (ws_rc == GGNN_OK) ws_rc = ::gemm_tn(e, st, ws, ws_floats, segs, nseg, a_vec, B, ldb, C, ldc, c_stride, bias, M, N, K);
    };
    const int TD = T * D;
    for (int l = L - 1; l >= 0; --l) {
        const int R = e->nres[l], din = D * (1 + R), ldx = din + D;
        const ggnn_layer_weights& w = e->w[l];
        ggnn_layer_grads gw = grads[l];
        const std::array<size_t, 8> gfloats = layer_grad_floats(e, l);
        if (e->det) {
            float* p = (float*)(bb + o_gsum);
            for (int i = 0; i < 8; ++i) {
                float** f = grad_field(gw, i);
                if (!*f) continue;
                *f = gfloats[i] ? p : nullptr;
                p += align_up(gfloats[i], 64);
            }
            CU_TRY(e, cudaMemsetAsync(bb + o_gsum, 0, (char*)p - (bb + o_gsum), st));
        }
        if (R > 0) {
            float* hp[MAX_RES];
            for (int i = 0; i < R; ++i) hp[i] = dstate + (size_t)e->res[l][i] * vd;
            CU_TRY(e, cudaMemcpyAsync(d_ptrs, hp, sizeof(float*) * R, cudaMemcpyHostToDevice, st));
        }
        float* dhn = dstate + (size_t)(l + 1) * vd;   // gradient wrt the state leaving the current step
        float* dh_new = dha;
        for (int s = e->steps[l] - 1; s >= 0; --s) {
            const SaveDev sv = saved_step(e, e->step_base[l] + s);
            const float *h = sv.h_in, *x = sv.agg;
            if (e->saved_drop_keep < 1.0f) {
                dropout_grad_kernel<<<eb, 256, 0, st>>>(dhn, e->saved_drop_seed, e->step_base[l] + s, V, D, e->saved_drop_keep, n);
                ++e->last_launches;
            }
            // the cell input row [res_0 .. res_{R-1} | x | last], one [V,D] array per piece
            auto cell_segs = [&](const float* last) {
                SegList sl;
                memset(&sl, 0, sizeof sl);
                for (int i = 0; i < R; ++i) { sl.p[i] = fstate[e->res[l][i]]; sl.ld[i] = D; }
                sl.p[R] = x; sl.ld[R] = D;
                sl.p[R + 1] = last; sl.ld[R + 1] = D;
                return sl;
            };
            if (e->cell == CELL_GRU) {
                const float *r = sv.r, *u = sv.u, *c = sv.c;
                gru_bwd1_kernel<<<eb, 256, 0, st>>>(dhn, h, r, u, c, dpc, dpg, dh_new, rh, n, D, e->act); ++e->last_launches;
                gemm_nt(false, dpc, D, 0, w.cand_kernel, D, 0, 1, dxc, ldx, V, ldx, D);
                gemm_tn(cell_segs(rh), R + 2, true, dpc, D, gw.cand_kernel, D, (size_t)D * D, gw.cand_bias, V, D, D);
                gru_bwd2_kernel<<<eb, 256, 0, st>>>(dxc, ldx, (R + 1) * D, h, r, dpg, dh_new, n, D); ++e->last_launches;
                gemm_nt(false, dpg, 2 * D, 0, w.gate_kernel, 2 * D, 0, 1, dxg, ldx, V, ldx, 2 * D);
                gemm_tn(cell_segs(h), R + 2, true, dpg, 2 * D, gw.gate_kernel, 2 * D, (size_t)D * 2 * D, gw.gate_bias, V, 2 * D, D);
                split_input_grad_kernel<<<eb, 256, 0, st>>>(dxc, dxg, ldx, R, d_ptrs, dxp, e->use_avg ? gd.denom : nullptr, dh_new, 0, 1, 1, n, D);
                ++e->last_launches;
            } else if (e->cell == CELL_CUDNN_GRU) {
                // c = act(x.K_in + b_in + r*q), q = h.K_hid + b_hid: the candidate kernel's first din rows see [res.., x], its last D rows see h
                const float *r = sv.r, *u = sv.u, *c = sv.c, *q = sv.q;
                float* dq = rh;   // the r*h scratch of the GRU branch is free here
                cudnn_gru_bwd1_kernel<<<eb, 256, 0, st>>>(dhn, h, r, u, c, q, dpc, dq, dpg, dh_new, n, D, e->act); ++e->last_launches;
                gemm_nt(false, dpc, D, 0, w.cand_kernel, D, 0, 1, dxc, ldx, V, din, D);                                  // d[res.., x] = dpc . K_in^T
                gemm_nt(true, dq, D, 0, w.cand_kernel + (size_t)din * D, D, 0, 1, dh_new, D, V, D, D);                   // dh += dq . K_hid^T
                gemm_tn(cell_segs(nullptr), R + 1, true, dpc, D, gw.cand_kernel, D, (size_t)D * D, gw.cand_bias, V, D, D);
                {
                    SegList sl;
                    memset(&sl, 0, sizeof sl);
                    sl.p[0] = h; sl.ld[0] = D;
                    gemm_tn(sl, 1, true, dq, D, gw.cand_kernel ? gw.cand_kernel + (size_t)din * D : nullptr, D, 0, gw.cand_hidden_bias, V, D, D);
                }
                gemm_nt(false, dpg, 2 * D, 0, w.gate_kernel, 2 * D, 0, 1, dxg, ldx, V, ldx, 2 * D);
                gemm_tn(cell_segs(h), R + 2, true, dpg, 2 * D, gw.gate_kernel, 2 * D, (size_t)D * 2 * D, gw.gate_bias, V, 2 * D, D);
                // dxc holds only the din input columns: the recurrent gradient of the candidate went into dh_new through dq above
                split_input_grad_kernel<<<eb, 256, 0, st>>>(dxc, dxg, ldx, R, d_ptrs, dxp, e->use_avg ? gd.denom : nullptr, dh_new, 0, 1, 1, n, D);
                ++e->last_launches;
            } else {
                const float* hnew = (s == e->steps[l] - 1) ? fstate[l + 1] : saved_step(e, e->step_base[l] + s + 1).h_in;
                rnn_bwd1_kernel<<<eb, 256, 0, st>>>(dhn, hnew, dpc, n, e->act, e->saved_drop_keep < 1.0f ? e->saved_drop_keep : 1.0f); ++e->last_launches;
                gemm_nt(false, dpc, D, 0, w.cand_kernel, D, 0, 1, dxc, ldx, V, ldx, D);
                gemm_tn(cell_segs(h), R + 2, true, dpc, D, gw.cand_kernel, D, (size_t)D * D, gw.cand_bias, V, D, D);
                split_input_grad_kernel<<<eb, 256, 0, st>>>(dxc, nullptr, ldx, R, d_ptrs, dxp, e->use_avg ? gd.denom : nullptr, dh_new, 1, 0, 0, n, D);
                ++e->last_launches;
            }
            // ---- messages: all edge types at once.  At[v, t*D..] = sum of h over the type-t sources of v, Gt[s, t*D..] = sum of dx' over
            // the type-t targets of s.  A weighted batch weights both by the adjacency entry of the slot.
            GatherJob j0{gd.row_ptr, gd.src, h, At, nullptr, nullptr}, j1{gd.trow, gd.ttgt, dxp, Gt, nullptr, nullptr};
            if (e->dense_device) {   // the matrix products of the dense kernels instead of the gathers, and dA += <P_t[i], h[j]> + <dx'[i], b_t>
                const float* A = (const float*)e->dense_adj.ptr;
                if (d_dA) {
                    gemm_nt(false, dxp, D, 0, w.edge_weights, D, 0, 1, Pall, TD, V, TD, D);   // P[v, t*D+k] = <dx'[v], W_t[k, :]>
                    dense_adj_launch(e, st, Pall, h, dxp, e->use_bias ? w.edge_biases : nullptr, d_dA);
                    ++e->last_launches;
                }
                dense_apply_launch(e, st, false, A, h, At, nullptr);
                dense_apply_launch(e, st, true, A, dxp, Gt, nullptr);
                e->last_launches += 2;
            } else if (e->use_att) {   // softmax backward first (it adds to dh_new), then the gathers are weighted by the probabilities
                const float* alpha = (const float*)e->att_buf.ptr + (size_t)(e->step_base[l] + s) * (size_t)std::max<int64_t>(e->M, 1);
                gemm_nt(false, dxp, D, 0, w.edge_weights, D, 0, 1, Pall, TD, V, TD, D);   // P[v, t*D+k] = <dx'[v], W_t[k, :]>
                // the target kernel holds 8 columns of d h[v] per lane up to hidden 256, 16 above
                if (e->det && gw.edge_type_attention_weights) {   // per-block d a_t into ws, then added over the blocks in a fixed order
                    (D <= 256 ? attention_bwd_target_ordered_kernel<8> : attention_bwd_target_ordered_kernel<16>)<<<nodes_blocks, 256, 0, st>>>(
                        gd.row_ptr, gd.src, h, Pall, alpha, w.edge_type_attention_weights, dsa, dh_new, ws, V, D, T);
                    ordered_colsum_kernel<<<T, 256, 0, st>>>(ws, nodes_blocks, T, gw.edge_type_attention_weights);
                    ++e->last_launches;
                } else {
                    (D <= 256 ? attention_bwd_target_kernel<8> : attention_bwd_target_kernel<16>)<<<nodes_blocks, 256, 0, st>>>(
                        gd.row_ptr, gd.src, h, Pall, alpha, w.edge_type_attention_weights, dsa, dh_new, gw.edge_type_attention_weights, V, D, T);
                }
                attention_bwd_source_kernel<<<nodes_blocks, 256, 0, st>>>(gd.trow, gd.ttgt, gd.tslot, h, dsa, dh_new, V, D, T);
                e->last_launches += 2;
                j0.w = j1.w = alpha;
                j1.widx = gd.tslot;
            } else if (e->weighted) {
                j0.w = gd.slotw;
                j1.w = gd.tslotw;
                if (d_dw) {   // d w_m += <P[v, t], h[src_m]>: the message's own term of the gathered sum
                    gemm_nt(false, dxp, D, 0, w.edge_weights, D, 0, 1, Pall, TD, V, TD, D);   // P[v, t*D+k] = <dx'[v], W_t[k, :]>
                    msgw::message_weight_grad_kernel<<<nodes_blocks, 256, 0, st>>>(gd.row_ptr, gd.src, Pall, h, dw_slot, V, D, T);
                    ++e->last_launches;
                }
            }
            if (!e->dense_device) {
                csr_gather_all_kernel<<<dim3(nodes_blocks, 2), 256, 0, st>>>(j0, j1, V, D, T);
                ++e->last_launches;
            }
            if (e->use_bias && gw.edge_biases) {   // dB[t,:] += sum_v indeg[v,t] dx'[v,:]  =  indeg^T . dx'
                SegList sl;
                memset(&sl, 0, sizeof sl);
                sl.p[0] = gd.indeg; sl.ld[0] = T;
                gemm_tn(sl, 1, false, dxp, D, gw.edge_biases, D, 0, nullptr, V, D, T);
            }
            if (gw.edge_weights) {
                for (int t0 = 0; t0 < T; t0 += MAX_SEGS) {
                    SegList sl;
                    memset(&sl, 0, sizeof sl);
                    const int nt = std::min(MAX_SEGS, T - t0);
                    for (int t = 0; t < nt; ++t) { sl.p[t] = At + (size_t)(t0 + t) * D; sl.ld[t] = TD; }
                    gemm_tn(sl, nt, true, dxp, D, gw.edge_weights + (size_t)t0 * D * D, D, (size_t)D * D, nullptr, V, D, D);
                }
            }
            gemm_nt(true, Gt, TD, D, w.edge_weights, D, D * D, T, dh_new, D, V, D, D);
            dhn = dh_new;
            dh_new = (dh_new == dha) ? dhb : dha;
        }
        if (e->det) {
            ggnn_layer_grads out = grads[l];
            for (int i = 0; i < 8; ++i) {
                float *dst = *grad_field(out, i), *src = *grad_field(gw, i);
                if (!dst || !src) continue;
                add_inplace_kernel<<<(int)std::min<size_t>((gfloats[i] + 255) / 256, 4096), 256, 0, st>>>(dst, src, (long long)gfloats[i]);
                ++e->last_launches;
            }
        }
        if (e->steps[l] > 0) { add_inplace_kernel<<<eb, 256, 0, st>>>(dstate + (size_t)l * vd, dhn, n); ++e->last_launches; }
        else { add_inplace_kernel<<<eb, 256, 0, st>>>(dstate + (size_t)l * vd, dstate + (size_t)(l + 1) * vd, n); ++e->last_launches; }
    }
    if (ws_rc != GGNN_OK) return ws_rc;
    if (d_dw && e->M > 0) {
        msgw::add_slot_grads_kernel<<<(int)std::min<int64_t>((e->M + 255) / 256, 4096), 256, 0, st>>>(gd.msg, dw_slot, d_dw, e->M);
        ++e->last_launches;
    }
    if (d_h0) CU_TRY(e, cudaMemcpyAsync(d_h0, dstate, vd * sizeof(float), cudaMemcpyDeviceToDevice, st));
    CU_TRY(e, cudaGetLastError());
    return GGNN_OK;
}

// ------------------------------------------------------------------------------------------ C ABI
extern "C" {

const char* ggnn_last_error(const ggnn_engine* e) { return e ? e->err.c_str() : g_create_error.c_str(); }

// The checks and fields both model configs have; no CUDA (the text goes to `err`: this may run in any thread).
// `max_hidden`: the widest hidden size of the model's kernels (GGNN 512: the readout and the attention backward hold 16 columns per lane;
// GCN 256 by default, as before its streaming plan existed; 512 with wide_hidden).
static int init_common_shape(ModelShape& s, int hidden_size, int max_hidden, int num_layers, int precision, int device, std::string& err) {
    if (hidden_size <= 0 || hidden_size % 4 != 0) { err = "hidden_size must be a positive multiple of 4"; return GGNN_EINVAL; }
    if (hidden_size > max_hidden) { err = "hidden_size > " + std::to_string(max_hidden) + " is not supported by this build"; return GGNN_EUNSUPPORTED; }
    if (num_layers <= 0 || num_layers > MAX_LAYERS) { err = "num_layers must be in 1..16"; return GGNN_EINVAL; }
    if (precision != GGNN_PREC_FP32 && precision != GGNN_PREC_BF16X3 && precision != GGNN_PREC_BF16) { err = "unknown precision"; return GGNN_EINVAL; }
    s.D = hidden_size; s.L = num_layers; s.precision = precision; s.device = device;
    s.DP = (s.D + 15) / 16 * 16;
    return GGNN_OK;
}

// The model shape of a ggnn_config (what prepare_specific_graph_model fixes).  Shared by ggnn_create and the host-only constructor of
// prepared graphs.  Returns GGNN_OK or an error code.
static int init_model_shape(ModelShape& s, const ggnn_config* cfg, std::string& err) {
    auto bad = [&](const char* msg) { err = msg; return (int)GGNN_EINVAL; };
    if (int rc = init_common_shape(s, cfg->hidden_size, 512, cfg->num_layers, cfg->precision, cfg->device, err)) return rc;
    if (cfg->num_edge_types <= 0 || cfg->num_edge_types > 32) return bad("num_edge_types must be in 1..32");
    if (!cfg->layer_timesteps) return bad("layer_timesteps is null");
    const bool cudnn_tc = cfg->cell == GGNN_CELL_CUDNN_GRU_TENSOR_CORES;
    if (cfg->cell != GGNN_CELL_GRU && cfg->cell != GGNN_CELL_RNN && cfg->cell != GGNN_CELL_CUDNN_GRU && !cudnn_tc)
        return bad("Unknown RNN cell type");   // sparse:112
    if ((cfg->cell == GGNN_CELL_CUDNN_GRU || cudnn_tc) && cfg->activation != GGNN_ACT_TANH)
        return bad("CudnnCompatibleGRUCell requires the tanh activation");   // sparse:106
    if (cfg->activation != GGNN_ACT_TANH && cfg->activation != GGNN_ACT_RELU) return bad("Unknown activation function type");  // sparse:81
    s.T = cfg->num_edge_types;
    s.use_bias = cfg->use_edge_bias != 0; s.use_avg = cfg->use_edge_msg_avg_aggregation != 0;
    s.cell = cudnn_tc ? (int)CELL_CUDNN_GRU : cfg->cell; s.act = cfg->activation;
    s.cudnn_tc = cudnn_tc ? 1 : 0;
    s.use_att = cfg->use_propagation_attention != 0;
    if (s.use_att && s.T > 16) { err = "propagation attention supports at most 16 edge types"; return GGNN_EUNSUPPORTED; }
    // GGNN_ATT_FP32: the softmax-weighted gather runs on the fp32 kernels (the plan text says so); GGNN_ATT_TENSOR_CORES keeps the precision,
    // so attention at a tensor-core precision means the streaming plan with its attention pre-pass
    const bool cudnn_fp32 = s.cell == CELL_CUDNN_GRU && !cudnn_tc;
    if (s.use_att && (cfg->use_propagation_attention != GGNN_ATT_TENSOR_CORES || cudnn_fp32)) s.precision = GGNN_PREC_FP32;
    // so does the reset-after-matmul candidate of CudnnCompatibleGRUCell, unless GGNN_CELL_CUDNN_GRU_TENSOR_CORES asks for the streaming plan
    if (cudnn_fp32) s.precision = GGNN_PREC_FP32;
    int total = 0;
    for (int l = 0; l < s.L; ++l) {
        if (cfg->layer_timesteps[l] < 0) return bad("negative layer_timesteps entry");
        s.steps[l] = cfg->layer_timesteps[l];
        s.step_base[l] = total;
        total += s.steps[l];
        int nr = 0;
        if (cfg->residual_offsets && cfg->residual_layers) {
            nr = cfg->residual_offsets[l + 1] - cfg->residual_offsets[l];
            if (nr < 0 || nr > MAX_RES) return bad("a layer has more than 4 residual inputs");
            for (int i = 0; i < nr; ++i) {
                int r = cfg->residual_layers[cfg->residual_offsets[l] + i];
                // node_states_per_layer has l+1 entries when layer l is built (sparse:144: IndexError otherwise)
                if (r < 0 || r > l) return bad("residual connection refers to a layer that does not exist yet");
                s.res[l][i] = r;
            }
        }
        s.nres[l] = nr;
    }
    s.total_steps = total;
    return GGNN_OK;
}

// The model shape of a ggnn_gcn_config (chem_tensorflow_gcn.py:42-82): one edge type, one "timestep" per layer (the dropout's global step
// is the layer index).
static int init_gcn_shape(ModelShape& s, const ggnn_gcn_config* cfg, std::string& err) {
    const int max_hidden = cfg->wide_hidden ? 512 : 256;
    if (int rc = init_common_shape(s, cfg->hidden_size, max_hidden, cfg->num_layers, cfg->precision, cfg->device, err)) return rc;
    s.model = MODEL_GCN;
    s.wide_hidden = cfg->wide_hidden != 0;
    s.T = 1;
    s.use_bias = cfg->use_bias != 0;
    s.cell = CELL_RNN; s.act = ACT_RELU;
    for (int l = 0; l < s.L; ++l) { s.steps[l] = 1; s.step_base[l] = l; s.nres[l] = 0; }
    s.total_steps = s.L;
    return GGNN_OK;
}

// The device half of ggnn_create / ggnn_gcn_create: takes ownership of `e` (deleted on failure) and publishes it in *out.
static int attach_device(ggnn_engine* e, ggnn_engine** out) {
    cudaError_t st = cudaSetDevice(e->device);
    cudaDeviceProp prop;
    if (st == cudaSuccess) st = cudaGetDeviceProperties(&prop, e->device);
    if (st != cudaSuccess) {
        g_create_error = std::string("CUDA device unavailable: ") + cudaGetErrorString(st);
        delete e;
        return GGNN_ECUDA;
    }
    e->num_sms = prop.multiProcessorCount;
    e->max_smem = prop.sharedMemPerBlockOptin;
    memset(e->w, 0, sizeof e->w);
    if (e->err_flag.reserve(sizeof(int)) != cudaSuccess || cudaMemset(e->err_flag.ptr, 0, sizeof(int)) != cudaSuccess) {
        g_create_error = "cudaMalloc failed";
        delete e;
        return GGNN_ECUDA;
    }
    *out = e;
    return GGNN_OK;
}

int ggnn_create(const ggnn_config* cfg, ggnn_engine** out) {
    if (!cfg || !out) { g_create_error = "null argument"; return GGNN_EINVAL; }
    *out = nullptr;
    ggnn_engine* e = new ggnn_engine();
    if (int rc = init_model_shape(*e, cfg, g_create_error)) { delete e; return rc; }
    return attach_device(e, out);
}

int ggnn_destroy(ggnn_engine* e) {
    if (!e) return GGNN_OK;
    cudaSetDevice(e->device);
    e->graph_buf.release(); e->ds_table.release(); e->state_buf.release(); e->save_bufs.release(); e->io_buf.release(); e->bwd_buf.release();
    e->tc_tiles.buf.release(); e->tc_respre.release(); e->ts_tiles.buf.release(); e->ts_images.release(); e->ts_virt.release(); e->err_flag.release();
    e->step_wt.buf.release(); e->step_buf.release(); e->dense_adj.release();
    if (e->own_prep) { ggnn_free_prepared_graph(e->own_prep); e->own_prep = nullptr; }
    e->ro_buf.release(); e->ro_stage.release(); e->att_buf.release(); e->ro_ws.release(); e->ro_kval.release();
    delete e;
    return GGNN_OK;
}

int ggnn_set_weights(ggnn_engine* e, const ggnn_layer_weights* layers, int32_t num_layers) {
    if (!e) return GGNN_EINVAL;
    GGNN_REQUIRE_MODEL(e, MODEL_GGNN);
    if (!layers || num_layers != e->L) return e->fail(GGNN_EINVAL, "expected %d layers of weights, got %d", e->L, num_layers);
    for (int l = 0; l < e->L; ++l) {
        const ggnn_layer_weights& w = layers[l];
        if (!w.edge_weights || !w.cand_kernel || !w.cand_bias) return e->fail(GGNN_EINVAL, "layer %d: null edge_weights/cand_kernel/cand_bias", l);
        if (e->use_bias && !w.edge_biases) return e->fail(GGNN_EINVAL, "layer %d: use_edge_bias set but edge_biases is null", l);
        if (e->cell != CELL_RNN && (!w.gate_kernel || !w.gate_bias)) return e->fail(GGNN_EINVAL, "layer %d: GRU needs gate_kernel/gate_bias", l);
        if (e->cell == CELL_CUDNN_GRU && !w.cand_hidden_bias) return e->fail(GGNN_EINVAL, "layer %d: CudnnCompatibleGRUCell needs cand_hidden_bias", l);
        if (e->use_att && !w.edge_type_attention_weights) return e->fail(GGNN_EINVAL, "layer %d: use_propagation_attention set but edge_type_attention_weights is null", l);
        const void* ps[7] = {w.edge_weights, w.edge_biases, w.gate_kernel, w.gate_bias, w.cand_kernel, w.cand_bias, w.cand_hidden_bias};
        for (const void* q : ps)
            if (q && ((uintptr_t)q & 15)) return e->fail(GGNN_EINVAL, "layer %d: weight pointers must be 16-byte aligned", l);
    }
    for (int l = 0; l < e->L; ++l) e->w[l] = layers[l];   // all or nothing: a refused call leaves the previous weights bound
    e->weights_set = true;
    ++e->weights_gen;       // the tensor-core paths re-tile their bf16 copies at their next forward
    e->saved_valid = false;   // a backward combines the saved activations with the bound weights: both must be the last forward's
    return GGNN_OK;
}

static int reserve_states(ggnn_engine* e) {
    const size_t vd = (size_t)std::max(e->V, 1) * e->D * sizeof(float);
    CU_TRY(e, e->state_buf.reserve(vd * (size_t)(e->L + 1)));
    if (e->save && e->model == MODEL_GGNN) CU_TRY(e, e->save_bufs.reserve(vd * (e->cell == CELL_CUDNN_GRU ? 6 : 5) * (size_t)std::max(e->total_steps, 1)));
    return GGNN_OK;
}

// Stable counting sort of the messages by (target, type): counts[k + 1] holds the number of messages of row k = target*T + type on
// entry (it is reused as the write cursors).  Messages are visited in the reference's order (type-major, then list order,
// sparse:124-129), so within a row they stay in message order -- this IS NumPy's stable argsort by target.
static void fill_target_csr(int V, int T, const int32_t* const* adj, const int32_t* num_edges, std::vector<int>& counts, int* row_ptr,
                            int* csr_src, int* csr_msg) {
    row_ptr[0] = 0;
    for (size_t k = 1; k <= (size_t)V * T; ++k) row_ptr[k] = row_ptr[k - 1] + counts[k];
    std::vector<int>& pos = counts;
    for (size_t k = 0; k < (size_t)V * T; ++k) pos[k] = row_ptr[k];
    int m = 0;
    for (int t = 0; t < T; ++t) {
        const int32_t* a = adj[t];
        for (int i = 0; i < num_edges[t]; ++i, ++m) {
            const int slot = pos[(size_t)a[2 * i + 1] * T + t]++;
            csr_src[slot] = a[2 * i];
            csr_msg[slot] = m;
        }
    }
}

// Streaming plan: number the (target, type) pairs marked -2 ("several messages") in row order, replace the mark by -(2 + vid) and list
// their sources (vptr / vsrc).  `pair` already holds -1 / the single source.  The independent reference of ggnn_host_stream_tables, which
// the CPU tests hold the builder's own tables (stream_rows) against.
static void number_virtual_rows(int ntiles, int T, const int* tile_start, const int* row_ptr, const int* csr_src, int* pair, int* vptr, int* vsrc,
                                int* tvp) {
    int vid = 0, vm = 0;
    vptr[0] = 0;
    for (int i = 0; i < ntiles; ++i) {
        tvp[i] = vid;
        for (size_t k = (size_t)tile_start[i] * T, kend = (size_t)tile_start[i + 1] * T; k < kend; ++k) {
            if (pair[k] != -2) continue;
            const int b = row_ptr[k], cnt = row_ptr[k + 1] - b;
            pair[k] = -(2 + vid);
            for (int m = 0; m < cnt; ++m) vsrc[vm++] = csr_src[b + m];
            vptr[++vid] = vm;
        }
    }
    tvp[ntiles] = vid;
}

// The tile plan ggnn_set_graph_sparse would make for this batch, without an engine or a GPU: the cut points (node boundaries no edge
// crosses, found by a single-threaded pass of its own) and build_plan().
int ggnn_host_tile_plan(int32_t hidden_size, int32_t num_edge_types, int32_t precision, int32_t num_sms, int32_t V, const int32_t* const* adj,
                        const int32_t* num_edges, int32_t* tile_start, int32_t tile_capacity, int32_t* num_tiles, char* plan_text,
                        int32_t plan_text_capacity) {
    if (hidden_size <= 0 || num_edge_types <= 0 || V < 0 || !adj || !num_edges || !tile_start || !num_tiles || num_sms <= 0) return GGNN_EINVAL;
    // same cut detection as ggnn_set_graph_sparse: reach[j] = farthest node an edge starting at node j touches
    std::vector<int> reach((size_t)V + 1, 0);
    for (int t = 0; t < num_edge_types; ++t)
        for (int i = 0; i < num_edges[t]; ++i) {
            const int s = adj[t][2 * i], d = adj[t][2 * i + 1];
            if ((unsigned)s >= (unsigned)V || (unsigned)d >= (unsigned)V) return GGNN_ERANGE;
            const int lo = std::min(s, d), hi = std::max(s, d);
            if (hi > reach[lo]) reach[lo] = hi;
        }
    std::vector<int> cuts;
    find_cuts(reach.data(), V, cuts);
    ModelShape s;
    s.D = hidden_size; s.T = num_edge_types; s.precision = precision; s.num_sms = num_sms; s.max_smem = HOST_MAX_SMEM;
    if (precision != GGNN_PREC_FP32) s.DP = (hidden_size + 15) / 16 * 16;
    BatchPlan p;
    std::string err;
    std::vector<int> ts;
    int rc = build_plan(s, V, false, cuts, p, ts, err);
    if (rc) return rc;
    *num_tiles = p.ntiles;
    if ((int)ts.size() > tile_capacity) return GGNN_EINVAL;
    for (size_t i = 0; i < ts.size(); ++i) tile_start[i] = ts[i];
    if (plan_text && plan_text_capacity > 0) snprintf(plan_text, (size_t)plan_text_capacity, "%s", p.plan_text.c_str());
    return GGNN_OK;
}

// The same CSR build without an engine or a GPU (host arithmetic only): lets the CPU test-suite pin the integer path bit for bit.
int ggnn_host_target_csr(int32_t V, int32_t T, const int32_t* const* adj, const int32_t* num_edges, int32_t* row_ptr, int32_t* src,
                         int32_t* msg) {
    if (V < 0 || T <= 0 || !adj || !num_edges || !row_ptr) return GGNN_EINVAL;
    std::vector<int> counts((size_t)V * T + 1, 0);
    int64_t M = 0;
    for (int t = 0; t < T; ++t) {
        if (num_edges[t] < 0 || (num_edges[t] > 0 && !adj[t])) return GGNN_EINVAL;
        M += num_edges[t];
        for (int i = 0; i < num_edges[t]; ++i) {
            const int s = adj[t][2 * i], d = adj[t][2 * i + 1];
            if ((unsigned)s >= (unsigned)V || (unsigned)d >= (unsigned)V) return GGNN_ERANGE;
            ++counts[(size_t)d * T + t + 1];
        }
    }
    if (M > 0 && (!src || !msg)) return GGNN_EINVAL;
    fill_target_csr(V, T, adj, num_edges, counts, row_ptr, src, msg);
    return GGNN_OK;
}

int ggnn_host_stream_tables(int32_t V, int32_t T, const int32_t* const* adj, const int32_t* num_edges, int32_t* pair_src, int32_t* vrow_ptr,
                            int32_t vrow_capacity, int32_t* vsrc, int32_t vsrc_capacity, int32_t* tile_vptr, int32_t* num_virtual_rows) {
    if (V < 0 || T <= 0 || !adj || !num_edges || !pair_src || !vrow_ptr || !vsrc || !tile_vptr || !num_virtual_rows) return GGNN_EINVAL;
    std::vector<int> row_ptr((size_t)V * T + 1), src, msg;
    int64_t M = 0;
    for (int t = 0; t < T; ++t) M += num_edges[t];
    src.resize((size_t)std::max<int64_t>(M, 1)); msg.resize((size_t)std::max<int64_t>(M, 1));
    int rc = ggnn_host_target_csr(V, T, adj, num_edges, row_ptr.data(), src.data(), msg.data());
    if (rc) return rc;
    const int ntiles = (V + ts::TILE_M - 1) / ts::TILE_M;
    std::vector<int> tile_start(ntiles + 1);
    for (int i = 0; i <= ntiles; ++i) tile_start[i] = std::min(i * ts::TILE_M, V);
    int nv = 0; int64_t nvm = 0;
    for (size_t k = 0; k < (size_t)V * T; ++k) {
        const int cnt = row_ptr[k + 1] - row_ptr[k];
        pair_src[k] = cnt == 0 ? -1 : (cnt == 1 ? src[row_ptr[k]] : -2);
        if (cnt >= 2) { ++nv; nvm += cnt; }
    }
    for (size_t k = (size_t)V * T; k < (size_t)ntiles * ts::TILE_M * T; ++k) pair_src[k] = -1;
    if (nv + 1 > vrow_capacity || nvm > vsrc_capacity) return GGNN_EINVAL;
    number_virtual_rows(ntiles, T, tile_start.data(), row_ptr.data(), src.data(), pair_src, vrow_ptr, vsrc, tile_vptr);
    *num_virtual_rows = nv;
    return GGNN_OK;
}

#ifdef _OPENMP
// Size of the host team for the per-batch graph builders: up to 8 threads, bounded by the cores this process may run on divided by the
// number of ranks on the node (LOCAL_WORLD_SIZE, set by torchrun).  Deliberately NOT omp_get_max_threads(): torchrun exports
// OMP_NUM_THREADS=1 to every rank by default ("to avoid your system being overloaded"), which would silently serialise the builders of
// exactly the multi-GPU runs (measured at N = 2: dense batch e2e 0.77 ms against 0.41 ms at N = 1); 8 ranks x 8 short-lived builder threads
// are far below a GPU host's core count.  GGNN_HOST_THREADS overrides.
static int host_team_size() {
    int avail = 0;
    cpu_set_t set;
    if (sched_getaffinity(0, sizeof set, &set) == 0) avail = CPU_COUNT(&set);
    if (avail <= 0) avail = omp_get_num_procs();
    int ranks = 1;
    if (const char* lws = getenv("LOCAL_WORLD_SIZE")) ranks = std::max(1, atoi(lws));
    return std::max(1, std::min(8, avail / ranks));
}

// One-time probe per process: is a parallel region of `team` threads cheap to enter here?  (Third of three empty regions under 150 us.)
static bool host_team_is_fast(int team) {
    static int verdict[65] = {0};   // 0 unknown, 1 fast, -1 slow; a benign race at worst probes twice
    if (team < 2 || team > 64) return false;
    if (verdict[team] == 0) {
        double us = 0.0;
        for (int rep = 0; rep < 3; ++rep) {
            const auto t0 = std::chrono::steady_clock::now();
            int seen = 0;
#pragma omp parallel num_threads(team) reduction(+ : seen)
            { seen += 1; }
            us = std::chrono::duration<double, std::micro>(std::chrono::steady_clock::now() - t0).count();
            if (seen < 1) us = 1e9;
        }
        verdict[team] = us < 150.0 ? 1 : -1;
        if (getenv("GGNN_HOST_TIMING")) fprintf(stderr, "[ggnn host] OpenMP team of %d: region entry %.1f us -> %s\n", team, us, us < 150.0 ? "used" : "not used");
    }
    return verdict[team] > 0;
}
#endif

// The layout of a batch's graph image from its plan (V, ntiles, stream, weighted) and sizes: M messages, nv virtual rows holding nvm
// messages (streaming plan); `save`: the image carries the source-keyed CSR.  Fills the plan's offsets and returns the image's size.  Shared
// by the edge-list builder and the device-resident dataset (ggnn_dataset_prepare_batch), whose kernels write the same sections.
static size_t layout_image(const ModelShape& shape, BatchPlan& p, bool save, int64_t M, int nv, int64_t nvm) {
    const int V = p.V, T = shape.T, ntiles = p.ntiles;
    size_t off = 0;
    p.M = M;
    p.pads.clear();
    // a section whose builders write its first `used` bytes, in room for `room` bytes (at least one element), 16-byte aligned; the bytes
    // after `used` up to the next section are recorded in p.pads
    auto place = [&](size_t used, size_t room) {
        const size_t at = off;
        off = align_up(at + room, 16);
        if (off > at + used) p.pads.push_back({at + used, off - at - used});
        return at;
    };
    const size_t I = sizeof(int), Mu = (size_t)M, Mr = (size_t)std::max<int64_t>(M, 1);
    const size_t VT = (size_t)V * T, nvu = (size_t)nv, nvr = (size_t)std::max(nv, 1), nvmu = (size_t)nvm;
    p.off_row_ptr = place(I * (VT + 1), I * (VT + 1));
    p.off_src = place(I * Mu, I * Mr);
    p.off_msg = place(I * Mu, I * Mr);
    p.off_indeg = place(sizeof(float) * VT, sizeof(float) * (size_t)std::max(V, 1) * T);
    p.off_denom = place(sizeof(float) * (size_t)V, sizeof(float) * (size_t)std::max(V, 1));
    p.off_tiles = place(I * (size_t)(ntiles + 1), I * (size_t)(ntiles + 1));
    p.off_mask = place(sizeof(unsigned) * (size_t)ntiles, sizeof(unsigned) * (size_t)std::max(ntiles, 1));
    p.has_transpose = save;
    if (p.has_transpose) {
        p.off_trow = place(I * (VT + 1), I * (VT + 1));
        p.off_ttgt = place(I * Mu, I * Mr);
        p.off_tslot = shape.use_att || p.msg_weighted ? place(I * Mu, I * Mr) : off;
    }
    // streaming plan: per (target, type) pair the ONE node to copy from (or none / a virtual row), see ggnn_fwd_stream.cuh
    if (p.stream) {
        const size_t pairs = I * (size_t)std::max(ntiles, 1) * ts::TILE_M * T;
        p.off_pair = place(pairs, pairs);
        p.off_vptr = place(I * (nvu + 1), I * (nvu + 1));
        p.off_vsrc = place(I * nvmu, I * (size_t)std::max<int64_t>(nvm, 1));
        p.off_tvp = place(I * (size_t)(ntiles + 1), I * (size_t)(ntiles + 1));
        p.off_vinfo = place(I * 8 * nvu, I * 8 * nvr);
        if (p.weighted || p.all_virtual) p.off_vslot = place(I * nvu, I * nvr);
    }
    if (p.weighted) {   // per-slot adjacency weights
        p.off_slotw = place(sizeof(float) * Mu, sizeof(float) * Mr);
        if (p.has_transpose) p.off_tslotw = place(sizeof(float) * Mu, sizeof(float) * Mr);
    }
    p.ts_nv = nv;
    return off;
}

// The typed view of an image laid out by plan `p` (layout_image) at `base`.  The one statement of which sections a plan carries: the
// source-keyed CSR with save_for_backward (its slot map with attention and on a message-weighted batch, its weights on a weighted batch), the streaming tables on the
// streaming plan (the virtual rows' first slots on a weighted one and with attention), the slot weights on a weighted batch.  Every other section is null.
static ImageView image_view(const BatchPlan& p, bool use_att, char* base) {
    auto sec = [&](size_t off, bool present) { return present ? (void*)(base + off) : nullptr; };
    ImageView v;
    v.row_ptr = (int*)sec(p.off_row_ptr, true); v.src = (int*)sec(p.off_src, true); v.msg = (int*)sec(p.off_msg, true);
    v.indeg = (float*)sec(p.off_indeg, true); v.denom = (float*)sec(p.off_denom, true);
    v.tile_start = (int*)sec(p.off_tiles, true); v.tile_mask = (unsigned*)sec(p.off_mask, true);
    v.trow = (int*)sec(p.off_trow, p.has_transpose); v.ttgt = (int*)sec(p.off_ttgt, p.has_transpose);
    v.tslot = (int*)sec(p.off_tslot, p.has_transpose && (use_att || p.msg_weighted));
    v.pair = (int*)sec(p.off_pair, p.stream); v.vptr = (int*)sec(p.off_vptr, p.stream); v.vsrc = (int*)sec(p.off_vsrc, p.stream);
    v.tvp = (int*)sec(p.off_tvp, p.stream); v.vinfo = (int*)sec(p.off_vinfo, p.stream); v.vslot = (int*)sec(p.off_vslot, p.stream && (p.weighted || p.all_virtual));
    v.slotw = (float*)sec(p.off_slotw, p.weighted); v.tslotw = (float*)sec(p.off_tslotw, p.weighted && p.has_transpose);
    return v;
}

// ---- the sections' builders: the batch builder below runs them over a whole batch, ds_add_graph over one graph of a dataset, so every
// section has one format.

// Pass 1 over the edge lists (adj[t]: type t's (source, target) pairs; type_base[t]: the position of its first message in the reference's
// type-major message order, type_base[T] = M): checks every edge against V nodes, counts the messages of every (target, type) row into
// counts[k + 1] (V*T + 1 entries) and, with `reach` (V + 1 entries), sets reach[j] = the farthest node an edge whose lower end is node j
// touches.  Split over `nth` threads by EDGE ranges: counting is commutative, so the threads add into the shared per-row counts with relaxed
// atomic increments (and an atomic max for `reach`) -- same totals for every thread count; a single thread uses plain increments.  Returns
// false when an edge is out of range (first_bad_edge names it).
static bool count_edges(int V, int T, const int32_t* const* adj, const int64_t* type_base, int nth, int* counts, int* reach) {
    const int64_t M = type_base[T];
    const bool need_cuts = reach != nullptr;
    int bad_edge = 0;
#ifdef _OPENMP
#pragma omp parallel num_threads(nth) if (nth > 1)
#endif
    {
        int k = 0, n = 1;
#ifdef _OPENMP
        k = omp_get_thread_num(); n = omp_get_num_threads();
#endif
        {   // clear this thread's slice of the scratch arrays
            const size_t nc = (size_t)V * T + 1, c0 = nc * k / n, c1 = nc * (k + 1) / n;
            std::fill(counts + c0, counts + c1, 0);
            if (need_cuts) {
                const size_t nr = (size_t)V + 1, r0 = nr * k / n, r1 = nr * (k + 1) / n;
                std::fill(reach + r0, reach + r1, 0);
            }
        }
#ifdef _OPENMP
#pragma omp barrier
#endif
        const int64_t e0 = M * k / n, e1 = M * (k + 1) / n;   // this thread's messages, in the type-major order
        int* const cnt = counts;
        int* const rch = reach;
        bool bad = false;
        for (int t = 0; t < T && !bad; ++t) {
            const int32_t* a = adj[t];
            const int i0 = (int)(std::max(e0, type_base[t]) - type_base[t]);
            const int i1 = (int)(std::min(e1, type_base[t + 1]) - type_base[t]);
            if (n == 1) {
                for (int i = i0; i < i1; ++i) {
                    const int s = a[2 * i], d = a[2 * i + 1];
                    if ((unsigned)s >= (unsigned)V || (unsigned)d >= (unsigned)V) { bad = true; break; }
                    ++cnt[(size_t)d * T + t + 1];
                    if (need_cuts) {
                        const int lo = std::min(s, d), hi = std::max(s, d);
                        rch[lo] = std::max(rch[lo], hi);   // unconditional store: the compare-and-branch form mispredicts on every other edge
                    }
                }
            } else {
                for (int i = i0; i < i1; ++i) {
                    const int s = a[2 * i], d = a[2 * i + 1];
                    if ((unsigned)s >= (unsigned)V || (unsigned)d >= (unsigned)V) { bad = true; break; }
                    __atomic_fetch_add(cnt + ((size_t)d * T + t + 1), 1, __ATOMIC_RELAXED);
                    if (need_cuts) {
                        const int lo = std::min(s, d), hi = std::max(s, d);
                        int cur = __atomic_load_n(rch + lo, __ATOMIC_RELAXED);
                        while (hi > cur && !__atomic_compare_exchange_n(rch + lo, &cur, hi, true, __ATOMIC_RELAXED, __ATOMIC_RELAXED)) {}
                    }
                }
            }
        }
        if (bad) {
#ifdef _OPENMP
#pragma omp atomic write
#endif
            bad_edge = 1;
        }
    }
    return !bad_edge;
}

// The first edge in the lists' order that is out of range for V nodes (after count_edges found one): its type and index.
static void first_bad_edge(int V, int T, const int32_t* const* adj, const int32_t* num_edges, int& bad_t, int& bad_i) {
    bad_t = bad_i = 0;
    for (int t = 0; t < T; ++t)
        for (int i = 0; i < num_edges[t]; ++i) {
            const int s = adj[t][2 * i], d = adj[t][2 * i + 1];
            if ((unsigned)s >= (unsigned)V || (unsigned)d >= (unsigned)V) { bad_t = t; bad_i = i; return; }
        }
}

// The denominators of nodes [v0, v1) from the [V][T] in-degrees: tf.reduce_sum over the type axis in fp32 (sparse:207), then
// + SMALL_NUMBER (:209).
static void fill_denominators(int v0, int v1, int T, const float* indeg, float* denom) {
    for (int v = v0; v < v1; ++v) {
        const float* row = indeg + (size_t)v * T;
        float s = 0.0f;
        for (int t = 0; t < T; ++t) s += row[t];
        denom[v] = s + 1e-7f;
    }
}

// The source-keyed CSR of the backward pass (rows source*T+type -> targets, in message order), which turns its scatter into a gather:
// trow [V*T + 1], ttgt [M]; `tslot` (when non-null) the target-CSR slot of every entry, from csr_msg (the message of every target-CSR slot);
// `tslotw` (when non-null) its weight, from the per-message weights w (zero without them).
static void fill_source_csr(int V, int T, const int32_t* const* adj, const int32_t* num_edges, int64_t M, const int* csr_msg, const float* w,
                            int* trow, int* ttgt, int* tslot, float* tslotw) {
    std::vector<int> cnt((size_t)V * T + 1, 0);
    for (int t = 0; t < T; ++t)
        for (int i = 0; i < num_edges[t]; ++i) ++cnt[(size_t)adj[t][2 * i] * T + t + 1];
    trow[0] = 0;
    for (size_t k = 1; k <= (size_t)V * T; ++k) trow[k] = trow[k - 1] + cnt[k];
    for (size_t k = 0; k < (size_t)V * T; ++k) cnt[k] = trow[k];
    std::vector<int> slot_of_msg;
    if (tslot) {
        slot_of_msg.resize((size_t)std::max<int64_t>(M, 1));
        for (int64_t k = 0; k < M; ++k) slot_of_msg[csr_msg[k]] = (int)k;
    }
    int m = 0;
    for (int t = 0; t < T; ++t)
        for (int i = 0; i < num_edges[t]; ++i, ++m) {
            const int j = cnt[(size_t)adj[t][2 * i] * T + t]++;
            ttgt[j] = adj[t][2 * i + 1];
            if (tslot) tslot[j] = slot_of_msg[m];
            if (tslotw) tslotw[j] = w ? w[m] : 0.0f;
        }
}

// The streaming plan's tables of the (target, type) rows [r0, r1), one sequential pass: pair[r] = -1 (no message), its one source, or
// -(2 + vid) for a virtual row (several messages), numbered on from `vid`; a virtual row's sources go to vsrc from `vm` on, its end to
// vptr[vid + 1] and, when `vinfo` is non-null, its count and first seven sources to vinfo[8 * vid ..].  Advances vid and vm.
// Weighted batches (`slotw`: the slot weights of these rows, in target-CSR order): a row is a copy only if its one message weighs exactly
// 1.0f, every other row with messages is a virtual row, and vslot[vid] = its first slot.  `all_virtual` (attention, whose probability of a
// lone message is 1 / (1 + 1e-7), not 1): every row with messages is a virtual row.
static void stream_rows(size_t r0, size_t r1, const int* row_ptr, const int* csr_src, const float* slotw, bool all_virtual, int* pair, int* vptr,
                        int* vsrc, int* vinfo, int* vslot, int& vid, int& vm) {
    for (size_t r = r0; r < r1; ++r) {
        const int b = row_ptr[r], cnt = row_ptr[r + 1] - b;
        if (cnt == 0) pair[r] = -1;
        else if (cnt == 1 && !all_virtual && (!slotw || slotw[b] == 1.0f)) pair[r] = csr_src[b];
        else {
            pair[r] = -(2 + vid);
            if (vslot) vslot[vid] = b;
            if (vinfo) {
                vinfo[8 * vid] = cnt;
                for (int m = 0; m < 7; ++m) vinfo[8 * vid + 1 + m] = m < cnt ? csr_src[b + m] : 0;
            }
            for (int m = 0; m < cnt; ++m) vsrc[vm++] = csr_src[b + m];
            vptr[++vid] = vm;
        }
    }
}

// GCN entries (row i = output, column j = input, int64) as one edge type j -> i: checks every entry against V nodes and writes the int32
// (source j, target i) pairs in list order.  Returns the index of the first entry out of range, or -1.
static int64_t gcn_pairs(int64_t V, int64_t nnz, const int64_t* list, int32_t* pairs) {
    for (int64_t k = 0; k < nnz; ++k) {
        const int64_t i = list[2 * k], j = list[2 * k + 1];
        if (i < 0 || i >= V || j < 0 || j >= V) return k;
        pairs[2 * k] = (int32_t)j;
        pairs[2 * k + 1] = (int32_t)i;
    }
    return -1;
}

// ---- the host half of ggnn_set_graph_sparse: validation, tile plan, stable target-sorted CSR, streaming tables -> g->image.
// `weighted`: the batch has one weight per message, `w`, in the type-major message order (required when there are messages); the image
// then carries them in target-CSR order and, with the source-keyed CSR, in source-CSR order.  `stream_weighted`: see build_plan.
// `msg_weighted` (with weighted and w null; for the GGNN with stream_weighted): the weights come later, on the device -- the weight sections
// are zero and the plan is the one every weight vector shares.
// Nothing here touches the device except the pinned allocation of the image and the wait for the previous upload out of it.
static int build_sparse_image(ggnn_prepared_graph* g, int32_t V, const int32_t* const* adj, const int32_t* num_edges, const float* indeg,
                              bool weighted, const float* w, bool stream_weighted = false, bool msg_weighted = false) {
    const ModelShape& shape = g->shape;
    BatchPlan& p = g->plan;
    g->valid = false;
    static const bool host_timing = getenv("GGNN_HOST_TIMING") != nullptr;
    const auto t_begin = std::chrono::steady_clock::now();
    auto lap = [&](const char* what, std::chrono::steady_clock::time_point& t) {
        if (!host_timing) return;
        const auto now = std::chrono::steady_clock::now();
        fprintf(stderr, "[ggnn host] %-18s %7.1f us\n", what, std::chrono::duration<double, std::micro>(now - t).count());
        t = now;
    };
    auto t_lap = t_begin;
    if (V < 0 || !adj || !num_edges || (!indeg && V > 0)) return g->fail(GGNN_EINVAL, "null/negative argument");
    const int T = shape.T;
    int64_t M = 0;
    for (int t = 0; t < T; ++t) {
        if (num_edges[t] < 0 || (num_edges[t] > 0 && !adj[t])) return g->fail(GGNN_EINVAL, "adjacency list %d is null/negative", t);
        M += num_edges[t];
    }
    if (M > 0x7fffffff || (int64_t)V * T + 1 > 0x7fffffff) return g->fail(GGNN_EUNSUPPORTED, "batch too large for int32 indexing");
    if (weighted && !msg_weighted && M > 0 && !w) return g->fail(GGNN_EINVAL, "null message weights");

    // ---- host threads.  Every pass below is split over `nth` threads by TARGET ranges (pass 1: equal node ranges; later passes: equal
    // tile ranges): each thread scans the whole edge list (sequential reads) and performs only the scattered writes of its own rows, in the
    // list's order -- so every row keeps the reference's message order and the image is bit-identical for every thread count
    // (tests/test_prepared_graph_cpu.py pins it against the single-pass ggnn_host_target_csr and NumPy's stable sort).
    // Small batches stay on one thread (a cfg2-sized build is ~80 us: less than a team's wake-up).  Large ones use ONE team size per
    // process, and only after host_team_is_fast() has seen that entering a parallel region of that size is cheap here: libgomp's region
    // entry can cost milliseconds in some containers (measured: 8-18 ms per region for 2-3 threads on an 8-CPU box, 2 us for 8).
    int nth = 1;
#ifdef _OPENMP
    if (M >= 24000) {
        const int team = host_team_size();
        if (team > 1 && host_team_is_fast(team)) nth = team;
    }
    if (const char* nt = getenv("GGNN_HOST_THREADS")) nth = std::max(1, std::min(atoi(nt), 64));
#endif
    // ---- pass 1: validate, count per (target,type), mark which node boundaries are spanned by an edge (the cut points of the tile-local
    // plans; the streaming plan of hidden sizes > 128 and the per-timestep fp32 path above 256 tile by fixed 128-row blocks and skip that part.
    // A GCN needs them only on its wgmma kernel (DP <= 128 on bf16x3 / bf16): its fp32 kernel and its streaming plan tile by fixed blocks)
    std::vector<int>& counts = g->h_counts;
    std::vector<int>& reach = g->h_diff;   // reach[j] = the farthest node an edge whose lower end is node j touches
    const bool need_cuts = shape.precision == GGNN_PREC_FP32 ? shape.D <= 256 : shape.DP <= 128;
    counts.resize((size_t)V * T + 1);
    if (need_cuts) reach.resize((size_t)V + 1);
    std::vector<int64_t> type_base(T + 1, 0);   // position of every type's first message in the reference's type-major message order
    for (int t = 0; t < T; ++t) type_base[t + 1] = type_base[t] + num_edges[t];
    if (!count_edges(V, T, adj, type_base.data(), nth, counts.data(), need_cuts ? reach.data() : nullptr)) {
        int t, i;
        first_bad_edge(V, T, adj, num_edges, t, i);
        return g->fail(GGNN_ERANGE, "edge %d of type %d = (%d,%d) is out of range for %d nodes", i, t, adj[t][2 * i], adj[t][2 * i + 1], V);
    }
    lap("  edges pass 1", t_lap);
    std::vector<int> cuts;
    find_cuts(need_cuts ? reach.data() : nullptr, V, cuts);
    lap("validate+count", t_lap);
    std::vector<int> tile_start;
    int rc = build_plan(shape, V, weighted, cuts, p, tile_start, g->err, stream_weighted, msg_weighted);
    if (rc) return rc;
    p.M = M;
    const int ntiles = p.ntiles;
    lap("tile plan", t_lap);
    nth = std::max(1, std::min(nth, ntiles));
    // tile ranges of the threads for all later passes: tiles [tb[k], tb[k+1]), i.e. nodes [tile_start[tb[k]], tile_start[tb[k+1]])
    std::vector<int> tb(nth + 1);
    for (int k = 0; k <= nth; ++k) tb[k] = (int)((int64_t)ntiles * k / nth);
    // weighted streaming plan: the rows whose one message weighs other than 1.0f, which stream_rows makes virtual rows too (each such row
    // has one message, so no two writes meet).  Not on an all-virtual plan, whose rows with messages are all virtual whatever the weights
    std::vector<uint8_t> scaled_single;
    if (p.stream && weighted && !p.all_virtual) {
        scaled_single.assign((size_t)V * T, 0);
        for (int t = 0; t < T; ++t)
            for (int i = 0; i < num_edges[t]; ++i) {
                const size_t r = (size_t)adj[t][2 * i + 1] * T + t;
                if (counts[r + 1] == 1 && w[type_base[t] + i] != 1.0f) scaled_single[r] = 1;
            }
    }
    const uint8_t* scaled = scaled_single.empty() ? nullptr : scaled_single.data();
    // per-range totals: messages, and (streaming plan) virtual rows = (target, type) pairs with several messages, with their message count
    std::vector<int64_t> part_msgs(nth + 1, 0), part_nv(nth + 1, 0), part_nvm(nth + 1, 0);
#ifdef _OPENMP
#pragma omp parallel for schedule(static, 1) num_threads(nth) if (nth > 1)
#endif
    for (int k = 0; k < nth; ++k) {
        int64_t sm = 0, nv = 0, nvm = 0;
        const size_t k0 = (size_t)tile_start[tb[k]] * T, k1 = (size_t)tile_start[tb[k + 1]] * T;
        if (p.stream) {
            for (size_t r = k0; r < k1; ++r) {
                const int c = counts[r + 1];
                sm += c;
                if (c >= 2 || (scaled && scaled[r]) || (p.all_virtual && c == 1)) { ++nv; nvm += c; }
            }
        } else {
            for (size_t r = k0; r < k1; ++r) sm += counts[r + 1];
        }
        part_msgs[k + 1] = sm; part_nv[k + 1] = nv; part_nvm[k + 1] = nvm;
    }
    for (int k = 0; k < nth; ++k) { part_msgs[k + 1] += part_msgs[k]; part_nv[k + 1] += part_nv[k]; part_nvm[k + 1] += part_nvm[k]; }

    const size_t off = layout_image(shape, p, g->save, M, (int)part_nv[nth], part_nvm[nth]);
    CU_TRY(g, g->image.begin(off));
    g->bytes = off;
    const ImageView img = image_view(p, shape.use_att, g->image.ptr);
    for (const auto& pad : p.pads) memset(g->image.ptr + pad.first, 0, pad.second);
    lap("stage reserve", t_lap);

    // ---- pass 2, per thread over its tile range: exclusive scan of the (target, type) rows -> row_ptr, fill cursors, the tiles'
    // edge-type masks and the largest per-tile message count; then the stable fill -- every thread walks the
    // lists in the reference's order (type-major, then list order, sparse:124-129) and places the messages of ITS rows, so within a row
    // they stay in message order: this IS NumPy's stable argsort by target, tests pin it bit for bit; then (streaming plan) the gather
    // table and the virtual rows of its range, numbered from the range's offset; then in-degrees / denominators of its nodes.
    std::vector<int>& cursor = g->h_cursor;   // next free slot of every (target, type) row (its own array: the counts of a range's last
    cursor.resize((size_t)V * T + 1);         // row are read by one thread while the next range's thread already writes cursors)
    int max_tile_msgs = 0, max_tile_types = 0;
    img.row_ptr[0] = 0;
    if (img.vptr) img.vptr[0] = 0;
#ifdef _OPENMP
#pragma omp parallel for schedule(static, 1) num_threads(nth) if (nth > 1) reduction(max : max_tile_msgs, max_tile_types)
#endif
    for (int k = 0; k < nth; ++k) {
        int run = (int)part_msgs[k];
        for (int i = tb[k]; i < tb[k + 1]; ++i) {
            unsigned mask = 0;
            const int tile_first = run;
            for (size_t r = (size_t)tile_start[i] * T, rend = (size_t)tile_start[i + 1] * T; r < rend; r += T)
                for (int t = 0; t < T; ++t) {
                    const int c = counts[r + t + 1];
                    cursor[r + t] = run;
                    run += c;
                    img.row_ptr[r + t + 1] = run;
                    mask |= (unsigned)(c > 0) << t;
                }
            img.tile_mask[i] = mask;
            max_tile_msgs = std::max(max_tile_msgs, run - tile_first);
            max_tile_types = std::max(max_tile_types, __builtin_popcount(mask));
            img.tile_start[i] = tile_start[i];
        }
        if (k == nth - 1) img.tile_start[ntiles] = tile_start[ntiles];
    }
    p.max_tile_msgs = max_tile_msgs;
    p.max_tile_types = max_tile_types;
    lap("row sweep", t_lap);
#ifdef _OPENMP
#pragma omp parallel for schedule(static, 1) num_threads(nth) if (nth > 1)
#endif
    for (int k = 0; k < nth; ++k) {
        const int v0 = tile_start[tb[k]], v1 = tile_start[tb[k + 1]];
        int* const csr_src = img.src;
        int* const csr_msg = img.msg;
        for (int t = 0; t < T; ++t) {
            const int32_t* a = adj[t];
            const int ne = num_edges[t];
            const int mb = (int)type_base[t];
            if (nth == 1) {
                for (int i = 0; i < ne; ++i) {
                    const int slot = cursor[(size_t)a[2 * i + 1] * T + t]++;
                    csr_src[slot] = a[2 * i];
                    csr_msg[slot] = mb + i;
                }
            } else {
                int dummy_cursor = 0, dummy_src = 0, dummy_msg = 0;   // see pass 1: select, do not branch
                int* const cur = cursor.data();
                const unsigned span = (unsigned)(v1 - v0);
                for (int i = 0; i < ne; ++i) {
                    const int d = a[2 * i + 1];
                    const bool mine = (unsigned)(d - v0) < span;
                    int* pc = mine ? cur + ((size_t)d * T + t) : &dummy_cursor;
                    const int slot = *pc;
                    *pc = slot + 1;
                    *(mine ? csr_src + slot : &dummy_src) = a[2 * i];
                    *(mine ? csr_msg + slot : &dummy_msg) = mb + i;
                }
            }
        }
        if (img.slotw)   // the weights of this range's slots, in target-CSR order
            for (int64_t m = part_msgs[k]; m < part_msgs[k + 1]; ++m) img.slotw[m] = w ? w[csr_msg[m]] : 0.0f;
        if (img.pair) {   // the range's rows: no message -> -1, one -> its source, several -> virtual row; then the last tile's rows beyond V
            int vid = (int)part_nv[k], vm = (int)part_nvm[k];
            for (int i = tb[k]; i < tb[k + 1]; ++i) {
                img.tvp[i] = vid;
                const size_t rend = (size_t)tile_start[i + 1] * T, rpad = (size_t)(i + 1) * ts::TILE_M * T;
                stream_rows((size_t)tile_start[i] * T, rend, img.row_ptr, csr_src, img.slotw, p.all_virtual, img.pair, img.vptr, img.vsrc, img.vinfo,
                            img.vslot, vid, vm);
                for (size_t r = rend; r < rpad; ++r) img.pair[r] = -1;
            }
            if (k == nth - 1) img.tvp[ntiles] = vid;
        }
        if (v1 > v0) memcpy(img.indeg + (size_t)v0 * T, indeg + (size_t)v0 * T, sizeof(float) * (size_t)(v1 - v0) * T);
        fill_denominators(v0, v1, T, indeg, img.denom);
    }
    if (ntiles == 0) {
        img.tile_start[0] = 0;
        if (img.pair) { for (size_t r = 0; r < (size_t)ts::TILE_M * T; ++r) img.pair[r] = -1; img.tvp[0] = 0; }
    }
    lap("csr fill", t_lap);
    if (img.trow) fill_source_csr(V, T, adj, num_edges, M, img.msg, w, img.trow, img.ttgt, img.tslot, img.tslotw);
    lap("denom+masks+extra", t_lap);
    g->valid = true;
    return GGNN_OK;
}

int ggnn_free_prepared_graph(ggnn_prepared_graph* g) {
    if (!g) return GGNN_OK;
    if (g->image.use_cuda) {
        cudaSetDevice(g->shape.device);
        g->image.release();
    }
    delete g;
    return GGNN_OK;
}

const char* ggnn_prepared_graph_error(const ggnn_prepared_graph* g) { return g ? g->err.c_str() : "null prepared graph"; }

}  // extern "C"

// The model shape of a prepared graph or a dataset (`t` takes the error): with an engine `e`, which must be a `model` engine (the model of
// Config), the engine's, made current on this thread -- which may be a producer thread; without one, the shape `cfg` describes for a host
// of `num_sms` SMs with HOST_MAX_SMEM of shared memory each.
template <class Config>
static int model_shape_for(ErrorText* t, ModelShape& s, const ggnn_engine* e, const Config* cfg, int32_t num_sms, const char* fn) {
    constexpr int model = std::is_same<Config, ggnn_gcn_config>::value ? MODEL_GCN : MODEL_GGNN;
    if (e) {
        s = *e;
        if (e->model != model) return wrong_model(t, fn, e->model, model);
        if (cudaSetDevice(e->device) != cudaSuccess) return t->fail(GGNN_ECUDA, "cudaSetDevice(%d) failed", e->device);
        return GGNN_OK;
    }
    s = ModelShape();
    int rc;
    if constexpr (model == MODEL_GCN) rc = init_gcn_shape(s, cfg, t->err);
    else rc = init_model_shape(s, cfg, t->err);
    if (rc) return rc;
    s.num_sms = num_sms; s.max_smem = HOST_MAX_SMEM;
    return GGNN_OK;
}

// The prologue of the six prepare calls: reuse or allocate *inout and give it a model shape (model_shape_for).  With an engine, the save
// flag for save_for_backward = -1 is the engine's and the image is pinned on its device; without one, the image is plain memory.
template <class Config>
static int begin_prepare(ggnn_prepared_graph** inout, const ggnn_engine* e, const Config* cfg, int32_t num_sms, int32_t save_for_backward,
                         const char* fn) {
    if (!inout || (!e && (!cfg || num_sms <= 0))) return GGNN_EINVAL;
    ggnn_prepared_graph* g = *inout;
    if (!g) { g = new ggnn_prepared_graph(); *inout = g; }
    g->valid = false;
    g->image.use_cuda = e != nullptr;
    if (int rc = model_shape_for(g, g->shape, e, cfg, num_sms, fn)) return rc;
    g->save = e && save_for_backward < 0 ? e->save : save_for_backward != 0;   // a producer thread says what the batch will be used for
    return GGNN_OK;
}

// The plan fields the info calls of a prepared graph and a dataset batch report (image_bytes: the size of its image); null outputs are skipped.
static void report_plan(const BatchPlan& q, size_t bytes, int32_t* num_nodes, int64_t* num_messages, int32_t* num_tiles, int64_t* image_bytes,
                        int32_t* is_streaming, char* plan_text, int32_t plan_text_capacity, int32_t* max_tile_msgs, int32_t* max_tile_types) {
    if (num_nodes) *num_nodes = q.V;
    if (num_messages) *num_messages = q.M;
    if (num_tiles) *num_tiles = q.ntiles;
    if (image_bytes) *image_bytes = (int64_t)bytes;
    if (is_streaming) *is_streaming = q.stream ? 1 : 0;
    if (plan_text && plan_text_capacity > 0) snprintf(plan_text, (size_t)plan_text_capacity, "%s", q.plan_text.c_str());
    if (max_tile_msgs) *max_tile_msgs = q.max_tile_msgs;
    if (max_tile_types) *max_tile_types = q.max_tile_types;
}

// The common body of the ggnn_set_graph_* calls: build(&e->own_prep) prepares the batch in the engine's own prepared graph (the same two
// halves a caller can run on two threads), then the engine uploads it.
template <class Build>
static int set_graph_from_own_prep(ggnn_engine* e, ggnn_stream_t stream, Build build) {
    forget_batch(e);
    int rc = build(&e->own_prep);
    if (rc) { if (e->own_prep) e->err = e->own_prep->err; return rc; }
    return ggnn_set_graph_prepared(e, e->own_prep, stream);
}

extern "C" {

int ggnn_host_prepare_graph_sparse(const ggnn_config* cfg, int32_t num_sms, int32_t save_for_backward, int32_t V, const int32_t* const* adj,
                                   const int32_t* num_edges, const float* indeg, ggnn_prepared_graph** inout) {
    if (int rc = begin_prepare(inout, nullptr, cfg, num_sms, save_for_backward, __func__)) return rc;
    return build_sparse_image(*inout, V, adj, num_edges, indeg, false, nullptr);
}

int ggnn_prepared_graph_info(const ggnn_prepared_graph* g, int32_t* num_nodes, int64_t* num_messages, int32_t* num_tiles, int64_t* image_bytes,
                             int32_t* is_streaming, char* plan_text, int32_t plan_text_capacity) {
    if (!g || !g->valid) return GGNN_ESTATE;
    report_plan(g->plan, g->bytes, num_nodes, num_messages, num_tiles, image_bytes, is_streaming, plan_text, plan_text_capacity, nullptr, nullptr);
    return GGNN_OK;
}

int ggnn_prepared_graph_arrays(const ggnn_prepared_graph* g, int32_t* row_ptr, int32_t* src, int32_t* msg, int32_t* tile_start, float* denom,
                               int32_t* pair_src) {
    if (!g || !g->valid) return GGNN_ESTATE;
    const BatchPlan& q = g->plan;
    const ImageView img = image_view(q, g->shape.use_att, g->image.ptr);
    const size_t V = (size_t)q.V, T = (size_t)g->shape.T, M = q.dense_device ? 0 : (size_t)q.M;   // (a dense-device image lists none)
    if (row_ptr) memcpy(row_ptr, img.row_ptr, sizeof(int) * (V * T + 1));
    if (src && M) memcpy(src, img.src, sizeof(int) * M);
    if (msg && M) memcpy(msg, img.msg, sizeof(int) * M);
    if (tile_start) memcpy(tile_start, img.tile_start, sizeof(int) * (size_t)(q.ntiles + 1));
    if (denom && V) memcpy(denom, img.denom, sizeof(float) * V);
    if (pair_src && img.pair) memcpy(pair_src, img.pair, sizeof(int) * (size_t)std::max(q.ntiles, 1) * ts::TILE_M * T);
    return GGNN_OK;
}

int ggnn_prepared_graph_stream_tables(const ggnn_prepared_graph* g, int32_t* num_virtual_rows, int64_t* num_virtual_messages, int32_t* vrow_ptr,
                                      int32_t* vsrc, int32_t* vinfo, int32_t* vslot, int32_t* tile_vptr) {
    if (!g || !g->valid || !g->plan.stream) return GGNN_ESTATE;
    const BatchPlan& q = g->plan;
    const ImageView img = image_view(q, g->shape.use_att, g->image.ptr);
    if (vslot && !img.vslot) return GGNN_ESTATE;
    if (q.dense_device) {   // V*T virtual rows, whose image rows the dense aggregation kernel writes: no row lists a source
        const size_t nv = (size_t)q.ts_nv;
        if (num_virtual_rows) *num_virtual_rows = (int32_t)nv;
        if (num_virtual_messages) *num_virtual_messages = 0;
        if (vrow_ptr) memset(vrow_ptr, 0, sizeof(int) * (nv + 1));
        if (vinfo && nv) memset(vinfo, 0, sizeof(int) * 8 * nv);
        if (tile_vptr) memcpy(tile_vptr, img.tvp, sizeof(int) * (size_t)(q.ntiles + 1));
        return GGNN_OK;
    }
    const size_t nv = (size_t)q.ts_nv, nvm = (size_t)img.vptr[nv];
    if (num_virtual_rows) *num_virtual_rows = (int32_t)nv;
    if (num_virtual_messages) *num_virtual_messages = (int64_t)nvm;
    if (vrow_ptr) memcpy(vrow_ptr, img.vptr, sizeof(int) * (nv + 1));
    if (vsrc && nvm) memcpy(vsrc, img.vsrc, sizeof(int) * nvm);
    if (vinfo && nv) memcpy(vinfo, img.vinfo, sizeof(int) * 8 * nv);
    if (vslot && nv) memcpy(vslot, img.vslot, sizeof(int) * nv);
    if (tile_vptr) memcpy(tile_vptr, img.tvp, sizeof(int) * (size_t)(q.ntiles + 1));
    return GGNN_OK;
}

int ggnn_prepared_graph_tile_stats(const ggnn_prepared_graph* g, int32_t* max_tile_msgs, int32_t* max_tile_types) {
    if (!g || !g->valid) return GGNN_ESTATE;
    report_plan(g->plan, g->bytes, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, 0, max_tile_msgs, max_tile_types);
    return GGNN_OK;
}

int ggnn_prepared_graph_image(const ggnn_prepared_graph* g, void* dst, int64_t capacity) {
    if (!g || !g->valid || !dst) return GGNN_ESTATE;
    if (capacity < (int64_t)g->bytes) return GGNN_EINVAL;
    memcpy(dst, g->image.ptr, g->bytes);
    return GGNN_OK;
}

int ggnn_prepare_graph_sparse(const ggnn_engine* e, int32_t save_for_backward, int32_t V, const int32_t* const* adj, const int32_t* num_edges,
                              const float* indeg, ggnn_prepared_graph** inout) {
    if (int rc = begin_prepare<ggnn_config>(inout, e, nullptr, 0, save_for_backward, __func__)) return rc;
    return build_sparse_image(*inout, V, adj, num_edges, indeg, false, nullptr);
}

}  // extern "C"

// The host half of the two message-weighted prepare calls: the sparse builder with zero weight sections and the value-independent plan.
static int build_message_weighted_image(ggnn_prepared_graph* g, int32_t V, const int32_t* const* adj, const int32_t* num_edges, const float* indeg) {
    g->valid = false;
    if (g->shape.use_att)
        return g->fail(GGNN_EUNSUPPORTED, "message weights with propagation attention are not supported (the probabilities are the slot weights)");
    if (int rc = build_sparse_image(g, V, adj, num_edges, indeg, true, nullptr, true, true)) return rc;
    g->plan.plan_text += " [message-weighted]";
    return GGNN_OK;
}

extern "C" {

int ggnn_prepare_graph_sparse_weighted(const ggnn_engine* e, int32_t save_for_backward, int32_t V, const int32_t* const* adj,
                                       const int32_t* num_edges, const float* indeg, ggnn_prepared_graph** inout) {
    if (int rc = begin_prepare<ggnn_config>(inout, e, nullptr, 0, save_for_backward, __func__)) return rc;
    return build_message_weighted_image(*inout, V, adj, num_edges, indeg);
}

int ggnn_host_prepare_graph_sparse_weighted(const ggnn_config* cfg, int32_t num_sms, int32_t save_for_backward, int32_t V,
                                            const int32_t* const* adj, const int32_t* num_edges, const float* indeg, ggnn_prepared_graph** inout) {
    if (int rc = begin_prepare(inout, nullptr, cfg, num_sms, save_for_backward, __func__)) return rc;
    return build_message_weighted_image(*inout, V, adj, num_edges, indeg);
}

}  // extern "C"

// Whether a batch planned for model shape `q` (`what` names it) may be adopted by engine `e`; with save_for_backward on, the plan must carry
// the source-keyed CSR.
static int check_batch_shape(ggnn_engine* e, const ModelShape& q, const BatchPlan& p, const char* what) {
    if (q.model != e->model)
        return e->fail(GGNN_ESTATE, "the %s was built for a %s engine, this is a %s engine", what, q.model == MODEL_GCN ? "GCN" : "GGNN",
                       e->model == MODEL_GCN ? "GCN" : "GGNN");
    if (q.D != e->D || q.T != e->T || q.precision != e->precision || q.DP != e->DP || q.num_sms != e->num_sms || q.cell != e->cell || q.use_att != e->use_att ||
        q.wide_hidden != e->wide_hidden)
        return e->fail(GGNN_EINVAL, "the %s was built for a different engine configuration", what);
    if (e->save && !p.has_transpose)
        return e->fail(GGNN_ESTATE, "save_for_backward is on but the %s was prepared without it (the source-keyed CSR is built at prepare time)", what);
    return GGNN_OK;
}

// The typed view of the graph image in graph_buf (laid out by e's plan), then room for the states of the batch: the end of every graph upload.
static int bind_graph(ggnn_engine* e) {
    e->gd = image_view(*e, e->use_att, (char*)e->graph_buf.ptr);
    int rc = reserve_states(e);
    if (rc) return rc;
    e->graph_set = true;
    return GGNN_OK;
}

extern "C" {

int ggnn_set_graph_prepared(ggnn_engine* e, ggnn_prepared_graph* g, ggnn_stream_t stream) {
    if (!e) return GGNN_EINVAL;
    forget_batch(e);
    if (!g || !g->valid) return e->fail(GGNN_ESTATE, "the prepared graph is empty (its build failed or never ran)");
    if (int rc = check_batch_shape(e, g->shape, g->plan, "prepared graph")) return rc;
    CU_TRY(e, cudaSetDevice(e->device));
    static_cast<BatchPlan&>(*e) = g->plan;
    CU_TRY(e, e->graph_buf.reserve(g->bytes));
    e->graph_bytes = g->bytes;
    CU_TRY(e, g->image.upload(e->graph_buf.ptr, g->bytes, (cudaStream_t)stream));
    return bind_graph(e);
}

int ggnn_set_graph_sparse(ggnn_engine* e, int32_t V, const int32_t* const* adj, const int32_t* num_edges,
                          const float* indeg, ggnn_stream_t stream) {
    if (!e) return GGNN_EINVAL;
    GGNN_REQUIRE_MODEL(e, MODEL_GGNN);
    return set_graph_from_own_prep(e, stream, [&](ggnn_prepared_graph** g) { return ggnn_prepare_graph_sparse(e, -1, V, adj, num_edges, indeg, g); });
}


// The reference only ever feeds 0/1 adjacency (dense:30-36).  An adjacency IS a list of weighted messages: A_t.(h W_t + b_t) =
// (sum of A_t[i,j] h_j over the row's sources j) W_t + rowsum(A_t) b_t, which is the CSR path with one weight per message and in-degree =
// row sums (dense:107-112 adds the bias to every source row before A.m).  One scan of [b, T, v, v] -> per-type (source, target) lists and
// their matrix entries in the order (graph, target row, source column), and the fp32 row sums in column order (the zero entries add
// nothing); returns whether some nonzero entry differs from 1.  `weights` is filled, in the type-major message order, only then.
// The scan is a stream over b*T*v*v floats (4 MB at cfg3) of which ~99 % are zero: memory-bound on one core (~0.5 ms), so the
// graphs are split into contiguous ranges over a few OpenMP threads; every thread appends to its own per-type lists (order inside
// a range: graph, target row, source column) and the ranges are concatenated in order -- the result is the single-thread list.
static bool scan_dense(int T, int b, int v, const float* adjm, std::vector<std::vector<int32_t>>& lists, std::vector<float>& weights,
                       std::vector<float>& indeg) {
    const int V = b * v;
    lists.assign(T, std::vector<int32_t>());
    weights.clear();
    indeg.assign((size_t)std::max(V, 1) * T, 0.0f);
    int nthreads = 1;   // graph ranges scanned concurrently
    int team = 1;       // OpenMP team size: ONE size per process (the sparse builder's), used only if its region entry is cheap here
#ifdef _OPENMP
    team = b >= 16 ? host_team_size() : 1;
    if (team > 1 && !host_team_is_fast(team)) team = 1;
    nthreads = std::max(1, std::min(team, b / 8));
    if (const char* nt = getenv("GGNN_HOST_THREADS")) { nthreads = std::max(1, std::min(atoi(nt), std::max(b, 1))); team = nthreads; }
#endif
    std::vector<std::vector<std::vector<int32_t>>> part(nthreads, std::vector<std::vector<int32_t>>(T));
    std::vector<std::vector<std::vector<float>>> part_w(nthreads, std::vector<std::vector<float>>(T));
    std::vector<int> part_weighted(nthreads, 0);
    const int chunk = (b + nthreads - 1) / std::max(nthreads, 1);
#ifdef _OPENMP
#pragma omp parallel for schedule(static, 1) num_threads(team) if (team > 1)
#endif
    for (int k = 0; k < nthreads; ++k) {
        const int g0 = k * chunk, g1 = std::min(b, g0 + chunk);
        for (int t = 0; t < T; ++t) {
            part[k][t].reserve((size_t)std::max(g1 - g0, 0) * v * 3);
            part_w[k][t].reserve((size_t)std::max(g1 - g0, 0) * v * 3 / 2);
        }
        bool weighted = false;
        for (int g = g0; g < g1; ++g)
            for (int t = 0; t < T; ++t) {
                const float* m = adjm + ((size_t)g * T + t) * v * v;
                std::vector<int32_t>& lst = part[k][t];
                std::vector<float>& wl = part_w[k][t];
                for (int i = 0; i < v; ++i) {
                    const float* row = m + (size_t)i * v;
                    float sum = 0.0f;
                    auto visit = [&](int j) {
                        const float a = row[j];
                        if (a != 0.0f) {
                            lst.push_back(g * v + j);   // source
                            lst.push_back(g * v + i);   // target
                            wl.push_back(a);
                            sum += a;
                            weighted |= a != 1.0f;
                        }
                    };
                    int j = 0;
                    for (; j + 4 <= v; j += 4) {   // test 16 bytes at a time
                        uint64_t w0, w1;
                        memcpy(&w0, row + j, 8); memcpy(&w1, row + j + 2, 8);
                        if ((w0 | w1) == 0) continue;
                        visit(j); visit(j + 1); visit(j + 2); visit(j + 3);
                    }
                    for (; j < v; ++j) visit(j);
                    indeg[((size_t)g * v + i) * T + t] = sum;
                }
            }
        part_weighted[k] = weighted ? 1 : 0;
    }
    const bool weighted = std::find(part_weighted.begin(), part_weighted.end(), 1) != part_weighted.end();
    for (int t = 0; t < T; ++t) {
        size_t total = 0;
        for (int k = 0; k < nthreads; ++k) total += part[k][t].size();
        lists[t].resize(total);
        size_t off = 0;
        for (int k = 0; k < nthreads; ++k) {
            if (!part[k][t].empty()) memcpy(lists[t].data() + off, part[k][t].data(), part[k][t].size() * sizeof(int32_t));
            off += part[k][t].size();
            if (weighted) weights.insert(weights.end(), part_w[k][t].begin(), part_w[k][t].end());
        }
    }
    return weighted;
}

// How the dense entries take a weighted matrix: refused (the binary prepare calls), as weighted messages that run on the tile kernel or on
// fp32 (ggnn_set_graph_dense), or also on the streaming wgmma kernels above hidden 128 (the ..._dense_weighted entries).
enum DenseWeights { DENSE_BINARY_ONLY, DENSE_WEIGHTED, DENSE_WEIGHTED_STREAM };

// Host half of ggnn_set_graph_dense: the matrix is scanned to message lists for the CSR builder.  A 0/1 matrix builds the image of its
// edge lists; a weighted one (refused with GGNN_EUNSUPPORTED under DENSE_BINARY_ONLY) also carries its entries as slot weights.
static int build_dense_image(ggnn_prepared_graph* g, int32_t b, int32_t v, const float* adjm, DenseWeights mode) {
    g->valid = false;
    if (b < 0 || v <= 0 || (!adjm && b > 0)) return g->fail(GGNN_EINVAL, "null/negative argument");
    if (g->shape.use_att) return g->fail(GGNN_EUNSUPPORTED, "propagation attention exists only in the sparse model (sparse:170-196)");
    if (g->shape.cudnn_tc) return g->fail(GGNN_EUNSUPPORTED, "CudnnCompatibleGRUCell exists only in the sparse model (sparse:105-108)");
    const int T = g->shape.T;
    if ((int64_t)b * v > 0x7fffffff / std::max(T, 1)) return g->fail(GGNN_EUNSUPPORTED, "batch too large for int32 indexing");
    std::vector<std::vector<int32_t>> lists;
    std::vector<float> weights, indeg;
    const bool weighted = scan_dense(T, b, v, adjm, lists, weights, indeg);
    if (weighted && mode == DENSE_BINARY_ONLY)
        return g->fail(GGNN_EUNSUPPORTED, "the adjacency matrix is not 0/1: a weighted matrix is fed through ggnn_set_graph_dense");
    std::vector<const int32_t*> ptrs(T);
    std::vector<int32_t> counts(T);
    for (int t = 0; t < T; ++t) { ptrs[t] = lists[t].data(); counts[t] = (int32_t)(lists[t].size() / 2); }
    int rc = build_sparse_image(g, b * v, ptrs.data(), counts.data(), indeg.data(), weighted, weights.data(), mode == DENSE_WEIGHTED_STREAM);
    if (rc) return rc;
    g->plan.plan_text += weighted ? " [weighted dense adjacency -> weighted CSR]" : " [binary dense adjacency -> CSR]";
    return GGNN_OK;
}

int ggnn_prepare_graph_dense(const ggnn_engine* e, int32_t save_for_backward, int32_t b, int32_t v, const float* adjm, ggnn_prepared_graph** inout) {
    if (int rc = begin_prepare<ggnn_config>(inout, e, nullptr, 0, save_for_backward, __func__)) return rc;
    return build_dense_image(*inout, b, v, adjm, DENSE_BINARY_ONLY);
}

int ggnn_host_prepare_graph_dense(const ggnn_config* cfg, int32_t num_sms, int32_t save_for_backward, int32_t b, int32_t v, const float* adjm,
                                  ggnn_prepared_graph** inout) {
    if (int rc = begin_prepare(inout, nullptr, cfg, num_sms, save_for_backward, __func__)) return rc;
    return build_dense_image(*inout, b, v, adjm, DENSE_BINARY_ONLY);
}

int ggnn_host_prepare_graph_dense_weighted(const ggnn_config* cfg, int32_t num_sms, int32_t save_for_backward, int32_t b, int32_t v,
                                           const float* adjm, ggnn_prepared_graph** inout) {
    if (int rc = begin_prepare(inout, nullptr, cfg, num_sms, save_for_backward, __func__)) return rc;
    return build_dense_image(*inout, b, v, adjm, DENSE_WEIGHTED_STREAM);
}

int ggnn_prepare_graph_dense_weighted(const ggnn_engine* e, int32_t save_for_backward, int32_t b, int32_t v, const float* adjm,
                                      ggnn_prepared_graph** inout) {
    if (int rc = begin_prepare<ggnn_config>(inout, e, nullptr, 0, save_for_backward, __func__)) return rc;
    return build_dense_image(*inout, b, v, adjm, DENSE_WEIGHTED_STREAM);
}

}  // extern "C"

// Host half of ggnn_prepare_graph_dense_device: the plan and the image of b graphs of v rows, from (b, v) and the model shape alone.  The
// tensor-core precisions take the streaming plan at every hidden size (fixed 128-row tiles, every tile's mask has all T types, every
// (row, type) pair is virtual row row*T + type, no tile lists virtual-row sources); fp32 takes the per-timestep path at every hidden size.
// The image's CSR sections are empty and its in-degree section zero until ggnn_set_message_weights writes the row sums.  One thread: the
// work is a few integers per row.
static int build_dense_device_image(ggnn_prepared_graph* g, int32_t b, int32_t v) {
    const ModelShape& shape = g->shape;
    BatchPlan& p = g->plan;
    g->valid = false;
    if (b < 0 || v <= 0) return g->fail(GGNN_EINVAL, "null/negative argument");
    if (shape.use_att) return g->fail(GGNN_EUNSUPPORTED, "propagation attention exists only in the sparse model (sparse:170-196)");
    if (shape.cudnn_tc) return g->fail(GGNN_EUNSUPPORTED, "CudnnCompatibleGRUCell exists only in the sparse model (sparse:105-108)");
    if (shape.use_avg)
        return g->fail(GGNN_EUNSUPPORTED, "use_edge_msg_avg_aggregation with a device adjacency is not supported (its denominator would depend on A)");
    const int T = shape.T;
    const int64_t V64 = (int64_t)b * v;
    if (V64 * T + 1 > 0x7fffffff) return g->fail(GGNN_EUNSUPPORTED, "batch too large for int32 indexing");
    const int V = (int)V64;
    p = BatchPlan();
    p.V = V;
    p.msg_weighted = p.dense_device = true;
    p.dense_b = b; p.dense_v = v;
    std::vector<int> tile_start;
    fixed_tiles(V, ts::TILE_M, tile_start);
    p.ntiles = (int)tile_start.size() - 1;
    char buf[320];
    if (shape.precision != GGNN_PREC_FP32) {
        p.stream = true; p.variant = 3;
        for (int i = 0; i < 2; ++i) { p.ts_nblk[i] = ((i + 1) * shape.DP + ts::MMA_N - 1) / ts::MMA_N; p.ts_nc[i] = ts::MMA_N; }
        snprintf(buf, sizeof buf, "wgmma-%s STREAM(4 launches per step: dense aggregation, gather-GEMM, gate GEMM, candidate GEMM) tiles=%d DP=%d "
                 "N-blocks agg/cand=%dx%d gate=%dx%d [dense adjacency on the device]", shape.precision == GGNN_PREC_BF16X3 ? "bf16x3" : "bf16",
                 p.ntiles, shape.DP, p.ts_nblk[0], p.ts_nc[0], p.ts_nblk[1], p.ts_nc[1]);
    } else {
        p.stepwise = true;
        snprintf(buf, sizeof buf, "fp32-stepwise%s (%d launches per step) V=%d D=%d T=%d [dense adjacency on the device]",
                 shape.cell == CELL_CUDNN_GRU ? "+cudnn-gru" : "", stepwise_launches(shape), V, shape.D, T);
    }
    p.plan_text = buf;
    const size_t off = layout_image(shape, p, g->save, 0, 0, 0);
    p.M = V64 * T * v;
    if (p.stream) p.ts_nv = V * T;
    CU_TRY(g, g->image.begin(off));
    g->bytes = off;
    const ImageView img = image_view(p, shape.use_att, g->image.ptr);
    for (const auto& pad : p.pads) memset(g->image.ptr + pad.first, 0, pad.second);
    const size_t VT = (size_t)V * T;
    memset(img.row_ptr, 0, sizeof(int) * (VT + 1));
    memset(img.indeg, 0, sizeof(float) * VT);
    fill_denominators(0, V, T, img.indeg, img.denom);
    const unsigned all_types = T == 32 ? 0xffffffffu : (1u << T) - 1u;
    for (int i = 0; i <= p.ntiles; ++i) img.tile_start[i] = tile_start[i];
    for (int i = 0; i < p.ntiles; ++i) img.tile_mask[i] = all_types;
    if (img.trow) memset(img.trow, 0, sizeof(int) * (VT + 1));
    if (img.pair) {
        const size_t rows = (size_t)std::max(p.ntiles, 1) * ts::TILE_M * T;
        for (size_t r = 0; r < rows; ++r) img.pair[r] = r < VT ? -(2 + (int)r) : -1;
        img.vptr[0] = 0;
        for (int i = 0; i <= p.ntiles; ++i) img.tvp[i] = 0;
    }
    g->valid = true;
    return GGNN_OK;
}

extern "C" {

int ggnn_prepare_graph_dense_device(const ggnn_engine* e, int32_t save_for_backward, int32_t b, int32_t v, ggnn_prepared_graph** inout) {
    if (int rc = begin_prepare<ggnn_config>(inout, e, nullptr, 0, save_for_backward, __func__)) return rc;
    return build_dense_device_image(*inout, b, v);
}

int ggnn_host_prepare_graph_dense_device(const ggnn_config* cfg, int32_t num_sms, int32_t save_for_backward, int32_t b, int32_t v,
                                         ggnn_prepared_graph** inout) {
    if (int rc = begin_prepare(inout, nullptr, cfg, num_sms, save_for_backward, __func__)) return rc;
    return build_dense_device_image(*inout, b, v);
}

int ggnn_set_graph_dense(ggnn_engine* e, int32_t b, int32_t v, const float* adjm, ggnn_stream_t stream) {
    if (!e) return GGNN_EINVAL;
    GGNN_REQUIRE_MODEL(e, MODEL_GGNN);
    return set_graph_from_own_prep(e, stream, [&](ggnn_prepared_graph** g) {
        if (int rc = begin_prepare<ggnn_config>(g, e, nullptr, 0, -1, "ggnn_set_graph_dense")) return rc;
        return build_dense_image(*g, b, v, adjm, DENSE_WEIGHTED);
    });
}

int ggnn_set_graph_dense_weighted(ggnn_engine* e, int32_t b, int32_t v, const float* adjm, ggnn_stream_t stream) {
    if (!e) return GGNN_EINVAL;
    GGNN_REQUIRE_MODEL(e, MODEL_GGNN);
    return set_graph_from_own_prep(e, stream, [&](ggnn_prepared_graph** g) {
        if (int rc = begin_prepare<ggnn_config>(g, e, nullptr, 0, -1, "ggnn_set_graph_dense_weighted")) return rc;
        return build_dense_image(*g, b, v, adjm, DENSE_WEIGHTED_STREAM);
    });
}

// ------------------------------------------------------------------------------------------ forward drivers (host)
// fp32 CUDA-core path (ggnn_fwd_ffma.cuh); the only one with propagation attention and CudnnCompatibleGRUCell.
static int forward_ffma(ggnn_engine* e, const float* h0, float* h_out, cudaStream_t st) {
    if (e->use_att)
        CU_TRY(e, e->att_buf.reserve(sizeof(float) * (size_t)std::max<int64_t>(e->M, 1) * (size_t)(e->save ? std::max(e->total_steps, 1) : 1)));
    FwdParams p;
    fill_common_params(e, p, h0, h_out);
    p.use_att = e->use_att; p.att = (float*)e->att_buf.ptr; p.att_stride = e->save ? (size_t)std::max<int64_t>(e->M, 1) : 0;
    for (int l = 0; l < e->L; ++l) {
        LayerDev& ld = p.layer[l];
        ld.edge_w = e->w[l].edge_weights; ld.edge_b = e->w[l].edge_biases;
        ld.gate_k = e->w[l].gate_kernel; ld.gate_b = e->w[l].gate_bias;
        ld.cand_k = e->w[l].cand_kernel; ld.cand_b = e->w[l].cand_bias;
        ld.att_w = e->use_att ? e->w[l].edge_type_attention_weights : nullptr;
        ld.cand_hb = e->cell == CELL_CUDNN_GRU ? e->w[l].cand_hidden_bias : nullptr;
    }
    FwdKernel k = pick_fwd_kernel(e->variant, e->nb1, e->local);
    if (!k) return e->fail(GGNN_EUNSUPPORTED, "no kernel for variant=%d nb1=%d", e->variant, e->nb1);
    const size_t smem = fwd_smem_bytes(e->variant, e->nb1, e->D, e->T);
    CU_TRY(e, cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    return launch_steps(e, p, st, [&](const FwdParams& q) { k<<<e->ntiles, 256, smem, st>>>(q); });
}

// The per-timestep fp32 path (ggnn_fwd_step.cuh) multiplies with bwd::gemm_nt_kernel, C = A . B^T: it reads transposed fp32 copies of the
// weights, per layer the T edge matrices, the gate kernel and the candidate kernel.  Made again when the weights changed since (the
// weights generation), at no other time.
static int step_prepare_weights(ggnn_engine* e, cudaStream_t st) {
    const size_t D = e->D, T = e->T;
    WeightTiles& c = e->step_wt;
    size_t off = 0;
    for (int l = 0; l < e->L; ++l) {
        const size_t rows = D * (e->nres[l] + 2);
        c.off_edge[l] = off; off += T * D * D;
        c.off_gate[l] = off; off += e->cell != CELL_RNN ? rows * 2 * D : 0;
        c.off_cand[l] = off; off += rows * D;
    }
    bool retile = false;
    CU_TRY(e, c.reserve(off * sizeof(float), 0, 0, e->weights_gen, retile));
    if (!retile) return GGNN_OK;
    float* base = (float*)c.buf.ptr;
    auto transpose = [&](const float* W, size_t out, int rows, int cols, int batch) {
        step::transpose_kernel<<<dim3((cols + 31) / 32, (rows + 31) / 32, batch), dim3(32, 8), 0, st>>>(W, base + out, rows, cols);
        ++e->last_launches;
    };
    for (int l = 0; l < e->L; ++l) {
        const int rows = (int)D * (e->nres[l] + 2);
        transpose(e->w[l].edge_weights, c.off_edge[l], (int)D, (int)D, (int)T);
        if (e->cell != CELL_RNN) transpose(e->w[l].gate_kernel, c.off_gate[l], rows, 2 * (int)D, 1);
        transpose(e->w[l].cand_kernel, c.off_cand[l], rows, (int)D, 1);
    }
    CU_TRY(e, cudaGetLastError());
    c.gen = e->weights_gen;
    return GGNN_OK;
}

static int forward_stepwise(ggnn_engine* e, const float* h0, float* h_out, cudaStream_t st) {
    using namespace ggnn::bwd;
    if (int rc = step_prepare_weights(e, st)) return rc;
    const int V = e->V, D = e->D, T = e->T;
    const bool gru = e->cell != CELL_RNN, cudnn = e->cell == CELL_CUDNN_GRU;
    int maxres = 0;
    for (int l = 0; l < e->L; ++l) maxres = std::max(maxres, e->nres[l]);
    const size_t vd = (size_t)V * D;
    // scratch: gathered messages [V, T*D] | cell input row [V, D*(R+2)] | gates [V, 2D] | candidate GEMM [V, D] | q GEMM [V, D]
    size_t off = 0;
    auto take = [&](size_t floats) { size_t o = off; off = align_up(off + floats * sizeof(float), 256); return o; };
    const size_t o_at = take(vd * T), o_x = take(vd * (maxres + 2)), o_g = take(gru ? 2 * vd : 0), o_c = take(vd), o_q = take(cudnn ? vd : 0);
    CU_TRY(e, e->step_buf.reserve(off));
    if (e->use_att)
        CU_TRY(e, e->att_buf.reserve(sizeof(float) * (size_t)std::max<int64_t>(e->M, 1) * (size_t)(e->save ? std::max(e->total_steps, 1) : 1)));
    char* sb = (char*)e->step_buf.ptr;
    float *At = (float*)(sb + o_at), *X = (float*)(sb + o_x), *Gb = (float*)(sb + o_g), *Cb = (float*)(sb + o_c), *Qb = (float*)(sb + o_q);
    const float* wt = (const float*)e->step_wt.buf.ptr;
    const ImageView& gd = e->gd;
    const long long n = (long long)vd;
    const int eb = (int)std::min<long long>((n + 255) / 256, 4096), nodes_blocks = (V + 7) / 8;
    auto gemm = [&](const float* A, int lda, int a_stride, const float* B, int ldb, int b_stride, int nseg, float* C, int ldc, int N, int K) {
        gemm_nt_kernel<false><<<dim3((N + NT_BN - 1) / NT_BN, (V + NT_BM - 1) / NT_BM), 128, 0, st>>>(A, lda, a_stride, B, ldb, b_stride, nseg, C,
                                                                                                    ldc, V, N, K);
    };
    FwdParams p;   // the layer states and the step ping-pong of launch_steps
    fill_common_params(e, p, h0, h_out);
    cudaError_t copy_st = cudaSuccess;
    const int rc = launch_steps(e, p, st, [&](const FwdParams& q) {
        const int l = q.g_layer, R = e->nres[l], ldx = D * (R + 2), gs = e->step_base[l] + q.g_step;
        const ggnn_layer_weights& w = e->w[l];
        const float* h = q.g_in;
        const SaveDev sv = saved_step(e, gs);
        // the residual inputs are node_states_per_layer entries before this layer: fixed for all of its steps
        if (q.g_step == 0)
            for (int i = 0; i < R && copy_st == cudaSuccess; ++i)
                copy_st = cudaMemcpy2DAsync(X + (size_t)i * D, sizeof(float) * ldx, q.state[e->res[l][i]], sizeof(float) * D, sizeof(float) * D, V,
                                            cudaMemcpyDeviceToDevice, st);
        const float* msg_w = q.slot_w;
        if (e->use_att) {
            float* att = (float*)e->att_buf.ptr + (size_t)gs * (e->save ? (size_t)std::max<int64_t>(e->M, 1) : 0);
            step::attention_kernel<<<nodes_blocks, 256, 0, st>>>(gd.row_ptr, gd.src, h, w.edge_type_attention_weights, att, V, D, T);
            msg_w = att;
        }
        if (e->dense_device) {   // X = [A_0 h | .. | A_{T-1} h] where the gather would write it
            dense_apply_launch(e, st, false, (const float*)e->dense_adj.ptr, h, At, nullptr);
        } else {
            const GatherJob gj{gd.row_ptr, gd.src, h, At, msg_w, nullptr};
            csr_gather_all_kernel<<<dim3(nodes_blocks, 1), 256, 0, st>>>(gj, gj, V, D, T);
        }
        gemm(At, T * D, D, wt + e->step_wt.off_edge[l], D, D * D, T, X + (size_t)R * D, ldx, D, D);
        step::agg_epilogue_kernel<<<eb, 256, 0, st>>>(X, ldx, R * D, (R + 1) * D, h, e->use_bias ? w.edge_biases : nullptr, gd.indeg,
                                                      e->use_avg ? gd.denom : nullptr, sv.agg, sv.h_in, n, D, T);
        if (gru) {
            gemm(X, ldx, 0, wt + e->step_wt.off_gate[l], ldx, 0, 1, Gb, 2 * D, 2 * D, ldx);
            step::gate_epilogue_kernel<<<eb, 256, 0, st>>>(Gb, w.gate_bias, h, cudnn ? nullptr : X, ldx, (R + 1) * D, sv.r, sv.u, n, D);
            if (cudnn) gemm(h, D, 0, wt + e->step_wt.off_cand[l] + (size_t)(R + 1) * D, ldx, 0, 1, Qb, D, D, D);
        }
        // CudnnCompatibleGRUCell: the candidate's first D*(R+1) kernel rows see [res.., agg]; its recurrent rows went into q
        gemm(X, ldx, 0, wt + e->step_wt.off_cand[l], ldx, 0, 1, Cb, D, D, cudnn ? ldx - D : ldx);
        step::update_kernel<<<eb, 256, 0, st>>>(Cb, w.cand_bias, gru ? Gb : nullptr, cudnn ? Qb : nullptr, w.cand_hidden_bias, h, q.g_out, sv.c,
                                                sv.q, e->act, e->drop_keep, e->drop_seed, gs, V, n, D);
        e->last_launches += stepwise_launches(*e) - 1;   // launch_steps counts one per step
    });
    if (copy_st != cudaSuccess) return e->fail(GGNN_ECUDA, "residual input copy failed: %s", cudaGetErrorString(copy_st));
    return rc;
}

// The tile-local wgmma layout (ggnn_fwd_tc.cuh): per layer the T edge blocks, then the gate and the candidate kernel in nres + 2 input
// segments.  A GCN layer is one edge block.
static int tc_prepare_weights(ggnn_engine* e, cudaStream_t st) {
    const bool gcn = e->model == MODEL_GCN;
    const int D = e->D, DP = e->DP, T = e->T, NKS = DP / 16;
    WeightTiles& c = e->tc_tiles;
    size_t off = 0;
    for (int l = 0; l < e->L; ++l) {
        const int nseg = e->nres[l] + 2;
        c.off_edge[l] = off; off += (size_t)T * NKS * 64 * DP;
        if (gcn) continue;
        c.off_gate[l] = off; off += (size_t)nseg * NKS * 128 * DP;
        c.off_cand[l] = off; off += (size_t)nseg * NKS * 64 * DP;
    }
    bool retile = false;
    CU_TRY(e, c.reserve(off, 0, 0, e->weights_gen, retile));
    if (!retile) return GGNN_OK;
    uint8_t* base = (uint8_t*)c.buf.ptr;
    auto launch = [&](const float* W, size_t out, int segs, int blks, int src_ld) {
        const long long total = (long long)segs * NKS * 2 * blks * DP;
        const int blocks = (int)std::min<long long>((total + 255) / 256, 1024);
        tc::ggnn_tile_weights_kernel<<<blocks, 256, 0, st>>>(W, base + out, D, DP, segs, blks, src_ld, 0);
        ++e->last_launches;
    };
    for (int l = 0; l < e->L; ++l) {
        const int nseg = e->nres[l] + 2;
        if (gcn) { launch(e->gcn_w[l].kernel, c.off_edge[l], 1, 1, D); continue; }
        launch(e->w[l].edge_weights, c.off_edge[l], T, 1, D);
        if (e->cell == CELL_GRU) launch(e->w[l].gate_kernel, c.off_gate[l], nseg, 2, 2 * D);
        launch(e->w[l].cand_kernel, c.off_cand[l], nseg, 1, D);
    }
    CU_TRY(e, cudaGetLastError());
    c.gen = e->weights_gen;
    return GGNN_OK;
}

static int forward_tc(ggnn_engine* e, const float* h0, float* h_out, cudaStream_t st) {
    const int DP = e->DP;
    int rc = tc_prepare_weights(e, st);
    if (rc) return rc;
    bool any_res = false;
    for (int l = 0; l < e->L; ++l) any_res |= e->nres[l] > 0;
    if (any_res) CU_TRY(e, e->tc_respre.reserve((size_t)e->ntiles * tc::TILE_M * 3 * DP * sizeof(float)));
    tc::TcParams p;
    fill_common_params(e, p, h0, h_out);
    p.DP = DP;
    p.nparts = e->precision == GGNN_PREC_BF16X3 ? 3 : 1;
    p.kgs = e->tc_kgs;
    const size_t avail = e->max_smem > 1024 ? e->max_smem - 1024 : 0;
    // the shared-memory plan (ggnn_tc_smem.h): the CSR slice of tile-local graphs when it fits beside the two ring slots a worker holds
    // at once (DP 128 with 128-row tiles has room for two slots only without it), the number of gather tiles (GGNN_TC_GATHER_TILES=<n>
    // overrides the edge types per tile, clamped to what fits), the ring depth
    static_assert(tc::TILE_M == 128, "ggnn_tc_smem.h sizes the CSR slice for 128-row tiles");
    int ng_request = 0;
    if (const char* g = getenv("GGNN_TC_GATHER_TILES")) ng_request = std::max(2, atoi(g));
    const TcSmemPlan sp = tc_smem_plan(DP, p.kgs, e->T, e->local, !e->weighted, e->use_bias != 0, e->max_tile_msgs,
                                       e->max_tile_types, avail, tc::MAX_STAGES, ng_request);
    if (sp.nstages < 2) return e->fail(GGNN_EUNSUPPORTED, "not enough shared memory for the tensor-core tile (DP=%d)", DP);
    p.csr_cache = sp.csr_cache;
    p.csr_cap_msgs = sp.csr_cap_msgs;
    p.ngather = sp.ngather;
    p.nstages = sp.nstages;
    const size_t smem = sp.smem;
    const WeightTiles& wt = e->tc_tiles;
    const uint8_t* wb = (const uint8_t*)wt.buf.ptr;
    for (int l = 0; l < e->L; ++l) {
        tc::TcLayer& ld = p.layer[l];
        ld.w_edge = wb + wt.off_edge[l]; ld.w_gate = wb + wt.off_gate[l]; ld.w_cand = wb + wt.off_cand[l];
        ld.edge_b = e->w[l].edge_biases; ld.gate_b = e->w[l].gate_bias; ld.cand_b = e->w[l].cand_bias;
    }
    p.res_pre = (float*)e->tc_respre.ptr;
    p.error_flag = (int*)e->err_flag.ptr;
    // the wgmma N of a warpgroup's columns is an instruction immediate: one kernel per padded hidden size, layout (compact tiles
    // split the columns four ways, 128-row tiles two ways) and precision (bf16x3 / bf16: the MMA path is straight-line code)
    void (*kern)(tc::TcParams) = nullptr;
    const bool compact = e->tc_kgs == 1024, x3 = p.nparts == 3;
    switch (DP / 2) {
#define GGNN_TC_LAYOUTS(nh, x3)                                                                                                       \
    (!e->local ? tc::ggnn_fwd_tc_kernel<false, nh, false, x3>                                                                         \
               : (compact ? tc::ggnn_fwd_tc_kernel<true, nh, true, x3> : tc::ggnn_fwd_tc_kernel<true, nh, false, x3>))
#define GGNN_TC_CASE(nh)                                                                                                              \
    case nh:                                                                                                                          \
        kern = x3 ? GGNN_TC_LAYOUTS(nh, true) : GGNN_TC_LAYOUTS(nh, false);                                                           \
        break;
        GGNN_TC_CASE(8) GGNN_TC_CASE(16) GGNN_TC_CASE(24) GGNN_TC_CASE(32) GGNN_TC_CASE(40) GGNN_TC_CASE(48) GGNN_TC_CASE(56) GGNN_TC_CASE(64)
#undef GGNN_TC_CASE
#undef GGNN_TC_LAYOUTS
        default: return e->fail(GGNN_EUNSUPPORTED, "no tile-local tensor-core kernel for DP=%d", DP);
    }
    CU_TRY(e, cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    const int nthreads = e->local && compact ? tc::NTHREADS<true> : tc::NTHREADS<false>;
    return launch_steps(e, p, st, [&](const tc::TcParams& q) { kern<<<e->ntiles, nthreads, smem, st>>>(q); });
}

// ------------------------------------------------------------------------------------------ streaming tensor-core path (host)
// The streaming layout (ggnn_fwd_stream.cuh): per layer, in N blocks of ts_nc columns, the T edge blocks, the gate and the candidate kernel.
// CudnnCompatibleGRUCell splits the candidate kernel in two: K_in (its first (R+1) D rows, the [res.. | agg] segments) and, at off_hproj,
// K_hid (its last D rows, one segment).  A GCN layer is one segment: W_l at off_edge.
static int ts_prepare_weights(ggnn_engine* e, cudaStream_t st) {
    const int D = e->D, DP = e->DP, T = e->T, NKS = DP / 16;
    const int nc0 = e->ts_nc[0], nb0 = e->ts_nblk[0], nc1 = e->ts_nc[1], nb1 = e->ts_nblk[1];
    const bool cudnn = e->cell == CELL_CUDNN_GRU, gcn = e->model == MODEL_GCN;
    WeightTiles& c = e->ts_tiles;
    size_t off = 0;
    for (int l = 0; l < e->L; ++l) {
        if (gcn) { c.off_edge[l] = off; off += (size_t)nb0 * NKS * 64 * nc0; continue; }
        const int nseg = e->nres[l] + 2, ncand = cudnn ? nseg - 1 : nseg;
        c.off_edge[l] = off; off += (size_t)nb0 * T * NKS * 64 * nc0;
        c.off_gate[l] = off; off += (size_t)nb1 * nseg * NKS * 64 * nc1;
        c.off_cand[l] = off; off += (size_t)nb0 * ncand * NKS * 64 * nc0;
        c.off_hproj[l] = off; off += cudnn ? (size_t)nb0 * NKS * 64 * nc0 : 0;
    }
    bool retile = false;
    CU_TRY(e, c.reserve(off, nc0, nc1, e->weights_gen, retile));
    if (!retile) return GGNN_OK;
    uint8_t* base = (uint8_t*)c.buf.ptr;
    for (int l = 0; l < e->L; ++l) {
        const int nseg = e->nres[l] + 2;
        auto launch = [&](const float* W, uint8_t* out, int segs, int ncolblk, int src_ld, int NC, int nblk) {
            const long long total = (long long)nblk * segs * NKS * 2 * NC;
            const int blocks = (int)std::min<long long>((total + 255) / 256, 2048);
            ts::ggnn_tile_weights_stream_kernel<<<blocks, 256, 0, st>>>(W, out, D, DP, segs, ncolblk, src_ld, NC, nblk);
            ++e->last_launches;
        };
        if (gcn) { launch(e->gcn_w[l].kernel, base + c.off_edge[l], 1, 1, D, nc0, nb0); continue; }
        launch(e->w[l].edge_weights, base + c.off_edge[l], T, 1, D, nc0, nb0);
        if (e->cell != CELL_RNN) launch(e->w[l].gate_kernel, base + c.off_gate[l], nseg, 2, 2 * D, nc1, nb1);
        if (cudnn) {
            launch(e->w[l].cand_kernel, base + c.off_cand[l], nseg - 1, 1, D, nc0, nb0);
            launch(e->w[l].cand_kernel + (size_t)(nseg - 1) * D * D, base + c.off_hproj[l], 1, 1, D, nc0, nb0);
        } else {
            launch(e->w[l].cand_kernel, base + c.off_cand[l], nseg, 1, D, nc0, nb0);
        }
    }
    CU_TRY(e, cudaGetLastError());
    c.gen = e->weights_gen;
    return GGNN_OK;
}

// The ring of the streaming kernels and the two instances a forward launches (the GGNN's and the GCN's streaming forward).  A ring stage
// carries KS K-steps, the largest of 4, 2, 1 that divides the K-steps of a segment (the producer thread pays several hundred cycles per bulk
// copy whatever its size; KS is a template parameter so that a stage's MMAs are straight-line code); GGNN_TS_KSTEPS caps it and
// GGNN_TS_STAGES caps the ring depth.  `edge` is the gather-fed instance, `fed` the TMA-fed one.
struct StreamLaunch {
    int KS = 4;
    int max_ns = ts::MAX_NS;   // the kernel has MAX_NS stage barriers
    void (*edge)(ts::StreamParams) = nullptr;
    void (*fed)(ts::StreamParams) = nullptr;
    size_t stage_bytes(int NC) const { return (size_t)KS * ((size_t)ts::A_STAGE_B + 64 * (size_t)NC); }
    int stages(int NC, size_t budget) const { return (int)std::min<size_t>((size_t)max_ns, budget / stage_bytes(NC)); }
    size_t smem(int NC, int ns, size_t extra) const { return (size_t)1024 + ts::ring_bytes(ns, stage_bytes(NC)) + extra; }
};

static StreamLaunch stream_launch(const ggnn_engine* e) {
    StreamLaunch k;
    const int NKS = e->DP / 16;
    const char* env_ks = getenv("GGNN_TS_KSTEPS");
    const char* env_ns = getenv("GGNN_TS_STAGES");
    if (env_ks) k.KS = atoi(env_ks) >= 4 ? 4 : (atoi(env_ks) >= 2 ? 2 : 1);
    while (NKS % k.KS) k.KS /= 2;
    if (env_ns) k.max_ns = std::max(0, std::min(atoi(env_ns), ts::MAX_NS));
    const bool x3 = e->precision == GGNN_PREC_BF16X3;
    const int KS = k.KS;
#define GGNN_TS_PICK(X, K)                              \
    if (x3 == X && KS == K) {                           \
        k.edge = ts::ggnn_stream_kernel<true, X, K>;    \
        k.fed = ts::ggnn_stream_kernel<false, X, K>;    \
    }
    GGNN_TS_PICK(true, 4) GGNN_TS_PICK(true, 2) GGNN_TS_PICK(true, 1) GGNN_TS_PICK(false, 4) GGNN_TS_PICK(false, 2) GGNN_TS_PICK(false, 1)
#undef GGNN_TS_PICK
    return k;
}

static int forward_stream(ggnn_engine* e, const float* h0, float* h_out, cudaStream_t st) {
    const int D = e->D, DP = e->DP, T = e->T, L = e->L, V = e->V, NKS = DP / 16;
    const int ntiles = e->ntiles;
    int rc = ts_prepare_weights(e, st);
    if (rc) return rc;
    const size_t img_b = (size_t)ntiles * NKS * ts::A_STAGE_B;   // one operand image == one chunk-major fp32 copy, in bytes
    // images: node_states_per_layer, two step temporaries, agg, r*h (CudnnCompatibleGRUCell: the same bytes hold r, then r*q, chunk-major fp32)
    const int n_img = L + 1 + 4;
    const int n_chk = L + 1 + 3;    // chunk-major fp32: node_states_per_layer, two step temporaries, u
    CU_TRY(e, e->ts_images.reserve(img_b * (n_img + n_chk)));
    uint8_t* ib = (uint8_t*)e->ts_images.ptr;
    auto img_state = [&](int l) { return ib + (size_t)l * img_b; };
    uint8_t* img_tmp[2] = {ib + (size_t)(L + 1) * img_b, ib + (size_t)(L + 2) * img_b};
    uint8_t* img_agg = ib + (size_t)(L + 3) * img_b;
    uint8_t* img_rh = ib + (size_t)(L + 4) * img_b;
    uint8_t* cb = ib + (size_t)n_img * img_b;
    auto chk_state = [&](int l) { return (float*)(cb + (size_t)l * img_b); };
    float* chk_tmp[2] = {(float*)(cb + (size_t)(L + 1) * img_b), (float*)(cb + (size_t)(L + 2) * img_b)};
    float* u_chk = (float*)(cb + (size_t)(L + 3) * img_b);
    const size_t vd_bytes = (size_t)V * D * sizeof(float);
    const bool gated = e->cell != CELL_RNN, cudnn = e->cell == CELL_CUDNN_GRU;
    float* rq_chk = (float*)img_rh;   // CudnnCompatibleGRUCell: r (gate launch), then r*q (hidden-projection launch)
    const ImageView& gd = e->gd;

    // shared-memory budgets
    const size_t avail = (e->max_smem > 2048 ? e->max_smem - 2048 : 0);
    const size_t csr_b = (size_t)ts::TILE_M * T * 4;   // the tile's (target, type) -> source table
    CU_TRY(e, e->ts_virt.reserve((size_t)((e->ts_nv + ts::TILE_M - 1) / ts::TILE_M + 1) * NKS * ts::A_STAGE_B));
    const size_t att_stride = e->save ? (size_t)std::max<int64_t>(e->M, 1) : 0;   // attention probabilities of a step, [steps][M] when saving
    if (e->use_att) CU_TRY(e, e->att_buf.reserve(sizeof(float) * (size_t)std::max<int64_t>(e->M, 1) * (size_t)(e->save ? std::max(e->total_steps, 1) : 1)));
    const StreamLaunch kl = stream_launch(e);
    auto stages_for = [&](int NC, size_t budget) { return kl.stages(NC, budget); };
    ts::StreamParams base;
    memset(&base, 0, sizeof base);
    base.V = V; base.D = D; base.DP = DP; base.T = T;
    base.nparts = e->precision == GGNN_PREC_BF16X3 ? 3 : 1;
    base.cell = e->cell; base.act = e->act; base.use_bias = e->use_bias; base.use_avg = e->use_avg;
    base.tile_mask = gd.tile_mask;
    base.pair_src = gd.pair; base.vrow_ptr = gd.vptr; base.vsrc = gd.vsrc; base.tile_vptr = gd.tvp; base.vinfo = (const int4*)gd.vinfo;
    base.virt_img = (uint8_t*)e->ts_virt.ptr;   // pairs with several messages, pre-summed by the prologue of every gather launch
    base.slot_w = gd.slotw; base.vslot = gd.vslot;   // weighted batches: the virtual rows' message weights (null for a binary batch; with
                                                     // attention the step's probabilities, set per step)
    base.indeg = gd.indeg; base.denom = gd.denom;
    base.drop_keep = e->drop_keep; base.drop_seed = e->drop_seed;
    base.error_flag = (int*)e->err_flag.ptr;
    const int nc0 = e->ts_nc[0], nb0 = e->ts_nblk[0], nc1 = e->ts_nc[1], nb1 = e->ts_nblk[1];
    // one CTA per SM for all three kernels: the whole shared memory is the ring (CudnnCompatibleGRUCell's hidden-projection launch has the
    // candidate's N blocks, and so its ring)
    const int ns_edge = stages_for(nc0, avail > csr_b ? avail - csr_b : 0);
    const int ns_gate = stages_for(nc1, avail), ns_cand = stages_for(nc0, avail);
    // the kernel's parity waits are only sound if every ring has at least as many stages as there are gather groups (ts::MIN_NS)
    const int ns_min = std::min({ns_edge, ns_gate, ns_cand});
    if (ns_min < ts::MIN_NS)
        return e->fail(GGNN_EUNSUPPORTED, "streaming ring of %d stages (DP=%d): it needs at least %d, one per gather group", ns_min, DP,
                       ts::MIN_NS);
    auto smem_of = [&](int NC, int ns, bool gather) { return kl.smem(NC, ns, gather ? csr_b : 0); };
    void (*k_edge)(ts::StreamParams) = kl.edge;
    void (*k_fed)(ts::StreamParams) = kl.fed;
    const size_t sm_edge = smem_of(nc0, ns_edge, true);
    const size_t sm_fed = std::max(smem_of(nc1, ns_gate, false), smem_of(nc0, ns_cand, false));
    CU_TRY(e, cudaFuncSetAttribute(k_edge, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm_edge));
    CU_TRY(e, cudaFuncSetAttribute(k_fed, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm_fed));

    {   // node_states_per_layer[0] -> operand image
        const long long total = (long long)ntiles * ts::TILE_M * (DP / 8);
        ts::ggnn_image_kernel<<<(int)std::min<long long>((total + 255) / 256, 4096), 256, 0, st>>>(h0, img_state(0), chk_state(0), V, D, DP, ntiles);
        ++e->last_launches;
    }
    const WeightTiles& wt = e->ts_tiles;
    const uint8_t* wb = (const uint8_t*)wt.buf.ptr;
    for (int l = 0; l < L; ++l) {
        const uint8_t* img_in = img_state(l);
        const float* chk_in = chk_state(l);
        if (e->steps[l] == 0) {   // a layer without timesteps aliases the previous state (sparse:152)
            CU_TRY(e, cudaMemcpyAsync(layer_state(e, l + 1, h0, h_out), layer_state(e, l, h0, h_out), vd_bytes, cudaMemcpyDeviceToDevice, st));
            CU_TRY(e, cudaMemcpyAsync(img_state(l + 1), img_in, img_b, cudaMemcpyDeviceToDevice, st));
            CU_TRY(e, cudaMemcpyAsync(chk_state(l + 1), chk_in, img_b, cudaMemcpyDeviceToDevice, st));
            continue;
        }
        const int R = e->nres[l], nseg = R + 2;
        for (int s = 0; s < e->steps[l]; ++s) {
            const bool last = s == e->steps[l] - 1;
            float* out = last ? layer_state(e, l + 1, h0, h_out) : nullptr;   // the row-major copy exists only for node_states_per_layer entries
            uint8_t* img_out = last ? img_state(l + 1) : img_tmp[s & 1];
            float* chk_out = last ? chk_state(l + 1) : chk_tmp[s & 1];
            const int gs = e->step_base[l] + s;
            const SaveDev sv = saved_step(e, gs);
            // ---- aggregated messages (with attention: the step's probabilities first, the gather's slot weights)
            ts::StreamParams p = base;
            if (e->use_att) {
                float* att = (float*)e->att_buf.ptr + (size_t)gs * att_stride;
                ts::attention_chunk_kernel<<<(V + 7) / 8, 256, 0, st>>>(gd.row_ptr, gd.src, chk_in, e->w[l].edge_type_attention_weights, att, V, D,
                                                                        DP, T);
                ++e->last_launches;
                p.slot_w = att;
            }
            if (e->dense_device) {   // every (row, type) pair's A_t . h row, into its virtual row
                dense_apply_launch(e, st, false, (const float*)e->dense_adj.ptr, chk_in, nullptr, (uint8_t*)e->ts_virt.ptr);
                ++e->last_launches;
            }
            p.epi = ts::EPI_AGG; p.NC = nc0; p.nstages = ns_edge;
            p.g_img = img_in; p.w = wb + wt.off_edge[l]; p.kt_all = T * NKS;
            p.bias = e->use_bias ? e->w[l].edge_biases : nullptr;
            p.img_out = img_agg; p.sv_agg = sv.agg; p.gstep = gs;
            k_edge<<<dim3(ntiles, nb0), ts::NTHREADS, sm_edge, st>>>(p);
            ++e->last_launches;
            // [res.. | agg | last_img], or without last_img (null: CudnnCompatibleGRUCell's candidate, whose recurrent half is its own launch)
            auto set_segs = [&](ts::StreamParams& q, const uint8_t* last_img) {
                q.nseg = last_img ? nseg : nseg - 1;
                for (int i = 0; i < R; ++i) q.seg[i] = img_state(e->res[l][i]);
                q.seg[R] = img_agg;
                if (last_img) q.seg[R + 1] = last_img;
                q.kt_all = q.nseg * NKS;
            };
            if (gated) {
                ts::StreamParams q = base;
                q.epi = ts::EPI_GATE; q.NC = nc1; q.nstages = ns_gate;
                set_segs(q, img_in);
                q.w = wb + wt.off_gate[l]; q.bias = e->w[l].gate_bias; q.h_chk = chk_in; q.u_buf = u_chk;
                if (cudnn) q.rq_chk = rq_chk; else q.img_out = img_rh;
                q.sv_r = sv.r; q.sv_h = sv.h_in; q.sv_u = sv.u;
                q.gstep = gs;
                k_fed<<<dim3(ntiles, nb1), ts::NTHREADS, smem_of(nc1, ns_gate, false), st>>>(q);
                ++e->last_launches;
            }
            if (cudnn) {   // q = h . K_hid + b_hid over the step's input state; r <- r*q
                ts::StreamParams q = base;
                q.epi = ts::EPI_HPROJ; q.NC = nc0; q.nstages = ns_cand;
                q.nseg = 1; q.seg[0] = img_in; q.kt_all = NKS;
                q.w = wb + wt.off_hproj[l]; q.b_hid = e->w[l].cand_hidden_bias; q.rq_chk = rq_chk; q.sv_q = sv.q;
                q.gstep = gs;
                k_fed<<<dim3(ntiles, nb0), ts::NTHREADS, smem_of(nc0, ns_cand, false), st>>>(q);
                ++e->last_launches;
            }
            ts::StreamParams c = base;
            c.epi = ts::EPI_CAND; c.NC = nc0; c.nstages = ns_cand;
            set_segs(c, cudnn ? nullptr : (gated ? img_rh : img_in));
            c.w = wb + wt.off_cand[l]; c.bias = e->w[l].cand_bias; c.h_chk = chk_in; c.u_buf = u_chk; c.h_chk_out = chk_out; c.h_out = out; c.img_out = img_out;
            if (cudnn) c.rq_chk = rq_chk;
            if (gated) c.sv_c = sv.c; else c.sv_h = sv.h_in;
            c.gstep = gs;
            k_fed<<<dim3(ntiles, nb0), ts::NTHREADS, smem_of(nc0, ns_cand, false), st>>>(c);
            ++e->last_launches;
            img_in = img_out; chk_in = chk_out;
        }
    }
    return GGNN_OK;
}

// ------------------------------------------------------------------------------------------ sparse GCN (chem_tensorflow_gcn.py:42-82)
// Host half of a GCN batch: validate the int64 (row i = output, column j = input) list, feed it to the GGNN builder as one edge type
// (source j -> target i, list order kept) with the weights as per-message weights.  `msg_weighted` (w null): the weights come later, on the
// device (ggnn_set_message_weights) -- the weight sections are zero and, with save_for_backward, the image carries the source-keyed CSR's
// slot map.  No GCN plan depends on the weights' values.
static int build_gcn_image(ggnn_prepared_graph* g, int32_t V, int64_t nnz, const int64_t* list, const float* w, bool msg_weighted = false) {
    g->valid = false;
    if (V < 0 || nnz < 0 || (nnz > 0 && (!list || (!w && !msg_weighted)))) return g->fail(GGNN_EINVAL, "null/negative argument");
    if (nnz > 0x7fffffff) return g->fail(GGNN_EUNSUPPORTED, "batch too large for int32 indexing");
    std::vector<int32_t> pairs((size_t)nnz * 2);
    if (const int64_t k = gcn_pairs(V, nnz, list, pairs.data()); k >= 0)
        return g->fail(GGNN_ERANGE, "adjacency_list[%lld] = (%lld, %lld) is out of range for %d nodes", (long long)k, (long long)list[2 * k],
                       (long long)list[2 * k + 1], V);
    const std::vector<float> indeg((size_t)std::max(V, 1), 0.0f);
    const int32_t* lists[1] = {pairs.data()};
    const int32_t counts[1] = {(int32_t)nnz};
    if (!msg_weighted) return build_sparse_image(g, V, lists, counts, indeg.data(), true, w);
    if (int rc = build_sparse_image(g, V, lists, counts, indeg.data(), true, nullptr, false, true)) return rc;
    g->plan.plan_text += " [message-weighted]";
    return GGNN_OK;
}

int ggnn_gcn_create(const ggnn_gcn_config* cfg, ggnn_engine** out) {
    if (!cfg || !out) { g_create_error = "null argument"; return GGNN_EINVAL; }
    *out = nullptr;
    ggnn_engine* e = new ggnn_engine();
    if (int rc = init_gcn_shape(*e, cfg, g_create_error)) { delete e; return rc; }
    return attach_device(e, out);
}

int ggnn_gcn_set_weights(ggnn_engine* e, const ggnn_gcn_layer_weights* layers, int32_t num_layers) {
    if (!e) return GGNN_EINVAL;
    GGNN_REQUIRE_MODEL(e, MODEL_GCN);
    if (!layers || num_layers != e->L) return e->fail(GGNN_EINVAL, "expected %d layers of weights, got %d", e->L, num_layers);
    for (int l = 0; l < e->L; ++l) {
        const ggnn_gcn_layer_weights& w = layers[l];
        if (!w.kernel) return e->fail(GGNN_EINVAL, "layer %d: null kernel", l);
        if (e->use_bias && !w.bias) return e->fail(GGNN_EINVAL, "layer %d: use_bias set but bias is null", l);
        if (((uintptr_t)w.kernel & 15) || ((uintptr_t)w.bias & 15)) return e->fail(GGNN_EINVAL, "layer %d: weight pointers must be 16-byte aligned", l);
    }
    for (int l = 0; l < e->L; ++l) { e->gcn_w[l] = layers[l]; if (!e->use_bias) e->gcn_w[l].bias = nullptr; }
    e->weights_set = true;
    ++e->weights_gen;
    e->saved_valid = false;   // as in ggnn_set_weights
    return GGNN_OK;
}

int ggnn_prepare_graph_gcn(const ggnn_engine* e, int32_t save_for_backward, int32_t V, int64_t nnz, const int64_t* list, const float* w,
                           ggnn_prepared_graph** inout) {
    if (int rc = begin_prepare<ggnn_gcn_config>(inout, e, nullptr, 0, save_for_backward, __func__)) return rc;
    return build_gcn_image(*inout, V, nnz, list, w);
}

int ggnn_host_prepare_graph_gcn(const ggnn_gcn_config* cfg, int32_t num_sms, int32_t save_for_backward, int32_t V, int64_t nnz,
                                const int64_t* list, const float* w, ggnn_prepared_graph** inout) {
    if (int rc = begin_prepare(inout, nullptr, cfg, num_sms, save_for_backward, __func__)) return rc;
    return build_gcn_image(*inout, V, nnz, list, w);
}

int ggnn_prepare_graph_gcn_message_weighted(const ggnn_engine* e, int32_t save_for_backward, int32_t V, int64_t nnz, const int64_t* list,
                                            ggnn_prepared_graph** inout) {
    if (int rc = begin_prepare<ggnn_gcn_config>(inout, e, nullptr, 0, save_for_backward, __func__)) return rc;
    return build_gcn_image(*inout, V, nnz, list, nullptr, true);
}

int ggnn_host_prepare_graph_gcn_message_weighted(const ggnn_gcn_config* cfg, int32_t num_sms, int32_t save_for_backward, int32_t V,
                                                 int64_t nnz, const int64_t* list, ggnn_prepared_graph** inout) {
    if (int rc = begin_prepare(inout, nullptr, cfg, num_sms, save_for_backward, __func__)) return rc;
    return build_gcn_image(*inout, V, nnz, list, nullptr, true);
}

int ggnn_set_graph_gcn(ggnn_engine* e, int32_t V, int64_t nnz, const int64_t* list, const float* w, ggnn_stream_t stream) {
    if (!e) return GGNN_EINVAL;
    GGNN_REQUIRE_MODEL(e, MODEL_GCN);
    return set_graph_from_own_prep(e, stream, [&](ggnn_prepared_graph** g) { return ggnn_prepare_graph_gcn(e, -1, V, nnz, list, w, g); });
}

int ggnn_prepared_graph_slot_weights(const ggnn_prepared_graph* g, float* target_csr_w, float* source_csr_w) {
    if (!g || !g->valid || !g->plan.weighted) return GGNN_ESTATE;
    const BatchPlan& q = g->plan;
    const ImageView img = image_view(q, g->shape.use_att, g->image.ptr);
    if (source_csr_w && !img.tslotw) return GGNN_ESTATE;
    if (target_csr_w && q.M) memcpy(target_csr_w, img.slotw, sizeof(float) * (size_t)q.M);
    if (source_csr_w && q.M) memcpy(source_csr_w, img.tslotw, sizeof(float) * (size_t)q.M);
    return GGNN_OK;
}

// Whether the GCN runs on its fused wgmma kernel (hidden <= 128); else on the streaming plan (gcn_streams) or on the fp32 kernel, one launch
// per layer.
static bool gcn_on_tensor_cores(const ggnn_engine* e) { return e->precision != GGNN_PREC_FP32 && e->DP <= 128; }

// The GCN's streaming plan (wide_hidden, hidden > 128 on bf16x3 / bf16), two launches per layer on fixed 128-row tiles:
//   gcn_gather_image_kernel  S = A . H_l from the row-major fp32 state -> the operand image (one, reused by every layer)
//   ggnn_stream_kernel       TMA-fed, one segment: S . W_l, then EPI_GCN (bias; relu and state dropout but on the last layer) -> H_{l+1},
//                            row-major fp32, on every layer (the backward and ggnn_layer_state read them)
static int forward_gcn_stream(ggnn_engine* e, const float* h0, float* h_out, cudaStream_t st) {
    const int D = e->D, DP = e->DP, L = e->L, V = e->V, NKS = DP / 16, ntiles = e->ntiles;
    if (int rc = ts_prepare_weights(e, st)) return rc;
    CU_TRY(e, e->ts_images.reserve((size_t)ntiles * NKS * ts::A_STAGE_B));
    uint8_t* img_s = (uint8_t*)e->ts_images.ptr;
    const StreamLaunch kl = stream_launch(e);
    const int nc = e->ts_nc[0], nb = e->ts_nblk[0];
    const int ns = kl.stages(nc, e->max_smem > 2048 ? e->max_smem - 2048 : 0);
    if (ns < ts::MIN_NS)
        return e->fail(GGNN_EUNSUPPORTED, "streaming ring of %d stages (DP=%d): it needs at least %d, one per gather group", ns, DP, ts::MIN_NS);
    const size_t smem = kl.smem(nc, ns, 0);
    CU_TRY(e, cudaFuncSetAttribute(kl.fed, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    ts::StreamParams p;
    memset(&p, 0, sizeof p);
    p.V = V; p.D = D; p.DP = DP; p.T = 1;
    p.nparts = e->precision == GGNN_PREC_BF16X3 ? 3 : 1;
    p.epi = ts::EPI_GCN; p.NC = nc; p.nstages = ns;
    p.nseg = 1; p.seg[0] = img_s; p.kt_all = NKS;
    p.drop_keep = e->drop_keep; p.drop_seed = e->drop_seed;
    p.error_flag = (int*)e->err_flag.ptr;
    const WeightTiles& wt = e->ts_tiles;
    const ImageView& gd = e->gd;
    const long long gather_threads = (long long)ntiles * (ts::TILE_M / 4) * ((DP / 8 + 7) / 8) * 32;
    for (int l = 0; l < L; ++l) {
        gcn::gcn_gather_image_kernel<<<(int)((gather_threads + 255) / 256), 256, 0, st>>>(gd.row_ptr, gd.src, gd.slotw,
                                                                                      layer_state(e, l, h0, h_out), img_s, V, D, DP, ntiles);
        p.w = (const uint8_t*)wt.buf.ptr + wt.off_edge[l];
        p.bias = e->gcn_w[l].bias;
        p.relu_dropout = l < L - 1;
        p.gstep = l;   // the dropout's global step is the layer index
        p.h_out = layer_state(e, l + 1, h0, h_out);
        kl.fed<<<dim3(ntiles, nb), ts::NTHREADS, smem, st>>>(p);
        e->last_launches += 2;
    }
    return GGNN_OK;
}

static int forward_gcn(ggnn_engine* e, const float* h0, float* h_out, cudaStream_t st) {
    if (gcn_streams(*e)) return forward_gcn_stream(e, h0, h_out, st);
    const int D = e->D, DP = e->DP, L = e->L, V = e->V;
    const bool tcore = gcn_on_tensor_cores(e);
    gcn::GcnParams p;
    memset(&p, 0, sizeof p);
    p.V = V; p.D = D; p.DP = DP; p.L = L;
    p.nparts = e->precision == GGNN_PREC_BF16X3 ? 3 : 1;
    p.save = e->save ? 1 : 0;
    p.tile_start = e->gd.tile_start; p.row_ptr = e->gd.row_ptr; p.csr_src = e->gd.src; p.slot_w = e->gd.slotw;
    set_layer_states(e, p, h0, h_out);
    for (int l = 0; l < L; ++l) { p.kernel[l] = e->gcn_w[l].kernel; p.bias[l] = e->gcn_w[l].bias; }
    p.drop_keep = e->drop_keep; p.drop_seed = e->drop_seed;
    p.error_flag = (int*)e->err_flag.ptr;
    if (tcore) {
        int rc = tc_prepare_weights(e, st);
        if (rc) return rc;
        const WeightTiles& wt = e->tc_tiles;
        for (int l = 0; l < L; ++l) p.w_tiled[l] = (const uint8_t*)wt.buf.ptr + wt.off_edge[l];
        const size_t opb = (size_t)DP * gcn::KGS / 4, slot_b = (size_t)DP * 128, sh_b = e->local ? (size_t)tc::TILE_M * DP * sizeof(float) : 0;
        const size_t avail = e->max_smem > 1024 ? e->max_smem - 1024 : 0;
        p.nstages = (int)std::min<size_t>(gcn::MAX_STAGES, avail > opb + sh_b ? (avail - opb - sh_b) / slot_b : 0);
        if (p.nstages < 2) return e->fail(GGNN_EUNSUPPORTED, "not enough shared memory for the GCN tensor-core tile (DP=%d)", DP);
        const size_t smem = opb + (size_t)p.nstages * slot_b + sh_b;
        void (*kern)(gcn::GcnParams) = nullptr;
        switch (DP / 2) {
#define GGNN_GCN_CASE(nh)                                                                                                    \
    case nh:                                                                                                                 \
        kern = e->local ? (p.nparts == 3 ? gcn::gcn_wgmma_kernel<true, nh, true> : gcn::gcn_wgmma_kernel<true, nh, false>)   \
                        : (p.nparts == 3 ? gcn::gcn_wgmma_kernel<false, nh, true> : gcn::gcn_wgmma_kernel<false, nh, false>); \
        break;
            GGNN_GCN_CASE(8) GGNN_GCN_CASE(16) GGNN_GCN_CASE(24) GGNN_GCN_CASE(32) GGNN_GCN_CASE(40) GGNN_GCN_CASE(48) GGNN_GCN_CASE(56) GGNN_GCN_CASE(64)
#undef GGNN_GCN_CASE
            default: return e->fail(GGNN_EUNSUPPORTED, "no GCN tensor-core kernel for DP=%d", DP);
        }
        CU_TRY(e, cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        for (int l = 0; l < (e->local ? 1 : L); ++l) {
            p.g_layer = l;
            kern<<<e->ntiles, gcn::NTHREADS, smem, st>>>(p);
            ++e->last_launches;
        }
    } else {
        const size_t smem = (size_t)gcn::F32_ROWS * D * sizeof(float);
        CU_TRY(e, cudaFuncSetAttribute(gcn::gcn_fp32_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        for (int l = 0; l < L; ++l) {
            p.g_layer = l;
            gcn::gcn_fp32_kernel<<<(V + gcn::F32_ROWS - 1) / gcn::F32_ROWS, gcn::F32_THREADS, smem, st>>>(p);
            ++e->last_launches;
        }
    }
    return GGNN_OK;
}

// Backward of the GCN layers, per layer in reverse (the two GEMMs on FFMA, or on bf16x3 wgmma: ggnn_set_backward_precision):
//   dPre = dOut (last layer) or dOut * relu'(y) * mask / keep (gcn_relu_dropout_grad_kernel, from the saved output y)
//   S    = A . H_l (recomputed from the saved layer input: one gather instead of L saved [V, D] arrays)
//   dW  += S^T . dPre,  db += sum dPre            (gemm_tn: atomic or fixed-order split sums, the bias rides along)
//   dS   = dPre . W^T                             (gemm_nt)
//   dH_l = A^T . dS                               (csr_gather_all_kernel over the source-keyed CSR with its per-slot weights: no float atomics)
// With d_dw (DEVICE [nnz] or null: the adjacency weights' gradient of a message-weighted batch, accumulated into) dS is formed on every
// layer, layer 0 included, and gcn_source_grad_kernel replaces the last gather: the same dH_l bits, and d w_k += <dS_l[i_k], H_l[j_k]> into
// a per-target-slot sum (dw_slot) that msgw::add_slot_grads_kernel adds into d_dw at the end.
static int gcn_backward_impl(ggnn_engine* e, const float* d_h_out, const ggnn_gcn_layer_grads* grads, int32_t num_layers, float* d_h0,
                             float* d_dw, ggnn_stream_t stream) {
    using namespace ggnn::bwd;
    if (int rc = begin_backward(e, "ggnn_gcn_backward", "setting the graph", d_h_out, grads, num_layers, d_h0)) return rc;
    cudaStream_t st = (cudaStream_t)stream;
    const int V = e->V, D = e->D, L = e->L;
    if (V == 0) return GGNN_OK;
    const size_t vd = (size_t)V * D;
    const size_t slab = align_up(vd * sizeof(float), 256);
    const size_t ws_floats = std::max(gemm_tn_workspace(e, true, e->use_bias, V, D, D, 1), gemm_tn_workspace(e, false, e->use_bias, V, D, D, 1));
    const bool want_dw = d_dw && e->M > 0;
    const size_t o_dws = align_up(4 * slab + ws_floats * sizeof(float), 256);
    CU_TRY(e, e->bwd_buf.reserve(want_dw ? o_dws + sizeof(float) * (size_t)e->M : 4 * slab + ws_floats * sizeof(float)));
    char* bb = (char*)e->bwd_buf.ptr;
    float *dH = (float*)bb, *dP = (float*)(bb + slab), *S = (float*)(bb + 2 * slab), *dS = (float*)(bb + 3 * slab), *ws = (float*)(bb + 4 * slab);
    float* dw_slot = (float*)(bb + o_dws);
    if (want_dw) CU_TRY(e, cudaMemsetAsync(dw_slot, 0, sizeof(float) * (size_t)e->M, st));
    const ImageView& gd = e->gd;
    std::vector<const float*> fstate(L + 1);
    for (int l = 0; l <= L; ++l) fstate[l] = layer_state(e, l, e->last_h0, e->last_out);
    const long long n = (long long)vd;
    const int eb = (int)std::min<long long>((n + 255) / 256, 4096);
    const dim3 gather_grid((V + 7) / 8, 1);
    const float* dout = d_h_out;
    for (int l = L - 1; l >= 0; --l) {
        const float* dpre = dout;
        if (l < L - 1) {
            const float keep = e->saved_drop_keep < 1.0f ? e->saved_drop_keep : 1.0f;
            gcn::gcn_relu_dropout_grad_kernel<<<eb, 256, 0, st>>>(dout, fstate[l + 1], dP, 1.0f / keep, n);
            ++e->last_launches;
            dpre = dP;
        }
        const ggnn_gcn_layer_grads& gw = grads[l];
        if (gw.kernel) {
            GatherJob j{gd.row_ptr, gd.src, fstate[l], S, gd.slotw, nullptr};
            csr_gather_all_kernel<<<gather_grid, 256, 0, st>>>(j, j, V, D, 1);
            ++e->last_launches;
            SegList sl;
            memset(&sl, 0, sizeof sl);
            sl.p[0] = S; sl.ld[0] = D;
            if (int rc = gemm_tn(e, st, ws, ws_floats, sl, 1, true, dpre, D, gw.kernel, D, 0, e->use_bias ? gw.bias : nullptr, V, D, D)) return rc;
        } else if (e->use_bias && gw.bias) {
            SegList none;
            memset(&none, 0, sizeof none);
            if (int rc = gemm_tn(e, st, ws, ws_floats, none, 1, true, dpre, D, nullptr, D, 0, gw.bias, V, D, D)) return rc;
        }
        if (l == 0 && !d_h0 && !want_dw) break;
        gemm_nt(e, st, false, dpre, D, 0, e->gcn_w[l].kernel, D, 0, 1, dS, D, V, D, D);
        float* dst = l == 0 ? d_h0 : dH;
        if (want_dw) {
            const bool want_dh = dst != nullptr;
            void (*kern)(const int*, const int*, const int*, const float*, const float*, const float*, float*, float*, int, int) = nullptr;
            switch ((D + 127) / 128) {
#define GGNN_GCN_SRC_CASE(ch) \
    case ch: kern = want_dh ? gcn::gcn_source_grad_kernel<ch, true> : gcn::gcn_source_grad_kernel<ch, false>; break;
                GGNN_GCN_SRC_CASE(1) GGNN_GCN_SRC_CASE(2) GGNN_GCN_SRC_CASE(3) GGNN_GCN_SRC_CASE(4)
#undef GGNN_GCN_SRC_CASE
                default: return e->fail(GGNN_EUNSUPPORTED, "no GCN source-row gradient kernel for D=%d", D);
            }
            kern<<<gather_grid, 256, 0, st>>>(gd.trow, gd.ttgt, gd.tslot, gd.tslotw, dS, fstate[l], dst, dw_slot, V, D);
        } else {
            GatherJob j{gd.trow, gd.ttgt, dS, dst, gd.tslotw, nullptr};
            csr_gather_all_kernel<<<gather_grid, 256, 0, st>>>(j, j, V, D, 1);
        }
        ++e->last_launches;
        dout = dst;
    }
    if (want_dw) {
        msgw::add_slot_grads_kernel<<<(int)std::min<int64_t>((e->M + 255) / 256, 4096), 256, 0, st>>>(gd.msg, dw_slot, d_dw, e->M);
        ++e->last_launches;
    }
    CU_TRY(e, cudaGetLastError());
    return GGNN_OK;
}

int ggnn_gcn_backward(ggnn_engine* e, const float* d_h_out, const ggnn_gcn_layer_grads* grads, int32_t num_layers, float* d_h0, ggnn_stream_t stream) {
    if (!e) return GGNN_EINVAL;
    GGNN_REQUIRE_MODEL(e, MODEL_GCN);
    return gcn_backward_impl(e, d_h_out, grads, num_layers, d_h0, nullptr, stream);
}

int ggnn_gcn_backward_weighted(ggnn_engine* e, const float* d_h_out, const ggnn_gcn_layer_grads* grads, int32_t num_layers, float* d_h0,
                               float* d_adjacency_weights, ggnn_stream_t stream) {
    if (!e) return GGNN_EINVAL;
    GGNN_REQUIRE_MODEL(e, MODEL_GCN);
    if (d_adjacency_weights && !e->msg_weighted)
        return e->fail(GGNN_ESTATE, "d_adjacency_weights needs a message-weighted batch (ggnn_prepare_graph_gcn_message_weighted)");
    return gcn_backward_impl(e, d_h_out, grads, num_layers, d_h0, d_adjacency_weights, stream);
}

int ggnn_forward(ggnn_engine* e, const float* h0, float* h_out, ggnn_stream_t stream) {
    if (!e) return GGNN_EINVAL;
    const bool gcn = e->model == MODEL_GCN;
    if (!e->weights_set) return e->fail(GGNN_ESTATE, "%s has not been called", gcn ? "ggnn_gcn_set_weights" : "ggnn_set_weights");
    if (!e->graph_set) return no_graph(e);
    if (e->msg_weighted && !e->msg_weights_set)
        return e->fail(GGNN_ESTATE, "the batch is message-weighted: ggnn_set_message_weights must follow its upload before a forward");
    if ((!h0 || !h_out) && e->V > 0) return e->fail(GGNN_EINVAL, "null state pointer");
    if (((uintptr_t)h0 & 15) || ((uintptr_t)h_out & 15)) return e->fail(GGNN_EINVAL, "state pointers must be 16-byte aligned");
    // In place is refused: the GLOBAL launches gather h0 rows that other CTAs of the same launch overwrite, and the backward reads h0 as
    // node_states_per_layer[0] after the forward.
    const uintptr_t vd_bytes = (uintptr_t)e->V * e->D * sizeof(float), a = (uintptr_t)h0, b = (uintptr_t)h_out;
    if (vd_bytes > 0 && a < b + vd_bytes && b < a + vd_bytes)
        return e->fail(GGNN_EINVAL, "h_out (%p) overlaps h0 (%p) over their %zu bytes: the forward does not run in place", (const void*)h_out,
                       (const void*)h0, (size_t)vd_bytes);
    CU_TRY(e, cudaSetDevice(e->device));
    cudaStream_t st = (cudaStream_t)stream;
    e->last_launches = 0;
    e->fwd_valid = false; e->layers_written = false; e->saved_valid = false;
    const auto done = [&](bool layers_written, bool saved) {
        e->last_h0 = h0; e->last_out = h_out; e->fwd_valid = true; e->layers_written = layers_written;
        if (saved) { e->saved_valid = true; e->saved_drop_keep = e->drop_keep; e->saved_drop_seed = e->drop_seed; }
        return GGNN_OK;
    };
    if (e->V == 0) return done(true, e->save);   // the backward of an empty batch has nothing to compute either
    if (e->save) { int rc = reserve_states(e); if (rc) return rc; }
    if (!gcn && e->total_steps == 0) {  // no propagation at all: result is the input (sparse:152 with empty loops)
        CU_TRY(e, cudaMemcpyAsync(h_out, h0, (size_t)e->V * e->D * sizeof(float), cudaMemcpyDeviceToDevice, st));
        return done(false, false);
    }
    int rc;
    if (gcn) rc = forward_gcn(e, h0, h_out, st);
    else if (e->precision == GGNN_PREC_FP32) rc = e->stepwise ? forward_stepwise(e, h0, h_out, st) : forward_ffma(e, h0, h_out, st);
    else rc = e->stream ? forward_stream(e, h0, h_out, st) : forward_tc(e, h0, h_out, st);
    if (rc) return rc;
    CU_TRY(e, cudaGetLastError());
    return done(!(gcn && e->local && gcn_on_tensor_cores(e) && !e->save), e->save);
}

int ggnn_forward_host_async(ggnn_engine* e, const float* h0_host, float* h_out_host, ggnn_stream_t stream) {
    if (!e) return GGNN_EINVAL;
    if (!e->graph_set) return no_graph(e);
    if ((!h0_host || !h_out_host) && e->V > 0) return e->fail(GGNN_EINVAL, "null host pointer");
    const size_t bytes = (size_t)e->V * e->D * sizeof(float);
    IoSlots io;
    if (int rc = stage_io(e, h0_host, bytes, 0, (cudaStream_t)stream, io)) return rc;
    int rc = ggnn_forward(e, io.in, io.out, stream);
    if (rc) return rc;
    if (bytes) CU_TRY(e, cudaMemcpyAsync(h_out_host, io.out, bytes, cudaMemcpyDeviceToHost, (cudaStream_t)stream));
    return GGNN_OK;
}

int ggnn_forward_host(ggnn_engine* e, const float* h0_host, float* h_out_host, ggnn_stream_t stream) {
    int rc = ggnn_forward_host_async(e, h0_host, h_out_host, stream);
    if (rc) return rc;
    CU_TRY(e, cudaStreamSynchronize((cudaStream_t)stream));
    return GGNN_OK;
}

}  // extern "C"

// One call per batch, the shape of the reference's sess.run(fetch, feed_dict) (chem_tensorflow.py:235): the h0 upload is
// enqueued FIRST so the host-side CSR build of set_graph overlaps it.
template <class SetGraph>
static int run_host(ggnn_engine* e, int64_t V, const float* h0_host, float* h_out_host, cudaStream_t st, SetGraph set_graph) {
    if (!e) return GGNN_EINVAL;
    if (V < 0 || ((!h0_host || !h_out_host) && V > 0)) return e->fail(GGNN_EINVAL, "null host pointer / negative size");
    const size_t bytes = (size_t)V * e->D * sizeof(float);
    IoSlots io;
    int rc = stage_io(e, h0_host, bytes, 0, st, io);
    if (rc) return rc;
    rc = set_graph();
    if (rc) return rc;
    if ((int64_t)e->V != V) return e->fail(GGNN_EINVAL, "graph has %d nodes, h0 has %lld rows", e->V, (long long)V);
    rc = ggnn_forward(e, io.in, io.out, (ggnn_stream_t)st);
    if (rc) return rc;
    if (bytes) CU_TRY(e, cudaMemcpyAsync(h_out_host, io.out, bytes, cudaMemcpyDeviceToHost, st));
    CU_TRY(e, cudaStreamSynchronize(st));
    return GGNN_OK;
}

extern "C" {

int ggnn_run_sparse_host(ggnn_engine* e, int32_t V, const int32_t* const* adjacency_lists, const int32_t* num_edges,
                         const float* num_incoming_edges_per_type, const float* h0_host, float* h_out_host, ggnn_stream_t stream) {
    return run_host(e, V, h0_host, h_out_host, (cudaStream_t)stream,
                    [&]() { return ggnn_set_graph_sparse(e, V, adjacency_lists, num_edges, num_incoming_edges_per_type, stream); });
}

int ggnn_run_dense_host(ggnn_engine* e, int32_t b, int32_t v, const float* adjacency_matrix, const float* h0_host, float* h_out_host,
                        ggnn_stream_t stream) {
    return run_host(e, (int64_t)b * v, h0_host, h_out_host, (cudaStream_t)stream,
                    [&]() { return ggnn_set_graph_dense(e, b, v, adjacency_matrix, stream); });
}

// ------------------------------------------------------------------------------------------ readout (SURVEY 8f-1)
}  // extern "C"

// The layout of the readout map in ro_buf for V nodes in G graphs: graph_of [V] | start [G+1] | mask [V] | perm [V] | the device-only
// per-node gated values.  Returns the offset of the values (the bytes an upload may fill).
static size_t readout_layout(ggnn_engine* e, int V, int G) {
    size_t off = 0;
    e->ro_off_graph_of = off; off = align_up(off + sizeof(int) * (size_t)std::max(V, 1), 16);
    e->ro_off_start = off;    off = align_up(off + sizeof(int) * (size_t)(G + 1), 16);
    e->ro_off_mask = off;     off = align_up(off + sizeof(float) * (size_t)std::max(V, 1), 16);
    e->ro_off_perm = off;     off = align_up(off + sizeof(int) * (size_t)std::max(V, 1), 16);   // uploaded for ungrouped lists only
    e->ro_off_val = off;      // device-only scratch: per-node gated value
    return off;
}

extern "C" {

int ggnn_readout_set_graphs(ggnn_engine* e, int32_t num_nodes, const int32_t* graph_nodes_list, int32_t num_graphs,
                            int32_t nodes_per_graph, const float* node_mask, ggnn_stream_t stream) {
    if (!e) return GGNN_EINVAL;
    e->ro_V = -1;
    if (num_nodes < 0 || num_graphs < 0) return e->fail(GGNN_EINVAL, "negative size");
    if (!graph_nodes_list && (nodes_per_graph <= 0 || (int64_t)nodes_per_graph * num_graphs != num_nodes))
        return e->fail(GGNN_EINVAL, "without a graph_nodes_list the batch must be num_graphs x nodes_per_graph (%d x %d != %d)", num_graphs, nodes_per_graph, num_nodes);
    CU_TRY(e, cudaSetDevice(e->device));
    const int V = num_nodes, G = num_graphs;
    const size_t off = readout_layout(e, V, G);
    const size_t dev_bytes = align_up(off + sizeof(float) * (size_t)std::max(V, 1), 16);
    CU_TRY(e, e->ro_stage.begin(off));
    CU_TRY(e, e->ro_buf.reserve(dev_bytes));
    char* base = e->ro_stage.ptr;
    int* graph_of = (int*)(base + e->ro_off_graph_of);
    int* start = (int*)(base + e->ro_off_start);
    bool grouped = true;
    for (int v = 0; v < V; ++v) {
        const int g = graph_nodes_list ? graph_nodes_list[v] : v / nodes_per_graph;
        if ((unsigned)g >= (unsigned)G) return e->fail(GGNN_ERANGE, "graph_nodes_list[%d] = %d is out of range for %d graphs", v, g, G);
        if (v > 0 && g < graph_of[v - 1]) grouped = false;
        graph_of[v] = g;
    }
    if (grouped) {   // graph g owns the contiguous node range [start[g], start[g+1])
        int v = 0;
        for (int g = 0; g <= G; ++g) {
            while (v < V && graph_of[v] < g) ++v;
            start[g] = v;
        }
    } else {   // the stable counting sort by graph: graph g owns perm[start[g] .. start[g+1]), its nodes in index order (deterministic mode)
        int* perm = (int*)(base + e->ro_off_perm);
        std::fill(start, start + G + 1, 0);
        for (int v = 0; v < V; ++v) ++start[graph_of[v] + 1];
        for (int g = 0; g < G; ++g) start[g + 1] += start[g];
        std::vector<int> cursor(start, start + G);
        for (int v = 0; v < V; ++v) perm[cursor[graph_of[v]]++] = v;
    }
    if (node_mask) memcpy(base + e->ro_off_mask, node_mask, sizeof(float) * (size_t)V);
    CU_TRY(e, e->ro_stage.upload(e->ro_buf.ptr, grouped ? e->ro_off_perm : off, (cudaStream_t)stream));
    e->ro_V = V; e->ro_G = G; e->ro_grouped = grouped; e->ro_has_mask = node_mask != nullptr; e->ro_from_dataset = false;
    return GGNN_OK;
}

static int readout_check(ggnn_engine* e, const void* const* ptrs, int n) {
    if (e->ro_V < 0) return e->fail(GGNN_ESTATE, "ggnn_readout_set_graphs has not been called for this batch");
    if (e->D > 32 * readout::MAX_D_PER_LANE) return e->fail(GGNN_EUNSUPPORTED, "readout supports hidden_size <= %d", 32 * readout::MAX_D_PER_LANE);
    for (int i = 0; i < n; ++i) {
        if (!ptrs[i]) return e->fail(GGNN_EINVAL, "null readout argument %d", i);
        if (i != 3 && i != 5 && ((uintptr_t)ptrs[i] & 15)) return e->fail(GGNN_EINVAL, "readout argument %d must be 16-byte aligned", i);
    }
    return GGNN_OK;
}

}  // extern "C"

// The readout forward of K tasks over the current map: stage 1 into val [K][V] (device scratch), stage 2 into out[k * stride + slot[g]].
static int readout_run(ggnn_engine* e, const float* h_last, const float* h0, int K, const readout::TaskWeights& tw, const int* slot, int stride,
                       float* out, float* val, cudaStream_t st) {
    const int V = e->ro_V, G = e->ro_G;
    char* g = (char*)e->ro_buf.ptr;
    const float* mask = e->ro_has_mask ? (const float*)(g + e->ro_off_mask) : nullptr;
    if (V > 0) {
        if (K == 1) readout::readout_node_kernel<1><<<(V + 7) / 8, 256, 0, st>>>(h_last, h0, tw, K, mask, val, V, e->D);
        else readout::readout_node_kernel<readout::MAX_TASKS><<<(V + 7) / 8, 256, 0, st>>>(h_last, h0, tw, K, mask, val, V, e->D);
    }
    const dim3 per_graph((G + 127) / 128, K);
    if (e->ro_grouped || V == 0) {
        readout::readout_sum_grouped_kernel<<<per_graph, 128, 0, st>>>(val, (const int*)(g + e->ro_off_start), slot, out, G, V, stride);
    } else if (e->det) {
        readout::readout_sum_permuted_kernel<<<per_graph, 128, 0, st>>>(val, (const int*)(g + e->ro_off_start), (const int*)(g + e->ro_off_perm),
                                                                       slot, out, G, V, stride);
    } else {
        readout::readout_zero_kernel<<<per_graph, 128, 0, st>>>(slot, out, G, stride);
        readout::readout_sum_atomic_kernel<<<dim3((V + 255) / 256, K), 256, 0, st>>>(val, (const int*)(g + e->ro_off_graph_of), slot, out, V,
                                                                                      stride);
    }
    CU_TRY(e, cudaGetLastError());
    return GGNN_OK;
}

extern "C" {

int ggnn_readout_forward(ggnn_engine* e, const float* h_last, const float* h0, const float* w_gate, const float* b_gate,
                         const float* w_trans, const float* b_trans, float* out, ggnn_stream_t stream) {
    if (!e) return GGNN_EINVAL;
    const void* ps[7] = {h_last, h0, w_gate, b_gate, w_trans, b_trans, out};
    if (int rc = readout_check(e, ps, e->ro_V > 0 ? 7 : 0)) return rc;
    CU_TRY(e, cudaSetDevice(e->device));
    if (e->ro_G == 0) return GGNN_OK;
    if (!out) return e->fail(GGNN_EINVAL, "null output");
    readout::TaskWeights tw{};
    tw.w[0] = readout::Weights{w_gate, b_gate, w_trans, b_trans};
    return readout_run(e, h_last, h0, 1, tw, nullptr, e->ro_G, out, (float*)((char*)e->ro_buf.ptr + e->ro_off_val), (cudaStream_t)stream);
}

int ggnn_readout_predict(ggnn_engine* e, const float* h_last, const float* h0, int32_t num_tasks, const ggnn_readout_task* tasks,
                         const int32_t* slot, int32_t out_stride, float* out, ggnn_stream_t stream) {
    if (!e) return GGNN_EINVAL;
    if (num_tasks < 1 || num_tasks > readout::MAX_TASKS)
        return e->fail(GGNN_EINVAL, "num_tasks = %d: the readout runs 1 .. %d tasks per call", (int)num_tasks, readout::MAX_TASKS);
    if (!tasks) return e->fail(GGNN_EINVAL, "null tasks");
    const void* ps[2] = {h_last, h0};
    if (int rc = readout_check(e, ps, e->ro_V > 0 ? 2 : 0)) return rc;
    const int V = e->ro_V, G = e->ro_G;
    readout::TaskWeights tw{};
    for (int k = 0; k < num_tasks; ++k) {
        const void* w[4] = {tasks[k].w_gate, tasks[k].b_gate, tasks[k].w_trans, tasks[k].b_trans};
        for (int i = 0; i < 4; ++i) {
            if (!w[i]) return e->fail(GGNN_EINVAL, "task %d: null readout weight %d", k, i);
            if ((i == 0 || i == 2) && ((uintptr_t)w[i] & 15)) return e->fail(GGNN_EINVAL, "task %d: readout weight %d must be 16-byte aligned", k, i);
        }
        tw.w[k] = readout::Weights{tasks[k].w_gate, tasks[k].b_gate, tasks[k].w_trans, tasks[k].b_trans};
    }
    if (G == 0) return GGNN_OK;
    if (!out) return e->fail(GGNN_EINVAL, "null output");
    if (out_stride < 1 || (!slot && out_stride < G))
        return e->fail(GGNN_EINVAL, "out_stride = %d: without a slot map each task's row needs the batch's %d graphs", (int)out_stride, G);
    CU_TRY(e, cudaSetDevice(e->device));
    CU_TRY(e, e->ro_kval.reserve(sizeof(float) * (size_t)num_tasks * std::max(V, 1)));
    return readout_run(e, h_last, h0, num_tasks, tw, slot, out_stride, out, (float*)e->ro_kval.ptr, (cudaStream_t)stream);
}

int ggnn_dataset_batch_slots(const ggnn_engine* e, const int32_t** slot) {
    if (!e || !slot) return GGNN_EINVAL;
    if (e->ro_V < 0 || !e->ro_from_dataset) return GGNN_ESTATE;
    *slot = e->ro_dataset_slots;
    return GGNN_OK;
}

int ggnn_readout_backward(ggnn_engine* e, const float* h_last, const float* h0, const float* w_gate, const float* b_gate,
                          const float* w_trans, const float* b_trans, const float* d_out, float* d_h_last, float* d_w_gate,
                          float* d_b_gate, float* d_w_trans, float* d_b_trans, ggnn_stream_t stream) {
    if (!e) return GGNN_EINVAL;
    const void* ps[8] = {h_last, h0, w_gate, b_gate, w_trans, b_trans, d_out, d_h_last};
    if (int rc = readout_check(e, ps, e->ro_V > 0 ? 8 : 0)) return rc;
    CU_TRY(e, cudaSetDevice(e->device));
    const int V = e->ro_V;
    if (V == 0) return GGNN_OK;
    char* g = (char*)e->ro_buf.ptr;
    const float* mask = e->ro_has_mask ? (const float*)(g + e->ro_off_mask) : nullptr;
    readout::Weights w{w_gate, b_gate, w_trans, b_trans};
    if (e->det) {   // a grid fixed by V alone, per-block partials, then every gradient entry summed over the blocks in a fixed order
        const int blocks = std::max(1, std::min((V + 7) / 8, readout::RO_ORDERED_BLOCKS)), cols = 3 * e->D + 2;
        CU_TRY(e, e->ro_ws.reserve(sizeof(float) * (size_t)blocks * cols));
        float* part = (float*)e->ro_ws.ptr;
        // 8 columns per lane up to hidden 256, 16 above (its 8 warp rows then need dynamic shared memory)
        if (e->D <= 256) {
            readout::readout_bwd_ordered_kernel<8><<<blocks, 256, 0, (cudaStream_t)stream>>>(h_last, h0, w, (const int*)(g + e->ro_off_graph_of), mask,
                                                                                            d_out, d_h_last, part, V, e->D);
        } else {
            const size_t smem = readout::ro_ordered_smem<16>();
            CU_TRY(e, cudaFuncSetAttribute(readout::readout_bwd_ordered_kernel<16>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
            readout::readout_bwd_ordered_kernel<16><<<blocks, 256, smem, (cudaStream_t)stream>>>(h_last, h0, w, (const int*)(g + e->ro_off_graph_of),
                                                                                                mask, d_out, d_h_last, part, V, e->D);
        }
        readout::readout_bwd_reduce_kernel<<<cols, 256, 0, (cudaStream_t)stream>>>(part, blocks, e->D, d_w_gate, d_b_gate, d_w_trans, d_b_trans);
        CU_TRY(e, cudaGetLastError());
        return GGNN_OK;
    }
    const int blocks = std::max(1, std::min((V + 7) / 8, 4 * e->num_sms));
    (e->D <= 256 ? readout::readout_bwd_kernel<8> : readout::readout_bwd_kernel<16>)<<<blocks, 256, 0, (cudaStream_t)stream>>>(
        h_last, h0, w, (const int*)(g + e->ro_off_graph_of), mask, d_out, d_h_last, d_w_gate, d_b_gate, d_w_trans, d_b_trans, V, e->D);
    CU_TRY(e, cudaGetLastError());
    return GGNN_OK;
}

int ggnn_run_sparse_host_readout(ggnn_engine* e, int32_t V, const int32_t* const* adjacency_lists, const int32_t* num_edges,
                                 const float* indeg, const float* h0_host, const int32_t* graph_nodes_list, int32_t G, int32_t num_tasks,
                                 const ggnn_readout_task* tasks, const float* target_values, const float* target_mask, float* loss_out,
                                 float* accuracy_out, ggnn_stream_t stream) {
    if (!e) return GGNN_EINVAL;
    if (V < 0 || G < 0 || num_tasks <= 0 || !tasks || !loss_out || !accuracy_out || (V > 0 && (!h0_host || !graph_nodes_list)) ||
        (G > 0 && (!target_values || !target_mask)))
        return e->fail(GGNN_EINVAL, "null / negative argument");
    cudaStream_t st = (cudaStream_t)stream;
    const size_t tg = (size_t)num_tasks * std::max(G, 1);
    // device scratch behind the two state slots: targets | masks | per-task readout [tasks][G] | results [2*tasks]
    const size_t o_tm = align_up(tg * 4, 256), o_ro = 2 * o_tm, o_res = 3 * o_tm;
    IoSlots io;   // the h0 upload overlaps the host-side CSR build below
    int rc = stage_io(e, h0_host, (size_t)V * e->D * sizeof(float), o_res + align_up((size_t)2 * num_tasks * 4, 256), st, io);
    if (rc) return rc;
    char* sc = io.scratch;
    if (G > 0) {
        CU_TRY(e, cudaMemcpyAsync(sc, target_values, tg * 4, cudaMemcpyHostToDevice, st));
        CU_TRY(e, cudaMemcpyAsync(sc + o_tm, target_mask, tg * 4, cudaMemcpyHostToDevice, st));
    }
    rc = ggnn_set_graph_sparse(e, V, adjacency_lists, num_edges, indeg, stream);
    if (rc) return rc;
    rc = ggnn_readout_set_graphs(e, V, graph_nodes_list, G, 0, nullptr, stream);
    if (rc) return rc;
    rc = ggnn_forward(e, io.in, io.out, stream);
    if (rc) return rc;
    for (int t = 0; t < num_tasks; ++t) {
        rc = ggnn_readout_forward(e, io.out, io.in, tasks[t].w_gate, tasks[t].b_gate, tasks[t].w_trans, tasks[t].b_trans,
                                  (float*)(sc + o_ro) + (size_t)t * G, stream);
        if (rc) return rc;
    }
    readout::masked_loss_kernel<<<num_tasks, 256, 0, st>>>((const float*)(sc + o_ro), (const float*)sc, (const float*)(sc + o_tm),
                                                           (float*)(sc + o_res), G, num_tasks);
    CU_TRY(e, cudaGetLastError());
    std::vector<float> res((size_t)2 * num_tasks);
    CU_TRY(e, cudaMemcpyAsync(res.data(), sc + o_res, sizeof(float) * 2 * num_tasks, cudaMemcpyDeviceToHost, st));
    CU_TRY(e, cudaStreamSynchronize(st));
    for (int t = 0; t < num_tasks; ++t) { loss_out[t] = res[t]; accuracy_out[t] = res[num_tasks + t]; }
    return GGNN_OK;
}

}  // extern "C"

// The reference's evaluate_one_batch (sparse:352-362, dense:230-249) in one call: the upload and the forward without saving for backward
// (the save flag is restored afterwards), the readout map, every task's readout into [num_tasks][G] on the device, one D2H copy.
template <class SetGraph, class SetMap>
static int run_host_predict(ggnn_engine* e, int64_t V, const float* h0_host, int32_t G, int32_t num_tasks, const ggnn_readout_task* tasks,
                            float* out_host, cudaStream_t st, SetGraph set_graph, SetMap set_map) {
    if (!e) return GGNN_EINVAL;
    if (V < 0 || G < 0 || (V > 0 && !h0_host) || (G > 0 && !out_host)) return e->fail(GGNN_EINVAL, "null host pointer / negative size");
    const size_t bytes = (size_t)V * e->D * sizeof(float), kg = (size_t)std::max(num_tasks, 1) * std::max(G, 1);
    IoSlots io;
    int rc = stage_io(e, h0_host, bytes, sizeof(float) * kg, st, io);
    if (rc) return rc;
    const bool save = e->save;
    e->save = false;
    rc = set_graph();
    if (!rc && (int64_t)e->V != V) rc = e->fail(GGNN_EINVAL, "graph has %d nodes, h0 has %lld rows", e->V, (long long)V);
    if (!rc) rc = set_map();
    if (!rc) rc = ggnn_forward(e, io.in, io.out, (ggnn_stream_t)st);
    e->save = save;
    e->saved_valid = false;
    if (rc) return rc;
    float* res = (float*)io.scratch;
    rc = ggnn_readout_predict(e, io.out, io.in, num_tasks, tasks, nullptr, G, res, (ggnn_stream_t)st);
    if (rc) return rc;
    if (G > 0) CU_TRY(e, cudaMemcpyAsync(out_host, res, sizeof(float) * (size_t)num_tasks * G, cudaMemcpyDeviceToHost, st));
    CU_TRY(e, cudaStreamSynchronize(st));
    return GGNN_OK;
}

extern "C" {

int ggnn_run_sparse_host_predict(ggnn_engine* e, int32_t V, const int32_t* const* adjacency_lists, const int32_t* num_edges, const float* indeg,
                                 const float* h0_host, const int32_t* graph_nodes_list, int32_t G, int32_t num_tasks,
                                 const ggnn_readout_task* tasks, float* out_host, ggnn_stream_t stream) {
    if (e && V > 0 && !graph_nodes_list) return e->fail(GGNN_EINVAL, "null graph_nodes_list");
    return run_host_predict(e, V, h0_host, G, num_tasks, tasks, out_host, (cudaStream_t)stream,
                            [&]() { return ggnn_set_graph_sparse(e, V, adjacency_lists, num_edges, indeg, stream); },
                            [&]() { return ggnn_readout_set_graphs(e, V, graph_nodes_list, G, 0, nullptr, stream); });
}

int ggnn_run_dense_host_predict(ggnn_engine* e, int32_t b, int32_t v, const float* adjacency_matrix, const float* h0_host, const float* node_mask,
                                int32_t num_tasks, const ggnn_readout_task* tasks, float* out_host, ggnn_stream_t stream) {
    return run_host_predict(e, (int64_t)b * v, h0_host, b, num_tasks, tasks, out_host, (cudaStream_t)stream,
                            [&]() { return ggnn_set_graph_dense(e, b, v, adjacency_matrix, stream); },
                            [&]() { return ggnn_readout_set_graphs(e, b * v, nullptr, b, v, node_mask, stream); });
}

int ggnn_sync_check(ggnn_engine* e, ggnn_stream_t stream) {
    if (!e) return GGNN_EINVAL;
    CU_TRY(e, cudaSetDevice(e->device));
    CU_TRY(e, cudaStreamSynchronize((cudaStream_t)stream));
    int flag = 0;
    CU_TRY(e, cudaMemcpy(&flag, e->err_flag.ptr, sizeof(int), cudaMemcpyDeviceToHost));
    if (flag != 0) {
        cudaMemset(e->err_flag.ptr, 0, sizeof(int));
        return e->fail(GGNN_ECUDA, "propagation kernel reported a barrier timeout (role code %d)", flag);
    }
    return GGNN_OK;
}

int ggnn_set_save_for_backward(ggnn_engine* e, int32_t enable) {
    if (!e) return GGNN_EINVAL;
    e->save = enable != 0;
    e->saved_valid = false;
    return GGNN_OK;
}

int ggnn_set_deterministic(ggnn_engine* e, int32_t enable) {
    if (!e) return GGNN_EINVAL;
    e->det = enable != 0;
    return GGNN_OK;
}

int ggnn_set_backward_precision(ggnn_engine* e, int32_t precision) {
    if (!e) return GGNN_EINVAL;
    if (precision != GGNN_PREC_FP32 && precision != GGNN_PREC_BF16X3)
        return e->fail(GGNN_EINVAL, "backward precision must be GGNN_PREC_FP32 (%d) or GGNN_PREC_BF16X3 (%d), got %d", GGNN_PREC_FP32,
                       GGNN_PREC_BF16X3, (int)precision);
    e->bwd_precision = precision;
    return GGNN_OK;
}

int ggnn_set_state_dropout(ggnn_engine* e, float keep_prob, uint64_t seed) {
    if (!e) return GGNN_EINVAL;
    if (!(keep_prob > 0.0f) || keep_prob > 1.0f) return e->fail(GGNN_EINVAL, "state keep probability must be in (0, 1], got %g", (double)keep_prob);
    e->drop_keep = keep_prob;
    e->drop_seed = (unsigned long long)seed;
    return GGNN_OK;
}

int ggnn_state_dropout_mask(int32_t V, int32_t D, int32_t global_step, float keep_prob, uint64_t seed, uint8_t* mask_out) {
    if (V < 0 || D <= 0 || (!mask_out && V > 0)) return GGNN_EINVAL;
    for (int r = 0; r < V; ++r)
        for (int c = 0; c < D; ++c)
            mask_out[(size_t)r * D + c] = dropout_keeps((unsigned long long)seed, global_step, V, D, r, c, keep_prob) ? 1 : 0;
    return GGNN_OK;
}

int ggnn_backward(ggnn_engine* e, const float* d_h_out, const ggnn_layer_grads* grads, int32_t num_layers,
                  float* d_h0, ggnn_stream_t stream) {
    if (!e) return GGNN_EINVAL;
    GGNN_REQUIRE_MODEL(e, MODEL_GGNN);
    return ggnn_backward_impl(e, d_h_out, grads, num_layers, d_h0, nullptr, stream);
}

int ggnn_backward_weighted(ggnn_engine* e, const float* d_h_out, const ggnn_layer_grads* grads, int32_t num_layers, float* d_h0,
                           float* d_message_weights, ggnn_stream_t stream) {
    if (!e) return GGNN_EINVAL;
    GGNN_REQUIRE_MODEL(e, MODEL_GGNN);
    if (d_message_weights && !e->msg_weighted)
        return e->fail(GGNN_ESTATE, "d_message_weights needs a message-weighted batch (ggnn_prepare_graph_sparse_weighted)");
    return ggnn_backward_impl(e, d_h_out, grads, num_layers, d_h0, d_message_weights, stream);
}

// GGNN and GCN engines: a GCN's adjacency weights are its one edge type's message weights, in list order.
int ggnn_set_message_weights(ggnn_engine* e, const float* message_weights, ggnn_stream_t stream) {
    if (!e) return GGNN_EINVAL;
    if (!e->graph_set) return no_graph(e);
    if (!e->msg_weighted)
        return e->fail(GGNN_ESTATE, "the current batch is not message-weighted (%s)",
                       e->model == MODEL_GCN ? "ggnn_prepare_graph_gcn_message_weighted" : "ggnn_prepare_graph_sparse_weighted");
    if (!message_weights && e->M > 0) return e->fail(GGNN_EINVAL, "null message weights");
    CU_TRY(e, cudaSetDevice(e->device));
    e->msg_weights_set = false;
    e->saved_valid = false;   // the backward's gathers read the slot weights: they must be the saved forward's
    if (e->dense_device) {   // the engine's own copy of the [b, T, v, v] matrix, and its row sums as the in-degree table
        if (e->M > 0) {
            const size_t bytes = sizeof(float) * (size_t)e->M;
            CU_TRY(e, e->dense_adj.reserve(bytes));
            CU_TRY(e, cudaMemcpyAsync(e->dense_adj.ptr, message_weights, bytes, cudaMemcpyDeviceToDevice, (cudaStream_t)stream));
            const int64_t rows = (int64_t)e->dense_b * e->T * e->dense_v;
            dadj::dense_row_sums_kernel<<<(int)std::min<int64_t>((rows + 255) / 256, 4096), 256, 0, (cudaStream_t)stream>>>(
                (const float*)e->dense_adj.ptr, e->gd.indeg, e->dense_b, e->dense_v, e->T);
            CU_TRY(e, cudaGetLastError());
        }
    } else if (e->M > 0) {
        const ImageView& gd = e->gd;
        msgw::scatter_message_weights_kernel<<<(int)std::min<int64_t>((e->M + 255) / 256, 4096), 256, 0, (cudaStream_t)stream>>>(
            message_weights, gd.msg, gd.tslot, gd.slotw, gd.tslotw, e->M);
        CU_TRY(e, cudaGetLastError());
    }
    e->msg_weights_set = true;
    return GGNN_OK;
}

int ggnn_num_messages(const ggnn_engine* e, int64_t* out) {
    if (!e || !out) return GGNN_EINVAL;
    *out = e->M;
    return GGNN_OK;
}

int ggnn_get_csr(ggnn_engine* e, int32_t* row_ptr, int32_t* src, int32_t* msg) {
    if (!e) return GGNN_EINVAL;
    if (!e->graph_set) return e->fail(GGNN_ESTATE, "no graph set");
    CU_TRY(e, cudaSetDevice(e->device));
    CU_TRY(e, cudaDeviceSynchronize());
    if (row_ptr) CU_TRY(e, cudaMemcpy(row_ptr, e->gd.row_ptr, sizeof(int) * ((size_t)e->V * e->T + 1), cudaMemcpyDeviceToHost));
    const size_t M = e->dense_device ? 0 : (size_t)e->M;   // (a dense-device image lists no messages)
    if (src && M) CU_TRY(e, cudaMemcpy(src, e->gd.src, sizeof(int) * M, cudaMemcpyDeviceToHost));
    if (msg && M) CU_TRY(e, cudaMemcpy(msg, e->gd.msg, sizeof(int) * M, cudaMemcpyDeviceToHost));
    return GGNN_OK;
}

int ggnn_layer_state(ggnn_engine* e, int32_t layer, const float** dev_ptr) {
    if (!e || !dev_ptr) return GGNN_EINVAL;
    if (layer < 0 || layer > e->L) return e->fail(GGNN_EINVAL, "layer index %d out of range", layer);
    if (!e->graph_set || !e->fwd_valid) return e->fail(GGNN_ESTATE, "no forward has run on the current graph");
    if (layer > 0 && layer < e->L && !e->layers_written)
        return e->fail(GGNN_ESTATE, "layer %d: the last forward did not write the layers between h0 and the result (enable save_for_backward)", layer);
    *dev_ptr = layer_state(e, layer, e->last_h0, e->last_out);
    return GGNN_OK;
}

int ggnn_copy_layer_state(ggnn_engine* e, int32_t layer, float* dst, ggnn_stream_t stream) {
    const float* src = nullptr;
    int rc = ggnn_layer_state(e, layer, &src);
    if (rc) return rc;
    if (!dst) return e->fail(GGNN_EINVAL, "null destination");
    CU_TRY(e, cudaSetDevice(e->device));
    if (e->V > 0)
        CU_TRY(e, cudaMemcpyAsync(dst, src, (size_t)e->V * e->D * sizeof(float), cudaMemcpyDeviceToDevice, (cudaStream_t)stream));
    return GGNN_OK;
}

int ggnn_last_launch_count(const ggnn_engine* e) { return e ? e->last_launches : 0; }
const char* ggnn_plan_description(const ggnn_engine* e) { return e ? e->plan_text.c_str() : ""; }

}  // extern "C"

// ------------------------------------------------------------------------------------------ device-resident datasets (ggnn_dataset.cuh)
// A dataset holds every graph's pieces of a batch image in graph-local numbering, uploaded once: its target-CSR rows and slots, in-degrees
// and denominators, the source-keyed CSR (training datasets), the streaming tables (GGNN on tensor cores), the slot weights (GCN), and its
// annotations and labels.  The host keeps what a batch plan needs and no edge: per graph its sizes and the dataset offsets of its pieces,
// per edge type its message count, and per cut segment (node range between two cut points) its message count and edge-type mask.
struct DsGraph {
    int V = 0, M = 0, nv = 0, nvm = 0;
    int seg0 = 0, nseg = 0;   // its segments in ggnn_dataset::seg_*
};

struct ggnn_dataset : ErrorText {
    ModelShape shape;
    bool train = false, stream_tables = false, weighted = false, on_device = false;
    bool dense = false;   // ggnn_dataset_create_dense: batches of nodes_per_graph rows per graph (ggnn_dataset_prepare_batch_dense)
    int N = 0, ann = 0, tasks = 0;
    std::vector<DsGraph> graphs;
    std::vector<int> type_msgs;   // [N][T]
    std::vector<int> seg_end, seg_msgs;   // graph-local end node and messages (by target) of every cut segment
    std::vector<unsigned> seg_mask;
    DevBuf buf;
    ds::DsArrays dev{};
};

struct ggnn_dataset_batch : ErrorText {
    const ggnn_dataset* ds = nullptr;
    ModelShape shape;
    BatchPlan plan;
    size_t bytes = 0;
    int G = 0;
    int v = 0;               // a dense batch's rows per graph; 0 for sparse and GCN batches
    StagedImage table;       // tile starts [ntiles + 1] | the per-graph records [G][R_MBASE + T] | the graphs' dataset indices [G] (16-byte aligned)
    size_t table_bytes = 0, off_records = 0, off_slots = 0;
    bool valid = false;
};

// The host arrays of a dataset before its upload, section by section (each 16-byte aligned in the one image).
struct DsHost {
    std::vector<int> base, row_end, src, pos, trow_end, ttgt, tslot, pair, vend, vsrc, vpre, vslot, nfeat;
    std::vector<float> indeg, denom, slotw, tslotw;
};

// Adds one graph of V nodes: per edge type t its graph-local (source, target) list adj[t] of ne[t] messages in the reference's order, its
// [V][T] in-degrees, and (weighted datasets) its per-message weights w in type-major order.  Builds its pieces with the batch builder's
// section builders (count_edges, fill_denominators, fill_source_csr, stream_rows; find_cuts) and its target CSR with fill_target_csr, on
// the graph alone, and appends them.
static int ds_add_graph(ggnn_dataset* d, DsHost& h, int gi, int V, const int32_t* const* adj, const int32_t* ne, const float* indeg, const float* w) {
    const int T = d->shape.T;
    DsGraph g;
    g.V = V;
    std::vector<int64_t> type_base(T + 1, 0);
    for (int t = 0; t < T; ++t) type_base[t + 1] = type_base[t] + ne[t];
    std::vector<int> counts((size_t)V * T + 1), reach((size_t)V + 1);
    if (!count_edges(V, T, adj, type_base.data(), 1, counts.data(), reach.data())) {
        int t, i;
        first_bad_edge(V, T, adj, ne, t, i);
        return d->fail(GGNN_ERANGE, "graph %d: edge %d of type %d = (%d,%d) is out of range for its %d nodes", gi, i, t, adj[t][2 * i],
                       adj[t][2 * i + 1], V);
    }
    d->type_msgs.insert(d->type_msgs.end(), ne, ne + T);
    const int M = (int)type_base[T];
    g.M = M;
    std::vector<int> row_ptr((size_t)V * T + 1), src((size_t)std::max(M, 1)), msg((size_t)std::max(M, 1));
    fill_target_csr(V, T, adj, ne, counts, row_ptr.data(), src.data(), msg.data());
    h.row_end.insert(h.row_end.end(), row_ptr.begin() + 1, row_ptr.end());
    h.src.insert(h.src.end(), src.begin(), src.begin() + M);
    for (size_t k = 0; k < (size_t)V * T; ++k)
        for (int m = row_ptr[k]; m < row_ptr[k + 1]; ++m) h.pos.push_back(msg[m] - (int)type_base[k % T]);
    h.indeg.insert(h.indeg.end(), indeg, indeg + (size_t)V * T);
    const size_t d0 = h.denom.size();
    h.denom.resize(d0 + V);
    fill_denominators(0, V, T, indeg, h.denom.data() + d0);
    if (d->weighted)
        for (int m = 0; m < M; ++m) h.slotw.push_back(w[msg[m]]);
    if (d->train) {
        std::vector<int> trow((size_t)V * T + 1);
        const size_t t0 = h.ttgt.size();
        h.ttgt.resize(t0 + M);
        if (d->shape.use_att) h.tslot.resize(t0 + M);
        if (d->weighted) h.tslotw.resize(t0 + M);
        fill_source_csr(V, T, adj, ne, M, msg.data(), w, trow.data(), h.ttgt.data() + t0, d->shape.use_att ? h.tslot.data() + t0 : nullptr,
                        d->weighted ? h.tslotw.data() + t0 : nullptr);
        h.trow_end.insert(h.trow_end.end(), trow.begin() + 1, trow.end());
    }
    if (d->stream_tables) {   // the graph's streaming tables on its own, virtual rows numbered in row order from 0 (with attention every row
                              // with messages, and vslot graph-local)
        const bool att = d->shape.use_att != 0;
        std::vector<int> pair((size_t)V * T), vptr((size_t)V * T + 1, 0), vsrc((size_t)std::max(M, 1)), vslot(att ? (size_t)V * T : 0);
        int nv = 0, nvm = 0;
        stream_rows(0, (size_t)V * T, row_ptr.data(), src.data(), nullptr, att, pair.data(), vptr.data(), vsrc.data(), nullptr,
                    att ? vslot.data() : nullptr, nv, nvm);
        if (att) h.vslot.insert(h.vslot.end(), vslot.begin(), vslot.begin() + nv);
        g.nv = nv; g.nvm = nvm;
        int before = 0;
        for (int v = 0; v < V; ++v) {
            h.vpre.push_back(before);
            for (int t = 0; t < T; ++t) before += pair[(size_t)v * T + t] <= -2;
        }
        h.pair.insert(h.pair.end(), pair.begin(), pair.end());
        h.vend.insert(h.vend.end(), vptr.begin() + 1, vptr.begin() + 1 + nv);
        h.vsrc.insert(h.vsrc.end(), vsrc.begin(), vsrc.begin() + nvm);
    }
    std::vector<int> cuts;
    find_cuts(reach.data(), V, cuts);
    g.seg0 = (int)d->seg_end.size();
    g.nseg = (int)cuts.size() - 1;
    for (int k = 0; k < g.nseg; ++k) {
        unsigned mask = 0;
        for (size_t r = (size_t)cuts[k] * T; r < (size_t)cuts[k + 1] * T; ++r) mask |= (unsigned)(row_ptr[r + 1] > row_ptr[r]) << (r % T);
        d->seg_end.push_back(cuts[k + 1]);
        d->seg_msgs.push_back(row_ptr[(size_t)cuts[k + 1] * T] - row_ptr[(size_t)cuts[k] * T]);
        d->seg_mask.push_back(mask);
    }
    d->graphs.push_back(g);
    return GGNN_OK;
}

// After the graphs: the per-graph base table, the annotations and labels, and (with a device) the one upload of every section.
static int ds_finish(ggnn_dataset* d, DsHost& h, const float* ann, const float* labels, const float* lmask, cudaStream_t stream) {
    int64_t node = 0, slot = 0, vrow = 0, vs = 0;
    for (const DsGraph& g : d->graphs) {
        h.base.insert(h.base.end(), {(int)node, (int)slot, (int)vrow, (int)vs});
        node += g.V; slot += g.M; vrow += g.nv; vs += g.nvm;
        if (node * d->shape.T > 0x7fffffff || slot > 0x7fffffff || vs > 0x7fffffff)
            return d->fail(GGNN_EUNSUPPORTED, "dataset too large for int32 indexing");
    }
    h.base.insert(h.base.end(), {(int)node, (int)slot, (int)vrow, (int)vs});
    if (!d->on_device) return GGNN_OK;
    const size_t nann = (size_t)node * d->ann, nlab = (size_t)d->N * d->tasks;
    struct Section { const void* src; size_t bytes; const void** dst; };
    ds::DsArrays& a = d->dev;
    a = ds::DsArrays{};
    a.ann_size = d->ann; a.tasks = d->tasks;
    auto I = [](const std::vector<int>& v, const int** dst) { return Section{v.data(), v.size() * sizeof(int), (const void**)dst}; };
    auto F = [](const std::vector<float>& v, const float** dst) { return Section{v.data(), v.size() * sizeof(float), (const void**)dst}; };
    const Section secs[] = {I(h.base, &a.base), I(h.row_end, &a.row_end), I(h.src, &a.src), I(h.pos, &a.pos), F(h.indeg, &a.indeg),
                            F(h.denom, &a.denom), I(h.trow_end, &a.trow_end), I(h.ttgt, &a.ttgt), I(h.tslot, &a.tslot), I(h.pair, &a.pair),
                            I(h.vend, &a.vend), I(h.vsrc, &a.vsrc), I(h.vpre, &a.vpre), I(h.vslot, &a.vslot), F(h.slotw, &a.slotw), F(h.tslotw, &a.tslotw),
                            {ann, nann * sizeof(float), (const void**)&a.ann}, {labels, nlab * sizeof(float), (const void**)&a.labels},
                            {lmask, nlab * sizeof(float), (const void**)&a.lmask}, I(h.nfeat, &a.nfeat)};
    const bool present[] = {true, true, true, true, true, true, d->train, d->train, d->train && d->shape.use_att, d->stream_tables,
                            d->stream_tables, d->stream_tables, d->stream_tables, d->stream_tables && d->shape.use_att, d->weighted,
                            d->weighted && d->train, true, d->tasks > 0,
                            d->tasks > 0, d->dense};
    size_t total = 0;
    for (const Section& s : secs) total = align_up(total + s.bytes, 16);
    std::vector<char> image(total);
    size_t off = 0;
    std::vector<size_t> offs;
    for (const Section& s : secs) {
        if (s.bytes) memcpy(image.data() + off, s.src, s.bytes);
        offs.push_back(off);
        off = align_up(off + s.bytes, 16);
    }
    if (d->buf.reserve(std::max<size_t>(total, 16)) != cudaSuccess) {
        cudaGetLastError();
        return d->fail(GGNN_ECUDA, "cudaMalloc of the dataset's %zu bytes failed", total);
    }
    CU_TRY(d, cudaMemcpyAsync(d->buf.ptr, image.data(), total, cudaMemcpyHostToDevice, stream));
    CU_TRY(d, cudaStreamSynchronize(stream));   // the staging image is pageable and freed on return
    for (size_t i = 0; i < sizeof secs / sizeof secs[0]; ++i) *secs[i].dst = present[i] ? (const char*)d->buf.ptr + offs[i] : nullptr;
    return GGNN_OK;
}

// The prologue of the four create calls: the model shape (model_shape_for), then the argument checks; the handle is allocated here and
// returned even on failure, with the text in ggnn_dataset_error.
template <class Config>
static int begin_dataset(ggnn_dataset** out, const ggnn_engine* e, const Config* cfg, int32_t num_sms, int32_t for_training, int32_t N,
                         const int64_t* node_counts, int32_t ann, const float* annotations, int32_t tasks, const float* labels,
                         const float* lmask, const char* fn) {
    if (!out || (!e && (!cfg || num_sms <= 0))) return GGNN_EINVAL;
    ggnn_dataset* d = new ggnn_dataset();
    *out = d;
    if (int rc = model_shape_for(d, d->shape, e, cfg, num_sms, fn)) return rc;
    d->on_device = e != nullptr;
    d->train = for_training != 0;
    d->weighted = d->shape.model == MODEL_GCN;
    d->stream_tables = d->shape.model == MODEL_GGNN && d->shape.precision != GGNN_PREC_FP32;
    d->N = N; d->ann = ann; d->tasks = tasks;
    if (N < 0 || ann < 0 || tasks < 0 || (N > 0 && !node_counts) || (ann > 0 && N > 0 && !annotations) || (tasks > 0 && N > 0 && (!labels || !lmask)))
        return d->fail(GGNN_EINVAL, "null/negative argument");
    if (ann > d->shape.D) return d->fail(GGNN_EINVAL, "annotation_size %d exceeds hidden_size %d", ann, d->shape.D);
    for (int i = 0; i < N; ++i)
        if (node_counts[i] < 0 || node_counts[i] > 0x7fffffff) return d->fail(GGNN_EINVAL, "graph %d: node count %lld", i, (long long)node_counts[i]);
    return GGNN_OK;
}

template <class Config>
static int create_dataset_sparse(ggnn_dataset** out, const ggnn_engine* e, const Config* cfg, int32_t num_sms, int32_t for_training, int32_t N,
                                 const int64_t* node_counts, const int32_t* const* edge_lists, const int64_t* edge_offsets, const float* indeg,
                                 int32_t ann, const float* annotations, int32_t tasks, const float* labels, const float* lmask,
                                 cudaStream_t stream, const char* fn) {
    if (int rc = begin_dataset(out, e, cfg, num_sms, for_training, N, node_counts, ann, annotations, tasks, labels, lmask, fn)) return rc;
    ggnn_dataset* d = *out;
    const int T = d->shape.T;
    if (N > 0 && (!edge_lists || !edge_offsets || !indeg)) return d->fail(GGNN_EINVAL, "null edge lists / offsets / in-degrees");
    DsHost h;
    std::vector<const int32_t*> adj(T);
    std::vector<int32_t> ne(T);
    int64_t node = 0;
    for (int i = 0; i < N; ++i) {
        for (int t = 0; t < T; ++t) {
            const int64_t* eo = edge_offsets + (size_t)t * (N + 1);
            if (eo[i] < 0 || eo[i + 1] < eo[i] || eo[i + 1] - eo[i] > 0x7fffffff || (eo[i + 1] > eo[i] && !edge_lists[t]))
                return d->fail(GGNN_EINVAL, "graph %d: bad edge offsets of type %d", i, t);
            adj[t] = eo[i + 1] > eo[i] ? edge_lists[t] + 2 * eo[i] : nullptr;
            ne[t] = (int32_t)(eo[i + 1] - eo[i]);
        }
        if (int rc = ds_add_graph(d, h, i, (int)node_counts[i], adj.data(), ne.data(), indeg + (size_t)node * T, nullptr)) return rc;
        node += node_counts[i];
    }
    return ds_finish(d, h, annotations, labels, lmask, stream);
}

// GCN entries (row i = output, column j = input, int64, graph-local) become one edge type j -> i with fp32 weights, as in build_gcn_image.
template <class Config>
static int create_dataset_gcn(ggnn_dataset** out, const ggnn_engine* e, const Config* cfg, int32_t num_sms, int32_t for_training, int32_t N,
                              const int64_t* node_counts, const int64_t* lists, const int64_t* entry_offsets, const float* weights, int32_t ann,
                              const float* annotations, int32_t tasks, const float* labels, const float* lmask, cudaStream_t stream,
                              const char* fn) {
    if (int rc = begin_dataset(out, e, cfg, num_sms, for_training, N, node_counts, ann, annotations, tasks, labels, lmask, fn)) return rc;
    ggnn_dataset* d = *out;
    if (N > 0 && !entry_offsets) return d->fail(GGNN_EINVAL, "null entry offsets");
    DsHost h;
    std::vector<int32_t> pairs;
    for (int i = 0; i < N; ++i) {
        const int64_t e0 = entry_offsets[i], e1 = entry_offsets[i + 1], V = node_counts[i];
        if (e0 < 0 || e1 < e0 || e1 - e0 > 0x7fffffff || (e1 > e0 && (!lists || !weights))) return d->fail(GGNN_EINVAL, "graph %d: bad entry offsets", i);
        pairs.resize((size_t)(e1 - e0) * 2);
        if (const int64_t k = gcn_pairs(V, e1 - e0, lists + 2 * e0, pairs.data()); k >= 0)
            return d->fail(GGNN_ERANGE, "graph %d: entry %lld = (%lld, %lld) is out of range for its %lld nodes", i, (long long)k,
                           (long long)lists[2 * (e0 + k)], (long long)lists[2 * (e0 + k) + 1], (long long)V);
        const std::vector<float> indeg((size_t)V, 0.0f);
        const int32_t* adj[1] = {pairs.data()};
        const int32_t ne[1] = {(int32_t)(e1 - e0)};
        if (int rc = ds_add_graph(d, h, i, (int)V, adj, ne, indeg.data(), weights + e0)) return rc;
    }
    return ds_finish(d, h, annotations, labels, lmask, stream);
}

// Dense graphs: the reference's raw (src, bond, dest) triples, int64 [sum E, 3] with graph offsets [N+1], and each graph's feature count.
// Each triple sets A[bond-1, dest, src] and A[bond-1+bwd, src, dest] (dense:30-36, bwd = 0 tied, T/2 untied); as assignments, duplicates
// collapse.  The graph's per-type lists are those entries in the order scan_dense emits them -- target row, then source column -- and
// its in-degrees the number of distinct sources.  A graph spans V_g = max(features, largest id + 1) rows; annotations arrive for its
// feature rows only and are stored for all V_g (zero beyond the features), so that the kernels read them like a sparse graph's.
template <class Config>
static int create_dataset_dense(ggnn_dataset** out, const ggnn_engine* e, const Config* cfg, int32_t num_sms, int32_t for_training, int32_t N,
                                const int64_t* feature_counts, const int64_t* triples, const int64_t* graph_offsets, int32_t tie_fwd_bkwd,
                                int32_t ann, const float* annotations, int32_t tasks, const float* labels, const float* lmask,
                                cudaStream_t stream, const char* fn) {
    if (int rc = begin_dataset(out, e, cfg, num_sms, for_training, N, feature_counts, ann, annotations, tasks, labels, lmask, fn)) return rc;
    ggnn_dataset* d = *out;
    d->dense = true;
    if (d->shape.use_att) return d->fail(GGNN_EUNSUPPORTED, "propagation attention exists only in the sparse model (sparse:170-196)");
    if (d->shape.cudnn_tc) return d->fail(GGNN_EUNSUPPORTED, "CudnnCompatibleGRUCell exists only in the sparse model (sparse:105-108)");
    if (N > 0 && !graph_offsets) return d->fail(GGNN_EINVAL, "null graph offsets");
    const int T = d->shape.T, bwd = tie_fwd_bkwd ? 0 : T / 2;
    DsHost h;
    std::vector<float> ann_rows;   // [sum V_g][ann]
    std::vector<std::array<int, 3>> ent;   // (type, target, source)
    std::vector<std::vector<int32_t>> lists(T);
    std::vector<const int32_t*> adj(T);
    std::vector<int32_t> ne(T);
    int64_t feat_row = 0;
    for (int i = 0; i < N; ++i) {
        const int64_t e0 = graph_offsets[i], e1 = graph_offsets[i + 1];
        if (e0 < 0 || e1 < e0 || (e1 > e0 && !triples)) return d->fail(GGNN_EINVAL, "graph %d: bad graph offsets", i);
        int64_t Vg = feature_counts[i];
        ent.clear();
        for (int64_t k = e0; k < e1; ++k) {
            const int64_t s = triples[3 * k], b = triples[3 * k + 1], t = triples[3 * k + 2];
            if (s < 0 || t < 0 || s >= 0x7fffffff || t >= 0x7fffffff || b < 1 || b - 1 + bwd >= T)
                return d->fail(GGNN_ERANGE, "graph %d: edge %lld = (%lld, %lld, %lld) is out of range (node ids >= 0, bond types 1..%d)", i,
                               (long long)(k - e0), (long long)s, (long long)b, (long long)t, T - bwd);
            ent.push_back({(int)(b - 1), (int)t, (int)s});
            ent.push_back({(int)(b - 1 + bwd), (int)s, (int)t});
            Vg = std::max(Vg, std::max(s, t) + 1);
        }
        std::sort(ent.begin(), ent.end());
        ent.erase(std::unique(ent.begin(), ent.end()), ent.end());
        for (int t = 0; t < T; ++t) lists[t].clear();
        std::vector<float> indeg((size_t)Vg * T, 0.0f);
        for (const auto& x : ent) {
            lists[x[0]].push_back(x[2]);
            lists[x[0]].push_back(x[1]);
            indeg[(size_t)x[1] * T + x[0]] += 1.0f;
        }
        for (int t = 0; t < T; ++t) { adj[t] = lists[t].data(); ne[t] = (int32_t)(lists[t].size() / 2); }
        if (int rc = ds_add_graph(d, h, i, (int)Vg, adj.data(), ne.data(), indeg.data(), nullptr)) return rc;
        h.nfeat.push_back((int)feature_counts[i]);
        if (ann > 0) {
            ann_rows.insert(ann_rows.end(), annotations + feat_row * ann, annotations + (feat_row + feature_counts[i]) * ann);
            ann_rows.resize(ann_rows.size() + (size_t)(Vg - feature_counts[i]) * ann, 0.0f);
        }
        feat_row += feature_counts[i];
    }
    return ds_finish(d, h, ann_rows.data(), labels, lmask, stream);
}

extern "C" {

int ggnn_dataset_create_sparse(const ggnn_engine* e, int32_t for_training, int32_t num_graphs, const int64_t* node_counts,
                               const int32_t* const* edge_lists, const int64_t* edge_offsets, const float* num_incoming_edges_per_type,
                               int32_t annotation_size, const float* annotations, int32_t num_tasks, const float* labels, const float* label_mask,
                               ggnn_stream_t stream, ggnn_dataset** out) {
    if (!e) return GGNN_EINVAL;
    return create_dataset_sparse<ggnn_config>(out, e, nullptr, 0, for_training, num_graphs, node_counts, edge_lists, edge_offsets,
                                              num_incoming_edges_per_type, annotation_size, annotations, num_tasks, labels, label_mask,
                                              (cudaStream_t)stream, __func__);
}

int ggnn_host_dataset_create_sparse(const ggnn_config* cfg, int32_t num_sms, int32_t for_training, int32_t num_graphs, const int64_t* node_counts,
                                    const int32_t* const* edge_lists, const int64_t* edge_offsets, const float* num_incoming_edges_per_type,
                                    int32_t annotation_size, const float* annotations, int32_t num_tasks, const float* labels,
                                    const float* label_mask, ggnn_dataset** out) {
    return create_dataset_sparse(out, nullptr, cfg, num_sms, for_training, num_graphs, node_counts, edge_lists, edge_offsets,
                                 num_incoming_edges_per_type, annotation_size, annotations, num_tasks, labels, label_mask, nullptr, __func__);
}

int ggnn_dataset_create_gcn(const ggnn_engine* e, int32_t for_training, int32_t num_graphs, const int64_t* node_counts, const int64_t* adjacency_lists,
                            const int64_t* entry_offsets, const float* adjacency_weights, int32_t annotation_size, const float* annotations,
                            int32_t num_tasks, const float* labels, const float* label_mask, ggnn_stream_t stream, ggnn_dataset** out) {
    if (!e) return GGNN_EINVAL;
    return create_dataset_gcn<ggnn_gcn_config>(out, e, nullptr, 0, for_training, num_graphs, node_counts, adjacency_lists, entry_offsets,
                                               adjacency_weights, annotation_size, annotations, num_tasks, labels, label_mask,
                                               (cudaStream_t)stream, __func__);
}

int ggnn_host_dataset_create_gcn(const ggnn_gcn_config* cfg, int32_t num_sms, int32_t for_training, int32_t num_graphs, const int64_t* node_counts,
                                 const int64_t* adjacency_lists, const int64_t* entry_offsets, const float* adjacency_weights,
                                 int32_t annotation_size, const float* annotations, int32_t num_tasks, const float* labels,
                                 const float* label_mask, ggnn_dataset** out) {
    return create_dataset_gcn(out, nullptr, cfg, num_sms, for_training, num_graphs, node_counts, adjacency_lists, entry_offsets, adjacency_weights,
                              annotation_size, annotations, num_tasks, labels, label_mask, nullptr, __func__);
}

int ggnn_dataset_create_dense(const ggnn_engine* e, int32_t for_training, int32_t num_graphs, const int64_t* feature_counts, const int64_t* graphs,
                              const int64_t* graph_offsets, int32_t tie_fwd_bkwd, int32_t annotation_size, const float* annotations,
                              int32_t num_tasks, const float* labels, const float* label_mask, ggnn_stream_t stream, ggnn_dataset** out) {
    if (!e) return GGNN_EINVAL;
    return create_dataset_dense<ggnn_config>(out, e, nullptr, 0, for_training, num_graphs, feature_counts, graphs, graph_offsets, tie_fwd_bkwd,
                                             annotation_size, annotations, num_tasks, labels, label_mask, (cudaStream_t)stream, __func__);
}

int ggnn_host_dataset_create_dense(const ggnn_config* cfg, int32_t num_sms, int32_t for_training, int32_t num_graphs, const int64_t* feature_counts,
                                   const int64_t* graphs, const int64_t* graph_offsets, int32_t tie_fwd_bkwd, int32_t annotation_size,
                                   const float* annotations, int32_t num_tasks, const float* labels, const float* label_mask, ggnn_dataset** out) {
    return create_dataset_dense(out, nullptr, cfg, num_sms, for_training, num_graphs, feature_counts, graphs, graph_offsets, tie_fwd_bkwd,
                                annotation_size, annotations, num_tasks, labels, label_mask, nullptr, __func__);
}

int ggnn_free_dataset(ggnn_dataset* d) {
    if (!d) return GGNN_OK;
    if (d->on_device) { cudaSetDevice(d->shape.device); d->buf.release(); }
    delete d;
    return GGNN_OK;
}

const char* ggnn_dataset_error(const ggnn_dataset* d) { return d ? d->err.c_str() : "null dataset"; }

}  // extern "C"

// The host half of both batch kinds.  v = 0: a sparse or GCN batch, graphs end to end.  v > 0: a dense batch, graph i at node offset i*v
// followed by its padding rows, each an isolated node -- a cut point after every one, as the host builder finds them.
static int prepare_dataset_batch(const ggnn_dataset* d, int32_t save_for_backward, const int64_t* graph_ids, int32_t num_graphs, bool dense,
                                 int v, ggnn_dataset_batch** inout) {
    if (!d || !inout || num_graphs < 0 || (num_graphs > 0 && !graph_ids)) return GGNN_EINVAL;
    ggnn_dataset_batch* b = *inout;
    if (!b) { b = new ggnn_dataset_batch(); *inout = b; }
    b->valid = false;
    b->ds = d;
    b->shape = d->shape;
    b->v = dense ? v : 0;
    b->table.use_cuda = d->on_device;
    if (d->dense != dense)
        return b->fail(GGNN_EINVAL, d->dense ? "a dense dataset's batches are prepared with ggnn_dataset_prepare_batch_dense"
                                             : "ggnn_dataset_prepare_batch_dense needs a dataset made by ggnn_dataset_create_dense");
    if (dense && v <= 0) return b->fail(GGNN_EINVAL, "nodes_per_graph = %d", v);
    v = b->v;
    const bool save = save_for_backward != 0;
    if (save && !d->train) return b->fail(GGNN_ESTATE, "save_for_backward needs a dataset created for training (the source-keyed CSR is built there)");
    if (save && d->tasks == 0) return b->fail(GGNN_EINVAL, "the dataset has no targets: its batches can be predicted, not trained on");
    const int T = d->shape.T, G = num_graphs;
    for (int i = 0; i < G; ++i)
        if (graph_ids[i] < 0 || graph_ids[i] >= d->N)
            return b->fail(GGNN_ERANGE, "graph_ids[%d] = %lld is out of range for a dataset of %d graphs", i, (long long)graph_ids[i], d->N);
    for (int i = 0; i < G && v > 0; ++i)
        if (d->graphs[graph_ids[i]].V > v)
            return b->fail(GGNN_EINVAL, "graph_ids[%d] = %lld: graph of %d nodes does not fit nodes_per_graph = %d", i, (long long)graph_ids[i],
                           d->graphs[graph_ids[i]].V, v);
    // offsets and the cut points: every graph's segments, shifted by its node offset (dense: then one per padding row)
    int64_t V = 0, M = 0, nv = 0, nvm = 0;
    std::vector<int64_t> type_tot(T, 0);
    std::vector<int> cuts(1, 0);
    for (int i = 0; i < G; ++i) {
        const DsGraph& g = d->graphs[graph_ids[i]];
        for (int k = 0; k < g.nseg; ++k) cuts.push_back((int)(V + d->seg_end[g.seg0 + k]));
        for (int r = g.V + 1; r <= v; ++r) cuts.push_back((int)(V + r));
        V += v > 0 ? v : g.V; M += g.M; nv += g.nv; nvm += g.nvm;
        for (int t = 0; t < T; ++t) type_tot[t] += d->type_msgs[(size_t)graph_ids[i] * T + t];
        if (M > 0x7fffffff || V * T + 1 > 0x7fffffff) return b->fail(GGNN_EUNSUPPORTED, "batch too large for int32 indexing");
    }
    BatchPlan& p = b->plan;
    std::vector<int> tile_start;
    if (int rc = build_plan(d->shape, (int)V, d->weighted, cuts, p, tile_start, b->err)) return rc;
    if (d->dense) p.plan_text += " [binary dense adjacency -> CSR]";
    b->bytes = layout_image(d->shape, p, save, M, (int)nv, nvm);
    if (p.local) {   // tiles of whole segments: their message counts and edge types from the segment summaries (only LOCAL launches read them)
        // (a dense batch's padding rows are segments of no message and no edge type: a tile may end inside them)
        size_t tile = 1;
        int msgs = 0; unsigned mask = 0;
        int64_t node = 0;
        for (int i = 0; i < G; ++i) {
            const DsGraph& g = d->graphs[graph_ids[i]];
            for (int k = 0; k < g.nseg; ++k) {
                msgs += d->seg_msgs[g.seg0 + k]; mask |= d->seg_mask[g.seg0 + k];
                if (node + d->seg_end[g.seg0 + k] == tile_start[tile]) {
                    p.max_tile_msgs = std::max(p.max_tile_msgs, msgs);
                    p.max_tile_types = std::max(p.max_tile_types, __builtin_popcount(mask));
                    msgs = 0; mask = 0; ++tile;
                }
            }
            for (int r = g.V + 1; r <= v; ++r)
                if (node + r == tile_start[tile]) {
                    p.max_tile_msgs = std::max(p.max_tile_msgs, msgs);
                    p.max_tile_types = std::max(p.max_tile_types, __builtin_popcount(mask));
                    msgs = 0; mask = 0; ++tile;
                }
            node += v > 0 ? v : g.V;
        }
    }
    // the batch table: tile starts, then per graph its id, offsets and per-type message bases (type base of the batch + earlier graphs')
    const int rec = ds::R_MBASE + T;
    b->off_records = align_up(sizeof(int) * tile_start.size(), 16);
    b->off_slots = align_up(b->off_records + sizeof(int) * (size_t)rec * G, 16);
    b->table_bytes = b->off_slots + sizeof(int) * (size_t)G;
    CU_TRY(b, b->table.begin(std::max<size_t>(b->table_bytes, 16)));
    memcpy(b->table.ptr, tile_start.data(), sizeof(int) * tile_start.size());
    int* r = (int*)(b->table.ptr + b->off_records);
    std::vector<int64_t> mbase(T, 0);
    for (int t = 1; t < T; ++t) mbase[t] = mbase[t - 1] + type_tot[t - 1];
    int64_t node = 0, slot = 0, vrow = 0, vs = 0;
    for (int i = 0; i < G; ++i, r += rec) {
        const DsGraph& g = d->graphs[graph_ids[i]];
        r[ds::R_GID] = (int)graph_ids[i]; r[ds::R_NODE] = (int)node; r[ds::R_SLOT] = (int)slot; r[ds::R_VROW] = (int)vrow; r[ds::R_VSRC] = (int)vs;
        for (int t = 0; t < T; ++t) {
            r[ds::R_MBASE + t] = (int)mbase[t];
            mbase[t] += d->type_msgs[(size_t)graph_ids[i] * T + t];
        }
        node += v > 0 ? v : g.V; slot += g.M; vrow += g.nv; vs += g.nvm;
    }
    int* slots = (int*)(b->table.ptr + b->off_slots);   // the slot map of ggnn_readout_predict: batch graph i -> its dataset index
    for (int i = 0; i < G; ++i) slots[i] = (int)graph_ids[i];
    b->G = G;
    b->valid = true;
    return GGNN_OK;
}

extern "C" {

int ggnn_dataset_prepare_batch(const ggnn_dataset* d, int32_t save_for_backward, const int64_t* graph_ids, int32_t num_graphs,
                               ggnn_dataset_batch** inout) {
    return prepare_dataset_batch(d, save_for_backward, graph_ids, num_graphs, false, 0, inout);
}

int ggnn_dataset_prepare_batch_dense(const ggnn_dataset* d, int32_t save_for_backward, const int64_t* graph_ids, int32_t num_graphs,
                                     int32_t nodes_per_graph, ggnn_dataset_batch** inout) {
    return prepare_dataset_batch(d, save_for_backward, graph_ids, num_graphs, true, nodes_per_graph, inout);
}

int ggnn_dataset_batch_info(const ggnn_dataset_batch* b, int32_t* num_nodes, int64_t* num_messages, int32_t* num_tiles, int64_t* image_bytes,
                            int32_t* is_streaming, char* plan_text, int32_t plan_text_capacity, int32_t* tile_start, int32_t* max_tile_msgs,
                            int32_t* max_tile_types) {
    if (!b || !b->valid) return GGNN_ESTATE;
    report_plan(b->plan, b->bytes, num_nodes, num_messages, num_tiles, image_bytes, is_streaming, plan_text, plan_text_capacity, max_tile_msgs,
                max_tile_types);
    if (tile_start) memcpy(tile_start, b->table.ptr, sizeof(int) * (size_t)(b->plan.ntiles + 1));
    return GGNN_OK;
}

int ggnn_free_dataset_batch(ggnn_dataset_batch* b) {
    if (!b) return GGNN_OK;
    if (b->table.use_cuda) { cudaSetDevice(b->shape.device); b->table.release(); }
    delete b;
    return GGNN_OK;
}

const char* ggnn_dataset_batch_error(const ggnn_dataset_batch* b) { return b ? b->err.c_str() : "null dataset batch"; }

}  // extern "C"

// The device half of both batch kinds: node_mask is the dense call's [V] output (null for the sparse call, which refuses a dense batch).
static int set_graph_dataset(ggnn_engine* e, ggnn_dataset_batch* b, float* h0, float* target_values, float* target_mask, bool dense,
                             float* node_mask, ggnn_stream_t stream) {
    if (!e) return GGNN_EINVAL;
    forget_batch(e);
    if (!b || !b->valid) return e->fail(GGNN_ESTATE, "the dataset batch is empty (its prepare failed or never ran)");
    if ((b->v > 0) != dense)
        return e->fail(GGNN_EINVAL, dense ? "ggnn_set_graph_dataset_dense needs a dense dataset batch" : "a dense dataset batch is adopted with ggnn_set_graph_dataset_dense");
    const ggnn_dataset* d = b->ds;
    if (!d->on_device) return e->fail(GGNN_EINVAL, "a host-only dataset has no device copy");
    if (int rc = check_batch_shape(e, b->shape, b->plan, "dataset")) return rc;
    if (b->shape.device != e->device)   // its arrays live in another GPU's memory
        return e->fail(GGNN_EINVAL, "the dataset was built for an engine on device %d, this engine is on device %d", b->shape.device, e->device);
    const BatchPlan& q = b->plan;
    if ((q.V > 0 && (!h0 || (dense && !node_mask))) || (d->tasks > 0 && b->G > 0 && (!target_values || !target_mask)))
        return e->fail(GGNN_EINVAL, "null output buffer");
    CU_TRY(e, cudaSetDevice(e->device));
    cudaStream_t st = (cudaStream_t)stream;
    static_cast<BatchPlan&>(*e) = q;
    CU_TRY(e, e->graph_buf.reserve(b->bytes));
    e->graph_bytes = b->bytes;
    CU_TRY(e, e->ds_table.reserve(std::max<size_t>(b->table_bytes, 16)));
    const size_t ro_bytes = readout_layout(e, q.V, b->G);
    CU_TRY(e, e->ro_buf.reserve(align_up(ro_bytes + sizeof(float) * (size_t)std::max(q.V, 1), 16)));
    CU_TRY(e, b->table.upload(e->ds_table.ptr, b->table_bytes, st));
    CU_TRY(e, cudaMemsetAsync(e->graph_buf.ptr, 0, b->bytes, st));   // the alignment gaps, as in a fresh host image
    CU_TRY(e, cudaMemsetAsync(e->ro_buf.ptr, 0, e->ro_off_perm, st));
    ds::DsOut o;
    o.img = image_view(q, e->use_att, (char*)e->graph_buf.ptr);
    o.h0 = h0; o.tv = target_values; o.tm = target_mask;
    o.ro_graph_of = (int*)((char*)e->ro_buf.ptr + e->ro_off_graph_of); o.ro_start = (int*)((char*)e->ro_buf.ptr + e->ro_off_start);
    o.node_mask = node_mask; o.ro_mask = dense ? (float*)((char*)e->ro_buf.ptr + e->ro_off_mask) : nullptr;
    o.V = q.V; o.D = e->D; o.T = e->T; o.G = b->G; o.ntiles = q.ntiles; o.nv = q.ts_nv; o.rec = ds::R_MBASE + e->T; o.v = b->v;
    const int* table = (const int*)((const char*)e->ds_table.ptr + b->off_records);
    if (b->G > 0) ds::ds_graph_kernel<<<b->G, 256, 0, st>>>(d->dev, o, table);
    const int tile_work = std::max(q.ntiles + 1, q.stream ? ts::TILE_M * e->T : 0);
    ds::ds_tile_kernel<<<std::min(e->num_sms * 4, (tile_work + 255) / 256), 256, 0, st>>>(
        d->dev, o, table, (const int*)e->ds_table.ptr);
    CU_TRY(e, cudaGetLastError());
    if (int rc = bind_graph(e)) return rc;
    e->ro_V = q.V; e->ro_G = b->G; e->ro_grouped = true; e->ro_has_mask = dense;
    e->ro_from_dataset = true; e->ro_dataset_slots = (const int*)((const char*)e->ds_table.ptr + b->off_slots);
    return GGNN_OK;
}

extern "C" {

int ggnn_set_graph_dataset(ggnn_engine* e, ggnn_dataset_batch* b, float* h0, float* target_values, float* target_mask, ggnn_stream_t stream) {
    return set_graph_dataset(e, b, h0, target_values, target_mask, false, nullptr, stream);
}

int ggnn_set_graph_dataset_dense(ggnn_engine* e, ggnn_dataset_batch* b, float* h0, float* target_values, float* target_mask, float* node_mask,
                                 ggnn_stream_t stream) {
    return set_graph_dataset(e, b, h0, target_values, target_mask, true, node_mask, stream);
}

int ggnn_graph_image(ggnn_engine* e, void* dst, int64_t capacity, int64_t* image_bytes, ggnn_stream_t stream) {
    if (!e) return GGNN_EINVAL;
    if (!e->graph_set) return no_graph(e);
    if (image_bytes) *image_bytes = (int64_t)e->graph_bytes;
    if (!dst) return GGNN_OK;
    if (capacity < (int64_t)e->graph_bytes) return e->fail(GGNN_EINVAL, "the image has %zu bytes, the buffer %lld", e->graph_bytes, (long long)capacity);
    CU_TRY(e, cudaSetDevice(e->device));
    CU_TRY(e, cudaMemcpyAsync(dst, e->graph_buf.ptr, e->graph_bytes, cudaMemcpyDeviceToHost, (cudaStream_t)stream));
    CU_TRY(e, cudaStreamSynchronize((cudaStream_t)stream));
    return GGNN_OK;
}

}  // extern "C"
