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
    int use_att = 0;    // use_propagation_attention (sparse:170-196): fp32 path only
    int num_sms = 132;
    size_t max_smem = 0;
};

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
    size_t off_slotw = 0, off_tslotw = 0;   // weighted: per-slot adjacency weights in target-CSR order / source-CSR order (with the transpose)
};

// Typed device pointers into the uploaded graph image of the current batch, made once per upload by ggnn_set_graph_prepared.  An array
// the plan does not carry points at the start of the image.
struct GraphDev {
    const int *row_ptr, *csr_src, *csr_msg;
    const float *indeg, *denom;
    const int* tile_start;
    const unsigned* tile_mask;
    const int *trow, *ttgt, *tslot;                      // source-keyed CSR (save_for_backward)
    const int *pair_src, *vrow_ptr, *vsrc, *tile_vptr;   // streaming plan
    const int4* vinfo;
    const float *slot_w, *tslot_w;                       // weighted batches: per-slot adjacency weights
};

// The weights in the pre-split, pre-tiled bf16 layout of one tensor-core kernel family, with each layer's offsets.  The tiles are rebuilt
// when the weights changed since they were made (ggnn_set_weights / ggnn_gcn_set_weights bump the engine's weights generation) or when
// the layout changed, and at no other time.
struct WeightTiles {
    DevBuf buf;
    size_t off_edge[MAX_LAYERS] = {0}, off_gate[MAX_LAYERS] = {0}, off_cand[MAX_LAYERS] = {0};
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

    // device memory
    DevBuf graph_buf;   // the graph image of the current batch
    GraphDev gd;        // ... and the view of it every driver reads
    // readout (gated_regression): node -> graph map of the current batch
    DevBuf ro_buf; StagedImage ro_stage;
    int ro_V = -1, ro_G = 0; bool ro_grouped = false, ro_has_mask = false;
    size_t ro_off_graph_of = 0, ro_off_start = 0, ro_off_mask = 0, ro_off_val = 0;
    size_t ro_off_perm = 0;   // ungrouped lists: the stable by-graph node permutation (graph g owns perm[start[g] .. start[g+1]))
    DevBuf ro_ws;             // deterministic readout backward: per-block partials of the weight gradients
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
    const GraphDev& gd = e->gd;
    p.tile_start = gd.tile_start; p.tile_mask = gd.tile_mask; p.row_ptr = gd.row_ptr; p.csr_src = gd.csr_src;
    p.slot_w = e->weighted ? gd.slot_w : nullptr; p.indeg = gd.indeg; p.denom = gd.denom;
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
    e->graph_set = false; e->saved_valid = false;
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

// The tile plan of a batch of V nodes: which kernel, and the tiles.  `cuts` are the sorted node indices where the batch may be split
// between connected components (cuts.front() == 0, cuts.back() == V); `weighted`: every message has a weight.  Starts `p` afresh; the image
// builders fill in the rest.
int build_plan(const ModelShape& s, int V, bool weighted, const std::vector<int>& cuts, BatchPlan& p, std::vector<int>& tile_start,
               std::string& err) {
    p = BatchPlan();
    p.V = V;
    p.weighted = weighted;
    int max_span = 0;
    for (size_t i = 1; i < cuts.size(); ++i) max_span = std::max(max_span, cuts[i] - cuts[i - 1]);
    p.max_span = max_span;
    const char* fg = getenv("GGNN_FORCE_GLOBAL");
    const bool force_global = fg && fg[0] == '1';
    const char* prec = s.precision == GGNN_PREC_BF16X3 ? "bf16x3" : "bf16";
    char buf[256];
    if (s.model == MODEL_GCN) {
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
        // The streaming kernels sum unweighted messages only: a weighted batch stays on the tile kernel.
        const bool big_component = max_span > tc::TILE_M && !weighted && !force_global && !(fs && fs[0] == '0');
        if (s.DP > 128 || big_component || (fs && fs[0] == '1' && !weighted)) {
            // streaming plan: fixed 128-row tiles (the gather reads the previous state from L2, so tiles need not respect components),
            // one launch per GEMM of a timestep; N blocks sized so that small batches still spread over the chip
            if (weighted) {
                err = "hidden_size > 128 on the tensor-core path needs unweighted messages (a weighted dense adjacency runs on GGNN_PREC_FP32)";
                return GGNN_EUNSUPPORTED;
            }
            p.stream = true; p.variant = 3;
            fixed_tiles(V, ts::TILE_M, tile_start);
            p.ntiles = (int)tile_start.size() - 1;
            for (int i = 0; i < 2; ++i) {
                const int width = (i + 1) * s.DP;
                // one wgmma accumulator of MMA_N columns per CTA (the MMA warpgroup holds both 64-row halves in registers)
                p.ts_nblk[i] = (width + ts::MMA_N - 1) / ts::MMA_N;
                p.ts_nc[i] = ts::MMA_N;
            }
            int len = snprintf(buf, sizeof buf, "wgmma-%s STREAM(3 launches per step: gather-GEMM, gate GEMM, candidate GEMM) tiles=%d DP=%d N-blocks agg/cand=%dx%d gate=%dx%d",
                               prec, p.ntiles, s.DP, p.ts_nblk[0], p.ts_nc[0], p.ts_nblk[1], p.ts_nc[1]);
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

static int ggnn_backward_impl(ggnn_engine* e, const float* d_h_out, const ggnn_layer_grads* grads, int32_t num_layers,
                              float* d_h0, ggnn_stream_t stream) {
    using namespace ggnn::bwd;
    if (int rc = begin_backward(e, "ggnn_backward", "ggnn_set_graph_sparse", d_h_out, grads, num_layers, d_h0)) return rc;
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
    const size_t o_pall = take(e->use_att ? vd * T : 0), o_dsa = take(e->use_att ? (size_t)std::max<int64_t>(e->M, 1) : 0);
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
    CU_TRY(e, cudaMemsetAsync(dstate, 0, vd * L * sizeof(float), st));
    CU_TRY(e, cudaMemcpyAsync(dstate + vd * L, d_h_out, vd * sizeof(float), cudaMemcpyDeviceToDevice, st));
    // forward values of node_states_per_layer
    std::vector<const float*> fstate(L + 1);
    for (int l = 0; l <= L; ++l) fstate[l] = layer_state(e, l, e->last_h0, e->last_out);
    const GraphDev& gd = e->gd;
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
            GatherJob j0{gd.row_ptr, gd.csr_src, h, At, nullptr, nullptr}, j1{gd.trow, gd.ttgt, dxp, Gt, nullptr, nullptr};
            if (e->use_att) {   // softmax backward first (it adds to dh_new), then the gathers are weighted by the probabilities
                const float* alpha = (const float*)e->att_buf.ptr + (size_t)(e->step_base[l] + s) * (size_t)std::max<int64_t>(e->M, 1);
                gemm_nt(false, dxp, D, 0, w.edge_weights, D, 0, 1, Pall, TD, V, TD, D);   // P[v, t*D+k] = <dx'[v], W_t[k, :]>
                // the target kernel holds 8 columns of d h[v] per lane up to hidden 256, 16 above
                if (e->det && gw.edge_type_attention_weights) {   // per-block d a_t into ws, then added over the blocks in a fixed order
                    (D <= 256 ? attention_bwd_target_ordered_kernel<8> : attention_bwd_target_ordered_kernel<16>)<<<nodes_blocks, 256, 0, st>>>(
                        gd.row_ptr, gd.csr_src, h, Pall, alpha, w.edge_type_attention_weights, dsa, dh_new, ws, V, D, T);
                    ordered_colsum_kernel<<<T, 256, 0, st>>>(ws, nodes_blocks, T, gw.edge_type_attention_weights);
                    ++e->last_launches;
                } else {
                    (D <= 256 ? attention_bwd_target_kernel<8> : attention_bwd_target_kernel<16>)<<<nodes_blocks, 256, 0, st>>>(
                        gd.row_ptr, gd.csr_src, h, Pall, alpha, w.edge_type_attention_weights, dsa, dh_new, gw.edge_type_attention_weights, V, D, T);
                }
                attention_bwd_source_kernel<<<nodes_blocks, 256, 0, st>>>(gd.trow, gd.ttgt, gd.tslot, h, dsa, dh_new, V, D, T);
                e->last_launches += 2;
                j0.w = j1.w = alpha;
                j1.widx = gd.tslot;
            } else if (e->weighted) {
                j0.w = gd.slot_w;
                j1.w = gd.tslot_w;
            }
            csr_gather_all_kernel<<<dim3(nodes_blocks, 2), 256, 0, st>>>(j0, j1, V, D, T);
            ++e->last_launches;
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
    if (d_h0) CU_TRY(e, cudaMemcpyAsync(d_h0, dstate, vd * sizeof(float), cudaMemcpyDeviceToDevice, st));
    CU_TRY(e, cudaGetLastError());
    return GGNN_OK;
}

// ------------------------------------------------------------------------------------------ C ABI
extern "C" {

const char* ggnn_last_error(const ggnn_engine* e) { return e ? e->err.c_str() : g_create_error.c_str(); }

// The checks and fields both model configs have; no CUDA (the text goes to `err`: this may run in any thread).
// `max_hidden`: the widest hidden size of the model's kernels (GGNN 512: the readout and the attention backward hold 16 columns per lane;
// GCN 256: its fp32 kernel).
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
    if (cfg->cell != GGNN_CELL_GRU && cfg->cell != GGNN_CELL_RNN && cfg->cell != GGNN_CELL_CUDNN_GRU) return bad("Unknown RNN cell type");   // sparse:112
    if (cfg->cell == GGNN_CELL_CUDNN_GRU && cfg->activation != GGNN_ACT_TANH) return bad("CudnnCompatibleGRUCell requires the tanh activation");   // sparse:106
    if (cfg->activation != GGNN_ACT_TANH && cfg->activation != GGNN_ACT_RELU) return bad("Unknown activation function type");  // sparse:81
    s.T = cfg->num_edge_types;
    s.use_bias = cfg->use_edge_bias != 0; s.use_avg = cfg->use_edge_msg_avg_aggregation != 0;
    s.cell = cfg->cell; s.act = cfg->activation;
    s.use_att = cfg->use_propagation_attention != 0;
    if (s.use_att && s.T > 16) { err = "propagation attention supports at most 16 edge types"; return GGNN_EUNSUPPORTED; }
    if (s.use_att) s.precision = GGNN_PREC_FP32;   // the softmax-weighted gather lives in the fp32 kernel only (the plan text says so)
    if (s.cell == CELL_CUDNN_GRU) s.precision = GGNN_PREC_FP32;   // so does the reset-after-matmul candidate of CudnnCompatibleGRUCell
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
    if (int rc = init_common_shape(s, cfg->hidden_size, 256, cfg->num_layers, cfg->precision, cfg->device, err)) return rc;
    s.model = MODEL_GCN;
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
    e->graph_buf.release(); e->state_buf.release(); e->save_bufs.release(); e->io_buf.release(); e->bwd_buf.release();
    e->tc_tiles.buf.release(); e->tc_respre.release(); e->ts_tiles.buf.release(); e->ts_images.release(); e->ts_virt.release(); e->err_flag.release();
    e->step_wt.buf.release(); e->step_buf.release();
    if (e->own_prep) { ggnn_free_prepared_graph(e->own_prep); e->own_prep = nullptr; }
    e->ro_buf.release(); e->ro_stage.release(); e->att_buf.release(); e->ro_ws.release();
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
// their sources (vinfo: count + the first seven inline; vptr / vsrc: the complete lists).  `pair` already holds -1 / the single source.
static void number_virtual_rows(int ntiles, int T, const int* tile_start, const int* row_ptr, const int* csr_src, int* pair, int* vptr, int* vsrc,
                                int* tvp, int* vinfo) {
    int vid = 0, vm = 0;
    vptr[0] = 0;
    for (int i = 0; i < ntiles; ++i) {
        tvp[i] = vid;
        for (size_t k = (size_t)tile_start[i] * T, kend = (size_t)tile_start[i + 1] * T; k < kend; ++k) {
            if (pair[k] != -2) continue;
            const int b = row_ptr[k], cnt = row_ptr[k + 1] - b;
            pair[k] = -(2 + vid);
            if (vinfo) {
                vinfo[8 * vid] = cnt;
                for (int m = 0; m < 7; ++m) vinfo[8 * vid + 1 + m] = m < cnt ? csr_src[b + m] : 0;
            }
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
    s.D = hidden_size; s.T = num_edge_types; s.precision = precision; s.num_sms = num_sms; s.max_smem = 227 * 1024;
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
    number_virtual_rows(ntiles, T, tile_start.data(), row_ptr.data(), src.data(), pair_src, vrow_ptr, vsrc, tile_vptr, nullptr);
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

// ---- the host half of ggnn_set_graph_sparse: validation, tile plan, stable target-sorted CSR, streaming tables -> g->image.
// `weighted`: the batch has one weight per message, `w`, in the type-major message order (required when there are messages); the image
// then carries them in target-CSR order and, with the source-keyed CSR, in source-CSR order.
// Nothing here touches the device except the pinned allocation of the image and the wait for the previous upload out of it.
static int build_sparse_image(ggnn_prepared_graph* g, int32_t V, const int32_t* const* adj, const int32_t* num_edges, const float* indeg,
                              bool weighted, const float* w) {
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
    if (weighted && M > 0 && !w) return g->fail(GGNN_EINVAL, "null message weights");

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
    // plans; the streaming plan of hidden sizes > 128 and the per-timestep fp32 path above 256 tile by fixed 128-row blocks and skip that part)
    std::vector<int>& counts = g->h_counts;
    std::vector<int>& reach = g->h_diff;   // reach[j] = the farthest node an edge whose lower end is node j touches
    const bool need_cuts = shape.precision == GGNN_PREC_FP32 ? shape.D <= 256 : shape.DP <= 128;
    counts.resize((size_t)V * T + 1);
    if (need_cuts) reach.resize((size_t)V + 1);
    std::vector<int64_t> type_base(T + 1, 0);   // position of every type's first message in the reference's type-major message order
    for (int t = 0; t < T; ++t) type_base[t + 1] = type_base[t] + num_edges[t];
    int bad_edge = 0;
    // Pass 1 is split by EDGE ranges: counting is commutative, so the threads add into the shared per-row counts with relaxed atomic
    // increments (and an atomic max for `reach`) -- same totals for every thread count; a single thread uses plain increments.
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
            std::fill(counts.begin() + c0, counts.begin() + c1, 0);
            if (need_cuts) {
                const size_t nr = (size_t)V + 1, r0 = nr * k / n, r1 = nr * (k + 1) / n;
                std::fill(reach.begin() + r0, reach.begin() + r1, 0);
            }
        }
#ifdef _OPENMP
#pragma omp barrier
#endif
        const int64_t e0 = M * k / n, e1 = M * (k + 1) / n;   // this thread's messages, in the type-major order
        int* const cnt = counts.data();
        int* const rch = need_cuts ? reach.data() : nullptr;
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
    if (bad_edge) {   // name the first offending edge, like the single pass did
        for (int t = 0; t < T; ++t)
            for (int i = 0; i < num_edges[t]; ++i) {
                const int s = adj[t][2 * i], d = adj[t][2 * i + 1];
                if ((unsigned)s >= (unsigned)V || (unsigned)d >= (unsigned)V)
                    return g->fail(GGNN_ERANGE, "edge %d of type %d = (%d,%d) is out of range for %d nodes", i, t, s, d, V);
            }
    }
    lap("  edges pass 1", t_lap);
    std::vector<int> cuts;
    find_cuts(need_cuts ? reach.data() : nullptr, V, cuts);
    lap("validate+count", t_lap);
    std::vector<int> tile_start;
    int rc = build_plan(shape, V, weighted, cuts, p, tile_start, g->err);
    if (rc) return rc;
    p.M = M;
    const int ntiles = p.ntiles;
    lap("tile plan", t_lap);
    nth = std::max(1, std::min(nth, ntiles));
    // tile ranges of the threads for all later passes: tiles [tb[k], tb[k+1]), i.e. nodes [tile_start[tb[k]], tile_start[tb[k+1]])
    std::vector<int> tb(nth + 1);
    for (int k = 0; k <= nth; ++k) tb[k] = (int)((int64_t)ntiles * k / nth);
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
                if (c >= 2) { ++nv; nvm += c; }
            }
        } else {
            for (size_t r = k0; r < k1; ++r) sm += counts[r + 1];
        }
        part_msgs[k + 1] = sm; part_nv[k + 1] = nv; part_nvm[k + 1] = nvm;
    }
    for (int k = 0; k < nth; ++k) { part_msgs[k + 1] += part_msgs[k]; part_nv[k + 1] += part_nv[k]; part_nvm[k + 1] += part_nvm[k]; }

    // ---- layout of the packed upload
    size_t off = 0;
    p.off_row_ptr = off; off = align_up(off + sizeof(int) * ((size_t)V * T + 1), 16);
    p.off_src = off;     off = align_up(off + sizeof(int) * (size_t)std::max<int64_t>(M, 1), 16);
    p.off_msg = off;     off = align_up(off + sizeof(int) * (size_t)std::max<int64_t>(M, 1), 16);
    p.off_indeg = off;   off = align_up(off + sizeof(float) * (size_t)std::max(V, 1) * T, 16);
    p.off_denom = off;   off = align_up(off + sizeof(float) * (size_t)std::max(V, 1), 16);
    p.off_tiles = off;   off = align_up(off + sizeof(int) * (size_t)(ntiles + 1), 16);
    p.off_mask = off;    off = align_up(off + sizeof(unsigned) * (size_t)std::max(ntiles, 1), 16);
    p.has_transpose = g->save;
    if (p.has_transpose) {
        p.off_trow = off; off = align_up(off + sizeof(int) * ((size_t)V * T + 1), 16);
        p.off_ttgt = off; off = align_up(off + sizeof(int) * (size_t)std::max<int64_t>(M, 1), 16);
        p.off_tslot = off;
        if (shape.use_att) off = align_up(off + sizeof(int) * (size_t)std::max<int64_t>(M, 1), 16);
    }
    // streaming plan: per (target, type) pair the ONE node to copy from (or none / a virtual row), see ggnn_fwd_stream.cuh
    const int nv = (int)part_nv[nth];
    const int64_t nvm = part_nvm[nth];
    if (p.stream) {
        p.off_pair = off; off = align_up(off + sizeof(int) * (size_t)std::max(ntiles, 1) * ts::TILE_M * T, 16);
        p.off_vptr = off; off = align_up(off + sizeof(int) * (size_t)(nv + 1), 16);
        p.off_vsrc = off; off = align_up(off + sizeof(int) * (size_t)std::max<int64_t>(nvm, 1), 16);
        p.off_tvp = off;  off = align_up(off + sizeof(int) * (size_t)(ntiles + 1), 16);
        p.off_vinfo = off; off = align_up(off + sizeof(int) * 8 * (size_t)std::max(nv, 1), 16);
    }
    if (p.weighted) {   // per-slot adjacency weights
        p.off_slotw = off; off = align_up(off + sizeof(float) * (size_t)std::max<int64_t>(M, 1), 16);
        if (p.has_transpose) { p.off_tslotw = off; off = align_up(off + sizeof(float) * (size_t)std::max<int64_t>(M, 1), 16); }
    }
    p.ts_nv = nv;
    CU_TRY(g, g->image.begin(off));
    g->bytes = off;
    char* base = g->image.ptr;
    int* row_ptr = (int*)(base + p.off_row_ptr);
    int* csr_src = (int*)(base + p.off_src);
    int* csr_msg = (int*)(base + p.off_msg);
    float* h_indeg = (float*)(base + p.off_indeg);
    float* h_denom = (float*)(base + p.off_denom);
    int* h_tiles = (int*)(base + p.off_tiles);
    unsigned* h_mask = (unsigned*)(base + p.off_mask);
    int* pair = p.stream ? (int*)(base + p.off_pair) : nullptr;   // streaming plan: (target, type) -> its one source / virtual row
    int* vptr = p.stream ? (int*)(base + p.off_vptr) : nullptr;
    int* vsrc = p.stream ? (int*)(base + p.off_vsrc) : nullptr;
    int* tvp = p.stream ? (int*)(base + p.off_tvp) : nullptr;
    int* vinfo = p.stream ? (int*)(base + p.off_vinfo) : nullptr;
    lap("stage reserve", t_lap);

    // ---- pass 2, per thread over its tile range: exclusive scan of the (target, type) rows -> row_ptr, fill cursors, the tiles'
    // edge-type masks and the largest per-tile message count; then the stable fill -- every thread walks the
    // lists in the reference's order (type-major, then list order, sparse:124-129) and places the messages of ITS rows, so within a row
    // they stay in message order: this IS NumPy's stable argsort by target, tests pin it bit for bit; then (streaming plan) the gather
    // table and the virtual rows of its range, numbered from the range's offset; then in-degrees / denominators of its nodes.
    std::vector<int>& cursor = g->h_cursor;   // next free slot of every (target, type) row (its own array: the counts of a range's last
    cursor.resize((size_t)V * T + 1);         // row are read by one thread while the next range's thread already writes cursors)
    int max_tile_msgs = 0, max_tile_types = 0;
    row_ptr[0] = 0;
    if (vptr) vptr[0] = 0;
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
                    row_ptr[r + t + 1] = run;
                    mask |= (unsigned)(c > 0) << t;
                }
            h_mask[i] = mask;
            max_tile_msgs = std::max(max_tile_msgs, run - tile_first);
            max_tile_types = std::max(max_tile_types, __builtin_popcount(mask));
            h_tiles[i] = tile_start[i];
        }
        if (k == nth - 1) h_tiles[ntiles] = tile_start[ntiles];
    }
    p.max_tile_msgs = max_tile_msgs;
    p.max_tile_types = max_tile_types;
    lap("row sweep", t_lap);
#ifdef _OPENMP
#pragma omp parallel for schedule(static, 1) num_threads(nth) if (nth > 1)
#endif
    for (int k = 0; k < nth; ++k) {
        const int v0 = tile_start[tb[k]], v1 = tile_start[tb[k + 1]];
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
        if (pair) {   // one sequential pass over the range's rows: no message -> -1, one -> its source, several -> virtual row
            int vid = (int)part_nv[k], vm = (int)part_nvm[k];
            for (int i = tb[k]; i < tb[k + 1]; ++i) {
                tvp[i] = vid;
                size_t r = (size_t)tile_start[i] * T;
                const size_t rend = (size_t)tile_start[i + 1] * T, rpad = (size_t)(i + 1) * ts::TILE_M * T;
                for (; r < rend; ++r) {
                    const int b = row_ptr[r], cnt = row_ptr[r + 1] - b;
                    if (cnt == 0) pair[r] = -1;
                    else if (cnt == 1) pair[r] = csr_src[b];
                    else {
                        pair[r] = -(2 + vid);
                        vinfo[8 * vid] = cnt;
                        for (int m = 0; m < 7; ++m) vinfo[8 * vid + 1 + m] = m < cnt ? csr_src[b + m] : 0;
                        for (int m = 0; m < cnt; ++m) vsrc[vm++] = csr_src[b + m];
                        vptr[++vid] = vm;
                    }
                }
                for (; r < rpad; ++r) pair[r] = -1;   // rows of the last tile beyond V
            }
            if (k == nth - 1) tvp[ntiles] = vid;
        }
        if (weighted) {   // the weights of this range's slots, in target-CSR order
            float* slotw = (float*)(base + p.off_slotw);
            for (int64_t m = part_msgs[k]; m < part_msgs[k + 1]; ++m) slotw[m] = w[csr_msg[m]];
        }
        if (v1 > v0) memcpy(h_indeg + (size_t)v0 * T, indeg + (size_t)v0 * T, sizeof(float) * (size_t)(v1 - v0) * T);
        for (int v = v0; v < v1; ++v) {
            const float* row = indeg + (size_t)v * T;
            float s = 0.0f;  // tf.reduce_sum over the type axis in fp32 (sparse:207), then + SMALL_NUMBER (:209)
            for (int t = 0; t < T; ++t) s += row[t];
            h_denom[v] = s + 1e-7f;
        }
    }
    if (ntiles == 0) {
        h_tiles[0] = 0;
        if (pair) { for (size_t r = 0; r < (size_t)ts::TILE_M * T; ++r) pair[r] = -1; tvp[0] = 0; }
    }
    lap("csr fill", t_lap);
    if (p.has_transpose) {   // messages keyed by (source, type): the scatter of the backward pass becomes a gather
        int* trow = (int*)(base + p.off_trow);
        int* ttgt = (int*)(base + p.off_ttgt);
        std::vector<int> cnt((size_t)V * T + 1, 0);
        for (int t = 0; t < T; ++t)
            for (int i = 0; i < num_edges[t]; ++i) ++cnt[(size_t)adj[t][2 * i] * T + t + 1];
        trow[0] = 0;
        for (size_t k = 1; k <= (size_t)V * T; ++k) trow[k] = trow[k - 1] + cnt[k];
        for (size_t k = 0; k < (size_t)V * T; ++k) cnt[k] = trow[k];
        std::vector<int> slot_of_msg;
        int* tslot = shape.use_att ? (int*)(base + p.off_tslot) : nullptr;
        float* tslotw = weighted ? (float*)(base + p.off_tslotw) : nullptr;
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
                if (tslotw) tslotw[j] = w[m];
            }
    }
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

// The prologue of the six prepare calls: reuse or allocate *inout and give it a model shape.  With an engine `e` (which must be a
// `model` engine, the model of Config), the shape and -- for save_for_backward = -1 -- the save flag are the engine's, and the image
// is pinned on its device; without one, the shape comes from `cfg` for a host of `num_sms` SMs with 227 KiB of shared memory each,
// and the image is plain memory.
template <class Config>
static int begin_prepare(ggnn_prepared_graph** inout, const ggnn_engine* e, const Config* cfg, int32_t num_sms, int32_t save_for_backward,
                         const char* fn) {
    constexpr int model = std::is_same<Config, ggnn_gcn_config>::value ? MODEL_GCN : MODEL_GGNN;
    if (!inout || (!e && (!cfg || num_sms <= 0))) return GGNN_EINVAL;
    ggnn_prepared_graph* g = *inout;
    if (!g) { g = new ggnn_prepared_graph(); *inout = g; }
    g->valid = false;
    g->image.use_cuda = e != nullptr;
    if (e) {
        g->shape = *e;
        if (e->model != model) return wrong_model(g, fn, e->model, model);
        g->save = save_for_backward >= 0 ? save_for_backward != 0 : e->save;   // a producer thread says what the batch will be used for
        if (cudaSetDevice(e->device) != cudaSuccess) return g->fail(GGNN_ECUDA, "cudaSetDevice(%d) failed", e->device);   // this may be a producer thread
        return GGNN_OK;
    }
    g->shape = ModelShape();
    int rc;
    if constexpr (model == MODEL_GCN) rc = init_gcn_shape(g->shape, cfg, g->err);
    else rc = init_model_shape(g->shape, cfg, g->err);
    if (rc) return rc;
    g->shape.num_sms = num_sms; g->shape.max_smem = 227 * 1024;
    g->save = save_for_backward != 0;
    return GGNN_OK;
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
    if (num_nodes) *num_nodes = g->plan.V;
    if (num_messages) *num_messages = g->plan.M;
    if (num_tiles) *num_tiles = g->plan.ntiles;
    if (image_bytes) *image_bytes = (int64_t)g->bytes;
    if (is_streaming) *is_streaming = g->plan.stream ? 1 : 0;
    if (plan_text && plan_text_capacity > 0) snprintf(plan_text, (size_t)plan_text_capacity, "%s", g->plan.plan_text.c_str());
    return GGNN_OK;
}

int ggnn_prepared_graph_arrays(const ggnn_prepared_graph* g, int32_t* row_ptr, int32_t* src, int32_t* msg, int32_t* tile_start, float* denom,
                               int32_t* pair_src) {
    if (!g || !g->valid) return GGNN_ESTATE;
    const BatchPlan& q = g->plan;
    const char* base = g->image.ptr;
    const size_t V = (size_t)q.V, T = (size_t)g->shape.T, M = (size_t)q.M;
    if (row_ptr) memcpy(row_ptr, base + q.off_row_ptr, sizeof(int) * (V * T + 1));
    if (src && M) memcpy(src, base + q.off_src, sizeof(int) * M);
    if (msg && M) memcpy(msg, base + q.off_msg, sizeof(int) * M);
    if (tile_start) memcpy(tile_start, base + q.off_tiles, sizeof(int) * (size_t)(q.ntiles + 1));
    if (denom && V) memcpy(denom, base + q.off_denom, sizeof(float) * V);
    if (pair_src && q.stream) memcpy(pair_src, base + q.off_pair, sizeof(int) * (size_t)std::max(q.ntiles, 1) * ts::TILE_M * T);
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

int ggnn_set_graph_prepared(ggnn_engine* e, ggnn_prepared_graph* g, ggnn_stream_t stream) {
    if (!e) return GGNN_EINVAL;
    forget_batch(e);
    if (!g || !g->valid) return e->fail(GGNN_ESTATE, "the prepared graph is empty (its build failed or never ran)");
    const ModelShape& q = g->shape;
    if (q.model != e->model)
        return e->fail(GGNN_ESTATE, "the prepared graph was built for a %s engine, this is a %s engine", q.model == MODEL_GCN ? "GCN" : "GGNN",
                       e->model == MODEL_GCN ? "GCN" : "GGNN");
    if (q.D != e->D || q.T != e->T || q.precision != e->precision || q.DP != e->DP || q.num_sms != e->num_sms || q.cell != e->cell || q.use_att != e->use_att)
        return e->fail(GGNN_EINVAL, "the prepared graph was built for a different engine configuration");
    if (e->save && !g->plan.has_transpose)
        return e->fail(GGNN_ESTATE, "save_for_backward is on but the graph was prepared without it (the source-keyed CSR is built at prepare time)");
    CU_TRY(e, cudaSetDevice(e->device));
    static_cast<BatchPlan&>(*e) = g->plan;
    CU_TRY(e, e->graph_buf.reserve(g->bytes));
    CU_TRY(e, g->image.upload(e->graph_buf.ptr, g->bytes, (cudaStream_t)stream));
    const char* b = (const char*)e->graph_buf.ptr;
    GraphDev& d = e->gd;
    d.row_ptr = (const int*)(b + e->off_row_ptr); d.csr_src = (const int*)(b + e->off_src); d.csr_msg = (const int*)(b + e->off_msg);
    d.indeg = (const float*)(b + e->off_indeg); d.denom = (const float*)(b + e->off_denom);
    d.tile_start = (const int*)(b + e->off_tiles); d.tile_mask = (const unsigned*)(b + e->off_mask);
    d.trow = (const int*)(b + e->off_trow); d.ttgt = (const int*)(b + e->off_ttgt); d.tslot = (const int*)(b + e->off_tslot);
    d.pair_src = (const int*)(b + e->off_pair); d.vrow_ptr = (const int*)(b + e->off_vptr); d.vsrc = (const int*)(b + e->off_vsrc);
    d.tile_vptr = (const int*)(b + e->off_tvp); d.vinfo = (const int4*)(b + e->off_vinfo);
    d.slot_w = (const float*)(b + e->off_slotw); d.tslot_w = (const float*)(b + e->off_tslotw);
    int rc = reserve_states(e);
    if (rc) return rc;
    e->graph_set = true;
    return GGNN_OK;
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

// Host half of ggnn_set_graph_dense: the matrix is scanned to message lists for the CSR builder.  A 0/1 matrix builds the image of its
// edge lists; a weighted one (when `weighted_ok`, else it is refused with GGNN_EUNSUPPORTED) also carries its entries as slot weights.
static int build_dense_image(ggnn_prepared_graph* g, int32_t b, int32_t v, const float* adjm, bool weighted_ok) {
    g->valid = false;
    if (b < 0 || v <= 0 || (!adjm && b > 0)) return g->fail(GGNN_EINVAL, "null/negative argument");
    if (g->shape.use_att) return g->fail(GGNN_EUNSUPPORTED, "propagation attention exists only in the sparse model (sparse:170-196)");
    const int T = g->shape.T;
    if ((int64_t)b * v > 0x7fffffff / std::max(T, 1)) return g->fail(GGNN_EUNSUPPORTED, "batch too large for int32 indexing");
    std::vector<std::vector<int32_t>> lists;
    std::vector<float> weights, indeg;
    const bool weighted = scan_dense(T, b, v, adjm, lists, weights, indeg);
    if (weighted && !weighted_ok)
        return g->fail(GGNN_EUNSUPPORTED, "the adjacency matrix is not 0/1: a weighted matrix is fed through ggnn_set_graph_dense");
    std::vector<const int32_t*> ptrs(T);
    std::vector<int32_t> counts(T);
    for (int t = 0; t < T; ++t) { ptrs[t] = lists[t].data(); counts[t] = (int32_t)(lists[t].size() / 2); }
    int rc = build_sparse_image(g, b * v, ptrs.data(), counts.data(), indeg.data(), weighted, weights.data());
    if (rc) return rc;
    g->plan.plan_text += weighted ? " [weighted dense adjacency -> weighted CSR]" : " [binary dense adjacency -> CSR]";
    return GGNN_OK;
}

int ggnn_prepare_graph_dense(const ggnn_engine* e, int32_t save_for_backward, int32_t b, int32_t v, const float* adjm, ggnn_prepared_graph** inout) {
    if (int rc = begin_prepare<ggnn_config>(inout, e, nullptr, 0, save_for_backward, __func__)) return rc;
    return build_dense_image(*inout, b, v, adjm, false);
}

int ggnn_host_prepare_graph_dense(const ggnn_config* cfg, int32_t num_sms, int32_t save_for_backward, int32_t b, int32_t v, const float* adjm,
                                  ggnn_prepared_graph** inout) {
    if (int rc = begin_prepare(inout, nullptr, cfg, num_sms, save_for_backward, __func__)) return rc;
    return build_dense_image(*inout, b, v, adjm, false);
}

int ggnn_set_graph_dense(ggnn_engine* e, int32_t b, int32_t v, const float* adjm, ggnn_stream_t stream) {
    if (!e) return GGNN_EINVAL;
    GGNN_REQUIRE_MODEL(e, MODEL_GGNN);
    return set_graph_from_own_prep(e, stream, [&](ggnn_prepared_graph** g) {
        if (int rc = begin_prepare<ggnn_config>(g, e, nullptr, 0, -1, "ggnn_set_graph_dense")) return rc;
        return build_dense_image(*g, b, v, adjm, true);
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
    const GraphDev& gd = e->gd;
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
            step::attention_kernel<<<nodes_blocks, 256, 0, st>>>(gd.row_ptr, gd.csr_src, h, w.edge_type_attention_weights, att, V, D, T);
            msg_w = att;
        }
        const GatherJob gj{gd.row_ptr, gd.csr_src, h, At, msg_w, nullptr};
        csr_gather_all_kernel<<<dim3(nodes_blocks, 1), 256, 0, st>>>(gj, gj, V, D, T);
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
static int ts_prepare_weights(ggnn_engine* e, cudaStream_t st) {
    const int D = e->D, DP = e->DP, T = e->T, NKS = DP / 16;
    const int nc0 = e->ts_nc[0], nb0 = e->ts_nblk[0], nc1 = e->ts_nc[1], nb1 = e->ts_nblk[1];
    WeightTiles& c = e->ts_tiles;
    size_t off = 0;
    for (int l = 0; l < e->L; ++l) {
        const int nseg = e->nres[l] + 2;
        c.off_edge[l] = off; off += (size_t)nb0 * T * NKS * 64 * nc0;
        c.off_gate[l] = off; off += (size_t)nb1 * nseg * NKS * 64 * nc1;
        c.off_cand[l] = off; off += (size_t)nb0 * nseg * NKS * 64 * nc0;
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
        launch(e->w[l].edge_weights, base + c.off_edge[l], T, 1, D, nc0, nb0);
        if (e->cell == CELL_GRU) launch(e->w[l].gate_kernel, base + c.off_gate[l], nseg, 2, 2 * D, nc1, nb1);
        launch(e->w[l].cand_kernel, base + c.off_cand[l], nseg, 1, D, nc0, nb0);
    }
    CU_TRY(e, cudaGetLastError());
    c.gen = e->weights_gen;
    return GGNN_OK;
}

static int forward_stream(ggnn_engine* e, const float* h0, float* h_out, cudaStream_t st) {
    const int D = e->D, DP = e->DP, T = e->T, L = e->L, V = e->V, NKS = DP / 16;
    const int ntiles = e->ntiles;
    int rc = ts_prepare_weights(e, st);
    if (rc) return rc;
    const size_t img_b = (size_t)ntiles * NKS * ts::A_STAGE_B;   // one operand image == one chunk-major fp32 copy, in bytes
    const int n_img = L + 1 + 4;    // images: node_states_per_layer, two step temporaries, agg, r*h
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
    const bool gru = e->cell == CELL_GRU;
    const GraphDev& gd = e->gd;

    // shared-memory budgets
    const size_t avail = (e->max_smem > 2048 ? e->max_smem - 2048 : 0);
    const size_t csr_b = (size_t)ts::TILE_M * T * 4;   // the tile's (target, type) -> source table
    CU_TRY(e, e->ts_virt.reserve((size_t)((e->ts_nv + ts::TILE_M - 1) / ts::TILE_M + 1) * NKS * ts::A_STAGE_B));
    // a ring stage carries KS K-steps, the largest of 4, 2, 1 that divides the K-steps of a segment (the producer thread pays several
    // hundred cycles per bulk copy whatever its size; KS is a template parameter so that a stage's MMAs are straight-line code)
    const char* env_ks = getenv("GGNN_TS_KSTEPS");
    const char* env_ns = getenv("GGNN_TS_STAGES");
    int KS = 4;
    if (env_ks) KS = atoi(env_ks) >= 4 ? 4 : (atoi(env_ks) >= 2 ? 2 : 1);
    while (NKS % KS) KS /= 2;
    auto stage_bytes = [&](int NC) { return (size_t)KS * ((size_t)ts::A_STAGE_B + 64 * (size_t)NC); };
    const int max_ns = env_ns ? std::max(0, std::min(atoi(env_ns), ts::MAX_NS)) : ts::MAX_NS;   // the kernel has MAX_NS stage barriers
    auto stages_for = [&](int NC, size_t budget) { return (int)std::min<size_t>((size_t)max_ns, budget / stage_bytes(NC)); };
    ts::StreamParams base;
    memset(&base, 0, sizeof base);
    base.V = V; base.D = D; base.DP = DP; base.T = T;
    base.nparts = e->precision == GGNN_PREC_BF16X3 ? 3 : 1;
    base.cell = e->cell; base.act = e->act; base.use_bias = e->use_bias; base.use_avg = e->use_avg;
    base.tile_mask = gd.tile_mask;
    base.pair_src = gd.pair_src; base.vrow_ptr = gd.vrow_ptr; base.vsrc = gd.vsrc; base.tile_vptr = gd.tile_vptr; base.vinfo = gd.vinfo;
    base.virt_img = (uint8_t*)e->ts_virt.ptr;   // pairs with several messages, pre-summed by the prologue of every gather launch
    base.indeg = gd.indeg; base.denom = gd.denom;
    base.drop_keep = e->drop_keep; base.drop_seed = e->drop_seed;
    base.error_flag = (int*)e->err_flag.ptr;
    const int nc0 = e->ts_nc[0], nb0 = e->ts_nblk[0], nc1 = e->ts_nc[1], nb1 = e->ts_nblk[1];
    // one CTA per SM for all three kernels: the whole shared memory is the ring
    const int ns_edge = stages_for(nc0, avail > csr_b ? avail - csr_b : 0);
    const int ns_gate = stages_for(nc1, avail), ns_cand = stages_for(nc0, avail);
    // the kernel's parity waits are only sound if every ring has at least as many stages as there are gather groups (ts::MIN_NS)
    const int ns_min = std::min({ns_edge, ns_gate, ns_cand});
    if (ns_min < ts::MIN_NS)
        return e->fail(GGNN_EUNSUPPORTED, "streaming ring of %d stages (DP=%d): it needs at least %d, one per gather group", ns_min, DP,
                       ts::MIN_NS);
    auto smem_of = [&](int NC, int ns, bool gather) { return (size_t)1024 + ts::ring_bytes(ns, stage_bytes(NC)) + (gather ? csr_b : 0); };
    const bool x3 = e->precision == GGNN_PREC_BF16X3;
    void (*k_edge)(ts::StreamParams) = nullptr;
    void (*k_fed)(ts::StreamParams) = nullptr;
#define GGNN_TS_PICK(X, K)                              \
    if (x3 == X && KS == K) {                           \
        k_edge = ts::ggnn_stream_kernel<true, X, K>;    \
        k_fed = ts::ggnn_stream_kernel<false, X, K>;    \
    }
    GGNN_TS_PICK(true, 4) GGNN_TS_PICK(true, 2) GGNN_TS_PICK(true, 1) GGNN_TS_PICK(false, 4) GGNN_TS_PICK(false, 2) GGNN_TS_PICK(false, 1)
#undef GGNN_TS_PICK
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
            // ---- aggregated messages
            ts::StreamParams p = base;
            p.epi = ts::EPI_AGG; p.NC = nc0; p.nstages = ns_edge;
            p.g_img = img_in; p.w = wb + wt.off_edge[l]; p.kt_all = T * NKS;
            p.bias = e->use_bias ? e->w[l].edge_biases : nullptr;
            p.img_out = img_agg; p.sv_agg = sv.agg; p.gstep = gs;
            k_edge<<<dim3(ntiles, nb0), ts::NTHREADS, sm_edge, st>>>(p);
            ++e->last_launches;
            auto set_segs = [&](ts::StreamParams& q, const uint8_t* last_img) {
                q.nseg = nseg;
                for (int i = 0; i < R; ++i) q.seg[i] = img_state(e->res[l][i]);
                q.seg[R] = img_agg; q.seg[R + 1] = last_img;
                q.kt_all = nseg * NKS;
            };
            if (gru) {
                ts::StreamParams q = base;
                q.epi = ts::EPI_GATE; q.NC = nc1; q.nstages = ns_gate;
                set_segs(q, img_in);
                q.w = wb + wt.off_gate[l]; q.bias = e->w[l].gate_bias; q.h_chk = chk_in; q.u_buf = u_chk; q.img_out = img_rh;
                q.sv_r = sv.r; q.sv_h = sv.h_in; q.sv_u = sv.u;
                q.gstep = gs;
                k_fed<<<dim3(ntiles, nb1), ts::NTHREADS, smem_of(nc1, ns_gate, false), st>>>(q);
                ++e->last_launches;
            }
            ts::StreamParams c = base;
            c.epi = ts::EPI_CAND; c.NC = nc0; c.nstages = ns_cand;
            set_segs(c, gru ? img_rh : img_in);
            c.w = wb + wt.off_cand[l]; c.bias = e->w[l].cand_bias; c.h_chk = chk_in; c.u_buf = u_chk; c.h_chk_out = chk_out; c.h_out = out; c.img_out = img_out;
            if (gru) c.sv_c = sv.c; else c.sv_h = sv.h_in;
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
// (source j -> target i, list order kept) with the weights as per-message weights.
static int build_gcn_image(ggnn_prepared_graph* g, int32_t V, int64_t nnz, const int64_t* list, const float* w) {
    g->valid = false;
    if (V < 0 || nnz < 0 || (nnz > 0 && (!list || !w))) return g->fail(GGNN_EINVAL, "null/negative argument");
    if (nnz > 0x7fffffff) return g->fail(GGNN_EUNSUPPORTED, "batch too large for int32 indexing");
    std::vector<int32_t> pairs((size_t)nnz * 2);
    for (int64_t k = 0; k < nnz; ++k) {
        const int64_t i = list[2 * k], j = list[2 * k + 1];
        if (i < 0 || i >= V || j < 0 || j >= V)
            return g->fail(GGNN_ERANGE, "adjacency_list[%lld] = (%lld, %lld) is out of range for %d nodes", (long long)k, (long long)i, (long long)j, V);
        pairs[2 * k] = (int32_t)j;
        pairs[2 * k + 1] = (int32_t)i;
    }
    const std::vector<float> indeg((size_t)std::max(V, 1), 0.0f);
    const int32_t* lists[1] = {pairs.data()};
    const int32_t counts[1] = {(int32_t)nnz};
    return build_sparse_image(g, V, lists, counts, indeg.data(), true, w);
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

int ggnn_set_graph_gcn(ggnn_engine* e, int32_t V, int64_t nnz, const int64_t* list, const float* w, ggnn_stream_t stream) {
    if (!e) return GGNN_EINVAL;
    GGNN_REQUIRE_MODEL(e, MODEL_GCN);
    return set_graph_from_own_prep(e, stream, [&](ggnn_prepared_graph** g) { return ggnn_prepare_graph_gcn(e, -1, V, nnz, list, w, g); });
}

int ggnn_prepared_graph_slot_weights(const ggnn_prepared_graph* g, float* target_csr_w, float* source_csr_w) {
    if (!g || !g->valid || !g->plan.weighted) return GGNN_ESTATE;
    const BatchPlan& q = g->plan;
    if (source_csr_w && !q.has_transpose) return GGNN_ESTATE;
    if (target_csr_w && q.M) memcpy(target_csr_w, g->image.ptr + q.off_slotw, sizeof(float) * (size_t)q.M);
    if (source_csr_w && q.M) memcpy(source_csr_w, g->image.ptr + q.off_tslotw, sizeof(float) * (size_t)q.M);
    return GGNN_OK;
}

// Whether the GCN runs on its wgmma kernel (else on the fp32 kernel, one launch per layer).
static bool gcn_on_tensor_cores(const ggnn_engine* e) { return e->precision != GGNN_PREC_FP32 && e->DP <= 128; }

static int forward_gcn(ggnn_engine* e, const float* h0, float* h_out, cudaStream_t st) {
    const int D = e->D, DP = e->DP, L = e->L, V = e->V;
    const bool tcore = gcn_on_tensor_cores(e);
    gcn::GcnParams p;
    memset(&p, 0, sizeof p);
    p.V = V; p.D = D; p.DP = DP; p.L = L;
    p.nparts = e->precision == GGNN_PREC_BF16X3 ? 3 : 1;
    p.save = e->save ? 1 : 0;
    p.tile_start = e->gd.tile_start; p.row_ptr = e->gd.row_ptr; p.csr_src = e->gd.csr_src; p.slot_w = e->gd.slot_w;
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
int ggnn_gcn_backward(ggnn_engine* e, const float* d_h_out, const ggnn_gcn_layer_grads* grads, int32_t num_layers, float* d_h0, ggnn_stream_t stream) {
    using namespace ggnn::bwd;
    if (!e) return GGNN_EINVAL;
    GGNN_REQUIRE_MODEL(e, MODEL_GCN);
    if (int rc = begin_backward(e, "ggnn_gcn_backward", "setting the graph", d_h_out, grads, num_layers, d_h0)) return rc;
    cudaStream_t st = (cudaStream_t)stream;
    const int V = e->V, D = e->D, L = e->L;
    if (V == 0) return GGNN_OK;
    const size_t vd = (size_t)V * D;
    const size_t slab = align_up(vd * sizeof(float), 256);
    const size_t ws_floats = std::max(gemm_tn_workspace(e, true, e->use_bias, V, D, D, 1), gemm_tn_workspace(e, false, e->use_bias, V, D, D, 1));
    CU_TRY(e, e->bwd_buf.reserve(4 * slab + ws_floats * sizeof(float)));
    char* bb = (char*)e->bwd_buf.ptr;
    float *dH = (float*)bb, *dP = (float*)(bb + slab), *S = (float*)(bb + 2 * slab), *dS = (float*)(bb + 3 * slab), *ws = (float*)(bb + 4 * slab);
    const GraphDev& gd = e->gd;
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
            GatherJob j{gd.row_ptr, gd.csr_src, fstate[l], S, gd.slot_w, nullptr};
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
        if (l == 0 && !d_h0) break;
        gemm_nt(e, st, false, dpre, D, 0, e->gcn_w[l].kernel, D, 0, 1, dS, D, V, D, D);
        float* dst = l == 0 ? d_h0 : dH;
        GatherJob j{gd.trow, gd.ttgt, dS, dst, gd.tslot_w, nullptr};
        csr_gather_all_kernel<<<gather_grid, 256, 0, st>>>(j, j, V, D, 1);
        ++e->last_launches;
        dout = dst;
    }
    CU_TRY(e, cudaGetLastError());
    return GGNN_OK;
}

int ggnn_forward(ggnn_engine* e, const float* h0, float* h_out, ggnn_stream_t stream) {
    if (!e) return GGNN_EINVAL;
    const bool gcn = e->model == MODEL_GCN;
    if (!e->weights_set) return e->fail(GGNN_ESTATE, "%s has not been called", gcn ? "ggnn_gcn_set_weights" : "ggnn_set_weights");
    if (!e->graph_set) return no_graph(e);
    if ((!h0 || !h_out) && e->V > 0) return e->fail(GGNN_EINVAL, "null state pointer");
    if (((uintptr_t)h0 & 15) || ((uintptr_t)h_out & 15)) return e->fail(GGNN_EINVAL, "state pointers must be 16-byte aligned");
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
        if (h_out != h0) CU_TRY(e, cudaMemcpyAsync(h_out, h0, (size_t)e->V * e->D * sizeof(float), cudaMemcpyDeviceToDevice, st));
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
int ggnn_readout_set_graphs(ggnn_engine* e, int32_t num_nodes, const int32_t* graph_nodes_list, int32_t num_graphs,
                            int32_t nodes_per_graph, const float* node_mask, ggnn_stream_t stream) {
    if (!e) return GGNN_EINVAL;
    e->ro_V = -1;
    if (num_nodes < 0 || num_graphs < 0) return e->fail(GGNN_EINVAL, "negative size");
    if (!graph_nodes_list && (nodes_per_graph <= 0 || (int64_t)nodes_per_graph * num_graphs != num_nodes))
        return e->fail(GGNN_EINVAL, "without a graph_nodes_list the batch must be num_graphs x nodes_per_graph (%d x %d != %d)", num_graphs, nodes_per_graph, num_nodes);
    CU_TRY(e, cudaSetDevice(e->device));
    const int V = num_nodes, G = num_graphs;
    size_t off = 0;
    e->ro_off_graph_of = off; off = align_up(off + sizeof(int) * (size_t)std::max(V, 1), 16);
    e->ro_off_start = off;    off = align_up(off + sizeof(int) * (size_t)(G + 1), 16);
    e->ro_off_mask = off;     off = align_up(off + sizeof(float) * (size_t)std::max(V, 1), 16);
    e->ro_off_perm = off;     off = align_up(off + sizeof(int) * (size_t)std::max(V, 1), 16);   // uploaded for ungrouped lists only
    e->ro_off_val = off;      // device-only scratch: per-node gated value
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
    e->ro_V = V; e->ro_G = G; e->ro_grouped = grouped; e->ro_has_mask = node_mask != nullptr;
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

int ggnn_readout_forward(ggnn_engine* e, const float* h_last, const float* h0, const float* w_gate, const float* b_gate,
                         const float* w_trans, const float* b_trans, float* out, ggnn_stream_t stream) {
    if (!e) return GGNN_EINVAL;
    const void* ps[7] = {h_last, h0, w_gate, b_gate, w_trans, b_trans, out};
    if (int rc = readout_check(e, ps, e->ro_V > 0 ? 7 : 0)) return rc;
    CU_TRY(e, cudaSetDevice(e->device));
    cudaStream_t st = (cudaStream_t)stream;
    const int V = e->ro_V, G = e->ro_G;
    if (G == 0) return GGNN_OK;
    if (!out) return e->fail(GGNN_EINVAL, "null output");
    char* g = (char*)e->ro_buf.ptr;
    const float* mask = e->ro_has_mask ? (const float*)(g + e->ro_off_mask) : nullptr;
    readout::Weights w{w_gate, b_gate, w_trans, b_trans};
    float* val = (float*)(g + e->ro_off_val);
    if (V > 0) readout::readout_node_kernel<<<(V + 7) / 8, 256, 0, st>>>(h_last, h0, w, mask, val, V, e->D);
    if (e->ro_grouped || V == 0) {
        readout::readout_sum_grouped_kernel<<<(G + 127) / 128, 128, 0, st>>>(val, (const int*)(g + e->ro_off_start), out, G);
    } else if (e->det) {
        readout::readout_sum_permuted_kernel<<<(G + 127) / 128, 128, 0, st>>>(val, (const int*)(g + e->ro_off_start), (const int*)(g + e->ro_off_perm),
                                                                            out, G);
    } else {
        CU_TRY(e, cudaMemsetAsync(out, 0, sizeof(float) * (size_t)G, st));
        readout::readout_sum_atomic_kernel<<<(V + 255) / 256, 256, 0, st>>>(val, (const int*)(g + e->ro_off_graph_of), out, V);
    }
    CU_TRY(e, cudaGetLastError());
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
    return ggnn_backward_impl(e, d_h_out, grads, num_layers, d_h0, stream);
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
    if (src && e->M) CU_TRY(e, cudaMemcpy(src, e->gd.csr_src, sizeof(int) * (size_t)e->M, cudaMemcpyDeviceToHost));
    if (msg && e->M) CU_TRY(e, cudaMemcpy(msg, e->gd.csr_msg, sizeof(int) * (size_t)e->M, cudaMemcpyDeviceToHost));
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
