/*
 * ggnn_b200.h -- C ABI of the H100-native GGNN propagation engine (libggnn_b200.so).
 *
 * This is the drop-in boundary for ONE path of microsoft/gated-graph-neural-network-samples: the
 * propagation step behind ChemModel's two graph-model hooks
 *
 *     prepare_specific_graph_model()          chem_tensorflow.py:205  (sparse:63-115, dense:68-91)
 *     compute_final_node_representations()    chem_tensorflow.py:208  (sparse:117-218, dense:93-117)
 *
 * The reference has no FFI (it is TF-1 graph construction in Python), so these entry points are what
 * a ctypes binding inside those two hooks calls (INTEGRATION.md shows the stub).  Plain pointers and
 * sizes only; no torch/TF types.  All functions return 0 on success or a negative GGNN_E* code; the
 * text is available from ggnn_last_error().  Nothing throws across the ABI.
 *
 * Ownership: the caller owns every tensor it passes (node states, weights, gradients); they must stay
 * valid until the stream work completes.  The engine owns its handle, the device copy of the batch's
 * graph structure (CSR + tiling) and its scratch.  One engine per GPU/stream; not thread-safe.
 * Launches are asynchronous on the caller's stream; there is no hidden device synchronisation except
 * in the *_host convenience calls, which return after the result is in host memory.
 */
#ifndef GGNN_B200_H
#define GGNN_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct ggnn_engine ggnn_engine;
typedef void* ggnn_stream_t; /* a cudaStream_t (0 = default stream) */

enum { GGNN_OK = 0, GGNN_EINVAL = -1, GGNN_ECUDA = -2, GGNN_ESTATE = -3, GGNN_EUNSUPPORTED = -4, GGNN_ERANGE = -5 };
enum { GGNN_CELL_GRU = 0, GGNN_CELL_RNN = 1,    /* params['graph_rnn_cell']        sparse:102-112 */
       GGNN_CELL_CUDNN_GRU = 2,                 /* 'CudnnCompatibleGRUCell', sparse:105-108 (fp32 path at every precision; tanh only, as the
                                                   reference asserts) */
       GGNN_CELL_CUDNN_GRU_TENSOR_CORES = 3 };  /* CudnnCompatibleGRUCell at the configured precision: the same weights, cand_hidden_bias, tanh
                                                   requirement and gradients as GGNN_CELL_CUDNN_GRU; on GGNN_PREC_BF16X3 / GGNN_PREC_BF16 every batch
                                                   takes the streaming wgmma plan (a hidden-projection GEMM per step), on GGNN_PREC_FP32 and with
                                                   GGNN_ATT_FP32 attention exactly GGNN_CELL_CUDNN_GRU.  Sparse model only: the dense entries and
                                                   the dense dataset refuse it (GGNN_EUNSUPPORTED) */
enum { GGNN_ACT_TANH = 0, GGNN_ACT_RELU = 1 };  /* params['graph_rnn_activation']  sparse:75-81   */
/* arithmetic of the dense contractions */
enum { GGNN_PREC_FP32 = 0,   /* fp32 FFMA on CUDA cores (bit-for-bit fp32 semantics, order aside) */
       GGNN_PREC_BF16X3 = 1, /* wgmma tensor cores, bf16 hi/lo split, 3 MMAs (~2^-16 rel / product) */
       GGNN_PREC_BF16 = 2 }; /* wgmma tensor cores, single bf16 MMA ("fast", outside the 1e-4 bar) */
/* values of ggnn_config.use_propagation_attention */
enum { GGNN_ATT_OFF = 0,
       GGNN_ATT_FP32 = 1,           /* attention on the fp32 kernels whatever the precision (every nonzero value but 2 means this) */
       GGNN_ATT_TENSOR_CORES = 2 }; /* attention at the configured precision: on GGNN_PREC_BF16X3 / GGNN_PREC_BF16 every batch takes the
                                       streaming wgmma plan (a softmax pre-pass per step feeding the slot-weighted gather); on
                                       GGNN_PREC_FP32, and with GGNN_CELL_CUDNN_GRU, exactly GGNN_ATT_FP32; with
                                       GGNN_CELL_CUDNN_GRU_TENSOR_CORES the streaming plan runs both the pre-pass and the cell's
                                       hidden-projection GEMM */

/* Mirrors the keys of self.params the two hooks read (sparse:40-61, chem_tensorflow.py:17-37). */
typedef struct ggnn_config {
    int32_t hidden_size;                  /* params['hidden_size'] (D)                                 */
    int32_t num_edge_types;               /* self.num_edge_types (T), chem_tensorflow.py:120           */
    int32_t num_layers;                   /* len(params['layer_timesteps'])                            */
    const int32_t* layer_timesteps;       /* [num_layers]                        sparse:53,131         */
    const int32_t* residual_offsets;      /* [num_layers+1] CSR over layers      sparse:48-51,140-145  */
    const int32_t* residual_layers;       /* [residual_offsets[num_layers]] indices into node_states_per_layer */
    int32_t use_edge_bias;                /* sparse:45,98,202                                          */
    int32_t use_edge_msg_avg_aggregation; /* sparse:47,206                                             */
    int32_t cell;                         /* GGNN_CELL_*                                               */
    int32_t activation;                   /* GGNN_ACT_*                                                */
    int32_t precision;                    /* GGNN_PREC_*                                               */
    int32_t device;                       /* CUDA device ordinal                                       */
    int32_t use_propagation_attention;    /* GGNN_ATT_*, sparse:46,94-96,147-149,170-196 (<= 16 edge types) */
} ggnn_config;

/* Device pointers to one layer's trainables, fp32 row-major, shapes as created at sparse:86-115:
 *   edge_weights [T, D, D]   (the reference Variable is [T*D, D]; same bytes, sparse:88-90)
 *   edge_biases  [T, D]      or NULL when !use_edge_bias (dense model: [T,1,D], same bytes)
 *   GRU: gate_kernel [Din+D, 2D], gate_bias [2D]  (columns: r first, u second)
 *        cand_kernel [Din+D, D],  cand_bias [D]
 *   RNN: cand_kernel [Din+D, D], cand_bias [D] hold BasicRNNCell's kernel/bias; gate_* are NULL.
 *   CudnnCompatibleGRUCell (tf.contrib.cudnn_rnn, sparse:105-108): gates as GRU;
 *        c = tanh(x . K_in + b_in + r * (h . K_hid + b_hid)) -- the reset gate is applied AFTER the recurrent product.
 *        cand_kernel [Din+D, D] = [candidate/input_projection/kernel ; candidate/hidden_projection/kernel] (rows stacked in that
 *        order, so the row order below still holds), cand_bias [D] = b_in, cand_hidden_bias [D] = b_hid.
 * Din = D * (1 + number of residual inputs of the layer); kernel rows are ordered
 * [residual states ..., aggregated messages, recurrent state] (sparse:211-216 + TF-1.3 _linear).   */
typedef struct ggnn_layer_weights {
    const float* edge_weights;
    const float* edge_biases;
    const float* gate_kernel;
    const float* gate_bias;
    const float* cand_kernel;
    const float* cand_bias;
    const float* edge_type_attention_weights; /* [T] (sparse:94-96) or NULL when !use_propagation_attention */
    const float* cand_hidden_bias;            /* [D] CudnnCompatibleGRUCell only (candidate/hidden_projection/bias), else NULL */
} ggnn_layer_weights;

/* Same layout, device pointers the backward pass ACCUMULATES into (caller zeroes them). */
typedef struct ggnn_layer_grads {
    float* edge_weights;
    float* edge_biases;
    float* gate_kernel;
    float* gate_bias;
    float* cand_kernel;
    float* cand_bias;
    float* edge_type_attention_weights;
    float* cand_hidden_bias;
} ggnn_layer_grads;

/* prepare_specific_graph_model (sparse:63-115 / dense:68-91): fix the model shape.
 * Limits: hidden_size a positive multiple of 4 and <= 512 (larger: GGNN_EUNSUPPORTED), 1 <= num_edge_types <= 32 (<= 16 with propagation
 * attention), 1 <= num_layers <= 16, at most 4 residual inputs per layer.  Kernels by hidden size: GGNN_PREC_BF16X3 / GGNN_PREC_BF16 run
 * the tile-local wgmma kernel up to 128 and the streaming wgmma kernels above; attention with GGNN_ATT_TENSOR_CORES, and
 * GGNN_CELL_CUDNN_GRU_TENSOR_CORES, run the streaming wgmma kernels at every hidden size.  GGNN_PREC_FP32 (and GGNN_ATT_FP32 attention, and
 * GGNN_CELL_CUDNN_GRU, at any precision) runs the fused fp32 tile kernel up to 256 and the per-timestep fp32 path above 256.  A weighted dense adjacency runs on
 * tensor cores up to hidden 128 on the tile-local kernel (GLOBAL when a component exceeds 128 rows) whichever dense entry feeds it; above
 * 128, ggnn_set_graph_dense / ggnn_run_dense_host(_predict) refuse it as before (run it on GGNN_PREC_FP32), and the ..._dense_weighted
 * entries run it on the streaming kernels, whose gather sums each weighted (target, type) pair into a virtual row. */
int ggnn_create(const ggnn_config* cfg, ggnn_engine** out);
int ggnn_destroy(ggnn_engine* e);
const char* ggnn_last_error(const ggnn_engine* e); /* e may be NULL: error of the last failed ggnn_create */

/* Bind the trainables (device pointers, one entry per layer); pointers are read at every forward.  A refused call binds nothing.  The
 * saved activations of the last forward are dropped: ggnn_backward then returns GGNN_ESTATE until the next forward with save_for_backward,
 * so a backward never combines one forward's activations with other weights. */
int ggnn_set_weights(ggnn_engine* e, const ggnn_layer_weights* layers, int32_t num_layers);

/* Feed one batch's graph structure in the reference wire format (sparse:331-348), HOST pointers:
 *   adjacency_lists[t] -> [num_edges[t], 2] int32 (col 0 = source, col 1 = target), message order kept
 *   num_incoming_edges_per_type -> [V, T] float32
 * Validates indices (TF-CPU gather raises on OOB), builds the stable target-sorted CSR and the tile
 * plan, and uploads them on `stream`. */
int ggnn_set_graph_sparse(ggnn_engine* e, int32_t num_nodes, const int32_t* const* adjacency_lists,
                          const int32_t* num_edges, const float* num_incoming_edges_per_type,
                          ggnn_stream_t stream);

/* The two halves of ggnn_set_graph_sparse as separate calls, so that the host half can run in a PRODUCER THREAD while the engine's
 * stream is still busy with the previous batch -- the overlap the reference gets from ThreadedIterator around its batch packer
 * (chem_tensorflow.py:225, utils.py:16-36; SURVEY 8 f3):
 *   ggnn_prepare_graph_sparse   host only: index validation, stable target-sorted CSR, tile plan, streaming tables, packed into ONE
 *                               pinned image.  Reads the engine's configuration and nothing else of it: thread-safe against calls on the
 *                               engine from another thread.  save_for_backward: 1 / 0 = whether the batch will be trained on (the
 *                               source-keyed CSR of ggnn_backward is part of the image), -1 = the engine's flag at this moment.
 *                               *inout = NULL allocates a prepared graph, a non-NULL one is rebuilt in place (it first waits for its own
 *                               previous upload).
 *   ggnn_set_graph_prepared     engine thread: adopts the plan and enqueues the single H2D copy of the image on `stream`.  The prepared
 *                               graph must stay alive (and must not be rebuilt from a thread that skips the wait above) until that copy ran.
 * Every graph upload, failed ones included, first forgets the previous batch: its forward (ggnn_layer_state), its saved activations
 * (ggnn_backward) and its readout map (ggnn_readout_set_graphs must follow the upload).
 * ggnn_set_graph_sparse is exactly these two calls on an engine-owned prepared graph.  On failure the text is in
 * ggnn_prepared_graph_error (prepare) / ggnn_last_error (set). */
typedef struct ggnn_prepared_graph ggnn_prepared_graph;
int ggnn_prepare_graph_sparse(const ggnn_engine* e, int32_t save_for_backward, int32_t num_nodes, const int32_t* const* adjacency_lists,
                              const int32_t* num_edges, const float* num_incoming_edges_per_type, ggnn_prepared_graph** inout);
int ggnn_set_graph_prepared(ggnn_engine* e, ggnn_prepared_graph* g, ggnn_stream_t stream);
int ggnn_free_prepared_graph(ggnn_prepared_graph* g);
const char* ggnn_prepared_graph_error(const ggnn_prepared_graph* g);
/* The same host half without an engine or a GPU (plain memory instead of pinned): what the CPU test-suite pins against
 * ggnn_host_target_csr / ggnn_host_tile_plan / ggnn_host_stream_tables, and a way to prepare batches on a machine without a device. */
int ggnn_host_prepare_graph_sparse(const ggnn_config* cfg, int32_t num_sms, int32_t save_for_backward, int32_t num_nodes,
                                   const int32_t* const* adjacency_lists, const int32_t* num_edges,
                                   const float* num_incoming_edges_per_type, ggnn_prepared_graph** inout);
/* The dense wire format through the same two halves: a 0/1 adjacency_matrix [b, T, v, v] (all the reference ever feeds, dense:30-36) is
 * scanned into edge lists (order: graph, target row, source column; in-degree = row sums) and built like a sparse batch; the result is
 * adopted with ggnn_set_graph_prepared.  A matrix with other entries returns GGNN_EUNSUPPORTED: feed it with ggnn_set_graph_dense, which
 * builds it the same way with its entries as per-message weights. */
int ggnn_prepare_graph_dense(const ggnn_engine* e, int32_t save_for_backward, int32_t num_graphs, int32_t num_vertices,
                             const float* adjacency_matrix, ggnn_prepared_graph** inout);
int ggnn_host_prepare_graph_dense(const ggnn_config* cfg, int32_t num_sms, int32_t save_for_backward, int32_t num_graphs,
                                  int32_t num_vertices, const float* adjacency_matrix, ggnn_prepared_graph** inout);
/* Any matrix, a weighted one with its entries as per-message (slot) weights and the plan text ending in
 * " [weighted dense adjacency -> weighted CSR]"; a 0/1 matrix exactly as ggnn_prepare_graph_dense builds it.  Unlike ggnn_set_graph_dense,
 * a weighted matrix above hidden 128 on GGNN_PREC_BF16X3 / GGNN_PREC_BF16 takes the streaming plan.  ggnn_set_graph_dense_weighted (below)
 * is the prepare and the upload in one call; the host-only form needs no engine or GPU. */
int ggnn_prepare_graph_dense_weighted(const ggnn_engine* e, int32_t save_for_backward, int32_t num_graphs, int32_t num_vertices,
                                      const float* adjacency_matrix, ggnn_prepared_graph** inout);
int ggnn_host_prepare_graph_dense_weighted(const ggnn_config* cfg, int32_t num_sms, int32_t save_for_backward, int32_t num_graphs,
                                           int32_t num_vertices, const float* adjacency_matrix, ggnn_prepared_graph** inout);
/* ---- Message weights (sparse GGNN model): message m of type t, from source s to target v, weighs w_m, the messages numbered in the
 * reference's type-major order (type t's list, in fed order, starts at sum_{t' < t} E_t'):
 *     incoming[v] = ( sum_t (sum_{m into v, type t} w_m h[s_m]) W_t  +  sum_t indeg[v,t] b_t ) / denom[v]      (/ only with avg aggregation)
 * The weight scales the state term only: the in-degree table is used as fed, for the edge bias and the mean, and is data (no gradient).
 * Weights may be zero, negative or any finite value; weights of 1.0 give the unweighted model.  The gradient, per timestep of every layer
 * with step input state h:  d w_m += <P[v, t], h[s_m]>,  P = dx' . W_t^T, dx' the gradient of the pre-mean message sum.
 *   ggnn_prepare_graph_sparse_weighted   as ggnn_prepare_graph_sparse (same validation, CSR, tile plan, pinned image), the batch marked
 *                                        message-weighted and its plan text ending in " [message-weighted]".  Its slot-weight sections
 *                                        are zero until ggnn_set_message_weights writes them on the device; with save_for_backward the image
 *                                        also carries the source-keyed CSR's slot map.  The plan depends on the structure alone: on the
 *                                        streaming plan (hidden sizes above 128 on GGNN_PREC_BF16X3 / GGNN_PREC_BF16, and
 *                                        GGNN_CELL_CUDNN_GRU_TENSOR_CORES) every (target, type) pair with messages is a virtual row.  Refused:
 *                                        propagation attention (GGNN_EUNSUPPORTED: its probabilities are the slot weights), a GCN engine
 *                                        (GGNN_ESTATE).  The host-only twin needs no engine or GPU.
 *   ggnn_set_message_weights             message_weights DEVICE fp32 [M] (ggnn_num_messages), in the order above: one kernel on `stream`
 *                                        scatters them into the current batch's slot weights; the buffer is free once the stream passed
 *                                        the call.  GGNN_ESTATE when the current batch is not message-weighted.  Every graph upload forgets
 *                                        the weights, and ggnn_forward on a message-weighted batch without them is GGNN_ESTATE.  Like
 *                                        ggnn_set_weights it drops the saved activations of the last forward.
 *   ggnn_backward_weighted               ggnn_backward, and with d_message_weights (DEVICE fp32 [M], accumulated into) the weights' gradient:
 *                                        one P GEMM per timestep (wgmma under ggnn_set_backward_precision(GGNN_PREC_BF16X3)) and a per-slot
 *                                        sum in a fixed order, without atomics -- bit-identical from call to call in both deterministic
 *                                        modes.  ggnn_backward is this call with d_message_weights = NULL; a non-NULL one on a batch that is not
 *                                        message-weighted is GGNN_ESTATE. */
int ggnn_prepare_graph_sparse_weighted(const ggnn_engine* e, int32_t save_for_backward, int32_t num_nodes, const int32_t* const* adjacency_lists,
                                       const int32_t* num_edges, const float* num_incoming_edges_per_type, ggnn_prepared_graph** inout);
int ggnn_host_prepare_graph_sparse_weighted(const ggnn_config* cfg, int32_t num_sms, int32_t save_for_backward, int32_t num_nodes,
                                            const int32_t* const* adjacency_lists, const int32_t* num_edges,
                                            const float* num_incoming_edges_per_type, ggnn_prepared_graph** inout);
int ggnn_set_message_weights(ggnn_engine* e, const float* message_weights, ggnn_stream_t stream);
/* ---- Dense adjacency on the device (dense GGNN model): the [b, T, v, v] matrix A of the reference's dense model (dense:78-80, 110-112) as a
 * DEVICE fp32 buffer, A[g, t, i, j] the weight of the type-t message from node j to node i of graph g, the batch's rows g*v + i.  Any finite
 * values (negative, zero, or a full matrix).  Per timestep with input state h (no averaging):
 *     X_t[g*v+i] = sum_j A[g,t,i,j] h[g*v+j]    (j ascending, fmaf from +0)
 *     agg        = sum_t X_t W_t + sum_t rowsum(A[g,t,i,:]) b_t       (fp32 row sums in column order, on the device)
 * and the gradient at every entry, zeros included:  dA[g,t,i,j] += <P_t[g*v+i], h[g*v+j]> + <dx'[g*v+i], b_t>,  P = dx' . W_t^T.
 *   ggnn_prepare_graph_dense_device      the plan and image of b graphs of v rows from (b, v) alone: no matrix is read.  ggnn_num_messages
 *                                        of the batch is b*T*v*v and its plan text ends in " [dense adjacency on the device]".
 *                                        GGNN_PREC_BF16X3 / GGNN_PREC_BF16 run the streaming plan at every hidden size (a dense aggregation
 *                                        launch before every gather-GEMM), GGNN_PREC_FP32 the per-timestep fp32 path at every hidden size.
 *                                        Refused with GGNN_EUNSUPPORTED: propagation attention, use_edge_msg_avg_aggregation (its denominator
 *                                        would depend on A), GGNN_CELL_CUDNN_GRU_TENSOR_CORES.  Adopt it with ggnn_set_graph_prepared; the
 *                                        host-only twin needs no engine or GPU.
 *   ggnn_set_message_weights             on such a batch: message_weights = A [b, T, v, v], copied into an engine buffer on `stream` (the
 *                                        caller's buffer is free once the stream passed the call), its row sums computed in the same call.
 *                                        The rules above hold: every upload forgets A, a forward without it is GGNN_ESTATE, setting it drops
 *                                        the saved activations.  A new A on the same batch needs no new prepare.
 *   ggnn_backward_weighted               d_message_weights = dA [b, T, v, v], accumulated into; every entry has one writer per timestep and
 *                                        the timesteps are added in the backward's fixed order, so dA repeats bit for bit in both
 *                                        deterministic modes. */
int ggnn_prepare_graph_dense_device(const ggnn_engine* e, int32_t save_for_backward, int32_t num_graphs, int32_t num_vertices,
                                    ggnn_prepared_graph** inout);
int ggnn_host_prepare_graph_dense_device(const ggnn_config* cfg, int32_t num_sms, int32_t save_for_backward, int32_t num_graphs,
                                         int32_t num_vertices, ggnn_prepared_graph** inout);
/* Introspection of a prepared graph: sizes and plan text; copies of its CSR (row_ptr [V*T+1], src [M], msg [M]), tile starts
 * [num_tiles+1], per-node mean-aggregation denominators [V] and, for a streaming plan, the (target, type) -> source table
 * [ceil(V/128)*128*T] (NULL pointers are skipped; pair_src of a non-streaming plan is left untouched and *is_streaming = 0). */
int ggnn_prepared_graph_info(const ggnn_prepared_graph* g, int32_t* num_nodes, int64_t* num_messages, int32_t* num_tiles, int64_t* image_bytes,
                             int32_t* is_streaming, char* plan_text, int32_t plan_text_capacity);
int ggnn_prepared_graph_arrays(const ggnn_prepared_graph* g, int32_t* row_ptr, int32_t* src, int32_t* msg, int32_t* tile_start, float* denom,
                               int32_t* pair_src);
/* The whole packed image (image_bytes of ggnn_prepared_graph_info) -- exactly the bytes ggnn_set_graph_prepared uploads.  The builder
 * splits its passes over host threads by target ranges (GGNN_HOST_THREADS overrides the count); the tests require identical bytes for
 * every thread count. */
int ggnn_prepared_graph_image(const ggnn_prepared_graph* g, void* dst, int64_t capacity);
/* The plan's largest message count and largest number of edge types present in one tile: what the tile-local wgmma kernel sizes its shared
 * memory by (its CSR cache and its gather tiles). */
int ggnn_prepared_graph_tile_stats(const ggnn_prepared_graph* g, int32_t* max_tile_msgs, int32_t* max_tile_types);
/* A streaming plan's virtual rows (the (target, type) pairs the gather sums before copying; pair_src of ggnn_prepared_graph_arrays holds
 * -(2 + vid) for them): their count NV and message count, vrow_ptr [NV+1] / vsrc (their sources in target-CSR order), vinfo [8*NV] (count,
 * then the first seven sources, zero-filled), tile_vptr [num_tiles+1] (first vid of every tile) and, on a weighted batch only, vslot [NV]
 * (the first target-CSR slot of every virtual row: message m weighs slot weight vslot[vid] + m).  In a weighted batch a pair is a virtual
 * row unless it has exactly one message of weight exactly 1.0f.  NULL pointers are skipped; GGNN_ESTATE for a plan that does not stream,
 * and for vslot on a binary one. */
int ggnn_prepared_graph_stream_tables(const ggnn_prepared_graph* g, int32_t* num_virtual_rows, int64_t* num_virtual_messages, int32_t* vrow_ptr,
                                      int32_t* vsrc, int32_t* vinfo, int32_t* vslot, int32_t* tile_vptr);

/* Dense wire format (dense:214-224): adjacency_matrix [b, T, v, v] float32 HOST pointer with
 * A[g, t, dest, src] (dense:30-36).  Rows are the b*v padded nodes. */
int ggnn_set_graph_dense(ggnn_engine* e, int32_t num_graphs, int32_t num_vertices,
                         const float* adjacency_matrix, ggnn_stream_t stream);
/* The same, and a weighted matrix above hidden 128 on the tensor-core precisions runs on the streaming kernels (ggnn_set_graph_dense
 * refuses it there with GGNN_EUNSUPPORTED). */
int ggnn_set_graph_dense_weighted(ggnn_engine* e, int32_t num_graphs, int32_t num_vertices,
                                  const float* adjacency_matrix, ggnn_stream_t stream);

/* compute_final_node_representations (sparse:117-218 / dense:93-117).
 * h0, h_out: DEVICE [V, D] fp32 (dense: [b*v, D]).  Asynchronous on `stream`.
 * Aliasing: the V*D floats at h_out must not overlap those at h0, on any model and plan (the GLOBAL launches gather h0 rows that other
 * blocks overwrite, and the backward reads h0 again); an overlap returns GGNN_EINVAL naming both pointers, before any launch and with the
 * engine's state untouched.  ggnn_backward / ggnn_gcn_backward and ggnn_layer_state read h0 and h_out of the last forward again (they are
 * node_states_per_layer[0] and [L]): both must stay unchanged until the backward has run. */
int ggnn_forward(ggnn_engine* e, const float* h0, float* h_out, ggnn_stream_t stream);

/* Same with HOST buffers: H2D copy of h0, propagation, D2H copy of the result, stream-synchronised. */
int ggnn_forward_host(ggnn_engine* e, const float* h0_host, float* h_out_host, ggnn_stream_t stream);
/* One call per batch -- the shape of the reference's sess.run(fetch_list, feed_dict=batch) (chem_tensorflow.py:235): graph
 * structure + initial states in, final node states out, all HOST buffers, synchronous.  Equivalent to ggnn_set_graph_* followed
 * by ggnn_forward_host, except that the h0 upload is enqueued first so the host-side CSR build overlaps it. */
int ggnn_run_sparse_host(ggnn_engine* e, int32_t num_nodes, const int32_t* const* adjacency_lists, const int32_t* num_edges,
                         const float* num_incoming_edges_per_type, const float* h0_host, float* h_out_host, ggnn_stream_t stream);
int ggnn_run_dense_host(ggnn_engine* e, int32_t num_graphs, int32_t num_vertices, const float* adjacency_matrix,
                        const float* h0_host, float* h_out_host, ggnn_stream_t stream);
/* ... without the final synchronisation (pinned host buffers; pair with ggnn_sync_check): lets a caller keep two batches in
 * flight on two engines/streams, the way ChemModel's ThreadedIterator overlaps packing with sess.run (chem_tensorflow.py:225). */
int ggnn_forward_host_async(ggnn_engine* e, const float* h0_host, float* h_out_host, ggnn_stream_t stream);

/* ---- Readout: gated_regression (sparse:220-231, dense:119-129), the op right after the propagation (SURVEY 8f-1), one task:
 *   out[g] = sum over the nodes v of graph g of  sigmoid([h_T[v] | h_0[v]] . w_gate + b_gate) * (h_T[v] . w_trans + b_trans) * mask[v]
 * The reference's two readout MLPs have no hidden layers (chem_tensorflow.py:153-157): w_gate is the [2D,1] kernel, w_trans the [D,1]
 * kernel.  ggnn_readout_set_graphs feeds the batch's node -> graph map in the reference wire format, HOST pointers:
 *   sparse: graph_nodes_list [V] int32 (sparse:337), node_mask NULL
 *   dense : graph_nodes_list NULL, nodes_per_graph = num_vertices (graph = row / num_vertices), node_mask [b*v] float32 (dense:126)
 * Nodes grouped by graph (what the packers produce) are summed in node order, deterministically, like TF's CPU
 * unsorted_segment_sum; an ungrouped list falls back to float atomics (with ggnn_set_deterministic on, each graph's nodes are summed in
 * node order through a stable by-graph permutation built here).  All other pointers are DEVICE fp32; `out` is [num_graphs].
 * ggnn_readout_backward writes d_h_last [V,D] and ACCUMULATES into the weight gradients (caller zeroes; any may be NULL).  The map belongs
 * to the current batch: a graph upload drops it, and the readout calls return GGNN_ESTATE until ggnn_readout_set_graphs runs again. */
int ggnn_readout_set_graphs(ggnn_engine* e, int32_t num_nodes, const int32_t* graph_nodes_list, int32_t num_graphs,
                            int32_t nodes_per_graph, const float* node_mask, ggnn_stream_t stream);
int ggnn_readout_forward(ggnn_engine* e, const float* h_last, const float* h0, const float* w_gate, const float* b_gate,
                         const float* w_trans, const float* b_trans, float* out, ggnn_stream_t stream);
int ggnn_readout_backward(ggnn_engine* e, const float* h_last, const float* h0, const float* w_gate, const float* b_gate,
                          const float* w_trans, const float* b_trans, const float* d_out, float* d_h_last, float* d_w_gate,
                          float* d_b_gate, float* d_w_trans, float* d_b_trans, ggnn_stream_t stream);

/* The whole fetch of the reference's training/validation step in ONE call -- sess.run([loss, accuracy_task*], feed_dict=batch),
 * chem_tensorflow.py:231-235 with the ops of :145-170: propagation (sparse:117-218), gated_regression per task (sparse:220-231), masked
 * 1/2-MSE loss and MAE per task (chem_tensorflow.py:161-166; the 1/task_sample_ratio factor of :168 is left to the caller).
 * The batch comes in HOST buffers in the reference wire format (sparse:331-348): graph structure, h0 [V, D], graph_nodes_list [V],
 * target_values / target_mask [num_tasks, num_graphs]; the readout trainables are DEVICE pointers, one ggnn_readout_task per task.
 * Only 2 * num_tasks floats come back: loss_out [num_tasks], accuracy_out [num_tasks] (HOST).  Synchronous. */
typedef struct ggnn_readout_task {
    const float* w_gate;  /* [2D] regression_gate MLP kernel      (chem_tensorflow.py:153-154) */
    const float* b_gate;  /* [1]                                                               */
    const float* w_trans; /* [D]  regression_transform MLP kernel (chem_tensorflow.py:155-157) */
    const float* b_trans; /* [1]                                                               */
} ggnn_readout_task;
int ggnn_run_sparse_host_readout(ggnn_engine* e, int32_t num_nodes, const int32_t* const* adjacency_lists, const int32_t* num_edges,
                                 const float* num_incoming_edges_per_type, const float* h0_host, const int32_t* graph_nodes_list,
                                 int32_t num_graphs, int32_t num_tasks, const ggnn_readout_task* tasks, const float* target_values,
                                 const float* target_mask, float* loss_out, float* accuracy_out, ggnn_stream_t stream);

/* ---- Prediction: every task's readout in one pass over the node rows (the reference's evaluate_one_batch, sparse:352-362 / dense:230-249,
 * fetches self.output; here all tasks come back).  Over the current readout map (ggnn_readout_set_graphs or a dataset batch), task k of batch
 * graph g is written to out[k * out_stride + slot[g]]:
 *   slot      DEVICE int32 [num_graphs], or NULL for slot[g] = g (out_stride >= num_graphs then).  Each task's values are those
 *             ggnn_readout_forward computes with that task's weights, bit for bit when the sums are ordered (grouped node lists, or
 *             ggnn_set_deterministic).  Entries must be distinct and below out_stride: nothing else of `out` is written.
 *   tasks     1 .. 16 tasks (more is GGNN_EINVAL), DEVICE weights as for ggnn_readout_forward (w_gate / w_trans 16-byte aligned).
 * ggnn_dataset_batch_slots: the slot table of the dataset batch the engine adopted last -- its graphs' dataset indices [G], DEVICE, valid
 * until the next graph upload -- so that a whole dataset's predictions land in one [num_tasks, N] buffer; GGNN_ESTATE when the current
 * readout map did not come from a dataset batch.
 * ggnn_run_sparse_host_predict / ggnn_run_dense_host_predict: one synchronous call per batch with HOST buffers and no targets, the shape of
 * sess.run(self.output, feed) -- upload, the forward without saving for backward, the readout map (sparse: graph_nodes_list [V]; dense:
 * num_graphs x num_vertices with node_mask [b*v]), every task, and out_host [num_tasks, num_graphs] back. */
int ggnn_readout_predict(ggnn_engine* e, const float* h_last, const float* h0, int32_t num_tasks, const ggnn_readout_task* tasks,
                         const int32_t* slot, int32_t out_stride, float* out, ggnn_stream_t stream);
int ggnn_dataset_batch_slots(const ggnn_engine* e, const int32_t** slot);
int ggnn_run_sparse_host_predict(ggnn_engine* e, int32_t num_nodes, const int32_t* const* adjacency_lists, const int32_t* num_edges,
                                 const float* num_incoming_edges_per_type, const float* h0_host, const int32_t* graph_nodes_list,
                                 int32_t num_graphs, int32_t num_tasks, const ggnn_readout_task* tasks, float* out_host, ggnn_stream_t stream);
int ggnn_run_dense_host_predict(ggnn_engine* e, int32_t num_graphs, int32_t num_vertices, const float* adjacency_matrix, const float* h0_host,
                                const float* node_mask, int32_t num_tasks, const ggnn_readout_task* tasks, float* out_host,
                                ggnn_stream_t stream);

/* Synchronises `stream` and reports asynchronous kernel-side failures (a bounded barrier wait that expired). */
int ggnn_sync_check(ggnn_engine* e, ggnn_stream_t stream);

/* DropoutWrapper(cell, state_keep_prob) of sparse:113-114 / dense:89 (the reference keeps element [1], the dropped STATE,
 * sparse:216): every timestep's new state is multiplied by a keep mask and DIVIDED by keep_prob before it is stored and
 * carried on.  keep_prob = 1 (the default, and what the reference feeds in evaluation, sparse:284) turns it off.  The mask is
 * a counter-based hash of (seed, global timestep, node, column) -- TensorFlow's own random stream cannot be reproduced -- so
 * ggnn_backward regenerates it; use a fresh seed per training step.  Applies to the following ggnn_forward calls. */
int ggnn_set_state_dropout(ggnn_engine* e, float keep_prob, uint64_t seed);
/* The same mask on the host ([V, D] bytes, 1 = kept) for timestep `global_step` (layers' timesteps numbered consecutively):
 * lets a caller or a test restate the dropped forward. */
int ggnn_state_dropout_mask(int32_t V, int32_t D, int32_t global_step, float keep_prob, uint64_t seed, uint8_t* mask_out);

/* Gradient of the propagation (what optimizer.compute_gradients builds, chem_tensorflow.py:184).
 * Must follow a ggnn_forward on the same graph with save_for_backward enabled.
 * d_h_out: DEVICE [V, D]; grads: per layer, accumulated into; d_h0: DEVICE [V, D] or NULL.  d_h0 may be d_h_out or overlap it (here and
 * in ggnn_gcn_backward): d_h_out is read in full before d_h0 is written, so the result is the out-of-place one, bit for bit. */
int ggnn_set_save_for_backward(ggnn_engine* e, int32_t enable);
/* Deterministic mode (off by default; GGNN and GCN engines; takes effect from the next call).  With it on, the same engine configuration,
 * batch, weights, dropout seed and caller buffer contents produce identical bits in every output and every accumulated gradient buffer,
 * from call to call, engine to engine and process to process.  It governs ggnn_backward, ggnn_gcn_backward, ggnn_readout_forward /
 * ggnn_readout_backward and ggnn_run_sparse_host_readout: every weight and bias gradient G is summed in a fixed order over row splits that
 * depend only on the problem's shape (not on the GPU's SM count), and then added once (C <- C + G, as with it off); an ungrouped
 * graph_nodes_list is summed per graph in node order.  The forward and d h0 are bit-reproducible in either mode.  With it off the weight
 * gradients and an ungrouped readout sum are added with float atomics, equal only within their ordering noise. */
int ggnn_set_deterministic(ggnn_engine* e, int32_t enable);
/* Precision of the backward pass's GEMMs (GGNN and GCN engines; GGNN_PREC_FP32 by default).  GGNN_PREC_FP32: FFMA on CUDA cores.
 * GGNN_PREC_BF16X3: sm_90a wgmma tensor cores with the forward's hi/lo split (three bf16 MMAs per product, fp32 accumulators) for every data
 * gradient (the cell kernels, dh += sum_t G_t . W_t^T, attention's dx' . W^T, the GCN's dS) and every weight gradient but the edge biases;
 * bias gradients stay fp32 column sums, the elementwise, gather and attention kernels are unchanged.  Expect each gradient tensor within
 * max|err| / max|ref| < 2e-4 of float64 (the forward's bf16x3 bar).  Independent of the forward's precision and of ggnn_set_deterministic
 * (which keeps its guarantees: d h0 bit-reproducible, the weight gradients too with it on).  Takes effect at the next backward call and
 * touches nothing else (the forward, the saved activations, the plan): switching between two backward calls on one saved forward is fine.
 * GGNN_PREC_BF16 and unknown values return GGNN_EINVAL and keep the setting. */
int ggnn_set_backward_precision(ggnn_engine* e, int32_t precision);
int ggnn_backward(ggnn_engine* e, const float* d_h_out, const ggnn_layer_grads* grads, int32_t num_layers,
                  float* d_h0, ggnn_stream_t stream);
/* ggnn_backward with the message weights' gradient (see ggnn_set_message_weights above). */
int ggnn_backward_weighted(ggnn_engine* e, const float* d_h_out, const ggnn_layer_grads* grads, int32_t num_layers, float* d_h0,
                           float* d_message_weights, ggnn_stream_t stream);

/* The CSR build of ggnn_set_graph_sparse on its own -- host arithmetic only, no engine, no GPU: row_ptr [V*T+1], src [M], msg [M]
 * (msg = position of the slot's message in the reference's type-major message order, sparse:124-129).  Returns GGNN_ERANGE for an
 * out-of-range edge.  Used by the CPU test-suite to pin the integer path against NumPy's stable sort. */
int ggnn_host_target_csr(int32_t num_nodes, int32_t num_edge_types, const int32_t* const* adjacency_lists, const int32_t* num_edges,
                         int32_t* row_ptr, int32_t* src, int32_t* msg);

/* The streaming plan's gather tables on their own (host arithmetic only; what ggnn_set_graph_sparse uploads when hidden_size > 128 or a
 * component exceeds a tile): pair_src [ceil(V/128)*128*T] -- per (target, type) pair -1 (no message), the source node (exactly one) or
 * -(2 + vid) (several messages: "virtual row" vid, numbered in (target, type) order); vrow_ptr [NV+1] / vsrc: the sources of every virtual
 * row in message order; tile_vptr [ceil(V/128)+1]: first vid of every 128-row tile.  Capacities in entries; returns the counts. */
int ggnn_host_stream_tables(int32_t num_nodes, int32_t num_edge_types, const int32_t* const* adjacency_lists, const int32_t* num_edges,
                            int32_t* pair_src, int32_t* vrow_ptr, int32_t vrow_capacity, int32_t* vsrc, int32_t vsrc_capacity,
                            int32_t* tile_vptr, int32_t* num_virtual_rows);

/* The tile plan ggnn_set_graph_sparse would make for this batch on a GPU with `num_sms` SMs -- host arithmetic only: tile_start
 * [num_tiles + 1] (first node of every tile; tile_capacity entries available) and the plan description.  Tiles are unions of whole
 * connected components whenever the largest component fits a tile (LOCAL plan); used by the CPU test-suite. */
int ggnn_host_tile_plan(int32_t hidden_size, int32_t num_edge_types, int32_t precision, int32_t num_sms, int32_t num_nodes,
                        const int32_t* const* adjacency_lists, const int32_t* num_edges, int32_t* tile_start, int32_t tile_capacity,
                        int32_t* num_tiles, char* plan_text, int32_t plan_text_capacity);

/* ---- Sparse GCN (Kipf & Welling; the reference's chem_tensorflow_gcn.py:42-82) on the same engine handle.
 * Per layer l:  S = A . H  (A sparse, S[i] += w * H[j] over the nonzeros (i, j, w) in list order),  H' = S . W_l (+ b_l),
 * then relu and state dropout on every layer but the last (the last layer is linear).
 * A GCN engine is created with ggnn_gcn_create.  ggnn_set_graph_prepared, ggnn_forward(_host/_host_async), ggnn_sync_check,
 * ggnn_set_state_dropout (outputs of layers 0..L-2, global step = layer index), ggnn_set_save_for_backward, ggnn_readout_*,
 * ggnn_layer_state (intermediate layers: after a forward with save_for_backward on), ggnn_plan_description,
 * ggnn_last_launch_count, ggnn_prepared_graph_info and ggnn_prepared_graph_arrays (T = 1: row_ptr [V+1] keyed by the output row i,
 * src = the input column j, msg = position in the input list) work on it as on a GGNN engine, and so does ggnn_set_message_weights on a
 * message-weighted GCN batch (below).  The GGNN-only calls (ggnn_set_weights, ggnn_set_graph_sparse/dense,
 * ggnn_prepare_graph_sparse/dense, ggnn_prepare_graph_sparse_weighted, ggnn_run_*, ggnn_backward, ggnn_backward_weighted) return
 * GGNN_ESTATE on a GCN engine, and the GCN calls below return GGNN_ESTATE on a GGNN engine.
 * Limits: hidden_size a positive multiple of 4 and <= 256 (<= 512 with wide_hidden), 1 <= num_layers <= 16.  precision
 * GGNN_PREC_BF16X3 / GGNN_PREC_BF16 run the fused wgmma kernel for hidden_size <= 128; GGNN_PREC_FP32 runs the fp32 CUDA-core kernel at
 * every hidden size.  Above 128 on GGNN_PREC_BF16X3 / GGNN_PREC_BF16:
 *   wide_hidden = 0  hidden sizes up to 256 run the fp32 CUDA-core kernel (the plan says gcn-fp32-ffma), larger ones are refused;
 *   wide_hidden = 1  every layer is two launches on fixed 128-row tiles (the plan says gcn-stream-...): a weighted gather writes S = A . H
 *                    as a bf16 hi/lo operand image, and the streaming wgmma kernel of the GGNN model's wide hidden sizes multiplies it by
 *                    W_l, adds the bias and applies relu and state dropout (the same masks as the fp32 kernel's).
 * At hidden_size <= 128 the flag changes nothing: the same plans and the same image bytes.  The two paths from 129 to 256 exist only because
 * the default, 0, is kept as it was; a batch or dataset prepared with one value of the flag is refused by an engine created with the other. */
typedef struct ggnn_gcn_config {
    int32_t hidden_size; /* params['hidden_size'] (D)                   */
    int32_t num_layers;  /* params['num_timesteps']                     */
    int32_t use_bias;    /* params['gcn_use_bias']                      */
    int32_t precision;   /* GGNN_PREC_*                                 */
    int32_t device;      /* CUDA device ordinal                         */
    int32_t wide_hidden; /* 0: as above; 1: hidden sizes up to 512, on the streaming wgmma plan above 128 on bf16x3 / bf16 */
} ggnn_gcn_config;
/* DEVICE pointers, fp32: kernel [D, D] row-major (gcn_weights_l), bias [D] (gcn_bias_l) or NULL when !use_bias. */
typedef struct ggnn_gcn_layer_weights { const float* kernel; const float* bias; } ggnn_gcn_layer_weights;
/* Same layout; ggnn_gcn_backward ACCUMULATES into them (caller zeroes; either may be NULL; 16-byte aligned). */
typedef struct ggnn_gcn_layer_grads { float* kernel; float* bias; } ggnn_gcn_layer_grads;
int ggnn_gcn_create(const ggnn_gcn_config* cfg, ggnn_engine** out);
int ggnn_gcn_set_weights(ggnn_engine* e, const ggnn_gcn_layer_weights* layers, int32_t num_layers);
/* The reference's feed (chem_tensorflow_gcn.py:44-47), HOST pointers: adjacency_list [nnz, 2] int64 with column 0 = the OUTPUT row i and
 * column 1 = the INPUT column j, adjacency_weights [nnz] fp32.  Any list a TF SparseTensor accepts: unsorted, duplicate (i, j) entries
 * (summed), rows without entries, nnz = 0; an index outside [0, num_nodes) returns GGNN_ERANGE.  The host half is the GGNN builder (stable
 * counting sort by output row, tile plan over whole connected components, one pinned image) plus the per-slot weights in target-CSR order
 * and, when saving for backward, in source-CSR order.  save_for_backward and *inout as for ggnn_prepare_graph_sparse. */
int ggnn_prepare_graph_gcn(const ggnn_engine* e, int32_t save_for_backward, int32_t num_nodes, int64_t nnz, const int64_t* adjacency_list,
                           const float* adjacency_weights, ggnn_prepared_graph** inout);
int ggnn_host_prepare_graph_gcn(const ggnn_gcn_config* cfg, int32_t num_sms, int32_t save_for_backward, int32_t num_nodes, int64_t nnz,
                                const int64_t* adjacency_list, const float* adjacency_weights, ggnn_prepared_graph** inout);
/* ggnn_prepare_graph_gcn into an engine-owned prepared graph + ggnn_set_graph_prepared. */
int ggnn_set_graph_gcn(ggnn_engine* e, int32_t num_nodes, int64_t nnz, const int64_t* adjacency_list, const float* adjacency_weights,
                       ggnn_stream_t stream);
/* Copies of a GCN prepared graph's per-slot weights: target_csr_w [nnz] (= adjacency_weights[msg]), source_csr_w [nnz] (weights in the
 * order of the source-keyed CSR; only present when the graph was prepared for backward, else GGNN_ESTATE if requested). */
int ggnn_prepared_graph_slot_weights(const ggnn_prepared_graph* g, float* target_csr_w, float* source_csr_w);
/* Gradient of the GCN propagation; must follow a ggnn_forward with save_for_backward on.  d_h_out [V, D] DEVICE; grads: one entry per
 * layer, accumulated into; d_h0 [V, D] DEVICE or NULL.  fp32 on CUDA cores whatever the forward precision. */
int ggnn_gcn_backward(ggnn_engine* e, const float* d_h_out, const ggnn_gcn_layer_grads* grads, int32_t num_layers, float* d_h0,
                      ggnn_stream_t stream);
/* ---- Adjacency weights on the device (GCN engine).  Entry k of the list, (i_k, j_k), weighs w_k, from a DEVICE fp32 [nnz] buffer in list
 * order; per layer l with input H_l:
 *     S_l[i] = sum_{k : i_k = i} w_k H_l[j_k]   (list order, as above)      d w_k = sum_l <dS_l[i_k], H_l[j_k]>,  dS_l = dPre_l . W_l^T
 * Duplicate entries keep their own weight and gradient; any finite weight is allowed.  The same values fed as host weights through
 * ggnn_prepare_graph_gcn give the same forward and the same d_h0 / kernel / bias gradients, bit for bit.
 *   ggnn_prepare_graph_gcn_message_weighted   ggnn_prepare_graph_gcn without host weights (same validation and GGNN_ERANGE, CSR, tile plan,
 *                                             pinned image; no plan depends on the weights' values): the batch is marked message-weighted,
 *                                             its slot-weight sections are zero until ggnn_set_message_weights writes them on the device, and
 *                                             with save_for_backward the image also carries the source-keyed CSR's slot map.  The plan text
 *                                             ends in " [message-weighted]".  The host-only twin needs no engine or GPU.
 *   ggnn_set_message_weights                  (see the sparse GGNN's message weights above) message_weights = w, [nnz] (ggnn_num_messages):
 *                                             GGNN_ESTATE on a batch that is not message-weighted; every upload forgets the weights, a forward
 *                                             without them is GGNN_ESTATE, and setting them drops the saved activations.
 *   ggnn_gcn_backward_weighted                ggnn_gcn_backward, and with d_adjacency_weights (DEVICE fp32 [nnz], accumulated into) the weights'
 *                                             gradient: dS_l on every layer and one source-row pass per layer that forms dH_l (the same bits as
 *                                             ggnn_gcn_backward's gather) and each entry's dot product into a per-entry sum, without atomics --
 *                                             bit-identical from call to call in both deterministic modes.  ggnn_gcn_backward is this call with
 *                                             d_adjacency_weights = NULL; a non-NULL one on a batch that is not message-weighted is GGNN_ESTATE. */
int ggnn_prepare_graph_gcn_message_weighted(const ggnn_engine* e, int32_t save_for_backward, int32_t num_nodes, int64_t nnz,
                                            const int64_t* adjacency_list, ggnn_prepared_graph** inout);
int ggnn_host_prepare_graph_gcn_message_weighted(const ggnn_gcn_config* cfg, int32_t num_sms, int32_t save_for_backward, int32_t num_nodes,
                                                 int64_t nnz, const int64_t* adjacency_list, ggnn_prepared_graph** inout);
int ggnn_gcn_backward_weighted(ggnn_engine* e, const float* d_h_out, const ggnn_gcn_layer_grads* grads, int32_t num_layers, float* d_h0,
                               float* d_adjacency_weights, ggnn_stream_t stream);

/* ---- Device-resident datasets: the training graphs uploaded once, every batch of whole graphs assembled on the device.
 * Graphs never share edges, so a batch's graph image is its graphs' pieces (CSR slice, in-degrees, denominators, source-keyed CSR,
 * attention slot map, streaming tables, slot weights) laid end to end with offsets.  A dataset holds those pieces, built once per graph at
 * creation; a batch then costs O(number of graphs) on the host and a few kernels on the device, with no per-batch PCIe traffic but its
 * table of per-graph offsets.  Batches are bit for bit the batches the packers build: the same image as ggnn_prepared_graph_image, the
 * same h0, targets and readout map.
 *
 *   ggnn_dataset_create_sparse   GGNN engine.  num_graphs graphs; node_counts [N]; per edge type t, edge_lists[t] -> [E_t, 2] int32
 *                                GRAPH-LOCAL (source, target) pairs of all graphs in graph order, each graph's in the reference's message
 *                                order, with edge_offsets [T][N+1] int64 (graph i's type-t edges are rows edge_offsets[t][i] ..
 *                                edge_offsets[t][i+1]); num_incoming_edges_per_type [sum V, T]; annotations [sum V, annotation_size] (the
 *                                first columns of h0; annotation_size <= hidden_size); labels / label_mask [N, num_tasks].
 *   ggnn_dataset_create_gcn      GCN engine.  adjacency_lists [sum nnz, 2] int64 graph-local (row i = output, column j = input) with
 *                                entry_offsets [N+1], adjacency_weights [sum nnz] fp32 (as ggnn_prepare_graph_gcn takes them); the rest as above.
 * Both validate every index (GGNN_ERANGE names the graph and the edge), record the engine's model shape (model, T, D, precision, SM count),
 * build the pieces and upload them in one copy on `stream`, returning after it completed.  for_training = 1 also builds the source-keyed
 * CSR that batches with save_for_backward need.  The source arrays stay the caller's; the dataset owns its device memory (an allocation
 * failure returns GGNN_ECUDA naming the size).  *out is allocated even when the call fails: read ggnn_dataset_error, then free it.  The
 * ggnn_host_* twins build the same host summaries without an engine or a GPU (for a host of num_sms SMs): their batches can be planned
 * and inspected, not adopted.
 *   ggnn_dataset_create_dense    GGNN engine, the dense model's graphs (dense:30-36, 132-164).  feature_counts [N] (rows of node_features);
 *                                graphs [sum E, 3] int64, the reference's raw (src, bond, dest) triples with graph_offsets [N+1]
 *                                (graph i's rows graph_offsets[i] .. graph_offsets[i+1]); tie_fwd_bkwd as the model's parameter (0: the
 *                                reverse direction is type bond-1 + T/2); annotations [sum features, annotation_size]; labels / label_mask
 *                                as above.  Every triple is the two 0/1 entries A[bond-1, dest, src] and A[bond-1+bwd, src, dest]:
 *                                duplicates collapse, a self-loop is one entry, the in-degree is the number of distinct sources, and each
 *                                type's messages are in the order ggnn_prepare_graph_dense scans the matrix (target row, source column).
 *                                A graph spans V_g = max(features, largest id + 1) nodes, stored unpadded; rows at or beyond its feature
 *                                count are masked out (node_mask 0, h0 zero) but still send and receive messages.  A bond type outside
 *                                1 .. T - bwd or a negative id is GGNN_ERANGE naming the graph and the edge; an attention model is
 *                                GGNN_EUNSUPPORTED (the dense model has none). */
typedef struct ggnn_dataset ggnn_dataset;
int ggnn_dataset_create_sparse(const ggnn_engine* e, int32_t for_training, int32_t num_graphs, const int64_t* node_counts,
                               const int32_t* const* edge_lists, const int64_t* edge_offsets, const float* num_incoming_edges_per_type,
                               int32_t annotation_size, const float* annotations, int32_t num_tasks, const float* labels, const float* label_mask,
                               ggnn_stream_t stream, ggnn_dataset** out);
int ggnn_host_dataset_create_sparse(const ggnn_config* cfg, int32_t num_sms, int32_t for_training, int32_t num_graphs, const int64_t* node_counts,
                                    const int32_t* const* edge_lists, const int64_t* edge_offsets, const float* num_incoming_edges_per_type,
                                    int32_t annotation_size, const float* annotations, int32_t num_tasks, const float* labels,
                                    const float* label_mask, ggnn_dataset** out);
int ggnn_dataset_create_gcn(const ggnn_engine* e, int32_t for_training, int32_t num_graphs, const int64_t* node_counts, const int64_t* adjacency_lists,
                            const int64_t* entry_offsets, const float* adjacency_weights, int32_t annotation_size, const float* annotations,
                            int32_t num_tasks, const float* labels, const float* label_mask, ggnn_stream_t stream, ggnn_dataset** out);
int ggnn_host_dataset_create_gcn(const ggnn_gcn_config* cfg, int32_t num_sms, int32_t for_training, int32_t num_graphs, const int64_t* node_counts,
                                 const int64_t* adjacency_lists, const int64_t* entry_offsets, const float* adjacency_weights,
                                 int32_t annotation_size, const float* annotations, int32_t num_tasks, const float* labels,
                                 const float* label_mask, ggnn_dataset** out);
int ggnn_free_dataset(ggnn_dataset* d);
const char* ggnn_dataset_error(const ggnn_dataset* d);
/* The two halves of a dataset batch, like ggnn_prepare_graph_* / ggnn_set_graph_prepared:
 *   ggnn_dataset_prepare_batch   host only, from the dataset's summaries (no edge is read, the device is not touched but for the pinned
 *                                table): the batch of graph_ids [num_graphs] (int64 dataset indices, in batch order; an id out of range is
 *                                GGNN_ERANGE) -- its offsets, its cut points through the same tile planner, the image layout -- and a small
 *                                pinned table of tile starts, per-graph offsets and the graph ids (ggnn_dataset_batch_slots).  Reads the
 *                                dataset and nothing else: callable from a producer thread.  save_for_backward 1 needs a training dataset
 *                                with targets (a dataset created with num_tasks = 0 is for prediction: GGNN_EINVAL).  *inout as for ggnn_prepare_graph_sparse
 *                                (a rebuilt batch first waits for its previous table upload).
 *   ggnn_set_graph_dataset       engine thread: adopts the plan and enqueues on `stream` the table upload and the kernels that write the
 *                                batch's graph image into the engine's graph buffer, h0 [V, D] (the annotation columns, zeros elsewhere),
 *                                target_values / target_mask [num_tasks, num_graphs] (DEVICE buffers of the caller) and the readout map
 *                                (what ggnn_readout_set_graphs builds from the batch's graph_nodes_list).  No host synchronisation, no
 *                                atomics, no allocation but the engine's buffers growing as for any upload.  The batch must stay alive
 *                                until the stream passed it.  Like every graph upload it first forgets the previous batch (ggnn_layer_state,
 *                                saved activations) -- and the readout map it replaces.  A batch prepared for an engine of another shape or
 *                                on another device is refused (GGNN_EINVAL; another model: GGNN_ESTATE).
 * A batch reads its dataset in every call: the dataset must outlive every batch prepared from it (free the batches first).
 * ggnn_dataset_batch_info: as ggnn_prepared_graph_info, plus the tile starts [num_tiles + 1] and, for LOCAL (tile-local) plans, the values of
 * ggnn_prepared_graph_tile_stats -- other plans' launches do not read them, and they are 0 there.  NULL pointers are skipped.
 *
 * Dense datasets have their own pair of calls; each kind refuses the other's dataset or batch with GGNN_EINVAL:
 *   ggnn_dataset_prepare_batch_dense   the batch ggnn_prepare_graph_dense builds from pack_dense_batch's [b, T, v, v] matrix, with
 *                                      v = nodes_per_graph: graph i owns rows i*v .. i*v+v-1, its V_g rows first, then v - V_g isolated
 *                                      padding rows.  A graph with V_g > v is GGNN_EINVAL naming it.  Plan text, tile starts, layout and
 *                                      image are those of the host-built batch, the plan text ending in " [binary dense adjacency -> CSR]".
 *   ggnn_set_graph_dataset_dense       as ggnn_set_graph_dataset, plus node_mask [V = b*v] (DEVICE, the caller's): 1 for the rows below
 *                                      the graph's feature count, 0 elsewhere.  The readout map is that of ggnn_readout_set_graphs(b,
 *                                      nodes_per_graph = v, node_mask): the fused readout sums each graph's masked rows. */
typedef struct ggnn_dataset_batch ggnn_dataset_batch;
int ggnn_dataset_prepare_batch(const ggnn_dataset* d, int32_t save_for_backward, const int64_t* graph_ids, int32_t num_graphs,
                               ggnn_dataset_batch** inout);
int ggnn_dataset_batch_info(const ggnn_dataset_batch* b, int32_t* num_nodes, int64_t* num_messages, int32_t* num_tiles, int64_t* image_bytes,
                            int32_t* is_streaming, char* plan_text, int32_t plan_text_capacity, int32_t* tile_start, int32_t* max_tile_msgs,
                            int32_t* max_tile_types);
int ggnn_free_dataset_batch(ggnn_dataset_batch* b);
const char* ggnn_dataset_batch_error(const ggnn_dataset_batch* b);
int ggnn_set_graph_dataset(ggnn_engine* e, ggnn_dataset_batch* b, float* h0, float* target_values, float* target_mask, ggnn_stream_t stream);
int ggnn_dataset_create_dense(const ggnn_engine* e, int32_t for_training, int32_t num_graphs, const int64_t* feature_counts, const int64_t* graphs,
                              const int64_t* graph_offsets, int32_t tie_fwd_bkwd, int32_t annotation_size, const float* annotations,
                              int32_t num_tasks, const float* labels, const float* label_mask, ggnn_stream_t stream, ggnn_dataset** out);
int ggnn_host_dataset_create_dense(const ggnn_config* cfg, int32_t num_sms, int32_t for_training, int32_t num_graphs, const int64_t* feature_counts,
                                   const int64_t* graphs, const int64_t* graph_offsets, int32_t tie_fwd_bkwd, int32_t annotation_size,
                                   const float* annotations, int32_t num_tasks, const float* labels, const float* label_mask, ggnn_dataset** out);
int ggnn_dataset_prepare_batch_dense(const ggnn_dataset* d, int32_t save_for_backward, const int64_t* graph_ids, int32_t num_graphs,
                                     int32_t nodes_per_graph, ggnn_dataset_batch** inout);
int ggnn_set_graph_dataset_dense(ggnn_engine* e, ggnn_dataset_batch* b, float* h0, float* target_values, float* target_mask, float* node_mask,
                                 ggnn_stream_t stream);
/* The engine's current graph image copied back to the host (the counterpart of ggnn_prepared_graph_image, whatever upload made it):
 * *image_bytes gets its size; dst NULL only asks for it.  Synchronises `stream`. */
int ggnn_graph_image(ggnn_engine* e, void* dst, int64_t capacity, int64_t* image_bytes, ggnn_stream_t stream);

/* Introspection used by the parity tests and the benchmark. */
int ggnn_num_messages(const ggnn_engine* e, int64_t* out);
/* Copies the engine's device CSR back: row_ptr [V*T+1] (rows keyed target*T+type), src [M], msg [M]. */
int ggnn_get_csr(ggnn_engine* e, int32_t* row_ptr, int32_t* src, int32_t* msg);
/* Pointer to node_states_per_layer[layer] (layer 0 = h0, num_layers = final) of the last forward.  GGNN_ESTATE until a forward has run on
 * the current graph (every graph upload clears it), and for 0 < layer < num_layers when the last forward did not write those layers: the
 * GCN wgmma kernel's LOCAL plan without save_for_backward, and a model without timesteps. */
int ggnn_layer_state(ggnn_engine* e, int32_t layer, const float** dev_ptr);
/* Device-to-device copy of that state into dst [V, D] on `stream`. */
int ggnn_copy_layer_state(ggnn_engine* e, int32_t layer, float* dst, ggnn_stream_t stream);
/* Kernel launches issued by the last forward / backward call, and plan description text. */
int ggnn_last_launch_count(const ggnn_engine* e);
const char* ggnn_plan_description(const ggnn_engine* e);

#ifdef __cplusplus
}
#endif
#endif /* GGNN_B200_H */
