"""CPU ORACLE for the GGNN propagation step -- TEST INFRASTRUCTURE ONLY.

This file restates, on the CPU, the arithmetic of the reference's hot path:

* ``chem_tensorflow_sparse.py:117-218``  (``SparseGGNNChemModel.compute_final_node_representations``)
* ``chem_tensorflow_sparse.py:63-115``   (weight shapes / initialisers)
* ``chem_tensorflow_dense.py:93-117``    (``DenseGGNNChemModel.compute_final_node_representations``)
* ``chem_tensorflow_dense.py:30-36``     (dense adjacency layout ``amat[e, dest, src]``)
* ``utils.py:8-13``                      (``SMALL_NUMBER``, ``glorot_init``)

The cell arithmetic lives in an un-vendored third-party dependency, ``tensorflow==1.3.0``
(``requirements.txt:2``): ``tf.nn.rnn_cell.GRUCell`` / ``BasicRNNCell`` / ``_linear`` /
``DropoutWrapper`` in ``tensorflow/python/ops/rnn_cell_impl.py`` of that release.  Its published
algorithm is restated here from knowledge of the release (TF is not installable in this image, see
SURVEY.md section 8c):

    GRUCell:       [r|u] = sigmoid([x, h] . K_g + b_g)          (b_g initialised to 1.0)
                   c     = act([x, r*h] . K_c + b_c)
                   h'    = u*h + (1-u)*c
    BasicRNNCell:  h'    = act([x, h] . K + b)
    CudnnCompatibleGRUCell (tf.contrib.cudnn_rnn, TF >= 1.4 -- what sparse:105-108 instantiates; not in 1.3.0 itself):
                   gates as GRUCell;  c = tanh(x . K_in + b_in + r * (h . K_hid + b_hid));  h' = u*h + (1-u)*c
    DropoutWrapper(state_keep_prob=1.0): identity on the new state.

PARITY: the reference ships no tests, golden vectors or fixtures and TensorFlow 1.3 cannot run here, so the reference itself pins
nothing ("parity unpinned" in the strict sense).  What pins this oracle instead:
(1) fixtures computed by the reference's OWN graph-building code: ``prepare_specific_graph_model`` /
    ``compute_final_node_representations`` / ``gated_regression`` of both model files are imported unmodified and evaluated in float64
    over a NumPy stand-in for the ``tf.*`` calls they make (tests/golden/tf_shim.py, generator make_reference_graph_golden.py, batches
    from the reference's own packers); every statement of this oracle reproduces them to 1e-12 (tests/test_oracle.py).  That fixes
    the dataflow -- gather/matmul/concat/segment-sum order, bias and mean, residual selection, the attention softmax, the readout --
    to the reference's code.  NOT covered: the arithmetic inside TensorFlow's own ops (GRUCell / BasicRNNCell, see above), restated
    from the 1.3 release in both places;
(2) its own float64 loop-level statement vs. its vectorised fp32 statements, and an independent plain-C restatement
    (oracle/ggnn_oracle.c, message by message in double precision, no shared code) that must agree to 1e-12;
(3) the sparse == dense cross-implementation identity the reference's two model files imply;
(4) hand-derived closed-form tiny graphs;
(5) batches produced by the reference's *own* NumPy packing code (tests/golden/make_golden.py).

Only ``tests/``, ``__graft_entry__.smoke()`` and ``bench.py``'s CPU-baseline legs may import this
module.  The product path (``gated_graph_neural_network_samples_b200``) never does.
"""
from __future__ import annotations

import numpy as np

SMALL_NUMBER = 1e-7  # utils.py:8


# ----------------------------------------------------------------------------------------------
# Initialisers (utils.py:11-13, chem_tensorflow_sparse.py:86-115, chem_tensorflow_dense.py:84-91)
# ----------------------------------------------------------------------------------------------
def glorot_init(shape, rng):
    """utils.py:11-13 -- uniform(+-sqrt(6/(shape[-2]+shape[-1]))) as float32."""
    r = np.sqrt(6.0 / (shape[-2] + shape[-1]))
    return rng.uniform(low=-r, high=r, size=shape).astype(np.float32)


def residual_inputs_of_layer(params, layer_idx):
    """chem_tensorflow_sparse.py:140-145 -- list of layer indices whose states feed layer_idx."""
    res = params.get("residual_connections", {}) or {}
    lst = res.get(str(layer_idx))
    return [] if lst is None else list(lst)


def init_sparse_weights(params, num_edge_types, rng, edge_bias_scale=0.1, attention_scale=0.0):
    """Per-layer weights with the shapes of chem_tensorflow_sparse.py:86-115.

    edge_weights:  glorot on the *stacked* [T*D, D] shape (sparse:88) reshaped to [T, D, D] (sparse:90)
    edge_biases:   [T, D]; the reference initialises zeros (sparse:99) -- we draw U(-s, s) so the bias
                   path is exercised (SURVEY 8d)
    cell kernels:  glorot-uniform (TF default initializer for ``_linear``), gate bias 1.0, cand bias 0.
    """
    D = int(params["hidden_size"])
    T = int(num_edge_types)
    layers = []
    for layer_idx, _ in enumerate(params["layer_timesteps"]):
        R = len(residual_inputs_of_layer(params, layer_idx))
        din = D * (1 + R)
        w = {"edge_weights": glorot_init([T * D, D], rng).reshape(T, D, D)}
        if params.get("use_edge_bias", False):
            w["edge_biases"] = rng.uniform(-edge_bias_scale, edge_bias_scale, size=(T, D)).astype(np.float32)
        if params.get("use_propagation_attention", False):   # sparse:94-96: ones; attention_scale > 0 perturbs them for the tests
            w["edge_type_attention_weights"] = (np.ones(T) + attention_scale * rng.uniform(-1, 1, T)).astype(np.float32)
        cell = params.get("graph_rnn_cell", "GRU").lower()
        if cell == "gru":
            w["gate_kernel"] = glorot_init([din + D, 2 * D], rng)
            w["gate_bias"] = np.ones([2 * D], dtype=np.float32)
            w["cand_kernel"] = glorot_init([din + D, D], rng)
            w["cand_bias"] = np.zeros([D], dtype=np.float32)
        elif cell == "cudnncompatiblegrucell":   # sparse:105-108; _linear initialises each projection on its own shape
            w["gate_kernel"] = glorot_init([din + D, 2 * D], rng)
            w["gate_bias"] = np.ones([2 * D], dtype=np.float32)
            w["cand_kernel"] = np.concatenate([glorot_init([din, D], rng), glorot_init([D, D], rng)], axis=0)
            w["cand_bias"] = rng.uniform(-0.1, 0.1, size=D).astype(np.float32)          # the reference initialises zeros: perturbed so that
            w["cand_hidden_bias"] = rng.uniform(-0.1, 0.1, size=D).astype(np.float32)   # both bias paths are exercised
        elif cell == "rnn":
            w["rnn_kernel"] = glorot_init([din + D, D], rng)
            w["rnn_bias"] = np.zeros([D], dtype=np.float32)
        else:
            raise Exception("Unknown RNN cell type '%s'." % cell)  # sparse:112
        layers.append(w)
    return layers


def init_dense_weights(params, num_edge_types, rng, edge_bias_scale=0.1):
    """chem_tensorflow_dense.py:84-91 -- one shared [T,D,D] weight, [T,1,D] bias, one GRU cell."""
    D = int(params["hidden_size"])
    T = int(num_edge_types)
    w = {"edge_weights": glorot_init([T, D, D], rng)}
    if params.get("use_edge_bias", True):
        w["edge_biases"] = rng.uniform(-edge_bias_scale, edge_bias_scale, size=(T, 1, D)).astype(np.float32)
    w["gate_kernel"] = glorot_init([2 * D, 2 * D], rng)
    w["gate_bias"] = np.ones([2 * D], dtype=np.float32)
    w["cand_kernel"] = glorot_init([2 * D, D], rng)
    w["cand_bias"] = np.zeros([D], dtype=np.float32)
    return w


# ----------------------------------------------------------------------------------------------
# Cells (tensorflow==1.3.0 rnn_cell_impl.py semantics, see module docstring)
# ----------------------------------------------------------------------------------------------
def _activation(name):
    name = name.lower()
    if name == "tanh":
        return np.tanh
    if name == "relu":
        return lambda v: np.maximum(v, 0)
    raise Exception("Unknown activation function type '%s'." % name)  # sparse:81


def _sigmoid(v):
    return 1.0 / (1.0 + np.exp(-v))


def gru_cell(x, h, w, act):
    """TF-1.3 GRUCell.__call__: rows of the kernels are ordered [inputs ; state]."""
    D = h.shape[-1]
    ru = _sigmoid(np.concatenate([x, h], axis=-1) @ w["gate_kernel"] + w["gate_bias"])
    r, u = ru[..., :D], ru[..., D:]
    c = act(np.concatenate([x, r * h], axis=-1) @ w["cand_kernel"] + w["cand_bias"])
    return u * h + (1.0 - u) * c


def cudnn_gru_cell(x, h, w, act):
    """tf.contrib.cudnn_rnn.CudnnCompatibleGRUCell.call (TF >= 1.4; the class the reference instantiates at sparse:105-108):
    gates as GRUCell; c = act(_linear(x; candidate/input_projection) + r * _linear(h; candidate/hidden_projection)) -- the reset gate is
    applied AFTER the recurrent product.  ``cand_kernel`` stacks [input_projection/kernel ; hidden_projection/kernel]."""
    D = h.shape[-1]
    din = x.shape[-1]
    ru = _sigmoid(np.concatenate([x, h], axis=-1) @ w["gate_kernel"] + w["gate_bias"])
    r, u = ru[..., :D], ru[..., D:]
    c = act(x @ w["cand_kernel"][:din] + w["cand_bias"] + r * (h @ w["cand_kernel"][din:] + w["cand_hidden_bias"]))
    return u * h + (1.0 - u) * c


def rnn_cell(x, h, w, act):
    """TF-1.3 BasicRNNCell.__call__."""
    return act(np.concatenate([x, h], axis=-1) @ w["rnn_kernel"] + w["rnn_bias"])


def _cell_fn(params):
    act = _activation(params.get("graph_rnn_activation", "tanh"))
    cell = params.get("graph_rnn_cell", "GRU").lower()
    if cell == "gru":
        return lambda x, h, w: gru_cell(x, h, w, act)
    if cell == "rnn":
        return lambda x, h, w: rnn_cell(x, h, w, act)
    if cell == "cudnncompatiblegrucell":
        return lambda x, h, w: cudnn_gru_cell(x, h, w, act)
    raise Exception("Unknown RNN cell type '%s'." % cell)


def _cast_weights(weights, dtype):
    if isinstance(weights, dict):
        return {k: np.asarray(v, dtype=dtype) for k, v in weights.items()}
    return [{k: np.asarray(v, dtype=dtype) for k, v in w.items()} for w in weights]


# ----------------------------------------------------------------------------------------------
# Sparse propagation, loop-level literal statement (float64 by default) -- THE SPEC
# ----------------------------------------------------------------------------------------------
def sparse_propagation_loops(h0, adjacency_lists, num_incoming_edges_per_type, weights, params,
                             dtype=np.float64, return_all_layers=False):
    """Literal restatement of chem_tensorflow_sparse.py:117-218 with explicit Python loops.

    h0:                            [V, D]     initial_node_representation        (sparse:65)
    adjacency_lists[e]:            [E_e, 2]   int32, col0 = source, col1 = target (sparse:67,125,160)
    num_incoming_edges_per_type:   [V, T]     float                               (sparse:69)
    The scatter-add runs serially in message order (type-major, sparse:124-129,168), which is what the
    TF-1.3 CPU ``unsorted_segment_sum`` functor does.
    """
    h0 = np.asarray(h0, dtype=dtype)
    indeg = np.asarray(num_incoming_edges_per_type, dtype=dtype)
    weights = _cast_weights(weights, dtype)
    V, D = h0.shape
    cell = _cell_fn(params)
    node_states_per_layer = [h0]                                                   # sparse:118-119
    for layer_idx, num_timesteps in enumerate(params["layer_timesteps"]):          # sparse:131
        w = weights[layer_idx]
        residual_states = [node_states_per_layer[i]
                           for i in residual_inputs_of_layer(params, layer_idx)]    # sparse:140-145
        node_states_per_layer.append(node_states_per_layer[-1])                    # sparse:152
        for _step in range(num_timesteps):                                         # sparse:153
            h = node_states_per_layer[-1]
            incoming = np.zeros((V, D), dtype=dtype)
            attention = None
            if params.get("use_propagation_attention", False):                     # sparse:170-196, message by message
                scores = {}
                for e, adj in enumerate(adjacency_lists):
                    for i, (src, tgt) in enumerate(np.asarray(adj).reshape(-1, 2)):
                        scores[(e, i)] = (int(tgt), float(h[src] @ h[tgt]) * float(w["edge_type_attention_weights"][e]))
                mx, ssum = {}, {}
                for tgt, sc in scores.values():
                    mx[tgt] = max(mx.get(tgt, -np.inf), sc)
                for tgt, sc in scores.values():
                    ssum[tgt] = ssum.get(tgt, 0.0) + np.exp(sc - mx[tgt])
                attention = {k: np.exp(sc - mx[tgt]) / (ssum[tgt] + SMALL_NUMBER) for k, (tgt, sc) in scores.items()}
            for e, adj in enumerate(adjacency_lists):                              # sparse:159
                adj = np.asarray(adj).reshape(-1, 2)
                for i, (src, tgt) in enumerate(adj):                               # gather :161, matmul :163
                    if not (0 <= src < V and 0 <= tgt < V):
                        raise IndexError("edge (%d,%d) out of range for V=%d" % (src, tgt, V))
                    msg = h[src] @ w["edge_weights"][e]
                    incoming[tgt] += msg if attention is None else msg * attention[(e, i)]   # segment_sum :198
            if params.get("use_edge_bias", False):                                 # sparse:202-204
                incoming = incoming + indeg @ w["edge_biases"].reshape(-1, D)
            if params.get("use_edge_msg_avg_aggregation", False):                  # sparse:206-209
                incoming = incoming / (indeg.sum(axis=-1, keepdims=True) + dtype(SMALL_NUMBER))
            x = np.concatenate(residual_states + [incoming], axis=-1)              # sparse:211-212
            node_states_per_layer[-1] = cell(x, h, w)                              # sparse:215-216
    if return_all_layers:
        return node_states_per_layer
    return node_states_per_layer[-1]                                               # sparse:218


# ----------------------------------------------------------------------------------------------
# Sparse propagation, vectorised NumPy (same op order as the TF graph; any dtype)
# ----------------------------------------------------------------------------------------------
def sparse_propagation_np(h0, adjacency_lists, num_incoming_edges_per_type, weights, params,
                          dtype=np.float32, return_all_layers=False):
    """Vectorised statement: gather -> per-type matmul -> concat -> ordered scatter-add -> (+bias)
    -> (/deg) -> concat residuals -> cell.  ``np.add.at`` accumulates in index order like the serial
    CPU segment-sum."""
    h0 = np.asarray(h0, dtype=dtype)
    indeg = np.asarray(num_incoming_edges_per_type, dtype=dtype)
    weights = _cast_weights(weights, dtype)
    V, D = h0.shape
    cell = _cell_fn(params)
    adjs = [np.asarray(a, dtype=np.int64).reshape(-1, 2) for a in adjacency_lists]
    for a in adjs:
        if a.size and (a.min() < 0 or a.max() >= V):
            raise IndexError("edge index out of range")
    message_targets = np.concatenate([a[:, 1] for a in adjs]) if adjs else np.zeros(0, np.int64)
    states = [h0]
    for layer_idx, num_timesteps in enumerate(params["layer_timesteps"]):
        w = weights[layer_idx]
        residual_states = [states[i] for i in residual_inputs_of_layer(params, layer_idx)]
        states.append(states[-1])
        for _ in range(num_timesteps):
            h = states[-1]
            msgs = [h[a[:, 0]] @ w["edge_weights"][e] for e, a in enumerate(adjs)]
            messages = np.concatenate(msgs, axis=0) if msgs else np.zeros((0, D), dtype)
            if params.get("use_propagation_attention", False) and messages.shape[0]:             # sparse:170-196
                message_types = np.concatenate([np.full(a.shape[0], e, np.int64) for e, a in enumerate(adjs)])
                src_states = np.concatenate([h[a[:, 0]] for a in adjs], axis=0)
                scores = np.einsum("mi,mi->m", src_states, h[message_targets]) * w["edge_type_attention_weights"][message_types]
                mx = np.full(V, -np.inf, dtype); np.maximum.at(mx, message_targets, scores)      # unsorted_segment_max
                exped = np.exp(scores - mx[message_targets])
                ssum = np.zeros(V, dtype); np.add.at(ssum, message_targets, exped)
                messages = messages * (exped / (ssum[message_targets] + dtype(SMALL_NUMBER)))[:, None]
            incoming = np.zeros((V, D), dtype=dtype)
            np.add.at(incoming, message_targets, messages)
            if params.get("use_edge_bias", False):
                incoming = incoming + indeg @ w["edge_biases"].reshape(-1, D)
            if params.get("use_edge_msg_avg_aggregation", False):
                incoming = incoming / (indeg.sum(axis=-1, keepdims=True) + dtype(SMALL_NUMBER))
            x = np.concatenate(residual_states + [incoming], axis=-1)
            states[-1] = cell(x, h, w).astype(dtype)
    return states if return_all_layers else states[-1]


# ----------------------------------------------------------------------------------------------
# Dense propagation (chem_tensorflow_dense.py:93-117)
# ----------------------------------------------------------------------------------------------
def graph_to_adj_mat(graph, max_n_vertices, num_edge_types, tie_fwd_bkwd=True):
    """chem_tensorflow_dense.py:30-36 -- amat[e-1, dest, src] = 1 (assignment: duplicates collapse)."""
    bwd = 0 if tie_fwd_bkwd else (num_edge_types // 2)
    amat = np.zeros((num_edge_types, max_n_vertices, max_n_vertices))
    for src, e, dest in graph:
        amat[e - 1, dest, src] = 1
        amat[e - 1 + bwd, src, dest] = 1
    return amat


def dense_propagation_loops(h0, adjacency_matrix, weights, params, dtype=np.float64):
    """Literal restatement of chem_tensorflow_dense.py:93-117.

    h0: [b, v, D]; adjacency_matrix: [b, T, v, v] (dense:78-80, transposed to [T,b,v,v] there).
    Padded rows are updated like any other (they are masked only at the readout, dense:126).
    """
    h0 = np.asarray(h0, dtype=dtype)
    A = np.asarray(adjacency_matrix, dtype=dtype)
    w = _cast_weights(weights, dtype)
    b, v, D = h0.shape
    T = A.shape[1]
    act = np.tanh  # tf.contrib.rnn.GRUCell default (dense:88)
    h = h0.reshape(-1, D)                                                          # dense:97
    for _ in range(int(params["num_timesteps"])):                                  # dense:100
        acts = None
        for e in range(T):                                                         # dense:103
            m = (h @ w["edge_weights"][e]).reshape(b, v, D)                        # dense:104-106
            if params.get("use_edge_bias", True):
                m = m + w["edge_biases"].reshape(T, 1, D)[e]                       # dense:107-108
            contrib = np.einsum("bij,bjd->bid", A[:, e], m)                        # dense:110-112
            acts = contrib if acts is None else acts + contrib
        acts = acts.reshape(-1, D)                                                 # dense:113
        h = gru_cell(acts, h, w, act)                                              # dense:115
    return h.reshape(b, v, D)                                                      # dense:116


# ----------------------------------------------------------------------------------------------
# Integer path: the target-sorted CSR an engine must reproduce bit-exactly
# ----------------------------------------------------------------------------------------------
def message_arrays(adjacency_lists):
    """sparse:122-129 -- type-major message order: (src, tgt, type) per message."""
    srcs, tgts, typs = [], [], []
    for e, a in enumerate(adjacency_lists):
        a = np.asarray(a, dtype=np.int32).reshape(-1, 2)
        srcs.append(a[:, 0]); tgts.append(a[:, 1]); typs.append(np.full(a.shape[0], e, np.int32))
    cat = lambda xs: np.concatenate(xs) if xs else np.zeros(0, np.int32)
    return cat(srcs).astype(np.int32), cat(tgts).astype(np.int32), cat(typs).astype(np.int32)


def stable_target_csr(adjacency_lists, V):
    """Stable sort of the messages by target: row_ptr [V+1], then per slot the source node, the edge
    type and the original message id.  Stable => within a target the reference's message order."""
    src, tgt, typ = message_arrays(adjacency_lists)
    order = np.argsort(tgt, kind="stable").astype(np.int32)
    row_ptr = np.zeros(V + 1, dtype=np.int32)
    np.cumsum(np.bincount(tgt, minlength=V), out=row_ptr[1:])
    return row_ptr, src[order], typ[order], order


# ----------------------------------------------------------------------------------------------
# fp32 PyTorch-CPU restatement at the TF graph's op granularity -- the timed "reference CPU path"
# ----------------------------------------------------------------------------------------------
def state_dropout_mask(seed, global_step, V, D, keep):
    """The engine's state-dropout keep mask ([V, D] bool), restated: splitmix64 finaliser of
    ((global_step*V + node)*D + column) + (seed+1)*golden-ratio, top 24 bits as a uniform in [0,1), kept iff < fp32(keep).
    (DropoutWrapper's own random stream is TensorFlow's and cannot be reproduced -- sparse:113-114.)"""
    M = np.uint64(0xFFFFFFFFFFFFFFFF)
    with np.errstate(over="ignore"):
        idx = (np.uint64(global_step) * np.uint64(V) + np.arange(V, dtype=np.uint64)[:, None]) * np.uint64(D) + np.arange(D, dtype=np.uint64)[None, :]
        x = idx + np.uint64((int(seed) + 1) * 0x9E3779B97F4A7C15 & 0xFFFFFFFFFFFFFFFF)
        x ^= x >> np.uint64(30); x *= np.uint64(0xBF58476D1CE4E5B9)
        x ^= x >> np.uint64(27); x *= np.uint64(0x94D049BB133111EB)
        x ^= x >> np.uint64(31)
    u = (x >> np.uint64(40)).astype(np.float32) * np.float32(1.0 / 16777216.0)
    return u < np.float32(keep)


def _apply_state_dropout(h, state_dropout, global_step, mask_width):
    """DropoutWrapper on the new state with the engine's mask (state_dropout_mask).  An engine running a hidden size zero-padded to a
    multiple of 4 draws its mask at the padded width: ``mask_width`` is that width, and the first D columns of its mask apply."""
    import torch
    if state_dropout is None or state_dropout[0] >= 1.0:
        return h
    keep, seed = state_dropout
    V, D = h.shape
    mask = torch.from_numpy(state_dropout_mask(seed, global_step, V, mask_width or D, keep)[:, :D])
    return torch.where(mask, h / float(np.float32(keep)), torch.zeros((), dtype=h.dtype))


def sparse_propagation_torch(h0, adjacency_lists, num_incoming_edges_per_type, weights, params,
                             return_all_layers=False, dtype=None, state_dropout=None, mask_width=None):
    """Same ops and materialisations as sparse:159-216 with torch CPU fp32 kernels:
    index_select (embedding_lookup) -> matmul -> cat -> index_add_ (unsorted_segment_sum) -> matmul bias
    -> divide -> cat -> explicit GRUCell/BasicRNNCell arithmetic.  Inputs may be NumPy or torch.
    ``state_dropout`` = (keep, seed) and ``mask_width``: see _apply_state_dropout."""
    import torch
    dtype = dtype or torch.float32   # float64 + requires_grad tensors give the autograd reference for the backward tests
    t = lambda a: a if isinstance(a, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(a))
    h0 = t(h0).to(dtype)
    indeg = t(num_incoming_edges_per_type).to(dtype)
    adjs = [t(np.asarray(a).reshape(-1, 2) if not isinstance(a, torch.Tensor) else a).long() for a in adjacency_lists]
    V, D = h0.shape
    act_name = params.get("graph_rnn_activation", "tanh").lower()
    act = torch.tanh if act_name == "tanh" else torch.relu
    cell_type = params.get("graph_rnn_cell", "GRU").lower()
    message_targets = torch.cat([a[:, 1] for a in adjs])
    states = [h0]
    global_step = 0   # state_dropout = (keep, seed): DropoutWrapper on the state after every timestep (sparse:113-114,216)
    for layer_idx, num_timesteps in enumerate(params["layer_timesteps"]):
        w = {k: t(v).to(dtype) for k, v in weights[layer_idx].items()}
        residual_states = [states[i] for i in residual_inputs_of_layer(params, layer_idx)]
        states.append(states[-1])
        for _ in range(num_timesteps):
            h = states[-1]
            msgs = []
            for e, a in enumerate(adjs):
                edge_source_states = torch.index_select(h, 0, a[:, 0])
                msgs.append(torch.matmul(edge_source_states, w["edge_weights"][e]))
            messages = torch.cat(msgs, dim=0)
            if params.get("use_propagation_attention", False) and messages.shape[0]:             # sparse:170-196
                message_types = torch.cat([torch.full((a.shape[0],), e, dtype=torch.long) for e, a in enumerate(adjs)])
                src_states = torch.cat([torch.index_select(h, 0, a[:, 0]) for a in adjs], dim=0)
                scores = (src_states * torch.index_select(h, 0, message_targets)).sum(-1) * w["edge_type_attention_weights"][message_types]
                mx = torch.full((V,), -float("inf"), dtype=dtype).scatter_reduce(0, message_targets, scores.detach(), reduce="amax")
                exped = torch.exp(scores - mx[message_targets])
                ssum = torch.zeros(V, dtype=dtype).index_add_(0, message_targets, exped)
                messages = messages * (exped / (ssum[message_targets] + SMALL_NUMBER)).unsqueeze(-1)
            incoming = torch.zeros(V, D, dtype=dtype).index_add_(0, message_targets, messages)
            if params.get("use_edge_bias", False):
                incoming = incoming + torch.matmul(indeg, w["edge_biases"].reshape(-1, D))
            if params.get("use_edge_msg_avg_aggregation", False):
                incoming = incoming / (indeg.sum(dim=-1, keepdim=True) + SMALL_NUMBER)
            x = torch.cat(residual_states + [incoming], dim=-1)
            if cell_type == "gru":
                ru = torch.sigmoid(torch.matmul(torch.cat([x, h], -1), w["gate_kernel"]) + w["gate_bias"])
                r, u = ru[:, :D], ru[:, D:]
                c = act(torch.matmul(torch.cat([x, r * h], -1), w["cand_kernel"]) + w["cand_bias"])
                states[-1] = u * h + (1 - u) * c
            elif cell_type == "cudnncompatiblegrucell":                                          # sparse:105-108
                ru = torch.sigmoid(torch.matmul(torch.cat([x, h], -1), w["gate_kernel"]) + w["gate_bias"])
                r, u = ru[:, :D], ru[:, D:]
                din = x.shape[-1]
                c = act(torch.matmul(x, w["cand_kernel"][:din]) + w["cand_bias"]
                        + r * (torch.matmul(h, w["cand_kernel"][din:]) + w["cand_hidden_bias"]))
                states[-1] = u * h + (1 - u) * c
            else:
                states[-1] = act(torch.matmul(torch.cat([x, h], -1), w["rnn_kernel"]) + w["rnn_bias"])
            states[-1] = _apply_state_dropout(states[-1], state_dropout, global_step, mask_width)
            global_step += 1
    return states if return_all_layers else states[-1]


def dense_propagation_torch(h0, adjacency_matrix, weights, params, dtype=None, state_dropout=None, mask_width=None):
    """dense:100-115 with torch CPU fp32 kernels (matmul / batched matmul / GRUCell arithmetic).  ``state_dropout`` (DropoutWrapper,
    dense:89) as in sparse_propagation_torch, over the [b*v, D] state rows, one global step per timestep."""
    import torch
    dtype = dtype or torch.float32
    t = lambda a: a if isinstance(a, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(a))
    h0 = t(h0).to(dtype)
    A = t(adjacency_matrix).to(dtype).permute(1, 0, 2, 3).contiguous()             # dense:80
    w = {k: t(v).to(dtype) for k, v in weights.items()}
    b, v, D = h0.shape
    T = A.shape[0]
    h = h0.reshape(-1, D)
    for step in range(int(params["num_timesteps"])):
        acts = None
        for e in range(T):
            m = torch.matmul(h, w["edge_weights"][e]).reshape(b, v, D)
            if params.get("use_edge_bias", True):
                m = m + w["edge_biases"].reshape(T, 1, D)[e]
            contrib = torch.matmul(A[e], m)
            acts = contrib if acts is None else acts + contrib
        acts = acts.reshape(-1, D)
        ru = torch.sigmoid(torch.matmul(torch.cat([acts, h], -1), w["gate_kernel"]) + w["gate_bias"])
        r, u = ru[:, :D], ru[:, D:]
        c = torch.tanh(torch.matmul(torch.cat([acts, r * h], -1), w["cand_kernel"]) + w["cand_bias"])
        h = _apply_state_dropout(u * h + (1 - u) * c, state_dropout, step, mask_width)
    return h.reshape(b, v, D)


def gated_regression_torch(last_h, h0, w_gate, b_gate, w_trans, b_trans, graph_nodes_list=None, num_graphs=None, node_mask=None,
                           dtype=None):
    """gated_regression of sparse:220-231 (``graph_nodes_list`` given: unsorted_segment_sum over graphs) or dense:119-129
    (``last_h`` [b, v, D] with ``node_mask`` [b, v]) for readout MLPs without hidden layers (chem_tensorflow.py:153-157,
    utils.py:65-71: one affine map each).  torch CPU; float64 + requires_grad inputs give the autograd reference."""
    import torch
    dtype = dtype or torch.float32
    t = lambda a: a if isinstance(a, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(a))
    last_h, h0 = t(last_h).to(dtype), t(h0).to(dtype)
    w_gate, b_gate, w_trans, b_trans = (t(x).to(dtype) for x in (w_gate, b_gate, w_trans, b_trans))
    D = last_h.shape[-1]
    gate_input = torch.cat([last_h, h0], dim=-1).reshape(-1, 2 * D)
    gated = torch.sigmoid(gate_input @ w_gate.reshape(2 * D, 1) + b_gate) * (last_h.reshape(-1, D) @ w_trans.reshape(D, 1) + b_trans)
    if graph_nodes_list is not None:
        ids = t(np.asarray(graph_nodes_list)).long()
        return torch.zeros(int(num_graphs), 1, dtype=dtype).index_add_(0, ids, gated).squeeze(-1)
    gated = gated.reshape(last_h.shape[0], last_h.shape[1])
    return (gated * t(node_mask).to(dtype)).sum(dim=1)
