"""Python face of the C ABI (include/ggnn_b200.h): one ``PropagationEngine`` per model instance and GPU.

PyTorch is used for device memory and streams only; all arithmetic of the propagation step runs in
libggnn_b200.so (hand-written sm_90a kernels).  There is no fallback: a missing library or GPU raises.
"""
from __future__ import annotations

import ctypes as C
from typing import Dict, List, Optional, Sequence

import numpy as np

from . import _lib, packing

PRECISIONS = {"fp32": 0, "bf16x3": 1, "bf16": 2}
BACKWARD_PRECISIONS = ("fp32", "bf16x3")   # ggnn_set_backward_precision
WEIGHT_FIELDS = ("edge_weights", "edge_biases", "gate_kernel", "gate_bias", "cand_kernel", "cand_bias", "edge_type_attention_weights",
                 "cand_hidden_bias")
# params['graph_rnn_cell'].lower() (sparse:102-112) -> GGNN_CELL_*
CELL_CODES = {"gru": 0, "rnn": 1, "cudnncompatiblegrucell": 2}


def residual_inputs_of_layer(params: dict, layer_idx: int) -> List[int]:
    """sparse:140-145 -- ``params['residual_connections'].get(str(layer_idx))``."""
    lst = (params.get("residual_connections") or {}).get(str(layer_idx))
    return [] if lst is None else [int(x) for x in lst]


def layer_input_width(params: dict, layer_idx: int) -> int:
    return int(params["hidden_size"]) * (1 + len(residual_inputs_of_layer(params, layer_idx)))


def weight_shapes(params: dict, num_edge_types: int, layer_idx: int) -> Dict[str, tuple]:
    """Shapes of one layer's trainables exactly as created at sparse:86-115 (+ TF-1.3 cell variables)."""
    D, T = int(params["hidden_size"]), int(num_edge_types)
    din = layer_input_width(params, layer_idx)
    shapes = {"edge_weights": (T, D, D)}
    if params.get("use_edge_bias", False):
        shapes["edge_biases"] = (T, D)
    if params.get("use_propagation_attention", False):
        shapes["edge_type_attention_weights"] = (T,)                                            # sparse:94-96
    cell = params.get("graph_rnn_cell", "GRU").lower()
    if cell == "gru":
        shapes.update(gate_kernel=(din + D, 2 * D), gate_bias=(2 * D,), cand_kernel=(din + D, D), cand_bias=(D,))
    elif cell == "cudnncompatiblegrucell":   # sparse:105-108: cand_kernel = [input_projection/kernel ; hidden_projection/kernel]
        shapes.update(gate_kernel=(din + D, 2 * D), gate_bias=(2 * D,), cand_kernel=(din + D, D), cand_bias=(D,), cand_hidden_bias=(D,))
    else:
        shapes.update(cand_kernel=(din + D, D), cand_bias=(D,))
    return shapes


def make_config(params: dict, num_edge_types: int, device: int = 0, precision: str = "fp32", attention_tensor_cores: bool = False,
                cudnn_gru_tensor_cores: bool = False):
    """``ggnn_config`` of a parameter dict (the keys the two hooks read, sparse:40-61) + the ctypes arrays it points into (keep them alive).
    ``attention_tensor_cores``: propagation attention runs at ``precision`` (GGNN_ATT_TENSOR_CORES: on bf16x3 / bf16 the streaming wgmma
    plan) instead of on the fp32 kernels; it changes nothing when attention is off.  ``cudnn_gru_tensor_cores``: CudnnCompatibleGRUCell
    runs at ``precision`` (GGNN_CELL_CUDNN_GRU_TENSOR_CORES: on bf16x3 / bf16 the streaming wgmma plan) instead of on the fp32 kernels; it
    changes nothing for the other cells."""
    steps = [int(s) for s in params["layer_timesteps"]]
    L = len(steps)
    act = params.get("graph_rnn_activation", "tanh").lower()
    if act not in ("tanh", "relu"):
        raise Exception("Unknown activation function type '%s'." % act)                      # sparse:81
    cell = params.get("graph_rnn_cell", "GRU").lower()
    if cell not in CELL_CODES:
        raise Exception("Unknown RNN cell type '%s'." % cell)                                # sparse:112
    if cell == "cudnncompatiblegrucell":
        assert act == "tanh"                                                                 # sparse:106
    offs, flat = [0], []
    for l in range(L):
        flat += residual_inputs_of_layer(params, l)
        offs.append(len(flat))
    keep = ((C.c_int32 * L)(*steps), (C.c_int32 * (L + 1))(*offs), (C.c_int32 * max(len(flat), 1))(*flat))
    att = _lib.ATT_OFF
    if params.get("use_propagation_attention", False):
        att = _lib.ATT_TENSOR_CORES if attention_tensor_cores else _lib.ATT_FP32
    code = CELL_CODES[cell]
    if cell == "cudnncompatiblegrucell" and cudnn_gru_tensor_cores:
        code = _lib.CELL_CUDNN_GRU_TENSOR_CORES
    cfg = _lib.GgnnConfig(int(params["hidden_size"]), int(num_edge_types), L, keep[0], keep[1], keep[2],
                          int(bool(params.get("use_edge_bias", False))), int(bool(params.get("use_edge_msg_avg_aggregation", False))),
                          code, 0 if act == "tanh" else 1, PRECISIONS[precision], int(device), att)
    return cfg, keep


class GgnnError(Exception):
    """Raised for every non-zero return of the C ABI (the reference raises plain ``Exception``s too)."""


def _gcn_list(adjacency_list):
    """A GCN adjacency list as the C ABI takes it: ``[nnz, 2]`` int64, contiguous."""
    lst = np.asarray(adjacency_list)
    if lst.size == 0:
        lst = lst.reshape(0, 2)
    if lst.ndim != 2 or lst.shape[1] != 2:
        raise GgnnError("adjacency_list must be [nnz, 2] (row i = output, column j = input), got shape %s" % (lst.shape,))
    return np.ascontiguousarray(lst, dtype=np.int64)


def _gcn_arrays(adjacency_list, adjacency_weights):
    """The GCN feed as the C ABI takes it: ``[nnz, 2]`` int64 and ``[nnz]`` float32, contiguous (float64 packer weights are cast here,
    as the reference's float32 placeholder does at the feed)."""
    lst = _gcn_list(adjacency_list)
    w = np.asarray(adjacency_weights)
    if w.ndim != 1:
        raise GgnnError("adjacency_weights must be [nnz], got shape %s" % (w.shape,))
    w = np.ascontiguousarray(w, dtype=np.float32)
    if w.shape[0] != lst.shape[0]:
        raise GgnnError("adjacency_weights has %d entries for %d adjacency_list rows" % (w.shape[0], lst.shape[0]))
    return lst, w


class PreparedGraph:
    """Handle of a ``ggnn_prepared_graph`` (include/ggnn_b200.h): the host half of one batch's graph structure."""

    def __init__(self, lib=None):
        self.lib = lib or _lib.load()
        self._h = C.c_void_p()
        self.V = 0

    @classmethod
    def host_only(cls, params: dict, num_edge_types: int, adjacency_lists, num_incoming_edges_per_type, precision: str = "fp32",
                  num_sms: int = 132, save_for_backward: bool = False, reuse: Optional["PreparedGraph"] = None,
                  attention_tensor_cores: bool = False, cudnn_gru_tensor_cores: bool = False) -> "PreparedGraph":
        """``ggnn_host_prepare_graph_sparse``: no engine, no GPU (plain memory instead of pinned).  ``attention_tensor_cores``,
        ``cudnn_gru_tensor_cores``: as in ``make_config``."""
        g = reuse if reuse is not None else cls()
        cfg, keep = make_config(params, num_edge_types, 0, precision, attention_tensor_cores, cudnn_gru_tensor_cores)
        T = int(num_edge_types)
        adjs = [np.ascontiguousarray(np.asarray(a, dtype=np.int32).reshape(-1, 2)) for a in adjacency_lists]
        indeg = np.ascontiguousarray(np.asarray(num_incoming_edges_per_type, dtype=np.float32))
        ptrs = (C.c_void_p * T)(*[a.ctypes.data for a in adjs])
        counts = (C.c_int32 * T)(*[a.shape[0] for a in adjs])
        return g._fill(g.lib.ggnn_host_prepare_graph_sparse, indeg.shape[0], T, C.byref(cfg), int(num_sms), int(bool(save_for_backward)),
                       indeg.shape[0], ptrs, counts, indeg.ctypes.data)

    @classmethod
    def host_only_dense(cls, params: dict, num_edge_types: int, adjacency_matrix, precision: str = "fp32", num_sms: int = 132,
                        save_for_backward: bool = False, reuse: Optional["PreparedGraph"] = None) -> "PreparedGraph":
        """``ggnn_host_prepare_graph_dense``: a 0/1 ``[b, T, v, v]`` adjacency through the CSR builder, no engine, no GPU."""
        g = reuse if reuse is not None else cls()
        cfg, keep = make_config(params, num_edge_types, 0, precision)
        a = np.ascontiguousarray(np.asarray(adjacency_matrix, dtype=np.float32))
        return g._fill(g.lib.ggnn_host_prepare_graph_dense, a.shape[0] * a.shape[2], int(num_edge_types), C.byref(cfg), int(num_sms),
                       int(bool(save_for_backward)), a.shape[0], a.shape[2], a.ctypes.data)

    @classmethod
    def host_only_dense_weighted(cls, params: dict, num_edge_types: int, adjacency_matrix, precision: str = "fp32", num_sms: int = 132,
                                 save_for_backward: bool = False, reuse: Optional["PreparedGraph"] = None) -> "PreparedGraph":
        """``ggnn_host_prepare_graph_dense_weighted``: any ``[b, T, v, v]`` adjacency as ``set_graph_dense_weighted`` builds it (a weighted one
        with its entries as slot weights), no engine, no GPU."""
        g = reuse if reuse is not None else cls()
        cfg, keep = make_config(params, num_edge_types, 0, precision)
        a = np.ascontiguousarray(np.asarray(adjacency_matrix, dtype=np.float32))
        return g._fill(g.lib.ggnn_host_prepare_graph_dense_weighted, a.shape[0] * a.shape[2], int(num_edge_types), C.byref(cfg), int(num_sms),
                       int(bool(save_for_backward)), a.shape[0], a.shape[2], a.ctypes.data)

    @classmethod
    def host_only_dense_device(cls, params: dict, num_edge_types: int, num_graphs: int, num_vertices: int, precision: str = "fp32",
                               num_sms: int = 132, save_for_backward: bool = False, reuse: Optional["PreparedGraph"] = None,
                               cudnn_gru_tensor_cores: bool = False) -> "PreparedGraph":
        """``ggnn_host_prepare_graph_dense_device``: a dense batch whose adjacency comes later on the device (see
        ``PropagationEngine.prepare_graph_dense_device``), from its shape alone, no engine, no GPU."""
        g = reuse if reuse is not None else cls()
        cfg, keep = make_config(params, num_edge_types, 0, precision, False, cudnn_gru_tensor_cores)
        return g._fill(g.lib.ggnn_host_prepare_graph_dense_device, int(num_graphs) * int(num_vertices), int(num_edge_types), C.byref(cfg),
                       int(num_sms), int(bool(save_for_backward)), int(num_graphs), int(num_vertices))

    @classmethod
    def host_only_weighted(cls, params: dict, num_edge_types: int, adjacency_lists, num_incoming_edges_per_type, precision: str = "fp32",
                           num_sms: int = 132, save_for_backward: bool = False, reuse: Optional["PreparedGraph"] = None,
                           cudnn_gru_tensor_cores: bool = False) -> "PreparedGraph":
        """``ggnn_host_prepare_graph_sparse_weighted``: a message-weighted sparse batch (see
        ``PropagationEngine.prepare_graph_sparse_weighted``), no engine, no GPU."""
        g = reuse if reuse is not None else cls()
        cfg, keep = make_config(params, num_edge_types, 0, precision, False, cudnn_gru_tensor_cores)
        T = int(num_edge_types)
        adjs = [np.ascontiguousarray(np.asarray(a, dtype=np.int32).reshape(-1, 2)) for a in adjacency_lists]
        indeg = np.ascontiguousarray(np.asarray(num_incoming_edges_per_type, dtype=np.float32))
        ptrs = (C.c_void_p * T)(*[a.ctypes.data for a in adjs])
        counts = (C.c_int32 * T)(*[a.shape[0] for a in adjs])
        return g._fill(g.lib.ggnn_host_prepare_graph_sparse_weighted, indeg.shape[0], T, C.byref(cfg), int(num_sms), int(bool(save_for_backward)),
                       indeg.shape[0], ptrs, counts, indeg.ctypes.data)

    @classmethod
    def host_only_gcn(cls, hidden_size: int, num_layers: int, num_nodes: int, adjacency_list, adjacency_weights, use_bias: bool = False,
                      precision: str = "fp32", num_sms: int = 132, save_for_backward: bool = False,
                      reuse: Optional["PreparedGraph"] = None, wide_hidden: bool = False) -> "PreparedGraph":
        """``ggnn_host_prepare_graph_gcn``: a GCN batch (``[nnz, 2]`` int64 (row i = output, column j = input) list and ``[nnz]`` weights)
        through the same builder, no engine, no GPU.  ``wide_hidden``: as for ``GCNEngine``."""
        g = reuse if reuse is not None else cls()
        cfg = _lib.GcnConfig(int(hidden_size), int(num_layers), int(bool(use_bias)), PRECISIONS[precision], 0, int(bool(wide_hidden)))
        lst, w = _gcn_arrays(adjacency_list, adjacency_weights)
        return g._fill(g.lib.ggnn_host_prepare_graph_gcn, int(num_nodes), 1, C.byref(cfg), int(num_sms), int(bool(save_for_backward)),
                       int(num_nodes), lst.shape[0], lst.ctypes.data, w.ctypes.data)

    @classmethod
    def host_only_gcn_message_weighted(cls, hidden_size: int, num_layers: int, num_nodes: int, adjacency_list, use_bias: bool = False,
                                       precision: str = "fp32", num_sms: int = 132, save_for_backward: bool = False,
                                       reuse: Optional["PreparedGraph"] = None, wide_hidden: bool = False) -> "PreparedGraph":
        """``ggnn_host_prepare_graph_gcn_message_weighted``: a GCN batch whose adjacency weights come later on the device (see
        ``GCNEngine.prepare_graph_gcn_message_weighted``), no engine, no GPU."""
        g = reuse if reuse is not None else cls()
        cfg = _lib.GcnConfig(int(hidden_size), int(num_layers), int(bool(use_bias)), PRECISIONS[precision], 0, int(bool(wide_hidden)))
        lst = _gcn_list(adjacency_list)
        return g._fill(g.lib.ggnn_host_prepare_graph_gcn_message_weighted, int(num_nodes), 1, C.byref(cfg), int(num_sms),
                       int(bool(save_for_backward)), int(num_nodes), lst.shape[0], lst.ctypes.data)

    def _fill(self, prepare, V: int, T: int, *args) -> "PreparedGraph":
        """Runs the C prepare call ``prepare(*args, &handle)`` into this handle (the call allocates it when empty)."""
        h = C.c_void_p(self._h.value)
        rc = prepare(*args, C.byref(h))
        self._h = h
        if rc != 0:
            raise GgnnError(self.lib.ggnn_prepared_graph_error(self._h).decode())
        self.V, self.T = V, T
        return self

    def slot_weights(self, source_order: bool = False) -> np.ndarray:
        """A GCN graph's per-slot adjacency weights in target-CSR order (``source_order``: in source-CSR order, backward graphs only)."""
        out = np.empty(self.info()["num_messages"], np.float32)
        rc = self.lib.ggnn_prepared_graph_slot_weights(self._h, None if source_order else out.ctypes.data, out.ctypes.data if source_order else None)
        if rc != 0:
            raise GgnnError("not a GCN prepared graph%s" % (" prepared for backward" if source_order else ""))
        return out

    def info(self) -> dict:
        V, M, nt, nb, st = C.c_int32(), C.c_int64(), C.c_int32(), C.c_int64(), C.c_int32()
        buf = C.create_string_buffer(512)
        if self.lib.ggnn_prepared_graph_info(self._h, C.byref(V), C.byref(M), C.byref(nt), C.byref(nb), C.byref(st), buf, 512) != 0:
            raise GgnnError("the prepared graph is empty")
        return {"num_nodes": V.value, "num_messages": M.value, "num_tiles": nt.value, "image_bytes": nb.value, "streaming": bool(st.value),
                "plan": buf.value.decode()}

    def arrays(self, T: int) -> dict:
        i = self.info()
        V, M = i["num_nodes"], i["num_messages"]
        out = {"row_ptr": np.empty(V * T + 1, np.int32), "src": np.empty(M, np.int32), "msg": np.empty(M, np.int32),
               "tile_start": np.empty(i["num_tiles"] + 1, np.int32), "denom": np.empty(V, np.float32)}
        pair = np.empty(((V + 127) // 128) * 128 * T, np.int32) if i["streaming"] else None
        if self.lib.ggnn_prepared_graph_arrays(self._h, out["row_ptr"].ctypes.data, out["src"].ctypes.data, out["msg"].ctypes.data,
                                               out["tile_start"].ctypes.data, out["denom"].ctypes.data,
                                               None if pair is None else pair.ctypes.data) != 0:
            raise GgnnError("the prepared graph is empty")
        if pair is not None:
            out["pair_src"] = pair
        return out

    def stream_tables(self) -> dict:
        """A streaming plan's virtual rows: ``vrow_ptr`` [NV+1], ``vsrc``, ``vinfo`` [NV, 8], ``tile_vptr`` [num_tiles+1] and, on a weighted
        batch or with attention, ``vslot`` [NV] (the first target-CSR slot of every virtual row; None on a binary batch)."""
        nv, nvm = C.c_int32(), C.c_int64()
        if self.lib.ggnn_prepared_graph_stream_tables(self._h, C.byref(nv), C.byref(nvm), None, None, None, None, None) != 0:
            raise GgnnError("the prepared graph is empty or does not stream")
        out = {"vrow_ptr": np.empty(nv.value + 1, np.int32), "vsrc": np.empty(nvm.value, np.int32), "vinfo": np.empty((nv.value, 8), np.int32),
               "tile_vptr": np.empty(self.info()["num_tiles"] + 1, np.int32), "vslot": np.empty(nv.value, np.int32)}
        weighted = self.lib.ggnn_prepared_graph_stream_tables(self._h, None, None, None, None, None, out["vslot"].ctypes.data, None) == 0
        if not weighted:
            out["vslot"] = None
        if self.lib.ggnn_prepared_graph_stream_tables(self._h, None, None, out["vrow_ptr"].ctypes.data, out["vsrc"].ctypes.data,
                                                      out["vinfo"].ctypes.data, None, out["tile_vptr"].ctypes.data) != 0:
            raise GgnnError("the prepared graph is empty or does not stream")
        return out

    def tile_stats(self) -> tuple:
        """(largest message count, largest number of edge types) of one tile: what the tile-local wgmma kernel sizes its shared memory by."""
        mm, mt = C.c_int32(), C.c_int32()
        if self.lib.ggnn_prepared_graph_tile_stats(self._h, C.byref(mm), C.byref(mt)) != 0:
            raise GgnnError("the prepared graph is empty")
        return mm.value, mt.value

    def image(self) -> np.ndarray:
        """The packed image, byte for byte what ``set_graph_prepared`` uploads."""
        out = np.empty(self.info()["image_bytes"], np.uint8)
        if self.lib.ggnn_prepared_graph_image(self._h, out.ctypes.data, out.nbytes) != 0:
            raise GgnnError("the prepared graph is empty")
        return out

    def close(self):
        if getattr(self, "_h", None) is not None and self._h.value:
            self.lib.ggnn_free_prepared_graph(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class DeviceDataset:
    """Handle of a ``ggnn_dataset`` (include/ggnn_b200.h): a whole graph set on the GPU, from which every batch of whole graphs is assembled on
    the device.  Built from a ``packing.FlatSparseGraphs`` or ``packing.FlatDenseGraphs`` (GGNN engines) or ``packing.FlatGCNGraphs`` (GCN
    engines), whose arrays it reads as they are.  ``for_engine`` uploads it for an engine; ``host_only`` / ``host_only_dense`` /
    ``host_only_gcn`` build the same host summaries without a GPU, so that batch plans can be checked anywhere.  A dense dataset's batches
    have ``nodes_per_graph`` rows per graph, as the dense model's bucketed batches."""

    def __init__(self, lib=None):
        self.lib = lib or _lib.load()
        self._h = C.c_void_p()
        self.num_tasks = 0

    @staticmethod
    def _common(flat):
        labels = np.ascontiguousarray(flat.labels, np.float32)
        mask = np.ascontiguousarray(flat.mask, np.float32)
        ann = np.ascontiguousarray(flat.feat, np.float32)
        return [np.ascontiguousarray(flat.n_nodes, np.int64), ann, labels, mask]

    @staticmethod
    def _sparse_arrays(flat, T: int):
        if flat.num_edge_types != T:
            raise GgnnError("the graph set has %d edge types, the engine %d" % (flat.num_edge_types, T))
        edges = [np.ascontiguousarray(e, np.int32).reshape(-1, 2) for e in flat.edges]
        offsets = np.ascontiguousarray(np.stack(flat.edge_off), np.int64) if T else np.zeros((0, 1), np.int64)
        indeg = np.ascontiguousarray(flat.indeg, np.float32)
        return edges, offsets, indeg

    def _create(self, fn, flat, head, tail, keep):
        """``fn(*head, N, node_counts, *tail, ann_size, ann, tasks, labels, mask, *stream, &handle)``; raises with the dataset's text."""
        counts, ann, labels, mask = self._common(flat)
        keep += [counts, ann, labels, mask]
        h = C.c_void_p()
        rc = fn(*head[0], int(flat.num_graphs), counts.ctypes.data, *tail, ann.shape[1] if ann.ndim == 2 else 0, ann.ctypes.data,
                labels.shape[1], labels.ctypes.data, mask.ctypes.data, *head[1], C.byref(h))
        self._h = h
        if rc != 0:
            err = GgnnError(self.lib.ggnn_dataset_error(h).decode() if h.value else "invalid argument")
            err.code = rc
            self.close()
            raise err
        self.num_tasks = labels.shape[1]
        self.num_graphs = int(flat.num_graphs)
        self.dense = isinstance(flat, packing.FlatDenseGraphs)
        return self

    @classmethod
    def for_engine(cls, engine: "PropagationEngine", flat, for_training: bool = True, stream: Optional[int] = None) -> "DeviceDataset":
        """Validates, builds and uploads ``flat`` for ``engine`` on ``stream`` (default: torch's current stream) and returns once the upload
        completed.  ``for_training``: also build the source-keyed CSR that batches trained on need."""
        d = cls(engine.lib)
        d.engine_T, d.D = engine.T, engine.D
        keep = []
        head = ((engine._h, int(bool(for_training))), (engine._stream() if stream is None else int(stream),))
        if isinstance(engine, GCNEngine):
            lst, w = _gcn_arrays(flat.lists, flat.weights)
            off = np.ascontiguousarray(flat.entry_off, np.int64)
            keep += [lst, w, off]
            return d._create(d.lib.ggnn_dataset_create_gcn, flat, head, (lst.ctypes.data, off.ctypes.data, w.ctypes.data), keep)
        if isinstance(flat, packing.FlatDenseGraphs):
            tri, off = cls._dense_arrays(flat)
            keep += [tri, off]
            return d._create(d.lib.ggnn_dataset_create_dense, flat, head, (tri.ctypes.data, off.ctypes.data, int(flat.tie_fwd_bkwd)), keep)
        edges, offsets, indeg = cls._sparse_arrays(flat, engine.T)
        keep += [edges, offsets, indeg]
        ptrs = (C.c_void_p * max(engine.T, 1))(*[e.ctypes.data for e in edges])
        return d._create(d.lib.ggnn_dataset_create_sparse, flat, head, (ptrs, offsets.ctypes.data, indeg.ctypes.data), keep)

    @staticmethod
    def _dense_arrays(flat):
        return (np.ascontiguousarray(flat.triples, np.int64).reshape(-1, 3), np.ascontiguousarray(flat.edge_off, np.int64))

    @classmethod
    def host_only_dense(cls, params: dict, num_edge_types: int, flat, precision: str = "fp32", num_sms: int = 132,
                        for_training: bool = True) -> "DeviceDataset":
        """``ggnn_host_dataset_create_dense``: the dense dataset's host summaries (from a ``packing.FlatDenseGraphs``), no engine, no GPU."""
        d = cls()
        cfg, keep = make_config(params, num_edge_types, 0, precision)
        tri, off = cls._dense_arrays(flat)
        head = ((C.byref(cfg), int(num_sms), int(bool(for_training))), ())
        return d._create(d.lib.ggnn_host_dataset_create_dense, flat, head, (tri.ctypes.data, off.ctypes.data, int(flat.tie_fwd_bkwd)),
                         [keep, tri, off])

    @classmethod
    def host_only(cls, params: dict, num_edge_types: int, flat, precision: str = "fp32", num_sms: int = 132,
                  for_training: bool = True, attention_tensor_cores: bool = False, cudnn_gru_tensor_cores: bool = False) -> "DeviceDataset":
        """``ggnn_host_dataset_create_sparse``: the GGNN dataset's host summaries, no engine, no GPU.  ``attention_tensor_cores``,
        ``cudnn_gru_tensor_cores``: as in ``make_config``."""
        d = cls()
        cfg, keep = make_config(params, num_edge_types, 0, precision, attention_tensor_cores, cudnn_gru_tensor_cores)
        edges, offsets, indeg = cls._sparse_arrays(flat, int(num_edge_types))
        keep = [keep, edges, offsets, indeg]
        ptrs = (C.c_void_p * max(int(num_edge_types), 1))(*[e.ctypes.data for e in edges])
        head = ((C.byref(cfg), int(num_sms), int(bool(for_training))), ())
        return d._create(d.lib.ggnn_host_dataset_create_sparse, flat, head, (ptrs, offsets.ctypes.data, indeg.ctypes.data), keep)

    @classmethod
    def host_only_gcn(cls, hidden_size: int, num_layers: int, flat, use_bias: bool = False, precision: str = "fp32", num_sms: int = 132,
                      for_training: bool = True, wide_hidden: bool = False) -> "DeviceDataset":
        """``ggnn_host_dataset_create_gcn``: the GCN dataset's host summaries, no engine, no GPU.  ``wide_hidden``: as for ``GCNEngine``."""
        d = cls()
        cfg = _lib.GcnConfig(int(hidden_size), int(num_layers), int(bool(use_bias)), PRECISIONS[precision], 0, int(bool(wide_hidden)))
        lst, w = _gcn_arrays(flat.lists, flat.weights)
        off = np.ascontiguousarray(flat.entry_off, np.int64)
        head = ((C.byref(cfg), int(num_sms), int(bool(for_training))), ())
        return d._create(d.lib.ggnn_host_dataset_create_gcn, flat, head, (lst.ctypes.data, off.ctypes.data, w.ctypes.data), [lst, w, off])

    def prepare_batch(self, ids, save_for_backward: bool = True, reuse: Optional["DatasetBatch"] = None,
                      nodes_per_graph: Optional[int] = None) -> "DatasetBatch":
        """The HOST half of a batch of the graphs ``ids`` (dataset indices, in batch order): offsets, tile plan, image layout and a pinned
        table of per-graph offsets, from the dataset's summaries alone -- may run in a producer thread.  ``reuse`` rebuilds a batch in place.
        A dense dataset's batch needs ``nodes_per_graph`` (the bucket size v: graph i owns rows i*v .. i*v+v-1); other datasets take none."""
        ids = np.ascontiguousarray(np.asarray(ids, dtype=np.int64).reshape(-1))
        b = reuse if reuse is not None else DatasetBatch(self)
        h = C.c_void_p(b._h.value)
        if nodes_per_graph is not None or self.dense:
            rc = self.lib.ggnn_dataset_prepare_batch_dense(self._h, int(bool(save_for_backward)), ids.ctypes.data, ids.shape[0],
                                                           int(nodes_per_graph or 0), C.byref(h))
        else:
            rc = self.lib.ggnn_dataset_prepare_batch(self._h, int(bool(save_for_backward)), ids.ctypes.data, ids.shape[0], C.byref(h))
        b._h = h
        if rc != 0:
            err = GgnnError(self.lib.ggnn_dataset_batch_error(h).decode() if h.value else "invalid argument")
            err.code = rc
            raise err
        b.dataset, b.G, b.ids = self, ids.shape[0], ids
        b.V = b.info()["num_nodes"]
        b.nodes_per_graph = int(nodes_per_graph) if self.dense else 0
        return b

    def close(self):
        if getattr(self, "_h", None) is not None and self._h.value:
            self.lib.ggnn_free_dataset(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class DatasetBatch:
    """Handle of a ``ggnn_dataset_batch``: the host half of one dataset batch (adopt it with ``set_graph_from_dataset``)."""

    def __init__(self, dataset: DeviceDataset):
        self.lib = dataset.lib
        self.dataset = dataset   # the dataset must outlive its batches
        self._h = C.c_void_p()
        self.V = self.G = self.nodes_per_graph = 0
        self.ids = np.zeros(0, np.int64)   # the batch's graphs' dataset indices, in batch order
        # the same ids as the engine's DEVICE int32 table [G] once the batch is adopted (set_graph_from_dataset): the slot map with which
        # readout_predict writes each graph's predictions at its dataset index; valid until the engine's next graph upload
        self.slot_table = None

    def info(self) -> dict:
        V, M, nt, nb, st = C.c_int32(), C.c_int64(), C.c_int32(), C.c_int64(), C.c_int32()
        buf = C.create_string_buffer(512)
        if self.lib.ggnn_dataset_batch_info(self._h, C.byref(V), C.byref(M), C.byref(nt), C.byref(nb), C.byref(st), buf, 512, None, None, None) != 0:
            raise GgnnError("the dataset batch is empty")
        tiles = np.empty(nt.value + 1, np.int32)
        mm, mt = C.c_int32(), C.c_int32()
        self.lib.ggnn_dataset_batch_info(self._h, None, None, None, None, None, None, 0, tiles.ctypes.data, C.byref(mm), C.byref(mt))
        return {"num_nodes": V.value, "num_messages": M.value, "num_tiles": nt.value, "image_bytes": nb.value, "streaming": bool(st.value),
                "plan": buf.value.decode(), "tile_start": tiles, "max_tile_msgs": mm.value, "max_tile_types": mt.value}

    def close(self):
        if getattr(self, "_h", None) is not None and self._h.value:
            self.lib.ggnn_free_dataset_batch(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class PropagationEngine:
    def __init__(self, params: dict, num_edge_types: int, device: int = 0, precision: str = "fp32", attention_tensor_cores: bool = False,
                 cudnn_gru_tensor_cores: bool = False):
        """``attention_tensor_cores``: propagation attention at ``precision`` instead of on the fp32 kernels; ``cudnn_gru_tensor_cores``:
        CudnnCompatibleGRUCell at ``precision`` likewise (see ``make_config``)."""
        self._h = C.c_void_p()
        self.lib = _lib.load()
        self.params = dict(params)
        self.D = int(params["hidden_size"])
        self.T = int(num_edge_types)
        self.L = len(params["layer_timesteps"])
        cfg, self._cfg_keepalive = make_config(params, num_edge_types, device, precision, attention_tensor_cores, cudnn_gru_tensor_cores)
        rc = self.lib.ggnn_create(C.byref(cfg), C.byref(self._h))
        if rc != 0:
            self._h = C.c_void_p()
            raise GgnnError(self.lib.ggnn_last_error(None).decode())
        self.device = int(device)
        self.V = 0
        self.serial = 0   # bumped by every forward, graph upload and weight binding: see require_serial
        self._weights_keepalive = None
        self._graph_keepalive = None

    # ------------------------------------------------------------------ plumbing
    def _check(self, rc: int):
        if rc != 0:
            err = GgnnError(self.lib.ggnn_last_error(self._h).decode())
            err.code = rc   # the GGNN_E* code of the call
            raise err

    def close(self):
        if getattr(self, "_h", None) and self._h.value:
            self.lib.ggnn_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    @staticmethod
    def _stream() -> int:
        import torch
        return int(torch.cuda.current_stream().cuda_stream)

    # ------------------------------------------------------------------ model
    def set_weights(self, layers: Sequence[dict]):
        """``layers[l]``: dict of contiguous fp32 CUDA tensors keyed like ``ggnn_layer_weights``."""
        arr = (_lib.GgnnLayerWeights * len(layers))()
        keep = []
        for l, w in enumerate(layers):
            shapes = weight_shapes(self.params, self.T, l)
            for f in WEIGHT_FIELDS:
                t = w.get(f)
                if t is None or f not in shapes:
                    setattr(arr[l], f, None)
                    continue
                if not (t.is_cuda and t.is_contiguous() and t.dtype.is_floating_point and t.element_size() == 4):
                    raise GgnnError("layer %d %s must be a contiguous fp32 CUDA tensor" % (l, f))
                if tuple(t.reshape(shapes[f]).shape) != shapes[f]:
                    raise GgnnError("layer %d %s has shape %s, expected %s" % (l, f, tuple(t.shape), shapes[f]))
                setattr(arr[l], f, t.data_ptr())
                keep.append(t)
        self.serial += 1
        self._check(self.lib.ggnn_set_weights(self._h, arr, len(layers)))
        self._weights_keepalive = keep

    # ------------------------------------------------------------------ batch
    def _sparse_args(self, adjacency_lists, num_incoming_edges_per_type):
        if len(adjacency_lists) != self.T:
            raise GgnnError("expected %d adjacency lists, got %d" % (self.T, len(adjacency_lists)))
        adjs = [np.ascontiguousarray(np.asarray(a, dtype=np.int32).reshape(-1, 2)) for a in adjacency_lists]
        indeg = np.ascontiguousarray(np.asarray(num_incoming_edges_per_type, dtype=np.float32))
        if indeg.ndim != 2 or indeg.shape[1] != self.T:
            raise GgnnError("num_incoming_edges_per_type must be [V, %d]" % self.T)
        ptrs = (C.c_void_p * self.T)(*[a.ctypes.data for a in adjs])
        counts = (C.c_int32 * self.T)(*[a.shape[0] for a in adjs])
        return adjs, indeg, ptrs, counts

    def set_graph_sparse(self, adjacency_lists: Sequence[np.ndarray], num_incoming_edges_per_type: np.ndarray):
        """Reference wire format (sparse:331-348): per type an ``[E_t, 2]`` int32 (source, target) list and the
        ``[V, T]`` in-degree table.  HOST arrays; index validation, CSR build and upload happen in the library."""
        adjs, indeg, ptrs, counts = self._sparse_args(adjacency_lists, num_incoming_edges_per_type)
        V = indeg.shape[0]
        self.serial += 1
        self._check(self.lib.ggnn_set_graph_sparse(self._h, V, ptrs, counts, indeg.ctypes.data, self._stream()))
        self.V = V
        self._graph_keepalive = (adjs, indeg)

    def _sparse_device_args(self, num_nodes, adjacency_lists, num_incoming_edges_per_type):
        """Checks and marshals the feeds of ``set_graph_sparse_device``; raises ``GgnnError`` before any call into the library."""
        import torch
        V = int(num_nodes)
        if V < 0:
            raise GgnnError("num_nodes must be >= 0, got %d" % V)
        if len(adjacency_lists) != self.T:
            raise GgnnError("expected %d adjacency lists, got %d" % (self.T, len(adjacency_lists)))
        dev = torch.device("cuda", self.device)
        for t, a in enumerate(adjacency_lists):
            if not isinstance(a, torch.Tensor) or a.device != dev:
                raise GgnnError("adjacency list %d must be a torch tensor on cuda:%d" % (t, self.device))
            if a.dtype != torch.int32 or a.dim() != 2 or a.shape[1] != 2 or not a.is_contiguous():
                raise GgnnError("adjacency list %d must be a contiguous int32 [E, 2] tensor, got %s %s" % (t, a.dtype, tuple(a.shape)))
        indeg = num_incoming_edges_per_type
        if indeg is not None:
            if not isinstance(indeg, torch.Tensor) or indeg.device != dev:
                raise GgnnError("num_incoming_edges_per_type must be a torch tensor on cuda:%d or None" % self.device)
            if indeg.dtype != torch.float32 or tuple(indeg.shape) != (V, self.T) or not indeg.is_contiguous():
                raise GgnnError("num_incoming_edges_per_type must be a contiguous float32 [%d, %d] tensor, got %s %s"
                                % (V, self.T, indeg.dtype, tuple(indeg.shape)))
        ptrs = (C.c_void_p * self.T)(*[a.data_ptr() if a.shape[0] else None for a in adjacency_lists])
        counts = (C.c_int32 * self.T)(*[a.shape[0] for a in adjacency_lists])
        return V, ptrs, counts, indeg

    def set_graph_sparse_device(self, num_nodes: int, adjacency_lists, num_incoming_edges_per_type=None, message_weighted: bool = False):
        """``set_graph_sparse`` with the graph already on the GPU (``ggnn_set_graph_sparse_device``): per type a contiguous int32 CUDA tensor
        ``[E_t, 2]`` of (source, target) pairs on the engine's device, and optionally the fp32 CUDA ``[V, T]`` in-degree table (None: the
        per-(target, type) message counts, which is what the reference's packer feeds).  The batch is built on the device, with the host's
        plan, into the image ``prepare_graph_sparse`` (``message_weighted``: ``prepare_graph_sparse_weighted``, then ``set_message_weights``)
        would upload, byte for byte.  The call waits for the current stream for three small reads at most; the tensors are kept alive until
        the next graph upload."""
        V, ptrs, counts, indeg = self._sparse_device_args(num_nodes, adjacency_lists, num_incoming_edges_per_type)
        self.serial += 1
        self._check(self.lib.ggnn_set_graph_sparse_device(self._h, V, ptrs, counts, indeg.data_ptr() if indeg is not None and V else None,
                                                          int(bool(message_weighted)), self._stream()))
        self.V = V
        self._graph_keepalive = (list(adjacency_lists), indeg)

    def marshal_sparse(self, adjacency_lists, num_incoming_edges_per_type):
        """The ctypes view of one batch's graph feeds (contiguous int32 / float32 arrays, pointer and count tables), reusable across calls:
        pass it as ``marshalled=`` to keep a producer thread's time under the GIL to a few microseconds per batch."""
        return self._sparse_args(adjacency_lists, num_incoming_edges_per_type)

    def prepare_graph_sparse(self, adjacency_lists=None, num_incoming_edges_per_type=None, save_for_backward: Optional[bool] = None,
                             reuse: Optional["PreparedGraph"] = None, marshalled=None) -> "PreparedGraph":
        """The HOST half of ``set_graph_sparse`` (validation, CSR, tile plan, one pinned image) -- may run in a producer thread while the
        engine's stream works on the previous batch (ThreadedIterator, chem_tensorflow.py:225).  ``save_for_backward``: whether the batch
        will be trained on (None = the engine's current flag).  ``reuse``: rebuild a prepared graph in place (its pinned image is kept; the
        call waits for its previous upload first)."""
        adjs, indeg, ptrs, counts = marshalled if marshalled is not None else self._sparse_args(adjacency_lists, num_incoming_edges_per_type)
        g = reuse if reuse is not None else PreparedGraph(self.lib)
        return g._fill(self.lib.ggnn_prepare_graph_sparse, indeg.shape[0], self.T, self._h,
                       -1 if save_for_backward is None else int(bool(save_for_backward)), indeg.shape[0], ptrs, counts, indeg.ctypes.data)

    def prepare_graph_sparse_weighted(self, adjacency_lists=None, num_incoming_edges_per_type=None, save_for_backward: Optional[bool] = None,
                                      reuse: Optional["PreparedGraph"] = None, marshalled=None) -> "PreparedGraph":
        """``prepare_graph_sparse`` for a MESSAGE-WEIGHTED batch (``ggnn_prepare_graph_sparse_weighted``): after ``set_graph_prepared``,
        ``set_message_weights`` puts one weight per message on the device, and every forward scales message m's state term by w_m:
        incoming[v] = (sum_t (sum_m w_m h[s_m]) W_t + sum_t indeg[v,t] b_t) / denom[v].  The in-degree table is used as fed, for the edge bias
        and the mean, and gets no gradient: to weight the bias too (A.(hW + b)), feed the weighted row sums as the table -- the weights'
        gradient then lacks the bias path.  Refused with propagation attention."""
        adjs, indeg, ptrs, counts = marshalled if marshalled is not None else self._sparse_args(adjacency_lists, num_incoming_edges_per_type)
        g = reuse if reuse is not None else PreparedGraph(self.lib)
        return g._fill(self.lib.ggnn_prepare_graph_sparse_weighted, indeg.shape[0], self.T, self._h,
                       -1 if save_for_backward is None else int(bool(save_for_backward)), indeg.shape[0], ptrs, counts, indeg.ctypes.data)

    def prepare_graph_dense_device(self, num_graphs: int, num_vertices: int, save_for_backward: Optional[bool] = None,
                                   reuse: Optional["PreparedGraph"] = None) -> "PreparedGraph":
        """The batch of ``num_graphs`` dense graphs of ``num_vertices`` rows whose ``[b, T, v, v]`` adjacency lives on the device
        (``ggnn_prepare_graph_dense_device``): after ``set_graph_prepared``, ``set_message_weights(A)`` sets the matrix (any finite values)
        and ``backward(..., d_message_weights=dA)`` returns its gradient at every entry.  The plan depends on (b, v) only, so a new matrix on
        the same batch needs no new prepare.  Refused with propagation attention, mean aggregation and ``cudnn_gru_tensor_cores``."""
        g = reuse if reuse is not None else PreparedGraph(self.lib)
        return g._fill(self.lib.ggnn_prepare_graph_dense_device, int(num_graphs) * int(num_vertices), self.T, self._h,
                       -1 if save_for_backward is None else int(bool(save_for_backward)), int(num_graphs), int(num_vertices))

    def set_message_weights(self, w):
        """``ggnn_set_message_weights``: ``w`` a contiguous fp32 CUDA tensor of ``num_messages()`` entries, message m of type t at position
        ``sum_{t' < t} E_t' + i`` (the reference's type-major order, ``oracle.ggnn_oracle.message_arrays``), for the current
        message-weighted batch (``prepare_graph_sparse_weighted`` + ``set_graph_prepared``, or
        ``set_graph_sparse_device(..., message_weighted=True)``); on a batch of ``prepare_graph_dense_device``, the ``[b, T, v, v]`` adjacency itself.  The engine copies
        them on its stream; ``w`` may be reused once the stream passed the call."""
        import torch
        if not (isinstance(w, torch.Tensor) and w.is_cuda and w.dtype == torch.float32 and w.is_contiguous()):
            raise GgnnError("message weights must be a contiguous fp32 CUDA tensor")
        M = self.num_messages()
        if w.numel() != M:
            raise GgnnError("message weights have %d entries, the batch has %d messages" % (w.numel(), M))
        self.serial += 1
        self._check(self.lib.ggnn_set_message_weights(self._h, w.data_ptr() if M else None, self._stream()))

    def prepare_graph_dense(self, adjacency_matrix, save_for_backward: Optional[bool] = None,
                            reuse: Optional["PreparedGraph"] = None) -> "PreparedGraph":
        """The HOST half of ``set_graph_dense`` for a 0/1 adjacency ``[b, T, v, v]`` (scan to edge lists + the CSR builder); raises
        ``GgnnError`` for a weighted matrix, which ``set_graph_dense`` and ``prepare_graph_dense_weighted`` take."""
        return self._prepare_dense(self.lib.ggnn_prepare_graph_dense, adjacency_matrix, save_for_backward, reuse)

    def prepare_graph_dense_weighted(self, adjacency_matrix, save_for_backward: Optional[bool] = None,
                                     reuse: Optional["PreparedGraph"] = None) -> "PreparedGraph":
        """The HOST half of ``set_graph_dense_weighted``: any ``[b, T, v, v]`` adjacency, a weighted one with its entries as slot weights
        and, above hidden 128 on bf16x3 / bf16, on the streaming wgmma kernels."""
        return self._prepare_dense(self.lib.ggnn_prepare_graph_dense_weighted, adjacency_matrix, save_for_backward, reuse)

    def _prepare_dense(self, fn, adjacency_matrix, save_for_backward, reuse):
        a = self._dense_matrix(adjacency_matrix)
        g = reuse if reuse is not None else PreparedGraph(self.lib)
        return g._fill(fn, a.shape[0] * a.shape[2], self.T, self._h, -1 if save_for_backward is None else int(bool(save_for_backward)),
                       a.shape[0], a.shape[2], a.ctypes.data)

    def _dense_matrix(self, adjacency_matrix) -> np.ndarray:
        a = np.ascontiguousarray(np.asarray(adjacency_matrix, dtype=np.float32))
        if a.ndim != 4 or a.shape[1] != self.T or a.shape[2] != a.shape[3]:
            raise GgnnError("adjacency_matrix must be [b, %d, v, v]" % self.T)
        return a

    def set_graph_prepared(self, g: "PreparedGraph"):
        """The DEVICE half: adopt the plan, enqueue the one H2D copy of the image.  Keep ``g`` alive until the stream has passed it."""
        self.serial += 1
        self._check(self.lib.ggnn_set_graph_prepared(self._h, g._h, self._stream()))
        self.V = g.V
        self._graph_keepalive = (g,)

    def set_graph_from_dataset(self, batch: "DatasetBatch"):
        """The DEVICE half of a dataset batch: adopts its plan and assembles its graph image, h0, targets and readout map on the engine's
        stream.  Returns ``(h0 [V, D], target_values [tasks, G], target_mask [tasks, G])`` as CUDA tensors, and for a dense batch also its
        ``node_mask [G, nodes_per_graph]``; the readout map (with a dense batch's mask) is set (no ``readout_set_graphs`` needed).  Keep
        ``batch`` alive until the stream has passed it."""
        import torch
        dev = "cuda:%d" % self.device
        h0 = torch.empty(batch.V, self.D, dtype=torch.float32, device=dev)
        tv = torch.empty(batch.dataset.num_tasks, batch.G, dtype=torch.float32, device=dev)
        tm = torch.empty_like(tv)
        ptr = lambda t: t.data_ptr() if t.numel() else None
        self.serial += 1
        if batch.dataset.dense:
            mask = torch.empty(batch.G, batch.nodes_per_graph, dtype=torch.float32, device=dev)
            self._check(self.lib.ggnn_set_graph_dataset_dense(self._h, batch._h, ptr(h0), ptr(tv), ptr(tm), ptr(mask), self._stream()))
        else:
            self._check(self.lib.ggnn_set_graph_dataset(self._h, batch._h, ptr(h0), ptr(tv), ptr(tm), self._stream()))
        self.V = batch.V
        self._graph_keepalive = (batch,)
        self._readout_keepalive = None
        self._readout_shape = (batch.V, batch.G)
        slots = C.c_void_p()
        self._check(self.lib.ggnn_dataset_batch_slots(self._h, C.byref(slots)))
        batch.slot_table = slots.value
        return (h0, tv, tm, mask) if batch.dataset.dense else (h0, tv, tm)

    def graph_image(self) -> np.ndarray:
        """The engine's current graph image copied back (``ggnn_graph_image``): the bytes ``PreparedGraph.image`` holds for the same batch."""
        n = C.c_int64()
        self._check(self.lib.ggnn_graph_image(self._h, None, 0, C.byref(n), self._stream()))
        out = np.empty(n.value, np.uint8)
        self._check(self.lib.ggnn_graph_image(self._h, out.ctypes.data, out.nbytes, C.byref(n), self._stream()))
        return out

    def run_sparse_host(self, adjacency_lists, num_incoming_edges_per_type, h0: np.ndarray, out: Optional[np.ndarray] = None) -> np.ndarray:
        """One call per batch (the shape of ``sess.run(fetch, feed_dict)``, chem_tensorflow.py:235): graph + initial
        states in, final node states out, HOST arrays, synchronous; the h0 upload overlaps the host-side CSR build."""
        adjs, indeg, ptrs, counts = self._sparse_args(adjacency_lists, num_incoming_edges_per_type)
        V = indeg.shape[0]
        h0 = np.ascontiguousarray(h0, dtype=np.float32)
        if h0.size != V * self.D:
            raise GgnnError("h0 has %d elements, the graph has %d nodes x %d" % (h0.size, V, self.D))
        if out is None:
            out = np.empty_like(h0)
        self.serial += 1
        self._check(self.lib.ggnn_run_sparse_host(self._h, V, ptrs, counts, indeg.ctypes.data, h0.ctypes.data, out.ctypes.data, self._stream()))
        self.V = V
        self._graph_keepalive = (adjs, indeg)
        return out

    def run_sparse_host_readout(self, adjacency_lists, num_incoming_edges_per_type, h0, graph_nodes_list, num_graphs, readout_tasks,
                                target_values, target_mask):
        """The fetches of the reference's ``sess.run([loss, accuracy_task*], feed_dict)`` (chem_tensorflow.py:231-235) in one call: the
        batch in HOST arrays (reference wire format), per task the readout trainables as CUDA tensors ``(w_gate [2D], b_gate [1],
        w_trans [D], b_trans [1])``; returns ``(loss [tasks], accuracy [tasks])`` -- 2*tasks floats are all that cross PCIe on the way back."""
        adjs, indeg, ptrs, counts = self._sparse_args(adjacency_lists, num_incoming_edges_per_type)
        V, nt, G = indeg.shape[0], len(readout_tasks), int(num_graphs)
        h0 = np.ascontiguousarray(h0, dtype=np.float32)
        gnl = np.ascontiguousarray(np.asarray(graph_nodes_list, dtype=np.int32).reshape(-1))
        tv = np.ascontiguousarray(np.asarray(target_values, dtype=np.float32).reshape(nt, G))
        tm = np.ascontiguousarray(np.asarray(target_mask, dtype=np.float32).reshape(nt, G))
        if h0.size != V * self.D or gnl.shape[0] != V:
            raise GgnnError("h0 / graph_nodes_list do not match the %d nodes of the graph" % V)
        arr = self._readout_tasks(readout_tasks)
        loss, acc = np.empty(nt, np.float32), np.empty(nt, np.float32)
        self.serial += 1
        self._check(self.lib.ggnn_run_sparse_host_readout(self._h, V, ptrs, counts, indeg.ctypes.data, h0.ctypes.data, gnl.ctypes.data, G, nt, arr,
                                                          tv.ctypes.data, tm.ctypes.data, loss.ctypes.data, acc.ctypes.data, self._stream()))
        self.V = V
        self._graph_keepalive = (adjs, indeg)
        return loss, acc

    def _readout_tasks(self, readout_tasks):
        """``ggnn_readout_task[]`` of ``(w_gate [2D], b_gate [1], w_trans [D], b_trans [1])`` CUDA tensors, one tuple per task."""
        arr = (_lib.GgnnReadoutTask * len(readout_tasks))()
        for i, (wg, bg, wt, bt) in enumerate(readout_tasks):
            arr[i].w_gate, arr[i].b_gate = self._f32(wg, 2 * self.D, "w_gate"), self._f32(bg, 1, "b_gate")
            arr[i].w_trans, arr[i].b_trans = self._f32(wt, self.D, "w_trans"), self._f32(bt, 1, "b_trans")
        return arr

    def run_sparse_host_predict(self, adjacency_lists, num_incoming_edges_per_type, h0, graph_nodes_list, num_graphs, readout_tasks) -> np.ndarray:
        """``sess.run(self.output, feed)`` of the reference's evaluate_one_batch (sparse:352-362) for every task in one call: the batch in
        HOST arrays without targets, the readout trainables as for ``run_sparse_host_readout``; returns ``[tasks, num_graphs]`` (HOST)."""
        adjs, indeg, ptrs, counts = self._sparse_args(adjacency_lists, num_incoming_edges_per_type)
        V, G = indeg.shape[0], int(num_graphs)
        h0 = np.ascontiguousarray(h0, dtype=np.float32)
        gnl = np.ascontiguousarray(np.asarray(graph_nodes_list, dtype=np.int32).reshape(-1))
        if h0.size != V * self.D or gnl.shape[0] != V:
            raise GgnnError("h0 / graph_nodes_list do not match the %d nodes of the graph" % V)
        arr = self._readout_tasks(readout_tasks)
        out = np.empty((len(readout_tasks), G), np.float32)
        self.serial += 1
        self._check(self.lib.ggnn_run_sparse_host_predict(self._h, V, ptrs, counts, indeg.ctypes.data, h0.ctypes.data, gnl.ctypes.data, G,
                                                          len(readout_tasks), arr, out.ctypes.data, self._stream()))
        self.V = V
        self._graph_keepalive = (adjs, indeg)
        self._readout_shape = (V, G)
        return out

    def run_dense_host_predict(self, adjacency_matrix, h0, node_mask, readout_tasks) -> np.ndarray:
        """The dense evaluate_one_batch (dense:230-249) in one call: ``[b, T, v, v]`` adjacency, ``h0 [b*v, D]`` and ``node_mask [b, v]``
        HOST arrays; returns ``[tasks, b]`` (HOST)."""
        a = np.ascontiguousarray(np.asarray(adjacency_matrix, dtype=np.float32))
        if a.ndim != 4 or a.shape[1] != self.T or a.shape[2] != a.shape[3]:
            raise GgnnError("adjacency_matrix must be [b, %d, v, v]" % self.T)
        b, v = a.shape[0], a.shape[2]
        h0 = np.ascontiguousarray(h0, dtype=np.float32)
        mask = np.ascontiguousarray(np.asarray(node_mask, dtype=np.float32).reshape(-1))
        if h0.size != b * v * self.D or mask.shape[0] != b * v:
            raise GgnnError("h0 / node_mask do not match the %d x %d nodes of the batch" % (b, v))
        arr = self._readout_tasks(readout_tasks)
        out = np.empty((len(readout_tasks), b), np.float32)
        self.serial += 1
        self._check(self.lib.ggnn_run_dense_host_predict(self._h, b, v, a.ctypes.data, h0.ctypes.data, mask.ctypes.data, len(readout_tasks), arr,
                                                         out.ctypes.data, self._stream()))
        self.V = b * v
        self._graph_keepalive = (a,)
        self._readout_shape = (b * v, b)
        return out

    def run_dense_host(self, adjacency_matrix: np.ndarray, h0: np.ndarray, out: Optional[np.ndarray] = None) -> np.ndarray:
        a = np.ascontiguousarray(np.asarray(adjacency_matrix, dtype=np.float32))
        if a.ndim != 4 or a.shape[1] != self.T or a.shape[2] != a.shape[3]:
            raise GgnnError("adjacency_matrix must be [b, %d, v, v]" % self.T)
        h0 = np.ascontiguousarray(h0, dtype=np.float32)
        V = a.shape[0] * a.shape[2]
        if h0.size != V * self.D:
            raise GgnnError("h0 has %d elements, the graph has %d nodes x %d" % (h0.size, V, self.D))
        if out is None:
            out = np.empty_like(h0)
        self.serial += 1
        self._check(self.lib.ggnn_run_dense_host(self._h, a.shape[0], a.shape[2], a.ctypes.data, h0.ctypes.data, out.ctypes.data, self._stream()))
        self.V = V
        self._graph_keepalive = (a,)
        return out

    def set_graph_dense(self, adjacency_matrix: np.ndarray):
        """Dense wire format (dense:214-224): ``[b, T, v, v]`` float32 with ``A[g, t, dest, src]``."""
        self._set_dense(self.lib.ggnn_set_graph_dense, adjacency_matrix)

    def set_graph_dense_weighted(self, adjacency_matrix: np.ndarray):
        """``set_graph_dense`` that also runs a weighted matrix above hidden 128 on bf16x3 / bf16, on the streaming wgmma kernels (where
        ``set_graph_dense`` refuses it)."""
        self._set_dense(self.lib.ggnn_set_graph_dense_weighted, adjacency_matrix)

    def _set_dense(self, fn, adjacency_matrix):
        a = self._dense_matrix(adjacency_matrix)
        self.serial += 1
        self._check(fn(self._h, a.shape[0], a.shape[2], a.ctypes.data, self._stream()))
        self.V = a.shape[0] * a.shape[2]
        self._graph_keepalive = (a,)

    # ------------------------------------------------------------------ the hot path
    def forward(self, h0, out=None):
        """compute_final_node_representations on device tensors: ``h0`` [V, D] fp32 CUDA -> [V, D]."""
        import torch
        if not (h0.is_cuda and h0.dtype == torch.float32 and h0.is_contiguous()):
            raise GgnnError("h0 must be a contiguous fp32 CUDA tensor")
        if h0.numel() != self.V * self.D:
            raise GgnnError("h0 has %d elements, the graph has %d nodes x %d" % (h0.numel(), self.V, self.D))
        if out is None:
            out = torch.empty_like(h0)
        self.serial += 1
        self._check(self.lib.ggnn_forward(self._h, h0.data_ptr(), out.data_ptr(), self._stream()))
        return out

    def forward_host(self, h0: np.ndarray, out: Optional[np.ndarray] = None, sync: bool = True) -> np.ndarray:
        """Same through HOST buffers (H2D + propagation + D2H inside the call).  ``sync=False`` returns right after
        enqueueing (pinned buffers required); the result is valid after ``sync_check()``."""
        h0 = np.ascontiguousarray(h0, dtype=np.float32)
        if h0.size != self.V * self.D:
            raise GgnnError("h0 has %d elements, the graph has %d nodes x %d" % (h0.size, self.V, self.D))
        if out is None:
            out = np.empty_like(h0)
        fn = self.lib.ggnn_forward_host if sync else self.lib.ggnn_forward_host_async
        self.serial += 1
        self._check(fn(self._h, h0.ctypes.data, out.ctypes.data, self._stream()))
        return out

    def require_serial(self, serial: int, what: str = "this backward"):
        """Raises ``GgnnError`` unless the engine's serial is still ``serial``.  An autograd node records the serial after its forward:
        ``backward`` reads the engine's saved activations, states and weights, which any later forward, graph upload or weight binding
        replaces.  Repeated backward calls of one forward keep the serial."""
        if self.serial != serial:
            raise GgnnError("%s belongs to an earlier forward: the engine has run %d forward / graph / weight call(s) since, so its saved "
                            "activations are not this forward's" % (what, self.serial - serial))

    def sync_check(self):
        """Synchronise the stream and raise if a kernel reported an (always bounded) barrier timeout."""
        self._check(self.lib.ggnn_sync_check(self._h, self._stream()))

    def set_state_dropout(self, keep_prob: float, seed: int = 0):
        """DropoutWrapper(state_keep_prob) (sparse:113-114): applies to the following forwards; 1.0 = off."""
        self._check(self.lib.ggnn_set_state_dropout(self._h, float(keep_prob), int(seed) & 0xFFFFFFFFFFFFFFFF))

    def state_dropout_mask(self, global_step: int, keep_prob: float, seed: int, V: Optional[int] = None) -> np.ndarray:
        V = self.V if V is None else V
        m = np.empty((V, self.D), np.uint8)
        self._check(self.lib.ggnn_state_dropout_mask(V, self.D, int(global_step), float(keep_prob), int(seed) & 0xFFFFFFFFFFFFFFFF, m.ctypes.data))
        return m

    def set_save_for_backward(self, enable: bool):
        self._check(self.lib.ggnn_set_save_for_backward(self._h, int(bool(enable))))

    def set_deterministic(self, enable: bool):
        """``ggnn_set_deterministic``: fixed-order weight-gradient and readout sums from the next call on, so that the same inputs give
        the same bits in every output and gradient (the autograd nodes set it from ``torch.are_deterministic_algorithms_enabled()``)."""
        self._check(self.lib.ggnn_set_deterministic(self._h, int(bool(enable))))

    def set_backward_precision(self, precision: str):
        """``ggnn_set_backward_precision``: "fp32" (the default, FFMA) or "bf16x3" (the backward's GEMMs on tensor cores, each gradient
        within 2e-4 of float64 relative to its largest entry).  Takes effect at the next backward; the forward is not touched."""
        if precision not in BACKWARD_PRECISIONS:
            raise ValueError("unknown backward precision %r (expected one of %s)" % (precision, ", ".join(BACKWARD_PRECISIONS)))
        self._check(self.lib.ggnn_set_backward_precision(self._h, PRECISIONS[precision]))

    def backward(self, d_out, grads: Sequence[dict], d_h0=None, d_message_weights=None):
        """``ggnn_backward``; with ``d_message_weights`` (fp32 CUDA [num_messages()], accumulated into; message-weighted batches only)
        ``ggnn_backward_weighted``, which also forms the message weights' gradient (on a dense-device batch: dA, ``[b, T, v, v]``)."""
        arr = (_lib.GgnnLayerGrads * len(grads))()
        for l, g in enumerate(grads):
            for f in WEIGHT_FIELDS:
                t = g.get(f)
                setattr(arr[l], f, None if t is None else t.data_ptr())
        if d_message_weights is None:
            self._check(self.lib.ggnn_backward(self._h, d_out.data_ptr(), arr, len(grads),
                                               None if d_h0 is None else d_h0.data_ptr(), self._stream()))
            return
        import torch
        if not (d_message_weights.is_cuda and d_message_weights.dtype == torch.float32 and d_message_weights.is_contiguous()
                and d_message_weights.numel() == self.num_messages()):
            raise GgnnError("d_message_weights must be a contiguous fp32 CUDA tensor of num_messages() entries")
        self._check(self.lib.ggnn_backward_weighted(self._h, d_out.data_ptr(), arr, len(grads), None if d_h0 is None else d_h0.data_ptr(),
                                                    d_message_weights.data_ptr() if d_message_weights.numel() else None, self._stream()))

    # ------------------------------------------------------------------ readout (gated_regression, sparse:220-231 / dense:119-129)
    def readout_set_graphs(self, num_graphs: int, graph_nodes_list=None, nodes_per_graph: int = 0, node_mask=None):
        """The batch's node -> graph map in the reference wire format: sparse ``graph_nodes_list`` [V] int32 (sparse:337), or
        dense ``nodes_per_graph`` = num_vertices with ``node_mask`` [b, v] (dense:126).  HOST arrays, or CUDA tensors on the engine's device
        (``ggnn_readout_set_graphs_device``: a contiguous int32 ``[V]`` list, a contiguous fp32 mask of V entries): the map is then built on
        the GPU, the same map the host arrays give, and a list costs one wait for the current stream.  Host and CUDA arguments do not mix;
        ``num_graphs`` is a host int either way."""
        import torch
        cuda = [torch.is_tensor(a) and a.is_cuda for a in (graph_nodes_list, node_mask) if a is not None]
        if any(cuda):
            if not all(cuda):
                raise GgnnError("graph_nodes_list and node_mask must both be CUDA tensors or both host arrays")
            return self._readout_set_graphs_device(int(num_graphs), graph_nodes_list, int(nodes_per_graph), node_mask)
        gnl = mask = None
        if graph_nodes_list is not None:
            gnl = np.ascontiguousarray(np.asarray(graph_nodes_list, dtype=np.int32).reshape(-1))
            V = gnl.shape[0]
        else:
            V = int(num_graphs) * int(nodes_per_graph)
        if node_mask is not None:
            mask = np.ascontiguousarray(np.asarray(node_mask, dtype=np.float32).reshape(-1))
            if mask.shape[0] != V:
                raise GgnnError("node_mask has %d entries for %d nodes" % (mask.shape[0], V))
        self._check(self.lib.ggnn_readout_set_graphs(self._h, V, None if gnl is None else gnl.ctypes.data, int(num_graphs), int(nodes_per_graph),
                                                     None if mask is None else mask.ctypes.data, self._stream()))
        self._readout_keepalive = (gnl, mask)
        self._readout_shape = (V, int(num_graphs))

    def _readout_set_graphs_device(self, G: int, gnl, npg: int, mask):
        """``readout_set_graphs`` with CUDA tensors: checks them, then ``ggnn_readout_set_graphs_device``; raises ``GgnnError`` before the
        call for a bad feed.  The tensors are kept alive until the next map."""
        import torch
        dev = torch.device("cuda", self.device)
        if gnl is not None:
            if gnl.dtype != torch.int32:
                raise GgnnError("graph_nodes_list must be int32, got %s" % gnl.dtype)
            if gnl.dim() != 1:
                raise GgnnError("graph_nodes_list must be [V], got %s" % (tuple(gnl.shape),))
            if not gnl.is_contiguous():
                raise GgnnError("graph_nodes_list must be contiguous")
            if gnl.device != dev:
                raise GgnnError("graph_nodes_list must be on cuda:%d, got %s" % (self.device, gnl.device))
            V = gnl.shape[0]
        else:
            V = G * npg
        if mask is not None:
            if mask.dtype != torch.float32:
                raise GgnnError("node_mask must be float32, got %s" % mask.dtype)
            if not mask.is_contiguous():
                raise GgnnError("node_mask must be contiguous")
            if mask.device != dev:
                raise GgnnError("node_mask must be on cuda:%d, got %s" % (self.device, mask.device))
            if mask.numel() != V:
                raise GgnnError("node_mask has %d entries for %d nodes" % (mask.numel(), V))
        # an empty tensor has no storage, and NULL means "no list" / "no mask" to the entry: one element stands in (none of it is read)
        ptr = lambda t: None if t is None else (t if V else torch.empty(1, dtype=t.dtype, device=dev)).data_ptr()
        lp, mp = ptr(gnl), ptr(mask)
        self._check(self.lib.ggnn_readout_set_graphs_device(self._h, V, lp, G, npg, mp, self._stream()))
        self._readout_keepalive = (gnl, mask)
        self._readout_shape = (V, G)

    def readout_map(self) -> dict:
        """The current readout map copied back (``ggnn_readout_map``): ``graph_of`` [V], ``start`` [G+1], ``grouped``, ``perm`` [V] (an
        ungrouped list's stable by-graph order, else None) and ``node_mask`` [V] (None without one), as NumPy arrays."""
        V, G, flags = C.c_int32(), C.c_int32(), C.c_int32()
        self._check(self.lib.ggnn_readout_map(self._h, C.byref(V), C.byref(G), C.byref(flags), None, None, None, None, self._stream()))
        V, G, flags = V.value, G.value, flags.value
        graph_of, start, perm, mask = np.empty(V, np.int32), np.empty(G + 1, np.int32), np.empty(V, np.int32), np.empty(V, np.float32)
        self._check(self.lib.ggnn_readout_map(self._h, None, None, None, graph_of.ctypes.data, start.ctypes.data, perm.ctypes.data,
                                              mask.ctypes.data, self._stream()))
        grouped, has_mask = bool(flags & 1), bool(flags & 2)
        return {"graph_of": graph_of, "start": start, "grouped": grouped, "perm": None if grouped else perm,
                "node_mask": mask if has_mask else None}

    @staticmethod
    def _f32(t, n, what):
        if not (t.is_cuda and t.is_contiguous() and t.element_size() == 4 and t.dtype.is_floating_point and t.numel() == n):
            raise GgnnError("%s must be a contiguous fp32 CUDA tensor with %d elements" % (what, n))
        return t.data_ptr()

    def readout_forward(self, h_last, h0, w_gate, b_gate, w_trans, b_trans):
        import torch
        V, G = self._readout_shape
        D = self.D
        out = torch.empty(G, dtype=torch.float32, device=h_last.device)
        self._check(self.lib.ggnn_readout_forward(
            self._h, self._f32(h_last, V * D, "h_last"), self._f32(h0, V * D, "h0"), self._f32(w_gate, 2 * D, "w_gate"), self._f32(b_gate, 1, "b_gate"),
            self._f32(w_trans, D, "w_trans"), self._f32(b_trans, 1, "b_trans"), out.data_ptr(), self._stream()))
        return out

    def readout_predict(self, h_last, h0, readout_tasks, slot=None, out=None, out_stride: Optional[int] = None):
        """``ggnn_readout_predict``: every task's readout over the current map in one pass over the node rows.  ``readout_tasks``: one
        ``(w_gate, b_gate, w_trans, b_trans)`` tuple of CUDA tensors per task (at most 16).  Task k of batch graph g goes to
        ``out.view(-1)[k * out_stride + slot[g]]``: ``slot`` None (slot[g] = g), an int32 CUDA tensor [G], or a device address such as
        ``DatasetBatch.slot_table``.  ``out`` defaults to a new ``[tasks, G]`` tensor; returns it."""
        import torch
        V, G = self._readout_shape
        D, K = self.D, len(readout_tasks)
        if out is None:
            out = torch.empty(K, G, dtype=torch.float32, device=h_last.device)
            out_stride = G
        if not (out.is_cuda and out.is_contiguous() and out.dtype == torch.float32):
            raise GgnnError("out must be a contiguous fp32 CUDA tensor")
        stride = G if out_stride is None else int(out_stride)
        if torch.is_tensor(slot):
            if not (slot.is_cuda and slot.dtype == torch.int32 and slot.is_contiguous() and slot.numel() == G):
                raise GgnnError("slot must be a contiguous int32 CUDA tensor with %d elements" % G)
            slot_ptr = slot.data_ptr()
        else:
            slot_ptr = slot
        if G and out.numel() < (K - 1) * stride + 1:
            raise GgnnError("out has %d elements for %d tasks at stride %d" % (out.numel(), K, stride))
        self._check(self.lib.ggnn_readout_predict(self._h, self._f32(h_last, V * D, "h_last"), self._f32(h0, V * D, "h0"), K,
                                                  self._readout_tasks(readout_tasks), slot_ptr, stride, out.data_ptr(), self._stream()))
        return out

    def readout_backward(self, h_last, h0, w_gate, b_gate, w_trans, b_trans, d_out):
        import torch
        V, G = self._readout_shape
        D = self.D
        d_h = torch.empty(V, D, dtype=torch.float32, device=h_last.device)
        d_wg = torch.zeros(2 * D, dtype=torch.float32, device=h_last.device)
        d_wt = torch.zeros(D, dtype=torch.float32, device=h_last.device)
        d_b = torch.zeros(2, dtype=torch.float32, device=h_last.device)
        self._check(self.lib.ggnn_readout_backward(
            self._h, self._f32(h_last, V * D, "h_last"), self._f32(h0, V * D, "h0"), self._f32(w_gate, 2 * D, "w_gate"), self._f32(b_gate, 1, "b_gate"),
            self._f32(w_trans, D, "w_trans"), self._f32(b_trans, 1, "b_trans"), self._f32(d_out, G, "d_out"), d_h.data_ptr(), d_wg.data_ptr(),
            d_b.data_ptr(), d_wt.data_ptr(), d_b.data_ptr() + 4, self._stream()))
        return d_h, d_wg, d_b[0:1], d_wt, d_b[1:2]

    # ------------------------------------------------------------------ introspection
    def num_messages(self) -> int:
        m = C.c_int64()
        self._check(self.lib.ggnn_num_messages(self._h, C.byref(m)))
        return int(m.value)

    def csr(self):
        M = self.num_messages()
        row_ptr = np.empty(self.V * self.T + 1, np.int32)
        src = np.empty(M, np.int32)
        msg = np.empty(M, np.int32)
        self._check(self.lib.ggnn_get_csr(self._h, row_ptr.ctypes.data, src.ctypes.data, msg.ctypes.data))
        return row_ptr, src, msg

    def layer_state(self, layer: int):
        """Copy of node_states_per_layer[layer] (0 = h0, L = result) of the last forward, as a CUDA tensor."""
        import torch
        out = torch.empty(self.V, self.D, dtype=torch.float32, device="cuda:%d" % self.device)
        if self.V == 0:   # nothing to copy (an empty tensor has no storage); the engine still says whether the state exists
            self._check(self.lib.ggnn_layer_state(self._h, int(layer), C.byref(C.c_void_p())))
            return out
        self._check(self.lib.ggnn_copy_layer_state(self._h, int(layer), out.data_ptr(), self._stream()))
        return out

    @property
    def last_launch_count(self) -> int:
        return int(self.lib.ggnn_last_launch_count(self._h))

    @property
    def plan(self) -> str:
        return self.lib.ggnn_plan_description(self._h).decode()


class GCNEngine(PropagationEngine):
    """The sparse GCN model (chem_tensorflow_gcn.py:42-82) on the same C ABI: ``ggnn_gcn_create`` / ``ggnn_gcn_set_weights`` /
    ``ggnn_set_graph_gcn`` / ``ggnn_gcn_backward``; forward, readout, dropout, save-for-backward, prepared graphs and introspection are
    the inherited calls.  The GGNN-only calls raise ``GgnnError`` (the library refuses them on a GCN engine).

    ``wide_hidden`` (``ggnn_gcn_config.wide_hidden``): hidden sizes up to 512, and above 128 on bf16x3 / bf16 the streaming wgmma plan
    (a weighted gather and one GEMM launch per layer) instead of the fp32 kernel.  Batches and datasets must be prepared with the same value.

    Adjacency weights on the device: ``prepare_graph_gcn_message_weighted`` + ``set_graph_prepared`` (or, with the list on the GPU,
    ``set_graph_gcn_device``), then ``set_message_weights(w)`` (the inherited call) before every forward that should use new weights, and
    ``backward(..., d_adjacency_weights=)`` for their gradient."""

    def __init__(self, hidden_size: int, num_layers: int, use_bias: bool = False, device: int = 0, precision: str = "fp32",
                 wide_hidden: bool = False):
        self._h = C.c_void_p()
        self.lib = _lib.load()
        self.params = {"hidden_size": int(hidden_size), "num_timesteps": int(num_layers), "gcn_use_bias": bool(use_bias)}
        self.D, self.T, self.L = int(hidden_size), 1, int(num_layers)
        self.use_bias = bool(use_bias)
        self.wide_hidden = bool(wide_hidden)
        cfg = _lib.GcnConfig(self.D, self.L, int(self.use_bias), PRECISIONS[precision], int(device), int(self.wide_hidden))
        rc = self.lib.ggnn_gcn_create(C.byref(cfg), C.byref(self._h))
        if rc != 0:
            self._h = C.c_void_p()
            raise GgnnError(self.lib.ggnn_last_error(None).decode())
        self.device = int(device)
        self.V = 0
        self.serial = 0   # bumped by every forward, graph upload and weight binding: see require_serial
        self._weights_keepalive = None
        self._graph_keepalive = None

    def set_weights(self, kernels: Sequence, biases: Optional[Sequence] = None):
        """``kernels[l]``: [D, D] fp32 CUDA tensor (gcn_weights_l); ``biases[l]``: [D] (gcn_bias_l) when the engine uses biases."""
        arr = (_lib.GcnLayerWeights * len(kernels))()
        keep = []
        for l, k in enumerate(kernels):
            arr[l].kernel = self._f32(k, self.D * self.D, "layer %d kernel" % l)
            keep.append(k)
            if self.use_bias:
                if biases is None:
                    raise GgnnError("the engine uses biases: pass biases")
                arr[l].bias = self._f32(biases[l], self.D, "layer %d bias" % l)
                keep.append(biases[l])
        self.serial += 1
        self._check(self.lib.ggnn_gcn_set_weights(self._h, arr, len(kernels)))
        self._weights_keepalive = keep

    def set_graph_gcn(self, num_nodes: int, adjacency_list, adjacency_weights):
        """The reference's feed (chem_tensorflow_gcn.py:44-47): ``[nnz, 2]`` (row i = output, column j = input) and ``[nnz]`` weights, HOST
        arrays; validation, stable CSR build, tile plan and upload happen in the library."""
        lst, w = _gcn_arrays(adjacency_list, adjacency_weights)
        self.serial += 1
        self._check(self.lib.ggnn_set_graph_gcn(self._h, int(num_nodes), lst.shape[0], lst.ctypes.data, w.ctypes.data, self._stream()))
        self.V = int(num_nodes)
        self._graph_keepalive = (lst, w)

    def prepare_graph_gcn(self, num_nodes: int, adjacency_list, adjacency_weights, save_for_backward: Optional[bool] = None,
                          reuse: Optional[PreparedGraph] = None) -> PreparedGraph:
        """The HOST half of ``set_graph_gcn`` (may run in a producer thread); adopt the result with ``set_graph_prepared``."""
        lst, w = _gcn_arrays(adjacency_list, adjacency_weights)
        g = reuse if reuse is not None else PreparedGraph(self.lib)
        return g._fill(self.lib.ggnn_prepare_graph_gcn, int(num_nodes), 1, self._h, -1 if save_for_backward is None else int(bool(save_for_backward)),
                       int(num_nodes), lst.shape[0], lst.ctypes.data, w.ctypes.data)

    def prepare_graph_gcn_message_weighted(self, num_nodes: int, adjacency_list, save_for_backward: Optional[bool] = None,
                                           reuse: Optional[PreparedGraph] = None) -> PreparedGraph:
        """``prepare_graph_gcn`` for a MESSAGE-WEIGHTED batch (``ggnn_prepare_graph_gcn_message_weighted``): the list alone, no host weights.
        After ``set_graph_prepared``, ``set_message_weights(w)`` puts the adjacency weights on the device -- ``w`` a contiguous fp32 CUDA
        tensor of ``num_messages()`` = nnz entries in list order -- and every forward uses them as ``adjacency_weights``; ``backward(...,
        d_adjacency_weights=)`` adds their gradient.  One prepared batch takes new weights every step (learned edge weights, DropEdge with
        renormalization) without host work."""
        lst = _gcn_list(adjacency_list)
        g = reuse if reuse is not None else PreparedGraph(self.lib)
        return g._fill(self.lib.ggnn_prepare_graph_gcn_message_weighted, int(num_nodes), 1, self._h,
                       -1 if save_for_backward is None else int(bool(save_for_backward)), int(num_nodes), lst.shape[0], lst.ctypes.data)

    def set_graph_gcn_device(self, num_nodes: int, adjacency_list):
        """``prepare_graph_gcn_message_weighted`` + ``set_graph_prepared`` with the list already on the GPU (``ggnn_set_graph_gcn_device``):
        ``adjacency_list`` a contiguous int64 CUDA tensor ``[nnz, 2]`` (row i = output, column j = input) on the engine's device.  The batch
        is built on the device, with the host's plan, into the image the host builder would upload, byte for byte; follow with
        ``set_message_weights(w)`` (``w`` fp32 CUDA ``[nnz]`` in list order) before a forward.  The call waits for the current stream for
        three small reads at most; the tensor is kept alive until the next graph upload."""
        import torch
        V = int(num_nodes)
        if V < 0:
            raise GgnnError("num_nodes must be >= 0, got %d" % V)
        a = adjacency_list
        if not isinstance(a, torch.Tensor):
            raise GgnnError("adjacency_list must be a torch tensor, got %s" % type(a).__name__)
        if a.dtype != torch.int64:
            raise GgnnError("adjacency_list must be int64, got %s" % a.dtype)
        if a.dim() != 2 or a.shape[1] != 2:
            raise GgnnError("adjacency_list must be [nnz, 2], got %s" % (tuple(a.shape),))
        if not a.is_contiguous():
            raise GgnnError("adjacency_list must be contiguous")
        if a.device != torch.device("cuda", self.device):
            raise GgnnError("adjacency_list must be on cuda:%d, got %s" % (self.device, a.device))
        self.serial += 1
        self._check(self.lib.ggnn_set_graph_gcn_device(self._h, V, a.shape[0], a.data_ptr() if a.shape[0] else None, self._stream()))
        self.V = V
        self._graph_keepalive = (a,)

    def backward(self, d_out, grads: Sequence[dict], d_h0=None, d_adjacency_weights=None):
        """``grads[l]``: dict with optional ``kernel`` [D, D] / ``bias`` [D] fp32 CUDA tensors, accumulated into.  With
        ``d_adjacency_weights`` (fp32 CUDA [num_messages()], accumulated into; message-weighted batches only) ``ggnn_gcn_backward_weighted``,
        which also forms the adjacency weights' gradient."""
        arr = (_lib.GcnLayerWeights * len(grads))()
        for l, g in enumerate(grads):
            arr[l].kernel = None if g.get("kernel") is None else g["kernel"].data_ptr()
            arr[l].bias = None if g.get("bias") is None else g["bias"].data_ptr()
        if d_adjacency_weights is None:
            self._check(self.lib.ggnn_gcn_backward(self._h, d_out.data_ptr(), arr, len(grads), None if d_h0 is None else d_h0.data_ptr(),
                                                   self._stream()))
            return
        import torch
        if not (isinstance(d_adjacency_weights, torch.Tensor) and d_adjacency_weights.is_cuda and d_adjacency_weights.dtype == torch.float32
                and d_adjacency_weights.is_contiguous() and d_adjacency_weights.numel() == self.num_messages()):
            raise GgnnError("d_adjacency_weights must be a contiguous fp32 CUDA tensor of num_messages() entries")
        self._check(self.lib.ggnn_gcn_backward_weighted(self._h, d_out.data_ptr(), arr, len(grads), None if d_h0 is None else d_h0.data_ptr(),
                                                        d_adjacency_weights.data_ptr() if d_adjacency_weights.numel() else None,
                                                        self._stream()))
