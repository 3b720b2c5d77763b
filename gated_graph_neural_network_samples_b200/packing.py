"""Host-side batch packing: raw molecule dicts -> the wire format the propagation engine consumes.

Mirrors (behaviour, not code) the reference packers that sit just before the hot path:

* sparse: ``chem_tensorflow_sparse.py:234-276`` (``process_raw_graphs`` / ``__graph_to_adjacency_lists``)
  and ``:278-350`` (``make_minibatch_iterator``): per edge type an ``[E_e, 2]`` int32 list of
  ``(source, target)`` sorted by (source, target), both directions when ``tie_fwd_bkwd``; per node and
  type the in-degree (multi-edges counted); graphs concatenated into one disconnected batch with node
  offsets until the *node* budget ``batch_size`` would be reached (strict ``<``, sparse:297).
* dense: ``chem_tensorflow_dense.py:30-36,132-228``: ``amat[e, dest, src] = 1`` (assignment, duplicates
  collapse), features and mask padded to the bucket size.

Outputs are keyed like the reference's ``self.placeholders`` feed-dict slots (sparse:331-348,
dense:214-224).  tests/test_packing.py checks them against batches produced by the reference's own
NumPy code (tests/golden/make_golden.py).
"""
from __future__ import annotations

from typing import Dict, Iterable, List, Sequence

import numpy as np


# ------------------------------------------------------------------------------------------ sparse
def graph_to_adjacency_lists(graph: Sequence[Sequence[int]], tie_fwd_bkwd: bool = True):
    """One molecule's ``[[src, bond(1..), dst], ...]`` -> ({type: [E,2] int32 sorted}, {type: {node: indeg}}).

    Only ``tie_fwd_bkwd=True`` is supported: the reference's untied branch indexes past
    ``num_edge_types`` (sparse:271 vs chem_tensorflow.py:120; SURVEY 8a "latent bugs")."""
    if not tie_fwd_bkwd:
        raise Exception("tie_fwd_bkwd=False is broken in the reference sparse model and not supported")
    g = np.asarray(graph, dtype=np.int64).reshape(-1, 3)
    adj: Dict[int, np.ndarray] = {}
    indeg: Dict[int, Dict[int, int]] = {}
    for t in np.unique(g[:, 1]):
        rows = g[g[:, 1] == t]
        src = np.concatenate([rows[:, 0], rows[:, 2]])
        dst = np.concatenate([rows[:, 2], rows[:, 0]])
        order = np.lexsort((dst, src))  # == sorted(list of (src, dst) tuples), sparse:265
        e = int(t) - 1                  # sparse:258
        adj[e] = np.stack([src[order], dst[order]], axis=1).astype(np.int32)
        nodes, counts = np.unique(dst, return_counts=True)
        indeg[e] = {int(n): int(c) for n, c in zip(nodes, counts)}
    return adj, indeg


def process_raw_graphs_sparse(raw_data: Iterable[dict], task_ids=(0,), tie_fwd_bkwd: bool = True, labels: bool = True) -> List[dict]:
    """sparse:234-252 without the training-time shuffle / task sub-sampling (caller's business).  ``labels=False``: graphs to predict,
    which need no ``"targets"`` key -- every graph gets an empty label list (batches of them have ``[0, G]`` targets)."""
    out = []
    for d in raw_data:
        adj, indeg = graph_to_adjacency_lists(d["graph"], tie_fwd_bkwd)
        out.append({"adjacency_lists": adj, "num_incoming_edge_per_type": indeg, "init": d["node_features"],
                    "labels": [d["targets"][t][0] for t in task_ids] if labels else []})
    return out


def pack_sparse_batch(graphs: Sequence[dict], hidden_size: int, num_edge_types: int) -> dict:
    """Concatenate processed graphs into one disconnected batch (sparse:288-350)."""
    feats, gnl, indeg_rows, tv, tm = [], [], [], [], []
    per_type: List[List[np.ndarray]] = [[] for _ in range(num_edge_types)]
    offset = 0
    for gi, g in enumerate(graphs):
        init = np.asarray(g["init"], dtype=np.float32)
        n, ann = init.shape
        padded = np.zeros((n, hidden_size), dtype=np.float32)                  # sparse:300-302
        padded[:, :ann] = init
        feats.append(padded)
        gnl.append(np.full(n, gi, dtype=np.int32))                             # sparse:304
        for e in range(num_edge_types):                                        # sparse:305-307
            a = g["adjacency_lists"].get(e)
            if a is not None:
                per_type[e].append(a + np.int32(offset))
        deg = np.zeros((n, num_edge_types), dtype=np.float32)                  # sparse:310-313
        for e, dct in g["num_incoming_edge_per_type"].items():
            for node, cnt in dct.items():
                deg[node, e] = cnt
        indeg_rows.append(deg)
        tv.append([0.0 if v is None else v for v in g["labels"]])              # sparse:316-326
        tm.append([0.0 if v is None else 1.0 for v in g["labels"]])
        offset += n
    adjacency_lists = [np.concatenate(l).astype(np.int32) if l else np.zeros((0, 2), np.int32)  # sparse:343-347
                       for l in per_type]
    return {
        "initial_node_representation": np.concatenate(feats, axis=0) if feats else np.zeros((0, hidden_size), np.float32),
        "adjacency_lists": adjacency_lists,
        "num_incoming_edges_per_type": np.concatenate(indeg_rows, axis=0) if indeg_rows
        else np.zeros((0, num_edge_types), np.float32),
        "graph_nodes_list": np.concatenate(gnl) if gnl else np.zeros(0, np.int32),
        "target_values": np.asarray(tv, dtype=np.float32).T.reshape(-1, len(graphs)),
        "target_mask": np.asarray(tm, dtype=np.float32).T.reshape(-1, len(graphs)),
        "num_graphs": len(graphs),
    }


def iter_sparse_minibatches(data: Sequence[dict], batch_size_nodes: int, hidden_size: int, num_edge_types: int):
    """sparse:286-350: greedy packing while ``node_offset + len(graph) < batch_size`` (strict)."""
    i = 0
    while i < len(data):
        start, nodes = i, 0
        while i < len(data) and nodes + len(data[i]["init"]) < batch_size_nodes:
            nodes += len(data[i]["init"])
            i += 1
        if i == start:
            raise Exception("graph %d has %d nodes and does not fit batch_size=%d"
                            % (i, len(data[i]["init"]), batch_size_nodes))  # the reference loops forever here
        yield pack_sparse_batch(data[start:i], hidden_size, num_edge_types)


class _FlatGraphs:
    """What the flattened graph sets share: ``n_nodes`` per graph, ``pack(idx, hidden_size)`` for one batch, and the node-budget batching."""

    @staticmethod
    def _ranges(starts: np.ndarray, lengths: np.ndarray) -> np.ndarray:
        """Concatenation of arange(starts[i], starts[i] + lengths[i])."""
        total = int(lengths.sum())
        if total == 0:
            return np.zeros(0, np.int64)
        out_off = np.cumsum(lengths) - lengths
        return np.arange(total, dtype=np.int64) + np.repeat(starts - out_off, lengths)

    def iter_minibatches(self, order, batch_size_nodes: int, hidden_size: int):
        """The greedy node-budget batching of sparse:286-297 / gcn:150-162 over the graphs in ``order`` (flat ids)."""
        for idx in self.iter_batch_ids(order, batch_size_nodes):
            yield self.pack(idx, hidden_size)

    def iter_batch_ids(self, order, batch_size_nodes: int):
        """The flat ids of every batch ``iter_minibatches`` packs, in its order (what a device-resident dataset assembles batches from)."""
        order = np.asarray(order, dtype=np.int64)
        csum = np.cumsum(self.n_nodes[order])
        start, N = 0, order.shape[0]
        while start < N:
            base = int(csum[start - 1]) if start else 0
            end = int(np.searchsorted(csum, base + batch_size_nodes, side="left"))   # graphs whose running node count stays < budget
            if end == start:
                raise Exception("graph %d has %d nodes and does not fit batch_size=%d"
                                % (start, int(self.n_nodes[order[start]]), batch_size_nodes))
            yield order[start:end]
            start = end


class FlatSparseGraphs(_FlatGraphs):
    """Processed graphs (``process_raw_graphs_sparse``) flattened ONCE into a few contiguous arrays, so that assembling a batch
    is a constant number of NumPy gathers instead of the per-graph Python loop of sparse:288-350 (SURVEY 8f-3: at a 100 k-node
    batch the loop costs ~0.26 s against a 9 ms training step).  ``pack(idx)`` returns exactly what
    ``pack_sparse_batch([graphs[i] for i in idx])`` returns -- same keys, dtypes, values (tests/test_packing.py)."""

    def __init__(self, graphs: Sequence[dict], num_edge_types: int):
        T, N = int(num_edge_types), len(graphs)
        self.num_edge_types, self.num_graphs = T, N
        self.n_nodes = np.fromiter((len(g["init"]) for g in graphs), dtype=np.int64, count=N)
        self.node_off = np.concatenate([[0], np.cumsum(self.n_nodes)])
        V = int(self.node_off[-1])
        self.ann = max((np.asarray(g["init"]).shape[1] for g in graphs), default=0)
        self.feat = np.zeros((V, self.ann), np.float32)
        self.indeg = np.zeros((V, T), np.float32)
        ntasks = len(graphs[0]["labels"]) if N else 0
        self.labels = np.zeros((N, ntasks), np.float32)
        self.mask = np.zeros((N, ntasks), np.float32)
        counts = np.zeros((T, N), np.int64)
        for i, g in enumerate(graphs):
            for e, a in g["adjacency_lists"].items():
                if e < T:
                    counts[e, i] = len(a)
        self.edge_off = [np.concatenate([[0], np.cumsum(counts[e])]) for e in range(T)]
        self.edges = [np.zeros((int(self.edge_off[e][-1]), 2), np.int32) for e in range(T)]
        for i, g in enumerate(graphs):
            o = int(self.node_off[i])
            init = np.asarray(g["init"], np.float32)
            self.feat[o:o + init.shape[0], :init.shape[1]] = init
            for e, a in g["adjacency_lists"].items():
                if e < T and len(a):
                    self.edges[e][self.edge_off[e][i]:self.edge_off[e][i + 1]] = a
            for e, dct in g["num_incoming_edge_per_type"].items():
                for node, cnt in dct.items():
                    self.indeg[o + node, e] = cnt
            for k, v in enumerate(g["labels"]):
                if v is not None:
                    self.labels[i, k] = v
                    self.mask[i, k] = 1.0

    def pack(self, idx, hidden_size: int) -> dict:
        idx = np.asarray(idx, dtype=np.int64)
        G, T = idx.shape[0], self.num_edge_types
        n = self.n_nodes[idx]
        batch_off = np.cumsum(n) - n                                            # node offset of each graph in the batch
        nodes = self._ranges(self.node_off[idx], n)
        V = nodes.shape[0]
        feats = np.zeros((V, hidden_size), np.float32)                          # sparse:300-302
        feats[:, :self.ann] = self.feat[nodes]
        adjacency_lists = []
        for e in range(T):                                                      # sparse:305-307, 343-347
            m = self.edge_off[e][idx + 1] - self.edge_off[e][idx]
            rows = self._ranges(self.edge_off[e][idx], m)
            adjacency_lists.append((self.edges[e][rows] + np.repeat(batch_off, m).astype(np.int32)[:, None]).astype(np.int32)
                                   if rows.shape[0] else np.zeros((0, 2), np.int32))
        return {
            "initial_node_representation": feats,
            "adjacency_lists": adjacency_lists,
            "num_incoming_edges_per_type": self.indeg[nodes] if V else np.zeros((0, T), np.float32),
            "graph_nodes_list": np.repeat(np.arange(G, dtype=np.int32), n),     # sparse:304
            "target_values": np.ascontiguousarray(self.labels[idx].T).reshape(-1, G),
            "target_mask": np.ascontiguousarray(self.mask[idx].T).reshape(-1, G),
            "num_graphs": G,
        }


# ------------------------------------------------------------------------------------------- dense
DEFAULT_BUCKET_SIZES = np.array(list(range(4, 28, 2)) + [29])  # dense:134


def graph_to_adj_mat(graph, max_n_vertices: int, num_edge_types: int, tie_fwd_bkwd: bool = True) -> np.ndarray:
    """dense:30-36 -- [T, v, v] with amat[e-1, dest, src] = 1 and the tied reverse entry."""
    g = np.asarray(graph, dtype=np.int64).reshape(-1, 3)
    bwd = 0 if tie_fwd_bkwd else num_edge_types // 2
    amat = np.zeros((num_edge_types, max_n_vertices, max_n_vertices), dtype=np.float32)
    amat[g[:, 1] - 1, g[:, 2], g[:, 0]] = 1.0
    amat[g[:, 1] - 1 + bwd, g[:, 0], g[:, 2]] = 1.0
    return amat


def pack_dense_batch(raw_graphs: Sequence[dict], bucket_size: int, hidden_size: int, num_edge_types: int,
                     task_ids=(0,), tie_fwd_bkwd: bool = True) -> dict:
    """dense:142-148,172-224 for one bucket: [b,T,v,v] adjacency, [b,v,D] features, [b,v] mask."""
    b = len(raw_graphs)
    adj = np.zeros((b, num_edge_types, bucket_size, bucket_size), dtype=np.float32)
    init = np.zeros((b, bucket_size, hidden_size), dtype=np.float32)
    mask = np.zeros((b, bucket_size), dtype=np.float32)
    # all graphs' edge triples in one array with their graph index: the adjacency is filled by two fancy-index assignments
    # (same semantics as graph_to_adj_mat per graph: assignment, duplicates collapse, dense:30-36) instead of b small ones
    edges = [np.asarray(d["graph"], dtype=np.int64).reshape(-1, 3) for d in raw_graphs]
    if b:
        counts = np.fromiter((e.shape[0] for e in edges), dtype=np.int64, count=b)
        g = np.concatenate(edges, axis=0)
        gi = np.repeat(np.arange(b), counts)
        bwd = 0 if tie_fwd_bkwd else num_edge_types // 2
        adj[gi, g[:, 1] - 1, g[:, 2], g[:, 0]] = 1.0
        adj[gi, g[:, 1] - 1 + bwd, g[:, 0], g[:, 2]] = 1.0
    tv = np.zeros((b, len(task_ids)), np.float32)
    tm = np.zeros((b, len(task_ids)), np.float32)
    for i, d in enumerate(raw_graphs):
        f = np.asarray(d["node_features"], dtype=np.float32)
        init[i, :f.shape[0], :f.shape[1]] = f
        mask[i, :f.shape[0]] = 1.0
        for k, t in enumerate(task_ids):
            v = d["targets"][t][0]
            if v is not None:
                tv[i, k] = v
                tm[i, k] = 1.0
    tv, tm = tv.tolist(), tm.tolist()
    return {"initial_node_representation": init, "adjacency_matrix": adj, "node_mask": mask,
            "num_vertices": int(bucket_size), "num_graphs": b,
            "target_values": np.asarray(tv, np.float32).T.reshape(-1, b),
            "target_mask": np.asarray(tm, np.float32).T.reshape(-1, b)}


class FlatDenseGraphs:
    """The dense plug-in's processed graphs (raw molecule dicts, ``DenseGGNNChemModel.process_raw_graphs``) flattened ONCE for a
    device-resident dataset (``engine.DeviceDataset``): ``n_nodes`` the node_features rows of every graph (its node mask's extent; edges may
    name nodes beyond it), ``triples`` the raw ``(src, bond, dest)`` rows ``[sum E, 3]`` int64 with ``edge_off`` ``[N+1]``, ``feat`` the
    node features ``[sum n_nodes, ann]``, and per task of ``task_ids`` the label and its mask ``[N, tasks]`` -- a ``None`` target (dropped
    by ``task_sample_ratios``, dense:153-158) has mask 0, as ``pack_dense_batch`` gives it."""

    def __init__(self, graphs: Sequence[dict], task_ids=(0,), tie_fwd_bkwd: bool = True):
        N = len(graphs)
        self.num_graphs, self.tie_fwd_bkwd = N, bool(tie_fwd_bkwd)
        edges = [np.asarray(d["graph"], dtype=np.int64).reshape(-1, 3) for d in graphs]
        self.edge_off = np.concatenate([[0], np.cumsum([e.shape[0] for e in edges])]).astype(np.int64)
        self.triples = np.concatenate(edges, axis=0) if N else np.zeros((0, 3), np.int64)
        feats = [np.asarray(d["node_features"], dtype=np.float32) for d in graphs]
        self.n_nodes = np.fromiter((f.shape[0] for f in feats), dtype=np.int64, count=N)
        self.ann = max((f.shape[1] for f in feats if f.ndim == 2), default=0)
        self.feat = np.zeros((int(self.n_nodes.sum()), self.ann), np.float32)
        self.labels = np.zeros((N, len(task_ids)), np.float32)
        self.mask = np.zeros((N, len(task_ids)), np.float32)
        o = 0
        for i, (d, f) in enumerate(zip(graphs, feats)):
            if f.size:
                self.feat[o:o + f.shape[0], :f.shape[1]] = f
            o += f.shape[0]
            for k, t in enumerate(task_ids):
                v = d["targets"][t][0]
                if v is not None:
                    self.labels[i, k] = v
                    self.mask[i, k] = 1.0


def bucket_batches(raw_graphs: Sequence[dict], batch_size: int, bucket_sizes=DEFAULT_BUCKET_SIZES):
    """The dense model's bucketing (dense:132-141) for prediction: ``(bucket size, input indices)`` of every batch -- each bucket's graphs
    in input order, cut into batches of at most ``batch_size`` graphs, the last one short (training drops it, dense:159-160; a prediction
    needs every graph).  Reads no ``"targets"``: pack the batches with ``pack_dense_batch(..., task_ids=())``."""
    by_bucket: Dict[int, List[int]] = {}
    for i, d in enumerate(raw_graphs):
        by_bucket.setdefault(choose_bucket(d["graph"], bucket_sizes), []).append(i)
    for b, idx in by_bucket.items():
        for s in range(0, len(idx), batch_size):
            yield int(bucket_sizes[b]), np.asarray(idx[s:s + batch_size], np.int64)


def choose_bucket(graph, bucket_sizes=DEFAULT_BUCKET_SIZES) -> int:
    """dense:138-140 -- first bucket strictly larger than the largest node id."""
    g = np.asarray(graph).reshape(-1, 3)
    mx = int(max(g[:, 0].max(), g[:, 2].max()))
    return int(np.argmax(np.asarray(bucket_sizes) > mx))


# ------------------------------------------------------------------------------------------- sparse GCN
def graph_to_gcn_adjacency(graph, num_nodes: int):
    """chem_tensorflow_gcn.py:116-142 in float64: ``A[src, dst] = A[dst, src] = 1`` (assignment: duplicate bonds collapse, bond types are
    ignored), ``A += I``, ``d = rowsum(A)^-0.5 + 1e-7``, ``diag(d) A diag(d)``; the nonzeros in row-major ``(i, j)`` order as
    ``([nnz, 2] int64, [nnz] float64)``."""
    a = np.zeros((num_nodes, num_nodes))
    g = np.asarray(graph, dtype=np.int64).reshape(-1, 3)
    a[g[:, 0], g[:, 2]] = 1
    a[g[:, 2], g[:, 0]] = 1
    a += np.eye(num_nodes)
    d = np.diag(np.power(np.sum(a, axis=-1), -0.5).flatten() + 1e-7)
    a = d.dot(a).dot(d)
    i, j = np.nonzero(a)   # row-major order, exactly the reference's double loop over w != 0
    return np.stack([i, j], axis=1).astype(np.int64).reshape(-1, 2), a[i, j]


def process_raw_graphs_gcn(raw_data: Iterable[dict], task_ids=(0,), labels: bool = True) -> List[dict]:
    """chem_tensorflow_gcn.py:96-103 without the training-time shuffle / task sub-sampling (caller's business).  ``labels=False`` as for
    ``process_raw_graphs_sparse``."""
    out = []
    for d in raw_data:
        lst, w = graph_to_gcn_adjacency(d["graph"], len(d["node_features"]))
        out.append({"adjacency_list": lst, "adjacency_weights": w, "init": d["node_features"],
                    "labels": [d["targets"][t][0] for t in task_ids] if labels else []})
    return out


def pack_gcn_batch(graphs: Sequence[dict], hidden_size: int) -> dict:
    """One batch of chem_tensorflow_gcn.py:150-197: features padded to ``hidden_size``, adjacency lists offset by the node offset of their
    graph and concatenated (weights stay float64, as the reference feeds them), ``graph_nodes_list``, targets / mask ``[tasks, graphs]``."""
    feats, gnl, lists, weights, tv, tm = [], [], [], [], [], []
    offset = 0
    for gi, g in enumerate(graphs):
        init = np.asarray(g["init"], dtype=np.float32)
        n, ann = init.shape
        padded = np.zeros((n, hidden_size), dtype=np.float32)                  # gcn:165-167
        padded[:, :ann] = init
        feats.append(padded)
        gnl.append(np.full(n, gi, dtype=np.int32))                             # gcn:169
        lists.append(np.asarray(g["adjacency_list"], np.int64).reshape(-1, 2) + offset)   # gcn:170
        weights.append(np.asarray(g["adjacency_weights"], np.float64).reshape(-1))
        tv.append([0.0 if v is None else v for v in g["labels"]])              # gcn:173-183
        tm.append([0.0 if v is None else 1.0 for v in g["labels"]])
        offset += n
    return {
        "initial_node_representation": np.concatenate(feats, axis=0) if feats else np.zeros((0, hidden_size), np.float32),
        "adjacency_list": np.concatenate(lists, axis=0) if lists else np.zeros((0, 2), np.int64),
        "adjacency_weights": np.concatenate(weights) if weights else np.zeros(0, np.float64),
        "graph_nodes_list": np.concatenate(gnl) if gnl else np.zeros(0, np.int32),
        "target_values": np.asarray(tv, dtype=np.float32).T.reshape(-1, len(graphs)),
        "target_mask": np.asarray(tm, dtype=np.float32).T.reshape(-1, len(graphs)),
        "num_graphs": len(graphs),
    }


def iter_gcn_minibatches(data: Sequence[dict], batch_size_nodes: int, hidden_size: int):
    """gcn:150-199: greedy packing while ``node_offset + len(graph) < batch_size`` (strict), like the sparse GGNN packer."""
    i = 0
    while i < len(data):
        start, nodes = i, 0
        while i < len(data) and nodes + len(data[i]["init"]) < batch_size_nodes:
            nodes += len(data[i]["init"])
            i += 1
        if i == start:
            raise Exception("graph %d has %d nodes and does not fit batch_size=%d"
                            % (i, len(data[i]["init"]), batch_size_nodes))  # the reference loops forever here
        yield pack_gcn_batch(data[start:i], hidden_size)


class FlatGCNGraphs(_FlatGraphs):
    """Processed GCN graphs (``process_raw_graphs_gcn``) flattened ONCE -- features, graph-local adjacency lists, float64 weights, labels,
    node and entry offsets -- so that a batch is a few NumPy gathers instead of the per-graph loop of gcn:150-197 (at the default
    100 000-node budget that loop is the producer thread's whole cost).  ``pack(idx)`` returns exactly what
    ``pack_gcn_batch([graphs[i] for i in idx])`` returns: same keys, dtypes and values."""

    def __init__(self, graphs: Sequence[dict]):
        N = len(graphs)
        self.num_graphs = N
        self.n_nodes = np.fromiter((len(g["init"]) for g in graphs), dtype=np.int64, count=N)
        self.node_off = np.concatenate([[0], np.cumsum(self.n_nodes)])
        lists = [np.asarray(g["adjacency_list"], np.int64).reshape(-1, 2) for g in graphs]
        self.entry_off = np.concatenate([[0], np.cumsum([l.shape[0] for l in lists])]).astype(np.int64)
        self.lists = np.concatenate(lists, axis=0) if N else np.zeros((0, 2), np.int64)
        self.weights = (np.concatenate([np.asarray(g["adjacency_weights"], np.float64).reshape(-1) for g in graphs]) if N
                        else np.zeros(0, np.float64))
        self.ann = max((np.asarray(g["init"]).shape[1] for g in graphs), default=0)
        self.feat = np.zeros((int(self.node_off[-1]), self.ann), np.float32)
        ntasks = len(graphs[0]["labels"]) if N else 0
        self.labels = np.zeros((N, ntasks), np.float32)
        self.mask = np.zeros((N, ntasks), np.float32)
        for i, g in enumerate(graphs):
            init = np.asarray(g["init"], np.float32)
            o = int(self.node_off[i])
            self.feat[o:o + init.shape[0], :init.shape[1]] = init
            for k, v in enumerate(g["labels"]):
                if v is not None:
                    self.labels[i, k] = v
                    self.mask[i, k] = 1.0

    def pack(self, idx, hidden_size: int) -> dict:
        idx = np.asarray(idx, dtype=np.int64)
        G = idx.shape[0]
        n = self.n_nodes[idx]
        batch_off = np.cumsum(n) - n                                            # node offset of each graph in the batch (gcn:170)
        nodes = self._ranges(self.node_off[idx], n)
        feats = np.zeros((nodes.shape[0], hidden_size), np.float32)             # gcn:165-167
        feats[:, :self.ann] = self.feat[nodes]
        m = self.entry_off[idx + 1] - self.entry_off[idx]
        rows = self._ranges(self.entry_off[idx], m)
        return {
            "initial_node_representation": feats,
            "adjacency_list": self.lists[rows] + np.repeat(batch_off, m)[:, None],
            "adjacency_weights": self.weights[rows],
            "graph_nodes_list": np.repeat(np.arange(G, dtype=np.int32), n),     # gcn:169
            "target_values": np.ascontiguousarray(self.labels[idx].T).reshape(-1, G),
            "target_mask": np.ascontiguousarray(self.mask[idx].T).reshape(-1, G),
            "num_graphs": G,
        }
