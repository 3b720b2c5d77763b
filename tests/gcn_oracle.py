"""Reference restatements of the sparse GCN propagation (chem_tensorflow_gcn.py:59-82) the engine is checked against.

* ``gcn_propagation_loops``: float64, one nonzero at a time in list order -- the specification.
* ``gcn_propagation_torch``: torch on the CPU, autograd-capable (float64 for gradient references, fp32 for a CPU baseline).

State dropout uses the engine's counter-based mask (``PropagationEngine.state_dropout_mask`` with global step = layer index); pass the
per-layer ``[V, D]`` 0/1 masks of layers ``0 .. L-2`` as ``masks``.
"""
import numpy as np


def gcn_propagation_loops(h0, adjacency_list, adjacency_weights, kernels, biases=None, masks=None, keep_prob=1.0):
    h = np.asarray(h0, np.float64)
    lst = np.asarray(adjacency_list, np.int64).reshape(-1, 2)
    w = np.asarray(adjacency_weights, np.float64).reshape(-1)
    L = len(kernels)
    for l in range(L):
        s = np.zeros_like(h)
        for k in range(lst.shape[0]):   # S[i] += w * H[j], in list order
            s[lst[k, 0]] += w[k] * h[lst[k, 1]]
        h = s @ np.asarray(kernels[l], np.float64)
        if biases is not None:
            h = h + np.asarray(biases[l], np.float64)
        if l < L - 1:
            h = np.maximum(h, 0.0)
            if masks is not None:
                h = h * masks[l] / np.float64(np.float32(keep_prob))
    return h


def gcn_propagation_torch(h0, adjacency_list, adjacency_weights, kernels, biases=None, masks=None, keep_prob=1.0):
    """Torch tensors in (any dtype, autograd allowed); ``masks`` as for the loops."""
    import torch
    lst = torch.as_tensor(np.asarray(adjacency_list, np.int64).reshape(-1, 2))
    rows, cols = lst[:, 0], lst[:, 1]
    h = h0
    w = adjacency_weights.to(h0.dtype)
    L = len(kernels)
    for l in range(L):
        s = torch.zeros_like(h).index_add_(0, rows, w[:, None] * h[cols])
        h = s @ kernels[l]
        if biases is not None:
            h = h + biases[l]
        if l < L - 1:
            h = torch.relu(h)
            if masks is not None:
                h = h * torch.as_tensor(masks[l], dtype=h.dtype) / float(np.float32(keep_prob))
    return h


def random_gcn_list(V, nnz, rng, symmetric=False, isolated=()):
    """An unsorted, duplicate-bearing, non-symmetric weighted list over V nodes (nodes in ``isolated`` have no entries at all)."""
    live = np.setdiff1d(np.arange(V), np.asarray(isolated, np.int64))
    lst = np.stack([rng.choice(live, nnz), rng.choice(live, nnz)], axis=1).astype(np.int64)
    if nnz >= 4:
        lst[nnz // 2] = lst[0]        # duplicate (i, j) entries are summed
        lst[nnz // 3] = lst[1]
    if symmetric:
        lst = np.concatenate([lst, lst[:, ::-1]], axis=0)
    w = rng.uniform(-1.0, 1.0, lst.shape[0]).astype(np.float32)
    return lst, w


def component_list(sizes, rng, density=3):
    """Disjoint components of the given sizes (block-diagonal batch, like packed molecules): random non-symmetric entries inside each
    component plus self loops, shuffled over the whole batch."""
    lists, off = [], 0
    for n in sizes:
        m = density * n
        lists.append(np.stack([rng.integers(0, n, m), rng.integers(0, n, m)], axis=1) + off)
        lists.append(np.stack([np.arange(n), np.arange(n)], axis=1) + off)
        off += n
    lst = np.concatenate(lists, axis=0).astype(np.int64)
    lst = lst[rng.permutation(lst.shape[0])]
    w = rng.uniform(-1.0, 1.0, lst.shape[0]).astype(np.float32)
    return off, lst, w


def glorot(shape, rng):
    r = np.sqrt(6.0 / (shape[-2] + shape[-1]))
    return rng.uniform(-r, r, size=shape).astype(np.float32)
