"""CPU: message weights in the sparse GGNN model (ggnn_prepare_graph_sparse_weighted, ggnn_set_message_weights, ggnn_backward_weighted).

A message-weighted batch is the sparse batch with one weight per message that arrives on the device after the upload.  Without a GPU this
file checks:

* the three entries: exported, declared in include/ggnn_b200.h with the argument count the ctypes binding gives them;
* the host-only image (``ggnn_host_prepare_graph_sparse_weighted``) at hidden 100 / fp32, 100 / bf16x3, 256 / bf16x3 and 512 / fp32, with
  and without the source-keyed CSR: CSR, ``msg``, tile plan and denominators are those of the unweighted prepare of the same lists and
  NumPy's stable argsort; the weight sections are zero; the plan text is the unweighted one with " [message-weighted]" appended; on the
  streaming plan the virtual rows are exactly the (target, type) pairs with messages, whatever their count; the image bytes are the same
  at 1, 2, 3, 5 and 8 host threads;
* the refusal of propagation attention (GGNN_EUNSUPPORTED);
* the float64 restatement the GPU tests use (tests/message_weights_oracle.py): all-ones weights give the unweighted oracle, and without
  edge bias and mean a weighted batch is ``dense_propagation_loops`` on the matching weighted matrix;
* the new kernels use no stack and spill nothing.
"""
import ctypes as C
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

from oracle import ggnn_oracle as O
from tests import _util as U
from tests import message_weights_oracle as MW

NUM_SMS = 132
TAG = " [message-weighted]"
ENTRIES = ("ggnn_prepare_graph_sparse_weighted", "ggnn_host_prepare_graph_sparse_weighted", "ggnn_set_message_weights",
           "ggnn_backward_weighted")
SHAPES = [(100, "fp32"), (100, "bf16x3"), (256, "bf16x3"), (512, "fp32")]
HOST_THREADS = (1, 2, 3, 5, 8)
# registers of the new kernels as ptxas made them for sm_90a (none has a stack frame or spills)
KERNEL_REGS = {"scatter_message_weights_kernel": 32, "message_weight_grad_kernel": 40, "add_slot_grads_kernel": 32}


def params(D, cell="GRU", att=False):
    return {"hidden_size": D, "layer_timesteps": [2, 1], "residual_connections": {"1": [0]}, "use_edge_bias": True,
            "use_edge_msg_avg_aggregation": True, "graph_rnn_cell": cell, "graph_rnn_activation": "tanh",
            "use_propagation_attention": att}


def molecules(n, D=100, T=4, seed=0):
    """A packed batch of ``n`` synthetic molecules, with hub rows: node 0 of the batch receives 9 type-0 messages and one type-1 message."""
    _, b = U.molecule_batch(n, D, T, seed)
    adj = [np.asarray(a, np.int32).reshape(-1, 2) for a in b["adjacency_lists"]]
    hub = np.array([[s, 0] for s in range(1, 10)], np.int32)
    adj[0] = np.concatenate([adj[0], hub])
    adj[1] = np.concatenate([adj[1], np.array([[3, 0]], np.int32)])
    V = b["num_incoming_edges_per_type"].shape[0]
    indeg = np.zeros((V, T), np.float32)
    for t, a in enumerate(adj):
        np.add.at(indeg[:, t], a[:, 1], 1.0)
    return adj, indeg


def prepare(D, precision, adj, indeg, weighted=True, save=False, p=None):
    from gated_graph_neural_network_samples_b200.engine import PreparedGraph
    f = PreparedGraph.host_only_weighted if weighted else PreparedGraph.host_only
    return f(p or params(D), len(adj), adj, indeg, precision=precision, num_sms=NUM_SMS, save_for_backward=save)


# ---------------------------------------------------------------------------------------------------------------- ABI
def test_entries_are_exported_declared_and_bound():
    from gated_graph_neural_network_samples_b200 import _lib
    lib = _lib.load()
    header = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "ggnn_b200.h")).read()
    for name in ENTRIES:
        getattr(lib, name)
        m = re.search(r"\bint %s\(([^;]*)\);" % name, header)
        assert m, name
        nargs = len([a for a in m.group(1).split(",") if a.strip()])
        assert len(_lib.SYMBOLS[name][1]) == nargs, (name, nargs)
    # ggnn_backward_weighted is ggnn_backward with one more argument, before the stream
    bw, b = _lib.SYMBOLS["ggnn_backward_weighted"][1], _lib.SYMBOLS["ggnn_backward"][1]
    assert bw[:5] == b[:5] and bw[-1] == b[-1] and len(bw) == len(b) + 1


# ---------------------------------------------------------------------------------------------------------------- the image
@pytest.mark.parametrize("save", [False, True])
@pytest.mark.parametrize("D,precision", SHAPES)
def test_image_is_the_unweighted_batch_with_zero_weights(D, precision, save):
    adj, indeg = molecules(40, D)
    T = len(adj)
    V = indeg.shape[0]
    g = prepare(D, precision, adj, indeg, save=save)
    u = prepare(D, precision, adj, indeg, weighted=False, save=save)
    gi, ui = g.info(), u.info()
    assert gi["plan"] == ui["plan"] + TAG, (gi["plan"], ui["plan"])
    assert gi["num_messages"] == ui["num_messages"] == sum(a.shape[0] for a in adj)
    ga, ua = g.arrays(T), u.arrays(T)
    for k in ("row_ptr", "src", "msg", "tile_start", "denom"):
        np.testing.assert_array_equal(ga[k], ua[k], err_msg=k)
    # NumPy's stable argsort by (target, type) in the reference's message order
    src, tgt, typ = O.message_arrays(adj)
    order = np.argsort(tgt.astype(np.int64) * T + typ, kind="stable")
    np.testing.assert_array_equal(ga["msg"], order)
    np.testing.assert_array_equal(ga["src"], src[order])
    np.testing.assert_array_equal(ga["row_ptr"][1:], np.cumsum(np.bincount(tgt.astype(np.int64) * T + typ, minlength=V * T)))
    np.testing.assert_array_equal(g.slot_weights(), np.zeros(gi["num_messages"], np.float32))
    if save:
        np.testing.assert_array_equal(g.slot_weights(source_order=True), np.zeros(gi["num_messages"], np.float32))
    assert gi["streaming"] == (precision != "fp32" and D > 128)
    if gi["streaming"]:
        rp = ga["row_ptr"]
        counts = np.diff(rp)
        rows = np.nonzero(counts)[0]
        pair = ga["pair_src"][:V * T]
        assert np.all(pair[counts == 0] == -1)
        np.testing.assert_array_equal(pair[rows], -(2 + np.arange(rows.size)))   # every pair with messages, singles included
        st = g.stream_tables()
        np.testing.assert_array_equal(np.diff(st["vrow_ptr"]), counts[rows])
        np.testing.assert_array_equal(st["vslot"], rp[rows])
        np.testing.assert_array_equal(st["vsrc"], ga["src"])
        assert st["vinfo"][:, 0].tolist() == counts[rows].tolist()
        assert np.any(counts[rows] == 1) and np.any(counts[rows] > 7)


@pytest.mark.parametrize("D,precision", [(100, "bf16x3"), (256, "bf16x3"), (512, "fp32")])
def test_image_bytes_do_not_depend_on_host_threads(D, precision, monkeypatch):
    adj, indeg = molecules(300, D, seed=1)
    images = []
    for n in HOST_THREADS:
        monkeypatch.setenv("GGNN_HOST_THREADS", str(n))
        images.append(prepare(D, precision, adj, indeg, save=True).image())
    for n, img in zip(HOST_THREADS[1:], images[1:]):
        np.testing.assert_array_equal(img, images[0], err_msg="%d host threads" % n)


def test_plan_texts():
    adj, indeg = molecules(12)
    expect = {(100, "fp32"): r"^fp32-ffma LOCAL\(", (100, "bf16x3"): r"^wgmma-bf16x3 LOCAL\(", (256, "bf16x3"): r"^wgmma-bf16x3 STREAM\(",
              (512, "fp32"): r"^fp32-stepwise "}
    for (D, precision), pat in expect.items():
        plan = prepare(D, precision, adj, indeg).info()["plan"]
        assert re.match(pat, plan) and plan.endswith(TAG), (D, precision, plan)
    # CudnnCompatibleGRUCell on the tensor cores streams at every hidden size, all pairs virtual as well
    p = params(100, cell="CudnnCompatibleGRUCell")
    from gated_graph_neural_network_samples_b200.engine import PreparedGraph
    g = PreparedGraph.host_only_weighted(p, len(adj), adj, indeg, precision="bf16x3", num_sms=NUM_SMS, cudnn_gru_tensor_cores=True)
    assert "STREAM+cudnn-gru" in g.info()["plan"] and g.info()["plan"].endswith(TAG)
    assert g.stream_tables()["vrow_ptr"].shape[0] - 1 == np.count_nonzero(np.diff(g.arrays(len(adj))["row_ptr"]))


def test_attention_is_refused():
    from gated_graph_neural_network_samples_b200 import _lib
    from gated_graph_neural_network_samples_b200.engine import GgnnError, make_config
    adj, indeg = molecules(4)
    T = len(adj)
    for tc in (False, True):
        cfg, keep = make_config(params(100, att=True), T, 0, "bf16x3", attention_tensor_cores=tc)
        ptrs = (C.c_void_p * T)(*[a.ctypes.data for a in adj])
        counts = (C.c_int32 * T)(*[a.shape[0] for a in adj])
        lib = _lib.load()
        h = C.c_void_p()
        rc = lib.ggnn_host_prepare_graph_sparse_weighted(C.byref(cfg), NUM_SMS, 1, indeg.shape[0], ptrs, counts, indeg.ctypes.data, C.byref(h))
        assert rc == -4, rc   # GGNN_EUNSUPPORTED
        assert "attention" in lib.ggnn_prepared_graph_error(h).decode()
        lib.ggnn_free_prepared_graph(h)
        with pytest.raises(GgnnError, match="attention"):
            prepare(100, "bf16x3", adj, indeg, p=params(100, att=True))


# ---------------------------------------------------------------------------------------------------------------- the oracle
def _small(D=8, T=3, seed=0):
    rng = np.random.default_rng(seed)
    V = 9
    adj = [rng.integers(0, V, size=(int(rng.integers(3, 9)), 2)).astype(np.int32) for _ in range(T)]
    adj[0] = np.concatenate([adj[0], np.array([[4, 4]], np.int32)])   # a self-loop
    indeg = np.zeros((V, T), np.float32)
    for t, a in enumerate(adj):
        np.add.at(indeg[:, t], a[:, 1], 1.0)
    return adj, indeg, rng.normal(0, 0.5, (V, D))


@pytest.mark.parametrize("cell", ["GRU", "RNN", "CudnnCompatibleGRUCell"])
def test_oracle_all_ones_is_the_unweighted_model(cell):
    import torch
    adj, indeg, h0 = _small()
    p = dict(params(8, cell=cell))
    w = O.init_sparse_weights(p, 3, np.random.default_rng(1))
    M = sum(a.shape[0] for a in adj)
    ref = O.sparse_propagation_loops(h0, adj, indeg, w, p)
    np.testing.assert_allclose(MW.propagation_loops(h0, adj, indeg, w, p, np.ones(M)), ref, rtol=1e-12, atol=1e-12)
    got = MW.propagation_torch(h0, adj, indeg, w, p, np.ones(M), dtype=torch.float64).numpy()
    np.testing.assert_allclose(got, ref, rtol=1e-10, atol=1e-12)


@pytest.mark.parametrize("cell", ["GRU", "RNN", "CudnnCompatibleGRUCell"])
def test_oracle_torch_restatement_is_the_loop_statement(cell):
    import torch
    adj, indeg, h0 = _small(seed=2)
    p = dict(params(8, cell=cell))
    w = O.init_sparse_weights(p, 3, np.random.default_rng(3))
    mw = np.random.default_rng(4).normal(size=sum(a.shape[0] for a in adj))
    got = MW.propagation_torch(h0, adj, indeg, w, p, mw, dtype=torch.float64).numpy()
    np.testing.assert_allclose(got, MW.propagation_loops(h0, adj, indeg, w, p, mw), rtol=1e-10, atol=1e-12)


def test_oracle_matches_the_weighted_dense_model():
    """Without edge bias and mean, message weights are the entries of a weighted adjacency: ``dense_propagation_loops``."""
    rng = np.random.default_rng(3)
    b, T, v, D, steps = 3, 2, 5, 8, 3
    A = (rng.random((b, T, v, v)) < 0.4) * rng.normal(0, 1.0, (b, T, v, v))
    adj, mw = [], []
    for t in range(T):
        lst = []
        for g in range(b):
            for i in range(v):
                for j in range(v):
                    if A[g, t, i, j] != 0:
                        lst.append((g * v + j, g * v + i))
                        mw.append(A[g, t, i, j])
        adj.append(np.array(lst, np.int32).reshape(-1, 2))
    dw = O.init_dense_weights({"hidden_size": D, "use_edge_bias": False}, T, rng)
    h0 = rng.normal(0, 0.5, (b, v, D))
    ref = O.dense_propagation_loops(h0, A, dw, {"num_timesteps": steps, "use_edge_bias": False})
    p = {"hidden_size": D, "layer_timesteps": [steps], "residual_connections": {}, "use_edge_bias": False,
         "use_edge_msg_avg_aggregation": False, "graph_rnn_cell": "GRU", "graph_rnn_activation": "tanh"}
    indeg = np.zeros((b * v, T), np.float32)
    got = MW.propagation_loops(h0.reshape(-1, D), adj, indeg, [dw], p, np.array(mw))
    np.testing.assert_allclose(got.reshape(b, v, D), ref, rtol=1e-12, atol=1e-12)


def test_oracle_weight_gradient_is_the_step_sum_of_P_dot_h():
    """d w_m = sum over steps of <P[v, t], h[s_m]>, P = dx' . W_t^T: the torch restatement's autograd against that formula on a one-step
    RNN model (the step input is h0, dx' is the gradient at the pre-mean sum)."""
    import torch
    adj, indeg, h0 = _small(seed=4)
    p = {"hidden_size": 8, "layer_timesteps": [1], "residual_connections": {}, "use_edge_bias": True, "use_edge_msg_avg_aggregation": True,
         "graph_rnn_cell": "RNN", "graph_rnn_activation": "tanh"}
    w = O.init_sparse_weights(p, 3, np.random.default_rng(2))
    M = sum(a.shape[0] for a in adj)
    mw = torch.tensor(np.random.default_rng(5).normal(size=M), dtype=torch.float64, requires_grad=True)
    out = MW.propagation_torch(h0, adj, indeg, w, p, mw, dtype=torch.float64)
    g = torch.tensor(np.random.default_rng(6).normal(size=out.shape), dtype=torch.float64)
    (out * g).sum().backward()
    # by hand: out = tanh([x, h] K + b), x = (sum_m w_m h[s] W_t + indeg B) / denom
    K = torch.tensor(w[0]["rnn_kernel"], dtype=torch.float64)
    src, tgt, typ = O.message_arrays(adj)
    dpre = g * (1 - out.detach() ** 2)
    dx = (dpre @ K[:8].T) / torch.tensor(indeg.astype(np.float64).sum(-1, keepdims=True) + O.SMALL_NUMBER)
    W = torch.tensor(w[0]["edge_weights"], dtype=torch.float64)
    want = [float(dx[tgt[m]] @ W[typ[m]].T @ torch.tensor(h0[src[m]])) for m in range(M)]
    np.testing.assert_allclose(mw.grad.numpy(), want, rtol=1e-10, atol=1e-12)


# ---------------------------------------------------------------------------------------------------------------- the kernels
def _cuobjdump():
    exe = shutil.which("cuobjdump")
    if exe is None:
        cand = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "cuobjdump")
        exe = cand if os.path.exists(cand) else None
    return exe


def test_new_kernels_use_no_stack_and_do_not_spill():
    exe = _cuobjdump()
    if exe is None:
        pytest.skip("cuobjdump is not available")
    from gated_graph_neural_network_samples_b200 import _build, _lib
    _lib.load()
    out = subprocess.run([exe, "-res-usage", _build.LIB_PATH], capture_output=True, text=True, check=True).stdout
    found, name = {}, None
    for line in out.splitlines():
        m = re.match(r"\s*Function (\S+):", line)
        if m:
            name = next((k for k in KERNEL_REGS if k in m.group(1) and "msgw" in m.group(1)), None)
            continue
        if name is not None and "REG:" in line:
            found[name] = {n: int(v) for n, v in re.findall(r"([A-Z_]+):(\d+)", line)}
            name = None
    assert sorted(found) == sorted(KERNEL_REGS), sorted(found)
    for k, r in found.items():
        print("%s %s" % (k, r))
        assert r["STACK"] == 0 and r.get("LOCAL", 0) == 0, (k, r)
        assert r["REG"] <= KERNEL_REGS[k], (k, r)
