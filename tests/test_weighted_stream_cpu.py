"""CPU: weighted dense adjacency on the streaming wgmma plan (hidden sizes above 128 on bf16x3 / bf16).

The streaming gather copies the image row of a (target, type) pair's one source, or of a "virtual row" that the gather launch sums first.
In a weighted batch a pair is a copy only when its one message weighs exactly 1.0f; every other pair with messages is a virtual row, whose
messages are its target-CSR row and whose weights are ``slot_w[vslot[vid] + m]``.  Without a GPU this file checks:

* the plan of every weighted case of tests/test_gpu_weighted_stream.py, at 132 SMs, through ``ggnn_host_prepare_graph_dense_weighted``:
  hidden 132 ... 512 on bf16x3 and bf16, save on and off, is the STREAM plan with the weighted suffix;
* ``pair_src`` and the virtual-row tables against a NumPy restatement from the builder's own CSR and slot weights, on every weight
  regime, hub rows of more than seven messages and 1, 2, 3 and 8 host threads (identical image bytes at each);
* binary matrices: the weighted entry builds the bytes of the binary entry, and their tables keep the binary rule with no ``vslot``;
* up to hidden 128 every weighted case of tests/test_weighted_dense_cpu.py keeps the plan it had (``GGNN_TC_STREAM=1`` ignored);
* the float64 weighted oracle the GPU file uses (any cell, residual inputs, state dropout, every layer's state) agrees with the dense
  oracle on GRU batches and with the sparse oracle on 0/1 batches.
"""
import os
import re

import numpy as np
import pytest

from oracle import ggnn_oracle as O
from tests import _util as U
from tests.test_backward_plans_cpu import plan_matches
from tests.test_forward_plans_cpu import pad16
from tests.test_weighted_dense_cpu import ALL_CASES, BINARY_TAG, HOST_THREADS, NUM_SMS, WEIGHTED_TAG, binary, weigh

STREAM_SIZES = (132, 144, 192, 256, 260, 384, 512)
TC_PRECISIONS = ("bf16x3", "bf16")
HUB_SOURCES = 12        # messages into each hub row: past vinfo's seven inline sources


def stream_pattern(prec, D):
    return r"^wgmma-%s STREAM\(.* DP=%d " % (prec, pad16(D))


def with_hubs(A, sources=HUB_SOURCES):
    """``A`` with a hub row in every other graph: node 0 receives type-0 messages from nodes 1 .. ``sources`` (entries 1.0 where the
    pattern had none, so that a weighing of the result sees them)."""
    A = A.copy()
    A[::2, 0, 0, 1:sources + 1] = np.where(A[::2, 0, 0, 1:sources + 1] != 0, A[::2, 0, 0, 1:sources + 1], 1.0)
    return A


def batch(name):
    """The 0/1 patterns of this file: the weighted dense file's batches, and ``hub`` / ``hub64`` (10 / 64 molecules with hub rows)."""
    if name == "hub":
        return with_hubs(binary("mol"))
    if name == "hub64":
        return with_hubs(binary("mol64"))
    return binary(name)


def matrix(name, regime):
    return weigh(batch(name), regime)


def params(D, steps=3, bias=True, cell="GRU", act="tanh", residual=False):
    """Engine params of a dense-model batch: one layer of ``steps`` timesteps, or with ``residual`` two layers ([2, 1]) whose second
    reads node_states_per_layer[0]."""
    p = U.dense_params_as_engine_params({"num_timesteps": steps, "use_edge_bias": bias}, D)
    p.update(graph_rnn_cell=cell, graph_rnn_activation=act)
    if residual:
        p.update(layer_timesteps=[2, 1], residual_connections={"1": [0]})
    return p


def prepare(A, D, precision, save=False, p=None):
    from gated_graph_neural_network_samples_b200.engine import PreparedGraph
    return PreparedGraph.host_only_dense_weighted(p or params(D), A.shape[1], A, precision=precision, num_sms=NUM_SMS,
                                                  save_for_backward=save)


# ---------------------------------------------------------------------------------------------------------------- the restatement
def restate_stream_tables(row_ptr, src, slot_w, tile_start, T):
    """pair_src, vrow_ptr, vsrc, vinfo, vslot and tile_vptr of a streaming plan from its CSR (``slot_w`` None: a binary batch)."""
    ntiles = len(tile_start) - 1
    pair = np.full(max(ntiles, 1) * 128 * T, -1, np.int32)
    vptr, vsrc, vinfo, vslot, tvp = [0], [], [], [], []
    for i in range(ntiles):
        tvp.append(len(vslot))
        for r in range(tile_start[i] * T, tile_start[i + 1] * T):
            b, e = int(row_ptr[r]), int(row_ptr[r + 1])
            if e == b:
                continue
            if e - b == 1 and (slot_w is None or slot_w[b] == np.float32(1.0)):
                pair[r] = src[b]
                continue
            pair[r] = -(2 + len(vslot))
            vslot.append(b)
            vsrc += [int(s) for s in src[b:e]]
            vptr.append(len(vsrc))
            vinfo.append([e - b] + [int(src[b + m]) if m < e - b else 0 for m in range(7)])
    tvp.append(len(vslot))
    return {"pair_src": pair, "vrow_ptr": np.array(vptr, np.int32), "vsrc": np.array(vsrc, np.int32),
            "vinfo": np.array(vinfo, np.int32).reshape(-1, 8), "vslot": np.array(vslot, np.int32), "tile_vptr": np.array(tvp, np.int32)}


def check_tables(g, A, weighted):
    """Holds g's streaming tables to the restatement from its own CSR and slot weights, and those weights to the matrix entries.
    Returns the tables."""
    T = A.shape[1]
    v = A.shape[2]
    arr = g.arrays(T)
    sw = g.slot_weights() if weighted else None
    if weighted:   # slot m of row (node, type) holds A[graph, type, node % v, source % v]
        rows = np.repeat(np.arange(len(arr["row_ptr"]) - 1), np.diff(arr["row_ptr"]))
        node, t = rows // T, rows % T
        np.testing.assert_array_equal(sw, A[node // v, t, node % v, arr["src"] - (node // v) * v])
    want = restate_stream_tables(arr["row_ptr"], arr["src"], sw, arr["tile_start"], T)
    got = g.stream_tables()
    np.testing.assert_array_equal(arr["pair_src"], want["pair_src"])
    for k in ("vrow_ptr", "vsrc", "vinfo", "tile_vptr"):
        np.testing.assert_array_equal(got[k], want[k], err_msg=k)
    if weighted:
        np.testing.assert_array_equal(got["vslot"], want["vslot"])
    else:
        assert got["vslot"] is None
    return got, arr, sw


# ---------------------------------------------------------------------------------------------------------------- tests
@pytest.mark.parametrize("save", [False, True], ids=["infer", "save"])
@pytest.mark.parametrize("precision", TC_PRECISIONS)
@pytest.mark.parametrize("D", STREAM_SIZES)
def test_weighted_batches_above_hidden_128_stream(D, precision, save):
    plan = prepare(matrix("mol", "uniform"), D, precision, save).info()["plan"]
    assert plan.endswith(WEIGHTED_TAG), plan
    assert plan_matches(plan, stream_pattern(precision, D)), plan


REGIMES = ("uniform", "signed", "ones", "scales", "lastonly")


@pytest.mark.parametrize("regime", REGIMES)
@pytest.mark.parametrize("name", ["hub64", "one200"])
def test_stream_tables_match_the_restatement_at_every_thread_count(name, regime, monkeypatch):
    """Every regime on 64 molecules with hub rows and on two 200-node components, at 1, 2, 3 and 8 host threads: tables equal to the
    restatement, and the same image bytes at every count."""
    A = matrix(name, regime)
    images = []
    for n in HOST_THREADS:
        monkeypatch.setenv("GGNN_HOST_THREADS", str(n))
        g = prepare(A, 256, "bf16x3", save=True)
        assert g.info()["plan"].endswith(WEIGHTED_TAG)
        check_tables(g, A, True)
        images.append(g.image())
    for im in images[1:]:
        np.testing.assert_array_equal(im, images[0])


def test_the_batches_hold_what_the_tables_must_cover():
    """hub64 / uniform: hub rows past vinfo's inline sources; ones: single messages of weight exactly 1 (copies) and of other weights
    (virtual rows of one message); signed: virtual rows whose fp32 weight sum is exactly 0."""
    A = matrix("hub64", "ones")
    tabs, arr, sw = check_tables(prepare(A, 256, "bf16x3"), A, True)
    counts = np.diff(tabs["vrow_ptr"])
    assert counts.max() > 7 and (counts == 1).any() and (counts >= 2).any()
    pair, rp = arr["pair_src"], arr["row_ptr"]
    singles = np.flatnonzero(np.diff(rp) == 1)
    assert (pair[singles] >= 0).any() and (pair[singles] < -1).any()
    assert np.all(sw[rp[singles][pair[singles] >= 0]] == 1.0) and np.all(sw[rp[singles][pair[singles] < -1]] != 1.0)
    S = matrix("hub64", "signed")
    tabs, arr, sw = check_tables(prepare(S, 256, "bf16x3"), S, True)
    sums = np.array([np.add.reduce(sw[s:s + c], dtype=np.float32) for s, c in zip(tabs["vslot"], np.diff(tabs["vrow_ptr"]))])
    assert (sums == 0).any() and (sums != 0).any()
    # a weighted molecule batch makes almost every pair with messages a virtual row; its binary twin only the pairs with several
    Au = matrix("hub64", "uniform")
    nv_w = len(prepare(Au, 256, "bf16x3").stream_tables()["vslot"])
    nv_b = len(prepare(batch("hub64"), 256, "bf16x3").stream_tables()["vrow_ptr"]) - 1
    nonempty = int((np.diff(arr["row_ptr"]) > 0).sum())
    assert nv_w == nonempty and nv_b < nonempty


@pytest.mark.parametrize("D", [132, 256, 512])
@pytest.mark.parametrize("name", ["hub", "one200", "mol64"])
def test_binary_matrices_keep_their_image(name, D, monkeypatch):
    """A 0/1 matrix through the weighted entry: the bytes of the binary entry, the binary plan suffix, the binary table rule (a pair of
    one message is a copy) and no vslot -- at 1 and 8 host threads."""
    from gated_graph_neural_network_samples_b200.engine import PreparedGraph
    A = batch(name)
    p = params(D)
    for n in (1, 8):
        monkeypatch.setenv("GGNN_HOST_THREADS", str(n))
        for save in (False, True):
            gw = prepare(A, D, "bf16x3", save)
            gb = PreparedGraph.host_only_dense(p, A.shape[1], A, precision="bf16x3", num_sms=NUM_SMS, save_for_backward=save)
            assert gw.info()["plan"] == gb.info()["plan"] and gb.info()["plan"].endswith(BINARY_TAG)
            np.testing.assert_array_equal(gw.image(), gb.image())
            check_tables(gb, A, False)


def test_binary_tables_equal_the_independent_reference():
    """The binary dense batch's tables against ggnn_host_stream_tables, the builder-independent statement of the binary rule."""
    import ctypes as C
    from gated_graph_neural_network_samples_b200 import _lib
    A = batch("hub64")
    b, T, v, _ = A.shape
    g = prepare(A, 256, "bf16x3")
    tabs = g.stream_tables()
    lists = []
    for t in range(T):
        gi, i, j = np.nonzero(A[:, t])
        lists.append(np.ascontiguousarray(np.stack([gi * v + j, gi * v + i], 1), np.int32))
    V = b * v
    lib = _lib.load()
    pair = np.empty(((V + 127) // 128) * 128 * T, np.int32)
    vptr, vsrc, tvp = np.empty(V * T + 1, np.int32), np.empty(sum(len(a) for a in lists) + 1, np.int32), np.empty(V // 128 + 2, np.int32)
    nv = C.c_int32()
    rc = lib.ggnn_host_stream_tables(V, T, (C.c_void_p * T)(*[a.ctypes.data for a in lists]), (C.c_int32 * T)(*[len(a) for a in lists]),
                                     pair.ctypes.data, vptr.ctypes.data, len(vptr), vsrc.ctypes.data, len(vsrc), tvp.ctypes.data, C.byref(nv))
    assert rc == 0
    np.testing.assert_array_equal(g.arrays(T)["pair_src"], pair)
    np.testing.assert_array_equal(tabs["vrow_ptr"], vptr[:nv.value + 1])
    np.testing.assert_array_equal(tabs["vsrc"], vsrc[:vptr[nv.value]])
    np.testing.assert_array_equal(tabs["tile_vptr"], tvp[:len(tabs["tile_vptr"])])


def test_stream_tables_refuse_what_a_plan_does_not_carry():
    from gated_graph_neural_network_samples_b200.engine import GgnnError
    with pytest.raises(GgnnError):
        prepare(matrix("mol", "uniform"), 100, "bf16x3").stream_tables()          # hidden 100: the tile kernel, no tables
    import ctypes as C
    g = prepare(batch("mol"), 256, "bf16x3")
    vslot = np.empty(4096, np.int32)
    assert g.lib.ggnn_prepared_graph_stream_tables(g._h, None, None, None, None, None, vslot.ctypes.data, None) != 0   # binary: no vslot


def _with_env(env, fn):
    saved = {k: os.environ.get(k) for k in env}
    os.environ.update(env)
    try:
        return fn()
    finally:
        for k, val in saved.items():
            if val is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = val


@pytest.mark.parametrize("name", sorted(ALL_CASES))
def test_weighted_plans_up_to_hidden_128_are_unchanged(name):
    """Every weighted case of tests/test_weighted_dense_cpu.py (each asserted on the device there) keeps its plan under its environment,
    now pinned without a GPU through the weighted entry; on tensor cores also with GGNN_TC_STREAM=1, which a weighted batch ignores."""
    c = ALL_CASES[name]
    A = c.matrix()
    plan = _with_env(c.env, lambda: prepare(A, c.D, c.precision, p=c.params).info()["plan"])
    assert plan.endswith(WEIGHTED_TAG) and plan_matches(plan, c.pattern), (c.pattern, plan)
    if c.precision != "fp32":
        forced = _with_env(dict(c.env, GGNN_TC_STREAM="1"), lambda: prepare(A, c.D, c.precision, p=c.params).info()["plan"])
        assert forced == plan


# ---------------------------------------------------------------------------------------------------------------- the oracle
def weighted_propagation_torch(h0, A, weights, p, dtype=None, state_dropout=None, return_all_layers=False):
    """float64 reference of the engine on a weighted ``[b, T, v, v]`` matrix, for any cell, residual inputs and state dropout: the sparse
    model's step (sparse:159-216) with message j -> i of type t scaled by A[g, t, i, j] and the in-degrees replaced by the fp32 row sums
    (so the edge-bias term is rowsum . b_t; the engine's fp32 row sums are within its bars of these).  ``weights``: per layer, the sparse oracle's names (``rnn_kernel`` for the RNN cell).
    Returns [b*v, D] (or every node_states_per_layer entry)."""
    import torch
    dtype = dtype or torch.float64
    t = lambda a: a if isinstance(a, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(a))
    b, T, v, _ = A.shape
    h0 = t(h0).to(dtype).reshape(b * v, -1)
    V, D = h0.shape
    gi, ti, ii, jj = np.nonzero(A)
    wmsg = torch.from_numpy(A[gi, ti, ii, jj].astype(np.float64)).to(dtype)
    src, tgt, typ = torch.from_numpy(gi * v + jj), torch.from_numpy(gi * v + ii), torch.from_numpy(ti)
    indeg = torch.from_numpy(A.astype(np.float64).sum(-1).transpose(0, 2, 1).reshape(V, T)).to(dtype)
    act = torch.tanh if p.get("graph_rnn_activation", "tanh").lower() == "tanh" else torch.relu
    cell = p.get("graph_rnn_cell", "GRU").lower()
    states, gs = [h0], 0
    for l, steps in enumerate(p["layer_timesteps"]):
        w = {k: t(x).to(dtype) for k, x in weights[l].items()}
        res = [states[i] for i in O.residual_inputs_of_layer(p, l)]
        states.append(states[-1])
        for _ in range(steps):
            h = states[-1]
            incoming = torch.zeros(V, D, dtype=dtype)
            for e in range(T):
                sel = typ == e
                msgs = (h[src[sel]] @ w["edge_weights"].reshape(T, D, D)[e]) * wmsg[sel][:, None]
                incoming = incoming.index_add(0, tgt[sel], msgs)
            if p.get("use_edge_bias", False):
                incoming = incoming + indeg @ w["edge_biases"].reshape(T, D)
            x = torch.cat(res + [incoming], -1)
            if cell == "gru":
                ru = torch.sigmoid(torch.cat([x, h], -1) @ w["gate_kernel"] + w["gate_bias"])
                r, u = ru[:, :D], ru[:, D:]
                c = act(torch.cat([x, r * h], -1) @ w["cand_kernel"] + w["cand_bias"])
                hn = u * h + (1 - u) * c
            else:
                hn = act(torch.cat([x, h], -1) @ w["rnn_kernel"] + w["rnn_bias"])
            states[-1] = O._apply_state_dropout(hn, state_dropout, gs, None)
            gs += 1
    return states if return_all_layers else states[-1]


@pytest.mark.parametrize("regime", ["uniform", "signed"])
@pytest.mark.parametrize("keep", [1.0, 0.8])
def test_weighted_oracle_agrees_with_the_dense_oracle(regime, keep):
    import torch
    A = matrix("hub", regime)
    D, T = 8, A.shape[1]
    h0 = np.random.default_rng(1).normal(0, 1, (A.shape[0], A.shape[2], D))
    dw = O.init_dense_weights({"hidden_size": D, "use_edge_bias": True}, T, np.random.default_rng(5))
    drop = (keep, 11) if keep < 1 else None
    want = O.dense_propagation_torch(h0, A, dw, {"num_timesteps": 3, "use_edge_bias": True}, dtype=torch.float64, state_dropout=drop)
    got = weighted_propagation_torch(h0, A, [dw], params(D), state_dropout=drop)
    assert U.max_rel_err(got.numpy(), want.numpy().reshape(-1, D)) < 1e-12


@pytest.mark.parametrize("cell,act", [("GRU", "tanh"), ("RNN", "relu")])
def test_weighted_oracle_agrees_with_the_sparse_oracle_on_binary_batches(cell, act):
    import torch
    A = batch("hub")
    b, T, v, _ = A.shape
    D = 8
    p = params(D, cell=cell, act=act, residual=True)
    w = O.init_sparse_weights(p, T, np.random.default_rng(3))
    h0 = np.random.default_rng(1).normal(0, 1, (b * v, D))
    lists = []
    for t in range(T):
        gi, i, j = np.nonzero(A[:, t])
        lists.append(np.stack([gi * v + j, gi * v + i], 1))
    indeg = A.sum(-1).transpose(0, 2, 1).reshape(b * v, T)
    want = O.sparse_propagation_torch(h0, lists, indeg, w, p, return_all_layers=True, dtype=torch.float64)
    got = weighted_propagation_torch(h0, A, w, p, return_all_layers=True)
    assert len(got) == len(want) == 3
    for a, r in zip(got, want):
        assert U.max_rel_err(a.numpy(), r.numpy()) < 1e-12
