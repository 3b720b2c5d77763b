"""GPU: every compiled forward kernel instance and every accepted hidden size against the float64 oracle.

The cases and the instance each one claims live in tests/test_forward_plans_cpu.py, which pins them without a GPU and checks that
together they launch every instance the dispatch code compiles.  Here each case runs on the device, asserts the instance its plan text
names, and compares the final state and every ``layer_state(l)`` with the float64 oracle:

* GGNN: ``sparse_propagation_np`` (``sparse_propagation_torch`` with the engine's counter-based mask for state dropout); the dense model:
  ``dense_propagation_loops``; the GCN: ``gcn_propagation_loops``; the readout: ``gated_regression_torch`` under float64 autograd.
* Every bias is drawn nonzero (the initialisers leave the candidate biases at 0), so a kernel that drops one fails.
* Bars, as max|err| / max|ref| per state: ``BARS`` below (fp32 1e-5, bf16x3 1e-4, bf16 2e-2).
"""
import numpy as np
import pytest

from oracle import ggnn_oracle as O
from tests import _util as U
from tests import gcn_oracle as G
from tests.test_forward_plans_cpu import (CASES, FFMA, GCN, GCN_LAYERS, HIDDEN_SIZES, STREAM, SWEEP, TILE, dense_batch, gcn_graph, graph,
                                          h0_for, instance_of_plan)

pytestmark = pytest.mark.gpu

# Worst max|err| / max|ref| over this file's cases, measured on an H100 80GB HBM3 at a 700 W power limit:
#   fp32 1.5e-6 (FFMA, hidden 232), bf16x3 1.3e-5 (GCN hidden 4; GGNN tile kernel 1.3e-5), bf16 7.2e-3 (GCN NH 24 LOCAL; GGNN 4.1e-3).
# fp32 is held to 10x DESIGN §5's ~1e-6, bf16x3 to the north-star 1e-4, bf16 (one bf16 product per operand) to 2.8x its worst case.
BARS = {"fp32": 1e-5, "bf16x3": 1e-4, "bf16": 2e-2}
DROP_SEED = 20261015


def _weights(p, T, seed=1):
    """The oracle's initialisers with the zero candidate biases drawn, so that every bias enters the forward."""
    rng = np.random.default_rng(seed)
    w = O.init_sparse_weights(p, T, rng, attention_scale=0.5)
    for lw in w:
        for k in ("cand_bias", "rnn_bias"):
            if k in lw:
                lw[k] = rng.normal(0, 0.1, lw[k].shape).astype(np.float32)
    return w


def _compare(c, got_states, ref_states):
    """Every node_states_per_layer entry at the case's bar; prints the worst."""
    bar = BARS[c.precision]
    errs = [U.max_rel_err(g, r) for g, r in zip(got_states, ref_states)]
    worst = max(errs[1:])
    print("\nFWDERR %-8s %-7s %-40s %.3e" % (c.instance[0], c.precision, c.name, worst))
    for l, e in enumerate(errs):
        assert e < bar, (c.name, "layer %d" % l, e, bar)


def _set_env(monkeypatch, env):
    for k, v in env.items():
        monkeypatch.setenv(k, v)


def _check_plan(c, plan):
    assert instance_of_plan(plan, c.env) == c.instance, (c.name, c.instance, plan)


def _run_ggnn(c, monkeypatch):
    import torch
    from gated_graph_neural_network_samples_b200.engine import PropagationEngine
    _set_env(monkeypatch, c.env)
    L = len(c.params["layer_timesteps"])
    if c.kind == "dense":
        A, h0 = dense_batch(c.D, True)
        b, v, D = h0.shape
        dw = O.init_dense_weights({"hidden_size": D}, c.T, np.random.default_rng(5))
        dw["cand_bias"] = np.random.default_rng(6).normal(0, 0.1, D).astype(np.float32)
        ref = O.dense_propagation_loops(h0, A, dw, {"num_timesteps": c.params["layer_timesteps"][0], "use_edge_bias": True}, dtype=np.float64)
        refs = [h0.reshape(b * v, D), ref.reshape(b * v, D)]
        w = [dict(dw, edge_biases=dw["edge_biases"].reshape(c.T, D))]
        h0 = h0.reshape(b * v, D)
    else:
        adj, indeg = graph(c.batch, c.T)
        h0 = h0_for(indeg.shape[0], c.D)
        w = _weights(c.params, c.T)
        if c.keep < 1.0:
            refs = [s.numpy() for s in O.sparse_propagation_torch(h0, adj, indeg, w, c.params, dtype=torch.float64, return_all_layers=True,
                                                                  state_dropout=(c.keep, DROP_SEED))]
        else:
            refs = O.sparse_propagation_np(h0, adj, indeg, w, c.params, dtype=np.float64, return_all_layers=True)
    eng = PropagationEngine(c.params, c.T, precision=c.precision)
    eng.set_weights(U.to_cuda_weights(w))
    if c.keep < 1.0:
        eng.set_state_dropout(c.keep, DROP_SEED)
    if c.kind == "dense":
        eng.set_graph_dense(A)
    else:
        eng.set_graph_sparse(adj, indeg)
    _check_plan(c, eng.plan)
    th0 = torch.from_numpy(h0).cuda()
    out = eng.forward(th0)
    eng.sync_check()
    states = [eng.layer_state(l).cpu().numpy() for l in range(L + 1)]
    np.testing.assert_array_equal(states[L], out.cpu().numpy())
    np.testing.assert_array_equal(states[0], h0)
    _compare(c, states, refs)


@pytest.mark.parametrize("case", [c.name for c in SWEEP])
def test_hidden_size_sweep(case, monkeypatch):
    """Every hidden size 4..256: bf16x3 on its default plan, fp32 on both tile variants.  Two layers with a residual, edge bias, avg
    aggregation; GRU / tanh and RNN / ReLU alternate with the hidden size."""
    _run_ggnn(CASES[case], monkeypatch)


@pytest.mark.parametrize("case", [c.name for c in TILE])
def test_tile_wgmma_instances(case, monkeypatch):
    """The tile-local wgmma kernel at every NH: compact 64-row and 128-row LOCAL tiles, GLOBAL, bf16 LOCAL and GLOBAL, T = 17 / 32 (no
    shared-memory CSR cache; type 31 sets the tile mask's top bit), a tile with more than 4096 messages, state dropout, and a weighted
    dense matrix (weighted CSR)."""
    _run_ggnn(CASES[case], monkeypatch)


@pytest.mark.parametrize("case", [c.name for c in STREAM])
def test_streaming_instances(case, monkeypatch):
    """Every (X3, KS) streaming instance with GRU and RNN at column tails (DP 144 / 160 / 192), T = 32, dropout, forced streaming at DP 32
    and 48, and GGNN_TS_KSTEPS below the natural KS."""
    _run_ggnn(CASES[case], monkeypatch)


@pytest.mark.parametrize("case", [c.name for c in FFMA])
def test_ffma_instances(case, monkeypatch):
    """All twelve fp32 instances (variant x nb1 x LOCAL / GLOBAL) with GRU, RNN / ReLU, CudnnCompatibleGRUCell and attention."""
    _run_ggnn(CASES[case], monkeypatch)


def _gcn_reference(h0, lst, w, ks, bs, masks, keep):
    """node_states_per_layer of the GCN from the list-order loops: layer l < L is relu(prefix) * mask / keep, layer L the loops' result."""
    refs = [np.asarray(h0, np.float64)]
    for l in range(1, GCN_LAYERS + 1):
        pre = G.gcn_propagation_loops(h0, lst, w, ks[:l], bs[:l], masks, keep)
        if l < GCN_LAYERS:
            pre = np.maximum(pre, 0.0)
            if masks is not None:
                pre = pre * masks[l - 1] / np.float64(np.float32(keep))
        refs.append(pre)
    return refs


@pytest.mark.parametrize("case", [c.name for c in GCN])
def test_gcn_instances(case, monkeypatch):
    """Every GCN wgmma instance at bf16x3 and bf16, and every hidden size on bf16x3 and fp32.  The final state without save; then every
    layer's state with save (a LOCAL launch writes intermediate layers only then)."""
    from tests.test_gpu_gcn import run
    c = CASES[case]
    _set_env(monkeypatch, c.env)
    V, lst, w = gcn_graph(c.D, c.batch)
    rng = np.random.default_rng(c.D)
    ks = [G.glorot((c.D, c.D), rng) for _ in range(GCN_LAYERS)]
    bs = [rng.normal(0, 0.2, c.D).astype(np.float32) for _ in range(GCN_LAYERS)]
    h0 = rng.normal(0, 1, (V, c.D)).astype(np.float32)
    got, eng = run(c.D, GCN_LAYERS, V, lst, w, h0, ks, bs, c.precision, keep=c.keep, seed=DROP_SEED)
    _check_plan(c, eng.plan)
    masks = [eng.state_dropout_mask(l, c.keep, DROP_SEED) for l in range(GCN_LAYERS - 1)] if c.keep < 1 else None
    refs = _gcn_reference(h0, lst, w, ks, bs, masks, c.keep)
    assert U.max_rel_err(got, refs[-1]) < BARS[c.precision], (case, U.max_rel_err(got, refs[-1]))
    _, eng = run(c.D, GCN_LAYERS, V, lst, w, h0, ks, bs, c.precision, keep=c.keep, seed=DROP_SEED, save=True)
    _compare(c, [eng.layer_state(l).cpu().numpy() for l in range(GCN_LAYERS + 1)], refs)


# ---------------------------------------------------------------------------------------------------------------- readout
def _readout_case(D, shuffled):
    from tests.test_gpu_readout import _case
    Gn = 37
    sizes = np.random.default_rng(3 + D).integers(1, 30, Gn)
    sizes[5] = 0                                               # a graph without nodes
    gnl = np.repeat(np.arange(Gn, dtype=np.int32), sizes)
    if shuffled:
        gnl = np.random.default_rng(4 + D).permutation(gnl)   # not grouped: the atomic variant
    last_h, h0, w, Gw = _case(gnl.shape[0], D, Gn, 11 + D)
    return gnl, Gn, last_h, h0, w, Gw


@pytest.mark.parametrize("D", HIDDEN_SIZES)
def test_readout_every_hidden_size(D):
    """Grouped node lists (graphs summed in node order) at every hidden size: the float4 rows and the per-lane column loop."""
    _check_readout(D, False)


@pytest.mark.parametrize("D", [4, 12, 60, 132, 252])
def test_readout_shuffled(D):
    """Shuffled node lists: the atomic variant."""
    _check_readout(D, True)


def _check_readout(D, shuffled):
    """Forward and the five gradients (d h_last, w_gate, b_gate, w_trans, b_trans) of the fused readout against float64 autograd."""
    from tests.test_gpu_readout import _engine, _ref, _run
    gnl, Gn, last_h, h0, w, Gw = _readout_case(D, shuffled)
    eng = _engine(D)
    eng.readout_set_graphs(Gn, graph_nodes_list=gnl)
    out, dh, dw = _run(eng, last_h, h0, w, Gw)
    r_out, r_dh, r_dw = _ref(last_h, h0, w, Gw, graph_nodes_list=gnl, num_graphs=Gn)
    errs = [("forward", U.max_rel_err(out, r_out)), ("d h_last", U.max_rel_err(dh, r_dh))]
    errs += [("d " + k, U.max_rel_err(dw[k], r_dw[k])) for k in sorted(r_dw)]
    print("\nFWDERR %-8s %-7s %-40s %.3e" % ("readout", "fp32", "readout-D%d%s" % (D, "-shuffled" if shuffled else ""), max(e for _, e in errs)))
    for n, e in errs:
        assert e < BARS["fp32"], (D, shuffled, n, e)
