"""GPU: hidden sizes 260 .. 512 on every precision and cell, against float64.

Above hidden 256 the tensor-core precisions run the streaming wgmma kernels, and fp32, propagation attention and CudnnCompatibleGRUCell
run the per-timestep fp32 path (ggnn_fwd_step.cuh); the readout and the attention backward switch to their 16-columns-per-lane
instances.  Every case asserts its plan text on the device (tests/test_wide_hidden_cpu.py pins the same plans without a GPU) and compares
with the float64 oracle:

* forward: the final state and every ``node_states_per_layer`` entry, every bias drawn nonzero; bars max|err| / max|ref| of
  tests/test_gpu_forward_plans.py (fp32 1e-5, bf16x3 1e-4, bf16 2e-2);
* gradients: ``d h0`` and every weight and bias gradient against float64 autograd (2.5e-5 on fp32-saved plans, 2e-4 on bf16x3);
* determinism: forward bits on one engine and a fresh one; under ``ggnn_set_deterministic`` the same gradient bits across calls, engines
  and a prefilled buffer;
* the fused readout, the two plug-ins' training gradients, a two-epoch ``train()`` with a checkpoint, one engine across mixed batches.
"""
import numpy as np
import pytest

from oracle import ggnn_oracle as O
from tests import _util as U
from tests.test_backward_plans_cpu import component_graph, dense_batch, dense_params, model, sparse_batch
from tests.test_forward_plans_cpu import pad16, stream_ksteps

pytestmark = pytest.mark.gpu

BARS = {"fp32": 1e-5, "bf16x3": 1e-4, "bf16": 2e-2}
GRAD_BARS = {"fp32": 2.5e-5, "bf16x3": 2e-4}
DROP_SEED = 20261017
REN = {"rnn_kernel": "cand_kernel", "rnn_bias": "cand_bias"}


def _weights(p, T, seed=1):
    """The oracle's initialisers with the zero candidate biases drawn, so that every bias enters the forward."""
    rng = np.random.default_rng(seed)
    w = O.init_sparse_weights(p, T, rng, attention_scale=0.5)
    for lw in w:
        for k in ("cand_bias", "rnn_bias", "cand_hidden_bias"):
            if k in lw:
                lw[k] = rng.normal(0, 0.1, lw[k].shape).astype(np.float32)
    return w


def _plan_pattern(p, precision):
    """The plan family a model lands on at hidden > 256."""
    D = p["hidden_size"]
    if precision == "fp32" or p.get("use_propagation_attention") or p["graph_rnn_cell"] == "CudnnCompatibleGRUCell":
        tag = ("+attention" if p.get("use_propagation_attention") else "") + ("+cudnn-gru" if p["graph_rnn_cell"] == "CudnnCompatibleGRUCell" else "")
        return "fp32-stepwise%s (" % tag, "fp32"
    return "wgmma-%s STREAM(" % precision, precision


def _engine(p, T, w, precision, keep=1.0):
    from gated_graph_neural_network_samples_b200.engine import PropagationEngine
    eng = PropagationEngine(p, T, precision=precision)
    eng.set_weights(U.to_cuda_weights(w))
    if keep < 1.0:
        eng.set_state_dropout(keep, DROP_SEED)
    return eng


def _forward_states(eng, h0):
    import torch
    L = eng.L
    th0 = torch.from_numpy(np.ascontiguousarray(h0, np.float32)).cuda()
    out = eng.forward(th0)
    eng.sync_check()
    states = [eng.layer_state(l).cpu().numpy() for l in range(L + 1)]
    np.testing.assert_array_equal(states[L], out.cpu().numpy())
    return states


def _reference_states(p, adj, indeg, h0, w, keep=1.0):
    import torch
    if keep < 1.0:
        return [s.numpy() for s in O.sparse_propagation_torch(h0, adj, indeg, w, p, dtype=torch.float64, return_all_layers=True,
                                                              state_dropout=(keep, DROP_SEED))]
    return O.sparse_propagation_np(h0, adj, indeg, w, p, dtype=np.float64, return_all_layers=True)


def _compare_states(tag, bar, got, ref):
    errs = [U.max_rel_err(g, r) if r.size else 0.0 for g, r in zip(got, ref)]
    print("\nWIDEERR %-48s %.3e" % (tag, max(errs)))
    for l, e in enumerate(errs):
        assert e < bar, (tag, "layer %d" % l, e, bar)


def _check_forward(tag, p, T, adj, indeg, precision, keep=1.0, seed=0):
    D = p["hidden_size"]
    h0 = np.random.default_rng(300 + D + seed).normal(0, 1, (indeg.shape[0], D)).astype(np.float32)
    w = _weights(p, T)
    eng = _engine(p, T, w, precision, keep)
    eng.set_graph_sparse(adj, indeg)
    prefix, fam = _plan_pattern(p, precision)
    assert eng.plan.startswith(prefix), (tag, eng.plan)
    if fam != "fp32":
        assert "DP=%d " % pad16(D) in eng.plan
    _compare_states(tag, BARS[fam], _forward_states(eng, h0), _reference_states(p, adj, indeg, h0, w, keep))


# ---------------------------------------------------------------------------------------------------------------- forward
WIDTHS = (260, 272, 288, 320, 384, 512)


@pytest.mark.parametrize("precision", ("bf16x3", "bf16", "fp32"))
@pytest.mark.parametrize("D", WIDTHS)
def test_gru_forward_at_every_width(D, precision):
    """GRU / tanh, two layers with a residual, edge bias, avg aggregation: the streaming instances with KS 1 (DP 272), 2 (288), 4 (320,
    384, 512) and the per-timestep fp32 path."""
    adj, indeg, _ = sparse_batch("mol24", D, 4)
    _check_forward("gru-D%d-%s" % (D, precision), model("GRU", D, act="tanh", avg=True), 4, adj, indeg, precision)


CELLS = {
    "rnn-relu-bias": lambda D: model("RNN", D, act="ReLU"),
    "cudnn": lambda D: model("CudnnCompatibleGRUCell", D, act="tanh", avg=True),
    "attention": lambda D: model("GRU", D, act="tanh", attention=True),
    "attention-rnn": lambda D: model("RNN", D, act="tanh", attention=True, avg=True),
}


@pytest.mark.parametrize("precision", ("fp32", "bf16x3"))
@pytest.mark.parametrize("D", (260, 512))
@pytest.mark.parametrize("cell", sorted(CELLS))
def test_cells_forward(cell, D, precision):
    """RNN / ReLU with edge bias (streaming on bf16x3), CudnnCompatibleGRUCell and attention (the fp32 path at every precision)."""
    adj, indeg, _ = sparse_batch("mol24", D, 4)
    _check_forward("%s-D%d-%s" % (cell, D, precision), CELLS[cell](D), 4, adj, indeg, precision)


SHAPES = {   # name: (params at hidden D, T, batch, keep)
    "T1": (lambda D: model("GRU", D, act="tanh", avg=True), 1, "comp", 1.0),
    "T32": (lambda D: model("RNN", D, act="tanh", avg=True), 32, "comp", 1.0),
    "res4-self": (lambda D: model("GRU", D, layer_timesteps=(1, 1, 1, 2), residual_connections={"3": [0, 1, 2, 3]}, act="tanh", avg=True),
                  4, "mol24", 1.0),
    "zero-step": (lambda D: model("GRU", D, layer_timesteps=(2, 0, 1), residual_connections={"2": [1, 2]}, act="tanh"), 4, "mol24", 1.0),
    "dropout-gru": (lambda D: model("GRU", D, act="tanh", avg=True), 4, "mol24", 0.8),
    "dropout-rnn": (lambda D: model("RNN", D, act="tanh"), 4, "mol24", 0.8),
    "isolated-avg-cudnn": (lambda D: model("CudnnCompatibleGRUCell", D, act="tanh", avg=True), 3, "comp", 1.0),
}


@pytest.mark.parametrize("precision", ("fp32", "bf16x3"))
@pytest.mark.parametrize("shape", sorted(SHAPES))
def test_shapes_at_512(shape, precision):
    """T = 1 and 32, four residual inputs into one layer (one of them the layer's own input), a zero-step layer read through a residual,
    state dropout 0.8, and a batch with isolated nodes under avg aggregation."""
    make, T, batch, keep = SHAPES[shape]
    adj, indeg, _ = sparse_batch(batch, 512, T)
    if batch == "comp":
        assert np.sum(indeg.sum(1) == 0) >= 2
    _check_forward("%s-D512-%s" % (shape, precision), make(512), T, adj, indeg, precision, keep)


@pytest.mark.parametrize("precision", ("fp32", "bf16x3"))
def test_a_10k_node_component(precision):
    """One connected component of 10 000 nodes: no tile or component logic on either plan."""
    rng = np.random.default_rng(7)
    V = 10000
    chain = np.stack([np.arange(V - 1), np.arange(1, V)], 1)
    extra = rng.integers(0, V, (6000, 2))
    adj = [np.concatenate([chain, chain[:, ::-1]]).astype(np.int32), np.concatenate([extra, extra[:, ::-1]]).astype(np.int32)]
    indeg = np.zeros((V, 2), np.float32)
    for t, a in enumerate(adj):
        np.add.at(indeg[:, t], a[:, 1], 1.0)
    _check_forward("10k-D512-%s" % precision, model("GRU", 512, act="tanh", avg=True), 2, adj, indeg, precision)


@pytest.mark.parametrize("precision", ("fp32", "bf16x3"))
def test_an_empty_batch(precision):
    import torch
    p = model("GRU", 512, act="tanh")
    w = _weights(p, 4)
    eng = _engine(p, 4, w, precision)
    eng.set_save_for_backward(True)
    eng.set_graph_sparse([np.zeros((0, 2), np.int32)] * 4, np.zeros((0, 4), np.float32))
    assert eng.plan.startswith(_plan_pattern(p, precision)[0]), eng.plan
    out = eng.forward(torch.zeros(0, 512, device="cuda"))
    eng.sync_check()
    assert tuple(out.shape) == (0, 512)
    grads = [{k: torch.zeros_like(v) for k, v in lw.items()} for lw in U.to_cuda_weights(w)]
    eng.backward(torch.zeros(0, 512, device="cuda"), grads, torch.zeros(0, 512, device="cuda"))
    eng.sync_check()
    assert all(not torch.any(g) for lw in grads for g in lw.values())


@pytest.mark.parametrize("precision,weighted", [("fp32", False), ("bf16x3", False), ("fp32", True)])
def test_dense_matrices(precision, weighted):
    """A binary [b, T, v, v] adjacency on both families, a weighted one on the fp32 path (slot weights in the gather)."""
    import torch
    D = 512
    A, h0 = dense_batch(D, weighted)
    b, v, _ = h0.shape
    dw = O.init_dense_weights({"hidden_size": D}, 4, np.random.default_rng(5))
    dw["cand_bias"] = np.random.default_rng(6).normal(0, 0.1, D).astype(np.float32)
    ref = O.dense_propagation_loops(h0, A, dw, {"num_timesteps": 3, "use_edge_bias": True}, dtype=np.float64)
    p = dense_params(D)
    eng = _engine(p, 4, [dict(dw, edge_biases=dw["edge_biases"].reshape(4, D))], precision)
    eng.set_graph_dense(A)
    fam = "fp32-stepwise (" if precision == "fp32" else "wgmma-bf16x3 STREAM("
    assert eng.plan.startswith(fam) and eng.plan.endswith("[weighted dense adjacency -> weighted CSR]" if weighted else "[binary dense adjacency -> CSR]"), eng.plan
    out = eng.forward(torch.from_numpy(h0.reshape(b * v, D)).cuda())
    eng.sync_check()
    _compare_states("dense-%s-%s" % ("weighted" if weighted else "binary", precision), BARS[precision], [out.cpu().numpy()], [ref.reshape(b * v, D)])


# ---------------------------------------------------------------------------------------------------------------- gradients
def _autograd(p, T, w, adj, indeg, h0, g_out, keep=1.0):
    import torch
    tw = [{k: torch.tensor(v, dtype=torch.float64, requires_grad=True) for k, v in lw.items()} for lw in w]
    th0 = torch.tensor(h0, dtype=torch.float64, requires_grad=True)
    out = O.sparse_propagation_torch(th0, adj, indeg, tw, p, dtype=torch.float64, state_dropout=(keep, DROP_SEED) if keep < 1.0 else None)
    (out * torch.tensor(g_out, dtype=torch.float64)).sum().backward()
    zero_if_none = lambda v: np.zeros(v.shape) if v.grad is None else v.grad.numpy()
    return out.detach().numpy(), th0.grad.numpy(), [{REN.get(k, k): zero_if_none(v) for k, v in lw.items()} for lw in tw]


class _Trained:
    """An engine after a forward with save_for_backward; ``backward(into)`` runs ggnn_backward and returns (d h0, gradients) as NumPy."""

    def __init__(self, p, T, batch, precision, keep=1.0, det=False):
        import torch
        D = p["hidden_size"]
        self.adj, self.indeg, self.h0 = sparse_batch(batch, D, T)
        self.w = _weights(p, T)
        self.eng = _engine(p, T, self.w, precision, keep)
        self.eng.set_deterministic(det)
        self.eng.set_save_for_backward(True)
        self.eng.set_graph_sparse(self.adj, self.indeg)
        self.th0 = torch.from_numpy(self.h0).cuda()
        self.out = self.eng.forward(self.th0)
        self.g_out = np.random.default_rng(5).normal(size=self.h0.shape).astype(np.float32)
        self.dev_w = U.to_cuda_weights(self.w)

    def backward(self, into=None):
        import torch
        grads = [{k: torch.zeros_like(v) for k, v in lw.items()} for lw in self.dev_w] if into is None else into
        dh0 = torch.zeros_like(self.th0)
        self.eng.backward(torch.from_numpy(self.g_out).cuda(), grads, dh0)
        self.eng.sync_check()
        return dh0.cpu().numpy(), [{k: v.cpu().numpy() for k, v in lw.items()} for lw in grads]


GRAD_CASES = {   # name: (params at hidden D, T, batch, keep)
    "gru": (lambda D: model("GRU", D, act="tanh", avg=True), 4, "mol24", 1.0),
    "rnn": (lambda D: model("RNN", D, act="tanh"), 4, "mol24", 1.0),
    "cudnn": (lambda D: model("CudnnCompatibleGRUCell", D, act="tanh", avg=True), 4, "mol24", 1.0),
    "attention": (lambda D: model("GRU", D, act="tanh", attention=True, avg=True), 4, "mol24", 1.0),
    "res4-dropout": (lambda D: model("GRU", D, layer_timesteps=(1, 1, 1, 2), residual_connections={"3": [0, 1, 2, 3]}, act="tanh", avg=True),
                     4, "mol24", 0.8),
    "T32": (lambda D: model("RNN", D, act="tanh", avg=True), 32, "comp", 1.0),
}


@pytest.mark.parametrize("precision", ("fp32", "bf16x3"))
@pytest.mark.parametrize("D", (260, 512))
@pytest.mark.parametrize("name", sorted(GRAD_CASES))
def test_gradients_against_float64_autograd(name, D, precision):
    """d h0 and every weight and bias gradient, including edge_type_attention_weights and cand_hidden_bias, on the streaming and the
    per-timestep fp32 plans."""
    make, T, batch, keep = GRAD_CASES[name]
    p = make(D)
    prefix, fam = _plan_pattern(p, precision)
    t = _Trained(p, T, batch, precision, keep)
    assert t.eng.plan.startswith(prefix), t.eng.plan
    dh0, gw = t.backward()
    out, rdh0, rgw = _autograd(p, T, t.w, t.adj, t.indeg, t.h0, t.g_out, keep)
    pairs = [("forward", t.out.cpu().numpy(), out), ("d h0", dh0, rdh0)]
    pairs += [("layer %d %s" % (l, k), a[k], r[k]) for l, (a, r) in enumerate(zip(gw, rgw)) for k in sorted(r)]
    errs = [(U.max_rel_err(g, r) if np.any(r) else float(np.max(np.abs(g))), n) for n, g, r in pairs]
    print("\nWIDEGRAD %-36s worst %.2e on %s" % ("%s-D%d-%s" % (name, D, precision), *max(errs[1:])))
    for e, n in errs:
        assert e < GRAD_BARS[fam], (name, D, precision, n, e)


# ---------------------------------------------------------------------------------------------------------------- determinism
@pytest.mark.parametrize("precision", ("fp32", "bf16x3"))
@pytest.mark.parametrize("name", ("gru", "attention", "cudnn"))
def test_forward_bits_repeat(name, precision):
    p = GRAD_CASES[name][0](512)
    adj, indeg, h0 = sparse_batch("mol24", 512, 4)
    w = _weights(p, 4)
    runs = []
    for fresh in (False, False, True):
        if fresh or not runs:
            eng = _engine(p, 4, w, precision)
            eng.set_graph_sparse(adj, indeg)
        runs.append(_forward_states(eng, h0))
    for other in runs[1:]:
        for a, b in zip(runs[0], other):
            np.testing.assert_array_equal(a, b)


@pytest.mark.parametrize("precision", ("fp32", "bf16x3"))
@pytest.mark.parametrize("name", ("gru", "attention", "cudnn", "res4-dropout"))
def test_deterministic_gradients_repeat(name, precision):
    """Under ggnn_set_deterministic: the same gradient bits on two calls, on a fresh engine, and prefill + G in a prefilled buffer."""
    import torch
    make, T, batch, keep = GRAD_CASES[name]
    a = _Trained(make(512), T, batch, precision, keep, det=True)
    dh0, g1 = a.backward()
    _, g2 = a.backward()
    b = _Trained(make(512), T, batch, precision, keep, det=True)
    dh0b, g3 = b.backward()
    np.testing.assert_array_equal(dh0, dh0b)
    prefill = [{k: torch.full_like(v, 0.375) for k, v in lw.items()} for lw in a.dev_w]
    _, g4 = a.backward(into=prefill)
    for l in range(len(g1)):
        for k in g1[l]:
            np.testing.assert_array_equal(g1[l][k], g2[l][k], err_msg="layer %d %s" % (l, k))
            np.testing.assert_array_equal(g1[l][k], g3[l][k], err_msg="layer %d %s" % (l, k))
            np.testing.assert_array_equal(g4[l][k], np.float32(0.375) + g1[l][k], err_msg="layer %d %s" % (l, k))


# ---------------------------------------------------------------------------------------------------------------- readout
@pytest.mark.parametrize("det", (False, True))
@pytest.mark.parametrize("layout", ("grouped", "shuffled", "masked"))
@pytest.mark.parametrize("D", (260, 512))
def test_readout(D, layout, det):
    """The fused readout forward and its five gradients; the deterministic mode runs the ordered backward."""
    from tests.test_gpu_readout import _case, _engine as ro_engine, _ref, _run
    if layout == "masked":
        b, v = 9, 16
        last_h, h0, w, Gw = _case(b * v, D, b, 5 + D)
        mask = (np.random.default_rng(6).random((b, v)) < 0.7).astype(np.float32)
        eng = ro_engine(D)
        eng.readout_set_graphs(b, nodes_per_graph=v, node_mask=mask)
        ref = _ref(last_h.reshape(b, v, D), h0.reshape(b, v, D), w, Gw, node_mask=mask)
        ref = (ref[0], ref[1].reshape(b * v, D), ref[2])
    else:
        Gn = 37
        sizes = np.random.default_rng(3 + D).integers(1, 30, Gn)
        sizes[5] = 0
        gnl = np.repeat(np.arange(Gn, dtype=np.int32), sizes)
        if layout == "shuffled":
            gnl = np.random.default_rng(4 + D).permutation(gnl)
        last_h, h0, w, Gw = _case(gnl.shape[0], D, Gn, 11 + D)
        eng = ro_engine(D)
        eng.readout_set_graphs(Gn, graph_nodes_list=gnl)
        ref = _ref(last_h, h0, w, Gw, graph_nodes_list=gnl, num_graphs=Gn)
    import torch
    was = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(det)   # the readout's autograd nodes set the engine's mode from it
    try:
        out, dh, dw = _run(eng, last_h, h0, w, Gw)
        again = _run(eng, last_h, h0, w, Gw) if det else None
    finally:
        torch.use_deterministic_algorithms(was)
    errs = [("forward", U.max_rel_err(out, ref[0])), ("d h_last", U.max_rel_err(dh, ref[1]))]
    errs += [("d " + k, U.max_rel_err(dw[k], ref[2][k])) for k in sorted(ref[2])]
    print("\nWIDEERR readout-D%d-%s%s %.3e" % (D, layout, "-det" if det else "", max(e for _, e in errs)))
    for n, e in errs:
        assert e < BARS["fp32"], (D, layout, det, n, e)
    if det:
        out2, dh2, dw2 = again
        np.testing.assert_array_equal(out, out2)
        np.testing.assert_array_equal(dh, dh2)
        for k in dw:
            np.testing.assert_array_equal(dw[k], dw2[k])


# ---------------------------------------------------------------------------------------------------------------- plug-ins
@pytest.mark.parametrize("hidden,precision", [(512, "fp32"), (512, "bf16x3"), (510, "fp32"), (510, "bf16x3")])
def test_sparse_plugin_training_gradients(tmp_path, monkeypatch, hidden, precision):
    """forward_batch + loss.backward() of SparseGGNNChemModel against float64 autograd of the same model, its dropout draws replayed;
    at 510 the plug-in pads to 512 at the engine boundary."""
    from tests.test_gpu_chem_ggnn_gradients import SPARSE_TRAINING, _check, _sparse_model, _training_feed, _two_task_molecules
    m = _sparse_model(tmp_path, precision, _two_task_molecules(64, seed=1), **dict(SPARSE_TRAINING, hidden_size=hidden, graph_rnn_activation="tanh"))
    assert m.engine.D == 512
    plan = r"^fp32-stepwise " if precision == "fp32" else r"^wgmma-bf16x3 STREAM\("
    _check("sparse wide %d %s" % (hidden, precision), m, _training_feed(m), monkeypatch, plan, precision)


@pytest.mark.parametrize("hidden,precision", [(512, "fp32"), (512, "bf16x3"), (510, "fp32")])
def test_dense_plugin_training_gradients(tmp_path, monkeypatch, hidden, precision):
    from tests.test_gpu_chem_ggnn_gradients import DENSE_TRAINING, _check, _dense_model, _training_feed, _two_task_molecules
    m = _dense_model(tmp_path, precision, _two_task_molecules(64, seed=2), **dict(DENSE_TRAINING, hidden_size=hidden))
    assert m.engine.D == 512
    plan = r"^fp32-stepwise " if precision == "fp32" else r"^wgmma-bf16x3 STREAM\("
    _check("dense wide %d %s" % (hidden, precision), m, _training_feed(m), monkeypatch, plan, precision)


@pytest.mark.parametrize("precision", ("fp32", "bf16x3"))
def test_two_epoch_train_saves_and_restores(tmp_path, precision):
    import pickle
    from gated_graph_neural_network_samples_b200 import synthetic
    from gated_graph_neural_network_samples_b200.chem_sparse import SparseGGNNChemModel
    mols = synthetic.make_molecules(40, seed=5)
    cfg = {"hidden_size": 512, "batch_size": 400, "layer_timesteps": [2, 1], "residual_connections": {"1": [0]}, "use_edge_bias": True,
           "learning_rate": 0.001, "num_epochs": 2}
    args = lambda: {"--log_dir": str(tmp_path), "--precision": precision, "--train_data": mols[:32], "--valid_data": mols[32:], "--config": dict(cfg)}
    a = SparseGGNNChemModel(args())
    a.train()
    saved = pickle.load(open(a.best_model_file, "rb"))
    assert "graph_model/gnn_layer_0/gnn_edge_weights_0/Adam_1:0" in saved["weights"]
    b = SparseGGNNChemModel(args())
    b.restore_progress(a.best_model_file)
    names = dict(b.trainable_variables())
    for n, v in saved["weights"].items():
        if n in names:
            np.testing.assert_array_equal(names[n].detach().cpu().numpy(), v, err_msg=n)
    assert np.isfinite(b.run_epoch("valid", b.valid_data, False)[0])


# ---------------------------------------------------------------------------------------------------------------- engine lifetime
def test_one_engine_across_mixed_512_wide_batches():
    """One engine per family alternates large, small and empty batches at hidden 512; every forward against float64."""
    p = model("GRU", 512, act="tanh", avg=True)
    w = _weights(p, 4)
    big = component_graph(4, V_target=2000, seed=9)
    small = sparse_batch("mol24", 512, 4)[:2]
    empty = ([np.zeros((0, 2), np.int32)] * 4, np.zeros((0, 4), np.float32))
    for precision in ("bf16x3", "fp32"):
        prefix, fam = _plan_pattern(p, precision)
        eng = _engine(p, 4, w, precision)
        for i, (adj, indeg) in enumerate([big, small, empty, big, small]):
            eng.set_graph_sparse(adj, indeg)
            assert eng.plan.startswith(prefix), eng.plan
            h0 = np.random.default_rng(i).normal(0, 1, (indeg.shape[0], 512)).astype(np.float32)
            got = _forward_states(eng, h0)
            if indeg.shape[0]:
                _compare_states("lifetime-%d-%s" % (i, precision), BARS[fam], got, _reference_states(p, adj, indeg, h0, w))
