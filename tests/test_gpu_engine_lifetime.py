"""GPU: one engine across long mixed batch sequences, against float64 and against a fresh engine, and the refusal of state left over
from an earlier batch.

Every other GPU test builds a fresh engine per case.  In training one engine serves thousands of batches in a row, and between two
batches the node and message counts, the plan, the save flag, the dropout seed and the weights may all change while the engine keeps
its graph image, state and save buffers, weight tiles, streaming images, attention buffer and readout map.  Each sequence here runs on
ONE engine (scripts and their plans: tests/test_engine_lifetime_cpu.py) and checks every step four ways:

(i)   the final state and every ``layer_state(l)`` against the float64 oracle (fp32 1e-5, bf16x3 1e-4, bf16 2e-2);
(ii)  the step's result against a fresh engine given the same batch, weights, dropout and environment: identical bits on the fp32,
      streaming and GCN kernels, within 1e-6 on the tile-local wgmma kernel (its MMA issue order is not fixed); ``d h0`` identical bits
      on every plan;
(iii) with save on, every weight, bias and ``d h0`` gradient against float64 autograd with the step's dropout mask (2e-4; the GCN 2.5e-5);
(iv)  the plan text.

The refusal tests at the end show the stale-state findings so that an engine without the checks reads only allocated memory and fails
an assertion: the second batch is smaller than the first, the second forward runs on the same graph, the new readout graph has the
same node count.
"""
import re

import numpy as np
import pytest

from gated_graph_neural_network_samples_b200.engine import GgnnError
from oracle import ggnn_oracle as O
from tests import _util as U
from tests import gcn_oracle as G
from tests import test_engine_lifetime_cpu as S
from tests.test_backward_plans_cpu import dense_params
from tests.test_gpu_backward_plans import _weights
from tests.test_gpu_forward_plans import _gcn_reference

pytestmark = pytest.mark.gpu

BARS = {"fp32": 1e-5, "bf16x3": 1e-4, "bf16": 2e-2}
GRAD_BAR = 2e-4
GCN_GRAD_BAR = 2.5e-5
TILE_LOCAL_NOISE = 1e-6
REN = {"rnn_kernel": "cand_kernel", "rnn_bias": "cand_bias"}


def _env(monkeypatch, env):
    for k in ("GGNN_FORCE_GLOBAL", "GGNN_TC_STREAM"):
        monkeypatch.delenv(k, raising=False)
    for k, v in env.items():
        monkeypatch.setenv(k, v)


def _dev(w):
    import torch
    return [{REN.get(k, k): torch.from_numpy(np.ascontiguousarray(v, np.float32)).cuda() for k, v in lw.items()} for lw in w]


def _rel(a, b):
    return U.max_rel_err(a, b) if b.size and np.any(b) else (float(np.max(np.abs(a))) if a.size else 0.0)


def _same(got, fresh, plan, tag):
    """(ii): identical bits, or within TILE_LOCAL_NOISE on the tile-local wgmma kernel."""
    if re.match(r"^wgmma-bf16x?3? (LOCAL|GLOBAL)\(", plan):
        assert _rel(got, fresh) <= TILE_LOCAL_NOISE, (tag, _rel(got, fresh))
    else:
        np.testing.assert_array_equal(got, fresh, err_msg=tag)


class Worst:
    """The worst error per check of one sequence, printed at its end."""

    def __init__(self, tag):
        self.tag, self.e = tag, {}

    def add(self, what, err):
        self.e[what] = max(self.e.get(what, 0.0), err)
        return err

    def report(self):
        print("\n[lifetime %s] worst: %s" % (self.tag, "  ".join("%s %.2e" % kv for kv in sorted(self.e.items()))))


# ---------------------------------------------------------------------------------------------------------------- the GGNN runner
class GgnnRun:
    """Runs the forward (and with save the backward) of one batch on an engine, keeping every buffer the engine points into alive."""

    def __init__(self, eng, params, T):
        self.eng, self.p, self.T = eng, params, T

    def run(self, step, dev_w, adj, indeg, h0, g_out, monkeypatch):
        import torch
        _env(monkeypatch, step.env)
        eng = self.eng
        if dev_w is not None:
            eng.set_weights(dev_w)
        eng.set_save_for_backward(step.save)
        eng.set_graph_sparse(adj, indeg)
        eng.set_state_dropout(step.keep, step.seed)
        self.h0 = torch.from_numpy(h0).cuda()
        self.out = eng.forward(self.h0)
        states = [eng.layer_state(l).cpu().numpy() for l in range(eng.L + 1)]
        res = {"plan": eng.plan, "states": states}
        if step.save:
            self.grads = [{k: torch.zeros_like(v) for k, v in lw.items()} for lw in self.dev_w_for_grads]
            self.dh0 = torch.zeros_like(self.h0)
            eng.backward(torch.from_numpy(g_out).cuda(), self.grads, self.dh0)
            res["dh0"] = self.dh0.cpu().numpy()
            res["grads"] = [{k: v.cpu().numpy() for k, v in lw.items()} for lw in self.grads]
        eng.sync_check()
        return res


def _reference(params, T, w, adj, indeg, h0, g_out, step):
    """float64: every layer state, and with save the gradients of sum(out * g_out) (zero where a weight does not reach the output)."""
    import torch
    drop = (step.keep, step.seed) if step.keep < 1.0 else None
    if not step.save:
        if drop is None:
            return {"states": O.sparse_propagation_np(h0, adj, indeg, w, params, dtype=np.float64, return_all_layers=True)}
        return {"states": [s.numpy() for s in O.sparse_propagation_torch(h0, adj, indeg, w, params, dtype=torch.float64, return_all_layers=True,
                                                                        state_dropout=drop)]}
    tw = [{k: torch.tensor(v, dtype=torch.float64, requires_grad=True) for k, v in lw.items()} for lw in w]
    th0 = torch.tensor(h0, dtype=torch.float64, requires_grad=True)
    states = O.sparse_propagation_torch(th0, adj, indeg, tw, params, dtype=torch.float64, return_all_layers=True, state_dropout=drop)
    (states[-1] * torch.tensor(g_out, dtype=torch.float64)).sum().backward()
    z = lambda v: np.zeros(v.shape) if v.grad is None else v.grad.numpy()
    return {"states": [s.detach().numpy() for s in states], "dh0": th0.grad.numpy(),
            "grads": [{REN.get(k, k): z(v) for k, v in lw.items()} for lw in tw]}


def _check_step(tag, res, ref, bar, worst):
    for l, (g, r) in enumerate(zip(res["states"], ref["states"])):
        assert g.shape == np.shape(r), (tag, l, g.shape)
        assert worst.add("oracle", _rel(g, r)) < bar, (tag, "layer %d" % l, _rel(g, r))
    if "grads" in ref:
        assert worst.add("d h0", _rel(res["dh0"], ref["dh0"])) < GRAD_BAR, (tag, "d h0", _rel(res["dh0"], ref["dh0"]))
        for l, (a, r) in enumerate(zip(res["grads"], ref["grads"])):
            for k in r:
                e = _rel(a[k], r[k]) if np.any(r[k]) else float(np.max(np.abs(a[k])))
                assert worst.add("gradient", e) < GRAD_BAR, (tag, "layer %d %s" % (l, k), e)


def _run_ggnn_script(tag, params, T, precision, steps, monkeypatch, check_grads=True):
    from gated_graph_neural_network_samples_b200.engine import PropagationEngine
    D = params["hidden_size"]
    eng = PropagationEngine(params, T, precision=precision)
    runner = GgnnRun(eng, params, T)
    worst = Worst(tag)
    weights, bound, memo = {}, None, {}
    for i, s in enumerate(steps):
        if s.weights is not None and s.weights not in weights:
            w = _weights(params, T, seed=s.weights)
            weights[s.weights] = (w, _dev(w))
        new = s.weights is not None
        if new:
            bound = s.weights
        w, dev_w = weights[bound]
        adj, indeg, h0 = S.batch(s.kind, D, T)
        g_out = np.random.default_rng(100 + i).normal(size=h0.shape).astype(np.float32)
        runner.dev_w_for_grads = dev_w
        st = "%s step %d %r" % (tag, i + 1, s)
        res = runner.run(s, dev_w if new else None, adj, indeg, h0, g_out, monkeypatch)
        if s.plan is not None:                                                                     # (iv)
            assert re.search(s.plan, res["plan"]), (st, res["plan"])
        keep_alive = (runner.h0, runner.out)
        if h0.shape[0] > 0:                                                                        # (i), (iii)
            bar = BARS["fp32" if res["plan"].startswith("fp32") else precision]
            ref_step = s if check_grads else S.Step(s.kind, None, False, s.keep, s.seed, None)
            _check_step(st, res, _reference(params, T, w, adj, indeg, h0, g_out, ref_step), bar, worst)
        else:
            assert all(x.shape == (0, D) for x in res["states"])
        fresh = GgnnRun(PropagationEngine(params, T, precision=precision), params, T)             # (ii)
        fresh.dev_w_for_grads = dev_w
        f = fresh.run(s, dev_w, adj, indeg, h0, g_out, monkeypatch)
        assert f["plan"] == res["plan"], (st, f["plan"], res["plan"])
        _same(res["states"][-1], f["states"][-1], res["plan"], st + " final vs a fresh engine")
        if s.save:
            np.testing.assert_array_equal(res["dh0"], f["dh0"], err_msg=st + " d h0 vs a fresh engine")
        key = (s.kind, bound, s.save, s.keep, s.seed)
        if key in memo:   # the same batch with the same weights bound again: the same result as the first time
            _same(res["states"][-1], memo[key], res["plan"], st + " final vs the same batch earlier in the sequence")
        memo[key] = res["states"][-1]
        del keep_alive
    worst.report()
    return worst


@pytest.mark.parametrize("precision", ["bf16x3", "fp32"])
def test_default_model_sequence(precision, monkeypatch):
    """The reference's default model with edge bias: compact LOCAL -> 128-row LOCAL -> the big component -> forced GLOBAL with the
    weights of two steps back -> empty -> one node -> a small validation batch -> the 128-row batch with its weights bound again."""
    _run_ggnn_script("default " + precision, S.DEFAULT, 4, precision, S.ggnn_script(precision), monkeypatch)


def test_default_model_sequence_bf16(monkeypatch):
    """The same plan switches on the single-bf16 kernels (forward only against float64: the gradient bars are those of bf16x3)."""
    _run_ggnn_script("default bf16", S.DEFAULT, 4, "bf16", S.ggnn_script("bf16", short=True), monkeypatch, check_grads=False)


@pytest.mark.parametrize("model", ["attention", "cudnn"])
def test_attention_and_cudnn_gru_sequences(model, monkeypatch):
    """Attention: save off at a small M, save on at a larger M (att_buf grows to [steps][M]), then back.  CudnnCompatibleGRUCell: the
    sixth saved array."""
    params, T, precision, steps = S.SCRIPTS[model]
    _run_ggnn_script(model, params, T, precision, steps, monkeypatch)


def test_cfg4_streaming_sequence_with_hub_nodes(monkeypatch):
    """Hidden 256, 8 edge types: V grows and shrinks, a hub batch (virtual rows longer than the 7 inline sources) is followed by one
    without any, then by one with fewer; save toggles."""
    params, T, precision, steps = S.SCRIPTS["cfg4"]
    _run_ggnn_script("cfg4", params, T, precision, steps, monkeypatch)


# ---------------------------------------------------------------------------------------------------------------- dense
@pytest.mark.parametrize("precision", ["fp32", "bf16x3"])
def test_dense_sequence_alternates_binary_and_weighted_matrices(precision):
    """Binary matrices (CSR) alternate with weighted ones (CSR with slot weights) on one engine, with b and v changing."""
    import torch
    from gated_graph_neural_network_samples_b200.engine import PropagationEngine
    D = 100
    eng = PropagationEngine(dense_params(D), S.DENSE_T, precision=precision)
    worst = Worst("dense " + precision)
    for i, (weighted, b, v) in enumerate(S.DENSE_SCRIPT):
        A = S.dense_matrix(weighted, b, v)
        dw = O.init_dense_weights({"hidden_size": D}, S.DENSE_T, np.random.default_rng(50 + i))
        dw["cand_bias"] = np.random.default_rng(60 + i).normal(0, 0.1, D).astype(np.float32)
        dev = _dev([dict(dw, edge_biases=dw["edge_biases"].reshape(S.DENSE_T, D))])
        h0 = np.random.default_rng(70 + i).normal(0, 1, (b, v, D)).astype(np.float32)
        g_out = np.random.default_rng(80 + i).normal(size=h0.shape).astype(np.float32)

        def run(e):
            e.set_weights(dev)
            e.set_save_for_backward(True)
            e.set_graph_dense(A)
            th0 = torch.from_numpy(h0.reshape(b * v, D)).cuda()
            out = e.forward(th0)
            grads = [{k: torch.zeros_like(x) for k, x in dev[0].items()}]
            dh0 = torch.zeros_like(th0)
            e.backward(torch.from_numpy(g_out.reshape(b * v, D)).cuda(), grads, dh0)
            e.sync_check()
            return e.plan, out.cpu().numpy().reshape(b, v, D), dh0.cpu().numpy().reshape(b, v, D), {k: x.cpu().numpy() for k, x in grads[0].items()}

        plan, out, dh0, gw = run(eng)
        tag = "dense step %d weighted=%s b=%d v=%d" % (i + 1, weighted, b, v)
        assert ("binary dense adjacency -> CSR" in plan) == (not weighted), (tag, plan)
        tw = {k: torch.tensor(x, dtype=torch.float64, requires_grad=True) for k, x in dw.items()}
        th0 = torch.tensor(h0, dtype=torch.float64, requires_grad=True)
        ref = O.dense_propagation_torch(th0, A, tw, {"num_timesteps": S.DENSE_STEPS, "use_edge_bias": True}, dtype=torch.float64)
        (ref * torch.tensor(g_out, dtype=torch.float64)).sum().backward()
        assert worst.add("oracle", _rel(out, ref.detach().numpy())) < BARS[precision], (tag, _rel(out, ref.detach().numpy()))
        assert worst.add("d h0", _rel(dh0, th0.grad.numpy())) < GRAD_BAR, tag
        for k in tw:
            assert worst.add("gradient", _rel(gw[k].reshape(tw[k].shape), tw[k].grad.numpy())) < GRAD_BAR, (tag, k)
        f_plan, f_out, f_dh0, _ = run(PropagationEngine(dense_params(D), S.DENSE_T, precision=precision))
        assert f_plan == plan
        _same(out, f_out, plan, tag + " vs a fresh engine")
        np.testing.assert_array_equal(dh0, f_dh0, err_msg=tag)
    worst.report()


# ---------------------------------------------------------------------------------------------------------------- GCN
@pytest.mark.parametrize("precision", ["bf16x3", "fp32"])
def test_gcn_sequence(precision):
    """LOCAL -> GLOBAL (a 200-node component) -> empty -> LOCAL, weights set every step, save and dropout varied; intermediate layer
    states are checked after save forwards (without save the fused LOCAL kernel keeps them on chip, and the engine refuses them)."""
    import torch
    from gated_graph_neural_network_samples_b200.engine import GCNEngine
    D, L = S.GCN_D, S.GCN_L
    eng = GCNEngine(D, L, use_bias=True, precision=precision)
    worst = Worst("gcn " + precision)
    for i, (kind, wseed, save, keep, seed, plan) in enumerate(S.GCN_SCRIPT):
        V, lst, w = S.gcn_graph(kind)
        rng = np.random.default_rng(wseed)
        ks = [G.glorot((D, D), rng) for _ in range(L)]
        bs = [rng.normal(0, 0.2, D).astype(np.float32) for _ in range(L)]
        h0 = rng.normal(0, 1, (V, D)).astype(np.float32)
        g_out = rng.normal(size=(V, D)).astype(np.float32)
        dk, db = [torch.from_numpy(k).cuda() for k in ks], [torch.from_numpy(b).cuda() for b in bs]
        tag = "gcn step %d %s save=%d keep=%g" % (i + 1, kind, save, keep)

        def run(e):
            e.set_weights(dk, db)
            e.set_save_for_backward(save)
            e.set_graph_gcn(V, lst, w)
            e.set_state_dropout(keep, seed)
            th0 = torch.from_numpy(h0).cuda()
            out = e.forward(th0)
            r = {"plan": e.plan, "out": out.cpu().numpy(), "keep": (th0, out)}
            inter = range(L + 1) if save or e.plan.startswith("gcn-fp32") or "GLOBAL" in e.plan else (0, L)
            r["states"] = {l: e.layer_state(l).cpu().numpy() for l in inter}
            if save:
                gk, gb = [torch.zeros(D, D, device="cuda") for _ in range(L)], [torch.zeros(D, device="cuda") for _ in range(L)]
                dh0 = torch.zeros_like(th0)
                e.backward(torch.from_numpy(g_out).cuda(), [{"kernel": a, "bias": b} for a, b in zip(gk, gb)], d_h0=dh0)
                r["dh0"], r["gk"], r["gb"] = dh0.cpu().numpy(), [a.cpu().numpy() for a in gk], [b.cpu().numpy() for b in gb]
            e.sync_check()
            return r

        r = run(eng)
        if plan is not None:
            assert re.search(S.GCN_PLANS[precision][plan], r["plan"]), (tag, r["plan"])
        if not save and "LOCAL" in r["plan"] and not r["plan"].startswith("gcn-fp32"):
            with pytest.raises(GgnnError, match="did not write the layers"):
                eng.layer_state(1)
        f = run(GCNEngine(D, L, use_bias=True, precision=precision))
        np.testing.assert_array_equal(r["out"], f["out"], err_msg=tag + " vs a fresh engine")
        if V == 0:
            continue
        masks = [eng.state_dropout_mask(l, keep, seed) for l in range(L - 1)] if keep < 1 else None
        th0 = torch.from_numpy(h0).double().requires_grad_()
        tk = [torch.from_numpy(k).double().requires_grad_() for k in ks]
        tb = [torch.from_numpy(b).double().requires_grad_() for b in bs]
        refs = _gcn_reference(h0, lst, w, ks, bs, masks, keep)
        for l, got in r["states"].items():
            ref_l = refs[l]
            assert worst.add("oracle", _rel(got, ref_l)) < BARS[precision], (tag, l, _rel(got, ref_l))
        if save:
            np.testing.assert_array_equal(r["dh0"], f["dh0"], err_msg=tag)
            # ReLU's derivative jumps at 0: where a pre-activation lies within the forward's rounding of 0, float64 and the engine take
            # opposite sides (tests/test_backward_plans_cpu.py, smooth_on_tensor_cores).  The reference therefore takes the engine's side:
            # relu(x) = x * [engine state > 0], the same forward wherever the two agree, and the engine's decision where they do not.
            rows, cols = torch.from_numpy(lst[:, 0]), torch.from_numpy(lst[:, 1])
            wt, out = torch.from_numpy(w).double(), th0
            for l in range(L):
                out = torch.zeros_like(out).index_add_(0, rows, wt[:, None] * out[cols]) @ tk[l] + tb[l]
                if l < L - 1:
                    out = out * torch.from_numpy((r["states"][l + 1] > 0).astype(np.float64))
                    if masks is not None:
                        out = out * torch.from_numpy(masks[l].astype(np.float64)) / float(np.float32(keep))
            out.backward(torch.from_numpy(g_out).double())
            errs = [_rel(r["dh0"], th0.grad.numpy())] + [_rel(a, t.grad.numpy()) for a, t in zip(r["gk"] + r["gb"], tk + tb)]
            assert worst.add("gradient", max(errs)) < GCN_GRAD_BAR, (tag, errs)
    worst.report()


# ---------------------------------------------------------------------------------------------------------------- entry points
def test_entry_points_and_prepared_graphs_on_one_engine():
    """set_graph_sparse + forward, forward_host, run_sparse_host, run_sparse_host_readout (loss and MAE against the torch restatement)
    and prepared graphs from a pool of two, uploaded in another order than they were prepared in, on one bf16x3 engine."""
    import torch
    from gated_graph_neural_network_samples_b200.engine import PropagationEngine
    p, T, D = S.DEFAULT, 4, 100
    w = _weights(p, T, seed=9)
    eng = PropagationEngine(p, T, precision="bf16x3")
    eng.set_weights(_dev(w))
    bar = BARS["bf16x3"]
    ref = lambda adj, indeg, h0: O.sparse_propagation_np(h0, adj, indeg, w, p, dtype=np.float64)
    A, B, C = (S.batch(k, D, T) for k in ("mol40+300", "mol24", "mol1024"))
    # set_graph_sparse + forward, then forward_host on the same graph
    eng.set_graph_sparse(A[0], A[1])
    out = eng.forward(torch.from_numpy(A[2]).cuda()).cpu().numpy()
    assert U.max_rel_err(out, ref(*A)) < bar
    assert U.max_rel_err(eng.forward_host(A[2]), ref(*A)) < bar
    # two prepared graphs (B, C), built before either is uploaded, uploaded C first
    gB = eng.prepare_graph_sparse(B[0], B[1])
    gC = eng.prepare_graph_sparse(C[0], C[1])
    for g, (adj, indeg, h0) in ((gC, C), (gB, B)):
        eng.set_graph_prepared(g)
        assert U.max_rel_err(eng.forward_host(h0), ref(adj, indeg, h0)) < bar
    # the one-call entry points between them
    assert U.max_rel_err(eng.run_sparse_host(A[0], A[1], A[2]), ref(*A)) < bar
    _, b = U.molecule_batch(40, D, seed=3)
    G_, rng = 40, np.random.default_rng(2)
    tasks = [tuple(torch.from_numpy(a.astype(np.float32)).cuda() for a in (rng.normal(0, 0.2, 2 * D), rng.normal(0, 0.1, 1),
                                                                           rng.normal(0, 0.2, D), rng.normal(0, 0.1, 1))) for _ in range(2)]
    tv = rng.normal(size=(2, G_)).astype(np.float32)
    tm = (rng.random((2, G_)) < 0.7).astype(np.float32)
    loss, acc = eng.run_sparse_host_readout(b["adjacency_lists"], b["num_incoming_edges_per_type"], b["initial_node_representation"],
                                            b["graph_nodes_list"], G_, tasks, tv, tm)
    final = torch.from_numpy(ref(b["adjacency_lists"], b["num_incoming_edges_per_type"], b["initial_node_representation"]))
    h0t = torch.from_numpy(b["initial_node_representation"]).double()
    gnl = torch.from_numpy(np.asarray(b["graph_nodes_list"])).long()
    for t, (wg, bg, wt, bt) in enumerate(tasks):
        wg, bg, wt, bt = (x.double().cpu() for x in (wg, bg, wt, bt))
        gated = torch.sigmoid(torch.cat([final, h0t], -1) @ wg.view(-1, 1) + bg) * (final @ wt.view(-1, 1) + bt)
        pred = torch.zeros(G_, 1, dtype=torch.float64).index_add_(0, gnl, gated).squeeze(-1)
        diff = (pred - torch.from_numpy(tv[t]).double()) * torch.from_numpy(tm[t]).double()
        num = float(tm[t].sum()) + 1e-7
        assert abs(loss[t] - float((0.5 * diff * diff).sum()) / num) < 1e-4 * max(1.0, abs(float(loss[t])))
        assert abs(acc[t] - float(diff.abs().sum()) / num) < 1e-4 * max(1.0, abs(float(acc[t])))
    # the pool reused: C rebuilt into B's prepared graph, B into C's, uploaded B first
    gB2 = eng.prepare_graph_sparse(C[0], C[1], reuse=gB)
    gC2 = eng.prepare_graph_sparse(B[0], B[1], reuse=gC)
    for g, (adj, indeg, h0) in ((gC2, B), (gB2, C)):
        eng.set_graph_prepared(g)
        th0 = torch.from_numpy(h0).cuda()   # layer 0 is the caller's h0: kept alive while its states are read
        got = eng.forward(th0)
        assert U.max_rel_err(got.cpu().numpy(), ref(adj, indeg, h0)) < bar
        for l in (0, 2):
            assert eng.layer_state(l).shape == (h0.shape[0], D)
        np.testing.assert_array_equal(eng.layer_state(0).cpu().numpy(), h0)
    eng.sync_check()


# ---------------------------------------------------------------------------------------------------------------- operation order
def _trained(precision="bf16x3", keep=0.8, seed=5):
    import torch
    from gated_graph_neural_network_samples_b200.engine import PropagationEngine
    p, T, D = S.DEFAULT, 4, 100
    w = _weights(p, T, seed=3)
    dev = _dev(w)
    adj, indeg, h0 = S.batch("mol24", D, T)
    eng = PropagationEngine(p, T, precision=precision)
    eng.set_weights(dev)
    eng.set_save_for_backward(True)
    eng.set_graph_sparse(adj, indeg)
    eng.set_state_dropout(keep, seed)
    th0 = torch.from_numpy(h0).cuda()
    out = eng.forward(th0)
    g_out = np.random.default_rng(4).normal(size=h0.shape).astype(np.float32)

    def backward():
        grads = [{k: torch.zeros_like(v) for k, v in lw.items()} for lw in dev]
        dh0 = torch.zeros_like(th0)
        eng.backward(torch.from_numpy(g_out).cuda(), grads, dh0)
        eng.sync_check()
        return dh0.cpu().numpy(), [{k: v.cpu().numpy() for k, v in lw.items()} for lw in grads]

    return eng, backward, (p, T, w, adj, indeg, h0, g_out, (th0, out, dev))


def test_backward_uses_the_forwards_dropout_mask_after_set_state_dropout_changes():
    eng, backward, (p, T, w, adj, indeg, h0, g_out, _) = _trained(keep=0.8, seed=5)
    eng.set_state_dropout(0.5, 99)   # for the next forward; the saved forward ran at (0.8, 5)
    dh0, gw = backward()
    ref = _reference(p, T, w, adj, indeg, h0, g_out, S.Step("mol24", 0, True, 0.8, 5, None))
    _check_step("dropout changed before backward", {"states": [], "dh0": dh0, "grads": gw}, ref, 0, Worst("order"))


def test_two_backward_calls_of_one_forward_agree():
    """What reduce_gradients does once per task: d h0 identical bits, weight gradients within the backward bar (atomic sums)."""
    _, backward, _ = _trained(keep=0.9, seed=6)
    a_dh0, a = backward()
    b_dh0, b = backward()
    np.testing.assert_array_equal(a_dh0, b_dh0)
    for x, y in zip(a, b):
        for k in x:
            assert _rel(y[k], x[k]) < GRAD_BAR, k


# ---------------------------------------------------------------------------------------------------------------- refusals
def test_layer_state_is_refused_after_a_new_graph_until_a_forward_ran_on_it():
    """Batch B (5 molecules) after batch A (24): until a forward ran on B, layer_state of any layer refuses (it would return A's h0
    pointer, or offsets computed with B's V into A's states).  A failed upload refuses too.  After B's forward every layer is B's."""
    import torch
    from gated_graph_neural_network_samples_b200.engine import PropagationEngine
    p, T, D = S.DEFAULT, 4, 100
    w = _weights(p, T, seed=2)
    eng = PropagationEngine(p, T, precision="bf16x3")
    eng.set_weights(_dev(w))
    A, B = S.batch("mol24", D, T), S.batch("mol5", D, T)
    eng.set_graph_sparse(A[0], A[1])
    hA = torch.from_numpy(A[2]).cuda()
    outA = eng.forward(hA)
    eng.layer_state(2)
    eng.set_graph_sparse(B[0], B[1])
    for l in range(eng.L + 1):
        with pytest.raises(GgnnError, match="no forward has run on the current graph"):
            eng.layer_state(l)
    hB = torch.from_numpy(B[2]).cuda()
    outB = eng.forward(hB)
    ref = O.sparse_propagation_np(B[2], B[0], B[1], w, p, dtype=np.float64, return_all_layers=True)
    for l in range(eng.L + 1):
        assert U.max_rel_err(eng.layer_state(l).cpu().numpy(), ref[l]) < BARS["bf16x3"], l
    bad = [a.copy() for a in A[0]]
    bad[0][0, 0] = 10 ** 6                                                     # an out-of-range source: the upload fails
    with pytest.raises(GgnnError):
        eng.set_graph_sparse(bad, A[1])
    with pytest.raises(GgnnError, match="no forward has run on the current graph"):
        eng.layer_state(0)
    del outA, outB


def test_gcn_layer_state_between_layers_is_refused_after_a_fused_forward_without_save():
    """The LOCAL GCN wgmma kernel without save_for_backward keeps the layers between h0 and the result on chip: layer_state refuses
    them (it returned whatever an earlier save forward left in the state buffer); layers 0 and L stay available."""
    import torch
    from gated_graph_neural_network_samples_b200.engine import GCNEngine
    D, L = S.GCN_D, S.GCN_L
    V, lst, w = S.gcn_graph("small")
    rng = np.random.default_rng(1)
    ks = [G.glorot((D, D), rng) for _ in range(L)]
    h0 = rng.normal(0, 1, (V, D)).astype(np.float32)
    eng = GCNEngine(D, L, precision="bf16x3")
    eng.set_weights([torch.from_numpy(k).cuda() for k in ks])
    eng.set_save_for_backward(True)
    eng.set_graph_gcn(V, lst, w)
    th0 = torch.from_numpy(h0).cuda()
    eng.forward(th0)
    assert U.max_rel_err(eng.layer_state(1).cpu().numpy(), _gcn_reference(h0, lst, w, ks, [np.zeros(D, np.float32)] * L, None, 1.0)[1]) < BARS["bf16x3"]
    eng.set_save_for_backward(False)
    eng.set_graph_gcn(V, lst, w)
    th1 = torch.from_numpy(h0 * 0.5).cuda()
    out = eng.forward(th1)
    assert "LOCAL" in eng.plan
    for l in range(1, L):
        with pytest.raises(GgnnError, match="did not write the layers"):
            eng.layer_state(l)
    np.testing.assert_array_equal(eng.layer_state(0).cpu().numpy(), h0 * 0.5)
    np.testing.assert_array_equal(eng.layer_state(L).cpu().numpy(), out.cpu().numpy())


def _sparse_node(eng, dev):
    from gated_graph_neural_network_samples_b200.chem_sparse import _propagation_function
    flat, layout = [], []
    for lw in dev:
        lay = {}
        for k, v in lw.items():
            lay[k] = len(flat)
            flat.append(v.clone().requires_grad_(True))
        layout.append(lay)
    return _propagation_function(), layout, flat


def test_autograd_node_refuses_a_backward_after_another_forward_on_its_engine():
    """Two forwards of the propagation node on one engine (same graph, different h0), then the first one's backward: the engine's saved
    activations are the second's, so the backward must raise instead of returning the second forward's gradients.  The second one's
    backward works, twice."""
    import torch
    from gated_graph_neural_network_samples_b200.engine import PropagationEngine
    p, T, D = S.DEFAULT, 4, 100
    adj, indeg, h0 = S.batch("mol24", D, T)
    eng = PropagationEngine(p, T, precision="bf16x3")
    eng.set_save_for_backward(True)
    eng.set_graph_sparse(adj, indeg)
    P, layout, flat = _sparse_node(eng, _dev(_weights(p, T, seed=1)))
    ha = torch.from_numpy(h0).cuda().requires_grad_(True)
    hb = torch.from_numpy(h0 * 0.5).cuda().requires_grad_(True)
    out_a = P.apply(eng, layout, ha, *flat)
    out_b = P.apply(eng, layout, hb, *flat)
    with pytest.raises(GgnnError, match="earlier forward"):
        out_a.sum().backward()
    g1 = torch.autograd.grad(out_b.sum(), [hb], retain_graph=True)[0]
    g2 = torch.autograd.grad(out_b.sum(), [hb])[0]
    np.testing.assert_array_equal(g1.cpu().numpy(), g2.cpu().numpy())


def test_gcn_autograd_node_refuses_a_backward_after_another_forward_on_its_engine():
    import torch
    from gated_graph_neural_network_samples_b200.chem_gcn import _propagation_function
    from gated_graph_neural_network_samples_b200.engine import GCNEngine
    D, L = S.GCN_D, S.GCN_L
    V, lst, w = S.gcn_graph("small")
    rng = np.random.default_rng(1)
    ks = [torch.from_numpy(G.glorot((D, D), rng)).cuda().requires_grad_(True) for _ in range(L)]
    h0 = rng.normal(0, 1, (V, D)).astype(np.float32)
    eng = GCNEngine(D, L, precision="bf16x3")
    eng.set_save_for_backward(True)
    eng.set_graph_gcn(V, lst, w)
    P = _propagation_function()
    out_a = P.apply(eng, torch.from_numpy(h0).cuda().requires_grad_(True), *ks)
    out_b = P.apply(eng, torch.from_numpy(h0 * 0.5).cuda().requires_grad_(True), *ks)
    with pytest.raises(GgnnError, match="earlier forward"):
        out_a.sum().backward()
    out_b.sum().backward()


def test_backward_after_new_weights_is_refused():
    """set_weights between a forward and its backward: the backward would combine the old activations with the new weights."""
    import torch
    from gated_graph_neural_network_samples_b200.engine import GCNEngine
    eng, backward, (p, T, w, *_rest) = _trained()
    eng.set_weights(_dev(_weights(p, T, seed=4)))
    with pytest.raises(GgnnError, match="needs a preceding ggnn_forward"):
        backward()
    D, L = S.GCN_D, S.GCN_L
    V, lst, wg = S.gcn_graph("small")
    ks = [torch.from_numpy(G.glorot((D, D), np.random.default_rng(l))).cuda() for l in range(L)]
    g = GCNEngine(D, L, precision="bf16x3")
    g.set_weights(ks)
    g.set_save_for_backward(True)
    g.set_graph_gcn(V, lst, wg)
    th0 = torch.zeros(V, D, device="cuda")
    g.forward(th0)
    g.set_weights([k * 2 for k in ks])
    with pytest.raises(GgnnError, match="needs a preceding ggnn_forward"):
        g.backward(torch.ones(V, D, device="cuda"), [{"kernel": torch.zeros(D, D, device="cuda")} for _ in range(L)])


def test_readout_map_is_dropped_by_a_new_graph():
    """readout_set_graphs belongs to one batch: after a new graph (same node count) the readout refuses until it is called again."""
    import torch
    from gated_graph_neural_network_samples_b200.engine import PropagationEngine
    p, T, D = S.DEFAULT, 4, 100
    _, b = U.molecule_batch(24, D, seed=3)
    adj, indeg, h0 = b["adjacency_lists"], b["num_incoming_edges_per_type"], b["initial_node_representation"]
    eng = PropagationEngine(p, T, precision="bf16x3")
    eng.set_weights(_dev(_weights(p, T, seed=1)))
    eng.set_graph_sparse(adj, indeg)
    th0 = torch.from_numpy(h0).cuda()
    out = eng.forward(th0)
    eng.readout_set_graphs(24, graph_nodes_list=b["graph_nodes_list"])
    ro = [torch.full((2 * D,), 0.01, device="cuda"), torch.zeros(1, device="cuda"), torch.full((D,), 0.01, device="cuda"), torch.zeros(1, device="cuda")]
    eng.readout_forward(out, th0, *ro)
    eng.set_graph_sparse(adj, indeg)                                 # a new batch with the same node count
    with pytest.raises(GgnnError, match="ggnn_readout_set_graphs has not been called for this batch"):
        eng.readout_forward(out, th0, *ro)
    eng.readout_set_graphs(24, graph_nodes_list=b["graph_nodes_list"])
    eng.readout_forward(out, th0, *ro)
    eng.sync_check()
