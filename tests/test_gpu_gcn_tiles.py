"""GPU: the fused GCN kernel on full 128-row LOCAL tiles, and the GCN at the benchmarked 100 000-node batch, against float64.

The batches are tests/test_gcn_tiles_cpu.py's, which pins their plans and tiles without a GPU.  Here every graph goes through the engine's
own ``prepare_graph_gcn`` and its tiles are checked again before ``set_graph_prepared``, so that an H100 with another SM count cannot
silently run smaller tiles.  Groups:

1. Forward at every row position of a LOCAL tile: every ``span*`` batch and ``mol1200``, bf16x3 at hidden 12 / 64 / 100 / 128 (NH 8 / 32 /
   56 / 64) and bf16 at 100 / 128, state keep 1.0 and 0.8 (the engine's mask replayed), three layers, biases drawn nonzero.  Without
   save the final state, with save every ``layer_state(l)``, against the float64 list-order loops (``span*``) or the float64 torch
   statement (``mol1200``).  Bars ``test_gpu_forward_plans.BARS``: bf16x3 1e-4, bf16 2e-2 (max|err| / max|ref| per state).
2. LOCAL = GLOBAL bit for bit on 128-row tiles: each LOCAL batch again under ``GGNN_FORCE_GLOBAL=1`` with the same weights; the final
   state, and with save every layer state, at keep 1.0 and 0.8.  This has no tolerance: a row of ``sH`` read or written wrong shows.
3. The benchmarked batch (tools/gcn_bench.py: 5 500 molecules, 99 046 nodes, hidden 100, four layers), bias off (the benchmark's model)
   and on: the forward on bf16x3 LOCAL, bf16, forced GLOBAL (bit-identical to LOCAL) and fp32; the backward on LOCAL-with-save and fp32,
   on this batch and on ``mol1200``, ``d h0`` and every kernel and bias gradient against float64 autograd of the torch statement at
   2.5e-5.  The gradient reference takes ReLU's pattern from the engine's saved states (``x * [state > 0]``): a pre-activation within
   the forward's rounding of 0 lies on the other side in float64, and ReLU's derivative jumps there.  Every node / column where the two
   patterns disagree must have |float64 pre-activation| below the forward bar times its layer's max|pre|; the count is printed.  The
   SparseGCNChemModel plug-in on this batch (forward_batch + loss.backward(), grouped readout over 5 500 graphs): every trainable's
   gradient against float64 autograd through readout and masked loss, at ``test_gpu_training_steps.GCN_BARS`` (fp32 2.5e-5, bf16x3
   2e-4).
4. Partial backward requests on ``mol1200`` (LOCAL-with-save and fp32): only ``d h0``, only kernels, only biases (the column-sum
   branch), kernels and biases without ``d h0`` (the early exit at layer 0), and kernels or biases with ``d h0``, against a full request:
   ``d h0`` bit for bit, weight gradients within the atomics' order noise (1e-5 of the largest entry).  Calls into prefilled buffers add
   exactly one gradient each and overwrite ``d h0``; ``d h0`` is bit-identical run to run.

The worst error of each group is printed at the end (``-s``).  Measured on an H100 80GB HBM3 at a 400 W power limit (164 tests, 70 s):
1. bf16x3 1.3e-5 (span65, hidden 12), bf16 5.6e-3 (span65, hidden 100);  2. bit-identical everywhere;  3. forward bf16x3 9.1e-6, bf16
4.8e-3, fp32 3.1e-7; backward bf16x3 5.0e-6 (a layer-3 kernel at 99 k nodes), fp32 6.8e-7; 32-34 ReLU pattern disagreements on bf16x3 at
99 k nodes, 8 on mol1200, none on fp32; plug-in bf16x3 6.3e-6, fp32 6.1e-7 (both the readout's transform weights);  4. weight-gradient
order noise 7.0e-7.  The weight gradients at 99 k nodes stay 5x inside 2.5e-5: the 132-way row split of their GEMM shows no summation
growth at that bar.
"""
import functools
import re

import numpy as np
import pytest

from gated_graph_neural_network_samples_b200.utils import SMALL_NUMBER
from tests import gcn_oracle as G
from tests._util import max_rel_err
from tests.test_gcn_tiles_cpu import LOCAL_BATCHES, SPANS, batch, check_tiles, molecule_feed, plan_pattern
from tests.test_gpu_forward_plans import BARS, _gcn_reference
from tests.test_forward_plans_cpu import GCN_LAYERS
from tests.test_gpu_training_steps import GCN_BARS

pytestmark = pytest.mark.gpu

GRAD_BAR = 2.5e-5
NOISE = 1e-5          # order noise of the weight-gradient atomics, relative to the largest entry
DROP_SEED = 20261016
BENCH_LAYERS = 4
WORST = {}            # group -> (err, case)


@pytest.fixture(scope="module", autouse=True)
def _report_worst():
    yield
    if WORST:
        print("\n\nworst max|err|/max|ref| per group:")
        for g, (e, name) in WORST.items():
            print("  %-34s %.2e (%s)" % (g, e, name))


def _note(group, err, name):
    WORST[group] = max(WORST.get(group, (0.0, "")), (err, name))


def _set_global(monkeypatch, force):
    if force:
        monkeypatch.setenv("GGNN_FORCE_GLOBAL", "1")
    else:
        monkeypatch.delenv("GGNN_FORCE_GLOBAL", raising=False)


# ---------------------------------------------------------------------------------------------------------------- inputs and runs
@functools.lru_cache(maxsize=4)
def _inputs(name, D, L, bias=True, feed_h0=False):
    """(h0, kernels, biases or None) of a batch at hidden D: glorot kernels, N(0, 0.2) biases, N(0, 1) states (``feed_h0``: the packed
    molecule features, the benchmark's own input)."""
    V, _, _ = batch(name)
    rng = np.random.default_rng([V, D, L, int(bias)])
    ks = [G.glorot((D, D), rng) for _ in range(L)]
    bs = [rng.normal(0, 0.2, D).astype(np.float32) for _ in range(L)] if bias else None
    h0 = molecule_feed(name)["initial_node_representation"] if feed_h0 else rng.normal(0, 1, (V, D)).astype(np.float32)
    return np.ascontiguousarray(h0, np.float32), ks, bs


class Run:
    """One GCNEngine on a batch: weights bound, save / dropout set, the graph prepared, its tiles checked, uploaded, one forward."""

    def __init__(self, name, D, L, precision, h0, ks, bs, save=False, keep=1.0):
        import torch
        from gated_graph_neural_network_samples_b200.engine import GCNEngine
        V, lst, w = batch(name)
        self.eng = eng = GCNEngine(D, L, use_bias=bs is not None, precision=precision)
        self.dk = [torch.from_numpy(k).cuda() for k in ks]
        self.db = None if bs is None else [torch.from_numpy(b).cuda() for b in bs]
        eng.set_weights(self.dk, self.db)
        eng.set_save_for_backward(save)
        g = eng.prepare_graph_gcn(V, lst, w)
        self.plan = g.info()["plan"]
        if precision != "fp32":
            check_tiles(name, g.arrays(1)["tile_start"], lst, "LOCAL" in self.plan)
        eng.set_graph_prepared(g)
        eng.set_state_dropout(keep, DROP_SEED)
        self.h0 = torch.from_numpy(h0).cuda()
        self.L, self.keep = L, keep
        self.out = self.forward()

    def forward(self):
        # the engine reads h0 and the output buffer again (layer_state(0) / layer_state(L), the backward): both stay alive here
        self.d_out = self.eng.forward(self.h0)
        self.eng.sync_check()
        return self.d_out.cpu().numpy()

    def states(self):
        return [self.eng.layer_state(l).cpu().numpy() for l in range(self.L + 1)]

    def masks(self):
        return [self.eng.state_dropout_mask(l, self.keep, DROP_SEED) for l in range(self.L - 1)] if self.keep < 1 else None

    def backward(self, g_out, fields, d_h0=True, into=None):
        """ggnn_gcn_backward into fresh zeroed buffers (or ``into``) for the requested fields of every layer; returns (d h0 or None,
        [{field: array}])."""
        import torch
        grads = into if into is not None else [{f: torch.zeros_like(dict(kernel=k, bias=b)[f]) for f in fields}
                                               for k, b in zip(self.dk, self.db or [None] * self.L)]
        dh0 = torch.full_like(self.h0, np.nan) if d_h0 else None     # overwritten, not accumulated into
        self.eng.backward(g_out, grads, d_h0=dh0)
        self.eng.sync_check()
        return (None if dh0 is None else dh0.cpu().numpy()), [{f: t.cpu().numpy() for f, t in lg.items()} for lg in grads]


def _torch_reference(name, h0, ks, bs, masks=None, keep=1.0):
    """node_states_per_layer and the pre-activation of every layer from the float64 torch statement (prefix by prefix, like
    ``_gcn_reference`` does with the loops)."""
    import torch
    _, lst, w = batch(name)
    L = len(ks)
    th0, tw = torch.from_numpy(h0).double(), torch.from_numpy(w).double()
    tk = [torch.from_numpy(k).double() for k in ks]
    tb = None if bs is None else [torch.from_numpy(b).double() for b in bs]
    states, pres = [np.asarray(h0, np.float64)], []
    for l in range(1, L + 1):
        pre = G.gcn_propagation_torch(th0, lst, tw, tk[:l], None if tb is None else tb[:l], masks, keep).numpy()
        pres.append(pre)
        if l < L:
            pre = np.maximum(pre, 0.0)
            if masks is not None:
                pre = pre * masks[l - 1] / np.float64(np.float32(keep))
        states.append(pre)
    return states, pres


def _pattern_propagation(th0, lst, w, tk, tb, patterns):
    """The float64 forward with ReLU replaced by ``x * patterns[l]`` (the engine's side of the kink), differentiable in h0 and weights."""
    import torch
    rows, cols = torch.from_numpy(np.asarray(lst[:, 0], np.int64)), torch.from_numpy(np.asarray(lst[:, 1], np.int64))
    wt, h = torch.from_numpy(w).double(), th0
    for l in range(len(tk)):
        h = torch.zeros_like(h).index_add_(0, rows, wt[:, None] * h[cols]) @ tk[l]
        if tb is not None:
            h = h + tb[l]
        if l < len(tk) - 1:
            h = h * torch.from_numpy(patterns[l].astype(np.float64))
    return h


def _kink_check(tag, patterns, pres, bar):
    """Where the engine's ReLU pattern and float64's ``pre > 0`` disagree, |float64 pre| must lie within the forward's rounding of 0."""
    count = 0
    for l, (p, pre) in enumerate(zip(patterns, pres)):
        dis = p != (pre > 0)
        count += int(dis.sum())
        lim = bar * float(np.max(np.abs(pre)))
        if dis.any():
            assert float(np.max(np.abs(pre[dis]))) < lim, (tag, "layer %d" % l, float(np.max(np.abs(pre[dis]))), lim)
    print("\n%-40s ReLU pattern disagreements with float64: %d" % (tag, count))
    return count


# ---------------------------------------------------------------------------------------------------------------- 1. forward
FWD_BATCHES = ["span%d" % S for S in SPANS] + ["span129", "mol1200"]
FWD_CASES = [(name, prec, D, keep) for name in FWD_BATCHES for D in (12, 64, 100, 128) for keep in (1.0, 0.8)
             for prec in ("bf16x3", "bf16") if prec == "bf16x3" or D >= 100]
_REFS = {}


def _reference_states(name, D, keep, masks):
    """Cached per (batch, hidden, keep): the precisions and save on / off share it (the cases run in that order: two entries suffice)."""
    key = (name, D, keep)
    if key not in _REFS:
        while len(_REFS) >= 2:
            _REFS.pop(next(iter(_REFS)))
        h0, ks, bs = _inputs(name, D, GCN_LAYERS)
        if name.startswith("span"):
            _REFS[key] = _gcn_reference(h0, batch(name)[1], batch(name)[2], ks, bs, masks, keep)
        else:
            _REFS[key] = _torch_reference(name, h0, ks, bs, masks, keep)[0]
    return _REFS[key]


@pytest.mark.parametrize("name,precision,D,keep", FWD_CASES, ids=["%s-%s-D%d-keep%g" % c for c in FWD_CASES])
def test_forward_at_every_row_position(name, precision, D, keep):
    tag = "%s-%s-D%d-keep%g" % (name, precision, D, keep)
    h0, ks, bs = _inputs(name, D, GCN_LAYERS)
    r = Run(name, D, GCN_LAYERS, precision, h0, ks, bs, save=False, keep=keep)
    assert re.search(plan_pattern(name, precision), r.plan), (tag, r.plan)
    refs = _reference_states(name, D, keep, r.masks())
    bar = BARS[precision]
    err = max_rel_err(r.out, refs[-1])
    assert err < bar, (tag, "final", err)
    s = Run(name, D, GCN_LAYERS, precision, h0, ks, bs, save=True, keep=keep)
    states = s.states()
    np.testing.assert_array_equal(states[0], h0)
    np.testing.assert_array_equal(states[-1], s.out)
    np.testing.assert_array_equal(s.out, r.out, err_msg=tag + ": save on / off")
    errs = [max_rel_err(g, ref) for g, ref in zip(states, refs)]
    print("\n%-32s %s" % (tag, " ".join("%.2e" % e for e in errs[1:])))
    _note("forward %s" % precision, max([err] + errs), tag)
    for l, e in enumerate(errs):
        assert e < bar, (tag, "layer %d" % l, e)


# ---------------------------------------------------------------------------------------------------------------- 2. LOCAL = GLOBAL
LG_BATCHES = [b for b in LOCAL_BATCHES if b != "bench"]
LG_CASES = [(name, prec, D, keep) for name in LG_BATCHES for prec, D in (("bf16x3", 12), ("bf16x3", 64), ("bf16x3", 128), ("bf16", 100))
            for keep in (1.0, 0.8)]


@pytest.mark.parametrize("name,precision,D,keep", LG_CASES, ids=["%s-%s-D%d-keep%g" % c for c in LG_CASES])
def test_local_equals_global_on_128_row_tiles(name, precision, D, keep, monkeypatch):
    """Same gather order, operand split, MMAs and epilogue: only where the previous layer's state is read from differs."""
    h0, ks, bs = _inputs(name, D, GCN_LAYERS)
    for save in (False, True):
        runs = []
        for force in (False, True):
            _set_global(monkeypatch, force)
            runs.append(Run(name, D, GCN_LAYERS, precision, h0, ks, bs, save=save, keep=keep))
        loc, glo = runs
        assert " LOCAL(" in loc.plan and " GLOBAL(" in glo.plan, (loc.plan, glo.plan)
        np.testing.assert_array_equal(loc.out, glo.out, err_msg="%s save=%s: final state" % (name, save))
        if save:
            for l, (a, b) in enumerate(zip(loc.states(), glo.states())):
                np.testing.assert_array_equal(a, b, err_msg="%s: layer %d" % (name, l))
    _set_global(monkeypatch, False)


# ---------------------------------------------------------------------------------------------------------------- 3. the benchmarked batch
@pytest.mark.parametrize("bias", [False, True], ids=["nobias", "bias"])
def test_benchmarked_batch_forward(bias, monkeypatch):
    """Hidden 100, four layers; bias off with the packed molecule features as h0 is tools/gcn_bench.py's model and input."""
    h0, ks, bs = _inputs("bench", 100, BENCH_LAYERS, bias=bias, feed_h0=not bias)
    ref = _torch_reference("bench", h0, ks, bs)[0][-1]
    outs = {}
    for label, precision, force in (("bf16x3 LOCAL", "bf16x3", False), ("bf16", "bf16", False), ("bf16x3 forced GLOBAL", "bf16x3", True),
                                    ("fp32", "fp32", False)):
        _set_global(monkeypatch, force)
        r = Run("bench", 100, BENCH_LAYERS, precision, h0, ks, bs)
        assert (" GLOBAL(" if force or precision == "fp32" else " LOCAL(") in r.plan, (label, r.plan)
        err = max_rel_err(r.out, ref)
        tag = "bench-%s-%s" % ("bias" if bias else "nobias", label)
        print("\n%-40s %.2e  %s" % (tag, err, r.plan[:60]))
        _note("bench forward %s" % precision, err, tag)
        assert err < BARS[precision], (tag, err)
        outs[label] = r.out
    _set_global(monkeypatch, False)
    np.testing.assert_array_equal(outs["bf16x3 LOCAL"], outs["bf16x3 forced GLOBAL"])


BWD_CASES = [("bench", "bf16x3", False), ("bench", "bf16x3", True), ("bench", "fp32", False), ("bench", "fp32", True),
             ("mol1200", "bf16x3", True), ("mol1200", "fp32", True)]


@pytest.mark.parametrize("name,precision,bias", BWD_CASES, ids=["%s-%s-%s" % (n, p, "bias" if b else "nobias") for n, p, b in BWD_CASES])
def test_backward_against_float64_autograd(name, precision, bias, monkeypatch):
    import torch
    _set_global(monkeypatch, False)
    tag = "%s-%s-%s" % (name, precision, "bias" if bias else "nobias")
    L = BENCH_LAYERS
    h0, ks, bs = _inputs(name, 100, L, bias=bias, feed_h0=name == "bench" and not bias)
    r = Run(name, 100, L, precision, h0, ks, bs, save=True)
    assert (" LOCAL(" if precision != "fp32" else "gcn-fp32") in r.plan, r.plan
    states = r.states()
    ref_states, pres = _torch_reference(name, h0, ks, bs)
    f_err = max(max_rel_err(g, ref) for g, ref in zip(states, ref_states))
    assert f_err < BARS[precision], (tag, "forward", f_err)
    g_out = np.random.default_rng(5).normal(0, 1, h0.shape).astype(np.float32)
    fields = ["kernel", "bias"] if bias else ["kernel"]
    dh0, grads = r.backward(torch.from_numpy(g_out).cuda(), fields)
    patterns = [states[l + 1] > 0 for l in range(L - 1)]
    _kink_check(tag, patterns, pres[:-1], BARS[precision])
    _, lst, w = batch(name)
    th0 = torch.from_numpy(h0).double().requires_grad_()
    tk = [torch.from_numpy(k).double().requires_grad_() for k in ks]
    tb = None if bs is None else [torch.from_numpy(b).double().requires_grad_() for b in bs]
    _pattern_propagation(th0, lst, w, tk, tb, patterns).backward(torch.from_numpy(g_out).double())
    pairs = [("d h0", dh0, th0.grad)] + [("layer %d kernel" % l, grads[l]["kernel"], tk[l].grad) for l in range(L)]
    if bias:
        pairs += [("layer %d bias" % l, grads[l]["bias"], tb[l].grad) for l in range(L)]
    errs = [(max_rel_err(g, ref.numpy()), n) for n, g, ref in pairs]
    worst = max(errs)
    print("\n%-40s forward %.2e  worst gradient %.2e on %s" % (tag, f_err, worst[0], worst[1]))
    _note("backward %s" % precision, worst[0], "%s %s" % (tag, worst[1]))
    bad = [(n, e) for e, n in errs if not e < GRAD_BAR]
    assert not bad, (tag, bad)


@pytest.mark.parametrize("precision", ["fp32", "bf16x3"])
def test_plugin_gradients_on_the_benchmarked_batch(tmp_path, precision):
    """SparseGCNChemModel (hidden 100, four layers, no bias: the benchmark's model) on the benchmark's batch: forward_batch and
    loss.backward() through the engine's backward and the grouped readout over 5 500 graphs; every trainable against float64 autograd."""
    import torch
    from gated_graph_neural_network_samples_b200 import synthetic
    from gated_graph_neural_network_samples_b200.chem_gcn import SparseGCNChemModel
    L = BENCH_LAYERS
    mols = synthetic.make_molecules(8, seed=1)
    m = SparseGCNChemModel({"--log_dir": str(tmp_path), "--precision": precision, "--train_data": mols[:4], "--valid_data": mols[4:],
                            "--config": {"batch_size": 100000, "hidden_size": 100, "num_timesteps": L, "gcn_use_bias": False,
                                         "random_seed": 0}})
    feed = dict(molecule_feed("bench"), graph_state_keep_prob=1.0, out_layer_dropout_keep_prob=1.0)
    loss, _ = m.forward_batch(feed)
    loss.backward()
    torch.cuda.synchronize()
    m.engine.sync_check()
    assert m.engine.plan.startswith("gcn-fp32" if precision == "fp32" else "gcn-wgmma-bf16x3 LOCAL("), m.engine.plan
    patterns = [m.engine.layer_state(l + 1).cpu().numpy() > 0 for l in range(L - 1)]
    named = dict(m.trainable_variables())
    assert len(named) == L + 4
    ref = {n: v.detach().cpu().double().requires_grad_() for n, v in named.items()}
    ks = [ref["graph_model/gcn_scope/gcn_weights_%d:0" % l] for l in range(L)]
    h0 = np.asarray(feed["initial_node_representation"], np.float32)
    _, pres = _torch_reference("bench", h0, [k.detach().numpy().astype(np.float32) for k in ks], None)
    _kink_check("plug-in %s" % precision, patterns, pres[:-1], BARS[precision])
    th0 = torch.from_numpy(h0).double()
    final = _pattern_propagation(th0, feed["adjacency_list"], np.asarray(feed["adjacency_weights"], np.float32), ks, None, patterns)
    wg, bg = ref["out_layer_task0/regression_gate/MLP_W_layer0:0"], ref["out_layer_task0/regression_gate/MLP_b_layer0:0"]
    wt, bt = ref["out_layer_task0/regression/MLP_W_layer0:0"], ref["out_layer_task0/regression/MLP_b_layer0:0"]
    gated = torch.sigmoid(torch.cat([final, th0], 1) @ wg + bg) * (final @ wt + bt)
    gnl = torch.from_numpy(np.asarray(feed["graph_nodes_list"], np.int64))
    ro = torch.zeros(int(feed["num_graphs"]), 1, dtype=torch.float64).index_add_(0, gnl, gated).squeeze(-1)
    tv = torch.from_numpy(np.asarray(feed["target_values"], np.float64)[0])
    tm = torch.from_numpy(np.asarray(feed["target_mask"], np.float64)[0])
    diff = (ro - tv) * tm
    ((0.5 * diff * diff).sum() / (tm.sum() + SMALL_NUMBER)).backward()
    errs = []
    for n, v in named.items():
        assert v.grad is not None, n
        errs.append((max_rel_err(v.grad.cpu().numpy(), ref[n].grad.numpy()), n))
    worst = max(errs)
    print("\nplug-in %-8s worst gradient %.2e on %s" % (precision, worst[0], worst[1]))
    _note("plug-in %s" % precision, worst[0], worst[1])
    bad = [(n, e) for e, n in errs if not e < GCN_BARS[precision]]
    assert not bad, (precision, bad)


# ---------------------------------------------------------------------------------------------------------------- 4. partial requests
REQUESTS = {"d h0": ((), True), "kernels": (("kernel",), False), "biases": (("bias",), False), "kernels+biases": (("kernel", "bias"), False),
            "kernels+d h0": (("kernel",), True), "biases+d h0": (("bias",), True)}


@pytest.mark.parametrize("precision", ["bf16x3", "fp32"])
def test_partial_backward_requests(precision, monkeypatch):
    import torch
    _set_global(monkeypatch, False)
    L = BENCH_LAYERS
    h0, ks, bs = _inputs("mol1200", 100, L)
    r = Run("mol1200", 100, L, precision, h0, ks, bs, save=True)
    assert (" LOCAL(" if precision != "fp32" else "gcn-fp32") in r.plan, r.plan
    g_out = torch.from_numpy(np.random.default_rng(6).normal(0, 1, h0.shape).astype(np.float32)).cuda()
    full_dh0, full = r.backward(g_out, ("kernel", "bias"))
    assert np.all(np.isfinite(full_dh0))
    noise = 0.0
    for req, (fields, want_dh0) in REQUESTS.items():
        dh0, part = r.backward(g_out, fields, d_h0=want_dh0)
        if want_dh0:
            np.testing.assert_array_equal(dh0, full_dh0, err_msg=req)
        for l, (p, f) in enumerate(zip(part, full)):
            assert sorted(p) == sorted(fields), (req, l)
            for k in p:
                e = max_rel_err(p[k], f[k])
                noise = max(noise, e)
                assert e < NOISE, (precision, req, l, k, e)
    _note("partial requests %s" % precision, noise, "order noise")
    # prefilled buffers: each call adds one gradient and overwrites d h0
    rng = np.random.default_rng(9)
    pre = [{k: (rng.normal(size=v.shape) * np.max(np.abs(v))).astype(np.float32) for k, v in lw.items()} for lw in full]
    bufs = [{k: torch.from_numpy(v.copy()).cuda() for k, v in lw.items()} for lw in pre]
    for n in (1, 2):
        dh0, acc = r.backward(g_out, ("kernel", "bias"), into=bufs)
        np.testing.assert_array_equal(dh0, full_dh0)
        for l, (a, p, f) in enumerate(zip(acc, pre, full)):
            for k in a:
                err = np.max(np.abs(a[k] - (p[k].astype(np.float64) + n * f[k].astype(np.float64))))
                assert err <= 2 * n * NOISE * np.max(np.abs(f[k])), (precision, n, l, k, err)
    # run to run: a second forward and backward give the same state and d h0, bit for bit
    out_b = r.forward()
    dh0_b, _ = r.backward(g_out, ("kernel", "bias"))
    np.testing.assert_array_equal(out_b, r.out)
    np.testing.assert_array_equal(dh0_b, full_dh0)
