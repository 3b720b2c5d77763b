"""GPU: adjacency weights on the device in the sparse GCN model, against the host-weighted batch and float64.

A batch prepared with ``prepare_graph_gcn_message_weighted`` takes its adjacency weights on the device (``set_message_weights``);
``backward(..., d_adjacency_weights=)`` adds their gradient  d w_k = sum_l <dS_l[i_k], H_l[j_k]>.  On every GCN plan (the wgmma kernel
LOCAL at 12 / 100 / 128 and GLOBAL at 128, bf16 at 100, the fp32 kernel at 100 / 132 / 256 and bf16x3 at 256 without wide_hidden, the
streaming plan at 256 / 384 / 512):

* the forward and every layer state are bit-identical to the host-weighted batch with the same weights, and within 1e-4 (bf16x3),
  2e-2 (bf16) and 1e-5 (fp32) of float64;
* d h0, dW and db with d w requested are bit-identical to ``ggnn_gcn_backward`` on the host-weighted batch (deterministic mode);
* d w is within 2.5e-5 (fp32 backward) / 2e-4 (bf16x3 backward) of float64 autograd through the engine's relu / dropout pattern.

Then edge cases (duplicates, self-loops, isolated nodes, nnz = 0, zero / negative / mixed weights, a one-entry list, L = 1, d w alone),
bit-repeatability in both deterministic modes, two weight vectors on one upload, refusals, the 100 000-node batch, guard bands, a NaN
component, and an end-to-end learned normalization through ``chem_gcn.propagate``.
"""
import numpy as np
import pytest

from tests import gcn_oracle as G
from tests._util import max_rel_err

pytestmark = pytest.mark.gpu

BARS = {"bf16x3": 1e-4, "bf16": 2e-2, "fp32": 1e-5}
GRAD_BARS = {"fp32": 2.5e-5, "bf16x3": 2e-4}
SEED = 4242
TAG = " [message-weighted]"

# name -> (hidden size, precision, wide_hidden, state dropout keep, batch kind, plan pattern)
PLANS = {
    "local-12": (12, "bf16x3", False, 1.0, "mol", r"^gcn-wgmma-bf16x3 LOCAL\("),
    "local-100": (100, "bf16x3", False, 1.0, "mol", r"^gcn-wgmma-bf16x3 LOCAL\("),
    "local-100-drop": (100, "bf16x3", False, 0.8, "mol", r"^gcn-wgmma-bf16x3 LOCAL\("),
    "local-128": (128, "bf16x3", False, 1.0, "mol", r"^gcn-wgmma-bf16x3 LOCAL\("),
    "local-128-drop": (128, "bf16x3", False, 0.8, "mol", r"^gcn-wgmma-bf16x3 LOCAL\("),
    "bf16-100": (100, "bf16", False, 1.0, "mol", r"^gcn-wgmma-bf16 LOCAL\("),
    "global-128": (128, "bf16x3", False, 1.0, "big", r"^gcn-wgmma-bf16x3 GLOBAL\("),
    "fp32-100": (100, "fp32", False, 1.0, "mol", r"^gcn-fp32-ffma GLOBAL\("),
    "fp32-132": (132, "fp32", False, 0.8, "big", r"^gcn-fp32-ffma GLOBAL\("),
    "fp32-256": (256, "fp32", False, 1.0, "mol", r"^gcn-fp32-ffma GLOBAL\("),
    "x3-256-narrow": (256, "bf16x3", False, 1.0, "mol", r"^gcn-fp32-ffma GLOBAL\("),
    "stream-256": (256, "bf16x3", True, 1.0, "mol", r"^gcn-stream-bf16x3 \("),
    "stream-384": (384, "bf16x3", True, 0.8, "big", r"^gcn-stream-bf16x3 \("),
    "stream-512": (512, "bf16x3", True, 1.0, "mol", r"^gcn-stream-bf16x3 \("),
}


def _cuda(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a, np.float32)).cuda()


def graph(kind, seed=0):
    """(V, list, weights): ``mol`` is 40 components of 2-60 nodes with self-loops, ``big`` adds a 150-node component (a GLOBAL plan on
    the wgmma kernel); both have duplicate entries, isolated nodes at the end and mixed-sign weights with zeros."""
    rng = np.random.default_rng(seed)
    sizes = [int(x) for x in rng.integers(2, 60, 40)] + ([150] if kind == "big" else [])
    V, lst, w = G.component_list(sizes, rng)
    lst = np.concatenate([lst, lst[::17]])
    w = np.concatenate([w, rng.normal(0, 1, lst.shape[0] - w.shape[0]).astype(np.float32)])
    w[::9] = 0.0
    return V + 3, lst, w


def weights(D, L, bias, seed):
    rng = np.random.default_rng([D, L, seed])
    ks = [G.glorot((D, D), rng) for _ in range(L)]
    bs = [rng.normal(0, 0.2, D).astype(np.float32) for _ in range(L)] if bias else None
    return ks, bs


class Run:
    """Two GCN engines on one batch: ``host`` with the weights fed on the host (ggnn_prepare_graph_gcn), ``dev`` message-weighted with the
    same weights set on the device."""

    def __init__(self, name, L=3, bias=True, det=False, bwd="fp32", V=None, lst=None, w=None, seed=0):
        import re
        import torch
        from gated_graph_neural_network_samples_b200.engine import GCNEngine
        self.D, precision, wide, self.keep, kind, pat = PLANS[name]
        self.precision, self.L = precision, L
        if lst is None:
            V, lst, w = graph(kind, seed)
        self.V, self.lst, self.w = V, lst, np.asarray(w, np.float32)
        self.ks, self.bs = weights(self.D, L, bias, seed)
        rng = np.random.default_rng(seed + 1)
        self.h0 = rng.normal(0, 1, (V, self.D)).astype(np.float32)
        self.dk = [_cuda(k) for k in self.ks]
        self.db = None if self.bs is None else [_cuda(b) for b in self.bs]
        self.engines = {}
        for side in ("host", "dev"):
            eng = GCNEngine(self.D, L, use_bias=bias, precision=precision, wide_hidden=wide)
            eng.set_weights(self.dk, self.db)
            eng.set_save_for_backward(True)
            eng.set_deterministic(det)
            eng.set_backward_precision(bwd)
            eng.set_state_dropout(self.keep, SEED)
            if side == "host":
                eng.set_graph_gcn(V, lst, self.w)
            else:
                eng.set_graph_prepared(eng.prepare_graph_gcn_message_weighted(V, lst))
                assert eng.plan == self.engines["host"].plan + TAG, eng.plan
                assert eng.num_messages() == lst.shape[0]
                eng.set_message_weights(_cuda(self.w))
            assert re.search(pat, eng.plan), (name, eng.plan)
            self.engines[side] = eng
        self.dev = self.engines["dev"]
        self.th0 = _cuda(self.h0)
        self.outs = {s: torch.empty_like(self.th0) for s in self.engines}

    def forward(self, side="dev"):
        self.engines[side].forward(self.th0, self.outs[side])
        self.engines[side].sync_check()
        return self.outs[side].cpu().numpy()

    def states(self, side="dev"):
        return [self.engines[side].layer_state(l).cpu().numpy() for l in range(1, self.L + 1)]

    def backward(self, g_out, side="dev", dw=True, dh0=True, layer_grads=True, dw_buf=None):
        import torch
        grads = [{"kernel": torch.zeros_like(k), **({"bias": torch.zeros_like(self.db[l])} if self.db else {})} if layer_grads else {}
                 for l, k in enumerate(self.dk)]
        d_h0 = torch.full_like(self.th0, np.nan) if dh0 else None
        d_w = None
        if dw:
            d_w = dw_buf if dw_buf is not None else torch.zeros(self.lst.shape[0], dtype=torch.float32, device="cuda")
        self.engines[side].backward(_cuda(g_out), grads, d_h0, d_adjacency_weights=d_w)
        self.engines[side].sync_check()
        return (None if d_w is None else d_w.cpu().numpy(), None if d_h0 is None else d_h0.cpu().numpy(),
                [{k: v.cpu().numpy() for k, v in g.items()} for g in grads])

    def masks(self):
        return [self.dev.state_dropout_mask(l, self.keep, SEED) for l in range(self.L - 1)] if self.keep < 1.0 else None

    def oracle_states(self):
        """Every layer's state in float64, the list-order statement."""
        out, h, masks = [], np.asarray(self.h0, np.float64), self.masks()
        for l in range(self.L):
            h = G.gcn_propagation_loops(h, self.lst, self.w, [self.ks[l]], None if self.bs is None else [self.bs[l]])
            if l < self.L - 1:
                h = np.maximum(h, 0.0)
                if masks is not None:
                    h = h * masks[l] / np.float64(np.float32(self.keep))
            out.append(h)
        return out

    def autograd(self, g_out, states, device="cpu"):
        """float64 autograd of (h0, kernels, biases, w) through the engine's relu / dropout pattern (its saved states' y > 0)."""
        import torch
        rows = torch.from_numpy(np.ascontiguousarray(self.lst[:, 0])).to(device)
        cols = torch.from_numpy(np.ascontiguousarray(self.lst[:, 1])).to(device)
        t = lambda a: torch.from_numpy(np.asarray(a, np.float64)).to(device).requires_grad_()   # noqa: E731
        th0, tw = t(self.h0), t(self.w)
        tk = [t(k) for k in self.ks]
        tb = [t(b) for b in self.bs] if self.bs is not None else None
        h = th0
        for l in range(self.L):
            h = torch.zeros_like(h).index_add_(0, rows, tw[:, None] * h[cols]) @ tk[l]
            if tb is not None:
                h = h + tb[l]
            if l < self.L - 1:
                h = h * torch.from_numpy(states[l] > 0).to(device).double() / float(np.float32(self.keep))
        h.backward(torch.from_numpy(np.asarray(g_out, np.float64)).to(device))
        return tw.grad.cpu().numpy(), th0.grad.cpu().numpy(), tk, tb


def _g_out(V, D, seed=6):
    return np.random.default_rng(seed).normal(0, 1, (V, D)).astype(np.float32)


# ---------------------------------------------------------------------------------------------------------------- every plan
@pytest.mark.parametrize("name", sorted(PLANS))
def test_forward_is_the_host_weighted_batch_and_matches_float64(name):
    r = Run(name)
    dev, host = r.forward("dev"), r.forward("host")
    np.testing.assert_array_equal(dev, host)
    ref = r.oracle_states()
    for l, (a, b) in enumerate(zip(r.states("dev"), r.states("host"))):
        np.testing.assert_array_equal(a, b, err_msg="layer %d" % (l + 1))
        err = max_rel_err(a, ref[l])
        assert err < BARS[r.precision], (name, l + 1, err)
    for _ in range(2):
        np.testing.assert_array_equal(r.forward("dev"), dev)


@pytest.mark.parametrize("bwd", ["fp32", "bf16x3"])
@pytest.mark.parametrize("name", sorted(PLANS))
def test_gradients_are_the_host_weighted_ones_and_d_w_matches_float64(name, bwd):
    # deterministic mode: dW and db are fixed-order sums there (else atomics, which differ between any two calls)
    r = Run(name, bwd=bwd, det=True)
    r.forward("host")
    out = r.forward("dev")
    g_out = _g_out(r.V, r.D)
    dw, dh0, gw = r.backward(g_out, "dev")
    _, hdh0, hgw = r.backward(g_out, "host", dw=False)
    np.testing.assert_array_equal(dh0, hdh0)
    for l in range(r.L):
        for k in gw[l]:
            np.testing.assert_array_equal(gw[l][k], hgw[l][k], err_msg="layer %d %s" % (l, k))
    assert np.all(np.isfinite(dw)) and np.all(np.isfinite(out))
    if r.precision == "bf16":
        return   # the bf16 forward's states are 2e-2 from float64: d w is pinned to the host-weighted batch's gradients above
    states = r.states("dev")
    rdw, rdh0, tk, tb = r.autograd(g_out, states[:-1])
    err = max_rel_err(dw, rdw)
    print("\nGCNMW %-16s bwd %-6s d w %.2e  d h0 %.2e" % (name, bwd, err, max_rel_err(dh0, rdh0)))
    assert err < GRAD_BARS[bwd], (name, bwd, err)
    assert max_rel_err(dh0, rdh0) < GRAD_BARS[bwd]
    for l in range(r.L):
        assert max_rel_err(gw[l]["kernel"], tk[l].grad.numpy()) < GRAD_BARS[bwd], (l, "kernel")
        assert max_rel_err(gw[l]["bias"], tb[l].grad.numpy()) < GRAD_BARS[bwd], (l, "bias")


# ---------------------------------------------------------------------------------------------------------------- edge cases
@pytest.mark.parametrize("regime", ["zero", "negative", "mixed"])
@pytest.mark.parametrize("name", ["local-100", "fp32-100", "stream-384"])
def test_weight_regimes(name, regime):
    V, lst, w = graph("mol", 3)
    rng = np.random.default_rng(4)
    w = {"zero": np.zeros_like(w), "negative": -rng.uniform(0.1, 1.5, w.shape), "mixed": rng.normal(0, 1, w.shape)}[regime]
    r = Run(name, V=V, lst=lst, w=w.astype(np.float32))
    np.testing.assert_array_equal(r.forward("dev"), r.forward("host"))
    g_out = _g_out(V, r.D, 7)
    dw, dh0, _ = r.backward(g_out)
    rdw, rdh0, _, _ = r.autograd(g_out, r.states()[:-1])
    assert max_rel_err(dw, rdw) < GRAD_BARS["fp32"] and max_rel_err(dh0, rdh0) < GRAD_BARS["fp32"], regime


@pytest.mark.parametrize("name", ["local-100", "fp32-256", "stream-256"])
def test_empty_list(name):
    """nnz = 0: every state is the bias; d w has no entries, and the other gradients are the host-weighted batch's."""
    import torch
    V = 70
    lst, w = np.zeros((0, 2), np.int64), np.zeros(0, np.float32)
    r = Run(name, V=V, lst=lst, w=w)
    np.testing.assert_array_equal(r.forward("dev"), r.forward("host"))
    g_out = _g_out(V, r.D)
    dw, dh0, gw = r.backward(g_out)
    _, hdh0, hgw = r.backward(g_out, "host", dw=False)
    assert dw.shape == (0,)
    np.testing.assert_array_equal(dh0, hdh0)
    np.testing.assert_array_equal(gw[0]["bias"], hgw[0]["bias"])
    assert torch.isfinite(torch.from_numpy(dh0)).all()


@pytest.mark.parametrize("name", ["local-100", "fp32-100", "stream-256"])
def test_one_entry_list_pins_the_orientation(name):
    """One entry (i, j) = (0, 1), L = 1, no bias: d w = <dS[0], H[1]> with dS = d_out . W^T -- not <dS[1], H[0]>."""
    lst = np.array([[0, 1]], np.int64)
    r = Run(name, L=1, bias=False, V=2, lst=lst, w=np.array([0.75], np.float32))
    out = r.forward()
    assert np.all(out[1] == 0)   # row 1 has no entries
    g_out = _g_out(2, r.D, 8)
    dw, dh0, _ = r.backward(g_out)
    dS = g_out.astype(np.float64) @ r.ks[0].astype(np.float64).T
    want, wrong = dS[0] @ r.h0[1], dS[1] @ r.h0[0]
    assert abs(dw[0] - want) < 1e-4 * max(abs(want), 1.0), (dw[0], want, wrong)
    assert abs(want - wrong) > 1e-2
    np.testing.assert_allclose(dh0[1], 0.75 * dS[0], rtol=1e-4, atol=1e-5)
    assert np.all(dh0[0] == 0)


@pytest.mark.parametrize("name", ["local-100", "fp32-132", "stream-512"])
def test_one_layer_and_d_w_alone(name):
    """L = 1 with and without d h0, and d w alone (no layer gradient, no d h0): the same d w every time."""
    r = Run(name, L=1)
    r.forward()
    g_out = _g_out(r.V, r.D, 9)
    full = r.backward(g_out)[0]
    no_h0 = r.backward(g_out, dh0=False)[0]
    alone = r.backward(g_out, dh0=False, layer_grads=False)[0]
    np.testing.assert_array_equal(no_h0, full)
    np.testing.assert_array_equal(alone, full)
    rdw, _, _, _ = r.autograd(g_out, [])
    assert max_rel_err(full, rdw) < GRAD_BARS["fp32"]
    r3 = Run(name, L=3)
    r3.forward()
    g3 = _g_out(r3.V, r3.D, 10)
    a = r3.backward(g3, dh0=False, layer_grads=False)[0]
    np.testing.assert_array_equal(a, r3.backward(g3)[0])


@pytest.mark.parametrize("det", [False, True])
@pytest.mark.parametrize("bwd", ["fp32", "bf16x3"])
@pytest.mark.parametrize("name", ["local-100-drop", "global-128", "stream-384"])
def test_d_w_repeats_bit_for_bit(name, bwd, det):
    r = Run(name, det=det, bwd=bwd)
    r.forward()
    g_out = _g_out(r.V, r.D, 11)
    first, second = r.backward(g_out), r.backward(g_out)
    np.testing.assert_array_equal(first[0], second[0])
    np.testing.assert_array_equal(first[1], second[1])
    if det:
        for a, b in zip(first[2], second[2]):
            for k in a:
                np.testing.assert_array_equal(a[k], b[k], err_msg=k)


@pytest.mark.parametrize("name", ["local-100", "fp32-100", "stream-256"])
def test_two_weight_vectors_on_one_upload(name):
    """One upload, two weight vectors: each forward is its host-weighted batch's; a backward after the second set and before a forward is
    refused (setting the weights drops the saved activations)."""
    from gated_graph_neural_network_samples_b200.engine import GgnnError
    r = Run(name)
    w2 = np.random.default_rng(12).normal(0, 1, r.w.shape).astype(np.float32)
    first = r.forward()
    r.dev.set_message_weights(_cuda(w2))
    g_out = _g_out(r.V, r.D, 13)
    with pytest.raises(GgnnError) as e:
        r.backward(g_out)
    assert e.value.code == -3
    second = r.forward()
    assert not np.array_equal(first, second)
    r.engines["host"].set_graph_gcn(r.V, r.lst, w2)
    np.testing.assert_array_equal(second, r.forward("host"))
    r.w = w2
    dw = r.backward(g_out)[0]
    rdw, _, _, _ = r.autograd(g_out, r.states()[:-1])
    assert max_rel_err(dw, rdw) < GRAD_BARS["fp32"]


def test_refusals():
    import torch
    from gated_graph_neural_network_samples_b200.engine import GCNEngine, GgnnError
    V, lst, w = graph("mol", 5)
    D, L = 100, 2
    ks, _ = weights(D, L, False, 5)
    eng = GCNEngine(D, L, precision="bf16x3")
    eng.set_weights([_cuda(k) for k in ks])
    eng.set_save_for_backward(True)
    g = eng.prepare_graph_gcn_message_weighted(V, lst)
    eng.set_graph_prepared(g)
    th0 = _cuda(np.ones((V, D)))
    with pytest.raises(GgnnError) as e:   # a forward before the weights
        eng.forward(th0)
    assert e.value.code == -3
    with pytest.raises(GgnnError, match="entries"):   # a weight tensor of the wrong length
        eng.set_message_weights(_cuda(np.ones(lst.shape[0] + 1)))
    eng.set_message_weights(_cuda(w))
    out = eng.forward(th0)
    grads = [{"kernel": torch.zeros(D, D, device="cuda")} for _ in range(L)]
    with pytest.raises(GgnnError, match="num_messages"):
        eng.backward(torch.ones_like(out), grads, None, d_adjacency_weights=torch.zeros(lst.shape[0] - 1, device="cuda"))
    eng.set_graph_prepared(g)   # an upload forgets the weights
    with pytest.raises(GgnnError) as e:
        eng.forward(th0)
    assert e.value.code == -3
    eng.set_graph_gcn(V, lst, w)   # an ordinary batch takes no weights, and no d w
    with pytest.raises(GgnnError) as e:
        eng.set_message_weights(_cuda(w))
    assert e.value.code == -3
    out = eng.forward(th0)
    with pytest.raises(GgnnError) as e:
        eng.backward(torch.ones_like(out), grads, None, d_adjacency_weights=torch.zeros(lst.shape[0], device="cuda"))
    assert e.value.code == -3
    eng.backward(torch.ones_like(out), grads, None)   # the ordinary backward still runs
    eng.sync_check()


# ---------------------------------------------------------------------------------------------------------------- the benchmark batch
def test_100k_node_batch():
    """The plug-in's 100 000-node batch (99 046 nodes, nnz 302 492) at hidden 100, 4 layers on the LOCAL wgmma kernel: forward bits against
    the host-weighted batch, d w against float64 autograd on the device."""
    from tests.test_gcn_tiles_cpu import batch
    V, lst, w = batch("bench")
    r = Run("local-100", L=4, bias=False, V=V, lst=lst, w=w)
    np.testing.assert_array_equal(r.forward("dev"), r.forward("host"))
    g_out = _g_out(V, r.D, 14)
    dw, dh0, _ = r.backward(g_out)
    rdw, rdh0, _, _ = r.autograd(g_out, r.states()[:-1], device="cuda")
    print("\nGCNMW 100k d w %.2e  d h0 %.2e" % (max_rel_err(dw, rdw), max_rel_err(dh0, rdh0)))
    assert max_rel_err(dw, rdw) < GRAD_BARS["fp32"] and max_rel_err(dh0, rdh0) < GRAD_BARS["fp32"]


# ---------------------------------------------------------------------------------------------------------------- canaries
def _guarded(n, fill):
    """A [n] view between two bands of 64 payload NaNs, in one allocation; the view starts as ``fill``."""
    import torch
    buf = torch.full((n + 128,), float("nan"), device="cuda")
    view = buf[64:64 + n]
    view.fill_(fill)
    return buf, view


@pytest.mark.parametrize("name", ["local-100", "global-128", "fp32-100", "stream-384"])
def test_guard_bands(name):
    """The weights and their gradient between NaN bands: the same forward bits and d w as on plain buffers, and the bands intact."""
    import torch
    r = Run(name, det=True)
    plain = r.forward()
    g_out = _g_out(r.V, r.D, 15)
    dw_plain = r.backward(g_out)[0]
    M = r.lst.shape[0]
    wbuf, wview = _guarded(M, 0.0)
    wview.copy_(_cuda(r.w))
    r.dev.set_message_weights(wview)
    np.testing.assert_array_equal(r.forward(), plain)
    gbuf, gview = _guarded(M, 0.25)
    r.backward(g_out, dw_buf=gview)
    want = (torch.from_numpy(dw_plain) + torch.tensor(0.25)).numpy()
    np.testing.assert_array_equal(gview.cpu().numpy(), want)
    for buf in (wbuf, gbuf):
        b = buf.cpu().numpy()
        assert np.all(np.isnan(b[:64])) and np.all(np.isnan(b[-64:]))


@pytest.mark.parametrize("name", ["local-100", "fp32-100", "stream-256"])
def test_nan_component_stays_in_its_rows(name):
    """The first component's h0 rows, weights and d_out rows NaN: every other node's final state and d h0, and every other entry's d w,
    are finite and equal the run with that component finite."""
    rng = np.random.default_rng(16)
    sizes = [int(x) for x in rng.integers(2, 40, 30)]
    V, lst, w = G.component_list(sizes, rng)
    first = np.zeros(V, bool)
    first[:sizes[0]] = True
    poison = first[lst[:, 0]]
    results = []
    for poisoned in (False, True):
        r = Run(name, det=True, V=V, lst=lst, w=np.where(poison, np.nan, w) if poisoned else w)
        if poisoned:
            r.h0[first] = np.nan
            r.th0 = _cuda(r.h0)
        out = r.forward()
        g_out = _g_out(V, r.D, 17)
        if poisoned:
            g_out[first] = np.nan
        dw, dh0, _ = r.backward(g_out)
        results.append((out[~first], dh0[~first], dw[~poison]))
    for a, b, what in zip(results[0], results[1], ("state", "d h0", "d w")):
        assert np.all(np.isfinite(b)), what
        if PLANS[name][1] == "fp32":
            np.testing.assert_array_equal(b, a, err_msg=what)
        else:
            assert max_rel_err(b, a) < 1e-6, (what, max_rel_err(b, a))


# ---------------------------------------------------------------------------------------------------------------- end to end
def test_learned_normalization_end_to_end():
    """theta [E] per undirected edge; the reference's normalization  D^-1/2 (A+I) D^-1/2  with A's entries softplus(theta), computed in
    torch, weighs the entries through ``chem_gcn.propagate``; then a sum readout per graph and a squared loss.  theta's gradient (and h0's
    and the layers') against a float64 all-torch restatement."""
    import torch
    from gated_graph_neural_network_samples_b200.chem_gcn import propagate
    from gated_graph_neural_network_samples_b200.engine import GCNEngine
    rng = np.random.default_rng(18)
    D, L = 100, 3
    sizes = [int(x) for x in rng.integers(3, 30, 24)]
    V = sum(sizes)
    gid = np.repeat(np.arange(len(sizes)), sizes)
    edges, off = [], 0
    for n in sizes:   # a path and a few chords per graph
        e = [(off + i, off + i + 1) for i in range(n - 1)] + [tuple(sorted(off + rng.choice(n, 2, replace=False))) for _ in range(n // 3)]
        edges += e
        off += n
    E = np.array(edges, np.int64)
    lst = np.concatenate([E, E[:, ::-1], np.stack([np.arange(V), np.arange(V)], 1)])   # both directions, then the self-loops
    perm = rng.permutation(lst.shape[0])
    lst = np.ascontiguousarray(lst[perm])
    theta0 = rng.normal(0, 0.5, E.shape[0])
    ks, bs = weights(D, L, True, 19)
    h0 = rng.normal(0, 1, (V, D)).astype(np.float32)
    target = rng.normal(0, 1, len(sizes))

    def loss_of(theta, h0t, prop, dev, dtype):
        a = torch.nn.functional.softplus(theta)
        vals = torch.cat([a, a, torch.ones(V, dtype=dtype, device=dev)])[torch.from_numpy(perm).to(dev)]
        rows, cols = torch.from_numpy(lst[:, 0]).to(dev), torch.from_numpy(lst[:, 1]).to(dev)
        deg = torch.zeros(V, dtype=dtype, device=dev).index_add(0, rows, vals)
        w = vals * deg[rows].rsqrt() * deg[cols].rsqrt()
        out = prop(h0t, w)
        pred = torch.zeros(len(sizes), dtype=dtype, device=dev).index_add(0, torch.from_numpy(gid).to(dev), out.sum(1))
        return ((pred - torch.tensor(target, dtype=dtype, device=dev)) ** 2).sum()

    eng = GCNEngine(D, L, use_bias=True, precision="bf16x3")
    eng.set_graph_prepared(eng.prepare_graph_gcn_message_weighted(V, lst, save_for_backward=True))
    tk = [_cuda(k).requires_grad_() for k in ks]
    tb = [_cuda(b).requires_grad_() for b in bs]
    theta = torch.tensor(theta0, dtype=torch.float32, device="cuda", requires_grad=True)
    th0 = _cuda(h0).requires_grad_()
    loss = loss_of(theta, th0, lambda h, w: propagate(eng, h, tk, tb, w), "cuda", torch.float32)
    loss.backward()
    rtheta = torch.tensor(theta0, dtype=torch.float64, requires_grad=True)
    rh0 = torch.tensor(h0, dtype=torch.float64, requires_grad=True)
    rk = [torch.tensor(k, dtype=torch.float64, requires_grad=True) for k in ks]
    rb = [torch.tensor(b, dtype=torch.float64, requires_grad=True) for b in bs]
    rloss = loss_of(rtheta, rh0, lambda h, w: G.gcn_propagation_torch(h, lst, w, rk, rb), "cpu", torch.float64)
    rloss.backward()
    print("\nGCNMW e2e loss %.6e / %.6e  d theta %.2e" % (float(loss), float(rloss), max_rel_err(theta.grad.cpu().numpy(), rtheta.grad.numpy())))
    assert abs(float(loss) - float(rloss)) <= 1e-4 * abs(float(rloss)) + 1e-6
    assert max_rel_err(theta.grad.cpu().numpy(), rtheta.grad.numpy()) < 2e-4
    assert max_rel_err(th0.grad.cpu().numpy(), rh0.grad.numpy()) < 2e-4
    for l in range(L):
        assert max_rel_err(tk[l].grad.cpu().numpy(), rk[l].grad.numpy()) < 2e-4, l
        assert max_rel_err(tb[l].grad.cpu().numpy(), rb[l].grad.numpy()) < 2e-4, l
