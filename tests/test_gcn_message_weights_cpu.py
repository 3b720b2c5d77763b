"""CPU: adjacency weights on the device in the sparse GCN model (ggnn_prepare_graph_gcn_message_weighted, ggnn_set_message_weights on a
GCN engine, ggnn_gcn_backward_weighted).

A message-weighted GCN batch is the GCN batch without host weights: they arrive on the device after the upload.  Without a GPU this file
checks:

* the three entries: exported, declared in include/ggnn_b200.h with the argument count the ctypes binding gives them;
* the host-only image (``PreparedGraph.host_only_gcn_message_weighted``) against ``ggnn_host_prepare_graph_gcn``'s image of the same list
  with zero weights, at hidden 12 / 100 / 128 on bf16x3, 256 on fp32 and 512 with ``wide_hidden``, with and without the source-keyed CSR:
  the same bytes, but for the source-CSR -> target-slot map (``tslot``) a backward image adds, which equals its NumPy restatement; CSR,
  ``msg`` and tiles are those of the ordinary prepare; the slot weights are zero; the image bytes are the same at 1, 2, 3 and 8 host threads;
* the plan texts of every GCN plan (LOCAL, GLOBAL, fp32, stream): the ordinary ones with " [message-weighted]" appended;
* the float64 gradient the GPU tests compare against: autograd through ``tests/gcn_oracle.gcn_propagation_torch`` with a weight leaf is
  the loop statement  d w_k = sum_l <dS_l[i_k], H_l[j_k]>;
* the new kernel's instances use no stack and spill nothing.
"""
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

from tests import gcn_oracle as G

NUM_SMS = 132
TAG = " [message-weighted]"
ENTRIES = ("ggnn_prepare_graph_gcn_message_weighted", "ggnn_host_prepare_graph_gcn_message_weighted", "ggnn_gcn_backward_weighted")
# (hidden size, precision, wide_hidden): the wgmma kernel at three widths, the fp32 kernel, the streaming plan
SHAPES = [(12, "bf16x3", False), (100, "bf16x3", False), (128, "bf16x3", False), (256, "fp32", False), (512, "bf16x3", True)]
HOST_THREADS = (1, 2, 3, 8)


def batch(seed=0, sizes=(5, 30, 64, 17, 100, 3, 41)):
    """(V, list, weights): disjoint components with self-loops, shuffled, plus duplicates and an isolated node at the end."""
    rng = np.random.default_rng(seed)
    V, lst, w = G.component_list(list(sizes), rng)
    lst = np.concatenate([lst, lst[:7]])   # duplicate entries
    return V + 1, lst, np.concatenate([w, w[:7]])


def prepare(D, precision, wide, V, lst, w=None, save=False, L=3):
    """The message-weighted host-only prepare (``w`` None), else the ordinary one with host weights ``w``."""
    from gated_graph_neural_network_samples_b200.engine import PreparedGraph
    if w is None:
        return PreparedGraph.host_only_gcn_message_weighted(D, L, V, lst, use_bias=True, precision=precision, num_sms=NUM_SMS,
                                                            save_for_backward=save, wide_hidden=wide)
    return PreparedGraph.host_only_gcn(D, L, V, lst, w, use_bias=True, precision=precision, num_sms=NUM_SMS, save_for_backward=save,
                                       wide_hidden=wide)


def expected_tslot(lst):
    """The target-CSR slot of every source-CSR entry: slots are the list sorted stably by output row i, source entries the list sorted
    stably by input column j."""
    lst = np.asarray(lst, np.int64).reshape(-1, 2)
    by_target = np.argsort(lst[:, 0], kind="stable")
    slot_of = np.empty(lst.shape[0], np.int64)
    slot_of[by_target] = np.arange(lst.shape[0])
    return slot_of[np.argsort(lst[:, 1], kind="stable")].astype(np.int32)


def _find(haystack, needle):
    """Byte offsets of ``needle`` in ``haystack`` (uint8 arrays), at 4-byte alignment."""
    h = haystack[: haystack.size // 4 * 4].view(np.int32)
    n = needle.view(np.int32)
    starts = np.nonzero(h[: h.size - n.size + 1] == n[0])[0]
    return [4 * int(s) for s in starts if np.array_equal(h[s:s + n.size], n)]


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
    # ggnn_gcn_backward_weighted is ggnn_gcn_backward with one more argument, before the stream; the prepare calls are the ordinary ones
    # without the weights
    bw, b = _lib.SYMBOLS["ggnn_gcn_backward_weighted"][1], _lib.SYMBOLS["ggnn_gcn_backward"][1]
    assert bw[:5] == b[:5] and bw[-1] == b[-1] and len(bw) == len(b) + 1
    for name in ("ggnn_prepare_graph_gcn", "ggnn_host_prepare_graph_gcn"):
        mw, plain = _lib.SYMBOLS[name + "_message_weighted"][1], _lib.SYMBOLS[name][1]
        assert mw == plain[:-2] + plain[-1:], name


# ---------------------------------------------------------------------------------------------------------------- the image
@pytest.mark.parametrize("save", [False, True])
@pytest.mark.parametrize("D,precision,wide", SHAPES)
def test_image_is_the_ordinary_batch_with_zero_weights(D, precision, wide, save):
    V, lst, w = batch(D)
    g = prepare(D, precision, wide, V, lst, save=save)
    u = prepare(D, precision, wide, V, lst, w, save=save)
    z = prepare(D, precision, wide, V, lst, np.zeros_like(w), save=save)
    gi, ui = g.info(), u.info()
    assert gi["plan"] == ui["plan"] + TAG, (gi["plan"], ui["plan"])
    assert gi["num_messages"] == ui["num_messages"] == lst.shape[0]
    assert gi["num_tiles"] == ui["num_tiles"] and gi["streaming"] == ui["streaming"]
    ga, ua = g.arrays(1), u.arrays(1)
    for k in ("row_ptr", "src", "msg", "tile_start", "denom"):
        np.testing.assert_array_equal(ga[k], ua[k], err_msg=k)
    np.testing.assert_array_equal(ga["msg"], np.argsort(lst[:, 0], kind="stable"))
    np.testing.assert_array_equal(g.slot_weights(), np.zeros(lst.shape[0], np.float32))
    np.testing.assert_array_equal(u.slot_weights(), w[ga["msg"]])
    gimg, zimg = g.image(), z.image()
    if not save:   # no source-keyed CSR: the zero-weight ordinary image, byte for byte
        np.testing.assert_array_equal(gimg, zimg)
        return
    np.testing.assert_array_equal(g.slot_weights(source_order=True), np.zeros(lst.shape[0], np.float32))
    # with it: the zero-weight ordinary image with one more section, tslot, placed behind the source CSR
    tslot = expected_tslot(lst)
    extra = gimg.size - zimg.size
    assert extra == (tslot.nbytes + 15) // 16 * 16, extra   # sections are 16-byte aligned
    hits = _find(gimg, tslot.view(np.uint8))
    assert len(hits) == 1, hits
    off = hits[0]
    np.testing.assert_array_equal(gimg[:off], zimg[:off])
    np.testing.assert_array_equal(gimg[off + extra:], zimg[off:])
    assert not gimg[off + tslot.nbytes:off + extra].any()


@pytest.mark.parametrize("D,precision,wide", [(100, "bf16x3", False), (256, "fp32", False), (512, "bf16x3", True)])
def test_image_bytes_do_not_depend_on_host_threads(D, precision, wide, monkeypatch):
    from tests.test_gcn_tiles_cpu import batch as tiles_batch
    V, lst, _ = tiles_batch("mol1200")
    images = []
    for n in HOST_THREADS:
        monkeypatch.setenv("GGNN_HOST_THREADS", str(n))
        images.append(prepare(D, precision, wide, V, lst, save=True).image())
    for n, img in zip(HOST_THREADS[1:], images[1:]):
        np.testing.assert_array_equal(img, images[0], err_msg="%d host threads" % n)


def test_plan_texts_on_every_gcn_plan(monkeypatch):
    monkeypatch.delenv("GGNN_FORCE_GLOBAL", raising=False)
    from tests.test_gcn_tiles_cpu import batch as tiles_batch
    expect = [("span64", 100, "bf16x3", False, r"^gcn-wgmma-bf16x3 LOCAL\("), ("span129", 128, "bf16x3", False, r"^gcn-wgmma-bf16x3 GLOBAL\("),
              ("span64", 100, "bf16", False, r"^gcn-wgmma-bf16 LOCAL\("), ("span64", 100, "fp32", False, r"^gcn-fp32-ffma GLOBAL\("),
              ("span64", 256, "bf16x3", False, r"^gcn-fp32-ffma GLOBAL\("), ("span129", 384, "bf16x3", True, r"^gcn-stream-bf16x3 \(")]
    for name, D, precision, wide, pat in expect:
        V, lst, w = tiles_batch(name)
        for save in (False, True):
            plan = prepare(D, precision, wide, V, lst, save=save).info()["plan"]
            assert re.match(pat, plan) and plan == prepare(D, precision, wide, V, lst, w, save=save).info()["plan"] + TAG, (name, D, plan)


def test_refusals_of_the_host_prepare():
    from gated_graph_neural_network_samples_b200.engine import GgnnError
    with pytest.raises(GgnnError, match="out of range"):
        prepare(100, "bf16x3", False, 4, np.array([[0, 1], [2, 4]], np.int64))
    with pytest.raises(GgnnError, match="out of range"):
        prepare(100, "bf16x3", False, 4, np.array([[-1, 1]], np.int64))
    g = prepare(100, "bf16x3", False, 6, np.zeros((0, 2), np.int64), save=True)   # nnz = 0
    assert g.info()["num_messages"] == 0 and g.info()["plan"].endswith(TAG)


# ---------------------------------------------------------------------------------------------------------------- the float64 gradient
def loop_gradient(h0, lst, w, ks, bs, g_out, masks=None, keep=1.0):
    """d w by the loop statement: the float64 forward keeping every layer input H_l and pre-activation, then per layer in reverse
    dPre_l, dS_l = dPre_l . W_l^T, d w_k += <dS_l[i_k], H_l[j_k]> and dH_l = A^T dS_l."""
    L = len(ks)
    H, pre = [np.asarray(h0, np.float64)], []
    for l in range(L):
        s = np.zeros_like(H[-1])
        for k in range(lst.shape[0]):
            s[lst[k, 0]] += w[k] * H[-1][lst[k, 1]]
        p = s @ ks[l] + bs[l]
        pre.append(p)
        h = p
        if l < L - 1:
            h = np.maximum(p, 0.0)
            if masks is not None:
                h = h * masks[l] / np.float64(np.float32(keep))
        H.append(h)
    dw = np.zeros(lst.shape[0])
    dh = np.asarray(g_out, np.float64)
    for l in range(L - 1, -1, -1):
        dpre = dh
        if l < L - 1:
            dpre = dh * (pre[l] > 0)
            if masks is not None:
                dpre = dpre * masks[l] / np.float64(np.float32(keep))
        dS = dpre @ ks[l].T
        for k in range(lst.shape[0]):
            dw[k] += dS[lst[k, 0]] @ H[l][lst[k, 1]]
        dh = np.zeros_like(dh)
        for k in range(lst.shape[0]):
            dh[lst[k, 1]] += w[k] * dS[lst[k, 0]]
    return dw


@pytest.mark.parametrize("L,keep", [(1, 1.0), (3, 1.0), (3, 0.7)])
def test_autograd_through_the_torch_oracle_is_the_loop_statement(L, keep):
    import torch
    rng = np.random.default_rng(L)
    V, lst, w = batch(L, sizes=(4, 7, 1, 9))
    lst = np.concatenate([lst, [[2, 3]]])   # one entry whose transpose is not in the list
    w = np.concatenate([w, [-0.5]]).astype(np.float32)
    w[::5] = 0.0
    D = 6
    ks = [G.glorot((D, D), rng).astype(np.float64) for _ in range(L)]
    bs = [rng.normal(0, 0.3, D) for _ in range(L)]
    h0 = rng.normal(0, 1, (V, D))
    masks = [(rng.random((V, D)) < keep).astype(np.float64) for _ in range(L - 1)] if keep < 1.0 else None
    g_out = rng.normal(0, 1, (V, D))
    tw = torch.tensor(w, dtype=torch.float64, requires_grad=True)
    out = G.gcn_propagation_torch(torch.tensor(h0), lst, tw, [torch.tensor(k) for k in ks], [torch.tensor(b) for b in bs], masks, keep)
    (out * torch.tensor(g_out)).sum().backward()
    want = loop_gradient(h0, lst, w.astype(np.float64), ks, bs, g_out, masks, keep)
    np.testing.assert_allclose(tw.grad.numpy(), want, rtol=1e-10, atol=1e-12)
    # the orientation: a one-entry list (i, j) = (0, 1) gives d w = <dS[0], H[1]>, not <dS[1], H[0]>
    one = np.array([[0, 1]], np.int64)
    tw1 = torch.tensor([0.7], dtype=torch.float64, requires_grad=True)
    h = torch.tensor(h0[:2])
    out = G.gcn_propagation_torch(h, one, tw1, [torch.tensor(ks[0])])
    (out * torch.tensor(g_out[:2])).sum().backward()
    dS = g_out[:2] @ ks[0].T
    assert abs(float(tw1.grad[0]) - float(dS[0] @ h0[1])) < 1e-12
    assert abs(float(dS[0] @ h0[1]) - float(dS[1] @ h0[0])) > 1e-3


# ---------------------------------------------------------------------------------------------------------------- the kernel
def _cuobjdump():
    exe = shutil.which("cuobjdump")
    if exe is None:
        cand = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "cuobjdump")
        exe = cand if os.path.exists(cand) else None
    return exe


def test_source_grad_kernel_uses_no_stack_and_does_not_spill():
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
            name = m.group(1) if "gcn_source_grad_kernel" in m.group(1) else None
            continue
        if name is not None and "REG:" in line:
            found[name] = {n: int(v) for n, v in re.findall(r"([A-Z_]+):(\d+)", line)}
            name = None
    assert len(found) == 8, sorted(found)   # CHUNKS 1..4, with and without dH
    for k, r in found.items():
        print("%s %s" % (k, r))
        assert r["STACK"] == 0 and r.get("LOCAL", 0) == 0, (k, r)
