"""CPU: every forward kernel instance the engine compiles, and the case of tests/test_gpu_forward_plans.py that launches it.

Each forward kernel family is a set of template instances chosen at run time from the padded hidden size DP, the tile variant and the
precision (``ggnn_engine.cu``: ``GGNN_TC_CASE``, ``GGNN_GCN_CASE``, ``GGNN_TS_PICK``, ``pick_fwd_kernel``, ``gcn_fp32_kernel``).  An
instance no test launches can be wrong, or fail to launch, while the suite passes.  Here:

* the instance inventory is read from the dispatch code itself, so a new case in a dispatch list is seen without editing this file;
* every case of the GPU file is built through the host-only prepare calls at 132 SMs (an H100 SXM) with the case's environment, and the
  instance its plan text names must be the one the case claims;
* the union of the cases must cover every inventoried instance at every precision it serves.  A dispatch case without a test fails here.

The batches are chosen so that the plan does not depend on the SM count: 128-row LOCAL tiles come from components of 65-128 nodes, not
from a batch with more tiles than SMs.  (The weighted dense cases cannot be pinned here: the host-only dense prepare refuses weighted
matrices.  The GPU test checks their plan on the device.)
"""
import functools
import os
import re

import numpy as np
import pytest

from tests import gcn_oracle as G
from tests.test_backward_plans_cpu import dense_batch, dense_params, model, sparse_batch  # noqa: F401  (dense_batch: used by the GPU file)

NUM_SMS = 132
ENGINE_CU = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "gated_graph_neural_network_samples_b200", "csrc",
                         "ggnn_engine.cu")
HIDDEN_SIZES = list(range(4, 257, 4))       # every hidden size the ABI accepts
WGMMA_PRECISIONS = ("bf16x3", "bf16")

FORCE_GLOBAL = {"GGNN_FORCE_GLOBAL": "1"}
FORCE_STREAM = {"GGNN_TC_STREAM": "1"}


# ---------------------------------------------------------------------------------------------------------------- the inventory
@functools.lru_cache(maxsize=None)
def _source():
    with open(ENGINE_CU) as f:
        return f.read()


def inventory():
    """The instances the dispatch code compiles, as the instance tuples ``instance_of_plan`` returns."""
    src = _source()
    tc_nh = [int(n) for n in re.findall(r"GGNN_TC_CASE\((\d+)\)", src)]
    gcn_nh = [int(n) for n in re.findall(r"GGNN_GCN_CASE\((\d+)\)", src)]
    ts = [(x == "true", int(k)) for x, k in re.findall(r"GGNN_TS_PICK\((true|false),\s*(\d+)\)", src)]
    body = re.search(r"FwdKernel pick_fwd_kernel\(.*?\n}\n", src, re.S)
    ffma = [(int(rg), int(cs), int(nb1), loc == "true")
            for rg, cs, nb1, loc in re.findall(r"fwd_kernel_ptr<(\d+),\s*(\d+),\s*(\d+),\s*(true|false)>", body.group(0) if body else "")]
    gcn_fp32 = re.findall(r"gcn::gcn_fp32_kernel<<<", src)
    return {"tc": tc_nh, "gcn": gcn_nh, "stream": ts, "ffma": ffma, "gcn-fp32": gcn_fp32}


def required_instances():
    inv = inventory()
    req = {("tc", loc, nh, p) for nh in inv["tc"] for loc in (True, False) for p in WGMMA_PRECISIONS}
    req |= {("gcn", loc, nh, p) for nh in inv["gcn"] for loc in (True, False) for p in WGMMA_PRECISIONS}
    req |= {("stream", x3, ks) for x3, ks in inv["stream"]}
    req |= {("ffma",) + t for t in inv["ffma"]}
    if inv["gcn-fp32"]:
        req.add(("gcn-fp32",))
    return req


# ---------------------------------------------------------------------------------------------------------------- plan text -> instance
def stream_ksteps(DP, env):
    """K-steps per ring stage of the streaming kernels, as ``forward_stream`` chooses it: the largest of 4 / 2 / 1 (at most
    ``GGNN_TS_KSTEPS``) that divides the DP / 16 K-steps of a segment."""
    ks = 4
    if env.get("GGNN_TS_KSTEPS") is not None:
        v = int(env["GGNN_TS_KSTEPS"])
        ks = 4 if v >= 4 else (2 if v >= 2 else 1)
    while (DP // 16) % ks:
        ks //= 2
    return ks


def instance_of_plan(plan, env):
    """The kernel instance a plan text launches: ``("tc", LOCAL, NH, precision)``, ``("stream", X3, KS)``, ``("ffma", RG, CS, NB1, LOCAL)``,
    ``("gcn", LOCAL, NH, precision)`` or ``("gcn-fp32",)``.  Raises on a plan text it cannot read."""
    m = re.match(r"^wgmma-(bf16x3|bf16) (LOCAL|GLOBAL)\(.* DP=(\d+) ", plan)
    if m:
        return ("tc", m.group(2) == "LOCAL", int(m.group(3)) // 2, m.group(1))
    m = re.match(r"^wgmma-(bf16x3|bf16) STREAM\(.* DP=(\d+) ", plan)
    if m:
        return ("stream", m.group(1) == "bf16x3", stream_ksteps(int(m.group(2)), env))
    m = re.match(r"^fp32-ffma(?:\+attention)?(?:\+cudnn-gru)? (LOCAL|GLOBAL)\(.* rows/tile<=(\d+) warps=(\d+) colsplit=(\d+) nb1=(\d+) ", plan)
    if m:
        rows, warps = int(m.group(2)), int(m.group(3))
        return ("ffma", rows // warps, int(m.group(4)), int(m.group(5)), m.group(1) == "LOCAL")
    m = re.match(r"^gcn-wgmma-(bf16x3|bf16) (LOCAL|GLOBAL)\(.* DP=(\d+) ", plan)
    if m:
        return ("gcn", m.group(2) == "LOCAL", int(m.group(3)) // 2, m.group(1))
    if plan.startswith("gcn-fp32-ffma GLOBAL("):
        return ("gcn-fp32",)
    raise ValueError("unrecognised plan text: %r" % plan)


def pad16(D):
    return (D + 15) // 16 * 16


# ---------------------------------------------------------------------------------------------------------------- batches
def sized_components(sizes, edges, T, seed):
    """Components of ``sizes`` nodes, component i a random spanning tree plus random distinct extra pairs up to ``edges[i]`` undirected
    edges, each in both directions, with types uniform over ``T`` (every type occurs).  Reference wire format, like component_graph."""
    rng = np.random.default_rng(seed)
    und, off = [], 0
    for n, m in zip(sizes, edges):
        pairs = {(int(rng.integers(0, i)), i) for i in range(1, n)}
        m = min(m, n * (n - 1) // 2)
        while len(pairs) < m:
            a, b = sorted(int(x) for x in rng.choice(n, 2, replace=False))
            pairs.add((a, b))
        und += [(off + a, off + b) for a, b in sorted(pairs)]
        off += n
    types = rng.integers(0, T, len(und))
    types[:T] = np.arange(T)
    adj = []
    for t in range(T):
        e = np.asarray([u for u, k in zip(und, types) if k == t], np.int32).reshape(-1, 2)
        adj.append(np.concatenate([e, e[:, ::-1]], axis=0).astype(np.int32))
    indeg = np.zeros((off, T), np.float32)
    for t, a in enumerate(adj):
        np.add.at(indeg[:, t], a[:, 1], 1.0)
    return adj, indeg


# components of 65-128 nodes: whole-component LOCAL tiles of more than 64 rows (2048-byte k-group stride) on any SM count above 5
BIG_SIZES = (120, 90, 70, 100, 66)
# one 100-node component with 2200 undirected edges: a tile with 4400 messages, above the 4096 of the shared-memory CSR cache
MSG_SIZES, MSG_EDGES = (100, 40, 30, 20), (2200, 80, 60, 40)
CSR_CACHE_MSGS = 4096


def graph(kind, T):
    """(adjacency lists, in-degree table) of a batch kind: ``mol24`` (24 synthetic molecules), ``comp`` (component_graph(T)),
    ``big`` (components of 66-120 nodes), ``msgs`` (a tile with more than 4096 messages)."""
    if kind in ("mol24", "comp"):
        adj, indeg, _ = sparse_batch(kind, 4, T)
        return adj, indeg
    if kind == "big":
        return sized_components(BIG_SIZES, [2 * n for n in BIG_SIZES], T, 40 + T)
    if kind == "msgs":
        return sized_components(MSG_SIZES, MSG_EDGES, T, 50 + T)
    raise ValueError(kind)


def h0_for(V, D, seed=0):
    return np.random.default_rng(1000 + 7 * D + seed).normal(0, 1, (V, D)).astype(np.float32)


GCN_LAYERS = 3


def gcn_graph(D, kind):
    """(V, [nnz, 2] list, [nnz] weights): ``components`` = 40 components of 3-29 nodes (LOCAL), ``random`` = one graph over 300 nodes
    (GLOBAL: a component larger than a tile)."""
    rng = np.random.default_rng(3 + D)
    if kind == "components":
        V, lst, w = G.component_list(list(rng.integers(3, 30, 40)), rng)
    else:
        V = 300
        lst, w = G.random_gcn_list(V, 2000, rng, isolated=(0, 7))
    return V, lst, w


# ---------------------------------------------------------------------------------------------------------------- the cases
class Case:
    """One forward of the GPU file.  ``kind``: ``sparse`` (GGNN on a batch kind), ``dense`` (weighted dense matrix, weighted CSR) or
    ``gcn``.  ``instance``: the kernel instance the case claims; ``keep``: state-dropout keep probability."""

    def __init__(self, name, kind, params, T, batch, precision, env, instance, keep=1.0):
        self.name, self.kind, self.params, self.T, self.batch = name, kind, params, T, batch
        self.precision, self.env, self.instance, self.keep = precision, dict(env), instance, keep

    @property
    def D(self):
        return self.params["hidden_size"]

    def __repr__(self):
        return self.name


def _cell(D):
    """GRU and RNN alternate with the hidden size, so that each DP class (four hidden sizes) sees both."""
    return "GRU" if (D // 4) % 2 else "RNN"


def _act(cell):
    return "tanh" if cell == "GRU" else "ReLU"


def sweep_model(D, cell=None):
    cell = cell or _cell(D)
    return model(cell, D, act=_act(cell), avg=True)


def _sweep_cases():
    """a. Every hidden size: bf16x3 on its default plan (LOCAL up to DP 128, STREAM above), fp32 on tile variant 0 (D <= 128) and 1."""
    out = []
    for D in HIDDEN_SIZES:
        p = sweep_model(D)
        if pad16(D) <= 128:
            inst = ("tc", True, pad16(D) // 2, "bf16x3")
        else:
            inst = ("stream", True, stream_ksteps(pad16(D), {}))
        out.append(Case("sweep-D%d-bf16x3" % D, "sparse", p, 4, "mol24", "bf16x3", {}, inst))
        for v, (rg, cs, per) in enumerate(((8, 1, 32), (4, 2, 64))):
            if v == 0 and D > 128:
                continue
            nb1 = next(n for n in (1, 2, 4) if D <= n * per)
            out.append(Case("sweep-D%d-fp32-v%d" % (D, v), "sparse", p, 4, "mol24", "fp32", {"GGNN_FFMA_VARIANT": str(v)},
                            ("ffma", rg, cs, nb1, True)))
    return out


def _tile_cases():
    """b. The tile-local wgmma kernel per NH = DP / 2, at D = DP and D = DP - 4 in turn (a column tail inside the last 16)."""
    out = []
    for i, nh in enumerate(range(8, 65, 8)):
        DP = 2 * nh
        Da, Db = DP, max(DP - 4, 4)     # (DP 16: D 16 and 12)
        g = lambda D, cell="GRU", **kw: model(cell, D, act=_act(cell), avg=True, **kw)
        tc = lambda loc, prec="bf16x3": ("tc", loc, nh, prec)
        out += [
            Case("tc-nh%d-local-compact-D%d" % (nh, Da), "sparse", g(Da), 4, "mol24", "bf16x3", {}, tc(True)),
            Case("tc-nh%d-local-128-D%d" % (nh, Db), "sparse", g(Db, "RNN"), 4, "big", "bf16x3", {}, tc(True)),
            Case("tc-nh%d-global-D%d" % (nh, Db), "sparse", g(Db), 4, "mol24", "bf16x3", FORCE_GLOBAL, tc(False)),
            Case("tc-nh%d-bf16-local-D%d" % (nh, Db), "sparse", g(Db), 4, "mol24", "bf16", {}, tc(True, "bf16")),
            Case("tc-nh%d-bf16-global-D%d" % (nh, Da), "sparse", g(Da, "RNN"), 4, "mol24", "bf16", FORCE_GLOBAL, tc(False, "bf16")),
            Case("tc-nh%d-T17-D%d" % (nh, Da), "sparse", g(Da, "RNN"), 17, "comp", "bf16x3", {}, tc(True)),
            Case("tc-nh%d-T32-D%d" % (nh, Db), "sparse", g(Db), 32, "comp", "bf16x3", {}, tc(True)),
            Case("tc-nh%d-msgs4k-D%d" % (nh, Da), "sparse", g(Da), 4, "msgs", "bf16x3", {}, tc(True)),
            Case("tc-nh%d-dropout-D%d" % (nh, Db), "sparse", g(Db, "RNN" if i % 2 else "GRU"), 4, "mol24", "bf16x3", {}, tc(True), keep=0.8),
            Case("tc-nh%d-dense-D%d" % (nh, Da), "dense", dense_params(Da), 4, "dense", "bf16x3", {}, tc(True)),
        ]
    return out


def _stream_cases():
    """c. The streaming kernels: each (X3, KS) pair with GRU and RNN at a hidden size whose DP is not a multiple of 128 (KS 1: DP 144,
    KS 2: DP 160, KS 4: DP 192); T = 32 and dropout; forced streaming at small DP (KS 2: DP 32, KS 1: DP 48); GGNN_TS_KSTEPS below the
    natural KS at hidden 256."""
    out = []
    for prec in WGMMA_PRECISIONS:
        x3 = prec == "bf16x3"
        for D, ks in ((132, 1), (148, 2), (180, 4)):
            for cell in ("GRU", "RNN"):
                out.append(Case("stream-%s-ks%d-%s-D%d" % (prec, ks, cell.lower(), D), "sparse", sweep_model(D, cell), 4, "mol24", prec, {},
                                ("stream", x3, ks)))
        for D, ks in ((20, 2), (40, 1)):
            out.append(Case("stream-%s-forced-ks%d-D%d" % (prec, ks, D), "sparse", sweep_model(D, "GRU"), 4, "mol24", prec, FORCE_STREAM,
                            ("stream", x3, ks)))
        out.append(Case("stream-%s-T32-D148" % prec, "sparse", sweep_model(148, "GRU"), 32, "comp", prec, {}, ("stream", x3, 2)))
        out.append(Case("stream-%s-dropout-D132" % prec, "sparse", sweep_model(132, "RNN"), 4, "mol24", prec, {}, ("stream", x3, 1), keep=0.8))
        for ks in (2, 1):
            out.append(Case("stream-%s-ksteps%d-D256" % (prec, ks), "sparse", sweep_model(256, "GRU"), 4, "mol24", prec,
                            {"GGNN_TS_KSTEPS": str(ks)}, ("stream", x3, ks)))
    return out


def _ffma_cases():
    """d. The fp32 kernel: all (variant, nb1, LOCAL / GLOBAL) instances with GRU / tanh and RNN / ReLU, and CudnnCompatibleGRUCell and
    attention on each of them."""
    out = []
    for v, (rg, cs, sizes) in enumerate(((8, 1, (28, 60, 100)), (4, 2, (44, 116, 196)))):
        for nb1, D in zip((1, 2, 4), sizes):
            for loc in (True, False):
                env = {"GGNN_FFMA_VARIANT": str(v)}
                env.update({} if loc else FORCE_GLOBAL)
                tag = "ffma-v%d-nb%d-%s" % (v, nb1, "local" if loc else "global")
                inst = ("ffma", rg, cs, nb1, loc)
                out += [Case("%s-gru-D%d" % (tag, D), "sparse", model("GRU", D, act="tanh", avg=True), 4, "mol24", "fp32", env, inst),
                        Case("%s-rnn-D%d" % (tag, D), "sparse", model("RNN", D, act="ReLU"), 4, "mol24", "fp32", env, inst),
                        Case("%s-cudnn-D%d" % (tag, D), "sparse", model("CudnnCompatibleGRUCell", D, act="tanh", avg=True), 4, "mol24", "fp32",
                             env, inst),
                        Case("%s-attention-D%d" % (tag, D), "sparse", model("GRU", D, act="tanh", attention=True), 4, "mol24", "fp32", env, inst)]
    return out


def _gcn_cases():
    """e. The GCN: every wgmma instance (NH x LOCAL / GLOBAL) at bf16x3 and bf16, and every hidden size at bf16x3 (wgmma up to DP 128,
    the fp32 kernel above) and fp32."""
    out = []
    for nh in range(8, 65, 8):
        for i, prec in enumerate(WGMMA_PRECISIONS):
            D = 2 * nh - 4 * i
            out += [Case("gcn-nh%d-%s-local-D%d" % (nh, prec, D), "gcn", {"hidden_size": D}, 1, "components", prec, {}, ("gcn", True, nh, prec)),
                    Case("gcn-nh%d-%s-global-D%d" % (nh, prec, D), "gcn", {"hidden_size": D}, 1, "random", prec, {}, ("gcn", False, nh, prec))]
    for D in HIDDEN_SIZES:
        inst = ("gcn", True, pad16(D) // 2, "bf16x3") if pad16(D) <= 128 else ("gcn-fp32",)
        out.append(Case("gcn-sweep-D%d-bf16x3" % D, "gcn", {"hidden_size": D}, 1, "components", "bf16x3", {}, inst))
        out.append(Case("gcn-sweep-D%d-fp32" % D, "gcn", {"hidden_size": D}, 1, "components", "fp32", {}, ("gcn-fp32",)))
    out.append(Case("gcn-fp32-dropout-D100", "gcn", {"hidden_size": 100}, 1, "random", "fp32", {}, ("gcn-fp32",), keep=0.8))
    out.append(Case("gcn-nh48-dropout-D92", "gcn", {"hidden_size": 92}, 1, "components", "bf16x3", {}, ("gcn", True, 48, "bf16x3"), keep=0.8))
    return out


SWEEP, TILE, STREAM, FFMA, GCN = _sweep_cases(), _tile_cases(), _stream_cases(), _ffma_cases(), _gcn_cases()
CASES = {c.name: c for c in SWEEP + TILE + STREAM + FFMA + GCN}
assert len(CASES) == len(SWEEP + TILE + STREAM + FFMA + GCN), "duplicate case names"
PINNABLE = sorted(n for n, c in CASES.items() if c.kind != "dense")


@functools.lru_cache(maxsize=None)
def host_plan(name):
    """The plan text of a case, from the host-only prepare call at 132 SMs under the case's environment."""
    from gated_graph_neural_network_samples_b200.engine import PreparedGraph
    c = CASES[name]
    saved = {k: os.environ.get(k) for k in c.env}
    os.environ.update(c.env)
    try:
        if c.kind == "gcn":
            V, lst, w = gcn_graph(c.D, c.batch)
            g = PreparedGraph.host_only_gcn(c.D, GCN_LAYERS, V, lst, w, use_bias=True, precision=c.precision, num_sms=NUM_SMS)
        else:
            adj, indeg = graph(c.batch, c.T)
            g = PreparedGraph.host_only(c.params, c.T, adj, indeg, precision=c.precision, num_sms=NUM_SMS)
        return g.info()
    finally:
        for k, v in saved.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


# ---------------------------------------------------------------------------------------------------------------- tests
def test_inventory_is_read_from_the_dispatch_code():
    """A renamed macro or kernel must fail here, not leave an empty inventory that every case set covers."""
    inv = inventory()
    assert inv["tc"] == [8, 16, 24, 32, 40, 48, 56, 64], inv["tc"]
    assert inv["gcn"] == [8, 16, 24, 32, 40, 48, 56, 64], inv["gcn"]
    assert sorted(inv["stream"]) == [(False, 1), (False, 2), (False, 4), (True, 1), (True, 2), (True, 4)], inv["stream"]
    assert len(inv["ffma"]) == 12 and len(set(inv["ffma"])) == 12, inv["ffma"]
    assert {(rg, cs) for rg, cs, _, _ in inv["ffma"]} == {(8, 1), (4, 2)}
    assert len(inv["gcn-fp32"]) == 1
    assert len(required_instances()) == 16 * 2 + 16 * 2 + 6 + 12 + 1


@pytest.mark.parametrize("name", PINNABLE)
def test_case_reaches_its_instance(name):
    c = CASES[name]
    plan = host_plan(name)["plan"]
    assert instance_of_plan(plan, c.env) == c.instance, (c.instance, plan)


def test_every_instance_is_launched_by_a_case():
    covered = {instance_of_plan(host_plan(n)["plan"], CASES[n].env) for n in PINNABLE}
    missing = sorted(required_instances() - covered, key=str)
    assert not missing, "compiled forward instances no case launches: %s" % missing


def test_batches_have_the_shapes_the_cases_claim():
    """The 128-row tiles come from components of 65-128 nodes; the message-heavy batch has a tile above the CSR cache's 4096 messages;
    the molecule batch fits the LOCAL tiles of both fp32 variants (components of at most 32 nodes)."""
    from gated_graph_neural_network_samples_b200.engine import PreparedGraph
    p = model("GRU", 100)
    adj, indeg = graph("big", 4)
    plan = PreparedGraph.host_only(p, 4, adj, indeg, precision="bf16x3", num_sms=NUM_SMS).info()["plan"]
    budget = int(re.search(r"rows/tile<=(\d+)", plan).group(1))
    assert 64 < budget <= 128 and "compact" not in plan, plan
    adj, indeg = graph("msgs", 4)
    g = PreparedGraph.host_only(p, 4, adj, indeg, precision="bf16x3", num_sms=NUM_SMS)
    a = g.arrays(4)
    ts, rp = a["tile_start"], a["row_ptr"]
    tile_msgs = [rp[ts[i + 1] * 4] - rp[ts[i] * 4] for i in range(len(ts) - 1)]
    assert max(tile_msgs) > CSR_CACHE_MSGS, tile_msgs
    assert int(re.search(r"max_component=(\d+)", host_plan("sweep-D100-fp32-v1")["plan"]).group(1)) <= 32
    for T in (17, 32):
        adj, _ = graph("comp", T)
        assert all(x.shape[0] > 0 for x in adj)    # every type occurs: type 31 sets the top bit of the 32-bit tile mask


def test_instance_of_plan_reads_every_plan_family():
    assert instance_of_plan("wgmma-bf16 GLOBAL(1 launch per step) tiles=3 rows/tile<=128 DP=80 max_component=30", {}) == ("tc", False, 40, "bf16")
    assert instance_of_plan("wgmma-bf16x3 STREAM(3 launches) tiles=3 DP=160 N-blocks agg/cand=2x128 gate=3x128", {}) == ("stream", True, 2)
    assert instance_of_plan("wgmma-bf16x3 STREAM(3 launches) tiles=3 DP=256 N-blocks x", {"GGNN_TS_KSTEPS": "1"}) == ("stream", True, 1)
    with pytest.raises(ValueError):
        instance_of_plan("something else", {})
    assert [stream_ksteps(dp, {}) for dp in (16, 32, 48, 64, 144, 160, 192, 208, 256)] == [1, 2, 1, 4, 1, 2, 4, 1, 4]
