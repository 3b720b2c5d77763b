"""CPU-only: the MMA path of the tile kernels as the compiler made it, read from ``cuobjdump`` of the built library (skipped without it).

``gcn_wgmma_kernel<LOCAL, NH, X3>`` and the compact instances of ``ggnn_fwd_tc_kernel<LOCAL, NH, COMPACT, X3>`` issue their wgmma MMAs as
straight-line code -- the precision, DP = 2*NH and every K-step trip count are template constants -- and keep one weight slot's MMA group
in flight (``wgmma.wait_group 1``) while the next slot's MMAs are issued.  Where ptxas cannot keep a wgmma pipeline it serialises every
MMA instead: one ``WARPGROUP.DEPBAR`` after each ``HGMMA``.  The 128-row instances of the tile kernel issue one slot at a time on purpose
(their fragments are twice as wide; a pipelined body only spills more).  Here:

* every GCN instance, and every compact LOCAL instance at NH 8, 16 and 40-64 (cfg2 runs NH 56), has fewer ``WARPGROUP.DEPBAR`` than
  ``HGMMA`` (a GEMM of a single MMA has one of each);
* no 128-row instance, at either precision, has a larger stack frame than the single instance of the build whose MMA path was not yet
  straight-line (``SERIAL_STACK``), but for the few listed in ``SERIAL_STACK_EXCEPTIONS`` (8-48 bytes more); no compact instance a
  larger one than ``COMPACT_STACK``;
* every NH has a bf16x3 and a bf16 instance of each layout, and every compiled instance is launched by a case -- of
  tests/test_forward_plans_cpu.py, or the 128-row LOCAL bf16 cases below (run on the GPU by tests/test_gpu_tile_bf16.py).

Not pipelined: the compact instances at NH 24 and 32.  The compact instances spill: keeping the accumulators of the MMAs in flight
locked, the cfg2 instance needs more than 200 registers per worker thread for a spill-free body, and four worker warpgroups get at most
112 (setmaxnreg, with the producer warpgroup at 32).  COMPACT_STACK holds them at this layout's stack frames.
"""
import functools
import os
import re
import shutil
import subprocess

import pytest

from tests.test_backward_plans_cpu import model
from tests.test_forward_plans_cpu import CASES, NUM_SMS, PINNABLE, Case, graph, host_plan, inventory


def _bf16_128_cases():
    """The 128-row LOCAL tile kernel at bf16 for every NH (components of 66-120 nodes), GRU and RNN alternating, D = DP and DP - 4."""
    out = []
    for i, nh in enumerate(range(8, 65, 8)):
        DP = 2 * nh
        D = DP if i % 2 else max(DP - 4, 4)
        cell = "RNN" if i % 2 else "GRU"
        p = model(cell, D, act="ReLU" if cell == "RNN" else "tanh", avg=True)
        out.append(Case("tc-nh%d-bf16-local-128-D%d" % (nh, D), "sparse", p, 4, "big", "bf16", {}, ("tc", True, nh, "bf16")))
    return out


BF16_128 = {c.name: c for c in _bf16_128_cases()}
assert not set(BF16_128) & set(CASES)


# ---------------------------------------------------------------------------------------------------------------- the binary
def _cuobjdump():
    exe = shutil.which("cuobjdump")
    if exe is None:
        cand = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "cuobjdump")
        exe = cand if os.path.exists(cand) else None
    if exe is None:
        pytest.skip("cuobjdump is not available")
    return exe


def _lib():
    from gated_graph_neural_network_samples_b200 import _build, _lib
    _lib.load()
    return _build.LIB_PATH


def instance_of_symbol(name):
    """``("tc", LOCAL, NH, COMPACT, precision)`` or ``("gcn", LOCAL, NH, precision)`` of a mangled kernel name, else None."""
    m = re.search(r"ggnn_fwd_tc_kernelILb([01])ELi(\d+)ELb([01])ELb([01])EE", name)
    if m:
        return ("tc", m.group(1) == "1", int(m.group(2)), m.group(3) == "1", "bf16x3" if m.group(4) == "1" else "bf16")
    m = re.search(r"gcn_wgmma_kernelILb([01])ELi(\d+)ELb([01])EE", name)
    if m:
        return ("gcn", m.group(1) == "1", int(m.group(2)), "bf16x3" if m.group(3) == "1" else "bf16")
    return None


@functools.lru_cache(maxsize=None)
def resources():
    """{instance: {"REG": n, "STACK": n, ...}} from ``cuobjdump -res-usage``."""
    out = subprocess.run([_cuobjdump(), "-res-usage", _lib()], capture_output=True, text=True, check=True).stdout
    res, key = {}, None
    for line in out.splitlines():
        m = re.match(r"\s*Function (\S+):", line)
        if m:
            key = instance_of_symbol(m.group(1))
            continue
        if key is not None and "REG:" in line:
            res[key] = {n: int(v) for n, v in re.findall(r"([A-Z_]+):(\d+)", line)}
            key = None
    return res


@functools.lru_cache(maxsize=None)
def mma_counts():
    """{instance: (HGMMA count, WARPGROUP.DEPBAR count)} from ``cuobjdump -sass``."""
    proc = subprocess.Popen([_cuobjdump(), "-sass", _lib()], stdout=subprocess.PIPE, text=True)
    counts, key = {}, None
    for line in proc.stdout:
        if "Function :" in line:
            key = instance_of_symbol(line.split("Function :", 1)[1].strip())
            if key is not None:
                counts[key] = [0, 0]
            continue
        if key is not None:
            if "HGMMA." in line:
                counts[key][0] += 1
            elif "WARPGROUP.DEPBAR" in line:
                counts[key][1] += 1
    assert proc.wait() == 0
    return {k: tuple(v) for k, v in counts.items()}


def _plan_instance(plan):
    """The plan text of a tile-kernel case -> the instance as ``instance_of_symbol`` names it (None for the other kernel families)."""
    m = re.match(r"^wgmma-(bf16x3|bf16) (LOCAL|GLOBAL)\(.* DP=(\d+) ", plan)
    if m:
        return ("tc", m.group(2) == "LOCAL", int(m.group(3)) // 2, "compact 64-row operand tiles" in plan, m.group(1))
    m = re.match(r"^gcn-wgmma-(bf16x3|bf16) (LOCAL|GLOBAL)\(.* DP=(\d+) ", plan)
    if m:
        return ("gcn", m.group(2) == "LOCAL", int(m.group(3)) // 2, m.group(1))
    return None


@functools.lru_cache(maxsize=None)
def bf16_128_plan(name):
    from gated_graph_neural_network_samples_b200.engine import PreparedGraph
    c = BF16_128[name]
    adj, indeg = graph(c.batch, c.T)
    return PreparedGraph.host_only(c.params, c.T, adj, indeg, precision=c.precision, num_sms=NUM_SMS).info()["plan"]


# ---------------------------------------------------------------------------------------------------------------- tests
def test_every_nh_has_both_precisions_of_every_layout():
    nh = inventory()["tc"]
    want = {("tc", loc, n, compact, prec) for n in nh for loc, compact in ((True, True), (True, False), (False, False))
            for prec in ("bf16x3", "bf16")}
    want |= {("gcn", loc, n, prec) for n in inventory()["gcn"] for loc in (True, False) for prec in ("bf16x3", "bf16")}
    assert set(resources()) == want, sorted(set(resources()) ^ want, key=str)


PIPELINED_COMPACT_NH = (8, 16, 40, 48, 56, 64)
# Stack frames in bytes, CUDA 12.9 with the NVCC flags of _build.py.  SERIAL_STACK: the 128-row instances (LOCAL True / False) of the
# build in which one instance served both precisions.  COMPACT_STACK: the pipelined compact instances (bf16x3 / bf16 share the ceiling).
SERIAL_STACK = {
    True: {8: 8, 16: 16, 24: 72, 32: 152, 40: 208, 48: 400, 56: 552, 64: 1240},
    False: {8: 24, 16: 208, 24: 264, 32: 288, 40: 464, 48: 880, 56: 1032, 64: 1680},
}
COMPACT_STACK = {8: 0, 16: 0, 24: 16, 32: 24, 40: 120, 48: 120, 56: 336, 64: 344}
# 128-row instances whose stack frame is larger than SERIAL_STACK, and the largest frame accepted (bytes): the per-precision instances at
# NH 8 (LOCAL bf16x3 +8, GLOBAL +24) and LOCAL NH 48 (+24 bf16, +48 bf16x3).  Every other 128-row instance is at or below SERIAL_STACK.
SERIAL_STACK_EXCEPTIONS = {(True, 8, "bf16x3"): 16, (False, 8, "bf16x3"): 48, (False, 8, "bf16"): 48, (True, 48, "bf16"): 424,
                           (True, 48, "bf16x3"): 448}


def _pipelined(inst):
    return inst[0] == "gcn" or (inst[1] and inst[3] and inst[2] in PIPELINED_COMPACT_NH)


def test_mmas_are_not_serialised():
    counts = mma_counts()
    assert set(counts) == set(resources())
    checked = 0
    for inst, (hgmma, depbar) in sorted(counts.items(), key=str):
        assert hgmma > 0, inst
        if _pipelined(inst) and hgmma > 1:
            assert depbar < hgmma, "%s: %d WARPGROUP.DEPBAR for %d HGMMA: every MMA waits for the one before it" % (inst, depbar, hgmma)
            checked += 1
    # every GCN instance but NH 8 at bf16 (DP 16: one K-step, one MMA), LOCAL and GLOBAL; every pipelined compact NH at both precisions
    gcn = [nh for nh in inventory()["gcn"] for _ in range(2 * 2)]
    assert checked == len(gcn) - 2 * (8 in inventory()["gcn"]) + len(PIPELINED_COMPACT_NH) * 2


def test_tile_kernel_stacks_no_larger_than_before():
    for inst, r in resources().items():
        if inst[0] != "tc":
            continue
        _, loc, nh, compact, prec = inst
        bound = COMPACT_STACK[nh] if compact else SERIAL_STACK_EXCEPTIONS.get((loc, nh, prec), SERIAL_STACK[loc][nh])
        assert r["STACK"] <= bound, (inst, r["STACK"], bound)


def test_gcn_instances_do_not_spill():
    for inst, r in resources().items():
        if inst[0] == "gcn":
            assert r["STACK"] == 0, (inst, r["STACK"])


@pytest.mark.parametrize("name", sorted(BF16_128))
def test_bf16_128_row_case_reaches_its_instance(name):
    assert _plan_instance(bf16_128_plan(name)) == ("tc", True, BF16_128[name].instance[2], False, "bf16")


def test_every_compiled_instance_is_launched_by_a_case():
    covered = {_plan_instance(host_plan(n)["plan"]) for n in PINNABLE} | {_plan_instance(bf16_128_plan(n)) for n in BF16_128}
    missing = sorted(set(resources()) - covered, key=str)
    assert not missing, "compiled tile-kernel instances no case launches: %s" % missing
