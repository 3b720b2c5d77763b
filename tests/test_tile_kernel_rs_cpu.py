"""CPU-only: where the compact tile kernel's MMAs take their A operand from, read from ``cuobjdump -sass`` of the built library (skipped
without it).

On compact tiles (<= 64 rows) each worker warp loads a K-step's A fragment into registers once (``ldmatrix``) and feeds every MMA of that
K-step from there (wgmma's register-A form), instead of each MMA reading A from shared memory again.  In SASS a register-A MMA reads
``HGMMA.<shape> Rd, Ra, gdesc[..]``, a shared-memory one ``HGMMA.<shape> Rd, gdesc[..]``.  Per K-step (NKS = DP / 16 = NH / 8 of them per
DP-wide operand):

* bf16x3: the edge-type GEMM (3 MMAs), the gate GEMM's two segments (6 each) and the candidate's two (3 each) take A from registers --
  21 * NKS HGMMA; only the residual pre-products, once per layer, keep A in shared memory (6 + 3) -- 9 * NKS;
* bf16: the gate GEMM's two segments (2 MMAs each, r and u sharing one A fragment) take A from registers -- 4 * NKS; the rest keeps it in
  shared memory (one MMA per A fragment reads the same bytes either way);
* the 128-row tile kernel and the GCN kernel never take A from registers.
"""
import functools
import re
import subprocess

from tests.test_tile_kernel_mma_cpu import _cuobjdump, _lib, instance_of_symbol

_RS = re.compile(r"HGMMA\.\S+ R\d+, R\d+, gdesc")


@functools.lru_cache(maxsize=None)
def a_sources():
    """{instance: (register-A HGMMA count, shared-memory-A HGMMA count)} of every tile-kernel instance."""
    proc = subprocess.Popen([_cuobjdump(), "-sass", _lib()], stdout=subprocess.PIPE, text=True)
    counts, key = {}, None
    for line in proc.stdout:
        if "Function :" in line:
            key = instance_of_symbol(line.split("Function :", 1)[1].strip())
            if key is not None:
                counts[key] = [0, 0]
            continue
        if key is not None and "HGMMA." in line:
            counts[key][0 if _RS.search(line) else 1] += 1
    assert proc.wait() == 0
    return {k: tuple(v) for k, v in counts.items()}


def test_compact_bf16x3_mmas_take_a_from_registers():
    compact = {k: v for k, v in a_sources().items() if k[0] == "tc" and k[3] and k[4] == "bf16x3"}
    assert sorted(k[2] for k in compact) == [8, 16, 24, 32, 40, 48, 56, 64]
    for (_, _, nh, _, _), (rs, ss) in sorted(compact.items()):
        nks = nh // 8
        assert (rs, ss) == (21 * nks, 9 * nks), "NH=%d: %d register-A / %d shared-A HGMMA" % (nh, rs, ss)


def test_compact_bf16_gate_mmas_take_a_from_registers():
    compact = {k: v for k, v in a_sources().items() if k[0] == "tc" and k[3] and k[4] == "bf16"}
    assert sorted(k[2] for k in compact) == [8, 16, 24, 32, 40, 48, 56, 64]
    for (_, _, nh, _, _), (rs, ss) in sorted(compact.items()):
        assert rs == 4 * (nh // 8) and ss > 0, "NH=%d: %d register-A / %d shared-A HGMMA" % (nh, rs, ss)


def test_other_tile_kernels_keep_a_in_shared_memory():
    others = {k: v for k, v in a_sources().items() if k[0] == "gcn" or not k[3]}
    assert others
    for inst, (rs, ss) in sorted(others.items(), key=str):
        assert rs == 0 and ss > 0, (inst, rs, ss)
