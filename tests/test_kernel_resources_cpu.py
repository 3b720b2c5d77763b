"""CPU-only: what the compiler made of the tile-local wgmma kernel.  On compact tiles (every tile <= 64 rows) the four worker warpgroups
split the output columns, so each thread holds a quarter-width accumulator fragment per quantity instead of a half-width one.  That must
show in the binary: a compact instance exists for every padded hidden size, and its stack frame (register spills under the 96-register cap
of a 17-warp CTA) is no larger than that of the 128-row instance of the same size.  Read from ``cuobjdump -res-usage`` of the built
library; skipped without cuobjdump."""
import os
import re
import shutil
import subprocess

import pytest


def _cuobjdump():
    exe = shutil.which("cuobjdump")
    if exe is None:
        cand = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "cuobjdump")
        exe = cand if os.path.exists(cand) else None
    return exe


def _tile_kernels():
    """{(LOCAL, NH, COMPACT): {"REG": n, "STACK": n, ...}} of the ggnn_fwd_tc_kernel instances in libggnn_b200.so."""
    exe = _cuobjdump()
    if exe is None:
        pytest.skip("cuobjdump is not available")
    from gated_graph_neural_network_samples_b200 import _build, _lib
    _lib.load()
    out = subprocess.run([exe, "-res-usage", _build.LIB_PATH], capture_output=True, text=True, check=True).stdout
    kernels, key = {}, None
    for line in out.splitlines():
        m = re.match(r"\s*Function (\S+):", line)
        if m:
            k = re.search(r"ggnn_fwd_tc_kernelILb([01])ELi(\d+)ELb([01])E", m.group(1))
            key = (k.group(1) == "1", int(k.group(2)), k.group(3) == "1") if k else None
            continue
        if key is not None and "REG:" in line:
            kernels[key] = {n: int(v) for n, v in re.findall(r"([A-Z_]+):(\d+)", line)}
            key = None
    return kernels


def test_compact_tile_kernels_spill_no_more_than_the_128_row_layout():
    kernels = _tile_kernels()
    compact = sorted(nh for local, nh, c in kernels if c)
    assert compact == [8, 16, 24, 32, 40, 48, 56, 64], sorted(kernels)
    for nh in compact:
        assert (False, nh, True) not in kernels, "compact tiles are tile-local"
        small, full = kernels[(True, nh, True)], kernels[(True, nh, False)]
        assert small["REG"] <= 96, "NH=%d: %d registers do not fit 17 warps per SM" % (nh, small["REG"])
        assert small["STACK"] <= full["STACK"], "NH=%d: compact stack %d > 128-row stack %d" % (nh, small["STACK"], full["STACK"])
