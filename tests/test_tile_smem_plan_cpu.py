"""CPU-only: the shared-memory plan of the tile-local wgmma kernel (csrc/ggnn_tc_smem.h), compiled into a small host program.

The plan places the h operand, the gather tiles, the weight ring, the biases, the per-row constants and the CSR slice.  Here, for every
padded hidden size of the tile kernel, 4 / 17 / 32 edge types, with and without edge bias:

* every plan fits the H100's 227 KB opt-in shared memory (less the kernel's static 1 KB) and its parts add up to the launch's size;
* compact tile-local launches get min(edge types per tile, what fits) gather tiles, never fewer than 2, and whenever they get more
  than 2 the weight ring keeps at least 4 slots; 128-row and GLOBAL launches keep 2;
* GGNN_TC_GATHER_TILES (the request) is clamped to what fits, and a request of 2 leaves the CSR slice as it is by default;
* cfg2 (DP 112, 4 edge types) gets 4 gather tiles and 5 ring slots.
"""
import os
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "gated_graph_neural_network_samples_b200", "csrc", "ggnn_tc_smem.h")
AVAIL = 227 * 1024 - 1024
MAX_STAGES = 10

DRIVER = r"""
#include <cstdio>
#include <cstdlib>
#include "%s"
int main(int argc, char** argv) {
    int DP, kgs, T, local, sparse, bias, msgs, types, req;
    while (std::scanf("%%d %%d %%d %%d %%d %%d %%d %%d %%d", &DP, &kgs, &T, &local, &sparse, &bias, &msgs, &types, &req) == 9) {
        const ggnn::TcSmemPlan p = ggnn::tc_smem_plan(DP, kgs, T, local, sparse, bias, msgs, types, %d, %d, req);
        std::printf("%%d %%d %%d %%d %%zu\n", p.ngather, p.nstages, p.csr_cache, p.csr_cap_msgs, p.smem);
    }
    return 0;
}
"""


@pytest.fixture(scope="module")
def plan(tmp_path_factory):
    cxx = shutil.which("g++") or shutil.which("c++")
    if cxx is None:
        pytest.skip("no host C++ compiler")
    d = tmp_path_factory.mktemp("smem_plan")
    src, exe = d / "plan.cpp", d / "plan"
    src.write_text(DRIVER % (HEADER, AVAIL, MAX_STAGES))
    subprocess.run([cxx, "-std=c++17", "-O1", "-o", str(exe), str(src)], check=True)

    def run(cases):
        text = "".join(" ".join(str(int(v)) for v in c) + "\n" for c in cases)
        out = subprocess.run([str(exe)], input=text, capture_output=True, text=True, check=True).stdout.split("\n")
        keys = ("ngather", "nstages", "csr_cache", "csr_cap", "smem")
        return [dict(zip(keys, map(int, line.split()))) for line in out if line.strip()]
    return run


def _layout_bytes(DP, kgs, T, local, bias, p):
    opb, stage = DP * kgs // 4, DP * 128
    csr = ((128 * T + 1 + 7) & ~7) * 2 + p["csr_cap"] if p["csr_cache"] else 0
    rows = (kgs // 16) * (1 + (T if bias else 0)) * 4 if local and kgs == 1024 else 0
    return (1 + p["ngather"]) * opb + p["nstages"] * stage + 3 * DP * 4 + 64 + rows + csr


def _cases():
    out = []
    for DP in range(16, 129, 16):
        for T in (4, 17, 32):
            for bias in (0, 1):
                for kgs, local in ((1024, 1), (2048, 1), (2048, 0)):
                    for req in (0, 2, 3, 64):
                        out.append((DP, kgs, T, local, 1, bias, 40 * T, T, req))
    return out


def test_every_plan_fits_and_keeps_the_ring(plan):
    cases = _cases()
    for c, p in zip(cases, plan(cases)):
        DP, kgs, T, local, _, bias, _, types, req = c
        assert 2 <= p["nstages"] <= MAX_STAGES, (c, p)
        assert p["smem"] <= AVAIL and p["smem"] == _layout_bytes(DP, kgs, T, local, bias, p), (c, p)
        if local and kgs == 1024:
            want = req if req else types
            assert 2 <= p["ngather"] <= max(2, want), (c, p)
            if p["ngather"] > 2:
                assert p["nstages"] >= 4, (c, p)
            if 2 < want and p["ngather"] < min(want, 32):   # limited by shared memory: one more tile would leave fewer than 4 slots
                fixed = p["smem"] - p["nstages"] * DP * 128
                assert AVAIL - fixed - DP * kgs // 4 < 4 * DP * 128, (c, p)
        else:
            assert p["ngather"] == 2, (c, p)
        if not local:
            assert not p["csr_cache"], (c, p)


def test_two_gather_tiles_keep_the_default_csr_slice(plan):
    cases = [c for c in _cases() if c[8] == 0]
    default, two = plan(cases), plan([c[:8] + (2,) for c in cases])
    for c, a, b in zip(cases, default, two):
        assert b["ngather"] == 2, (c, b)
        assert a["csr_cache"] == b["csr_cache"], (c, a, b)


def test_cfg2_plan(plan):
    cfg2, dp128, dp128_wide = plan([(112, 1024, 4, 1, 1, 0, 300, 4, 0), (128, 1024, 4, 1, 1, 0, 300, 4, 0),
                                    (128, 2048, 32, 1, 1, 1, 300, 32, 0)])
    assert (cfg2["ngather"], cfg2["nstages"], cfg2["csr_cache"]) == (4, 5, 1), cfg2
    assert dp128["ngather"] == 3 and dp128["nstages"] >= 4, dp128
    # 128-row tiles at DP 128 have room for two ring slots only
    assert (dp128_wide["ngather"], dp128_wide["nstages"]) == (2, 2), dp128_wide
