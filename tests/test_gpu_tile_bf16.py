"""GPU: the 128-row LOCAL tile kernel at bf16 precision for every NH, against the float64 oracle.

The precision is a template parameter of the tile kernel, so 128-row LOCAL tiles at bf16 run an instance of their own.  The cases and the
instance each one claims are in tests/test_tile_kernel_mma_cpu.py; each runs as the cases of tests/test_gpu_forward_plans.py do (plan text,
final state and every layer state at the bf16 bar).
"""
import pytest

from tests.test_gpu_forward_plans import _run_ggnn
from tests.test_tile_kernel_mma_cpu import BF16_128

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("case", sorted(BF16_128))
def test_128_row_bf16_instances(case, monkeypatch):
    _run_ggnn(BF16_128[case], monkeypatch)
