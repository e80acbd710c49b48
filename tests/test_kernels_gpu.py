"""GPU parity tests of the normalisation, attention, loss and element-wise kernels behind the C ABI against plain PyTorch
fp32 references of the same op (tolerances are relative L2 errors of bf16 results vs the fp32 reference; written in
tools/gpu_kernel_check.py).  The GEMM is checked element by element against fp64 in tests/test_gemm_paths_gpu.py."""
import os
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools"))


@pytest.fixture(scope="module")
def chk():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    import gpu_kernel_check as c
    return c


@pytest.mark.parametrize("group", ["norm", "attn", "loss", "act_bwd_colsum"])
def test_kernel_group(chk, group):
    chk.RESULTS.clear()
    chk.GROUPS[group]()
    torch.cuda.synchronize()
    bad = [r for r in chk.RESULTS if not r["ok"]]
    assert not bad, "\n".join(f"{r['name']}: err={r['err']:.3e} tol={r['tol']:.1e} {r['extra']}" for r in bad)
    assert len(chk.RESULTS) > 0
