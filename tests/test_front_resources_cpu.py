"""Compiler resource report of the speech front-end's implicit-conv2 kernels (no GPU needed): the implicit conv2 GEMM entry
point (tc_gemm_conv_kernel, the tc_gemm_kernel body with the shifted-box A operand) and the 16-bit normalised-save conv1
kernels — the forward that also writes the parity-class planes and the backward that holds conv1's filter-gradient
accumulators in registers — keep everything in registers (no stack frame, no spills)."""
import os
import subprocess
import tempfile

import pytest

from neurst_b200.csrc import build as B
from tests.test_kernel_resources_cpu import ptxas_report, spill_table  # noqa: F401  (module-scoped fixture: tc_gemm.cu)


@pytest.fixture(scope="module")
def conv_report():
    if not os.path.exists(B.NVCC):
        pytest.skip("nvcc not available (%s)" % B.NVCC)
    with tempfile.TemporaryDirectory() as tmp:
        r = subprocess.run([B.NVCC] + B.FLAGS + ["-Xptxas", "-v", "-c", os.path.join(B.HERE, "conv_kernels.cu"), "-o",
                            os.path.join(tmp, "conv_kernels.o")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-4000:]
    return r.stdout + r.stderr


def test_conv_gemm_kernels_do_not_spill(ptxas_report):  # noqa: F811
    table = {k: v for k, v in spill_table(ptxas_report).items() if "tc_gemm_conv_kernel" in k}
    # K-major (data gradient) / MN-major (forward) weights x bf16 / fp16
    assert len(table) == 4, sorted(table)
    bad = {k: v for k, v in table.items() if any(v)}
    assert not bad, bad


def test_conv1_implicit_kernels_do_not_spill(conv_report):
    table = spill_table(conv_report)
    # conv1_bwd_xhat_c256_kernel<T, IMPLICIT = true> and conv1_fwd_c256_kernel<T, SAVE = true>, T = __half / __nv_bfloat16
    picked = {k: v for k, v in table.items()
              if ("conv1_bwd_xhat_c256_kernel" in k or "conv1_fwd_c256_kernel" in k) and "Lb1E" in k and "IfLb1E" not in k}
    assert len(picked) == 4, sorted(table)
    bad = {k: v for k, v in picked.items() if any(v)}
    assert not bad, bad
