"""Compiler resource report of the wide decode step (decode_rows.cu, no GPU needed): every rows-GEMM instantiation keeps its
accumulators and split-term operands in registers (zero spill bytes) and ptxas keeps its wgmma asynchronous (no C7512)."""
import os
import subprocess
import tempfile

import pytest

from neurst_b200.csrc import build as B
from tests.test_kernel_resources_cpu import spill_table

SRC = os.path.join(B.HERE, "decode_rows.cu")


@pytest.fixture(scope="module")
def ptxas_report():
    if not os.path.exists(B.NVCC):
        pytest.skip("nvcc not available (%s)" % B.NVCC)
    with tempfile.TemporaryDirectory() as tmp:
        r = subprocess.run([B.NVCC] + B.FLAGS + ["-Xptxas", "-v", "-c", SRC, "-o", os.path.join(tmp, "decode_rows.o")],
                           capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-4000:]
    return r.stdout + r.stderr


def test_no_serialized_wgmma(ptxas_report):
    bad = [l for l in ptxas_report.splitlines() if "C7512" in l or "serialized" in l]
    assert not bad, "\n".join(bad)


def test_rows_gemm_kernels_do_not_spill(ptxas_report):
    table = {k: v for k, v in spill_table(ptxas_report).items() if "rows_gemm_kernel" in k}
    # fp16 / bf16 x (LayerNorm -> store, MN-major) (none -> add) (relu(a + b1) -> add) (LayerNorm -> store, K-major logits)
    assert len(table) == 8, sorted(table)
    spilled = {k: v for k, v in table.items() if v[1] or v[2]}
    assert not spilled, spilled
