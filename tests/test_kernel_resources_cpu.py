"""Compiler resource report of the tensor-core kernels (no GPU needed): ptxas must keep every wgmma asynchronous (no C7512
"wgmma.mma_async instructions are serialized due to insufficient register resources") and the fused FFN kernel's
accumulators in registers (zero spill bytes for every fused_mlp_fwd_kernel instantiation)."""
import os
import re
import subprocess
import tempfile

import pytest

from neurst_b200.csrc import build as B

SRC = os.path.join(B.HERE, "tc_gemm.cu")


@pytest.fixture(scope="module")
def ptxas_report():
    if not os.path.exists(B.NVCC):
        pytest.skip("nvcc not available (%s)" % B.NVCC)
    with tempfile.TemporaryDirectory() as tmp:
        r = subprocess.run([B.NVCC] + B.FLAGS + ["-Xptxas", "-v", "-c", SRC, "-o", os.path.join(tmp, "tc_gemm.o")],
                           capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-4000:]
    return r.stdout + r.stderr


def spill_table(report):
    """{mangled kernel name: (stack frame, spill store, spill load) bytes} from ptxas -v output."""
    out, fn = {}, None
    for line in report.splitlines():
        m = re.search(r"Function properties for (\S+)", line)
        if m:
            fn = m.group(1)
            continue
        m = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m and fn is not None:
            out[fn] = tuple(int(x) for x in m.groups())
            fn = None
    return out


def test_no_serialized_wgmma(ptxas_report):
    bad = [l for l in ptxas_report.splitlines() if "C7512" in l]
    assert not bad, "\n".join(bad)


def test_fused_mlp_kernels_do_not_spill(ptxas_report):
    table = {k: v for k, v in spill_table(ptxas_report).items() if "fused_mlp_fwd_kernel" in k}
    # F16 / BF16 x forward (MN-major weights) / backward (K-major) x d in {128, 256}
    assert len(table) == 8, sorted(table)
    spilled = {k: v for k, v in table.items() if v[1] or v[2]}
    assert not spilled, spilled
