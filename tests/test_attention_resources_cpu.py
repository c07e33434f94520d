"""Compiler resource report of the fused attention kernels (no GPU needed): every attn_fwd_kernel / attn_bwd_kernel
instantiation keeps its fp32 accumulators in registers (zero spill bytes) and every wgmma asynchronous (no C7512)."""
import os
import subprocess
import tempfile

import pytest

from neurst_b200.csrc import build as B
from tests.test_kernel_resources_cpu import spill_table

SRC = os.path.join(B.HERE, "attention.cu")


@pytest.fixture(scope="module")
def attention_report():
    if not os.path.exists(B.NVCC):
        pytest.skip("nvcc not available (%s)" % B.NVCC)
    with tempfile.TemporaryDirectory() as tmp:
        r = subprocess.run([B.NVCC] + B.FLAGS + ["-Xptxas", "-v", "-c", SRC, "-o", os.path.join(tmp, "attention.o")],
                           capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-4000:]
    return r.stdout + r.stderr


def test_attention_wgmma_not_serialized(attention_report):
    bad = [l for l in attention_report.splitlines() if "C7512" in l]
    assert not bad, "\n".join(bad)


def test_attention_kernels_do_not_spill(attention_report):
    table = {k: v for k, v in spill_table(attention_report).items() if "attn_fwd_kernel" in k or "attn_bwd_kernel" in k}
    # forward / backward x causal / not x bf16 / fp16
    assert len(table) == 8, sorted(table)
    spilled = {k: v for k, v in table.items() if v[1] or v[2]}
    assert not spilled, spilled
