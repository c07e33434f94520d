"""Compiler resource report of the partial-tuning kernels (no GPU needed): the FREEZE instantiations of adam_kernel and
apply_mask_kernel keep everything in registers (no stack frame, no spills)."""
import os
import subprocess
import tempfile

import pytest

from neurst_b200.csrc import build as B
from tests.test_kernel_resources_cpu import spill_table


def _report(name):
    if not os.path.exists(B.NVCC):
        pytest.skip("nvcc not available (%s)" % B.NVCC)
    with tempfile.TemporaryDirectory() as tmp:
        r = subprocess.run([B.NVCC] + B.FLAGS + ["-Xptxas", "-v", "-c", os.path.join(B.HERE, name), "-o", os.path.join(tmp, "k.o")],
                           capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-4000:]
    return spill_table(r.stdout + r.stderr)


def test_freeze_adam_and_apply_mask_kernels_do_not_spill():
    adam = {k: v for k, v in _report("optim.cu").items() if "adam_kernel" in k}
    freeze = {k: v for k, v in adam.items() if "MaskModeE2E" in k}
    assert len(adam) == 6 and len(freeze) == 2, sorted(adam)           # {clip_norm, plain} x {NONE, PRUNE, FREEZE}
    mask = {k: v for k, v in _report("prune.cu").items() if "apply_mask_kernel" in k}
    assert len(mask) == 1, sorted(mask)
    bad = {k: v for k, v in {**freeze, **mask}.items() if any(v)}
    assert not bad, bad
