"""Compiler resource report of the GEMM kernels (no GPU needed): every tc_gemm_kernel and tc_wgrad_group_kernel
instantiation keeps its fp32 accumulators in registers (zero spill bytes) within the 168-register budget of a 384-thread CTA."""
from tests.test_kernel_resources_cpu import ptxas_report, spill_table  # noqa: F401  (module fixture: one ptxas run here)


def test_gemm_kernels_do_not_spill(ptxas_report):  # noqa: F811
    table = spill_table(ptxas_report)
    gemm = {k: v for k, v in table.items() if "tc_gemm_kernel" in k}
    wgrad = {k: v for k, v in table.items() if "tc_wgrad_group_kernel" in k}
    # BN in {64, 128} x 4 operand layouts x bf16 / fp16; the grouped weight-gradient kernel in bf16 / fp16
    assert len(gemm) == 16, sorted(gemm)
    assert len(wgrad) == 2, sorted(wgrad)
    spilled = {k: v for k, v in {**gemm, **wgrad}.items() if v[1] or v[2]}
    assert not spilled, spilled
