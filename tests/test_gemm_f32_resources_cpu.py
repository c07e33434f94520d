"""Compiler resource report of tc_gemm_f32_kernel (no GPU needed): its fp32-output epilogue is an entry point of its own
because, next to the general loop, it spilled the BN = 128 accumulators; every instantiation must stay spill-free."""
from tests.test_kernel_resources_cpu import ptxas_report, spill_table  # noqa: F401  (module fixture: one ptxas run here)


def test_f32_output_gemm_kernels_do_not_spill(ptxas_report):  # noqa: F811
    table = {k: v for k, v in spill_table(ptxas_report).items() if "tc_gemm_f32_kernel" in k}
    # BN in {64, 128} x 4 operand layouts x bf16 / fp16
    assert len(table) == 16, sorted(table)
    spilled = {k: v for k, v in table.items() if v[1] or v[2]}
    assert not spilled, spilled
