"""Compiler resource report of conv1's 16-bit implicit backward (conv1_bwd_xhat_c256_kernel<T, IMPLICIT = true>), no GPU
needed.  The kernel is meant to run at HBM bandwidth with two 256-thread CTAs per SM (16 warps, twice the positions in
flight of one CTA per SM), which needs at most 65536 / (2 * 256) = 128 registers per thread, no stack frame, and its
static shared memory (two filter-gradient staging buffers and the reduction rows) within two CTAs' share of the SM."""
import re

from tests.test_front_resources_cpu import conv_report  # noqa: F401  (module-scoped fixture: conv_kernels.cu)


def implicit_backward_resources(report):
    """{mangled name: (registers, stack bytes, smem bytes)} of conv1_bwd_xhat_c256_kernel<16-bit T, true>."""
    out, fn = {}, None
    for line in report.splitlines():
        m = re.search(r"Compiling entry function '(\S+)'", line)
        if m:
            fn = m.group(1) if "conv1_bwd_xhat_c256_kernel" in m.group(1) and "Lb1E" in m.group(1) else None
            continue
        if fn is None:
            continue
        m = re.search(r"(\d+) bytes stack frame", line)
        if m:
            stack = int(m.group(1))
        m = re.search(r"Used (\d+) registers.*?(\d+) bytes smem", line)
        if m:
            out[fn] = (int(m.group(1)), stack, int(m.group(2)))
            fn = None
    return out


def test_conv1_implicit_backward_fits_two_ctas_per_sm(conv_report):  # noqa: F811
    res = implicit_backward_resources(conv_report)
    assert len(res) == 2, res           # __half and __nv_bfloat16
    for name, (regs, stack, smem) in res.items():
        assert regs <= 128, (name, regs)
        assert stack == 0, (name, stack)
        assert 2 * (smem + 1024) <= 228 * 1024, (name, smem)
