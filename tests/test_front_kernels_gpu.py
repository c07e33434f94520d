"""The speech front-end's C-ABI kernels per element against fp64:

- b200st_conv1_ln_relu_fwd: conv 3x3 / stride 2 / pad 1 (+ LayerNorm, eps 1e-6) + ReLU, through every dispatch branch:
  the register-filter kernel (C == 256, Cin == 1, LN, 16-byte aligned) and the generic kernel with and without 16-byte
  vectors, 8 or 16 channels per lane, one or several input channels.
- b200st_layernorm_fwd / b200st_layernorm_bwd (ReLU and residual gradient): the vector kernels (2 rows per warp up to
  65536 rows, 1 above; 4-column groups up to 512 columns), the scalar kernels (cols % 4 != 0, cols > 512, or a view that is
  not 16-byte aligned), and the dgamma / dbeta reduction over many rows.

16-bit outputs may differ from the fp64 value rounded to their type by one unit in the last place, plus the fp32
arithmetic of the kernel (which can only matter where that unit is smaller, near zero)."""
import ctypes as C

import pytest
import torch
import torch.nn.functional as Fn

from neurst_b200 import lib as L

pytestmark = pytest.mark.gpu

DT = {"fp32": torch.float32, "bf16": torch.bfloat16, "fp16": torch.float16}


def spacing(ref, dtype):
    """Distance between consecutive values of `dtype` around ref (fp64 tensor)."""
    fi = torch.finfo(dtype)
    mant = {torch.float32: 23, torch.bfloat16: 7, torch.float16: 10}[dtype]
    a = ref.abs().clamp(min=fi.smallest_normal)
    return torch.exp2(torch.floor(torch.log2(a)) - mant)


def assert_close(got, ref, dtype, atol, what):
    """|got - ref| <= 1 ulp of ref in `dtype` (16-bit) + atol; fp32: <= atol."""
    got, ref = got.double(), ref.double()
    bound = atol + (spacing(ref.to(dtype).double(), dtype) if dtype != torch.float32 else 0.0)
    err = (got - ref).abs()
    excess = err - bound
    i = int(torch.argmax(excess.flatten()))
    assert float(excess.flatten()[i]) <= 0, "%s: |got - ref| = %.3e > bound %.3e at flat index %d (got %.6e, ref %.6e)" % (
        what, float(err.flatten()[i]), float(torch.as_tensor(bound).expand_as(err).flatten()[i]), i,
        float(got.flatten()[i]), float(ref.flatten()[i]))


# ---------------------------------------------------------------------------------------------------------------------
# conv1 + LN + ReLU forward
# ---------------------------------------------------------------------------------------------------------------------
def conv1_ref(src, w, b, gamma, beta, use_ln):
    """fp64: src [B,T,F,Cin], w HWIO [3,3,Cin,C] -> [B,T1,F1,C]."""
    x = src.double().permute(0, 3, 1, 2)
    z = Fn.conv2d(x, w.double().permute(3, 2, 0, 1), b.double(), stride=2, padding=1).permute(0, 2, 3, 1)
    if use_ln:
        mean = z.mean(-1, keepdim=True)
        var = ((z - mean) ** 2).mean(-1, keepdim=True)
        z = (z - mean) / torch.sqrt(var + 1e-6) * gamma.double() + beta.double()
    return torch.relu(z)


def conv1_device(src, w, b, gamma, beta, dtype, C_, use_ln, misalign=False):
    B, T, F, Cin = src.shape
    T1, F1 = (T + 1) // 2, (F + 1) // 2
    n = B * T1 * F1 * C_
    buf = torch.full((n + 1,), float("nan"), dtype=dtype, device="cuda")
    y = buf[1:] if misalign else buf[:n]
    args = [C.c_void_p(t.data_ptr()) for t in (src, w, b, gamma, beta)]
    rc = L.load().b200st_conv1_ln_relu_fwd(*args, C.c_void_p(y.data_ptr()), C.c_int32(L._dt(y)), C.c_int32(B), C.c_int32(T),
                                          C.c_int32(F), C.c_int32(Cin), C.c_int32(C_), C.c_int32(int(use_ln)), L._stream())
    L.check(rc)
    torch.cuda.synchronize()
    return y.view(B, T1, F1, C_)


# (C, Cin, use_ln, misaligned output) -> kernel
CONV_CASES = [
    (256, 1, 1, False),   # conv1_fwd_c256_kernel (filter in registers)
    (256, 1, 0, False),   # generic, VEC, CPL 8, Cin 1 (no LN: the register-filter kernel needs LN)
    (256, 1, 1, True),    # generic, scalar stores (output not 16-byte aligned), CPL 8, Cin 1
    (64, 2, 1, False),    # generic, VEC, CPL 8, Cin > 1
    (256, 4, 0, False),   # generic, VEC, CPL 8, Cin 4 (36 taps)
    (320, 1, 1, False),   # generic, VEC, CPL 16, Cin 1
    (512, 2, 1, False),   # generic, VEC, CPL 16, Cin > 1 (largest C)
    (5, 1, 1, False),     # generic, scalar, CPL 8, Cin 1 (C < 8)
    (100, 3, 0, False),   # generic, scalar (C % 8 != 0), CPL 8, Cin > 1
    (300, 1, 1, False),   # generic, scalar, CPL 16, Cin 1
    (300, 2, 0, False),   # generic, scalar, CPL 16, Cin > 1
]


@pytest.mark.parametrize("dtype", ["fp32", "bf16", "fp16"])
@pytest.mark.parametrize("T,F", [(11, 80), (12, 7), (5, 83)])
@pytest.mark.parametrize("C_,Cin,use_ln,misalign", CONV_CASES)
def test_conv1_ln_relu_fwd_vs_fp64(C_, Cin, use_ln, misalign, T, F, dtype):
    g = torch.Generator().manual_seed(C_ * 31 + Cin * 7 + T + F)
    B = 3
    src = torch.randn(B, T, F, Cin, generator=g)
    w = torch.randn(3, 3, Cin, C_, generator=g) / (3.0 * Cin ** 0.5)       # O(1) pre-activations
    b = 0.2 * torch.randn(C_, generator=g)
    gamma = 1.0 + 0.2 * torch.randn(C_, generator=g)
    beta = 0.2 * torch.randn(C_, generator=g)
    ref = conv1_ref(src, w, b, gamma, beta, use_ln)
    got = conv1_device(*(t.cuda() for t in (src, w, b, gamma, beta)), DT[dtype], C_, use_ln, misalign).cpu()
    assert torch.isfinite(got.float()).all()
    assert_close(got, ref, DT[dtype], 1e-5, "conv1 C=%d Cin=%d ln=%d" % (C_, Cin, use_ln))


def test_conv1_filter_beyond_shared_memory_is_refused():
    src = torch.zeros(1, 4, 8, 3, device="cuda")
    w = torch.zeros(3, 3, 3, 512, device="cuda")
    v = torch.zeros(512, device="cuda")
    with pytest.raises(L.B200STError, match="shared memory"):
        conv1_device(src, w, v, v, v, torch.float32, 512, 1)


# ---------------------------------------------------------------------------------------------------------------------
# LayerNorm forward / backward
# ---------------------------------------------------------------------------------------------------------------------
def ln_case(rows, cols, dtype, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = (0.5 + torch.randn(rows, cols, generator=g, device="cuda")).to(dtype)
    dy = torch.randn(rows, cols, generator=g, device="cuda").to(dtype)
    dres = torch.randn(rows, cols, generator=g, device="cuda")
    gamma = 1.0 + 0.2 * torch.randn(cols, generator=g, device="cuda")
    beta = 0.3 * torch.randn(cols, generator=g, device="cuda")
    return x, dy, dres, gamma, beta


def placed(t, misalign):
    """t itself, or a copy that starts one element into its buffer (breaks 16-byte alignment)."""
    if not misalign:
        return t.contiguous()
    buf = torch.empty(t.numel() + 1, dtype=t.dtype, device=t.device)
    v = buf[1:].view(t.shape)
    v.copy_(t)
    return v


def ln_fwd(x, gamma, beta, y_dtype, relu, misalign):
    rows, cols = x.shape
    y = placed(torch.full_like(x, float("nan"), dtype=y_dtype), misalign)
    mean = torch.full((rows,), float("nan"), device="cuda")
    rstd = torch.full((rows,), float("nan"), device="cuda")
    L.check(L.load().b200st_layernorm_fwd(x.data_ptr(), L._dt(x), gamma.data_ptr(), beta.data_ptr(), 1e-6, y.data_ptr(),
                                          L._dt(y), mean.data_ptr(), rstd.data_ptr(), rows, cols, int(relu), L._stream()))
    return y, mean, rstd


def run_layernorm(rows, cols, dtype, relu, with_dres, misalign, seed=0):
    dt = DT[dtype]
    x, dy, dres, gamma, beta = ln_case(rows, cols, dt, seed)
    x, dy = placed(x, misalign), placed(dy, misalign)
    dres = placed(dres, misalign) if with_dres else None
    y, mean, rstd = ln_fwd(x, gamma, beta, dt, relu, misalign)
    # the same forward with an fp32 output: the ReLU mask exactly as the kernels see it (no 16-bit rounding to zero)
    y32, _, _ = ln_fwd(x, gamma, beta, torch.float32, relu, False)
    dx = placed(torch.full_like(x, float("nan")), misalign)
    g = torch.Generator(device="cuda").manual_seed(seed + 1)
    dg0 = torch.randn(cols, generator=g, device="cuda")      # the kernel accumulates into dgamma / dbeta
    db0 = torch.randn(cols, generator=g, device="cuda")
    dgamma, dbeta = dg0.clone(), db0.clone()
    L.check(L.load().b200st_layernorm_bwd(dy.data_ptr(), L._dt(dy), x.data_ptr(), L._dt(x), mean.data_ptr(), rstd.data_ptr(),
                                          gamma.data_ptr(), beta.data_ptr(), dres.data_ptr() if dres is not None else None,
                                          dx.data_ptr(), L._dt(dx), dgamma.data_ptr(), dbeta.data_ptr(), rows, cols, int(relu),
                                          L._stream()))
    torch.cuda.synchronize()

    # fp64 reference on the same (rounded) inputs
    xd = x.double()
    m = xd.mean(-1, keepdim=True)
    r = 1.0 / torch.sqrt(((xd - m) ** 2).mean(-1, keepdim=True) + 1e-6)
    xh = (xd - m) * r
    yref = xh * gamma.double() + beta.double()
    d = dy.double()
    if relu:
        yref = torch.relu(yref)
        d = d * (y32 > 0).double()
    gg = d * gamma.double()
    dxref = r * (gg - gg.mean(-1, keepdim=True) - xh * (gg * xh).mean(-1, keepdim=True))
    if dres is not None:
        dxref = dxref + dres.double()
    dgref = dg0.double() + (d * xh).sum(0)
    dbref = db0.double() + d.sum(0)
    return dict(y=(y, yref), mean=(mean, m.squeeze(-1)), rstd=(rstd, r.squeeze(-1)), dx=(dx, dxref), dgamma=(dgamma, dgref),
                dbeta=(dbeta, dbref))


def check_layernorm(res, rows, dtype):
    dt = DT[dtype]
    y, yref = res["y"]
    assert_close(y, yref, dt, 1e-5, "y")
    mean, mref = res["mean"]
    rstd, rref = res["rstd"]
    assert_close(mean, mref, torch.float32, 2e-6, "mean")
    assert_close(rstd / rref, torch.ones_like(rref), torch.float32, 2e-6, "rstd (relative)")
    dx, dxref = res["dx"]
    assert_close(dx, dxref, dt, 2e-5, "dx")
    # column sums over `rows` rows of O(1) terms in fp32: rounding grows like sqrt(rows)
    tol = 1e-5 * rows ** 0.5
    for k in ("dgamma", "dbeta"):
        got, ref = res[k]
        assert_close(got, ref, torch.float32, tol, k)


LN_COLS = [5, 64, 250, 256, 320, 512, 1024]


@pytest.mark.parametrize("dtype", ["fp32", "bf16", "fp16"])
@pytest.mark.parametrize("rows", [1, 37, 65537])
@pytest.mark.parametrize("cols", LN_COLS)
def test_layernorm_relu_dres_vs_fp64(cols, rows, dtype):
    check_layernorm(run_layernorm(rows, cols, dtype, relu=True, with_dres=True, misalign=False), rows, dtype)


@pytest.mark.parametrize("dtype", ["fp32", "bf16", "fp16"])
@pytest.mark.parametrize("cols", LN_COLS)
def test_layernorm_plain_vs_fp64(cols, dtype):
    check_layernorm(run_layernorm(37, cols, dtype, relu=False, with_dres=False, misalign=False), 37, dtype)


# many rows: 65536 is the last row count of the two-rows-per-warp backward kernel, 200000 runs the one-row kernel and
# the dgamma / dbeta reduction over ~12 rows per warp (the speech front-end's ln2: 256 columns, ReLU, > 65536 rows)
@pytest.mark.parametrize("dtype", ["fp32", "bf16", "fp16"])
@pytest.mark.parametrize("rows", [65536, 200000])
@pytest.mark.parametrize("cols", [64, 256, 320])
def test_layernorm_many_rows_vs_fp64(cols, rows, dtype):
    check_layernorm(run_layernorm(rows, cols, dtype, relu=True, with_dres=False, misalign=False), rows, dtype)


# a view one element into its buffer: not 16-byte aligned, so the scalar kernels run whatever the column count
@pytest.mark.parametrize("dtype", ["fp32", "bf16", "fp16"])
@pytest.mark.parametrize("rows", [37, 65537])
@pytest.mark.parametrize("cols", [64, 256, 1024])
def test_layernorm_misaligned_view_vs_fp64(cols, rows, dtype):
    check_layernorm(run_layernorm(rows, cols, dtype, relu=True, with_dres=True, misalign=True), rows, dtype)
