// fp32 CUDA-core GEMM with the same GemmArgs contract as the wgmma kernel.
//
// Used (a) for the fp32 parity mode — every contraction in full fp32 FMA so the CUDA path can be held to
// the reference's own KAT tolerances (tests/neurst/**: sum(d^2) < 1e-9) at the toy shapes of those tests
// (d = 4..16, which no tensor-core tile fits) — and (b) as the on-device cross-check of the wgmma kernel.
// Operands may be fp32 or bf16 in memory; accumulation is always fp32.
#include "gemm.cuh"
#include "pdl.cuh"

namespace b200st {
namespace {

constexpr int TM = 64, TN = 64, TK = 16;

__global__ void __launch_bounds__(256) simt_gemm_kernel(const GemmArgs g) {
  pdl_wait();
  pdl_trigger();
  __shared__ float As[TK][TM + 1];
  __shared__ float Bs[TK][TN + 1];
  const int b = blockIdx.z;
  const int b1 = b % g.nb1, b2 = b / g.nb1;
  const int m0 = blockIdx.y * TM, n0 = blockIdx.x * TN;
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
  const int64_t a_off = (int64_t)b2 * g.A.sb2 + (int64_t)b1 * g.A.sb1;
  const int64_t b_off = (int64_t)b2 * g.B.sb2 + (int64_t)b1 * g.B.sb1;
  const int64_t sam = g.A.mn_major ? 1 : g.A.ld, sak = g.A.mn_major ? g.A.ld : 1;
  const int64_t sbn = g.B.mn_major ? 1 : g.B.ld, sbk = g.B.mn_major ? g.B.ld : 1;
  float acc[4][4] = {};
  for (int k0 = 0; k0 < g.K; k0 += TK) {
    for (int i = threadIdx.x; i < TM * TK; i += 256) {
      int mm, kk;
      if (g.A.mn_major) { mm = i % TM; kk = i / TM; } else { kk = i % TK; mm = i / TK; }
      const int m = m0 + mm, k = k0 + kk;
      As[kk][mm] = (m < g.M && k < g.K) ? load_as_f32(g.A.ptr, g.A.dtype, a_off + m * sam + k * sak) : 0.f;
    }
    for (int i = threadIdx.x; i < TN * TK; i += 256) {
      int nn, kk;
      if (g.B.mn_major) { nn = i % TN; kk = i / TN; } else { kk = i % TK; nn = i / TK; }
      const int n = n0 + nn, k = k0 + kk;
      Bs[kk][nn] = (n < g.N && k < g.K) ? load_as_f32(g.B.ptr, g.B.dtype, b_off + n * sbn + k * sbk) : 0.f;
    }
    __syncthreads();
#pragma unroll
    for (int kk = 0; kk < TK; ++kk) {
      float a[4], bb[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) { a[i] = As[kk][ty * 4 + i]; bb[i] = Bs[kk][tx * 4 + i]; }
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(a[i], bb[j], acc[i][j]);
    }
    __syncthreads();
  }
  const GemmEpilogue& ep = g.epi;
  const int64_t bidx = (int64_t)b2 * g.nb1 + b1;
  const int64_t boff_c = (int64_t)b2 * g.c_sb2 + (int64_t)b1 * g.c_sb1;
  const int64_t boff_mask = (int64_t)b2 * ep.mask_sb2 + (int64_t)b1 * ep.mask_sb1;
  const int64_t boff_res = (int64_t)b2 * ep.res_sb2 + (int64_t)b1 * ep.res_sb1;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int m = m0 + ty * 4 + i;
    if (m >= g.M) continue;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int n = n0 + tx * 4 + j;
      if (n >= g.N) continue;
      const uint64_t e_idx = (uint64_t)((bidx * g.M + m) * (int64_t)g.N + n);
      float v = gemm_epilogue_value(ep, acc[i][j], m, n, boff_mask, boff_res, e_idx);
      const int64_t idx = boff_c + (int64_t)m * g.ldc + n;
      if (ep.accumulate) v += reinterpret_cast<float*>(g.C)[idx];
      store_from_f32(g.C, g.c_dtype, idx, v);
    }
  }
}

}  // namespace

int gemm_simt_f32(const GemmArgs& g, cudaStream_t stream) {
  B200ST_CHECK(g.M > 0 && g.N > 0 && g.K > 0 && g.nb1 > 0 && g.nb2 > 0, "empty GEMM");
  if (g.epi.accumulate) B200ST_CHECK(g.c_dtype == F32, "accumulate needs fp32 C");
  const int64_t nb = (int64_t)g.nb1 * g.nb2;
  B200ST_CHECK(nb <= 65535 && ceil_div(g.M, TM) <= 65535, "grid too large for SIMT GEMM");
  dim3 grid(ceil_div(g.N, TN), ceil_div(g.M, TM), (unsigned)nb);
  return launch(simt_gemm_kernel, grid, 256, 0, stream, g);
}

int gemm(const GemmArgs& g, cudaStream_t stream) {
  if (is16(g.A.dtype) && is16(g.B.dtype)) return gemm_tc_bf16(g, stream);
  B200ST_CHECK(g.A.dtype == F32 && g.B.dtype == F32, "mixed-dtype GEMM operands");
  return gemm_simt_f32(g, stream);
}

}  // namespace b200st
