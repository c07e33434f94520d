// LayerNorm / softmax / dropout-cast / reductions / positions / embedding / label-smoothed CE / Adam.
// HBM-bound kernels: coalesced accesses along the feature axis, warp-shuffle reductions, fp32 math.
#include "kernels.cuh"
#include "pdl.cuh"
#include <math.h>

namespace b200st {

// three tensors that are either all fp32 or all the same 16-bit type (keeps the instantiation count linear)
#define DISPATCH_UNIFORM3(d0, d1, d2, T, ...)                                                 \
  do {                                                                                        \
    if ((d0) != (d1) || (d1) != (d2)) B200ST_FAIL("the three tensors must share one dtype"); \
    DISPATCH_DTYPE(d0, T, __VA_ARGS__);                                                       \
  } while (0)


// ---- 4-wide vector access along the feature axis (16-byte fp32 / 8-byte bf16) ------------------------------------
template <typename T> __device__ __forceinline__ void load4(const T* p, float (&v)[4]);
template <> __device__ __forceinline__ void load4<float>(const float* p, float (&v)[4]) {
  const float4 a = *reinterpret_cast<const float4*>(p);
  v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w;
}
template <int DT> __device__ __forceinline__ void load4_16(const void* p, float (&v)[4]) {
  const uint2 pk = *reinterpret_cast<const uint2*>(p);
  const float2 a = unpack2_16(pk.x, DT), b = unpack2_16(pk.y, DT);
  v[0] = a.x; v[1] = a.y; v[2] = b.x; v[3] = b.y;
}
template <> __device__ __forceinline__ void load4<__nv_bfloat16>(const __nv_bfloat16* p, float (&v)[4]) { load4_16<BF16>(p, v); }
template <> __device__ __forceinline__ void load4<__half>(const __half* p, float (&v)[4]) { load4_16<F16>(p, v); }
template <typename T> __device__ __forceinline__ void store4(T* p, const float (&v)[4]);
template <> __device__ __forceinline__ void store4<float>(float* p, const float (&v)[4]) {
  *reinterpret_cast<float4*>(p) = make_float4(v[0], v[1], v[2], v[3]);
}
template <int DT> __device__ __forceinline__ void store4_16(void* p, const float (&v)[4]) {
  uint2 pk;
  pk.x = pack2_16(v[0], v[1], DT); pk.y = pack2_16(v[2], v[3], DT);
  *reinterpret_cast<uint2*>(p) = pk;
}
template <> __device__ __forceinline__ void store4<__nv_bfloat16>(__nv_bfloat16* p, const float (&v)[4]) { store4_16<BF16>(p, v); }
template <> __device__ __forceinline__ void store4<__half>(__half* p, const float (&v)[4]) { store4_16<F16>(p, v); }

// =============================================================================================
// LayerNorm forward: one warp per row, values cached in registers for cols <= 1024
// =============================================================================================
template <typename TX, typename TY>
__global__ void __launch_bounds__(256) ln_fwd_kernel(const TX* __restrict__ x, const float* __restrict__ gamma,
                                                      const float* __restrict__ beta, float eps, TY* __restrict__ y,
                                                      float* __restrict__ y32, float* __restrict__ mean_out,
                                                      float* __restrict__ rstd_out, int64_t rows, int cols, int relu) {
  pdl_wait();
  pdl_trigger();
  const int lane = threadIdx.x & 31;
  const int64_t warps_total = (int64_t)gridDim.x * (blockDim.x >> 5);
  for (int64_t row = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); row < rows; row += warps_total) {
    const TX* xr = x + row * cols;
    float sum = 0.f;
    for (int c = lane; c < cols; c += 32) sum += to_f32(xr[c]);
    const float mean = warp_sum(sum) / cols;
    float sq = 0.f;
    for (int c = lane; c < cols; c += 32) { float dlt = to_f32(xr[c]) - mean; sq += dlt * dlt; }
    const float var = warp_sum(sq) / cols;
    const float rstd = 1.0f / sqrtf(var + eps);
    for (int c = lane; c < cols; c += 32) {
      float v = (to_f32(xr[c]) - mean) * rstd;
      v = v * gamma[c] + beta[c];
      if (relu) v = fmaxf(v, 0.f);
      y[row * cols + c] = from_f32<TY>(v);
      if (y32) y32[row * cols + c] = v;
    }
    if (lane == 0) {
      if (mean_out) mean_out[row] = mean;
      if (rstd_out) rstd_out[row] = rstd;
    }
  }
}

// cols % 4 == 0, cols <= 128*NV: each lane owns NV groups of 4 contiguous columns (c = 4*lane + 128*g); row in registers
template <typename TX, typename TY, int NV>
__global__ void __launch_bounds__(256) ln_fwd_vec_kernel(const TX* __restrict__ x, const float* __restrict__ gamma,
                                                          const float* __restrict__ beta, float eps, TY* __restrict__ y,
                                                          float* __restrict__ y32, float* __restrict__ mean_out,
                                                          float* __restrict__ rstd_out, int64_t rows, int cols, int relu,
                                                          float* __restrict__ xcopy) {
  pdl_wait();
  pdl_trigger();
  const int lane = threadIdx.x & 31;
  const int64_t warps_total = (int64_t)gridDim.x * (blockDim.x >> 5);
  float g[NV][4], bt[NV][4];
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    const int c = 4 * lane + 128 * i;
    if (c < cols) { load4<float>(gamma + c, g[i]); load4<float>(beta + c, bt[i]); }
  }
  for (int64_t row = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); row < rows; row += warps_total) {
    float v[NV][4];
    float sum = 0.f;
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      const int c = 4 * lane + 128 * i;
      if (c < cols) {
        load4<TX>(x + row * cols + c, v[i]);
        sum += v[i][0] + v[i][1] + v[i][2] + v[i][3];
        if (xcopy) store4<float>(xcopy + row * cols + c, v[i]);     // fp32 copy of the input row (residual base of a fused consumer)
      }
    }
    const float mean = warp_sum(sum) / cols;
    float sq = 0.f;
#pragma unroll
    for (int i = 0; i < NV; ++i)
      if (4 * lane + 128 * i < cols) {
#pragma unroll
        for (int j = 0; j < 4; ++j) { const float dl = v[i][j] - mean; sq += dl * dl; }
      }
    const float rstd = 1.0f / sqrtf(warp_sum(sq) / cols + eps);
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      const int c = 4 * lane + 128 * i;
      if (c < cols) {
        float o[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          o[j] = (v[i][j] - mean) * rstd * g[i][j] + bt[i][j];
          if (relu) o[j] = fmaxf(o[j], 0.f);
        }
        store4<TY>(y + row * cols + c, o);
        if (y32) store4<float>(y32 + row * cols + c, o);
      }
    }
    if (lane == 0) {
      if (mean_out) mean_out[row] = mean;
      if (rstd_out) rstd_out[row] = rstd;
    }
  }
}

int layernorm_fwd(const void* x, int x_dtype, const float* gamma, const float* beta, float eps, void* y, int y_dtype,
                  float* y32, float* mean, float* rstd, int64_t rows, int cols, int relu, cudaStream_t s) {
  return layernorm_fwd_copy(x, x_dtype, gamma, beta, eps, y, y_dtype, y32, mean, rstd, rows, cols, relu, nullptr, s);
}
// + xcopy (optional): fp32 copy of the input rows, written in the same pass
int layernorm_fwd_copy(const void* x, int x_dtype, const float* gamma, const float* beta, float eps, void* y, int y_dtype,
                       float* y32, float* mean, float* rstd, int64_t rows, int cols, int relu, float* xcopy, cudaStream_t s) {
  if (rows == 0) return 0;
  const int grid = grid_for(rows, 8 * 2);
  const bool vec = (cols % 4 == 0) && cols <= 1024 && ((reinterpret_cast<uintptr_t>(x) & 15) == 0) &&
                   ((reinterpret_cast<uintptr_t>(y) & 15) == 0) && ((reinterpret_cast<uintptr_t>(gamma) & 15) == 0) &&
                   ((reinterpret_cast<uintptr_t>(beta) & 15) == 0) && (!y32 || (reinterpret_cast<uintptr_t>(y32) & 15) == 0);
  // x and y dtypes are independent: the inner dispatch runs in a lambda so that the outer one gets its result
#define LN_FWD(...) DISPATCH_DTYPE(x_dtype, TX, [&] { DISPATCH_DTYPE(y_dtype, TY, __VA_ARGS__); return 0; }())
#define LN_FWD_VEC(NV)                                                                                                  \
  LN_FWD(launch(ln_fwd_vec_kernel<TX, TY, NV>, grid, 256, 0, s, (const TX*)x, gamma, beta, eps, (TY*)y, y32, mean, rstd, rows, cols, relu, \
                (vec && x_dtype == F32 && (reinterpret_cast<uintptr_t>(xcopy) & 15) == 0) ? xcopy : (float*)nullptr))
  if (vec && cols <= 256) LN_FWD_VEC(2);
  else if (vec && cols <= 512) LN_FWD_VEC(4);
  else if (vec) LN_FWD_VEC(8);
  else LN_FWD(launch(ln_fwd_kernel<TX, TY>, grid, 256, 0, s, (const TX*)x, gamma, beta, eps, (TY*)y, y32, mean, rstd, rows, cols, relu));
#undef LN_FWD_VEC
#undef LN_FWD
  if (xcopy && !(vec && x_dtype == F32 && (reinterpret_cast<uintptr_t>(xcopy) & 15) == 0)) {
    B200ST_CHECK(x_dtype == F32, "layernorm_fwd_copy needs fp32 input rows");
    B200ST_CUDA(cudaMemcpyAsync(xcopy, x, sizeof(float) * (size_t)rows * cols, cudaMemcpyDeviceToDevice, s));
  }
  return 0;
}

// =============================================================================================
// LayerNorm backward: warp per row for dx; per-lane column partials for dgamma/dbeta, block-reduced
// =============================================================================================
template <typename TDY, typename TX, typename TDX, int CPL>
__global__ void __launch_bounds__(256) ln_bwd_kernel(const TDY* __restrict__ dy, const TX* __restrict__ x,
                                                      const float* __restrict__ mean, const float* __restrict__ rstd,
                                                      const float* __restrict__ gamma, const float* __restrict__ beta,
                                                      const float* __restrict__ dres, TDX* __restrict__ dx,
                                                      float* __restrict__ dgamma, float* __restrict__ dbeta, int64_t rows,
                                                      int cols, int relu) {
  pdl_wait();
  pdl_trigger();
  extern __shared__ float sm[];   // [2][cols] block partials
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
  for (int c = threadIdx.x; c < 2 * cols; c += blockDim.x) sm[c] = 0.f;
  __syncthreads();
  float gam[CPL], bet[CPL], dg_acc[CPL], db_acc[CPL];
#pragma unroll
  for (int i = 0; i < CPL; ++i) {
    const int c = lane + 32 * i;
    gam[i] = c < cols ? gamma[c] : 0.f; bet[i] = c < cols ? beta[c] : 0.f;
    dg_acc[i] = 0.f; db_acc[i] = 0.f;
  }
  const int64_t warps_total = (int64_t)gridDim.x * nwarps;
  for (int64_t row = (int64_t)blockIdx.x * nwarps + warp; row < rows; row += warps_total) {
    const float mu = mean[row], rs = rstd[row];
    float xh[CPL], d[CPL];
    float c1 = 0.f, c2 = 0.f;
#pragma unroll
    for (int i = 0; i < CPL; ++i) {
      const int c = lane + 32 * i;
      xh[i] = 0.f; d[i] = 0.f;
      if (c < cols) {
        xh[i] = (to_f32(x[row * cols + c]) - mu) * rs;
        float dd = to_f32(dy[row * cols + c]);
        if (relu && (xh[i] * gam[i] + bet[i]) <= 0.f) dd = 0.f;
        d[i] = dd;
        const float g = dd * gam[i];
        c1 += g; c2 += g * xh[i];
        dg_acc[i] += dd * xh[i]; db_acc[i] += dd;
      }
    }
    c1 = warp_sum(c1) / cols; c2 = warp_sum(c2) / cols;
#pragma unroll
    for (int i = 0; i < CPL; ++i) {
      const int c = lane + 32 * i;
      if (c < cols) {
        float v = rs * (d[i] * gam[i] - c1 - xh[i] * c2);
        if (dres) v += dres[row * cols + c];
        dx[row * cols + c] = from_f32<TDX>(v);
      }
    }
  }
#pragma unroll
  for (int i = 0; i < CPL; ++i) {
    const int c = lane + 32 * i;
    if (c < cols) { atomicAdd(&sm[c], dg_acc[i]); atomicAdd(&sm[cols + c], db_acc[i]); }
  }
  __syncthreads();
  for (int c = threadIdx.x; c < cols; c += blockDim.x) {
    if (dgamma) atomicAdd(&dgamma[c], sm[c]);
    if (dbeta) atomicAdd(&dbeta[c], sm[cols + c]);
  }
}

// vector variant: cols % 4 == 0, lane owns NV groups of 4 contiguous columns
template <typename TDY, typename TX, typename TDX, int NV, int R>
__global__ void __launch_bounds__(256, 2) ln_bwd_vec_kernel(const TDY* __restrict__ dy, const TX* __restrict__ x,
                                                          const float* __restrict__ mean, const float* __restrict__ rstd,
                                                          const float* __restrict__ gamma, const float* __restrict__ beta,
                                                          const float* __restrict__ dres, TDX* __restrict__ dx,
                                                          float* __restrict__ dgamma, float* __restrict__ dbeta, int64_t rows,
                                                          int cols, int relu, void* __restrict__ dnext, int dnext_dt,
                                                          const DropoutSpec ndrop) {
  pdl_wait();
  pdl_trigger();
  extern __shared__ float sm[];   // [nwarps][2][cols] per-warp partials (no shared-memory atomics)
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
  float gam[NV][4], bet[NV][4], dg_acc[NV][4], db_acc[NV][4];
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    const int c = 4 * lane + 128 * i;
#pragma unroll
    for (int j = 0; j < 4; ++j) { gam[i][j] = 0.f; bet[i][j] = 0.f; dg_acc[i][j] = 0.f; db_acc[i][j] = 0.f; }
    if (c < cols) { load4<float>(gamma + c, gam[i]); load4<float>(beta + c, bet[i]); }
  }
  // R rows per warp iteration with every global load (x, dy, residual gradient, statistics) issued up front: with a few
  // rows per warp the kernel is bound by bytes in flight (Little's law), not by bandwidth
  const int64_t warps_total = (int64_t)gridDim.x * nwarps;
  for (int64_t row0 = ((int64_t)blockIdx.x * nwarps + warp) * R; row0 < rows; row0 += warps_total * R) {
    float xh[R][NV][4], d[R][NV][4], rr[R][NV][4], mu[R], rs[R];
    uint32_t kb[R][NV];          // keep-bits of the NEXT block's post-dropout for this lane's 4-column groups (dnext only)
#pragma unroll
    for (int r = 0; r < R; ++r) {
      const int64_t row = row0 + r;
      const bool rv = row < rows;
      mu[r] = rv ? mean[row] : 0.f; rs[r] = rv ? rstd[row] : 0.f;
#pragma unroll
      for (int i = 0; i < NV; ++i) {
        const int c = 4 * lane + 128 * i;
#pragma unroll
        for (int j = 0; j < 4; ++j) { xh[r][i][j] = 0.f; d[r][i][j] = 0.f; rr[r][i][j] = 0.f; }
        if (rv && c < cols) {
          load4<TX>(x + row * cols + c, xh[r][i]);
          load4<TDY>(dy + row * cols + c, d[r][i]);
          if (dres) load4<float>(dres + row * cols + c, rr[r][i]);
          kb[r][i] = 0xffu;
          if (dnext && ndrop.bits) kb[r][i] = __ldg(ndrop.bits + ((uint64_t)(row * cols + c) >> 3));   // bitmap only (host guarantees); raw byte, used after the math
        }
      }
    }
    float c1[R], c2[R];
#pragma unroll
    for (int r = 0; r < R; ++r) {
      c1[r] = 0.f; c2[r] = 0.f;
      const bool rv = row0 + r < rows;
#pragma unroll
      for (int i = 0; i < NV; ++i) {
        const int c = 4 * lane + 128 * i;
        if (rv && c < cols) {
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            xh[r][i][j] = (xh[r][i][j] - mu[r]) * rs[r];
            if (relu && (xh[r][i][j] * gam[i][j] + bet[i][j]) <= 0.f) d[r][i][j] = 0.f;
            const float g = d[r][i][j] * gam[i][j];
            c1[r] += g; c2[r] += g * xh[r][i][j];
            dg_acc[i][j] += d[r][i][j] * xh[r][i][j]; db_acc[i][j] += d[r][i][j];
          }
        }
      }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
#pragma unroll
      for (int r = 0; r < R; ++r) { c1[r] += __shfl_xor_sync(0xffffffffu, c1[r], o); c2[r] += __shfl_xor_sync(0xffffffffu, c2[r], o); }
    }
#pragma unroll
    for (int r = 0; r < R; ++r) {
      const int64_t row = row0 + r;
      if (row >= rows) continue;
      const float m1 = c1[r] / cols, m2 = c2[r] / cols;
#pragma unroll
      for (int i = 0; i < NV; ++i) {
        const int c = 4 * lane + 128 * i;
        if (c < cols) {
          float o[4];
#pragma unroll
          for (int j = 0; j < 4; ++j) o[j] = rs[r] * (d[r][i][j] * gam[i][j] - m1 - xh[r][i][j] * m2) + rr[r][i][j];
          store4<TDX>(dx + row * cols + c, o);
          if (dnext) {
            // the consumer block's first op fused here: dY = cast(dropout'(dx)) in the activation dtype
            const float nscale = ndrop.p > 0.f ? ndrop.scale : 1.f;
            // element e = row * cols + c + j keeps bit e & 7 of byte e >> 3; c % 4 == 0, so that bit is
            // ((row * cols + c) & 4) + j (not (c & 4) + j: row * cols need not be a multiple of 8, e.g. cols % 8 == 4)
            const int bit0 = (int)((row * cols + c) & 4);
#pragma unroll
            for (int j = 0; j < 4; ++j) o[j] = ((kb[r][i] >> (bit0 + j)) & 1u) ? o[j] * nscale : 0.f;
            if (dnext_dt == BF16) store4<__nv_bfloat16>(reinterpret_cast<__nv_bfloat16*>(dnext) + row * cols + c, o);
            else if (dnext_dt == F16) store4<__half>(reinterpret_cast<__half*>(dnext) + row * cols + c, o);
            else store4<float>(reinterpret_cast<float*>(dnext) + row * cols + c, o);
          }
        }
      }
    }
  }
  float* mine = sm + (size_t)warp * 2 * cols;
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    const int c = 4 * lane + 128 * i;
    if (c < cols) {
      *reinterpret_cast<float4*>(mine + c) = make_float4(dg_acc[i][0], dg_acc[i][1], dg_acc[i][2], dg_acc[i][3]);
      *reinterpret_cast<float4*>(mine + cols + c) = make_float4(db_acc[i][0], db_acc[i][1], db_acc[i][2], db_acc[i][3]);
    }
  }
  __syncthreads();
  // one 16-byte vector reduction per 4 columns per block (4x fewer same-address L2 atomics than scalar atomicAdd)
  for (int v = threadIdx.x; v < 2 * (cols / 4); v += blockDim.x) {
    float4 a = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int w = 0; w < nwarps; ++w) {
      const float4 t = *reinterpret_cast<const float4*>(sm + (size_t)w * 2 * cols + 4 * v);
      a.x += t.x; a.y += t.y; a.z += t.z; a.w += t.w;
    }
    float* dst = (4 * v < cols) ? (dgamma ? dgamma + 4 * v : nullptr) : (dbeta ? dbeta + (4 * v - cols) : nullptr);
    if (dst) asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(dst), "f"(a.x), "f"(a.y), "f"(a.z), "f"(a.w) : "memory");
  }
}

int layernorm_bwd(const void* dy, int dy_dtype, const void* x, int x_dtype, const float* mean, const float* rstd,
                  const float* gamma, const float* beta, const float* dres, void* dx, int dx_dtype, float* dgamma,
                  float* dbeta, int64_t rows, int cols, int relu, cudaStream_t s) {
  return layernorm_bwd_next(dy, dy_dtype, x, x_dtype, mean, rstd, gamma, beta, dres, dx, dx_dtype, dgamma, dbeta, rows, cols, relu,
                            nullptr, F32, no_dropout(), s);
}

// Same, plus (dnext != null) dnext = cast(dropout'(dx)) in `dnext_dtype` with the NEXT backward block's post-dropout
// site — that block's first kernel, fused into this one.
int layernorm_bwd_next(const void* dy, int dy_dtype, const void* x, int x_dtype, const float* mean, const float* rstd,
                       const float* gamma, const float* beta, const float* dres, void* dx, int dx_dtype, float* dgamma,
                       float* dbeta, int64_t rows, int cols, int relu, void* dnext, int dnext_dtype, DropoutSpec ndrop,
                       cudaStream_t s) {
  if (rows == 0) return 0;
  B200ST_CHECK(cols <= 1024, "layernorm_bwd supports cols <= 1024");
  const int grid = grid_for(rows, 8 * 2, 132 * 8);      // 2 rows in flight per warp; long inputs loop
  const size_t smem = 2 * (size_t)cols * sizeof(float);
#define LN_BWD_LAUNCH(CPL)                                                                                              \
  DISPATCH_UNIFORM3(dy_dtype, x_dtype, dx_dtype, TT,                                                                    \
      (launch(ln_bwd_kernel<TT, TT, TT, CPL>, grid, 256, smem, s, (const TT*)dy, (const TT*)x, mean, rstd, gamma, beta, dres, \
                                                                (TT*)dx, dgamma, dbeta, rows, cols, relu)))
  const bool vec = (cols % 4 == 0) && ((reinterpret_cast<uintptr_t>(x) & 15) == 0) && ((reinterpret_cast<uintptr_t>(dy) & 15) == 0) &&
                   ((reinterpret_cast<uintptr_t>(dx) & 15) == 0) && ((reinterpret_cast<uintptr_t>(gamma) & 15) == 0) &&
                   ((reinterpret_cast<uintptr_t>(beta) & 15) == 0) && (!dres || (reinterpret_cast<uintptr_t>(dres) & 15) == 0);
#define LN_BWD_VEC(NV, RR)                                                                                                \
  DISPATCH_UNIFORM3(dy_dtype, x_dtype, dx_dtype, TT,                                                                    \
      (launch(ln_bwd_vec_kernel<TT, TT, TT, NV, RR>, grid, 256, smem * 8, s, (const TT*)dy, (const TT*)x, mean, rstd, gamma, beta, dres, \
                                                                   (TT*)dx, dgamma, dbeta, rows, cols, relu, fused_next ? dnext : nullptr, dnext_dtype, ndrop)))
  const bool vec_ok = vec && ((reinterpret_cast<uintptr_t>(dgamma) & 15) == 0) && ((reinterpret_cast<uintptr_t>(dbeta) & 15) == 0);
  const bool fused_next = dnext && vec_ok && cols <= 512 && ((reinterpret_cast<uintptr_t>(dnext) & 15) == 0) &&
                          (ndrop.p <= 0.f || ndrop.bits != nullptr);      // on-the-fly Philox sites use the separate kernel
  // short inputs (a few rows per warp) are bound by bytes in flight: 2 rows per warp iteration; long ones by occupancy
  if (vec_ok && cols <= 256 && rows <= 65536) LN_BWD_VEC(2, 2);
  else if (vec_ok && cols <= 256) LN_BWD_VEC(2, 1);
  else if (vec_ok && cols <= 512) LN_BWD_VEC(4, 1);      // 8 warps x 2 x 512 floats = 32 KB of per-warp partials
  else if (cols <= 256) LN_BWD_LAUNCH(8);
  else if (cols <= 512) LN_BWD_LAUNCH(16);
  else LN_BWD_LAUNCH(32);
#undef LN_BWD_VEC
#undef LN_BWD_LAUNCH
  if (dnext && !fused_next) {         // shapes outside the vector kernel: the separate kernel the fusion replaces
    B200ST_CHECK(dx_dtype == F32, "layernorm_bwd_next fallback needs an fp32 dx");
    B200ST_TRY(cast_dropout(reinterpret_cast<const float*>(dx), dnext, dnext_dtype, rows * cols, ndrop, s));
  }
  return 0;
}

// =============================================================================================
// softmax (+ additive key bias, diagonal key mask (KeyMask), dropout) : one warp per (b,h,q) row
// =============================================================================================
constexpr float kFloatMin = -1.0e9f;   // neurst/utils/compat.py:24

// Each lane owns groups of 8 consecutive keys (k = 8*(lane + 32*s) + j): 32-byte loads of S, 16-byte stores of P,
// one Philox call per group.  Dropout element index = row * ldP + k (ldP = Tk rounded up to 8), so groups never
// straddle rows.  The row (Tk <= 256*STEPS) lives in registers: S is read exactly once.
__device__ __forceinline__ float masked_logit(float v, const float* br, int k, int causal, int kmax_visible) {
  if (br) v += br[k];
  if (causal && k > kmax_visible) v += kFloatMin;
  return v;
}

template <typename T> __device__ __forceinline__ void load8(const T* src, float (&v)[8]);
template <> __device__ __forceinline__ void load8<float>(const float* src, float (&v)[8]) {
  const float4 a = *reinterpret_cast<const float4*>(src), b = *reinterpret_cast<const float4*>(src + 4);
  v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
}
template <int DT> __device__ __forceinline__ void load8_16(const void* src, float (&v)[8]) {
  const uint4 pk = *reinterpret_cast<const uint4*>(src);
  unpack8_16<DT>(pk, v);
}
template <> __device__ __forceinline__ void load8<__nv_bfloat16>(const __nv_bfloat16* src, float (&v)[8]) { load8_16<BF16>(src, v); }
template <> __device__ __forceinline__ void load8<__half>(const __half* src, float (&v)[8]) { load8_16<F16>(src, v); }

template <typename T, int STEPS>
__global__ void __launch_bounds__(256) softmax_fwd_kernel(const float* __restrict__ S, int64_t ldS,
                                                           const float* __restrict__ bias, KeyMask mask,
                                                           T* __restrict__ P_pre, T* __restrict__ P_drop, int64_t ldP,
                                                           int B, int H, int Tq, int Tk, DropoutSpec drop) {
  pdl_wait();
  pdl_trigger();
  const int lane = threadIdx.x & 31;
  const int64_t rows = (int64_t)B * H * Tq;
  const int64_t warps_total = (int64_t)gridDim.x * (blockDim.x >> 5);
  const uint32_t thresh = dropout_thresh16(drop.p);
  const int causal = mask.on, moff = mask.on ? key_mask_off(mask, Tk) : 0;
  for (int64_t row = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); row < rows; row += warps_total) {
    const int q = (int)(row % Tq);
    const int b = (int)(row / ((int64_t)H * Tq));
    const float* sr = S + row * ldS;
    const float* br = bias ? bias + (int64_t)b * Tk : nullptr;
    const int kmax_visible = q + moff;
    float v[STEPS][8];
    float mx = -INFINITY;
#pragma unroll
    for (int st = 0; st < STEPS; ++st) {
      const int k0 = 8 * (lane + 32 * st);
      if (k0 < Tk) {
        load8<float>(sr + k0, v[st]);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          v[st][j] = (k0 + j < Tk) ? masked_logit(v[st][j], br, k0 + j, causal, kmax_visible) : -INFINITY;
          mx = fmaxf(mx, v[st][j]);
        }
      }
    }
    mx = warp_max(mx);
    float sum = 0.f;
#pragma unroll
    for (int st = 0; st < STEPS; ++st) {
      const int k0 = 8 * (lane + 32 * st);
      if (k0 < Tk) {
#pragma unroll
        for (int j = 0; j < 8; ++j) { v[st][j] = (k0 + j < Tk) ? expf(v[st][j] - mx) : 0.f; sum += v[st][j]; }
      }
    }
    sum = warp_sum(sum);
    const float inv = 1.0f / sum;
#pragma unroll
    for (int st = 0; st < STEPS; ++st) {
      const int k0 = 8 * (lane + 32 * st);
      if (k0 < Tk) {
#pragma unroll
        for (int j = 0; j < 8; ++j) v[st][j] *= inv;
        store8<T>(P_pre + row * ldP + k0, v[st]);
        if (drop.p > 0.f) {
          const uint32_t keep = drop_keep8(drop, (uint64_t)(row * ldP + k0) >> 3, thresh);
          float w[8];
#pragma unroll
          for (int j = 0; j < 8; ++j) {
            // dropout acts on the stored (rounded) probability so that backward sees identical values
            const float ps = to_f32(from_f32<T>(v[st][j]));
            w[j] = ((keep >> j) & 1u) ? ps * drop.scale : 0.f;
          }
          store8<T>(P_drop + row * ldP + k0, w);
        }
      }
    }
  }
}

int softmax_fwd(const float* S, int64_t ldS, const float* bias, KeyMask mask, void* P_pre, void* P_drop, int p_dtype,
                int64_t ldP, int B, int H, int Tq, int Tk, DropoutSpec drop, cudaStream_t s) {
  const int64_t rows = (int64_t)B * H * Tq;
  if (rows == 0) return 0;
  B200ST_CHECK(ldS % 8 == 0 && ldP % 8 == 0 && ldS >= Tk && ldP >= Tk, "softmax needs row strides padded to 8");
  B200ST_CHECK((reinterpret_cast<uintptr_t>(S) & 31) == 0 && (reinterpret_cast<uintptr_t>(P_pre) & 15) == 0, "softmax alignment");
  B200ST_CHECK(Tk <= 2048, "softmax supports up to 2048 keys");
  const int grid = grid_for(rows, 8);
#define SM_FWD(ST) DISPATCH_DTYPE(p_dtype, T, (launch(softmax_fwd_kernel<T, ST>, grid, 256, 0, s, S, ldS, bias, mask, (T*)P_pre, \
                                                                                   (T*)P_drop, ldP, B, H, Tq, Tk, drop)))
  if (Tk <= 256) SM_FWD(1); else if (Tk <= 512) SM_FWD(2); else if (Tk <= 1024) SM_FWD(4); else SM_FWD(8);
#undef SM_FWD
  return 0;
}

template <typename T, int STEPS>
__global__ void __launch_bounds__(256) softmax_bwd_kernel(const float* __restrict__ dP, int64_t ldS,
                                                           const T* __restrict__ P_pre, T* __restrict__ dS, int64_t ldP,
                                                           int64_t rows, int Tk, DropoutSpec drop) {
  pdl_wait();
  pdl_trigger();
  const int lane = threadIdx.x & 31;
  const int64_t warps_total = (int64_t)gridDim.x * (blockDim.x >> 5);
  const uint32_t thresh = dropout_thresh16(drop.p);
  for (int64_t row = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); row < rows; row += warps_total) {
    float d[STEPS][8], pr[STEPS][8];
    float dot = 0.f;
#pragma unroll
    for (int st = 0; st < STEPS; ++st) {
      const int k0 = 8 * (lane + 32 * st);
      if (k0 < Tk) {
        load8<float>(dP + row * ldS + k0, d[st]);
        load8<T>(P_pre + row * ldP + k0, pr[st]);
        uint32_t keep = 0xffu;
        if (drop.p > 0.f) keep = drop_keep8(drop, (uint64_t)(row * ldP + k0) >> 3, thresh);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          if (k0 + j >= Tk) { d[st][j] = 0.f; pr[st][j] = 0.f; }
          if (drop.p > 0.f) d[st][j] = ((keep >> j) & 1u) ? d[st][j] * drop.scale : 0.f;
          dot += d[st][j] * pr[st][j];
        }
      }
    }
    dot = warp_sum(dot);
#pragma unroll
    for (int st = 0; st < STEPS; ++st) {
      const int k0 = 8 * (lane + 32 * st);
      if (k0 < Tk) {
        float o[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) o[j] = pr[st][j] * (d[st][j] - dot);
        store8<T>(dS + row * ldP + k0, o);
      }
    }
  }
}

int softmax_bwd(const float* dP, int64_t ldS, const void* P_pre, void* dS, int p_dtype, int64_t ldP, int64_t rows,
                int Tk, DropoutSpec drop, cudaStream_t s) {
  if (rows == 0) return 0;
  B200ST_CHECK(ldS % 8 == 0 && ldP % 8 == 0 && Tk <= 2048, "softmax_bwd needs row strides padded to 8 and Tk <= 2048");
  const int grid = grid_for(rows, 8);
#define SM_BWD(ST) DISPATCH_DTYPE(p_dtype, T, (launch(softmax_bwd_kernel<T, ST>, grid, 256, 0, s, dP, ldS, (const T*)P_pre, (T*)dS, \
                                                                                   ldP, rows, Tk, drop)))
  if (Tk <= 256) SM_BWD(1); else if (Tk <= 512) SM_BWD(2); else if (Tk <= 1024) SM_BWD(4); else SM_BWD(8);
#undef SM_BWD
  return 0;
}

// =============================================================================================
// elementwise: cast + dropout, posenc, fill, param cast
// =============================================================================================
template <typename T>
__global__ void __launch_bounds__(256) cast_dropout_kernel(const float* __restrict__ x, T* __restrict__ y, int64_t n,
                                                           DropoutSpec drop) {
  pdl_wait();
  pdl_trigger();
  const uint32_t thresh = dropout_thresh16(drop.p);
  const int64_t ngroups = (n + 7) / 8;
  const bool vec = (n % 8 == 0) && ((reinterpret_cast<uintptr_t>(x) & 31) == 0) && ((reinterpret_cast<uintptr_t>(y) & 15) == 0);
  for (int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; g < ngroups; g += (int64_t)gridDim.x * blockDim.x) {
    const uint32_t keep = drop.p > 0.f ? drop_keep8(drop, (uint64_t)g, thresh) : 0xffu;
    float v[8];
    if (vec) {
      load8<float>(x + g * 8, v);
#pragma unroll
      for (int j = 0; j < 8; ++j) v[j] = ((keep >> j) & 1u) ? v[j] * drop.scale : 0.f;
      store8<T>(y + g * 8, v);
    } else {
      for (int j = 0; j < 8 && g * 8 + j < n; ++j)
        y[g * 8 + j] = from_f32<T>(((keep >> j) & 1u) ? x[g * 8 + j] * drop.scale : 0.f);
    }
  }
}
int cast_dropout(const float* x, void* y, int y_dtype, int64_t n, DropoutSpec drop, cudaStream_t s) {
  if (n == 0) return 0;
  DISPATCH_DTYPE(y_dtype, T, (launch(cast_dropout_kernel<T>, grid_for((n + 7) / 8, 256), 256, 0, s, x, (T*)y, n, drop)));
  return 0;
}

// db[n] += sum_m dY[m,n].  Vector path: each thread owns 8 contiguous columns (16-byte bf16 / 32-byte fp32 loads), a warp
// covers 256 columns of one row, the 8 warps of a block stride over rows; partials meet in shared memory, one atomic per
// (block, column).
template <typename T>
__global__ void __launch_bounds__(256) colsum_vec_kernel(const T* __restrict__ dY, int64_t M, int N, int64_t ld, float* __restrict__ db) {
  pdl_wait();
  pdl_trigger();
  __shared__ float red[8][256 + 8];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int n0 = blockIdx.x * 256 + lane * 8;
  float acc[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) acc[j] = 0.f;
  if (n0 < N) {
    for (int64_t m = (int64_t)blockIdx.y * 8 + warp; m < M; m += (int64_t)gridDim.y * 8) {
      float v[8];
      load8<T>(dY + m * ld + n0, v);
#pragma unroll
      for (int j = 0; j < 8; ++j) acc[j] += v[j];
    }
  }
#pragma unroll
  for (int j = 0; j < 8; ++j) red[warp][lane * 8 + j] = acc[j];
  __syncthreads();
  const int c = threadIdx.x;
  const int n = blockIdx.x * 256 + c;
  if (n < N) {
    float t = 0.f;
#pragma unroll
    for (int w = 0; w < 8; ++w) t += red[w][c];
    atomicAdd(&db[n], t);
  }
}

template <typename T>
__global__ void colsum_kernel(const T* __restrict__ dY, int64_t M, int N, int64_t ld, float* __restrict__ db) {
  pdl_wait();
  pdl_trigger();
  __shared__ float red[8][33];
  const int n = blockIdx.x * 32 + threadIdx.x;
  float acc = 0.f;
  if (n < N)
    for (int64_t m = (int64_t)blockIdx.y * 8 + threadIdx.y; m < M; m += (int64_t)gridDim.y * 8) acc += to_f32(dY[m * ld + n]);
  red[threadIdx.y][threadIdx.x] = acc;
  __syncthreads();
  if (threadIdx.y == 0 && n < N) {
    float t = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) t += red[i][threadIdx.x];
    atomicAdd(&db[n], t);
  }
}
int colsum_accum(const void* dY, int dtype, int64_t M, int N, int64_t ld, float* db, cudaStream_t s) {
  if (M == 0 || N == 0) return 0;
  const int esz = dtype_size(dtype);
  const bool vec = (N % 8 == 0) && ((ld * esz) % (8 * esz) == 0) && ((reinterpret_cast<uintptr_t>(dY) & (8 * esz - 1)) == 0);
  if (vec) {
    const int gx = ceil_div(N, 256);
    int gy = (int)((M + 63) / 64);
    const int cap = (132 * 4 + gx - 1) / gx;
    if (gy > cap) gy = cap;
    if (gy < 1) gy = 1;
    DISPATCH_DTYPE(dtype, T, (launch(colsum_vec_kernel<T>, dim3(gx, gy), 256, 0, s, (const T*)dY, M, N, ld, db)));
  } else {
    dim3 block(32, 8);
    int gy = (int)((M + 255) / 256);
    if (gy > 64) gy = 64;
    if (gy < 1) gy = 1;
    dim3 grid(ceil_div(N, 32), gy);
    DISPATCH_DTYPE(dtype, T, (launch(colsum_kernel<T>, grid, block, 0, s, (const T*)dY, M, N, ld, db)));
  }
  return 0;
}

// sinusoid(t, c): [sin(t*w_i) | cos(t*w_i)], w_i = exp(-i * ln(1e4)/(d/2-1))  (common_layers.py:400-408)
__device__ __forceinline__ float sinusoid(int t, int c, int d) {
  const int half = d / 2;
  if (c >= 2 * half) return 0.f;   // odd d: zero pad
  const int i = c < half ? c : c - half;
  const double inc = log(1.0e4) / ((double)half - 1.0);
  const double arg = (double)t * exp(-(double)i * inc);
  return (float)(c < half ? sin(arg) : cos(arg));
}

__global__ void posenc_fwd_kernel(const float* __restrict__ v, float* __restrict__ x, int B, int T, int d, float scale,
                                  int t0, DropoutSpec drop) {
  pdl_wait();
  pdl_trigger();
  const int64_t n = (int64_t)B * T * d;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const int c = (int)(i % d);
    const int t = (int)((i / d) % T);
    float val = v[i] * scale + sinusoid(t + t0, c, d);
    if (drop.p > 0.f) val = drop_keep1(drop, (uint64_t)i) ? val * drop.scale : 0.f;
    x[i] = val;
  }
}
int posenc_fwd(const float* v, float* x, int B, int T, int d, float scale, int t0, DropoutSpec drop, cudaStream_t s) {
  const int64_t n = (int64_t)B * T * d;
  if (n == 0) return 0;
  return launch(posenc_fwd_kernel, grid_for(n, 256 * 2), 256, 0, s, v, x, B, T, d, scale, t0, drop);
}

template <typename T>
__global__ void posenc_bwd_kernel(const float* __restrict__ dx, T* __restrict__ dv, int64_t n, float scale, DropoutSpec drop) {
  pdl_wait();
  pdl_trigger();
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    float g = dx[i];
    if (drop.p > 0.f) g = drop_keep1(drop, (uint64_t)i) ? g * drop.scale : 0.f;
    dv[i] = from_f32<T>(g * scale);
  }
}
int posenc_bwd(const float* dx, void* dv, int dv_dtype, int64_t n, float scale, DropoutSpec drop, cudaStream_t s) {
  if (n == 0) return 0;
  DISPATCH_DTYPE(dv_dtype, T, (launch(posenc_bwd_kernel<T>, grid_for(n, 256 * 4), 256, 0, s, dx, (T*)dv, n, scale, drop)));
  return 0;
}

__global__ void embed_fwd_kernel(const int64_t* __restrict__ ids, const float* __restrict__ E, float* __restrict__ x, int B,
                                 int L, int d, int V, int t0, float scale, DropoutSpec drop) {
  pdl_wait();
  pdl_trigger();
  const int64_t n = (int64_t)B * L * d;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const int c = (int)(i % d);
    const int64_t bl = i / d;
    const int l = (int)(bl % L);
    int64_t id = ids[bl];
    id = id < 0 ? 0 : (id >= V ? V - 1 : id);
    float val = E[id * d + c] * scale + sinusoid(l + t0, c, d);
    if (drop.p > 0.f) val = drop_keep1(drop, (uint64_t)i) ? val * drop.scale : 0.f;
    x[i] = val;
  }
}
int embed_fwd(const int64_t* ids, const float* E, float* x, int B, int L, int d, int V, int t0, DropoutSpec drop,
              cudaStream_t s) {
  const int64_t n = (int64_t)B * L * d;
  if (n == 0) return 0;
  return launch(embed_fwd_kernel, grid_for(n, 256 * 2), 256, 0, s, ids, E, x, B, L, d, V, t0, sqrtf((float)d), drop);
}
__global__ void embed_bwd_kernel(const int64_t* __restrict__ ids, const float* __restrict__ dx, float* __restrict__ dE,
                                 int B, int L, int d, int V, float scale, DropoutSpec drop) {
  pdl_wait();
  pdl_trigger();
  const int64_t n = (int64_t)B * L * d;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const int c = (int)(i % d);
    const int64_t bl = i / d;
    int64_t id = ids[bl];
    id = id < 0 ? 0 : (id >= V ? V - 1 : id);
    float g = dx[i];
    if (drop.p > 0.f) g = drop_keep1(drop, (uint64_t)i) ? g * drop.scale : 0.f;
    atomicAdd(&dE[id * d + c], g * scale);
  }
}
int embed_bwd(const int64_t* ids, const float* dx, float* dE, int B, int L, int d, int V, DropoutSpec drop, cudaStream_t s) {
  const int64_t n = (int64_t)B * L * d;
  if (n == 0) return 0;
  return launch(embed_bwd_kernel, grid_for(n, 256 * 2), 256, 0, s, ids, dx, dE, B, L, d, V, sqrtf((float)d), drop);
}

__global__ void length_to_bias_kernel(const int64_t* __restrict__ lengths, float* __restrict__ bias, int B, int T, int n_halvings,
                                      int32_t* __restrict__ klen) {
  pdl_wait();
  pdl_trigger();
  const int64_t n = (int64_t)B * T;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const int b = (int)(i / T), t = (int)(i % T);
    int64_t len = lengths[b];
    for (int h = 0; h < n_halvings; ++h) len = (len + 1) / 2;
    bias[i] = t >= len ? kFloatMin : 0.f;
    if (klen && t == 0) klen[b] = (int32_t)(len < 1 ? T : (len > T ? T : len));     // number of leading non-padded keys
  }
}
int length_to_bias(const int64_t* lengths, float* bias, int B, int T, int n_halvings, cudaStream_t s, int32_t* klen) {
  if ((int64_t)B * T == 0) return 0;
  return launch(length_to_bias_kernel, grid_for((int64_t)B * T, 256), 256, 0, s, lengths, bias, B, T, n_halvings, klen);
}
__global__ void padding_to_bias_kernel(const float* __restrict__ padding, float* __restrict__ bias, int64_t n) {
  pdl_wait();
  pdl_trigger();
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    bias[i] = padding[i] * kFloatMin;
}
int padding_to_bias(const float* padding, float* bias, int64_t n, cudaStream_t s) {
  if (n == 0) return 0;
  return launch(padding_to_bias_kernel, grid_for(n, 256), 256, 0, s, padding, bias, n);
}

// =============================================================================================
// label-smoothed cross entropy: one block per (b,l) row of V logits
// =============================================================================================
__device__ __forceinline__ float block_reduce(float v, float* sm, bool is_max) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  v = is_max ? warp_max(v) : warp_sum(v);
  __syncthreads();
  if (lane == 0) sm[warp] = v;
  __syncthreads();
  float r = (threadIdx.x < (blockDim.x >> 5)) ? sm[threadIdx.x] : (is_max ? -INFINITY : 0.f);
  if (warp == 0) {
    r = is_max ? warp_max(r) : warp_sum(r);
    if (lane == 0) sm[0] = r;
  }
  __syncthreads();
  return sm[0];
}

template <typename T>
__global__ void __launch_bounds__(256) lsce_kernel(const float* __restrict__ logits, const int64_t* __restrict__ trg,
                                                    const int64_t* __restrict__ trg_length, int B, int L, int V,
                                                    float eps_ls, float* __restrict__ nll_sum, T* __restrict__ dlogits,
                                                    float loss_scale, const float* __restrict__ loss_scale_dev) {
  pdl_wait();
  pdl_trigger();
  if (loss_scale_dev) loss_scale *= *loss_scale_dev;
  __shared__ float sm[32];
  const int64_t row = blockIdx.x;
  const int b = (int)(row / L), l = (int)(row % L);
  const float w = (l < trg_length[b]) ? 1.f : 0.f;
  // total token count (every block recomputes it: B is small)
  float tok = 0.f;
  for (int i = threadIdx.x; i < B; i += blockDim.x) { int64_t len = trg_length[i]; tok += (float)(len < L ? (len < 0 ? 0 : len) : L); }
  const float total_tokens = block_reduce(tok, sm, false);
  const float* z = logits + row * V;
  float mx = -INFINITY;
  for (int v = threadIdx.x; v < V; v += blockDim.x) mx = fmaxf(mx, z[v]);
  mx = block_reduce(mx, sm, true);
  float se = 0.f, sz = 0.f;
  for (int v = threadIdx.x; v < V; v += blockDim.x) { se += expf(z[v] - mx); sz += z[v]; }
  se = block_reduce(se, sm, false);
  sz = block_reduce(sz, sm, false);
  const float lse = mx + logf(se);
  int64_t label = trg[row];
  label = label < 0 ? 0 : (label >= V ? V - 1 : label);
  const float conf = 1.f - eps_ls;
  const float low = eps_ls / (float)(V - 1);
  if (threadIdx.x == 0) {
    const float lp_label = z[label] - lse;
    const float sum_lp = sz - (float)V * lse;
    float xent = -((conf - low) * lp_label + low * sum_lp);
    if (eps_ls > 0.f) xent -= -(conf * logf(conf) + (float)(V - 1) * low * logf(low + 1e-20f));
    atomicAdd(&nll_sum[b], xent * w);
  }
  if (dlogits) {
    const float coef = (total_tokens > 0.f) ? w * loss_scale / total_tokens : 0.f;
    T* dz = dlogits + row * V;
    for (int v = threadIdx.x; v < V; v += blockDim.x) {
      const float p = expf(z[v] - lse);
      dz[v] = from_f32<T>(coef * (p - (v == label ? conf : low)));
    }
  }
}

// Row held in registers (V <= 1024 * NV, V % 4 == 0): the fp32 logits are read from HBM exactly once.
template <typename T, int NV>
__global__ void __launch_bounds__(256) lsce_vec_kernel(const float* __restrict__ logits, const int64_t* __restrict__ trg,
                                                        const int64_t* __restrict__ trg_length, int B, int L, int V,
                                                        float eps_ls, float* __restrict__ nll_sum, T* __restrict__ dlogits,
                                                        float loss_scale, const float* __restrict__ loss_scale_dev) {
  pdl_wait();
  pdl_trigger();
  if (loss_scale_dev) loss_scale *= *loss_scale_dev;
  __shared__ float sm[32];
  const int64_t row = blockIdx.x;
  const int b = (int)(row / L), l = (int)(row % L);
  const float w = (l < trg_length[b]) ? 1.f : 0.f;
  float tok = 0.f;
  for (int i = threadIdx.x; i < B; i += blockDim.x) { int64_t len = trg_length[i]; tok += (float)(len < L ? (len < 0 ? 0 : len) : L); }
  const float total_tokens = block_reduce(tok, sm, false);
  const float* z = logits + row * V;
  float4 r[NV];
  float mx = -INFINITY, sz = 0.f;
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    const int v = 4 * (threadIdx.x + 256 * i);
    if (v < V) {
      r[i] = __ldg(reinterpret_cast<const float4*>(z + v));
      mx = fmaxf(fmaxf(mx, fmaxf(r[i].x, r[i].y)), fmaxf(r[i].z, r[i].w));
      sz += (r[i].x + r[i].y) + (r[i].z + r[i].w);
    }
  }
  mx = block_reduce(mx, sm, true);
  float se = 0.f;
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    const int v = 4 * (threadIdx.x + 256 * i);
    if (v < V) {
      r[i].x = expf(r[i].x - mx); r[i].y = expf(r[i].y - mx); r[i].z = expf(r[i].z - mx); r[i].w = expf(r[i].w - mx);
      se += (r[i].x + r[i].y) + (r[i].z + r[i].w);
    }
  }
  se = block_reduce(se, sm, false);
  sz = block_reduce(sz, sm, false);
  const float lse = mx + logf(se);
  int64_t label = trg[row];
  label = label < 0 ? 0 : (label >= V ? V - 1 : label);
  const float conf = 1.f - eps_ls;
  const float low = eps_ls / (float)(V - 1);
  if (threadIdx.x == 0) {
    const float lp_label = z[label] - lse;
    const float sum_lp = sz - (float)V * lse;
    float xent = -((conf - low) * lp_label + low * sum_lp);
    if (eps_ls > 0.f) xent -= -(conf * logf(conf) + (float)(V - 1) * low * logf(low + 1e-20f));
    atomicAdd(&nll_sum[b], xent * w);
  }
  if (dlogits) {
    const float coef = (total_tokens > 0.f) ? w * loss_scale / total_tokens : 0.f;
    const float inv_se = 1.0f / se;
    T* dz = dlogits + row * V;
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      const int v = 4 * (threadIdx.x + 256 * i);
      if (v < V) {
        float o[4] = {r[i].x * inv_se, r[i].y * inv_se, r[i].z * inv_se, r[i].w * inv_se};
#pragma unroll
        for (int j = 0; j < 4; ++j) o[j] = coef * (o[j] - ((v + j) == label ? conf : low));
        store4<T>(dz + v, o);
      }
    }
  }
}

__global__ void lsce_finalize_kernel(const float* __restrict__ nll_sum, const int64_t* __restrict__ trg_length, int B, int L,
                                     float* __restrict__ n_tokens, float* __restrict__ loss) {
  pdl_wait();
  pdl_trigger();
  __shared__ float sm[32];
  float a = 0.f, t = 0.f;
  for (int i = threadIdx.x; i < B; i += blockDim.x) {
    int64_t len = trg_length[i];
    const float tk = (float)(len < L ? (len < 0 ? 0 : len) : L);
    n_tokens[i] = tk;
    a += nll_sum[i]; t += tk;
  }
  a = block_reduce(a, sm, false);
  t = block_reduce(t, sm, false);
  if (threadIdx.x == 0) loss[0] = a / t;
}

int lsce_fwd_bwd(const float* logits, const int64_t* trg, const int64_t* trg_length, int B, int L, int V,
                 float label_smoothing, float* nll_sum, float* n_tokens, float* loss, void* dlogits, int d_dtype,
                 float loss_scale, const float* loss_scale_dev, cudaStream_t s) {
  if (B * L == 0) return 0;
  B200ST_CUDA(cudaMemsetAsync(nll_sum, 0, sizeof(float) * B, s));
  const bool vec = (V % 4 == 0) && ((reinterpret_cast<uintptr_t>(logits) & 15) == 0) && (!dlogits || (reinterpret_cast<uintptr_t>(dlogits) & 15) == 0);
  if (vec && V <= 8192)
    DISPATCH_DTYPE(d_dtype, T, (launch(lsce_vec_kernel<T, 8>, B * L, 256, 0, s, logits, trg, trg_length, B, L, V, label_smoothing,
                                           nll_sum, (T*)dlogits, loss_scale, loss_scale_dev)));
  else if (vec && V <= 32768)
    DISPATCH_DTYPE(d_dtype, T, (launch(lsce_vec_kernel<T, 32>, B * L, 256, 0, s, logits, trg, trg_length, B, L, V, label_smoothing,
                                           nll_sum, (T*)dlogits, loss_scale, loss_scale_dev)));
  else
    DISPATCH_DTYPE(d_dtype, T, (launch(lsce_kernel<T>, B * L, 256, 0, s, logits, trg, trg_length, B, L, V, label_smoothing, nll_sum,
                                           (T*)dlogits, loss_scale, loss_scale_dev)));
  return launch(lsce_finalize_kernel, 1, 256, 0, s, nll_sum, trg_length, B, L, n_tokens, loss);
}

__global__ void dropout_bits_kernel(DropoutSpec drop, int64_t ngroups, uint8_t* __restrict__ out) {
  pdl_wait();
  pdl_trigger();
  const uint32_t thresh = dropout_thresh16(drop.p);
  const uint64_t seed = dropout_seed(drop);
  for (int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; g < ngroups; g += (int64_t)gridDim.x * blockDim.x)
    out[g] = (uint8_t)dropout_keep8(seed, drop.stream, (uint64_t)g, thresh);
}
int dropout_bits(DropoutSpec drop, int64_t n_elems, uint8_t* out, cudaStream_t s) {
  const int64_t ng = (n_elems + 7) / 8;
  if (ng == 0) return 0;
  return launch(dropout_bits_kernel, grid_for(ng, 256), 256, 0, s, drop, ng, out);
}
__global__ void __launch_bounds__(256) dropout_bits_multi_kernel(const DropBitsTable t, uint64_t seed, const uint64_t* seed_ptr,
                                                                  uint8_t* __restrict__ base) {
  pdl_wait();
  pdl_trigger();
  const uint64_t sd = seed_ptr ? *seed_ptr : seed;
  const int64_t total = t.goff[t.n];
  // 4 consecutive groups (= 4 output bytes) per thread: one site lookup and one 32-bit store when the 4 groups lie in one
  // site and the destination is 4-byte aligned (site byte offsets are 256-byte aligned, so this is the common case)
  const int64_t total4 = (total + 3) >> 2;
  for (int64_t q = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; q < total4; q += (int64_t)gridDim.x * blockDim.x) {
    const int64_t g0 = q << 2;
    int lo = 0, hi = t.n - 1;                      // last site whose first group <= g0
    while (lo < hi) { const int mid = (lo + hi + 1) >> 1; if (t.goff[mid] <= g0) lo = mid; else hi = mid - 1; }
    const int64_t local = g0 - t.goff[lo];
    if (g0 + 3 < t.goff[lo + 1] && ((t.boff[lo] + local) & 3) == 0) {
      uint32_t w = 0;
#pragma unroll
      for (int j = 0; j < 4; ++j) w |= dropout_keep8(sd, t.stream[lo], (uint64_t)(local + j), t.thresh[lo]) << (8 * j);
      *reinterpret_cast<uint32_t*>(base + t.boff[lo] + local) = w;
    } else {
      for (int64_t g = g0; g < g0 + 4 && g < total; ++g) {
        int l2 = lo;
        while (l2 + 1 < t.n && t.goff[l2 + 1] <= g) ++l2;
        const int64_t loc = g - t.goff[l2];
        base[t.boff[l2] + loc] = (uint8_t)dropout_keep8(sd, t.stream[l2], (uint64_t)loc, t.thresh[l2]);
      }
    }
  }
}
int dropout_bits_multi(const DropBitsTable& t, uint64_t seed, const uint64_t* seed_ptr, uint8_t* base, cudaStream_t s) {
  if (t.n == 0 || t.goff[t.n] == 0) return 0;
  return launch(dropout_bits_multi_kernel, grid_for((t.goff[t.n] + 3) / 4, 256, 132 * 8), 256, 0, s, t, seed, seed_ptr, base);
}
__global__ void fill_kernel(float* __restrict__ x, float v, int64_t n) {
  pdl_wait();
  pdl_trigger();
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) x[i] = v;
}
int fill_f32(float* x, float v, int64_t n, cudaStream_t s) {
  if (n == 0) return 0;
  return launch(fill_kernel, grid_for(n, 256 * 4), 256, 0, s, x, v, n);
}

}  // namespace b200st
