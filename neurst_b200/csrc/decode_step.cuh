// The per-row kernels of a decoding step on at most 8 rows (decode.cu), shared with the streaming session (stream.cu): the
// embedding of the current symbols, the split-K GEMV with its LayerNorm / ReLU prologue, and the tied logits product.
#pragma once
#include "common.cuh"
#include "pdl.cuh"

namespace b200st {

namespace {

constexpr int MAXB = 8;        // rows per step (batch x beam = batch for greedy)

template <typename TW> __device__ __forceinline__ float wf(const TW* p, int64_t i) { return to_f32(p[i]); }

__device__ __forceinline__ float sinusoid_at(int t, int c, int d) {   // common_layers.py:400-408 (concat(sin, cos))
  const int half = d / 2;
  if (c >= 2 * half) return 0.f;
  const int i = c < half ? c : c - half;
  const double inc = log(1.0e4) / ((double)half - 1.0);
  const double arg = (double)t * exp(-(double)i * inc);
  return (float)(c < half ? sin(arg) : cos(arg));
}

// x[b,:] = E[ids[b],:] * sqrt(d) + sinusoid(time)   (text_modalities.py:84-92, common_layers.py:395-397,427-434)
template <typename TW>
__global__ void embed_step_kernel(const int64_t* __restrict__ ids, const TW* __restrict__ E, float* __restrict__ x, int B, int d, int V,
                                  const int* __restrict__ time_dev) {
  pdl_wait();
  pdl_trigger();
  const int t = *time_dev;
  const float scale = sqrtf((float)d);
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < B * d; i += gridDim.x * blockDim.x) {
    const int b = i / d, c = i % d;
    int64_t id = ids[b];
    id = id < 0 ? 0 : (id >= V ? V - 1 : id);
    x[i] = wf(E, id * d + c) * scale + sinusoid_at(t, c, d);
  }
}

// y[b, n] += sum_{k in this block's K slice} f(in[b, k]) * W[k, n]  (+ bias[n] from the first K slice), y zero-initialised
// or the residual stream itself.  PRE: 0 = LayerNorm(in) with gamma/beta (pre-norm block input, common_layers.py:73-85),
// 1 = relu(in + pre_bias) (FFN hidden, common_layers.py:156-160).  W is [K, N] row-major (TF [in, out]): a warp reads
// 32 consecutive columns of one row = one coalesced 64/128-byte segment.  grid = (N / 128 tiles, K / 32 slices).
template <typename TW, int PRE>
__global__ void __launch_bounds__(128) gemv_kernel(const float* __restrict__ in, const float* __restrict__ gamma, const float* __restrict__ beta,
                                                   const float* __restrict__ pre_bias, float eps, const TW* __restrict__ W,
                                                   const float* __restrict__ bias, float* __restrict__ y, int B, int K, int N) {
  pdl_wait();
  pdl_trigger();
  constexpr int KS = 32;
  __shared__ float xs[MAXB][KS];
  __shared__ float red[8];
  const int k0 = blockIdx.y * KS;
  const int kn = min(KS, K - k0);
  for (int b = 0; b < B; ++b) {
    float mean = 0.f, rstd = 1.f;
    if (PRE == 0) {
      float s = 0.f;
      for (int k = threadIdx.x; k < K; k += blockDim.x) s += in[(int64_t)b * K + k];
      mean = block_sum(s, red) / (float)K;
      float q = 0.f;
      for (int k = threadIdx.x; k < K; k += blockDim.x) { const float dlt = in[(int64_t)b * K + k] - mean; q += dlt * dlt; }
      rstd = rsqrtf(block_sum(q, red) / (float)K + eps);
    }
    if ((int)threadIdx.x < kn) {
      const int k = k0 + threadIdx.x;
      float v = in[(int64_t)b * K + k];
      if (PRE == 0) v = (v - mean) * rstd * gamma[k] + beta[k];
      else if (PRE == 1) v = fmaxf(v + pre_bias[k], 0.f);
      xs[b][threadIdx.x] = v;
    }
  }
  __syncthreads();
  const int n = blockIdx.x * 128 + threadIdx.x;
  if (n >= N) return;
  float acc[MAXB];
#pragma unroll
  for (int b = 0; b < MAXB; ++b) acc[b] = 0.f;
  const TW* wp = W + (int64_t)k0 * N + n;
#pragma unroll 8
  for (int k = 0; k < kn; ++k) {
    const float w = wf(wp, (int64_t)k * N);
#pragma unroll
    for (int b = 0; b < MAXB; ++b) acc[b] = fmaf(xs[b][k], w, acc[b]);
  }
  const float bb = (bias && blockIdx.y == 0) ? bias[n] : 0.f;
#pragma unroll
  for (int b = 0; b < MAXB; ++b)
    if (b < B) atomicAdd(y + (int64_t)b * N + n, acc[b] + bb);
}


// logits[b, v] = LN(x[b]) . E[v, :] + bias[v]   (tied output layer, text_modalities.py:104-108): warp per vocabulary row
template <typename TW>
__global__ void __launch_bounds__(256) logits_step_kernel(const float* __restrict__ x, const float* __restrict__ gamma,
                                                          const float* __restrict__ beta, float eps, const TW* __restrict__ E,
                                                          const float* __restrict__ bias, float* __restrict__ logits, int B, int d, int V) {
  pdl_wait();
  pdl_trigger();
  extern __shared__ float xs[];          // [B][d] normalised rows
  __shared__ float red[8];
  for (int b = 0; b < B; ++b) {
    float s = 0.f;
    for (int k = threadIdx.x; k < d; k += blockDim.x) s += x[(int64_t)b * d + k];
    const float mean = block_sum(s, red) / (float)d;
    float q = 0.f;
    for (int k = threadIdx.x; k < d; k += blockDim.x) { const float dlt = x[(int64_t)b * d + k] - mean; q += dlt * dlt; }
    const float rstd = rsqrtf(block_sum(q, red) / (float)d + eps);
    for (int k = threadIdx.x; k < d; k += blockDim.x) xs[b * d + k] = (x[(int64_t)b * d + k] - mean) * rstd * gamma[k] + beta[k];
  }
  __syncthreads();
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  for (int v = blockIdx.x * 8 + w; v < V; v += gridDim.x * 8) {
    float acc[MAXB];
#pragma unroll
    for (int b = 0; b < MAXB; ++b) acc[b] = 0.f;
    for (int k = lane; k < d; k += 32) {
      const float e = wf(E, (int64_t)v * d + k);
#pragma unroll
      for (int b = 0; b < MAXB; ++b) if (b < B) acc[b] = fmaf(xs[b * d + k], e, acc[b]);
    }
#pragma unroll
    for (int b = 0; b < MAXB; ++b) {
      if (b < B) {
        const float s = warp_sum(acc[b]);
        if (lane == 0) logits[(int64_t)b * V + v] = s + (bias ? bias[v] : 0.f);
      }
    }
  }
}

}  // namespace

}  // namespace b200st
