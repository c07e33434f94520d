// Incremental (cached) decoding and greedy search on the device — SURVEY.md §8 f1, BASELINE cfg-5.
//
// Replaces, for beam_size = 1, the loop  sequence_beam_search -> symbols_to_logits_fn -> TransformerDecoder.call(cache)
//   neurst/layers/search/beam_search.py:254-439 (search loop, finished / EOS / UNK / min-length masking :70-138,373-395)
//   neurst/models/encoder_decoder_model.py:211-261 (symbols_to_logits_fn: embed(time) -> decoder(cache) -> logits)
//   neurst/layers/decoders/transformer_decoder.py:105-147,171-228 (cache creation, cached step)
//   neurst/layers/decoders/transformer_layers.py:156-170 (memorize_memory: the encoder output is projected to K/V once)
//   neurst/layers/attentions/multi_head_attention.py:271-289 (self-attention key/value cache)
//
// A decoding step has M = B rows: every contraction is a matrix-vector product bound by reading the weights once
// (21.6 MB in 16-bit per token for speech_transformer_s, SURVEY §8d: >= 4 us/token at HBM speed), so this is plain
// CUDA-core code: split-K GEMV kernels whose blocks stream disjoint weight tiles with coalesced loads and reduce with
// fp32 atomics, one block per (head, batch) for the two attentions (fused with their output projection), the final
// LayerNorm fused into the tied logits product, and one block for argmax / finished masks / log-probabilities.  The
// key/value caches are preallocated ([layers][2][B][max_len][d]) — nothing grows, nothing is copied.  One step is ~40
// launches; the whole step is captured ONCE into a CUDA graph (the position `time` and the token ids live in device
// memory) and replayed per token.
//
// Weights are read either from the fp32 master arena (token ids identical to an fp32 reference) or from the 16-bit
// shadow (half the bytes).  All arithmetic and both caches are fp32.
#include "model.cuh"
#include "pdl.cuh"

#include <cmath>
#include <vector>

namespace b200st {

namespace {

constexpr int MAXB = 8;        // rows per step (batch x beam = batch for greedy)
constexpr float kFloatMin = -1.0e9f;

template <typename TW> __device__ __forceinline__ float wf(const TW* p, int64_t i) { return to_f32(p[i]); }

__device__ __forceinline__ float block_sum(float v, float* sm) {
  v = warp_sum(v);
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5, nw = (blockDim.x + 31) >> 5;
  __syncthreads();
  if (lane == 0) sm[w] = v;
  __syncthreads();
  float t = (threadIdx.x < nw) ? sm[threadIdx.x] : 0.f;
  if (w == 0) { t = warp_sum(t); if (lane == 0) sm[0] = t; }
  __syncthreads();
  return sm[0];
}
__device__ __forceinline__ float block_max(float v, float* sm) {
  v = warp_max(v);
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5, nw = (blockDim.x + 31) >> 5;
  __syncthreads();
  if (lane == 0) sm[w] = v;
  __syncthreads();
  float t = (threadIdx.x < nw) ? sm[threadIdx.x] : -INFINITY;
  if (w == 0) { t = warp_max(t); if (lane == 0) sm[0] = t; }
  __syncthreads();
  return sm[0];
}

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

// One block per (head, row): attention of the current position over the cached keys, fused with the output projection
// (accumulated straight into the residual stream x).  SELF: q/k/v come from the qkv accumulator, k/v are appended to the
// cache at position `time` (multi_head_attention.py:271-276); else q from `qsrc`, keys = pre-projected memory with the
// additive memory bias.  q is scaled by dh^-0.5 after the projection bias (multi_head_attention.py:203).
template <typename TW, bool SELF>
__global__ void __launch_bounds__(256) attn_step_kernel(const float* __restrict__ qsrc, int q_ld, float* __restrict__ kcache,
                                                        float* __restrict__ vcache, int kv_ld, int cache_rows,
                                                        const float* __restrict__ mem_bias, const TW* __restrict__ Wo,
                                                        const float* __restrict__ bo, float* __restrict__ x, int d, int dh, int Tm,
                                                        const int* __restrict__ time_dev) {
  pdl_wait();
  pdl_trigger();
  extern __shared__ float sm[];          // q[dh] | ctx[dh] | scores[nk] | red[8]
  const int h = blockIdx.x, b = blockIdx.y;
  const int t = *time_dev;
  const int nk = SELF ? t + 1 : Tm;
  float* q = sm;
  float* ctx = sm + dh;
  float* sc = sm + 2 * dh;
  float* red = sc + nk;
  const float* qrow = qsrc + (int64_t)b * q_ld + h * dh;
  float* kbase = kcache + (int64_t)b * cache_rows * kv_ld + h * dh;
  float* vbase = vcache + (int64_t)b * cache_rows * kv_ld + h * dh;
  const float alpha = rsqrtf((float)dh);
  for (int c = threadIdx.x; c < dh; c += blockDim.x) {
    q[c] = qrow[c] * alpha;
    if (SELF) {
      kbase[(int64_t)t * kv_ld + c] = qrow[d + c];
      vbase[(int64_t)t * kv_ld + c] = qrow[2 * d + c];
    }
  }
  __syncthreads();
  // scores: one thread per key — its dh-float key row is read with independent 16-byte loads (no cross-lane reduction,
  // every load of the row in flight at once: the loop is latency-bound otherwise)
  for (int j = threadIdx.x; j < nk; j += blockDim.x) {
    const float* kr = kbase + (int64_t)j * kv_ld;
    float s = 0.f;
    if ((dh & 3) == 0) {
#pragma unroll 4
      for (int c = 0; c < dh; c += 4) {
        const float4 kk = *reinterpret_cast<const float4*>(kr + c);
        s = fmaf(q[c], kk.x, fmaf(q[c + 1], kk.y, fmaf(q[c + 2], kk.z, fmaf(q[c + 3], kk.w, s))));
      }
    } else {
      for (int c = 0; c < dh; ++c) s = fmaf(q[c], kr[c], s);
    }
    sc[j] = s + ((!SELF && mem_bias) ? mem_bias[(int64_t)b * Tm + j] : 0.f);
  }
  __syncthreads();
  float mx = -INFINITY;
  for (int j = threadIdx.x; j < nk; j += blockDim.x) mx = fmaxf(mx, sc[j]);
  mx = block_max(mx, red);
  float se = 0.f;
  for (int j = threadIdx.x; j < nk; j += blockDim.x) { const float e = expf(sc[j] - mx); sc[j] = e; se += e; }
  se = block_sum(se, red);
  const float inv = 1.f / se;
  // ctx[c] = sum_j p_j V[j][c]: thread = (column c, key partition); 4 independent partial sums per thread
  for (int c = threadIdx.x; c < dh; c += blockDim.x) ctx[c] = 0.f;
  __syncthreads();
  {
    const int c = threadIdx.x % dh, part = threadIdx.x / dh, nparts = blockDim.x / dh > 0 ? blockDim.x / dh : 1;
    if (part < nparts) {
      float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;
      int j = part;
      for (; j + 3 * nparts < nk; j += 4 * nparts) {
        a0 = fmaf(sc[j], vbase[(int64_t)j * kv_ld + c], a0);
        a1 = fmaf(sc[j + nparts], vbase[(int64_t)(j + nparts) * kv_ld + c], a1);
        a2 = fmaf(sc[j + 2 * nparts], vbase[(int64_t)(j + 2 * nparts) * kv_ld + c], a2);
        a3 = fmaf(sc[j + 3 * nparts], vbase[(int64_t)(j + 3 * nparts) * kv_ld + c], a3);
      }
      for (; j < nk; j += nparts) a0 = fmaf(sc[j], vbase[(int64_t)j * kv_ld + c], a0);
      atomicAdd(&ctx[c], (a0 + a1 + a2 + a3) * inv);
    }
  }
  __syncthreads();
  // output projection of this head's slice: x[b, n] += sum_c ctx[c] * Wo[h*dh + c, n]  (+ bias once)
  for (int n = threadIdx.x; n < d; n += blockDim.x) {
    float a = (h == 0 && bo) ? bo[n] : 0.f;
    const TW* wp = Wo + (int64_t)h * dh * d + n;
#pragma unroll 8
    for (int c = 0; c < dh; ++c) a = fmaf(ctx[c], wf(wp, (int64_t)c * d), a);
    atomicAdd(x + (int64_t)b * d + n, a);
  }
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

// Greedy selection of the reference's search step with beam_size = 1 (beam_search.py:70-138,373-395): log_softmax; rows
// already finished emit EOS; UNK masked by FLOAT_MIN unless enabled; EOS masked while time < min_len - 1; argmax (lowest
// index on ties, like tf.nn.top_k); finished <- (token == EOS); accumulated log-probability and length.
struct GreedyState {
  int64_t* ids;          // [B] current input ids (in/out)
  int32_t* finished;     // [B]
  int32_t* length;       // [B] decoding length
  float* logprob;        // [B] accumulated log probability
  int64_t* out;          // [B, max_steps]
  int32_t* time;         // [1]
  int32_t* all_finished; // [1]
};
__global__ void __launch_bounds__(1024) greedy_pick_kernel(const float* __restrict__ logits, GreedyState g, int B, int V, int eos, int unk,
                                                           int min_len, int max_steps) {
  pdl_wait();
  pdl_trigger();
  __shared__ float red[32];
  __shared__ float sval[32];
  __shared__ int sidx[32];
  const int t = *g.time;
  int fin_all = 1;
  for (int b = 0; b < B; ++b) {
    const float* z = logits + (int64_t)b * V;
    const bool was_finished = g.finished[b] != 0;
    float mx = -INFINITY;
    for (int v = threadIdx.x; v < V; v += blockDim.x) mx = fmaxf(mx, z[v]);
    mx = block_max(mx, red);
    float se = 0.f;
    for (int v = threadIdx.x; v < V; v += blockDim.x) se += expf(z[v] - mx);
    se = block_sum(se, red);
    const float lse = mx + logf(se);
    float best = -INFINITY; int bi = 0x7fffffff;
    for (int v = threadIdx.x; v < V; v += blockDim.x) {
      float lp = z[v] - lse;
      if (was_finished) lp = (v == eos) ? 0.f : kFloatMin;
      if (v == unk) lp += kFloatMin;
      if (v == eos && t < min_len - 1) lp += kFloatMin;
      if (lp > best || (lp == best && v < bi)) { best = lp; bi = v; }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float ob = __shfl_xor_sync(0xffffffffu, best, o);
      const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
      if (ob > best || (ob == best && oi < bi)) { best = ob; bi = oi; }
    }
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    __syncthreads();
    if (lane == 0) { sval[w] = best; sidx[w] = bi; }
    __syncthreads();
    if (threadIdx.x == 0) {
      for (int i = 1; i < (int)(blockDim.x >> 5); ++i)
        if (sval[i] > sval[0] || (sval[i] == sval[0] && sidx[i] < sidx[0])) { sval[0] = sval[i]; sidx[0] = sidx[i]; }
      const int tok = sidx[0];
      g.out[(int64_t)b * max_steps + t] = tok;
      g.ids[b] = tok;
      g.logprob[b] += sval[0];
      g.length[b] += was_finished ? 0 : 1;
      g.finished[b] = (tok == eos) ? 1 : 0;
    }
    __syncthreads();
    fin_all &= (sidx[0] == eos) ? 1 : 0;
    __syncthreads();
  }
  if (threadIdx.x == 0) { *g.time = t + 1; *g.all_finished = fin_all; }
}

__global__ void greedy_init_kernel(GreedyState g, const int64_t* __restrict__ bos, int B, int max_steps, int eos) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < B) { g.ids[i] = bos[i]; g.finished[i] = 0; g.length[i] = 0; g.logprob[i] = 0.f; }
  if (i == 0) { *g.time = 0; *g.all_finished = 0; }
  for (int j = i; j < B * max_steps; j += gridDim.x * blockDim.x) g.out[j] = eos;   // padded with EOS (beam_search.py:428-436)
}


// =============================================================================================================
// Persistent greedy search: ONE cooperative launch decodes the whole hypothesis.  Every block is resident (grid = #SMs),
// the phases of a token (embed | per layer: LN+QKV, self-attention+out-proj, LN+Q, cross-attention+out-proj, LN+FFN1,
// ReLU+FFN2 | LN+logits | pick) are separated by a grid-wide barrier (one atomic + spin on a monotonic counter)
// instead of a kernel boundary (a launch latency each), work items of a phase are distributed round-robin over
// the blocks.  Data produced by other blocks in an earlier phase is read with ld.global.cg (L1 is not coherent);
// weights and the cross-attention memory never change and go through the read-only path.
// =============================================================================================================
struct LayerOffs {          // arena offsets (elements) of one decoder layer's tensors
  int64_t s_lng, s_lnb, s_qkv, s_qkvb, s_out, s_outb;
  int64_t c_lng, c_lnb, c_q, c_qb, c_out, c_outb;
  int64_t f_lng, f_lnb, f_w1, f_b1, f_w2, f_b2;
};
constexpr int kMaxDecLayers = 12;
struct PersistentArgs {
  LayerOffs layer[kMaxDecLayers];
  int64_t emb, emb_bias, out_lng, out_lnb;
  int n_layers, B, d, H, ffn, V, Tm, max_len, cross;
  float eps;
  const float* params;            // fp32 master arena (biases, LayerNorm parameters; weights too when TW = float)
  float* scratch;                 // layout_of(): x | qkv | qc | hid | logits
  int64_t o_x, o_qkv, o_qc, o_hid, o_logits;
  float* self_kv; float* cross_kv; const float* mem_bias;
  GreedyState g;
  int eos, unk, min_len, max_steps;
  unsigned int* barrier;          // monotonic arrival counter (zeroed before the launch)
};

__device__ __forceinline__ void grid_barrier(unsigned int* ctr, unsigned int& target) {
  __syncthreads();
  if (threadIdx.x == 0) {
    target += gridDim.x;
    __threadfence();
    atomicAdd(ctr, 1u);
    while (*reinterpret_cast<volatile unsigned int*>(ctr) < target) { }
    __threadfence();
  }
  __syncthreads();
}

// one (column tile of 256, K slice of 16) work item of  y[b, n] += sum_k f(in[b, k]) W[k, n]   (256 threads)
template <typename TW, int PRE>
__device__ __forceinline__ void gemv_item(int item, const float* in, const float* gamma, const float* beta, const float* pre_bias, float eps,
                                          const TW* __restrict__ W, const float* bias, float* y, int B, int K, int N, float* xs, float* red) {
  constexpr int KS = 16;
  const int n_tiles = (N + 255) / 256;
  const int nt = item % n_tiles, ks = item / n_tiles;
  const int k0 = ks * KS, kn = min(KS, K - k0);
  for (int b = 0; b < B; ++b) {
    float mean = 0.f, rstd = 1.f;
    if (PRE == 0) {
      float s = 0.f;
      for (int k = threadIdx.x; k < K; k += blockDim.x) s += __ldcg(in + (int64_t)b * K + k);
      mean = block_sum(s, red) / (float)K;
      float q = 0.f;
      for (int k = threadIdx.x; k < K; k += blockDim.x) { const float dlt = __ldcg(in + (int64_t)b * K + k) - mean; q += dlt * dlt; }
      rstd = rsqrtf(block_sum(q, red) / (float)K + eps);
    }
    if ((int)threadIdx.x < kn) {
      const int k = k0 + threadIdx.x;
      float v = __ldcg(in + (int64_t)b * K + k);
      if (PRE == 0) v = (v - mean) * rstd * gamma[k] + beta[k];
      else v = fmaxf(v + pre_bias[k], 0.f);
      xs[b * KS + threadIdx.x] = v;
    }
  }
  __syncthreads();
  const int n = nt * 256 + threadIdx.x;
  if (n < N) {
    float acc[MAXB];
#pragma unroll
    for (int b = 0; b < MAXB; ++b) acc[b] = 0.f;
    const TW* wp = W + (int64_t)k0 * N + n;
#pragma unroll 8
    for (int k = 0; k < kn; ++k) {
      const float w = wf(wp, (int64_t)k * N);
#pragma unroll
      for (int b = 0; b < MAXB; ++b) acc[b] = fmaf(xs[b * KS + k], w, acc[b]);
    }
    const float bb = (bias && ks == 0) ? bias[n] : 0.f;
#pragma unroll
    for (int b = 0; b < MAXB; ++b)
      if (b < B) atomicAdd(y + (int64_t)b * N + n, acc[b] + bb);
  }
  __syncthreads();
}

// one (head, row) work item: attention of the current position over the cached keys + output projection into x
template <typename TW, bool SELF>
__device__ __forceinline__ void attn_item(int h, int b, int t, const float* qsrc, int q_ld, float* kcache, float* vcache, int kv_ld,
                                          int cache_rows, const float* mem_bias, const TW* __restrict__ Wo, const float* bo, float* x, int d,
                                          int dh, int Tm, float* sm) {
  const int nk = SELF ? t + 1 : Tm;
  float* q = sm;
  float* ctx = sm + dh;
  float* sc = sm + 2 * dh;
  float* red = sc + nk;
  const float* qrow = qsrc + (int64_t)b * q_ld + h * dh;
  float* kbase = kcache + (int64_t)b * cache_rows * kv_ld + h * dh;
  float* vbase = vcache + (int64_t)b * cache_rows * kv_ld + h * dh;
  const float alpha = rsqrtf((float)dh);
  for (int c = threadIdx.x; c < dh; c += blockDim.x) {
    q[c] = __ldcg(qrow + c) * alpha;
    if (SELF) {
      kbase[(int64_t)t * kv_ld + c] = __ldcg(qrow + d + c);
      vbase[(int64_t)t * kv_ld + c] = __ldcg(qrow + 2 * d + c);
    }
    ctx[c] = 0.f;
  }
  __syncthreads();
  for (int j = threadIdx.x; j < nk; j += blockDim.x) {
    const float* kr = kbase + (int64_t)j * kv_ld;
    float s = 0.f;
    if ((dh & 3) == 0) {
#pragma unroll 4
      for (int c = 0; c < dh; c += 4) {
        const float4 kk = SELF ? __ldcg(reinterpret_cast<const float4*>(kr + c)) : __ldg(reinterpret_cast<const float4*>(kr + c));
        s = fmaf(q[c], kk.x, fmaf(q[c + 1], kk.y, fmaf(q[c + 2], kk.z, fmaf(q[c + 3], kk.w, s))));
      }
    } else {
      for (int c = 0; c < dh; ++c) s = fmaf(q[c], SELF ? __ldcg(kr + c) : __ldg(kr + c), s);
    }
    sc[j] = s + ((!SELF && mem_bias) ? mem_bias[(int64_t)b * Tm + j] : 0.f);
  }
  __syncthreads();
  float mx = -INFINITY;
  for (int j = threadIdx.x; j < nk; j += blockDim.x) mx = fmaxf(mx, sc[j]);
  mx = block_max(mx, red);
  float se = 0.f;
  for (int j = threadIdx.x; j < nk; j += blockDim.x) { const float e = expf(sc[j] - mx); sc[j] = e; se += e; }
  se = block_sum(se, red);
  const float inv = 1.f / se;
  {
    const int c = threadIdx.x % dh, part = threadIdx.x / dh, nparts = blockDim.x / dh > 0 ? blockDim.x / dh : 1;
    if (part < nparts) {
      float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;
      int j = part;
      for (; j + 3 * nparts < nk; j += 4 * nparts) {
        const float* v0 = vbase + (int64_t)j * kv_ld + c;
        a0 = fmaf(sc[j], SELF ? __ldcg(v0) : __ldg(v0), a0);
        a1 = fmaf(sc[j + nparts], SELF ? __ldcg(v0 + (int64_t)nparts * kv_ld) : __ldg(v0 + (int64_t)nparts * kv_ld), a1);
        a2 = fmaf(sc[j + 2 * nparts], SELF ? __ldcg(v0 + (int64_t)2 * nparts * kv_ld) : __ldg(v0 + (int64_t)2 * nparts * kv_ld), a2);
        a3 = fmaf(sc[j + 3 * nparts], SELF ? __ldcg(v0 + (int64_t)3 * nparts * kv_ld) : __ldg(v0 + (int64_t)3 * nparts * kv_ld), a3);
      }
      for (; j < nk; j += nparts) { const float* v0 = vbase + (int64_t)j * kv_ld + c; a0 = fmaf(sc[j], SELF ? __ldcg(v0) : __ldg(v0), a0); }
      atomicAdd(&ctx[c], (a0 + a1 + a2 + a3) * inv);
    }
  }
  __syncthreads();
  for (int n = threadIdx.x; n < d; n += blockDim.x) {
    float a = (h == 0 && bo) ? bo[n] : 0.f;
    const TW* wp = Wo + (int64_t)h * dh * d + n;
#pragma unroll 8
    for (int c = 0; c < dh; ++c) a = fmaf(ctx[c], wf(wp, (int64_t)c * d), a);
    atomicAdd(x + (int64_t)b * d + n, a);
  }
  __syncthreads();
}

template <typename TW>
__global__ void __launch_bounds__(256, 1) greedy_persistent_kernel(const __grid_constant__ PersistentArgs a, const TW* __restrict__ wbase) {
  extern __shared__ float dsm[];            // attention: q | ctx | scores | red ;  logits: normalised rows [B][d]
  __shared__ float xs[MAXB * 16];
  __shared__ float red[32];
  __shared__ float sval[32];
  __shared__ int sidx[32];
  const int B = a.B, d = a.d, H = a.H, dh = a.d / a.H, f = a.ffn, V = a.V;
  const float* P = a.params;
  float* x = a.scratch + a.o_x;
  float* logits = a.scratch + a.o_logits;
  unsigned int target = 0;
  const int nb = gridDim.x, bid = blockIdx.x;
  const float scale = sqrtf((float)d);
  for (int t = 0; t < a.max_steps; ++t) {
    // ---- embed the current symbols (position = t) and clear every accumulator of this token ----
    for (int i = bid * blockDim.x + threadIdx.x; i < B * d; i += nb * blockDim.x) {
      const int b = i / d, c = i % d;
      int64_t id = __ldcg(a.g.ids + b);
      id = id < 0 ? 0 : (id >= V ? V - 1 : id);
      x[i] = wf(wbase + a.emb, id * d + c) * scale + sinusoid_at(t, c, d);
    }
    for (int64_t i = (int64_t)bid * blockDim.x + threadIdx.x; i < a.o_logits - a.o_qkv; i += (int64_t)nb * blockDim.x)
      a.scratch[a.o_qkv + i] = 0.f;
    grid_barrier(a.barrier, target);
    for (int l = 0; l < a.n_layers; ++l) {
      const LayerOffs& L = a.layer[l];
      float* qkv = a.scratch + a.o_qkv + (int64_t)l * B * 3 * d;
      float* qc = a.scratch + a.o_qc + (int64_t)l * B * d;
      float* hid = a.scratch + a.o_hid + (int64_t)l * B * f;
      {
        const int items = ((3 * d + 255) / 256) * ((d + 15) / 16);
        for (int it = bid; it < items; it += nb)
          gemv_item<TW, 0>(it, x, P + L.s_lng, P + L.s_lnb, nullptr, a.eps, wbase + L.s_qkv, P + L.s_qkvb, qkv, B, d, 3 * d, xs, red);
      }
      grid_barrier(a.barrier, target);
      {
        float* sk = a.self_kv + (int64_t)l * 2 * B * a.max_len * d;
        float* sv = sk + (int64_t)B * a.max_len * d;
        for (int it = bid; it < H * B; it += nb)
          attn_item<TW, true>(it % H, it / H, t, qkv, 3 * d, sk, sv, d, a.max_len, nullptr, wbase + L.s_out, P + L.s_outb, x, d, dh, 0, dsm);
      }
      grid_barrier(a.barrier, target);
      if (a.cross) {
        {
          const int items = ((d + 255) / 256) * ((d + 15) / 16);
          for (int it = bid; it < items; it += nb)
            gemv_item<TW, 0>(it, x, P + L.c_lng, P + L.c_lnb, nullptr, a.eps, wbase + L.c_q, P + L.c_qb, qc, B, d, d, xs, red);
        }
        grid_barrier(a.barrier, target);
        {
          float* ck = a.cross_kv + (int64_t)l * B * a.Tm * 2 * d;
          for (int it = bid; it < H * B; it += nb)
            attn_item<TW, false>(it % H, it / H, t, qc, d, ck, ck + d, 2 * d, a.Tm, a.mem_bias, wbase + L.c_out, P + L.c_outb, x, d, dh, a.Tm, dsm);
        }
        grid_barrier(a.barrier, target);
      }
      {
        const int items = ((f + 255) / 256) * ((d + 15) / 16);
        for (int it = bid; it < items; it += nb)
          gemv_item<TW, 0>(it, x, P + L.f_lng, P + L.f_lnb, nullptr, a.eps, wbase + L.f_w1, nullptr, hid, B, d, f, xs, red);
      }
      grid_barrier(a.barrier, target);
      {
        const int items = ((d + 255) / 256) * ((f + 15) / 16);
        for (int it = bid; it < items; it += nb)
          gemv_item<TW, 1>(it, hid, nullptr, nullptr, P + L.f_b1, 0.f, wbase + L.f_w2, P + L.f_b2, x, B, f, d, xs, red);
      }
      grid_barrier(a.barrier, target);
    }
    // ---- final LayerNorm + tied logits: a warp per vocabulary row ----
    {
      float* xn = dsm;
      for (int b = 0; b < B; ++b) {
        float s = 0.f;
        for (int k = threadIdx.x; k < d; k += blockDim.x) s += __ldcg(x + (int64_t)b * d + k);
        const float mean = block_sum(s, red) / (float)d;
        float q = 0.f;
        for (int k = threadIdx.x; k < d; k += blockDim.x) { const float dlt = __ldcg(x + (int64_t)b * d + k) - mean; q += dlt * dlt; }
        const float rstd = rsqrtf(block_sum(q, red) / (float)d + a.eps);
        for (int k = threadIdx.x; k < d; k += blockDim.x)
          xn[b * d + k] = (__ldcg(x + (int64_t)b * d + k) - mean) * rstd * P[a.out_lng + k] + P[a.out_lnb + k];
      }
      __syncthreads();
      const int lane = threadIdx.x & 31, w = threadIdx.x >> 5, nw = blockDim.x >> 5;
      for (int v = bid * nw + w; v < V; v += nb * nw) {
        float acc[MAXB];
#pragma unroll
        for (int b = 0; b < MAXB; ++b) acc[b] = 0.f;
        for (int k = lane; k < d; k += 32) {
          const float e = wf(wbase + a.emb, (int64_t)v * d + k);
#pragma unroll
          for (int b = 0; b < MAXB; ++b) if (b < B) acc[b] = fmaf(xn[b * d + k], e, acc[b]);
        }
#pragma unroll
        for (int b = 0; b < MAXB; ++b) {
          if (b < B) {
            const float sres = warp_sum(acc[b]);
            if (lane == 0) logits[(int64_t)b * V + v] = sres + P[a.emb_bias + v];
          }
        }
      }
    }
    grid_barrier(a.barrier, target);
    // ---- greedy pick (block 0): the search step of sequence_beam_search with beam 1 ----
    if (bid == 0) {
      int fin_all = 1;
      for (int b = 0; b < B; ++b) {
        const float* z = logits + (int64_t)b * V;
        const bool was_finished = a.g.finished[b] != 0;
        float mx = -INFINITY;
        for (int v = threadIdx.x; v < V; v += blockDim.x) mx = fmaxf(mx, __ldcg(z + v));
        mx = block_max(mx, red);
        float se = 0.f;
        for (int v = threadIdx.x; v < V; v += blockDim.x) se += expf(__ldcg(z + v) - mx);
        se = block_sum(se, red);
        const float lse = mx + logf(se);
        float best = -INFINITY; int bi = 0x7fffffff;
        for (int v = threadIdx.x; v < V; v += blockDim.x) {
          float lp = __ldcg(z + v) - lse;
          if (was_finished) lp = (v == a.eos) ? 0.f : kFloatMin;
          if (v == a.unk) lp += kFloatMin;
          if (v == a.eos && t < a.min_len - 1) lp += kFloatMin;
          if (lp > best || (lp == best && v < bi)) { best = lp; bi = v; }
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
          const float ob = __shfl_xor_sync(0xffffffffu, best, o);
          const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
          if (ob > best || (ob == best && oi < bi)) { best = ob; bi = oi; }
        }
        const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
        __syncthreads();
        if (lane == 0) { sval[w] = best; sidx[w] = bi; }
        __syncthreads();
        if (threadIdx.x == 0) {
          for (int i = 1; i < (int)(blockDim.x >> 5); ++i)
            if (sval[i] > sval[0] || (sval[i] == sval[0] && sidx[i] < sidx[0])) { sval[0] = sval[i]; sidx[0] = sidx[i]; }
          const int tok = sidx[0];
          a.g.out[(int64_t)b * a.max_steps + t] = tok;
          a.g.ids[b] = tok;
          a.g.logprob[b] += sval[0];
          a.g.length[b] += was_finished ? 0 : 1;
          a.g.finished[b] = (tok == a.eos) ? 1 : 0;
        }
        __syncthreads();
        fin_all &= (sidx[0] == a.eos) ? 1 : 0;
        __syncthreads();
      }
      if (threadIdx.x == 0) { *a.g.time = t + 1; *a.g.all_finished = fin_all; }
    }
    grid_barrier(a.barrier, target);
    if (__ldcg(a.g.all_finished)) break;             // while not all finished (beam_search.py:414-418)
  }
}

struct DecodeLayout {      // offsets (floats) inside the scratch buffer
  int64_t x, qkv, qc, hid, logits, total;
};
DecodeLayout layout_of(const Config& c, int B) {
  DecodeLayout l{};
  int64_t o = 0;
  l.x = o; o += (int64_t)B * c.d;
  l.qkv = o; o += (int64_t)c.dec_layers * B * 3 * c.d;
  l.qc = o; o += (int64_t)c.dec_layers * B * c.d;
  l.hid = o; o += (int64_t)c.dec_layers * B * c.ffn;
  l.logits = o; o += (int64_t)B * c.vocab;
  l.total = o;
  return l;
}

struct StepCtx {
  const Model& m;
  Buffers buf;
  DecodeState st;
  cudaStream_t s;
  const float* P(const std::string& n) const { const int i = m.find(n); return i < 0 ? nullptr : buf.params + m.params[i].offset; }
  int64_t off(const std::string& n) const { const int i = m.find(n); return i < 0 ? -1 : m.params[i].offset; }
};

template <typename TW>
int step_launch(const StepCtx& c, const TW* wbase, const int64_t* ids, const int32_t* time_dev, float* logits_out) {
  const Config& cf = c.m.cfg;
  const DecodeState& st = c.st;
  const int B = st.B, d = cf.d, H = cf.heads, dh = d / H, f = cf.ffn, V = cf.vocab;
  const DecodeLayout lo = layout_of(cf, B);
  float* x = st.scratch + lo.x;
  // zero every accumulator of the step in one node (qkv / q / ffn hidden of all layers; logits are plain stores)
  B200ST_CUDA(cudaMemsetAsync(st.scratch + lo.qkv, 0, sizeof(float) * (size_t)(lo.logits - lo.qkv), c.s));
  auto W = [&](const std::string& n) { return wbase + c.off(n); };
  launch_pdl(embed_step_kernel<TW>, (B * d + 255) / 256, 256, 0, c.s, ids, W("trg.emb"), x, B, d, V, time_dev);
  const int64_t self_layer = 2 * (int64_t)B * st.max_len * d, cross_layer = (int64_t)B * st.Tm * 2 * d;
  for (int i = 0; i < cf.dec_layers; ++i) {
    const std::string p = "dec." + std::to_string(i);
    float* qkv = st.scratch + lo.qkv + (int64_t)i * B * 3 * d;
    float* qc = st.scratch + lo.qc + (int64_t)i * B * d;
    float* hid = st.scratch + lo.hid + (int64_t)i * B * f;
    // self attention block
    launch_pdl(gemv_kernel<TW, 0>, dim3((3 * d + 127) / 128, (d + 31) / 32), 128, 0, c.s, (const float*)x, c.P(p + ".self.ln.gamma"),
               c.P(p + ".self.ln.beta"), (const float*)nullptr, cf.ln_eps, W(p + ".self.qkv.kernel"), c.P(p + ".self.qkv.bias"), qkv, B, d, 3 * d);
    float* sk = st.self_kv + (int64_t)i * self_layer;
    float* sv = sk + (int64_t)B * st.max_len * d;
    const size_t smem_self = sizeof(float) * (size_t)(2 * dh + st.max_len + 8);
    launch_pdl(attn_step_kernel<TW, true>, dim3(H, B), 256, smem_self, c.s, (const float*)qkv, 3 * d, sk, sv, d, st.max_len,
               (const float*)nullptr, W(p + ".self.out.kernel"), c.P(p + ".self.out.bias"), x, d, dh, 0, time_dev);
    // encoder-decoder attention block over the pre-projected memory
    if (cf.with_cross_attention && st.Tm > 0) {
      launch_pdl(gemv_kernel<TW, 0>, dim3((d + 127) / 128, (d + 31) / 32), 128, 0, c.s, (const float*)x, c.P(p + ".cross.ln.gamma"),
                 c.P(p + ".cross.ln.beta"), (const float*)nullptr, cf.ln_eps, W(p + ".cross.q.kernel"), c.P(p + ".cross.q.bias"), qc, B, d, d);
      float* ck = st.cross_kv + (int64_t)i * cross_layer;
      const size_t smem_cross = sizeof(float) * (size_t)(2 * dh + st.Tm + 8);
      launch_pdl(attn_step_kernel<TW, false>, dim3(H, B), 256, smem_cross, c.s, (const float*)qc, d, ck, ck + d, 2 * d, st.Tm,
                 st.memory_bias, W(p + ".cross.out.kernel"), c.P(p + ".cross.out.bias"), x, d, dh, st.Tm, time_dev);
    }
    // feed-forward block
    launch_pdl(gemv_kernel<TW, 0>, dim3((f + 127) / 128, (d + 31) / 32), 128, 0, c.s, (const float*)x, c.P(p + ".ffn.ln.gamma"),
               c.P(p + ".ffn.ln.beta"), (const float*)nullptr, cf.ln_eps, W(p + ".ffn.w1"), (const float*)nullptr, hid, B, d, f);
    launch_pdl(gemv_kernel<TW, 1>, dim3((d + 127) / 128, (f + 31) / 32), 128, 0, c.s, (const float*)hid, (const float*)nullptr,
               (const float*)nullptr, c.P(p + ".ffn.b1"), 0.f, W(p + ".ffn.w2"), c.P(p + ".ffn.b2"), x, B, f, d);
    g_kernel_launches += cf.with_cross_attention && st.Tm > 0 ? 6 : 4;
  }
  launch_pdl(logits_step_kernel<TW>, 132 * 2, 256, sizeof(float) * (size_t)B * d, c.s, (const float*)x, c.P("dec.out_ln.gamma"),
             c.P("dec.out_ln.beta"), cf.ln_eps, W("trg.emb"), c.P("trg.bias"), logits_out, B, d, V);
  g_kernel_launches += 2;
  B200ST_LAUNCH_CHECK();
  return 0;
}

int step_dispatch(const StepCtx& c, const int64_t* ids, const int32_t* time_dev, float* logits_out) {
  if (c.st.use_shadow) {
    B200ST_CHECK(is16(c.m.adt) && c.buf.shadow, "use_shadow needs a 16-bit precision handle and its shadow arena");
    if (c.m.adt == F16) return step_launch(c, reinterpret_cast<const __half*>(c.buf.shadow), ids, time_dev, logits_out);
    return step_launch(c, reinterpret_cast<const __nv_bfloat16*>(c.buf.shadow), ids, time_dev, logits_out);
  }
  return step_launch(c, c.buf.params, ids, time_dev, logits_out);
}


// Whole search in one cooperative launch (greedy_persistent_kernel).  Returns 1 and leaves `done` false when the device
// cannot co-schedule the grid (the caller then falls back to the per-token graph).
template <typename TW>
int launch_persistent(const Model& m, const Buffers& buf, const DecodeState& st, const GreedyArgs& ga, const GreedyState& g,
                      const TW* wbase, cudaStream_t s, bool* done) {
  const Config& cf = m.cfg;
  *done = false;
  if (cf.dec_layers > kMaxDecLayers) return 0;
  PersistentArgs a{};
  auto off = [&](const std::string& n) -> int64_t { const int i = m.find(n); return i < 0 ? 0 : m.params[i].offset; };
  for (int i = 0; i < cf.dec_layers; ++i) {
    const std::string p = "dec." + std::to_string(i);
    LayerOffs& L = a.layer[i];
    L.s_lng = off(p + ".self.ln.gamma"); L.s_lnb = off(p + ".self.ln.beta"); L.s_qkv = off(p + ".self.qkv.kernel");
    L.s_qkvb = off(p + ".self.qkv.bias"); L.s_out = off(p + ".self.out.kernel"); L.s_outb = off(p + ".self.out.bias");
    L.c_lng = off(p + ".cross.ln.gamma"); L.c_lnb = off(p + ".cross.ln.beta"); L.c_q = off(p + ".cross.q.kernel");
    L.c_qb = off(p + ".cross.q.bias"); L.c_out = off(p + ".cross.out.kernel"); L.c_outb = off(p + ".cross.out.bias");
    L.f_lng = off(p + ".ffn.ln.gamma"); L.f_lnb = off(p + ".ffn.ln.beta"); L.f_w1 = off(p + ".ffn.w1"); L.f_b1 = off(p + ".ffn.b1");
    L.f_w2 = off(p + ".ffn.w2"); L.f_b2 = off(p + ".ffn.b2");
  }
  a.emb = off("trg.emb"); a.emb_bias = off("trg.bias"); a.out_lng = off("dec.out_ln.gamma"); a.out_lnb = off("dec.out_ln.beta");
  a.n_layers = cf.dec_layers; a.B = st.B; a.d = cf.d; a.H = cf.heads; a.ffn = cf.ffn; a.V = cf.vocab; a.Tm = st.Tm; a.max_len = st.max_len;
  a.cross = (cf.with_cross_attention && st.Tm > 0) ? 1 : 0;
  a.eps = cf.ln_eps;
  a.params = buf.params; a.scratch = st.scratch;
  const DecodeLayout lo = layout_of(cf, st.B);
  a.o_x = lo.x; a.o_qkv = lo.qkv; a.o_qc = lo.qc; a.o_hid = lo.hid; a.o_logits = lo.logits;
  a.self_kv = st.self_kv; a.cross_kv = st.cross_kv; a.mem_bias = st.memory_bias;
  a.g = g;
  a.eos = ga.eos_id; a.unk = ga.unk_id; a.min_len = ga.min_len; a.max_steps = ga.max_steps;
  a.barrier = reinterpret_cast<unsigned int*>(reinterpret_cast<char*>(ga.state_words) + 128);   // after ids / flags / time words
  const int dh = cf.d / cf.heads;
  size_t smem = sizeof(float) * (size_t)(2 * dh + (st.Tm > st.max_len ? st.Tm : st.max_len) + 8);
  const size_t smem_logits = sizeof(float) * (size_t)st.B * cf.d;
  if (smem_logits > smem) smem = smem_logits;
  auto kern = greedy_persistent_kernel<TW>;
  if (smem > 48 * 1024) B200ST_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  int dev = 0, sms = 0, coop = 0, per_sm = 0;
  B200ST_CUDA(cudaGetDevice(&dev));
  B200ST_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
  B200ST_CUDA(cudaDeviceGetAttribute(&coop, cudaDevAttrCooperativeLaunch, dev));
  B200ST_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, 256, smem));
  if (!coop || per_sm < 1) return 0;
  B200ST_CUDA(cudaMemsetAsync(a.barrier, 0, sizeof(unsigned int), s));
  void* args[2] = {(void*)&a, (void*)&wbase};
  const cudaError_t e = cudaLaunchCooperativeKernel((const void*)kern, dim3(sms), dim3(256), args, smem, s);
  if (e != cudaSuccess) { cudaGetLastError(); return 0; }
  ++g_kernel_launches;
  *done = true;
  return 0;
}

int check_state(const Model& m, const DecodeState& st) {
  const Config& cf = m.cfg;
  B200ST_CHECK(cf.model_type == MODEL_SPEECH || cf.model_type == MODEL_TEXT, "decoding needs an encoder-decoder handle");
  B200ST_CHECK(st.B >= 1 && st.B <= MAXB, "decode batch must be 1.." + std::to_string(MAXB));
  B200ST_CHECK(st.max_len >= 1 && st.Tm >= 0, "bad decode lengths");
  B200ST_CHECK(st.self_kv && st.scratch && (st.Tm == 0 || st.cross_kv), "decode state buffers missing");
  const int dh = cf.d / cf.heads;
  B200ST_CHECK(dh <= 256 && 256 % dh == 0, "decode kernels need a head dim that divides 256");
  const size_t smem = sizeof(float) * (size_t)(2 * dh + (st.Tm > st.max_len ? st.Tm : st.max_len) + 8);
  B200ST_CHECK(smem <= 200 * 1024, "decode: too many keys for the shared-memory score buffer");
  return 0;
}

template <typename K>
int raise_smem(K kern, size_t smem) {
  if (smem > 48 * 1024) B200ST_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  return 0;
}
int raise_all_smem(const Config& cf, const DecodeState& st) {
  const int dh = cf.d / cf.heads;
  const size_t smem = sizeof(float) * (size_t)(2 * dh + (st.Tm > st.max_len ? st.Tm : st.max_len) + 8);
  B200ST_TRY(raise_smem(attn_step_kernel<float, true>, smem)); B200ST_TRY(raise_smem(attn_step_kernel<float, false>, smem));
  B200ST_TRY(raise_smem(attn_step_kernel<__half, true>, smem)); B200ST_TRY(raise_smem(attn_step_kernel<__half, false>, smem));
  B200ST_TRY(raise_smem(attn_step_kernel<__nv_bfloat16, true>, smem)); B200ST_TRY(raise_smem(attn_step_kernel<__nv_bfloat16, false>, smem));
  return 0;
}

}  // namespace

static int g_last_greedy_graph = -1;
int last_greedy_used_graph() { return g_last_greedy_graph; }

int64_t decode_scratch_floats(const Model& m, int B) { return layout_of(m.cfg, B).total + 64; }

// memorize_memory (transformer_layers.py:156-160): K/V projections of the encoder output, once per utterance, fp32
int decode_init(const Model& m, const Buffers& buf, const float* enc_out, const DecodeState& st, cudaStream_t s) {
  B200ST_TRY(check_state(m, st));
  const Config& cf = m.cfg;
  if (!cf.with_cross_attention || st.Tm == 0) return 0;
  B200ST_CHECK(enc_out != nullptr && buf.params != nullptr, "decode_init needs the encoder output and the parameters");
  const int d = cf.d;
  for (int i = 0; i < cf.dec_layers; ++i) {
    const std::string p = "dec." + std::to_string(i) + ".cross.kv";
    const int wi = m.find(p + ".kernel"), bi = m.find(p + ".bias");
    B200ST_CHECK(wi >= 0 && bi >= 0, "cross-attention parameters missing");
    GemmArgs g = gemm_defaults();
    g.M = st.B * st.Tm; g.N = 2 * d; g.K = d;
    g.A = GemmOperand{enc_out, F32, 0, d, 0, 0};
    g.B = GemmOperand{buf.params + m.params[wi].offset, F32, 1, 2 * d, 0, 0};
    g.C = st.cross_kv + (int64_t)i * st.B * st.Tm * 2 * d; g.c_dtype = F32; g.ldc = 2 * d;
    g.epi.bias = buf.params + m.params[bi].offset;
    B200ST_TRY(gemm_simt_f32(g, s));
    ++g_kernel_launches;
  }
  return 0;
}

int decode_step(const Model& m, const Buffers& buf, const DecodeState& st, const int64_t* symbols, const int32_t* time_dev,
                float* logits, cudaStream_t s) {
  B200ST_TRY(check_state(m, st));
  B200ST_CHECK(symbols && time_dev && logits, "decode_step: null argument");
  B200ST_TRY(raise_all_smem(m.cfg, st));
  StepCtx c{m, buf, st, s};
  return step_dispatch(c, symbols, time_dev, logits);
}

// Whole greedy search: init -> [capture one step into a CUDA graph] -> replay until every row has emitted EOS (checked
// every 8 tokens through a pinned flag) or `max_steps`.  The caller's stream must not be capturing.
int greedy_search(const Model& m, const Buffers& buf, const DecodeState& st, const GreedyArgs& ga, cudaStream_t s) {
  B200ST_TRY(check_state(m, st));
  const Config& cf = m.cfg;
  B200ST_CHECK(ga.max_steps >= 1 && ga.max_steps <= st.max_len, "max_steps must be within the cache length");
  B200ST_CHECK(ga.bos_ids && ga.out_ids && ga.out_len && ga.out_logprob && ga.state_words, "greedy_search: null argument");
  B200ST_TRY(raise_all_smem(cf, st));
  // device words: [ids B x int64][finished B][length B][time][all_finished]
  char* w = reinterpret_cast<char*>(ga.state_words);
  GreedyState g{};
  g.ids = reinterpret_cast<int64_t*>(w); w += sizeof(int64_t) * MAXB;
  g.finished = reinterpret_cast<int32_t*>(w); w += sizeof(int32_t) * MAXB;
  g.length = ga.out_len;
  g.logprob = ga.out_logprob;
  g.out = ga.out_ids;
  g.time = reinterpret_cast<int32_t*>(w); w += sizeof(int32_t);
  g.all_finished = reinterpret_cast<int32_t*>(w);
  const DecodeLayout lo = layout_of(cf, st.B);
  float* logits = st.scratch + lo.logits;
  greedy_init_kernel<<<8, 256, 0, s>>>(g, ga.bos_ids, st.B, ga.max_steps, ga.eos_id);
  B200ST_CUDA(cudaGetLastError());
  if (ga.use_graph == 2) {       // persistent mode: one cooperative launch for the whole search
    bool done = false;
    if (st.use_shadow) {
      B200ST_CHECK(is16(m.adt) && buf.shadow, "use_shadow needs a 16-bit precision handle and its shadow arena");
      if (m.adt == F16) B200ST_TRY(launch_persistent(m, buf, st, ga, g, reinterpret_cast<const __half*>(buf.shadow), s, &done));
      else B200ST_TRY(launch_persistent(m, buf, st, ga, g, reinterpret_cast<const __nv_bfloat16*>(buf.shadow), s, &done));
    } else {
      B200ST_TRY(launch_persistent(m, buf, st, ga, g, buf.params, s, &done));
    }
    if (done) { g_last_greedy_graph = 2; return 0; }
  }
  StepCtx c{m, buf, st, s};
  auto one_step = [&]() -> int {
    B200ST_TRY(step_dispatch(c, g.ids, g.time, logits));
    launch_pdl(greedy_pick_kernel, 1, 1024, 0, s, (const float*)logits, g, st.B, cf.vocab, ga.eos_id, ga.unk_id, ga.min_len, ga.max_steps);
    ++g_kernel_launches;
    B200ST_LAUNCH_CHECK();
    return 0;
  };
  cudaGraph_t graph = nullptr;
  cudaGraphExec_t exec = nullptr;
  bool graphed = false;
  if (ga.use_graph) {
    B200ST_TRY(one_step());                     // step 0 eagerly (also warms function attributes outside the capture)
    if (cudaStreamBeginCapture(s, cudaStreamCaptureModeThreadLocal) == cudaSuccess) {
      const int rc = one_step();
      cudaError_t e = cudaStreamEndCapture(s, &graph);
      if (rc == 0 && e == cudaSuccess && graph && cudaGraphInstantiate(&exec, graph, 0) == cudaSuccess) graphed = true;
      else { cudaGetLastError(); pdl_launch_error() = cudaSuccess; }
    } else {
      cudaGetLastError();
    }
  }
  g_last_greedy_graph = graphed ? 1 : 0;
  static thread_local int32_t* flag_host = nullptr;     // pinned word for the "all rows finished" poll
  if (!flag_host) B200ST_CUDA(cudaMallocHost(&flag_host, sizeof(int32_t)));
  *flag_host = 0;
  int rc = 0;
  for (int t = ga.use_graph ? 1 : 0; t < ga.max_steps && rc == 0; ++t) {
    if (graphed) { if (cudaGraphLaunch(exec, s) != cudaSuccess) { set_last_error("decode graph launch failed"); rc = 1; } }
    else rc = one_step();
    if (rc == 0 && (t % 8 == 7 || t + 1 == ga.max_steps)) {
      cudaMemcpyAsync(flag_host, g.all_finished, sizeof(int32_t), cudaMemcpyDeviceToHost, s);
      if (cudaStreamSynchronize(s) != cudaSuccess) { set_last_error("decode step failed"); rc = 1; }
      if (*flag_host) break;
    }
  }
  if (exec) cudaGraphExecDestroy(exec);
  if (graph) cudaGraphDestroy(graph);
  return rc;
}

}  // namespace b200st
