// Top-k / nucleus sampling (TopSampling, neurst/layers/search/sampling.py): the per-row selection of
// sequence_sampling_search (:103-250) with top_k_logits / top_p_logits (:76-100) and one categorical draw per row, and the
// state set-up of the search.  The search driver, which runs the decoder step on the utterances x sample_num rows, is
// sampling_search in decode.cu.
//
// A draw is keyed, not sequenced: row g (the global row index, row_offset + row) at step t takes
//   u = (x >> 8) * 2^-24,  x = the first word of philox4x32(seed, t, g)  (common.cuh, the dropout generator)
// and picks the first vocabulary index, in index order, whose running sum of kept weights exp(z_v - max) exceeds u * W
// (W their total).  Every reduction has a fixed order and no floating-point atomic is used, so a row's id depends only on
// its logits and its key: on the bit-reproducible wide step the sampled ids do not depend on the batch a row is decoded in.
#include "beam.cuh"

#include <algorithm>
#include <cmath>
#include <string>

namespace b200st {

namespace {

constexpr int kSampleThreads = 512;
constexpr int kRadixBits = 4;
constexpr int kRadixBuckets = 1 << kRadixBits;

// order-preserving uint32 key of a float: a < b  <=>  key(a) < key(b) (NaN aside)
__device__ __forceinline__ uint32_t order_key(float f) {
  const uint32_t u = __float_as_uint(f);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

// out[b] = sum over the block's threads of acc[b], lane order within a warp, then warp order.  sm: [32][kRadixBuckets].
__device__ __forceinline__ void block_sum_buckets(const float (&acc)[kRadixBuckets], float* sm, float* out) {
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5, nw = blockDim.x >> 5;
#pragma unroll
  for (int b = 0; b < kRadixBuckets; ++b) {
    const float v = warp_sum(acc[b]);
    if (lane == 0) sm[w * kRadixBuckets + b] = v;
  }
  __syncthreads();
  if ((int)threadIdx.x < kRadixBuckets) {
    float s = 0.f;
    for (int i = 0; i < nw; ++i) s += sm[i * kRadixBuckets + threadIdx.x];
    out[threadIdx.x] = s;
  }
  __syncthreads();
}

// The filter's threshold without sorting the row: the largest order key k* for which the weight of {v : key(z_v) >= k*}
// reaches `target` (> 0).  count: every element weighs 1 and target = k, so k* is the key of the k-th largest value,
// duplicates counted (top_k_logits).  Else an element weighs exp(z_v - mx) and target = p * W, so k* is the key of the
// largest value whose upper tail holds probability >= p (top_p_logits).  Radix select over the key, 4 bits per pass from
// the top: a pass sums the weights of the elements that share the prefix found so far into 16 buckets (per-thread
// registers, then a fixed-order block reduction) and descends into the highest bucket at which the weight at or above
// it reaches the target.  When none does (the prefix's weight, summed in another order, falls short of the target by
// rounding), the lowest bucket is taken: the threshold then keeps the whole prefix.
template <typename ZF>
__device__ uint32_t radix_threshold(ZF zf, int V, bool count, float mx, float target, float* sm, float* hist, uint32_t* sel) {
  uint32_t prefix = 0;
  float above = 0.f;                                   // thread 0: weight of the elements above the prefix
  for (int shift = 32 - kRadixBits; shift >= 0; shift -= kRadixBits) {
    const uint32_t hi_mask = shift + kRadixBits >= 32 ? 0u : (0xffffffffu << (shift + kRadixBits));
    float acc[kRadixBuckets];
#pragma unroll
    for (int b = 0; b < kRadixBuckets; ++b) acc[b] = 0.f;
    for (int v = threadIdx.x; v < V; v += blockDim.x) {
      const float z = zf(v);
      const uint32_t k = order_key(z);
      if ((k & hi_mask) == prefix) {
        const uint32_t digit = (k >> shift) & (kRadixBuckets - 1);
        const float w = count ? 1.f : expf(z - mx);
#pragma unroll
        for (int b = 0; b < kRadixBuckets; ++b) acc[b] += digit == (uint32_t)b ? w : 0.f;
      }
    }
    block_sum_buckets(acc, sm, hist);
    if (threadIdx.x == 0) {
      int d = 0;
      for (int b = kRadixBuckets - 1; b > 0; --b) {
        if (above + hist[b] >= target) { d = b; break; }
        above += hist[b];
      }
      *sel = prefix | ((uint32_t)d << shift);
    }
    __syncthreads();
    prefix = *sel;
  }
  return prefix;
}

// The draw: the first index v, in index order, whose running sum of weights wf(v) exceeds u * W.  Thread i owns the
// contiguous chunk [i*C, (i+1)*C); the chunk sums are scanned in thread order (a shuffle scan within the warp, then the
// warp totals in order), so a running sum has one association and the chunk intervals [lo, hi) of consecutive threads
// share their ends exactly.  The thread whose interval holds the target walks its chunk; if rounding leaves it short,
// the chunk's last positive weight is drawn.  A zero weight is never drawn.  Returns the index in every thread.
template <typename WF>
__device__ int draw_index(WF wf, int V, float u, float* sm, int* who, int* pick) {
  const int C = (V + blockDim.x - 1) / blockDim.x;
  const int lo_v = min(V, (int)threadIdx.x * C), hi_v = min(V, lo_v + C);
  float s = 0.f;
  for (int v = lo_v; v < hi_v; ++v) s += wf(v);
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5, nw = blockDim.x >> 5;
  float incl = s;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const float n = __shfl_up_sync(0xffffffffu, incl, o);
    if (lane >= o) incl += n;
  }
  float prev = __shfl_up_sync(0xffffffffu, incl, 1);
  if (lane == 0) prev = 0.f;
  if (lane == 31) sm[w] = incl;
  if (threadIdx.x == 0) { *who = 0x7fffffff; *pick = -1; }
  __syncthreads();
  if (threadIdx.x == 0) {
    float a = 0.f;
    for (int i = 0; i < nw; ++i) { const float t = sm[i]; sm[32 + i] = a; a += t; }
    sm[64] = a;
  }
  __syncthreads();
  const float lo = sm[32 + w] + prev, hi = sm[32 + w] + incl;
  const float target = u * sm[64];
  if (hi > target) atomicMin(who, (int)threadIdx.x);
  __syncthreads();
  int owner = *who;
  if (owner == 0x7fffffff) {
    // u * W rounded up to W: the last thread holding weight draws its chunk's last positive element
    __syncthreads();
    if (threadIdx.x == 0) *who = -1;
    __syncthreads();
    if (s > 0.f) atomicMax(who, (int)threadIdx.x);
    __syncthreads();
    owner = *who;
  }
  if ((int)threadIdx.x == owner) {
    float run = lo;
    int last = -1, got = -1;
    for (int v = lo_v; v < hi_v; ++v) {
      const float x = wf(v);
      if (x > 0.f) {
        last = v;
        run += x;
        if (run > target) { got = v; break; }
      }
    }
    *pick = got >= 0 ? got : last;
  }
  __syncthreads();
  return *pick;
}

// One block per row.  The search (SEARCH): a finished row emits EOS and keeps its length and log-probability; otherwise
// UNK is masked to FLOAT_MIN (_calculate_logits, :48-73) and so is EOS while time < min_len - 1 (:213-221), the filter
// keeps the logits at or above the threshold (top_p_logits when top_p < 1, else top_k_logits, top_k 0 keeping all), one
// id is drawn, and the row's log-probability grows by the masked, unfiltered log-softmax of that id.  The last block of
// the step publishes all_finished and advances `time`, as beam_select_kernel does.  Without SEARCH (b200st_sample_logits)
// the row is the caller's logits as they are and the draw is written to out[row].
template <bool SEARCH>
__global__ void __launch_bounds__(kSampleThreads) sample_select_kernel(const __grid_constant__ SampleRows a) {
  pdl_wait();
  pdl_trigger();
  __shared__ float red[32];
  __shared__ float sm[32 * kRadixBuckets];
  __shared__ float hist[kRadixBuckets];
  __shared__ uint32_t sel;
  __shared__ int who[2];
  const int r = blockIdx.x;
  const int t = SEARCH ? *a.time : a.step;
  const bool was_finished = SEARCH && a.finished[r] != 0;
  if (!was_finished) {
    const float* z = a.logits + (int64_t)r * a.V;
    const bool eos_masked = SEARCH && t < a.min_len - 1;
    auto zf = [&](int v) -> float {
      const float x = z[v];
      return (v == a.unk || (eos_masked && v == a.eos)) ? kFloatMin : x;
    };
    float mx = -INFINITY;
    for (int v = threadIdx.x; v < a.V; v += blockDim.x) mx = fmaxf(mx, zf(v));
    mx = block_max(mx, red);
    float se = 0.f;
    for (int v = threadIdx.x; v < a.V; v += blockDim.x) se += expf(zf(v) - mx);
    se = block_sum(se, red);
    uint32_t thr = 0;                                  // every key is >= 0: no filter
    if (a.top_p < 1.f) thr = radix_threshold(zf, a.V, false, mx, fmaxf(a.top_p * se, 1e-30f), sm, hist, &sel);
    else if (a.top_k > 0) thr = radix_threshold(zf, a.V, true, mx, (float)a.top_k, sm, hist, &sel);
    const Philox4 rnd = philox4x32(a.seed, (uint64_t)t, (uint64_t)(a.row_offset + r));
    const float u = (float)(rnd.x >> 8) * (1.f / 16777216.f);
    auto wf = [&](int v) -> float {
      const float x = zf(v);
      return order_key(x) >= thr ? expf(x - mx) : 0.f;
    };
    const int id = draw_index(wf, a.V, u, sm, who, who + 1);
    if (threadIdx.x == 0) {
      if (SEARCH) {
        a.out[(int64_t)r * a.max_steps + t] = id;
        a.ids[r] = id;
        a.logprob[r] += zf(id) - (mx + logf(se));
        a.length[r] += 1;
        a.finished[r] = id == a.eos ? 1 : 0;
      } else {
        a.out[r] = id;
      }
    }
  } else if (threadIdx.x == 0) {
    a.out[(int64_t)r * a.max_steps + t] = a.eos;
    a.ids[r] = a.eos;
  }
  if (SEARCH) {
    __threadfence();
    __syncthreads();
    if (threadIdx.x == 0) {
      __threadfence();
      if (atomicAdd(a.ticket, 1u) == gridDim.x - 1) {
        __threadfence();
        int all = 1;
        for (int i = 0; i < (int)gridDim.x; ++i) all &= __ldcg(a.finished + i) != 0 ? 1 : 0;
        *a.all_finished = all;
        *a.ticket = 0;
        *a.time = t + 1;
      }
    }
  }
}

// stack_beam_size of the decoder input, the row state, the identity ancestry table (every row reads its own
// self-attention cache) and the output rows padded with EOS (sampling.py:253-256)
__global__ void sample_init_kernel(BeamState s, const int64_t* __restrict__ bos, int rows, int sample_num, int max_len,
                                   int64_t* __restrict__ out, int max_steps, int eos, float* __restrict__ logprob,
                                   int32_t* __restrict__ length) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < rows) { s.ids[i] = bos[i / sample_num]; s.finished[i] = 0; logprob[i] = 0.f; length[i] = 0; }
  if (i == 0) { *s.time = 0; *s.all_finished = 0; *s.ticket = 0; }
  for (int64_t j = i; j < (int64_t)rows * max_len; j += (int64_t)gridDim.x * blockDim.x) s.anc[j] = (int)(j / max_len);
  for (int64_t j = i; j < (int64_t)rows * max_steps; j += (int64_t)gridDim.x * blockDim.x) out[j] = eos;
}

}  // namespace

int check_sample_filter(int top_k, float top_p, int V) {
  B200ST_CHECK(std::isfinite(top_p), "top_p must be finite, got " + std::to_string(top_p));
  B200ST_CHECK(top_k >= 0, "top_k must be >= 0 (0: no top-k filter), got " + std::to_string(top_k));
  B200ST_CHECK(top_k <= V, "top_k " + std::to_string(top_k) + " exceeds the vocabulary of " + std::to_string(V));
  B200ST_CHECK(!(top_k > 0 && top_p < 1.f), "Not implemented search logic when top_k > 0 and top_p < 1.");
  return 0;
}

int sample_init(const BeamState& bs, const int64_t* bos, int rows, int sample_num, int max_len, int64_t* out, int max_steps,
                int eos, float* logprob, int32_t* length, cudaStream_t s) {
  const int64_t work = (int64_t)rows * (max_len > max_steps ? max_len : max_steps);
  const int grid = (int)std::min<int64_t>((work + 255) / 256, 132 * 8);
  return launch_serial(sample_init_kernel, grid, 256, 0, s, bs, bos, rows, sample_num, max_len, out, max_steps, eos, logprob, length);
}

int sample_select(const SampleRows& a, int rows, cudaStream_t s) {
  return launch(sample_select_kernel<true>, rows, kSampleThreads, 0, s, a);
}

int sample_logits(const float* logits, int rows, int V, int top_k, float top_p, uint64_t seed, int64_t row_offset, int step,
                  int64_t* out, cudaStream_t s) {
  B200ST_CHECK(logits && out, "sample_logits: null argument");
  B200ST_CHECK(rows >= 1 && V >= 1, "sample_logits: rows and V must be >= 1");
  B200ST_CHECK(step >= 0 && row_offset >= 0, "sample_logits: step and row_offset must be >= 0");
  B200ST_TRY(check_sample_filter(top_k, top_p, V));
  SampleRows a{};
  a.logits = logits; a.V = V; a.eos = -1; a.unk = -1; a.min_len = 0;
  a.top_k = top_k; a.top_p = top_p; a.seed = seed; a.row_offset = row_offset; a.step = step;
  a.out = out; a.max_steps = 1;
  return launch(sample_select_kernel<false>, rows, kSampleThreads, 0, s, a);
}

}  // namespace b200st
