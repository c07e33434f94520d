// Beam-search state and selection step, shared by the single-model search (decode.cu) and the ensemble's selection over
// mixed log-probabilities (ensemble.cu).
#pragma once
#include "model.cuh"
#include "pdl.cuh"

namespace b200st {

constexpr int kBeamMaxK = 8;          // largest beam: every beam of an utterance is a row of the same step

// ---- beam search (beam_search.py:71-251,380-437): rows = utterances x beam, row u*beam + k holds beam k of utterance u ----
struct BeamState {
  int64_t* ids;          // [rows] current input ids
  float* logprob;        // [rows] accumulated log probability
  int32_t* finished;     // [rows]
  int32_t* length;       // [rows] decoding length
  int32_t* anc;          // [rows][max_len] cache row whose slot holds position j of the hypothesis now in row r
  int32_t* hist;         // [rows][max_len] word chosen at step j for row r
  int32_t* time;         // [1]
  int32_t* all_finished; // [1]
  uint32_t* ticket;      // [1] blocks done with the current step (the last one publishes time / all_finished)
};

// Per-step inputs of ensemble_logprob: each member's fp32 logits [rows, V] and its normalised log-weight.  The mixture is
// written over z[0].
struct EnsembleMix {
  float* z[kEnsembleMaxModels];
  float logw[kEnsembleMaxModels];
  int n;
};

// One step of the sampling search over `rows` rows (sampling.cu), or one draw per row of caller logits (step >= 0, no
// masks, out[row]).  Row r draws with the key (seed, row_offset + r, step); the search reads the step from *time.
struct SampleRows {
  const float* logits;   // [rows, V]
  int V;
  int eos, unk, min_len; // UNK masked unless unk < 0; EOS masked while time < min_len - 1
  int top_k;             // 0: no top-k filter
  float top_p;           // < 1: the nucleus filter (top_k must be 0)
  uint64_t seed;
  int64_t row_offset;    // global index of row 0
  int step;              // b200st_sample_logits: the step index of the key
  int64_t* ids;          // [rows] current input ids
  int32_t* finished;     // [rows]
  int32_t* length;       // [rows]
  float* logprob;        // [rows]
  int64_t* out;          // [rows, max_steps] (b200st_sample_logits: [rows])
  int max_steps;
  int32_t* time;
  int32_t* all_finished;
  uint32_t* ticket;
};
// top_k / top_p as TopSampling takes them (finite top_p, 0 <= top_k <= V, not both filters)
int check_sample_filter(int top_k, float top_p, int V);
// sequence_sampling_search's initial state on rows = utterances x sample_num, the identity ancestry table and EOS-padded
// output rows
int sample_init(const BeamState& bs, const int64_t* bos, int rows, int sample_num, int max_len, int64_t* out, int max_steps,
                int eos, float* logprob, int32_t* length, cudaStream_t s);
int sample_select(const SampleRows& a, int rows, cudaStream_t s);

// lp[r, v] = log sum_m w_m softmax(z_m[r])[v], written over member 0's logits (one block per row, members in order)
int ensemble_logprob(const EnsembleMix& mix, int rows, int V, cudaStream_t s);
// beam_select_kernel on rows that already hold log-probabilities (the ensemble's mixture)
int beam_select_logprobs(const float* logprobs, const BeamState& bs, int utterances, int beam, int V, int eos, int unk, int min_len,
                         float alpha, int max_len, cudaStream_t s);

namespace {

constexpr float kFloatMin = -1.0e9f;
constexpr int KMAX = kBeamMaxK;

// _calculate_length_penalty (beam_search.py:24-40): 1/len for alpha < 0, else ((5 + len) / 6)^-alpha
__device__ __forceinline__ float length_penalty(int len, float alpha) {
  return alpha < 0.f ? 1.f / (float)len : powf((5.f + (float)len) / 6.f, -alpha);
}
// tf.nn.top_k order: higher score first, the lower flat index on ties
__device__ __forceinline__ bool cand_better(float s, int i, float s2, int i2) { return s > s2 || (s == s2 && i < i2); }

// One search step of one utterance (block = utterance, so every row it reads or reorders is its own): log_softmax of each
// beam row with the finished / UNK / min-length masks (:71-142,380-388), accumulated log-probabilities times the length
// penalty of next_length = length + 1 - finished (:145-179), top-`beam` over the beam*V candidates (only the first beam's
// V at time 0; :181-190), then the reorder of the row state and of the ancestry table (:395-404).  The top-k is a
// per-thread register top-KMAX over the thread's candidates followed by `beam` rounds of a block-wide arg-max.
// LOGP: the rows already hold log-probabilities (an ensemble's mixture, :101-115), so the log_softmax pass is skipped.
template <bool LOGP>
__global__ void __launch_bounds__(1024) beam_select_kernel(const float* __restrict__ logits, BeamState s, int beam, int V, int eos,
                                                           int unk, int min_len, float alpha, int max_len) {
  pdl_wait();
  pdl_trigger();
  __shared__ float red[32];
  __shared__ float sval[32];
  __shared__ int sidx[32];
  __shared__ float lse[KMAX], pen[KMAX], lprev[KMAX];
  __shared__ int fin[KMAX], nlen[KMAX], win[KMAX];
  const int r0 = blockIdx.x * beam;
  const int t = *s.time;
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5, nw = blockDim.x >> 5;
  for (int b = 0; b < beam; ++b) {
    float mx = 0.f, se = 1.f;
    if (!LOGP) {
      const float* z = logits + (int64_t)(r0 + b) * V;
      mx = -INFINITY;
      for (int v = threadIdx.x; v < V; v += blockDim.x) mx = fmaxf(mx, z[v]);
      mx = block_max(mx, red);
      se = 0.f;
      for (int v = threadIdx.x; v < V; v += blockDim.x) se += expf(z[v] - mx);
      se = block_sum(se, red);
    }
    if (threadIdx.x == 0) {
      lse[b] = LOGP ? 0.f : mx + logf(se);
      fin[b] = s.finished[r0 + b] != 0;
      lprev[b] = s.logprob[r0 + b];
      nlen[b] = s.length[r0 + b] + 1 - fin[b];
      pen[b] = length_penalty(nlen[b], alpha);
    }
  }
  __syncthreads();
  // accumulated log-probability of candidate (beam b, word v), un-penalised
  auto acc_of = [&](int b, int v) -> float {
    float lp = logits[(int64_t)(r0 + b) * V + v] - lse[b];
    if (fin[b]) lp = (v == eos) ? 0.f : kFloatMin;
    if (v == unk) lp += kFloatMin;
    if (v == eos && t < min_len - 1) lp += kFloatMin;
    return lp + lprev[b];
  };
  float vs[KMAX];
  int is[KMAX];
#pragma unroll
  for (int q = 0; q < KMAX; ++q) { vs[q] = -INFINITY; is[q] = 0x7fffffff; }
  const int nb = t == 0 ? 1 : beam;
  for (int b = 0; b < nb; ++b) {
    for (int v = threadIdx.x; v < V; v += blockDim.x) {
      const float sc = acc_of(b, v) * pen[b];
      const int i = b * V + v;
      if (cand_better(sc, i, vs[KMAX - 1], is[KMAX - 1])) {
        vs[KMAX - 1] = sc; is[KMAX - 1] = i;
#pragma unroll
        for (int q = KMAX - 1; q > 0; --q) {
          if (cand_better(vs[q], is[q], vs[q - 1], is[q - 1])) {
            const float tv = vs[q]; vs[q] = vs[q - 1]; vs[q - 1] = tv;
            const int ti = is[q]; is[q] = is[q - 1]; is[q - 1] = ti;
          }
        }
      }
    }
  }
  for (int k = 0; k < beam; ++k) {
    float bv = vs[0];
    int bi = is[0];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float ov = __shfl_xor_sync(0xffffffffu, bv, o);
      const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
      if (cand_better(ov, oi, bv, bi)) { bv = ov; bi = oi; }
    }
    __syncthreads();
    if (lane == 0) { sval[w] = bv; sidx[w] = bi; }
    __syncthreads();
    if (threadIdx.x == 0) {
      for (int i = 1; i < nw; ++i)
        if (cand_better(sval[i], sidx[i], bv, bi)) { bv = sval[i]; bi = sidx[i]; }
      win[k] = bi < nb * V ? bi : 0;
    }
    __syncthreads();
    if (is[0] == win[k]) {                        // flat indices are unique: exactly one thread pops its head
#pragma unroll
      for (int q = 0; q < KMAX - 1; ++q) { vs[q] = vs[q + 1]; is[q] = is[q + 1]; }
      vs[KMAX - 1] = -INFINITY; is[KMAX - 1] = 0x7fffffff;
    }
  }
  // new row r0 + j continues beam p = win[j] / V with word win[j] % V (every old value was read into shared memory above)
  if ((int)threadIdx.x < beam) {
    const int j = threadIdx.x, p = win[j] / V, word = win[j] % V;
    const int r = r0 + j;
    s.ids[r] = word;
    s.logprob[r] = acc_of(p, word);
    s.length[r] = nlen[p];
    s.finished[r] = word == eos ? 1 : 0;
    s.hist[(int64_t)r * max_len + t] = word;
  }
  // ancestry: anc'[r0 + j][col] = anc[r0 + p][col] for col < t, and r0 + p at col = t (the parent's own slot).  A thread
  // owns whole columns, so reading every parent's entry before writing needs no barrier.
  for (int col = threadIdx.x; col <= t; col += blockDim.x) {
    int nv[KMAX];
#pragma unroll
    for (int j = 0; j < KMAX; ++j) {
      if (j < beam) {
        const int p = r0 + win[j] / V;
        nv[j] = col == t ? p : s.anc[(int64_t)p * max_len + col];
      }
    }
#pragma unroll
    for (int j = 0; j < KMAX; ++j)
      if (j < beam) s.anc[(int64_t)(r0 + j) * max_len + col] = nv[j];
  }
  // the last block of the step publishes all_finished (every row of every utterance) and advances time: every block has
  // read `time` before it takes its ticket
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence();
    if (atomicAdd(s.ticket, 1u) == gridDim.x - 1) {
      __threadfence();
      int all = 1;
      for (int r = 0; r < (int)gridDim.x * beam; ++r) all &= __ldcg(s.finished + r) != 0 ? 1 : 0;
      *s.all_finished = all;
      *s.ticket = 0;
      *s.time = t + 1;
    }
  }
}

}  // namespace
}  // namespace b200st
