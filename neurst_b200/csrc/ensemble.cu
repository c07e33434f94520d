// Per-step kernels of ensemble decoding (EncoderDecoderEnsembleModel under sequence_beam_search,
//   neurst/models/encoder_decoder_ensemble_model.py, neurst/layers/search/beam_search.py:97-115):
// the mixture of the members' next-token distributions, and the beam selection on that mixture.  The search driver, which
// steps every member against one beam state, is ensemble_beam_search in decode.cu.
#include "beam.cuh"

namespace b200st {

namespace {

constexpr int kMixThreads = 512;

// One block per row.  For every member m, lse_m = log sum_v exp(z_m[v]); then
//   lp[v] = log sum_m exp(log w_m + z_m[v] - lse_m)
// as a log-sum-exp over the members: in exact arithmetic the reference's log(sum_m w_m softmax(z_m)[v]), but it does not
// underflow to -inf where every member's probability does.  A zero weight (log w = -inf) contributes exp(-inf) = 0.
// The result is written over member 0's logits.  Members are combined in index order and every block reduction has a
// fixed order (no atomics): the step stays bit-reproducible and a row's result does not depend on the other rows.
__global__ void __launch_bounds__(kMixThreads) ensemble_logprob_kernel(const __grid_constant__ EnsembleMix mix, int V) {
  pdl_wait();
  pdl_trigger();
  __shared__ float red[32];
  __shared__ float shift[kEnsembleMaxModels];      // log w_m - lse_m
  const int64_t base = (int64_t)blockIdx.x * V;
  for (int m = 0; m < mix.n; ++m) {
    const float* z = mix.z[m] + base;
    float mx = -INFINITY;
    for (int v = threadIdx.x; v < V; v += blockDim.x) mx = fmaxf(mx, z[v]);
    mx = block_max(mx, red);
    float se = 0.f;
    for (int v = threadIdx.x; v < V; v += blockDim.x) se += expf(z[v] - mx);
    se = block_sum(se, red);
    if (threadIdx.x == 0) shift[m] = mix.logw[m] - (mx + logf(se));
  }
  __syncthreads();
  float* out = mix.z[0] + base;
  for (int v = threadIdx.x; v < V; v += blockDim.x) {
    float a[kEnsembleMaxModels];
    float hi = -INFINITY;
#pragma unroll
    for (int m = 0; m < kEnsembleMaxModels; ++m) {
      if (m < mix.n) {
        a[m] = mix.z[m][base + v] + shift[m];
        hi = fmaxf(hi, a[m]);
      }
    }
    float s = 0.f;
#pragma unroll
    for (int m = 0; m < kEnsembleMaxModels; ++m)
      if (m < mix.n) s += expf(a[m] - hi);
    out[v] = hi + logf(s);
  }
}

}  // namespace

int ensemble_logprob(const EnsembleMix& mix, int rows, int V, cudaStream_t s) {
  return launch(ensemble_logprob_kernel, rows, kMixThreads, 0, s, mix, V);
}

int beam_select_logprobs(const float* logprobs, const BeamState& bs, int utterances, int beam, int V, int eos, int unk, int min_len,
                         float alpha, int max_len, cudaStream_t s) {
  return launch(beam_select_kernel<true>, utterances, 1024, 0, s, logprobs, bs, beam, V, eos, unk, min_len, alpha, max_len);
}

}  // namespace b200st
