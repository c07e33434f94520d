// Cascade ST handoff: the ASR search's top-1 hypotheses (device ids) -> the MT model's source batch, without a host
// round trip.  One block per utterance:
//   n = position of the first ASR EOS in the hypothesis (its whole length when none),
//   source = remap[hyp[0..n)] (ASR target vocabulary -> MT source vocabulary; an ASR id outside the table maps to the MT
//            UNK) followed by the MT EOS, i.e. TextDataPipeline.encode(is_processed=True) of the hypothesis' tokens,
//   max_src_len > 0: Seq2Seq's truncation rule (seq2seq.py:171-176), the first max_src_len - 1 ids and the EOS,
//   src_ids / src_padding [B][out_stride] padded with the MT pad id / 1.0 beyond the length, src_len [B].
// Integer work only: no floating-point atomic, and every output element is written exactly once.
#include "../../include/b200st.h"
#include "common.cuh"
#include "kernels.cuh"
#include "pdl.cuh"

#include <string>

namespace b200st {
namespace {

constexpr int kCascadeThreads = 128;

__global__ void __launch_bounds__(kCascadeThreads) cascade_source_kernel(const b200st_cascade_source_args a) {
  __shared__ int warp_min[kCascadeThreads / 32];
  const int b = blockIdx.x;
  const int64_t* hyp = a.hyp_ids + (int64_t)b * a.hyp_stride;
  int first = a.hyp_len;                                   // first EOS position (hyp_len when the row never emits one)
  for (int i = threadIdx.x; i < a.hyp_len; i += blockDim.x)
    if (hyp[i] == (int64_t)a.asr_eos_id) first = min(first, i);
  first = __reduce_min_sync(0xffffffffu, first);
  if ((threadIdx.x & 31) == 0) warp_min[threadIdx.x >> 5] = first;
  __syncthreads();
  int n = warp_min[0];
#pragma unroll
  for (int w = 1; w < kCascadeThreads / 32; ++w) n = min(n, warp_min[w]);
  int len = n + 1;                                         // tokens + EOS
  if (a.max_src_len > 0 && len > a.max_src_len) len = a.max_src_len;
  int64_t* out = a.src_ids + (int64_t)b * a.out_stride;
  float* pad = a.src_padding + (int64_t)b * a.out_stride;
  for (int j = threadIdx.x; j < a.out_stride; j += blockDim.x) {
    int64_t v;
    if (j < len - 1) {
      const int64_t id = hyp[j];
      v = (id >= 0 && id < (int64_t)a.asr_vocab) ? (int64_t)a.remap[id] : (int64_t)a.mt_unk_id;
    } else {
      v = j == len - 1 ? (int64_t)a.mt_eos_id : (int64_t)a.mt_pad_id;
    }
    out[j] = v;
    pad[j] = j < len ? 0.f : 1.f;
  }
  if (threadIdx.x == 0) a.src_len[b] = len;
}

}  // namespace

static int cascade_source(const b200st_cascade_source_args& a, cudaStream_t s) {
  B200ST_CHECK(a.hyp_ids && a.remap && a.src_ids && a.src_padding && a.src_len, "cascade_source: null argument");
  B200ST_CHECK(a.B >= 1 && a.B <= 65535, "cascade_source: B must be in 1..65535, got " + std::to_string(a.B));
  B200ST_CHECK(a.hyp_len >= 1 && a.hyp_stride >= a.hyp_len, "cascade_source: need 1 <= hyp_len <= hyp_stride");
  B200ST_CHECK(a.asr_vocab >= 1 && a.mt_vocab >= 1, "cascade_source: the remap table needs asr_vocab >= 1 entries into an "
               "MT vocabulary of mt_vocab >= 1 ids");
  B200ST_CHECK(a.asr_eos_id >= 0 && a.asr_eos_id < a.asr_vocab, "cascade_source: asr_eos_id outside the ASR vocabulary");
  for (int32_t id : {a.mt_eos_id, a.mt_pad_id, a.mt_unk_id})
    B200ST_CHECK(id >= 0 && id < a.mt_vocab, "cascade_source: MT eos / pad / unk id " + std::to_string(id) + " outside the MT "
                 "vocabulary of " + std::to_string(a.mt_vocab));
  B200ST_CHECK(a.max_src_len == 0 || a.max_src_len >= 2, "cascade_source: max_src_len must be 0 (none) or >= 2");
  const int need = a.max_src_len > 0 && a.max_src_len < a.hyp_len + 1 ? a.max_src_len : a.hyp_len + 1;
  B200ST_CHECK(a.out_stride >= need, "cascade_source: out_stride " + std::to_string(a.out_stride) + " < the longest source " +
               std::to_string(need));
  return launch_serial(cascade_source_kernel, a.B, kCascadeThreads, 0, s, a);
}

}  // namespace b200st

extern "C" int b200st_cascade_source(const b200st_cascade_source_args* a, void* stream) {
  if (!a) {
    b200st::set_last_error("cascade_source: null argument");
    return 1;
  }
  return b200st::cascade_source(*a, reinterpret_cast<cudaStream_t>(stream));
}
