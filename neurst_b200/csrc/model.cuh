// Model runtime of libb200st: configuration, parameter table (flat fp32 arena in the reference's TF layouts),
// workspace planning and the forward / backward orchestration of the SpeechTransformer hot path.
#pragma once
#include "common.cuh"
#include "gemm.cuh"
#include "kernels.cuh"

#include <string>
#include <unordered_map>
#include <vector>

namespace b200st {

enum ModelType : int { MODEL_SPEECH = 0, MODEL_TEXT = 1, MODEL_ENCODER = 2, MODEL_DECODER = 3, MODEL_MHA = 4 };

struct Config {
  int model_type;
  int d, heads, ffn, enc_layers, dec_layers, vocab, src_vocab;
  int feat, in_channels, channels, conv_layer_norm;
  int precision;              // F32: fp32 FMA kernels (parity mode); BF16 / F16: wgmma kernels with that 16-bit type
  float ln_eps, attention_dropout, ffn_dropout, postprocess_dropout, label_smoothing;
  int share_src_trg_embedding;
  // MODEL_MHA only
  int mha_self, mha_din, mha_dmem, mha_dout;
  int with_cross_attention;   // decoder stack: 1 (default)
  int disable_fused_attention; // tests: use the materialised (GEMM + softmax) attention path in bf16 mode
  int deterministic;           // fused FFN: slices reduce in slice order (bit-reproducible)
  int encoder_monotonic;       // MODEL_TEXT: causal encoder self-attention (transformer_encoder.py:119-123)
};

struct ParamInfo {
  std::string name;
  int64_t offset;   // elements in the arena (multiple of 8)
  int ndim;
  int64_t shape[4];
  int64_t numel;
};

struct GradSync;     // comm.cu: NCCL communicator + communication stream of a data-parallel replica
int comm_unique_id(char* out128);
int comm_init(GradSync** out, const char* id128, int nranks, int rank);
void comm_destroy(GradSync* g);
int comm_world(const GradSync* g);
int comm_reserved_sms(const GradSync* g);    // SMs the communicator's kernels may hold while the backward pass runs
int64_t comm_reduced_elems(const GradSync* g);
int comm_calls(const GradSync* g);
void comm_begin_step(GradSync* g);
int comm_reduce_range(GradSync* g, float* grads, int64_t lo, int64_t hi, cudaStream_t compute, cudaEvent_t extra0, cudaEvent_t extra1);
int comm_join(GradSync* g, cudaStream_t compute);
int comm_broadcast(GradSync* g, float* buf, int64_t n, int root, cudaStream_t compute);

struct Model {
  Config cfg;
  std::vector<ParamInfo> params;
  std::unordered_map<std::string, int> index;
  int64_t arena_numel = 0;
  int adt = F32;              // activation dtype
  GradSync* sync = nullptr;   // set by b200st_comm_init: gradients are all-reduced inside forward_backward when asked
  int find(const std::string& n) const {
    auto it = index.find(n);
    return it == index.end() ? -1 : it->second;
  }
};

int build_param_table(Model& m);

// Caller-provided device memory for one call.
struct Buffers {
  const float* params;                 // fp32 master arena
  const void* shadow;                  // 16-bit copy of the arena in the handle's precision (bf16 / fp16 modes)
  float* grads;                        // fp32 gradient arena (accumulated into; null for inference)
  void* workspace;
  size_t workspace_bytes;
};

struct Batch {
  // speech: src fp32 [B,T,feat,in_channels] + src_length[B]; text: src_ids [B,T] + src_padding [B,T]
  const float* src;
  const int64_t* src_ids;
  const int64_t* src_length;
  const float* src_padding;
  const int64_t* trg_input;            // [B,L]
  const int64_t* trg;                  // [B,L] (loss) or null
  const int64_t* trg_length;           // [B]
  int B, T, L;
  int training;                        // dropout on
  uint64_t seed;
  const uint64_t* seed_dev;            // optional: device-resident seed (overrides `seed`)
  float loss_scale;                    // multiplies dlogits (1/world for DP mean, gradient-accumulation factor, ...)
  const float* loss_scale_dev;         // optional device word multiplied in as well (dynamic loss scale of the fp16 mode)
  int wait_k;                          // decoder cross-attention lag k (0: none): target i sees memory keys j < i + k
  const int32_t* wait_k_dev;           // optional device-resident lag, read at kernel run time (overrides wait_k)
  // outputs (device, optional)
  float* logits;                       // fp32 [B,L,V]
  float* loss;                         // [1]
  float* nll_sum;                      // [B]
  float* n_tokens;                     // [B]
  float* enc_out;                      // fp32 [B,T',d]
  // b200st_encode: stop after the encoder stack; enc_bias_out receives the additive key bias [B,T'] (0 / -1e9)
  int allreduce_grads = 0;             // backward: bucketed NCCL all-reduce of the gradient arena, overlapped (needs Model::sync)
  int stop_after_encoder = 0;
  float* enc_bias_out = nullptr;
};

size_t model_workspace_bytes(const Model& m, int B, int T, int L, int training);
int model_forward(const Model& m, const Buffers& buf, const Batch& b, bool backward, cudaStream_t st);

// stack-level entry points (layer API; inference/eval forward only)
// When `need` is non-null the call only reports the workspace bytes it would use (nothing is launched).
int encoder_forward_api(const Model& m, const Buffers& buf, const float* x, const float* padding, int B, int T, float* out,
                        int training, uint64_t seed, cudaStream_t st, size_t* need);
int decoder_forward_api(const Model& m, const Buffers& buf, const float* x, const float* memory, const float* memory_padding,
                        int B, int L, int Tm, float* out, int training, uint64_t seed, cudaStream_t st, size_t* need);
int mha_forward_api(const Model& m, const Buffers& buf, const float* query, const float* memory, const float* bias, int B, int Tq,
                    int Tk, float* out, cudaStream_t st, size_t* need);

uint64_t dropout_stream_id(const std::string& site);

// ---- incremental decoding (decode.cu) ----------------------------------------------------------------------------
struct DecodeState {
  int B, Tm, max_len;            // rows, encoder length T', cache length (maximum number of decoded positions)
  float* cross_kv;               // [dec_layers][B][Tm][2d] fp32: pre-projected memory keys | values
  float* self_kv;                // [dec_layers][2][B][max_len][d] fp32
  const float* memory_bias;      // [B, Tm] additive (0 / -1e9) or null
  float* scratch;                // decode_scratch_floats(B) floats
  int use_shadow;                // 0: fp32 master weights, 1: the handle's 16-bit shadow
  int wait_k;                    // wait-k lag (0: none): step t attends to the memory keys j < min(Tm, wait_k + t)
};
struct GreedyArgs {
  const int64_t* bos_ids;        // [B] device: first decoder input (generation_initializer["decoder_input"])
  int eos_id, unk_id;            // unk_id < 0: UNK allowed
  int min_len, max_steps;
  int64_t* out_ids;              // [B, max_steps] device, padded with EOS
  int32_t* out_len;              // [B] device
  float* out_logprob;            // [B] device: accumulated log-probability of the hypothesis
  void* state_words;             // >= 256 bytes of device memory (ids, finished flags, time, grid barrier)
  int use_graph;
};
int64_t decode_scratch_floats(const Model& m, int B);
int decode_init(const Model& m, const Buffers& buf, const float* enc_out, const DecodeState& st, cudaStream_t s);
int decode_step(const Model& m, const Buffers& buf, const DecodeState& st, const int64_t* symbols, const int32_t* time_dev,
                float* logits, cudaStream_t s);
int last_greedy_used_graph();      // 1 / 0 for the last greedy_search of this process (-1: none yet)
int greedy_search(const Model& m, const Buffers& buf, const DecodeState& st, const GreedyArgs& ga, cudaStream_t s);
struct BeamArgs {
  const int64_t* bos_ids;        // [B] device, one per utterance
  int eos_id, unk_id;            // unk_id < 0: UNK allowed
  int min_len, max_steps;
  int beam_size, top_k;
  float length_penalty;          // alpha; < 0: 1 / length
  int64_t* out_ids;              // [B * top_k, max_steps] device, padded with EOS
  float* out_scores;             // [B * top_k] logprob * length penalty, best first per utterance
  float* out_logprob;            // [B * top_k]
  int32_t* out_len;              // [B * top_k]
  void* state_words;             // >= beam_state_bytes(B, beam_size, max_len)
  int use_graph;
};
int64_t beam_state_bytes(int B, int beam, int max_len);
// st.B counts utterances; self_kv and scratch are sized for B * beam_size rows, cross_kv / memory_bias for B
int beam_search(const Model& m, const Buffers& buf, const DecodeState& st, const BeamArgs& a, cudaStream_t s);
struct SamplingArgs {
  const int64_t* bos_ids;        // [B] device, one per utterance
  int eos_id, unk_id;            // unk_id < 0: UNK allowed
  int min_len, max_steps;
  int sample_num, top_k;         // top_k 0: no top-k filter
  float top_p;                   // < 1: nucleus filter
  uint64_t seed;
  int64_t row_offset;            // global index of row 0 (the draws' key)
  int64_t* out_ids;              // [B * sample_num, max_steps] device, padded with EOS
  float* out_logprob;            // [B * sample_num]
  int32_t* out_len;              // [B * sample_num]
  void* state_words;             // >= beam_state_bytes(B, sample_num, max_len)
  int use_graph;
};
// sequence_sampling_search (TopSampling) with the per-token step of beam_search on B x sample_num rows; st as beam_search's
int sampling_search(const Model& m, const Buffers& buf, const DecodeState& st, const SamplingArgs& a, cudaStream_t s);
// one draw per row of caller logits [rows, V], no masks: out[r] with the key (seed, row_offset + r, step) (sampling.cu)
int sample_logits(const float* logits, int rows, int V, int top_k, float top_p, uint64_t seed, int64_t row_offset, int step,
                  int64_t* out, cudaStream_t s);
constexpr int kEnsembleMaxModels = 8;      // B200ST_ENSEMBLE_MAX_MODELS
struct EnsembleMember {
  const Model* m;
  Buffers buf;
  DecodeState st;                // as beam_search's: B utterances, self_kv / scratch for B * beam_size rows
  float weight;                  // >= 0, normalised over the members
};
// beam_search over the weighted mixture of n members' next-token distributions, one beam state for all members
int ensemble_beam_search(const EnsembleMember* members, int n, const BeamArgs& a, cudaStream_t s);

// ---- streaming simultaneous translation (stream.cu) ------------------------------------------------------------------
struct StreamState {
  int max_src, max_trg;
  float* enc_kv;                 // [enc_layers][2][max_src][d] fp32: each encoder layer's self-attention keys / values
  float* cross_kv;               // [dec_layers][max_src][2d] fp32: memory keys | values
  float* self_kv;                // [dec_layers][2][max_trg][d] fp32
  float* enc_out;                // optional [max_src][d] fp32: the encoder output rows (final LayerNorm)
  float* scratch;                // stream_scratch_floats() floats
  int use_shadow;
};
struct StreamMember {
  const Model* m;
  Buffers buf;
  StreamState st;
};
struct StreamSession;
int64_t stream_scratch_floats(const Model& m);
int stream_create(const StreamMember* members, int n, int32_t* lens_dev, StreamSession** out);
void stream_destroy(StreamSession* s);
int stream_reset(StreamSession* s, cudaStream_t st);
int stream_read(StreamSession* s, int n, const int64_t* ids, cudaStream_t st);
int stream_write(StreamSession* s, const float* weights, int64_t* out_id, cudaStream_t st);
void stream_lengths(const StreamSession* s, int* src_len, int* trg_len);

}  // namespace b200st
