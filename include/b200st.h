/* libb200st — C ABI of the H100-native SpeechTransformer hot path.
 *
 * Drop-in boundary for bytedance/neurst (reference @ /root/reference).  The reference is pure Python; its
 * "FFI" for this path is the class registry (neurst/utils/registry.py:24-137) through which Trainer and the
 * models reach the neurst/layers and neurst/criterions packages.  Each entry point below replaces the TF/PyTorch
 * library ops behind one reference function (file:line cited per function); INTEGRATION.md shows the
 * ctypes binding a maintainer adds.
 *
 * Conventions: every pointer is a DEVICE pointer owned by the caller (weights, activations, workspace);
 * every call is asynchronous on the given cudaStream_t (passed as void*); return 0 = ok, non-zero = error
 * with a thread-local message from b200st_last_error(); no exceptions cross the ABI; the library never
 * allocates device memory.  dtype codes: 0 = fp32, 1 = bf16.
 */
#ifndef B200ST_H_
#define B200ST_H_
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif

#define B200ST_F32 0
#define B200ST_BF16 1
#define B200ST_F16 2   /* IEEE half: forward values of the mixed16 precision */

const char* b200st_last_error(void);
int b200st_version(void);
/* number of hand-written kernels launched by this process so far (bench.py "gpu_launches") */
int64_t b200st_launch_count(void);

/* ---- generic contraction (tf.einsum / Dense / tf.matmul sites; neurst/layers/common_layers.py:270,276-288,
 *      multi_head_attention.py:145,215; text_modalities.py:104-108) ---------------------------------------
 * C[b2][b1][m][n] = epi(alpha * sum_k A(m,k) B(n,k)); operands K-major (mn_major=0) or MN-major (1).
 * bf16 operands -> wgmma/TMA kernel; fp32 operands -> fp32 FMA kernel (parity mode). */
typedef struct {
  const void* ptr; int32_t dtype; int32_t mn_major; int64_t ld, sb1, sb2;
} b200st_operand;
typedef struct {
  int32_t M, N, K, nb1, nb2;
  b200st_operand A, B;
  void* C; int32_t c_dtype; int64_t ldc, c_sb1, c_sb2;
  float alpha;
  const float* bias;
  int32_t relu;
  const void* mask_src; int32_t mask_dtype; int64_t mask_ld, mask_sb1, mask_sb2;
  float dropout_p; uint64_t dropout_seed, dropout_stream;
  const float* residual; int64_t res_ld, res_sb1, res_sb2;
  int32_t accumulate;
  int32_t splitk;        /* 1 = none, 0 = auto (linear fp32 accumulate epilogues only) */
  int32_t force_simt;    /* tests: run the fp32-FMA kernel even on bf16 operands */
} b200st_gemm_args;
int b200st_gemm(const b200st_gemm_args* args, void* stream);


/* ---- model handle ------------------------------------------------------------------------------------
 * model_type: 0 = SpeechTransformer (neurst/models/speech_transformer.py:27-280), 1 = text Transformer
 * (neurst/models/transformer.py), 2 = TransformerEncoder stack only (layers/encoders/transformer_encoder.py:23-136),
 * 3 = TransformerDecoder stack only (layers/decoders/transformer_decoder.py:23-228), 4 = MultiHeadAttention /
 * MultiHeadSelfAttention (layers/attentions/multi_head_attention.py:21-290).
 * precision: B200ST_F32 = fp32 FMA kernels (parity mode, any shape); B200ST_F16 / B200ST_BF16 = wgmma kernels with every
 * 16-bit tensor (weights shadow, activations, activation gradients) in that type, fp32 accumulation, fp32 master weights,
 * fp32 parameter gradients.  B200ST_F16 is the reference's own mixed precision (mixed_float16 + dynamic loss scaling,
 * neurst/training/training_utils.py:73-81,413-416): 11-bit significands, needs loss scaling (b200st_batch.loss_scale_dev +
 * b200st_optimizer_step); B200ST_BF16 needs none but carries 8-bit significands. */
typedef struct b200st_model* b200st_handle;
typedef struct {
  int32_t model_type;
  int32_t d, heads, ffn, enc_layers, dec_layers, vocab, src_vocab;
  int32_t feat, in_channels, channels, conv_layer_norm;
  int32_t precision;
  float ln_eps, attention_dropout, ffn_dropout, postprocess_dropout, label_smoothing;
  int32_t share_src_trg_embedding;
  int32_t mha_self, mha_din, mha_dmem, mha_dout;
  int32_t with_cross_attention;
  int32_t disable_fused_attention;   /* tests: materialised attention (GEMM + softmax kernels) and unfused FFN in the 16-bit modes */
  int32_t deterministic;             /* 1: the hidden-dimension slices of the fused FFN kernel reduce into the output in slice
                                      * order (ticket per row tile) instead of arrival order: bit-reproducible steps for a few
                                      * microseconds per FFN launch (default 0: fp32 sums in arrival order) */
  int32_t encoder_monotonic;         /* 1: causal encoder self-attention, query i sees keys j <= i (transformer_encoder.py:119-123,
                                      * the wait-k model's encoder).  Text model (model_type 1) only; other models refuse it. */
} b200st_config;

int b200st_create(const b200st_config* cfg, b200st_handle* out);   /* host object only; no device memory */
int b200st_destroy(b200st_handle h);

/* Parameter arena: one flat fp32 buffer; tensors in the reference's TF layouts (dense [in,out], conv HWIO,
 * embedding [V,d]; SURVEY.md Appendix B), each starting at a multiple of 8 elements. */
int64_t b200st_param_arena_numel(b200st_handle h);
int32_t b200st_param_count(b200st_handle h);
int b200st_param_info(b200st_handle h, int32_t i, char* name, int32_t name_cap, int64_t* offset, int32_t* ndim,
                      int64_t* shape4);

typedef struct {
  const float* params;      /* fp32 master arena */
  const void* shadow;       /* 16-bit copy of the arena in the handle's precision (b200st_refresh_shadow / b200st_optimizer_step) */
  float* grads;             /* fp32, same layout; gradients are ACCUMULATED into it */
  void* workspace; uint64_t workspace_bytes;   /* >= b200st_workspace_bytes(...) , 256-byte aligned */
} b200st_buffers;

/* One batch in the reference's input-dict form (neurst/tasks/speech2text.py:135-161). */
typedef struct {
  const float* src;             /* speech: fp32 [B,T,feat,in_channels] */
  const int64_t* src_ids;       /* text:   [B,T] */
  const int64_t* src_length;    /* speech: [B] frames */
  const float* src_padding;     /* text:   [B,T] 1.0 = pad */
  const int64_t* trg_input;     /* [B,L] */
  const int64_t* trg;           /* [B,L] or NULL */
  const int64_t* trg_length;    /* [B]   or NULL */
  int32_t B, T, L;
  int32_t training;             /* dropout on */
  uint64_t seed;                /* dropout seed of this step */
  const uint64_t* seed_dev;     /* optional device-resident seed (read at kernel run time: CUDA-graph replay) */
  float loss_scale;             /* multiplies the loss gradient (0 => 1) */
  const float* loss_scale_dev;  /* optional device word, multiplied in too: the dynamic loss scale (element 0 of the
                                 * b200st_optimizer_step state), read at kernel run time so CUDA-graph replays follow it */
  float* logits;                /* out, optional: fp32 [B,L,V] */
  float* loss;                  /* out, optional: [1] = sum(nll)/sum(tokens) (label_smoothed_cross_entropy.py:46-53) */
  float* nll_sum;               /* out, optional: [B] */
  float* n_tokens;              /* out, optional: [B] */
  float* enc_out;               /* out, optional: fp32 [B,T',d] */
  int32_t wait_k;               /* wait-k lag of the decoder's cross-attention (0: none): target position i (0-based) sees the
                                 * memory keys j < i + wait_k (transformer_decoder.py:194-208).  < 0, or > 0 on a model without
                                 * cross-attention, fails before anything is launched. */
  const int32_t* wait_k_dev;    /* optional device int32 lag, read at kernel run time instead of wait_k (CUDA-graph replay with a
                                 * fresh lag per step); a value < 1 there means no lag */
} b200st_batch;

int64_t b200st_workspace_bytes(b200st_handle h, int32_t B, int32_t T, int32_t L, int32_t training);
/* EncoderDecoderModel.call (+ criterion when trg given): neurst/models/encoder_decoder_model.py:263-279 */
int b200st_forward(b200st_handle h, const b200st_buffers* buf, const b200st_batch* batch, void* stream);
/* forward + label-smoothed CE + full backward (GradAccumKerasModel.train_step, gradaccum_keras_model.py:190-245) */
int b200st_forward_backward(b200st_handle h, const b200st_buffers* buf, const b200st_batch* batch, void* stream);

/* ---- data-parallel training step (SURVEY.md 8b/8e): NCCL over NVLink only, inside the library -----------------------------
 * One process per GPU.  Rank 0 calls b200st_comm_unique_id, the 128 bytes travel to the other ranks by any host channel,
 * every rank calls b200st_comm_init (ncclCommInitRank; libnccl.so.2 is dlopen'ed from the process or the system).
 * b200st_train_step = forward + loss + backward (+ allreduce_grads: ncclAllReduce(sum) of the fp32 gradient arena in
 * reverse-order buckets — decoder+output layer / upper encoder half / lower encoder half / front-end — each issued on the
 * library's communication stream the moment its last gradient kernel has been enqueued, so the transfers run under the
 * rest of the backward pass; `stream` waits for them at the end) (+ optim != NULL: b200st_optimizer_step with
 * grad_scale = 1/(replicas * update_cycle) = hvd.Average, neurst/training/hvd_utils.py:48-62).
 * b200st_comm_broadcast: rank-0 parameters to all (neurst/exps/trainer.py:285). */
int b200st_comm_unique_id(char* out128);
int b200st_comm_init(b200st_handle h, const char* id128, int32_t nranks, int32_t rank);
int b200st_comm_broadcast(b200st_handle h, float* buf, int64_t numel, int32_t root, void* stream);
/* call on every rank before the process group goes away; destroy every CUDA graph that captured b200st_train_step with
 * allreduce_grads first: ncclCommDestroy waits for the graphs that reference the communicator */
int b200st_comm_destroy(b200st_handle h);
int b200st_comm_stats(b200st_handle h, int64_t* reduced_elems, int32_t* calls, int32_t* world);   /* of the last step */
struct b200st_optim_args_;
typedef struct {
  int32_t allreduce_grads;
  const struct b200st_optim_args_* optim;     /* NULL: no optimizer step (gradient accumulation micro-step) */
} b200st_step_opts;
int b200st_train_step(b200st_handle h, const b200st_buffers* buf, const b200st_batch* batch, const b200st_step_opts* opts,
                      void* stream);

/* ---- inference: encoder pass, cached decoder step, greedy search (SURVEY.md 8 f1, BASELINE cfg-5) ---------------------
 * b200st_encode: modality + TransformerEncoder only (EncoderDecoderModel.get_symbols_to_logits_fn up to
 * create_decoding_internal_cache, neurst/models/encoder_decoder_model.py:230-241): enc_out fp32 [B,T',d], enc_bias fp32
 * [B,T'] = the additive memory bias (0 / -1e9).  Uses batch->src, src_length (speech) or src_ids, src_padding (text). */
int b200st_encode(b200st_handle h, const b200st_buffers* buf, const b200st_batch* batch, float* enc_out, float* enc_bias,
                  void* stream);
int64_t b200st_encode_workspace_bytes(b200st_handle h, int32_t B, int32_t T);
/* Decoding state, caller-owned device buffers (nothing grows during decoding):
 *   cross_kv  fp32 [dec_layers][B][Tm][2d]: memory keys | values, projected once (transformer_layers.py:156-170)
 *   self_kv   fp32 [dec_layers][2][B][max_len][d]: self-attention key / value cache (multi_head_attention.py:271-289)
 *   scratch   b200st_decode_scratch_floats(h, B) floats
 * use_shadow 0: weights read from the fp32 master arena (token ids identical to an fp32 reference); 1: the handle's
 *   16-bit shadow (half the bytes) for trg.emb (embedding and tied logits) and, per decoder layer, self.qkv.kernel,
 *   self.out.kernel, cross.q.kernel, cross.out.kernel, ffn.w1 and ffn.w2.  Biases, LayerNorm parameters and the
 *   cross-attention K/V projection (b200st_decode_init) always use the fp32 master arena; all arithmetic is fp32.
 * Rows per step (B, or B*beam_size in beam search): 1..8 with use_shadow 0; 1..B200ST_DECODE_MAX_ROWS with use_shadow 1.
 *   Above 8 rows the step runs its projections on the tensor cores: each fp32 activation is split into a sum of 16-bit
 *   terms (2 for fp16, 3 for bf16) multiplied by the same 16-bit weights with fp32 accumulation, so the step keeps the
 *   contract above (and needs d, ffn multiples of 64 and vocab a multiple of 8).  With fp16 weights every activation
 *   entering a projection must lie within the fp16 range, as in the reference's mixed_float16.  That step uses no
 *   floating-point atomics: it is bit-reproducible, and a row's result does not depend on the other rows of the step. */
#define B200ST_DECODE_MAX_ROWS 256
typedef struct {
  int32_t B, Tm, max_len;
  float* cross_kv; float* self_kv;
  const float* memory_bias;
  float* scratch;
  int32_t use_shadow;
  int32_t wait_k;               /* wait-k lag (0: none): decoding step t attends to the memory keys j < min(Tm, wait_k + t), the
                                 * offline form of the streaming agent (waitk_transformer.py:102-110).  < 0, or > 0 on a model
                                 * without cross-attention or in b200st_ensemble_beam_search, fails before anything is launched. */
} b200st_decode_state;
int64_t b200st_decode_scratch_floats(b200st_handle h, int32_t B);
/* TransformerDecoder.create_decoding_internal_cache + memorize_memory (transformer_decoder.py:105-147) */
int b200st_decode_init(b200st_handle h, const b200st_buffers* buf, const float* enc_out, const b200st_decode_state* st, void* stream);
/* symbols_to_logits_fn(symbols, cache, time) (encoder_decoder_model.py:243-253): symbols int64 [B] and the position *time_dev
 * are device-resident; appends this position's keys/values to self_kv; logits fp32 [B,V]. */
int b200st_decode_step(b200st_handle h, const b200st_buffers* buf, const b200st_decode_state* st, const int64_t* symbols,
                       const int32_t* time_dev, float* logits, void* stream);
/* sequence_beam_search with beam_size = 1 (neurst/layers/search/beam_search.py:254-439): log_softmax, finished rows emit EOS,
 * UNK masked unless unk_id < 0, EOS masked before min_len, argmax (lowest index on ties), stop when every row has finished
 * or after max_steps = min(T' + extra_decode_length, maximum_decode_length); out_ids [B,max_steps] is padded with EOS.
 * The step is captured once into a CUDA graph and replayed (use_graph); `stream` must not be capturing. */
typedef struct {
  const int64_t* bos_ids;
  int32_t eos_id, unk_id, min_len, max_steps;
  int64_t* out_ids; int32_t* out_len; float* out_logprob;
  void* state_words;            /* >= 256 bytes of device memory for B <= 8; above 8 rows
                                 * b200st_beam_state_bytes(h, B, 1, st->max_len) bytes */
  int32_t use_graph;            /* 2: ONE persistent cooperative kernel for the whole search (grid-wide barriers between the
                                 * phases of a token; falls back to 1 when the grid cannot be co-scheduled, and always above
                                 * 8 rows); 1: one captured CUDA graph of ~40 kernels replayed per token; 0: eager launches */
} b200st_greedy_args;
int b200st_greedy_search(b200st_handle h, const b200st_buffers* buf, const b200st_decode_state* st, const b200st_greedy_args* a,
                         void* stream);
/* mode the last b200st_greedy_search actually ran in: 2 persistent kernel, 1 captured graph, 0 eager launches */
int32_t b200st_greedy_used_graph(void);
/* sequence_beam_search (neurst/layers/search/beam_search.py:254-439): per step, log_softmax with the greedy search's masks,
 * accumulated log-probability times the length penalty (1/len for length_penalty < 0, else ((5+len)/6)^-length_penalty),
 * top-beam_size over the beam_size*V candidates of each utterance (only the first beam's at step 0; lower flat index on
 * ties), then the top_k beams of each utterance by logprob * penalty(length), best first.
 *   st->B counts UTTERANCES: cross_kv and memory_bias are b200st_decode_init's for the B utterances (the memory is not
 *   tiled per beam), while self_kv [dec_layers][2][B*beam_size][max_len][d] and scratch
 *   (b200st_decode_scratch_floats(h, B*beam_size) floats) are sized for B*beam_size rows.  B*beam_size <= 8 with
 *   st->use_shadow 0, <= B200ST_DECODE_MAX_ROWS with use_shadow 1; beam_size <= 8.
 *   out_ids [B*top_k][max_steps] padded with EOS, out_scores / out_logprob / out_len [B*top_k], utterance-major.
 *   state_words: b200st_beam_state_bytes(h, B, beam_size, st->max_len) bytes of device memory.
 *   use_graph: 1 = the step captured once into a CUDA graph and replayed, 0 = eager launches.  beam_size == 1 is the greedy
 *   search (b200st_greedy_search, where use_graph 2 selects its persistent kernel) with the score computed from its result.
 * Invalid arguments (too many rows, beam_size > 8, top_k outside 1..beam_size, max_steps > max_len, null buffers) fail
 * before anything is launched. */
typedef struct {
  const int64_t* bos_ids;       /* [B] */
  int32_t eos_id, unk_id, min_len, max_steps;
  int32_t beam_size, top_k;
  float length_penalty;
  int64_t* out_ids; float* out_scores; float* out_logprob; int32_t* out_len;
  void* state_words;
  int32_t use_graph;
} b200st_beam_args;
int64_t b200st_beam_state_bytes(b200st_handle h, int32_t B, int32_t beam_size, int32_t max_len);
int b200st_beam_search(b200st_handle h, const b200st_buffers* buf, const b200st_decode_state* st, const b200st_beam_args* a,
                       void* stream);
/* Top-k / nucleus sampling: sequence_sampling_search of TopSampling (neurst/layers/search/sampling.py:76-250).  Each utterance
 * is tiled sample_num times (row b*sample_num + s is sample s of utterance b).  Per step and row: UNK is masked to FLOAT_MIN
 * (unk_id < 0: not masked), EOS too while time < min_len - 1; the filter keeps the logits >= the k-th largest (top_k > 0,
 * ties kept) or >= the largest value whose upper tail holds softmax mass >= top_p (top_p < 1; everything when no value
 * reaches it); then one id is drawn.  The draw of global row g = row_offset + row at step t: x = the first word of
 * Philox4x32-7(key seed, counter t, stream g) (the dropout generator), u = (x >> 8) * 2^-24, and the id is the first
 * vocabulary index, in index order, whose running sum of kept weights exp(z - max) exceeds u * (their total).  A row that
 * has emitted EOS emits EOS; the search stops when every row has, or after max_steps = max(min(T' + extra_decode_length,
 * maximum_decode_length), minimum_decode_length).  out_logprob: the sum over the drawn ids of the masked, unfiltered
 * log-softmax (the model's log-probability of the sample); out_len: the ids drawn up to and including the first EOS.
 *   st as for b200st_beam_search with beam_size = sample_num (st->B counts utterances); sample_num <= 8; B*sample_num <= 8
 *   with st->use_shadow 0, <= B200ST_DECODE_MAX_ROWS with use_shadow 1.  out_ids [B*sample_num][max_steps] padded with EOS.
 *   state_words: b200st_beam_state_bytes(h, B, sample_num, st->max_len) bytes.  use_graph: 1 = captured step graph, 0 = eager.
 * The selection uses fixed-order reductions only: on the wide step (above 8 rows) the ids are bit-reproducible and a row's
 * ids do not depend on the other rows of the call.  Invalid arguments (top_k < 0 or > vocab, top_k > 0 with top_p < 1, a
 * non-finite top_p, too many rows, max_steps > max_len, null buffers) fail before anything is launched. */
typedef struct {
  const int64_t* bos_ids;       /* [B] */
  int32_t eos_id, unk_id, min_len, max_steps;
  int32_t sample_num, top_k;
  float top_p;
  uint64_t seed;
  int64_t row_offset;           /* global index of row 0 in the draws' key */
  int64_t* out_ids; float* out_logprob; int32_t* out_len;
  void* state_words;
  int32_t use_graph;
} b200st_sampling_args;
int b200st_sampling_search(b200st_handle h, const b200st_buffers* buf, const b200st_decode_state* st, const b200st_sampling_args* a,
                           void* stream);
/* The same selection on caller logits fp32 [rows, V], without masks (top_k_logits / top_p_logits + one categorical draw):
 * out_ids[r] draws with the key (seed, row_offset + r, step). */
int b200st_sample_logits(const float* logits, int32_t rows, int32_t V, int32_t top_k, float top_p, uint64_t seed, int64_t row_offset,
                         int32_t step, int64_t* out_ids, void* stream);
/* Cascade ST handoff (ASR -> MT on the device): one block per utterance reads the ASR search's top-1 hypothesis ids
 * hyp_ids [B][hyp_stride] (first hyp_len columns), truncates at the first asr_eos_id, maps each id through remap
 * [asr_vocab] (int32, ASR target id -> MT source id; an ASR id outside 0..asr_vocab-1 maps to mt_unk_id), applies the MT
 * side's truncation (max_src_len > 0: the first max_src_len - 1 ids and EOS; 0: none), appends mt_eos_id, and writes
 * src_ids [B][out_stride] (padded with mt_pad_id), src_padding [B][out_stride] (1.0 beyond the length) and src_len [B].
 * The remap values must lie in 0..mt_vocab-1 (the caller builds the table).  Bad sizes or ids (B, hyp_len > hyp_stride,
 * table sizes < 1, eos / pad / unk ids outside their vocabulary, out_stride below the longest source) fail before anything is
 * launched.  Integer work only: the outputs do not depend on the launch. */
typedef struct {
  const int64_t* hyp_ids;
  int32_t B, hyp_len, hyp_stride;
  int32_t asr_eos_id, asr_vocab;
  const int32_t* remap;
  int32_t mt_vocab, mt_eos_id, mt_pad_id, mt_unk_id;
  int32_t max_src_len, out_stride;
  int64_t* src_ids;
  float* src_padding;
  int32_t* src_len;
} b200st_cascade_source_args;
int b200st_cascade_source(const b200st_cascade_source_args* a, void* stream);
/* Ensemble decoding: sequence_beam_search over EncoderDecoderEnsembleModel (neurst/models/encoder_decoder_ensemble_model.py;
 * neurst/layers/search/beam_search.py:97-115,486-515).  Per step every member runs its decoder step on the same rows, and the
 * search continues from log(sum_m w_m softmax(logits_m)) (evaluated as a log-sum-exp over the members) with the masks,
 * scores and outputs of b200st_beam_search.
 *   members[m]: a handle, its buffers and its decode state, each as for b200st_beam_search (st->B counts utterances; cross_kv
 *   and memory_bias are that member's b200st_decode_init for the B utterances; self_kv and scratch are sized for
 *   B*beam_size rows of that member's handle).  Every member keeps its own caches and scratch; they share the beam state.
 *   Must agree across members: vocab, st->B, st->Tm and st->max_len.  d, heads and the layer counts may differ, and the
 *   members' precisions and use_shadow too, as long as every member can decode B*beam_size rows: above 8 rows every member
 *   needs use_shadow 1 and a 16-bit handle.
 *   weight: finite and >= 0 with a positive sum; the library normalises the weights to sum 1 (BeamSearch's
 *   ensemble_weights: "average" is 1/n each).  A zero weight leaves that member out of the mixture.
 *   a: as for b200st_beam_search; state_words holds b200st_beam_state_bytes(members[0].h, B, beam_size, st->max_len) bytes.
 *   beam_size 1 runs the beam path with one beam (the reference's greedy search is sequence_beam_search(beam_size=1)).
 * n_members is 1..B200ST_ENSEMBLE_MAX_MODELS; one member is exactly b200st_beam_search.  Invalid arguments fail before anything
 * is launched. */
#define B200ST_ENSEMBLE_MAX_MODELS 8
typedef struct {
  b200st_handle h; const b200st_buffers* buf; const b200st_decode_state* st;
  float weight;                 /* >= 0; normalised by the library */
} b200st_ensemble_member;
int b200st_ensemble_beam_search(const b200st_ensemble_member* members, int32_t n_members, const b200st_beam_args* a, void* stream);

/* Streaming simultaneous translation: the wait-k agent's read / write loop on one source stream (SimulTransTextAgent,
 * neurst/utils/simuleval_agents/simul_trans_text_agent.py; WaitkTransformer.incremental_encode / incremental_decode,
 * neurst/models/waitk_transformer.py:119-140).  A session decodes one stream with 1..B200ST_ENSEMBLE_MAX_MODELS text
 * Transformer members with a monotonic encoder (encoder_monotonic = 1), sharing the target vocabulary and d.
 *   Per member, caller-owned device buffers (nothing is allocated on the device after set-up):
 *     enc_kv   fp32 [enc_layers][2][max_src][d]: each encoder layer's self-attention keys / values
 *     cross_kv fp32 [dec_layers][max_src][2d]: the memory keys | values, appended as the source grows
 *     self_kv  fp32 [dec_layers][2][max_trg][d]
 *     enc_out  optional fp32 [max_src][d]: the encoder output rows (after its final LayerNorm), NULL: not written
 *     scratch  b200st_stream_scratch_floats(h) floats
 *   use_shadow as for b200st_decode_state: 1 reads the embeddings, the attention projections (qkv / q / out) and the FFN
 *   kernels of both stacks from the 16-bit shadow; the cross K/V projection, biases and LayerNorm parameters always come from
 *   the master arena, and all arithmetic is fp32.
 *   lens_dev: device int32[2] = {src_len (source ids encoded), trg_len (decoder positions used)}, caller-owned; the session
 *   keeps host mirrors of both to check calls before anything is launched.
 * b200st_stream_read appends n >= 1 source ids (device int64 [n]) at positions src_len .. src_len + n - 1 for every member:
 *   embedding + sinusoid at the absolute positions, each encoder layer (the new rows attend causally to the cached keys and
 *   to each other), the final LayerNorm, and each decoder layer's cross K/V of the new rows; then src_len += n.
 * b200st_stream_write runs one decoder step per member at position trg_len on the symbol in *out_id_dev, attending to the
 *   memory [0, src_len) with no lag mask; mixes the members' log-probabilities (weights NULL: equal, the agent's
 *   logsumexp_m(log_softmax_m) - log n; otherwise normalised to sum 1; one member: log_softmax); takes the argmax (lower index
 *   on ties, no UNK or minimum-length mask); writes the id to *out_id_dev (the next step's symbol) and sets trg_len += 1.  The
 *   step is captured once into a CUDA graph (again when out_id_dev or the weights change) and replayed: `stream` must be a
 *   stream that can capture (not capturing already, not the legacy default stream).
 * Invalid calls fail before anything is launched: src_len + n > max_src, trg_len == max_trg, a write before any read,
 * members with different vocabularies or d, a handle without a monotonic encoder. */
typedef struct {
  int32_t max_src, max_trg;
  float* enc_kv; float* cross_kv; float* self_kv; float* enc_out;
  float* scratch;
  int32_t use_shadow;
} b200st_stream_state;
typedef struct {
  b200st_handle h; const b200st_buffers* buf; const b200st_stream_state* st;
} b200st_stream_member;
typedef struct b200st_stream_session* b200st_stream;
int64_t b200st_stream_scratch_floats(b200st_handle h);
/* host object only; the members' buffers must outlive it */
int b200st_stream_create(const b200st_stream_member* members, int32_t n_members, int32_t* lens_dev, b200st_stream* out);
int b200st_stream_destroy(b200st_stream s);
/* zeroes src_len and trg_len (the caches need no clearing: the lengths bound every read of them) */
int b200st_stream_reset(b200st_stream s, void* stream);
int b200st_stream_read(b200st_stream s, int32_t n, const int64_t* ids, void* stream);
int b200st_stream_write(b200st_stream s, const float* weights, int64_t* out_id_dev, void* stream);
/* the host mirrors of src_len and trg_len */
int b200st_stream_lengths(b200st_stream s, int32_t* src_len, int32_t* trg_len);

/* 16-bit shadow of the parameter arena (wgmma operands); shadow_dtype = B200ST_BF16 or B200ST_F16 */
int b200st_refresh_shadow(const float* params, void* shadow, int32_t shadow_dtype, int64_t numel, void* stream);

/* Optimizer step of GradAccumKerasModel.train_step (neurst/training/gradaccum_keras_model.py:222-240): unscale ->
 * tf.clip_by_value / tf.clip_by_norm PER GRADIENT TENSOR -> Keras Adam (epsilon-hat form), with the 16-bit shadow refresh and
 * gradient zeroing in the same pass.  loss_scale_state != NULL enables the reference's dynamic loss scale
 * (neurst/training/revised_dynamic_loss_scale.py:60-107): device float[8] = {scale, finite steps in a row, last step skipped,
 * skipped steps, applied steps, global gradient norm, 1/scale latch, reserved}; a step whose gradients are not all finite
 * is skipped (parameters untouched, gradients zeroed) and halves the scale; `growth_steps` finite steps double it.
 * h may be NULL (whole arena = one tensor); numel must then be a multiple of 8, as every arena the library lays out is
 * (refused otherwise, before any launch).  clip_value keeps a NaN gradient NaN, as tf.clip_by_value does.
 * tensor_sumsq: device float[param_count + 1] scratch (clip_norm / loss scale).
 *
 * An optional per-element mask makes it one of two other steps; setting both, or either without a handle, is refused
 * before any launch.  Their bitmaps are device, numel / 8 bytes, bit j of byte b is element 8b + j.
 *
 * prune: weight pruning during training, the reference's pruning optimizer (neurst/sparsity/pruning_optimizer.py, built
 *   with keep_prune_property=True), with its schedules (neurst/sparsity/pruning_schedule.py).  state[0] counts the updates
 *   applied in this run (the optimizer's iterations, from 1; a step the dynamic loss scale skips does not count).  A pruning
 *   turn is an applied update with step >= begin_step, (step <= end_step or end_step < 0) and
 *   (step - begin_step) % frequency == 0.  Off a turn: Adam, then w *= mask.  On a turn: Adam without the old mask, then per
 *   pruned tensor k = round(size * (1 - sparsity)) in float32 (half to even), threshold = the k-th largest |w| counting
 *   duplicates, mask = |w| >= threshold and w *= mask.  The sparsity is target_sparsity (B200ST_PRUNE_CONSTANT) or
 *   (initial - target) * (1 - clip((step - begin) / (end - begin), 0, 1)) ** polynomial_power + target
 *   (B200ST_PRUNE_POLYNOMIAL), in float32.  Masked weights are written as zero in the parameter and shadow arenas; their Adam
 *   moments keep moving, so a later turn can bring them back.  Gradients are never masked.  Nothing synchronises with the
 *   host.  The schedule is refused as the reference's constructors refuse it (and PolynomialDecay with
 *   end_step == begin_step), and so is a sparsity that leaves some pruned tensor with k == 0.
 * frozen: partial tuning of a pruned model (Prune-Tune, examples/prune_tune/src/partial_tuning_optimizer.py): every element
 *   whose bit is 1 keeps the weight it had before the step, in the parameter arena and in the 16-bit shadow
 *   (w = w_orig * original_mask + w * tuning_mask); 1 in the alignment padding.  The Adam moments, the gradient statistics
 *   and the loss-scale state advance exactly as in the plain step, and the free elements get its weights bit for bit. */
#define B200ST_PRUNE_CONSTANT 0
#define B200ST_PRUNE_POLYNOMIAL 1
#define B200ST_PRUNE_MAX_TENSORS 512
typedef struct {
  uint8_t* mask;                /* device, numel / 8 bytes: bit j of byte b = 1 keeps element 8b + j; 1 outside the pruned
                                 * tensors.  The owner derives it from weight != 0 when a run starts (masks are not checkpointed) */
  const int32_t* tensor_ids;    /* host: the pruned tensors' indices (b200st_param_info order), each once */
  int32_t n_tensors;            /* 1..B200ST_PRUNE_MAX_TENSORS */
  int32_t schedule;             /* B200ST_PRUNE_CONSTANT or B200ST_PRUNE_POLYNOMIAL */
  double initial_sparsity, target_sparsity;   /* float32(initial - target), taken in double, and float32(target) enter the
                                               * float32 formula, as the reference's Python floats do */
  float polynomial_power;
  int64_t begin_step, end_step, frequency;
  int32_t* state;               /* device int32[4], zero when a run starts: {applied updates, this update was a pruning turn,
                                 * pruning turns so far, float bits of the last turn's sparsity} */
  float* thresholds;            /* device float[n_tensors] or NULL: each tensor's |w| threshold at the last turn */
  void* scratch;                /* device, b200st_prune_scratch_bytes(n_tensors) bytes, zero-filled once before the first call */
} b200st_prune_args;
typedef struct b200st_optim_args_ {
  float* params; float* grads; float* m; float* v;
  void* shadow; int32_t shadow_dtype;
  int64_t numel;
  float lr, beta1, beta2, eps;
  int64_t step_t;               /* Adam's t (from 1) when loss_scale_state is NULL; else t = applied steps on the device */
  float grad_scale;             /* 1 / (replicas * update_cycle) */
  int32_t zero_grad;
  float clip_value, clip_norm;  /* <= 0: off */
  float* tensor_sumsq;
  float* loss_scale_state;
  float growth_steps, multiplier;   /* 0 => 2000, 2 */
  const b200st_prune_args* prune;   /* NULL: no pruning */
  const uint8_t* frozen;            /* NULL: no frozen elements */
} b200st_optim_args;
int b200st_optimizer_step(b200st_handle h, const b200st_optim_args* a, void* stream);
int64_t b200st_prune_scratch_bytes(int32_t n_tensors);
/* The selection alone on n tensors of an arena: tensor i = params[offsets[i], offsets[i] + sizes[i]), offsets multiples of 8,
 * each tensor's slot padded to a multiple of 8 elements.  k: device int64[n], 1 <= k[i] <= sizes[i].  Writes the mask bytes of
 * the tensors, the thresholds (device float[n] or NULL) and zeroes the pruned elements of params and of the 16-bit shadow
 * (or NULL).  scratch as for b200st_prune_args. */
int b200st_prune_select(float* params, void* shadow, const int64_t* offsets, const int64_t* sizes, const int64_t* k, int32_t n,
                        uint8_t* mask, float* thresholds, void* scratch, void* stream);
/* params[i] = 0 (and shadow[i] = +0 when shadow is not NULL; shadow_dtype B200ST_F16 or B200ST_BF16) for every element whose
 * bit of `keep` (same layout) is 0.  n: a multiple of 8. */
int b200st_apply_mask(float* params, void* shadow, int shadow_dtype, const uint8_t* keep, int64_t n, void* stream);

/* layer-level forward (reference layer API).  need_bytes != NULL: only report the workspace size. */
int b200st_encoder_forward(b200st_handle h, const b200st_buffers* buf, const float* x, const float* padding, int32_t B,
                           int32_t T, float* out, int32_t training, uint64_t seed, void* stream, uint64_t* need_bytes);
int b200st_decoder_forward(b200st_handle h, const b200st_buffers* buf, const float* x, const float* memory,
                           const float* memory_padding, int32_t B, int32_t L, int32_t Tm, float* out, int32_t training,
                           uint64_t seed, void* stream, uint64_t* need_bytes);
int b200st_mha_forward(b200st_handle h, const b200st_buffers* buf, const float* query, const float* memory,
                       const float* bias_2d, int32_t B, int32_t Tq, int32_t Tk, float* out, void* stream,
                       uint64_t* need_bytes);

/* criterion alone: LabelSmoothedCrossEntropy.__call__/reduce_loss (label_smoothed_cross_entropy.py:94-157,46-53) */
int b200st_lsce(const float* logits, const int64_t* trg, const int64_t* trg_length, int32_t B, int32_t L, int32_t V,
                float label_smoothing, float* nll_sum, float* n_tokens, float* loss, void* dlogits, int32_t dlogits_dtype,
                float loss_scale, void* stream);
/* LayerNormalization (common_layers.py:64-65) */
int b200st_layernorm_fwd(const void* x, int32_t x_dtype, const float* gamma, const float* beta, float eps, void* y,
                         int32_t y_dtype, float* mean, float* rstd, int64_t rows, int32_t cols, int32_t relu, void* stream);
int b200st_layernorm_bwd(const void* dy, int32_t dy_dtype, const void* x, int32_t x_dtype, const float* mean,
                         const float* rstd, const float* gamma, const float* beta, const float* dres, void* dx,
                         int32_t dx_dtype, float* dgamma, float* dbeta, int64_t rows, int32_t cols, int32_t relu, void* stream);
/* softmax over keys with additive [B,Tk] bias / causal mask (multi_head_attention.py:147-160); S fp32 [B,H,Tq,ldS] */
int b200st_softmax_fwd(const float* S, int64_t ldS, const float* bias_2d, int32_t causal, void* P, int32_t p_dtype,
                       int64_t ldP, int32_t B, int32_t H, int32_t Tq, int32_t Tk, void* stream);
/* conv subsampling front-end pieces (audio_modalities.py:84-109) */
int b200st_conv1_ln_relu_fwd(const float* src, const float* w, const float* b, const float* gamma, const float* beta,
                             void* y1, int32_t dtype, int32_t B, int32_t T, int32_t F, int32_t Cin, int32_t C,
                             int32_t use_ln, void* stream);

/* dropout bookkeeping for tests: the keep-mask (uint8) of site `stream_id` under `seed`, element i in [0,n) */
uint64_t b200st_dropout_stream_id(const char* site);
int b200st_dropout_mask(uint64_t seed, uint64_t stream_id, int64_t n, float p, uint8_t* out, void* stream);

/* tests/bench only: time `iters` back-to-back launches of one GEMM with CUDA events on `stream` (no host overhead) */
int b200st_gemm_bench(const b200st_gemm_args* args, int32_t iters, float* ms_per_iter, void* stream);

/* bench only: per-launch CUDA-event timing of the wgmma GEMM launches issued between begin and end
 * (sum of kernel durations in ms, sum of their algorithmic FLOPs, number of launches) */
int b200st_profile_begin(void);
int b200st_profile_end(double* gemm_ms, double* gemm_flops, int64_t* gemm_launches);

#ifdef __cplusplus
}
#endif
#endif /* B200ST_H_ */
