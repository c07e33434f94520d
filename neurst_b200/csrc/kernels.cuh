// Host launchers of the non-GEMM kernels (LayerNorm, softmax, dropout casts, reductions, positions,
// embedding, label-smoothed CE, Adam, conv front-end).  All activations are `dtype`-tagged raw pointers
// (F32 in the fp32 parity mode, BF16 in the wgmma mode); statistics, residual stream, gradients of
// parameters and the loss are always fp32.
#pragma once
#include "common.cuh"

namespace b200st {

extern int64_t g_kernel_launches;

// y = LN(x) (* gamma + beta) [relu]; x: [rows, cols] in x_dtype; y in y_dtype; optional fp32 copy y32.
// mean / rstd (fp32 [rows]) may be null.  (neurst/layers/common_layers.py:64-65,77; audio_modalities.py:73-74,103-104)
int layernorm_fwd(const void* x, int x_dtype, const float* gamma, const float* beta, float eps, void* y, int y_dtype,
                  float* y32, float* mean, float* rstd, int64_t rows, int cols, int relu, cudaStream_t s);
int layernorm_fwd_copy(const void* x, int x_dtype, const float* gamma, const float* beta, float eps, void* y, int y_dtype,
                       float* y32, float* mean, float* rstd, int64_t rows, int cols, int relu, float* xcopy, cudaStream_t s);
// dx = [dres +] LN'(dy) ; dgamma/dbeta += ; relu: dy is masked where LN(x)*gamma+beta <= 0 (conv front-end).
int layernorm_bwd(const void* dy, int dy_dtype, const void* x, int x_dtype, const float* mean, const float* rstd,
                  const float* gamma, const float* beta, const float* dres, void* dx, int dx_dtype, float* dgamma,
                  float* dbeta, int64_t rows, int cols, int relu, cudaStream_t s);
// + dnext = cast(dropout'(dx)) for the next backward block (its first kernel fused into this one)
int layernorm_bwd_next(const void* dy, int dy_dtype, const void* x, int x_dtype, const float* mean, const float* rstd,
                       const float* gamma, const float* beta, const float* dres, void* dx, int dx_dtype, float* dgamma,
                       float* dbeta, int64_t rows, int cols, int relu, void* dnext, int dnext_dtype, DropoutSpec ndrop,
                       cudaStream_t s);

// P = softmax(S + bias[b, k] + causal) over k (multi_head_attention.py:147-160,207-208).
// S fp32 [B,H,Tq,ldS]; bias fp32 [B,Tk] or null; causal: key k visible to query q iff k <= q + (Tk - Tq).
// Writes P_pre and (if drop.p > 0) P_drop = dropout(P_pre), both `p_dtype` with row stride ldP.
int softmax_fwd(const float* S, int64_t ldS, const float* bias, int causal, void* P_pre, void* P_drop, int p_dtype,
                int64_t ldP, int B, int H, int Tq, int Tk, DropoutSpec drop, cudaStream_t s);
// dS = P * (dP' - sum_k dP' P), dP' = dropout'(dP); dP fp32 [rows, ldS], output `p_dtype` [rows, ldP].
int softmax_bwd(const float* dP, int64_t ldS, const void* P_pre, void* dS, int p_dtype, int64_t ldP, int64_t rows,
                int Tk, DropoutSpec drop, cudaStream_t s);

// y(dtype) = dropout(x fp32) over n elements (post-process dropout backward: common_layers.py:80-83)
int cast_dropout(const float* x, void* y, int y_dtype, int64_t n, DropoutSpec drop, cudaStream_t s);
// db[n] += sum_m dY[m, n]
int colsum_accum(const void* dY, int dtype, int64_t M, int N, int64_t ld, float* db, cudaStream_t s);

// x[b,t,:] = dropout(v[b,t,:] * scale + sinusoid(t + t0)) (common_layers.py:357-434); v fp32 -> x fp32
int posenc_fwd(const float* v, float* x, int B, int T, int d, float scale, int t0, DropoutSpec drop, cudaStream_t s);
// dv(dtype) = dropout'(dx) * scale
int posenc_bwd(const float* dx, void* dv, int dv_dtype, int64_t n, float scale, DropoutSpec drop, cudaStream_t s);

// x[b,l,:] = dropout(E[ids[b,l]] * sqrt(d) + sinusoid(l + t0)) (text_modalities.py:84-92)
int embed_fwd(const int64_t* ids, const float* E, float* x, int B, int L, int d, int V, int t0, DropoutSpec drop,
              cudaStream_t s);
int embed_bwd(const int64_t* ids, const float* dx, float* dE, int B, int L, int d, int V, DropoutSpec drop,
              cudaStream_t s);

// bias[b,k] = (k >= len[b]) ? -1e9 : 0   with len from `lengths` after `n_conv` ceil-halvings
// (speech_transformer.py:179-189, layer_utils.py:19-32)
// klen (optional): int32 [B] = number of leading non-padded keys (the fused attention skips key blocks beyond it)
int length_to_bias(const int64_t* lengths, float* bias, int B, int T, int n_halvings, cudaStream_t s, int32_t* klen = nullptr);
int padding_to_bias(const float* padding, float* bias, int64_t n, cudaStream_t s);

// label-smoothed CE forward (+ backward when dlogits != null) (label_smoothed_cross_entropy.py:94-157,46-53)
// logits fp32 [B*L, V]; outputs nll_sum[B], n_tokens[B], loss[1] = sum nll / sum tokens;
// dlogits(dtype)[B*L, V] = w/sum_tokens * loss_scale * (softmax - soft_target)
int lsce_fwd_bwd(const float* logits, const int64_t* trg, const int64_t* trg_length, int B, int L, int V,
                 float label_smoothing, float* nll_sum, float* n_tokens, float* loss, void* dlogits, int d_dtype,
                 float loss_scale, const float* loss_scale_dev, cudaStream_t s);

// ---- optimizer step (optim.cu) --------------------------------------------------------------------------------------
// Offsets of the parameter tensors inside the flat arena (each a multiple of 8 elements; tensor i = [off[i], off[i+1]))
// travel as a kernel argument: per-tensor gradient norms and the per-tensor clip need no device-side table.
struct TensorTable {
  int n;
  uint32_t off8[513];      // offsets / 8
};
// Device-resident control block of the step (6 floats), caller-owned:
//   [0] loss scale S (fp16 precision: the loss gradient was multiplied by S)   [1] consecutive finite steps
//   [2] 1 when the LAST step was skipped (non-finite gradients)                [3] number of skipped steps so far
//   [4] number of applied steps (Adam's t)                                      [5] global gradient norm of the last step
struct OptimArgs {
  float* p; float* g; float* m; float* v;
  void* shadow; int shadow_dtype;     // 16-bit copy of the arena refreshed in the same pass (or null)
  int64_t n;
  float lr, beta1, beta2, eps;
  int64_t step_t;                     // Adam's t when `ctl` is null (host-counted); with `ctl` t = ctl[4] + 1
  float grad_scale;                   // 1 / (replicas * update_cycle)
  int zero_grad;
  float clip_value, clip_norm;        // <= 0: off.  tf.clip_by_value / tf.clip_by_norm PER TENSOR (gradaccum_keras_model.py:228-233)
  float* tensor_sumsq;                // [n_tensors + 1] scratch (needed for clip_norm or ctl); last = total
  float* ctl;                         // dynamic loss scale state or null
  float growth_steps, multiplier;     // revised_dynamic_loss_scale.py:82-107 (2000, 2)
};
int optimizer_step(const OptimArgs& a, const TensorTable& tt, cudaStream_t s);
int cast_f32_to_16(const float* x, void* y, int y_dtype, int64_t n, cudaStream_t s);
// out[g] = keep-bits of elements [8g, 8g+8) of the dropout site (identical to the on-the-fly Philox decisions)
int dropout_bits(DropoutSpec drop, int64_t n_elems, uint8_t* out, cudaStream_t s);
// all dropout sites of a step in one launch: site i covers groups [goff[i], goff[i+1]) and writes base[boff[i] + local]
struct DropBitsTable {
  int n;
  uint64_t stream[128];
  uint32_t thresh[128];
  int64_t goff[129];
  int64_t boff[128];
};
int dropout_bits_multi(const DropBitsTable& t, uint64_t seed, const uint64_t* seed_ptr, uint8_t* base, cudaStream_t s);
int fill_f32(float* x, float v, int64_t n, cudaStream_t s);

// ---- fused attention (16-bit operand type `dt` = BF16 or F16, head dim 64): wgmma QK^T / PV with on-chip online softmax (attention.cu) ----
// q/k/v/ctx/dctx/dq/dk/dv: bf16 views [B*T, ld], head h at columns [h*64, h*64+64); bias fp32 [B,Tk] or null;
// lse fp32 [B,H,Tq] (written by forward, read by backward); dq_scratch fp32 [B*Tq, H*64] followed by [B*H*Tq] floats (rowsum(dO*O)).
// kv_len (optional, int32 [B]): keys >= kv_len[b] all carry the -1e9 padding bias — their probabilities are exactly 0 in
// fp32, so whole key blocks beyond it are skipped (bit-identical result; ragged batches of cfg-4)
int attention_fwd_fused(int dt, const void* q, int64_t q_ld, const void* k, int64_t k_ld, const void* v, int64_t v_ld, int B, int H,
                        int Tq, int Tk, const float* bias, int causal, DropoutSpec drop, void* ctx, int64_t ctx_ld, float* lse,
                        cudaStream_t s, const int32_t* kv_len = nullptr);
int attention_bwd_fused(int dt, const void* q, int64_t q_ld, const void* k, int64_t k_ld, const void* v, int64_t v_ld, const void* ctx,
                        int64_t ctx_ld, const void* dctx, int64_t dctx_ld, const float* lse, int B, int H, int Tq, int Tk,
                        const float* bias, int causal, DropoutSpec drop, float* dq_scratch, void* dq, int64_t dq_ld, void* dk,
                        int64_t dk_ld, void* dv, int64_t dv_ld, cudaStream_t s, const int32_t* kv_len = nullptr);

// ---- conv front-end (audio_modalities.py:84-109) ----
// y1 = relu(LN(conv3x3s2(src) + b)); src fp32 [B,T,F,Cin]; w fp32 HWIO [3,3,Cin,C]; y1 (dtype) [B,T1,F1,C]
int conv1_ln_relu_fwd(const float* src, const float* w, const float* b, const float* gamma, const float* beta, float eps,
                      void* y1, int y_dtype, int B, int T, int F, int Cin, int C, int use_ln, cudaStream_t s);
// Fused backward of conv1's LN+ReLU fed by conv2's dgrad: dy1 = col2im(dcol) (transpose of im2col), ReLU mask from y1,
// z1 recomputed from src, dz1 = LN'(dy1) written in `dtype`, col1[pos, 0..K1p) = im2col row of src (zero padded) for the
// filter-gradient GEMM, and db / dgamma / dbeta accumulated.
int conv1_bwd_fused(const float* src, const float* w, const float* b, const float* gamma, const float* beta, float eps,
                    const void* y1, const void* dcol, int dtype, void* dz1, void* col1, int K1p, float* db, float* dgamma,
                    float* dbeta, int B, int T, int F, int Cin, int C, int use_ln, cudaStream_t s);
// col[(b,t2,f2), (kh,kw,c)] = y1[b, 2*t2+kh-1, 2*f2+kw-1, c] (zero outside)
int im2col_3x3s2(const void* y1, void* col, int dtype, int B, int T1, int F1, int C, cudaStream_t s);
// normalised-save front-end (training path at C == 256, Cin == 1): conv1 stores xhat + 1/sigma, the im2col applies
// gamma / beta / ReLU in flight, the backward reads xhat back instead of recomputing the convolution
int conv1_norm_fwd(const float* src, const float* w, const float* b, float eps, void* xhat, int dtype, float* rstd, int B, int T,
                   int F, int Cin, int C, cudaStream_t s);
int im2col_3x3s2_affine(const void* y1, void* col, int dtype, int B, int T1, int F1, int C, const void* gamma, const void* beta,
                        cudaStream_t s);   // gamma / beta in the activation dtype (bf16 shadow or fp32 master)
int conv1_bwd_from_xhat(const float* src, const void* gamma, const void* beta, const void* xhat, const float* rstd,
                        const void* dcol, int dtype, void* dz1, void* col1, int K1p, float* db, float* dgamma, float* dbeta, int B,
                        int T, int F, int C, cudaStream_t s, int implicit_tiles = 0);
// conv2 data gradient as four implicit GEMMs (tc_gemm.cu); da = class-major padded tiles, conv2_dgrad_implicit_elems() elements
int conv2_dgrad_implicit(const void* dy, const void* w16, void* da, int dtype, int B, int T2, int F2, int C, cudaStream_t stream);
int64_t conv2_dgrad_implicit_elems(int B, int T2, int F2, int C);

}  // namespace b200st
