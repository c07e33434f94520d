// Streaming simultaneous translation on the device: the wait-k agent's incremental encoding and decoding.
//
// Replaces, for one source stream decoded by 1..8 members,
//   WaitkTransformer.incremental_encode      neurst/models/waitk_transformer.py:119-130
//   TransformerEncoder.incremental_encode    neurst/layers/encoders/transformer_encoder.py:138-175 (per-layer self-attention
//                                            caches; the new rows attend causally to the cache and to each other)
//   TransformerDecoder.update_incremental_cache  neurst/layers/decoders/transformer_decoder.py:149-169 (the new memory rows'
//                                            cross-attention keys / values are appended)
//   WaitkTransformer.incremental_decode + the agent's mixing and top_k(1)
//                                            neurst/utils/simuleval_agents/simul_trans_text_agent.py (predict)
//
// A READ of n source ids runs, per member, in pieces of at most 8 rows (the GEMV kernels' row limit; the encoder is causal,
// so a piece sees exactly the keys the whole chunk would): the embedding at the absolute positions, each encoder layer
// (LN + QKV GEMV, stream_attn_kernel appending the keys / values to the layer's cache and attending causally, fused with
// the output projection into the residual stream, LN + FFN), then each decoder layer's cross K/V projection of the final
// LayerNorm of the new rows.  Positions come from the host mirror of src_len, so a READ is a handful of eager launches.
// A WRITE is one decoder step per member at position trg_len over the memory prefix [0, src_len) (both device words,
// read at run time), the agent's equal-weight mixture, the argmax and the length update: nothing in it depends on a host
// value that changes between calls, so it is captured once into a CUDA graph and replayed.
//
// Weights are read from the fp32 master arena or, with use_shadow, from the 16-bit shadow: the source and target
// embeddings, and per layer the attention projections (qkv / q / out) and the FFN kernels.  Biases, LayerNorm parameters
// and the cross-attention K/V projection always come from the master arena; all arithmetic and every cache are fp32.
#include "beam.cuh"
#include "decode_step.cuh"
#include "model.cuh"
#include "pdl.cuh"

#include <cmath>
#include <string>
#include <vector>

namespace b200st {

namespace {

// x[r,:] = E[ids[r],:] * sqrt(d) + sinusoid(pos0 + r)   (_src_modality(..., time=pos0), text_modalities.py:84-92)
template <typename TW>
__global__ void stream_embed_kernel(const int64_t* __restrict__ ids, const TW* __restrict__ E, float* __restrict__ x, int n, int d,
                                    int V, int pos0) {
  pdl_wait();
  pdl_trigger();
  const float scale = sqrtf((float)d);
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n * d; i += gridDim.x * blockDim.x) {
    const int r = i / d, c = i % d;
    int64_t id = ids[r];
    id = id < 0 ? 0 : (id >= V ? V - 1 : id);
    x[i] = wf(E, id * d + c) * scale + sinusoid_at(pos0 + r, c, d);
  }
}

// One block per (head, new row r) of a chunk whose first row sits at position base = (*len_dev, or 0) + pos0.
// SELF (encoder chunk / decoder step self-attention, multi_head_attention.py:271-289): q / k / v of the new rows come from
// the qkv accumulator [rows][3d]; row r's key and value are stored at cache position base + r, and row r attends to the
// keys 0 .. base + r: the cached ones (< base) from the cache, those of the chunk's own rows from the accumulator (another
// block of this launch writes them to the cache).  Cross (!SELF): q from qsrc [rows][d], keys = the memory rows
// 0 .. base - 1 of the pre-projected cross K/V, with no bias: an unpadded stream's memory_bias is all zeros.
// q is scaled by dh^-0.5 after the projection bias (multi_head_attention.py:203); the context goes through this head's
// slice of the output projection into the residual stream x[r] (+ the bias once, from head 0).
template <typename TW, bool SELF>
__global__ void __launch_bounds__(256) stream_attn_kernel(const float* __restrict__ qsrc, int q_ld, float* __restrict__ kcache,
                                                          float* __restrict__ vcache, int kv_ld, const int* __restrict__ len_dev, int pos0,
                                                          const TW* __restrict__ Wo, const float* __restrict__ bo, float* __restrict__ x,
                                                          int d, int dh) {
  pdl_wait();
  pdl_trigger();
  extern __shared__ float sm[];          // q[dh] | ctx[dh] | scores[nk] | red[8]
  const int h = blockIdx.x, r = blockIdx.y;
  const int base = (len_dev ? *len_dev : 0) + pos0;
  const int nk = SELF ? base + r + 1 : base;
  float* q = sm;
  float* ctx = sm + dh;
  float* sc = sm + 2 * dh;
  float* red = sc + nk;
  const float* qrow = qsrc + (int64_t)r * q_ld + h * dh;
  // key / value j: the cache row j, or (SELF, j >= base) the accumulator row j - base
  const float* kb = kcache + h * dh;
  const float* vb = vcache + h * dh;
  const float* kn = qsrc + d + h * dh;
  const float* vn = qsrc + 2 * d + h * dh;
  const float alpha = rsqrtf((float)dh);
  for (int c = threadIdx.x; c < dh; c += blockDim.x) {
    q[c] = qrow[c] * alpha;
    ctx[c] = 0.f;
    if (SELF) {
      kcache[(int64_t)(base + r) * kv_ld + h * dh + c] = qrow[d + c];
      vcache[(int64_t)(base + r) * kv_ld + h * dh + c] = qrow[2 * d + c];
    }
  }
  __syncthreads();
  for (int j = threadIdx.x; j < nk; j += blockDim.x) {
    const float* kr = (SELF && j >= base) ? kn + (int64_t)(j - base) * q_ld : kb + (int64_t)j * kv_ld;
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
    sc[j] = s;
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
      // the cached keys' values, then (SELF) the chunk's own rows' from the accumulator
      const int ncache = nk < base ? nk : base;
      float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;
      int j = part;
      for (; j + 3 * nparts < ncache; j += 4 * nparts) {
        a0 = fmaf(sc[j], vb[(int64_t)j * kv_ld + c], a0);
        a1 = fmaf(sc[j + nparts], vb[(int64_t)(j + nparts) * kv_ld + c], a1);
        a2 = fmaf(sc[j + 2 * nparts], vb[(int64_t)(j + 2 * nparts) * kv_ld + c], a2);
        a3 = fmaf(sc[j + 3 * nparts], vb[(int64_t)(j + 3 * nparts) * kv_ld + c], a3);
      }
      for (; j < ncache; j += nparts) a0 = fmaf(sc[j], vb[(int64_t)j * kv_ld + c], a0);
      if (SELF)
        for (; j < nk; j += nparts) a1 = fmaf(sc[j], vn[(int64_t)(j - base) * q_ld + c], a1);
      atomicAdd(&ctx[c], (a0 + a1 + a2 + a3) * inv);
    }
  }
  __syncthreads();
  for (int n = threadIdx.x; n < d; n += blockDim.x) {
    float a = (h == 0 && bo) ? bo[n] : 0.f;
    const TW* wp = Wo + (int64_t)h * dh * d + n;
#pragma unroll 8
    for (int c = 0; c < dh; ++c) a = fmaf(ctx[c], wf(wp, (int64_t)c * d), a);
    atomicAdd(x + (int64_t)r * d + n, a);
  }
}

// The agent's choice (simul_trans_text_agent.py predict): top_k(1) of the log-probabilities — log_softmax of one member's
// logits (raw), or the members' mixture, already log-probabilities — the lower index on ties, with no UNK or minimum-length
// mask.  The id becomes the next decoder input and trg_len advances.
__global__ void __launch_bounds__(1024) stream_pick_kernel(const float* __restrict__ z, int V, int raw, int64_t* __restrict__ out_id,
                                                           int32_t* __restrict__ lens) {
  pdl_wait();
  pdl_trigger();
  __shared__ float red[32];
  __shared__ float sval[32];
  __shared__ int sidx[32];
  float lse = 0.f;
  if (raw) {
    float mx = -INFINITY;
    for (int v = threadIdx.x; v < V; v += blockDim.x) mx = fmaxf(mx, z[v]);
    mx = block_max(mx, red);
    float se = 0.f;
    for (int v = threadIdx.x; v < V; v += blockDim.x) se += expf(z[v] - mx);
    se = block_sum(se, red);
    lse = mx + logf(se);
  }
  float best = -INFINITY; int bi = 0x7fffffff;
  for (int v = threadIdx.x; v < V; v += blockDim.x) {
    const float lp = z[v] - lse;
    if (lp > best || (lp == best && v < bi)) { best = lp; bi = v; }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float ob = __shfl_xor_sync(0xffffffffu, best, o);
    const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
    if (ob > best || (ob == best && oi < bi)) { best = ob; bi = oi; }
  }
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  if (lane == 0) { sval[w] = best; sidx[w] = bi; }
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int i = 1; i < (int)(blockDim.x >> 5); ++i)
      if (sval[i] > sval[0] || (sval[i] == sval[0] && sidx[i] < sidx[0])) { sval[0] = sval[i]; sidx[0] = sidx[i]; }
    *out_id = sidx[0];
    lens[1] += 1;
  }
}

// src_len += n after every member has read the chunk
__global__ void stream_advance_kernel(int32_t* __restrict__ lens, int n) {
  pdl_wait();
  pdl_trigger();
  if (threadIdx.x == 0) lens[0] += n;
}

// Offsets (floats) inside a member's scratch: the encoder piece (x, per-layer qkv / FFN hidden accumulators) and the
// decoder step (x, per-layer qkv / cross q / FFN hidden accumulators, logits).  Each group of accumulators is contiguous,
// so one memset clears it.
struct StreamLayout {
  int64_t ex, eqkv, ehid, eend, dx, dqkv, dqc, dhid, dend, logits, total;
};
StreamLayout stream_layout(const Config& c) {
  StreamLayout l{};
  int64_t o = 0;
  l.ex = o; o += (int64_t)MAXB * c.d;
  l.eqkv = o; o += (int64_t)c.enc_layers * MAXB * 3 * c.d;
  l.ehid = o; o += (int64_t)c.enc_layers * MAXB * c.ffn;
  l.eend = o;
  l.dx = o; o += c.d;
  l.dqkv = o; o += (int64_t)c.dec_layers * 3 * c.d;
  l.dqc = o; o += (int64_t)c.dec_layers * c.d;
  l.dhid = o; o += (int64_t)c.dec_layers * c.ffn;
  l.dend = o;
  l.logits = o; o += c.vocab;
  l.total = o;
  return l;
}

size_t stream_attn_smem(const Config& c, int keys) { return sizeof(float) * (size_t)(2 * (c.d / c.heads) + keys + 8); }

template <typename K>
int raise_smem_to(K kern, size_t smem) {
  if (smem > 48 * 1024) B200ST_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  return 0;
}

}  // namespace

struct StreamSession {
  std::vector<StreamMember> mem;
  int32_t* lens = nullptr;       // device {src_len, trg_len}
  int src_len = 0, trg_len = 0;  // host mirrors
  cudaGraph_t graph = nullptr;
  cudaGraphExec_t exec = nullptr;
  int64_t* graph_out = nullptr;  // the out_id word and the weights the captured step was built with
  std::vector<float> graph_w;
  int graph_raw = 0;
  void drop_graph() {
    if (exec) cudaGraphExecDestroy(exec);
    if (graph) cudaGraphDestroy(graph);
    exec = nullptr; graph = nullptr;
  }
};

namespace {

struct MemberCtx {
  const StreamMember& sm;
  cudaStream_t s;
  const float* P(const std::string& n) const { return sm.buf.params + sm.m->params[sm.m->find(n)].offset; }
  int64_t off(const std::string& n) const { return sm.m->params[sm.m->find(n)].offset; }
};

// One piece of m <= 8 source rows at the absolute position pos of one member.
template <typename TW>
int read_piece(const MemberCtx& c, const TW* wb, const int64_t* ids, int m, int pos) {
  const Config& cf = c.sm.m->cfg;
  const StreamState& st = c.sm.st;
  const int d = cf.d, H = cf.heads, dh = d / H, f = cf.ffn;
  const StreamLayout lo = stream_layout(cf);
  float* x = st.scratch + lo.ex;
  auto W = [&](const std::string& n) { return wb + c.off(n); };
  B200ST_CUDA(cudaMemsetAsync(st.scratch + lo.eqkv, 0, sizeof(float) * (size_t)(lo.eend - lo.eqkv), c.s));
  for (int i = 0; i < cf.dec_layers; ++i)
    B200ST_CUDA(cudaMemsetAsync(st.cross_kv + ((int64_t)i * st.max_src + pos) * 2 * d, 0, sizeof(float) * (size_t)m * 2 * d, c.s));
  const bool shared = cf.share_src_trg_embedding != 0;
  const std::string tab = shared ? "trg.emb" : "srcemb.emb";
  B200ST_TRY(launch(stream_embed_kernel<TW>, (m * d + 255) / 256, 256, 0, c.s, ids, (const TW*)W(tab), x, m, d,
                    shared ? cf.vocab : cf.src_vocab, pos));
  const size_t smem = stream_attn_smem(cf, st.max_src);
  for (int i = 0; i < cf.enc_layers; ++i) {
    const std::string p = "enc." + std::to_string(i);
    float* qkv = st.scratch + lo.eqkv + (int64_t)i * MAXB * 3 * d;
    float* hid = st.scratch + lo.ehid + (int64_t)i * MAXB * f;
    float* ek = st.enc_kv + (int64_t)i * 2 * st.max_src * d;
    float* ev = ek + (int64_t)st.max_src * d;
    B200ST_TRY(launch(gemv_kernel<TW, 0>, dim3((3 * d + 127) / 128, (d + 31) / 32), 128, 0, c.s, (const float*)x, c.P(p + ".att.ln.gamma"),
                      c.P(p + ".att.ln.beta"), (const float*)nullptr, cf.ln_eps, W(p + ".att.qkv.kernel"), c.P(p + ".att.qkv.bias"), qkv, m, d, 3 * d));
    B200ST_TRY(launch(stream_attn_kernel<TW, true>, dim3(H, m), 256, smem, c.s, (const float*)qkv, 3 * d, ek, ev, d, (const int*)nullptr, pos,
                      W(p + ".att.out.kernel"), c.P(p + ".att.out.bias"), x, d, dh));
    B200ST_TRY(launch(gemv_kernel<TW, 0>, dim3((f + 127) / 128, (d + 31) / 32), 128, 0, c.s, (const float*)x, c.P(p + ".ffn.ln.gamma"),
                      c.P(p + ".ffn.ln.beta"), (const float*)nullptr, cf.ln_eps, W(p + ".ffn.w1"), (const float*)nullptr, hid, m, d, f));
    B200ST_TRY(launch(gemv_kernel<TW, 1>, dim3((d + 127) / 128, (f + 31) / 32), 128, 0, c.s, (const float*)hid, (const float*)nullptr,
                      (const float*)nullptr, c.P(p + ".ffn.b1"), 0.f, W(p + ".ffn.w2"), c.P(p + ".ffn.b2"), x, m, f, d));
  }
  if (st.enc_out)
    B200ST_TRY(layernorm_fwd(x, F32, c.P("enc.out_ln.gamma"), c.P("enc.out_ln.beta"), cf.ln_eps, st.enc_out + (int64_t)pos * d, F32,
                             nullptr, nullptr, nullptr, m, d, 0, c.s));
  // memorize the new memory rows: cross K/V = LN_enc(x) . kv.kernel + kv.bias (fp32 master weights, as b200st_decode_init)
  for (int i = 0; i < cf.dec_layers; ++i) {
    const std::string p = "dec." + std::to_string(i) + ".cross.kv";
    B200ST_TRY(launch(gemv_kernel<float, 0>, dim3((2 * d + 127) / 128, (d + 31) / 32), 128, 0, c.s, (const float*)x, c.P("enc.out_ln.gamma"),
                      c.P("enc.out_ln.beta"), (const float*)nullptr, cf.ln_eps, c.P(p + ".kernel"), c.P(p + ".bias"),
                      st.cross_kv + ((int64_t)i * st.max_src + pos) * 2 * d, m, d, 2 * d));
  }
  return 0;
}

// One decoder step of one member at position trg_len over the memory prefix [0, src_len); logits [V] in its scratch.
template <typename TW>
int write_step(const MemberCtx& c, const TW* wb, const int64_t* sym, const int32_t* lens) {
  const Config& cf = c.sm.m->cfg;
  const StreamState& st = c.sm.st;
  const int d = cf.d, H = cf.heads, dh = d / H, f = cf.ffn, V = cf.vocab;
  const StreamLayout lo = stream_layout(cf);
  float* x = st.scratch + lo.dx;
  auto W = [&](const std::string& n) { return wb + c.off(n); };
  B200ST_CUDA(cudaMemsetAsync(st.scratch + lo.dqkv, 0, sizeof(float) * (size_t)(lo.dend - lo.dqkv), c.s));
  B200ST_TRY(launch(embed_step_kernel<TW>, (d + 255) / 256, 256, 0, c.s, sym, W("trg.emb"), x, 1, d, V, lens + 1));
  const size_t smem_self = stream_attn_smem(cf, st.max_trg), smem_cross = stream_attn_smem(cf, st.max_src);
  for (int i = 0; i < cf.dec_layers; ++i) {
    const std::string p = "dec." + std::to_string(i);
    float* qkv = st.scratch + lo.dqkv + (int64_t)i * 3 * d;
    float* qc = st.scratch + lo.dqc + (int64_t)i * d;
    float* hid = st.scratch + lo.dhid + (int64_t)i * f;
    float* sk = st.self_kv + (int64_t)i * 2 * st.max_trg * d;
    float* sv = sk + (int64_t)st.max_trg * d;
    float* ck = st.cross_kv + (int64_t)i * st.max_src * 2 * d;
    B200ST_TRY(launch(gemv_kernel<TW, 0>, dim3((3 * d + 127) / 128, (d + 31) / 32), 128, 0, c.s, (const float*)x, c.P(p + ".self.ln.gamma"),
                      c.P(p + ".self.ln.beta"), (const float*)nullptr, cf.ln_eps, W(p + ".self.qkv.kernel"), c.P(p + ".self.qkv.bias"), qkv, 1, d, 3 * d));
    B200ST_TRY(launch(stream_attn_kernel<TW, true>, dim3(H, 1), 256, smem_self, c.s, (const float*)qkv, 3 * d, sk, sv, d, lens + 1, 0,
                      W(p + ".self.out.kernel"), c.P(p + ".self.out.bias"), x, d, dh));
    B200ST_TRY(launch(gemv_kernel<TW, 0>, dim3((d + 127) / 128, (d + 31) / 32), 128, 0, c.s, (const float*)x, c.P(p + ".cross.ln.gamma"),
                      c.P(p + ".cross.ln.beta"), (const float*)nullptr, cf.ln_eps, W(p + ".cross.q.kernel"), c.P(p + ".cross.q.bias"), qc, 1, d, d));
    B200ST_TRY(launch(stream_attn_kernel<TW, false>, dim3(H, 1), 256, smem_cross, c.s, (const float*)qc, d, ck, ck + d, 2 * d, lens, 0,
                      W(p + ".cross.out.kernel"), c.P(p + ".cross.out.bias"), x, d, dh));
    B200ST_TRY(launch(gemv_kernel<TW, 0>, dim3((f + 127) / 128, (d + 31) / 32), 128, 0, c.s, (const float*)x, c.P(p + ".ffn.ln.gamma"),
                      c.P(p + ".ffn.ln.beta"), (const float*)nullptr, cf.ln_eps, W(p + ".ffn.w1"), (const float*)nullptr, hid, 1, d, f));
    B200ST_TRY(launch(gemv_kernel<TW, 1>, dim3((d + 127) / 128, (f + 31) / 32), 128, 0, c.s, (const float*)hid, (const float*)nullptr,
                      (const float*)nullptr, c.P(p + ".ffn.b1"), 0.f, W(p + ".ffn.w2"), c.P(p + ".ffn.b2"), x, 1, f, d));
  }
  return launch(logits_step_kernel<TW>, 132 * 2, 256, sizeof(float) * (size_t)d, c.s, (const float*)x, c.P("dec.out_ln.gamma"),
                c.P("dec.out_ln.beta"), cf.ln_eps, W("trg.emb"), c.P("trg.bias"), st.scratch + lo.logits, 1, d, V);
}

// Runs fn(wbase) with the member's weights: the 16-bit shadow (use_shadow) or the fp32 master arena.
template <typename Fn>
int with_weights(const StreamMember& sm, Fn&& fn) {
  if (sm.st.use_shadow) {
    if (sm.m->adt == F16) return fn(reinterpret_cast<const __half*>(sm.buf.shadow));
    return fn(reinterpret_cast<const __nv_bfloat16*>(sm.buf.shadow));
  }
  return fn(sm.buf.params);
}

int raise_stream_smem(size_t smem) {
  B200ST_TRY(raise_smem_to(stream_attn_kernel<float, true>, smem)); B200ST_TRY(raise_smem_to(stream_attn_kernel<float, false>, smem));
  B200ST_TRY(raise_smem_to(stream_attn_kernel<__half, true>, smem)); B200ST_TRY(raise_smem_to(stream_attn_kernel<__half, false>, smem));
  B200ST_TRY(raise_smem_to(stream_attn_kernel<__nv_bfloat16, true>, smem));
  return raise_smem_to(stream_attn_kernel<__nv_bfloat16, false>, smem);
}

// The captured WRITE: every member's step, the mixture (several members), the pick.
int write_body(StreamSession& ss, const std::vector<float>& w, int64_t* out_id, cudaStream_t s) {
  const int n = (int)ss.mem.size();
  for (const StreamMember& sm : ss.mem) {
    const MemberCtx c{sm, s};
    B200ST_TRY(with_weights(sm, [&](auto wb) { return write_step(c, wb, out_id, ss.lens); }));
  }
  const int V = ss.mem[0].m->cfg.vocab;
  float* z0 = ss.mem[0].st.scratch + stream_layout(ss.mem[0].m->cfg).logits;
  if (n > 1) {
    EnsembleMix mix{};
    mix.n = n;
    for (int i = 0; i < n; ++i) {
      mix.z[i] = ss.mem[i].st.scratch + stream_layout(ss.mem[i].m->cfg).logits;
      mix.logw[i] = w[i];
    }
    B200ST_TRY(ensemble_logprob(mix, 1, V, s));
  }
  return launch(stream_pick_kernel, 1, 1024, 0, s, (const float*)z0, V, n > 1 ? 0 : 1, out_id, ss.lens);
}

}  // namespace

int64_t stream_scratch_floats(const Model& m) { return stream_layout(m.cfg).total + 64; }

int stream_create(const StreamMember* mem, int n, int32_t* lens_dev, StreamSession** out) {
  B200ST_CHECK(out != nullptr && mem != nullptr && lens_dev != nullptr, "stream_create: null argument");
  B200ST_CHECK(n >= 1 && n <= kEnsembleMaxModels,
               "a streaming session has 1.." + std::to_string(kEnsembleMaxModels) + " members, got " + std::to_string(n));
  size_t smem = 0;
  for (int i = 0; i < n; ++i) {
    const std::string who = "stream member " + std::to_string(i) + ": ";
    B200ST_CHECK(mem[i].m != nullptr, who + "null handle");
    const Config& cf = mem[i].m->cfg;
    const StreamState& st = mem[i].st;
    B200ST_CHECK(cf.model_type == MODEL_TEXT && cf.with_cross_attention, who + "streaming needs a text Transformer handle");
    B200ST_CHECK(cf.encoder_monotonic, who + "streaming needs a monotonic encoder (encoder_monotonic = 1): the incremental "
                                             "encoding equals the whole-prefix encoding only when no row sees later rows");
    B200ST_CHECK(cf.vocab == mem[0].m->cfg.vocab,
                 who + "vocabulary of " + std::to_string(cf.vocab) + " differs from member 0's " + std::to_string(mem[0].m->cfg.vocab));
    B200ST_CHECK(cf.d == mem[0].m->cfg.d, who + "d = " + std::to_string(cf.d) + " differs from member 0's " + std::to_string(mem[0].m->cfg.d));
    B200ST_CHECK(st.max_src >= 1 && st.max_trg >= 1, who + "max_src and max_trg must be >= 1");
    B200ST_CHECK(st.max_src == mem[0].st.max_src && st.max_trg == mem[0].st.max_trg, who + "max_src / max_trg differ from member 0's");
    B200ST_CHECK(st.enc_kv && st.cross_kv && st.self_kv && st.scratch && mem[i].buf.params, who + "state buffers missing");
    B200ST_CHECK(!st.use_shadow || (is16(mem[i].m->adt) && mem[i].buf.shadow),
                 who + "use_shadow needs a 16-bit precision handle and its shadow arena");
    const int dh = cf.d / cf.heads;
    B200ST_CHECK(dh <= 256 && 256 % dh == 0, who + "the stream kernels need a head dim that divides 256");
    const size_t need = stream_attn_smem(cf, st.max_src > st.max_trg ? st.max_src : st.max_trg);
    B200ST_CHECK(need <= 200 * 1024, who + "too many keys for the shared-memory score buffer");
    smem = need > smem ? need : smem;
  }
  B200ST_TRY(raise_stream_smem(smem));
  StreamSession* ss = new StreamSession();
  ss->mem.assign(mem, mem + n);
  ss->lens = lens_dev;
  *out = ss;
  return 0;
}

void stream_destroy(StreamSession* ss) {
  if (!ss) return;
  ss->drop_graph();
  delete ss;
}

int stream_reset(StreamSession* ss, cudaStream_t s) {
  B200ST_CUDA(cudaMemsetAsync(ss->lens, 0, 2 * sizeof(int32_t), s));
  ss->src_len = 0;
  ss->trg_len = 0;
  return 0;
}

void stream_lengths(const StreamSession* ss, int* src_len, int* trg_len) {
  if (src_len) *src_len = ss->src_len;
  if (trg_len) *trg_len = ss->trg_len;
}

int stream_read(StreamSession* ss, int n, const int64_t* ids, cudaStream_t s) {
  const int max_src = ss->mem[0].st.max_src;
  B200ST_CHECK(n >= 1 && ids != nullptr, "stream_read needs n >= 1 source ids");
  B200ST_CHECK(ss->src_len + n <= max_src, "stream_read: src_len + n = " + std::to_string(ss->src_len) + " + " + std::to_string(n) +
                                               " exceeds max_src = " + std::to_string(max_src));
  for (const StreamMember& sm : ss->mem) {
    const MemberCtx c{sm, s};
    for (int o = 0; o < n; o += MAXB) {
      const int m = n - o < MAXB ? n - o : MAXB;
      B200ST_TRY(with_weights(sm, [&](auto wb) { return read_piece(c, wb, ids + o, m, ss->src_len + o); }));
    }
  }
  B200ST_TRY(launch(stream_advance_kernel, 1, 32, 0, s, ss->lens, n));
  ss->src_len += n;
  return 0;
}

int stream_write(StreamSession* ss, const float* weights, int64_t* out_id, cudaStream_t s) {
  const int n = (int)ss->mem.size();
  B200ST_CHECK(out_id != nullptr, "stream_write: null out_id");
  B200ST_CHECK(ss->src_len >= 1, "stream_write needs at least one source token read");
  B200ST_CHECK(ss->trg_len < ss->mem[0].st.max_trg, "stream_write: trg_len has reached max_trg = " + std::to_string(ss->mem[0].st.max_trg));
  std::vector<float> w(n, -std::log((float)n));          // the agent's mixture: logsumexp_m(log_softmax_m) - log n
  if (weights) {
    double sum = 0.0;
    for (int i = 0; i < n; ++i) {
      B200ST_CHECK(std::isfinite(weights[i]) && weights[i] >= 0.f, "stream weights must be finite and >= 0");
      sum += weights[i];
    }
    B200ST_CHECK(sum > 0.0, "stream weights must have a positive sum");
    for (int i = 0; i < n; ++i) w[i] = (float)std::log((double)weights[i] / sum);
  }
  if (!ss->exec || ss->graph_out != out_id || ss->graph_w != w) {
    ss->drop_graph();
    B200ST_CUDA(cudaStreamBeginCapture(s, cudaStreamCaptureModeThreadLocal));
    const int rc = write_body(*ss, w, out_id, s);
    const cudaError_t e = cudaStreamEndCapture(s, &ss->graph);
    if (rc != 0) { ss->drop_graph(); return rc; }
    if (e != cudaSuccess || !ss->graph || cudaGraphInstantiate(&ss->exec, ss->graph, 0) != cudaSuccess) {
      cudaGetLastError();
      ss->drop_graph();
      B200ST_FAIL("stream_write could not capture its step into a CUDA graph (is the stream capturing or the legacy default stream?)");
    }
    ss->graph_out = out_id;
    ss->graph_w = w;
  }
  B200ST_CUDA(cudaGraphLaunch(ss->exec, s));
  ss->trg_len += 1;
  return 0;
}

}  // namespace b200st
