// Decoder step on 9..256 rows (utterances x beam) with the 16-bit shadow weights — DESIGN.md §4, "the wide step".
//
// The <= 8-row step (decode.cu) is a set of GEMV kernels with one fp32 accumulator per row in registers; at the recipes'
// 64 utterances x beam 4 the same contractions are 2.8 G FMA per token, which belongs on the tensor cores.  Here every
// projection is one rows-GEMM launch  C[rows, N] = epi(pre(A)[rows, K] . W)  on wgmma:
//   pre: the pre-norm LayerNorm (per-row mean / rstd computed by the block), relu(a + b1) (the FFN's second product) or none
//   A:   fp32 activations split into 16-bit terms in registers (fp16: hi + lo, bf16: hi + mid + lo; term i is the rounded
//        residual of the terms before it) and fed to wgmma as register A operands; every term is multiplied by the same
//        weight tile and accumulated in fp32, so the product keeps fp32 accuracy on the shadow's rounded weights.  The fp16
//        split needs every GEMM input within the fp16 range (|a| < 65504), as the reference's mixed_float16 does.
//   W:   the shadow tensor through TMA into a 4-stage ring of 128B-swizzled [64 k x 64 n] tiles: MN-major [in, out] for the
//        projections, K-major [V, d] for the tied logits
//   epi: fp32 store (+ bias) or fp32 add (+ bias) into the residual stream x in place (one owner per element)
// Block = one warpgroup on a 64-row x 64-column tile; thread 0 also issues the TMA loads.  Only the products into the d-wide
// residual stream with K >= 512 are split along K (the FFN's second product; the output projections from d = 512 on), into
// slices of at least 256, at most 8 (k_splits): the rule reads K, N and d, never the row count, so a row's arithmetic does
// not depend on how many rows share the step; slices store fp32 partials and the last slice to arrive (ticket per tile)
// sums them in slice order.  No floating-point atomics anywhere in the step: it is bit-reproducible.
// The tile, ring depth and slice rule are first estimates, not tuned on measurements.
//
// The attentions run on CUDA cores in fp32 and write their context to scratch (the output projection is a rows GEMM):
// self-attention one block per (head, row) over the cache as attn_step_kernel does (ancestry table in beam search);
// cross-attention one block per (head, utterance) serving every beam row of the utterance, so the memory keys / values are
// read once per utterance instead of once per beam.  Partial sums are combined in a fixed order.
#include "decode_rows.cuh"
#include "pdl.cuh"
#include "ptx.cuh"

#include <type_traits>

namespace b200st {

int make_tma_map_16(const void* ptr, int dtype, uint64_t inner, uint64_t rows, int nb1, int nb2, int64_t ld, int64_t sb1, int64_t sb2,
                    uint32_t box_rows, CUtensorMap* out);

namespace {

constexpr int kRowsThreads = 128;                // one warpgroup
constexpr int kRowsStages = 4;
constexpr uint32_t kRowsStageBytes = 64 * 64 * 2;
constexpr size_t kRowsSmem = 1024 + kRowsStages * kRowsStageBytes + 2 * 8 * kRowsStages;
constexpr int kMaxSplits = 8;
constexpr int kMaxTickets = 1024;
constexpr int kBeamMax = 8;                      // KMAX of decode.cu
constexpr int kAttnThreads = 256;
enum { PRE_LN = 0, PRE_RELU_BIAS = 1, PRE_NONE = 2 };
enum { EPI_STORE = 0, EPI_ADD = 1 };

struct RowsParams {
  const float* A;                // [M, K] fp32
  int M, K, N;
  const float* gamma; const float* beta; float eps;     // PRE_LN
  const float* pre_bias;                                // PRE_RELU_BIAS
  const float* bias;             // [N] or null
  float* C;                      // [M, N] fp32
  int splits, kb_per_split;      // K slices (gridDim.z) and 64-wide k-blocks per slice
  float* partial;                // [splits][M][N] when splits > 1
  int* tickets;                  // [m tiles * n tiles], zero between launches (the last slice resets its tile's)
};

template <int PRE>
__device__ __forceinline__ float2 pre_value(const RowsParams& p, float2 v, int col, float mean, float rstd) {
  if (PRE == PRE_LN) {
    const float2 g = __ldg(reinterpret_cast<const float2*>(p.gamma + col)), b = __ldg(reinterpret_cast<const float2*>(p.beta + col));
    return make_float2((v.x - mean) * rstd * g.x + b.x, (v.y - mean) * rstd * g.y + b.y);
  }
  if (PRE == PRE_RELU_BIAS) {
    const float2 b = __ldg(reinterpret_cast<const float2*>(p.pre_bias + col));
    return make_float2(fmaxf(v.x + b.x, 0.f), fmaxf(v.y + b.y, 0.f));
  }
  return v;
}

template <bool BF, bool B_MN, int PRE, int EPI>
__global__ void __launch_bounds__(kRowsThreads) rows_gemm_kernel(const __grid_constant__ CUtensorMap tmW, const RowsParams p) {
  extern __shared__ uint8_t smem_raw[];
  __shared__ float s_mean[64], s_rstd[64];
  __shared__ int s_last;
  constexpr int DT = BF ? BF16 : F16;
  constexpr int TERMS = BF ? 3 : 2;
  const uint32_t base = (ptx::smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t sW = base;
  const uint32_t bars = sW + kRowsStages * kRowsStageBytes;
  auto full = [&](int s2) { return bars + 8u * s2; };
  auto empty = [&](int s2) { return bars + 8u * (kRowsStages + s2); };
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, q = lane & 3;
  const int n0 = blockIdx.x * 64, m_blk = blockIdx.y, split = blockIdx.z;
  const int nkb = p.kb_per_split, kb0 = split * nkb;
  const bool producer = threadIdx.x == 0;
  if (producer) {
    ptx::prefetch_tensormap(&tmW);
    for (int s2 = 0; s2 < kRowsStages; ++s2) { ptx::mbar_init(full(s2), 1); ptx::mbar_init(empty(s2), kRowsThreads / 32); }
    ptx::fence_mbar_init();
  }
  __syncthreads();
  pdl_wait();
  pdl_trigger();
  auto issue = [&](int it) {
    if (it >= nkb) return;
    const int st = it % kRowsStages;
    ptx::mbar_wait(empty(st), (((uint32_t)(it / kRowsStages)) & 1u) ^ 1u);
    ptx::mbar_arrive_expect_tx(full(st), kRowsStageBytes);
    const int k0 = (kb0 + it) * 64;
    if (B_MN) ptx::tma_load_4d(sW + st * kRowsStageBytes, &tmW, full(st), n0, k0, 0, 0);     // W [K, N]: 64 n x 64 k box
    else ptx::tma_load_4d(sW + st * kRowsStageBytes, &tmW, full(st), k0, n0, 0, 0);          // E [N, K]: 64 k x 64 n box
  };
  if (producer)
    for (int it = 0; it < kRowsStages; ++it) issue(it);

  // this thread's rows of the tile: r0 and r0 + 8 (the wgmma fragment rows of its warp)
  const int r0 = warp * 16 + g;
  const int mA = m_blk * 64 + r0, mB = mA + 8;
  const bool okA = mA < p.M, okB = mB < p.M;
  if (PRE == PRE_LN) {
    // per-row statistics of the whole row (two passes, fp32), a warp per 16 rows
    for (int r = warp * 16; r < warp * 16 + 16; ++r) {
      const int m = m_blk * 64 + r;
      float mean = 0.f, rstd = 0.f;
      if (m < p.M) {
        const float* row = p.A + (int64_t)m * p.K;
        float s = 0.f;
        for (int k = lane; k < p.K; k += 32) s += row[k];
        mean = warp_sum(s) / (float)p.K;
        float v = 0.f;
        for (int k = lane; k < p.K; k += 32) { const float dl = row[k] - mean; v += dl * dl; }
        rstd = rsqrtf(warp_sum(v) / (float)p.K + p.eps);
      }
      if (lane == 0) { s_mean[r] = mean; s_rstd[r] = rstd; }
    }
    __syncwarp();
  }
  const float meanA = PRE == PRE_LN ? s_mean[r0] : 0.f, rstdA = PRE == PRE_LN ? s_rstd[r0] : 0.f;
  const float meanB = PRE == PRE_LN ? s_mean[r0 + 8] : 0.f, rstdB = PRE == PRE_LN ? s_rstd[r0 + 8] : 0.f;
  const float* rowA = p.A + (int64_t)(okA ? mA : 0) * p.K;
  const float* rowB = p.A + (int64_t)(okB ? mB : 0) * p.K;

  // raw[s][h][r]: rows (r0, r0 + 8) x columns 16 s + 8 h + 2 q + {0, 1} of a 64-wide k-block
  float2 raw[4][2][2];
  auto load_raw = [&](int it) {
    const int k0 = (kb0 + it) * 64 + 2 * q;
#pragma unroll
    for (int s2 = 0; s2 < 4; ++s2)
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int k = k0 + 16 * s2 + 8 * h;
        raw[s2][h][0] = okA ? *reinterpret_cast<const float2*>(rowA + k) : make_float2(0.f, 0.f);
        raw[s2][h][1] = okB ? *reinterpret_cast<const float2*>(rowB + k) : make_float2(0.f, 0.f);
      }
  };
  float acc[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) acc[i] = 0.f;
  load_raw(0);
  for (int it = 0; it < nkb; ++it) {
    // split-term A fragments: a[t][s][2 h + r] = term t of (row r0 + 8 r, columns 16 s + 8 h + 2 q + {0, 1})
    uint32_t a[TERMS][4][4];
    const int k0 = (kb0 + it) * 64 + 2 * q;
#pragma unroll
    for (int s2 = 0; s2 < 4; ++s2)
#pragma unroll
      for (int h = 0; h < 2; ++h)
#pragma unroll
        for (int r = 0; r < 2; ++r) {
          const int col = k0 + 16 * s2 + 8 * h;
          float2 v = pre_value<PRE>(p, raw[s2][h][r], col, r ? meanB : meanA, r ? rstdB : rstdA);
          if (!(r ? okB : okA)) v = make_float2(0.f, 0.f);
#pragma unroll
          for (int t = 0; t < TERMS; ++t) {
            const uint32_t pk = pack2_16(v.x, v.y, DT);
            a[t][s2][2 * h + r] = pk;
            const float2 back = unpack2_16(pk, DT);
            v = make_float2(v.x - back.x, v.y - back.y);     // exact in fp32: the residual the next term rounds
          }
        }
    if (it + 1 < nkb) load_raw(it + 1);                    // in flight while the tensor cores run
    const int st = it % kRowsStages;
    ptx::mbar_wait(full(st), ((uint32_t)(it / kRowsStages)) & 1u);
    const uint32_t tile = sW + st * kRowsStageBytes;
    ptx::fence_acc(acc);
    ptx::wgmma_fence();
#pragma unroll
    for (int s2 = 0; s2 < 4; ++s2)
#pragma unroll
      for (int t = TERMS - 1; t >= 0; --t)                 // smallest term first
        ptx::WgmmaRS<64, BF, B_MN ? 1 : 0>::mma(acc, a[t][s2], B_MN ? ptx::desc_mnmajor(tile, s2) : ptx::desc_kmajor(tile, s2), 1);
    ptx::wgmma_commit();
    ptx::wgmma_wait<0>();
    ptx::fence_acc(acc);
    if (lane == 0) ptx::mbar_arrive(empty(st));
    if (producer) issue(it + kRowsStages);
    __syncwarp();
  }

  // epilogue: acc[4 j + 2 hr + {0, 1}] = D[r0 + 8 hr][8 j + 2 q + {0, 1}]
  auto finish = [&](int m, int n, float2 v) {
    float2 b = make_float2(0.f, 0.f);
    if (p.bias) b = __ldg(reinterpret_cast<const float2*>(p.bias + n));
    float2* c = reinterpret_cast<float2*>(p.C + (int64_t)m * p.N + n);
    if (EPI == EPI_ADD) { const float2 x = *c; *c = make_float2(x.x + (v.x + b.x), x.y + (v.y + b.y)); }
    else *c = make_float2(v.x + b.x, v.y + b.y);
  };
  if (p.splits == 1) {
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int n = n0 + 8 * j + 2 * q;
#pragma unroll
      for (int hr = 0; hr < 2; ++hr) {
        const int m = hr ? mB : mA;
        if (m < p.M && n < p.N) finish(m, n, make_float2(acc[4 * j + 2 * hr], acc[4 * j + 2 * hr + 1]));
      }
    }
    return;
  }
  // K slices: store the partial, the last slice of the tile sums the partials in slice order
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const int n = n0 + 8 * j + 2 * q;
#pragma unroll
    for (int hr = 0; hr < 2; ++hr) {
      const int m = hr ? mB : mA;
      if (m < p.M && n < p.N)
        *reinterpret_cast<float2*>(p.partial + ((int64_t)split * p.M + m) * p.N + n) = make_float2(acc[4 * j + 2 * hr], acc[4 * j + 2 * hr + 1]);
    }
  }
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) {
    int* tk = p.tickets + blockIdx.y * gridDim.x + blockIdx.x;
    const int prev = atomicAdd(tk, 1);
    s_last = prev == p.splits - 1;
    if (s_last) *tk = 0;
  }
  __syncthreads();
  if (!s_last) return;
  __threadfence();
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const int n = n0 + 8 * j + 2 * q;
#pragma unroll
    for (int hr = 0; hr < 2; ++hr) {
      const int m = hr ? mB : mA;
      if (m < p.M && n < p.N) {
        float2 v = make_float2(0.f, 0.f);
        for (int s2 = 0; s2 < p.splits; ++s2) {
          const float2 x = __ldcg(reinterpret_cast<const float2*>(p.partial + ((int64_t)s2 * p.M + m) * p.N + n));
          v.x += x.x; v.y += x.y;
        }
        finish(m, n, v);
      }
    }
  }
}

// Self-attention of row b, head h over positions 0..time; appends this position's key / value at `time`.  anc != null (beam
// search): position j < time of row b lives in the cache slot of row anc[b][j].  ctx [rows, d] gets the head's context.
// smem: q[dh] | scores[time + 1] | partial context[blockDim] | red[32] | slot[time + 1]
__global__ void __launch_bounds__(kAttnThreads) rows_self_attn_kernel(const float* __restrict__ qkv, float* __restrict__ kcache,
                                                                     float* __restrict__ vcache, int d, int dh, int max_len,
                                                                     const int32_t* __restrict__ time_dev, const int* __restrict__ anc,
                                                                     float* __restrict__ ctx) {
  pdl_wait();
  pdl_trigger();
  extern __shared__ float sm[];
  const int h = blockIdx.x, b = blockIdx.y;
  const int t = *time_dev, nk = t + 1;
  float* q = sm;
  float* sc = q + dh;
  float* part = sc + nk;
  float* red = part + blockDim.x;
  int* slot = reinterpret_cast<int*>(red + 32);
  const float* qrow = qkv + (int64_t)b * 3 * d + h * dh;
  const float alpha = rsqrtf((float)dh);
  for (int c = threadIdx.x; c < dh; c += blockDim.x) {
    q[c] = qrow[c] * alpha;
    kcache[((int64_t)b * max_len + t) * d + h * dh + c] = qrow[d + c];
    vcache[((int64_t)b * max_len + t) * d + h * dh + c] = qrow[2 * d + c];
  }
  for (int j = threadIdx.x; j < nk; j += blockDim.x) slot[j] = (anc && j < t ? anc[(int64_t)b * max_len + j] : b) * max_len + j;
  __syncthreads();
  const float* kb = kcache + h * dh;
  const float* vb = vcache + h * dh;
  for (int j = threadIdx.x; j < nk; j += blockDim.x) {
    const float* kr = kb + (int64_t)slot[j] * d;
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
  // thread = (column c, key partition): partials in shared memory, summed in partition order
  const int c = threadIdx.x % dh, pt = threadIdx.x / dh, np = blockDim.x / dh;
  float a0 = 0.f, a1 = 0.f;
  int j = pt;
  for (; j + np < nk; j += 2 * np) {
    a0 = fmaf(sc[j], vb[(int64_t)slot[j] * d + c], a0);
    a1 = fmaf(sc[j + np], vb[(int64_t)slot[j + np] * d + c], a1);
  }
  if (j < nk) a0 = fmaf(sc[j], vb[(int64_t)slot[j] * d + c], a0);
  part[threadIdx.x] = a0 + a1;
  __syncthreads();
  if ((int)threadIdx.x < dh) {
    float s = 0.f;
    for (int i = 0; i < np; ++i) s += part[i * dh + threadIdx.x];
    ctx[(int64_t)b * d + h * dh + threadIdx.x] = s * inv;
  }
}

// Cross-attention of the `beam` rows of utterance u, head h over the pre-projected memory ([u][Tm][2d]: keys | values) with
// the additive memory bias: every key and value row is read once for all the utterance's rows.  wait_k > 0: step t scans
// the visible keys j < min(Tm, wait_k + t) only, as attn_step_kernel (decode.cu).
// smem: q[beam][dh] | scores[beam][Tm] | partial context[beam][blockDim] | inv[beam] | red[32]
__global__ void __launch_bounds__(kAttnThreads) rows_cross_attn_kernel(const float* __restrict__ qc, const float* __restrict__ mem,
                                                                      const float* __restrict__ mem_bias, int d, int dh, int Tm,
                                                                      int wait_k, const int32_t* __restrict__ time_dev, int beam,
                                                                      float* __restrict__ ctx) {
  pdl_wait();
  pdl_trigger();
  extern __shared__ float sm[];
  const int h = blockIdx.x, u = blockIdx.y, r0 = u * beam;
  const int nk = wait_k > 0 ? min(Tm, wait_k + *time_dev) : Tm;
  float* q = sm;
  float* sc = q + beam * dh;
  float* part = sc + (int64_t)beam * Tm;
  float* inv = part + beam * blockDim.x;
  float* red = inv + kBeamMax;
  const float alpha = rsqrtf((float)dh);
  for (int i = threadIdx.x; i < beam * dh; i += blockDim.x) q[i] = qc[(int64_t)(r0 + i / dh) * d + h * dh + i % dh] * alpha;
  __syncthreads();
  const float* kb = mem + (int64_t)u * Tm * 2 * d + h * dh;
  const float* vb = kb + d;
  for (int j = threadIdx.x; j < nk; j += blockDim.x) {
    const float* kr = kb + (int64_t)j * 2 * d;
    float s[kBeamMax];
#pragma unroll
    for (int r = 0; r < kBeamMax; ++r) s[r] = 0.f;
    if ((dh & 3) == 0) {
      for (int c = 0; c < dh; c += 4) {
        const float4 kk = *reinterpret_cast<const float4*>(kr + c);
#pragma unroll
        for (int r = 0; r < kBeamMax; ++r) {
          if (r < beam) {
            const float* qr = q + r * dh + c;
            s[r] = fmaf(qr[0], kk.x, fmaf(qr[1], kk.y, fmaf(qr[2], kk.z, fmaf(qr[3], kk.w, s[r]))));
          }
        }
      }
    } else {
      for (int c = 0; c < dh; ++c) {
        const float kk = kr[c];
#pragma unroll
        for (int r = 0; r < kBeamMax; ++r) if (r < beam) s[r] = fmaf(q[r * dh + c], kk, s[r]);
      }
    }
    const float mb = mem_bias ? mem_bias[(int64_t)u * Tm + j] : 0.f;
#pragma unroll
    for (int r = 0; r < kBeamMax; ++r) if (r < beam) sc[(int64_t)r * Tm + j] = s[r] + mb;
  }
  __syncthreads();
  for (int r = 0; r < beam; ++r) {
    float* z = sc + (int64_t)r * Tm;
    float mx = -INFINITY;
    for (int j = threadIdx.x; j < nk; j += blockDim.x) mx = fmaxf(mx, z[j]);
    mx = block_max(mx, red);
    float se = 0.f;
    for (int j = threadIdx.x; j < nk; j += blockDim.x) { const float e = expf(z[j] - mx); z[j] = e; se += e; }
    se = block_sum(se, red);
    if (threadIdx.x == 0) inv[r] = 1.f / se;
  }
  __syncthreads();
  const int c = threadIdx.x % dh, pt = threadIdx.x / dh, np = blockDim.x / dh;
  float a[kBeamMax];
#pragma unroll
  for (int r = 0; r < kBeamMax; ++r) a[r] = 0.f;
  for (int j = pt; j < nk; j += np) {
    const float v = vb[(int64_t)j * 2 * d + c];
#pragma unroll
    for (int r = 0; r < kBeamMax; ++r) if (r < beam) a[r] = fmaf(sc[(int64_t)r * Tm + j], v, a[r]);
  }
#pragma unroll
  for (int r = 0; r < kBeamMax; ++r) if (r < beam) part[r * blockDim.x + threadIdx.x] = a[r];
  __syncthreads();
  for (int i = threadIdx.x; i < beam * dh; i += blockDim.x) {
    const int r = i / dh, cc = i % dh;
    float s = 0.f;
    for (int k = 0; k < np; ++k) s += part[r * blockDim.x + k * dh + cc];
    ctx[(int64_t)(r0 + r) * d + h * dh + cc] = s * inv[r];
  }
}

// greedy_pick_kernel (decode.cu) for row blockIdx.x: log_softmax, finished rows emit EOS, UNK / early-EOS masks, argmax
// with the lowest index on ties
__global__ void __launch_bounds__(1024) rows_greedy_pick_kernel(const float* __restrict__ logits, int64_t* ids, int32_t* finished,
                                                               int32_t* length, float* logprob, int64_t* out, int32_t* time,
                                                               int32_t* all_finished, uint32_t* ticket, int V, int eos, int unk,
                                                               int min_len, int max_steps) {
  pdl_wait();
  pdl_trigger();
  __shared__ float red[32];
  __shared__ float sval[32];
  __shared__ int sidx[32];
  const int b = blockIdx.x;
  const int t = *time;
  const float* z = logits + (int64_t)b * V;
  const bool was_finished = finished[b] != 0;
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
    if (was_finished) lp = (v == eos) ? 0.f : -1.0e9f;
    if (v == unk) lp += -1.0e9f;
    if (v == eos && t < min_len - 1) lp += -1.0e9f;
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
    const int tok = sidx[0];
    out[(int64_t)b * max_steps + t] = tok;
    ids[b] = tok;
    logprob[b] += sval[0];
    length[b] += was_finished ? 0 : 1;
    finished[b] = (tok == eos) ? 1 : 0;
    // the last block of the step publishes all_finished and advances time: every block has read `time` before its ticket
    __threadfence();
    if (atomicAdd(ticket, 1u) == gridDim.x - 1) {
      __threadfence();
      int all = 1;
      for (int r = 0; r < (int)gridDim.x; ++r) all &= __ldcg(finished + r) != 0 ? 1 : 0;
      *all_finished = all;
      *ticket = 0;
      *time = t + 1;
    }
  }
}

struct RowsLayout {          // offsets (floats) inside the scratch buffer
  int64_t x, qkv, qc, ctx, hid, logits, partial, tickets, total;
  int d;
};
RowsLayout rows_layout(const Config& c, int B) {
  RowsLayout l{};
  l.d = c.d;
  int64_t o = 0;
  auto take = [&](int64_t n) { const int64_t at = o; o += (n + 63) / 64 * 64; return at; };
  l.x = take((int64_t)B * c.d);
  l.qkv = take((int64_t)B * 3 * c.d);
  l.qc = take((int64_t)B * c.d);
  l.ctx = take((int64_t)B * c.d);
  l.hid = take((int64_t)B * c.ffn);
  l.logits = take((int64_t)B * c.vocab);
  l.partial = take((int64_t)kMaxSplits * B * c.d);      // split-K partials: k_splits splits only GEMMs with N <= d
  l.tickets = take(kMaxTickets);
  l.total = o;
  return l;
}

template <bool BF, bool B_MN, int PRE, int EPI>
int launch_rows_gemm(const CUtensorMap& tm, const RowsParams& p, dim3 grid, cudaStream_t s) {
  return launch(rows_gemm_kernel<BF, B_MN, PRE, EPI>, grid, kRowsThreads, kRowsSmem, s, tm, p);
}

// K slices of one rows GEMM.  Only the products into the d-wide residual stream (N <= d: the output projections and the
// FFN's second product) are split, into slices of at least 4 k-blocks of 64, at most kMaxSplits, so the partials always fit
// the [kMaxSplits][rows][d] area.  The rule reads K, N and d, never the row count: a row's sums do not depend on how many
// rows share the step.
int k_splits(int K, int N, int d) {
  if (N > d || K < 512) return 1;
  const int kb = K / 64;
  int splits = kMaxSplits;
  while (splits > 1 && (kb % splits != 0 || kb / splits < 4)) --splits;
  return splits;
}

// C[M, N] (=|+=) pre(A)[M, K] . W + bias; W_mn: W is [K, N] (TF [in, out]), else [N, K] (the tied embedding).  rows_check has
// validated the shapes and the split-K scratch of every call.
template <typename TW>
int rows_gemm(const float* A, int M, int K, const TW* W, bool w_mn, int N, int pre, const float* gamma, const float* beta, float eps,
              const float* pre_bias, const float* bias, float* C, int epi, const RowsLayout& lo, float* scratch, cudaStream_t s) {
  constexpr bool BF = std::is_same<TW, __nv_bfloat16>::value;
  CUtensorMap tm;
  if (w_mn) B200ST_TRY(make_tma_map_16(W, BF ? BF16 : F16, (uint64_t)N, (uint64_t)K, 1, 1, N, 0, 0, 64, &tm));
  else B200ST_TRY(make_tma_map_16(W, BF ? BF16 : F16, (uint64_t)K, (uint64_t)N, 1, 1, K, 0, 0, 64, &tm));
  RowsParams p{};
  p.A = A; p.M = M; p.K = K; p.N = N;
  p.gamma = gamma; p.beta = beta; p.eps = eps; p.pre_bias = pre_bias; p.bias = bias; p.C = C;
  const int splits = k_splits(K, N, lo.d);
  const int m_tiles = (M + 63) / 64, n_tiles = (N + 63) / 64;
  p.splits = splits; p.kb_per_split = K / 64 / splits;
  p.partial = scratch + lo.partial;
  p.tickets = reinterpret_cast<int*>(scratch + lo.tickets);
  const dim3 grid(n_tiles, m_tiles, splits);
  if (!w_mn) {
    B200ST_CHECK(pre == PRE_LN && epi == EPI_STORE, "wide decode: unsupported K-major GEMM");
    return launch_rows_gemm<BF, false, PRE_LN, EPI_STORE>(tm, p, grid, s);
  }
  if (pre == PRE_LN && epi == EPI_STORE) return launch_rows_gemm<BF, true, PRE_LN, EPI_STORE>(tm, p, grid, s);
  if (pre == PRE_NONE && epi == EPI_ADD) return launch_rows_gemm<BF, true, PRE_NONE, EPI_ADD>(tm, p, grid, s);
  if (pre == PRE_RELU_BIAS && epi == EPI_ADD) return launch_rows_gemm<BF, true, PRE_RELU_BIAS, EPI_ADD>(tm, p, grid, s);
  B200ST_FAIL("wide decode: unsupported GEMM variant");
}

size_t self_smem(const Config& cf, int max_len) {
  return sizeof(float) * (size_t)(cf.d / cf.heads + max_len + kAttnThreads + 32) + sizeof(int) * (size_t)max_len;
}
size_t cross_smem(const Config& cf, int Tm, int beam) {
  return sizeof(float) * ((size_t)beam * (cf.d / cf.heads + Tm + kAttnThreads) + kBeamMax + 32);
}

template <typename TW>
int rows_step_t(const Model& m, const Buffers& buf, const DecodeState& st, const TW* wbase, const int32_t* time_dev, float* logits,
                const int* anc, int beam, cudaStream_t s) {
  const Config& cf = m.cfg;
  const int B = st.B, d = cf.d, H = cf.heads, dh = d / H, f = cf.ffn, V = cf.vocab;
  const RowsLayout lo = rows_layout(cf, B);
  float* sc = st.scratch;
  float* x = sc + lo.x;
  float* qkv = sc + lo.qkv;
  float* qc = sc + lo.qc;
  float* ctx = sc + lo.ctx;
  float* hid = sc + lo.hid;
  auto P = [&](const std::string& n) -> const float* { const int i = m.find(n); return i < 0 ? nullptr : buf.params + m.params[i].offset; };
  auto W = [&](const std::string& n) -> const TW* { const int i = m.find(n); return i < 0 ? nullptr : wbase + m.params[i].offset; };
  const int64_t self_layer = 2 * (int64_t)B * st.max_len * d, cross_layer = (int64_t)(B / beam) * st.Tm * 2 * d;
  const bool cross = cf.with_cross_attention && st.Tm > 0;
  const size_t smem_self = self_smem(cf, st.max_len), smem_cross = cross_smem(cf, st.Tm, beam);
  B200ST_CUDA(cudaMemsetAsync(sc + lo.tickets, 0, sizeof(int) * kMaxTickets, s));     // split-K tickets of the step
  for (int i = 0; i < cf.dec_layers; ++i) {
    const std::string p = "dec." + std::to_string(i);
    B200ST_TRY(rows_gemm(x, B, d, W(p + ".self.qkv.kernel"), true, 3 * d, PRE_LN, P(p + ".self.ln.gamma"), P(p + ".self.ln.beta"),
                         cf.ln_eps, nullptr, P(p + ".self.qkv.bias"), qkv, EPI_STORE, lo, sc, s));
    float* sk = st.self_kv + (int64_t)i * self_layer;
    B200ST_TRY(launch(rows_self_attn_kernel, dim3(H, B), kAttnThreads, smem_self, s, (const float*)qkv, sk, sk + (int64_t)B * st.max_len * d,
                      d, dh, st.max_len, time_dev, anc, ctx));
    B200ST_TRY(rows_gemm(ctx, B, d, W(p + ".self.out.kernel"), true, d, PRE_NONE, nullptr, nullptr, 0.f, nullptr,
                         P(p + ".self.out.bias"), x, EPI_ADD, lo, sc, s));
    if (cross) {
      B200ST_TRY(rows_gemm(x, B, d, W(p + ".cross.q.kernel"), true, d, PRE_LN, P(p + ".cross.ln.gamma"), P(p + ".cross.ln.beta"),
                           cf.ln_eps, nullptr, P(p + ".cross.q.bias"), qc, EPI_STORE, lo, sc, s));
      B200ST_TRY(launch(rows_cross_attn_kernel, dim3(H, B / beam), kAttnThreads, smem_cross, s, (const float*)qc,
                        (const float*)(st.cross_kv + (int64_t)i * cross_layer), st.memory_bias, d, dh, st.Tm, st.wait_k, time_dev, beam, ctx));
      B200ST_TRY(rows_gemm(ctx, B, d, W(p + ".cross.out.kernel"), true, d, PRE_NONE, nullptr, nullptr, 0.f, nullptr,
                           P(p + ".cross.out.bias"), x, EPI_ADD, lo, sc, s));
    }
    B200ST_TRY(rows_gemm(x, B, d, W(p + ".ffn.w1"), true, f, PRE_LN, P(p + ".ffn.ln.gamma"), P(p + ".ffn.ln.beta"), cf.ln_eps,
                         nullptr, nullptr, hid, EPI_STORE, lo, sc, s));
    B200ST_TRY(rows_gemm(hid, B, f, W(p + ".ffn.w2"), true, d, PRE_RELU_BIAS, nullptr, nullptr, 0.f, P(p + ".ffn.b1"),
                         P(p + ".ffn.b2"), x, EPI_ADD, lo, sc, s));
  }
  B200ST_TRY(rows_gemm(x, B, d, W("trg.emb"), false, V, PRE_LN, P("dec.out_ln.gamma"), P("dec.out_ln.beta"), cf.ln_eps, nullptr,
                       P("trg.bias"), logits, EPI_STORE, lo, sc, s));
  return 0;
}

}  // namespace

int64_t rows_scratch_floats(const Config& c, int B) { return rows_layout(c, B).total + 64; }
int64_t rows_logits_offset(const Config& c, int B) { return rows_layout(c, B).logits; }

int rows_check(const Model& m, const Buffers& buf, const DecodeState& st, int beam) {
  const Config& cf = m.cfg;
  B200ST_CHECK(st.use_shadow && is16(m.adt) && buf.shadow, "decoding more than 8 rows per step needs use_shadow = 1 and the 16-bit shadow");
  B200ST_CHECK(cf.d % 64 == 0 && cf.ffn % 64 == 0 && cf.vocab % 8 == 0,
               "the wide decode step needs d and ffn multiples of 64 and a vocabulary multiple of 8");
  B200ST_CHECK(beam >= 1 && beam <= kBeamMax && st.B % beam == 0, "wide decode: bad beam size");
  const int dh = cf.d / cf.heads;
  B200ST_CHECK(dh <= kAttnThreads && kAttnThreads % dh == 0, "the wide decode step needs a head dim that divides 256");
  // every rows GEMM of the step: its K slices fit the partial area and its tiles the ticket words
  const RowsLayout lo = rows_layout(cf, st.B);
  const int shapes[5][2] = {{cf.d, 3 * cf.d}, {cf.d, cf.d}, {cf.d, cf.ffn}, {cf.ffn, cf.d}, {cf.d, cf.vocab}};   // K, N
  for (const auto& kn : shapes) {
    const int splits = k_splits(kn[0], kn[1], cf.d);
    const int64_t tiles = (int64_t)((st.B + 63) / 64) * ((kn[1] + 63) / 64);
    B200ST_CHECK(splits == 1 || ((int64_t)splits * st.B * kn[1] <= lo.tickets - lo.partial && tiles <= kMaxTickets),
                 "wide decode: split-K scratch too small");
  }
  const size_t ss = self_smem(cf, st.max_len), cs = cross_smem(cf, st.Tm, beam);
  B200ST_CHECK(ss <= 200 * 1024 && cs <= 200 * 1024, "decode: too many keys for the shared-memory score buffer");
  return 0;
}

size_t rows_self_smem(const Config& c, int max_len) { return self_smem(c, max_len); }
size_t rows_cross_smem(const Config& c, int Tm, int beam) { return cross_smem(c, Tm, beam); }

int rows_raise_smem(size_t ss, size_t cs) {
  if (ss > 48 * 1024) B200ST_CUDA(cudaFuncSetAttribute(rows_self_attn_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)ss));
  if (cs > 48 * 1024) B200ST_CUDA(cudaFuncSetAttribute(rows_cross_attn_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)cs));
  return 0;
}

int rows_step(const Model& m, const Buffers& buf, const DecodeState& st, const int32_t* time_dev, float* logits, const int* anc,
              int beam, cudaStream_t s) {
  if (m.adt == F16) return rows_step_t(m, buf, st, reinterpret_cast<const __half*>(buf.shadow), time_dev, logits, anc, beam, s);
  return rows_step_t(m, buf, st, reinterpret_cast<const __nv_bfloat16*>(buf.shadow), time_dev, logits, anc, beam, s);
}

int rows_greedy_pick(const float* logits, int64_t* ids, int32_t* finished, int32_t* length, float* logprob, int64_t* out,
                     int32_t* time, int32_t* all_finished, uint32_t* ticket, int B, int V, int eos, int unk, int min_len,
                     int max_steps, cudaStream_t s) {
  return launch(rows_greedy_pick_kernel, B, 1024, 0, s, logits, ids, finished, length, logprob, out, time, all_finished, ticket, V, eos,
                unk, min_len, max_steps);
}

}  // namespace b200st
