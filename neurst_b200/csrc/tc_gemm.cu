// wgmma / TMA 16-bit GEMM for sm_90a.
//
// Persistent, warp-specialised kernel (one CTA per SM, 384 threads = 3 warpgroups):
//   warpgroup 0    : TMA producer (one thread: cp.async.bulk.tensor -> 128B-swizzled smem ring, mbarrier complete_tx);
//                    gives its registers to the consumers (setmaxnreg)
//   warpgroups 1, 2: consumers, 64 rows of the 128-row tile each: wgmma.mma_async from the smem ring into fp32 register
//                    accumulators (one k-block in flight behind the one being issued), then the fused epilogue straight
//                    from the accumulator fragments to global memory (plain stores, or fp32 atomics for split-K / accumulate)
// Tile: 128 x BN x 64 (BN in {64,128,256}); operands may be K-major or MN-major (wgrad / PV products),
// batched through 4-D tensor maps; optional split-K.  Every launch is a programmatic dependent launch (pdl.cuh).
//
// Replaces the cuBLAS calls behind tf.einsum / Dense / Conv2D at the reference sites listed in
// SURVEY.md §2.3 (K3,K4,K8,K9,K10,K11,K13,K15), e.g. neurst/layers/common_layers.py:270,276-288.
#include "gemm.cuh"
#include "pdl.cuh"
#include "ptx.cuh"

#include <mutex>
#include <unordered_map>
#include <vector>
#include <cstring>
#include <cstdlib>

namespace b200st {

namespace {

constexpr int BM = 128;
constexpr int BK = 64;                  // 64 bf16 = 128 B = one swizzle row
constexpr int kThreads = 384;           // producer warpgroup + 2 consumer warpgroups
constexpr int kConsumerWarps = 8;
constexpr int kSmemLimit = 232448;      // 227 KB
constexpr uint32_t kABytes = BM * BK * 2;
constexpr int kProducerRegs = 40, kConsumerRegs = 232;   // 128 * 40 + 256 * 232 = 384 * 168 registers

struct TcParams {
  int M, N, K;
  int nb1, nb2;
  int m_tiles, n_tiles, splitk, kb_total, kb_per_split;
  int64_t num_tiles;
  int stages;
  void* C;
  int c_dtype;
  int64_t ldc, c_sb1, c_sb2;
  GemmEpilogue epi;
  int atomic;           // C += through fp32 atomics (split-K or accumulate)
  int vec2;             // C may be written two columns at a time (even N, ld and batch strides; 8-byte aligned base)
  // implicit transposed-convolution A operand (conv2 data gradient, see gemm_conv2_dgrad): A tile = a [conv_tu x conv_v]
  // patch of positions x 64 channels of dY[B, T2, F2, C], shifted by the tap; k-block kb = (tap, 64-channel chunk)
  int conv;             // 0 = off
  int conv_ub;          // row tiles per utterance
  int conv_tu;          // time rows per tile
  int conv_kpc;         // k-blocks per tap (C / 64)
  int conv_dt[4], conv_df[4], conv_wrow[4];   // per tap: time / frequency shift into dY, first row of the tap in the weight matrix
  uint32_t conv_a_bytes;                      // bytes one A box delivers (64 ch x conv_v x conv_tu x 2)
};

struct TileCoord { int b2, b1, m_blk, n_blk, split; };

__device__ __forceinline__ TileCoord decode_tile(const TcParams& p, int64_t tile) {
  TileCoord t;
  t.split = (int)(tile % p.splitk); tile /= p.splitk;
  t.n_blk = (int)(tile % p.n_tiles); tile /= p.n_tiles;
  t.m_blk = (int)(tile % p.m_tiles); tile /= p.m_tiles;
  t.b1 = (int)(tile % p.nb1);
  t.b2 = (int)(tile / p.nb1);
  return t;
}

// The smem operand ring shared by the producer thread and the consumer warps: `full` barriers count the producer's
// expect_tx arrival, `empty` barriers one arrival per consumer warp.
struct Ring {
  uint32_t smem, bars, stage_bytes;
  int stages, stage;
  uint32_t phase;
  __device__ __forceinline__ uint32_t full() const { return bars + 8u * stage; }
  __device__ __forceinline__ uint32_t empty(int s) const { return bars + 8u * (stages + s); }
  __device__ __forceinline__ uint32_t slot() const { return smem + (uint32_t)stage * stage_bytes; }
  __device__ __forceinline__ void advance() { if (++stage == stages) { stage = 0; phase ^= 1u; } }
  __device__ __forceinline__ void init() const {
    for (int s = 0; s < stages; ++s) { ptx::mbar_init(bars + 8u * s, 1); ptx::mbar_init(empty(s), kConsumerWarps); }
  }
};

// Consumer warpgroup `wg`: acc[64 x BN] = sum over the next nkb ring slots of A_slot[64 wg .. 64 wg + 64, :] B_slot^T.
// The wgmma group of slot i stays in flight while slot i + 1 is issued; a slot is released once its group has retired.
template <int BN, bool A_MN, bool B_MN, bool BF>
__device__ __forceinline__ void consume_kblocks(float (&acc)[BN / 2], Ring& r, int nkb, int wg, int lane) {
  int prev = -1;
  for (int i = 0; i < nkb; ++i) {
    ptx::mbar_wait(r.full(), r.phase);
    const uint32_t sa = r.slot() + (uint32_t)wg * 8192u, sb = r.slot() + kABytes;
    ptx::fence_acc(acc);
    ptx::wgmma_fence();
#pragma unroll
    for (int k = 0; k < BK / 16; ++k)
      ptx::WgmmaSS<BN, BF, A_MN, B_MN>::mma(acc, A_MN ? ptx::desc_mnmajor(sa, k) : ptx::desc_kmajor(sa, k),
                                             B_MN ? ptx::desc_mnmajor(sb, k) : ptx::desc_kmajor(sb, k), (i > 0 || k > 0) ? 1 : 0);
    ptx::wgmma_commit();
    if (prev >= 0) {
      ptx::wgmma_wait<1>();
      if (lane == 0) ptx::mbar_arrive(r.empty(prev));
    }
    prev = r.stage;
    r.advance();
  }
  ptx::wgmma_wait<0>();
  ptx::fence_acc(acc);
  if (prev >= 0 && lane == 0) ptx::mbar_arrive(r.empty(prev));
}

// Fused epilogue of one accumulator pair (row m, columns n and n + 1): alpha / bias / relu / mask / dropout / residual as
// gemm_epilogue_value defines them, then a store or an fp32 atomic add.
__device__ __forceinline__ void epilogue_pair(const TcParams& p, float a0, float a1, int m, int n, int64_t bidx, int64_t boff_c,
                                              int64_t boff_mask, int64_t boff_res) {
  const uint64_t e_idx = (uint64_t)((bidx * p.M + m) * (int64_t)p.N + n);
  const bool two = n + 1 < p.N;
  const float v0 = gemm_epilogue_value(p.epi, a0, m, n, boff_mask, boff_res, e_idx);
  const float v1 = two ? gemm_epilogue_value(p.epi, a1, m, n + 1, boff_mask, boff_res, e_idx + 1) : 0.f;
  const int64_t idx = boff_c + (int64_t)m * p.ldc + n;
  if (p.atomic) {
    float* c = reinterpret_cast<float*>(p.C) + idx;
    if (p.vec2 && two) atomicAdd(reinterpret_cast<float2*>(c), make_float2(v0, v1));
    else { atomicAdd(c, v0); if (two) atomicAdd(c + 1, v1); }
  } else if (p.c_dtype == F32) {
    float* c = reinterpret_cast<float*>(p.C) + idx;
    if (p.vec2 && two) *reinterpret_cast<float2*>(c) = make_float2(v0, v1);
    else { c[0] = v0; if (two) c[1] = v1; }
  } else {
    if (p.vec2 && two) reinterpret_cast<uint32_t*>(p.C)[idx >> 1] = pack2_16(v0, v1, p.c_dtype);
    else { store_from_f32(p.C, p.c_dtype, idx, v0); if (two) store_from_f32(p.C, p.c_dtype, idx + 1, v1); }
  }
}

template <int BN, bool A_MN, bool B_MN, bool BF>
__global__ void __launch_bounds__(kThreads, 1)
tc_gemm_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, const TcParams p) {
  extern __shared__ uint8_t smem_raw[];
  constexpr uint32_t kBBytes = BN * BK * 2;
  constexpr uint32_t kStageBytes = kABytes + kBBytes;

  Ring ring;
  ring.smem = (ptx::smem_u32(smem_raw) + 1023u) & ~1023u;
  ring.stages = p.stages;
  ring.stage_bytes = kStageBytes;
  ring.bars = ring.smem + (uint32_t)p.stages * kStageBytes;
  ring.stage = 0; ring.phase = 0;

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;

  if (warp == 0 && lane == 0) {
    ptx::prefetch_tensormap(&tmA);
    ptx::prefetch_tensormap(&tmB);
    ring.init();
    ptx::fence_mbar_init();
  }
  __syncthreads();
  pdl_wait();      // everything above (barriers, descriptor prefetch) overlaps the previous kernel's tail
  pdl_trigger();

  if (warp < 4) {
    // ===================== TMA producer =====================
    ptx::reg_dealloc<kProducerRegs>();
    if (warp == 0 && lane == 0) {
      for (int64_t tile = blockIdx.x; tile < p.num_tiles; tile += gridDim.x) {
        const TileCoord t = decode_tile(p, tile);
        const int kb0 = t.split * p.kb_per_split;
        const int kb1 = min(p.kb_total, kb0 + p.kb_per_split);
        for (int kb = kb0; kb < kb1; ++kb) {
          ptx::mbar_wait(ring.empty(ring.stage), ring.phase ^ 1u);
          const uint32_t sa = ring.slot();
          const uint32_t sb = sa + kABytes;
          if constexpr (!A_MN && !B_MN) {
            if (p.conv) {
              const int tap = kb / p.conv_kpc, c0 = (kb - tap * p.conv_kpc) * BK;
              ptx::mbar_arrive_expect_tx(ring.full(), p.conv_a_bytes + kBBytes);
              ptx::tma_load_4d(sa, &tmA, ring.full(), c0, p.conv_df[tap], (t.m_blk % p.conv_ub) * p.conv_tu + p.conv_dt[tap],
                               t.m_blk / p.conv_ub);
              ptx::tma_load_4d(sb, &tmB, ring.full(), c0, p.conv_wrow[tap] + t.n_blk * BN, 0, 0);
              ring.advance();
              continue;
            }
          }
          ptx::mbar_arrive_expect_tx(ring.full(), kStageBytes);
          if (A_MN) {
#pragma unroll
            for (int c = 0; c < BM / 64; ++c)
              ptx::tma_load_4d(sa + c * (64 * BK * 2), &tmA, ring.full(), t.m_blk * BM + c * 64, kb * BK, t.b1, t.b2);
          } else {
            ptx::tma_load_4d(sa, &tmA, ring.full(), kb * BK, t.m_blk * BM, t.b1, t.b2);
          }
          if (B_MN) {
#pragma unroll
            for (int c = 0; c < BN / 64; ++c)
              ptx::tma_load_4d(sb + c * (64 * BK * 2), &tmB, ring.full(), t.n_blk * BN + c * 64, kb * BK, t.b1, t.b2);
          } else {
            ptx::tma_load_4d(sb, &tmB, ring.full(), kb * BK, t.n_blk * BN, t.b1, t.b2);
          }
          ring.advance();
        }
      }
    }
  } else {
    // ===================== consumer warpgroups =====================
    ptx::reg_alloc<kConsumerRegs>();
    const int wg = (warp >> 2) - 1, g = lane >> 2, q = lane & 3;
    const GemmEpilogue& ep = p.epi;
    float acc[BN / 2];
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
    for (int64_t tile = blockIdx.x; tile < p.num_tiles; tile += gridDim.x) {
      const TileCoord t = decode_tile(p, tile);
      const int kb0 = t.split * p.kb_per_split;
      const int kb1 = min(p.kb_total, kb0 + p.kb_per_split);
      consume_kblocks<BN, A_MN, B_MN, BF>(acc, ring, kb1 - kb0, wg, lane);
      const int m0 = t.m_blk * BM + wg * 64 + (warp & 3) * 16 + g;
      const int n0 = t.n_blk * BN + 2 * q;
      const int64_t bidx = (int64_t)t.b2 * p.nb1 + t.b1;
      const int64_t boff_c = (int64_t)t.b2 * p.c_sb2 + (int64_t)t.b1 * p.c_sb1;
      const int64_t boff_mask = (int64_t)t.b2 * ep.mask_sb2 + (int64_t)t.b1 * ep.mask_sb1;
      const int64_t boff_res = (int64_t)t.b2 * ep.res_sb2 + (int64_t)t.b1 * ep.res_sb1;
#pragma unroll
      for (int j = 0; j < BN / 8; ++j) {
        const int n = n0 + 8 * j;
        if (n < p.N) {
          if (m0 < p.M) epilogue_pair(p, acc[4 * j], acc[4 * j + 1], m0, n, bidx, boff_c, boff_mask, boff_res);
          if (m0 + 8 < p.M) epilogue_pair(p, acc[4 * j + 2], acc[4 * j + 3], m0 + 8, n, bidx, boff_c, boff_mask, boff_res);
        }
      }
    }
  }
}


// =============================================================================================================
// Grouped weight-gradient GEMM: up to kMaxGroup products  dW_g[K_in, N_out] += X_g^T dY_g  of one backward block in ONE
// persistent launch (TF autodiff of the Dense / einsum sites of a sublayer: neurst/layers/common_layers.py:270-288,
// multi_head_attention.py:145-215).  Each product alone has 2..16 output tiles and needs split-K over the B*T rows to fill
// the SMs, i.e. every CTA reduce-adds a full 128 x 256 fp32 tile for a handful of k-blocks of MMA work and every launch pays
// its fixed cost; together the products of a block give one wave of work units with k-ranges several times longer.
// Same pipeline as tc_gemm_kernel<256, true, true>; a work unit = (product, m tile, n tile, k split).
// =============================================================================================================
constexpr int kMaxGroup = 4;
struct TcGroupProb {
  CUtensorMap ta, tb;
  float* C;
  int64_t ldc;
  int m_tiles, n_tiles, splitk, kb_total, kb_per_split, tile_begin;
  float alpha;
  int pad_;
};
struct TcGroup {
  TcGroupProb prob[kMaxGroup];
  int n, num_tiles, stages;
};
struct GroupTile { int gi, m_blk, n_blk, kb0, kb1; };
__device__ __forceinline__ GroupTile group_tile(const TcGroup& g, int tile) {
  GroupTile t;
  t.gi = 0;
#pragma unroll
  for (int i = 1; i < kMaxGroup; ++i)
    if (i < g.n && tile >= g.prob[i].tile_begin) t.gi = i;
  const TcGroupProb& q = g.prob[t.gi];
  int local = tile - q.tile_begin;
  const int split = local % q.splitk; local /= q.splitk;
  t.n_blk = local % q.n_tiles;
  t.m_blk = local / q.n_tiles;
  t.kb0 = split * q.kb_per_split;
  t.kb1 = min(q.kb_total, t.kb0 + q.kb_per_split);
  return t;
}

template <bool BF>
__global__ void __launch_bounds__(kThreads, 1) tc_wgrad_group_kernel(const __grid_constant__ TcGroup grp) {
  extern __shared__ uint8_t smem_raw[];
  constexpr int BN = 256;
  constexpr uint32_t kBBytes = BN * BK * 2;
  constexpr uint32_t kStageBytes = kABytes + kBBytes;

  Ring ring;
  ring.smem = (ptx::smem_u32(smem_raw) + 1023u) & ~1023u;
  ring.stages = grp.stages;
  ring.stage_bytes = kStageBytes;
  ring.bars = ring.smem + (uint32_t)grp.stages * kStageBytes;
  ring.stage = 0; ring.phase = 0;

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  if (warp == 0 && lane == 0) {
    for (int i = 0; i < grp.n; ++i) {
      ptx::prefetch_tensormap(&grp.prob[i].ta);
      ptx::prefetch_tensormap(&grp.prob[i].tb);
    }
    ring.init();
    ptx::fence_mbar_init();
  }
  __syncthreads();
  pdl_wait();
  pdl_trigger();

  if (warp < 4) {
    ptx::reg_dealloc<kProducerRegs>();
    if (warp == 0 && lane == 0) {
      for (int tile = blockIdx.x; tile < grp.num_tiles; tile += gridDim.x) {
        const GroupTile t = group_tile(grp, tile);
        const CUtensorMap* ma = &grp.prob[t.gi].ta;
        const CUtensorMap* mb = &grp.prob[t.gi].tb;
        for (int kb = t.kb0; kb < t.kb1; ++kb) {
          ptx::mbar_wait(ring.empty(ring.stage), ring.phase ^ 1u);
          const uint32_t sa = ring.slot();
          const uint32_t sb = sa + kABytes;
          ptx::mbar_arrive_expect_tx(ring.full(), kStageBytes);
#pragma unroll
          for (int c = 0; c < BM / 64; ++c)
            ptx::tma_load_4d(sa + c * (64 * BK * 2), ma, ring.full(), t.m_blk * BM + c * 64, kb * BK, 0, 0);
#pragma unroll
          for (int c = 0; c < BN / 64; ++c)
            ptx::tma_load_4d(sb + c * (64 * BK * 2), mb, ring.full(), t.n_blk * BN + c * 64, kb * BK, 0, 0);
          ring.advance();
        }
      }
    }
  } else {
    ptx::reg_alloc<kConsumerRegs>();
    const int wg = (warp >> 2) - 1, g = lane >> 2, q = lane & 3;
    float acc[BN / 2];
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
    for (int tile = blockIdx.x; tile < grp.num_tiles; tile += gridDim.x) {
      const GroupTile t = group_tile(grp, tile);
      const float alpha = grp.prob[t.gi].alpha;
      consume_kblocks<BN, true, true, BF>(acc, ring, t.kb1 - t.kb0, wg, lane);
      // M % 128 == 0 and N % 256 == 0 (gemm_wgrad_group): no edge tiles
      float* c = grp.prob[t.gi].C + (int64_t)(t.m_blk * BM + wg * 64 + (warp & 3) * 16 + g) * grp.prob[t.gi].ldc + t.n_blk * BN + 2 * q;
      const int64_t row8 = 8 * grp.prob[t.gi].ldc;
#pragma unroll
      for (int j = 0; j < BN / 8; ++j) {
        atomicAdd(reinterpret_cast<float2*>(c + 8 * j), make_float2(acc[4 * j] * alpha, acc[4 * j + 1] * alpha));
        atomicAdd(reinterpret_cast<float2*>(c + row8 + 8 * j), make_float2(acc[4 * j + 2] * alpha, acc[4 * j + 3] * alpha));
      }
    }
  }
}


// =============================================================================================================
// Fused Transformer FFN forward (SURVEY K11):  x_out += dropout_post( dropout_ffn(relu(X W1 + b1)) W2 + b2 )
//   neurst/layers/common_layers.py:145-160 (TransformerFFN) inside the pre-norm wrapper (:73-85); X = LN(x_in) (16-bit),
//   x_out is pre-initialised with the residual x_in by the LayerNorm kernel.
// One CTA = (128-row tile, slice of the hidden dimension); each consumer warpgroup owns 64 of the rows.  The X tile
// (128 x D, D in {128, 256}) stays in shared memory; the hidden activations of a 128-column chunk are accumulated in
// registers (GEMM1), get bias, ReLU and dropout there, are written to HBM only because the backward pass needs them, and
// go, packed to 16 bits, straight back into the tensor cores as the register A operand of GEMM2, which accumulates the
// [64 x D] output rows in registers across all chunks.  Only the weights stream (L2 -> smem), and the [M, ffn] hidden
// tensor is never read back.  Slices of the hidden dimension reduce into x_out with fp32 atomics (dropout is a mask: linear).
//   warpgroup 0: TMA producer (X once, then per chunk the W1 stages and the W2 stages, in consumption order)
//   smem: X 64 KB | weight ring 3 x 32 KB
// =============================================================================================================
struct MlpParams {
  int M, d, ffn;
  int chunks_per_cta;          // 128-column hidden chunks per CTA
  int splits;                  // hidden slices (gridDim.x = m_tiles * splits)
  const float* b1; const float* b2;
  DropoutSpec drop_ffn, drop_post;
  // backward (dgrad chain) variant: hidden epilogue = alpha * acc masked by (mask_src > 0), no bias / ReLU / dropout bits
  int relu;
  float alpha;
  const void* mask_src; int64_t mask_ld;
  uint16_t* F1;                // [M, ffn] hidden activations (forward) / hidden gradient (backward), 16-bit
  float* out;                  // [M, d] fp32, added into
  int* tickets;                // deterministic mode: [m_tiles] zero-initialised; slice s adds after slices < s (self-resetting)
};
constexpr int kMlpStages = 3;
constexpr uint32_t kMlpStageBytes = 32768;
constexpr uint32_t kMlpXBytes = 65536;
constexpr size_t kMlpSmem = 1024 + kMlpXBytes + kMlpStages * kMlpStageBytes + 256;

// B_MN: weights as MN-major B operands (forward: W1 [d, ffn], W2 [ffn, d] in the TF [in, out] layout) or K-major (backward:
// the same arrays read transposed: G1 uses W2 rows = hidden units, G2 uses W1 rows = model dims)
template <int DT, bool B_MN, int D>
__global__ void __launch_bounds__(kThreads, 1)
fused_mlp_fwd_kernel(const __grid_constant__ CUtensorMap tmX, const __grid_constant__ CUtensorMap tmW1,
                     const __grid_constant__ CUtensorMap tmW2, const MlpParams p) {
  extern __shared__ uint8_t smem_raw[];
  constexpr bool BF = DT == BF16;
  constexpr int kbx = D / BK;                  // k-blocks of GEMM1
  const uint32_t base = (ptx::smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t sX = base;
  const uint32_t sW = sX + kMlpXBytes;
  const uint32_t bars = sW + kMlpStages * kMlpStageBytes;
  const uint32_t x_full = bars;
  auto w_full = [&](int s2) { return bars + 8u * (1 + s2); };
  auto w_empty = [&](int s2) { return bars + 8u * (1 + kMlpStages + s2); };

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int m_blk = blockIdx.x / p.splits, split = blockIdx.x % p.splits;
  const int C = p.chunks_per_cta;
  const int chunk0 = split * C;

  if (warp == 0 && lane == 0) {
    ptx::prefetch_tensormap(&tmX); ptx::prefetch_tensormap(&tmW1); ptx::prefetch_tensormap(&tmW2);
    ptx::mbar_init(x_full, 1);
    for (int s2 = 0; s2 < kMlpStages; ++s2) { ptx::mbar_init(w_full(s2), 1); ptx::mbar_init(w_empty(s2), kConsumerWarps); }
    ptx::fence_mbar_init();
  }
  __syncthreads();
  pdl_wait();
  pdl_trigger();

  if (warp < 4) {
    ptx::reg_dealloc<kProducerRegs>();
    if (warp == 0 && lane == 0) {
      ptx::mbar_arrive_expect_tx(x_full, (uint32_t)kbx * kABytes);
      for (int kb = 0; kb < kbx; ++kb) ptx::tma_load_4d(sX + kb * kABytes, &tmX, x_full, kb * BK, m_blk * BM, 0, 0);
      int it = 0;
      auto stage_wait = [&](int& st, uint32_t& dst) {
        st = it % kMlpStages;
        ptx::mbar_wait(w_empty(st), (((uint32_t)(it / kMlpStages)) & 1u) ^ 1u);
        dst = sW + st * kMlpStageBytes;
        ++it;
      };
      for (int c = 0; c < C; ++c) {
        // GEMM1 B operand of chunk c: [K = d rows, N = 128 cols] as 2 k-blocks per stage
        const int n0 = (chunk0 + c) * 128;
        for (int s2 = 0; s2 < kbx; s2 += 2) {
          int st; uint32_t dst;
          stage_wait(st, dst);
          ptx::mbar_arrive_expect_tx(w_full(st), 2u * 16384u);
          for (int j = 0; j < 2; ++j) {
            if (B_MN) {
              for (int i = 0; i < 2; ++i)
                ptx::tma_load_4d(dst + j * 16384 + i * 8192, &tmW1, w_full(st), n0 + i * 64, (s2 + j) * BK, 0, 0);
            } else {
              ptx::tma_load_4d(dst + j * 16384, &tmW1, w_full(st), (s2 + j) * BK, n0, 0, 0);      // [128 rows x 64 k]
            }
          }
        }
        // GEMM2 B operand of chunk c: [K = 128 hidden rows, N = d cols], one k-block per stage
        for (int kb = 0; kb < 2; ++kb) {
          int st; uint32_t dst;
          stage_wait(st, dst);
          ptx::mbar_arrive_expect_tx(w_full(st), (uint32_t)(D / 64) * 8192u);
          if (B_MN) {
            for (int i = 0; i < D / 64; ++i)
              ptx::tma_load_4d(dst + i * 8192, &tmW2, w_full(st), i * 64, n0 + kb * BK, 0, 0);
          } else {
            ptx::tma_load_4d(dst, &tmW2, w_full(st), n0 + kb * BK, 0, 0, 0);                        // [d rows x 64 k]
          }
        }
      }
    }
  } else {
    ptx::reg_alloc<kConsumerRegs>();
    const int wg = (warp >> 2) - 1, g = lane >> 2, q = lane & 3;
    const int m0 = m_blk * BM + wg * 64 + (warp & 3) * 16 + g;       // this thread's rows: m0 and m0 + 8
    const bool use_bits = p.drop_ffn.p > 0.f;
    const float dscale = use_bits ? p.drop_ffn.scale : 1.f;
    const float hidden_floor = p.relu ? 0.f : -INFINITY;
    int it = 0;
    auto stage_get = [&](uint32_t& src) {
      const int st = it % kMlpStages;
      ptx::mbar_wait(w_full(st), ((uint32_t)(it / kMlpStages)) & 1u);
      src = sW + st * kMlpStageBytes;
      ++it;
      return st;
    };
    float out[D / 2];
#pragma unroll
    for (int i = 0; i < D / 2; ++i) out[i] = 0.f;
    ptx::mbar_wait(x_full, 0);
    for (int c = 0; c < C; ++c) {
      // The 128 hidden columns of chunk c go through the registers as two halves of 64 (GEMM1 half, epilogue, GEMM2 k-block),
      // so that the [64 x D] output accumulator and the hidden fragments fit the register file; the W1 stages are read by
      // both halves and released after the second.
      uint32_t w1src[kbx / 2];
      int w1st[kbx / 2];
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        // ---- GEMM1: hidden accumulator [64 x 64] ----
        float hid[32];
#pragma unroll
        for (int i = 0; i < 32; ++i) hid[i] = 0.f;
        if (h == 0) {
#pragma unroll
          for (int s2 = 0; s2 < kbx / 2; ++s2) w1st[s2] = stage_get(w1src[s2]);
        }
        ptx::fence_acc(hid);
        ptx::wgmma_fence();
#pragma unroll
        for (int kb = 0; kb < kbx; ++kb) {
          const uint32_t sa = sX + (uint32_t)kb * kABytes + (uint32_t)wg * 8192u;
          const uint32_t sb = w1src[kb >> 1] + (uint32_t)(kb & 1) * 16384u + (uint32_t)h * 8192u;
#pragma unroll
          for (int k = 0; k < BK / 16; ++k)
            ptx::WgmmaSS<64, BF, 0, B_MN>::mma(hid, ptx::desc_kmajor(sa, k), B_MN ? ptx::desc_mnmajor(sb, k) : ptx::desc_kmajor(sb, k),
                                               (kb > 0 || k > 0) ? 1 : 0);
        }
        ptx::wgmma_commit();
        ptx::wgmma_wait<0>();
        ptx::fence_acc(hid);
        if (h == 1 && lane == 0) {
#pragma unroll
          for (int s2 = 0; s2 < kbx / 2; ++s2) ptx::mbar_arrive(w_empty(w1st[s2]));
        }
        // ---- hidden epilogue on the fragments: bias, ReLU, dropout (forward) / relu'-dropout' mask (backward); store; pack ----
        const int n0 = (chunk0 + c) * 128 + h * 64 + 2 * q;
        uint32_t a16[4][4];
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const int n = n0 + 8 * j;
          float2 bb = make_float2(0.f, 0.f);
          if (p.b1) bb = __ldg(reinterpret_cast<const float2*>(p.b1 + n));
#pragma unroll
          for (int hr = 0; hr < 2; ++hr) {
            const int m = m0 + 8 * hr;
            const bool row_ok = m < p.M;
            float v0 = fmaxf(fmaf(hid[4 * j + 2 * hr], p.alpha, bb.x), hidden_floor);
            float v1 = fmaxf(fmaf(hid[4 * j + 2 * hr + 1], p.alpha, bb.y), hidden_floor);
            if (use_bits && row_ok) {
              const uint32_t kb = (uint32_t)__ldg(p.drop_ffn.bits + ((uint64_t)((int64_t)m * p.ffn + n) >> 3)) >> (2 * q);
              v0 = (kb & 1u) ? v0 * dscale : 0.f;
              v1 = (kb & 2u) ? v1 * dscale : 0.f;
            }
            if (!B_MN && p.mask_src && row_ok) {
              // 16-bit mask source (bf16 / fp16): "> 0" <=> sign clear and magnitude bits non-zero
              const uint32_t w = __ldg(reinterpret_cast<const uint32_t*>(reinterpret_cast<const uint16_t*>(p.mask_src) + (int64_t)m * p.mask_ld + n));
              const uint32_t lo = w & 0xffffu, hi = w >> 16;
              if (!(lo != 0u && lo < 0x8000u)) v0 = 0.f;
              if (!(hi != 0u && hi < 0x8000u)) v1 = 0.f;
            }
            const uint32_t pk = pack2_16(v0, v1, DT);
            if (row_ok) *reinterpret_cast<uint32_t*>(p.F1 + (int64_t)m * p.ffn + n) = pk;
            a16[j >> 1][(j & 1) * 2 + hr] = pk;
          }
        }
        // ---- GEMM2: out[64 x D] += hidden half (registers) x the matching 64 rows of the W2 chunk ----
        uint32_t src;
        const int st = stage_get(src);
        ptx::fence_acc(out);
        ptx::wgmma_fence();
#pragma unroll
        for (int k = 0; k < BK / 16; ++k)
          ptx::WgmmaRS<D, BF, B_MN>::mma(out, a16[k], B_MN ? ptx::desc_mnmajor(src, k) : ptx::desc_kmajor(src, k),
                                         (c > 0 || h > 0 || k > 0) ? 1 : 0);
        ptx::wgmma_commit();
        ptx::wgmma_wait<0>();
        ptx::fence_acc(out);
        if (lane == 0) ptx::mbar_arrive(w_empty(st));
      }
    }
    // ---- output rows: (+ b2 on slice 0) -> post dropout -> fp32 add into x_out ----
    const bool add_b2 = split == 0 && p.b2 != nullptr;
    const bool post = p.drop_post.p > 0.f;
    const float pscale = post ? p.drop_post.scale : 1.f;
    if (p.tickets && p.splits > 1) {
      // deterministic reduction order: slice s adds only after slices 0 .. s-1 of this row tile have completed theirs
      if (lane == 0) {
        const volatile int* tk = p.tickets + m_blk;
        while (*tk != split) { }
        __threadfence();
      }
      __syncwarp();
    }
#pragma unroll
    for (int j = 0; j < D / 8; ++j) {
      const int n = 8 * j + 2 * q;
      float2 bb = make_float2(0.f, 0.f);
      if (add_b2) bb = __ldg(reinterpret_cast<const float2*>(p.b2 + n));
#pragma unroll
      for (int hr = 0; hr < 2; ++hr) {
        const int m = m0 + 8 * hr;
        if (m < p.M) {
          float v0 = out[4 * j + 2 * hr] + bb.x, v1 = out[4 * j + 2 * hr + 1] + bb.y;
          if (post) {
            const uint32_t kb = (uint32_t)__ldg(p.drop_post.bits + ((uint64_t)((int64_t)m * p.d + n) >> 3)) >> (2 * q);
            v0 = (kb & 1u) ? v0 * pscale : 0.f;
            v1 = (kb & 2u) ? v1 * pscale : 0.f;
          }
          atomicAdd(reinterpret_cast<float2*>(p.out + (int64_t)m * p.d + n), make_float2(v0, v1));
        }
      }
    }
    if (p.tickets && p.splits > 1) {
      __threadfence();
      asm volatile("bar.sync 1, 256;" ::: "memory");      // all 8 warps' additions have been performed
      if (threadIdx.x == 128) atomicExch(p.tickets + m_blk, split + 1 == p.splits ? 0 : split + 1);
    }
  }
}

// -------------------------------------------------------------------------------------------
// Host side: tensor-map construction (driver entry point fetched at run time; no libcuda link)
// -------------------------------------------------------------------------------------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

EncodeTiledFn get_encode_fn() {
  static EncodeTiledFn fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(p);
  });
  return fn;
}

struct MapKey {
  uint64_t v[10];
  bool operator==(const MapKey& o) const { return std::memcmp(v, o.v, sizeof(v)) == 0; }
};
struct MapKeyHash {
  size_t operator()(const MapKey& k) const {
    uint64_t h = 1469598103934665603ull;
    for (uint64_t x : k.v) { h ^= x; h *= 1099511628211ull; }
    return (size_t)h;
  }
};
std::mutex g_map_mu;
std::unordered_map<MapKey, CUtensorMap, MapKeyHash> g_map_cache;

// Operand tensor map: dims (inner, outer, nb1, nb2); inner = K (K-major) or M/N (MN-major).
int make_operand_map(const GemmOperand& op, int rows, int K, int nb1, int nb2, int box_rows_kmajor, CUtensorMap* out) {
  EncodeTiledFn fn = get_encode_fn();
  B200ST_CHECK(fn != nullptr, "cuTensorMapEncodeTiled unavailable (no CUDA driver?)");
  const uint64_t es = 2;
  uint64_t inner = op.mn_major ? (uint64_t)rows : (uint64_t)K;
  uint64_t outer = op.mn_major ? (uint64_t)K : (uint64_t)rows;
  uint64_t sb1 = nb1 > 1 ? (uint64_t)op.sb1 : (uint64_t)op.ld * outer;
  uint64_t sb2 = nb2 > 1 ? (uint64_t)op.sb2 : sb1 * (uint64_t)nb1;
  if (sb1 == 0) sb1 = (uint64_t)op.ld * outer;   // broadcast batch strides are not used by callers of the TC path
  if (sb2 == 0) sb2 = sb1 * (uint64_t)nb1;
  cuuint64_t dims[4] = {inner, outer, (cuuint64_t)nb1, (cuuint64_t)nb2};
  cuuint64_t strides[3] = {(cuuint64_t)op.ld * es, sb1 * es, sb2 * es};
  cuuint32_t box[4] = {64u, (cuuint32_t)(op.mn_major ? BK : box_rows_kmajor), 1u, 1u};
  cuuint32_t estr[4] = {1u, 1u, 1u, 1u};
  B200ST_CHECK((reinterpret_cast<uintptr_t>(op.ptr) & 15) == 0, "TMA operand base must be 16-byte aligned");
  B200ST_CHECK(strides[0] % 16 == 0 && strides[1] % 16 == 0 && strides[2] % 16 == 0,
               "TMA operand strides must be multiples of 16 bytes (ld % 8 == 0 for bf16)");
  MapKey key{{(uint64_t)(uintptr_t)op.ptr, inner, outer, (uint64_t)nb1, (uint64_t)nb2, strides[0], strides[1], strides[2],
              box[1], (uint64_t)op.mn_major | ((uint64_t)op.dtype << 8)}};
  {
    std::lock_guard<std::mutex> lk(g_map_mu);
    auto it = g_map_cache.find(key);
    if (it != g_map_cache.end()) { *out = it->second; return 0; }
  }
  CUresult r = fn(out, op.dtype == F16 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4,
                  const_cast<void*>(op.ptr), dims, strides, box, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) B200ST_FAIL("cuTensorMapEncodeTiled failed with CUresult " + std::to_string((int)r));
  std::lock_guard<std::mutex> lk(g_map_mu);
  if (g_map_cache.size() > 65536) g_map_cache.clear();
  g_map_cache.emplace(key, *out);
  return 0;
}

int g_num_sms = 0;
int64_t g_launches = 0;
}  // namespace

// 16-bit 4-D tensor map (inner, rows, nb1, nb2) with a {box_inner<=64, box_rows} box, 128B swizzle.
int make_tma_map_16(const void* ptr, int dtype, uint64_t inner, uint64_t rows, int nb1, int nb2, int64_t ld, int64_t sb1, int64_t sb2,
                    uint32_t box_rows, CUtensorMap* out) {
  GemmOperand op{ptr, dtype, 0, ld, sb1, sb2};
  return make_operand_map(op, (int)rows, (int)inner, nb1, nb2, (int)box_rows, out);
}
void tc_count_launch() { ++g_launches; }

namespace {

// optional GEMM profile (bench.py roofline pass; off in the timed region): every tensor-core GEMM issued between begin and
// end is RECORDED (arguments only); tc_profile_end() then replays each recorded GEMM back to back (1 warm-up + kReps timed
// launches bracketed by one event pair, no host gap between them) and reports the per-launch average.  The buffers of the
// step are still alive (same workspace), accumulate / reduce epilogues only add into gradients nobody reads afterwards.
// conv2 data gradient as an implicit GEMM (see conv2_dgrad_implicit): replaces the A tensor map and the k-block -> coordinates rule
struct ConvA {
  const void* dy; int B, T2, F2, C;     // dY [B, T2, F2, C]
  int tu, ub, ntaps;
  int dt[4], df[4], wrow[4];
};
struct ProfRec { GemmArgs g; cudaStream_t stream; int bn, splitk; int group_n = 0; GemmArgs rest[3]; bool has_conv = false; ConvA conv; };   // group_n > 1: grouped weight-gradient launch (g + rest)
bool g_prof = false;
std::vector<ProfRec> g_prof_recs;

template <int BN, bool A_MN, bool B_MN, bool BF>
int launch_kernel(const CUtensorMap& ta, const CUtensorMap& tb, const TcParams& p, int grid, size_t smem, cudaStream_t stream) {
  auto kern = tc_gemm_kernel<BN, A_MN, B_MN, BF>;
  static bool attr_set = false;
  if (!attr_set) {
    B200ST_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemLimit));
    attr_set = true;
  }
  launch_pdl(kern, grid, kThreads, smem, stream, ta, tb, p);
  B200ST_LAUNCH_CHECK();
  return 0;
}

template <int BN, bool A_MN, bool B_MN>
int launch_variant(bool bf, const CUtensorMap& ta, const CUtensorMap& tb, const TcParams& p, int grid, size_t smem, cudaStream_t stream) {
  if (bf) return launch_kernel<BN, A_MN, B_MN, true>(ta, tb, p, grid, smem, stream);
  return launch_kernel<BN, A_MN, B_MN, false>(ta, tb, p, grid, smem, stream);
}

template <int BN>
int launch_bn(bool a_mn, bool b_mn, bool bf, const CUtensorMap& ta, const CUtensorMap& tb, const TcParams& p, int grid, size_t smem,
              cudaStream_t stream) {
  if (!a_mn && !b_mn) return launch_variant<BN, false, false>(bf, ta, tb, p, grid, smem, stream);
  if (!a_mn && b_mn) return launch_variant<BN, false, true>(bf, ta, tb, p, grid, smem, stream);
  if (a_mn && !b_mn) return launch_variant<BN, true, false>(bf, ta, tb, p, grid, smem, stream);
  return launch_variant<BN, true, true>(bf, ta, tb, p, grid, smem, stream);
}

}  // namespace

TcDebug& tc_debug() {
  static TcDebug d{};
  return d;
}
int64_t tc_launch_count() { return g_launches; }

namespace {
int gemm_tc_impl(const GemmArgs& g, cudaStream_t stream, const ConvA* conv);
}  // namespace
int gemm_tc_bf16(const GemmArgs& g, cudaStream_t stream) { return gemm_tc_impl(g, stream, nullptr); }

namespace {
int gemm_tc_impl(const GemmArgs& g, cudaStream_t stream, const ConvA* conv) {
  B200ST_CHECK(is16(g.A.dtype) && is16(g.B.dtype), "tensor-core GEMM needs 16-bit (bf16 / fp16) operands");
  // wgmma has no mixed bf16 x fp16 form: the library refuses mixed products up front
  B200ST_CHECK(g.A.dtype == g.B.dtype, "wgmma needs A and B in the same 16-bit format (both bf16 or both fp16)");
  B200ST_CHECK(g.M > 0 && g.N > 0 && g.K > 0 && g.nb1 > 0 && g.nb2 > 0, "empty GEMM");
  if (const int abl = ablate_mask()) {
    const bool wgrad = g.A.mn_major && g.B.mn_major;
    if ((wgrad && (abl & ABL_WGRAD)) || (!wgrad && (abl & ABL_GEMM))) return 0;
  }
  if (g_num_sms == 0) {
    int dev = 0;
    B200ST_CUDA(cudaGetDevice(&dev));
    B200ST_CUDA(cudaDeviceGetAttribute(&g_num_sms, cudaDevAttrMultiProcessorCount, dev));
  }
  const TcDebug& dbg = tc_debug();
  const int num_sms = dbg.max_ctas > 0 ? dbg.max_ctas : (dbg.reserve_sms > 0 && dbg.reserve_sms < g_num_sms ? g_num_sms - dbg.reserve_sms : g_num_sms);

  TcParams p{};
  p.M = g.M; p.N = g.N; p.K = g.K; p.nb1 = g.nb1; p.nb2 = g.nb2;
  p.m_tiles = ceil_div(g.M, BM);
  p.kb_total = ceil_div(g.K, BK);
  const int64_t batch = (int64_t)g.nb1 * g.nb2;

  // ---- joint choice of the N tile and the split-K factor ----
  // Cost model per k-block of a CTA: max(tensor time, L2->smem fill time): the wgmmas of a 128 x c x 64 block take about
  // 4c cycles, the operand bytes (16 KB + 128c B) are assumed to arrive at ~44 B/cycle/SM (an estimate, not measured on
  // H100).  The epilogue runs after the main loop of its tile.  Split-K (fp32 atomic epilogue) is allowed for linear
  // accumulate epilogues only and is chosen so that the tile count fills the SMs once.
  const bool linear_epi = !g.epi.relu && !g.epi.mask_src && g.epi.drop.p == 0.f && !g.epi.residual && !g.epi.bias;
  const bool split_ok = linear_epi && g.c_dtype == F32 && g.epi.accumulate;
  if (g.splitk > 1) B200ST_CHECK(split_ok, "split-K needs a linear fp32 accumulate epilogue");
  int bn = dbg.force_bn, splitk = g.splitk >= 1 ? g.splitk : 1;
  {
    double best = 1e30;
    int best_bn = 0, best_sk = 1;
    const int cands[3] = {256, 128, 64};
    for (int c : cands) {
      if (dbg.force_bn && c != dbg.force_bn) continue;
      if (conv && c != 256) continue;
      if (!dbg.force_bn && c > 64 && c >= 2 * ((g.N + 63) / 64 * 64)) continue;   // do not pad N by 2x or more
      const int64_t tiles0 = batch * p.m_tiles * ceil_div(g.N, c);
      int sk_lo = splitk, sk_hi = splitk;
      if (g.splitk == 0 && split_ok) {
        sk_lo = 1;
        sk_hi = (int)(num_sms / tiles0);
        const int cap = p.kb_total / 4 > 0 ? p.kb_total / 4 : 1;
        if (sk_hi > cap) sk_hi = cap;
        if (sk_hi < 1) sk_hi = 1;
      }
      for (int sk = sk_hi; sk >= sk_lo; sk = (sk > sk_lo && sk > 1) ? (sk == sk_hi && sk_hi > 2 ? sk / 2 : sk - 1) : sk_lo - 1) {
        const int kb_per = ceil_div(p.kb_total, sk);
        const int64_t tiles = tiles0 * ceil_div(p.kb_total, kb_per);
        const int64_t waves = (tiles + num_sms - 1) / num_sms;
        const double fill = (16384.0 + 128.0 * c) / 44.0, mma = 4.0 * c;
        const double mainloop = kb_per * (fill > mma ? fill : mma);
        const double epi = (sk > 1 ? 14.0 : 10.0) * c + 600.0;
        const double cost = (double)waves * (mainloop + epi + 800.0) + (sk > 1 ? 500.0 : 0.0);
        if (cost < best) { best = cost; best_bn = c; best_sk = sk; }
        if (sk <= sk_lo) break;
      }
    }
    bn = best_bn;
    splitk = best_sk;
  }
  if (splitk > p.kb_total) splitk = p.kb_total;
  p.kb_per_split = ceil_div(p.kb_total, splitk);
  splitk = ceil_div(p.kb_total, p.kb_per_split);   // no empty trailing split
  p.splitk = splitk;
  p.n_tiles = ceil_div(g.N, bn);
  p.num_tiles = batch * p.m_tiles * p.n_tiles * splitk;

  const uint32_t stage_bytes = kABytes + (uint32_t)bn * BK * 2;
  int stages = dbg.force_stages > 0 ? dbg.force_stages : (int)((kSmemLimit - 2048) / stage_bytes);
  if (stages > 8) stages = 8;
  if (stages < 2) stages = 2;      // consume_kblocks keeps one slot in flight before it releases the previous one
  p.stages = stages;
  const size_t smem = 1024 + (size_t)stages * stage_bytes + 16 * stages + 16;
  B200ST_CHECK(smem <= (size_t)kSmemLimit, "smem budget exceeded");

  p.C = g.C; p.c_dtype = g.c_dtype; p.ldc = g.ldc; p.c_sb1 = g.c_sb1; p.c_sb2 = g.c_sb2;
  p.epi = g.epi;
  if (g.epi.accumulate) B200ST_CHECK(g.c_dtype == F32, "accumulate needs fp32 C");
  p.atomic = (splitk > 1 || g.epi.accumulate) ? 1 : 0;
  // paired stores / atomics need every (row, even column) element of C 8-byte (fp32) or 4-byte (16-bit) aligned
  const uintptr_t pair_bytes = g.c_dtype == F32 ? 8 : 4;
  p.vec2 = ((reinterpret_cast<uintptr_t>(g.C) % pair_bytes) == 0 && g.ldc % 2 == 0 && (g.nb1 == 1 || g.c_sb1 % 2 == 0) &&
            (g.nb2 == 1 || g.c_sb2 % 2 == 0)) ? 1 : 0;

  CUtensorMap ta, tb;
  if (conv) {
    B200ST_CHECK(bn == 256 && splitk == 1 && !g.A.mn_major && !g.B.mn_major && g.nb1 == 1 && g.nb2 == 1 && conv->C % BK == 0 &&
                     g.K == conv->ntaps * conv->C && g.M == conv->B * conv->ub * BM && conv->F2 * conv->tu <= BM && conv->ntaps <= 4,
                 "implicit conv dgrad: unsupported shape");
    p.conv = 1; p.conv_ub = conv->ub; p.conv_tu = conv->tu; p.conv_kpc = conv->C / BK;
    for (int i = 0; i < conv->ntaps; ++i) { p.conv_dt[i] = conv->dt[i]; p.conv_df[i] = conv->df[i]; p.conv_wrow[i] = conv->wrow[i]; }
    p.conv_a_bytes = (uint32_t)(BK * conv->F2 * conv->tu * 2);
    // A: dY as a 4-D tensor (C, F2, T2, B); one box = 64 channels x all F2 frequencies x tu time rows of one utterance — rows
    // beyond the tensor (the shifted taps at the far edge) are zero-filled by the TMA unit, i.e. the convolution's border
    EncodeTiledFn fn = get_encode_fn();
    B200ST_CHECK(fn != nullptr, "cuTensorMapEncodeTiled unavailable (no CUDA driver?)");
    B200ST_CHECK((reinterpret_cast<uintptr_t>(conv->dy) & 15) == 0, "TMA operand base must be 16-byte aligned");
    cuuint64_t dims[4] = {(cuuint64_t)conv->C, (cuuint64_t)conv->F2, (cuuint64_t)conv->T2, (cuuint64_t)conv->B};
    cuuint64_t strides[3] = {(cuuint64_t)conv->C * 2, (cuuint64_t)conv->F2 * conv->C * 2, (cuuint64_t)conv->T2 * conv->F2 * conv->C * 2};
    cuuint32_t box[4] = {(cuuint32_t)BK, (cuuint32_t)conv->F2, (cuuint32_t)conv->tu, 1u};
    cuuint32_t estr[4] = {1u, 1u, 1u, 1u};
    CUresult r = fn(&ta, g.A.dtype == F16 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, const_cast<void*>(conv->dy),
                    dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                    CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) B200ST_FAIL("cuTensorMapEncodeTiled (conv dY) failed with CUresult " + std::to_string((int)r));
    B200ST_TRY(make_operand_map(g.B, 9 * conv->C, conv->C, 1, 1, bn, &tb));      // all 9 taps of the [9C, C] weight matrix
  } else {
    B200ST_TRY(make_operand_map(g.A, g.M, g.K, g.nb1, g.nb2, BM, &ta));
    B200ST_TRY(make_operand_map(g.B, g.N, g.K, g.nb1, g.nb2, bn, &tb));
  }

  const int max_grid = num_sms;
  const int grid = (int)(p.num_tiles < max_grid ? p.num_tiles : max_grid);
  ++g_launches;
  if (g_prof) {
    ProfRec r{g, stream, bn, splitk};
    if (conv) { r.has_conv = true; r.conv = *conv; }
    g_prof_recs.push_back(r);
  }
  int rc = 0;
  const bool bf = g.A.dtype == BF16;
  switch (bn) {
    case 64: rc = launch_bn<64>(g.A.mn_major, g.B.mn_major, bf, ta, tb, p, grid, smem, stream); break;
    case 128: rc = launch_bn<128>(g.A.mn_major, g.B.mn_major, bf, ta, tb, p, grid, smem, stream); break;
    case 256: rc = launch_bn<256>(g.A.mn_major, g.B.mn_major, bf, ta, tb, p, grid, smem, stream); break;
    default: B200ST_FAIL("unsupported BN");
  }
  return rc;
}
}  // namespace

// Data gradient of the 3x3 / stride-2 / pad-1 convolution (Conv2D#2 of AudioConv2dSubsamplingLayer,
// neurst/layers/modalities/audio_modalities.py:96-104) as four implicit GEMMs, one per parity class (t1 & 1, f1 & 1) of the
// input position: dA[b, t1, f1, :] = sum over the taps (kh, kw) with t1 = 2 t2 + kh - 1, f1 = 2 f2 + kw - 1 of
// dY[b, t2, f2, :] W[kh, kw]^T — 1 tap for (even, even), 2 for the mixed classes, 4 for (odd, odd).  The A operand is read
// straight out of dY by 4-D TMA boxes shifted by the tap (zero fill = border), so neither the [rows, 9C] column gradient
// (737 MB at cfg-2) nor its col2im gather exist.  Output: class-major padded tiles
//   dA[cls][b][tile][128 rows = tu x F2 positions (+ unused rows)][C],   tile = (t1 >> 1) / tu,   row = ((t1 >> 1) % tu) * F2 + (f1 >> 1)
// which conv1's backward kernel reads back with the same arithmetic.
int conv2_dgrad_implicit(const void* dy, const void* w16, void* da, int dtype, int B, int T2, int F2, int C, cudaStream_t stream) {
  B200ST_CHECK(is16(dtype) && C == 256 && F2 >= 1 && F2 <= BM, "implicit conv2 dgrad: 16-bit, C == 256, F2 <= 128");
  ConvA ca{};
  ca.dy = dy; ca.B = B; ca.T2 = T2; ca.F2 = F2; ca.C = C;
  ca.tu = BM / F2;
  ca.ub = ceil_div(T2, ca.tu);
  const int64_t cls_elems = (int64_t)B * ca.ub * BM * C;
  for (int cls = 0; cls < 4; ++cls) {
    const int pt = cls >> 1, pf = cls & 1;
    // per axis: even position -> centre tap, same index; odd position -> tap 2 at the same index and tap 0 at index + 1
    const int nt = pt ? 2 : 1, nf = pf ? 2 : 1;
    const int kh_of[2] = {pt ? 2 : 1, 0}, dt_of[2] = {0, 1};
    const int kw_of[2] = {pf ? 2 : 1, 0}, df_of[2] = {0, 1};
    ca.ntaps = nt * nf;
    for (int a = 0; a < nt; ++a)
      for (int b2 = 0; b2 < nf; ++b2) {
        const int i = a * nf + b2;
        ca.dt[i] = dt_of[a]; ca.df[i] = df_of[b2]; ca.wrow[i] = (kh_of[a] * 3 + kw_of[b2]) * C;
      }
    GemmArgs g = gemm_defaults();
    g.M = B * ca.ub * BM; g.N = C; g.K = ca.ntaps * C;
    g.A = GemmOperand{dy, dtype, 0, C, 0, 0};
    g.B = GemmOperand{w16, dtype, 0, C, 0, 0};
    g.C = reinterpret_cast<char*>(da) + (size_t)cls * cls_elems * 2; g.c_dtype = dtype; g.ldc = C;
    B200ST_TRY(gemm_tc_impl(g, stream, &ca));
  }
  return 0;
}
int64_t conv2_dgrad_implicit_elems(int B, int T2, int F2, int C) {
  const int tu = BM / F2;
  return 4 * (int64_t)B * ceil_div(T2, tu) * BM * C;
}


// One launch for the weight gradients of a backward block (see tc_wgrad_group_kernel).  Every product must be a plain
// fp32-accumulate MN-major x MN-major 16-bit GEMM with M % 128 == 0 and N % 256 == 0; returns 2 (nothing launched) when the
// group does not qualify, so that the caller issues the products one by one.
int gemm_wgrad_group(const GemmArgs* gs, int n, cudaStream_t stream) {
  if (n < 2 || n > kMaxGroup || getenv("B200ST_NO_GROUPED_WGRAD")) return 2;
  for (int i = 0; i < n; ++i) {
    const GemmArgs& g = gs[i];
    const bool plain = !g.epi.relu && !g.epi.mask_src && g.epi.drop.p == 0.f && !g.epi.residual && !g.epi.bias && g.epi.accumulate;
    if (!(is16(g.A.dtype) && g.A.dtype == g.B.dtype && g.A.dtype == gs[0].A.dtype && g.A.mn_major && g.B.mn_major && plain &&
          g.c_dtype == F32 && g.nb1 == 1 && g.nb2 == 1 && g.M % BM == 0 && g.N % 256 == 0 && g.K > 0 && g.splitk <= 1 &&
          (reinterpret_cast<uintptr_t>(g.C) & 7) == 0 && g.ldc % 2 == 0))
      return 2;
  }
  if (ablate_mask() & ABL_WGRAD) return 0;
  if (g_num_sms == 0) {
    int dev = 0;
    B200ST_CUDA(cudaGetDevice(&dev));
    B200ST_CUDA(cudaDeviceGetAttribute(&g_num_sms, cudaDevAttrMultiProcessorCount, dev));
  }
  const TcDebug& dbg = tc_debug();
  const int num_sms = dbg.max_ctas > 0 ? dbg.max_ctas : (dbg.reserve_sms > 0 && dbg.reserve_sms < g_num_sms ? g_num_sms - dbg.reserve_sms : g_num_sms);
  TcGroup grp;
  std::memset(&grp, 0, sizeof(grp));
  grp.n = n;
  int64_t work = 0;
  int tiles0[kMaxGroup], kbt[kMaxGroup];
  for (int i = 0; i < n; ++i) {
    tiles0[i] = (gs[i].M / BM) * (gs[i].N / 256);
    kbt[i] = ceil_div(gs[i].K, BK);
    work += (int64_t)tiles0[i] * kbt[i];
  }
  // smallest common k-range L (in 64-row blocks) whose work units fit one wave of `num_sms` CTAs
  int L = (int)((work + num_sms - 1) / num_sms);
  if (L < 2) L = 2;
  for (;; ++L) {
    int64_t units = 0;
    for (int i = 0; i < n; ++i) units += (int64_t)tiles0[i] * ceil_div(kbt[i], L);
    if (units <= num_sms || L >= 4096) break;
  }
  int tile = 0;
  for (int i = 0; i < n; ++i) {
    const GemmArgs& g = gs[i];
    TcGroupProb& q = grp.prob[i];
    q.m_tiles = g.M / BM; q.n_tiles = g.N / 256; q.kb_total = kbt[i];
    q.kb_per_split = L < kbt[i] ? L : kbt[i];
    q.splitk = ceil_div(kbt[i], q.kb_per_split);
    q.tile_begin = tile;
    q.alpha = g.epi.alpha;
    tile += q.m_tiles * q.n_tiles * q.splitk;
    B200ST_TRY(make_operand_map(g.A, g.M, g.K, 1, 1, BM, &q.ta));
    B200ST_TRY(make_operand_map(g.B, g.N, g.K, 1, 1, 256, &q.tb));
    q.C = reinterpret_cast<float*>(g.C); q.ldc = g.ldc;
  }
  grp.num_tiles = tile;
  const uint32_t stage_bytes = kABytes + 256u * BK * 2;
  int stages = (int)((kSmemLimit - 2048) / stage_bytes);
  if (stages > 8) stages = 8;
  grp.stages = stages;
  const size_t smem = 1024 + (size_t)stages * stage_bytes + 16 * stages + 16;
  B200ST_CHECK(smem <= (size_t)kSmemLimit, "smem budget exceeded");
  auto kern = gs[0].A.dtype == BF16 ? tc_wgrad_group_kernel<true> : tc_wgrad_group_kernel<false>;
  static bool attr_set[2] = {false, false};
  if (!attr_set[gs[0].A.dtype == BF16]) {
    B200ST_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemLimit));
    attr_set[gs[0].A.dtype == BF16] = true;
  }
  const int grid = grp.num_tiles < num_sms ? grp.num_tiles : num_sms;
  ++g_launches;
  if (g_prof) {
    ProfRec r{gs[0], stream, 256, grp.prob[0].splitk};
    r.group_n = n;
    for (int i = 1; i < n; ++i) r.rest[i - 1] = gs[i];
    g_prof_recs.push_back(r);
  }
  launch_pdl(kern, grid, kThreads, smem, stream, grp);
  B200ST_LAUNCH_CHECK();
  return 0;
}


// Fused FFN forward (see fused_mlp_fwd_kernel).  X: 16-bit [M, d] (LayerNorm output); W1 [d, ffn], W2 [ffn, d] in the same
// 16-bit type (TF layouts); F1 out [M, ffn] (saved for the backward pass); x_out fp32 [M, d] must already hold the residual.
bool fused_mlp_supported(int M, int d, int ffn, int dtype) {
  return is16(dtype) && (d == 128 || d == 256) && ffn % 128 == 0 && M > 0 && !getenv("B200ST_NO_FUSED_MLP");
}
int fused_mlp_fwd(const void* X, int dtype, int M, int d, int ffn, const void* W1, const float* b1, const void* W2, const float* b2,
                  DropoutSpec drop_ffn, DropoutSpec drop_post, void* F1, float* x_out, cudaStream_t stream, int* tickets) {
  if (ablate_mask() & ABL_MLP_FWD) return 0;
  B200ST_CHECK(fused_mlp_supported(M, d, ffn, dtype), "fused MLP: unsupported shape / dtype");
  if (g_num_sms == 0) {
    int dev = 0;
    B200ST_CUDA(cudaGetDevice(&dev));
    B200ST_CUDA(cudaDeviceGetAttribute(&g_num_sms, cudaDevAttrMultiProcessorCount, dev));
  }
  if (drop_ffn.p > 0.f) B200ST_CHECK(drop_ffn.bits != nullptr, "fused MLP needs precomputed dropout bits");
  if (drop_post.p > 0.f) B200ST_CHECK(drop_post.bits != nullptr, "fused MLP needs precomputed dropout bits");
  const int m_tiles = ceil_div(M, BM), chunks = ffn / 128;
  // slices of the hidden dimension: the most CTAs that still fit one wave, with an equal number of chunks per slice
  int splits = 1;
  for (int s2 = 1; s2 <= chunks; ++s2)
    if (chunks % s2 == 0 && (int64_t)m_tiles * s2 <= g_num_sms - tc_debug().reserve_sms) splits = s2;
  if (getenv("B200ST_MLP_SPLITS")) { const int f = atoi(getenv("B200ST_MLP_SPLITS")); if (f >= 1 && chunks % f == 0) splits = f; }
  MlpParams p{};
  p.M = M; p.d = d; p.ffn = ffn; p.splits = splits; p.chunks_per_cta = chunks / splits;
  p.b1 = b1; p.b2 = b2; p.drop_ffn = drop_ffn; p.drop_post = drop_post;
  p.relu = 1; p.alpha = 1.f; p.mask_src = nullptr; p.mask_ld = 0; p.tickets = tickets;
  p.F1 = reinterpret_cast<uint16_t*>(F1); p.out = x_out;
  B200ST_CHECK((reinterpret_cast<uintptr_t>(F1) & 3) == 0 && (reinterpret_cast<uintptr_t>(x_out) & 7) == 0, "fused MLP: unaligned output");
  CUtensorMap tx, tw1, tw2;
  B200ST_TRY(make_operand_map(GemmOperand{X, dtype, 0, d, 0, 0}, M, d, 1, 1, BM, &tx));
  B200ST_TRY(make_operand_map(GemmOperand{W1, dtype, 1, ffn, 0, 0}, ffn, d, 1, 1, 64, &tw1));
  B200ST_TRY(make_operand_map(GemmOperand{W2, dtype, 1, d, 0, 0}, d, ffn, 1, 1, 64, &tw2));
  auto kern = d == 256 ? (dtype == F16 ? fused_mlp_fwd_kernel<F16, true, 256> : fused_mlp_fwd_kernel<BF16, true, 256>)
                       : (dtype == F16 ? fused_mlp_fwd_kernel<F16, true, 128> : fused_mlp_fwd_kernel<BF16, true, 128>);
  static bool attr[4] = {false, false, false, false};
  const int ai = (dtype == F16 ? 1 : 0) + (d == 256 ? 2 : 0);
  if (!attr[ai]) {
    B200ST_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kMlpSmem));
    attr[ai] = true;
  }
  launch_pdl(kern, m_tiles * splits, kThreads, kMlpSmem, stream, tx, tw1, tw2, p);
  ++g_launches;
  B200ST_LAUNCH_CHECK();
  return 0;
}

// Fused FFN backward, data-gradient chain: dF1 = scale * (dY W2^T) masked by (F1 > 0)  [written for the W1 weight gradient],
// dH += dF1 W1^T (fp32, dH must be zero-initialised).  Same kernel, weights read as K-major B operands.
int fused_mlp_bwd(const void* dY, int dtype, int M, int d, int ffn, const void* W1, const void* W2, const void* F1, float scale,
                  void* dF1, float* dH, cudaStream_t stream, int* tickets) {
  if (ablate_mask() & ABL_MLP_BWD) return 0;
  B200ST_CHECK(fused_mlp_supported(M, d, ffn, dtype), "fused MLP: unsupported shape / dtype");
  if (g_num_sms == 0) {
    int dev = 0;
    B200ST_CUDA(cudaGetDevice(&dev));
    B200ST_CUDA(cudaDeviceGetAttribute(&g_num_sms, cudaDevAttrMultiProcessorCount, dev));
  }
  const int m_tiles = ceil_div(M, BM), chunks = ffn / 128;
  int splits = 1;
  for (int s2 = 1; s2 <= chunks; ++s2)
    if (chunks % s2 == 0 && (int64_t)m_tiles * s2 <= g_num_sms - tc_debug().reserve_sms) splits = s2;
  if (getenv("B200ST_MLP_SPLITS")) { const int f = atoi(getenv("B200ST_MLP_SPLITS")); if (f >= 1 && chunks % f == 0) splits = f; }
  MlpParams p{};
  p.M = M; p.d = d; p.ffn = ffn; p.splits = splits; p.chunks_per_cta = chunks / splits;
  p.b1 = nullptr; p.b2 = nullptr; p.drop_ffn = no_dropout(); p.drop_post = no_dropout();
  p.relu = 0; p.alpha = scale; p.mask_src = F1; p.mask_ld = ffn; p.tickets = tickets;
  p.F1 = reinterpret_cast<uint16_t*>(dF1); p.out = dH;
  B200ST_CHECK((reinterpret_cast<uintptr_t>(dF1) & 3) == 0 && (reinterpret_cast<uintptr_t>(dH) & 7) == 0 &&
               (reinterpret_cast<uintptr_t>(F1) & 3) == 0, "fused MLP: unaligned buffer");
  CUtensorMap tx, tw1, tw2;
  B200ST_TRY(make_operand_map(GemmOperand{dY, dtype, 0, d, 0, 0}, M, d, 1, 1, BM, &tx));
  B200ST_TRY(make_operand_map(GemmOperand{W2, dtype, 0, d, 0, 0}, ffn, d, 1, 1, 128, &tw1));     // G1: rows = hidden units, k = d
  B200ST_TRY(make_operand_map(GemmOperand{W1, dtype, 0, ffn, 0, 0}, d, ffn, 1, 1, d, &tw2));      // G2: rows = model dims, k = hidden
  auto kern = d == 256 ? (dtype == F16 ? fused_mlp_fwd_kernel<F16, false, 256> : fused_mlp_fwd_kernel<BF16, false, 256>)
                       : (dtype == F16 ? fused_mlp_fwd_kernel<F16, false, 128> : fused_mlp_fwd_kernel<BF16, false, 128>);
  static bool attr[4] = {false, false, false, false};
  const int ai = (dtype == F16 ? 1 : 0) + (d == 256 ? 2 : 0);
  if (!attr[ai]) {
    B200ST_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kMlpSmem));
    attr[ai] = true;
  }
  launch_pdl(kern, m_tiles * splits, kThreads, kMlpSmem, stream, tx, tw1, tw2, p);
  ++g_launches;
  B200ST_LAUNCH_CHECK();
  return 0;
}

void tc_profile_begin() {
  g_prof_recs.clear();
  g_prof = true;
}
bool tc_profile_active() { return g_prof; }
int tc_profile_end(double* ms, double* flops, int64_t* launches) {
  g_prof = false;
  constexpr int kReps = 4;
  double tms = 0, tf = 0;
  FILE* dump = getenv("B200ST_PROFILE_CSV") ? fopen(getenv("B200ST_PROFILE_CSV"), "w") : nullptr;
  if (dump) fprintf(dump, "M,N,K,batch,bn,splitk,a_mn,b_mn,epi,us,tflops\n");
  cudaEvent_t e0, e1;
  B200ST_CUDA(cudaEventCreate(&e0));
  B200ST_CUDA(cudaEventCreate(&e1));
  std::vector<ProfRec> recs;
  recs.swap(g_prof_recs);
  for (const ProfRec& r : recs) {
    const cudaStream_t st = r.stream;
    GemmArgs grp_args[4];
    grp_args[0] = r.g;
    for (int i = 1; i < r.group_n; ++i) grp_args[i] = r.rest[i - 1];
    auto run = [&]() -> int {
      if (r.has_conv) return gemm_tc_impl(r.g, st, &r.conv);
      return r.group_n > 1 ? gemm_wgrad_group(grp_args, r.group_n, st) : gemm_tc_bf16(r.g, st);
    };
    B200ST_TRY(run());                                          // warm-up (tensor maps, instruction cache)
    B200ST_CUDA(cudaEventRecord(e0, st));
    for (int i = 0; i < kReps; ++i) B200ST_TRY(run());
    B200ST_CUDA(cudaEventRecord(e1, st));
    B200ST_CUDA(cudaEventSynchronize(e1));
    float t = 0.f;
    B200ST_CUDA(cudaEventElapsedTime(&t, e0, e1));
    t /= kReps;
    double fl = 2.0 * (double)r.g.M * r.g.N * r.g.K * (double)r.g.nb1 * r.g.nb2;
    for (int i = 1; i < r.group_n; ++i) fl += 2.0 * (double)grp_args[i].M * grp_args[i].N * grp_args[i].K;
    const int epi = (r.g.epi.bias ? 1 : 0) | (r.g.epi.relu ? 2 : 0) | (r.g.epi.mask_src ? 4 : 0) | (r.g.epi.drop.p > 0.f ? 8 : 0) |
                    (r.g.epi.residual ? 16 : 0) | (r.g.c_dtype == F32 ? 32 : 0);
    if (dump) fprintf(dump, "%d,%d,%d,%d,%d,%d,%d,%d,%d,%.2f,%.1f\n", r.g.M, r.g.N, r.g.K, r.group_n > 1 ? -r.group_n : r.g.nb1 * r.g.nb2, r.bn,
                      r.splitk, r.g.A.mn_major, r.g.B.mn_major, epi, t * 1e3, fl / (t * 1e-3) / 1e12);   // batch = -n: grouped launch of n products (first one listed)
    tms += t; tf += fl;
  }
  if (dump) fclose(dump);
  cudaEventDestroy(e0); cudaEventDestroy(e1);
  if (ms) *ms = tms;
  if (flops) *flops = tf;
  if (launches) *launches = (int64_t)recs.size();
  return 0;
}

}  // namespace b200st
