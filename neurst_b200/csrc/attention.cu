// Fused multi-head attention for sm_90a (head dim 64): S = QK^T and O = PV on wgmma with fp32 accumulators in
// registers, operands staged by TMA, online softmax on the accumulator fragments (a query row lives in the four lanes of a
// quad), additive key bias / diagonal key mask (KeyMask: causal, monotonic or wait-k) exactly as the reference
// (multi_head_attention.py:145-160: logits + bias, FLOAT_MIN = -1e9), dropout on the probabilities (:207-208) from the precomputed keep-bit bitmap.  The [B,H,Tq,Tk] score /
// probability tensors never touch HBM: forward keeps only the per-row log-sum-exp; backward recomputes P from Q, K and the
// LSE (flash-attention style).
//
// forward : grid (q tiles of 128, H, B), 384 threads: warpgroup 0 = TMA producer, warpgroups 1-2 = 64 query rows each; the
//           probabilities go back into the tensor cores as the register A operand of the PV product.
// backward: attn_bwd_prep_kernel (zero dQ, D = rowsum(dO * O)), then grid (kv blocks of 128, H, B), 256 threads = two
//           compute warpgroups (255-register budget; thread 0 also issues the TMA loads of a two-stage Q / dO ring): K_j / V_j
//           resident, each warpgroup owns 64 keys and computes the transposed tiles S^T = K Q^T and dP^T = V dO^T, so
//           that P^T and dS^T are register A operands of the dV / dK products (accumulated in registers over the q tiles);
//           dS^T also goes through shared memory as the MN-major A operand of dQ = dS K.  The next 64-query half's S^T / dP^T
//           and its keep-bit loads are issued before the wait on the current dV / dK / dQ group; the two warpgroups' dQ
//           partials are summed through shared memory and reduced across kv blocks with one fp32 RED per element into a
//           scratch buffer (cast_rows_kernel -> bf16).
#include "gemm.cuh"
#include "kernels.cuh"
#include "pdl.cuh"
#include "ptx.cuh"

namespace b200st {

int make_tma_map_16(const void* ptr, int dtype, uint64_t inner, uint64_t rows, int nb1, int nb2, int64_t ld, int64_t sb1, int64_t sb2,
                    uint32_t box_rows, CUtensorMap* out);

namespace {

constexpr int BQ = 128, BKV = 128, DH = 64;
constexpr float kLog2e = 1.4426950408889634f;
constexpr float kLn2 = 0.6931471805599453f;
constexpr float kMaskMin = -1.0e9f;   // neurst/utils/compat.py:24
constexpr uint32_t kTile16K = 128 * 64 * 2;      // [128 rows x 64 bf16] swizzled tile
constexpr int kAttnThreads = 384;                // forward: TMA warpgroup + 2 compute warpgroups
constexpr int kBwdThreads = 256;                 // 2 compute warpgroups; thread 0 also issues the TMA loads
constexpr int kAttnConsumerWarps = 8;

struct AttnParams {
  int B, H, Tq, Tk, Tkp;
  float alpha;                 // dh^-0.5
  const float* bias;           // [B, Tk] additive or null
  const int32_t* kv_len;       // [B] or null: keys >= kv_len[b] are padding (bias -1e9): their key blocks are skipped
  KeyMask mask;                // CAUSAL kernels: key k hidden from query q when k > q + key_mask_off(mask, Tk)
  DropoutSpec drop;
  uint16_t* ctx; int64_t ctx_ld;          // [B*Tq, H*64], 16-bit type DT (bf16 or fp16)
  float* lse;                  // [B, H, Tq]  (natural log)
  // backward only
  const uint16_t* dctx; int64_t dctx_ld;
  float* dq_acc; int64_t dq_ld;           // fp32 [B*Tq, H*64] (zeroed by attn_bwd_prep_kernel)
  const float* dvec;                      // [B, H, Tq] rowsum(dO * O) (attn_bwd_prep_kernel)
  uint16_t* dk; int64_t dk_ld;            // [B*Tk, ...] view base already offset to the K columns; + h*64
  uint16_t* dv; int64_t dv_ld;
};

// every kernel below is templated on DT, the 16-bit operand type (BF16 or F16): it only selects the MMA operand format
// and the fp32 <-> 16-bit conversions
#define pack_bf16(a, b) pack2_16((a), (b), DT)

__device__ __forceinline__ float ex2_approx(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
// 64 keep-bits (keys k0 .. k0+63 of one query row) from the precomputed bitmap or regenerated; bits of keys >= Tkp read as 1
__device__ __forceinline__ void load_keep64(const DropoutSpec& d, bool row_ok, int64_t row_bit0, int k0, int Tkp, uint32_t thresh,
                                            uint32_t (&keep)[2]) {
  keep[0] = keep[1] = 0xffffffffu;
  if (!(d.p > 0.f) || !row_ok) return;
  if (d.bits && (Tkp & 63) == 0) {        // rows are 8-byte aligned in the bitmap: one 64-bit load
    if (k0 < Tkp) {
      const uint2 w = __ldg(reinterpret_cast<const uint2*>(d.bits + ((uint64_t)(row_bit0 + k0) >> 3)));
      keep[0] = w.x; keep[1] = w.y;
    }
    return;
  }
  if (d.bits) {                           // bitmap, unaligned rows: 8 byte loads (all issued before the first use)
    uint32_t byte[8];
    const uint8_t* bp = d.bits + ((uint64_t)(row_bit0 + k0) >> 3);
#pragma unroll
    for (int g = 0; g < 8; ++g) byte[g] = (k0 + 8 * g < Tkp) ? (uint32_t)__ldg(bp + g) : 0xffu;
    keep[0] = byte[0] | (byte[1] << 8) | (byte[2] << 16) | (byte[3] << 24);
    keep[1] = byte[4] | (byte[5] << 8) | (byte[6] << 16) | (byte[7] << 24);
    return;
  }
  // no bitmap: regenerate with Philox (stand-alone attention API); rolled, and each word indexed by a constant so that
  // keep[] stays in registers
#pragma unroll
  for (int w = 0; w < 2; ++w) {
#pragma unroll 1
    for (int g = 0; g < 4; ++g) {
      const int k8 = k0 + 32 * w + 8 * g;
      if (k8 < Tkp) {
        const uint32_t byte = dropout_keep8(dropout_seed(d), d.stream, (uint64_t)(row_bit0 + k8) >> 3, thresh);
        keep[w] = (keep[w] & ~(0xffu << (8 * g))) | (byte << (8 * g));
      }
    }
  }
}
// the keep-bits of keys [k16, k16 + 16) of one query row (k16 % 16 == 0; Tkp % 8 == 0 keeps rows byte-aligned); bits of keys
// >= Tkp read as 1.  When the row's byte offset is even (always when Tkp % 16 == 0) the two bytes are one 16-bit load.
__device__ __forceinline__ uint32_t load_keep16(const DropoutSpec& d, bool ok, int64_t row_bit0, int k16, int Tkp, uint32_t thresh) {
  if (!ok || k16 >= Tkp) return 0xffffu;
  const uint64_t byte = (uint64_t)(row_bit0 + k16) >> 3;
  const bool hi = k16 + 8 < Tkp;
  if (d.bits && hi && (byte & 1u) == 0) return __ldg(reinterpret_cast<const uint16_t*>(d.bits + byte));
  return drop_keep8(d, byte, thresh) | ((hi ? drop_keep8(d, byte + 1, thresh) : 0xffu) << 8);
}

// ==============================================================================================================
// forward.  K is double-buffered (the next K load runs behind the current block), V single-buffered.
// Element math is branch-free: the key bias (times log2 e, -inf beyond Tk) sits in a shared-memory table, the logit is
// one FFMA, exp is one MUFU.EX2, the dropout scale is folded into the final 1/l.
// ==============================================================================================================
template <bool CAUSAL, int DT>
__global__ void __launch_bounds__(kAttnThreads, 1)
attn_fwd_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK,
                const __grid_constant__ CUtensorMap tmV, const AttnParams p) {
  extern __shared__ uint8_t smem_raw[];
  constexpr bool BF = DT == BF16;
  const uint32_t base = (ptx::smem_u32(smem_raw) + 1023u) & ~1023u;
  const int nblk_all = (p.Tk + BKV - 1) / BKV;       // sizes the bias table (launch-time shared memory)
  // key blocks that hold at least one non-padded key (kv_len is written at the very start of the step, many kernels back:
  // complete and visible before this kernel's predecessor could start, so it may be read ahead of griddepcontrol.wait)
  const int nblk = p.kv_len ? max(1, min(nblk_all, (__ldg(p.kv_len + blockIdx.z) + BKV - 1) / BKV)) : nblk_all;
  const uint32_t sQ = base;                          // 16 KB
  const uint32_t sK = sQ + kTile16K;                 // 2 x 16 KB
  const uint32_t sV = sK + 2 * kTile16K;             // 16 KB
  const uint32_t sB = sV + kTile16K;                 // key bias * log2(e), [nblk * 128] floats
  const uint32_t bars = sB + (uint32_t)nblk_all * 512u;
  const uint32_t q_full = bars, v_full = bars + 8, v_empty = bars + 16;
  auto k_full = [&](int s2) { return bars + 24u + 8u * s2; };
  auto k_empty = [&](int s2) { return bars + 40u + 8u * s2; };
  float* btab = reinterpret_cast<float*>(smem_raw + (sB - ptx::smem_u32(smem_raw)));

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int qt = blockIdx.x, h = blockIdx.y, b = blockIdx.z;

  if (warp == 0 && lane == 0) {
    ptx::prefetch_tensormap(&tmQ); ptx::prefetch_tensormap(&tmK); ptx::prefetch_tensormap(&tmV);
    ptx::mbar_init(q_full, 1);
    ptx::mbar_init(v_full, 1); ptx::mbar_init(v_empty, kAttnConsumerWarps);
    for (int s2 = 0; s2 < 2; ++s2) { ptx::mbar_init(k_full(s2), 1); ptx::mbar_init(k_empty(s2), kAttnConsumerWarps); }
    ptx::fence_mbar_init();
  }
  __syncthreads();
  pdl_wait();      // everything above (barriers, descriptor prefetch) overlaps the previous kernel's tail
  pdl_trigger();

  if (warp < 4) {
    ptx::reg_dealloc<40>();
    if (warp == 0 && lane == 0) {
      ptx::mbar_arrive_expect_tx(q_full, kTile16K);
      ptx::tma_load_4d(sQ, &tmQ, q_full, 0, qt * BQ, h, b);
      for (int j = 0; j < nblk; ++j) {
        const int s2 = j & 1;
        ptx::mbar_wait(k_empty(s2), (((uint32_t)j >> 1) & 1u) ^ 1u);
        ptx::mbar_arrive_expect_tx(k_full(s2), kTile16K);
        ptx::tma_load_4d(sK + s2 * kTile16K, &tmK, k_full(s2), 0, j * BKV, h, b);
        ptx::mbar_wait(v_empty, ((uint32_t)j & 1u) ^ 1u);
        ptx::mbar_arrive_expect_tx(v_full, kTile16K);
        ptx::tma_load_4d(sV, &tmV, v_full, 0, j * BKV, h, b);
      }
    }
  } else {
    // ---------------- compute warpgroups: thread = 2 query rows (g, g + 8 of the warp's 16) x 32 key columns ----------------
    ptx::reg_alloc<232>();
    const int wg = (warp >> 2) - 1, g = lane >> 2, qd = lane & 3;
    const int row0 = wg * 64 + (warp & 3) * 16 + g;            // + 8 for the second row
    const uint32_t thresh = dropout_thresh16(p.drop.p);
    const float a2 = p.alpha * kLog2e;
    const float cmask = kMaskMin * kLog2e;
    const bool use_drop = p.drop.p > 0.f;
    const int moff = CAUSAL ? key_mask_off(p.mask, p.Tk) : 0;
    {
      const float* bias_row = p.bias ? p.bias + (int64_t)b * p.Tk : nullptr;
      for (int k = threadIdx.x - 128; k < nblk * BKV; k += 256)
        btab[k] = (k < p.Tk) ? (bias_row ? __ldg(bias_row + k) * kLog2e : 0.f) : -INFINITY;
      asm volatile("bar.sync 1, 256;" ::: "memory");
    }
    int qrow[2]; bool qok[2];
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      qrow[r] = qt * BQ + row0 + 8 * r;
      qok[r] = qrow[r] < p.Tq;
    }
    const int64_t bit0 = (((int64_t)b * p.H + h) * p.Tq + qrow[0]) * p.Tkp;   // keep-bit of row qrow[0], key 0 (row + 8: + 8 Tkp)
    float m[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};   // running row max (log2 domain), this thread's partial row sums
    float o[32];
#pragma unroll
    for (int i = 0; i < 32; ++i) o[i] = 0.f;
    ptx::mbar_wait(q_full, 0);
    for (int j = 0; j < nblk; ++j) {
      const uint32_t k_s = sK + (uint32_t)(j & 1) * kTile16K;
      float s[64];
#pragma unroll
      for (int i = 0; i < 64; ++i) s[i] = 0.f;
      ptx::mbar_wait(k_full(j & 1), ((uint32_t)j >> 1) & 1u);
      ptx::fence_acc(s);
      ptx::wgmma_fence();
#pragma unroll
      for (int k = 0; k < DH / 16; ++k)
        ptx::WgmmaSS<BKV, BF, 0, 0>::mma(s, ptx::desc_kmajor(sQ + (uint32_t)wg * 8192u, k), ptx::desc_kmajor(k_s, k), k > 0 ? 1 : 0);
      ptx::wgmma_commit();
      uint32_t keep[2][4];                 // keep bits of the block's 128 keys for both rows (in flight during the MMA)
#pragma unroll
      for (int r = 0; r < 2; ++r) {
        uint32_t k2[2];
        load_keep64(p.drop, qok[r] && use_drop, bit0 + 8 * r * p.Tkp, j * BKV, p.Tkp, thresh, k2);
        keep[r][0] = k2[0]; keep[r][1] = k2[1];
        load_keep64(p.drop, qok[r] && use_drop, bit0 + 8 * r * p.Tkp, j * BKV + 64, p.Tkp, thresh, k2);
        keep[r][2] = k2[0]; keep[r][3] = k2[1];
      }
      ptx::wgmma_wait<0>();
      ptx::fence_acc(s);
      if (lane == 0) ptx::mbar_arrive(k_empty(j & 1));
      // logits (log2 domain) and block row max
      float bmax[2] = {-INFINITY, -INFINITY};
#pragma unroll
      for (int c8 = 0; c8 < 16; ++c8) {
        const int kcol = j * BKV + 8 * c8 + 2 * qd;
        const float2 bb = *reinterpret_cast<const float2*>(btab + kcol);
#pragma unroll
        for (int r = 0; r < 2; ++r) {
          float x0 = fmaf(s[4 * c8 + 2 * r], a2, bb.x), x1 = fmaf(s[4 * c8 + 2 * r + 1], a2, bb.y);
          if (CAUSAL) {
            const int qlim = qrow[r] + moff;                  // keys k > qlim get the additive FLOAT_MIN
            x0 = (kcol > qlim) ? x0 + cmask : x0;
            x1 = (kcol + 1 > qlim) ? x1 + cmask : x1;
          }
          s[4 * c8 + 2 * r] = x0; s[4 * c8 + 2 * r + 1] = x1;
          bmax[r] = fmaxf(bmax[r], fmaxf(x0, x1));
        }
      }
      float corr[2], m_new[2];
#pragma unroll
      for (int r = 0; r < 2; ++r) {
        bmax[r] = fmaxf(bmax[r], __shfl_xor_sync(0xffffffffu, bmax[r], 1));
        bmax[r] = fmaxf(bmax[r], __shfl_xor_sync(0xffffffffu, bmax[r], 2));
        m_new[r] = fmaxf(m[r], bmax[r]);
        corr[r] = ex2_approx(m[r] - m_new[r]);       // 0 on the first block (m = -inf)
        m[r] = m_new[r];
      }
      // probabilities -> 16-bit register A operand of the PV product; dropout scale applied at the end
      uint32_t p16[8][4];
      float bsum[2] = {0.f, 0.f};
#pragma unroll
      for (int c8 = 0; c8 < 16; ++c8) {
#pragma unroll
        for (int r = 0; r < 2; ++r) {
          const float p0 = ex2_approx(s[4 * c8 + 2 * r] - m_new[r]), p1 = ex2_approx(s[4 * c8 + 2 * r + 1] - m_new[r]);
          bsum[r] += p0 + p1;
          const uint32_t kb = keep[r][c8 >> 2] >> (8 * (c8 & 3) + 2 * qd);
          p16[c8 >> 1][(c8 & 1) * 2 + r] = pack_bf16((kb & 1u) ? p0 : 0.f, (kb & 2u) ? p1 : 0.f);
        }
      }
#pragma unroll
      for (int r = 0; r < 2; ++r) l[r] = l[r] * corr[r] + bsum[r];
#pragma unroll
      for (int c8 = 0; c8 < 8; ++c8) {
        o[4 * c8] *= corr[0]; o[4 * c8 + 1] *= corr[0];
        o[4 * c8 + 2] *= corr[1]; o[4 * c8 + 3] *= corr[1];
      }
      ptx::mbar_wait(v_full, (uint32_t)j & 1u);
      ptx::fence_acc(o);
      ptx::wgmma_fence();
#pragma unroll
      for (int k = 0; k < BKV / 16; ++k)
        ptx::WgmmaRS<DH, BF, 1>::mma(o, p16[k], ptx::desc_mnmajor(sV, k), 1);
      ptx::wgmma_commit();
      ptx::wgmma_wait<0>();
      ptx::fence_acc(o);
      if (lane == 0) ptx::mbar_arrive(v_empty);
    }
    // ---- epilogue: O * scale / l -> ctx, LSE ----
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      l[r] += __shfl_xor_sync(0xffffffffu, l[r], 1);
      l[r] += __shfl_xor_sync(0xffffffffu, l[r], 2);
      if (qok[r]) {
        const float inv_l = (use_drop ? p.drop.scale : 1.0f) / l[r];
        uint16_t* dst = p.ctx + ((int64_t)b * p.Tq + qrow[r]) * p.ctx_ld + h * DH + 2 * qd;
#pragma unroll
        for (int c8 = 0; c8 < 8; ++c8)
          *reinterpret_cast<uint32_t*>(dst + 8 * c8) = pack_bf16(o[4 * c8 + 2 * r] * inv_l, o[4 * c8 + 2 * r + 1] * inv_l);
        if (qd == 0 && p.lse) p.lse[((int64_t)b * p.H + h) * p.Tq + qrow[r]] = m[r] * kLn2 + logf(l[r]);
      }
    }
  }
}

// ==============================================================================================================
// backward: one CTA per (kv block, head, batch)
// ==============================================================================================================
__device__ __forceinline__ void red_add_v2(float* addr, float a, float b) {
  asm volatile("red.global.add.v2.f32 [%0], {%1, %2};" ::"l"(addr), "f"(a), "f"(b) : "memory");
}

template <bool CAUSAL, int DT>
__global__ void __launch_bounds__(kBwdThreads, 1)
attn_bwd_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK,
                const __grid_constant__ CUtensorMap tmV, const __grid_constant__ CUtensorMap tmdO, const AttnParams p) {
  extern __shared__ uint8_t smem_raw[];
  constexpr bool BF = DT == BF16;
  const uint32_t base = (ptx::smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t sK = base;                          // 16 KB
  const uint32_t sV = sK + kTile16K;                 // 16 KB
  const uint32_t sQ = sV + kTile16K;                 // 2 stages x 16 KB
  const uint32_t sdO = sQ + 2 * kTile16K;            // 2 stages x 16 KB
  const uint32_t sdS = sdO + 2 * kTile16K;           // 2 warpgroups x 2 halves x 8 KB: dS^T [64 keys x 64 queries]
  const uint32_t sX = sdS + 2 * kTile16K;            // 2 warpgroups x 2 halves x 8 KB: dQ partials handed to the other warpgroup
  const uint32_t sLD = sX + 2 * kTile16K;            // 2 stages x (LSE[128] * log2(e), D[128]) fp32
  const uint32_t sB = sLD + 2048;                    // key bias * log2(e) of this kv block, 128 floats
  const uint32_t bars = sB + 512;
  const uint32_t kv_full = bars;
  auto qdo_full = [&](int s) { return bars + 8u * (1 + s); };
  auto qdo_empty = [&](int s) { return bars + 8u * (3 + s); };
  auto smem_f = [&](uint32_t a) { return reinterpret_cast<float*>(smem_raw + (a - ptx::smem_u32(smem_raw))); };

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int jb = blockIdx.x, h = blockIdx.y, b = blockIdx.z;
  const int nq = (p.Tq + BQ - 1) / BQ;
  if (p.kv_len && jb > 0 && jb * BKV >= __ldg(p.kv_len + b)) {
    // every key of this block is padding: P = 0 exactly, so dK = dV = 0 and the block adds nothing to dQ
    pdl_wait();
    pdl_trigger();
    for (int i = threadIdx.x; i < BKV * (DH / 8); i += blockDim.x) {
      const int r = i / (DH / 8), c8 = (i % (DH / 8)) * 8, kk = jb * BKV + r;
      if (kk < p.Tk) {
        *reinterpret_cast<uint4*>(p.dv + ((int64_t)b * p.Tk + kk) * p.dv_ld + h * DH + c8) = make_uint4(0, 0, 0, 0);
        *reinterpret_cast<uint4*>(p.dk + ((int64_t)b * p.Tk + kk) * p.dk_ld + h * DH + c8) = make_uint4(0, 0, 0, 0);
      }
    }
    return;
  }

  const bool producer = threadIdx.x == 0;
  const int row_lse = (b * p.H + h) * p.Tq;         // first LSE / D element of this (b, h)
  if (producer) {
    ptx::prefetch_tensormap(&tmQ); ptx::prefetch_tensormap(&tmK); ptx::prefetch_tensormap(&tmV); ptx::prefetch_tensormap(&tmdO);
    ptx::mbar_init(kv_full, 1);
    for (int s = 0; s < 2; ++s) { ptx::mbar_init(qdo_full(s), 1); ptx::mbar_init(qdo_empty(s), kAttnConsumerWarps); }
    ptx::fence_mbar_init();
  }
  __syncthreads();
  pdl_wait();      // everything above (barriers, descriptor prefetch) overlaps the previous kernel's tail
  pdl_trigger();

  // Producer side (thread 0 only): query tile i (Q and dO) goes to stage i % 2 once all 8 warps have released tile i - 2.
  auto load_tile = [&](int i) {
    const int st = i & 1;
    ptx::mbar_arrive_expect_tx(qdo_full(st), 2 * kTile16K);
    ptx::tma_load_4d(sQ + st * kTile16K, &tmQ, qdo_full(st), 0, i * BQ, h, b);
    ptx::tma_load_4d(sdO + st * kTile16K, &tmdO, qdo_full(st), 0, i * BQ, h, b);
  };
  // The tile's 128 LSE (times log2 e; +inf past Tq, so that P = 0 there) and 128 D values go to the LSE / D stage i % 2, one
  // value per thread.  The loads are issued under the MMAs of the tile before; a 256-thread barrier precedes every first read,
  // and a stage is rewritten only after the barrier that follows the last read of the tile it held.
  auto load_lse_d = [&](int i) {
    const int t = threadIdx.x & 127, q = i * BQ + t;
    float v;
    if (threadIdx.x < 128) v = q < p.Tq ? __ldg(p.lse + row_lse + q) * kLog2e : INFINITY;
    else v = q < p.Tq ? __ldg(p.dvec + row_lse + q) : 0.f;
    smem_f(sLD + (i & 1) * 1024)[threadIdx.x] = v;
  };
  if (producer) {
    ptx::mbar_arrive_expect_tx(kv_full, 2 * kTile16K);
    ptx::tma_load_4d(sK, &tmK, kv_full, 0, jb * BKV, h, b);
    ptx::tma_load_4d(sV, &tmV, kv_full, 0, jb * BKV, h, b);
    for (int i = 0; i < nq && i < 2; ++i) load_tile(i);
  }
  load_lse_d(0);
  {
    float* btab = smem_f(sB);
    const float* bias_row = p.bias ? p.bias + (int64_t)b * p.Tk : nullptr;
    const int t = threadIdx.x, k = jb * BKV + t;
    if (t < BKV) btab[t] = (k < p.Tk) ? (bias_row ? __ldg(bias_row + k) * kLog2e : 0.f) : -INFINITY;
    __syncthreads();
  }

  // Warpgroup wg owns keys [64 wg, 64 wg + 64) of the block; thread = 2 keys (g, g + 8 of the warp's 16) x the query columns
  // 8 c + 2 qd + {0, 1} of the transposed tiles.  Branch-free element math as in the forward kernel; the dropout scale is
  // folded into dS (FFMA) and into the dV epilogue.
  const int wg = warp >> 2, g = lane >> 2, qd = lane & 3;
  const int krow0 = wg * 64 + (warp & 3) * 16 + g;          // key row inside the block (+ 8 for the second)
  const uint32_t thresh = dropout_thresh16(p.drop.p);
  const float a2 = p.alpha * kLog2e;
  const float cmask = kMaskMin * kLog2e;
  const bool use_drop = p.drop.p > 0.f;
  const float dscale = use_drop ? p.drop.scale : 1.0f;
  const int moff = CAUSAL ? key_mask_off(p.mask, p.Tk) : 0;
  const float kbias[2] = {smem_f(sB)[krow0], smem_f(sB)[krow0 + 8]};
  const int key[2] = {jb * BKV + krow0, jb * BKV + krow0 + 8};
  const int key16 = key[0] & ~15;                           // key[0] & 7 == g, key[1] = key[0] + 8
  const uint32_t sK_wg = sK + (uint32_t)wg * 8192u, sV_wg = sV + (uint32_t)wg * 8192u;
  const int nu = 2 * nq;                                    // units of work: the two 64-query halves of every query tile

  float dv[32], dk[32], st_[32], dpt[32];
  uint32_t kb[16];                                          // keep bits of (query column 2 c8 + e) x keys key16 .. key16 + 15
#pragma unroll
  for (int t = 0; t < 32; ++t) { dv[t] = 0.f; dk[t] = 0.f; }
  // S^T = K Q^T ; dP^T = V dO^T ([64 keys x 64 queries] each) of unit u, and its keep bits (loaded while the MMAs run)
  auto issue_sdp = [&](int u) {
    const uint32_t q_h = sQ + ((u >> 1) & 1) * kTile16K + (uint32_t)(u & 1) * 8192u;
    const uint32_t do_h = sdO + ((u >> 1) & 1) * kTile16K + (uint32_t)(u & 1) * 8192u;
#pragma unroll
    for (int t = 0; t < 32; ++t) { st_[t] = 0.f; dpt[t] = 0.f; }
    ptx::fence_acc(st_); ptx::fence_acc(dpt);
    ptx::wgmma_fence();
#pragma unroll
    for (int k = 0; k < DH / 16; ++k)
      ptx::WgmmaSS<64, BF, 0, 0>::mma(st_, ptx::desc_kmajor(sK_wg, k), ptx::desc_kmajor(q_h, k), k > 0 ? 1 : 0);
#pragma unroll
    for (int k = 0; k < DH / 16; ++k)
      ptx::WgmmaSS<64, BF, 0, 0>::mma(dpt, ptx::desc_kmajor(sV_wg, k), ptx::desc_kmajor(do_h, k), k > 0 ? 1 : 0);
    ptx::wgmma_commit();
#pragma unroll
    for (int t = 0; t < 16; ++t) {
      const int q = (u >> 1) * BQ + (u & 1) * 64 + 8 * (t >> 1) + 2 * qd + (t & 1);
      kb[t] = load_keep16(p.drop, use_drop && q < p.Tq, ((int64_t)row_lse + q) * p.Tkp, key16, p.Tkp, thresh);
    }
  };

  ptx::mbar_wait(kv_full, 0);
  ptx::mbar_wait(qdo_full(0), 0);
  issue_sdp(0);
  for (int u = 0; u < nu; ++u) {
    const int i = u >> 1, hq = u & 1, st = i & 1;
    const uint32_t q_h = sQ + st * kTile16K + (uint32_t)hq * 8192u, do_h = sdO + st * kTile16K + (uint32_t)hq * 8192u;
    const float* lse_s = smem_f(sLD + st * 1024) + hq * 64;
    const float* d_s = lse_s + 128;
    ptx::wgmma_wait<0>();
    ptx::fence_acc(st_); ptx::fence_acc(dpt);
    uint32_t p16[4][4], ds16[4][4];
    const uint32_t ds_buf = sdS + (uint32_t)(2 * wg + hq) * 8192u;
#pragma unroll
    for (int c8 = 0; c8 < 8; ++c8) {
      const int ql = 8 * c8 + 2 * qd;                   // query column inside the half
      const int q0 = i * BQ + hq * 64 + ql;
      const float2 lse2 = *reinterpret_cast<const float2*>(lse_s + ql), Dq = *reinterpret_cast<const float2*>(d_s + ql);
#pragma unroll
      for (int r = 0; r < 2; ++r) {
        float pd[2], ds[2];
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          float x = fmaf(st_[4 * c8 + 2 * r + e], a2, kbias[r]);
          if (CAUSAL) x = (key[r] > q0 + e + moff) ? x + cmask : x;
          const float pr = ex2_approx(x - (e ? lse2.y : lse2.x));
          const bool kp = (kb[2 * c8 + e] >> (8 * r + g)) & 1u;
          const float dpv = kp ? dpt[4 * c8 + 2 * r + e] : 0.f;
          pd[e] = kp ? pr : 0.f;
          ds[e] = pr * fmaf(dpv, dscale, -(e ? Dq.y : Dq.x));
        }
        const uint32_t pp = pack_bf16(pd[0], pd[1]), dd = pack_bf16(ds[0], ds[1]);
        p16[c8 >> 1][(c8 & 1) * 2 + r] = pp;
        ds16[c8 >> 1][(c8 & 1) * 2 + r] = dd;
        // dS^T -> shared memory, MN-major A operand of dQ = dS K: row = key (128 B = 64 queries), 128B swizzle
        const int kr = krow0 - wg * 64 + 8 * r;
        const uint32_t addr = ds_buf + (uint32_t)kr * 128u + ((uint32_t)(c8 ^ (kr & 7)) << 4) + (uint32_t)qd * 4u;
        asm volatile("st.shared.b32 [%0], %1;" ::"r"(addr), "r"(dd) : "memory");
      }
    }
    ptx::fence_proxy_async_smem();       // dS^T (generic-proxy writes) -> visible to the tensor-core (async) proxy
    ptx::named_bar_sync(1 + wg, 128);
    // dV += P^T dO ; dK += dS^T Q (contraction over the 64 queries) ; dQ[64 queries x 64] = dS K (over this warpgroup's 64 keys)
    float dq[32];
#pragma unroll
    for (int t = 0; t < 32; ++t) dq[t] = 0.f;
    ptx::fence_acc(dv); ptx::fence_acc(dk); ptx::fence_acc(dq);
    ptx::wgmma_fence();
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      ptx::WgmmaRS<DH, BF, 1>::mma(dv, p16[k], ptx::desc_mnmajor(do_h, k), 1);
      ptx::WgmmaRS<DH, BF, 1>::mma(dk, ds16[k], ptx::desc_mnmajor(q_h, k), 1);
      ptx::WgmmaSS<DH, BF, 1, 1>::mma(dq, ptx::desc_mnmajor(ds_buf, k), ptx::desc_mnmajor(sK_wg, k), k > 0 ? 1 : 0);
    }
    ptx::wgmma_commit();
    // the next unit's S^T / dP^T run under this unit's dQ reduction
    if (u + 1 < nu) {
      if (hq == 1) ptx::mbar_wait(qdo_full((i + 1) & 1), ((uint32_t)(i + 1) >> 1) & 1u);
      issue_sdp(u + 1);
      if (hq == 1) load_lse_d(i + 1);
      ptx::wgmma_wait<1>();
    } else {
      ptx::wgmma_wait<0>();
    }
    ptx::fence_acc(dv); ptx::fence_acc(dk); ptx::fence_acc(dq);
    // dQ: both warpgroups hold partials of the same 64 x 64 block (over different keys).  Warpgroup 0 sums and reduces
    // columns [0, 32), warpgroup 1 columns [32, 64): each hands the other half of its fragment over through shared memory,
    // laid out [float4 j][thread] so that the stores and loads are free of bank conflicts.  The buffers alternate with
    // hq, so one barrier per unit also orders a buffer's reads before its next writes.
    {
      const int tw = threadIdx.x & 127;
      float4* xo = reinterpret_cast<float4*>(smem_f(sX + (uint32_t)(2 * wg + hq) * 8192u));
      const float4* xi = reinterpret_cast<const float4*>(smem_f(sX + (uint32_t)(2 * (1 - wg) + hq) * 8192u));
#pragma unroll
      for (int j = 0; j < 4; ++j) {                   // fragment indices stay compile-time: select, do not index by wg
        const int a = 4 * j, c = 16 + 4 * j;
        xo[j * 128 + tw] = wg ? make_float4(dq[a], dq[a + 1], dq[a + 2], dq[a + 3]) : make_float4(dq[c], dq[c + 1], dq[c + 2], dq[c + 3]);
      }
      ptx::named_bar_sync(3, 256);
      float sum[16];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float4 o = xi[j * 128 + tw];
        const int a = 4 * j, c = 16 + 4 * j;
        sum[4 * j] = o.x + (wg ? dq[c] : dq[a]);
        sum[4 * j + 1] = o.y + (wg ? dq[c + 1] : dq[a + 1]);
        sum[4 * j + 2] = o.z + (wg ? dq[c + 2] : dq[a + 2]);
        sum[4 * j + 3] = o.w + (wg ? dq[c + 3] : dq[a + 3]);
      }
#pragma unroll
      for (int r = 0; r < 2; ++r) {
        const int q = i * BQ + hq * 64 + (warp & 3) * 16 + g + 8 * r;
        if (q < p.Tq) {
          float* dq_row = p.dq_acc + ((int64_t)b * p.Tq + q) * p.dq_ld + h * DH + wg * 32 + 2 * qd;
#pragma unroll
          for (int c8 = 0; c8 < 4; ++c8) red_add_v2(dq_row + 8 * c8, sum[4 * c8 + 2 * r] * p.alpha, sum[4 * c8 + 2 * r + 1] * p.alpha);
        }
      }
    }
    if (hq == 1) {
      if (lane == 0) ptx::mbar_arrive(qdo_empty(st));
      if (producer && i + 2 < nq) {
        ptx::mbar_wait(qdo_empty(st), ((uint32_t)i >> 1) & 1u);
        load_tile(i + 2);
      }
      __syncwarp();
    }
  }
  ptx::wgmma_wait<0>();      // nothing is pending after the last unit; ptxas cannot tell, and would insert this wait itself
  ptx::fence_acc(dv); ptx::fence_acc(dk);
  // ---- dV, dK of this warpgroup's keys ----
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    if (key[r] < p.Tk) {
      uint16_t* dv_row = p.dv + ((int64_t)b * p.Tk + key[r]) * p.dv_ld + h * DH + 2 * qd;
      uint16_t* dk_row = p.dk + ((int64_t)b * p.Tk + key[r]) * p.dk_ld + h * DH + 2 * qd;
#pragma unroll
      for (int c8 = 0; c8 < 8; ++c8) {
        *reinterpret_cast<uint32_t*>(dv_row + 8 * c8) = pack_bf16(dv[4 * c8 + 2 * r] * dscale, dv[4 * c8 + 2 * r + 1] * dscale);
        *reinterpret_cast<uint32_t*>(dk_row + 8 * c8) = pack_bf16(dk[4 * c8 + 2 * r] * p.alpha, dk[4 * c8 + 2 * r + 1] * p.alpha);
      }
    }
  }
}

constexpr size_t kBwdSmem = 1024 + (size_t)(2 + 2 + 2 + 2 + 2 + 2) * kTile16K + 2048 + 512 + 64;

// One warp per (b, q) row: zero the fp32 dQ accumulator row and compute D[b,h,q] = sum_c dO[b,q,h,c] * O[b,q,h,c].
template <int DT>
__global__ void attn_bwd_prep_kernel(const uint16_t* __restrict__ o, int64_t o_ld, const uint16_t* __restrict__ dout,
                                     int64_t do_ld, float* __restrict__ dq_acc, float* __restrict__ dvec, int B, int H, int Tq) {
  pdl_wait();
  pdl_trigger();
  const int lane = threadIdx.x & 31;
  const int64_t rows = (int64_t)B * Tq;
  const int chunks = H * (DH / 8);                  // 16-byte chunks per row; 8 chunks per head
  for (int64_t r = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); r < rows; r += (int64_t)gridDim.x * (blockDim.x >> 5)) {
    const int b = (int)(r / Tq), q = (int)(r % Tq);
    for (int c0 = 0; c0 < chunks; c0 += 32) {
      const int c = c0 + lane;
      float part = 0.f;
      if (c < chunks) {
        const uint4 a = __ldg(reinterpret_cast<const uint4*>(o + r * o_ld + 8 * c)), d = __ldg(reinterpret_cast<const uint4*>(dout + r * do_ld + 8 * c));
        const uint32_t aw[4] = {a.x, a.y, a.z, a.w}, dw[4] = {d.x, d.y, d.z, d.w};
#pragma unroll
        for (int t = 0; t < 4; ++t) {
          const float2 x = unpack2_16(aw[t], DT), y = unpack2_16(dw[t], DT);
          part = fmaf(x.x, y.x, fmaf(x.y, y.y, part));
        }
        float4* z = reinterpret_cast<float4*>(dq_acc + r * (int64_t)H * DH + 8 * c);
        z[0] = make_float4(0.f, 0.f, 0.f, 0.f); z[1] = make_float4(0.f, 0.f, 0.f, 0.f);
      }
      part += __shfl_xor_sync(0xffffffffu, part, 1);
      part += __shfl_xor_sync(0xffffffffu, part, 2);
      part += __shfl_xor_sync(0xffffffffu, part, 4);
      if (c < chunks && (lane & 7) == 0) dvec[((int64_t)b * H + (c >> 3)) * Tq + q] = part;
    }
  }
}

// dst(bf16)[r, 0..cols) = src(fp32)[r, 0..cols)   (dq scratch -> the q columns of the fused dqkv buffer)
template <int DT>
__global__ void cast_rows_kernel(const float* __restrict__ src, int64_t ld_src, uint16_t* __restrict__ dst, int64_t ld_dst,
                                 int64_t rows, int cols) {
  pdl_wait();
  pdl_trigger();
  const int64_t n8 = rows * (cols / 8);
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n8; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r = i / (cols / 8);
    const int c = (int)(i % (cols / 8)) * 8;
    const float4 a = *reinterpret_cast<const float4*>(src + r * ld_src + c), b2 = *reinterpret_cast<const float4*>(src + r * ld_src + c + 4);
    uint4 pk;
    pk.x = pack_bf16(a.x, a.y); pk.y = pack_bf16(a.z, a.w); pk.z = pack_bf16(b2.x, b2.y); pk.w = pack_bf16(b2.z, b2.w);
    *reinterpret_cast<uint4*>(dst + r * ld_dst + c) = pk;
  }
}

constexpr size_t kFwdSmemFixed = 1024 + (size_t)(1 + 2 + 1) * kTile16K + 8 * 7 + 64;   // + 512 B per kv block (bias table)

}  // namespace

// q/k/v: bf16 views [B*T, ld] with head h at columns [h*64, h*64+64)
int attention_fwd_fused(int dt, const void* q, int64_t q_ld, const void* k, int64_t k_ld, const void* v, int64_t v_ld, int B, int H,
                        int Tq, int Tk, const float* bias, KeyMask mask, DropoutSpec drop, void* ctx, int64_t ctx_ld, float* lse,
                        cudaStream_t s, const int32_t* kv_len) {
  B200ST_CHECK(Tq > 0 && Tk > 0 && B > 0 && H > 0, "empty attention");
  B200ST_CHECK(B <= 65535 && H <= 65535, "attention grid too large");
  B200ST_CHECK(is16(dt), "fused attention needs a 16-bit operand type");
  CUtensorMap tq, tk, tv;
  B200ST_TRY(make_tma_map_16(q, dt, DH, Tq, H, B, q_ld, DH, (int64_t)Tq * q_ld, BQ, &tq));
  B200ST_TRY(make_tma_map_16(k, dt, DH, Tk, H, B, k_ld, DH, (int64_t)Tk * k_ld, BKV, &tk));
  B200ST_TRY(make_tma_map_16(v, dt, DH, Tk, H, B, v_ld, DH, (int64_t)Tk * v_ld, BKV, &tv));
  AttnParams p{};
  p.B = B; p.H = H; p.Tq = Tq; p.Tk = Tk; p.Tkp = (Tk + 7) / 8 * 8;
  p.alpha = 0.125f;                     // 64^-0.5 (multi_head_attention.py:203)
  p.bias = bias; p.mask = mask; p.drop = drop; p.kv_len = kv_len;
  p.ctx = reinterpret_cast<uint16_t*>(ctx); p.ctx_ld = ctx_ld; p.lse = lse;
  B200ST_CHECK((reinterpret_cast<uintptr_t>(ctx) & 15) == 0 && ctx_ld % 8 == 0, "ctx must be 16-byte aligned");
  const size_t smem = kFwdSmemFixed + (size_t)((Tk + BKV - 1) / BKV) * 512;
  B200ST_CHECK(smem <= 227 * 1024, "fused attention: Tk too large for the shared-memory bias table");
  const bool causal = mask.on != 0;
  auto kern = causal ? (dt == F16 ? attn_fwd_kernel<true, F16> : attn_fwd_kernel<true, BF16>)
                     : (dt == F16 ? attn_fwd_kernel<false, F16> : attn_fwd_kernel<false, BF16>);
  static size_t attr[4] = {0, 0, 0, 0};
  const int ai = (causal ? 1 : 0) + (dt == F16 ? 2 : 0);
  if (smem > attr[ai]) {
    B200ST_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    attr[ai] = smem;
  }
  dim3 grid((Tq + BQ - 1) / BQ, H, B);
  return launch(kern, grid, kAttnThreads, smem, s, tq, tk, tv, p);
}


// dq_scratch: fp32 [B*Tq, H*64] (overwritten).  dq/dk/dv: bf16 views like q/k/v.  lse / ctx from the forward pass.
int attention_bwd_fused(int dt, const void* q, int64_t q_ld, const void* k, int64_t k_ld, const void* v, int64_t v_ld, const void* ctx,
                        int64_t ctx_ld, const void* dctx, int64_t dctx_ld, const float* lse, int B, int H, int Tq, int Tk,
                        const float* bias, KeyMask mask, DropoutSpec drop, float* dq_scratch, void* dq, int64_t dq_ld, void* dk,
                        int64_t dk_ld, void* dv, int64_t dv_ld, cudaStream_t s, const int32_t* kv_len) {
  B200ST_CHECK(Tq > 0 && Tk > 0 && B > 0 && H > 0 && B <= 65535 && H <= 65535, "bad attention shape");
  B200ST_CHECK(is16(dt), "fused attention needs a 16-bit operand type");
  CUtensorMap tq, tk, tv, tdo;
  B200ST_TRY(make_tma_map_16(q, dt, DH, Tq, H, B, q_ld, DH, (int64_t)Tq * q_ld, BQ, &tq));
  B200ST_TRY(make_tma_map_16(k, dt, DH, Tk, H, B, k_ld, DH, (int64_t)Tk * k_ld, BKV, &tk));
  B200ST_TRY(make_tma_map_16(v, dt, DH, Tk, H, B, v_ld, DH, (int64_t)Tk * v_ld, BKV, &tv));
  B200ST_TRY(make_tma_map_16(dctx, dt, DH, Tq, H, B, dctx_ld, DH, (int64_t)Tq * dctx_ld, BQ, &tdo));
  AttnParams p{};
  p.B = B; p.H = H; p.Tq = Tq; p.Tk = Tk; p.Tkp = (Tk + 7) / 8 * 8;
  p.alpha = 0.125f;
  p.bias = bias; p.mask = mask; p.drop = drop; p.kv_len = kv_len;
  p.ctx = reinterpret_cast<uint16_t*>(const_cast<void*>(ctx)); p.ctx_ld = ctx_ld;
  p.lse = const_cast<float*>(lse);
  p.dctx = reinterpret_cast<const uint16_t*>(dctx); p.dctx_ld = dctx_ld;
  p.dq_acc = dq_scratch; p.dq_ld = (int64_t)H * DH;
  p.dk = reinterpret_cast<uint16_t*>(dk); p.dk_ld = dk_ld;
  p.dv = reinterpret_cast<uint16_t*>(dv); p.dv_ld = dv_ld;
  B200ST_CHECK(((reinterpret_cast<uintptr_t>(dk) | reinterpret_cast<uintptr_t>(dv) | reinterpret_cast<uintptr_t>(dq) |
                 reinterpret_cast<uintptr_t>(dq_scratch)) & 15) == 0, "attention gradient buffers must be 16-byte aligned");
  static bool attr = false;
  if (!attr) {
    B200ST_CUDA(cudaFuncSetAttribute(attn_bwd_kernel<false, BF16>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kBwdSmem));
    B200ST_CUDA(cudaFuncSetAttribute(attn_bwd_kernel<true, BF16>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kBwdSmem));
    B200ST_CUDA(cudaFuncSetAttribute(attn_bwd_kernel<false, F16>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kBwdSmem));
    B200ST_CUDA(cudaFuncSetAttribute(attn_bwd_kernel<true, F16>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kBwdSmem));
    attr = true;
  }
  const int64_t rows = (int64_t)B * Tq;
  float* dvec = dq_scratch + rows * H * DH;
  p.dvec = dvec;
  B200ST_CHECK((reinterpret_cast<uintptr_t>(ctx) & 15) == 0 && (reinterpret_cast<uintptr_t>(dctx) & 15) == 0 && ctx_ld % 8 == 0 &&
               dctx_ld % 8 == 0, "attention ctx / dctx must be 16-byte aligned");
  {
    int64_t gp = (rows + 7) / 8;
    if (gp > 132 * 8) gp = 132 * 8;
    B200ST_TRY(launch(dt == F16 ? attn_bwd_prep_kernel<F16> : attn_bwd_prep_kernel<BF16>, (int)gp, 256, 0, s,
                      reinterpret_cast<const uint16_t*>(ctx), ctx_ld, reinterpret_cast<const uint16_t*>(dctx), dctx_ld, dq_scratch, dvec, B, H, Tq));
  }
  dim3 grid((Tk + BKV - 1) / BKV, H, B);
  const bool causal = mask.on != 0;
  auto kern = causal ? (dt == F16 ? attn_bwd_kernel<true, F16> : attn_bwd_kernel<true, BF16>)
                     : (dt == F16 ? attn_bwd_kernel<false, F16> : attn_bwd_kernel<false, BF16>);
  B200ST_TRY(launch(kern, grid, kBwdThreads, kBwdSmem, s, tq, tk, tv, tdo, p));
  const int64_t n8 = rows * (H * DH / 8);
  int64_t g = (n8 + 255) / 256;
  if (g > 132 * 8) g = 132 * 8;
  return launch(dt == F16 ? cast_rows_kernel<F16> : cast_rows_kernel<BF16>, (int)g, 256, 0, s, dq_scratch, (int64_t)H * DH,
                reinterpret_cast<uint16_t*>(dq), dq_ld, rows, H * DH);
}

}  // namespace b200st
