// wgmma / TMA 16-bit GEMM for sm_90a.
//
// Persistent, warp-specialised kernel (one CTA per SM, 384 threads = 3 warpgroups):
//   warpgroup 0    : TMA producer (one thread: cp.async.bulk.tensor -> 128B-swizzled smem ring, mbarrier complete_tx), filling
//                    the ring with the k-blocks of the CTA's tiles in tile order; gives its registers to the consumers (setmaxnreg)
//   warpgroups 1, 2: ping-pong consumers.  Each owns whole 128 x BN output tiles, alternating over the CTA's tiles, and
//                    accumulates one with two m64 wgmma.mma_async per k16 step into fp32 registers (one k-block in flight
//                    behind the one being issued).  Their main loops take turns through an ordered hand-off on two named
//                    barriers, so one warpgroup's fused epilogue runs while the other's wgmmas keep the tensor cores busy.
//                    Epilogue: per 64-row half, the fragments go to the warpgroup's own fp32 staging buffer in shared memory;
//                    the warpgroup then reads it back row by row (a warp covers 64 consecutive columns) and applies the fused
//                    epilogue with coalesced plain stores, or fp32 atomics for split-K / accumulate.  The generic epilogue
//                    code exists once in a rolled loop instead of once per fragment register.
// Tile: 128 x BN x 64 (BN in {64,128}: the 128 x 128 accumulator is 128 registers per thread of the 168-register budget of a
// 384-thread CTA); operands may be K-major or MN-major (wgrad / PV products), batched through 4-D tensor maps; optional
// split-K.  Every launch is a programmatic dependent launch (pdl.cuh).
//
// Replaces the cuBLAS calls behind tf.einsum / Dense / Conv2D at the reference sites listed in
// SURVEY.md §2.3 (K3,K4,K8,K9,K10,K11,K13,K15), e.g. neurst/layers/common_layers.py:270,276-288.
#include "gemm.cuh"
#include "pdl.cuh"
#include "ptx.cuh"

#include <mutex>
#include <type_traits>
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
constexpr int kOrderBar = 1;            // named barriers kOrderBar + wg: "consumer warpgroup wg may start its main loop"
constexpr int kEpiBar = 3;              // named barriers kEpiBar + wg: the 4 warps of warpgroup wg around its staging buffer
// Epilogue staging buffer of one consumer warpgroup: 64 rows x BN fp32 accumulators.  Rows are BN + 8 floats apart, so the
// 8-byte fragment stores of a half-warp (rows g..g+3, columns 2q) hit 32 distinct banks.
__host__ __device__ constexpr uint32_t staging_bytes(int bn) { return 64u * (uint32_t)(bn + 8) * 4u; }
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
  int plain16;          // 16-bit C, plain stores, epilogue = alpha (+ bias) only: the short epilogue loop applies
  int c_reduce;         // tc_gemm_f32_kernel: bulk reduce-adds (split-K / accumulate) instead of bulk stores
  // Implicit convolution A operand (tc_gemm_kernel<..., CONV = true>; conv2 of the speech front-end, see ConvA): A tile = conv_tu time rows x F2 positions of
  // one plane x 64 channels, read as a 4-D box (channels, F2, time rows, plane) shifted by the tap — coordinates outside the
  // tensor are zero-filled by the TMA unit, which is the convolution's pad-1 border; k-block kb = (tap, 64-channel chunk).
  // The data gradient writes the tiles as they are (class-major tiles); the forward (conv_remap) sends tile rows to the
  // dense [B, T2, F2] rows of its output and drops the rows past the image.
  int conv_ub;          // row tiles per utterance
  int conv_tu;          // time rows per tile
  int conv_kpc;         // k-blocks per tap (C / 64)
  int conv_remap, conv_T2, conv_F2;
  int conv_dt[9], conv_df[9], conv_wrow[9], conv_plane[9];   // per tap: time / frequency shift, first weight row, first plane
  uint32_t conv_a_bytes;                      // bytes one A box delivers (64 ch x F2 x conv_tu x 2)
  // Data gradient (tc_gemm_conv_kernel<B_MN = false>): the four parity classes in one launch.  Tile = unit * 4 + cls, unit =
  // (row tile, n tile); class cls has the taps conv_tap0[cls] .. conv_tap0[cls] + conv_ntap[cls] - 1 (the classes' taps
  // follow each other, 9 in all) and writes C + cls * conv_cls_elems.  See dgrad_first_tile.
  int conv_tap0[4], conv_ntap[4];
  int64_t conv_cls_elems;
};
constexpr int kConvRows = 1, kConvWgrad = 2;   // ConvA::mode: tc_gemm_kernel's A operand, or tc_wgrad_group_kernel's operands

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

// Static schedule of the conv2 data gradient's tiles over its persistent CTAs.  The tiles, in (unit, class) order, form one
// sequence of W = units * 9 * conv_kpc k-blocks; CTA c owns the tiles whose first k-block lies in [ceil(c W / G),
// ceil((c + 1) W / G)) for a grid of G CTAs.  Each CTA's k-blocks therefore differ from the mean W / G by less than one tile
// (at most 4 taps * conv_kpc k-blocks), and the four class tiles of a unit, which read the same dZ2 rows, run back to back on
// one SM.  Returns the first tile of CTA c (c = G: the tile count).
__device__ __forceinline__ int64_t dgrad_first_tile(const TcParams& p, int c) {
  const int64_t per_unit = 9 * p.conv_kpc;
  const int64_t s = ((int64_t)c * (p.num_tiles / 4) * per_unit + gridDim.x - 1) / gridDim.x;
  int64_t unit = s / per_unit;
  const int rem = (int)(s - unit * per_unit);
  int cls = 0;
  while (cls < 4 && p.conv_tap0[cls] * p.conv_kpc < rem) ++cls;
  if (cls == 4) { ++unit; cls = 0; }
  return unit * 4 + cls;
}

// Coordinates of data-gradient tile `tile` (parity class tile & 3): its row / n tile and its k-blocks [kb0, kb1) in the
// 9-tap k-block numbering (k-block kb is tap kb / conv_kpc).
__device__ __forceinline__ TileCoord decode_dgrad_tile(const TcParams& p, int64_t tile, int& kb0, int& kb1) {
  const int cls = (int)(tile & 3);
  const int64_t unit = tile >> 2;
  TileCoord t;
  t.split = 0; t.b1 = 0; t.b2 = 0;
  t.n_blk = (int)(unit % p.n_tiles);
  t.m_blk = (int)(unit / p.n_tiles);
  kb0 = p.conv_tap0[cls] * p.conv_kpc;
  kb1 = kb0 + p.conv_ntap[cls] * p.conv_kpc;
  return t;
}

// The smem operand ring shared by the producer thread and the consumer warps: `full` barriers count the producer's
// expect_tx arrival, `empty` barriers one arrival per warp that reads the slot (init(releasers)).
struct Ring {
  uint32_t smem, bars, stage_bytes;
  int stages, stage;
  uint32_t phase;
  __device__ __forceinline__ uint32_t full() const { return bars + 8u * stage; }
  __device__ __forceinline__ uint32_t empty(int s) const { return bars + 8u * (stages + s); }
  __device__ __forceinline__ uint32_t slot() const { return smem + (uint32_t)stage * stage_bytes; }
  __device__ __forceinline__ void advance() { if (++stage == stages) { stage = 0; phase ^= 1u; } }
  // step over n slots that another warpgroup consumes
  __device__ __forceinline__ void skip(int n) {
    stage += n;
    const int wraps = stage / stages;
    stage -= wraps * stages;
    phase ^= (uint32_t)wraps & 1u;
  }
  __device__ __forceinline__ void init(int releasers) const {
    for (int s = 0; s < stages; ++s) { ptx::mbar_init(bars + 8u * s, 1); ptx::mbar_init(empty(s), releasers); }
  }
};

// fp32 output rows of one consumer warpgroup on their way to global memory through a 128B-swizzled fp32 tensor map
// (make_out_map_f32): [64 rows x 32 columns] boxes, box b (columns 32 b ..) at base + 8 KB * b, rows 128 B apart, the
// 16-byte chunks XOR-swizzled by row % 8 as the map's 128B swizzle expects (a warp's fragment stores hit all 32 banks).
// base must be 1024-byte aligned.  Stores the warpgroup's [64 x N] wgmma accumulator fragment (layout: ptx.cuh) times alpha.
template <int N>
__device__ __forceinline__ void stage_rows_sw128(uint32_t base, const float (&acc)[N / 2], float alpha, int warp, int lane) {
  const int g = lane >> 2, q = lane & 3;
  // this thread's rows (warp & 3) * 16 + g + 8 hr of the warpgroup's 64: row % 8 = g
  const uint32_t row = base + (uint32_t)((warp & 3) * 16 + g) * 128u + (uint32_t)(q & 1) * 8u;
#pragma unroll
  for (int j = 0; j < N / 8; ++j) {
#pragma unroll
    for (int hr = 0; hr < 2; ++hr) {
      const uint32_t chunk = (uint32_t)(((j & 3) * 2 + (q >> 1)) ^ g);
      const uint32_t dst = row + (uint32_t)(j >> 2) * 8192u + (uint32_t)hr * 1024u + chunk * 16u;
      asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(dst), "f"(acc[4 * j + 2 * hr] * alpha), "f"(acc[4 * j + 2 * hr + 1] * alpha)
                   : "memory");
    }
  }
}
// One thread, after the warpgroup's stage_rows_sw128 stores, fence_proxy_async_smem and a warpgroup barrier:
// C[row0 .., col0 .. col0 + N) += the staged rows as N / 32 bulk reduce-adds (fp32 adds performed at L2, element-wise atomic
// with respect to other writers; rows and columns outside the map are skipped).  Returns once they are performed, so the
// staging may be reused and the sums are visible to whatever runs after the kernel.
template <int N>
__device__ __forceinline__ void reduce_add_rows_sw128(const CUtensorMap* tm, uint32_t base, int col0, int row0) {
#pragma unroll
  for (int b = 0; b < N / 32; ++b) ptx::tma_reduce_add_2d(tm, base + (uint32_t)b * 8192u, col0 + b * 32, row0);
  ptx::bulk_commit();
  ptx::bulk_wait_all();
}

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

// Consumer warpgroup main loop of one whole 128 x BN tile: acc[h] (rows 64 h .. 64 h + 63) = sum over the next nkb ring slots
// of A_slot[64 h .. 64 h + 63, :] B_slot^T.  Same pipelining as consume_kblocks; the slots are released by this warpgroup's 4
// warps alone.  `handoff` (bar.arrive on the other warpgroup's order barrier) runs once the last k-block's wgmmas are issued,
// so the other warpgroup's main loop queues behind them while this one drains its last group and runs its epilogue.
template <int BN, bool A_MN, bool B_MN, bool BF>
__device__ __forceinline__ void consume_tile(float (&acc)[2][BN / 2], Ring& r, int nkb, int lane, int handoff) {
  int prev = -1;
  for (int i = 0; i < nkb; ++i) {
    ptx::mbar_wait(r.full(), r.phase);
    const uint32_t sa = r.slot(), sb = r.slot() + kABytes;
    ptx::fence_acc(acc[0]);
    ptx::fence_acc(acc[1]);
    ptx::wgmma_fence();
#pragma unroll
    for (int k = 0; k < BK / 16; ++k) {
      const uint64_t db = B_MN ? ptx::desc_mnmajor(sb, k) : ptx::desc_kmajor(sb, k);
#pragma unroll
      for (int h = 0; h < 2; ++h)
        ptx::WgmmaSS<BN, BF, A_MN, B_MN>::mma(acc[h], A_MN ? ptx::desc_mnmajor(sa + h * 8192u, k) : ptx::desc_kmajor(sa + h * 8192u, k),
                                               db, (i > 0 || k > 0) ? 1 : 0);
    }
    ptx::wgmma_commit();
    if (prev >= 0) {
      ptx::wgmma_wait<1>();
      if (lane == 0) ptx::mbar_arrive(r.empty(prev));
    }
    prev = r.stage;
    r.advance();
  }
  if (handoff >= 0) ptx::named_bar_arrive(handoff, 256);
  ptx::wgmma_wait<0>();
  ptx::fence_acc(acc[0]);
  ptx::fence_acc(acc[1]);
  if (prev >= 0 && lane == 0) ptx::mbar_arrive(r.empty(prev));
}

// CONV: implicit conv2 A operand (TcParams conv fields; K-major A only), compiled into an entry point of its own
// (tc_gemm_conv_kernel) so that the plain GEMMs carry none of its code.
// F32C: fp32 C written through the tensor map tmC (bulk stores, or reduce-adds when p.c_reduce), epilogue alpha (+ bias);
// an entry point of its own (tc_gemm_f32_kernel): next to the general loop, its code spilled the BN = 128 accumulators.
template <int BN, bool A_MN, bool B_MN, bool BF, bool CONV, bool F32C = false>
__device__ __forceinline__ void tc_gemm_body(const CUtensorMap& tmA, const CUtensorMap& tmB, const CUtensorMap& tmC, const TcParams& p) {
  static_assert(BN <= 128, "a consumer warpgroup holds the whole 128 x BN accumulator");
  static_assert(!CONV || !A_MN, "the implicit conv A operand is K-major");
  extern __shared__ uint8_t smem_raw[];
  constexpr uint32_t kBBytes = BN * BK * 2;
  constexpr uint32_t kStageBytes = kABytes + kBBytes;

  Ring ring;
  ring.smem = (ptx::smem_u32(smem_raw) + 1023u) & ~1023u;
  ring.stages = p.stages;
  ring.stage_bytes = kStageBytes;
  const uint32_t staging = ring.smem + (uint32_t)p.stages * kStageBytes;      // 2 x staging_bytes(BN)
  ring.bars = staging + 2u * staging_bytes(BN);
  ring.stage = 0; ring.phase = 0;

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  // the CTA's tiles: blockIdx.x, + gridDim.x, ... (the conv2 data gradient: a contiguous run, dgrad_first_tile)
  constexpr bool DGRAD = CONV && !B_MN;
  auto first_tile = [&]() -> int64_t { if constexpr (DGRAD) return dgrad_first_tile(p, blockIdx.x); else return blockIdx.x; };
  auto end_tile = [&]() -> int64_t { if constexpr (DGRAD) return dgrad_first_tile(p, blockIdx.x + 1); else return p.num_tiles; };
  auto next_tile = [&](int64_t tile) -> int64_t { if constexpr (DGRAD) return tile + 1; else return tile + gridDim.x; };

  if (warp == 0 && lane == 0) {
    ptx::prefetch_tensormap(&tmA);
    ptx::prefetch_tensormap(&tmB);
    if constexpr (F32C) ptx::prefetch_tensormap(&tmC);
    ring.init(4);         // a slot is read by the 4 warps of the warpgroup that owns its tile
    ptx::fence_mbar_init();
  }
  __syncthreads();
  pdl_wait();      // everything above (barriers, descriptor prefetch) overlaps the previous kernel's tail
  pdl_trigger();

  if (warp < 4) {
    // ===================== TMA producer =====================
    ptx::reg_dealloc<kProducerRegs>();
    if (warp == 0 && lane == 0) {
      for (int64_t tile = first_tile(), end = end_tile(); tile < end; tile = next_tile(tile)) {
        TileCoord t;
        int kb0, kb1;
        if constexpr (DGRAD) {
          t = decode_dgrad_tile(p, tile, kb0, kb1);
        } else {
          t = decode_tile(p, tile);
          kb0 = t.split * p.kb_per_split;
          kb1 = min(p.kb_total, kb0 + p.kb_per_split);
        }
        for (int kb = kb0; kb < kb1; ++kb) {
          ptx::mbar_wait(ring.empty(ring.stage), ring.phase ^ 1u);
          const uint32_t sa = ring.slot();
          const uint32_t sb = sa + kABytes;
          if constexpr (CONV) {
            const int tap = kb / p.conv_kpc, c0 = (kb - tap * p.conv_kpc) * BK;
            ptx::mbar_arrive_expect_tx(ring.full(), p.conv_a_bytes + kBBytes);
            ptx::tma_load_4d(sa, &tmA, ring.full(), c0, p.conv_df[tap], (t.m_blk % p.conv_ub) * p.conv_tu + p.conv_dt[tap],
                             p.conv_plane[tap] + t.m_blk / p.conv_ub);
            if (B_MN) {
#pragma unroll
              for (int c = 0; c < BN / 64; ++c)
                ptx::tma_load_4d(sb + c * (64 * BK * 2), &tmB, ring.full(), t.n_blk * BN + c * 64, p.conv_wrow[tap] + c0, 0, 0);
            } else {
              ptx::tma_load_4d(sb, &tmB, ring.full(), c0, p.conv_wrow[tap] + t.n_blk * BN, 0, 0);
            }
            ring.advance();
            continue;
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
    // ===================== consumer warpgroups (ping-pong) =====================
    // Warpgroup wg takes the CTA's tiles j = wg, wg + 2, ...  The main loop of tile j starts after that of tile j - 1 has
    // been issued: the warpgroup waits on its own order barrier (except for tile 0) and, when tile j + 1 exists, arrives on
    // the other's.  Every arrive is matched by exactly one wait of the other warpgroup.
    ptx::reg_alloc<kConsumerRegs>();
    const int wg = (warp >> 2) - 1, g = lane >> 2, q = lane & 3;
    const GemmEpilogue& ep = p.epi;
    const int tid = threadIdx.x & 127;
    float* stg = reinterpret_cast<float*>(smem_raw + (staging - ptx::smem_u32(smem_raw)) + (uint32_t)wg * staging_bytes(BN));
    float acc[2][BN / 2];
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) acc[0][i] = acc[1][i] = 0.f;
    int j = 0;
    for (int64_t tile = first_tile(), end = end_tile(); tile < end; tile = next_tile(tile), ++j) {
      TileCoord t;
      int kb0, kb1;
      if constexpr (DGRAD) {
        t = decode_dgrad_tile(p, tile, kb0, kb1);
      } else {
        t = decode_tile(p, tile);
        kb0 = t.split * p.kb_per_split;
        kb1 = min(p.kb_total, kb0 + p.kb_per_split);
      }
      if ((j & 1) != wg) {
        ring.skip(kb1 - kb0);
        continue;
      }
      if (j > 0) ptx::named_bar_sync(kOrderBar + wg, 256);
      const int handoff = next_tile(tile) < end ? kOrderBar + (wg ^ 1) : -1;
      consume_tile<BN, A_MN, B_MN, BF>(acc, ring, kb1 - kb0, lane, handoff);
      const int64_t bidx = (int64_t)t.b2 * p.nb1 + t.b1;
      int64_t boff_c;
      if constexpr (DGRAD) boff_c = (tile & 3) * p.conv_cls_elems;      // the tile's parity class
      else boff_c = (int64_t)t.b2 * p.c_sb2 + (int64_t)t.b1 * p.c_sb1;
      const int64_t boff_mask = (int64_t)t.b2 * ep.mask_sb2 + (int64_t)t.b1 * ep.mask_sb1;
      const int64_t boff_res = (int64_t)t.b2 * ep.res_sb2 + (int64_t)t.b1 * ep.res_sb1;
      constexpr int kLd = BN + 8, kPairs = BN / 2, kRowStep = 128 / kPairs;
      const int cp = tid % kPairs, n = t.n_blk * BN + 2 * cp;
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        if constexpr (F32C) {
          // the half's raw accumulators go to the staging buffer as swizzled [64 x 32] boxes; alpha (+ bias) is applied
          // there as gemm_epilogue_value computes it, and one thread issues a bulk store or reduce-add per box that starts
          // inside C (the map clips rows past M and columns past N).  The buffer is refilled only after that thread has
          // seen the previous half's bulk operations finish reading it.
          const uint32_t sbuf = staging + (uint32_t)wg * staging_bytes(BN);
          if (tid == 0) ptx::bulk_wait_read_all();
          ptx::named_bar_sync(kEpiBar + wg, 128);
          stage_rows_sw128<BN>(sbuf, acc[h], 1.f, warp, lane);
          if (ep.alpha != 1.f || ep.bias) {
            ptx::named_bar_sync(kEpiBar + wg, 128);
            const int c = 2 * cp;                            // a column pair per thread, its bias pair loaded once per tile
            const float b0 = ep.bias && n < p.N ? __ldg(ep.bias + n) : 0.f, b1 = ep.bias && n + 1 < p.N ? __ldg(ep.bias + n + 1) : 0.f;
            const uint32_t col = sbuf + (uint32_t)(c >> 5) * 8192u + (uint32_t)(c & 3) * 4u;
#pragma unroll 4
            for (int r = tid / kPairs; r < 64; r += kRowStep) {
              const uint32_t a = col + (uint32_t)r * 128u + ((uint32_t)(((c & 31) >> 2) ^ (r & 7)) << 4);
              float v0, v1;
              asm volatile("ld.shared.v2.f32 {%0, %1}, [%2];" : "=f"(v0), "=f"(v1) : "r"(a) : "memory");
              v0 = v0 * ep.alpha;
              v1 = v1 * ep.alpha;
              if (ep.bias) { v0 += b0; v1 += b1; }
              asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(a), "f"(v0), "f"(v1) : "memory");
            }
          }
          ptx::fence_proxy_async_smem();               // the generic-proxy stores, visible to the bulk operations
          ptx::named_bar_sync(kEpiBar + wg, 128);
          const int r0 = t.m_blk * BM + h * 64;
          if (tid == 0 && r0 < p.M) {
#pragma unroll
            for (int b = 0; b < BN / 32; ++b) {
              const int c0 = t.n_blk * BN + b * 32;
              if (c0 >= p.N) break;
              if (p.c_reduce) ptx::tma_reduce_add_2d(&tmC, sbuf + (uint32_t)b * 8192u, c0, r0);
              else ptx::tma_store_2d(&tmC, sbuf + (uint32_t)b * 8192u, c0, r0);
            }
            ptx::bulk_commit();
          }
          continue;
        }
        ptx::named_bar_sync(kEpiBar + wg, 128);          // the previous half's reads are done
#pragma unroll
        for (int jj = 0; jj < BN / 8; ++jj) {
          const int r = (warp & 3) * 16 + g, c = 8 * jj + 2 * q;
          *reinterpret_cast<float2*>(stg + r * kLd + c) = make_float2(acc[h][4 * jj], acc[h][4 * jj + 1]);
          *reinterpret_cast<float2*>(stg + (r + 8) * kLd + c) = make_float2(acc[h][4 * jj + 2], acc[h][4 * jj + 3]);
        }
        ptx::named_bar_sync(kEpiBar + wg, 128);
        if (p.plain16 && n + 1 < p.N) {
          // alpha (+ bias) into 16-bit C, a column pair per thread: the bias pair and the column offset are fixed for the
          // tile, so a row costs one shared load, the arithmetic and one store (the general loop below re-derives every
          // epilogue option per element, and its instruction count, not memory, bounded the short-K GEMMs)
          const float b0 = ep.bias ? __ldg(ep.bias + n) : 0.f, b1 = ep.bias ? __ldg(ep.bias + n + 1) : 0.f;
          uint32_t* c32 = reinterpret_cast<uint32_t*>(p.C);
          const int64_t col = boff_c + n;
          auto store = [&](int r, int m) {
            const float2 v = *reinterpret_cast<const float2*>(stg + r * kLd + 2 * cp);
            float v0 = v.x * ep.alpha, v1 = v.y * ep.alpha;
            if (ep.bias) { v0 += b0; v1 += b1; }
            c32[(col + (int64_t)m * p.ldc) >> 1] = pack2_16(v0, v1, p.c_dtype);
          };
          bool remap = false;
          if constexpr (CONV) remap = p.conv_remap;
          if (remap) {
            // implicit conv2 forward: tile row rr is position (rr / F2, rr % F2) of the tile's conv_tu time rows; rows past the
            // tile's positions or past T2 are dropped (a loop of its own: the plain loop's instruction count sets short-K GEMMs)
            const int u0 = (t.m_blk % p.conv_ub) * p.conv_tu, b = t.m_blk / p.conv_ub;
#pragma unroll 4
            for (int r = tid / kPairs; r < 64; r += kRowStep) {
              const int rr = h * 64 + r, tr = rr / p.conv_F2, t2 = u0 + tr;
              if (tr < p.conv_tu && t2 < p.conv_T2) store(r, (b * p.conv_T2 + t2) * p.conv_F2 + (rr - tr * p.conv_F2));
            }
          } else {
#pragma unroll 8
            for (int r = tid / kPairs; r < 64; r += kRowStep) {
              const int m = t.m_blk * BM + h * 64 + r;
              if (m < p.M) store(r, m);
            }
          }
        } else if (n < p.N) {
#pragma unroll 4
          for (int r = tid / kPairs; r < 64; r += kRowStep) {
            const int m = t.m_blk * BM + h * 64 + r;
            if (m < p.M) {
              const float2 v = *reinterpret_cast<const float2*>(stg + r * kLd + 2 * cp);
              epilogue_pair(p, v.x, v.y, m, n, bidx, boff_c, boff_mask, boff_res);
            }
          }
        }
      }
    }
    if constexpr (F32C) {
      if (tid == 0) ptx::bulk_wait_all();      // the staging stays allocated until the last bulk operations are done
    }
  }
}


template <int BN, bool A_MN, bool B_MN, bool BF>
__global__ void __launch_bounds__(kThreads, 1)
tc_gemm_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, const TcParams p) {
  tc_gemm_body<BN, A_MN, B_MN, BF, false>(tmA, tmB, tmA, p);
}
// non-batched GEMMs with fp32 C that fits a tensor map and an alpha (+ bias) epilogue (gemm_tc_impl: TcParams::c_reduce)
template <int BN, bool A_MN, bool B_MN, bool BF>
__global__ void __launch_bounds__(kThreads, 1)
tc_gemm_f32_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                   const __grid_constant__ CUtensorMap tmC, const TcParams p) {
  tc_gemm_body<BN, A_MN, B_MN, BF, false, true>(tmA, tmB, tmC, p);
}
// the implicit conv2 GEMMs (conv2_fwd_implicit: MN-major weights, conv2_dgrad_implicit: K-major weights)
template <bool B_MN, bool BF>
__global__ void __launch_bounds__(kThreads, 1)
tc_gemm_conv_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, const TcParams p) {
  tc_gemm_body<128, false, B_MN, BF, true>(tmA, tmB, tmA, p);
}

// =============================================================================================================
// Grouped weight-gradient GEMM: up to kMaxGroup products  dW_g[K_in, N_out] += X_g^T dY_g  of one backward block in ONE
// persistent launch (TF autodiff of the Dense / einsum sites of a sublayer: neurst/layers/common_layers.py:270-288,
// multi_head_attention.py:145-215).  Each product alone has 2..16 output tiles and needs split-K over the B*T rows to fill
// the SMs, i.e. every CTA reduce-adds a full 128 x 256 fp32 tile for a handful of k-blocks of MMA work and every launch pays
// its fixed cost; together the products of a block give one wave of work units with k-ranges several times longer.
// Same pipeline as tc_gemm_kernel<256, true, true>; a work unit = (product, m tile, n tile, k split), exactly one per CTA
// (launch_wgrad_group).  Every CTA of the wave finishes at about the same time, so the units' fp32 tiles leave as bulk
// reduce-adds staged in the drained operand ring, not as per-thread atomics (see the fused FFN kernel's tail).
// =============================================================================================================
constexpr int kMaxGroup = 4;
struct TcGroupProb {
  CUtensorMap ta, tb;
  CUtensorMap tc;           // fp32 C (make_out_map_f32), the bulk reduce-add target
  int m_tiles, n_tiles, splitk, kb_total, kb_per_split, tile_begin;
  float alpha;
};
// Implicit conv2 filter gradient (conv2_wgrad_implicit, one product): m = (tap, input channel), k-block kb = (utterance, chunk
// of kt time rows x fw frequencies); A = the tap's parity-class plane shifted by the tap, B = dZ2 at the same positions, both
// MN-major 4-D boxes.  Both deliver krows of the 64 k rows; the rest stay zero (set up at kernel start).
struct ConvWgrad {
  int on, kpc, kc, fc, kt, fw, krows;     // m tiles per tap, k-blocks per utterance, frequency chunks per row group
  int dt[9], df[9], plane[9];
};
struct TcGroup {
  TcGroupProb prob[kMaxGroup];
  int n, num_tiles, stages;
  ConvWgrad cw;
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
      ptx::prefetch_tensormap(&grp.prob[i].tc);
    }
    ring.init(kConsumerWarps);
    ptx::fence_mbar_init();
  }
  if (grp.cw.on && grp.cw.krows < BK) {
    // k rows krows..63 of every 64 x 64 operand block are never written by the TMA unit: zero them once in every stage, in
    // both operands (a stale value times zero can still be NaN)
    constexpr int kBlocks = (BM + BN) / 64;
    const int tail16 = (BK - grp.cw.krows) * 8;           // 16-byte words per block tail
    uint8_t* ring0 = smem_raw + (ring.smem - ptx::smem_u32(smem_raw));
    for (int i = threadIdx.x; i < grp.stages * kBlocks * tail16; i += blockDim.x) {
      const int blk = i / tail16, w = i - blk * tail16;
      reinterpret_cast<uint4*>(ring0 + (uint32_t)blk * (64 * BK * 2) + grp.cw.krows * 128)[w] = make_uint4(0, 0, 0, 0);
    }
    ptx::fence_proxy_async_smem();
  }
  __syncthreads();
  pdl_wait();
  pdl_trigger();

  const GroupTile t = group_tile(grp, blockIdx.x);         // the CTA's one work unit (gridDim.x == grp.num_tiles)
  if (warp < 4) {
    ptx::reg_dealloc<kProducerRegs>();
    if (warp == 0 && lane == 0) {
      const CUtensorMap* ma = &grp.prob[t.gi].ta;
      const CUtensorMap* mb = &grp.prob[t.gi].tb;
      for (int kb = t.kb0; kb < t.kb1; ++kb) {
        ptx::mbar_wait(ring.empty(ring.stage), ring.phase ^ 1u);
        const uint32_t sa = ring.slot();
        const uint32_t sb = sa + kABytes;
        if (grp.cw.on) {
          const ConvWgrad& cw = grp.cw;
          const int tap = t.m_blk / cw.kpc, ci0 = (t.m_blk - tap * cw.kpc) * BM;
          const int b = kb / cw.kc, ch = kb - b * cw.kc;
          const int t0 = (ch / cw.fc) * cw.kt, f0 = (ch % cw.fc) * cw.fw;
          ptx::mbar_arrive_expect_tx(ring.full(), (uint32_t)((BM + BN) * cw.krows * 2));
#pragma unroll
          for (int c = 0; c < BM / 64; ++c)
            ptx::tma_load_4d(sa + c * (64 * BK * 2), ma, ring.full(), ci0 + c * 64, f0 + cw.df[tap], t0 + cw.dt[tap], cw.plane[tap] + b);
#pragma unroll
          for (int c = 0; c < BN / 64; ++c)
            ptx::tma_load_4d(sb + c * (64 * BK * 2), mb, ring.full(), t.n_blk * BN + c * 64, f0, t0, b);
          ring.advance();
          continue;
        }
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
  } else {
    ptx::reg_alloc<kConsumerRegs>();
    const int wg = (warp >> 2) - 1;
    float acc[BN / 2];
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
    consume_kblocks<BN, true, true, BF>(acc, ring, t.kb1 - t.kb0, wg, lane);
    // Both warpgroups read every slot, so the ring is free once both are past their last wgmma wait (all TMA loads of the
    // unit have landed by then).  Warpgroup wg's [64 x 256] fp32 rows go to ring.smem + 64 KB * wg (launch_wgrad_group
    // sizes the ring for both); M % 128 == 0 and N % 256 == 0 (gemm_wgrad_group): no edge tiles.
    ptx::named_bar_sync(kOrderBar, 256);
    const uint32_t stg = ring.smem + (uint32_t)wg * (64u * BN * 4u);
    stage_rows_sw128<BN>(stg, acc, grp.prob[t.gi].alpha, warp, lane);
    ptx::fence_proxy_async_smem();             // the generic-proxy stores, visible to the bulk reductions
    ptx::named_bar_sync(kEpiBar + wg, 128);
    if ((threadIdx.x & 127) == 0) reduce_add_rows_sw128<BN>(&grp.prob[t.gi].tc, stg, t.n_blk * BN, t.m_blk * BM + wg * 64);
  }
}


// =============================================================================================================
// Fused Transformer FFN forward (SURVEY K11):  x_out += dropout_post( dropout_ffn(relu(X W1 + b1)) W2 + b2 )
//   neurst/layers/common_layers.py:145-160 (TransformerFFN) inside the pre-norm wrapper (:73-85); X = LN(x_in) (16-bit),
//   x_out is pre-initialised with the residual x_in by the LayerNorm kernel.
// One CTA = (128-row tile, slice of the hidden dimension); each consumer warpgroup owns 64 of the rows.  The X tile
// (128 x D, D in {128, 256}) stays in shared memory; the hidden activations of a 64-column half are accumulated in
// registers (GEMM1), get bias, ReLU and dropout there, are written to HBM only because the backward pass needs them, and
// go, packed to 16 bits, straight back into the tensor cores as the register A operand of GEMM2, which accumulates the
// [64 x D] output rows in registers across all halves.  Only the weights stream (L2 -> smem), and the [M, ffn] hidden
// tensor is never read back.  Slices of the hidden dimension reduce into x_out with fp32 bulk reductions (dropout is a mask: linear).
//   256 threads = the two consumer warpgroups and nothing else: a CTA of at most two warpgroups is compiled to a 255-register
//   budget, which the [64 x 256] output accumulator plus the hidden fragments need for the wgmmas to stay asynchronous (with a
//   third, producer warpgroup the budget is 168 and the d = 256 accumulators spill).
//   Step s of a warpgroup issues GEMM2 of half s - 1 and GEMM1 of half s back to back and waits for both; the hidden
//   epilogue of half s follows on CUDA cores.  The two warpgroups take turns through two named barriers, as in
//   tc_gemm_kernel: warpgroup 0 issues step s once warpgroup 1 has issued step s - 1, and warpgroup 1 issues step s once
//   warpgroup 0 has, so one warpgroup's wait and epilogue run while the other's wgmmas keep the tensor cores busy.  The
//   epilogue's reads that do not depend on the accumulator (dropout-bit bytes / F1 mask words) are issued a step ahead.
//   Weight ring: item 2s = the W1 columns of half s, item 2s + 1 = the W2 rows of half s (D x 64 16-bit weights each); step
//   s reads items 2s - 1 and 2s and releases both after its wait.  Warpgroup 1 releases every item after warpgroup 0, so
//   its first thread issues the TMA loads (X once, then the refill of a stage once all eight warps have released it) and
//   warpgroup 0 never waits for a refill it did not need.  With 5 stages, the items of step s are requested when step
//   s - 3 (item 2s - 1) and step s - 2 (item 2s) release theirs.
//   smem: X 64 KB | weight ring 5 x 32 KB (after the last step: the fp32 output rows on their way to x_out)
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
constexpr int kMlpThreads = 256;
constexpr int kMlpStages = 5;
constexpr uint32_t kMlpStageBytes = 32768;     // one ring item at d = 256
constexpr uint32_t kMlpXBytes = 65536;
constexpr size_t kMlpSmem = 1024 + kMlpXBytes + kMlpStages * kMlpStageBytes + 256;
static_assert(kMlpSmem <= (size_t)kSmemLimit, "fused MLP smem");

// Timeline of the fused FFN kernel for tools/ffn_bench.py, compiled only into that tool's own library: the first thread of
// each warpgroup writes clock64 stamps to g_mlp_timeline[(blockIdx.x * 2 + warpgroup) * kMlpTlSlots + slot].  Slots: 0 / 1
// globaltimer / clock64 at entry, 2 after the X tile arrived, 3 tail start, 4 output rows staged in shared memory, 5 / 6
// clock64 / globaltimer at exit (after the bulk reductions completed); step s (0 .. H) at 8 + 6 s + e: e = 0 entry, 1 hidden epilogue done, 2 turn taken (named barrier),
// 3 ring items arrived, 4 wgmmas issued (before the wait), 5 wgmmas complete (after the W2 item's release).  No stamps are
// written while the buffer pointer is null; without the macro nothing is emitted.
#ifdef B200ST_MLP_TIMELINE
constexpr int kMlpTlSlots = 256;
__device__ unsigned long long* g_mlp_timeline;
__device__ __forceinline__ unsigned long long mlp_globaltimer() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}
#define MLP_STAMP_AT(slot, value)                                                                                       \
  do {                                                                                                                  \
    if ((threadIdx.x & 127) == 0 && g_mlp_timeline != nullptr)                                                          \
      g_mlp_timeline[((size_t)blockIdx.x * 2 + (threadIdx.x >> 7)) * kMlpTlSlots + (slot)] = (value);                 \
  } while (0)
#define MLP_STAMP(slot) MLP_STAMP_AT(slot, (unsigned long long)clock64())
#else
#define MLP_STAMP_AT(slot, value) ((void)0)
#define MLP_STAMP(slot) ((void)0)
#endif

// B_MN: weights as MN-major B operands (forward: W1 [d, ffn], W2 [ffn, d] in the TF [in, out] layout) or K-major (backward:
// the same arrays read transposed: G1 uses W2 rows = hidden units, G2 uses W1 rows = model dims)
template <int DT, bool B_MN, int D>
__global__ void __launch_bounds__(kMlpThreads, 1)
fused_mlp_fwd_kernel(const __grid_constant__ CUtensorMap tmX, const __grid_constant__ CUtensorMap tmW1,
                     const __grid_constant__ CUtensorMap tmW2, const __grid_constant__ CUtensorMap tmO, const MlpParams p) {
  extern __shared__ uint8_t smem_raw[];
  constexpr bool BF = DT == BF16;
  constexpr int kbx = D / BK;                  // k-blocks of GEMM1
  constexpr uint32_t kItemBytes = D * 128u;    // D x 64 16-bit weights
  static_assert(kItemBytes <= kMlpStageBytes, "a ring item fits one stage");
  static_assert(kMlpStages >= 4, "the refills a step waits for are issued by earlier steps' releases");
  const uint32_t base = (ptx::smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t sX = base;
  const uint32_t sW = sX + kMlpXBytes;
  const uint32_t bars = sW + kMlpStages * kMlpStageBytes;
  const uint32_t x_full = bars;
  auto w_full = [&](int s2) { return bars + 8u * (1 + s2); };
  auto w_empty = [&](int s2) { return bars + 8u * (1 + kMlpStages + s2); };

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int m_blk = blockIdx.x / p.splits, split = blockIdx.x % p.splits;
  const int H = 2 * p.chunks_per_cta;                  // 64-column hidden halves of this CTA's slice
  const int hid0 = split * p.chunks_per_cta * 128;     // first hidden unit of the slice
  const bool producer = threadIdx.x == 128;            // first thread of warpgroup 1
  MLP_STAMP_AT(0, mlp_globaltimer());
  MLP_STAMP(1);

  if (producer) {
    ptx::prefetch_tensormap(&tmX); ptx::prefetch_tensormap(&tmW1); ptx::prefetch_tensormap(&tmW2); ptx::prefetch_tensormap(&tmO);
    ptx::mbar_init(x_full, 1);
    for (int s2 = 0; s2 < kMlpStages; ++s2) { ptx::mbar_init(w_full(s2), 1); ptx::mbar_init(w_empty(s2), kConsumerWarps); }
    ptx::fence_mbar_init();
  }
  __syncthreads();
  pdl_wait();
  pdl_trigger();

  // Producer side: ring item `it` goes to stage it % kMlpStages once all 8 warps have released the item kMlpStages before
  // it.  It is called from warpgroup 1's release of that item, and warpgroup 0 releases an item before it waits for any
  // later one, so this wait never depends on a load that has not been issued yet.
  auto issue = [&](int it) {
    if (it >= 2 * H) return;
    const int st = it % kMlpStages;
    const int h0 = hid0 + (it >> 1) * 64;              // first hidden unit of the item's half
    const uint32_t dst = sW + st * kMlpStageBytes;
    ptx::mbar_wait(w_empty(st), (((uint32_t)(it / kMlpStages)) & 1u) ^ 1u);
    ptx::mbar_arrive_expect_tx(w_full(st), kItemBytes);
    if ((it & 1) == 0) {
      // GEMM1 B operand of the half: [K = d, N = 64 hidden units], one 8 KB box per k-block
      for (int kb = 0; kb < kbx; ++kb) {
        if (B_MN) ptx::tma_load_4d(dst + kb * 8192, &tmW1, w_full(st), h0, kb * BK, 0, 0);
        else ptx::tma_load_4d(dst + kb * 8192, &tmW1, w_full(st), kb * BK, h0, 0, 0);        // [64 hidden rows x 64 k]
      }
    } else {
      // GEMM2 B operand of the half: [K = 64 hidden rows, N = d]
      if (B_MN) {
        for (int i = 0; i < D / 64; ++i) ptx::tma_load_4d(dst + i * 8192, &tmW2, w_full(st), i * 64, h0, 0, 0);
      } else {
        ptx::tma_load_4d(dst, &tmW2, w_full(st), h0, 0, 0, 0);                                 // [d rows x 64 k]
      }
    }
  };
  if (producer) {
    ptx::mbar_arrive_expect_tx(x_full, (uint32_t)kbx * kABytes);
    for (int kb = 0; kb < kbx; ++kb) ptx::tma_load_4d(sX + kb * kABytes, &tmX, x_full, kb * BK, m_blk * BM, 0, 0);
    for (int it = 0; it < kMlpStages; ++it) issue(it);
  }
  __syncwarp();

  const int wg = warp >> 2, g = lane >> 2, q = lane & 3;
  const int m0 = m_blk * BM + wg * 64 + (warp & 3) * 16 + g;       // this thread's rows: m0 and m0 + 8
  const bool use_bits = B_MN && p.drop_ffn.p > 0.f;
  const bool use_mask = !B_MN && p.mask_src != nullptr;
  const float dscale = use_bits ? p.drop_ffn.scale : 1.f;
  const float hidden_floor = p.relu ? 0.f : -INFINITY;
  auto stage_get = [&](int it) {
    const int st = it % kMlpStages;
    ptx::mbar_wait(w_full(st), ((uint32_t)(it / kMlpStages)) & 1u);
    return sW + st * kMlpStageBytes;
  };
  auto release = [&](int it) {
    if (lane == 0) ptx::mbar_arrive(w_empty(it % kMlpStages));
    if (producer) issue(it + kMlpStages);
    __syncwarp();
  };
  // The epilogue's inputs of half s that do not depend on the accumulator, loaded a step before they are folded into keep
  // bits.  Forward: the dropout-bit bytes of columns n0 + 8 j (j < 8) of a row are 8 consecutive bytes, one 8-byte load;
  // backward: the 16-bit F1 pairs at the thread's fragment positions.
  uint32_t ew[2][8];
  auto load_ew = [&](int s) {
    const int n0 = hid0 + s * 64 + 2 * q;
#pragma unroll
    for (int hr = 0; hr < 2; ++hr) {
      const int m = m0 + 8 * hr;
#pragma unroll
      for (int j = 0; j < 8; ++j) ew[hr][j] = 0u;
      if (use_bits && m < p.M) {
        const uint2 w = __ldg(reinterpret_cast<const uint2*>(p.drop_ffn.bits + (((int64_t)m * p.ffn + hid0 + s * 64) >> 3)));
        ew[hr][0] = w.x; ew[hr][1] = w.y;
      }
      if (use_mask && m < p.M) {
#pragma unroll
        for (int j = 0; j < 8; ++j)
          ew[hr][j] = __ldg(reinterpret_cast<const uint32_t*>(reinterpret_cast<const uint16_t*>(p.mask_src) + (int64_t)m * p.mask_ld + n0 + 8 * j));
      }
    }
  };
  // keep bits of element pair (row m0 + 8 hr, columns n0 + 8 j + {0, 1}): bits 16 hr + 2 j + {0, 1}
  auto fold_keep = [&]() {
    uint32_t keep = 0u;
#pragma unroll
    for (int hr = 0; hr < 2; ++hr) {
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        uint32_t k2;
        if (B_MN) {
          k2 = (ew[hr][j >> 2] >> (8 * (j & 3) + 2 * q)) & 3u;
        } else {
          // 16-bit mask source (bf16 / fp16): "> 0" <=> sign clear and magnitude bits non-zero
          const uint32_t lo = ew[hr][j] & 0xffffu, hi = ew[hr][j] >> 16;
          k2 = ((lo != 0u && lo < 0x8000u) ? 1u : 0u) | ((hi != 0u && hi < 0x8000u) ? 2u : 0u);
        }
        keep |= k2 << (16 * hr + 2 * j);
      }
    }
    return keep;
  };

  float out[D / 2];
#pragma unroll
  for (int i = 0; i < D / 2; ++i) out[i] = 0.f;
  float hid[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) hid[i] = 0.f;           // the first wgmma of every GEMM1 ignores the accumulator (scale-d 0)
  uint32_t a16[4][4];
#pragma unroll
  for (int k = 0; k < 4; ++k)
#pragma unroll
    for (int i = 0; i < 4; ++i) a16[k][i] = 0u;
  float2 bias[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) bias[j] = make_float2(0.f, 0.f);
  uint32_t keep = 0u;
  // Step s; G2 / G1 are compile-time flags (false for the first / last step), so that no wgmma sits on a path the compiler
  // must treat as divergent (ptxas would serialize them).
  auto step = [&](const int s, auto G2, auto G1) {
    MLP_STAMP(8 + 6 * s);
    if constexpr (decltype(G2)::value) {
      // ---- hidden epilogue of half s - 1: bias, ReLU, dropout (forward) / relu'-dropout' mask (backward); store; pack ----
      const int n0 = hid0 + (s - 1) * 64 + 2 * q;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const int n = n0 + 8 * j;
#pragma unroll
        for (int hr = 0; hr < 2; ++hr) {
          const int m = m0 + 8 * hr;
          const bool row_ok = m < p.M;
          float v0 = fmaxf(fmaf(hid[4 * j + 2 * hr], p.alpha, bias[j].x), hidden_floor);
          float v1 = fmaxf(fmaf(hid[4 * j + 2 * hr + 1], p.alpha, bias[j].y), hidden_floor);
          const uint32_t k2 = keep >> (16 * hr + 2 * j);
          if ((use_bits || use_mask) && row_ok) {
            v0 = (k2 & 1u) ? v0 * dscale : 0.f;
            v1 = (k2 & 2u) ? v1 * dscale : 0.f;
          }
          const uint32_t pk = pack2_16(v0, v1, DT);
          if (row_ok) *reinterpret_cast<uint32_t*>(p.F1 + (int64_t)m * p.ffn + n) = pk;
          a16[j >> 1][(j & 1) * 2 + hr] = pk;
        }
      }
    }
    // ---- step s, in this warpgroup's turn: GEMM2 of half s - 1 (out[64 x D] += hidden half x W2 rows), GEMM1 of half s ----
    MLP_STAMP(8 + 6 * s + 1);
    if (G2 || wg == 1) ptx::named_bar_sync(kOrderBar + wg, 256);
    MLP_STAMP(8 + 6 * s + 2);
    const uint32_t src = G2 ? stage_get(2 * s - 1) : 0u;          // both waits before the wgmmas: none sits between them
    const uint32_t w1 = G1 ? stage_get(2 * s) : 0u;
    MLP_STAMP(8 + 6 * s + 3);
    ptx::fence_acc(out);
    ptx::fence_acc(hid);
    ptx::wgmma_fence();
    if constexpr (decltype(G2)::value) {
#pragma unroll
      for (int k = 0; k < BK / 16; ++k)
        ptx::WgmmaRS<D, BF, B_MN>::mma(out, a16[k], B_MN ? ptx::desc_mnmajor(src, k) : ptx::desc_kmajor(src, k),
                                       (s > 1 || k > 0) ? 1 : 0);
      ptx::wgmma_commit();
    }
    if constexpr (decltype(G1)::value) {
#pragma unroll
      for (int kb = 0; kb < kbx; ++kb) {
        const uint32_t sa = sX + (uint32_t)kb * kABytes + (uint32_t)wg * 8192u;
        const uint32_t sb = w1 + (uint32_t)kb * 8192u;
#pragma unroll
        for (int k = 0; k < BK / 16; ++k)
          ptx::WgmmaSS<64, BF, 0, B_MN>::mma(hid, ptx::desc_kmajor(sa, k), B_MN ? ptx::desc_mnmajor(sb, k) : ptx::desc_kmajor(sb, k),
                                             (kb > 0 || k > 0) ? 1 : 0);
      }
      ptx::wgmma_commit();
    }
    if (G1 || wg == 0) ptx::named_bar_arrive(kOrderBar + (wg ^ 1), 256);
    if constexpr (decltype(G1)::value) {
      keep = fold_keep();
      if (s + 1 < H) load_ew(s + 1);
      if (B_MN && p.b1) {
#pragma unroll
        for (int j = 0; j < 8; ++j) bias[j] = __ldg(reinterpret_cast<const float2*>(p.b1 + hid0 + s * 64 + 8 * j + 2 * q));
      }
    }
    asm volatile("" : "+r"(keep));            // folded while the wgmmas run, not after the wait
    MLP_STAMP(8 + 6 * s + 4);
    ptx::wgmma_wait<0>();
    MLP_STAMP(8 + 6 * s + 5);
    ptx::fence_acc(out);
    ptx::fence_acc(hid);
#pragma unroll
    for (int k = 0; k < 4; ++k)
#pragma unroll
      for (int i = 0; i < 4; ++i) asm volatile("" : "+r"(a16[k][i]) :: "memory");   // GEMM2 reads them until the wait
    if (G2) release(2 * s - 1);
    if (G1) release(2 * s);
  };
  load_ew(0);
  ptx::mbar_wait(x_full, 0);
  MLP_STAMP(2);
  step(0, std::false_type{}, std::true_type{});
  for (int s = 1; s < H; ++s) step(s, std::true_type{}, std::true_type{});
  step(H, std::true_type{}, std::false_type{});
  MLP_STAMP(3);
  // ---- output rows: (+ b2 on slice 0) -> post dropout -> shared memory -> TMA reduce-add into x_out ----
  // Every CTA of the wave reaches this tail at about the same time.  Per-thread 8-byte atomics (each warp instruction
  // touching 8 rows) ran at the L2's rate for such requests, about half the launch at M = 8000; staged through shared
  // memory, the tile goes out as D / 32 bulk reductions per warpgroup of [64 rows x 32 columns] each, added at L2.
  // Once both warpgroups are past their last wgmma wait no ring item is read any more, so the ring holds the staging:
  // warpgroup wg's [64 x D] fp32 rows at sW + wg * 64 * D * 4 (stage_rows_sw128).
  const bool add_b2 = split == 0 && p.b2 != nullptr;
  const bool post = p.drop_post.p > 0.f;
  const float pscale = post ? p.drop_post.scale : 1.f;
  __syncthreads();
  const uint32_t stg = sW + (uint32_t)wg * (64u * D * 4u);
  uint2 pbits[2];                              // post-dropout bytes of columns 8 j' .. 8 j' + 63 of the thread's two rows
#pragma unroll
  for (int j = 0; j < D / 8; ++j) {
    const int n = 8 * j + 2 * q;
    float2 bb = make_float2(0.f, 0.f);
    if (add_b2) bb = __ldg(reinterpret_cast<const float2*>(p.b2 + n));
#pragma unroll
    for (int hr = 0; hr < 2; ++hr) {
      const int m = m0 + 8 * hr;
      if ((j & 7) == 0)
        pbits[hr] = post && m < p.M ? __ldg(reinterpret_cast<const uint2*>(p.drop_post.bits + (((int64_t)m * p.d + 8 * j) >> 3)))
                                    : make_uint2(0u, 0u);
      float v0 = out[4 * j + 2 * hr] + bb.x, v1 = out[4 * j + 2 * hr + 1] + bb.y;
      if (post) {
        const uint32_t kb = ((j & 4) ? pbits[hr].y : pbits[hr].x) >> (8 * (j & 3) + 2 * q);
        v0 = (kb & 1u) ? v0 * pscale : 0.f;
        v1 = (kb & 2u) ? v1 * pscale : 0.f;
      }
      out[4 * j + 2 * hr] = v0;
      out[4 * j + 2 * hr + 1] = v1;
    }
  }
  stage_rows_sw128<D>(stg, out, 1.f, warp, lane);   // rows >= M are staged but not added
  ptx::fence_proxy_async_smem();               // the generic-proxy stores, visible to the bulk reductions
  ptx::named_bar_sync(kEpiBar + wg, 128);
  MLP_STAMP(4);
  const bool ordered = p.tickets && p.splits > 1;
  if ((threadIdx.x & 127) == 0) {
    if (ordered) {
      // deterministic reduction order: slice s adds only after slices 0 .. s-1 of this row tile have completed theirs
      const volatile int* tk = p.tickets + m_blk;
      while (*tk != split) { }
      __threadfence();
      asm volatile("fence.proxy.async.global;" ::: "memory");
    }
    reduce_add_rows_sw128<D>(&tmO, stg, 0, m_blk * BM + wg * 64);
    if (ordered) {
      asm volatile("fence.proxy.async.global;" ::: "memory");
      __threadfence();
    }
  }
  if (ordered) {
    __syncthreads();                           // both warpgroups' reductions have completed
    if (threadIdx.x == 0) atomicExch(p.tickets + m_blk, split + 1 == p.splits ? 0 : split + 1);
  }
  MLP_STAMP(5);
  MLP_STAMP_AT(6, mlp_globaltimer());
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

// fp32 [M, d] row-major output (rows ld floats apart) of the fused FFN, grouped weight-gradient and fp32 GEMM kernels: [64 rows
// x 32 columns] boxes, 128B swizzle (bulk store / reduce-add target; stage_rows_sw128 writes the layout; boxes are clipped)
int make_out_map_f32(float* ptr, int M, int d, int64_t ld, CUtensorMap* out) {
  EncodeTiledFn fn = get_encode_fn();
  B200ST_CHECK(fn != nullptr, "cuTensorMapEncodeTiled unavailable (no CUDA driver?)");
  B200ST_CHECK((reinterpret_cast<uintptr_t>(ptr) & 15) == 0 && ld >= d && ld % 4 == 0, "fp32 output map: unaligned base or row stride");
  cuuint64_t dims[2] = {(cuuint64_t)d, (cuuint64_t)M};
  cuuint64_t strides[1] = {(cuuint64_t)ld * 4};
  cuuint32_t box[2] = {32u, 64u};
  cuuint32_t estr[2] = {1u, 1u};
  MapKey key{{(uint64_t)(uintptr_t)ptr, (uint64_t)d, (uint64_t)M, 1, 1, strides[0], 0, 0, box[1], (uint64_t)F32 << 8 | 0x10000u}};
  {
    std::lock_guard<std::mutex> lk(g_map_mu);
    auto it = g_map_cache.find(key);
    if (it != g_map_cache.end()) { *out = it->second; return 0; }
  }
  CUresult r = fn(out, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, ptr, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                  CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) B200ST_FAIL("cuTensorMapEncodeTiled failed with CUresult " + std::to_string((int)r));
  std::lock_guard<std::mutex> lk(g_map_mu);
  if (g_map_cache.size() > 65536) g_map_cache.clear();
  g_map_cache.emplace(key, *out);
  return 0;
}

// [planes][T2][F2][C] 16-bit activation as a 4-D tensor (C, F2, T2, planes) with a {64, box_f, box_t, 1} box, 128B swizzle.
// Boxes that reach outside the tensor (negative or past-the-end shifted coordinates) are zero-filled: the conv's border.
int make_conv_map(const void* ptr, int dtype, int C, int F2, int T2, int planes, int box_f, int box_t, CUtensorMap* out) {
  EncodeTiledFn fn = get_encode_fn();
  B200ST_CHECK(fn != nullptr, "cuTensorMapEncodeTiled unavailable (no CUDA driver?)");
  B200ST_CHECK((reinterpret_cast<uintptr_t>(ptr) & 15) == 0, "TMA operand base must be 16-byte aligned");
  cuuint64_t dims[4] = {(cuuint64_t)C, (cuuint64_t)F2, (cuuint64_t)T2, (cuuint64_t)planes};
  cuuint64_t strides[3] = {(cuuint64_t)C * 2, (cuuint64_t)F2 * C * 2, (cuuint64_t)T2 * F2 * C * 2};
  cuuint32_t box[4] = {(cuuint32_t)BK, (cuuint32_t)box_f, (cuuint32_t)box_t, 1u};
  cuuint32_t estr[4] = {1u, 1u, 1u, 1u};
  CUresult r = fn(out, dtype == F16 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, const_cast<void*>(ptr),
                  dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) B200ST_FAIL("cuTensorMapEncodeTiled (conv operand) failed with CUresult " + std::to_string((int)r));
  return 0;
}

int g_num_sms = 0;
int g_reserved_sms = 0;

// SMs a persistent grid may fill: the device's, less those reserved for communication kernels (set_reserved_sms)
int usable_sms(int* out) {
  if (g_num_sms == 0) {
    int dev = 0;
    B200ST_CUDA(cudaGetDevice(&dev));
    B200ST_CUDA(cudaDeviceGetAttribute(&g_num_sms, cudaDevAttrMultiProcessorCount, dev));
  }
  *out = g_reserved_sms > 0 && g_reserved_sms < g_num_sms ? g_num_sms - g_reserved_sms : g_num_sms;
  return 0;
}
}  // namespace

// 16-bit 4-D tensor map (inner, rows, nb1, nb2) with a {box_inner<=64, box_rows} box, 128B swizzle.
int make_tma_map_16(const void* ptr, int dtype, uint64_t inner, uint64_t rows, int nb1, int nb2, int64_t ld, int64_t sb1, int64_t sb2,
                    uint32_t box_rows, CUtensorMap* out) {
  GemmOperand op{ptr, dtype, 0, ld, sb1, sb2};
  return make_operand_map(op, (int)rows, (int)inner, nb1, nb2, (int)box_rows, out);
}

namespace {

// optional GEMM profile (bench.py roofline pass; off in the timed region): every tensor-core GEMM issued between begin and
// end is RECORDED (arguments only); tc_profile_end() then replays each recorded GEMM back to back (1 warm-up + kReps timed
// launches bracketed by one event pair, no host gap between them) and reports the per-launch average.  The buffers of the
// step are still alive (same workspace), accumulate / reduce epilogues only add into gradients nobody reads afterwards.
// Implicit conv2 GEMM (conv2_fwd_implicit, conv2_dgrad_implicit, conv2_wgrad_implicit): replaces the operand tensor maps and
// the k-block -> coordinates rule.  x: [planes][T2][F2][C] (dY: one plane per utterance; the parity-split activation: 4 B
// planes, class-major); dy: the wgrad's B operand dZ2 [B, T2, F2, C].
struct ConvA {
  int mode;                              // kConvRows or kConvWgrad
  const void* x; int planes, T2, F2, C;
  const void* dy; int B;
  int tu, ub, remap;                     // kConvRows
  int ntaps;
  int dt[9], df[9], wrow[9], plane[9];
  int tap0[4], ntap[4];                  // data gradient: each parity class's taps (TcParams::conv_tap0 ...)
  int64_t cls_elems;
};
struct ProfRec { GemmArgs g; cudaStream_t stream; int bn, splitk; int group_n = 0; GemmArgs rest[3]; bool has_conv = false; ConvA conv; };   // group_n > 1: grouped weight-gradient launch (g + rest)
bool g_prof = false;
std::vector<ProfRec> g_prof_recs;

// tc: the fp32 C map of a tc_gemm_f32_kernel launch, or null
template <int BN, bool A_MN, bool B_MN, bool BF, bool CONV>
int launch_kernel(const CUtensorMap& ta, const CUtensorMap& tb, const CUtensorMap* tc, const TcParams& p, int grid, size_t smem,
                  cudaStream_t stream) {
  if constexpr (!CONV) {
    if (tc) {
      auto kf = tc_gemm_f32_kernel<BN, A_MN, B_MN, BF>;
      static bool attr_f32 = false;
      if (!attr_f32) {
        B200ST_CUDA(cudaFuncSetAttribute(kf, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemLimit));
        attr_f32 = true;
      }
      return launch(kf, grid, kThreads, smem, stream, ta, tb, *tc, p);
    }
  }
  void (*kern)(const CUtensorMap, const CUtensorMap, const TcParams);
  if constexpr (CONV) kern = tc_gemm_conv_kernel<B_MN, BF>;
  else kern = tc_gemm_kernel<BN, A_MN, B_MN, BF>;
  static bool attr_set = false;
  if (!attr_set) {
    B200ST_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemLimit));
    attr_set = true;
  }
  return launch(kern, grid, kThreads, smem, stream, ta, tb, p);
}

template <int BN, bool A_MN, bool B_MN, bool CONV = false>
int launch_variant(bool bf, const CUtensorMap& ta, const CUtensorMap& tb, const CUtensorMap* tc, const TcParams& p, int grid, size_t smem,
                   cudaStream_t stream) {
  if (bf) return launch_kernel<BN, A_MN, B_MN, true, CONV>(ta, tb, tc, p, grid, smem, stream);
  return launch_kernel<BN, A_MN, B_MN, false, CONV>(ta, tb, tc, p, grid, smem, stream);
}

template <int BN>
int launch_bn(bool a_mn, bool b_mn, bool bf, const CUtensorMap& ta, const CUtensorMap& tb, const CUtensorMap* tc, const TcParams& p, int grid,
              size_t smem, cudaStream_t stream) {
  if (!a_mn && !b_mn) return launch_variant<BN, false, false>(bf, ta, tb, tc, p, grid, smem, stream);
  if (!a_mn && b_mn) return launch_variant<BN, false, true>(bf, ta, tb, tc, p, grid, smem, stream);
  if (a_mn && !b_mn) return launch_variant<BN, true, false>(bf, ta, tb, tc, p, grid, smem, stream);
  return launch_variant<BN, true, true>(bf, ta, tb, tc, p, grid, smem, stream);
}

}  // namespace

void set_reserved_sms(int n) { g_reserved_sms = n; }

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
  int num_sms = 0;
  B200ST_TRY(usable_sms(&num_sms));

  TcParams p{};
  p.M = g.M; p.N = g.N; p.K = g.K; p.nb1 = g.nb1; p.nb2 = g.nb2;
  p.m_tiles = ceil_div(g.M, BM);
  p.kb_total = ceil_div(g.K, BK);
  const int64_t batch = (int64_t)g.nb1 * g.nb2;

  // ---- joint choice of the N tile and the split-K factor ----
  // Cost model of a CTA's share of the tiles.  Main loop of one tile, per k-block: max(tensor time, L2->smem fill time): the
  // wgmmas of a 128 x c x 64 block take about 4c cycles, the operand bytes (16 KB + 128c B) are assumed to arrive at
  // ~44 B/cycle/SM (an estimate, not measured on H100).  The two consumer warpgroups take turns on the tensor cores, so a
  // tile's epilogue (one warpgroup, 128 rows) hides under the other warpgroup's main loop as far as that is long enough.
  // Split-K (fp32 atomic epilogue) is allowed for linear accumulate epilogues only and is chosen so that the tile count fills
  // the SMs once.
  const bool linear_epi = !g.epi.relu && !g.epi.mask_src && g.epi.drop.p == 0.f && !g.epi.residual && !g.epi.bias;
  const bool split_ok = linear_epi && g.c_dtype == F32 && g.epi.accumulate;
  if (g.splitk > 1) B200ST_CHECK(split_ok, "split-K needs a linear fp32 accumulate epilogue");
  int bn = 0, splitk = g.splitk >= 1 ? g.splitk : 1;
  {
    double best = 1e30;
    int best_bn = 0, best_sk = 1;
    const int cands[2] = {128, 64};
    for (int c : cands) {
      if (conv && c != 128) continue;
      if (c > 64 && c >= 2 * ((g.N + 63) / 64 * 64)) continue;   // do not pad N by 2x or more
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
        const int64_t per_cta = (tiles + num_sms - 1) / num_sms;
        const double fill = (16384.0 + 128.0 * c) / 44.0, mma = 4.0 * c;
        const double mainloop = kb_per * (fill > mma ? fill : mma);
        const double epi = (sk > 1 ? 28.0 : 20.0) * c + 600.0;
        const double per_tile = mainloop > 0.5 * (mainloop + epi) ? mainloop : 0.5 * (mainloop + epi);
        const double cost = (double)per_cta * per_tile + 0.5 * epi + 800.0 + (sk > 1 ? 500.0 : 0.0);
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
  int stages = (int)((kSmemLimit - 2048 - 2 * staging_bytes(bn)) / stage_bytes);
  if (stages > 8) stages = 8;
  if (stages < 2) stages = 2;      // consume_tile keeps one slot in flight before it releases the previous one
  p.stages = stages;
  const size_t smem = 1024 + (size_t)stages * stage_bytes + 2 * staging_bytes(bn) + 16 * stages + 16;
  B200ST_CHECK(smem <= (size_t)kSmemLimit, "smem budget exceeded");

  p.C = g.C; p.c_dtype = g.c_dtype; p.ldc = g.ldc; p.c_sb1 = g.c_sb1; p.c_sb2 = g.c_sb2;
  p.epi = g.epi;
  if (g.epi.accumulate) B200ST_CHECK(g.c_dtype == F32, "accumulate needs fp32 C");
  p.atomic = (splitk > 1 || g.epi.accumulate) ? 1 : 0;
  // paired stores / atomics need every (row, even column) element of C 8-byte (fp32) or 4-byte (16-bit) aligned
  const uintptr_t pair_bytes = g.c_dtype == F32 ? 8 : 4;
  p.vec2 = ((reinterpret_cast<uintptr_t>(g.C) % pair_bytes) == 0 && g.ldc % 2 == 0 && (g.nb1 == 1 || g.c_sb1 % 2 == 0) &&
            (g.nb2 == 1 || g.c_sb2 % 2 == 0)) ? 1 : 0;
  p.plain16 = (!p.atomic && g.c_dtype != F32 && p.vec2 && !g.epi.relu && !g.epi.mask_src && g.epi.drop.p == 0.f && !g.epi.residual) ? 1 : 0;
  // fp32 C of a non-batched GEMM that fits a tensor map, epilogue alpha (+ bias unless added): tc_gemm_f32_kernel's bulk
  // stores or, for split-K / accumulate, bulk reduce-adds instead of the general loop's per-element stores and atomics
  const bool f32c = g.c_dtype == F32 && !conv && g.nb1 == 1 && g.nb2 == 1 && (reinterpret_cast<uintptr_t>(g.C) & 15) == 0 &&
                    g.ldc >= g.N && g.ldc % 4 == 0 && !g.epi.relu && !g.epi.mask_src && g.epi.drop.p == 0.f && !g.epi.residual &&
                    !(p.atomic && g.epi.bias);
  p.c_reduce = p.atomic;

  CUtensorMap ta, tb, tc;
  if (f32c) B200ST_TRY(make_out_map_f32(reinterpret_cast<float*>(g.C), g.M, g.N, g.ldc, &tc));
  if (conv) {
    B200ST_CHECK(conv->mode == kConvRows && bn == 128 && splitk == 1 && !g.A.mn_major && g.nb1 == 1 && g.nb2 == 1 && conv->C % BK == 0 && conv->ntaps <= 9 &&
                     g.K == conv->ntaps * conv->C && g.M == conv->B * conv->ub * BM && conv->F2 * conv->tu <= BM &&
                     (!conv->remap || p.plain16),
                 "implicit conv2 GEMM: unsupported shape");
    p.conv_ub = conv->ub; p.conv_tu = conv->tu; p.conv_kpc = conv->C / BK;
    p.conv_remap = conv->remap; p.conv_T2 = conv->T2; p.conv_F2 = conv->F2;
    for (int i = 0; i < conv->ntaps; ++i) {
      p.conv_dt[i] = conv->dt[i]; p.conv_df[i] = conv->df[i]; p.conv_wrow[i] = conv->wrow[i]; p.conv_plane[i] = conv->plane[i];
    }
    p.conv_a_bytes = (uint32_t)(BK * conv->F2 * conv->tu * 2);
    if (!g.B.mn_major) {
      // data gradient: g.K is the four classes' K together (9 C), the tiles are the four class tiles of every unit
      for (int c = 0; c < 4; ++c) { p.conv_tap0[c] = conv->tap0[c]; p.conv_ntap[c] = conv->ntap[c]; }
      p.conv_cls_elems = conv->cls_elems;
      p.num_tiles = 4 * (int64_t)p.m_tiles * p.n_tiles;
    }
    // A: one box = 64 channels x all F2 frequencies x tu time rows of one plane
    B200ST_TRY(make_conv_map(conv->x, g.A.dtype, conv->C, conv->F2, conv->T2, conv->planes, conv->F2, conv->tu, &ta));
    // B: all 9 taps of the [9C, C] weight matrix (K-major for the data gradient, MN-major for the forward)
    if (g.B.mn_major) B200ST_TRY(make_operand_map(g.B, conv->C, 9 * conv->C, 1, 1, bn, &tb));
    else B200ST_TRY(make_operand_map(g.B, 9 * conv->C, conv->C, 1, 1, bn, &tb));
  } else {
    B200ST_TRY(make_operand_map(g.A, g.M, g.K, g.nb1, g.nb2, BM, &ta));
    B200ST_TRY(make_operand_map(g.B, g.N, g.K, g.nb1, g.nb2, bn, &tb));
  }

  const int max_grid = num_sms;
  const int grid = (int)(p.num_tiles < max_grid ? p.num_tiles : max_grid);
  if (g_prof) {
    ProfRec r{g, stream, bn, splitk};
    if (conv) { r.has_conv = true; r.conv = *conv; }
    g_prof_recs.push_back(r);
  }
  int rc = 0;
  const bool bf = g.A.dtype == BF16;
  if (conv) {
    if (g.B.mn_major) return launch_variant<128, false, true, true>(bf, ta, tb, nullptr, p, grid, smem, stream);
    return launch_variant<128, false, false, true>(bf, ta, tb, nullptr, p, grid, smem, stream);
  }
  switch (bn) {
    case 64: rc = launch_bn<64>(g.A.mn_major, g.B.mn_major, bf, ta, tb, f32c ? &tc : nullptr, p, grid, smem, stream); break;
    case 128: rc = launch_bn<128>(g.A.mn_major, g.B.mn_major, bf, ta, tb, f32c ? &tc : nullptr, p, grid, smem, stream); break;
    default: B200ST_FAIL("unsupported BN");
  }
  return rc;
}
}  // namespace

// Conv2D#2 of AudioConv2dSubsamplingLayer (neurst/layers/modalities/audio_modalities.py:96-104): 3x3, stride 2, pad 1, as
// implicit GEMMs.  Tap (kh, kw) of output position (t2, f2) reads input position (2 t2 + kh - 1, 2 f2 + kw - 1); stored split
// by parity class cls = ((t1 & 1) << 1) | (f1 & 1) at plane position (t1 >> 1, f1 >> 1), that is plane position
// (t2 + dt, f2 + df) of class plane cls with dt = -1 for kh = 0 and 0 otherwise (df alike) — dense unit-stride boxes
// shifted per tap.  conv1's forward writes the activation in that layout (conv_kernels.cu), zero at the class positions
// past the image.
static void conv2_fwd_taps(ConvA& ca, int B, int C) {
  ca.ntaps = 9;
  for (int kh = 0; kh < 3; ++kh)
    for (int kw = 0; kw < 3; ++kw) {
      const int tap = kh * 3 + kw, cls = ((kh != 1) << 1) | (kw != 1);
      ca.dt[tap] = kh == 0 ? -1 : 0; ca.df[tap] = kw == 0 ? -1 : 0;
      ca.wrow[tap] = tap * C; ca.plane[tap] = cls * B;
    }
}

// z2[b, t2, f2, :] = bias + sum over taps of a1_tap W[tap]: a 128-row tile = tu = 128 / F2 time rows of one utterance, k-blocks
// in the (kh, kw, channel) order of the explicit column matrix, so every output element sums the same products in the same
// order as the explicit GEMM did.
int conv2_fwd_implicit(const void* a1, const void* w16, const float* bias, void* z2, int dtype, int B, int T2, int F2, int C,
                       cudaStream_t stream) {
  B200ST_CHECK(is16(dtype) && C == 256 && F2 >= 1 && F2 <= BM, "implicit conv2 forward: 16-bit, C == 256, F2 <= 128");
  ConvA ca{};
  ca.mode = kConvRows; ca.x = a1; ca.planes = 4 * B; ca.T2 = T2; ca.F2 = F2; ca.C = C; ca.B = B;
  ca.tu = BM / F2; ca.ub = ceil_div(T2, ca.tu); ca.remap = 1;
  conv2_fwd_taps(ca, B, C);
  GemmArgs g = gemm_defaults();
  g.M = B * ca.ub * BM; g.N = C; g.K = 9 * C;
  g.A = GemmOperand{a1, dtype, 0, C, 0, 0};
  g.B = GemmOperand{w16, dtype, 1, C, 0, 0};
  g.C = z2; g.c_dtype = dtype; g.ldc = C;
  g.epi.bias = bias;
  return gemm_tc_impl(g, stream, &ca);
}

// dW[(kh, kw, ci), co] += sum over positions p of a1_tap(p)[ci] dZ2[p][co]: both operands MN-major, a k-block = a chunk of whole
// time rows x F2 frequencies of one utterance (F2 <= 64: 64 / F2 rows; 64 < F2 <= 128: one row in two halves of 64).
// Split-K with fp32 atomics; all work units run in one wave and walk their k ranges in step, so the 18 m tiles (9 taps x 2
// channel halves) of a k range read the four class planes of the same positions at about the same time, from L2.
namespace { int conv_wgrad_launch(const GemmArgs& g, const ConvA& ca, cudaStream_t stream); }
int conv2_wgrad_implicit(const void* a1, const void* dz2, float* dw, int dtype, int B, int T2, int F2, int C, cudaStream_t stream) {
  B200ST_CHECK(is16(dtype) && C == 256 && F2 >= 1 && F2 <= BM, "implicit conv2 filter gradient: 16-bit, C == 256, F2 <= 128");
  ConvA ca{};
  ca.mode = kConvWgrad; ca.x = a1; ca.planes = 4 * B; ca.T2 = T2; ca.F2 = F2; ca.C = C; ca.dy = dz2; ca.B = B;
  conv2_fwd_taps(ca, B, C);
  const int kt = F2 < BK ? BK / F2 : 1, fc = F2 <= BK ? 1 : 2;
  GemmArgs g = gemm_defaults();
  g.M = 9 * C; g.N = C; g.K = B * ceil_div(T2, kt) * fc * BK;
  g.A = GemmOperand{a1, dtype, 1, 9 * C, 0, 0};
  g.B = GemmOperand{dz2, dtype, 1, C, 0, 0};
  g.C = dw; g.c_dtype = F32; g.ldc = C;
  g.epi.accumulate = 1;
  return conv_wgrad_launch(g, ca, stream);
}

// Data gradient of the same convolution as one implicit GEMM launch over the four parity classes (t1 & 1, f1 & 1) of the input
// position: dA[b, t1, f1, :] = sum over the taps (kh, kw) with t1 = 2 t2 + kh - 1, f1 = 2 f2 + kw - 1 of dY[b, t2, f2, :]
// W[kh, kw]^T — 1 tap for (even, even), 2 for the mixed classes, 4 for (odd, odd), 9 in all.  The A operand is read straight
// out of dY by 4-D TMA boxes shifted by the tap (zero fill = border), so neither the [rows, 9C] column gradient (737 MB at
// cfg-2) nor its col2im gather exist.  The four class tiles of one (row tile, n tile) are consecutive tiles of one CTA
// (dgrad_first_tile), so they share their dY rows in L2.  Output: class-major padded tiles
//   dA[cls][b][tile][128 rows = tu x F2 positions (+ unused rows)][C],   tile = (t1 >> 1) / tu,   row = ((t1 >> 1) % tu) * F2 + (f1 >> 1)
// which conv1's backward kernel reads back with the same arithmetic.
int conv2_dgrad_implicit(const void* dy, const void* w16, void* da, int dtype, int B, int T2, int F2, int C, cudaStream_t stream) {
  B200ST_CHECK(is16(dtype) && C == 256 && F2 >= 1 && F2 <= BM, "implicit conv2 dgrad: 16-bit, C == 256, F2 <= 128");
  ConvA ca{};
  ca.mode = kConvRows; ca.x = dy; ca.planes = B; ca.B = B; ca.T2 = T2; ca.F2 = F2; ca.C = C;
  ca.tu = BM / F2;
  ca.ub = ceil_div(T2, ca.tu);
  ca.cls_elems = (int64_t)B * ca.ub * BM * C;
  ca.ntaps = 0;
  for (int cls = 0; cls < 4; ++cls) {
    const int pt = cls >> 1, pf = cls & 1;
    // per axis: even position -> centre tap, same index; odd position -> tap 2 at the same index and tap 0 at index + 1
    const int nt = pt ? 2 : 1, nf = pf ? 2 : 1;
    const int kh_of[2] = {pt ? 2 : 1, 0}, dt_of[2] = {0, 1};
    const int kw_of[2] = {pf ? 2 : 1, 0}, df_of[2] = {0, 1};
    ca.tap0[cls] = ca.ntaps;
    ca.ntap[cls] = nt * nf;
    for (int a = 0; a < nt; ++a)
      for (int b2 = 0; b2 < nf; ++b2) {
        const int i = ca.ntaps++;
        ca.dt[i] = dt_of[a]; ca.df[i] = df_of[b2]; ca.wrow[i] = (kh_of[a] * 3 + kw_of[b2]) * C; ca.plane[i] = 0;
      }
  }
  GemmArgs g = gemm_defaults();
  g.M = B * ca.ub * BM; g.N = C; g.K = ca.ntaps * C;      // M per class; K = the classes' K together (profile FLOPs 2 M N K)
  g.A = GemmOperand{dy, dtype, 0, C, 0, 0};
  g.B = GemmOperand{w16, dtype, 0, C, 0, 0};
  g.C = da; g.c_dtype = dtype; g.ldc = C;
  return gemm_tc_impl(g, stream, &ca);
}
int64_t conv2_dgrad_implicit_elems(int B, int T2, int F2, int C) {
  const int tu = BM / F2;
  return 4 * (int64_t)B * ceil_div(T2, tu) * BM * C;
}


// One launch for the weight gradients of a backward block (see tc_wgrad_group_kernel).  Every product must be a plain
// fp32-accumulate MN-major x MN-major 16-bit GEMM with M % 128 == 0 and N % 256 == 0, whose C fits an fp32 tensor map, and
// the group's output tiles must fit one wave; gemm_wgrad_group returns 2 (nothing launched) when the group does not
// qualify, so that the caller issues the products one by one.
// Output tiles of the group's products: at most one wave, since every tile is at least one work unit.
static int64_t wgrad_group_tiles(const TcGroup& grp) {
  int64_t tiles = 0;
  for (int i = 0; i < grp.n; ++i) tiles += (int64_t)grp.prob[i].m_tiles * grp.prob[i].n_tiles;
  return tiles;
}
// Splits the products of `grp` (tensor maps and alpha set; m_tiles, n_tiles and kb_total given) into work units of one
// common k-range length and launches them as one wave, one unit per CTA: the kernel's tail stages the unit's sums in the
// operand ring, which is only drained for good when no further unit follows.
static int launch_wgrad_group(TcGroup& grp, bool bf, cudaStream_t stream) {
  int num_sms = 0;
  B200ST_TRY(usable_sms(&num_sms));
  B200ST_CHECK(wgrad_group_tiles(grp) <= num_sms, "grouped weight gradient: more output tiles than SMs");
  int64_t work = 0;
  for (int i = 0; i < grp.n; ++i) work += (int64_t)grp.prob[i].m_tiles * grp.prob[i].n_tiles * grp.prob[i].kb_total;
  // smallest common k-range L (in 64-row blocks) whose work units fit one wave of `num_sms` CTAs; it exists (at the longest
  // product's kb_total every product is one unit per tile)
  int L = (int)((work + num_sms - 1) / num_sms);
  if (L < 2) L = 2;
  for (;; ++L) {
    int64_t units = 0;
    for (int i = 0; i < grp.n; ++i) units += (int64_t)grp.prob[i].m_tiles * grp.prob[i].n_tiles * ceil_div(grp.prob[i].kb_total, L);
    if (units <= num_sms) break;
  }
  int tile = 0;
  for (int i = 0; i < grp.n; ++i) {
    TcGroupProb& q = grp.prob[i];
    q.kb_per_split = L < q.kb_total ? L : q.kb_total;
    q.splitk = ceil_div(q.kb_total, q.kb_per_split);
    q.tile_begin = tile;
    tile += q.m_tiles * q.n_tiles * q.splitk;
  }
  grp.num_tiles = tile;
  B200ST_CHECK(grp.num_tiles <= num_sms, "grouped weight gradient: one work unit per CTA");
  const uint32_t stage_bytes = kABytes + 256u * BK * 2;
  int stages = (int)((kSmemLimit - 2048) / stage_bytes);
  if (stages > 8) stages = 8;
  grp.stages = stages;
  const size_t smem = 1024 + (size_t)stages * stage_bytes + 16 * stages + 16;
  B200ST_CHECK(smem <= (size_t)kSmemLimit, "smem budget exceeded");
  B200ST_CHECK((size_t)stages * stage_bytes >= 2 * 64 * 256 * 4, "grouped weight gradient: the ring holds both warpgroups' output rows");
  auto kern = bf ? tc_wgrad_group_kernel<true> : tc_wgrad_group_kernel<false>;
  static bool attr_set[2] = {false, false};
  if (!attr_set[bf]) {
    B200ST_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemLimit));
    attr_set[bf] = true;
  }
  return launch(kern, grp.num_tiles, kThreads, smem, stream, grp);
}

int gemm_wgrad_group(const GemmArgs* gs, int n, cudaStream_t stream) {
  if (n < 2 || n > kMaxGroup) return 2;
  for (int i = 0; i < n; ++i) {
    const GemmArgs& g = gs[i];
    const bool plain = !g.epi.relu && !g.epi.mask_src && g.epi.drop.p == 0.f && !g.epi.residual && !g.epi.bias && g.epi.accumulate;
    if (!(is16(g.A.dtype) && g.A.dtype == g.B.dtype && g.A.dtype == gs[0].A.dtype && g.A.mn_major && g.B.mn_major && plain &&
          g.c_dtype == F32 && g.nb1 == 1 && g.nb2 == 1 && g.M % BM == 0 && g.N % 256 == 0 && g.K > 0 && g.splitk <= 1 &&
          (reinterpret_cast<uintptr_t>(g.C) & 15) == 0 && g.ldc >= g.N && g.ldc % 4 == 0))     // C fits an fp32 tensor map
      return 2;
  }
  TcGroup grp;
  std::memset(&grp, 0, sizeof(grp));
  grp.n = n;
  for (int i = 0; i < n; ++i) {
    grp.prob[i].m_tiles = gs[i].M / BM;
    grp.prob[i].n_tiles = gs[i].N / 256;
  }
  int num_sms = 0;
  B200ST_TRY(usable_sms(&num_sms));
  if (wgrad_group_tiles(grp) > num_sms) return 2;
  for (int i = 0; i < n; ++i) {
    const GemmArgs& g = gs[i];
    TcGroupProb& q = grp.prob[i];
    q.kb_total = ceil_div(g.K, BK);
    q.alpha = g.epi.alpha;
    B200ST_TRY(make_operand_map(g.A, g.M, g.K, 1, 1, BM, &q.ta));
    B200ST_TRY(make_operand_map(g.B, g.N, g.K, 1, 1, 256, &q.tb));
    B200ST_TRY(make_out_map_f32(reinterpret_cast<float*>(g.C), g.M, g.N, g.ldc, &q.tc));
  }
  B200ST_TRY(launch_wgrad_group(grp, gs[0].A.dtype == BF16, stream));
  if (g_prof) {
    ProfRec r{gs[0], stream, 256, grp.prob[0].splitk};
    r.group_n = n;
    for (int i = 1; i < n; ++i) r.rest[i - 1] = gs[i];
    g_prof_recs.push_back(r);
  }
  return 0;
}

namespace {
// dW[(kh, kw, ci), co] += sum over positions of a1_tap[ci] dZ2[co] as one tc_wgrad_group_kernel product (128 x 256 tiles: each
// k-block of the two operands feeds twice the MMA work of a 128 x 128 tile, which sets this GEMM's time: it is bound by
// operand traffic from L2, not by HBM)
int conv_wgrad_launch(const GemmArgs& g, const ConvA& ca, cudaStream_t stream) {
  B200ST_CHECK(ca.mode == kConvWgrad && is16(g.A.dtype) && g.A.dtype == g.B.dtype && ca.C % BM == 0 && ca.ntaps == 9 &&
                   g.M == 9 * ca.C && g.N == ca.C && ca.C % 256 == 0 && ca.F2 >= 1 && ca.F2 <= 2 * BK && g.c_dtype == F32,
               "implicit conv2 filter gradient: unsupported shape");
  const int fw = ca.F2 < BK ? ca.F2 : BK, kt = ca.F2 < BK ? BK / ca.F2 : 1;
  TcGroup grp;
  std::memset(&grp, 0, sizeof(grp));
  grp.n = 1;
  ConvWgrad& cw = grp.cw;
  cw.on = 1; cw.kpc = ca.C / BM; cw.fw = fw; cw.kt = kt; cw.fc = ceil_div(ca.F2, fw); cw.krows = fw * kt;
  cw.kc = ceil_div(ca.T2, kt) * cw.fc;
  for (int i = 0; i < 9; ++i) { cw.dt[i] = ca.dt[i]; cw.df[i] = ca.df[i]; cw.plane[i] = ca.plane[i]; }
  TcGroupProb& q = grp.prob[0];
  q.m_tiles = g.M / BM; q.n_tiles = g.N / 256; q.kb_total = ca.B * cw.kc;
  B200ST_CHECK(ceil_div(g.K, BK) == q.kb_total, "implicit conv2 filter gradient: k-blocks do not match the chunking");
  q.alpha = g.epi.alpha;
  B200ST_TRY(make_out_map_f32(reinterpret_cast<float*>(g.C), g.M, g.N, g.ldc, &q.tc));
  B200ST_TRY(make_conv_map(ca.x, g.A.dtype, ca.C, ca.F2, ca.T2, ca.planes, fw, kt, &q.ta));
  B200ST_TRY(make_conv_map(ca.dy, g.B.dtype, ca.C, ca.F2, ca.T2, ca.B, fw, kt, &q.tb));
  B200ST_TRY(launch_wgrad_group(grp, g.A.dtype == BF16, stream));
  if (g_prof) {
    ProfRec r{g, stream, 256, q.splitk};
    r.has_conv = true; r.conv = ca;
    g_prof_recs.push_back(r);
  }
  return 0;
}
}  // namespace


// Fused FFN forward (see fused_mlp_fwd_kernel).  X: 16-bit [M, d] (LayerNorm output); W1 [d, ffn], W2 [ffn, d] in the same
// 16-bit type (TF layouts); F1 out [M, ffn] (saved for the backward pass); x_out fp32 [M, d] must already hold the residual.
bool fused_mlp_supported(int M, int d, int ffn, int dtype) {
  return is16(dtype) && (d == 128 || d == 256) && ffn % 128 == 0 && M > 0;
}
// slices of the hidden dimension: the most CTAs that still fit one wave, with an equal number of chunks per slice
static int mlp_splits(int m_tiles, int chunks, int* splits) {
  int num_sms = 0;
  B200ST_TRY(usable_sms(&num_sms));
  *splits = 1;
  for (int s = 1; s <= chunks; ++s)
    if (chunks % s == 0 && (int64_t)m_tiles * s <= num_sms) *splits = s;
  return 0;
}
int fused_mlp_fwd(const void* X, int dtype, int M, int d, int ffn, const void* W1, const float* b1, const void* W2, const float* b2,
                  DropoutSpec drop_ffn, DropoutSpec drop_post, void* F1, float* x_out, cudaStream_t stream, int* tickets) {
  B200ST_CHECK(fused_mlp_supported(M, d, ffn, dtype), "fused MLP: unsupported shape / dtype");
  if (drop_ffn.p > 0.f)
    B200ST_CHECK(drop_ffn.bits != nullptr && (reinterpret_cast<uintptr_t>(drop_ffn.bits) & 7) == 0,
                 "fused MLP needs precomputed, 8-byte aligned dropout bits");
  if (drop_post.p > 0.f)
    B200ST_CHECK(drop_post.bits != nullptr && (reinterpret_cast<uintptr_t>(drop_post.bits) & 7) == 0,
                 "fused MLP needs precomputed, 8-byte aligned dropout bits");
  const int m_tiles = ceil_div(M, BM), chunks = ffn / 128;
  int splits = 1;
  B200ST_TRY(mlp_splits(m_tiles, chunks, &splits));
  MlpParams p{};
  p.M = M; p.d = d; p.ffn = ffn; p.splits = splits; p.chunks_per_cta = chunks / splits;
  p.b1 = b1; p.b2 = b2; p.drop_ffn = drop_ffn; p.drop_post = drop_post;
  p.relu = 1; p.alpha = 1.f; p.mask_src = nullptr; p.mask_ld = 0; p.tickets = tickets;
  p.F1 = reinterpret_cast<uint16_t*>(F1); p.out = x_out;
  B200ST_CHECK((reinterpret_cast<uintptr_t>(F1) & 3) == 0 && (reinterpret_cast<uintptr_t>(x_out) & 15) == 0, "fused MLP: unaligned output");
  CUtensorMap tx, tw1, tw2;
  B200ST_TRY(make_operand_map(GemmOperand{X, dtype, 0, d, 0, 0}, M, d, 1, 1, BM, &tx));
  B200ST_TRY(make_operand_map(GemmOperand{W1, dtype, 1, ffn, 0, 0}, ffn, d, 1, 1, 64, &tw1));
  B200ST_TRY(make_operand_map(GemmOperand{W2, dtype, 1, d, 0, 0}, d, ffn, 1, 1, 64, &tw2));
  CUtensorMap to;
  B200ST_TRY(make_out_map_f32(x_out, M, d, d, &to));
  auto kern = d == 256 ? (dtype == F16 ? fused_mlp_fwd_kernel<F16, true, 256> : fused_mlp_fwd_kernel<BF16, true, 256>)
                       : (dtype == F16 ? fused_mlp_fwd_kernel<F16, true, 128> : fused_mlp_fwd_kernel<BF16, true, 128>);
  static bool attr[4] = {false, false, false, false};
  const int ai = (dtype == F16 ? 1 : 0) + (d == 256 ? 2 : 0);
  if (!attr[ai]) {
    B200ST_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kMlpSmem));
    attr[ai] = true;
  }
  return launch(kern, m_tiles * splits, kMlpThreads, kMlpSmem, stream, tx, tw1, tw2, to, p);
}

// Fused FFN backward, data-gradient chain: dF1 = scale * (dY W2^T) masked by (F1 > 0)  [written for the W1 weight gradient],
// dH += dF1 W1^T (fp32, dH must be zero-initialised).  Same kernel, weights read as K-major B operands.
int fused_mlp_bwd(const void* dY, int dtype, int M, int d, int ffn, const void* W1, const void* W2, const void* F1, float scale,
                  void* dF1, float* dH, cudaStream_t stream, int* tickets) {
  B200ST_CHECK(fused_mlp_supported(M, d, ffn, dtype), "fused MLP: unsupported shape / dtype");
  const int m_tiles = ceil_div(M, BM), chunks = ffn / 128;
  int splits = 1;
  B200ST_TRY(mlp_splits(m_tiles, chunks, &splits));
  MlpParams p{};
  p.M = M; p.d = d; p.ffn = ffn; p.splits = splits; p.chunks_per_cta = chunks / splits;
  p.b1 = nullptr; p.b2 = nullptr; p.drop_ffn = no_dropout(); p.drop_post = no_dropout();
  p.relu = 0; p.alpha = scale; p.mask_src = F1; p.mask_ld = ffn; p.tickets = tickets;
  p.F1 = reinterpret_cast<uint16_t*>(dF1); p.out = dH;
  B200ST_CHECK((reinterpret_cast<uintptr_t>(dF1) & 3) == 0 && (reinterpret_cast<uintptr_t>(dH) & 15) == 0 &&
               (reinterpret_cast<uintptr_t>(F1) & 3) == 0, "fused MLP: unaligned buffer");
  CUtensorMap tx, tw1, tw2;
  B200ST_TRY(make_operand_map(GemmOperand{dY, dtype, 0, d, 0, 0}, M, d, 1, 1, BM, &tx));
  B200ST_TRY(make_operand_map(GemmOperand{W2, dtype, 0, d, 0, 0}, ffn, d, 1, 1, 64, &tw1));      // G1: rows = hidden units, k = d
  B200ST_TRY(make_operand_map(GemmOperand{W1, dtype, 0, ffn, 0, 0}, d, ffn, 1, 1, d, &tw2));      // G2: rows = model dims, k = hidden
  CUtensorMap to;
  B200ST_TRY(make_out_map_f32(dH, M, d, d, &to));
  auto kern = d == 256 ? (dtype == F16 ? fused_mlp_fwd_kernel<F16, false, 256> : fused_mlp_fwd_kernel<BF16, false, 256>)
                       : (dtype == F16 ? fused_mlp_fwd_kernel<F16, false, 128> : fused_mlp_fwd_kernel<BF16, false, 128>);
  static bool attr[4] = {false, false, false, false};
  const int ai = (dtype == F16 ? 1 : 0) + (d == 256 ? 2 : 0);
  if (!attr[ai]) {
    B200ST_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kMlpSmem));
    attr[ai] = true;
  }
  return launch(kern, m_tiles * splits, kMlpThreads, kMlpSmem, stream, tx, tw1, tw2, to, p);
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
  // B200ST_PROFILE_CSV only names a file for the per-GEMM rows (tools/step_profile.py reads it); nothing computed changes
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
      if (r.has_conv) return r.conv.mode == kConvWgrad ? conv_wgrad_launch(r.g, r.conv, st) : gemm_tc_impl(r.g, st, &r.conv);
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
