// Weight pruning of the training loop: the reference's pruning schedules (neurst/sparsity/pruning_schedule.py) evaluated on
// the device, and its mask update (neurst/sparsity/pruning_optimizer.py:106-119): per pruned tensor
// k = round(size * (1 - sparsity)), threshold = the k-th largest |w| counting duplicates (top_k(...).values[k-1]),
// mask = |w| >= threshold, w *= mask.
//
// Selection: an exact radix select over the bit patterns of |w| (non-negative floats order like uint32), all pruned tensors
// together in each launch.  Three digit passes (bits 31..21, 20..10, 9..0); each pass builds a shared-memory histogram per
// chunk of one tensor over the elements whose higher digits match the ones chosen so far, adds it into that tensor's global
// counts, and one CTA per tensor then picks the digit holding the k-th largest and the rank left inside it.  The counts are
// integers, so the threshold is exact and identical on every data-parallel rank; there is no sort and no host round-trip.
#include "kernels.cuh"
#include "pdl.cuh"

namespace b200st {
namespace {

__device__ __forceinline__ int chunk_tensor(const PruneTable& tb, uint32_t c) {   // largest i with cbase[i] <= c
  int lo = 0, hi = tb.n;
  while (hi - lo > 1) {
    const int mid = (lo + hi) >> 1;
    if (tb.cbase[mid] <= c) lo = mid; else hi = mid;
  }
  return lo;
}

__device__ __forceinline__ uint32_t abs_bits(float x) { return __float_as_uint(x) & 0x7fffffffu; }

// one thread block: the schedule's step, the turn decision and, on a turn, every tensor's k (float32 as in the reference)
__global__ void prune_control_kernel(const __grid_constant__ PruneTable tb, const PruneSchedule sc, const float* __restrict__ ctl,
                                     int32_t* __restrict__ state, uint32_t* __restrict__ rank, uint32_t* __restrict__ prefix) {
  __shared__ int turn_s;
  __shared__ float sparsity_s;
  pdl_wait();
  pdl_trigger();
  if (threadIdx.x == 0) {
    // under the dynamic loss scale a skipped update applies nothing: the optimizer's iterations do not advance
    const bool applied = ctl == nullptr || ctl[2] == 0.f;
    const int64_t step = (int64_t)state[0] + (applied ? 1 : 0);
    state[0] = (int32_t)step;
    const bool in_range = step >= sc.begin && (step <= sc.end || sc.end < 0);
    const bool turn = applied && in_range && (step - sc.begin) % sc.frequency == 0;
    float sp = sc.target;
    if (sc.polynomial) {
      float p = (float)(step - sc.begin) / (float)(sc.end - sc.begin);
      p = fminf(1.f, fmaxf(0.f, p));
      sp = __fadd_rn(__fmul_rn(sc.delta, powf(1.f - p, sc.power)), sc.target);    // no FMA contraction
    }
    state[1] = turn ? 1 : 0;
    if (turn) { state[2] += 1; state[3] = __float_as_int(sp); }
    turn_s = turn;
    sparsity_s = sp;
  }
  __syncthreads();
  if (!turn_s) return;
  for (int i = threadIdx.x; i < tb.n; i += blockDim.x) {
    const float kf = rintf((float)tb.size[i] * (1.f - sparsity_s));          // round half to even, as tf.math.round
    const uint32_t k = kf < 1.f ? 1u : kf > (float)tb.size[i] ? tb.size[i] : (uint32_t)kf;
    rank[i] = k;
    prefix[i] = 0u;
  }
}

// rank / prefix from host-given k and the turn word set (prune_select)
__global__ void prune_seed_kernel(const __grid_constant__ PruneTable tb, const int64_t* __restrict__ k, uint32_t* __restrict__ scratch) {
  pdl_wait();
  pdl_trigger();
  for (int i = threadIdx.x; i < tb.n; i += blockDim.x) {
    scratch[i] = (uint32_t)k[i];
    scratch[kPruneMaxTensors + i] = 0u;
  }
  if (threadIdx.x == 0) scratch[2 * kPruneMaxTensors] = 1u;
}

// histogram of digit (u >> SHIFT) & (2^BITS - 1) over the elements whose digits above SHIFT + BITS equal the prefix
template <int SHIFT, int BITS>
__global__ void __launch_bounds__(256) prune_hist_kernel(const float* __restrict__ p, const __grid_constant__ PruneTable tb,
                                                         const int32_t* __restrict__ turn, const uint32_t* __restrict__ prefix,
                                                         uint32_t* __restrict__ counts) {
  constexpr int BINS = 1 << BITS;
  constexpr int HI = SHIFT + BITS;
  __shared__ uint32_t h[BINS];
  pdl_wait();
  pdl_trigger();
  if (*turn == 0) return;
  const uint32_t n_chunks = tb.cbase[tb.n];
  for (uint32_t c = blockIdx.x; c < n_chunks; c += gridDim.x) {
    const int t = chunk_tensor(tb, c);
    for (int b = threadIdx.x; b < BINS; b += blockDim.x) h[b] = 0u;
    __syncthreads();
    const uint32_t size = tb.size[t];
    const uint32_t lo = (c - tb.cbase[t]) * (uint32_t)kPruneChunk;
    const uint32_t hi = min(lo + (uint32_t)kPruneChunk, size);
    const float* __restrict__ w = p + (size_t)tb.off8[t] * 8;
    const uint32_t pre = prefix[t];
#pragma unroll 4
    for (uint32_t e = lo + threadIdx.x * 4; e < hi; e += blockDim.x * 4) {
      // the tensor's slot is padded to 8 elements: the vector load stays inside it, the padding is not counted
      const float4 q = *reinterpret_cast<const float4*>(w + e);
      const float v[4] = {q.x, q.y, q.z, q.w};
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const uint32_t u = abs_bits(v[j]);
        bool match = e + j < hi;
        if constexpr (HI < 32) match = match && (u >> HI) == (pre >> HI);
        if (match) atomicAdd(&h[(u >> SHIFT) & (BINS - 1)], 1u);
      }
    }
    __syncthreads();
    uint32_t* ct = counts + (size_t)t * kPruneBins;
    for (int b = threadIdx.x; b < BINS; b += blockDim.x)
      if (h[b]) atomicAdd(ct + b, h[b]);
    __syncthreads();
  }
}

// one CTA per tensor: the digit that holds the rank-th largest, counted from the top bin; the counts are zeroed after reading
template <int SHIFT, int BITS, bool LAST>
__global__ void __launch_bounds__(256) prune_pick_kernel(const int32_t* __restrict__ turn, uint32_t* __restrict__ rank,
                                                         uint32_t* __restrict__ prefix, uint32_t* __restrict__ counts,
                                                         float* __restrict__ thresholds) {
  constexpr int BINS = 1 << BITS;
  constexpr int PER = BINS / 256;
  __shared__ uint32_t part[256];
  pdl_wait();
  pdl_trigger();
  if (*turn == 0) return;
  const int t = blockIdx.x, j = threadIdx.x;
  uint32_t* ct = counts + (size_t)t * kPruneBins;
  uint32_t c[PER];
  uint32_t s = 0;
#pragma unroll
  for (int q = 0; q < PER; ++q) {          // thread j owns bins BINS-1-j*PER .. BINS-PER-j*PER (descending)
    const int b = BINS - 1 - j * PER - q;
    c[q] = ct[b];
    ct[b] = 0u;
    s += c[q];
  }
  part[j] = s;
  __syncthreads();
  for (int off = 1; off < 256; off <<= 1) {  // inclusive scan over the threads (descending bin order)
    const uint32_t v = j >= off ? part[j - off] : 0u;
    __syncthreads();
    part[j] += v;
    __syncthreads();
  }
  const uint32_t incl = part[j], excl = incl - s;
  const uint32_t r = rank[t];
  __syncthreads();
  if (excl < r && r <= incl) {
    uint32_t cum = excl;
    bool found = false;
#pragma unroll
    for (int q = 0; q < PER; ++q) {
      if (!found && cum + c[q] >= r) {
        found = true;
        const uint32_t pre = prefix[t] | ((uint32_t)(BINS - 1 - j * PER - q) << SHIFT);
        rank[t] = r - cum;
        prefix[t] = pre;
        if (LAST && thresholds) thresholds[t] = __uint_as_float(pre);
      }
      cum += c[q];
    }
  }
}

// mask = |w| >= threshold over every byte of the pruned tensors (the padding bits stay 1); pruned elements -> 0 in both arenas
__global__ void __launch_bounds__(256) prune_apply_kernel(float* __restrict__ p, uint16_t* __restrict__ shadow,
                                                          const __grid_constant__ PruneTable tb, const int32_t* __restrict__ turn,
                                                          const uint32_t* __restrict__ thr, uint8_t* __restrict__ mask) {
  pdl_wait();
  pdl_trigger();
  if (*turn == 0) return;
  const uint32_t n_chunks = tb.cbase[tb.n];
  for (uint32_t c = blockIdx.x; c < n_chunks; c += gridDim.x) {
    const int t = chunk_tensor(tb, c);
    const uint32_t size = tb.size[t];
    const uint32_t lo = (c - tb.cbase[t]) * (uint32_t)kPruneChunk;
    const uint32_t hi = min(lo + (uint32_t)kPruneChunk, size);
    const size_t base = (size_t)tb.off8[t] * 8;
    const uint32_t th = thr[t];
    for (uint32_t e = lo + threadIdx.x * 8; e < hi; e += blockDim.x * 8) {
      const float4 a = *reinterpret_cast<const float4*>(p + base + e);
      const float4 b = *reinterpret_cast<const float4*>(p + base + e + 4);
      const float v[8] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w};
      uint32_t bits = 0;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const bool keep = e + j >= size || abs_bits(v[j]) >= th;
        bits |= (uint32_t)keep << j;
        if (!keep) {
          p[base + e + j] = 0.f;
          if (shadow) shadow[base + e + j] = 0;       // +0 in both 16-bit formats
        }
      }
      mask[(base + e) >> 3] = (uint8_t)bits;
    }
  }
}

// one thread per mask byte: the elements of its 8 whose bit is 0 -> +0 in the master and the 16-bit shadow (or null)
__global__ void __launch_bounds__(256) apply_mask_kernel(float* __restrict__ p, uint16_t* __restrict__ shadow,
                                                         const uint8_t* __restrict__ keep, int64_t n_bytes) {
  pdl_wait();
  pdl_trigger();
  for (int64_t b = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; b < n_bytes; b += (int64_t)gridDim.x * blockDim.x) {
    const uint32_t bits = keep[b];
    if (bits == 0xFFu) continue;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      if ((bits >> j) & 1u) continue;
      p[b * 8 + j] = 0.f;
      if (shadow) shadow[b * 8 + j] = 0;
    }
  }
}

int grid_chunks(const PruneTable& pt) {
  const uint32_t n = pt.cbase[pt.n];
  return (int)(n < 1 ? 1 : n > 132 * 8 ? 132 * 8 : n);
}

}  // namespace

size_t prune_scratch_bytes(int n) { return sizeof(uint32_t) * ((size_t)kPruneScratchHead + (size_t)n * kPruneBins); }

int check_prune_table(const PruneTable& pt) {
  B200ST_CHECK(pt.n >= 1 && pt.n <= kPruneMaxTensors, "pruning takes 1.." + std::to_string(kPruneMaxTensors) + " tensors");
  // the table is a kernel argument of ~6 KB: kernel arguments above 4 KB need a CUDA 12.1 driver
  static int driver = -1;
  if (driver < 0) B200ST_CUDA(cudaDriverGetVersion(&driver));
  B200ST_CHECK(driver >= 12010, "weight pruning needs a CUDA 12.1 or newer driver (kernel arguments above 4 KB)");
  return 0;
}

int prune_control(const PruneTable& pt, const PruneSchedule& sc, const float* ctl, const PruneDev& pd, cudaStream_t s) {
  return launch(prune_control_kernel, 1, 256, 0, s, pt, sc, ctl, pd.state, pd.scratch, pd.scratch + kPruneMaxTensors);
}

int prune_select_apply(float* p, void* shadow, const PruneTable& pt, const PruneDev& pd, const int32_t* turn, cudaStream_t s) {
  uint32_t* rank = pd.scratch;
  uint32_t* prefix = pd.scratch + kPruneMaxTensors;
  uint32_t* counts = pd.scratch + kPruneScratchHead;
  const int grid = grid_chunks(pt);
  B200ST_TRY(launch(prune_hist_kernel<21, 11>, grid, 256, 0, s, (const float*)p, pt, turn, (const uint32_t*)prefix, counts));
  B200ST_TRY(launch(prune_pick_kernel<21, 11, false>, pt.n, 256, 0, s, turn, rank, prefix, counts, pd.thresholds));
  B200ST_TRY(launch(prune_hist_kernel<10, 11>, grid, 256, 0, s, (const float*)p, pt, turn, (const uint32_t*)prefix, counts));
  B200ST_TRY(launch(prune_pick_kernel<10, 11, false>, pt.n, 256, 0, s, turn, rank, prefix, counts, pd.thresholds));
  B200ST_TRY(launch(prune_hist_kernel<0, 10>, grid, 256, 0, s, (const float*)p, pt, turn, (const uint32_t*)prefix, counts));
  B200ST_TRY(launch(prune_pick_kernel<0, 10, true>, pt.n, 256, 0, s, turn, rank, prefix, counts, pd.thresholds));
  return launch(prune_apply_kernel, grid, 256, 0, s, p, reinterpret_cast<uint16_t*>(shadow), pt, turn, (const uint32_t*)prefix, pd.mask);
}

int prune_select(float* p, void* shadow, const PruneTable& pt, const int64_t* k, const PruneDev& pd, cudaStream_t s) {
  B200ST_TRY(check_prune_table(pt));
  B200ST_TRY(launch(prune_seed_kernel, 1, 256, 0, s, pt, k, pd.scratch));
  return prune_select_apply(p, shadow, pt, pd, reinterpret_cast<const int32_t*>(pd.scratch + 2 * kPruneMaxTensors), s);
}

int apply_mask(float* p, void* shadow, const uint8_t* keep, int64_t n, cudaStream_t s) {
  if (n == 0) return 0;
  B200ST_CHECK(n > 0 && n % 8 == 0, "apply_mask: the arena must be padded to a multiple of 8 elements");
  return launch(apply_mask_kernel, grid_for(n / 8, 256, 132 * 8), 256, 0, s, p, reinterpret_cast<uint16_t*>(shadow), keep, n / 8);
}

}  // namespace b200st
