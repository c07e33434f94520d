// Optimizer step of the training loop: gradient statistics (per-tensor sum of squares + finite check), dynamic loss-scale
// control, clip-by-value / per-tensor clip-by-norm and the Keras Adam update with the 16-bit shadow refresh — HBM-bound
// streaming kernels over the flat arenas (34 B per parameter for Adam, 4 B for the statistics pass); the pruned step adds
// the weight mask (1 bit per parameter) to the Adam pass and the selection kernels of prune.cu, the partial-tuning step
// the frozen-element bitmap (1 bit per parameter) to the Adam pass.
//
// Reference: GradAccumKerasModel.train_step (neurst/training/gradaccum_keras_model.py:222-240): unscale -> clip_by_value
// or clip_by_norm per gradient tensor -> apply_gradients; Keras Adam, epsilon-hat form (neurst/optimizers/__init__.py:21,
// hparams neurst/models/speech_transformer.py:265-270); dynamic loss scale (neurst/training/revised_dynamic_loss_scale.py:
// 60-107: skip the update and halve the scale on non-finite gradients, double it after `growth_steps` finite steps).
#include "kernels.cuh"
#include "pdl.cuh"

namespace b200st {
namespace {

__device__ __forceinline__ int tensor_of(const TensorTable& tt, uint32_t e8) {   // largest i with off8[i] <= e8
  int lo = 0, hi = tt.n;
  while (hi - lo > 1) {
    const int mid = (lo + hi) >> 1;
    if (tt.off8[mid] <= e8) lo = mid; else hi = mid;
  }
  return lo;
}

// sumsq[t] += sum of g^2 over tensor t.  A warp owns 1024 consecutive elements per iteration (4 x 16-byte loads per lane in
// flight, coalesced 512-byte rows); tensors start at multiples of 8 elements, so a lane's 4-element vector never straddles
// two tensors.  Usually the whole warp range lies inside one tensor: one atomic per warp.
__global__ void __launch_bounds__(256) grad_stats_kernel(const float* __restrict__ g, int64_t n, const __grid_constant__ TensorTable tt,
                                                         float* __restrict__ sumsq) {
  pdl_wait();
  pdl_trigger();
  const int lane = threadIdx.x & 31;
  const int64_t warp_id = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int64_t n_warps = (int64_t)gridDim.x * (blockDim.x >> 5);
  const int64_t n4 = n >> 2;                       // arenas are padded to multiples of 8 elements
  for (int64_t base = warp_id * 256; base < n4; base += n_warps * 256) {      // in float4 units: 256 vectors = 1024 elements
    float4 v[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int64_t i = base + j * 32 + lane;
      v[j] = i < n4 ? __ldg(reinterpret_cast<const float4*>(g) + i) : make_float4(0.f, 0.f, 0.f, 0.f);
    }
    const int64_t last = (base + 255 < n4 ? base + 255 : n4 - 1);
    const int t_first = tensor_of(tt, (uint32_t)(base >> 1)), t_last = tensor_of(tt, (uint32_t)(last >> 1));
    if (t_first == t_last) {
      float acc = 0.f;
#pragma unroll
      for (int j = 0; j < 8; ++j) acc += v[j].x * v[j].x + v[j].y * v[j].y + v[j].z * v[j].z + v[j].w * v[j].w;
      acc = warp_sum(acc);
      if (lane == 0) atomicAdd(sumsq + t_first, acc);
    } else {
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const int64_t i = base + j * 32 + lane;
        if (i < n4) atomicAdd(sumsq + tensor_of(tt, (uint32_t)(i >> 1)), v[j].x * v[j].x + v[j].y * v[j].y + v[j].z * v[j].z + v[j].w * v[j].w);
      }
    }
  }
}

// one thread: total norm, finite check, loss-scale state machine
__global__ void step_control_kernel(float* __restrict__ sumsq, int n_tensors, float* __restrict__ ctl, float grad_scale,
                                    float growth_steps, float multiplier) {
  pdl_wait();
  pdl_trigger();
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  float tot = 0.f;
  for (int i = 0; i < n_tensors; ++i) tot += sumsq[i];
  sumsq[n_tensors] = tot;
  if (!ctl) return;
  const float S = ctl[0] > 0.f ? ctl[0] : 1.f;
  const bool finite = isfinite(tot);
  ctl[5] = finite ? sqrtf(tot) * grad_scale / S : INFINITY;
  if (finite) {
    ctl[2] = 0.f;
    ctl[4] += 1.f;
    if (ctl[1] + 1.f >= growth_steps) { const float ns = S * multiplier; if (isfinite(ns)) ctl[0] = ns; ctl[1] = 0.f; }
    else ctl[1] += 1.f;
  } else {
    ctl[2] = 1.f;
    ctl[3] += 1.f;
    ctl[1] = 0.f;
    ctl[0] = fmaxf(S / multiplier, 1.f);
  }
}

// What the Adam pass does with the 1-bit-per-parameter `mask` (bit j of byte b is element 8b + j):
//   NONE    no mask.
//   PRUNE   the pruned step: off a pruning turn, the elements whose bit is 0 are written as zero in the master and shadow
//           arenas after their update (their Adam moments still move, so a later turn can bring them back); on a turn
//           (*turn != 0) the mask is not applied, the selection that follows sets the new one.
//   FREEZE  the partial-tuning step: the elements whose bit is 1 keep their old weight in the master and shadow arenas
//           (the shadow is the rounding of the master, so rounding the old weight rewrites the old 16-bit value); their
//           Adam moments still move, as the reference's Keras Adam updates every slot before the restore.  `turn` unused.
enum class MaskMode { NONE, PRUNE, FREEZE };

template <bool CLIP_NORM, MaskMode MODE>
__global__ void __launch_bounds__(256) adam_kernel(const OptimArgs a, const __grid_constant__ TensorTable tt, float unscale_host,
                                                   const uint8_t* __restrict__ mask, const int32_t* __restrict__ turn) {
  pdl_wait();
  pdl_trigger();
  bool apply_mask = false;
  if constexpr (MODE == MaskMode::PRUNE) apply_mask = *turn == 0;
  float gs = a.grad_scale * unscale_host;
  float t = (float)a.step_t;
  bool skip = false;
  if (a.ctl) {
    // the control kernel has already advanced the state: the scale that produced THESE gradients is recovered from it
    skip = a.ctl[2] != 0.f;
    t = a.ctl[4];
  }
  const float* __restrict__ unscale_dev = a.ctl ? a.ctl + 6 : nullptr;   // [6] = 1 / (scale used by this step)
  if (unscale_dev) gs *= *unscale_dev;
  const float b1 = a.beta1, b2 = a.beta2;
  const float lr_t = a.lr * sqrtf(1.f - powf(b2, t)) / (1.f - powf(b1, t));
  const int64_t n4 = a.n >> 2;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (int64_t)gridDim.x * blockDim.x) {
    if (skip) {
      if (a.zero_grad) reinterpret_cast<float4*>(a.g)[i] = make_float4(0.f, 0.f, 0.f, 0.f);
      continue;
    }
    const float4 g4 = reinterpret_cast<const float4*>(a.g)[i], m4 = reinterpret_cast<const float4*>(a.m)[i];
    const float4 v4 = reinterpret_cast<const float4*>(a.v)[i], p4 = reinterpret_cast<const float4*>(a.p)[i];
    float sc = gs;
    if (CLIP_NORM) {
      // tf.clip_by_norm(g, c): g * c / max(||g||, c) with the norm of the UNSCALED tensor
      const float nrm = sqrtf(a.tensor_sumsq[tensor_of(tt, (uint32_t)(i >> 1))]) * gs;
      sc = gs * a.clip_norm / fmaxf(nrm, a.clip_norm);
    }
    float gi[4] = {g4.x * sc, g4.y * sc, g4.z * sc, g4.w * sc};
    if (a.clip_value > 0.f) {
      // tf.clip_by_value keeps a NaN (its minimum / maximum propagate it); fminf / fmaxf would return the bound instead
#pragma unroll
      for (int j = 0; j < 4; ++j) gi[j] = gi[j] > a.clip_value ? a.clip_value : (gi[j] < -a.clip_value ? -a.clip_value : gi[j]);
    }
    const float mo[4] = {m4.x, m4.y, m4.z, m4.w}, vo[4] = {v4.x, v4.y, v4.z, v4.w}, po[4] = {p4.x, p4.y, p4.z, p4.w};
    float mi[4], vi[4], pi[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      mi[j] = b1 * mo[j] + (1.f - b1) * gi[j];
      vi[j] = b2 * vo[j] + (1.f - b2) * gi[j] * gi[j];
      pi[j] = po[j] - lr_t * mi[j] / (sqrtf(vi[j]) + a.eps);
    }
    if constexpr (MODE == MaskMode::PRUNE) {
      if (apply_mask) {
        const uint32_t bits = mask[i >> 1] >> ((i & 1) * 4);     // the 4 elements of vector i: bits 4(i&1) .. 4(i&1)+3
#pragma unroll
        for (int j = 0; j < 4; ++j) if (!((bits >> j) & 1u)) pi[j] = 0.f;
      }
    }
    if constexpr (MODE == MaskMode::FREEZE) {
      const uint32_t bits = mask[i >> 1] >> ((i & 1) * 4);
#pragma unroll
      for (int j = 0; j < 4; ++j) if ((bits >> j) & 1u) pi[j] = po[j];
    }
    reinterpret_cast<float4*>(a.m)[i] = make_float4(mi[0], mi[1], mi[2], mi[3]);
    reinterpret_cast<float4*>(a.v)[i] = make_float4(vi[0], vi[1], vi[2], vi[3]);
    reinterpret_cast<float4*>(a.p)[i] = make_float4(pi[0], pi[1], pi[2], pi[3]);
    if (a.shadow) {
      uint2 pk;
      pk.x = pack2_16(pi[0], pi[1], a.shadow_dtype); pk.y = pack2_16(pi[2], pi[3], a.shadow_dtype);
      reinterpret_cast<uint2*>(a.shadow)[i] = pk;
    }
    if (a.zero_grad) reinterpret_cast<float4*>(a.g)[i] = make_float4(0.f, 0.f, 0.f, 0.f);
  }
}

// ctl[6] = 1 / ctl[0]: latched BEFORE the control kernel changes the scale (the gradients were produced under ctl[0])
__global__ void latch_unscale_kernel(float* __restrict__ ctl) {
  pdl_wait();
  pdl_trigger();
  if (threadIdx.x == 0 && blockIdx.x == 0) ctl[6] = 1.f / (ctl[0] > 0.f ? ctl[0] : 1.f);
}

template <typename T>
__global__ void cast16_kernel(const float* __restrict__ x, T* __restrict__ y, int64_t n) {
  pdl_wait();
  pdl_trigger();
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    y[i] = from_f32<T>(x[i]);
}

}  // namespace

int cast_f32_to_16(const float* x, void* y, int y_dtype, int64_t n, cudaStream_t s) {
  if (n == 0) return 0;
  B200ST_CHECK(is16(y_dtype), "cast_f32_to_16 needs a 16-bit destination type");
  if (y_dtype == F16) return launch(cast16_kernel<__half>, grid_for(n, 256 * 4), 256, 0, s, x, reinterpret_cast<__half*>(y), n);
  return launch(cast16_kernel<__nv_bfloat16>, grid_for(n, 256 * 4), 256, 0, s, x, reinterpret_cast<__nv_bfloat16*>(y), n);
}

// gradient statistics + loss-scale control when clip_norm or the dynamic loss scale needs them
static int step_stats(const OptimArgs& a, const TensorTable& tt, cudaStream_t s) {
  const bool need_stats = a.clip_norm > 0.f || a.ctl != nullptr;
  if (!need_stats) return 0;
  B200ST_CHECK(a.tensor_sumsq != nullptr, "clip_norm / dynamic loss scale need the tensor_sumsq scratch [n_tensors + 1]");
  B200ST_CHECK(tt.n > 0 && tt.n <= 512, "clip_norm / dynamic loss scale support up to 512 parameter tensors");
  B200ST_CHECK(a.n % 8 == 0, "clip_norm / dynamic loss scale need an arena padded to a multiple of 8 elements");
  B200ST_CUDA(cudaMemsetAsync(a.tensor_sumsq, 0, sizeof(float) * (size_t)(tt.n + 1), s));
  B200ST_TRY(launch(grad_stats_kernel, grid_for(a.n, 8192, 132 * 8), 256, 0, s, (const float*)a.g, a.n, tt, a.tensor_sumsq));
  if (a.ctl) B200ST_TRY(launch(latch_unscale_kernel, 1, 32, 0, s, a.ctl));
  return launch(step_control_kernel, 1, 32, 0, s, a.tensor_sumsq, tt.n, a.ctl, a.grad_scale, a.growth_steps > 0.f ? a.growth_steps : 2000.f,
                a.multiplier > 1.f ? a.multiplier : 2.f);
}

static int check_arenas(const OptimArgs& a) {
  B200ST_CHECK(((reinterpret_cast<uintptr_t>(a.p) | reinterpret_cast<uintptr_t>(a.g) | reinterpret_cast<uintptr_t>(a.m) |
                 reinterpret_cast<uintptr_t>(a.v)) & 15) == 0 && (reinterpret_cast<uintptr_t>(a.shadow) & 7) == 0,
               "optimizer: arenas must be 16-byte aligned");
  B200ST_CHECK(!a.shadow || is16(a.shadow_dtype), "optimizer: the shadow arena must be a 16-bit type");
  return 0;
}

int optimizer_step(const OptimArgs& a, const TensorTable& tt, cudaStream_t s) {
  if (a.n == 0) return 0;
  B200ST_TRY(check_arenas(a));
  B200ST_TRY(step_stats(a, tt, s));
  const int grid = grid_for(a.n, 256 * 4 * 4);
  const uint8_t* no_mask = nullptr;
  const int32_t* no_turn = nullptr;
  if (a.clip_norm > 0.f) return launch(adam_kernel<true, MaskMode::NONE>, grid, 256, 0, s, a, tt, 1.f, no_mask, no_turn);
  return launch(adam_kernel<false, MaskMode::NONE>, grid, 256, 0, s, a, tt, 1.f, no_mask, no_turn);
}

// The reference's pruning optimizer (neurst/sparsity/pruning_optimizer.py) inside the loss-scale optimizer: statistics and
// loss-scale control, the pruning control (which sees whether this update is applied), Adam with the mask off-turn, and
// the selection + new mask on a turn.  No host synchronisation: the turn is a device word every kernel reads.
int optimizer_step_pruned(const OptimArgs& a, const TensorTable& tt, const PruneTable& pt, const PruneSchedule& sc,
                          const PruneDev& pd, cudaStream_t s) {
  B200ST_CHECK(a.n > 0 && a.n % 8 == 0, "the pruned step needs an arena padded to a multiple of 8 elements");
  B200ST_CHECK(pd.mask && pd.state && pd.scratch, "the pruned step needs the mask, the state words and the scratch");
  B200ST_TRY(check_arenas(a));
  B200ST_TRY(check_prune_table(pt));
  B200ST_TRY(step_stats(a, tt, s));
  B200ST_TRY(prune_control(pt, sc, a.ctl, pd, s));
  const int grid = grid_for(a.n, 256 * 4 * 4);
  const uint8_t* mask = pd.mask;
  const int32_t* turn = pd.state + 1;
  if (a.clip_norm > 0.f) B200ST_TRY(launch(adam_kernel<true, MaskMode::PRUNE>, grid, 256, 0, s, a, tt, 1.f, mask, turn));
  else B200ST_TRY(launch(adam_kernel<false, MaskMode::PRUNE>, grid, 256, 0, s, a, tt, 1.f, mask, turn));
  return prune_select_apply(a.p, a.shadow, pt, pd, turn, s);
}

// The reference's partial-tuning optimizer (examples/prune_tune/src/partial_tuning_optimizer.py:79-88): the plain step, then
// w = w_orig * original_mask + w * tuning_mask, i.e. the elements whose bit of `frozen` is 1 keep their weight.  Same
// statistics, loss-scale control and launches as optimizer_step; the Adam pass reads numel / 8 bytes more.
int optimizer_step_partial(const OptimArgs& a, const TensorTable& tt, const uint8_t* frozen, cudaStream_t s) {
  B200ST_CHECK(a.n > 0 && a.n % 8 == 0, "the partial-tuning step needs an arena padded to a multiple of 8 elements");
  B200ST_CHECK(frozen != nullptr, "the partial-tuning step needs the frozen-element bitmap");
  B200ST_TRY(check_arenas(a));
  B200ST_TRY(step_stats(a, tt, s));
  const int grid = grid_for(a.n, 256 * 4 * 4);
  const int32_t* no_turn = nullptr;
  if (a.clip_norm > 0.f) return launch(adam_kernel<true, MaskMode::FREEZE>, grid, 256, 0, s, a, tt, 1.f, frozen, no_turn);
  return launch(adam_kernel<false, MaskMode::FREEZE>, grid, 256, 0, s, a, tt, 1.f, frozen, no_turn);
}

}  // namespace b200st
