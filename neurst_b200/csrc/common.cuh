// Shared device/host helpers for libb200st (sm_90a only).
#pragma once
#include <cstdlib>
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <stdint.h>
#include <stdio.h>
#include <string>

namespace b200st {

// F16 (IEEE half): forward values in the "mixed16" precision (11-bit significand: 8x finer than bf16, the reference's own
// mixed_float16 compute type, neurst/training/training_utils.py:73-81); BF16: gradients (fp32 exponent range, no loss scaling).
enum DType : int { F32 = 0, BF16 = 1, F16 = 2 };
__host__ __device__ __forceinline__ bool is16(int dt) { return dt == BF16 || dt == F16; }
__host__ __device__ __forceinline__ int dtype_size(int dt) { return dt == F32 ? 4 : 2; }

// ---- error plumbing (thread-local last error string, C-ABI returns int) -----------------
void set_last_error(const std::string& s);
#define B200ST_FAIL(msg)                                                                   \
  do {                                                                                     \
    ::b200st::set_last_error(std::string(__FILE__) + ":" + std::to_string(__LINE__) + ": " + (msg)); \
    return 1;                                                                              \
  } while (0)
#define B200ST_CHECK(cond, msg)                                                            \
  do {                                                                                     \
    if (!(cond)) B200ST_FAIL(std::string("check failed: " #cond " — ") + (msg));          \
  } while (0)
#define B200ST_CUDA(expr)                                                                  \
  do {                                                                                     \
    cudaError_t _e = (expr);                                                               \
    if (_e != cudaSuccess) B200ST_FAIL(std::string(#expr ": ") + cudaGetErrorString(_e));  \
  } while (0)
#define B200ST_TRY(expr)                                                                   \
  do {                                                                                     \
    int _r = (expr);                                                                       \
    if (_r != 0) return _r;                                                                \
  } while (0)
// Runs the launch expression (0 or 1, as launch() in pdl.cuh returns) with T bound to the C++ type of dtype `dt`, and
// returns from the caller when it fails.
#define DISPATCH_DTYPE(dt, T, ...)                                                    \
  do {                                                                                \
    if ((dt) == F32) { using T = float; B200ST_TRY(__VA_ARGS__); }                    \
    else if ((dt) == BF16) { using T = __nv_bfloat16; B200ST_TRY(__VA_ARGS__); }      \
    else if ((dt) == F16) { using T = __half; B200ST_TRY(__VA_ARGS__); }              \
    else B200ST_FAIL("bad dtype");                                                    \
  } while (0)

// ---- dtype helpers -----------------------------------------------------------------------
template <typename T> struct DTypeOf;
template <> struct DTypeOf<float> { static constexpr int value = F32; };
template <> struct DTypeOf<__nv_bfloat16> { static constexpr int value = BF16; };
template <> struct DTypeOf<__half> { static constexpr int value = F16; };

__device__ __forceinline__ float to_f32(float v) { return v; }
__device__ __forceinline__ float to_f32(__nv_bfloat16 v) { return __bfloat162float(v); }
__device__ __forceinline__ float to_f32(__half v) { return __half2float(v); }
template <typename T> __device__ __forceinline__ T from_f32(float v);
template <> __device__ __forceinline__ float from_f32<float>(float v) { return v; }
template <> __device__ __forceinline__ __nv_bfloat16 from_f32<__nv_bfloat16>(float v) { return __float2bfloat16_rn(v); }
template <> __device__ __forceinline__ __half from_f32<__half>(float v) { return __float2half_rn(v); }

// two fp32 -> one packed 16-bit pair (low half = a) in the 16-bit type `dt`
__device__ __forceinline__ uint32_t pack2_16(float a, float b, int dt) {
  if (dt == F16) { __half2 h = __floats2half2_rn(a, b); return *reinterpret_cast<uint32_t*>(&h); }
  __nv_bfloat162 h = __floats2bfloat162_rn(a, b);
  return *reinterpret_cast<uint32_t*>(&h);
}
__device__ __forceinline__ float2 unpack2_16(uint32_t u, int dt) {
  if (dt == F16) return __half22float2(*reinterpret_cast<const __half2*>(&u));
  return __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&u));
}
// 8 consecutive elements: 16 bytes of a 16-bit type `DT` -> fp32, and fp32 -> 32 bytes of fp32 / 16 bytes of a 16-bit type
template <int DT> __device__ __forceinline__ void unpack8_16(const uint4& pk, float (&v)[8]) {
  const uint32_t w[4] = {pk.x, pk.y, pk.z, pk.w};
#pragma unroll
  for (int i = 0; i < 4; ++i) { const float2 f = unpack2_16(w[i], DT); v[2 * i] = f.x; v[2 * i + 1] = f.y; }
}
template <typename T> __device__ __forceinline__ void store8(T* dst, const float (&v)[8]);
template <> __device__ __forceinline__ void store8<float>(float* dst, const float (&v)[8]) {
  *reinterpret_cast<float4*>(dst) = make_float4(v[0], v[1], v[2], v[3]);
  *reinterpret_cast<float4*>(dst + 4) = make_float4(v[4], v[5], v[6], v[7]);
}
template <int DT> __device__ __forceinline__ void store8_16(void* dst, const float (&v)[8]) {
  uint4 pk;
  pk.x = pack2_16(v[0], v[1], DT); pk.y = pack2_16(v[2], v[3], DT);
  pk.z = pack2_16(v[4], v[5], DT); pk.w = pack2_16(v[6], v[7], DT);
  *reinterpret_cast<uint4*>(dst) = pk;
}
template <> __device__ __forceinline__ void store8<__nv_bfloat16>(__nv_bfloat16* dst, const float (&v)[8]) { store8_16<BF16>(dst, v); }
template <> __device__ __forceinline__ void store8<__half>(__half* dst, const float (&v)[8]) { store8_16<F16>(dst, v); }

__device__ __forceinline__ float load_as_f32(const void* p, int dtype, int64_t idx) {
  return dtype == F32 ? reinterpret_cast<const float*>(p)[idx]
         : dtype == F16 ? __half2float(reinterpret_cast<const __half*>(p)[idx])
                        : __bfloat162float(reinterpret_cast<const __nv_bfloat16*>(p)[idx]);
}
__device__ __forceinline__ void store_from_f32(void* p, int dtype, int64_t idx, float v) {
  if (dtype == F32) reinterpret_cast<float*>(p)[idx] = v;
  else if (dtype == F16) reinterpret_cast<__half*>(p)[idx] = __float2half_rn(v);
  else reinterpret_cast<__nv_bfloat16*>(p)[idx] = __float2bfloat16_rn(v);
}

// ---- warp / block reductions ------------------------------------------------------------
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
// block-wide sum / max (every thread gets the result); sm: >= 32 floats of shared memory.  Fixed reduction order.
__device__ __forceinline__ float block_sum(float v, float* sm) {
  v = warp_sum(v);
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5, nw = (blockDim.x + 31) >> 5;
  __syncthreads();
  if (lane == 0) sm[w] = v;
  __syncthreads();
  float t = (threadIdx.x < nw) ? sm[threadIdx.x] : 0.f;
  if (w == 0) { t = warp_sum(t); if (lane == 0) sm[0] = t; }
  __syncthreads();
  return sm[0];
}
__device__ __forceinline__ float block_max(float v, float* sm) {
  v = warp_max(v);
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5, nw = (blockDim.x + 31) >> 5;
  __syncthreads();
  if (lane == 0) sm[w] = v;
  __syncthreads();
  float t = (threadIdx.x < nw) ? sm[threadIdx.x] : -INFINITY;
  if (w == 0) { t = warp_max(t); if (lane == 0) sm[0] = t; }
  __syncthreads();
  return sm[0];
}

// ---- counter-based RNG for dropout: Philox4x32-7 ---------------------------------------
// (7 rounds: the smallest round count of Philox4x32 that Salmon et al. report as passing BigCrush; the generator of all
// keep-bits of a step is integer-ALU bound, so fewer rounds are directly fewer instructions)
// One call yields 4 x 32 random bits for counter (idx4, stream) under key (seed).  Dropout at element
// index e uses call (e >> 2) and lane (e & 3), so forward and backward regenerate identical masks.
struct Philox4 { uint32_t x, y, z, w; };
constexpr int kPhiloxRounds = 7;
__host__ __device__ __forceinline__ uint32_t mulhilo32(uint32_t a, uint32_t b, uint32_t* hi) {
  uint64_t p = (uint64_t)a * (uint64_t)b;
  *hi = (uint32_t)(p >> 32);
  return (uint32_t)p;
}
__host__ __device__ __forceinline__ Philox4 philox4x32(uint64_t seed, uint64_t counter, uint64_t stream) {
  uint32_t k0 = (uint32_t)seed, k1 = (uint32_t)(seed >> 32);
  uint32_t c0 = (uint32_t)counter, c1 = (uint32_t)(counter >> 32);
  uint32_t c2 = (uint32_t)stream, c3 = (uint32_t)(stream >> 32);
#pragma unroll
  for (int r = 0; r < kPhiloxRounds; ++r) {
    uint32_t hi0, hi1;
    uint32_t lo0 = mulhilo32(0xD2511F53u, c0, &hi0);
    uint32_t lo1 = mulhilo32(0xCD9E8D57u, c2, &hi1);
    uint32_t n0 = hi1 ^ c1 ^ k0, n1 = lo1, n2 = hi0 ^ c3 ^ k1, n3 = lo0;
    c0 = n0; c1 = n1; c2 = n2; c3 = n3;
    k0 += 0x9E3779B9u; k1 += 0xBB67AE85u;
  }
  return Philox4{c0, c1, c2, c3};
}
// Dropout keep-decisions come 8 at a time: one Philox call yields 128 bits = 8 x 16-bit uniforms for the elements
// [8g, 8g+8) of dropout site `stream`; element e is kept iff its u16 >= thresh, thresh = round(p * 65536).
__host__ __device__ __forceinline__ uint32_t dropout_thresh16(float p) {
  float t = p * 65536.0f + 0.5f;
  return t <= 0.f ? 0u : (t >= 65535.f ? 65535u : (uint32_t)t);
}
__host__ __device__ __forceinline__ uint32_t dropout_keep8(uint64_t seed, uint64_t stream, uint64_t group, uint32_t thresh) {
  const Philox4 r = philox4x32(seed, group, stream);
  uint32_t m = 0;
  m |= ((r.x & 0xffffu) >= thresh ? 1u : 0u) << 0; m |= ((r.x >> 16) >= thresh ? 1u : 0u) << 1;
  m |= ((r.y & 0xffffu) >= thresh ? 1u : 0u) << 2; m |= ((r.y >> 16) >= thresh ? 1u : 0u) << 3;
  m |= ((r.z & 0xffffu) >= thresh ? 1u : 0u) << 4; m |= ((r.z >> 16) >= thresh ? 1u : 0u) << 5;
  m |= ((r.w & 0xffffu) >= thresh ? 1u : 0u) << 6; m |= ((r.w >> 16) >= thresh ? 1u : 0u) << 7;
  return m;
}
__host__ __device__ __forceinline__ bool dropout_keep(uint64_t seed, uint64_t stream, uint64_t e, float p) {
  return (dropout_keep8(seed, stream, e >> 3, dropout_thresh16(p)) >> (e & 7)) & 1u;
}

struct DropoutSpec {
  float p;          // 0 => disabled
  float scale;      // 1/(1-p)
  uint64_t seed;
  uint64_t stream;  // unique id of the dropout site (layer, op)
  const uint64_t* seed_ptr;   // optional device address of the seed (CUDA-graph replay with a fresh seed per step)
  const uint8_t* bits;        // optional precomputed keep-bits (byte g = dropout_keep8 of group g); same values as Philox
};
__host__ __device__ __forceinline__ DropoutSpec no_dropout() { return DropoutSpec{0.f, 1.f, 0, 0, nullptr, nullptr}; }
__device__ __forceinline__ uint64_t dropout_seed(const DropoutSpec& d) { return d.seed_ptr ? *d.seed_ptr : d.seed; }
// keep-bits of group g (elements [8g, 8g+8)): from the precomputed bitmap when present, else regenerated
__device__ __forceinline__ uint32_t drop_keep8(const DropoutSpec& d, uint64_t group, uint32_t thresh) {
  return d.bits ? (uint32_t)__ldg(d.bits + group) : dropout_keep8(dropout_seed(d), d.stream, group, thresh);
}
__device__ __forceinline__ bool drop_keep1(const DropoutSpec& d, uint64_t e) {
  return (drop_keep8(d, e >> 3, dropout_thresh16(d.p)) >> (e & 7)) & 1u;
}

static inline int ceil_div(int64_t a, int64_t b) { return (int)((a + b - 1) / b); }
// blocks for `work` items at `per_block` items per block, clamped to [1, cap] (grid-stride kernels loop over the rest)
static inline int grid_for(int64_t work, int per_block, int cap = 132 * 16) {
  int64_t g = (work + per_block - 1) / per_block;
  if (g < 1) g = 1;
  return (int)(g > cap ? cap : g);
}

}  // namespace b200st
