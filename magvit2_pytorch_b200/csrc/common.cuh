// Shared helpers for libmagvit2_b200.so (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <stdint.h>
#include <stdio.h>
#include <stdarg.h>
#include <mutex>
#include "../../include/magvit2_b200.h"

namespace mv2 {

void set_error(const char* fmt, ...);

#define MV2_CHECK_ARG(cond, ...)                                  \
  do {                                                            \
    if (!(cond)) {                                                \
      mv2::set_error("%s:%d: argument check failed: %s", __FILE__, __LINE__, #cond); \
      return MV2_E_ARG;                                           \
    }                                                             \
  } while (0)

#define MV2_CHECK_LAUNCH()                                        \
  do {                                                            \
    cudaError_t e__ = cudaGetLastError();                         \
    if (e__ != cudaSuccess) {                                     \
      mv2::set_error("%s:%d: CUDA launch failed: %s", __FILE__, __LINE__, cudaGetErrorString(e__)); \
      return MV2_E_CUDA;                                          \
    }                                                             \
  } while (0)

#define MV2_CHECK_CUDA(expr)                                      \
  do {                                                            \
    cudaError_t e__ = (expr);                                     \
    if (e__ != cudaSuccess) {                                     \
      mv2::set_error("%s:%d: %s failed: %s", __FILE__, __LINE__, #expr, cudaGetErrorString(e__)); \
      return MV2_E_CUDA;                                          \
    }                                                             \
  } while (0)

template <typename T> __device__ __forceinline__ float to_f32(T v);
template <> __device__ __forceinline__ float to_f32<float>(float v) { return v; }
template <> __device__ __forceinline__ float to_f32<__nv_bfloat16>(__nv_bfloat16 v) { return __bfloat162float(v); }
// MV2_U8 sources (decoded video frames): the data loaders' normalisation x / 255 (reference data.py:103 ToTensor,
// data.py:188 `frames_torch /= 255.`) -- a correctly rounded fp32 division, so the result is bit-identical to theirs
template <> __device__ __forceinline__ float to_f32<uint8_t>(uint8_t v) { return __fdiv_rn((float)v, 255.f); }

template <typename T> __device__ __forceinline__ T from_f32(float v);
template <> __device__ __forceinline__ float from_f32<float>(float v) { return v; }
template <> __device__ __forceinline__ __nv_bfloat16 from_f32<__nv_bfloat16>(float v) { return __float2bfloat16_rn(v); }
template <> __device__ __forceinline__ float to_f32<__half>(__half v) { return __half2float(v); }
template <> __device__ __forceinline__ __half from_f32<__half>(float v) { return __float2half_rn(v); }

// The two 16-bit activation dtypes (MV2_BF16, MV2_F16): fp32 accumulation, one round-to-nearest-even per stored value.
// pair_t<T> is the 2-element vector type of T; pair_to_f2 / f2_to_pair convert it to and from fp32.
template <typename T> struct pair_of;
template <> struct pair_of<__nv_bfloat16> { typedef __nv_bfloat162 type; };
template <> struct pair_of<__half> { typedef __half2 type; };
template <typename T> using pair_t = typename pair_of<T>::type;
__device__ __forceinline__ float2 pair_to_f2(__nv_bfloat162 v) { return __bfloat1622float2(v); }
__device__ __forceinline__ float2 pair_to_f2(__half2 v) { return __half22float2(v); }
template <typename T> __device__ __forceinline__ pair_t<T> f2_to_pair(float a, float b);
template <> __device__ __forceinline__ __nv_bfloat162 f2_to_pair<__nv_bfloat16>(float a, float b) { return __floats2bfloat162_rn(a, b); }
template <> __device__ __forceinline__ __half2 f2_to_pair<__half>(float a, float b) { return __floats2half2_rn(a, b); }

// Activations.  expm1f / expf (not the fast intrinsics): the fp32 path must track the
// reference's libm-based CPU results to ~1 ulp.
__device__ __forceinline__ float act_elu(float v) { return v > 0.f ? v : expm1f(v); }
__device__ __forceinline__ float act_silu(float v) { return v / (1.f + expf(-v)); }
__device__ __forceinline__ float apply_act(float v, int act) {
  if (act == MV2_ACT_ELU) return act_elu(v);
  if (act == MV2_ACT_SILU) return act_silu(v);
  if (act == MV2_ACT_LEAKY_RELU) return v > 0.f ? v : 0.1f * v;
  if (act == MV2_ACT_RELU) return v < 0.f ? 0.f : v;     // NaN passes, as torch.relu
  return v;
}

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

static inline int ceil_div(int64_t a, int64_t b) { return (int)((a + b - 1) / b); }

// ---- attention dropout: counter-based Philox4x32-10 (Salmon et al., SC'11; Random123's constants) ------------------------
// The keep mask is a pure function of (seed, call, sequence, head, query i, key j): word j & 3 of
// philox(counter (i, j >> 2, seq, h | call << 16), key seed) is kept iff >= thr = floor(p * 2^32).  No kernel, tiling or
// dtype enters it, so every attention kernel, mv2_attention_dropout_mask and a numpy replica agree bit for bit.
__device__ __forceinline__ uint4 philox4x32_10(uint4 c, uint32_t k0, uint32_t k1) {
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    if (r) { k0 += 0x9E3779B9u; k1 += 0xBB67AE85u; }
    const uint32_t lo0 = 0xD2511F53u * c.x, hi0 = __umulhi(0xD2511F53u, c.x);
    const uint32_t lo1 = 0xCD9E8D57u * c.z, hi1 = __umulhi(0xCD9E8D57u, c.z);
    c = make_uint4(hi1 ^ c.y ^ k0, lo1, hi0 ^ c.w ^ k1, lo0);
  }
  return c;
}

struct AttnDrop {           // kernel-side form of mv2_dropout_args
  uint32_t k0, k1;          // seed, low / high word
  uint32_t call_hi;         // call << 16
  uint32_t thr;             // keep iff word >= thr
  float scale;              // fp32(1 / (1 - p))
};

// keep bits (bit w = word w >= thr) of the 4-key group `grp` (keys 4 grp .. 4 grp + 3) of query i
__device__ __forceinline__ uint32_t attn_keep4(const AttnDrop& d, uint32_t i, uint32_t grp, uint32_t seq, uint32_t h) {
  const uint4 r = philox4x32_10(make_uint4(i, grp, seq, h | d.call_hi), d.k0, d.k1);
  return (uint32_t)(r.x >= d.thr) | (uint32_t)(r.y >= d.thr) << 1 | (uint32_t)(r.z >= d.thr) << 2 | (uint32_t)(r.w >= d.thr) << 3;
}

// ---- per-device one-time initialisation ----------------------------------------------------------------------
// cudaFuncSetAttribute (the > 48 KB dynamic shared memory opt-in) applies to the CURRENT device only, so a process that
// drives several GPUs must repeat it on each of them: the flag is kept per device ordinal, not per process.
struct PerDeviceOnce {
  std::mutex mu;
  bool done[64] = {};
  cudaError_t err[64] = {};
  template <typename F>
  cudaError_t run(F&& f) {
    int dev = 0;
    cudaError_t e = cudaGetDevice(&dev);
    if (e != cudaSuccess) return e;
    if (dev < 0 || dev >= 64) return cudaErrorInvalidDevice;
    std::lock_guard<std::mutex> lk(mu);
    if (!done[dev]) { err[dev] = f(); done[dev] = true; }
    return err[dev];
  }
};

// ---- programmatic dependent launch (PDL) ---------------------------------------------------------------------
// Every kernel of the library starts with pdl_wait() (everything before it -- barrier init, bias
// staging -- may overlap the tail of the previous kernel in the stream) and signals pdl_launch_dependents() right
// after, so the next kernel's CTAs move in as this kernel's CTAs retire.  Without the launch attribute both
// instructions are no-ops.  mv2_set_pdl(1) turns the attribute on for all launches.
extern int g_pdl;
// kernels launched from this thread (mv2_launch_count)
extern thread_local uint64_t g_launches;
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }

template <typename... KArgs, typename... Args>
static inline void launch_k(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, Args&&... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  cudaLaunchAttribute attr;
  attr.id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr.val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = &attr;
  cfg.numAttrs = g_pdl ? 1 : 0;
  // a refused launch is not counted; its error surfaces through MV2_CHECK_LAUNCH
  if (cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...) == cudaSuccess) ++g_launches;
}

}  // namespace mv2
