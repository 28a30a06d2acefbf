// Shared device-side PTX wrappers (mbarrier / TMA / wgmma) and host-side tensor-map helpers for the Hopper
// tensor-core kernels (tc_conv.cu, tc_slab.cu).  sm_90a only.
#pragma once
#include "common.cuh"
#include <cuda.h>
#include <mutex>
#include <type_traits>

namespace mv2 {


// ------------------------------------------------------------------------------------------
// PTX wrappers
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  asm volatile(
      "{\n\t"
      ".reg .pred P1;\n\t"
      "WAIT_LOOP:\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 P1, [%0], %1, 0x989680;\n\t"
      "@P1 bra DONE;\n\t"
      "bra WAIT_LOOP;\n\t"
      "DONE:\n\t"
      "}" ::"r"(bar), "r"(parity) : "memory");
}
__device__ __forceinline__ void fence_barrier_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

__device__ __forceinline__ void tma_load_5d(uint32_t dst, const CUtensorMap* map, uint32_t bar, int c0, int c1, int c2,
                                            int c3, int c4) {
  asm volatile(
      "cp.async.bulk.tensor.5d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6, %7}], [%2];"
      ::"r"(dst), "l"(map), "r"(bar), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "r"(c4) : "memory");
}
__device__ __forceinline__ void tma_load_2d(uint32_t dst, const CUtensorMap* map, uint32_t bar, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
      ::"r"(dst), "l"(map), "r"(bar), "r"(c0), "r"(c1) : "memory");
}
__device__ __forceinline__ void tma_load_3d(uint32_t dst, const CUtensorMap* map, uint32_t bar, int c0, int c1, int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
      ::"r"(dst), "l"(map), "r"(bar), "r"(c0), "r"(c1), "r"(c2) : "memory");
}
// shared -> global box store, completed through this thread's bulk async-groups
__device__ __forceinline__ void tma_store_5d(const CUtensorMap* map, uint32_t src, int c0, int c1, int c2, int c3, int c4) {
  asm volatile("cp.async.bulk.tensor.5d.global.shared::cta.bulk_group [%0, {%2, %3, %4, %5, %6}], [%1];"
               ::"l"(map), "r"(src), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "r"(c4) : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
// waits until this thread's bulk stores have read their shared-memory sources (the buffers may be written again)
__device__ __forceinline__ void bulk_wait_read_all() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }
// waits until this thread's bulk stores are complete
__device__ __forceinline__ void bulk_wait_all() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* map) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(map) : "memory");
}

// ---- wgmma (sm_90a warpgroup MMA): D[regs] (+)= A[smem] * B[smem], bf16, fp16 or tf32 in, fp32 accumulate ----
// Every wgmma instruction is issued by all 128 threads of a warpgroup; the 64 x N fp32 accumulator lives in their
// registers (m64nNk16 / m64nNk8 fragment: thread t holds rows 16 (t / 32) + (t % 32) / 4 (+ 8), columns 8 j + 2 (t % 4) (+ 1)).
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_wait_all() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }
// waits until at most N committed groups of this warpgroup are still in flight
template <int N> __device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }

// Per-warpgroup register budget (setmaxnreg): all four warps of a warpgroup execute it.  A warp-specialised kernel lowers
// its producer warpgroup's budget so that its consumer warpgroups can raise theirs within the SM's 64 K registers.
template <int N> __device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(N)); }
template <int N> __device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(N)); }
// One specialisation per (element type, N): the element type selects the PTX operand type, .bf16 or .f16 (the same
// tensor-core rate on sm_90a; fp16 keeps 3 more mantissa bits, bf16 8 more exponent bits), or .tf32 for fp32 storage.
// One MMA reads 32 bytes of K either way: k16 of a 16-bit type, k8 of tf32 (which has no transpose operands: both are
// K-major, as here).  The tensor core reads a tf32 operand as the top 19 bits of its fp32 word (sign, 8-bit exponent,
// 10-bit mantissa): the low 13 mantissa bits are dropped, not rounded.
template <typename T, int N> __device__ __forceinline__ void wgmma_mma(float (&d)[N / 2], uint64_t da, uint64_t db, uint32_t scale_d);
#define MV2_WGMMA_DEF(T, TY, K, TR, N, REGS, DA, DB, P, ...)                                                     \
  template <> __device__ __forceinline__ void wgmma_mma<T, N>(float (&d)[N / 2], uint64_t da, uint64_t db, uint32_t scale_d) { \
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, " P ", 0;\n\t"                                           \
                 "wgmma.mma_async.sync.aligned.m64n" #N K ".f32." TY "." TY " " REGS ", " DA ", " DB ", p, 1, 1" TR ";\n\t}" \
                 : __VA_ARGS__ : "l"(da), "l"(db), "r"(scale_d));                                                     \
  }
#define MV2_WGMMA_N8(T, TY, K, TR) MV2_WGMMA_DEF(T, TY, K, TR, 8, "{%0, %1, %2, %3}", "%4", "%5", "%6", "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]))
#define MV2_WGMMA_N16(T, TY, K, TR) MV2_WGMMA_DEF(T, TY, K, TR, 16, "{%0, %1, %2, %3, %4, %5, %6, %7}", "%8", "%9", "%10", "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]))
#define MV2_WGMMA_N32(T, TY, K, TR) MV2_WGMMA_DEF(T, TY, K, TR, 32, "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}", "%16", "%17", "%18", "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]))
#define MV2_WGMMA_N64(T, TY, K, TR) MV2_WGMMA_DEF(T, TY, K, TR, 64, "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}", "%32", "%33", "%34", "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]))
#define MV2_WGMMA_N128(T, TY, K, TR) MV2_WGMMA_DEF(T, TY, K, TR, 128, "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}", "%64", "%65", "%66", "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]))
#define MV2_WGMMA_ALL(T, TY, K, TR) MV2_WGMMA_N8(T, TY, K, TR) MV2_WGMMA_N16(T, TY, K, TR) MV2_WGMMA_N32(T, TY, K, TR) \
  MV2_WGMMA_N64(T, TY, K, TR) MV2_WGMMA_N128(T, TY, K, TR)
MV2_WGMMA_ALL(__nv_bfloat16, "bf16", "k16", ", 0, 0")
MV2_WGMMA_ALL(__half, "f16", "k16", ", 0, 0")
MV2_WGMMA_ALL(float, "tf32", "k8", "")
#undef MV2_WGMMA_ALL
#undef MV2_WGMMA_N8
#undef MV2_WGMMA_N16
#undef MV2_WGMMA_N32
#undef MV2_WGMMA_N64
#undef MV2_WGMMA_N128
#undef MV2_WGMMA_DEF

// wgmma shared-memory matrix descriptor, K-major operand with hardware swizzle (128 B rows -> SWIZZLE_128B, 64 B ->
// SWIZZLE_64B, 32 B -> SWIZZLE_32B), without the start address:
//   bits [0,14) start address >> 4      bits [16,30) leading byte offset >> 4 (unused for swizzled K-major)
//   bits [32,46) stride byte offset >> 4 (distance between 8-row core groups)      bits [62,64) swizzle: 1 = 128B, 2 = 64B, 3 = 32B
// The swizzle is a function of the absolute shared-memory address (as for TMA), so a start address moved by whole rows
// or by 32-byte K steps inside a 1024-byte-aligned tile still addresses what TMA wrote; the base-offset field stays 0.
__host__ __device__ __forceinline__ uint64_t gmma_desc_hi(uint32_t sbo, uint32_t row_bytes) {
  const uint64_t layout = row_bytes == 128 ? 1 : (row_bytes == 64 ? 2 : 3);
  return ((uint64_t)1 << 16) | ((uint64_t)(sbo >> 4) << 32) | (layout << 62);
}
__device__ __forceinline__ uint32_t desc_lo(uint32_t saddr) { return (saddr & 0x3FFFF) >> 4; }

// Accumulator staging: a warpgroup writes its 64 x N fragment to shared memory ([64][N + 4] fp32: the padding makes the
// row-per-thread reads below conflict-free), so that the epilogue can work on one output row per thread.
template <int N> __device__ __forceinline__ void stage_acc(const float (&d)[N / 2], float* stg, int t) {
  const int r = 16 * (t >> 5) + ((t & 31) >> 2), c = 2 * (t & 3);
#pragma unroll
  for (int j = 0; j < N / 8; ++j) {
    *reinterpret_cast<float2*>(stg + r * (N + 4) + 8 * j + c) = make_float2(d[4 * j], d[4 * j + 1]);
    *reinterpret_cast<float2*>(stg + (r + 8) * (N + 4) + 8 * j + c) = make_float2(d[4 * j + 2], d[4 * j + 3]);
  }
}
// 32 (or, at the end of a 16-column-wide tile, 16) consecutive accumulator columns of one staged row
__device__ __forceinline__ void load_row32(const float* src, int ncols, uint32_t (&r)[32]) {
#pragma unroll
  for (int g = 0; g < 8; ++g) {
    if (g * 4 >= ncols) break;
    const float4 v = *reinterpret_cast<const float4*>(src + 4 * g);
    r[4 * g] = __float_as_uint(v.x); r[4 * g + 1] = __float_as_uint(v.y);
    r[4 * g + 2] = __float_as_uint(v.z); r[4 * g + 3] = __float_as_uint(v.w);
  }
}
__device__ __forceinline__ void named_bar_sync(uint32_t id, uint32_t nthreads) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}

// Two fp32 values rounded (RN) into one 32-bit word of the element type T, and the two halves of such a word back in fp32
template <typename T> __device__ __forceinline__ uint32_t pack2(float a, float b) {
  pair_t<T> v = f2_to_pair<T>(a, b);
  return *reinterpret_cast<uint32_t*>(&v);
}
template <typename T> __device__ __forceinline__ float2 unpack2(uint32_t r) {
  if constexpr (std::is_same<T, __nv_bfloat16>::value) return make_float2(__uint_as_float(r << 16), __uint_as_float(r & 0xffff0000u));
  else return pair_to_f2(*reinterpret_cast<const pair_t<T>*>(&r));
}



// ------------------------------------------------------------------------------------------
// shared epilogue: fp32 accumulator chunk -> bias -> activation -> (GEGLU | shuffle) -> residual -> bf16 / fp16 / fp32 store
// ------------------------------------------------------------------------------------------
struct TcEpi {
  const float* bias;             // global, packed column order (only used to decide has-bias; values come from smem)
  const void* res;               // element type of the kernel (bf16 / fp16 / fp32)
  void* y;
  int act, shuffle, mode;        // mode 0 plain; 1 GEGLU: packed cols [16g, 16g+8) = x, [16g+8, 16g+16) = gate (M:466-469);
                                 // 2 scaled residual: (act(acc + bias) + res) * 2^-0.5 (DiscriminatorBlock, M:585)
  int Co;                        // packed GEMM output columns
  int To, Ho, Wo;                // output volume before any depth-to-space/time shuffle
  int out_cf;                    // 1: y is channels-first (B, Co, To, Ho, Wo) -- EPI_RAGGED scalar stores only (conv_out,
                                 // the video's data gradient)
  const float* oscale;           // [B][Co] or null: accumulator multiplier per (clip, output channel) before bias / activation
};

// 8 consecutive elements of T from / to fp32: 16 bytes of bf16 / fp16 (one rounding each), 32 bytes of fp32
template <typename T> __device__ __forceinline__ void store8(T* dst, const float (&v)[8]) {
  if constexpr (std::is_same<T, float>::value) {
    reinterpret_cast<float4*>(dst)[0] = make_float4(v[0], v[1], v[2], v[3]);
    reinterpret_cast<float4*>(dst)[1] = make_float4(v[4], v[5], v[6], v[7]);
  } else {
    uint4 o;
    o.x = pack2<T>(v[0], v[1]); o.y = pack2<T>(v[2], v[3]);
    o.z = pack2<T>(v[4], v[5]); o.w = pack2<T>(v[6], v[7]);
    *reinterpret_cast<uint4*>(dst) = o;
  }
}
template <typename T> __device__ __forceinline__ void load8(const T* src, float (&f)[8]) {
  if constexpr (std::is_same<T, float>::value) {
    const float4 a = reinterpret_cast<const float4*>(src)[0], b = reinterpret_cast<const float4*>(src)[1];
    f[0] = a.x; f[1] = a.y; f[2] = a.z; f[3] = a.w; f[4] = b.x; f[5] = b.y; f[6] = b.z; f[7] = b.w;
  } else {
    const uint4 rv = *reinterpret_cast<const uint4*>(src);
    const pair_t<T>* rb = reinterpret_cast<const pair_t<T>*>(&rv);
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const float2 p = pair_to_f2(rb[q]);
      f[2 * q] = p.x; f[2 * q + 1] = p.y;
    }
  }
}

// Epilogue flavours are compile-time so each kernel instance carries only the code it runs (the generic version was
// ~2300 SASS instructions per 32-column chunk and thrashed the instruction cache of the 8 epilogue warps).
// EPI_PLAIN (slab kernel only) additionally requires Co % 8 == 0; its epilogue runs on the accumulator fragments and
// stores through TMA (tc_slab.cu: slab_epi_fragment);
// EPI_RAGGED is the direct per-row path with scalar tails (conv_out's 3 channels, and the tap kernel's plain mode).
// EPI_PLAIN_RES is EPI_PLAIN with a residual input (TMA-loaded into shared memory under the main loop): act(conv + bias)
// + res is summed in fp32 and rounded to bf16 ONCE (the reference's bf16 `fn(x) + x` rounds twice; the single rounding
// is strictly closer to the fp32 result).
// EPI_FUSED_RU (slab kernel only): the whole conv half of a ResidualUnit in one launch -- the ELU'd 3x3x3 tile goes to
// shared memory as the A operand of a second wgmma against the 1x1x1 weights, and the second epilogue emits the
// SqueezeExcite online-softmax pool partials next to y (see tc_slab.cu).
// EPI_SHUFFLE_ST (slab kernel only): depth-to-space / depth-to-time stores through a shared-memory transpose of the
// staged accumulators (64 contiguous bytes per output position and store instruction); needs Cy % 32 == 0 so that a 32-column chunk
// stays inside one sub-pixel phase.  EPI_SHUFFLE is the direct 16-byte-piece path for the other widths.
// EPI_DOWN_SPACE (slab kernel only): SpatialDownsample2x (3x3, stride 2) -- plain epilogue, but the slab is two row-parity
// sub-slabs of the input viewed as (W/2) x (2C) and the taps follow a small offset table (see tc_slab.cu).
enum { EPI_PLAIN = 0, EPI_GEGLU = 1, EPI_SHUFFLE = 2, EPI_RAGGED = 3, EPI_PLAIN_RES = 4, EPI_FUSED_RU = 5, EPI_SHUFFLE_ST = 6,
       EPI_DOWN_SPACE = 7 };

// Branch-free activations on the bare MUFU approximations (ex2/rcp with flush-to-zero): the results are rounded to
// bf16 right after, and __expf's denormal range handling costs ~5 extra instructions per element.
__device__ __forceinline__ float ex2_approx(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ float rcp_approx(float x) {
  float y;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
// erf by Abramowitz & Stegun 7.1.26 (|error| <= 1.5e-7, far below the bf16 rounding of the result): 2 MUFU + ~12 FP32
// instructions, about half of libdevice's erff; the GEGLU epilogue of the feed-forward runs 16 of them per 32 columns.
__device__ __forceinline__ float erf_fast(float x) {
  const float ax = fabsf(x);
  const float t = rcp_approx(fmaf(0.3275911f, ax, 1.f));
  float p = fmaf(1.061405429f, t, -1.453152027f);
  p = fmaf(p, t, 1.421413741f);
  p = fmaf(p, t, -0.284496736f);
  p = fmaf(p, t, 0.254829592f);
  const float e = ex2_approx(-1.4426950408889634f * ax * ax);
  return copysignf(fmaf(-p * t, e, 1.f), x);
}

// gelu(g) = g * Phi(g) with Phi(g) = 0.5 (1 + erf(g / sqrt 2)) and erf by Abramowitz & Stegun 7.1.26 in z = |g| / sqrt 2
// (|error| <= 1.5e-7): with q = 0.5 * t * poly(t) * exp(-g^2 / 2), t = 1 / (1 + 0.3275911 z),
//   Phi(g) = 1 - q (g >= 0), q (g < 0)   =>   gelu(g) = max(g, 0) - |g| * q.
// All constant factors (1 / sqrt 2, 0.5, log2 e) are folded into the coefficients: 2 MUFU + 12 FP32 instructions per value
// (the erf_fast form above costs 16); the fc1 + GEGLU epilogue is bound by instruction issue.
__device__ __forceinline__ float gelu_fast(float g) {
  const float ag = fabsf(g);
  const float t = rcp_approx(fmaf(0.3275911f * 0.70710678118654752440f, ag, 1.f));
  float p = fmaf(0.5f * 1.061405429f, t, 0.5f * -1.453152027f);
  p = fmaf(p, t, 0.5f * 1.421413741f);
  p = fmaf(p, t, 0.5f * -0.284496736f);
  p = fmaf(p, t, 0.5f * 0.254829592f);
  const float e = ex2_approx((g * g) * (-0.5f * 1.4426950408889634f));
  const float q = (p * t) * e;
  return fmaf(-ag, q, fmaxf(g, 0.f));
}

// ReLU shares the LeakyReLU instantiation (a runtime flag), so the epilogues carry no extra code path
template <int ACT>
__device__ __forceinline__ float act_ct(float x, bool relu = false) {
  if (ACT == MV2_ACT_ELU) {
    const float e = ex2_approx(x * 1.4426950408889634f) - 1.f;
    return x > 0.f ? x : e;
  }
  if (ACT == MV2_ACT_SILU) return x * rcp_approx(1.f + ex2_approx(-1.4426950408889634f * x));
  if (ACT == MV2_ACT_LEAKY_RELU) return x > 0.f ? x : (relu ? 0.f * x : 0.1f * x);   // ReLU: NaN * 0 passes NaN, as torch
  return x;
}

// r: 32 raw accumulator columns of ONE output row (position b,to,ho,wo); n = first packed column; sb = smem bias of
// these columns (always valid memory; zeros when there is no bias).
// row_base = linear position index * Co (plain mode), computed once per row by the caller.
template <typename T, int MODE, int ACT>
__device__ __forceinline__ void epi_chunk32_t(const TcEpi& e, const uint32_t (&r)[32], int ncols, int n, const float* sb,
                                              int b, int to, int ho, int wo, int64_t row_base, bool relu = false) {
  if (MODE == EPI_GEGLU) {
    const int I = e.Co >> 1;
    const int64_t pos = (((int64_t)b * e.To + to) * e.Ho + ho) * e.Wo + wo;
#pragma unroll
    for (int g = 0; g < 2; ++g) {
      if (g * 16 >= ncols || n + g * 16 >= e.Co) break;
      float v[8];
#pragma unroll
      for (int q = 0; q < 8; ++q) {
        const float xv = __uint_as_float(r[g * 16 + q]) + sb[g * 16 + q];
        const float gt = __uint_as_float(r[g * 16 + 8 + q]) + sb[g * 16 + 8 + q];
        v[q] = gelu_fast(gt) * xv;
      }
      store8<T>((T*)e.y + pos * I + ((n + g * 16) >> 1), v);
    }
    return;
  }
  const int cy = MODE == EPI_SHUFFLE ? (e.shuffle == MV2_SHUFFLE_SPACE ? (e.Co >> 2) : (e.Co >> 1)) : e.Co;
  const bool vec_ok = (cy & 7) == 0;
#pragma unroll
  for (int g = 0; g < 4; ++g) {
    const int ng = n + g * 8;
    if (g * 8 >= ncols || ng >= e.Co) break;
    float v[8];
    {
      const float4 b0 = *reinterpret_cast<const float4*>(sb + g * 8), b1 = *reinterpret_cast<const float4*>(sb + g * 8 + 4);
      const float bb[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
      if (MODE != EPI_SHUFFLE && e.oscale) {      // Conv3DMod demodulation (M:741-742)
#pragma unroll
        for (int q = 0; q < 8; ++q) {
          const float os = ng + q < e.Co ? e.oscale[(int64_t)b * e.Co + ng + q] : 0.f;
          v[q] = act_ct<ACT>(__uint_as_float(r[g * 8 + q]) * os + bb[q], relu);
        }
      } else
#pragma unroll
      for (int q = 0; q < 8; ++q) v[q] = act_ct<ACT>(__uint_as_float(r[g * 8 + q]) + bb[q], relu);
    }
    int64_t off;
    if (MODE == EPI_SHUFFLE) {
      const int qd = ng / cy, c = ng - qd * cy;
      if (e.shuffle == MV2_SHUFFLE_SPACE) {
        const int p1 = qd >> 1, p2 = qd & 1;
        off = ((((int64_t)b * e.To + to) * (2 * e.Ho) + (2 * ho + p1)) * (2 * e.Wo) + (2 * wo + p2)) * cy + c;
      } else {
        off = ((((int64_t)b * (2 * e.To) + (2 * to + qd)) * e.Ho + ho) * e.Wo + wo) * cy + c;
      }
    } else {
      off = row_base + ng;
    }
    const float rscale = e.mode == 2 ? 0.70710678118654752440f : 1.f;
    if (vec_ok && ng + 8 <= e.Co) {
      if (e.res) {
        float rf[8];
        load8<T>((const T*)e.res + off, rf);
#pragma unroll
        for (int q = 0; q < 8; ++q) v[q] = (v[q] + rf[q]) * rscale;
      }
      store8<T>((T*)e.y + off, v);
    } else {
      if (MODE == EPI_RAGGED && e.out_cf) {            // conv_out: the reconstruction goes out in torch's (B, C, T, H, W)
        const int64_t plane = (int64_t)e.Ho * e.Wo;
        const int64_t o0 = ((int64_t)b * e.Co * e.To + to) * plane + (int64_t)ho * e.Wo + wo;
        for (int q = 0; q < 8 && ng + q < e.Co; ++q) ((T*)e.y)[o0 + (int64_t)(ng + q) * e.To * plane] = from_f32<T>(v[q]);
      } else
      for (int q = 0; q < 8 && ng + q < e.Co; ++q) {   // scalar tail (Co % 8 != 0, e.g. conv_out's 3 channels)
        float x = v[q];
        if (e.res) x = (x + to_f32(((const T*)e.res)[off + q])) * rscale;
        ((T*)e.y)[off + q] = from_f32<T>(x);
      }
    }
  }
}

// bias + activation + packing into T of one 32-column chunk (row-per-lane), for the staged epilogue
template <typename T, int ACT>
__device__ __forceinline__ void epi_pack32_t(const uint32_t (&r)[32], const float* sb, uint32_t (&pk)[16], bool relu = false) {
#pragma unroll
  for (int g = 0; g < 8; ++g) {
    const float4 b = *reinterpret_cast<const float4*>(sb + g * 4);
    pk[2 * g] = pack2<T>(act_ct<ACT>(__uint_as_float(r[4 * g]) + b.x, relu), act_ct<ACT>(__uint_as_float(r[4 * g + 1]) + b.y, relu));
    pk[2 * g + 1] = pack2<T>(act_ct<ACT>(__uint_as_float(r[4 * g + 2]) + b.z, relu), act_ct<ACT>(__uint_as_float(r[4 * g + 3]) + b.w, relu));
  }
}
template <typename T>
__device__ __forceinline__ void epi_pack32(int act, const uint32_t (&r)[32], const float* sb, uint32_t (&pk)[16]) {
  if (act == MV2_ACT_ELU) epi_pack32_t<T, MV2_ACT_ELU>(r, sb, pk);
  else if (act == MV2_ACT_SILU) epi_pack32_t<T, MV2_ACT_SILU>(r, sb, pk);
  else if (act == MV2_ACT_LEAKY_RELU || act == MV2_ACT_RELU) epi_pack32_t<T, MV2_ACT_LEAKY_RELU>(r, sb, pk, act == MV2_ACT_RELU);
  else epi_pack32_t<T, MV2_ACT_NONE>(r, sb, pk);
}

// activation is a kernel argument; dispatch once per chunk (warp uniform) into the compile-time variants
template <typename T, int MODE>
__device__ __forceinline__ void epi_chunk32(const TcEpi& e, const uint32_t (&r)[32], int ncols, int n, const float* sb,
                                            int b, int to, int ho, int wo, int64_t row_base) {
  if (MODE == EPI_GEGLU) { epi_chunk32_t<T, EPI_GEGLU, MV2_ACT_NONE>(e, r, ncols, n, sb, b, to, ho, wo, row_base); return; }
  if (e.act == MV2_ACT_ELU) epi_chunk32_t<T, MODE, MV2_ACT_ELU>(e, r, ncols, n, sb, b, to, ho, wo, row_base);
  else if (e.act == MV2_ACT_SILU) epi_chunk32_t<T, MODE, MV2_ACT_SILU>(e, r, ncols, n, sb, b, to, ho, wo, row_base);
  else if (e.act == MV2_ACT_LEAKY_RELU || e.act == MV2_ACT_RELU)
    epi_chunk32_t<T, MODE, MV2_ACT_LEAKY_RELU>(e, r, ncols, n, sb, b, to, ho, wo, row_base, e.act == MV2_ACT_RELU);
  else epi_chunk32_t<T, MODE, MV2_ACT_NONE>(e, r, ncols, n, sb, b, to, ho, wo, row_base);
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static inline EncodeTiledFn get_encode_fn() {
  static EncodeTiledFn fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* f = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &f, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = (EncodeTiledFn)f;
  });
  return fn;
}

// Hardware swizzle of a K-major operand tile with rows of row_bytes (128 / 64 / 32 bytes), as gmma_desc_hi describes it
static inline CUtensorMapSwizzle swizzle_of_row(int row_bytes) {
  return row_bytes == 128 ? CU_TENSOR_MAP_SWIZZLE_128B : (row_bytes == 64 ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_32B);
}

// One tiled tensor map of the elements of a tensor-core conv (dtype MV2_BF16, MV2_F16 or MV2_TF32: fp32): dims and box
// innermost first, byte strides of dims 1 .. rank-1, unit element strides, 256-byte L2 promotion; box elements outside the
// tensor are zero-filled.  `what` names the map in the error message.
static inline int encode_tc_map(CUtensorMap* map, int dtype, int rank, const void* base, const cuuint64_t* dims,
                                const cuuint64_t* strides, const cuuint32_t* box, CUtensorMapSwizzle swz, const char* what) {
  const EncodeTiledFn enc = get_encode_fn();
  if (!enc) { set_error("cuTensorMapEncodeTiled entry point unavailable"); return MV2_E_CUDA; }
  const cuuint32_t es[5] = {1, 1, 1, 1, 1};
  const CUtensorMapDataType dt = dtype == MV2_F16 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16
                                 : (dtype == MV2_TF32 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16);
  const CUresult r = enc(map, dt, (cuuint32_t)rank, const_cast<void*>(base), dims, strides, box, es,
                         CU_TENSOR_MAP_INTERLEAVE_NONE, swz, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) { set_error("cuTensorMapEncodeTiled(%s) failed: %d", what, (int)r); return MV2_E_CUDA; }
  return MV2_OK;
}

// Epilogue arguments of a tensor-core conv launch
static inline TcEpi tc_epi_of(const mv2_tc_conv_args* a) {
  TcEpi e = {};
  e.bias = a->bias; e.res = a->res; e.y = a->y;
  e.act = a->act; e.shuffle = a->shuffle; e.mode = a->epi_mode; e.Co = a->Co;
  e.To = a->To; e.Ho = a->Ho; e.Wo = a->Wo; e.out_cf = a->out_layout == 1; e.oscale = a->oscale;
  return e;
}

// Element type of a tensor-core conv launch: MV2_BF16 (also for 0, the value of a zero-initialised struct), MV2_F16 or
// MV2_TF32; -1 for anything else
static inline int tc_dtype_of(int32_t d) {
  return d == 0 || d == MV2_BF16 ? MV2_BF16 : (d == MV2_F16 || d == MV2_TF32 ? d : -1);
}
static inline int tc_dtype(const mv2_tc_conv_args* a) { return tc_dtype_of(a->dtype); }
// Bytes per stored element of a tensor-core dtype: the host plans and maps in bytes, the kernels in elements of T
static inline int tc_esize(int dtype) { return dtype == MV2_TF32 ? 4 : 2; }

static inline int pow2_ceil(int v) { int r = 1; while (r < v) r <<= 1; return r; }
static inline int floor_div(int a, int b) { int q = a / b; if ((a % b != 0) && ((a < 0) != (b < 0))) --q; return q; }


}  // namespace mv2
