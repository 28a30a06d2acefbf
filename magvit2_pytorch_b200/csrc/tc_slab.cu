// wgmma / TMA "slab" implicit-GEMM kernel for stride-1 k_t x k_h x k_w convolutions (the causal 3x3x3 residual
// convs carry most of the path's FLOPs), bf16, fp16 or fp32 (TF32 multiply) in (the element type T is a template
// parameter of every kernel) / fp32 accumulate in registers, persistent CTAs, sm_90a.  The host plans in bytes: a 128-byte
// K row holds 64 bf16 / fp16 channels or 32 fp32 ones and takes the same four 32-byte MMA K steps.
//
// Why a second kernel: tc_conv.cu reloads the activation tile from L2 once per tap (27x) and the weight tile once per
// 128 output positions.  Here
//   * one TMA box load brings a haloed activation slab {64 ch, 8*mw + kw - 1, 16 + kh - 1} (one frame, one 64-channel
//     slice) into shared memory ONCE and all k_h*k_w in-plane taps are fed from it: the wgmma A descriptor is simply
//     started (dh*pitch + dw) rows further into the slab (128-byte rows; the hardware SWIZZLE_128B is a function of the
//     absolute shared-memory address, so row-shifted starts stay consistent with what TMA wrote; 8-row core groups are
//     8 consecutive w positions, group stride (SBO) = slab row pitch);
//   * a macro tile is mw (1|2|4) M-tiles of 16(h) x 8(w) positions side by side; all of them consume the same weight
//     tile from shared memory, dividing weight traffic by mw (mw * bn <= 128: the mw accumulators of a consumer
//     warpgroup fit 64 fp32 registers per thread);
//   * CTAs are persistent with a static, cost-sorted serpentine tile schedule (slab_frame_of / slab_tile_of);
//   * causal frames in front of the clip (t + dt - pt < 0) come from the history map (hmap: the tail of the previous chunk
//     of a streamed clip, hist_T frames); those in front of the history are all-zero and are skipped outright;
//   * N tiles need not divide Co (TMA clips the plain / GEGLU stores at Co): wide outputs without a
//     128-column divisor take 128-column tiles with a ragged last one;
//   * the kernel is instantiated per epilogue flavour (tc_common.cuh: EPI_*) and N tile (32 / 64 / 128); the plain,
//     residual, GEGLU, SpatialDownsample2x and fused ResidualUnit flavours run the epilogue on the accumulator fragments
//     and store bf16 / fp16 boxes through TMA (slab_epi_mtile), the others stage the accumulators in shared memory first.
//     The channels-first flavour (EPI_RAGGED: fewer than 32 output channels, so never a wider tile than 32) has narrow
//     8- and 16-column tiles (wgmma m64n8k16 / m64n16k16) instead, for the data gradient of conv_in with respect to the
//     video: 3 output channels, 7 x 7 in-plane taps (slab_narrow).
// Warp roles (384 threads): w0 slab TMA producer, w1 residual TMA producer (EPI_PLAIN_RES), w2 weight TMA producer
// (40 registers each, setmaxnreg), w4-7 / w8-11 two consumer warpgroups (232 registers): each issues the wgmma of 64 of
// the 128 positions of every M-tile, with one commit group in flight across ring stages, and runs the epilogue.
#include "common.cuh"
#include "tc_common.cuh"
#include <cuda.h>
#include <algorithm>
#include <type_traits>
#include <mutex>
#include <map>
#include <vector>
#include <string.h>

namespace mv2 {

struct alignas(64) SlabParams {
  CUtensorMap amap;
  CUtensorMap hmap;      // history frames in front of x (mv2_conv_hist), hist_T of them; unused when hist_T = 0
  CUtensorMap wmap;      // weights as {ci, co, tap} (3-D boxes of tpw taps)
  CUtensorMap wmap2;     // weights as {k, co} (2-D boxes, used when tpw == 1)
  int kt, kh, kw, pt, ph, pw;
  int st;                // stride along t (1, or 2: TimeDownsample2x); spatial strides are always 1 in this kernel
  int hist_T;
  int Ci, kchunks, row_bytes;
  int B, T, H, W, Co;
  int mw, pitch, slab_h, slab_bytes, slab_stride;
  int bn, n_tiles_n, tiles_w, tiles_h, total_tiles;
  int slab_stages, w_stages;
  int tpw;               // in-plane taps per weight stage (one 3-D TMA box {bk, bn, tpw})
  TcEpi epi;
  int dtype;             // host side: MV2_BF16, MV2_F16 or MV2_TF32, selects the kernel instance and the tensor maps' element type
  // ---- EPI_FUSED_RU only (mv2_tc_ru_forward) ----
  CUtensorMap w1map;     // 1x1x1 weights [Co][Ci] as {ci, co}: 2-D boxes {64, bn}
  const float* bias1;    // 1x1x1 bias [C]
  const float* se_wk;    // SqueezeExcite to_k weight [C]
  float se_bk;
  float* se_ws;          // SE pool records [B*T][recs_per_frame][C + 2] = (max, sum, sum e*y[C]) per 32-position row group
  // ---- EPI_DOWN_SPACE only (mv2_tc_down_space_forward) ----
  CUtensorMap amap_odd;  // odd input rows (amap: even rows), both over x viewed as {2C, W/2, H/2, T, B}
  int dn_e_off;          // byte offset of the even-row sub-slab inside a slab stage
  int dn_aoff[6];        // per tap' = dh * 2 + (dw2 + 1): A-descriptor start offset inside the stage, in 16-byte units
  int dn_lower;          // K-chunks of the lower (pw = 0) half of the 2C axis: they only see the dw2 = 0 taps
  int h_stride;          // bytes of the shared-memory H buffer (ELU'd 3x3x3 tile of one M-tile) = kchunks * 16 KB
  // ---- TMA-store flavours (slab_tma_epi: EPI_PLAIN, EPI_PLAIN_RES, EPI_GEGLU, EPI_DOWN_SPACE; and EPI_FUSED_RU) ----
  CUtensorMap ymap;      // y as {Co (GEGLU: Co / 2), W, H, T, B}: boxes {cb, 8, 8, 1, 1}, one per 64 positions and cb channels
  CUtensorMap rmap;      // EPI_PLAIN_RES: the residual, same view and boxes as ymap
};

// Flavours whose epilogue runs on the accumulator fragments and stores through TMA (slab_epi_fragment).  The fused
// ResidualUnit does both too, with its own epilogue around the second GEMM; the others stage the accumulators in shared
// memory first (the channels-first and shuffled stores need a row per thread).
__host__ __device__ constexpr bool slab_tma_epi(int mode) {
  return mode == EPI_PLAIN || mode == EPI_PLAIN_RES || mode == EPI_GEGLU || mode == EPI_DOWN_SPACE;
}
// Channels of one output box of a TMA-store flavour with an N tile of bn columns and es-byte elements: one 128-byte
// swizzled row (64 bf16 / fp16 or 32 fp32 channels), or the whole tile when its output is narrower (GEGLU writes bn / 2
// channels)
__host__ __device__ constexpr int slab_out_box_ch(int mode, int bn, int es) {
  return (mode == EPI_GEGLU ? bn / 2 : bn) < 128 / es ? (mode == EPI_GEGLU ? bn / 2 : bn) : 128 / es;
}

// Frames are enumerated most-expensive first: the B * (T - pt) frames that see all kt frame taps, then the frames
// t = pt-1, pt-2, ..., 0 of every clip (their leading taps fall into the causal padding and are skipped, so their tiles
// cost (kt-1)/kt ... 1/kt of a full one).  Together with the serpentine CTA assignment (slab_tile_of) a static schedule
// then behaves like longest-processing-time-first list scheduling: with few tiles per CTA no CTA gets three full tiles
// while others get two.  Pure index arithmetic, shared by every warp of the CTA and by the host-side tests.
__host__ __device__ __forceinline__ void slab_frame_of(const SlabParams& p, int slot, int& b, int& t) {
  const int ptc = p.pt > 0 ? (p.pt + p.st - 1) / p.st : 0;   // output frames whose leading taps fall into the causal padding
                                                              // (pt < 0: cropped conv_out output, none)
  const int n_cheap = ptc < p.T ? ptc : p.T, n_full = p.T - n_cheap;
  const int full_slots = p.B * n_full;
  if (slot < full_slots) { b = slot / n_full; t = n_cheap + slot - b * n_full; }
  else { const int r = slot - full_slots; const int level = r / p.B; b = r - level * p.B; t = n_cheap - 1 - level; }
}
// k-th tile of CTA `cta` of `grid`: waves alternate direction (serpentine) so the CTAs that finish a wave first start the
// next one first.  (mv2_tc_slab_tile exposes the same function to the host-side tests.)
__host__ __device__ __forceinline__ int slab_tile_of_cta(const SlabParams& p, int k, int cta, int grid) {
  const int tile = k * grid + ((k & 1) ? grid - 1 - cta : cta);
  return tile < p.total_tiles ? tile : -1;
}
__device__ __forceinline__ int slab_tile_of(const SlabParams& p, int k) { return slab_tile_of_cta(p, k, blockIdx.x, gridDim.x); }

struct TileCoord { int b, t, h0, w0, n0; };
__host__ __device__ __forceinline__ TileCoord decode_tile(const SlabParams& p, int tile) {
  TileCoord c;
  // n-tile fastest: CTAs running side by side share the activation slab through L2
  const int nt = tile % p.n_tiles_n; tile /= p.n_tiles_n;
  const int tw = tile % p.tiles_w; tile /= p.tiles_w;
  const int th = tile % p.tiles_h; tile /= p.tiles_h;
  slab_frame_of(p, tile, c.b, c.t);
  c.h0 = th * 16;
  c.w0 = tw * 8 * p.mw;
  c.n0 = nt * p.bn;
  return c;
}

// Shared-memory layout behind the two TMA rings (host and kernel must agree): barriers, bias, the eight 2 KB
// epilogue transpose buffers, the fp32 accumulator staging of both consumer warpgroups (mw M-tiles x 64 rows x (bn + 4)
// each).
// The TMA-store flavours use the span of the transpose buffers and the staging for other things: the residual
// full / empty barriers of both warpgroups, then (1024-byte aligned, for the swizzled boxes) the output tiles and
// the residual tiles of both warpgroups, 2 x mw x 64 x bn x es bytes each (es-byte elements).  With 16-bit elements
// they take at most 32 + 1023 + 512 mw bn bytes of the 16 KB + 512 mw (bn + 4) the span has, so the span, and with it
// every launch's plan, is the same for all flavours but the fused one.  fp32 tiles take twice that: the output tiles
// still fit the span, the residual tiles (launches with a residual only) extend it.
// The fused ResidualUnit stages nothing: bias, logit partials, then (1024-byte aligned) the H buffer and the output
// tiles of both warpgroups.
struct SlabSmem { uint32_t sbias, stage0, lpart, accstg, hbuf, end, rbar, otile, rtile; };
__host__ __device__ __forceinline__ SlabSmem slab_smem_layout(const SlabParams& p, uint32_t bar0, bool fused, uint32_t es) {
  SlabSmem m = {};
  m.sbias = (bar0 + 8 * (2 * p.slab_stages + 2 * p.w_stages) + 15) & ~15u;
  m.stage0 = m.sbias + (uint32_t)(p.n_tiles_n * p.bn) * 4 * (fused ? 3 : 1);   // fused: [conv3 bias][conv1 bias][SE to_k weight]
  if (fused) {
    m.lpart = m.stage0;
    m.hbuf = (m.lpart + 2048 + 1023u) & ~1023u;          // SWIZZLE_128B tiles: 1024-byte aligned
    m.otile = m.hbuf + (uint32_t)p.h_stride;
    m.end = m.otile + 2u * p.mw * 64 * p.bn * es;
    return m;
  }
  m.accstg = m.stage0 + 8 * 2048;
  m.end = m.accstg + 2u * p.mw * 64 * (p.bn + 4) * 4;
  m.rbar = m.stage0;
  m.otile = (m.rbar + 32 + 1023u) & ~1023u;
  m.rtile = m.otile + 2u * p.mw * 64 * p.bn * es;
  const uint32_t tiles_end = m.rtile + (p.epi.res ? 2u * p.mw * 64 * p.bn * es : 0u);   // residual tiles: EPI_PLAIN_RES only
  if (tiles_end > m.end) m.end = tiles_end;
  return m;
}

// Epilogue of the TMA-store flavours on one M-tile of a consumer warpgroup's accumulators, in fragment layout: thread
// (warp wq of the warpgroup, lane) holds rows m0 = 16 wq + lane / 4 and m0 + 8 of the M-tile (row m = output position
// (h0 + 8 wg + m / 8, w0 + 8 j + m % 8)) and columns 8 g + 2 (lane % 4) + {0, 1}.  The math per element is that of the
// staged epilogue, in the same order: x oscale, + bias and activation, [+ residual in fp32, x 2^-0.5 in mode 2], one
// rounding to bf16 / fp16 (fp32 is stored as computed); GEGLU pairs packed column 16 g + c (x) with 16 g + 8 + c (its
// gate), which the same thread holds.
// Results go to `ot` as [boxes][64 rows][cb channels] boxes of T in the swizzle TMA uses for their row width; the
// residual is read from `rt` in the same layout.  Bank-conflict free: the 8 rows of a warp's access fall on 8 different
// 16-byte units of the swizzle.  With 128-byte rows this is also the layout of a K-major SWIZZLE_128B wgmma operand of
// 64 rows (one 8 KB K-chunk per box), which the fused ResidualUnit's second GEMM reads.
template <typename T, int MODE, int BN, int ACT>
__device__ __forceinline__ void slab_epi_mtile(const SlabParams& p, const float (&acc)[BN / 2], const TileCoord& c,
                                               const float* sbias, uint32_t ot, uint32_t rt, int wq, int lane, bool relu) {
  constexpr int ES = sizeof(T);
  constexpr int CB = slab_out_box_ch(MODE, BN, ES);
  constexpr uint32_t RB = CB * ES, BOX = 64 * RB, SWZ = (RB / 16 - 1) << 4;
  const uint32_t m0 = 16 * wq + (lane >> 2), q4 = (lane & 3) * 2 * ES;
  auto at = [&](int col, uint32_t m) {               // byte offset of (row m, output columns col, col + 1)
    const uint32_t off = m * RB + (uint32_t)(col % CB) * ES + q4;
    return (uint32_t)(col / CB) * BOX + (off ^ ((off >> 3) & SWZ));
  };
  auto st2 = [](uint32_t a, float v0, float v1) {   // two adjacent output columns
    if constexpr (ES == 4) asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(a), "f"(v0), "f"(v1) : "memory");
    else asm volatile("st.shared.b32 [%0], %1;" ::"r"(a), "r"(pack2<T>(v0, v1)) : "memory");
  };
  const float* os = (MODE == EPI_PLAIN || MODE == EPI_PLAIN_RES) && p.epi.oscale ? p.epi.oscale + (int64_t)c.b * p.Co : nullptr;
  const float rs = MODE == EPI_PLAIN_RES && p.epi.mode == 2 ? 0.70710678118654752440f : 1.f;
  if (MODE == EPI_GEGLU) {
#pragma unroll
    for (int g = 0; g < BN / 16; ++g) {
      const int n = c.n0 + 16 * g + 2 * (lane & 3);
      const float2 bx = *reinterpret_cast<const float2*>(sbias + n), bg = *reinterpret_cast<const float2*>(sbias + n + 8);
#pragma unroll
      for (int hr = 0; hr < 2; ++hr) {
        const float* xv = &acc[8 * g + 2 * hr];
        const float* gv = &acc[8 * g + 4 + 2 * hr];
        const float v0 = gelu_fast(gv[0] + bg.x) * (xv[0] + bx.x);
        const float v1 = gelu_fast(gv[1] + bg.y) * (xv[1] + bx.y);
        st2(ot + at(8 * g, m0 + 8 * hr), v0, v1);
      }
    }
  } else {
#pragma unroll
    for (int g = 0; g < BN / 8; ++g) {
      const int col = 8 * g, n = c.n0 + col + 2 * (lane & 3);
      const float2 b = *reinterpret_cast<const float2*>(sbias + n);
      float o0 = 1.f, o1 = 1.f;
      if (os) { o0 = n < p.Co ? os[n] : 0.f; o1 = n + 1 < p.Co ? os[n + 1] : 0.f; }
#pragma unroll
      for (int hr = 0; hr < 2; ++hr) {
        float v0 = acc[4 * g + 2 * hr], v1 = acc[4 * g + 2 * hr + 1];
        if (os) { v0 *= o0; v1 *= o1; }
        v0 = act_ct<ACT>(v0 + b.x, relu);
        v1 = act_ct<ACT>(v1 + b.y, relu);
        const uint32_t a = at(col, m0 + 8 * hr);
        if (MODE == EPI_PLAIN_RES) {
          float2 rf;
          if constexpr (ES == 4) {
            asm volatile("ld.shared.v2.f32 {%0, %1}, [%2];" : "=f"(rf.x), "=f"(rf.y) : "r"(rt + a) : "memory");
          } else {
            uint32_t r;
            asm volatile("ld.shared.b32 %0, [%1];" : "=r"(r) : "r"(rt + a) : "memory");
            rf = unpack2<T>(r);
          }
          v0 = (v0 + rf.x) * rs;
          v1 = (v1 + rf.y) * rs;
        }
        st2(ot + a, v0, v1);
      }
    }
  }
}
// All M-tiles of a warpgroup: output and residual tiles as [mw][boxes][64 rows][cb channels]
template <typename T, int MODE, int BN, int ACT, int MWMAX>
__device__ __forceinline__ void slab_epi_fragment(const SlabParams& p, const float (&acc)[MWMAX][BN / 2], const TileCoord& c,
                                                  const float* sbias, uint32_t ot, uint32_t rt, int wq, int lane, bool relu) {
  constexpr uint32_t MTILE = (MODE == EPI_GEGLU ? BN / 2 : BN) * 64 * (int)sizeof(T);   // bytes of one M-tile's boxes
#pragma unroll
  for (int j = 0; j < MWMAX; ++j) {
    if (j >= p.mw) break;
    slab_epi_mtile<T, MODE, BN, ACT>(p, acc[j], c, sbias, ot + j * MTILE, rt + j * MTILE, wq, lane, relu);
  }
}

// Every instantiation runs 384 threads: warp 0 slab TMA producer, warp 2 weight TMA producer, warp 1 residual TMA producer
// (EPI_PLAIN_RES; otherwise idle, as is warp 3), warps
// 4-11 are two consumer warpgroups.  Consumer warpgroup g issues the wgmma of output rows h0 + 8g .. h0 + 8g + 7 of every
// M-tile (64 positions) against all bn columns, keeping mw accumulators of 64 x bn in registers (mw * bn <= 128: at most
// 64 fp32 registers per thread), then runs the epilogue on them.
// Register split: the launch gives every thread 168 registers (384 x 168 = 64,512); the producer warpgroup drops to
// SLAB_PRODUCER_REGS and the consumers take the freed registers (128 x 40 + 256 x 232 = 64,512).
constexpr int SLAB_PRODUCER_REGS = 40, SLAB_CONSUMER_REGS = 232;
template <typename T, int MODE, int BN>
__device__ __forceinline__ void tc_slab_body(const SlabParams& p) {
  constexpr int MWMAX = BN >= 32 ? 128 / BN : 4;        // mw <= 4 (slab_default_mw)
  constexpr int KC1 = BN >= 64 ? BN / 64 : 1;   // EPI_FUSED_RU (bn = C = 64 | 128): 64-channel K-chunks of the 1x1x1 GEMM
  constexpr bool TMA_STORE = slab_tma_epi(MODE) || MODE == EPI_FUSED_RU;   // y leaves through TMA box stores
  extern __shared__ uint8_t smem_raw[];
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const uint32_t row_bytes = p.row_bytes;          // 128 (SWIZZLE_128B) or 64 (SWIZZLE_64B)
  const uint32_t bk = row_bytes / (uint32_t)sizeof(T);   // channels of one K row
  const uint32_t w_tile = p.bn * row_bytes;          // one tap's weight tile
  const uint32_t w_bytes = w_tile * p.tpw;           // one ring stage = tpw consecutive in-plane taps
  const uint32_t slab0 = smem_base;
  const uint32_t wst0 = smem_base + p.slab_stages * p.slab_stride;
  const uint32_t bar0 = wst0 + p.w_stages * w_bytes;
  // barrier table (8 bytes each)
  const uint32_t slab_full = bar0, slab_empty = slab_full + 8 * p.slab_stages;
  const uint32_t w_full = slab_empty + 8 * p.slab_stages, w_empty = w_full + 8 * p.w_stages;
  const SlabSmem L = slab_smem_layout(p, bar0, MODE == EPI_FUSED_RU, (uint32_t)sizeof(T));
  auto gen = [&](uint32_t u) { return smem_raw + (u - smem_u32(smem_raw)); };
  float* sbias = reinterpret_cast<float*>(gen(L.sbias));   // padded Co floats, 16-byte aligned
  const uint32_t nbias = (uint32_t)(p.n_tiles_n * p.bn);
  const uint32_t stage0 = L.stage0;                        // one 2 KB transpose buffer per epilogue warp (32 rows x 64 B)

  if (threadIdx.x == 0) {
    // empty barriers: one arrival per consumer warp once its wgmma of the stage have completed
    for (int s = 0; s < p.slab_stages; ++s) { mbar_init(slab_full + 8 * s, 1); mbar_init(slab_empty + 8 * s, 8); }
    for (int s = 0; s < p.w_stages; ++s) { mbar_init(w_full + 8 * s, 1); mbar_init(w_empty + 8 * s, 8); }
    // residual tile of each consumer warpgroup: full = the producer's TMA loads, empty = one arrival per consumer warp
    if (MODE == EPI_PLAIN_RES)
      for (int g = 0; g < 2; ++g) { mbar_init(L.rbar + 8 * g, 1); mbar_init(L.rbar + 16 + 8 * g, 4); }
    fence_barrier_init();
  }
  if (warp == 0 && lane == 0) {
    tma_prefetch_desc(&p.amap);
    if (MODE == EPI_DOWN_SPACE) tma_prefetch_desc(&p.amap_odd);
    else if (p.hist_T > 0) tma_prefetch_desc(&p.hmap);
  }
  if (warp == 2 && lane == 0) {
    tma_prefetch_desc(&p.wmap); tma_prefetch_desc(&p.wmap2);
    if (MODE == EPI_FUSED_RU) tma_prefetch_desc(&p.w1map);
  }
  if (TMA_STORE && warp == 1 && lane == 0) {
    tma_prefetch_desc(&p.ymap);
    if (MODE == EPI_PLAIN_RES) tma_prefetch_desc(&p.rmap);
  }
  if (warp >= 4) {
    const int nb = p.n_tiles_n * p.bn;   // >= Co; padded columns read zeros
    for (int i = threadIdx.x - 128; i < nb; i += 256) sbias[i] = (p.epi.bias && i < p.Co) ? p.epi.bias[i] : 0.f;
    if (MODE == EPI_FUSED_RU)
      for (int i = threadIdx.x - 128; i < nb; i += 256) {
        sbias[nb + i] = (p.bias1 && i < p.Co) ? p.bias1[i] : 0.f;
        sbias[2 * nb + i] = i < p.Co ? p.se_wk[i] : 0.f;
      }
  }
  __syncthreads();
  // everything above overlapped the previous kernel's tail (PDL); activations may only be touched from here on
  pdl_wait();
  pdl_launch_dependents();

  const int taps2d = p.kh * p.kw;

  if (warp < 4) {
    // every warp of the producer warpgroup, the idle ones included, gives up its registers (one setmaxnreg for the
    // warpgroup) before any of them returns: the consumers' setmaxnreg.inc waits until the SM's register file has them
    setmaxnreg_dec<SLAB_PRODUCER_REGS>();
    if (warp == 0) {
      // ------------------------------ slab producer ------------------------------
      if (MODE == EPI_DOWN_SPACE) {
        // one stage = the odd-row sub-slab (input rows 2*ho - 1: 17 rows for 16 output rows) + the even-row sub-slab (rows 2*ho)
        // of one 64-channel chunk of the (W/2) x (2C) view; w2 starts one position to the left (the dw = 0 tap), OOB = zero pad
        if (lane == 0) {
          uint32_t s = 0, ph = 0;
          for (int tk = 0, tile; (tile = slab_tile_of(p, tk)) >= 0; ++tk) {
            const TileCoord c = decode_tile(p, tile);
            for (int kc = 0; kc < p.kchunks; ++kc) {
              mbar_wait(slab_empty + 8 * s, ph ^ 1);
              mbar_expect_tx(slab_full + 8 * s, p.slab_bytes);
              tma_load_5d(slab0 + s * p.slab_stride, &p.amap_odd, slab_full + 8 * s, kc * bk, c.w0 - 1, c.h0 - 1, c.t, c.b);
              tma_load_5d(slab0 + s * p.slab_stride + p.dn_e_off, &p.amap, slab_full + 8 * s, kc * bk, c.w0 - 1, c.h0, c.t, c.b);
              if (++s == (uint32_t)p.slab_stages) { s = 0; ph ^= 1; }
            }
          }
        }
      } else
      if (lane == 0) {
        uint32_t s = 0, ph = 0;
        for (int tk = 0, tile; (tile = slab_tile_of(p, tk)) >= 0; ++tk) {
          const TileCoord c = decode_tile(p, tile);
          const int dt0 = max(0, p.pt - c.t * p.st - p.hist_T);
          for (int dt = dt0; dt < p.kt; ++dt)
            for (int kc = 0; kc < p.kchunks; ++kc) {
              mbar_wait(slab_empty + 8 * s, ph ^ 1);
              mbar_expect_tx(slab_full + 8 * s, p.slab_bytes);
              const int ti = c.t * p.st + dt - p.pt;
              tma_load_5d(slab0 + s * p.slab_stride, ti >= 0 ? &p.amap : &p.hmap, slab_full + 8 * s, kc * bk, c.w0 - p.pw,
                          c.h0 - p.ph, ti >= 0 ? ti : ti + p.hist_T, c.b);
              if (++s == (uint32_t)p.slab_stages) { s = 0; ph ^= 1; }
            }
        }
      }
    } else if (warp == 1) {
      // ------------------------------ residual producer (EPI_PLAIN_RES) ------------------------------
      // loads the boxes of a tile's residual that hold output positions and channels (the boxes of slab_epi_fragment)
      // as soon as the warpgroup has read the previous tile's, so that they arrive under the tile's main loop
      if (MODE == EPI_PLAIN_RES && lane == 0) {
        constexpr int CB = slab_out_box_ch(MODE, BN, sizeof(T)), NB = BN / CB;
        constexpr uint32_t BOX = 64 * CB * (uint32_t)sizeof(T);
        uint32_t ph = 0;
        for (int tk = 0, tile; (tile = slab_tile_of(p, tk)) >= 0; ++tk) {
          const TileCoord c = decode_tile(p, tile);
          for (int g = 0; g < 2; ++g) {
            const uint32_t rt = L.rtile + (uint32_t)(g * p.mw * NB) * BOX;
            const int h = c.h0 + 8 * g;
            int nbox = 0;
            for (int j = 0; j < p.mw; ++j)
              for (int b = 0; b < NB; ++b) nbox += h < p.H && c.w0 + 8 * j < p.W && c.n0 + b * CB < p.Co;
            mbar_wait(L.rbar + 16 + 8 * g, ph ^ 1);
            mbar_expect_tx(L.rbar + 8 * g, (uint32_t)nbox * BOX);
            for (int j = 0; j < p.mw; ++j)
              for (int b = 0; b < NB; ++b)
                if (h < p.H && c.w0 + 8 * j < p.W && c.n0 + b * CB < p.Co)
                  tma_load_5d(rt + (uint32_t)(j * NB + b) * BOX, &p.rmap, L.rbar + 8 * g, c.n0 + b * CB, c.w0 + 8 * j, h, c.t, c.b);
          }
          ph ^= 1;
        }
      }
    } else if (warp == 2) {
      // ------------------------------ weight producer ------------------------------
      if (MODE == EPI_DOWN_SPACE) {
        if (lane == 0) {
          uint32_t s = 0, ph = 0;
          const int C2 = p.Ci;                 // channels of the paired view (2C)
          for (int tk = 0, tile; (tile = slab_tile_of(p, tk)) >= 0; ++tk) {
            const TileCoord c = decode_tile(p, tile);
            for (int kc = 0; kc < p.kchunks; ++kc)
              for (int tap = kc < p.dn_lower ? 1 : 0; tap < 6; tap += kc < p.dn_lower ? 2 : 1) {
                mbar_wait(w_empty + 8 * s, ph ^ 1);
                mbar_expect_tx(w_full + 8 * s, w_tile);
                tma_load_2d(wst0 + s * w_bytes, &p.wmap2, w_full + 8 * s, tap * C2 + kc * (int)bk, c.n0);
                if (++s == (uint32_t)p.w_stages) { s = 0; ph ^= 1; }
              }
          }
        }
      } else
      if (lane == 0) {
        uint32_t s = 0, ph = 0;
        for (int tk = 0, tile; (tile = slab_tile_of(p, tk)) >= 0; ++tk) {
          const TileCoord c = decode_tile(p, tile);
          const int dt0 = max(0, p.pt - c.t * p.st - p.hist_T);
          for (int dt = dt0; dt < p.kt; ++dt)
            for (int kc = 0; kc < p.kchunks; ++kc)
              for (int tp = 0; tp < taps2d; tp += p.tpw) {
                mbar_wait(w_empty + 8 * s, ph ^ 1);
                mbar_expect_tx(w_full + 8 * s, w_bytes);
                if (p.tpw == 1) tma_load_2d(wst0 + s * w_bytes, &p.wmap2, w_full + 8 * s, (dt * taps2d + tp) * p.Ci + kc * bk, c.n0);
                else tma_load_3d(wst0 + s * w_bytes, &p.wmap, w_full + 8 * s, kc * bk, c.n0, dt * taps2d + tp);
                if (++s == (uint32_t)p.w_stages) { s = 0; ph ^= 1; }
              }
          // EPI_FUSED_RU: the tile's last KC1 stages are the 1x1x1 weights (tpw = 1, one 64-channel K-chunk each), which
          // the second GEMM of every M-tile of the tile reads
          if (MODE == EPI_FUSED_RU)
            for (int kc2 = 0; kc2 < KC1; ++kc2) {
              mbar_wait(w_empty + 8 * s, ph ^ 1);
              mbar_expect_tx(w_full + 8 * s, w_tile);
              tma_load_2d(wst0 + s * w_bytes, &p.w1map, w_full + 8 * s, kc2 * (int)bk, 0);
              if (++s == (uint32_t)p.w_stages) { s = 0; ph ^= 1; }
            }
        }
      }
    }
  } else {
    setmaxnreg_inc<SLAB_CONSUMER_REGS>();
    // ------------------------------ consumer warpgroups: wgmma main loop + epilogue ------------------------------
    const int wg = (warp - 4) >> 2, wq = warp & 3, tid = threadIdx.x & 127;
    // epilogue roles: 32-row quarter `sub` of the M-tile (rows sub*32 .. +31 = output rows h0 + 4 sub .. +3, all 8 w) and
    // column half `half`; ew numbers the 8 epilogue warps (transpose buffer, logit exchange)
    const int sub = 2 * wg + (wq & 1), half = wq >> 1, ew = sub + 4 * half;
    const int row = sub * 32 + lane;
    const int lh = row >> 3, lw = row & 7;
    float* stg = reinterpret_cast<float*>(gen(L.accstg)) + (size_t)wg * p.mw * 64 * (BN + 4);   // [mw][64][BN + 4]
    const uint32_t wg_bar = 5 + wg;                          // named barrier of this warpgroup (1..4: logit exchange pairs)
    const uint32_t sbo = (uint32_t)p.pitch * row_bytes;
    const uint64_t a_hi = gmma_desc_hi(sbo, row_bytes);
    const uint64_t b_hi = gmma_desc_hi(8 * row_bytes, row_bytes);
    const bool k4 = row_bytes == 128;
    // All ring bookkeeping is incremental (stage index, parity, descriptor low words).
    const uint32_t a_row = row_bytes >> 4;                       // descriptor-address units per slab row
    const uint32_t a_wg = (uint32_t)wg * 8 * (sbo >> 4);         // this warpgroup's first output row: 8 slab rows (h) down
    const uint32_t a_next_dh = (uint32_t)(p.pitch - p.kw + 1) * a_row;
    const uint32_t a_mtile = 8 * a_row;                          // next M-tile: 8 positions further along w
    const uint32_t w_tile16 = w_tile >> 4, w_stage16 = w_bytes >> 4;
    const uint32_t b_lo0 = desc_lo(wst0);
    uint32_t s_idx = 0, s_par = 0;                               // slab ring
    uint32_t w_idx = 0, w_par = 0, b_lo = b_lo0;                 // weight ring
    uint32_t ecount = 0;       // EPI_FUSED_RU: M-tiles processed (selects the logit exchange buffer)
    uint32_t r_par = 0;        // EPI_PLAIN_RES: parity of the residual tile's full barrier
    float acc[MWMAX][BN / 2];
    // Main loop of one tile, compiled per M-tile count MW (= p.mw) and K steps per 64-byte half row (K4: 128-byte rows),
    // so that every commit group is straight-line code with constant accumulator indices: ptxas closes a group early at
    // any branch inside it, which would leave nothing but an empty MMA in flight.
    // One commit group (the MMAs of one tap) stays in flight: after committing group g the warpgroup waits until g - 1
    // has completed (wait_group 1).  When g - 1 was the last tap of its weight stage, that weight slot is released, and
    // when it was also the last reading its slab stage, that slab slot too (one arrival per consumer warp and slot).
    // The tile's last group is retired with wait_group 0.
    auto mainloop = [&](const TileCoord& c, auto mw_c, auto k4_c) {
      constexpr int MW = decltype(mw_c)::value;
      constexpr bool K4 = decltype(k4_c)::value;
      constexpr uint32_t NONE = ~0u;
      uint32_t accum = 0, pend_w = NONE, pend_s = NONE;
      auto release_pending = [&]() {
        __syncwarp();
        if (lane == 0) {
          if (pend_w != NONE) mbar_arrive(w_empty + 8 * pend_w);
          if (pend_s != NONE) mbar_arrive(slab_empty + 8 * pend_s);
        }
      };
      // after a commit: retire the previous group, then hold the slots (or NONE) the group just committed frees once done
      auto retire_previous = [&](uint32_t w_last, uint32_t s_last) {
        wgmma_wait<1>();
        release_pending();
        pend_w = w_last; pend_s = s_last;
      };
      auto next_w_stage = [&]() {
        if (++w_idx == (uint32_t)p.w_stages) { w_idx = 0; w_par ^= 1; b_lo = b_lo0; } else { b_lo += w_stage16; }
      };
      if (MODE == EPI_DOWN_SPACE) {
        for (int kc = 0; kc < p.kchunks; ++kc) {
          mbar_wait(slab_full + 8 * s_idx, s_par);
          const uint32_t a_base = desc_lo(slab0 + s_idx * p.slab_stride) + a_wg;
          const int t0 = kc < p.dn_lower ? 1 : 0, tstep = kc < p.dn_lower ? 2 : 1;
          for (int tap = t0; tap < 6; tap += tstep) {
            mbar_wait(w_full + 8 * w_idx, w_par);
            wgmma_fence();
            const uint64_t bd = b_hi | (uint64_t)b_lo;
#pragma unroll
            for (int j = 0; j < MW; ++j) {
              const uint64_t ad = a_hi | (uint64_t)(a_base + (uint32_t)p.dn_aoff[tap] + j * a_mtile);
              wgmma_mma<T, BN>(acc[j], ad, bd, accum);
              wgmma_mma<T, BN>(acc[j], ad + 2, bd + 2, 1u);
              wgmma_mma<T, BN>(acc[j], ad + 4, bd + 4, 1u);
              wgmma_mma<T, BN>(acc[j], ad + 6, bd + 6, 1u);
            }
            wgmma_commit();
            retire_previous(w_idx, tap + tstep >= 6 ? s_idx : NONE);
            accum = 1;
            next_w_stage();
          }
          if (++s_idx == (uint32_t)p.slab_stages) { s_idx = 0; s_par ^= 1; }
        }
      } else {
        const int dt0 = max(0, p.pt - c.t * p.st - p.hist_T);
        for (int dt = dt0; dt < p.kt; ++dt)
          for (int kc = 0; kc < p.kchunks; ++kc) {
            mbar_wait(slab_full + 8 * s_idx, s_par);
            uint32_t a_lo = desc_lo(slab0 + s_idx * p.slab_stride) + a_wg;   // descriptor low word of tap (0, 0)
            int dw = 0;
            for (int tp0 = 0; tp0 < taps2d; tp0 += p.tpw) {
              mbar_wait(w_full + 8 * w_idx, w_par);
              const bool slab_last = tp0 + p.tpw >= taps2d;
              uint32_t b_cur = b_lo;
              for (int u = 0; u < p.tpw; ++u) {
                wgmma_fence();
                const uint64_t bd = b_hi | (uint64_t)b_cur;
#pragma unroll
                for (int j = 0; j < MW; ++j) {
                  const uint64_t ad = a_hi | (uint64_t)(a_lo + j * a_mtile);
                  wgmma_mma<T, BN>(acc[j], ad, bd, accum);
                  wgmma_mma<T, BN>(acc[j], ad + 2, bd + 2, 1u);
                  if (K4) {
                    wgmma_mma<T, BN>(acc[j], ad + 4, bd + 4, 1u);
                    wgmma_mma<T, BN>(acc[j], ad + 6, bd + 6, 1u);
                  }
                }
                wgmma_commit();
                const bool w_last = u == p.tpw - 1;
                retire_previous(w_last ? w_idx : NONE, w_last && slab_last ? s_idx : NONE);
                accum = 1;
                b_cur += w_tile16;
                if (++dw == p.kw) { dw = 0; a_lo += a_next_dh; } else { a_lo += a_row; }
              }
              next_w_stage();
            }
            if (++s_idx == (uint32_t)p.slab_stages) { s_idx = 0; s_par ^= 1; }
          }
      }
      wgmma_wait<0>();
      release_pending();
    };
    // 64-byte rows (k4 false) occur only in the plain slab flavours; the fused ResidualUnit and SpatialDownsample2x
    // always read 128-byte rows
    auto mainloop_k = [&](const TileCoord& c, auto mw_c) {
      if (MODE != EPI_FUSED_RU && MODE != EPI_DOWN_SPACE && !k4) mainloop(c, mw_c, std::false_type());
      else mainloop(c, mw_c, std::true_type());
    };
    for (int tk = 0, tile; (tile = slab_tile_of(p, tk)) >= 0; ++tk) {
      const TileCoord c = decode_tile(p, tile);
      if (MWMAX >= 4 && p.mw == 4) mainloop_k(c, std::integral_constant<int, (MWMAX >= 4 ? 4 : 1)>());
      else if (MWMAX >= 2 && p.mw == 2) mainloop_k(c, std::integral_constant<int, (MWMAX >= 2 ? 2 : 1)>());
      else mainloop_k(c, std::integral_constant<int, 1>());
      if (slab_tma_epi(MODE)) {
        // ---- register epilogue: results -> this warpgroup's output tile -> TMA box stores ----
        constexpr int CB = slab_out_box_ch(MODE, BN, sizeof(T)), NB = (MODE == EPI_GEGLU ? BN / 2 : BN) / CB;
        constexpr uint32_t BOX = 64 * CB * (uint32_t)sizeof(T);
        const uint32_t ot = L.otile + (uint32_t)(wg * p.mw * NB) * BOX, rt = L.rtile + (uint32_t)(wg * p.mw) * 64 * BN * (uint32_t)sizeof(T);
        if (tid == 0) bulk_wait_read_all();     // the previous tile's stores have read the output tile
        named_bar_sync(wg_bar, 128);
        if (MODE == EPI_PLAIN_RES) mbar_wait(L.rbar + 8 * wg, r_par);
        const int act = p.epi.act;
        if (MODE == EPI_GEGLU || act == MV2_ACT_NONE)
          slab_epi_fragment<T, MODE, BN, MV2_ACT_NONE>(p, acc, c, sbias, ot, rt, wq, lane, false);
        else if (act == MV2_ACT_ELU) slab_epi_fragment<T, MODE, BN, MV2_ACT_ELU>(p, acc, c, sbias, ot, rt, wq, lane, false);
        else if (act == MV2_ACT_SILU) slab_epi_fragment<T, MODE, BN, MV2_ACT_SILU>(p, acc, c, sbias, ot, rt, wq, lane, false);
        else slab_epi_fragment<T, MODE, BN, MV2_ACT_LEAKY_RELU>(p, acc, c, sbias, ot, rt, wq, lane, act == MV2_ACT_RELU);
        if (MODE == EPI_PLAIN_RES) {
          __syncwarp();
          if (lane == 0) mbar_arrive(L.rbar + 16 + 8 * wg);
          r_par ^= 1;
        }
        fence_proxy_async();                    // generic-proxy writes -> visible to the TMA engine's reads
        named_bar_sync(wg_bar, 128);
        if (tid == 0) {
          // boxes without an output position or channel are skipped; TMA clips the others at the H, W and Co edges
          const int oc0 = MODE == EPI_GEGLU ? c.n0 / 2 : c.n0, oco = MODE == EPI_GEGLU ? p.Co / 2 : p.Co;
          const int h = c.h0 + 8 * wg;
          for (int j = 0; j < p.mw; ++j)
            for (int b = 0; b < NB; ++b)
              if (h < p.H && c.w0 + 8 * j < p.W && oc0 + b * CB < oco)
                tma_store_5d(&p.ymap, ot + (uint32_t)(j * NB + b) * BOX, oc0 + b * CB, c.w0 + 8 * j, h, c.t, c.b);
          bulk_commit();
        }
        continue;
      }
      if constexpr (MODE == EPI_FUSED_RU) {
        // ---------------- fused ResidualUnit epilogue (reference M:937-941 + the pooling half of M:229-233), per M-tile j
        //      on the accumulator fragments: E1 writes h = bf16(ELU(conv3 + b3)) into the H buffer, the A operand of the
        //      1x1x1 GEMM; E2 writes y = bf16(ELU(conv1 + b1)) into this warpgroup's output tile, TMA stores it and the
        //      SE pooling reads it back.  H and the output tiles are laid out as slab_epi_mtile writes them (bn = C = 64 |
        //      128: 128-byte rows, one 8 KB box per 64 channels); each warpgroup has its own 64 rows of both ----------------
        static_assert(sizeof(T) == 2, "the fused ResidualUnit has 16-bit instances only");
        constexpr int CB = slab_out_box_ch(MODE, BN, 2), NB = BN / CB;
        constexpr uint32_t BOX = 64 * CB * 2;
        const float* sb1 = sbias + nbias;
        const float* swk = sbias + 2 * nbias;
        float* lpart = reinterpret_cast<float*>(gen(L.lpart));
        const uint32_t hb = L.hbuf + (uint32_t)wg * KC1 * BOX, ot = L.otile + (uint32_t)(wg * p.mw * NB) * BOX;
        const int h = c.h0 + lh;
        const int rl = lane >> 2, piece = lane & 3;
        // rows of the warpgroup's 64 this thread reads back: its own (the logit), and 8 k + rl of its warp's 32 (pooling)
        const uint32_t mrow = (uint32_t)(row & 63), mq = mrow & ~31u;
        // one record per (tile, lane quarter): the M-tiles of the tile are folded in registers (online softmax over j)
        const int recs_per_frame = p.tiles_h * p.tiles_w * 4;
        float* rec = p.se_ws + ((int64_t)(c.b * p.T + c.t) * recs_per_frame + ((c.h0 >> 4) * p.tiles_w + c.w0 / (8 * p.mw)) * 4 + sub) * (p.Co + 2);
        float run_m = -INFINITY, run_s = 0.f, run_acc[2][8];
#pragma unroll
        for (int q = 0; q < 2; ++q)
#pragma unroll
          for (int i = 0; i < 8; ++i) run_acc[q][i] = 0.f;
        const uint64_t h_hi = gmma_desc_hi(1024, 128);
        const uint32_t h_lo = desc_lo(hb);
        // the 1x1x1 weights: the tile's last KC1 weight-ring stages (the producer appends them after the conv's stages);
        // they stay held until the last M-tile's second GEMM has read them
        uint32_t w1_slot[KC1], w1_par[KC1], w1_lo[KC1];
#pragma unroll
        for (int kc2 = 0; kc2 < KC1; ++kc2) {
          w1_slot[kc2] = w_idx; w1_par[kc2] = w_par; w1_lo[kc2] = b_lo;
          if (++w_idx == (uint32_t)p.w_stages) { w_idx = 0; w_par ^= 1; b_lo = b_lo0; } else { b_lo += w_stage16; }
        }
        // the previous tile's y stores have read the output tile (E2 writes it after the barrier that follows E1)
        if (tid == 0) bulk_wait_read_all();
#pragma unroll
        for (int j = 0; j < MWMAX; ++j) {
          if (j >= p.mw) break;
          // E1 (H is free: the previous second GEMM completed before the barrier that follows its E2)
          slab_epi_mtile<T, MODE, BN, MV2_ACT_ELU>(p, acc[j], c, sbias, hb, 0, wq, lane, false);
          fence_proxy_async();      // generic-proxy writes -> visible to the tensor core's async-proxy reads
          named_bar_sync(wg_bar, 128);
          // second GEMM: acc[0] = H (this warpgroup's 64 rows) x W1^T
#pragma unroll
          for (int kc2 = 0; kc2 < KC1; ++kc2) mbar_wait(w_full + 8 * w1_slot[kc2], w1_par[kc2]);
          wgmma_fence();
#pragma unroll
          for (int kc2 = 0; kc2 < KC1; ++kc2) {
            const uint64_t ad = h_hi | (uint64_t)(h_lo + kc2 * (BOX >> 4)), bd = h_hi | (uint64_t)w1_lo[kc2];
            wgmma_mma<T, BN>(acc[0], ad, bd, kc2 > 0 ? 1u : 0u);
            wgmma_mma<T, BN>(acc[0], ad + 2, bd + 2, 1u);
            wgmma_mma<T, BN>(acc[0], ad + 4, bd + 4, 1u);
            wgmma_mma<T, BN>(acc[0], ad + 6, bd + 6, 1u);
          }
          wgmma_commit();
          wgmma_wait<0>();
          if (j == p.mw - 1) {
            __syncwarp();
            if (lane == 0)
#pragma unroll
              for (int kc2 = 0; kc2 < KC1; ++kc2) mbar_arrive(w_empty + 8 * w1_slot[kc2]);
          }
          // E2 -> output tile of M-tile j -> TMA box stores (boxes without an output position are skipped; TMA clips
          // the others at the H and W edges)
          const uint32_t otj = ot + (uint32_t)(j * NB) * BOX;
          slab_epi_mtile<T, MODE, BN, MV2_ACT_ELU>(p, acc[0], c, sb1, otj, 0, wq, lane, false);
          fence_proxy_async();
          named_bar_sync(wg_bar, 128);
          if (tid == 0) {
            if (c.h0 + 8 * wg < p.H && c.w0 + 8 * j < p.W)
#pragma unroll
              for (int b = 0; b < NB; ++b) tma_store_5d(&p.ymap, otj + (uint32_t)b * BOX, b * CB, c.w0 + 8 * j, c.h0 + 8 * wg, c.t, c.b);
            bulk_commit();
          }
          // SE logit of this thread's row on the rounded y, like the unfused path reads it: channels half * 32 + 64 q + 0..31
          // in order, one fma chain
          auto ld_y = [&](int q, uint32_t m, uint32_t u) {   // 16-byte unit u (channels 8 u ..) of row m, box q
            uint4 v;
            asm volatile("ld.shared.v4.b32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w)
                         : "r"(otj + (uint32_t)q * BOX + m * 128 + ((u ^ (m & 7)) << 4)) : "memory");
            return v;
          };
          const int w = c.w0 + 8 * j + lw;
          const bool row_ok = h < p.H && w < p.W;
          float lp = 0.f;
#pragma unroll
          for (int q = 0; q < NB; ++q)
#pragma unroll
            for (int g = 0; g < 4; ++g) {
              const uint4 v = ld_y(q, mrow, 4 * half + g);
              const float4 wa = *reinterpret_cast<const float4*>(swk + half * 32 + 64 * q + 8 * g);
              const float4 wb = *reinterpret_cast<const float4*>(swk + half * 32 + 64 * q + 8 * g + 4);
              const float2 f0 = unpack2<T>(v.x), f1 = unpack2<T>(v.y), f2 = unpack2<T>(v.z), f3 = unpack2<T>(v.w);
              lp = fmaf(f0.x, wa.x, lp);
              lp = fmaf(f0.y, wa.y, lp);
              lp = fmaf(f1.x, wa.z, lp);
              lp = fmaf(f1.y, wa.w, lp);
              lp = fmaf(f2.x, wb.x, lp);
              lp = fmaf(f2.y, wb.y, lp);
              lp = fmaf(f3.x, wb.z, lp);
              lp = fmaf(f3.y, wb.w, lp);
            }
          // the two warps of this lane quarter hold the two halves of every row's channels: exchange the logit partials
          float* lpb = lpart + (ecount & 1u) * 256;
          ++ecount;
          lpb[ew * 32 + lane] = lp;
          asm volatile("bar.sync %0, 64;" ::"r"(1 + sub) : "memory");
          float lg = lpb[sub * 32 + lane] + lpb[(sub + 4) * 32 + lane] + p.se_bk;
          lg = row_ok ? lg : -INFINITY;
          const float mx = warp_max(lg);
          const float ev = lg > -INFINITY ? ex2_approx((lg - mx) * 1.4426950408889634f) : 0.f;
          const float es = warp_sum(ev);
          float e4[4];
#pragma unroll
          for (int k = 0; k < 4; ++k) e4[k] = __shfl_sync(0xffffffffu, ev, 8 * k + rl);
          const float new_m = fmaxf(run_m, mx);
          const float ca = run_m > -INFINITY ? ex2_approx((run_m - new_m) * 1.4426950408889634f) : 0.f;   // rescales what is held
          const float cb = mx > -INFINITY ? ex2_approx((mx - new_m) * 1.4426950408889634f) : 0.f;         // weights this M-tile
          run_s = fmaf(run_s, ca, es * cb);
          run_m = new_m;
          // pool sums: this lane's 8 channels (16-byte piece) of rows 8 k + rl (output rows h0 + 4 sub + k, w = w0 + 8 j + rl)
#pragma unroll
          for (int q = 0; q < NB; ++q) {
            float t[8];
#pragma unroll
            for (int i = 0; i < 8; ++i) t[i] = 0.f;
#pragma unroll
            for (int k = 0; k < 4; ++k) {
              const uint4 v = ld_y(q, mq + 8 * k + rl, 4 * half + piece);
              const uint32_t vv[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
              for (int i = 0; i < 4; ++i) {
                const float2 f = unpack2<T>(vv[i]);
                t[2 * i] = fmaf(e4[k], f.x, t[2 * i]);
                t[2 * i + 1] = fmaf(e4[k], f.y, t[2 * i + 1]);
              }
            }
#pragma unroll
            for (int i = 0; i < 8; ++i) {
              t[i] += __shfl_xor_sync(0xffffffffu, t[i], 4);
              t[i] += __shfl_xor_sync(0xffffffffu, t[i], 8);
              t[i] += __shfl_xor_sync(0xffffffffu, t[i], 16);
            }
#pragma unroll
            for (int i = 0; i < 8; ++i) run_acc[q][i] = fmaf(run_acc[q][i], ca, t[i] * cb);
          }
        }
        if (half == 0 && lane == 0) { rec[0] = run_m; rec[1] = run_s; }
        if (rl == 0) {
#pragma unroll
          for (int q = 0; q < NB; ++q) {
            float2* dst = reinterpret_cast<float2*>(rec + 2 + half * 32 + 64 * q + piece * 8);
            dst[0] = make_float2(run_acc[q][0], run_acc[q][1]); dst[1] = make_float2(run_acc[q][2], run_acc[q][3]);
            dst[2] = make_float2(run_acc[q][4], run_acc[q][5]); dst[3] = make_float2(run_acc[q][6], run_acc[q][7]);
          }
        }
        continue;
      }
      // ---- accumulators -> shared-memory staging (one [64][BN + 4] block per M-tile), once the previous tile's epilogue
      //      of this warpgroup has read its staging ----
      named_bar_sync(wg_bar, 128);
#pragma unroll
      for (int j = 0; j < MWMAX; ++j) {
        if (j >= p.mw) break;
        stage_acc<BN>(acc[j], stg + j * 64 * (BN + 4), tid);
      }
      named_bar_sync(wg_bar, 128);
      const int h = c.h0 + lh;
      for (int j = 0; j < p.mw; ++j) {
        const int w = c.w0 + 8 * j + lw;
        const bool row_ok = h < p.H && w < p.W;
        const float* srow = stg + (j * 64 + row - 64 * wg) * (BN + 4);
        const int64_t row_base = ((((int64_t)c.b * p.T + c.t) * p.H + h) * p.W + w) * p.Co;
        // column chunks are dealt round-robin to the two warps that share this lane quarter
        if constexpr (MODE == EPI_SHUFFLE_ST) {
          static_assert(sizeof(T) == 2, "the transposed shuffle stores have 16-bit instances only");
          // Row-per-lane results are transposed through shared memory so that every store instruction writes 8 rows
          // x 64 contiguous bytes (full sectors; the 8 rows are neighbours along w) instead of 32 scattered 16-byte pieces.
          const uint32_t stg = stage0 + (uint32_t)ew * 2048;
          const uint32_t wr = stg + lane * 64, wsw = (lane >> 1) & 3;
          const int rl = lane >> 2, piece = lane & 3;                 // read side: row within an 8-row group, 16-byte piece
          const int w2 = c.w0 + 8 * j + rl;
          const uint32_t rd = stg + rl * 64;
          const int h20 = c.h0 + sub * 4;
          const int kmax = w2 < p.W ? p.H - h20 : 0;                   // rows k < kmax are inside the frame
          for (int c0 = ((j + half) & 1) * 32; c0 < p.bn; c0 += 64) {
            uint32_t r[32], pk[16];
            load_row32(srow + c0, 32, r);
            epi_pack32<T>(p.epi.act, r, sbias + c.n0 + c0, pk);
#pragma unroll
            for (int g = 0; g < 4; ++g)
              asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(wr + ((g ^ wsw) << 4)), "r"(pk[4 * g]),
                           "r"(pk[4 * g + 1]), "r"(pk[4 * g + 2]), "r"(pk[4 * g + 3]) : "memory");
            __syncwarp();
            const bool col_ok = c.n0 + c0 + piece * 8 < p.Co && c0 + piece * 8 < p.bn;
            const int klim = col_ok ? kmax : 0;
            // packed GEMM columns are (q, c): this chunk's 32 columns share one sub-pixel phase q (Cy % 32 == 0), so a
            // row's 64 bytes land contiguously at its shuffled position (reference M:824 / M:861 rearranges)
            T* yp;
            int64_t ks;
            const int n = c.n0 + c0;
            if (p.epi.shuffle == MV2_SHUFFLE_SPACE) {
              const int cy = p.Co >> 2, qd = n / cy, cb = n - qd * cy;
              yp = (T*)p.epi.y + ((((int64_t)c.b * p.T + c.t) * (2 * p.H) + (2 * h20 + (qd >> 1))) * (2 * p.W) + (2 * w2 + (qd & 1))) * cy + cb + piece * 8;
              ks = (int64_t)4 * p.W * cy;          // next h row = two output rows further
            } else {
              const int cy = p.Co >> 1, qd = n / cy, cb = n - qd * cy;
              yp = (T*)p.epi.y + ((((int64_t)c.b * (2 * p.T) + (2 * c.t + qd)) * p.H + h20) * p.W + w2) * cy + cb + piece * 8;
              ks = (int64_t)p.W * cy;
            }
#pragma unroll
            for (int k = 0; k < 4; ++k) {
              uint4 v;
              asm volatile("ld.shared.v4.b32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w)
                           : "r"(rd + k * 512 + ((piece ^ (((8 * k + rl) >> 1) & 3)) << 4)));
              if (k < klim) *reinterpret_cast<uint4*>(yp + k * ks) = v;
            }
            __syncwarp();
          }
        } else {
          for (int c0 = ((j + half) & 1) * 32; c0 < p.bn; c0 += 64) {
            uint32_t r[32];
            load_row32(srow + c0, BN < 32 ? BN : 32, r);     // a narrow tile's staged rows hold BN + 4 floats
            if (row_ok) epi_chunk32<T, MODE>(p.epi, r, min(32, p.bn - c0), c.n0 + c0, sbias + c.n0 + c0, c.b, c.t, h, w, row_base);
          }
        }
      }
    }
    if (TMA_STORE && tid == 0) bulk_wait_all();   // the output is written before the CTA exits
  }
}

// One kernel per element type (the names of the bf16 instances are those of the library before fp16 existed)
template <int MODE, int BN>
__global__ void __launch_bounds__(384, 1) tc_slab_kernel(const __grid_constant__ SlabParams p) { tc_slab_body<__nv_bfloat16, MODE, BN>(p); }
template <int MODE, int BN>
__global__ void __launch_bounds__(384, 1) tc_slab_f16_kernel(const __grid_constant__ SlabParams p) { tc_slab_body<__half, MODE, BN>(p); }
template <int MODE, int BN>
__global__ void __launch_bounds__(384, 1) tc_slab_tf32_kernel(const __grid_constant__ SlabParams p) { tc_slab_body<float, MODE, BN>(p); }

}  // namespace mv2

using namespace mv2;

// Channels-first outputs of at most 16 channels whose in-plane taps are wider than 3 -- the data gradient of a 7 x 7 x 7
// conv_in (or its 1 x 7 x 7 first-frame conv) with respect to the video -- run on the narrow N tiles (8 / 16 columns):
// a 32-column tile would spend 29 of every 32 MMA columns and weight rows on padding.
static bool slab_narrow(const mv2_tc_conv_args* a) { return a->out_layout == 1 && a->Co <= 16 && a->kw > 3; }

extern "C" int mv2_tc_slab_supported(const mv2_tc_conv_args* a) {
  if (!a || tc_dtype(a) < 0) return 0;
  const int ci_bytes = a->Ci * tc_esize(tc_dtype(a));      // bytes of one position's input channels
  if (a->sh != 1 || a->sw != 1) return 0;
  if (a->st != 1) {      // TimeDownsample2x (M:796-807): stride 2 along t only, plain epilogue
    if (a->st != 2 || a->out_layout != 0 || a->epi_mode != 0 || a->shuffle != MV2_SHUFFLE_NONE) return 0;
    if (a->To != (a->Ti + a->pt - a->kt) / a->st + 1 || a->To < 1) return 0;
  }
  if (ci_bytes % 64 != 0 || a->Co > 4096) return 0;
  if (a->oscale && (a->epi_mode != 0 || a->shuffle != MV2_SHUFFLE_NONE)) return 0;   // demodulation: plain / ragged epilogues only
  if (a->epi_mode == 1 && (a->Co % 64 != 0 || a->shuffle != MV2_SHUFFLE_NONE || a->res)) return 0;   // fused GEGLU (64-column epilogue chunks)
  if (a->epi_mode == 2 && (!a->res || a->shuffle != MV2_SHUFFLE_NONE)) return 0;   // scaled residual
  if (a->epi_mode < 0 || a->epi_mode > 2) return 0;
  if (a->Co % 32 != 0 && a->Co > 32) return 0;           // ragged N only as a single (zero padded) 32-column tile
  if (ci_bytes % 128 != 0 && a->kw != 1) return 0;       // 64-byte rows: only h-shifted taps (1024 B multiples)
  if (a->res && a->Co % 8 != 0) return 0;
  if (a->shuffle != MV2_SHUFFLE_NONE && ((a->shuffle == MV2_SHUFFLE_SPACE ? a->Co / 4 : a->Co / 2) % 8 != 0 || a->Co % 32 != 0)) return 0;
  if (a->kh > 7 || a->kw > (slab_narrow(a) ? 7 : 3) || a->kt > 8) return 0;
  if (a->Ho != a->Hi || a->Wo != a->Wi) return 0;
  if (a->out_layout == 1) {   // channels-first output: the ragged scalar-store epilogue only; may drop leading frames
    if (a->Co % 8 == 0 || a->res || a->shuffle != MV2_SHUFFLE_NONE || a->epi_mode != 0) return 0;
    if (a->To > a->Ti || a->To < 1) return 0;
    // conv_out (causal, the first Ti - To output frames not computed) or the data gradient of a causal conv (the transposed
    // conv: no leading pad, output frame t reads input frames t + Ti - To ..; the first Ti - To frames not computed)
    if (a->pt != a->kt - 1 - (a->Ti - a->To) && a->pt != -(a->Ti - a->To)) return 0;
  } else if (a->out_layout != 0 || (a->st == 1 && a->To != a->Ti)) return 0;
  return 1;
}

// Shared memory left for the two TMA rings of a launch: 227 KB minus what follows them (barrier table sized for the deepest
// rings, bias, transpose buffers, accumulator staging or, fused, logit partials, H buffer and output tiles) and the
// alignment slack.
static int slab_ring_budget(const SlabParams& p, bool fused) {
  SlabParams q = p;
  q.slab_stages = 3; q.w_stages = 12;      // upper bounds for the barrier table
  return 227 * 1024 - 2048 - (int)slab_smem_layout(q, 0, fused, tc_esize(p.dtype)).end;
}
// Dynamic shared memory of a launch: alignment slack, the slab and weight rings, then slab_smem_layout
static size_t slab_smem_bytes(const SlabParams& p, bool fused) {
  const uint32_t rings = (uint32_t)(p.slab_stages * p.slab_stride + p.w_stages * p.bn * p.row_bytes * p.tpw);
  return 1024 + slab_smem_layout(p, rings, fused, tc_esize(p.dtype)).end;
}
// M-tiles side by side per weight tile: as many as the frame width uses, while their accumulators fit 64 fp32 registers
// per consumer thread (mw * bn <= 128); this divides the weight traffic by mw
static int slab_default_mw(int bn, int Wo) { return bn <= 32 && Wo > 16 ? 4 : (bn <= 64 && Wo > 8 ? 2 : 1); }
// Slab geometry of a macro tile of mw M-tiles: slab row pitch, bytes of one slab (slab_h rows) and its 1024-byte aligned
// ring stride, tile counts.  Needs kw, slab_h, row_bytes, B, T, W, tiles_h and n_tiles_n.
static void slab_set_geometry(SlabParams& p, int mw) {
  p.mw = mw;
  p.pitch = 8 * mw + p.kw - 1;
  p.slab_bytes = p.pitch * p.slab_h * p.row_bytes;
  p.slab_stride = (p.slab_bytes + 1023) / 1024 * 1024;
  p.tiles_w = ceil_div(p.W, 8 * mw);
  p.total_tiles = (int)((int64_t)p.B * p.T * p.tiles_h * p.tiles_w * p.n_tiles_n);
}

// Everything the launch derives from the layer shape alone (tiling, ring depths, tile count): pure host arithmetic, no
// CUDA calls -- also reachable through mv2_tc_slab_plan / mv2_tc_slab_tile for the CPU-side tests.
static int slab_fill_plan(const mv2_tc_conv_args* a, SlabParams& p) {
  memset(&p, 0, sizeof(p));
  p.kt = a->kt; p.kh = a->kh; p.kw = a->kw; p.pt = a->pt; p.ph = a->ph; p.pw = a->pw;
  p.st = a->st;
  p.dtype = tc_dtype(a);
  const int ci_bytes = a->Ci * tc_esize(p.dtype);
  p.row_bytes = ci_bytes % 128 == 0 ? 128 : 64;
  p.Ci = a->Ci; p.kchunks = ci_bytes / p.row_bytes;
  p.B = a->B; p.T = a->To; p.H = a->Ho; p.W = a->Wo; p.Co = a->Co;
  p.epi = tc_epi_of(a);

  // ---- tiling: widest N tile (<= 128 columns), then as many M-tiles per weight tile as slab_default_mw allows ----
  const int co_pad = (a->Co + 31) / 32 * 32;
  int best_bn = 32;
  for (int bn = 128; bn >= 32; bn >>= 1)
    if (co_pad % bn == 0) { best_bn = bn; break; }
  // wide outputs whose width has no large power-of-two divisor (the GEGLU feed-forward: 2 * 1365 -> 2752 packed columns
  // would run 43 tiles of 64): take 128-column tiles and let the last one be ragged (the plain and GEGLU epilogues guard
  // every stored column against Co)
  const bool ragged_ok = a->epi_mode == 0 && a->shuffle == MV2_SHUFFLE_NONE && a->Co % 8 == 0;
  if ((ragged_ok || a->epi_mode == 1) && best_bn <= 64 && co_pad >= 512 && (co_pad + 127) / 128 * 128 * 100 <= co_pad * 108)
    best_bn = 128;
  p.bn = slab_narrow(a) ? (a->Co <= 8 ? 8 : 16) : best_bn;
  // a ragged last tile reads zero-filled weight rows and stores nothing for them; a narrow tile covers all of Co (<= bn)
  p.n_tiles_n = slab_narrow(a) ? 1 : (co_pad + p.bn - 1) / p.bn;
  p.tiles_h = ceil_div(a->Ho, 16);
  p.slab_h = 16 + a->kh - 1;
  int budget;
  for (int mw = slab_default_mw(p.bn, a->Wo);; mw >>= 1) {   // two slab stages and the staging of a wide macro tile do not fit: narrow it
    slab_set_geometry(p, mw);
    budget = slab_ring_budget(p, false);
    if (mw == 1 || 2 * p.slab_stride + 2 * p.bn * p.row_bytes <= budget) break;
  }
  // weight ring stage = tpw consecutive in-plane taps (fewer barrier round trips for small tiles), <= 32 KB
  const int taps2d = a->kh * a->kw;
  p.tpw = 1;
  for (int d = taps2d; d >= 1; --d)
    if (taps2d % d == 0 && d * p.bn * p.row_bytes <= 32 * 1024) { p.tpw = d; break; }
  int w_bytes = p.bn * p.row_bytes * p.tpw;
  p.slab_stages = p.slab_stride * 3 + w_bytes * 3 <= budget ? 3 : 2;
  p.w_stages = std::min(12, (budget - p.slab_stages * p.slab_stride) / w_bytes);
  if (p.w_stages < 2 && p.slab_stages > 2) { p.slab_stages = 2; p.w_stages = std::min(12, (budget - 2 * p.slab_stride) / w_bytes); }
  while (p.w_stages < 2 && p.tpw > 1) {   // wide slabs: fall back to fewer taps per weight stage
    int d = p.tpw - 1;
    while (d > 1 && taps2d % d != 0) --d;
    p.tpw = d;
    w_bytes = p.bn * p.row_bytes * p.tpw;
    p.w_stages = std::min(12, (budget - p.slab_stages * p.slab_stride) / w_bytes);
  }
  MV2_CHECK_ARG(p.w_stages >= 2);
  return MV2_OK;
}

// TMA maps of a stride-1 slab conv: the activation slab (box {bk, pitch, slab_h, 1, 1} of x as {Ci, Wi, Hi, Ti, B}) and the
// weights [Co][tap][Ci] as {ci, co, tap} (box {bk, bn, tpw}: tpw consecutive K-major tiles) and as {k, co} (box {bk, bn}).
static int slab_encode_maps(SlabParams& p, const mv2_tc_conv_args* a, const mv2_conv_hist* hist = nullptr) {
  const CUtensorMapSwizzle swz = swizzle_of_row(p.row_bytes);
  const int es = tc_esize(p.dtype);
  const int64_t C = a->Ci, W = a->Wi, H = a->Hi, T = a->Ti;
  const cuuint64_t xdims[5] = {(cuuint64_t)C, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)T, (cuuint64_t)a->B};
  const cuuint64_t xstrides[4] = {(cuuint64_t)(C * es), (cuuint64_t)(W * C * es), (cuuint64_t)(H * W * C * es), (cuuint64_t)(T * H * W * C * es)};
  const cuuint32_t xbox[5] = {(cuuint32_t)(p.row_bytes / es), (cuuint32_t)p.pitch, (cuuint32_t)p.slab_h, 1, 1};
  if (const int rc = encode_tc_map(&p.amap, p.dtype, 5, a->x, xdims, xstrides, xbox, swz, "slab")) return rc;
  p.hist_T = hist ? hist->T_h : 0;
  if (p.hist_T > 0) {     // the same boxes over the history: (T_h frames, clip stride of the tensor it lives in)
    const cuuint64_t hdims[5] = {(cuuint64_t)C, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)p.hist_T, (cuuint64_t)a->B};
    const cuuint64_t hstrides[4] = {xstrides[0], xstrides[1], xstrides[2], (cuuint64_t)(hist->clip_stride * es)};
    if (const int rc = encode_tc_map(&p.hmap, p.dtype, 5, hist->h, hdims, hstrides, xbox, swz, "history")) return rc;
  }
  const int64_t ntaps = (int64_t)a->kt * a->kh * a->kw, K = ntaps * C;
  const cuuint64_t wdims[3] = {(cuuint64_t)C, (cuuint64_t)a->Co, (cuuint64_t)ntaps}, kdims[2] = {(cuuint64_t)K, (cuuint64_t)a->Co};
  const cuuint64_t wstrides[2] = {(cuuint64_t)(K * es), (cuuint64_t)(C * es)};
  const cuuint32_t wbox[3] = {(cuuint32_t)(p.row_bytes / es), (cuuint32_t)p.bn, (cuuint32_t)p.tpw};
  if (const int rc = encode_tc_map(&p.wmap, p.dtype, 3, a->w, wdims, wstrides, wbox, swz, "weights")) return rc;
  return encode_tc_map(&p.wmap2, p.dtype, 2, a->w, kdims, wstrides, wbox, swz, "weights 2-D");
}
// Output (and residual) maps of the TMA-store flavours: y as {oc, W, H, T, B} (oc = Co, or Co / 2 for GEGLU), boxes of
// slab_out_box_ch channels x 8 (w) x 8 (h) in the swizzle of their row width
static int slab_encode_out_maps(SlabParams& p, int mode) {
  const int es = tc_esize(p.dtype);
  const int cb = slab_out_box_ch(mode, p.bn, es);
  const int64_t oc = mode == EPI_GEGLU ? p.Co / 2 : p.Co;
  const cuuint64_t dims[5] = {(cuuint64_t)oc, (cuuint64_t)p.W, (cuuint64_t)p.H, (cuuint64_t)p.T, (cuuint64_t)p.B};
  const cuuint64_t strides[4] = {(cuuint64_t)(oc * es), (cuuint64_t)(p.W * oc * es), (cuuint64_t)(p.H * p.W * oc * es),
                                 (cuuint64_t)(p.T * p.H * p.W * oc * es)};
  const cuuint32_t box[5] = {(cuuint32_t)cb, 8, 8, 1, 1};
  const CUtensorMapSwizzle swz = swizzle_of_row(cb * es);
  if (const int rc = encode_tc_map(&p.ymap, p.dtype, 5, p.epi.y, dims, strides, box, swz, "output")) return rc;
  if (mode != EPI_PLAIN_RES) return MV2_OK;
  return encode_tc_map(&p.rmap, p.dtype, 5, p.epi.res, dims, strides, box, swz, "residual");
}

// Launches one slab-kernel flavour: persistent CTAs, one per SM of the current device (fewer when there are fewer tiles)
static int slab_launch(int mode, const SlabParams& p, void* stream) {
  // kernel instance per (epilogue flavour, N tile); every instance may use up to 227 KB of dynamic shared memory.  The
  // channels-first flavour EPI_RAGGED (< 32 channels) has the 32-column tile and the narrow 16- and 8-column ones.
  // [0] bf16, [1] fp16, [2] TF32, which has no fused ResidualUnit and no transposed shuffle stores (null: never chosen).
#define MV2_SLAB_BN(K, M) {K<M, 32>, K<M, 64>, K<M, 128>}
#define MV2_SLAB_NONE {nullptr, nullptr, nullptr}
#define MV2_SLAB_FLAVOURS(K, FUSED_RU, SHUFFLE_ST)                                                                       \
  {MV2_SLAB_BN(K, EPI_PLAIN), MV2_SLAB_BN(K, EPI_GEGLU), MV2_SLAB_BN(K, EPI_SHUFFLE),                                 \
   {K<EPI_RAGGED, 32>, K<EPI_RAGGED, 16>, K<EPI_RAGGED, 8>},                                                           \
   MV2_SLAB_BN(K, EPI_PLAIN_RES), FUSED_RU, SHUFFLE_ST, MV2_SLAB_BN(K, EPI_DOWN_SPACE)}
  static void (*const kernels[3][8][3])(SlabParams) = {
      MV2_SLAB_FLAVOURS(tc_slab_kernel, MV2_SLAB_BN(tc_slab_kernel, EPI_FUSED_RU), MV2_SLAB_BN(tc_slab_kernel, EPI_SHUFFLE_ST)),
      MV2_SLAB_FLAVOURS(tc_slab_f16_kernel, MV2_SLAB_BN(tc_slab_f16_kernel, EPI_FUSED_RU),
                        MV2_SLAB_BN(tc_slab_f16_kernel, EPI_SHUFFLE_ST)),
      MV2_SLAB_FLAVOURS(tc_slab_tf32_kernel, MV2_SLAB_NONE, MV2_SLAB_NONE)};
#undef MV2_SLAB_FLAVOURS
#undef MV2_SLAB_NONE
#undef MV2_SLAB_BN
  static PerDeviceOnce attr_once;
  const cudaError_t attr_err = attr_once.run([] {
    cudaError_t e = cudaSuccess;
    for (auto& type : kernels)
      for (auto& row : type)
        for (auto k : row)
          if (e == cudaSuccess && k) e = cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024);
    return e;
  });
  if (attr_err != cudaSuccess) { set_error("cudaFuncSetAttribute failed: %s", cudaGetErrorString(attr_err)); return MV2_E_CUDA; }
  const size_t smem = slab_smem_bytes(p, mode == EPI_FUSED_RU);
  MV2_CHECK_ARG(smem <= 227 * 1024);
  int dev = 0, n_sm = 132;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&n_sm, cudaDevAttrMultiProcessorCount, dev);
  MV2_CHECK_ARG(p.bn >= 32 || mode == EPI_RAGGED);
  const int slot = p.bn == 32 ? 0 : (p.bn == 64 || p.bn == 16 ? 1 : 2);
  const auto kernel = kernels[p.dtype == MV2_F16 ? 1 : (p.dtype == MV2_TF32 ? 2 : 0)][mode][slot];
  MV2_CHECK_ARG(kernel != nullptr);
  launch_k(kernel, dim3(std::min(p.total_tiles, n_sm)), dim3(384), smem, (cudaStream_t)stream, p);
  MV2_CHECK_LAUNCH();
  return MV2_OK;
}

extern "C" int mv2_tc_slab_plan(const mv2_tc_conv_args* a, int n_sm, int* out6) {
  MV2_CHECK_ARG(a && out6 && n_sm > 0);
  if (!mv2_tc_slab_supported(a)) { set_error("mv2_tc_slab_plan: unsupported shape"); return MV2_E_UNSUPPORTED; }
  SlabParams p;
  if (const int rc = slab_fill_plan(a, p)) return rc;
  const int grid = std::min(p.total_tiles, n_sm);
  out6[0] = p.mw; out6[1] = p.bn; out6[2] = p.n_tiles_n; out6[3] = p.total_tiles; out6[4] = grid; out6[5] = p.slab_stages;
  return MV2_OK;
}

extern "C" int mv2_tc_slab_tile(const mv2_tc_conv_args* a, int n_sm, int cta, int k, int* out6) {
  MV2_CHECK_ARG(a && out6 && n_sm > 0 && cta >= 0 && k >= 0);
  if (!mv2_tc_slab_supported(a)) { set_error("mv2_tc_slab_tile: unsupported shape"); return MV2_E_UNSUPPORTED; }
  SlabParams p;
  if (const int rc = slab_fill_plan(a, p)) return rc;
  const int grid = std::min(p.total_tiles, n_sm);
  MV2_CHECK_ARG(cta < grid);
  const int tile = slab_tile_of_cta(p, k, cta, grid);
  out6[0] = tile;                                // -1: this CTA has no k-th tile
  if (tile >= 0) {
    const TileCoord c = decode_tile(p, tile);
    out6[1] = c.b; out6[2] = c.t; out6[3] = c.h0; out6[4] = c.w0; out6[5] = c.n0;
  }
  return MV2_OK;
}

extern "C" int mv2_tc_slab_forward(const mv2_tc_conv_args* a, const mv2_conv_hist* hist, void* stream) {
  MV2_CHECK_ARG(a && a->x && a->w && a->y);
  MV2_CHECK_ARG(!hist || (hist->T_h >= 0 && (hist->T_h == 0 || (hist->h && hist->clip_stride > 0))));
  if (!mv2_tc_slab_supported(a)) { set_error("mv2_tc_slab_forward: unsupported shape"); return MV2_E_UNSUPPORTED; }
  SlabParams p;
  if (const int rc = slab_fill_plan(a, p)) return rc;
  if (const int rc = slab_encode_maps(p, a, hist)) return rc;
  int mode = EPI_PLAIN;
  if (a->epi_mode == 1) mode = EPI_GEGLU;
  else if (a->shuffle != MV2_SHUFFLE_NONE && (a->Co / (a->shuffle == MV2_SHUFFLE_SPACE ? 4 : 2)) % 32 == 0 && p.dtype != MV2_TF32)
    mode = EPI_SHUFFLE_ST;     // TF32: a 32-column chunk of fp32 is 128 bytes per row, twice a transpose buffer's rows
  else if (a->shuffle != MV2_SHUFFLE_NONE) mode = EPI_SHUFFLE;
  else if (a->Co % 8 != 0) mode = EPI_RAGGED;
  else if (a->res) mode = EPI_PLAIN_RES;
  if (slab_tma_epi(mode))
    if (const int rc = slab_encode_out_maps(p, mode)) return rc;
  return slab_launch(mode, p, stream);
}


// =====================================================================================================================
// Fused ResidualUnit front half: y = ELU(conv1x1x1(ELU(causal_conv3x3x3(x)))) + SqueezeExcite pool partials, one launch.
// =====================================================================================================================
static void ru_as_conv_args(const mv2_tc_ru_args* a, mv2_tc_conv_args* c) {
  memset(c, 0, sizeof(*c));
  c->x = a->x; c->w = a->w3; c->bias = a->b3; c->res = nullptr; c->y = a->y;
  c->B = a->B; c->Ti = c->To = a->T; c->Hi = c->Ho = a->H; c->Wi = c->Wo = a->W; c->Ci = c->Co = a->C;
  c->kt = a->kt; c->kh = a->kh; c->kw = a->kw; c->st = c->sh = c->sw = 1;
  c->pt = a->kt - 1; c->ph = a->kh / 2; c->pw = a->kw / 2;
  c->act = MV2_ACT_ELU; c->shuffle = MV2_SHUFFLE_NONE; c->epi_mode = 0;
  c->dtype = a->dtype;
}

extern "C" int mv2_tc_ru_supported(const mv2_tc_ru_args* a) {
  if (!a) return 0;
  if (tc_dtype_of(a->dtype) == MV2_TF32) return 0;     // 16-bit only: TF32 units take the unfused convs (DESIGN.md)
  if (a->C != 64 && a->C != 128) return 0;            // all of Co in one N tile (bn = C)
  if (a->W <= 8) return 0;                            // narrow frames take the unfused path
  if (a->kt < 1 || a->kt > 8 || a->kh < 1 || a->kh > 7 || a->kw < 1 || a->kw > 3) return 0;
  if ((a->kh & 1) == 0 || (a->kw & 1) == 0) return 0;
  mv2_tc_conv_args c;
  ru_as_conv_args(a, &c);
  return mv2_tc_slab_supported(&c);
}

// tiling + shared-memory plan of the fused kernel (host arithmetic only): the slab plan of the 3x3x3 conv (one N tile of
// bn = C; its M-tile rule gives mw = 2 at C = 64 and 1 at C = 128), one tap per weight stage, three slab stages when they
// leave room for two weight stages next to the H buffer and the output tiles, and as many weight stages as then fit (the
// 1x1x1 weights stream through the same ring, C / 64 stages per tile): 3 + 6 at C = 64, 3 + 5 at C = 128 (3x3x3)
static int ru_fill_plan(const mv2_tc_ru_args* a, SlabParams& p) {
  mv2_tc_conv_args c;
  ru_as_conv_args(a, &c);
  if (const int rc = slab_fill_plan(&c, p)) return rc;
  MV2_CHECK_ARG(p.bn == a->C && p.n_tiles_n == 1 && p.row_bytes == 128);
  p.tpw = 1;
  p.h_stride = p.kchunks * 16384;
  const int budget = slab_ring_budget(p, true), w_bytes = p.bn * p.row_bytes;
  p.slab_stages = 3 * p.slab_stride + 2 * w_bytes <= budget ? 3 : 2;
  p.w_stages = std::min(12, (budget - p.slab_stages * p.slab_stride) / w_bytes);
  MV2_CHECK_ARG(p.w_stages >= 2);
  p.bias1 = a->b1; p.se_wk = a->se_wk; p.se_bk = a->se_bk; p.se_ws = a->se_ws;
  return MV2_OK;
}

extern "C" int mv2_tc_ru_records(const mv2_tc_ru_args* a) {
  if (!mv2_tc_ru_supported(a)) { set_error("mv2_tc_ru_records: unsupported shape"); return MV2_E_UNSUPPORTED; }
  SlabParams p;
  if (const int rc = ru_fill_plan(a, p)) return rc;
  return p.tiles_h * p.tiles_w * 4;
}

extern "C" size_t mv2_tc_ru_workspace_bytes(const mv2_tc_ru_args* a) {
  const int recs = mv2_tc_ru_records(a);
  if (recs <= 0) return 0;
  const size_t F = (size_t)a->B * a->T;
  return (F * recs * (a->C + 2) + F * (a->C + 16)) * sizeof(float);    // pool records + the SE hidden layer (mv2_se_gate_records)
}

extern "C" int mv2_tc_ru_forward(const mv2_tc_ru_args* a, const mv2_conv_hist* hist, void* stream) {
  MV2_CHECK_ARG(a && a->x && a->w3 && a->w1 && a->y && a->se_wk && a->se_ws);
  MV2_CHECK_ARG(!hist || (hist->T_h >= 0 && (hist->T_h == 0 || (hist->h && hist->clip_stride > 0))));
  if (!mv2_tc_ru_supported(a)) { set_error("mv2_tc_ru_forward: unsupported shape"); return MV2_E_UNSUPPORTED; }
  SlabParams p;
  if (const int rc = ru_fill_plan(a, p)) return rc;
  mv2_tc_conv_args c;
  ru_as_conv_args(a, &c);
  if (const int rc = slab_encode_maps(p, &c, hist)) return rc;
  const cuuint64_t dims1[2] = {(cuuint64_t)a->C, (cuuint64_t)a->C};
  const cuuint64_t strides1[1] = {(cuuint64_t)a->C * 2};
  const cuuint32_t box1[2] = {64, (cuuint32_t)p.bn};
  if (const int rc = encode_tc_map(&p.w1map, p.dtype, 2, a->w1, dims1, strides1, box1, CU_TENSOR_MAP_SWIZZLE_128B, "w1")) return rc;
  if (const int rc = slab_encode_out_maps(p, EPI_FUSED_RU)) return rc;
  return slab_launch(EPI_FUSED_RU, p, stream);
}


// =====================================================================================================================
// SpatialDownsample2x (reference M:770-780: per-frame Conv2d k3 s2 p1) on the slab design.
// The input (H x W x C) is read as (H) x (W/2) x (2C): output column wo needs input columns 2wo-1, 2wo, 2wo+1 =
// (w2 = wo-1, second half of the 2C axis), (w2 = wo, first half), (w2 = wo, second half), i.e. a 2-tap conv along w2 whose
// dw2 = -1 tap only touches the upper C channels.  Rows: output row ho needs input rows 2ho-1, 2ho, 2ho+1: the slab stage
// holds the odd rows and the even rows as two sub-slabs (two TMA box loads through row-parity tensor maps), and the three dh
// taps start in (odd, row 0), (even, row 0), (odd, row 1).  Weights are packed by the host as w[co][tap'][2C],
// tap' = dh * 2 + (dw2 + 1), lower half of the dw2 = -1 taps zero (and never loaded).
// =====================================================================================================================
extern "C" int mv2_tc_down_space_supported(const mv2_tc_conv_args* a) {
  if (!a || tc_dtype(a) < 0) return 0;
  const int es = tc_esize(tc_dtype(a));
  if (a->kt != 1 || a->kh != 3 || a->kw != 3 || a->st != 1 || a->sh != 2 || a->sw != 2) return 0;
  if (a->pt != 0 || a->ph != 1 || a->pw != 1) return 0;
  if ((a->Hi & 1) || (a->Wi & 1) || a->Ho != a->Hi / 2 || a->Wo != a->Wi / 2 || a->To != a->Ti) return 0;
  if ((a->Ci * es) % 128 != 0 || a->Co % 32 != 0 || a->Co > 4096) return 0;    // 128-byte K rows
  if (a->res || a->shuffle != MV2_SHUFFLE_NONE || a->epi_mode != 0 || a->out_layout != 0 || a->oscale) return 0;
  return 1;
}

extern "C" int mv2_tc_down_space_forward(const mv2_tc_conv_args* a, void* stream) {
  MV2_CHECK_ARG(a && a->x && a->w && a->y);
  if (!mv2_tc_down_space_supported(a)) { set_error("mv2_tc_down_space_forward: unsupported shape"); return MV2_E_UNSUPPORTED; }
  SlabParams p;
  memset(&p, 0, sizeof(p));
  p.dtype = tc_dtype(a);
  const int es = tc_esize(p.dtype);
  const int C2 = 2 * a->Ci, bk = 128 / es;     // channels of one 128-byte K row
  p.kt = 1; p.kh = 3; p.kw = 2; p.pt = 0; p.ph = 1; p.pw = 1; p.st = 1;
  p.row_bytes = 128; p.Ci = C2; p.kchunks = C2 / bk; p.dn_lower = a->Ci / bk;
  p.B = a->B; p.T = a->To; p.H = a->Ho; p.W = a->Wo; p.Co = a->Co;
  p.epi = tc_epi_of(a);
  int bn = 32;
  for (int c = 128; c >= 32; c >>= 1) if (a->Co % c == 0) { bn = c; break; }
  const int w_bytes = bn * 128;
  p.bn = bn; p.n_tiles_n = a->Co / bn; p.tpw = 1;
  p.tiles_h = ceil_div(a->Ho, 16);
  p.slab_h = 17;       // the odd-row sub-slab (input rows 2 ho - 1: 17 rows for 16 output rows) is an ordinary slab ...
  int budget;
  for (int mw = slab_default_mw(bn, a->Wo);; mw >>= 1) {   // the two sub-slabs of a wide macro tile do not fit twice: narrow it
    slab_set_geometry(p, mw);
    p.dn_e_off = p.slab_stride;    // ... and the 16-row even-row sub-slab follows it at the next 1024-byte boundary
    const int e_bytes = 16 * p.pitch * 128;
    p.slab_bytes += e_bytes;
    p.slab_stride += (e_bytes + 1023) / 1024 * 1024;
    budget = slab_ring_budget(p, false);
    if (mw == 1 || 2 * p.slab_stride + 3 * w_bytes <= budget) break;
  }
  for (int dh = 0; dh < 3; ++dh)
    for (int q = 0; q < 2; ++q)      // q = dw2 + 1
      p.dn_aoff[dh * 2 + q] = ((dh == 1 ? p.dn_e_off : 0) + ((dh == 2 ? p.pitch : 0) + q) * 128) >> 4;
  p.slab_stages = p.slab_stride * 3 + w_bytes * 4 <= budget ? 3 : 2;
  p.w_stages = std::min(12, (budget - p.slab_stages * p.slab_stride) / w_bytes);
  MV2_CHECK_ARG(p.w_stages >= 2);

  const int64_t rowb = (int64_t)a->Wi * a->Ci * es;
  const cuuint64_t dims[5] = {(cuuint64_t)C2, (cuuint64_t)(a->Wi / 2), (cuuint64_t)(a->Hi / 2), (cuuint64_t)a->Ti, (cuuint64_t)a->B};
  const cuuint64_t strides[4] = {(cuuint64_t)(C2 * es), (cuuint64_t)(2 * rowb), (cuuint64_t)(a->Hi * rowb), (cuuint64_t)(a->Ti * a->Hi * rowb)};
  const cuuint32_t box_e[5] = {(cuuint32_t)bk, (cuuint32_t)p.pitch, 16, 1, 1}, box_o[5] = {(cuuint32_t)bk, (cuuint32_t)p.pitch, 17, 1, 1};
  if (const int rc = encode_tc_map(&p.amap, p.dtype, 5, a->x, dims, strides, box_e, CU_TENSOR_MAP_SWIZZLE_128B, "even rows")) return rc;
  if (const int rc = encode_tc_map(&p.amap_odd, p.dtype, 5, (const char*)a->x + rowb, dims, strides, box_o, CU_TENSOR_MAP_SWIZZLE_128B, "odd rows")) return rc;
  const int64_t K = 6 * (int64_t)C2;
  const cuuint64_t wdims[2] = {(cuuint64_t)K, (cuuint64_t)a->Co};
  const cuuint64_t wstrides[1] = {(cuuint64_t)(K * es)};
  const cuuint32_t wbox[2] = {(cuuint32_t)bk, (cuuint32_t)bn};
  if (const int rc = encode_tc_map(&p.wmap2, p.dtype, 2, a->w, wdims, wstrides, wbox, CU_TENSOR_MAP_SWIZZLE_128B, "weights")) return rc;
  p.wmap = p.wmap2;
  if (const int rc = slab_encode_out_maps(p, EPI_DOWN_SPACE)) return rc;
  return slab_launch(EPI_DOWN_SPACE, p, stream);
}
