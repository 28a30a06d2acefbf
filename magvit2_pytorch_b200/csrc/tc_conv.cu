// wgmma / TMA implicit-GEMM convolution for sm_90a (bf16, fp16 or fp32 with TF32 multiply in, fp32 accumulate in registers).
//
// One kernel covers the whole dense-contraction family of the VideoTokenizer forward path:
// causal 3x3x3 convs, 1x1x1 convs / Linear layers, the strided compress_space / compress_time
// convs and the 1x1 up-samplers with their depth-to-space / depth-to-time stores.
//
// GEMM view:  D[m][n] = sum_{tap, c} X[pos(m) + off(tap)][c] * W[n][tap][c]
//   M = 128 output positions per CTA, laid out as a (bt, bh, bw) box of the output volume
//   N = 32, 64 or 128 output channels per CTA
//   K = taps x Ci, walked in BK-channel slices of one tap at a time
// Operand staging: one TMA box load per (tap, slice) for A -- the box {BK, bw, bh, bt, 1} of the
// channels-last activation tensor shifted by the tap offset; out-of-bounds elements (the causal
// time halo, the spatial halo, ragged tile edges) are zero-filled by the TMA unit, so no padded
// copy of the activations is ever materialised (the reference does F.pad + conv, M:924-928).
// Strided convs read through "parity view" tensor maps (one per stride phase).  Both operands are
// K-major in shared memory with the hardware 128B/64B/32B swizzle (BK = 64/32/16 16-bit or 32/16/8 fp32 channels).
// Warp roles (384 threads): warp 0 = TMA producer, warps 4-11 = two consumer warpgroups (rows 0-63 / 64-127 of the
// tile): wgmma into registers, then the epilogue (accumulator -> shared-memory staging -> bias/activation/residual
// -> global, one output row per thread and 32-column chunk).
#include "common.cuh"
#include "tc_common.cuh"
#include <cuda.h>
#include <mutex>
#include <algorithm>
#include <string.h>

namespace mv2 {

// ------------------------------------------------------------------------------------------
// kernel
// ------------------------------------------------------------------------------------------
constexpr int TC_MAX_TAPS = 64;
constexpr int TC_MAX_MAPS = 8;
constexpr int TC_BM = 128;

struct alignas(64) TcParams {
  CUtensorMap amap[TC_MAX_MAPS];
  CUtensorMap hmap;      // history frames in front of x (mv2_conv_hist; stride 1 only): used when frame_loads > 1
  CUtensorMap wmap;
  int8_t tap_map[TC_MAX_TAPS], tap_dt[TC_MAX_TAPS], tap_dh[TC_MAX_TAPS], tap_dw[TC_MAX_TAPS];
  int ntaps, kchunks, ci_pad, bk;
  int B, To, Ho, Wo, Co;
  int bt, bh, bw, tt, th, tw;
  int bn, stages;
  int hist_T;
  int frame_loads;       // hist_T = 0: 1 box of bt frames per stage; else bt boxes of one frame, each from x or the history
  TcEpi epi;
};

template <typename T, int MODE, int BN>
__device__ __forceinline__ void tc_conv_body(const TcParams& p) {
  extern __shared__ uint8_t smem_raw[];
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int bk = p.bk;
  const uint32_t row_bytes = bk * (int)sizeof(T);
  const uint32_t a_bytes = TC_BM * row_bytes;
  const uint32_t b_bytes = BN * row_bytes;
  const uint32_t stage_bytes = a_bytes + b_bytes;   // both multiples of 1024 (BN >= 32, bk >= 16)
  const uint32_t bar_base = smem_base + p.stages * stage_bytes;
  // barriers: full[s] at +8s, empty[s] at +8(S+s)
  const uint32_t full0 = bar_base, empty0 = bar_base + 8 * p.stages;
  const uint32_t sbias_u = (empty0 + 8 * p.stages + 15) & ~15u;
  float* sbias = reinterpret_cast<float*>(smem_raw + (sbias_u - smem_u32(smem_raw)));   // BN floats, 16-byte aligned
  float* stg_all = sbias + BN;                                                            // 2 x [64][BN + 4] fp32 staging

  // tile coordinates
  int tile = blockIdx.x;
  const int iw = tile % p.tw; tile /= p.tw;
  const int ih = tile % p.th; tile /= p.th;
  const int it = tile % p.tt; tile /= p.tt;
  const int b = tile;
  const int w0 = iw * p.bw, h0 = ih * p.bh, t0 = it * p.bt;
  const int n0 = blockIdx.y * BN;

  if (threadIdx.x == 0) {
    for (int s = 0; s < p.stages; ++s) {
      mbar_init(full0 + 8 * s, 1);
      mbar_init(empty0 + 8 * s, 8);     // one arrival per consumer warp
    }
    fence_barrier_init();
  }
  if (warp == 0 && lane == 0) {
    tma_prefetch_desc(&p.wmap);
    tma_prefetch_desc(&p.amap[0]);
  }
  if (warp >= 4)
    for (int i = threadIdx.x - 128; i < BN; i += 256) sbias[i] = (p.epi.bias && n0 + i < p.Co) ? p.epi.bias[n0 + i] : 0.f;
  __syncthreads();
  // everything above overlapped the previous kernel's tail (PDL); activations may only be touched from here on
  pdl_wait();
  pdl_launch_dependents();

  const int n_iters = p.ntaps * p.kchunks;
  if (warp == 0) {
    if (lane == 0) {
      // incremental ring / tap bookkeeping: no division or modulo in the loop
      uint32_t s = 0, ph = 0;
      int tap = 0, kc = 0;
      for (int i = 0; i < n_iters; ++i) {
        mbar_wait(empty0 + 8 * s, ph ^ 1);
        mbar_expect_tx(full0 + 8 * s, stage_bytes);
        const uint32_t sa = smem_base + s * stage_bytes;
        if (p.hist_T == 0)
          tma_load_5d(sa, &p.amap[p.tap_map[tap]], full0 + 8 * s, kc * bk, w0 + p.tap_dw[tap], h0 + p.tap_dh[tap],
                      t0 + p.tap_dt[tap], b);
        else
          for (int lt = 0; lt < p.frame_loads; ++lt) {     // frames in front of the chunk come from the history
            const int ti = t0 + lt + p.tap_dt[tap];
            tma_load_5d(sa + lt * (uint32_t)(p.bw * p.bh) * row_bytes, ti >= 0 ? &p.amap[0] : &p.hmap, full0 + 8 * s, kc * bk,
                        w0 + p.tap_dw[tap], h0 + p.tap_dh[tap], ti >= 0 ? ti : ti + p.hist_T, b);
          }
        tma_load_2d(sa + a_bytes, &p.wmap, full0 + 8 * s, tap * p.ci_pad + kc * bk, n0);
        if (++kc == p.kchunks) { kc = 0; ++tap; }
        if (++s == (uint32_t)p.stages) { s = 0; ph ^= 1; }
      }
    }
  } else if (warp >= 4) {
    // ---------------- consumer warpgroups: wgmma main loop ----------------
    const int wg = (warp - 4) >> 2, t = threadIdx.x & 127;
    const uint64_t d_hi = gmma_desc_hi(8 * row_bytes, row_bytes);
    const int ksteps = bk >> (sizeof(T) == 4 ? 3 : 4);   // 32-byte MMA K steps per K row
    // this warpgroup's 64 rows start 64 rows into the A tile; one MMA K step (16 bf16 / fp16 or 8 fp32) = +32 bytes = +2
    // address units
    const uint32_t stage16 = stage_bytes >> 4, a16 = a_bytes >> 4, wg16 = (uint32_t)wg * ((64 * row_bytes) >> 4);
    uint32_t s = 0, ph = 0, lo = desc_lo(smem_base);
    float acc[BN / 2];
    for (int i = 0; i < n_iters; ++i) {
      mbar_wait(full0 + 8 * s, ph);
      wgmma_fence();
      const uint64_t ad = d_hi | (uint64_t)(lo + wg16);
      const uint64_t bd = d_hi | (uint64_t)(lo + a16);
      wgmma_mma<T, BN>(acc, ad, bd, i > 0 ? 1u : 0u);
      if (ksteps > 1) wgmma_mma<T, BN>(acc, ad + 2, bd + 2, 1u);
      if (ksteps > 2) {
        wgmma_mma<T, BN>(acc, ad + 4, bd + 4, 1u);
        wgmma_mma<T, BN>(acc, ad + 6, bd + 6, 1u);
      }
      wgmma_commit();
      wgmma_wait_all();
      __syncwarp();
      if (lane == 0) mbar_arrive(empty0 + 8 * s);   // frees the smem slot: these MMAs have read it
      if (++s == (uint32_t)p.stages) { s = 0; ph ^= 1; lo = desc_lo(smem_base); } else { lo += stage16; }
    }
    // ---------------- epilogue: one output row per thread, the two warps of a 32-row quarter split the columns ----------------
    float* stg = stg_all + wg * 64 * (BN + 4);
    stage_acc<BN>(acc, stg, t);
    named_bar_sync(1 + wg, 128);
    const int wq = warp & 3;
    const int sub = 2 * wg + (wq & 1), half = wq >> 1;
    const int row = sub * 32 + lane;
    const int lw = row % p.bw, lh = (row / p.bw) % p.bh, lt = row / (p.bw * p.bh);
    const int wo = w0 + lw, ho = h0 + lh, to = t0 + lt;
    const bool row_ok = wo < p.Wo && ho < p.Ho && to < p.To;
    const int64_t row_base = ((((int64_t)b * p.To + to) * p.Ho + ho) * p.Wo + wo) * p.Co;
    const float* srow = stg + (row - 64 * wg) * (BN + 4);
    for (int c0 = half * 32; c0 < BN; c0 += 64) {
      uint32_t r[32];
      load_row32(srow + c0, 32, r);
      if (row_ok) epi_chunk32<T, MODE>(p.epi, r, 32, n0 + c0, sbias + c0, b, to, ho, wo, row_base);
    }
  }
}

// ------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------
// kernel instance per (element type, epilogue flavour, N tile); every instance may use up to 227 KB of dynamic shared
// memory.  [0] bf16, [1] fp16, [2] TF32; rows: ragged (plain) stores, GEGLU, depth-to-space / depth-to-time shuffle.
// One kernel per element type (the names of the bf16 instances are those of the library before fp16 existed)
template <int MODE, int BN>
__global__ void __launch_bounds__(384, 1) tc_conv_kernel(const __grid_constant__ TcParams p) { tc_conv_body<__nv_bfloat16, MODE, BN>(p); }
template <int MODE, int BN>
__global__ void __launch_bounds__(384, 1) tc_conv_f16_kernel(const __grid_constant__ TcParams p) { tc_conv_body<__half, MODE, BN>(p); }
template <int MODE, int BN>
__global__ void __launch_bounds__(384, 1) tc_conv_tf32_kernel(const __grid_constant__ TcParams p) { tc_conv_body<float, MODE, BN>(p); }
#define MV2_TC_BN(K, M) {K<M, 32>, K<M, 64>, K<M, 128>}
#define MV2_TC_FLAVOURS(K) {MV2_TC_BN(K, EPI_RAGGED), MV2_TC_BN(K, EPI_GEGLU), MV2_TC_BN(K, EPI_SHUFFLE)}
static void (*const g_tc_kernels[3][3][3])(TcParams) = {MV2_TC_FLAVOURS(tc_conv_kernel), MV2_TC_FLAVOURS(tc_conv_f16_kernel),
                                                        MV2_TC_FLAVOURS(tc_conv_tf32_kernel)};
#undef MV2_TC_FLAVOURS
#undef MV2_TC_BN

}  // namespace mv2

using namespace mv2;

extern "C" {

// output tile box of a launch: bw * bh * bt = 128 positions
static void tc_tile_box(const mv2_tc_conv_args* a, int& bw, int& bh, int& bt) {
  bw = std::min(128, pow2_ceil(a->Wo));
  bh = std::min(128 / bw, pow2_ceil(a->Ho));
  bt = 128 / (bw * bh);
}

int mv2_tc_conv_hist_supported(const mv2_tc_conv_args* a) {
  if (!mv2_tc_conv_supported(a) || a->st != 1 || a->sh != 1 || a->sw != 1) return 0;
  int bw, bh, bt;
  tc_tile_box(a, bw, bh, bt);
  return bt == 1 || (bw * bh) % 8 == 0;      // one box per frame: each must start on a whole swizzle pattern (8 rows)
}

int mv2_tc_conv_supported(const mv2_tc_conv_args* a) {
  if (!a) return 0;
  if (tc_dtype(a) < 0) return 0;
  if (a->Ci * tc_esize(tc_dtype(a)) % 32 != 0) return 0;   // TMA inner box = 32/64/128 B, global strides multiple of 16 B
  if (a->kt * a->kh * a->kw > TC_MAX_TAPS) return 0;
  if (a->st < 1 || a->st > 2 || a->sh < 1 || a->sh > 2 || a->sw < 1 || a->sw > 2) return 0;
  if (a->shuffle != MV2_SHUFFLE_NONE && ((a->shuffle == MV2_SHUFFLE_SPACE ? a->Co / 4 : a->Co / 2) % 8 != 0)) return 0;
  if (a->res && a->Co % 8 != 0) return 0;
  if (a->epi_mode == 1 && (a->Co % 32 != 0 || a->shuffle != MV2_SHUFFLE_NONE || a->res)) return 0;   // GEGLU pairs
  if (a->epi_mode == 2 && (!a->res || a->shuffle != MV2_SHUFFLE_NONE)) return 0;   // scaled residual
  if (a->epi_mode < 0 || a->epi_mode > 2) return 0;
  if (a->out_layout != 0) return 0;
  if (a->oscale && (a->epi_mode != 0 || a->shuffle != MV2_SHUFFLE_NONE)) return 0;
  return 1;
}

int mv2_tc_conv_forward(const mv2_tc_conv_args* a, const mv2_conv_hist* hist, void* stream) {
  MV2_CHECK_ARG(a && a->x && a->w && a->y);
  MV2_CHECK_ARG(!hist || (hist->T_h >= 0 && (hist->T_h == 0 || (hist->h && hist->clip_stride > 0))));
  const int hist_T = hist ? hist->T_h : 0;
  if (!mv2_tc_conv_supported(a)) { set_error("mv2_tc_conv_forward: unsupported shape (Ci=%d Co=%d)", a->Ci, a->Co); return MV2_E_UNSUPPORTED; }

  const int dt = tc_dtype(a), es = tc_esize(dt);
  TcParams p;
  memset(&p, 0, sizeof(p));
  const int ci_bytes = a->Ci * es;
  const int row_bytes = ci_bytes % 128 == 0 ? 128 : (ci_bytes % 64 == 0 ? 64 : 32);   // one K row of the operand tiles
  const int bk = row_bytes / es;
  const CUtensorMapSwizzle swz = swizzle_of_row(row_bytes);
  p.bk = bk;
  p.ci_pad = a->Ci;
  p.kchunks = a->Ci / bk;
  p.B = a->B; p.To = a->To; p.Ho = a->Ho; p.Wo = a->Wo; p.Co = a->Co;
  // output tile box: bw * bh * bt = 128
  tc_tile_box(a, p.bw, p.bh, p.bt);
  p.tw = ceil_div(a->Wo, p.bw); p.th = ceil_div(a->Ho, p.bh); p.tt = ceil_div(a->To, p.bt);
  p.hist_T = hist_T;
  p.frame_loads = hist_T > 0 ? p.bt : 1;
  if (hist_T > 0 && !mv2_tc_conv_hist_supported(a)) {
    set_error("mv2_tc_conv_forward: unsupported shape with history (mv2_tc_conv_hist_supported)");
    return MV2_E_UNSUPPORTED;
  }
  // N tile: 32, 64 or 128 columns (a wgmma N, 64 fp32 accumulator registers per thread at 128); wider outputs take
  // several N tiles, a ragged last one reads zero-filled weight rows and stores nothing for them
  const int bn = a->Co <= 32 ? 32 : (a->Co <= 64 ? 64 : 128);
  p.bn = bn;
  const int stage_bytes = TC_BM * row_bytes + bn * row_bytes;
  MV2_CHECK_ARG((TC_BM * row_bytes) % 1024 == 0 && (bn * row_bytes) % 1024 == 0);
  const int stg_bytes = 2 * 64 * (bn + 4) * 4;         // accumulator staging of the two consumer warpgroups
  // ring depth: no deeper than the K loop
  int stages = (200 * 1024 - stg_bytes) / stage_bytes;
  stages = std::max(2, std::min(stages, 8));
  stages = std::max(1, std::min(stages, a->kt * a->kh * a->kw * (a->Ci / bk)));
  p.stages = stages;
  p.epi = tc_epi_of(a);

  // ---- activation tensor maps: one per stride-parity phase ----
  const int st = a->st, sh = a->sh, sw = a->sw;
  const int nmaps = st * sh * sw;
  MV2_CHECK_ARG(nmaps <= TC_MAX_MAPS);
  const int64_t C = a->Ci, W = a->Wi, H = a->Hi, T = a->Ti;
  for (int pt = 0; pt < st; ++pt)
    for (int ph = 0; ph < sh; ++ph)
      for (int pw = 0; pw < sw; ++pw) {
        const int id = (pt * sh + ph) * sw + pw;
        const int64_t nW = (W - pw + sw - 1) / sw, nH = (H - ph + sh - 1) / sh, nT = (T - pt + st - 1) / st;
        if (nW <= 0 || nH <= 0 || nT <= 0) { set_error("empty stride phase (dimension smaller than stride)"); return MV2_E_UNSUPPORTED; }
        const cuuint64_t dims[5] = {(cuuint64_t)C, (cuuint64_t)nW, (cuuint64_t)nH, (cuuint64_t)nT, (cuuint64_t)a->B};
        const cuuint64_t strides[4] = {(cuuint64_t)(sw * C * es), (cuuint64_t)(sh * W * C * es), (cuuint64_t)(st * H * W * C * es),
                                       (cuuint64_t)(T * H * W * C * es)};
        const cuuint32_t box[5] = {(cuuint32_t)bk, (cuuint32_t)p.bw, (cuuint32_t)p.bh, (cuuint32_t)(128 / (p.bw * p.bh * p.frame_loads)), 1};
        const char* base = (const char*)a->x + ((int64_t)pt * H * W + (int64_t)ph * W + pw) * C * es;
        char what[32];
        snprintf(what, sizeof(what), "activations, phase %d", id);
        if (const int rc = encode_tc_map(&p.amap[id], dt, 5, base, dims, strides, box, swz, what)) return rc;
      }
  if (hist_T > 0) {
    const cuuint64_t dims[5] = {(cuuint64_t)C, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)hist_T, (cuuint64_t)a->B};
    const cuuint64_t strides[4] = {(cuuint64_t)(C * es), (cuuint64_t)(W * C * es), (cuuint64_t)(H * W * C * es), (cuuint64_t)(hist->clip_stride * es)};
    const cuuint32_t box[5] = {(cuuint32_t)bk, (cuuint32_t)p.bw, (cuuint32_t)p.bh, 1, 1};
    if (const int rc = encode_tc_map(&p.hmap, dt, 5, hist->h, dims, strides, box, swz, "history")) return rc;
  }
  // ---- taps ----
  p.ntaps = a->kt * a->kh * a->kw;
  for (int dt = 0; dt < a->kt; ++dt)
    for (int dh = 0; dh < a->kh; ++dh)
      for (int dw = 0; dw < a->kw; ++dw) {
        const int tap = (dt * a->kh + dh) * a->kw + dw;
        const int ot = dt - a->pt, oh = dh - a->ph, ow = dw - a->pw;
        const int pt = ((ot % st) + st) % st, ph = ((oh % sh) + sh) % sh, pw = ((ow % sw) + sw) % sw;
        p.tap_map[tap] = (int8_t)((pt * sh + ph) * sw + pw);
        p.tap_dt[tap] = (int8_t)floor_div(ot, st);
        p.tap_dh[tap] = (int8_t)floor_div(oh, sh);
        p.tap_dw[tap] = (int8_t)floor_div(ow, sw);
      }
  // ---- weights map: [Co][taps * Ci] K-major ----
  const int64_t K = (int64_t)p.ntaps * a->Ci;
  const cuuint64_t wdims[2] = {(cuuint64_t)K, (cuuint64_t)a->Co};
  const cuuint64_t wstrides[1] = {(cuuint64_t)(K * es)};
  const cuuint32_t wbox[2] = {(cuuint32_t)bk, (cuuint32_t)bn};
  if (const int rc = encode_tc_map(&p.wmap, dt, 2, a->w, wdims, wstrides, wbox, swz, "weights")) return rc;

  const size_t smem = 1024 + (size_t)stages * stage_bytes + 16 * stages + 16 + (size_t)bn * 4 + stg_bytes;
  static PerDeviceOnce attr_once;
  const cudaError_t attr_err = attr_once.run([] {
    cudaError_t e = cudaSuccess;
    for (auto& type : g_tc_kernels)
      for (auto& row : type)
        for (auto k : row)
          if (e == cudaSuccess) e = cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024);
    return e;
  });
  if (attr_err != cudaSuccess) { set_error("cudaFuncSetAttribute failed: %s", cudaGetErrorString(attr_err)); return MV2_E_CUDA; }
  MV2_CHECK_ARG(smem <= 227 * 1024);
  dim3 grid((unsigned)((int64_t)a->B * p.tt * p.th * p.tw), (unsigned)ceil_div(a->Co, bn));
  const int flavour = a->epi_mode == 1 ? 1 : (a->shuffle != MV2_SHUFFLE_NONE ? 2 : 0);   // row of g_tc_kernels
  launch_k(g_tc_kernels[dt == MV2_F16 ? 1 : (dt == MV2_TF32 ? 2 : 0)][flavour][bn == 32 ? 0 : (bn == 64 ? 1 : 2)], grid, dim3(384), smem, (cudaStream_t)stream, p);
  MV2_CHECK_LAUNCH();
  return MV2_OK;
}

}  // extern "C"
