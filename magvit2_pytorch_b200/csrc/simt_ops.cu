// CUDA-core (fp32-accumulate) kernels of libmagvit2_b200.so.
//
// These cover every operator of the VideoTokenizer forward path for ANY shape and for both
// activation dtypes.  They are (a) the whole fp32 parity path (fp32 storage + fp32 FMA, no
// TF32), (b) the memory-bound operators of the bf16 path (SqueezeExcite, norms, attention
// cores, GEGLU, quantisers, layout), and (c) the on-device cross-check for the wgmma
// implicit-GEMM kernels in tc_conv.cu, which take over the dense contractions in bf16.
//
// Reference semantics are cited per entry point in include/magvit2_b200.h.
#include "common.cuh"
#include <type_traits>
#include <math.h>
#include <stdlib.h>
#include <mutex>
#include <algorithm>

namespace mv2 {

int g_pdl = 0;

// Cap for the grid of a grid-stride elementwise kernel: `per_sm` blocks on every SM of the current device.
static int grid_cap(int per_sm) {
  static thread_local int dev_cached = -1, n_sm = 132;
  int dev = 0;
  if (cudaGetDevice(&dev) == cudaSuccess && dev != dev_cached) {
    int v = 0;
    if (cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, dev) == cudaSuccess && v > 0) n_sm = v;
    dev_cached = dev;
  }
  return n_sm * per_sm;
}
static thread_local char g_err[512] = "";
thread_local uint64_t g_launches = 0;
void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

// ------------------------------------------------------------------------------------------
// layout
// ------------------------------------------------------------------------------------------
// src [B][R][S] -> dst [B][S_dst][R]  (R = channels rows, S = positions), dst position = s + s_off_dst,
// src position = s + s_off_src.  Classic 32x32 smem tile transpose.
template <typename TS, typename TD>
__global__ void transpose_rs_kernel(const TS* __restrict__ src, TD* __restrict__ dst, int R, int64_t S,
                                    int64_t src_S_total, int64_t dst_S_total, int64_t s_off_src,
                                    int64_t s_off_dst, bool src_is_rs) {
  pdl_wait();
  pdl_launch_dependents();
  __shared__ float tile[32][33];
  const int b = blockIdx.z;
  const int64_t s0 = (int64_t)blockIdx.x * 32;
  const int r0 = blockIdx.y * 32;
  const int tx = threadIdx.x, ty = threadIdx.y;
  if (src_is_rs) {
    // src [B][R][S_total] -> dst [B][S_total'][R]
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      int r = r0 + ty + 8 * j;
      int64_t s = s0 + tx;
      float v = 0.f;
      if (r < R && s < S) v = to_f32<TS>(src[((int64_t)b * R + r) * src_S_total + s + s_off_src]);
      tile[ty + 8 * j][tx] = v;
    }
    __syncthreads();
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      int64_t s = s0 + ty + 8 * j;
      int r = r0 + tx;
      if (r < R && s < S) dst[((int64_t)b * dst_S_total + s + s_off_dst) * R + r] = from_f32<TD>(tile[tx][ty + 8 * j]);
    }
  } else {
    // src [B][S_total][R] -> dst [B][R][S_total']
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      int64_t s = s0 + ty + 8 * j;
      int r = r0 + tx;
      float v = 0.f;
      if (r < R && s < S) v = to_f32<TS>(src[((int64_t)b * src_S_total + s + s_off_src) * R + r]);
      tile[ty + 8 * j][tx] = v;
    }
    __syncthreads();
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      int r = r0 + ty + 8 * j;
      int64_t s = s0 + tx;
      if (r < R && s < S) dst[((int64_t)b * R + r) * dst_S_total + s + s_off_dst] = from_f32<TD>(tile[tx][ty + 8 * j]);
    }
  }
}

template <typename TS, typename TD>
static int launch_transpose(const void* src, void* dst, int B, int R, int64_t S, int64_t src_S_total,
                            int64_t dst_S_total, int64_t s_off_src, int64_t s_off_dst, bool src_is_rs,
                            cudaStream_t st) {
  dim3 grid(ceil_div(S, 32), ceil_div(R, 32), B), block(32, 8);
  launch_k(transpose_rs_kernel<TS, TD>, dim3(grid), dim3(block), 0, st, (const TS*)src, (TD*)dst, R, S, src_S_total, dst_S_total,
                                                      s_off_src, s_off_dst, src_is_rs);
  MV2_CHECK_LAUNCH();
  return MV2_OK;
}

static int dispatch_transpose(const void* src, int sd, void* dst, int dd, int B, int R, int64_t S,
                              int64_t src_S_total, int64_t dst_S_total, int64_t s_off_src, int64_t s_off_dst,
                              bool src_is_rs, cudaStream_t st) {
  if (sd == MV2_F32 && dd == MV2_F32)
    return launch_transpose<float, float>(src, dst, B, R, S, src_S_total, dst_S_total, s_off_src, s_off_dst, src_is_rs, st);
  if (sd == MV2_F32 && dd == MV2_BF16)
    return launch_transpose<float, __nv_bfloat16>(src, dst, B, R, S, src_S_total, dst_S_total, s_off_src, s_off_dst, src_is_rs, st);
  if (sd == MV2_BF16 && dd == MV2_F32)
    return launch_transpose<__nv_bfloat16, float>(src, dst, B, R, S, src_S_total, dst_S_total, s_off_src, s_off_dst, src_is_rs, st);
  if (sd == MV2_BF16 && dd == MV2_BF16)
    return launch_transpose<__nv_bfloat16, __nv_bfloat16>(src, dst, B, R, S, src_S_total, dst_S_total, s_off_src, s_off_dst, src_is_rs, st);
  if (sd == MV2_U8 && dd == MV2_F32)
    return launch_transpose<uint8_t, float>(src, dst, B, R, S, src_S_total, dst_S_total, s_off_src, s_off_dst, src_is_rs, st);
  if (sd == MV2_U8 && dd == MV2_BF16)
    return launch_transpose<uint8_t, __nv_bfloat16>(src, dst, B, R, S, src_S_total, dst_S_total, s_off_src, s_off_dst, src_is_rs, st);
  if (sd == MV2_F32 && dd == MV2_F16)
    return launch_transpose<float, __half>(src, dst, B, R, S, src_S_total, dst_S_total, s_off_src, s_off_dst, src_is_rs, st);
  if (sd == MV2_F16 && dd == MV2_F32)
    return launch_transpose<__half, float>(src, dst, B, R, S, src_S_total, dst_S_total, s_off_src, s_off_dst, src_is_rs, st);
  if (sd == MV2_F16 && dd == MV2_F16)
    return launch_transpose<__half, __half>(src, dst, B, R, S, src_S_total, dst_S_total, s_off_src, s_off_dst, src_is_rs, st);
  if (sd == MV2_U8 && dd == MV2_F16)
    return launch_transpose<uint8_t, __half>(src, dst, B, R, S, src_S_total, dst_S_total, s_off_src, s_off_dst, src_is_rs, st);
  set_error("unsupported dtype pair %d -> %d", sd, dd);
  return MV2_E_ARG;
}


// Video ingest for the tensor-core conv_in: packs the k_w taps of the (tiny-channel) input into the channel axis so the
// 7x7x7, C_in = 3 conv becomes a (7x7x1)-tap conv over 32 "channels":
//   dst[b][t + t_pad][h][w][dw * C + c] = src[b][c][t][h][w + dw - pw]   (0 outside the image / for padded channels)
// One block per (b, t, h) image row: the C source rows are staged in shared memory with a zero halo (coalesced
// loads, each source element read once), then every thread assembles groups of 8 packed channels from them (16 bytes of
// bf16 / fp16, 32 bytes of fp32).
template <typename TS, typename TD>
__global__ void __launch_bounds__(256) ingest_kwpack_kernel(const TS* __restrict__ src, TD* __restrict__ dst,
                                                            int B, int C, int T, int H, int W, int t_pad, int kw, int pw,
                                                            int cpack) {
  pdl_wait();
  pdl_launch_dependents();
  extern __shared__ float srow[];            // [C][W + kw - 1]
  const int pitch = W + kw - 1;
  const int groups = cpack >> 3;
  int r = blockIdx.x;
  const int h = r % H; r /= H;
  const int t = r % (T + t_pad);
  const int b = r / (T + t_pad);
  const int ts = t - t_pad;
  for (int i = threadIdx.x; i < C * pitch; i += blockDim.x) {
    const int c = i / pitch, ws = i - c * pitch - pw;
    float x = 0.f;
    if (ts >= 0 && ws >= 0 && ws < W) x = to_f32<TS>(src[((((int64_t)b * C + c) * T + ts) * H + h) * W + ws]);
    srow[i] = x;
  }
  __syncthreads();
  TD* drow = dst + (((int64_t)b * (T + t_pad) + t) * H + h) * (int64_t)W * cpack;
  for (int i = threadIdx.x; i < W * groups; i += blockDim.x) {
    const int g = i % groups, w = i / groups;
    int dw = (g * 8) / C, c = g * 8 - dw * C;
    float v[8];
#pragma unroll
    for (int q = 0; q < 8; ++q) {
      v[q] = dw < kw ? srow[c * pitch + w + dw] : 0.f;     // srow index w + dw  <->  source column w + dw - pw
      if (++c == C) { c = 0; ++dw; }
    }
    if constexpr (std::is_same<TD, float>::value) {
      float4* d4 = reinterpret_cast<float4*>(drow + (int64_t)i * 8);
      d4[0] = make_float4(v[0], v[1], v[2], v[3]);
      d4[1] = make_float4(v[4], v[5], v[6], v[7]);
    } else {
      uint4 o;
      pair_t<TD> p0 = f2_to_pair<TD>(v[0], v[1]), p1 = f2_to_pair<TD>(v[2], v[3]);
      pair_t<TD> p2 = f2_to_pair<TD>(v[4], v[5]), p3 = f2_to_pair<TD>(v[6], v[7]);
      o.x = *reinterpret_cast<uint32_t*>(&p0); o.y = *reinterpret_cast<uint32_t*>(&p1);
      o.z = *reinterpret_cast<uint32_t*>(&p2); o.w = *reinterpret_cast<uint32_t*>(&p3);
      *reinterpret_cast<uint4*>(drow + (int64_t)i * 8) = o;
    }
  }
}

// ------------------------------------------------------------------------------------------
// generic convolution (implicit GEMM on CUDA cores)
// ------------------------------------------------------------------------------------------
constexpr int CBM = 64, CBN = 64, CBK = 16;

template <typename T>
__global__ void __launch_bounds__(256) conv_simt_kernel(const mv2_conv_args a, const mv2_conv_hist hh) {
  pdl_wait();
  pdl_launch_dependents();
  __shared__ float As[CBK][CBM + 4];
  __shared__ float Bs[CBK][CBN + 4];
  const T* __restrict__ x = (const T*)a.x;
  const T* __restrict__ w = (const T*)a.w;
  const int tid = threadIdx.x;
  const int tx = tid & 15, ty = tid >> 4;
  const int64_t M = (int64_t)a.B * a.To * a.Ho * a.Wo;
  const int64_t m0 = (int64_t)blockIdx.x * CBM;
  const int n0 = blockIdx.y * CBN;

  // loader role: position lp (0..63), 4 consecutive channels at (tid & 3) * 4
  const int lp = tid >> 2, lk = (tid & 3) * 4;
  const int64_t lm = m0 + lp;
  const bool lvalid = lm < M;
  int lb = 0, lto = 0, lho = 0, lwo = 0;
  if (lvalid) {
    int64_t r = lm;
    lwo = (int)(r % a.Wo); r /= a.Wo;
    lho = (int)(r % a.Ho); r /= a.Ho;
    lto = (int)(r % a.To); r /= a.To;
    lb = (int)r;
  }
  // weight loader role: k row = tid >> 4, 4 columns at (tid & 15) * 4
  const int wk = tid >> 4, wn = (tid & 15) * 4;

  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;

  const int ntaps = a.kt * a.kh * a.kw;
  const int half_c = (a.Ci + 1) >> 1;      // torch.chunk(2): the first (unshifted) half takes ceil(C / 2) channels (M:250)
  for (int tap = 0; tap < ntaps; ++tap) {
    const int dw = tap % a.kw, dh = (tap / a.kw) % a.kh, dt = tap / (a.kw * a.kh);
    const int ti = lto * a.st - a.pt + dt;
    const int hi = lho * a.sh - a.ph + dh;
    const int wi = lwo * a.sw - a.pw + dw;
    const bool sp_ok = lvalid && hi >= 0 && hi < a.Hi && wi >= 0 && wi < a.Wi;
    for (int c0 = 0; c0 < a.Ci; c0 += CBK) {
      // ---- stage A (im2col gather) ----
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int c = c0 + lk + j;
        float v = 0.f;
        if (sp_ok && c < a.Ci) {
          int tt = ti;
          if (a.x_token_shift && c >= half_c) tt -= 1;
          if (tt >= 0 && tt < a.Ti)
            v = to_f32<T>(x[((((int64_t)lb * a.Ti + tt) * a.Hi + hi) * a.Wi + wi) * a.Ci + c]);
          else if (tt < 0 && tt >= -hh.T_h)       // frames in front of the chunk: the carried history (T_h = 0: none)
            v = to_f32<T>(((const T*)hh.h)[(int64_t)lb * hh.clip_stride + (((int64_t)(hh.T_h + tt) * a.Hi + hi) * a.Wi + wi) * a.Ci + c]);
        }
        As[lk + j][lp] = v;
      }
      // ---- stage B (weights) ----
      {
        const int c = c0 + wk;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const int n = n0 + wn + j;
          float v = 0.f;
          if (c < a.Ci && n < a.Co) v = to_f32<T>(w[((int64_t)tap * a.Ci + c) * a.Co + n]);
          Bs[wk][wn + j] = v;
        }
      }
      __syncthreads();
#pragma unroll
      for (int k = 0; k < CBK; ++k) {
        float av[4], bv[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) av[i] = As[k][ty * 4 + i];
#pragma unroll
        for (int j = 0; j < 4; ++j) bv[j] = Bs[k][tx * 4 + j];
#pragma unroll
        for (int i = 0; i < 4; ++i)
#pragma unroll
          for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
      }
      __syncthreads();
    }
  }

  // ---- epilogue: bias, activation, depth-to-space/time shuffle, residual ----
  T* __restrict__ y = (T*)a.y;
  const T* __restrict__ res = (const T*)a.res;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int64_t m = m0 + ty * 4 + i;
    if (m >= M) continue;
    int64_t r = m;
    const int wo = (int)(r % a.Wo); r /= a.Wo;
    const int ho = (int)(r % a.Ho); r /= a.Ho;
    const int to = (int)(r % a.To); r /= a.To;
    const int b = (int)r;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int n = n0 + tx * 4 + j;
      if (n >= a.Co) continue;
      float v = acc[i][j];
      if (a.oscale) v *= a.oscale[(int64_t)b * a.Co + n];          // Conv3DMod demodulation (M:741-742)
      v += a.bias ? a.bias[n] : 0.f;
      v = apply_act(v, a.act);
      int64_t off;
      if (a.shuffle == MV2_SHUFFLE_SPACE) {
        const int cy = a.Co >> 2, c = n >> 2, p1 = (n >> 1) & 1, p2 = n & 1;
        off = ((((int64_t)b * a.To + to) * (2 * a.Ho) + (2 * ho + p1)) * (2 * a.Wo) + (2 * wo + p2)) * cy + c;
      } else if (a.shuffle == MV2_SHUFFLE_TIME) {
        const int cy = a.Co >> 1, c = n >> 1, p = n & 1;
        off = ((((int64_t)b * (2 * a.To) + (2 * to + p)) * a.Ho + ho) * a.Wo + wo) * cy + c;
      } else {
        off = m * a.Co + n;
      }
      if (res) v += to_f32<T>(res[off]);
      y[off] = from_f32<T>(v);
    }
  }
}

// ------------------------------------------------------------------------------------------
// SqueezeExcite
// ------------------------------------------------------------------------------------------
constexpr int SE_CHUNK = 128;     // rows per block of the generic kernel
constexpr int SE_MIN_ROWS = 32;   // smallest chunk the single-pass bf16 kernel may use (sizes the workspace)

template <typename T>
__global__ void __launch_bounds__(256) se_pool_kernel(const T* __restrict__ y, int P, int C,
                                                      const float* __restrict__ wk, float bk,
                                                      float* __restrict__ ws, int n_chunks) {
  pdl_wait();
  pdl_launch_dependents();
  __shared__ float e[SE_CHUNK];
  __shared__ float red[8];
  __shared__ float bcast[2];
  const int f = blockIdx.y, chunk = blockIdx.x;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int p0 = chunk * SE_CHUNK;
  const T* yf = y + (int64_t)f * P * C;
  for (int n = warp; n < SE_CHUNK; n += 8) {
    const int p = p0 + n;
    float s = 0.f;
    if (p < P) {
      const T* row = yf + (int64_t)p * C;
      for (int c = lane; c < C; c += 32) s = fmaf(to_f32<T>(row[c]), wk[c], s);
    }
    s = warp_sum(s);
    if (lane == 0) e[n] = (p < P) ? s + bk : -INFINITY;
  }
  __syncthreads();
  float v = (tid < SE_CHUNK) ? e[tid] : -INFINITY;
  float mx = warp_max(v);
  if (lane == 0) red[warp] = mx;
  __syncthreads();
  if (tid == 0) {
    float m = red[0];
    for (int i = 1; i < 8; ++i) m = fmaxf(m, red[i]);
    bcast[0] = m;
  }
  __syncthreads();
  const float m = bcast[0];
  float ev = (tid < SE_CHUNK && v > -INFINITY) ? expf(v - m) : 0.f;
  __syncthreads();
  if (tid < SE_CHUNK) e[tid] = ev;
  float sm = warp_sum(ev);
  if (lane == 0) red[warp] = sm;
  __syncthreads();
  float* out = ws + ((int64_t)f * n_chunks + chunk) * (C + 2);
  if (tid == 0) {
    float s = 0.f;
    for (int i = 0; i < 8; ++i) s += red[i];
    out[0] = m;
    out[1] = s;
  }
  const int cnt = min(SE_CHUNK, P - p0);
  for (int c = tid; c < C; c += 256) {
    float acc = 0.f;
    for (int n = 0; n < cnt; ++n) acc = fmaf(e[n], to_f32<T>(yf[(int64_t)(p0 + n) * C + c]), acc);
    out[2 + c] = acc;
  }
}

// bf16 single-pass variant of se_pool_kernel (online softmax): a row's C channels are spread over G = C / VEC lanes
// (VEC = 8, 16 or 32 bf16 per lane, G <= 32 a power of two), 256 / G row groups per block walk the chunk's rows once:
//   logit (lane-group shuffle reduce) -> running max / rescale -> acc[c] += exp(l - m) * y[c].
// The row groups' partial (m, s, acc) are merged through shared memory and one (m, s, pooled[C]) record per chunk is
// written, same workspace format as se_pool_kernel.
// exp for the online softmax: bare MUFU.EX2 (flush-to-zero; arguments are <= 0, and exp(-inf) = 0 as required)
__device__ __forceinline__ float se_exp(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x * 1.4426950408889634f));
  return y;
}

// The chunk is streamed through shared memory by the bulk-copy engine (cp.async.bulk, one batch of R * U rows per ring
// stage, SE_STAGES stages): loads run ahead of the arithmetic independently of how many registers / warps the SM
// has left, which is what bounded the direct-load version to ~3.5 TB/s.
constexpr int SE_STAGES = 3;
__device__ __forceinline__ void se_mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void se_mbar_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void se_mbar_wait(uint32_t bar, uint32_t parity) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "WAIT_%=:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
      "@p bra DONE_%=;\n"
      "bra WAIT_%=;\n"
      "DONE_%=:\n"
      "}\n" ::"r"(bar), "r"(parity) : "memory");
}
__device__ __forceinline__ void se_bulk_load(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
               ::"r"(dst), "l"(src), "r"(bytes), "r"(bar) : "memory");
}

template <typename T, int VEC, int G>   // G = C / VEC lanes per row (compile time: the shuffle reductions unroll)
__global__ void __launch_bounds__(256) se_pool_online_kernel(const T* __restrict__ y, int P, int C,
                                                             const float* __restrict__ wk, float bk,
                                                             float* __restrict__ ws, int n_chunks, int chunk_rows) {
  extern __shared__ __align__(128) float dyn[];   // ring of SE_STAGES batches; reused as [R][C + 2] + [R] for the merge
  __shared__ __align__(8) uint64_t full_bar[SE_STAGES];
  const int f = blockIdx.y, chunk = blockIdx.x;
  const int tid = threadIdx.x;
  constexpr int R = 256 / G;
  const int g = tid % G, rsub = tid / G;
  const int p0 = chunk * chunk_rows;
  const int cnt = min(chunk_rows, P - p0);
  constexpr int U = (VEC == 8) ? 4 : 2;
  const int batch_rows = R * U;
  const uint32_t stage_bytes = (uint32_t)batch_rows * C * 2;
  const int n_batches = (cnt + batch_rows - 1) / batch_rows;
  const uint32_t ring = (uint32_t)__cvta_generic_to_shared(dyn);
  const uint32_t bar0 = (uint32_t)__cvta_generic_to_shared(full_bar);
  const T* ychunk = y + ((int64_t)f * P + p0) * C;
  if (tid == 0) {
    for (int s_ = 0; s_ < SE_STAGES; ++s_) se_mbar_init(bar0 + 8 * s_, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  pdl_wait();
  pdl_launch_dependents();
  auto issue = [&](int bi) {     // thread 0 only
    const int st_ = bi % SE_STAGES;
    const int rows = min(batch_rows, cnt - bi * batch_rows);
    const uint32_t bytes = (uint32_t)rows * C * 2;
    se_mbar_expect_tx(bar0 + 8 * st_, bytes);
    se_bulk_load(ring + st_ * stage_bytes, ychunk + (int64_t)bi * batch_rows * C, bytes, bar0 + 8 * st_);
  };
  if (tid == 0)
    for (int bi = 0; bi < SE_STAGES && bi < n_batches; ++bi) issue(bi);
  float wv[VEC], acc[VEC];
#pragma unroll
  for (int q = 0; q < VEC; ++q) { wv[q] = wk[g * VEC + q]; acc[q] = 0.f; }
  float m = -INFINITY, ssum = 0.f;
  for (int bi = 0; bi < n_batches; ++bi) {
    const int st_ = bi % SE_STAGES;
    const int nb = bi * batch_rows;
    se_mbar_wait(bar0 + 8 * st_, (uint32_t)(bi / SE_STAGES) & 1u);
    const unsigned char* sbase = reinterpret_cast<const unsigned char*>(dyn) + (size_t)st_ * stage_bytes + (size_t)g * VEC * 2;
    uint4 raw[U][VEC / 8];
    bool ok[U];
#pragma unroll
    for (int uu = 0; uu < U; ++uu) {
      const int rr = uu * R + rsub;                 // row inside the batch
      ok[uu] = nb + rr < cnt;
      const uint4* src = reinterpret_cast<const uint4*>(sbase + (size_t)rr * C * 2);
#pragma unroll
      for (int u = 0; u < VEC / 8; ++u) raw[uu][u] = ok[uu] ? src[u] : make_uint4(0, 0, 0, 0);
    }
    // every thread has its rows in registers: the stage can be refilled.  The refill is an async-proxy write, so the
    // generic-proxy reads above must be ordered before it explicitly; without the fence the bulk copy may overwrite rows
    // that have not been read yet.
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    __syncthreads();
    if (tid == 0 && bi + SE_STAGES < n_batches) issue(bi + SE_STAGES);
    // the U rows are folded in together: one running-max update, one rescale of the accumulators and U + 1 exponentials
    // per batch (the row-at-a-time recurrence serialised 2 exponentials and a full rescale per row)
    float v[U][VEC], l[U];
#pragma unroll
    for (int uu = 0; uu < U; ++uu) {
      float dot = 0.f;
#pragma unroll
      for (int u = 0; u < VEC / 8; ++u) {
        const pair_t<T>* vb = reinterpret_cast<const pair_t<T>*>(&raw[uu][u]);
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          const float2 fv = pair_to_f2(vb[q]);
          v[uu][u * 8 + 2 * q] = fv.x;
          v[uu][u * 8 + 2 * q + 1] = fv.y;
        }
      }
#pragma unroll
      for (int q = 0; q < VEC; ++q) dot = fmaf(v[uu][q], wv[q], dot);
#pragma unroll
      for (int o = G >> 1; o > 0; o >>= 1) dot += __shfl_xor_sync(0xffffffffu, dot, o);
      l[uu] = ok[uu] ? dot + bk : -INFINITY;
    }
    float mn = m;
#pragma unroll
    for (int uu = 0; uu < U; ++uu) mn = fmaxf(mn, l[uu]);
    if (mn > -INFINITY) {
      const float sc = se_exp(m - mn);
      float e[U], es = 0.f;
#pragma unroll
      for (int uu = 0; uu < U; ++uu) { e[uu] = se_exp(l[uu] - mn); es += e[uu]; }
      ssum = fmaf(ssum, sc, es);
#pragma unroll
      for (int q = 0; q < VEC; ++q) {
        float t = acc[q] * sc;
#pragma unroll
        for (int uu = 0; uu < U; ++uu) t = fmaf(e[uu], v[uu][q], t);
        acc[q] = t;
      }
      m = mn;
    }
  }
  float* mine = dyn + (size_t)rsub * (C + 2);
  if (g == 0) { mine[0] = m; mine[1] = ssum; }
#pragma unroll
  for (int q = 0; q < VEC; ++q) mine[2 + g * VEC + q] = acc[q];
  __syncthreads();
  // merge the R row groups: warp 0 turns the group maxima into coefficients, then every thread sums its channels
  float* coefs = dyn + (size_t)R * (C + 2);   // [R]
  float* out = ws + ((int64_t)f * n_chunks + chunk) * (C + 2);
  if (tid < 32) {   // R may exceed 32 (narrow layers: C = 16 -> 128 row groups)
    float mx = -INFINITY;
    for (int r = tid; r < R; r += 32) mx = fmaxf(mx, dyn[(size_t)r * (C + 2)]);
    const float M = warp_max(mx);
    float sp = 0.f;
    for (int r = tid; r < R; r += 32) {
      const float mr = dyn[(size_t)r * (C + 2)];
      const float cf = mr > -INFINITY ? __expf(mr - M) : 0.f;
      coefs[r] = cf;
      sp = fmaf(cf, dyn[(size_t)r * (C + 2) + 1], sp);
    }
    const float S = warp_sum(sp);
    if (tid == 0) { out[0] = M; out[1] = S; }
  }
  __syncthreads();
  for (int c = tid; c < C; c += 256) {
    float t = 0.f;
    for (int r = 0; r < R; ++r) t = fmaf(dyn[(size_t)r * (C + 2) + 2 + c], coefs[r], t);
    out[2 + c] = t;
  }
}

// NARROW (C <= 128, a power of two): 256 / C thread groups each fold a strided subset of the chunk records (the fused
// ResidualUnit kernel writes ~100 small records per frame), then the groups are summed through shared memory.
template <bool NARROW>
__global__ void __launch_bounds__(256) se_hidden_kernel(const float* __restrict__ ws, int n_chunks, int C, int Hd,
                                                        const float* __restrict__ w1, const float* __restrict__ b1,
                                                        float* __restrict__ hidden_out) {
  pdl_wait();
  pdl_launch_dependents();
  // grid (F, ceil(Hd / 32)): combine the chunk partials into pooled[C] (redundantly per block: cheap), then 32 hidden units.
  extern __shared__ float sm[];
  float* pooled = sm;          // [C]
  float* coef = sm + C;        // [n_chunks]
  __shared__ float s_inv;
  const int f = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const float* wf = ws + (int64_t)f * n_chunks * (C + 2);
  if (warp == 0) {
    float m = -INFINITY;
    for (int k = lane; k < n_chunks; k += 32) m = fmaxf(m, wf[(int64_t)k * (C + 2)]);
    m = warp_max(m);
    float s = 0.f;
    for (int k = lane; k < n_chunks; k += 32) {
      float cf = expf(wf[(int64_t)k * (C + 2)] - m);
      coef[k] = cf;
      s += cf * wf[(int64_t)k * (C + 2) + 1];
    }
    s = warp_sum(s);
    if (lane == 0) s_inv = 1.f / s;
  }
  __syncthreads();
  if (NARROW) {
    float* part = sm + C + n_chunks;                  // [256]
    const int nparts = 256 / C, c = tid & (C - 1), pi = tid / C;
    float acc = 0.f;
    for (int k = pi; k < n_chunks; k += nparts) acc = fmaf(coef[k], wf[(int64_t)k * (C + 2) + 2 + c], acc);
    part[tid] = acc;
    __syncthreads();
    if (tid < C) {
      float t = 0.f;
      for (int q = 0; q < nparts; ++q) t += part[q * C + tid];
      pooled[tid] = t * s_inv;
    }
  } else {
    for (int c = tid; c < C; c += 256) {
      float acc = 0.f;
      for (int k = 0; k < n_chunks; ++k) acc = fmaf(coef[k], wf[(int64_t)k * (C + 2) + 2 + c], acc);
      pooled[c] = acc * s_inv;
    }
  }
  __syncthreads();
  const int j0 = blockIdx.y * 32 + warp * 4;
  float acc[4] = {0.f, 0.f, 0.f, 0.f};
  for (int c = lane; c < C; c += 32) {
    const float pv = pooled[c];
#pragma unroll
    for (int u = 0; u < 4; ++u)
      if (j0 + u < Hd) acc[u] = fmaf(w1[(int64_t)(j0 + u) * C + c], pv, acc[u]);
  }
#pragma unroll
  for (int u = 0; u < 4; ++u) {
    const float a = warp_sum(acc[u]);
    if (lane == 0 && j0 + u < Hd) {
      const float h = a + b1[j0 + u];
      hidden_out[(int64_t)f * Hd + j0 + u] = h > 0.f ? h : 0.1f * h;
    }
  }
}

__global__ void __launch_bounds__(256) se_out_kernel(const float* __restrict__ hidden, int C, int Hd,
                                                     const float* __restrict__ w2, const float* __restrict__ b2,
                                                     float* __restrict__ gates) {
  pdl_wait();
  pdl_launch_dependents();
  // grid (F, ceil(C / 64)): 8 warps x 8 output channels each
  extern __shared__ float sm[];   // hidden[Hd]
  const int f = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  for (int j = tid; j < Hd; j += 256) sm[j] = hidden[(int64_t)f * Hd + j];
  __syncthreads();
  const int c0 = blockIdx.y * 64 + warp * 8;
  float acc[8];
#pragma unroll
  for (int u = 0; u < 8; ++u) acc[u] = 0.f;
  // unrolled so that the weight loads of 8 steps are in flight together: the kernel is a chain of load latencies
#pragma unroll 8
  for (int j = lane; j < Hd; j += 32) {
    const float hv = sm[j];
#pragma unroll
    for (int u = 0; u < 8; ++u)
      if (c0 + u < C) acc[u] = fmaf(w2[(int64_t)(c0 + u) * Hd + j], hv, acc[u]);
  }
#pragma unroll
  for (int u = 0; u < 8; ++u) {
    const float a = warp_sum(acc[u]);
    if (lane == 0 && c0 + u < C) gates[(int64_t)f * C + c0 + u] = 1.f / (1.f + expf(-(a + b2[c0 + u])));
  }
}

template <typename T>
__global__ void gate_residual_kernel(const T* __restrict__ y, const T* __restrict__ x,
                                     const float* __restrict__ gates, T* __restrict__ out,
                                     int64_t total, int64_t PC, int C) {
  pdl_wait();
  pdl_launch_dependents();
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t f = i / PC;
    const int c = (int)(i % C);
    out[i] = from_f32<T>(fmaf(gates[f * C + c], to_f32<T>(y[i]), to_f32<T>(x[i])));
  }
}

// 8 bf16 per thread (16-byte accesses); requires C % 8 == 0
template <typename T>
__global__ void gate_residual_x8_kernel(const uint4* __restrict__ y, const uint4* __restrict__ x,
                                            const float* __restrict__ gates, uint4* __restrict__ out,
                                            int64_t total8, int64_t PC8, int C8) {
  pdl_wait();
  pdl_launch_dependents();
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total8; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t f = i / PC8;
    const int c = (int)(i % C8) * 8;
    const uint4 yv = y[i], xv = x[i];
    const float4 g0 = *reinterpret_cast<const float4*>(gates + f * (C8 * 8) + c);
    const float4 g1 = *reinterpret_cast<const float4*>(gates + f * (C8 * 8) + c + 4);
    const pair_t<T>* yb = reinterpret_cast<const pair_t<T>*>(&yv);
    const pair_t<T>* xb = reinterpret_cast<const pair_t<T>*>(&xv);
    const float gg[8] = {g0.x, g0.y, g0.z, g0.w, g1.x, g1.y, g1.z, g1.w};
    uint4 o;
    uint32_t* ob = reinterpret_cast<uint32_t*>(&o);
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const float2 yf = pair_to_f2(yb[q]), xf = pair_to_f2(xb[q]);
      pair_t<T> r = f2_to_pair<T>(fmaf(gg[2 * q], yf.x, xf.x), fmaf(gg[2 * q + 1], yf.y, xf.y));
      ob[q] = *reinterpret_cast<uint32_t*>(&r);
    }
    out[i] = o;
  }
}


// ------------------------------------------------------------------------------------------
// conditioning helpers (cond_residual; reference M:680-753, M:946-988, M:1344-1352)
// ------------------------------------------------------------------------------------------
// y[b][n] = act(sum_k x[b][k] w[n][k] + bias[n]); one warp per output, grid (ceil(N / 8), B)
__global__ void __launch_bounds__(256) dense_small_kernel(const float* __restrict__ x, const float* __restrict__ w,
                                                          const float* __restrict__ bias, float* __restrict__ y, int K, int N, int act) {
  pdl_wait();
  pdl_launch_dependents();
  const int b = blockIdx.y, n = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (n >= N) return;
  float acc = 0.f;
  for (int k = lane; k < K; k += 32) acc = fmaf(x[(int64_t)b * K + k], w[(int64_t)n * K + k], acc);
  acc = warp_sum(acc);
  if (lane == 0) y[(int64_t)b * N + n] = apply_act(acc + (bias ? bias[n] : 0.f), act);
}

// scale_in[b][i] = cond[b][i] + 1;  inv_norm[b][o] = rsqrt(max(sum_i (cond[b][i] + 1)^2 S[o][i], eps))
__global__ void __launch_bounds__(256) mod_prepare_kernel(const float* __restrict__ cond, const float* __restrict__ S, float eps,
                                                          float* __restrict__ scale_in, float* __restrict__ inv_norm, int Ci, int Co) {
  pdl_wait();
  pdl_launch_dependents();
  const int b = blockIdx.y, lane = threadIdx.x & 31;
  if (blockIdx.x == 0)
    for (int i = threadIdx.x; i < Ci; i += 256) scale_in[(int64_t)b * Ci + i] = cond[(int64_t)b * Ci + i] + 1.f;
  const int o = blockIdx.x * 8 + (threadIdx.x >> 5);
  if (o >= Co) return;
  float acc = 0.f;
  for (int i = lane; i < Ci; i += 32) {
    const float m = cond[(int64_t)b * Ci + i] + 1.f;
    acc = fmaf(m * m, S[(int64_t)o * Ci + i], acc);
  }
  acc = warp_sum(acc);
  if (lane == 0) inv_norm[(int64_t)b * Co + o] = rsqrtf(fmaxf(acc, eps));
}

template <typename T>
__global__ void scale_channels_kernel(const T* __restrict__ x, const float* __restrict__ scale, T* __restrict__ out,
                                      int64_t total, int64_t per_clip, int C) {
  pdl_wait();
  pdl_launch_dependents();
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t b = i / per_clip;
    const int c = (int)(i % C);
    out[i] = from_f32<T>(to_f32<T>(x[i]) * scale[b * C + c]);
  }
}

// ------------------------------------------------------------------------------------------
// explicit padding for CausalConv3d with pad_mode != 'constant' (M:925-927: F.pad(x, (pw, pw, ph, ph, kt-1, 0), mode))
// dst (B, T + pt, H + 2 ph, W + 2 pw, C) <- src (B, T, H, W, C), channels-last; mode 1 reflect, 2 replicate, 3 circular
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ int pad_src_index(int i, int n, int mode) {
  if (i >= 0 && i < n) return i;
  if (mode == 1) { if (i < 0) i = -i; if (i >= n) i = 2 * (n - 1) - i; return i; }      // reflect (no edge repeat)
  if (mode == 2) return i < 0 ? 0 : n - 1;                                             // replicate
  i %= n;                                                                               // circular
  return i < 0 ? i + n : i;
}
template <typename T>
__global__ void pad_cl_kernel(const T* __restrict__ src, T* __restrict__ dst, int B, int Tn, int H, int W, int C, int pt, int ph,
                              int pw, int mode) {
  pdl_wait();
  pdl_launch_dependents();
  const int To = Tn + pt, Ho = H + 2 * ph, Wo = W + 2 * pw;
  const int64_t total = (int64_t)B * To * Ho * Wo * C;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    int64_t r = i;
    const int c = (int)(r % C); r /= C;
    const int w = (int)(r % Wo); r /= Wo;
    const int h = (int)(r % Ho); r /= Ho;
    const int t = (int)(r % To); r /= To;
    const int b = (int)r;
    const int ts = pad_src_index(t - pt, Tn, mode), hs = pad_src_index(h - ph, H, mode), ws = pad_src_index(w - pw, W, mode);
    dst[i] = src[((((int64_t)b * Tn + ts) * H + hs) * W + ws) * C + c];
  }
}

// ------------------------------------------------------------------------------------------
// RMSNorm (+ token shift addressing)
// ------------------------------------------------------------------------------------------
template <typename T>
__global__ void __launch_bounds__(256) rmsnorm_kernel(const T* __restrict__ x, T* __restrict__ out,
                                                      const float* __restrict__ gamma, int64_t n_tok, int T_,
                                                      int P, int C, int token_shift, const T* __restrict__ prev,
                                                      int64_t prev_stride) {
  pdl_wait();
  pdl_launch_dependents();
  const int lane = threadIdx.x & 31;
  const int64_t tok = (int64_t)blockIdx.x * 8 + (threadIdx.x >> 5);
  if (tok >= n_tok) return;
  const int t = (int)((tok / P) % T_);
  const int half = (C + 1) >> 1;           // torch.chunk(2): the first (unshifted) half takes ceil(C / 2) channels (M:250)
  const T* row = x + tok * C;
  // frame -1 of a chunk that continues a clip: the previous chunk's last frame (prev), else the zero shift
  const T* prow = t > 0 || !prev ? row - (int64_t)P * C : prev + (tok / ((int64_t)T_ * P)) * prev_stride + (tok % P) * C;
  const bool has_prev = t > 0 || prev;
  float ss = 0.f;
  for (int c = lane; c < C; c += 32) {
    float v;
    if (token_shift && c >= half) v = has_prev ? to_f32<T>(prow[c]) : 0.f;
    else v = to_f32<T>(row[c]);
    ss = fmaf(v, v, ss);
  }
  ss = warp_sum(ss);
  const float denom = fmaxf(sqrtf(ss), 1e-12f);
  const float scale = sqrtf((float)C);
  T* orow = out + tok * C;
  for (int c = lane; c < C; c += 32) {
    float v;
    if (token_shift && c >= half) v = has_prev ? to_f32<T>(prow[c]) : 0.f;
    else v = to_f32<T>(row[c]);
    orow[c] = from_f32<T>(((v / denom) * scale) * gamma[c]);
  }
}


// bf16, C % 8 == 0: one warp per token, 16-byte accesses, the row is held in registers between the two phases
// (C <= 1024: at most 4 uint4 per lane).
// One warp normalises RN_TPW (template) tokens: all of their 16-byte loads are issued before the first reduction (one token per
// warp left a single load in flight per lane and ran at a third of the HBM rate).
template <typename T, int NU, int RN_TPW>   // 256-channel slabs per token: C <= 256 * NU
__global__ void __launch_bounds__(256) rmsnorm_x8_kernel(const T* __restrict__ x, T* __restrict__ out,
                                                             const float* __restrict__ gamma, int64_t n_tok, int T_,
                                                             int P, int C, int token_shift,
                                                             const T* __restrict__ prev, int64_t prev_stride) {
  pdl_wait();
  pdl_launch_dependents();
  const int lane = threadIdx.x & 31;
  const int64_t tok0 = ((int64_t)blockIdx.x * 8 + (threadIdx.x >> 5)) * RN_TPW;
  if (tok0 >= n_tok) return;
  const int half = C >> 1;
  uint4 v[RN_TPW][NU];
#pragma unroll
  for (int i = 0; i < RN_TPW; ++i) {
    const int64_t tok = tok0 + i;
    const bool valid = tok < n_tok;
    const int t = valid ? (int)((tok / P) % T_) : 0;
    const T* row = x + (valid ? tok : tok0) * C;
    const T* prow = t > 0 || !prev ? row - (int64_t)P * C
                                               : prev + ((valid ? tok : tok0) / ((int64_t)T_ * P)) * prev_stride + ((valid ? tok : tok0) % P) * C;
    const bool has_prev = t > 0 || prev;
#pragma unroll
    for (int u = 0; u < NU; ++u) {
      const int c = (u * 32 + lane) * 8;
      v[i][u] = make_uint4(0, 0, 0, 0);
      if (valid && c < C) {
        if (token_shift && c >= half) { if (has_prev) v[i][u] = *reinterpret_cast<const uint4*>(prow + c); }
        else v[i][u] = *reinterpret_cast<const uint4*>(row + c);
      }
    }
  }
  float ss[RN_TPW];
#pragma unroll
  for (int i = 0; i < RN_TPW; ++i) {
    float a = 0.f;
#pragma unroll
    for (int u = 0; u < NU; ++u) {
      const pair_t<T>* vb = reinterpret_cast<const pair_t<T>*>(&v[i][u]);
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const float2 f = pair_to_f2(vb[q]);
        a = fmaf(f.x, f.x, a);
        a = fmaf(f.y, f.y, a);
      }
    }
    ss[i] = a;
  }
#pragma unroll
  for (int i = 0; i < RN_TPW; ++i) ss[i] = warp_sum(ss[i]);
  const float scale = sqrtf((float)C);
#pragma unroll
  for (int u = 0; u < NU; ++u) {
    const int c = (u * 32 + lane) * 8;
    if (c < C) {
      const float4 g0 = *reinterpret_cast<const float4*>(gamma + c), g1 = *reinterpret_cast<const float4*>(gamma + c + 4);
      const float gg[8] = {g0.x, g0.y, g0.z, g0.w, g1.x, g1.y, g1.z, g1.w};
#pragma unroll
      for (int i = 0; i < RN_TPW; ++i) {
        if (tok0 + i < n_tok) {
          const float rinv = 1.f / fmaxf(sqrtf(ss[i]), 1e-12f);   // x / max(|x|, eps) as one reciprocal per token
          const pair_t<T>* vb = reinterpret_cast<const pair_t<T>*>(&v[i][u]);
          uint4 o;
          uint32_t* ob = reinterpret_cast<uint32_t*>(&o);
#pragma unroll
          for (int q = 0; q < 4; ++q) {
            const float2 f = pair_to_f2(vb[q]);
            pair_t<T> r = f2_to_pair<T>(((f.x * rinv) * scale) * gg[2 * q], ((f.y * rinv) * scale) * gg[2 * q + 1]);
            ob[q] = *reinterpret_cast<uint32_t*>(&r);
          }
          *reinterpret_cast<uint4*>(out + (tok0 + i) * C + c) = o;
        }
      }
    }
  }
}

// ------------------------------------------------------------------------------------------
// softmax attention core
// ------------------------------------------------------------------------------------------
// Every softmax kernel body below takes a DROP parameter: DROP = false is the plain kernel; DROP = true drops the softmax
// weights with the Philox mask of common.cuh (attn_keep4).  The denominator sums the undropped weights; only the P.V operand
// is masked, and 1 / (1 - p) is folded into the final 1 / l.
constexpr int AT_Q = 32;  // queries per block
// Rows [q_begin, L) of a call (mv2_attention_tail): a.qkv is then a K/V cache ('(kv h d)' rows of 2 * heads * dim_head), the
// queries are rows 0.. of the chunk's qkv rows q (sequences q_outer tokens apart), and the output rows are stored alike
// (out_outer).  A whole call is {0, -1, nullptr, 0}: queries, keys and values from a.qkv.
struct AttnTail { int q_begin; int64_t out_outer; const void* q; int64_t q_outer; };
template <typename T, int DPL, bool DROP>
__device__ __forceinline__ void attention_body(const mv2_attn_args& a, const AttnDrop& dr, const AttnTail tl = AttnTail{0, -1, nullptr, 0}) {
  pdl_wait();
  pdl_launch_dependents();
  constexpr int D = DPL * 32;
  __shared__ float Qs[AT_Q][D];
  __shared__ float Ks[32][D + 1];
  __shared__ float Vs[32][D + 1];
  const T* __restrict__ qkv = (const T*)a.qkv;
  T* __restrict__ out = (T*)a.out;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int h = blockIdx.y;
  const int64_t seq = blockIdx.x;
  const int64_t so = seq / a.n_inner, sn = seq % a.n_inner;
  const int64_t base = so * a.outer_stride + sn * a.inner_stride;
  const int q0 = tl.q_begin + blockIdx.z * AT_Q;
  const int HD = a.heads * D;
  const int64_t row_stride = 3 * (int64_t)HD;
  const int64_t kv_stride = tl.q ? 2 * (int64_t)HD : row_stride, k_off = tl.q ? 0 : HD;   // K/V cache rows: '(kv h d)'
  const float scale = rsqrtf((float)D);
  const bool causal = a.causal && a.L > 1;
  const int Ltot = a.n_mem + a.L;

  for (int idx = tid; idx < AT_Q * D; idx += 128) {
    const int qi = idx / D, d = idx % D;
    const int i = q0 + qi;
    float v = 0.f;
    if (i < a.L) {
      if (tl.q) v = to_f32<T>(((const T*)tl.q)[(so * tl.q_outer + sn * a.inner_stride + (int64_t)(i - tl.q_begin) * a.tok_stride) * row_stride + h * D + d]);
      else v = to_f32<T>(qkv[(base + (int64_t)i * a.tok_stride) * row_stride + h * D + d]);
    }
    Qs[qi][d] = v;
  }
  float m[8], l[8], o[8][DPL];
#pragma unroll
  for (int r = 0; r < 8; ++r) {
    m[r] = -INFINITY;
    l[r] = 0.f;
#pragma unroll
    for (int dd = 0; dd < DPL; ++dd) o[r][dd] = 0.f;
  }
  // keys visible to the last query of this block bound the tile loop under causal masking
  int last_key = Ltot;
  if (causal) last_key = min(Ltot, min(q0 + AT_Q, a.L) + a.n_mem);
  for (int j0 = 0; j0 < last_key; j0 += 32) {
    __syncthreads();
    for (int idx = tid; idx < 32 * D; idx += 128) {
      const int j = idx / D, d = idx % D;
      const int jg = j0 + j;
      float kv = 0.f, vv = 0.f;
      if (jg < a.n_mem) {
        kv = a.mem_kv[(((int64_t)0 * a.heads + h) * a.n_mem + jg) * D + d];
        vv = a.mem_kv[(((int64_t)1 * a.heads + h) * a.n_mem + jg) * D + d];
      } else if (jg < Ltot) {
        const int64_t tokrow = (base + (int64_t)(jg - a.n_mem) * a.tok_stride) * kv_stride + k_off;
        kv = to_f32<T>(qkv[tokrow + h * D + d]);
        vv = to_f32<T>(qkv[tokrow + HD + h * D + d]);
      }
      Ks[j][d] = kv;
      Vs[j][d] = vv;
    }
    __syncthreads();
    const int jg = j0 + lane;
#pragma unroll
    for (int r = 0; r < 8; ++r) {
      const int qi = warp * 8 + r;
      const int i = q0 + qi;
      if (i >= a.L) continue;  // warp-uniform
      float s = 0.f;
#pragma unroll 8
      for (int d = 0; d < D; ++d) s = fmaf(Qs[qi][d], Ks[lane][d], s);
      s *= scale;
      const bool valid = jg < Ltot && (!causal || jg <= i + a.n_mem);
      s = valid ? s : -INFINITY;
      const float m_new = fmaxf(m[r], warp_max(s));
      const float p = valid ? expf(s - m_new) : 0.f;
      const float corr = expf(m[r] - m_new);
      l[r] = l[r] * corr + warp_sum(p);
      m[r] = m_new;
#pragma unroll
      for (int dd = 0; dd < DPL; ++dd) o[r][dd] *= corr;
      float pv = p;
      if (DROP) pv = (attn_keep4(dr, i, jg >> 2, blockIdx.x, h) >> (jg & 3)) & 1u ? p : 0.f;
      for (int j = 0; j < 32; ++j) {
        const float pj = __shfl_sync(0xffffffffu, pv, j);
#pragma unroll
        for (int dd = 0; dd < DPL; ++dd) o[r][dd] = fmaf(pj, Vs[j][lane + 32 * dd], o[r][dd]);
      }
    }
  }
#pragma unroll
  for (int r = 0; r < 8; ++r) {
    const int i = q0 + warp * 8 + r;
    if (i >= a.L) continue;
    const float inv = DROP ? dr.scale / l[r] : 1.f / l[r];
    const int64_t obase = tl.out_outer < 0 ? base : so * tl.out_outer + sn * a.inner_stride;
    T* orow = out + (obase + (int64_t)(i - tl.q_begin) * a.tok_stride) * HD + h * D;
#pragma unroll
    for (int dd = 0; dd < DPL; ++dd) orow[lane + 32 * dd] = from_f32<T>(o[r][dd] * inv);
  }
}
template <typename T, int DPL>
__global__ void __launch_bounds__(128) attention_kernel(const mv2_attn_args a) { attention_body<T, DPL, false>(a, AttnDrop{}); }
template <typename T, int DPL>
__global__ void __launch_bounds__(128) attention_tail_kernel(const mv2_attn_args a, const AttnTail tl) {
  attention_body<T, DPL, false>(a, AttnDrop{}, tl);
}
template <typename T, int DPL>
__global__ void __launch_bounds__(128) attention_dropout_kernel(const mv2_attn_args a, const AttnDrop d) {
  attention_body<T, DPL, true>(a, d);
}

// ------------------------------------------------------------------------------------------
// softmax attention core for SHORT sequences (time attention: L = T' = 5 tokens + 4 memory key/values per pixel, M:456-464):
// one warp per (sequence, head), lane = head dimension; the whole (L x (n_mem + L)) score matrix lives in registers.  The
// general kernel above spends a 128-thread block with 32 query slots and two shared-memory key tiles on 5 queries.
// bf16 only (the fp32 path keeps the general kernel and its summation order).
// ------------------------------------------------------------------------------------------
constexpr int AS_L = 8, AS_M = 8;      // max tokens / memory slots
template <typename T, int DPL, bool DROP>
__device__ __forceinline__ void attention_small_body(const mv2_attn_args& a, const AttnDrop& dr, const AttnTail tl = AttnTail{0, -1, nullptr, 0}) {
  pdl_wait();
  pdl_launch_dependents();
  constexpr int D = DPL * 32;
  const T* __restrict__ qkv = (const T*)a.qkv;
  T* __restrict__ out = (T*)a.out;
  const int lane = threadIdx.x & 31;
  const int64_t wid = (int64_t)blockIdx.x * 8 + (threadIdx.x >> 5);       // (sequence, head)
  const int64_t n_seq = (int64_t)a.n_outer * a.n_inner;
  if (wid >= n_seq * a.heads) return;
  const int h = (int)(wid % a.heads);
  const int64_t seq = wid / a.heads;
  const int64_t base = (seq / a.n_inner) * a.outer_stride + (seq % a.n_inner) * a.inner_stride;
  const int HD = a.heads * D;
  const int64_t row_stride = 3 * (int64_t)HD;
  const float scale = rsqrtf((float)D);
  const bool causal = a.causal && a.L > 1;
  const int L = a.L, NM = a.n_mem;
  float q[AS_L][DPL], k[AS_M + AS_L][DPL], v[AS_M + AS_L][DPL];
#pragma unroll
  for (int j = 0; j < AS_M; ++j)
#pragma unroll
    for (int dd = 0; dd < DPL; ++dd) {
      const int d = lane + 32 * dd;
      k[j][dd] = j < NM ? a.mem_kv[(((int64_t)0 * a.heads + h) * NM + j) * D + d] : 0.f;
      v[j][dd] = j < NM ? a.mem_kv[(((int64_t)1 * a.heads + h) * NM + j) * D + d] : 0.f;
    }
#pragma unroll
  for (int i = 0; i < AS_L; ++i)
#pragma unroll
    for (int dd = 0; dd < DPL; ++dd) {
      const int d = lane + 32 * dd;
      float qv = 0.f, kv = 0.f, vv = 0.f;
      if (i < L && tl.q) {        // K/V cache rows '(kv h d)'; the queries of rows >= q_begin from the chunk
        const int64_t row = (base + (int64_t)i * a.tok_stride) * (2 * (int64_t)HD) + h * D + d;
        kv = to_f32(qkv[row]); vv = to_f32(qkv[row + HD]);
        if (i >= tl.q_begin)
          qv = to_f32(((const T*)tl.q)[((seq / a.n_inner) * tl.q_outer + (seq % a.n_inner) * a.inner_stride +
                                                            (int64_t)(i - tl.q_begin) * a.tok_stride) * row_stride + h * D + d]);
      } else if (i < L) {
        const int64_t row = (base + (int64_t)i * a.tok_stride) * row_stride + h * D + d;
        qv = to_f32(qkv[row]); kv = to_f32(qkv[row + HD]); vv = to_f32(qkv[row + 2 * HD]);
      }
      q[i][dd] = qv; k[AS_M + i][dd] = kv; v[AS_M + i][dd] = vv;
    }
  // dropout: NM + L <= 16 keys are 4 Philox groups per query, so lane 4 i + grp draws group grp of query i once; the quad's
  // OR leaves query i's 16 keep bits (bit = key index, memory first) in lanes 4 i .. 4 i + 3
  uint32_t keep = 0;
  if (DROP) {
    keep = attn_keep4(dr, lane >> 2, lane & 3, (uint32_t)seq, h) << (4 * (lane & 3));
    keep |= __shfl_xor_sync(0xffffffffu, keep, 1);
    keep |= __shfl_xor_sync(0xffffffffu, keep, 2);
  }
#pragma unroll
  for (int i = 0; i < AS_L; ++i) {
    if (i >= L) break;
    if (i < tl.q_begin) continue;
    const uint32_t keep_i = DROP ? __shfl_sync(0xffffffffu, keep, 4 * i) : 0u;
    float sc[AS_M + AS_L], mx = -INFINITY;
#pragma unroll
    for (int j = 0; j < AS_M + AS_L; ++j) {
      const int jk = j - AS_M;                               // key index among the tokens (memory slots: j < AS_M)
      const bool valid = j < AS_M ? j < NM : (jk < L && (!causal || jk <= i));
      float p = 0.f;
#pragma unroll
      for (int dd = 0; dd < DPL; ++dd) p = fmaf(q[i][dd], k[j][dd], p);
      p = warp_sum(p) * scale;
      sc[j] = valid ? p : -INFINITY;
      mx = fmaxf(mx, sc[j]);
    }
    float den = 0.f, o[DPL];
#pragma unroll
    for (int dd = 0; dd < DPL; ++dd) o[dd] = 0.f;
#pragma unroll
    for (int j = 0; j < AS_M + AS_L; ++j) {
      const float e = sc[j] > -INFINITY ? __expf(sc[j] - mx) : 0.f;
      den += e;
      float ev = e;
      if (DROP) ev = (keep_i >> (j < AS_M ? j : NM + j - AS_M)) & 1u ? e : 0.f;
#pragma unroll
      for (int dd = 0; dd < DPL; ++dd) o[dd] = fmaf(ev, v[j][dd], o[dd]);
    }
    const float inv = DROP ? dr.scale / den : 1.f / den;
    const int64_t obase = tl.out_outer < 0 ? base : (seq / a.n_inner) * tl.out_outer + (seq % a.n_inner) * a.inner_stride;
    T* orow = out + (obase + (int64_t)(i - tl.q_begin) * a.tok_stride) * HD + h * D;
#pragma unroll
    for (int dd = 0; dd < DPL; ++dd) orow[lane + 32 * dd] = from_f32<T>(o[dd] * inv);
  }
}
// bf16 kernels keep their names; the fp16 ones are the _f16_ twins of the same bodies (AttnK16<T> picks one)
template <int DPL>
__global__ void __launch_bounds__(256) attention_small_kernel(const mv2_attn_args a) { attention_small_body<__nv_bfloat16, DPL, false>(a, AttnDrop{}); }
template <int DPL>
__global__ void __launch_bounds__(256) attention_small_tail_kernel(const mv2_attn_args a, const AttnTail tl) {
  attention_small_body<__nv_bfloat16, DPL, false>(a, AttnDrop{}, tl);
}
template <int DPL>
__global__ void __launch_bounds__(256) attention_small_dropout_kernel(const mv2_attn_args a, const AttnDrop d) {
  attention_small_body<__nv_bfloat16, DPL, true>(a, d);
}
template <int DPL>
__global__ void __launch_bounds__(256) attention_small_f16_kernel(const mv2_attn_args a) { attention_small_body<__half, DPL, false>(a, AttnDrop{}); }
template <int DPL>
__global__ void __launch_bounds__(256) attention_small_tail_f16_kernel(const mv2_attn_args a, const AttnTail tl) {
  attention_small_body<__half, DPL, false>(a, AttnDrop{}, tl);
}
template <int DPL>
__global__ void __launch_bounds__(256) attention_small_dropout_f16_kernel(const mv2_attn_args a, const AttnDrop d) {
  attention_small_body<__half, DPL, true>(a, d);
}


// ------------------------------------------------------------------------------------------
// softmax attention core on tensor cores (warp-level mma.sync m16n8k16, bf16 in / fp32 accumulate):
// flash-style, non-causal, memory key/values prepended, sequences addressed through strides.
// 8 warps x 16 queries per block; keys/values staged per 64-key tile (V transposed) in shared memory, loads prefetched one tile ahead;
// online softmax with quad shuffles.  Used for bf16 sequences with L >= 64 (space attention).
// ------------------------------------------------------------------------------------------
constexpr int FA_Q = 128, FA_KT = 64;     // 8 warps x 16 queries per block; keys / values staged 64 at a time

// T = __nv_bfloat16 or __half selects the operand type of the MMA (ldmatrix and the fragment layouts are the same)
template <typename T>
__device__ __forceinline__ void mma_16816(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  if constexpr (std::is_same<T, __half>::value)
    asm volatile(
        "mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
  else
    asm volatile(
        "mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
template <typename T>
__device__ __forceinline__ uint32_t pack2_16(float lo, float hi) {
  pair_t<T> v = f2_to_pair<T>(lo, hi);
  return *reinterpret_cast<uint32_t*>(&v);
}

template <typename T, int D, bool DROP>
__device__ __forceinline__ void attention_mma_body(const mv2_attn_args& a, const AttnDrop& dr) {
  pdl_wait();
  pdl_launch_dependents();
  constexpr int DK = D / 16, DN = D / 8;
  __shared__ __align__(16) T Ks[FA_KT][D + 8];
  __shared__ __align__(16) T Vt[D][FA_KT + 8];
  const T* __restrict__ qkv = (const T*)a.qkv;
  T* __restrict__ out = (T*)a.out;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int g = lane >> 2, t = lane & 3;
  const int h = blockIdx.y;
  const int64_t seq = blockIdx.x;
  const int64_t so = seq / a.n_inner, sn = seq % a.n_inner;
  const int64_t base = so * a.outer_stride + sn * a.inner_stride;
  const int q0 = blockIdx.z * FA_Q + warp * 16;
  const int HD = a.heads * D;
  const int64_t row_stride = 3 * (int64_t)HD;
  const float sc = rsqrtf((float)D) * 1.4426950408889634f;   // softmax scale folded with log2(e)
  const int Ltot = a.n_mem + a.L;

  // Q fragments for rows q0+g and q0+g+8
  uint32_t qa[DK][4];
  {
    const int r0 = q0 + g, r1 = q0 + g + 8;
    const T* p0 = qkv + (base + (int64_t)min(r0, a.L - 1) * a.tok_stride) * row_stride + h * D;
    const T* p1 = qkv + (base + (int64_t)min(r1, a.L - 1) * a.tok_stride) * row_stride + h * D;
#pragma unroll
    for (int k = 0; k < DK; ++k) {
      qa[k][0] = *reinterpret_cast<const uint32_t*>(p0 + k * 16 + t * 2);
      qa[k][1] = *reinterpret_cast<const uint32_t*>(p1 + k * 16 + t * 2);
      qa[k][2] = *reinterpret_cast<const uint32_t*>(p0 + k * 16 + 8 + t * 2);
      qa[k][3] = *reinterpret_cast<const uint32_t*>(p1 + k * 16 + 8 + t * 2);
    }
  }
  float o[DN][4];
#pragma unroll
  for (int i = 0; i < DN; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) o[i][j] = 0.f;
  float m0 = -INFINITY, m1 = -INFINITY, l0 = 0.f, l1 = 0.f;

  // K / V staging is software pipelined: the global loads of tile j0 + 64 are issued before tile j0 is consumed, so their
  // latency hides under the MMAs / softmax of the current tile (each thread owns ITEMS 16-byte pieces of a tile)
  constexpr int ITEMS = FA_KT * (D / 8) / 256;
  uint4 kr[ITEMS], vr[ITEMS];
  auto fetch = [&](int j0) {
#pragma unroll
    for (int it = 0; it < ITEMS; ++it) {
      const int idx = tid + it * 256;
      const int j = idx / (D / 8), c = (idx % (D / 8)) * 8;
      const int jg = j0 + j;
      uint4 kv4 = make_uint4(0, 0, 0, 0), vv4 = make_uint4(0, 0, 0, 0);
      if (jg < a.n_mem) {
        const float* mk = a.mem_kv + (((int64_t)0 * a.heads + h) * a.n_mem + jg) * D + c;
        const float* mv = a.mem_kv + (((int64_t)1 * a.heads + h) * a.n_mem + jg) * D + c;
        kv4.x = pack2_16<T>(mk[0], mk[1]); kv4.y = pack2_16<T>(mk[2], mk[3]);
        kv4.z = pack2_16<T>(mk[4], mk[5]); kv4.w = pack2_16<T>(mk[6], mk[7]);
        vv4.x = pack2_16<T>(mv[0], mv[1]); vv4.y = pack2_16<T>(mv[2], mv[3]);
        vv4.z = pack2_16<T>(mv[4], mv[5]); vv4.w = pack2_16<T>(mv[6], mv[7]);
      } else if (jg < Ltot) {
        const T* row = qkv + (base + (int64_t)(jg - a.n_mem) * a.tok_stride) * row_stride;
        kv4 = *reinterpret_cast<const uint4*>(row + HD + h * D + c);
        vv4 = *reinterpret_cast<const uint4*>(row + 2 * HD + h * D + c);
      }
      kr[it] = kv4;
      vr[it] = vv4;
    }
  };
  fetch(0);
  for (int j0 = 0; j0 < Ltot; j0 += FA_KT) {
    __syncthreads();
    // ---- stage K (row major) and V (transposed) for keys j0 .. j0+63 ----
#pragma unroll
    for (int it = 0; it < ITEMS; ++it) {
      const int idx = tid + it * 256;
      const int j = idx / (D / 8), c = (idx % (D / 8)) * 8;
      *reinterpret_cast<uint4*>(&Ks[j][c]) = kr[it];
      const T* vb = reinterpret_cast<const T*>(&vr[it]);
#pragma unroll
      for (int q = 0; q < 8; ++q) Vt[c + q][j] = vb[q];
    }
    __syncthreads();
    if (j0 + FA_KT < Ltot) fetch(j0 + FA_KT);
    // ---- S = Q K^T (16 x 64 per warp) ----
    float sfr[FA_KT / 8][4];
#pragma unroll
    for (int nt = 0; nt < FA_KT / 8; ++nt) {
#pragma unroll
      for (int j = 0; j < 4; ++j) sfr[nt][j] = 0.f;
#pragma unroll
      for (int k = 0; k < DK; ++k) {
        const uint32_t b0 = *reinterpret_cast<const uint32_t*>(&Ks[nt * 8 + g][k * 16 + t * 2]);
        const uint32_t b1 = *reinterpret_cast<const uint32_t*>(&Ks[nt * 8 + g][k * 16 + 8 + t * 2]);
        mma_16816<T>(sfr[nt], qa[k], b0, b1);
      }
    }
    // ---- online softmax ----
    float tm0 = -INFINITY, tm1 = -INFINITY;
#pragma unroll
    for (int nt = 0; nt < FA_KT / 8; ++nt) {
      const int kcol = j0 + nt * 8 + t * 2;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const bool valid = (kcol + (j & 1)) < Ltot;
        sfr[nt][j] = valid ? sfr[nt][j] * sc : -INFINITY;
      }
      tm0 = fmaxf(tm0, fmaxf(sfr[nt][0], sfr[nt][1]));
      tm1 = fmaxf(tm1, fmaxf(sfr[nt][2], sfr[nt][3]));
    }
    tm0 = fmaxf(tm0, __shfl_xor_sync(0xffffffffu, tm0, 1));
    tm0 = fmaxf(tm0, __shfl_xor_sync(0xffffffffu, tm0, 2));
    tm1 = fmaxf(tm1, __shfl_xor_sync(0xffffffffu, tm1, 1));
    tm1 = fmaxf(tm1, __shfl_xor_sync(0xffffffffu, tm1, 2));
    const float mn0 = fmaxf(m0, tm0), mn1 = fmaxf(m1, tm1);   // finite: every tile holds >= 1 valid key
    const float c0 = exp2f(m0 - mn0), c1 = exp2f(m1 - mn1);
    m0 = mn0; m1 = mn1;
    l0 *= c0; l1 *= c1;
#pragma unroll
    for (int i = 0; i < DN; ++i) { o[i][0] *= c0; o[i][1] *= c0; o[i][2] *= c1; o[i][3] *= c1; }
#pragma unroll
    for (int nt = 0; nt < FA_KT / 8; ++nt) {
      sfr[nt][0] = exp2f(sfr[nt][0] - mn0); sfr[nt][1] = exp2f(sfr[nt][1] - mn0);
      sfr[nt][2] = exp2f(sfr[nt][2] - mn1); sfr[nt][3] = exp2f(sfr[nt][3] - mn1);
      l0 += sfr[nt][0] + sfr[nt][1];
      l1 += sfr[nt][2] + sfr[nt][3];
    }
    if (DROP) {
      // keys j0 + nt*8 + 4*(t>>1) .. +3 are one Philox group, shared by threads t and t^1 for rows q0+g and q0+g+8: the even
      // thread draws row q0+g, the odd one row q0+g+8, and each passes the partner the two keep bits it needs
#pragma unroll
      for (int nt = 0; nt < FA_KT / 8; ++nt) {
        const uint32_t odd = t & 1;
        const uint32_t kb = attn_keep4(dr, q0 + g + 8 * odd, (j0 + nt * 8) / 4 + (t >> 1), blockIdx.x, h);
        const uint32_t other = __shfl_xor_sync(0xffffffffu, odd ? kb & 3u : kb >> 2, 1);
        const uint32_t k0 = odd ? other : kb & 3u, k1 = odd ? kb >> 2 : other;    // row q0+g / q0+g+8: bit c = column 2t + c
        sfr[nt][0] = k0 & 1u ? sfr[nt][0] : 0.f; sfr[nt][1] = k0 & 2u ? sfr[nt][1] : 0.f;
        sfr[nt][2] = k1 & 1u ? sfr[nt][2] : 0.f; sfr[nt][3] = k1 & 2u ? sfr[nt][3] : 0.f;
      }
    }
    // ---- O += P V ----
#pragma unroll
    for (int kk = 0; kk < FA_KT / 16; ++kk) {
      uint32_t pa[4];
      pa[0] = pack2_16<T>(sfr[2 * kk][0], sfr[2 * kk][1]);
      pa[1] = pack2_16<T>(sfr[2 * kk][2], sfr[2 * kk][3]);
      pa[2] = pack2_16<T>(sfr[2 * kk + 1][0], sfr[2 * kk + 1][1]);
      pa[3] = pack2_16<T>(sfr[2 * kk + 1][2], sfr[2 * kk + 1][3]);
#pragma unroll
      for (int dn = 0; dn < DN; ++dn) {
        const uint32_t b0 = *reinterpret_cast<const uint32_t*>(&Vt[dn * 8 + g][kk * 16 + t * 2]);
        const uint32_t b1 = *reinterpret_cast<const uint32_t*>(&Vt[dn * 8 + g][kk * 16 + 8 + t * 2]);
        mma_16816<T>(o[dn], pa, b0, b1);
      }
    }
  }
  l0 += __shfl_xor_sync(0xffffffffu, l0, 1);
  l0 += __shfl_xor_sync(0xffffffffu, l0, 2);
  l1 += __shfl_xor_sync(0xffffffffu, l1, 1);
  l1 += __shfl_xor_sync(0xffffffffu, l1, 2);
  const float i0 = DROP ? dr.scale / l0 : 1.f / l0, i1 = DROP ? dr.scale / l1 : 1.f / l1;
  const int r0 = q0 + g, r1 = q0 + g + 8;
  if (r0 < a.L) {
    T* orow = out + (base + (int64_t)r0 * a.tok_stride) * HD + h * D;
#pragma unroll
    for (int dn = 0; dn < DN; ++dn) *reinterpret_cast<uint32_t*>(orow + dn * 8 + t * 2) = pack2_16<T>(o[dn][0] * i0, o[dn][1] * i0);
  }
  if (r1 < a.L) {
    T* orow = out + (base + (int64_t)r1 * a.tok_stride) * HD + h * D;
#pragma unroll
    for (int dn = 0; dn < DN; ++dn) *reinterpret_cast<uint32_t*>(orow + dn * 8 + t * 2) = pack2_16<T>(o[dn][2] * i1, o[dn][3] * i1);
  }
}
template <int D>
__global__ void __launch_bounds__(256) attention_mma_kernel(const mv2_attn_args a) { attention_mma_body<__nv_bfloat16, D, false>(a, AttnDrop{}); }
template <int D>
__global__ void __launch_bounds__(256) attention_mma_dropout_kernel(const mv2_attn_args a, const AttnDrop d) {
  attention_mma_body<__nv_bfloat16, D, true>(a, d);
}
template <int D>
__global__ void __launch_bounds__(256) attention_mma_f16_kernel(const mv2_attn_args a) { attention_mma_body<__half, D, false>(a, AttnDrop{}); }
template <int D>
__global__ void __launch_bounds__(256) attention_mma_dropout_f16_kernel(const mv2_attn_args a, const AttnDrop d) {
  attention_mma_body<__half, D, true>(a, d);
}

// the kernels of one 16-bit element type
template <typename T> struct AttnK16;
template <> struct AttnK16<__nv_bfloat16> {
  template <int D> static constexpr auto mma() { return attention_mma_kernel<D>; }
  template <int D> static constexpr auto mma_drop() { return attention_mma_dropout_kernel<D>; }
  template <int P> static constexpr auto small() { return attention_small_kernel<P>; }
  template <int P> static constexpr auto small_drop() { return attention_small_dropout_kernel<P>; }
  template <int P> static constexpr auto small_tail() { return attention_small_tail_kernel<P>; }
};
template <> struct AttnK16<__half> {
  template <int D> static constexpr auto mma() { return attention_mma_f16_kernel<D>; }
  template <int D> static constexpr auto mma_drop() { return attention_mma_dropout_f16_kernel<D>; }
  template <int P> static constexpr auto small() { return attention_small_f16_kernel<P>; }
  template <int P> static constexpr auto small_drop() { return attention_small_dropout_f16_kernel<P>; }
  template <int P> static constexpr auto small_tail() { return attention_small_tail_f16_kernel<P>; }
};

// keep mask of mv2_attention_dropout_mask: one thread per (sequence, head, query, 4-key group), keep[seq][h][i][n_mem + L]
__global__ void __launch_bounds__(256) attention_dropout_mask_kernel(int64_t n_groups, int heads, int L, int Ltot, const AttnDrop d,
                                                                     uint8_t* __restrict__ keep) {
  pdl_wait();
  pdl_launch_dependents();
  const int gpr = (Ltot + 3) / 4;                                  // groups per query row
  for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < n_groups; idx += (int64_t)gridDim.x * blockDim.x) {
    const int grp = (int)(idx % gpr);
    const int64_t row = idx / gpr;                                 // (seq * heads + h) * L + i
    const int i = (int)(row % L);
    const int h = (int)((row / L) % heads);
    const uint32_t seq = (uint32_t)(row / ((int64_t)L * heads));
    const uint32_t kb = attn_keep4(d, i, grp, seq, h);
    uint8_t* dst = keep + row * Ltot + 4 * grp;
#pragma unroll
    for (int w = 0; w < 4; ++w)
      if (4 * grp + w < Ltot) dst[w] = (uint8_t)((kb >> w) & 1u);
  }
}

// ------------------------------------------------------------------------------------------
// Taylor-series linear attention core (dim_head = 8, feature dim 1 + 8 + 64 = 73)
// ------------------------------------------------------------------------------------------
constexpr int LA_D = 8, LA_F = 73, LA_ST = LA_F * (LA_D + 1);  // 657 state values per (seq, head)
constexpr int LA_CHUNK = 256;

__device__ __forceinline__ float taylor_feat(const float* v, int f) {
  if (f == 0) return 1.f;
  if (f <= LA_D) return v[f - 1];
  const int ij = f - 1 - LA_D;
  return v[ij >> 3] * v[ij & 7] * 0.70710678118654752440f;
}

template <typename T>
__global__ void __launch_bounds__(256) linattn_reduce_kernel(const T* __restrict__ kv, float* __restrict__ ws,
                                                             int L, int heads, int n_chunks) {
  pdl_wait();
  pdl_launch_dependents();
  // S[f][e] = sum_n phi(k_n)[f] * [v_n, 1][e].  phi is evaluated once per token into shared memory; thread (slice, f)
  // owns the 9 outputs of feature f for every third token: per token it reads phi[n][f] (conflict free) and the 9
  // values [v_n, 1] (warp broadcast) for 9 FMAs.  The three slices are summed through shared memory at the end.
  constexpr int TB = 64, NS = 3;
  __shared__ float phi[TB][LA_F + 1];
  __shared__ __align__(16) float vs[TB][12];
  __shared__ float ks[TB][LA_D];
  __shared__ float part[NS][LA_ST];
  const int chunk = blockIdx.x, h = blockIdx.y;
  const int64_t seq = blockIdx.z;
  const int tid = threadIdx.x;
  const int HD = heads * LA_D;
  const bool worker = tid < NS * LA_F;
  const int slice = tid / LA_F, f = tid % LA_F;
  float acc[LA_D + 1];
#pragma unroll
  for (int e = 0; e <= LA_D; ++e) acc[e] = 0.f;
  const int t_begin = chunk * LA_CHUNK, t_end = min(L, t_begin + LA_CHUNK);
  for (int t0 = t_begin; t0 < t_end; t0 += TB) {
    __syncthreads();
    for (int idx = tid; idx < TB * LA_D; idx += 256) {
      const int n = idx / LA_D, d = idx % LA_D;
      const int t = t0 + n;
      float kk = 0.f, vv = 0.f;
      if (t < t_end) {
        const int64_t row = (seq * L + t) * (2 * (int64_t)HD);
        kk = to_f32<T>(kv[row + h * LA_D + d]);
        vv = to_f32<T>(kv[row + HD + h * LA_D + d]);
      }
      ks[n][d] = kk;
      vs[n][d] = vv;
    }
    for (int n = tid; n < TB; n += 256) vs[n][LA_D] = (t0 + n < t_end) ? 1.f : 0.f;
    __syncthreads();
    for (int idx = tid; idx < TB * LA_F; idx += 256) {
      const int n = idx / LA_F, ff = idx % LA_F;
      phi[n][ff] = (t0 + n < t_end) ? taylor_feat(ks[n], ff) : 0.f;
    }
    __syncthreads();
    if (worker) {
#pragma unroll 4
      for (int n = slice; n < TB; n += NS) {
        const float pf = phi[n][f];
        const float4 v0 = *reinterpret_cast<const float4*>(&vs[n][0]);
        const float4 v1 = *reinterpret_cast<const float4*>(&vs[n][4]);
        const float v8 = vs[n][8];
        acc[0] = fmaf(pf, v0.x, acc[0]); acc[1] = fmaf(pf, v0.y, acc[1]);
        acc[2] = fmaf(pf, v0.z, acc[2]); acc[3] = fmaf(pf, v0.w, acc[3]);
        acc[4] = fmaf(pf, v1.x, acc[4]); acc[5] = fmaf(pf, v1.y, acc[5]);
        acc[6] = fmaf(pf, v1.z, acc[6]); acc[7] = fmaf(pf, v1.w, acc[7]);
        acc[8] = fmaf(pf, v8, acc[8]);
      }
    }
  }
  if (worker) {
#pragma unroll
    for (int e = 0; e <= LA_D; ++e) part[slice][f * (LA_D + 1) + e] = acc[e];
  }
  __syncthreads();
  float* o = ws + ((seq * heads + h) * n_chunks + chunk) * LA_ST;
  for (int idx = tid; idx < LA_ST; idx += 256) o[idx] = part[0][idx] + part[1][idx] + part[2][idx];
}

template <typename T>
__global__ void __launch_bounds__(64) linattn_apply_kernel(const T* __restrict__ q, const float* __restrict__ ws,
                                                           T* __restrict__ out, int L, int heads, int n_chunks) {
  pdl_wait();
  pdl_launch_dependents();
  // block = 64 threads x 4 tokens = one LA_CHUNK of tokens; every state value read from smem feeds 4 tokens
  __shared__ float S[LA_ST];
  const int chunk = blockIdx.x, h = blockIdx.y;
  const int64_t seq = blockIdx.z;
  const int tid = threadIdx.x;
  const int HD = heads * LA_D;
  const float* wsh = ws + (seq * heads + h) * (int64_t)n_chunks * LA_ST;
  for (int idx = tid; idx < LA_ST; idx += 64) {
    float s = 0.f;
    for (int k = 0; k < n_chunks; ++k) s += wsh[(int64_t)k * LA_ST + idx];
    S[idx] = s;
  }
  __syncthreads();
  constexpr int TPT = LA_CHUNK / 64;   // 4 tokens per thread, strided by 64 for coalescing
  float qv[TPT][LA_D], num[TPT][LA_D], den[TPT];
  const float qscale = rsqrtf((float)LA_D);
  bool ok[TPT];
#pragma unroll
  for (int u = 0; u < TPT; ++u) {
    const int t = chunk * LA_CHUNK + u * 64 + tid;
    ok[u] = t < L;
    const int64_t tok = seq * L + (ok[u] ? t : 0);
#pragma unroll
    for (int d = 0; d < LA_D; ++d) {
      qv[u][d] = ok[u] ? to_f32<T>(q[tok * HD + h * LA_D + d]) * qscale : 0.f;
      num[u][d] = 0.f;
    }
    den[u] = 0.f;
  }
  // f = 0 (constant feature)
#pragma unroll
  for (int u = 0; u < TPT; ++u) {
#pragma unroll
    for (int e = 0; e < LA_D; ++e) num[u][e] = S[e];
    den[u] = S[LA_D];
  }
  // linear features
#pragma unroll
  for (int i = 0; i < LA_D; ++i) {
    const float* Sr = S + (1 + i) * (LA_D + 1);
    float sv[LA_D + 1];
#pragma unroll
    for (int e = 0; e <= LA_D; ++e) sv[e] = Sr[e];
#pragma unroll
    for (int u = 0; u < TPT; ++u) {
      const float pf = qv[u][i];
#pragma unroll
      for (int e = 0; e < LA_D; ++e) num[u][e] = fmaf(pf, sv[e], num[u][e]);
      den[u] = fmaf(pf, sv[LA_D], den[u]);
    }
  }
  // quadratic features
#pragma unroll
  for (int i = 0; i < LA_D; ++i)
#pragma unroll
    for (int j = 0; j < LA_D; ++j) {
      const float* Sr = S + (1 + LA_D + i * LA_D + j) * (LA_D + 1);
      float sv[LA_D + 1];
#pragma unroll
      for (int e = 0; e <= LA_D; ++e) sv[e] = Sr[e];
#pragma unroll
      for (int u = 0; u < TPT; ++u) {
        const float pf = qv[u][i] * qv[u][j] * 0.70710678118654752440f;
#pragma unroll
        for (int e = 0; e < LA_D; ++e) num[u][e] = fmaf(pf, sv[e], num[u][e]);
        den[u] = fmaf(pf, sv[LA_D], den[u]);
      }
    }
#pragma unroll
  for (int u = 0; u < TPT; ++u) {
    if (!ok[u]) continue;
    const int64_t tok = seq * L + chunk * LA_CHUNK + u * 64 + tid;
    const float dn = fmaxf(den[u], 1e-5f);
#pragma unroll
    for (int e = 0; e < LA_D; ++e) out[tok * HD + h * LA_D + e] = from_f32<T>(num[u][e] / dn);
  }
}


// ------------------------------------------------------------------------------------------
// Taylor linear attention on tensor cores (bf16 path): both contractions are small GEMMs
//   reduce:  S[f][e]   = sum_n phi_f(k_n) * [v_n, 1][e]        (M = 80 padded features, N = 16, K = tokens)
//   apply :  out[n][e] = sum_f phi_f(q_n) * S[f][e]             (M = tokens, N = 16, K = 80)
// evaluated with warp-level mma.sync m16n8k16 (bf16 operands, fp32 accumulate); the feature map phi is evaluated once
// per token into shared memory by the thread that owns the token (compile-time feature index -> registers only).
// ------------------------------------------------------------------------------------------
constexpr int LAM_F = 80;      // 73 features padded to 5 x 16
constexpr int LAM_TB = 128;    // tokens per staging batch

template <int F_IDX>
__device__ __forceinline__ float taylor_feat_ct(const float (&k)[LA_D]) {
  if (F_IDX == 0) return 1.f;
  if (F_IDX <= LA_D) return k[(F_IDX - 1) & 7];
  if (F_IDX < LA_F) return k[((F_IDX - 1 - LA_D) >> 3) & 7] * k[(F_IDX - 1 - LA_D) & 7] * 0.70710678118654752440f;
  return 0.f;
}
template <int F0, typename Fn>
__device__ __forceinline__ void for_each_feature_pair(const float (&k)[LA_D], Fn&& fn) {
  if constexpr (F0 < LAM_F) {
    fn(F0, taylor_feat_ct<F0>(k), taylor_feat_ct<F0 + 1>(k));
    for_each_feature_pair<F0 + 2>(k, fn);
  }
}

// ldmatrix of four 8x8 b16 tiles, transposed: thread (g = lane / 4, t = lane % 4) receives, from the tile whose 8 row addresses
// lanes 8j .. 8j+7 supplied, the elements [row 2t][col g] and [row 2t+1][col g]
__device__ __forceinline__ void ldmatrix_x4_trans(uint32_t (&r)[4], const void* smem_row) {
  const uint32_t addr = (uint32_t)__cvta_generic_to_shared(smem_row);
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0, %1, %2, %3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(addr));
}

constexpr int LAM_RS = LAM_F + 8;                                            // bf16 elements per token row (176 B: conflict-free)
constexpr size_t LAM_REDUCE_SMEM = (size_t)2 * LAM_TB * LAM_RS * 2 + (size_t)16 * (LAM_TB + 8) * 2;   // phi hi + lo, v^T
constexpr size_t LAM_REDUCE_SMEM_F16 = LAM_REDUCE_SMEM + (size_t)16 * (LAM_TB + 8) * 2;                // + the v^T lo part

// T: element type of kv (bf16 or fp16).  The MMA operands are bf16 in both cases: the values are widened to fp32 at the
// load and split into bf16 hi + lo pairs, so only the loads depend on T.
template <typename T>
__device__ __forceinline__ void linattn_reduce_mma_body(const T* __restrict__ kv, float* __restrict__ ws, int L, int heads,
                                                        int n_chunks) {
  constexpr bool V_LO = std::is_same<T, __half>::value;
  // phi is carried as a bf16 hi + lo pair (two MMAs) so the quadratic features keep ~16 mantissa bits; a bf16 v is exact in
  // bf16, an fp16 v (11 significant bits) is exact as a bf16 hi + lo pair (a third MMA: phi hi x v lo).
  // Token-major staging [token][feature] (one token per thread, 16-byte stores: a 176-byte row pitch puts the 32 rows of a warp
  // in 8 distinct bank groups = the minimal 4 wavefronts per store); the MMA wants A = phi^T [feature][token], which
  // ldmatrix.trans delivers straight from the token-major tile.  (The former feature-major layout needed 160 two-byte stores
  // per token and was bound by shared-memory wavefronts.)
  extern __shared__ __align__(16) unsigned char lam_dyn[];
  __nv_bfloat16 (*phi_s)[LAM_RS] = reinterpret_cast<__nv_bfloat16 (*)[LAM_RS]>(lam_dyn);                                // [token][feature] hi
  __nv_bfloat16 (*phi_l)[LAM_RS] = reinterpret_cast<__nv_bfloat16 (*)[LAM_RS]>(lam_dyn + (size_t)LAM_TB * LAM_RS * 2);  // lo
  __nv_bfloat16 (*vt)[LAM_TB + 8] = reinterpret_cast<__nv_bfloat16 (*)[LAM_TB + 8]>(lam_dyn + (size_t)2 * LAM_TB * LAM_RS * 2);   // [e][token]; e = 8: ones
  __nv_bfloat16 (*vtl)[LAM_TB + 8] = reinterpret_cast<__nv_bfloat16 (*)[LAM_TB + 8]>(lam_dyn + LAM_REDUCE_SMEM);   // V_LO: lo part
  const int chunk = blockIdx.x, h = blockIdx.y;
  const int64_t seq = blockIdx.z;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int g = lane >> 2, t = lane & 3;
  const int HD = heads * LA_D;
  float acc[5][2][4];
#pragma unroll
  for (int a = 0; a < 5; ++a)
#pragma unroll
    for (int b = 0; b < 2; ++b)
#pragma unroll
      for (int c = 0; c < 4; ++c) acc[a][b][c] = 0.f;
#pragma unroll
  for (int e = LA_D + 1; e < 16; ++e) vt[e][tid] = __float2bfloat16_rn(0.f);      // padding rows of the B operand: written once
  if (V_LO)
    for (int e = LA_D; e < 16; ++e) vtl[e][tid] = __float2bfloat16_rn(0.f);       // the ones row is exact: its lo part is 0
  const int t_begin = chunk * LA_CHUNK, t_end = min(L, t_begin + LA_CHUNK);
  // ldmatrix row address of this lane inside a 16-token x 16-feature block: tile j = lane / 8 covers tokens (j & 2 ? 8 : 0) + r,
  // features (j & 1 ? 8 : 0) .. +7   ->   a[0], a[1], a[2], a[3] of the m16n8k16 A fragment (rows = features, k = tokens)
  const int lm_tok = ((lane >> 3) & 2 ? 8 : 0) + (lane & 7), lm_feat = ((lane >> 3) & 1) ? 8 : 0;
  for (int t0 = t_begin; t0 < t_end; t0 += LAM_TB) {
    __syncthreads();
    {   // stage: thread = token
      const int tok = t0 + tid;
      const bool ok = tok < t_end;
      float kk[LA_D], vv[LA_D];
      if (ok) {
        const T* row = kv + (seq * L + tok) * (2 * (int64_t)HD);
        const uint4 kr = *reinterpret_cast<const uint4*>(row + h * LA_D);
        const uint4 vr = *reinterpret_cast<const uint4*>(row + HD + h * LA_D);
        const pair_t<T>* kb = reinterpret_cast<const pair_t<T>*>(&kr);
        const pair_t<T>* vb = reinterpret_cast<const pair_t<T>*>(&vr);
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          const float2 a = pair_to_f2(kb[q]), b = pair_to_f2(vb[q]);
          kk[2 * q] = a.x; kk[2 * q + 1] = a.y; vv[2 * q] = b.x; vv[2 * q + 1] = b.y;
        }
      } else {
#pragma unroll
        for (int q = 0; q < LA_D; ++q) { kk[q] = 0.f; vv[q] = 0.f; }
      }
      uint32_t fh[LAM_F / 2], fl[LAM_F / 2];
      for_each_feature_pair<0>(kk, [&](int f, float a, float b) {
        a = ok ? a : 0.f;
        b = ok ? b : 0.f;
        const __nv_bfloat16 ah = __float2bfloat16_rn(a), bh = __float2bfloat16_rn(b);
        __nv_bfloat162 hi; hi.x = ah; hi.y = bh;
        fh[f >> 1] = *reinterpret_cast<uint32_t*>(&hi);
        fl[f >> 1] = pack2_16<__nv_bfloat16>(a - __bfloat162float(ah), b - __bfloat162float(bh));
      });
#pragma unroll
      for (int v = 0; v < LAM_F / 8; ++v) {
        *reinterpret_cast<uint4*>(&phi_s[tid][v * 8]) = make_uint4(fh[4 * v], fh[4 * v + 1], fh[4 * v + 2], fh[4 * v + 3]);
        *reinterpret_cast<uint4*>(&phi_l[tid][v * 8]) = make_uint4(fl[4 * v], fl[4 * v + 1], fl[4 * v + 2], fl[4 * v + 3]);
      }
#pragma unroll
      for (int e = 0; e < LA_D; ++e) {
        const __nv_bfloat16 vh = __float2bfloat16_rn(vv[e]);
        vt[e][tid] = vh;
        if (V_LO) vtl[e][tid] = __float2bfloat16_rn(vv[e] - __bfloat162float(vh));
      }
      vt[LA_D][tid] = __float2bfloat16_rn(ok ? 1.f : 0.f);
    }
    __syncthreads();
    // each warp contracts its 32 tokens (2 k-steps of 16)
#pragma unroll
    for (int ks = 0; ks < 2; ++ks) {
      const int n0 = warp * 32 + ks * 16;
      uint32_t b[2][2], bl[2][2];
#pragma unroll
      for (int nt = 0; nt < 2; ++nt) {
        b[nt][0] = *reinterpret_cast<const uint32_t*>(&vt[nt * 8 + g][n0 + t * 2]);
        b[nt][1] = *reinterpret_cast<const uint32_t*>(&vt[nt * 8 + g][n0 + 8 + t * 2]);
        if (V_LO) {
          bl[nt][0] = *reinterpret_cast<const uint32_t*>(&vtl[nt * 8 + g][n0 + t * 2]);
          bl[nt][1] = *reinterpret_cast<const uint32_t*>(&vtl[nt * 8 + g][n0 + 8 + t * 2]);
        }
      }
#pragma unroll
      for (int mt = 0; mt < 5; ++mt) {
        uint32_t a[4];
        ldmatrix_x4_trans(a, &phi_s[n0 + lm_tok][mt * 16 + lm_feat]);
        mma_16816<__nv_bfloat16>(acc[mt][0], a, b[0][0], b[0][1]);
        mma_16816<__nv_bfloat16>(acc[mt][1], a, b[1][0], b[1][1]);
        if (V_LO) {
          mma_16816<__nv_bfloat16>(acc[mt][0], a, bl[0][0], bl[0][1]);
          mma_16816<__nv_bfloat16>(acc[mt][1], a, bl[1][0], bl[1][1]);
        }
        ldmatrix_x4_trans(a, &phi_l[n0 + lm_tok][mt * 16 + lm_feat]);
        mma_16816<__nv_bfloat16>(acc[mt][0], a, b[0][0], b[0][1]);
        mma_16816<__nv_bfloat16>(acc[mt][1], a, b[1][0], b[1][1]);
      }
    }
  }
  // cross-warp reduction through shared memory (the phi hi tile is reused as fp32 [4 warps][80 * 16]: 20480 B <= 22528 B)
  __syncthreads();
  float* red = reinterpret_cast<float*>(lam_dyn);
#pragma unroll
  for (int mt = 0; mt < 5; ++mt)
#pragma unroll
    for (int nt = 0; nt < 2; ++nt) {
      const int f0 = mt * 16 + g, e0 = nt * 8 + t * 2;
      float* w = red + warp * (LAM_F * 16);
      w[f0 * 16 + e0] = acc[mt][nt][0];
      w[f0 * 16 + e0 + 1] = acc[mt][nt][1];
      w[(f0 + 8) * 16 + e0] = acc[mt][nt][2];
      w[(f0 + 8) * 16 + e0 + 1] = acc[mt][nt][3];
    }
  __syncthreads();
  float* o = ws + ((seq * heads + h) * n_chunks + chunk) * LA_ST;
  for (int idx = tid; idx < LA_ST; idx += 128) {
    const int f = idx / (LA_D + 1), e = idx % (LA_D + 1);
    const int si = f * 16 + e;
    o[idx] = red[si] + red[LAM_F * 16 + si] + red[2 * LAM_F * 16 + si] + red[3 * LAM_F * 16 + si];
  }
}
// bf16 keeps the kernel's name; the fp16 form is its _f16_ twin
__global__ void __launch_bounds__(128) linattn_reduce_mma_kernel(const __nv_bfloat16* __restrict__ kv, float* __restrict__ ws,
                                                                 int L, int heads, int n_chunks) {
  pdl_wait();
  pdl_launch_dependents();
  linattn_reduce_mma_body(kv, ws, L, heads, n_chunks);
}
__global__ void __launch_bounds__(128) linattn_reduce_mma_f16_kernel(const __half* __restrict__ kv, float* __restrict__ ws,
                                                                     int L, int heads, int n_chunks) {
  pdl_wait();
  pdl_launch_dependents();
  linattn_reduce_mma_body(kv, ws, L, heads, n_chunks);
}

constexpr int LAM_AT = 64;     // tokens per block in the apply kernel (2 warps x 32)
constexpr int LAM_SW = 16 * (LAM_F + 8);   // bf16 elements of one transposed state operand [e][feature]

// Sums the per-chunk partial states of one (sequence, head) and writes the transposed MMA B operand as a bf16
// hi + lo pair, once, so the apply blocks only copy 5.6 KB instead of re-reducing the partials.
__global__ void __launch_bounds__(128) linattn_finalize_kernel(const float* __restrict__ ws, __nv_bfloat16* __restrict__ sw,
                                                               int heads, int n_chunks) {
  pdl_wait();
  pdl_launch_dependents();
  const int h = blockIdx.x;
  const int64_t seq = blockIdx.y;
  const float* wsh = ws + (seq * heads + h) * (int64_t)n_chunks * LA_ST;
  __nv_bfloat16* o = sw + (seq * heads + h) * (int64_t)(2 * LAM_SW);
  for (int idx = threadIdx.x; idx < LAM_SW; idx += 128) {
    const int e = idx / (LAM_F + 8), f = idx % (LAM_F + 8);
    float sv = 0.f;
    if (e <= LA_D && f < LA_F)
      for (int k = 0; k < n_chunks; ++k) sv += wsh[(int64_t)k * LA_ST + f * (LA_D + 1) + e];
    const __nv_bfloat16 hi = __float2bfloat16_rn(sv);
    o[idx] = hi;
    o[LAM_SW + idx] = __float2bfloat16_rn(sv - __bfloat162float(hi));
  }
}

constexpr int LAM_AB = 4;      // 64-token sub-blocks per apply block: the 5.6 KB state operand is loaded once per 256 tokens
// T: element type of q and out (bf16 or fp16); the MMA operands are bf16 hi + lo pairs of fp32 values either way
template <typename T>
__device__ __forceinline__ void linattn_apply_mma_body(const T* __restrict__ q, const __nv_bfloat16* __restrict__ sw,
                                                       T* __restrict__ out, int L, int heads) {
  // both operands are carried as bf16 hi + lo pairs (3 MMAs: hi*hi + lo*hi + hi*lo) -> ~fp32-level accuracy
  __shared__ __align__(16) __nv_bfloat16 phi_s[LAM_AT][LAM_F + 8];   // [token][feature] hi
  __shared__ __align__(16) __nv_bfloat16 phi_l[LAM_AT][LAM_F + 8];   // lo
  __shared__ __align__(16) __nv_bfloat16 st[16][LAM_F + 8];          // [e][feature] hi  (S transposed; e = 8 is the denominator)
  __shared__ __align__(16) __nv_bfloat16 sl[16][LAM_F + 8];          // lo
  const int h = blockIdx.y;
  const int64_t seq = blockIdx.z;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int g = lane >> 2, t = lane & 3;
  const int HD = heads * LA_D;
  {
    const uint4* src = reinterpret_cast<const uint4*>(sw + (seq * heads + h) * (int64_t)(2 * LAM_SW));
    uint4* d0 = reinterpret_cast<uint4*>(&st[0][0]);
    uint4* d1 = reinterpret_cast<uint4*>(&sl[0][0]);
    constexpr int NV = LAM_SW / 8;
    for (int i = tid; i < NV; i += 64) { d0[i] = src[i]; d1[i] = src[NV + i]; }
  }
  for (int sb = 0; sb < LAM_AB; ++sb) {
    const int blk = blockIdx.x * LAM_AB + sb;
    if (blk * LAM_AT >= L) break;
    __syncthreads();                 // the previous sub-block's fragment loads are done (first pass: state copy ordering below)
    {
      const int tok = blk * LAM_AT + tid;
      const bool ok = tok < L;
      float qq[LA_D];
      if (ok) {
        const uint4 qr = *reinterpret_cast<const uint4*>(q + (seq * L + tok) * HD + h * LA_D);
        const pair_t<T>* qb = reinterpret_cast<const pair_t<T>*>(&qr);
        const float qs = rsqrtf((float)LA_D);
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const float2 a = pair_to_f2(qb[i]);
          qq[2 * i] = a.x * qs; qq[2 * i + 1] = a.y * qs;
        }
      } else {
#pragma unroll
        for (int i = 0; i < LA_D; ++i) qq[i] = 0.f;
      }
      // the 80 features of this token, as 40 packed hi pairs + 40 packed lo pairs, written with 16-byte stores: a token row is
      // 176 bytes, so the 32 rows of a warp start in 8 distinct bank groups and a 16-byte store takes the minimal 4 wavefronts
      // (the former 4-byte stores were 4-way bank conflicted and dominated the kernel's shared-memory traffic)
      uint32_t fh[LAM_F / 2], fl[LAM_F / 2];
      for_each_feature_pair<0>(qq, [&](int f, float a, float b) {
        const __nv_bfloat16 ah = __float2bfloat16_rn(a), bh = __float2bfloat16_rn(b);
        __nv_bfloat162 hi; hi.x = ah; hi.y = bh;
        fh[f >> 1] = *reinterpret_cast<uint32_t*>(&hi);
        fl[f >> 1] = pack2_16<__nv_bfloat16>(a - __bfloat162float(ah), b - __bfloat162float(bh));
      });
#pragma unroll
      for (int v = 0; v < LAM_F / 8; ++v) {
        *reinterpret_cast<uint4*>(&phi_s[tid][v * 8]) = make_uint4(fh[4 * v], fh[4 * v + 1], fh[4 * v + 2], fh[4 * v + 3]);
        *reinterpret_cast<uint4*>(&phi_l[tid][v * 8]) = make_uint4(fl[4 * v], fl[4 * v + 1], fl[4 * v + 2], fl[4 * v + 3]);
      }
    }
    __syncthreads();
#pragma unroll
    for (int mi = 0; mi < 2; ++mi) {
      const int n0 = warp * 32 + mi * 16;
      float c[2][4];
#pragma unroll
      for (int nt = 0; nt < 2; ++nt)
#pragma unroll
        for (int j = 0; j < 4; ++j) c[nt][j] = 0.f;
#pragma unroll
      for (int ks = 0; ks < LAM_F / 16; ++ks) {
        uint32_t ah[4], al[4];
        ah[0] = *reinterpret_cast<const uint32_t*>(&phi_s[n0 + g][ks * 16 + t * 2]);
        ah[1] = *reinterpret_cast<const uint32_t*>(&phi_s[n0 + g + 8][ks * 16 + t * 2]);
        ah[2] = *reinterpret_cast<const uint32_t*>(&phi_s[n0 + g][ks * 16 + 8 + t * 2]);
        ah[3] = *reinterpret_cast<const uint32_t*>(&phi_s[n0 + g + 8][ks * 16 + 8 + t * 2]);
        al[0] = *reinterpret_cast<const uint32_t*>(&phi_l[n0 + g][ks * 16 + t * 2]);
        al[1] = *reinterpret_cast<const uint32_t*>(&phi_l[n0 + g + 8][ks * 16 + t * 2]);
        al[2] = *reinterpret_cast<const uint32_t*>(&phi_l[n0 + g][ks * 16 + 8 + t * 2]);
        al[3] = *reinterpret_cast<const uint32_t*>(&phi_l[n0 + g + 8][ks * 16 + 8 + t * 2]);
#pragma unroll
        for (int nt = 0; nt < 2; ++nt) {
          const uint32_t bh0 = *reinterpret_cast<const uint32_t*>(&st[nt * 8 + g][ks * 16 + t * 2]);
          const uint32_t bh1 = *reinterpret_cast<const uint32_t*>(&st[nt * 8 + g][ks * 16 + 8 + t * 2]);
          const uint32_t bl0 = *reinterpret_cast<const uint32_t*>(&sl[nt * 8 + g][ks * 16 + t * 2]);
          const uint32_t bl1 = *reinterpret_cast<const uint32_t*>(&sl[nt * 8 + g][ks * 16 + 8 + t * 2]);
          mma_16816<__nv_bfloat16>(c[nt], ah, bh0, bh1);
          mma_16816<__nv_bfloat16>(c[nt], al, bh0, bh1);
          mma_16816<__nv_bfloat16>(c[nt], ah, bl0, bl1);
        }
      }
      // denominator = column 8 = c[1][0] (row g) / c[1][2] (row g+8) of the quad's t == 0 lane
      const float d0 = fmaxf(__shfl_sync(0xffffffffu, c[1][0], lane & ~3), 1e-5f);
      const float d1 = fmaxf(__shfl_sync(0xffffffffu, c[1][2], lane & ~3), 1e-5f);
      const int r0 = blk * LAM_AT + n0 + g, r1 = r0 + 8;
      if (r0 < L) *reinterpret_cast<uint32_t*>(out + (seq * L + r0) * HD + h * LA_D + t * 2) = pack2_16<T>(c[0][0] / d0, c[0][1] / d0);
      if (r1 < L) *reinterpret_cast<uint32_t*>(out + (seq * L + r1) * HD + h * LA_D + t * 2) = pack2_16<T>(c[0][2] / d1, c[0][3] / d1);
    }
  }
}
__global__ void __launch_bounds__(64) linattn_apply_mma_kernel(const __nv_bfloat16* __restrict__ q, const __nv_bfloat16* __restrict__ sw,
                                                               __nv_bfloat16* __restrict__ out, int L, int heads) {
  pdl_wait();
  pdl_launch_dependents();
  linattn_apply_mma_body(q, sw, out, L, heads);
}
__global__ void __launch_bounds__(64) linattn_apply_mma_f16_kernel(const __half* __restrict__ q, const __nv_bfloat16* __restrict__ sw,
                                                                   __half* __restrict__ out, int L, int heads) {
  pdl_wait();
  pdl_launch_dependents();
  linattn_apply_mma_body(q, sw, out, L, heads);
}

// ------------------------------------------------------------------------------------------
// GEGLU
// ------------------------------------------------------------------------------------------
template <typename T>
__global__ void geglu_kernel(const T* __restrict__ in, T* __restrict__ out, int64_t N, int I) {
  pdl_wait();
  pdl_launch_dependents();
  const int64_t total = N * I;
  for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
    const int64_t n = idx / I;
    const int i = (int)(idx % I);
    const float xv = to_f32<T>(in[n * 2 * I + i]);
    const float g = to_f32<T>(in[n * 2 * I + I + i]);
    const float ge = 0.5f * g * (1.f + erff(g * 0.70710678118654752440f));
    out[idx] = from_f32<T>(ge * xv);
  }
}

// ------------------------------------------------------------------------------------------
// quantisers
// ------------------------------------------------------------------------------------------
// projected dims per token: D <= 16 runs the original instantiation, 17 <= D <= 32 (e.g. MAGVIT-v2's 2^18 codes, or 2 x 2^16)
// the wide one, so the narrow configurations keep their register budget and results
constexpr int Q_MAXD = 16, Q_MAXD_WIDE = 32;
template <int MAXD>
struct FsqLevelsT { int32_t lv[MAXD]; };

// mode 0: LFQ, mode 1: FSQ.  One warp per token.  `d` = dims per codebook, `nc` codebooks (d * nc <= MAXD projected dims,
// reference kwarg num_codebooks M:1057 -> M:1367 / M:1381): one index per (token, codebook), idx[tok * nc + cb].
// spherical (LFQ, M:1070 -> A.1 step 4): the per-codebook d-vector is L2-normalised before the sign / the auxiliary terms; the
// quantised output (+-1) and the indices do not depend on it.
template <typename T, int MODE, int MAXD>
__global__ void __launch_bounds__(256) quant_forward_kernel(const T* __restrict__ x, int64_t N, int C, int d, int nc,
                                                            const float* __restrict__ win, const float* __restrict__ bin,
                                                            const float* __restrict__ wout, const float* __restrict__ bout,
                                                            float clamp, int spherical, FsqLevelsT<MAXD> lv, int64_t* __restrict__ idx64,
                                                            int32_t* __restrict__ idx32, T* __restrict__ quant,
                                                            float* __restrict__ aux) {
  pdl_wait();
  pdl_launch_dependents();
  const int lane = threadIdx.x & 31;
  const int64_t tok = (int64_t)blockIdx.x * 8 + (threadIdx.x >> 5);
  if (tok >= N) return;
  const int D = d * nc;
  const T* row = x + tok * C;
  float acc[MAXD];
#pragma unroll
  for (int i = 0; i < MAXD; ++i) acc[i] = 0.f;
  for (int c = lane; c < C; c += 32) {
    const float xv = to_f32<T>(row[c]);
#pragma unroll
    for (int i = 0; i < MAXD; ++i)
      if (i < D) acc[i] = fmaf(xv, win[(int64_t)i * C + c], acc[i]);
  }
  float code[MAXD], pv[MAXD];
#pragma unroll
  for (int i = 0; i < MAXD; ++i) {
    pv[i] = 0.f;
    if (i < D) {
      float p = warp_sum(acc[i]) + bin[i];
      if (MODE == 0 && clamp > 0.f) p = tanhf(p / clamp) * clamp;
      pv[i] = p;
    }
  }
  if (MODE == 0 && spherical) {          // F.normalize(x, dim = -1) per codebook: x / max(||x||, 1e-12)
    for (int cb = 0; cb < nc; ++cb) {
      float ss = 0.f;
#pragma unroll
      for (int i = 0; i < MAXD; ++i)
        if (i >= cb * d && i < (cb + 1) * d) ss = fmaf(pv[i], pv[i], ss);
      const float inv = 1.f / fmaxf(sqrtf(ss), 1e-12f);
#pragma unroll
      for (int i = 0; i < MAXD; ++i)
        if (i >= cb * d && i < (cb + 1) * d) pv[i] *= inv;
    }
  }
  int64_t index = 0;
  int32_t basis = 1;
  int j = 0, cb = 0;                      // position inside the current codebook
#pragma unroll
  for (int i = 0; i < MAXD; ++i) {
    code[i] = 0.f;
    if (i < D) {
      const float p = pv[i];
      if (MODE == 0) {
        const bool bit = p > 0.f;
        code[i] = bit ? 1.f : -1.f;
        if (bit) index |= (int64_t)1 << (d - 1 - j);
        if (aux && lane == 0) aux[tok * D + i] = p;
      } else {
        const int L = lv.lv[j];
        const float half_l = (float)(L - 1) * (1.f + 1e-3f) * 0.5f;
        const float offset = (L % 2 == 0) ? 0.5f : 0.f;
        const float shift = atanhf(offset / half_l);
        const float bnd = tanhf(p + shift) * half_l - offset;
        const float q = rintf(bnd);  // round half to even, as torch.round
        const int half_w = L / 2;
        code[i] = q / (float)half_w;
        index += (int64_t)((int)q + half_w) * basis;
        basis *= L;
        if (aux && lane == 0) aux[tok * D + i] = bnd;
      }
      if (++j == d) {
        if (lane == 0) {
          if (idx64) idx64[tok * nc + cb] = index;
          if (idx32) idx32[tok * nc + cb] = (int32_t)index;
        }
        j = 0; ++cb; index = 0; basis = 1;
      }
    }
  }
  if (quant) {
    T* qrow = quant + tok * C;
    for (int c = lane; c < C; c += 32) {
      float o = bout[c];
#pragma unroll
      for (int i = 0; i < MAXD; ++i)
        if (i < D) o = fmaf(code[i], wout[(int64_t)c * D + i], o);
      qrow[c] = from_f32<T>(o);
    }
  }
}

template <typename T, int MODE, int MAXD>
__global__ void __launch_bounds__(256) quant_decode_kernel(const void* __restrict__ indices, int is64, int64_t N, int C,
                                                           int d, int nc, FsqLevelsT<MAXD> lv, const float* __restrict__ wout,
                                                           const float* __restrict__ bout, T* __restrict__ quant) {
  pdl_wait();
  pdl_launch_dependents();
  const int lane = threadIdx.x & 31;
  const int64_t tok = (int64_t)blockIdx.x * 8 + (threadIdx.x >> 5);
  if (tok >= N) return;
  const int D = d * nc;
  float code[MAXD];
  int64_t index = 0, rem = 0;
  int j = 0, cb = 0;
#pragma unroll
  for (int i = 0; i < MAXD; ++i) {
    code[i] = 0.f;
    if (i < D) {
      if (j == 0) {
        index = is64 ? ((const int64_t*)indices)[tok * nc + cb] : (int64_t)((const int32_t*)indices)[tok * nc + cb];
        rem = index;
      }
      if (MODE == 0) {
        code[i] = ((index >> (d - 1 - j)) & 1) ? 1.f : -1.f;
      } else {
        const int L = lv.lv[j];
        const int digit = (int)(rem % L);
        rem /= L;
        const int half_w = L / 2;
        code[i] = (float)(digit - half_w) / (float)half_w;
      }
      if (++j == d) { j = 0; ++cb; }
    }
  }
  T* qrow = quant + tok * C;
  for (int c = lane; c < C; c += 32) {
    float o = bout[c];
#pragma unroll
    for (int i = 0; i < MAXD; ++i)
      if (i < D) o = fmaf(code[i], wout[(int64_t)c * D + i], o);
    qrow[c] = from_f32<T>(o);
  }
}

// LFQ training-mode entropy / commitment partial sums.  One block handles LE_TOK tokens of ONE codebook (blockIdx.y):
// presign is [N][nc][d], avg_prob [nc][K].
constexpr int LE_TOK = 32;
__global__ void __launch_bounds__(256) lfq_entropy_kernel(const float* __restrict__ presign_all, int64_t N, int d, int nc,
                                                          float inv_temp, float* __restrict__ avg_prob_all,
                                                          float* __restrict__ stats) {
  pdl_wait();
  pdl_launch_dependents();
  extern __shared__ float probs[];  // [K]
  __shared__ float red[8];
  __shared__ float bc;
  const int K = 1 << d;
  const float* presign = presign_all + (int64_t)blockIdx.y * d;     // token stride below is nc * d
  float* avg_prob = avg_prob_all + (int64_t)blockIdx.y * K;
  const int tstride = nc * d;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  float ent_sum = 0.f, commit_sum = 0.f;
  const int64_t t0 = (int64_t)blockIdx.x * LE_TOK;
  // per-thread running sum of probabilities for codes k = tid, tid+256, ...
  float pacc[16];
#pragma unroll
  for (int r = 0; r < 16; ++r) pacc[r] = 0.f;
  for (int64_t t = t0; t < min(N, t0 + LE_TOK); ++t) {
    float p[12];
#pragma unroll
    for (int i = 0; i < 12; ++i) p[i] = (i < d) ? presign[t * tstride + i] : 0.f;
    float mx = -INFINITY;
    for (int k = tid; k < K; k += 256) {
      float s = 0.f;
#pragma unroll
      for (int i = 0; i < 12; ++i)
        if (i < d) s += ((k >> (d - 1 - i)) & 1) ? p[i] : -p[i];
      s *= 2.f * inv_temp;
      probs[k] = s;
      mx = fmaxf(mx, s);
    }
    mx = warp_max(mx);
    if (lane == 0) red[warp] = mx;
    __syncthreads();
    if (tid == 0) { float m = red[0]; for (int i = 1; i < 8; ++i) m = fmaxf(m, red[i]); bc = m; }
    __syncthreads();
    mx = bc;
    float sm = 0.f;
    for (int k = tid; k < K; k += 256) { float e = expf(probs[k] - mx); probs[k] = e; sm += e; }
    sm = warp_sum(sm);
    __syncthreads();
    if (lane == 0) red[warp] = sm;
    __syncthreads();
    if (tid == 0) { float s = 0.f; for (int i = 0; i < 8; ++i) s += red[i]; bc = 1.f / s; }
    __syncthreads();
    const float inv = bc;
    float ent = 0.f;
    int r = 0;
    for (int k = tid; k < K; k += 256, ++r) {
      const float pr = probs[k] * inv;
      ent -= pr * logf(fmaxf(pr, 1e-5f));
      if (r < 16) pacc[r] += pr;
    }
    ent_sum += ent;
    if (tid == 0) {
      float cs = 0.f;
      for (int i = 0; i < d; ++i) { float q = p[i] > 0.f ? 1.f : -1.f; cs += (p[i] - q) * (p[i] - q); }
      commit_sum += cs;
    }
    __syncthreads();
  }
  {
    int r = 0;
    for (int k = tid; k < K; k += 256, ++r)
      if (r < 16) atomicAdd(&avg_prob[k], pacc[r]);
  }
  ent_sum = warp_sum(ent_sum);
  if (lane == 0) atomicAdd(&stats[0], ent_sum);
  if (tid == 0) atomicAdd(&stats[1], commit_sum);
}


// ------------------------------------------------------------------------------------------
// LFQ entropy terms of large codebooks (1 <= d <= 20), factorised over bits.  The code distribution
//   prob_k = softmax_k(2 tau <p, c_k>),  c_k in {+-1}^d,   equals   prod_i sigma(4 tau p_i s_ki)
// (s_ki = +-1: bit i of code k, MSB first as LFQ's mask), so one (token, code) probability is the product of two or three entries
// of small per-token tables of bit-probability products and nothing of size K is kept per token.  The clamped entropy
// -x log max(x, 1e-5) is not a sum over bits, so both passes still visit every (token, code) pair -- but they take a log only
// where x > 1e-5.  Every sum runs in a fixed order (per-thread registers, fixed shuffle trees, fixed-order partial reductions;
// no float atomics), so two runs give bit-identical results.
// ------------------------------------------------------------------------------------------
constexpr int LF_MAXD = 20;
constexpr int LF_TT = 32;                 // tokens staged per chunk (partials)
constexpr int LF_R = 16;                  // codes per thread (partials)
constexpr int LF_TARGET_BLOCKS = 264;     // partials grid: code tiles x token splits x codebooks ~ 2 waves of 132 SMs
constexpr int LF_BW_WARPS = 4;            // backward: warps per block (~150 registers per thread: 3 blocks per SM)
constexpr float LF_LOG_INV_EPS = 11.512925464970229f;   // -log(1e-5): -x log max(x, 1e-5) = x * this for x <= 1e-5

// code bit layout of the partials kernel (LSB first): lb = min(d, 8) bits -> threadIdx.x (split into lo4 = min(lb, 4) and the rest),
// rb = min(d - lb, 4) bits -> the thread's LF_R register codes, the top tb = d - lb - rb bits -> blockIdx.x (one code tile)
struct LfLayout {
  int lb, lo4, rb, tb;
  __host__ __device__ explicit LfLayout(int d) {
    lb = d < 8 ? d : 8;
    lo4 = lb < 4 ? lb : 4;
    rb = d - lb < 4 ? d - lb : 4;
    tb = d - lb - rb;
  }
};

struct LfSplit { int tiles, splits; int64_t per; };
static inline LfSplit lf_split(int64_t N, int d, int nc) {
  const LfLayout L(d);
  LfSplit s;
  s.tiles = 1 << L.tb;
  const int64_t want = std::max<int64_t>(1, (LF_TARGET_BLOCKS + (int64_t)s.tiles * nc - 1) / ((int64_t)s.tiles * nc));
  const int64_t chunks = (N + LF_TT - 1) / LF_TT;
  const int64_t sp = std::min<int64_t>(want, chunks);
  s.per = (chunks + sp - 1) / sp * LF_TT;           // tokens per split, a whole number of chunks
  s.splits = (int)((N + s.per - 1) / s.per);        // no empty split
  return s;
}

// product of the bit probabilities of `v` (nbits bits) over dims [i0, i0 + nbits): dim i0 + j <-> bit nbits - 1 - j of v
__device__ __forceinline__ float lf_bits_prod(const float (*sg)[2], int i0, int nbits, int v) {
  float a = 1.f;
  for (int j = 0; j < nbits; ++j) a *= sg[i0 + j][(v >> (nbits - 1 - j)) & 1];
  return a;
}

__device__ __forceinline__ float lf_plogp(float x) {     // -x log max(x, 1e-5)
  return x > 1e-5f ? -x * __logf(x) : x * LF_LOG_INV_EPS;
}

// one block: one code tile (LF_R x 256 codes) of one codebook (blockIdx.z) over one token split (blockIdx.y).  Per code: the sum of
// prob over the split's tokens; per block: the sum of the clamped entropy terms.  Both into fp64 workspace partials.
__global__ void __launch_bounds__(256, 1) lfq_fact_partials_kernel(const float* __restrict__ presign, int64_t N, int d, int nc,
                                                                float inv_temp, int64_t per, double* __restrict__ ws_avg,
                                                                double* __restrict__ ws_ent) {
  pdl_wait();
  pdl_launch_dependents();
  __shared__ float sg[LF_TT][LF_MAXD][2];       // sigma(-4 tau p), sigma(+4 tau p): probability of code bit 0 / 1
  __shared__ float tab[LF_TT][3][16];           // per token: low-4-bit products, next-4-bit products, Q[r] = tile factor x r factor
  __shared__ double red[8];
  const LfLayout L(d);
  const int K = 1 << d, tid = threadIdx.x, tile = blockIdx.x, split = blockIdx.y, c = blockIdx.z;
  const int64_t tbeg = (int64_t)split * per, tend = min(N, tbeg + per);
  double accd[LF_R], entd = 0.0;
#pragma unroll
  for (int r = 0; r < LF_R; ++r) accd[r] = 0.0;
  for (int64_t t0 = tbeg; t0 < tend; t0 += LF_TT) {
    const int nt = (int)min((int64_t)LF_TT, tend - t0);
    for (int e = tid; e < nt * d; e += 256) {
      const int t = e / d, i = e - t * d;
      const float x = 4.f * inv_temp * presign[((t0 + t) * nc + c) * d + i];
      sg[t][i][1] = 1.f / (1.f + expf(-x));
      sg[t][i][0] = 1.f / (1.f + expf(x));
    }
    __syncthreads();
    for (int e = tid; e < LF_TT * 48; e += 256) {
      const int t = e / 48, w = e - t * 48, which = w >> 4, v = w & 15;
      float a = 0.f;
      if (t < nt) {
        if (which == 0) a = v < (1 << L.lo4) ? lf_bits_prod(sg[t], d - L.lo4, L.lo4, v) : 0.f;
        else if (which == 1) a = v < (1 << (L.lb - L.lo4)) ? lf_bits_prod(sg[t], d - L.lb, L.lb - L.lo4, v) : 0.f;
        else a = v < (1 << L.rb) ? lf_bits_prod(sg[t], L.tb, L.rb, v) * lf_bits_prod(sg[t], 0, L.tb, tile) : 0.f;
      }
      tab[t][which][v] = a;
    }
    __syncthreads();
    float acc[LF_R], ent = 0.f;
#pragma unroll
    for (int r = 0; r < LF_R; ++r) acc[r] = 0.f;
    for (int t = 0; t < nt; ++t) {
      const float b = tab[t][0][tid & 15] * tab[t][1][tid >> 4];     // 0 for the threads past 2^lb codes
#pragma unroll
      for (int r = 0; r < LF_R; ++r) {
        const float pr = tab[t][2][r] * b;
        acc[r] += pr;
        ent += lf_plogp(pr);
      }
    }
#pragma unroll
    for (int r = 0; r < LF_R; ++r) accd[r] += (double)acc[r];
    entd += (double)ent;
    __syncthreads();               // sg / tab are rewritten by the next chunk
  }
  if (tid < (1 << L.lb)) {
    double* out = ws_avg + ((int64_t)split * nc + c) * K + ((int64_t)tile << (L.rb + L.lb)) + tid;
#pragma unroll
    for (int r = 0; r < LF_R; ++r)
      if (r < (1 << L.rb)) out[(int64_t)r << L.lb] = accd[r];
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) entd += __shfl_xor_sync(0xffffffffu, entd, o);
  if ((tid & 31) == 0) red[tid >> 5] = entd;
  __syncthreads();
  if (tid == 0) {
    double s = 0.0;
    for (int w = 0; w < 8; ++w) s += red[w];
    ws_ent[((int64_t)split * nc + c) * gridDim.x + tile] = s;
  }
}

// avg_prob[i] = sum over the token splits, in split order
__global__ void __launch_bounds__(256) lfq_fact_avg_kernel(const double* __restrict__ ws_avg, int64_t n, int splits,
                                                           float* __restrict__ avg_prob) {
  pdl_wait();
  pdl_launch_dependents();
  const int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x;
  if (i >= n) return;
  double s = 0.0;
  for (int k = 0; k < splits; ++k) s += ws_avg[(int64_t)k * n + i];
  avg_prob[i] = (float)s;
}

// stats[0] = entropy partials summed in a fixed order, stats[1] = commitment sum  sum (p - sign p)^2  over [N][nc][d]
__global__ void __launch_bounds__(256) lfq_fact_stats_kernel(const double* __restrict__ ws_ent, int n_ent, const float* __restrict__ presign,
                                                             int64_t n_pre, float* __restrict__ stats) {
  pdl_wait();
  pdl_launch_dependents();
  __shared__ double red[2][8];
  double e = 0.0, cm = 0.0;
  for (int i = threadIdx.x; i < n_ent; i += 256) e += ws_ent[i];
  for (int64_t i = threadIdx.x; i < n_pre; i += 256) {
    const float p = presign[i], q = p > 0.f ? 1.f : -1.f;
    cm += (double)((p - q) * (p - q));
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    e += __shfl_xor_sync(0xffffffffu, e, o);
    cm += __shfl_xor_sync(0xffffffffu, cm, o);
  }
  if ((threadIdx.x & 31) == 0) { red[0][threadIdx.x >> 5] = e; red[1][threadIdx.x >> 5] = cm; }
  __syncthreads();
  if (threadIdx.x == 0) {
    double a = 0.0, b = 0.0;
    for (int w = 0; w < 8; ++w) { a += red[0][w]; b += red[1][w]; }
    stats[0] = (float)a;
    stats[1] = (float)b;
  }
}

// hga[i] = coef_batch * h'(avg_global[i]),  h'(x) = -(log x + 1) for x > 1e-5, -log 1e-5 below the clamp
__global__ void __launch_bounds__(256) lfq_fact_hga_kernel(const float* __restrict__ avg, int64_t n, float coef_batch,
                                                           float* __restrict__ hga) {
  pdl_wait();
  pdl_launch_dependents();
  const int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x;
  if (i >= n) return;
  const float a = avg[i];
  hga[i] = coef_batch * (a > 1e-5f ? -(logf(a) + 1.f) : LF_LOG_INV_EPS);
}

// Backward of  coef_sample * sum_t H(prob_t) - coef_batch * <h'(avg_global), sum_t prob_t>  (the entropy part of LFQ's aux loss,
// with avg entering as avg_local + (avg_global - avg_local).detach()) with respect to the pre-sign values:
//   c_tk = prob_tk (coef_sample h'(prob_tk) - coef_batch h'(avg_global_k)),   dp_ti = 2 tau (sum_k c_tk s_ki - tanh(2 tau p_ti) sum_k c_tk)
// One warp per (token, codebook) walks all 2^d codes.  Code bit layout (LSB first): min(d, 5) bits -> lane, the next min(d - 5, 5)
// bits -> the warp's 32 register columns j, the rest -> the outer loop.  The bit sums come from the per-column sums M[j], the
// per-outer-step sums and the lane's total, so the cost is O(2^d) per token, not O(2^d d).
__global__ void __launch_bounds__(LF_BW_WARPS * 32) lfq_fact_backward_kernel(const float* __restrict__ presign, const float* __restrict__ hga,
                                                                int64_t N, int d, int nc, float inv_temp, float coef_sample,
                                                                float* __restrict__ grad) {
  pdl_wait();
  pdl_launch_dependents();
  __shared__ float sgw[LF_BW_WARPS][LF_MAXD][2];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int64_t pair = (int64_t)blockIdx.x * LF_BW_WARPS + warp;   // token * nc + codebook
  if (pair >= N * nc) return;
  const int c = (int)(pair % nc), K = 1 << d;
  const int lbb = d < 5 ? d : 5, mbb = d - lbb < 5 ? d - lbb : 5, tbb = d - lbb - mbb;
  const float* pp = presign + pair * d;
  float pi = 0.f;
  if (lane < d) {
    pi = pp[lane];
    const float x = 4.f * inv_temp * pi;
    sgw[warp][lane][1] = 1.f / (1.f + expf(-x));
    sgw[warp][lane][0] = 1.f / (1.f + expf(x));
  }
  __syncwarp();
  const float (*sg)[2] = sgw[warp];
  const float b = lane < (1 << lbb) ? lf_bits_prod(sg, d - lbb, lbb, lane) : 0.f;
  const float am = lane < (1 << mbb) ? lf_bits_prod(sg, tbb, mbb, lane) : 0.f;
  float P[32], M[32], Ht[LF_MAXD - 10];
#pragma unroll
  for (int j = 0; j < 32; ++j) { P[j] = __shfl_sync(0xffffffffu, am, j) * b; M[j] = 0.f; }
#pragma unroll
  for (int i = 0; i < LF_MAXD - 10; ++i) Ht[i] = 0.f;
  const float* hg = hga + (int64_t)c * K;
  const bool live = lane < (1 << lbb);
  for (int tp = 0; tp < (1 << tbb); ++tp) {
    const float at = lf_bits_prod(sg, 0, tbb, tp);
    const int base = (tp << (mbb + lbb)) + lane;
    float u = 0.f;
#pragma unroll
    for (int j = 0; j < 32; ++j) {
      if (j < (1 << mbb)) {
        const float pr = at * P[j];
        const float h = live ? __ldg(hg + base + (j << lbb)) : 0.f;
        const float hp = pr > 1e-5f ? -(__logf(pr) + 1.f) : LF_LOG_INV_EPS;
        const float cv = pr * fmaf(coef_sample, hp, -h);
        M[j] += cv;
        u += cv;
      }
    }
#pragma unroll
    for (int i = 0; i < LF_MAXD - 10; ++i)
      if (i < tbb) Ht[i] += ((tp >> (tbb - 1 - i)) & 1) ? u : -u;
  }
  float T = 0.f;
#pragma unroll
  for (int j = 0; j < 32; ++j) T += M[j];
  float g = 0.f;
#pragma unroll
  for (int i = 0; i < LF_MAXD; ++i) {
    if (i < d) {
      float v = 0.f;
      if (i < tbb) {
        if (i < LF_MAXD - 10) v = Ht[i];
      } else if (i < tbb + mbb) {
        const int q = mbb - 1 - (i - tbb);
#pragma unroll
        for (int j = 0; j < 32; ++j) v += ((j >> q) & 1) ? M[j] : -M[j];
      } else {
        v = ((lane >> (d - 1 - i)) & 1) ? T : -T;
      }
      v = warp_sum(v);
      if (lane == i) g = v;
    }
  }
  T = warp_sum(T);
  if (lane < d) grad[pair * d + lane] = 2.f * inv_temp * (g - tanhf(2.f * inv_temp * pi) * T);
}

// LFQ auxiliary loss for codebooks past the one-block 256-thread finalize (d > 12): the same terms, fp64 sums in a fixed order
__global__ void __launch_bounds__(1024) lfq_aux_final_wide_kernel(const float* __restrict__ avg_prob_sum, const float* __restrict__ stats,
                                                                  int64_t n, int nc, float inv_tokens_global, float inv_tokens,
                                                                  float inv_elems, float gamma, float w_entropy, float w_commit,
                                                                  float* __restrict__ out) {
  pdl_wait();
  pdl_launch_dependents();
  __shared__ double sw[32];
  double t = 0.0;
  for (int64_t k = threadIdx.x; k < n; k += 1024) {
    const float p = avg_prob_sum[k] * inv_tokens_global;
    t += (double)(-p * logf(fmaxf(p, 1e-5f)));
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) t += __shfl_xor_sync(0xffffffffu, t, o);
  if ((threadIdx.x & 31) == 0) sw[threadIdx.x >> 5] = t;
  __syncthreads();
  if (threadIdx.x == 0) {
    double s = 0.0;
    for (int w = 0; w < 32; ++w) s += sw[w];
    const float be = (float)(s / nc);
    const float ps = stats[0] * inv_tokens, cm = stats[1] * inv_elems;
    out[0] = ps; out[1] = be; out[2] = cm;
    out[3] = (ps - gamma * be) * w_entropy + cm * w_commit;
  }
}

// ------------------------------------------------------------------------------------------
// gateloop_time (reference M:1216-1222: ToTimeSequence(Residual(SimpleGateLoopLayer))): per (clip, pixel, channel) the gated
// recurrence over time  s_t = sigmoid(a_t) s_{t-1} + kv_t,  out_t = q_t s_t + x_t  (residual fused), with q / kv / a the three
// channel thirds of the Linear(dim, 3 dim) output.  One thread per (b, pixel, channel); consecutive threads = consecutive
// channels, so every time step is a coalesced row access.  State in fp32.
// ------------------------------------------------------------------------------------------
template <typename T>
__global__ void __launch_bounds__(256) gateloop_scan_kernel(const T* __restrict__ qkva, const T* __restrict__ res, T* __restrict__ out,
                                                            int Tn, int64_t PC, int C, int64_t total, float* __restrict__ state) {
  pdl_wait();
  pdl_launch_dependents();
  const int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x;      // over B * P * C
  if (i >= total) return;
  const int64_t b = i / PC, pc = i - b * PC;
  const int64_t p = pc / C;
  const int c = (int)(pc - p * C);
  const int64_t P = PC / C;
  float s = state ? state[i] : 0.f;
  for (int t = 0; t < Tn; ++t) {
    const int64_t pos = (b * Tn + t) * P + p;
    const T* row = qkva + pos * 3 * C;
    const float q = to_f32<T>(row[c]), kv = to_f32<T>(row[C + c]), a = to_f32<T>(row[2 * C + c]);
    s = fmaf(1.f / (1.f + expf(-a)), s, kv);
    out[pos * C + c] = from_f32<T>(fmaf(q, s, to_f32<T>(res[pos * C + c])));
  }
  if (state) state[i] = s;
}

// ------------------------------------------------------------------------------------------
// reconstruction loss F.mse_loss(video, recon_video) (reference M:1722): mean over all elements of (a - b)^2.
// Deterministic two-stage reduction: MSE_BLOCKS blocks accumulate strided fp32 partial sums (one double per block),
// then one warp folds the block partials in a fixed order.  a may be MV2_U8 (frames, x / 255).
// ------------------------------------------------------------------------------------------
constexpr int MSE_BLOCKS = 592;      // 4 per SM
template <typename TA, typename TB>
__global__ void __launch_bounds__(256) mse_partial_kernel(const TA* __restrict__ a, const TB* __restrict__ b, int64_t n,
                                                          double* __restrict__ partials) {
  pdl_wait();
  pdl_launch_dependents();
  float acc[4] = {0.f, 0.f, 0.f, 0.f};
  const int64_t stride = (int64_t)gridDim.x * 256;
  int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x;
  for (; i + 3 * stride < n; i += 4 * stride) {
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const float dlt = to_f32<TA>(a[i + u * stride]) - to_f32<TB>(b[i + u * stride]);
      acc[u] = fmaf(dlt, dlt, acc[u]);
    }
  }
  for (; i < n; i += stride) {
    const float dlt = to_f32<TA>(a[i]) - to_f32<TB>(b[i]);
    acc[0] = fmaf(dlt, dlt, acc[0]);
  }
  double t = (double)acc[0] + (double)acc[1] + (double)acc[2] + (double)acc[3];
  __shared__ double sw[8];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) t += __shfl_xor_sync(0xffffffffu, t, o);
  if ((threadIdx.x & 31) == 0) sw[threadIdx.x >> 5] = t;
  __syncthreads();
  if (threadIdx.x == 0) {
    double r = 0.0;
#pragma unroll
    for (int w = 0; w < 8; ++w) r += sw[w];
    partials[blockIdx.x] = r;
  }
}

__global__ void __launch_bounds__(32) mse_final_kernel(const double* __restrict__ partials, int nb, double inv_n, float* __restrict__ out) {
  pdl_wait();
  pdl_launch_dependents();
  double t = 0.0;
  for (int k = threadIdx.x; k < nb; k += 32) t += partials[k];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) t += __shfl_xor_sync(0xffffffffu, t, o);
  if (threadIdx.x == 0) out[0] = (float)(t * inv_n);
}

// LFQ auxiliary loss from the (all-reduced) partial sums (A.1 steps 7-10):
//   per_sample = stats[0] / N, commitment = stats[1] / (N d), batch_entropy = sum_k -p_k log(max(p_k, 1e-5)) with
//   p = avg_prob_sum / (N_global), aux = (per_sample - gamma * batch_entropy) * w_entropy + commitment * w_commit.
// out[0..3] = per_sample, batch_entropy, commitment, aux.
__global__ void __launch_bounds__(256) lfq_aux_final_kernel(const float* __restrict__ avg_prob_sum, const float* __restrict__ stats, int K,
                                                            int nc, float inv_tokens_global, float inv_tokens, float inv_elems, float gamma,
                                                            float w_entropy, float w_commit, float* __restrict__ out) {
  pdl_wait();
  pdl_launch_dependents();
  float t = 0.f;
  for (int k = threadIdx.x; k < K * nc; k += 256) {     // codebook entropy: mean over the codebooks of sum_k -p log p
    const float p = avg_prob_sum[k] * inv_tokens_global;
    t += -p * logf(fmaxf(p, 1e-5f));
  }
  __shared__ float sw[8];
  t = warp_sum(t);
  if ((threadIdx.x & 31) == 0) sw[threadIdx.x >> 5] = t;
  __syncthreads();
  if (threadIdx.x == 0) {
    float be = 0.f;
#pragma unroll
    for (int w = 0; w < 8; ++w) be += sw[w];
    be /= (float)nc;
    const float ps = stats[0] * inv_tokens, cm = stats[1] * inv_elems;
    out[0] = ps; out[1] = be; out[2] = cm;
    out[3] = (ps - gamma * be) * w_entropy + cm * w_commit;
  }
}

// ------------------------------------------------------------------------------------------
// 2x2 max-pool of a VGG feature extractor (nn.MaxPool2d(2, 2), floor mode), channels-last, VEC channels per thread
// ------------------------------------------------------------------------------------------
template <typename T, int VEC>
struct alignas(sizeof(T) * VEC) VecT { T v[VEC]; };

// torch's rule (max_pool2d): a later element replaces the running maximum only when strictly larger or NaN, so ties go to
// the first element in row-major window order and a NaN, once taken, stays
__device__ __forceinline__ bool pool_takes(float v, float m) { return v > m || isnan(v); }

template <typename T, int VEC>
__global__ void __launch_bounds__(256) maxpool2x2_kernel(const T* __restrict__ x, T* __restrict__ y, int N, int H, int W, int C) {
  pdl_wait();
  pdl_launch_dependents();
  using V = VecT<T, VEC>;
  const int Ho = H >> 1, Wo = W >> 1, Cv = C / VEC;
  const int64_t total = (int64_t)N * Ho * Wo * Cv;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    int64_t r = i;
    const int cv = (int)(r % Cv); r /= Cv;
    const int wo = (int)(r % Wo); r /= Wo;
    const int ho = (int)(r % Ho);
    const int64_t n = r / Ho;
    const int64_t p0 = ((n * H + 2 * ho) * W + 2 * wo) * C + (int64_t)cv * VEC, row = (int64_t)W * C;
    const int64_t off[4] = {p0, p0 + C, p0 + row, p0 + row + C};
    float m[VEC];
    {
      const V a = *reinterpret_cast<const V*>(x + off[0]);
#pragma unroll
      for (int q = 0; q < VEC; ++q) m[q] = to_f32<T>(a.v[q]);
    }
#pragma unroll
    for (int k = 1; k < 4; ++k) {
      const V a = *reinterpret_cast<const V*>(x + off[k]);
#pragma unroll
      for (int q = 0; q < VEC; ++q) {
        const float v = to_f32<T>(a.v[q]);
        if (pool_takes(v, m[q])) m[q] = v;
      }
    }
    V o;
#pragma unroll
    for (int q = 0; q < VEC; ++q) o.v[q] = from_f32<T>(m[q]);      // exact: m is one of the inputs
    *reinterpret_cast<V*>(y + ((n * Ho + ho) * Wo + wo) * C + (int64_t)cv * VEC) = o;
  }
}

// one thread per (window, VEC channels) over ceil(H/2) x ceil(W/2) windows: the windows past the floor-mode output (odd H / W)
// only write zeros, so gx is written densely without a separate memset
template <typename T, int VEC>
__global__ void __launch_bounds__(256) maxpool2x2_backward_kernel(const T* __restrict__ gy, const T* __restrict__ x, T* __restrict__ gx,
                                                                  int N, int H, int W, int C) {
  pdl_wait();
  pdl_launch_dependents();
  using V = VecT<T, VEC>;
  const int Ho = H >> 1, Wo = W >> 1, Hw = (H + 1) >> 1, Ww = (W + 1) >> 1, Cv = C / VEC;
  const int64_t total = (int64_t)N * Hw * Ww * Cv;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    int64_t r = i;
    const int cv = (int)(r % Cv); r /= Cv;
    const int ww = (int)(r % Ww); r /= Ww;
    const int hh = (int)(r % Hw);
    const int64_t n = r / Hw;
    const bool pooled = hh < Ho && ww < Wo;
    const int64_t p0 = ((n * H + 2 * hh) * W + 2 * ww) * C + (int64_t)cv * VEC, row = (int64_t)W * C;
    const int64_t off[4] = {p0, p0 + C, p0 + row, p0 + row + C};
    float g[VEC];
    int arg[VEC];
#pragma unroll
    for (int q = 0; q < VEC; ++q) { g[q] = 0.f; arg[q] = -1; }
    if (pooled) {
      const V gv = *reinterpret_cast<const V*>(gy + ((n * Ho + hh) * Wo + ww) * C + (int64_t)cv * VEC);
      float m[VEC] = {};
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const V a = *reinterpret_cast<const V*>(x + off[k]);
#pragma unroll
        for (int q = 0; q < VEC; ++q) {
          const float v = to_f32<T>(a.v[q]);
          if (k == 0 || pool_takes(v, m[q])) { m[q] = v; arg[q] = k; }
        }
      }
#pragma unroll
      for (int q = 0; q < VEC; ++q) g[q] = m[q] <= 0.f ? 0.f : to_f32<T>(gv.v[q]);   // ReLU mask of the pooled conv (torch's threshold_backward)
    }
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      if (2 * hh + (k >> 1) >= H || 2 * ww + (k & 1) >= W) continue;
      V o;
#pragma unroll
      for (int q = 0; q < VEC; ++q) o.v[q] = from_f32<T>(arg[q] == k ? g[q] : 0.f);
      *reinterpret_cast<V*>(gx + off[k]) = o;
    }
  }
}

}  // namespace mv2

// ==========================================================================================
// C ABI
// ==========================================================================================
using namespace mv2;

// a softmax attention kernel, or its dropout twin when d is given
static void launch_attn_k(void (*plain)(mv2_attn_args), void (*drop)(mv2_attn_args, AttnDrop), dim3 grid, dim3 block,
                          cudaStream_t st, const mv2_attn_args* a, const AttnDrop* d) {
  if (d) launch_k(drop, grid, block, 0, st, *a, *d);
  else launch_k(plain, grid, block, 0, st, *a);
}

template <typename T>
static int launch_attention(const mv2_attn_args* a, const AttnDrop* d, cudaStream_t st) {
  dim3 grid((unsigned)((int64_t)a->n_outer * a->n_inner), a->heads, ceil_div(a->L, AT_Q));
  switch (a->dim_head / 32) {
    case 1: launch_attn_k(attention_kernel<T, 1>, attention_dropout_kernel<T, 1>, grid, dim3(128), st, a, d); break;
    case 2: launch_attn_k(attention_kernel<T, 2>, attention_dropout_kernel<T, 2>, grid, dim3(128), st, a, d); break;
    case 3: launch_attn_k(attention_kernel<T, 3>, attention_dropout_kernel<T, 3>, grid, dim3(128), st, a, d); break;
    default: set_error("dim_head %d unsupported", a->dim_head); return MV2_E_UNSUPPORTED;
  }
  MV2_CHECK_LAUNCH();
  return MV2_OK;
}

// kernel choice of the 16-bit dtypes (T = __nv_bfloat16 or __half)
template <typename T>
static int attention_dispatch16(const mv2_attn_args* a, const AttnDrop* d, cudaStream_t st) {
  if (!a->causal && a->L >= 64 && (a->dim_head == 32 || a->dim_head == 64) && a->heads * a->dim_head % 8 == 0) {
    dim3 grid((unsigned)((int64_t)a->n_outer * a->n_inner), a->heads, ceil_div(a->L, FA_Q));
    using K = AttnK16<T>;
    if (a->dim_head == 32) launch_attn_k(K::template mma<32>(), K::template mma_drop<32>(), grid, dim3(256), st, a, d);
    else launch_attn_k(K::template mma<64>(), K::template mma_drop<64>(), grid, dim3(256), st, a, d);
    MV2_CHECK_LAUNCH();
    return MV2_OK;
  }
  if (a->L <= AS_L && a->n_mem <= AS_M && (a->dim_head == 32 || a->dim_head == 64)) {
    const int64_t warps = (int64_t)a->n_outer * a->n_inner * a->heads;
    const dim3 grid((unsigned)ceil_div(warps, 8));
    using K = AttnK16<T>;
    if (a->dim_head == 32) launch_attn_k(K::template small<1>(), K::template small_drop<1>(), grid, dim3(256), st, a, d);
    else launch_attn_k(K::template small<2>(), K::template small_drop<2>(), grid, dim3(256), st, a, d);
    MV2_CHECK_LAUNCH();
    return MV2_OK;
  }
  return launch_attention<T>(a, d, st);
}

// mv2_attention's argument checks and kernel choice; d != NULL launches the dropout twins
static int attention_dispatch(const mv2_attn_args* a, const AttnDrop* d, void* stream) {
  MV2_CHECK_ARG(a && a->qkv && a->out && a->mem_kv);
  MV2_CHECK_ARG(a->heads > 0 && a->dim_head > 0 && a->dim_head % 32 == 0 && a->dim_head <= 96);
  MV2_CHECK_ARG(a->n_mem >= 0 && a->n_outer > 0 && a->n_inner > 0 && a->L > 0);
  MV2_CHECK_ARG((int64_t)a->n_outer * a->n_inner <= 2147483647LL && ceil_div(a->L, AT_Q) <= 65535);
  cudaStream_t st = (cudaStream_t)stream;
  if (a->dtype == MV2_F32) return launch_attention<float>(a, d, st);
  if (a->dtype == MV2_BF16) return attention_dispatch16<__nv_bfloat16>(a, d, st);
  if (a->dtype == MV2_F16) return attention_dispatch16<__half>(a, d, st);
  set_error("bad dtype %d", a->dtype);
  return MV2_E_ARG;
}

// mv2_dropout_args -> AttnDrop, after the checks both dropout entry points share
static int attn_drop_from(const mv2_dropout_args* dp, int heads, AttnDrop* out) {
  MV2_CHECK_ARG(dp && dp->p > 0.f && dp->p < 1.f);                 // NaN fails too
  MV2_CHECK_ARG(heads > 0 && heads < 65536 && dp->call < 65536u);  // h | call << 16 is one 32-bit counter word
  out->k0 = (uint32_t)dp->seed;
  out->k1 = (uint32_t)(dp->seed >> 32);
  out->call_hi = dp->call << 16;
  out->thr = (uint32_t)floor((double)dp->p * 4294967296.0);        // < 2^32 for p < 1
  out->scale = (float)(1.0 / (1.0 - (double)dp->p));
  return MV2_OK;
}

// quantiser launches for one max-dims instantiation (MODE 0: LFQ, 1: FSQ); `levels` (FSQ) has d entries, checked by the caller
template <int MODE, int MAXD>
static int launch_quant_forward(const void* x, int dtype, int64_t N, int C, int d, int nc, const float* win, const float* bin,
                                const float* wout, const float* bout, float clamp, int spherical, const int32_t* levels,
                                int64_t* idx64, int32_t* idx32, void* quantized, float* aux, cudaStream_t st) {
  FsqLevelsT<MAXD> lv = {};
  for (int i = 0; levels && i < d; ++i) lv.lv[i] = levels[i];
  const int blocks = ceil_div(N, 8);
  if (dtype == MV2_F32)
    launch_k(quant_forward_kernel<float, MODE, MAXD>, dim3(blocks), dim3(256), 0, st, (const float*)x, N, C, d, nc, win, bin, wout, bout,
             clamp, spherical, lv, idx64, idx32, (float*)quantized, aux);
  else if (dtype == MV2_BF16)
    launch_k(quant_forward_kernel<__nv_bfloat16, MODE, MAXD>, dim3(blocks), dim3(256), 0, st, (const __nv_bfloat16*)x, N, C, d, nc, win,
             bin, wout, bout, clamp, spherical, lv, idx64, idx32, (__nv_bfloat16*)quantized, aux);
  else if (dtype == MV2_F16)
    launch_k(quant_forward_kernel<__half, MODE, MAXD>, dim3(blocks), dim3(256), 0, st, (const __half*)x, N, C, d, nc, win,
             bin, wout, bout, clamp, spherical, lv, idx64, idx32, (__half*)quantized, aux);
  else { set_error("bad dtype %d", dtype); return MV2_E_ARG; }
  MV2_CHECK_LAUNCH();
  return MV2_OK;
}

template <int MODE, int MAXD>
static int launch_quant_decode(const void* indices, int is64, int64_t N, int C, int d, int nc, const int32_t* levels,
                               const float* wout, const float* bout, void* quantized, int dtype, cudaStream_t st) {
  FsqLevelsT<MAXD> lv = {};
  for (int i = 0; levels && i < d; ++i) lv.lv[i] = levels[i];
  const int blocks = ceil_div(N, 8);
  if (dtype == MV2_F32)
    launch_k(quant_decode_kernel<float, MODE, MAXD>, dim3(blocks), dim3(256), 0, st, indices, is64, N, C, d, nc, lv, wout, bout,
             (float*)quantized);
  else if (dtype == MV2_BF16)
    launch_k(quant_decode_kernel<__nv_bfloat16, MODE, MAXD>, dim3(blocks), dim3(256), 0, st, indices, is64, N, C, d, nc, lv, wout, bout,
             (__nv_bfloat16*)quantized);
  else if (dtype == MV2_F16)
    launch_k(quant_decode_kernel<__half, MODE, MAXD>, dim3(blocks), dim3(256), 0, st, indices, is64, N, C, d, nc, lv, wout, bout,
             (__half*)quantized);
  else { set_error("bad dtype %d", dtype); return MV2_E_ARG; }
  MV2_CHECK_LAUNCH();
  return MV2_OK;
}

extern "C" {

int mv2_abi_version(void) { return MV2_ABI_VERSION; }
const char* mv2_last_error(void) { return mv2::g_err; }
uint64_t mv2_launch_count(void) { return mv2::g_launches; }

int mv2_set_pdl(int on) {
  const int prev = mv2::g_pdl;
  mv2::g_pdl = on ? 1 : 0;
  return prev;
}

int mv2_device_arch(void) {
  int dev = 0, major = 0, minor = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) { set_error("cudaGetDevice failed"); return MV2_E_CUDA; }
  cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, dev);
  cudaDeviceGetAttribute(&minor, cudaDevAttrComputeCapabilityMinor, dev);
  return major * 10 + minor;
}

int mv2_to_channels_last(const void* src, int src_dtype, void* dst, int dst_dtype, int B, int C, int T, int H, int W,
                         int t_pad, void* stream) {
  MV2_CHECK_ARG(src && dst && B > 0 && C > 0 && T > 0 && H > 0 && W > 0 && t_pad >= 0);
  cudaStream_t st = (cudaStream_t)stream;
  const int64_t HW = (int64_t)H * W, S = (int64_t)T * HW, Sd = (int64_t)(T + t_pad) * HW;
  const size_t es = dst_dtype == MV2_F32 ? 4 : 2;
  if (t_pad > 0)
    MV2_CHECK_CUDA(cudaMemset2DAsync(dst, (size_t)Sd * C * es, 0, (size_t)t_pad * HW * C * es, B, st));
  return dispatch_transpose(src, src_dtype, dst, dst_dtype, B, C, S, S, Sd, 0, (int64_t)t_pad * HW, true, st);
}

int mv2_to_channels_first(const void* src, int src_dtype, void* dst, int dst_dtype, int B, int C, int T, int H, int W,
                          int t_crop, void* stream) {
  MV2_CHECK_ARG(src && dst && B > 0 && C > 0 && T > t_crop && H > 0 && W > 0 && t_crop >= 0);
  cudaStream_t st = (cudaStream_t)stream;
  const int64_t HW = (int64_t)H * W, Ss = (int64_t)T * HW, S = (int64_t)(T - t_crop) * HW;
  return dispatch_transpose(src, src_dtype, dst, dst_dtype, B, C, S, Ss, S, (int64_t)t_crop * HW, 0, false, st);
}

int mv2_ingest_kwpack(const void* src, int src_dtype, void* dst, int B, int C, int T, int H, int W, int t_pad, int kw,
                      int pw, int cpack, void* stream) {
  MV2_CHECK_ARG(src && dst && B > 0 && C > 0 && T > 0 && H > 0 && W > 0 && t_pad >= 0 && kw > 0);
  MV2_CHECK_ARG(cpack % 8 == 0 && kw * C <= cpack);
  const int64_t rows = (int64_t)B * (T + t_pad) * H;
  const size_t smem = (size_t)C * (W + kw - 1) * sizeof(float);
  MV2_CHECK_ARG(rows <= 2147483647LL && smem <= 48 * 1024);
  const int blocks = (int)rows;
  cudaStream_t st = (cudaStream_t)stream;
  if (src_dtype & MV2_KWPACK_F32_DST) {        // fp32 destination: the TF32 conv_in
    src_dtype &= ~MV2_KWPACK_F32_DST;
    if (src_dtype == MV2_F32)
      launch_k(ingest_kwpack_kernel<float, float>, dim3(blocks), dim3(256), smem, st, (const float*)src, (float*)dst, B, C, T, H, W, t_pad, kw, pw, cpack);
    else if (src_dtype == MV2_BF16)
      launch_k(ingest_kwpack_kernel<__nv_bfloat16, float>, dim3(blocks), dim3(256), smem, st, (const __nv_bfloat16*)src, (float*)dst, B, C, T, H, W, t_pad, kw, pw, cpack);
    else if (src_dtype == MV2_U8)
      launch_k(ingest_kwpack_kernel<uint8_t, float>, dim3(blocks), dim3(256), smem, st, (const uint8_t*)src, (float*)dst, B, C, T, H, W, t_pad, kw, pw, cpack);
    else { set_error("bad dtype %d", src_dtype); return MV2_E_ARG; }
  } else if (src_dtype == MV2_F32)
    launch_k(ingest_kwpack_kernel<float, __nv_bfloat16>, dim3(blocks), dim3(256), smem, st, (const float*)src, (__nv_bfloat16*)dst, B, C, T, H, W, t_pad, kw, pw, cpack);
  else if (src_dtype == MV2_BF16)
    launch_k(ingest_kwpack_kernel<__nv_bfloat16, __nv_bfloat16>, dim3(blocks), dim3(256), smem, st, (const __nv_bfloat16*)src, (__nv_bfloat16*)dst, B, C, T, H, W, t_pad, kw, pw, cpack);
  else if (src_dtype == MV2_F16)
    launch_k(ingest_kwpack_kernel<__half, __half>, dim3(blocks), dim3(256), smem, st, (const __half*)src, (__half*)dst, B, C, T, H, W, t_pad, kw, pw, cpack);
  else if (src_dtype == MV2_U8)
    launch_k(ingest_kwpack_kernel<uint8_t, __nv_bfloat16>, dim3(blocks), dim3(256), smem, st, (const uint8_t*)src, (__nv_bfloat16*)dst, B, C, T, H, W, t_pad, kw, pw, cpack);
  else { set_error("bad dtype %d", src_dtype); return MV2_E_ARG; }
  MV2_CHECK_LAUNCH();
  return MV2_OK;
}

int mv2_conv_forward(const mv2_conv_args* a, const mv2_conv_hist* hist, void* stream) {
  const mv2_conv_hist none = {nullptr, 0, 0};
  if (!hist) hist = &none;
  MV2_CHECK_ARG(a && a->x && a->w && a->y && hist->T_h >= 0 && (hist->T_h == 0 || hist->h));
  MV2_CHECK_ARG(a->B > 0 && a->Ti > 0 && a->Hi > 0 && a->Wi > 0 && a->Ci > 0);
  MV2_CHECK_ARG(a->To > 0 && a->Ho > 0 && a->Wo > 0 && a->Co > 0);
  MV2_CHECK_ARG(a->kt > 0 && a->kh > 0 && a->kw > 0 && a->st > 0 && a->sh > 0 && a->sw > 0);
  MV2_CHECK_ARG(a->shuffle != MV2_SHUFFLE_SPACE || a->Co % 4 == 0);
  MV2_CHECK_ARG(a->shuffle != MV2_SHUFFLE_TIME || a->Co % 2 == 0);
  const int64_t M = (int64_t)a->B * a->To * a->Ho * a->Wo;
  dim3 grid(ceil_div(M, CBM), ceil_div(a->Co, CBN));
  cudaStream_t st = (cudaStream_t)stream;
  if (a->dtype == MV2_F32) launch_k(conv_simt_kernel<float>, dim3(grid), dim3(256), 0, st, *a, *hist);
  else if (a->dtype == MV2_BF16) launch_k(conv_simt_kernel<__nv_bfloat16>, dim3(grid), dim3(256), 0, st, *a, *hist);
  else if (a->dtype == MV2_F16) launch_k(conv_simt_kernel<__half>, dim3(grid), dim3(256), 0, st, *a, *hist);
  else { set_error("bad dtype %d", a->dtype); return MV2_E_ARG; }
  MV2_CHECK_LAUNCH();
  return MV2_OK;
}

size_t mv2_se_workspace_bytes(int F, int P, int C) {
  // chunk partials + room for the SE hidden layer (at most max(16, C/2) <= C + 16 units per frame)
  return ((size_t)F * ceil_div(P, SE_MIN_ROWS) * (C + 2) + (size_t)F * (C + 16)) * sizeof(float);
}

// the single-pass bf16 kernel processes SE_CHUNK * se_chunk_mult(P) rows per block but keeps the workspace stride of
// ceil(P / SE_CHUNK) records per frame (only the first ceil(P / rows) records are written; unused ones are skipped by
// passing the matching chunk count to se_hidden_kernel)
static int se_online_vec(int C) {
  for (int vec = 8; vec <= 32; vec <<= 1) {
    const int G = C / vec;
    if (C % vec == 0 && G >= 1 && G <= 32 && (G & (G - 1)) == 0) return vec;
  }
  return 0;
}
static int se_rows_per_block(int dtype, int F, int P, int C) {
  (void)F;   // deliberately NOT a function of the frame count: the chunking fixes the summation order of the pooled vector, and
             // a clip's tokens must not depend on how many other clips share its batch (tests: ..._batch_independence)
  if (!((dtype == MV2_BF16 || dtype == MV2_F16) && se_online_vec(C) != 0)) return SE_CHUNK;
  // small (L2-resident) frames take 64 - 128-row chunks: fewer, longer bulk-copy pipelines and fewer records to merge than
  // 32-row chunks; large frames amortise the per-block merge over longer chunks
  if (P <= 256) return 64;
  if (P <= 1024) return 128;
  if (P <= 4096) return 512;
  return 2048;
}

static cudaError_t se_pool_smem_optin() {
  static PerDeviceOnce once;
  return once.run([] {
    cudaError_t err = cudaSuccess;
    auto set = [&](const void* fn) { if (err == cudaSuccess) err = cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, 96 * 1024); };
    auto set_all = [&](auto tag) {
      using T = decltype(tag);
      set((const void*)se_pool_online_kernel<T, 8, 1>); set((const void*)se_pool_online_kernel<T, 8, 2>); set((const void*)se_pool_online_kernel<T, 8, 4>);
      set((const void*)se_pool_online_kernel<T, 8, 8>); set((const void*)se_pool_online_kernel<T, 8, 16>); set((const void*)se_pool_online_kernel<T, 8, 32>);
      set((const void*)se_pool_online_kernel<T, 16, 32>); set((const void*)se_pool_online_kernel<T, 32, 32>);
    };
    set_all(__nv_bfloat16());
    set_all(__half());
    return err;
  });
}

extern "C++" {
// the single-pass kernel of a 16-bit y (T = __nv_bfloat16 or __half)
template <typename T>
static int se_pool_online_launch(const void* y, int P, int C, const float* wk, float bk, void* workspace, dim3 grid, int nc,
                                 int rows, cudaStream_t st) {
  const int vec = se_online_vec(C);
  const int R_ = 256 / (C / vec), U_ = vec == 8 ? 4 : 2;
  // SE_STAGES batches of R * U rows, reused afterwards for R records of (m, s, acc[C]) + R merge coefficients
  const size_t dsm = std::max((size_t)SE_STAGES * R_ * U_ * C * 2, (size_t)R_ * (C + 3) * sizeof(float));
  if (dsm > 96 * 1024) { set_error("se_pool: C = %d needs %zu bytes of shared memory", C, dsm); return MV2_E_ARG; }
  const T* yb = (const T*)y;
  if (const cudaError_t e = se_pool_smem_optin()) { set_error("cudaFuncSetAttribute failed: %s", cudaGetErrorString(e)); return MV2_E_CUDA; }
  const int G_ = C / vec;
#define MV2_SE_POOL_CASE(V, GG) \
  else if (vec == V && G_ == GG) launch_k(se_pool_online_kernel<T, V, GG>, dim3(grid), dim3(256), dsm, st, yb, P, C, wk, bk, (float*)workspace, nc, rows)
  if (false) {}
  MV2_SE_POOL_CASE(8, 1); MV2_SE_POOL_CASE(8, 2); MV2_SE_POOL_CASE(8, 4); MV2_SE_POOL_CASE(8, 8); MV2_SE_POOL_CASE(8, 16);
  MV2_SE_POOL_CASE(8, 32); MV2_SE_POOL_CASE(16, 32); MV2_SE_POOL_CASE(32, 32);
  else { set_error("se_pool: no kernel for C = %d", C); return MV2_E_UNSUPPORTED; }
#undef MV2_SE_POOL_CASE
  MV2_CHECK_LAUNCH();
  return MV2_OK;
}
}  // extern "C++"

int mv2_se_pool(const void* y, int dtype, int F, int P, int C, const float* wk, float bk, void* workspace,
                void* stream) {
  MV2_CHECK_ARG(y && wk && workspace && F > 0 && P > 0 && C > 0);
  const int rows = se_rows_per_block(dtype, F, P, C);
  const int nc = ceil_div(P, rows);
  dim3 grid(nc, F);
  cudaStream_t st = (cudaStream_t)stream;
  if (dtype == MV2_F32) launch_k(se_pool_kernel<float>, dim3(grid), dim3(256), 0, st, (const float*)y, P, C, wk, bk, (float*)workspace, nc);
  else if ((dtype == MV2_BF16 || dtype == MV2_F16) && se_online_vec(C) != 0)
    return dtype == MV2_F16 ? se_pool_online_launch<__half>(y, P, C, wk, bk, workspace, grid, nc, rows, st)
                            : se_pool_online_launch<__nv_bfloat16>(y, P, C, wk, bk, workspace, grid, nc, rows, st);
  else if (dtype == MV2_BF16) launch_k(se_pool_kernel<__nv_bfloat16>, dim3(grid), dim3(256), 0, st, (const __nv_bfloat16*)y, P, C, wk, bk, (float*)workspace, nc);
  else if (dtype == MV2_F16) launch_k(se_pool_kernel<__half>, dim3(grid), dim3(256), 0, st, (const __half*)y, P, C, wk, bk, (float*)workspace, nc);
  else { set_error("bad dtype %d", dtype); return MV2_E_ARG; }
  MV2_CHECK_LAUNCH();
  return MV2_OK;
}

int mv2_se_gate(const void* workspace, int dtype, int F, int P, int C, int Hd, const float* w1, const float* b1,
                const float* w2, const float* b2, float* gates, void* stream) {
  MV2_CHECK_ARG(workspace && w1 && b1 && w2 && b2 && gates && F > 0 && P > 0 && C > 0 && Hd > 0);
  MV2_CHECK_ARG(Hd <= C + 16);     // the hidden layer scratch mv2_se_workspace_bytes reserves: F * (C + 16) floats
  const int nc = ceil_div(P, se_rows_per_block(dtype, F, P, C));   // chunk records se_pool wrote per frame
  const size_t smem1 = (size_t)(C + nc + 256) * sizeof(float), smem2 = (size_t)Hd * sizeof(float);
  MV2_CHECK_ARG(smem1 <= 48 * 1024 && smem2 <= 48 * 1024);
  // hidden activations live behind the chunk partials (mv2_se_workspace_bytes reserves F*Hd_max floats)
  float* hidden = (float*)workspace + (size_t)F * ceil_div(P, SE_MIN_ROWS) * (C + 2);
  cudaStream_t st = (cudaStream_t)stream;
  launch_k(se_hidden_kernel<false>, dim3(dim3(F, ceil_div(Hd, 32))), dim3(256), smem1, st, (const float*)workspace, nc, C, Hd, w1, b1, hidden);
  MV2_CHECK_LAUNCH();
  launch_k(se_out_kernel, dim3(dim3(F, ceil_div(C, 64))), dim3(256), smem2, st, hidden, C, Hd, w2, b2, gates);
  MV2_CHECK_LAUNCH();
  return MV2_OK;
}

int mv2_se_gate_records(const void* workspace, int nrec, int F, int C, int Hd, const float* w1, const float* b1,
                        const float* w2, const float* b2, float* gates, void* stream) {
  MV2_CHECK_ARG(workspace && w1 && b1 && w2 && b2 && gates && F > 0 && nrec > 0 && C > 0 && Hd > 0);
  MV2_CHECK_ARG(Hd <= C + 16);     // the hidden layer scratch mv2_tc_ru_workspace_bytes reserves: F * (C + 16) floats
  const size_t smem1 = (size_t)(C + nrec + 256) * sizeof(float), smem2 = (size_t)Hd * sizeof(float);
  MV2_CHECK_ARG(smem1 <= 48 * 1024 && smem2 <= 48 * 1024);
  float* hidden = (float*)workspace + (size_t)F * nrec * (C + 2);
  cudaStream_t st = (cudaStream_t)stream;
  if (C <= 128 && (C & (C - 1)) == 0 && nrec > 16)
    launch_k(se_hidden_kernel<true>, dim3(dim3(F, ceil_div(Hd, 32))), dim3(256), smem1, st, (const float*)workspace, nrec, C, Hd, w1, b1, hidden);
  else
    launch_k(se_hidden_kernel<false>, dim3(dim3(F, ceil_div(Hd, 32))), dim3(256), smem1, st, (const float*)workspace, nrec, C, Hd, w1, b1, hidden);
  MV2_CHECK_LAUNCH();
  launch_k(se_out_kernel, dim3(dim3(F, ceil_div(C, 64))), dim3(256), smem2, st, hidden, C, Hd, w2, b2, gates);
  MV2_CHECK_LAUNCH();
  return MV2_OK;
}

int mv2_dense_small(const float* x, const float* w, const float* bias, float* y, int B, int K, int N, int act, void* stream) {
  MV2_CHECK_ARG(x && w && y && B > 0 && K > 0 && N > 0 && B <= 65535);
  launch_k(dense_small_kernel, dim3(ceil_div(N, 8), B), dim3(256), 0, (cudaStream_t)stream, x, w, bias, y, K, N, act);
  MV2_CHECK_LAUNCH();
  return MV2_OK;
}

int mv2_mod_prepare(const float* cond, const float* S, float eps, float* scale_in, float* inv_norm, int B, int Ci, int Co,
                    void* stream) {
  MV2_CHECK_ARG(cond && S && scale_in && inv_norm && B > 0 && Ci > 0 && Co > 0 && B <= 65535);
  launch_k(mod_prepare_kernel, dim3(ceil_div(Co, 8), B), dim3(256), 0, (cudaStream_t)stream, cond, S, eps, scale_in, inv_norm, Ci, Co);
  MV2_CHECK_LAUNCH();
  return MV2_OK;
}

int mv2_scale_channels(const void* x, const float* scale, void* out, int dtype, int B, int64_t positions_per_clip, int C,
                       void* stream) {
  MV2_CHECK_ARG(x && scale && out && B > 0 && positions_per_clip > 0 && C > 0);
  const int64_t per_clip = positions_per_clip * C, total = per_clip * B;
  const int blocks = (int)std::min<int64_t>((total + 255) / 256, grid_cap(32));
  cudaStream_t st = (cudaStream_t)stream;
  if (dtype == MV2_F32) launch_k(scale_channels_kernel<float>, dim3(blocks), dim3(256), 0, st, (const float*)x, scale, (float*)out, total, per_clip, C);
  else if (dtype == MV2_BF16) launch_k(scale_channels_kernel<__nv_bfloat16>, dim3(blocks), dim3(256), 0, st, (const __nv_bfloat16*)x, scale, (__nv_bfloat16*)out, total, per_clip, C);
  else if (dtype == MV2_F16) launch_k(scale_channels_kernel<__half>, dim3(blocks), dim3(256), 0, st, (const __half*)x, scale, (__half*)out, total, per_clip, C);
  else { set_error("bad dtype %d", dtype); return MV2_E_ARG; }
  MV2_CHECK_LAUNCH();
  return MV2_OK;
}

int mv2_copy_frames(const void* src, void* dst, int B, int src_T, int dst_T, int src_t0, int dst_t0, int n_frames,
                    size_t frame_bytes, int zero_front, void* stream) {
  MV2_CHECK_ARG(src && dst && B > 0 && n_frames > 0 && frame_bytes > 0);
  MV2_CHECK_ARG(src_t0 >= 0 && dst_t0 >= 0 && src_t0 + n_frames <= src_T && dst_t0 + n_frames <= dst_T);
  cudaStream_t st = (cudaStream_t)stream;
  if (zero_front && dst_t0 > 0)
    MV2_CHECK_CUDA(cudaMemset2DAsync(dst, (size_t)dst_T * frame_bytes, 0, (size_t)dst_t0 * frame_bytes, B, st));
  MV2_CHECK_CUDA(cudaMemcpy2DAsync((char*)dst + (size_t)dst_t0 * frame_bytes, (size_t)dst_T * frame_bytes,
                                   (const char*)src + (size_t)src_t0 * frame_bytes, (size_t)src_T * frame_bytes,
                                   (size_t)n_frames * frame_bytes, B, cudaMemcpyDeviceToDevice, st));
  return MV2_OK;
}

int mv2_pad_cl(const void* src, void* dst, int dtype, int B, int T, int H, int W, int C, int pt, int ph, int pw, int mode,
               void* stream) {
  MV2_CHECK_ARG(src && dst && B > 0 && T > 0 && H > 0 && W > 0 && C > 0 && pt >= 0 && ph >= 0 && pw >= 0);
  MV2_CHECK_ARG(mode >= 1 && mode <= 3);
  if (mode == 1) MV2_CHECK_ARG(pt < T && ph < H && pw < W);          // torch's reflection padding requires pad < size
  if (mode == 3) MV2_CHECK_ARG(pt <= T && ph <= H && pw <= W);
  const int64_t total = (int64_t)B * (T + pt) * (H + 2 * ph) * (W + 2 * pw) * C;
  const int blocks = (int)std::min<int64_t>((total + 255) / 256, grid_cap(32));
  cudaStream_t st = (cudaStream_t)stream;
  if (dtype == MV2_F32) launch_k(pad_cl_kernel<float>, dim3(blocks), dim3(256), 0, st, (const float*)src, (float*)dst, B, T, H, W, C, pt, ph, pw, mode);
  else if (dtype == MV2_BF16) launch_k(pad_cl_kernel<__nv_bfloat16>, dim3(blocks), dim3(256), 0, st, (const __nv_bfloat16*)src, (__nv_bfloat16*)dst, B, T, H, W, C, pt, ph, pw, mode);
  else if (dtype == MV2_F16) launch_k(pad_cl_kernel<__half>, dim3(blocks), dim3(256), 0, st, (const __half*)src, (__half*)dst, B, T, H, W, C, pt, ph, pw, mode);
  else { set_error("bad dtype %d", dtype); return MV2_E_ARG; }
  MV2_CHECK_LAUNCH();
  return MV2_OK;
}

int mv2_gate_residual(const void* y, const void* x, const float* gates, void* out, int dtype, int F, int P, int C,
                      void* stream) {
  MV2_CHECK_ARG(y && x && gates && out && F > 0 && P > 0 && C > 0);
  const int64_t total = (int64_t)F * P * C;
  const int blocks = (int)std::min<int64_t>((total + 255) / 256, grid_cap(32));
  cudaStream_t st = (cudaStream_t)stream;
  if (dtype == MV2_F32)
    launch_k(gate_residual_kernel<float>, dim3(blocks), dim3(256), 0, st, (const float*)y, (const float*)x, gates, (float*)out, total, (int64_t)P * C, C);
  else if ((dtype == MV2_BF16 || dtype == MV2_F16) && C % 8 == 0) {
    const int64_t total8 = total / 8;
    const int b8 = (int)std::min<int64_t>((total8 + 255) / 256, grid_cap(16));
    launch_k(dtype == MV2_F16 ? gate_residual_x8_kernel<__half> : gate_residual_x8_kernel<__nv_bfloat16>, dim3(b8), dim3(256), 0, st,
             (const uint4*)y, (const uint4*)x, gates, (uint4*)out, total8, (int64_t)P * C / 8, C / 8);
  } else if (dtype == MV2_BF16)
    launch_k(gate_residual_kernel<__nv_bfloat16>, dim3(blocks), dim3(256), 0, st, (const __nv_bfloat16*)y, (const __nv_bfloat16*)x, gates, (__nv_bfloat16*)out, total, (int64_t)P * C, C);
  else if (dtype == MV2_F16)
    launch_k(gate_residual_kernel<__half>, dim3(blocks), dim3(256), 0, st, (const __half*)y, (const __half*)x, gates, (__half*)out, total, (int64_t)P * C, C);
  else { set_error("bad dtype %d", dtype); return MV2_E_ARG; }
  MV2_CHECK_LAUNCH();
  return MV2_OK;
}

extern "C++" {
// the one-warp-per-token kernel of a 16-bit x (T = __nv_bfloat16 or __half), C % 8 == 0, C <= 1024
template <typename T>
static void rmsnorm_x8_launch(const void* x, void* out, const float* gamma, int64_t n_tok, int Tn, int P, int C, int token_shift,
                              const void* prev, int64_t prev_stride, cudaStream_t st) {
  const T* xb = (const T*)x;
  T* ob = (T*)out;
  const T* pb = (const T*)prev;
  // one token per warp up to C = 512 keeps the most warps in flight on the small README shapes; the widest rows take 4
  if (C <= 256) launch_k(rmsnorm_x8_kernel<T, 1, 1>, dim3(ceil_div(n_tok, 8 * 1)), dim3(256), 0, st, xb, ob, gamma, n_tok, Tn, P, C, token_shift, pb, prev_stride);
  else if (C <= 512) launch_k(rmsnorm_x8_kernel<T, 2, 1>, dim3(ceil_div(n_tok, 8 * 1)), dim3(256), 0, st, xb, ob, gamma, n_tok, Tn, P, C, token_shift, pb, prev_stride);
  else launch_k(rmsnorm_x8_kernel<T, 4, 4>, dim3(ceil_div(n_tok, 8 * 4)), dim3(256), 0, st, xb, ob, gamma, n_tok, Tn, P, C, token_shift, pb, prev_stride);
}
}  // extern "C++"

static int rmsnorm_launch(const void* x, void* out, int dtype, const float* gamma, int B, int T, int P, int C, int token_shift,
                          const void* prev, int64_t prev_stride, void* stream) {
  MV2_CHECK_ARG(x && out && gamma && B > 0 && T > 0 && P > 0 && C > 0);
  const int64_t n_tok = (int64_t)B * T * P;
  const int blocks = ceil_div(n_tok, 8);
  cudaStream_t st = (cudaStream_t)stream;
  if (dtype == MV2_F32)
    launch_k(rmsnorm_kernel<float>, dim3(blocks), dim3(256), 0, st, (const float*)x, (float*)out, gamma, n_tok, T, P, C, token_shift, (const float*)prev, prev_stride);
  else if ((dtype == MV2_BF16 || dtype == MV2_F16) && C % 8 == 0 && C <= 1024 && (!token_shift || (C / 2) % 8 == 0)) {
    if (dtype == MV2_F16) rmsnorm_x8_launch<__half>(x, out, gamma, n_tok, T, P, C, token_shift, prev, prev_stride, st);
    else rmsnorm_x8_launch<__nv_bfloat16>(x, out, gamma, n_tok, T, P, C, token_shift, prev, prev_stride, st);
  }
  else if (dtype == MV2_BF16)
    launch_k(rmsnorm_kernel<__nv_bfloat16>, dim3(blocks), dim3(256), 0, st, (const __nv_bfloat16*)x, (__nv_bfloat16*)out, gamma, n_tok, T, P, C, token_shift, (const __nv_bfloat16*)prev, prev_stride);
  else if (dtype == MV2_F16)
    launch_k(rmsnorm_kernel<__half>, dim3(blocks), dim3(256), 0, st, (const __half*)x, (__half*)out, gamma, n_tok, T, P, C, token_shift, (const __half*)prev, prev_stride);
  else { set_error("bad dtype %d", dtype); return MV2_E_ARG; }
  MV2_CHECK_LAUNCH();
  return MV2_OK;
}

int mv2_rmsnorm(const void* x, void* out, int dtype, const float* gamma, int B, int T, int P, int C, int token_shift,
                void* stream) {
  return rmsnorm_launch(x, out, dtype, gamma, B, T, P, C, token_shift, nullptr, 0, stream);
}

int mv2_rmsnorm_prev(const void* x, const void* prev, int64_t prev_clip_stride, void* out, int dtype, const float* gamma,
                     int B, int T, int P, int C, void* stream) {
  MV2_CHECK_ARG(prev && prev_clip_stride >= (int64_t)P * C);
  return rmsnorm_launch(x, out, dtype, gamma, B, T, P, C, 1, prev, prev_clip_stride, stream);
}

int mv2_attention(const mv2_attn_args* a, void* stream) { return attention_dispatch(a, nullptr, stream); }

// the kernel mv2_attention picks for a causal call of this L (the tensor-core kernel is non-causal only), on rows [q_begin, L)
int mv2_attention_tail(const mv2_attn_args* a, const void* q, int64_t q_outer_stride, int q_begin, void* out,
                       int64_t out_outer_stride, void* stream) {
  MV2_CHECK_ARG(a && a->qkv && q && out && a->mem_kv && a->causal && q_outer_stride >= 0);
  MV2_CHECK_ARG(a->heads > 0 && a->dim_head > 0 && a->dim_head % 32 == 0 && a->dim_head <= 96);
  MV2_CHECK_ARG(a->n_mem >= 0 && a->n_outer > 0 && a->n_inner > 0 && a->L > 0 && q_begin >= 0 && q_begin < a->L);
  MV2_CHECK_ARG(out_outer_stride >= 0 && (int64_t)a->n_outer * a->n_inner <= 2147483647LL);
  const AttnTail tl{q_begin, out_outer_stride, q, q_outer_stride};
  mv2_attn_args o = *a;
  o.out = out;
  cudaStream_t st = (cudaStream_t)stream;
  const int dpl = a->dim_head / 32;
  if (a->dtype != MV2_F32 && a->dtype != MV2_BF16 && a->dtype != MV2_F16) { set_error("bad dtype %d", a->dtype); return MV2_E_ARG; }
  auto go = [&](auto tag) {
    using T = decltype(tag);
    if (!std::is_same<T, float>::value && a->L <= AS_L && a->n_mem <= AS_M && (dpl == 1 || dpl == 2)) {
      using T16 = typename std::conditional<std::is_same<T, float>::value, __nv_bfloat16, T>::type;
      const dim3 grid((unsigned)ceil_div((int64_t)a->n_outer * a->n_inner * a->heads, 8));
      if (dpl == 1) launch_k(AttnK16<T16>::template small_tail<1>(), grid, dim3(256), 0, st, o, tl);
      else launch_k(AttnK16<T16>::template small_tail<2>(), grid, dim3(256), 0, st, o, tl);
    } else {
      const dim3 grid((unsigned)((int64_t)a->n_outer * a->n_inner), a->heads, ceil_div(a->L - q_begin, AT_Q));
      if (dpl == 1) launch_k(attention_tail_kernel<T, 1>, grid, dim3(128), 0, st, o, tl);
      else if (dpl == 2) launch_k(attention_tail_kernel<T, 2>, grid, dim3(128), 0, st, o, tl);
      else launch_k(attention_tail_kernel<T, 3>, grid, dim3(128), 0, st, o, tl);
    }
  };
  if (a->dtype == MV2_F32) go(float());
  else if (a->dtype == MV2_BF16) go(__nv_bfloat16());
  else go(__half());
  MV2_CHECK_LAUNCH();
  return MV2_OK;
}

int mv2_attention_dropout(const mv2_attn_args* a, const mv2_dropout_args* dp, void* stream) {
  MV2_CHECK_ARG(a);
  AttnDrop d;
  const int rc = attn_drop_from(dp, a->heads, &d);
  if (rc != MV2_OK) return rc;
  return attention_dispatch(a, &d, stream);
}

int mv2_attention_dropout_mask(int n_seq, int heads, int L, int n_mem, const mv2_dropout_args* dp, uint8_t* keep, void* stream) {
  MV2_CHECK_ARG(keep && n_seq > 0 && L > 0 && n_mem >= 0);
  AttnDrop d;
  const int rc = attn_drop_from(dp, heads, &d);
  if (rc != MV2_OK) return rc;
  const int Ltot = n_mem + L;
  const int64_t n_groups = (int64_t)n_seq * heads * L * ((Ltot + 3) / 4);
  const int blocks = (int)std::min<int64_t>((n_groups + 255) / 256, 1 << 20);
  launch_k(attention_dropout_mask_kernel, dim3(blocks), dim3(256), 0, (cudaStream_t)stream, n_groups, heads, L, Ltot, d, keep);
  MV2_CHECK_LAUNCH();
  return MV2_OK;
}

size_t mv2_linattn_workspace_bytes(int n_seq, int heads, int L) {
  // per-chunk fp32 partial states + the finalised bf16 hi/lo MMA operand of every (sequence, head)
  const size_t part_bytes = ((size_t)n_seq * heads * ceil_div(L, LA_CHUNK) * LA_ST * sizeof(float) + 15) / 16 * 16;
  return part_bytes + (size_t)n_seq * heads * 2 * LAM_SW * 2;
}

int mv2_linear_attention(const void* q, const void* kv, void* out, int dtype, int n_seq, int L, int heads,
                         int dim_head, void* workspace, void* stream) {
  MV2_CHECK_ARG(q && kv && out && workspace && n_seq > 0 && L > 0 && heads > 0);
  if (dim_head != LA_D) { set_error("linear attention dim_head %d unsupported (only 8)", dim_head); return MV2_E_UNSUPPORTED; }
  const int nc = ceil_div(L, LA_CHUNK);
  dim3 grid(nc, heads, n_seq);
  cudaStream_t st = (cudaStream_t)stream;
  if (dtype == MV2_F32) {
    launch_k(linattn_reduce_kernel<float>, dim3(grid), dim3(256), 0, st, (const float*)kv, (float*)workspace, L, heads, nc);
    MV2_CHECK_LAUNCH();
    launch_k(linattn_apply_kernel<float>, dim3(grid), dim3(64), 0, st, (const float*)q, (const float*)workspace, (float*)out, L, heads, nc);
  } else if ((dtype == MV2_BF16 || dtype == MV2_F16) && (heads * LA_D) % 8 == 0) {
    const bool f16 = dtype == MV2_F16;
    {
      static PerDeviceOnce once;
      MV2_CHECK_CUDA(once.run([] {
        cudaError_t e = cudaFuncSetAttribute(linattn_reduce_mma_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)LAM_REDUCE_SMEM);
        if (e == cudaSuccess)
          e = cudaFuncSetAttribute(linattn_reduce_mma_f16_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)LAM_REDUCE_SMEM_F16);
        return e;
      }));
    }
    if (f16)
      launch_k(linattn_reduce_mma_f16_kernel, dim3(grid), dim3(128), LAM_REDUCE_SMEM_F16, st, (const __half*)kv, (float*)workspace, L, heads, nc);
    else
      launch_k(linattn_reduce_mma_kernel, dim3(grid), dim3(128), LAM_REDUCE_SMEM, st, (const __nv_bfloat16*)kv, (float*)workspace, L, heads, nc);
    MV2_CHECK_LAUNCH();
    const size_t part_bytes = ((size_t)n_seq * heads * nc * LA_ST * sizeof(float) + 15) / 16 * 16;
    __nv_bfloat16* sw = reinterpret_cast<__nv_bfloat16*>((char*)workspace + part_bytes);
    launch_k(linattn_finalize_kernel, dim3(heads, n_seq), dim3(128), 0, st, (const float*)workspace, sw, heads, nc);
    MV2_CHECK_LAUNCH();
    dim3 grid2(ceil_div(L, LAM_AT * LAM_AB), heads, n_seq);
    if (f16)
      launch_k(linattn_apply_mma_f16_kernel, dim3(grid2), dim3(64), 0, st, (const __half*)q, (const __nv_bfloat16*)sw, (__half*)out, L, heads);
    else
      launch_k(linattn_apply_mma_kernel, dim3(grid2), dim3(64), 0, st, (const __nv_bfloat16*)q, (const __nv_bfloat16*)sw, (__nv_bfloat16*)out, L, heads);
  } else if (dtype == MV2_BF16) {
    launch_k(linattn_reduce_kernel<__nv_bfloat16>, dim3(grid), dim3(256), 0, st, (const __nv_bfloat16*)kv, (float*)workspace, L, heads, nc);
    MV2_CHECK_LAUNCH();
    launch_k(linattn_apply_kernel<__nv_bfloat16>, dim3(grid), dim3(64), 0, st, (const __nv_bfloat16*)q, (const float*)workspace, (__nv_bfloat16*)out, L, heads, nc);
  } else if (dtype == MV2_F16) {
    launch_k(linattn_reduce_kernel<__half>, dim3(grid), dim3(256), 0, st, (const __half*)kv, (float*)workspace, L, heads, nc);
    MV2_CHECK_LAUNCH();
    launch_k(linattn_apply_kernel<__half>, dim3(grid), dim3(64), 0, st, (const __half*)q, (const float*)workspace, (__half*)out, L, heads, nc);
  } else { set_error("bad dtype %d", dtype); return MV2_E_ARG; }
  MV2_CHECK_LAUNCH();
  return MV2_OK;
}

int mv2_geglu(const void* in, void* out, int dtype, int64_t N, int I, void* stream) {
  MV2_CHECK_ARG(in && out && N > 0 && I > 0);
  const int64_t total = N * I;
  const int blocks = (int)std::min<int64_t>((total + 255) / 256, grid_cap(32));
  cudaStream_t st = (cudaStream_t)stream;
  if (dtype == MV2_F32) launch_k(geglu_kernel<float>, dim3(blocks), dim3(256), 0, st, (const float*)in, (float*)out, N, I);
  else if (dtype == MV2_BF16) launch_k(geglu_kernel<__nv_bfloat16>, dim3(blocks), dim3(256), 0, st, (const __nv_bfloat16*)in, (__nv_bfloat16*)out, N, I);
  else if (dtype == MV2_F16) launch_k(geglu_kernel<__half>, dim3(blocks), dim3(256), 0, st, (const __half*)in, (__half*)out, N, I);
  else { set_error("bad dtype %d", dtype); return MV2_E_ARG; }
  MV2_CHECK_LAUNCH();
  return MV2_OK;
}

int mv2_lfq_forward(const void* x, int dtype, int64_t N, int C, int d, int num_codebooks, const float* win, const float* bin,
                    const float* wout, const float* bout, float clamp, int spherical, int64_t* indices, void* quantized,
                    float* presign, void* stream) {
  const int nc = num_codebooks;
  MV2_CHECK_ARG(x && win && bin && N > 0 && C > 0 && d > 0 && nc > 0 && d * nc <= Q_MAXD_WIDE);
  MV2_CHECK_ARG(!quantized || (wout && bout));
  return d * nc <= Q_MAXD ? launch_quant_forward<0, Q_MAXD>(x, dtype, N, C, d, nc, win, bin, wout, bout, clamp, spherical, nullptr,
                                                            indices, nullptr, quantized, presign, (cudaStream_t)stream)
                          : launch_quant_forward<0, Q_MAXD_WIDE>(x, dtype, N, C, d, nc, win, bin, wout, bout, clamp, spherical, nullptr,
                                                                 indices, nullptr, quantized, presign, (cudaStream_t)stream);
}

int mv2_lfq_decode(const void* indices, int index_is_i64, int64_t N, int C, int d, int num_codebooks, const float* wout,
                   const float* bout, void* quantized, int dtype, void* stream) {
  const int nc = num_codebooks;
  MV2_CHECK_ARG(indices && wout && bout && quantized && N > 0 && C > 0 && d > 0 && nc > 0 && d * nc <= Q_MAXD_WIDE);
  return d * nc <= Q_MAXD ? launch_quant_decode<0, Q_MAXD>(indices, index_is_i64, N, C, d, nc, nullptr, wout, bout, quantized, dtype,
                                                           (cudaStream_t)stream)
                          : launch_quant_decode<0, Q_MAXD_WIDE>(indices, index_is_i64, N, C, d, nc, nullptr, wout, bout, quantized, dtype,
                                                                (cudaStream_t)stream);
}

int mv2_fsq_forward(const void* x, int dtype, int64_t N, int C, int d, int num_codebooks, const int32_t* levels, const float* win,
                    const float* bin, const float* wout, const float* bout, int32_t* indices, void* quantized,
                    float* bounded, void* stream) {
  const int nc = num_codebooks;
  MV2_CHECK_ARG(x && levels && win && bin && N > 0 && C > 0 && d > 0 && nc > 0 && d * nc <= Q_MAXD_WIDE);
  MV2_CHECK_ARG(!quantized || (wout && bout));
  for (int i = 0; i < d; ++i) MV2_CHECK_ARG(levels[i] >= 2);
  return d * nc <= Q_MAXD ? launch_quant_forward<1, Q_MAXD>(x, dtype, N, C, d, nc, win, bin, wout, bout, 0.f, 0, levels, nullptr,
                                                            indices, quantized, bounded, (cudaStream_t)stream)
                          : launch_quant_forward<1, Q_MAXD_WIDE>(x, dtype, N, C, d, nc, win, bin, wout, bout, 0.f, 0, levels, nullptr,
                                                                 indices, quantized, bounded, (cudaStream_t)stream);
}

int mv2_fsq_decode(const void* indices, int index_is_i64, int64_t N, int C, int d, int num_codebooks, const int32_t* levels,
                   const float* wout, const float* bout, void* quantized, int dtype, void* stream) {
  const int nc = num_codebooks;
  MV2_CHECK_ARG(indices && levels && wout && bout && quantized && N > 0 && C > 0 && d > 0 && nc > 0 && d * nc <= Q_MAXD_WIDE);
  for (int i = 0; i < d; ++i) MV2_CHECK_ARG(levels[i] >= 2);
  return d * nc <= Q_MAXD ? launch_quant_decode<1, Q_MAXD>(indices, index_is_i64, N, C, d, nc, levels, wout, bout, quantized, dtype,
                                                           (cudaStream_t)stream)
                          : launch_quant_decode<1, Q_MAXD_WIDE>(indices, index_is_i64, N, C, d, nc, levels, wout, bout, quantized, dtype,
                                                                (cudaStream_t)stream);
}

int mv2_lfq_entropy_partials(const float* presign, int64_t N, int d, int num_codebooks, float inv_temperature, float* avg_prob,
                             float* stats, void* stream) {
  MV2_CHECK_ARG(presign && avg_prob && stats && N > 0 && d > 0 && d <= 12 && num_codebooks > 0 && num_codebooks <= 65535);
  const int K = 1 << d;
  const int blocks = ceil_div(N, LE_TOK);
  launch_k(lfq_entropy_kernel, dim3(dim3(blocks, num_codebooks)), dim3(256), K * sizeof(float), (cudaStream_t)stream, presign, N, d, num_codebooks,
           inv_temperature, avg_prob, stats);
  MV2_CHECK_LAUNCH();
  return MV2_OK;
}

size_t mv2_lfq_entropy_fact_workspace_bytes(int64_t n_tokens, int d, int num_codebooks) {
  if (n_tokens <= 0 || d < 1 || d > LF_MAXD || num_codebooks <= 0) return 0;
  const LfSplit s = lf_split(n_tokens, d, num_codebooks);
  const size_t K = (size_t)1 << d, nc = (size_t)num_codebooks;
  const size_t fwd = (size_t)s.splits * nc * (K + (size_t)s.tiles) * sizeof(double), bwd = nc * K * sizeof(float);
  return std::max(fwd, bwd);
}

int mv2_lfq_entropy_fact_partials(const float* presign, int64_t N, int d, int num_codebooks, float inv_temperature, float* avg_prob,
                                  float* stats, void* workspace, void* stream) {
  const int nc = num_codebooks;
  MV2_CHECK_ARG(presign && avg_prob && stats && workspace && N > 0 && d >= 1 && d <= LF_MAXD && nc > 0 && d * nc <= Q_MAXD_WIDE);
  const LfSplit s = lf_split(N, d, nc);
  cudaStream_t st = (cudaStream_t)stream;
  double* ws_avg = (double*)workspace;
  const int64_t n = (int64_t)nc << d;
  double* ws_ent = ws_avg + (int64_t)s.splits * n;
  launch_k(lfq_fact_partials_kernel, dim3(s.tiles, s.splits, nc), dim3(256), 0, st, presign, N, d, nc, inv_temperature, s.per,
           ws_avg, ws_ent);
  MV2_CHECK_LAUNCH();
  launch_k(lfq_fact_avg_kernel, dim3(ceil_div(n, 256)), dim3(256), 0, st, (const double*)ws_avg, n, s.splits, avg_prob);
  MV2_CHECK_LAUNCH();
  launch_k(lfq_fact_stats_kernel, dim3(1), dim3(256), 0, st, (const double*)ws_ent, s.splits * nc * s.tiles, presign, N * nc * d, stats);
  MV2_CHECK_LAUNCH();
  return MV2_OK;
}

int mv2_lfq_entropy_fact_backward(const float* presign, const float* avg_global, int64_t N, int d, int num_codebooks,
                                  float inv_temperature, float coef_sample, float coef_batch, float* grad_presign, void* workspace,
                                  void* stream) {
  const int nc = num_codebooks;
  MV2_CHECK_ARG(presign && avg_global && grad_presign && workspace && N > 0 && d >= 1 && d <= LF_MAXD && nc > 0 &&
                d * nc <= Q_MAXD_WIDE);
  cudaStream_t st = (cudaStream_t)stream;
  const int64_t n = (int64_t)nc << d;
  float* hga = (float*)workspace;
  launch_k(lfq_fact_hga_kernel, dim3(ceil_div(n, 256)), dim3(256), 0, st, avg_global, n, coef_batch, hga);
  MV2_CHECK_LAUNCH();
  launch_k(lfq_fact_backward_kernel, dim3(ceil_div(N * nc, LF_BW_WARPS)), dim3(LF_BW_WARPS * 32), 0, st, presign, (const float*)hga, N, d, nc, inv_temperature,
           coef_sample, grad_presign);
  MV2_CHECK_LAUNCH();
  return MV2_OK;
}

int mv2_mse(const void* a, int a_dtype, const void* b, int b_dtype, int64_t n, void* workspace, float* out, void* stream) {
  MV2_CHECK_ARG(a && b && workspace && out && n > 0);
  cudaStream_t st = (cudaStream_t)stream;
  double* part = (double*)workspace;
  const int nb = (int)std::min<int64_t>(MSE_BLOCKS, ceil_div(n, (int64_t)256));
#define MV2_MSE_CASE(DA, TA, DB, TB) \
  else if (a_dtype == DA && b_dtype == DB) launch_k(mse_partial_kernel<TA, TB>, dim3(nb), dim3(256), 0, st, (const TA*)a, (const TB*)b, n, part)
  if (false) {}
  MV2_MSE_CASE(MV2_F32, float, MV2_F32, float); MV2_MSE_CASE(MV2_F32, float, MV2_BF16, __nv_bfloat16);
  MV2_MSE_CASE(MV2_BF16, __nv_bfloat16, MV2_F32, float); MV2_MSE_CASE(MV2_BF16, __nv_bfloat16, MV2_BF16, __nv_bfloat16);
  MV2_MSE_CASE(MV2_U8, uint8_t, MV2_F32, float); MV2_MSE_CASE(MV2_U8, uint8_t, MV2_BF16, __nv_bfloat16);
  MV2_MSE_CASE(MV2_F32, float, MV2_F16, __half); MV2_MSE_CASE(MV2_F16, __half, MV2_F32, float);
  MV2_MSE_CASE(MV2_F16, __half, MV2_F16, __half); MV2_MSE_CASE(MV2_U8, uint8_t, MV2_F16, __half);
  else { set_error("mse: unsupported dtype pair %d, %d", a_dtype, b_dtype); return MV2_E_ARG; }
#undef MV2_MSE_CASE
  MV2_CHECK_LAUNCH();
  launch_k(mse_final_kernel, dim3(1), dim3(32), 0, st, (const double*)part, nb, 1.0 / (double)n, out);
  MV2_CHECK_LAUNCH();
  return MV2_OK;
}
size_t mv2_mse_workspace_bytes(void) { return (size_t)MSE_BLOCKS * sizeof(double); }

int mv2_lfq_aux_finalize(const float* avg_prob_sum, const float* stats, int d, int num_codebooks, int64_t n_tokens, int64_t n_tokens_global,
                         float diversity_gamma, float entropy_weight, float commitment_weight, float* out4, void* stream) {
  const int nc = num_codebooks;
  MV2_CHECK_ARG(avg_prob_sum && stats && out4 && d > 0 && d <= LF_MAXD && nc > 0 && n_tokens > 0 && n_tokens_global > 0);
  const float inv_g = (float)(1.0 / (double)n_tokens_global), inv_t = (float)(1.0 / ((double)n_tokens * nc)),
              inv_e = (float)(1.0 / ((double)n_tokens * nc * d));
  if (d <= 12)
    launch_k(lfq_aux_final_kernel, dim3(1), dim3(256), 0, (cudaStream_t)stream, avg_prob_sum, stats, 1 << d, nc, inv_g, inv_t, inv_e,
             diversity_gamma, entropy_weight, commitment_weight, out4);
  else
    launch_k(lfq_aux_final_wide_kernel, dim3(1), dim3(1024), 0, (cudaStream_t)stream, avg_prob_sum, stats, (int64_t)nc << d, nc, inv_g,
             inv_t, inv_e, diversity_gamma, entropy_weight, commitment_weight, out4);
  MV2_CHECK_LAUNCH();
  return MV2_OK;
}

int mv2_gateloop_scan(const void* qkva, const void* res, void* out, int dtype, int B, int T, int P, int C, void* stream) {
  return mv2_gateloop_scan_state(qkva, res, out, dtype, B, T, P, C, nullptr, stream);
}

int mv2_gateloop_scan_state(const void* qkva, const void* res, void* out, int dtype, int B, int T, int P, int C, float* state,
                            void* stream) {
  MV2_CHECK_ARG(qkva && res && out && B > 0 && T > 0 && P > 0 && C > 0);
  const int64_t total = (int64_t)B * P * C;
  const int64_t blocks = ceil_div(total, (int64_t)256);
  MV2_CHECK_ARG(blocks <= 2147483647LL);
  cudaStream_t st = (cudaStream_t)stream;
  if (dtype == MV2_F32)
    launch_k(gateloop_scan_kernel<float>, dim3((unsigned)blocks), dim3(256), 0, st, (const float*)qkva, (const float*)res, (float*)out, T, (int64_t)P * C, C, total, state);
  else if (dtype == MV2_BF16)
    launch_k(gateloop_scan_kernel<__nv_bfloat16>, dim3((unsigned)blocks), dim3(256), 0, st, (const __nv_bfloat16*)qkva, (const __nv_bfloat16*)res, (__nv_bfloat16*)out, T, (int64_t)P * C, C, total, state);
  else if (dtype == MV2_F16)
    launch_k(gateloop_scan_kernel<__half>, dim3((unsigned)blocks), dim3(256), 0, st, (const __half*)qkva, (const __half*)res, (__half*)out, T, (int64_t)P * C, C, total, state);
  else { set_error("bad dtype %d", dtype); return MV2_E_ARG; }
  MV2_CHECK_LAUNCH();
  return MV2_OK;
}

// 16-byte vectors over C when every pointer and the channel count allow them, else one channel per thread
static bool pool_vec_ok(int C, int vec, std::initializer_list<const void*> ps) {
  if (C % vec != 0) return false;
  for (const void* p : ps)
    if ((uintptr_t)p % 16 != 0) return false;
  return true;
}

int mv2_maxpool2x2(const void* x, void* y, int dtype, int N, int H, int W, int C, void* stream) {
  MV2_CHECK_ARG(x && y && N > 0 && H >= 2 && W >= 2 && C > 0);
  const int vec = dtype == MV2_BF16 ? 8 : 4;
  const bool v = pool_vec_ok(C, vec, {x, y});
  const int64_t total = (int64_t)N * (H / 2) * (W / 2) * (v ? C / vec : C);
  const int blocks = (int)std::min<int64_t>((total + 255) / 256, grid_cap(32));
  cudaStream_t st = (cudaStream_t)stream;
  if (dtype == MV2_F32) {
    if (v) launch_k(maxpool2x2_kernel<float, 4>, dim3(blocks), dim3(256), 0, st, (const float*)x, (float*)y, N, H, W, C);
    else launch_k(maxpool2x2_kernel<float, 1>, dim3(blocks), dim3(256), 0, st, (const float*)x, (float*)y, N, H, W, C);
  } else if (dtype == MV2_BF16) {
    using B16 = __nv_bfloat16;
    if (v) launch_k(maxpool2x2_kernel<B16, 8>, dim3(blocks), dim3(256), 0, st, (const B16*)x, (B16*)y, N, H, W, C);
    else launch_k(maxpool2x2_kernel<B16, 1>, dim3(blocks), dim3(256), 0, st, (const B16*)x, (B16*)y, N, H, W, C);
  } else { set_error("bad dtype %d", dtype); return MV2_E_ARG; }
  MV2_CHECK_LAUNCH();
  return MV2_OK;
}

int mv2_maxpool2x2_backward(const void* gy, const void* x, void* gx, int dtype, int N, int H, int W, int C, void* stream) {
  MV2_CHECK_ARG(gy && x && gx && N > 0 && H >= 2 && W >= 2 && C > 0);
  const int vec = dtype == MV2_BF16 ? 8 : 4;
  const bool v = pool_vec_ok(C, vec, {gy, x, gx});
  const int64_t total = (int64_t)N * ((H + 1) / 2) * ((W + 1) / 2) * (v ? C / vec : C);
  const int blocks = (int)std::min<int64_t>((total + 255) / 256, grid_cap(32));
  cudaStream_t st = (cudaStream_t)stream;
  if (dtype == MV2_F32) {
    if (v) launch_k(maxpool2x2_backward_kernel<float, 4>, dim3(blocks), dim3(256), 0, st, (const float*)gy, (const float*)x, (float*)gx, N, H, W, C);
    else launch_k(maxpool2x2_backward_kernel<float, 1>, dim3(blocks), dim3(256), 0, st, (const float*)gy, (const float*)x, (float*)gx, N, H, W, C);
  } else if (dtype == MV2_BF16) {
    using B16 = __nv_bfloat16;
    if (v) launch_k(maxpool2x2_backward_kernel<B16, 8>, dim3(blocks), dim3(256), 0, st, (const B16*)gy, (const B16*)x, (B16*)gx, N, H, W, C);
    else launch_k(maxpool2x2_backward_kernel<B16, 1>, dim3(blocks), dim3(256), 0, st, (const B16*)gy, (const B16*)x, (B16*)gx, N, H, W, C);
  } else { set_error("bad dtype %d", dtype); return MV2_E_ARG; }
  MV2_CHECK_LAUNCH();
  return MV2_OK;
}

}  // extern "C"
