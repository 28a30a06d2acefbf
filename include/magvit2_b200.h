/*
 * magvit2_b200.h -- C ABI of libmagvit2_b200.so, the sm_90a compute library behind
 * the VideoTokenizer forward path (tokenize / decode_from_code_indices / forward).
 *
 * The reference (lucidrains/magvit2-pytorch @ a00519fa) has NO native / FFI layer of
 * its own: its boundary is the Python class magvit2_pytorch.VideoTokenizer
 * (magvit2_pytorch/magvit2_pytorch.py:1045) whose forward dispatches ~730 ATen calls.
 * Each entry point below replaces the ATen call sequence of one reference module
 * (cited as M:line = magvit2_pytorch.py, A:line = attend.py).  The Python host class
 * magvit2_pytorch_b200.VideoTokenizer binds them with ctypes (INTEGRATION.md).
 *
 * Conventions
 *   - plain C: pointers, sizes, POD structs; no torch / C++ types cross the boundary.
 *   - every call returns 0 on success or a negative MV2_E_* code; mv2_last_error()
 *     returns a thread-local message.  Nothing throws across the boundary.
 *   - all device pointers are borrowed for the duration of the call; the library
 *     never allocates device memory: the caller supplies workspaces.
 *   - stream ordered, no implicit synchronisation; `stream` is a cudaStream_t passed
 *     as void*.
 *   - activations are channels-last ("NDHWC"): x[b][t][h][w][c], dtype MV2_F32, MV2_BF16
 *     or MV2_F16 (wherever MV2_BF16 is accepted for activations, so is MV2_F16: same
 *     kernels, fp16 storage with one round-to-nearest-even per stored value);
 *     accumulation is always fp32; biases / gammas / tiny SE + quantiser weights are fp32.
 *   - there is NO CPU fallback: every function launches sm_90a kernels.
 */
#ifndef MAGVIT2_B200_H
#define MAGVIT2_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define MV2_ABI_VERSION 5   /* 2: mv2_conv_args.oscale, mv2_tc_conv_args.{oscale,out_layout}; 3: num_codebooks / spherical in the quantiser entry points;
                               4: the two entry points of the one-launch SqueezeExcite tail for small frames are removed: the
                               engine never enabled it by default, so the separate pool / gate / gate_residual calls are the only SE path;
                               5: the conv entry points take the streaming history (mv2_conv_hist, NULL for none) as an argument,
                               their four _hist twins are removed */

enum { MV2_F32 = 0, MV2_BF16 = 1,
       MV2_U8 = 2,  /* source dtype of the two layout-in entry points and of mv2_mse only: decoded uint8 frames, x / 255 */
       MV2_F16 = 3, /* IEEE half: fp16 storage, fp32 accumulation */
       MV2_TF32 = 4 /* tensor-core convs only: fp32 storage, TF32 multiply (the top 19 bits of each fp32 operand),
                       fp32 accumulation */ };
/* The tensor-core conv structs (mv2_tc_conv_args, mv2_tc_ru_args) carry their element type in a `dtype` field that sits
 * in what was padding before fp16 existed: 0 there means bf16, so a zero-initialised struct of an older caller keeps its
 * meaning.  MV2_F32 (also 0) is therefore not a distinct value there: fp32 activations run on the tensor cores as
 * MV2_TF32 (the tap-wise and slab convs, SpatialDownsample2x; not the fused ResidualUnit, whose _supported refuses it). */
enum { MV2_ACT_NONE = 0, MV2_ACT_ELU = 1, MV2_ACT_SILU = 2,
       MV2_ACT_LEAKY_RELU = 3,  /* LeakyReLU(0.1), the discriminator's activation (M:117-118) */
       MV2_ACT_RELU = 4         /* ReLU, the activation of a VGG feature extractor (perceptual loss, M:1397-1405) */ };
enum { MV2_SHUFFLE_NONE = 0, MV2_SHUFFLE_SPACE = 1, MV2_SHUFFLE_TIME = 2 };
enum {
  MV2_OK = 0,
  MV2_E_ARG = -1,       /* bad argument / unsupported shape */
  MV2_E_CUDA = -2,      /* CUDA runtime / driver error (see mv2_last_error) */
  MV2_E_UNSUPPORTED = -3
};

int mv2_abi_version(void);
const char* mv2_last_error(void);
/* Number of kernels the library has launched from the calling thread (thread-local, from 0).  A kernel counts when its
 * launch is accepted, including a launch into a stream under graph capture; a call refused by its argument checks adds
 * nothing.  Memsets and copies are not kernels and are not counted: the copy of mv2_copy_frames and the zero-filled
 * t_pad frames of mv2_to_channels_last. */
uint64_t mv2_launch_count(void);
/* Compute capability of the current device as major*10+minor (90 on H100), <0 on error. */
int mv2_device_arch(void);
/* The frames in front of a streamed chunk that the conv entry points read (see "streaming" below); NULL: none. */
typedef struct mv2_conv_hist mv2_conv_hist;
/* Programmatic dependent launch: when on, every kernel is launched with
 * cudaLaunchAttributeProgrammaticStreamSerialization so its prologue (barrier init, bias staging,
 * block scheduling) overlaps the tail of the previous kernel of the stream; all kernels execute griddepcontrol.wait
 * before touching activations.  Returns the previous setting.  Off by default. */
int mv2_set_pdl(int on);

/* ---- layout: torch (B,C,T,H,W) <-> channels-last activations ------------------
 * mv2_to_channels_last : video ingest.  Replaces pad_at_dim (M:86-89, use M:1537) +
 *   the implicit layout of every later conv: dst[b][t+t_pad][h][w][c] = src[b][c][t][h][w],
 *   frames [0,t_pad) of dst are zero-filled.
 * mv2_to_channels_first: replaces the frame crop at M:1646-1647 and the layout return:
 *   dst[b][c][t][h][w] = src[b][t+t_crop][h][w][c],  dst has T - t_crop frames.            */
int mv2_to_channels_last(const void* src, int src_dtype, void* dst, int dst_dtype,
                         int B, int C, int T, int H, int W, int t_pad, void* stream);
int mv2_to_channels_first(const void* src, int src_dtype, void* dst, int dst_dtype,
                          int B, int C, int T, int H, int W, int t_crop, void* stream);
/* mv2_ingest_kwpack: ingest for the tensor-core conv_in (M:1109, 7x7x7 with C_in = 3): besides the layout change and
 *   the time_padding zero frames it packs the k_w taps into the channel axis,
 *   dst[b][t+t_pad][h][w][dw*C + c] = src[b][c][t][h][w + dw - pw]  (cpack channels, zero padded; fp16 for an MV2_F16
 *   source, bf16 for the others),
 *   so conv_in becomes a (k_t x k_h x 1)-tap implicit GEMM over cpack = 32 channels.                            */
int mv2_ingest_kwpack(const void* src, int src_dtype, void* dst, int B, int C, int T, int H, int W,
                      int t_pad, int kw, int pw, int cpack, void* stream);
/* MV2_KWPACK_F32_DST OR'd into mv2_ingest_kwpack's src_dtype (MV2_F32, MV2_BF16 or MV2_U8) writes fp32 instead: the
 *   ingest of the TF32 conv_in, 7 x 3 packed channels zero padded to cpack = 32, one 128-byte K row.                  */
#define MV2_KWPACK_F32_DST 0x100

/* mv2_copy_frames: frame-range copy between channels-last clips (device memcpy2D, no kernel):
 *   dst[b][dst_t0 + i] = src[b][src_t0 + i], i < n_frames; zero_front != 0 also zero-fills dst frames [0, dst_t0).
 * Used to split off / re-attach the first frame for separate_first_frame_encoding (reference M:1553-1561, M:1633-1639:
 * unpack / pack / pad_at_dim on the time axis).                                                                           */
int mv2_copy_frames(const void* src, void* dst, int B, int src_T, int dst_T, int src_t0, int dst_t0, int n_frames,
                    size_t frame_bytes, int zero_front, void* stream);

/* mv2_pad_cl: explicit causal / spatial padding for CausalConv3d with pad_mode != 'constant' (reference M:925-927:
 *   F.pad(x, (pw, pw, ph, ph, pt, 0), mode)): dst (B, T+pt, H+2ph, W+2pw, C) from src (B,T,H,W,C), channels-last;
 *   mode 1 = 'reflect', 2 = 'replicate', 3 = 'circular'.  The conv then runs with zero leading padding on dst.
 *   ('constant' never materialises its padding: TMA out-of-bounds fill / bounds checks.)                                   */
int mv2_pad_cl(const void* src, void* dst, int dtype, int B, int T, int H, int W, int C, int pt, int ph, int pw, int mode,
               void* stream);

/* ---- convolution family (CUDA-core fp32-accumulate path; any shape) -----------
 * One generic strided N-d convolution over channels-last activations with a fused
 * epilogue  y = shuffle(act(conv(x) + bias)) + res.   Replaces
 *   CausalConv3d.forward           F.pad + nn.Conv3d            M:924-928  (pt = kt-1, ph = kh/2, pw = kw/2)
 *   nn.Conv3d 1x1x1 / nn.Linear    M:939, M:352, M:367, M:493-495
 *   SpatialDownsample2x.forward    Conv2d k3 s2 p1 per frame    M:770-780
 *   TimeDownsample2x.forward       F.pad(2,0) + Conv1d k3 s2    M:796-807
 *   SpatialUpsample2x / TimeUpsample2x  1x1 conv + SiLU + depth-to-space/time  M:838-846, M:875-883
 *   Residual.forward               "+ x"                         M:173-174 (res)
 *   TokenShift.forward             half-channel one-frame delay  M:250-254 (x_token_shift)
 * Weights are packed by the host as w[tap][ci][co] (tap = (dt*kh + dh)*kw + dw) in the
 * activation dtype; bias is fp32[Co] or NULL.                                            */
typedef struct mv2_conv_args {
  const void* x;       /* (B, Ti, Hi, Wi, Ci) */
  const void* w;       /* [kt*kh*kw][Ci][Co]  */
  const float* bias;   /* [Co] or NULL */
  const void* res;     /* same shape as y, or NULL */
  void* y;             /* (B, To, Ho, Wo, Co) or its depth-to-space/time shuffle */
  int32_t dtype;
  int32_t B, Ti, Hi, Wi, Ci;
  int32_t To, Ho, Wo, Co;
  int32_t kt, kh, kw;
  int32_t st, sh, sw;
  int32_t pt, ph, pw;        /* leading zero padding; trailing padding is implied by To/Ho/Wo */
  int32_t act;               /* MV2_ACT_* */
  int32_t shuffle;           /* MV2_SHUFFLE_*: SPACE: y (B,To,2Ho,2Wo,Co/4), co=(c,p1,p2); TIME: y (B,2To,Ho,Wo,Co/2), co=(c,p) */
  int32_t x_token_shift;     /* 1: input channels >= ceil(Ci/2) are read from frame t-1 (zero at t = 0) */
  const float* oscale;       /* fp32 [B][Co] or NULL: per-(clip, output channel) multiplier applied to the accumulator BEFORE
                                bias / activation -- the demodulation factor of Conv3DMod (M:741-742), see mv2_mod_prepare */
} mv2_conv_args;
int mv2_conv_forward(const mv2_conv_args* a, const mv2_conv_hist* hist, void* stream);

/* ---- SqueezeExcite (M:221-240) --------------------------------------------------
 * se_pool  : per frame f (F = B*T frames of P = H*W positions, C channels):
 *            logit[n] = <y[f,n,:], wk> + bk; a = softmax_n(logit); pooled[f,c] = sum_n a[n] y[f,n,c]
 *            done as chunk partials (online softmax) + a combine fused into se_gate.
 * se_gate  : gate[f,:] = sigmoid(W2 leaky_relu_0.1(W1 pooled + b1) + b2)   (fp32 [F][C])
 * gate_residual : out = gate[f(m), c] * y[m, c] + x[m, c]                    (M:240 + M:174)
 * workspace for se_pool: mv2_se_workspace_bytes(F, P, C).  se_gate keeps its F * Hd hidden activations in the same
 * workspace, which reserves F * (C + 16) floats for them: Hd <= C + 16, else MV2_E_ARG.                             */
size_t mv2_se_workspace_bytes(int F, int P, int C);
int mv2_se_pool(const void* y, int dtype, int F, int P, int C, const float* wk, float bk,
                void* workspace, void* stream);
int mv2_se_gate(const void* workspace, int dtype /* of the y passed to mv2_se_pool */, int F, int P, int C, int Hd,
                const float* w1, const float* b1, const float* w2, const float* b2,
                float* gates, void* stream);
int mv2_gate_residual(const void* y, const void* x, const float* gates, void* out, int dtype,
                      int F, int P, int C, void* stream);

/* ---- RMSNorm (M:275-276): out = x / max(||x||_2, 1e-12) * sqrt(C) * gamma over the channel
 * axis of channels-last tokens; token_shift as in mv2_conv_args (M:250-254).               */
int mv2_rmsnorm(const void* x, void* out, int dtype, const float* gamma,
                int B, int T, int P, int C, int token_shift, void* stream);

/* ---- axial softmax attention core (Attention.forward M:379-388 + Attend A:186-243) ------
 * qkv: [Ntok][3*heads*dim_head] laid out '(qkv h d)' (M:353); out: [Ntok][heads*dim_head] '(h d)'.
 * Sequence s = (o, n): token(i) = o*outer_stride + n*inner_stride + i*tok_stride, i in [0, L).
 *   space attention (M:444-454): n_outer = B*T, n_inner = 1, outer_stride = H*W, tok_stride = 1, L = H*W
 *   time  attention (M:456-464): n_outer = B, outer_stride = T*H*W, n_inner = H*W, inner_stride = 1,
 *                                tok_stride = H*W, L = T, causal = 1
 * n_mem learned key/values (mem_kv fp32 [2][heads][n_mem][dim_head], M:357, M:383-385) are
 * prepended; causal masking is right aligned (A:46-47, A:123-129): query i sees mem + keys <= i;
 * it is disabled when L == 1 (A:209-210).  dim_head must be a multiple of 32, <= 96.           */
typedef struct mv2_attn_args {
  const void* qkv; void* out; const float* mem_kv;
  int32_t dtype, heads, dim_head, n_mem, causal;
  int32_t n_outer, n_inner, L;
  int64_t outer_stride, inner_stride, tok_stride;
} mv2_attn_args;
int mv2_attention(const mv2_attn_args* a, void* stream);

/* ---- attention dropout (Attend's dropout on the softmax weights in training mode, A:175 / A:239) --------------------
 * mv2_attention_dropout: mv2_attention (same kernels choice, same arguments) with every softmax weight, memory key/values
 *   included, kept with probability 1 - p and scaled by 1 / (1 - p); the softmax denominator is the undropped one:
 *     o_i = fp32(1 / (1 - p)) * sum_j keep_ij softmax_ij v_j.
 * keep_ij is a pure function of (seed, call, sequence s = o * n_inner + n, head h, query i, key j), j in [0, n_mem + L)
 *   counting the memory slots first: with r = Philox4x32-10(counter (i, j >> 2, s, h | call << 16), key (seed low, seed
 *   high word)), keep_ij = r[j & 3] >= floor(p * 2^32) (p the fp32 value, widened to double).
 * mv2_attention_dropout_mask: writes that mask, uint8 keep[s][h][i][n_mem + L] (s < n_seq), including the entries a
 *   causal mask hides.  Both need 0 < p < 1, heads < 2^16 and call < 2^16 (MV2_E_ARG otherwise).                      */
typedef struct mv2_dropout_args {
  uint64_t seed;
  uint32_t call;   /* index of the attention call within one forward: distinct calls draw independent masks */
  float p;
} mv2_dropout_args;
int mv2_attention_dropout(const mv2_attn_args* a, const mv2_dropout_args* d, void* stream);
int mv2_attention_dropout_mask(int n_seq, int heads, int L, int n_mem, const mv2_dropout_args* d, uint8_t* keep, void* stream);

/* ---- Taylor-series linear attention core (TaylorSeriesLinearAttn, un-vendored dependency;
 * SURVEY.md Appendix A.3; called at M:430).  q: [Ntok][heads*8], kv: [Ntok][2*heads*8] '(kv h d)',
 * out: [Ntok][heads*8]; sequences are n_seq contiguous runs of L tokens.  dim_head must be 8.
 * workspace: mv2_linattn_workspace_bytes(n_seq, heads, L).                                    */
size_t mv2_linattn_workspace_bytes(int n_seq, int heads, int L);
int mv2_linear_attention(const void* q, const void* kv, void* out, int dtype,
                         int n_seq, int L, int heads, int dim_head, void* workspace, void* stream);

/* ---- GEGLU (M:466-469): out[n][i] = gelu_erf(in[n][I + i]) * in[n][i] ------------------------- */
int mv2_geglu(const void* in, void* out, int dtype, int64_t N, int I, void* stream);

/* ---- quantisers (un-vendored vector-quantize-pytorch LFQ / FSQ; SURVEY.md Appendix A.1/A.2;
 * reference call sites M:1576, M:1593, M:1700, M:1705; constructor kwargs num_codebooks M:1057, lfq_spherical M:1070) ------
 * d = dims per codebook, num_codebooks = nc, D = d * nc <= 32 projected dims; one index per (token, codebook):
 *   indices [N][nc].
 * lfq_forward : x [N][C] -> p = tanh((Win x + bin)/clamp)*clamp (fp32), per codebook (L2-normalised first when
 *               spherical != 0): bit_j = p_j > 0, index = sum bit_j << (d-1-j) (int64), quantized [N][C] = Wout (+-1) + bout.
 *               presign (fp32 [N][D], after the optional normalisation) is optional (diagnostics / training losses).
 * lfq_decode  : indices -> quantized (LFQ.indices_to_codes).
 * fsq_*       : same with tanh-bound + round-half-even + mixed-radix int32 index (levels[d], shared by the codebooks).
 * win [D][C], bin [D], wout [C][D], bout [C] are fp32.                                         */
int mv2_lfq_forward(const void* x, int dtype, int64_t N, int C, int d, int num_codebooks,
                    const float* win, const float* bin, const float* wout, const float* bout,
                    float clamp, int spherical, int64_t* indices, void* quantized, float* presign, void* stream);
int mv2_lfq_decode(const void* indices, int index_is_i64, int64_t N, int C, int d, int num_codebooks,
                   const float* wout, const float* bout, void* quantized, int dtype, void* stream);
int mv2_fsq_forward(const void* x, int dtype, int64_t N, int C, int d, int num_codebooks, const int32_t* levels /* host */,
                    const float* win, const float* bin, const float* wout, const float* bout,
                    int32_t* indices, void* quantized, float* bounded, void* stream);
int mv2_fsq_decode(const void* indices, int index_is_i64, int64_t N, int C, int d, int num_codebooks, const int32_t* levels /* host */,
                   const float* wout, const float* bout, void* quantized, int dtype, void* stream);

/* ---- LFQ training-mode auxiliary terms (A.1 steps 7-8; the one collective on the path) -------
 * lfq_entropy_partials: from presign [N][nc][d] (d <= 12) accumulates, for this rank,
 *   stats[0] = sum_{tokens, codebooks} H(softmax_K(2*inv_temp*<p, code_k>)), stats[1] = sum (p - sign p)^2,
 *   avg_prob[nc][K] += sum_tokens prob (un-normalised; caller divides by the token count, then the cross-rank SUM
 *   all-reduce of avg_prob -- nc * 2^d * 4 bytes, 4 KiB at the README config).
 * stats and avg_prob must be zeroed by the caller.                                             */
int mv2_lfq_entropy_partials(const float* presign, int64_t N, int d, int num_codebooks, float inv_temperature,
                             float* avg_prob, float* stats, void* stream);

/* lfq_entropy_fact_*: the same terms for 1 <= d <= 20 (D = d * nc <= 32), factorised over bits:
 *   prob_k = prod_i sigmoid(4 inv_temp p_i s_ki)  (s_ki = +-1: bit i of code k, MSB first), so nothing of size
 *   [tokens][2^d] is materialised; O(N nc 2^d) work, a log only where prob > 1e-5.  Deterministic: fixed-order sums, no
 *   float atomics, bit-identical across runs.  workspace: mv2_lfq_entropy_fact_workspace_bytes(N, d, nc) bytes (covers both).
 * fact_partials: OVERWRITES avg_prob[nc][2^d] = sum_tokens prob and stats[2] (as lfq_entropy_partials; no zeroing needed).
 * fact_backward: grad_presign [N][nc][d] of  coef_sample * sum_{t,c} H(prob_tc) - coef_batch * sum_{t,c,k} h'(avg_global_ck) prob_tck
 *   (h'(x) = -(log x + 1) above 1e-5, -log 1e-5 below), i.e. the entropy part of the aux loss with the batch term taken at the
 *   cross-rank mean avg_global [nc][2^d]: coef_sample = entropy_weight / (N nc), coef_batch = entropy_weight * diversity_gamma / (N nc).
 *   grad = 2 inv_temp (sum_k c_k s_ki - tanh(2 inv_temp p_i) sum_k c_k),  c_k = prob_k (coef_sample h'(prob_k) - coef_batch h'(avg_k)). */
size_t mv2_lfq_entropy_fact_workspace_bytes(int64_t n_tokens, int d, int num_codebooks);
int mv2_lfq_entropy_fact_partials(const float* presign, int64_t N, int d, int num_codebooks, float inv_temperature,
                                  float* avg_prob, float* stats, void* workspace, void* stream);
int mv2_lfq_entropy_fact_backward(const float* presign, const float* avg_global, int64_t N, int d, int num_codebooks,
                                  float inv_temperature, float coef_sample, float coef_batch, float* grad_presign,
                                  void* workspace, void* stream);

/* mv2_lfq_aux_finalize: out4 = {per_sample_entropy, batch_entropy, commitment, aux_loss} from the partial sums above
 * (A.1 steps 7-10): per_sample = stats[0] / (n_tokens nc), commitment = stats[1] / (n_tokens nc d),
 * batch_entropy = mean over codebooks of sum_k -p_k log(max(p_k, 1e-5)), p = avg_prob_sum / n_tokens_global
 * (avg_prob_sum = the cross-rank SUM), aux = (per_sample - diversity_gamma * batch_entropy) * entropy_weight
 * + commitment * commitment_weight.  d <= 20 (d > 12: one 1024-thread block, fp64 sums in a fixed order).             */
int mv2_lfq_aux_finalize(const float* avg_prob_sum, const float* stats, int d, int num_codebooks, int64_t n_tokens,
                         int64_t n_tokens_global, float diversity_gamma, float entropy_weight, float commitment_weight,
                         float* out4, void* stream);

/* ---- gateloop_time (reference M:1216-1222: ToTimeSequence(Residual(SimpleGateLoopLayer(dim)))) -----------
 * qkva [B][T][P][3C] = Linear(dim, 3 dim) of the RMSNorm'ed activations (q | kv | a thirds), res / out [B][T][P][C]:
 *   s_t = sigmoid(a_t) * s_{t-1} + kv_t  (s_{-1} = 0, fp32 state),   out_t = q_t * s_t + res_t
 * per (b, pixel p, channel).  The norm and the projection run through mv2_rmsnorm and the conv entry points.   */
int mv2_gateloop_scan(const void* qkva, const void* res, void* out, int dtype, int B, int T, int P, int C, void* stream);

/* ---- reconstruction loss (reference M:1722 F.mse_loss(video, recon_video)) ------------------
 * out[0] = mean_i (a[i] - b[i])^2 over n elements of two same-layout tensors; a_dtype may be MV2_U8 (frames, x / 255).
 * Deterministic (fixed-order two-stage reduction); workspace: mv2_mse_workspace_bytes() bytes.                          */
int mv2_mse(const void* a, int a_dtype, const void* b, int b_dtype, int64_t n, void* workspace, float* out, void* stream);
size_t mv2_mse_workspace_bytes(void);

/* ---- 2x2 max-pool of a VGG feature extractor (nn.MaxPool2d(2, 2), floor mode) over channels-last maps ------------------
 * mv2_maxpool2x2         : x (N, H, W, C) -> y (N, H/2, W/2, C), y = max of each 2x2 window (NaN propagates, as in torch).
 * mv2_maxpool2x2_backward: gy (N, H/2, W/2, C) and the saved pool input x (N, H, W, C), the output of a conv with ReLU in its
 *   epilogue -> gx (N, H, W, C), dense: each window's gradient goes to its first maximum in row-major order (torch's tie
 *   rule) and is masked by x > 0 (the ReLU's gradient); every other element, including the row / column that floor mode
 *   drops for odd H / W, is zero.  Windows do not overlap: no atomics.  dtype MV2_F32 or MV2_BF16.                      */
int mv2_maxpool2x2(const void* x, void* y, int dtype, int N, int H, int W, int C, void* stream);
int mv2_maxpool2x2_backward(const void* gy, const void* x, void* gx, int dtype, int N, int H, int W, int C, void* stream);

/* ---- wgmma / TMA implicit-GEMM convolution (bf16, fp16 or TF32 in, fp32 accumulate in registers) ------------
 * Same operator family and epilogue as mv2_conv_forward, for bf16, fp16 or fp32 (TF32 multiply) activations
 * (mv2_tc_conv_args.dtype), executed on the
 * Hopper tensor cores (wgmma): TMA box loads with out-of-bounds zero fill implement the causal /
 * spatial halo (no padded copy, reference M:924-928), strided convs read through stride-phase
 * tensor maps, accumulators live in registers.  Weights are packed K-major: w[co][tap][ci] (bf16);
 * for depth-to-space / depth-to-time stores the host permutes the Co rows to co' = q*Cy + c
 * (q = p1*2+p2 or p) so that the shuffled stores are channel-contiguous; bias is permuted alike.
 * Requirements (mv2_tc_conv_supported): Ci * element size % 32 == 0 (Ci % 16 for 16-bit, Ci % 8 for fp32), strides in
 * {1,2}, <= 64 taps.                                                                                                  */
typedef struct mv2_tc_conv_args {
  const void* x;       /* bf16 (B, Ti, Hi, Wi, Ci) */
  const void* w;       /* bf16 [Co][kt*kh*kw*Ci] */
  const float* bias;   /* fp32 [Co] or NULL */
  const void* res;     /* bf16, same shape as y, or NULL */
  void* y;             /* bf16 */
  int32_t B, Ti, Hi, Wi, Ci;
  int32_t To, Ho, Wo, Co;
  int32_t kt, kh, kw;
  int32_t st, sh, sw;
  int32_t pt, ph, pw;
  int32_t act;
  int32_t shuffle;
  int32_t epi_mode;    /* 0 plain; 1 fused GEGLU (M:466-469): packed columns come in groups of 16 = 8 x-columns then
                          their 8 gate-columns, output has Co/2 channels: y = gelu_erf(gate) * x;
                          2 scaled residual (needs res, no shuffle): y = (act(acc + bias) + res) * 2^-0.5, the
                          DiscriminatorBlock output (M:585), rounded to bf16 once */
  const float* oscale; /* as mv2_conv_args.oscale (plain / ragged epilogues only) */
  int32_t out_layout;  /* 0: y is channels-last (B,To,Ho,Wo,Co).  1: y is torch's channels-first (B,Co,To,Ho,Wo) -- the slab
                          kernel's conv_out (Co % 8 != 0) writes the reconstruction directly in the caller's layout; with
                          To < Ti and pt = kt - 1 - (Ti - To) the leading time_padding frames are never computed
                          (reference M:1642-1647: conv_out, then video[:, :, time_padding:]).  pt = -(Ti - To) is the
                          data gradient of a causal conv (the transposed conv, no leading pad) without its first Ti - To
                          frames: the video's gradient through conv_in; with Co <= 16 and kw > 3 (up to 7) it runs on
                          8- / 16-column N tiles.                                                                        */
  int32_t dtype;       /* element type of x, w, res and y: MV2_F16, MV2_TF32 (fp32), or MV2_BF16 (0, as in a
                          zero-initialised struct, also means MV2_BF16).  It sits in what was the struct's tail padding:
                          size and offsets are unchanged.  Channel rules are rules on bytes: a K row is 32 / 64 / 128 bytes,
                          16 / 32 / 64 16-bit or 8 / 16 / 32 fp32 channels */
} mv2_tc_conv_args;
int mv2_tc_conv_supported(const mv2_tc_conv_args* a);
int mv2_tc_conv_forward(const mv2_tc_conv_args* a, const mv2_conv_hist* hist, void* stream);
/* "Slab" variant for stride-1 convs with an in-plane kernel (the causal 3x3x3 residual convs): persistent
 * CTAs, one haloed activation slab per (frame, 64-channel slice) staged in shared memory once and reused by
 * all k_h*k_w in-plane taps, up to four 128-position M-tiles sharing each weight tile (mw * N tile <= 128 columns of
 * register accumulators).  Requirements (mv2_tc_slab_supported): stride 1, Ci % 64 == 0, Co % 32 == 0, no shuffle.   */
int mv2_tc_slab_supported(const mv2_tc_conv_args* a);
int mv2_tc_slab_forward(const mv2_tc_conv_args* a, const mv2_conv_hist* hist, void* stream);
/* SpatialDownsample2x (M:770-780: per-frame Conv2d k3 s2 p1) on the slab design: the input is read as (W/2) x (2C) with
 * row-parity sub-slabs, so no tap reloads its tile from L2.  `a` describes the conv as usual (kh = kw = 3, sh = sw = 2,
 * ph = pw = 1, kt = 1), but w is packed as bf16 [Co][6][2*Ci]: tap' = dh * 2 + q, q = 0: [zeros(Ci) | w[:, :, dh, 0]],
 * q = 1: [w[:, :, dh, 1] | w[:, :, dh, 2]].  Requirements: Hi, Wi even, Ci % 64 == 0, Co % 32 == 0.                       */
int mv2_tc_down_space_supported(const mv2_tc_conv_args* a);
int mv2_tc_down_space_forward(const mv2_tc_conv_args* a, void* stream);
/* Launch plan of mv2_tc_slab_forward for a layer shape on a device with n_sm SMs -- pure host arithmetic (no CUDA call,
 * the pointers in `a` are not dereferenced), exposed so the tiling rule and the static tile schedule can be checked
 * without a GPU.  mv2_tc_slab_plan: out6 = {M-tiles per weight tile (mw), N tile width (bn), N tiles, total tiles,
 * grid size, activation-slab ring depth}.  mv2_tc_slab_tile: the k-th tile that persistent CTA `cta` processes:
 * out6 = {tile id or -1 when the CTA has no k-th tile, clip b, frame t, h0, w0, first output column n0}. */
int mv2_tc_slab_plan(const mv2_tc_conv_args* a, int n_sm, int* out6);
int mv2_tc_slab_tile(const mv2_tc_conv_args* a, int n_sm, int cta, int k, int* out6);


/* ---- conditioning (cond_residual = ResidualUnitMod / Conv3DMod, reference M:680-753, M:946-988; stems M:1344-1352) -------
 * Conv3DMod applies per-clip weights  w_b = w * (cond_b + 1)  (over input channels), demodulated by
 * rsqrt(max(sum_{i,taps} w_b^2, eps)) per output channel, as a grouped conv.  The per-clip weights never need to exist:
 *     y[b, o] = inv_norm[b, o] * conv(x[b] * (cond[b] + 1), w)[o],   inv_norm[b,o] = rsqrt(max(sum_i (cond[b,i]+1)^2 S[o,i], eps)),
 * with S[o, i] = sum_taps w[o, i, tap]^2 packed once by the host.  So the shared-weight conv kernels run unchanged with
 *   mv2_dense_small   : y[b][n] = act(sum_k x[b][k] w[n][k] + bias[n])   (cond stems: Linear + SiLU; to_cond: Linear), fp32
 *   mv2_mod_prepare   : scale_in[b][i] = cond[b][i] + 1,  inv_norm[b][o] as above                                  , fp32
 *   mv2_scale_channels: out[b, pos, c] = x[b, pos, c] * scale[b][c]        (activation dtype)
 * and mv2_*conv_args.oscale = inv_norm.                                                                                   */
int mv2_dense_small(const float* x, const float* w, const float* bias, float* y, int B, int K, int N, int act, void* stream);
int mv2_mod_prepare(const float* cond, const float* S, float eps, float* scale_in, float* inv_norm, int B, int Ci, int Co,
                    void* stream);
int mv2_scale_channels(const void* x, const float* scale, void* out, int dtype, int B, int64_t positions_per_clip, int C,
                       void* stream);

/* ---- fused ResidualUnit front half (reference M:937-941 + the pooling half of SqueezeExcite M:229-233) ----------------
 * One launch computes  y = ELU(Conv3d_1x1x1(ELU(CausalConv3d_ktxkhxkw(x))))  for C -> C channels (C = 64 or 128, the
 * HBM-bound levels of the README config): the ELU'd 3x3x3 tile never leaves the SM -- it is written to shared memory as the
 * A operand of a second wgmma against the 1x1x1 weights -- and the second epilogue emits, next to y, one SqueezeExcite
 * pool record (max logit, sum e, sum e * y[C]; e = exp(logit - max), logit = <y, se_wk> + se_bk) per 32-position quarter of a tile,
 * which mv2_se_gate_records combines (replaces mv2_conv_forward x2 + mv2_se_pool for these layers).
 * w3: bf16 [C][kt*kh*kw*C] (K-major, as mv2_tc_conv_args.w); w1: bf16 [C][C]; b3 / b1 / se_wk: fp32 [C].
 * se_ws: workspace of mv2_tc_ru_workspace_bytes(a) bytes; records per frame = mv2_tc_ru_records(a).                     */
typedef struct mv2_tc_ru_args {
  const void* x;        /* bf16 (B, T, H, W, C) */
  const void* w3; const float* b3;
  const void* w1; const float* b1;
  const float* se_wk; float se_bk;
  int32_t dtype;        /* element type of x, w3, w1 and y, as mv2_tc_conv_args.dtype (in what was padding) */
  void* y;              /* bf16 / fp16 (B, T, H, W, C) */
  float* se_ws;
  int32_t B, T, H, W, C;
  int32_t kt, kh, kw;
} mv2_tc_ru_args;
int mv2_tc_ru_supported(const mv2_tc_ru_args* a);
int mv2_tc_ru_records(const mv2_tc_ru_args* a);
size_t mv2_tc_ru_workspace_bytes(const mv2_tc_ru_args* a);
int mv2_tc_ru_forward(const mv2_tc_ru_args* a, const mv2_conv_hist* hist, void* stream);
/* SE gate from pool records in the (max, sum, acc[C]) format, nrec records per frame laid out [F][nrec][C + 2], with the
 * hidden layer scratch (F * Hd floats) right behind them: gate[f,:] = sigmoid(W2 leaky_relu_0.1(W1 pooled + b1) + b2).
 * mv2_tc_ru_workspace_bytes reserves F * (C + 16) floats for that scratch: Hd <= C + 16, else MV2_E_ARG.                  */
int mv2_se_gate_records(const void* workspace, int nrec, int F, int C, int Hd,
                        const float* w1, const float* b1, const float* w2, const float* b2,
                        float* gates, void* stream);

/* ---- streaming: causal state carried from one chunk of a clip to the next (magvit2_pytorch_b200/stream.py) ------------
 * A chunked call must give exactly what the whole-clip call gives, so the kernels read the state in place instead of
 * re-running earlier frames.
 *
 * mv2_conv_hist: the frames in front of a causal conv's input x.  Input frame t < 0 of clip b is history frame T_h + t,
 *   read from h + b * clip_stride (elements) as a (T_h, Hi, Wi, Ci) block; frames older than the history (t < -T_h) are the
 *   causal zero padding, exactly as frame t < 0 is without history.  The history may be the tail of the previous chunk's
 *   input itself (clip_stride = that tensor's frames per clip * Hi * Wi * Ci): nothing is copied.
 * The `hist` argument of mv2_conv_forward, mv2_tc_conv_forward, mv2_tc_slab_forward and mv2_tc_ru_forward: NULL or T_h = 0
 *   means no history.  Each output element accumulates the same products in the same order as the whole-clip call; the
 *   slab kernels skip the taps older than the history as they skip the padding.  mv2_tc_conv_forward takes a history only
 *   on the shapes mv2_tc_conv_hist_supported accepts (pure host arithmetic): stride 1 and an output tile of one frame or of
 *   >= 8 positions per frame.  For the others a caller runs it without history on a copy of [history | x] with pt reduced
 *   by T_h, which gives the same values.                                                                                    */
struct mv2_conv_hist {
  const void* h;
  int32_t T_h;
  int64_t clip_stride;
};
int mv2_tc_conv_hist_supported(const mv2_tc_conv_args* a);
/* mv2_rmsnorm_prev: mv2_rmsnorm whose token shift reads frame -1 of clip b from prev + b * prev_clip_stride (elements,
 *   a (P, C) frame) instead of zeros: the TokenShift (M:250-254) of a chunk that continues a clip.                        */
int mv2_rmsnorm_prev(const void* x, const void* prev, int64_t prev_clip_stride, void* out, int dtype, const float* gamma,
                     int B, int T, int P, int C, void* stream);
/* mv2_attention_tail: rows [q_begin, a->L) of a causal mv2_attention call over L tokens (the same kernel choice for that L,
 *   so the same values).  a->qkv is a K/V cache holding the keys and values of all L tokens, rows of 2 * heads * dim_head
 *   laid out '(kv h d)', addressed with a's strides; the queries are rows 0 .. L - q_begin - 1 of q (the chunk's qkv rows,
 *   '(qkv h d)', sequences q_outer_stride tokens apart, same inner / token strides) and the output rows are written alike to
 *   out (out_outer_stride).  The cost grows with the key count only.                                                      */
int mv2_attention_tail(const mv2_attn_args* a, const void* q, int64_t q_outer_stride, int q_begin, void* out,
                       int64_t out_outer_stride, void* stream);
/* mv2_gateloop_scan_state: mv2_gateloop_scan starting from s_{-1} = state (fp32 [B][P][C]) instead of 0; the state after
 *   the last frame is written back to it.                                                                                  */
int mv2_gateloop_scan_state(const void* qkva, const void* res, void* out, int dtype, int B, int T, int P, int C, float* state,
                            void* stream);

#ifdef __cplusplus
}
#endif
#endif /* MAGVIT2_B200_H */
