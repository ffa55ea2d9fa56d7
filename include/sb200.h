/*
 * sb200.h — C ABI of the sliders_b200 CUDA extension (libsb200.so, sm_90a only).
 *
 * This is the drop-in boundary for the per-timestep UNet denoise of rohitgandikota/sliders. The reference
 * has no FFI of its own (it is pure Python on top of diffusers/torch); the entry points below are what a
 * Python host binds with ctypes (see INTEGRATION.md) and each one names the reference call it replaces
 * (paths relative to the reference repo).
 *
 * Conventions
 *   - every function returns 0 on success, a negative sb200_status on failure; the message of the last
 *     failure on the calling thread is returned by sb200_last_error();
 *   - no function allocates device memory, owns a buffer or synchronises: the caller (torch) owns every
 *     tensor and passes raw device pointers, element counts / strides in ELEMENTS, and the cudaStream_t
 *     (as void*) the work is enqueued on; all entry points are capturable in a CUDA graph;
 *   - activations are bf16, channels-last: an image tensor is [B, H, W, C] == a token matrix [B*H*W, C];
 *   - nothing throws across the boundary; shapes are validated on the host.
 */
#ifndef SB200_H_
#define SB200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef enum sb200_status {
  SB200_OK = 0,
  SB200_ERR_INVALID = -1,   /* bad shape / alignment / flag combination */
  SB200_ERR_CUDA = -2,      /* a CUDA runtime / driver call failed */
  SB200_ERR_UNSUPPORTED = -3 /* device is not sm_90 */
} sb200_status;

/* epilogue flags of sb200_gemm / sb200_conv3x3 */
enum {
  SB200_EPI_BIAS = 1,     /* + bias[n] */
  SB200_EPI_ROWBIAS = 2,  /* + rowbias[(m / rows_per_batch) * N + n]   (ResnetBlock2D time-embedding add) */
  SB200_EPI_RESID = 4,    /* + resid[m * ldr + n] */
  SB200_EPI_GEGLU = 8,    /* out[m, j] = acc[m, j] * gelu_erf(acc[m, N/2 + j]),  j < N/2 */
  SB200_EPI_LORA = 16     /* + scale * (X . down^T) . up^T, rank r, computed in the same tile loop */
};

/* ABI / build identification: "sb200 <version> sm_90a". */
const char* sb200_version(void);
const char* sb200_last_error(void);

/* Per-device context: caches TMA descriptors and the SM count. */
int sb200_create(int device, void** handle);
int sb200_destroy(void* handle);

/* LoRA side inputs of a fused GEMM / conv (reference: LoRAModule.forward, trainscripts/textsliders/lora.py:108-112).
 *   down : [rt, K] bf16, row j = lora_down.weight row (conv: [r, kh, kw, Cin] flattened tap-major); rows
 *          beyond the used ranks must be zero; rt is 16 or 32.
 *   up   : [N, r] FP32 (lora_up.weight, widened once at pack time so the epilogue spends no cycles on
 *          conversion); output column n uses down rows [(n / group_n) * r, +r), so one call
 *          can carry several adapted leaves that share an input (to_q|to_k|to_v fused: group_n = C).
 *   scale: multiplier * alpha / rank, a run-time scalar (the slider value changes per denoise step,
 *          eval-scripts/generate_images_xl.py:327-330).
 *   scale_dev: optional device pointer to one float multiplied into scale when the kernel runs, so a
 *          captured CUDA graph can be replayed with a different slider value (NULL = unused). */
typedef struct sb200_lora {
  const void* down;
  const void* up;
  int r;
  int rt;
  int group_n;
  float scale;
  const float* scale_dev;
} sb200_lora;

/* out[M, N] = epilogue( X[M, K] . W[N, K]^T )  — every nn.Linear on the path and the 1x1 conv_shortcut.
 * Replaces: torch Linear inside diffusers Attention / FeedForward / Transformer2DModel as called from
 * trainscripts/textsliders/train_util.py:242-247, with lora.py:108-112 folded in.
 * X may be split along K into two sources (skip-connection concat): columns [0, K0) come from x0 and
 * [K0, K) from x1 (x1 == NULL, K0 == K for a single source). K0 and K must be multiples of 64, N of 16.
 * bn is the N tile (0 = choose by the cost model; | 0x1000 forces the CTA-pair (cta_group::2) kernel,
 * | 0x2000 the single-CTA kernel — used by the tests). */
int sb200_gemm(void* handle, void* stream, const void* x0, int ldx0, const void* x1, int ldx1, int K0,
               const void* w, int ldw, void* out, int ldo, int M, int N, int K, int flags,
               const void* bias, const void* rowbias, int rows_per_batch, const void* resid, int ldr,
               const sb200_lora* lora, int bn);

/* LayerNorm folded into the projection that consumes it (BasicTransformerBlock: norm1 -> attn1.to_q|k|v, norm2 ->
 * attn2.to_q, norm3 -> ff GEGLU; diffusers models/attention.py).  With W' = W * gamma (per input column),
 *   LN(x) . W^T + b  =  rstd[m] * (x . W'^T)[m, n]  -  rstd[m] * mean[m] * c[n]  +  d[n],
 *   c[n] = sum_k W'[n, k],  d[n] = sum_k beta[k] W[n, k] + b[n],
 * so the kernel multiplies the UN-normalised rows by W' and its epilogue applies the per-row (mean, rstd), which it
 * derives from per-row partial sums (sum x, sum x^2) that the GEMM producing x left behind (`rowstats` below).  The
 * LoRA-down rows are folded the same way (c_lora / d_lora over the rt stacked rows). */
typedef struct sb200_lnfold {
  const float* stats;   /* [parts, M, 2] partial (sum, sum of squares) per row of x, fp32 (part-major) */
  int parts;
  int C;                /* row length of x the statistics run over (= K) */
  float eps;
  const float* c;       /* [N] */
  const float* d;       /* [N]  (includes the bias: call without SB200_EPI_BIAS) */
  const float* c_lora;  /* [rt] or NULL */
  const float* d_lora;  /* [rt] or NULL */
} sb200_lnfold;

/* sb200_gemm with the two LayerNorm-fusion hooks:
 *   ln        (optional) this projection consumes LN(x): see sb200_lnfold;
 *   rowstats  (optional) [rowstats_cap, M, 2] fp32: the epilogue leaves per-row partial (sum, sum of squares) of the
 *             bf16 values it writes, one slot per N tile (part-major); *rowstats_parts receives the number of slots
 *             used per row (<= rowstats_cap, else SB200_ERR_INVALID).  Written without atomics: every slot has one
 *             owner, so the statistics are bit-reproducible. */
int sb200_gemm_ln(void* handle, void* stream, const void* x0, int ldx0, const void* x1, int ldx1, int K0,
                  const void* w, int ldw, void* out, int ldo, int M, int N, int K, int flags,
                  const void* bias, const void* rowbias, int rows_per_batch, const void* resid, int ldr,
                  const sb200_lora* lora, int bn, const sb200_lnfold* ln, float* rowstats, int rowstats_cap,
                  int* rowstats_parts);

/* 3x3 convolution, padding 1, stride 1 or 2, as an implicit GEMM over NHWC activations.
 * Replaces: torch Conv2d inside diffusers ResnetBlock2D / Downsample2D / Upsample2D (same call site).
 *   x0/x1: [B, Hin, Win, C0] / [B, Hin, Win, C1] (x1 may be NULL), pixel strides ldx0 / ldx1 elements;
 *   w    : [Cout, 3, 3, C0 + C1] bf16 (tap-major repack of the HF [Cout, Cin, 3, 3] weight);
 *   out  : [B, Hout, Wout, Cout], Hout = Hin / stride.
 * C0, C1 multiples of 64, Cout of 16. Epilogue flags as sb200_gemm (no GEGLU). */
int sb200_conv3x3(void* handle, void* stream, const void* x0, int ldx0, const void* x1, int ldx1, int C0,
                  int C1, const void* w, void* out, int ldo, int B, int Hin, int Win, int Cout,
                  int stride, int flags, const void* bias, const void* rowbias, const void* resid,
                  int ldr, const sb200_lora* lora, int bn);

/* softmax(Q K^T * scale) V per (batch, head); head_dim a multiple of 8 up to 192 (SDXL 64; SD1.x 40 / 80 / 160).
 * Q/K/V/O are token matrices with row strides in elements; head h occupies columns [h*head_dim, (h+1)*head_dim).
 * Replaces the attention processor called by diffusers Attention (xformers / SDPA; train_lora_xl.py:79-80).
 *   Q: [B*Sq, ldq]  K,V: [B*Skv, ldk/ldv]  O: [B*Sq, ldo] */
int sb200_attention(void* handle, void* stream, const void* q, int ldq, const void* k, int ldk,
                    const void* v, int ldv, void* o, int ldo, int B, int heads, int Sq, int Skv,
                    int head_dim, float scale, float* lse /* optional [B, heads, Sq] fp32, for sb200_attention_bwd */);

/* ------------------------------------------------------------------------------------------------------------------
 * Backward-to-LoRA pass: `loss.backward()` at trainscripts/textsliders/train_lora_xl.py:345 (train_lora.py:298,
 * imagesliders/train_lora-scale-xl.py:340,372) through the frozen UNet to the lora_down / lora_up weights
 * (lora.py:108-112), and `optimizer.step()` (:346; AdamW built at train_util.py:362-363).
 * Dense input gradients reuse sb200_gemm / sb200_conv3x3 with transposed weights (dX = dY W; for a 3x3 conv the
 * flipped-tap, channel-transposed weight; for stride 2 on the sb200_zero_stuff'ed gradient).
 * ---------------------------------------------------------------------------------------------------------------- */

/* Flash-attention backward.  q/k/v/o/dout and lse as in sb200_attention; dsum: caller scratch [B*heads*Sq] fp32.
 * dq always; dk and dv both or neither (NULL for cross-attention whose K/V need no gradient). */
int sb200_attention_bwd(void* handle, void* stream, const void* q, int ldq, const void* k, int ldk, const void* v,
                        int ldv, const void* o, int ldo, const void* dout, int lddo, const float* lse, float* dsum,
                        void* dq, int lddq, void* dk, int lddk, void* dv, int lddv, int B, int heads, int Sq,
                        int Skv, int head_dim, float scale);

/* sb200_attention_bwd with caller scratch for a query-split dK / dV.  When the keys fit one resident tile (Skv <= 128)
 * and heads * B leaves most of the 132 SMs of an H100 idle (cross-attention: 8 CTAs for SD1.x at batch 1), the dV and
 * dK launches run SB200_ATTN_BWD_SPLITS query ranges per (head, batch) as separate CTAs that write fp32 partial tiles to
 * ws, and a reduction sums them in split order (no atomics: bit-reproducible).  Other shapes take the unsplit path and
 * leave ws untouched.  dQ is computed exactly as by sb200_attention_bwd.  The split count depends on the shape only.
 * ws: SB200_ATTN_BWD_WS_FLOATS(B, heads, Sq, Skv, head_dim) floats. */
#define SB200_ATTN_BWD_SPLITS_WANT(B, heads, Sq) \
  ((132 + (B) * (heads) - 1) / ((B) * (heads)) < ((Sq) + 63) / 64 ? (132 + (B) * (heads) - 1) / ((B) * (heads)) : ((Sq) + 63) / 64)
#define SB200_ATTN_BWD_SPLITS(B, heads, Sq, Skv) \
  (((Skv) <= 128 && 2 * (B) * (heads) <= 132) ? SB200_ATTN_BWD_SPLITS_WANT(B, heads, Sq) : 1)
#define SB200_ATTN_BWD_WS_FLOATS(B, heads, Sq, Skv, head_dim) \
  ((size_t)2 * SB200_ATTN_BWD_SPLITS(B, heads, Sq, Skv) * (B) * (Skv) * (heads) * (head_dim))
int sb200_attention_bwd_ws(void* handle, void* stream, const void* q, int ldq, const void* k, int ldk, const void* v,
                           int ldv, const void* o, int ldo, const void* dout, int lddo, const float* lse, float* dsum,
                           void* dq, int lddq, void* dk, int lddk, void* dv, int lddv, int B, int heads, int Sq,
                           int Skv, int head_dim, float scale, float* ws, size_t ws_floats);

/* out[M, N] (fp32, row stride ldo) = X[M, K] . W[N, K]^T as a split-K GEMM for few rows and a long K: the gradient
 * w.r.t. encoder_hidden_states, d_ctx = dKV_all . W_kv, where K runs over the stacked to_k | to_v rows of every
 * cross-attention block (77 * B rows, K up to 166 400 for SDXL).  Each CTA of the wgmma GEMM owns one 128 x bn tile
 * and one range of SB200_GEMM_SPLITK_KB k-blocks (64 deep) and stores its fp32 accumulator tile to ws; a reduction
 * sums the splits in order (no atomics: bit-reproducible).  The split depends on the shape only, sized for about one
 * wave on 132 SMs.  N a multiple of 16, K and the leading dims multiples of 8.
 * ws: SB200_GEMM_SPLITK_WS_FLOATS(M, N, K) floats. */
#define SB200_GEMM_SPLITK_TILES(M, N) ((((M) + 127) / 128) * ((N) % 128 == 0 ? (N) / 128 : ((N) + 63) / 64))
#define SB200_GEMM_SPLITK_KB_(M, N, K) \
  ((((K) + 63) / 64 + (132 + SB200_GEMM_SPLITK_TILES(M, N) - 1) / SB200_GEMM_SPLITK_TILES(M, N) - 1) / \
   ((132 + SB200_GEMM_SPLITK_TILES(M, N) - 1) / SB200_GEMM_SPLITK_TILES(M, N)))
#define SB200_GEMM_SPLITK_KB(M, N, K) (SB200_GEMM_SPLITK_KB_(M, N, K) < 8 ? 8 : SB200_GEMM_SPLITK_KB_(M, N, K))
#define SB200_GEMM_SPLITK_SPLITS(M, N, K) ((((K) + 63) / 64 + SB200_GEMM_SPLITK_KB(M, N, K) - 1) / SB200_GEMM_SPLITK_KB(M, N, K))
#define SB200_GEMM_SPLITK_WS_FLOATS(M, N, K) ((size_t)SB200_GEMM_SPLITK_SPLITS(M, N, K) * (M) * (N))
int sb200_gemm_splitk_f32(void* handle, void* stream, const void* x, int ldx, const void* w, int ldw, float* out,
                          int ldo, int M, int N, int K, float* ws, size_t ws_floats);

/* GroupNorm(+SiLU) backward w.r.t. the input (gamma / beta are frozen).  fwd_stats: the [B][groups][2] (mean, rstd)
 * block the forward left at stats_ws + SB200_GN_STATS_OFFSET(B, groups); ws: SB200_GN_WS_FLOATS scratch.
 * dx = dGN(dy) (+ add), written as the channel concat [B, HW, C0 + C1] with row stride lddx. */
#define SB200_GN_STATS_OFFSET(B, groups) ((size_t)(B) * (groups) * 2 * 128)
int sb200_groupnorm_bwd(void* handle, void* stream, const void* x0, int ldx0, int C0, const void* x1, int ldx1,
                        int C1, const void* gamma, const void* beta, const void* dy, int lddy, const void* add,
                        int ldadd, void* dx, int lddx, int B, int HW, int groups, int silu, const float* fwd_stats,
                        float* ws);

/* LayerNorm backward w.r.t. the input: dx = dLN(dy) (+ add). */
int sb200_layernorm_bwd(void* handle, void* stream, const void* x, int ldx, const void* gamma, const void* dy,
                        int lddy, const void* add, int ldadd, void* dx, int lddx, int M, int C, float eps);

/* Unfused GEGLU for the training forward (pre = [a | g], out = a * gelu(g)) and its backward. */
int sb200_geglu(void* handle, void* stream, const void* pre, int ldp, void* out, int ldo, int M, int F);
int sb200_geglu_bwd(void* handle, void* stream, const void* pre, int ldp, const void* dout, int lddo, void* dpre,
                    int lddp, int M, int F);

/* out = a + b (+ c): gradient joins at residual / skip connections (2-D bf16, row strides in elements). */
int sb200_add(void* handle, void* stream, const void* a, int lda, const void* b, int ldb, const void* c, int ldc,
              void* out, int ldo, int M, int C);

/* Upsample2D (nearest x2) backward: dy [B,2H,2W,C] -> dx [B,H,W,C]. */
int sb200_upsample2x_bwd(void* handle, void* stream, const void* dy, void* dx, int B, int H, int W, int C);
/* z[b,2i,2j,:] = dy[b,i,j,:], zeros elsewhere ([B,2Ho,2Wo,C]): input of the stride-1 conv that yields the input
 * gradient of a stride-2 conv (Downsample2D). */
int sb200_zero_stuff(void* handle, void* stream, const void* dy, void* z, int B, int Ho, int Wo, int C);
/* conv_out (C -> 4, 3x3) backward: d_eps NCHW [B,4,H,W] (fp32 or bf16) -> dx NHWC [B,H,W,C]. w: [4,3,3,C]. */
int sb200_conv_out_bwd(void* handle, void* stream, const void* deps, int deps_f32, const void* w, void* dx, int B,
                       int H, int W, int C);
/* out[b, c] = sum_hw dy[b, hw, c] (fp32): gradient reaching time_emb_proj's output. */
int sb200_colsum(void* handle, void* stream, const void* dy, int ld, float* out, int B, int HW, int C);

/* Rank-r (r = 4 or 8) LoRA gradient pieces for y = W x + s * up (down x), lora.py:108-112:
 *   t = x down^T, u = dY up        : sb200_lora_proj   (T[M,r] (+)= A[M,C] Bt[r,C]^T, fp32 out)
 *   d_up = s dY^T t, d_down = s u^T x : sb200_lora_wgrad  (G[c*gs_c + j*gs_r] (+)= scale * sum_m A[m,c] T[m,j])
 *   dX += s u down                 : sb200_lora_rank_update
 * and the 3x3-conv forms (down is a 3x3 conv with the leaf's stride, D = lora_down packed [r,3,3,C]).
 * ws: SB200_WGRAD_WS_FLOATS(C, r) floats (C = 9 * channels for the conv form). */
#define SB200_WGRAD_CBLOCKS(C) (((C) / 8 + 31) / 32)
#define SB200_WGRAD_CHUNKS(cblocks) ((264 + (cblocks) - 1) / (cblocks) > 256 ? 256 : (264 + (cblocks) - 1) / (cblocks))
#define SB200_WGRAD_WS_FLOATS(C, r) ((size_t)SB200_WGRAD_CHUNKS(SB200_WGRAD_CBLOCKS(C)) * (C) * (r))
int sb200_lora_proj(void* handle, void* stream, const void* A, int lda, const void* Bt, int ldb, float* T, int M,
                    int C, int r, int accumulate);
int sb200_lora_wgrad(void* handle, void* stream, const void* A, int lda, const float* T, float* G, int gs_c,
                     int gs_r, float scale, int accumulate, int M, int C, int r, float* ws);
int sb200_lora_rank_update(void* handle, void* stream, void* dX, int ldx, const float* U, const void* D, int ldd,
                           float scale, int M, int C, int r);
int sb200_lora_conv_proj(void* handle, void* stream, const void* x0, int ldx0, int C0, const void* x1, int ldx1,
                         int C1, const void* D, float* T, int B, int H, int W, int stride, int r);
int sb200_lora_conv_wgrad(void* handle, void* stream, const void* x0, int ldx0, int C0, const void* x1, int ldx1,
                          int C1, const float* U, float* G, float scale, int accumulate, int B, int H, int W,
                          int stride, int r, float* ws);
int sb200_lora_conv_rank_update(void* handle, void* stream, void* dX, const float* U, const void* D, float scale,
                                int B, int H, int W, int C, int stride, int r);

/* torch.optim.AdamW step on bf16 parameters with bf16 moments (every intermediate torch materialises as a bf16
 * tensor is rounded to bf16).  table: device array of n_tensors records {p, g, m, v: device pointers; n: int64}. */
int sb200_adamw(void* handle, void* stream, const void* table, int n_tensors, long long max_numel, double lr,
                double beta1, double beta2, double eps, double weight_decay, int step);

/* torch.optim.Adam step (L2 weight decay folded into the gradient, no amsgrad) on fp32 parameters with fp32
 * moments: the optimiser of null-text inversion over the [1, 77, D] unconditional embedding.  table: device array of
 * n_tensors records {p, g, m, v: fp32 device pointers; n: int64}. */
int sb200_adam_f32(void* handle, void* stream, const void* table, int n_tensors, long long max_numel, double lr,
                   double beta1, double beta2, double eps, double weight_decay, int step);

/* GroupNorm (+ optional SiLU) over an NHWC tensor that may be the channel concat of two sources.
 * Replaces torch GroupNorm + SiLU in ResnetBlock2D / Transformer2DModel / conv_norm_out.
 * stats_ws: caller-owned fp32 scratch of at least SB200_GN_WS_FLOATS(B, groups) floats. The reduction is
 * atomic-free, so results are bit-reproducible run to run. */
#define SB200_GN_WS_FLOATS(B, groups) ((size_t)(B) * (groups) * 2 * (128 + 1))
int sb200_groupnorm(void* handle, void* stream, const void* x0, int ldx0, int C0, const void* x1,
                    int ldx1, int C1, const void* gamma, const void* beta, void* out, int ldo, int B,
                    int HW, int groups, float eps, int silu, float* stats_ws);

/* LayerNorm over the last dim of [M, C]. */
int sb200_layernorm(void* handle, void* stream, const void* x, int ldx, const void* gamma,
                    const void* beta, void* out, int ldo, int M, int C, float eps);

/* Small dense layers with M <= 64 rows (time / add embeddings, time_emb_proj):
 * y = act_in(x)[M, K] . W[N, K]^T + bias (+ LoRA);  act_in: 0 none, 1 SiLU;  resid (row stride N) may be NULL;
 *   act_out 0: out = y + resid      act_out 1: out = SiLU(y) + resid      act_out 2: out = SiLU(bf16(y + resid))
 * (2 is how the summed time embedding reaches every ResnetBlock2D: emb is a bf16 tensor, then SiLU). */
int sb200_small_linear(void* handle, void* stream, const void* x, int ldx, const void* w, int ldw,
                       const void* bias, void* out, int ldo, int M, int N, int K, int act_in,
                       int act_out, const sb200_lora* lora, const void* resid);

/* Sinusoidal embedding (diffusers get_timestep_embedding, flip_sin_to_cos=True, shift 0):
 * out[i, :] = [cos(v_i f_j) | sin(v_i f_j)], f_j = exp(-ln(10000) j / (dim/2)); fp32 math, bf16 out. */
int sb200_sinusoid(void* handle, void* stream, const float* values, int n, int dim, void* out, int ldo);

/* conv_in: 3x3, 4 -> Cout, NCHW fp32/bf16 latent in, NHWC bf16 out. w: [Cout, 3, 3, 4]. */
int sb200_conv_in(void* handle, void* stream, const void* latent_nchw, int latent_is_f32, const void* w,
                  const void* bias, void* out, int B, int H, int W, int Cout);
/* conv_out: 3x3, Cin -> 4 on an NHWC bf16 tensor (already normalised + SiLU), NCHW out (bf16 or fp32).
 * w: [4, 3, 3, Cin]. */
int sb200_conv_out(void* handle, void* stream, const void* x, const void* w, const void* bias, void* out,
                   int out_is_f32, int B, int H, int W, int Cin);

/* nearest-neighbour x2 upsample of an NHWC tensor (Upsample2D before its conv). */
int sb200_upsample2x(void* handle, void* stream, const void* x, void* out, int B, int H, int W, int C);

/* Classifier-free guidance + DDIM step on NCHW latents (train_util.py:250-253 + scheduler.step, :291):
 *   eps = eps_u + g (eps_c - eps_u);  x0 = (x - sqrt(1-a_t) eps) / sqrt(a_t);
 *   x_prev = sqrt(a_prev) x0 + sqrt(1-a_prev) eps.
 * eps2 holds the unconditional batch followed by the conditional batch (n elements each). If x is NULL
 * only the guided eps is written to eps_out. */
int sb200_cfg_ddim(void* handle, void* stream, const void* eps2, int eps_is_f32, float g, const void* x,
                   float a_t, float a_prev, void* x_prev, void* eps_out, int out_is_f32, int64_t n);

/* Classifier-free guidance + a scheduler step that is affine in (x, eps): x_prev = cx x + ce eps with host-side
 * coefficients.  EulerDiscreteScheduler.step (the scheduler the SDXL pipeline of eval-scripts/generate_images_xl.py:358
 * carries): cx = 1, ce = sigma_next - sigma. */
int sb200_cfg_step(void* handle, void* stream, const void* eps2, int eps_is_f32, float g, const void* x, float cx,
                   float ce, void* x_prev, void* eps_out, int out_is_f32, int64_t n);

/* Loss of one null-text inversion inner step (fp32, n elements each):
 *   eps = eps_u + g (eps_c - eps_u);  x_rec = cx x + ce eps  (a scheduler step affine in (x, eps));
 *   loss = mean((x_rec - target)^2)
 * mode 0 writes *loss (two-stage reduction over SB200_GUIDED_LOSS_BLOCKS(n) partial sums in ws, no atomics);
 * mode 1 writes d_eps_u = dloss[0] (1 - g) ce 2 (x_rec - target) / n, dloss a device scalar (the incoming gradient). */
#define SB200_GUIDED_LOSS_BLOCKS(n) ((n) / 2048 + 1 > 256 ? 256 : (n) / 2048 + 1)
int sb200_guided_step_loss(void* handle, void* stream, const float* eps_u, const float* eps_c, float g, const float* x,
                           float cx, float ce, const float* target, int64_t n, int mode, float* loss, float* ws,
                           const float* dloss, float* d_eps_u);

#ifdef __cplusplus
}
#endif
#endif /* SB200_H_ */
