/*
 * sb200_vae.h — C ABI of the SD / SDXL VAE pieces of libsb200.so (diffusers 0.20.2 AutoencoderKL: the VAE that decodes
 * every result of eval-scripts/generate_images_xl.py:368-378 and encodes the image pairs of
 * imagesliders/train_util.py:201-235).  Conventions as in sb200.h: 0 or a negative sb200_status, caller-owned device
 * buffers, the cudaStream_t as void*, nothing allocated or synchronised, capturable in a CUDA graph.
 *
 * The VAE's resnets, GroupNorms, upsamplers and attention projections run on the entry points of sb200.h, and its
 * downsamplers on sb200_conv3x3 with SB200_CONV_PAD_BR; these entry points are the rest.
 */
#ifndef SB200_VAE_H_
#define SB200_VAE_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* Encoder.conv_in on pixels: img uint8 [B, H, W, 3] (a PIL array), normalised as v / 255 * 2 - 1 in fp32
 * (VaeImageProcessor.preprocess), then 3x3 pad 1, 3 -> Cout.  w: [Cout, 3, 3, 3] bf16; out NHWC bf16 [B, H, W, Cout]. */
int sb200_vae_conv_in_u8(void* handle, void* stream, const uint8_t* img, const void* w, const void* bias, void* out,
                         int B, int H, int W, int Cout);
/* Decoder.conv_out (3x3 pad 1, Cin -> 3) on the normalised + SiLU'd NHWC bf16 x, then VaeImageProcessor.postprocess and
 * numpy_to_pil: img[b, h, w, c] = rint(clamp(y / 2 + 0.5, 0, 1) * 255) (round half to even, as numpy's round).
 * w: [3, 3, 3, Cin] bf16.  y_f32: optional fp32 NCHW [B, 3, H, W] copy of y (the decoder's `sample`; NULL = none). */
int sb200_vae_conv_out_u8(void* handle, void* stream, const void* x, const void* w, const void* bias, uint8_t* img,
                          float* y_f32, int B, int H, int W, int Cin);
/* Encoder.conv_out (3x3 pad 1, Cin -> 8, w [8, 3, 3, Cin] bf16) + quant_conv (1x1 8 -> 8, fp32 quant_w [8, 8] and
 * quant_b [8]) + DiagonalGaussianDistribution + scaling_factor, per latent pixel:
 *   mean = m[0:4], logvar = clamp(m[4:8], -30, 20), z = (mean + exp(0.5 logvar) eps) * scaling
 * eps: fp32 NCHW [B, 4, H, W] standard normal draws (latent_dist.sample()), or NULL for latent_dist.mean / mode().
 * z: fp32 NCHW [B, 4, H, W]. */
int sb200_vae_moments(void* handle, void* stream, const void* x, const void* w, const void* bias, const float* quant_w,
                      const float* quant_b, const float* eps, float scaling, float* z, int B, int H, int W, int Cin);
/* The decoder's latent input: out = post_quant_conv(z / scaling) on fp32 NCHW [B, 4, HW] (post_w [4, 4], post_b [4]
 * fp32); sb200_conv_in (latent_is_f32) then runs Decoder.conv_in on it. */
int sb200_vae_post_quant(void* handle, void* stream, const float* z, const float* post_w, const float* post_b,
                         float scaling, float* out, int B, int HW);
/* P[r, :] = softmax(scale * S[r, :]) for fp32 scores S [rows, cols] (row stride lds), bf16 P (row stride ldp), max and
 * sum in fp32: the softmax of the VAE mid-block attention (one head of width 512 over h * w tokens), whose scores
 * sb200_gemm_splitk_f32 computes and whose P . V runs on sb200_gemm.  cols, lds, ldp multiples of 4; scale > 0. */
int sb200_softmax_rows(void* handle, void* stream, const float* s, int lds, void* p, int ldp, int rows, int cols,
                       float scale);

#ifdef __cplusplus
}
#endif
#endif /* SB200_VAE_H_ */
