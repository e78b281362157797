/* emu_b200 — C ABI of the diffusion kernels as stand-alone operators.
 *
 * Every UNet step and every VAE decode runs the same bandwidth-bound kernels around its convolutions and GEMMs: GroupNorm
 * (+SiLU), the sinusoidal timestep / time-id embedding, the skip-connection concat, nearest 2x upsample, im2col for the
 * stride-2 downsamplers, the NCHW <-> NHWC boundaries, the token mean of the text embeddings, the PNDM step of the Emu1
 * pipeline and the VAE post-process; the VAE decoder adds its single-head mid-block attention.  These entry points call
 * exactly the launchers the engine calls, so tests and micro-benchmarks reach the product path at any shape.  Conventions
 * as in emu_b200.h: device pointers, the caller's stream, no synchronisation, EMU_* return codes.  Every argument is
 * checked before any CUDA call: a NULL pointer, a non-positive size, a channel count that is not a multiple of 8 where the
 * kernel moves 8-channel vectors, and the per-entry limits below are EMU_ERR_INVALID.
 *
 * Layouts: activations NHWC bf16 ([NB, H, W, C], or [NB, HW, C]) unless noted.
 */
#ifndef EMU_B200_DIFFUSION_OPS_H
#define EMU_B200_DIFFUSION_OPS_H

#include "emu_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* y = GroupNorm(x) * w + b, then SiLU when silu != 0 (the norm output is rounded to bf16 before the SiLU, as F.silu of a
 * bf16 group_norm).  x, y [NB, HW, C]; w, b [C].  C % 8 == 0, C % groups == 0, C <= 4096.  The partial-sum scratch is
 * owned here.  Deterministic: the statistics are summed in a fixed order. */
int emu_op_groupnorm(const void* x, const void* w, const void* b, void* y, int NB, int HW, int C, int groups, float eps,
                     int silu, emu_stream_t s);

/* Sinusoidal embedding [cos(t f_j) | sin(t f_j)], f_j = exp(-ln(1e4) j / (dim/2)), of t fp32 [rows]: row r goes to output
 * row r / grp at columns col_off + (r % grp) * dim of out (row stride ld).  grp = 1 is the timestep embedding, grp = 6 the
 * SDXL time-id packing after the text embedding.  dim even, ld >= col_off + grp * dim. */
int emu_op_timestep_embedding(const float* t, void* out, int rows, int dim, int ld, int col_off, int grp, emu_stream_t s);

/* Nearest 2x upsample: x [NB, H, W, C] -> y [NB, 2H, 2W, C].  C % 8 == 0. */
int emu_op_upsample2x(const void* x, void* y, int NB, int H, int W, int C, emu_stream_t s);

/* im2col of a 3x3 pad-1 convolution with stride 1 or 2: x [NB, H, W, C] -> out [NB, Ho, Wo, 9 C], column (r*3 + s) C + c,
 * Ho = (H - 1) / stride + 1 (likewise Wo), zeros outside the image.  C % 8 == 0. */
int emu_op_im2col3x3(const void* x, void* out, int NB, int H, int W, int C, int stride, emu_stream_t s);

/* dst[r, col_off + c] = src[r, c] for r < rows, c < cols (row strides lds, ldd): the channel concat of the skip
 * connections.  cols, lds, ldd, col_off multiples of 8; lds >= cols, ldd >= col_off + cols. */
int emu_op_copy_cols(const void* src, void* dst, int64_t rows, int cols, int lds, int ldd, int col_off, emu_stream_t s);

/* x NCHW [NB, C, HW] -> y NHWC [NB, HW, Cp], channels C..Cp-1 zero, every value bf16(x * scale).  Cp >= C. */
int emu_op_nchw_to_nhwc(const void* x, void* y, int NB, int C, int HW, int Cp, float scale, emu_stream_t s);

/* x NHWC [NB, HW, ldx] (the first C channels) -> y NCHW [NB, C, HW].  ldx >= C. */
int emu_op_nhwc_to_nchw(const void* x, void* y, int NB, int C, int HW, int ldx, emu_stream_t s);

/* y [B, C] = mean over L of x [B, L, C], summed in fp32. */
int emu_op_mean_tokens(const void* x, void* y, int B, int L, int C, emu_stream_t s);

/* Image post-process: y fp32 [n_pix, C] = clamp(x / 2 + 0.5, 0, 1) with the bf16 rounding after each step, x [n_pix, ldx]
 * bf16.  ldx >= C. */
int emu_op_vae_post(const void* x, float* y, int64_t n_pix, int C, int ldx, emu_stream_t s);

/* CFG combine + one linear-multistep (PNDM / PLMS) update of the Emu1 pipeline, as emu_denoise_step_multistep runs it after
 * the UNet: lat, saved fp32 [B, C, HW]; hist fp32 [3][B, C, HW] (newest first); eps NHWC bf16 [B or 2B, HW, ld] (cond rows
 * first, then uncond when cfg = 1).  params fp32 [8] on the device: a, b, wc, w0, w1, w2, guidance, flags (bit 0 push the
 * combined eps into hist, bit 1 read x from saved, bit 2 store the incoming lat in saved);  lat = a x + b (wc e + w0 h0 +
 * w1 h1 + w2 h2).  cfg 0 or 1, ld >= C. */
int emu_op_denoise_multistep(float* lat, const void* eps, float* hist, float* saved, int B, int C, int HW, int ld,
                             const float* params, int cfg, emu_stream_t s);

/* The VAE mid-block attention core, single head: out[b] = softmax(q[b] k[b]^T / sqrt(C)) v[b], q / k / v / out [B, T, C]
 * (before to_out).  Scores are kept in fp32.  T % 8 == 0, C % 8 == 0.  The workspace is owned here. */
int emu_op_vae_attention(const void* q, const void* k, const void* v, void* out, int B, int T, int C, emu_stream_t s);

#ifdef __cplusplus
}
#endif
#endif /* EMU_B200_DIFFUSION_OPS_H */
