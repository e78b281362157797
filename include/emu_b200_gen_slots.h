/* emu_b200 — C ABI of latent slots: continuous batching for image generation.
 *
 * A slot holds one request's latents at its own denoise step.  One emu_denoise_step_slots runs one UNet pass over the
 * conditional and unconditional rows of B slots and moves every live slot one Euler step along its own schedule, with its
 * own guidance; requests join and leave between steps.  Each slot's result is the one emu_denoise_step gives that request
 * alone: the UNet treats its rows independently, and the glue below reads only the slot's own rows and parameters.
 * Conventions as in emu_b200.h (device pointers, the caller's stream, no synchronisation, EMU_* return codes); every argument
 * is checked before any CUDA call.  NULL required pointers, a slot count outside 1..32 and non-positive sizes are
 * EMU_ERR_INVALID.
 *
 * Layouts:
 *   params   DEVICE fp32 [B][4]: {sigma, sigma_next, timestep, guidance} of every slot's current step
 *   live     DEVICE int32 [B]: 0 = free slot (its UNet rows are computed and ignored, its latents are not written)
 *   UNet rows of slot b: conditional row b*cs, unconditional row ub + b*cs.  emu_denoise_step_slots uses cs = 2, ub = 1
 *   (rows 2b and 2b+1); emu_denoise_step uses [cond_1..B; uncond_1..B], cs = 1, ub = B.
 */
#ifndef EMU_B200_GEN_SLOTS_H
#define EMU_B200_GEN_SLOTS_H

#include "emu_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* One denoise iteration over B (1..32) latent slots.  latents [B, C, h, w] fp32 updated in place; ctx [2B, L, Cc],
 * text_embeds [2B, Cc] bf16 and time_ids [2B, 6] int32 hold slot b's conditional row at 2b and its unconditional row at 2b+1.
 * A slot with guidance <= 1 takes its conditional prediction as it is (its unconditional row is computed and ignored).
 * params and live are read when the step runs, so one CUDA graph per (B, pointers) serves every step.
 * EMU_ERR_UNSUPPORTED on a CFG-parallel pair (tensor parallelism with the prediction exchange). */
int emu_denoise_step_slots(EmuEngine* e, float* latents_inout, const float* params, const int32_t* live, const void* ctx,
                           int L, const void* text_embeds, const int32_t* time_ids, int B, int h, int w, emu_stream_t s);

/* The step's input glue, stand-alone: latents [B, C, HW] fp32 -> UNet input NHWC bf16 [rows, HW, Cp] (channels C..Cp-1
 * zero), bf16(bf16(latent) / sqrt(sigma_b^2 + 1)) in the `copies` (1 or 2) rows of slot b, and t_rows[row] = timestep_b (fp32).
 * params at params + b*ps (ps 0: one set for all slots, or 4).  Layout (cs, ub) is (1, B), with rows = copies*B, or (2, 1)
 * with copies = 2 and rows = 2B. */
int emu_op_denoise_prepare(const float* latents, void* xin, float* t_rows, int B, int C, int HW, int Cp, const float* params,
                           int ps, int copies, int cs, int ub, emu_stream_t s);

/* The step's output glue, stand-alone: noise prediction eps NHWC bf16 [rows, HW, ld] -> latents [B, C, HW] fp32 in place:
 * e = round_bf16(eu + round_bf16(g * round_bf16(ec - eu))) (g > 1) or ec (g <= 1), latent += e * (sigma_next - sigma), for
 * every slot with live[b] != 0 (live NULL: all).  Arguments as emu_op_denoise_prepare; C <= ld. */
int emu_op_denoise_euler(float* latents, const void* eps, const int32_t* live, int B, int C, int HW, int ld,
                         const float* params, int ps, int cs, int ub, emu_stream_t s);

#ifdef __cplusplus
}
#endif
#endif /* EMU_B200_GEN_SLOTS_H */
