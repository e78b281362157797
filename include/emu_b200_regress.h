/* emu_b200 — C ABI of regression slots: Emu2-Gen's prompt encoding (EmuModel.generate_image) for every slot of slot mode at
 * once, so that newcomers' visual embeddings are regressed together and a scheduler can interleave their steps with other work.
 *
 * A regression slot holds one prompt ending in [IMG].  After its prefill it produces L embeddings of vit_width: embedding 0 is
 * project_down of the last prompt position's final-normed hidden state, and embedding k + 1 is project_down of the hidden
 * state the decoder gives for the input project_up(embedding k).  The engine keeps, per slot, in device memory: the last
 * embedding (the feedback of the next step) and the index k of the next output row.  The slots leave through emu_llm_leave.
 *
 * Bit-for-bit guarantee: a slot's embeddings depend only on its prompt, its slot index, the pool's n_slots and the B of the
 * steps it runs in.  The join normalises each segment's last row on its own and always projects n_slots rows, so it gives a
 * segment the same bits whatever else joins with it; a step projects B rows.
 *
 * Conventions as in emu_b200_slots.h (HOST slot lists, the caller's stream, no synchronisation, EMU_* return codes, every
 * argument checked before any CUDA call, messages name the slot).  Under tensor parallelism or with EMU_KV_COPY=1 (neither
 * has slot mode) they return EMU_ERR_UNSUPPORTED.  Both need the project_up and project_down weights.
 */
#ifndef EMU_B200_REGRESS_H
#define EMU_B200_REGRESS_H

#include "emu_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* Prefill n prompts into the free slots host_slots[0..n) (HOST int32, distinct) and regress their first embedding.
 * embeds [sum(host_new), hidden] bf16: the prompts back to back without padding, host_new[i] >= 1 tokens each at positions
 * 0 .. host_new[i] - 1 (at most llm_max_seq).  Slot host_slots[i] becomes live at host_new[i] and a regression slot:
 * out [n_slots, L, vit_width] bf16 gets row out[slot][0], the slot's feedback is that row and its k is 1.  Other slots'
 * rows of out are not written.  Joining an occupied slot: EMU_ERR_STATE. */
int emu_llm_regress_join(EmuEngine* e, const int32_t* host_slots, const int32_t* host_new, int n, const void* embeds, void* out,
                         int L, emu_stream_t s);

/* One regression step for every live slot below B: x = project_up(feedback); one slot-mode decode step on x (the hidden
 * state after the final norm, no lm_head); r = project_down(hidden); feedback = r; out[slot][k] = r while k < L; k += 1.
 * out [n_slots, L, vit_width] bf16.  B covers the highest live slot and stays within n_slots; every live slot below B must
 * be a regression slot (joined through emu_llm_regress_join), else EMU_ERR_STATE; free slots below B are computed and
 * dropped, as emu_llm_decode does.  "KV cache full" is checked per live slot.  A fixed launch sequence without host
 * read-back, captured as one CUDA graph per (B, out, L, stream) unless EMU_NO_GRAPH=1. */
int emu_llm_regress_step(EmuEngine* e, int B, void* out, int L, emu_stream_t s);

#ifdef __cplusplus
}
#endif
#endif /* EMU_B200_REGRESS_H */
