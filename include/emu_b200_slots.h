/* emu_b200 — C ABI of slot mode: the LLaMA KV cache as independent slots, for continuous batching.
 *
 * In slot mode every cache row is a slot that holds one sequence of its own length.  Sequences join (prefill into free
 * slots) and leave between decode steps while the other slots keep decoding; one emu_llm_decode advances every live slot
 * by one token.  A beam search takes one slot per beam: the prompt joins into one slot and is forked to the others, which
 * form its group.  Conventions as in emu_b200.h (device pointers unless marked HOST, the caller's stream, no
 * synchronisation, EMU_* return codes); every argument is checked before any CUDA call.
 *
 * Not available with EMU_KV_COPY=1 or tensor parallelism (EMU_ERR_UNSUPPORTED).  In slot mode emu_llm_prefill and
 * emu_llm_expand return EMU_ERR_STATE, emu_llm_reset leaves slot mode, and emu_llm_decode works per slot:
 *   - B may be anything from the highest occupied slot + 1 up to n_slots.  Free slots below B are computed, their outputs
 *     are meaningless, and they write only into their own cache row; their position stays 0.
 *   - live slots advance by one; "KV cache full" is checked per live slot and names it.
 *   - beam_src_idx [B] re-parents every slot up to its own length; it may map a slot only to a slot of its own group
 *     (identity for every slot outside a beam group).
 */
#ifndef EMU_B200_SLOTS_H
#define EMU_B200_SLOTS_H

#include "emu_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* Forget the cache and enter slot mode with n_slots (1 .. llm_max_batch) slots, all free. */
int emu_llm_slots_begin(EmuEngine* e, int n_slots, emu_stream_t s);

/* Prefill n new sequences into the free slots host_slots[0..n) (HOST int32, distinct), with HF positions
 * (position = index among the unmasked tokens).  inputs_embeds [n, N, hidden] bf16; attention_mask [n, N] int32, left
 * padded, or NULL = no padding; logits_last [n, vocab] fp32 (logits of every sequence's last position) or NULL.
 * The slots' length becomes N.  Live slots keep their cache untouched.  Joining an occupied slot: EMU_ERR_STATE. */
int emu_llm_join(EmuEngine* e, const int32_t* host_slots, int n, const void* inputs_embeds, const int32_t* attention_mask,
                 int N, float* logits_last, emu_stream_t s);

/* The free slots host_dst_slots[0..n) (HOST) continue the sequence of the live slot src_slot (beam expansion): no KV is
 * moved, the row table the decode attention reads through is copied.  Source and destinations form one group. */
int emu_llm_fork(EmuEngine* e, int src_slot, const int32_t* host_dst_slots, int n, emu_stream_t s);

/* Free the live slots host_slots[0..n) (HOST).  A beam group leaves together: every slot of a group named here must have
 * all of its group named. */
int emu_llm_leave(EmuEngine* e, const int32_t* host_slots, int n, emu_stream_t s);

/* The cached length of a slot (0 = free), from the host mirror; -1 outside slot mode or for a bad index. */
int emu_llm_slot_len(EmuEngine* e, int slot);

#ifdef __cplusplus
}
#endif
#endif /* EMU_B200_SLOTS_H */
