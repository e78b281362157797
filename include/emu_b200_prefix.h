/* emu_b200 — C ABI of prefix caching in slot mode: a slot may leave but keep the start of its cache, and a later sequence
 * that begins with the same tokens resumes from it and prefills only what follows.
 *
 * A slot's own-row length is how many leading positions of its row-table entry are its own physical cache row: its whole
 * length if it was never re-parented, the join length for the first slot of a beam group (generated beam positions are
 * scattered over the group's rows), 0 for a forked slot.  A kept slot is free: the decode step does not advance it, and
 * emu_llm_join, emu_llm_fork, emu_llm_extend and emu_llm_copy_prefix into it discard what it held.  Free slots below the
 * decode step's B are computed as before; a kept slot is parked so that this work writes only past its kept positions.
 *
 * Conventions as in emu_b200_slots.h (HOST slot lists, the caller's stream, no synchronisation, EMU_* return codes, every
 * argument checked before any CUDA call, messages name the slot).  Under tensor parallelism every entry point that takes an
 * engine returns EMU_ERR_UNSUPPORTED.
 */
#ifndef EMU_B200_PREFIX_H
#define EMU_B200_PREFIX_H

#include "emu_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* emu_llm_leave, but slot host_slots[i] keeps its first host_keep[i] cache positions (HOST int32; 0 = keep nothing), at most
 * its own-row length and at most llm_max_seq - 1.  Its left-pad start and position offset are kept with it. */
int emu_llm_leave_keep(EmuEngine* e, const int32_t* host_slots, const int32_t* host_keep, int n, emu_stream_t s);

/* The kept length of a free slot (0 = none), from the host mirror; -1 outside slot mode or for a bad index. */
int emu_llm_slot_kept(EmuEngine* e, int slot);

/* Copy positions [0, P) of the own row of src_slot (live, or kept) into the row of the free slot dst_slot, for every layer,
 * K and V, together with its start and position offset.  dst_slot becomes kept with length P. */
int emu_llm_copy_prefix(EmuEngine* e, int src_slot, int dst_slot, int P, emu_stream_t s);

/* The free slots host_slots[0..n) become live: slot i continues at length host_prefix[i] (at most its kept length; 0 starts
 * from nothing), and host_new[i] (1 .. N) tokens, right-padded to N in inputs_embeds [n, N, hidden] bf16, are prefilled after
 * it with HF positions continuing the slot's own.  logits_last [n, vocab] fp32: the logits of each row's last real token, or
 * NULL.  One weight pass for all n rows: the rows are compacted as they are staged, so no padding token is computed. */
int emu_llm_extend(EmuEngine* e, const int32_t* host_slots, const int32_t* host_prefix, const int32_t* host_new, int n,
                   const void* inputs_embeds, int N, float* logits_last, emu_stream_t s);

/* The engine's KV cache, for inspection: *kv = its device base (bf16), dims5 = {layers * 2 (K, V), llm_max_batch rows,
 * heads, llm_max_seq, head dim}.  The pointer stays valid until the engine is destroyed. */
int emu_llm_kv_cache(EmuEngine* e, void** kv, int64_t* dims5);

/* ---- the kernel behind emu_llm_copy_prefix as a stand-alone operator (device pointers) ---- */

/* Positions [0, P) of cache row src -> row dst in every plane of a bf16 cache [outer][rows][H][t_max][D]. */
int emu_op_kv_prefix_copy(void* cache, int outer, int rows, int H, int D, int t_max, int src, int dst, int P, emu_stream_t s);

#ifdef __cplusplus
}
#endif
#endif /* EMU_B200_PREFIX_H */
