/* emu_b200 — C ABI of chunked prefill in slot mode: one call runs the live slots' decode step and bounded chunks of newcomers'
 * prompts as ONE pass over the weights, so a long prompt never holds the live sequences for more than one such step.
 *
 * The rows of a mixed step are packed without padding: first the B decode rows (row b = slot b, as in emu_llm_decode), then
 * the n prompt segments one after the other.  Every per-layer GEMM runs once over all M = B + sum(host_new) rows.
 *
 * Guarantee against the hazard of a mixed step: a decode row whose slot is not live (free, kept, or mid-prefill) writes NO
 * K/V in it.  (emu_llm_decode parks such a slot and lets its junk token land past its data; here that position may be one a
 * segment of the same step writes, so the junk write is dropped instead.)  Such a row's logits are meaningless.
 *
 * A segment's slot that ends the call not final is kept at prefix + new, exactly as emu_llm_leave_keep leaves a slot: free,
 * parked, its left-pad start and position offset saved.  The next chunk continues it with host_prefix = prefix + new; it may
 * also be overwritten like any kept slot.  No other slot state exists.
 *
 * Conventions as in emu_b200_slots.h / emu_b200_prefix.h (HOST slot lists, the caller's stream, no synchronisation, EMU_*
 * return codes, every argument checked before any CUDA call, messages name the slot).  Under tensor parallelism or with
 * EMU_KV_COPY=1 (neither has slot mode) the entry points that take an engine return EMU_ERR_UNSUPPORTED.
 */
#ifndef EMU_B200_CHUNKED_H
#define EMU_B200_CHUNKED_H

#include "emu_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* One mixed step.
 * Decode part (B = 0: none): as emu_llm_decode in slot mode with token_ids [B] int32 (device) — live slots below B advance by
 * one token, beam_src_idx [B] (device, or NULL) re-parents them first, "KV cache full" is checked per live slot; B must cover
 * the highest live slot and stay within n_slots.  logits [B, vocab] fp32 or NULL.
 * Prefill part (n >= 1; n = 0 is emu_llm_decode): segment i continues the free slot host_slots[i] as emu_llm_extend does — at
 * length host_prefix[i] (at most its kept length), with host_new[i] >= 1 tokens of embeds, HF positions continuing the slot's
 * own.  embeds [sum(host_new), hidden] bf16 (device), the segments back to back.  host_final[i] = 1: the slot becomes live at
 * prefix + new (at most llm_max_seq), as after emu_llm_extend; 0: it is kept at prefix + new (at most llm_max_seq - 1).
 * logits_last [n, vocab] fp32: the logits of each segment's last token, or NULL.
 * The segments' slots are distinct and not live; they may lie below B.
 * Logits rows (the decode rows and the segments' last tokens) take the prefill rule: the final norm fused into the lm_head
 * GEMV at up to 8 rows, norm then GEMM above that.  emu_llm_join and emu_llm_extend are this call with B = 0 and every
 * segment final. */
int emu_llm_step(EmuEngine* e, const int32_t* token_ids, const int32_t* beam_src_idx, int B, float* logits,
                 const int32_t* host_slots, const int32_t* host_prefix, const int32_t* host_new, const int32_t* host_final, int n,
                 const void* embeds, float* logits_last, emu_stream_t s);

/* ---- the kernels behind slot mode's prefill (emu_llm_join, emu_llm_extend and emu_llm_step all run it) as stand-alone
 * operators (device pointers, B <= 32, n <= 32) ---- */

/* RoPE + KV append of a packed mixed step: qkv [M, 3*H*D] bf16 (q / k pair-interleaved per head), M >= B + n.
 * Row b < B (decode): rotated at pos[b] - pos_off[b]; q goes compact to q_out [B, H*D]; its k / v go to slot pos[b] of cache
 * row b only if active[b] != 0.  Rows B.. (segments, seg_new[i] rows each, in order): row j of segment i is rotated at
 * seg_q0[i] + j - seg_posoff[i] (q in place) and its k / v go to slot seg_q0[i] + j of cache row seg_row[i].  Rows past the
 * last segment are not touched.  pos, pos_off, active: device int32 [B]; seg_*: device int32 [n] (seg_posoff NULL = 0).
 * Caches [rows, H, t_max, D].  D = 64 or 128. */
int emu_op_rope_kv_write_packed(void* qkv, int M, int B, int n, int H, int D, const void* rope_cos, const void* rope_sin,
                                const int32_t* pos, const int32_t* pos_off, const int32_t* active, void* q_out,
                                const int32_t* seg_row, const int32_t* seg_q0, const int32_t* seg_new, const int32_t* seg_posoff,
                                void* k_cache, void* v_cache, int t_max, emu_stream_t s);

/* Causal prefill attention over packed queries: batch b's q_len[b] queries are rows q_row0[b] .. q_row0[b] + q_len[b] - 1 of
 * ONE [rows, H, D] view of q, and its outputs the same rows of out; query i sits at key position q_off[b] + i and sees keys
 * [kv_start[b], q_off[b] + i] (kv_start NULL = 0) of K/V batch kv_row[b] (NULL = b; kv_rows = batches the K/V views span).
 * Nq = the longest q_len.  Rows of q / out outside the batches are neither read into an output nor written; keys at or past
 * q_off[b] + q_len[b] are never read into an output, so they may hold anything.  st10, in elements: {q token, q head,
 * k batch, k token, k head, v batch, v token, v head, out token, out head}.  D = 64 or 128.  Nq >= 128 runs the wgmma kernel,
 * shorter the mma.sync one. */
int emu_op_attn_prefill_packed(const void* q, const void* k, const void* v, void* out, int rows, int B, int H, int Nq, int Nk,
                               int D, const int64_t* st10, float scale, const int32_t* q_row0, const int32_t* q_len,
                               const int32_t* q_off, const int32_t* kv_start, const int32_t* kv_row, int kv_rows, emu_stream_t s);

#ifdef __cplusplus
}
#endif
#endif /* EMU_B200_CHUNKED_H */
