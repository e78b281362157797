/* emu_b200 — C ABI of prompt-lookup speculative decoding: greedy search at batch 1 that checks several drafted tokens in one
 * pass over the weights.
 *
 * A step: emu_spec_draft proposes d tokens from the token history; emu_llm_verify runs the decoder over the last committed
 * token and the d drafts (n = d + 1 rows) and takes the arg-max of every row; emu_spec_accept keeps the drafts that equal the
 * arg-max before them and appends them and the arg-max after the last of them to the history; emu_llm_commit makes those
 * positions part of the cache.  Greedy output is that of one token per step; only the number of weight passes changes.
 *
 * Conventions as in emu_b200.h: the caller's stream, no synchronisation, EMU_* return codes, every argument checked before
 * any CUDA call, emu_last_error names the cause.
 */
#ifndef EMU_B200_SPEC_H
#define EMU_B200_SPEC_H

#include "emu_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* One pass of the decoder over n <= min(8, llm_max_batch) consecutive tokens of the batch-1 sequence in plain mode, whose
 * cache holds L positions: tokens [n] (device int32), row j at position L + j (row 0 the last committed token, rows 1.. the
 * drafts).  Every layer runs the decode GEMV at B = n, RoPE and the K/V append at positions L .. L + n - 1 of the sequence's
 * cache row, and the verify attention (row j sees positions start .. L + j).  Then the final norm and lm_head of every row:
 * logits [n, vocab] fp32 and / or next_ids [n] int32 (their arg-max; rows j < ban_rows exclude ban_id), either may be NULL.
 * The cache length stays L; positions L .. L + n - 1 hold uncommitted K/V until emu_llm_commit.  Positions come from device
 * memory: the call is one CUDA graph per (n, arguments), unless EMU_NO_GRAPH=1.
 * Refusals: slot mode EMU_ERR_STATE; tensor parallelism EMU_ERR_UNSUPPORTED; no prefill EMU_ERR_STATE; batch != 1, n out of
 * range, ban_rows outside [0, n] or L + n > llm_max_seq (KV cache full) EMU_ERR_INVALID. */
int emu_llm_verify(EmuEngine* e, const int32_t* tokens, int n, float* logits, int32_t* next_ids, int ban_id, int ban_rows,
                   emu_stream_t s);

/* Keep the first m (1 <= m <= n of the last verify) positions the last verify wrote: the cache length becomes L + m.  The
 * positions after it are dead and the next verify overwrites them.  No verify since the cache last changed: EMU_ERR_STATE;
 * m out of range: EMU_ERR_INVALID. */
int emu_llm_commit(EmuEngine* e, int m, emu_stream_t s);

/* The prompt-lookup draft (transformers 5.5 PromptLookupCandidateGenerator.get_candidates) over hist[0 .. *hist_len) (device
 * int32, *hist_len >= 1): n-gram sizes min(max_ngram, len - 1) down to 1; the leftmost earlier occurrence of the history's last
 * n-gram with a non-empty continuation, at most k tokens and within min(len, max_length); cut before its first eos_id; none
 * when max_length == len + 1.  out [1 + k] (device int32): out[0] = hist[len - 1], out[1 .. 1 + d) = the draft; *out_len = d
 * (device int32). */
int emu_spec_draft(const int32_t* hist, int32_t* hist_len, int k, int max_ngram, int max_length, int eos_id, int32_t* out,
                   int32_t* out_len, emu_stream_t s);

/* Acceptance after a verify of n rows: tokens [n] the verify's input (tokens[1 ..] the drafts), next_ids [n] its arg-max.  The
 * a leading drafts equal to next_ids[0 .. a) are accepted; next_ids[0 .. a] are appended to hist at *hist_len, stopping
 * after eos_id and when the history reaches max_len entries; *hist_len advances.  stats [2] (device int32): the number of
 * tokens appended (the positions to commit) and 1 when generation has finished. */
int emu_spec_accept(int32_t* hist, int32_t* hist_len, const int32_t* tokens, const int32_t* next_ids, int n, int eos_id,
                    int max_len, int32_t* stats, emu_stream_t s);

/* The verify attention as a stand-alone operator: q [n, q_ts] bf16 (head h of row j at j * q_ts + h * D), the cache
 * [rows, H, t_max, D] bf16 of one layer, cache row `row`; query j sees positions start[0] .. pos[0] + j (device int32 [1]
 * each, start may be NULL); indir (NULL or device int32 [t_max]) the cache row holding each position; out [n, H * D] bf16.
 * n <= 8, D of 64 or 128, pos[0] + n <= t_max. */
int emu_op_attn_verify(const void* q, long q_ts, const void* k_cache, const void* v_cache, int n, int H, int D, int t_max,
                       int row, const int32_t* pos, const int32_t* start, const int32_t* indir, float scale, void* out,
                       emu_stream_t s);

#ifdef __cplusplus
}
#endif
#endif /* EMU_B200_SPEC_H */
