/* emu_b200 — C ABI of the decode-step kernels as stand-alone operators.
 *
 * Every generated token runs the same few small kernels after its projections: RoPE plus the KV-cache append, attention
 * over the cache through the beam row table, beam re-parenting (row-table update or cache reorder) and the greedy argmax.
 * Prefill into chosen cache rows (a continuous-batching join) runs the prefill attention with a per-sequence cache row.
 * These entry points call exactly the launchers the engine calls, so tests and micro-benchmarks reach the product path
 * at any shape.  Conventions as in emu_b200.h: device pointers, the caller's stream, no synchronisation, EMU_* return
 * codes.  Every argument is checked before any CUDA call: NULL required pointers, a batch outside 1..32, an unsupported
 * head width and a non-positive size are EMU_ERR_INVALID.
 *
 * Layouts (bf16 unless noted):
 *   KV cache of one layer   [rows][H][t_max][D]; q and k head dims pair-interleaved (element 2j = original j,
 *                           2j+1 = original j + D/2), v in natural order
 *   row table `indir`       int32 [rows][t_max]: the cache row that holds token t of sequence b
 *   rope tables cos / sin   [positions][D/2]
 */
#ifndef EMU_B200_OPS_H
#define EMU_B200_OPS_H

#include "emu_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* Decode attention, one query per sequence: out[b] = softmax(scale q[b] K^T) V over the tokens t in [start[b], pos[b]] of
 * sequence b, read from cache row indir[b][t] (indir NULL: row b).  q, out [B, H*D]; pos, start int32 [B] (start NULL = 0).
 * B 1..32, D 64 or 128.  max_len_hint (1..t_max) bounds every pos[b] + 1 and sets the split-KV count like the engine, which
 * passes t_max.  The split workspace and combine counters are owned here. */
int emu_op_attn_decode_rows(const void* q, const void* k_cache, const void* v_cache, int B, int H, int D, int t_max,
                            const int32_t* pos, const int32_t* start, const int32_t* indir, float scale, void* out,
                            int max_len_hint, emu_stream_t s);

/* RoPE + KV-cache append.  qkv [B, N, 3*H*D] (q heads | k heads | v heads).  Token n of batch b goes to cache slot
 * p + n of row kv_row[b] (kv_row NULL: row b), p = pos_dev[b] (device int32 [B]) or pos0 when pos_dev is NULL, and is
 * rotated at position max(0, p + n - pos_off[b]) (pos_off NULL = 0).  The rotated q is written in place, or compact
 * [B*N, H*D] to q_out when it is given (the decode form).  B 1..32, D 64 or 128. */
int emu_op_rope_kv_write(void* qkv, int B, int N, int H, int D, const void* rope_cos, const void* rope_sin,
                         const int32_t* pos_off, int pos0, const int32_t* pos_dev, void* q_out, const int32_t* kv_row,
                         void* k_cache, void* v_cache, int t_max, emu_stream_t s);

/* Beam re-parenting of the row table, in place: indir[b][t] <- indir[src_idx[b]][t] for b < B and t < n_tok, and with
 * row_len (device int32 [B]) only for t < row_len[b].  B 1..32, 1 <= n_tok <= t_max. */
int emu_op_kv_indir_update(int32_t* indir, const int32_t* src_idx, const int32_t* row_len, int B, int t_max, int n_tok,
                           emu_stream_t s);

/* Beam re-parenting by moving the cache, in place (HF _reorder_cache): cache [outer][Bcap][H][t_max][D], row b <- row
 * src_idx[b] for b < B and the slots t < n_used_tokens.  B 1..32 <= Bcap, D 64 or 128, 1 <= n_used_tokens <= t_max. */
int emu_op_kv_reorder(void* cache, int Bcap, const int32_t* src_idx, int B, int outer, int n_used_tokens, int H, int D,
                      int t_max, emu_stream_t s);

/* First-max argmax of every row of logits fp32 [rows, cols] (contiguous) -> out int32 [rows]. */
int emu_op_argmax_rows(const float* logits, int rows, int cols, int32_t* out, emu_stream_t s);

/* emu_op_attn_prefill with the K / V batch of query batch b taken from kv_row[b] (device int32 [B]); the k / v views then
 * span kv_rows (1..32) batch entries, the whole cache.  kv_row NULL: batch b, kv_rows ignored.  B 1..32. */
int emu_op_attn_prefill_rows(const void* q, const void* k, const void* v, void* out, int B, int H, int Nq, int Nk, int D,
                             const int64_t* st12, float scale, int causal, const int32_t* kv_start, const int32_t* kv_row,
                             int kv_rows, emu_stream_t s);

#ifdef __cplusplus
}
#endif
#endif /* EMU_B200_OPS_H */
