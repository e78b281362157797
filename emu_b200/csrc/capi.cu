// emu_b200 — C ABI wrappers for the stand-alone operators (include/emu_b200.h, "stand-alone operators").
// These expose exactly the kernels the engine launches, so the parity tests exercise the product path.
#include "common.cuh"
#include "engine.h"
#include "../../include/emu_b200_ops.h"
#include "../../include/emu_b200_prefix.h"
#include "../../include/emu_b200_chunked.h"
#include "../../include/emu_b200_gen_slots.h"
#include "../../include/emu_b200_diffusion_ops.h"
#include "../../include/emu_b200_spec.h"
#include "diffusion_common.h"

using namespace emu;

extern "C" int emu_op_gemm(const void* A, int lda, const void* W, int ldw, int M, int N, int K, const void* bias,
                           const void* residual, int ldr, int epi_mode, void* C, int ldc, int out_fp32, int force_bn,
                           emu_stream_t s) {
  if (!A || !W || !C) return EMU_ERR_INVALID;
  GemmEpilogue e;
  e.C = C; e.ldc = ldc; e.bias = (const bf16*)bias; e.residual = (const bf16*)residual; e.ldr = ldr;
  e.mode = epi_mode; e.out_fp32 = out_fp32; e.force_bn = force_bn;
  count_launch();
  return gemm_bf16((const bf16*)A, lda, (const bf16*)W, ldw, M, N, K, e, (cudaStream_t)s);
}

// the wide-decode projection kernel (weights as the 128-row MMA operand, K-split partial sums), stand-alone
extern "C" int emu_op_gemm_skinny(const void* X, int ldx, const void* W, int ldw, int B, int N, int K, const void* residual,
                                  int ldr, int epi_mode, void* C, int ldc, int out_fp32, emu_stream_t s) {
  if (!X || !W || !C) return EMU_ERR_INVALID;
  static float* ws = nullptr;
  static int* counters = nullptr;
  if (!ws) {
    if (cudaMalloc((void**)&ws, gemm_skinny_workspace_bytes()) != cudaSuccess) return EMU_ERR_NOMEM;
    if (cudaMalloc((void**)&counters, kSkinnyMaxTiles * sizeof(int)) != cudaSuccess) return EMU_ERR_NOMEM;
    if (cudaMemset(counters, 0, kSkinnyMaxTiles * sizeof(int)) != cudaSuccess) return EMU_ERR_CUDA;
  }
  GemmEpilogue e;
  e.C = C; e.ldc = ldc; e.residual = (const bf16*)residual; e.ldr = ldr; e.mode = epi_mode; e.out_fp32 = out_fp32;
  count_launch();
  return gemm_skinny_bf16((const bf16*)X, ldx, (const bf16*)W, ldw, B, N, K, e, ws, counters, (cudaStream_t)s);
}

extern "C" int emu_debug_gemm_phases(const void* A, int lda, const void* W, int ldw, int M, int N, int K, const void* bias,
                                     const void* residual, int ldr, int epi_mode, void* C, int ldc, int force_bn,
                                     unsigned long long* stamps /*[grid][8] device*/, emu_stream_t s) {
  if (!A || !W || !C || !stamps) return EMU_ERR_INVALID;
  GemmEpilogue e;
  e.C = C; e.ldc = ldc; e.bias = (const bf16*)bias; e.residual = (const bf16*)residual; e.ldr = ldr;
  e.mode = epi_mode; e.force_bn = force_bn; e.dbg = stamps;
  count_launch();
  return gemm_bf16((const bf16*)A, lda, (const bf16*)W, ldw, M, N, K, e, (cudaStream_t)s);
}

extern "C" int emu_op_conv3x3(const void* x, int NB, int H, int W, int Cin, const void* wk, int Cout, const void* bias,
                              const void* residual, void* y, emu_stream_t s) {
  if (!x || !wk || !y) return EMU_ERR_INVALID;
  GemmEpilogue e;
  e.C = y; e.ldc = Cout; e.bias = (const bf16*)bias; e.residual = (const bf16*)residual; e.ldr = Cout;
  count_launch();
  return conv3x3_bf16((const bf16*)x, NB, H, W, Cin, (const bf16*)wk, Cout, e, (cudaStream_t)s);
}

extern "C" int emu_op_gemv(const void* W, int N, int K, const void* x, int ldx, int B, const void* norm_w, float eps,
                           int mode, const void* bias, const void* residual, int ldr, void* y, int ldy, int out_fp32,
                           int pdl, emu_stream_t s) {
  if (!W || !x || !y) return EMU_ERR_INVALID;
  if (mode != EPI_NONE && mode != EPI_SWIGLU) return EMU_ERR_INVALID;
  GemvArgs a;
  a.W = (const bf16*)W; a.N = N; a.K = K; a.x = (const bf16*)x; a.ldx = ldx; a.B = B;
  a.norm_w = (const bf16*)norm_w; a.norm_eps = eps; a.mode = mode; a.bias = (const bf16*)bias;
  a.residual = (const bf16*)residual; a.ldr = ldr; a.y = y; a.ldy = ldy; a.out_fp32 = out_fp32; a.pdl = pdl;
  count_launch();
  return gemv_bf16(a, (cudaStream_t)s);
}

extern "C" int emu_debug_gemv_phases(const void* W, int N, int K, const void* x, int ldx, int B, const void* norm_w, float eps,
                                     int mode, const void* residual, int ldr, void* y, int ldy, int pdl,
                                     unsigned long long* stamps /*[grid][8] device*/, emu_stream_t s) {
  if (!W || !x || !y || !stamps) return EMU_ERR_INVALID;
  GemvArgs a;
  a.W = (const bf16*)W; a.N = N; a.K = K; a.x = (const bf16*)x; a.ldx = ldx; a.B = B;
  a.norm_w = (const bf16*)norm_w; a.norm_eps = eps; a.mode = mode;
  a.residual = (const bf16*)residual; a.ldr = ldr; a.y = y; a.ldy = ldy; a.pdl = pdl; a.dbg = stamps;
  count_launch();
  return gemv_bf16(a, (cudaStream_t)s);
}

extern "C" int emu_op_gemv_rope_qkv(const void* W, int n_heads, int head_dim, int K, const void* x, int ldx, int B,
                                    const void* norm_w, float eps, const void* rope_cos, const void* rope_sin,
                                    const int32_t* pos, const int32_t* pos_off, void* q_out, void* k_cache,
                                    void* v_cache, int t_max, emu_stream_t s) {
  if (!W || !x || !q_out || !k_cache || !v_cache || !rope_cos || !rope_sin || !pos) return EMU_ERR_INVALID;
  GemvArgs a;
  a.W = (const bf16*)W; a.N = 3 * n_heads * head_dim; a.K = K; a.x = (const bf16*)x; a.ldx = ldx; a.B = B;
  a.norm_w = (const bf16*)norm_w; a.norm_eps = eps; a.mode = GEMV_ROPE_QKV;
  a.y = q_out; a.ldy = n_heads * head_dim; a.n_heads = n_heads; a.head_dim = head_dim;
  a.rope_cos = (const bf16*)rope_cos; a.rope_sin = (const bf16*)rope_sin; a.pos = pos; a.pos_off = pos_off;
  a.k_cache = (bf16*)k_cache; a.v_cache = (bf16*)v_cache; a.t_max = t_max;
  count_launch();
  return gemv_bf16(a, (cudaStream_t)s);
}

extern "C" int emu_op_attn_prefill(const void* q, const void* k, const void* v, void* out, int B, int H, int Nq, int Nk,
                                   int D, const int64_t* st12, float scale, int causal, const int32_t* kv_start,
                                   const float* bias, emu_stream_t s) {
  if (!q || !k || !v || !out || !st12) return EMU_ERR_INVALID;
  AttnArgs a;
  a.q = (const bf16*)q; a.k = (const bf16*)k; a.v = (const bf16*)v; a.out = (bf16*)out;
  a.q_bs = st12[0]; a.q_ts = st12[1]; a.q_hs = st12[2];
  a.k_bs = st12[3]; a.k_ts = st12[4]; a.k_hs = st12[5];
  a.v_bs = st12[6]; a.v_ts = st12[7]; a.v_hs = st12[8];
  a.o_bs = st12[9]; a.o_ts = st12[10]; a.o_hs = st12[11];
  a.B = B; a.H = H; a.Nq = Nq; a.Nk = Nk; a.D = D; a.scale = scale; a.causal = causal; a.kv_start = kv_start;
  a.bias = bias;
  count_launch();
  return attn_prefill(a, (cudaStream_t)s);
}

extern "C" int emu_op_attn_decode(const void* q, const void* k_cache, const void* v_cache, int B, int H, int D,
                                  int t_max, const int32_t* pos, const int32_t* start, float scale, void* out,
                                  int max_len, emu_stream_t s) {
  if (!q || !k_cache || !v_cache || !pos || !out || B < 1 || B > 8) return EMU_ERR_INVALID;
  // scratch for the split-KV combine (sized for the largest legal problem; allocated once)
  static float* ws = nullptr;
  static int* counters = nullptr;
  static size_t ws_bytes = 0;
  const size_t need = attn_decode_workspace_bytes(B, H, D);
  if (need > ws_bytes) {
    if (ws) cudaFree(ws);
    if (counters) cudaFree(counters);
    if (cudaMalloc((void**)&ws, need) != cudaSuccess) return EMU_ERR_NOMEM;
    if (cudaMalloc((void**)&counters, (size_t)8 * 1024 * sizeof(int)) != cudaSuccess) return EMU_ERR_NOMEM;
    cudaMemset(counters, 0, (size_t)8 * 1024 * sizeof(int));
    ws_bytes = need;
  }
  if (B * H > 8 * 1024) return EMU_ERR_UNSUPPORTED;
  count_launch();
  return attn_decode((const bf16*)q, (const bf16*)k_cache, (const bf16*)v_cache, B, H, D, t_max, pos, start, scale,
                     (bf16*)out, ws, counters, max_len, 0, (cudaStream_t)s);
}

// ---- the decode-step kernels (include/emu_b200_ops.h): the engine's launchers at any shape, arguments checked first ----
static bool llm_head_dim_ok(int D) { return D == 64 || D == 128; }

extern "C" int emu_op_attn_decode_rows(const void* q, const void* k_cache, const void* v_cache, int B, int H, int D,
                                       int t_max, const int32_t* pos, const int32_t* start, const int32_t* indir, float scale,
                                       void* out, int max_len_hint, emu_stream_t s) {
  if (!q || !k_cache || !v_cache || !pos || !out) return EMU_ERR_INVALID;
  if (B < 1 || B > kLlmMaxRows || H < 1 || !llm_head_dim_ok(D) || t_max < 1) return EMU_ERR_INVALID;
  if (max_len_hint < 1 || max_len_hint > t_max) return EMU_ERR_INVALID;
  // split workspace and combine counters for kLlmMaxRows x H (re)allocated when a wider head set arrives; the kernel
  // resets every counter it uses, so they are zeroed once per allocation
  static float* ws = nullptr;
  static int* counters = nullptr;
  static int cap_h = 0, cap_d = 0;
  if (H > cap_h || D > cap_d) {
    const int h = H > cap_h ? H : cap_h, d = D > cap_d ? D : cap_d;
    if (ws) cudaFree(ws);
    if (counters) cudaFree(counters);
    ws = nullptr;
    counters = nullptr;
    cap_h = cap_d = 0;
    const size_t n_ctr = (size_t)kLlmMaxRows * h * sizeof(int);
    if (cudaMalloc((void**)&ws, attn_decode_workspace_bytes(kLlmMaxRows, h, d)) != cudaSuccess) return EMU_ERR_NOMEM;
    if (cudaMalloc((void**)&counters, n_ctr) != cudaSuccess) return EMU_ERR_NOMEM;
    if (cudaMemset(counters, 0, n_ctr) != cudaSuccess) return EMU_ERR_CUDA;
    cap_h = h;
    cap_d = d;
  }
  count_launch();
  return attn_decode((const bf16*)q, (const bf16*)k_cache, (const bf16*)v_cache, B, H, D, t_max, pos, start, scale,
                     (bf16*)out, ws, counters, max_len_hint, 0, (cudaStream_t)s, indir);
}

extern "C" int emu_op_rope_kv_write(void* qkv, int B, int N, int H, int D, const void* rope_cos, const void* rope_sin,
                                    const int32_t* pos_off, int pos0, const int32_t* pos_dev, void* q_out,
                                    const int32_t* kv_row, void* k_cache, void* v_cache, int t_max, emu_stream_t s) {
  if (!qkv || !rope_cos || !rope_sin || !k_cache || !v_cache) return EMU_ERR_INVALID;
  if (B < 1 || B > kLlmMaxRows || N < 1 || H < 1 || !llm_head_dim_ok(D) || t_max < 1 || pos0 < 0) return EMU_ERR_INVALID;
  if (!pos_dev && pos0 + N > t_max) return EMU_ERR_INVALID;
  count_launch();
  return rope_kv_write((bf16*)qkv, B, N, H, D, (const bf16*)rope_cos, (const bf16*)rope_sin, pos_off, pos0, (bf16*)k_cache,
                       (bf16*)v_cache, t_max, (cudaStream_t)s, pos_dev, (bf16*)q_out, kv_row);
}

extern "C" int emu_op_kv_indir_update(int32_t* indir, const int32_t* src_idx, const int32_t* row_len, int B, int t_max,
                                      int n_tok, emu_stream_t s) {
  if (!indir || !src_idx) return EMU_ERR_INVALID;
  if (B < 1 || B > kLlmMaxRows || t_max < 1 || n_tok < 1 || n_tok > t_max) return EMU_ERR_INVALID;
  count_launch();
  return kv_indir_update(indir, src_idx, B, t_max, n_tok, (cudaStream_t)s, row_len);
}

extern "C" int emu_op_kv_reorder(void* cache, int Bcap, const int32_t* src_idx, int B, int outer, int n_used_tokens, int H,
                                 int D, int t_max, emu_stream_t s) {
  if (!cache || !src_idx) return EMU_ERR_INVALID;
  if (B < 1 || B > kLlmMaxRows || Bcap < B || outer < 1 || H < 1 || !llm_head_dim_ok(D) || t_max < 1) return EMU_ERR_INVALID;
  if (n_used_tokens < 1 || n_used_tokens > t_max) return EMU_ERR_INVALID;
  count_launch();
  return kv_reorder((bf16*)cache, Bcap, src_idx, B, outer, n_used_tokens, H, D, t_max, (cudaStream_t)s);
}

// the verify attention of speculative decoding (include/emu_b200_spec.h), with its own workspace as above
extern "C" int emu_op_attn_verify(const void* q, long q_ts, const void* k_cache, const void* v_cache, int n, int H, int D,
                                  int t_max, int row, const int32_t* pos, const int32_t* start, const int32_t* indir,
                                  float scale, void* out, emu_stream_t s) {
  if (!q || !k_cache || !v_cache || !pos || !out) return EMU_ERR_INVALID;
  if (n < 1 || n > 8 || H < 1 || !llm_head_dim_ok(D) || t_max < 1 || row < 0 || q_ts < (long)H * D) return EMU_ERR_INVALID;
  static float* ws = nullptr;
  static int* counters = nullptr;
  static int cap_h = 0, cap_d = 0;
  if (H > cap_h || D > cap_d) {
    const int h = H > cap_h ? H : cap_h, d = D > cap_d ? D : cap_d;
    if (ws) cudaFree(ws);
    if (counters) cudaFree(counters);
    ws = nullptr;
    counters = nullptr;
    cap_h = cap_d = 0;
    if (cudaMalloc((void**)&ws, attn_verify_workspace_bytes(h, d)) != cudaSuccess) return EMU_ERR_NOMEM;
    if (cudaMalloc((void**)&counters, (size_t)h * sizeof(int)) != cudaSuccess) return EMU_ERR_NOMEM;
    if (cudaMemset(counters, 0, (size_t)h * sizeof(int)) != cudaSuccess) return EMU_ERR_CUDA;
    cap_h = h;
    cap_d = d;
  }
  count_launch();
  return attn_verify((const bf16*)q, q_ts, (const bf16*)k_cache, (const bf16*)v_cache, n, H, D, t_max, row, pos, start, scale,
                     (bf16*)out, ws, counters, t_max, (cudaStream_t)s, indir);
}

extern "C" int emu_op_argmax_rows(const float* logits, int rows, int cols, int32_t* out, emu_stream_t s) {
  if (!logits || !out || rows < 1 || cols < 1) return EMU_ERR_INVALID;
  count_launch();
  return argmax_rows(logits, rows, cols, out, (cudaStream_t)s);
}

extern "C" int emu_op_attn_prefill_rows(const void* q, const void* k, const void* v, void* out, int B, int H, int Nq, int Nk,
                                        int D, const int64_t* st12, float scale, int causal, const int32_t* kv_start,
                                        const int32_t* kv_row, int kv_rows, emu_stream_t s) {
  if (!q || !k || !v || !out || !st12) return EMU_ERR_INVALID;
  if (B < 1 || B > kLlmMaxRows || H < 1 || Nq < 1 || Nk < 1 || D < 8 || D > 160 || D % 8) return EMU_ERR_INVALID;
  if (kv_row && (kv_rows < 1 || kv_rows > kLlmMaxRows)) return EMU_ERR_INVALID;
  AttnArgs a;
  a.q = (const bf16*)q; a.k = (const bf16*)k; a.v = (const bf16*)v; a.out = (bf16*)out;
  a.q_bs = st12[0]; a.q_ts = st12[1]; a.q_hs = st12[2];
  a.k_bs = st12[3]; a.k_ts = st12[4]; a.k_hs = st12[5];
  a.v_bs = st12[6]; a.v_ts = st12[7]; a.v_hs = st12[8];
  a.o_bs = st12[9]; a.o_ts = st12[10]; a.o_hs = st12[11];
  a.B = B; a.H = H; a.Nq = Nq; a.Nk = Nk; a.D = D; a.scale = scale; a.causal = causal; a.kv_start = kv_start;
  a.kv_row = kv_row; a.kv_rows = kv_row ? kv_rows : 0;
  count_launch();
  return attn_prefill(a, (cudaStream_t)s);
}

extern "C" int emu_op_kv_prefix_copy(void* cache, int outer, int rows, int H, int D, int t_max, int src, int dst, int P,
                                     emu_stream_t s) {
  if (!cache || (reinterpret_cast<uintptr_t>(cache) & 15)) return EMU_ERR_INVALID;  // moved as 16-byte words
  if (outer < 1 || rows < 1 || H < 1 || D < 8 || D % 8 || t_max < 1) return EMU_ERR_INVALID;
  if (src < 0 || src >= rows || dst < 0 || dst >= rows || src == dst || P < 1 || P > t_max) return EMU_ERR_INVALID;
  count_launch();
  return kv_prefix_copy((bf16*)cache, outer, rows, H, D, t_max, src, dst, P, (cudaStream_t)s);
}

// ---- the kernels behind emu_llm_step (include/emu_b200_chunked.h) ----
extern "C" int emu_op_rope_kv_write_packed(void* qkv, int M, int B, int n, int H, int D, const void* rope_cos, const void* rope_sin,
                                           const int32_t* pos, const int32_t* pos_off, const int32_t* active, void* q_out,
                                           const int32_t* seg_row, const int32_t* seg_q0, const int32_t* seg_new,
                                           const int32_t* seg_posoff, void* k_cache, void* v_cache, int t_max, emu_stream_t s) {
  if (!qkv || !rope_cos || !rope_sin || !k_cache || !v_cache) return EMU_ERR_INVALID;
  if (B > 0 && (!pos || !pos_off || !active || !q_out)) return EMU_ERR_INVALID;
  if (n > 0 && (!seg_row || !seg_q0 || !seg_new)) return EMU_ERR_INVALID;
  if (B < 0 || B > kLlmMaxRows || n < 0 || n > kLlmMaxRows || B + n < 1 || M < B + n) return EMU_ERR_INVALID;
  if (H < 1 || !llm_head_dim_ok(D) || t_max < 1) return EMU_ERR_INVALID;
  count_launch();
  return rope_kv_write_packed((bf16*)qkv, M, B, n, H, D, (const bf16*)rope_cos, (const bf16*)rope_sin, pos, pos_off, active,
                              (bf16*)q_out, seg_row, seg_q0, seg_new, seg_posoff, (bf16*)k_cache, (bf16*)v_cache, t_max,
                              (cudaStream_t)s);
}

extern "C" int emu_op_attn_prefill_packed(const void* q, const void* k, const void* v, void* out, int rows, int B, int H, int Nq,
                                          int Nk, int D, const int64_t* st10, float scale, const int32_t* q_row0,
                                          const int32_t* q_len, const int32_t* q_off, const int32_t* kv_start, const int32_t* kv_row,
                                          int kv_rows, emu_stream_t s) {
  if (!q || !k || !v || !out || !st10 || !q_row0 || !q_len || !q_off) return EMU_ERR_INVALID;
  if (rows < 1 || B < 1 || B > kLlmMaxRows || H < 1 || Nq < 1 || Nk < 1 || !llm_head_dim_ok(D)) return EMU_ERR_INVALID;
  if (kv_row && (kv_rows < 1 || kv_rows > kLlmMaxRows)) return EMU_ERR_INVALID;
  AttnArgs a;
  a.q = (const bf16*)q; a.k = (const bf16*)k; a.v = (const bf16*)v; a.out = (bf16*)out;
  a.q_ts = st10[0]; a.q_hs = st10[1];
  a.k_bs = st10[2]; a.k_ts = st10[3]; a.k_hs = st10[4];
  a.v_bs = st10[5]; a.v_ts = st10[6]; a.v_hs = st10[7];
  a.o_ts = st10[8]; a.o_hs = st10[9];
  a.B = B; a.H = H; a.Nq = Nq; a.Nk = Nk; a.D = D; a.scale = scale; a.causal = 1; a.kv_start = kv_start;
  a.kv_row = kv_row; a.kv_rows = kv_row ? kv_rows : 0; a.q_off = q_off; a.q_len = q_len; a.q_row0 = q_row0; a.q_rows = rows;
  count_launch();
  return attn_prefill(a, (cudaStream_t)s);
}

extern "C" int emu_op_rmsnorm(const void* x, const void* w, void* y, int rows, int cols, float eps, emu_stream_t s) {
  if (!x || !w || !y) return EMU_ERR_INVALID;
  count_launch();
  return rmsnorm((const bf16*)x, (const bf16*)w, (bf16*)y, rows, cols, eps, 0, (cudaStream_t)s);
}

extern "C" int emu_op_layernorm(const void* x, const void* w, const void* b, const void* residual, void* y, int rows,
                                int cols, float eps, emu_stream_t s) {
  if (!x || !w || !y) return EMU_ERR_INVALID;
  count_launch();
  return layernorm((const bf16*)x, (const bf16*)w, (const bf16*)b, (const bf16*)residual, (bf16*)y, rows, cols, eps,
                   (cudaStream_t)s);
}

// ---- the denoise-step glue of include/emu_b200_gen_slots.h ----
static bool denoise_glue_args_ok(int B, int C, int HW, int ps, int cs, int ub) {
  if (B < 1 || B > kMaxLatentSlots || C < 1 || HW < 1) return false;
  if (ps != 0 && ps != 4) return false;
  return (cs == 1 && ub == B) || (cs == 2 && ub == 1);  // the two row layouts; anything else could alias two slots' rows
}

extern "C" int emu_op_denoise_prepare(const float* latents, void* xin, float* t_rows, int B, int C, int HW, int Cp,
                                      const float* params, int ps, int copies, int cs, int ub, emu_stream_t s) {
  if (!latents || !xin || !t_rows || !params) return EMU_ERR_INVALID;
  if (!denoise_glue_args_ok(B, C, HW, ps, cs, ub) || Cp < C || (copies != 1 && copies != 2)) return EMU_ERR_INVALID;
  if (cs == 2 && copies != 2) return EMU_ERR_INVALID;  // adjacent rows: every slot owns two, the output holds 2B
  count_launch();
  return slot_prepare(latents, (bf16*)xin, t_rows, B, C, HW, Cp, params, ps, copies, cs, ub, (cudaStream_t)s);
}

extern "C" int emu_op_denoise_euler(float* latents, const void* eps, const int32_t* live, int B, int C, int HW, int ld,
                                    const float* params, int ps, int cs, int ub, emu_stream_t s) {
  if (!latents || !eps || !params) return EMU_ERR_INVALID;
  if (!denoise_glue_args_ok(B, C, HW, ps, cs, ub) || ld < C) return EMU_ERR_INVALID;
  count_launch();
  return slot_cfg_euler(latents, (const bf16*)eps, live, B, C, HW, ld, params, ps, cs, ub, (cudaStream_t)s);
}

// ---- the diffusion kernels (include/emu_b200_diffusion_ops.h): the engine's launchers at any shape, arguments checked first ----
// a device workspace owned by one entry point, grown on demand (cudaFree waits for the work that still uses the old one)
static int grow_workspace(void** buf, size_t* cap, size_t need) {
  if (need <= *cap) return EMU_OK;
  if (*buf) cudaFree(*buf);
  *buf = nullptr;
  *cap = 0;
  if (cudaMalloc(buf, need) != cudaSuccess) return EMU_ERR_NOMEM;
  *cap = need;
  return EMU_OK;
}

extern "C" int emu_op_groupnorm(const void* x, const void* w, const void* b, void* y, int NB, int HW, int C, int groups,
                                float eps, int silu, emu_stream_t s) {
  if (!x || !w || !b || !y) return EMU_ERR_INVALID;
  if (NB < 1 || HW < 1 || C < 1 || groups < 1 || C % 8 || C % groups || C > 4096) return EMU_ERR_INVALID;
  static void* scratch = nullptr;
  static size_t cap = 0;
  EMU_TRY(grow_workspace(&scratch, &cap, groupnorm_scratch_bytes(NB, groups)));
  count_launch(2);
  return groupnorm_nhwc((const bf16*)x, (const bf16*)w, (const bf16*)b, (bf16*)y, (float*)scratch, NB, HW, C, groups, eps,
                        silu ? 1 : 0, (cudaStream_t)s);
}

extern "C" int emu_op_timestep_embedding(const float* t, void* out, int rows, int dim, int ld, int col_off, int grp,
                                         emu_stream_t s) {
  if (!t || !out) return EMU_ERR_INVALID;
  if (rows < 1 || dim < 2 || dim % 2 || grp < 1 || col_off < 0 || (long)ld < (long)col_off + (long)grp * dim)
    return EMU_ERR_INVALID;
  count_launch();
  return timestep_embedding(t, (bf16*)out, rows, dim, ld, col_off, grp, (cudaStream_t)s);
}

extern "C" int emu_op_upsample2x(const void* x, void* y, int NB, int H, int W, int C, emu_stream_t s) {
  if (!x || !y || NB < 1 || H < 1 || W < 1 || C < 1 || C % 8) return EMU_ERR_INVALID;
  count_launch();
  return upsample2x_nhwc((const bf16*)x, (bf16*)y, NB, H, W, C, (cudaStream_t)s);
}

extern "C" int emu_op_im2col3x3(const void* x, void* out, int NB, int H, int W, int C, int stride, emu_stream_t s) {
  if (!x || !out || NB < 1 || H < 1 || W < 1 || C < 1 || C % 8) return EMU_ERR_INVALID;
  if (stride != 1 && stride != 2) return EMU_ERR_INVALID;
  count_launch();
  return im2col3x3((const bf16*)x, (bf16*)out, NB, H, W, C, stride, (cudaStream_t)s);
}

extern "C" int emu_op_copy_cols(const void* src, void* dst, int64_t rows, int cols, int lds, int ldd, int col_off,
                                emu_stream_t s) {
  if (!src || !dst || rows < 1 || cols < 1 || col_off < 0 || (cols | lds | ldd | col_off) % 8) return EMU_ERR_INVALID;
  if (lds < cols || (long)ldd < (long)col_off + cols) return EMU_ERR_INVALID;
  count_launch();
  return copy_cols((const bf16*)src, (bf16*)dst, rows, cols, lds, ldd, col_off, (cudaStream_t)s);
}

extern "C" int emu_op_nchw_to_nhwc(const void* x, void* y, int NB, int C, int HW, int Cp, float scale, emu_stream_t s) {
  if (!x || !y || NB < 1 || C < 1 || HW < 1 || Cp < C) return EMU_ERR_INVALID;
  count_launch();
  return nchw_to_nhwc((const bf16*)x, (bf16*)y, NB, C, HW, Cp, scale, (cudaStream_t)s);
}

extern "C" int emu_op_nhwc_to_nchw(const void* x, void* y, int NB, int C, int HW, int ldx, emu_stream_t s) {
  if (!x || !y || NB < 1 || C < 1 || HW < 1 || ldx < C) return EMU_ERR_INVALID;
  count_launch();
  return nhwc_to_nchw((const bf16*)x, (bf16*)y, NB, C, HW, ldx, (cudaStream_t)s);
}

extern "C" int emu_op_mean_tokens(const void* x, void* y, int B, int L, int C, emu_stream_t s) {
  if (!x || !y || B < 1 || L < 1 || C < 1) return EMU_ERR_INVALID;
  count_launch();
  return mean_tokens((const bf16*)x, (bf16*)y, B, L, C, (cudaStream_t)s);
}

extern "C" int emu_op_vae_post(const void* x, float* y, int64_t n_pix, int C, int ldx, emu_stream_t s) {
  if (!x || !y || n_pix < 1 || C < 1 || ldx < C) return EMU_ERR_INVALID;
  count_launch();
  return vae_post((const bf16*)x, y, n_pix, C, ldx, (cudaStream_t)s);
}

extern "C" int emu_op_denoise_multistep(float* lat, const void* eps, float* hist, float* saved, int B, int C, int HW, int ld,
                                        const float* params, int cfg, emu_stream_t s) {
  if (!lat || !eps || !hist || !saved || !params) return EMU_ERR_INVALID;
  if (B < 1 || C < 1 || HW < 1 || ld < C || (cfg != 0 && cfg != 1)) return EMU_ERR_INVALID;
  count_launch();
  return cfg_multistep(lat, (const bf16*)eps, hist, saved, B, C, HW, ld, params, cfg, (cudaStream_t)s);
}

extern "C" int emu_op_vae_attention(const void* q, const void* k, const void* v, void* out, int B, int T, int C,
                                    emu_stream_t s) {
  if (!q || !k || !v || !out || B < 1 || T < 1 || C < 1 || T % 8 || C % 8) return EMU_ERR_INVALID;
  static void* ws = nullptr;
  static size_t cap = 0;
  EMU_TRY(grow_workspace(&ws, &cap, vae_attention_workspace_bytes(T, C)));
  int nl = 0;
  const int rc = vae_attention((const bf16*)q, (const bf16*)k, (const bf16*)v, (bf16*)out, B, T, C, ws, (cudaStream_t)s, &nl);
  count_launch(nl);
  return rc;
}
