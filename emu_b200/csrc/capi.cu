// emu_b200 — C ABI wrappers for the stand-alone operators (include/emu_b200.h, "stand-alone operators").
// These expose exactly the kernels the engine launches, so the parity tests exercise the product path.
#include "common.cuh"
#include "engine.h"

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
