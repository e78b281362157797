// emu_b200 — internal op launchers (C++ side of the C ABI declared in include/emu_b200.h).
// Every launcher enqueues work on the caller's stream, never synchronises, and returns an EMU_* code.
#pragma once
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace emu {

typedef __nv_bfloat16 bf16;

enum EpiMode {
  EPI_NONE = 0,    // C = A W^T (+bias) (+residual)
  EPI_GELU = 1,    // C = gelu_erf(A W^T + bias)
  EPI_SWIGLU = 2,  // W rows interleaved (gate_j, up_j): C[:, j] = silu(g_j) * u_j          (N_out = N/2)
  EPI_GEGLU = 3,   // W rows interleaved (hidden_j, gate_j): C[:, j] = h_j * gelu_erf(g_j)   (N_out = N/2)
  EPI_RELU = 4,    // C = relu(A W^T + bias)   (T5 DenseReluDense)
};

struct GemmEpilogue {
  void* C = nullptr;
  int ldc = 0;
  const bf16* bias = nullptr;
  const bf16* residual = nullptr;
  int ldr = 0;
  const bf16* bias2 = nullptr;  // [M / bias2_rows, N] per-row-group bias (time embedding of a ResnetBlock2D)
  int bias2_rows = 0;
  int mode = EPI_NONE;
  int out_fp32 = 0;
  int force_bn = 0;  // tests only: force the N tile (64/128/256)
  unsigned long long* dbg = nullptr;  // diagnostics: per-CTA phase time stamps (emu_debug_gemm_phases)
};

// ---- gemm_tc.cu : wgmma GEMM / implicit-GEMM conv ----
int gemm_bf16(const bf16* A, int lda, const bf16* W, int ldw, int M, int N, int K, const GemmEpilogue& e,
              cudaStream_t st);
int conv3x3_bf16(const bf16* X_nhwc, int NB, int H, int W, int Cin, const bf16* Wk, int Cout, const GemmEpilogue& e,
                 cudaStream_t st);

// ---- gemm_skinny.cu : wgmma GEMM with the WEIGHTS as the 128-row operand, activations B <= 32 rows (wide decode) ----
// plain / +residual / EPI_SWIGLU epilogues, bf16 or fp32 output; K-split partial sums through `ws` (gemm_skinny_workspace_bytes())
// and `counters` (kSkinnyMaxTiles ints, zeroed once).  EMU_ERR_UNSUPPORTED: shape / epilogue outside this kernel -> gemm_bf16.
constexpr int kSkinnyMaxUnits = 1024;
constexpr int kSkinnyMaxTiles = 4096;
size_t gemm_skinny_workspace_bytes();
int gemm_skinny_init();
int gemm_skinny_bf16(const bf16* X, int ldx, const bf16* W, int ldw, int B, int N, int K, const GemmEpilogue& e, float* ws,
                     int* counters, cudaStream_t st);

// ---- gemv.cu : weight-streaming skinny GEMM for the decode loop (batch <= 8) ----
struct GemvArgs {
  const bf16* W = nullptr;  // [N, K] row-major
  int N = 0, K = 0;
  const bf16* x = nullptr;  // [B, ldx]
  int ldx = 0;
  int B = 0;
  const bf16* norm_w = nullptr;  // fused RMSNorm prologue on x (HF LlamaRMSNorm rounding), or null
  float norm_eps = 1e-6f;
  int mode = EPI_NONE;           // EPI_NONE / EPI_SWIGLU, or GEMV_ROPE_QKV below
  const bf16* bias = nullptr;    // [N] or null
  const bf16* residual = nullptr;  // [B, ldr]
  int ldr = 0;
  void* y = nullptr;  // [B, ldy] bf16 (or fp32 if out_fp32)
  int ldy = 0;
  int out_fp32 = 0;
  // mode == GEMV_ROPE_QKV: rows are [q heads | k heads | v heads], q/k head rows pair-interleaved
  // (row 2j <- orig j, row 2j+1 <- orig j + D/2). Epilogue applies RoPE to q,k, writes q to y and k,v
  // straight into the KV cache at slot pos[b].
  int n_heads = 0, head_dim = 0;
  const bf16* rope_cos = nullptr;  // [max_pos, D/2] bf16
  const bf16* rope_sin = nullptr;
  const int* pos = nullptr;      // [B] cache slot of the new token
  const int* pos_off = nullptr;  // [B] rope position = pos - pos_off
  bf16* k_cache = nullptr;       // [B, n_heads, T_max, D] (this layer)
  bf16* v_cache = nullptr;
  int t_max = 0;
  int pdl = 0;  // launch with programmatic dependent launch
  // Tensor-parallel fused exchange (tp_exchange.cu), mode == EPI_NONE only: instead of writing y, the epilogue stores
  // every fp32 output as an 8-byte {value, flag} word straight into each rank's receive slot over NVLink
  // (flag = *ll_step * 256 + ll_idx + 1, slot = parity ll_idx & 1, source ll_rank); ll_n == 0 disables.
  void* ll_peer[8] = {};
  int ll_n = 0, ll_rank = 0, ll_idx = 0;
  long ll_slot_elems = 0;
  const unsigned* ll_step = nullptr;
  // ... and, when ll_h is set, the first ll_red CTAs of the SAME kernel finish the exchange once their own rows are out:
  // they poll the {value, flag} words of all ranks in this rank's receive buffer (ll_peer[ll_rank]), add the fixed-order sum
  // to the residual stream ll_h [B, ldy] in place (projection rounded to bf16 first, like the unsharded model).  No
  // separate poll + reduce launch, and the successor's CTAs start filling their weight rings on the SMs that are done.
  bf16* ll_h = nullptr;
  int ll_red = 0;
  unsigned long long* dbg = nullptr;  // diagnostics: per-CTA phase time stamps (emu_debug_gemv_phases)
};
constexpr int GEMV_ROPE_QKV = 16;
int gemv_bf16(const GemvArgs& a, cudaStream_t st);
int gemv_init();  // allocate the stream-K workspace (must run once outside stream capture)

// ---- attention.cu ----
// decode: one query token per sequence against the KV cache (slots [start[b], pos[b]] inclusive)
int attn_decode(const bf16* q /*[B, H*D] pair-interleaved like k*/, const bf16* k_cache, const bf16* v_cache,
                int B, int H, int D, int t_max, const int* pos, const int* start, float scale, bf16* out /*[B,H*D]*/,
                float* workspace, int* counters, int max_len_hint, int pdl, cudaStream_t st,
                const int* indir = nullptr /*[rows][t_max] cache row holding token t of sequence b; null = own row*/);
size_t attn_decode_workspace_bytes(int B, int H, int D);
// prefill / encoder attention (flash style, mma.sync): q,k,v given as strided [B, N, H, D] views
struct AttnArgs {
  const bf16* q = nullptr; const bf16* k = nullptr; const bf16* v = nullptr;
  long q_bs = 0, q_ts = 0, q_hs = 0;  // element strides: batch, token, head
  long k_bs = 0, k_ts = 0, k_hs = 0;
  long v_bs = 0, v_ts = 0, v_hs = 0;
  bf16* out = nullptr; long o_bs = 0, o_ts = 0, o_hs = 0;
  int B = 0, H = 0, Nq = 0, Nk = 0, D = 0;
  float scale = 1.f;
  int causal = 0;                 // query i attends keys j <= i + (Nk - Nq)
  const int* kv_start = nullptr;  // [B] first valid key (left padding) or null
  const float* bias = nullptr;    // [H, Nq, Nk] additive (T5 relative position bias) or null
};
int attn_prefill(const AttnArgs& a, cudaStream_t st);
int attn_prefill_tc(const AttnArgs& a, cudaStream_t st);  // attention_tc.cu; EMU_ERR_UNSUPPORTED -> use attn_prefill's own kernel

// ---- programmatic dependent launch for kernel chains (UNet / ViT / prefill) ----
// While a PdlScope is alive on this thread, the PDL-aware launchers (GEMM / conv, wgmma attention, LayerNorm,
// GroupNorm, copy_cols) launch with cudaLaunchAttributeProgrammaticStreamSerialization: the kernel's prologue (CTA launch,
// barrier init, tensor-map prefetch) overlaps the predecessor's tail, and the kernel executes
// griddepcontrol.wait before it touches anything a predecessor wrote.  EMU_NO_PDL=1 disables.
extern thread_local int g_pdl_chain;
struct PdlScope {
  int prev;
  explicit PdlScope(int on);
  ~PdlScope() { g_pdl_chain = prev; }
};
template <typename... KArgs, typename... Args>
inline int launch_kernel(void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, int pdl, Args... args) {
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = pdl ? 1 : 0;
  return cudaLaunchKernelEx(&cfg, kern, static_cast<KArgs>(args)...) == cudaSuccess ? EMU_OK : EMU_ERR_CUDA;
}

// ---- elementwise.cu ----
int rmsnorm(const bf16* x, const bf16* w, bf16* y, int rows, int cols, float eps, int t5_style, cudaStream_t st);
int layernorm(const bf16* x, const bf16* w, const bf16* b, const bf16* residual, bf16* y, int rows, int cols, float eps,
              cudaStream_t st);  // y = residual + LN(x)  (residual may be null)
int rope_kv_write(bf16* qkv /*[B,N,3*H*D] pair-interleaved q,k*/, int B, int N, int H, int D, const bf16* cos,
                  const bf16* sin, const int* pos_off /*[B]*/, int pos0, bf16* k_cache, bf16* v_cache, int t_max,
                  cudaStream_t st, const int* pos_dev = nullptr /*device slot of the new token (N == 1), overrides pos0*/,
                  bf16* q_out = nullptr /*decode: the rotated q goes compact [B*N, H*D] here instead of in place*/);
int embed_gather(const bf16* table, const int* ids, bf16* out, int n, int dim, cudaStream_t st);
int argmax_rows(const float* logits, int rows, int cols, int* out_idx, cudaStream_t st);
int vit_im2col(const bf16* img_nchw, bf16* out, int B, int C, int HW, int P, int Kpad, cudaStream_t st);
int vit_assemble(const bf16* patches, const bf16* cls, const bf16* pos, bf16* x, int B, int Np, int dim,
                 cudaStream_t st);
int vit_pool(const bf16* x /*[B,1+G*G,dim]*/, bf16* out /*[B,n_query,dim]*/, int B, int G, int dim, int stride,
             cudaStream_t st);
int kv_reorder(bf16* cache /*[outer][Bcap][H][t_max][D]*/, int Bcap, const int* src_idx, int B, long outer,
               int n_used_tokens, int H, int D, int t_max, cudaStream_t st);
// beam re-parenting without moving the cache: indir[b][t] <- indir[src[b]][t] for t < n_tok (in place, column-wise)
int kv_indir_update(int* indir /*[rows][t_max]*/, const int* src_idx, int B, int t_max, int n_tok, cudaStream_t st);
int kv_indir_identity(int* indir, int rows, int t_max, cudaStream_t st);
int add_rows(const bf16* a, const bf16* b, bf16* out, long n, cudaStream_t st);

}  // namespace emu
