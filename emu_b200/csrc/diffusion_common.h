// emu_b200 — shared pieces of the diffusion sub-models (UNet in unet.cu, VAE decoder in vae.cu).
#pragma once
#include <map>
#include <string>
#include <vector>

#include "common.cuh"
#include "engine.h"

#ifndef EMU_TRY
#define EMU_TRY(x)                 \
  do {                             \
    int rc_ = (x);                 \
    if (rc_ != EMU_OK) return rc_; \
  } while (0)
#endif

namespace emu {

constexpr int kMaxLatentSlots = 32;  // include/emu_b200_gen_slots.h: B of a latent-slot step

// diffusion_ops.cu
int groupnorm_nhwc(const bf16* x, const bf16* w, const bf16* b, bf16* y, float* scratch, int NB, int HW, int C,
                   int groups, float eps, int do_silu, cudaStream_t st);
size_t groupnorm_scratch_bytes(int NB, int groups);
int timestep_embedding(const float* t, bf16* out, int rows, int dim, int ld, int col_off, int grp, cudaStream_t st);
int silu_rows(const bf16* x, bf16* y, long n, cudaStream_t st);
int copy_cols(const bf16* src, bf16* dst, long rows, int cols, int lds, int ldd, int col_off, cudaStream_t st);
int upsample2x_nhwc(const bf16* x, bf16* y, int NB, int H, int W, int C, cudaStream_t st);
int im2col3x3(const bf16* x, bf16* out, int NB, int H, int W, int C, int stride, cudaStream_t st);
int nchw_to_nhwc(const bf16* x, bf16* y, int NB, int C, int HW, int Cp, float scale, cudaStream_t st);
int nhwc_to_nchw(const bf16* x, bf16* y, int NB, int C, int HW, int ldx, cudaStream_t st);
int slot_prepare(const float* lat, bf16* xin, float* t_rows, int B, int C, int HW, int Cp, const float* params, int ps,
                 int copies, int cs, int ub, cudaStream_t st);
int slot_cfg_euler(float* lat, const bf16* eps_nhwc, const int* live, int B, int C, int HW, int ld, const float* params, int ps,
                   int cs, int ub, cudaStream_t st);
int cfg_multistep(float* lat, const bf16* eps_nhwc, float* hist, float* saved, int B, int C, int HW, int ld,
                  const float* params, int cfg, cudaStream_t st);
int int_to_float(const int* x, float* y, int n, cudaStream_t st);

#define EMU_TRY(x)                 \
  do {                             \
    int rc_ = (x);                 \
    if (rc_ != EMU_OK) return rc_; \
  } while (0)

struct Lin { bf16 *w = nullptr, *b = nullptr; int out = 0, in = 0; };
struct Conv { bf16 *w = nullptr, *b = nullptr; int cout = 0, cin = 0 /*padded to 8*/, k = 3; };
struct Norm { bf16 *w = nullptr, *b = nullptr; int c = 0; };
struct ResnetW { Norm n1, n2; Conv c1, c2, sc; Lin temb; bool has_sc = false; int cin = 0, cout = 0; };
struct TBlockW {
  Norm n1, n2, n3;
  bf16 *wqkv = nullptr, *wq2 = nullptr, *wkv2 = nullptr;
  Lin o1, o2, ff1, ff2;
  long kv_off = -1;  // column offset of this block's [k | v] in the batched cross-attention projection (unet.cu)
};
struct TransW { Norm gn; Lin pin, pout; std::vector<TBlockW> blocks; int c = 0, hd = 64; };

enum LoadKind { LK_COPY = 0, LK_CONV3 = 1, LK_ROWS = 2, LK_GEGLU_W = 3, LK_GEGLU_B = 4 };
struct LoadSpec {
  bf16** dst;
  int kind;
  long alloc_elems;  // elements of the destination buffer
  int rows, cols;    // source matrix view
  int row_off;       // LK_ROWS: destination row offset
  int cin_pad;       // LK_CONV3
};
typedef std::map<std::string, LoadSpec> SpecMap;
void reg_lin(SpecMap& m, const std::string& p, Lin& l, int out, int in, bool bias = true);
void reg_conv(SpecMap& m, const std::string& p, Conv& c, int cout, int cin, int k);
void reg_norm(SpecMap& m, const std::string& p, Norm& n, int c);
int load_by_spec(EmuEngine* e, const SpecMap& specs, const char* what, const std::string& key, const bf16* src,
                 const int64_t* shape, int ndim, cudaStream_t st);

// per-forward context: named, grow-on-demand device workspaces + launch counter
struct Ctx {
  EmuEngine* e;
  std::map<std::string, DevBuf>* bufs;
  bool* grew;
  cudaStream_t st;
  int B2;
  int groups;
  float gn_eps;
  int nl = 0;
  const bf16* kv_all = nullptr;  // [B2*L, kv_ld]: every transformer block's cross-attention K|V, projected in ONE GEMM
  long kv_ld = 0;
  bf16* buf(const char* name, size_t elems);
};
#define BUF(var, name, elems)               \
  bf16* var = c.buf(name, (size_t)(elems)); \
  if (!var) return c.e->fail(EMU_ERR_NOMEM, "diffusion workspace alloc failed")

int lin_rows(Ctx& c, const bf16* x, int M, const Lin& l, bf16* y, const bf16* residual = nullptr, int mode = EPI_NONE);
int conv3(Ctx& c, const bf16* x, int NB, int H, int W, const Conv& cv, int stride, bf16* y, const bf16* bias2,
          const bf16* residual, int ldy = 0);
int gnorm(Ctx& c, const bf16* x, const Norm& n, bf16* y, int NB, int HW, float eps, int do_silu);
int softmax_rows(const float* s, bf16* p, long rows, int cols, float scale, cudaStream_t st);
int transpose_2d(const bf16* x, bf16* y, int rows, int cols, cudaStream_t st);
int vae_post(const bf16* x, float* y, long n_pix, int C, int ldx, cudaStream_t st);
int mean_tokens(const bf16* x, bf16* y, int B, int L, int C, cudaStream_t st);

// vae.cu: the VAE mid-block attention core, o[b] = softmax(q[b] k[b]^T / sqrt(C)) v[b] for q / k / v / o [B, T, C] bf16
// (T % 8 == 0, C % 8 == 0), in query-row chunks of vae_attention_chunk_rows(T) over a workspace of
// vae_attention_workspace_bytes(T, C) (16-byte aligned).  *launches (optional) receives the kernel count.
int vae_attention_chunk_rows(int T);
size_t vae_attention_workspace_bytes(int T, int C);
int vae_attention(const bf16* q, const bf16* k, const bf16* v, bf16* o, int B, int T, int C, void* ws, cudaStream_t st,
                  int* launches = nullptr);

}  // namespace emu
