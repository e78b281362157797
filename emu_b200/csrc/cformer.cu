// emu_b200 — Emu1 Causal-Former: 32 learned causal query tokens through a T5-base *decoder* stack that
// cross-attends to the EVA-CLIP-g tokens, then a Linear to the LLaMA width.
//
// Reference: Emu1/models/causal_former.py:15-62 (module, forward) over the vendored T5 decoder
// Emu1/models/modeling_t5.py — T5LayerNorm :309-331, T5Attention :407-689 (no 1/sqrt(d) scaling; relative position
// bias computed by block 0 and shared; fp32 softmax :666; cross-attention K/V are Linear(encoder_width -> inner)
// :422-424), T5LayerFF / T5DenseActDense :352-365 (ReLU), T5Block :766-905, T5Stack.forward :1100-1366 (causal mask
// for the decoder self-attention, final_layer_norm).
//
// All contractions are tiny (32 queries): they go through the same wgmma GEMM and flash-attention kernels as the
// rest of the engine (additive bias + causal mask for self-attention, plain cross-attention over the 257 ViT tokens).
#include <math.h>

#include "diffusion_common.h"

namespace emu {

struct CfBlock {
  bf16 *ln0 = nullptr, *ln1 = nullptr, *ln2 = nullptr;
  bf16 *wqkv = nullptr, *wo = nullptr;   // self-attention [3*inner, d], [d, inner]
  bf16 *wq2 = nullptr, *wkv2 = nullptr, *wo2 = nullptr;  // cross [inner, d], [2*inner, enc], [d, inner]
  bf16 *wi = nullptr, *wff = nullptr;    // [ffn, d], [d, ffn]
};
struct CFormerModel {
  SpecMap specs;
  std::vector<CfBlock> blocks;
  bf16 *rel_table = nullptr, *final_ln = nullptr, *tokens = nullptr, *proj_w = nullptr, *proj_b = nullptr;
  float* bias = nullptr;  // [heads, Q, Q] relative position bias, built on first forward
  std::map<std::string, DevBuf> bufs;
  bool grew = false;
};

void cformer_destroy(CFormerModel* m) { delete m; }

static CFormerModel* cf_get(EmuEngine* e) {
  if (e->cformer) return e->cformer;
  const EmuConfig& c = e->cfg;
  if (c.cf_layers < 1) return nullptr;
  CFormerModel* m = new CFormerModel();
  const int d = c.cf_dim, inner = d, enc = c.cf_enc_width, ffn = c.cf_ffn;
  m->blocks.resize(c.cf_layers);
  for (int i = 0; i < c.cf_layers; ++i) {
    CfBlock& b = m->blocks[i];
    const std::string p = "cformer.block." + std::to_string(i) + ".layer.";
    m->specs[p + "0.layer_norm.weight"] = {&b.ln0, LK_COPY, (long)d, 1, d, 0, 0};
    m->specs[p + "0.SelfAttention.q.weight"] = {&b.wqkv, LK_ROWS, (long)3 * inner * d, inner, d, 0, 0};
    m->specs[p + "0.SelfAttention.k.weight"] = {&b.wqkv, LK_ROWS, (long)3 * inner * d, inner, d, inner, 0};
    m->specs[p + "0.SelfAttention.v.weight"] = {&b.wqkv, LK_ROWS, (long)3 * inner * d, inner, d, 2 * inner, 0};
    m->specs[p + "0.SelfAttention.o.weight"] = {&b.wo, LK_COPY, (long)d * inner, d, inner, 0, 0};
    if (i == 0)
      m->specs[p + "0.SelfAttention.relative_attention_bias.weight"] = {&m->rel_table, LK_COPY, (long)c.cf_buckets * c.cf_heads, c.cf_buckets, c.cf_heads, 0, 0};
    m->specs[p + "1.layer_norm.weight"] = {&b.ln1, LK_COPY, (long)d, 1, d, 0, 0};
    m->specs[p + "1.EncDecAttention.q.weight"] = {&b.wq2, LK_COPY, (long)inner * d, inner, d, 0, 0};
    m->specs[p + "1.EncDecAttention.k.weight"] = {&b.wkv2, LK_ROWS, (long)2 * inner * enc, inner, enc, 0, 0};
    m->specs[p + "1.EncDecAttention.v.weight"] = {&b.wkv2, LK_ROWS, (long)2 * inner * enc, inner, enc, inner, 0};
    m->specs[p + "1.EncDecAttention.o.weight"] = {&b.wo2, LK_COPY, (long)d * inner, d, inner, 0, 0};
    m->specs[p + "2.layer_norm.weight"] = {&b.ln2, LK_COPY, (long)d, 1, d, 0, 0};
    m->specs[p + "2.DenseReluDense.wi.weight"] = {&b.wi, LK_COPY, (long)ffn * d, ffn, d, 0, 0};
    m->specs[p + "2.DenseReluDense.wo.weight"] = {&b.wff, LK_COPY, (long)d * ffn, d, ffn, 0, 0};
  }
  m->specs["cformer.final_layer_norm.weight"] = {&m->final_ln, LK_COPY, (long)d, 1, d, 0, 0};
  m->specs["causal_tokens"] = {&m->tokens, LK_COPY, (long)c.cf_queries * d, c.cf_queries, d, 0, 0};
  m->specs["projection.weight"] = {&m->proj_w, LK_COPY, (long)c.cf_out_dim * d, c.cf_out_dim, d, 0, 0};
  m->specs["projection.bias"] = {&m->proj_b, LK_COPY, (long)c.cf_out_dim, 1, c.cf_out_dim, 0, 0};
  e->cformer = m;
  return m;
}

int cformer_load_tensor(EmuEngine* e, const std::string& key, const bf16* src, const int64_t* shape, int ndim,
                        cudaStream_t st) {
  CFormerModel* m = cf_get(e);
  if (!m) return e->fail(EMU_ERR_STATE, "engine was created without a Causal-Former (cf_layers = 0)");
  return load_by_spec(e, m->specs, "cformer", key, src, shape, ndim, st);
}

// T5Attention._relative_position_bucket with bidirectional=False (decoder) — modeling_t5.py:455-508
static int rel_bucket(int relative_position, int num_buckets, int max_distance) {
  int rp = -(relative_position < 0 ? relative_position : 0);  // -min(rp, 0)
  const int max_exact = num_buckets / 2;
  if (rp < max_exact) return rp;
  int large = max_exact + (int)(logf((float)rp / (float)max_exact) / logf((float)max_distance / (float)max_exact) *
                                (float)(num_buckets - max_exact));
  return large < num_buckets - 1 ? large : num_buckets - 1;
}

static int build_bias(EmuEngine* e, CFormerModel* m, cudaStream_t st) {
  const EmuConfig& c = e->cfg;
  const int Q = c.cf_queries, Hh = c.cf_heads, NBk = c.cf_buckets;
  std::vector<uint16_t> tab((size_t)NBk * Hh);
  if (cudaMemcpyAsync(tab.data(), m->rel_table, tab.size() * 2, cudaMemcpyDeviceToHost, st) != cudaSuccess)
    return e->fail(EMU_ERR_CUDA, "rel table copy");
  cudaStreamSynchronize(st);
  std::vector<float> bias((size_t)Hh * Q * Q);
  for (int h = 0; h < Hh; ++h)
    for (int i = 0; i < Q; ++i)
      for (int j = 0; j < Q; ++j) {
        const int bkt = rel_bucket(j - i, NBk, c.cf_max_distance);
        const uint32_t bits = (uint32_t)tab[(size_t)bkt * Hh + h] << 16;
        float f;
        memcpy(&f, &bits, 4);
        bias[((size_t)h * Q + i) * Q + j] = f;
      }
  m->bias = (float*)e->dmalloc(bias.size() * sizeof(float));
  if (!m->bias) return e->fail(EMU_ERR_NOMEM, "bias alloc");
  if (cudaMemcpyAsync(m->bias, bias.data(), bias.size() * sizeof(float), cudaMemcpyHostToDevice, st) != cudaSuccess)
    return e->fail(EMU_ERR_CUDA, "bias copy");
  cudaStreamSynchronize(st);
  return EMU_OK;
}

}  // namespace emu
using namespace emu;

extern "C" int emu_cformer_forward(EmuEngine* e, const void* vit_tokens, int B, int Nv, void* out, emu_stream_t stream) {
  if (!e || !vit_tokens || !out || B < 1 || Nv < 1) return EMU_ERR_INVALID;
  CFormerModel* m = cf_get(e);
  if (!m) return e->fail(EMU_ERR_STATE, "engine was created without a Causal-Former (cf_layers = 0)");
  for (auto& kv : m->specs)
    if (!*kv.second.dst) return e->fail(EMU_ERR_STATE, "Causal-Former weight missing: " + kv.first);
  cudaStream_t st = (cudaStream_t)stream;
  const EmuConfig& cf = e->cfg;
  const int d = cf.cf_dim, Hh = cf.cf_heads, D = d / Hh, Q = cf.cf_queries, enc = cf.cf_enc_width, ffn = cf.cf_ffn;
  if (!m->bias) EMU_TRY(build_bias(e, m, st));
  Ctx c{e, &m->bufs, &m->grew, st, B, 1, 1e-6f};
  const long M = (long)B * Q;
  BUF(h, "cf_h", M * d);
  BUF(n, "cf_n", M * d);
  BUF(qkv, "cf_qkv", M * 3 * d);
  BUF(att, "cf_att", M * d);
  BUF(kv, "cf_kv", (size_t)B * Nv * 2 * d);
  BUF(ff, "cf_ff", M * ffn);
  for (int b = 0; b < B; ++b)  // causal_tokens.expand(B, -1, -1)
    if (cudaMemcpyAsync(h + (size_t)b * Q * d, m->tokens, (size_t)Q * d * 2, cudaMemcpyDeviceToDevice, st) != cudaSuccess)
      return e->fail(EMU_ERR_CUDA, "token copy");
  int nl = 0;
  for (const CfBlock& blk : m->blocks) {
    // layer[0]: self-attention (causal, shared relative position bias, no score scaling)
    EMU_TRY(rmsnorm(h, blk.ln0, n, (int)M, d, 1e-6f, 1, st));
    GemmEpilogue e1;
    e1.C = qkv; e1.ldc = 3 * d;
    EMU_TRY(gemm_bf16(n, d, blk.wqkv, d, (int)M, 3 * d, d, e1, st));
    AttnArgs a;
    a.q = qkv; a.k = qkv + d; a.v = qkv + 2 * d;
    a.q_bs = a.k_bs = a.v_bs = (long)Q * 3 * d; a.q_ts = a.k_ts = a.v_ts = 3 * d; a.q_hs = a.k_hs = a.v_hs = D;
    a.out = att; a.o_bs = (long)Q * d; a.o_ts = d; a.o_hs = D;
    a.B = B; a.H = Hh; a.Nq = Q; a.Nk = Q; a.D = D; a.scale = 1.0f; a.causal = 1; a.bias = m->bias;
    EMU_TRY(attn_prefill(a, st));
    GemmEpilogue e2;
    e2.C = h; e2.ldc = d; e2.residual = h; e2.ldr = d;
    EMU_TRY(gemm_bf16(att, d, blk.wo, d, (int)M, d, d, e2, st));
    // layer[1]: cross-attention over the ViT tokens (K/V projected from encoder_width)
    EMU_TRY(rmsnorm(h, blk.ln1, n, (int)M, d, 1e-6f, 1, st));
    GemmEpilogue e3;
    e3.C = qkv; e3.ldc = d;
    EMU_TRY(gemm_bf16(n, d, blk.wq2, d, (int)M, d, d, e3, st));
    GemmEpilogue e4;
    e4.C = kv; e4.ldc = 2 * d;
    EMU_TRY(gemm_bf16((const bf16*)vit_tokens, enc, blk.wkv2, enc, B * Nv, 2 * d, enc, e4, st));
    AttnArgs x;
    x.q = qkv; x.q_bs = (long)Q * d; x.q_ts = d; x.q_hs = D;
    x.k = kv; x.v = kv + d; x.k_bs = x.v_bs = (long)Nv * 2 * d; x.k_ts = x.v_ts = 2 * d; x.k_hs = x.v_hs = D;
    x.out = att; x.o_bs = (long)Q * d; x.o_ts = d; x.o_hs = D;
    x.B = B; x.H = Hh; x.Nq = Q; x.Nk = Nv; x.D = D; x.scale = 1.0f;
    EMU_TRY(attn_prefill(x, st));
    GemmEpilogue e5;
    e5.C = h; e5.ldc = d; e5.residual = h; e5.ldr = d;
    EMU_TRY(gemm_bf16(att, d, blk.wo2, d, (int)M, d, d, e5, st));
    // layer[2]: ReLU feed-forward
    EMU_TRY(rmsnorm(h, blk.ln2, n, (int)M, d, 1e-6f, 1, st));
    GemmEpilogue e6;
    e6.C = ff; e6.ldc = ffn; e6.mode = EPI_RELU;
    EMU_TRY(gemm_bf16(n, d, blk.wi, d, (int)M, ffn, d, e6, st));
    GemmEpilogue e7;
    e7.C = h; e7.ldc = d; e7.residual = h; e7.ldr = d;
    EMU_TRY(gemm_bf16(ff, ffn, blk.wff, ffn, (int)M, d, ffn, e7, st));
    nl += 12;
  }
  EMU_TRY(rmsnorm(h, m->final_ln, n, (int)M, d, 1e-6f, 1, st));
  GemmEpilogue ep;
  ep.C = out; ep.ldc = cf.cf_out_dim; ep.bias = m->proj_b;
  EMU_TRY(gemm_bf16(n, d, m->proj_w, d, (int)M, cf.cf_out_dim, d, ep, st));
  count_launch(nl + 2);
  return EMU_OK;
}
