// emu_b200 — AutoencoderKL decoder (SDXL VAE) for Emu2-Gen: latents -> image.
//
// Reference call site: Emu2/emu/diffusion.py:214-219 (`vae.decode(latents / scaling_factor)`, then
// (x/2 + 0.5).clamp(0,1), NHWC float32), configured by Emu2/emu/conf/diffusion_config/vae/config.json.  The module
// arithmetic is diffusers==0.24.0 (third party, not vendored) restated in oracle/diffusion_oracle.py
// ("parity unpinned").  The pipeline runs the VAE in bf16 (force_upcast is not honoured by the reference pipeline).
//
// Same building blocks as the UNet: NHWC bf16, wgmma implicit-GEMM 3x3 convs, 2-kernel GroupNorm+SiLU.  The
// mid-block attention is single-head with head_dim = 512 (> the flash tile), so it is three GEMMs on wgmma
// (S = Q K^T, O = P V with V transposed once) around a row-softmax kernel; it runs once per image.
#include <math.h>

#include "diffusion_common.h"

namespace emu {

struct VaeResnet { Norm n1, n2; Conv c1, c2, sc; bool has_sc = false; int cin = 0, cout = 0; };
struct VaeModel {
  EmuVAEConfig cfg{};
  SpecMap specs;
  Conv post_quant, conv_in, conv_out;
  VaeResnet mid0, mid1;
  Norm attn_gn;
  Lin aq, ak, av, ao;
  std::vector<std::vector<VaeResnet>> up_res;
  std::vector<Conv> up_samp;
  Norm norm_out;
  std::map<std::string, DevBuf> bufs;
  bool grew = false;
};

static void reg_vres(VaeModel* m, const std::string& p, VaeResnet& r, int cin, int cout) {
  r.cin = cin; r.cout = cout;
  reg_norm(m->specs, p + "norm1", r.n1, cin);
  reg_conv(m->specs, p + "conv1", r.c1, cout, cin, 3);
  reg_norm(m->specs, p + "norm2", r.n2, cout);
  reg_conv(m->specs, p + "conv2", r.c2, cout, cout, 3);
  r.has_sc = cin != cout;
  if (r.has_sc) reg_conv(m->specs, p + "conv_shortcut", r.sc, cout, cin, 1);
}

void vae_destroy(VaeModel* m) { delete m; }

int vae_load_tensor(EmuEngine* e, const std::string& key, const bf16* src, const int64_t* shape, int ndim,
                    cudaStream_t st) {
  if (!e->vae) return e->fail(EMU_ERR_STATE, "emu_vae_configure must be called before loading vae.* tensors");
  return load_by_spec(e, e->vae->specs, "vae", key, src, shape, ndim, st);
}

static int vae_resnet(Ctx& c, const VaeResnet& r, const bf16* x, bf16* y, int NB, int H, int W) {
  const long M = (long)NB * H * W;
  BUF(g, "v_norm", M * (r.cin > r.cout ? r.cin : r.cout));
  BUF(t1, "v_t1", M * r.cout);
  EMU_TRY(gnorm(c, x, r.n1, g, NB, H * W, 1e-6f, 1));
  EMU_TRY(conv3(c, g, NB, H, W, r.c1, 1, t1, nullptr, nullptr));
  EMU_TRY(gnorm(c, t1, r.n2, g, NB, H * W, 1e-6f, 1));
  const bf16* shortcut = x;
  if (r.has_sc) {
    BUF(sc, "v_sc", M * r.cout);
    GemmEpilogue ep;
    ep.C = sc; ep.ldc = r.cout; ep.bias = r.sc.b;
    EMU_TRY(gemm_bf16(x, r.cin, r.sc.w, r.cin, (int)M, r.cout, r.cin, ep, c.st));
    ++c.nl;
    shortcut = sc;
  }
  return conv3(c, g, NB, H, W, r.c2, 1, y, nullptr, shortcut);
}

}  // namespace emu
using namespace emu;

extern "C" int emu_vae_configure(EmuEngine* e, const EmuVAEConfig* cfg) {
  if (!e || !cfg) return EMU_ERR_INVALID;
  if (cfg->n_blocks < 1 || cfg->n_blocks > 4) return e->fail(EMU_ERR_UNSUPPORTED, "vae config");
  if (e->vae) { vae_destroy(e->vae); e->vae = nullptr; }
  VaeModel* m = new VaeModel();
  m->cfg = *cfg;
  const int nb = cfg->n_blocks, lpb = cfg->layers_per_block, lc = cfg->latent_channels;
  const int* boc = cfg->block_out_channels;
  const int top = boc[nb - 1];
  reg_conv(m->specs, "post_quant_conv", m->post_quant, lc, lc, 1);
  reg_conv(m->specs, "decoder.conv_in", m->conv_in, top, lc, 3);
  reg_vres(m, "decoder.mid_block.resnets.0.", m->mid0, top, top);
  reg_norm(m->specs, "decoder.mid_block.attentions.0.group_norm", m->attn_gn, top);
  reg_lin(m->specs, "decoder.mid_block.attentions.0.to_q", m->aq, top, top);
  reg_lin(m->specs, "decoder.mid_block.attentions.0.to_k", m->ak, top, top);
  reg_lin(m->specs, "decoder.mid_block.attentions.0.to_v", m->av, top, top);
  reg_lin(m->specs, "decoder.mid_block.attentions.0.to_out.0", m->ao, top, top);
  reg_vres(m, "decoder.mid_block.resnets.1.", m->mid1, top, top);
  m->up_res.resize(nb);
  m->up_samp.resize(nb);
  int cin = top;
  for (int i = 0; i < nb; ++i) {
    const int cout = boc[nb - 1 - i];
    m->up_res[i].resize(lpb + 1);
    for (int j = 0; j < lpb + 1; ++j) {
      reg_vres(m, "decoder.up_blocks." + std::to_string(i) + ".resnets." + std::to_string(j) + ".", m->up_res[i][j], cin, cout);
      cin = cout;
    }
    if (i < nb - 1) reg_conv(m->specs, "decoder.up_blocks." + std::to_string(i) + ".upsamplers.0.conv", m->up_samp[i], cout, cout, 3);
  }
  reg_norm(m->specs, "decoder.conv_norm_out", m->norm_out, boc[0]);
  reg_conv(m->specs, "decoder.conv_out", m->conv_out, cfg->out_channels, boc[0], 3);
  e->vae = m;
  return EMU_OK;
}

extern "C" int emu_vae_decode(EmuEngine* e, const void* latents_nchw, int B, int h, int w, float* image_nhwc,
                              emu_stream_t stream) {
  if (!e || !latents_nchw || !image_nhwc || B < 1) return EMU_ERR_INVALID;
  VaeModel* m = e->vae;
  if (!m) return e->fail(EMU_ERR_STATE, "VAE not configured");
  for (auto& kv : m->specs)
    if (!*kv.second.dst) return e->fail(EMU_ERR_STATE, "VAE weight missing: " + kv.first);
  cudaStream_t st = (cudaStream_t)stream;
  const EmuVAEConfig& cf = m->cfg;
  Ctx c{e, &m->bufs, &m->grew, st, B, cf.norm_groups, 1e-6f};
  const int lc = cf.latent_channels, nb = cf.n_blocks, top = cf.block_out_channels[nb - 1];
  const int lcp = (lc + 7) / 8 * 8;
  int H = h, W = w;
  const long M0 = (long)B * H * W;
  BUF(z0, "v_z0", M0 * lcp);
  BUF(z1, "v_z1", M0 * lcp);
  EMU_TRY(nchw_to_nhwc((const bf16*)latents_nchw, z0, B, lc, H * W, lcp, 1.0f, st));
  {  // post_quant_conv (1x1): weight [lc, lc] against the zero-padded NHWC latents -> K = lcp with padded weight
    BUF(wq, "v_pq_w", (size_t)lcp * lcp);
    cudaMemsetAsync(wq, 0, (size_t)lcp * lcp * 2, st);
    cudaMemcpy2DAsync(wq, (size_t)lcp * 2, m->post_quant.w, (size_t)lc * 2, (size_t)lc * 2, lc, cudaMemcpyDeviceToDevice, st);
    cudaMemsetAsync(z1, 0, (size_t)M0 * lcp * 2, st);
    GemmEpilogue ep;
    ep.C = z1; ep.ldc = lcp; ep.bias = m->post_quant.b;
    EMU_TRY(gemm_bf16(z0, lcp, wq, lcp, (int)M0, lc, lcp, ep, st));
  }
  BUF(a, "v_a", M0 * top);
  BUF(b, "v_b", M0 * top);
  EMU_TRY(conv3(c, z1, B, H, W, m->conv_in, 1, a, nullptr, nullptr));
  EMU_TRY(vae_resnet(c, m->mid0, a, b, B, H, W));
  {  // single-head attention over H*W tokens, dim = top
    const int T = H * W, C = top;
    BUF(n, "v_an", M0 * C);
    BUF(q, "v_q", M0 * C);
    BUF(k, "v_k", M0 * C);
    BUF(v, "v_v", M0 * C);
    BUF(vt, "v_vt", (size_t)C * T);
    BUF(s, "v_s", (size_t)T * T);
    BUF(o, "v_o", (size_t)T * C);
    EMU_TRY(gnorm(c, b, m->attn_gn, n, B, T, 1e-6f, 0));
    EMU_TRY(lin_rows(c, n, (int)M0, m->aq, q));
    EMU_TRY(lin_rows(c, n, (int)M0, m->ak, k));
    EMU_TRY(lin_rows(c, n, (int)M0, m->av, v));
    for (int bi = 0; bi < B; ++bi) {
      const bf16* qb = q + (size_t)bi * T * C;
      const bf16* kb = k + (size_t)bi * T * C;
      const bf16* vb = v + (size_t)bi * T * C;
      GemmEpilogue es;
      es.C = s; es.ldc = T;
      EMU_TRY(gemm_bf16(qb, C, kb, C, T, T, C, es, st));          // S = Q K^T
      EMU_TRY(softmax_rows(s, T, T, 1.0f / sqrtf((float)C), st));  // P = softmax(S / sqrt(C))
      EMU_TRY(transpose_2d(vb, vt, T, C, st));                     // V^T [C, T] (K-major for the second GEMM)
      GemmEpilogue eo;
      eo.C = o; eo.ldc = C;
      EMU_TRY(gemm_bf16(s, T, vt, T, T, C, T, eo, st));            // O = P V
      // to_out + residual (b) -> a
      GemmEpilogue ef;
      ef.C = a + (size_t)bi * T * C; ef.ldc = C; ef.bias = m->ao.b; ef.residual = b + (size_t)bi * T * C; ef.ldr = C;
      EMU_TRY(gemm_bf16(o, C, m->ao.w, C, T, C, C, ef, st));
      c.nl += 5;
    }
  }
  EMU_TRY(vae_resnet(c, m->mid1, a, b, B, H, W));
  bf16* cur = b;
  int C = top;
  int pp = 0;
  for (int i = 0; i < nb; ++i) {
    for (int j = 0; j < cf.layers_per_block + 1; ++j) {
      const VaeResnet& r = m->up_res[i][j];
      char nm[16];
      snprintf(nm, sizeof(nm), "v_u%d", pp ^= 1);
      BUF(out, nm, (size_t)B * H * W * r.cout);
      EMU_TRY(vae_resnet(c, r, cur, out, B, H, W));
      cur = out; C = r.cout;
    }
    if (i < nb - 1) {
      BUF(up, "v_up", (size_t)B * 4 * H * W * C);
      EMU_TRY(upsample2x_nhwc(cur, up, B, H, W, C, st));
      H *= 2; W *= 2;
      char nm[16];
      snprintf(nm, sizeof(nm), "v_u%d", pp ^= 1);
      BUF(out, nm, (size_t)B * H * W * C);
      EMU_TRY(conv3(c, up, B, H, W, m->up_samp[i], 1, out, nullptr, nullptr));
      cur = out;
      ++c.nl;
    }
  }
  BUF(g, "v_norm", (size_t)B * H * W * C);
  EMU_TRY(gnorm(c, cur, m->norm_out, g, B, H * W, 1e-6f, 1));
  BUF(rgb, "v_rgb", (size_t)B * H * W * 8);
  EMU_TRY(conv3(c, g, B, H, W, m->conv_out, 1, rgb, nullptr, nullptr, 8));
  EMU_TRY(vae_post(rgb, image_nhwc, (long)B * H * W, cf.out_channels, 8, st));
  count_launch(c.nl + 6);
  return EMU_OK;
}
