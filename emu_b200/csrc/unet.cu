// emu_b200 — SDXL-topology UNet (diffusers UNet2DConditionModel) and the fused denoise step of Emu2-Gen.
//
// Reference call sites: Emu2/emu/diffusion.py:136-141 (unet forward), :131-149 (denoise loop body: cat for CFG,
// scale_model_input, UNet, CFG combine, Euler step), configured by Emu2/emu/conf/diffusion_config/unet/config.json.
// The module arithmetic itself is diffusers==0.24.0 (third party, not vendored): restated from the published
// algorithm, see oracle/diffusion_oracle.py ("parity unpinned").
//
// H100 mapping: activations live in HBM as NHWC bf16, so every 3x3 convolution is an implicit GEMM on wgmma
// (4-D TMA tile loads, halo = TMA out-of-bounds zero fill — csrc/gemm_tc.cu) and every Linear is the same kernel
// with a 2-D A tile; GroupNorm+SiLU is a 2-kernel bandwidth pass; time-embedding add, bias, residual and GEGLU are
// GEMM epilogues; attention is the flash kernel (head_dim 64).  The whole denoise step (≈1.5 k launches) is
// captured once into a CUDA graph; per-step scalars (sigma, timestep, guidance) are read from device memory.
#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include "diffusion_common.h"

namespace emu {


struct UNetModel {
  EmuUNetConfig cfg{};
  SpecMap specs;
  Conv conv_in, conv_out;
  Lin te1, te2, ae1, ae2;
  Norm norm_out;
  std::vector<std::vector<ResnetW>> down_res, up_res;
  std::vector<std::vector<TransW>> down_att, up_att;
  std::vector<Conv> down_samp, up_samp;
  ResnetW mid_r0, mid_r1;
  TransW mid_att;
  std::map<std::string, DevBuf> bufs;
  bool grew = false;
  // denoise-step graph
  typedef std::tuple<const void*, const void*, const void*, const void*, int, int, int, int> StepKey;
  std::map<StepKey, cudaGraphExec_t> graphs;
  std::map<StepKey, int> warmed;
  float* step_params = nullptr;  // device [4]: sigma, sigma_next, guidance, timestep
  int n_launch = 0;
  // all cross-attention to_k / to_v weights stacked row-wise: the context is the same for every block, so ONE
  // [B2*L, sum 2C] GEMM at the top of the forward replaces 70 tiny per-block launches (same arithmetic per element)
  bf16* kv_all_w = nullptr;
  long kv_all_n = 0;
  bool kv_all_ready = false;
  // CFG-parallel denoising on a pair of GPUs (engine created with tp_size == 2): rank 0 runs the conditional half of the
  // UNet batch, rank 1 the unconditional half, and the two noise predictions are swapped through NVLink peer memory
  // inside the CFG + Euler kernel (cfg_exchange_euler_kernel below)
  unsigned char* xch = nullptr;       // this rank's exchange buffer (cudaMalloc: IPC-exportable)
  unsigned char* xch_peer = nullptr;  // the other rank's, mapped through CUDA IPC
};

// exchange buffer layout (bytes): [2 parities][kXchSlot] noise predictions | [kXchCtas] flags | [kXchCtas] sequence counters
constexpr size_t kXchSlot = (size_t)4 << 20;  // 4 MiB per slot: batch * h * w <= 262144 latent pixels (16 samples of 128x128)
constexpr int kXchCtas = 64;
constexpr size_t kXchBytes = 2 * kXchSlot + 2 * kXchCtas * sizeof(unsigned);

// ----------------------------------------------------------------------------------------------
// configuration: builds the module tree and the key -> destination table
// ----------------------------------------------------------------------------------------------
static int unet_exchange_setup(EmuEngine* e, UNetModel* m);

void reg_lin(SpecMap& specs, const std::string& p, Lin& l, int out, int in, bool bias) {
  l.out = out; l.in = in;
  specs[p + ".weight"] = {&l.w, LK_COPY, (long)out * in, out, in, 0, 0};
  if (bias) specs[p + ".bias"] = {&l.b, LK_COPY, (long)out, 1, out, 0, 0};
}
void reg_conv(SpecMap& specs, const std::string& p, Conv& c, int cout, int cin, int k) {
  c.cout = cout; c.k = k;
  c.cin = (cin + 7) / 8 * 8;
  if (k == 3) specs[p + ".weight"] = {&c.w, LK_CONV3, (long)cout * 9 * c.cin, cout, cin, 0, c.cin};
  else specs[p + ".weight"] = {&c.w, LK_COPY, (long)cout * cin, cout, cin, 0, 0};
  specs[p + ".bias"] = {&c.b, LK_COPY, (long)cout, 1, cout, 0, 0};
}
void reg_norm(SpecMap& specs, const std::string& p, Norm& n, int c) {
  n.c = c;
  specs[p + ".weight"] = {&n.w, LK_COPY, (long)c, 1, c, 0, 0};
  specs[p + ".bias"] = {&n.b, LK_COPY, (long)c, 1, c, 0, 0};
}
static void reg_resnet(UNetModel* m, const std::string& p, ResnetW& r, int cin, int cout, int temb) {
  r.cin = cin; r.cout = cout;
  reg_norm(m->specs, p + "norm1", r.n1, cin);
  reg_conv(m->specs, p + "conv1", r.c1, cout, cin, 3);
  reg_lin(m->specs, p + "time_emb_proj", r.temb, cout, temb);
  reg_norm(m->specs, p + "norm2", r.n2, cout);
  reg_conv(m->specs, p + "conv2", r.c2, cout, cout, 3);
  r.has_sc = cin != cout;
  if (r.has_sc) reg_conv(m->specs, p + "conv_shortcut", r.sc, cout, cin, 1);
}
static void reg_trans(UNetModel* m, const std::string& p, TransW& t, int c, int layers, int cd) {
  t.c = c;
  t.hd = m->cfg.head_dim > 0 ? m->cfg.head_dim : c / m->cfg.num_heads;
  reg_norm(m->specs, p + "norm", t.gn, c);
  reg_lin(m->specs, p + "proj_in", t.pin, c, c);
  reg_lin(m->specs, p + "proj_out", t.pout, c, c);
  t.blocks.resize(layers);
  for (int k = 0; k < layers; ++k) {
    TBlockW& b = t.blocks[k];
    const std::string q = p + "transformer_blocks." + std::to_string(k) + ".";
    reg_norm(m->specs, q + "norm1", b.n1, c);
    reg_norm(m->specs, q + "norm2", b.n2, c);
    reg_norm(m->specs, q + "norm3", b.n3, c);
    // self-attention q|k|v fused into one [3C, C] matrix
    m->specs[q + "attn1.to_q.weight"] = {&b.wqkv, LK_ROWS, (long)3 * c * c, c, c, 0, 0};
    m->specs[q + "attn1.to_k.weight"] = {&b.wqkv, LK_ROWS, (long)3 * c * c, c, c, c, 0};
    m->specs[q + "attn1.to_v.weight"] = {&b.wqkv, LK_ROWS, (long)3 * c * c, c, c, 2 * c, 0};
    reg_lin(m->specs, q + "attn1.to_out.0", b.o1, c, c);
    m->specs[q + "attn2.to_q.weight"] = {&b.wq2, LK_COPY, (long)c * c, c, c, 0, 0};
    m->specs[q + "attn2.to_k.weight"] = {&b.wkv2, LK_ROWS, (long)2 * c * cd, c, cd, 0, 0};
    m->specs[q + "attn2.to_v.weight"] = {&b.wkv2, LK_ROWS, (long)2 * c * cd, c, cd, c, 0};
    reg_lin(m->specs, q + "attn2.to_out.0", b.o2, c, c);
    // GEGLU: rows (hidden_j, gate_j) interleaved so the activation is a pairwise GEMM epilogue
    b.ff1.out = 8 * c; b.ff1.in = c;
    m->specs[q + "ff.net.0.proj.weight"] = {&b.ff1.w, LK_GEGLU_W, (long)8 * c * c, 8 * c, c, 0, 0};
    m->specs[q + "ff.net.0.proj.bias"] = {&b.ff1.b, LK_GEGLU_B, (long)8 * c, 1, 8 * c, 0, 0};
    reg_lin(m->specs, q + "ff.net.2", b.ff2, c, 4 * c);
  }
}

}  // namespace emu
using namespace emu;

extern "C" int emu_unet_configure(EmuEngine* e, const EmuUNetConfig* cfg) {
  if (!e || !cfg) return EMU_ERR_INVALID;
  if (cfg->n_blocks < 2 || cfg->n_blocks > 4) return e->fail(EMU_ERR_UNSUPPORTED, "unet config: 2..4 blocks");
  for (int i = 0; i < cfg->n_blocks; ++i) {  // head width per level: fixed (SDXL) or C / num_heads (SD-1.5)
    if (cfg->transformer_layers[i] <= 0 && !(i == cfg->n_blocks - 1 && cfg->mid_transformer_layers > 0)) continue;
    const int C = cfg->block_out_channels[i];
    const int hd = cfg->head_dim > 0 ? cfg->head_dim : (cfg->num_heads > 0 ? C / cfg->num_heads : 0);
    if (hd < 8 || hd > 160 || hd % 8 || C % hd) return e->fail(EMU_ERR_UNSUPPORTED, "unet config: head width");
  }
  if (e->unet) { unet_destroy(e->unet); e->unet = nullptr; }
  UNetModel* m = new UNetModel();
  m->cfg = *cfg;
  const int nb = cfg->n_blocks, lpb = cfg->layers_per_block, cd = cfg->cross_attention_dim;
  const int* boc = cfg->block_out_channels;
  const int* tl = cfg->transformer_layers;
  const int temb = boc[0] * 4;
  reg_conv(m->specs, "conv_in", m->conv_in, boc[0], cfg->in_channels, 3);
  reg_lin(m->specs, "time_embedding.linear_1", m->te1, temb, boc[0]);
  reg_lin(m->specs, "time_embedding.linear_2", m->te2, temb, temb);
  if (cfg->addition_time_embed_dim > 0) {
    reg_lin(m->specs, "add_embedding.linear_1", m->ae1, temb, cfg->projection_class_embeddings_input_dim);
    reg_lin(m->specs, "add_embedding.linear_2", m->ae2, temb, temb);
  }
  m->down_res.resize(nb); m->down_att.resize(nb); m->down_samp.resize(nb);
  m->up_res.resize(nb); m->up_att.resize(nb); m->up_samp.resize(nb);
  std::vector<int> skip = {boc[0]};
  int cin = boc[0];
  for (int i = 0; i < nb; ++i) {
    m->down_res[i].resize(lpb);
    m->down_att[i].resize(tl[i] > 0 ? lpb : 0);
    for (int j = 0; j < lpb; ++j) {
      const std::string p = "down_blocks." + std::to_string(i);
      reg_resnet(m, p + ".resnets." + std::to_string(j) + ".", m->down_res[i][j], cin, boc[i], temb);
      cin = boc[i];
      if (tl[i] > 0) reg_trans(m, p + ".attentions." + std::to_string(j) + ".", m->down_att[i][j], cin, tl[i], cd);
      skip.push_back(cin);
    }
    if (i < nb - 1) {
      reg_conv(m->specs, "down_blocks." + std::to_string(i) + ".downsamplers.0.conv", m->down_samp[i], cin, cin, 3);
      skip.push_back(cin);
    }
  }
  reg_resnet(m, "mid_block.resnets.0.", m->mid_r0, cin, cin, temb);
  const int mid_layers = cfg->mid_transformer_layers > 0 ? cfg->mid_transformer_layers : tl[nb - 1];
  if (mid_layers > 0) reg_trans(m, "mid_block.attentions.0.", m->mid_att, cin, mid_layers, cd);
  reg_resnet(m, "mid_block.resnets.1.", m->mid_r1, cin, cin, temb);
  for (int i = 0; i < nb; ++i) {
    const int ri = nb - 1 - i;
    m->up_res[i].resize(lpb + 1);
    m->up_att[i].resize(tl[ri] > 0 ? lpb + 1 : 0);
    for (int j = 0; j < lpb + 1; ++j) {
      const std::string p = "up_blocks." + std::to_string(i);
      const int sc = skip.back();
      skip.pop_back();
      reg_resnet(m, p + ".resnets." + std::to_string(j) + ".", m->up_res[i][j], cin + sc, boc[ri], temb);
      cin = boc[ri];
      if (tl[ri] > 0) reg_trans(m, p + ".attentions." + std::to_string(j) + ".", m->up_att[i][j], cin, tl[ri], cd);
    }
    if (i < nb - 1) reg_conv(m->specs, "up_blocks." + std::to_string(i) + ".upsamplers.0.conv", m->up_samp[i], cin, cin, 3);
  }
  reg_norm(m->specs, "conv_norm_out", m->norm_out, boc[0]);
  reg_conv(m->specs, "conv_out", m->conv_out, cfg->out_channels, boc[0], 3);
  m->step_params = (float*)e->dmalloc(16 * sizeof(float));
  if (!m->step_params) { delete m; return e->fail(EMU_ERR_NOMEM, "unet params alloc"); }
  // engines created as a pair (tp_size == 2) set up the CFG-parallel exchange here: COLLECTIVE over both ranks
  const int xrc = unet_exchange_setup(e, m);
  if (xrc != EMU_OK) { unet_destroy(m); return xrc; }
  e->unet = m;
  return EMU_OK;
}

namespace emu {

__global__ void conv3_repack_kernel(const bf16* __restrict__ src, bf16* dst, int O, int I, int Ip) {
  // src [O, I, 3, 3] -> dst [O, 9*Ip], k = (r*3+s)*Ip + c, zero for c >= I
  const long total = (long)O * 9 * Ip;
  for (long idx = blockIdx.x * (long)blockDim.x + threadIdx.x; idx < total; idx += (long)gridDim.x * blockDim.x) {
    const int c = idx % Ip;
    const int tap = (idx / Ip) % 9;
    const long o = idx / ((long)Ip * 9);
    dst[idx] = c < I ? src[(o * I + c) * 9 + tap] : __float2bfloat16(0.f);
  }
}
__global__ void geglu_interleave_kernel(const bf16* __restrict__ src, bf16* dst, long half_rows, int cols) {
  // src rows [0,half) = hidden, [half, 2*half) = gate  ->  dst row 2j = hidden_j, 2j+1 = gate_j
  const long total = 2 * half_rows * cols;
  for (long idx = blockIdx.x * (long)blockDim.x + threadIdx.x; idx < total; idx += (long)gridDim.x * blockDim.x) {
    const int c = idx % cols;
    const long r = idx / cols;
    const long sr = (r & 1) ? half_rows + (r >> 1) : (r >> 1);
    dst[idx] = src[sr * cols + c];
  }
}

void unet_destroy(UNetModel* m) {
  if (!m) return;
  for (auto& g : m->graphs) cudaGraphExecDestroy(g.second);
  if (m->xch_peer) cudaIpcCloseMemHandle(m->xch_peer);
  if (m->xch) cudaFree(m->xch);
  cudaGetLastError();
  delete m;
}

int load_by_spec(EmuEngine* e, const SpecMap& specs, const char* what, const std::string& key, const bf16* src,
                 const int64_t* shape, int ndim, cudaStream_t st) {
  auto it = specs.find(key);
  if (it == specs.end()) return e->fail(EMU_ERR_INVALID, std::string("unknown ") + what + " key " + key);
  const LoadSpec& s = it->second;
  long n = 1;
  for (int i = 0; i < ndim; ++i) n *= shape[i];
  if (n != (long)s.rows * s.cols * (s.kind == LK_CONV3 ? 9 : 1))
    return e->fail(EMU_ERR_INVALID, std::string("shape mismatch for ") + what + "." + key);
  if (!*s.dst) {
    *s.dst = (bf16*)e->dmalloc((size_t)s.alloc_elems * 2);
    if (!*s.dst) return e->fail(EMU_ERR_NOMEM, "weight alloc");
  }
  switch (s.kind) {
    case LK_COPY:
      if (cudaMemcpyAsync(*s.dst, src, (size_t)n * 2, cudaMemcpyDeviceToDevice, st) != cudaSuccess) return e->fail(EMU_ERR_CUDA, "copy");
      break;
    case LK_ROWS:
      if (cudaMemcpyAsync(*s.dst + (size_t)s.row_off * s.cols, src, (size_t)n * 2, cudaMemcpyDeviceToDevice, st) != cudaSuccess)
        return e->fail(EMU_ERR_CUDA, "copy");
      break;
    case LK_CONV3:
      conv3_repack_kernel<<<4 * kNumSMs, 256, 0, st>>>(src, *s.dst, s.rows, s.cols, s.cin_pad);
      break;
    case LK_GEGLU_W:
      geglu_interleave_kernel<<<4 * kNumSMs, 256, 0, st>>>(src, *s.dst, s.rows / 2, s.cols);
      break;
    case LK_GEGLU_B:
      geglu_interleave_kernel<<<4, 256, 0, st>>>(src, *s.dst, s.cols / 2, 1);
      break;
  }
  return cudaGetLastError() == cudaSuccess ? EMU_OK : e->fail(EMU_ERR_CUDA, "weight repack kernel");
}

int unet_load_tensor(EmuEngine* e, const std::string& key, const bf16* src, const int64_t* shape, int ndim,
                     cudaStream_t st) {
  if (!e->unet) return e->fail(EMU_ERR_STATE, "emu_unet_configure must be called before loading unet.* tensors");
  UNetModel* m = e->unet;
  m->kv_all_ready = false;  // re-stack the cross-attention weights on the next forward ...
  if (!m->graphs.empty()) {  // ... which must run eagerly: captured steps read the (now stale) stacked copy
    cudaDeviceSynchronize();
    for (auto& g : m->graphs) cudaGraphExecDestroy(g.second);
    m->graphs.clear();
    m->warmed.clear();
  }
  return load_by_spec(e, e->unet->specs, "unet", key, src, shape, ndim, st);
}

// ----------------------------------------------------------------------------------------------
// CFG-parallel: exchange of the noise prediction + CFG combine + Euler step in one kernel
// ----------------------------------------------------------------------------------------------
// Each CTA owns a contiguous slice of the NHWC noise prediction (ld = 8 channels -> one 16-byte word per latent pixel):
//   1. pushes its slice of THIS rank's prediction into the peer's receive slot (16-byte NVLink stores),
//   2. publishes a sequence flag with a system-scope release and spins (acquire) on the flag the peer wrote into OUR memory,
//   3. combines cond (rank 0's prediction) and uncond (rank 1's) exactly like cfg_euler_kernel and applies the Euler step.
// Both ranks hold the same fp32 latents and perform the same arithmetic in the same order, so their latents stay bitwise
// identical — and identical to the single-GPU path.  Two receive slots (sequence parity): a rank can run at most one
// exchange ahead of its peer.  All state is on the device, so the kernel is captured in the denoise CUDA graph.
__global__ void __launch_bounds__(256) cfg_exchange_euler_kernel(float* lat, const bf16* __restrict__ eps_mine,
                                                                 unsigned char* xch_local, unsigned char* xch_peer, int rank,
                                                                 int B, int C, int HW, const float* __restrict__ params) {
  __shared__ unsigned s_seq;
  unsigned* flags_local = reinterpret_cast<unsigned*>(xch_local + 2 * kXchSlot);
  unsigned* flags_peer = reinterpret_cast<unsigned*>(xch_peer + 2 * kXchSlot);
  unsigned* seq_ptr = flags_local + kXchCtas + blockIdx.x;
  if (threadIdx.x == 0) s_seq = *seq_ptr;
  __syncthreads();
  const unsigned seq = s_seq, parity = seq & 1u;
  const long n_pix = (long)B * HW;
  const long per = (n_pix + gridDim.x - 1) / gridDim.x;
  const long p0 = (long)blockIdx.x * per, p1 = min(n_pix, p0 + per);
  const uint4* mine = reinterpret_cast<const uint4*>(eps_mine);
  uint4* out = reinterpret_cast<uint4*>(xch_peer + parity * kXchSlot);
  for (long i = p0 + threadIdx.x; i < p1; i += blockDim.x) out[i] = mine[i];  // NVLink peer store
  __threadfence_system();
  __syncthreads();
  if (threadIdx.x == 0) {
    asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(flags_peer + blockIdx.x), "r"(seq + 1) : "memory");
    unsigned long long t0 = 0, now;
    for (;;) {
      unsigned v;
      asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(flags_local + blockIdx.x) : "memory");
      if ((int)(v - (seq + 1)) >= 0) break;
      asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(now));
      if (t0 == 0) t0 = now;
      else if (now - t0 > 20000000000ull) {  // 20 s: the peer died — fail loudly instead of hanging the GPU
        printf("emu_b200: CFG-parallel exchange timed out (rank %d)\n", rank);
        __trap();
      }
    }
  }
  __syncthreads();
  const uint4* theirs = reinterpret_cast<const uint4*>(xch_local + parity * kXchSlot);
  const float dt = params[1] - params[0], g = params[2];
  for (long i = p0 + threadIdx.x; i < p1; i += blockDim.x) {
    const uint4 a = mine[i];
    uint4 o;
    asm volatile("ld.volatile.global.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(o.x), "=r"(o.y), "=r"(o.z), "=r"(o.w) : "l"(theirs + i));
    const uint4 cond = rank == 0 ? a : o, unc = rank == 0 ? o : a;
    const uint32_t cw[4] = {cond.x, cond.y, cond.z, cond.w}, uw[4] = {unc.x, unc.y, unc.z, unc.w};
    const long b = i / HW, p = i - b * HW;
    for (int c = 0; c < C && c < 8; ++c) {
      const float ec = (c & 1) ? bf16_hi(cw[c >> 1]) : bf16_lo(cw[c >> 1]);
      const float eu = (c & 1) ? bf16_hi(uw[c >> 1]) : bf16_lo(uw[c >> 1]);
      const float e = round_bf16(eu + round_bf16(g * round_bf16(ec - eu)));  // same rounding points as cfg_euler_kernel
      lat[((long)b * C + c) * HW + p] += e * dt;
    }
  }
  if (threadIdx.x == 0) *seq_ptr = seq + 1;
}

int engine_allgather_bytes(EmuEngine* e, const void* src, void* dst, size_t bytes);  // engine.cu (NCCL, host buffers)
int engine_allreduce_min_int(EmuEngine* e, int* v);

// collective over the pair: allocate, swap IPC handles, map the peer's buffer; leaves m->xch null when unavailable
static int unet_exchange_setup(EmuEngine* e, UNetModel* m) {
  if (e->tp_size != 2 || !e->nccl_comm) return EMU_OK;
  const char* env = getenv("EMU_CFG_PARALLEL");
  int ok = !(env && atoi(env) == 0);
  unsigned char* buf = nullptr;
  cudaIpcMemHandle_t mine;
  memset(&mine, 0, sizeof(mine));
  if (ok) {
    if (cudaMalloc((void**)&buf, kXchBytes) != cudaSuccess) ok = 0;
    if (ok && cudaMemset(buf, 0, kXchBytes) != cudaSuccess) ok = 0;
    if (ok && cudaIpcGetMemHandle(&mine, buf) != cudaSuccess) ok = 0;
    cudaGetLastError();
  }
  char all[2 * sizeof(cudaIpcMemHandle_t)];
  if (engine_allgather_bytes(e, &mine, all, sizeof(mine)) != EMU_OK) return e->fail(EMU_ERR_NCCL, "CFG-parallel handle exchange failed");
  void* peer = nullptr;
  if (ok) {
    cudaIpcMemHandle_t h;
    memcpy(&h, all + (size_t)(1 - e->tp_rank) * sizeof(h), sizeof(h));
    if (cudaIpcOpenMemHandle(&peer, h, cudaIpcMemLazyEnablePeerAccess) != cudaSuccess) {
      cudaGetLastError();
      ok = 0;
    }
  }
  int all_ok = ok;
  if (engine_allreduce_min_int(e, &all_ok) != EMU_OK) return e->fail(EMU_ERR_NCCL, "CFG-parallel setup reduce failed");
  if (!all_ok) {
    if (peer) cudaIpcCloseMemHandle(peer);
    if (buf) cudaFree(buf);
    return EMU_OK;  // both ranks fall back to running the whole CFG batch locally
  }
  m->xch = buf;
  m->xch_peer = (unsigned char*)peer;
  return EMU_OK;
}

// ----------------------------------------------------------------------------------------------
// forward helpers
// ----------------------------------------------------------------------------------------------
bf16* Ctx::buf(const char* name, size_t elems) {
  DevBuf& b = (*bufs)[name];
  if (b.bytes < elems * 2) {
    void* p = e->dmalloc(elems * 2);
    if (!p) return nullptr;
    b.p = p;
    b.bytes = elems * 2;
    *grew = true;
  }
  return (bf16*)b.p;
}

int lin_rows(Ctx& c, const bf16* x, int M, const Lin& l, bf16* y, const bf16* residual, int mode) {
  ++c.nl;
  if (M <= 8 && l.in % 32 == 0 && mode == EPI_NONE) {
    GemvArgs a;
    a.W = l.w; a.N = l.out; a.K = l.in; a.x = x; a.ldx = l.in; a.B = M; a.bias = l.b;
    a.residual = residual; a.ldr = l.out; a.y = y; a.ldy = l.out;
    return gemv_bf16(a, c.st);
  }
  GemmEpilogue ep;
  const int n_out = (mode == EPI_GEGLU || mode == EPI_SWIGLU) ? l.out / 2 : l.out;
  ep.C = y; ep.ldc = n_out; ep.bias = l.b; ep.residual = residual; ep.ldr = n_out; ep.mode = mode;
  return gemm_bf16(x, l.in, l.w, l.in, M, l.out, l.in, ep, c.st);
}

static bool conv_tileable(int H, int W) {
  const int tw = W >= 128 ? 128 : W;
  if (tw < 8 || (128 % tw)) return false;
  const int th = 128 / tw;
  return (H % th == 0) && (W % tw == 0);
}

// 3x3 pad-1 conv (stride 1 or 2) on NHWC; epilogue: + bias (+ bias2 per image) (+ residual)
int conv3(Ctx& c, const bf16* x, int NB, int H, int W, const Conv& cv, int stride, bf16* y, const bf16* bias2,
          const bf16* residual, int ldy) {
  const int Ho = (H - 1) / stride + 1, Wo = (W - 1) / stride + 1;
  GemmEpilogue ep;
  ep.C = y; ep.ldc = ldy ? ldy : cv.cout; ep.bias = cv.b; ep.residual = residual; ep.ldr = cv.cout;
  ep.bias2 = bias2; ep.bias2_rows = Ho * Wo;
  ++c.nl;
  if (stride == 1 && conv_tileable(H, W)) return conv3x3_bf16(x, NB, H, W, cv.cin, cv.w, cv.cout, ep, c.st);
  BUF(cols, "im2col", (size_t)NB * Ho * Wo * 9 * cv.cin);
  EMU_TRY(im2col3x3(x, cols, NB, H, W, cv.cin, stride, c.st));
  ++c.nl;
  return gemm_bf16(cols, 9 * cv.cin, cv.w, 9 * cv.cin, NB * Ho * Wo, cv.cout, 9 * cv.cin, ep, c.st);
}

int gnorm(Ctx& c, const bf16* x, const Norm& n, bf16* y, int NB, int HW, float eps, int do_silu) {
  const size_t sb = groupnorm_scratch_bytes(NB, c.groups);
  BUF(scr, "gn_scratch", sb / 2 + 8);
  c.nl += 2;
  return groupnorm_nhwc(x, n.w, n.b, y, (float*)scr, NB, HW, n.c, c.groups, eps, do_silu, c.st);
}

// ResnetBlock2D: x [NB,H,W,cin] -> y [NB,H,W,cout];  emb_act = silu(emb) [NB, temb]
static int resnet(Ctx& c, const ResnetW& r, const bf16* x, bf16* y, int NB, int H, int W, const bf16* emb_act) {
  const long M = (long)NB * H * W;
  BUF(g, "rs_norm", M * (r.cin > r.cout ? r.cin : r.cout));
  BUF(t1, "rs_t1", M * r.cout);
  BUF(tp, "rs_temb", (size_t)NB * r.cout);
  EMU_TRY(lin_rows(c, emb_act, NB, r.temb, tp));
  EMU_TRY(gnorm(c, x, r.n1, g, NB, H * W, c.gn_eps, 1));
  EMU_TRY(conv3(c, g, NB, H, W, r.c1, 1, t1, tp, nullptr));
  EMU_TRY(gnorm(c, t1, r.n2, g, NB, H * W, c.gn_eps, 1));
  const bf16* shortcut = x;
  if (r.has_sc) {
    BUF(sc, "rs_sc", M * r.cout);
    GemmEpilogue ep;
    ep.C = sc; ep.ldc = r.cout; ep.bias = r.sc.b;
    EMU_TRY(gemm_bf16(x, r.cin, r.sc.w, r.cin, (int)M, r.cout, r.cin, ep, c.st));
    ++c.nl;
    shortcut = sc;
  }
  return conv3(c, g, NB, H, W, r.c2, 1, y, nullptr, shortcut);
}

// Transformer2DModel (linear projections): x [NB, T, C] (NHWC tokens) -> y
static int transformer2d(Ctx& c, const TransW& t, const bf16* x, bf16* y, int NB, int T, const bf16* ctxv, int L, int cd) {
  const int C = t.c, hd = t.hd, Hh = C / hd;
  const long M = (long)NB * T;
  BUF(n, "tf_norm", M * C);
  BUF(h, "tf_h", M * C);
  BUF(qkv, "tf_qkv", M * 3 * C);
  BUF(att, "tf_att", M * C);
  BUF(kv, "tf_kv", (size_t)NB * L * 2 * C);
  BUF(ff, "tf_ff", M * 4 * C);
  EMU_TRY(gnorm(c, x, t.gn, n, NB, T, 1e-6f, 0));
  EMU_TRY(lin_rows(c, n, (int)M, t.pin, h));
  const float scale = 1.0f / sqrtf((float)hd);
  for (const TBlockW& b : t.blocks) {
    // self-attention
    EMU_TRY(layernorm(h, b.n1.w, b.n1.b, nullptr, n, (int)M, C, 1e-5f, c.st));
    GemmEpilogue e1;
    e1.C = qkv; e1.ldc = 3 * C;
    EMU_TRY(gemm_bf16(n, C, b.wqkv, C, (int)M, 3 * C, C, e1, c.st));
    AttnArgs a;
    a.q = qkv; a.k = qkv + C; a.v = qkv + 2 * C;
    a.q_bs = a.k_bs = a.v_bs = (long)T * 3 * C; a.q_ts = a.k_ts = a.v_ts = 3 * C; a.q_hs = a.k_hs = a.v_hs = hd;
    a.out = att; a.o_bs = (long)T * C; a.o_ts = C; a.o_hs = hd;
    a.B = NB; a.H = Hh; a.Nq = T; a.Nk = T; a.D = hd; a.scale = scale;
    EMU_TRY(attn_prefill(a, c.st));
    EMU_TRY(lin_rows(c, att, (int)M, b.o1, h, h));
    // cross-attention to the 64 regressed visual tokens
    EMU_TRY(layernorm(h, b.n2.w, b.n2.b, nullptr, n, (int)M, C, 1e-5f, c.st));
    GemmEpilogue e2;
    e2.C = qkv; e2.ldc = C;
    EMU_TRY(gemm_bf16(n, C, b.wq2, C, (int)M, C, C, e2, c.st));
    AttnArgs x2;
    x2.q = qkv; x2.q_bs = (long)T * C; x2.q_ts = C; x2.q_hs = hd;
    if (c.kv_all && b.kv_off >= 0) {
      x2.k = c.kv_all + b.kv_off; x2.v = x2.k + C;
      x2.k_bs = x2.v_bs = (long)L * c.kv_ld; x2.k_ts = x2.v_ts = c.kv_ld; x2.k_hs = x2.v_hs = hd;
    } else {
      GemmEpilogue e3;
      e3.C = kv; e3.ldc = 2 * C;
      EMU_TRY(gemm_bf16(ctxv, cd, b.wkv2, cd, NB * L, 2 * C, cd, e3, c.st));
      x2.k = kv; x2.v = kv + C; x2.k_bs = x2.v_bs = (long)L * 2 * C; x2.k_ts = x2.v_ts = 2 * C; x2.k_hs = x2.v_hs = hd;
    }
    x2.out = att; x2.o_bs = (long)T * C; x2.o_ts = C; x2.o_hs = hd;
    x2.B = NB; x2.H = Hh; x2.Nq = T; x2.Nk = L; x2.D = hd; x2.scale = scale;
    EMU_TRY(attn_prefill(x2, c.st));
    EMU_TRY(lin_rows(c, att, (int)M, b.o2, h, h));
    // GEGLU feed-forward
    EMU_TRY(layernorm(h, b.n3.w, b.n3.b, nullptr, n, (int)M, C, 1e-5f, c.st));
    EMU_TRY(lin_rows(c, n, (int)M, b.ff1, ff, nullptr, EPI_GEGLU));
    EMU_TRY(lin_rows(c, ff, (int)M, b.ff2, h, h));
    c.nl += (c.kv_all && b.kv_off >= 0) ? 7 : 8;
  }
  return lin_rows(c, h, (int)M, t.pout, y, x);
}

// stack every block's [to_k; to_v] rows into one matrix (done once after the weights are loaded, outside graph capture)
static int unet_stack_kv(EmuEngine* e, UNetModel* m, cudaStream_t st) {
  if (m->kv_all_ready) return EMU_OK;
  const int cd = m->cfg.cross_attention_dim;
  std::vector<TBlockW*> blocks;
  std::vector<int> widths;
  auto visit = [&](TransW& t) {
    for (TBlockW& b : t.blocks) {
      blocks.push_back(&b);
      widths.push_back(2 * t.c);
    }
  };
  for (auto& v : m->down_att) for (TransW& t : v) visit(t);
  visit(m->mid_att);
  for (auto& v : m->up_att) for (TransW& t : v) visit(t);
  long n = 0;
  for (int w : widths) n += w;
  if (n == 0) {
    m->kv_all_ready = true;
    return EMU_OK;
  }
  cudaStreamCaptureStatus cs = cudaStreamCaptureStatusNone;
  cudaStreamIsCapturing(st, &cs);
  if (cs != cudaStreamCaptureStatusNone) return EMU_OK;  // never allocate / restack inside a capture: keep the per-block path
  if (m->kv_all_n != n || !m->kv_all_w) {
    m->kv_all_w = (bf16*)e->dmalloc((size_t)n * cd * 2);
    if (!m->kv_all_w) return e->fail(EMU_ERR_NOMEM, "cross-attention weight stack alloc failed");
    m->kv_all_n = n;
  }
  long off = 0;
  for (size_t i = 0; i < blocks.size(); ++i) {
    if (!blocks[i]->wkv2) return e->fail(EMU_ERR_STATE, "unet cross-attention weights missing");
    if (cudaMemcpyAsync(m->kv_all_w + off * cd, blocks[i]->wkv2, (size_t)widths[i] * cd * 2, cudaMemcpyDeviceToDevice, st) !=
        cudaSuccess)
      return e->fail(EMU_ERR_CUDA, "cross-attention weight stack copy failed");
    blocks[i]->kv_off = off;
    off += widths[i];
  }
  m->kv_all_ready = true;
  return EMU_OK;
}

// UNet2DConditionModel.forward on NHWC input [B2, h, w, cin_pad]; t_dev [B2] fp32; returns eps in `eps` [B2*h*w, ld 8]
static int unet_core(Ctx& c, UNetModel* m, const bf16* x_in, const float* t_dev, const bf16* ctxv, int L, const bf16* text_embeds,
                     const int* time_ids, int h, int w, bf16* eps) {
  const EmuUNetConfig& cf = m->cfg;
  const int nb = cf.n_blocks, lpb = cf.layers_per_block, B2 = c.B2;
  const int* boc = cf.block_out_channels;
  const int temb = boc[0] * 4;
  PdlScope pdl_chain(1);  // ~1000 short kernels per forward: overlap every prologue with its predecessor's tail
  EMU_TRY(unet_stack_kv(c.e, m, c.st));
  c.kv_all = nullptr;
  if (m->kv_all_ready && m->kv_all_n > 0) {
    BUF(kv_all, "kv_all", (size_t)B2 * L * m->kv_all_n);
    GemmEpilogue ek;
    ek.C = kv_all; ek.ldc = (int)m->kv_all_n;
    EMU_TRY(gemm_bf16(ctxv, cf.cross_attention_dim, m->kv_all_w, cf.cross_attention_dim, B2 * L, (int)m->kv_all_n,
                      cf.cross_attention_dim, ek, c.st));
    ++c.nl;
    c.kv_all = kv_all;
    c.kv_ld = m->kv_all_n;
  }
  // ---- time / added-condition embeddings ----
  BUF(te_in, "te_in", (size_t)B2 * boc[0]);
  BUF(te_mid, "te_mid", (size_t)B2 * temb);
  BUF(emb, "emb", (size_t)B2 * temb);
  BUF(emb_act, "emb_act", (size_t)B2 * temb);
  EMU_TRY(timestep_embedding(t_dev, te_in, B2, boc[0], boc[0], 0, 1, c.st));
  EMU_TRY(lin_rows(c, te_in, B2, m->te1, te_mid));
  EMU_TRY(silu_rows(te_mid, te_mid, (long)B2 * temb, c.st));
  EMU_TRY(lin_rows(c, te_mid, B2, m->te2, emb));
  c.nl += 2;
  if (cf.addition_time_embed_dim > 0) {
    if (!text_embeds || !time_ids) return c.e->fail(EMU_ERR_INVALID, "text_time conditioning needs text_embeds and time_ids");
    const int ad = cf.addition_time_embed_dim, pin = cf.projection_class_embeddings_input_dim, cd = cf.cross_attention_dim;
    if (pin != cd + 6 * ad) return c.e->fail(EMU_ERR_INVALID, "projection_class_embeddings_input_dim mismatch");
    BUF(add_in, "add_in", (size_t)B2 * pin);
    BUF(tidf, "tid_f", (size_t)B2 * 6 * 2 + 8);
    EMU_TRY(int_to_float(time_ids, (float*)tidf, B2 * 6, c.st));
    EMU_TRY(copy_cols(text_embeds, add_in, B2, cd, cd, pin, 0, c.st));
    EMU_TRY(timestep_embedding((const float*)tidf, add_in, B2 * 6, ad, pin, cd, 6, c.st));
    EMU_TRY(lin_rows(c, add_in, B2, m->ae1, te_mid));
    EMU_TRY(silu_rows(te_mid, te_mid, (long)B2 * temb, c.st));
    EMU_TRY(lin_rows(c, te_mid, B2, m->ae2, emb, emb));  // emb = emb + aug_emb
    c.nl += 4;
  }
  EMU_TRY(silu_rows(emb, emb_act, (long)B2 * temb, c.st));
  ++c.nl;

  // ---- down path ----
  struct Skip { bf16* p; int C, H, W; };
  std::vector<Skip> skips;
  int H = h, W = w, C = boc[0];
  int sid = 0;
  auto skip_buf = [&](int Cc, int Hh, int Ww) -> bf16* {
    char name[32];
    snprintf(name, sizeof(name), "skip%d", sid++);
    return c.buf(name, (size_t)B2 * Hh * Ww * Cc);
  };
  bf16* cur = skip_buf(C, H, W);
  if (!cur) return c.e->fail(EMU_ERR_NOMEM, "skip alloc");
  EMU_TRY(conv3(c, x_in, B2, H, W, m->conv_in, 1, cur, nullptr, nullptr));
  skips.push_back({cur, C, H, W});
  for (int i = 0; i < nb; ++i) {
    for (int j = 0; j < lpb; ++j) {
      const ResnetW& r = m->down_res[i][j];
      const bool has_att = !m->down_att[i].empty();
      bf16* out = skip_buf(r.cout, H, W);
      if (!out) return c.e->fail(EMU_ERR_NOMEM, "skip alloc");
      if (has_att) {
        BUF(tmp, "blk_tmp", (size_t)B2 * H * W * r.cout);
        EMU_TRY(resnet(c, r, cur, tmp, B2, H, W, emb_act));
        EMU_TRY(transformer2d(c, m->down_att[i][j], tmp, out, B2, H * W, ctxv, L, cf.cross_attention_dim));
      } else {
        EMU_TRY(resnet(c, r, cur, out, B2, H, W, emb_act));
      }
      cur = out; C = r.cout;
      skips.push_back({cur, C, H, W});
    }
    if (i < nb - 1) {
      bf16* out = skip_buf(C, H / 2, W / 2);
      if (!out) return c.e->fail(EMU_ERR_NOMEM, "skip alloc");
      EMU_TRY(conv3(c, cur, B2, H, W, m->down_samp[i], 2, out, nullptr, nullptr));
      H /= 2; W /= 2;
      cur = out;
      skips.push_back({cur, C, H, W});
    }
  }
  // ---- mid ----
  {
    BUF(ma, "mid_a", (size_t)B2 * H * W * C);
    BUF(mb, "mid_b", (size_t)B2 * H * W * C);
    EMU_TRY(resnet(c, m->mid_r0, cur, ma, B2, H, W, emb_act));
    if (!m->mid_att.blocks.empty()) {
      EMU_TRY(transformer2d(c, m->mid_att, ma, mb, B2, H * W, ctxv, L, cf.cross_attention_dim));
      EMU_TRY(resnet(c, m->mid_r1, mb, ma, B2, H, W, emb_act));
      cur = ma;
    } else {
      EMU_TRY(resnet(c, m->mid_r1, ma, mb, B2, H, W, emb_act));
      cur = mb;
    }
  }
  // ---- up path ----
  int pp = 0;
  for (int i = 0; i < nb; ++i) {
    for (int j = 0; j < lpb + 1; ++j) {
      const ResnetW& r = m->up_res[i][j];
      const Skip s = skips.back();
      skips.pop_back();
      const long M = (long)B2 * H * W;
      BUF(cat, "up_cat", M * (C + s.C));
      EMU_TRY(copy_cols(cur, cat, M, C, C, C + s.C, 0, c.st));
      EMU_TRY(copy_cols(s.p, cat, M, s.C, s.C, C + s.C, C, c.st));
      c.nl += 2;
      char nm[32];
      snprintf(nm, sizeof(nm), "up_out%d", pp ^= 1);
      BUF(out, nm, M * r.cout);
      if (!m->up_att[i].empty()) {
        BUF(tmp, "blk_tmp", M * r.cout);
        EMU_TRY(resnet(c, r, cat, tmp, B2, H, W, emb_act));
        EMU_TRY(transformer2d(c, m->up_att[i][j], tmp, out, B2, H * W, ctxv, L, cf.cross_attention_dim));
      } else {
        EMU_TRY(resnet(c, r, cat, out, B2, H, W, emb_act));
      }
      cur = out; C = r.cout;
    }
    if (i < nb - 1) {
      BUF(up, "up_big", (size_t)B2 * 4 * H * W * C);
      EMU_TRY(upsample2x_nhwc(cur, up, B2, H, W, C, c.st));
      ++c.nl;
      H *= 2; W *= 2;
      char nm[32];
      snprintf(nm, sizeof(nm), "up_out%d", pp ^= 1);
      BUF(out, nm, (size_t)B2 * H * W * C);
      EMU_TRY(conv3(c, up, B2, H, W, m->up_samp[i], 1, out, nullptr, nullptr));
      cur = out;
    }
  }
  // ---- out ----
  BUF(g, "rs_norm", (size_t)B2 * H * W * C);
  EMU_TRY(gnorm(c, cur, m->norm_out, g, B2, H * W, cf.norm_eps, 1));
  return conv3(c, g, B2, H, W, m->conv_out, 1, eps, nullptr, nullptr, 8);
}

static int unet_ready(EmuEngine* e) {
  if (!e->unet) return e->fail(EMU_ERR_STATE, "UNet not configured");
  for (auto& kv : e->unet->specs)
    if (!*kv.second.dst) return e->fail(EMU_ERR_STATE, "UNet weight missing: " + kv.first);
  return EMU_OK;
}

}  // namespace emu

extern "C" int emu_unet_forward(EmuEngine* e, const void* latents_nchw, float timestep, const void* ctxv, int L,
                                const void* text_embeds, const int32_t* time_ids, int B2, int h, int w, void* noise_pred,
                                emu_stream_t stream) {
  if (!e || !latents_nchw || !ctxv || !noise_pred || B2 < 1) return EMU_ERR_INVALID;
  EMU_TRY(unet_ready(e));
  UNetModel* m = e->unet;
  cudaStream_t st = (cudaStream_t)stream;
  Ctx c{e, &m->bufs, &m->grew, st, B2, m->cfg.norm_groups, m->cfg.norm_eps};
  const int Cin = m->cfg.in_channels, Cp = m->conv_in.cin;
  BUF(xin, "x_in", (size_t)B2 * h * w * Cp);
  BUF(eps, "eps", (size_t)B2 * h * w * 8);
  BUF(tdev, "t_dev_big", (size_t)B2 * 2 + 8);
  {
    std::vector<float> tt(B2, timestep);
    if (cudaMemcpyAsync(tdev, tt.data(), B2 * sizeof(float), cudaMemcpyHostToDevice, st) != cudaSuccess)
      return e->fail(EMU_ERR_CUDA, "timestep copy");
    cudaStreamSynchronize(st);  // tt goes out of scope (stand-alone entry point; the denoise step uses device params)
  }
  EMU_TRY(nchw_to_nhwc((const bf16*)latents_nchw, xin, B2, Cin, h * w, Cp, 1.0f, st));
  EMU_TRY(unet_core(c, m, xin, (const float*)tdev, (const bf16*)ctxv, L, (const bf16*)text_embeds, time_ids, h, w, eps));
  EMU_TRY(nhwc_to_nchw(eps, (bf16*)noise_pred, B2, m->cfg.out_channels, h * w, 8, st));
  count_launch(c.nl + 2);
  return EMU_OK;
}

// One denoise iteration.  ms == nullptr: Euler (Emu2-Gen); otherwise the 8 linear-multistep scalars of cfg_multistep_kernel
// (PNDM, Emu1) with `state` = [4][B*C*h*w] fp32 (3 history planes + the saved sample).
static int denoise_step_impl(EmuEngine* e, float* latents, float sigma, float sigma_next, float timestep, float guidance,
                             const float* ms, float* state, const void* ctxv, int L, const void* text_embeds,
                             const int32_t* time_ids, int B, int h, int w, emu_stream_t stream) {
  if (!e || !latents || !ctxv || B < 1) return EMU_ERR_INVALID;
  EMU_TRY(unet_ready(e));
  UNetModel* m = e->unet;
  cudaStream_t st = (cudaStream_t)stream;
  const int cfg = guidance > 1.0f ? 1 : 0;  // do_classifier_free_guidance (Emu2/emu/diffusion.py:97)
  // CFG-parallel pair: this rank runs only its half of the [cond; uncond] UNet batch (SURVEY.md §8e "UNet, batch 1")
  const int split = (cfg && m->xch && m->xch_peer && e->tp_size == 2) ? 1 : 0;
  if (split && (size_t)B * h * w * 16 > kXchSlot) return e->fail(EMU_ERR_INVALID, "batch too large for the CFG-parallel exchange");
  if (split && (m->cfg.out_channels > 8)) return e->fail(EMU_ERR_UNSUPPORTED, "CFG-parallel exchange: out_channels > 8");
  const int B2 = (cfg && !split) ? 2 * B : B;
  const int Cin = m->cfg.in_channels, Cp = m->conv_in.cin;
  const int cd = m->cfg.cross_attention_dim;
  if (split) {  // the caller passes the full [2B, ...] conditioning on both ranks (same API); take this rank's half
    ctxv = (const bf16*)ctxv + (size_t)e->tp_rank * B * L * cd;
    if (text_embeds) text_embeds = (const bf16*)text_embeds + (size_t)e->tp_rank * B * cd;
    if (time_ids) time_ids = time_ids + (size_t)e->tp_rank * B * 6;
  }
  // per-step scalars go through device memory so the captured graph is step-independent
  float hp[12] = {sigma, sigma_next, guidance, timestep, 0, 0, 0, 0, 0, 0, 0, 0};
  if (ms) {
    for (int i = 0; i < 6; ++i) hp[4 + i] = ms[i];
    hp[10] = guidance;
    hp[11] = ms[7];
  }
  if (ms && split) return e->fail(EMU_ERR_UNSUPPORTED, "CFG-parallel exchange with the multistep scheduler");
  if (cudaMemcpyAsync(m->step_params, hp, sizeof(hp), cudaMemcpyHostToDevice, st) != cudaSuccess)
    return e->fail(EMU_ERR_CUDA, "step params copy");
  cudaStreamSynchronize(st);  // hp is a stack buffer

  auto body = [&](cudaStream_t s, int* nl) -> int {
    Ctx c{e, &m->bufs, &m->grew, s, B2, m->cfg.norm_groups, m->cfg.norm_eps};
    BUF(xin, "x_in", (size_t)B2 * h * w * Cp);
    BUF(eps, "eps", (size_t)B2 * h * w * 8);
    BUF(tdev, "t_dev_big", (size_t)B2 * 2 + 8);
    EMU_TRY(fill_float((float*)tdev, B2, m->step_params + 3, s));
    EMU_TRY(cfg_prepare(latents, xin, B, Cin, h * w, Cp, m->step_params, (cfg && !split) ? 2 : 1, s));
    EMU_TRY(unet_core(c, m, xin, (const float*)tdev, (const bf16*)ctxv, L, (const bf16*)text_embeds, time_ids, h, w, eps));
    if (split) {
      const long n_pix = (long)B * h * w;
      int grid = (int)((n_pix + 2047) / 2048);
      if (grid > kXchCtas) grid = kXchCtas;
      cfg_exchange_euler_kernel<<<grid, 256, 0, s>>>(latents, eps, m->xch, m->xch_peer, e->tp_rank, B, m->cfg.out_channels,
                                                     h * w, m->step_params);
      if (cudaGetLastError() != cudaSuccess) return e->fail(EMU_ERR_CUDA, "CFG-parallel exchange launch failed");
    } else if (ms) {
      const long n = (long)B * m->cfg.out_channels * h * w;
      EMU_TRY(cfg_multistep(latents, eps, state, state + 3 * n, B, m->cfg.out_channels, h * w, 8, m->step_params + 4, cfg, s));
    } else {
      EMU_TRY(cfg_euler(latents, eps, B, m->cfg.out_channels, h * w, 8, m->step_params, cfg, s));
    }
    *nl = c.nl + 3;
    return EMU_OK;
  };
  const char* no_graph = getenv("EMU_NO_GRAPH");
  const bool use_graph = e->use_graphs && !(no_graph && no_graph[0] == '1');
  auto key = std::make_tuple((const void*)latents, (const void*)ctxv, (const void*)text_embeds,
                             ms ? (const void*)state : (const void*)time_ids, B, h, w * 4 + cfg + 2 * split, L);
  auto it = m->graphs.find(key);
  if (use_graph && it != m->graphs.end()) {
    if (cudaGraphLaunch(it->second, st) != cudaSuccess) return e->fail(EMU_ERR_CUDA, "denoise graph launch failed");
    count_launch(m->n_launch);
    return EMU_OK;
  }
  // first call with these shapes runs eagerly (sizes every workspace); the second call captures
  m->grew = false;
  int nl = 0;
  if (!use_graph || !m->warmed.count(key)) {
    EMU_TRY(body(st, &nl));
    count_launch(nl);
    m->warmed[key] = 1;
    if (m->grew) {
      for (auto& g : m->graphs) cudaGraphExecDestroy(g.second);
      m->graphs.clear();
    }
    return EMU_OK;
  }
  if (!e->cap_stream && cudaStreamCreateWithFlags(&e->cap_stream, cudaStreamNonBlocking) != cudaSuccess)
    return e->fail(EMU_ERR_CUDA, "capture stream create failed");
  if (cudaStreamBeginCapture(e->cap_stream, cudaStreamCaptureModeRelaxed) != cudaSuccess)
    return e->fail(EMU_ERR_CUDA, "denoise graph capture begin failed");
  int rc = body(e->cap_stream, &nl);
  cudaGraph_t graph = nullptr;
  cudaError_t ce = cudaStreamEndCapture(e->cap_stream, &graph);
  if (rc != EMU_OK || ce != cudaSuccess || !graph || m->grew) {
    if (graph) cudaGraphDestroy(graph);
    cudaGetLastError();
    if (rc != EMU_OK) return rc;
    return e->fail(EMU_ERR_CUDA, "denoise graph capture failed");
  }
  cudaGraphExec_t exec = nullptr;
  ce = cudaGraphInstantiate(&exec, graph, 0);
  cudaGraphDestroy(graph);
  if (ce != cudaSuccess) return e->fail(EMU_ERR_CUDA, "denoise graph instantiate failed");
  m->graphs[key] = exec;
  m->n_launch = nl;
  if (cudaGraphLaunch(exec, st) != cudaSuccess) return e->fail(EMU_ERR_CUDA, "denoise graph launch failed");
  count_launch(nl);
  return EMU_OK;
}

extern "C" int emu_denoise_step(EmuEngine* e, float* latents, float sigma, float sigma_next, float timestep,
                                float guidance, const void* ctxv, int L, const void* text_embeds,
                                const int32_t* time_ids, int B, int h, int w, emu_stream_t stream) {
  return denoise_step_impl(e, latents, sigma, sigma_next, timestep, guidance, nullptr, nullptr, ctxv, L, text_embeds, time_ids,
                           B, h, w, stream);
}

extern "C" int emu_denoise_step_multistep(EmuEngine* e, float* latents, float* state, const float* host_coef8, float timestep,
                                          float guidance, const void* ctxv, int L, int B, int h, int w, emu_stream_t stream) {
  if (!state || !host_coef8) return EMU_ERR_INVALID;
  return denoise_step_impl(e, latents, 0.f, 0.f, timestep, guidance, host_coef8, state, ctxv, L, nullptr, nullptr, B, h, w,
                           stream);
}
