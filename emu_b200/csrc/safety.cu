// emu_b200 — the pipelines' NSFW safety checker (include/emu_b200_safety.h).
//
// Reference: StableDiffusionSafetyChecker (diffusers 0.24.0, pipelines/stable_diffusion/safety_checker.py — third-party and
// unpinned, restated here) as called from Emu2/emu/diffusion.py:236-249 and Emu1/models/pipeline.py:203-215, in bf16 (both
// pipelines cast the checker and its input to bf16):
//   pre-processing : CLIPImageProcessor, preprocess.cu (clip_plan / clip_launch)
//   tower          : transformers CLIPVisionModel — patch conv (no bias), [class_embedding | patches] + position_embedding,
//                    pre_layrnorm, pre-LN blocks x += out_proj(attn(LN1 x)); x += fc2(quick_gelu(fc1(LN2 x))),
//                    pooled = post_layernorm(x[:, 0]); image_embeds = visual_projection(pooled)  (gemm_tc / attention /
//                    layernorm, the EVA tower's kernels)
//   head           : cosine_distance against special_care_embeds / concept_embeds, the ordered special-care adjustment
//                    and the concept thresholds; flagged images are blacked out — safety_score_kernel below
// Under tensor / CFG parallelism every rank holds the whole checker and computes the same flags: no collective.
#include <math.h>
#include <string.h>

#include <map>
#include <utility>

#include "../../include/emu_b200_safety.h"
#include "common.cuh"
#include "engine.h"

namespace emu {

constexpr int kMaxConcepts = 64;

#define EMU_CHECK_RC(x)            \
  do {                             \
    int rc_ = (x);                 \
    if (rc_ != EMU_OK) return rc_; \
  } while (0)

static long numel_of(const int64_t* shape, int ndim) {
  long n = 1;
  for (int i = 0; i < ndim; ++i) n *= shape[i];
  return n;
}

struct SafetyBlock {
  bf16 *ln1w = nullptr, *ln1b = nullptr, *ln2w = nullptr, *ln2b = nullptr;
  bf16 *wqkv = nullptr, *bqkv = nullptr, *wo = nullptr, *bo = nullptr;
  bf16 *w1 = nullptr, *b1 = nullptr, *w2 = nullptr, *b2 = nullptr;
  unsigned loaded = 0;  // one bit per reference tensor (q / k / v share the fused buffers)
  static constexpr unsigned kAll = (1u << 16) - 1;
};
static const char* kBlockParts[16] = {"layer_norm1.weight", "layer_norm1.bias", "layer_norm2.weight", "layer_norm2.bias",
                                      "self_attn.q_proj.weight", "self_attn.k_proj.weight", "self_attn.v_proj.weight",
                                      "self_attn.q_proj.bias", "self_attn.k_proj.bias", "self_attn.v_proj.bias",
                                      "self_attn.out_proj.weight", "self_attn.out_proj.bias", "mlp.fc1.weight",
                                      "mlp.fc1.bias", "mlp.fc2.weight", "mlp.fc2.bias"};

struct ClipTables {  // one input size: the sliced coefficient tables on the device (uploaded once, from pinned memory)
  ClipPlan plan;
  int* host = nullptr;
  int* dev = nullptr;
};

struct SafetyModel {
  EmuSafetyConfig cfg{};
  int kpad = 0;
  std::vector<SafetyBlock> blocks;
  bf16 *cls = nullptr, *pos = nullptr, *wpatch = nullptr, *pre_w = nullptr, *pre_b = nullptr, *post_w = nullptr,
       *post_b = nullptr, *proj = nullptr, *special = nullptr, *concepts = nullptr, *special_w = nullptr, *concept_w = nullptr;
  std::vector<void*> owned;
  DevBuf pix, tmp, cols, x, y, qkv, att, mlp, emb;
  std::map<std::pair<int, int>, ClipTables> tables;

  bf16* alloc(size_t n) {
    void* p = nullptr;
    if (cudaMalloc(&p, n * 2) != cudaSuccess) { cudaGetLastError(); return nullptr; }
    owned.push_back(p);
    return (bf16*)p;
  }
  int ensure(DevBuf& b, size_t bytes) {
    if (b.bytes >= bytes) return EMU_OK;
    void* p = nullptr;
    if (cudaMalloc(&p, bytes) != cudaSuccess) { cudaGetLastError(); return EMU_ERR_NOMEM; }
    owned.push_back(p);
    b.p = p;
    b.bytes = bytes;
    return EMU_OK;
  }
};

void safety_destroy(SafetyModel* m) {
  if (!m) return;
  for (auto& t : m->tables) {
    if (t.second.host) cudaFreeHost(t.second.host);
  }
  for (void* p : m->owned) cudaFree(p);
  cudaGetLastError();
  delete m;
}

__global__ void safety_zero_kernel(bf16* d, size_t n) {
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
    d[i] = __float2bfloat16(0.f);
}
// dst[r, c] = src[r, c] for r < rows, c < cols; dst row stride ld (the patch kernel padded to K = kpad)
__global__ void safety_copy_rows_kernel(bf16* dst, const bf16* __restrict__ src, int rows, int cols, int ld) {
  const long total = (long)rows * cols;
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x)
    dst[(i / cols) * ld + i % cols] = src[i];
}

static bool shape_is(const int64_t* shape, int ndim, std::initializer_list<long> want) {
  if ((size_t)ndim != want.size()) return false;
  int i = 0;
  for (long w : want)
    if (shape[i++] != w) return false;
  return true;
}

int safety_load_tensor(EmuEngine* e, const std::string& key, const bf16* src, const int64_t* shape, int ndim,
                       cudaStream_t st) {
  SafetyModel* m = e->safety;
  if (!m) return e->fail(EMU_ERR_STATE, "emu_safety_configure must be called before loading safety_checker.* tensors");
  const EmuSafetyConfig& c = m->cfg;
  const int W = c.width, P = c.patch_size, G = c.image_size / P, N = G * G + 1;
  auto put = [&](bf16** dst, size_t n, size_t off) -> int {
    if (!*dst) {
      *dst = m->alloc(n);
      if (!*dst) return e->fail(EMU_ERR_NOMEM, "safety checker weight alloc failed");
    }
    const long cnt = numel_of(shape, ndim);
    return cudaMemcpyAsync(*dst + off, src, (size_t)cnt * 2, cudaMemcpyDeviceToDevice, st) == cudaSuccess
               ? EMU_OK : e->fail(EMU_ERR_CUDA, "safety checker weight copy failed");
  };
  auto bad = [&]() { return e->fail(EMU_ERR_INVALID, "shape mismatch for safety_checker." + key); };
  // head (diffusers StableDiffusionSafetyChecker parameters)
  if (key == "concept_embeds") return shape_is(shape, ndim, {c.n_concepts, c.proj_dim}) ? put(&m->concepts, (size_t)c.n_concepts * c.proj_dim, 0) : bad();
  if (key == "special_care_embeds") return shape_is(shape, ndim, {c.n_special, c.proj_dim}) ? put(&m->special, (size_t)c.n_special * c.proj_dim, 0) : bad();
  if (key == "concept_embeds_weights") return shape_is(shape, ndim, {c.n_concepts}) ? put(&m->concept_w, c.n_concepts, 0) : bad();
  if (key == "special_care_embeds_weights") return shape_is(shape, ndim, {c.n_special}) ? put(&m->special_w, c.n_special, 0) : bad();
  if (key == "visual_projection.weight") return shape_is(shape, ndim, {c.proj_dim, W}) ? put(&m->proj, (size_t)c.proj_dim * W, 0) : bad();
  // tower: transformers CLIPVisionModel names, under diffusers' `vision_model.` (CLIPVisionModel.vision_model.*)
  std::string k;
  if (key.compare(0, 26, "vision_model.vision_model.") == 0) k = key.substr(26);
  else if (key.compare(0, 13, "vision_model.") == 0) k = key.substr(13);
  else return e->fail(EMU_ERR_INVALID, "unknown safety_checker key " + key);
  if (k == "embeddings.position_ids") return EMU_OK;  // a buffer (arange), not a weight
  if (k == "embeddings.class_embedding") return shape_is(shape, ndim, {W}) ? put(&m->cls, W, 0) : bad();
  if (k == "embeddings.position_embedding.weight") return shape_is(shape, ndim, {N, W}) ? put(&m->pos, (size_t)N * W, 0) : bad();
  if (k == "embeddings.patch_embedding.weight") {
    if (!shape_is(shape, ndim, {W, 3, P, P})) return bad();
    if (!m->wpatch) {  // [W, 3*P*P] zero-padded to K = kpad (the EVA tower's layout: TMA wants 16-byte rows)
      m->wpatch = m->alloc((size_t)W * m->kpad);
      if (!m->wpatch) return e->fail(EMU_ERR_NOMEM, "safety checker weight alloc failed");
      safety_zero_kernel<<<4 * kNumSMs, 256, 0, st>>>(m->wpatch, (size_t)W * m->kpad);
    }
    safety_copy_rows_kernel<<<4 * kNumSMs, 256, 0, st>>>(m->wpatch, src, W, 3 * P * P, m->kpad);
    count_launch(2);
    return cudaGetLastError() == cudaSuccess ? EMU_OK : e->fail(EMU_ERR_CUDA, "patch kernel repack failed");
  }
  if (k == "pre_layrnorm.weight") return shape_is(shape, ndim, {W}) ? put(&m->pre_w, W, 0) : bad();
  if (k == "pre_layrnorm.bias") return shape_is(shape, ndim, {W}) ? put(&m->pre_b, W, 0) : bad();
  if (k == "post_layernorm.weight") return shape_is(shape, ndim, {W}) ? put(&m->post_w, W, 0) : bad();
  if (k == "post_layernorm.bias") return shape_is(shape, ndim, {W}) ? put(&m->post_b, W, 0) : bad();
  const char* pre = "encoder.layers.";
  if (k.compare(0, strlen(pre), pre) != 0) return e->fail(EMU_ERR_INVALID, "unknown safety_checker key " + key);
  const size_t p0 = strlen(pre), p1 = k.find('.', p0);
  if (p1 == std::string::npos) return e->fail(EMU_ERR_INVALID, "unknown safety_checker key " + key);
  const int li = atoi(k.substr(p0, p1 - p0).c_str());
  if (li < 0 || li >= c.layers) return e->fail(EMU_ERR_INVALID, "safety checker layer index out of range: " + key);
  const std::string sub = k.substr(p1 + 1);
  SafetyBlock& b = m->blocks[li];
  int part = -1;
  for (int i = 0; i < 16; ++i)
    if (sub == kBlockParts[i]) part = i;
  if (part < 0) return e->fail(EMU_ERR_INVALID, "unknown safety_checker key " + key);
  int rc;
  switch (part) {
    case 0: rc = shape_is(shape, ndim, {W}) ? put(&b.ln1w, W, 0) : bad(); break;
    case 1: rc = shape_is(shape, ndim, {W}) ? put(&b.ln1b, W, 0) : bad(); break;
    case 2: rc = shape_is(shape, ndim, {W}) ? put(&b.ln2w, W, 0) : bad(); break;
    case 3: rc = shape_is(shape, ndim, {W}) ? put(&b.ln2b, W, 0) : bad(); break;
    // q, k, v fused into one [3W, W] weight and one [3W] bias (unlike the EVA tower, k has a bias)
    case 4: case 5: case 6: rc = shape_is(shape, ndim, {W, W}) ? put(&b.wqkv, (size_t)3 * W * W, (size_t)(part - 4) * W * W) : bad(); break;
    case 7: case 8: case 9: rc = shape_is(shape, ndim, {W}) ? put(&b.bqkv, (size_t)3 * W, (size_t)(part - 7) * W) : bad(); break;
    case 10: rc = shape_is(shape, ndim, {W, W}) ? put(&b.wo, (size_t)W * W, 0) : bad(); break;
    case 11: rc = shape_is(shape, ndim, {W}) ? put(&b.bo, W, 0) : bad(); break;
    case 12: rc = shape_is(shape, ndim, {c.mlp, W}) ? put(&b.w1, (size_t)c.mlp * W, 0) : bad(); break;
    case 13: rc = shape_is(shape, ndim, {c.mlp}) ? put(&b.b1, c.mlp, 0) : bad(); break;
    case 14: rc = shape_is(shape, ndim, {W, c.mlp}) ? put(&b.w2, (size_t)W * c.mlp, 0) : bad(); break;
    default: rc = shape_is(shape, ndim, {W}) ? put(&b.b2, W, 0) : bad(); break;
  }
  if (rc == EMU_OK) b.loaded |= 1u << part;
  return rc;
}

static int safety_ready(EmuEngine* e) {
  SafetyModel* m = e->safety;
  if (!m) return e->fail(EMU_ERR_STATE, "safety checker not configured (emu_safety_configure)");
  struct { const void* p; const char* name; } stem[] = {
      {m->wpatch, "embeddings.patch_embedding"}, {m->cls, "embeddings.class_embedding"},
      {m->pos, "embeddings.position_embedding"}, {m->pre_w, "pre_layrnorm.weight"}, {m->pre_b, "pre_layrnorm.bias"},
      {m->post_w, "post_layernorm.weight"}, {m->post_b, "post_layernorm.bias"}, {m->proj, "visual_projection"},
      {m->special, "special_care_embeds"}, {m->concepts, "concept_embeds"},
      {m->special_w, "special_care_embeds_weights"}, {m->concept_w, "concept_embeds_weights"}};
  for (auto& s : stem)
    if (!s.p) return e->fail(EMU_ERR_STATE, std::string("safety checker is missing ") + s.name);
  for (size_t l = 0; l < m->blocks.size(); ++l) {
    const unsigned ld = m->blocks[l].loaded;
    if (ld == SafetyBlock::kAll) continue;
    std::string miss;
    for (int i = 0; i < 16; ++i)
      if (!(ld & (1u << i))) miss += std::string(miss.empty() ? "" : ", ") + kBlockParts[i];
    return e->fail(EMU_ERR_STATE, "safety checker layer " + std::to_string(l) + " is missing " + miss);
  }
  return EMU_OK;
}

// ---- the tower: pixel_values [B, 3, S, S] bf16 -> image_embeds [B, proj] bf16 ----
static int safety_tower(EmuEngine* e, const bf16* pix, int B, bf16* out, cudaStream_t st) {
  SafetyModel* m = e->safety;
  const EmuSafetyConfig& c = m->cfg;
  PdlScope pdl_chain(1);
  const int W = c.width, G = c.image_size / c.patch_size, Np = G * G, N = Np + 1, Hh = c.heads, D = W / Hh;
  const long M = (long)B * N;
  int rc = EMU_OK;
  if ((rc = m->ensure(m->cols, (size_t)B * Np * (m->kpad + W) * 2)) || (rc = m->ensure(m->x, (size_t)M * W * 2)) ||
      (rc = m->ensure(m->y, (size_t)M * W * 2)) || (rc = m->ensure(m->qkv, (size_t)M * 3 * W * 2)) ||
      (rc = m->ensure(m->att, (size_t)M * W * 2)) || (rc = m->ensure(m->mlp, (size_t)M * c.mlp * 2)))
    return e->fail(rc, "safety checker workspace alloc failed");
  bf16 *x = (bf16*)m->x.p, *y = (bf16*)m->y.p, *qkv = (bf16*)m->qkv.p, *att = (bf16*)m->att.p, *mlp = (bf16*)m->mlp.p;
  bf16* cols = (bf16*)m->cols.p;
  bf16* pemb = cols + (size_t)B * Np * m->kpad;

  // embeddings: patch conv (no bias) as im2col + GEMM, [class_embedding | patches] + position_embedding, pre_layrnorm
  EMU_CHECK_RC(vit_im2col(pix, cols, B, 3, c.image_size, c.patch_size, m->kpad, st));
  {
    GemmEpilogue ep;
    ep.C = pemb; ep.ldc = W;
    EMU_CHECK_RC(gemm_bf16(cols, m->kpad, m->wpatch, m->kpad, B * Np, W, m->kpad, ep, st));
  }
  EMU_CHECK_RC(vit_assemble(pemb, m->cls, m->pos, y, B, Np, W, st));
  EMU_CHECK_RC(layernorm(y, m->pre_w, m->pre_b, nullptr, x, (int)M, W, c.ln_eps, st));
  count_launch(4);

  const float scale = 1.0f / sqrtf((float)D);
  for (int l = 0; l < c.layers; ++l) {
    const SafetyBlock& b = m->blocks[l];
    EMU_CHECK_RC(layernorm(x, b.ln1w, b.ln1b, nullptr, y, (int)M, W, c.ln_eps, st));
    GemmEpilogue ep;
    ep.C = qkv; ep.ldc = 3 * W; ep.bias = b.bqkv;
    EMU_CHECK_RC(gemm_bf16(y, W, b.wqkv, W, (int)M, 3 * W, W, ep, st));
    AttnArgs a;
    a.q = qkv; a.k = qkv + W; a.v = qkv + 2 * W;
    a.q_bs = a.k_bs = a.v_bs = (long)N * 3 * W;
    a.q_ts = a.k_ts = a.v_ts = 3 * W;
    a.q_hs = a.k_hs = a.v_hs = D;
    a.out = att; a.o_bs = (long)N * W; a.o_ts = W; a.o_hs = D;
    a.B = B; a.H = Hh; a.Nq = N; a.Nk = N; a.D = D; a.scale = scale; a.causal = 0;
    EMU_CHECK_RC(attn_prefill(a, st));
    GemmEpilogue ep2;
    ep2.C = x; ep2.ldc = W; ep2.bias = b.bo; ep2.residual = x; ep2.ldr = W;  // x = x + out_proj(attn(LN1 x))
    EMU_CHECK_RC(gemm_bf16(att, W, b.wo, W, (int)M, W, W, ep2, st));
    EMU_CHECK_RC(layernorm(x, b.ln2w, b.ln2b, nullptr, y, (int)M, W, c.ln_eps, st));
    GemmEpilogue ep3;
    ep3.C = mlp; ep3.ldc = c.mlp; ep3.bias = b.b1; ep3.mode = EPI_QUICK_GELU;
    EMU_CHECK_RC(gemm_bf16(y, W, b.w1, W, (int)M, c.mlp, W, ep3, st));
    GemmEpilogue ep4;
    ep4.C = x; ep4.ldc = W; ep4.bias = b.b2; ep4.residual = x; ep4.ldr = W;  // x = x + fc2(quick_gelu(fc1(LN2 x)))
    EMU_CHECK_RC(gemm_bf16(mlp, c.mlp, b.w2, c.mlp, (int)M, W, c.mlp, ep4, st));
    count_launch(7);
  }
  // pooled = post_layernorm(x[:, 0]) (every row is normalised; the projection reads the CLS rows at a row stride of N * W)
  EMU_CHECK_RC(layernorm(x, m->post_w, m->post_b, nullptr, y, (int)M, W, c.ln_eps, st));
  GemmEpilogue ep;
  ep.C = out; ep.ldc = c.proj_dim;
  EMU_CHECK_RC(gemm_bf16(y, N * W, m->proj, W, B, c.proj_dim, W, ep, st));
  count_launch(2);
  return EMU_OK;
}

// ---- the head: one CTA per image ----
// diffusers cosine_distance(image_embeds, E) = normalize(image_embeds) @ normalize(E).T, in bf16: the L2 norm accumulates in
// fp32 and is rounded to bf16, every x / norm is rounded to bf16, the dot products accumulate in fp32 and are rounded to bf16,
// and the pipeline reads them back with .float().  Then, per image, in order:
//   adjustment = 0; for j in special-care: s = cos - threshold_j + adjustment; if round(s, 3) > 0: adjustment = 0.01
//   (the new value applies to the later special-care concepts too); for j in concepts: s likewise, round(s, 3) > 0 = bad
// s is formed in double from the bf16 values (which double holds exactly), as numpy does with the thresholds' .item().
// round(s, 3) > 0 is numpy's round-half-even rint(s * 1000) / 1000 > 0, i.e. fl64(s * 1000) > 0.5.  (NumPy 1 evaluates
// cos - threshold in double, NumPy 2 in float32; the two can only disagree exactly at that boundary.)
__global__ void __launch_bounds__(256) safety_score_kernel(const bf16* __restrict__ emb, const bf16* __restrict__ special,
                                                           const bf16* __restrict__ concepts, const bf16* __restrict__ sw,
                                                           const bf16* __restrict__ cw, int P, int S, int Cn, int32_t* flags,
                                                           float* scores, uint8_t* images, long img_bytes) {
  extern __shared__ float xs[];  // [P] normalised image embedding
  __shared__ float red[33];
  __shared__ float cosv[kMaxConcepts];
  __shared__ int flag;
  const int b = blockIdx.x;
  const bf16* x = emb + (long)b * P;
  float ss = 0.f;
  for (int k = threadIdx.x; k < P; k += blockDim.x) {
    const float v = __bfloat162float(x[k]);
    ss += v * v;
  }
  float nx = round_bf16(sqrtf(block_sum(ss, red)));
  nx = fmaxf(nx, 1e-12f);  // F.normalize's clamp_min(eps)
  for (int k = threadIdx.x; k < P; k += blockDim.x) xs[k] = round_bf16(__fdiv_rn(__bfloat162float(x[k]), nx));
  for (int j = 0; j < S + Cn; ++j) {
    const bf16* e = j < S ? special + (long)j * P : concepts + (long)(j - S) * P;
    float es = 0.f;
    for (int k = threadIdx.x; k < P; k += blockDim.x) {
      const float v = __bfloat162float(e[k]);
      es += v * v;
    }
    const float ne = fmaxf(round_bf16(sqrtf(block_sum(es, red))), 1e-12f);
    float dot = 0.f;
    for (int k = threadIdx.x; k < P; k += blockDim.x) dot += xs[k] * round_bf16(__fdiv_rn(__bfloat162float(e[k]), ne));
    const float cs = round_bf16(block_sum(dot, red));
    if (threadIdx.x == 0) cosv[j] = cs;
  }
  if (threadIdx.x == 0) {
    double adj = 0.0;
    int bad = 0;
    for (int j = 0; j < S + Cn; ++j) {
      const double thr = (double)__bfloat162float(j < S ? sw[j] : cw[j - S]);
      const double s = __dadd_rn(__dsub_rn((double)cosv[j], thr), adj);
      const bool hit = __dmul_rn(s, 1000.0) > 0.5;
      if (j < S) {
        if (hit) adj = 0.01;
      } else if (hit) {
        bad = 1;
      }
      if (scores) scores[(long)b * (S + Cn) + j] = (float)s;
    }
    flags[b] = bad;
    flag = bad;
  }
  __syncthreads();
  if (!flag) return;
  // black out: images[idx] = np.zeros(...)
  uint8_t* img = images + b * img_bytes;
  const long head = (16 - ((uintptr_t)img & 15)) & 15;
  const long pre = head < img_bytes ? head : img_bytes;
  for (long i = threadIdx.x; i < pre; i += blockDim.x) img[i] = 0;
  const long n16 = (img_bytes - pre) / 16;
  uint4* v = reinterpret_cast<uint4*>(img + pre);
  for (long i = threadIdx.x; i < n16; i += blockDim.x) v[i] = make_uint4(0, 0, 0, 0);
  for (long i = pre + n16 * 16 + threadIdx.x; i < img_bytes; i += blockDim.x) img[i] = 0;
}

}  // namespace emu

using namespace emu;

extern "C" int emu_safety_configure(EmuEngine* e, const EmuSafetyConfig* cfg) {
  if (!e || !cfg) return EMU_ERR_INVALID;
  const EmuSafetyConfig& c = *cfg;
  if (c.image_size < 1 || c.patch_size < 1 || c.image_size % c.patch_size || c.width < 8 || c.width % 8 || c.layers < 1 ||
      c.heads < 1 || c.width % c.heads || (c.width / c.heads) % 8 || c.mlp < 8 || c.mlp % 8 || c.proj_dim < 8 ||
      c.proj_dim % 8 || c.n_special < 0 || c.n_concepts < 1 || c.n_special + c.n_concepts > kMaxConcepts ||
      !(c.ln_eps > 0.f) || c.resize_shortest_edge < c.crop_size || c.crop_size != c.image_size)
    return e->fail(EMU_ERR_INVALID, "safety checker config out of range");
  for (int i = 0; i < 3; ++i)
    if (!(c.image_std[i] > 0.f)) return e->fail(EMU_ERR_INVALID, "safety checker config: image_std must be positive");
  if (e->safety) {
    cudaDeviceSynchronize();  // the old weights may still be read by queued work
    safety_destroy(e->safety);
    e->safety = nullptr;
  }
  SafetyModel* m = new SafetyModel();
  m->cfg = c;
  m->kpad = (3 * c.patch_size * c.patch_size + 7) / 8 * 8;
  m->blocks.resize(c.layers);
  e->safety = m;
  return EMU_OK;
}

extern "C" int emu_safety_embed(EmuEngine* e, const void* pixel_values, int B, void* image_embeds, emu_stream_t stream) {
  if (!e || !pixel_values || !image_embeds || B < 1) return EMU_ERR_INVALID;
  EMU_CHECK_RC(safety_ready(e));
  return safety_tower(e, (const bf16*)pixel_values, B, (bf16*)image_embeds, (cudaStream_t)stream);
}

extern "C" int emu_safety_check(EmuEngine* e, uint8_t* images, int B, int H, int W, int32_t* flags, float* scores,
                                emu_stream_t stream) {
  if (!e || !images || !flags || B < 1 || H < 1 || W < 1) return EMU_ERR_INVALID;
  EMU_CHECK_RC(safety_ready(e));
  SafetyModel* m = e->safety;
  const EmuSafetyConfig& c = m->cfg;
  cudaStream_t st = (cudaStream_t)stream;
  auto it = m->tables.find({H, W});
  if (it == m->tables.end()) {
    ClipTables t;
    if (clip_plan(H, W, c.resize_shortest_edge, c.crop_size, &t.plan) != EMU_OK)
      return e->fail(EMU_ERR_INVALID, "image too small for the feature extractor");
    const size_t bytes = t.plan.tab.size() * sizeof(int);
    if (cudaMallocHost((void**)&t.host, bytes) != cudaSuccess) { cudaGetLastError(); return e->fail(EMU_ERR_NOMEM, "pinned alloc failed"); }
    memcpy(t.host, t.plan.tab.data(), bytes);
    if (cudaMalloc((void**)&t.dev, bytes) != cudaSuccess) {
      cudaGetLastError();
      cudaFreeHost(t.host);
      return e->fail(EMU_ERR_NOMEM, "coefficient table alloc failed");
    }
    m->owned.push_back(t.dev);
    if (cudaMemcpyAsync(t.dev, t.host, bytes, cudaMemcpyHostToDevice, st) != cudaSuccess) {
      cudaFreeHost(t.host);
      return e->fail(EMU_ERR_CUDA, "coefficient table upload failed");
    }
    it = m->tables.emplace(std::make_pair(H, W), t).first;
  }
  const ClipTables& t = it->second;
  const int S = c.crop_size;
  int rc;
  if ((rc = m->ensure(m->pix, (size_t)B * 3 * S * S * 2)) || (rc = m->ensure(m->tmp, clip_tmp_bytes(t.plan, B) + 16)) ||
      (rc = m->ensure(m->emb, (size_t)B * c.proj_dim * 2)))
    return e->fail(rc, "safety checker workspace alloc failed");
  // CLIPImageProcessor -> pixel_values.to(bf16)
  if (clip_launch(t.plan, t.dev, images, B, (uint8_t*)m->tmp.p, m->pix.p, c.image_mean, c.image_std, 1, st) != EMU_OK)
    return e->fail(EMU_ERR_CUDA, "feature extractor launch failed");
  EMU_CHECK_RC(safety_tower(e, (const bf16*)m->pix.p, B, (bf16*)m->emb.p, st));
  safety_score_kernel<<<B, 256, c.proj_dim * sizeof(float), st>>>((const bf16*)m->emb.p, m->special, m->concepts, m->special_w,
                                                                  m->concept_w, c.proj_dim, c.n_special, c.n_concepts, flags,
                                                                  scores, images, (long)H * W * 3);
  count_launch();
  return cudaGetLastError() == cudaSuccess ? EMU_OK : e->fail(EMU_ERR_CUDA, "safety score launch failed");
}
