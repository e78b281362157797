// emu_b200 — engine: weight ingestion/packing, EVA ViT forward, LLaMA prefill + CUDA-graphed decode step.
//
// Orchestrates the kernels of gemm_tc.cu / gemv.cu / attention.cu / elementwise.cu into the reference's
// module boundaries (SURVEY.md §8a rows a1-a12):
//   ViT      : Emu2/emu/eva_vit.py:402-431 (post-norm) and Emu1/models/eva_vit_model.py:636-665 (pre-norm)
//   LLaMA    : HF LlamaModel.forward as driven by Emu2/emu/emu.py:133-138 (prefill, hidden_states[-1]) and
//              :213-229 (generate: prefill + one-token steps with KV cache)
#include "engine.h"

#include <dlfcn.h>
#include <math.h>
#include <stdlib.h>
#include <string.h>

#include "common.cuh"

namespace emu {

unsigned long long g_launches = 0;

#define EMU_TRY(x)            \
  do {                        \
    int rc_ = (x);            \
    if (rc_ != EMU_OK) return rc_; \
  } while (0)

// ----------------------------------------------------------------------------------------------
// packing kernels
// ----------------------------------------------------------------------------------------------
// dst[(dst_row_off + r*dst_row_stride) * dst_ld + c] = src[map(r) * src_ld + col_off + c]
// map: mode 0 -> row_off + r ; mode 1 -> RoPE pair interleave inside heads of size D
__global__ void pack_rows_kernel(bf16* dst, const bf16* __restrict__ src, long rows, int cols, long src_ld, long dst_ld,
                                 long row_off, int col_off, int mode, int D, long dst_row_off, int dst_row_stride) {
  const long total = rows * cols;
  for (long idx = blockIdx.x * (long)blockDim.x + threadIdx.x; idx < total; idx += (long)gridDim.x * blockDim.x) {
    const long r = idx / cols;
    const int c = idx % cols;
    long sr;
    if (mode == 0) sr = row_off + r;
    else {
      const long head = r / D;
      const int i = r % D;
      sr = row_off + head * D + (i >> 1) + (i & 1) * (D >> 1);
    }
    dst[(dst_row_off + r * dst_row_stride) * dst_ld + c] = src[sr * src_ld + col_off + c];
  }
}
static int pack_rows(bf16* dst, const bf16* src, long rows, int cols, long src_ld, long dst_ld, long row_off, int col_off,
                     int mode, int D, long dst_row_off, int dst_row_stride, cudaStream_t st) {
  pack_rows_kernel<<<8 * kNumSMs, 256, 0, st>>>(dst, src, rows, cols, src_ld, dst_ld, row_off, col_off, mode, D,
                                                dst_row_off, dst_row_stride);
  count_launch();
  return cudaGetLastError() == cudaSuccess ? EMU_OK : EMU_ERR_CUDA;
}

__global__ void cvt_f32_bf16_kernel(const float* __restrict__ s, bf16* d, size_t n) {
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
    d[i] = __float2bfloat16_rn(s[i]);
}
__global__ void cvt_f16_bf16_kernel(const __half* __restrict__ s, bf16* d, size_t n) {
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
    d[i] = __float2bfloat16_rn(__half2float(s[i]));
}
__global__ void fill_zero_kernel(bf16* d, size_t n) {
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
    d[i] = __float2bfloat16(0.f);
}
__global__ void rope_table_kernel(bf16* cos_t, bf16* sin_t, int max_pos, int half, float theta) {
  // HF LlamaRotaryEmbedding: inv_freq = 1/theta^(2j/D) (fp32), freqs = pos * inv_freq (fp32), cos/sin -> bf16
  const long total = (long)max_pos * half;
  for (long idx = blockIdx.x * (long)blockDim.x + threadIdx.x; idx < total; idx += (long)gridDim.x * blockDim.x) {
    const int j = idx % half;
    const int p = idx / half;
    const float inv_freq = 1.0f / powf(theta, (float)(2 * j) / (float)(2 * half));
    const float ang = (float)p * inv_freq;
    cos_t[idx] = __float2bfloat16_rn(cosf(ang));
    sin_t[idx] = __float2bfloat16_rn(sinf(ang));
  }
}
__global__ void set_int_kernel(int* p, int n, int v) {
  if (threadIdx.x < n) p[threadIdx.x] = v;
}
__global__ void advance_pos_kernel(int* p, int n, unsigned* tp_step) {
  if (threadIdx.x < n) p[threadIdx.x] += 1;
  if (tp_step && threadIdx.x == 0) *tp_step += 1;  // decode-step counter behind the tensor-parallel exchange flags
}
// start[b] = number of leading zeros in mask row b; posoff[b] = hf ? start[b] : 0
__global__ void mask_start_kernel(const int* __restrict__ mask, int N, int* start, int* posoff, int hf, int base) {
  const int b = blockIdx.x;
  if (threadIdx.x == 0) {
    int s = 0;
    while (s < N && mask[(long)b * N + s] == 0) ++s;
    start[b] = base + s;
    posoff[b] = hf ? base + s : 0;
  }
}
__global__ void argmax_ban_kernel(float* logits, int cols, int ban) {
  if (ban >= 0 && ban < cols) logits[(long)blockIdx.x * cols + ban] = -INFINITY;
}

int to_bf16_device(EmuEngine* e, const void* src, int dtype, size_t n, bf16** out, bool* temp, cudaStream_t st) {
  cudaPointerAttributes attr;
  bool on_device = false;
  if (cudaPointerGetAttributes(&attr, src) == cudaSuccess)
    on_device = (attr.type == cudaMemoryTypeDevice || attr.type == cudaMemoryTypeManaged);
  else
    cudaGetLastError();
  const size_t esz = dtype == EMU_DTYPE_F32 ? 4 : 2;
  const void* dsrc = src;
  void* staged = nullptr;
  if (!on_device) {
    if (cudaMalloc(&staged, n * esz) != cudaSuccess) return e->fail(EMU_ERR_NOMEM, "staging alloc failed");
    if (cudaMemcpyAsync(staged, src, n * esz, cudaMemcpyHostToDevice, st) != cudaSuccess) {
      cudaFree(staged);
      return e->fail(EMU_ERR_CUDA, "H2D copy failed");
    }
    dsrc = staged;
  }
  if (dtype == EMU_DTYPE_BF16) {
    *out = (bf16*)dsrc;
    *temp = staged != nullptr;
    return EMU_OK;
  }
  bf16* conv = nullptr;
  if (cudaMalloc((void**)&conv, n * 2) != cudaSuccess) {
    if (staged) cudaFree(staged);
    return e->fail(EMU_ERR_NOMEM, "convert alloc failed");
  }
  if (dtype == EMU_DTYPE_F32) cvt_f32_bf16_kernel<<<4 * kNumSMs, 256, 0, st>>>((const float*)dsrc, conv, n);
  else cvt_f16_bf16_kernel<<<4 * kNumSMs, 256, 0, st>>>((const __half*)dsrc, conv, n);
  count_launch();
  if (staged) {
    cudaStreamSynchronize(st);
    cudaFree(staged);
  }
  *out = conv;
  *temp = true;
  return EMU_OK;
}

// ----------------------------------------------------------------------------------------------
// NCCL (resolved lazily from the torch-bundled libnccl.so.2; only touched when tp_size > 1)
// ----------------------------------------------------------------------------------------------
struct NcclUid {
  char b[128];  // ncclUniqueId is passed BY VALUE to ncclCommInitRank
};
struct NcclApi {
  void* h = nullptr;
  int (*GetUniqueId)(void*) = nullptr;
  int (*CommInitRank)(void**, int, NcclUid, int) = nullptr;
  int (*AllReduce)(const void*, void*, size_t, int, int, void*, cudaStream_t) = nullptr;
  int (*AllGather)(const void*, void*, size_t, int, void*, cudaStream_t) = nullptr;
  int (*CommDestroy)(void*) = nullptr;
};
static NcclApi g_nccl;
static bool nccl_load() {
  if (g_nccl.h) return true;
  void* h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_GLOBAL);
  if (!h) return false;
  g_nccl.GetUniqueId = (int (*)(void*))dlsym(h, "ncclGetUniqueId");
  *(void**)(&g_nccl.CommInitRank) = dlsym(h, "ncclCommInitRank");
  *(void**)(&g_nccl.AllReduce) = dlsym(h, "ncclAllReduce");
  *(void**)(&g_nccl.CommDestroy) = dlsym(h, "ncclCommDestroy");
  *(void**)(&g_nccl.AllGather) = dlsym(h, "ncclAllGather");
  if (!g_nccl.GetUniqueId || !g_nccl.CommInitRank || !g_nccl.AllReduce || !g_nccl.AllGather) return false;
  g_nccl.h = h;
  return true;
}
int nccl_allreduce_bf16(EmuEngine* e, bf16* buf, size_t n, cudaStream_t st) {
  if (e->tp_size == 1) return EMU_OK;
  // ncclBfloat16 = 9, ncclSum = 0
  if (g_nccl.AllReduce(buf, buf, n, 9, 0, e->nccl_comm, st) != 0) return e->fail(EMU_ERR_NCCL, "ncclAllReduce failed");
  return EMU_OK;
}

// host-buffer helpers used once at engine creation to swap CUDA IPC handles (tp_exchange.cu)
static int nccl_allgather_bytes(EmuEngine* e, const void* src, void* dst, size_t bytes) {
  char* d = nullptr;
  if (cudaMalloc((void**)&d, bytes * (e->tp_size + 1)) != cudaSuccess) return EMU_ERR_NOMEM;
  int rc = EMU_OK;
  if (cudaMemcpy(d, src, bytes, cudaMemcpyHostToDevice) != cudaSuccess) rc = EMU_ERR_CUDA;
  // ncclInt8 = 0
  if (!rc && g_nccl.AllGather(d, d + bytes, bytes, 0, e->nccl_comm, nullptr) != 0) rc = EMU_ERR_NCCL;
  if (!rc && cudaDeviceSynchronize() != cudaSuccess) rc = EMU_ERR_CUDA;
  if (!rc && cudaMemcpy(dst, d + bytes, bytes * e->tp_size, cudaMemcpyDeviceToHost) != cudaSuccess) rc = EMU_ERR_CUDA;
  cudaFree(d);
  return rc;
}
static int nccl_allreduce_min_int(EmuEngine* e, int* v) {
  int* d = nullptr;
  if (cudaMalloc((void**)&d, sizeof(int)) != cudaSuccess) return EMU_ERR_NOMEM;
  int rc = EMU_OK;
  if (cudaMemcpy(d, v, sizeof(int), cudaMemcpyHostToDevice) != cudaSuccess) rc = EMU_ERR_CUDA;
  // ncclInt32 = 2, ncclMin = 3
  if (!rc && g_nccl.AllReduce(d, d, 1, 2, 3, e->nccl_comm, nullptr) != 0) rc = EMU_ERR_NCCL;
  if (!rc && cudaDeviceSynchronize() != cudaSuccess) rc = EMU_ERR_CUDA;
  if (!rc && cudaMemcpy(v, d, sizeof(int), cudaMemcpyDeviceToHost) != cudaSuccess) rc = EMU_ERR_CUDA;
  cudaFree(d);
  return rc;
}
int tp_setup(EmuEngine* e) { return tp_exchange_setup(e, nccl_allgather_bytes, nccl_allreduce_min_int); }
int engine_allgather_bytes(EmuEngine* e, const void* src, void* dst, size_t bytes) { return nccl_allgather_bytes(e, src, dst, bytes); }
int engine_allreduce_min_int(EmuEngine* e, int* v) { return nccl_allreduce_min_int(e, v); }

// vocab-sharded logits: local [B, Vl] fp32 -> all ranks' shards [tp][B][Vl] -> logits [B, V]
__global__ void logits_unshard_kernel(const float* __restrict__ g, float* out, int tp, int B, int Vl, int V) {
  const long total = (long)tp * B * Vl;
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const int v = i % Vl;
    const int b = (i / Vl) % B;
    const int r = i / ((long)Vl * B);
    const long col = (long)r * Vl + v;
    if (col < V) out[(long)b * V + col] = g[i];  // rows past V are the zero padding of the last shard
  }
}
int gather_logits(EmuEngine* e, const float* local, float* gathered, float* out, int B, cudaStream_t st) {
  // ncclFloat32 = 7
  if (g_nccl.AllGather(local, gathered, (size_t)B * e->Vl, 7, e->nccl_comm, st) != 0) return e->fail(EMU_ERR_NCCL, "ncclAllGather failed");
  logits_unshard_kernel<<<2 * kNumSMs, 256, 0, st>>>(gathered, out, e->tp_size, B, e->Vl, e->cfg.llm_vocab);
  return cudaGetLastError() == cudaSuccess ? EMU_OK : EMU_ERR_CUDA;
}

}  // namespace emu

using namespace emu;

void* EmuEngine::dmalloc(size_t bytes) {
  void* p = nullptr;
  if (cudaMalloc(&p, bytes ? bytes : 16) != cudaSuccess) {
    cudaGetLastError();
    return nullptr;
  }
  owned.push_back(p);
  return p;
}
int EmuEngine::ensure(DevBuf& b, size_t bytes) {
  if (b.bytes >= bytes) return EMU_OK;
  // growing a workspace invalidates graphs that baked the old pointer
  void* p = dmalloc(bytes);
  if (!p) return fail(EMU_ERR_NOMEM, "workspace alloc failed");
  b.p = p;
  b.bytes = bytes;
  return EMU_OK;
}

// ================================================================================================
// life cycle
// ================================================================================================
extern "C" int emu_tp_head_range(int n_heads, int tp_size, int tp_rank, int* start, int* count) {
  if (n_heads < 1 || tp_size < 1 || tp_rank < 0 || tp_rank >= tp_size || !start || !count) return EMU_ERR_INVALID;
  const int base = n_heads / tp_size, rem = n_heads % tp_size;
  *count = base + (tp_rank < rem ? 1 : 0);
  *start = tp_rank * base + (tp_rank < rem ? tp_rank : rem);
  return EMU_OK;
}

extern "C" int emu_nccl_unique_id(void* out128) {
  if (!nccl_load()) return EMU_ERR_NCCL;
  return g_nccl.GetUniqueId(out128) == 0 ? EMU_OK : EMU_ERR_NCCL;
}

extern "C" int emu_engine_create(const EmuConfig* cfg, int tp_rank, int tp_size, const void* uid, EmuEngine** out) {
  if (!cfg || !out || tp_size < 1 || tp_rank < 0 || tp_rank >= tp_size) return EMU_ERR_INVALID;
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) {
    cudaGetLastError();
    return EMU_ERR_CUDA;  // no CPU fallback
  }
  if (gemv_init() != EMU_OK) return EMU_ERR_NOMEM;
  EmuEngine* e = new EmuEngine();
  e->cfg = *cfg;
  e->tp_rank = tp_rank;
  e->tp_size = tp_size;
  const EmuConfig& c = e->cfg;
  if (c.llm_layers > 0) {
    if (c.llm_ffn % tp_size || c.llm_max_batch < 1 ||
        c.llm_max_batch > kLlmMaxRows || c.llm_hidden % 32 || c.llm_ffn % (32 * tp_size) || (c.llm_head_dim != 64 && c.llm_head_dim != 128)) {
      delete e;
      return EMU_ERR_UNSUPPORTED;
    }
    // heads need not divide the TP degree (Emu2: 52 heads on 8 GPUs): every rank allocates ceil(H/tp) head slots,
    // ranks past the remainder own one fewer real head and keep a zero-weight slot (exact: a zero head adds zero)
    e->Hl = (c.llm_heads + tp_size - 1) / tp_size;
    emu_tp_head_range(c.llm_heads, tp_size, tp_rank, &e->head_start, &e->head_count);
    e->Fl = c.llm_ffn / tp_size;
    // the vocabulary need not divide the TP degree either (Emu2-Chat: 32274, Emu1: 32004): every rank holds ceil(V/tp)
    // lm_head rows, rows past V are zero and are dropped when the shards are gathered
    e->Vl = (c.llm_vocab + tp_size - 1) / tp_size;
    e->layers.resize(c.llm_layers);
    const int half = c.llm_head_dim / 2;
    const int max_pos = c.llm_max_seq + 8;
    e->rope_cos = (bf16*)e->dmalloc((size_t)max_pos * half * 2);
    e->rope_sin = (bf16*)e->dmalloc((size_t)max_pos * half * 2);
    const size_t kv_elems = (size_t)c.llm_layers * 2 * c.llm_max_batch * e->Hl * c.llm_max_seq * c.llm_head_dim;
    e->kv = (bf16*)e->dmalloc(kv_elems * 2);
    e->d_pos = (int*)e->dmalloc(3 * kLlmMaxRows * sizeof(int));
    e->d_start = e->d_pos + kLlmMaxRows;
    e->d_posoff = e->d_pos + 2 * kLlmMaxRows;
    if (c.llm_max_batch > 8) {  // wide decode (more than 8 cache rows: the C4 workload, 4 prompts x 5 beams) runs on the GEMM path
      e->dec_xn = (bf16*)e->dmalloc((size_t)c.llm_max_batch * c.llm_hidden * 2);
      e->dec_qkv = (bf16*)e->dmalloc((size_t)c.llm_max_batch * 3 * e->Hl * c.llm_head_dim * 2);
      e->sk_ws = (float*)e->dmalloc(gemm_skinny_workspace_bytes());
      e->sk_counters = (int*)e->dmalloc(kSkinnyMaxTiles * sizeof(int));
      if (!e->dec_xn || !e->dec_qkv || !e->sk_ws || !e->sk_counters || gemm_skinny_init() != EMU_OK) {
        emu_engine_destroy(e);
        return EMU_ERR_NOMEM;
      }
      cudaMemset(e->sk_counters, 0, kSkinnyMaxTiles * sizeof(int));
      const char* wsk = getenv("EMU_WIDE_SKINNY");
      e->wide_skinny = !(wsk && wsk[0] == '0');
    }
    const int Bm = c.llm_max_batch;
    e->dec_h = (bf16*)e->dmalloc((size_t)Bm * c.llm_hidden * 2);
    e->dec_q = (bf16*)e->dmalloc((size_t)Bm * e->Hl * c.llm_head_dim * 2);
    e->dec_attn = (bf16*)e->dmalloc((size_t)Bm * e->Hl * c.llm_head_dim * 2);
    e->dec_act = (bf16*)e->dmalloc((size_t)Bm * e->Fl * 2);
    e->dec_tmp = (bf16*)e->dmalloc((size_t)Bm * c.llm_hidden * 2);
    e->dec_attn_ws = (float*)e->dmalloc(attn_decode_workspace_bytes(Bm, e->Hl, c.llm_head_dim));
    e->dec_counters = (int*)e->dmalloc((size_t)Bm * e->Hl * sizeof(int));
    e->kv_indir = (int*)e->dmalloc((size_t)Bm * c.llm_max_seq * sizeof(int));
    {
      const char* kc = getenv("EMU_KV_COPY");
      e->kv_copy = kc && kc[0] == '1';
    }
    e->dec_logits_local = (float*)e->dmalloc((size_t)Bm * c.llm_vocab * sizeof(float));
    e->dec_logits_shard = (float*)e->dmalloc(((size_t)Bm * e->Vl + 4) * sizeof(float));
    e->dec_part = (float*)e->dmalloc((size_t)Bm * c.llm_hidden * sizeof(float));
    e->dec_logits_gather = (float*)e->dmalloc((size_t)Bm * e->Vl * tp_size * sizeof(float));
    if (!e->rope_cos || !e->rope_sin || !e->kv || !e->d_pos || !e->dec_h || !e->dec_q || !e->dec_attn || !e->dec_act ||
        !e->dec_tmp || !e->dec_attn_ws || !e->dec_counters || !e->dec_logits_local || !e->kv_indir) {
      emu_engine_destroy(e);
      return EMU_ERR_NOMEM;
    }
    rope_table_kernel<<<2 * kNumSMs, 256>>>(e->rope_cos, e->rope_sin, max_pos, half, c.llm_rope_theta);
    cudaMemset(e->dec_counters, 0, (size_t)Bm * e->Hl * sizeof(int));
    cudaMemset(e->d_pos, 0, 3 * kLlmMaxRows * sizeof(int));
    kv_indir_identity(e->kv_indir, Bm, c.llm_max_seq, 0);
  }
  if (c.vit_layers > 0) {
    if (c.vit_width % c.vit_heads || c.vit_image % c.vit_patch || c.vit_width % 8) {
      emu_engine_destroy(e);
      return EMU_ERR_UNSUPPORTED;
    }
    e->vit.resize(c.vit_layers);
    e->vit_kpad = (3 * c.vit_patch * c.vit_patch + 7) / 8 * 8;
  }
  if (tp_size > 1) {
    if (!uid || !nccl_load()) {
      emu_engine_destroy(e);
      return EMU_ERR_NCCL;
    }
    NcclUid u;
    memcpy(u.b, uid, 128);
    if (g_nccl.CommInitRank(&e->nccl_comm, tp_size, u, tp_rank) != 0) {
      emu_engine_destroy(e);
      return EMU_ERR_NCCL;
    }
    if (c.llm_layers > 0 && emu::tp_setup(e) != EMU_OK) {
      emu_engine_destroy(e);
      return EMU_ERR_NCCL;
    }
  }
  if (cudaDeviceSynchronize() != cudaSuccess) {
    emu_engine_destroy(e);
    return EMU_ERR_CUDA;
  }
  *out = e;
  return EMU_OK;
}

extern "C" void emu_engine_destroy(EmuEngine* e) {
  if (!e) return;
  cudaDeviceSynchronize();
  for (auto& g : e->graphs) cudaGraphExecDestroy(g.second);
  if (e->cap_stream) cudaStreamDestroy(e->cap_stream);
  if (e->unet) unet_destroy(e->unet);
  if (e->vae) vae_destroy(e->vae);
  if (e->cformer) cformer_destroy(e->cformer);
  for (void* p : e->owned) cudaFree(p);
  tp_exchange_teardown(e);
  if (e->nccl_comm && g_nccl.CommDestroy) g_nccl.CommDestroy(e->nccl_comm);
  delete e;
}

extern "C" const char* emu_last_error(EmuEngine* e) { return e ? e->err.c_str() : "null engine"; }
extern "C" uint64_t emu_launch_count(void) { return g_launches; }
extern "C" const char* emu_version(void) { return "emu_b200 0.1 (sm_90a)"; }

// ================================================================================================
// weight ingestion
// ================================================================================================
static bool starts_with(const std::string& s, const char* p) { return s.compare(0, strlen(p), p) == 0; }
static bool ends_with(const std::string& s, const char* p) {
  const size_t n = strlen(p);
  return s.size() >= n && s.compare(s.size() - n, n, p) == 0;
}
static long numel(const int64_t* shape, int ndim) {
  long n = 1;
  for (int i = 0; i < ndim; ++i) n *= shape[i];
  return n;
}

static int alloc_copy(EmuEngine* e, bf16** dst, const bf16* src, size_t n, cudaStream_t st) {
  if (!*dst) *dst = (bf16*)e->dmalloc(n * 2);
  if (!*dst) return e->fail(EMU_ERR_NOMEM, "weight alloc failed");
  if (cudaMemcpyAsync(*dst, src, n * 2, cudaMemcpyDeviceToDevice, st) != cudaSuccess)
    return e->fail(EMU_ERR_CUDA, "weight copy failed");
  return EMU_OK;
}
static int alloc_zero(EmuEngine* e, bf16** dst, size_t n, cudaStream_t st) {
  if (*dst) return EMU_OK;
  *dst = (bf16*)e->dmalloc(n * 2);
  if (!*dst) return e->fail(EMU_ERR_NOMEM, "weight alloc failed");
  fill_zero_kernel<<<4 * kNumSMs, 256, 0, st>>>(*dst, n);
  return EMU_OK;
}

static int load_llm(EmuEngine* e, const std::string& key, const bf16* src, const int64_t* shape, int ndim,
                    cudaStream_t st) {
  const EmuConfig& c = e->cfg;
  const int Hd = c.llm_hidden, D = c.llm_head_dim, Hl = e->Hl, Fl = e->Fl;
  const long n = numel(shape, ndim);
  if (key == "decoder.lm.model.embed_tokens.weight") {
    if (n != (long)c.llm_vocab * Hd) return e->fail(EMU_ERR_INVALID, "embed_tokens shape");
    return alloc_copy(e, &e->embed, src, n, st);
  }
  if (key == "decoder.lm.model.norm.weight") {
    if (n != Hd) return e->fail(EMU_ERR_INVALID, "final norm shape");
    return alloc_copy(e, &e->final_norm, src, Hd, st);
  }
  if (key == "decoder.lm.lm_head.weight") {
    if (n != (long)c.llm_vocab * Hd) return e->fail(EMU_ERR_INVALID, "lm_head shape");
    EMU_TRY(alloc_zero(e, &e->lm_head, (size_t)e->Vl * Hd, st));
    const long row0 = (long)e->tp_rank * e->Vl;
    const long rows = row0 >= c.llm_vocab ? 0 : (row0 + e->Vl <= c.llm_vocab ? e->Vl : c.llm_vocab - row0);
    if (rows == 0) return EMU_OK;
    return pack_rows(e->lm_head, src, rows, Hd, Hd, Hd, row0, 0, 0, D, 0, 1, st);
  }
  if (key == "decoder.lm.stu_regress_head.weight") {
    if (ndim != 2) return e->fail(EMU_ERR_INVALID, "stu_regress_head shape");
    e->stu_out = (int)shape[0];
    e->stu_in = (int)shape[1];
    return alloc_copy(e, &e->stu_head, src, n, st);
  }
  const char* pre = "decoder.lm.model.layers.";
  if (!starts_with(key, pre)) return e->fail(EMU_ERR_INVALID, "unknown llm key " + key);
  const size_t p0 = strlen(pre);
  const size_t p1 = key.find('.', p0);
  const int li = atoi(key.substr(p0, p1 - p0).c_str());
  if (li < 0 || li >= c.llm_layers) return e->fail(EMU_ERR_INVALID, "layer index out of range: " + key);
  const std::string sub = key.substr(p1 + 1);
  LlmLayer& L = e->layers[li];
  if (sub == "input_layernorm.weight" || sub == "post_attention_layernorm.weight") {
    if (n != Hd) return e->fail(EMU_ERR_INVALID, "norm shape " + key);
    const bool first = sub[0] == 'i';
    L.loaded |= first ? 128u : 256u;
    return alloc_copy(e, first ? &L.ln1 : &L.ln2, src, Hd, st);
  }
  if (sub == "self_attn.q_proj.weight" || sub == "self_attn.k_proj.weight" || sub == "self_attn.v_proj.weight") {
    if (n != (long)c.llm_heads * D * Hd) return e->fail(EMU_ERR_INVALID, "qkv shape " + key);
    EMU_TRY(alloc_zero(e, &L.wqkv, (size_t)3 * Hl * D * Hd, st));
    const int which = sub[10] == 'q' ? 0 : (sub[10] == 'k' ? 1 : 2);
    L.loaded |= 1u << which;
    // q,k rows are pair-interleaved per head so a RoPE rotation pair is adjacent (see gemv.cu / elementwise.cu)
    return pack_rows(L.wqkv, src, (long)e->head_count * D, Hd, Hd, Hd, (long)e->head_start * D, 0, which < 2 ? 1 : 0, D,
                     (long)which * Hl * D, 1, st);
  }
  if (sub == "self_attn.o_proj.weight") {
    if (n != (long)c.llm_heads * D * Hd) return e->fail(EMU_ERR_INVALID, "o_proj shape " + key);
    L.loaded |= 8u;
    EMU_TRY(alloc_zero(e, &L.wo, (size_t)Hd * Hl * D, st));
    return pack_rows(L.wo, src, Hd, e->head_count * D, (long)c.llm_heads * D, (long)Hl * D, 0, e->head_start * D, 0, D, 0, 1, st);
  }
  if (sub == "mlp.gate_proj.weight" || sub == "mlp.up_proj.weight") {
    if (n != (long)c.llm_ffn * Hd) return e->fail(EMU_ERR_INVALID, "mlp shape " + key);
    if (!L.wgu) L.wgu = (bf16*)e->dmalloc((size_t)2 * Fl * Hd * 2);
    if (!L.wgu) return e->fail(EMU_ERR_NOMEM, "wgu alloc");
    const int which = sub[4] == 'g' ? 0 : 1;
    L.loaded |= 16u << which;
    return pack_rows(L.wgu, src, Fl, Hd, Hd, Hd, (long)e->tp_rank * Fl, 0, 0, D, which, 2, st);
  }
  if (sub == "mlp.down_proj.weight") {
    if (n != (long)c.llm_ffn * Hd) return e->fail(EMU_ERR_INVALID, "mlp shape " + key);
    L.loaded |= 64u;
    if (!L.wdown) L.wdown = (bf16*)e->dmalloc((size_t)Hd * Fl * 2);
    if (!L.wdown) return e->fail(EMU_ERR_NOMEM, "wdown alloc");
    return pack_rows(L.wdown, src, Hd, Fl, c.llm_ffn, Fl, 0, e->tp_rank * Fl, 0, D, 0, 1, st);
  }
  if (ends_with(sub, "rotary_emb.inv_freq")) return EMU_OK;
  return e->fail(EMU_ERR_INVALID, "unknown llm key " + key);
}

static int load_vit(EmuEngine* e, const std::string& key, const bf16* src, const int64_t* shape, int ndim,
                    cudaStream_t st) {
  const EmuConfig& c = e->cfg;
  const int W = c.vit_width;
  const long n = numel(shape, ndim);
  const int G = c.vit_image / c.vit_patch;
  auto sized = [&](long want, bf16** dst) -> int {
    if (n != want) return e->fail(EMU_ERR_INVALID, "shape mismatch for " + key);
    return alloc_copy(e, dst, src, (size_t)want, st);
  };
  if (key == "visual.cls_token") return sized(W, &e->vit_cls);
  if (key == "visual.pos_embed") {
    if (n != (long)(G * G + 1) * W) return e->fail(EMU_ERR_INVALID, "pos_embed shape");
    return alloc_copy(e, &e->vit_pos, src, n, st);
  }
  if (key == "visual.patch_embed.proj.weight") {
    const int kin = 3 * c.vit_patch * c.vit_patch;
    if (n != (long)W * kin) return e->fail(EMU_ERR_INVALID, "patch_embed shape");
    EMU_TRY(alloc_zero(e, &e->vit_wpatch, (size_t)W * e->vit_kpad, st));
    return pack_rows(e->vit_wpatch, src, W, kin, kin, e->vit_kpad, 0, 0, 0, 1, 0, 1, st);
  }
  if (key == "visual.patch_embed.proj.bias") return sized(W, &e->vit_bpatch);
  if (key == "ln_visual.weight") return sized(W, &e->vit_lnf_w);
  if (key == "ln_visual.bias") return sized(W, &e->vit_lnf_b);
  // unused-by-forward_features members of the Emu1 EVA tower (Emu1/models/eva_vit_model.py: head / norm / fc_norm / rope)
  if (starts_with(key, "visual.head.") || starts_with(key, "visual.norm.") || starts_with(key, "visual.fc_norm.") ||
      starts_with(key, "visual.rope."))
    return EMU_OK;
  const char* pre = "visual.blocks.";
  if (!starts_with(key, pre)) return e->fail(EMU_ERR_INVALID, "unknown vit key " + key);
  const size_t p0 = strlen(pre);
  const size_t p1 = key.find('.', p0);
  const int li = atoi(key.substr(p0, p1 - p0).c_str());
  if (li < 0 || li >= c.vit_layers) return e->fail(EMU_ERR_INVALID, "vit block index out of range");
  const std::string sub = key.substr(p1 + 1);
  VitBlock& B = e->vit[li];
  if (sub == "norm1.weight") return sized(W, &B.ln1w);
  if (sub == "norm1.bias") return sized(W, &B.ln1b);
  if (sub == "norm2.weight") return sized(W, &B.ln2w);
  if (sub == "norm2.bias") return sized(W, &B.ln2b);
  if (sub == "attn.qkv.weight") return sized((long)3 * W * W, &B.wqkv);
  if (sub == "attn.q_bias" || sub == "attn.v_bias") {
    // qkv bias = cat(q_bias, zeros, v_bias): K has no bias (Emu2/emu/eva_vit.py:194-196)
    if (n != W) return e->fail(EMU_ERR_INVALID, "shape mismatch for " + key);
    EMU_TRY(alloc_zero(e, &B.bqkv, (size_t)3 * W, st));
    B.bias_loaded |= sub == "attn.q_bias" ? 1u : 2u;
    const size_t off = sub == "attn.q_bias" ? 0 : (size_t)2 * W;
    return cudaMemcpyAsync(B.bqkv + off, src, (size_t)W * 2, cudaMemcpyDeviceToDevice, st) == cudaSuccess
               ? EMU_OK
               : e->fail(EMU_ERR_CUDA, "bias copy");
  }
  if (sub == "attn.proj.weight") return sized((long)W * W, &B.wproj);
  if (sub == "attn.proj.bias") return sized(W, &B.bproj);
  if (sub == "mlp.fc1.weight") return sized((long)c.vit_mlp * W, &B.wfc1);
  if (sub == "mlp.fc1.bias") return sized(c.vit_mlp, &B.bfc1);
  if (sub == "mlp.fc2.weight") return sized((long)c.vit_mlp * W, &B.wfc2);
  if (sub == "mlp.fc2.bias") return sized(W, &B.bfc2);
  if (starts_with(sub, "attn.rope.") || starts_with(sub, "attn.inner_attn_ln.")) return EMU_OK;
  return e->fail(EMU_ERR_INVALID, "unknown vit key " + key);
}

extern "C" int emu_engine_load_tensor(EmuEngine* e, const char* state_dict_key, const void* src, int dtype,
                                      const int64_t* shape, int ndim, emu_stream_t stream) {
  if (!e || !state_dict_key || !src || !shape || ndim < 1) return EMU_ERR_INVALID;
  cudaStream_t st = (cudaStream_t)stream;
  std::string key(state_dict_key);
  if (starts_with(key, "multimodal_encoder.")) key = key.substr(strlen("multimodal_encoder."));
  const long n = numel(shape, ndim);
  bf16* dsrc = nullptr;
  bool temp = false;
  EMU_TRY(to_bf16_device(e, src, dtype, (size_t)n, &dsrc, &temp, st));
  int rc;
  if (starts_with(key, "visual.") || starts_with(key, "ln_visual.")) rc = load_vit(e, key, dsrc, shape, ndim, st);
  else if (starts_with(key, "decoder.")) rc = load_llm(e, key, dsrc, shape, ndim, st);
  else if ((key == "project_up.weight" || key == "project_down.weight") && ndim != 2)
    rc = e->fail(EMU_ERR_INVALID, "projection shape " + key);
  else if (key == "project_up.weight") {
    e->proj_up_out = (int)shape[0];
    e->proj_up_in = (int)shape[1];
    rc = alloc_copy(e, &e->proj_up, dsrc, n, st);
  } else if (key == "project_down.weight") {
    e->proj_down_out = (int)shape[0];
    e->proj_down_in = (int)shape[1];
    rc = alloc_copy(e, &e->proj_down, dsrc, n, st);
  } else if (starts_with(key, "unet.")) rc = unet_load_tensor(e, key.substr(5), dsrc, shape, ndim, st);
  else if (starts_with(key, "vae.")) rc = vae_load_tensor(e, key.substr(4), dsrc, shape, ndim, st);
  else if (starts_with(key, "cformer.")) rc = cformer_load_tensor(e, key.substr(8), dsrc, shape, ndim, st);
  else rc = e->fail(EMU_ERR_INVALID, "unknown state-dict key " + key);
  if (temp) {
    cudaStreamSynchronize(st);
    cudaFree(dsrc);
  }
  return rc;
}

// ================================================================================================
// EVA ViT
// ================================================================================================
extern "C" int emu_vit_forward(EmuEngine* e, const void* image, int B, void* out, int n_query, int pool,
                               emu_stream_t stream) {
  if (!e || !image || !out || B < 1) return EMU_ERR_INVALID;
  const EmuConfig& c = e->cfg;
  if (c.vit_layers < 1) return e->fail(EMU_ERR_STATE, "engine has no ViT");
  cudaStream_t st = (cudaStream_t)stream;
  PdlScope pdl_chain(1);
  const int W = c.vit_width, G = c.vit_image / c.vit_patch, Np = G * G, N = Np + 1, Hh = c.vit_heads, D = W / Hh;
  const long M = (long)B * N;
  if (!e->vit_wpatch || !e->vit_bpatch || !e->vit_cls || !e->vit_pos) return e->fail(EMU_ERR_STATE, "ViT stem weights missing");
  for (auto& b : e->vit)
    if (!b.wqkv || !b.bqkv || b.bias_loaded != 3u || !b.wproj || !b.bproj || !b.wfc1 || !b.bfc1 || !b.wfc2 || !b.bfc2 ||
        !b.ln1w || !b.ln1b || !b.ln2w || !b.ln2b)
      return e->fail(EMU_ERR_STATE, "ViT block weights missing");
  EMU_TRY(e->ensure(e->vit_patches, (size_t)B * Np * (e->vit_kpad > W ? e->vit_kpad : W) * 2 * 2));
  EMU_TRY(e->ensure(e->vit_x, (size_t)M * W * 2));
  EMU_TRY(e->ensure(e->vit_y, (size_t)M * W * 2));
  EMU_TRY(e->ensure(e->vit_qkv, (size_t)M * 3 * W * 2));
  EMU_TRY(e->ensure(e->vit_att, (size_t)M * W * 2));
  EMU_TRY(e->ensure(e->vit_mlp, (size_t)M * c.vit_mlp * 2));
  bf16* x = (bf16*)e->vit_x.p;
  bf16* y = (bf16*)e->vit_y.p;
  bf16* qkv = (bf16*)e->vit_qkv.p;
  bf16* att = (bf16*)e->vit_att.p;
  bf16* mlp = (bf16*)e->vit_mlp.p;
  bf16* cols = (bf16*)e->vit_patches.p;
  bf16* pemb = cols + (size_t)B * Np * e->vit_kpad;

  // patch embedding: im2col -> GEMM(+bias) -> [CLS | patches] + pos_embed
  EMU_TRY(vit_im2col((const bf16*)image, cols, B, 3, c.vit_image, c.vit_patch, e->vit_kpad, st));
  {
    GemmEpilogue ep;
    ep.C = pemb; ep.ldc = W; ep.bias = e->vit_bpatch;
    EMU_TRY(gemm_bf16(cols, e->vit_kpad, e->vit_wpatch, e->vit_kpad, B * Np, W, e->vit_kpad, ep, st));
  }
  EMU_TRY(vit_assemble(pemb, e->vit_cls, e->vit_pos, x, B, Np, W, st));
  count_launch(3);

  const float scale = 1.0f / sqrtf((float)D);
  for (int l = 0; l < c.vit_layers; ++l) {
    const VitBlock& b = e->vit[l];
    const bf16* attn_in = x;
    if (!c.vit_postnorm) {  // Emu1 pre-norm
      EMU_TRY(layernorm(x, b.ln1w, b.ln1b, nullptr, y, (int)M, W, c.vit_ln_eps, st));
      attn_in = y;
      count_launch();
    }
    GemmEpilogue ep;
    ep.C = qkv; ep.ldc = 3 * W; ep.bias = b.bqkv;
    EMU_TRY(gemm_bf16(attn_in, W, b.wqkv, W, (int)M, 3 * W, W, ep, st));
    AttnArgs a;
    a.q = qkv; a.k = qkv + W; a.v = qkv + 2 * W;
    a.q_bs = a.k_bs = a.v_bs = (long)N * 3 * W;
    a.q_ts = a.k_ts = a.v_ts = 3 * W;
    a.q_hs = a.k_hs = a.v_hs = D;
    a.out = att; a.o_bs = (long)N * W; a.o_ts = W; a.o_hs = D;
    a.B = B; a.H = Hh; a.Nq = N; a.Nk = N; a.D = D; a.scale = scale; a.causal = 0;
    EMU_TRY(attn_prefill(a, st));
    if (c.vit_postnorm) {
      GemmEpilogue ep2;
      ep2.C = y; ep2.ldc = W; ep2.bias = b.bproj;
      EMU_TRY(gemm_bf16(att, W, b.wproj, W, (int)M, W, W, ep2, st));
      EMU_TRY(layernorm(y, b.ln1w, b.ln1b, x, x, (int)M, W, c.vit_ln_eps, st));  // x = x + LN(attn(x))
      GemmEpilogue ep3;
      ep3.C = mlp; ep3.ldc = c.vit_mlp; ep3.bias = b.bfc1; ep3.mode = EPI_GELU;
      EMU_TRY(gemm_bf16(x, W, b.wfc1, W, (int)M, c.vit_mlp, W, ep3, st));
      GemmEpilogue ep4;
      ep4.C = y; ep4.ldc = W; ep4.bias = b.bfc2;
      EMU_TRY(gemm_bf16(mlp, c.vit_mlp, b.wfc2, c.vit_mlp, (int)M, W, c.vit_mlp, ep4, st));
      EMU_TRY(layernorm(y, b.ln2w, b.ln2b, x, x, (int)M, W, c.vit_ln_eps, st));  // x = x + LN(mlp(x))
      count_launch(7);
    } else {
      GemmEpilogue ep2;
      ep2.C = x; ep2.ldc = W; ep2.bias = b.bproj; ep2.residual = x; ep2.ldr = W;  // x = x + attn(LN(x))
      EMU_TRY(gemm_bf16(att, W, b.wproj, W, (int)M, W, W, ep2, st));
      EMU_TRY(layernorm(x, b.ln2w, b.ln2b, nullptr, y, (int)M, W, c.vit_ln_eps, st));
      GemmEpilogue ep3;
      ep3.C = mlp; ep3.ldc = c.vit_mlp; ep3.bias = b.bfc1; ep3.mode = EPI_GELU;
      EMU_TRY(gemm_bf16(y, W, b.wfc1, W, (int)M, c.vit_mlp, W, ep3, st));
      GemmEpilogue ep4;
      ep4.C = x; ep4.ldc = W; ep4.bias = b.bfc2; ep4.residual = x; ep4.ldr = W;  // x = x + mlp(LN(x))
      EMU_TRY(gemm_bf16(mlp, c.vit_mlp, b.wfc2, c.vit_mlp, (int)M, W, c.vit_mlp, ep4, st));
      count_launch(6);
    }
  }
  if (pool) {
    int q = 1;
    while (q * q < n_query) ++q;
    if (q * q != n_query || G % q) return e->fail(EMU_ERR_INVALID, "n_query must be a square dividing the token grid");
    EMU_TRY(vit_pool(x, (bf16*)out, B, G, W, G / q, st));
    count_launch();
  } else if (c.vit_final_ln) {
    if (!e->vit_lnf_w || !e->vit_lnf_b) return e->fail(EMU_ERR_STATE, "ln_visual missing");
    EMU_TRY(layernorm(x, e->vit_lnf_w, e->vit_lnf_b, nullptr, (bf16*)out, (int)M, W, c.vit_ln_eps, st));
    count_launch();
  } else {
    if (cudaMemcpyAsync(out, x, (size_t)M * W * 2, cudaMemcpyDeviceToDevice, st) != cudaSuccess)
      return e->fail(EMU_ERR_CUDA, "copy out failed");
  }
  return EMU_OK;
}

// ================================================================================================
// LLaMA decoder
// ================================================================================================
static inline bf16* kv_layer(EmuEngine* e, int layer, int kv) {
  const EmuConfig& c = e->cfg;
  const size_t per = (size_t)c.llm_max_batch * e->Hl * c.llm_max_seq * c.llm_head_dim;
  return e->kv + ((size_t)layer * 2 + kv) * per;
}

static int llm_ready(EmuEngine* e) {
  if (e->cfg.llm_layers < 1) return e->fail(EMU_ERR_STATE, "engine has no LLM");
  if (!e->embed || !e->final_norm || !e->lm_head) return e->fail(EMU_ERR_STATE, "LLM embed/norm/lm_head missing");
  for (size_t l = 0; l < e->layers.size(); ++l) {
    const LlmLayer& L = e->layers[l];
    if (!L.wqkv || !L.wo || !L.wgu || !L.wdown || !L.ln1 || !L.ln2 || L.loaded != LlmLayer::kAll) {
      static const char* names[9] = {"q_proj", "k_proj", "v_proj", "o_proj", "gate_proj", "up_proj", "down_proj",
                                     "input_layernorm", "post_attention_layernorm"};
      std::string miss;
      for (int b = 0; b < 9; ++b)
        if (!(L.loaded & (1u << b))) miss += std::string(miss.empty() ? "" : ", ") + names[b];
      return e->fail(EMU_ERR_STATE, "LLM layer " + std::to_string(l) + " is missing " + miss);
    }
  }
  return EMU_OK;
}

extern "C" int emu_llm_reset(EmuEngine* e, emu_stream_t s) {
  if (!e) return EMU_ERR_INVALID;
  e->cur_len = 0;
  e->cache_B = 0;
  if (e->d_pos && cudaMemsetAsync(e->d_pos, 0, 3 * kLlmMaxRows * sizeof(int), (cudaStream_t)s) != cudaSuccess) return EMU_ERR_CUDA;
  if (e->kv_indir && e->kv_indir_dirty) {
    EMU_TRY(kv_indir_identity(e->kv_indir, e->cfg.llm_max_batch, e->cfg.llm_max_seq, (cudaStream_t)s));
    e->kv_indir_dirty = false;
  }
  return EMU_OK;
}
extern "C" int emu_llm_cur_len(EmuEngine* e) { return e ? e->cur_len : -1; }

__global__ void gather_rows_int_kernel(int* start, int* posoff, const int* __restrict__ src, int n) {
  __shared__ int a[emu::kLlmMaxRows], b[emu::kLlmMaxRows];
  if (threadIdx.x < n) {
    a[threadIdx.x] = start[src[threadIdx.x]];
    b[threadIdx.x] = posoff[src[threadIdx.x]];
  }
  __syncthreads();
  if (threadIdx.x < n) {
    start[threadIdx.x] = a[threadIdx.x];
    posoff[threadIdx.x] = b[threadIdx.x];
  }
}

// re-parent the cached sequences: row b continues the sequence row src[b] held.  Default: rewrite the row table the
// decode attention reads through (a few hundred KB); EMU_KV_COPY=1 moves the cache itself like HF does.
static int kv_reparent(EmuEngine* e, const int32_t* src_idx, int B, cudaStream_t st) {
  const EmuConfig& c = e->cfg;
  if (e->kv_copy)
    return kv_reorder(e->kv, c.llm_max_batch, src_idx, B, (long)c.llm_layers * 2, e->cur_len, e->Hl, c.llm_head_dim,
                      c.llm_max_seq, st);
  e->kv_indir_dirty = true;
  return kv_indir_update(e->kv_indir, src_idx, B, c.llm_max_seq, e->cur_len, st);
}

extern "C" int emu_llm_expand(EmuEngine* e, const int32_t* src_idx, int new_B, emu_stream_t stream) {
  if (!e || !src_idx || new_B < 1) return EMU_ERR_INVALID;
  const EmuConfig& c = e->cfg;
  if (new_B > c.llm_max_batch) return e->fail(EMU_ERR_INVALID, "expanded batch exceeds llm_max_batch");
  if (e->cur_len < 1) return e->fail(EMU_ERR_STATE, "expand before prefill");
  cudaStream_t st = (cudaStream_t)stream;
  EMU_TRY(kv_reparent(e, src_idx, new_B, st));
  gather_rows_int_kernel<<<1, 32, 0, st>>>(e->d_start, e->d_posoff, src_idx, new_B);
  count_launch(2);
  e->cache_B = new_B;
  return cudaGetLastError() == cudaSuccess ? EMU_OK : e->fail(EMU_ERR_CUDA, "cache expand failed");
}

extern "C" int emu_llm_embed(EmuEngine* e, const int32_t* ids, int n, void* out, emu_stream_t s) {
  if (!e || !ids || !out || n < 1) return EMU_ERR_INVALID;
  if (!e->embed) return e->fail(EMU_ERR_STATE, "embed_tokens missing");
  count_launch();
  return embed_gather(e->embed, ids, (bf16*)out, n, e->cfg.llm_hidden, (cudaStream_t)s);
}

extern "C" int emu_project(EmuEngine* e, int which, const void* x, int M, void* y, emu_stream_t s) {
  if (!e || !x || !y || M < 1) return EMU_ERR_INVALID;
  const bf16* W = which == 0 ? e->proj_up : (which == 1 ? e->proj_down : e->stu_head);
  const int in = which == 0 ? e->proj_up_in : (which == 1 ? e->proj_down_in : e->stu_in);
  const int out = which == 0 ? e->proj_up_out : (which == 1 ? e->proj_down_out : e->stu_out);
  if (!W) return e->fail(EMU_ERR_STATE, "projection weight missing");
  cudaStream_t st = (cudaStream_t)s;
  count_launch();
  if (M <= 8 && in % 32 == 0) {
    GemvArgs a;
    a.W = W; a.N = out; a.K = in; a.x = (const bf16*)x; a.ldx = in; a.B = M; a.y = y; a.ldy = out;
    return gemv_bf16(a, st);
  }
  GemmEpilogue ep;
  ep.C = y; ep.ldc = out;
  return gemm_bf16((const bf16*)x, in, W, in, M, out, in, ep, st);
}

extern "C" int emu_llm_prefill(EmuEngine* e, const void* inputs_embeds, const int32_t* attention_mask, int B, int N,
                               int hf_positions, void* last_hidden, float* logits_last, emu_stream_t stream) {
  if (!e || !inputs_embeds || B < 1 || N < 1) return EMU_ERR_INVALID;
  EMU_TRY(llm_ready(e));
  const EmuConfig& c = e->cfg;
  cudaStream_t st = (cudaStream_t)stream;
  PdlScope pdl_chain(1);
  if (B > c.llm_max_batch) return e->fail(EMU_ERR_INVALID, "batch exceeds llm_max_batch");
  if (e->cur_len + N > c.llm_max_seq) return e->fail(EMU_ERR_INVALID, "sequence exceeds llm_max_seq");
  if (e->cur_len > 0 && B != e->cache_B) return e->fail(EMU_ERR_STATE, "batch differs from cached batch");
  if (e->cur_len > 0 && e->kv_indir_dirty)
    return e->fail(EMU_ERR_STATE, "a further prompt chunk after a beam re-parent needs EMU_KV_COPY=1 (the prefill attention reads rows directly)");
  const int Hd = c.llm_hidden, D = c.llm_head_dim, Hl = e->Hl, Fl = e->Fl;
  const long M = (long)B * N;
  const int pos0 = e->cur_len;
  EMU_TRY(e->ensure(e->pf_h, (size_t)M * Hd * 2));
  EMU_TRY(e->ensure(e->pf_xn, (size_t)M * Hd * 2));
  EMU_TRY(e->ensure(e->pf_qkv, (size_t)M * 3 * Hl * D * 2));
  EMU_TRY(e->ensure(e->pf_attn, (size_t)M * Hl * D * 2));
  EMU_TRY(e->ensure(e->pf_act, (size_t)M * Fl * 2));
  if (e->tp_size > 1) EMU_TRY(e->ensure(e->pf_tmp, (size_t)M * Hd * 2));
  bf16* h = (bf16*)e->pf_h.p;
  bf16* xn = (bf16*)e->pf_xn.p;
  bf16* qkv = (bf16*)e->pf_qkv.p;
  bf16* att = (bf16*)e->pf_attn.p;
  bf16* act = (bf16*)e->pf_act.p;
  bf16* tmp = (bf16*)e->pf_tmp.p;
  if (cudaMemcpyAsync(h, inputs_embeds, (size_t)M * Hd * 2, cudaMemcpyDeviceToDevice, st) != cudaSuccess)
    return e->fail(EMU_ERR_CUDA, "embeds copy failed");
  if (pos0 == 0) {
    if (attention_mask) mask_start_kernel<<<B, 32, 0, st>>>(attention_mask, N, e->d_start, e->d_posoff, hf_positions, 0);
    else cudaMemsetAsync(e->d_start, 0, 2 * kLlmMaxRows * sizeof(int), st);
    count_launch();
    e->cache_B = B;
  }
  const float scale = 1.0f / sqrtf((float)D);
  for (int l = 0; l < c.llm_layers; ++l) {
    const LlmLayer& L = e->layers[l];
    bf16* kc = kv_layer(e, l, 0);
    bf16* vc = kv_layer(e, l, 1);
    EMU_TRY(rmsnorm(h, L.ln1, xn, (int)M, Hd, c.llm_rms_eps, 0, st));
    GemmEpilogue ep;
    ep.C = qkv; ep.ldc = 3 * Hl * D;
    EMU_TRY(gemm_bf16(xn, Hd, L.wqkv, Hd, (int)M, 3 * Hl * D, Hd, ep, st));
    EMU_TRY(rope_kv_write(qkv, B, N, Hl, D, e->rope_cos, e->rope_sin, e->d_posoff, pos0, kc, vc, c.llm_max_seq, st));
    AttnArgs a;
    a.q = qkv; a.q_bs = (long)N * 3 * Hl * D; a.q_ts = 3 * Hl * D; a.q_hs = D;
    a.k = kc; a.k_bs = (long)Hl * c.llm_max_seq * D; a.k_hs = (long)c.llm_max_seq * D; a.k_ts = D;
    a.v = vc; a.v_bs = a.k_bs; a.v_hs = a.k_hs; a.v_ts = D;
    a.out = att; a.o_bs = (long)N * Hl * D; a.o_ts = Hl * D; a.o_hs = D;
    a.B = B; a.H = Hl; a.Nq = N; a.Nk = pos0 + N; a.D = D; a.scale = scale; a.causal = 1; a.kv_start = e->d_start;
    EMU_TRY(attn_prefill(a, st));
    if (e->tp_size == 1) {
      GemmEpilogue eo;
      eo.C = h; eo.ldc = Hd; eo.residual = h; eo.ldr = Hd;
      EMU_TRY(gemm_bf16(att, Hl * D, L.wo, Hl * D, (int)M, Hd, Hl * D, eo, st));
    } else {
      GemmEpilogue eo;
      eo.C = tmp; eo.ldc = Hd;
      EMU_TRY(gemm_bf16(att, Hl * D, L.wo, Hl * D, (int)M, Hd, Hl * D, eo, st));
      EMU_TRY(nccl_allreduce_bf16(e, tmp, (size_t)M * Hd, st));
      EMU_TRY(add_rows(h, tmp, h, M * Hd, st));
      count_launch(2);
    }
    EMU_TRY(rmsnorm(h, L.ln2, xn, (int)M, Hd, c.llm_rms_eps, 0, st));
    GemmEpilogue eg;
    eg.C = act; eg.ldc = Fl; eg.mode = EPI_SWIGLU;
    EMU_TRY(gemm_bf16(xn, Hd, L.wgu, Hd, (int)M, 2 * Fl, Hd, eg, st));
    if (e->tp_size == 1) {
      GemmEpilogue ed;
      ed.C = h; ed.ldc = Hd; ed.residual = h; ed.ldr = Hd;
      EMU_TRY(gemm_bf16(act, Fl, L.wdown, Fl, (int)M, Hd, Fl, ed, st));
    } else {
      GemmEpilogue ed;
      ed.C = tmp; ed.ldc = Hd;
      EMU_TRY(gemm_bf16(act, Fl, L.wdown, Fl, (int)M, Hd, Fl, ed, st));
      EMU_TRY(nccl_allreduce_bf16(e, tmp, (size_t)M * Hd, st));
      EMU_TRY(add_rows(h, tmp, h, M * Hd, st));
      count_launch(2);
    }
    count_launch(8);
  }
  e->cur_len = pos0 + N;
  set_int_kernel<<<1, 32, 0, st>>>(e->d_pos, kLlmMaxRows, e->cur_len);  // slot of the next token
  count_launch();
  if (last_hidden) {
    EMU_TRY(rmsnorm(h, e->final_norm, (bf16*)last_hidden, (int)M, Hd, c.llm_rms_eps, 0, st));
    count_launch();
  }
  if (logits_last && B > 8) {
    // more rows than the skinny GEMV takes: final norm of the last position of every sequence, then the wgmma GEMM
    EMU_TRY(e->ensure(e->pf_last, (size_t)B * Hd * 2));
    bf16* last = (bf16*)e->pf_last.p;
    if (cudaMemcpy2DAsync(last, (size_t)Hd * 2, h + (size_t)(N - 1) * Hd, (size_t)N * Hd * 2, (size_t)Hd * 2, B,
                          cudaMemcpyDeviceToDevice, st) != cudaSuccess)
      return e->fail(EMU_ERR_CUDA, "last-position gather failed");
    EMU_TRY(rmsnorm(last, e->final_norm, last, B, Hd, c.llm_rms_eps, 0, st));
    GemmEpilogue el;
    el.out_fp32 = 1;
    if (e->tp_size == 1) {
      el.C = logits_last; el.ldc = c.llm_vocab;
      EMU_TRY(gemm_bf16(last, Hd, e->lm_head, Hd, B, e->Vl, Hd, el, st));
    } else {
      el.C = e->dec_logits_shard; el.ldc = e->Vl;
      EMU_TRY(gemm_bf16(last, Hd, e->lm_head, Hd, B, e->Vl, Hd, el, st));
      EMU_TRY(gather_logits(e, e->dec_logits_shard, e->dec_logits_gather, logits_last, B, st));
      count_launch(2);
    }
    count_launch(2);
  } else if (logits_last) {
    GemvArgs g;
    g.W = e->lm_head; g.N = e->Vl; g.K = Hd;
    g.x = h + (size_t)(N - 1) * Hd; g.ldx = N * Hd; g.B = B;
    g.norm_w = e->final_norm; g.norm_eps = c.llm_rms_eps;
    g.out_fp32 = 1;
    if (e->tp_size == 1) {
      g.y = logits_last; g.ldy = c.llm_vocab;
      EMU_TRY(gemv_bf16(g, st));
    } else {
      g.y = e->dec_logits_shard; g.ldy = e->Vl;
      EMU_TRY(gemv_bf16(g, st));
      EMU_TRY(gather_logits(e, e->dec_logits_shard, e->dec_logits_gather, logits_last, B, st));
      count_launch(2);
    }
    count_launch();
  }
  return EMU_OK;
}

// tensor-parallel tail of a row-parallel projection (o_proj / down_proj) in the decode loop: h += sum over ranks of W_r x_r.
// Preferred: fp32 partial -> NVLink peer-memory push + flag + fixed-order reduce in ONE kernel (tp_exchange.cu);
// otherwise NCCL all-reduce of the bf16 partial + add.
static int row_parallel_tail(EmuEngine* e, GemvArgs& g, bf16* h, int B, int Hd, int idx, cudaStream_t st, int* nl) {
  if (e->tp_p2p && e->tp_ll) {
    // fused: the GEMV epilogue itself pushes {value, flag} words to every rank; the poll + fixed-order reduce + residual
    // add is done by the first CTAs of the same kernel once their rows are out (tp_fold) or by one small kernel
    GemvArgs f = g;
    f.ldy = Hd;
    if (tp_ll_prepare(e, f, idx) == EMU_OK) {
      if (e->tp_fold) {
        f.ll_h = h;
        f.ll_red = 32;
      }
      const int rc = gemv_bf16(f, st);
      if (rc == EMU_OK) {
        if (e->tp_fold) return EMU_OK;
        EMU_TRY(tp_ll_reduce(e, h, (long)B * Hd, idx, g.pdl, st));
        *nl += 1;
        return EMU_OK;
      }
      if (rc != EMU_ERR_UNSUPPORTED) return rc;
    }
  }
  if (e->tp_p2p) {
    g.y = e->dec_part; g.ldy = Hd; g.out_fp32 = 1;
    EMU_TRY(gemv_bf16(g, st));
    EMU_TRY(tp_reduce_add(e, e->dec_part, h, (long)B * Hd, g.pdl, st));
    *nl += 1;
    return EMU_OK;
  }
  g.y = e->dec_tmp; g.ldy = Hd;
  EMU_TRY(gemv_bf16(g, st));
  EMU_TRY(nccl_allreduce_bf16(e, e->dec_tmp, (size_t)B * Hd, st));
  EMU_TRY(add_rows(h, e->dec_tmp, h, (long)B * Hd, st));
  *nl += 2;
  return EMU_OK;
}

// One decode step for MORE than 8 cache rows (BASELINE config 4: 4 prompts x 5 beams = 20 rows): the skinny GEMV takes at most
// 8 activation rows, so the projections run on the wgmma GEMM with M = B (one 128-row tile, weights streamed once — still
// HBM-bound), RoPE + cache append as in prefill but at the device-side slot, the split-KV decode attention over the cache,
// NCCL all-reduce on the row-parallel outputs under tensor parallelism.  Same arithmetic / rounding points as the narrow
// path; captured into the same CUDA-graph cache.
// a projection of the wide decode step: weights as the 128-row MMA operand (gemm_skinny.cu); shapes or epilogues that kernel
// does not take go to the general GEMM
static int wide_gemm(EmuEngine* e, const bf16* X, int ldx, const bf16* W, int ldw, int B, int N, int K, const GemmEpilogue& ep,
                     cudaStream_t st) {
  if (e->wide_skinny && e->sk_ws) {
    const int rc = gemm_skinny_bf16(X, ldx, W, ldw, B, N, K, ep, e->sk_ws, e->sk_counters, st);
    if (rc != EMU_ERR_UNSUPPORTED) return rc;
  }
  return gemm_bf16(X, ldx, W, ldw, B, N, K, ep, st);
}

// tensor-parallel tail of a row-parallel projection of the wide step: h += sum over ranks of X_r W_r^T.  With the peer-memory
// exchange: fp32 partial -> one kernel that pushes it to every rank over NVLink, waits for the others and adds the fixed-order
// sum to h (no NCCL launch; the partials meet in fp32 and are rounded once, as in the unsharded model).  Otherwise NCCL.
static int wide_row_parallel(EmuEngine* e, const bf16* X, int ldx, const bf16* W, int ldw, int B, int Hd, int K, bf16* h,
                             cudaStream_t st, int* nl) {
  GemmEpilogue ep;
  if (e->tp_p2p && !((long)B * Hd & 3)) {
    ep.C = e->dec_part; ep.ldc = Hd; ep.out_fp32 = 1;
    EMU_TRY(wide_gemm(e, X, ldx, W, ldw, B, Hd, K, ep, st));
    EMU_TRY(tp_reduce_add(e, e->dec_part, h, (long)B * Hd, g_pdl_chain, st));
    *nl += 1;
    return EMU_OK;
  }
  ep.C = e->dec_tmp; ep.ldc = Hd;
  EMU_TRY(wide_gemm(e, X, ldx, W, ldw, B, Hd, K, ep, st));
  EMU_TRY(nccl_allreduce_bf16(e, e->dec_tmp, (size_t)B * Hd, st));
  EMU_TRY(add_rows(h, e->dec_tmp, h, (long)B * Hd, st));
  *nl += 2;
  return EMU_OK;
}

static int decode_step_body_wide(EmuEngine* e, const int32_t* token_ids, const void* embeds, int B, float* logits,
                                 void* hidden, int32_t* next_ids, int ban_id, cudaStream_t st, int* n_launch) {
  const EmuConfig& c = e->cfg;
  const int Hd = c.llm_hidden, D = c.llm_head_dim, Hl = e->Hl, Fl = e->Fl;
  int nl = 0;
  bf16* h = e->dec_h;
  bf16* xn = e->dec_xn;
  bf16* qkv = e->dec_qkv;
  if (token_ids) {
    EMU_TRY(embed_gather(e->embed, token_ids, h, B, Hd, st));
    ++nl;
  } else if (cudaMemcpyAsync(h, embeds, (size_t)B * Hd * 2, cudaMemcpyDeviceToDevice, st) != cudaSuccess) {
    return e->fail(EMU_ERR_CUDA, "embeds copy failed");
  }
  const float scale = 1.0f / sqrtf((float)D);
  PdlScope pdl_chain(1);
  for (int l = 0; l < c.llm_layers; ++l) {
    const LlmLayer& L = e->layers[l];
    bf16* kc = kv_layer(e, l, 0);
    bf16* vc = kv_layer(e, l, 1);
    EMU_TRY(rmsnorm(h, L.ln1, xn, B, Hd, c.llm_rms_eps, 0, st));
    GemmEpilogue ep;
    ep.C = qkv; ep.ldc = 3 * Hl * D;
    EMU_TRY(wide_gemm(e, xn, Hd, L.wqkv, Hd, B, 3 * Hl * D, Hd, ep, st));
    EMU_TRY(rope_kv_write(qkv, B, 1, Hl, D, e->rope_cos, e->rope_sin, e->d_posoff, 0, kc, vc, c.llm_max_seq, st, e->d_pos,
                          e->dec_q));
    EMU_TRY(attn_decode(e->dec_q, kc, vc, B, Hl, D, c.llm_max_seq, e->d_pos, e->d_start, scale, e->dec_attn, e->dec_attn_ws,
                        e->dec_counters, c.llm_max_seq, 0, st, e->kv_indir));
    GemmEpilogue eo;
    if (e->tp_size == 1) {
      eo.C = h; eo.ldc = Hd; eo.residual = h; eo.ldr = Hd;
      EMU_TRY(wide_gemm(e, e->dec_attn, Hl * D, L.wo, Hl * D, B, Hd, Hl * D, eo, st));
    } else {
      EMU_TRY(wide_row_parallel(e, e->dec_attn, Hl * D, L.wo, Hl * D, B, Hd, Hl * D, h, st, &nl));
    }
    EMU_TRY(rmsnorm(h, L.ln2, xn, B, Hd, c.llm_rms_eps, 0, st));
    GemmEpilogue eg;
    eg.C = e->dec_act; eg.ldc = Fl; eg.mode = EPI_SWIGLU;
    EMU_TRY(wide_gemm(e, xn, Hd, L.wgu, Hd, B, 2 * Fl, Hd, eg, st));
    GemmEpilogue ed;
    if (e->tp_size == 1) {
      ed.C = h; ed.ldc = Hd; ed.residual = h; ed.ldr = Hd;
      EMU_TRY(wide_gemm(e, e->dec_act, Fl, L.wdown, Fl, B, Hd, Fl, ed, st));
    } else {
      EMU_TRY(wide_row_parallel(e, e->dec_act, Fl, L.wdown, Fl, B, Hd, Fl, h, st, &nl));
    }
    nl += 8;
  }
  if (hidden) {
    EMU_TRY(rmsnorm(h, e->final_norm, (bf16*)hidden, B, Hd, c.llm_rms_eps, 0, st));
    ++nl;
  }
  if (logits || next_ids) {
    float* lg = logits ? logits : e->dec_logits_local;
    EMU_TRY(rmsnorm(h, e->final_norm, xn, B, Hd, c.llm_rms_eps, 0, st));
    GemmEpilogue el;
    el.out_fp32 = 1;
    if (e->tp_size == 1) {
      el.C = lg; el.ldc = c.llm_vocab;
      EMU_TRY(wide_gemm(e, xn, Hd, e->lm_head, Hd, B, e->Vl, Hd, el, st));
    } else {
      el.C = e->dec_logits_shard; el.ldc = e->Vl;
      EMU_TRY(wide_gemm(e, xn, Hd, e->lm_head, Hd, B, e->Vl, Hd, el, st));
      EMU_TRY(gather_logits(e, e->dec_logits_shard, e->dec_logits_gather, lg, B, st));
      nl += 2;
    }
    nl += 2;
    if (next_ids) {
      if (ban_id >= 0) {
        argmax_ban_kernel<<<B, 1, 0, st>>>(lg, c.llm_vocab, ban_id);
        ++nl;
      }
      EMU_TRY(argmax_rows(lg, B, c.llm_vocab, next_ids, st));
      ++nl;
    }
  }
  advance_pos_kernel<<<1, 32, 0, st>>>(e->d_pos, kLlmMaxRows, tp_step_counter(e));
  ++nl;
  *n_launch = nl;
  return EMU_OK;
}

// the kernels of one decode step (captured into a CUDA graph by emu_llm_decode)
static int decode_step_body(EmuEngine* e, const int32_t* token_ids, const void* embeds, int B, float* logits,
                            void* hidden, int32_t* next_ids, int ban_id, cudaStream_t st, int* n_launch) {
  if (B > 8) return decode_step_body_wide(e, token_ids, embeds, B, logits, hidden, next_ids, ban_id, st, n_launch);
  const EmuConfig& c = e->cfg;
  const int Hd = c.llm_hidden, D = c.llm_head_dim, Hl = e->Hl, Fl = e->Fl;
  int nl = 0;
  bf16* h = e->dec_h;
  if (token_ids) {
    EMU_TRY(embed_gather(e->embed, token_ids, h, B, Hd, st));
    ++nl;
  } else {
    if (cudaMemcpyAsync(h, embeds, (size_t)B * Hd * 2, cudaMemcpyDeviceToDevice, st) != cudaSuccess)
      return e->fail(EMU_ERR_CUDA, "embeds copy failed");
  }
  const float scale = 1.0f / sqrtf((float)D);
  const int pdl = 1;
  for (int l = 0; l < c.llm_layers; ++l) {
    const LlmLayer& L = e->layers[l];
    bf16* kc = kv_layer(e, l, 0);
    bf16* vc = kv_layer(e, l, 1);
    GemvArgs q;
    q.W = L.wqkv; q.N = 3 * Hl * D; q.K = Hd; q.x = h; q.ldx = Hd; q.B = B;
    q.norm_w = L.ln1; q.norm_eps = c.llm_rms_eps; q.mode = GEMV_ROPE_QKV;
    q.y = e->dec_q; q.ldy = Hl * D; q.n_heads = Hl; q.head_dim = D;
    q.rope_cos = e->rope_cos; q.rope_sin = e->rope_sin; q.pos = e->d_pos; q.pos_off = e->d_posoff;
    q.k_cache = kc; q.v_cache = vc; q.t_max = c.llm_max_seq; q.pdl = (l > 0 || token_ids) ? pdl : 0;
    EMU_TRY(gemv_bf16(q, st));
    EMU_TRY(attn_decode(e->dec_q, kc, vc, B, Hl, D, c.llm_max_seq, e->d_pos, e->d_start, scale, e->dec_attn,
                        e->dec_attn_ws, e->dec_counters, c.llm_max_seq, pdl, st, e->kv_indir));
    GemvArgs o;
    o.W = L.wo; o.N = Hd; o.K = Hl * D; o.x = e->dec_attn; o.ldx = Hl * D; o.B = B; o.pdl = pdl;
    if (e->tp_size == 1) {
      o.residual = h; o.ldr = Hd; o.y = h; o.ldy = Hd;
      EMU_TRY(gemv_bf16(o, st));
    } else {
      EMU_TRY(row_parallel_tail(e, o, h, B, Hd, 2 * l, st, &nl));
    }
    GemvArgs g;
    g.W = L.wgu; g.N = 2 * Fl; g.K = Hd; g.x = h; g.ldx = Hd; g.B = B;
    g.norm_w = L.ln2; g.norm_eps = c.llm_rms_eps; g.mode = EPI_SWIGLU; g.y = e->dec_act; g.ldy = Fl;
    g.pdl = pdl;
    EMU_TRY(gemv_bf16(g, st));
    GemvArgs d;
    d.W = L.wdown; d.N = Hd; d.K = Fl; d.x = e->dec_act; d.ldx = Fl; d.B = B; d.pdl = pdl;
    if (e->tp_size == 1) {
      d.residual = h; d.ldr = Hd; d.y = h; d.ldy = Hd;
      EMU_TRY(gemv_bf16(d, st));
    } else {
      EMU_TRY(row_parallel_tail(e, d, h, B, Hd, 2 * l + 1, st, &nl));
    }
    nl += 5;
  }
  if (hidden) {
    EMU_TRY(rmsnorm(h, e->final_norm, (bf16*)hidden, B, Hd, c.llm_rms_eps, 0, st));
    ++nl;
  }
  if (logits || next_ids) {
    float* lg = logits ? logits : e->dec_logits_local;
    GemvArgs g;
    g.W = e->lm_head; g.N = e->Vl; g.K = Hd; g.x = h; g.ldx = Hd; g.B = B;
    g.norm_w = e->final_norm; g.norm_eps = c.llm_rms_eps;
    g.out_fp32 = 1; g.pdl = pdl;
    if (e->tp_size == 1) {
      g.y = lg; g.ldy = c.llm_vocab;
      EMU_TRY(gemv_bf16(g, st));
    } else {
      g.y = e->dec_logits_shard; g.ldy = e->Vl;
      EMU_TRY(gemv_bf16(g, st));
      if (e->tp_p2p) {
        EMU_TRY(tp_gather_logits(e, e->dec_logits_shard, lg, B, pdl, st));
        nl += 1;
      } else {
        EMU_TRY(gather_logits(e, e->dec_logits_shard, e->dec_logits_gather, lg, B, st));
        nl += 2;
      }
    }
    ++nl;
    if (next_ids) {
      if (ban_id >= 0) {
        argmax_ban_kernel<<<B, 1, 0, st>>>(lg, c.llm_vocab, ban_id);
        ++nl;
      }
      EMU_TRY(argmax_rows(lg, B, c.llm_vocab, next_ids, st));
      ++nl;
    }
  }
  advance_pos_kernel<<<1, 32, 0, st>>>(e->d_pos, kLlmMaxRows, tp_step_counter(e));
  ++nl;
  *n_launch = nl;
  return EMU_OK;
}

extern "C" int emu_llm_decode(EmuEngine* e, const int32_t* token_ids, const void* embeds, const int32_t* beam_src_idx,
                              int B, float* logits, void* hidden, int32_t* next_ids, int ban_id, emu_stream_t stream) {
  if (!e || B < 1 || ((token_ids == nullptr) == (embeds == nullptr))) return EMU_ERR_INVALID;
  EMU_TRY(llm_ready(e));
  const EmuConfig& c = e->cfg;
  cudaStream_t st = (cudaStream_t)stream;
  if (e->cur_len < 1) return e->fail(EMU_ERR_STATE, "decode before prefill");
  if (B != e->cache_B) return e->fail(EMU_ERR_STATE, "batch differs from cached batch");
  if (e->cur_len + 1 > c.llm_max_seq) return e->fail(EMU_ERR_INVALID, "KV cache full");
  if (beam_src_idx) {
    EMU_TRY(kv_reparent(e, beam_src_idx, B, st));
    count_launch();
  }
  int nl = 0;
  const char* no_graph = getenv("EMU_NO_GRAPH");  // debugging / parity switch: launch the step eagerly
  const bool graphable = e->use_graphs && !(no_graph && no_graph[0] == '1');  // NCCL collectives are graph-capturable
  if (!graphable) {
    EMU_TRY(decode_step_body(e, token_ids, embeds, B, logits, hidden, next_ids, ban_id, st, &nl));
    count_launch(nl);
  } else {
    EmuEngine::GraphKey key(B, token_ids, embeds, logits, hidden, next_ids, (const void*)st, ban_id);
    auto it = e->graphs.find(key);
    if (it == e->graphs.end()) {
      if (e->graphs.size() > 64) {
        for (auto& g : e->graphs) cudaGraphExecDestroy(g.second);
        e->graphs.clear();
        e->graph_nodes.clear();
      }
      // capture on an engine-owned stream: the caller's stream may be the legacy default stream, which cannot
      // be captured; the instantiated graph is then launched on the caller's stream
      if (!e->cap_stream && cudaStreamCreateWithFlags(&e->cap_stream, cudaStreamNonBlocking) != cudaSuccess)
        return e->fail(EMU_ERR_CUDA, "capture stream create failed");
      if (cudaStreamBeginCapture(e->cap_stream, cudaStreamCaptureModeRelaxed) != cudaSuccess)
        return e->fail(EMU_ERR_CUDA, std::string("graph capture begin failed: ") + cudaGetErrorString(cudaGetLastError()));
      int rc = decode_step_body(e, token_ids, embeds, B, logits, hidden, next_ids, ban_id, e->cap_stream, &nl);
      cudaGraph_t graph = nullptr;
      cudaError_t ce = cudaStreamEndCapture(e->cap_stream, &graph);
      if (rc != EMU_OK || ce != cudaSuccess || !graph) {
        if (graph) cudaGraphDestroy(graph);
        cudaGetLastError();
        return rc != EMU_OK ? rc : e->fail(EMU_ERR_CUDA, std::string("graph capture failed: ") + cudaGetErrorString(ce));
      }
      cudaGraphExec_t exec = nullptr;
      ce = cudaGraphInstantiate(&exec, graph, 0);
      cudaGraphDestroy(graph);
      if (ce != cudaSuccess) return e->fail(EMU_ERR_CUDA, std::string("graph instantiate failed: ") + cudaGetErrorString(ce));
      e->graphs[key] = exec;
      e->graph_nodes[key] = nl;
      it = e->graphs.find(key);
    }
    if (cudaGraphLaunch(it->second, st) != cudaSuccess) return e->fail(EMU_ERR_CUDA, "graph launch failed");
    count_launch(e->graph_nodes[key]);
  }
  e->cur_len += 1;
  return EMU_OK;
}
