// emu_b200 — engine: weight ingestion/packing, EVA ViT forward, LLaMA prefill + CUDA-graphed decode step.
//
// Orchestrates the kernels of gemm_tc.cu / gemv.cu / attention.cu / elementwise.cu into the reference's
// module boundaries (SURVEY.md §8a rows a1-a12):
//   ViT      : Emu2/emu/eva_vit.py:402-431 (post-norm) and Emu1/models/eva_vit_model.py:636-665 (pre-norm)
//   LLaMA    : HF LlamaModel.forward as driven by Emu2/emu/emu.py:133-138 (prefill, hidden_states[-1]) and
//              :213-229 (generate: prefill + one-token steps with KV cache)
#include "engine.h"
#include "../../include/emu_b200_chunked.h"
#include "../../include/emu_b200_prefix.h"
#include "../../include/emu_b200_regress.h"
#include "../../include/emu_b200_slots.h"
#include "../../include/emu_b200_spec.h"

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
// active: slot mode's live-row mask (a free slot's position stays 0), or null = every row
__global__ void advance_pos_kernel(int* p, int n, unsigned* tp_step, const int* __restrict__ active) {
  if (threadIdx.x < n) p[threadIdx.x] += active ? active[threadIdx.x] : 1;
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
// slot mode: a host list of slots (or of per-slot values) passed to a kernel by value.  A kernel that frees a slot or makes
// it live resets the slot's row of the re-parenting table to identity (it may have belonged to a beam group).
struct SlotList {
  int r[kLlmMaxRows];
};
// slot mode: the slots dst continue slot src's sequence — its table row up to its length (identity beyond: a slot's own
// new tokens are in its own row), its length, start and position offset.  One CTA per destination.
__global__ void slot_fork_kernel(int src, SlotList dst, int* pos, int* start, int* posoff, int* active, int* indir, int t_max) {
  const int row = dst.r[blockIdx.x];
  const int len = pos[src];
  for (int t = threadIdx.x; t < t_max; t += blockDim.x)
    indir[(long)row * t_max + t] = t < len ? indir[(long)src * t_max + t] : row;
  if (threadIdx.x == 0) {
    pos[row] = len;
    start[row] = start[src];
    posoff[row] = posoff[src];
    active[row] = 1;
  }
}
// slots leave keeping their first keep.r[b] cache positions (0 = a plain leave, prefix caching otherwise).  The real
// left-pad start / position offset move to the kept arrays, and the slot is parked at pos = start = keep: the decode step
// computes every free slot below B and appends its junk token at pos, which then lands at position keep, past the kept
// prefix (a resume overwrites it before anything reads it), and its attention reads that one key.
__global__ void slot_keep_kernel(SlotList rows, SlotList keep, int* pos, int* start, int* posoff, int* active, int* kept_start,
                                 int* kept_posoff, int* indir, int t_max) {
  const int b = blockIdx.x, row = rows.r[b], k = keep.r[b];
  if (threadIdx.x == 0) {
    kept_start[row] = k > 0 ? start[row] : 0;
    kept_posoff[row] = k > 0 ? posoff[row] : 0;
    pos[row] = k;
    start[row] = k;
    posoff[row] = 0;
    active[row] = 0;
  }
  for (int t = threadIdx.x; t < t_max; t += blockDim.x) indir[(long)row * t_max + t] = row;
}
// prefix caching: free slot dst becomes kept with P positions copied from src (live: its current start / offset; kept: its
// saved ones).  One CTA.
__global__ void slot_copy_state_kernel(int src, int src_kept, int dst, int P, int* pos, int* start, int* posoff, int* active,
                                       int* kept_start, int* kept_posoff, int* indir, int t_max) {
  if (threadIdx.x == 0) {
    kept_start[dst] = src_kept ? kept_start[src] : start[src];
    kept_posoff[dst] = src_kept ? kept_posoff[src] : posoff[src];
    pos[dst] = P;
    start[dst] = P;
    posoff[dst] = 0;
    active[dst] = 0;
  }
  for (int t = threadIdx.x; t < t_max; t += blockDim.x) indir[(long)dst * t_max + t] = dst;
}
// slot-mode prefill, before the layers: the join-local start / position offset of every segment's slot (its kept ones; zero
// for a slot that starts from nothing).  One thread per slot.
__global__ void slot_resume_begin_kernel(SlotList rows, SlotList prefix, const int* __restrict__ kept_start,
                                         const int* __restrict__ kept_posoff, int* join_start, int* join_posoff, int n) {
  const int b = threadIdx.x;
  if (b >= n) return;
  const int row = rows.r[b], p = prefix.r[b];
  join_start[b] = p > 0 ? kept_start[row] : 0;
  join_posoff[b] = p > 0 ? kept_posoff[row] : 0;
}
// ... after the layers: segment b's slot becomes live at len.r[b] (final.r[b]) or is kept there, as slot_keep_kernel
// leaves a slot (its start / position offset saved, parked at pos = start = len).  One CTA per slot.
__global__ void slot_step_end_kernel(SlotList rows, SlotList len, SlotList final_, const int* __restrict__ join_start,
                                     const int* __restrict__ join_posoff, int* pos, int* start, int* posoff, int* active,
                                     int* kept_start, int* kept_posoff, int* indir, int t_max) {
  const int b = blockIdx.x, row = rows.r[b], n = len.r[b];
  if (threadIdx.x == 0) {
    if (final_.r[b]) {
      start[row] = join_start[b];
      posoff[row] = join_posoff[b];
    } else {
      kept_start[row] = join_start[b];
      kept_posoff[row] = join_posoff[b];
      start[row] = n;
      posoff[row] = 0;
    }
    pos[row] = n;
    active[row] = final_.r[b] ? 1 : 0;
  }
  for (int t = threadIdx.x; t < t_max; t += blockDim.x) indir[(long)row * t_max + t] = row;
}
// hidden rows idx[b] -> out row b (16-byte words)
__global__ void gather_rows_kernel(const bf16* __restrict__ h, int Hd, const int* __restrict__ idx, bf16* out) {
  const int b = blockIdx.x;
  const uint4* src = reinterpret_cast<const uint4*>(h + (long)idx[b] * Hd);
  uint4* dst = reinterpret_cast<uint4*>(out + (long)b * Hd);
  for (int i = threadIdx.x; i < Hd / 8; i += blockDim.x) dst[i] = src[i];
}
// regression join: the last packed row of segment b (rows row0[b] .. row0[b] + n_new[b] - 1 of h) -> row slot[b] of out
__global__ void gather_last_to_slot_kernel(const bf16* __restrict__ h, int Hd, const int* __restrict__ slot,
                                           const int* __restrict__ n_new, const int* __restrict__ row0, bf16* out) {
  const int b = blockIdx.x;
  const uint4* src = reinterpret_cast<const uint4*>(h + (long)(row0[b] + n_new[b] - 1) * Hd);
  uint4* dst = reinterpret_cast<uint4*>(out + (long)slot[b] * Hd);
  for (int i = threadIdx.x; i < Hd / 8; i += blockDim.x) dst[i] = src[i];
}
// regression slots: the projected row r[s] [w] of slot s becomes its feedback fb[s] and, while k[s] < L, its output row
// out[s][k[s]]; then k[s] += 1 (at most L).  One CTA per slot: CTA b is slot join.r[b] starting from k = 0 (a join of n_join
// slots), or, with n_join = 0, slot b if active[b] (a step; the rows of the other slots are dropped).  w % 8 == 0.
__global__ void regress_emit_kernel(const bf16* __restrict__ r, bf16* fb, int* k, bf16* out, int L, int w, SlotList join,
                                    int n_join, const int* __restrict__ active) {
  const int s = n_join ? join.r[blockIdx.x] : blockIdx.x;
  if (!n_join && !active[s]) return;
  const int kk = n_join ? 0 : k[s];
  const uint4* src = reinterpret_cast<const uint4*>(r + (long)s * w);
  uint4* f = reinterpret_cast<uint4*>(fb + (long)s * w);
  uint4* o = reinterpret_cast<uint4*>(out + ((long)s * L + kk) * w);
  for (int i = threadIdx.x; i < w / 8; i += blockDim.x) {
    const uint4 v = src[i];
    f[i] = v;
    if (kk < L) o[i] = v;
  }
  __syncthreads();  // every thread has read k[s]
  if (threadIdx.x == 0) k[s] = kk < L ? kk + 1 : L;
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
    e->d_active = (int*)e->dmalloc(3 * kLlmMaxRows * sizeof(int));
    e->d_join_start = e->d_active + kLlmMaxRows;
    e->d_join_posoff = e->d_active + 2 * kLlmMaxRows;
    e->d_kept_start = (int*)e->dmalloc(2 * kLlmMaxRows * sizeof(int));
    e->d_kept_posoff = e->d_kept_start + kLlmMaxRows;
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
    if (!e->rope_cos || !e->rope_sin || !e->kv || !e->d_pos || !e->d_active || !e->d_kept_start || !e->dec_h || !e->dec_q || !e->dec_attn || !e->dec_act ||
        !e->dec_tmp || !e->dec_attn_ws || !e->dec_counters || !e->dec_logits_local || !e->kv_indir) {
      emu_engine_destroy(e);
      return EMU_ERR_NOMEM;
    }
    rope_table_kernel<<<2 * kNumSMs, 256>>>(e->rope_cos, e->rope_sin, max_pos, half, c.llm_rope_theta);
    cudaMemset(e->dec_counters, 0, (size_t)Bm * e->Hl * sizeof(int));
    cudaMemset(e->d_pos, 0, 3 * kLlmMaxRows * sizeof(int));
    cudaMemset(e->d_active, 0, 3 * kLlmMaxRows * sizeof(int));
    cudaMemset(e->d_kept_start, 0, 2 * kLlmMaxRows * sizeof(int));
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
  if (e->safety) safety_destroy(e->safety);
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
  else if (starts_with(key, "safety_checker.")) rc = safety_load_tensor(e, key.substr(15), dsrc, shape, ndim, st);
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
  e->spec_n = 0;
  e->n_slots = 0;
  e->slots.clear();
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
  if (e->n_slots > 0) {  // slots differ in length: every row copies its own, read from the device positions
    int n_tok = 0;
    for (int b = 0; b < B; ++b) n_tok = e->slots[b].len > n_tok ? e->slots[b].len : n_tok;
    return kv_indir_update(e->kv_indir, src_idx, B, c.llm_max_seq, n_tok, st, e->d_pos);
  }
  return kv_indir_update(e->kv_indir, src_idx, B, c.llm_max_seq, e->cur_len, st);
}

extern "C" int emu_llm_expand(EmuEngine* e, const int32_t* src_idx, int new_B, emu_stream_t stream) {
  if (!e || !src_idx || new_B < 1) return EMU_ERR_INVALID;
  const EmuConfig& c = e->cfg;
  if (new_B > c.llm_max_batch) return e->fail(EMU_ERR_INVALID, "expanded batch exceeds llm_max_batch");
  if (e->n_slots > 0) return e->fail(EMU_ERR_STATE, "expand in slot mode: use emu_llm_fork");
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

// y [M, out] = x [M, in] W^T of projection `which` (0 project_up, 1 project_down, 2 the student head; its weight loaded):
// the GEMV up to 8 rows, the GEMM above
static int project_rows(EmuEngine* e, int which, const void* x, int M, void* y, cudaStream_t st) {
  const bf16* W = which == 0 ? e->proj_up : (which == 1 ? e->proj_down : e->stu_head);
  const int in = which == 0 ? e->proj_up_in : (which == 1 ? e->proj_down_in : e->stu_in);
  const int out = which == 0 ? e->proj_up_out : (which == 1 ? e->proj_down_out : e->stu_out);
  if (M <= 8 && in % 32 == 0) {
    GemvArgs a;
    a.W = W; a.N = out; a.K = in; a.x = (const bf16*)x; a.ldx = in; a.B = M; a.y = y; a.ldy = out;
    return gemv_bf16(a, st);
  }
  GemmEpilogue ep;
  ep.C = y; ep.ldc = out;
  return gemm_bf16((const bf16*)x, in, W, in, M, out, in, ep, st);
}

extern "C" int emu_project(EmuEngine* e, int which, const void* x, int M, void* y, emu_stream_t s) {
  if (!e || !x || !y || M < 1) return EMU_ERR_INVALID;
  if (!(which == 0 ? e->proj_up : (which == 1 ? e->proj_down : e->stu_head)))
    return e->fail(EMU_ERR_STATE, "projection weight missing");
  count_launch();
  return project_rows(e, which, x, M, y, (cudaStream_t)s);
}

// prefill workspaces for M prompt tokens; the embeddings go to pf_h (null: the caller stages them)
static int prefill_stage(EmuEngine* e, const void* inputs_embeds, long M, cudaStream_t st) {
  const EmuConfig& c = e->cfg;
  const int Hd = c.llm_hidden, D = c.llm_head_dim, Hl = e->Hl, Fl = e->Fl;
  EMU_TRY(e->ensure(e->pf_h, (size_t)M * Hd * 2));
  EMU_TRY(e->ensure(e->pf_xn, (size_t)M * Hd * 2));
  EMU_TRY(e->ensure(e->pf_qkv, (size_t)M * 3 * Hl * D * 2));
  EMU_TRY(e->ensure(e->pf_attn, (size_t)M * Hl * D * 2));
  EMU_TRY(e->ensure(e->pf_act, (size_t)M * Fl * 2));
  if (e->tp_size > 1) EMU_TRY(e->ensure(e->pf_tmp, (size_t)M * Hd * 2));
  if (inputs_embeds && cudaMemcpyAsync(e->pf_h.p, inputs_embeds, (size_t)M * Hd * 2, cudaMemcpyDeviceToDevice, st) != cudaSuccess)
    return e->fail(EMU_ERR_CUDA, "embeds copy failed");
  return EMU_OK;
}

// slot-mode prefill: B decode rows, then n segments packed back to back; M rows in all.  Device [n]: the segments' cache
// rows, prefix lengths, token counts and first packed rows.
struct MixedRows {
  int B, n, M, max_new, Nk;
  const int *seg_row, *seg_q0, *seg_new, *seg_row0;
};

// one layer's RoPE / KV append and attention of slot-mode rows: the decode rows through the row-table decode attention, written
// straight into the first B rows of att; the segments through the packed-query prefill attention
static int mixed_attention(EmuEngine* e, const MixedRows& m, bf16* qkv, bf16* att, bf16* kc, bf16* vc, float scale,
                           cudaStream_t st) {
  const EmuConfig& c = e->cfg;
  const int D = c.llm_head_dim, Hl = e->Hl;
  EMU_TRY(rope_kv_write_packed(qkv, m.M, m.B, m.n, Hl, D, e->rope_cos, e->rope_sin, e->d_pos, e->d_posoff, e->d_active, e->dec_q,
                               m.seg_row, m.seg_q0, m.seg_new, e->d_join_posoff, kc, vc, c.llm_max_seq, st));
  if (m.B > 0)
    EMU_TRY(attn_decode(e->dec_q, kc, vc, m.B, Hl, D, c.llm_max_seq, e->d_pos, e->d_start, scale, att, e->dec_attn_ws,
                        e->dec_counters, c.llm_max_seq, 0, st, e->kv_indir));
  AttnArgs a;
  a.q = qkv; a.q_ts = 3 * Hl * D; a.q_hs = D;
  a.k = kc; a.k_bs = (long)Hl * c.llm_max_seq * D; a.k_hs = (long)c.llm_max_seq * D; a.k_ts = D;
  a.v = vc; a.v_bs = a.k_bs; a.v_hs = a.k_hs; a.v_ts = D;
  a.out = att; a.o_ts = Hl * D; a.o_hs = D;
  a.B = m.n; a.H = Hl; a.Nq = m.max_new; a.Nk = m.Nk; a.D = D; a.scale = scale; a.causal = 1; a.kv_start = e->d_join_start;
  a.kv_row = m.seg_row; a.kv_rows = c.llm_max_batch;
  a.q_off = m.seg_q0; a.q_len = m.seg_new; a.q_row0 = m.seg_row0; a.q_rows = m.M;
  if (m.B > 0) count_launch();  // the layer's count has one RoPE and one attention launch
  return attn_prefill(a, st);
}

// the decoder layers over the B x N prompt tokens in pf_h: k / v of batch b go to cache row b at slots [pos0, pos0 + N),
// rotated at position slot - posoff[b]; the attention reads keys [start[b], pos0 + N) of that row.
// With mix (slot mode): the M = mix->M packed rows of mix instead, attention by mixed_attention.
static int prefill_layers(EmuEngine* e, int B, int N, int pos0, const int* start, const int* posoff, cudaStream_t st,
                          const MixedRows* mix = nullptr) {
  const EmuConfig& c = e->cfg;
  const int Hd = c.llm_hidden, D = c.llm_head_dim, Hl = e->Hl, Fl = e->Fl;
  const long M = mix ? (long)mix->M : (long)B * N;
  bf16* h = (bf16*)e->pf_h.p;
  bf16* xn = (bf16*)e->pf_xn.p;
  bf16* qkv = (bf16*)e->pf_qkv.p;
  bf16* att = (bf16*)e->pf_attn.p;
  bf16* act = (bf16*)e->pf_act.p;
  bf16* tmp = (bf16*)e->pf_tmp.p;
  const float scale = 1.0f / sqrtf((float)D);
  for (int l = 0; l < c.llm_layers; ++l) {
    const LlmLayer& L = e->layers[l];
    bf16* kc = kv_layer(e, l, 0);
    bf16* vc = kv_layer(e, l, 1);
    EMU_TRY(rmsnorm(h, L.ln1, xn, (int)M, Hd, c.llm_rms_eps, 0, st));
    GemmEpilogue ep;
    ep.C = qkv; ep.ldc = 3 * Hl * D;
    EMU_TRY(gemm_bf16(xn, Hd, L.wqkv, Hd, (int)M, 3 * Hl * D, Hd, ep, st));
    if (mix) {
      EMU_TRY(mixed_attention(e, *mix, qkv, att, kc, vc, scale, st));
    } else {
      EMU_TRY(rope_kv_write(qkv, B, N, Hl, D, e->rope_cos, e->rope_sin, posoff, pos0, kc, vc, c.llm_max_seq, st));
      AttnArgs a;
      a.q = qkv; a.q_bs = (long)N * 3 * Hl * D; a.q_ts = 3 * Hl * D; a.q_hs = D;
      a.k = kc; a.k_bs = (long)Hl * c.llm_max_seq * D; a.k_hs = (long)c.llm_max_seq * D; a.k_ts = D;
      a.v = vc; a.v_bs = a.k_bs; a.v_hs = a.k_hs; a.v_ts = D;
      a.out = att; a.o_bs = (long)N * Hl * D; a.o_ts = Hl * D; a.o_hs = D;
      a.B = B; a.H = Hl; a.Nq = N; a.Nk = pos0 + N; a.D = D; a.scale = scale; a.causal = 1; a.kv_start = start;
      EMU_TRY(attn_prefill(a, st));
    }
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
  return EMU_OK;
}

// final norm of every prompt token (last_hidden) and the logits of every sequence's last position (logits_last).  With rows
// (device [B], slot mode): the logits of hidden rows rows[0 .. B) of pf_h instead, gathered to pf_last first (N = 1).
static int prefill_outputs(EmuEngine* e, int B, int N, void* last_hidden, float* logits_last, cudaStream_t st,
                           const int* rows = nullptr) {
  const EmuConfig& c = e->cfg;
  const int Hd = c.llm_hidden;
  const long M = (long)B * N;
  bf16* h = (bf16*)e->pf_h.p;
  if (rows && logits_last) {
    EMU_TRY(e->ensure(e->pf_last, (size_t)B * Hd * 2));
    gather_rows_kernel<<<B, 128, 0, st>>>(h, Hd, rows, (bf16*)e->pf_last.p);
    count_launch();
    if (cudaGetLastError() != cudaSuccess) return e->fail(EMU_ERR_CUDA, "logits row gather failed");
    h = (bf16*)e->pf_last.p;
    N = 1;
  }
  if (last_hidden) {
    EMU_TRY(rmsnorm(h, e->final_norm, (bf16*)last_hidden, (int)M, Hd, c.llm_rms_eps, 0, st));
    count_launch();
  }
  if (logits_last && B > 8) {
    // more rows than the skinny GEMV takes: final norm of the last position of every sequence, then the wgmma GEMM
    EMU_TRY(e->ensure(e->pf_last, (size_t)B * Hd * 2));
    bf16* last = (bf16*)e->pf_last.p;
    if (!rows && cudaMemcpy2DAsync(last, (size_t)Hd * 2, h + (size_t)(N - 1) * Hd, (size_t)N * Hd * 2, (size_t)Hd * 2, B,
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

extern "C" int emu_llm_prefill(EmuEngine* e, const void* inputs_embeds, const int32_t* attention_mask, int B, int N,
                               int hf_positions, void* last_hidden, float* logits_last, emu_stream_t stream) {
  if (!e || !inputs_embeds || B < 1 || N < 1) return EMU_ERR_INVALID;
  EMU_TRY(llm_ready(e));
  const EmuConfig& c = e->cfg;
  cudaStream_t st = (cudaStream_t)stream;
  PdlScope pdl_chain(1);
  if (e->n_slots > 0) return e->fail(EMU_ERR_STATE, "prefill in slot mode: use emu_llm_join (emu_llm_reset leaves slot mode)");
  if (B > c.llm_max_batch) return e->fail(EMU_ERR_INVALID, "batch exceeds llm_max_batch");
  if (e->cur_len + N > c.llm_max_seq) return e->fail(EMU_ERR_INVALID, "sequence exceeds llm_max_seq");
  if (e->cur_len > 0 && B != e->cache_B) return e->fail(EMU_ERR_STATE, "batch differs from cached batch");
  if (e->cur_len > 0 && e->kv_indir_dirty)
    return e->fail(EMU_ERR_STATE, "a further prompt chunk after a beam re-parent needs EMU_KV_COPY=1 (the prefill attention reads rows directly)");
  const int pos0 = e->cur_len;
  EMU_TRY(prefill_stage(e, inputs_embeds, (long)B * N, st));
  if (pos0 == 0) {
    if (attention_mask) mask_start_kernel<<<B, 32, 0, st>>>(attention_mask, N, e->d_start, e->d_posoff, hf_positions, 0);
    else cudaMemsetAsync(e->d_start, 0, 2 * kLlmMaxRows * sizeof(int), st);
    count_launch();
    e->cache_B = B;
  }
  EMU_TRY(prefill_layers(e, B, N, pos0, e->d_start, e->d_posoff, st));
  e->cur_len = pos0 + N;
  set_int_kernel<<<1, 32, 0, st>>>(e->d_pos, kLlmMaxRows, e->cur_len);  // slot of the next token
  count_launch();
  return prefill_outputs(e, B, N, last_hidden, logits_last, st);
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
  advance_pos_kernel<<<1, 32, 0, st>>>(e->d_pos, kLlmMaxRows, tp_step_counter(e), e->n_slots > 0 ? e->d_active : nullptr);
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
  advance_pos_kernel<<<1, 32, 0, st>>>(e->d_pos, kLlmMaxRows, tp_step_counter(e), e->n_slots > 0 ? e->d_active : nullptr);
  ++nl;
  *n_launch = nl;
  return EMU_OK;
}

// slot mode's decode rows 0 .. B - 1: B covers the highest live slot and stays within the slots, and every live slot among
// them has room for one more token
static int check_decode_rows(EmuEngine* e, int B, const std::string& none_live) {
  int hi = -1;
  for (int b = 0; b < e->n_slots; ++b)
    if (e->slots[b].live()) hi = b;
  if (hi < 0) return e->fail(EMU_ERR_STATE, none_live);
  if (B <= hi || B > e->n_slots)
    return e->fail(EMU_ERR_INVALID, "slot mode: B = " + std::to_string(B) + " must cover the highest live slot " +
                                        std::to_string(hi) + " and stay within " + std::to_string(e->n_slots) + " slots");
  for (int b = 0; b < B; ++b)
    if (e->slots[b].live() && e->slots[b].len + 1 > e->cfg.llm_max_seq)
      return e->fail(EMU_ERR_INVALID, "KV cache full at slot " + std::to_string(b));
  return EMU_OK;
}

// launch body(stream, &n_launches) — a fixed launch sequence — on st as the CUDA graph cached under key (captured on first use),
// or eagerly with EMU_NO_GRAPH=1 (debugging / parity switch) or without graphs
template <class Body>
static int run_graphed(EmuEngine* e, const EmuEngine::GraphKey& key, cudaStream_t st, Body body) {
  int nl = 0;
  const char* no_graph = getenv("EMU_NO_GRAPH");
  const bool graphable = e->use_graphs && !(no_graph && no_graph[0] == '1');  // NCCL collectives are graph-capturable
  if (!graphable) {
    EMU_TRY(body(st, &nl));
    count_launch(nl);
    return EMU_OK;
  }
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
    int rc = body(e->cap_stream, &nl);
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
  return EMU_OK;
}

extern "C" int emu_llm_decode(EmuEngine* e, const int32_t* token_ids, const void* embeds, const int32_t* beam_src_idx,
                              int B, float* logits, void* hidden, int32_t* next_ids, int ban_id, emu_stream_t stream) {
  if (!e || B < 1 || ((token_ids == nullptr) == (embeds == nullptr))) return EMU_ERR_INVALID;
  EMU_TRY(llm_ready(e));
  const EmuConfig& c = e->cfg;
  cudaStream_t st = (cudaStream_t)stream;
  if (e->n_slots > 0) {
    EMU_TRY(check_decode_rows(e, B, "decode with no live slot"));
  } else {
    if (e->cur_len < 1) return e->fail(EMU_ERR_STATE, "decode before prefill");
    if (B != e->cache_B) return e->fail(EMU_ERR_STATE, "batch differs from cached batch");
    if (e->cur_len + 1 > c.llm_max_seq) return e->fail(EMU_ERR_INVALID, "KV cache full");
  }
  if (beam_src_idx) {
    EMU_TRY(kv_reparent(e, beam_src_idx, B, st));
    count_launch();
  }
  EmuEngine::GraphKey key(B, token_ids, embeds, logits, hidden, next_ids, (const void*)st, ban_id, e->n_slots > 0 ? 1 : 0);
  auto body = [&](cudaStream_t cs, int* nl) {
    return decode_step_body(e, token_ids, embeds, B, logits, hidden, next_ids, ban_id, cs, nl);
  };
  EMU_TRY(run_graphed(e, key, st, body));
  if (e->n_slots > 0) {
    for (int b = 0; b < B; ++b) e->slots[b].advance();
  } else {
    e->cur_len += 1;
  }
  return EMU_OK;
}

// ================================================================================================
// speculative decoding: verify n consecutive tokens of the batch-1 sequence in one weight pass (include/emu_b200_spec.h)
// ================================================================================================
static int spec_alloc(EmuEngine* e) {
  if (e->sp_idx) return EMU_OK;
  const EmuConfig& c = e->cfg;
  bf16* qkv = (bf16*)e->dmalloc((size_t)8 * 3 * e->Hl * c.llm_head_dim * 2);
  float* ws = (float*)e->dmalloc(attn_verify_workspace_bytes(e->Hl, c.llm_head_dim));
  int* counters = (int*)e->dmalloc((size_t)e->Hl * sizeof(int));
  int* idx = (int*)e->dmalloc(16 * sizeof(int));
  if (!qkv || !ws || !counters || !idx) return e->fail(EMU_ERR_NOMEM, "speculative decoding buffers");
  int iota[16];
  for (int i = 0; i < 16; ++i) iota[i] = i;
  if (cudaMemset(counters, 0, (size_t)e->Hl * sizeof(int)) != cudaSuccess ||
      cudaMemcpy(idx, iota, sizeof(iota), cudaMemcpyHostToDevice) != cudaSuccess)
    return e->fail(EMU_ERR_CUDA, "speculative decoding buffers init failed");
  e->sp_qkv = qkv; e->sp_ws = ws; e->sp_counters = counters; e->sp_idx = idx;
  return EMU_OK;
}

// the kernels of one verify (captured into a CUDA graph by emu_llm_verify): the decode step's GEMVs at B = n, the packed
// RoPE / KV append of one segment (cache row 0, positions d_pos[0] ..), the verify attention, and the lm_head of every row
static int verify_body(EmuEngine* e, const int32_t* tokens, int n, float* logits, int32_t* next_ids, int ban_id, int ban_rows,
                       cudaStream_t st, int* n_launch) {
  const EmuConfig& c = e->cfg;
  const int Hd = c.llm_hidden, D = c.llm_head_dim, Hl = e->Hl, Fl = e->Fl;
  const float scale = 1.0f / sqrtf((float)D);
  const int pdl = 1;
  int nl = 1;
  bf16* h = e->dec_h;
  EMU_TRY(embed_gather(e->embed, tokens, h, n, Hd, st));
  for (int l = 0; l < c.llm_layers; ++l) {
    const LlmLayer& L = e->layers[l];
    bf16* kc = kv_layer(e, l, 0);
    bf16* vc = kv_layer(e, l, 1);
    GemvArgs q;
    q.W = L.wqkv; q.N = 3 * Hl * D; q.K = Hd; q.x = h; q.ldx = Hd; q.B = n;
    q.norm_w = L.ln1; q.norm_eps = c.llm_rms_eps; q.y = e->sp_qkv; q.ldy = 3 * Hl * D; q.pdl = pdl;
    EMU_TRY(gemv_bf16(q, st));
    EMU_TRY(rope_kv_write_packed(e->sp_qkv, n, 0, 1, Hl, D, e->rope_cos, e->rope_sin, nullptr, nullptr, nullptr, nullptr,
                                 e->sp_idx, e->d_pos, e->sp_idx + n, e->d_posoff, kc, vc, c.llm_max_seq, st));
    EMU_TRY(attn_verify(e->sp_qkv, 3L * Hl * D, kc, vc, n, Hl, D, c.llm_max_seq, 0, e->d_pos, e->d_start, scale, e->dec_attn,
                        e->sp_ws, e->sp_counters, c.llm_max_seq, st, e->kv_indir));
    GemvArgs o;
    o.W = L.wo; o.N = Hd; o.K = Hl * D; o.x = e->dec_attn; o.ldx = Hl * D; o.B = n; o.pdl = pdl;
    o.residual = h; o.ldr = Hd; o.y = h; o.ldy = Hd;
    EMU_TRY(gemv_bf16(o, st));
    GemvArgs g;
    g.W = L.wgu; g.N = 2 * Fl; g.K = Hd; g.x = h; g.ldx = Hd; g.B = n;
    g.norm_w = L.ln2; g.norm_eps = c.llm_rms_eps; g.mode = EPI_SWIGLU; g.y = e->dec_act; g.ldy = Fl; g.pdl = pdl;
    EMU_TRY(gemv_bf16(g, st));
    GemvArgs d;
    d.W = L.wdown; d.N = Hd; d.K = Fl; d.x = e->dec_act; d.ldx = Fl; d.B = n; d.pdl = pdl;
    d.residual = h; d.ldr = Hd; d.y = h; d.ldy = Hd;
    EMU_TRY(gemv_bf16(d, st));
    nl += 6;
  }
  if (logits || next_ids) {
    float* lg = logits ? logits : e->dec_logits_local;
    GemvArgs g;
    g.W = e->lm_head; g.N = e->Vl; g.K = Hd; g.x = h; g.ldx = Hd; g.B = n;
    g.norm_w = e->final_norm; g.norm_eps = c.llm_rms_eps;
    g.out_fp32 = 1; g.pdl = pdl; g.y = lg; g.ldy = c.llm_vocab;
    EMU_TRY(gemv_bf16(g, st));
    ++nl;
    if (next_ids) {
      if (ban_id >= 0 && ban_rows > 0) {
        argmax_ban_kernel<<<ban_rows, 1, 0, st>>>(lg, c.llm_vocab, ban_id);
        ++nl;
      }
      EMU_TRY(argmax_rows(lg, n, c.llm_vocab, next_ids, st));
      ++nl;
    }
  }
  *n_launch = nl;
  return cudaGetLastError() == cudaSuccess ? EMU_OK : e->fail(EMU_ERR_CUDA, "verify launch failed");
}

extern "C" int emu_llm_verify(EmuEngine* e, const int32_t* tokens, int n, float* logits, int32_t* next_ids, int ban_id,
                              int ban_rows, emu_stream_t stream) {
  if (!e) return EMU_ERR_INVALID;
  if (!tokens) return e->fail(EMU_ERR_INVALID, "verify: tokens is null");
  EMU_TRY(llm_ready(e));
  const EmuConfig& c = e->cfg;
  if (e->n_slots > 0) return e->fail(EMU_ERR_STATE, "verify in slot mode (emu_llm_reset leaves it)");
  if (e->tp_size > 1) return e->fail(EMU_ERR_UNSUPPORTED, "verify under tensor parallelism");
  if (c.llm_head_dim != 64 && c.llm_head_dim != 128)
    return e->fail(EMU_ERR_UNSUPPORTED, "verify needs head_dim 64 or 128");
  if (e->cur_len < 1) return e->fail(EMU_ERR_STATE, "verify before prefill");
  if (e->cache_B != 1) return e->fail(EMU_ERR_INVALID, "verify needs batch 1, the cache holds " + std::to_string(e->cache_B));
  const int n_max = c.llm_max_batch < 8 ? c.llm_max_batch : 8;
  if (n < 1 || n > n_max)
    return e->fail(EMU_ERR_INVALID, "verify: n = " + std::to_string(n) + " outside [1, min(8, llm_max_batch) = " +
                                        std::to_string(n_max) + "]");
  if (ban_rows < 0 || ban_rows > n) return e->fail(EMU_ERR_INVALID, "verify: ban_rows outside [0, n]");
  if (e->cur_len + n > c.llm_max_seq)
    return e->fail(EMU_ERR_INVALID, "KV cache full: verify of " + std::to_string(n) + " rows at length " +
                                        std::to_string(e->cur_len) + " exceeds llm_max_seq " + std::to_string(c.llm_max_seq));
  EMU_TRY(spec_alloc(e));
  cudaStream_t st = (cudaStream_t)stream;
  PdlScope pdl_chain(1);
  EmuEngine::GraphKey key(n, tokens, nullptr, logits, nullptr, next_ids, (const void*)st, ban_id, 16 + ban_rows);
  auto body = [&](cudaStream_t cs, int* nl) { return verify_body(e, tokens, n, logits, next_ids, ban_id, ban_rows, cs, nl); };
  EMU_TRY(run_graphed(e, key, st, body));
  e->spec_n = n;
  e->spec_len = e->cur_len;
  return EMU_OK;
}

extern "C" int emu_llm_commit(EmuEngine* e, int m, emu_stream_t stream) {
  if (!e) return EMU_ERR_INVALID;
  if (e->spec_n < 1 || e->n_slots > 0 || e->spec_len != e->cur_len)
    return e->fail(EMU_ERR_STATE, "commit without a verify since the cache last changed");
  if (m < 1 || m > e->spec_n)
    return e->fail(EMU_ERR_INVALID, "commit: m = " + std::to_string(m) + " outside [1, " + std::to_string(e->spec_n) + "]");
  e->cur_len += m;
  e->spec_n = 0;
  set_int_kernel<<<1, 32, 0, (cudaStream_t)stream>>>(e->d_pos, kLlmMaxRows, e->cur_len);
  count_launch();
  return cudaGetLastError() == cudaSuccess ? EMU_OK : e->fail(EMU_ERR_CUDA, "commit failed");
}

// ================================================================================================
// slot mode: continuous batching (include/emu_b200_slots.h)
// ================================================================================================
static int slot_mode_ok(EmuEngine* e) {
  if (e->cfg.llm_layers < 1) return e->fail(EMU_ERR_STATE, "engine has no LLM");
  if (e->tp_size > 1) return e->fail(EMU_ERR_UNSUPPORTED, "slot mode under tensor parallelism");
  if (e->n_slots < 1) return e->fail(EMU_ERR_STATE, "not in slot mode (emu_llm_slots_begin)");
  return EMU_OK;
}

// a host slot list: n in [1, n_slots], every index in range, distinct, and free (want_free) or live
static int check_slots(EmuEngine* e, const int32_t* slots, int n, bool want_free, SlotList* out) {
  if (n < 1 || n > e->n_slots) return e->fail(EMU_ERR_INVALID, "slot count " + std::to_string(n) + " out of range");
  for (int i = 0; i < n; ++i) {
    const int s = slots[i];
    if (s < 0 || s >= e->n_slots)
      return e->fail(EMU_ERR_INVALID, "slot " + std::to_string(s) + " out of range [0, " + std::to_string(e->n_slots) + ")");
    for (int j = 0; j < i; ++j)
      if (slots[j] == s) return e->fail(EMU_ERR_INVALID, "slot " + std::to_string(s) + " named twice");
    if (want_free && e->slots[s].live()) return e->fail(EMU_ERR_STATE, "slot " + std::to_string(s) + " is occupied");
    if (!want_free && !e->slots[s].live()) return e->fail(EMU_ERR_STATE, "slot " + std::to_string(s) + " is free");
    out->r[i] = s;
  }
  return EMU_OK;
}

// a beam group leaves together: its slots' table rows point into each other
static int check_groups_leave(EmuEngine* e, const SlotList& rows, int n) {
  for (int b = 0; b < e->n_slots; ++b) {
    if (!e->slots[b].live()) continue;
    bool named = false, group_named = false;
    for (int i = 0; i < n; ++i) {
      named |= rows.r[i] == b;
      group_named |= e->slots[rows.r[i]].group == e->slots[b].group;
    }
    if (group_named && !named)
      return e->fail(EMU_ERR_STATE, "slot " + std::to_string(b) + " belongs to a leaving beam group and must leave with it");
  }
  return EMU_OK;
}

// the segments of a slot-mode prefill: free slot slot.r[i] continues after its first prefix.r[i] kept positions with
// n_new.r[i] tokens and ends live (final_.r[i]) or kept at prefix + n_new
struct Segments {
  int n = 0;
  SlotList slot, prefix, n_new, final_;
};

// slot mode's one prefill path, behind emu_llm_join, emu_llm_extend and emu_llm_step, in one pass over the weights: B decode
// rows (token_ids, beams re-parented by beam_src_idx first; B may be 0), then the segments' tokens packed back to back.
// Segment i's embeddings are rows [i * ld, i * ld + n_new[i]) of embeds (ld = 0: already packed).  mask [n, N], every segment
// starting from nothing with N tokens: the left-pad starts and HF position offsets.  logits [B, vocab] of the decode rows
// and logits_last [n, vocab] of each segment's last token, either may be null.  `what` names the call in a CUDA failure.
// hidden_rows [n_slots, hidden] (or null): each segment's last row after the final norm, at row slot.r[i] (the rows of the
// other slots are scratch: they are normed in place too).
static int slot_prefill(EmuEngine* e, const int32_t* token_ids, const int32_t* beam_src_idx, int B, float* logits,
                        const Segments& sg, const void* embeds, int ld, const int32_t* mask, float* logits_last,
                        const char* what, cudaStream_t st, bf16* hidden_rows = nullptr) {
  const EmuConfig& c = e->cfg;
  const int Hd = c.llm_hidden, n = sg.n, K = kLlmMaxRows;
  int host_idx[6 * K];  // cache rows, prefixes, token counts, first packed rows, then the rows whose logits are read
  SlotList len;
  MixedRows m;
  m.B = B; m.n = n; m.M = B; m.max_new = 0; m.Nk = 0;
  for (int i = 0; i < n; ++i) {
    const int k = sg.n_new.r[i];
    host_idx[i] = sg.slot.r[i];
    host_idx[K + i] = sg.prefix.r[i];
    host_idx[2 * K + i] = k;
    host_idx[3 * K + i] = m.M;
    len.r[i] = sg.prefix.r[i] + k;
    m.M += k;
    m.max_new = k > m.max_new ? k : m.max_new;
    m.Nk = len.r[i] > m.Nk ? len.r[i] : m.Nk;
  }
  int n_out = 0;  // logits rows: the decode rows, then each segment's last row
  if (logits)
    for (int b = 0; b < B; ++b) host_idx[4 * K + n_out++] = b;
  if (logits_last)
    for (int i = 0; i < n; ++i) host_idx[4 * K + n_out++] = host_idx[3 * K + i] + sg.n_new.r[i] - 1;
  EMU_TRY(e->ensure(e->step_idx, sizeof(host_idx)));
  int* d_idx = (int*)e->step_idx.p;
  m.seg_row = d_idx;
  m.seg_q0 = d_idx + K;
  m.seg_new = d_idx + 2 * K;
  m.seg_row0 = d_idx + 3 * K;
  PdlScope pdl_chain(1);
  if (cudaMemcpyAsync(d_idx, host_idx, sizeof(host_idx), cudaMemcpyHostToDevice, st) != cudaSuccess)
    return e->fail(EMU_ERR_CUDA, "slot list upload failed");
  EMU_TRY(prefill_stage(e, nullptr, m.M, st));
  bf16* h = (bf16*)e->pf_h.p;
  for (int i = 0; i < (ld > 0 ? n : 1); ++i) {  // one copy per segment; packed embeddings in one
    const long dst = ld > 0 ? host_idx[3 * K + i] : B, rows = ld > 0 ? sg.n_new.r[i] : m.M - B;
    if (cudaMemcpyAsync(h + dst * Hd, (const bf16*)embeds + (long)i * ld * Hd, (size_t)rows * Hd * 2, cudaMemcpyDeviceToDevice,
                        st) != cudaSuccess)
      return e->fail(EMU_ERR_CUDA, "embeds copy failed");
  }
  if (B > 0) {
    EMU_TRY(embed_gather(e->embed, token_ids, h, B, Hd, st));
    count_launch();
  }
  if (beam_src_idx) {
    EMU_TRY(kv_reparent(e, beam_src_idx, B, st));
    count_launch();
  }
  slot_resume_begin_kernel<<<1, 32, 0, st>>>(sg.slot, sg.prefix, e->d_kept_start, e->d_kept_posoff, e->d_join_start,
                                             e->d_join_posoff, n);
  if (mask) mask_start_kernel<<<n, 32, 0, st>>>(mask, sg.n_new.r[0], e->d_join_start, e->d_join_posoff, 1, 0);
  count_launch(mask ? 2 : 1);
  EMU_TRY(prefill_layers(e, 0, 0, 0, nullptr, nullptr, st, &m));
  // live decode slots advance (before the segments' slots may become live), then the segments' slots take their state
  if (B > 0) advance_pos_kernel<<<1, 32, 0, st>>>(e->d_pos, B, nullptr, e->d_active);
  slot_step_end_kernel<<<n, 256, 0, st>>>(sg.slot, len, sg.final_, e->d_join_start, e->d_join_posoff, e->d_pos, e->d_start,
                                          e->d_posoff, e->d_active, e->d_kept_start, e->d_kept_posoff, e->kv_indir, c.llm_max_seq);
  count_launch(B > 0 ? 2 : 1);
  if (cudaGetLastError() != cudaSuccess) return e->fail(EMU_ERR_CUDA, std::string(what) + " failed");
  for (int b = 0; b < B; ++b) e->slots[b].advance();
  for (int i = 0; i < n; ++i) {
    Slot& s = e->slots[sg.slot.r[i]];
    if (sg.final_.r[i]) s.set_live(sg.slot.r[i], len.r[i]);
    else s.set_kept(len.r[i]);
  }
  if (hidden_rows) {  // row by row, as the prefill's last_hidden: a row's bits do not depend on the others
    gather_last_to_slot_kernel<<<n, 128, 0, st>>>(h, Hd, m.seg_row, m.seg_new, m.seg_row0, hidden_rows);
    count_launch();
    if (cudaGetLastError() != cudaSuccess) return e->fail(EMU_ERR_CUDA, std::string(what) + ": last-row gather failed");
    EMU_TRY(rmsnorm(hidden_rows, e->final_norm, hidden_rows, e->n_slots, Hd, c.llm_rms_eps, 0, st));
    count_launch();
  }
  if (n_out == 0) return EMU_OK;
  // the rows' logits in one pass over lm_head, written straight to the one output asked for, or split to both
  float* out = logits ? logits : logits_last;
  if (logits && logits_last) {
    EMU_TRY(e->ensure(e->step_logits, (size_t)n_out * c.llm_vocab * sizeof(float)));
    out = (float*)e->step_logits.p;
  }
  EMU_TRY(prefill_outputs(e, n_out, 1, nullptr, out, st, d_idx + 4 * K));
  if (logits && logits_last) {
    const size_t row_bytes = (size_t)c.llm_vocab * sizeof(float);
    if (cudaMemcpyAsync(logits, out, B * row_bytes, cudaMemcpyDeviceToDevice, st) != cudaSuccess)
      return e->fail(EMU_ERR_CUDA, "decode logits copy failed");
    if (cudaMemcpyAsync(logits_last, out + (size_t)B * c.llm_vocab, n * row_bytes, cudaMemcpyDeviceToDevice, st) != cudaSuccess)
      return e->fail(EMU_ERR_CUDA, "segment logits copy failed");
  }
  return EMU_OK;
}

extern "C" int emu_llm_slots_begin(EmuEngine* e, int n_slots, emu_stream_t s) {
  if (!e) return EMU_ERR_INVALID;
  const EmuConfig& c = e->cfg;
  if (c.llm_layers < 1) return e->fail(EMU_ERR_STATE, "engine has no LLM");
  if (n_slots < 1 || n_slots > c.llm_max_batch)
    return e->fail(EMU_ERR_INVALID, "n_slots = " + std::to_string(n_slots) + " must be in [1, llm_max_batch = " +
                                        std::to_string(c.llm_max_batch) + "]");
  if (e->tp_size > 1) return e->fail(EMU_ERR_UNSUPPORTED, "slot mode under tensor parallelism");
  if (e->kv_copy) return e->fail(EMU_ERR_UNSUPPORTED, "slot mode with EMU_KV_COPY=1 (slots re-parent through the row table)");
  EMU_TRY(emu_llm_reset(e, s));
  if (cudaMemsetAsync(e->d_active, 0, kLlmMaxRows * sizeof(int), (cudaStream_t)s) != cudaSuccess)
    return e->fail(EMU_ERR_CUDA, "slot state reset failed");
  e->n_slots = n_slots;
  e->slots.assign(n_slots, Slot());
  e->kv_indir_dirty = true;  // joins, forks and leaves rewrite table rows: emu_llm_reset restores the identity
  return EMU_OK;
}

extern "C" int emu_llm_join(EmuEngine* e, const int32_t* host_slots, int n, const void* inputs_embeds,
                            const int32_t* attention_mask, int N, float* logits_last, emu_stream_t stream) {
  if (!e || !host_slots || !inputs_embeds || n < 1 || N < 1) return EMU_ERR_INVALID;
  EMU_TRY(slot_mode_ok(e));
  EMU_TRY(llm_ready(e));
  const EmuConfig& c = e->cfg;
  if (N > c.llm_max_seq) return e->fail(EMU_ERR_INVALID, "prompt of " + std::to_string(N) + " tokens exceeds llm_max_seq");
  Segments sg;
  sg.n = n;
  EMU_TRY(check_slots(e, host_slots, n, true, &sg.slot));
  for (int i = 0; i < n; ++i) {
    sg.prefix.r[i] = 0;
    sg.n_new.r[i] = N;
    sg.final_.r[i] = 1;
  }
  return slot_prefill(e, nullptr, nullptr, 0, nullptr, sg, inputs_embeds, 0, attention_mask, logits_last, "slot join",
                      (cudaStream_t)stream);
}

extern "C" int emu_llm_fork(EmuEngine* e, int src_slot, const int32_t* host_dst_slots, int n, emu_stream_t stream) {
  if (!e || !host_dst_slots || n < 1) return EMU_ERR_INVALID;
  EMU_TRY(slot_mode_ok(e));
  if (src_slot < 0 || src_slot >= e->n_slots) return e->fail(EMU_ERR_INVALID, "source slot " + std::to_string(src_slot) + " out of range");
  if (!e->slots[src_slot].live()) return e->fail(EMU_ERR_STATE, "source slot " + std::to_string(src_slot) + " is free");
  SlotList dst;
  EMU_TRY(check_slots(e, host_dst_slots, n, true, &dst));
  const EmuConfig& c = e->cfg;
  slot_fork_kernel<<<n, 256, 0, (cudaStream_t)stream>>>(src_slot, dst, e->d_pos, e->d_start, e->d_posoff, e->d_active, e->kv_indir,
                                                        c.llm_max_seq);
  count_launch();
  if (cudaGetLastError() != cudaSuccess) return e->fail(EMU_ERR_CUDA, "slot fork failed");
  for (int i = 0; i < n; ++i) e->slots[dst.r[i]].set_fork(e->slots[src_slot]);
  e->slots[src_slot].grows = false;  // beam re-parenting scatters the group's new positions over its rows
  return EMU_OK;
}

extern "C" int emu_llm_leave(EmuEngine* e, const int32_t* host_slots, int n, emu_stream_t stream) {
  static const int32_t keep_none[kLlmMaxRows] = {};  // n is checked against n_slots <= kLlmMaxRows before it is read
  return emu_llm_leave_keep(e, host_slots, keep_none, n, stream);
}

extern "C" int emu_llm_slot_len(EmuEngine* e, int slot) {
  if (!e || e->n_slots < 1 || slot < 0 || slot >= e->n_slots) return -1;
  return e->slots[slot].len;
}

// ================================================================================================
// prefix caching: kept slots and per-slot continuation (include/emu_b200_prefix.h)
// ================================================================================================
extern "C" int emu_llm_leave_keep(EmuEngine* e, const int32_t* host_slots, const int32_t* host_keep, int n, emu_stream_t stream) {
  if (!e || !host_slots || !host_keep || n < 1) return EMU_ERR_INVALID;
  EMU_TRY(slot_mode_ok(e));
  SlotList rows, keep;
  EMU_TRY(check_slots(e, host_slots, n, false, &rows));
  EMU_TRY(check_groups_leave(e, rows, n));
  const EmuConfig& c = e->cfg;
  for (int i = 0; i < n; ++i) {
    const int s = rows.r[i], k = host_keep[i];
    const int own = e->slots[s].own;
    if (k < 0 || k > own || k > c.llm_max_seq - 1)
      return e->fail(EMU_ERR_INVALID, "slot " + std::to_string(s) + " may keep 0 .. " +
                                          std::to_string(own < c.llm_max_seq - 1 ? own : c.llm_max_seq - 1) +
                                          " positions (its own-row length " + std::to_string(own) + "), asked for " +
                                          std::to_string(k));
    keep.r[i] = k;
  }
  slot_keep_kernel<<<n, 256, 0, (cudaStream_t)stream>>>(rows, keep, e->d_pos, e->d_start, e->d_posoff, e->d_active, e->d_kept_start,
                                                        e->d_kept_posoff, e->kv_indir, c.llm_max_seq);
  count_launch();
  if (cudaGetLastError() != cudaSuccess) return e->fail(EMU_ERR_CUDA, "slot leave failed");
  for (int i = 0; i < n; ++i) e->slots[rows.r[i]].set_kept(keep.r[i]);
  return EMU_OK;
}

extern "C" int emu_llm_slot_kept(EmuEngine* e, int slot) {
  if (!e || e->n_slots < 1 || slot < 0 || slot >= e->n_slots) return -1;
  return e->slots[slot].kept;
}

extern "C" int emu_llm_copy_prefix(EmuEngine* e, int src_slot, int dst_slot, int P, emu_stream_t stream) {
  if (!e) return EMU_ERR_INVALID;
  EMU_TRY(slot_mode_ok(e));
  const EmuConfig& c = e->cfg;
  if (src_slot < 0 || src_slot >= e->n_slots) return e->fail(EMU_ERR_INVALID, "source slot " + std::to_string(src_slot) + " out of range");
  if (dst_slot < 0 || dst_slot >= e->n_slots)
    return e->fail(EMU_ERR_INVALID, "destination slot " + std::to_string(dst_slot) + " out of range");
  if (dst_slot == src_slot) return e->fail(EMU_ERR_INVALID, "slot " + std::to_string(src_slot) + " copied onto itself");
  if (e->slots[dst_slot].live()) return e->fail(EMU_ERR_STATE, "destination slot " + std::to_string(dst_slot) + " is occupied");
  const bool live = e->slots[src_slot].live();
  const int avail = live ? e->slots[src_slot].own : e->slots[src_slot].kept;
  if (!live && avail == 0) return e->fail(EMU_ERR_STATE, "source slot " + std::to_string(src_slot) + " is free and keeps nothing");
  if (P < 1 || P > avail || P > c.llm_max_seq - 1)
    return e->fail(EMU_ERR_INVALID, "slot " + std::to_string(src_slot) + " holds " + std::to_string(avail) +
                                        " positions of its own row, asked to copy " + std::to_string(P));
  cudaStream_t st = (cudaStream_t)stream;
  EMU_TRY(kv_prefix_copy(e->kv, (long)c.llm_layers * 2, c.llm_max_batch, e->Hl, c.llm_head_dim, c.llm_max_seq, src_slot, dst_slot, P,
                         st));
  slot_copy_state_kernel<<<1, 256, 0, st>>>(src_slot, live ? 0 : 1, dst_slot, P, e->d_pos, e->d_start, e->d_posoff, e->d_active,
                                            e->d_kept_start, e->d_kept_posoff, e->kv_indir, c.llm_max_seq);
  count_launch(2);
  if (cudaGetLastError() != cudaSuccess) return e->fail(EMU_ERR_CUDA, "prefix copy failed");
  e->slots[dst_slot].set_kept(P);
  return EMU_OK;
}

extern "C" int emu_llm_extend(EmuEngine* e, const int32_t* host_slots, const int32_t* host_prefix, const int32_t* host_new, int n,
                              const void* inputs_embeds, int N, float* logits_last, emu_stream_t stream) {
  if (!e || !host_slots || !host_prefix || !host_new || !inputs_embeds || n < 1 || N < 1) return EMU_ERR_INVALID;
  EMU_TRY(slot_mode_ok(e));
  EMU_TRY(llm_ready(e));
  const EmuConfig& c = e->cfg;
  if (N > c.llm_max_seq) return e->fail(EMU_ERR_INVALID, "suffix of " + std::to_string(N) + " tokens exceeds llm_max_seq");
  Segments sg;
  sg.n = n;
  EMU_TRY(check_slots(e, host_slots, n, true, &sg.slot));
  for (int i = 0; i < n; ++i) {
    const int s = sg.slot.r[i], p = host_prefix[i], k = host_new[i];
    if (p < 0 || p > e->slots[s].kept)
      return e->fail(EMU_ERR_INVALID, "slot " + std::to_string(s) + " keeps " + std::to_string(e->slots[s].kept) +
                                          " positions, asked to resume at " + std::to_string(p));
    if (k < 1 || k > N)
      return e->fail(EMU_ERR_INVALID, "slot " + std::to_string(s) + ": " + std::to_string(k) + " new tokens, N = " + std::to_string(N));
    if (p + k > c.llm_max_seq)
      return e->fail(EMU_ERR_INVALID, "slot " + std::to_string(s) + ": " + std::to_string(p) + " + " + std::to_string(k) +
                                          " positions exceed llm_max_seq");
    sg.prefix.r[i] = p;
    sg.n_new.r[i] = k;
    sg.final_.r[i] = 1;
  }
  // the right-padded [n, N] rows are compacted as they are staged: no kernel sees a padding row
  return slot_prefill(e, nullptr, nullptr, 0, nullptr, sg, inputs_embeds, N, nullptr, logits_last, "slot extend",
                      (cudaStream_t)stream);
}

extern "C" int emu_llm_kv_cache(EmuEngine* e, void** kv, int64_t* dims5) {
  if (!e || !kv || !dims5) return EMU_ERR_INVALID;
  const EmuConfig& c = e->cfg;
  if (c.llm_layers < 1 || !e->kv) return e->fail(EMU_ERR_STATE, "engine has no LLM");
  *kv = e->kv;
  dims5[0] = (int64_t)c.llm_layers * 2;
  dims5[1] = c.llm_max_batch;
  dims5[2] = e->Hl;
  dims5[3] = c.llm_max_seq;
  dims5[4] = c.llm_head_dim;
  return EMU_OK;
}

// ================================================================================================
// chunked prefill: the mixed decode + prefill step (include/emu_b200_chunked.h)
// ================================================================================================
extern "C" int emu_llm_step(EmuEngine* e, const int32_t* token_ids, const int32_t* beam_src_idx, int B, float* logits,
                            const int32_t* host_slots, const int32_t* host_prefix, const int32_t* host_new, const int32_t* host_final,
                            int n, const void* embeds, float* logits_last, emu_stream_t stream) {
  if (!e || !host_slots || !host_prefix || !host_new || !host_final || !embeds || n < 1 || B < 0) return EMU_ERR_INVALID;
  if (B > 0 && !token_ids) return EMU_ERR_INVALID;
  if (B == 0 && (beam_src_idx || logits)) return EMU_ERR_INVALID;
  EMU_TRY(slot_mode_ok(e));
  EMU_TRY(llm_ready(e));
  const EmuConfig& c = e->cfg;
  if (B > 0) EMU_TRY(check_decode_rows(e, B, "a decode part of " + std::to_string(B) + " rows with no live slot"));
  // the segments: as emu_llm_extend, each ending live (final) or kept
  Segments sg;
  sg.n = n;
  EMU_TRY(check_slots(e, host_slots, n, true, &sg.slot));
  for (int i = 0; i < n; ++i) {
    const int s = sg.slot.r[i], p = host_prefix[i], k = host_new[i], f = host_final[i];
    if (f != 0 && f != 1) return e->fail(EMU_ERR_INVALID, "slot " + std::to_string(s) + ": final must be 0 or 1, got " + std::to_string(f));
    if (p < 0 || p > e->slots[s].kept)
      return e->fail(EMU_ERR_INVALID, "slot " + std::to_string(s) + " keeps " + std::to_string(e->slots[s].kept) +
                                          " positions, asked to resume at " + std::to_string(p));
    const int room = f ? c.llm_max_seq : c.llm_max_seq - 1;  // a slot left mid-prefill is kept: at most llm_max_seq - 1
    if (k < 1 || k > room - p)
      return e->fail(EMU_ERR_INVALID, "slot " + std::to_string(s) + ": " + std::to_string(k) + " new tokens after " + std::to_string(p) +
                                          " must be in [1, " + std::to_string(room - p) + "] (" + (f ? "final" : "not final") + ")");
    sg.prefix.r[i] = p;
    sg.n_new.r[i] = k;
    sg.final_.r[i] = f;
  }
  return slot_prefill(e, token_ids, beam_src_idx, B, logits, sg, embeds, 0, nullptr, logits_last, "mixed step", (cudaStream_t)stream);
}

// ================================================================================================
// regression slots: Emu2-Gen's prompt encoding in slot mode (include/emu_b200_regress.h)
// ================================================================================================
// project_down and project_up chain hidden -> width -> hidden
static int regress_ready(EmuEngine* e) {
  const int Hd = e->cfg.llm_hidden;
  if (!e->proj_up || !e->proj_down) return e->fail(EMU_ERR_STATE, "regression slots need the project_up and project_down weights");
  if (e->proj_down_in != Hd || e->proj_up_out != Hd || e->proj_up_in != e->proj_down_out)
    return e->fail(EMU_ERR_STATE, "project_down [" + std::to_string(e->proj_down_out) + ", " + std::to_string(e->proj_down_in) +
                                      "] and project_up [" + std::to_string(e->proj_up_out) + ", " + std::to_string(e->proj_up_in) +
                                      "] do not chain through hidden " + std::to_string(Hd));
  if (e->proj_down_out % 8)
    return e->fail(EMU_ERR_UNSUPPORTED, "regression width " + std::to_string(e->proj_down_out) + " is not a multiple of 8");
  return EMU_OK;
}

// the regression buffers, allocated once at kLlmMaxRows rows so the pointers the step graphs bake in never change; zeroed
static int regress_alloc(EmuEngine* e, cudaStream_t st) {
  if (e->rg_fb) return EMU_OK;
  const size_t K = kLlmMaxRows, wb = K * e->proj_down_out * 2, hb = K * e->cfg.llm_hidden * 2;
  bf16 *fb = (bf16*)e->dmalloc(wb), *r = (bf16*)e->dmalloc(wb), *x = (bf16*)e->dmalloc(hb), *h = (bf16*)e->dmalloc(hb);
  int* k = (int*)e->dmalloc(K * sizeof(int));
  if (!fb || !r || !x || !h || !k) return e->fail(EMU_ERR_NOMEM, "regression buffers");
  if (cudaMemsetAsync(fb, 0, wb, st) != cudaSuccess || cudaMemsetAsync(r, 0, wb, st) != cudaSuccess ||
      cudaMemsetAsync(x, 0, hb, st) != cudaSuccess || cudaMemsetAsync(h, 0, hb, st) != cudaSuccess ||
      cudaMemsetAsync(k, 0, K * sizeof(int), st) != cudaSuccess)
    return e->fail(EMU_ERR_CUDA, "regression buffers reset failed");
  e->rg_fb = fb; e->rg_r = r; e->rg_x = x; e->rg_h = h; e->rg_k = k;
  return EMU_OK;
}

extern "C" int emu_llm_regress_join(EmuEngine* e, const int32_t* host_slots, const int32_t* host_new, int n, const void* embeds,
                                    void* out, int L, emu_stream_t stream) {
  if (!e || !host_slots || !host_new || !embeds || !out || n < 1 || n > kLlmMaxRows || L < 1) return EMU_ERR_INVALID;
  for (int i = 0; i < n; ++i)
    if (host_slots[i] < 0 || host_slots[i] >= kLlmMaxRows || host_new[i] < 1) return EMU_ERR_INVALID;
  if (e->kv_copy) return e->fail(EMU_ERR_UNSUPPORTED, "regression slots with EMU_KV_COPY=1 (no slot mode)");
  EMU_TRY(slot_mode_ok(e));
  EMU_TRY(llm_ready(e));
  EMU_TRY(regress_ready(e));
  const EmuConfig& c = e->cfg;
  Segments sg;
  sg.n = n;
  EMU_TRY(check_slots(e, host_slots, n, true, &sg.slot));
  for (int i = 0; i < n; ++i) {
    if (host_new[i] > c.llm_max_seq)
      return e->fail(EMU_ERR_INVALID, "slot " + std::to_string(sg.slot.r[i]) + ": prompt of " + std::to_string(host_new[i]) +
                                          " tokens exceeds llm_max_seq = " + std::to_string(c.llm_max_seq));
    sg.prefix.r[i] = 0;
    sg.n_new.r[i] = host_new[i];
    sg.final_.r[i] = 1;
  }
  cudaStream_t st = (cudaStream_t)stream;
  EMU_TRY(regress_alloc(e, st));
  EMU_TRY(slot_prefill(e, nullptr, nullptr, 0, nullptr, sg, embeds, 0, nullptr, nullptr, "regression join", st, e->rg_h));
  // always n_slots rows: a segment's projection is the same bits however many joined with it
  EMU_TRY(project_rows(e, 1, e->rg_h, e->n_slots, e->rg_r, st));
  regress_emit_kernel<<<n, 128, 0, st>>>(e->rg_r, e->rg_fb, e->rg_k, (bf16*)out, L, e->proj_down_out, sg.slot, n, e->d_active);
  count_launch(2);
  if (cudaGetLastError() != cudaSuccess) return e->fail(EMU_ERR_CUDA, "regression join failed");
  for (int i = 0; i < n; ++i) e->slots[sg.slot.r[i]].regress = true;
  return EMU_OK;
}

extern "C" int emu_llm_regress_step(EmuEngine* e, int B, void* out, int L, emu_stream_t stream) {
  if (!e || !out || B < 1 || B > kLlmMaxRows || L < 1) return EMU_ERR_INVALID;
  if (e->kv_copy) return e->fail(EMU_ERR_UNSUPPORTED, "regression slots with EMU_KV_COPY=1 (no slot mode)");
  EMU_TRY(slot_mode_ok(e));
  EMU_TRY(llm_ready(e));
  EMU_TRY(regress_ready(e));
  EMU_TRY(check_decode_rows(e, B, "regression step with no live slot"));
  for (int b = 0; b < B; ++b)
    if (e->slots[b].live() && !e->slots[b].regress)
      return e->fail(EMU_ERR_STATE, "slot " + std::to_string(b) + " is live but did not join through emu_llm_regress_join");
  cudaStream_t st = (cudaStream_t)stream;
  const int w = e->proj_down_out;
  auto body = [&](cudaStream_t cs, int* nl) {
    int n_dec = 0;
    EMU_TRY(project_rows(e, 0, e->rg_fb, B, e->rg_x, cs));
    EMU_TRY(decode_step_body(e, nullptr, e->rg_x, B, nullptr, e->rg_h, nullptr, -1, cs, &n_dec));
    EMU_TRY(project_rows(e, 1, e->rg_h, B, e->rg_r, cs));
    regress_emit_kernel<<<B, 128, 0, cs>>>(e->rg_r, e->rg_fb, e->rg_k, (bf16*)out, L, w, SlotList{}, 0, e->d_active);
    *nl = n_dec + 3;
    return cudaGetLastError() == cudaSuccess ? EMU_OK : e->fail(EMU_ERR_CUDA, "regression step failed");
  };
  EmuEngine::GraphKey key(B, nullptr, e->rg_x, nullptr, out, nullptr, (const void*)st, L, 2);
  EMU_TRY(run_graphed(e, key, st, body));
  for (int b = 0; b < B; ++b) e->slots[b].advance();
  return EMU_OK;
}
