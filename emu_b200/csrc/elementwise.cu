// emu_b200 — bandwidth-bound glue kernels of the generate path (norms, RoPE + KV-cache writes, embedding gather,
// argmax, ViT patch gather / CLS+pos assembly / average pooling, beam KV reorder).  All are 16-byte vectorised,
// one pass over the data, fp32 math with the reference's bf16 rounding points.
#include <cstdlib>

#include "common.cuh"
#include "ops.h"

namespace emu {

thread_local int g_pdl_chain = 0;
PdlScope::PdlScope(int on) {
  static int disabled = -1;
  if (disabled < 0) {
    const char* v = getenv("EMU_NO_PDL");
    disabled = (v && atoi(v) != 0) ? 1 : 0;
  }
  prev = g_pdl_chain;
  g_pdl_chain = (on && !disabled) ? 1 : 0;
}

// ----------------------------------------------------------------------------------------------
// RMSNorm (HF LlamaRMSNorm / T5LayerNorm — Emu1/models/modeling_t5.py:318-331): one CTA per row
// ----------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) rmsnorm_kernel(const bf16* __restrict__ x, const bf16* __restrict__ w,
                                                      bf16* __restrict__ y, int cols, float eps) {
  __shared__ float red[33];
  const long row = blockIdx.x;
  const uint4* src = reinterpret_cast<const uint4*>(x + row * cols);
  const uint4* wsrc = reinterpret_cast<const uint4*>(w);
  uint4* dst = reinterpret_cast<uint4*>(y + row * cols);
  const int nv = cols >> 3;
  float s = 0.f;
  for (int i = threadIdx.x; i < nv; i += blockDim.x) {
    const uint4 v = src[i];
    const uint32_t v4[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float lo = bf16_lo(v4[j]), hi = bf16_hi(v4[j]);
      s += lo * lo + hi * hi;
    }
  }
  const float tot = block_sum(s, red);
  const float rstd = rsqrtf(tot / (float)cols + eps);
  for (int i = threadIdx.x; i < nv; i += blockDim.x) {
    const uint4 v = src[i], ww = wsrc[i];
    const uint32_t v4[4] = {v.x, v.y, v.z, v.w}, w4[4] = {ww.x, ww.y, ww.z, ww.w};
    uint32_t o[4];
#pragma unroll
    for (int j = 0; j < 4; ++j)
      o[j] = pack_bf16(round_bf16(bf16_lo(v4[j]) * rstd) * bf16_lo(w4[j]),
                       round_bf16(bf16_hi(v4[j]) * rstd) * bf16_hi(w4[j]));
    dst[i] = make_uint4(o[0], o[1], o[2], o[3]);
  }
}

int rmsnorm(const bf16* x, const bf16* w, bf16* y, int rows, int cols, float eps, int, cudaStream_t st) {
  if (cols % 8) return EMU_ERR_INVALID;
  rmsnorm_kernel<<<rows, 256, 0, st>>>(x, w, y, cols, eps);
  return cudaGetLastError() == cudaSuccess ? EMU_OK : EMU_ERR_CUDA;
}

// ----------------------------------------------------------------------------------------------
// LayerNorm with fused residual: y = residual + LN(x) (Emu2 post-norm block, Emu2/emu/eva_vit.py:298-300);
// residual == null gives plain LN (Emu1 pre-norm, ln_visual, UNet transformer norms).
// ----------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) layernorm_kernel(const bf16* __restrict__ x, const bf16* __restrict__ w,
                                                        const bf16* __restrict__ b, const bf16* residual, bf16* y,
                                                        int cols, float eps) {
  __shared__ float red[33];
  const long row = blockIdx.x;
  const uint4* src = reinterpret_cast<const uint4*>(x + row * cols);
  const int nv = cols >> 3;
  float s = 0.f;
  for (int i = threadIdx.x; i < nv; i += blockDim.x) {
    const uint4 v = src[i];
    const uint32_t v4[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
    for (int j = 0; j < 4; ++j) s += bf16_lo(v4[j]) + bf16_hi(v4[j]);
  }
  const float mean = block_sum(s, red) / (float)cols;
  float s2 = 0.f;
  for (int i = threadIdx.x; i < nv; i += blockDim.x) {
    const uint4 v = src[i];
    const uint32_t v4[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float lo = bf16_lo(v4[j]) - mean, hi = bf16_hi(v4[j]) - mean;
      s2 += lo * lo + hi * hi;
    }
  }
  const float rstd = rsqrtf(block_sum(s2, red) / (float)cols + eps);
  const uint4* wsrc = reinterpret_cast<const uint4*>(w);
  const uint4* bsrc = reinterpret_cast<const uint4*>(b);
  const uint4* rsrc = residual ? reinterpret_cast<const uint4*>(residual + row * cols) : nullptr;
  uint4* dst = reinterpret_cast<uint4*>(y + row * cols);
  for (int i = threadIdx.x; i < nv; i += blockDim.x) {
    const uint4 v = src[i], ww = wsrc[i];
    const uint4 bb = bsrc ? bsrc[i] : make_uint4(0, 0, 0, 0);
    const uint4 rr = rsrc ? rsrc[i] : make_uint4(0, 0, 0, 0);
    const uint32_t v4[4] = {v.x, v.y, v.z, v.w}, w4[4] = {ww.x, ww.y, ww.z, ww.w}, b4[4] = {bb.x, bb.y, bb.z, bb.w},
                   r4[4] = {rr.x, rr.y, rr.z, rr.w};
    uint32_t o[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      float lo = (bf16_lo(v4[j]) - mean) * rstd * bf16_lo(w4[j]) + bf16_lo(b4[j]);
      float hi = (bf16_hi(v4[j]) - mean) * rstd * bf16_hi(w4[j]) + bf16_hi(b4[j]);
      if (rsrc) {
        lo = round_bf16(lo) + bf16_lo(r4[j]);
        hi = round_bf16(hi) + bf16_hi(r4[j]);
      }
      o[j] = pack_bf16(lo, hi);
    }
    dst[i] = make_uint4(o[0], o[1], o[2], o[3]);
  }
}

// rows of <= 2048 elements: one WARP per row, the row lives in registers (one global read, no block barriers)
__global__ void __launch_bounds__(256) layernorm_warp_kernel(const bf16* __restrict__ x, const bf16* __restrict__ w,
                                                             const bf16* __restrict__ b, const bf16* residual, bf16* y,
                                                             int rows, int cols, float eps, int pdl) {
  if (pdl) {
    pdl_launch_dependents();
    pdl_wait();
  }
  const int lane = threadIdx.x & 31;
  const long row = (long)blockIdx.x * 8 + (threadIdx.x >> 5);
  if (row >= rows) return;
  const int nv = cols >> 3;
  const uint4* src = reinterpret_cast<const uint4*>(x + row * cols);
  uint4 v[8];
  float s = 0.f;
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    const int i = lane + 32 * k;
    v[k] = i < nv ? src[i] : make_uint4(0, 0, 0, 0);
    const uint32_t v4[4] = {v[k].x, v[k].y, v[k].z, v[k].w};
#pragma unroll
    for (int j = 0; j < 4; ++j) s += bf16_lo(v4[j]) + bf16_hi(v4[j]);
  }
  const float mean = warp_sum(s) / (float)cols;
  float s2 = 0.f;
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    if (lane + 32 * k < nv) {
      const uint32_t v4[4] = {v[k].x, v[k].y, v[k].z, v[k].w};
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float lo = bf16_lo(v4[j]) - mean, hi = bf16_hi(v4[j]) - mean;
        s2 += lo * lo + hi * hi;
      }
    }
  }
  const float rstd = rsqrtf(warp_sum(s2) / (float)cols + eps);
  const uint4* wsrc = reinterpret_cast<const uint4*>(w);
  const uint4* bsrc = reinterpret_cast<const uint4*>(b);
  const uint4* rsrc = residual ? reinterpret_cast<const uint4*>(residual + row * cols) : nullptr;
  uint4* dst = reinterpret_cast<uint4*>(y + row * cols);
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    const int i = lane + 32 * k;
    if (i < nv) {
      const uint4 ww = __ldg(wsrc + i);
      const uint4 bb = bsrc ? __ldg(bsrc + i) : make_uint4(0, 0, 0, 0);
      const uint4 rr = rsrc ? rsrc[i] : make_uint4(0, 0, 0, 0);
      const uint32_t v4[4] = {v[k].x, v[k].y, v[k].z, v[k].w}, w4[4] = {ww.x, ww.y, ww.z, ww.w},
                     b4[4] = {bb.x, bb.y, bb.z, bb.w}, r4[4] = {rr.x, rr.y, rr.z, rr.w};
      uint32_t o[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        float lo = (bf16_lo(v4[j]) - mean) * rstd * bf16_lo(w4[j]) + bf16_lo(b4[j]);
        float hi = (bf16_hi(v4[j]) - mean) * rstd * bf16_hi(w4[j]) + bf16_hi(b4[j]);
        if (rsrc) {
          lo = round_bf16(lo) + bf16_lo(r4[j]);
          hi = round_bf16(hi) + bf16_hi(r4[j]);
        }
        o[j] = pack_bf16(lo, hi);
      }
      dst[i] = make_uint4(o[0], o[1], o[2], o[3]);
    }
  }
}

int layernorm(const bf16* x, const bf16* w, const bf16* b, const bf16* residual, bf16* y, int rows, int cols, float eps,
              cudaStream_t st) {
  if (cols % 8) return EMU_ERR_INVALID;
  if (cols <= 2048)
    return launch_kernel(layernorm_warp_kernel, dim3((rows + 7) / 8), dim3(256), 0, st, g_pdl_chain, x, w, b, residual, y,
                         rows, cols, eps, g_pdl_chain);
  layernorm_kernel<<<rows, 256, 0, st>>>(x, w, b, residual, y, cols, eps);
  return cudaGetLastError() == cudaSuccess ? EMU_OK : EMU_ERR_CUDA;
}

// ----------------------------------------------------------------------------------------------
// prefill: RoPE on q (in place) and k, append k/v to the cache.  q/k head dims are pair-interleaved
// (element 2j = original j, 2j+1 = original j + D/2) by the weight packer, so a rotation pair is one 4-byte word.
// ----------------------------------------------------------------------------------------------
__global__ void rope_kv_write_kernel(bf16* qkv, int B, int N, int H, int D, const bf16* __restrict__ cos_t,
                                     const bf16* __restrict__ sin_t, const int* pos_off, int pos0, bf16* k_cache,
                                     bf16* v_cache, int t_max, const int* __restrict__ pos_dev, bf16* q_out,
                                     const int* __restrict__ kv_row) {
  const int half = D >> 1;
  const long total = (long)B * N * H * half;
  for (long idx = blockIdx.x * (long)blockDim.x + threadIdx.x; idx < total; idx += (long)gridDim.x * blockDim.x) {
    const int j = idx % half;
    const int h = (idx / half) % H;
    const int n = (idx / ((long)half * H)) % N;
    const int b = idx / ((long)half * H * N);
    bf16* base = qkv + ((long)b * N + n) * 3 * H * D;
    // CUDA-graphed decode: the cache slot of every row's new token lives on the device (rows differ in slot mode)
    const int p0 = pos_dev ? pos_dev[b] : pos0;
    const int row = kv_row ? kv_row[b] : b;
    int rp = p0 + n - (pos_off ? pos_off[b] : 0);
    rp = rp < 0 ? 0 : rp;
    const float c = __bfloat162float(cos_t[(long)rp * half + j]);
    const float s = __bfloat162float(sin_t[(long)rp * half + j]);
    uint32_t* qp = reinterpret_cast<uint32_t*>(base + h * D + 2 * j);
    const uint32_t qv = *qp;
    const float q1 = bf16_lo(qv), q2 = bf16_hi(qv);
    // decode (N == 1) may want the rotated q compact [B, H*D] for the attention kernel instead of in place
    uint32_t* qd = q_out ? reinterpret_cast<uint32_t*>(q_out + ((long)b * N + n) * H * D + h * D + 2 * j) : qp;
    *qd = pack_bf16(round_bf16(q1 * c) + round_bf16(-q2 * s), round_bf16(q2 * c) + round_bf16(q1 * s));
    const uint32_t kv = *reinterpret_cast<const uint32_t*>(base + (H + h) * D + 2 * j);
    const float k1 = bf16_lo(kv), k2 = bf16_hi(kv);
    const long coff = (((long)row * H + h) * t_max + p0 + n) * D + 2 * j;
    *reinterpret_cast<uint32_t*>(k_cache + coff) =
        pack_bf16(round_bf16(k1 * c) + round_bf16(-k2 * s), round_bf16(k2 * c) + round_bf16(k1 * s));
    *reinterpret_cast<uint32_t*>(v_cache + coff) = *reinterpret_cast<const uint32_t*>(base + (2 * H + h) * D + 2 * j);
  }
}

int rope_kv_write(bf16* qkv, int B, int N, int H, int D, const bf16* cos_t, const bf16* sin_t, const int* pos_off,
                  int pos0, bf16* k_cache, bf16* v_cache, int t_max, cudaStream_t st, const int* pos_dev, bf16* q_out,
                  const int* kv_row) {
  const long total = (long)B * N * H * (D / 2);
  const int grid = (int)((total + 255) / 256 < 4 * kNumSMs ? (total + 255) / 256 : 4 * kNumSMs);
  rope_kv_write_kernel<<<grid, 256, 0, st>>>(qkv, B, N, H, D, cos_t, sin_t, pos_off, pos0, k_cache, v_cache, t_max, pos_dev, q_out,
                                             kv_row);
  return cudaGetLastError() == cudaSuccess ? EMU_OK : EMU_ERR_CUDA;
}

// slot mode (emu_llm_join, emu_llm_extend, emu_llm_step): the M packed rows of a mixed step, one CTA per row.  Row m < B is the decode token of slot m
// (cache slot pos[m], q compact to q_out, k / v only if the slot is live); the rows after it are the segments back to back,
// row j of segment i at cache slot seg_q0[i] + j of row seg_row[i] (q in place).  Same rotation and rounding as above.
__global__ void rope_kv_write_packed_kernel(bf16* qkv, int B, int n, int H, int D, const bf16* __restrict__ cos_t,
                                            const bf16* __restrict__ sin_t, const int* __restrict__ pos,
                                            const int* __restrict__ pos_off, const int* __restrict__ active, bf16* q_out,
                                            const int* __restrict__ seg_row, const int* __restrict__ seg_q0,
                                            const int* __restrict__ seg_new, const int* __restrict__ seg_posoff,
                                            bf16* k_cache, bf16* v_cache, int t_max) {
  const int m = blockIdx.x, half = D >> 1;
  int row, slot, off;
  bool write_kv = true;
  if (m < B) {
    row = m;
    slot = pos[m];
    off = pos_off ? pos_off[m] : 0;
    write_kv = active[m] != 0;
  } else {
    int r = m - B, i = 0;
    while (i < n && r >= seg_new[i]) r -= seg_new[i++];
    if (i == n) return;  // past the last segment
    row = seg_row[i];
    slot = seg_q0[i] + r;
    off = seg_posoff ? seg_posoff[i] : 0;
  }
  bf16* base = qkv + (long)m * 3 * H * D;
  int rp = slot - off;
  rp = rp < 0 ? 0 : rp;
  for (int idx = threadIdx.x; idx < H * half; idx += blockDim.x) {
    const int j = idx % half, h = idx / half;
    const float c = __bfloat162float(cos_t[(long)rp * half + j]);
    const float s = __bfloat162float(sin_t[(long)rp * half + j]);
    uint32_t* qp = reinterpret_cast<uint32_t*>(base + h * D + 2 * j);
    const uint32_t qv = *qp;
    const float q1 = bf16_lo(qv), q2 = bf16_hi(qv);
    uint32_t* qd = m < B ? reinterpret_cast<uint32_t*>(q_out + (long)m * H * D + h * D + 2 * j) : qp;
    *qd = pack_bf16(round_bf16(q1 * c) + round_bf16(-q2 * s), round_bf16(q2 * c) + round_bf16(q1 * s));
    if (!write_kv) continue;
    const uint32_t kv = *reinterpret_cast<const uint32_t*>(base + (H + h) * D + 2 * j);
    const float k1 = bf16_lo(kv), k2 = bf16_hi(kv);
    const long coff = (((long)row * H + h) * t_max + slot) * D + 2 * j;
    *reinterpret_cast<uint32_t*>(k_cache + coff) =
        pack_bf16(round_bf16(k1 * c) + round_bf16(-k2 * s), round_bf16(k2 * c) + round_bf16(k1 * s));
    *reinterpret_cast<uint32_t*>(v_cache + coff) = *reinterpret_cast<const uint32_t*>(base + (2 * H + h) * D + 2 * j);
  }
}

int rope_kv_write_packed(bf16* qkv, int M, int B, int n, int H, int D, const bf16* cos_t, const bf16* sin_t, const int* pos,
                         const int* pos_off, const int* active, bf16* q_out, const int* seg_row, const int* seg_q0,
                         const int* seg_new, const int* seg_posoff, bf16* k_cache, bf16* v_cache, int t_max, cudaStream_t st) {
  // one CTA per row with a thread for each of its H * D / 2 rotation pairs (up to 1024): a short prefill has few rows, and a
  // CTA that loops over its row would leave most of the GPU idle
  const int pairs = H * (D / 2), threads = pairs < 1024 ? (pairs + 31) / 32 * 32 : 1024;
  rope_kv_write_packed_kernel<<<M, threads, 0, st>>>(qkv, B, n, H, D, cos_t, sin_t, pos, pos_off, active, q_out, seg_row, seg_q0,
                                                     seg_new, seg_posoff, k_cache, v_cache, t_max);
  return cudaGetLastError() == cudaSuccess ? EMU_OK : EMU_ERR_CUDA;
}

// prefix caching: cache positions [0, P) of row src -> row dst in every (layer, k/v, head) plane of a [outer][rows][H][t_max][D]
// cache.  Each plane's prefix is P*D contiguous elements, moved as 16-byte words; 4 independent words in flight per thread
// keep enough loads outstanding for a copy that is bound by HBM bandwidth.
__global__ void kv_prefix_copy_kernel(bf16* cache, int rows, int H, int t_max, int D, int src, int dst, long per, long total) {
  const long stride = (long)gridDim.x * blockDim.x;
  for (long i0 = blockIdx.x * (long)blockDim.x + threadIdx.x; i0 < total; i0 += 4 * stride) {
    uint4 v[4];
    long off[4];
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const long idx = i0 + u * stride;
      off[u] = -1;
      if (idx < total) {
        const long w = idx % per, plane = idx / per;  // plane = o * H + h
        const long o = plane / H, h = plane % H;
        const long base = ((o * rows) * H + h) * t_max * D / 8 + w;
        off[u] = base;
        v[u] = __ldg(reinterpret_cast<const uint4*>(cache) + base + (long)src * H * t_max * D / 8);
      }
    }
#pragma unroll
    for (int u = 0; u < 4; ++u)
      if (off[u] >= 0) reinterpret_cast<uint4*>(cache)[off[u] + (long)dst * H * t_max * D / 8] = v[u];
  }
}

int kv_prefix_copy(bf16* cache, long outer, int rows, int H, int D, int t_max, int src, int dst, int P, cudaStream_t st) {
  const long per = (long)P * D / 8;  // 16-byte words per plane
  const long total = outer * H * per;
  const long want = (total + 4 * 256 - 1) / (4 * 256);
  const int grid = (int)(want < 8 * kNumSMs ? want : 8 * kNumSMs);
  kv_prefix_copy_kernel<<<grid, 256, 0, st>>>(cache, rows, H, t_max, D, src, dst, per, total);
  return cudaGetLastError() == cudaSuccess ? EMU_OK : EMU_ERR_CUDA;
}

// ----------------------------------------------------------------------------------------------
__global__ void embed_gather_kernel(const bf16* __restrict__ table, const int* __restrict__ ids, bf16* out, int dim) {
  const long row = blockIdx.x;
  const uint4* src = reinterpret_cast<const uint4*>(table + (long)ids[row] * dim);
  uint4* dst = reinterpret_cast<uint4*>(out + row * dim);
  for (int i = threadIdx.x; i < (dim >> 3); i += blockDim.x) dst[i] = src[i];
}
int embed_gather(const bf16* table, const int* ids, bf16* out, int n, int dim, cudaStream_t st) {
  if (dim % 8) return EMU_ERR_INVALID;
  embed_gather_kernel<<<n, 128, 0, st>>>(table, ids, out, dim);
  return cudaGetLastError() == cudaSuccess ? EMU_OK : EMU_ERR_CUDA;
}

// first-max argmax per row of fp32 logits (greedy decoding): one 1024-thread CTA per row, 16-byte loads
__global__ void __launch_bounds__(1024) argmax_kernel(const float* __restrict__ logits, int cols, int* out) {
  __shared__ float sv[32];
  __shared__ int si[32];
  const float* row = logits + (long)blockIdx.x * cols;
  float best = -INFINITY;
  int bi = 0x7fffffff;
  auto take = [&](float v, int i) {
    if (v > best || (v == best && i < bi)) { best = v; bi = i; }
  };
  if ((cols & 3) == 0 && (reinterpret_cast<uintptr_t>(row) & 15) == 0) {
    const float4* r4 = reinterpret_cast<const float4*>(row);
    const int n4 = cols >> 2;
#pragma unroll 4
    for (int i = threadIdx.x; i < n4; i += blockDim.x) {
      const float4 v = __ldcg(r4 + i);
      take(v.x, 4 * i); take(v.y, 4 * i + 1); take(v.z, 4 * i + 2); take(v.w, 4 * i + 3);
    }
  } else {
    for (int i = threadIdx.x; i < cols; i += blockDim.x) take(row[i], i);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float ov = __shfl_xor_sync(0xffffffffu, best, o);
    const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
    if (ov > best || (ov == best && oi < bi)) { best = ov; bi = oi; }
  }
  if ((threadIdx.x & 31) == 0) { sv[threadIdx.x >> 5] = best; si[threadIdx.x >> 5] = bi; }
  __syncthreads();
  if (threadIdx.x < 32) {
    best = sv[threadIdx.x];
    bi = si[threadIdx.x];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float ov = __shfl_xor_sync(0xffffffffu, best, o);
      const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
      if (ov > best || (ov == best && oi < bi)) { best = ov; bi = oi; }
    }
    if (threadIdx.x == 0) out[blockIdx.x] = bi;
  }
}
int argmax_rows(const float* logits, int rows, int cols, int* out_idx, cudaStream_t st) {
  argmax_kernel<<<rows, 1024, 0, st>>>(logits, cols, out_idx);
  return cudaGetLastError() == cudaSuccess ? EMU_OK : EMU_ERR_CUDA;
}

// ----------------------------------------------------------------------------------------------
// ViT front/back ends (Emu2/emu/eva_vit.py:329-335, 406-409; Emu2/emu/emu.py:82-89)
// ----------------------------------------------------------------------------------------------
// NCHW image -> patch rows [B*G*G, Kpad], k = c*P*P + py*P + px (Conv2d weight flatten order), zero padded
__global__ void vit_im2col_kernel(const bf16* __restrict__ img, bf16* out, int B, int C, int HW, int P, int Kpad) {
  const int G = HW / P;
  const long total = (long)B * G * G * Kpad;
  for (long idx = blockIdx.x * (long)blockDim.x + threadIdx.x; idx < total; idx += (long)gridDim.x * blockDim.x) {
    const int k = idx % Kpad;
    const long prow = idx / Kpad;
    bf16 v = __float2bfloat16(0.f);
    if (k < C * P * P) {
      const int c = k / (P * P), py = (k / P) % P, px = k % P;
      const int gx = prow % G, gy = (prow / G) % G;
      const int b = prow / ((long)G * G);
      v = img[(((long)b * C + c) * HW + gy * P + py) * HW + gx * P + px];
    }
    out[idx] = v;
  }
}
int vit_im2col(const bf16* img, bf16* out, int B, int C, int HW, int P, int Kpad, cudaStream_t st) {
  vit_im2col_kernel<<<4 * kNumSMs, 256, 0, st>>>(img, out, B, C, HW, P, Kpad);
  return cudaGetLastError() == cudaSuccess ? EMU_OK : EMU_ERR_CUDA;
}

// x[b,0] = cls + pos[0];  x[b,1+i] = patches[b*Np+i] + pos[1+i]
__global__ void vit_assemble_kernel(const bf16* __restrict__ patches, const bf16* __restrict__ cls,
                                    const bf16* __restrict__ pos, bf16* x, int Np, int dim) {
  const int tok = blockIdx.x % (Np + 1);
  const int b = blockIdx.x / (Np + 1);
  const bf16* src = tok == 0 ? cls : patches + ((long)b * Np + tok - 1) * dim;
  const bf16* ps = pos + (long)tok * dim;
  bf16* dst = x + ((long)b * (Np + 1) + tok) * dim;
  for (int i = threadIdx.x; i < dim; i += blockDim.x)
    dst[i] = __float2bfloat16_rn(__bfloat162float(src[i]) + __bfloat162float(ps[i]));
}
int vit_assemble(const bf16* patches, const bf16* cls, const bf16* pos, bf16* x, int B, int Np, int dim,
                 cudaStream_t st) {
  vit_assemble_kernel<<<B * (Np + 1), 256, 0, st>>>(patches, cls, pos, x, Np, dim);
  return cudaGetLastError() == cudaSuccess ? EMU_OK : EMU_ERR_CUDA;
}

// drop CLS, average stride x stride windows of the G x G token grid
__global__ void vit_pool_kernel(const bf16* __restrict__ x, bf16* out, int G, int dim, int stride) {
  const int Q = G / stride;
  const int q = blockIdx.x % (Q * Q), b = blockIdx.x / (Q * Q);
  const int qy = q / Q, qx = q % Q;
  for (int c = threadIdx.x; c < dim; c += blockDim.x) {
    float s = 0.f;
    for (int dy = 0; dy < stride; ++dy)
      for (int dx = 0; dx < stride; ++dx)
        s += __bfloat162float(x[((long)b * (G * G + 1) + 1 + (qy * stride + dy) * G + qx * stride + dx) * dim + c]);
    out[((long)b * Q * Q + q) * dim + c] = __float2bfloat16_rn(s / (float)(stride * stride));
  }
}
int vit_pool(const bf16* x, bf16* out, int B, int G, int dim, int stride, cudaStream_t st) {
  if (stride < 1 || G % stride) return EMU_ERR_INVALID;
  const int Q = G / stride;
  vit_pool_kernel<<<B * Q * Q, 256, 0, st>>>(x, out, G, dim, stride);
  return cudaGetLastError() == cudaSuccess ? EMU_OK : EMU_ERR_CUDA;
}

// ----------------------------------------------------------------------------------------------
// beam-search KV reorder (HF _reorder_cache): cache[..., b, ...] <- cache[..., src[b], ...] in place.
// cache is viewed as [outer, B, H*t_max*D-with-holes]; each thread owns one 16-byte column position
// for ALL beams, so the in-place permutation needs no scratch.
// ----------------------------------------------------------------------------------------------
template <int MAXB>
__global__ void kv_reorder_kernel(bf16* cache, const int* __restrict__ src_idx, int outer, int B, int Bcap, int H,
                                  int t_max, int D, int n_tok) {
  const int vec_per_tok = D >> 3;
  const long per_outer = (long)H * n_tok * vec_per_tok;
  const long total = (long)outer * per_outer;
  int src[MAXB];
#pragma unroll
  for (int b = 0; b < MAXB; ++b) src[b] = b < B ? src_idx[b] : 0;
  for (long idx = blockIdx.x * (long)blockDim.x + threadIdx.x; idx < total; idx += (long)gridDim.x * blockDim.x) {
    const int v = idx % vec_per_tok;
    const int t = (idx / vec_per_tok) % n_tok;
    const int h = (idx / ((long)vec_per_tok * n_tok)) % H;
    const long o = idx / per_outer;
    // the cache holds Bcap sequences per (layer, k/v) slab; only the first B are live
    uint4* base = reinterpret_cast<uint4*>(cache) + ((o * Bcap * H + h) * (long)t_max + t) * vec_per_tok + v;
    const long bstride = (long)H * t_max * vec_per_tok;
    uint4 vals[MAXB];
#pragma unroll
    for (int b = 0; b < MAXB; ++b)
      if (b < B) vals[b] = base[src[b] * bstride];
#pragma unroll
    for (int b = 0; b < MAXB; ++b)
      if (b < B) base[b * bstride] = vals[b];
  }
}
int kv_reorder(bf16* cache, int Bcap, const int* src_idx, int B, long outer, int n_used_tokens, int H, int D, int t_max,
               cudaStream_t st) {
  if (B > 32 || D % 8) return EMU_ERR_INVALID;
  if (n_used_tokens <= 0) return EMU_OK;
  if (B <= 8) kv_reorder_kernel<8><<<8 * kNumSMs, 256, 0, st>>>(cache, src_idx, (int)outer, B, Bcap, H, t_max, D, n_used_tokens);
  else kv_reorder_kernel<32><<<8 * kNumSMs, 256, 0, st>>>(cache, src_idx, (int)outer, B, Bcap, H, t_max, D, n_used_tokens);
  return cudaGetLastError() == cudaSuccess ? EMU_OK : EMU_ERR_CUDA;
}

__global__ void kv_indir_update_kernel(int* indir, const int* __restrict__ src_idx, int B, int t_max, int n_tok,
                                       const int* __restrict__ row_len) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n_tok) return;
  int vals[32];
#pragma unroll
  for (int b = 0; b < 32; ++b)
    if (b < B && (!row_len || t < row_len[b])) vals[b] = indir[(long)src_idx[b] * t_max + t];
#pragma unroll
  for (int b = 0; b < 32; ++b)
    if (b < B && (!row_len || t < row_len[b])) indir[(long)b * t_max + t] = vals[b];
}
int kv_indir_update(int* indir, const int* src_idx, int B, int t_max, int n_tok, cudaStream_t st, const int* row_len) {
  if (B > 32) return EMU_ERR_INVALID;
  if (n_tok <= 0) return EMU_OK;
  kv_indir_update_kernel<<<(n_tok + 127) / 128, 128, 0, st>>>(indir, src_idx, B, t_max, n_tok, row_len);
  return cudaGetLastError() == cudaSuccess ? EMU_OK : EMU_ERR_CUDA;
}
__global__ void kv_indir_identity_kernel(int* indir, int rows, int t_max) {
  const long n = (long)rows * t_max;
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x)
    indir[i] = (int)(i / t_max);
}
int kv_indir_identity(int* indir, int rows, int t_max, cudaStream_t st) {
  kv_indir_identity_kernel<<<kNumSMs, 256, 0, st>>>(indir, rows, t_max);
  return cudaGetLastError() == cudaSuccess ? EMU_OK : EMU_ERR_CUDA;
}

__global__ void add_rows_kernel(const bf16* __restrict__ a, const bf16* __restrict__ b, bf16* out, long n) {
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x)
    out[i] = __float2bfloat16_rn(__bfloat162float(a[i]) + __bfloat162float(b[i]));
}
int add_rows(const bf16* a, const bf16* b, bf16* out, long n, cudaStream_t st) {
  add_rows_kernel<<<4 * kNumSMs, 256, 0, st>>>(a, b, out, n);
  return cudaGetLastError() == cudaSuccess ? EMU_OK : EMU_ERR_CUDA;
}

}  // namespace emu
