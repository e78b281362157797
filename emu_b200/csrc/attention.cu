// emu_b200 — attention kernels.
//
//  attn_decode : one new query per sequence against the bf16 KV cache (HF LlamaAttention with past_key_values,
//                reached from Emu2/emu/emu.py:213-229).  Pure KV streaming -> HBM-bound: split-KV CTAs with
//                16-byte coalesced row loads, warp-shuffle dot products, fp32 softmax, last-CTA combine.
//  attn_prefill: flash-style fused softmax(QK^T)V for prompts / encoders — causal + left-padding (LLaMA prefill),
//                bidirectional (EVA ViT, Emu2/emu/eva_vit.py:226-248; head_dim 112 and 88), additive bias
//                (T5 relative position, Emu1/models/modeling_t5.py:537-689) and cross attention (Nq != Nk).
//                Scores never touch HBM (the reference materialises [B,16,1025,1025] per ViT layer).
#include "common.cuh"
#include "ops.h"

namespace emu {

// ================================================================================================
// decode
// ================================================================================================
constexpr int kDecThreads = 128;

template <int D>
__global__ void __launch_bounds__(kDecThreads) attn_decode_kernel(
    const bf16* __restrict__ q, const bf16* __restrict__ k_cache, const bf16* __restrict__ v_cache, int H, int t_max,
    const int* __restrict__ pos, const int* __restrict__ start, float scale, bf16* out, float* ws_o, float* ws_ml,
    int* counters, int nsplit, int pdl, const int* __restrict__ indir) {
  // indir (optional, [rows][t_max]): cache row that holds token t of sequence b — beam search re-parents sequences by
  // rewriting this table instead of moving the cache (HF's `_reorder_cache` moves it; at 4k tokens x 20 rows that is
  // 2x the whole cache per step).
  constexpr int EPL = D / 8;  // elements per lane (8 lanes per token)
  constexpr int VPL = EPL / 8;  // uint4 per lane
  extern __shared__ __align__(16) float sm[];
  float* sc = sm;  // scores [per]
  __shared__ float qs[D];
  __shared__ float red[33];
  __shared__ float opart[16][D];
  __shared__ int s_last;

  const int h = blockIdx.x, b = blockIdx.y, sp = blockIdx.z;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  if (pdl) {
    pdl_launch_dependents();
    pdl_wait();
  }
  const int t_end = pos[b] + 1;
  const int t_begin = start ? start[b] : 0;
  const int n = t_end - t_begin;
  const int per = (n + nsplit - 1) / nsplit;
  const int t0 = t_begin + sp * per;
  const int t1 = min(t0 + per, t_end);

  for (int i = tid; i < D; i += kDecThreads) qs[i] = __bfloat162float(q[((long)b * H + h) * D + i]) * scale;
  __syncthreads();

  const long row_stride = (long)H * t_max * D;
  const bf16* kb = k_cache + (long)h * t_max * D;
  const bf16* vb = v_cache + (long)h * t_max * D;
  const int* ind = indir ? indir + (long)b * t_max : nullptr;

  // ---- phase 1: scores ----
  const int part = lane & 7, tig = lane >> 3;  // 8 lanes per token, 4 tokens per warp pass
  float qreg[EPL];
#pragma unroll
  for (int i = 0; i < EPL; ++i) qreg[i] = qs[part * EPL + i];
  float lmax = -INFINITY;
  // two token groups per trip: both K rows are requested before either is reduced (the long-context case has few CTAs per
  // SM, so the bytes in flight have to come from each warp)
  for (int tb = t0 + warp * 4; tb < t1; tb += 32) {  // warp-uniform trip count (shuffles below need all lanes)
    const int ta = tb + tig, tc = tb + 16 + tig;
    const bool oka = ta < t1, okc = tc < t1;
    uint4 ka[VPL], kc[VPL];
    if (oka) {
      const int row = ind ? __ldg(ind + ta) : b;
      const uint4* kr = reinterpret_cast<const uint4*>(kb + row * row_stride + (long)ta * D + part * EPL);
#pragma unroll
      for (int v = 0; v < VPL; ++v) ka[v] = ldg_stream(kr + v);
    }
    if (okc) {
      const int row = ind ? __ldg(ind + tc) : b;
      const uint4* kr = reinterpret_cast<const uint4*>(kb + row * row_stride + (long)tc * D + part * EPL);
#pragma unroll
      for (int v = 0; v < VPL; ++v) kc[v] = ldg_stream(kr + v);
    }
    float sa = 0.f, sc2 = 0.f;
    if (oka) {
#pragma unroll
      for (int v = 0; v < VPL; ++v) {
        const uint32_t k4[4] = {ka[v].x, ka[v].y, ka[v].z, ka[v].w};
#pragma unroll
        for (int j = 0; j < 4; ++j)
          sa += bf16_lo(k4[j]) * qreg[v * 8 + 2 * j] + bf16_hi(k4[j]) * qreg[v * 8 + 2 * j + 1];
      }
    }
    if (okc) {
#pragma unroll
      for (int v = 0; v < VPL; ++v) {
        const uint32_t k4[4] = {kc[v].x, kc[v].y, kc[v].z, kc[v].w};
#pragma unroll
        for (int j = 0; j < 4; ++j)
          sc2 += bf16_lo(k4[j]) * qreg[v * 8 + 2 * j] + bf16_hi(k4[j]) * qreg[v * 8 + 2 * j + 1];
      }
    }
    sa += __shfl_xor_sync(0xffffffffu, sa, 4);
    sc2 += __shfl_xor_sync(0xffffffffu, sc2, 4);
    sa += __shfl_xor_sync(0xffffffffu, sa, 2);
    sc2 += __shfl_xor_sync(0xffffffffu, sc2, 2);
    sa += __shfl_xor_sync(0xffffffffu, sa, 1);
    sc2 += __shfl_xor_sync(0xffffffffu, sc2, 1);
    if (oka && part == 0) sc[ta - t0] = sa;
    if (okc && part == 0) sc[tc - t0] = sc2;
    if (oka) lmax = fmaxf(lmax, sa);
    if (okc) lmax = fmaxf(lmax, sc2);
  }
  lmax = warp_max(lmax);
  if (lane == 0) red[warp] = lmax;
  __syncthreads();
  const float m = fmaxf(fmaxf(red[0], red[1]), fmaxf(red[2], red[3]));
  __syncthreads();
  // ---- phase 2: exp / sum ----
  float lsum = 0.f;
  for (int i = tid; i < t1 - t0; i += kDecThreads) {
    const float p = __expf(sc[i] - m);
    sc[i] = p;
    lsum += p;
  }
  const float l = block_sum(lsum, red);
  // ---- phase 3: P·V ----
  const int dpart = tid & 7, tl = tid >> 3;  // 16 token lanes x 8 d-slices
  float acc[EPL];
#pragma unroll
  for (int i = 0; i < EPL; ++i) acc[i] = 0.f;
#pragma unroll 4
  for (int t = t0 + tl; t < t1; t += 16) {
    const float p = sc[t - t0];
    const int row = ind ? __ldg(ind + t) : b;
    const uint4* vr = reinterpret_cast<const uint4*>(vb + row * row_stride + (long)t * D + dpart * EPL);
#pragma unroll
    for (int v = 0; v < VPL; ++v) {
      const uint4 vv = ldg_stream(vr + v);
      const uint32_t v4[4] = {vv.x, vv.y, vv.z, vv.w};
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        acc[v * 8 + 2 * j] += p * bf16_lo(v4[j]);
        acc[v * 8 + 2 * j + 1] += p * bf16_hi(v4[j]);
      }
    }
  }
#pragma unroll
  for (int i = 0; i < EPL; ++i) opart[tl][dpart * EPL + i] = acc[i];
  __syncthreads();
  float o = 0.f;  // thread d < D owns output element d
  if (tid < D) {
#pragma unroll
    for (int j = 0; j < 16; ++j) o += opart[j][tid];
  }
  if (nsplit == 1) {
    if (tid < D) out[((long)b * H + h) * D + tid] = __float2bfloat16_rn(l > 0.f ? o / l : 0.f);
    return;
  }
  const long bh = (long)b * H + h;
  if (tid < D) ws_o[(bh * nsplit + sp) * D + tid] = o;
  if (tid == 0) {
    ws_ml[(bh * nsplit + sp) * 2] = m;
    ws_ml[(bh * nsplit + sp) * 2 + 1] = l;
  }
  __threadfence();
  __syncthreads();
  if (tid == 0) {
    const int prev = atomicAdd(&counters[bh], 1);
    s_last = (prev == nsplit - 1);
    if (s_last) counters[bh] = 0;  // self-reset for the next launch / graph replay
  }
  __syncthreads();
  if (!s_last) return;
  __threadfence();
  if (tid < D) {
    float M = -INFINITY;
    for (int i = 0; i < nsplit; ++i) M = fmaxf(M, __ldcg(&ws_ml[(bh * nsplit + i) * 2]));
    float L = 0.f, O = 0.f;
    for (int i = 0; i < nsplit; ++i) {
      const float mi = __ldcg(&ws_ml[(bh * nsplit + i) * 2]), li = __ldcg(&ws_ml[(bh * nsplit + i) * 2 + 1]);
      const float w = (li > 0.f) ? __expf(mi - M) : 0.f;
      L += li * w;
      O += __ldcg(&ws_o[(bh * nsplit + i) * D + tid]) * w;
    }
    out[bh * D + tid] = __float2bfloat16_rn(L > 0.f ? O / L : 0.f);
  }
}

size_t attn_decode_workspace_bytes(int B, int H, int D) { return (size_t)B * H * 16 * (D + 2) * sizeof(float); }

int attn_decode(const bf16* q, const bf16* k_cache, const bf16* v_cache, int B, int H, int D, int t_max,
                const int* pos, const int* start, float scale, bf16* out, float* workspace, int* counters,
                int max_len_hint, int pdl, cudaStream_t st, const int* indir) {
  if (D != 64 && D != 128) return EMU_ERR_UNSUPPORTED;
  int nsplit = (2 * kNumSMs + H * B - 1) / (H * B);
  const int by_len = (max_len_hint + 63) / 64;
  if (nsplit > by_len) nsplit = by_len;
  {
    // long contexts: aim for ~8 CTAs (32 warps) per SM so that enough loads are in flight, in splits of >= 512 tokens
    // (4 prompts x 5 beams x 26 heads at 4k context was ONE split: 3.5 CTAs per SM, half the HBM rate)
    int want = (8 * kNumSMs + H * B - 1) / (H * B);
    const int cap = max_len_hint / 512;
    if (want > cap) want = cap;
    if (nsplit < want) nsplit = want;
  }
  if (nsplit > 16) nsplit = 16;
  if (nsplit < 1) nsplit = 1;
  const int per = (max_len_hint + nsplit - 1) / nsplit + 8;
  const size_t smem = (size_t)per * sizeof(float);
  if (smem > 160 * 1024) return EMU_ERR_UNSUPPORTED;
  float* ws_o = workspace;
  float* ws_ml = workspace + (size_t)B * H * 16 * D;
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = dim3(H, B, nsplit);
  cfg.blockDim = dim3(kDecThreads);
  cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = pdl ? 1 : 0;
  cudaError_t e;
  if (D == 128) {
    static size_t mx = 48 * 1024;
    if (smem > mx) {
      if (cudaFuncSetAttribute(attn_decode_kernel<128>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess)
        return EMU_ERR_CUDA;
      mx = smem;
    }
    e = cudaLaunchKernelEx(&cfg, attn_decode_kernel<128>, q, k_cache, v_cache, H, t_max, pos, start, scale, out, ws_o,
                           ws_ml, counters, nsplit, pdl, indir);
  } else {
    static size_t mx = 48 * 1024;
    if (smem > mx) {
      if (cudaFuncSetAttribute(attn_decode_kernel<64>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess)
        return EMU_ERR_CUDA;
      mx = smem;
    }
    e = cudaLaunchKernelEx(&cfg, attn_decode_kernel<64>, q, k_cache, v_cache, H, t_max, pos, start, scale, out, ws_o,
                           ws_ml, counters, nsplit, pdl, indir);
  }
  return e == cudaSuccess ? EMU_OK : EMU_ERR_CUDA;
}

// ================================================================================================
// verify (speculative decoding): NQ <= 8 consecutive queries of ONE sequence, query j at position L + j = pos[0] + j sees
// keys [start[0], L + j].  Split-KV CTAs (head, split) read every K / V element of their key range once for all NQ queries;
// the causal limit only touches the last NQ keys.  The splits are combined by the last CTA of a head in split order, so the
// result does not depend on which CTA finishes last.  Keys at or past L + NQ are never loaded.
// ================================================================================================
constexpr int kVerThreads = 128;
constexpr int kVerMaxSplit = 32;

template <int D, int NQ>
__global__ void __launch_bounds__(kVerThreads) attn_verify_kernel(
    const bf16* __restrict__ q, long q_ts, const bf16* __restrict__ k_cache, const bf16* __restrict__ v_cache, int H,
    int t_max, int row, const int* __restrict__ pos, const int* __restrict__ start, float scale, bf16* out, float* ws_o,
    float* ws_ml, int* counters, int nsplit, int per_cap, const int* __restrict__ indir) {
  constexpr int EPL = D / 8;     // K elements per lane in the score phase (8 lanes per key)
  constexpr int VPL = EPL / 8;   // uint4 per lane
  constexpr int DV = 4;          // V elements per thread in the P·V phase
  constexpr int TPR = D / DV;    // threads per V row
  constexpr int TL = kVerThreads / TPR;  // V rows in flight per CTA pass
  extern __shared__ __align__(16) float sc[];  // scores / probabilities [NQ][per_cap]
  __shared__ __align__(16) float qs[NQ][D];
  __shared__ float red[NQ][kVerThreads / 32];
  __shared__ float s_m[NQ], s_l[NQ];
  __shared__ float opart[TL][NQ][D];
  __shared__ int s_last;

  const int h = blockIdx.x, sp = blockIdx.y;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int L = pos[0];
  const int t_end = L + NQ;
  const int t_begin = start ? start[0] : 0;
  const int per = (t_end - t_begin + nsplit - 1) / nsplit;
  const int t0 = t_begin + sp * per;
  const int t1 = min(t0 + per, t_end);

  for (int i = tid; i < NQ * D; i += kVerThreads)
    qs[i / D][i % D] = __bfloat162float(q[(long)(i / D) * q_ts + (long)h * D + i % D]) * scale;
  __syncthreads();

  const long row_stride = (long)H * t_max * D;
  const bf16* kb = k_cache + (long)h * t_max * D;
  const bf16* vb = v_cache + (long)h * t_max * D;

  // ---- phase 1: scores.  Lane `part` of a key's 8 lanes holds elements (v * 8 + part) * 8 .. + 8: each v is one coalesced
  // 128-byte row segment, and the float4 reads of qs by the 8 parts fall in distinct banks.
  const int part = lane & 7, tig = lane >> 3;
  for (int tb = t0 + warp * 4; tb < t1; tb += 32) {  // warp-uniform trip count; two key groups in flight per trip
    int tk[2] = {tb + tig, tb + 16 + tig};
    uint4 kr[2][VPL];
#pragma unroll
    for (int g = 0; g < 2; ++g) {
      if (tk[g] < t1) {
        const int r = indir ? __ldg(indir + tk[g]) : row;
        const uint4* p = reinterpret_cast<const uint4*>(kb + r * row_stride + (long)tk[g] * D);
#pragma unroll
        for (int v = 0; v < VPL; ++v) kr[g][v] = ldg_stream(p + v * 8 + part);
      }
    }
#pragma unroll
    for (int g = 0; g < 2; ++g) {
      float s[NQ];
#pragma unroll
      for (int j = 0; j < NQ; ++j) s[j] = 0.f;
      if (tk[g] < t1) {
#pragma unroll
        for (int v = 0; v < VPL; ++v) {
          const uint32_t k4[4] = {kr[g][v].x, kr[g][v].y, kr[g][v].z, kr[g][v].w};
          float kf[8];
#pragma unroll
          for (int c = 0; c < 4; ++c) {
            kf[2 * c] = bf16_lo(k4[c]);
            kf[2 * c + 1] = bf16_hi(k4[c]);
          }
          const int e0 = (v * 8 + part) * 8;
#pragma unroll
          for (int j = 0; j < NQ; ++j) {
            const float4 a = *reinterpret_cast<const float4*>(&qs[j][e0]);
            const float4 b = *reinterpret_cast<const float4*>(&qs[j][e0 + 4]);
            s[j] += kf[0] * a.x + kf[1] * a.y + kf[2] * a.z + kf[3] * a.w + kf[4] * b.x + kf[5] * b.y + kf[6] * b.z +
                    kf[7] * b.w;
          }
        }
      }
#pragma unroll
      for (int j = 0; j < NQ; ++j) {
        s[j] += __shfl_xor_sync(0xffffffffu, s[j], 4);
        s[j] += __shfl_xor_sync(0xffffffffu, s[j], 2);
        s[j] += __shfl_xor_sync(0xffffffffu, s[j], 1);
      }
      if (tk[g] < t1 && part == 0) {
#pragma unroll
        for (int j = 0; j < NQ; ++j) sc[j * per_cap + tk[g] - t0] = tk[g] <= L + j ? s[j] : -INFINITY;
      }
    }
  }
  __syncthreads();

  // ---- phase 2: per-query max, exp, sum ----
  const int nk = t1 > t0 ? t1 - t0 : 0;
  float mx[NQ];
#pragma unroll
  for (int j = 0; j < NQ; ++j) mx[j] = -INFINITY;
  for (int i = tid; i < nk; i += kVerThreads)
#pragma unroll
    for (int j = 0; j < NQ; ++j) mx[j] = fmaxf(mx[j], sc[j * per_cap + i]);
#pragma unroll
  for (int j = 0; j < NQ; ++j) {
    mx[j] = warp_max(mx[j]);
    if (lane == 0) red[j][warp] = mx[j];
  }
  __syncthreads();
  if (tid < NQ) {
    float m = red[tid][0];
    for (int w = 1; w < kVerThreads / 32; ++w) m = fmaxf(m, red[tid][w]);
    s_m[tid] = m;
  }
  __syncthreads();
  float ls[NQ];
#pragma unroll
  for (int j = 0; j < NQ; ++j) ls[j] = 0.f;
  for (int i = tid; i < nk; i += kVerThreads) {
#pragma unroll
    for (int j = 0; j < NQ; ++j) {
      const float m = s_m[j];
      const float p = m == -INFINITY ? 0.f : __expf(sc[j * per_cap + i] - m);
      sc[j * per_cap + i] = p;
      ls[j] += p;
    }
  }
#pragma unroll
  for (int j = 0; j < NQ; ++j) {
    ls[j] = warp_sum(ls[j]);
    if (lane == 0) red[j][warp] = ls[j];
  }
  __syncthreads();
  if (tid < NQ) {
    float l = 0.f;
    for (int w = 0; w < kVerThreads / 32; ++w) l += red[tid][w];
    s_l[tid] = l;
  }

  // ---- phase 3: P·V, each V row loaded once for all NQ queries ----
  const int dq = tid % TPR, tl = tid / TPR;
  float acc[NQ][DV];
#pragma unroll
  for (int j = 0; j < NQ; ++j)
#pragma unroll
    for (int c = 0; c < DV; ++c) acc[j][c] = 0.f;
#pragma unroll 2
  for (int t = t0 + tl; t < t1; t += TL) {
    const int r = indir ? __ldg(indir + t) : row;
    const uint2 vv = __ldg(reinterpret_cast<const uint2*>(vb + r * row_stride + (long)t * D + dq * DV));
    const float vf[4] = {bf16_lo(vv.x), bf16_hi(vv.x), bf16_lo(vv.y), bf16_hi(vv.y)};
#pragma unroll
    for (int j = 0; j < NQ; ++j) {
      const float p = sc[j * per_cap + t - t0];
#pragma unroll
      for (int c = 0; c < DV; ++c) acc[j][c] += p * vf[c];
    }
  }
#pragma unroll
  for (int j = 0; j < NQ; ++j)
#pragma unroll
    for (int c = 0; c < DV; ++c) opart[tl][j][dq * DV + c] = acc[j][c];
  __syncthreads();

  const long hs = (long)h * nsplit + sp;
  for (int i = tid; i < NQ * D; i += kVerThreads) {
    const int j = i / D, d = i % D;
    float o = 0.f;
#pragma unroll
    for (int w = 0; w < TL; ++w) o += opart[w][j][d];
    if (nsplit == 1) {
      const float l = s_l[j];
      out[(long)j * H * D + (long)h * D + d] = __float2bfloat16_rn(l > 0.f ? o / l : 0.f);
    } else {
      ws_o[(hs * NQ + j) * D + d] = o;
    }
  }
  if (nsplit == 1) return;
  if (tid < NQ) {
    ws_ml[(hs * NQ + tid) * 2] = s_m[tid];
    ws_ml[(hs * NQ + tid) * 2 + 1] = s_l[tid];
  }
  __threadfence();
  __syncthreads();
  if (tid == 0) {
    const int prev = atomicAdd(&counters[h], 1);
    s_last = (prev == nsplit - 1);
    if (s_last) counters[h] = 0;  // self-reset for the next launch / graph replay
  }
  __syncthreads();
  if (!s_last) return;
  __threadfence();
  for (int i = tid; i < NQ * D; i += kVerThreads) {
    const int j = i / D, d = i % D;
    const long base = (long)h * nsplit;
    float M = -INFINITY;
    for (int s = 0; s < nsplit; ++s) M = fmaxf(M, __ldcg(&ws_ml[((base + s) * NQ + j) * 2]));
    float Ls = 0.f, O = 0.f;
    for (int s = 0; s < nsplit; ++s) {
      const float mi = __ldcg(&ws_ml[((base + s) * NQ + j) * 2]), li = __ldcg(&ws_ml[((base + s) * NQ + j) * 2 + 1]);
      const float w = li > 0.f ? __expf(mi - M) : 0.f;
      Ls += li * w;
      O += __ldcg(&ws_o[((base + s) * NQ + j) * D + d]) * w;
    }
    out[(long)j * H * D + (long)h * D + d] = __float2bfloat16_rn(Ls > 0.f ? O / Ls : 0.f);
  }
}

size_t attn_verify_workspace_bytes(int H, int D) { return (size_t)H * kVerMaxSplit * 8 * (D + 2) * sizeof(float); }

template <int D, int NQ>
static int launch_verify(const bf16* q, long q_ts, const bf16* k_cache, const bf16* v_cache, int H, int t_max, int row,
                         const int* pos, const int* start, float scale, bf16* out, float* ws, int* counters, int nsplit,
                         int per_cap, cudaStream_t st, const int* indir) {
  const size_t smem = (size_t)NQ * per_cap * sizeof(float);
  static size_t mx = 0;
  if (smem > mx) {
    if (cudaFuncSetAttribute(attn_verify_kernel<D, NQ>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess)
      return EMU_ERR_CUDA;
    mx = smem;
  }
  float* ws_o = ws;
  float* ws_ml = ws + (size_t)H * kVerMaxSplit * 8 * D;
  attn_verify_kernel<D, NQ><<<dim3(H, nsplit), kVerThreads, smem, st>>>(q, q_ts, k_cache, v_cache, H, t_max, row, pos, start,
                                                                        scale, out, ws_o, ws_ml, counters, nsplit, per_cap,
                                                                        indir);
  return cudaGetLastError() == cudaSuccess ? EMU_OK : EMU_ERR_CUDA;
}

template <int D>
static int verify_dispatch(int n, const bf16* q, long q_ts, const bf16* k_cache, const bf16* v_cache, int H, int t_max, int row,
                           const int* pos, const int* start, float scale, bf16* out, float* ws, int* counters, int nsplit,
                           int per_cap, cudaStream_t st, const int* indir) {
#define EMU_VERIFY_CASE(N)                                                                                              \
  case N:                                                                                                               \
    return launch_verify<D, N>(q, q_ts, k_cache, v_cache, H, t_max, row, pos, start, scale, out, ws, counters, nsplit, \
                               per_cap, st, indir);
  switch (n) {
    EMU_VERIFY_CASE(1)
    EMU_VERIFY_CASE(2)
    EMU_VERIFY_CASE(3)
    EMU_VERIFY_CASE(4)
    EMU_VERIFY_CASE(5)
    EMU_VERIFY_CASE(6)
    EMU_VERIFY_CASE(7)
    EMU_VERIFY_CASE(8)
  }
#undef EMU_VERIFY_CASE
  return EMU_ERR_INVALID;
}

int attn_verify(const bf16* q, long q_ts, const bf16* k_cache, const bf16* v_cache, int n, int H, int D, int t_max, int row,
                const int* pos, const int* start, float scale, bf16* out, float* workspace, int* counters, int max_len_hint,
                cudaStream_t st, const int* indir) {
  if (D != 64 && D != 128) return EMU_ERR_UNSUPPORTED;
  if (n < 1 || n > 8 || H < 1 || max_len_hint < 1 || (q_ts % 8)) return EMU_ERR_INVALID;
  // about 8 CTAs per SM over the heads, and at least 32 keys per split
  int nsplit = (8 * kNumSMs + H - 1) / H;
  if (nsplit > max_len_hint / 32) nsplit = max_len_hint / 32;
  if (nsplit > kVerMaxSplit) nsplit = kVerMaxSplit;
  if (nsplit < 1) nsplit = 1;
  const int per_cap = (max_len_hint + nsplit - 1) / nsplit;
  if ((size_t)8 * per_cap * sizeof(float) > 160 * 1024) return EMU_ERR_UNSUPPORTED;
  if (D == 128)
    return verify_dispatch<128>(n, q, q_ts, k_cache, v_cache, H, t_max, row, pos, start, scale, out, workspace, counters,
                                nsplit, per_cap, st, indir);
  return verify_dispatch<64>(n, q, q_ts, k_cache, v_cache, H, t_max, row, pos, start, scale, out, workspace, counters, nsplit,
                             per_cap, st, indir);
}

// ================================================================================================
// prefill / encoder flash attention (mma.sync m16n8k16, 4 warps x 16 query rows, 64-key blocks)
// ================================================================================================
constexpr int kFaThreads = 128;
constexpr int kFaBM = 64;
constexpr int kFaBN = 64;

template <int DP>
struct FaSmem {
  static constexpr int LD = DP + 8;  // row stride (elements): odd multiple of 16 B -> conflict-free ldmatrix
  static constexpr int kTile = 64 * LD;
  static constexpr int kBytes = (kTile /*Q*/ + 4 * kTile /*K,V double buffered*/) * 2;
};

template <int DP>
__device__ __forceinline__ void fa_load_tile(bf16* dst, const bf16* src, long ts, int row0, int nrows_valid, int D) {
  // 64 rows x DP cols, 16-byte chunks, zero fill outside [0,nrows_valid) x [0,D)
  constexpr int LD = FaSmem<DP>::LD;
  constexpr int CPR = DP / 8;
  for (int c = threadIdx.x; c < 64 * CPR; c += kFaThreads) {
    const int r = c / CPR, ch = c % CPR;
    const bool ok = (row0 + r) < nrows_valid && ch * 8 < D;
    const bf16* g = ok ? src + (long)(row0 + r) * ts + ch * 8 : src;
    cp_async16(dst + r * LD + ch * 8, g, ok);
  }
}

// kPacked (slot mode): batch b's queries are the rows a.q_row0[b] .. + a.q_len[b] of one packed view, at key positions
// a.q_off[b] + i; rows past its q_len are neither loaded nor stored, and keys at or past a.q_off[b] + a.q_len[b] load as zeros.
template <int DP, bool kPacked>
__global__ void __launch_bounds__(kFaThreads) attn_prefill_kernel(const AttnArgs a) {
  constexpr int LD = FaSmem<DP>::LD;
  constexpr int KS = DP / 16;  // k-steps over the head dim
  constexpr int NT = DP / 8;   // output n-tiles
  extern __shared__ __align__(16) uint8_t smraw[];
  bf16* sQ = reinterpret_cast<bf16*>(smraw);
  bf16* sK = sQ + FaSmem<DP>::kTile;
  bf16* sV = sK + 2 * FaSmem<DP>::kTile;

  const int qb = blockIdx.x, h = blockIdx.y, b = blockIdx.z;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int g = lane >> 2, t = lane & 3;
  const int q0 = qb * kFaBM;
  const int q_n = kPacked ? a.q_len[b] : a.Nq;  // this batch's query rows
  if (kPacked && q0 >= q_n) return;

  const bf16* qp = a.q + (kPacked ? (long)a.q_row0[b] * a.q_ts : (long)b * a.q_bs) + (long)h * a.q_hs;
  const int kvb = a.kv_row ? a.kv_row[b] : b;
  const bf16* kp = a.k + (long)kvb * a.k_bs + (long)h * a.k_hs;
  const bf16* vp = a.v + (long)kvb * a.v_bs + (long)h * a.v_hs;
  const int kv_lo = a.kv_start ? a.kv_start[b] : 0;
  const int shift = kPacked ? a.q_off[b] : a.Nk - a.Nq;  // causal: key j visible to query i iff j <= i + shift
  // keys of this batch: all Nk, or (kPacked) up to the end of its rows; past it the tiles load as zeros
  const int kv_n = kPacked ? min(a.Nk, shift + (a.q_len ? a.q_len[b] : a.Nq)) : a.Nk;
  int kv_hi = kv_n;
  if (a.causal) kv_hi = min(kv_n, q0 + kFaBM + shift);
  const int nb0 = kv_lo / kFaBN;
  const int nb1 = (kv_hi + kFaBN - 1) / kFaBN;

  fa_load_tile<DP>(sQ, qp, a.q_ts, q0, q_n, a.D);
  if (nb0 < nb1) {
    fa_load_tile<DP>(sK, kp, a.k_ts, nb0 * kFaBN, kv_n, a.D);
    fa_load_tile<DP>(sV, vp, a.v_ts, nb0 * kFaBN, kv_n, a.D);
  }
  cp_async_commit();

  float o_acc[NT][4];
#pragma unroll
  for (int i = 0; i < NT; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) o_acc[i][j] = 0.f;
  float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};
  uint32_t qf[KS][4];
  bool q_loaded = false;

  const int qrow0 = q0 + warp * 16 + g;  // rows qrow0 and qrow0 + 8
  for (int nb = nb0; nb < nb1; ++nb) {
    const int buf = (nb - nb0) & 1;
    if (nb + 1 < nb1) {
      fa_load_tile<DP>(sK + (buf ^ 1) * FaSmem<DP>::kTile, kp, a.k_ts, (nb + 1) * kFaBN, kv_n, a.D);
      fa_load_tile<DP>(sV + (buf ^ 1) * FaSmem<DP>::kTile, vp, a.v_ts, (nb + 1) * kFaBN, kv_n, a.D);
      cp_async_commit();
      cp_async_wait<1>();
    } else {
      cp_async_wait<0>();
    }
    __syncthreads();
    if (!q_loaded) {
#pragma unroll
      for (int ks = 0; ks < KS; ++ks) {
        const int r = warp * 16 + (lane & 15);
        const int c = ks * 16 + (lane >> 4) * 8;
        ldmatrix_x4(qf[ks], smem_u32(sQ + r * LD + c));
      }
      q_loaded = true;
    }
    const bf16* tK = sK + buf * FaSmem<DP>::kTile;
    const bf16* tV = sV + buf * FaSmem<DP>::kTile;

    // ---- S = Q K^T (16 x 64 per warp) ----
    float s[8][4];
#pragma unroll
    for (int i = 0; i < 8; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j) s[i][j] = 0.f;
#pragma unroll
    for (int ks = 0; ks < KS; ++ks) {
#pragma unroll
      for (int np = 0; np < 4; ++np) {  // pairs of 8-key n-tiles
        uint32_t kf[4];
        const int mi = lane >> 3, rr = lane & 7;
        const int key = np * 16 + (mi >> 1) * 8 + rr;
        const int dd = ks * 16 + (mi & 1) * 8;
        ldmatrix_x4(kf, smem_u32(tK + key * LD + dd));
        mma_bf16_16816(s[2 * np], qf[ks], kf);
        mma_bf16_16816(s[2 * np + 1], qf[ks], kf + 2);
      }
    }
    // ---- scale, bias, mask, online softmax ----
    const int key0 = nb * kFaBN;
    float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
    for (int nt = 0; nt < 8; ++nt) {
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int qi = qrow0 + (j >> 1) * 8;
        const int kj = key0 + nt * 8 + 2 * t + (j & 1);
        float x = s[nt][j] * a.scale;
        if (a.bias != nullptr && qi < a.Nq && kj < a.Nk) x += a.bias[((long)h * a.Nq + qi) * a.Nk + kj];
        const bool vis = kj < kv_n && kj >= kv_lo && (!a.causal || kj <= qi + shift);
        x = vis ? x : -INFINITY;
        s[nt][j] = x;
        mx[j >> 1] = fmaxf(mx[j >> 1], x);
      }
    }
    float corr[2], m_use[2];
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 1));
      mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 2));
      const float m_new = fmaxf(m_run[r], mx[r]);
      m_use[r] = (m_new == -INFINITY) ? 0.f : m_new;  // fully masked row so far
      corr[r] = (m_run[r] == -INFINITY) ? 0.f : __expf(m_run[r] - m_use[r]);
      m_run[r] = m_new;
    }
    float rs[2] = {0.f, 0.f};
    uint32_t pf[4][4];  // P as A fragments for 4 k-steps of 16 keys
#pragma unroll
    for (int nt = 0; nt < 8; ++nt) {
      const float p0 = __expf(s[nt][0] - m_use[0]), p1 = __expf(s[nt][1] - m_use[0]);
      const float p2 = __expf(s[nt][2] - m_use[1]), p3 = __expf(s[nt][3] - m_use[1]);
      rs[0] += p0 + p1;
      rs[1] += p2 + p3;
      pf[nt >> 1][(nt & 1) * 2] = pack_bf16(p0, p1);
      pf[nt >> 1][(nt & 1) * 2 + 1] = pack_bf16(p2, p3);
    }
#pragma unroll
    for (int r = 0; r < 2; ++r) l_run[r] = l_run[r] * corr[r] + rs[r];
#pragma unroll
    for (int i = 0; i < NT; ++i) {
      o_acc[i][0] *= corr[0];
      o_acc[i][1] *= corr[0];
      o_acc[i][2] *= corr[1];
      o_acc[i][3] *= corr[1];
    }
    // ---- O += P V ----
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {  // 16 keys per step
#pragma unroll
      for (int dp = 0; dp < NT / 2; ++dp) {  // pairs of 8-wide d tiles
        uint32_t vf[4];
        const int mi = lane >> 3, rr = lane & 7;
        const int key = kk * 16 + (mi & 1) * 8 + rr;
        const int dd = dp * 16 + (mi >> 1) * 8;
        ldmatrix_x4_trans(vf, smem_u32(tV + key * LD + dd));
        mma_bf16_16816(o_acc[2 * dp], pf[kk], vf);
        mma_bf16_16816(o_acc[2 * dp + 1], pf[kk], vf + 2);
      }
    }
    __syncthreads();
  }
  cp_async_wait<0>();

  // ---- normalise and store ----
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    l_run[r] += __shfl_xor_sync(0xffffffffu, l_run[r], 1);
    l_run[r] += __shfl_xor_sync(0xffffffffu, l_run[r], 2);
  }
  bf16* op = a.out + (kPacked ? (long)a.q_row0[b] * a.o_ts : (long)b * a.o_bs) + (long)h * a.o_hs;
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int qi = qrow0 + r * 8;
    if (qi >= q_n) continue;
    const float inv = l_run[r] > 0.f ? 1.f / l_run[r] : 0.f;
#pragma unroll
    for (int nt = 0; nt < NT; ++nt) {
      const int d = nt * 8 + 2 * t;
      if (d < a.D)
        *reinterpret_cast<uint32_t*>(op + (long)qi * a.o_ts + d) =
            pack_bf16(o_acc[nt][2 * r] * inv, o_acc[nt][2 * r + 1] * inv);
    }
  }
}

template <int DP, bool kPacked = false>
static int launch_fa(const AttnArgs& a, cudaStream_t st) {
  static bool set = false;
  if (!set) {
    if (cudaFuncSetAttribute(attn_prefill_kernel<DP, kPacked>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                             FaSmem<DP>::kBytes) != cudaSuccess)
      return EMU_ERR_CUDA;
    set = true;
  }
  dim3 grid((a.Nq + kFaBM - 1) / kFaBM, a.H, a.B);
  attn_prefill_kernel<DP, kPacked><<<grid, kFaThreads, FaSmem<DP>::kBytes, st>>>(a);
  return cudaGetLastError() == cudaSuccess ? EMU_OK : EMU_ERR_CUDA;
}

int attn_prefill(const AttnArgs& a, cudaStream_t st) {
  if (a.D % 8 || a.D > 160 || a.Nq < 1 || a.Nk < 1) return EMU_ERR_INVALID;
  // strides must keep 16-byte alignment of every row
  if ((a.q_ts % 8) || (a.k_ts % 8) || (a.v_ts % 8) || (a.q_hs % 8) || (a.k_hs % 8) || (a.v_hs % 8) ||
      (a.q_bs % 8) || (a.k_bs % 8) || (a.v_bs % 8) || (a.o_ts % 2) || (a.o_hs % 2) || (a.o_bs % 2))
    return EMU_ERR_INVALID;
  // dense problems go to the wgmma kernel (attention_tc.cu); EMU_ATTN=legacy forces this file's mma.sync kernel
  static int legacy = -1;
  if (legacy < 0) {
    const char* v = getenv("EMU_ATTN");
    legacy = (v && v[0] == 'l') ? 1 : 0;
  }
  if (!legacy) {
    const int rc = attn_prefill_tc(a, st);
    if (rc != EMU_ERR_UNSUPPORTED) return rc;
  }
  if (a.q_off || a.q_len || a.q_row0) {  // packed queries (slot mode): causal, the LLaMA head dims only
    if (!a.q_off || !a.q_len || !a.q_row0 || !a.causal || a.bias) return EMU_ERR_INVALID;
    if (a.D == 64) return launch_fa<64, true>(a, st);
    if (a.D == 128) return launch_fa<128, true>(a, st);
    return EMU_ERR_INVALID;
  }
  if (a.D <= 32) return launch_fa<32>(a, st);
  if (a.D <= 64) return launch_fa<64>(a, st);
  if (a.D <= 96) return launch_fa<96>(a, st);
  if (a.D <= 112) return launch_fa<112>(a, st);
  if (a.D <= 128) return launch_fa<128>(a, st);
  return launch_fa<160>(a, st);  // SD-1.5 class UNets: 8 heads of 160 at the 1280-channel levels (Emu1 pipeline)
}

}  // namespace emu
