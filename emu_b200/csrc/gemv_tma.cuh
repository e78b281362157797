// emu_b200 — device-side building blocks of the TMA-fed skinny GEMM (gemv_tma.cu has the design notes).
#pragma once
#include <stdlib.h>

#include "common.cuh"
#include "ops.h"

namespace emu {

int make_tmap_2d(CUtensorMap* out, const void* base, long rows, long cols, long ld, int box_rows);  // gemm_tc.cu

constexpr int kTW = 8;                  // consumer warps
constexpr int kTThreads = (kTW + 1) * 32;  // + 1 producer warp
constexpr int kTRT = 2;                 // 16-row tiles per chunk
constexpr int kTRows = 16 * kTRT;       // 32 rows
constexpr int kTCols = 256;             // columns per chunk (4 TMA tiles of 64)
constexpr int kTStageBytes = kTRows * kTCols * 2;  // 16 KB
constexpr int kTStages = 10;  // ring slots carved; p.nstages of them are used
constexpr int kTMaxParts = 8;
constexpr int kTWsGroups = 8192;

struct GemvTmaParams {
  GemvArgs a;
  int ldxs;      // smem row stride of staged x (elements), = Kpad + 8
  int kpad;      // K rounded up to 256
  int cpt;       // chunks per row group
  int xsc;       // chunks of x staged in shared memory at a time (0 or >= cpt: the whole row; smaller: K segments that
                 //   are re-staged as the chunk stream crosses them — batch x K too large for shared memory, e.g. 5 x 17920)
  int xbulk;     // x reaches shared memory by cp.async.bulk row copies (aligned rows; normalised in place afterwards)
  int nstages;   // ring depth actually used (<= kTStages)
  int geff;      // number of CTAs that share this matrix's chunks (<= gridDim.x); CTAs >= geff get none
  long total;    // total chunks
  float* ws;     // [groups][kTMaxParts][kTRT*128]
  int* counters;
};

static __device__ __forceinline__ void consumer_bar() { asm volatile("bar.sync 1, 256;" ::: "memory"); }

// finish k-segment [kc_lo, kc_hi] of row group grp (consumer threads only; `red` already holds per-warp partials)
static __device__ __noinline__ void gemv_tma_flush(const GemvTmaParams* sp, float* red, float* fin, int* s_last_p, int grp,
                                            int kc_lo, int kc_hi) {
  const GemvTmaParams& p = *sp;
  const GemvArgs& a = p.a;
  const int N = a.N, B = a.B, CPT = p.cpt;
  constexpr int nval = kTRT * 128;
  const long G = p.geff;
  const int tid = threadIdx.x;  // < 256
  consumer_bar();
  const bool whole = (kc_lo == 0 && kc_hi == CPT - 1);
  bool do_epilogue = whole;
  float v = 0.f;
#pragma unroll
  for (int w = 0; w < kTW; ++w) v += red[w * nval + tid];
  if (whole) {
    fin[tid] = v;
  } else {
    const long first_chunk = (long)grp * CPT;
    const int first_owner = (int)(((first_chunk + 1) * G - 1) / p.total);
    const int last_owner = (int)(((first_chunk + CPT) * G - 1) / p.total);
    const int nparts = last_owner - first_owner + 1;
    const int my = (int)blockIdx.x - first_owner;
    float* wt = p.ws + ((long)grp * kTMaxParts) * nval;
    wt[my * nval + tid] = v;
    __threadfence();
    consumer_bar();
    if (tid == 0) {
      const int prev = atomicAdd(&p.counters[grp], 1);
      *s_last_p = (prev == nparts - 1);
      if (prev == nparts - 1) p.counters[grp] = 0;
    }
    consumer_bar();
    do_epilogue = *s_last_p != 0;
    if (do_epilogue) {
      __threadfence();
      float s = 0.f;
      for (int q = 0; q < nparts; ++q) s += __ldcg(&wt[q * nval + tid]);  // fixed order: deterministic
      fin[tid] = s;
    }
  }
  if (do_epilogue) {
    consumer_bar();
    const int rt = tid >> 7, r = tid & 15, b = (tid >> 4) & 7;
    const float* f = fin + rt * 128;
    const int nrow = (grp * kTRT + rt) * 16 + r;
    if (b < B && nrow < N) {
      if (a.mode == EPI_NONE && a.ll_n > 0) {
        // fused tensor-parallel push: {value, flag} words are self-validating, so no fence / separate flag round trip
        const unsigned flag = __ldcg(a.ll_step) * 256u + (unsigned)a.ll_idx + 1u;
        const unsigned bits = __float_as_uint(f[r * 8 + b]);
        const size_t off = ((size_t)(a.ll_idx & 1) * a.ll_n + a.ll_rank) * a.ll_slot_elems + (size_t)b * a.ldy + nrow;
        for (int pr = 0; pr < a.ll_n; ++pr)
          asm volatile("st.global.v2.b32 [%0], {%1, %2};" ::"l"(reinterpret_cast<uint2*>(a.ll_peer[pr]) + off), "r"(bits),
                       "r"(flag)
                       : "memory");
      } else if (a.mode == EPI_NONE) {
        float o = f[r * 8 + b];
        if (a.bias) o += __bfloat162float(a.bias[nrow]);
        if (a.residual)
          o = round_bf16(o) + __uint_as_float((uint32_t)__ldcg(reinterpret_cast<const unsigned short*>(a.residual) + (long)b * a.ldr + nrow) << 16);
        if (a.out_fp32) reinterpret_cast<float*>(a.y)[(long)b * a.ldy + nrow] = o;
        else reinterpret_cast<bf16*>(a.y)[(long)b * a.ldy + nrow] = __float2bfloat16_rn(o);
      } else if (a.mode == EPI_SWIGLU) {
        if (!(r & 1)) {
          const float gate = round_bf16(f[r * 8 + b]), up = round_bf16(f[(r + 1) * 8 + b]);
          reinterpret_cast<bf16*>(a.y)[(long)b * a.ldy + (nrow >> 1)] = __float2bfloat16_rn(round_bf16(silu(gate)) * up);
        }
      } else {  // GEMV_ROPE_QKV
        const int D = a.head_dim, H = a.n_heads;
        const int hh = nrow / D, i = nrow - hh * D;
        const int slot = a.pos[b];
        if (hh < 2 * H) {
          if (!(r & 1)) {
            const float x1 = round_bf16(f[r * 8 + b]), x2 = round_bf16(f[(r + 1) * 8 + b]);
            const int rp = slot - (a.pos_off ? a.pos_off[b] : 0);
            const float c = __bfloat162float(a.rope_cos[(long)rp * (D / 2) + (i >> 1)]);
            const float s = __bfloat162float(a.rope_sin[(long)rp * (D / 2) + (i >> 1)]);
            const float o1 = round_bf16(x1 * c) + round_bf16(-x2 * s);
            const float o2 = round_bf16(x2 * c) + round_bf16(x1 * s);
            bf16* dst;
            if (hh < H) dst = reinterpret_cast<bf16*>(a.y) + (long)b * a.ldy + nrow;
            else dst = a.k_cache + (((long)b * H + (hh - H)) * a.t_max + slot) * D + i;
            *reinterpret_cast<uint32_t*>(dst) = pack_bf16(o1, o2);
          }
        } else {
          a.v_cache[(((long)b * H + (hh - 2 * H)) * a.t_max + slot) * D + i] = __float2bfloat16_rn(f[r * 8 + b]);
        }
      }
    }
  }
  consumer_bar();
}


// ---- producer: stream this CTA's chunk range [c0, c1) of one weight matrix through the ring ----
static __device__ __forceinline__ void tma_produce(const CUtensorMap* tm, int cpt, long c0, long c1, uint8_t* ring,
                                                   uint64_t* full_bar, uint64_t* empty_bar, int nstages, int& stage,
                                                   uint32_t& phase) {
  int grp = (int)(c0 / cpt), kc = (int)(c0 % cpt);
  for (long i = c0; i < c1; ++i) {
    mbar_wait(&empty_bar[stage], phase ^ 1);
    uint8_t* dst = ring + stage * kTStageBytes;
    mbar_expect_tx(&full_bar[stage], kTStageBytes);
#pragma unroll
    for (int j = 0; j < 4; ++j)
      tma_load_2d(dst + j * (kTRows * 128), tm, &full_bar[stage], kc * kTCols + j * 64, grp * kTRows);
    if (++stage == nstages) { stage = 0; phase ^= 1; }
    if (++kc == cpt) { kc = 0; ++grp; }
  }
}

// ---- consumers: stage x (optionally RMS-normalised, zero padded to kpad) into shared memory ----
// Staging sits on the critical path of every GEMV (the weight ring is full long before it ends), so it is written for
// latency: loads are issued four deep per thread before anything is consumed, and the norm weights —
// which do not depend on the predecessor kernel — are fetched by the caller before griddepcontrol.wait (XPre).
// LlamaRMSNorm on two packed bf16: w * bf16(x * rstd).  cvt.rn.bf16x2.f32 rounds both products in one instruction and
// mul.rn.bf16x2 rounds the exact bf16 x bf16 product once — bit-identical to round_bf16(round_bf16(x * rstd) * w) in fp32.
static __device__ __forceinline__ uint32_t rmsnorm_pair(uint32_t x2, float rstd, uint32_t w2) {
  const float lo = __uint_as_float(x2 << 16) * rstd, hi = __uint_as_float(x2 & 0xffff0000u) * rstd;
  uint32_t n2, o2;
  asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(n2) : "f"(hi), "f"(lo));
  asm("mul.rn.bf16x2 %0, %1, %2;" : "=r"(o2) : "r"(n2), "r"(w2));
  return o2;
}
struct XPre {
  uint4 w[4];  // this thread's norm-weight vectors of columns (threadIdx.x + 256 j) * 8, j < 4 (K <= 8192)
  bool have = false;
};
static __device__ __forceinline__ void tma_prefetch_norm_w(const GemvTmaParams& p, XPre& pre) {
  const GemvArgs& a = p.a;
  pre.have = false;
  if (a.norm_w == nullptr || (a.K >> 3) > 1024) return;
  const uint4* wsrc = reinterpret_cast<const uint4*>(a.norm_w);
  const int vec_per_row = a.K >> 3;
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const int gi = (int)threadIdx.x + 256 * j;
    pre.w[j] = gi < vec_per_row ? __ldg(wsrc + gi) : make_uint4(0, 0, 0, 0);
  }
  pre.have = true;
}

// columns [seg * xsc * 256, (seg + 1) * xsc * 256) of every batch row (the whole row when xsc covers it)
static __device__ __forceinline__ void tma_stage_x_seg(const GemvTmaParams& p, bf16* xs, const float* s_rstd, int seg,
                                                       const XPre* pre = nullptr) {
  const GemvArgs& a = p.a;
  const int K = a.K, B = a.B;
  const int vec_per_row = K >> 3;
  const int xsc = (p.xsc > 0 && p.xsc < p.cpt) ? p.xsc : p.cpt;
  const int v0 = seg * xsc * (kTCols >> 3);                       // first 16-byte vector of the segment
  const int nv = min(xsc, p.cpt - seg * xsc) * (kTCols >> 3);     // vectors in this segment (zero padded past K)
  const bool use_pre = pre != nullptr && pre->have && v0 == 0;
  const uint4* wsrc = reinterpret_cast<const uint4*>(a.norm_w);
  for (int b = 0; b < B; ++b) {
    const float rstd = a.norm_w ? s_rstd[b] : 1.f;
    const uint4* src = reinterpret_cast<const uint4*>(a.x + (long)b * a.ldx);
    uint4* dst = reinterpret_cast<uint4*>(xs + (long)b * p.ldxs);
    for (int i0 = 0; i0 < nv; i0 += 1024) {
      uint4 v[4], w[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) {  // four independent loads in flight per thread
        const int gi = v0 + i0 + (int)threadIdx.x + 256 * j;
        // activations may have been produced by other CTAs of this very kernel's predecessor: bypass L1
        v[j] = (i0 + (int)threadIdx.x + 256 * j < nv && gi < vec_per_row) ? __ldcg(src + gi) : make_uint4(0, 0, 0, 0);
        if (a.norm_w) w[j] = (use_pre && i0 == 0) ? pre->w[j] : (gi < vec_per_row ? __ldg(wsrc + gi) : make_uint4(0, 0, 0, 0));
      }
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int i = i0 + (int)threadIdx.x + 256 * j;
        if (i >= nv) continue;
        uint4 o = v[j];
        if (a.norm_w) {
          const uint32_t v4[4] = {v[j].x, v[j].y, v[j].z, v[j].w}, w4[4] = {w[j].x, w[j].y, w[j].z, w[j].w};
          uint32_t o4[4];
#pragma unroll
          for (int q = 0; q < 4; ++q) o4[q] = rmsnorm_pair(v4[q], rstd, w4[q]);  // HF: weight * (x.float() * rsqrt(var + eps)).to(bf16)
          o = make_uint4(o4[0], o4[1], o4[2], o4[3]);
        }
        dst[i] = o;
      }
    }
  }
  consumer_bar();
}

static __device__ __forceinline__ void tma_stage_x(const GemvTmaParams& p, bf16* xs, float (*s_ss)[8], float* s_rstd,
                                                   int seg = 0, const XPre* pre = nullptr) {
  const GemvArgs& a = p.a;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int K = a.K, B = a.B;
  const int vec_per_row = K >> 3;
  if (a.norm_w != nullptr) {
    float ss[8];
#pragma unroll
    for (int b = 0; b < 8; ++b) ss[b] = 0.f;
    for (int b = 0; b < B; ++b) {
      const uint4* src = reinterpret_cast<const uint4*>(a.x + (long)b * a.ldx);
      float s = 0.f;
      for (int i0 = 0; i0 < vec_per_row; i0 += 1024) {
        uint4 v[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const int i = i0 + (int)threadIdx.x + 256 * j;
          v[j] = i < vec_per_row ? __ldcg(src + i) : make_uint4(0, 0, 0, 0);
        }
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const uint32_t w4[4] = {v[j].x, v[j].y, v[j].z, v[j].w};
#pragma unroll
          for (int q = 0; q < 4; ++q) {
            const float lo = bf16_lo(w4[q]), hi = bf16_hi(w4[q]);
            s += lo * lo + hi * hi;
          }
        }
      }
      ss[b] = warp_sum(s);
    }
    if (lane == 0) {
#pragma unroll
      for (int b = 0; b < 8; ++b) s_ss[warp][b] = ss[b];
    }
    consumer_bar();
    if (threadIdx.x < 8) {
      float tot = 0.f;
#pragma unroll
      for (int w = 0; w < kTW; ++w) tot += s_ss[w][threadIdx.x];
      s_rstd[threadIdx.x] = rsqrtf(tot / (float)K + a.norm_eps);
    }
    consumer_bar();
  }
  tma_stage_x_seg(p, xs, s_rstd, seg, pre);
}

// ---- bulk-copy staging: every batch row of the segment flies at once (one latency, no registers) ----
// The per-row load loops above pay one L2 round trip per batch row and pass (sum of squares, then the copy): ~10 us per
// GEMV at 5 beams.  Here thread 0 issues one cp.async.bulk per row, all 256 consumers wait on one mbarrier, and the
// RMSNorm (whole-row staging only) is applied in place from shared memory.
static __device__ __forceinline__ void bulk_g2s(void* dst, const void* src, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(dst)),
               "l"(src), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}
static __device__ __forceinline__ void tma_stage_x_bulk(const GemvTmaParams& p, bf16* xs, float (*s_ss)[8], float* s_rstd,
                                                        int seg, const XPre* pre, uint64_t* xbar, uint32_t& xphase) {
  const GemvArgs& a = p.a;
  const int K = a.K, B = a.B;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int xsc = (p.xsc > 0 && p.xsc < p.cpt) ? p.xsc : p.cpt;
  const int col0 = seg * xsc * kTCols;
  const int ncols_pad = min(xsc, p.cpt - seg * xsc) * kTCols;
  const int ncols = min(ncols_pad, K - col0);
  if (threadIdx.x == 0) {
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");  // earlier reads of xs are ordered before the async writes
    mbar_expect_tx(xbar, (uint32_t)B * (uint32_t)ncols * 2u);
    for (int b = 0; b < B; ++b) bulk_g2s(xs + (long)b * p.ldxs, a.x + (long)b * a.ldx + col0, (uint32_t)ncols * 2u, xbar);
  }
  const int padv = (ncols_pad - ncols) >> 3;  // zero the columns past K (generic writes, disjoint from the copies)
  for (int i = threadIdx.x; i < B * padv; i += 256) {
    const int b = i / padv, j = i - b * padv;
    reinterpret_cast<uint4*>(xs + (long)b * p.ldxs + ncols)[j] = make_uint4(0, 0, 0, 0);
  }
  mbar_wait(xbar, xphase);
  xphase ^= 1;
  if (a.norm_w != nullptr) {  // whole row staged (host guarantees it): LlamaRMSNorm in place
    const int vec_per_row = K >> 3;
    float ss[8];
#pragma unroll
    for (int b = 0; b < 8; ++b) ss[b] = 0.f;
#pragma unroll
    for (int b = 0; b < 8; ++b) {
      if (b < B) {
        const uint4* row = reinterpret_cast<const uint4*>(xs + (long)b * p.ldxs);
        float s = 0.f;
        for (int i = threadIdx.x; i < vec_per_row; i += 256) {
          const uint4 v = row[i];
          const uint32_t w4[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
          for (int q = 0; q < 4; ++q) {
            const float lo = bf16_lo(w4[q]), hi = bf16_hi(w4[q]);
            s += lo * lo + hi * hi;
          }
        }
        ss[b] = warp_sum(s);
      }
    }
    if (lane == 0) {
#pragma unroll
      for (int b = 0; b < 8; ++b) s_ss[warp][b] = ss[b];
    }
    consumer_bar();
    if (threadIdx.x < 8) {
      float tot = 0.f;
#pragma unroll
      for (int w = 0; w < kTW; ++w) tot += s_ss[w][threadIdx.x];
      s_rstd[threadIdx.x] = rsqrtf(tot / (float)K + a.norm_eps);
    }
    consumer_bar();
    const uint4* wsrc = reinterpret_cast<const uint4*>(a.norm_w);
    const bool use_pre = pre != nullptr && pre->have;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int i = (int)threadIdx.x + 256 * j;
      if (i >= vec_per_row) break;
      const uint4 w = use_pre ? pre->w[j] : __ldg(wsrc + i);
      const uint32_t w4[4] = {w.x, w.y, w.z, w.w};
      uint4 v[8];
#pragma unroll
      for (int b = 0; b < 8; ++b)  // every row's vector is requested before the first is used
        if (b < B) v[b] = reinterpret_cast<const uint4*>(xs + (long)b * p.ldxs)[i];
#pragma unroll
      for (int b = 0; b < 8; ++b) {
        if (b < B) {
          const float rstd = s_rstd[b];
          const uint32_t v4[4] = {v[b].x, v[b].y, v[b].z, v[b].w};
          uint32_t o4[4];
#pragma unroll
          for (int q = 0; q < 4; ++q) o4[q] = rmsnorm_pair(v4[q], rstd, w4[q]);  // HF: weight * (x.float() * rsqrt(var + eps)).to(bf16)
          reinterpret_cast<uint4*>(xs + (long)b * p.ldxs)[i] = make_uint4(o4[0], o4[1], o4[2], o4[3]);
        }
      }
    }
    for (int i = (int)threadIdx.x + 1024; i < vec_per_row; i += 256) {  // K > 8192
      const uint4 w = __ldg(wsrc + i);
      const uint32_t w4[4] = {w.x, w.y, w.z, w.w};
      for (int b = 0; b < B; ++b) {
        uint4* row = reinterpret_cast<uint4*>(xs + (long)b * p.ldxs);
        const float rstd = s_rstd[b];
        const uint4 v = row[i];
        const uint32_t v4[4] = {v.x, v.y, v.z, v.w};
        uint32_t o4[4];
#pragma unroll
        for (int q = 0; q < 4; ++q) o4[q] = rmsnorm_pair(v4[q], rstd, w4[q]);
        row[i] = make_uint4(o4[0], o4[1], o4[2], o4[3]);
      }
    }
  }
  consumer_bar();
}

// ---- consumers: pull this CTA's chunks [c0, c1) out of the ring, mma them against xs, finish row groups ----
static __device__ __forceinline__ void tma_consume(const GemvTmaParams* sp, long c0, long c1, uint8_t* ring,
                                                   uint64_t* full_bar, uint64_t* empty_bar, float* red, float* fin,
                                                   bf16* xs, int* s_last, int& stage, uint32_t& phase,
                                                   const float* s_rstd = nullptr, uint64_t* xbar = nullptr,
                                                   uint32_t* xphase = nullptr) {
  const GemvTmaParams& p = *sp;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int g = lane >> 2, t = lane & 3;
  const int B = p.a.B, CPT = p.cpt;
  const int n = (int)(c1 - c0);
  float acc[kTRT][4];
#pragma unroll
  for (int rt = 0; rt < kTRT; ++rt)
#pragma unroll
    for (int q = 0; q < 4; ++q) acc[rt][q] = 0.f;
  // fragment addressing inside a 128B-swizzled [32 rows x 64 cols] TMA tile
  const int tile_j = warp >> 1;                   // which 64-column tile of the chunk this warp reads
  const int cbase = (warp & 1) * 4;               // first logical 16-byte chunk of this warp's 32 columns
  const int lrow = lane & 15, lhalf = lane >> 4;  // ldmatrix.x4 lane -> (row, k-half)
  const bool has_x = g < B;
  const bf16* xrow = xs + (long)g * p.ldxs + warp * 32 + 2 * t;
  int cp_grp = (int)(c0 / CPT), cp_kc = (int)(c0 % CPT);
  int seg_lo = cp_kc;
  const int xsc = (p.xsc > 0 && p.xsc < CPT) ? p.xsc : CPT;  // chunks per staged x segment
  int cur_seg = cp_kc / xsc;                                  // the caller staged this segment (tma_stage_x(.., seg))
  int k_in_seg = cp_kc - cur_seg * xsc;                       // tracked incrementally: no division in the chunk loop
  for (int i = 0; i < n; ++i) {
    // leave the staged K segment?  (never when the whole row is staged: xsc == CPT)
    bool restage = false;
    if (cp_kc == 0) {  // a new row group starts at column 0
      if (cur_seg != 0) { cur_seg = 0; restage = true; }
      k_in_seg = 0;
    } else if (k_in_seg == xsc) {  // ran off the end of the segment inside a row
      ++cur_seg;
      k_in_seg = 0;
      restage = true;
    }
    if (restage) {  // all 8 consumer warps take this branch together (same chunk stream)
      consumer_bar();
      if (p.xbulk) tma_stage_x_bulk(p, xs, nullptr, nullptr, cur_seg, nullptr, xbar, *xphase);  // segmented => no norm
      else tma_stage_x_seg(p, xs, s_rstd, cur_seg);
    }
    mbar_wait(&full_bar[stage], phase);
    const uint32_t tbase = smem_u32(ring + stage * kTStageBytes + tile_j * (kTRows * 128));
    const bf16* xk = xrow + k_in_seg * kTCols;
#pragma unroll
    for (int ks = 0; ks < 2; ++ks) {
      uint32_t bfr[2] = {0u, 0u};
      if (has_x) {
        bfr[0] = *reinterpret_cast<const uint32_t*>(xk + ks * 16);
        bfr[1] = *reinterpret_cast<const uint32_t*>(xk + ks * 16 + 8);
      }
#pragma unroll
      for (int rt = 0; rt < kTRT; ++rt) {
        const int r = rt * 16 + lrow;
        const int c = cbase + ks * 2 + lhalf;
        uint32_t af[4];
        ldmatrix_x4(af, tbase + r * 128 + ((c ^ (r & 7)) << 4));
        mma_bf16_16816(acc[rt], af, bfr);
      }
    }
    __syncwarp();
    if (lane == 0) mbar_arrive(&empty_bar[stage]);
    if (++stage == p.nstages) { stage = 0; phase ^= 1; }
    const bool grp_done = (cp_kc == CPT - 1) || (i == n - 1);
    if (grp_done) {
#pragma unroll
      for (int rt = 0; rt < kTRT; ++rt) {
        float* r = red + (warp * kTRT + rt) * 128;
        r[g * 8 + 2 * t] = acc[rt][0];
        r[g * 8 + 2 * t + 1] = acc[rt][1];
        r[(g + 8) * 8 + 2 * t] = acc[rt][2];
        r[(g + 8) * 8 + 2 * t + 1] = acc[rt][3];
        acc[rt][0] = acc[rt][1] = acc[rt][2] = acc[rt][3] = 0.f;
      }
      gemv_tma_flush(sp, red, fin, s_last, cp_grp, seg_lo, cp_kc);
    }
    ++k_in_seg;
    if (++cp_kc == CPT) { cp_kc = 0; ++cp_grp; }
    if (grp_done) seg_lo = cp_kc;
  }
}

}  // namespace emu
