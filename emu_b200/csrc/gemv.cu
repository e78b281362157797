// emu_b200 — weight-streaming skinny GEMM for the autoregressive decode loop.
//
// y[b, n] = epilogue( sum_k x[b, k] * W[n, k] ),  1 <= b <= 8 (batch x beams), W bf16 row-major [N, K].
//
// This is the dominant kernel of the headline metric: per decoded token the LLaMA-33B decoder streams
// 64.6 GB of bf16 weights (HF LlamaDecoderLayer q/k/v/o/gate/up/down + lm_head, driven from
// Emu2/emu/emu.py:213-229 and :133-138), so the kernel is judged on HBM GB/s, not FLOPs.
//
// The bytes in flight live in shared memory:
//   * one producer thread issues cp.async.bulk.tensor (TMA) loads of [32 rows x 64 cols] 128B-swizzled tiles into an
//     8-stage x 16 KB ring signalled by mbarriers — 128 KB in flight per SM with zero registers and zero address math
//     (a deep prefetch rather than a shallower ring that would let the PDL successor co-reside);
//   * 8 consumer warps pull A fragments with ldmatrix (conflict-free through the swizzle) and run mma.sync.m16n8k16 with
//     the staged x rows as the 8-wide N operand, then release the stage — batch 1..8 (greedy .. 5-beam search) all run
//     at the same bandwidth-bound speed;
//   * ONE persistent CTA per SM (grid = kNumSMs), stream-K over (row group, k chunk) units: every CTA gets the same
//     number of consecutive chunks (+-1), so all SMs stream the same number of bytes whatever N and K are.  A row group
//     whose chunks straddle CTAs is finished by whichever CTA arrives last (per-group counter; partial sums are added in a
//     fixed order, so results are run-to-run deterministic).  With PDL the producer starts streaming weights before
//     griddepcontrol.wait resolves.
// x (batch <= 8 rows) reaches shared memory by one cp.async.bulk per row, optionally through a fused RMSNorm (HF
// LlamaRMSNorm rounding) applied in place.  When batch x K does not fit next to the ring (5 beams x 17920) x is staged in
// K segments that are re-staged as the chunk stream crosses them (GemvTmaParams::xsc).
// Ragged N and K tails cost nothing (TMA zero-fills out-of-bounds rows/columns).
// Epilogues: bias / residual / SwiGLU / RoPE + KV-cache append / tensor-parallel {value, flag} push.
#include <stdio.h>

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
  int ldxs;      // smem row stride of staged x (elements), = xsc * 256 + 8
  int kpad;      // K rounded up to 256
  int cpt;       // chunks per row group
  int xsc;       // chunks of x staged in shared memory at a time (== cpt: the whole row; smaller: K segments that are
                 //   re-staged as the chunk stream crosses them — batch x K too large for shared memory, e.g. 5 x 17920)
  int nstages;   // ring depth actually used (<= kTStages)
  int geff;      // number of CTAs that share this matrix's chunks (<= gridDim.x); CTAs >= geff get none
  long total;    // total chunks
  float* ws;     // [groups][kTMaxParts][kTRT*128]
  int* counters;
};

static __device__ __forceinline__ void consumer_bar() { asm volatile("bar.sync 1, 256;" ::: "memory"); }

// finish k-segment [kc_lo, kc_hi] of row group grp (consumer threads only; `red` already holds per-warp partials).
// Kept out of line: it runs once per row group, and inlining it into the chunk loop bloats the instruction stream.
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
    // owner(x) = largest c with floor(c*total/G) <= x  =  floor(((x+1)*G - 1) / total)
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
      if (prev == nparts - 1) p.counters[grp] = 0;  // self-reset for the next launch / graph replay
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
    // fin[rt*128 + r*8 + b] holds the full dot product of row (grp*kTRT + rt)*16 + r with x[b]
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
            // HF apply_rotary_pos_emb in bf16: (q*cos) + (rotate_half(q)*sin), each op rounded
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
// latency: every batch row of a segment is one bulk copy, all in flight at once, and the norm weights — which do not
// depend on the predecessor kernel — are fetched by the caller before griddepcontrol.wait (XPre).
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

// per-warp sums of squares of every batch row -> s_rstd[b], folded over the warps in a fixed order
static __device__ __forceinline__ void rstd_from_ss(const float (&ss)[8], float (*s_ss)[8], float* s_rstd, int K, float eps) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (lane == 0) {
#pragma unroll
    for (int b = 0; b < 8; ++b) s_ss[warp][b] = ss[b];
  }
  consumer_bar();
  if (threadIdx.x < 8) {
    float tot = 0.f;
#pragma unroll
    for (int w = 0; w < kTW; ++w) tot += s_ss[w][threadIdx.x];
    s_rstd[threadIdx.x] = rsqrtf(tot / (float)K + eps);
  }
  consumer_bar();
}

// RMSNorm statistics of x read from global memory: a segmented row is never whole in shared memory
static __device__ __forceinline__ void x_norm_stats_global(const GemvTmaParams& p, float (*s_ss)[8], float* s_rstd) {
  const GemvArgs& a = p.a;
  const int K = a.K, B = a.B;
  const int vec_per_row = K >> 3;
  float ss[8];
#pragma unroll
  for (int b = 0; b < 8; ++b) ss[b] = 0.f;
  for (int b = 0; b < B; ++b) {
    const uint4* src = reinterpret_cast<const uint4*>(a.x + (long)b * a.ldx);
    float s = 0.f;
    for (int i0 = 0; i0 < vec_per_row; i0 += 1024) {
      uint4 v[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) {  // four independent loads in flight per thread
        const int i = i0 + (int)threadIdx.x + 256 * j;
        // activations may have been produced by other CTAs of this very kernel's predecessor: bypass L1
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
  rstd_from_ss(ss, s_ss, s_rstd, K, a.norm_eps);
}

// Columns [seg * xsc * 256, (seg + 1) * xsc * 256) of every batch row (the whole row when xsc == cpt): thread 0 issues one
// cp.async.bulk per row, all 256 consumers wait on one mbarrier, and the RMSNorm is applied in place.  Its statistics come
// from shared memory when the whole row is staged; a segmented row's are already in s_rstd (x_norm_stats_global).
static __device__ __forceinline__ void stage_x(const GemvTmaParams& p, bf16* xs, float (*s_ss)[8], float* s_rstd, int seg,
                                               const XPre* pre, uint64_t* xbar, uint32_t& xphase) {
  const GemvArgs& a = p.a;
  const int K = a.K, B = a.B;
  const int col0 = seg * p.xsc * kTCols;
  const int ncols_pad = min(p.xsc, p.cpt - seg * p.xsc) * kTCols;
  const int ncols = min(ncols_pad, K - col0);
  if (threadIdx.x == 0) {
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");  // earlier accesses of xs are ordered before the async writes
    mbar_expect_tx(xbar, (uint32_t)B * (uint32_t)ncols * 2u);
    for (int b = 0; b < B; ++b) bulk_load_1d(xs + (long)b * p.ldxs, a.x + (long)b * a.ldx + col0, (uint32_t)ncols * 2u, xbar);
  }
  const int padv = (ncols_pad - ncols) >> 3;  // zero the columns past K (generic writes, disjoint from the copies)
  for (int i = threadIdx.x; i < B * padv; i += 256) {
    const int b = i / padv, j = i - b * padv;
    reinterpret_cast<uint4*>(xs + (long)b * p.ldxs + ncols)[j] = make_uint4(0, 0, 0, 0);
  }
  mbar_wait(xbar, xphase);
  xphase ^= 1;
  if (a.norm_w != nullptr) {
    const int nvec = ncols >> 3;  // 16-byte vectors of this segment inside K
    if (p.xsc == p.cpt) {
      float ss[8];
#pragma unroll
      for (int b = 0; b < 8; ++b) ss[b] = 0.f;
#pragma unroll
      for (int b = 0; b < 8; ++b) {
        if (b < B) {
          const uint4* row = reinterpret_cast<const uint4*>(xs + (long)b * p.ldxs);
          float s = 0.f;
          for (int i = threadIdx.x; i < nvec; i += 256) {
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
      rstd_from_ss(ss, s_ss, s_rstd, K, a.norm_eps);
    }
    const uint4* wsrc = reinterpret_cast<const uint4*>(a.norm_w) + (col0 >> 3);
    // The first stage requests every row's vector before it uses the first.  Re-stages (no XPre) normalise row by row:
    // they are inlined into the chunk loop, whose registers the batched loads would spill.
    int i = threadIdx.x;
    if (pre != nullptr) {
      const bool use_pre = seg == 0 && pre->have;
#pragma unroll
      for (int j = 0; j < 4; ++j, i += 256) {
        if (i >= nvec) break;
        const uint4 w = use_pre ? pre->w[j] : __ldg(wsrc + i);
        const uint32_t w4[4] = {w.x, w.y, w.z, w.w};
        uint4 v[8];
#pragma unroll
        for (int b = 0; b < 8; ++b)
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
    }
    for (; i < nvec; i += 256) {  // re-stages, and the columns past 8192 of the first stage
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
                                                   bf16* xs, int* s_last, int& stage, uint32_t& phase, float* s_rstd,
                                                   uint64_t* xbar, uint32_t& xphase) {
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
  const int xsc = p.xsc;       // chunks per staged x segment
  int cur_seg = cp_kc / xsc;   // the caller staged this segment
  int k_in_seg = cp_kc - cur_seg * xsc;  // tracked incrementally: no division in the chunk loop
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
      stage_x(p, xs, nullptr, s_rstd, cur_seg, nullptr, xbar, xphase);  // segmented: the statistics are in s_rstd
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

// consumer threads (256) of the first ll_red CTAs, after their own rows are pushed: finish the tensor-parallel exchange
// (GemvArgs::ll_h).  The words polled here are written by the epilogues of this very kernel — on this rank (all CTAs are
// resident: grid <= SM count) and on the peers.
static __device__ __forceinline__ void gemv_tail_reduce(const GemvArgs& a) {
  const unsigned epoch = __ldcg(a.ll_step) * 256u + (unsigned)a.ll_idx + 1u;
  const int R = a.ll_red;
  const uint4* base = reinterpret_cast<const uint4*>(a.ll_peer[a.ll_rank]) + ((size_t)(a.ll_idx & 1) * a.ll_n * a.ll_slot_elems) / 2;
  const long n2 = ((long)a.B * a.ldy) >> 1;  // element pairs of h [B, ldy]
  const long per = (n2 + R - 1) / R;
  const long i0 = (long)blockIdx.x * per, i1 = min(n2, i0 + per);
  uint32_t* h = reinterpret_cast<uint32_t*>(a.ll_h);
  for (long i = i0 + threadIdx.x; i < i1; i += 256) {
    float a0 = 0.f, a1 = 0.f;
    for (int r = 0; r < a.ll_n; ++r) {
      const uint4* w = base + ((size_t)r * a.ll_slot_elems) / 2 + i;
      uint4 v;
      unsigned long long t0 = 0, now;
      for (;;) {
        asm volatile("ld.volatile.global.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(w));
        if (v.y == epoch && v.w == epoch) break;
        asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(now));
        if (t0 == 0) t0 = now;
        else if (now - t0 > 20000000000ull) {  // 20 s: a peer died — fail loudly instead of hanging the GPU
          printf("emu_b200: tensor-parallel exchange %d timed out waiting for rank %d\n", a.ll_idx, r);
          __trap();
        }
      }
      a0 += __uint_as_float(v.x);  // fixed rank order: bitwise identical on every rank
      a1 += __uint_as_float(v.z);
    }
    const uint32_t hv = __ldcg(h + i);
    h[i] = pack_bf16(bf16_lo(hv) + round_bf16(a0), bf16_hi(hv) + round_bf16(a1));
  }
}

__global__ void __launch_bounds__(kTThreads, 2) gemv_tma_kernel(const __grid_constant__ CUtensorMap tmW,
                                                                const __grid_constant__ GemvTmaParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* ring = smem;                                                   // nstages x 16 KB
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(ring + p.nstages * kTStageBytes);
  uint64_t* empty_bar = full_bar + kTStages;
  float* red = reinterpret_cast<float*>(empty_bar + kTStages);            // [8 warps][kTRT*128]
  float* fin = red + kTW * kTRT * 128;                                    // [kTRT*128]
  bf16* xs = reinterpret_cast<bf16*>(fin + kTRT * 128);                   // [B][ldxs]
  __shared__ float s_ss[kTW][8];
  __shared__ float s_rstd[8];
  __shared__ int s_last;
  __shared__ GemvTmaParams s_params;
  __shared__ __align__(8) uint64_t s_xbar;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  // diagnostics: {globaltimer at entry; clock64 at entry, barriers ready, dependency resolved, x staged, first weight chunk
  // landed (consumer side), own chunks consumed + rows flushed, exit}
  unsigned long long* dbg = p.a.dbg ? p.a.dbg + (size_t)blockIdx.x * 8 : nullptr;
  auto clk = [] { unsigned long long t; asm volatile("mov.u64 %0, %%clock64;" : "=l"(t)); return t; };
  if (dbg && threadIdx.x == 0) {
    unsigned long long g;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(g));
    dbg[0] = g;
    dbg[1] = clk();
  }
  const long G = p.geff;  // == gridDim.x for this kernel
  const long c0 = (long)blockIdx.x * p.total / G, c1 = ((long)blockIdx.x + 1) * p.total / G;
  // the launch parameters are re-read from shared memory by the flush routine: copy them with the whole CTA (one word
  // per thread) instead of one thread walking ~350 bytes
  for (int i = threadIdx.x; i < (int)(sizeof(GemvTmaParams) / 4); i += blockDim.x)
    reinterpret_cast<uint32_t*>(&s_params)[i] = reinterpret_cast<const uint32_t*>(&p)[i];
  if (threadIdx.x == 0) tma_prefetch_desc(&tmW);
  if (threadIdx.x < kTStages) {  // one barrier pair per thread: a single thread walking 20 inits costs ~0.3 us per launch
    mbar_init(&full_bar[threadIdx.x], 1);
    mbar_init(&empty_bar[threadIdx.x], kTW);
    mbar_fence_init();
  } else if (threadIdx.x == 32) {
    mbar_init(&s_xbar, 1);
    mbar_fence_init();
  }
  __syncthreads();
  if (dbg && threadIdx.x == 0) dbg[2] = clk();
  if (p.a.pdl) pdl_launch_dependents();
  int stage = 0;
  uint32_t phase = 0;
  if (warp == kTW) {
    // producer: weights do not depend on the previous kernel, so the ring fills before griddepcontrol.wait resolves
    if (lane == 0) tma_produce(&tmW, p.cpt, c0, c1, ring, full_bar, empty_bar, p.nstages, stage, phase);
    return;
  }
  XPre pre;
  tma_prefetch_norm_w(p, pre);  // weights of the fused RMSNorm: independent of the predecessor, fetched while it drains
  if (p.a.pdl) pdl_wait();
  if (dbg && threadIdx.x == 0) dbg[3] = clk();
  if (p.a.norm_w != nullptr && p.xsc < p.cpt) x_norm_stats_global(p, s_ss, s_rstd);
  uint32_t xphase = 0;
  stage_x(p, xs, s_ss, s_rstd, (int)(c0 % p.cpt) / p.xsc, &pre, &s_xbar, xphase);
  if (dbg && threadIdx.x == 0) {
    dbg[4] = clk();
    if (c0 < c1) mbar_wait(&full_bar[0], 0);  // (diagnostic only) when did the first chunk land?
    dbg[5] = clk();
  }
  tma_consume(&s_params, c0, c1, ring, full_bar, empty_bar, red, fin, xs, &s_last, stage, phase, s_rstd, &s_xbar, xphase);
  if (dbg && threadIdx.x == 0) dbg[6] = clk();
  if (p.a.ll_n > 0 && p.a.ll_h != nullptr && (int)blockIdx.x < p.a.ll_red) gemv_tail_reduce(p.a);
  if (dbg && threadIdx.x == 0) dbg[7] = clk();
}

static float* g_tws = nullptr;
static int* g_tcounters = nullptr;

int gemv_init() {
  if (g_tws) return EMU_OK;
  if (cudaMalloc((void**)&g_tws, (size_t)kTWsGroups * kTMaxParts * kTRT * 128 * sizeof(float)) != cudaSuccess) return EMU_ERR_NOMEM;
  if (cudaMalloc((void**)&g_tcounters, (size_t)kTWsGroups * sizeof(int)) != cudaSuccess) return EMU_ERR_NOMEM;
  if (cudaMemset(g_tcounters, 0, (size_t)kTWsGroups * sizeof(int)) != cudaSuccess) return EMU_ERR_CUDA;
  if (cudaFuncSetAttribute(gemv_tma_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024) != cudaSuccess)
    return EMU_ERR_CUDA;
  // ask for the largest shared-memory carve-out so that this kernel's CTA and its PDL successor's CTA (2 x ~105 KB)
  // can be resident on one SM at the same time
  if (cudaFuncSetAttribute(gemv_tma_kernel, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared) !=
      cudaSuccess)
    return EMU_ERR_CUDA;
  return EMU_OK;
}

int gemv_bf16(const GemvArgs& a, cudaStream_t st) {
  // everything the kernel cannot take is refused here, before any CUDA call
  if (a.B < 1 || a.B > 8 || a.N < 1 || a.K < 32 || (a.K % 32) || (a.ldx % 8)) return EMU_ERR_INVALID;
  if ((a.mode == EPI_SWIGLU || a.mode == GEMV_ROPE_QKV) && (a.N % 16)) return EMU_ERR_INVALID;
  // W is read by TMA and x by bulk copies: both need 16-byte aligned rows (ldx % 8 == 0 carries x's alignment to every row)
  if ((reinterpret_cast<uintptr_t>(a.W) | reinterpret_cast<uintptr_t>(a.x)) & 15) return EMU_ERR_INVALID;
  const int groups = (a.N + kTRows - 1) / kTRows;
  if (groups > kTWsGroups) return EMU_ERR_INVALID;  // the stream-K workspace holds N <= 262144 rows
  if (a.ll_n > 0 && a.ll_h && (a.ll_red < 1 || (a.ldy & 1))) return EMU_ERR_INVALID;
  if (!g_tws) {  // first use must happen outside stream capture (the engine calls gemv_init() at create)
    int rc = gemv_init();
    if (rc) return rc;
  }
  GemvTmaParams p;
  p.a = a;
  p.kpad = (a.K + kTCols - 1) / kTCols * kTCols;
  p.cpt = p.kpad / kTCols;
  p.xsc = p.cpt;
  p.ldxs = p.kpad + 8;  // row stride = 16 B (mod 128 B): the 8 batch rows hit distinct bank groups
  // batch x K too large to keep all of x in shared memory next to a deep ring (5 beams x 17920 = 179 KB): stage x in K
  // segments of <= 88 KB instead, re-staged as the chunk stream crosses them.  With B <= 8 a segment holds >= 21 chunks.
  const size_t budget = 88 * 1024;
  if ((size_t)a.B * p.ldxs * 2 > budget) {
    p.xsc = (int)((budget / ((size_t)a.B * 2) - 8) / kTCols);
    p.ldxs = p.xsc * kTCols + 8;
  }
  p.total = (long)groups * p.cpt;
  p.ws = g_tws;
  p.counters = g_tcounters;
  const size_t xs_bytes = (size_t)a.B * p.ldxs * 2;
  // the ring buffers are carved for kTStages; 8 stages = 128 KB in flight per SM, and a CTA with a wide x uses fewer so
  // that this kernel (<= ~110 KB) and its PDL successor still fit one SM together.  x is at most 88 KB, so even the
  // 3-stage floor fits the 200 KB the kernel is allowed.
  p.nstages = 8;
  size_t smem;
  for (;;) {  // shrink the ring until the CTA fits (wide x at batch > 1)
    smem = 1024 + (size_t)p.nstages * kTStageBytes + 2 * kTStages * 8 + (size_t)(kTW + 1) * kTRT * 128 * 4 + xs_bytes + 64;
    if (smem <= 200 * 1024 || p.nstages <= 3) break;
    --p.nstages;
  }
  long grid = kNumSMs;
  if (grid > p.total) grid = p.total;
  const long max_grid = (long)groups * (kTMaxParts - 3);  // a row group is shared by at most kTMaxParts CTAs
  if (grid > max_grid) grid = max_grid;
  p.geff = (int)grid;
  if (p.a.ll_n > 0 && p.a.ll_h && p.a.ll_red > (int)grid) p.a.ll_red = (int)grid;
  CUtensorMap tm;
  if (int rc = make_tmap_2d(&tm, a.W, a.N, a.K, a.K, kTRows)) return rc;
  return launch_kernel(gemv_tma_kernel, dim3((unsigned)grid), dim3(kTThreads), smem, st, a.pdl, tm, p);
}

}  // namespace emu
