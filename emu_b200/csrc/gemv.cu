// emu_b200 — weight-streaming skinny GEMM for the autoregressive decode loop.
//
// y[b, n] = epilogue( sum_k x[b, k] * W[n, k] ),  1 <= b <= 8 (batch x beams), W bf16 row-major [N, K].
//
// This is the dominant kernel of the headline metric: per decoded token the LLaMA-33B decoder streams
// 64.6 GB of bf16 weights (HF LlamaDecoderLayer q/k/v/o/gate/up/down + lm_head, driven from
// Emu2/emu/emu.py:213-229 and :133-138), so the kernel is judged on HBM GB/s, not FLOPs.
//
// Work decomposition ("stream-K"): the weight matrix is cut into chunks of (16*RT rows) x 256 columns.  A
// persistent grid of 2 CTAs per SM gives every CTA the SAME number of consecutive chunks (+-1), so all SMs stream
// the same number of bytes and finish together — no wave quantisation whatever N and K are.  A row group whose chunks straddle
// CTAs is finished by whichever CTA arrives last (per-group counter; partial sums are added in a fixed order, so
// results are run-to-run deterministic).
//
// Inside a CTA the 8 warps each own one 32-column block of the current chunk; every lane streams 16-byte pieces
// of 2*RT rows with ld.global.nc.L1::no_allocate (each request = 64 B contiguous per row, 8 rows) through a
// register ring holding 16 loads in flight per lane (128 KB per SM), with plain pointer increments in the steady
// state (~11 SASS instructions per KB; a first stream-K cut with 16-row chunks and per-chunk address math was
// instruction-issue bound at 3 TB/s).  The tiny x operand (<= 8 rows) is staged once per CTA in shared memory —
// optionally through a fused RMSNorm prologue (HF LlamaRMSNorm rounding) — and fed as the 8-wide N operand of
// mma.sync.m16n8k16, so batch 1..8 (greedy .. 5-beam search) all run at the same bandwidth-bound speed.
// Epilogues: bias / residual / SwiGLU / RoPE + KV-cache append.  Launched with programmatic dependent launch: the
// ring is filled before griddepcontrol.wait, so HBM keeps streaming while the previous kernel drains.
#include <stdlib.h>

#include "common.cuh"
#include "ops.h"

namespace emu {

int gemv_tma_bf16(const GemvArgs& a, cudaStream_t st);  // gemv_tma.cu
int gemv_tma_init();
int gemv_reg_bf16(const GemvArgs& a, cudaStream_t st);

constexpr int kGemvWarps = 8;
constexpr int kGemvThreads = kGemvWarps * 32;
constexpr int kMaxParts = 8;    // CTAs that may share one row group
constexpr int kWsTiles = 8192;  // workspace capacity in 16-row tiles (N <= 131072)

struct GemvParams {
  GemvArgs a;
  int ldxs;       // smem row stride of staged x (elements)
  int red_off;    // byte offset of the reduction buffers
  int cpt;        // chunks per row group (= ceil(K / 256))
  int rt;         // 16-row tiles per group
  long total;     // total chunks
  float* ws;      // [groups][kMaxParts][rt*128]
  int* counters;  // [groups], self-resetting
};

// Finish the k-segment [kc_lo, kc_hi] of row group `grp`; per-warp partial sums are already in `red`.
// Called uniformly by all threads of the CTA.  Kept out of line: it runs once per row group, and inlining it into
// the unrolled streaming loop blew the instruction cache.
__device__ __noinline__ void gemv_flush(const GemvParams* sp, float* red, float* fin, int* s_last_p, int grp, int kc_lo,
                                        int kc_hi) {
  const GemvParams& p = *sp;
  const GemvArgs& a = p.a;
  const int N = a.N, B = a.B, CPT = p.cpt, RT = p.rt;
  const int nval = RT * 128;
  const long G = gridDim.x;
  __syncthreads();
  const bool whole = (kc_lo == 0 && kc_hi == CPT - 1);
  bool do_epilogue = whole;
  if (whole) {
    for (int idx = threadIdx.x; idx < nval; idx += kGemvThreads) {
      float v = 0.f;
#pragma unroll
      for (int w = 0; w < kGemvWarps; ++w) v += red[w * nval + idx];
      fin[idx] = v;
    }
  } else {
    // owner(x) = largest c with floor(c*total/G) <= x  =  floor(((x+1)*G - 1) / total)
    const long first_chunk = (long)grp * CPT;
    const int first_owner = (int)(((first_chunk + 1) * G - 1) / p.total);
    const int last_owner = (int)(((first_chunk + CPT) * G - 1) / p.total);
    const int nparts = last_owner - first_owner + 1;
    const int my = (int)blockIdx.x - first_owner;
    float* wt = p.ws + ((long)grp * kMaxParts) * nval;
    for (int idx = threadIdx.x; idx < nval; idx += kGemvThreads) {
      float v = 0.f;
#pragma unroll
      for (int w = 0; w < kGemvWarps; ++w) v += red[w * nval + idx];
      wt[my * nval + idx] = v;
    }
    __threadfence();
    __syncthreads();
    if (threadIdx.x == 0) {
      const int prev = atomicAdd(&p.counters[grp], 1);
      *s_last_p = (prev == nparts - 1);
      if (prev == nparts - 1) p.counters[grp] = 0;  // self-reset for the next launch / graph replay
    }
    __syncthreads();
    do_epilogue = *s_last_p != 0;
    if (do_epilogue) {
      __threadfence();
      for (int idx = threadIdx.x; idx < nval; idx += kGemvThreads) {
        float s = 0.f;
        for (int q = 0; q < nparts; ++q) s += __ldcg(&wt[q * nval + idx]);  // fixed order: deterministic
        fin[idx] = s;
      }
    }
  }
  if (do_epilogue) {  // uniform across the CTA
    __syncthreads();
    // fin[rt*128 + r*8 + b] holds the full dot product of row (grp*RT + rt)*16 + r with x[b]
    for (int idx = threadIdx.x; idx < nval; idx += kGemvThreads) {
      const int rt = idx >> 7, r = idx & 15, b = (idx >> 4) & 7;
      const float* f = fin + rt * 128;
      const int nrow = (grp * RT + rt) * 16 + r;
      if (b >= B || nrow >= N) continue;
      if (a.mode == EPI_NONE) {
        float v = f[r * 8 + b];
        if (a.bias) v += __bfloat162float(a.bias[nrow]);
        if (a.residual) v = round_bf16(v) + __bfloat162float(a.residual[(long)b * a.ldr + nrow]);
        if (a.out_fp32) reinterpret_cast<float*>(a.y)[(long)b * a.ldy + nrow] = v;
        else reinterpret_cast<bf16*>(a.y)[(long)b * a.ldy + nrow] = __float2bfloat16_rn(v);
      } else if (a.mode == EPI_SWIGLU) {
        if (r & 1) continue;
        const float gate = round_bf16(f[r * 8 + b]), up = round_bf16(f[(r + 1) * 8 + b]);
        const float v = round_bf16(silu(gate)) * up;
        reinterpret_cast<bf16*>(a.y)[(long)b * a.ldy + (nrow >> 1)] = __float2bfloat16_rn(v);
      } else {  // GEMV_ROPE_QKV
        const int D = a.head_dim, H = a.n_heads;
        const int hh = nrow / D, i = nrow - hh * D;
        const int slot = a.pos[b];
        if (hh < 2 * H) {
          if (r & 1) continue;
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
        } else {
          a.v_cache[(((long)b * H + (hh - 2 * H)) * a.t_max + slot) * D + i] = __float2bfloat16_rn(f[r * 8 + b]);
        }
      }
    }
  }
  __syncthreads();
}

// RT: 16-row tiles per chunk (1/2/4).  KFULL: K % 256 == 0, i.e. every warp's k-block is valid in every chunk.
template <int RT, bool KFULL>
__global__ void __launch_bounds__(kGemvThreads, 2) gemv_kernel(const GemvParams p) {
  constexpr int SLOTS = 8 / RT;  // ring slots, each RT*2 loads: 16 loads in flight per lane
  const GemvArgs& a = p.a;
  extern __shared__ __align__(16) uint8_t smem[];
  bf16* xs = reinterpret_cast<bf16*>(smem);
  float* red = reinterpret_cast<float*>(smem + p.red_off);  // [8 warps][RT][16][8]
  float* fin = red + kGemvWarps * RT * 128;                 // [RT][16][8]
  __shared__ float s_ss[kGemvWarps][8];
  __shared__ float s_rstd[8];
  __shared__ int s_last;
  __shared__ GemvParams s_params;
  if (threadIdx.x == 0) s_params = p;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int g = lane >> 2, t = lane & 3;
  const int K = a.K, N = a.N, B = a.B;
  const int KB = K >> 5, CPT = p.cpt;
  const long G = gridDim.x;
  const long c0 = (long)blockIdx.x * p.total / G, c1 = ((long)blockIdx.x + 1) * p.total / G;
  const int n = (int)(c1 - c0);

  // ---- load stream state: 2*RT row pointers that advance by 256 elements per chunk ----
  int ld_grp = (int)(c0 / CPT), ld_kc = (int)(c0 % CPT);
  const bf16* lp[RT][2];
  auto set_ptrs = [&](int grp, int kc) {
#pragma unroll
    for (int rt = 0; rt < RT; ++rt)
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        int row = (grp * RT + rt) * 16 + g + 8 * h;
        row = row < N ? row : N - 1;  // ragged last group: clamp (results of clamped rows are never stored)
        lp[rt][h] = a.W + (long)row * K + ((long)kc * kGemvWarps + warp) * 32 + t * 8;
      }
  };
  set_ptrs(ld_grp, ld_kc);
  uint4 ring[SLOTS][RT][2];
  auto load_next = [&](uint4(&slot)[RT][2]) {
    const bool valid = KFULL || (ld_kc * kGemvWarps + warp < KB);
#pragma unroll
    for (int rt = 0; rt < RT; ++rt)
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        slot[rt][h] = valid ? ldg_stream(lp[rt][h]) : make_uint4(0, 0, 0, 0);
        lp[rt][h] += 256;
      }
    if (++ld_kc == CPT) {
      ld_kc = 0;
      ++ld_grp;
      set_ptrs(ld_grp, 0);
    }
  };
  // weights do not depend on the previous kernel: fill the ring before the grid dependency resolves
#pragma unroll
  for (int j = 0; j < SLOTS; ++j)
    if (j < n) load_next(ring[j]);
  if (a.pdl) {
    pdl_launch_dependents();
    pdl_wait();
  }

  // ---- stage x (optionally RMS-normalised) into shared memory ----
  const int vec_per_row = K >> 3;
  if (a.norm_w != nullptr) {
    float ss[8];
#pragma unroll
    for (int b = 0; b < 8; ++b) ss[b] = 0.f;
    for (int b = 0; b < B; ++b) {
      const uint4* src = reinterpret_cast<const uint4*>(a.x + (long)b * a.ldx);
      float s = 0.f;
      for (int i = threadIdx.x; i < vec_per_row; i += kGemvThreads) {
        const uint4 v = src[i];
        const uint32_t w4[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const float lo = bf16_lo(w4[j]), hi = bf16_hi(w4[j]);
          s += lo * lo + hi * hi;
        }
      }
      ss[b] = warp_sum(s);
    }
    if (lane == 0) {
#pragma unroll
      for (int b = 0; b < 8; ++b) s_ss[warp][b] = ss[b];
    }
    __syncthreads();
    if (threadIdx.x < 8) {
      float tot = 0.f;
#pragma unroll
      for (int w = 0; w < kGemvWarps; ++w) tot += s_ss[w][threadIdx.x];
      s_rstd[threadIdx.x] = rsqrtf(tot / (float)K + a.norm_eps);
    }
    __syncthreads();
    for (int b = 0; b < B; ++b) {
      const float rstd = s_rstd[b];
      const uint4* src = reinterpret_cast<const uint4*>(a.x + (long)b * a.ldx);
      const uint4* wsrc = reinterpret_cast<const uint4*>(a.norm_w);
      uint4* dst = reinterpret_cast<uint4*>(xs + (long)b * p.ldxs);
      for (int i = threadIdx.x; i < vec_per_row; i += kGemvThreads) {
        const uint4 v = src[i], w = wsrc[i];
        const uint32_t v4[4] = {v.x, v.y, v.z, v.w}, w4[4] = {w.x, w.y, w.z, w.w};
        uint32_t o4[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          // HF: weight * (x.float() * rsqrt(var + eps)).to(bf16)
          const float lo = round_bf16(bf16_lo(v4[j]) * rstd) * bf16_lo(w4[j]);
          const float hi = round_bf16(bf16_hi(v4[j]) * rstd) * bf16_hi(w4[j]);
          o4[j] = pack_bf16(lo, hi);
        }
        dst[i] = make_uint4(o4[0], o4[1], o4[2], o4[3]);
      }
    }
  } else {
    for (int b = 0; b < B; ++b) {
      const uint4* src = reinterpret_cast<const uint4*>(a.x + (long)b * a.ldx);
      uint4* dst = reinterpret_cast<uint4*>(xs + (long)b * p.ldxs);
      for (int i = threadIdx.x; i < vec_per_row; i += kGemvThreads) dst[i] = src[i];
    }
  }
  __syncthreads();

  float acc[RT][4];
#pragma unroll
  for (int rt = 0; rt < RT; ++rt)
#pragma unroll
    for (int q = 0; q < 4; ++q) acc[rt][q] = 0.f;

  const bf16* xrow = xs + (long)g * p.ldxs + t * 8;
  const bool has_x = g < B;
  int cp_grp = (int)(c0 / CPT), cp_kc = (int)(c0 % CPT);
  int seg_lo = cp_kc;
  const bf16* xp = xrow + (cp_kc * kGemvWarps + warp) * 32;
  for (int base = 0; base < n; base += SLOTS) {
#pragma unroll
    for (int j = 0; j < SLOTS; ++j) {
      const int i = base + j;
      if (i < n) {
        if (KFULL || cp_kc * kGemvWarps + warp < KB) {
          uint4 xb = make_uint4(0, 0, 0, 0);
          if (has_x) xb = *reinterpret_cast<const uint4*>(xp);
          const uint32_t b1[2] = {xb.x, xb.y};
          const uint32_t b2[2] = {xb.z, xb.w};
#pragma unroll
          for (int rt = 0; rt < RT; ++rt) {
            const uint4 wa = ring[j][rt][0], wb = ring[j][rt][1];
            // K permutation shared by A and B: lane t feeds elements t*8+{0,1 | 2,3} to mma #1, {4,5 | 6,7} to #2
            const uint32_t a1[4] = {wa.x, wb.x, wa.y, wb.y};
            mma_bf16_16816(acc[rt], a1, b1);
            const uint32_t a2[4] = {wa.z, wb.z, wa.w, wb.w};
            mma_bf16_16816(acc[rt], a2, b2);
          }
        }
        xp += 256;
        if (i + SLOTS < n) load_next(ring[j]);
        const bool grp_done = (cp_kc == CPT - 1) || (i == n - 1);
        if (grp_done) {
#pragma unroll
          for (int rt = 0; rt < RT; ++rt) {
            float* r = red + (warp * RT + rt) * 128;
            r[g * 8 + 2 * t] = acc[rt][0];
            r[g * 8 + 2 * t + 1] = acc[rt][1];
            r[(g + 8) * 8 + 2 * t] = acc[rt][2];
            r[(g + 8) * 8 + 2 * t + 1] = acc[rt][3];
            acc[rt][0] = acc[rt][1] = acc[rt][2] = acc[rt][3] = 0.f;
          }
          gemv_flush(&s_params, red, fin, &s_last, cp_grp, seg_lo, cp_kc);
        }
        if (++cp_kc == CPT) { cp_kc = 0; ++cp_grp; xp = xrow + warp * 32; }
        if (grp_done) seg_lo = cp_kc;
      }
    }
  }
}

static float* g_ws = nullptr;
static int* g_counters = nullptr;

static int ensure_ws() {
  if (g_ws) return EMU_OK;
  if (cudaMalloc((void**)&g_ws, (size_t)kWsTiles * kMaxParts * 128 * sizeof(float)) != cudaSuccess) return EMU_ERR_NOMEM;
  if (cudaMalloc((void**)&g_counters, (size_t)kWsTiles * sizeof(int)) != cudaSuccess) return EMU_ERR_NOMEM;
  if (cudaMemset(g_counters, 0, (size_t)kWsTiles * sizeof(int)) != cudaSuccess) return EMU_ERR_CUDA;
  return EMU_OK;
}
int gemv_init() {
  int rc = ensure_ws();
  if (rc) return rc;
  return gemv_tma_init();
}

template <int RT, bool KFULL>
static int launch_gemv(const GemvParams& p, int grid, size_t smem, cudaStream_t st) {
  static size_t cur_max = 0;
  if (smem > cur_max) {
    if (cudaFuncSetAttribute(gemv_kernel<RT, KFULL>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess)
      return EMU_ERR_CUDA;
    cur_max = smem;
  }
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = dim3((unsigned)grid);
  cfg.blockDim = dim3(kGemvThreads);
  cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = p.a.pdl ? 1 : 0;
  return cudaLaunchKernelEx(&cfg, gemv_kernel<RT, KFULL>, p) == cudaSuccess ? EMU_OK : EMU_ERR_CUDA;
}

// dispatcher: TMA-fed kernel whenever the shape fits, register-ring kernel otherwise (EMU_GEMV=reg forces the latter)
int gemv_bf16(const GemvArgs& a, cudaStream_t st) {
  if (a.B < 1 || a.B > 8 || a.N < 1 || a.K < 32 || (a.K % 32) || (a.ldx % 8)) return EMU_ERR_INVALID;
  if ((a.mode == EPI_SWIGLU || a.mode == GEMV_ROPE_QKV) && (a.N % 16)) return EMU_ERR_INVALID;
  static int force_reg = -1;
  if (force_reg < 0) {
    const char* v = getenv("EMU_GEMV");
    force_reg = (v && v[0] == 'r') ? 1 : 0;
  }
  if (!force_reg) {
    const int rc = gemv_tma_bf16(a, st);
    if (rc != EMU_ERR_UNSUPPORTED) return rc;
  }
  if (a.ll_n > 0) return EMU_ERR_UNSUPPORTED;  // the fused exchange epilogue exists in the TMA kernel only
  return gemv_reg_bf16(a, st);
}

int gemv_reg_bf16(const GemvArgs& a, cudaStream_t st) {
  if (a.B < 1 || a.B > 8 || a.N < 1 || a.K < 32 || (a.K % 32) || (a.ldx % 8)) return EMU_ERR_INVALID;
  if ((a.mode == EPI_SWIGLU || a.mode == GEMV_ROPE_QKV) && (a.N % 16)) return EMU_ERR_INVALID;
  const int tiles = (a.N + 15) / 16;
  if (tiles > kWsTiles) return EMU_ERR_UNSUPPORTED;
  int rc = ensure_ws();  // NOTE: first use must happen outside stream capture (the engine calls gemv_init())
  if (rc) return rc;
  GemvParams p;
  p.a = a;
  p.ldxs = a.K + 32;  // row stride = 64 B (mod 128 B): conflict-free B-fragment reads
  p.ws = g_ws;
  p.counters = g_counters;
  const int KB = a.K / 32;
  p.cpt = (KB + kGemvWarps - 1) / kGemvWarps;
  const size_t xs_bytes = (size_t)a.B * p.ldxs * sizeof(bf16);
  p.red_off = (int)((xs_bytes + 15) & ~size_t(15));
  // tallest row group that still leaves >= 9 chunks per CTA: the RT=4 inner loop is ~4x leaner in instructions
  // per byte than RT=1, which outweighs up to ~10 % chunk-count imbalance (measured on the 6656x6656 o_proj)
  const long slots = 2L * kNumSMs;
  int rt = 1;
  if ((long)((tiles + 3) / 4) * p.cpt >= 9 * slots) rt = 4;
  else if ((long)((tiles + 1) / 2) * p.cpt >= 9 * slots) rt = 2;
  const size_t smem = p.red_off + (size_t)(kGemvWarps + 1) * rt * 128 * sizeof(float);
  if (smem > 220 * 1024) return EMU_ERR_UNSUPPORTED;
  const int occ = smem > 100 * 1024 ? 1 : 2;
  p.rt = rt;
  const int groups = (tiles + rt - 1) / rt;
  p.total = (long)groups * p.cpt;
  long grid = (long)kNumSMs * occ;
  if (grid > p.total) grid = p.total;
  // a row group may be shared by at most kMaxParts CTAs: keep every CTA's share >= cpt / (kMaxParts - 3)
  const long max_grid = (long)groups * (kMaxParts - 3);
  if (grid > max_grid) grid = max_grid;
  const bool kfull = (a.K % 256) == 0;
  if (kfull) {
    if (rt == 4) return launch_gemv<4, true>(p, (int)grid, smem, st);
    if (rt == 2) return launch_gemv<2, true>(p, (int)grid, smem, st);
    return launch_gemv<1, true>(p, (int)grid, smem, st);
  }
  if (rt == 4) return launch_gemv<4, false>(p, (int)grid, smem, st);
  if (rt == 2) return launch_gemv<2, false>(p, (int)grid, smem, st);
  return launch_gemv<1, false>(p, (int)grid, smem, st);
}

}  // namespace emu
