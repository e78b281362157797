// emu_b200 — TMA-fed variant of the decode-loop skinny GEMM (see gemv.cu for the problem statement and the
// stream-K decomposition; this file is the production path whenever the shape allows, gemv.cu is the fallback).
//
// Why a second kernel: gemv.cu keeps its bytes-in-flight in registers (16 x 16 B per lane).  That needs two 256-thread
// CTAs per SM to cover HBM latency and fills the register file.  Here the bytes in flight live in shared memory instead:
//   * one producer thread issues cp.async.bulk.tensor (TMA) loads of [32 rows x 64 cols] 128B-swizzled tiles into an
//     8-stage x 16 KB ring signalled by mbarriers — 128 KB in flight per SM with zero registers and zero address math
//     (a deep prefetch rather than a shallower ring that would let the PDL successor co-reside);
//   * 8 consumer warps pull A fragments with ldmatrix (conflict-free through the swizzle) and run mma.sync with the
//     staged x rows as the 8-wide N operand, then release the stage;
//   * ONE persistent CTA per SM (grid = kNumSMs), stream-K over (row group, k chunk) units, last-arriver fix-up in fixed
//     order; with PDL the producer starts streaming weights before griddepcontrol.wait resolves.
// x (batch <= 8 rows) is staged in shared memory once per CTA; when batch x K does not fit next to the ring (5 beams x
// 17920) it is staged in K segments that are re-staged as the chunk stream crosses them (GemvTmaParams::xsc).
// Ragged N and K tails cost nothing (TMA zero-fills out-of-bounds rows/columns).
#include <stdio.h>

#include "gemv_tma.cuh"

namespace emu {

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
  const int xsc = (p.xsc > 0 && p.xsc < p.cpt) ? p.xsc : p.cpt;
  uint32_t xphase = 0;
  if (p.xbulk) tma_stage_x_bulk(p, xs, s_ss, s_rstd, (int)(c0 % p.cpt) / xsc, &pre, &s_xbar, xphase);
  else tma_stage_x(p, xs, s_ss, s_rstd, (int)(c0 % p.cpt) / xsc, &pre);
  if (dbg && threadIdx.x == 0) {
    dbg[4] = clk();
    if (c0 < c1) mbar_wait(&full_bar[0], 0);  // (diagnostic only) when did the first chunk land?
    dbg[5] = clk();
  }
  tma_consume(&s_params, c0, c1, ring, full_bar, empty_bar, red, fin, xs, &s_last, stage, phase, s_rstd, &s_xbar, &xphase);
  if (dbg && threadIdx.x == 0) dbg[6] = clk();
  if (p.a.ll_n > 0 && p.a.ll_h != nullptr && (int)blockIdx.x < p.a.ll_red) gemv_tail_reduce(p.a);
  if (dbg && threadIdx.x == 0) dbg[7] = clk();
}

static float* g_tws = nullptr;
static int* g_tcounters = nullptr;

int gemv_tma_init() {
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

// returns EMU_ERR_UNSUPPORTED when the shape does not fit this kernel (caller falls back to gemv.cu)
int gemv_tma_bf16(const GemvArgs& a, cudaStream_t st) {
  if (a.K % 8 || (reinterpret_cast<uintptr_t>(a.W) & 15)) return EMU_ERR_UNSUPPORTED;
  const int groups = (a.N + kTRows - 1) / kTRows;
  if (groups > kTWsGroups) return EMU_ERR_UNSUPPORTED;
  if (!g_tws) {  // first use must happen outside stream capture (the engine calls gemv_init() at create)
    int rc = gemv_tma_init();
    if (rc) return rc;
  }
  GemvTmaParams p;
  p.a = a;
  p.kpad = (a.K + kTCols - 1) / kTCols * kTCols;
  p.ldxs = p.kpad + 8;  // row stride = 16 B (mod 128 B): the 8 batch rows hit distinct bank groups
  p.cpt = p.kpad / kTCols;
  p.xsc = 0;
  {
    // batch x K too large to keep all of x in shared memory next to a deep ring (5 beams x 17920 = 179 KB): stage x in K
    // segments of <= 88 KB instead, re-staged as the chunk stream crosses them
    const size_t budget = 88 * 1024;
    if ((size_t)a.B * p.ldxs * 2 > budget) {
      int xsc = (int)((budget / ((size_t)a.B * 2) - 8) / kTCols);
      if (xsc < 1) return EMU_ERR_UNSUPPORTED;
      p.xsc = xsc;
      p.ldxs = xsc * kTCols + 8;
    }
  }
  {
    static int env_bulk = -1;
    if (env_bulk < 0) {
      const char* v = getenv("EMU_GEMV_XBULK");
      env_bulk = v ? atoi(v) : 1;
    }
    // bulk row copies need 16-byte aligned rows; the in-place norm needs the whole row in shared memory
    p.xbulk = env_bulk && (a.ldx % 8 == 0) && !(reinterpret_cast<uintptr_t>(a.x) & 15) && (a.norm_w == nullptr || p.xsc == 0);
  }
  p.total = (long)groups * p.cpt;
  p.ws = g_tws;
  p.counters = g_tcounters;
  const size_t xs_bytes = (size_t)a.B * p.ldxs * 2;
  // the ring buffers are carved for kTStages; a CTA with a wide x uses fewer so that this kernel (<= ~110 KB) and its
  // PDL successor still fit one SM together
  static int env_stages = -1;
  if (env_stages < 0) {
    const char* v = getenv("EMU_GEMV_STAGES");
    env_stages = v ? atoi(v) : 0;
  }
  // default 8 stages = 128 KB in flight per SM (EMU_GEMV_STAGES overrides it for A-B runs)
  p.nstages = env_stages > 0 ? env_stages : 8;
  if (p.nstages > kTStages) p.nstages = kTStages;
  size_t smem;
  for (;;) {  // shrink the ring until the CTA fits (wide x at batch > 1)
    smem = 1024 + (size_t)p.nstages * kTStageBytes + 2 * kTStages * 8 + (size_t)(kTW + 1) * kTRT * 128 * 4 + xs_bytes + 64;
    if (smem <= 200 * 1024 || p.nstages <= 3) break;
    --p.nstages;
  }
  if (smem > 200 * 1024) return EMU_ERR_UNSUPPORTED;
  long grid = kNumSMs;
  if (grid > p.total) grid = p.total;
  const long max_grid = (long)groups * (kTMaxParts - 3);
  if (grid > max_grid) grid = max_grid;
  p.geff = (int)grid;
  if (p.a.ll_n > 0 && p.a.ll_h) {
    if (p.a.ll_red < 1 || (a.ldy & 1)) return EMU_ERR_INVALID;
    if (p.a.ll_red > (int)grid) p.a.ll_red = (int)grid;
  }
  CUtensorMap tm;
  if (make_tmap_2d(&tm, a.W, a.N, a.K, a.K, kTRows) != EMU_OK) return EMU_ERR_UNSUPPORTED;
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = dim3((unsigned)grid);
  cfg.blockDim = dim3(kTThreads);
  cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = a.pdl ? 1 : 0;
  return cudaLaunchKernelEx(&cfg, gemv_tma_kernel, tm, p) == cudaSuccess ? EMU_OK : EMU_ERR_CUDA;
}

}  // namespace emu
