// emu_b200 — wgmma skinny GEMM for the wide decode step:  C[B,N] = epilogue( X[B,K] · W[N,K]^T ),  B <= 32.
//
// The decode step of more than 8 cache rows (BASELINE config 4: 4 prompts x 5 beams = 20 rows; reference call site
// Emu2/emu/emu.py:213-229 -> HF beam search) streams every weight once per token: HBM-bound, so what matters is how many
// weight bytes each SM keeps in flight.  gemm_tc.cu treats the activations as the 128-row MMA operand: at 20 rows most of
// every pipeline stage is zero padding.  Here the operands are swapped:
//   A operand (2 x M = 64) : a tile of 128 WEIGHT rows x 64 k      (16 KB per stage)
//   B operand (N = 32)     : the activations, 32 rows (zero-filled past B) x 64 k   (4 KB per stage)
//   accumulators           : [128 weight rows] x [32 batch columns] fp32 in the registers of one warpgroup
// -> 10 stages x 16 KB = 160 KB of weights in flight per SM.  Work units are (weight-row tile, K split): projections with
// few tiles are split along K so that every SM streams; the partial sums go through an fp32 workspace and the CTA that
// arrives last at a tile adds them in split order (deterministic) and runs the epilogue.
//   warp 4     : TMA producer (weight tiles are requested before griddepcontrol.wait — they do not depend on the predecessor)
//   warps 0..3 : wgmma m64n32k16 (two per 16-deep k step) and the epilogue: plain / +residual / SwiGLU (gate and up rows
//                interleaved: one shuffle), bf16 or fp32 output.
#include "common.cuh"
#include "ops.h"
#include "wgmma.cuh"

namespace emu {

int make_tmap_2d(CUtensorMap* out, const void* base, long rows, long cols, long ld, int box_rows);  // gemm_tc.cu

namespace {

constexpr int SKM = 128;  // weight rows per tile
constexpr int SKN = 32;   // activation rows (MMA N)
constexpr int SKK = 64;   // k per stage: 64 bf16 = one 128-byte swizzle row
constexpr int kSkStageBytes = (SKM + SKN) * SKK * 2;  // 20480
constexpr int kSkStages = 10;
constexpr int kSkThreads = 160;  // warps 0..3 = the consumer warpgroup, warp 4 = TMA producer
constexpr int kSkSmem = kSkStages * kSkStageBytes + 1024 /*align*/ + 256 /*barriers*/;

struct SkinnyParams {
  int B, N, K;
  void* C;
  int ldc;
  int out_fp32;
  const bf16* residual;
  int ldr;
  int mode;  // EPI_NONE / EPI_SWIGLU
  int tiles, splits, kb_per_split, num_kb;
  float* ws;      // [tiles * splits][32][128] fp32 partial sums (splits > 1)
  int* counters;  // [tiles], zero between launches (self-resetting)
  int pdl;
};

__device__ __forceinline__ void sk_named_bar(int id, int n) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(n) : "memory"); }

__global__ void __launch_bounds__(kSkThreads, 1)
gemm_skinny_kernel(const __grid_constant__ CUtensorMap tmW, const __grid_constant__ CUtensorMap tmX, const SkinnyParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + kSkStages * kSkStageBytes);
  uint64_t* empty_bar = full_bar + kSkStages;
  __shared__ int s_last;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int units = p.tiles * p.splits;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmW);
    tma_prefetch_desc(&tmX);
  }
  if (threadIdx.x < kSkStages) {
    mbar_init(&full_bar[threadIdx.x], 1);
    mbar_init(&empty_bar[threadIdx.x], 4);  // lane 0 of every consumer warp
    mbar_fence_init();
  }
  if (p.pdl) pdl_launch_dependents();
  __syncthreads();

  if (warp == 4) {
    // ===================== TMA producer =====================
    if (lane == 0) {
      int stage = 0;
      uint32_t phase = 0;
      int pre = 0;  // stages of the first unit whose weight tiles were requested before the dependency resolved
      if (p.pdl) {
        if ((int)blockIdx.x < units) {
          const int tile = blockIdx.x / p.splits, s = blockIdx.x % p.splits;
          const int kb0 = s * p.kb_per_split, kb1 = min(p.num_kb, kb0 + p.kb_per_split);
          pre = min(kSkStages, kb1 - kb0);
          for (int i = 0; i < pre; ++i) {
            mbar_expect_tx(&full_bar[i], kSkStageBytes);
            tma_load_2d(smem + i * kSkStageBytes, &tmW, &full_bar[i], (kb0 + i) * SKK, tile * SKM);
          }
          pdl_wait();  // the activations are the predecessor's output
          for (int i = 0; i < pre; ++i)
            tma_load_2d(smem + i * kSkStageBytes + SKM * SKK * 2, &tmX, &full_bar[i], (kb0 + i) * SKK, 0);
        } else {
          pdl_wait();
        }
      }
      bool first = true;
      for (int u = blockIdx.x; u < units; u += gridDim.x) {
        const int tile = u / p.splits, s = u % p.splits;
        const int kb0 = s * p.kb_per_split, kb1 = min(p.num_kb, kb0 + p.kb_per_split);
        for (int kb = kb0; kb < kb1; ++kb) {
          if (!(first && kb - kb0 < pre)) {
            mbar_wait(&empty_bar[stage], phase ^ 1);
            uint8_t* sa = smem + stage * kSkStageBytes;
            mbar_expect_tx(&full_bar[stage], kSkStageBytes);
            tma_load_2d(sa, &tmW, &full_bar[stage], kb * SKK, tile * SKM);
            tma_load_2d(sa + SKM * SKK * 2, &tmX, &full_bar[stage], kb * SKK, 0);
          }
          if (++stage == kSkStages) { stage = 0; phase ^= 1; }
        }
        first = false;
      }
    }
  } else {
    // ===================== consumer warpgroup: wgmma + epilogue =====================
    // v[16 m + 4 j + 2 h + e] = weight row 64 m + 16 warp + lane / 4 + 8 h of the tile, batch row 8 j + 2 (lane % 4) + e
    if (p.pdl) pdl_wait();  // residual is a predecessor output and C may alias a buffer it still reads
    const int B = p.B;
    int stage = 0;
    uint32_t phase = 0;
    for (int u = blockIdx.x; u < units; u += gridDim.x) {
      const int tile = u / p.splits, s = u % p.splits;
      const int kb0 = s * p.kb_per_split, kb1 = min(p.num_kb, kb0 + p.kb_per_split);
      float v[32];
      int prev = -1;
      for (int kb = kb0; kb < kb1; ++kb) {
        mbar_wait(&full_bar[stage], phase);
        const uint32_t sa = smem_u32(smem + stage * kSkStageBytes);
        const uint64_t da0 = wgmma_desc_sw128(sa), da1 = wgmma_desc_sw128(sa + 64 * SKK * 2);
        const uint64_t db = wgmma_desc_sw128(sa + SKM * SKK * 2);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < SKK / 16; ++k) {
          const int acc = (kb != kb0 || k != 0) ? 1 : 0;
          WgmmaSS<SKN>::run(v, da0 + 2 * k, db + 2 * k, acc);
          WgmmaSS<SKN>::run(v + 16, da1 + 2 * k, db + 2 * k, acc);
        }
        wgmma_commit();
        wgmma_wait<1>();
        if (prev >= 0) {
          __syncwarp();
          if (lane == 0) mbar_arrive(&empty_bar[prev]);
        }
        prev = stage;
        if (++stage == kSkStages) { stage = 0; phase ^= 1; }
      }
      wgmma_wait<0>();
      __syncwarp();
      if (lane == 0) mbar_arrive(&empty_bar[prev]);
      const int rbase = 16 * warp + (lane >> 2), bbase = 2 * (lane & 3);
      bool fin = true;
      if (p.splits > 1) {
        float* wt = p.ws + ((long)(tile * p.splits + s) * 32) * SKM;
#pragma unroll
        for (int i = 0; i < 32; ++i) {
          const int r = 64 * (i >> 4) + rbase + 8 * ((i >> 1) & 1), b = 8 * ((i >> 2) & 3) + bbase + (i & 1);
          if (b < B) wt[b * SKM + r] = v[i];
        }
        __threadfence();
        sk_named_bar(1, 128);
        if (threadIdx.x == 0) {
          const int prev_cnt = atomicAdd(&p.counters[tile], 1);
          s_last = prev_cnt == p.splits - 1;
          if (prev_cnt == p.splits - 1) p.counters[tile] = 0;  // self-reset for the next launch / graph replay
        }
        sk_named_bar(1, 128);
        fin = s_last != 0;
        if (fin) {
          __threadfence();
          const float* base = p.ws + ((long)tile * p.splits * 32) * SKM;
#pragma unroll
          for (int i = 0; i < 32; ++i) v[i] = 0.f;
          for (int s2 = 0; s2 < p.splits; ++s2) {  // split order: deterministic.  All values of one split are loaded before
            const float* src = base + (long)s2 * 32 * SKM;  // any is added: one L2 round trip per split, not per value
            float t[32];
#pragma unroll
            for (int i = 0; i < 32; ++i) {
              const int r = 64 * (i >> 4) + rbase + 8 * ((i >> 1) & 1), b = 8 * ((i >> 2) & 3) + bbase + (i & 1);
              t[i] = b < B ? __ldcg(src + b * SKM + r) : 0.f;
            }
#pragma unroll
            for (int i = 0; i < 32; ++i) v[i] += t[i];
          }
        }
        sk_named_bar(1, 128);  // s_last is rewritten by the next unit
      }
      if (!fin) continue;
      if (p.mode == EPI_SWIGLU) {
        // rows 2j / 2j+1 of W are gate_j / up_j (lanes l and l ^ 4): silu(gate) * up with HF's bf16 rounding points
        bf16* out = reinterpret_cast<bf16*>(p.C);
#pragma unroll
        for (int i = 0; i < 32; ++i) {
          const float other = __shfl_xor_sync(0xffffffffu, v[i], 4);
          const long n = (long)tile * SKM + 64 * (i >> 4) + rbase + 8 * ((i >> 1) & 1);
          const int b = 8 * ((i >> 2) & 3) + bbase + (i & 1);
          if (!((lane >> 2) & 1) && n < p.N && b < B) {
            const float gate = round_bf16(v[i]), up = round_bf16(other);
            out[(long)b * p.ldc + (n >> 1)] = __float2bfloat16_rn(round_bf16(silu(gate)) * up);
          }
        }
      } else {
        float rs[32];
        if (p.residual != nullptr) {  // all residual values in flight before the first is consumed
#pragma unroll
          for (int i = 0; i < 32; ++i) {
            const long n = (long)tile * SKM + 64 * (i >> 4) + rbase + 8 * ((i >> 1) & 1);
            const int b = 8 * ((i >> 2) & 3) + bbase + (i & 1);
            rs[i] = (b < B && n < p.N)
                        ? __uint_as_float((uint32_t)__ldcg(reinterpret_cast<const unsigned short*>(p.residual) + (long)b * p.ldr + n) << 16)
                        : 0.f;
          }
#pragma unroll
          for (int i = 0; i < 32; ++i) v[i] = round_bf16(v[i]) + rs[i];
        }
#pragma unroll
        for (int i = 0; i < 32; ++i) {
          const long n = (long)tile * SKM + 64 * (i >> 4) + rbase + 8 * ((i >> 1) & 1);
          const int b = 8 * ((i >> 2) & 3) + bbase + (i & 1);
          if (b < B && n < p.N) {
            if (p.out_fp32) reinterpret_cast<float*>(p.C)[(long)b * p.ldc + n] = v[i];
            else reinterpret_cast<bf16*>(p.C)[(long)b * p.ldc + n] = __float2bfloat16_rn(v[i]);
          }
        }
      }
    }
  }
}

}  // namespace

int gemm_skinny_init() {  // the engine calls this at create: the first real launch may sit inside a stream capture
  static bool attr_set = false;
  if (!attr_set) {
    if (cudaFuncSetAttribute(gemm_skinny_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kSkSmem) != cudaSuccess)
      return EMU_ERR_CUDA;
    attr_set = true;
  }
  return EMU_OK;
}

size_t gemm_skinny_workspace_bytes() { return (size_t)kSkinnyMaxUnits * 32 * SKM * sizeof(float); }

int gemm_skinny_bf16(const bf16* X, int ldx, const bf16* W, int ldw, int B, int N, int K, const GemmEpilogue& e, float* ws,
                     int* counters, cudaStream_t st) {
  if (B < 1 || B > SKN || N < 1 || K < 1) return EMU_ERR_UNSUPPORTED;
  if ((ldx % 8) || (ldw % 8) || (K % 8) || (reinterpret_cast<uintptr_t>(X) & 15) || (reinterpret_cast<uintptr_t>(W) & 15))
    return EMU_ERR_UNSUPPORTED;
  if (e.bias || e.bias2 || (e.mode != EPI_NONE && e.mode != EPI_SWIGLU)) return EMU_ERR_UNSUPPORTED;
  if (e.mode == EPI_SWIGLU && (e.residual || e.out_fp32 || (N & 1))) return EMU_ERR_UNSUPPORTED;
  SkinnyParams p;
  p.B = B; p.N = N; p.K = K;
  p.C = e.C; p.ldc = e.ldc; p.out_fp32 = e.out_fp32;
  p.residual = e.residual; p.ldr = e.ldr; p.mode = e.mode;
  p.tiles = (N + SKM - 1) / SKM;
  p.num_kb = (K + SKK - 1) / SKK;
  p.ws = ws; p.counters = counters;
  p.pdl = g_pdl_chain;
  // K splits: every SM should stream.  cost(S) = waves x (k-blocks per unit x ~420 cycles [10 stages in flight against the
  // loaded HBM latency] + fill / epilogue / partial-sum round trip)
  int best_s = 1;
  double best_cost = 1e30;
  const int max_s = (ws && counters) ? 16 : 1;
  // every weight byte crosses HBM once: no split can beat tiles x k-blocks x 16 KB at ~1800 B/clk
  const double hbm_floor = (double)p.tiles * p.num_kb * (SKM * SKK * 2) / 1800.0;
  for (int S = 1; S <= max_s; ++S) {
    const int kbs = (p.num_kb + S - 1) / S;
    if (S > 1 && (kbs < 4 || (long)p.tiles * S > kSkinnyMaxUnits || p.tiles > kSkinnyMaxTiles)) break;
    if ((S - 1) * kbs >= p.num_kb) continue;  // an empty last split
    const long units = (long)p.tiles * S;
    const long per_sm = (units + kNumSMs - 1) / kNumSMs;  // units the busiest SM works through
    double cost = (double)per_sm * ((double)kbs * 420.0 + 3000.0);
    if (cost < hbm_floor) cost = hbm_floor;
    if (S > 1) cost += 3000.0 + 700.0 * S;  // partial sums out, counter round trip, S loads back
    if (cost < best_cost - 1e-9) {
      best_cost = cost;
      best_s = S;
    }
  }
  p.splits = best_s;
  p.kb_per_split = (p.num_kb + best_s - 1) / best_s;
  CUtensorMap tmW, tmX;
  if (make_tmap_2d(&tmW, W, N, K, ldw, SKM) != EMU_OK) return EMU_ERR_UNSUPPORTED;
  if (make_tmap_2d(&tmX, X, B, K, ldx, SKN) != EMU_OK) return EMU_ERR_UNSUPPORTED;
  if (gemm_skinny_init() != EMU_OK) return EMU_ERR_CUDA;
  const long units = (long)p.tiles * p.splits;
  const unsigned grid = (unsigned)(units < kNumSMs ? units : kNumSMs);
  return launch_kernel(gemm_skinny_kernel, dim3(grid), dim3(kSkThreads), kSkSmem, st, p.pdl, tmW, tmX, p);
}

}  // namespace emu
