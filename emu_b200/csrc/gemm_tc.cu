// emu_b200 — wgmma GEMM:  C[M,N] = epilogue( A[M,K] · W[N,K]^T )
//
// The dense-contraction workhorse of the generate path: ViT QKV/proj/MLP (Emu2/emu/eva_vit.py:194-200,
// 105-114), LLaMA prefill q/k/v/o/gate/up/down (HF LlamaDecoderLayer, called from Emu2/emu/emu.py:133-138,
// 213-229), project_up/project_down (emu.py:53-55), UNet linears and — through the 4-D TMA "conv" A-loader —
// the UNet/VAE 3x3 convolutions (diffusers UNet2DConditionModel, called from Emu2/emu/diffusion.py:136-141).
//
// 128 x BN output tiles, persistent CTAs (one per SM), a TMA producer feeding a ring of 128B-swizzled stages and two
// consumer warpgroups that run wgmma (fp32 accumulators in registers) and the fused epilogue — bias / GELU / quick GELU / residual /
// SwiGLU / GEGLU.  bf16 outputs are STAGED: the tile is assembled in shared memory as 64B-swizzled [rows x 32 columns]
// slabs and leaves with TMA stores; a residual tile arrives the same way (TMA load issued before the tile's main loop
// ends).  fp32 outputs, unaligned or very wide (> 192 columns) tiles store straight from registers.
// A and W are both K-major, so neither operand needs a transpose anywhere in the model.
#include <cstdlib>
#include <cstring>
#include <type_traits>

#include "common.cuh"
#include "ops.h"
#include "wgmma.cuh"

namespace emu {

constexpr int BM = 128;
constexpr int BK = 64;  // 64 bf16 = 128 B = one swizzle row
constexpr int kGemmThreads = 384;  // producer warpgroup + two consumer warpgroups

__device__ __forceinline__ void tma_store_2d(const CUtensorMap* m, const void* smem, int c0, int c1) {
  asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];" ::"l"(m), "r"(smem_u32(smem)),
               "r"(c0), "r"(c1)
               : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
__device__ __forceinline__ void bulk_wait_read0() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }
__device__ __forceinline__ void bulk_wait0() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }
__device__ __forceinline__ void fence_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void named_bar(int id, int n) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(n) : "memory"); }
__device__ __forceinline__ void sts128(uint32_t saddr, uint4 v) {
  asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(saddr), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
}
__device__ __forceinline__ uint4 lds128(uint32_t saddr) {
  uint4 v;
  asm volatile("ld.shared.v4.b32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(saddr) : "memory");
  return v;
}

template <int BN>
struct GemmSmem {
  static_assert(BN % 32 == 0 && BN >= 64 && BN <= 256, "BN: multiple of 32 (epilogue slabs) within the wgmma N range");
  static constexpr int kStageBytes = (BM + BN) * BK * 2;
  // staging for the TMA-store epilogue: [slabs of 32 output columns][128 rows][64 B].  Tiles wider than 192 columns are
  // only staged by the pair epilogues (SwiGLU / GEGLU), which emit BN / 2 columns.
  static constexpr int kStagingBytes = BM * (BN <= 192 ? BN : BN / 2) * 2;
  static constexpr int kFit = (227 * 1024 - 1024 - 512 - kStagingBytes) / kStageBytes;
  static constexpr int kStages = kFit > 8 ? 8 : kFit;  // 8 / 7 / 6 / 5 / 4 / 4 / 4 for BN = 64 .. 256
  static constexpr int kBytes = kStages * kStageBytes + kStagingBytes + 1024 /*align slack*/ + 512 /*barriers*/;
  static_assert(kStages >= 3, "pipeline too shallow");
};

struct GemmParams {
  int M, N, K;
  // epilogue
  void* C;         // bf16 or fp32
  int ldc;         // elements
  const bf16* bias;      // [N] or null
  const bf16* residual;  // [M, ldr] or null (added AFTER rounding the linear output to bf16, like `x + lin(x)`)
  int ldr;
  const bf16* bias2;     // [M / bias2_rows, N] or null: per-row-group bias (ResnetBlock2D time embedding), added after
  int bias2_rows;        //   rounding like `conv(x) + temb[:, :, None, None]`
  int epi;         // EpiMode
  int out_fp32;
  // conv A-loader (mode 1): A is an NHWC tensor [NB, H, W, Cin]; M = NB*H*W output pixels (stride 1, pad 1),
  // K index = tap * Cin + c.  tile rows = th x tw spatial patch (th*tw == 128)
  int conv;        // 0 = plain 2-D A, 1 = 3x3 conv (pad 1), 2 = 3x3 conv stride 2 is NOT handled here
  int H, W, Cin, tw, th;
  int pdl;  // launched with programmatic dependent launch: griddepcontrol.wait before touching activations
  int staged;    // bf16 output through shared memory + TMA store (tmC)
  int res_smem;  // residual tile through TMA load into the staging buffer (tmR); else direct global loads
  // diagnostics (emu_debug_gemm_phases): when non-null, every CTA writes 8 x u64 = {globaltimer at entry, clock64 at entry,
  // after set-up, first TMA issued, first stage landed (MMA side), last MMA of the tile retired, epilogue started,
  // epilogue done} for its FIRST tile
  unsigned long long* dbg;
};
__device__ __forceinline__ unsigned long long clk64() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%clock64;" : "=l"(t));
  return t;
}
__device__ __forceinline__ unsigned long long gtimer() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}

// two consecutive bf16 at p (the second only if `two`) as floats; 4-byte load when aligned
__device__ __forceinline__ float2 ld_bf16x2(const bf16* p, bool two) {
  if (two && !(reinterpret_cast<uintptr_t>(p) & 3)) {
    const uint32_t v = *reinterpret_cast<const uint32_t*>(p);
    return make_float2(bf16_lo(v), bf16_hi(v));
  }
  return make_float2(__bfloat162float(p[0]), two ? __bfloat162float(p[1]) : 0.f);
}
__device__ __forceinline__ uint32_t lds32(uint32_t saddr) {
  uint32_t v;
  asm volatile("ld.shared.b32 %0, [%1];" : "=r"(v) : "r"(saddr) : "memory");
  return v;
}
__device__ __forceinline__ void sts32(uint32_t saddr, uint32_t v) { asm volatile("st.shared.b32 [%0], %1;" ::"r"(saddr), "r"(v) : "memory"); }
__device__ __forceinline__ void sts16(uint32_t saddr, uint16_t v) { asm volatile("st.shared.b16 [%0], %1;" ::"r"(saddr), "h"(v) : "memory"); }
// byte offset of (row, column c < 32) inside a 64B-swizzled [rows][32 bf16] slab (the TMA SWIZZLE_64B pattern)
__device__ __forceinline__ uint32_t slab_off(int row, int c) {
  return (uint32_t)row * 64u + ((((uint32_t)c >> 3) ^ (((uint32_t)row >> 1) & 3u)) << 4) + ((uint32_t)c & 7u) * 2u;
}

// Warp roles (384 threads = 3 warpgroups, one CTA per SM, persistent over output tiles):
//   warpgroup 0 : TMA producer (one thread) — 128x64 (A) and BNx64 (W) bf16 tiles into a kStages-deep ring of
//                 128B-swizzled shared-memory stages, completion on mbarriers; the other warps give their registers away
//   warpgroups 1/2 : consumers of tile rows 0..63 / 64..127 — wgmma m64nBNk16 from shared memory into fp32 registers,
//                 then the fused epilogue of their 64 rows.
// CL = thread-block cluster size along M (1 or 2).  With CL == 2 the two CTAs of a cluster work on vertically adjacent
// output tiles (same weight columns): each loads HALF of the W tile and TMA-multicasts it into both CTAs' shared memory,
// so W crosses the L2->SM fabric once per pair; a stage is released in both CTAs once both have consumed it.
// CLF = CL, or CL | kQuickGeluKernel for the instantiations with the quick-GELU epilogue (CLIP MLP): that epilogue is a
// compile-time choice, so the kernels every other model runs carry no trace of it.
constexpr int kQuickGeluKernel = 16;
template <int BN, int CLF>
__global__ void __launch_bounds__(kGemmThreads, 1)
gemm_tc_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
               const __grid_constant__ CUtensorMap tmC, const __grid_constant__ CUtensorMap tmR, const GemmParams p) {
  constexpr int CL = CLF & (kQuickGeluKernel - 1);
  constexpr bool QG = (CLF & kQuickGeluKernel) != 0;
  constexpr int kStages = GemmSmem<BN>::kStages;
  constexpr int kStageBytes = GemmSmem<BN>::kStageBytes;

  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* staging = smem + kStages * kStageBytes;  // 1024-aligned: kStageBytes is a multiple of 4096
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(staging + GemmSmem<BN>::kStagingBytes);
  uint64_t* empty_bar = full_bar + kStages;
  uint64_t* res_full = empty_bar + kStages;  // [2] residual slabs of consumer 0 / 1 have landed

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;

  const int tiles_m = (p.M + BM - 1) / BM;
  const int tiles_n = (p.N + BN - 1) / BN;
  // work units: one tile (CL == 1) or one vertical tile pair (CL == 2; a ragged last pair computes a dummy tile whose
  // loads are out of bounds = zeros and whose rows fail the epilogue's row check, keeping the pair in lock step)
  const int units_m = (tiles_m + CL - 1) / CL;
  const int num_tiles = units_m * tiles_n;
  const int crank = CL > 1 ? (int)cluster_ctarank() : 0;
  const int unit0 = blockIdx.x / CL, unit_step = gridDim.x / CL;
  const int kblocks_per_tap = p.conv ? (p.Cin + BK - 1) / BK : (p.K + BK - 1) / BK;
  const int num_kb = p.conv ? 9 * kblocks_per_tap : kblocks_per_tap;

  unsigned long long* dbg = p.dbg ? p.dbg + (size_t)blockIdx.x * 8 : nullptr;
  if (dbg && threadIdx.x == 0) { dbg[0] = gtimer(); dbg[1] = clk64(); }
  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
    if (p.staged) tma_prefetch_desc(&tmC);
    if (p.res_smem) tma_prefetch_desc(&tmR);
  }
  if (threadIdx.x < kStages) {
    mbar_init(&full_bar[threadIdx.x], 1);
    mbar_init(&empty_bar[threadIdx.x], 8 * CL);  // lane 0 of every consumer warp, in every CTA that reads the stage
    mbar_fence_init();
  } else if (threadIdx.x >= 32 && threadIdx.x < 34) {
    mbar_init(&res_full[threadIdx.x - 32], 1);
    mbar_fence_init();
  }
  if (p.pdl) pdl_launch_dependents();  // the next kernel of the chain may start its own prologue now
  if (CL > 1) cluster_sync_all();  // the peer's barriers must be initialised before anything is multicast at them
  else __syncthreads();
  if (dbg && threadIdx.x == 0) dbg[2] = clk64();

  if (warp < 4) {
    // ===================== TMA producer =====================
    asm volatile("setmaxnreg.dec.sync.aligned.u32 40;");
    if (warp == 0 && lane == 0) {
      if (p.pdl) pdl_wait();  // activations (A) come from the predecessor; everything above overlapped its tail
      if (dbg) dbg[3] = clk64();
      int stage = 0;
      uint32_t phase = 0;
      for (int tile = unit0; tile < num_tiles; tile += unit_step) {
        const int tm = (tile % units_m) * CL + crank, tn = tile / units_m;
        int img = 0, h0 = 0, w0 = 0;
        if (p.conv) {
          const int tiles_w = p.W / p.tw, tiles_h = p.H / p.th;
          w0 = (tm % tiles_w) * p.tw;
          h0 = ((tm / tiles_w) % tiles_h) * p.th;
          img = tm / (tiles_w * tiles_h);
        }
        for (int kb = 0; kb < num_kb; ++kb) {
          mbar_wait(&empty_bar[stage], phase ^ 1);
          uint8_t* sa = smem + stage * kStageBytes;
          uint8_t* sb = sa + BM * BK * 2;
          mbar_expect_tx(&full_bar[stage], kStageBytes);
          int kcol;
          if (p.conv) {
            const int tap = kb / kblocks_per_tap, cb = kb % kblocks_per_tap;
            const int r = tap / 3, s = tap % 3;
            tma_load_4d(sa, &tmA, &full_bar[stage], cb * BK, w0 + s - 1, h0 + r - 1, img);
            kcol = tap * p.Cin + cb * BK;
          } else {
            tma_load_2d(sa, &tmA, &full_bar[stage], kb * BK, tm * BM);
            kcol = kb * BK;
          }
          if (CL > 1) {
            // my half of the W tile, written to the same offset in both CTAs; the peer supplies the other half
            constexpr int kHalf = BN / CL;
            tma_load_2d_mc(sb + crank * kHalf * BK * 2, &tmB, &full_bar[stage], kcol, tn * BN + crank * kHalf,
                           (uint16_t)((1u << CL) - 1));
          } else {
            tma_load_2d(sb, &tmB, &full_bar[stage], kcol, tn * BN);
          }
          if (++stage == kStages) { stage = 0; phase ^= 1; }
        }
      }
    }
  } else {
    // ===================== consumers: wgmma main loop + epilogue of 64 rows =====================
    asm volatile("setmaxnreg.inc.sync.aligned.u32 232;");
    const int wg = (warp >> 2) - 1;                   // 0 / 1: tile rows 64 wg ..
    const int rl = 64 * wg + 16 * (warp & 3) + (lane >> 2);  // tile rows rl and rl + 8 of this thread
    const int cq = 2 * (lane & 3);                    // column pair offset inside every 8-column group
    const bool pair = (p.epi == EPI_SWIGLU || p.epi == EPI_GEGLU);
    const int n_out = pair ? (p.N >> 1) : p.N;        // output columns of the whole matrix
    const int bn_out = pair ? BN / 2 : BN;            // ... of one tile
    const int n_units = bn_out / 32;
    const uint32_t stg = smem_u32(staging);
    const bool issuer = (threadIdx.x & 127) == 0;
    const int bar_id = 1 + wg;
    if (p.pdl) pdl_wait();  // residual / bias2 are predecessor outputs and C may alias a buffer it still reads
    auto tile_row0 = [&](int tm) -> long {
      if (!p.conv) return (long)tm * BM;
      const int tiles_w = p.W / p.tw, tiles_h = p.H / p.th;
      const int w0 = (tm % tiles_w) * p.tw, h0 = ((tm / tiles_w) % tiles_h) * p.th, img = tm / (tiles_w * tiles_h);
      return ((long)img * p.H + h0) * p.W + w0;  // a tile is th full-width rows or one 128-pixel run: 128 consecutive rows
    };
    auto load_residual = [&](int tile) {  // issuer only: this consumer's 64 residual rows of every slab of `tile` -> staging
      const int tm = (tile % units_m) * CL + crank, tn = tile / units_m;
      int cnt = 0;
      for (int u = 0; u < n_units; ++u)
        if (tn * bn_out + u * 32 < n_out) ++cnt;
      if (tm >= tiles_m) cnt = 0;
      mbar_expect_tx(&res_full[wg], (uint32_t)cnt * 4096u);  // arrive + expect: with 0 bytes the phase completes at once
      if (cnt == 0) return;
      const int row0 = (int)tile_row0(tm) + 64 * wg;
      for (int u = 0; u < n_units; ++u)
        if (tn * bn_out + u * 32 < n_out)
          tma_load_2d(staging + u * 8192 + wg * 4096, &tmR, &res_full[wg], tn * bn_out + u * 32, row0);
    };
    if (p.staged && p.res_smem && issuer && unit0 < num_tiles) load_residual(unit0);
    uint32_t res_phase = 0;
    int stage = 0;
    uint32_t phase = 0;
    float d[BN / 2];
    for (int tile = unit0; tile < num_tiles; tile += unit_step) {
      const int tm = (tile % units_m) * CL + crank, tn = tile / units_m;
      // ---------- main loop: one k block = 4 x wgmma k16; the stage of k block kb - 1 is released once kb's are issued ----------
      int prev = -1;
      for (int kb = 0; kb < num_kb; ++kb) {
        mbar_wait(&full_bar[stage], phase);
        if (dbg && kb == 0 && tile == unit0 && threadIdx.x == 128) dbg[4] = clk64();
        const uint32_t sa = smem_u32(smem + stage * kStageBytes) + wg * (64 * BK * 2);
        const uint32_t sb = smem_u32(smem + stage * kStageBytes) + BM * BK * 2;
        const uint64_t da = wgmma_desc_sw128(sa), db = wgmma_desc_sw128(sb);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < BK / 16; ++k)  // 16 elements (32 B) along K inside the 128 B swizzle row: +2 in the (addr>>4) field
          WgmmaSS<BN>::run(d, da + 2 * k, db + 2 * k, (kb | k) != 0);
        wgmma_commit();
        wgmma_wait<1>();
        if (prev >= 0) {
          __syncwarp();
          if (lane == 0) {
            if (CL > 1) {
              for (int c = 0; c < CL; ++c) mbar_arrive_cluster(&empty_bar[prev], (uint32_t)c);
            } else {
              mbar_arrive(&empty_bar[prev]);
            }
          }
        }
        prev = stage;
        if (++stage == kStages) { stage = 0; phase ^= 1; }
      }
      wgmma_wait<0>();
      __syncwarp();
      if (lane == 0) {
        if (CL > 1) {
          for (int c = 0; c < CL; ++c) mbar_arrive_cluster(&empty_bar[prev], (uint32_t)c);
        } else {
          mbar_arrive(&empty_bar[prev]);
        }
      }
      if (dbg && tile == unit0 && threadIdx.x == 128) dbg[5] = dbg[6] = clk64();

      // ---------- epilogue ----------
      const long row0 = tile_row0(tm);
      const bool tile_ok = tm < tiles_m;
      long rows[2];
      bool row_ok[2];
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int r = rl + 8 * h;
        if (p.conv && !p.staged) {
          const int tiles_w = p.W / p.tw, tiles_h = p.H / p.th;
          const int w0 = (tm % tiles_w) * p.tw, h0 = ((tm / tiles_w) % tiles_h) * p.th, img = tm / (tiles_w * tiles_h);
          rows[h] = ((long)img * p.H + h0 + r / p.tw) * p.W + w0 + r % p.tw;
        } else {
          rows[h] = row0 + r;
        }
        row_ok[h] = tile_ok && rows[h] < p.M;
      }
      if (p.staged && p.res_smem) mbar_wait(&res_full[wg], res_phase);
#pragma unroll
      for (int j = 0; j < BN / 8; ++j) {
        const int ct = 8 * j + cq;      // accumulator column inside the tile (even)
        const int col = tn * BN + ct;   // ... of the matrix
        if (col >= p.N) continue;
        const bool two = col + 1 < p.N;
        float2 b = make_float2(0.f, 0.f);
        if (p.bias != nullptr) b = ld_bf16x2(p.bias + col, two);
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          float f0 = d[4 * j + 2 * h] + b.x, f1 = d[4 * j + 2 * h + 1] + b.y;
          const int r = rl + 8 * h;
          if (p.bias2 != nullptr && row_ok[h]) {
            const float2 b2 = ld_bf16x2(p.bias2 + (rows[h] / p.bias2_rows) * p.N + col, two);
            round_bf16x2(f0, f1);
            f0 += b2.x;
            f1 += b2.y;
          }
          if (pair) {
            // interleaved (a_j, b_j) accumulator columns -> output column j; rounding points of the reference
            // (Linear -> bf16, activation -> bf16, product -> bf16).  SwiGLU: silu(gate) * up; GEGLU: hidden * gelu(gate)
            round_bf16x2(f0, f1);
            const float o = (p.epi == EPI_SWIGLU) ? round_bf16(silu(f0)) * f1 : f0 * round_bf16(gelu_erf_fast(f1));
            const int oct = ct >> 1;  // output column inside the tile
            if (p.staged) {
              sts16(stg + (uint32_t)(oct >> 5) * 8192u + slab_off(r, oct & 31), __bfloat16_as_ushort(__float2bfloat16_rn(o)));
            } else if (row_ok[h]) {
              reinterpret_cast<bf16*>(p.C)[rows[h] * p.ldc + (col >> 1)] = __float2bfloat16_rn(o);
            }
            continue;
          }
          if (QG) {
            // transformers QuickGELUActivation on the bf16 Linear output, x * sigmoid(1.702 * x), with the rounding points
            // of its bf16 eager run: Linear -> bf16, 1.702 * x -> bf16, sigmoid -> bf16, product -> bf16 (at the store)
            round_bf16x2(f0, f1);
            f0 *= round_bf16(sigmoid_f(round_bf16(1.702f * f0)));
            f1 *= round_bf16(sigmoid_f(round_bf16(1.702f * f1)));
          } else if (p.epi == EPI_GELU) {
            round_bf16x2(f0, f1);
            f0 = gelu_erf_fast(f0);
            f1 = gelu_erf_fast(f1);
          } else if (p.epi == EPI_RELU) {
            f0 = fmaxf(f0, 0.f);
            f1 = fmaxf(f1, 0.f);
          }
          if (p.staged) {
            const uint32_t a = stg + (uint32_t)(ct >> 5) * 8192u + slab_off(r, ct & 31);
            if (p.res_smem) {
              const uint32_t rv = lds32(a);
              round_bf16x2(f0, f1);
              f0 += bf16_lo(rv);
              f1 += bf16_hi(rv);
            } else if (p.residual != nullptr && row_ok[h]) {
              const float2 rv = ld_bf16x2(p.residual + rows[h] * p.ldr + col, two);
              round_bf16x2(f0, f1);
              f0 += rv.x;
              f1 += rv.y;
            }
            sts32(a, pack_bf16(f0, f1));
            continue;
          }
          if (!row_ok[h]) continue;
          if (p.residual != nullptr) {
            const float2 rv = ld_bf16x2(p.residual + rows[h] * p.ldr + col, two);
            round_bf16x2(f0, f1);
            f0 += rv.x;
            f1 += rv.y;
          }
          if (p.out_fp32) {
            float* dst = reinterpret_cast<float*>(p.C) + rows[h] * p.ldc + col;
            if (two && !(reinterpret_cast<uintptr_t>(dst) & 7)) *reinterpret_cast<float2*>(dst) = make_float2(f0, f1);
            else { dst[0] = f0; if (two) dst[1] = f1; }
          } else {
            bf16* dst = reinterpret_cast<bf16*>(p.C) + rows[h] * p.ldc + col;
            if (two && !(reinterpret_cast<uintptr_t>(dst) & 3)) *reinterpret_cast<uint32_t*>(dst) = pack_bf16(f0, f1);
            else { dst[0] = __float2bfloat16_rn(f0); if (two) dst[1] = __float2bfloat16_rn(f1); }
          }
        }
      }
      if (p.staged) {
        // this consumer's 64 rows of every slab leave with TMA stores (rows / columns past the matrix are clipped)
        fence_async_smem();  // generic-proxy slab writes -> visible to the TMA engine
        named_bar(bar_id, 128);
        if (issuer) {
          if (tile_ok) {
            for (int u = 0; u < n_units; ++u) {
              const int oc0 = tn * bn_out + u * 32;
              if (oc0 < n_out) tma_store_2d(&tmC, staging + u * 8192 + wg * 4096, oc0, (int)row0 + 64 * wg);
            }
          }
          bulk_commit();
          bulk_wait_read0();  // the slabs may be overwritten once the stores have READ them
          if (p.res_smem && tile + unit_step < num_tiles) load_residual(tile + unit_step);
        }
        named_bar(bar_id, 128);  // nobody of the group touches the slabs before the issuer got here
        res_phase ^= 1;
      }
      if (dbg && tile == unit0 && threadIdx.x == 128) dbg[7] = clk64();
    }
    if (p.staged && issuer) bulk_wait0();  // all stores complete (global writes performed) before the CTA retires
  }

  if (CL > 1) cluster_sync_all();  // nobody leaves while the peer can still multicast into / arrive on its shared memory
}

// ----------------------------------------------------------------------------------------------
// host side
// ----------------------------------------------------------------------------------------------
typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                    const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                    CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static PFN_encodeTiled get_encode() {
  static PFN_encodeTiled fn = nullptr;
  if (fn) return fn;
  void* ptr = nullptr;
  cudaDriverEntryPointQueryResult qres;
  if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &ptr, cudaEnableDefault, &qres) != cudaSuccess ||
      qres != cudaDriverEntryPointSuccess)
    return nullptr;
  fn = reinterpret_cast<PFN_encodeTiled>(ptr);
  return fn;
}

// 2-D K-major bf16 matrix [rows, cols] with row stride ld (elements); box = box_rows x 64 cols, 128B swizzle
int make_tmap_2d(CUtensorMap* out, const void* base, long rows, long cols, long ld, int box_rows) {
  PFN_encodeTiled enc = get_encode();
  if (!enc) return EMU_ERR_CUDA;
  cuuint64_t dims[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
  cuuint64_t strides[1] = {(cuuint64_t)ld * 2};
  cuuint32_t box[2] = {(cuuint32_t)BK, (cuuint32_t)box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = enc(out, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(base), dims, strides, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS ? EMU_OK : EMU_ERR_CUDA;
}

// bf16 [rows, cols] output / residual matrix for the staged epilogue: box = 64 rows (one consumer warpgroup) x 32 columns
// (64 B), 64B swizzle.
// TMA clips the rows / columns of a box that fall outside the matrix on a store and zero-fills them on a load.
int make_tmap_out(CUtensorMap* out, const void* base, long rows, long cols, long ld) {
  PFN_encodeTiled enc = get_encode();
  if (!enc) return EMU_ERR_CUDA;
  cuuint64_t dims[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
  cuuint64_t strides[1] = {(cuuint64_t)ld * 2};
  cuuint32_t box[2] = {32, 64};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = enc(out, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(base), dims, strides, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_64B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS ? EMU_OK : EMU_ERR_CUDA;
}

// 4-D NHWC bf16 activation [NB, H, W, C]; box = {64 ch, tw, th, 1}; out-of-bounds (the conv halo) reads as zero
int make_tmap_nhwc(CUtensorMap* out, const void* base, int NB, int H, int W, int C, int tw, int th) {
  PFN_encodeTiled enc = get_encode();
  if (!enc) return EMU_ERR_CUDA;
  cuuint64_t dims[4] = {(cuuint64_t)C, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)NB};
  cuuint64_t strides[3] = {(cuuint64_t)C * 2, (cuuint64_t)W * C * 2, (cuuint64_t)H * W * C * 2};
  cuuint32_t box[4] = {(cuuint32_t)BK, (cuuint32_t)tw, (cuuint32_t)th, 1};
  cuuint32_t estr[4] = {1, 1, 1, 1};
  CUresult r = enc(out, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, const_cast<void*>(base), dims, strides, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS ? EMU_OK : EMU_ERR_CUDA;
}

// strided [B, N, H, D] bf16 view (attention operands) as a 4-D map; box = {64 d, box_rows tokens, 1 head, 1 batch}.
// Dimensions are ordered by stride (head-before-token when heads are interleaved inside a token row, as in fused QKV
// outputs); *head_first tells the kernel which coordinate order to use.  Head-dim padding and rows past N read as zero.
int make_tmap_bnhd(CUtensorMap* out, const void* base, int D, long N, int H, int B, long ts, long hs, long bs, int box_rows,
                   int* head_first) {
  PFN_encodeTiled enc = get_encode();
  if (!enc) return EMU_ERR_CUDA;
  if ((ts % 8) || (hs % 8) || (bs % 8) || (reinterpret_cast<uintptr_t>(base) & 15)) return EMU_ERR_INVALID;
  const bool hf = hs < ts;
  *head_first = hf ? 1 : 0;
  cuuint64_t bstride = bs > 0 ? (cuuint64_t)bs * 2 : 16;
  cuuint64_t tstride = ts > 0 ? (cuuint64_t)ts * 2 : 16;
  cuuint64_t hstride = hs > 0 ? (cuuint64_t)hs * 2 : 16;
  cuuint64_t dims[4], strides[3];
  cuuint32_t box[4];
  dims[0] = (cuuint64_t)D;
  box[0] = 64;
  if (hf) {
    dims[1] = (cuuint64_t)H; dims[2] = (cuuint64_t)N; strides[0] = hstride; strides[1] = tstride;
    box[1] = 1; box[2] = (cuuint32_t)box_rows;
  } else {
    dims[1] = (cuuint64_t)N; dims[2] = (cuuint64_t)H; strides[0] = tstride; strides[1] = hstride;
    box[1] = (cuuint32_t)box_rows; box[2] = 1;
  }
  dims[3] = (cuuint64_t)B;
  strides[2] = bstride;
  box[3] = 1;
  cuuint32_t estr[4] = {1, 1, 1, 1};
  CUresult r = enc(out, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, const_cast<void*>(base), dims, strides, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS ? EMU_OK : EMU_ERR_CUDA;
}

template <int BN, int CL, bool QG = false>
static int launch_gemm_cl(const CUtensorMap& tmA, const CUtensorMap& tmB, const CUtensorMap& tmC, const CUtensorMap& tmR,
                          const GemmParams& p, cudaStream_t st) {
  static_assert(!QG || CL == 1, "the quick-GELU kernels are built without clusters");
  auto kern = gemm_tc_kernel<BN, QG ? (CL | kQuickGeluKernel) : CL>;
  static bool attr_set = false;
  static int max_ctas = kNumSMs;
  if (!attr_set) {
    if (cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, GemmSmem<BN>::kBytes) !=
        cudaSuccess)
      return EMU_ERR_CUDA;
    if (CL > 1) {
      // how many clusters can be resident at once (GPC boundaries may leave an SM without a partner)
      cudaLaunchConfig_t q{};
      q.gridDim = dim3(kNumSMs / CL * CL);
      q.blockDim = dim3(kGemmThreads);
      q.dynamicSmemBytes = GemmSmem<BN>::kBytes;
      cudaLaunchAttribute a[1];
      a[0].id = cudaLaunchAttributeClusterDimension;
      a[0].val.clusterDim.x = CL; a[0].val.clusterDim.y = 1; a[0].val.clusterDim.z = 1;
      q.attrs = a;
      q.numAttrs = 1;
      int n = 0;
      if (cudaOccupancyMaxActiveClusters(&n, gemm_tc_kernel<BN, CL>, &q) == cudaSuccess && n > 0) max_ctas = n * CL;
      else cudaGetLastError();
      if (max_ctas > kNumSMs) max_ctas = kNumSMs / CL * CL;
    }
    attr_set = true;
  }
  const int units = (((p.M + BM - 1) / BM + CL - 1) / CL) * ((p.N + BN - 1) / BN);
  int grid = units * CL < max_ctas ? units * CL : max_ctas;
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = dim3(grid);
  cfg.blockDim = dim3(kGemmThreads);
  cfg.dynamicSmemBytes = GemmSmem<BN>::kBytes;
  cfg.stream = st;
  cudaLaunchAttribute attr[2];
  int na = 0;
  if (CL > 1) {
    attr[na].id = cudaLaunchAttributeClusterDimension;
    attr[na].val.clusterDim.x = CL; attr[na].val.clusterDim.y = 1; attr[na].val.clusterDim.z = 1;
    ++na;
  }
  if (p.pdl) {
    attr[na].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[na].val.programmaticStreamSerializationAllowed = 1;
    ++na;
  }
  cfg.attrs = attr;
  cfg.numAttrs = na;
  return cudaLaunchKernelEx(&cfg, kern, tmA, tmB, tmC, tmR, p) == cudaSuccess ? EMU_OK : EMU_ERR_CUDA;
}

// Cluster mode (W tile TMA-multicast over a 2-CTA cluster): halves the W traffic into shared memory at the price of
// cluster start-up and lock step.  Default: convolutions only (K >= 5760 for most UNet convs).  EMU_GEMM_CLUSTER = 0
// (never), 1 (always), unset (convs); force bits: 1024 = off, 2048 = on (tests / A-B runs).
static bool use_cluster(int M, int force, bool is_conv) {
  static int env = -2;
  if (env == -2) {
    const char* v = getenv("EMU_GEMM_CLUSTER");
    env = v ? atoi(v) : -1;
  }
  if (force & 1024) return false;
  const int tiles_m = (M + BM - 1) / BM;
  if (force & 2048) return tiles_m >= 1;
  if (env == 0 || (env < 0 && !is_conv)) return false;
  return tiles_m >= 2 && (tiles_m % 2 == 0 || tiles_m >= 7);
}

// Can this problem use the staged (shared memory + TMA store) epilogue at tile width bn?
static bool can_stage(const GemmEpilogue& e, int N, int bn) {
  if (e.out_fp32 || e.C == nullptr) return false;
  const bool pair = e.mode == EPI_SWIGLU || e.mode == EPI_GEGLU;
  const int n_out = pair ? N / 2 : N;
  if ((reinterpret_cast<uintptr_t>(e.C) & 15) || (e.ldc % 8) || (n_out % 8)) return false;
  if (pair) return bn % 64 == 0;  // a 32-column output slab = 64 accumulator columns
  return bn <= 192;               // the staging buffer holds at most 192 columns
}
static bool env_no_stage() {
  static int v = -1;
  if (v < 0) {
    const char* s = getenv("EMU_GEMM_DIRECT");
    v = (s && atoi(s) == 1) ? 1 : 0;
  }
  return v == 1;
}

// Tile width: minimise the modelled time of one CTA's tile stream over the instantiated widths.  Per tile the main loop
// costs kblocks x max(tensor pipe: 4 x bn cycles per 128-row, 64-deep k block at H100's 1024 bf16 FMA / clk / SM, L2 ->
// shared-memory operand traffic: (128 + bn) x 128 B at ~64 B/cycle/SM); the epilogue runs after the main loop in the same
// warps and costs a few cycles per output column (more with activations or a residual).  Odd widths such as 160 exist
// because e.g. M=2048, N=1280 is 160 tiles at BN=128 (two waves on 132 SMs, the second 21 % full) but 128 tiles at BN=160
// (one wave).
static int pick_bn(int M, int N, int K, const GemmEpilogue& e) {
  static const int cand[] = {256, 224, 192, 160, 128, 96, 64};
  const long tm = (M + BM - 1) / BM;
  const long kb = (K + BK - 1) / BK;
  const bool act = e.mode == EPI_GELU || e.mode == EPI_SWIGLU || e.mode == EPI_GEGLU || e.mode == EPI_QUICK_GELU;
  int best = 128;
  double best_cost = 1e30;
  for (int bn : cand) {
    const long tiles = tm * ((N + bn - 1) / bn);
    const long waves = (tiles + kNumSMs - 1) / kNumSMs;
    const double a_rows = M < 128 ? (double)M : 128.0;  // rows past M are zero-filled by TMA, not fetched
    const double mma = 4.0 * bn, l2 = (a_rows + bn) * 128.0 / 64.0;
    double per_kb = mma > l2 ? mma : l2;
    if (tm == 1) {  // one row of tiles: every weight byte comes from HBM exactly once, shared by the busy SMs (~1800 B/clk)
      const double active = tiles < kNumSMs ? (double)tiles : (double)kNumSMs;
      const double hbm = bn * 128.0 * active / 1800.0;
      if (hbm > per_kb) per_kb = hbm;
    }
    const double ml = (double)kb * per_kb + 1500.0;  // + pipeline fill
    const bool staged = !env_no_stage() && can_stage(e, N, bn);
    double per_col = staged ? (act ? 20.0 : 8.0) : (act ? 40.0 : (e.residual ? 30.0 : 16.0));
    const double epi = per_col * bn + 400.0;
    const double cost = (double)waves * (ml + epi);
    if (cost < best_cost - 1e-9) {
      best_cost = cost;
      best = bn;
    }
  }
  return best;
}

template <typename F>
static int dispatch_bn(int bn, F&& f) {
  switch (bn) {
    case 256: return f(std::integral_constant<int, 256>());
    case 224: return f(std::integral_constant<int, 224>());
    case 192: return f(std::integral_constant<int, 192>());
    case 160: return f(std::integral_constant<int, 160>());
    case 128: return f(std::integral_constant<int, 128>());
    case 96: return f(std::integral_constant<int, 96>());
    case 64: return f(std::integral_constant<int, 64>());
  }
  return EMU_ERR_INVALID;
}

// decide the epilogue style of this launch and build the tensor maps it needs (dummies otherwise: the kernel never touches
// a map whose flag is off)
static int setup_staging(GemmParams& p, const GemmEpilogue& e, int M, int N, int bn, CUtensorMap* tmC, CUtensorMap* tmR) {
  memset(tmC, 0, sizeof(*tmC));
  memset(tmR, 0, sizeof(*tmR));
  p.staged = 0;
  p.res_smem = 0;
  const bool forced_direct = (e.force_bn & 4096) != 0;
  if (forced_direct || env_no_stage() || !can_stage(e, N, bn)) return EMU_OK;
  const bool pair = e.mode == EPI_SWIGLU || e.mode == EPI_GEGLU;
  const int n_out = pair ? N / 2 : N;
  if (make_tmap_out(tmC, e.C, M, n_out, e.ldc) != EMU_OK) return EMU_OK;  // odd geometry: keep the direct path
  p.staged = 1;
  if (e.residual != nullptr && !pair && (e.ldr % 8 == 0) && !(reinterpret_cast<uintptr_t>(e.residual) & 15) &&
      make_tmap_out(tmR, e.residual, M, n_out, e.ldr) == EMU_OK)
    p.res_smem = 1;
  return EMU_OK;
}

int gemm_bf16(const bf16* A, int lda, const bf16* W, int ldw, int M, int N, int K, const GemmEpilogue& e,
              cudaStream_t st) {
  if (M <= 0 || N <= 0 || K <= 0) return EMU_ERR_INVALID;
  if ((lda % 8) || (ldw % 8) || (reinterpret_cast<uintptr_t>(A) & 15) || (reinterpret_cast<uintptr_t>(W) & 15))
    return EMU_ERR_INVALID;
  const bool pair = e.mode == EPI_SWIGLU || e.mode == EPI_GEGLU;
  if (pair && (N & 1)) return EMU_ERR_INVALID;
  const bool qg = e.mode == EPI_QUICK_GELU;
  GemmParams p{};
  p.M = M; p.N = N; p.K = K;
  p.C = e.C; p.ldc = e.ldc; p.bias = e.bias; p.residual = e.residual; p.ldr = e.ldr;
  p.bias2 = e.bias2; p.bias2_rows = e.bias2_rows > 0 ? e.bias2_rows : 1;
  p.epi = e.mode; p.out_fp32 = e.out_fp32; p.conv = 0; p.pdl = g_pdl_chain; p.dbg = e.dbg;
  const int bn = (e.force_bn & 1023) ? (e.force_bn & 1023) : pick_bn(M, N, K, e);
  const bool cl = !qg && use_cluster(M, e.force_bn, false);
  CUtensorMap tmA, tmB, tmC, tmR;
  int rc = make_tmap_2d(&tmA, A, M, K, lda, BM);
  if (rc) return rc;
  rc = make_tmap_2d(&tmB, W, N, K, ldw, cl ? bn / 2 : bn);
  if (rc) return rc;
  rc = setup_staging(p, e, M, N, bn, &tmC, &tmR);
  if (rc) return rc;
  return dispatch_bn(bn, [&](auto w) {
    constexpr int kBN = decltype(w)::value;
    if (qg) return launch_gemm_cl<kBN, 1, true>(tmA, tmB, tmC, tmR, p, st);
    return cl ? launch_gemm_cl<kBN, 2>(tmA, tmB, tmC, tmR, p, st) : launch_gemm_cl<kBN, 1>(tmA, tmB, tmC, tmR, p, st);
  });
}

// 3x3 stride-1 pad-1 convolution on NHWC bf16 as an implicit GEMM. Wk is [Cout, 9*Cin] with k = (r*3+s)*Cin + c.
int conv3x3_bf16(const bf16* X, int NB, int H, int W, int Cin, const bf16* Wk, int Cout, const GemmEpilogue& e,
                 cudaStream_t st) {
  if (Cin % 8 || e.mode == EPI_QUICK_GELU) return EMU_ERR_INVALID;  // quick GELU: Linear layers only
  int tw = W >= 128 ? 128 : W;  // tile = th x tw pixels, th*tw = 128
  if (128 % tw) return EMU_ERR_UNSUPPORTED;
  int th = 128 / tw;
  if (H % th || W % tw) return EMU_ERR_UNSUPPORTED;
  GemmParams p{};
  p.M = NB * H * W; p.N = Cout; p.K = 9 * Cin;
  p.C = e.C; p.ldc = e.ldc; p.bias = e.bias; p.residual = e.residual; p.ldr = e.ldr;
  p.bias2 = e.bias2; p.bias2_rows = e.bias2_rows > 0 ? e.bias2_rows : 1;
  p.epi = e.mode; p.out_fp32 = e.out_fp32; p.pdl = g_pdl_chain; p.dbg = e.dbg;
  p.conv = 1; p.H = H; p.W = W; p.Cin = Cin; p.tw = tw; p.th = th;
  const int bn = (e.force_bn & 1023) ? (e.force_bn & 1023) : pick_bn(p.M, Cout, 9 * Cin, e);
  const bool cl = use_cluster(p.M, e.force_bn, true);
  CUtensorMap tmA, tmB, tmC, tmR;
  int rc = make_tmap_nhwc(&tmA, X, NB, H, W, Cin, tw, th);
  if (rc) return rc;
  rc = make_tmap_2d(&tmB, Wk, Cout, 9L * Cin, 9L * Cin, cl ? bn / 2 : bn);
  if (rc) return rc;
  rc = setup_staging(p, e, p.M, Cout, bn, &tmC, &tmR);
  if (rc) return rc;
  return dispatch_bn(bn, [&](auto w) {
    constexpr int kBN = decltype(w)::value;
    return cl ? launch_gemm_cl<kBN, 2>(tmA, tmB, tmC, tmR, p, st) : launch_gemm_cl<kBN, 1>(tmA, tmB, tmC, tmR, p, st);
  });
}

}  // namespace emu
