// emu_b200 — flash attention on the Hopper tensor cores (wgmma + TMA), the dense-attention path of
//   * the EVA-CLIP ViT blocks            (reference: Emu2/emu/eva_vit.py:228-283 `Attention.forward`, non-causal, D=112)
//   * the SD-XL UNet self-attention      (diffusers 0.24 `Attention` via Emu2/emu/diffusion.py:136-141, D=64, 4096/1024 tokens)
//   * LLaMA prefill / `generate_image`   (transformers `LlamaAttention`, Emu2/emu/lm.py:37-41, causal + left padding, D=128)
// softmax(scale * Q K^T [+ mask]) V with fp32 scores / statistics and bf16 probabilities — the same rounding points as
// the mma.sync kernel in attention.cu, which stays the path for additive-bias (T5) and tiny problems.
//
// One CTA = 128 query rows of one (batch, head); K/V blocks stream through a 3-stage TMA ring (4-D tensor maps over the
// strided [B, N, H, D] views, 128B swizzle, out-of-bounds rows / head-dim padding arrive as zeros) and are shared by the
// two consumer warpgroups (64 query rows each).  Per KV block a consumer runs S = Q K^T as wgmma from shared memory,
// the online softmax on the S fragment in registers, and O += P V as wgmma with P as the register A operand and V used in
// place as an MN-major B operand (no transpose pass); O accumulates in registers.
#include <cstdlib>

#include <cuda.h>
#include <cuda_runtime.h>

#include "common.cuh"
#include "ops.h"
#include "wgmma.cuh"

namespace emu {

int make_tmap_bnhd(CUtensorMap* out, const void* base, int D, long N, int H, int B, long ts, long hs, long bs, int box_rows,
                   int* head_first);  // gemm_tc.cu

namespace {

constexpr int kAtStages = 3;

template <int DT, int BN>
struct AtCfg {
  static constexpr int kThreads = 384;             // warpgroup 0 = TMA producer, warpgroups 1/2 = query rows 0..63 / 64..127
  static constexpr int kDC = DT / 64;              // 64-wide head-dim chunks (one 128 B swizzle row each)
  static constexpr int kQBytes = 128 * DT * 2;     // the Q tile
  static constexpr int kKVBytes = BN * DT * 2;     // one K (or V) block
  static constexpr int kOffK = kQBytes;
  static constexpr int kOffV = kOffK + kAtStages * kKVBytes;
  static constexpr int kOffBar = kOffV + kAtStages * kKVBytes;
  static constexpr int kSmem = kOffBar + 32 * 8 + 1024;  // + 1024 B alignment slack
  static_assert(BN % 16 == 0 && DT % 64 == 0, "tile shapes");
  static_assert(kSmem <= 227 * 1024, "SMEM budget");
};

struct AtParams {
  bf16* out;
  long o_bs, o_ts, o_hs;
  const int* kv_start;
  const int* kv_row;  // [B] K/V batch coordinate of query batch b, or null = b
  const int* q_off;   // [B] kPacked: key position of query 0 of batch b (AttnArgs::q_off)
  const int* q_len;   // [B] kPacked: query rows of batch b (AttnArgs::q_len)
  int Nq, Nk, D;  // D = real head dim (<= DT)
  int causal;
  float scale_log2;  // scale * log2(e)
  int pdl;
  int q_hf, k_hf, v_hf;  // tensor-map coordinate order: 1 = (d, head, token, batch), 0 = (d, token, head, batch)
  const int* q_row0;     // [B] kPacked: first row of batch b in the one-batch q / out views (AttnArgs::q_row0)
};

__device__ __forceinline__ void load_rows(void* dst, const CUtensorMap* m, uint64_t* bar, int d0, int tok, int head, int batch,
                                          int head_first) {
  if (head_first) tma_load_4d(dst, m, bar, d0, head, tok, batch);
  else tma_load_4d(dst, m, bar, d0, tok, head, batch);
}

// kPacked (slot mode): batch b's queries are rows q_row0[b] .. + q_len[b] of ONE packed q / out view at key positions
// q_off[b] + i, so each CTA bounds its key loop by its own batch's offset; a CTA past its batch's rows does nothing, and rows
// past them (the next batch's, or zeros past the view) are never stored.
template <int DT, int BN, bool kPacked>
__global__ void __launch_bounds__(AtCfg<DT, BN>::kThreads, 1)
attn_tc_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK,
               const __grid_constant__ CUtensorMap tmV, const AtParams p) {
  using C = AtCfg<DT, BN>;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + C::kOffBar);
  uint64_t* q_full = bars;                 // [1]
  uint64_t* k_full = bars + 1;             // [3]
  uint64_t* k_empty = k_full + kAtStages;  // [3]
  uint64_t* v_full = k_empty + kAtStages;
  uint64_t* v_empty = v_full + kAtStages;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int q0 = blockIdx.x * 128, head = blockIdx.y, batch = blockIdx.z;
  const int off = kPacked ? p.q_off[batch] : p.Nk - p.Nq;
  // keys of this batch: all Nk, or (kPacked) up to the end of its rows, which is all the caller wrote
  const int kv_n = kPacked ? min(p.Nk, off + (p.q_len ? p.q_len[batch] : p.Nq)) : p.Nk;
  const int q_n = kPacked ? p.q_len[batch] : p.Nq;  // this batch's query rows
  int kmax = kv_n - 1;  // last key any query row of this CTA may see
  if (p.causal) kmax = min(kmax, min(q0 + 127, q_n - 1) + off);
  const int nb = kmax < 0 || (kPacked && q0 >= q_n) ? 0 : kmax / BN + 1;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmQ);
    tma_prefetch_desc(&tmK);
    tma_prefetch_desc(&tmV);
    mbar_init(q_full, 1);
    for (int i = 0; i < kAtStages; ++i) {
      mbar_init(&k_full[i], 1);
      mbar_init(&k_empty[i], 8);  // lane 0 of every consumer warp
      mbar_init(&v_full[i], 1);
      mbar_init(&v_empty[i], 8);
    }
    mbar_fence_init();
  }
  if (p.pdl) pdl_launch_dependents();
  __syncthreads();

  if (warp < 4) {
    // ===================== TMA producer =====================
    if (warp == 0 && lane == 0 && nb > 0) {
      if (p.pdl) pdl_wait();  // Q/K/V are the predecessor's output; all stores of this kernel happen after these loads
      const int kvb = p.kv_row ? p.kv_row[batch] : batch;
      mbar_expect_tx(q_full, C::kQBytes);
      if (kPacked) {
        for (int c = 0; c < C::kDC; ++c) load_rows(smem + c * (128 * 128), &tmQ, q_full, c * 64, p.q_row0[batch] + q0, head, 0, p.q_hf);
      } else {
        for (int c = 0; c < C::kDC; ++c) load_rows(smem + c * (128 * 128), &tmQ, q_full, c * 64, q0, head, batch, p.q_hf);
      }
      for (int j = 0; j < nb; ++j) {
        const int s = j % kAtStages;
        const uint32_t ph = (uint32_t)(j / kAtStages) & 1u;
        mbar_wait(&k_empty[s], ph ^ 1);
        mbar_expect_tx(&k_full[s], C::kKVBytes);
        for (int c = 0; c < C::kDC; ++c)
          load_rows(smem + C::kOffK + s * C::kKVBytes + c * (BN * 128), &tmK, &k_full[s], c * 64, j * BN, head, kvb, p.k_hf);
        mbar_wait(&v_empty[s], ph ^ 1);
        mbar_expect_tx(&v_full[s], C::kKVBytes);
        for (int c = 0; c < C::kDC; ++c)
          load_rows(smem + C::kOffV + s * C::kKVBytes + c * (BN * 128), &tmV, &v_full[s], c * 64, j * BN, head, kvb, p.v_hf);
      }
    }
  } else {
    // ===================== consumers: 64 query rows each =====================
    // S / O fragments (wgmma accumulator layout): rows qi[h] = q0 + 64 wg + 16 (warp % 4) + lane / 4 + 8 h, columns
    // 8 jj + 2 (lane % 4) + e at index 4 jj + 2 h + e.  P is re-packed from the S fragment into the register A operand.
    const int wg = (warp >> 2) - 1;
    const int t = lane & 3;
    int qi[2];
    qi[0] = q0 + 64 * wg + 16 * (warp & 3) + (lane >> 2);
    qi[1] = qi[0] + 8;
    const uint32_t sQ = smem_u32(smem) + wg * (64 * 128), sK = smem_u32(smem + C::kOffK), sV = smem_u32(smem + C::kOffV);
    const float c = p.scale_log2;
    const int lo = p.kv_start ? p.kv_start[batch] : 0;
    int hi[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) hi[h] = p.causal ? min(kv_n - 1, qi[h] + off) : kv_n - 1;
    float o[DT / 2];
#pragma unroll
    for (int i = 0; i < DT / 2; ++i) o[i] = 0.f;
    float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};
    if (nb > 0) mbar_wait(q_full, 0);
    for (int j = 0; j < nb; ++j) {
      const int s = j % kAtStages;
      const uint32_t ph = (uint32_t)(j / kAtStages) & 1u;
      // ---- S = Q K_j^T ----
      float sc[BN / 2];
      mbar_wait(&k_full[s], ph);
      wgmma_fence();
#pragma unroll
      for (int cc = 0; cc < C::kDC; ++cc) {
        const uint64_t da = wgmma_desc_sw128(sQ + cc * (128 * 128));
        const uint64_t db = wgmma_desc_sw128(sK + s * C::kKVBytes + cc * (BN * 128));
#pragma unroll
        for (int k = 0; k < 4; ++k) WgmmaSS<BN>::run(sc, da + 2 * k, db + 2 * k, (cc | k) != 0);
      }
      wgmma_commit();
      wgmma_wait<0>();
      __syncwarp();
      if (lane == 0) mbar_arrive(&k_empty[s]);
      // ---- mask, online softmax (log2 domain) ----
      const int k0 = j * BN;
      float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
      for (int i = 0; i < BN / 2; ++i) {
        const int h = (i >> 1) & 1;
        const int kj = k0 + 8 * (i >> 2) + 2 * t + (i & 1);
        const float x = (kj >= lo && kj <= hi[h]) ? sc[i] * c : -INFINITY;
        sc[i] = x;
        mx[h] = fmaxf(mx[h], x);
      }
      float m_use[2], corr[2];
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        mx[h] = fmaxf(mx[h], __shfl_xor_sync(0xffffffffu, mx[h], 1));
        mx[h] = fmaxf(mx[h], __shfl_xor_sync(0xffffffffu, mx[h], 2));
        const float m_new = fmaxf(m_run[h], mx[h]);
        m_use[h] = (m_new == -INFINITY) ? 0.f : m_new;  // fully masked row so far
        corr[h] = (m_run[h] == -INFINITY) ? 0.f : ex2_approx_ftz(m_run[h] - m_use[h]);
        m_run[h] = m_new;
      }
      float rs[2] = {0.f, 0.f};
      uint32_t pa[BN / 16][4];
#pragma unroll
      for (int jj = 0; jj < BN / 8; ++jj) {
        const float p0 = ex2_approx_ftz(sc[4 * jj] - m_use[0]), p1 = ex2_approx_ftz(sc[4 * jj + 1] - m_use[0]);
        const float p2 = ex2_approx_ftz(sc[4 * jj + 2] - m_use[1]), p3 = ex2_approx_ftz(sc[4 * jj + 3] - m_use[1]);
        rs[0] += p0 + p1;
        rs[1] += p2 + p3;
        pa[jj >> 1][(jj & 1) * 2] = pack_bf16(p0, p1);
        pa[jj >> 1][(jj & 1) * 2 + 1] = pack_bf16(p2, p3);
      }
#pragma unroll
      for (int h = 0; h < 2; ++h) l_run[h] = l_run[h] * corr[h] + rs[h];
#pragma unroll
      for (int i = 0; i < DT / 2; ++i) o[i] *= corr[(i >> 1) & 1];
      // ---- O += P V_j : V is used in place as an MN-major B operand (64-wide d chunks BN*128 B apart, 8-key groups 1 KB) ----
      mbar_wait(&v_full[s], ph);
      if (kPacked && k0 + BN > kv_n) {
        // the tile runs past this batch's last written key: zero those V rows (128 B each in every 64-wide chunk, whatever
        // the swizzle) so a stale non-finite value cannot reach O through a zero probability.  Both consumer warpgroups
        // write the same zeros; each makes its own writes visible to its wgmma before issuing it.
        uint8_t* vt = smem + C::kOffV + s * C::kKVBytes;
        const int r0 = kv_n - k0, units = (BN - r0) * 8, tid = threadIdx.x - 128 * (wg + 1);
        for (int cc = 0; cc < C::kDC; ++cc)
          for (int u = tid; u < units; u += 128)
            *reinterpret_cast<uint4*>(vt + cc * (BN * 128) + r0 * 128 + u * 16) = make_uint4(0u, 0u, 0u, 0u);
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
        asm volatile("bar.sync %0, 128;" ::"r"(wg + 1) : "memory");
      }
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < BN / 16; ++kk)
        WgmmaRS<DT, 1>::run(o, pa[kk], wgmma_desc_sw128(sV + s * C::kKVBytes + kk * 2048, BN * 128, 1024), 1);
      wgmma_commit();
      wgmma_wait<0>();
      __syncwarp();
      if (lane == 0) mbar_arrive(&v_empty[s]);
    }
    // ---- normalise and store ----
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      l_run[h] += __shfl_xor_sync(0xffffffffu, l_run[h], 1);
      l_run[h] += __shfl_xor_sync(0xffffffffu, l_run[h], 2);
    }
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      if (qi[h] >= q_n) continue;
      const float inv = l_run[h] > 0.f ? 1.f / l_run[h] : 0.f;
      bf16* dst = p.out + (kPacked ? (long)(p.q_row0[batch] + qi[h]) * p.o_ts : (long)batch * p.o_bs + (long)qi[h] * p.o_ts) +
                  (long)head * p.o_hs;
#pragma unroll
      for (int jj = 0; jj < DT / 8; ++jj) {
        const int d = 8 * jj + 2 * t;
        if (d < p.D) *reinterpret_cast<uint32_t*>(dst + d) = pack_bf16(o[4 * jj + 2 * h] * inv, o[4 * jj + 2 * h + 1] * inv);
      }
    }
  }
}

template <int DT, int BN, bool kPacked = false>
int launch_attn_tc(const AttnArgs& a, cudaStream_t st) {
  using C = AtCfg<DT, BN>;
  static bool attr_set = false;
  if (!attr_set) {
    if (cudaFuncSetAttribute(attn_tc_kernel<DT, BN, kPacked>, cudaFuncAttributeMaxDynamicSharedMemorySize, C::kSmem) !=
        cudaSuccess)
      return EMU_ERR_CUDA;
    attr_set = true;
  }
  CUtensorMap tq, tk, tv;
  AtParams p;
  if (kPacked) {  // one batch of q_rows rows: a tile past the last row loads zeros
    if (make_tmap_bnhd(&tq, a.q, a.D, a.q_rows, a.H, 1, a.q_ts, a.q_hs, 0, 128, &p.q_hf) != EMU_OK) return EMU_ERR_UNSUPPORTED;
  } else if (make_tmap_bnhd(&tq, a.q, a.D, a.Nq, a.H, a.B, a.q_ts, a.q_hs, a.q_bs, 128, &p.q_hf) != EMU_OK) {
    return EMU_ERR_UNSUPPORTED;
  }
  const int kvB = a.kv_row && a.kv_rows > 0 ? a.kv_rows : a.B;  // a row-mapped K/V map spans every cache row
  if (make_tmap_bnhd(&tk, a.k, a.D, a.Nk, a.H, kvB, a.k_ts, a.k_hs, a.k_bs, BN, &p.k_hf) != EMU_OK) return EMU_ERR_UNSUPPORTED;
  if (make_tmap_bnhd(&tv, a.v, a.D, a.Nk, a.H, kvB, a.v_ts, a.v_hs, a.v_bs, BN, &p.v_hf) != EMU_OK) return EMU_ERR_UNSUPPORTED;
  p.out = a.out; p.o_bs = a.o_bs; p.o_ts = a.o_ts; p.o_hs = a.o_hs;
  p.kv_start = a.kv_start; p.kv_row = a.kv_row; p.q_off = a.q_off; p.q_len = a.q_len; p.Nq = a.Nq; p.Nk = a.Nk; p.D = a.D; p.causal = a.causal;
  p.scale_log2 = a.scale * 1.4426950408889634f;
  p.pdl = g_pdl_chain;
  p.q_row0 = a.q_row0;
  dim3 grid((a.Nq + 127) / 128, a.H, a.B);
  return launch_kernel(attn_tc_kernel<DT, BN, kPacked>, grid, dim3(C::kThreads), C::kSmem, st, p.pdl, tq, tk, tv, p);
}

}  // namespace

// returns EMU_ERR_UNSUPPORTED when the problem should go to the mma.sync kernel instead
int attn_prefill_tc(const AttnArgs& a, cudaStream_t st) {
  if (a.bias != nullptr || a.D % 8 || a.D > 128 || a.D < 16) return EMU_ERR_UNSUPPORTED;
  if (a.Nq < 128 || a.Nk < 64) return EMU_ERR_UNSUPPORTED;        // tiny problems: launch-latency bound anyway
  if (a.causal && a.Nk < a.Nq) return EMU_ERR_UNSUPPORTED;
  if ((a.o_ts % 8) || (a.o_hs % 8) || (a.o_bs % 8) || (reinterpret_cast<uintptr_t>(a.out) & 15)) return EMU_ERR_UNSUPPORTED;
  if ((reinterpret_cast<uintptr_t>(a.q) & 15) || (reinterpret_cast<uintptr_t>(a.k) & 15) || (reinterpret_cast<uintptr_t>(a.v) & 15))
    return EMU_ERR_UNSUPPORTED;
  if (a.H > 65535 || a.B > 65535) return EMU_ERR_UNSUPPORTED;
  if (a.q_off || a.q_len || a.q_row0) {  // packed queries (slot mode): the LLaMA head dims only
    if (!a.q_off || !a.q_len || !a.q_row0 || a.q_rows < 1) return EMU_ERR_INVALID;
    if (!a.causal) return EMU_ERR_UNSUPPORTED;
    if (a.D == 64) return launch_attn_tc<64, 128, true>(a, st);
    if (a.D == 128) return launch_attn_tc<128, 64, true>(a, st);
    return EMU_ERR_UNSUPPORTED;
  }
  if (a.D <= 64) {
    if (a.Nk <= 64) return launch_attn_tc<64, 64>(a, st);  // cross-attention: 64 keys
    return launch_attn_tc<64, 128>(a, st);
  }
  return launch_attn_tc<128, 64>(a, st);
}

}  // namespace emu
