// emu_b200 — bandwidth-bound kernels of the diffusion half (UNet / VAE / Euler scheduler), NHWC bf16.
//
// GroupNorm(+SiLU) [diffusers ResnetBlock2D / Transformer2DModel norms], sinusoidal timestep embedding
// [diffusers get_timestep_embedding, flip_sin_to_cos=True], nearest 2x upsample, channel concat (UNet skip
// connections), explicit im2col (stride-2 downsamplers and non-tileable tiny feature maps), NCHW<->NHWC boundary
// conversion, fused CFG + Euler step (Emu2/emu/diffusion.py:131-149).
#include "common.cuh"
#include "ops.h"

namespace emu {

// ----------------------------------------------------------------------------------------------
// GroupNorm over NHWC: stage 1 — per (image, pixel-chunk) partial sums for every group (coalesced row reads)
// ----------------------------------------------------------------------------------------------
constexpr int kGnChunks = 128;  // partial-sum slots per image (x NB CTAs of 512 threads: ~2 CTAs per SM in flight)

// The sums are taken of x - pivot, the pivot being the first element of the (image, group) plane.  Without the shift,
// var = E[x^2] - mean^2 in fp32 cancels: its relative error grows as 2^-24 (mean/std)^2 times the summation length, which
// reaches the bf16 output's own rounding once |mean| is a few hundred standard deviations.  Shifted, mean/std is that of
// one sample's distance from the mean, so the cancellation is gone while the summation order (and determinism) is kept.
__device__ __forceinline__ float gn_pivot(const bf16* x_img, int c, int cpg) {
  return __bfloat162float(x_img[c / cpg * cpg]);
}

__global__ void __launch_bounds__(512) gn_partial_kernel(const bf16* __restrict__ x, float* __restrict__ part, int HW,
                                                         int C, int groups, int pdl) {
  // grid (kGnChunks, NB); part[((b*kGnChunks + chunk)*groups + g)*2 + {0,1}] = {sum, sumsq} of x - pivot
  __shared__ float stage[512 * 16];  // per-thread {sum[8], sumsq[8]}
  if (pdl) {
    pdl_launch_dependents();
    pdl_wait();
  }
  const int chunk = blockIdx.x, b = blockIdx.y;
  const int cpg = C / groups;
  const int p0 = (int)((long)HW * chunk / kGnChunks), p1 = (int)((long)HW * (chunk + 1) / kGnChunks);
  const int vecC = C >> 3;  // 8 channels per 16-byte vector
  // every active thread owns ONE channel vector and walks down the pixels: sums stay in registers
  const int stride = (blockDim.x / vecC) * vecC;
  if ((int)threadIdx.x < stride) {
    const int cv = threadIdx.x % vecC;
    const long total = (long)(p1 - p0) * vecC;
    const bf16* base = x + ((long)b * HW + p0) * C;
    float s[8], s2[8], piv[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      s[j] = s2[j] = 0.f;
      piv[j] = gn_pivot(x + (long)b * HW * C, cv * 8 + j, cpg);
    }
#pragma unroll 4
    for (long idx = threadIdx.x; idx < total; idx += stride) {
      const long pix = idx / vecC;
      const uint4 v = *reinterpret_cast<const uint4*>(base + pix * C + cv * 8);
      const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float lo = bf16_lo(w[j]) - piv[2 * j], hi = bf16_hi(w[j]) - piv[2 * j + 1];
        s[2 * j] += lo; s2[2 * j] += lo * lo;
        s[2 * j + 1] += hi; s2[2 * j + 1] += hi * hi;
      }
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      stage[threadIdx.x * 16 + j] = s[j];
      stage[threadIdx.x * 16 + 8 + j] = s2[j];
    }
  }
  __syncthreads();
  // fixed-order reduction (deterministic): group gi <- channels [gi*cpg, (gi+1)*cpg) x pixel lanes
  const int lanes = stride / vecC;
  for (int gi = threadIdx.x; gi < groups; gi += blockDim.x) {
    float a = 0.f, a2 = 0.f;
    for (int c = gi * cpg; c < (gi + 1) * cpg; ++c) {
      const int cvc = c >> 3, j = c & 7;
      for (int k = 0; k < lanes; ++k) {
        a += stage[(cvc + k * vecC) * 16 + j];
        a2 += stage[(cvc + k * vecC) * 16 + 8 + j];
      }
    }
    part[(((long)b * kGnChunks + chunk) * groups + gi) * 2] = a;
    part[(((long)b * kGnChunks + chunk) * groups + gi) * 2 + 1] = a2;
  }
}

// stage 2 — normalise (+ optional SiLU); mean/rstd are rebuilt from the partials by every CTA (fixed order)
__global__ void __launch_bounds__(256) gn_apply_kernel(const bf16* __restrict__ x, const float* __restrict__ part_,
                                                       const bf16* __restrict__ w, const bf16* __restrict__ bsh,
                                                       bf16* __restrict__ y, int HW, int C, int groups, float eps,
                                                       int do_silu, int pdl) {
  extern __shared__ float st[];  // [groups*2] mean, rstd
  if (pdl) {
    pdl_launch_dependents();
    pdl_wait();
  }
  const int b = blockIdx.y;
  const int cpg = C / groups;
  // rebuild mean / rstd from the kGnChunks partial sums: (group, chunk-slice) pairs spread over the whole CTA so the
  // dependent-load chain is kGnChunks / nparts long instead of kGnChunks; fixed summation order -> deterministic
  __shared__ float ps[256 * 2];
  const int nparts = groups <= 256 ? 256 / groups : 1;
  for (int g0 = 0; g0 < groups; g0 += 256) {
    const int g = g0 + (int)threadIdx.x % (groups < 256 ? groups : 256);
    const int part = (int)threadIdx.x / (groups < 256 ? groups : 256);
    float s = 0.f, s2 = 0.f;
    if (g < groups && part < nparts) {
      for (int c = part; c < kGnChunks; c += nparts) {
        s += part_[(((long)b * kGnChunks + c) * groups + g) * 2];
        s2 += part_[(((long)b * kGnChunks + c) * groups + g) * 2 + 1];
      }
    }
    ps[threadIdx.x * 2] = s;
    ps[threadIdx.x * 2 + 1] = s2;
    __syncthreads();
    if (part == 0 && g < groups) {
      const int gw = groups < 256 ? groups : 256;
      float a = 0.f, a2 = 0.f;
      for (int q = 0; q < nparts; ++q) {
        a += ps[(q * gw + (int)threadIdx.x) * 2];
        a2 += ps[(q * gw + (int)threadIdx.x) * 2 + 1];
      }
      const float n = (float)HW * cpg;
      const float dmean = a / n;  // mean of x - pivot
      const float var = fmaxf(a2 / n - dmean * dmean, 0.f);
      st[g * 2] = gn_pivot(x + (long)b * HW * C, g * cpg, cpg) + dmean;
      st[g * 2 + 1] = rsqrtf(var + eps);
    }
    __syncthreads();
  }
  __syncthreads();
  // every thread owns ONE 8-channel vector (its affine constants live in registers) and walks down the pixels
  const int vecC = C >> 3;
  const int nthreads = gridDim.x * blockDim.x;
  const int stride = (nthreads / vecC) * vecC;
  const int gtid = blockIdx.x * blockDim.x + threadIdx.x;
  if (gtid >= stride) return;
  const int cv = gtid % vecC;
  float mu[8], sc[8], wt[8], sh[8];
  {
    const uint4 wv = *reinterpret_cast<const uint4*>(w + cv * 8);
    const uint4 bv = *reinterpret_cast<const uint4*>(bsh + cv * 8);
    const uint32_t ww[4] = {wv.x, wv.y, wv.z, wv.w}, bb[4] = {bv.x, bv.y, bv.z, bv.w};
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int c = cv * 8 + 2 * j;
      const int g0 = c / cpg, g1 = (c + 1) / cpg;  // an 8-channel vector may straddle two groups
      mu[2 * j] = st[g0 * 2]; mu[2 * j + 1] = st[g1 * 2];
      sc[2 * j] = st[g0 * 2 + 1]; sc[2 * j + 1] = st[g1 * 2 + 1];
      wt[2 * j] = bf16_lo(ww[j]); wt[2 * j + 1] = bf16_hi(ww[j]);
      sh[2 * j] = bf16_lo(bb[j]); sh[2 * j + 1] = bf16_hi(bb[j]);
    }
  }
  const bf16* xb = x + (long)b * HW * C + cv * 8;
  bf16* yb = y + (long)b * HW * C + cv * 8;
  const int pstep = stride / vecC;
  for (long pix = gtid / vecC; pix < HW; pix += pstep) {
    const uint4 v = *reinterpret_cast<const uint4*>(xb + pix * C);
    const uint32_t xv[4] = {v.x, v.y, v.z, v.w};
    uint32_t o[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      float lo = (bf16_lo(xv[j]) - mu[2 * j]) * sc[2 * j] * wt[2 * j] + sh[2 * j];
      float hi = (bf16_hi(xv[j]) - mu[2 * j + 1]) * sc[2 * j + 1] * wt[2 * j + 1] + sh[2 * j + 1];
      if (do_silu) {  // F.silu(group_norm(x)) with the bf16 rounding of the norm output in between
        lo = silu(round_bf16(lo));
        hi = silu(round_bf16(hi));
      }
      o[j] = pack_bf16(lo, hi);
    }
    *reinterpret_cast<uint4*>(yb + pix * C) = make_uint4(o[0], o[1], o[2], o[3]);
  }
}

int groupnorm_nhwc(const bf16* x, const bf16* w, const bf16* b, bf16* y, float* scratch, int NB, int HW, int C,
                   int groups, float eps, int do_silu, cudaStream_t st) {
  if (C % 8 || C % groups || C > 4096) return EMU_ERR_INVALID;
  const int pdl = g_pdl_chain;
  {
    const int rc = launch_kernel(gn_partial_kernel, dim3(kGnChunks, NB), dim3(512), 0, st, pdl, x, scratch, HW, C, groups, pdl);
    if (rc) return rc;
  }
  const long total = (long)HW * (C >> 3);
  int gx = (int)((total + 255) / 256);
  const int cap = (4 * kNumSMs + NB - 1) / NB;
  if (gx > cap) gx = cap;
  if (gx < ((C >> 3) + 255) / 256) gx = ((C >> 3) + 255) / 256;  // at least one thread per 8-channel vector
  return launch_kernel(gn_apply_kernel, dim3(gx, NB), dim3(256), groups * 2 * sizeof(float), st, pdl, x, scratch, w, b, y, HW,
                       C, groups, eps, do_silu, pdl);
}
size_t groupnorm_scratch_bytes(int NB, int groups) { return (size_t)NB * kGnChunks * groups * 2 * sizeof(float); }

// ----------------------------------------------------------------------------------------------
// sinusoidal embedding: out[r, :] = [cos(t_r * f_j) | sin(t_r * f_j)], f_j = exp(-ln(1e4) * j / half)
// ----------------------------------------------------------------------------------------------
__global__ void timestep_embedding_kernel(const float* __restrict__ t, bf16* out, int rows, int dim, int ld,
                                          int col_off, int grp) {
  // row r belongs to output row r / grp, slot r % grp (grp = 6 packs the SDXL time_ids side by side)
  const int half = dim / 2;
  for (int idx = blockIdx.x * blockDim.x + threadIdx.x; idx < rows * half; idx += gridDim.x * blockDim.x) {
    const int r = idx / half, j = idx % half;
    const float f = expf(-9.210340371976184f * (float)j / (float)half);
    const float a = t[r] * f;
    bf16* o = out + (long)(r / grp) * ld + col_off + (r % grp) * dim;
    o[j] = __float2bfloat16_rn(cosf(a));
    o[half + j] = __float2bfloat16_rn(sinf(a));
  }
}
int timestep_embedding(const float* t, bf16* out, int rows, int dim, int ld, int col_off, int grp, cudaStream_t st) {
  timestep_embedding_kernel<<<(rows * dim / 2 + 255) / 256, 256, 0, st>>>(t, out, rows, dim, ld, col_off, grp);
  return cudaGetLastError() == cudaSuccess ? EMU_OK : EMU_ERR_CUDA;
}
__global__ void int_to_float_kernel(const int* __restrict__ x, float* y, int n) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) y[i] = (float)x[i];
}
int int_to_float(const int* x, float* y, int n, cudaStream_t st) {
  int_to_float_kernel<<<(n + 255) / 256, 256, 0, st>>>(x, y, n);
  return cudaGetLastError() == cudaSuccess ? EMU_OK : EMU_ERR_CUDA;
}

__global__ void silu_kernel(const bf16* __restrict__ x, bf16* y, long n) {
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x)
    y[i] = __float2bfloat16_rn(silu(__bfloat162float(x[i])));
}
int silu_rows(const bf16* x, bf16* y, long n, cudaStream_t st) {
  silu_kernel<<<(int)((n + 255) / 256 < 1024 ? (n + 255) / 256 : 1024), 256, 0, st>>>(x, y, n);
  return cudaGetLastError() == cudaSuccess ? EMU_OK : EMU_ERR_CUDA;
}

// copy [rows, cols] (src stride lds) into dst at column offset (dst stride ldd); used for channel concat
__global__ void copy_cols_kernel(const bf16* __restrict__ src, bf16* dst, long rows, int cols, int lds, int ldd,
                                 int col_off, int pdl) {
  if (pdl) {
    pdl_launch_dependents();
    pdl_wait();
  }
  const int vc = cols >> 3;
  const long total = rows * vc;
  for (long idx = blockIdx.x * (long)blockDim.x + threadIdx.x; idx < total; idx += (long)gridDim.x * blockDim.x) {
    const long r = idx / vc;
    const int c = (idx % vc) * 8;
    *reinterpret_cast<uint4*>(dst + r * ldd + col_off + c) = *reinterpret_cast<const uint4*>(src + r * lds + c);
  }
}
int copy_cols(const bf16* src, bf16* dst, long rows, int cols, int lds, int ldd, int col_off, cudaStream_t st) {
  if ((cols | lds | ldd | col_off) % 8) return EMU_ERR_INVALID;
  return launch_kernel(copy_cols_kernel, dim3(4 * kNumSMs), dim3(256), 0, st, g_pdl_chain, src, dst, rows, cols, lds, ldd,
                       col_off, g_pdl_chain);
}

// nearest-neighbour 2x upsample, NHWC
__global__ void upsample2x_kernel(const bf16* __restrict__ x, bf16* y, int NB, int H, int W, int C) {
  const int vc = C >> 3;
  const long total = (long)NB * 2 * H * 2 * W * vc;
  for (long idx = blockIdx.x * (long)blockDim.x + threadIdx.x; idx < total; idx += (long)gridDim.x * blockDim.x) {
    const int c = (idx % vc) * 8;
    long p = idx / vc;
    const int ox = p % (2 * W);
    p /= 2 * W;
    const int oy = p % (2 * H);
    const int b = p / (2 * H);
    *reinterpret_cast<uint4*>(y + (((long)b * 2 * H + oy) * 2 * W + ox) * C + c) =
        *reinterpret_cast<const uint4*>(x + (((long)b * H + (oy >> 1)) * W + (ox >> 1)) * C + c);
  }
}
int upsample2x_nhwc(const bf16* x, bf16* y, int NB, int H, int W, int C, cudaStream_t st) {
  if (C % 8) return EMU_ERR_INVALID;
  upsample2x_kernel<<<8 * kNumSMs, 256, 0, st>>>(x, y, NB, H, W, C);
  return cudaGetLastError() == cudaSuccess ? EMU_OK : EMU_ERR_CUDA;
}

// explicit im2col for 3x3 pad-1 convs with stride s: out[(b,oy,ox), (r*3+s_)*C + c]
__global__ void im2col3x3_kernel(const bf16* __restrict__ x, bf16* out, int NB, int H, int W, int C, int stride, int Ho,
                                 int Wo) {
  const int vc = C >> 3;
  const long total = (long)NB * Ho * Wo * 9 * vc;
  for (long idx = blockIdx.x * (long)blockDim.x + threadIdx.x; idx < total; idx += (long)gridDim.x * blockDim.x) {
    const int c = (idx % vc) * 8;
    long p = idx / vc;
    const int tap = p % 9;
    p /= 9;
    const int ox = p % Wo;
    p /= Wo;
    const int oy = p % Ho;
    const int b = p / Ho;
    const int iy = oy * stride + tap / 3 - 1, ix = ox * stride + tap % 3 - 1;
    uint4 v = make_uint4(0, 0, 0, 0);
    if (iy >= 0 && iy < H && ix >= 0 && ix < W) v = *reinterpret_cast<const uint4*>(x + (((long)b * H + iy) * W + ix) * C + c);
    *reinterpret_cast<uint4*>(out + (((long)b * Ho + oy) * Wo + ox) * 9 * C + tap * C + c) = v;
  }
}
int im2col3x3(const bf16* x, bf16* out, int NB, int H, int W, int C, int stride, cudaStream_t st) {
  if (C % 8) return EMU_ERR_INVALID;
  const int Ho = (H + 2 - 3) / stride + 1, Wo = (W + 2 - 3) / stride + 1;
  im2col3x3_kernel<<<8 * kNumSMs, 256, 0, st>>>(x, out, NB, H, W, C, stride, Ho, Wo);
  return cudaGetLastError() == cudaSuccess ? EMU_OK : EMU_ERR_CUDA;
}

// NCHW (C real channels) -> NHWC padded to Cp channels (zero fill), and back; optional input scale
__global__ void nchw_to_nhwc_kernel(const bf16* __restrict__ x, bf16* y, int NB, int C, int HW, int Cp, float scale) {
  const long total = (long)NB * HW * Cp;
  for (long idx = blockIdx.x * (long)blockDim.x + threadIdx.x; idx < total; idx += (long)gridDim.x * blockDim.x) {
    const int c = idx % Cp;
    const long p = (idx / Cp) % HW;
    const int b = idx / ((long)Cp * HW);
    y[idx] = c < C ? __float2bfloat16_rn(__bfloat162float(x[((long)b * C + c) * HW + p]) * scale) : __float2bfloat16(0.f);
  }
}
int nchw_to_nhwc(const bf16* x, bf16* y, int NB, int C, int HW, int Cp, float scale, cudaStream_t st) {
  nchw_to_nhwc_kernel<<<2 * kNumSMs, 256, 0, st>>>(x, y, NB, C, HW, Cp, scale);
  return cudaGetLastError() == cudaSuccess ? EMU_OK : EMU_ERR_CUDA;
}
__global__ void nhwc_to_nchw_kernel(const bf16* __restrict__ x, bf16* y, int NB, int C, int HW, int ldx) {
  const long total = (long)NB * C * HW;
  for (long idx = blockIdx.x * (long)blockDim.x + threadIdx.x; idx < total; idx += (long)gridDim.x * blockDim.x) {
    const long p = idx % HW;
    const int c = (idx / HW) % C;
    const int b = idx / ((long)HW * C);
    y[idx] = x[((long)b * HW + p) * ldx + c];
  }
}
int nhwc_to_nchw(const bf16* x, bf16* y, int NB, int C, int HW, int ldx, cudaStream_t st) {
  nhwc_to_nchw_kernel<<<2 * kNumSMs, 256, 0, st>>>(x, y, NB, C, HW, ldx);
  return cudaGetLastError() == cudaSuccess ? EMU_OK : EMU_ERR_CUDA;
}

// ----------------------------------------------------------------------------------------------
// denoise-step glue (Emu2/emu/diffusion.py:131-149)
// ----------------------------------------------------------------------------------------------
// The Euler glue serves B latent slots, each at its own step: slot b reads {sigma, sigma_next, timestep, guidance} at
// params + b * ps on the device (ps = 0: one set for all slots), so one captured graph serves every step.  Slot b's conditional
// UNet row is b * cs and its unconditional row ub + b * cs: [cond_1..B; uncond_1..B] is cs = 1, ub = B; slots whose two rows
// are adjacent are cs = 2, ub = 1.
//
// latent_model_input = cat([latents]*2) / sqrt(sigma^2+1), written straight as NHWC (Cp channels, zero padded) into the
// `copies` rows of every slot, and the slot's timestep into t_rows at the same rows
__global__ void slot_prepare_kernel(const float* __restrict__ lat, bf16* xin, float* t_rows, int B, int C, int HW, int Cp,
                                    const float* __restrict__ params, int ps, int copies, int cs, int ub) {
  const long first = blockIdx.x * (long)blockDim.x + threadIdx.x;
  if (first < (long)copies * B) {
    const int k = (int)first / B, b = (int)first % B;
    t_rows[k * ub + b * cs] = params[b * ps + 2];
  }
  const long per_row = (long)HW * Cp, total = (long)copies * B * per_row;
  for (long idx = first; idx < total; idx += (long)gridDim.x * blockDim.x) {
    const int c = idx % Cp;
    const long p = (idx / Cp) % HW;
    const int kb = idx / per_row, k = kb / B, b = kb % B;
    const float sigma = params[b * ps];
    const float inv = 1.0f / sqrtf(sigma * sigma + 1.0f);
    // the reference scales in the activation dtype: bf16(latent) / sqrt(sigma^2+1) -> bf16
    xin[((long)(k * ub + b * cs) * HW + p) * Cp + c] =
        c < C ? __float2bfloat16_rn(round_bf16(lat[((long)b * C + c) * HW + p]) * inv) : __float2bfloat16(0.f);
  }
}
int slot_prepare(const float* lat, bf16* xin, float* t_rows, int B, int C, int HW, int Cp, const float* params, int ps,
                 int copies, int cs, int ub, cudaStream_t st) {
  slot_prepare_kernel<<<2 * kNumSMs, 256, 0, st>>>(lat, xin, t_rows, B, C, HW, Cp, params, ps, copies, cs, ub);
  return cudaGetLastError() == cudaSuccess ? EMU_OK : EMU_ERR_CUDA;
}
// noise = uncond + g*(cond - uncond) (cond first, :145-146); latents += noise * (sigma_next - sigma)  (Euler, eps-pred).
// A slot with g <= 1 takes its conditional prediction as it is (forward without CFG has no unconditional row); a slot with
// live[b] == 0 (live NULL: every slot is live) is not written.
__global__ void slot_cfg_euler_kernel(float* lat, const bf16* __restrict__ eps_nhwc, const int* __restrict__ live, int B, int C,
                                      int HW, int ld, const float* __restrict__ params, int ps, int cs, int ub) {
  const long total = (long)B * C * HW;
  for (long idx = blockIdx.x * (long)blockDim.x + threadIdx.x; idx < total; idx += (long)gridDim.x * blockDim.x) {
    const long p = idx % HW;
    const int c = (idx / HW) % C;
    const int b = idx / ((long)HW * C);
    if (live && !live[b]) continue;
    const float* pr = params + b * ps;
    const float dt = pr[1] - pr[0], g = pr[3];
    const float ec = __bfloat162float(eps_nhwc[((long)(b * cs) * HW + p) * ld + c]);
    float e = ec;
    if (g > 1.0f) {
      const float eu = __bfloat162float(eps_nhwc[((long)(ub + b * cs) * HW + p) * ld + c]);
      e = round_bf16(eu + round_bf16(g * round_bf16(ec - eu)));  // bf16 rounding points of the reference expression
    }
    lat[idx] += e * dt;
  }
}
int slot_cfg_euler(float* lat, const bf16* eps_nhwc, const int* live, int B, int C, int HW, int ld, const float* params, int ps,
                   int cs, int ub, cudaStream_t st) {
  slot_cfg_euler_kernel<<<2 * kNumSMs, 256, 0, st>>>(lat, eps_nhwc, live, B, C, HW, ld, params, ps, cs, ub);
  return cudaGetLastError() == cudaSuccess ? EMU_OK : EMU_ERR_CUDA;
}

// CFG combine + one linear-multistep (PNDM / PLMS) update, the scheduler of the Emu1 pipeline (Emu1/models/pipeline.py:112-127
// with diffusers PNDMScheduler, skip_prk_steps):  e = CFG(eps);  m = wc*e + w0*h0 + w1*h1 + w2*h2 (h0 = newest stored eps);
// x_prev = a * x + b * m, where x is the latent or the sample saved at the first step.  params (device, fp32):
// [0] a, [1] b, [2] wc, [3] w0, [4] w1, [5] w2, [6] guidance, [7] flags as float: bit 0 push e into the history,
// bit 1 read x from `saved`, bit 2 store the incoming latent in `saved`.  hist = [3][n] fp32 planes (newest first).
__global__ void cfg_multistep_kernel(float* lat, const bf16* __restrict__ eps_nhwc, float* hist, float* saved, int B, int C,
                                     int HW, int ld, const float* __restrict__ params, int cfg) {
  const float a = params[0], b = params[1], wc = params[2], w0 = params[3], w1 = params[4], w2 = params[5], g = params[6];
  const int flags = (int)params[7];
  const long total = (long)B * C * HW;
  for (long idx = blockIdx.x * (long)blockDim.x + threadIdx.x; idx < total; idx += (long)gridDim.x * blockDim.x) {
    const long p = idx % HW;
    const int c = (idx / HW) % C;
    const int bb = idx / ((long)HW * C);
    const float ec = __bfloat162float(eps_nhwc[((long)bb * HW + p) * ld + c]);
    float e = ec;
    if (cfg) {
      const float eu = __bfloat162float(eps_nhwc[((long)(B + bb) * HW + p) * ld + c]);
      e = round_bf16(eu + round_bf16(g * round_bf16(ec - eu)));  // same rounding points as slot_cfg_euler_kernel
    }
    const float h0 = hist[idx], h1 = hist[total + idx], h2 = hist[2 * total + idx];
    const float m = wc * e + w0 * h0 + w1 * h1 + w2 * h2;
    const float x_in = lat[idx];
    const float x = (flags & 2) ? saved[idx] : x_in;
    if (flags & 4) saved[idx] = x_in;
    if (flags & 1) {
      hist[2 * total + idx] = h1;
      hist[total + idx] = h0;
      hist[idx] = e;
    }
    lat[idx] = a * x + b * m;
  }
}
int cfg_multistep(float* lat, const bf16* eps_nhwc, float* hist, float* saved, int B, int C, int HW, int ld,
                  const float* params, int cfg, cudaStream_t st) {
  cfg_multistep_kernel<<<2 * kNumSMs, 256, 0, st>>>(lat, eps_nhwc, hist, saved, B, C, HW, ld, params, cfg);
  return cudaGetLastError() == cudaSuccess ? EMU_OK : EMU_ERR_CUDA;
}

// mean over tokens: ctx [B, L, C] -> [B, C]   (text_embeds = prompt_embeds.mean(1), Emu2/emu/diffusion.py:113)
__global__ void mean_tokens_kernel(const bf16* __restrict__ x, bf16* y, int L, int C) {
  const int b = blockIdx.x;
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    float s = 0.f;
    for (int l = 0; l < L; ++l) s += __bfloat162float(x[((long)b * L + l) * C + c]);
    y[(long)b * C + c] = __float2bfloat16_rn(s / (float)L);
  }
}
int mean_tokens(const bf16* x, bf16* y, int B, int L, int C, cudaStream_t st) {
  mean_tokens_kernel<<<B, 256, 0, st>>>(x, y, L, C);
  return cudaGetLastError() == cudaSuccess ? EMU_OK : EMU_ERR_CUDA;
}

// row softmax of fp32 scores times `scale` -> bf16 probabilities (VAE mid-block single-head attention, D = 512 > flash tile)
__global__ void __launch_bounds__(256) softmax_rows_kernel(const float* __restrict__ s, bf16* __restrict__ p, int cols,
                                                           float scale) {
  __shared__ float red[33];
  const float* row = s + (long)blockIdx.x * cols;
  bf16* prow = p + (long)blockIdx.x * cols;
  float m = -INFINITY;
  for (int i = threadIdx.x; i < cols; i += blockDim.x) m = fmaxf(m, row[i] * scale);
  m = warp_max(m);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = m;
  __syncthreads();
  m = red[0];
  for (int w = 1; w < 8; ++w) m = fmaxf(m, red[w]);
  __syncthreads();
  float l = 0.f;
  for (int i = threadIdx.x; i < cols; i += blockDim.x) l += __expf(row[i] * scale - m);
  l = block_sum(l, red);
  const float inv = 1.f / l;
  for (int i = threadIdx.x; i < cols; i += blockDim.x) prow[i] = __float2bfloat16_rn(__expf(row[i] * scale - m) * inv);
}
int softmax_rows(const float* s, bf16* p, long rows, int cols, float scale, cudaStream_t st) {
  softmax_rows_kernel<<<(unsigned)rows, 256, 0, st>>>(s, p, cols, scale);
  return cudaGetLastError() == cudaSuccess ? EMU_OK : EMU_ERR_CUDA;
}

// transpose [rows, cols] -> [cols, rows] (bf16), 32x32 smem tiles
__global__ void transpose_kernel(const bf16* __restrict__ x, bf16* y, int rows, int cols) {
  __shared__ bf16 tile[32][33];
  const int bx = blockIdx.x * 32, by = blockIdx.y * 32;
  for (int j = threadIdx.y; j < 32; j += 8)
    if (by + j < rows && bx + threadIdx.x < cols) tile[j][threadIdx.x] = x[(long)(by + j) * cols + bx + threadIdx.x];
  __syncthreads();
  for (int j = threadIdx.y; j < 32; j += 8)
    if (bx + j < cols && by + threadIdx.x < rows) y[(long)(bx + j) * rows + by + threadIdx.x] = tile[threadIdx.x][j];
}
int transpose_2d(const bf16* x, bf16* y, int rows, int cols, cudaStream_t st) {
  transpose_kernel<<<dim3((cols + 31) / 32, (rows + 31) / 32), dim3(32, 8), 0, st>>>(x, y, rows, cols);
  return cudaGetLastError() == cudaSuccess ? EMU_OK : EMU_ERR_CUDA;
}

// image post-process: (x/2 + 0.5).clamp(0,1) -> fp32 NHWC (Emu2/emu/diffusion.py:217-218)
__global__ void vae_post_kernel(const bf16* __restrict__ x, float* y, long n_pix, int C, int ldx) {
  const long total = n_pix * C;
  for (long idx = blockIdx.x * (long)blockDim.x + threadIdx.x; idx < total; idx += (long)gridDim.x * blockDim.x) {
    const int c = idx % C;
    const long p = idx / C;
    const float v = round_bf16(round_bf16(__bfloat162float(x[p * ldx + c]) * 0.5f) + 0.5f);
    y[idx] = fminf(fmaxf(v, 0.f), 1.f);
  }
}
int vae_post(const bf16* x, float* y, long n_pix, int C, int ldx, cudaStream_t st) {
  vae_post_kernel<<<4 * kNumSMs, 256, 0, st>>>(x, y, n_pix, C, ldx);
  return cudaGetLastError() == cudaSuccess ? EMU_OK : EMU_ERR_CUDA;
}

}  // namespace emu
