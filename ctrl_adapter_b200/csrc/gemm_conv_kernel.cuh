// Multi-tap wgmma GEMM: the one contraction kernel behind every Linear, 1x1 / 3x3
// (stride 1 or 2) Conv2d and (3,1,1) temporal Conv3d on the denoising hot path.
//
//   out[row, n] = epilogue( sum_{tap} sum_{src} sum_{c} A_src[row + off(tap), c] * W[n, tap, src, c] )
//
// Activations live in HBM channels-last ([..., C] bf16).  "row" is a point of a 4-D output row space (e.g. x, y,
// sample for a conv); a 128-row tile is a 4-D box which TMA fetches as one 5-D box per (tap, 64-channel chunk) with
// hardware zero fill outside the tensor -- implicit-GEMM convolution with no im2col buffer.  Weights are
// [N][taps*K] bf16 (K contiguous).
//
// Per CTA (persistent over 128 x BN tiles, warp specialised, 384 threads = 3 warpgroups):
//   warpgroup 0, one thread : TMA producer (A box + W tile per k-iteration into a multi-stage shared-memory ring)
//   warpgroups 1, 2         : consumers.  Warpgroup g issues m64nBNk16 wgmma for rows [64g, 64g + 64) of the tile with
//                             both operands read from the 128B-swizzled ring, accumulates in registers, and releases
//                             a ring slot as soon as the wgmma that read it have retired.  Then the epilogue straight
//                             from the accumulator registers: bias / SiLU / GEGLU / scale / row vector / residual /
//                             AlphaBlender / fp32 output, with a bf16 rounding after each step (the autocast rounding
//                             points of the reference).
// setmaxnreg moves registers from the producer warpgroup to the consumers (BN = 256: 128 accumulators per thread).
#pragma once
#include "common.cuh"
#include "kernels.h"
#include "wgmma.cuh"

namespace ca {

static constexpr int kBM = 128;
static constexpr int kBK = 64;
static constexpr int kGemmThreads = 384;

template <int BN>
struct GemmCfg {
  static constexpr uint32_t kABytes = kBM * kBK * 2;  // 16 KB
  static constexpr uint32_t kBBytes = BN * kBK * 2;   // a multiple of the 1 KB swizzle atom for every BN used
  static constexpr uint32_t kStageBytes = kABytes + kBBytes;
  static constexpr uint32_t kBudget = 232448 - 1024 - 256;  // 227 KB per block on H100, minus alignment and barriers
  static constexpr int kStagesRaw = kBudget / kStageBytes;
  static constexpr int kStages = kStagesRaw > 8 ? 8 : kStagesRaw;
  static constexpr uint32_t kSmemBytes = kStages * kStageBytes + 1024 /*align slack*/ + 256 /*barriers*/;
};

// exact-erf GELU of a bf16-valued x (erf of Abramowitz & Stegun 7.1.26, |error| <= 1.5e-7), arranged as
// relu(x) - |x| * q(|x|) with q = 0.5 * erfc(|x| / sqrt 2): no cancellation for negative x, no branches
__device__ __forceinline__ float gelu_erf(float x) {
  const float a = fabsf(x);
  float t;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(t) : "f"(fmaf(0.3275911f * 0.70710678118654752440f, a, 1.0f)));
  float p = fmaf(0.5f * 1.061405429f, t, 0.5f * -1.453152027f);
  p = fmaf(p, t, 0.5f * 1.421413741f);
  p = fmaf(p, t, 0.5f * -0.284496736f);
  p = fmaf(p, t, 0.5f * 0.254829592f);
  float e;
  const float arg = (a * a) * (-0.5f * 1.4426950408889634f);
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(arg));
  const float q = (p * t) * e;
  return fmaf(-a, q, fmaxf(x, 0.0f));
}

// the epilogue after bias / activation of two adjacent columns (col, col + 1) of one row; `nv` of them exist
__device__ __forceinline__ void gemm_finish_pair(const GemmParams& p, float v0, float v1, int col, int nv,
                                                 long long out_off, long long res_off, long long rv_off,
                                                 float alpha_s, float alpha_t) {
  if (p.out_scale != 1.0f) {
    v0 *= p.out_scale;
    v1 *= p.out_scale;
    if (!p.out_fp32) round2_bf16(v0, v1);  // fp32 output (attention scores of the VAE): unrounded
  }
  if (p.rowvec != nullptr) {
    const __nv_bfloat16* rv = p.rowvec + rv_off + col;
    v0 = round_bf16(v0 + __bfloat162float(rv[0]));
    if (nv > 1) v1 = round_bf16(v1 + __bfloat162float(rv[1]));
  }
  if (p.out_fp32) {
    float* op = reinterpret_cast<float*>(p.out) + out_off + col;
    if (p.residual != nullptr) {
      v0 += __bfloat162float(p.residual[res_off + col]);
      if (nv > 1) v1 += __bfloat162float(p.residual[res_off + col + 1]);
    }
    op[0] = v0;
    if (nv > 1) op[1] = v1;
    return;
  }
  if (p.residual != nullptr) {
    const __nv_bfloat16* rs = p.residual + res_off + col;
    v0 += __bfloat162float(rs[0]);
    v1 += __bfloat162float(rs[1]);
    round2_bf16(v0, v1);
  }
  if (p.blend_src != nullptr) {
    const __nv_bfloat16* bs = p.blend_src + res_off + col;
    v0 = round_bf16(round_bf16(alpha_s * __bfloat162float(bs[0])) + round_bf16(alpha_t * v0));
    v1 = round_bf16(round_bf16(alpha_s * __bfloat162float(bs[1])) + round_bf16(alpha_t * v1));
  }
  __nv_bfloat16* op = reinterpret_cast<__nv_bfloat16*>(p.out) + out_off + col;
  if ((reinterpret_cast<uintptr_t>(op) & 3) == 0) {
    *reinterpret_cast<uint32_t*>(op) = pack_bf16x2(v0, v1);
  } else {
    op[0] = __float2bfloat16_rn(v0);
    op[1] = __float2bfloat16_rn(v1);
  }
}

template <int BN>
__global__ void __launch_bounds__(kGemmThreads, 1)
gemm_conv_kernel(const __grid_constant__ CUtensorMap tmap_a0, const __grid_constant__ CUtensorMap tmap_a1,
                 const __grid_constant__ CUtensorMap tmap_w, const GemmParams p) {
  using Cfg = GemmCfg<BN>;
  CA_PDL_TRIGGER();
  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw_addr = smem_u32(smem_raw);
  uint8_t* smem = smem_raw + ((1024u - (raw_addr & 1023u)) & 1023u);

  uint8_t* smem_a = smem;                                // kStages x 16 KB
  uint8_t* smem_b = smem + Cfg::kStages * Cfg::kABytes;  // kStages x BN*128 B
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + Cfg::kStages * Cfg::kStageBytes);
  uint64_t* full_bar = bars;                  // [kStages]
  uint64_t* empty_bar = bars + Cfg::kStages;  // [kStages]

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;

  const int tiles_m = p.ntile[0] * p.ntile[1] * p.ntile[2] * p.ntile[3];
  const int total_tiles = tiles_m * p.n_tiles_n;
  const int chunks0 = (p.src_c[0] + kBK - 1) / kBK;
  const int chunks1 = (p.nsrc > 1) ? (p.src_c[1] + kBK - 1) / kBK : 0;
  const int kiters = p.ntaps * (chunks0 + chunks1);

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmap_a0);
    if (p.nsrc > 1) tma_prefetch_desc(&tmap_a1);
    tma_prefetch_desc(&tmap_w);
    for (int s = 0; s < Cfg::kStages; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], 8);  // one arrive per consumer warp
    }
    fence_mbar_init();
  }
  __syncthreads();
  CA_PDL_WAIT();  // prologue done: the previous kernel's output (A, residual, bias ...) may be read from here on

  // decode tile -> (n tile, 4-D M tile origin)
  auto tile_coords = [&](int tile, int& tn, int (&org)[4]) {
    tn = tile % p.n_tiles_n;
    int tm = tile / p.n_tiles_n;
    org[0] = (tm % p.ntile[0]) * p.box[0]; tm /= p.ntile[0];
    org[1] = (tm % p.ntile[1]) * p.box[1]; tm /= p.ntile[1];
    org[2] = (tm % p.ntile[2]) * p.box[2]; tm /= p.ntile[2];
    org[3] = tm * p.box[3];
  };

  if (warp < 4) {
    // ===================== TMA producer =====================
    setmaxnreg_dec<40>();
    if (threadIdx.x == 0) {
      int stage = 0;
      uint32_t phase = 0;
      for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
        int tn, org[4];
        tile_coords(tile, tn, org);
        const int n0 = tn * BN;
        for (int tap = 0; tap < p.ntaps; ++tap) {
          const int c1 = org[0] + p.tap_off[tap][0], c2 = org[1] + p.tap_off[tap][1];
          const int c3 = org[2] + p.tap_off[tap][2], c4 = org[3] + p.tap_off[tap][3];
          const int kbase = tap * p.k_per_tap;
          for (int ch = 0; ch < chunks0 + chunks1; ++ch) {
            mbar_wait(&empty_bar[stage], phase ^ 1);
            const bool second = ch >= chunks0;
            const int cc = (second ? (ch - chunks0) : ch) * kBK;
            const int ca = cc + (second ? p.src_c0_off[1] : p.src_c0_off[0]) + p.tap_c_off[tap];
            const int kw = kbase + (second ? p.src_c[0] : 0) + cc;
            const CUtensorMap* ta = second ? &tmap_a1 : &tmap_a0;
            mbar_arrive_expect_tx(&full_bar[stage], Cfg::kStageBytes);
            tma_load_5d(smem_a + stage * Cfg::kABytes, ta, &full_bar[stage], ca, c1, c2, c3, c4);
            tma_load_2d(smem_b + stage * Cfg::kBBytes, &tmap_w, &full_bar[stage], kw, n0);
            if (++stage == Cfg::kStages) { stage = 0; phase ^= 1; }
          }
        }
      }
    }
    return;
  }

  // ===================== consumers: wgmma main loop + register epilogue =====================
  setmaxnreg_inc<232>();
  const int cw = (warp >> 2) - 1;   // consumer warpgroup: tile rows [64 cw, 64 cw + 64)
  const int wq = warp & 3;          // warp inside the warpgroup: rows [16 wq, 16 wq + 16) of those
  const bool geglu = (p.act == CA_ACT_GEGLU);
  float alpha_s = 0.f, alpha_t = 0.f;
  if (p.blend_src != nullptr) {
    const float a = *p.blend_alpha;  // bf16-valued
    alpha_s = a;
    alpha_t = round_bf16(1.0f - a);
  }
  float acc[BN / 2];
  int stage = 0;
  uint32_t phase = 0;
  for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
    int tn, org[4];
    tile_coords(tile, tn, org);
    int prev = -1;
    for (int it = 0; it < kiters; ++it) {
      mbar_wait(&full_bar[stage], phase);
      const uint32_t a_addr = smem_u32(smem_a + stage * Cfg::kABytes) + cw * 64 * 128;
      const uint32_t b_addr = smem_u32(smem_b + stage * Cfg::kBBytes);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < kBK / 16; ++k) {
        Wgmma<BN>::ss(acc, gmma_desc_sw128(a_addr + k * 32, 16, 1024), gmma_desc_sw128(b_addr + k * 32, 16, 1024),
                      (it | k) != 0 ? 1 : 0);
      }
      wgmma_commit();
      if (prev >= 0) {
        wgmma_wait<1>();  // the wgmma of the previous k-iteration retired: its ring slot may be refilled
        if (lane == 0) mbar_arrive(&empty_bar[prev]);
      }
      prev = stage;
      if (++stage == Cfg::kStages) { stage = 0; phase ^= 1; }
    }
    wgmma_wait<0>();
    reg_fence(acc);
    if (lane == 0) mbar_arrive(&empty_bar[prev]);

    // ---- epilogue: thread holds rows (r0, r0 + 8) x columns 8 j + 2 (lane & 3) + {0, 1} ----
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      int rr = cw * 64 + wq * 16 + (lane >> 2) + 8 * h;
      const int i1 = rr % p.box[0]; rr /= p.box[0];
      const int i2 = rr % p.box[1]; rr /= p.box[1];
      const int i3 = rr % p.box[2]; rr /= p.box[2];
      const int i4 = rr;
      const int o[4] = {org[0] + i1, org[1] + i2, org[2] + i3, org[3] + i4};
      const bool row_ok = o[0] < p.odim[0] && o[1] < p.odim[1] && o[2] < p.odim[2] && o[3] < p.odim[3];
      if (!row_ok) continue;
      const long long out_off = o[0] * p.ostride[0] + o[1] * p.ostride[1] + o[2] * p.ostride[2] + o[3] * p.ostride[3];
      const long long res_off = o[0] * p.rstride[0] + o[1] * p.rstride[1] + o[2] * p.rstride[2] + o[3] * p.rstride[3];
      const long long rv_off = (p.rowvec != nullptr)
                                   ? (o[0] * p.vstride[0] + o[1] * p.vstride[1] + o[2] * p.vstride[2] + o[3] * p.vstride[3])
                                   : 0;
      if (geglu) {
        // weight rows of tile tn: [value rows of BN/2 output columns][the matching gate rows]
#pragma unroll
        for (int j = 0; j < BN / 16; ++j) {
          const int c = 8 * j + 2 * (lane & 3);
          const int col = tn * (BN / 2) + c;
          if (col >= p.n_out) continue;  // n_out is a multiple of 8: both columns of the pair exist
          float a0 = acc[4 * j + 2 * h], a1 = acc[4 * j + 2 * h + 1];
          float g0 = acc[4 * (j + BN / 16) + 2 * h], g1 = acc[4 * (j + BN / 16) + 2 * h + 1];
          if (p.bias != nullptr) {
            const float2 ba = __ldg(reinterpret_cast<const float2*>(p.bias + tn * BN + c));
            const float2 bg = __ldg(reinterpret_cast<const float2*>(p.bias + tn * BN + BN / 2 + c));
            a0 += ba.x; a1 += ba.y; g0 += bg.x; g1 += bg.y;
          }
          round2_bf16(a0, a1);
          round2_bf16(g0, g1);
          float l0 = gelu_erf(g0), l1 = gelu_erf(g1);
          round2_bf16(l0, l1);
          float r0 = a0 * l0, r1 = a1 * l1;
          round2_bf16(r0, r1);
          gemm_finish_pair(p, r0, r1, col, 2, out_off, res_off, rv_off, alpha_s, alpha_t);
        }
      } else {
#pragma unroll
        for (int j = 0; j < BN / 8; ++j) {
          const int c = 8 * j + 2 * (lane & 3);
          const int col = tn * BN + c;
          if (col >= p.n_out) continue;
          const int nv = min(2, p.n_out - col);
          float v0 = acc[4 * j + 2 * h], v1 = acc[4 * j + 2 * h + 1];
          if (p.bias != nullptr) {
            v0 += __ldg(p.bias + col);
            v1 += __ldg(p.bias + min(col + 1, p.n_out - 1));
          }
          if (!p.out_fp32) round2_bf16(v0, v1);
          if (p.act == CA_ACT_SILU) {
            v0 = __fdividef(v0, 1.0f + __expf(-v0));
            v1 = __fdividef(v1, 1.0f + __expf(-v1));
            round2_bf16(v0, v1);
          }
          gemm_finish_pair(p, v0, v1, col, nv, out_off, res_off, rv_off, alpha_s, alpha_t);
        }
      }
    }
  }
}

// one translation unit per BN (gemm_conv_bn*.cu) instantiates its kernel through this
template <int BN>
static cudaError_t launch_bn(const CUtensorMap& a0, const CUtensorMap& a1, const CUtensorMap& w, const GemmParams& p,
                             int grid, cudaStream_t stream) {
  using Cfg = GemmCfg<BN>;
  static bool attr_set = false;
  auto kern = gemm_conv_kernel<BN>;
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         static_cast<int>(Cfg::kSmemBytes));
    if (e != cudaSuccess) return e;
    attr_set = true;
  }
  CA_KERNEL_LAUNCH(kern, grid, kGemmThreads, Cfg::kSmemBytes, stream, a0, a1, w, p);
  return cudaGetLastError();
}

}  // namespace ca
