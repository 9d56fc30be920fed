// Multi-tap wgmma GEMM: the one contraction kernel behind every Linear, 1x1 / 3x3
// (stride 1 or 2) Conv2d and (3,1,1) temporal Conv3d on the denoising hot path.
//
//   out[row, n] = epilogue( sum_{tap} sum_{src} sum_{c} A_src[row + off(tap), c] * W[n, tap, src, c] )
//
// Activations live in HBM channels-last ([..., C] bf16).  "row" is a point of a 4-D output row space (e.g. x, y,
// sample for a conv); a 128-row tile is a 4-D box which TMA fetches as one 5-D box per (tap, 64-channel chunk) with
// hardware zero fill outside the tensor -- implicit-GEMM convolution with no im2col buffer.  Weights are
// [N][taps*K] bf16 (K contiguous).  The box extents multiply to 128, so each is a power of two.
//
// Per CTA (persistent over 128 x BN tiles, warp specialised, 384 threads = 3 warpgroups):
//   warpgroup 0, thread 0   : TMA producer (A box + W tile per k-iteration into a multi-stage shared-memory ring);
//                             it runs ahead into the next tile's ring slots while the current tile is written out
//   warpgroup 0, warps 1-3  : storers (bf16 outputs).  Per tile: wait on `staged`, then read the staged tile, add
//                             row vector / residual / AlphaBlender with their bf16 roundings and write the output with
//                             16-byte loads and stores (element-wise when ca_gemm finds a pointer or stride that is
//                             not 16-byte aligned), skipping rows outside the output box; then arrive on `drained`
//   warpgroups 1, 2         : consumers.  Warpgroup g issues m64nBNk16 wgmma for rows [64g, 64g + 64) of the tile with
//                             both operands read from the 128B-swizzled ring, accumulates in registers, and releases
//                             a ring slot as soon as the wgmma that read it have retired.  After the last k-iteration
//                             they wait on `drained` (the storers have finished the previous tile), add the bias
//                             (copied to shared memory once per tile), round, apply SiLU or GEGLU and the output
//                             scale with their roundings, write bf16 into the staging tile, arrive on `staged` and
//                             go straight on to the next tile's main loop.  Consumers issue no global stores.
// Every rounding is a bf16 rounding of the reference's autocast chain; the order of the steps is that chain's.
// fp32 outputs (VAE attention scores, kernel checks) are a separate instantiation without staging: the consumers write
// them straight from the accumulator registers.
// setmaxnreg moves registers from warpgroup 0 to the consumers (BN = 256: 128 accumulators per thread).
#pragma once
#include "common.cuh"
#include "kernels.h"
#include "wgmma.cuh"

namespace ca {

static constexpr int kBM = 128;
static constexpr int kBK = 64;
static constexpr int kGemmThreads = 384;
static constexpr int kConsumerThreads = 256;  // warpgroups 1, 2
static constexpr int kStorerThreads = 96;     // warps 1-3 of warpgroup 0

enum GemmEpilogue { kEpiBf16 = 0, kEpiGeglu = 1, kEpiF32 = 2 };

template <int BN, int EPI>
struct GemmCfg {
  static constexpr uint32_t kABytes = kBM * kBK * 2;  // 16 KB
  static constexpr uint32_t kBBytes = BN * kBK * 2;   // a multiple of the 1 KB swizzle atom for every BN used
  static constexpr uint32_t kStageBytes = kABytes + kBBytes;
  // bf16 epilogues stage the tile as kBM rows of kOutCols bf16 in 16-byte chunks.  Rows of a multiple of 8 chunks
  // are XOR-swizzled (chunk ^ (row & 7)), other rows are padded by one chunk: either way a consumer store (8 rows x
  // 4 words per warp) and a storer read (8 chunks of one row per quarter warp) hit 32 distinct banks.
  static constexpr bool kStaged = EPI != kEpiF32;
  static constexpr int kOutCols = EPI == kEpiGeglu ? BN / 2 : BN;
  static constexpr int kChunks = kOutCols / 8;
  static constexpr bool kSwizzle = kChunks % 8 == 0;
  static constexpr uint32_t kPitch = kOutCols * 2 + (kSwizzle ? 0 : 16);
  static constexpr uint32_t kStagingBytes = kStaged ? kBM * kPitch : 0;
  static constexpr uint32_t kBiasBytes = kStaged ? BN * 4 : 0;
  // 227 KB per block on H100, minus alignment slack, barriers, staging tile and bias: BN 256 keeps 3 ring stages
  // (4 for GEGLU, whose staging tile is half as wide)
  static constexpr uint32_t kBudget = 232448 - 1024 - 256 - kStagingBytes - kBiasBytes;
  static constexpr int kStagesRaw = kBudget / kStageBytes;
  static constexpr int kStages = kStagesRaw > 8 ? 8 : kStagesRaw;
  static constexpr uint32_t kSmemBytes =
      kStages * kStageBytes + kStagingBytes + kBiasBytes + 1024 /*align slack*/ + 256 /*barriers*/;
  // registers per thread after setmaxnreg: 128 * kWg0Regs + 256 * kConsumerRegs = 384 * 168
  static constexpr int kWg0Regs = kStaged ? 72 : 40;
  static constexpr int kConsumerRegs = kStaged ? 216 : 232;

  __device__ __forceinline__ static uint32_t chunk_off(int row, int chunk) {
    return row * kPitch + ((kSwizzle ? (chunk ^ (row & 7)) : chunk) << 4);
  }
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

// output row r of a tile with origin `org` -> 4-D output point; lb = log2 of the box extents
struct GemmRow {
  bool ok;  // inside odim
  long long out, res, rv;  // element offsets of the row in out, residual / blend_src, rowvec
};
__device__ __forceinline__ GemmRow gemm_row(const GemmParams& p, const int (&org)[4], const int (&lb)[4], int r) {
  int o[4];
  o[0] = org[0] + (r & (p.box[0] - 1)); r >>= lb[0];
  o[1] = org[1] + (r & (p.box[1] - 1)); r >>= lb[1];
  o[2] = org[2] + (r & (p.box[2] - 1)); r >>= lb[2];
  o[3] = org[3] + r;
  GemmRow g;
  g.ok = o[0] < p.odim[0] && o[1] < p.odim[1] && o[2] < p.odim[2] && o[3] < p.odim[3];
  g.out = o[0] * p.ostride[0] + o[1] * p.ostride[1] + o[2] * p.ostride[2] + o[3] * p.ostride[3];
  g.res = o[0] * p.rstride[0] + o[1] * p.rstride[1] + o[2] * p.rstride[2] + o[3] * p.rstride[3];
  g.rv = o[0] * p.vstride[0] + o[1] * p.vstride[1] + o[2] * p.vstride[2] + o[3] * p.vstride[3];
  return g;
}

// 8 bf16 of global memory: one 16-byte access when kVec, else eight 2-byte ones
template <bool kVec>
__device__ __forceinline__ uint4 ld8_bf16(const __nv_bfloat16* g) {
  if constexpr (kVec) {
    return *reinterpret_cast<const uint4*>(g);
  } else {
    const unsigned short* h = reinterpret_cast<const unsigned short*>(g);
    return make_uint4(h[0] | (uint32_t(h[1]) << 16), h[2] | (uint32_t(h[3]) << 16), h[4] | (uint32_t(h[5]) << 16),
                      h[6] | (uint32_t(h[7]) << 16));
  }
}
template <bool kVec>
__device__ __forceinline__ void st8_bf16(__nv_bfloat16* g, uint4 v) {
  if constexpr (kVec) {
    *reinterpret_cast<uint4*>(g) = v;
  } else {
    unsigned short* h = reinterpret_cast<unsigned short*>(g);
    const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      h[2 * i] = static_cast<unsigned short>(w[i] & 0xffffu);
      h[2 * i + 1] = static_cast<unsigned short>(w[i] >> 16);
    }
  }
}

// the storer's part of the chain on one bf16 pair: row vector, residual, AlphaBlender, each rounded to bf16
__device__ __forceinline__ uint32_t gemm_finish_word(uint32_t v, bool rv_on, uint32_t rv, bool res_on, uint32_t rs,
                                                     bool blend_on, uint32_t bs, float alpha_s, float alpha_t) {
  float v0 = bf16lo_to_float(v), v1 = bf16hi_to_float(v);
  if (rv_on) {
    v0 += bf16lo_to_float(rv);
    v1 += bf16hi_to_float(rv);
    round2_bf16(v0, v1);
  }
  if (res_on) {
    v0 += bf16lo_to_float(rs);
    v1 += bf16hi_to_float(rs);
    round2_bf16(v0, v1);
  }
  if (blend_on) {
    float s0 = alpha_s * bf16lo_to_float(bs), s1 = alpha_s * bf16hi_to_float(bs);
    float t0 = alpha_t * v0, t1 = alpha_t * v1;
    round2_bf16(s0, s1);
    round2_bf16(t0, t1);
    v0 = s0 + t0;
    v1 = s1 + t1;
  }
  return pack_bf16x2(v0, v1);
}

// Storers: write one staged tile.  Thread s takes chunks s, s + 96, ... (row-major over 16-byte chunks, so a warp
// covers whole rows).  kVec: every source is 16-byte aligned, and kRv / kRes / kBlend say which exist; otherwise
// (element-wise path) the flags are read from p.
template <class Cfg, bool kVec, bool kRv, bool kRes, bool kBlend>
__device__ __forceinline__ void gemm_drain_tile(const GemmParams& p, const uint8_t* staging, int tn,
                                                const int (&org)[4], const int (&lb)[4], int s, float alpha_s,
                                                float alpha_t) {
  const bool rv_on = kVec ? kRv : p.rowvec != nullptr;
  const bool res_on = kVec ? kRes : p.residual != nullptr;
  const bool blend_on = kVec ? kBlend : p.blend_src != nullptr;
  __nv_bfloat16* out = static_cast<__nv_bfloat16*>(p.out);
  const int col0 = tn * Cfg::kOutCols;
  for (int q = s; q < kBM * Cfg::kChunks; q += kStorerThreads) {
    const int r = q / Cfg::kChunks, c = q % Cfg::kChunks, col = col0 + 8 * c;
    const GemmRow g = gemm_row(p, org, lb, r);
    if (!g.ok || col >= p.n_out) continue;
    uint4 rv, rs, bs;
    if (rv_on) rv = ld8_bf16<kVec>(p.rowvec + g.rv + col);
    if (res_on) rs = ld8_bf16<kVec>(p.residual + g.res + col);
    if (blend_on) bs = ld8_bf16<kVec>(p.blend_src + g.res + col);
    uint4 v = *reinterpret_cast<const uint4*>(staging + Cfg::chunk_off(r, c));
    if (rv_on || res_on || blend_on) {
      v.x = gemm_finish_word(v.x, rv_on, rv.x, res_on, rs.x, blend_on, bs.x, alpha_s, alpha_t);
      v.y = gemm_finish_word(v.y, rv_on, rv.y, res_on, rs.y, blend_on, bs.y, alpha_s, alpha_t);
      v.z = gemm_finish_word(v.z, rv_on, rv.z, res_on, rs.z, blend_on, bs.z, alpha_s, alpha_t);
      v.w = gemm_finish_word(v.w, rv_on, rv.w, res_on, rs.w, blend_on, bs.w, alpha_s, alpha_t);
    }
    st8_bf16<kVec>(out + g.out + col, v);
  }
}

// fp32 output, straight from the accumulators.  Thread holds rows (r0, r0 + 8) x columns 8 j + 2 (lane & 3) + {0, 1}.
// Rounded to bf16 only where the reference's chain is bf16: after SiLU and after the row vector.
template <int BN>
__device__ __forceinline__ void gemm_epilogue_f32(const GemmParams& p, const float (&acc)[BN / 2], int tn,
                                                  const int (&org)[4], int r0, int lane) {
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    int rr = r0 + 8 * h;
    const int i1 = rr % p.box[0]; rr /= p.box[0];
    const int i2 = rr % p.box[1]; rr /= p.box[1];
    const int i3 = rr % p.box[2]; rr /= p.box[2];
    const int o[4] = {org[0] + i1, org[1] + i2, org[2] + i3, org[3] + rr};
    if (!(o[0] < p.odim[0] && o[1] < p.odim[1] && o[2] < p.odim[2] && o[3] < p.odim[3])) continue;
    float* op = reinterpret_cast<float*>(p.out) +
                (o[0] * p.ostride[0] + o[1] * p.ostride[1] + o[2] * p.ostride[2] + o[3] * p.ostride[3]);
    const long long res_off = o[0] * p.rstride[0] + o[1] * p.rstride[1] + o[2] * p.rstride[2] + o[3] * p.rstride[3];
    const long long rv_off = o[0] * p.vstride[0] + o[1] * p.vstride[1] + o[2] * p.vstride[2] + o[3] * p.vstride[3];
#pragma unroll
    for (int j = 0; j < BN / 8; ++j) {
      const int col = tn * BN + 8 * j + 2 * (lane & 3);
      if (col >= p.n_out) continue;
      const int nv = min(2, p.n_out - col);
      float v0 = acc[4 * j + 2 * h], v1 = acc[4 * j + 2 * h + 1];
      if (p.bias != nullptr) {
        v0 += __ldg(p.bias + col);
        v1 += __ldg(p.bias + min(col + 1, p.n_out - 1));
      }
      if (p.act == CA_ACT_SILU) {
        v0 = __fdividef(v0, 1.0f + __expf(-v0));
        v1 = __fdividef(v1, 1.0f + __expf(-v1));
        round2_bf16(v0, v1);
      }
      if (p.out_scale != 1.0f) {
        v0 *= p.out_scale;
        v1 *= p.out_scale;
      }
      if (p.rowvec != nullptr) {
        v0 = round_bf16(v0 + __bfloat162float(p.rowvec[rv_off + col]));
        if (nv > 1) v1 = round_bf16(v1 + __bfloat162float(p.rowvec[rv_off + col + 1]));
      }
      if (p.residual != nullptr) {
        v0 += __bfloat162float(p.residual[res_off + col]);
        if (nv > 1) v1 += __bfloat162float(p.residual[res_off + col + 1]);
      }
      op[col] = v0;
      if (nv > 1) op[col + 1] = v1;
    }
  }
}

// Consumers, bf16 outputs: bias (from shared memory), rounding, activation and output scale of the thread's
// accumulators into the staging tile.  Adding -0.0 is exact for every value, so a missing bias is a bias of -0.0.
// Scaling a bf16-valued number by 1.0 and rounding it again is exact as well, so the scale is always applied.
template <class Cfg, int BN, bool kSilu>
__device__ __forceinline__ void gemm_stage_tile(const GemmParams& p, const float (&acc)[BN / 2], const float* bias_s,
                                                uint8_t* staging, int r0, int lane) {
  const int q = lane & 3;
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int r = r0 + 8 * h;
    if constexpr (Cfg::kOutCols == BN) {
#pragma unroll
      for (int j = 0; j < BN / 8; ++j) {
        const float2 b = *reinterpret_cast<const float2*>(bias_s + 8 * j + 2 * q);
        float v0 = acc[4 * j + 2 * h] + b.x, v1 = acc[4 * j + 2 * h + 1] + b.y;
        round2_bf16(v0, v1);
        if constexpr (kSilu) {
          v0 = __fdividef(v0, 1.0f + __expf(-v0));
          v1 = __fdividef(v1, 1.0f + __expf(-v1));
          round2_bf16(v0, v1);
        }
        v0 *= p.out_scale;
        v1 *= p.out_scale;
        *reinterpret_cast<uint32_t*>(staging + Cfg::chunk_off(r, j) + 4 * q) = pack_bf16x2(v0, v1);
      }
    } else {
      // GEGLU: weight rows of tile tn are [value rows of BN/2 output columns][the matching gate rows]
#pragma unroll
      for (int j = 0; j < BN / 16; ++j) {
        const float2 ba = *reinterpret_cast<const float2*>(bias_s + 8 * j + 2 * q);
        const float2 bg = *reinterpret_cast<const float2*>(bias_s + BN / 2 + 8 * j + 2 * q);
        float a0 = acc[4 * j + 2 * h] + ba.x, a1 = acc[4 * j + 2 * h + 1] + ba.y;
        float g0 = acc[4 * (j + BN / 16) + 2 * h] + bg.x, g1 = acc[4 * (j + BN / 16) + 2 * h + 1] + bg.y;
        round2_bf16(a0, a1);
        round2_bf16(g0, g1);
        float l0 = gelu_erf(g0), l1 = gelu_erf(g1);
        round2_bf16(l0, l1);
        float v0 = a0 * l0, v1 = a1 * l1;
        round2_bf16(v0, v1);
        v0 *= p.out_scale;
        v1 *= p.out_scale;
        *reinterpret_cast<uint32_t*>(staging + Cfg::chunk_off(r, j) + 4 * q) = pack_bf16x2(v0, v1);
      }
    }
  }
}

template <int BN, int EPI>
__global__ void __launch_bounds__(kGemmThreads, 1)
gemm_conv_kernel(const __grid_constant__ CUtensorMap tmap_a0, const __grid_constant__ CUtensorMap tmap_a1,
                 const __grid_constant__ CUtensorMap tmap_w, const GemmParams p) {
  using Cfg = GemmCfg<BN, EPI>;
  CA_PDL_TRIGGER();
  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw_addr = smem_u32(smem_raw);
  uint8_t* smem = smem_raw + ((1024u - (raw_addr & 1023u)) & 1023u);

  uint8_t* smem_a = smem;                                       // kStages x 16 KB
  uint8_t* smem_b = smem + Cfg::kStages * Cfg::kABytes;         // kStages x BN*128 B
  uint8_t* staging = smem + Cfg::kStages * Cfg::kStageBytes;    // kBM x kPitch B (bf16 outputs)
  float* bias_s = reinterpret_cast<float*>(staging + Cfg::kStagingBytes);  // [BN] (bf16 outputs)
  uint64_t* bars = reinterpret_cast<uint64_t*>(staging + Cfg::kStagingBytes + Cfg::kBiasBytes);
  uint64_t* full_bar = bars;                        // [kStages]
  uint64_t* empty_bar = bars + Cfg::kStages;        // [kStages]
  uint64_t* staged_bar = bars + 2 * Cfg::kStages;   // consumers -> storers: the staging tile holds tile i
  uint64_t* drained_bar = staged_bar + 1;           // storers -> consumers: the staging tile may be overwritten

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
    mbar_init(staged_bar, kConsumerThreads);
    mbar_init(drained_bar, kStorerThreads);
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
    setmaxnreg_dec<Cfg::kWg0Regs>();
    if (threadIdx.x == 0) {
      // ===================== TMA producer =====================
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
    } else if (Cfg::kStaged && warp > 0) {
      // ===================== storers =====================
      const int s = threadIdx.x - 32;
      float alpha_s = 0.f, alpha_t = 0.f;
      if (p.blend_src != nullptr) {
        const float a = *p.blend_alpha;  // bf16-valued
        alpha_s = a;
        alpha_t = round_bf16(1.0f - a);
      }
      const int lb[4] = {__ffs(p.box[0]) - 1, __ffs(p.box[1]) - 1, __ffs(p.box[2]) - 1, __ffs(p.box[3]) - 1};
      const int kind = (p.rowvec != nullptr ? 1 : 0) | (p.residual != nullptr ? 2 : 0) | (p.blend_src != nullptr ? 4 : 0);
      uint32_t phase = 0;
      for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
        int tn, org[4];
        tile_coords(tile, tn, org);
        mbar_wait(staged_bar, phase);
        if (!p.vec_ok) {
          gemm_drain_tile<Cfg, false, false, false, false>(p, staging, tn, org, lb, s, alpha_s, alpha_t);
        } else {
          switch (kind) {
            case 0: gemm_drain_tile<Cfg, true, false, false, false>(p, staging, tn, org, lb, s, alpha_s, alpha_t); break;
            case 1: gemm_drain_tile<Cfg, true, true, false, false>(p, staging, tn, org, lb, s, alpha_s, alpha_t); break;
            case 2: gemm_drain_tile<Cfg, true, false, true, false>(p, staging, tn, org, lb, s, alpha_s, alpha_t); break;
            case 3: gemm_drain_tile<Cfg, true, true, true, false>(p, staging, tn, org, lb, s, alpha_s, alpha_t); break;
            case 4: gemm_drain_tile<Cfg, true, false, false, true>(p, staging, tn, org, lb, s, alpha_s, alpha_t); break;
            case 5: gemm_drain_tile<Cfg, true, true, false, true>(p, staging, tn, org, lb, s, alpha_s, alpha_t); break;
            case 6: gemm_drain_tile<Cfg, true, false, true, true>(p, staging, tn, org, lb, s, alpha_s, alpha_t); break;
            default: gemm_drain_tile<Cfg, true, true, true, true>(p, staging, tn, org, lb, s, alpha_s, alpha_t); break;
          }
        }
        mbar_arrive(drained_bar);
        phase ^= 1;
      }
    }
    return;
  }

  // ===================== consumers: wgmma main loop + epilogue =====================
  setmaxnreg_inc<Cfg::kConsumerRegs>();
  const int cw = (warp >> 2) - 1;   // consumer warpgroup: tile rows [64 cw, 64 cw + 64)
  const int wq = warp & 3;          // warp inside the warpgroup: rows [16 wq, 16 wq + 16) of those
  const int ct = threadIdx.x - 128; // consumer thread 0..255
  const int r0 = cw * 64 + wq * 16 + (lane >> 2);  // the thread's accumulator rows are r0 and r0 + 8
  float acc[BN / 2];
  int stage = 0;
  uint32_t phase = 0, staged_phase = 0;
  for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
    int tn, org[4];
    tile_coords(tile, tn, org);
    // this thread's bias value of the tile, loaded now so that its latency hides behind the main loop
    float bias_v = -0.0f;
    if (Cfg::kStaged && p.bias != nullptr && ct < BN && (EPI == kEpiGeglu || tn * BN + ct < p.n_out))
      bias_v = __ldg(p.bias + tn * BN + ct);
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

    if constexpr (Cfg::kStaged) {
      mbar_wait(drained_bar, staged_phase ^ 1);  // the storers are done with the previous tile (and its bias)
      if (ct < BN) bias_s[ct] = bias_v;
      named_bar_sync(1, kConsumerThreads);
      if (EPI == kEpiBf16 && p.act == CA_ACT_SILU)
        gemm_stage_tile<Cfg, BN, true>(p, acc, bias_s, staging, r0, lane);
      else
        gemm_stage_tile<Cfg, BN, false>(p, acc, bias_s, staging, r0, lane);
      mbar_arrive(staged_bar);
      staged_phase ^= 1;
    } else {
      gemm_epilogue_f32<BN>(p, acc, tn, org, r0, lane);
    }
  }
}

template <int BN, int EPI>
static cudaError_t launch_epi(const CUtensorMap& a0, const CUtensorMap& a1, const CUtensorMap& w, const GemmParams& p,
                              int grid, cudaStream_t stream) {
  using Cfg = GemmCfg<BN, EPI>;
  static bool attr_set = false;
  auto kern = gemm_conv_kernel<BN, EPI>;
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         static_cast<int>(Cfg::kSmemBytes));
    if (e != cudaSuccess) return e;
    attr_set = true;
  }
  return launch_pdl(kern, grid, kGemmThreads, Cfg::kSmemBytes, stream, a0, a1, w, p);
}

// one translation unit per BN (gemm_conv_bn*.cu) instantiates its kernels through this
template <int BN>
static cudaError_t launch_bn(const CUtensorMap& a0, const CUtensorMap& a1, const CUtensorMap& w, const GemmParams& p,
                             int grid, cudaStream_t stream) {
  if (p.out_fp32) return launch_epi<BN, kEpiF32>(a0, a1, w, p, grid, stream);
  if (p.act == CA_ACT_GEGLU) return launch_epi<BN, kEpiGeglu>(a0, a1, w, p, grid, stream);
  return launch_epi<BN, kEpiBf16>(a0, a1, w, p, grid, stream);
}

}  // namespace ca
