// Temporal self-attention of the video adapters / UNets on the tensor cores: the sequence is the F <= 32 frames of one
// pixel (head dim 64), so one (pixel, head) problem is a 16 x 16 (or 32 x 32) score matrix -- far below a wgmma tile.
// A CTA therefore batches G = 128 / SEQ pixels of one (clip, head) into ONE 128-row tile:
//
//   TMA: the tensor map orders the global dims as (channel, FRAME, PIXEL, clip) -- strides are free, so the box
//        (64, SEQ, G, 1) lands in shared memory as rows (pixel g, frame f): each pixel's sequence is a contiguous block of
//        SEQ rows (frames >= F and pixels >= hw are zero-filled by the TMA unit).
//   MMA: SEQ divides 64, so no sequence straddles a 64-row half.  For each half, S = Q K^T as one m64n64k64 wgmma; only
//        the diagonal SEQ x SEQ blocks are meaningful, the others are masked.
//   softmax in registers (fp32 scores and row sum, P rounded to bf16), then O = P V as m64n64k64 with P from registers
//        and V read MN-major from shared memory; epilogue O / l -> global.
// One warpgroup per CTA (128 threads, 48 KB of shared memory), so several CTAs share an SM and one CTA's loads overlap
// another's MMAs.
#include "common.cuh"
#include "kernels.h"
#include "wgmma.cuh"

namespace ca {

static constexpr int kTaThreads = 128;
static constexpr uint32_t kTaTile = 128 * 64 * 2;  // one [128 rows x 64 dims] bf16 tile = 16 KB
static constexpr uint32_t kTaSmem = 3 * kTaTile + 1024 /*align slack*/ + 64 /*barrier*/;

struct TemporalAttnParams {
  int clips, frames, heads;
  long long hw;
  float scale_log2;            // softmax scale * log2(e)
  __nv_bfloat16* out;          // rows ((clip * frames + f) * hw + pixel), heads * 64 used columns
  long long out_row_stride;    // elements
};

template <int SEQ>
__global__ void __launch_bounds__(kTaThreads)
temporal_attention_tc_kernel(const __grid_constant__ CUtensorMap tmap_q, const __grid_constant__ CUtensorMap tmap_k,
                             const __grid_constant__ CUtensorMap tmap_v, const TemporalAttnParams p) {
  constexpr int G = 128 / SEQ;  // pixels per tile
  CA_PDL_TRIGGER();
  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw_addr = smem_u32(smem_raw);
  uint8_t* smem = smem_raw + ((1024u - (raw_addr & 1023u)) & 1023u);
  uint64_t* bar = reinterpret_cast<uint64_t*>(smem + 3 * kTaTile);

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int tig = lane & 3;
  const int ngroups = static_cast<int>((p.hw + G - 1) / G);
  const long long w = blockIdx.x;
  const int head = static_cast<int>(w % p.heads);
  const long long t = w / p.heads;
  const int pix0 = static_cast<int>(t % ngroups) * G;
  const int clip = static_cast<int>(t / ngroups);

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmap_q);
    tma_prefetch_desc(&tmap_k);
    tma_prefetch_desc(&tmap_v);
    mbar_init(bar, 1);
    fence_mbar_init();
  }
  __syncthreads();
  CA_PDL_WAIT();
  if (threadIdx.x == 0) {
    mbar_arrive_expect_tx(bar, 3 * kTaTile);
    tma_load_4d(smem, &tmap_q, bar, head * 64, 0, pix0, clip);
    tma_load_4d(smem + kTaTile, &tmap_k, bar, head * 64, 0, pix0, clip);
    tma_load_4d(smem + 2 * kTaTile, &tmap_v, bar, head * 64, 0, pix0, clip);
  }
  mbar_wait(bar, 0);
  const uint32_t base = smem_u32(smem);

#pragma unroll 1
  for (int half = 0; half < 2; ++half) {
    const uint32_t off = half * 64 * 128;  // rows [64 half, 64 half + 64)
    float s[32];
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      Wgmma<64>::ss(s, gmma_desc_sw128(base + off + k * 32, 16, 1024),
                    gmma_desc_sw128(base + kTaTile + off + k * 32, 16, 1024), k != 0 ? 1 : 0);
    }
    wgmma_commit();
    wgmma_wait<0>();
    reg_fence(s);

    // thread holds rows (r, r + 8) of this half x key columns 8 jj + 2 tig + {0, 1}
    const int r_lo = warp * 16 + (lane >> 2);
    float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
    for (int jj = 0; jj < 8; ++jj) {
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int row = r_lo + 8 * (e >> 1);
        const int col = 8 * jj + 2 * tig + (e & 1);
        const bool valid = (col / SEQ == row / SEQ) && (col % SEQ) < p.frames;
        const float x = valid ? s[4 * jj + e] * p.scale_log2 : -INFINITY;
        s[4 * jj + e] = x;
        mx[e >> 1] = fmaxf(mx[e >> 1], x);
      }
    }
    float l[2] = {0.f, 0.f};
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
      mx[hh] = fmaxf(mx[hh], __shfl_xor_sync(0xffffffffu, mx[hh], 1));
      mx[hh] = fmaxf(mx[hh], __shfl_xor_sync(0xffffffffu, mx[hh], 2));
    }
#pragma unroll
    for (int i = 0; i < 32; ++i) {
      const float pv = exp2f(s[i] - mx[(i >> 1) & 1]);
      s[i] = pv;
      l[(i >> 1) & 1] += pv;
    }
    uint32_t pa[4][4];  // P is bf16 in the fused SDPA kernels of the reference path
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {
      pa[kk][0] = pack_bf16x2(s[8 * kk + 0], s[8 * kk + 1]);
      pa[kk][1] = pack_bf16x2(s[8 * kk + 2], s[8 * kk + 3]);
      pa[kk][2] = pack_bf16x2(s[8 * kk + 4], s[8 * kk + 5]);
      pa[kk][3] = pack_bf16x2(s[8 * kk + 6], s[8 * kk + 7]);
    }
    float o[32];
#pragma unroll
    for (int i = 0; i < 32; ++i) o[i] = 0.f;
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < 4; ++kk)
      Wgmma<64>::rs_bt(o, pa[kk], gmma_desc_sw128(base + 2 * kTaTile + off + kk * 2048, 8192, 1024), 1);
    wgmma_commit();
    wgmma_wait<0>();
    reg_fence(o);

#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
      float lt = l[hh];
      lt += __shfl_xor_sync(0xffffffffu, lt, 1);
      lt += __shfl_xor_sync(0xffffffffu, lt, 2);
      const float inv_l = 1.0f / lt;
      const int row = half * 64 + r_lo + 8 * hh;  // tile row = g * SEQ + f
      const int f = row % SEQ;
      const long long pix = static_cast<long long>(pix0) + row / SEQ;
      if (f >= p.frames || pix >= p.hw) continue;
      __nv_bfloat16* orow =
          p.out + ((static_cast<long long>(clip) * p.frames + f) * p.hw + pix) * p.out_row_stride + head * 64;
#pragma unroll
      for (int jj = 0; jj < 8; ++jj) {
        *reinterpret_cast<uint32_t*>(orow + 8 * jj + 2 * tig) =
            pack_bf16x2(o[4 * jj + 2 * hh] * inv_l, o[4 * jj + 2 * hh + 1] * inv_l);
      }
    }
  }
}

template <int SEQ>
static cudaError_t launch_seq(const CUtensorMap& q, const CUtensorMap& k, const CUtensorMap& v,
                              const TemporalAttnParams& p, long long ctas, cudaStream_t stream) {
  static bool attr_set = false;
  auto kern = temporal_attention_tc_kernel<SEQ>;
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(kTaSmem));
    if (e != cudaSuccess) return e;
    attr_set = true;
  }
  return launch_pdl(kern, static_cast<unsigned>(ctas), kTaThreads, kTaSmem, stream, q, k, v, p);
}

extern "C" int ca_temporal_attention(const void* q, const void* k, const void* v, int32_t clips, int32_t frames,
                                     int64_t hw, int32_t heads, float scale, int64_t in_row_stride, void* out, void* s) {
  if (frames < 1 || frames > 32) return fail(CA_ERR_INVALID, "temporal_attention: frames must be 1..32 (got %d)", frames);
  if (clips < 1 || hw < 1 || heads < 1) return fail(CA_ERR_INVALID, "temporal_attention: empty problem (clips, hw, heads)");
  if ((in_row_stride & 7) != 0) return fail(CA_ERR_INVALID, "temporal_attention: in_row_stride must be a multiple of 8");
  // one CTA per (clip, group of 128 / SEQ pixels, head)
  const int seq = frames <= 16 ? 16 : 32;
  const long long ctas = static_cast<long long>(clips) * ((hw + 128 / seq - 1) / (128 / seq)) * heads;
  if (ctas > 0x7fffffffLL) return fail(CA_ERR_INVALID, "temporal_attention: clips * hw * heads too large");
  // global dims ordered (channel, frame, pixel, clip): a box then holds whole frame sequences of consecutive pixels
  const cuuint64_t dims[4] = {(cuuint64_t)heads * 64, (cuuint64_t)frames, (cuuint64_t)hw, (cuuint64_t)clips};
  const cuuint64_t st[3] = {(cuuint64_t)hw * in_row_stride * 2, (cuuint64_t)in_row_stride * 2,
                            (cuuint64_t)frames * hw * in_row_stride * 2};
  const cuuint32_t box[4] = {64, (cuuint32_t)seq, (cuuint32_t)(128 / seq), 1};
  CUtensorMap tq, tk, tv;
  int rc = make_tmap(&tq, q, 4, dims, st, box);
  if (rc) return rc;
  if ((rc = make_tmap(&tk, k, 4, dims, st, box))) return rc;
  if ((rc = make_tmap(&tv, v, 4, dims, st, box))) return rc;
  TemporalAttnParams p;
  p.clips = clips; p.frames = frames; p.heads = heads; p.hw = hw;
  p.scale_log2 = scale * 1.4426950408889634f;
  p.out = static_cast<__nv_bfloat16*>(out);
  p.out_row_stride = static_cast<long long>(heads) * 64;
  cudaStream_t stream = static_cast<cudaStream_t>(s);
  const cudaError_t e = seq == 16 ? launch_seq<16>(tq, tk, tv, p, ctas, stream) : launch_seq<32>(tq, tk, tv, p, ctas, stream);
  return launched(e, "temporal_attention");
}

}  // namespace ca
