// Fused softmax(Q K^T * scale) V for the spatial self / cross attention of the adapter, the ControlNet and the
// UNets: wgmma tensor-core MMAs, TMA-fed 128B-swizzled shared memory, online softmax in registers.
//
// One CTA = 128 query rows of one (batch, head) and one 64-wide slice of the value head dim; 384 threads:
//   warpgroup 0, one thread: TMA producer (Q once, then K and V tiles of 128 keys through a 2-stage ring)
//   warpgroups 1, 2        : 64 query rows each.  Per KV tile: S = Q K^T (m64n128, K = 64 * DQ, both operands K-major
//                            in shared memory) into registers; online softmax (exp2, running max and row sum in fp32);
//                            P is rounded to bf16 and fed from registers as the A operand of O += P V (m64n64, V read
//                            MN-major from shared memory).  The ring slot is released once both wgmma have retired.
// Epilogue: O / l, one bf16 rounding, 4-byte stores.  Head dims 128 / 192 (the zero-padded ControlNet heads) use
// DQ = 2 / 3 chunks of 64 for Q K^T.
#include "common.cuh"
#include "kernels.h"
#include "wgmma.cuh"

namespace ca {

static constexpr int kTileQ = 128;
static constexpr int kTileKV = 128;
static constexpr int kAttnThreads = 384;
static constexpr uint32_t kChunkBytes = 128 * 64 * 2;  // one [128 rows x 64 cols] bf16 swizzle tile = 16 KB

template <int DQ>
struct AttnCfg {
  static constexpr int kStages = 2;
  static constexpr uint32_t kQBytes = DQ * kChunkBytes;
  static constexpr uint32_t kStageBytes = (DQ + 1) * kChunkBytes;  // K chunks + one V slice
  static constexpr uint32_t kDataBytes = kQBytes + kStages * kStageBytes;
  static constexpr uint32_t kSmemBytes = kDataBytes + 1024 /*align slack*/ + 256 /*barriers*/;
};

__device__ __forceinline__ float fast_exp2(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

template <int DQ>
__global__ void __launch_bounds__(kAttnThreads, 1)
attention_kernel(const __grid_constant__ CUtensorMap tmap_q, const __grid_constant__ CUtensorMap tmap_k,
                 const __grid_constant__ CUtensorMap tmap_v, const AttnParams p) {
  using Cfg = AttnCfg<DQ>;
  CA_PDL_TRIGGER();
  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw_addr = smem_u32(smem_raw);
  uint8_t* smem = smem_raw + ((1024u - (raw_addr & 1023u)) & 1023u);
  uint8_t* smem_q = smem;
  uint8_t* smem_kv = smem + Cfg::kQBytes;
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + Cfg::kDataBytes);
  uint64_t* q_full = bars;
  uint64_t* full = bars + 1;   // [kStages]
  uint64_t* empty = bars + 3;  // [kStages]

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int q0 = blockIdx.x * kTileQ;
  const int h = blockIdx.y / p.v_slices;
  const int vs = blockIdx.y % p.v_slices;
  const int b = blockIdx.z;
  const int dpad = 64 * p.v_slices;  // padded head dim (elements) in the Q/K/V channel layout
  const int nkv = (p.lk + kTileKV - 1) / kTileKV;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmap_q);
    tma_prefetch_desc(&tmap_k);
    tma_prefetch_desc(&tmap_v);
    mbar_init(q_full, 1);
    for (int s = 0; s < Cfg::kStages; ++s) {
      mbar_init(&full[s], 1);
      mbar_init(&empty[s], 8);  // one arrive per consumer warp
    }
    fence_mbar_init();
  }
  __syncthreads();
  CA_PDL_WAIT();

  if (warp < 4) {
    // ===================== TMA producer =====================
    setmaxnreg_dec<40>();
    if (threadIdx.x == 0) {
      const int kvb = b / p.kv_batch_div;
      mbar_arrive_expect_tx(q_full, Cfg::kQBytes);
      for (int c = 0; c < DQ; ++c) tma_load_3d(smem_q + c * kChunkBytes, &tmap_q, q_full, h * dpad + c * 64, q0, b);
      int stage = 0;
      uint32_t phase = 0;
      for (int j = 0; j < nkv; ++j) {
        mbar_wait(&empty[stage], phase ^ 1);
        uint8_t* dst = smem_kv + stage * Cfg::kStageBytes;
        mbar_arrive_expect_tx(&full[stage], Cfg::kStageBytes);
        for (int c = 0; c < DQ; ++c)
          tma_load_3d(dst + c * kChunkBytes, &tmap_k, &full[stage], h * dpad + c * 64, j * kTileKV, kvb);
        tma_load_3d(dst + DQ * kChunkBytes, &tmap_v, &full[stage], h * dpad + vs * 64, j * kTileKV, kvb);
        if (++stage == Cfg::kStages) { stage = 0; phase ^= 1; }
      }
    }
    return;
  }

  // ===================== consumers =====================
  setmaxnreg_inc<232>();
  const int cw = (warp >> 2) - 1;  // query rows [64 cw, 64 cw + 64) of the tile
  const int wq = warp & 3;
  const int tig = lane & 3;
  float o[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) o[i] = 0.f;
  float m_run[2] = {-INFINITY, -INFINITY};
  float l_run[2] = {0.f, 0.f};
  const uint32_t q_addr = smem_u32(smem_q) + cw * 64 * 128;
  mbar_wait(q_full, 0);

  int stage = 0;
  uint32_t phase = 0;
  for (int j = 0; j < nkv; ++j) {
    mbar_wait(&full[stage], phase);
    const uint32_t kv_addr = smem_u32(smem_kv + stage * Cfg::kStageBytes);
    float s[64];
    wgmma_fence();
#pragma unroll
    for (int c = 0; c < DQ; ++c) {
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        Wgmma<128>::ss(s, gmma_desc_sw128(q_addr + c * kChunkBytes + k * 32, 16, 1024),
                       gmma_desc_sw128(kv_addr + c * kChunkBytes + k * 32, 16, 1024), (c | k) != 0 ? 1 : 0);
      }
    }
    wgmma_commit();
    wgmma_wait<0>();
    reg_fence(s);

    // ---- online softmax: thread holds rows (r, r + 8) x key columns 8 jj + 2 tig + {0, 1} ----
    const int kv_valid = min(kTileKV, p.lk - j * kTileKV);
    float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
    for (int jj = 0; jj < 16; ++jj) {
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int col = 8 * jj + 2 * tig + (e & 1);
        float x = s[4 * jj + e] * p.scale_log2;
        if (col >= kv_valid) x = -INFINITY;
        s[4 * jj + e] = x;
        mx[e >> 1] = fmaxf(mx[e >> 1], x);
      }
    }
    float corr[2];
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
      mx[hh] = fmaxf(mx[hh], __shfl_xor_sync(0xffffffffu, mx[hh], 1));
      mx[hh] = fmaxf(mx[hh], __shfl_xor_sync(0xffffffffu, mx[hh], 2));
      const float m_new = fmaxf(m_run[hh], mx[hh]);
      corr[hh] = fast_exp2(m_run[hh] - m_new);  // 0 on the first tile (m_run = -inf)
      m_run[hh] = m_new;
      l_run[hh] *= corr[hh];
    }
    uint32_t pa[8][4];
#pragma unroll
    for (int jj = 0; jj < 16; ++jj) {
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const float pv = fast_exp2(s[4 * jj + e] - m_run[e >> 1]);
        s[4 * jj + e] = pv;
        l_run[e >> 1] += pv;
      }
    }
#pragma unroll
    for (int kk = 0; kk < 8; ++kk) {
      pa[kk][0] = pack_bf16x2(s[8 * kk + 0], s[8 * kk + 1]);
      pa[kk][1] = pack_bf16x2(s[8 * kk + 2], s[8 * kk + 3]);
      pa[kk][2] = pack_bf16x2(s[8 * kk + 4], s[8 * kk + 5]);
      pa[kk][3] = pack_bf16x2(s[8 * kk + 6], s[8 * kk + 7]);
    }
#pragma unroll
    for (int i = 0; i < 32; ++i) o[i] *= corr[(i >> 1) & 1];

    // ---- O += P V ----
    const uint32_t v_addr = kv_addr + DQ * kChunkBytes;
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < 8; ++kk) Wgmma<64>::rs_bt(o, pa[kk], gmma_desc_sw128(v_addr + kk * 2048, 8192, 1024), 1);
    wgmma_commit();
    wgmma_wait<0>();
    reg_fence(o);
    if (lane == 0) mbar_arrive(&empty[stage]);
    if (++stage == Cfg::kStages) { stage = 0; phase ^= 1; }
  }

  // ---- epilogue: O / l ----
#pragma unroll
  for (int hh = 0; hh < 2; ++hh) {
    float l = l_run[hh];
    l += __shfl_xor_sync(0xffffffffu, l, 1);
    l += __shfl_xor_sync(0xffffffffu, l, 2);
    const float inv_l = 1.0f / l;
    const int row = q0 + cw * 64 + wq * 16 + (lane >> 2) + 8 * hh;
    if (row >= p.lq) continue;
    __nv_bfloat16* orow = p.out + static_cast<long long>(b) * p.out_batch_stride +
                          static_cast<long long>(row) * p.out_row_stride + h * dpad + vs * 64;
#pragma unroll
    for (int jj = 0; jj < 8; ++jj) {
      *reinterpret_cast<uint32_t*>(orow + 8 * jj + 2 * tig) =
          pack_bf16x2(o[4 * jj + 2 * hh] * inv_l, o[4 * jj + 2 * hh + 1] * inv_l);
    }
  }
}

template <int DQ>
static cudaError_t launch_dq(const CUtensorMap& q, const CUtensorMap& k, const CUtensorMap& v, const AttnParams& p,
                             cudaStream_t stream) {
  using Cfg = AttnCfg<DQ>;
  static bool attr_set = false;
  auto kern = attention_kernel<DQ>;
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         static_cast<int>(Cfg::kSmemBytes));
    if (e != cudaSuccess) return e;
    attr_set = true;
  }
  const dim3 grid((p.lq + kTileQ - 1) / kTileQ, p.heads * p.v_slices, p.batch);
  CA_KERNEL_LAUNCH(kern, grid, kAttnThreads, Cfg::kSmemBytes, stream, q, k, v, p);
  return cudaGetLastError();
}

cudaError_t launch_attention(const CUtensorMap& q, const CUtensorMap& k, const CUtensorMap& v, const AttnParams& p,
                             cudaStream_t stream) {
  switch (p.dqk_chunks) {
    case 1: return launch_dq<1>(q, k, v, p, stream);
    case 2: return launch_dq<2>(q, k, v, p, stream);
    case 3: return launch_dq<3>(q, k, v, p, stream);
    default: return cudaErrorInvalidValue;
  }
}

}  // namespace ca
