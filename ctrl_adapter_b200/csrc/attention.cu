// Fused softmax(Q K^T * scale) V for the spatial self / cross attention of the adapter, the ControlNet and the
// UNets: wgmma tensor-core MMAs, TMA-fed 128B-swizzled shared memory, online softmax in registers.
//
// One CTA = 64 * NWG query rows of one (batch, head) and one 64-wide slice of the value head dim; 128 * (NWG + 1)
// threads:
//   warpgroup 0, one thread: TMA producer.  Q once, then per tile of 128 keys the K chunks and then the V slice, each
//                            through its own ring of kStages slots (full / empty mbarrier pair per slot), so that
//                            Q K^T waits only for K.
//   warpgroups 1 .. NWG    : 64 query rows each.  S = Q K^T (m64n128, K = 64 * DQ, both operands K-major in shared
//                            memory) into registers; online softmax (exp2, running max and row sum in fp32); P is
//                            rounded to bf16 and fed from registers as the A operand of O += P V (m64n64, V read
//                            MN-major from shared memory).
// Two configurations: NWG = 3 (192 query rows, 512 threads) for head dim 64 with more than one KV tile, where the
// softmax is as expensive as the MMAs and a third warpgroup gives each SM sub-partition a third warp to hide it with;
// NWG = 2 (128 rows, 384 threads) for head dims 128 / 192, single-KV-tile calls and query lengths a 192-row tile pads
// badly (ca_attention's rule).
// Schedule of one consumer warpgroup: Q K_{j+1}^T and P_j V_j are issued back to back, and the softmax of S_{j+1} runs
// while P_j V_j is still on the tensor cores; O is rescaled by the new tile's correction once P_j V_j has retired.  The
// warpgroups take turns issuing (named barriers, round robin), so one's softmax overlaps the others' MMAs.  The
// arithmetic and its order are those of a plain tile-by-tile loop: only the schedule overlaps.
// Softmax: the row max is taken on the raw scores, so that each probability is exp2(fma(s, scale_log2, -max)), one
// FFMA and one exp2 per score.
// Epilogue: O / l, one bf16 rounding, 4-byte stores.  Head dims 128 / 192 (the zero-padded ControlNet heads) use
// DQ = 2 / 3 chunks of 64 for Q K^T.
#include "common.cuh"
#include "kernels.h"
#include "wgmma.cuh"

namespace ca {

static constexpr int kTileKV = 128;
static constexpr uint32_t kChunkBytes = 128 * 64 * 2;  // one [128 rows x 64 cols] bf16 swizzle tile = 16 KB

struct AttnParams {
  int batch, heads, lq, lk;
  int kv_batch_div;    // K/V batch index = query batch index / kv_batch_div (context shared by the frames of a clip)
  int dqk_chunks;      // padded head dim / 64 used for QK^T
  int v_slices;        // padded head dim / 64 (PV is computed one 64-wide slice per CTA)
  float scale_log2;    // softmax scale * log2(e)
  __nv_bfloat16* out;  // [batch, lq, heads * 64 * v_slices]
  long long out_batch_stride, out_row_stride;  // elements
};

template <int DQ, int NWG>
struct AttnCfg {
  static constexpr int kTileQ = 64 * NWG;
  static constexpr int kThreads = 128 * (NWG + 1);
  static constexpr uint32_t kQChunkBytes = kTileQ * 64 * 2;  // one [kTileQ rows x 64 cols] bf16 swizzle tile
  static constexpr uint32_t kQBytes = DQ * kQChunkBytes;
  static constexpr uint32_t kKBytes = DQ * kChunkBytes;  // one K slot: DQ chunks
  static constexpr uint32_t kVBytes = kChunkBytes;       // one V slot: one 64-wide slice
  // 227 KB per block on H100, minus Q, alignment slack and barriers: 4 stages at DQ 1 / 2, 2 at DQ 3
  static constexpr uint32_t kBudget = 232448 - kQBytes - 1024 - 256;
  static constexpr int kStagesRaw = kBudget / (kKBytes + kVBytes);
  static constexpr int kStages = kStagesRaw > 4 ? 4 : kStagesRaw;
  static constexpr uint32_t kDataBytes = kQBytes + kStages * (kKBytes + kVBytes);
  static constexpr uint32_t kSmemBytes = kDataBytes + 1024 /*align slack*/ + 256 /*barriers*/;
  // registers per thread after setmaxnreg: 128 * kProducerRegs + 128 * NWG * kConsumerRegs <= 65536
  static constexpr int kProducerRegs = NWG == 3 ? 24 : 40;
  static constexpr int kConsumerRegs = NWG == 3 ? 160 : 232;
  static_assert(128 * kProducerRegs + 128 * NWG * kConsumerRegs <= 65536, "register file");
  static_assert(kStages >= 2, "the K / V rings need two slots");
  static_assert((1 + 4 * kStages) * 8 <= 256, "barrier area");
};

// named barriers of the consumer warpgroups' issue turns (barrier 1 + w: warpgroup w may issue); a turn is handed from
// one warpgroup to the next, so each barrier has 2 warpgroups of threads
static constexpr int kTurnBar = 1;
static constexpr int kTurnThreads = 256;

__device__ __forceinline__ float fast_exp2(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

// Online softmax of one tile of raw scores s = Q K^T in place (s becomes the unrounded P), updating the running max
// (m_run, of the scaled scores in log2 units) and row sum; corr = the factor O must be scaled by before this tile's
// P V.  Thread holds rows (r, r + 8) x key columns 8 jj + 2 tig + {0, 1}.  The max is taken on the raw scores, which
// gives the scaled max because c = scale * log2(e) > 0 (ca_attention), so that each probability is one FFMA and one
// exp2.  kMask: keys past kv_valid (only the last KV tile has them) get the raw score -inf.
template <bool kMask>
__device__ __forceinline__ void online_softmax(float (&s)[64], float c, int kv_valid, int tig, float (&m_run)[2],
                                               float (&l_run)[2], float (&corr)[2]) {
  float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
  for (int jj = 0; jj < 16; ++jj) {
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      if (kMask && 8 * jj + 2 * tig + (e & 1) >= kv_valid) s[4 * jj + e] = -INFINITY;
      mx[e >> 1] = fmaxf(mx[e >> 1], s[4 * jj + e]);
    }
  }
  float neg_m[2];
#pragma unroll
  for (int hh = 0; hh < 2; ++hh) {
    mx[hh] = fmaxf(mx[hh], __shfl_xor_sync(0xffffffffu, mx[hh], 1));
    mx[hh] = fmaxf(mx[hh], __shfl_xor_sync(0xffffffffu, mx[hh], 2));
    const float m_new = fmaxf(m_run[hh], mx[hh] * c);
    corr[hh] = fast_exp2(m_run[hh] - m_new);  // 0 on the first tile (m_run = -inf)
    m_run[hh] = m_new;
    neg_m[hh] = -m_new;
    l_run[hh] *= corr[hh];
  }
#pragma unroll
  for (int jj = 0; jj < 16; ++jj) {
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const float pv = fast_exp2(fmaf(s[4 * jj + e], c, neg_m[e >> 1]));
      s[4 * jj + e] = pv;
      l_run[e >> 1] += pv;
    }
  }
}

template <int DQ, int NWG>
__global__ void __launch_bounds__(AttnCfg<DQ, NWG>::kThreads, 1)
attention_kernel(const __grid_constant__ CUtensorMap tmap_q, const __grid_constant__ CUtensorMap tmap_k,
                 const __grid_constant__ CUtensorMap tmap_v, const AttnParams p) {
  using Cfg = AttnCfg<DQ, NWG>;
  constexpr uint32_t S = Cfg::kStages;
  CA_PDL_TRIGGER();
  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw_addr = smem_u32(smem_raw);
  uint8_t* smem = smem_raw + ((1024u - (raw_addr & 1023u)) & 1023u);
  uint8_t* smem_q = smem;
  uint8_t* smem_k = smem + Cfg::kQBytes;            // [kStages] x kKBytes
  uint8_t* smem_v = smem_k + S * Cfg::kKBytes;      // [kStages] x kVBytes
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + Cfg::kDataBytes);
  uint64_t* q_full = bars;
  uint64_t* k_full = bars + 1;           // [kStages]
  uint64_t* k_empty = bars + 1 + S;      // [kStages]
  uint64_t* v_full = bars + 1 + 2 * S;   // [kStages]
  uint64_t* v_empty = bars + 1 + 3 * S;  // [kStages]

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int q0 = blockIdx.x * Cfg::kTileQ;
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
    for (uint32_t s = 0; s < S; ++s) {
      mbar_init(&k_full[s], 1);
      mbar_init(&k_empty[s], 4 * NWG);  // one arrive per consumer warp
      mbar_init(&v_full[s], 1);
      mbar_init(&v_empty[s], 4 * NWG);
    }
    fence_mbar_init();
  }
  __syncthreads();
  CA_PDL_WAIT();

  if (warp < 4) {
    // ===================== TMA producer =====================
    setmaxnreg_dec<Cfg::kProducerRegs>();
    if (threadIdx.x == 0) {
      const int kvb = b / p.kv_batch_div;
      mbar_arrive_expect_tx(q_full, Cfg::kQBytes);
      for (int c = 0; c < DQ; ++c)
        tma_load_3d(smem_q + c * Cfg::kQChunkBytes, &tmap_q, q_full, h * dpad + c * 64, q0, b);
      for (uint32_t j = 0; j < static_cast<uint32_t>(nkv); ++j) {
        const uint32_t slot = j % S;
        const uint32_t phase = (j / S) & 1u;
        mbar_wait(&k_empty[slot], phase ^ 1);
        uint8_t* kdst = smem_k + slot * Cfg::kKBytes;
        mbar_arrive_expect_tx(&k_full[slot], Cfg::kKBytes);
        for (int c = 0; c < DQ; ++c)
          tma_load_3d(kdst + c * kChunkBytes, &tmap_k, &k_full[slot], h * dpad + c * 64, j * kTileKV, kvb);
        mbar_wait(&v_empty[slot], phase ^ 1);
        mbar_arrive_expect_tx(&v_full[slot], Cfg::kVBytes);
        tma_load_3d(smem_v + slot * Cfg::kVBytes, &tmap_v, &v_full[slot], h * dpad + vs * 64, j * kTileKV, kvb);
      }
    }
    return;
  }

  // ===================== consumers =====================
  setmaxnreg_inc<Cfg::kConsumerRegs>();
  const int cw = (warp >> 2) - 1;  // query rows [64 cw, 64 cw + 64) of the tile
  const int wq = warp & 3;
  const int tig = lane & 3;
  float o[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) o[i] = 0.f;
  float m_run[2] = {-INFINITY, -INFINITY};
  float l_run[2] = {0.f, 0.f};
  float corr[2];
  float s[64];
  uint32_t pa[8][4];
  const uint32_t q_addr = smem_u32(smem_q) + cw * 64 * 128;
  const int last = nkv - 1;
  const int kv_valid_last = p.lk - last * kTileKV;

  // S = Q K_j^T (one commit group; K_j has landed)
  auto issue_qk = [&](uint32_t j) {
    const uint32_t k_addr = smem_u32(smem_k + (j % S) * Cfg::kKBytes);
#pragma unroll
    for (int c = 0; c < DQ; ++c) {
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        Wgmma<128>::ss(s, gmma_desc_sw128(q_addr + c * Cfg::kQChunkBytes + k * 32, 16, 1024),
                       gmma_desc_sw128(k_addr + c * kChunkBytes + k * 32, 16, 1024), (c | k) != 0 ? 1 : 0);
      }
    }
    wgmma_commit();
  };
  // O += P V_j (one commit group; V_j has landed)
  auto issue_pv = [&](uint32_t j) {
    const uint32_t v_addr = smem_u32(smem_v + (j % S) * Cfg::kVBytes);
#pragma unroll
    for (int kk = 0; kk < 8; ++kk) Wgmma<64>::rs_bt(o, pa[kk], gmma_desc_sw128(v_addr + kk * 2048, 8192, 1024), 1);
    wgmma_commit();
  };
  auto softmax = [&](int j) {
    if (j == last) online_softmax<true>(s, p.scale_log2, kv_valid_last, tig, m_run, l_run, corr);
    else online_softmax<false>(s, p.scale_log2, kTileKV, tig, m_run, l_run, corr);
  };
  auto pack_p = [&]() {
#pragma unroll
    for (int kk = 0; kk < 8; ++kk) {
      pa[kk][0] = pack_bf16x2(s[8 * kk + 0], s[8 * kk + 1]);
      pa[kk][1] = pack_bf16x2(s[8 * kk + 2], s[8 * kk + 3]);
      pa[kk][2] = pack_bf16x2(s[8 * kk + 4], s[8 * kk + 5]);
      pa[kk][3] = pack_bf16x2(s[8 * kk + 6], s[8 * kk + 7]);
    }
  };
  // Issue turns go round the warpgroups, nkv + 1 per warpgroup (S_0; S_{j+1} with P_j V_j; the last P V).  Warpgroup
  // 0 needs no go-ahead for its first turn and the last warpgroup gives none after its last, so every arrive is
  // matched by exactly one sync.
  auto turn_begin = [&](bool first) {
    if (!(first && cw == 0)) named_bar_sync(kTurnBar + cw, kTurnThreads);
  };
  auto turn_end = [&](bool final_turn) {
    if (!(final_turn && cw == NWG - 1)) named_bar_arrive(kTurnBar + (cw + 1) % NWG, kTurnThreads);
  };
  auto wait_full = [&](uint64_t* full, uint32_t j) { mbar_wait(&full[j % S], (j / S) & 1u); };
  auto release = [&](uint64_t* empty, uint32_t j) {
    if (lane == 0) mbar_arrive(&empty[j % S]);
  };

  mbar_wait(q_full, 0);

  // prologue: S_0 and its softmax (O is still 0: no rescale)
  wait_full(k_full, 0);
  turn_begin(true);
  wgmma_fence();
  issue_qk(0);
  turn_end(false);
  wgmma_wait<0>();
  reg_fence(s);
  release(k_empty, 0);
  softmax(0);
  pack_p();

  // steady state: S_{j+1} and P_j V_j in flight together; the softmax of S_{j+1} overlaps P_j V_j
  for (int j = 0; j < last; ++j) {
    wait_full(k_full, j + 1);
    wait_full(v_full, j);
    turn_begin(false);
    wgmma_fence();
    issue_qk(j + 1);
    issue_pv(j);
    turn_end(false);
    wgmma_wait<1>();
    reg_fence(s);
    release(k_empty, j + 1);
    softmax(j + 1);
    reg_fence(s);
    wgmma_wait<0>();
    reg_fence(o);
    release(v_empty, j);
#pragma unroll
    for (int i = 0; i < 32; ++i) o[i] *= corr[(i >> 1) & 1];
    pack_p();
  }

  // tail: the last P V
  wait_full(v_full, last);
  turn_begin(false);
  wgmma_fence();
  issue_pv(last);
  turn_end(true);
  wgmma_wait<0>();
  reg_fence(o);
  release(v_empty, last);

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

template <int DQ, int NWG>
static cudaError_t launch_cfg(const CUtensorMap& q, const CUtensorMap& k, const CUtensorMap& v, const AttnParams& p,
                              cudaStream_t stream) {
  using Cfg = AttnCfg<DQ, NWG>;
  static bool attr_set = false;
  auto kern = attention_kernel<DQ, NWG>;
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         static_cast<int>(Cfg::kSmemBytes));
    if (e != cudaSuccess) return e;
    attr_set = true;
  }
  const dim3 grid((p.lq + Cfg::kTileQ - 1) / Cfg::kTileQ, p.heads * p.v_slices, p.batch);
  return launch_pdl(kern, grid, Cfg::kThreads, Cfg::kSmemBytes, stream, q, k, v, p);
}

// Head dim 64 with more than one KV tile runs 192-row query tiles (three consumer warpgroups) unless their padding
// exceeds the 128-row tiles' by more than 1/25 of lq (L 1024: 128 rows; L 2304, 4096, 9216, 16384: 192 rows).
static bool use_wg3(int dqk_chunks, int lq, int lk) {
  if (dqk_chunks != 1 || lk <= kTileKV) return false;
  const long long pad192 = (lq + 191LL) / 192 * 192 - lq;
  const long long pad128 = (lq + 127LL) / 128 * 128 - lq;
  return 25 * (pad192 - pad128) <= lq;
}

extern "C" int ca_attention(const ca_attention_desc* d, void* cuda_stream) {
  if (!d) return fail(CA_ERR_INVALID, "null desc");
  cudaStream_t stream = static_cast<cudaStream_t>(cuda_stream);
  if (d->head_dim_pad != 64 && d->head_dim_pad != 128 && d->head_dim_pad != 192)
    return fail(CA_ERR_UNSUPPORTED, "head_dim_pad must be 64, 128 or 192 (got %d)", d->head_dim_pad);
  if (d->batch < 1 || d->heads < 1 || d->lq < 1 || d->lk < 1) return fail(CA_ERR_INVALID, "empty attention problem");
  const int kv_div = d->kv_batch_div > 0 ? d->kv_batch_div : 1;
  if (d->batch % kv_div != 0) return fail(CA_ERR_INVALID, "batch must be a multiple of kv_batch_div");
  // grid (q tiles, heads * head_dim_pad / 64, batch)
  if (d->batch > kMaxGridYZ) return fail(CA_ERR_INVALID, "batch (%d) must be <= 65535", d->batch);
  if (static_cast<long long>(d->heads) * (d->head_dim_pad / 64) > kMaxGridYZ)
    return fail(CA_ERR_INVALID, "heads * head_dim_pad / 64 (%d * %d) must be <= 65535", d->heads, d->head_dim_pad / 64);
  // the epilogue stores bf16 pairs as 4-byte words
  if (!aligned(d->out, 4) || (d->out_row_stride & 1) != 0 || (d->out_batch_stride & 1) != 0)
    return fail(CA_ERR_INVALID, "out must be 4-byte aligned with even out_row_stride, out_batch_stride (%lld, %lld)",
                (long long)d->out_row_stride, (long long)d->out_batch_stride);
  // the softmax takes its row max on the raw scores (online_softmax), which is the scaled max only for a positive scale
  const float scale_log2 = d->scale * 1.4426950408889634f;
  if (!(d->scale > 0.f) || !isfinite(scale_log2))
    return fail(CA_ERR_INVALID, "scale must be positive and finite (got %g)", (double)d->scale);
  const int dqk_chunks = d->head_dim_pad / 64;
  const bool wg3 = use_wg3(dqk_chunks, d->lq, d->lk);
  const cuuint64_t ctot = static_cast<cuuint64_t>(d->heads) * d->head_dim_pad;
  CUtensorMap tq, tk, tv;
  {
    const cuuint32_t box[3] = {64, wg3 ? 192u : 128u, 1};
    cuuint64_t dims[3] = {ctot, (cuuint64_t)d->lq, (cuuint64_t)d->batch};
    cuuint64_t st[2] = {(cuuint64_t)d->q_row_stride * 2, (cuuint64_t)d->q_batch_stride * 2};
    int rc = make_tmap(&tq, d->q, 3, dims, st, box);
    if (rc) return rc;
  }
  {
    const cuuint32_t box[3] = {64, kTileKV, 1};
    cuuint64_t dims[3] = {ctot, (cuuint64_t)d->lk, (cuuint64_t)(d->batch / kv_div)};
    cuuint64_t st[2] = {(cuuint64_t)d->k_row_stride * 2, (cuuint64_t)d->k_batch_stride * 2};
    int rc = make_tmap(&tk, d->k, 3, dims, st, box);
    if (rc) return rc;
    cuuint64_t sv[2] = {(cuuint64_t)d->v_row_stride * 2, (cuuint64_t)d->v_batch_stride * 2};
    rc = make_tmap(&tv, d->v, 3, dims, sv, box);
    if (rc) return rc;
  }
  AttnParams p;
  p.batch = d->batch; p.heads = d->heads; p.lq = d->lq; p.lk = d->lk;
  p.kv_batch_div = kv_div;
  p.dqk_chunks = dqk_chunks;
  p.v_slices = d->head_dim_pad / 64;
  p.scale_log2 = scale_log2;
  p.out = static_cast<__nv_bfloat16*>(d->out);
  p.out_batch_stride = d->out_batch_stride;
  p.out_row_stride = d->out_row_stride;
  const cudaError_t e = wg3                 ? launch_cfg<1, 3>(tq, tk, tv, p, stream)
                        : p.dqk_chunks == 1 ? launch_cfg<1, 2>(tq, tk, tv, p, stream)
                        : p.dqk_chunks == 2 ? launch_cfg<2, 2>(tq, tk, tv, p, stream)
                                            : launch_cfg<3, 2>(tq, tk, tv, p, stream);
  return launched(e, "attention launch");
}

}  // namespace ca
