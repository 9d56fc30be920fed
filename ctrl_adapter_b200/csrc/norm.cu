// GroupNorm (channels-last, two launches) and LayerNorm.  HBM-bound: 16-byte vector loads with several loads in
// flight per thread, fp32 math, fp64 only for the cross-block accumulation of the GroupNorm statistics.
#include "common.cuh"
#include "kernels.h"

namespace ca {

__device__ __forceinline__ uint4 ld_nc(const void* p) {
  uint4 r;
  asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0, %1, %2, %3}, [%4];"
               : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
               : "l"(p));
  return r;
}

// ---------------------------------------------------------------------------------------------
// GroupNorm statistics: sums[n][g] = {sum x, sum x^2} over rows x (C/groups) channels.
// grid (slabs, n); each thread owns one 8-channel vector column and strides over the rows of the slab,
// 4 rows per iteration so that 4 independent 16-byte loads are in flight.
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(512)
gn_stats_kernel(const __nv_bfloat16* __restrict__ x0, int c0, const __nv_bfloat16* __restrict__ x1, int c1,
                long long rows, int groups, int rows_per_block, double* __restrict__ sums) {
  CA_PDL_TRIGGER();
  CA_PDL_WAIT();
  __shared__ float s_acc[64][2];
  const int C = c0 + c1;
  const int nvec = C >> 3;
  const int cpg = C / groups;
  const int n = blockIdx.y;
  for (int i = threadIdx.x; i < groups * 2; i += blockDim.x) (&s_acc[0][0])[i] = 0.f;
  __syncthreads();
  const int rows_per_iter = blockDim.x / nvec;
  const int vec = threadIdx.x % nvec;
  const int rsub = threadIdx.x / nvec;
  if (rsub < rows_per_iter) {
    const long long r_begin = static_cast<long long>(blockIdx.x) * rows_per_block;
    const long long r_end = min(rows, r_begin + rows_per_block);
    const int ch = vec * 8;
    const bool second = ch >= c0;
    const int cs = second ? c1 : c0;
    const __nv_bfloat16* base = (second ? x1 + (ch - c0) : x0 + ch) + static_cast<long long>(n) * rows * cs;
    float s[8], ss[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) { s[e] = 0.f; ss[e] = 0.f; }
    long long r = r_begin + rsub;
    for (; r + 3LL * rows_per_iter < r_end; r += 4LL * rows_per_iter) {
      uint4 u[4];
#pragma unroll
      for (int k = 0; k < 4; ++k) u[k] = ld_nc(base + (r + static_cast<long long>(k) * rows_per_iter) * cs);
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&u[k]);
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const float2 f = __bfloat1622float2(h[e]);
          s[2 * e] += f.x; ss[2 * e] = fmaf(f.x, f.x, ss[2 * e]);
          s[2 * e + 1] += f.y; ss[2 * e + 1] = fmaf(f.y, f.y, ss[2 * e + 1]);
        }
      }
    }
    for (; r < r_end; r += rows_per_iter) {
      const uint4 u = ld_nc(base + r * cs);
      const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&u);
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const float2 f = __bfloat1622float2(h[e]);
        s[2 * e] += f.x; ss[2 * e] = fmaf(f.x, f.x, ss[2 * e]);
        s[2 * e + 1] += f.y; ss[2 * e + 1] = fmaf(f.y, f.y, ss[2 * e + 1]);
      }
    }
    // fold the 8 channels into (at most a few) groups
    int g_cur = ch / cpg;
    float a = 0.f, b = 0.f;
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      const int g = (ch + e) / cpg;
      if (g != g_cur) {
        atomicAdd(&s_acc[g_cur][0], a);
        atomicAdd(&s_acc[g_cur][1], b);
        a = 0.f; b = 0.f; g_cur = g;
      }
      a += s[e]; b += ss[e];
    }
    atomicAdd(&s_acc[g_cur][0], a);
    atomicAdd(&s_acc[g_cur][1], b);
  }
  __syncthreads();
  for (int i = threadIdx.x; i < groups * 2; i += blockDim.x)
    atomicAdd(&sums[static_cast<long long>(n) * groups * 2 + i], static_cast<double>((&s_acc[0][0])[i]));
}

// the GroupNorm channel layout both passes support: <= 64 groups of whole 8-channel vectors, <= 512 vectors per pixel
static int check_gn_channels(const char* what, int c0, int c1, int groups) {
  const int C = c0 + c1;
  if (groups < 1 || groups > 64) return fail(CA_ERR_INVALID, "%s: groups must be 1..64 (got %d)", what, groups);
  if (C % groups != 0) return fail(CA_ERR_INVALID, "%s: c0 + c1 (%d) must be a multiple of groups (%d)", what, C, groups);
  if ((c0 & 7) != 0 || (c1 & 7) != 0 || C < 8 || C > 4096)
    return fail(CA_ERR_INVALID, "%s: c0, c1 (%d, %d) must be multiples of 8 with 8 <= c0 + c1 <= 4096", what, c0, c1);
  return CA_OK;
}

extern "C" int ca_groupnorm_stats(const void* x0, int32_t c0, const void* x1, int32_t c1, int32_t n, int64_t rows,
                                  int32_t groups, double* sums, void* s) {
  if (int rc = check_gn_channels("groupnorm_stats", c0, c1, groups)) return rc;
  cudaStream_t stream = static_cast<cudaStream_t>(s);
  cudaError_t e = cudaMemsetAsync(sums, 0, sizeof(double) * n * groups * 2, stream);
  if (e != cudaSuccess) return launched(e, "groupnorm_stats");
  const int C = c0 + c1;
  const int threads = 512;
  // >= ~4 resident blocks per SM overall, while keeping the per-thread fp32 partial sums short (<= ~64 rows)
  const int rows_per_iter = threads / (C >> 3);
  long long want_blocks = (148LL * 4 + n - 1) / n;
  long long rpb = (rows + want_blocks - 1) / want_blocks;
  const long long min_rpb = 16LL * rows_per_iter, max_rpb = 64LL * rows_per_iter;
  if (rpb < min_rpb) rpb = min_rpb;
  if (rpb > max_rpb) rpb = max_rpb;
  const int slabs = static_cast<int>((rows + rpb - 1) / rpb);
  e = launch_pdl(gn_stats_kernel, dim3(slabs, n), threads, 0, stream, static_cast<const __nv_bfloat16*>(x0), c0,
                 static_cast<const __nv_bfloat16*>(x1), c1, rows, groups, static_cast<int>(rpb), sums);
  return launched(e, "groupnorm_stats");
}

// ---------------------------------------------------------------------------------------------
// GroupNorm apply (+SiLU, +2x nearest upsample, +concat of two sources), bf16 out.
// grid (pixel slabs, images); image i uses the statistics of sample i / imgs_per_sample.
// Same thread mapping as the statistics pass: a thread owns ONE 8-channel vector column for the whole slab, so its 8
// scale / shift pairs (gamma*rstd, beta - mean*gamma*rstd) live in registers and the pixel loop is pure streaming --
// 4 independent 16-byte loads in flight, no index arithmetic beyond one add per pixel, no shared-memory reads.
// ---------------------------------------------------------------------------------------------
template <bool SILU, bool UP>
__global__ void __launch_bounds__(512, 2)
gn_apply_kernel(const __nv_bfloat16* __restrict__ x0, int c0, const __nv_bfloat16* __restrict__ x1, int c1, int h,
                int w, int imgs_per_sample, int groups, float eps, const double* __restrict__ sums,
                const float* __restrict__ gamma, const float* __restrict__ beta, int pix_per_block,
                __nv_bfloat16* __restrict__ y) {
  CA_PDL_TRIGGER();
  CA_PDL_WAIT();
  __shared__ float s_mean[64], s_rstd[64];
  const int C = c0 + c1;
  const int nvec = C >> 3;
  const int cpg = C / groups;
  const int img = blockIdx.y;
  const int sample = img / imgs_per_sample;
  const int hw = h * w;
  if (threadIdx.x < groups) {
    const double cnt = static_cast<double>(hw) * imgs_per_sample * cpg;
    const double s = sums[(static_cast<long long>(sample) * groups + threadIdx.x) * 2];
    const double ss = sums[(static_cast<long long>(sample) * groups + threadIdx.x) * 2 + 1];
    const double mean = s / cnt;
    double var = ss / cnt - mean * mean;
    if (var < 0.0) var = 0.0;
    s_mean[threadIdx.x] = static_cast<float>(mean);
    s_rstd[threadIdx.x] = static_cast<float>(1.0 / sqrt(var + static_cast<double>(eps)));
  }
  __syncthreads();
  const int rows_per_iter = blockDim.x / nvec;  // the launcher makes blockDim.x an exact multiple of nvec
  const int vec = threadIdx.x % nvec;
  const int rsub = threadIdx.x / nvec;
  const int ch = vec * 8;
  float sc[8], sh[8];
#pragma unroll
  for (int e = 0; e < 8; ++e) {
    const int g = (ch + e) / cpg;
    sc[e] = s_rstd[g] * __ldg(gamma + ch + e);
    sh[e] = __ldg(beta + ch + e) - s_mean[g] * sc[e];
  }
  const bool second = ch >= c0;
  const int cs = second ? c1 : c0;
  const __nv_bfloat16* src = (second ? x1 + (ch - c0) : x0 + ch) + static_cast<long long>(img) * hw * cs;
  const int p_begin = blockIdx.x * pix_per_block;
  const int p_end = min(hw, p_begin + pix_per_block);

  auto emit = [&](const uint4& u, int pix) {
    const uint32_t wds[4] = {u.x, u.y, u.z, u.w};
    uint32_t o[4];
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      float v0 = fmaf(bf16lo_to_float(wds[e]), sc[2 * e], sh[2 * e]);
      float v1 = fmaf(bf16hi_to_float(wds[e]), sc[2 * e + 1], sh[2 * e + 1]);
      if (SILU) {
        v0 = __fdividef(v0, 1.0f + __expf(-v0));
        v1 = __fdividef(v1, 1.0f + __expf(-v1));
      }
      o[e] = pack_bf16x2(v0, v1);
    }
    const uint4 ov = make_uint4(o[0], o[1], o[2], o[3]);
    if (!UP) {
      *reinterpret_cast<uint4*>(y + (static_cast<long long>(img) * hw + pix) * C + ch) = ov;
    } else {
      const int py = pix / w, px = pix - py * w;
      const long long ow = 2LL * w;
      __nv_bfloat16* dst = y + ((static_cast<long long>(img) * 2 * h + 2 * py) * ow + 2 * px) * C + ch;
      *reinterpret_cast<uint4*>(dst) = ov;
      *reinterpret_cast<uint4*>(dst + C) = ov;
      *reinterpret_cast<uint4*>(dst + ow * C) = ov;
      *reinterpret_cast<uint4*>(dst + ow * C + C) = ov;
    }
  };

  // software pipeline: the four loads of the NEXT step are issued before the current four pixels are normalised (SiLU is
  // ~30 instructions per pixel-vector), so a thread always has loads in flight -- without it the kernel sat at ~3.5 TB/s
  // with half of its threads computing and not loading at any time
  int pix = p_begin + rsub;
  const int step = 4 * rows_per_iter;
  uint4 u[4];
  bool have = pix + 3 * rows_per_iter < p_end;
  if (have) {
#pragma unroll
    for (int k = 0; k < 4; ++k) u[k] = ld_nc(src + static_cast<long long>(pix + k * rows_per_iter) * cs);
  }
  while (have) {
    uint4 cur[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) cur[k] = u[k];
    const int pn = pix + step;
    have = pn + 3 * rows_per_iter < p_end;
    if (have) {
#pragma unroll
      for (int k = 0; k < 4; ++k) u[k] = ld_nc(src + static_cast<long long>(pn + k * rows_per_iter) * cs);
    }
#pragma unroll
    for (int k = 0; k < 4; ++k) emit(cur[k], pix + k * rows_per_iter);
    pix = pn;
  }
  for (; pix < p_end; pix += rows_per_iter) emit(ld_nc(src + static_cast<long long>(pix) * cs), pix);
}

extern "C" int ca_groupnorm_apply(const void* x0, int32_t c0, const void* x1, int32_t c1, int32_t n, int32_t h,
                                  int32_t w, int32_t imgs_per_sample, int32_t groups, float eps, const double* sums,
                                  const float* gamma, const float* beta, int32_t silu, int32_t up2x, void* y, void* s) {
  if (int rc = check_gn_channels("groupnorm_apply", c0, c1, groups)) return rc;
  const long long hw = static_cast<long long>(h) * w;
  if (hw > 0x3fffffffLL) return fail(CA_ERR_INVALID, "groupnorm_apply: h * w (%lld) must be < 2^30", hw);
  const int C = c0 + c1;
  const int nvec = C >> 3;
  const int rows_per_iter = 512 / nvec;  // >= 1 because C <= 4096
  const int threads = rows_per_iter * nvec;
  // about 6 slabs per SM over the whole launch, each a multiple of the 4-row unrolled step
  long long want_blocks = (148LL * 6 + n - 1) / n;
  const long long step = 4LL * rows_per_iter;
  long long ppb = ((hw + want_blocks - 1) / want_blocks + step - 1) / step * step;
  if (ppb < 2 * step) ppb = 2 * step;
  const int slabs = static_cast<int>((hw + ppb - 1) / ppb);
  auto kern = silu ? (up2x ? gn_apply_kernel<true, true> : gn_apply_kernel<true, false>)
                   : (up2x ? gn_apply_kernel<false, true> : gn_apply_kernel<false, false>);
  const cudaError_t e = launch_pdl(kern, dim3(slabs, n), threads, 0, static_cast<cudaStream_t>(s),
                                   static_cast<const __nv_bfloat16*>(x0), c0, static_cast<const __nv_bfloat16*>(x1), c1,
                                   h, w, imgs_per_sample, groups, eps, sums, gamma, beta, static_cast<int>(ppb),
                                   static_cast<__nv_bfloat16*>(y));
  return launched(e, "groupnorm_apply");
}

// ---------------------------------------------------------------------------------------------
// LayerNorm.  A group of L lanes (8, 16 or 32) normalises one row, so a warp works on G = 32 / L consecutive rows at a
// time and every lane owns NV = ceil(C / 8 / L) 16-byte vectors of its row: C = 320 / 640 / 1280 all map to NV = 5
// with no idle lanes (L = 8 / 16 / 32).  Resident warps walk the G-row steps with a grid-wide stride.
//  * Each warp owns a three-step ring in shared memory that one lane fills with 1-D bulk copies (cp.async.bulk +
//    mbarrier; the G rows of a step are contiguous in memory): the next steps are in flight while the warp works, at
//    no register cost.
//  * The rows are NOT held in registers: both passes re-read their vectors from the stage.  The registers hold gamma
//    and beta instead (16 x NV per lane; a lane's columns are the same for every row).  Loading them per row ran the
//    kernel at the L1 rate: 8 bytes of fp32 gamma / beta per 2-byte element.
//  * Statistics in ONE pass over d = x - K with K = the row's first element: mean = K + sum(d)/C,
//    var = (sum(d^2) - sum(d)^2 / C) / C.  K is an element of the row, so (K - mean)^2 <= (C - 1) var and the
//    cancellation costs at most ~C ulp of fp32 in var (1.5e-4 relative at C = 1280), far below the bf16 output grid.
// RV: fused pre-add of a broadcast row vector (frame position embedding / single-token cross-attention output),
// rounded to bf16 like the eager add it replaces, written back into the stage; optionally also written out (y_sum).
// ---------------------------------------------------------------------------------------------
constexpr int kLnWarps = 8;
constexpr int kLnStages = 3;
constexpr int kLnHoldMaxNV = 5;   // gamma / beta stay in registers up to 5 vectors per lane; wider rows reload them
constexpr int kLnMaxC = 8 * 32 * 8;
constexpr int kLnRingMaxBytes = kLnWarps * kLnStages * (kLnMaxC * 2 + 8);  // widest step the launcher builds
__host__ __device__ constexpr int ln_blocks_per_sm(int nv) { return nv <= 2 ? 3 : (nv <= kLnHoldMaxNV ? 2 : 3); }

__device__ __forceinline__ uint4 lds128(uint32_t saddr) {  // volatile: the passes must not be merged into registers
  uint4 q;
  asm volatile("ld.shared.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(q.x), "=r"(q.y), "=r"(q.z), "=r"(q.w) : "r"(saddr));
  return q;
}
__device__ __forceinline__ void sts128(uint32_t saddr, const uint4& q) {
  asm volatile("st.shared.v4.u32 [%0], {%1, %2, %3, %4};" ::"r"(saddr), "r"(q.x), "r"(q.y), "r"(q.z), "r"(q.w)
               : "memory");
}

template <int NV, int L, bool RV>
__global__ void __launch_bounds__(kLnWarps * 32, ln_blocks_per_sm(NV))
layernorm_kernel(const __nv_bfloat16* __restrict__ x, long long rows, int c, float eps,
                 const float* __restrict__ gamma, const float* __restrict__ beta,
                 const __nv_bfloat16* __restrict__ add_rowvec, long long rows_per_vec,
                 __nv_bfloat16* __restrict__ y_sum, __nv_bfloat16* __restrict__ y) {
  constexpr bool kHold = NV <= kLnHoldMaxNV;
  constexpr int G = 32 / L;
  extern __shared__ __align__(128) uint8_t ln_smem[];
  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int sub = lane / L;   // which row of the step
  const int ll = lane % L;    // position inside the row's lane group
  const int nvec = c >> 3;
  const uint32_t row_bytes = static_cast<uint32_t>(c) * 2u;
  const uint32_t step_bytes = G * row_bytes;
  uint8_t* ring = ln_smem + static_cast<size_t>(warp) * kLnStages * step_bytes;
  uint64_t* bars = reinterpret_cast<uint64_t*>(ln_smem + static_cast<size_t>(kLnWarps) * kLnStages * step_bytes) +
                   warp * kLnStages;
  if (lane == 0) {
#pragma unroll
    for (int s = 0; s < kLnStages; ++s) mbar_init(&bars[s], 1);
    fence_mbar_init();
    fence_proxy_async_smem();
  }
  __syncwarp();
  auto load_gb = [&](int v, float (&g)[8], float (&b)[8]) {
    const float4 g0 = __ldg(reinterpret_cast<const float4*>(gamma + v * 8));
    const float4 g1 = __ldg(reinterpret_cast<const float4*>(gamma + v * 8) + 1);
    const float4 b0 = __ldg(reinterpret_cast<const float4*>(beta + v * 8));
    const float4 b1 = __ldg(reinterpret_cast<const float4*>(beta + v * 8) + 1);
    g[0] = g0.x; g[1] = g0.y; g[2] = g0.z; g[3] = g0.w; g[4] = g1.x; g[5] = g1.y; g[6] = g1.z; g[7] = g1.w;
    b[0] = b0.x; b[1] = b0.y; b[2] = b0.z; b[3] = b0.w; b[4] = b1.x; b[5] = b1.y; b[6] = b1.z; b[7] = b1.w;
  };
  // vector k of this lane is column block v = ll + L k; only the last k can fall off the end of the row
  auto has = [&](int k) { return k < NV - 1 || ll + L * k < nvec; };
  // parameters, not produced by the previous kernel: loaded ahead of the programmatic-launch wait
  [[maybe_unused]] float gg[kHold ? NV : 1][8], bb[kHold ? NV : 1][8];
  if constexpr (kHold) {
#pragma unroll
    for (int k = 0; k < NV; ++k) {
#pragma unroll
      for (int e = 0; e < 8; ++e) gg[k][e] = bb[k][e] = 0.f;
      if (has(k)) load_gb(ll + L * k, gg[k], bb[k]);
    }
  }
  CA_PDL_TRIGGER();
  CA_PDL_WAIT();
  // step counters are 32-bit (the launcher rejects rows >= 2^31); only the element offsets need 64 bits
  const int nrows = static_cast<int>(rows);
  const int steps = (nrows + G - 1) / G;
  const int step_stride = static_cast<int>(gridDim.x) * kLnWarps;
  const int step0 = static_cast<int>(blockIdx.x) * kLnWarps + warp;
  auto fill = [&](uint32_t stage, int step) {  // lane 0 only
    const int r0 = step * G;
    const int left = nrows - r0;
    const uint32_t bytes = static_cast<uint32_t>(left < G ? left : G) * row_bytes;
    mbar_arrive_expect_tx(&bars[stage], bytes);
    bulk_load_1d(ring + stage * step_bytes, x + static_cast<long long>(r0) * c, bytes, &bars[stage]);
  };
  if (lane == 0) {
#pragma unroll
    for (int s = 0; s < kLnStages; ++s)
      if (step0 + s * step_stride < steps) fill(s, step0 + s * step_stride);
  }
  const float inv_c = 1.f / static_cast<float>(c);
  uint32_t stage = 0, phase = 0;
  for (int step = step0; step < steps; step += step_stride) {
    const int row = step * G + sub;
    const bool row_ok = row < nrows;  // a short last step leaves stale bytes in the stage: computed on, never stored
    [[maybe_unused]] const __nv_bfloat16* av = RV ? add_rowvec + (static_cast<long long>(row_ok ? row : 0) / rows_per_vec) * c : nullptr;
    // this lane's vector k sits at srow + 16 L k
    const uint32_t srow = smem_u32(ring + stage * step_bytes) + sub * row_bytes + ll * 16;
    mbar_wait(&bars[stage], phase);
    // the shift K: the row's first element (after the row-vector add, when there is one)
    uint32_t kw;
    asm volatile("ld.shared.u32 %0, [%1];" : "=r"(kw) : "r"(srow - ll * 16));
    if constexpr (RV) kw = add_bf16x2(kw, __ldg(reinterpret_cast<const uint32_t*>(av)));
    const float shift = bf16lo_to_float(kw);
    // pass 1: sum and sum of squares of d = x - K (and the fused row-vector add), even / odd columns apart
    float s_lo = 0.f, s_hi = 0.f, ss_lo = 0.f, ss_hi = 0.f;
#pragma unroll
    for (int k = 0; k < NV; ++k) {
      if (has(k)) {
        uint4 q = lds128(srow + 16 * L * k);
        if constexpr (RV) {
          const int v = ll + L * k;
          const uint4 ua = __ldg(reinterpret_cast<const uint4*>(av + v * 8));
          q.x = add_bf16x2(q.x, ua.x);  // bf16(x + rowvec), one rounding
          q.y = add_bf16x2(q.y, ua.y);
          q.z = add_bf16x2(q.z, ua.z);
          q.w = add_bf16x2(q.w, ua.w);
          sts128(srow + 16 * L * k, q);  // pass 2 of this lane reads it back
          if (y_sum != nullptr && row_ok) *reinterpret_cast<uint4*>(y_sum + static_cast<long long>(row) * c + v * 8) = q;
        }
        const uint32_t wds[4] = {q.x, q.y, q.z, q.w};
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const float d_lo = __fadd_rn(bf16lo_to_float(wds[e]), -shift);
          const float d_hi = __fadd_rn(bf16hi_to_float(wds[e]), -shift);
          s_lo = __fadd_rn(s_lo, d_lo);
          s_hi = __fadd_rn(s_hi, d_hi);
          ss_lo = __fmaf_rn(d_lo, d_lo, ss_lo);
          ss_hi = __fmaf_rn(d_hi, d_hi, ss_hi);
        }
      }
    }
    float sd = s_lo + s_hi, sq = ss_lo + ss_hi;
#pragma unroll
    for (int o = L / 2; o > 0; o >>= 1) {
      sd += __shfl_xor_sync(0xffffffffu, sd, o);
      sq += __shfl_xor_sync(0xffffffffu, sq, o);
    }
    const float mean_d = sd * inv_c;
    const float var = fmaxf((sq - sd * mean_d) * inv_c, 0.f);
    const float mean = shift + mean_d;
    const float rstd = rsqrtf(var + eps);
    // pass 2: normalise, scale, shift, store
#pragma unroll
    for (int k = 0; k < NV; ++k) {
      if (has(k)) {
        const int v = ll + L * k;
        const uint4 q = lds128(srow + 16 * L * k);
        const uint32_t wds[4] = {q.x, q.y, q.z, q.w};
        float ge[8], be[8];
        if constexpr (kHold) {
#pragma unroll
          for (int i = 0; i < 8; ++i) { ge[i] = gg[k][i]; be[i] = bb[k][i]; }
        } else {
          load_gb(v, ge, be);
        }
        uint32_t o[4];
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          // ((x - mean) * rstd) * gamma + beta, the association of the eager kernel
          const float r0 = __fmaf_rn(__fmul_rn(__fadd_rn(bf16lo_to_float(wds[e]), -mean), rstd), ge[2 * e], be[2 * e]);
          const float r1 =
              __fmaf_rn(__fmul_rn(__fadd_rn(bf16hi_to_float(wds[e]), -mean), rstd), ge[2 * e + 1], be[2 * e + 1]);
          o[e] = pack_bf16x2(r0, r1);
        }
        if (row_ok) *reinterpret_cast<uint4*>(y + static_cast<long long>(row) * c + v * 8) = make_uint4(o[0], o[1], o[2], o[3]);
      }
    }
    __syncwarp();  // every lane is done with the stage: refill it with the step kLnStages ahead
    if (lane == 0) {
      const int nxt = step + kLnStages * step_stride;
      // no proxy fence: every lane has consumed what it read from (or, RV, wrote to and read back from) the stage
      // before the __syncwarp above, the same release convention as the TMA rings of the GEMM kernels; a fence here
      // is a MEMBAR that also waits for this lane's row stores
      if (nxt < steps) fill(stage, nxt);
    }
    if (++stage == kLnStages) {
      stage = 0;
      phase ^= 1u;
    }
  }
}

template <int NV, int L>
static cudaError_t launch_layernorm(const __nv_bfloat16* x, long long rows, int c, float eps, const float* gamma,
                                   const float* beta, const __nv_bfloat16* add_rowvec, long long rpv,
                                   __nv_bfloat16* y_sum, __nv_bfloat16* y, cudaStream_t stream) {
  constexpr int G = 32 / L;
  static bool optin = false;  // the ring can exceed the 48 KB default: opt both variants in once
  if (!optin) {
    cudaError_t e = cudaFuncSetAttribute(layernorm_kernel<NV, L, true>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         kLnRingMaxBytes);
    if (e == cudaSuccess)
      e = cudaFuncSetAttribute(layernorm_kernel<NV, L, false>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                               kLnRingMaxBytes);
    if (e != cudaSuccess) return e;
    optin = true;
  }
  const size_t smem = static_cast<size_t>(kLnWarps) * kLnStages * (static_cast<size_t>(G) * c * 2 + sizeof(uint64_t));
  // blocks that fit one SM: the launch bound or the shared-memory ring (228 KB per SM, 1 KB reserved per block)
  int per_sm = ln_blocks_per_sm(NV);
  const int by_smem = static_cast<int>((228u * 1024u) / (smem + 1024u));
  if (by_smem < per_sm) per_sm = by_smem;
  const long long resident = static_cast<long long>(num_sms()) * per_sm;
  const long long steps = (rows + G - 1) / G;
  const long long need = (steps + kLnWarps - 1) / kLnWarps;
  const unsigned blocks = static_cast<unsigned>(need < resident ? need : resident);
  auto kern = (add_rowvec != nullptr) ? layernorm_kernel<NV, L, true> : layernorm_kernel<NV, L, false>;
  return launch_pdl(kern, blocks, kLnWarps * 32, smem, stream, x, rows, c, eps, gamma, beta, add_rowvec, rpv, y_sum, y);
}

extern "C" int ca_layernorm(const void* x_, int64_t rows, int32_t c, float eps, const float* gamma, const float* beta,
                            const void* add_rowvec_, int64_t rows_per_vec, void* y_sum_, void* y_, void* s) {
  if ((c & 7) != 0 || c < 8 || c > kLnMaxC)
    return fail(CA_ERR_INVALID, "layernorm: c (%d) must be a multiple of 8 in 8..%d", c, kLnMaxC);
  // whole rows travel as 1-D bulk copies
  if ((reinterpret_cast<uintptr_t>(x_) & 15) != 0) return fail(CA_ERR_INVALID, "layernorm: x must be 16-byte aligned");
  if (rows <= 0) return CA_OK;
  if (rows >= (1LL << 31) - 64) return fail(CA_ERR_INVALID, "layernorm: rows (%lld) must be < 2^31 - 64", (long long)rows);
  const auto* x = static_cast<const __nv_bfloat16*>(x_);
  const auto* add_rowvec = static_cast<const __nv_bfloat16*>(add_rowvec_);
  auto* y_sum = static_cast<__nv_bfloat16*>(y_sum_);
  auto* y = static_cast<__nv_bfloat16*>(y_);
  cudaStream_t stream = static_cast<cudaStream_t>(s);
  const long long rpv = rows_per_vec > 0 ? rows_per_vec : 1;
  const int nvec = c >> 3;
  // the narrowest lane group that still keeps gamma / beta in registers
  int lanes = 32;
  if ((nvec + 7) / 8 <= kLnHoldMaxNV) lanes = 8;
  else if ((nvec + 15) / 16 <= kLnHoldMaxNV) lanes = 16;
  const int nv = (nvec + lanes - 1) / lanes;
#define CA_LN(NV, L) \
  return launched(launch_layernorm<NV, L>(x, rows, c, eps, gamma, beta, add_rowvec, rpv, y_sum, y, stream), "layernorm")
  if (lanes == 8) {
    switch (nv) {
      case 1: CA_LN(1, 8);
      case 2: CA_LN(2, 8);
      case 3: CA_LN(3, 8);
      case 4: CA_LN(4, 8);
      default: CA_LN(5, 8);
    }
  }
  if (lanes == 16) {  // nv is 3..5 here: 1 and 2 fit eight lanes
    switch (nv) {
      case 3: CA_LN(3, 16);
      case 4: CA_LN(4, 16);
      default: CA_LN(5, 16);
    }
  }
  switch (nv) {       // nv is 3..8: at most 2 would fit sixteen lanes
    case 3: CA_LN(3, 32);
    case 4: CA_LN(4, 32);
    case 5: CA_LN(5, 32);
    case 6: CA_LN(6, 32);
    case 7: CA_LN(7, 32);
    default: CA_LN(8, 32);
  }
#undef CA_LN
}

}  // namespace ca
