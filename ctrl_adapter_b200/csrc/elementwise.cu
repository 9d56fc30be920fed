// Small HBM-bound kernels of the denoising step and their entry points: timestep sinusoid, layout changes at the
// module boundary, pooling / up-sampling, router softmax + weighted merge, CFG + scheduler update, the I2VGen-XL latent
// encoder, the SVD decoder's frame convolution and the VAE's row softmax.  All vectorised to 16-byte accesses where the
// layout allows.
#include "common.cuh"
#include "kernels.h"

namespace ca {

static inline unsigned blocks_for(long long n, int threads, long long cap = 148LL * 32) {
  long long b = (n + threads - 1) / threads;
  if (b > cap) b = cap;
  if (b < 1) b = 1;
  return static_cast<unsigned>(b);
}

// ---------------------------------------------------------------------------------------------
// diffusers Timesteps: emb = [sin(t f_k), cos(t f_k)], f_k = exp(-ln(1e4) k / (half - shift)); flip -> [cos, sin]
// ---------------------------------------------------------------------------------------------
__global__ void timestep_embedding_kernel(const float* __restrict__ t, int n, int dim, int flip, float shift,
                                          int round_t, __nv_bfloat16* __restrict__ out) {
  CA_PDL_TRIGGER();
  CA_PDL_WAIT();
  const int half = dim / 2;
  const long long total = static_cast<long long>(n) * half;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int row = static_cast<int>(i / half), k = static_cast<int>(i % half);
    float tv = t[row];
    if (round_t) tv = round_bf16(tv);
    const float exponent = -9.210340371976184f * static_cast<float>(k) / (static_cast<float>(half) - shift);
    const float arg = tv * expf(exponent);
    const float sv = sinf(arg), cv = cosf(arg);
    __nv_bfloat16* o = out + static_cast<long long>(row) * dim;
    if (flip) { o[k] = __float2bfloat16_rn(cv); o[half + k] = __float2bfloat16_rn(sv); }
    else      { o[k] = __float2bfloat16_rn(sv); o[half + k] = __float2bfloat16_rn(cv); }
    if ((dim & 1) && k == 0) o[dim - 1] = __float2bfloat16_rn(0.f);
  }
}
extern "C" int ca_timestep_embedding(const float* t, int32_t n, int32_t dim, int32_t flip_sin_to_cos, float freq_shift,
                                     int32_t round_t_bf16, void* out, void* s) {
  // dim 1 has no sinusoid pair: the kernel would never write its one (zero) column
  if (dim < 2) return fail(CA_ERR_INVALID, "timestep_embedding: dim (%d) must be >= 2", dim);
  if (n < 1) return fail(CA_ERR_INVALID, "timestep_embedding: n (%d) must be positive", n);
  const long long total = static_cast<long long>(n) * (dim / 2);
  return launched(launch_pdl(timestep_embedding_kernel, blocks_for(total, 256), 256, 0, static_cast<cudaStream_t>(s), t,
                             n, dim, flip_sin_to_cos, freq_shift, round_t_bf16, static_cast<__nv_bfloat16*>(out)),
                  "timestep_embedding");
}

// ---------------------------------------------------------------------------------------------
// silu / add (bf16, 8 elements per thread; n must be a multiple of 8 -- all channel counts here are)
// ---------------------------------------------------------------------------------------------
__global__ void silu_kernel(const uint4* __restrict__ x, long long nvec, uint4* __restrict__ y) {
  CA_PDL_TRIGGER();
  CA_PDL_WAIT();
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < nvec;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const uint4 u = x[i];
    const __nv_bfloat16* h = reinterpret_cast<const __nv_bfloat16*>(&u);
    float f[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) { const float v = __bfloat162float(h[e]); f[e] = v / (1.0f + __expf(-v)); }
    y[i] = make_uint4(pack_bf16x2(f[0], f[1]), pack_bf16x2(f[2], f[3]), pack_bf16x2(f[4], f[5]), pack_bf16x2(f[6], f[7]));
  }
}
extern "C" int ca_silu(const void* x, int64_t n, void* y, void* s) {
  if (n & 7) return fail(CA_ERR_INVALID, "silu: n (%lld) must be a multiple of 8", (long long)n);
  if (!aligned(x, 16) || !aligned(y, 16)) return fail(CA_ERR_INVALID, "silu: x, y must be 16-byte aligned");
  return launched(launch_pdl(silu_kernel, blocks_for(n / 8, 256), 256, 0, static_cast<cudaStream_t>(s),
                             static_cast<const uint4*>(x), n / 8, static_cast<uint4*>(y)),
                  "silu");
}
__global__ void add_kernel(const uint4* __restrict__ a, const uint4* __restrict__ b, long long nvec,
                           uint4* __restrict__ y) {
  CA_PDL_TRIGGER();
  CA_PDL_WAIT();
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < nvec;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const uint4 ua = a[i], ub = b[i];
    const __nv_bfloat162* ha = reinterpret_cast<const __nv_bfloat162*>(&ua);
    const __nv_bfloat162* hb = reinterpret_cast<const __nv_bfloat162*>(&ub);
    uint4 o;
    uint32_t* po = reinterpret_cast<uint32_t*>(&o);
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const float2 fa = __bfloat1622float2(ha[e]), fb = __bfloat1622float2(hb[e]);
      po[e] = pack_bf16x2(fa.x + fb.x, fa.y + fb.y);
    }
    y[i] = o;
  }
}
extern "C" int ca_add(const void* a, const void* b, int64_t n, void* y, void* s) {
  if (n & 7) return fail(CA_ERR_INVALID, "add: n (%lld) must be a multiple of 8", (long long)n);
  if (!aligned(a, 16) || !aligned(b, 16) || !aligned(y, 16))
    return fail(CA_ERR_INVALID, "add: a, b, y must be 16-byte aligned");
  return launched(launch_pdl(add_kernel, blocks_for(n / 8, 256), 256, 0, static_cast<cudaStream_t>(s),
                             static_cast<const uint4*>(a), static_cast<const uint4*>(b), n / 8, static_cast<uint4*>(y)),
                  "add");
}

// ---------------------------------------------------------------------------------------------
// NCHW <-> channels-last transposes through a 32x33 smem tile (coalesced on both sides)
// ---------------------------------------------------------------------------------------------
template <typename SrcT>
__global__ void nchw_to_nhwc_kernel(const SrcT* __restrict__ x, int c, long long hw, int c_pad,
                                    __nv_bfloat16* __restrict__ y) {
  CA_PDL_TRIGGER();
  CA_PDL_WAIT();
  __shared__ float tile[32][33];
  const int n = blockIdx.z;
  const long long p0 = static_cast<long long>(blockIdx.x) * 32;
  const int c0 = blockIdx.y * 32;
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    const int ch = c0 + i;
    const long long p = p0 + threadIdx.x;
    float v = 0.f;
    if (ch < c && p < hw) v = static_cast<float>(x[(static_cast<long long>(n) * c + ch) * hw + p]);
    tile[i][threadIdx.x] = v;
  }
  __syncthreads();
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    const long long p = p0 + i;
    const int ch = c0 + threadIdx.x;
    if (p < hw && ch < c_pad) y[(static_cast<long long>(n) * hw + p) * c_pad + ch] = __float2bfloat16_rn(tile[threadIdx.x][i]);
  }
}
extern "C" int ca_nchw_to_nhwc(const void* x, int32_t src_fp32, int32_t n, int32_t c, int64_t hw, int32_t c_pad,
                               void* y_, void* s) {
  if (n < 1 || c < 1 || hw < 1) return fail(CA_ERR_INVALID, "nchw_to_nhwc: n, c, hw (%d, %d, %lld) must be positive", n, c,
                                            (long long)hw);
  // c > c_pad would drop channels without a word
  if (c_pad < c) return fail(CA_ERR_INVALID, "nchw_to_nhwc: c_pad (%d) must be >= c (%d)", c_pad, c);
  if (n > kMaxGridYZ || (static_cast<long long>(c_pad) + 31) / 32 > kMaxGridYZ || hw > 0xffffffffLL)
    return fail(CA_ERR_INVALID, "nchw_to_nhwc: n (%d) must be <= 65535, c_pad (%d) <= 65535 * 32 and hw (%lld) < 2^32",
                n, c_pad, (long long)hw);
  const dim3 grid(static_cast<unsigned>((hw + 31) / 32), (c_pad + 31) / 32, n), block(32, 8);
  cudaStream_t stream = static_cast<cudaStream_t>(s);
  __nv_bfloat16* y = static_cast<__nv_bfloat16*>(y_);
  const cudaError_t e =
      src_fp32 ? launch_pdl(nchw_to_nhwc_kernel<float>, grid, block, 0, stream, static_cast<const float*>(x), c, hw, c_pad, y)
               : launch_pdl(nchw_to_nhwc_kernel<__nv_bfloat16>, grid, block, 0, stream,
                            static_cast<const __nv_bfloat16*>(x), c, hw, c_pad, y);
  return launched(e, "nchw_to_nhwc");
}
template <typename DstT>
__global__ void nhwc_to_nchw_kernel(const __nv_bfloat16* __restrict__ x, int c, int c_stride, long long hw,
                                    DstT* __restrict__ y) {
  CA_PDL_TRIGGER();
  CA_PDL_WAIT();
  __shared__ float tile[32][33];
  const int n = blockIdx.z;
  const long long p0 = static_cast<long long>(blockIdx.x) * 32;
  const int c0 = blockIdx.y * 32;
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    const long long p = p0 + i;
    const int ch = c0 + threadIdx.x;
    float v = 0.f;
    if (p < hw && ch < c) v = __bfloat162float(x[(static_cast<long long>(n) * hw + p) * c_stride + ch]);
    tile[i][threadIdx.x] = v;
  }
  __syncthreads();
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    const int ch = c0 + i;
    const long long p = p0 + threadIdx.x;
    if (ch < c && p < hw) y[(static_cast<long long>(n) * c + ch) * hw + p] = static_cast<DstT>(tile[threadIdx.x][i]);
  }
}
extern "C" int ca_nhwc_to_nchw(const void* x_, int32_t n, int32_t c, int32_t c_stride, int64_t hw, void* y,
                               int32_t dst_fp32, void* s) {
  if (n < 1 || c < 1 || hw < 1) return fail(CA_ERR_INVALID, "nhwc_to_nchw: n, c, hw (%d, %d, %lld) must be positive", n, c,
                                            (long long)hw);
  // c > c_stride would read channel c_stride.. from the next pixel
  if (c_stride < c) return fail(CA_ERR_INVALID, "nhwc_to_nchw: c_stride (%d) must be >= c (%d)", c_stride, c);
  if (n > kMaxGridYZ || (static_cast<long long>(c) + 31) / 32 > kMaxGridYZ || hw > 0xffffffffLL)
    return fail(CA_ERR_INVALID, "nhwc_to_nchw: n (%d) must be <= 65535, c (%d) <= 65535 * 32 and hw (%lld) < 2^32", n, c,
                (long long)hw);
  const dim3 grid(static_cast<unsigned>((hw + 31) / 32), (c + 31) / 32, n), block(32, 8);
  cudaStream_t stream = static_cast<cudaStream_t>(s);
  const __nv_bfloat16* x = static_cast<const __nv_bfloat16*>(x_);
  const cudaError_t e =
      dst_fp32 ? launch_pdl(nhwc_to_nchw_kernel<float>, grid, block, 0, stream, x, c, c_stride, hw, static_cast<float*>(y))
               : launch_pdl(nhwc_to_nchw_kernel<__nv_bfloat16>, grid, block, 0, stream, x, c, c_stride, hw,
                            static_cast<__nv_bfloat16*>(y));
  return launched(e, "nhwc_to_nchw");
}

// ---------------------------------------------------------------------------------------------
// adaptive average pool with integer ratio, channels-last (C small: latents / control image)
// ---------------------------------------------------------------------------------------------
__global__ void avgpool_kernel(const __nv_bfloat16* __restrict__ x, int h, int w, int c, int oh, int ow,
                               long long total, __nv_bfloat16* __restrict__ y) {
  CA_PDL_TRIGGER();
  CA_PDL_WAIT();
  const int ry = h / oh, rx = w / ow;
  const float inv = 1.0f / static_cast<float>(ry * rx);
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int ch = static_cast<int>(i % c);
    long long t = i / c;
    const int ox = static_cast<int>(t % ow); t /= ow;
    const int oy = static_cast<int>(t % oh);
    const long long n = t / oh;
    float acc = 0.f;
    for (int dy = 0; dy < ry; ++dy)
      for (int dx = 0; dx < rx; ++dx)
        acc += __bfloat162float(x[((n * h + oy * ry + dy) * w + ox * rx + dx) * c + ch]);
    y[i] = __float2bfloat16_rn(acc * inv);
  }
}
extern "C" int ca_avgpool(const void* x, int32_t n, int32_t h, int32_t w, int32_t c, int32_t oh, int32_t ow, void* y,
                          void* s) {
  if (oh < 1 || ow < 1 || h % oh != 0 || w % ow != 0)
    return fail(CA_ERR_INVALID, "avgpool: h, w (%d, %d) must be positive multiples of oh, ow (%d, %d)", h, w, oh, ow);
  const long long total = static_cast<long long>(n) * oh * ow * c;
  return launched(launch_pdl(avgpool_kernel, blocks_for(total, 256), 256, 0, static_cast<cudaStream_t>(s),
                             static_cast<const __nv_bfloat16*>(x), h, w, c, oh, ow, total, static_cast<__nv_bfloat16*>(y)),
                  "avgpool");
}

__global__ void upsample2x_kernel(const uint4* __restrict__ x, int h, int w, int nvec, long long total,
                                  uint4* __restrict__ y) {
  CA_PDL_TRIGGER();
  CA_PDL_WAIT();
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int v = static_cast<int>(i % nvec);
    long long t = i / nvec;
    const int px = static_cast<int>(t % w); t /= w;
    const int py = static_cast<int>(t % h);
    const long long n = t / h;
    const uint4 u = x[i];
    const long long ow = 2LL * w;
    uint4* dst = y + ((n * 2 * h + 2 * py) * ow + 2 * px) * nvec + v;
    dst[0] = u; dst[nvec] = u; dst[ow * nvec] = u; dst[ow * nvec + nvec] = u;
  }
}
extern "C" int ca_upsample2x(const void* x, int32_t n, int32_t h, int32_t w, int32_t c, void* y, void* s) {
  if (c & 7) return fail(CA_ERR_INVALID, "upsample2x: c (%d) must be a multiple of 8", c);
  if (!aligned(x, 16) || !aligned(y, 16)) return fail(CA_ERR_INVALID, "upsample2x: x, y must be 16-byte aligned");
  const long long total = static_cast<long long>(n) * h * w * (c / 8);
  return launched(launch_pdl(upsample2x_kernel, blocks_for(total, 256), 256, 0, static_cast<cudaStream_t>(s),
                             static_cast<const uint4*>(x), h, w, c / 8, total, static_cast<uint4*>(y)),
                  "upsample2x");
}

// ---------------------------------------------------------------------------------------------
// Router: one warp per router; masked softmax over <= 32 experts by warp shuffles (ctrl_router.py:96-107)
// ---------------------------------------------------------------------------------------------
__global__ void router_weights_kernel(const float* __restrict__ logits, const unsigned char* __restrict__ mask,
                                      int nrouters, int nexperts, float* __restrict__ weights) {
  CA_PDL_TRIGGER();
  CA_PDL_WAIT();
  const int r = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (r >= nrouters) return;
  const int lane = threadIdx.x & 31;
  float v = -INFINITY;
  if (lane < nexperts) {
    v = logits[r * nexperts + lane];
    if (mask != nullptr && mask[lane] == 0) v -= 1e6f;
  }
  float mx = v;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  float e = (lane < nexperts) ? expf(v - mx) : 0.f;
  float s = e;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if (lane < nexperts) weights[r * nexperts + lane] = e / s;
}
extern "C" int ca_router_weights(const float* logits, const uint8_t* mask, int32_t nrouters, int32_t nexperts,
                                 float* weights, void* s) {
  if (nexperts < 1 || nexperts > 32) return fail(CA_ERR_INVALID, "router_weights: nexperts must be 1..32 (got %d)", nexperts);
  if (nrouters < 1) return fail(CA_ERR_INVALID, "router_weights: nrouters (%d) must be positive", nrouters);
  const int wpb = 4;
  return launched(launch_pdl(router_weights_kernel, (nrouters + wpb - 1) / wpb, wpb * 32, 0, static_cast<cudaStream_t>(s),
                             logits, mask, nrouters, nexperts, weights),
                  "router_weights");
}

// y = sum_e w[e] * x_e with the reference's bf16 rounding after each multiply and add
constexpr int kMaxRouterExperts = 8;
struct RouterSources {  // expert tensors by value: nothing to stage on the device, so the launch is graph-capturable
  const __nv_bfloat16* p[kMaxRouterExperts];
};
__global__ void router_merge_kernel(const __grid_constant__ RouterSources xs, const float* __restrict__ w,
                                    int nactive, long long nvec, uint4* __restrict__ y) {
  CA_PDL_TRIGGER();
  CA_PDL_WAIT();
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < nvec;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    float acc[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) acc[e] = 0.f;
    for (int k = 0; k < nactive; ++k) {
      const float wk = round_bf16(w[k]);
      const uint4 u = __ldg(reinterpret_cast<const uint4*>(xs.p[k]) + i);
      const __nv_bfloat16* h = reinterpret_cast<const __nv_bfloat16*>(&u);
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        const float prod = round_bf16(__bfloat162float(h[e]) * wk);
        acc[e] = (k == 0) ? prod : round_bf16(acc[e] + prod);
      }
    }
    y[i] = make_uint4(pack_bf16x2(acc[0], acc[1]), pack_bf16x2(acc[2], acc[3]), pack_bf16x2(acc[4], acc[5]),
                      pack_bf16x2(acc[6], acc[7]));
  }
}
extern "C" int ca_router_merge(const void* const* xs, const float* w, int32_t nactive, int64_t n, void* y, void* s) {
  if (nactive < 1 || nactive > kMaxRouterExperts)
    return fail(CA_ERR_INVALID, "router_merge: nactive must be 1..%d (got %d)", kMaxRouterExperts, nactive);
  if (n & 7) return fail(CA_ERR_INVALID, "router_merge: n (%lld) must be a multiple of 8", (long long)n);
  if (xs == nullptr) return fail(CA_ERR_INVALID, "router_merge: null xs array");
  RouterSources src{};
  for (int k = 0; k < nactive; ++k) {
    if (!aligned(xs[k], 16)) return fail(CA_ERR_INVALID, "router_merge: xs[%d] must be 16-byte aligned", k);
    src.p[k] = static_cast<const __nv_bfloat16*>(xs[k]);
  }
  if (!aligned(y, 16)) return fail(CA_ERR_INVALID, "router_merge: y must be 16-byte aligned");
  return launched(launch_pdl(router_merge_kernel, blocks_for(n / 8, 256), 256, 0, static_cast<cudaStream_t>(s), src, w,
                             nactive, n / 8, static_cast<uint4*>(y)),
                  "router_merge");
}

// ---------------------------------------------------------------------------------------------
// CFG + scheduler step in one pass.  The per-step scalars come from a device row {t, a, b, c} so that the whole
// denoising step can be captured once in a CUDA graph and replayed for every timestep.
// Rounding points follow the reference's bf16 pipeline (latents are bf16 between steps, the scheduler up-casts
// internally): eps = u + g*(c-u) in bf16 ops; Euler: x0 = x - bf16(sigma*eps) (0-dim fp32 sigma times a bf16
// tensor yields bf16), d = (x-x0)/sigma, x' = bf16(x + d*(sigma_next-sigma)); next model input = bf16(x'/div).
// ---------------------------------------------------------------------------------------------
// the operands every CFG + scheduler entry point dereferences (model_in_next may be NULL: no next model input)
static int check_cfg(const char* what, const void* eu, const void* et, const float* lat, long long n, const float* row,
                     const float* lat_out) {
  if (n < 0) return fail(CA_ERR_INVALID, "%s: n (%lld) must be >= 0", what, n);
  if (!eu || !et || !lat) return fail(CA_ERR_INVALID, "%s: null eps_uncond, eps_text or latents_in", what);
  if (!row) return fail(CA_ERR_INVALID, "%s: null step_row", what);
  if (!lat_out) return fail(CA_ERR_INVALID, "%s: null latents_out", what);
  return CA_OK;
}
__global__ void cfg_euler_kernel(const __nv_bfloat16* __restrict__ eu, const __nv_bfloat16* __restrict__ et,
                                 const float* __restrict__ lat, long long n, float g, const float* __restrict__ row,
                                 int round_lat, float* __restrict__ lat_out, __nv_bfloat16* __restrict__ next_in) {
  CA_PDL_TRIGGER();
  CA_PDL_WAIT();
  // A 0-dim fp32 tensor combined with a bf16 tensor is first cast to bf16 by PyTorch's type promotion, so the
  // reference multiplies eps by bf16(sigma) and divides the next model input by bf16(sqrt(sigma_next^2+1)).
  const float sigma = row[1], sigma_next = row[2], next_div = round_bf16(row[3]);
  const float sigma_b = round_bf16(sigma);
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < n;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const float u = __bfloat162float(eu[i]), c = __bfloat162float(et[i]);
    const float eps = round_bf16(u + round_bf16(g * round_bf16(c - u)));
    const float x = lat[i];
    const float x0 = x - round_bf16(sigma_b * eps);
    const float d = (x - x0) / sigma;
    float xn = x + d * (sigma_next - sigma);
    if (round_lat) xn = round_bf16(xn);
    lat_out[i] = xn;
    if (next_in) next_in[i] = __float2bfloat16_rn(xn / next_div);
  }
}
extern "C" int ca_cfg_euler(const void* eu, const void* et, const float* lat, int64_t n, float g, const float* step_row,
                            int32_t round_latents_bf16, float* lat_out, void* next_in, void* s) {
  if (int rc = check_cfg("cfg_euler", eu, et, lat, n, step_row, lat_out)) return rc;
  return launched(launch_pdl(cfg_euler_kernel, blocks_for(n, 256), 256, 0, static_cast<cudaStream_t>(s),
                             static_cast<const __nv_bfloat16*>(eu), static_cast<const __nv_bfloat16*>(et), lat, n, g,
                             step_row, round_latents_bf16, lat_out, static_cast<__nv_bfloat16*>(next_in)),
                  "cfg_euler");
}
// Euler, v-prediction, per-frame guidance (SVD loop, svd/pipelines/svd_controlnet_adapter_pipeline.py:781-787 with the
// diffusers v0.27.2 EulerDiscreteScheduler.step): row = {t, sigma, sigma_next, sqrt(sigma_next^2+1)};
// guidance[f] (bf16-valued) for frame f = (i / frame_elems) % frames of a [clips, frames, C, H, W] latent.
//   mo   = u + g_f (c - u)                                  (bf16 ops)
//   x0   = mo * bf16(-sigma / sqrt(sigma^2+1)) + x / (sigma^2+1)   (bf16 product, then fp32: the scheduler up-casts x)
//   x'   = x + (x - x0) / sigma * (sigma_next - sigma)      -> rounded to the model dtype
__global__ void cfg_euler_v_kernel(const __nv_bfloat16* __restrict__ eu, const __nv_bfloat16* __restrict__ et,
                                   const float* __restrict__ lat, long long n, const float* __restrict__ guidance,
                                   int frames, long long frame_elems, const float* __restrict__ row, int round_lat,
                                   float* __restrict__ lat_out, __nv_bfloat16* __restrict__ next_in) {
  CA_PDL_TRIGGER();
  CA_PDL_WAIT();
  const float sigma = row[1], sigma_next = row[2], next_div = round_bf16(row[3]);
  const float c_out = round_bf16(-sigma / sqrtf(sigma * sigma + 1.0f));
  const float c_skip_den = sigma * sigma + 1.0f;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < n;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const float g = guidance[(i / frame_elems) % frames];
    const float u = __bfloat162float(eu[i]), c = __bfloat162float(et[i]);
    const float mo = round_bf16(u + round_bf16(g * round_bf16(c - u)));
    const float x = lat[i];
    const float x0 = round_bf16(mo * c_out) + x / c_skip_den;
    const float d = (x - x0) / sigma;
    float xn = x + d * (sigma_next - sigma);
    if (round_lat) xn = round_bf16(xn);
    lat_out[i] = xn;
    if (next_in) next_in[i] = __float2bfloat16_rn(xn / next_div);
  }
}
extern "C" int ca_cfg_euler_v(const void* eu, const void* et, const float* lat, int64_t n, const float* guidance,
                              int32_t frames, int64_t frame_elems, const float* step_row, int32_t round_latents_bf16,
                              float* lat_out, void* next_in, void* s) {
  if (int rc = check_cfg("cfg_euler_v", eu, et, lat, n, step_row, lat_out)) return rc;
  if (!guidance) return fail(CA_ERR_INVALID, "cfg_euler_v: null guidance");
  if (frames < 1 || frame_elems < 1 || n % (static_cast<long long>(frames) * frame_elems) != 0)
    return fail(CA_ERR_INVALID, "cfg_euler_v: n (%lld) must be a multiple of frames * frame_elems (%d * %lld)",
                (long long)n, frames, (long long)frame_elems);
  return launched(launch_pdl(cfg_euler_v_kernel, blocks_for(n, 256), 256, 0, static_cast<cudaStream_t>(s),
                             static_cast<const __nv_bfloat16*>(eu), static_cast<const __nv_bfloat16*>(et), lat, n,
                             guidance, frames, frame_elems, step_row, round_latents_bf16, lat_out,
                             static_cast<__nv_bfloat16*>(next_in)),
                  "cfg_euler_v");
}
// DDIM (eta 0): row = {t, alpha_prod_t, alpha_prod_prev, -}; epsilon- or v-prediction model output
__global__ void cfg_ddim_kernel(const __nv_bfloat16* __restrict__ eu, const __nv_bfloat16* __restrict__ et,
                                const float* __restrict__ lat, long long n, float g, const float* __restrict__ row,
                                int round_lat, int vpred, float* __restrict__ lat_out,
                                __nv_bfloat16* __restrict__ next_in) {
  CA_PDL_TRIGGER();
  CA_PDL_WAIT();
  const float a_t = row[1], a_prev = row[2];
  float sa = sqrtf(a_t), sb = sqrtf(1.f - a_t), sap = sqrtf(a_prev), sbp = sqrtf(1.f - a_prev);
  if (round_lat) {
    // diffusers' DDIMScheduler.step does not up-cast: with bf16 latents every product / sum below is a bf16 op and the
    // 0-dim fp32 coefficients are cast to bf16 by type promotion before they are used
    sa = round_bf16(sa); sb = round_bf16(sb); sap = round_bf16(sap); sbp = round_bf16(sbp);
  }
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < n;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const float u = __bfloat162float(eu[i]), c = __bfloat162float(et[i]);
    const float mo = round_bf16(u + round_bf16(g * round_bf16(c - u)));  // guided model output
    const float x = lat[i];
    float x0, eps, xn;
    if (round_lat) {
      if (vpred) {
        x0 = round_bf16(round_bf16(sa * x) - round_bf16(sb * mo));
        eps = round_bf16(round_bf16(sa * mo) + round_bf16(sb * x));
      } else {
        x0 = round_bf16(round_bf16(x - round_bf16(sb * mo)) / sa);
        eps = mo;
      }
      xn = round_bf16(round_bf16(sap * x0) + round_bf16(sbp * eps));
    } else {
      if (vpred) {
        x0 = sa * x - sb * mo;
        eps = sa * mo + sb * x;
      } else {
        x0 = (x - sb * mo) / sa;
        eps = mo;
      }
      xn = sap * x0 + sbp * eps;
    }
    lat_out[i] = xn;
    if (next_in) next_in[i] = __float2bfloat16_rn(xn);
  }
}
extern "C" int ca_cfg_ddim(const void* eu, const void* et, const float* lat, int64_t n, float g, const float* step_row,
                           int32_t round_latents_bf16, int32_t v_prediction, float* lat_out, void* next_in, void* s) {
  if (int rc = check_cfg("cfg_ddim", eu, et, lat, n, step_row, lat_out)) return rc;
  return launched(launch_pdl(cfg_ddim_kernel, blocks_for(n, 256), 256, 0, static_cast<cudaStream_t>(s),
                             static_cast<const __nv_bfloat16*>(eu), static_cast<const __nv_bfloat16*>(et), lat, n, g,
                             step_row, round_latents_bf16, v_prediction, lat_out, static_cast<__nv_bfloat16*>(next_in)),
                  "cfg_ddim");
}

// ---------------------------------------------------------------------------------------------
// I2VGen-XL image-latent temporal encoder: one thread per (clip, pixel); sequence = F frames x 4 channels.
// LN(4) -> 2-head attention (head dim 4) -> +x -> FF (4 -> 16 GELU -> 4) -> +h.  bf16 rounding after each
// Linear / attention output as on the autocast path.  Tiny and step-invariant (run once per generation).
// ---------------------------------------------------------------------------------------------
__global__ void i2vgen_latent_encoder_kernel(const __nv_bfloat16* __restrict__ x, int frames, long long hw,
                                             int c_stride, const float* __restrict__ prm, long long total,
                                             __nv_bfloat16* __restrict__ y) {
  CA_PDL_TRIGGER();
  CA_PDL_WAIT();
  __shared__ float sp[288];
  for (int i = threadIdx.x; i < 288; i += blockDim.x) sp[i] = prm[i];
  __syncthreads();
  const float* ln_w = sp; const float* ln_b = sp + 4; const float* wq = sp + 8; const float* wk = sp + 40;
  const float* wv = sp + 72; const float* wo = sp + 104; const float* bo = sp + 136; const float* w1 = sp + 140;
  const float* b1 = sp + 204; const float* w2 = sp + 220;
  // layout: ln_w[4] ln_b[4] wq[32] wk[32] wv[32] wo[32] bo[4] w1[64] b1[16] w2[64] b2[4]  (total 288)
  const long long idx = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;
  if (idx >= total) return;
  const long long pix = idx % hw, clip = idx / hw;
  const long long fstride = hw * c_stride;
  const __nv_bfloat16* xb = x + (clip * frames * hw + pix) * c_stride;
  __nv_bfloat16* yb = y + (clip * frames * hw + pix) * c_stride;
  float xin[32][4], q[32][8], k[32][8], v[32][8];
  for (int f = 0; f < frames; ++f) {
    float m = 0.f;
    for (int c = 0; c < 4; ++c) { xin[f][c] = __bfloat162float(xb[f * fstride + c]); m += xin[f][c]; }
    m *= 0.25f;
    float var = 0.f;
    for (int c = 0; c < 4; ++c) { const float d = xin[f][c] - m; var += d * d; }
    const float rstd = rsqrtf(var * 0.25f + 1e-5f);
    float n4[4];
    for (int c = 0; c < 4; ++c) n4[c] = round_bf16((xin[f][c] - m) * rstd * ln_w[c] + ln_b[c]);
    for (int o = 0; o < 8; ++o) {
      float aq = 0.f, ak = 0.f, av = 0.f;
      for (int c = 0; c < 4; ++c) { aq += wq[o * 4 + c] * n4[c]; ak += wk[o * 4 + c] * n4[c]; av += wv[o * 4 + c] * n4[c]; }
      q[f][o] = round_bf16(aq); k[f][o] = round_bf16(ak); v[f][o] = round_bf16(av);
    }
  }
  for (int f = 0; f < frames; ++f) {
    float att[8];
    for (int hd = 0; hd < 2; ++hd) {
      float s[32], mx = -INFINITY;
      for (int g2 = 0; g2 < frames; ++g2) {
        float d = 0.f;
        for (int e = 0; e < 4; ++e) d += q[f][hd * 4 + e] * k[g2][hd * 4 + e];
        s[g2] = d * 0.5f;  // head dim 4 -> scale 4^-0.5
        mx = fmaxf(mx, s[g2]);
      }
      float l = 0.f, o4[4] = {0.f, 0.f, 0.f, 0.f};
      for (int g2 = 0; g2 < frames; ++g2) {
        const float pe = __expf(s[g2] - mx);
        l += pe;
        for (int e = 0; e < 4; ++e) o4[e] += pe * v[g2][hd * 4 + e];
      }
      for (int e = 0; e < 4; ++e) att[hd * 4 + e] = round_bf16(o4[e] / l);
    }
    float h4[4];
    for (int c = 0; c < 4; ++c) {
      float a = bo[c];
      for (int o = 0; o < 8; ++o) a += wo[c * 8 + o] * att[o];
      h4[c] = round_bf16(round_bf16(a) + xin[f][c]);
    }
    float u16[16];
    for (int j = 0; j < 16; ++j) {
      float a = b1[j];
      for (int c = 0; c < 4; ++c) a += w1[j * 4 + c] * h4[c];
      a = round_bf16(a);
      u16[j] = round_bf16(0.5f * a * (1.0f + erff(a * 0.70710678118654752440f)));
    }
    const float* b2p = sp + 284;
    for (int c = 0; c < 4; ++c) {
      float a = b2p[c];
      for (int j = 0; j < 16; ++j) a += w2[c * 16 + j] * u16[j];
      yb[f * fstride + c] = __float2bfloat16_rn(round_bf16(a) + h4[c]);
    }
  }
}
extern "C" int ca_i2vgen_latent_encoder(const void* x, int32_t clips, int32_t frames, int64_t hw, int32_t c_stride,
                                        const float* params, void* y, void* s) {
  if (frames < 1 || frames > 32) return fail(CA_ERR_INVALID, "i2vgen_latent_encoder: frames must be 1..32 (got %d)", frames);
  if (c_stride < 4) return fail(CA_ERR_INVALID, "i2vgen_latent_encoder: c_stride (%d) must be >= 4", c_stride);
  if (clips < 1 || hw < 1)
    return fail(CA_ERR_INVALID, "i2vgen_latent_encoder: clips, hw (%d, %lld) must be positive", clips, (long long)hw);
  const long long total = static_cast<long long>(clips) * hw;
  return launched(launch_pdl(i2vgen_latent_encoder_kernel, static_cast<unsigned>((total + 63) / 64), 64, 0,
                             static_cast<cudaStream_t>(s), static_cast<const __nv_bfloat16*>(x), frames, hw, c_stride,
                             params, total, static_cast<__nv_bfloat16*>(y)),
                  "i2vgen_latent_encoder");
}

// ---------------------------------------------------------------------------------------------
// Conv3d (3,1,1), padding (1,0,0) over the frame axis for a handful of channels: the SVD temporal decoder's
// time_conv_out (3 -> 3 on the decoded RGB frames; diffusers TemporalDecoder.forward, reached from the svd pipeline's
// decode_latents :265-292).  Far too narrow for the tensor-core GEMM (K = 9), and HBM-bound: one thread per pixel pair
// reads the (up to) three frames' 16-byte channel vectors of conv_out's zero-padded channels-last output and writes the
// planes of the logical NCHW result directly (the layout conversion is fused).  fp32 accumulation, one rounding to bf16.
// The 27 + 3 parameters travel in the kernel parameter space.
// ---------------------------------------------------------------------------------------------
constexpr int kFrameConvMaxC = 4;
struct FrameConvSmallParams {
  float w[kFrameConvMaxC][kFrameConvMaxC][3];  // [out channel][in channel][frame tap]
  float b[kFrameConvMaxC];
};
__global__ void __launch_bounds__(256)
frame_conv_small_kernel(const __nv_bfloat16* __restrict__ x, int frames, long long hw, int c_stride, int cin, int cout,
                        FrameConvSmallParams prm, __nv_bfloat16* __restrict__ y) {
  CA_PDL_TRIGGER();
  CA_PDL_WAIT();
  const long long img = blockIdx.y;           // clip * frames + f
  const int f = static_cast<int>(img % frames);
  const long long p0 = (static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x) * 2;
  if (p0 >= hw) return;
  const bool two = p0 + 1 < hw;
  float acc[2][kFrameConvMaxC];
#pragma unroll
  for (int co = 0; co < kFrameConvMaxC; ++co) acc[0][co] = acc[1][co] = prm.b[co];
#pragma unroll
  for (int dt = 0; dt < 3; ++dt) {
    const int fs = f + dt - 1;
    if (fs < 0 || fs >= frames) continue;     // zero padding in time
    const __nv_bfloat16* src = x + ((img + dt - 1) * hw + p0) * c_stride;
#pragma unroll
    for (int q = 0; q < 2; ++q) {
      if (q == 1 && !two) break;
      const uint2 u = *reinterpret_cast<const uint2*>(src + static_cast<long long>(q) * c_stride);  // channels 0..3
      const float xv[4] = {bf16lo_to_float(u.x), bf16hi_to_float(u.x), bf16lo_to_float(u.y), bf16hi_to_float(u.y)};
#pragma unroll
      for (int co = 0; co < kFrameConvMaxC; ++co)
#pragma unroll
        for (int ci = 0; ci < kFrameConvMaxC; ++ci)
          if (co < cout && ci < cin) acc[q][co] = fmaf(prm.w[co][ci][dt], xv[ci], acc[q][co]);
    }
  }
#pragma unroll
  for (int co = 0; co < kFrameConvMaxC; ++co) {
    if (co >= cout) break;
    __nv_bfloat16* dst = y + (img * cout + co) * hw + p0;
    if (two && (hw & 1) == 0) {
      *reinterpret_cast<uint32_t*>(dst) = pack_bf16x2(acc[0][co], acc[1][co]);
    } else {
      dst[0] = __float2bfloat16_rn(acc[0][co]);
      if (two) dst[1] = __float2bfloat16_rn(acc[1][co]);
    }
  }
}
extern "C" int ca_frame_conv_small(const void* x, int32_t clips, int32_t frames, int64_t hw, int32_t c_stride,
                                   int32_t cin, int32_t cout, const float* w_host, const float* bias_host, void* y,
                                   void* s) {
  if (w_host == nullptr) return fail(CA_ERR_INVALID, "frame_conv_small: null weight pointer");
  if (cin < 1 || cout < 1 || cin > kFrameConvMaxC || cout > kFrameConvMaxC)
    return fail(CA_ERR_INVALID, "frame_conv_small: cin, cout (%d, %d) must be 1..%d", cin, cout, kFrameConvMaxC);
  if (c_stride < 4 || (c_stride & 3) != 0)
    return fail(CA_ERR_INVALID, "frame_conv_small: c_stride (%d) must be a positive multiple of 4", c_stride);
  // 8-byte loads of channels 0..3, 4-byte stores of pixel pairs
  if (!aligned(x, 8) || !aligned(y, 4)) return fail(CA_ERR_INVALID, "frame_conv_small: x must be 8-byte and y 4-byte aligned");
  if (clips < 1 || frames < 1 || hw < 1 || static_cast<long long>(clips) * frames > 65535)
    return fail(CA_ERR_INVALID, "frame_conv_small: clips, frames, hw (%d, %d, %lld) must be positive with clips * frames "
                "<= 65535", clips, frames, (long long)hw);
  FrameConvSmallParams prm = {};
  for (int co = 0; co < cout; ++co) {
    prm.b[co] = bias_host != nullptr ? bias_host[co] : 0.f;
    for (int ci = 0; ci < cin; ++ci)
      for (int dt = 0; dt < 3; ++dt) prm.w[co][ci][dt] = w_host[(co * cin + ci) * 3 + dt];
  }
  const dim3 grid(static_cast<unsigned>((hw + 511) / 512), static_cast<unsigned>(clips * frames));
  return launched(launch_pdl(frame_conv_small_kernel, grid, 256, 0, static_cast<cudaStream_t>(s),
                             static_cast<const __nv_bfloat16*>(x), frames, hw, c_stride, cin, cout, prm,
                             static_cast<__nv_bfloat16*>(y)),
                  "frame_conv_small");
}

// ---------------------------------------------------------------------------------------------
// Row softmax, fp32 scores -> bf16 probabilities: the VAE decoder's single 512-wide attention head (diffusers
// AutoencoderKL mid block) is run as  S = Q K^T (tensor-core GEMM, fp32 out)  ->  this kernel  ->  O = P V (GEMM); its
// head dim is outside attention_kernel's 64 / 128 / 192 and it runs once per generation, not per step.  One CTA per
// row, three passes over the row (max, sum, write); the row (<= 64 KB) stays in L1 / L2 between them.
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
softmax_rows_kernel(const float* __restrict__ x, long long cols, __nv_bfloat16* __restrict__ y) {
  CA_PDL_TRIGGER();
  CA_PDL_WAIT();
  __shared__ float red[8];
  const float4* row = reinterpret_cast<const float4*>(x + static_cast<long long>(blockIdx.x) * cols);
  uint2* out = reinterpret_cast<uint2*>(y + static_cast<long long>(blockIdx.x) * cols);
  const long long nv = cols >> 2;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  auto block_reduce = [&](float v, bool is_max) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float t = __shfl_xor_sync(0xffffffffu, v, o);
      v = is_max ? fmaxf(v, t) : v + t;
    }
    __syncthreads();
    if (lane == 0) red[warp] = v;
    __syncthreads();
    v = red[0];
#pragma unroll
    for (int i = 1; i < 8; ++i) v = is_max ? fmaxf(v, red[i]) : v + red[i];
    return v;
  };
  float m = -INFINITY;
  for (long long i = threadIdx.x; i < nv; i += 256) {
    const float4 v = row[i];
    m = fmaxf(m, fmaxf(fmaxf(v.x, v.y), fmaxf(v.z, v.w)));
  }
  m = block_reduce(m, true);
  float l = 0.f;
  for (long long i = threadIdx.x; i < nv; i += 256) {
    const float4 v = row[i];
    l += __expf(v.x - m) + __expf(v.y - m) + __expf(v.z - m) + __expf(v.w - m);
  }
  l = block_reduce(l, false);
  const float inv = 1.0f / l;
  for (long long i = threadIdx.x; i < nv; i += 256) {
    const float4 v = row[i];
    out[i] = make_uint2(pack_bf16x2(__expf(v.x - m) * inv, __expf(v.y - m) * inv),
                        pack_bf16x2(__expf(v.z - m) * inv, __expf(v.w - m) * inv));
  }
}
extern "C" int ca_softmax_rows(const float* x, int64_t rows, int64_t cols, void* y, void* s) {
  if (rows < 1 || rows > 0x7fffffffLL) return fail(CA_ERR_INVALID, "softmax_rows: rows (%lld) must be 1..2^31-1", (long long)rows);
  if (cols < 4 || (cols & 3) != 0) return fail(CA_ERR_INVALID, "softmax_rows: cols (%lld) must be a positive multiple of 4", (long long)cols);
  // float4 row loads, 8-byte stores of four probabilities
  if (!aligned(x, 16) || !aligned(y, 8)) return fail(CA_ERR_INVALID, "softmax_rows: x must be 16-byte and y 8-byte aligned");
  return launched(launch_pdl(softmax_rows_kernel, static_cast<unsigned>(rows), 256, 0, static_cast<cudaStream_t>(s), x,
                             cols, static_cast<__nv_bfloat16*>(y)),
                  "softmax_rows");
}

// ---------------------------------------------------------------------------------------------
// VAE encoder posterior -> image latents (diffusers DiagonalGaussianDistribution on the quant_conv output, then the
// image-latent assembly of the two video pipelines).  moments: channels-last bf16 [n, hw, 8] = (mean[4], logvar[4]);
// noise: optional fp32 NCHW [n, 4, hw].  v = mean + exp(0.5 * clamp(logvar, -30, 20)) * noise (v = mean without noise),
// fp32, one rounding to bf16 at the store.  One thread per (output batch row, pixel): it reads one 16-byte moment
// vector and writes its 4 channels into every frame the row has.
//   CA_VAE_POSTERIOR  out [n, 4, hw]: v
//   CA_VAE_I2VGEN     out [2*n*nv, 4, F, hw]: frame 0 = v * scale, frame k >= 1 = k / (F - 1); row r holds image r % n
//   CA_VAE_SVD        out [2*n*nv, F, 4, hw]: row r holds 0 when r % 2n < n, else image r % 2n - n (every frame)
// ---------------------------------------------------------------------------------------------
__global__ void vae_latents_kernel(const uint4* __restrict__ moments, const float* __restrict__ noise, int n,
                                   long long hw, int layout, int frames, long long rows, float scale,
                                   __nv_bfloat16* __restrict__ out) {
  CA_PDL_TRIGGER();
  CA_PDL_WAIT();
  const long long total = rows * hw;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long p = i % hw, r = i / hw;
    long long img = r % n;
    bool zero = false;
    if (layout == CA_VAE_SVD) {
      const long long q = r % (2LL * n);
      zero = q < n;
      img = zero ? 0 : q - n;
    }
    float v[4] = {0.f, 0.f, 0.f, 0.f};
    if (!zero) {
      const uint4 u = moments[img * hw + p];
      const float mean[4] = {bf16lo_to_float(u.x), bf16hi_to_float(u.x), bf16lo_to_float(u.y), bf16hi_to_float(u.y)};
      const float logvar[4] = {bf16lo_to_float(u.z), bf16hi_to_float(u.z), bf16lo_to_float(u.w), bf16hi_to_float(u.w)};
#pragma unroll
      for (int c = 0; c < 4; ++c) {
        v[c] = mean[c];
        if (noise != nullptr) {
          const float std = expf(0.5f * fminf(fmaxf(logvar[c], -30.f), 20.f));
          v[c] = fmaf(std, noise[(img * 4 + c) * hw + p], mean[c]);
        }
      }
    }
    if (layout == CA_VAE_I2VGEN) {
      __nv_bfloat16* o = out + r * 4LL * frames * hw + p;
#pragma unroll
      for (int c = 0; c < 4; ++c) {
        o[static_cast<long long>(c) * frames * hw] = __float2bfloat16_rn(v[c] * scale);
        for (int f = 1; f < frames; ++f)
          o[(static_cast<long long>(c) * frames + f) * hw] =
              __float2bfloat16_rn(static_cast<float>(f) / static_cast<float>(frames - 1));
      }
    } else {
      // CA_VAE_POSTERIOR has frames == 1: both layouts are [row, frame, channel, pixel]
      for (int f = 0; f < frames; ++f) {
        __nv_bfloat16* o = out + (r * frames + f) * 4LL * hw + p;
#pragma unroll
        for (int c = 0; c < 4; ++c) o[c * hw] = __float2bfloat16_rn(v[c]);
      }
    }
  }
}
extern "C" int ca_vae_latents(const void* moments, const float* noise, int32_t n, int64_t hw, int32_t latent_channels,
                              int32_t layout, int32_t frames, int32_t num_videos, float scale, void* out, void* s) {
  if (moments == nullptr) return fail(CA_ERR_INVALID, "vae_latents: null moments pointer");
  if (out == nullptr) return fail(CA_ERR_INVALID, "vae_latents: null out pointer");
  if (!aligned(moments, 16)) return fail(CA_ERR_INVALID, "vae_latents: moments must be 16-byte aligned");
  if (latent_channels != 4)
    return fail(CA_ERR_INVALID, "vae_latents: latent_channels (%d) must be 4 (moments carry 8 channels)", latent_channels);
  if (layout < CA_VAE_POSTERIOR || layout > CA_VAE_SVD)
    return fail(CA_ERR_INVALID, "vae_latents: layout (%d) must be 0, 1 or 2", layout);
  if (n < 1 || hw < 1) return fail(CA_ERR_INVALID, "vae_latents: n, hw (%d, %lld) must be positive", n, (long long)hw);
  if (frames < 1) return fail(CA_ERR_INVALID, "vae_latents: frames (%d) must be positive", frames);
  if (num_videos < 1) return fail(CA_ERR_INVALID, "vae_latents: num_videos (%d) must be positive", num_videos);
  if (layout == CA_VAE_POSTERIOR && (frames != 1 || num_videos != 1))
    return fail(CA_ERR_INVALID, "vae_latents: frames, num_videos (%d, %d) must be 1 for the posterior layout", frames,
                num_videos);
  const long long rows = layout == CA_VAE_POSTERIOR ? n : 2LL * n * num_videos;
  return launched(launch_pdl(vae_latents_kernel, blocks_for(rows * hw, 256), 256, 0, static_cast<cudaStream_t>(s),
                             static_cast<const uint4*>(moments), noise, n, hw, layout, frames, rows, scale,
                             static_cast<__nv_bfloat16*>(out)),
                  "vae_latents");
}

}  // namespace ca
