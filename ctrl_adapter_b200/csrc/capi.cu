// extern "C" entry points declared in include/ctrl_adapter_b200.h: argument validation, TMA tensor-map
// encoding and kernel launches.  cuTensorMapEncodeTiled is resolved at run time through the CUDA runtime
// (cudaGetDriverEntryPoint) so the library has no link-time dependency on libcuda and can be dlopen'ed
// (symbol check) on a machine without a driver.
#include <stdarg.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include "kernels.h"

namespace {

thread_local char g_err[512] = "";

int fail(int code, const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
  return code;
}
int cuda_fail(cudaError_t e, const char* what) {
  return fail(CA_ERR_CUDA, "%s: %s", what, cudaGetErrorString(e));
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

EncodeTiledFn get_encode_fn() {
  static EncodeTiledFn fn = nullptr;
  static bool tried = false;
  if (!tried) {
    tried = true;
    void* p = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) == cudaSuccess &&
        qres == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(p);
  }
  return fn;
}

// bf16 tensor map, 128B swizzle, zero OOB fill. dims/strides fastest-first; strides in BYTES for dims 1..rank-1.
int make_tmap(CUtensorMap* m, const void* base, int rank, const cuuint64_t* dims, const cuuint64_t* strides_bytes,
              const cuuint32_t* box) {
  EncodeTiledFn fn = get_encode_fn();
  if (!fn) return fail(CA_ERR_CUDA, "cuTensorMapEncodeTiled unavailable (no CUDA driver?)");
  cuuint32_t estr[5] = {1, 1, 1, 1, 1};
  if ((reinterpret_cast<uintptr_t>(base) & 15) != 0) return fail(CA_ERR_INVALID, "tensor base not 16-byte aligned");
  for (int i = 0; i + 1 < rank; ++i)
    if (strides_bytes[i] % 16 != 0) return fail(CA_ERR_INVALID, "tensor stride %d (%llu B) not a multiple of 16", i + 1,
                                                (unsigned long long)strides_bytes[i]);
  CUresult r = fn(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, rank, const_cast<void*>(base), dims, strides_bytes, box, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    return fail(CA_ERR_CUDA,
                "cuTensorMapEncodeTiled failed (%d): rank %d dims [%llu %llu %llu %llu %llu] box [%u %u %u %u %u]",
                (int)r, rank, (unsigned long long)dims[0], (unsigned long long)(rank > 1 ? dims[1] : 0),
                (unsigned long long)(rank > 2 ? dims[2] : 0), (unsigned long long)(rank > 3 ? dims[3] : 0),
                (unsigned long long)(rank > 4 ? dims[4] : 0), box[0], rank > 1 ? box[1] : 0, rank > 2 ? box[2] : 0,
                rank > 3 ? box[3] : 0, rank > 4 ? box[4] : 0);
  }
  return CA_OK;
}

int num_sms() {
  static int sms = 0;
  if (sms == 0) {
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) return 132;
    if (cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || sms <= 0) sms = 132;
  }
  return sms;
}

#define CA_LAUNCH(expr, what)                      \
  do {                                             \
    cudaError_t _e = (expr);                       \
    if (_e != cudaSuccess) return cuda_fail(_e, what); \
    return CA_OK;                                  \
  } while (0)

// developer instrumentation (only read by -DCA_TRACE builds): device buffer of 16 u64 counters per CTA
unsigned long long* trace_ptr() {
  static const char* env = getenv("CA_GEMM_TRACE_PTR");
  static unsigned long long* ptr = env ? reinterpret_cast<unsigned long long*>(strtoull(env, nullptr, 0)) : nullptr;
  return ptr;
}

}  // namespace

extern "C" {

int ca_abi_version(void) { return CA_ABI_VERSION; }
const char* ca_last_error(void) { return g_err; }

int ca_device_ok(void) {
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess || n <= 0) return fail(CA_ERR_CUDA, "no CUDA device");
  int dev = 0, major = 0;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, dev);
  if (major != 9) return fail(CA_ERR_UNSUPPORTED, "device compute capability %d.x, need 9.x (sm_90a)", major);
  return CA_OK;
}

int ca_gemm(const ca_gemm_desc* d, void* cuda_stream) {
  if (!d) return fail(CA_ERR_INVALID, "null desc");
  cudaStream_t stream = static_cast<cudaStream_t>(cuda_stream);
  if (d->nsrc < 1 || d->nsrc > 2) return fail(CA_ERR_INVALID, "nsrc must be 1 or 2");
  if (d->ntaps < 1 || d->ntaps > CA_MAX_TAPS) return fail(CA_ERR_INVALID, "ntaps out of range");
  if (d->box[0] < 1 || d->box[1] < 1 || d->box[2] < 1 || d->box[3] < 1 ||
      d->box[0] * d->box[1] * d->box[2] * d->box[3] != 128)
    return fail(CA_ERR_INVALID, "box extents must be positive with product 128");
  if (!d->a[0] || !d->w || !d->out) return fail(CA_ERR_INVALID, "null tensor pointer");
  const bool geglu = d->act == CA_ACT_GEGLU;
  if (geglu && d->n_out * 2 != d->w_rows) return fail(CA_ERR_INVALID, "GEGLU needs w_rows == 2*n_out");
  if (!geglu && d->n_out != d->w_rows) return fail(CA_ERR_INVALID, "n_out must equal w_rows");
  if ((d->n_out & 7) != 0 && !d->out_fp32) return fail(CA_ERR_INVALID, "n_out must be a multiple of 8");
  if (geglu && d->out_fp32) return fail(CA_ERR_UNSUPPORTED, "GEGLU output is bf16");
  // the fp32 epilogue has no blend term: refuse rather than silently return the unblended result
  if (d->blend_src && d->out_fp32) return fail(CA_ERR_UNSUPPORTED, "AlphaBlender (blend_src) output is bf16");

  ca::GemmParams p;
  memset(&p, 0, sizeof(p));
  int bn = d->bn;
  if (bn == 0) {
    if (geglu) bn = 256;
    else if (d->w_rows % 256 == 0) bn = 256;
    else if (d->w_rows % 160 == 0) bn = 160;
    else if (d->w_rows % 128 == 0) bn = 128;
    else if (d->w_rows <= 64) bn = 64;
    else if (d->w_rows <= 128) bn = 128;
    else bn = 256;
  }
  if (bn != 64 && bn != 128 && bn != 160 && bn != 256) return fail(CA_ERR_INVALID, "bn must be 0, 64, 128, 160 or 256");
  if (geglu && (d->w_rows % bn) != 0) return fail(CA_ERR_INVALID, "GEGLU needs w_rows %% bn == 0");

  int k_per_tap = 0;
  for (int s = 0; s < d->nsrc; ++s) {
    if (d->a_c_len[s] <= 0 || (d->a_c_off[s] & 7) != 0) return fail(CA_ERR_INVALID, "bad channel slice");
    if (s == 0 && d->nsrc == 2 && (d->a_c_len[0] % 64) != 0)
      return fail(CA_ERR_INVALID, "first of two sources must contribute a multiple of 64 channels");
    p.src_c[s] = d->a_c_len[s];
    p.src_c0_off[s] = d->a_c_off[s];
    k_per_tap += d->a_c_len[s];
  }
  p.nsrc = d->nsrc;
  if (d->w_k_per_tap < k_per_tap) return fail(CA_ERR_INVALID, "w_k_per_tap smaller than the A channels per tap");
  k_per_tap = d->w_k_per_tap;
  p.k_per_tap = k_per_tap;
  p.ntaps = d->ntaps;
  for (int t = 0; t < d->ntaps; ++t) {
    for (int i = 0; i < 4; ++i) p.tap_off[t][i] = d->tap_off[t][i];
    p.tap_c_off[t] = d->tap_c_off[t];
    if (d->tap_c_off[t] != 0 && (k_per_tap % 64) != 0)
      return fail(CA_ERR_INVALID, "tap_c_off needs w_k_per_tap %% 64 == 0");
  }
  for (int i = 0; i < 4; ++i) {
    p.box[i] = d->box[i];
    p.odim[i] = d->out_dims[i];
    p.ntile[i] = (d->out_dims[i] + d->box[i] - 1) / d->box[i];
    p.ostride[i] = d->out_strides[i];
    p.rstride[i] = d->res_strides[i];
    p.vstride[i] = d->rowvec_strides[i];
  }
  p.n_out = d->n_out;
  p.n_tiles_n = (d->w_rows + bn - 1) / bn;
  p.act = d->act;
  p.out_fp32 = d->out_fp32;
  p.out_scale = d->out_scale;
  p.bias = d->bias;
  p.rowvec = static_cast<const __nv_bfloat16*>(d->rowvec);
  p.residual = static_cast<const __nv_bfloat16*>(d->residual);
  p.blend_src = static_cast<const __nv_bfloat16*>(d->blend_src);
  p.blend_alpha = d->blend_alpha;
  if (p.blend_src && !p.blend_alpha) return fail(CA_ERR_INVALID, "blend_src without blend_alpha");
  p.out = d->out;
  p.trace = trace_ptr();
  {
    // the bf16 epilogue moves 8 columns per 16-byte access when every base and row stride it touches allows it
    auto a16 = [](const void* q) { return (reinterpret_cast<uintptr_t>(q) & 15) == 0; };
    bool vec = a16(p.out) && a16(p.residual) && a16(p.blend_src) && a16(p.rowvec);
    for (int i = 0; i < 4; ++i) {
      vec = vec && (p.ostride[i] % 8) == 0;
      if (p.residual || p.blend_src) vec = vec && (p.rstride[i] % 8) == 0;
      if (p.rowvec) vec = vec && (p.vstride[i] % 8) == 0;
    }
    p.vec_ok = vec ? 1 : 0;
  }

  CUtensorMap ta[2], tw;
  memset(ta, 0, sizeof(ta));
  for (int s = 0; s < d->nsrc; ++s) {
    // the map covers channels [0, c_off + c_len) so that chunks past the slice are zero filled
    int max_tap_c = 0;
    for (int t = 0; t < d->ntaps; ++t) max_tap_c = d->tap_c_off[t] > max_tap_c ? d->tap_c_off[t] : max_tap_c;
    cuuint64_t dims[5] = {static_cast<cuuint64_t>(max_tap_c + d->a_c_off[s] + d->a_c_len[s]), (cuuint64_t)d->a_dims[0],
                          (cuuint64_t)d->a_dims[1], (cuuint64_t)d->a_dims[2], (cuuint64_t)d->a_dims[3]};
    if (max_tap_c + d->a_c_off[s] + d->a_c_len[s] > d->a_channels[s]) return fail(CA_ERR_INVALID, "channel slice exceeds tensor");
    cuuint64_t strides[4];
    for (int i = 0; i < 4; ++i) strides[i] = static_cast<cuuint64_t>(d->a_strides[s][i]) * 2;
    cuuint32_t box[5] = {64, (cuuint32_t)d->box[0], (cuuint32_t)d->box[1], (cuuint32_t)d->box[2], (cuuint32_t)d->box[3]};
    int rc = make_tmap(&ta[s], d->a[s], 5, dims, strides, box);
    if (rc) return rc;
  }
  if (d->nsrc == 1) ta[1] = ta[0];
  {
    const cuuint64_t ktot = static_cast<cuuint64_t>(d->ntaps) * k_per_tap;
    if (ktot % 8 != 0) return fail(CA_ERR_INVALID, "weight row length must be a multiple of 8");
    cuuint64_t dims[2] = {ktot, static_cast<cuuint64_t>(d->w_rows)};
    cuuint64_t strides[1] = {ktot * 2};
    cuuint32_t box[2] = {64, static_cast<cuuint32_t>(bn)};
    int rc = make_tmap(&tw, d->w, 2, dims, strides, box);
    if (rc) return rc;
  }
  const long long tiles_m = static_cast<long long>(p.ntile[0]) * p.ntile[1] * p.ntile[2] * p.ntile[3];
  const long long tiles = tiles_m * p.n_tiles_n;
  if (tiles <= 0) return fail(CA_ERR_INVALID, "empty problem");
  const long long sms = num_sms();
  const int grid = static_cast<int>(tiles < sms ? tiles : sms);
  CA_LAUNCH(ca::launch_gemm_conv(bn, ta[0], ta[1], tw, p, grid, stream), "gemm_conv launch");
}

int ca_attention(const ca_attention_desc* d, void* cuda_stream) {
  if (!d) return fail(CA_ERR_INVALID, "null desc");
  cudaStream_t stream = static_cast<cudaStream_t>(cuda_stream);
  if (d->head_dim_pad != 64 && d->head_dim_pad != 128 && d->head_dim_pad != 192)
    return fail(CA_ERR_UNSUPPORTED, "head_dim_pad must be 64, 128 or 192 (got %d)", d->head_dim_pad);
  if (d->batch < 1 || d->heads < 1 || d->lq < 1 || d->lk < 1) return fail(CA_ERR_INVALID, "empty attention problem");
  const int kv_div = d->kv_batch_div > 0 ? d->kv_batch_div : 1;
  if (d->batch % kv_div != 0) return fail(CA_ERR_INVALID, "batch must be a multiple of kv_batch_div");
  const cuuint64_t ctot = static_cast<cuuint64_t>(d->heads) * d->head_dim_pad;
  CUtensorMap tq, tk, tv;
  const cuuint32_t box[3] = {64, 128, 1};
  {
    cuuint64_t dims[3] = {ctot, (cuuint64_t)d->lq, (cuuint64_t)d->batch};
    cuuint64_t st[2] = {(cuuint64_t)d->q_row_stride * 2, (cuuint64_t)d->q_batch_stride * 2};
    int rc = make_tmap(&tq, d->q, 3, dims, st, box);
    if (rc) return rc;
  }
  {
    cuuint64_t dims[3] = {ctot, (cuuint64_t)d->lk, (cuuint64_t)(d->batch / kv_div)};
    cuuint64_t st[2] = {(cuuint64_t)d->k_row_stride * 2, (cuuint64_t)d->k_batch_stride * 2};
    int rc = make_tmap(&tk, d->k, 3, dims, st, box);
    if (rc) return rc;
    cuuint64_t sv[2] = {(cuuint64_t)d->v_row_stride * 2, (cuuint64_t)d->v_batch_stride * 2};
    rc = make_tmap(&tv, d->v, 3, dims, sv, box);
    if (rc) return rc;
  }
  ca::AttnParams p;
  p.batch = d->batch; p.heads = d->heads; p.lq = d->lq; p.lk = d->lk;
  p.kv_batch_div = kv_div;
  p.dqk_chunks = d->head_dim_pad / 64;
  p.v_slices = d->head_dim_pad / 64;
  p.scale_log2 = d->scale * 1.4426950408889634f;
  p.out = static_cast<__nv_bfloat16*>(d->out);
  p.out_batch_stride = d->out_batch_stride;
  p.out_row_stride = d->out_row_stride;
  CA_LAUNCH(ca::launch_attention(tq, tk, tv, p, stream), "attention launch");
}

int ca_groupnorm_stats(const void* x0, int32_t c0, const void* x1, int32_t c1, int32_t n, int64_t rows, int32_t groups,
                       double* sums, void* s) {
  CA_LAUNCH(ca::launch_gn_stats((const __nv_bfloat16*)x0, c0, (const __nv_bfloat16*)x1, c1, n, rows, groups, sums,
                                (cudaStream_t)s), "groupnorm_stats");
}
int ca_groupnorm_apply(const void* x0, int32_t c0, const void* x1, int32_t c1, int32_t n, int32_t h, int32_t w,
                       int32_t imgs_per_sample, int32_t groups, float eps, const double* sums, const float* gamma,
                       const float* beta, int32_t silu, int32_t up2x, void* y, void* s) {
  CA_LAUNCH(ca::launch_gn_apply((const __nv_bfloat16*)x0, c0, (const __nv_bfloat16*)x1, c1, n, h, w, imgs_per_sample,
                                groups, eps, sums, gamma, beta, silu, up2x, (__nv_bfloat16*)y, (cudaStream_t)s),
            "groupnorm_apply");
}
int ca_layernorm(const void* x, int64_t rows, int32_t c, float eps, const float* gamma, const float* beta,
                 const void* add_rowvec, int64_t rows_per_vec, void* y_sum, void* y, void* s) {
  CA_LAUNCH(ca::launch_layernorm((const __nv_bfloat16*)x, rows, c, eps, gamma, beta, (const __nv_bfloat16*)add_rowvec,
                                 rows_per_vec, (__nv_bfloat16*)y_sum, (__nv_bfloat16*)y, (cudaStream_t)s), "layernorm");
}
int ca_timestep_embedding(const float* t, int32_t n, int32_t dim, int32_t flip, float shift, int32_t round_t, void* out,
                          void* s) {
  CA_LAUNCH(ca::launch_timestep_embedding(t, n, dim, flip, shift, round_t, (__nv_bfloat16*)out, (cudaStream_t)s),
            "timestep_embedding");
}
int ca_silu(const void* x, int64_t n, void* y, void* s) {
  CA_LAUNCH(ca::launch_silu((const __nv_bfloat16*)x, n, (__nv_bfloat16*)y, (cudaStream_t)s), "silu");
}
int ca_add(const void* a, const void* b, int64_t n, void* y, void* s) {
  CA_LAUNCH(ca::launch_add((const __nv_bfloat16*)a, (const __nv_bfloat16*)b, n, (__nv_bfloat16*)y, (cudaStream_t)s),
            "add");
}
int ca_nchw_to_nhwc(const void* x, int32_t src_fp32, int32_t n, int32_t c, int64_t hw, int32_t c_pad, void* y, void* s) {
  CA_LAUNCH(ca::launch_nchw_to_nhwc(x, src_fp32, n, c, hw, c_pad, (__nv_bfloat16*)y, (cudaStream_t)s), "nchw_to_nhwc");
}
int ca_nhwc_to_nchw(const void* x, int32_t n, int32_t c, int32_t c_stride, int64_t hw, void* y, int32_t dst_fp32,
                    void* s) {
  CA_LAUNCH(ca::launch_nhwc_to_nchw((const __nv_bfloat16*)x, n, c, c_stride, hw, y, dst_fp32, (cudaStream_t)s),
            "nhwc_to_nchw");
}
int ca_avgpool(const void* x, int32_t n, int32_t h, int32_t w, int32_t c, int32_t oh, int32_t ow, void* y, void* s) {
  CA_LAUNCH(ca::launch_avgpool((const __nv_bfloat16*)x, n, h, w, c, oh, ow, (__nv_bfloat16*)y, (cudaStream_t)s),
            "avgpool");
}
int ca_upsample2x(const void* x, int32_t n, int32_t h, int32_t w, int32_t c, void* y, void* s) {
  CA_LAUNCH(ca::launch_upsample2x((const __nv_bfloat16*)x, n, h, w, c, (__nv_bfloat16*)y, (cudaStream_t)s),
            "upsample2x");
}
int ca_router_weights(const float* logits, const uint8_t* mask, int32_t nrouters, int32_t nexperts, float* weights,
                      void* s) {
  CA_LAUNCH(ca::launch_router_weights(logits, mask, nrouters, nexperts, weights, (cudaStream_t)s), "router_weights");
}
int ca_router_merge(const void* const* xs, const float* w, int32_t nactive, int64_t n, void* y, void* s) {
  CA_LAUNCH(ca::launch_router_merge((const __nv_bfloat16* const*)xs, w, nactive, n, (__nv_bfloat16*)y, (cudaStream_t)s),
            "router_merge");
}
int ca_cfg_euler(const void* eu, const void* et, const float* lat, int64_t n, float g, const float* step_row,
                 int32_t round_latents_bf16, float* lat_out, void* next_in, void* s) {
  CA_LAUNCH(ca::launch_cfg_euler((const __nv_bfloat16*)eu, (const __nv_bfloat16*)et, lat, n, g, step_row,
                                 round_latents_bf16, lat_out, (__nv_bfloat16*)next_in, (cudaStream_t)s), "cfg_euler");
}
int ca_cfg_euler_v(const void* eu, const void* et, const float* lat, int64_t n, const float* guidance, int32_t frames,
                   int64_t frame_elems, const float* step_row, int32_t round_latents_bf16, float* lat_out, void* next_in,
                   void* s) {
  CA_LAUNCH(ca::launch_cfg_euler_v((const __nv_bfloat16*)eu, (const __nv_bfloat16*)et, lat, n, guidance, frames,
                                   frame_elems, step_row, round_latents_bf16, lat_out, (__nv_bfloat16*)next_in,
                                   (cudaStream_t)s), "cfg_euler_v");
}
int ca_cfg_ddim(const void* eu, const void* et, const float* lat, int64_t n, float g, const float* step_row,
                int32_t round_latents_bf16, int32_t v_prediction, float* lat_out, void* next_in, void* s) {
  CA_LAUNCH(ca::launch_cfg_ddim((const __nv_bfloat16*)eu, (const __nv_bfloat16*)et, lat, n, g, step_row,
                                round_latents_bf16, v_prediction, lat_out, (__nv_bfloat16*)next_in, (cudaStream_t)s),
            "cfg_ddim");
}
int ca_i2vgen_latent_encoder(const void* x, int32_t clips, int32_t frames, int64_t hw, int32_t c_stride,
                             const float* params, void* y, void* s) {
  CA_LAUNCH(ca::launch_i2vgen_latent_encoder((const __nv_bfloat16*)x, clips, frames, hw, c_stride, params,
                                             (__nv_bfloat16*)y, (cudaStream_t)s), "i2vgen_latent_encoder");
}
int ca_frame_conv_small(const void* x, int32_t clips, int32_t frames, int64_t hw, int32_t c_stride, int32_t cin,
                        int32_t cout, const float* w_host, const float* bias_host, void* y, void* s) {
  if (w_host == nullptr) return fail(CA_ERR_INVALID, "frame_conv_small: null weight pointer");
  CA_LAUNCH(ca::launch_frame_conv_small((const __nv_bfloat16*)x, clips, frames, hw, c_stride, cin, cout, w_host,
                                        bias_host, (__nv_bfloat16*)y, (cudaStream_t)s), "frame_conv_small");
}
int ca_softmax_rows(const float* x, int64_t rows, int64_t cols, void* y, void* s) {
  CA_LAUNCH(ca::launch_softmax_rows(x, rows, cols, (__nv_bfloat16*)y, (cudaStream_t)s), "softmax_rows");
}
int ca_temporal_attention(const void* q, const void* k, const void* v, int32_t clips, int32_t frames, int64_t hw,
                          int32_t heads, float scale, int64_t in_row_stride, void* out, void* s) {
  cudaStream_t stream = static_cast<cudaStream_t>(s);
  if (clips < 1 || frames < 1 || frames > 32 || hw < 1 || heads < 1) return fail(CA_ERR_INVALID, "empty temporal attention problem");
  if ((in_row_stride & 7) != 0) return fail(CA_ERR_INVALID, "row stride must be a multiple of 8 elements");
  static const bool fma = getenv("CA_TATTN_FMA") != nullptr;  // developer A/B knob: round 1's FMA kernel
  if (fma) {
    CA_LAUNCH(ca::launch_temporal_attention((const __nv_bfloat16*)q, (const __nv_bfloat16*)k, (const __nv_bfloat16*)v,
                                            clips, frames, hw, heads, scale, in_row_stride, (__nv_bfloat16*)out, stream),
              "temporal_attention");
  }
  // global dims ordered (channel, frame, pixel, clip): a box then holds whole frame sequences of consecutive pixels
  const int seq = frames <= 16 ? 16 : 32;
  const cuuint64_t dims[4] = {(cuuint64_t)heads * 64, (cuuint64_t)frames, (cuuint64_t)hw, (cuuint64_t)clips};
  const cuuint64_t st[3] = {(cuuint64_t)hw * in_row_stride * 2, (cuuint64_t)in_row_stride * 2,
                            (cuuint64_t)frames * hw * in_row_stride * 2};
  const cuuint32_t box[4] = {64, (cuuint32_t)seq, (cuuint32_t)(128 / seq), 1};
  CUtensorMap tq, tk, tv;
  int rc = make_tmap(&tq, q, 4, dims, st, box);
  if (rc) return rc;
  if ((rc = make_tmap(&tk, k, 4, dims, st, box))) return rc;
  if ((rc = make_tmap(&tv, v, 4, dims, st, box))) return rc;
  ca::TemporalAttnParams p;
  p.clips = clips; p.frames = frames; p.heads = heads; p.hw = hw;
  p.scale_log2 = scale * 1.4426950408889634f;
  p.out = static_cast<__nv_bfloat16*>(out);
  p.out_row_stride = static_cast<long long>(heads) * 64;
  CA_LAUNCH(ca::launch_temporal_attention_tc(tq, tk, tv, p, stream), "temporal_attention");
}

}  // extern "C"
