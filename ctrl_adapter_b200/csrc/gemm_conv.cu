// ca_gemm: argument validation, the TMA tensor maps of A and W, and dispatch of gemm_conv_kernel to the per-BN
// translation units (gemm_conv_bn*.cu; split so the kernel instantiations compile in parallel).
#include <string.h>

#include "kernels.h"

namespace ca {

extern "C" int ca_gemm(const ca_gemm_desc* d, void* cuda_stream) {
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

  GemmParams p;
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

  // the A maps cover channels [0, max tap_c_off + c_off + c_len) so that chunks past the slice are zero filled
  int max_tap_c = 0;
  for (int t = 0; t < d->ntaps; ++t) max_tap_c = d->tap_c_off[t] > max_tap_c ? d->tap_c_off[t] : max_tap_c;
  int k_per_tap = 0;
  for (int s = 0; s < d->nsrc; ++s) {
    if (d->a_c_len[s] <= 0 || (d->a_c_off[s] & 7) != 0) return fail(CA_ERR_INVALID, "bad channel slice");
    if (s == 0 && d->nsrc == 2 && (d->a_c_len[0] % 64) != 0)
      return fail(CA_ERR_INVALID, "first of two sources must contribute a multiple of 64 channels");
    if (max_tap_c + d->a_c_off[s] + d->a_c_len[s] > d->a_channels[s]) return fail(CA_ERR_INVALID, "channel slice exceeds tensor");
    p.src_c[s] = d->a_c_len[s];
    p.src_c0_off[s] = d->a_c_off[s];
    k_per_tap += d->a_c_len[s];
  }
  p.nsrc = d->nsrc;
  if (d->w_k_per_tap < k_per_tap) return fail(CA_ERR_INVALID, "w_k_per_tap smaller than the A channels per tap");
  k_per_tap = d->w_k_per_tap;
  p.k_per_tap = k_per_tap;
  const cuuint64_t ktot = static_cast<cuuint64_t>(d->ntaps) * k_per_tap;
  if (ktot % 8 != 0) return fail(CA_ERR_INVALID, "weight row length must be a multiple of 8");
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
  const long long tiles_m = static_cast<long long>(p.ntile[0]) * p.ntile[1] * p.ntile[2] * p.ntile[3];
  const long long tiles = tiles_m * p.n_tiles_n;
  if (tiles <= 0) return fail(CA_ERR_INVALID, "empty problem");

  CUtensorMap ta[2], tw;
  memset(ta, 0, sizeof(ta));
  for (int s = 0; s < d->nsrc; ++s) {
    cuuint64_t dims[5] = {static_cast<cuuint64_t>(max_tap_c + d->a_c_off[s] + d->a_c_len[s]), (cuuint64_t)d->a_dims[0],
                          (cuuint64_t)d->a_dims[1], (cuuint64_t)d->a_dims[2], (cuuint64_t)d->a_dims[3]};
    cuuint64_t strides[4];
    for (int i = 0; i < 4; ++i) strides[i] = static_cast<cuuint64_t>(d->a_strides[s][i]) * 2;
    cuuint32_t box[5] = {64, (cuuint32_t)d->box[0], (cuuint32_t)d->box[1], (cuuint32_t)d->box[2], (cuuint32_t)d->box[3]};
    int rc = make_tmap(&ta[s], d->a[s], 5, dims, strides, box);
    if (rc) return rc;
  }
  if (d->nsrc == 1) ta[1] = ta[0];
  {
    cuuint64_t dims[2] = {ktot, static_cast<cuuint64_t>(d->w_rows)};
    cuuint64_t strides[1] = {ktot * 2};
    cuuint32_t box[2] = {64, static_cast<cuuint32_t>(bn)};
    int rc = make_tmap(&tw, d->w, 2, dims, strides, box);
    if (rc) return rc;
  }
  const long long sms = num_sms();
  const int grid = static_cast<int>(tiles < sms ? tiles : sms);
  cudaError_t e;
  switch (bn) {
    case 64: e = launch_gemm_bn64(ta[0], ta[1], tw, p, grid, stream); break;
    case 128: e = launch_gemm_bn128(ta[0], ta[1], tw, p, grid, stream); break;
    case 160: e = launch_gemm_bn160(ta[0], ta[1], tw, p, grid, stream); break;
    default: e = launch_gemm_bn256(ta[0], ta[1], tw, p, grid, stream); break;
  }
  return launched(e, "gemm_conv launch");
}

}  // namespace ca
