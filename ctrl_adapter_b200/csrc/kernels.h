// Internal kernel-launch interface shared by the .cu translation units and capi.cu.
#pragma once
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/ctrl_adapter_b200.h"

namespace ca {

struct GemmParams {
  int box[4];             // row-space box extents (product == 128)
  int ntile[4];           // tiles along each row dim
  int odim[4];            // output extents (rows outside are computed but not stored)
  long long ostride[4];   // output element strides per row dim
  long long rstride[4];   // residual / blend_src element strides per row dim
  long long vstride[4];   // rowvec element strides per row dim
  int ntaps;
  int tap_off[CA_MAX_TAPS][4];  // A-coordinate offset of each tap, per row dim
  int tap_c_off[CA_MAX_TAPS];   // A channel offset of each tap (stride-2 parity views)
  int nsrc;
  int src_c[2];           // channels taken from each A source (K extent per tap = sum)
  int src_c0_off[2];      // first channel inside each source tensor
  int k_per_tap;          // weight row elements per tap (>= src_c[0] + src_c[1], zero padded)
  int n_out;              // output columns
  int n_tiles_n;
  int act;
  int out_fp32;
  int vec_ok;             // bf16 output: out / residual / blend_src / rowvec bases and strides allow 16-byte access
  float out_scale;
  const float* bias;               // [weight rows] fp32
  const __nv_bfloat16* rowvec;     // broadcast add, indexed through vstride
  const __nv_bfloat16* residual;   // indexed through rstride
  const __nv_bfloat16* blend_src;  // AlphaBlender x_spatial, indexed through rstride
  const float* blend_alpha;        // device scalar: sigmoid(mix_factor), bf16-valued
  void* out;
  unsigned long long* trace;  // developer builds (-DCA_TRACE) only: per-CTA role wait-cycle counters, else unused
};

cudaError_t launch_gemm_conv(int bn, const CUtensorMap& a0, const CUtensorMap& a1, const CUtensorMap& w,
                             const GemmParams& p, int grid, cudaStream_t stream);

struct AttnParams {
  int batch, heads, lq, lk;
  int kv_batch_div;    // K/V batch index = query batch index / kv_batch_div (context shared by the frames of a clip)
  int dqk_chunks;      // padded head dim / 64 used for QK^T
  int v_slices;        // padded head dim / 64 (PV is computed one 64-wide slice per CTA)
  float scale_log2;    // softmax scale * log2(e)
  __nv_bfloat16* out;  // [batch, lq, heads * 64 * v_slices]
  long long out_batch_stride, out_row_stride;  // elements
};
cudaError_t launch_attention(const CUtensorMap& q, const CUtensorMap& k, const CUtensorMap& v, const AttnParams& p,
                             cudaStream_t stream);

// --- temporal_attention.cu ---
struct TemporalAttnParams {
  int clips, frames, heads;
  long long hw;
  float scale_log2;            // softmax scale * log2(e)
  __nv_bfloat16* out;          // rows ((clip * frames + f) * hw + pixel), heads * 64 used columns
  long long out_row_stride;    // elements
};
cudaError_t launch_temporal_attention_tc(const CUtensorMap& q, const CUtensorMap& k, const CUtensorMap& v,
                                         const TemporalAttnParams& p, cudaStream_t stream);

// --- norm.cu ---
cudaError_t launch_gn_stats(const __nv_bfloat16* x0, int c0, const __nv_bfloat16* x1, int c1, int n, long long hw,
                            int groups, double* sums /*[n][groups][2], zeroed by the launcher*/, cudaStream_t stream);
cudaError_t launch_gn_apply(const __nv_bfloat16* x0, int c0, const __nv_bfloat16* x1, int c1, int n, int h, int w,
                            int imgs_per_sample, int groups, float eps, const double* sums, const float* gamma,
                            const float* beta, int silu, int up2x, __nv_bfloat16* y, cudaStream_t stream);
cudaError_t launch_layernorm(const __nv_bfloat16* x, long long rows, int c, float eps, const float* gamma,
                             const float* beta, const __nv_bfloat16* add_rowvec, long long rows_per_vec,
                             __nv_bfloat16* y_sum, __nv_bfloat16* y, cudaStream_t stream);

// --- elementwise.cu ---
cudaError_t launch_timestep_embedding(const float* t, int n, int dim, int flip_sin_to_cos, float freq_shift,
                                      int round_t_bf16, __nv_bfloat16* out, cudaStream_t stream);
cudaError_t launch_silu(const __nv_bfloat16* x, long long n, __nv_bfloat16* y, cudaStream_t stream);
cudaError_t launch_add(const __nv_bfloat16* a, const __nv_bfloat16* b, long long n, __nv_bfloat16* y,
                       cudaStream_t stream);
cudaError_t launch_nchw_to_nhwc(const void* x, int src_fp32, int n, int c, long long hw, int c_pad,
                                __nv_bfloat16* y, cudaStream_t stream);
cudaError_t launch_nhwc_to_nchw(const __nv_bfloat16* x, int n, int c, int c_stride, long long hw, void* y,
                                int dst_fp32, cudaStream_t stream);
cudaError_t launch_avgpool(const __nv_bfloat16* x, int n, int h, int w, int c, int oh, int ow, __nv_bfloat16* y,
                           cudaStream_t stream);
cudaError_t launch_upsample2x(const __nv_bfloat16* x, int n, int h, int w, int c, __nv_bfloat16* y,
                              cudaStream_t stream);
cudaError_t launch_router_weights(const float* logits, const unsigned char* mask, int nrouters, int nexperts,
                                  float* weights, cudaStream_t stream);
constexpr int kFrameConvMaxC = 4;
struct FrameConvSmallParams {
  float w[kFrameConvMaxC][kFrameConvMaxC][3];  // [out channel][in channel][frame tap]
  float b[kFrameConvMaxC];
};
cudaError_t launch_frame_conv_small(const __nv_bfloat16* x, int clips, int frames, long long hw, int c_stride, int cin,
                                    int cout, const float* w_host, const float* bias_host, __nv_bfloat16* y,
                                    cudaStream_t stream);
cudaError_t launch_softmax_rows(const float* x, long long rows, long long cols, __nv_bfloat16* y, cudaStream_t stream);
static constexpr int kMaxRouterExperts = 8;
cudaError_t launch_router_merge(const __nv_bfloat16* const* xs_host, const float* w, int nactive, long long n,
                                __nv_bfloat16* y, cudaStream_t stream);
cudaError_t launch_cfg_euler_v(const __nv_bfloat16* eps_uncond, const __nv_bfloat16* eps_text, const float* latents_in,
                               long long n, const float* guidance, int frames, long long frame_elems,
                               const float* step_row, int round_latents_bf16, float* latents_out,
                               __nv_bfloat16* model_in_next, cudaStream_t stream);
cudaError_t launch_cfg_euler(const __nv_bfloat16* eps_uncond, const __nv_bfloat16* eps_text, const float* latents_in,
                             long long n, float guidance, const float* step_row, int round_latents_bf16,
                             float* latents_out, __nv_bfloat16* model_in_next, cudaStream_t stream);
cudaError_t launch_cfg_ddim(const __nv_bfloat16* eps_uncond, const __nv_bfloat16* eps_text, const float* latents_in,
                            long long n, float guidance, const float* step_row, int round_latents_bf16,
                            int v_prediction, float* latents_out, __nv_bfloat16* model_in_next, cudaStream_t stream);
cudaError_t launch_i2vgen_latent_encoder(const __nv_bfloat16* x, int clips, int frames, long long hw, int c_stride,
                                         const float* params, __nv_bfloat16* y, cudaStream_t stream);
cudaError_t launch_temporal_attention(const __nv_bfloat16* q, const __nv_bfloat16* k, const __nv_bfloat16* v,
                                      int clips, int frames, long long hw, int heads, float scale,
                                      long long in_row_stride, __nv_bfloat16* out, cudaStream_t stream);

}  // namespace ca
