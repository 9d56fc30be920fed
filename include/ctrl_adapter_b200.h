/*
 * ctrl_adapter_b200 -- C ABI of the H100 (sm_90a) denoising hot path of Ctrl-Adapter.
 *
 * The reference (HL-hanlin/Ctrl-Adapter @ 4f495bd) has no FFI layer: its hot path is eager
 * PyTorch/diffusers `nn.Module.forward` calls (SURVEY.md section 8b).  This header is the boundary a
 * maintainer would bind instead of those library calls: plain pointers + sizes, a CUDA stream
 * handle, `int` status (0 = ok) with a thread-local message (ca_last_error), no torch types.
 * All device tensors are bf16 (uint16 payload) unless stated; activations are channels-last
 * ([..., C], C contiguous).  Every entry point is asynchronous on `stream`, never synchronises
 * the device and is CUDA-graph capturable.
 *
 * Each entry names the reference call site(s) it replaces (file:line under /root/reference, or the
 * diffusers v0.27.2 op the reference reaches through that line).
 */
#ifndef CTRL_ADAPTER_B200_H_
#define CTRL_ADAPTER_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define CA_MAX_TAPS 9

enum ca_status { CA_OK = 0, CA_ERR_INVALID = 1, CA_ERR_CUDA = 2, CA_ERR_UNSUPPORTED = 3 };
enum ca_act { CA_ACT_NONE = 0, CA_ACT_SILU = 1, CA_ACT_GEGLU = 2 };

/* ABI version of this header; bump on any struct change. */
#define CA_ABI_VERSION 1
int ca_abi_version(void);
/* Thread-local description of the last non-zero status returned on this thread. */
const char* ca_last_error(void);
/* 0 when a CUDA device with compute capability 9.x (sm_90a) is usable by this process, else non-zero. */
int ca_device_ok(void);

/*
 * ca_gemm -- multi-tap tensor-core contraction (wgmma) with fused epilogue.
 *
 *   out[row, n] = epi( sum_tap sum_src sum_c  A_src[row + tap_off[tap], c] * W[n, tap, src, c] )
 *
 * Replaces: F.linear / nn.Linear   (model/adapter_spatial_temporal.py:257,287; diffusers Attention to_q/k/v/out,
 *                                   FeedForward, TimestepEmbedding reached from :208,:265,:271,:280)
 *           F.conv2d 3x3 / 1x1     (model/resnet_block_2d.py:189,214,217; controlnet/controlnet.py:95-102,802,853,858;
 *                                   Downsample2D stride 2; UNet resnets / up-samplers)
 *           F.conv3d (3,1,1)       (diffusers TemporalResnetBlock reached from adapter_spatial_temporal.py:226)
 *
 * Row space: 4 dims (fastest first), e.g. (x, y, sample, 1) for a conv, (token, 1, 1, 1) for a Linear.
 * A sources are 5-D tensors (channel, then the 4 row dims) read through TMA with zero fill outside the tensor,
 * which implements the convolution padding.  Two sources are concatenated along the channel axis (UNet skip
 * connections) without materialising the concat.
 */
typedef struct ca_gemm_desc {
  /* A operand */
  int32_t nsrc;              /* 1 or 2 */
  const void* a[2];          /* bf16, 16-byte aligned */
  int32_t a_channels[2];     /* innermost extent of each source tensor (elements) */
  int32_t a_c_off[2];        /* first channel used from each source */
  int32_t a_c_len[2];        /* channels used from each source; K per tap = a_c_len[0] + a_c_len[1] */
  int64_t a_dims[4];         /* extents of the 4 row dims of the A tensors */
  int64_t a_strides[2][4];   /* element strides of the 4 row dims (multiples of 8) */
  int32_t box[4];            /* tile box over the row dims, product must be 128 */
  int32_t ntaps;             /* 1 (linear), 3 (temporal conv), 9 (3x3 conv) */
  int32_t tap_off[CA_MAX_TAPS][4];
  int32_t tap_c_off[CA_MAX_TAPS]; /* extra channel offset per tap (stride-2 convs read a parity view whose
                                     channel axis is [x parity][C]); 0 otherwise */
  /* weights: [w_rows][ntaps * w_k_per_tap] bf16, K contiguous, each tap's K zero padded to w_k_per_tap
   * (>= a_c_len[0]+a_c_len[1]; must be a multiple of 64 when tap_c_off is used); for CA_ACT_GEGLU the rows are
   * interleaved per n-tile: tile t holds value rows [t*bn/2,(t+1)*bn/2) then the matching gate rows */
  const void* w;
  int32_t w_rows;
  int32_t w_k_per_tap;
  const float* bias;         /* [w_rows] fp32 (bf16-valued) or NULL */
  /* output */
  void* out;
  int32_t out_fp32;          /* 0: bf16, 1: fp32 (test/debug) */
  int32_t n_out;             /* output columns (w_rows, or w_rows/2 for GEGLU) */
  int32_t out_dims[4];       /* extents of the output row space */
  int64_t out_strides[4];    /* element strides of the output rows */
  /* epilogue, applied in this order with a bf16 rounding after every step (autocast rounding points):
   *   v = acc + bias ; v = act(v) ; v *= out_scale ; v += rowvec ; v += residual ;
   *   v = alpha * blend_src + (1 - alpha) * v
   * out_fp32 = 1 rounds to bf16 only after act (SiLU) and after the rowvec add; bias, out_scale and the residual add
   * stay fp32; there is no GEGLU and no blend term (CA_ERR_UNSUPPORTED).                  */
  int32_t act;
  float out_scale;
  const void* rowvec;        /* bf16, addressed rowvec[sum_d o_d * rowvec_strides[d] + n] */
  int64_t rowvec_strides[4];
  const void* residual;      /* bf16, addressed with res_strides */
  const void* blend_src;     /* bf16, addressed with res_strides */
  int64_t res_strides[4];
  const float* blend_alpha;  /* device scalar */
  int32_t bn;                /* N tile: 0 = auto, else 64/128/160/256 */
} ca_gemm_desc;
int ca_gemm(const ca_gemm_desc* d, void* cuda_stream);

/*
 * ca_attention -- softmax(Q K^T * scale) V, flash-style, wgmma + TMA.
 * Replaces F.scaled_dot_product_attention (diffusers AttnProcessor2_0) reached from
 * model/adapter_spatial_temporal.py:271 (adapter spatial self / cross attention), the ControlNet
 * Transformer2DModel blocks built at controlnet/controlnet.py:371-424 and the UNet attention layers.
 * q/k/v: [batch, L, heads * head_dim_pad] bf16 with head_dim_pad a multiple of 64 (zero padded),
 * row strides given in elements.  out: [batch, lq, heads * head_dim_pad], 4-byte aligned, even out strides.
 * Constraints: batch <= 65535, heads * head_dim_pad / 64 <= 65535.
 */
typedef struct ca_attention_desc {
  const void* q; const void* k; const void* v; void* out;
  int32_t batch, heads, lq, lk;
  int32_t head_dim_pad;                 /* 64, 128 or 192 */
  float scale;                          /* softmax scale (1/sqrt(true head dim)): positive and finite, as is
                                           scale * log2(e) (the softmax works in base 2); others -> CA_ERR_INVALID */
  int64_t q_row_stride, q_batch_stride; /* elements */
  int64_t k_row_stride, k_batch_stride;
  int64_t v_row_stride, v_batch_stride;
  int64_t out_row_stride, out_batch_stride;
  int32_t kv_batch_div;                 /* K/V batch = query batch / kv_batch_div (>= 1): one context shared by the
                                           frames of a clip (I2VGen-XL `context_emb.repeat_interleave(num_frames)`) */
} ca_attention_desc;
int ca_attention(const ca_attention_desc* d, void* cuda_stream);

/*
 * GroupNorm on channels-last data, two launches: statistics (fp64 accumulation of sum / sum-of-squares per
 * (sample, group), of x minus the group's first channel at the sample's first pixel) and apply (+SiLU, + optional 2x
 * nearest up-sampling, + optional channel concat of two sources).
 * Replaces F.group_norm + F.silu (+ Upsample2D) at model/resnet_block_2d.py:171-184,199-211,
 * model/adapter_spatial_temporal.py:254, diffusers TemporalResnetBlock / Transformer2DModel norms.
 * `sums` is a caller-provided scratch of n*groups*2 doubles (zeroed by ca_groupnorm_stats).
 * A "sample" is `rows` consecutive channel vectors (h*w, or frames*h*w for the 5-D temporal GroupNorm).
 * Constraints (both passes): 1 <= groups <= 64 dividing c0 + c1; c0, c1 multiples of 8 with 8 <= c0 + c1 <= 4096;
 * 1 <= n <= 65535; x0 (and x1 when c1 > 0) and y 16-byte aligned; stats: rows >= 1; apply: h, w >= 1, h * w < 2^30,
 * imgs_per_sample >= 1 dividing n (apply's n counts images, stats' n samples); y must not alias x0 or x1 (apply reads
 * each sample's first pixel back in every block), and apply must see the data stats summed, with rows = h * w *
 * imgs_per_sample.
 */
int ca_groupnorm_stats(const void* x0, int32_t c0, const void* x1, int32_t c1, int32_t n, int64_t rows,
                       int32_t groups, double* sums, void* cuda_stream);
int ca_groupnorm_apply(const void* x0, int32_t c0, const void* x1, int32_t c1, int32_t n, int32_t h, int32_t w,
                       int32_t imgs_per_sample, int32_t groups, float eps, const double* sums, const float* gamma,
                       const float* beta, int32_t silu, int32_t up2x, void* y, void* cuda_stream);

/*
 * LayerNorm over the last dim (fp32 statistics) with an optional fused broadcast add before the norm:
 *   s = x + add_rowvec[row / rows_per_vec]   (written to y_sum when non-NULL) ; y = LN(s) * gamma + beta
 * Replaces F.layer_norm in diffusers BasicTransformerBlock / TemporalBasicTransformerBlock (norm1/2/3, norm_in)
 * and the `hidden_states + emb` add at model/adapter_spatial_temporal.py:279.
 * Constraints: c a multiple of 8, 8 <= c <= 2048; x contiguous [rows, c] and 16-byte aligned (whole rows travel as
 * 1-D bulk copies); gamma, beta, add_rowvec, y_sum and y 16-byte aligned; rows < 2^31 - 64.  y / y_sum may alias x
 * (each row is read before it is written).
 */
int ca_layernorm(const void* x, int64_t rows, int32_t c, float eps, const float* gamma, const float* beta,
                 const void* add_rowvec, int64_t rows_per_vec, void* y_sum, void* y, void* cuda_stream);

/* Sinusoidal timestep embedding (diffusers Timesteps; model/adapter_spatial_temporal.py:207,263;
 * controlnet/controlnet.py:751).  t: n fp32 device values.  round_t_bf16 reproduces the reference's
 * `timestep.to(bf16)` before the sinusoid (adapter_spatial_temporal.py:198).  out: [n, dim] bf16; an odd dim ends in
 * a zero column.  Constraints: n >= 1, dim >= 2. */
int ca_timestep_embedding(const float* t, int32_t n, int32_t dim, int32_t flip_sin_to_cos, float freq_shift,
                          int32_t round_t_bf16, void* out, void* cuda_stream);

/* Elementwise helpers (bf16 in/out): n a multiple of 8, every pointer 16-byte aligned. */
int ca_silu(const void* x, int64_t n, void* y, void* cuda_stream);
int ca_add(const void* a, const void* b, int64_t n, void* y, void* cuda_stream);
/* NCHW (bf16 or fp32) -> channels-last bf16 with the channel count zero padded to c_pad, and back (the first c of
 * c_stride channels).  Constraints: n, c, hw >= 1; c <= c_pad (c <= c_stride); n <= 65535; c_pad (c) <= 65535 * 32;
 * hw < 2^32. */
int ca_nchw_to_nhwc(const void* x, int32_t src_fp32, int32_t n, int32_t c, int64_t hw, int32_t c_pad, void* y,
                    void* cuda_stream);
int ca_nhwc_to_nchw(const void* x, int32_t n, int32_t c, int32_t c_stride, int64_t hw, void* y, int32_t dst_fp32,
                    void* cuda_stream);
/* F.adaptive_avg_pool2d for integer ratios (sdxl pipeline :1308-1309), channels-last: oh, ow >= 1 dividing h, w. */
int ca_avgpool(const void* x, int32_t n, int32_t h, int32_t w, int32_t c, int32_t oh, int32_t ow, void* y,
               void* cuda_stream);
/* nearest 2x up-sampling, channels-last (diffusers Upsample2D in the UNet up blocks): c a multiple of 8, x and y
 * 16-byte aligned. */
int ca_upsample2x(const void* x, int32_t n, int32_t h, int32_t w, int32_t c, void* y, void* cuda_stream);

/*
 * Router (model/ctrl_router.py:85-112): masked softmax over experts for all routers in one launch,
 * one warp per router (warp-shuffle reduction).  logits [nrouters, nexperts] fp32, mask [nexperts] (0 = masked).
 * Constraints: nrouters >= 1, 1 <= nexperts <= 32.
 */
int ca_router_weights(const float* logits, const uint8_t* mask, int32_t nrouters, int32_t nexperts, float* weights,
                      void* cuda_stream);
/* Row softmax, fp32 [rows, cols] -> bf16 probabilities (cols % 4 == 0): the VAE decoder's single 512-wide attention
 * head (diffusers AutoencoderKL mid block, reached from sdxl pipeline :1414 / i2vgen pipeline :398-418) runs as
 * GEMM (QK^T, fp32) -> this -> GEMM (PV).  softmax in fp32, one rounding to bf16 (torch SDPA math semantics).  x 16-byte, y 8-byte aligned;
 * 1 <= rows < 2^31. */
int ca_softmax_rows(const float* x, int64_t rows, int64_t cols, void* y, void* cuda_stream);
/* Conv3d (3,1,1), padding (1,0,0) over the frame axis for <= 4 channels: time_conv_out of the SVD VAE's TemporalDecoder
 * (diffusers AutoencoderKLTemporalDecoder, run by the svd pipeline's decode_latents :265-292).  x: channels-last bf16
 * [clips*frames, hw, c_stride] (the first cin channels are read); w / bias: HOST arrays [cout][cin][3] / [cout] (they
 * travel to the kernel by value, so the call is CUDA-graph capturable); y: bf16 [clips*frames, cout, hw] (logical NCHW).
 * Constraints: 1 <= cin, cout <= 4; c_stride a positive multiple of 4; clips * frames <= 65535; x 8-byte and y 4-byte
 * aligned. */
int ca_frame_conv_small(const void* x, int32_t clips, int32_t frames, int64_t hw, int32_t c_stride, int32_t cin,
                        int32_t cout, const float* w_host, const float* bias_host, void* y, void* cuda_stream);
/* Weighted merge of expert residuals (i2vgen_xl pipeline :1001-1022): y = sum_e w[e] * xs[e], bf16 rounding
 * after each multiply and each add as in the reference loop.  xs: HOST array of nactive (<= 8) device pointers; they
 * travel to the kernel by value, so the call is CUDA-graph capturable.  n a multiple of 8; every xs[k] and y 16-byte
 * aligned. */
int ca_router_merge(const void* const* xs, const float* w, int32_t nactive, int64_t n, void* y, void* cuda_stream);

/* Classifier-free guidance + scheduler update in one pass (latent-sized, HBM-bound).
 * `step_row` is a DEVICE pointer to 4 floats so that a captured CUDA graph of the step can be replayed for every
 * timestep:  Euler {t, sigma, sigma_next, sqrt(sigma_next^2+1)}   DDIM {t, alpha_prod_t, alpha_prod_prev, -}.
 * Euler = SDXL default EulerDiscreteScheduler, epsilon prediction (sdxl pipeline :1369-1378):
 *   eps = u + g (c - u); x0 = x - sigma*eps; d = (x - x0)/sigma; x' = x + d (sigma_next - sigma);
 *   also emits the next step's scaled model input x' / sqrt(sigma_next^2+1) in bf16 (scale_model_input, :1285).
 * DDIM = I2VGen-XL (i2vgen_xl pipeline :1102-1115), eta = 0, epsilon prediction.
 * round_latents_bf16 = 1 reproduces the reference's bf16 latents between steps.  All three: n >= 0; eps_uncond, eps_text,
 * latents_in, step_row and latents_out non-NULL (model_in_next may be NULL: no next model input). */
int ca_cfg_euler(const void* eps_uncond, const void* eps_text, const float* latents_in, int64_t n, float guidance,
                 const float* step_row, int32_t round_latents_bf16, float* latents_out, void* model_in_next,
                 void* cuda_stream);
/* Euler, v-prediction, per-frame guidance = the SVD loop (svd pipeline :781-787; EulerDiscreteScheduler with
 * prediction_type v_prediction): latents [clips, frames, C, H, W], guidance: DEVICE fp32 [frames] (bf16-valued, the
 * pipeline's linspace(min, max, F) in the latent dtype), frame_elems = C*H*W.  step_row as for ca_cfg_euler.
 *   mo = u + g_f (c - u);  x0 = mo * (-sigma / sqrt(sigma^2+1)) + x / (sigma^2+1);  x' = x + (x - x0)/sigma * (sigma_next - sigma)
 * frames, frame_elems >= 1, n a multiple of frames * frame_elems, guidance non-NULL. */
int ca_cfg_euler_v(const void* eps_uncond, const void* eps_text, const float* latents_in, int64_t n,
                   const float* guidance, int32_t frames, int64_t frame_elems, const float* step_row,
                   int32_t round_latents_bf16, float* latents_out, void* model_in_next, void* cuda_stream);
int ca_cfg_ddim(const void* eps_uncond, const void* eps_text, const float* latents_in, int64_t n, float guidance,
                const float* step_row, int32_t round_latents_bf16, int32_t v_prediction, float* latents_out,
                void* model_in_next, void* cuda_stream);

/* I2VGen-XL image-latent temporal encoder (unet_i2vgen_xl.py:51-101, called at :648): per pixel, over the F frames of a
 * clip, on 4 channels: h = x + to_out(attn(LN(x))) (2 heads x 4); y = h + W2 gelu(W1 h).  Step-invariant conditioning,
 * computed once per generation.  x/y: [clips*frames, hw, c_stride] bf16 (first 4 channels used).  params: fp32 device
 * array {ln_w[4], ln_b[4], wq[8*4], wk[8*4], wv[8*4], wo[4*8], bo[4], w1[16*4], b1[16], w2[4*16], b2[4]}.
 * Constraints: 1 <= frames <= 32, c_stride >= 4, clips, hw >= 1. */
int ca_i2vgen_latent_encoder(const void* x, int32_t clips, int32_t frames, int64_t hw, int32_t c_stride,
                             const float* params, void* y, void* cuda_stream);

/*
 * VAE encoder posterior and image-latent assembly: diffusers DiagonalGaussianDistribution on the quant_conv output
 * (reached from `self.vae.encode(image).latent_dist` in the i2vgen pipeline :496 and the svd pipeline :221), then the
 * layouts the two denoising loops take.  Run once per call, not per step.
 * moments: channels-last bf16 [n, hw, 8] = (mean[4], logvar[4]); noise: DEVICE fp32 [n, 4, hw] or NULL (no noise).
 *   v = mean + exp(0.5 * clamp(logvar, -30, 20)) * noise       (v = mean when noise is NULL; fp32, one rounding)
 * layout / out (bf16):
 *   CA_VAE_POSTERIOR  [n, 4, hw]             v  (latent_dist.sample() / .mode()); frames = num_videos = 1
 *   CA_VAE_I2VGEN     [2*n*nv, 4, frames, hw] frame 0 = v * scale, frame k >= 1 = k / (frames - 1); the n images tiled
 *                                            nv times, then twice for classifier-free guidance (i2vgen pipeline :487-517)
 *   CA_VAE_SVD        [2*n*nv, frames, 4, hw] cat([zeros, v]) repeated nv times, then repeated over the frames
 *                                            (svd pipeline :214-235, :580-583)
 * latent_channels must be 4; moments 16-byte aligned.
 */
enum ca_vae_layout { CA_VAE_POSTERIOR = 0, CA_VAE_I2VGEN = 1, CA_VAE_SVD = 2 };
int ca_vae_latents(const void* moments, const float* noise, int32_t n, int64_t hw, int32_t latent_channels,
                   int32_t layout, int32_t frames, int32_t num_videos, float scale, void* out, void* cuda_stream);

/*
 * Temporal self-attention over the frame axis (diffusers TemporalBasicTransformerBlock.attn1 reached from
 * model/adapter_spatial_temporal.py:280).  q/k/v: rows of heads*64 bf16 with stride in_row_stride elements (views of a
 * fused QKV buffer), out: [clips*frames*hw, heads*64] dense; rows in (clip, frame, pixel)
 * order -- the (b f) s c <-> (b s) f c permutes of the reference are folded into the addressing.
 * Constraints: 1 <= frames <= 32; in_row_stride a multiple of 8; out 4-byte aligned.
 */
int ca_temporal_attention(const void* q, const void* k, const void* v, int32_t clips, int32_t frames, int64_t hw,
                          int32_t heads, float scale, int64_t in_row_stride, void* out, void* cuda_stream);

#ifdef __cplusplus
}
#endif
#endif /* CTRL_ADAPTER_B200_H_ */
