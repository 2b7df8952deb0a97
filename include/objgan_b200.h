/* objgan_b200 -- C ABI of libobjgan_b200.so (sm_90a kernels for the Obj-GAN image_generation hot path).
 *
 * Plain pointers and sizes only; every pointer is a DEVICE pointer unless stated otherwise; every call is
 * asynchronous on `stream` and re-entrant (no global mutable state), which is what the reference's one FFI
 * crossing requires (models/roi_align/src/roi_align_cuda.c:5,31: global THCState, current-stream launch).
 *
 * Return convention: og_* functions return 0 on success, else the cudaError_t of the failed call.  The two
 * ROIAlign*Laucher symbols keep the reference convention (1 = ok, 0 = error) because they are the literal
 * drop-ins for models/roi_align/src/roi_align_kernel.h:13-27.  Nothing in this library calls exit().
 *
 * Activations are NHWC fp32 ("rows" = pixels, channels contiguous), channel counts padded to a multiple of
 * 8 with zero lanes; the module boundary (NCHW, unpadded -- the reference's public layout) is crossed with
 * og_nchw_to_nhwc / og_nhwc_to_nchw.  All "ref:" paths are relative to /root/reference/image_generation/.
 */
#ifndef OBJGAN_B200_H
#define OBJGAN_B200_H

#include <cuda_runtime_api.h>

#ifdef __cplusplus
extern "C" {
#endif

/* ---- codes ---- */
enum { OG_ACT_NONE = 0, OG_ACT_LRELU = 1, OG_ACT_TANH = 2, OG_ACT_SIGMOID = 3 };  /* conv epilogue activations  */
enum { OG_NA_NONE = 0, OG_NA_LRELU = 1, OG_NA_GLU = 2 };                          /* norm-apply fusions         */
enum { OG_PAD_ZERO = 0, OG_PAD_REFLECT = 1, OG_UPSAMPLE2X = 2, OG_TRANSPOSED = 3 }; /* conv source addressing   */

/* ------------------------------------------------------------------------------------------------------
 * ROIAlign -- replaces ref: models/roi_align/src/roi_align_kernel.h:13-27 (same names, argument order,
 * NCHW fp32 features, rois = [batch_idx, x1, y1, x2, y2] rows, caller zero-fills outputs;
 * callers: models/roi_align/src/roi_align_cuda.c:33-38, 70-73).
 * ---------------------------------------------------------------------------------------------------- */
int ROIAlignForwardLaucher(const float* bottom_data, const float spatial_scale, const int num_rois, const int height,
                           const int width, const int channels, const int aligned_height, const int aligned_width,
                           const float* bottom_rois, float* top_data, cudaStream_t stream);
int ROIAlignBackwardLaucher(const float* top_diff, const float spatial_scale, const int batch_size, const int num_rois,
                            const int height, const int width, const int channels, const int aligned_height,
                            const int aligned_width, const float* bottom_rois, float* bottom_diff, cudaStream_t stream);
/* fused RoIAlignAvg(AH, AW, scale) = align to (AH+1)x(AW+1) then avg_pool2d(2, 1)
 * -- replaces ref: models/roi_align/modules/roi_align.py:18-29 (used at model.py:1241, 1307). */
int og_roi_align_avg_fwd(const float* features, int height, int width, int channels, const float* rois, int num_rois,
                         int AH, int AW, float spatial_scale, float* out, cudaStream_t stream);
int og_roi_align_avg_bwd(const float* grad_out, int height, int width, int channels, const float* rois, int num_rois,
                         int AH, int AW, float spatial_scale, float* grad_features, cudaStream_t stream);

/* channels-last variant (features NHWC [B][H][W][C], out NHWC [R][AH][AW][C], C % 4 == 0): identical values, coalesced
 * 16-byte loads / stores / vector atomics; what the object discriminators use internally (their feature maps are
 * produced channels-last), the NCHW entry points above stay the drop-in for the reference's callers. */
int og_roi_align_avg_nhwc_fwd(const float* features, int height, int width, int channels, const float* rois,
                              int num_rois, int AH, int AW, float spatial_scale, float* out, cudaStream_t stream);
int og_roi_align_avg_nhwc_bwd(const float* grad_out, int height, int width, int channels, const float* rois,
                              int num_rois, int AH, int AW, float spatial_scale, float* grad_features,
                              cudaStream_t stream);

/* ------------------------------------------------------------------------------------------------------
 * Convolutions / linear layers as implicit GEMM -- replaces the cuDNN/cuBLAS calls behind nn.Conv2d /
 * nn.Linear in ref: model.py:36-39 (conv3x3), 43-49 (upBlock), 52-60 (downBlock_G), 63-81 (HmapResBlock),
 * 455-518 (CA_NET / INIT_STAGE_G fc), 589-617 (G_HMAP), 708-719 (GET_IMAGE_G), 999-1048 (D stacks).
 * x: source NHWC [N,H,W,C] with element strides (xsn,xsh,xsw); y likewise [N,OH,OW,K]; C % 8 == 0, K % 4 == 0.
 * mode selects how a (row pixel, tap) pair maps to a source pixel: zero padding, reflection padding
 * (nn.ReflectionPad2d), nearest-2x upsampling followed by zero padding (nn.Upsample + conv), or the
 * transposed map used for the input gradient.  wpacked is produced by og_pack_weights.  padh / padw: row / column
 * padding (they differ for the 1x7, 7x1, 1x3 and 3x1 kernels of the Inception-v3 image encoder).
 * ---------------------------------------------------------------------------------------------------- */
int og_conv2d_simt(const float* x, int N, int H, int W, int C, long long xsn, long long xsh, long long xsw,
                   const float* wpacked, float* y, int OH, int OW, int K, long long ysn, long long ysh, long long ysw,
                   int KH, int KW, int stride, int padh, int padw, int mode, const float* bias, int act, float slope,
                   int allow_splitk, cudaStream_t stream);
int og_conv2d_wgrad_simt(const float* x, int N, int H, int W, int C, long long xsn, long long xsh, long long xsw,
                         const float* g, int OH, int OW, int K, long long gsn, long long gsh, long long gsw,
                         float* dw_packed, int KH, int KW, int stride, int pad, int mode, cudaStream_t stream);
/* <= 8 output channels with a long reduction (the k4 s2 p0 logit heads, ref: model.py:1031-1033): dot-product
 * kernels instead of GEMM tiles.  Contiguous NHWC, zero padding, output channels padded to 8, wpacked [(kh,kw,ci)][8]. */
int og_conv2d_narrow_fwd(const float* x, int N, int H, int W, int C, const float* wpacked, float* y, int OH, int OW,
                         int KH, int KW, int stride, int pad, const float* bias, int act, float slope,
                         cudaStream_t stream);
int og_conv2d_narrow_dgrad(const float* g, int N, int H, int W, int C, const float* wpacked, float* gx, int OH, int OW,
                           int KH, int KW, int stride, int pad, cudaStream_t stream);
int og_conv2d_narrow_wgrad(const float* x, int N, int H, int W, int C, const float* g, float* dw_packed, int OH, int OW,
                           int KH, int KW, int stride, int pad, cudaStream_t stream);
/* OIHW parameter (state_dict layout, SURVEY 8b) <-> kernel-native matrices (csrc/operands.cu).  split/splitp: GLU
 * halves of the output channels are each padded to splitp.  transposed=1 gives the dgrad operand ([tap][co][ci]
 * instead of [tap][ci][co]).  og_pack_weights_f16 writes the same matrices as the fp16 hi/lo operand pair of the
 * tensor-core path, scaled by the power of two derived from *amax (og_amax over the parameter; see og_prep_split). */
int og_pack_weights(const float* w_oihw, int Co, int Ci, int KH, int KW, int Cip, int Kp, int split, int splitp,
                    int transposed, float* out, cudaStream_t stream);
int og_pack_weights_f16(const float* w_oihw, int Co, int Ci, int KH, int KW, int Cip, int Kp, int split, int splitp,
                        int transposed, const unsigned* amax, void* hi, void* lo, cudaStream_t stream);
int og_unpack_wgrad(const float* dw_packed, int Co, int Ci, int KH, int KW, int Cip, int Kp, int split, int splitp,
                    float* grad_oihw, int accumulate, int transposed, cudaStream_t stream);

/* upBlock (nearest 2x upsample + conv3x3, ref: model.py:43-49) as four 2x2 phase convolutions with pre-summed
 * weights (csrc/operands.cu): Wp[16][..] (tap t = ((p*2+q)*2+a)*2+b) from the OIHW parameter as fp16 hi/lo operands
 * (scale word *amax_up = 4 * *amax, the bound of the pre-sums), and the adjoint map for the gradient (accumulate = 1
 * adds it to grad_oihw, a persistent gradient buffer, like og_unpack_wgrad). */
int og_pack_upsample_weights(const float* w_oihw, int Co, int Ci, int Cip, int Kp, int split, int splitp,
                             int transposed, const unsigned* amax, unsigned* amax_up, void* hi, void* lo,
                             cudaStream_t stream);
int og_unpack_upsample_wgrad(const float* dwp, int Co, int Ci, int Cip, int Kp, int split, int splitp,
                             float* grad_oihw, int accumulate, cudaStream_t stream);

/* Tensor-core path (wgmma f16 with fp32 register accumulators, TMA operand staging) for the
 * contractions that dominate the step (HmapResBlock / upBlock / jointConv / discriminator convs: forward, input
 * and weight gradients).  Operands are fp16 hi/lo pairs (22 mantissa bits; "3xFP16": a*b ~ ah*bh + al*bh + ah*bl)
 * of x * 2^k, k = og_scale_exp(max|x|) per tensor; the word *amax holds max|x| as float bits and travels with the
 * operand (the format: csrc/operand.cuh).  og_prep_split (csrc/operands.cu) computes *amax and writes the pair for
 * an activation tensor (pad=1 also materialises the nn.ReflectionPad2d(1) halo, ref: model.py:67; s2d=1 writes the
 * four space-to-depth phase blocks used by the stride-2 convs of the discriminators and by the adjoint of the 2x
 * upsampling); og_conv2d_tc computes
 *     y[n, osy*h+opy, osx*w+opx, :] = act(bias + sum_t x[n+dn_t, h+dh_t, w+dw_t, :] * W[widx_t])   (x OOB = 0)
 * with taps = ntaps host quadruples (dh, dw, dn, widx), as the error-compensated product (fp32-level accuracy).
 * Every entry point that takes a hi / lo pair returns cudaErrorInvalidValue if either pointer is null. */
int og_amax(const float* x, long long n, unsigned* amax, cudaStream_t stream);
int og_prep_split(const float* x, int N, int H, int W, int C, int pad, int s2d, unsigned* amax, int amax_ready,
                  void* xh, void* xl, cudaStream_t stream);
int og_conv2d_tc(const void* xh, const void* xl, const unsigned* amax_x, int N, int SN, int SH, int SW, int C,
                 const void* wh, const void* wl, const unsigned* amax_w, int ntaps_w, int Kw, float* y, int OH, int OW,
                 int K, long long ysn, long long ysh, long long ysw, int OHf, int OWf, int osy, int osx, int opy,
                 int opx, const int* taps_host, int ntaps, const float* bias, int act, float slope,
                 cudaStream_t stream);
/* Weight gradient: dw[tap][co][ci] = sum_{n,h,w} G[n+gdn, h, w, co] * X[n+xdn, h+dh, w+dw, ci]  (X out of range = 0).
 * Both operands are the same NHWC fp16 hi/lo tensors og_prep_split writes for the forward / input-gradient kernels
 * (G: [GN][OH][OW][Kp], X: [XN][SH][SW][C]; GN / XN = N or 4N space-to-depth blocks), consumed MN-major by
 * wgmma; each needs 512 readable bytes after its last element.
 * entries_host: nentries quintuples (gdn, dh, dw, xdn, output tap); dw is [ntaps_out][Kp][C], zero-filled here. */
int og_conv2d_wgrad_tc(const void* gh, const void* gl, const unsigned* amax_g, int N, int GN, int OH, int OW, int Kp,
                       const void* xh, const void* xl, const unsigned* amax_x, int XN, int SH, int SW, int C, float* dw,
                       int ntaps_out, const int* entries_host, int nentries, cudaStream_t stream);

/* ------------------------------------------------------------------------------------------------------
 * InstanceNorm2d / BatchNorm (train and eval mode) + fused GLU / LeakyReLU / residual
 * -- replaces ref: model.py:19-27 (GLU), 47, 70, 75, 497, 602, 992, 1011 (norm layers).
 * groups = N (instance norm) or 1 (batch norm); P pixels per group; contiguous rows of C channels.
 * amax_out / amax_dy (optional): receive max|out| / max|dy| as float bits, so that a convolution consuming the
 * tensor can skip the amax pass of og_prep_split (amax_ready = 1).
 * ---------------------------------------------------------------------------------------------------- */
int og_norm_stats(const float* x, int groups, long long P, int C, float eps, double* stats, float* mean, float* rstd,
                  float* running_mean, float* running_var, float momentum, int real_c, long long* num_batches_tracked,
                  cudaStream_t stream);
int og_norm_apply(const float* y, int groups, long long P, int Cy, const float* mean, const float* rstd,
                  const float* gamma, const float* beta, const float* res, int act, float slope, float* out,
                  unsigned* amax_out, cudaStream_t stream);
/* og_norm_apply that also emits the fp16 hi / lo tensor-core operand copies of its output (what og_prep_split would
 * make of it, optionally with the reflection halo), scaled by the a-priori bound og_norm_bound leaves in bound_word;
 * out (fp32) may be null when nothing else reads the activation */
int og_norm_bound(const float* gamma, const float* beta, int C, long long count, const unsigned* res_word,
                  unsigned* out_word, cudaStream_t stream);
int og_norm_apply_split(const float* y, int N, int H, int W, int Cy, int instance, const float* mean,
                        const float* rstd, const float* gamma, const float* beta, const float* res, int act,
                        float slope, float* out, const unsigned* bound_word, int pad, void* xh, void* xl,
                        cudaStream_t stream);
int og_norm_backward(const float* y, const float* g, int groups, long long P, int Cy, const float* mean,
                     const float* rstd, const float* gamma, const float* beta, int act, float slope, double* bstats,
                     float* dy, float* dgamma, float* dbeta, int accumulate_param_grads, unsigned* amax_dy,
                     cudaStream_t stream);
/* BatchNorm in eval mode (ref: nn.BatchNorm{1,2}d after .eval(), evaluator.py:110): the running statistics, only read,
 * give mean = running_mean and rstd = 1 / sqrt(running_var + eps), which og_norm_apply (groups = 1) consumes.
 * og_bn_eval_backward is the matching backward: activation backward, then dy = g' * gamma * rstd,
 * dgamma = sum g' * (y - mean) * rstd, dbeta = sum g' (no batch-statistic terms; per-channel sums in a fixed order,
 * so repeated calls give identical results).  dgamma / dbeta may both be null. */
int og_bn_eval_coef(const float* running_mean, const float* running_var, int C, float eps, float* mean, float* rstd,
                    cudaStream_t stream);
int og_bn_eval_backward(const float* y, const float* g, long long P, int Cy, const float* mean, const float* rstd,
                        const float* gamma, const float* beta, int act, float slope, float* dy, float* dgamma,
                        float* dbeta, int accumulate_param_grads, unsigned* amax_dy, cudaStream_t stream);

/* ------------------------------------------------------------------------------------------------------
 * Attention -- replaces ref: GlobalAttention.py:32-70 (func_attention), 73-122 (GlobalAttentionGeneral),
 * 125-181 (GlobalBUAttentionGeneral) and miscc/utils.py:401-413 (pprocess_bt_attns).
 * mask: [B][L] bytes, 1 = padding word; the reference's mask-row permutation quirk is reproduced.
 * ---------------------------------------------------------------------------------------------------- */
int og_words_proj(const float* words, const float* W, int B, int idf, int cdf, int L, float* src, cudaStream_t stream);
int og_words_proj_bwd(const float* words, const float* W, const float* gsrc, int B, int idf, int cdf, int L, float* gW,
                      int accumulate, float* gwords, cudaStream_t stream);
int og_att_general_fwd(const float* h, const float* src, const unsigned char* mask, int B, int Q, int idf, int cs,
                       int L, float* wc, float* attn, cudaStream_t stream);
int og_att_general_bwd(const float* h, const float* src, const float* attn, const float* g_wc, int B, int Q, int idf,
                       int cs, int L, float* g_h, float* g_src, cudaStream_t stream);
int og_bu_att_fwd(const float* labels, const float* glove, const float* src, const unsigned char* mask, int B, int E,
                  int R, int L, int idf, int norm, float eps, float* wc, float* attn, cudaStream_t stream);
int og_bu_att_bwd(const float* attn, const float* g_wc, int B, int R, int L, int idf, float* g_src,
                  cudaStream_t stream);
int og_paint_max_fwd(const float* f, const float* m, int B, int num, int R, int Rtot, long long P, float* out,
                     int dstride, int doff, cudaStream_t stream);
int og_paint_max_bwd(const float* f, const float* m, const float* g, int gstride, int goff, int B, int num, int R,
                     int Rtot, long long P, float* g_f, cudaStream_t stream);
int og_func_attention_fwd(const float* query, const float* ctx, int B, int ndf, int Lq, int S, float gamma1, float* wc,
                          float* attn, cudaStream_t stream);
int og_func_attention_bwd(const float* query, const float* ctx, const float* attn, const float* g_wc,
                          const float* g_attn, int B, int ndf, int Lq, int S, float gamma1, float* g_query, float* g_ctx,
                          cudaStream_t stream);

/* ------------------------------------------------------------------------------------------------------
 * Layout, adjoints of pad / upsample, concat, losses, optimiser
 * -- replaces ATen elementwise kernels behind ref: model.py:45 (Upsample), 67 (ReflectionPad2d), torch.cat at
 * model.py:579, 697, 1041; nn.BCELoss in miscc/losses.py:178-208, 378-393; KL_loss miscc/losses.py:533-537;
 * CA_NET.reparametrize model.py:470-478; optim.Adam + EMA trainer.py:197-224, 461-462.
 * ---------------------------------------------------------------------------------------------------- */
int og_nchw_to_nhwc(const float* x, int N, int C, int H, int W, int Cp, float* y, cudaStream_t stream);
int og_nhwc_to_nchw(const float* y, int N, int C, int H, int W, int Cp, float* x, cudaStream_t stream);
int og_act_backward(const float* out, const float* g, long long n, int act, float slope, float* gin,
                    cudaStream_t stream);
int og_channel_sum(const float* x, long long P, int C, double* scratch, float* out, int n_out, int accumulate,
                   cudaStream_t stream);
int og_upsample2x_bwd(const float* gu, int N, int H, int W, int C, float* gx, cudaStream_t stream);
int og_reflect_pad_fwd(const float* x, int N, int H, int W, int C, float* xp, cudaStream_t stream);
int og_reflect_pad_bwd(const float* gpad, int N, int H, int W, int C, float* gx, cudaStream_t stream);
int og_copy_channels(const float* src, int sstride, int soff, float* dst, int dstride, int doff, int nch, long long P,
                     int accumulate, cudaStream_t stream);
int og_broadcast_channels(const float* c, int B, int Cc, float* dst, int dstride, int doff, long long pix_per_img,
                          cudaStream_t stream);
int og_broadcast_channels_bwd(const float* g, int B, int Cc, int gstride, int goff, long long pix_per_img, float* gc,
                              cudaStream_t stream);   /* gc[b][k] = sum_pixels g[pixel][goff + k] */
/* Row gather out[i,:] = x[idx[i],:] (idx: int64 device array) and its adjoint (gx zero-filled, then += g rows):
 * the roi compaction of feat_select (ref: miscc/utils.py:465-499) and the raw_conditions[classes] lookup of
 * objD_loss (ref: miscc/losses.py:280-281) without per-roi host loops. */
int og_gather_rows(const float* x, const long long* idx, long long n_out, long long rowlen, float* out,
                   cudaStream_t stream);
int og_scatter_rows_add(const float* g, const long long* idx, long long n_out, long long n_in, long long rowlen,
                        float* gx, cudaStream_t stream);
int og_add(const float* a, const float* b, float* out, long long n, cudaStream_t stream);
/* F.interpolate(bilinear, align_corners=True) on NHWC (ref: model.py:1217-1218, 1283-1284) and its adjoint */
int og_bilinear_fwd(const float* x, int N, int IH, int IW, int C, int OH, int OW, float* y, cudaStream_t stream);
int og_bilinear_bwd(const float* g, int N, int IH, int IW, int C, int OH, int OW, float* gx, cudaStream_t stream);
int og_glu_fwd(const float* x, long long P, int Ch, float* out, cudaStream_t stream);
int og_glu_bwd(const float* x, const float* g, long long P, int Ch, float* gx, cudaStream_t stream);
int og_reparam_fwd(const float* x, int xs, const float* eps, int B, int D, float* c, int cs, cudaStream_t stream);
int og_reparam_bwd(const float* x, int xs, const float* eps, const float* gc, int gcs, int B, int D, float* gx,
                   cudaStream_t stream);
int og_bce(const float* p, long long n, float target, float weight, float* loss_accum, float* gp, cudaStream_t stream);
int og_kl(const float* x, int xs, int B, int D, float weight, float* loss_accum, float* gx, cudaStream_t stream);
/* step: 1-based Adam step from the host, or (step_dev != NULL) read from a device counter so that a whole training
 * step can be replayed from a CUDA graph; og_inc_i64 bumps such a counter. */
int og_adam_ema(float* p, const float* g, float* m, float* v, float* avg, long long n, double lr, double b1, double b2,
                double eps, int step, const long long* step_dev, float gscale, float decay, cudaStream_t stream);
int og_inc_i64(long long* counter, cudaStream_t stream);

/* ------------------------------------------------------------------------------------------------------
 * DAMSM matching losses (ref: miscc/losses.py:22-71, 131-147: sent_loss and the cross-entropies of words_loss; the
 * word-level similarities are og_words_pairs_*).  Dense row-major fp32; B <= 128 captions (og_ce_pair: the R-precision pool of 100).
 *  og_cosine_matrix_* : out[i][j] = <a_i, b_j> / max(|a_i||b_j|, eps); backward w.r.t. a   (losses.py:43-50)
 *  og_ce_pair         : scores = gamma3 * sim with masked entries at -inf; loss0 = CrossEntropy(scores, labels),
 *                       loss1 = CrossEntropy(scores^T, labels) (means), their gradients G0 / G1 w.r.t. sim, and the
 *                       number of top-1 hits of both directions (losses.py:50-68, 131-147)
 *  og_ce_pair_bwd     : gsim = *g0 * G0 + *g1 * G1 (device scalars; NULL = 0)
 * ---------------------------------------------------------------------------------------------------- */
int og_cosine_matrix_fwd(const float* a, const float* b, int Ba, int Bb, int D, float eps, float* out,
                         cudaStream_t stream);
int og_cosine_matrix_bwd(const float* a, const float* b, const float* g, int Ba, int Bb, int D, float eps, float* ga,
                         cudaStream_t stream);
int og_ce_pair(const float* sim, const unsigned char* mask, const long long* labels, int B, float gamma3, float* loss0,
               float* loss1, float* G0, float* G1, float* correct, cudaStream_t stream);
int og_ce_pair_bwd(const float* G0, const float* G1, const float* g0, const float* g1, int n, float* gsim,
                   cudaStream_t stream);

/* All (image, caption) pairs of words_loss in ONE launch (ref: miscc/losses.py:87-127 -- the reference calls
 * func_attention once per caption in a Python loop).  words [NC][ndf][T] (caption i uses its first lens[i] words),
 * ctx [B][ndf][S] image region features (NCHW flattened), lens [NC] int64 on the device.  pair p = b * NC + i.
 *  fwd: wc [B*NC][ndf][T] (weighted contexts), attn [B*NC][T][S], sim [B][NC] = log sum_l exp(gamma2 * cos_l)
 *       (rows / columns beyond a caption's length are not written)
 *  bwd: g_ctx [B][ndf][S] = d (sum_p g_sim[p] * sim[p]) / d ctx  (zero-filled by the call, fp32 atomics) */
int og_words_pairs_fwd(const float* words, const float* ctx, const long long* lens, int B, int NC, int ndf, int T, int S,
                       float gamma1, float gamma2, float eps, float* wc, float* attn, float* sim, cudaStream_t stream);
int og_words_pairs_bwd(const float* words, const float* ctx, const long long* lens, const float* wc, const float* attn,
                       const float* g_sim, int B, int NC, int ndf, int T, int S, float gamma1, float gamma2, float eps,
                       float* g_ctx, cudaStream_t stream);

/* Device-side input preparation (ref: trainDataset.py:79-128, miscc/load.py:160-176, miscc/utils.py:502-522):
 *  og_form_hmaps        : out[b][cls[b][r]][p] += masks[b][r][p] for r < num_rois[b], in roi order (the loader's loop);
 *                         clamp_max > 0 additionally clamps the touched channels (synthetic inputs); out NCHW, zeroed here
 *  og_form_clabels_feat : out[b][e][r] = emb[cls[b][r]][e] for r < num_rois[b], else 0   (B, E, Rmax, 1) */
int og_form_hmaps(const float* masks, const long long* cls, const long long* num_rois, int B, int R, long long P,
                  int ncls, float clamp_max, float* out, cudaStream_t stream);
int og_form_clabels_feat(const float* emb, const long long* cls, const long long* num_rois, int B, int R, int Rmax, int E,
                         int ncls, float* out, cudaStream_t stream);

/* Whole-network weight re-packing after an optimiser step: og_amax + og_pack_weights_f16 for EVERY registered
 * (weight, layout) of a network in one launch each, from a device-resident int64 job table (csrc/operands.cu).
 *  amax job (4 fields): x, n, out word, first block index;  a block covers 4096 elements
 *  pack job (14 fields): w (OIHW), hi, lo (or 0), amax word, Co, Ci, taps, Cip, Kp, split, splitp, transposed, total,
 *                        first block index */
int og_amax_multi(const long long* jobs, int njobs, int total_blocks, cudaStream_t stream);
int og_pack_weights_f16_multi(const long long* jobs, int njobs, int total_blocks, cudaStream_t stream);

/* out[b][c] = x[b][perm[b][c]] over NCHW planes of P floats (permute_seg's class-channel shuffle, utils.py:445-462) */
int og_permute_channels(const float* x, const long long* perm, int B, int C, long long P, float* out,
                        cudaStream_t stream);

/* ------------------------------------------------------------------------------------------------------
 * Shape generator (SHP_G_NET, ref: model.py:798-985) and heat maps from generated masks (miscc/utils.py:524-584)
 *  og_form_bbox_maps : the loader's one-hot box maps (ref: miscc/load.py:178-189, 625-641) from the compact batch.
 *                      rois / fm_rois: float64 [B][boxes][*stride] rows (x, y, w, h, ...), cls / num_rois int64.
 *                      maps NHWC [2][B][R][S][S][Cp]: forward sequence (slot t), then backward (slot boxes-1-t: the
 *                      reversal covers all box slots before the [:R] slice); fmaps [B][R][F][F] from fm_rois / 2.
 *                      Box edges: min(round-half-even(v), size - 1), upper bound exclusive; slots >= num_rois are 0.
 *  og_clstm_cell     : one ConvLSTM step (ref: model.py:818-863) of BOTH directions.  gx_*: x-part of Gates incl. bias
 *                      for every step, NHWC [B*R][HW][4*Ch] (image b*R + t); gh_*: conv(h_{t-1}, W_h) [B][HW][4*Ch],
 *                      both null at t = 0 (zero state: c_prev = 0).  c_* [B][HW][Ch] updated in place; h_* [B][HW][Ch]
 *                      written; h also written to joint [B*R][HW][Cj]: forward at (b*R + t, channels [0, Ch)),
 *                      backward at (b*R + R-1-t, channels [Ch, 2Ch)).
 *  og_mul_pixels     : out[p][c] = x[p][c] * s[p] (the crop by the box feature maps, ref: model.py:969-972)
 *  og_gen_hmaps      : form_hmaps' normalisation and class composite.  slots NHWC [B][P][Cs] (lane t = roi slot t,
 *                      Cs <= 16): slots t < num_rois[b] normalised in place, the others left raw; hmap NHWC
 *                      [B][P][Cp] written (class channels, every present one renormalised).  cls [B][boxes].
 *                      Fixed-order reductions, no atomics. */
int og_form_bbox_maps(const double* rois, int rois_stride, const double* fm_rois, int fm_stride, const long long* cls,
                      const long long* num_rois, int B, int boxes, int R, int ncls, int Cp, int S, int F, float* maps,
                      float* fmaps, cudaStream_t stream);
int og_clstm_cell(const float* gx_f, const float* gx_b, const float* gh_f, const float* gh_b, float* c_f, float* c_b,
                  float* h_f, float* h_b, float* joint, int B, int R, int t, int HW, int Ch, int Cj,
                  cudaStream_t stream);
int og_mul_pixels(const float* x, const float* s, long long P, int C, float* out, cudaStream_t stream);
int og_gen_hmaps(float* slots, int B, long long P, int Cs, const long long* cls, int boxes, const long long* num_rois,
                 int ncls, int Cp, float* hmap, cudaStream_t stream);

/* ------------------------------------------------------------------------------------------------------
 * Text encoder and word inputs of caption-conditioned sampling (ref: model.py:85-179 RNN_ENCODER in eval mode,
 * evaluator.py:337-351, 148-164)
 *  og_lstm_bidir      : the whole recurrence of a one-layer bidirectional LSTM (H = 128 per direction) in one launch.
 *                       gx [B*L][8H]: x-part of the gates plus b_ih + b_hh at every step (row b*L + t; forward
 *                       direction in channels [0, 4H), backward in [4H, 8H), gate order i, f, g, o); whh_* [4H][H];
 *                       lens [B] int64 in [1, L].  Sample b runs its own lens[b] steps each way from a zero state;
 *                       words [B][2H][L] (forward in channels [0, H), backward in [H, 2H), every column t >= lens[b]
 *                       zero); sent [B][2H] = [forward h after token lens[b]-1, backward h after token 0].  Fixed-order
 *                       fp32 FMA, no atomics: a sample's outputs do not depend on B or on its place in the batch.
 *  og_text_inputs     : glove_words [B][E][L] = glove[glove_ids[b][t]] and mask [B][L] bytes = (captions[b][t] == 0),
 *                       t < L, from row-major int64 id tables with row strides cap_ld / glove_ld (>= L).
 *  og_class_label_emb : prepare_cat_emb: row k of the labels [n][lab_ld] is the mean of its first lens[k] GloVe vectors
 *                       when lens[k] is 1 or 2, else zeros; out [n][E] row i = row order[i]. */
int og_lstm_bidir(const float* gx, const float* whh_f, const float* whh_b, const long long* lens, int B, int L, int H,
                  float* words, float* sent, cudaStream_t stream);
int og_text_inputs(const long long* captions, int cap_ld, const long long* glove_ids, int glove_ld, const float* glove,
                   int E, int B, int L, float* glove_words, unsigned char* mask, cudaStream_t stream);
int og_class_label_emb(const float* glove, int E, const long long* labels, int lab_ld, const long long* lens,
                       const long long* order, int n, float* out, cudaStream_t stream);
/* og_lstm_bidir_state: og_lstm_bidir that also writes the final cell state cell [B][2H] in the layout of sent (the
 *                       forward c after token lens[b]-1, the backward c after token 0), the encoder state the box
 *                       decoder starts from (ref: box_generation/seq2seq/models/PreEncoderRNN.py:59-99). */
int og_lstm_bidir_state(const float* gx, const float* whh_f, const float* whh_b, const long long* lens, int B, int L,
                        int H, float* words, float* sent, float* cell, cudaStream_t stream);

/* ------------------------------------------------------------------------------------------------------
 * Box generator of caption-to-image sampling (ref: box_generation/seq2seq/models/DecoderRNN.py:81-183, 260-292,
 * 350-384 in inference; seq2seq/evaluator/evaluator.py:74-139; image_generation/miscc/load.py:653-776)
 *  og_box_label_table : table [NL][1024] = b_ih + b_hh + W_ih[:, 100:356] emb[l], one fmaf chain per entry in column
 *                       order; W_ih [1024][356] row-major, emb [NL][256].
 *  og_box_decode      : every decoding step of B samples in one launch.  h0 / c0 [B][256] (encoder directions
 *                       concatenated); wt [356][1024] = [W_ih[:, 0:100] | W_hh]^T; *_w (50, 2) and *_b (50,) of
 *                       xy_embedding / wh_embedding / next_xy_embedding; lout_t [256][NL], xyo_t [256+NL][30] and
 *                       who_t [256+NL+50][30] the transposed heads; noise [B][S][6] = (u_xy, n1, n2, u_wh, n3, n4),
 *                       uniforms in [0, 1) and standard normals.  The first step reads label sos and (x0, y0, w0, r0);
 *                       a sample stops after the step whose label is eos or after S steps.  labels [B][S] (-1 after
 *                       the end), samples [B][S][4] normalised (x, y, w, r; 0 after the end), steps [B]; dbg null or
 *                       [B][S][NL + 60]: p, then the xy and wh mixture parameters (pi, mu_x, mu_y, sigma_x, sigma_y,
 *                       rho, 5 each, sigma before the temperature), 0 after the end.  Fixed-order fp32, no atomics: a
 *                       sample's results do not depend on B or its place in the batch.  NL <= 128.
 *  og_box_layout      : the evaluator's post-processing and load_gen_insanns per sample, in float64: mean_std [4][2]
 *                       (mean, std of x, y, w, r), label_to_class [NL] (class row, -1 for the special tokens),
 *                       count_stats [C][2] (mu, sigma of the per-class count), noise_cnt [B][C] standard normals.
 *                       rois [3][B][R][6] at 64, 128 and 256 pixels, fm_rois [B][R][6], roi_cls [B][R], num_rois [B],
 *                       zero-padded to R slots.  S <= 16.  It is og_box_records' rows through the boxes.txt round
 *                       trip int(float('%.2f' % v)), the ROI_MIN_SIZE filter (min_size) and the three scales.
 *  og_box_records     : the rows Evaluator.evaluate writes to boxes.txt, per sample in float64, from the same inputs as
 *                       og_box_layout: rows [B][S][4] (x, y, w, h after the clip; not rounded, no size filter, zero
 *                       after the end), row_cls [B][S] (class row), n_rows [B], n_valid [B] (valid steps before the
 *                       last is dropped; the reference writes a dev_bbox_test.txt line only when it is > 1) and
 *                       n_special [B] (boxes dropped for a special label, where the reference raises).  S <= 16.
 *  og_box_noise       : noise_box [B][S][6] and noise_cnt [B][C] of captions first .. first + B - 1, each a function of
 *                       (seed, caption index) only: Philox4x32-10 of (value, stream, index) under the key seed >= 0;
 *                       columns 0 and 3 of noise_box uniform in [0, 1), every other value a standard normal. */
int og_box_label_table(const float* emb, const float* w_ih, const float* b_ih, const float* b_hh, int NL, float* table,
                       cudaStream_t stream);
int og_box_decode(const float* h0, const float* c0, const float* table, const float* wt, const float* xy_w,
                  const float* xy_b, const float* wh_w, const float* wh_b, const float* nxy_w, const float* nxy_b,
                  const float* lout_t, const float* lout_b, const float* xyo_t, const float* xyo_b, const float* who_t,
                  const float* who_b, const float* noise, int B, int S, int NL, int sos, int eos, float x0, float y0,
                  float w0, float r0, long long* labels, float* samples, long long* steps, float* dbg,
                  cudaStream_t stream);
int og_box_layout(const long long* labels, const float* samples, const long long* steps, const double* mean_std,
                  const long long* label_to_class, const double* count_stats, const float* noise_cnt, int B, int S,
                  int NL, int C, int R, int min_size, double* rois, double* fm_rois, long long* roi_cls,
                  long long* num_rois, cudaStream_t stream);
int og_box_records(const long long* labels, const float* samples, const long long* steps, const double* mean_std,
                   const long long* label_to_class, const double* count_stats, const float* noise_cnt, int B, int S,
                   int NL, int C, double* rows, long long* row_cls, long long* n_rows, long long* n_valid,
                   long long* n_special, cudaStream_t stream);
int og_box_noise(long long seed, long long first, int B, int S, int C, float* noise_box, float* noise_cnt,
                 cudaStream_t stream);

/* zero-fill (a memset node when captured in a CUDA graph; no kernel launch) */
int og_zero_bytes(float* p, long long bytes, cudaStream_t stream);

/* ----------------------------------------------------------------------------------------------------
 * Inception-v3 image encoder (CNN_ENCODER, ref: model.py:182-287; csrc/inception.cu).  NHWC fp32, C % 8 == 0.
 * Pooling: max_pool2d(3, 2) (output may be a channel slice: pixel stride ldy, offset yoff; the backward reads the
 * gradient slice the same way), avg_pool2d(3, 1, 1, count_include_pad=True), the global average over P pixels; every
 * backward is a deterministic gather.  og_bilinear_bwd_gather: adjoint of og_bilinear_fwd without atomics.
 * og_bn_fold: eval BatchNorm folded into a bias-free conv (wout = w * s, bout = beta - mean * s, s = gamma /
 * sqrt(var + eps), R = Ci * KH * KW).  og_prep_split_s2d (csrc/operands.cu): og_prep_split(s2d=1) for any H, W
 * (phase blocks of ceil(H/2) x ceil(W/2), zero past an odd edge).  og_relu_grad_slice: out[p, ooff + c] =
 * g[p, goff + c] masked by y[p, yoff + c] > 0 (relu = 1) or copied (relu = 0), c < nch.
 * ---------------------------------------------------------------------------------------------------- */
int og_maxpool3s2_fwd(const float* x, int N, int H, int W, int C, float* y, int ldy, int yoff, cudaStream_t stream);
int og_maxpool3s2_bwd(const float* x, const float* g, int ldg, int goff, int N, int H, int W, int C, float* gx,
                      cudaStream_t stream);
int og_avgpool3s1_fwd(const float* x, int N, int H, int W, int C, float* y, cudaStream_t stream);
int og_avgpool3s1_bwd(const float* g, int N, int H, int W, int C, float* gx, cudaStream_t stream);
int og_global_avg_fwd(const float* x, int N, int P, int C, float* y, cudaStream_t stream);
int og_global_avg_bwd(const float* g, int N, int P, int C, float* gx, cudaStream_t stream);
int og_bilinear_bwd_gather(const float* g, int N, int IH, int IW, int C, int OH, int OW, float* gx,
                           cudaStream_t stream);
int og_bn_fold(const float* w, int Co, long long R, const float* gamma, const float* beta, const float* mean,
               const float* var, float eps, float* wout, float* bout, cudaStream_t stream);
int og_prep_split_s2d(const float* x, int N, int H, int W, int C, unsigned* amax, int amax_ready, void* xh, void* xl,
                      cudaStream_t stream);
/* Scoring networks (INCEPTION_V3 / INCEPTION_V3_FID, ref: model.py:290-451; csrc/inception.cu).
 * og_inception_input: NCHW (N, 3, H, W) images in [-1, 1] -> NHWC (N, OS, OS, 8), pad lanes zero; mode 0 (IS): the
 * affine x * 0.5 + 0.5, (v - mean) / std, then the align_corners=True resize; mode 1 (FID): the half-pixel resize, then
 * x * 0.5 + 0.5, v * (std / 0.5) + (mean - 0.5) / 0.5.  og_softmax_rows: softmax over the C columns of each row,
 * deterministic.  og_moments_f64: adds one batch x (n, d) fp32 to the fp64 sums s1 = sum (x - k) and s2 = sum (x - k)
 * (x - k)^T (tiles on or above the diagonal); init = 1 sets k to the batch's first row and starts the sums. */
int og_inception_input(const float* x, int N, int H, int W, int OS, int mode, float* y, cudaStream_t stream);
int og_softmax_rows(const float* x, int rows, int C, float* y, cudaStream_t stream);
int og_moments_f64(const float* x, int n, int d, int init, double* k, double* s1, double* s2, cudaStream_t stream);
int og_relu_grad_slice(const float* y, int ldy, int yoff, const float* g, int ldg, int goff, float* out, int ldo,
                       int ooff, int nch, long long P, int relu, cudaStream_t stream);
/* og_images_to_u8: NCHW (N, 3, H, W) fp32 images -> NHWC (N, H, W, 3) bytes with the arithmetic of the evaluator's
 * save_singleimages (ref: evaluator.py:235-237): round(round(x + 1) * 0.5 * 255), clamped to [0, 255], truncated
 * toward zero; NaN gives 0 (csrc/elementwise.cu). */
int og_images_to_u8(const float* x, int N, int H, int W, unsigned char* out, cudaStream_t stream);

/* og_snapshot_canvas: the pixels of one attention-map snapshot PNG (ref: miscc/utils.py:59-306, build_super_images /
 * build_super_shape_images) for images i < nvis, without the caption glyphs: uint8 HWC `out` of
 * (nvis * (strip + 2 vis)) x ((words + 2) (vis + 2)) pixels.  img (>= nvis, 3, img_side, img_side) and lr (the same
 * with lr_side; NULL: img) are fp32 in [-1, 1]; maps (>= nvis, L, att, att) fp32; lens (>= nvis) int64 map counts
 * per image (NULL: L each).  vis must be a multiple of att; upscale vis / att > 1 expands every map with skimage
 * 0.14's pyramid_expand(sigma=20) in float64 (then vis must be a multiple of 4 and above 80).  per_map selects the
 * shape snapshots' per-map min / max (guarded by max != min) instead of one pair per image starting at (1, 0).
 * Workspaces: maxmap nvis att^2 floats; mm0 and stats nvis (L + 1) 2 doubles; with upscale > 1 also work
 * nvis (L + 1) vis^2 and part nvis (L + 1) (vis / 4) 2 doubles (else NULL).  words <= 20 (the caption colours).
 * Five launches with upscale > 1, three without (csrc/snapshot.cu). */
int og_snapshot_canvas(const float* img, int img_side, const float* lr, int lr_side, const float* maps, int L,
                       int att, const long long* lens, int nvis, int vis, int words, int strip, int per_map,
                       float* maxmap, double* mm0, double* work, double* part, double* stats, unsigned char* out,
                       cudaStream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* OBJGAN_B200_H */
