// Inception-v3 image encoder (the DAMSM CNN_ENCODER, ref: image_generation/model.py:182-287): the parts of its
// trunk that are not convolutions, and the helpers its convolutions need.  NHWC fp32, channels padded to 8.
//
//   * max_pool2d(3, 2) and avg_pool2d(3, 1, 1, count_include_pad=True), forward and backward;
//   * the final 8x8 average, forward and backward;
//   * the adjoint of F.interpolate(bilinear, align_corners=True) as a gather (og_bilinear_fwd is the forward);
//   * eval BatchNorm folded into the convolution: W' = W * s, b' = beta - mean * s, s = gamma / sqrt(var + eps);
//   * the gradient through a conv's ReLU epilogue between channel slices of concatenated block outputs.
//
// Every backward here is a gather: each input element sums its (at most a few) contributions in a fixed order, so two
// runs give the same bits.  No atomics.
#include "common.cuh"

namespace {

#define GRID_STRIDE(i, total) \
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < (total); i += (long long)gridDim.x * blockDim.x)

// ---------------------------------------------------------------------------------------------------------------
// max_pool2d(kernel 3, stride 2, no padding).  y may be a channel slice of a wider tensor: pixel stride ldy, offset
// yoff.  A window's maximum is the first maximum in PyTorch's scan order (row by row), NaN wins like in PyTorch.
// ---------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) maxpool3s2_fwd_kernel(const float* __restrict__ x, int H, int W, int C4, int OH,
                                                             int OW, long long total, float* __restrict__ y, int ldy,
                                                             int yoff) {
  GRID_STRIDE(i, total) {
    const int c = (int)(i % C4);
    long long t = i / C4;
    const int ow = (int)(t % OW);
    t /= OW;
    const int oh = (int)(t % OH);
    const long long n = t / OH;
    const float* src = x + ((n * H + 2 * oh) * W + 2 * ow) * (C4 * 4) + c * 4;
    float4 m = ldg4(src);
    for (int kh = 0; kh < 3; ++kh)
      for (int kw = 0; kw < 3; ++kw) {
        const float4 v = ldg4(src + ((long long)kh * W + kw) * (C4 * 4));
        if (v.x > m.x || isnan(v.x)) m.x = v.x;
        if (v.y > m.y || isnan(v.y)) m.y = v.y;
        if (v.z > m.z || isnan(v.z)) m.z = v.z;
        if (v.w > m.w || isnan(v.w)) m.w = v.w;
      }
    st4(y + ((n * OH + oh) * OW + ow) * ldy + yoff + c * 4, m);
  }
}

// gx[n, ih, iw, c] = sum over the windows (oh, ow) that contain (ih, iw) and whose first maximum is there of g
__global__ void __launch_bounds__(256) maxpool3s2_bwd_kernel(const float* __restrict__ x, const float* __restrict__ g,
                                                             int ldg, int goff, int H, int W, int C, int OH, int OW,
                                                             long long total, float* __restrict__ gx) {
  GRID_STRIDE(i, total) {
    const int c = (int)(i % C);
    long long t = i / C;
    const int iw = (int)(t % W);
    t /= W;
    const int ih = (int)(t % H);
    const long long n = t / H;
    const int oh0 = ih >= 2 ? (ih - 1) / 2 : 0, oh1 = min(ih / 2, OH - 1);
    const int ow0 = iw >= 2 ? (iw - 1) / 2 : 0, ow1 = min(iw / 2, OW - 1);
    const float* xn = x + n * H * W * C + c;
    float acc = 0.f;
    for (int oh = oh0; oh <= oh1; ++oh)
      for (int ow = ow0; ow <= ow1; ++ow) {
        int best = 0;
        float m = __ldg(xn + ((long long)(2 * oh) * W + 2 * ow) * C);
        for (int k = 1; k < 9; ++k) {
          const float v = __ldg(xn + ((long long)(2 * oh + k / 3) * W + 2 * ow + k % 3) * C);
          if (v > m || isnan(v)) {
            m = v;
            best = k;
          }
        }
        if (2 * oh + best / 3 == ih && 2 * ow + best % 3 == iw) acc += __ldg(g + ((n * OH + oh) * OW + ow) * ldg + goff + c);
      }
    gx[i] = acc;
  }
}

// ---------------------------------------------------------------------------------------------------------------
// avg_pool2d(kernel 3, stride 1, padding 1, count_include_pad=True): the sum of the window (zeros outside) over 9
// ---------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) avgpool3s1_kernel(const float* __restrict__ x, int H, int W, int C4,
                                                         long long total, float* __restrict__ y) {
  GRID_STRIDE(i, total) {
    const int c = (int)(i % C4);
    long long t = i / C4;
    const int w = (int)(t % W);
    t /= W;
    const int h = (int)(t % H);
    const long long n = t / H;
    float4 s = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int kh = -1; kh <= 1; ++kh) {
      if (h + kh < 0 || h + kh >= H) continue;
      for (int kw = -1; kw <= 1; ++kw) {
        if (w + kw < 0 || w + kw >= W) continue;
        const float4 v = ldg4(x + ((n * H + h + kh) * W + w + kw) * (C4 * 4) + c * 4);
        s.x += v.x; s.y += v.y; s.z += v.z; s.w += v.w;
      }
    }
    st4(y + i * 4, make_float4(s.x / 9.f, s.y / 9.f, s.z / 9.f, s.w / 9.f));
  }
}

// the adjoint: every window divides by 9, so gx[h, w] = sum over the windows centred at (h + kh, w + kw) of g / 9
__global__ void __launch_bounds__(256) avgpool3s1_bwd_kernel(const float* __restrict__ g, int H, int W, int C4,
                                                             long long total, float* __restrict__ gx) {
  GRID_STRIDE(i, total) {
    const int c = (int)(i % C4);
    long long t = i / C4;
    const int w = (int)(t % W);
    t /= W;
    const int h = (int)(t % H);
    const long long n = t / H;
    float4 s = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int kh = -1; kh <= 1; ++kh) {
      if (h + kh < 0 || h + kh >= H) continue;
      for (int kw = -1; kw <= 1; ++kw) {
        if (w + kw < 0 || w + kw >= W) continue;
        const float4 v = ldg4(g + ((n * H + h + kh) * W + w + kw) * (C4 * 4) + c * 4);
        s.x += v.x / 9.f; s.y += v.y / 9.f; s.z += v.z / 9.f; s.w += v.w / 9.f;
      }
    }
    st4(gx + i * 4, s);
  }
}

// ---------------------------------------------------------------------------------------------------------------
// global average over P pixels: y[n, c] = sum_p x[n, p, c] / P (pixels added in order), and its adjoint
// ---------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) global_avg_kernel(const float* __restrict__ x, int P, int C, long long total,
                                                         float* __restrict__ y) {
  GRID_STRIDE(i, total) {
    const int c = (int)(i % C);
    const long long n = i / C;
    const float* src = x + n * P * C + c;
    float s = 0.f;
    for (int p = 0; p < P; ++p) s += __ldg(src + (long long)p * C);
    y[i] = s / (float)P;
  }
}

__global__ void __launch_bounds__(256) global_avg_bwd_kernel(const float* __restrict__ g, int P, int C, long long total,
                                                             float* __restrict__ gx) {
  GRID_STRIDE(i, total) {
    const int c = (int)(i % C);
    const long long n = i / ((long long)P * C);
    gx[i] = __ldg(g + n * C + c) / (float)P;
  }
}

// ---------------------------------------------------------------------------------------------------------------
// adjoint of og_bilinear_fwd (align_corners=True) as a gather.  The forward maps output row o to source rows
// h0 = (int)(r * o) and h1 = h0 + (h0 < IH - 1) with weights 1 - l and l; input row i collects the rows o with h0 == i
// or h1 == i, which all lie in ((i - 1) / r, (i + 1) / r).  Same float arithmetic as the forward.
// ---------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ float bl_weight(int o, int i, float r, int IS) {
  const float f = r * o;
  const int a = (int)f;
  const int b = a + (a < IS - 1);
  const float l = f - a;
  return (a == i ? 1.f - l : 0.f) + (b == i ? l : 0.f);
}

// inv_r = 1 / r (0 when r == 0: every output row reads row 0); the range is widened by one row on each side
__device__ __forceinline__ void bl_range(int i, float inv_r, int OS, int& lo, int& hi) {
  if (inv_r == 0.f) {
    lo = 0;
    hi = OS - 1;
    return;
  }
  lo = max(0, (int)floorf((i - 1) * inv_r) - 1);
  hi = min(OS - 1, (int)ceilf((i + 1) * inv_r) + 1);
}

__global__ void __launch_bounds__(256) bilinear_bwd_gather_kernel(const float* __restrict__ g, int IH, int IW, int OH,
                                                                  int OW, int C, float rh, float rw, float inv_rh,
                                                                  float inv_rw, long long total, float* __restrict__ gx) {
  GRID_STRIDE(i, total) {
    const int c = (int)(i % C);
    long long t = i / C;
    const int iw = (int)(t % IW);
    t /= IW;
    const int ih = (int)(t % IH);
    const long long n = t / IH;
    int oh0, oh1, ow0, ow1;
    bl_range(ih, inv_rh, OH, oh0, oh1);
    bl_range(iw, inv_rw, OW, ow0, ow1);
    const float* gn = g + n * OH * OW * C + c;
    float acc = 0.f;
    for (int oh = oh0; oh <= oh1; ++oh) {
      const float wr = bl_weight(oh, ih, rh, IH);
      if (wr == 0.f) continue;
      for (int ow = ow0; ow <= ow1; ++ow) {
        const float wc = bl_weight(ow, iw, rw, IW);
        if (wc == 0.f) continue;
        acc += __ldg(gn + ((long long)oh * OW + ow) * C) * wr * wc;
      }
    }
    gx[i] = acc;
  }
}

// ---------------------------------------------------------------------------------------------------------------
// eval BatchNorm folded into a bias-free convolution: out channel co of w (R = Ci * KH * KW elements) times s[co]
// ---------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) bn_fold_kernel(const float* __restrict__ w, int Co, long long R,
                                                      const float* __restrict__ gamma, const float* __restrict__ beta,
                                                      const float* __restrict__ mean, const float* __restrict__ var,
                                                      float eps, float* __restrict__ wout, float* __restrict__ bout) {
  GRID_STRIDE(i, (long long)Co * R) {
    const int co = (int)(i / R);
    const double s = (double)gamma[co] / sqrt((double)var[co] + (double)eps);
    wout[i] = (float)((double)w[i] * s);
    if (i % R == 0) bout[co] = (float)((double)beta[co] - (double)mean[co] * s);
  }
}

// ---------------------------------------------------------------------------------------------------------------
// out[p, ooff + c] = (relu ? (y[p, yoff + c] > 0 ? g[p, goff + c] : 0) : g[p, goff + c]) for c < nch: the gradient
// through a conv's ReLU epilogue (torch's threshold_backward masks y > 0), between channel slices
// ---------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) relu_grad_slice_kernel(const float* __restrict__ y, int ldy, int yoff,
                                                              const float* __restrict__ g, int ldg, int goff,
                                                              float* __restrict__ out, int ldo, int ooff, int nch4,
                                                              int relu, long long total) {
  GRID_STRIDE(i, total) {
    const int c = (int)(i % nch4) * 4;
    const long long p = i / nch4;
    float4 v = ldg4(g + p * ldg + goff + c);
    if (relu) {
      const float4 o = ldg4(y + p * ldy + yoff + c);
      v.x = o.x > 0.f ? v.x : 0.f; v.y = o.y > 0.f ? v.y : 0.f;
      v.z = o.z > 0.f ? v.z : 0.f; v.w = o.w > 0.f ? v.w : 0.f;
    }
    st4(out + p * ldo + ooff + c, v);
  }
}

// ---------------------------------------------------------------------------------------------------------------
// The scoring networks' input (INCEPTION_V3 / INCEPTION_V3_FID, ref: model.py:301-315, 416-451): NCHW fp32 images
// in [-1, 1] -> the trunk's NHWC (N, 299, 299, 8) input, pad lanes zero, in one pass.
//   mode 0 (IS):  v = x * 0.5 + 0.5, v = (v - mean_c) / std_c, then bilinear resize with align_corners=True;
//   mode 1 (FID): bilinear resize with half-pixel centres (align_corners=False), then v = x * 0.5 + 0.5,
//                 v = v * a_c + b_c with a_c = std_c / 0.5, b_c = (mean_c - 0.5) / 0.5 (the reference's inverse of
//                 the usual normalisation, kept).
// Every step rounds to fp32 on its own as the reference's separate tensor ops do (no contraction into an FMA); the
// constants are the Python doubles rounded to fp32.  Mode 0 applies the affine to the four taps before they are
// blended, which is what affine-then-resize computes.
// ---------------------------------------------------------------------------------------------------------------
struct InceptionAffine {
  float m[3], s[3];      // mode 0: (v - m) / s;  mode 1: v * s + m
};

__device__ __forceinline__ float half_affine(float x) { return __fadd_rn(__fmul_rn(x, 0.5f), 0.5f); }

__device__ __forceinline__ void resize_coord(int o, int in, float r, int align, int& i0, int& i1, float& l) {
  float f = align ? r * o : fmaxf(__fsub_rn(__fmul_rn(r, o + 0.5f), 0.5f), 0.f);
  i0 = min((int)f, in - 1);
  i1 = i0 + (i0 < in - 1);
  l = fminf(f - i0, 1.f);
}

__global__ void __launch_bounds__(256) inception_input_kernel(const float* __restrict__ x, int H, int W, int OS,
                                                              int mode, float rh, float rw, InceptionAffine af,
                                                              long long total, float* __restrict__ y) {
  GRID_STRIDE(i, total) {
    const int ow = (int)(i % OS);
    long long t = i / OS;
    const int oh = (int)(t % OS);
    const long long n = t / OS;
    int h0, h1, w0, w1;
    float lh, lw;
    resize_coord(oh, H, rh, mode == 0, h0, h1, lh);
    resize_coord(ow, W, rw, mode == 0, w0, w1, lw);
    const float hh = 1.f - lh, hw = 1.f - lw;
    float v[3];
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const float* p = x + (n * 3 + c) * (long long)H * W;
      float a = __ldg(p + (long long)h0 * W + w0), b = __ldg(p + (long long)h0 * W + w1);
      float d = __ldg(p + (long long)h1 * W + w0), e = __ldg(p + (long long)h1 * W + w1);
      if (mode == 0) {
        a = __fdiv_rn(__fsub_rn(half_affine(a), af.m[c]), af.s[c]);
        b = __fdiv_rn(__fsub_rn(half_affine(b), af.m[c]), af.s[c]);
        d = __fdiv_rn(__fsub_rn(half_affine(d), af.m[c]), af.s[c]);
        e = __fdiv_rn(__fsub_rn(half_affine(e), af.m[c]), af.s[c]);
      }
      float r = hh * (hw * a + lw * b) + lh * (hw * d + lw * e);
      if (mode == 1) r = __fadd_rn(__fmul_rn(half_affine(r), af.s[c]), af.m[c]);
      v[c] = r;
    }
    st4(y + i * 8, make_float4(v[0], v[1], v[2], 0.f));
    st4(y + i * 8 + 4, make_float4(0.f, 0.f, 0.f, 0.f));
  }
}

// ---------------------------------------------------------------------------------------------------------------
// Row softmax y = exp(x - max) / sum exp(x - max) over C columns, one CTA per row.  Accurate expf; the per-thread
// partials (columns tid, tid + 256, ...) and the shared-memory tree combine in a fixed order, so results are
// deterministic.
// ---------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) softmax_rows_kernel(const float* __restrict__ x, int C, float* __restrict__ y) {
  __shared__ float red[256];
  const float* xr = x + (long long)blockIdx.x * C;
  float* yr = y + (long long)blockIdx.x * C;
  const int tid = threadIdx.x;
  float m = -INFINITY;
  for (int c = tid; c < C; c += 256) m = fmaxf(m, __ldg(xr + c));
  red[tid] = m;
  __syncthreads();
  for (int s = 128; s > 0; s >>= 1) {
    if (tid < s) red[tid] = fmaxf(red[tid], red[tid + s]);
    __syncthreads();
  }
  m = red[0];
  __syncthreads();
  float sum = 0.f;
  for (int c = tid; c < C; c += 256) {
    const float e = expf(__ldg(xr + c) - m);
    yr[c] = e;
    sum += e;
  }
  red[tid] = sum;
  __syncthreads();
  for (int s = 128; s > 0; s >>= 1) {
    if (tid < s) red[tid] += red[tid + s];
    __syncthreads();
  }
  const float total = red[0];
  for (int c = tid; c < C; c += 256) yr[c] = yr[c] / total;
}

// ---------------------------------------------------------------------------------------------------------------
// Streaming FID moments in fp64: for a batch x (n, d) fp32, s1[j] += sum_r (x[r, j] - k[j]) and
// s2[i, j] += sum_r (x[r, i] - k[i]) (x[r, j] - k[j]) for the tiles on or above the diagonal (tile row <= tile
// column; the caller mirrors the rest).  init = 1 starts the sums (s1, s2 are written, not added to).  k is the first row of the first batch (init = 1 also writes it): a sum of
// squares about a shift near the data does not cancel the way one about zero does.  Each element is summed by one
// thread over the rows in order, then added to the running total: deterministic.
// ---------------------------------------------------------------------------------------------------------------
constexpr int MT = 32;   // moment tile (MT x MT elements, 256 threads, 4 per thread)

__global__ void __launch_bounds__(256) moments_f64_kernel(const float* __restrict__ x, int n, int d, int init,
                                                          double* __restrict__ k, double* __restrict__ s1,
                                                          double* __restrict__ s2) {
  const int ti = blockIdx.y, tj = blockIdx.x;
  if (ti > tj) return;
  __shared__ double a[MT][MT + 1], b[MT][MT + 1];   // [row][column within the tile]
  const int tx = threadIdx.x % MT, ty = threadIdx.x / MT;
  const int i0 = ti * MT, j0 = tj * MT;
  const double ki = i0 + tx < d ? (init ? (double)__ldg(x + i0 + tx) : k[i0 + tx]) : 0.0;
  const double kj = j0 + tx < d ? (init ? (double)__ldg(x + j0 + tx) : k[j0 + tx]) : 0.0;
  double acc[4] = {0.0, 0.0, 0.0, 0.0}, acc1 = 0.0;
  for (int r0 = 0; r0 < n; r0 += MT) {
    __syncthreads();
    for (int r = ty; r < MT; r += 256 / MT) {
      const bool row = r0 + r < n;
      a[r][tx] = row && i0 + tx < d ? (double)__ldg(x + (long long)(r0 + r) * d + i0 + tx) - ki : 0.0;
      b[r][tx] = row && j0 + tx < d ? (double)__ldg(x + (long long)(r0 + r) * d + j0 + tx) - kj : 0.0;
    }
    __syncthreads();
    const int rn = min(MT, n - r0);
    for (int r = 0; r < rn; ++r) {
      const double bj = b[r][tx];
#pragma unroll
      for (int q = 0; q < 4; ++q) acc[q] = fma(a[r][ty + 8 * q], bj, acc[q]);
      if (ti == tj && ty == 0) acc1 += bj;
    }
  }
  if (j0 + tx >= d) return;
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    const int i = i0 + ty + 8 * q;
    double* o = s2 + (long long)i * d + j0 + tx;
    if (i < d) *o = init ? acc[q] : *o + acc[q];
  }
  if (ti == tj && ty == 0) {
    s1[j0 + tx] = init ? acc1 : s1[j0 + tx] + acc1;
    if (init) k[j0 + tx] = kj;
  }
}

}  // namespace

OG_API int og_maxpool3s2_fwd(const float* x, int N, int H, int W, int C, float* y, int ldy, int yoff,
                             cudaStream_t stream) {
  if (C % 4 || ldy % 4 || yoff % 4 || H < 3 || W < 3) return (int)cudaErrorInvalidValue;
  const int OH = (H - 3) / 2 + 1, OW = (W - 3) / 2 + 1;
  const long long total = (long long)N * OH * OW * (C / 4);
  if (total == 0) return 0;
  maxpool3s2_fwd_kernel<<<og_grid(total), 256, 0, stream>>>(x, H, W, C / 4, OH, OW, total, y, ldy, yoff);
  OG_RETURN_LAST_ERROR();
}

OG_API int og_maxpool3s2_bwd(const float* x, const float* g, int ldg, int goff, int N, int H, int W, int C, float* gx,
                             cudaStream_t stream) {
  if (H < 3 || W < 3) return (int)cudaErrorInvalidValue;
  const int OH = (H - 3) / 2 + 1, OW = (W - 3) / 2 + 1;
  const long long total = (long long)N * H * W * C;
  if (total == 0) return 0;
  maxpool3s2_bwd_kernel<<<og_grid(total), 256, 0, stream>>>(x, g, ldg, goff, H, W, C, OH, OW, total, gx);
  OG_RETURN_LAST_ERROR();
}

OG_API int og_avgpool3s1_fwd(const float* x, int N, int H, int W, int C, float* y, cudaStream_t stream) {
  if (C % 4) return (int)cudaErrorInvalidValue;
  const long long total = (long long)N * H * W * (C / 4);
  if (total == 0) return 0;
  avgpool3s1_kernel<<<og_grid(total), 256, 0, stream>>>(x, H, W, C / 4, total, y);
  OG_RETURN_LAST_ERROR();
}

OG_API int og_avgpool3s1_bwd(const float* g, int N, int H, int W, int C, float* gx, cudaStream_t stream) {
  if (C % 4) return (int)cudaErrorInvalidValue;
  const long long total = (long long)N * H * W * (C / 4);
  if (total == 0) return 0;
  avgpool3s1_bwd_kernel<<<og_grid(total), 256, 0, stream>>>(g, H, W, C / 4, total, gx);
  OG_RETURN_LAST_ERROR();
}

OG_API int og_global_avg_fwd(const float* x, int N, int P, int C, float* y, cudaStream_t stream) {
  const long long total = (long long)N * C;
  if (total == 0 || P == 0) return 0;
  global_avg_kernel<<<og_grid(total), 256, 0, stream>>>(x, P, C, total, y);
  OG_RETURN_LAST_ERROR();
}

OG_API int og_global_avg_bwd(const float* g, int N, int P, int C, float* gx, cudaStream_t stream) {
  const long long total = (long long)N * P * C;
  if (total == 0) return 0;
  global_avg_bwd_kernel<<<og_grid(total), 256, 0, stream>>>(g, P, C, total, gx);
  OG_RETURN_LAST_ERROR();
}

// gx is written (not accumulated); the same (rh, rw) as og_bilinear_fwd
OG_API int og_bilinear_bwd_gather(const float* g, int N, int IH, int IW, int C, int OH, int OW, float* gx,
                                  cudaStream_t stream) {
  const long long total = (long long)N * IH * IW * C;
  if (total == 0) return 0;
  const float rh = OH > 1 ? (float)(IH - 1) / (float)(OH - 1) : 0.f, rw = OW > 1 ? (float)(IW - 1) / (float)(OW - 1) : 0.f;
  bilinear_bwd_gather_kernel<<<og_grid(total), 256, 0, stream>>>(g, IH, IW, OH, OW, C, rh, rw, rh > 0.f ? 1.f / rh : 0.f,
                                                                   rw > 0.f ? 1.f / rw : 0.f, total, gx);
  OG_RETURN_LAST_ERROR();
}

OG_API int og_bn_fold(const float* w, int Co, long long R, const float* gamma, const float* beta, const float* mean,
                      const float* var, float eps, float* wout, float* bout, cudaStream_t stream) {
  if ((long long)Co * R == 0) return 0;
  bn_fold_kernel<<<og_grid((long long)Co * R), 256, 0, stream>>>(w, Co, R, gamma, beta, mean, var, eps, wout, bout);
  OG_RETURN_LAST_ERROR();
}

OG_API int og_relu_grad_slice(const float* y, int ldy, int yoff, const float* g, int ldg, int goff, float* out, int ldo,
                              int ooff, int nch, long long P, int relu, cudaStream_t stream) {
  if (nch % 4 || ldy % 4 || yoff % 4 || ldg % 4 || goff % 4 || ldo % 4 || ooff % 4) return (int)cudaErrorInvalidValue;
  const long long total = P * (nch / 4);
  if (total == 0) return 0;
  relu_grad_slice_kernel<<<og_grid(total), 256, 0, stream>>>(y, ldy, yoff, g, ldg, goff, out, ldo, ooff, nch / 4, relu,
                                                              total);
  OG_RETURN_LAST_ERROR();
}

// x: (N, 3, H, W) NCHW fp32 contiguous; y: (N, 299, 299, 8) -- OS x OS in general.  mode 0: IS, 1: FID (see above)
OG_API int og_inception_input(const float* x, int N, int H, int W, int OS, int mode, float* y, cudaStream_t stream) {
  if (H < 1 || W < 1 || OS < 1 || (mode != 0 && mode != 1)) return (int)cudaErrorInvalidValue;
  const long long total = (long long)N * OS * OS;
  if (total == 0) return 0;
  const double mean[3] = {0.485, 0.456, 0.406}, std_[3] = {0.229, 0.224, 0.225};
  InceptionAffine af;
  for (int c = 0; c < 3; ++c) {
    af.m[c] = mode == 0 ? (float)mean[c] : (float)((mean[c] - 0.5) / 0.5);
    af.s[c] = mode == 0 ? (float)std_[c] : (float)(std_[c] / 0.5);
  }
  float rh, rw;
  if (mode == 0) {
    rh = OS > 1 ? (float)(H - 1) / (float)(OS - 1) : 0.f;
    rw = OS > 1 ? (float)(W - 1) / (float)(OS - 1) : 0.f;
  } else {
    rh = (float)H / (float)OS;
    rw = (float)W / (float)OS;
  }
  inception_input_kernel<<<og_grid(total), 256, 0, stream>>>(x, H, W, OS, mode, rh, rw, af, total, y);
  OG_RETURN_LAST_ERROR();
}

OG_API int og_softmax_rows(const float* x, int rows, int C, float* y, cudaStream_t stream) {
  if (rows == 0 || C == 0) return 0;
  if (rows < 0 || C < 0) return (int)cudaErrorInvalidValue;
  softmax_rows_kernel<<<rows, 256, 0, stream>>>(x, C, y);
  OG_RETURN_LAST_ERROR();
}

// k, s1: (d) fp64, s2: (d, d) fp64 (only the tiles on or above the diagonal are written)
OG_API int og_moments_f64(const float* x, int n, int d, int init, double* k, double* s1, double* s2,
                          cudaStream_t stream) {
  if (n < 1 || d < 1 || (init != 0 && init != 1)) return (int)cudaErrorInvalidValue;
  const int t = (d + MT - 1) / MT;
  moments_f64_kernel<<<dim3(t, t), 256, 0, stream>>>(x, n, d, init, k, s1, s2);
  OG_RETURN_LAST_ERROR();
}
