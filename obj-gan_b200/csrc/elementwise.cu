// Bandwidth-bound helper kernels: layout conversion at the module boundary, activation / padding /
// upsampling adjoints, channel concat, losses (BCE, KL), CA_NET reparametrisation, fused Adam + EMA.
// Reference semantics cited per kernel (paths under /root/reference/image_generation/).
#include "common.cuh"

// ---------------------------------------------------------------------------------------------
// NCHW <-> NHWC(+channel padding).  Public tensors are NCHW fp32 like the reference's; kernels run NHWC.
// ---------------------------------------------------------------------------------------------
__global__ void nchw_to_nhwc_kernel(const float* __restrict__ x, int C, int HW, int Cp, float* __restrict__ y) {
  __shared__ float tile[32][33];
  const int n = blockIdx.z;
  const int p0 = blockIdx.x * 32, c0 = blockIdx.y * 32;
  const float* xn = x + (long long)n * C * HW;
  float* yn = y + (long long)n * HW * Cp;
  for (int j = threadIdx.y; j < 32; j += 8) {
    int c = c0 + j, p = p0 + threadIdx.x;
    tile[j][threadIdx.x] = (c < C && p < HW) ? xn[(long long)c * HW + p] : 0.f;
  }
  __syncthreads();
  for (int j = threadIdx.y; j < 32; j += 8) {
    int p = p0 + j, c = c0 + threadIdx.x;
    if (p < HW && c < Cp) yn[(long long)p * Cp + c] = tile[threadIdx.x][j];
  }
}

__global__ void nhwc_to_nchw_kernel(const float* __restrict__ y, int C, int HW, int Cp, float* __restrict__ x) {
  __shared__ float tile[32][33];
  const int n = blockIdx.z;
  const int p0 = blockIdx.x * 32, c0 = blockIdx.y * 32;
  const float* yn = y + (long long)n * HW * Cp;
  float* xn = x + (long long)n * C * HW;
  for (int j = threadIdx.y; j < 32; j += 8) {
    int p = p0 + j, c = c0 + threadIdx.x;
    tile[j][threadIdx.x] = (p < HW && c < Cp) ? yn[(long long)p * Cp + c] : 0.f;
  }
  __syncthreads();
  for (int j = threadIdx.y; j < 32; j += 8) {
    int c = c0 + j, p = p0 + threadIdx.x;
    if (c < C && p < HW) xn[(long long)c * HW + p] = tile[threadIdx.x][j];
  }
}

OG_API int og_nchw_to_nhwc(const float* x, int N, int C, int H, int W, int Cp, float* y, cudaStream_t stream) {
  if (N == 0) return 0;
  dim3 grid(og_cdiv((long long)H * W, 32), og_cdiv(Cp, 32), N), block(32, 8);
  nchw_to_nhwc_kernel<<<grid, block, 0, stream>>>(x, C, H * W, Cp, y);
  OG_RETURN_LAST_ERROR();
}
OG_API int og_nhwc_to_nchw(const float* y, int N, int C, int H, int W, int Cp, float* x, cudaStream_t stream) {
  if (N == 0) return 0;
  dim3 grid(og_cdiv((long long)H * W, 32), og_cdiv(Cp, 32), N), block(32, 8);
  nhwc_to_nchw_kernel<<<grid, block, 0, stream>>>(y, C, H * W, Cp, x);
  OG_RETURN_LAST_ERROR();
}

// ---------------------------------------------------------------------------------------------
// gradient through a conv-epilogue activation, from the saved OUTPUT (LeakyReLU / tanh / sigmoid)
// ---------------------------------------------------------------------------------------------
__global__ void act_backward_kernel(const float* __restrict__ out, const float* __restrict__ g, long long n4, int act,
                                    float slope, float* __restrict__ gin) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n4;
       i += (long long)gridDim.x * blockDim.x) {
    float4 o = ldg4(out + i * 4), gg = ldg4(g + i * 4), r;
    if (act == OG_ACT_LRELU) {
      r.x = o.x > 0.f ? gg.x : gg.x * slope; r.y = o.y > 0.f ? gg.y : gg.y * slope;
      r.z = o.z > 0.f ? gg.z : gg.z * slope; r.w = o.w > 0.f ? gg.w : gg.w * slope;
    } else if (act == OG_ACT_TANH) {
      r.x = gg.x * (1.f - o.x * o.x); r.y = gg.y * (1.f - o.y * o.y);
      r.z = gg.z * (1.f - o.z * o.z); r.w = gg.w * (1.f - o.w * o.w);
    } else if (act == OG_ACT_SIGMOID) {
      r.x = gg.x * o.x * (1.f - o.x); r.y = gg.y * o.y * (1.f - o.y);
      r.z = gg.z * o.z * (1.f - o.z); r.w = gg.w * o.w * (1.f - o.w);
    } else {
      r = gg;
    }
    st4(gin + i * 4, r);
  }
}
OG_API int og_act_backward(const float* out, const float* g, long long n, int act, float slope, float* gin,
                           cudaStream_t stream) {
  if (n % 4) return (int)cudaErrorInvalidValue;
  if (n == 0) return 0;
  act_backward_kernel<<<og_grid(n / 4), 256, 0, stream>>>(out, g, n / 4, act, slope, gin);
  OG_RETURN_LAST_ERROR();
}

// ---------------------------------------------------------------------------------------------
// per-channel sum over pixels (conv bias gradient).  fp64 partials: each CTA stores its sums to plane blockIdx.y of a
// [chunks][C] workspace, and store_sum_kernel adds the planes in a fixed order.
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) channel_sum_kernel(const float* __restrict__ x, int C, long long P,
                                                          int pix_per_block, double* __restrict__ part) {
  const int c4 = blockIdx.x * 32 + threadIdx.x;
  const int C4 = C >> 2;
  const long long p0 = (long long)blockIdx.y * pix_per_block, p1 = min(P, p0 + pix_per_block);
  double s[4] = {0, 0, 0, 0};
  if (c4 < C4)
    for (long long p = p0 + threadIdx.y; p < p1; p += 8) {
      float4 v = ldg4(x + p * C + c4 * 4);
      s[0] += v.x; s[1] += v.y; s[2] += v.z; s[3] += v.w;
    }
  og_cta_channel_sums(s, C4, C, C, part + (long long)blockIdx.y * C);
}
// one warp per channel: acc[c] = the fp64 sum, out[c] (c < n_out) = it rounded to fp32 (added to out[c] when accumulating)
__global__ void store_sum_kernel(const double* __restrict__ part, int S, int C, double* __restrict__ acc, int n_out,
                                 float* out, int accumulate) {
  const int i = (int)((blockIdx.x * (long long)blockDim.x + threadIdx.x) >> 5);
  if (i >= C) return;
  double a[1];
  og_plane_sum(part + i, 0, S, C, a);
  if (threadIdx.x & 31) return;
  acc[i] = a[0];
  if (i < n_out) out[i] = accumulate ? out[i] + (float)a[0] : (float)a[0];
}
OG_API int og_channel_sum(const float* x, long long P, int C, double* scratch, float* out, int n_out, int accumulate,
                          cudaStream_t stream) {
  if (C % 4) return (int)cudaErrorInvalidValue;
  int cg = og_cdiv(C / 4, 32);
  long long chunks = (long long)og_num_sms() * 8 / cg + 1;
  long long ppb = (P + chunks - 1) / chunks;
  if (ppb < 64) ppb = 64;
  dim3 grid(cg, og_cdiv(P, ppb)), block(32, 8);
  double* part = nullptr;
  if (P > 0) {
    OG_CHECK(og_work_alloc(&part, (size_t)grid.y * C, stream));
    channel_sum_kernel<<<grid, block, 0, stream>>>(x, C, P, (int)ppb, part);
  }
  store_sum_kernel<<<og_cdiv(C, 8), 256, 0, stream>>>(part, (int)grid.y, C, scratch, n_out, out, accumulate);
  const int rc = (int)cudaGetLastError();
  const cudaError_t e = part ? cudaFreeAsync(part, stream) : cudaSuccess;
  return rc ? rc : (int)e;
}

// ---------------------------------------------------------------------------------------------
// adjoint of nn.Upsample(scale_factor=2, mode='nearest') (model.py:45): sum of the 4 children
// ---------------------------------------------------------------------------------------------
__global__ void upsample2x_bwd_kernel(const float* __restrict__ gu, int H, int W, int C4, long long total,
                                      float* __restrict__ gx) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    int c = (int)(i % C4);
    long long t = i / C4;
    int w = (int)(t % W);
    t /= W;
    int h = (int)(t % H);
    long long n = t / H;
    const float* b = gu + (((n * 2 * H + 2 * h) * 2 * W + 2 * w) * C4 + c) * 4;
    long long rs = (long long)2 * W * C4 * 4;
    float4 a = ldg4(b), b1 = ldg4(b + C4 * 4), c0 = ldg4(b + rs), c1 = ldg4(b + rs + C4 * 4);
    st4(gx + i * 4, make_float4(a.x + b1.x + c0.x + c1.x, a.y + b1.y + c0.y + c1.y, a.z + b1.z + c0.z + c1.z,
                                a.w + b1.w + c0.w + c1.w));
  }
}
OG_API int og_upsample2x_bwd(const float* gu, int N, int H, int W, int C, float* gx, cudaStream_t stream) {
  if (C % 4) return (int)cudaErrorInvalidValue;
  long long total = (long long)N * H * W * (C / 4);
  if (total == 0) return 0;
  upsample2x_bwd_kernel<<<og_grid(total), 256, 0, stream>>>(gu, H, W, C / 4, total, gx);
  OG_RETURN_LAST_ERROR();
}

// ---------------------------------------------------------------------------------------------
// nn.ReflectionPad2d(1) (model.py:67, 72, 600): forward materialisation and adjoint (fold).
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ int refl(int i, int n) { return i < 0 ? -i : (i >= n ? 2 * n - 2 - i : i); }

__global__ void reflect_pad_fwd_kernel(const float* __restrict__ x, int H, int W, int C4, long long total,
                                       float* __restrict__ xp) {
  const int Hp = H + 2, Wp = W + 2;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    int c = (int)(i % C4);
    long long t = i / C4;
    int w = (int)(t % Wp);
    t /= Wp;
    int h = (int)(t % Hp);
    long long n = t / Hp;
    int sh = refl(h - 1, H), sw = refl(w - 1, W);
    st4(xp + i * 4, ldg4(x + (((n * H + sh) * W + sw) * C4 + c) * 4));
  }
}
OG_API int og_reflect_pad_fwd(const float* x, int N, int H, int W, int C, float* xp, cudaStream_t stream) {
  if (C % 4) return (int)cudaErrorInvalidValue;
  long long total = (long long)N * (H + 2) * (W + 2) * (C / 4);
  if (total == 0) return 0;
  reflect_pad_fwd_kernel<<<og_grid(total), 256, 0, stream>>>(x, H, W, C / 4, total, xp);
  OG_RETURN_LAST_ERROR();
}

__global__ void reflect_pad_bwd_kernel(const float* __restrict__ gp, int H, int W, int C4, long long total,
                                       float* __restrict__ gx) {
  const int Wp = W + 2, Hp = H + 2;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    int c = (int)(i % C4);
    long long t = i / C4;
    int w = (int)(t % W);
    t /= W;
    int h = (int)(t % H);
    long long n = t / H;
    // padded rows/cols that read input row h: h+1 always; row 0 if h == 1; row H+1 if h == H-2
    int hs[3], nh = 0, ws[3], nw = 0;
    hs[nh++] = h + 1;
    if (h == 1) hs[nh++] = 0;
    if (h == H - 2) hs[nh++] = H + 1;
    ws[nw++] = w + 1;
    if (w == 1) ws[nw++] = 0;
    if (w == W - 2) ws[nw++] = W + 1;
    float4 a = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int ih = 0; ih < nh; ++ih)
      for (int iw = 0; iw < nw; ++iw) {
        float4 v = ldg4(gp + (((n * Hp + hs[ih]) * Wp + ws[iw]) * C4 + c) * 4);
        a.x += v.x; a.y += v.y; a.z += v.z; a.w += v.w;
      }
    st4(gx + i * 4, a);
  }
}
OG_API int og_reflect_pad_bwd(const float* gpad, int N, int H, int W, int C, float* gx, cudaStream_t stream) {
  if (C % 4) return (int)cudaErrorInvalidValue;
  long long total = (long long)N * H * W * (C / 4);
  if (total == 0) return 0;
  reflect_pad_bwd_kernel<<<og_grid(total), 256, 0, stream>>>(gpad, H, W, C / 4, total, gx);
  OG_RETURN_LAST_ERROR();
}

// ---------------------------------------------------------------------------------------------
// channel-slice copy (torch.cat along channels and its adjoint), optional accumulate
// ---------------------------------------------------------------------------------------------
__global__ void copy_channels_kernel(const float* __restrict__ src, int sstride, int soff, float* __restrict__ dst,
                                     int dstride, int doff, int nch, long long P, int accumulate) {
  long long total = P * nch;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    long long p = i / nch;
    int c = (int)(i - p * nch);
    float v = src[p * sstride + soff + c];
    float* d = dst + p * dstride + doff + c;
    *d = accumulate ? *d + v : v;
  }
}
OG_API int og_copy_channels(const float* src, int sstride, int soff, float* dst, int dstride, int doff, int nch,
                            long long P, int accumulate, cudaStream_t stream) {
  if (P * nch == 0) return 0;
  copy_channels_kernel<<<og_grid(P * nch), 256, 0, stream>>>(src, sstride, soff, dst, dstride, doff, nch, P, accumulate);
  OG_RETURN_LAST_ERROR();
}

// adjoint of broadcast_channels w.r.t. the code: gc[b][k] = sum over the image's pixels of g[pixel][goff + k]
// (needed when the conditioning code carries a gradient: the object-discriminator terms of G_loss, losses.py:436-452)
__global__ void broadcast_channels_bwd_kernel(const float* __restrict__ g, int Cc, int gstride, int goff,
                                              long long pix_per_img, long long total, float* __restrict__ gc) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const long long b = i / Cc;
    const int k = (int)(i - b * Cc);
    const float* src = g + b * pix_per_img * gstride + goff + k;
    float acc = 0.f;
    for (long long p = 0; p < pix_per_img; ++p) acc += src[p * gstride];
    gc[i] = acc;
  }
}
OG_API int og_broadcast_channels_bwd(const float* g, int B, int Cc, int gstride, int goff, long long pix_per_img,
                                     float* gc, cudaStream_t stream) {
  long long total = (long long)B * Cc;
  if (total == 0) return 0;
  broadcast_channels_bwd_kernel<<<og_grid(total), 256, 0, stream>>>(g, Cc, gstride, goff, pix_per_img, total, gc);
  OG_RETURN_LAST_ERROR();
}

// row gather out[i, :] = x[idx[i], :] and its adjoint gx[idx[i], :] += g[i, :]  (feat_select's roi compaction,
// ref: miscc/utils.py:465-499, and the raw_conditions[classes] lookup, miscc/losses.py:280-281, without host loops)
__global__ void gather_rows_kernel(const float* __restrict__ x, const long long* __restrict__ idx, long long n_out,
                                   long long rowlen, float* __restrict__ out) {
  const long long total = n_out * rowlen;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const long long r = i / rowlen, c = i - r * rowlen;
    out[i] = x[idx[r] * rowlen + c];
  }
}
__global__ void scatter_rows_add_kernel(const float* __restrict__ g, const long long* __restrict__ idx, long long n_out,
                                        long long rowlen, float* __restrict__ gx) {
  const long long total = n_out * rowlen;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const long long r = i / rowlen, c = i - r * rowlen;
    atomicAdd(gx + idx[r] * rowlen + c, g[i]);
  }
}
OG_API int og_gather_rows(const float* x, const long long* idx, long long n_out, long long rowlen, float* out,
                          cudaStream_t stream) {
  if (n_out * rowlen == 0) return 0;
  gather_rows_kernel<<<og_grid(n_out * rowlen), 256, 0, stream>>>(x, idx, n_out, rowlen, out);
  OG_RETURN_LAST_ERROR();
}
// gx ([n_in][rowlen]) is zero-filled here, then receives the scattered rows
OG_API int og_scatter_rows_add(const float* g, const long long* idx, long long n_out, long long n_in, long long rowlen,
                               float* gx, cudaStream_t stream) {
  OG_CHECK(cudaMemsetAsync(gx, 0, sizeof(float) * (size_t)(n_in * rowlen), stream));
  if (n_out * rowlen == 0) return 0;
  scatter_rows_add_kernel<<<og_grid(n_out * rowlen), 256, 0, stream>>>(g, idx, n_out, rowlen, gx);
  OG_RETURN_LAST_ERROR();
}

// c_code (B, Cc) broadcast over each image's pixels into a channel slice (D_GET_LOGITS, model.py:1037-1041)
__global__ void broadcast_channels_kernel(const float* __restrict__ c, int Cc, float* __restrict__ dst, int dstride,
                                          int doff, long long pix_per_img, long long total) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    long long p = i / Cc;
    int k = (int)(i - p * Cc);
    long long b = p / pix_per_img;
    dst[p * dstride + doff + k] = c[b * Cc + k];
  }
}
OG_API int og_broadcast_channels(const float* c, int B, int Cc, float* dst, int dstride, int doff,
                                 long long pix_per_img, cudaStream_t stream) {
  long long total = (long long)B * pix_per_img * Cc;
  if (total == 0) return 0;
  broadcast_channels_kernel<<<og_grid(total), 256, 0, stream>>>(c, Cc, dst, dstride, doff, pix_per_img, total);
  OG_RETURN_LAST_ERROR();
}

__global__ void add_kernel(const float* __restrict__ a, const float* __restrict__ b, float* __restrict__ o,
                           long long n4) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n4;
       i += (long long)gridDim.x * blockDim.x) {
    float4 x = ldg4(a + i * 4), y = ldg4(b + i * 4);
    st4(o + i * 4, make_float4(x.x + y.x, x.y + y.y, x.z + y.z, x.w + y.w));
  }
}
OG_API int og_add(const float* a, const float* b, float* out, long long n, cudaStream_t stream) {
  if (n % 4) return (int)cudaErrorInvalidValue;
  if (n == 0) return 0;
  add_kernel<<<og_grid(n / 4), 256, 0, stream>>>(a, b, out, n / 4);
  OG_RETURN_LAST_ERROR();
}

// ---------------------------------------------------------------------------------------------
// GLU without normalisation (CA_NET, model.py:464-468): rows of 2*Ch channels -> Ch
// ---------------------------------------------------------------------------------------------
__global__ void glu_fwd_kernel(const float* __restrict__ x, int Ch, long long total, float* __restrict__ o) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    long long p = i / Ch;
    int c = (int)(i - p * Ch);
    o[i] = x[p * 2 * Ch + c] * og_sigmoid(x[p * 2 * Ch + Ch + c]);
  }
}
__global__ void glu_bwd_kernel(const float* __restrict__ x, const float* __restrict__ g, int Ch, long long total,
                               float* __restrict__ gx) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    long long p = i / Ch;
    int c = (int)(i - p * Ch);
    float a = x[p * 2 * Ch + c], s = og_sigmoid(x[p * 2 * Ch + Ch + c]), gg = g[i];
    gx[p * 2 * Ch + c] = gg * s;
    gx[p * 2 * Ch + Ch + c] = gg * a * s * (1.f - s);
  }
}
OG_API int og_glu_fwd(const float* x, long long P, int Ch, float* out, cudaStream_t stream) {
  if (P * Ch == 0) return 0;
  glu_fwd_kernel<<<og_grid(P * Ch), 256, 0, stream>>>(x, Ch, P * Ch, out);
  OG_RETURN_LAST_ERROR();
}
OG_API int og_glu_bwd(const float* x, const float* g, long long P, int Ch, float* gx, cudaStream_t stream) {
  if (P * Ch == 0) return 0;
  glu_bwd_kernel<<<og_grid(P * Ch), 256, 0, stream>>>(x, g, Ch, P * Ch, gx);
  OG_RETURN_LAST_ERROR();
}

// ---------------------------------------------------------------------------------------------
// CA_NET reparametrisation (model.py:470-478):  c = eps * exp(0.5 * logvar) + mu
// x rows hold [mu (D) | logvar (D)] (row stride xs); eps, c are (B, D) dense.
// ---------------------------------------------------------------------------------------------
__global__ void reparam_fwd_kernel(const float* __restrict__ x, int xs, const float* __restrict__ eps, int D,
                                   long long total, float* __restrict__ c, int cs) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    long long b = i / D;
    int k = (int)(i - b * D);
    c[b * cs + k] = eps[i] * expf(0.5f * x[b * xs + D + k]) + x[b * xs + k];
  }
}
__global__ void reparam_bwd_kernel(const float* __restrict__ x, int xs, const float* __restrict__ eps,
                                   const float* __restrict__ gc, int gcs, int D, long long total,
                                   float* __restrict__ gx) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    long long b = i / D;
    int k = (int)(i - b * D);
    float g = gc[b * gcs + k];
    gx[b * xs + k] += g;
    gx[b * xs + D + k] += g * eps[i] * 0.5f * expf(0.5f * x[b * xs + D + k]);
  }
}
OG_API int og_reparam_fwd(const float* x, int xs, const float* eps, int B, int D, float* c, int cs,
                          cudaStream_t stream) {
  reparam_fwd_kernel<<<og_grid((long long)B * D), 256, 0, stream>>>(x, xs, eps, D, (long long)B * D, c, cs);
  OG_RETURN_LAST_ERROR();
}
// accumulates into gx (caller zero-fills or pre-loads it with the KL gradient)
OG_API int og_reparam_bwd(const float* x, int xs, const float* eps, const float* gc, int gcs, int B, int D, float* gx,
                          cudaStream_t stream) {
  reparam_bwd_kernel<<<og_grid((long long)B * D), 256, 0, stream>>>(x, xs, eps, gc, gcs, D, (long long)B * D, gx);
  OG_RETURN_LAST_ERROR();
}

// ---------------------------------------------------------------------------------------------
// losses.  Each kernel adds  weight * mean(loss)  into *loss_accum (device scalar) and writes the
// gradient of that weighted mean w.r.t. its input.  One block: the sum is taken in a fixed order (the inputs are
// logits of patch heads and CA_NET rows, a few thousand elements), so the value does not change from run to run.
// nn.BCELoss (miscc/losses.py:178-208, 378-393): log terms clamped at -100, backward
// (p - t) / max(p (1 - p), 1e-12) like PyTorch.
// ---------------------------------------------------------------------------------------------
__global__ void bce_kernel(const float* __restrict__ p, long long n, float target, float weight, float* loss_accum,
                           float* __restrict__ gp) {
  float local = 0.f;
  const float inv = 1.f / (float)n;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n;
       i += (long long)gridDim.x * blockDim.x) {
    float v = p[i];
    float l1 = fmaxf(logf(v), -100.f), l0 = fmaxf(logf(1.f - v), -100.f);
    local += -(target * l1 + (1.f - target) * l0);
    if (gp) gp[i] = weight * inv * (v - target) / fmaxf(v * (1.f - v), 1e-12f);
  }
  local = warp_sum(local);
  __shared__ float sh[8];
  if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = local;
  __syncthreads();
  if (threadIdx.x == 0) {
    float s = 0.f;
    for (int i = 0; i < (blockDim.x >> 5); ++i) s += sh[i];
    *loss_accum += weight * inv * s;
  }
}
OG_API int og_bce(const float* p, long long n, float target, float weight, float* loss_accum, float* gp,
                  cudaStream_t stream) {
  if (n == 0) return 0;
  bce_kernel<<<1, 256, 0, stream>>>(p, n, target, weight, loss_accum, gp);
  OG_RETURN_LAST_ERROR();
}

// KL_loss (miscc/losses.py:533-537): -0.5 * mean(1 + logvar - mu^2 - exp(logvar)); x rows = [mu | logvar]
__global__ void kl_kernel(const float* __restrict__ x, int xs, int B, int D, float weight, float* loss_accum,
                          float* __restrict__ gx) {
  float local = 0.f;
  const long long n = (long long)B * D;
  const float inv = 1.f / (float)n;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n;
       i += (long long)gridDim.x * blockDim.x) {
    long long b = i / D;
    int k = (int)(i - b * D);
    float mu = x[b * xs + k], lv = x[b * xs + D + k], e = expf(lv);
    local += 1.f + lv - mu * mu - e;
    if (gx) {
      gx[b * xs + k] = weight * inv * mu;
      gx[b * xs + D + k] = weight * inv * (-0.5f) * (1.f - e);
    }
  }
  local = warp_sum(local);
  __shared__ float sh[8];
  if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = local;
  __syncthreads();
  if (threadIdx.x == 0) {
    float s = 0.f;
    for (int i = 0; i < (blockDim.x >> 5); ++i) s += sh[i];
    *loss_accum += -0.5f * weight * inv * s;
  }
}
OG_API int og_kl(const float* x, int xs, int B, int D, float weight, float* loss_accum, float* gx,
                 cudaStream_t stream) {
  kl_kernel<<<1, 256, 0, stream>>>(x, xs, B, D, weight, loss_accum, gx);
  OG_RETURN_LAST_ERROR();
}

// ---------------------------------------------------------------------------------------------
// fused Adam (+ gradient pre-scale for data-parallel averaging, + EMA of the generator weights)
// torch.optim.Adam(lr, betas=(0.5, 0.999)) as used in trainer.py:197-224; EMA trainer.py:461-462.
// ---------------------------------------------------------------------------------------------
__global__ void adam_ema_kernel(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ m,
                                float* __restrict__ v, float* __restrict__ avg, long long n, float lr, float b1,
                                float b2, float eps, double b1d, double b2d, int step_host,
                                const long long* __restrict__ step_dev, float gscale, float decay) {
  // bias corrections in double, like torch.optim.Adam's python scalars; the step count comes from the host or,
  // when the step is replayed from a CUDA graph, from a device counter (og_inc_i64 bumps it before this launch)
  const double st = step_dev ? (double)(*step_dev) : (double)step_host;
  const float bc1 = (float)(1.0 - pow(b1d, st));
  const float sqrt_bc2 = (float)sqrt(1.0 - pow(b2d, st));
  const float step_size = lr / bc1;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n;
       i += (long long)gridDim.x * blockDim.x) {
    float gg = g[i] * gscale;
    float mm = m[i] * b1 + (1.f - b1) * gg;
    float vv = v[i] * b2 + (1.f - b2) * gg * gg;
    m[i] = mm;
    v[i] = vv;
    float denom = sqrtf(vv) / sqrt_bc2 + eps;
    float pp = p[i] - step_size * (mm / denom);
    p[i] = pp;
    if (avg) avg[i] = avg[i] * decay + (1.f - decay) * pp;
  }
}
OG_API int og_adam_ema(float* p, const float* g, float* m, float* v, float* avg, long long n, double lr, double b1,
                       double b2, double eps, int step, const long long* step_dev, float gscale, float decay,
                       cudaStream_t stream) {
  if (n == 0) return 0;
  adam_ema_kernel<<<og_grid(n), 256, 0, stream>>>(p, g, m, v, avg, n, (float)lr, (float)b1, (float)b2, (float)eps, b1, b2,
                                                   step, step_dev, gscale, decay);
  OG_RETURN_LAST_ERROR();
}

__global__ void inc_i64_kernel(long long* c) { *c += 1; }
OG_API int og_inc_i64(long long* counter, cudaStream_t stream) {
  inc_i64_kernel<<<1, 1, 0, stream>>>(counter);
  OG_RETURN_LAST_ERROR();
}

// ---------------------------------------------------------------------------------------------
// F.interpolate(mode='bilinear', align_corners=True) on NHWC tensors (OBJ_SS_D_NET / OBJ_LS_D_NET front end,
// ref: model.py:1217-1218, 1283-1284): src index = dst * (in-1)/(out-1), weights in fp32 like ATen.
// ---------------------------------------------------------------------------------------------
__global__ void bilinear_fwd_kernel(const float* __restrict__ x, int IH, int IW, int OH, int OW, int C4, float rh,
                                    float rw, long long total, float* __restrict__ y) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    int c = (int)(i % C4);
    long long t = i / C4;
    int ow = (int)(t % OW);
    t /= OW;
    int oh = (int)(t % OH);
    long long n = t / OH;
    float fh = rh * oh, fw = rw * ow;
    int h0 = (int)fh, w0 = (int)fw;
    int h1 = h0 + (h0 < IH - 1), w1 = w0 + (w0 < IW - 1);
    float lh = fh - h0, lw = fw - w0, hh = 1.f - lh, hw = 1.f - lw;
    const float* b = x + n * IH * IW * C4 * 4;
    float4 a = ldg4(b + ((long long)h0 * IW + w0) * C4 * 4 + c * 4), bq = ldg4(b + ((long long)h0 * IW + w1) * C4 * 4 + c * 4);
    float4 cq = ldg4(b + ((long long)h1 * IW + w0) * C4 * 4 + c * 4), d = ldg4(b + ((long long)h1 * IW + w1) * C4 * 4 + c * 4);
    float4 o;
    o.x = hh * (hw * a.x + lw * bq.x) + lh * (hw * cq.x + lw * d.x);
    o.y = hh * (hw * a.y + lw * bq.y) + lh * (hw * cq.y + lw * d.y);
    o.z = hh * (hw * a.z + lw * bq.z) + lh * (hw * cq.z + lw * d.z);
    o.w = hh * (hw * a.w + lw * bq.w) + lh * (hw * cq.w + lw * d.w);
    st4(y + i * 4, o);
  }
}
__global__ void bilinear_bwd_kernel(const float* __restrict__ g, int IH, int IW, int OH, int OW, int C, float rh,
                                    float rw, long long total, float* __restrict__ gx) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    int c = (int)(i % C);
    long long t = i / C;
    int ow = (int)(t % OW);
    t /= OW;
    int oh = (int)(t % OH);
    long long n = t / OH;
    float fh = rh * oh, fw = rw * ow;
    int h0 = (int)fh, w0 = (int)fw;
    int h1 = h0 + (h0 < IH - 1), w1 = w0 + (w0 < IW - 1);
    float lh = fh - h0, lw = fw - w0, hh = 1.f - lh, hw = 1.f - lw;
    float gv = g[i];
    float* b = gx + n * IH * IW * C + c;
    atomicAdd(b + ((long long)h0 * IW + w0) * C, gv * hh * hw);
    atomicAdd(b + ((long long)h0 * IW + w1) * C, gv * hh * lw);
    atomicAdd(b + ((long long)h1 * IW + w0) * C, gv * lh * hw);
    atomicAdd(b + ((long long)h1 * IW + w1) * C, gv * lh * lw);
  }
}
OG_API int og_bilinear_fwd(const float* x, int N, int IH, int IW, int C, int OH, int OW, float* y, cudaStream_t stream) {
  if (C % 4) return (int)cudaErrorInvalidValue;
  long long total = (long long)N * OH * OW * (C / 4);
  if (total == 0) return 0;
  float rh = OH > 1 ? (float)(IH - 1) / (float)(OH - 1) : 0.f, rw = OW > 1 ? (float)(IW - 1) / (float)(OW - 1) : 0.f;
  bilinear_fwd_kernel<<<og_grid(total), 256, 0, stream>>>(x, IH, IW, OH, OW, C / 4, rh, rw, total, y);
  OG_RETURN_LAST_ERROR();
}
// gx is zero-filled here
OG_API int og_bilinear_bwd(const float* g, int N, int IH, int IW, int C, int OH, int OW, float* gx, cudaStream_t stream) {
  OG_CHECK(cudaMemsetAsync(gx, 0, sizeof(float) * (size_t)N * IH * IW * C, stream));
  long long total = (long long)N * OH * OW * C;
  if (total == 0) return 0;
  float rh = OH > 1 ? (float)(IH - 1) / (float)(OH - 1) : 0.f, rw = OW > 1 ? (float)(IW - 1) / (float)(OW - 1) : 0.f;
  bilinear_bwd_kernel<<<og_grid(total), 256, 0, stream>>>(g, IH, IW, OH, OW, C, rh, rw, total, gx);
  OG_RETURN_LAST_ERROR();
}

// ---------------------------------------------------------------------------------------------------------------
// Device-side input preparation (the part of the reference's host data path that only re-arranges what the loader
// already produced; ref: trainDataset.py:79-128 prepare_data, miscc/load.py:160-176 get_hmaps_rois,
// miscc/utils.py:502-522 form_clabels_feat).  The 80-channel class heat maps are, by construction, the per-class sums
// of the 10 per-roi masks (load.py:176: hmaps[cat] += re_mask), so only the masks cross PCIe (7x fewer bytes) and the
// heat maps are rebuilt here, in roi order like the loader's loop.
// ---------------------------------------------------------------------------------------------------------------
// masks [B][R][P], cls [B][R] (int64 class index per roi slot), num_rois [B] (int64) -> out [B][ncls][P] (NCHW)
__global__ void __launch_bounds__(256) form_hmaps_kernel(const float* __restrict__ masks, const long long* __restrict__ cls,
                                                         const long long* __restrict__ num_rois, int R, long long P,
                                                         int ncls, float clamp_max, float* __restrict__ out) {
  const int b = blockIdx.y;
  const int n = min((int)num_rois[b], R);
  __shared__ int scls[64];
  for (int r = threadIdx.x; r < n && r < 64; r += blockDim.x) scls[r] = (int)cls[(long long)b * R + r];
  __syncthreads();
  for (long long p = blockIdx.x * (long long)blockDim.x + threadIdx.x; p < P; p += (long long)gridDim.x * blockDim.x) {
    float* o = out + (long long)b * ncls * P + p;
    for (int r = 0; r < n; ++r) {                       // sequential, in roi order: same sums as the host loop
      const int c = scls[r];
      if (c < 0 || c >= ncls) continue;
      float v = o[(long long)c * P] + masks[((long long)b * R + r) * P + p];
      o[(long long)c * P] = v;
    }
    if (clamp_max > 0.f)
      for (int r = 0; r < n; ++r) {
        const int c = scls[r];
        if (c < 0 || c >= ncls) continue;
        o[(long long)c * P] = fminf(o[(long long)c * P], clamp_max);
      }
  }
}
OG_API int og_form_hmaps(const float* masks, const long long* cls, const long long* num_rois, int B, int R, long long P,
                         int ncls, float clamp_max, float* out, cudaStream_t stream) {
  if (R > 64) return (int)cudaErrorInvalidValue;
  OG_CHECK(cudaMemsetAsync(out, 0, sizeof(float) * (size_t)B * ncls * P, stream));
  if (B == 0 || P == 0) return 0;
  dim3 grid(og_cdiv(P, 256) < og_num_sms() * 4 ? og_cdiv(P, 256) : og_num_sms() * 4, B);
  form_hmaps_kernel<<<grid, 256, 0, stream>>>(masks, cls, num_rois, R, P, ncls, clamp_max, out);
  OG_RETURN_LAST_ERROR();
}
// emb [ncls][E], cls [B][R], num_rois [B] -> out [B][E][Rmax] (= (B, E, Rmax, 1)); slots r >= num_rois[b] are zero
__global__ void form_clabels_feat_kernel(const float* __restrict__ emb, const long long* __restrict__ cls,
                                         const long long* __restrict__ num_rois, int R, int Rmax, int E, int ncls,
                                         long long total, float* __restrict__ out) {
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int r = (int)(i % Rmax);
  const int e = (int)((i / Rmax) % E);
  const int b = (int)(i / ((long long)Rmax * E));
  float v = 0.f;
  if (r < (int)num_rois[b] && r < R) {
    const int c = (int)cls[(long long)b * R + r];
    if (c >= 0 && c < ncls) v = emb[(long long)c * E + e];
  }
  out[i] = v;
}
OG_API int og_form_clabels_feat(const float* emb, const long long* cls, const long long* num_rois, int B, int R, int Rmax,
                                int E, int ncls, float* out, cudaStream_t stream) {
  const long long total = (long long)B * E * Rmax;
  if (total == 0) return 0;
  form_clabels_feat_kernel<<<og_cdiv(total, 256), 256, 0, stream>>>(emb, cls, num_rois, R, Rmax, E, ncls, total, out);
  OG_RETURN_LAST_ERROR();
}

// out[b][c][:] = x[b][perm[b][c]][:]  (NCHW planes of P floats): the per-sample class-channel shuffle of permute_seg
// (ref: miscc/utils.py:445-462) as ONE pass over the maps, with the permutation table built on the host
__global__ void __launch_bounds__(256) permute_channels_kernel(const float* __restrict__ x,
                                                               const long long* __restrict__ perm, int C, long long P,
                                                               float* __restrict__ out) {
  const int c = blockIdx.y, b = blockIdx.z;
  const long long src = perm[(long long)b * C + c];
  const float* xp = x + ((long long)b * C + src) * P;
  float* op = out + ((long long)b * C + c) * P;
  if ((P & 3) == 0) {
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < P / 4; i += (long long)gridDim.x * blockDim.x)
      st4(op + i * 4, ldg4(xp + i * 4));
  } else {
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < P; i += (long long)gridDim.x * blockDim.x)
      op[i] = xp[i];
  }
}
OG_API int og_permute_channels(const float* x, const long long* perm, int B, int C, long long P, float* out,
                               cudaStream_t stream) {
  if (B == 0 || C == 0 || P == 0) return 0;
  int bx = og_cdiv(P / 4 > 0 ? P / 4 : P, 256);
  if (bx > 64) bx = 64;
  permute_channels_kernel<<<dim3(bx, C, B), 256, 0, stream>>>(x, perm, C, P, out);
  OG_RETURN_LAST_ERROR();
}

// NCHW (N, 3, H, W) fp32 images in [-1, 1] -> NHWC (N, H, W, 3) uint8, the arithmetic of the reference's
// save_singleimages (ref: evaluator.py:235-237): x.add(1).div(2).mul(255).clamp(0, 255).byte(), then permute(1, 2, 0).
// Each step is rounded on its own (__fadd_rn / __fmul_rn: no contraction into an FMA may move a value across a byte
// boundary); the halving is exact.  The clamp then the truncation toward zero of .byte(); fmaxf maps NaN to 0.
__global__ void __launch_bounds__(256) images_to_u8_kernel(const float* __restrict__ x, long long HW, long long total,
                                                           unsigned char* __restrict__ out) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const long long n = i / HW, p = i - n * HW;
    const float* xp = x + n * 3 * HW + p;
    unsigned char* op = out + i * 3;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      float v = __fmul_rn(__fmul_rn(__fadd_rn(__ldg(xp + c * HW), 1.f), 0.5f), 255.f);
      v = fminf(fmaxf(v, 0.f), 255.f);
      op[c] = (unsigned char)__float2uint_rz(v);
    }
  }
}
OG_API int og_images_to_u8(const float* x, int N, int H, int W, unsigned char* out, cudaStream_t stream) {
  const long long total = (long long)N * H * W;
  if (total == 0) return 0;
  images_to_u8_kernel<<<og_grid(total), 256, 0, stream>>>(x, (long long)H * W, total, out);
  OG_RETURN_LAST_ERROR();
}
