// InstanceNorm2d / BatchNorm{1,2}d (train and eval mode) with fused activation, forward and backward, NHWC.
//
// Reference semantics (image_generation/model.py): nn.InstanceNorm2d defaults (no affine, eps 1e-5, biased
// variance; model.py:70, 602, 1198) and nn.BatchNorm2d/1d in train mode (batch statistics, biased variance
// for normalisation, running stats with momentum 0.1 and the unbiased variance; model.py:47, 497, 992,
// 1011).  The activation that always follows is fused into the apply pass: GLU (model.py:19-27),
// LeakyReLU(0.2) or nothing (+ optional residual add, model.py:76-81).
//
// All kernels are HBM-bandwidth bound: one read of the conv output for the statistics, one read + one
// write for the apply.  Statistics are accumulated in fp64 (sum, sum of squares) so that the one-pass
// variance does not lose digits; the finalised mean / rstd are fp32.
//
// Layout: contiguous NHWC, rows = pixels, C % 4 == 0.  "groups" = N for instance norm, 1 for batch norm;
// each group covers P pixels (H*W, resp. N*H*W).
#include "common.cuh"
#include <cuda_fp16.h>

// grid: (ceil(C4/32), chunks, groups)   block: (32, 8)
// A thread owns one channel quad and walks the rows p0 + ty, p0 + ty + 8, ...: four rows are loaded back to back (four
// 16-byte loads in flight), summed pairwise in fp32 (<= 2 roundings: ~1e-7 relative, random) and only the 4-row partial
// enters the fp64 accumulators -- a quarter of the F2F / DADD / DFMA issue slots of per-element fp64.
__global__ void __launch_bounds__(256) norm_stats_kernel(const float* __restrict__ x, int C, long long P,
                                                         int pix_per_block, double* __restrict__ stats) {
  const int c4 = blockIdx.x * 32 + threadIdx.x;
  const int C4 = C >> 2;
  const long long g = blockIdx.z;
  const long long p0 = (long long)blockIdx.y * pix_per_block;
  const long long p1 = min(P, p0 + pix_per_block);
  double s[4] = {0, 0, 0, 0}, q[4] = {0, 0, 0, 0};
  if (c4 < C4) {
    const float* base = x + (g * P) * C + c4 * 4;
    long long p = p0 + threadIdx.y;
    for (; p + 24 < p1; p += 32) {
      const float4 a = ldg4(base + p * C), b = ldg4(base + (p + 8) * C);
      const float4 c = ldg4(base + (p + 16) * C), d = ldg4(base + (p + 24) * C);
      s[0] += (double)((a.x + b.x) + (c.x + d.x)); q[0] += (double)((a.x * a.x + b.x * b.x) + (c.x * c.x + d.x * d.x));
      s[1] += (double)((a.y + b.y) + (c.y + d.y)); q[1] += (double)((a.y * a.y + b.y * b.y) + (c.y * c.y + d.y * d.y));
      s[2] += (double)((a.z + b.z) + (c.z + d.z)); q[2] += (double)((a.z * a.z + b.z * b.z) + (c.z * c.z + d.z * d.z));
      s[3] += (double)((a.w + b.w) + (c.w + d.w)); q[3] += (double)((a.w * a.w + b.w * b.w) + (c.w * c.w + d.w * d.w));
    }
    for (; p < p1; p += 8) {
      float4 v = ldg4(base + p * C);
      s[0] += v.x; q[0] += (double)v.x * v.x;
      s[1] += v.y; q[1] += (double)v.y * v.y;
      s[2] += v.z; q[2] += (double)v.z * v.z;
      s[3] += v.w; q[3] += (double)v.w * v.w;
    }
  }
  __shared__ double sh[8][32][8];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    sh[threadIdx.y][threadIdx.x][i] = s[i];
    sh[threadIdx.y][threadIdx.x][4 + i] = q[i];
  }
  __syncthreads();
  // 256 threads reduce 32 x 8 values over the 8 pixel lanes
  const int t = threadIdx.y * 32 + threadIdx.x;
  const int cx = t >> 3, k = t & 7;
  double acc = 0;
#pragma unroll
  for (int j = 0; j < 8; ++j) acc += sh[j][cx][k];
  const int cc4 = blockIdx.x * 32 + cx;
  if (cc4 < C4) {
    int ch = cc4 * 4 + (k & 3);
    atomicAdd(&stats[(g * C + ch) * 2 + (k >> 2)], acc);
  }
}

// mean / rstd from (sum, sumsq); optional BatchNorm running-stat update.
__global__ void norm_finalize_kernel(const double* __restrict__ stats, int groups, int C, double count, float eps,
                                     float* __restrict__ mean, float* __restrict__ rstd, float* running_mean,
                                     float* running_var, float momentum, int real_c,
                                     long long* num_batches_tracked) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= groups * C) return;
  if (i == 0 && num_batches_tracked) *num_batches_tracked += 1;
  double m = stats[i * 2] / count;
  double var = stats[i * 2 + 1] / count - m * m;
  if (var < 0) var = 0;
  mean[i] = (float)m;
  rstd[i] = (float)(1.0 / sqrt(var + (double)eps));
  if (running_mean && groups == 1 && i < real_c) {
    double unbiased = count > 1 ? var * count / (count - 1.0) : var;
    running_mean[i] = (1.f - momentum) * running_mean[i] + momentum * (float)m;
    running_var[i] = (1.f - momentum) * running_var[i] + momentum * (float)unbiased;
  }
}

// forward apply.  y: conv output [G*P][Cy];  out: [G*P][Co] where Co = Cy (none / lrelu) or Cy/2 (GLU).
// gamma/beta (BatchNorm affine) may be null (InstanceNorm).  res (same shape as out) is added when non-null.
// max|.| of the values a 256-thread block has written, merged into *amax (float bits; non-negative floats order like
// unsigned integers).  The consumer convolution scales its fp16 operand copies by it (og_prep_split).
__device__ __forceinline__ float amax4(float m, const float4& o) {
  return fmaxf(fmaxf(m, fmaxf(fabsf(o.x), fabsf(o.y))), fmaxf(fabsf(o.z), fabsf(o.w)));
}
__device__ __forceinline__ void block_amax_256(float m, unsigned* amax) {
  __shared__ float sm_amax[8];
  const int tid = threadIdx.y * blockDim.x + threadIdx.x;       // 256 threads as (256) or (32, 8)
  m = warp_max(m);
  if ((tid & 31) == 0) sm_amax[tid >> 5] = m;
  __syncthreads();
  if (tid < 8) {
    m = sm_amax[tid];
#pragma unroll
    for (int o = 4; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffu, m, o));
    if (tid == 0) atomicMax(amax, __float_as_uint(m));
  }
}

// sigmoid on the SFU: ex2.approx + rcp.approx (~2 ulp; the libm expf + IEEE division it replaces made the GLU passes
// issue bound at half of the HBM bandwidth).  exp(-x) overflowing to +inf gives exactly 0.
__device__ __forceinline__ float sigmoid_fast(float x) { return __fdividef(1.0f, 1.0f + __expf(-x)); }

// Flat grid-stride walk over (pixel, channel quad): every lane of every warp carries a 16-byte load, which measured
// 0.92 of the copy bandwidth for the plain / LeakyReLU / residual forms (the channel-fixed mapping of the backward
// kernels below, with its idle lanes when C/4 is not a multiple of 32, measured 0.74 here).  The (pixel, quad, group)
// indices advance incrementally: no division per element.
template <int ACT>
__global__ void __launch_bounds__(256) norm_apply_kernel(const float* __restrict__ y, int Cy, long long P,
                                                         long long total_pix, const float* __restrict__ mean,
                                                         const float* __restrict__ rstd,
                                                         const float* __restrict__ gamma,
                                                         const float* __restrict__ beta,
                                                         const float* __restrict__ res, float slope,
                                                         float* __restrict__ out, unsigned* __restrict__ amax) {
  const int Co = (ACT == OG_NA_GLU) ? Cy / 2 : Cy;
  const int Co4 = Co >> 2;
  const long long total = total_pix * Co4;
  float mx = 0.f;
  // (pixel p, channel quad c4, group g, pixel-in-group pg) advance incrementally: no division per element
  const long long stride = (long long)gridDim.x * blockDim.x;
  const long long dp = stride / Co4;
  const int dc = (int)(stride - dp * Co4);
  long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  long long p = i / Co4;
  int c4i = (int)(i - p * Co4);
  long long g = p / P, pg = p - g * P;
  for (; i < total; i += stride, p += dp, pg += dp, c4i += dc) {
    if (c4i >= Co4) { c4i -= Co4; ++p; ++pg; }
    while (pg >= P) { pg -= P; ++g; }
    const int c = c4i * 4;
    const float* mrow = mean + g * Cy;
    const float* rrow = rstd + g * Cy;
    float4 v = ldg4(y + p * Cy + c);
    float4 m = ldg4(mrow + c), r = ldg4(rrow + c);
    float4 ga = gamma ? ldg4(gamma + c) : make_float4(1.f, 1.f, 1.f, 1.f);
    float4 be = beta ? ldg4(beta + c) : make_float4(0.f, 0.f, 0.f, 0.f);
    float4 a;
    a.x = (v.x - m.x) * r.x * ga.x + be.x;
    a.y = (v.y - m.y) * r.y * ga.y + be.y;
    a.z = (v.z - m.z) * r.z * ga.z + be.z;
    a.w = (v.w - m.w) * r.w * ga.w + be.w;
    float4 o;
    if (ACT == OG_NA_GLU) {
      float4 v2 = ldg4(y + p * Cy + Co + c);
      float4 m2 = ldg4(mrow + Co + c), r2 = ldg4(rrow + Co + c);
      float4 ga2 = gamma ? ldg4(gamma + Co + c) : make_float4(1.f, 1.f, 1.f, 1.f);
      float4 be2 = beta ? ldg4(beta + Co + c) : make_float4(0.f, 0.f, 0.f, 0.f);
      o.x = a.x * sigmoid_fast((v2.x - m2.x) * r2.x * ga2.x + be2.x);
      o.y = a.y * sigmoid_fast((v2.y - m2.y) * r2.y * ga2.y + be2.y);
      o.z = a.z * sigmoid_fast((v2.z - m2.z) * r2.z * ga2.z + be2.z);
      o.w = a.w * sigmoid_fast((v2.w - m2.w) * r2.w * ga2.w + be2.w);
    } else if (ACT == OG_NA_LRELU) {
      o.x = a.x > 0.f ? a.x : a.x * slope;
      o.y = a.y > 0.f ? a.y : a.y * slope;
      o.z = a.z > 0.f ? a.z : a.z * slope;
      o.w = a.w > 0.f ? a.w : a.w * slope;
    } else {
      o = a;
    }
    if (res) {
      float4 rr = ldg4(res + p * Co + c);
      o.x += rr.x; o.y += rr.y; o.z += rr.z; o.w += rr.w;
    }
    st4(out + p * Co + c, o);
    mx = amax4(mx, o);
  }
  if (amax) block_amax_256(mx, amax);
}

// Per-thread constants of the backward passes: statistics and affine parameters of the thread's channel quad (and of
// the gate quad Co channels further for GLU), loaded once.
struct ChanConst {
  float4 m, r, ga, be, m2, r2, ga2, be2;
};
template <int ACT>
__device__ __forceinline__ void load_chan(ChanConst& k, const float* __restrict__ mean, const float* __restrict__ rstd,
                                          const float* __restrict__ gamma, const float* __restrict__ beta,
                                          long long grp, int Cy, int Co, int c) {
  const float4 one = make_float4(1.f, 1.f, 1.f, 1.f), zero = make_float4(0.f, 0.f, 0.f, 0.f);
  k.m = ldg4(mean + grp * Cy + c); k.r = ldg4(rstd + grp * Cy + c);
  k.ga = gamma ? ldg4(gamma + c) : one; k.be = beta ? ldg4(beta + c) : zero;
  k.m2 = zero; k.r2 = one; k.ga2 = one; k.be2 = zero;
  if (ACT == OG_NA_GLU) {
    k.m2 = ldg4(mean + grp * Cy + Co + c); k.r2 = ldg4(rstd + grp * Cy + Co + c);
    if (gamma) k.ga2 = ldg4(gamma + Co + c);
    if (beta) k.be2 = ldg4(beta + Co + c);
  }
}

// gradient of the fused activation w.r.t. the normalised (+affine) values n, for 4 channels: v / v2 = the conv outputs
// of the "a" and gate quads, go = the incoming gradient.  Returns xhat and dn for the "a" half (and the gate half's).
template <int ACT>
__device__ __forceinline__ void act_grad4(const ChanConst& k, const float4& v, const float4& v2, const float4& go,
                                          float slope, float4& xh, float4& dn, float4& xh2, float4& dn2) {
  xh.x = (v.x - k.m.x) * k.r.x; xh.y = (v.y - k.m.y) * k.r.y; xh.z = (v.z - k.m.z) * k.r.z; xh.w = (v.w - k.m.w) * k.r.w;
  float4 n;
  n.x = xh.x * k.ga.x + k.be.x; n.y = xh.y * k.ga.y + k.be.y; n.z = xh.z * k.ga.z + k.be.z; n.w = xh.w * k.ga.w + k.be.w;
  if (ACT == OG_NA_GLU) {
    xh2.x = (v2.x - k.m2.x) * k.r2.x; xh2.y = (v2.y - k.m2.y) * k.r2.y;
    xh2.z = (v2.z - k.m2.z) * k.r2.z; xh2.w = (v2.w - k.m2.w) * k.r2.w;
    const float sx = sigmoid_fast(xh2.x * k.ga2.x + k.be2.x), sy = sigmoid_fast(xh2.y * k.ga2.y + k.be2.y);
    const float sz = sigmoid_fast(xh2.z * k.ga2.z + k.be2.z), sw = sigmoid_fast(xh2.w * k.ga2.w + k.be2.w);
    dn.x = go.x * sx; dn.y = go.y * sy; dn.z = go.z * sz; dn.w = go.w * sw;
    dn2.x = go.x * n.x * sx * (1.f - sx); dn2.y = go.y * n.y * sy * (1.f - sy);
    dn2.z = go.z * n.z * sz * (1.f - sz); dn2.w = go.w * n.w * sw * (1.f - sw);
  } else if (ACT == OG_NA_LRELU) {
    dn.x = n.x > 0.f ? go.x : go.x * slope; dn.y = n.y > 0.f ? go.y : go.y * slope;
    dn.z = n.z > 0.f ? go.z : go.z * slope; dn.w = n.w > 0.f ? go.w : go.w * slope;
  } else {
    dn = go;
  }
}

// backward reduce: per (group, channel of y):  bstats[.,0] = sum dn,  bstats[.,1] = sum dn * xhat   (fp64)
// grid: (ceil(Co4/32), chunks, groups)  block (32, 8).  Two rows per trip: their contributions are added in fp32 and the
// pair enters the fp64 accumulators (half of the fp64 issue slots; the pair sum costs one fp32 rounding).
template <int ACT>
__global__ void __launch_bounds__(256) norm_bwd_reduce_kernel(const float* __restrict__ y,
                                                              const float* __restrict__ g, int Cy, long long P,
                                                              int pix_per_block, const float* __restrict__ mean,
                                                              const float* __restrict__ rstd,
                                                              const float* __restrict__ gamma,
                                                              const float* __restrict__ beta, float slope,
                                                              double* __restrict__ bstats) {
  const int Co = (ACT == OG_NA_GLU) ? Cy / 2 : Cy;
  const int Co4 = Co >> 2;
  const int c4 = blockIdx.x * 32 + threadIdx.x;
  const long long grp = blockIdx.z;
  const long long p0 = (long long)blockIdx.y * pix_per_block;
  const long long p1 = min(P, p0 + pix_per_block);
  constexpr int NV = (ACT == OG_NA_GLU) ? 16 : 8;
  double acc[NV];
#pragma unroll
  for (int i = 0; i < NV; ++i) acc[i] = 0;
  if (c4 < Co4) {
    const int c = c4 * 4;
    ChanConst k;
    load_chan<ACT>(k, mean, rstd, gamma, beta, grp, Cy, Co, c);
    const float* yb = y + (grp * P) * Cy + c;
    const float* gb = g + (grp * P) * Co + c;
    const float4 zero = make_float4(0.f, 0.f, 0.f, 0.f);
    long long p = p0 + threadIdx.y;
    for (; p + 8 < p1; p += 16) {
      const float4 va = ldg4(yb + p * Cy), vb = ldg4(yb + (p + 8) * Cy);
      const float4 ga_ = ldg4(gb + p * Co), gb_ = ldg4(gb + (p + 8) * Co);
      float4 v2a = zero, v2b = zero;
      if (ACT == OG_NA_GLU) { v2a = ldg4(yb + p * Cy + Co); v2b = ldg4(yb + (p + 8) * Cy + Co); }
      float4 xa, da, x2a, d2a, xb, db, x2b, d2b;
      act_grad4<ACT>(k, va, v2a, ga_, slope, xa, da, x2a, d2a);
      act_grad4<ACT>(k, vb, v2b, gb_, slope, xb, db, x2b, d2b);
      acc[0] += (double)(da.x + db.x); acc[1] += (double)(da.y + db.y);
      acc[2] += (double)(da.z + db.z); acc[3] += (double)(da.w + db.w);
      acc[4] += (double)(da.x * xa.x + db.x * xb.x); acc[5] += (double)(da.y * xa.y + db.y * xb.y);
      acc[6] += (double)(da.z * xa.z + db.z * xb.z); acc[7] += (double)(da.w * xa.w + db.w * xb.w);
      if (ACT == OG_NA_GLU) {
        acc[NV - 8] += (double)(d2a.x + d2b.x); acc[NV - 7] += (double)(d2a.y + d2b.y);
        acc[NV - 6] += (double)(d2a.z + d2b.z); acc[NV - 5] += (double)(d2a.w + d2b.w);
        acc[NV - 4] += (double)(d2a.x * x2a.x + d2b.x * x2b.x); acc[NV - 3] += (double)(d2a.y * x2a.y + d2b.y * x2b.y);
        acc[NV - 2] += (double)(d2a.z * x2a.z + d2b.z * x2b.z); acc[NV - 1] += (double)(d2a.w * x2a.w + d2b.w * x2b.w);
      }
    }
    for (; p < p1; p += 8) {
      const float4 v = ldg4(yb + p * Cy), go = ldg4(gb + p * Co);
      const float4 v2 = (ACT == OG_NA_GLU) ? ldg4(yb + p * Cy + Co) : zero;
      float4 xh, dn, xh2, dn2;
      act_grad4<ACT>(k, v, v2, go, slope, xh, dn, xh2, dn2);
      acc[0] += dn.x; acc[1] += dn.y; acc[2] += dn.z; acc[3] += dn.w;
      acc[4] += (double)dn.x * xh.x; acc[5] += (double)dn.y * xh.y;
      acc[6] += (double)dn.z * xh.z; acc[7] += (double)dn.w * xh.w;
      if (ACT == OG_NA_GLU) {
        acc[NV - 8] += dn2.x; acc[NV - 7] += dn2.y; acc[NV - 6] += dn2.z; acc[NV - 5] += dn2.w;
        acc[NV - 4] += (double)dn2.x * xh2.x; acc[NV - 3] += (double)dn2.y * xh2.y;
        acc[NV - 2] += (double)dn2.z * xh2.z; acc[NV - 1] += (double)dn2.w * xh2.w;
      }
    }
  }
  __shared__ double sh[8][32][NV];
#pragma unroll
  for (int i = 0; i < NV; ++i) sh[threadIdx.y][threadIdx.x][i] = acc[i];
  __syncthreads();
  const int t = threadIdx.y * 32 + threadIdx.x;
  for (int item = t; item < 32 * NV; item += 256) {
    int cx = item / NV, k = item % NV;
    double a = 0;
#pragma unroll
    for (int j = 0; j < 8; ++j) a += sh[j][cx][k];
    int cc4 = blockIdx.x * 32 + cx;
    if (cc4 < Co4) {
      int half = k >> 3;            // 0: "a" half, 1: gate half (GLU only)
      int kk = k & 7;
      int ch = half * Co + cc4 * 4 + (kk & 3);
      atomicAdd(&bstats[(grp * Cy + ch) * 2 + (kk >> 2)], a);
    }
  }
}

// backward apply: dy = rstd * gamma * (dn - S1/cnt - xhat * S2/cnt).  Same thread mapping as the forward apply: the
// channel quad's statistics, affine parameters and the two reduction coefficients per channel stay in registers.
template <int ACT>
__global__ void __launch_bounds__(256) norm_bwd_apply_kernel(const float* __restrict__ y,
                                                             const float* __restrict__ g, int Cy, long long P,
                                                             int pix_per_block, const float* __restrict__ mean,
                                                             const float* __restrict__ rstd,
                                                             const float* __restrict__ gamma,
                                                             const float* __restrict__ beta, float slope,
                                                             const double* __restrict__ bstats,
                                                             float* __restrict__ dy, unsigned* __restrict__ amax) {
  const int Co = (ACT == OG_NA_GLU) ? Cy / 2 : Cy;
  const int Co4 = Co >> 2;
  const int c4 = blockIdx.x * 32 + threadIdx.x;
  const long long grp = blockIdx.z;
  const long long p0 = (long long)blockIdx.y * pix_per_block;
  const long long p1 = min(P, p0 + pix_per_block);
  float mx = 0.f;
  if (c4 < Co4) {
    const int c = c4 * 4;
    ChanConst k;
    load_chan<ACT>(k, mean, rstd, gamma, beta, grp, Cy, Co, c);
    // coef[(grp * Cy + ch) * 4 + {0, 1}] = (float)(S1 / count), (float)(S2 / count): written over the fp64 sums by
    // norm_bwd_coef_kernel (same float values the per-element double products gave)
    const float* coef = reinterpret_cast<const float*>(bstats);
    const float* bs = coef + (grp * Cy + c) * 4;
    const float2 k0 = *reinterpret_cast<const float2*>(bs), k1 = *reinterpret_cast<const float2*>(bs + 4);
    const float2 k2 = *reinterpret_cast<const float2*>(bs + 8), k3 = *reinterpret_cast<const float2*>(bs + 12);
    float2 j0 = make_float2(0.f, 0.f), j1 = j0, j2 = j0, j3 = j0;
    if (ACT == OG_NA_GLU) {
      const float* bs2 = coef + (grp * Cy + Co + c) * 4;
      j0 = *reinterpret_cast<const float2*>(bs2); j1 = *reinterpret_cast<const float2*>(bs2 + 4);
      j2 = *reinterpret_cast<const float2*>(bs2 + 8); j3 = *reinterpret_cast<const float2*>(bs2 + 12);
    }
    const float* yb = y + (grp * P) * Cy + c;
    const float* gb = g + (grp * P) * Co + c;
    float* db = dy + (grp * P) * Cy + c;
    const float4 zero = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll(ACT == OG_NA_GLU ? 2 : 4)
    for (long long p = p0 + threadIdx.y; p < p1; p += 8) {
      const float4 v = ldg4(yb + p * Cy), go = ldg4(gb + p * Co);
      const float4 v2 = (ACT == OG_NA_GLU) ? ldg4(yb + p * Cy + Co) : zero;
      float4 xh, dn, xh2, dn2;
      act_grad4<ACT>(k, v, v2, go, slope, xh, dn, xh2, dn2);
      float4 o;
      o.x = k.r.x * k.ga.x * (dn.x - k0.x - xh.x * k0.y);
      o.y = k.r.y * k.ga.y * (dn.y - k1.x - xh.y * k1.y);
      o.z = k.r.z * k.ga.z * (dn.z - k2.x - xh.z * k2.y);
      o.w = k.r.w * k.ga.w * (dn.w - k3.x - xh.w * k3.y);
      st4(db + p * Cy, o);
      mx = amax4(mx, o);
      if (ACT == OG_NA_GLU) {
        float4 o2;
        o2.x = k.r2.x * k.ga2.x * (dn2.x - j0.x - xh2.x * j0.y);
        o2.y = k.r2.y * k.ga2.y * (dn2.y - j1.x - xh2.y * j1.y);
        o2.z = k.r2.z * k.ga2.z * (dn2.z - j2.x - xh2.z * j2.y);
        o2.w = k.r2.w * k.ga2.w * (dn2.w - j3.x - xh2.w * j3.y);
        st4(db + p * Cy + Co, o2);
        mx = amax4(mx, o2);
      }
    }
  }
  if (amax) block_amax_256(mx, amax);
}

// (S1, S2) fp64 -> ((float)(S1 / count), (float)(S2 / count)) stored over the first 8 bytes of the same 16-byte slot
__global__ void norm_bwd_coef_kernel(double* __restrict__ bstats, long long n, double inv_count) {
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i >= n) return;
  const double s1 = bstats[i * 2], s2 = bstats[i * 2 + 1];
  float2 k = make_float2((float)(s1 * inv_count), (float)(s2 * inv_count));
  *reinterpret_cast<float2*>(bstats + i * 2) = k;
}

// dgamma = S2, dbeta = S1 for batch norm (groups == 1): copy fp64 sums to fp32 parameter-gradient vectors
__global__ void norm_param_grad_kernel(const double* __restrict__ bstats, int C, float* dgamma, float* dbeta,
                                       int accumulate) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= C) return;
  float db = (float)bstats[i * 2], dg = (float)bstats[i * 2 + 1];
  dgamma[i] = accumulate ? dgamma[i] + dg : dg;
  dbeta[i] = accumulate ? dbeta[i] + db : db;
}

// ------------------------------------------------------------------------------------------------
// Forward apply that ALSO emits the tensor-core operand copies of its output (what og_prep_split would make of it):
// fp16 hi / lo of out * 2^k, optionally with the ReflectionPad2d(1) halo of the consuming convolution.  The scale has to
// be known before the pass, so it comes from an a-priori bound of max|out| (og_norm_bound): a normalised value is at
// most sqrt(P - 1) in magnitude (biased variance over P values), so |out| <= max|gamma| sqrt(P) + max|beta| (+ the
// bound of the residual) whatever the data -- any upper bound is a valid operand scale, it only positions the 22-bit
// window (an element 2^-18 below the BOUND keeps all 22 bits; typical activations sit 2^-7 .. 2^-10 below it).
// The walk is over the DESTINATION grid [N][H + 2 pad][W + 2 pad][C / 8] (a halo position recomputes its source
// pixel: ~3 % more reads at 128^2); the fp32 output, when asked for, is written from the interior positions.
// ------------------------------------------------------------------------------------------------
__global__ void norm_bound_kernel(const float* __restrict__ gamma, const float* __restrict__ beta, int C, double count,
                                  const unsigned* __restrict__ res_word, unsigned* __restrict__ out_word) {
  float mg = gamma ? 0.f : 1.f, mb = 0.f;
  for (int i = threadIdx.x; i < C; i += blockDim.x) {
    if (gamma) mg = fmaxf(mg, fabsf(gamma[i]));
    if (beta) mb = fmaxf(mb, fabsf(beta[i]));
  }
  __shared__ float sg[8], sb[8];
  mg = warp_max(mg);
  mb = warp_max(mb);
  if ((threadIdx.x & 31) == 0) { sg[threadIdx.x >> 5] = mg; sb[threadIdx.x >> 5] = mb; }
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int i = 1; i < 8; ++i) { mg = fmaxf(mg, sg[i]); mb = fmaxf(mb, sb[i]); }
    float bound = mg * (float)(sqrt(count) * 1.001) + mb;
    if (res_word) bound += __uint_as_float(*res_word & 0x7fffffffu);
    *out_word = __float_as_uint(bound);
  }
}

template <int ACT>
__global__ void __launch_bounds__(256) norm_apply_split_kernel(
    const float* __restrict__ y, int N, int H, int W, int Cy, int instance, const float* __restrict__ mean,
    const float* __restrict__ rstd, const float* __restrict__ gamma, const float* __restrict__ beta,
    const float* __restrict__ res, float slope, float* __restrict__ out, const unsigned* __restrict__ bound_word,
    int pad, long long total, __half* __restrict__ xh, __half* __restrict__ xl) {
  const int Co = (ACT == OG_NA_GLU) ? Cy / 2 : Cy;
  const int C8 = Co >> 3;
  const int Hp = H + 2 * pad, Wp = W + 2 * pad;
  const float scale = og_exp2i(og_scale_exp(__ldg(bound_word)));
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(i % C8) * 8;
    long long t = i / C8;
    const int w = (int)(t % Wp);
    t /= Wp;
    const int h = (int)(t % Hp);
    const long long n = t / Hp;
    int sh = h - pad, sw = w - pad;
    const bool interior = sh >= 0 && sh < H && sw >= 0 && sw < W;
    if (sh < 0) sh = -sh;
    if (sh >= H) sh = 2 * H - 2 - sh;
    if (sw < 0) sw = -sw;
    if (sw >= W) sw = 2 * W - 2 - sw;
    const long long p = (n * H + sh) * W + sw;
    const long long g = instance ? n : 0;
    const float* yp = y + p * Cy + c;
    const float* mrow = mean + g * Cy + c;
    const float* rrow = rstd + g * Cy + c;
    float o[8];
#pragma unroll
    for (int q = 0; q < 2; ++q) {
      const float4 v = ldg4(yp + 4 * q), m = ldg4(mrow + 4 * q), r = ldg4(rrow + 4 * q);
      const float4 ga = gamma ? ldg4(gamma + c + 4 * q) : make_float4(1.f, 1.f, 1.f, 1.f);
      const float4 be = beta ? ldg4(beta + c + 4 * q) : make_float4(0.f, 0.f, 0.f, 0.f);
      float a[4] = {(v.x - m.x) * r.x * ga.x + be.x, (v.y - m.y) * r.y * ga.y + be.y,
                    (v.z - m.z) * r.z * ga.z + be.z, (v.w - m.w) * r.w * ga.w + be.w};
      if (ACT == OG_NA_GLU) {
        const float4 v2 = ldg4(yp + Co + 4 * q), m2 = ldg4(mrow + Co + 4 * q), r2 = ldg4(rrow + Co + 4 * q);
        const float4 ga2 = gamma ? ldg4(gamma + Co + c + 4 * q) : make_float4(1.f, 1.f, 1.f, 1.f);
        const float4 be2 = beta ? ldg4(beta + Co + c + 4 * q) : make_float4(0.f, 0.f, 0.f, 0.f);
        a[0] *= sigmoid_fast((v2.x - m2.x) * r2.x * ga2.x + be2.x);
        a[1] *= sigmoid_fast((v2.y - m2.y) * r2.y * ga2.y + be2.y);
        a[2] *= sigmoid_fast((v2.z - m2.z) * r2.z * ga2.z + be2.z);
        a[3] *= sigmoid_fast((v2.w - m2.w) * r2.w * ga2.w + be2.w);
      } else if (ACT == OG_NA_LRELU) {
#pragma unroll
        for (int j = 0; j < 4; ++j) a[j] = a[j] > 0.f ? a[j] : a[j] * slope;
      }
      if (res) {
        const float4 rr = ldg4(res + p * Co + c + 4 * q);
        a[0] += rr.x; a[1] += rr.y; a[2] += rr.z; a[3] += rr.w;
      }
#pragma unroll
      for (int j = 0; j < 4; ++j) o[4 * q + j] = a[j];
    }
    if (out && interior) {
      st4(out + p * Co + c, make_float4(o[0], o[1], o[2], o[3]));
      st4(out + p * Co + c + 4, make_float4(o[4], o[5], o[6], o[7]));
    }
    __align__(16) __half hi[8], lo[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const float v = o[j] * scale;
      hi[j] = __float2half_rn(v);
      lo[j] = __float2half_rn(v - __half2float(hi[j]));
    }
    *reinterpret_cast<uint4*>(xh + i * 8) = *reinterpret_cast<const uint4*>(hi);
    if (xl) *reinterpret_cast<uint4*>(xl + i * 8) = *reinterpret_cast<const uint4*>(lo);
  }
}

// ------------------------------------------------------------------------------------------------
// BatchNorm in eval mode (ref: nn.BatchNorm{1,2}d after .eval(), evaluator.py:110): the running statistics replace the
// batch statistics, so the normalisation is a fixed per-channel affine map.  The forward pass is og_bn_eval_coef
// (mean / rstd in the form og_norm_apply takes) followed by og_norm_apply with groups = 1.
// ------------------------------------------------------------------------------------------------
__global__ void bn_eval_coef_kernel(const float* __restrict__ running_mean, const float* __restrict__ running_var,
                                    int C, float eps, float* __restrict__ mean, float* __restrict__ rstd) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= C) return;
  mean[i] = running_mean[i];
  rstd[i] = (float)(1.0 / sqrt((double)running_var[i] + (double)eps));
}

// Backward of the fixed affine + activation: dy = dn * gamma * rstd, with no batch-statistic terms.  Same thread mapping
// as norm_bwd_apply_kernel (grid (ceil(Co4/32), chunks), block (32, 8)).  When part is non-null, the CTA's per-channel
// sums (sum dn, sum dn * xhat) are reduced inside the CTA in a fixed order (fp64) and stored to plane blockIdx.y of
// part ([chunks][2][Cy] doubles); bn_eval_param_grad_kernel adds the planes in a fixed order -- no atomics, so the
// parameter gradients are the same on every run.
template <int ACT>
__global__ void __launch_bounds__(256) bn_eval_bwd_kernel(const float* __restrict__ y, const float* __restrict__ g,
                                                          int Cy, long long P, int pix_per_block,
                                                          const float* __restrict__ mean,
                                                          const float* __restrict__ rstd,
                                                          const float* __restrict__ gamma,
                                                          const float* __restrict__ beta, float slope,
                                                          float* __restrict__ dy, double* __restrict__ part,
                                                          unsigned* __restrict__ amax) {
  const int Co = (ACT == OG_NA_GLU) ? Cy / 2 : Cy;
  const int Co4 = Co >> 2;
  const int c4 = blockIdx.x * 32 + threadIdx.x;
  const long long p0 = (long long)blockIdx.y * pix_per_block;
  const long long p1 = min(P, p0 + pix_per_block);
  constexpr int NV = (ACT == OG_NA_GLU) ? 16 : 8;
  double acc[NV];
#pragma unroll
  for (int i = 0; i < NV; ++i) acc[i] = 0;
  float mx = 0.f;
  if (c4 < Co4) {
    const int c = c4 * 4;
    ChanConst k;
    load_chan<ACT>(k, mean, rstd, gamma, beta, 0, Cy, Co, c);
    const float4 s = make_float4(k.r.x * k.ga.x, k.r.y * k.ga.y, k.r.z * k.ga.z, k.r.w * k.ga.w);
    const float4 s2 = make_float4(k.r2.x * k.ga2.x, k.r2.y * k.ga2.y, k.r2.z * k.ga2.z, k.r2.w * k.ga2.w);
    const float* yb = y + c;
    const float* gb = g + c;
    float* db = dy + c;
    const float4 zero = make_float4(0.f, 0.f, 0.f, 0.f);
    for (long long p = p0 + threadIdx.y; p < p1; p += 8) {
      const float4 v = ldg4(yb + p * Cy), go = ldg4(gb + p * Co);
      const float4 v2 = (ACT == OG_NA_GLU) ? ldg4(yb + p * Cy + Co) : zero;
      float4 xh, dn, xh2, dn2;
      act_grad4<ACT>(k, v, v2, go, slope, xh, dn, xh2, dn2);
      const float4 o = make_float4(dn.x * s.x, dn.y * s.y, dn.z * s.z, dn.w * s.w);
      st4(db + p * Cy, o);
      mx = amax4(mx, o);
      if (ACT == OG_NA_GLU) {
        const float4 o2 = make_float4(dn2.x * s2.x, dn2.y * s2.y, dn2.z * s2.z, dn2.w * s2.w);
        st4(db + p * Cy + Co, o2);
        mx = amax4(mx, o2);
      }
      acc[0] += dn.x; acc[1] += dn.y; acc[2] += dn.z; acc[3] += dn.w;
      acc[4] += (double)dn.x * xh.x; acc[5] += (double)dn.y * xh.y;
      acc[6] += (double)dn.z * xh.z; acc[7] += (double)dn.w * xh.w;
      if (ACT == OG_NA_GLU) {
        acc[NV - 8] += dn2.x; acc[NV - 7] += dn2.y; acc[NV - 6] += dn2.z; acc[NV - 5] += dn2.w;
        acc[NV - 4] += (double)dn2.x * xh2.x; acc[NV - 3] += (double)dn2.y * xh2.y;
        acc[NV - 2] += (double)dn2.z * xh2.z; acc[NV - 1] += (double)dn2.w * xh2.w;
      }
    }
  }
  if (amax) block_amax_256(mx, amax);
  if (!part) return;
  __shared__ double sh[8][32][NV];
#pragma unroll
  for (int i = 0; i < NV; ++i) sh[threadIdx.y][threadIdx.x][i] = acc[i];
  __syncthreads();
  const int t = threadIdx.y * 32 + threadIdx.x;
  double* plane = part + (long long)blockIdx.y * 2 * Cy;
  for (int item = t; item < 32 * NV; item += 256) {
    const int cx = item / NV, kk = item % NV;
    double a = 0;
#pragma unroll
    for (int j = 0; j < 8; ++j) a += sh[j][cx][kk];
    const int cc4 = blockIdx.x * 32 + cx;
    if (cc4 < Co4) {
      const int half = kk >> 3;              // 0: "a" half, 1: gate half (GLU only)
      const int ch = half * Co + cc4 * 4 + (kk & 3);
      plane[((kk & 7) >> 2) * Cy + ch] = a;  // [0][ch] = sum dn, [1][ch] = sum dn * xhat
    }
  }
}

// dbeta = sum_s part[s][0][c], dgamma = sum_s part[s][1][c], planes added in the order s = 0, 1, ...
__global__ void bn_eval_param_grad_kernel(const double* __restrict__ part, int S, int C, float* dgamma, float* dbeta,
                                          int accumulate) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= C) return;
  double sb = 0, sg = 0;
  for (int s = 0; s < S; ++s) {
    sb += part[(long long)s * 2 * C + i];
    sg += part[(long long)s * 2 * C + C + i];
  }
  dgamma[i] = accumulate ? dgamma[i] + (float)sg : (float)sg;
  dbeta[i] = accumulate ? dbeta[i] + (float)sb : (float)sb;
}

static int elem_blocks(long long total) {
  long long b = (total + 255) / 256;
  long long cap = (long long)og_num_sms() * 32;
  return (int)(b < cap ? (b < 1 ? 1 : b) : cap);
}
static int pix_chunk(long long P, int cgroups, int groups) {
  // aim for >= ~4 blocks per SM overall, at least 64 pixels per block
  long long want = (long long)og_num_sms() * 8;
  long long chunks = want / ((long long)cgroups * groups) + 1;
  long long ppb = (P + chunks - 1) / chunks;
  if (ppb < 64) ppb = 64;
  return (int)ppb;
}

// stats: fp64 [groups][C][2] (zeroed here); mean/rstd: fp32 [groups][C]
OG_API int og_norm_stats(const float* x, int groups, long long P, int C, float eps, double* stats, float* mean,
                         float* rstd, float* running_mean, float* running_var, float momentum, int real_c,
                         long long* num_batches_tracked, cudaStream_t stream) {
  if (C % 4) return (int)cudaErrorInvalidValue;
  OG_CHECK(cudaMemsetAsync(stats, 0, sizeof(double) * 2 * groups * C, stream));
  int cg = og_cdiv(C / 4, 32);
  int ppb = pix_chunk(P, cg, groups);
  dim3 grid(cg, og_cdiv(P, ppb), groups), block(32, 8);
  norm_stats_kernel<<<grid, block, 0, stream>>>(x, C, P, ppb, stats);
  norm_finalize_kernel<<<og_cdiv((long long)groups * C, 256), 256, 0, stream>>>(stats, groups, C, (double)P, eps, mean, rstd,
                                                                     running_mean, running_var, momentum, real_c,
                                                                     num_batches_tracked);
  OG_RETURN_LAST_ERROR();
}

OG_API int og_norm_apply(const float* y, int groups, long long P, int Cy, const float* mean, const float* rstd,
                         const float* gamma, const float* beta, const float* res, int act, float slope, float* out,
                         unsigned* amax_out, cudaStream_t stream) {
  long long tp = (long long)groups * P;
  int Co = act == OG_NA_GLU ? Cy / 2 : Cy;
  if (Cy % 4 || Co % 4) return (int)cudaErrorInvalidValue;
  if (amax_out) OG_CHECK(cudaMemsetAsync(amax_out, 0, sizeof(unsigned), stream));
  int blocks = elem_blocks(tp * (Co / 4));
  if (act == OG_NA_GLU)
    norm_apply_kernel<OG_NA_GLU><<<blocks, 256, 0, stream>>>(y, Cy, P, tp, mean, rstd, gamma, beta, res, slope, out, amax_out);
  else if (act == OG_NA_LRELU)
    norm_apply_kernel<OG_NA_LRELU><<<blocks, 256, 0, stream>>>(y, Cy, P, tp, mean, rstd, gamma, beta, res, slope, out, amax_out);
  else
    norm_apply_kernel<OG_NA_NONE><<<blocks, 256, 0, stream>>>(y, Cy, P, tp, mean, rstd, gamma, beta, res, slope, out, amax_out);
  OG_RETURN_LAST_ERROR();
}

// g: gradient w.r.t. the fused output ([groups*P][Co]); dy: gradient w.r.t. the conv output y.
// bstats: fp64 scratch [groups][Cy][2].  dgamma/dbeta optional (batch norm).
OG_API int og_norm_backward(const float* y, const float* g, int groups, long long P, int Cy, const float* mean,
                            const float* rstd, const float* gamma, const float* beta, int act, float slope,
                            double* bstats, float* dy, float* dgamma, float* dbeta, int accumulate_param_grads,
                            unsigned* amax_dy, cudaStream_t stream) {
  int Co = act == OG_NA_GLU ? Cy / 2 : Cy;
  if (Cy % 4 || Co % 4) return (int)cudaErrorInvalidValue;
  OG_CHECK(cudaMemsetAsync(bstats, 0, sizeof(double) * 2 * groups * Cy, stream));
  if (amax_dy) OG_CHECK(cudaMemsetAsync(amax_dy, 0, sizeof(unsigned), stream));
  int cg = og_cdiv(Co / 4, 32);
  int ppb = pix_chunk(P, cg, groups);
  dim3 grid(cg, og_cdiv(P, ppb), groups), block(32, 8);
  double inv = 1.0 / (double)P;
#define OG_LAUNCH_BWD(A)                                                                                           \
  norm_bwd_reduce_kernel<A><<<grid, block, 0, stream>>>(y, g, Cy, P, ppb, mean, rstd, gamma, beta, slope, bstats); \
  if (dgamma && groups == 1)                                                                                       \
    norm_param_grad_kernel<<<og_cdiv(Cy, 256), 256, 0, stream>>>(bstats, Cy, dgamma, dbeta, accumulate_param_grads); \
  norm_bwd_coef_kernel<<<og_cdiv((long long)groups * Cy, 256), 256, 0, stream>>>(bstats, (long long)groups * Cy, inv); \
  norm_bwd_apply_kernel<A><<<grid, block, 0, stream>>>(y, g, Cy, P, ppb, mean, rstd, gamma, beta, slope, bstats, dy, amax_dy);
  if (act == OG_NA_GLU) {
    OG_LAUNCH_BWD(OG_NA_GLU)
  } else if (act == OG_NA_LRELU) {
    OG_LAUNCH_BWD(OG_NA_LRELU)
  } else {
    OG_LAUNCH_BWD(OG_NA_NONE)
  }
#undef OG_LAUNCH_BWD
  OG_RETURN_LAST_ERROR();
}

// eval-mode BatchNorm: mean = running_mean, rstd = 1 / sqrt(running_var + eps) (fp32 [C]); the buffers are only read
OG_API int og_bn_eval_coef(const float* running_mean, const float* running_var, int C, float eps, float* mean,
                           float* rstd, cudaStream_t stream) {
  if (C <= 0) return (int)cudaErrorInvalidValue;
  bn_eval_coef_kernel<<<og_cdiv(C, 256), 256, 0, stream>>>(running_mean, running_var, C, eps, mean, rstd);
  OG_RETURN_LAST_ERROR();
}

// Backward of og_norm_apply (groups = 1) with og_bn_eval_coef's statistics.  g: gradient w.r.t. the fused output
// ([P][Co]); dy: gradient w.r.t. y ([P][Cy]).  dgamma / dbeta optional (both or neither); accumulate_param_grads adds
// into them instead of overwriting.
OG_API int og_bn_eval_backward(const float* y, const float* g, long long P, int Cy, const float* mean,
                               const float* rstd, const float* gamma, const float* beta, int act, float slope, float* dy,
                               float* dgamma, float* dbeta, int accumulate_param_grads, unsigned* amax_dy,
                               cudaStream_t stream) {
  const int Co = act == OG_NA_GLU ? Cy / 2 : Cy;
  if (Cy % 4 || Co % 4 || (dgamma == nullptr) != (dbeta == nullptr)) return (int)cudaErrorInvalidValue;
  if (amax_dy) OG_CHECK(cudaMemsetAsync(amax_dy, 0, sizeof(unsigned), stream));
  if (P == 0) {
    if (dgamma && !accumulate_param_grads) {
      OG_CHECK(cudaMemsetAsync(dgamma, 0, sizeof(float) * Cy, stream));
      OG_CHECK(cudaMemsetAsync(dbeta, 0, sizeof(float) * Cy, stream));
    }
    return 0;
  }
  const int cg = og_cdiv(Co / 4, 32);
  const int ppb = pix_chunk(P, cg, 1);
  const dim3 grid(cg, og_cdiv(P, ppb), 1), block(32, 8);
  double* part = nullptr;
  if (dgamma) {
    float* w = nullptr;
    OG_CHECK(og_work_alloc(&w, (size_t)grid.y * 2 * Cy * 2, stream));     // doubles as pairs of floats
    part = reinterpret_cast<double*>(w);
  }
  if (act == OG_NA_GLU)
    bn_eval_bwd_kernel<OG_NA_GLU><<<grid, block, 0, stream>>>(y, g, Cy, P, ppb, mean, rstd, gamma, beta, slope, dy, part, amax_dy);
  else if (act == OG_NA_LRELU)
    bn_eval_bwd_kernel<OG_NA_LRELU><<<grid, block, 0, stream>>>(y, g, Cy, P, ppb, mean, rstd, gamma, beta, slope, dy, part, amax_dy);
  else
    bn_eval_bwd_kernel<OG_NA_NONE><<<grid, block, 0, stream>>>(y, g, Cy, P, ppb, mean, rstd, gamma, beta, slope, dy, part, amax_dy);
  int rc = (int)cudaGetLastError();
  if (part) {
    if (!rc) {
      bn_eval_param_grad_kernel<<<og_cdiv(Cy, 256), 256, 0, stream>>>(part, (int)grid.y, Cy, dgamma, dbeta,
                                                                     accumulate_param_grads);
      rc = (int)cudaGetLastError();
    }
    const cudaError_t e = cudaFreeAsync(part, stream);
    if (!rc) rc = (int)e;
  }
  return rc;
}

// *out_word = float bits of an upper bound of max|og_norm_apply output| (see norm_apply_split_kernel): max|gamma| *
// sqrt(count) + max|beta| (+ the bound / amax word of the residual).  gamma / beta null = InstanceNorm without affine.
OG_API int og_norm_bound(const float* gamma, const float* beta, int C, long long count, const unsigned* res_word,
                         unsigned* out_word, cudaStream_t stream) {
  norm_bound_kernel<<<1, 256, 0, stream>>>(gamma, beta, C, (double)count, res_word, out_word);
  OG_RETURN_LAST_ERROR();
}

// og_norm_apply fused with og_prep_split of its output: y [N][H][W][Cy] -> fp16 hi / lo [N][H + 2 pad][W + 2 pad][Co]
// scaled by the power of two of *bound_word (og_norm_bound), pad = 1 adds the reflection halo; out (fp32, [N][H][W][Co])
// may be null when nothing else reads the activation; xl may be null (single-product mode).
OG_API int og_norm_apply_split(const float* y, int N, int H, int W, int Cy, int instance, const float* mean,
                               const float* rstd, const float* gamma, const float* beta, const float* res, int act,
                               float slope, float* out, const unsigned* bound_word, int pad, void* xh, void* xl,
                               cudaStream_t stream) {
  const int Co = act == OG_NA_GLU ? Cy / 2 : Cy;
  if (Co % 8 || pad < 0 || pad > 1 || (pad && (H < 2 || W < 2))) return (int)cudaErrorInvalidValue;
  const long long total = (long long)N * (H + 2 * pad) * (W + 2 * pad) * (Co / 8);
  if (total == 0) return 0;
  long long b = (total + 255) / 256;
  if (b > (long long)og_num_sms() * 32) b = (long long)og_num_sms() * 32;
#define OG_LAUNCH_AS(A)                                                                                              \
  norm_apply_split_kernel<A><<<(int)b, 256, 0, stream>>>(y, N, H, W, Cy, instance, mean, rstd, gamma, beta, res, slope, \
                                                         out, bound_word, pad, total, (__half*)xh, (__half*)xl)
  if (act == OG_NA_GLU) OG_LAUNCH_AS(OG_NA_GLU);
  else if (act == OG_NA_LRELU) OG_LAUNCH_AS(OG_NA_LRELU);
  else OG_LAUNCH_AS(OG_NA_NONE);
#undef OG_LAUNCH_AS
  OG_RETURN_LAST_ERROR();
}
