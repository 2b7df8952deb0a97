// Implicit-GEMM convolution on the CUDA cores (exact fp32 FMA arithmetic), NHWC activations.
//
// This is the general-purpose contraction kernel of the library: every conv / transposed conv /
// linear layer of G_NET and the PAT_D_NETs (reference image_generation/model.py:36-49, 63-81,
// 486-518, 589-617, 708-719, 999-1048) can run through it, in forward (fprop), input-gradient
// (dgrad == fprop in OG_TRANSPOSED addressing with re-packed weights) and weight-gradient (wgrad).
// The tensor-core path (conv_tc.cu) takes over the shapes that dominate the step; this kernel stays as
// the exact-fp32 path for small / odd shapes and as the on-device cross-check.
//
// GEMM view (fprop): rows m = (n, oh, ow) output pixels, cols = output channels (padded to 4),
// reduction k = (kh, kw, ci) with ci padded to 8.  A is gathered on the fly from the NHWC input
// with the addressing mode (zero pad / reflection pad / nearest-2x-upsample-then-zero-pad /
// transposed); B is a pre-packed [(kh,kw,ci)][co] matrix (og_pack_weights).
#include "common.cuh"

struct ConvArgs {
  const float* x;  // source NHWC
  int N, H, W, C;  // source dims (C % 8 == 0)
  long long xsn, xsh, xsw;
  const float* w;  // packed [(KH*KW*C)][K]
  float* y;        // result NHWC, channels K (K % 4 == 0)
  int OH, OW, K;
  long long ysn, ysh, ysw;
  int KH, KW, stride, pad, mode;
  const float* bias;  // [K] or null
  int act;
  float slope;
  float* work;       // split-K: slice z writes its partial result to work + z * work_plane (y's layout)
  long long work_plane;
  int padw;          // column padding (pad is the row padding)
};

__device__ __forceinline__ int src_coord(int mode, int o, int k, int stride, int pad, int Hs) {
  if (mode == OG_PAD_ZERO) {
    int i = o * stride + k - pad;
    return (i < 0 || i >= Hs) ? -1 : i;
  } else if (mode == OG_PAD_REFLECT) {
    int i = o * stride + k - pad;
    if (i < 0) i = -i;
    if (i >= Hs) i = 2 * Hs - 2 - i;
    return i;
  } else if (mode == OG_UPSAMPLE2X) {
    int u = o + k - pad;
    return (u < 0 || u >= 2 * Hs) ? -1 : (u >> 1);
  } else {  // OG_TRANSPOSED: rows are input pixels of the forward conv, source is the output gradient
    int t = o + pad - k;
    if (t < 0 || (t % stride) != 0) return -1;
    int i = t / stride;
    return i >= Hs ? -1 : i;
  }
}

__device__ __forceinline__ float apply_act(float v, int act, float slope) {
  if (act == OG_ACT_LRELU) return v > 0.f ? v : v * slope;
  if (act == OG_ACT_TANH) return tanhf(v);
  if (act == OG_ACT_SIGMOID) return og_sigmoid(v);
  return v;
}

constexpr int BM = 128, BK = 8, BMP = BM + 4;

template <int TN>
__device__ __forceinline__ void mma_tile(const float (*As)[BMP], const float* Bs, int bnp, float (&acc)[8][TN], int tx,
                                         int ty) {
#pragma unroll
  for (int k = 0; k < BK; ++k) {
    float a[8], b[TN];
    float4 a0 = *reinterpret_cast<const float4*>(&As[k][ty * 4]);
    float4 a1 = *reinterpret_cast<const float4*>(&As[k][64 + ty * 4]);
    a[0] = a0.x; a[1] = a0.y; a[2] = a0.z; a[3] = a0.w;
    a[4] = a1.x; a[5] = a1.y; a[6] = a1.z; a[7] = a1.w;
    const float* brow = Bs + k * bnp;
    if (TN == 8) {
      float4 b0 = *reinterpret_cast<const float4*>(brow + tx * 4);
      float4 b1 = *reinterpret_cast<const float4*>(brow + 64 + tx * 4);
      b[0] = b0.x; b[1] = b0.y; b[2] = b0.z; b[3] = b0.w;
      b[TN - 4] = b1.x; b[TN - 3] = b1.y; b[TN - 2] = b1.z; b[TN - 1] = b1.w;
    } else if (TN == 4) {
      float4 b0 = *reinterpret_cast<const float4*>(brow + tx * 4);
      b[0] = b0.x; b[1] = b0.y; b[2] = b0.z; b[3] = b0.w;
    } else {
      float2 b0 = *reinterpret_cast<const float2*>(brow + tx * 2);
      b[0] = b0.x; b[1] = b0.y;
    }
#pragma unroll
    for (int i = 0; i < 8; ++i)
#pragma unroll
      for (int j = 0; j < TN; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
  }
}

// column of accumulator j for thread tx
template <int TN>
__device__ __forceinline__ int acc_col(int tx, int j) {
  if (TN == 8) return j < 4 ? tx * 4 + j : 64 + tx * 4 + (j - 4);
  if (TN == 4) return tx * 4 + j;
  return tx * 2 + j;
}
__device__ __forceinline__ int acc_row(int ty, int i) { return i < 4 ? ty * 4 + i : 64 + ty * 4 + (i - 4); }

template <int TN>
__global__ void __launch_bounds__(256) conv_gemm_kernel(ConvArgs a) {
  constexpr int BN = 16 * TN;
  __shared__ __align__(16) float As[2][BK][BMP];
  __shared__ __align__(16) float Bs[2][BK * BN];
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
  const long long M = (long long)a.N * a.OH * a.OW;
  const long long m0 = (long long)blockIdx.x * BM;
  const int n0 = blockIdx.y * BN;
  const int cchunks = a.C / BK;
  const int nk_total = a.KH * a.KW * cchunks;
  // split-K range
  const int per = (nk_total + gridDim.z - 1) / gridDim.z;
  const int kt_beg = blockIdx.z * per;
  const int kt_end = min(nk_total, kt_beg + per);
  if (kt_beg >= kt_end) return;

  // A-load role: one float4 per thread
  const int ar = tid >> 1, ah = tid & 1;
  const long long am = m0 + ar;
  const bool am_ok = am < M;
  int an = 0, aoh = 0, aow = 0;
  if (am_ok) {
    an = (int)(am / ((long long)a.OH * a.OW));
    int rem = (int)(am - (long long)an * a.OH * a.OW);
    aoh = rem / a.OW;
    aow = rem - aoh * a.OW;
  }
  // B-load role
  constexpr int COLS4 = BN / 4;
  const int bk = tid / COLS4, bc4 = tid % COLS4;
  const bool b_ok = (bk < BK) && (n0 + bc4 * 4 < a.K);

  int tap = kt_beg / cchunks;
  int cc = kt_beg - tap * cchunks;
  const float* aptr = nullptr;
  auto set_tap = [&](int t) {
    aptr = nullptr;
    if (!am_ok) return;
    int kh = t / a.KW, kw = t - kh * a.KW;
    int ih = src_coord(a.mode, aoh, kh, a.stride, a.pad, a.H);
    int iw = src_coord(a.mode, aow, kw, a.stride, a.padw, a.W);
    if (ih < 0 || iw < 0) return;
    aptr = a.x + an * a.xsn + ih * a.xsh + iw * a.xsw + ah * 4;
  };
  set_tap(tap);

  float4 ra, rb;
  auto gload = [&](int kt) {
    ra = make_float4(0.f, 0.f, 0.f, 0.f);
    rb = ra;
    if (aptr) ra = ldg4(aptr + cc * BK);
    if (b_ok) rb = ldg4(a.w + (long long)(kt * BK + bk) * a.K + n0 + bc4 * 4);
  };
  auto sstore = [&](int buf) {
    As[buf][ah * 4 + 0][ar] = ra.x;
    As[buf][ah * 4 + 1][ar] = ra.y;
    As[buf][ah * 4 + 2][ar] = ra.z;
    As[buf][ah * 4 + 3][ar] = ra.w;
    if (bk < BK) *reinterpret_cast<float4*>(&Bs[buf][bk * BN + bc4 * 4]) = rb;
  };
  auto advance = [&]() {
    if (++cc == cchunks) {
      cc = 0;
      ++tap;
      if (tap < a.KH * a.KW) set_tap(tap);
    }
  };

  float acc[8][TN];
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int j = 0; j < TN; ++j) acc[i][j] = 0.f;

  gload(kt_beg);
  sstore(0);
  advance();
  __syncthreads();
  int cur = 0;
  for (int kt = kt_beg; kt < kt_end; ++kt) {
    const bool more = kt + 1 < kt_end;
    if (more) gload(kt + 1);
    mma_tile<TN>(As[cur], Bs[cur], BN, acc, tx, ty);
    if (more) {
      sstore(cur ^ 1);
      advance();
    }
    __syncthreads();
    cur ^= 1;
  }

  // epilogue
  const bool atomic = gridDim.z > 1;
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    long long m = m0 + acc_row(ty, i);
    if (m >= M) continue;
    int n = (int)(m / ((long long)a.OH * a.OW));
    int rem = (int)(m - (long long)n * a.OH * a.OW);
    int oh = rem / a.OW, ow = rem - oh * a.OW;
    float* yrow = a.y + n * a.ysn + oh * a.ysh + ow * a.ysw;
#pragma unroll
    for (int j = 0; j < TN; ++j) {
      int c = n0 + acc_col<TN>(tx, j);
      if (c >= a.K) continue;
      float v = acc[i][j];
      if (atomic) {
        a.work[(long long)blockIdx.z * a.work_plane + (yrow - a.y) + c] = v;
      } else {
        if (a.bias) v += __ldg(a.bias + c);
        yrow[c] = apply_act(v, a.act, a.slope);
      }
    }
  }
}

// ---------------------------------------------------------------------------------------------
// wgrad: dW[(kh,kw,ci)][co] += sum over output pixels m of  x[src(m,kh,kw)][ci] * g[m][co]
// ---------------------------------------------------------------------------------------------
struct WgradArgs {
  const float* x;  // forward input NHWC
  int N, H, W, C;
  long long xsn, xsh, xsw;
  const float* g;  // output gradient NHWC, K channels
  int OH, OW, K;
  long long gsn, gsh, gsw;
  float* dw;  // packed [(KH*KW*C)][K]: written by the one split, else the sum of the work planes (og_split_sum)
  int KH, KW, stride, pad, mode;
  int pix_per_split;  // multiple of 8
  float* work;       // pixel splits: split z writes its partial dw to work + z * R * K (null: one split, into dw)
};

template <int TN>
__global__ void __launch_bounds__(256) conv_wgrad_kernel(WgradArgs a) {
  constexpr int BN = 16 * TN;
  __shared__ __align__(16) float As[2][BK][BMP];
  __shared__ __align__(16) float Bs[2][BK * BN];
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
  const int R = a.KH * a.KW * a.C;
  const int r0 = blockIdx.x * BM;
  const int n0 = blockIdx.y * BN;
  const long long M = (long long)a.N * a.OH * a.OW;
  const long long mbeg = (long long)blockIdx.z * a.pix_per_split;
  const long long mend = min(M, mbeg + a.pix_per_split);
  if (mbeg >= mend) return;
  const int nk = (int)((mend - mbeg + BK - 1) / BK);

  // A-load role: pixel pj of the chunk, rows q*4..q*4+3 of the tile
  const int pj = tid >> 5, q = tid & 31;
  const int r = r0 + q * 4;
  const bool r_ok = r < R;
  int kh = 0, kw = 0, ci = 0;
  if (r_ok) {
    int tap = r / a.C;
    ci = r - tap * a.C;
    kh = tap / a.KW;
    kw = tap - kh * a.KW;
  }
  constexpr int COLS4 = BN / 4;
  const int bp = tid / COLS4, bc4 = tid % COLS4;
  const bool b_ok = (bp < BK) && (n0 + bc4 * 4 < a.K);
  const long long ohow = (long long)a.OH * a.OW;

  float4 ra, rb;
  auto gload = [&](int kt) {
    ra = make_float4(0.f, 0.f, 0.f, 0.f);
    rb = ra;
    long long m = mbeg + (long long)kt * BK + pj;
    if (r_ok && m < mend) {
      int n = (int)(m / ohow);
      int rem = (int)(m - n * ohow);
      int oh = rem / a.OW, ow = rem - oh * a.OW;
      int ih = src_coord(a.mode, oh, kh, a.stride, a.pad, a.H);
      int iw = src_coord(a.mode, ow, kw, a.stride, a.pad, a.W);
      if (ih >= 0 && iw >= 0) ra = ldg4(a.x + n * a.xsn + ih * a.xsh + iw * a.xsw + ci);
    }
    long long mb = mbeg + (long long)kt * BK + bp;
    if (b_ok && mb < mend) {
      int n = (int)(mb / ohow);
      int rem = (int)(mb - n * ohow);
      int oh = rem / a.OW, ow = rem - oh * a.OW;
      rb = ldg4(a.g + n * a.gsn + oh * a.gsh + ow * a.gsw + n0 + bc4 * 4);
    }
  };
  auto sstore = [&](int buf) {
    *reinterpret_cast<float4*>(&As[buf][pj][q * 4]) = ra;
    if (bp < BK) *reinterpret_cast<float4*>(&Bs[buf][bp * BN + bc4 * 4]) = rb;
  };

  float acc[8][TN];
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int j = 0; j < TN; ++j) acc[i][j] = 0.f;

  gload(0);
  sstore(0);
  __syncthreads();
  int cur = 0;
  for (int kt = 0; kt < nk; ++kt) {
    const bool more = kt + 1 < nk;
    if (more) gload(kt + 1);
    mma_tile<TN>(As[cur], Bs[cur], BN, acc, tx, ty);
    if (more) sstore(cur ^ 1);
    __syncthreads();
    cur ^= 1;
  }
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    int rr = r0 + acc_row(ty, i);
    if (rr >= R) continue;
#pragma unroll
    for (int j = 0; j < TN; ++j) {
      int c = n0 + acc_col<TN>(tx, j);
      if (c >= a.K) continue;
      (a.work ? a.work + (long long)blockIdx.z * R * a.K : a.dw)[(long long)rr * a.K + c] = acc[i][j];
    }
  }
}

// ---------------------------------------------------------------------------------------------
// "narrow" convolutions: at most 8 output channels and a long reduction (the k4 s2 p0 logit heads of
// D_GET_LOGITS, model.py:1031-1033: 768 -> 1 on 16x16 / 8x8 / 4x4 maps).  A GEMM tile is the wrong shape for
// them (7 CTAs, 1536 k-steps each); these are dot products: one warp per output pixel in the forward,
// one thread per input element in dgrad, one thread per weight row in wgrad.  Weights: packed [(kh,kw,ci)][8].
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) conv_narrow_fwd_kernel(const float* __restrict__ x, int N, int H, int W, int C,
                                                              const float* __restrict__ w, float* __restrict__ y,
                                                              int OH, int OW, int KH, int KW, int stride, int pad,
                                                              const float* __restrict__ bias, int act, float slope) {
  const int lane = threadIdx.x & 31;
  const long long pix = (long long)blockIdx.x * 8 + (threadIdx.x >> 5);
  if (pix >= (long long)N * OH * OW) return;
  const int n = (int)(pix / (OH * OW));
  const int rem = (int)(pix - (long long)n * OH * OW);
  const int oh = rem / OW, ow = rem - oh * OW;
  float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  const int C4 = C >> 2;
  for (int kh = 0; kh < KH; ++kh) {
    const int ih = oh * stride + kh - pad;
    if (ih < 0 || ih >= H) continue;
    for (int kw = 0; kw < KW; ++kw) {
      const int iw = ow * stride + kw - pad;
      if (iw < 0 || iw >= W) continue;
      const float* xp = x + (((long long)n * H + ih) * W + iw) * C;
      const float* wp = w + (long long)(kh * KW + kw) * C * 8;
      for (int c4 = lane; c4 < C4; c4 += 32) {
        const float4 xv = ldg4(xp + c4 * 4);
        const float xs[4] = {xv.x, xv.y, xv.z, xv.w};
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          const float4 w0 = ldg4(wp + (c4 * 4 + k) * 8), w1 = ldg4(wp + (c4 * 4 + k) * 8 + 4);
          acc[0] = fmaf(xs[k], w0.x, acc[0]); acc[1] = fmaf(xs[k], w0.y, acc[1]);
          acc[2] = fmaf(xs[k], w0.z, acc[2]); acc[3] = fmaf(xs[k], w0.w, acc[3]);
          acc[4] = fmaf(xs[k], w1.x, acc[4]); acc[5] = fmaf(xs[k], w1.y, acc[5]);
          acc[6] = fmaf(xs[k], w1.z, acc[6]); acc[7] = fmaf(xs[k], w1.w, acc[7]);
        }
      }
    }
  }
#pragma unroll
  for (int j = 0; j < 8; ++j) acc[j] = warp_sum(acc[j]);
  if (lane < 8) {
    float v = acc[0];
#pragma unroll
    for (int j = 1; j < 8; ++j)
      if (lane == j) v = acc[j];
    if (bias) v += bias[lane];
    y[pix * 8 + lane] = apply_act(v, act, slope);
  }
}

// Long reductions (the logit heads: 16 taps x 768 channels for a few hundred output pixels): one block = 8 output
// pixels, its 8 warps split the (tap, channel) range, so every weight vector is read once per 8 pixels and the
// reduction is 256-way parallel; partial sums meet in shared memory.
__global__ void __launch_bounds__(256) conv_narrow_fwd_long_kernel(const float* __restrict__ x, int N, int H, int W, int C,
                                                                   const float* __restrict__ w, float* __restrict__ y,
                                                                   int OH, int OW, int KH, int KW, int stride, int pad,
                                                                   const float* __restrict__ bias, int act, float slope) {
  constexpr int PPB = 8;
  __shared__ float red[8][PPB * 8];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const long long npix = (long long)N * OH * OW;
  const long long pix0 = (long long)blockIdx.x * PPB;
  int ih0[PPB], iw0[PPB];
  long long xoff[PPB];
#pragma unroll
  for (int p = 0; p < PPB; ++p) {
    const long long pix = pix0 + p;
    if (pix < npix) {
      const int n = (int)(pix / (OH * OW));
      const int rem = (int)(pix - (long long)n * OH * OW);
      const int oh = rem / OW, ow = rem - oh * OW;
      ih0[p] = oh * stride - pad;
      iw0[p] = ow * stride - pad;
      xoff[p] = (long long)n * H * W * C;
    } else {
      ih0[p] = -(1 << 20);     // never in range
      iw0[p] = 0;
      xoff[p] = 0;
    }
  }
  float acc[PPB][8];
#pragma unroll
  for (int p = 0; p < PPB; ++p)
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[p][j] = 0.f;
  const int C4 = C >> 2, items = KH * KW * C4;
  for (int i = threadIdx.x; i < items; i += 256) {
    const int tap = i / C4, c4 = i - tap * C4;
    const int kh = tap / KW, kw = tap - kh * KW;
    const float* wp = w + ((long long)tap * C + c4 * 4) * 8;
    float4 wv[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) wv[k] = ldg4(wp + k * 4);      // rows c4*4 .. c4*4+3, 8 outputs each
#pragma unroll
    for (int p = 0; p < PPB; ++p) {
      const int ih = ih0[p] + kh, iw = iw0[p] + kw;
      if (ih < 0 || ih >= H || iw < 0 || iw >= W) continue;
      const float4 xv = ldg4(x + xoff[p] + ((long long)ih * W + iw) * C + c4 * 4);
      const float xs[4] = {xv.x, xv.y, xv.z, xv.w};
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        acc[p][0] = fmaf(xs[k], wv[2 * k].x, acc[p][0]); acc[p][1] = fmaf(xs[k], wv[2 * k].y, acc[p][1]);
        acc[p][2] = fmaf(xs[k], wv[2 * k].z, acc[p][2]); acc[p][3] = fmaf(xs[k], wv[2 * k].w, acc[p][3]);
        acc[p][4] = fmaf(xs[k], wv[2 * k + 1].x, acc[p][4]); acc[p][5] = fmaf(xs[k], wv[2 * k + 1].y, acc[p][5]);
        acc[p][6] = fmaf(xs[k], wv[2 * k + 1].z, acc[p][6]); acc[p][7] = fmaf(xs[k], wv[2 * k + 1].w, acc[p][7]);
      }
    }
  }
#pragma unroll
  for (int p = 0; p < PPB; ++p)
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const float v = warp_sum(acc[p][j]);
      if (lane == 0) red[warp][p * 8 + j] = v;
    }
  __syncthreads();
  if (threadIdx.x < PPB * 8) {
    float v = 0.f;
#pragma unroll
    for (int wi = 0; wi < 8; ++wi) v += red[wi][threadIdx.x];
    const int p = threadIdx.x >> 3, j = threadIdx.x & 7;
    if (pix0 + p < npix) {
      if (bias) v += bias[j];
      y[(pix0 + p) * 8 + j] = apply_act(v, act, slope);
    }
  }
}

// gx[n,ih,iw,ci] = sum_{kh,kw: (ih+pad-kh) % stride == 0} sum_co g[n,oh,ow,co] * w[(kh,kw,ci)][co]
__global__ void conv_narrow_dgrad_kernel(const float* __restrict__ g, int N, int H, int W, int C,
                                         const float* __restrict__ w, float* __restrict__ gx, int OH, int OW, int KH,
                                         int KW, int stride, int pad, long long total) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int ci = (int)(i % C);
    long long t = i / C;
    const int iw = (int)(t % W);
    t /= W;
    const int ih = (int)(t % H);
    const int n = (int)(t / H);
    float acc = 0.f;
    for (int kh = 0; kh < KH; ++kh) {
      const int th = ih + pad - kh;
      if (th < 0 || th % stride) continue;
      const int oh = th / stride;
      if (oh >= OH) continue;
      for (int kw = 0; kw < KW; ++kw) {
        const int tw = iw + pad - kw;
        if (tw < 0 || tw % stride) continue;
        const int ow = tw / stride;
        if (ow >= OW) continue;
        const float* gp = g + (((long long)n * OH + oh) * OW + ow) * 8;
        const float* wp = w + ((long long)(kh * KW + kw) * C + ci) * 8;
        const float4 g0 = ldg4(gp), g1 = ldg4(gp + 4), w0 = ldg4(wp), w1 = ldg4(wp + 4);
        acc += g0.x * w0.x + g0.y * w0.y + g0.z * w0.z + g0.w * w0.w + g1.x * w1.x + g1.y * w1.y + g1.z * w1.z +
               g1.w * w1.w;
      }
    }
    gx[i] = acc;
  }
}

// dw[(kh,kw,ci)][co] = sum_{n,oh,ow} x[n,ih,iw,ci] * g[n,oh,ow,co]: one thread per weight row and slice of the output
// pixels (blockIdx.y); slice y writes its partial rows to dw + y * R * 8 (a workspace summed by og_split_sum)
__global__ void conv_narrow_wgrad_kernel(const float* __restrict__ x, int N, int H, int W, int C,
                                         const float* __restrict__ g, float* __restrict__ dw, int OH, int OW, int KH,
                                         int KW, int stride, int pad, int R, int pix_per_slice) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= R) return;
  const int ci = r % C, tap = r / C, kh = tap / KW, kw = tap - kh * KW;
  float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  const int npix = N * OH * OW;
  const int p0 = blockIdx.y * pix_per_slice, p1 = min(npix, p0 + pix_per_slice);
  int n = p0 / (OH * OW), rem = p0 - n * OH * OW;
  int oh = rem / OW, ow = rem - oh * OW;
  for (int p = p0; p < p1; ++p) {
    const int ih = oh * stride + kh - pad, iw = ow * stride + kw - pad;
    if (ih >= 0 && ih < H && iw >= 0 && iw < W) {
      const float xv = __ldg(x + (((long long)n * H + ih) * W + iw) * C + ci);
      const float* gp = g + (long long)p * 8;
      const float4 g0 = ldg4(gp), g1 = ldg4(gp + 4);
      acc[0] = fmaf(xv, g0.x, acc[0]); acc[1] = fmaf(xv, g0.y, acc[1]); acc[2] = fmaf(xv, g0.z, acc[2]);
      acc[3] = fmaf(xv, g0.w, acc[3]); acc[4] = fmaf(xv, g1.x, acc[4]); acc[5] = fmaf(xv, g1.y, acc[5]);
      acc[6] = fmaf(xv, g1.z, acc[6]); acc[7] = fmaf(xv, g1.w, acc[7]);
    }
    if (++ow == OW) {
      ow = 0;
      if (++oh == OH) { oh = 0; ++n; }
    }
  }
#pragma unroll
  for (int j = 0; j < 8; ++j) dw[(long long)blockIdx.y * R * 8 + (long long)r * 8 + j] = acc[j];
}

// ---------------------------------------------------------------------------------------------
// C ABI
// ---------------------------------------------------------------------------------------------
static int pick_splits(long long tiles, int nk, int want_ctas) {
  if (tiles >= want_ctas) return 1;
  int s = (int)((want_ctas + tiles - 1) / tiles);
  int maxs = nk / 16;  // keep at least 16 k-steps per split
  if (s > maxs) s = maxs;
  return s < 1 ? 1 : s;
}

// padh / padw: row / column padding (they differ for the 1x7 / 7x1 / 1x3 / 3x1 convolutions of Inception-v3)
OG_API int og_conv2d_simt(const float* x, int N, int H, int W, int C, long long xsn, long long xsh, long long xsw,
                          const float* wpacked, float* y, int OH, int OW, int K, long long ysn, long long ysh,
                          long long ysw, int KH, int KW, int stride, int padh, int padw, int mode, const float* bias,
                          int act, float slope, int allow_splitk, cudaStream_t stream) {
  if (C % 8 || K % 4) return (int)cudaErrorInvalidValue;
  ConvArgs a{x, N, H, W, C, xsn, xsh, xsw, wpacked, y, OH, OW, K, ysn, ysh, ysw, KH, KW, stride, padh, mode, bias, act, slope};
  a.padw = padw;
  long long M = (long long)N * OH * OW;
  if (M == 0) return 0;
  int TN = K > 64 ? 8 : (K > 32 ? 4 : 2);
  int BN = 16 * TN;
  dim3 grid(og_cdiv(M, BM), og_cdiv(K, BN), 1);
  int nk = KH * KW * (C / 8);
  if (allow_splitk && !bias && act == OG_ACT_NONE) {
    int s = pick_splits((long long)grid.x * grid.y, nk, 296);
    if (s > 1) {
      // split-K: every slice writes its partial result to its own plane of a workspace (no slice without work),
      // og_split_sum adds the planes in a fixed order
      if (ysw == K && ysh == (long long)OW * K && ysn == (long long)OH * OW * K) {
        grid.z = og_cdiv(nk, og_cdiv(nk, s));
        a.work_plane = M * K;
        OG_CHECK(og_work_alloc(&a.work, (size_t)grid.z * a.work_plane, stream));
      }
    }
  }
  if (TN == 8)
    conv_gemm_kernel<8><<<grid, 256, 0, stream>>>(a);
  else if (TN == 4)
    conv_gemm_kernel<4><<<grid, 256, 0, stream>>>(a);
  else
    conv_gemm_kernel<2><<<grid, 256, 0, stream>>>(a);
  int rc = (int)cudaGetLastError();
  if (grid.z > 1) {
    if (!rc) rc = og_split_sum(a.work, a.work_plane, (int)grid.z, y, stream);
    const cudaError_t e = cudaFreeAsync(a.work, stream);
    if (!rc) rc = (int)e;
  }
  return rc;
}

OG_API int og_conv2d_wgrad_simt(const float* x, int N, int H, int W, int C, long long xsn, long long xsh,
                                long long xsw, const float* g, int OH, int OW, int K, long long gsn, long long gsh,
                                long long gsw, float* dw_packed, int KH, int KW, int stride, int pad, int mode,
                                cudaStream_t stream) {
  if (C % 8 || K % 4) return (int)cudaErrorInvalidValue;
  long long M = (long long)N * OH * OW;
  int R = KH * KW * C;
  OG_CHECK(cudaMemsetAsync(dw_packed, 0, sizeof(float) * (long long)R * K, stream));
  if (M == 0) return 0;
  int TN = K > 64 ? 8 : (K > 32 ? 4 : 2);
  int BN = 16 * TN;
  dim3 grid(og_cdiv(R, BM), og_cdiv(K, BN), 1);
  long long tiles = (long long)grid.x * grid.y;
  long long splits = (592 + tiles - 1) / tiles;
  long long maxs = (M + 127) / 128;
  if (splits > maxs) splits = maxs;
  if (splits < 1) splits = 1;
  long long pps = (M + splits - 1) / splits;
  pps = (pps + 7) / 8 * 8;
  grid.z = og_cdiv(M, pps);
  WgradArgs a{x, N, H, W, C, xsn, xsh, xsw, g, OH, OW, K, gsn, gsh, gsw, dw_packed, KH, KW, stride, pad, mode, (int)pps};
  if (grid.z > 1) OG_CHECK(og_work_alloc(&a.work, (size_t)grid.z * R * K, stream));
  if (TN == 8)
    conv_wgrad_kernel<8><<<grid, 256, 0, stream>>>(a);
  else if (TN == 4)
    conv_wgrad_kernel<4><<<grid, 256, 0, stream>>>(a);
  else
    conv_wgrad_kernel<2><<<grid, 256, 0, stream>>>(a);
  int rc = (int)cudaGetLastError();
  if (grid.z > 1) {
    if (!rc) rc = og_split_sum(a.work, (long long)R * K, (int)grid.z, dw_packed, stream);
    const cudaError_t e = cudaFreeAsync(a.work, stream);
    if (!rc) rc = (int)e;
  }
  return rc;
}

// contiguous NHWC tensors, zero padding, output channels padded to exactly 8; wpacked = [(kh,kw,ci)][8]
OG_API int og_conv2d_narrow_fwd(const float* x, int N, int H, int W, int C, const float* wpacked, float* y, int OH,
                                int OW, int KH, int KW, int stride, int pad, const float* bias, int act, float slope,
                                cudaStream_t stream) {
  if (C % 4) return (int)cudaErrorInvalidValue;
  long long pix = (long long)N * OH * OW;
  if (pix == 0) return 0;
  if ((long long)KH * KW * (C / 4) >= 512)     // long reduction: split it over the block
    conv_narrow_fwd_long_kernel<<<og_cdiv(pix, 8), 256, 0, stream>>>(x, N, H, W, C, wpacked, y, OH, OW, KH, KW, stride,
                                                                     pad, bias, act, slope);
  else
    conv_narrow_fwd_kernel<<<og_cdiv(pix, 8), 256, 0, stream>>>(x, N, H, W, C, wpacked, y, OH, OW, KH, KW, stride, pad,
                                                                bias, act, slope);
  OG_RETURN_LAST_ERROR();
}
OG_API int og_conv2d_narrow_dgrad(const float* g, int N, int H, int W, int C, const float* wpacked, float* gx, int OH,
                                  int OW, int KH, int KW, int stride, int pad, cudaStream_t stream) {
  long long total = (long long)N * H * W * C;
  if (total == 0) return 0;
  long long b = (total + 255) / 256;
  if (b > (long long)og_num_sms() * 32) b = (long long)og_num_sms() * 32;
  conv_narrow_dgrad_kernel<<<(int)b, 256, 0, stream>>>(g, N, H, W, C, wpacked, gx, OH, OW, KH, KW, stride, pad, total);
  OG_RETURN_LAST_ERROR();
}
OG_API int og_conv2d_narrow_wgrad(const float* x, int N, int H, int W, int C, const float* g, float* dw_packed, int OH,
                                  int OW, int KH, int KW, int stride, int pad, cudaStream_t stream) {
  const int R = KH * KW * C;
  const long long npix = (long long)N * OH * OW;
  OG_CHECK(cudaMemsetAsync(dw_packed, 0, sizeof(float) * (size_t)R * 8, stream));
  if (npix == 0) return 0;
  // ~4 waves of 128-thread blocks over the GPU, at least 16 pixels per slice
  const int rb = og_cdiv(R, 128);
  long long slices = ((long long)og_num_sms() * 16 + rb - 1) / rb;
  if (slices > npix / 16) slices = npix / 16;
  if (slices < 1) slices = 1;
  if (slices > 65535) slices = 65535;
  const int pps = og_cdiv(npix, slices);
  dim3 grid(rb, og_cdiv(npix, pps));
  float* work = dw_packed;
  if (grid.y > 1) OG_CHECK(og_work_alloc(&work, (size_t)grid.y * R * 8, stream));
  conv_narrow_wgrad_kernel<<<grid, 128, 0, stream>>>(x, N, H, W, C, g, work, OH, OW, KH, KW, stride, pad, R, pps);
  int rc = (int)cudaGetLastError();
  if (grid.y > 1) {
    if (!rc) rc = og_split_sum(work, (long long)R * 8, (int)grid.y, dw_packed, stream);
    const cudaError_t e = cudaFreeAsync(work, stream);
    if (!rc) rc = (int)e;
  }
  return rc;
}
