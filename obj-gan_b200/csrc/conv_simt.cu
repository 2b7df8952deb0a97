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
#include <cuda_fp16.h>

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
  float* dw;  // packed [(KH*KW*C)][K], accumulated with atomicAdd
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
// weight (re)packing between the reference's OIHW parameter layout (state_dict shapes, SURVEY 8b)
// and the kernel-native K-major matrices.
//   co_map(co) = co < split ? co : co + (splitp - split)   (GLU halves each padded to splitp)
// ---------------------------------------------------------------------------------------------
// output-major: one thread per element of the packed matrix (coalesced writes, zero padding written in place; the
// strided OIHW reads hit the same 32-byte sectors for neighbouring taps and stay in L1/L2)
// F16 = true: fp16 hi/lo operands of the tensor-core path, scaled by the power of two derived from *amax
__device__ __forceinline__ void store_hilo_f16(float v, float scale, __half* hi, __half* lo, long long o) {
  v *= scale;
  const __half h = __float2half_rn(v);
  hi[o] = h;
  lo[o] = __float2half_rn(v - __half2float(h));
}

template <bool F16>
__global__ void pack_weights_kernel(const float* __restrict__ w, int Co, int Ci, int KH, int KW, int Cip, int Kp,
                                    int split, int splitp, int transposed, void* __restrict__ out_v,
                                    void* __restrict__ out_lo_v, const unsigned* __restrict__ amax) {
  float* out = (float*)out_v;
  float scale = 1.f;
  if (F16) scale = og_exp2i(og_scale_exp(__ldg(amax)));
  const long long total = (long long)KH * KW * Cip * Kp;
  const int taps = KH * KW;
  for (long long o = blockIdx.x * (long long)blockDim.x + threadIdx.x; o < total;
       o += (long long)gridDim.x * blockDim.x) {
    int cm, ci, tap;
    if (!transposed) {            // [(tap, ci)][cm]
      cm = (int)(o % Kp);
      long long t = o / Kp;
      ci = (int)(t % Cip);
      tap = (int)(t / Cip);
    } else {                      // [(tap, cm)][ci]
      ci = (int)(o % Cip);
      long long t = o / Cip;
      cm = (int)(t % Kp);
      tap = (int)(t / Kp);
    }
    // inverse of the GLU-half padding map: cm -> co (or a padding lane)
    int co;
    if (split > 0) {
      if (cm < split) co = cm;
      else if (cm >= splitp && cm < splitp + split) co = cm - (splitp - split);
      else co = -1;
    } else {
      co = cm < Co ? cm : -1;
    }
    float v = 0.f;
    if (co >= 0 && co < Co && ci < Ci) v = __ldg(w + ((long long)co * Ci + ci) * taps + tap);
    if (F16) store_hilo_f16(v, scale, (__half*)out_v, (__half*)out_lo_v, o);
    else out[o] = v;
  }
}

__global__ void unpack_wgrad_kernel(const float* __restrict__ dw, int Co, int Ci, int KH, int KW, int Cip, int Kp,
                                    int split, int splitp, float* __restrict__ grad, int accumulate,
                                    int transposed) {
  long long total = (long long)Co * Ci * KH * KW;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    int kw = (int)(i % KW);
    long long t = i / KW;
    int kh = (int)(t % KH);
    t /= KH;
    int ci = (int)(t % Ci);
    int co = (int)(t / Ci);
    int cm = (split > 0 && co >= split) ? co + (splitp - split) : co;
    float v = transposed ? dw[((long long)(kh * KW + kw) * Kp + cm) * Cip + ci]
                         : dw[((long long)(kh * KW + kw) * Cip + ci) * Kp + cm];
    grad[i] = accumulate ? grad[i] + v : v;
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

OG_API int og_pack_weights(const float* w_oihw, int Co, int Ci, int KH, int KW, int Cip, int Kp, int split,
                           int splitp, int transposed, float* out, cudaStream_t stream) {
  long long total = (long long)KH * KW * Cip * Kp;
  int blocks = (int)((total + 255) / 256);
  if (blocks > og_num_sms() * 16) blocks = og_num_sms() * 16;
  pack_weights_kernel<false><<<blocks, 256, 0, stream>>>(w_oihw, Co, Ci, KH, KW, Cip, Kp, split, splitp, transposed,
                                                         out, nullptr, nullptr);
  OG_RETURN_LAST_ERROR();
}
// fp16 hi/lo operands for og_conv2d_tc: same matrices, scaled by 2^og_scale_exp(*amax) (amax from og_amax over w)
OG_API int og_pack_weights_f16(const float* w_oihw, int Co, int Ci, int KH, int KW, int Cip, int Kp, int split,
                               int splitp, int transposed, const unsigned* amax, void* hi, void* lo,
                               cudaStream_t stream) {
  if (!hi || !lo) return (int)cudaErrorInvalidValue;
  long long total = (long long)KH * KW * Cip * Kp;
  int blocks = (int)((total + 255) / 256);
  if (blocks > og_num_sms() * 16) blocks = og_num_sms() * 16;
  pack_weights_kernel<true><<<blocks, 256, 0, stream>>>(w_oihw, Co, Ci, KH, KW, Cip, Kp, split, splitp, transposed,
                                                        hi, lo, amax);
  OG_RETURN_LAST_ERROR();
}

OG_API int og_unpack_wgrad(const float* dw_packed, int Co, int Ci, int KH, int KW, int Cip, int Kp, int split,
                           int splitp, float* grad_oihw, int accumulate, int transposed, cudaStream_t stream) {
  long long total = (long long)Co * Ci * KH * KW;
  int blocks = (int)((total + 255) / 256);
  if (blocks > og_num_sms() * 16) blocks = og_num_sms() * 16;
  unpack_wgrad_kernel<<<blocks, 256, 0, stream>>>(dw_packed, Co, Ci, KH, KW, Cip, Kp, split, splitp, grad_oihw,
                                                  accumulate, transposed);
  OG_RETURN_LAST_ERROR();
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

// ---------------------------------------------------------------------------------------------
// nearest-2x-upsample + conv3x3 as four 2x2 "phase" convolutions on the low-resolution tensor (upBlock,
// model.py:43-49).  Output pixel (2i+p, 2j+q) reads low-res rows i + {-1,0} (p = 0) or i + {0,+1} (p = 1), and the
// three kernel rows collapse onto those two offsets, so the weights can be pre-summed:
//     Wp[p][q][a][b] = sum_{kh in Sh(p,a)} sum_{kw in Sw(q,b)} W[kh][kw]      (2.25x fewer MACs, same result up to
// fp32 rounding of the pre-sums).  Tap index t = ((p*2+q)*2+a)*2+b.  up_row(p, k) = which of the two offsets
// kernel row k falls on: p = 0: {0,1,1}, p = 1: {0,0,1}.
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ int up_row(int p, int k) { return p == 0 ? (k >= 1) : (k >= 2); }

// amax_up receives 4 * amax(w): the pre-sums of up to four taps are bounded by it, and it is the scale word the conv
// kernel is given for this operand
__global__ void pack_upsample_weights_kernel(const float* __restrict__ w, int Co, int Ci, int Cip, int Kp, int split,
                                             int splitp, int transposed, const unsigned* __restrict__ amax,
                                             unsigned* __restrict__ amax_up, __half* __restrict__ out,
                                             __half* __restrict__ out_lo) {
  long long total = (long long)16 * Co * Ci;
  const float bound = 4.f * __uint_as_float(__ldg(amax));
  const float scale = og_exp2i(og_scale_exp(__float_as_uint(bound)));
  if (blockIdx.x == 0 && threadIdx.x == 0) *amax_up = __float_as_uint(bound);
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    int ci = (int)(i % Ci);
    long long t2 = i / Ci;
    int co = (int)(t2 % Co);
    int t = (int)(t2 / Co);
    int b = t & 1, a = (t >> 1) & 1, q = (t >> 2) & 1, p = (t >> 3) & 1;
    float v = 0.f;
    for (int kh = 0; kh < 3; ++kh) {
      if (up_row(p, kh) != a) continue;
      for (int kw = 0; kw < 3; ++kw)
        if (up_row(q, kw) == b) v += w[(((long long)co * Ci + ci) * 3 + kh) * 3 + kw];
    }
    int cm = (split > 0 && co >= split) ? co + (splitp - split) : co;
    long long o = transposed ? ((long long)t * Kp + cm) * Cip + ci : ((long long)t * Cip + ci) * Kp + cm;
    store_hilo_f16(v, scale, out, out_lo, o);
  }
}
// dW[kh][kw] = sum_{p,q} dWp[p][q][up_row(p,kh)][up_row(q,kw)]   (dWp packed [16][Kp][Cip], i.e. "transposed" layout)
__global__ void unpack_upsample_wgrad_kernel(const float* __restrict__ dwp, int Co, int Ci, int Cip, int Kp, int split,
                                             int splitp, float* __restrict__ grad, int accumulate) {
  long long total = (long long)Co * Ci * 9;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    int kw = (int)(i % 3);
    long long t2 = i / 3;
    int kh = (int)(t2 % 3);
    t2 /= 3;
    int ci = (int)(t2 % Ci);
    int co = (int)(t2 / Ci);
    int cm = (split > 0 && co >= split) ? co + (splitp - split) : co;
    float v = 0.f;
    for (int p = 0; p < 2; ++p)
      for (int q = 0; q < 2; ++q) {
        int t = ((p * 2 + q) * 2 + up_row(p, kh)) * 2 + up_row(q, kw);
        v += dwp[((long long)t * Kp + cm) * Cip + ci];
      }
    grad[i] = accumulate ? grad[i] + v : v;
  }
}
OG_API int og_pack_upsample_weights(const float* w_oihw, int Co, int Ci, int Cip, int Kp, int split, int splitp,
                                    int transposed, const unsigned* amax, unsigned* amax_up, void* hi, void* lo,
                                    cudaStream_t stream) {
  if (!hi || !lo) return (int)cudaErrorInvalidValue;
  long long n = (long long)16 * Cip * Kp;
  OG_CHECK(cudaMemsetAsync(hi, 0, sizeof(__half) * n, stream));
  OG_CHECK(cudaMemsetAsync(lo, 0, sizeof(__half) * n, stream));
  long long total = (long long)16 * Co * Ci;
  int blocks = (int)((total + 255) / 256);
  if (blocks > og_num_sms() * 16) blocks = og_num_sms() * 16;
  pack_upsample_weights_kernel<<<blocks, 256, 0, stream>>>(w_oihw, Co, Ci, Cip, Kp, split, splitp, transposed, amax,
                                                           amax_up, (__half*)hi, (__half*)lo);
  OG_RETURN_LAST_ERROR();
}
OG_API int og_unpack_upsample_wgrad(const float* dwp, int Co, int Ci, int Cip, int Kp, int split, int splitp,
                                    float* grad_oihw, int accumulate, cudaStream_t stream) {
  long long total = (long long)Co * Ci * 9;
  int blocks = (int)((total + 255) / 256);
  if (blocks > og_num_sms() * 16) blocks = og_num_sms() * 16;
  unpack_upsample_wgrad_kernel<<<blocks, 256, 0, stream>>>(dwp, Co, Ci, Cip, Kp, split, splitp, grad_oihw, accumulate);
  OG_RETURN_LAST_ERROR();
}

// ---------------------------------------------------------------------------------------------------------------
// Multi-tensor weight re-packing: after an optimiser step EVERY convolution weight of a network needs its max|w| and
// its fp16 hi/lo operand matrices again (og_amax + og_pack_weights_f16 per layer and layout: ~300 tiny launches per
// training step).  These two kernels do the whole network in one launch each from a device-resident job table
// (int64 fields), a block being assigned to (job, chunk) by its index.
//   amax job : [x, n, out, block_start]                                  (blocks of 256 threads x 16 floats)
//   pack job : [w, hi, lo, amax, Co, Ci, taps, Cip, Kp, split, splitp, transposed, total, block_start]
// ---------------------------------------------------------------------------------------------------------------
namespace {
constexpr int MJ_AMAX_FIELDS = 4, MJ_PACK_FIELDS = 14, MJ_CHUNK = 4096;

__device__ __forceinline__ int mj_find(const long long* __restrict__ jobs, int njobs, int fields, int start_field,
                                       long long blk) {
  int lo = 0, hi = njobs - 1;
  while (lo < hi) {                       // last job whose block_start <= blk
    const int mid = (lo + hi + 1) >> 1;
    if (jobs[(long long)mid * fields + start_field] <= blk) lo = mid; else hi = mid - 1;
  }
  return lo;
}

__global__ void __launch_bounds__(256) amax_multi_kernel(const long long* __restrict__ jobs, int njobs) {
  const int j = mj_find(jobs, njobs, MJ_AMAX_FIELDS, 3, blockIdx.x);
  const long long* f = jobs + (long long)j * MJ_AMAX_FIELDS;
  const float* x = reinterpret_cast<const float*>(f[0]);
  const long long n = f[1];
  unsigned* out = reinterpret_cast<unsigned*>(f[2]);
  const long long base = ((long long)blockIdx.x - f[3]) * MJ_CHUNK;
  float m = 0.f;
  for (long long i = base + threadIdx.x; i < n && i < base + MJ_CHUNK; i += 256) m = fmaxf(m, fabsf(__ldg(x + i)));
  m = warp_max(m);
  __shared__ float sm[8];
  if ((threadIdx.x & 31) == 0) sm[threadIdx.x >> 5] = m;
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int k = 1; k < 8; ++k) m = fmaxf(m, sm[k]);
    atomicMax(out, __float_as_uint(m));
  }
}
__global__ void amax_zero_multi_kernel(const long long* __restrict__ jobs, int njobs) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j < njobs) *reinterpret_cast<unsigned*>(jobs[(long long)j * MJ_AMAX_FIELDS + 2]) = 0u;
}

__global__ void __launch_bounds__(256) pack_multi_kernel(const long long* __restrict__ jobs, int njobs) {
  const int j = mj_find(jobs, njobs, MJ_PACK_FIELDS, 13, blockIdx.x);
  const long long* f = jobs + (long long)j * MJ_PACK_FIELDS;
  const float* w = reinterpret_cast<const float*>(f[0]);
  __half* hi = reinterpret_cast<__half*>(f[1]);
  __half* lo = reinterpret_cast<__half*>(f[2]);
  const float scale = og_exp2i(og_scale_exp(__ldg(reinterpret_cast<const unsigned*>(f[3]))));
  const int Co = (int)f[4], Ci = (int)f[5], taps = (int)f[6], Cip = (int)f[7], Kp = (int)f[8];
  const int split = (int)f[9], splitp = (int)f[10], transposed = (int)f[11];
  const long long total = f[12];
  const long long base = ((long long)blockIdx.x - f[13]) * MJ_CHUNK;
  for (long long o = base + threadIdx.x; o < total && o < base + MJ_CHUNK; o += 256) {
    int cm, ci, tap;
    if (!transposed) {            // [(tap, ci)][cm]
      cm = (int)(o % Kp);
      const long long t = o / Kp;
      ci = (int)(t % Cip);
      tap = (int)(t / Cip);
    } else {                      // [(tap, cm)][ci]
      ci = (int)(o % Cip);
      const long long t = o / Cip;
      cm = (int)(t % Kp);
      tap = (int)(t / Kp);
    }
    int co;
    if (split > 0) {
      if (cm < split) co = cm;
      else if (cm >= splitp && cm < splitp + split) co = cm - (splitp - split);
      else co = -1;
    } else {
      co = cm < Co ? cm : -1;
    }
    float v = 0.f;
    if (co >= 0 && co < Co && ci < Ci) v = __ldg(w + ((long long)co * Ci + ci) * taps + tap);
    store_hilo_f16(v, scale, hi, lo, o);
  }
}
}  // namespace

// jobs: device table of njobs x 4 int64 (see above), total_blocks = sum of ceil(n / 4096)
OG_API int og_amax_multi(const long long* jobs, int njobs, int total_blocks, cudaStream_t stream) {
  if (njobs <= 0) return 0;
  amax_zero_multi_kernel<<<og_cdiv(njobs, 128), 128, 0, stream>>>(jobs, njobs);
  if (total_blocks > 0) amax_multi_kernel<<<total_blocks, 256, 0, stream>>>(jobs, njobs);
  OG_RETURN_LAST_ERROR();
}
// jobs: device table of njobs x 14 int64, total_blocks = sum of ceil(total / 4096)
OG_API int og_pack_weights_f16_multi(const long long* jobs, int njobs, int total_blocks, cudaStream_t stream) {
  if (njobs <= 0 || total_blocks <= 0) return 0;
  pack_multi_kernel<<<total_blocks, 256, 0, stream>>>(jobs, njobs);
  OG_RETURN_LAST_ERROR();
}
