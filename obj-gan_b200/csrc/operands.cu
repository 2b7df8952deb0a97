// Producers of the tensor-core convolutions' operands (the format: operand.cuh), and the weight layouts of both
// convolution engines:
//   * og_amax: the scale word max|x| of a tensor;
//   * og_prep_split / og_prep_split_s2d: the fp16 hi / lo copies of an NHWC activation, plain, with the reflection
//     halo, or as four space-to-depth phase blocks;
//   * og_pack_weights (fp32, CUDA-core engine) / og_pack_weights_f16: OIHW parameters to the kernel-native K-major
//     matrices, og_unpack_wgrad back; og_pack_upsample_weights / og_unpack_upsample_wgrad: the pre-summed 2x2 phase
//     weights of nearest-2x-upsample + conv3x3;
//   * og_amax_multi + og_pack_weights_f16_multi: og_amax + og_pack_weights_f16 for every weight of a network in two
//     launches.
// (og_norm_apply_split in norm.cu writes the same copies from inside the normalisation pass.)
#include "operand.cuh"

// max|x| over a tensor as float bits
__global__ void __launch_bounds__(256) amax_kernel(const float* __restrict__ x, long long n4, int tail,
                                                   unsigned* __restrict__ out) {
  float m = 0.f;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n4; i += (long long)gridDim.x * blockDim.x)
    m = amax4(m, ldg4(x + i * 4));
  if (blockIdx.x == 0 && (int)threadIdx.x < tail) m = fmaxf(m, fabsf(x[n4 * 4 + threadIdx.x]));
  block_amax_256(m, out);
}

// output: [N][H+2p][W+2p][C] or, for s2d, [4][N][ceil(H/2)][ceil(W/2)][C] with phase block (a*2+b) = x[:, a::2, b::2],
// the row / column past an odd edge zero
__global__ void __launch_bounds__(256) prep_split_kernel(const float* __restrict__ x, int N, int H, int W, int C8, int pad,
                                                         int s2d, long long total, const unsigned* __restrict__ amax,
                                                         __half* __restrict__ xh, __half* __restrict__ xl) {
  const int Hp = s2d ? (H + 1) / 2 : H + 2 * pad, Wp = s2d ? (W + 1) / 2 : W + 2 * pad;
  const float scale = og_operand_scale(__ldg(amax));
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    int c = (int)(i % C8);
    long long t = i / C8;
    int w = (int)(t % Wp);
    t /= Wp;
    int h = (int)(t % Hp);
    long long n = t / Hp;
    int sh, sw;
    if (s2d) {
      int ph = (int)(n / N);
      n -= (long long)ph * N;
      sh = 2 * h + (ph >> 1);
      sw = 2 * w + (ph & 1);
    } else {
      sh = og_reflect(h - pad, H);
      sw = og_reflect(w - pad, W);
    }
    float v[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    if (sh < H && sw < W) {
      const float* src = x + (((n * H + sh) * W + sw) * C8 + c) * 8;
      const float4 v0 = ldg4(src), v1 = ldg4(src + 4);
      v[0] = v0.x; v[1] = v0.y; v[2] = v0.z; v[3] = v0.w; v[4] = v1.x; v[5] = v1.y; v[6] = v1.z; v[7] = v1.w;
    }
    og_encode8_store(v, scale, xh, xl, i);
  }
}

// One packed weight matrix (og_pack_source's layouts): hi receives the fp32 matrix, or hi and lo its fp16 operand pair
struct PackJob {
  const float* w;
  void* hi;
  void* lo;
  int Co, Ci, taps, Cip, Kp, split, splitp, transposed;
};

template <bool F16>
__device__ __forceinline__ void pack_element(const PackJob& j, long long o, float scale) {
  const long long s = og_pack_source(o, j.Co, j.Ci, j.taps, j.Cip, j.Kp, j.split, j.splitp, j.transposed);
  const float v = s < 0 ? 0.f : __ldg(j.w + s);
  if (F16) {
    __half h, l;
    og_encode(v, scale, h, l);
    static_cast<__half*>(j.hi)[o] = h;
    static_cast<__half*>(j.lo)[o] = l;
  } else {
    static_cast<float*>(j.hi)[o] = v;
  }
}

// output-major: one thread per element of the packed matrix (coalesced writes, zero padding written in place; the
// strided OIHW reads hit the same 32-byte sectors for neighbouring taps and stay in L1/L2).  F16: scaled by *amax's
// power of two.
template <bool F16>
__global__ void pack_weights_kernel(PackJob j, long long total, const unsigned* __restrict__ amax) {
  const float scale = F16 ? og_operand_scale(__ldg(amax)) : 1.f;
  for (long long o = blockIdx.x * (long long)blockDim.x + threadIdx.x; o < total;
       o += (long long)gridDim.x * blockDim.x)
    pack_element<F16>(j, o, scale);
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
  const float scale = og_operand_scale(__float_as_uint(bound));
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
    __half h, l;
    og_encode(v, scale, h, l);
    out[o] = h;
    out_lo[o] = l;
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
  const long long base = ((long long)blockIdx.x - f[3]) * MJ_CHUNK;
  float m = 0.f;
  for (long long i = base + threadIdx.x; i < n && i < base + MJ_CHUNK; i += 256) m = fmaxf(m, fabsf(__ldg(x + i)));
  block_amax_256(m, reinterpret_cast<unsigned*>(f[2]));
}
__global__ void amax_zero_multi_kernel(const long long* __restrict__ jobs, int njobs) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j < njobs) *reinterpret_cast<unsigned*>(jobs[(long long)j * MJ_AMAX_FIELDS + 2]) = 0u;
}

__global__ void __launch_bounds__(256) pack_multi_kernel(const long long* __restrict__ jobs, int njobs) {
  const long long* f = jobs + (long long)mj_find(jobs, njobs, MJ_PACK_FIELDS, 13, blockIdx.x) * MJ_PACK_FIELDS;
  const PackJob j{reinterpret_cast<const float*>(f[0]), reinterpret_cast<void*>(f[1]), reinterpret_cast<void*>(f[2]),
                  (int)f[4], (int)f[5], (int)f[6], (int)f[7], (int)f[8], (int)f[9], (int)f[10], (int)f[11]};
  const float scale = og_operand_scale(__ldg(reinterpret_cast<const unsigned*>(f[3])));
  const long long total = f[12];
  const long long base = ((long long)blockIdx.x - f[13]) * MJ_CHUNK;
  for (long long o = base + threadIdx.x; o < total && o < base + MJ_CHUNK; o += 256) pack_element<true>(j, o, scale);
}
}  // namespace

// ---------------------------------------------------------------------------------------------
// C ABI
// ---------------------------------------------------------------------------------------------
// *amax = float bits of max|x[0..n)| (x 16-byte aligned); used for the weight tensors before og_pack_weights_f16
OG_API int og_amax(const float* x, long long n, unsigned* amax, cudaStream_t stream) {
  OG_CHECK(cudaMemsetAsync(amax, 0, sizeof(unsigned), stream));
  if (n == 0) return 0;
  const long long n4 = n / 4;
  amax_kernel<<<og_grid(n4, 8), 256, 0, stream>>>(x, n4, (int)(n - n4 * 4), amax);
  OG_RETURN_LAST_ERROR();
}

// fp16 hi/lo operand copies of an NHWC fp32 tensor, scaled by the power of two that og_scale_exp derives from
// max|x| (*amax as float bits: computed here, or, with amax_ready, left there by the kernel that produced x --
// any upper bound of max|x| is valid, it only positions the 22-bit window).  pad = 0: plain; pad = 1: nn.ReflectionPad2d(1) halo (model.py:67)
// materialised while splitting; s2d = 1: four space-to-depth phase blocks.
OG_API int og_prep_split(const float* x, int N, int H, int W, int C, int pad, int s2d, unsigned* amax, int amax_ready,
                         void* xh, void* xl, cudaStream_t stream) {
  if (!xh || !xl || C % 8 || pad < 0 || pad > 1 || (s2d && (pad || (H & 1) || (W & 1)))) return (int)cudaErrorInvalidValue;
  const long long n4 = (long long)N * H * W * C / 4;
  if (!amax_ready) OG_CHECK(cudaMemsetAsync(amax, 0, sizeof(unsigned), stream));
  if (n4 == 0) return 0;
  if (!amax_ready)        // the producer of x did not leave max|x| behind: one extra read pass
    amax_kernel<<<og_grid(n4, 8), 256, 0, stream>>>(x, n4, 0, amax);
  long long total = s2d ? (long long)N * H * W * (C / 8) : (long long)N * (H + 2 * pad) * (W + 2 * pad) * (C / 8);
  prep_split_kernel<<<og_grid(total), 256, 0, stream>>>(x, N, H, W, C / 8, pad, s2d, total, amax, (__half*)xh, (__half*)xl);
  OG_RETURN_LAST_ERROR();
}

// og_prep_split(s2d=1) at any H, W: xh / xl [4N][ceil(H/2)][ceil(W/2)][C]; *amax as in og_prep_split
OG_API int og_prep_split_s2d(const float* x, int N, int H, int W, int C, unsigned* amax, int amax_ready, void* xh,
                             void* xl, cudaStream_t stream) {
  if (!xh || !xl || C % 8) return (int)cudaErrorInvalidValue;
  if (!amax_ready) {
    const int rc = og_amax(x, (long long)N * H * W * C, amax, stream);
    if (rc) return rc;
  }
  const long long total = 4LL * N * ((H + 1) / 2) * ((W + 1) / 2) * (C / 8);
  if (total == 0) return 0;
  prep_split_kernel<<<og_grid(total), 256, 0, stream>>>(x, N, H, W, C / 8, 0, 1, total, amax, (__half*)xh, (__half*)xl);
  OG_RETURN_LAST_ERROR();
}

OG_API int og_pack_weights(const float* w_oihw, int Co, int Ci, int KH, int KW, int Cip, int Kp, int split,
                           int splitp, int transposed, float* out, cudaStream_t stream) {
  long long total = (long long)KH * KW * Cip * Kp;
  int blocks = (int)((total + 255) / 256);
  if (blocks > og_num_sms() * 16) blocks = og_num_sms() * 16;
  pack_weights_kernel<false><<<blocks, 256, 0, stream>>>(
      PackJob{w_oihw, out, nullptr, Co, Ci, KH * KW, Cip, Kp, split, splitp, transposed}, total, nullptr);
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
  pack_weights_kernel<true><<<blocks, 256, 0, stream>>>(
      PackJob{w_oihw, hi, lo, Co, Ci, KH * KW, Cip, Kp, split, splitp, transposed}, total, amax);
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
