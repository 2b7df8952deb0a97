// Shared device/host helpers for the objgan_b200 kernels (sm_90a).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <math.h>

#define OG_API extern "C" __attribute__((visibility("default")))

// Every launcher returns 0 on success, else the cudaError_t of the failed launch.
// (The reference's launcher calls exit(-1) on failure -- roi_align_kernel.cu:84-88; we never do.)
#define OG_RETURN_LAST_ERROR()                      \
  do {                                              \
    cudaError_t e__ = cudaGetLastError();           \
    return (int)e__;                                \
  } while (0)

#define OG_CHECK(call)                              \
  do {                                              \
    cudaError_t e__ = (call);                       \
    if (e__ != cudaSuccess) return (int)e__;        \
  } while (0)

static inline int og_cdiv(long long a, long long b) { return (int)((a + b - 1) / b); }

// SM count of the current device (grid sizing: waves of CTAs)
static inline int og_num_sms() {
  int dev = 0, sms = 0;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  return sms > 0 ? sms : 1;
}

// blocks of 256 threads for a grid-stride walk over total items: one per 256 items, at least one, at most per_sm per SM
static inline int og_grid(long long total, int per_sm = 32) {
  const long long b = (total + 255) / 256, cap = (long long)og_num_sms() * per_sm;
  return (int)(b < 1 ? 1 : (b > cap ? cap : b));
}

// Stream-ordered scratch memory for elems values of type T (also valid inside CUDA graph capture).  The device's
// default pool keeps what is freed for the next call instead of returning it to the driver at every synchronisation.
template <typename T>
static inline cudaError_t og_work_alloc(T** p, size_t elems, cudaStream_t stream) {
  static bool pool_ready = false;
  if (!pool_ready) {
    int dev = 0;
    cudaMemPool_t pool;
    cudaGetDevice(&dev);
    if (cudaDeviceGetDefaultMemPool(&pool, dev) == cudaSuccess) {
      uint64_t keep = UINT64_MAX;
      cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &keep);
    }
    pool_ready = true;
  }
  return cudaMallocAsync(reinterpret_cast<void**>(p), elems * sizeof(T), stream);
}

// Deterministic split reductions: the S CTAs that share an output write their partial sums to S planes of a
// workspace, and this kernel adds them in the fixed order s = 0, 1, ... (fp32 atomics would add them in whatever
// order the CTAs finish, so results would change from run to run).  out[i] = sum_s work[s * plane + i].
static __global__ void __launch_bounds__(256) og_split_sum_kernel(const float* __restrict__ work, long long plane,
                                                                  int S, float* __restrict__ out) {
  for (long long i = blockIdx.x * 256LL + threadIdx.x; i < plane; i += (long long)gridDim.x * 256) {
    float a = 0.f;
    for (int s = 0; s < S; ++s) a += work[s * plane + i];
    out[i] = a;
  }
}
static inline int og_split_sum(const float* work, long long plane, int S, float* out, cudaStream_t stream) {
  if (plane == 0) return 0;
  long long b = (plane + 255) / 256;
  if (b > 65535) b = 65535;
  og_split_sum_kernel<<<(int)b, 256, 0, stream>>>(work, plane, S, out);
  return (int)cudaGetLastError();
}

__device__ __forceinline__ float og_sigmoid(float x) { return 1.0f / (1.0f + expf(-x)); }

__device__ __forceinline__ float4 ldg4(const float* p) { return __ldg(reinterpret_cast<const float4*>(p)); }
__device__ __forceinline__ void st4(float* p, float4 v) { *reinterpret_cast<float4*>(p) = v; }

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ double warp_sum_d(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// The fp64 per-channel reductions (normalisation statistics and their backward, bias gradients) split the pixels over
// the CTAs of grid row blockIdx.y; each CTA stores its sums to plane blockIdx.y of a workspace, and og_plane_sum adds
// the planes in a fixed order, so the totals do not depend on which CTA finishes first.
//
// A (32, 8) block: thread (x, y) holds the partials acc[k] of channel quad q = blockIdx.x * 32 + x over its rows.  Entry
// k belongs to component (k & 7) >> 2 of channel (k >> 3) * Co + 4 q + (k & 3): NV = 4 is one component per channel, 8
// two, 16 two for each half of a GLU pair (Co apart).  The 8 rows are added in the order y = 0 .. 7 and the sums of the
// quads q < Co4 stored to plane[component * C + channel], so the plane is written in full for the block's channels and
// needs no zeroing.  Every thread of the block must call it.
template <int NV>
__device__ __forceinline__ void og_cta_channel_sums(const double (&acc)[NV], int Co4, int Co, int C, double* plane) {
  __shared__ double sh[8][32][NV];
#pragma unroll
  for (int i = 0; i < NV; ++i) sh[threadIdx.y][threadIdx.x][i] = acc[i];
  __syncthreads();
  for (int item = threadIdx.y * 32 + threadIdx.x; item < 32 * NV; item += 256) {
    const int cx = item / NV, k = item % NV;
    double a = 0;
#pragma unroll
    for (int j = 0; j < 8; ++j) a += sh[j][cx][k];
    const int q = blockIdx.x * 32 + cx;
    if (q < Co4) plane[((k & 7) >> 2) * C + (k >> 3) * Co + q * 4 + (k & 3)] = a;
  }
}

// sum[k] = sum_s p[s * stride + k * off] over S planes, for K components, taken by a whole warp: lane l adds the planes
// l, l + 32, ... in that order and warp_sum_d's shuffle tree adds the lanes, so every lane returns the same totals on
// every run.  A split can have ~1000 planes (a train-mode BatchNorm over 64 channels on an H100), too many for one
// thread to walk; the unrolled loop keeps 8 K loads of each lane in flight.
template <int K>
__device__ __forceinline__ void og_plane_sum(const double* __restrict__ p, long long off, int S, long long stride,
                                             double (&sum)[K]) {
  double a[K] = {};
#pragma unroll 8
  for (int s = threadIdx.x & 31; s < S; s += 32)
#pragma unroll
    for (int k = 0; k < K; ++k) a[k] += p[s * stride + k * off];
#pragma unroll
  for (int k = 0; k < K; ++k) sum[k] = warp_sum_d(a[k]);
}

// Per-tensor power-of-two scaling of the fp16 tensor-core operands: amax_bits = float bits of max|x| over the tensor;
// the operand stores x * 2^k with k chosen so that max|x| * 2^k lies in [2^13, 2^14) (fp16 overflows at 65504).
__host__ __device__ __forceinline__ int og_scale_exp(unsigned amax_bits) {
  amax_bits &= 0x7fffffffu;
  if (amax_bits == 0) return 0;
  int k = 13 - ((int)(amax_bits >> 23) - 127);
  return k < -110 ? -110 : (k > 110 ? 110 : k);
}
__device__ __forceinline__ float og_exp2i(int k) { return __int_as_float((k + 127) << 23); }   // |k| <= 126

// activation codes shared by conv epilogues and the act-backward kernel
enum { OG_ACT_NONE = 0, OG_ACT_LRELU = 1, OG_ACT_TANH = 2, OG_ACT_SIGMOID = 3 };
// normalisation-apply fusions
enum { OG_NA_NONE = 0, OG_NA_LRELU = 1, OG_NA_GLU = 2 };
// conv input addressing modes
enum { OG_PAD_ZERO = 0, OG_PAD_REFLECT = 1, OG_UPSAMPLE2X = 2, OG_TRANSPOSED = 3 };
