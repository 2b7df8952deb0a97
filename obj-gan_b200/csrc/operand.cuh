// The fp16 hi/lo operand format of the tensor-core convolutions, and the device helpers every writer of it uses
// (operands.cu, norm.cu).  A tensor x is stored as x * 2^k split into
//     hi = fp16(x * 2^k),   lo = fp16(x * 2^k - hi)        (22 significant bits; the kernels add three products)
// with k = og_scale_exp(word) and word = the float bits of max|x|, or of any upper bound of it: the word only positions
// the 22-bit window.
#pragma once
#include <cuda_fp16.h>

#include "common.cuh"

// the power of two a scale word selects
__device__ __forceinline__ float og_operand_scale(unsigned word) { return og_exp2i(og_scale_exp(word)); }

__device__ __forceinline__ void og_encode(float v, float scale, __half& hi, __half& lo) {
  v *= scale;
  hi = __float2half_rn(v);
  lo = __float2half_rn(v - __half2float(hi));
}

// eight consecutive channels of an NHWC tensor: element i of the 8-lane walk, two 16-byte stores per copy
__device__ __forceinline__ void og_encode8_store(const float (&v)[8], float scale, __half* __restrict__ xh,
                                                 __half* __restrict__ xl, long long i) {
  __align__(16) __half hi[8], lo[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) og_encode(v[j], scale, hi[j], lo[j]);
  *reinterpret_cast<uint4*>(xh + i * 8) = *reinterpret_cast<const uint4*>(hi);
  *reinterpret_cast<uint4*>(xl + i * 8) = *reinterpret_cast<const uint4*>(lo);
}

// nn.ReflectionPad2d(1): the source index of a coordinate at most one step outside [0, n)
__device__ __forceinline__ int og_reflect(int i, int n) {
  if (i < 0) i = -i;
  if (i >= n) i = 2 * n - 2 - i;
  return i;
}

// max|x| reductions: as float bits, non-negative floats order like unsigned integers, so atomicMax merges them
__device__ __forceinline__ float amax4(float m, const float4& o) {
  return fmaxf(fmaxf(m, fmaxf(fabsf(o.x), fabsf(o.y))), fmaxf(fabsf(o.z), fabsf(o.w)));
}
// merges the per-thread maxima m of a 256-thread block, shaped (256) or (32, 8), into *amax
__device__ __forceinline__ void block_amax_256(float m, unsigned* amax) {
  __shared__ float sm_amax[8];
  const int tid = threadIdx.y * blockDim.x + threadIdx.x;
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

// Element o of a packed weight matrix, [(tap, ci)][cm] or, transposed, [(tap, cm)][ci] (Cip x Kp per tap), to the
// offset of its source in the OIHW parameter [Co][Ci][taps], or -1 for a padding lane.  cm = co, except that with a GLU
// split the second half co >= split moves to cm = co + (splitp - split), each half padded to splitp.
__device__ __forceinline__ long long og_pack_source(long long o, int Co, int Ci, int taps, int Cip, int Kp, int split,
                                                    int splitp, int transposed) {
  int cm, ci, tap;
  if (!transposed) {
    cm = (int)(o % Kp);
    const long long t = o / Kp;
    ci = (int)(t % Cip);
    tap = (int)(t / Cip);
  } else {
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
  if (co < 0 || co >= Co || ci >= Ci) return -1;
  return ((long long)co * Ci + ci) * taps + tap;
}
