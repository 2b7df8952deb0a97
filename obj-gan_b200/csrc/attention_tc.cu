// Grid attention forward (GlobalAttentionGeneral / ATT_NET, ref: GlobalAttention.py:83-122) on the tensor cores:
// a persistent wgmma kernel for the large maps of the hot path (Q % 128 == 0, 48 channels, L <= 32 words).
//
//   scores[q][l] = sum_c h[q][c] * src[c][l]      (128 x 48) x (48 x 32)   -> registers, staged to shared memory
//   p = softmax_l(scores) (caption mask quirk: GlobalAttention.py:108)       -> attn[b][l][q]
//   wc[q][c]     = sum_l p[q][l] * src[c][l]      (128 x 32) x (32 x 48)   -> registers, staged to shared memory
//
// Why tensor cores for a bandwidth-bound op: the two tiny GEMMs cost 1920 fp32 FMAs per query; on the CUDA cores that
// instruction stream (plus the shared-memory operand traffic it needs) bounds the kernel well below the HBM
// bandwidth.  Here the FMA work is a few small MMAs per 128 queries and the threads only move and convert data.
//
// fp32 parity: the convolution engine's error-compensated scheme (conv_tc.cu): x * 2^k = hi + lo with hi, lo fp16
// (22 mantissa bits), three products hi*hi + lo*hi + hi*lo into the fp32 accumulator.  The power of two comes from
// max|x| of the 32 rows a WARP stages (a register max + one shuffle reduction; no extra pass over the tensor, no block
// barrier: the same warp owns those rows in the softmax and undoes its factor there) resp. of the image's
// word projections; the accumulator is scaled back before the softmax / the store.  hi is the fp32 value truncated to
// 11 significant bits (one LOP3), lo the exact remainder; the only conversions are packed cvt.rn.f16x2 (no F2F).
//
// One CTA = one warpgroup = 128 threads = 128 queries per trip; thread t owns query row t in the softmax.  The MMAs
// (M = 64 per instruction: two row halves) leave the accumulator spread over the warpgroup's registers, so score
// and context rows pass through shared memory.  Per trip:
//   (1) the h tile (24 KB, contiguous) arrives through coalesced 16-byte loads issued one trip AHEAD (registers),
//       is split and stored into two K-major 128B-swizzled A tiles;                        -> MMA 1
//   (2) scores staged row-wise, softmax in registers, coalesced attn stores (lanes = adjacent queries),
//       the probabilities are split into the same two tiles (K = 32);                      -> MMA 2
//   (3) context rows staged through shared memory, written with coalesced 16-byte stores.
// CTAs are persistent over the query tiles of ONE image (the word-projection operand tiles are built once; tiles are
// dealt with a fixed stride).  70 KB of shared memory: three CTAs per SM cover each other's MMA round trips.
#include "common.cuh"
#include "operand.cuh"
#include "wgmma.cuh"
#include <stdlib.h>

namespace {

constexpr int AT_Q = 128;          // queries per tile = threads per CTA
constexpr int AT_C = 48;           // channels (idf == row stride)
constexpr int AT_LP = 32;          // words padded to the MMA N / K extent
constexpr uint32_t AT_A_BYTES = 128 * 128;            // one fp16 copy of the A tile: 128 rows x 128-byte swizzle rows
constexpr uint32_t AT_B1_BYTES = AT_LP * 128;         // src as [l][c]  (N = 32 rows, K = 48)
constexpr uint32_t AT_B2_BYTES = AT_C * 128;          // src as [c][l]  (N = 48 rows, K = 32)
constexpr int AT_SP = AT_LP + 4;                      // floats per staged score row
constexpr uint32_t AT_S_BYTES = AT_Q * AT_SP * 4;     // staged score rows
constexpr uint32_t AT_SMEM = 2 * AT_A_BYTES + 2 * AT_B1_BYTES + 2 * AT_B2_BYTES + AT_S_BYTES;   // 70 KB
constexpr int AT_STAGE_PITCH = AT_C + 4;              // floats per staged context row (conflict-free 16-byte accesses)
constexpr int AT_MAXB = 128;                          // batch sizes whose caption masks fit the bit table
constexpr int AT_PSCALE = 13;                          // probabilities enter MMA 2 as p * 2^13 (fp16 subnormals start at 7e-9)
constexpr uint32_t AT_HALF = 64 * 128;                // byte offset of the second 64-row half of an A tile
constexpr int AT_FWD_CTAS = 3, AT_BWD_CTAS = 2;       // CTAs per SM that fit the shared memory

// byte offset of element (row r, 16-bit column k) in a K-major SWIZZLE_128B tile
__device__ __forceinline__ uint32_t at_sw_off(int r, int k) {
  return (uint32_t)((r >> 3) * 1024 + (r & 7) * 128 + ((((k >> 3) ^ (r & 7)) & 7) << 4) + (k & 7) * 2);
}

// x (already scaled) = hi + lo: hi = x rounded to 11 significant bits in the fp32 domain (half an ulp added to the
// magnitude, then truncated: exact in fp16 while |x| >= 2^-14), lo = x - hi exactly (|lo| <= 2^-11 |x|)
__device__ __forceinline__ void at_hilo(float x, float& hi, float& lo) {
  hi = __uint_as_float((__float_as_uint(x) + 0x1000u) & 0xFFFFE000u);
  lo = x - hi;
}
// two floats -> packed f16x2 (first argument in the low half)
__device__ __forceinline__ uint32_t at_cvt2(float lo_el, float hi_el) {
  uint32_t r;
  asm("cvt.rn.f16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(hi_el), "f"(lo_el));
  return r;
}
__device__ __forceinline__ void at_sts16(uint32_t addr, uint32_t v) {
  asm volatile("st.shared.u16 [%0], %1;" ::"r"(addr), "h"((unsigned short)v) : "memory");
}
__device__ __forceinline__ void at_sts64(uint32_t addr, uint32_t x, uint32_t y) {
  asm volatile("st.shared.v2.b32 [%0], {%1, %2};" ::"r"(addr), "r"(x), "r"(y) : "memory");
}
__device__ __forceinline__ void at_sts128(uint32_t addr, uint32_t x, uint32_t y, uint32_t z, uint32_t w) {
  asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(addr), "r"(x), "r"(y), "r"(z), "r"(w) : "memory");
}
__device__ __forceinline__ float4 at_lds128(uint32_t addr) {
  float4 v;
  asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(addr));
  return v;
}
// max over the CTA's 128 threads (4 warps) through a 4-word shared scratch; every thread gets the result
__device__ __forceinline__ float at_cta_max(float m, float* scratch) {
  m = warp_max(m);
  if ((threadIdx.x & 31) == 0) scratch[threadIdx.x >> 5] = m;
  __syncthreads();
  m = fmaxf(fmaxf(scratch[0], scratch[1]), fmaxf(scratch[2], scratch[3]));
  return m;
}


// D (64 x N) (+)= A (64 x K) * B (K x N), three products per k-step, small terms first: lo*hi, hi*lo, hi*hi.
// a / b: {hi, lo} descriptors; a k-step advances both by KSTEP bytes (32: K-major, 2048: MN-major).
template <int N, int TA, int TB, int KS, uint32_t KSTEP>
__device__ __forceinline__ void at_issue(float (&d)[N / 2], const uint64_t (&a)[2], const uint64_t (&b)[2], uint32_t aoff) {
#pragma unroll
  for (int k = 0; k < KS; ++k) {
    const uint64_t koff = (uint64_t)((k * KSTEP) >> 4), ao = koff + (aoff >> 4);
    if constexpr (N == 32) {
      wg_mma_n32<TA, TB>(d, a[1] + ao, b[0] + koff, k > 0 ? 1 : 0);
      wg_mma_n32<TA, TB>(d, a[0] + ao, b[1] + koff, 1);
      wg_mma_n32<TA, TB>(d, a[0] + ao, b[0] + koff, 1);
    } else {
      wg_mma_n48<TA, TB>(d, a[1] + ao, b[0] + koff, k > 0 ? 1 : 0);
      wg_mma_n48<TA, TB>(d, a[0] + ao, b[1] + koff, 1);
      wg_mma_n48<TA, TB>(d, a[0] + ao, b[0] + koff, 1);
    }
  }
}
// row of accumulator element d[4i + 2h + e] of this thread inside a 64-row MMA half (column 8i + 2(lane % 4) + e)
__device__ __forceinline__ int at_frag_row(int h) { return ((threadIdx.x >> 5) & 3) * 16 + ((threadIdx.x & 31) >> 2) + 8 * h; }
__device__ __forceinline__ int at_frag_col(int i) { return 8 * i + 2 * (threadIdx.x & 3); }

// N-column accumulators of the two row halves -> rows of a shared fp32 staging area (pitch in floats), times s
template <int N>
__device__ __forceinline__ void at_stage(const float (&d)[2][N / 2], uint32_t base, int pitch, float s) {
#pragma unroll
  for (int hf = 0; hf < 2; ++hf)
#pragma unroll
    for (int i = 0; i < N / 8; ++i)
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const uint32_t a = base + (uint32_t)(((hf * 64 + at_frag_row(h)) * pitch + at_frag_col(i)) * 4);
        asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(a), "f"(d[hf][4 * i + 2 * h] * s),
                     "f"(d[hf][4 * i + 2 * h + 1] * s) : "memory");
      }
}

// word projections of image b -> the two operand layouts B1[l][c] and B2[c][l] as scaled fp16 hi / lo (zero beyond
// L), straight from registers: thread t holds word l = t & 31 of channels (t >> 5) + 4j.  Returns the scale exponent.
__device__ __forceinline__ int at_stage_src(const float* src, int b, int L, uint32_t sB1, uint32_t sB2, float* red) {
  const int t = threadIdx.x, warp = t >> 5, lane = t & 31;
  const float* sb = src + (long long)b * AT_C * L;
  const int l = lane, c0 = warp;
  float v[12];
  float m = 0.f;
#pragma unroll
  for (int j = 0; j < 12; ++j) {
    v[j] = l < L ? __ldg(sb + (c0 + 4 * j) * L + l) : 0.f;
    m = fmaxf(m, fabsf(v[j]));
  }
  m = at_cta_max(m, red);
  const int ksrc = og_scale_exp(__float_as_uint(m));
  const float s = og_exp2i(ksrc);
#pragma unroll
  for (int j = 0; j < 12; ++j) {
    const int c = c0 + 4 * j;
    float hi, lo;
    at_hilo(v[j] * s, hi, lo);
    const uint32_t pk = at_cvt2(hi, lo);             // low half = hi, high half = lo
    const uint32_t o1 = at_sw_off(l, c), o2 = at_sw_off(c, l);
    at_sts16(sB1 + o1, pk & 0xFFFFu);
    at_sts16(sB1 + AT_B1_BYTES + o1, pk >> 16);
    at_sts16(sB2 + o2, pk & 0xFFFFu);
    at_sts16(sB2 + AT_B2_BYTES + o2, pk >> 16);
  }
  return ksrc;
}

// LQ: words handled in registers (20 covers the 12..18-word captions of the hot path; 32 = the MMA extent)
//
// Thread <-> data mapping of the two coalesced passes over a tile (1536 float4 = 128 rows x 12): warp w owns rows
// [32w, 32w + 32); it walks them in four groups g of 8 rows (= 96 float4 = three warp-wide accesses j), so float4
// number 32j + lane of a group is (row r8[j], quad c8[j]) with r8 / c8 fixed per thread, and a group step is exactly
// one 1024-byte swizzle atom of the operand tile: every shared-memory offset is base[j] + g * constant.
template <int LQ>
__global__ void __launch_bounds__(AT_Q, AT_FWD_CTAS)
att_general_fwd_tc_kernel(const float* __restrict__ h, const float* __restrict__ src,
                          const unsigned char* __restrict__ mask, int B, int Q, int L, int nslots,
                          float* __restrict__ wc, float* __restrict__ attn) {
  extern __shared__ uint8_t at_smem_raw[];
  const uint32_t smem = (smem_u32(at_smem_raw) + 1023u) & ~1023u;   // shared-window address of the operand tiles
  const uint32_t sA = smem;                            // hi, lo; reused for the probabilities and the staged context
  const uint32_t sB1 = smem + 2 * AT_A_BYTES;
  const uint32_t sB2 = sB1 + 2 * AT_B1_BYTES;
  const uint32_t sS = sB2 + 2 * AT_B2_BYTES;           // staged score rows
  __shared__ float red[4];                             // CTA max scratch
  __shared__ uint32_t mbits[AT_MAXB];                  // caption masks of the batch, one bit per word

  const int t = threadIdx.x, warp = t >> 5, lane = t & 31;
  const int b = blockIdx.x / nslots, slot = blockIdx.x - b * nslots;
  const int ntiles = Q / AT_Q;

  // per-thread constants of the tile walk
  uint32_t offA[3], offS[3];
#pragma unroll
  for (int j = 0; j < 3; ++j) {
    const int f = j * 32 + lane, r8 = (f * 43691) >> 19, c8 = f - r8 * 12;        // f / 12 for f < 96
    offA[j] = (uint32_t)(warp * 4 * 1024) + at_sw_off(r8, c8 * 4);
    offS[j] = (uint32_t)(((warp * 32 + r8) * AT_STAGE_PITCH + c8 * 4) * 4);
  }
  // prefetch the first tile
  float4 hv[12];
  int qt = slot;
  {
    const float4* hp = reinterpret_cast<const float4*>(h + ((long long)b * Q + (long long)qt * AT_Q) * AT_C) + warp * 384 + lane;
#pragma unroll
    for (int i = 0; i < 12; ++i) hv[i] = __ldg(hp + i * 32);
  }
  if (mask && t < B) {
    uint32_t w = 0;
    for (int i = 0; i < L; ++i) w |= (mask[t * L + i] ? 1u : 0u) << i;
    mbits[t] = w;
  }
  const int ksrc = at_stage_src(src, b, L, sB1, sB2, red);
  __syncthreads();

  uint64_t dA[2], dB1[2], dB2[2];
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    dA[i] = wg_desc_k(sA + i * AT_A_BYTES);
    dB1[i] = wg_desc_k(sB1 + i * AT_B1_BYTES);
    dB2[i] = wg_desc_k(sB2 + i * AT_B2_BYTES);
  }
  const uint32_t rowP = sA + (uint32_t)((t >> 3) * 1024 + (t & 7) * 128);   // row t of an A tile; chunk ch at ((ch ^ (t & 7)) << 4)
  const uint32_t rowSc = sS + (uint32_t)(t * AT_SP * 4);
  const float so = og_exp2i(-AT_PSCALE) * og_exp2i(-ksrc);                   // context rows: undo both operand scales
  const float ss2 = og_exp2i(-ksrc);
  // caption-mask row of query (b, q): sample (b * Q + q) mod B (ref: GlobalAttention.py:108); advanced incrementally
  uint32_t mrow = ((uint32_t)b * (uint32_t)Q + (uint32_t)(qt * AT_Q + t)) % (uint32_t)B;
  const uint32_t mstep = ((uint32_t)nslots * AT_Q) % (uint32_t)B;

  for (; qt < ntiles; qt += nslots) {
    const int q0 = qt * AT_Q;
    // ---------------- (1) scale by a power of two, split into the two A copies ----------------
    // The scale is per WARP: warp w stages rows [32w, 32w + 32) here and owns the same rows in the softmax, where it
    // divides its scores by its own factor again -- a row scale of A is a row scale of A.B -- so a shuffle
    // reduction is enough (no block-wide barrier).
    float m = 0.f;
#pragma unroll
    for (int i = 0; i < 12; ++i) m = amax4(m, hv[i]);
    m = warp_max(m);
    const int kh = og_scale_exp(__float_as_uint(m));
    const float sh = og_exp2i(kh);
#pragma unroll
    for (int g = 0; g < 4; ++g)
#pragma unroll
      for (int j = 0; j < 3; ++j) {
        const float4 x = hv[g * 3 + j];
        float h0, l0, h1, l1, h2, l2, h3, l3;
        at_hilo(x.x * sh, h0, l0); at_hilo(x.y * sh, h1, l1);
        at_hilo(x.z * sh, h2, l2); at_hilo(x.w * sh, h3, l3);
        const uint32_t a = sA + offA[j] + g * 1024;
        at_sts64(a, at_cvt2(h0, h1), at_cvt2(h2, h3));
        at_sts64(a + AT_A_BYTES, at_cvt2(l0, l1), at_cvt2(l2, l3));
      }
    // the next tile's loads fly during the rest of this trip
    if (qt + nslots < ntiles) {
      const float4* hp = reinterpret_cast<const float4*>(h + ((long long)b * Q + (long long)(qt + nslots) * AT_Q) * AT_C) + warp * 384 + lane;
#pragma unroll
      for (int i = 0; i < 12; ++i) hv[i] = __ldg(hp + i * 32);
    }
    fence_proxy_async();
    __syncthreads();
    {
      float s[2][16];
      wg_fence();
      at_issue<32, 0, 0, AT_C / 16, 32>(s[0], dA, dB1, 0);
      at_issue<32, 0, 0, AT_C / 16, 32>(s[1], dA, dB1, AT_HALF);
      wg_commit();
      wg_wait<0>();
      wg_hold(s[0]);
      wg_hold(s[1]);
      at_stage<32>(s, sS, AT_SP, 1.f);
    }
    __syncthreads();                                     // scores staged; every warp's MMA 1 has finished with the A tiles
    // ---------------- (2) softmax over the words ----------------
    float sc[LQ];
    {
      const float ss1 = og_exp2i(-kh);
#pragma unroll
      for (int l = 0; l < LQ; l += 4) {
        const float4 v = at_lds128(rowSc + l * 4);
        sc[l] = v.x * ss1 * ss2; sc[l + 1] = v.y * ss1 * ss2; sc[l + 2] = v.z * ss1 * ss2; sc[l + 3] = v.w * ss1 * ss2;
      }
    }
    {
      // words beyond L and masked words leave the softmax (exp2(-inf) = 0)
      uint32_t dead = L >= 32 ? 0u : ~((1u << L) - 1u);
      if (mask) dead |= mbits[mrow];
      mrow += mstep;
      if (mrow >= (uint32_t)B) mrow -= (uint32_t)B;
      float mx = -INFINITY;
#pragma unroll
      for (int l = 0; l < LQ; ++l) {
        if ((dead >> l) & 1u) sc[l] = -INFINITY;
        mx = fmaxf(mx, sc[l]);
      }
      float sum = 0.f;
#pragma unroll
      for (int l = 0; l < LQ; ++l) {
        sc[l] = exp2f((sc[l] - mx) * 1.4426950408889634f);
        sum += sc[l];
      }
      const float inv = 1.f / sum;
      float* arow = attn + (long long)b * L * Q + (q0 + t);
#pragma unroll
      for (int l = 0; l < LQ; ++l) {
        sc[l] *= inv;
        if (l < L) *arow = sc[l];
        arow += Q;
      }
    }
    // probabilities * 2^13 -> the two A copies (row t, K = 32: four 16-byte chunks per copy; words >= LQ are zeros)
#pragma unroll
    for (int ch = 0; ch < 4; ++ch) {
      uint32_t yh[4], yl[4];
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int l0 = ch * 8 + 2 * e;
        float ha = 0.f, la = 0.f, hb = 0.f, lb = 0.f;
        if (l0 < LQ) at_hilo(sc[l0 < LQ ? l0 : 0] * (float)(1 << AT_PSCALE), ha, la);
        if (l0 + 1 < LQ) at_hilo(sc[l0 + 1 < LQ ? l0 + 1 : 0] * (float)(1 << AT_PSCALE), hb, lb);
        yh[e] = at_cvt2(ha, hb);
        yl[e] = at_cvt2(la, lb);
      }
      const uint32_t addr = rowP + (uint32_t)(((ch ^ (t & 7)) & 7) << 4);
      at_sts128(addr, yh[0], yh[1], yh[2], yh[3]);
      at_sts128(addr + AT_A_BYTES, yl[0], yl[1], yl[2], yl[3]);
    }
    fence_proxy_async();
    __syncthreads();
    // ---------------- (3) context rows: registers -> shared staging -> coalesced stores ----------------
    {
      float o[2][24];
      wg_fence();
      at_issue<48, 0, 0, AT_LP / 16, 32>(o[0], dA, dB2, 0);
      at_issue<48, 0, 0, AT_LP / 16, 32>(o[1], dA, dB2, AT_HALF);
      wg_commit();
      wg_wait<0>();
      wg_hold(o[0]);
      wg_hold(o[1]);
      __syncthreads();                                   // MMA 2 has completed in every warp: the A copies are free
      at_stage<48>(o, sA, AT_STAGE_PITCH, so);
    }
    __syncthreads();
    {
      float4* op = reinterpret_cast<float4*>(wc + ((long long)b * Q + q0) * AT_C) + warp * 384 + lane;
#pragma unroll
      for (int g = 0; g < 4; ++g)
#pragma unroll
        for (int j = 0; j < 3; ++j)
          op[g * 96 + j * 32] = at_lds128(sA + offS[j] + (uint32_t)(g * 8 * AT_STAGE_PITCH * 4));
    }
    __syncthreads();                                     // staging drained before the next trip overwrites the A copies
  }
}

// ------------------------------------------------------------------------------------------------
// Backward (the attention maps are only visualised, so they carry no gradient).  Per query q:
//   gP[l]   = sum_c g_wc[q][c] src[c][l]                          MMA 1:  Gw (128 x 48)   . B1
//   gS[l]   = P[l] (gP[l] - sum_l' P[l'] gP[l'])                  registers (P read from the saved attention map)
//   g_h[c]  = sum_l gS[l] src[c][l]                               MMA 2:  gS (128 x 32)   . B2
//   g_src[c][l] += sum_q g_wc[q][c] P[q][l] + h[q][c] gS[q][l]    MMA 3a: Gw^T . P, 3b: H^T . gS  (contraction over the
//       tile's 128 queries: the SAME shared-memory tiles read as MN-major operands, M = 64 channels of which 48 are
//       real, k-step = 16 rows = 2048 bytes)
// The two g_src terms carry different operand scales, so each tile's pair of 64 x 32 results is rescaled and summed
// into register accumulators that persist over the CTA's tiles; each CTA stores its share of g_src to a workspace
// plane at the end, and the planes are added in a fixed order (og_split_sum).
// Shared memory: X = {Gw, then H} hi / lo, Y = {P, then gS} hi / lo, B1, B2, staged rows: 102 KB, two CTAs per SM.
// ------------------------------------------------------------------------------------------------
// two CTA-wide maxima at once
__device__ __forceinline__ void at_cta_max2(float& m0, float& m1, float (*scratch)[4]) {
  m0 = warp_max(m0);
  m1 = warp_max(m1);
  if ((threadIdx.x & 31) == 0) { scratch[0][threadIdx.x >> 5] = m0; scratch[1][threadIdx.x >> 5] = m1; }
  __syncthreads();
  m0 = fmaxf(fmaxf(scratch[0][0], scratch[0][1]), fmaxf(scratch[0][2], scratch[0][3]));
  m1 = fmaxf(fmaxf(scratch[1][0], scratch[1][1]), fmaxf(scratch[1][2], scratch[1][3]));
}

template <int LQ>
__global__ void __launch_bounds__(AT_Q, AT_BWD_CTAS)
att_general_bwd_tc_kernel(const float* __restrict__ h, const float* __restrict__ src, const float* __restrict__ attn,
                          const float* __restrict__ g_wc, int B, int Q, int L, int nslots, float* __restrict__ g_h,
                          float* __restrict__ g_src) {
  extern __shared__ uint8_t at_smem_raw[];
  const uint32_t smem = (smem_u32(at_smem_raw) + 1023u) & ~1023u;
  const uint32_t sX = smem;                            // Gw, then H (hi, lo); finally the staged g_h rows
  const uint32_t sY = smem + 2 * AT_A_BYTES;           // P, then gS (hi, lo)
  const uint32_t sB1 = sY + 2 * AT_A_BYTES;
  const uint32_t sB2 = sB1 + 2 * AT_B1_BYTES;
  const uint32_t sS = sB2 + 2 * AT_B2_BYTES;           // staged gP rows
  __shared__ float red[4][4];

  const int t = threadIdx.x, warp = t >> 5, lane = t & 31;
  const int b = blockIdx.x / nslots, slot = blockIdx.x - b * nslots;
  const int ntiles = Q / AT_Q;

  uint32_t offA[3], offS[3];
#pragma unroll
  for (int j = 0; j < 3; ++j) {
    const int f = j * 32 + lane, r8 = (f * 43691) >> 19, c8 = f - r8 * 12;
    offA[j] = (uint32_t)(warp * 4 * 1024) + at_sw_off(r8, c8 * 4);
    offS[j] = (uint32_t)(((warp * 32 + r8) * AT_STAGE_PITCH + c8 * 4) * 4);
  }
  const int ksrc = at_stage_src(src, b, L, sB1, sB2, red[0]);
  __syncthreads();

  uint64_t dX[2], dY[2], dB1[2], dB2[2], dXmn[2], dYmn[2];
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    dX[i] = wg_desc_k(sX + i * AT_A_BYTES);
    dY[i] = wg_desc_k(sY + i * AT_A_BYTES);
    dB1[i] = wg_desc_k(sB1 + i * AT_B1_BYTES);
    dB2[i] = wg_desc_k(sB2 + i * AT_B2_BYTES);
    dXmn[i] = wg_desc(sX + i * AT_A_BYTES, AT_A_BYTES, 1024);
    dYmn[i] = wg_desc(sY + i * AT_A_BYTES, AT_A_BYTES, 1024);
  }
  const uint32_t rowY = sY + (uint32_t)((t >> 3) * 1024 + (t & 7) * 128);
  const uint32_t rowSc = sS + (uint32_t)(t * AT_SP * 4);
  const float ss2 = og_exp2i(-ksrc);

  float gacc[16];                                      // g_src[c][l] fragment (rows c = channels), over this CTA's tiles
#pragma unroll
  for (int i = 0; i < 16; ++i) gacc[i] = 0.f;

  // g_wc rows and the saved probabilities of a tile are loaded one tile AHEAD (into the registers the current tile has
  // finished with); h is loaded at the top of its own tile (it is needed last)
  float4 gw[12];
  float pr[LQ];
  auto load_gw = [&](int tileq) {
    const float4* gp = reinterpret_cast<const float4*>(g_wc + ((long long)b * Q + (long long)tileq * AT_Q) * AT_C) + warp * 384 + lane;
#pragma unroll
    for (int i = 0; i < 12; ++i) gw[i] = __ldg(gp + i * 32);
  };
  auto load_pr = [&](int tileq) {
    const float* arow = attn + (long long)b * L * Q + ((long long)tileq * AT_Q + t);
#pragma unroll
    for (int l = 0; l < LQ; ++l) {
      pr[l] = l < L ? __ldg(arow) : 0.f;
      arow += Q;
    }
  };
  if (slot < ntiles) {
    load_gw(slot);
    load_pr(slot);
  }
  for (int qt = slot; qt < ntiles; qt += nslots) {
    const int q0 = qt * AT_Q;
    const long long tile = ((long long)b * Q + q0) * AT_C;
    float4 hh[12];
    {
      const float4* hp = reinterpret_cast<const float4*>(h + tile) + warp * 384 + lane;
#pragma unroll
      for (int i = 0; i < 12; ++i) hh[i] = __ldg(hp + i * 32);
    }
    float prc[LQ];                                     // this tile's probabilities (pr is refilled below)
#pragma unroll
    for (int l = 0; l < LQ; ++l) prc[l] = pr[l];
    // ---- (1) Gw -> X, P -> Y ----
    float mg = 0.f, mh = 0.f;
#pragma unroll
    for (int i = 0; i < 12; ++i) { mg = amax4(mg, gw[i]); mh = amax4(mh, hh[i]); }
    at_cta_max2(mg, mh, red + 1);
    const int kg = og_scale_exp(__float_as_uint(mg)), kh = og_scale_exp(__float_as_uint(mh));
    {
      const float sg = og_exp2i(kg);
#pragma unroll
      for (int g = 0; g < 4; ++g)
#pragma unroll
        for (int j = 0; j < 3; ++j) {
          const float4 x = gw[g * 3 + j];
          float h0, l0, h1, l1, h2, l2, h3, l3;
          at_hilo(x.x * sg, h0, l0); at_hilo(x.y * sg, h1, l1);
          at_hilo(x.z * sg, h2, l2); at_hilo(x.w * sg, h3, l3);
          const uint32_t a = sX + offA[j] + g * 1024;
          at_sts64(a, at_cvt2(h0, h1), at_cvt2(h2, h3));
          at_sts64(a + AT_A_BYTES, at_cvt2(l0, l1), at_cvt2(l2, l3));
        }
    }
#pragma unroll
    for (int ch = 0; ch < 4; ++ch) {
      uint32_t yh[4], yl[4];
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int l0 = ch * 8 + 2 * e;
        float ha = 0.f, la = 0.f, hb = 0.f, lb = 0.f;
        if (l0 < LQ) at_hilo(prc[l0 < LQ ? l0 : 0] * (float)(1 << AT_PSCALE), ha, la);
        if (l0 + 1 < LQ) at_hilo(prc[l0 + 1 < LQ ? l0 + 1 : 0] * (float)(1 << AT_PSCALE), hb, lb);
        yh[e] = at_cvt2(ha, hb);
        yl[e] = at_cvt2(la, lb);
      }
      const uint32_t addr = rowY + (uint32_t)(((ch ^ (t & 7)) & 7) << 4);
      at_sts128(addr, yh[0], yh[1], yh[2], yh[3]);
      at_sts128(addr + AT_A_BYTES, yl[0], yl[1], yl[2], yl[3]);
    }
    if (qt + nslots < ntiles) {                        // gw and pr are dead from here on: next tile's loads
      load_gw(qt + nslots);
      load_pr(qt + nslots);
    }
    fence_proxy_async();
    __syncthreads();
    {
      float gp[2][16], d3[16];
      wg_fence();
      at_issue<32, 0, 0, AT_C / 16, 32>(gp[0], dX, dB1, 0);           // gP
      at_issue<32, 0, 0, AT_C / 16, 32>(gp[1], dX, dB1, AT_HALF);
      at_issue<32, 1, 1, AT_Q / 16, 2048>(d3, dXmn, dYmn, 0);          // Gw^T . P
      wg_commit();
      wg_wait<0>();
      wg_hold(gp[0]);
      wg_hold(gp[1]);
      wg_hold(d3);
      at_stage<32>(gp, sS, AT_SP, 1.f);
      // first g_src term of this tile: acc * 2^-(kg + 13)
      const float s3a = og_exp2i(-kg), s3b = og_exp2i(-AT_PSCALE);      // two factors: their product may underflow
#pragma unroll
      for (int i = 0; i < 16; ++i) gacc[i] = fmaf(d3[i] * s3a, s3b, gacc[i]);
    }
    __syncthreads();
    // ---- (2) softmax backward in registers ----
    float gs[LQ];
    {
      const float s1 = og_exp2i(-kg);
#pragma unroll
      for (int l = 0; l < LQ; l += 4) {
        const float4 v = at_lds128(rowSc + l * 4);
        gs[l] = v.x * s1 * ss2; gs[l + 1] = v.y * s1 * ss2; gs[l + 2] = v.z * s1 * ss2; gs[l + 3] = v.w * s1 * ss2;
      }
      float dot = 0.f;
#pragma unroll
      for (int l = 0; l < LQ; ++l) dot = fmaf(prc[l], gs[l], dot);
      float mgs = 0.f;
#pragma unroll
      for (int l = 0; l < LQ; ++l) {
        gs[l] = prc[l] * (gs[l] - dot);
        mgs = fmaxf(mgs, fabsf(gs[l]));
      }
      mgs = at_cta_max(mgs, red[3]);
      const int ks = og_scale_exp(__float_as_uint(mgs));
      const float sgs = og_exp2i(ks), shh = og_exp2i(kh);
      // ---- (3) gS -> Y, H -> X (MMA 1 / 3a have completed in every warp: both regions are free) ----
#pragma unroll
      for (int ch = 0; ch < 4; ++ch) {
        uint32_t yh[4], yl[4];
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const int l0 = ch * 8 + 2 * e;
          float ha = 0.f, la = 0.f, hb = 0.f, lb = 0.f;
          if (l0 < LQ) at_hilo(gs[l0 < LQ ? l0 : 0] * sgs, ha, la);
          if (l0 + 1 < LQ) at_hilo(gs[l0 + 1 < LQ ? l0 + 1 : 0] * sgs, hb, lb);
          yh[e] = at_cvt2(ha, hb);
          yl[e] = at_cvt2(la, lb);
        }
        const uint32_t addr = rowY + (uint32_t)(((ch ^ (t & 7)) & 7) << 4);
        at_sts128(addr, yh[0], yh[1], yh[2], yh[3]);
        at_sts128(addr + AT_A_BYTES, yl[0], yl[1], yl[2], yl[3]);
      }
#pragma unroll
      for (int g = 0; g < 4; ++g)
#pragma unroll
        for (int j = 0; j < 3; ++j) {
          const float4 x = hh[g * 3 + j];
          float h0, l0, h1, l1, h2, l2, h3, l3;
          at_hilo(x.x * shh, h0, l0); at_hilo(x.y * shh, h1, l1);
          at_hilo(x.z * shh, h2, l2); at_hilo(x.w * shh, h3, l3);
          const uint32_t a = sX + offA[j] + g * 1024;
          at_sts64(a, at_cvt2(h0, h1), at_cvt2(h2, h3));
          at_sts64(a + AT_A_BYTES, at_cvt2(l0, l1), at_cvt2(l2, l3));
        }
      fence_proxy_async();
      __syncthreads();
      // ---- (4) g_h rows and the second g_src term ----
      float o[2][24], d3[16];
      wg_fence();
      at_issue<48, 0, 0, AT_LP / 16, 32>(o[0], dY, dB2, 0);           // g_h
      at_issue<48, 0, 0, AT_LP / 16, 32>(o[1], dY, dB2, AT_HALF);
      at_issue<32, 1, 1, AT_Q / 16, 2048>(d3, dXmn, dYmn, 0);          // H^T . gS
      wg_commit();
      wg_wait<0>();
      wg_hold(o[0]);
      wg_hold(o[1]);
      wg_hold(d3);
      const float s3a = og_exp2i(-kh), s3b = og_exp2i(-ks);
#pragma unroll
      for (int i = 0; i < 16; ++i) gacc[i] = fmaf(d3[i] * s3a, s3b, gacc[i]);
      __syncthreads();                                 // MMA 2 / 3b have completed in every warp: X takes the staging
      at_stage<48>(o, sX, AT_STAGE_PITCH, og_exp2i(-ks) * ss2);
    }
    __syncthreads();
    {
      float4* op = reinterpret_cast<float4*>(g_h + tile) + warp * 384 + lane;
#pragma unroll
      for (int g = 0; g < 4; ++g)
#pragma unroll
        for (int j = 0; j < 3; ++j)
          op[g * 96 + j * 32] = at_lds128(sX + offS[j] + (uint32_t)(g * 8 * AT_STAGE_PITCH * 4));
    }
    __syncthreads();
  }
  // this CTA's share of g_src: plane (slot, b) of the workspace, summed over the slots in a fixed order afterwards
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int hh = 0; hh < 2; ++hh)
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int c = at_frag_row(hh), l = at_frag_col(i) + e;
        if (c < AT_C && l < L) g_src[(((long long)slot * B + b) * AT_C + c) * L + l] = gacc[4 * i + 2 * hh + e];
      }
}

}  // namespace

// Returns 0 when the tensor-core kernel ran, -1 when the shape is outside its envelope (the caller then uses the SIMT
// kernels of attention.cu), else a cudaError_t.
extern "C" int og_att_general_fwd_tc(const float* h, const float* src, const unsigned char* mask, int B, int Q, int idf,
                                     int cs, int L, float* wc, float* attn, cudaStream_t stream) {
  if (idf != AT_C || cs != AT_C || L < 1 || L > AT_LP || Q % AT_Q != 0 || Q < AT_Q || B < 1 ||
      (long long)B * Q >= (1LL << 31) || B > AT_MAXB)
    return -1;
  const int ntiles = Q / AT_Q;
  int nslots = (AT_FWD_CTAS * og_num_sms()) / B;       // every CTA stays inside one image
  if (nslots < 1) nslots = 1;
  if (nslots > ntiles) nslots = ntiles;
  const size_t smem = AT_SMEM + 1024;
  static bool configured = false;
  if (!configured) {
    OG_CHECK(cudaFuncSetAttribute(att_general_fwd_tc_kernel<20>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    OG_CHECK(cudaFuncSetAttribute(att_general_fwd_tc_kernel<32>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    configured = true;
  }
  if (L <= 20)
    att_general_fwd_tc_kernel<20><<<B * nslots, AT_Q, smem, stream>>>(h, src, mask, B, Q, L, nslots, wc, attn);
  else
    att_general_fwd_tc_kernel<32><<<B * nslots, AT_Q, smem, stream>>>(h, src, mask, B, Q, L, nslots, wc, attn);
  OG_RETURN_LAST_ERROR();
}

// Backward on the tensor cores; g_src is overwritten.  Same return convention.
extern "C" int og_att_general_bwd_tc(const float* h, const float* src, const float* attn, const float* g_wc, int B, int Q,
                                     int idf, int cs, int L, float* g_h, float* g_src, cudaStream_t stream) {
  if (idf != AT_C || cs != AT_C || L < 1 || L > AT_LP || Q % AT_Q != 0 || Q < AT_Q || B < 1) return -1;
  const int ntiles = Q / AT_Q;
  int nslots = (AT_BWD_CTAS * og_num_sms()) / B;
  if (nslots < 1) nslots = 1;
  if (nslots > ntiles) nslots = ntiles;
  const size_t smem = 4 * AT_A_BYTES + 2 * AT_B1_BYTES + 2 * AT_B2_BYTES + AT_S_BYTES + 1024;
  static bool configured = false;
  if (!configured) {
    OG_CHECK(cudaFuncSetAttribute(att_general_bwd_tc_kernel<20>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    OG_CHECK(cudaFuncSetAttribute(att_general_bwd_tc_kernel<32>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    configured = true;
  }
  float* work = g_src;
  if (nslots > 1) OG_CHECK(og_work_alloc(&work, (size_t)nslots * B * AT_C * L, stream));
  if (L <= 20)
    att_general_bwd_tc_kernel<20><<<B * nslots, AT_Q, smem, stream>>>(h, src, attn, g_wc, B, Q, L, nslots, g_h, work);
  else
    att_general_bwd_tc_kernel<32><<<B * nslots, AT_Q, smem, stream>>>(h, src, attn, g_wc, B, Q, L, nslots, g_h, work);
  int rc = (int)cudaGetLastError();
  if (nslots > 1) {
    if (!rc) rc = og_split_sum(work, (long long)B * AT_C * L, nslots, g_src, stream);
    const cudaError_t e = cudaFreeAsync(work, stream);
    if (!rc) rc = (int)e;
  }
  return rc;
}
