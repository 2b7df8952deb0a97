// Tensor-core implicit-GEMM convolution for sm_90a: wgmma (m64nNk16, fp16 inputs, fp32 register accumulators),
// operands staged by TMA (cp.async.bulk.tensor, 128-byte swizzle), mbarrier producer/consumer pipeline.
//
// Covers every stride-1 contraction of the hot path through a "tap list":
//     out[pix, :] = sum_t  src[pix + (dh_t, dw_t), :] * W[widx_t]          (src out-of-bounds = 0 via TMA fill)
// which is the forward of the reflection-padded 3x3 convs of HmapResBlock (model.py:63-81; the halo is
// materialised by og_prep_split), the zero-padded 3x3 convs (model.py:36-39, 1020-1048), their input
// gradients (taps mirrored, operand re-packed) and the four phases of nearest-2x-upsample + conv3x3
// (upBlock, model.py:43-49: tap offsets at low resolution, strided output pixels).
//
// Precision: fp32 parity (1e-3 end to end) is not reachable with one 11-bit product (2^-11 operand rounding,
// ~35 stacked convs), so by default each product is error-compensated:  a*b ~= ah*bh + al*bh + ah*bl  with
// ah = fp16(a), al = fp16(a - ah): 22 mantissa bits per operand, three MMAs into the same fp32 accumulator
// ("3xFP16").  fp16 has the mantissa of tf32 at twice the MMA rate and half the operand bytes; its narrow exponent
// range is handled by scaling every operand tensor by a power of two taken from its max|x| (og_prep_split /
// og_pack_weights_f16 write x * 2^k; the epilogue multiplies the accumulator by 2^-(ka+kb)): elements within
// 2^-18 of the tensor maximum keep all 22 bits, smaller ones an absolute error <= 2^-39 of the maximum.
//
// GEMM tiling: one CTA = 128 output pixels (a TN x TH x TW patch) x BN output channels (BN % 8 == 0,
// <= 128); K loop over taps x 64-channel chunks; STAGES-deep smem ring of {A_hi, A_lo, B_hi, B_lo}.
// Warpgroup roles: warpgroup 0 = TMA producer (one elected thread), warpgroups 1 and 2 = MMA + epilogue, each
// owning 64 of the 128 tile rows.  Both kernels issue one wgmma over the whole N extent per product and k-step (the A
// tile is read from shared memory once); in the weight-gradient kernel that B operand is MN-major and spans several
// 64-channel slabs.
#include "common.cuh"
#include "wgmma.cuh"
#include <cuda_fp16.h>
#include <stdlib.h>
#include <iterator>
#include <type_traits>
#include <utility>

namespace {

constexpr int TC_BM = 128;
constexpr int TC_BK = 64;              // fp16 elements per k-chunk = one 128-byte swizzle row (4 MMA k-steps of 16)
constexpr int TC_MAX_TAPS = 36;
constexpr int TC_THREADS = 384;        // producer warpgroup + two consumer warpgroups
constexpr int TC_CONSUMER_WARPS = 8;
constexpr size_t TC_SMEM_BUDGET = 200 * 1024;  // operand ring per CTA (one CTA per SM; 227 KB is the sm_90 limit)

struct TcTaps {
  int n;
  int dh[TC_MAX_TAPS], dw[TC_MAX_TAPS], dn[TC_MAX_TAPS], widx[TC_MAX_TAPS];
};

struct TcParams {
  int N, OH, OW;          // GEMM-row pixel grid (before the output stride/phase mapping)
  int TN, TH, TW;         // tile patch: TN*TH*TW == 128
  int tiles_h, tiles_w;   // tiles per image along h / w
  int cchunks;            // ceil(C / 64)
  int klast;              // MMA k-steps (16 channels each) that the last chunk really needs: 1..4
  const unsigned* amax_a; // float bits of max|x| of the two operand tensors (power-of-two operand scaling)
  const unsigned* amax_b;
  int K;                  // output channels actually stored (<= gridDim.y * BN)
  float* y;
  long long ysn, ysh, ysw;  // output strides (elements) of the FULL-resolution output tensor
  int osy, osx, opy, opx;   // output pixel = (osy * h + opy, osx * w + opx)
  int OHfull, OWfull;       // bounds of the output tensor
  const float* bias;        // [K] or null
  int act;
  float slope;
  int ksplit;               // > 1: gridDim.z CTAs share one output tile, each reduces a slice of the (tap, chunk) loop
  float* work;              // ksplit > 1: slice z writes its partial output to work + z * work_plane (y's layout)
  long long work_plane;
  // conv_tc_rows_kernel only: taps per row run, resident A slot sets (1 or 2), B ring stages
  int run, asets, bstages;
  TcTaps taps;
};

__device__ __forceinline__ float tc_act(float v, int act, float slope) {
  if (act == OG_ACT_LRELU) return v > 0.f ? v : v * slope;
  if (act == OG_ACT_TANH) return tanhf(v);
  if (act == OG_ACT_SIGMOID) return og_sigmoid(v);
  return v;
}

// accumulator -> fp32 result: undo the two power-of-two operand scales (two factors: their product may leave the
// float exponent range although each factor and the result do not)
struct TcScale { float fa, fb; };
__device__ __forceinline__ TcScale tc_scale(const unsigned* amax_a, const unsigned* amax_b) {
  TcScale s;
  s.fa = og_exp2i(-og_scale_exp(__ldg(amax_a)));
  s.fb = og_exp2i(-og_scale_exp(__ldg(amax_b)));
  return s;
}

// 64 x BN fp32 accumulator of one consumer warpgroup, issued as ONE wgmma per call.  TA / TB = 1: that operand is
// MN-major (the weight gradient's; an MN-major B wider than 64 spans several slabs, LBO apart in its descriptor).
template <int BN, int TA = 0, int TB = 0>
struct TcAccWide {
  float d[BN / 2];

  __device__ __forceinline__ void zero() {
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) d[i] = 0.f;
  }
  __device__ __forceinline__ void hold() { wg_hold(d); }
  // scale_d = 0: D = A * B (the accumulator's previous contents are dropped)
  __device__ __forceinline__ void mma(uint64_t a, uint64_t b, int scale_d) {
    static_assert(BN == 32 || BN == 48 || BN == 64 || BN == 96 || BN == 104 || BN == 112 || BN == 128,
                  "no wgmma wrapper for this tile width");
    if constexpr (BN == 32) wg_mma_n32<TA, TB>(d, a, b, scale_d);
    if constexpr (BN == 48) wg_mma_n48<TA, TB>(d, a, b, scale_d);
    if constexpr (BN == 64) wg_mma_n64<TA, TB>(d, a, b, scale_d);
    if constexpr (BN == 96) wg_mma_n96<TA, TB>(d, a, b, scale_d);
    if constexpr (BN == 104) wg_mma_n104<TA, TB>(d, a, b, scale_d);
    if constexpr (BN == 112) wg_mma_n112<TA, TB>(d, a, b, scale_d);
    if constexpr (BN == 128) wg_mma_n128<TA, TB>(d, a, b, scale_d);
  }
  __device__ __forceinline__ void add(const TcAccWide& o) {
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) d[i] += o.d[i];
  }
  // columns [0, BN/2) += columns [BN/2, BN): the same thread holds column c and c + BN/2 (n8 blocks i, i + BN/16)
  __device__ __forceinline__ void fold_halves() {
#pragma unroll
    for (int i = 0; i < BN / 16; ++i)
#pragma unroll
      for (int q = 0; q < 4; ++q) d[4 * i + q] += d[4 * (i + BN / 16) + q];
  }
  // fn(column, row half h, value at column, value at column + 1) for every accumulator pair of this thread
  template <class F>
  __device__ __forceinline__ void each(int lane, F&& fn) const {
    const int c2 = 2 * (lane & 3);
#pragma unroll
    for (int i = 0; i < BN / 8; ++i)
#pragma unroll
      for (int h = 0; h < 2; ++h) fn(8 * i + c2, h, d[4 * i + 2 * h], d[4 * i + 2 * h + 1]);
  }
};

// One stage's MMAs into a fresh partial sum: KS k-steps of 16, KSTEP bytes apart in the operand tiles, as ONE
// straight-line issue window (fence, the MMAs, commit), then the wait for them.  Nothing in the window branches or
// touches the accumulator registers; otherwise ptxas waits for every wgmma before issuing the next (C7520 / C7519 /
// C7514 warnings).  The wait sits in here too, so that tc_stage_mma, which chooses KS at run time, merges the
// accumulators only after it (C7517 otherwise).
// al*bh, ah*bl, ah*bh (small terms first); STACKED: al*[bh_hi | bh_lo], ah*[bh_hi | bh_lo].
template <int KS, uint32_t KSTEP, bool STACKED, class Acc>
__device__ __forceinline__ void tc_stage_window(Acc& part, uint64_t ah, uint64_t al, uint64_t bh, uint64_t bl) {
  wg_fence();
#pragma unroll
  for (int k = 0; k < KS; ++k) {
    const uint64_t koff = (uint64_t)((k * KSTEP) >> 4);
    if constexpr (STACKED) {
      part.mma(al + koff, bh + koff, k > 0);
      part.mma(ah + koff, bh + koff, 1);
    } else {
      part.mma(al + koff, bh + koff, k > 0);
      part.mma(ah + koff, bl + koff, 1);
      part.mma(ah + koff, bh + koff, 1);
    }
  }
  wg_commit();
  wg_wait<0>();
  part.hold();
}

// One stage's MMAs with ks = 1..4 k-steps (a last channel chunk of fewer than 64 real channels skips the k-steps that
// would multiply zeros): one issue window per count, since a window whose length is a run-time value is serialized.
template <uint32_t KSTEP, bool STACKED, class Acc>
__device__ __forceinline__ void tc_stage_mma(int ks, Acc& part, uint64_t ah, uint64_t al, uint64_t bh, uint64_t bl) {
  switch (ks) {
    case 1: tc_stage_window<1, KSTEP, STACKED>(part, ah, al, bh, bl); break;
    case 2: tc_stage_window<2, KSTEP, STACKED>(part, ah, al, bh, bl); break;
    case 3: tc_stage_window<3, KSTEP, STACKED>(part, ah, al, bh, bl); break;
    default: tc_stage_window<4, KSTEP, STACKED>(part, ah, al, bh, bl); break;
  }
}

// Warp index as a value ptxas knows to be warp-uniform (threadIdx.x >> 5 is, but the compiler cannot prove it, and
// a role branch it takes for divergent serializes every wgmma behind it)
__device__ __forceinline__ int tc_warp_uniform() { return __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 5), 0); }

// Kernel prologue: thread 0 prefetches the tensor maps and initialises the barriers of the operand ring (full: the
// producer's arrival with its TMA bytes; empty: one arrival per consumer warp) for the whole CTA.  Returns the dynamic
// shared memory aligned to 1024 bytes, the atom of the 128-byte swizzle.
template <class... Maps>
__device__ __forceinline__ uint8_t* tc_prologue(uint8_t* smem_raw, uint64_t* full, uint64_t* empty, int stages,
                                                const Maps&... maps) {
  if (threadIdx.x == 0) {
    (prefetch_tmap(&maps), ...);
    for (int s = 0; s < stages; ++s) {
      mbar_init(&full[s], 1);
      mbar_init(&empty[s], TC_CONSUMER_WARPS);
    }
    fence_barrier_init();
  }
  __syncthreads();
  return reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
}

// Steps a walk through a ring of depth pipeline slots to the next slot; the barrier parity flips at each wrap
__device__ __forceinline__ void tc_ring_next(int& stage, uint32_t& phase, int depth) {
  if (++stage == depth) {
    stage = 0;
    phase ^= 1;
  }
}

// Origin (image, row, column) of this CTA's TN x TH x TW output patch; blockIdx.x walks the patches w fastest.
// ONE_IMAGE: TN == 1.
struct TcTile { int n0, h0, w0; };
template <bool ONE_IMAGE = false>
__device__ __forceinline__ TcTile tc_tile_origin(const TcParams& p) {
  int t = blockIdx.x;
  const int tw_i = t % p.tiles_w;
  t /= p.tiles_w;
  const int th_i = t % p.tiles_h;
  const int tn_i = t / p.tiles_h;
  return {ONE_IMAGE ? tn_i : tn_i * p.TN, th_i * p.TH, tw_i * p.TW};
}

// ===================== epilogue: registers -> global (consumer warpgroup cg = (warp >> 2) - 1) =====================
template <int BN, bool STACKED>
__device__ __forceinline__ void tc_epilogue(TcAccWide<BN>& acc, const TcParams& p, int n0, int h0, int w0, int col0,
                                            int warp, int lane) {
  const int cg = (warp >> 2) - 1;
  float* yrow[2];
  bool row_ok[2];
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int row = cg * 64 + (warp & 3) * 16 + (lane >> 2) + 8 * h;   // tile row = output pixel within the patch
    const int tw = row % p.TW;
    const int th = (row / p.TW) % p.TH;
    const int tn = row / (p.TW * p.TH);
    const int n = n0 + tn, hh = h0 + th, w = w0 + tw;
    const int oy = p.osy * hh + p.opy, ox = p.osx * w + p.opx;
    row_ok[h] = (n < p.N) && (hh < p.OH) && (w < p.OW) && (oy < p.OHfull) && (ox < p.OWfull);
    yrow[h] = p.y + (long long)n * p.ysn + (long long)oy * p.ysh + (long long)ox * p.ysw + col0;
  }
  const TcScale sc = tc_scale(p.amax_a, p.amax_b);
  if (STACKED) acc.fold_halves();
  acc.each(lane, [&](int c, int h, float v0, float v1) {
    if (STACKED && c >= BN / 2) return;
    if (!row_ok[h] || col0 + c >= p.K) return;        // K % 4 == 0: the pair (c, c + 1) is in or out together
    float2 v = make_float2(v0 * sc.fa * sc.fb, v1 * sc.fa * sc.fb);
    if (p.bias) {
      const float2 b = __ldg(reinterpret_cast<const float2*>(p.bias + col0 + c));
      v.x += b.x; v.y += b.y;
    }
    if (p.act != OG_ACT_NONE) {
      v.x = tc_act(v.x, p.act, p.slope);
      v.y = tc_act(v.y, p.act, p.slope);
    }
    float* dst = yrow[h] + c;
    if (p.ksplit > 1) dst = p.work + (long long)blockIdx.z * p.work_plane + (dst - p.y);   // partial sum of this slice
    *reinterpret_cast<float2*>(dst) = v;
  });
}

// ------------------------------------------------------------------------------------------------
// STACKED (<= 32 output channels): B is [w_hi | w_lo] of the same BN / 2 output channels stacked along N, so a k-step
// is two MMAs, a_lo [w_hi | w_lo] and a_hi [w_hi | w_lo], and the epilogue adds the two column halves (the extra
// a_lo w_lo term is below the rounding of the others).  Each A copy is read from shared memory once per k-step
// instead of 1.5 times -- narrow layers are bound by those reads, not by the MMA rate.
template <int BN, int STAGES, bool STACKED>
__global__ void __launch_bounds__(TC_THREADS, 1)
conv_tc_kernel(const __grid_constant__ CUtensorMap map_ah, const __grid_constant__ CUtensorMap map_al,
               const __grid_constant__ CUtensorMap map_bh, const __grid_constant__ CUtensorMap map_bl,
               const TcParams p) {
  static_assert(BN % 8 == 0 && BN <= 128, "");
  constexpr uint32_t A_BYTES = TC_BM * 128;         // 128 rows of 128 bytes = 16 KB
  constexpr uint32_t B_BYTES = BN * 128;            // BN % 8 == 0: a whole number of 1024-byte swizzle atoms
  constexpr uint32_t STAGE_BYTES = 2 * A_BYTES + (STACKED ? 1 : 2) * B_BYTES;
  extern __shared__ uint8_t smem_raw[];
  __shared__ __align__(8) uint64_t full_bar[STAGES], empty_bar[STAGES];

  const int warp = tc_warp_uniform(), lane = threadIdx.x & 31;
  const auto [n0, h0, w0] = tc_tile_origin(p);
  const int col0 = blockIdx.y * (STACKED ? BN / 2 : BN);
  const int nk_total = p.taps.n * p.cchunks;
  const int per_split = (nk_total + p.ksplit - 1) / p.ksplit;
  const int it_beg = blockIdx.z * per_split;
  const int nk = min(nk_total, it_beg + per_split) - it_beg;
  if (nk <= 0) return;

  uint8_t* const smem = tc_prologue(smem_raw, full_bar, empty_bar, STAGES, map_ah, map_bh, map_al, map_bl);

  if (warp < 4) {
    // ===================== TMA producer =====================
    if (threadIdx.x == 0) {
      int stage = 0;
      uint32_t phase = 0;
      for (int it = 0; it < nk; ++it) {
        const int tap = (it_beg + it) / p.cchunks, cc = (it_beg + it) - tap * p.cchunks;
        uint64_t* const full = &full_bar[stage];
        mbar_wait(&empty_bar[stage], phase ^ 1);
        uint8_t* sa = smem + (size_t)stage * STAGE_BYTES;
        mbar_expect_tx(full, STAGE_BYTES);
        const int c0 = cc * TC_BK, ws = w0 + p.taps.dw[tap], hs = h0 + p.taps.dh[tap], widx = p.taps.widx[tap];
        const int ns = n0 + p.taps.dn[tap];   // image offset: selects a space-to-depth phase block of the source
        tma_load_4d(sa, &map_ah, full, c0, ws, hs, ns);
        tma_load_3d(sa + 2 * A_BYTES, &map_bh, full, c0, col0, widx);
        tma_load_4d(sa + A_BYTES, &map_al, full, c0, ws, hs, ns);
        // stacked: the lo rows follow the hi rows inside the same N extent (maps with a box of BN / 2 rows)
        tma_load_3d(sa + 2 * A_BYTES + (STACKED ? B_BYTES / 2 : B_BYTES), &map_bl, full, c0, col0, widx);
        tc_ring_next(stage, phase, STAGES);
      }
    }
    return;
  }

  // ===================== MMA: consumer warpgroup cg owns tile rows [64 cg, 64 cg + 64) =====================
  const int cg = (warp >> 2) - 1;
  // The tensor core adds its products into the fp32 accumulator with truncation; over the long K loops of this
  // library the bias that builds up is visible in end-to-end gradients.  So each stage's MMAs (K = 64) start a fresh
  // partial sum, which is then added into the register accumulator with round-to-nearest fp32 adds.
  TcAccWide<BN> acc, part;
  acc.zero();
  int stage = 0;
  uint32_t phase = 0;
  for (int it = 0; it < nk; ++it) {
    mbar_wait(&full_bar[stage], phase);
    const uint32_t sa = smem_u32(smem + (size_t)stage * STAGE_BYTES);
    const uint64_t ah = wg_desc_k(sa + cg * 64 * 128), al = wg_desc_k(sa + A_BYTES + cg * 64 * 128);
    const uint64_t bh = wg_desc_k(sa + 2 * A_BYTES), bl = wg_desc_k(sa + 2 * A_BYTES + B_BYTES);
    // A k-step advances 32 bytes (16 fp16) inside the swizzle row; stacked, bh addresses [w_hi | w_lo].
    const int ks = ((it_beg + it + 1) % p.cchunks == 0) ? p.klast : 4;
    tc_stage_mma<32, STACKED>(ks, part, ah, al, bh, bl);
    if (lane == 0) mbar_arrive(&empty_bar[stage]);   // this stage's MMAs have completed: free its slot
    acc.add(part);
    tc_ring_next(stage, phase, STAGES);
  }

  tc_epilogue<BN, STACKED>(acc, p, n0, h0, w0, col0, warp, lane);
}

// ------------------------------------------------------------------------------------------------
// Row runs: a tap list that splits into runs of R taps with equal (dw, dn) and R consecutive dh (the column-by-column
// order of the 3x3 stride-1 layers, R = 3).  With a TH x TW patch (TN = 1, TW % 8 == 0) the A tile of tap dh + 1 is
// the tile of tap dh moved down one image row = TW smem rows, a whole number of 1024-byte swizzle atoms.  So one
// (TH + R - 1) x TW box per channel chunk and operand holds the A operands of all R taps of a run; tap r is the
// ordinary K-major descriptor at r * TW * 128 bytes into it, and TMA's zero fill gives the box the values the per-tap
// boxes of conv_tc_kernel read.  A is loaded once per run instead of once per tap.
//
// Shared memory: asets x cchunks A slots (hi and lo box each), every chunk's slot resident across the run (chunk c
// is read at stages c, c + cchunks, ...), then a ring of bstages B tiles, one (tap, chunk) weight tile each.  Two
// producer threads in different warps: warp 0 refills A slots as they are released (after the consumers' last tap
// of the run for that chunk), warp 1 streams the B ring; neither blocks the other.  With two slot sets the next run's
// A loads as soon as the previous run of the same set is done.
// The consumers walk exactly the stages of conv_tc_kernel (tap-major, chunk-minor, one fresh partial sum per stage
// added into the accumulator, the same last-chunk k-steps and epilogue): only the A descriptor's address differs, so
// the results are bitwise those of conv_tc_kernel.  No reduction split (ksplit == 1).
constexpr int TC_ROWS_MAX_SLOTS = 8;
constexpr int TC_ROWS_MAX_BSTAGES = 4;
// dynamic shared memory per block, the 1024-byte alignment slack included: sm_90's opt-in limit of 227 KB, less room
// for the static barriers
constexpr size_t TC_ROWS_SMEM_LIMIT = 227 * 1024 - 1024;

template <int BN, bool STACKED>
__global__ void __launch_bounds__(TC_THREADS, 1)
conv_tc_rows_kernel(const __grid_constant__ CUtensorMap map_ah, const __grid_constant__ CUtensorMap map_al,
                    const __grid_constant__ CUtensorMap map_bh, const __grid_constant__ CUtensorMap map_bl,
                    const TcParams p) {
  static_assert(BN % 8 == 0 && BN <= 128, "");
  constexpr uint32_t B_BYTES = BN * 128;
  constexpr uint32_t B_STAGE = (STACKED ? 1 : 2) * B_BYTES;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  __shared__ __align__(8) uint64_t a_full[TC_ROWS_MAX_SLOTS], a_empty[TC_ROWS_MAX_SLOTS];
  __shared__ __align__(8) uint64_t b_full[TC_ROWS_MAX_BSTAGES], b_empty[TC_ROWS_MAX_BSTAGES];

  const int warp = tc_warp_uniform(), lane = threadIdx.x & 31;
  const int R = p.run;
  const uint32_t a_box = (uint32_t)((p.TH + R - 1) * p.TW) * 128;   // one operand of one slot; TW % 8 == 0: 1024 | a_box
  const uint32_t slot_bytes = 2 * a_box;
  const int nslots = p.asets * p.cchunks;
  uint8_t* const smem_b = smem + (size_t)nslots * slot_bytes;
  const auto [n0, h0, w0] = tc_tile_origin<true>(p);
  const int col0 = blockIdx.y * (STACKED ? BN / 2 : BN);
  const int nk = p.taps.n * p.cchunks;

  if (threadIdx.x == 0) {
    prefetch_tmap(&map_ah);
    prefetch_tmap(&map_bh);
    prefetch_tmap(&map_al);
    prefetch_tmap(&map_bl);
    for (int s = 0; s < nslots; ++s) {
      mbar_init(&a_full[s], 1);
      mbar_init(&a_empty[s], TC_CONSUMER_WARPS);
    }
    for (int s = 0; s < p.bstages; ++s) {
      mbar_init(&b_full[s], 1);
      mbar_init(&b_empty[s], TC_CONSUMER_WARPS);
    }
    fence_barrier_init();
  }
  __syncthreads();

  if (warp < 4) {
    // ===================== TMA producers =====================
    if (threadIdx.x == 0) {
      // A: run j fills slot set j % asets, one (TH + R - 1)-row box per chunk and operand from the run's first row
      for (int j = 0; j < p.taps.n / R; ++j) {
        const int t0 = j * R;
        const int hs = h0 + min(p.taps.dh[t0], p.taps.dh[t0 + R - 1]), ws = w0 + p.taps.dw[t0];
        const int ns = n0 + p.taps.dn[t0];
        const uint32_t phase = (j / p.asets) & 1;
        for (int cc = 0; cc < p.cchunks; ++cc) {
          const int s = (j % p.asets) * p.cchunks + cc;
          mbar_wait(&a_empty[s], phase ^ 1);
          uint8_t* sa = smem + (size_t)s * slot_bytes;
          mbar_expect_tx(&a_full[s], slot_bytes);
          tma_load_4d(sa, &map_ah, &a_full[s], cc * TC_BK, ws, hs, ns);
          tma_load_4d(sa + a_box, &map_al, &a_full[s], cc * TC_BK, ws, hs, ns);
        }
      }
    } else if (threadIdx.x == 32) {
      // B: one (tap, chunk) weight tile per stage, as conv_tc_kernel.  The ring's depth is a run-time value: it gets
      // as many stages as the shared memory left after the layer's A slots holds
      int stage = 0;
      uint32_t phase = 0;
      for (int it = 0; it < nk; ++it) {
        const int tap = it / p.cchunks, cc = it - tap * p.cchunks;
        uint64_t* const full = &b_full[stage];
        mbar_wait(&b_empty[stage], phase ^ 1);
        uint8_t* sb = smem_b + (size_t)stage * B_STAGE;
        mbar_expect_tx(full, B_STAGE);
        tma_load_3d(sb, &map_bh, full, cc * TC_BK, col0, p.taps.widx[tap]);
        tma_load_3d(sb + (STACKED ? B_BYTES / 2 : B_BYTES), &map_bl, full, cc * TC_BK, col0, p.taps.widx[tap]);
        tc_ring_next(stage, phase, p.bstages);
      }
    }
    return;
  }

  // ===================== MMA: consumer warpgroup cg owns tile rows [64 cg, 64 cg + 64) =====================
  const int cg = (warp >> 2) - 1;
  TcAccWide<BN> acc, part;
  acc.zero();
  int stage = 0;
  uint32_t phase = 0;
  for (int it = 0; it < nk; ++it) {
    const int tap = it / p.cchunks, cc = it - tap * p.cchunks;
    const int j = tap / R, t0 = j * R;
    const int s = (j % p.asets) * p.cchunks + cc;
    const int row = p.taps.dh[tap] - min(p.taps.dh[t0], p.taps.dh[t0 + R - 1]);   // tap's first row in the box
    mbar_wait(&a_full[s], (j / p.asets) & 1);
    mbar_wait(&b_full[stage], phase);
    const uint32_t sa = smem_u32(smem + (size_t)s * slot_bytes) + (uint32_t)(row * p.TW) * 128 + cg * 64 * 128;
    const uint32_t sb = smem_u32(smem_b + (size_t)stage * B_STAGE);
    const uint64_t ah = wg_desc_k(sa), al = wg_desc_k(sa + a_box);
    const uint64_t bh = wg_desc_k(sb), bl = wg_desc_k(sb + B_BYTES);
    tc_stage_mma<32, STACKED>(cc == p.cchunks - 1 ? p.klast : 4, part, ah, al, bh, bl);
    if (lane == 0) {
      mbar_arrive(&b_empty[stage]);
      if (tap - t0 == R - 1) mbar_arrive(&a_empty[s]);   // the run's last tap of this chunk: the slot is free
    }
    acc.add(part);
    tc_ring_next(stage, phase, p.bstages);
  }

  tc_epilogue<BN, STACKED>(acc, p, n0, h0, w0, col0, warp, lane);
}

// ------------------------------------------------------------------------------------------------
// host side: tensor maps
// ------------------------------------------------------------------------------------------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

EncodeTiledFn get_encode() {
  static EncodeTiledFn fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess) fn = (EncodeTiledFn)p;
  }
  return fn;
}

// fp16 tensor viewed as [d4][d3][d2][d1][d0] (d0 contiguous); strides in elements for d1..
int make_map(CUtensorMap* m, const void* base, int rank, const unsigned long long* dims,
             const unsigned long long* strides_elems, const unsigned* box) {
  EncodeTiledFn enc = get_encode();
  if (!enc) return (int)cudaErrorNotSupported;
  cuuint64_t gdim[5], gstr[4];
  cuuint32_t bx[5], es[5];
  for (int i = 0; i < rank; ++i) {
    gdim[i] = dims[i];
    bx[i] = box[i];
    es[i] = 1;
  }
  for (int i = 0; i < rank - 1; ++i) gstr[i] = strides_elems[i] * sizeof(__half);
  CUresult r = enc(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, (cuuint32_t)rank, (void*)base, gdim, gstr, bx, es,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS ? 0 : 1000 + (int)r;
}

// deepest operand ring that fits the shared-memory budget (at most 4 stages)
constexpr int tc_stages(size_t stage_bytes) {
  return TC_SMEM_BUDGET / stage_bytes >= 4 ? 4 : (int)(TC_SMEM_BUDGET / stage_bytes);
}

// Launches KERNEL with smem bytes of dynamic shared memory.  Its limit is raised to smem_limit on the first launch
// only: the attribute call would add host time to every convolution.
template <auto KERNEL, class... Args>
int tc_launch(size_t smem_limit, dim3 grid, size_t smem, cudaStream_t stream, const Args&... args) {
  static bool configured = false;
  if (!configured) {
    cudaError_t e = cudaFuncSetAttribute(KERNEL, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_limit);
    if (e != cudaSuccess) return (int)e;
    configured = true;
  }
  KERNEL<<<grid, TC_THREADS, smem, stream>>>(args...);
  return (int)cudaGetLastError();
}

// N tile widths with an instantiated kernel: the layers of the hot path (K = 400 -> 4 x 104, 200 -> 2 x 104,
// 96, 48, ...) each run within 8 columns of their real width
constexpr int TC_BN_SET[] = {32, 48, 64, 96, 104, 112, 128};

// fn(std::integral_constant<int, BN>()) for the width BN of TC_BN_SET equal to bn; cudaErrorInvalidValue for any other
template <class F, size_t... I>
int tc_with_width(int bn, F&& fn, std::index_sequence<I...>) {
  int rc = (int)cudaErrorInvalidValue;
  (void)((bn == TC_BN_SET[I] && (rc = fn(std::integral_constant<int, TC_BN_SET[I]>()), true)) || ...);
  return rc;
}
template <class F>
int tc_with_width(int bn, F&& fn) {
  return tc_with_width(bn, fn, std::make_index_sequence<std::size(TC_BN_SET)>());
}

// fn(BN, STACKED) as integral constants for a forward N tile: stacked, [w_hi | w_lo] of stk_rows = 16 or 32 output
// channels; else the instantiated width bn
template <class F>
int tc_with_tile(int bn, bool stacked, int stk_rows, F&& fn) {
  if (stacked)
    return stk_rows == 16 ? fn(std::integral_constant<int, 32>(), std::true_type())
                          : fn(std::integral_constant<int, 64>(), std::true_type());
  return tc_with_width(bn, [&](auto width) { return fn(width, std::false_type()); });
}

// Taps per row run if the tap list splits completely into runs of the same length R >= 2 (equal dw and dn, dh
// stepping by +1 or by -1 through the run), else 0
int tc_row_run(const TcTaps& t) {
  int R = 1;
  while (R < t.n && t.dw[R] == t.dw[0] && t.dn[R] == t.dn[0] && t.dh[R] - t.dh[R - 1] == t.dh[1] - t.dh[0]) ++R;
  if (R < 2 || t.n % R || abs(t.dh[1] - t.dh[0]) != 1) return 0;
  for (int b = 0; b < t.n; b += R)
    for (int i = b + 1; i < b + R; ++i)
      if (t.dw[i] != t.dw[b] || t.dn[i] != t.dn[b] || t.dh[i] - t.dh[i - 1] != t.dh[b + 1] - t.dh[b] ||
          abs(t.dh[i] - t.dh[i - 1]) != 1)
        return 0;
  return R;
}


// ------------------------------------------------------------------------------------------------
// weight gradient on the tensor cores.
//   dW[t][co][ci] += sum_{n,h,w} G[n,h,w,co] * X[n, h+dh_t, w+dw_t, ci]
// GEMM per tap: M = co, N = ci, reduction over pixels.  Both operands are read straight from the NHWC hi/lo
// tensors the forward / input-gradient kernels already use, i.e. they are "MN-major" for the MMA (channel index
// contiguous, reduction index = smem row; 16-bit operands take the ordinary 128B swizzle).  A smem operand is a
// stack of "slabs" (64 channels x 64 pixels = 64 rows of 128 bytes, lbo = 8192 apart; 8-row groups sbo = 1024
// apart); one 5-D TMA box (64 channels-in-slab, w, h, n, slab) fills all slabs of an operand, the tap shift is a
// plain coordinate offset with out-of-bounds zero fill.  One MMA consumes 16 pixel rows (K = 16); consumer
// warpgroup cg multiplies slab cg of the G operand (64 output channels) by the whole BNW-wide X operand, one wgmma
// per product and k-step.  A ci tile starts at any multiple of 8 channels (citile * BNW): the X map's channel
// dimension is the whole pixel vector, the slab dimension steps 64 channels on from the tile's first one.  A
// warpgroup whose G slab lies wholly past Kp issues nothing (it only releases the stages).  TAPS = 2: two entries
// with the same G image offset share the CTA and its G tile, one accumulator each.
// Grid: (co tiles x ci tiles, entries / TAPS, pixel splits); partial sums meet in a fixed order (wgrad_sum_kernel).
// ------------------------------------------------------------------------------------------------
struct TcWgradParams {
  int N, OH, OW;        // pixel grid of G
  int cw, chh, cn;      // pixel chunk of one stage: cw x chh x cn = 64 pixels (w fastest)
  int wchunks, hchunks; // chunks per row / per image column
  int total_chunks;
  int chunks_per_cta;
  int Kp, C;            // rows (co) and columns (ci) of each dW[t]
  int cotiles;          // blockIdx.x = citile * cotiles + cotile
  int nentries;         // blockIdx.y = group of TAPS consecutive entries sharing one G tile
  float* dw;            // [ntaps_out][Kp][C]; or, when work is set, work[(z * nentries + e) * Kp * C] per (split, entry)
  float* work;
  const unsigned* amax_g; // operand scales (see TcParams)
  const unsigned* amax_x;
  // entry e: dW[out[e]] += G[n + gdn[e], h, w]^T * X[n + xdn[e], h + xdh[e], w + xdw[e]]
  int gdn[TC_MAX_TAPS], xdh[TC_MAX_TAPS], xdw[TC_MAX_TAPS], xdn[TC_MAX_TAPS], out[TC_MAX_TAPS];
};

constexpr int WG_PIX = 64;                     // pixels per stage (4 MMA k-steps of 16)
constexpr int WG_CH = 64;                      // channels per slab = one 128-byte row
constexpr uint32_t WG_SLAB = WG_PIX * 128;     // bytes of one slab: 64 pixels x 64 channels

__device__ __forceinline__ uint64_t make_desc_mn(uint32_t saddr) { return wg_desc(saddr, WG_SLAB, 1024); }

template <int BNW, int STAGES, int TAPS>
__global__ void __launch_bounds__(TC_THREADS, 1)
conv_tc_wgrad_wide_kernel(const __grid_constant__ CUtensorMap map_gh, const __grid_constant__ CUtensorMap map_gl,
                          const __grid_constant__ CUtensorMap map_xh, const __grid_constant__ CUtensorMap map_xl,
                          const TcWgradParams p) {
  constexpr int NSB = (BNW + WG_CH - 1) / WG_CH;          // slabs of the X operand
  constexpr uint32_t A_BYTES = 2 * WG_SLAB;               // 128 co = 2 slabs = 16 KB
  constexpr uint32_t B_BYTES = NSB * WG_SLAB;
  constexpr uint32_t STAGE_BYTES = 2 * A_BYTES + TAPS * 2 * B_BYTES;   // G hi, G lo, then X hi, X lo per entry
  extern __shared__ uint8_t smem_raw[];
  __shared__ __align__(8) uint64_t full_bar[STAGES], empty_bar[STAGES];

  const int warp = tc_warp_uniform(), lane = threadIdx.x & 31;
  const int cotile = blockIdx.x % p.cotiles, citile = blockIdx.x / p.cotiles;
  const int e0 = blockIdx.y * TAPS;                       // this CTA's entries: e0 .. e0 + ne - 1
  const int ne = min(TAPS, p.nentries - e0);
  const int ch_beg = blockIdx.z * p.chunks_per_cta;
  const int ch_end = min(p.total_chunks, ch_beg + p.chunks_per_cta);
  const int nk = ch_end - ch_beg;
  const uint32_t tx_bytes = 2 * A_BYTES + ne * 2 * B_BYTES;
  if (nk <= 0) return;

  uint8_t* const smem = tc_prologue(smem_raw, full_bar, empty_bar, STAGES, map_gh, map_xh);

  if (warp < 4) {
    if (threadIdx.x == 0) {
      int stage = 0;
      uint32_t phase = 0;
      const int gdn = p.gdn[e0];                          // the same for every entry of the CTA (host)
      const int aslab = cotile * 2, ci0 = citile * BNW;
      for (int it = 0; it < nk; ++it) {
        const int ch = ch_beg + it;
        const int wc = ch % p.wchunks;
        const int t2 = ch / p.wchunks;
        const int hc = t2 % p.hchunks;
        const int w0 = wc * p.cw, h = hc * p.chh, n = (t2 / p.hchunks) * p.cn;
        uint64_t* const full = &full_bar[stage];
        mbar_wait(&empty_bar[stage], phase ^ 1);
        uint8_t* sa = smem + (size_t)stage * STAGE_BYTES;
        mbar_expect_tx(full, tx_bytes);
        tma_load_5d(sa, &map_gh, full, 0, w0, h, n + gdn, aslab);
        tma_load_5d(sa + A_BYTES, &map_gl, full, 0, w0, h, n + gdn, aslab);
        for (int t = 0; t < ne; ++t) {
          const int e = e0 + t;
          const int xw = w0 + p.xdw[e], xh = h + p.xdh[e], xn = n + p.xdn[e];
          uint8_t* sb = sa + 2 * A_BYTES + t * 2 * B_BYTES;
          tma_load_5d(sb, &map_xh, full, ci0, xw, xh, xn, 0);
          tma_load_5d(sb + B_BYTES, &map_xl, full, ci0, xw, xh, xn, 0);
        }
        if (++stage == STAGES) {
          stage = 0;
          phase ^= 1;
        }
      }
    }
    return;
  }

  const int cg = (warp >> 2) - 1;
  if ((cotile * 2 + cg) * WG_CH >= p.Kp) {   // G slab past the last row: zero-filled, no product to issue
    int stage = 0;
    uint32_t phase = 0;
    for (int it = 0; it < nk; ++it) {
      mbar_wait(&full_bar[stage], phase);
      if (lane == 0) mbar_arrive(&empty_bar[stage]);
      if (++stage == STAGES) {
        stage = 0;
        phase ^= 1;
      }
    }
    return;
  }
  // per-stage partial sums, as in conv_tc_kernel; one accumulator per entry, each entry's stages in the same order
  // as with one entry per CTA
  TcAccWide<BNW, 1, 1> acc[TAPS], part;
#pragma unroll
  for (int t = 0; t < TAPS; ++t) acc[t].zero();
  int stage = 0;
  uint32_t phase = 0;
  for (int it = 0; it < nk; ++it) {
    mbar_wait(&full_bar[stage], phase);
    const uint32_t sa = smem_u32(smem + (size_t)stage * STAGE_BYTES);
    const uint64_t ah = make_desc_mn(sa + cg * WG_SLAB), al = make_desc_mn(sa + A_BYTES + cg * WG_SLAB);
    const uint32_t sb = sa + 2 * A_BYTES;
    tc_stage_mma<16 * 128, false>(WG_PIX / 16, part, ah, al, make_desc_mn(sb), make_desc_mn(sb + B_BYTES));
    acc[0].add(part);
    if constexpr (TAPS == 2) {
      if (ne == 2) {
        const uint32_t sb1 = sb + 2 * B_BYTES;
        tc_stage_mma<16 * 128, false>(WG_PIX / 16, part, ah, al, make_desc_mn(sb1), make_desc_mn(sb1 + B_BYTES));
        acc[1].add(part);
      }
    }
    if (lane == 0) mbar_arrive(&empty_bar[stage]);     // this stage's MMAs have completed: free its slot
    if (++stage == STAGES) {
      stage = 0;
      phase ^= 1;
    }
  }

  const int co0 = cotile * TC_BM + cg * 64 + (warp & 3) * 16 + (lane >> 2);
  const int cleft = p.C - citile * BNW;          // a multiple of 8: the pair (c, c + 1) is in or out together
  const TcScale sc = tc_scale(p.amax_g, p.amax_x);
#pragma unroll
  for (int t = 0; t < TAPS; ++t) {
    if (t >= ne) break;
    const int e = e0 + t;
    float* base = p.work ? p.work + ((long long)blockIdx.z * p.nentries + e) * p.Kp * p.C
                         : p.dw + (long long)p.out[e] * p.Kp * p.C;
    acc[t].each(lane, [&](int c, int h, float v0, float v1) {
      const int co = co0 + 8 * h;
      if (co >= p.Kp || c >= cleft) return;
      *reinterpret_cast<float2*>(base + (long long)co * p.C + citile * BNW + c) = make_float2(v0 * sc.fa * sc.fb, v1 * sc.fa * sc.fb);
    });
  }
}

// dw[t][j] = sum over the entries e with out[e] == t, then over the splits z, of work[(z * nentries + e) * plane + j]
struct WgradSum {
  int nentries, splits;
  int out[TC_MAX_TAPS];
};
__global__ void __launch_bounds__(256) wgrad_sum_kernel(const float* __restrict__ work, long long plane, int ntaps_out,
                                                        const WgradSum ws, float* __restrict__ dw) {
  for (long long i = blockIdx.x * 256LL + threadIdx.x; i < ntaps_out * plane; i += (long long)gridDim.x * 256) {
    const int t = (int)(i / plane);
    const long long j = i - t * plane;
    float a = 0.f;
    for (int e = 0; e < ws.nentries; ++e) {
      if (ws.out[e] != t) continue;
      for (int z = 0; z < ws.splits; ++z) a += work[((long long)z * ws.nentries + e) * plane + j];
    }
    dw[i] = a;
  }
}

// widths up to 104 take two entries per CTA (three accumulator sets of BNW / 2 registers fit the 168 of a thread)
constexpr int WG_PAIR_MAX_BN = 104;

// ci tile: as the forward's N tile (og_conv2d_tc), the smallest number of equal tiles of <= 128 columns, rounded up
// to the wgmma N step of 8, then to the next instantiated width
int tc_fit_width(int cols) {
  const int ntile = og_cdiv(cols, 128);
  const int bn8 = (og_cdiv(cols, ntile) + 7) / 8 * 8;
  for (int b : TC_BN_SET)
    if (b >= bn8) return b;
  return 128;
}

}  // namespace

// ------------------------------------------------------------------------------------------------
// C ABI.
//   xh/xl : source activations, fp16 hi / lo parts (og_prep_split), NHWC [SN][SH][SW][C] contiguous, C % 8 == 0
//           (SN = N, or 4*N for a space-to-depth source: phase block (a*2+b) holds x[:, a::2, b::2])
//   wh/wl : weights fp16 hi / lo, [ntaps_w][Kw][C] (og_pack_weights_f16 with transposed=1 for fprop), Kw rows
//   amax_x / amax_w : device words holding the float bits of max|.| of the two operand tensors (their scaling)
//   y     : output NHWC, channel count K (K % 4 == 0), element strides ysn/ysh/ysw, spatial bounds OHf x OWf
//   rows of the GEMM are the pixel grid N x OH x OW; output pixel (osy*h + opy, osx*w + opx)
//   taps  : ntaps quadruples (dh, dw, dn, weight tap index): source pixel = image n + dn, (h + dh, w + dw), zero
//           outside [0,SH)x[0,SW);  bias/act: optional epilogue (bias[K], OG_ACT_*)
// ------------------------------------------------------------------------------------------------
OG_API int og_conv2d_tc(const void* xh, const void* xl, const unsigned* amax_x, int N, int SN, int SH, int SW, int C,
                        const void* wh, const void* wl, const unsigned* amax_w, int ntaps_w, int Kw, float* y, int OH,
                        int OW, int K, long long ysn,
                        long long ysh, long long ysw, int OHf, int OWf, int osy, int osx, int opy, int opx,
                        const int* taps_host, int ntaps, const float* bias, int act,
                        float slope, cudaStream_t stream) {
  if (!xh || !xl || !wh || !wl || C % 8 || K % 4 || ntaps < 1 || ntaps > TC_MAX_TAPS) return (int)cudaErrorInvalidValue;
  if ((long long)N * OH * OW == 0) return 0;
  TcParams p;
  p.N = N; p.OH = OH; p.OW = OW;
  // patch shape: TW = largest power of two <= min(OW, 16); TH fills up to 128 / TW within OH; TN the rest
  int TW = 1;
  while (TW * 2 <= OW && TW * 2 <= 16) TW *= 2;
  int TH = 1;
  while (TH * 2 <= OH && TW * TH * 2 <= TC_BM) TH *= 2;
  int TN = TC_BM / (TW * TH);
  // a tile must not straddle two space-to-depth phase blocks of the source (image index n + dn)
  // N need not be a multiple of TN: GEMM rows are independent, the last tile's rows n >= N are never stored (row_ok),
  // whatever they read (zero fill past the tensor, or -- in a phase-stacked source -- images of the next phase block)
  p.TN = TN; p.TH = TH; p.TW = TW;
  p.bias = bias; p.act = act; p.slope = slope;
  p.tiles_w = og_cdiv(OW, TW);
  p.tiles_h = og_cdiv(OH, TH);
  const int tiles_n = og_cdiv(N, TN);
  p.cchunks = og_cdiv(C, TC_BK);
  p.klast = og_cdiv(C - (p.cchunks - 1) * TC_BK, 16);
  p.amax_a = amax_x; p.amax_b = amax_w;
  p.K = K;
  p.y = y; p.ysn = ysn; p.ysh = ysh; p.ysw = ysw;
  p.osy = osy; p.osx = osx; p.opy = opy; p.opx = opx;
  p.OHfull = OHf; p.OWfull = OWf;
  p.taps.n = ntaps;
  for (int i = 0; i < ntaps; ++i) {
    p.taps.dh[i] = taps_host[4 * i];
    p.taps.dw[i] = taps_host[4 * i + 1];
    p.taps.dn[i] = taps_host[4 * i + 2];
    p.taps.widx[i] = taps_host[4 * i + 3];
  }
  // N tile: whole K if it fits 128 columns (a consumer thread holds two sets of BN / 2 accumulators), else the
  // smallest number of equal tiles; the width is rounded up to the wgmma N step of 8, then to the next instantiated
  // width.  An output element's k-sum does not depend on the tile width, so neither do the results.
  const int BNsel = tc_fit_width(K);
  dim3 grid(tiles_n * p.tiles_h * p.tiles_w, og_cdiv(K, BNsel), 1);
  // few output tiles (small feature maps): split the reduction over gridDim.z (about two CTAs per SM in all); the
  // slices' partial outputs are summed in a fixed order afterwards (og_split_sum)
  p.ksplit = 1;
  p.work = nullptr;
  p.work_plane = (long long)N * OH * OW * K;
  {
    const long long tiles = (long long)grid.x * grid.y;
    const int nk_total = ntaps * p.cchunks;
    const bool dense = ysw == K && ysh == (long long)OWf * K && ysn == (long long)OHf * OWf * K && osy == 1 && osx == 1 &&
                       OH == OHf && OW == OWf;
    if (tiles < 100 && nk_total >= 16 && !bias && act == OG_ACT_NONE && dense) {
      int s = (int)((2 * og_num_sms() + tiles - 1) / tiles);
      if (s > nk_total / 8) s = nk_total / 8;
      if (s > 1) s = og_cdiv(nk_total, og_cdiv(nk_total, s));   // no slice without work: each writes its whole plane
      if (s > 1) {
        p.ksplit = s;
        grid.z = s;
      }
    }
  }

  // <= 32 output channels: [w_hi | w_lo] stacked along N (see conv_tc_kernel)
  const int stk_rows = K <= 16 ? 16 : 32;
  const bool stacked = BNsel == 32 && K <= 32;

  // row runs (conv_tc_rows_kernel): every chunk's A slot resident, two slot sets if they fit, then as deep a B ring
  // (2 to 4 stages) as the rest of the shared memory holds.  Runs of three taps only: the kernel columns of the 3x3
  // stride-1 layers, where it was measured.  The 7-tap runs of a 7x1 convolution and the 2-tap runs of a stride-2
  // input-gradient phase keep conv_tc_kernel (a longer first fill, a shallower B ring; not measured).
  p.run = tc_row_run(p.taps);
  p.asets = 1;
  p.bstages = 0;
  size_t rows_smem = 0;
  if (p.run == 3 && TN == 1 && TW % 8 == 0 && p.ksplit == 1) {
    const size_t slot = 2 * (size_t)(TH + p.run - 1) * TW * 128;
    const size_t bstage = (size_t)2 * (stacked ? stk_rows : BNsel) * 128;   // hi and lo (stacked: the two halves)
    if (2 * p.cchunks <= TC_ROWS_MAX_SLOTS && 2 * p.cchunks * slot + 2 * bstage + 1024 <= TC_ROWS_SMEM_LIMIT) p.asets = 2;
    const size_t aslots = (size_t)p.asets * p.cchunks * slot;
    if (p.asets * p.cchunks <= TC_ROWS_MAX_SLOTS && aslots + 2 * bstage + 1024 <= TC_ROWS_SMEM_LIMIT) {
      p.bstages = (int)((TC_ROWS_SMEM_LIMIT - 1024 - aslots) / bstage);
      if (p.bstages > TC_ROWS_MAX_BSTAGES) p.bstages = TC_ROWS_MAX_BSTAGES;
      rows_smem = aslots + p.bstages * bstage + 1024;
    }
  }
  const bool rows = p.bstages >= 2;

  CUtensorMap mah, mal, mbh, mbl;
  unsigned long long adims[4] = {(unsigned long long)C, (unsigned long long)SW, (unsigned long long)SH, (unsigned long long)SN};
  unsigned long long astr[3] = {(unsigned long long)C, (unsigned long long)SW * C, (unsigned long long)SH * SW * C};
  // a row run's box holds all of its taps' rows
  unsigned abox[4] = {(unsigned)TC_BK, (unsigned)TW, (unsigned)(rows ? TH + p.run - 1 : TH), (unsigned)TN};
  unsigned long long bdims[3] = {(unsigned long long)C, (unsigned long long)Kw, (unsigned long long)ntaps_w};
  unsigned long long bstr[2] = {(unsigned long long)C, (unsigned long long)Kw * C};
  unsigned bbox[3] = {(unsigned)TC_BK, (unsigned)(stacked ? stk_rows : BNsel), 1u};
  int rc;
  if ((rc = make_map(&mah, xh, 4, adims, astr, abox))) return rc;
  if ((rc = make_map(&mbh, wh, 3, bdims, bstr, bbox))) return rc;
  if ((rc = make_map(&mal, xl, 4, adims, astr, abox))) return rc;
  if ((rc = make_map(&mbl, wl, 3, bdims, bstr, bbox))) return rc;
  if (p.ksplit > 1) OG_CHECK(og_work_alloc(&p.work, (size_t)p.ksplit * p.work_plane, stream));
  if (!rows) {
    rc = tc_with_tile(BNsel, stacked, stk_rows, [&](auto bn, auto stk) {
      constexpr int BN = decltype(bn)::value;
      constexpr bool STACKED = decltype(stk)::value;
      constexpr size_t stage = 2 * TC_BM * 128 + (STACKED ? 1 : 2) * BN * 128;
      constexpr size_t smem = (size_t)tc_stages(stage) * stage + 1024;
      return tc_launch<conv_tc_kernel<BN, tc_stages(stage), STACKED>>(smem, grid, smem, stream, mah, mal, mbh, mbl, p);
    });
  } else {
    rc = tc_with_tile(BNsel, stacked, stk_rows, [&](auto bn, auto stk) {
      return tc_launch<conv_tc_rows_kernel<decltype(bn)::value, decltype(stk)::value>>(
          TC_ROWS_SMEM_LIMIT, grid, rows_smem, stream, mah, mal, mbh, mbl, p);
    });
  }
  if (p.ksplit > 1) {
    if (!rc) rc = og_split_sum(p.work, p.work_plane, p.ksplit, y, stream);
    const cudaError_t e = cudaFreeAsync(p.work, stream);
    if (!rc) rc = (int)e;
  }
  return rc;
}


// ------------------------------------------------------------------------------------------------
// weight gradient:  dw[t][co][ci] (fp32, [ntaps][Kp][C], zero-filled here) = sum_pixels G^T * X(shifted by tap t)
//   gh/gl : output gradient fp16 hi/lo, NHWC [GN][OH][OW][Kp] (og_prep_split; GN = N, or 4N space-to-depth blocks)
//   xh/xl : source activations fp16 hi/lo, NHWC [XN][SH][SW][C] (og_prep_split: plain, reflection-padded or
//           space-to-depth); both need 512 readable bytes after the last element (partial last channel slab)
//   amax_g / amax_x : operand scales as in og_conv2d_tc
//   entries: nentries quintuples (g image offset, dh, dw, x image offset, output tap):
//           dw[tap] += sum_{n,h,w} G[n + gdn, h, w, :]^T  X[n + xdn, h + dh, w + dw, :]   (out of range = 0)
// ------------------------------------------------------------------------------------------------
OG_API int og_conv2d_wgrad_tc(const void* gh, const void* gl, const unsigned* amax_g, int N, int GN, int OH, int OW,
                              int Kp, const void* xh, const void* xl, const unsigned* amax_x, int XN, int SH, int SW,
                              int C, float* dw,
                              int ntaps_out, const int* entries_host, int nentries, cudaStream_t stream) {
  if (!gh || !gl || !xh || !xl || nentries < 1 || nentries > TC_MAX_TAPS || Kp % 8 || C % 8)
    return (int)cudaErrorInvalidValue;
  OG_CHECK(cudaMemsetAsync(dw, 0, sizeof(float) * (size_t)ntaps_out * Kp * C, stream));
  if ((long long)N * OH * OW == 0) return 0;
  TcWgradParams p;
  p.N = N; p.OH = OH; p.OW = OW;
  // one stage = 64 pixels: a cw x chh x cn patch of the gradient grid (w fastest)
  int cw = 1;
  while (cw * 2 <= WG_PIX && OW % (cw * 2) == 0) cw *= 2;
  int chh = 1;
  while (cw * chh * 2 <= WG_PIX && OH % (chh * 2) == 0) chh *= 2;
  const int cn = WG_PIX / (cw * chh);
  // a last image group with n >= N contributes nothing as long as ONE operand is unstacked (TMA zero-fills it there)
  if (N % cn != 0 && GN != N && XN != N) return (int)cudaErrorInvalidValue;
  p.cw = cw; p.chh = chh; p.cn = cn;
  p.wchunks = OW / cw;
  p.hchunks = OH / chh;
  p.total_chunks = p.wchunks * p.hchunks * og_cdiv(N, cn);
  p.Kp = Kp; p.C = C; p.dw = dw;
  p.amax_g = amax_g; p.amax_x = amax_x;
  for (int i = 0; i < nentries; ++i) {
    p.gdn[i] = entries_host[5 * i];
    p.xdh[i] = entries_host[5 * i + 1];
    p.xdw[i] = entries_host[5 * i + 2];
    p.xdn[i] = entries_host[5 * i + 3];
    p.out[i] = entries_host[5 * i + 4];
  }
  const int cotiles = og_cdiv(Kp, TC_BM);
  const int BNsel = tc_fit_width(C);      // C = 200: 2 x 104 columns
  const int citiles = og_cdiv(C, BNsel);  // = ceil(C / 128), as many as 128-wide tiles would take
  p.cotiles = cotiles;
  // pixel splits: the CTAs are equal-sized and run one per SM, so fill at most two full waves (one CTA more would
  // cost a whole extra round); at least 8 chunks per CTA.  The count depends on the number of tiles and entries only,
  // not on the tile width or on how many entries a CTA shares, and an element's k-sum has the same stages and order
  // in every form: results do not depend on BNsel or on the entry pairing below
  int splits = 2 * og_num_sms() / (cotiles * citiles * nentries);
  if (splits < 1) splits = 1;
  int maxs = p.total_chunks / 8;
  if (maxs < 1) maxs = 1;
  if (splits > maxs) splits = maxs;
  p.chunks_per_cta = og_cdiv(p.total_chunks, splits);
  splits = og_cdiv(p.total_chunks, p.chunks_per_cta);
  // entries 2j and 2j + 1 share one CTA when they read the same G tile (equal image offset: every entry of a stride-1
  // or space-to-depth layer, the two column taps of an upsample phase): G is loaded once for both, a stage moves
  // 96 KB instead of 2 x 64 KB at BNW = 104.  The kernel is bound by those bytes, so pair only where
  // (waves) x (bytes per stage) drops: res-block conv1, 216 CTAs in 2 waves -> 120 in 1; not conv2 (252 -> 140, 2 waves)
  bool pair = BNsel <= WG_PAIR_MAX_BN && nentries > 1;
  for (int e = 0; e + 1 < nentries; e += 2) pair &= p.gdn[e] == p.gdn[e + 1];
  // OG_WGRAD_PAIR=0 / 1: never / always pair where the entries allow it (the results are the same)
  const char* pair_env = getenv("OG_WGRAD_PAIR");
  if (pair_env && atoi(pair_env) == 0) pair = false;
  if (pair && !pair_env) {
    const int nsb = og_cdiv(BNsel, WG_CH), sms = og_num_sms();
    const long long waves1 = og_cdiv((long long)cotiles * citiles * nentries * splits, sms);
    const long long waves2 = og_cdiv((long long)cotiles * citiles * og_cdiv(nentries, 2) * splits, sms);
    pair = waves2 * (4 + 4 * nsb) < waves1 * (4 + 2 * nsb);   // G: 2 slabs, X: nsb slabs per entry (hi and lo alike)
  }
  p.nentries = nentries;
  dim3 grid(cotiles * citiles, pair ? og_cdiv(nentries, 2) : nentries, splits);
  CUtensorMap mgh, mgl, mxh, mxl;
  // [slab][n][h][w][64 channels of the slab]: the slab dimension strides by 64 halves inside a pixel's channel vector
  unsigned long long gd[5] = {(unsigned long long)WG_CH, (unsigned long long)OW, (unsigned long long)OH,
                              (unsigned long long)GN, (unsigned long long)og_cdiv(Kp, WG_CH)};
  unsigned long long gs[4] = {(unsigned long long)Kp, (unsigned long long)OW * Kp, (unsigned long long)OH * OW * Kp,
                              (unsigned long long)WG_CH};
  unsigned gb[5] = {(unsigned)WG_CH, (unsigned)cw, (unsigned)chh, (unsigned)cn, 2u};
  // X: [slab of the tile][n][h][w][channel of the whole pixel vector]; a tile's box starts at channel citile * BNsel
  // and its slab s holds channels from there + 64 s (those >= C are never stored: zero-filled in the first slab,
  // read from the next pixel -- or the readable bytes after the tensor -- in the others)
  const int xslabs = (BNsel + WG_CH - 1) / WG_CH;
  unsigned long long xd[5] = {(unsigned long long)C, (unsigned long long)SW, (unsigned long long)SH,
                              (unsigned long long)XN, (unsigned long long)xslabs};
  unsigned long long xs[4] = {(unsigned long long)C, (unsigned long long)SW * C, (unsigned long long)SH * SW * C,
                              (unsigned long long)WG_CH};
  unsigned xb[5] = {(unsigned)WG_CH, (unsigned)cw, (unsigned)chh, (unsigned)cn, (unsigned)xslabs};
  int rc;
  if ((rc = make_map(&mgh, gh, 5, gd, gs, gb))) return rc;
  if ((rc = make_map(&mxh, xh, 5, xd, xs, xb))) return rc;
  if ((rc = make_map(&mgl, gl, 5, gd, gs, gb))) return rc;
  if ((rc = make_map(&mxl, xl, 5, xd, xs, xb))) return rc;
  // every element of an output tap has one writer unless pixel splits or several entries meet there: then each
  // (split, entry) writes its own plane of a workspace, summed in a fixed order by wgrad_sum_kernel
  bool shared_out = splits > 1;
  for (int i = 0; i < nentries; ++i)
    for (int j = 0; j < i; ++j) shared_out |= p.out[i] == p.out[j];
  p.work = nullptr;
  const long long plane = (long long)Kp * C;
  if (shared_out) OG_CHECK(og_work_alloc(&p.work, (size_t)splits * nentries * plane, stream));
  const auto launch = [&](auto bnw, auto taps) {
    constexpr int BNW = decltype(bnw)::value, TAPS = decltype(taps)::value;
    constexpr size_t stage = 2 * 2 * WG_SLAB + TAPS * 2 * ((BNW + WG_CH - 1) / WG_CH) * WG_SLAB;
    constexpr size_t smem = (size_t)tc_stages(stage) * stage + 1024;
    return tc_launch<conv_tc_wgrad_wide_kernel<BNW, tc_stages(stage), TAPS>>(smem, grid, smem, stream, mgh, mgl, mxh,
                                                                            mxl, p);
  };
  rc = tc_with_width(BNsel, [&](auto bnw) {
    if constexpr (decltype(bnw)::value <= WG_PAIR_MAX_BN)
      if (pair) return launch(bnw, std::integral_constant<int, 2>());
    return launch(bnw, std::integral_constant<int, 1>());
  });
  if (shared_out) {
    if (!rc) {
      WgradSum ws;
      ws.nentries = nentries;
      ws.splits = splits;
      for (int i = 0; i < nentries; ++i) ws.out[i] = p.out[i];
      const long long total = (long long)ntaps_out * plane;
      long long b = (total + 255) / 256;
      if (b > 65535) b = 65535;
      wgrad_sum_kernel<<<(int)b, 256, 0, stream>>>(p.work, plane, ntaps_out, ws, dw);
      rc = (int)cudaGetLastError();
    }
    const cudaError_t e = cudaFreeAsync(p.work, stream);
    if (!rc) rc = (int)e;
  }
  return rc;
}
