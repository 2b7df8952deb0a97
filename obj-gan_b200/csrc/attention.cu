// Word- and object-level attention of GlobalAttention.py plus the mask-paint of miscc/utils.py,
// as fused bandwidth-bound kernels.  All "ref:" paths are under /root/reference/image_generation/.
//
//   og_words_proj*        conv1x1 of the word embeddings (ref: GlobalAttention.py:97-100, 151-154)
//   og_att_general_*      GlobalAttentionGeneral / ATT_NET    (ref: GlobalAttention.py:83-122)
//   og_bu_att_*           GlobalBUAttentionGeneral / BT_ATT_NET (ref: GlobalAttention.py:136-181)
//   og_paint_max_*        pprocess_bt_attns                   (ref: miscc/utils.py:401-413)
//   og_func_attention_fwd func_attention (DAMSM)              (ref: GlobalAttention.py:32-70)
//
// The grid attention streams h_code once (4*C bytes / query), writes the context once and the
// attention map once: algorithmic bytes 4*Q*(2C + L) per image (SURVEY.md 8d).
#include "common.cuh"

constexpr int LMAX = 32;   // max caption length handled in registers (reference uses 12..18)

// two independent fp32 FMAs on a pair of lanes
__device__ __forceinline__ float2 ffma2(float2 a, float2 b, float2 c) {
  return make_float2(fmaf(a.x, b.x, c.x), fmaf(a.y, b.y, c.y));
}
constexpr int ATT_Q = 128; // queries per block

// The grid-attention kernels stage rows of `cs` floats (row stride cs, cs % 4 == 0) in shared tiles of pitch cs + 1.
// Both walks move 16 bytes per thread and step, and advance the thread's (row, quad) position by ATT_Q quads without
// a division.
// Rows [0, nq) of g -> tile rows [0, nq); with ZERO_TAIL, tile rows [nq, ATT_Q) become zeros.
template <bool ZERO_TAIL>
__device__ __forceinline__ void rows_to_tile(float* tile, const float* __restrict__ g, int cs, int nq) {
  const int pitch = cs + 1, cs4 = cs >> 2, t = threadIdx.x;
  for (int r = t / cs4, c4 = t - (t / cs4) * cs4, i = t; i < (ZERO_TAIL ? ATT_Q : nq) * cs4; i += ATT_Q) {
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (!ZERO_TAIL || r < nq) v = ldg4(g + i * 4);
    float* d = tile + r * pitch + c4 * 4;
    d[0] = v.x; d[1] = v.y; d[2] = v.z; d[3] = v.w;
    c4 += ATT_Q % cs4;
    r += ATT_Q / cs4;
    if (c4 >= cs4) { c4 -= cs4; ++r; }
  }
}
// Tile rows [0, nq) -> rows [0, nq) of g.
__device__ __forceinline__ void tile_to_rows(float* __restrict__ g, const float* tile, int cs, int nq) {
  const int pitch = cs + 1, cs4 = cs >> 2, t = threadIdx.x;
  for (int r = t / cs4, c4 = t - (t / cs4) * cs4, i = t; i < nq * cs4; i += ATT_Q) {
    const float* d = tile + r * pitch + c4 * 4;
    st4(g + i * 4, make_float4(d[0], d[1], d[2], d[3]));
    c4 += ATT_Q % cs4;
    r += ATT_Q / cs4;
    if (c4 >= cs4) { c4 -= cs4; ++r; }
  }
}

// src[b][c][l] = sum_k W[c][k] * words[b][k][l]
__global__ void words_proj_kernel(const float* __restrict__ words, const float* __restrict__ W, int idf, int cdf,
                                  int L, float* __restrict__ src) {
  const int b = blockIdx.y;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < idf * L; i += gridDim.x * blockDim.x) {
    int c = i / L, l = i - c * L;
    const float* wr = W + c * cdf;
    const float* wd = words + (long long)b * cdf * L + l;
    float acc = 0.f;
    for (int k = 0; k < cdf; ++k) acc = fmaf(__ldg(wr + k), __ldg(wd + (long long)k * L), acc);
    src[((long long)b * idf + c) * L + l] = acc;
  }
}
// gW[c][k] += sum_b sum_l gsrc[b][c][l] * words[b][k][l];   gwords[b][k][l] = sum_c W[c][k] * gsrc[b][c][l]
__global__ void words_proj_bwd_w_kernel(const float* __restrict__ words, const float* __restrict__ gsrc, int B,
                                        int idf, int cdf, int L, float* __restrict__ gW, int accumulate) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < idf * cdf; i += gridDim.x * blockDim.x) {
    int c = i / cdf, k = i - c * cdf;
    float acc = 0.f;
    for (int b = 0; b < B; ++b) {
      const float* gs = gsrc + ((long long)b * idf + c) * L;
      const float* wd = words + ((long long)b * cdf + k) * L;
      for (int l = 0; l < L; ++l) acc = fmaf(gs[l], wd[l], acc);
    }
    gW[i] = accumulate ? gW[i] + acc : acc;
  }
}
__global__ void words_proj_bwd_x_kernel(const float* __restrict__ W, const float* __restrict__ gsrc, int idf, int cdf,
                                        int L, float* __restrict__ gwords) {
  const int b = blockIdx.y;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < cdf * L; i += gridDim.x * blockDim.x) {
    int k = i / L, l = i - k * L;
    float acc = 0.f;
    for (int c = 0; c < idf; ++c) acc = fmaf(W[c * cdf + k], gsrc[((long long)b * idf + c) * L + l], acc);
    gwords[(long long)b * cdf * L + i] = acc;
  }
}

OG_API int og_words_proj(const float* words, const float* W, int B, int idf, int cdf, int L, float* src,
                         cudaStream_t stream) {
  if (B == 0) return 0;
  dim3 grid(og_cdiv(idf * L, 128), B);
  words_proj_kernel<<<grid, 128, 0, stream>>>(words, W, idf, cdf, L, src);
  OG_RETURN_LAST_ERROR();
}
OG_API int og_words_proj_bwd(const float* words, const float* W, const float* gsrc, int B, int idf, int cdf, int L,
                             float* gW, int accumulate, float* gwords, cudaStream_t stream) {
  if (gW) words_proj_bwd_w_kernel<<<og_cdiv(idf * cdf, 128), 128, 0, stream>>>(words, gsrc, B, idf, cdf, L, gW, accumulate);
  if (gwords && B > 0) {
    dim3 grid(og_cdiv(cdf * L, 128), B);
    words_proj_bwd_x_kernel<<<grid, 128, 0, stream>>>(W, gsrc, idf, cdf, L, gwords);
  }
  OG_RETURN_LAST_ERROR();
}

// ---------------------------------------------------------------------------------------------
// grid attention forward.  h: [B][Q][cs] (NHWC, idf real channels, row stride cs), src: [B][idf][L],
// mask: [B][L] bytes (1 = padding word) or null.  wc: [B][Q][cs] (pad lanes zeroed), attn: [B][L][Q].
// Mask quirk (ref: GlobalAttention.py:108): row (b, q) uses the caption mask of sample (b*Q + q) mod B.
// ---------------------------------------------------------------------------------------------
template <int LM>
__global__ void __launch_bounds__(ATT_Q, 7)
att_general_fwd_kernel(const float* __restrict__ h, const float* __restrict__ src,
                       const unsigned char* __restrict__ mask, int B, int Q, int idf, int cs, int L,
                       float* __restrict__ wc, float* __restrict__ attn) {
  // The word projections src[c][0..L) live in shared memory as rows of LM floats (zero padded) and are read with
  // 128-bit broadcast loads: one LDS.128 feeds four FMAs.
  extern __shared__ __align__(16) float smem[];
  const int pitch = cs + 1;
  float* ssrc = smem;                    // [idf][LM]
  float* tile = smem + idf * LM;         // [ATT_Q][pitch]
  const int b = blockIdx.y, q0 = blockIdx.x * ATT_Q, t = threadIdx.x;
  const int nq = min(ATT_Q, Q - q0);
  for (int i = t; i < idf * LM; i += ATT_Q) {
    int c = i / LM, l = i - c * LM;
    ssrc[i] = l < L ? src[((long long)b * idf + c) * L + l] : 0.f;
  }
  rows_to_tile<false>(tile, h + ((long long)b * Q + q0) * cs, cs, nq);
  __syncthreads();
  float2 s2[LM / 2];
#pragma unroll
  for (int l = 0; l < LM / 2; ++l) s2[l] = make_float2(0.f, 0.f);
  // rows past nq hold stale shared memory: they are computed but never stored
  for (int c = 0; c < idf; ++c) {
    const float hv = tile[t * pitch + c];
    const float2 hv2 = make_float2(hv, hv);
    const float4* sr = reinterpret_cast<const float4*>(ssrc + c * LM);
#pragma unroll
    for (int l4 = 0; l4 < LM / 4; ++l4) {
      const float4 w = sr[l4];
      s2[2 * l4] = ffma2(hv2, make_float2(w.x, w.y), s2[2 * l4]);
      s2[2 * l4 + 1] = ffma2(hv2, make_float2(w.z, w.w), s2[2 * l4 + 1]);
    }
  }
  {
    const int q = q0 + t;
    const bool live = t < nq;
    float s[LM];
#pragma unroll
    for (int l = 0; l < LM / 2; ++l) {
      s[2 * l] = s2[l].x;
      s[2 * l + 1] = s2[l].y;
    }
    float mx = -INFINITY;
    if (mask && live) {
      const unsigned char* mr = mask + (((long long)b * Q + q) % B) * L;
#pragma unroll
      for (int l = 0; l < LM; ++l)
        if (l < L && mr[l]) s[l] = -INFINITY;
    }
#pragma unroll
    for (int l = 0; l < LM; ++l)
      if (l < L) mx = fmaxf(mx, s[l]);
    float sum = 0.f;
#pragma unroll
    for (int l = 0; l < LM; ++l) {
      s[l] = l < L ? expf(s[l] - mx) : 0.f;
      sum += s[l];
    }
    const float inv = 1.f / sum;
#pragma unroll
    for (int l = 0; l < LM; ++l) {
      s[l] *= inv;
      if (l < L && live) attn[((long long)b * L + l) * Q + q] = s[l];
    }
#pragma unroll
    for (int l = 0; l < LM / 2; ++l) s2[l] = make_float2(s[2 * l], s[2 * l + 1]);
  }
  for (int c = 0; c < cs; ++c) {
    float acc = 0.f;
    if (c < idf) {
      const float4* sr = reinterpret_cast<const float4*>(ssrc + c * LM);
      float2 a2 = make_float2(0.f, 0.f), b2 = a2;   // four interleaved partial sums: short dependent FMA chains
#pragma unroll
      for (int l4 = 0; l4 < LM / 4; ++l4) {
        const float4 w = sr[l4];
        a2 = ffma2(make_float2(w.x, w.y), s2[2 * l4], a2);
        b2 = ffma2(make_float2(w.z, w.w), s2[2 * l4 + 1], b2);
      }
      acc = (a2.x + b2.x) + (a2.y + b2.y);
    }
    tile[t * pitch + c] = acc;
  }
  __syncthreads();
  tile_to_rows(wc + ((long long)b * Q + q0) * cs, tile, cs, nq);
}

// attention_tc.cu: the tensor-core (wgmma) kernel for the large maps of the hot path; -1 = shape outside its envelope
extern "C" int og_att_general_fwd_tc(const float* h, const float* src, const unsigned char* mask, int B, int Q, int idf,
                                     int cs, int L, float* wc, float* attn, cudaStream_t stream);

OG_API int og_att_general_fwd(const float* h, const float* src, const unsigned char* mask, int B, int Q, int idf,
                              int cs, int L, float* wc, float* attn, cudaStream_t stream) {
  if (L > LMAX || cs % 4 || idf > cs) return (int)cudaErrorInvalidValue;
  if (B == 0 || Q == 0) return 0;
  if (Q >= 4096) {
    const int rc = og_att_general_fwd_tc(h, src, mask, B, Q, idf, cs, L, wc, attn, stream);
    if (rc >= 0) return rc;
  }
  const int LMsel = L <= 20 ? 20 : LMAX;
  size_t sm = sizeof(float) * (ATT_Q * (cs + 1) + idf * LMsel);
  dim3 grid(og_cdiv(Q, ATT_Q), B);
  if (L <= 20) {   // captions of the hot path have 12..18 words: keep the per-thread score vector small
    if (sm > 48 * 1024)
      OG_CHECK(cudaFuncSetAttribute(att_general_fwd_kernel<20>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm));
    att_general_fwd_kernel<20><<<grid, ATT_Q, sm, stream>>>(h, src, mask, B, Q, idf, cs, L, wc, attn);
  } else {
    OG_CHECK(cudaFuncSetAttribute(att_general_fwd_kernel<LMAX>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm));
    att_general_fwd_kernel<LMAX><<<grid, ATT_Q, sm, stream>>>(h, src, mask, B, Q, idf, cs, L, wc, attn);
  }
  OG_RETURN_LAST_ERROR();
}

// backward: g_h [B][Q][cs]; g_src: the CTA's contribution to the image's [idf][L] gradient goes to plane blockIdx.x of
// [gridDim.x][B][idf][L], which the launcher adds in a fixed order (og_split_sum).
// The attention map is an output the networks only visualise, so no gradient flows into it.
__global__ void __launch_bounds__(ATT_Q) att_general_bwd_kernel(const float* __restrict__ h,
                                                                const float* __restrict__ src,
                                                                const float* __restrict__ attn,
                                                                const float* __restrict__ g_wc, int B, int Q,
                                                                int idf, int cs, int L, float* __restrict__ g_h,
                                                                float* __restrict__ g_src) {
  extern __shared__ float smem[];
  const int pitch = cs + 1;
  float* th = smem;                         // [ATT_Q][pitch]  h rows, later g_h rows
  float* tg = th + ATT_Q * pitch;           // [ATT_Q][pitch]  g_wc rows
  float* sA = tg + ATT_Q * pitch;           // [ATT_Q][L]
  float* sG = sA + ATT_Q * L;               // [ATT_Q][L]     gS
  float* ssrc = sG + ATT_Q * L;             // [idf][L]
  const int b = blockIdx.y, q0 = blockIdx.x * ATT_Q, t = threadIdx.x;
  const int nq = min(ATT_Q, Q - q0);
  for (int i = t; i < idf * L; i += ATT_Q) ssrc[i] = src[(long long)b * idf * L + i];
  rows_to_tile<false>(th, h + ((long long)b * Q + q0) * cs, cs, nq);
  rows_to_tile<false>(tg, g_wc + ((long long)b * Q + q0) * cs, cs, nq);
  __syncthreads();
  float gS[LMAX];
  if (t < nq) {
    const int q = q0 + t;
    float A[LMAX], gA[LMAX];
#pragma unroll
    for (int l = 0; l < LMAX; ++l) {
      A[l] = 0.f;
      gA[l] = 0.f;
      if (l < L) A[l] = attn[((long long)b * L + l) * Q + q];
    }
    const float* grow = tg + t * pitch;
    for (int c = 0; c < idf; ++c) {
      float gv = grow[c];
      const float* sr = ssrc + c * L;
#pragma unroll
      for (int l = 0; l < LMAX; ++l)
        if (l < L) gA[l] = fmaf(gv, sr[l], gA[l]);
    }
    float dot = 0.f;
#pragma unroll
    for (int l = 0; l < LMAX; ++l)
      if (l < L) dot = fmaf(gA[l], A[l], dot);
#pragma unroll
    for (int l = 0; l < LMAX; ++l) {
      gS[l] = 0.f;
      if (l < L) {
        gS[l] = A[l] * (gA[l] - dot);
        sA[t * L + l] = A[l];
        sG[t * L + l] = gS[l];
      }
    }
  } else {
    for (int l = 0; l < L; ++l) {
      sA[t * L + l] = 0.f;
      sG[t * L + l] = 0.f;
    }
    for (int c = 0; c < cs; ++c) {
      th[t * pitch + c] = 0.f;
      tg[t * pitch + c] = 0.f;
    }
  }
  __syncthreads();
  // block-partial g_src[c][l] = sum_t h[t][c] * gS[t][l] + g_wc[t][c] * A[t][l]
  for (int i = t; i < idf * L; i += ATT_Q) {
    int c = i / L, l = i - c * L;
    float acc = 0.f;
    for (int r = 0; r < ATT_Q; ++r)
      acc = fmaf(th[r * pitch + c], sG[r * L + l], fmaf(tg[r * pitch + c], sA[r * L + l], acc));
    g_src[((long long)blockIdx.x * B + b) * idf * L + i] = acc;
  }
  __syncthreads();
  if (t < nq) {
    float* row = th + t * pitch;
    for (int c = 0; c < cs; ++c) {
      float acc = 0.f;
      if (c < idf) {
        const float* sr = ssrc + c * L;
#pragma unroll
        for (int l = 0; l < LMAX; ++l)
          if (l < L) acc = fmaf(gS[l], sr[l], acc);
      }
      row[c] = acc;
    }
  }
  __syncthreads();
  tile_to_rows(g_h + ((long long)b * Q + q0) * cs, th, cs, nq);
}

// Backward for L <= 20 (the hot path): same arithmetic as above with the forward kernel's register blocking --
// word-projection rows of 20 floats read with broadcast LDS.128, paired FMAs, no `l < L` predicates (rows are zero
// padded).  Phases: (A) gA = g_wc . src, softmax backward -> gS in registers; (C) the block's contribution to g_src
// ([48 c x 2 halves of 10 words] threads, reduction over the block's 128 queries from shared memory), stored to plane
// blockIdx.x as above; (B) g_h rows.
__global__ void __launch_bounds__(ATT_Q, 3)
att_general_bwd20_kernel(const float* __restrict__ h, const float* __restrict__ src, const float* __restrict__ attn,
                         const float* __restrict__ g_wc, int B, int Q, int idf, int cs, int L,
                         float* __restrict__ g_h, float* __restrict__ g_src) {
  constexpr int LM = 20;
  extern __shared__ __align__(16) float smem[];
  const int pitch = cs + 1;
  float* ssrc = smem;                         // [idf][LM] zero padded
  float* sA = ssrc + idf * LM;                // [ATT_Q][LM]
  float* sG = sA + ATT_Q * LM;                // [ATT_Q][LM]
  float* th = sG + ATT_Q * LM;                // [ATT_Q][pitch]  h rows, later g_h rows
  float* tg = th + ATT_Q * pitch;             // [ATT_Q][pitch]  g_wc rows
  const int b = blockIdx.y, q0 = blockIdx.x * ATT_Q, t = threadIdx.x;
  const int nq = min(ATT_Q, Q - q0);
  for (int i = t; i < idf * LM; i += ATT_Q) {
    const int c = i / LM, l = i - c * LM;
    ssrc[i] = l < L ? src[((long long)b * idf + c) * L + l] : 0.f;
  }
  rows_to_tile<true>(th, h + ((long long)b * Q + q0) * cs, cs, nq);
  rows_to_tile<true>(tg, g_wc + ((long long)b * Q + q0) * cs, cs, nq);
  __syncthreads();
  // (A) gA[l] = sum_c g_wc[q][c] * src[c][l]
  float2 s2[LM / 2];
#pragma unroll
  for (int l = 0; l < LM / 2; ++l) s2[l] = make_float2(0.f, 0.f);
  {
    const float* grow = tg + t * pitch;
    for (int c = 0; c < idf; ++c) {
      const float gv = grow[c];
      const float2 g2 = make_float2(gv, gv);
      const float4* sr = reinterpret_cast<const float4*>(ssrc + c * LM);
#pragma unroll
      for (int l4 = 0; l4 < LM / 4; ++l4) {
        const float4 w = sr[l4];
        s2[2 * l4] = ffma2(g2, make_float2(w.x, w.y), s2[2 * l4]);
        s2[2 * l4 + 1] = ffma2(g2, make_float2(w.z, w.w), s2[2 * l4 + 1]);
      }
    }
  }
  {
    float A[LM], gA[LM];
    const int q = q0 + t;
    const bool live = t < nq;
#pragma unroll
    for (int l = 0; l < LM / 2; ++l) {
      gA[2 * l] = s2[l].x;
      gA[2 * l + 1] = s2[l].y;
    }
    float dot = 0.f;
#pragma unroll
    for (int l = 0; l < LM; ++l) {
      A[l] = 0.f;
      if (l < L && live) A[l] = attn[((long long)b * L + l) * Q + q];
      dot = fmaf(gA[l], A[l], dot);
    }
#pragma unroll
    for (int l = 0; l < LM; ++l) gA[l] = A[l] * (gA[l] - dot);          // gS (zero for dead rows and l >= L)
#pragma unroll
    for (int l4 = 0; l4 < LM / 4; ++l4) {
      *reinterpret_cast<float4*>(sA + t * LM + 4 * l4) = make_float4(A[4 * l4], A[4 * l4 + 1], A[4 * l4 + 2], A[4 * l4 + 3]);
      *reinterpret_cast<float4*>(sG + t * LM + 4 * l4) =
          make_float4(gA[4 * l4], gA[4 * l4 + 1], gA[4 * l4 + 2], gA[4 * l4 + 3]);
    }
#pragma unroll
    for (int l = 0; l < LM / 2; ++l) s2[l] = make_float2(gA[2 * l], gA[2 * l + 1]);
  }
  __syncthreads();
  // (C) block-partial g_src[c][l] = sum_r h[r][c] * gS[r][l] + g_wc[r][c] * A[r][l]
  if (t < 2 * idf && idf <= 64) {
    const int c = t % idf, half = t / idf;              // words [10 * half, 10 * half + 10)
    float2 acc[5];
#pragma unroll
    for (int k = 0; k < 5; ++k) acc[k] = make_float2(0.f, 0.f);
    for (int r = 0; r < ATT_Q; ++r) {
      const float hv = th[r * pitch + c], gv = tg[r * pitch + c];
      const float2 h2 = make_float2(hv, hv), g2 = make_float2(gv, gv);
      const float2* pg = reinterpret_cast<const float2*>(sG + r * LM + 10 * half);
      const float2* pa = reinterpret_cast<const float2*>(sA + r * LM + 10 * half);
#pragma unroll
      for (int k = 0; k < 5; ++k) acc[k] = ffma2(h2, pg[k], ffma2(g2, pa[k], acc[k]));
    }
    float* dst = g_src + (((long long)blockIdx.x * B + b) * idf + c) * L;
#pragma unroll
    for (int k = 0; k < 5; ++k) {
      const int l = 10 * half + 2 * k;
      if (l < L) dst[l] = acc[k].x;
      if (l + 1 < L) dst[l + 1] = acc[k].y;
    }
  }
  __syncthreads();
  // (B) g_h[c] = sum_l gS[l] * src[c][l], written over the h rows
  {
    float* row = th + t * pitch;
    for (int c = 0; c < cs; ++c) {
      float acc = 0.f;
      if (c < idf) {
        const float4* sr = reinterpret_cast<const float4*>(ssrc + c * LM);
        float2 a2 = make_float2(0.f, 0.f), b2 = a2;
#pragma unroll
        for (int l4 = 0; l4 < LM / 4; ++l4) {
          const float4 w = sr[l4];
          a2 = ffma2(make_float2(w.x, w.y), s2[2 * l4], a2);
          b2 = ffma2(make_float2(w.z, w.w), s2[2 * l4 + 1], b2);
        }
        acc = (a2.x + b2.x) + (a2.y + b2.y);
      }
      row[c] = acc;
    }
  }
  __syncthreads();
  tile_to_rows(g_h + ((long long)b * Q + q0) * cs, th, cs, nq);
}

extern "C" int og_att_general_bwd_tc(const float* h, const float* src, const float* attn, const float* g_wc, int B, int Q,
                                     int idf, int cs, int L, float* g_h, float* g_src, cudaStream_t stream);

OG_API int og_att_general_bwd(const float* h, const float* src, const float* attn, const float* g_wc, int B, int Q,
                              int idf, int cs, int L, float* g_h, float* g_src, cudaStream_t stream) {
  if (L > LMAX || cs % 4 || idf > cs) return (int)cudaErrorInvalidValue;
  if (B == 0 || Q == 0) return (int)cudaMemsetAsync(g_src, 0, sizeof(float) * (size_t)B * idf * L, stream);
  if (Q >= 4096) {
    const int rc = og_att_general_bwd_tc(h, src, attn, g_wc, B, Q, idf, cs, L, g_h, g_src, stream);
    if (rc >= 0) return rc;
  }
  const bool k20 = L <= 20 && idf <= 64;
  const size_t sm20 = sizeof(float) * ((size_t)idf * 20 + 2 * ATT_Q * 20 + 2 * (size_t)ATT_Q * (cs + 1));
  const size_t sm = sizeof(float) * (2 * ATT_Q * (cs + 1) + 2 * ATT_Q * L + idf * L);
  static size_t configured20 = 0;
  if (k20 && sm20 > configured20) {
    OG_CHECK(cudaFuncSetAttribute(att_general_bwd20_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm20));
    configured20 = sm20;
  }
  if (!k20) OG_CHECK(cudaFuncSetAttribute(att_general_bwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm));
  const dim3 grid(og_cdiv(Q, ATT_Q), B);
  float* work = g_src;                   // one CTA per image: its plane is g_src itself
  if (grid.x > 1) OG_CHECK(og_work_alloc(&work, (size_t)grid.x * B * idf * L, stream));
  if (k20)
    att_general_bwd20_kernel<<<grid, ATT_Q, sm20, stream>>>(h, src, attn, g_wc, B, Q, idf, cs, L, g_h, work);
  else
    att_general_bwd_kernel<<<grid, ATT_Q, sm, stream>>>(h, src, attn, g_wc, B, Q, idf, cs, L, g_h, work);
  int rc = (int)cudaGetLastError();
  if (grid.x > 1) {
    if (!rc) rc = og_split_sum(work, (long long)B * idf * L, (int)grid.x, g_src, stream);
    const cudaError_t e = cudaFreeAsync(work, stream);
    if (!rc) rc = (int)e;
  }
  return rc;
}

// ---------------------------------------------------------------------------------------------
// bottom-up (object) attention: one block per sample.
// labels [B][E][R] (E = 50 GloVe dims), glove [B][E][L], src [B][idf][L], mask [B][L] bytes or null
// -> wc [B][idf][R], attn [B][L][R].   Cosine normalisation when `norm` (cfg.TRAIN.BUATTN_NORM).
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(128) bu_att_fwd_kernel(const float* __restrict__ labels,
                                                         const float* __restrict__ glove,
                                                         const float* __restrict__ src,
                                                         const unsigned char* __restrict__ mask, int B, int E, int R,
                                                         int L, int idf, int norm, float eps, float* __restrict__ wc,
                                                         float* __restrict__ attn) {
  extern __shared__ float smem[];
  float* S = smem;          // [R][L]
  float* nl = S + R * L;    // [R]
  float* ng = nl + R;       // [L]
  const int b = blockIdx.x, t = threadIdx.x;
  const float* lb = labels + (long long)b * E * R;
  const float* gb = glove + (long long)b * E * L;
  for (int r = t; r < R; r += 128) {
    float a = 0.f;
    for (int e = 0; e < E; ++e) a = fmaf(lb[e * R + r], lb[e * R + r], a);
    nl[r] = sqrtf(a);
  }
  for (int l = t; l < L; l += 128) {
    float a = 0.f;
    for (int e = 0; e < E; ++e) a = fmaf(gb[e * L + l], gb[e * L + l], a);
    ng[l] = sqrtf(a);
  }
  __syncthreads();
  for (int i = t; i < R * L; i += 128) {
    int r = i / L, l = i - r * L;
    float a = 0.f;
    for (int e = 0; e < E; ++e) a = fmaf(lb[e * R + r], gb[e * L + l], a);
    if (norm) a = a / fmaxf(nl[r] * ng[l], eps);
    if (mask && mask[(((long long)b * R + r) % B) * L + l]) a = -INFINITY;
    S[i] = a;
  }
  __syncthreads();
  for (int r = t; r < R; r += 128) {
    float mx = -INFINITY;
    for (int l = 0; l < L; ++l) mx = fmaxf(mx, S[r * L + l]);
    float sum = 0.f;
    for (int l = 0; l < L; ++l) {
      float e = expf(S[r * L + l] - mx);
      S[r * L + l] = e;
      sum += e;
    }
    float inv = 1.f / sum;
    for (int l = 0; l < L; ++l) {
      float a = S[r * L + l] * inv;
      S[r * L + l] = a;
      attn[((long long)b * L + l) * R + r] = a;
    }
  }
  __syncthreads();
  const float* sb = src + (long long)b * idf * L;
  for (int i = t; i < idf * R; i += 128) {
    int c = i / R, r = i - c * R;
    float a = 0.f;
    for (int l = 0; l < L; ++l) a = fmaf(sb[c * L + l], S[r * L + l], a);
    wc[(long long)b * idf * R + i] = a;
  }
}
OG_API int og_bu_att_fwd(const float* labels, const float* glove, const float* src, const unsigned char* mask, int B,
                         int E, int R, int L, int idf, int norm, float eps, float* wc, float* attn,
                         cudaStream_t stream) {
  if (B == 0 || R == 0) return 0;
  size_t sm = sizeof(float) * (R * L + R + L);
  bu_att_fwd_kernel<<<B, 128, sm, stream>>>(labels, glove, src, mask, B, E, R, L, idf, norm, eps, wc, attn);
  OG_RETURN_LAST_ERROR();
}
// the attention weights depend only on constants (labels, GloVe), so the only gradient path is
// g_src[b][c][l] = sum_r g_wc[b][c][r] * attn[b][l][r]
__global__ void bu_att_bwd_kernel(const float* __restrict__ attn, const float* __restrict__ g_wc, int R, int L,
                                  int idf, float* __restrict__ g_src) {
  const int b = blockIdx.x;
  for (int i = threadIdx.x; i < idf * L; i += blockDim.x) {
    int c = i / L, l = i - c * L;
    float a = 0.f;
    for (int r = 0; r < R; ++r)
      a = fmaf(g_wc[((long long)b * idf + c) * R + r], attn[((long long)b * L + l) * R + r], a);
    g_src[(long long)b * idf * L + i] = a;
  }
}
OG_API int og_bu_att_bwd(const float* attn, const float* g_wc, int B, int R, int L, int idf, float* g_src,
                         cudaStream_t stream) {
  if (B == 0) return 0;
  bu_att_bwd_kernel<<<B, 128, 0, stream>>>(attn, g_wc, R, L, idf, g_src);
  OG_RETURN_LAST_ERROR();
}

// ---------------------------------------------------------------------------------------------
// mask paint: out[b][p][doff + k] = max_{r < R} f[b][k][r] * m[b][r][p]
// f [B][num][R], m [B][Rtot][P] (first R roi slots used), out NHWC rows of stride dstride.
// ---------------------------------------------------------------------------------------------
constexpr int PAINT_PIX = 64;
__global__ void __launch_bounds__(256) paint_max_fwd_kernel(const float* __restrict__ f,
                                                            const float* __restrict__ m, int num, int R, int Rtot,
                                                            long long P, float* __restrict__ out, int dstride,
                                                            int doff) {
  extern __shared__ float smem[];
  float* sf = smem;             // [num][R]
  float* sm = smem + num * R;   // [R][PAINT_PIX]
  const int b = blockIdx.y, t = threadIdx.x;
  const long long p0 = (long long)blockIdx.x * PAINT_PIX;
  const int np = (int)min((long long)PAINT_PIX, P - p0);
  for (int i = t; i < num * R; i += 256) sf[i] = f[(long long)b * num * R + i];
  for (int i = t; i < R * PAINT_PIX; i += 256) {
    int r = i / PAINT_PIX, j = i - r * PAINT_PIX;
    sm[i] = j < np ? m[((long long)b * Rtot + r) * P + p0 + j] : 0.f;
  }
  __syncthreads();
  for (int i = t; i < np * num; i += 256) {
    int j = i / num, k = i - j * num;
    float v = sf[k * R] * sm[j];
    for (int r = 1; r < R; ++r) v = fmaxf(v, sf[k * R + r] * sm[r * PAINT_PIX + j]);
    out[((long long)b * P + p0 + j) * dstride + doff + k] = v;
  }
}
// Vectorised variant: a thread produces FOUR consecutive channels of one pixel (one 16-byte store; a warp writes
// whole 128-byte lines of the NHWC row), the roi features sit in shared memory channel-contiguous (one LDS.128 per roi),
// the block's mask tile is read once, and the (pixel, channel-quad) walk has no divisions.  Channels [num, 4*nq4) are
// written as zeros (the pad lanes of the NHWC tensor), so the caller needs no separate zero fill.
constexpr int PAINT2_PIX = 128;
__global__ void __launch_bounds__(256) paint_max_fwd4_kernel(const float* __restrict__ f, const float* __restrict__ m,
                                                             int num, int nq4, int R, int Rtot, long long P,
                                                             float* __restrict__ out, int dstride, int doff) {
  extern __shared__ __align__(16) float smem[];
  float* sf = smem;                      // [R][4 * nq4]  (channel-contiguous, zero padded)
  float* sm = smem + R * 4 * nq4;        // [R][PAINT2_PIX]
  const int b = blockIdx.y, t = threadIdx.x;
  const long long p0 = (long long)blockIdx.x * PAINT2_PIX;
  const int np = (int)min((long long)PAINT2_PIX, P - p0);
  const int nc = 4 * nq4;
  for (int i = t; i < R * nc; i += 256) {
    const int r = i / nc, k = i - r * nc;
    sf[i] = k < num ? f[((long long)b * num + k) * R + r] : 0.f;
  }
  for (int i = t; i < R * PAINT2_PIX; i += 256) {
    const int r = i / PAINT2_PIX, j = i - r * PAINT2_PIX;
    sm[i] = j < np ? m[((long long)b * Rtot + r) * P + p0 + j] : 0.f;
  }
  __syncthreads();
  const int dj = 256 / nq4, dk = 256 - dj * nq4;
  int j = t / nq4, k4 = t - j * nq4;
  for (; j < np; j += dj, k4 += dk) {
    if (k4 >= nq4) { k4 -= nq4; ++j; if (j >= np) break; }
    const float4 f0 = *reinterpret_cast<const float4*>(sf + 4 * k4);
    const float m0 = sm[j];
    float4 v = make_float4(f0.x * m0, f0.y * m0, f0.z * m0, f0.w * m0);
    for (int r = 1; r < R; ++r) {
      const float4 fr = *reinterpret_cast<const float4*>(sf + r * nc + 4 * k4);
      const float mr = sm[r * PAINT2_PIX + j];
      v.x = fmaxf(v.x, fr.x * mr); v.y = fmaxf(v.y, fr.y * mr);
      v.z = fmaxf(v.z, fr.z * mr); v.w = fmaxf(v.w, fr.w * mr);
    }
    st4(out + ((long long)b * P + p0 + j) * dstride + doff + 4 * k4, v);
  }
}

OG_API int og_paint_max_fwd(const float* f, const float* m, int B, int num, int R, int Rtot, long long P, float* out,
                            int dstride, int doff, cudaStream_t stream) {
  if (B == 0 || P == 0) return 0;
  if (R > 0 && dstride % 4 == 0 && doff % 4 == 0 && (num + 3) / 4 * 4 + doff <= dstride && (num + 3) / 4 <= 256) {
    const int nq4 = (num + 3) / 4;
    const size_t smb = sizeof(float) * ((size_t)R * 4 * nq4 + (size_t)R * PAINT2_PIX);
    if (smb <= 48 * 1024) {
      dim3 grid4(og_cdiv(P, PAINT2_PIX), B);
      paint_max_fwd4_kernel<<<grid4, 256, smb, stream>>>(f, m, num, nq4, R, Rtot, P, out, dstride, doff);
      OG_RETURN_LAST_ERROR();
    }
  }
  if (R == 0) {   // no boxes in the whole batch: the painted maps are zero (ref: model.py:571-576, 689-694)
    OG_CHECK(cudaMemset2DAsync(out + doff, sizeof(float) * (size_t)dstride, 0, sizeof(float) * (size_t)num,
                               (size_t)B * (size_t)P, stream));
    return 0;
  }
  size_t sm = sizeof(float) * (num * R + R * PAINT_PIX);
  if (sm > 48 * 1024)
    OG_CHECK(cudaFuncSetAttribute(paint_max_fwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm));
  dim3 grid(og_cdiv(P, PAINT_PIX), B);
  paint_max_fwd_kernel<<<grid, 256, sm, stream>>>(f, m, num, R, Rtot, P, out, dstride, doff);
  OG_RETURN_LAST_ERROR();
}
// g_f[b][k][r] += sum_p g[b][p][goff + k] * m[b][r][p] * [r == argmax_r f*m]   (first maximal r)
// Block x of image b writes the sums over its PAINT_PIX pixels to out[(x * gridDim.y + b) * num * R], each a
// sequential sum in pixel order, so that the result does not depend on thread scheduling.
__global__ void __launch_bounds__(256) paint_max_bwd_kernel(const float* __restrict__ f,
                                                            const float* __restrict__ m,
                                                            const float* __restrict__ g, int gstride, int goff,
                                                            int num, int R, int Rtot, long long P,
                                                            float* __restrict__ g_f) {
  extern __shared__ float smem[];
  float* sf = smem;                   // [num][R]
  float* sm = sf + num * R;           // [R][PAINT_PIX]
  float* sval = sm + R * PAINT_PIX;   // [PAINT_PIX][num]: pixel j's contribution to (k, its maximal r)
  int* sbr = reinterpret_cast<int*>(sval + PAINT_PIX * num);   // [PAINT_PIX][num]: that r
  const int b = blockIdx.y, t = threadIdx.x;
  const long long p0 = (long long)blockIdx.x * PAINT_PIX;
  const int np = (int)min((long long)PAINT_PIX, P - p0);
  for (int i = t; i < num * R; i += 256) sf[i] = f[(long long)b * num * R + i];
  for (int i = t; i < R * PAINT_PIX; i += 256) {
    int r = i / PAINT_PIX, j = i - r * PAINT_PIX;
    sm[i] = j < np ? m[((long long)b * Rtot + r) * P + p0 + j] : 0.f;
  }
  __syncthreads();
  for (int i = t; i < np * num; i += 256) {
    int j = i / num, k = i - j * num;
    float best = sf[k * R] * sm[j];
    int br = 0;
    for (int r = 1; r < R; ++r) {
      float v = sf[k * R + r] * sm[r * PAINT_PIX + j];
      if (v > best) {
        best = v;
        br = r;
      }
    }
    float mv = sm[br * PAINT_PIX + j];
    sval[i] = mv != 0.f ? g[((long long)b * P + p0 + j) * gstride + goff + k] * mv : 0.f;
    sbr[i] = br;
  }
  __syncthreads();
  for (int i = t; i < num * R; i += 256) {
    const int k = i / R, r = i - k * R;
    float a = 0.f;
    for (int j = 0; j < np; ++j)
      if (sbr[j * num + k] == r) a += sval[j * num + k];
    g_f[((long long)blockIdx.x * gridDim.y + b) * num * R + i] = a;
  }
}
OG_API int og_paint_max_bwd(const float* f, const float* m, const float* g, int gstride, int goff, int B, int num,
                            int R, int Rtot, long long P, float* g_f, cudaStream_t stream) {
  OG_CHECK(cudaMemsetAsync(g_f, 0, sizeof(float) * (size_t)B * num * R, stream));
  if (B == 0 || P == 0 || R == 0) return 0;
  size_t sm = sizeof(float) * (num * R + R * PAINT_PIX + 2 * PAINT_PIX * num);
  static bool configured = false;
  if (!configured) {
    OG_CHECK(cudaFuncSetAttribute(paint_max_bwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    configured = true;
  }
  dim3 grid(og_cdiv(P, PAINT_PIX), B);
  float* out = g_f;
  if (grid.x > 1) OG_CHECK(og_work_alloc(&out, (size_t)grid.x * B * num * R, stream));
  paint_max_bwd_kernel<<<grid, 256, sm, stream>>>(f, m, g, gstride, goff, num, R, Rtot, P, out);
  int rc = (int)cudaGetLastError();
  if (grid.x > 1) {   // per-block partial sums, added in block order
    if (!rc) rc = og_split_sum(out, (long long)B * num * R, (int)grid.x, g_f, stream);
    const cudaError_t e = cudaFreeAsync(out, stream);
    if (!rc) rc = (int)e;
  }
  return rc;
}

// ---------------------------------------------------------------------------------------------
// func_attention forward (DAMSM): one block per (image, caption) pair.
// query [B][ndf][Lq], context [B][ndf][S] (NCHW feature map flattened) -> wc [B][ndf][Lq], attn [B][Lq][S]
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) func_attention_fwd_kernel(const float* __restrict__ query,
                                                                 const float* __restrict__ ctx, int ndf, int Lq,
                                                                 int S, float gamma1, float* __restrict__ wc,
                                                                 float* __restrict__ attn) {
  extern __shared__ float smem[];
  float* sq = smem;              // [ndf][Lq]
  float* sp = smem + ndf * Lq;   // [S][Lq]  scores / probabilities
  const int b = blockIdx.x, t = threadIdx.x, lane = t & 31, warp = t >> 5;
  const float* qb = query + (long long)b * ndf * Lq;
  const float* cb = ctx + (long long)b * ndf * S;
  for (int i = t; i < ndf * Lq; i += 256) sq[i] = qb[i];
  __syncthreads();
  // phase 1+2: scores per region, softmax over the words (ref: GlobalAttention.py:49-53)
  for (int s = t; s < S; s += 256) {
    float acc[LMAX];
#pragma unroll
    for (int l = 0; l < LMAX; ++l) acc[l] = 0.f;
    for (int c = 0; c < ndf; ++c) {
      float cv = __ldg(cb + (long long)c * S + s);
      const float* qr = sq + c * Lq;
#pragma unroll
      for (int l = 0; l < LMAX; ++l)
        if (l < Lq) acc[l] = fmaf(cv, qr[l], acc[l]);
    }
    float mx = -INFINITY;
#pragma unroll
    for (int l = 0; l < LMAX; ++l)
      if (l < Lq) mx = fmaxf(mx, acc[l]);
    float sum = 0.f;
#pragma unroll
    for (int l = 0; l < LMAX; ++l)
      if (l < Lq) {
        acc[l] = expf(acc[l] - mx);
        sum += acc[l];
      }
    float inv = 1.f / sum;
#pragma unroll
    for (int l = 0; l < LMAX; ++l)
      if (l < Lq) sp[s * Lq + l] = acc[l] * inv;
  }
  __syncthreads();
  // phase 3: per word, softmax over the regions of gamma1 * p (ref: GlobalAttention.py:57-62)
  for (int l = warp; l < Lq; l += 8) {
    float mx = -INFINITY;
    for (int s = lane; s < S; s += 32) mx = fmaxf(mx, sp[s * Lq + l] * gamma1);
    mx = warp_max(mx);
    float sum = 0.f;
    for (int s = lane; s < S; s += 32) {
      float e = expf(sp[s * Lq + l] * gamma1 - mx);
      sp[s * Lq + l] = e;
      sum += e;
    }
    sum = warp_sum(sum);
    float inv = 1.f / sum;
    for (int s = lane; s < S; s += 32) {
      float a = sp[s * Lq + l] * inv;
      sp[s * Lq + l] = a;
      attn[((long long)b * Lq + l) * S + s] = a;
    }
  }
  __syncthreads();
  // phase 4: weighted context (ref: GlobalAttention.py:66-68); warp per channel, lanes over regions
  for (int c = warp; c < ndf; c += 8) {
    float acc[LMAX];
#pragma unroll
    for (int l = 0; l < LMAX; ++l) acc[l] = 0.f;
    for (int s = lane; s < S; s += 32) {
      float cv = __ldg(cb + (long long)c * S + s);
      const float* pr = sp + s * Lq;
#pragma unroll
      for (int l = 0; l < LMAX; ++l)
        if (l < Lq) acc[l] = fmaf(cv, pr[l], acc[l]);
    }
#pragma unroll
    for (int l = 0; l < LMAX; ++l)
      if (l < Lq) {
        float v = warp_sum(acc[l]);
        if (lane == 0) wc[((long long)b * ndf + c) * Lq + l] = v;
      }
  }
}
OG_API int og_func_attention_fwd(const float* query, const float* ctx, int B, int ndf, int Lq, int S, float gamma1,
                                 float* wc, float* attn, cudaStream_t stream) {
  if (Lq > LMAX) return (int)cudaErrorInvalidValue;
  if (B == 0) return 0;
  size_t sm = sizeof(float) * ((size_t)ndf * Lq + (size_t)S * Lq);
  OG_CHECK(cudaFuncSetAttribute(func_attention_fwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm));
  func_attention_fwd_kernel<<<B, 256, sm, stream>>>(query, ctx, ndf, Lq, S, gamma1, wc, attn);
  OG_RETURN_LAST_ERROR();
}

// ---------------------------------------------------------------------------------------------
// func_attention backward (ref: GlobalAttention.py:32-70): one block per (image, caption) pair.
//   S[s,l] = sum_c ctx[c,s] q[c,l];  P = softmax_l(S);  P2 = softmax_s(gamma1 * P^T);  wc[c,l] = sum_s ctx[c,s] P2[l,s]
// inputs: query, ctx, attn (= P2, the saved forward output), g_wc [B][ndf][Lq], g_attn [B][Lq][S] or null
// outputs: g_query [B][ndf][Lq], g_ctx [B][ndf][S]
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) func_attention_bwd_kernel(const float* __restrict__ query,
                                                                 const float* __restrict__ ctx,
                                                                 const float* __restrict__ attn,
                                                                 const float* __restrict__ g_wc,
                                                                 const float* __restrict__ g_attn, int ndf, int Lq,
                                                                 int S, float gamma1, float* __restrict__ g_query,
                                                                 float* __restrict__ g_ctx) {
  extern __shared__ float smem[];
  float* sq = smem;                 // [ndf][Lq]   query
  float* sg = sq + ndf * Lq;        // [ndf][Lq]   g_wc
  float* sP = sg + ndf * Lq;        // [S][Lq]     P, then gS
  float* sP2 = sP + S * Lq;         // [Lq][S]     P2
  float* sG = sP2 + Lq * S;         // [Lq][S]     gP2, then gT
  const int b = blockIdx.x, t = threadIdx.x, lane = t & 31, warp = t >> 5;
  const float* qb = query + (long long)b * ndf * Lq;
  const float* cb = ctx + (long long)b * ndf * S;
  const float* gb = g_wc + (long long)b * ndf * Lq;
  for (int i = t; i < ndf * Lq; i += 256) {
    sq[i] = qb[i];
    sg[i] = gb[i];
  }
  for (int i = t; i < Lq * S; i += 256) sP2[i] = attn[(long long)b * Lq * S + i];
  __syncthreads();
  // (1) recompute P (softmax over the words, per region) and gP2[l,s] = sum_c g_wc[c,l] ctx[c,s] (+ g_attn)
  for (int s = t; s < S; s += 256) {
    float acc[LMAX], gp[LMAX];
#pragma unroll
    for (int l = 0; l < LMAX; ++l) {
      acc[l] = 0.f;
      gp[l] = 0.f;
    }
    for (int c = 0; c < ndf; ++c) {
      const float cv = __ldg(cb + (long long)c * S + s);
      const float* qr = sq + c * Lq;
      const float* gr = sg + c * Lq;
#pragma unroll
      for (int l = 0; l < LMAX; ++l)
        if (l < Lq) {
          acc[l] = fmaf(cv, qr[l], acc[l]);
          gp[l] = fmaf(cv, gr[l], gp[l]);
        }
    }
    float mx = -INFINITY;
#pragma unroll
    for (int l = 0; l < LMAX; ++l)
      if (l < Lq) mx = fmaxf(mx, acc[l]);
    float sum = 0.f;
#pragma unroll
    for (int l = 0; l < LMAX; ++l)
      if (l < Lq) {
        acc[l] = expf(acc[l] - mx);
        sum += acc[l];
      }
    const float inv = 1.f / sum;
#pragma unroll
    for (int l = 0; l < LMAX; ++l)
      if (l < Lq) {
        sP[s * Lq + l] = acc[l] * inv;
        sG[l * S + s] = gp[l] + (g_attn ? g_attn[((long long)b * Lq + l) * S + s] : 0.f);
      }
  }
  __syncthreads();
  // (2) softmax backward over the regions, per word: gT = P2 * (gP2 - <gP2, P2>)
  for (int l = warp; l < Lq; l += 8) {
    float d = 0.f;
    for (int s = lane; s < S; s += 32) d = fmaf(sG[l * S + s], sP2[l * S + s], d);
    d = warp_sum(d);
    for (int s = lane; s < S; s += 32) sG[l * S + s] = sP2[l * S + s] * (sG[l * S + s] - d);
  }
  __syncthreads();
  // (3) softmax backward over the words, per region: gS = P * (gP - <gP, P>),  gP = gamma1 * gT^T
  for (int s = t; s < S; s += 256) {
    float d = 0.f;
    for (int l = 0; l < Lq; ++l) d = fmaf(gamma1 * sG[l * S + s], sP[s * Lq + l], d);
    for (int l = 0; l < Lq; ++l) sP[s * Lq + l] = sP[s * Lq + l] * (gamma1 * sG[l * S + s] - d);
  }
  __syncthreads();
  // (4) g_ctx[c,s] = sum_l g_wc[c,l] P2[l,s] + gS[s,l] q[c,l];   g_query[c,l] = sum_s gS[s,l] ctx[c,s]
  for (int c = warp; c < ndf; c += 8) {
    float gq[LMAX];
#pragma unroll
    for (int l = 0; l < LMAX; ++l) gq[l] = 0.f;
    const float* qr = sq + c * Lq;
    const float* gr = sg + c * Lq;
    for (int s = lane; s < S; s += 32) {
      const float cv = __ldg(cb + (long long)c * S + s);
      float a = 0.f;
#pragma unroll
      for (int l = 0; l < LMAX; ++l)
        if (l < Lq) {
          const float gs = sP[s * Lq + l];
          a = fmaf(gr[l], sP2[l * S + s], a);
          a = fmaf(gs, qr[l], a);
          gq[l] = fmaf(gs, cv, gq[l]);
        }
      g_ctx[((long long)b * ndf + c) * S + s] = a;
    }
#pragma unroll
    for (int l = 0; l < LMAX; ++l)
      if (l < Lq) {
        const float v = warp_sum(gq[l]);
        if (lane == 0) g_query[((long long)b * ndf + c) * Lq + l] = v;
      }
  }
}
OG_API int og_func_attention_bwd(const float* query, const float* ctx, const float* attn, const float* g_wc,
                                 const float* g_attn, int B, int ndf, int Lq, int S, float gamma1, float* g_query,
                                 float* g_ctx, cudaStream_t stream) {
  if (Lq > LMAX) return (int)cudaErrorInvalidValue;
  if (B == 0) return 0;
  size_t sm = sizeof(float) * (2 * (size_t)ndf * Lq + 3 * (size_t)S * Lq);
  OG_CHECK(cudaFuncSetAttribute(func_attention_bwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm));
  func_attention_bwd_kernel<<<B, 256, sm, stream>>>(query, ctx, attn, g_wc, g_attn, ndf, Lq, S, gamma1, g_query, g_ctx);
  OG_RETURN_LAST_ERROR();
}
