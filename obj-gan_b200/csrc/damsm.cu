// DAMSM matching losses around func_attention (ref: miscc/losses.py:13-159): the small reductions that sit between
// the attention kernel (attention.cu) and the two cross-entropy terms.  Problem sizes are tiny (B <= 64 captions,
// nef = 256, <= 32 words), so these are one-thread-per-output kernels; what matters is that no arithmetic is left to
// host loops or library calls and that the backward formulas match autograd on the reference's expressions.
#include "common.cuh"

namespace {
// largest B of og_ce_pair (one thread per row / column): the evaluator's R-precision pool is 100 (RP_POOL_SIZE)
constexpr int DM_MAXB = 128;

// ---- cosine_similarity(word, weiContext) over the feature axis (losses.py:13-19, 101-108) ----------------------
// word [D][L] (one caption, shared by all images), wei [B][D][L]  ->  out[b][l]
__global__ void cosine_cl_fwd_kernel(const float* __restrict__ word, const float* __restrict__ wei, int B, int D, int L,
                                     float eps, float* __restrict__ out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= B * L) return;
  const int b = i / L, l = i - b * L;
  float w12 = 0.f, w1 = 0.f, w2 = 0.f;
  for (int c = 0; c < D; ++c) {
    const float x = word[c * L + l], y = wei[((long long)b * D + c) * L + l];
    w12 = fmaf(x, y, w12);
    w1 = fmaf(x, x, w1);
    w2 = fmaf(y, y, w2);
  }
  out[i] = w12 / fmaxf(sqrtf(w1) * sqrtf(w2), eps);
}
// gradient w.r.t. wei only (the caption embedding is a constant of the generator update)
__global__ void cosine_cl_bwd_kernel(const float* __restrict__ word, const float* __restrict__ wei,
                                     const float* __restrict__ g, int B, int D, int L, float eps,
                                     float* __restrict__ gwei) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= B * L) return;
  const int b = i / L, l = i - b * L;
  float w12 = 0.f, w1 = 0.f, w2 = 0.f;
  for (int c = 0; c < D; ++c) {
    const float x = word[c * L + l], y = wei[((long long)b * D + c) * L + l];
    w12 = fmaf(x, y, w12);
    w1 = fmaf(x, x, w1);
    w2 = fmaf(y, y, w2);
  }
  const float n1 = sqrtf(w1), n2 = sqrtf(w2), prod = n1 * n2;
  const float go = g[i];
  if (prod >= eps) {
    // cos = w12 / (n1 n2):  d/dy_c = x_c / (n1 n2) - cos * y_c / n2^2
    const float inv = 1.f / prod, k = w12 * inv / w2;
    for (int c = 0; c < D; ++c) {
      const long long o = ((long long)b * D + c) * L + l;
      gwei[o] = go * (word[c * L + l] * inv - k * wei[o]);
    }
  } else {
    const float inv = 1.f / eps;     // clamped denominator: cos = w12 / eps
    for (int c = 0; c < D; ++c) gwei[((long long)b * D + c) * L + l] = go * word[c * L + l] * inv;
  }
}

// ---- Eq. (10): out[b] = log(sum_l exp(gamma * s[b][l]))  (losses.py:112-115; no max shift, like the reference) ----
__global__ void expsumlog_fwd_kernel(const float* __restrict__ s, int B, int L, float gamma, float* __restrict__ out) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  float acc = 0.f;
  for (int l = 0; l < L; ++l) acc += expf(gamma * s[b * L + l]);
  out[b] = logf(acc);
}
__global__ void expsumlog_bwd_kernel(const float* __restrict__ s, const float* __restrict__ g, int B, int L, float gamma,
                                     float* __restrict__ gs) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  float acc = 0.f;
  for (int l = 0; l < L; ++l) acc += expf(gamma * s[b * L + l]);
  const float k = g[b] * gamma / acc;
  for (int l = 0; l < L; ++l) gs[b * L + l] = k * expf(gamma * s[b * L + l]);
}

// ---- sent_loss scores (losses.py:43-50): out[i][j] = <a_i, b_j> / max(|a_i| |b_j|, eps) -----------------------------
__global__ void cosine_matrix_fwd_kernel(const float* __restrict__ a, const float* __restrict__ b, int Ba, int Bb, int D,
                                         float eps, float* __restrict__ out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= Ba * Bb) return;
  const int r = i / Bb, c = i - r * Bb;
  float w12 = 0.f, w1 = 0.f, w2 = 0.f;
  for (int k = 0; k < D; ++k) {
    const float x = a[r * D + k], y = b[c * D + k];
    w12 = fmaf(x, y, w12);
    w1 = fmaf(x, x, w1);
    w2 = fmaf(y, y, w2);
  }
  out[i] = w12 / fmaxf(sqrtf(w1) * sqrtf(w2), eps);
}
// gradient w.r.t. a: one thread per (row r, feature k), loop over the columns
__global__ void cosine_matrix_bwd_kernel(const float* __restrict__ a, const float* __restrict__ b,
                                         const float* __restrict__ g, int Ba, int Bb, int D, float eps,
                                         float* __restrict__ ga) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= Ba * D) return;
  const int r = i / D, k = i - r * D;
  float w1 = 0.f;
  for (int q = 0; q < D; ++q) w1 = fmaf(a[r * D + q], a[r * D + q], w1);
  const float n1 = sqrtf(w1);
  float acc = 0.f;
  for (int c = 0; c < Bb; ++c) {
    float w12 = 0.f, w2 = 0.f;
    for (int q = 0; q < D; ++q) {
      const float y = b[c * D + q];
      w12 = fmaf(a[r * D + q], y, w12);
      w2 = fmaf(y, y, w2);
    }
    const float prod = n1 * sqrtf(w2);
    const float go = g[r * Bb + c];
    if (prod >= eps) acc += go * (b[c * D + k] / prod - (w12 / prod) * a[r * D + k] / w1);
    else acc += go * b[c * D + k] / eps;
  }
  ga[i] = acc;
}

// ---- the two CrossEntropyLoss terms over a B x B similarity matrix (losses.py:50-58, 131-139) ------------------------
// scores = gamma3 * sim, entries with mask != 0 set to -inf;  loss0 = CE(scores, labels), loss1 = CE(scores^T, labels)
// (mean over the B rows).  G0 / G1 = d loss0 / d sim, d loss1 / d sim.  correct = top-1 hits of both directions.
__global__ void ce_pair_kernel(const float* __restrict__ sim, const unsigned char* __restrict__ mask,
                               const long long* __restrict__ labels, int B, float gamma3, float* __restrict__ loss0,
                               float* __restrict__ loss1, float* __restrict__ G0, float* __restrict__ G1,
                               float* __restrict__ correct) {
  __shared__ float t0[DM_MAXB], t1[DM_MAXB], hit[DM_MAXB];
  const int i = threadIdx.x;
  if (i < B) {
    const int lab = (int)labels[i];
    // direction 0: row i
    float m = -INFINITY;
    int arg = 0;
    for (int j = 0; j < B; ++j) {
      const float v = (mask && mask[i * B + j]) ? -INFINITY : gamma3 * sim[i * B + j];
      if (v > m) { m = v; arg = j; }
    }
    float sum = 0.f;
    for (int j = 0; j < B; ++j) {
      const float v = (mask && mask[i * B + j]) ? -INFINITY : gamma3 * sim[i * B + j];
      sum += expf(v - m);
    }
    const float vlab = (mask && mask[i * B + lab]) ? -INFINITY : gamma3 * sim[i * B + lab];
    t0[i] = (m + logf(sum)) - vlab;
    for (int j = 0; j < B; ++j) {
      const float v = (mask && mask[i * B + j]) ? -INFINITY : gamma3 * sim[i * B + j];
      G0[i * B + j] = gamma3 * (expf(v - m) / sum - (j == lab ? 1.f : 0.f)) / (float)B;
    }
    float h = (arg == lab) ? 1.f : 0.f;
    // direction 1: column i
    m = -INFINITY;
    arg = 0;
    for (int j = 0; j < B; ++j) {
      const float v = (mask && mask[j * B + i]) ? -INFINITY : gamma3 * sim[j * B + i];
      if (v > m) { m = v; arg = j; }
    }
    sum = 0.f;
    for (int j = 0; j < B; ++j) {
      const float v = (mask && mask[j * B + i]) ? -INFINITY : gamma3 * sim[j * B + i];
      sum += expf(v - m);
    }
    const float vlab1 = (mask && mask[lab * B + i]) ? -INFINITY : gamma3 * sim[lab * B + i];
    t1[i] = (m + logf(sum)) - vlab1;
    for (int j = 0; j < B; ++j) {
      const float v = (mask && mask[j * B + i]) ? -INFINITY : gamma3 * sim[j * B + i];
      G1[j * B + i] = gamma3 * (expf(v - m) / sum - (j == lab ? 1.f : 0.f)) / (float)B;
    }
    h += (arg == lab) ? 1.f : 0.f;
    hit[i] = h;
  }
  __syncthreads();
  if (i == 0) {
    float s0 = 0.f, s1 = 0.f, c = 0.f;
    for (int k = 0; k < B; ++k) { s0 += t0[k]; s1 += t1[k]; c += hit[k]; }
    *loss0 = s0 / (float)B;
    *loss1 = s1 / (float)B;
    *correct = c;
  }
}
// gsim = g0 * G0 + g1 * G1 (g0 / g1: device scalars, null = 0)
__global__ void ce_pair_bwd_kernel(const float* __restrict__ G0, const float* __restrict__ G1, const float* __restrict__ g0,
                                   const float* __restrict__ g1, int n, float* __restrict__ gsim) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float a = g0 ? *g0 : 0.f, b = g1 ? *g1 : 0.f;
  gsim[i] = a * G0[i] + b * G1[i];
}
}  // namespace

OG_API int og_cosine_cl_fwd(const float* word, const float* wei, int B, int D, int L, float eps, float* out,
                            cudaStream_t stream) {
  if (B * L == 0) return 0;
  cosine_cl_fwd_kernel<<<og_cdiv(B * L, 128), 128, 0, stream>>>(word, wei, B, D, L, eps, out);
  OG_RETURN_LAST_ERROR();
}
OG_API int og_cosine_cl_bwd(const float* word, const float* wei, const float* g, int B, int D, int L, float eps,
                            float* gwei, cudaStream_t stream) {
  if (B * L == 0) return 0;
  cosine_cl_bwd_kernel<<<og_cdiv(B * L, 128), 128, 0, stream>>>(word, wei, g, B, D, L, eps, gwei);
  OG_RETURN_LAST_ERROR();
}
OG_API int og_expsumlog_fwd(const float* s, int B, int L, float gamma, float* out, cudaStream_t stream) {
  if (B == 0) return 0;
  expsumlog_fwd_kernel<<<og_cdiv(B, 64), 64, 0, stream>>>(s, B, L, gamma, out);
  OG_RETURN_LAST_ERROR();
}
OG_API int og_expsumlog_bwd(const float* s, const float* g, int B, int L, float gamma, float* gs, cudaStream_t stream) {
  if (B == 0) return 0;
  expsumlog_bwd_kernel<<<og_cdiv(B, 64), 64, 0, stream>>>(s, g, B, L, gamma, gs);
  OG_RETURN_LAST_ERROR();
}
OG_API int og_cosine_matrix_fwd(const float* a, const float* b, int Ba, int Bb, int D, float eps, float* out,
                                cudaStream_t stream) {
  if (Ba * Bb == 0) return 0;
  cosine_matrix_fwd_kernel<<<og_cdiv(Ba * Bb, 128), 128, 0, stream>>>(a, b, Ba, Bb, D, eps, out);
  OG_RETURN_LAST_ERROR();
}
OG_API int og_cosine_matrix_bwd(const float* a, const float* b, const float* g, int Ba, int Bb, int D, float eps,
                                float* ga, cudaStream_t stream) {
  if (Ba * D == 0) return 0;
  cosine_matrix_bwd_kernel<<<og_cdiv(Ba * D, 128), 128, 0, stream>>>(a, b, g, Ba, Bb, D, eps, ga);
  OG_RETURN_LAST_ERROR();
}
OG_API int og_ce_pair(const float* sim, const unsigned char* mask, const long long* labels, int B, float gamma3,
                      float* loss0, float* loss1, float* G0, float* G1, float* correct, cudaStream_t stream) {
  if (B < 1 || B > DM_MAXB) return (int)cudaErrorInvalidValue;
  ce_pair_kernel<<<1, DM_MAXB, 0, stream>>>(sim, mask, labels, B, gamma3, loss0, loss1, G0, G1, correct);
  OG_RETURN_LAST_ERROR();
}
OG_API int og_ce_pair_bwd(const float* G0, const float* G1, const float* g0, const float* g1, int n, float* gsim,
                          cudaStream_t stream) {
  if (n == 0) return 0;
  ce_pair_bwd_kernel<<<og_cdiv(n, 128), 128, 0, stream>>>(G0, G1, g0, g1, n, gsim);
  OG_RETURN_LAST_ERROR();
}
