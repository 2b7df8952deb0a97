// Text stage of caption-conditioned sampling: the recurrence of the reference's text encoder (ref: model.py:85-179,
// RNN_ENCODER: a one-layer bidirectional nn.LSTM over packed captions, in eval mode), the GloVe word lookups and the
// padding mask of the evaluator (evaluator.py:337-351), and the class label embeddings of prepare_cat_emb
// (evaluator.py:148-164).  The input projection of the LSTM runs before the recurrence as one 1x1 og_conv2d_simt.
#include <cooperative_groups.h>

#include "common.cuh"

namespace cg = cooperative_groups;

static int tblocks(long long total) {
  long long b = (total + 255) / 256;
  long long cap = (long long)og_num_sms() * 32;
  return (int)(b < cap ? (b < 1 ? 1 : b) : cap);
}

// ---------------------------------------------------------------------------------------------------------------
// Bidirectional LSTM recurrence.  One thread-block cluster of LSTM_CLUSTER CTAs per (direction, batch tile).  CTA r of
// a cluster owns hidden units [32 r, 32 r + 32): it keeps their i, f, g, o rows of W_hh (128 rows x 128 fp32, 64 KB) in
// shared memory for all steps, and lane j of every warp is unit 32 r + j, so the cell update and c stay in registers.
// Warp w handles the SPW samples [w * SPW, (w + 1) * SPW) of the tile.  After each step every CTA stores its 32 new h
// values of each sample into the next h buffer of all four CTAs of its cluster (distributed shared memory); one
// cluster barrier per step orders those stores before the next step's reads, and the h buffers are double-buffered so
// that no second barrier is needed (a peer can only be one step behind, reading the other buffer).
//
// Each gate pre-activation is gx + sum_k W_hh[row][k] * h[k], the sum a chain of fmaf in k order 0..127 for every
// sample, so a sample's result does not depend on its position in the batch, on the tile size or on B.
// ---------------------------------------------------------------------------------------------------------------
constexpr int LSTM_H = 128;                       // hidden units per direction
constexpr int LSTM_CLUSTER = 4;                   // CTAs per direction and tile
constexpr int LSTM_UNITS = LSTM_H / LSTM_CLUSTER; // 32: one unit per lane
constexpr int LSTM_WARPS = 8;
constexpr int LSTM_THREADS = LSTM_WARPS * 32;
constexpr int LSTM_LD = LSTM_H + 4;               // padded smem row: the 8 lanes of a float4 phase hit distinct banks

static size_t lstm_smem_bytes(int spw) {
  return sizeof(float) * (size_t)LSTM_LD * (4 * LSTM_UNITS + 2 * LSTM_WARPS * spw);
}

struct LstmArgs {
  const float* gx;       // [B * L][2 * 4 * H]: x-part of the gates + b_ih + b_hh; direction d at channel d * 4H
  const float* whh_f;    // [4H][H] per direction, gate order i, f, g, o
  const float* whh_b;
  const long long* lens; // [B]
  float* words;          // [B][2H][L]
  float* sent;           // [B][2H]
  int B, L;
  float* cell;           // [B][2H]: c after the same token as sent (CELL instantiations only)
};

// CELL: also write the final cell state (the encoder state the box decoder starts from); the instantiations without it
// are the text encoder's.
template <int SPW, bool CELL>
__global__ void __cluster_dims__(LSTM_CLUSTER, 1, 1) __launch_bounds__(LSTM_THREADS, 1)
    lstm_bidir_kernel(LstmArgs a) {
  extern __shared__ float4 smem4[];
  float* sw = reinterpret_cast<float*>(smem4);               // [4 * 32][LD]: local row g * 32 + j
  float* sh = sw + 4 * LSTM_UNITS * LSTM_LD;                  // [2][8 * SPW][LD]
  constexpr int BT = LSTM_WARPS * SPW;
  cg::cluster_group cluster = cg::this_cluster();
  const int rank = (int)cluster.block_rank();
  const int dir = blockIdx.x / LSTM_CLUSTER;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int unit = rank * LSTM_UNITS + lane;

  const float* whh = dir ? a.whh_b : a.whh_f;
  for (int i = threadIdx.x; i < 4 * LSTM_UNITS * (LSTM_H / 4); i += LSTM_THREADS) {
    const int row = i / (LSTM_H / 4), q = i % (LSTM_H / 4);
    const int grow = (row / LSTM_UNITS) * LSTM_H + rank * LSTM_UNITS + row % LSTM_UNITS;
    st4(sw + row * LSTM_LD + q * 4, ldg4(whh + (long long)grow * LSTM_H + q * 4));
  }
  for (int i = threadIdx.x; i < 2 * BT * LSTM_LD; i += LSTM_THREADS) sh[i] = 0.f;   // h_0 = 0

  int len[SPW];
  long long bidx[SPW];
  float c[SPW];
#pragma unroll
  for (int s = 0; s < SPW; ++s) {
    bidx[s] = (long long)blockIdx.y * BT + warp * SPW + s;
    len[s] = bidx[s] < a.B ? (int)a.lens[bidx[s]] : 0;
    c[s] = 0.f;
  }
  float* peer[LSTM_CLUSTER];                         // sh of every CTA of the cluster (this one included)
#pragma unroll
  for (int r = 0; r < LSTM_CLUSTER; ++r) peer[r] = cluster.map_shared_rank(sh, r);
  cluster.sync();                                    // every CTA's buffers are zeroed before any peer writes to them

  const int G4 = 4 * LSTM_H;
  const int wout = dir * LSTM_H + unit;              // channel of this thread's unit in words / sent
  for (int t = 0; t < a.L; ++t) {
    const int cur = t & 1;
    bool any = false;
#pragma unroll
    for (int s = 0; s < SPW; ++s) any |= t < len[s];
    if (any) {                                       // warp-uniform: the warp's lanes share their samples
      float gxv[SPW][4];
#pragma unroll
      for (int s = 0; s < SPW; ++s) {
        const int p = dir ? len[s] - 1 - t : t;      // the backward direction starts at the last token
        const float* row = a.gx + (bidx[s] * a.L + p) * (2 * G4) + dir * G4 + unit;
#pragma unroll
        for (int g = 0; g < 4; ++g) gxv[s][g] = t < len[s] ? __ldg(row + g * LSTM_H) : 0.f;
      }
      float acc[SPW][4];
#pragma unroll
      for (int s = 0; s < SPW; ++s)
#pragma unroll
        for (int g = 0; g < 4; ++g) acc[s][g] = 0.f;
      const float* hb = sh + cur * BT * LSTM_LD + warp * SPW * LSTM_LD;
#pragma unroll 2
      for (int k = 0; k < LSTM_H; k += 4) {
        float4 w[4];
#pragma unroll
        for (int g = 0; g < 4; ++g) w[g] = *reinterpret_cast<const float4*>(sw + (g * LSTM_UNITS + lane) * LSTM_LD + k);
#pragma unroll
        for (int s = 0; s < SPW; ++s) {
          const float4 h = *reinterpret_cast<const float4*>(hb + s * LSTM_LD + k);
#pragma unroll
          for (int g = 0; g < 4; ++g) {
            acc[s][g] = fmaf(w[g].x, h.x, acc[s][g]);
            acc[s][g] = fmaf(w[g].y, h.y, acc[s][g]);
            acc[s][g] = fmaf(w[g].z, h.z, acc[s][g]);
            acc[s][g] = fmaf(w[g].w, h.w, acc[s][g]);
          }
        }
      }
#pragma unroll
      for (int s = 0; s < SPW; ++s) {
        if (t < len[s]) {
          const float ig = og_sigmoid(gxv[s][0] + acc[s][0]), fg = og_sigmoid(gxv[s][1] + acc[s][1]);
          const float gg = tanhf(gxv[s][2] + acc[s][2]), og = og_sigmoid(gxv[s][3] + acc[s][3]);
          c[s] = __fadd_rn(__fmul_rn(fg, c[s]), __fmul_rn(ig, gg));
          const float h = og * tanhf(c[s]);
          const int slot = ((cur ^ 1) * BT + warp * SPW + s) * LSTM_LD + unit;
#pragma unroll
          for (int r = 0; r < LSTM_CLUSTER; ++r) peer[r][slot] = h;
          const int p = dir ? len[s] - 1 - t : t;
          a.words[(bidx[s] * 2 * LSTM_H + wout) * a.L + p] = h;
          if (t == len[s] - 1) a.sent[bidx[s] * 2 * LSTM_H + wout] = h;   // fwd: h after the last token; bwd: at token 0
          if constexpr (CELL) {
            if (t == len[s] - 1) a.cell[bidx[s] * 2 * LSTM_H + wout] = c[s];
          }
        }
      }
    }
#pragma unroll
    for (int s = 0; s < SPW; ++s)                    // columns past the caption (pad_packed_sequence + post_process_words)
      if (bidx[s] < a.B && t >= len[s]) a.words[(bidx[s] * 2 * LSTM_H + wout) * a.L + t] = 0.f;
    cluster.sync();
  }
}

template <int SPW, bool CELL>
static int lstm_launch(const LstmArgs& a, cudaStream_t stream) {
  static bool ready = false;                          // dynamic smem above 48 KB is opt-in, once per instantiation
  const size_t smem = lstm_smem_bytes(SPW);
  if (!ready) {
    OG_CHECK(cudaFuncSetAttribute(lstm_bidir_kernel<SPW, CELL>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                  (int)smem));
    ready = true;
  }
  const int bt = LSTM_WARPS * SPW;
  const dim3 grid(2 * LSTM_CLUSTER, og_cdiv(a.B, bt));
  lstm_bidir_kernel<SPW, CELL><<<grid, LSTM_THREADS, smem, stream>>>(a);
  OG_RETURN_LAST_ERROR();
}

template <bool CELL>
static int lstm_dispatch(const float* gx, const float* whh_f, const float* whh_b, const long long* lens, int B, int L,
                         int H, float* words, float* sent, float* cell, cudaStream_t stream) {
  if (H != LSTM_H || B < 0 || L < 0) return (int)cudaErrorInvalidValue;
  if (B == 0 || L == 0) return 0;
  LstmArgs a;
  a.gx = gx; a.whh_f = whh_f; a.whh_b = whh_b; a.lens = lens; a.words = words; a.sent = sent; a.B = B; a.L = L;
  a.cell = cell;
  // the smallest tile that holds the batch (up to 64 samples): fewer samples per warp shorten each step's FMA chain
  if (B <= 8) return lstm_launch<1, CELL>(a, stream);
  if (B <= 16) return lstm_launch<2, CELL>(a, stream);
  if (B <= 32) return lstm_launch<4, CELL>(a, stream);
  return lstm_launch<8, CELL>(a, stream);
}

OG_API int og_lstm_bidir(const float* gx, const float* whh_f, const float* whh_b, const long long* lens, int B, int L,
                         int H, float* words, float* sent, cudaStream_t stream) {
  return lstm_dispatch<false>(gx, whh_f, whh_b, lens, B, L, H, words, sent, nullptr, stream);
}

OG_API int og_lstm_bidir_state(const float* gx, const float* whh_f, const float* whh_b, const long long* lens, int B,
                               int L, int H, float* words, float* sent, float* cell, cudaStream_t stream) {
  return lstm_dispatch<true>(gx, whh_f, whh_b, lens, B, L, H, words, sent, cell, stream);
}

// ---------------------------------------------------------------------------------------------------------------
// The evaluator's word inputs besides the encoder (evaluator.py:340-351): glove_words[b][e][t] =
// glove[glove_ids[b][t]][e] and mask[b][t] = (captions[b][t] == 0), t < L, in one launch.
// ---------------------------------------------------------------------------------------------------------------
__global__ void text_inputs_kernel(const long long* __restrict__ captions, int cap_ld,
                                   const long long* __restrict__ glove_ids, int glove_ld,
                                   const float* __restrict__ glove, int E, int B, int L, float* __restrict__ glove_words,
                                   unsigned char* __restrict__ mask) {
  const long long nw = (long long)B * E * L, total = nw + (long long)B * L;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    if (i < nw) {
      const int t = (int)(i % L);
      const int e = (int)((i / L) % E);
      const long long b = i / ((long long)L * E);
      glove_words[i] = glove[glove_ids[b * glove_ld + t] * E + e];
    } else {
      const long long j = i - nw;
      mask[j] = captions[(j / L) * cap_ld + j % L] == 0 ? 1 : 0;
    }
  }
}

OG_API int og_text_inputs(const long long* captions, int cap_ld, const long long* glove_ids, int glove_ld,
                          const float* glove, int E, int B, int L, float* glove_words, unsigned char* mask,
                          cudaStream_t stream) {
  if (L > cap_ld || L > glove_ld) return (int)cudaErrorInvalidValue;
  const long long total = (long long)B * (E + 1) * L;
  if (total == 0) return 0;
  text_inputs_kernel<<<tblocks(total), 256, 0, stream>>>(captions, cap_ld, glove_ids, glove_ld, glove, E, B, L,
                                                       glove_words, mask);
  OG_RETURN_LAST_ERROR();
}

// ---------------------------------------------------------------------------------------------------------------
// prepare_cat_emb (evaluator.py:148-164): row k of the length-sorted labels is the mean of its GloVe vectors when it
// has 1 or 2 tokens, else zeros; out[i] = row order[i].
// ---------------------------------------------------------------------------------------------------------------
__global__ void class_label_emb_kernel(const float* __restrict__ glove, int E, const long long* __restrict__ labels,
                                       int lab_ld, const long long* __restrict__ lens,
                                       const long long* __restrict__ order, int n, float* __restrict__ out) {
  const long long total = (long long)n * E;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const long long k = order[i / E];
    const int e = (int)(i % E);
    const long long len = lens[k];
    const long long* lab = labels + k * lab_ld;
    float v = 0.f;
    if (len == 1) v = glove[lab[0] * E + e];
    else if (len == 2) v = (glove[lab[0] * E + e] + glove[lab[1] * E + e]) / 2.f;
    out[i] = v;
  }
}

OG_API int og_class_label_emb(const float* glove, int E, const long long* labels, int lab_ld, const long long* lens,
                              const long long* order, int n, float* out, cudaStream_t stream) {
  const long long total = (long long)n * E;
  if (total == 0) return 0;
  class_label_emb_kernel<<<tblocks(total), 256, 0, stream>>>(glove, E, labels, lab_ld, lens, order, n, out);
  OG_RETURN_LAST_ERROR();
}
