// Box stage of caption-to-image sampling: the inference branch of the reference's box generator (box_generation/,
// seq2seq/models/DecoderRNN.py:81-183 and 260-292, an LSTM decoder with a label head and two 5-component Gaussian
// mixture heads) and the evaluator's post-processing of its samples into the layout the image stage reads
// (seq2seq/evaluator/evaluator.py:74-139, the boxes.txt round trip, image_generation/miscc/load.py:653-776).
#include "common.cuh"

static int tblocks(long long total) {
  long long b = (total + 255) / 256;
  long long cap = (long long)og_num_sms() * 32;
  return (int)(b < cap ? (b < 1 ? 1 : b) : cap);
}

constexpr int BOX_H = 256;                 // decoder hidden units
constexpr int BOX_G = 4 * BOX_H;           // gate rows, order i, f, g, o
constexpr int BOX_AUG = 50;                // xy / wh / next_xy embedding width
constexpr int BOX_XIN = 2 * BOX_AUG;       // LSTM input columns other than the label embedding
constexpr int BOX_K = 5;                   // mixture components
constexpr int BOX_P = 6 * BOX_K;           // raw mixture parameters per head: pi, mu_x, mu_y, sigma_x, sigma_y, rho
constexpr int BOX_MAX_LABELS = 128;
constexpr int BOX_THREADS = BOX_H;         // thread j owns hidden unit j (its i, f, g, o rows and its c)
constexpr float BOX_TEMP = 0.4f;

// ---------------------------------------------------------------------------------------------------------------
// Label table: table[l][r] = (b_ih[r] + b_hh[r]) + sum_k W_ih[r][BOX_XIN + k] * emb[l][k], an fmaf chain in k order.
// og_box_decode starts every gate pre-activation from this entry and continues the same chain, so the table is a
// cache of the label-embedding columns of W_ih x, not a change in rounding.
// ---------------------------------------------------------------------------------------------------------------
__global__ void box_label_table_kernel(const float* __restrict__ emb, const float* __restrict__ w_ih,
                                       const float* __restrict__ b_ih, const float* __restrict__ b_hh, int NL,
                                       float* __restrict__ table) {
  const long long total = (long long)NL * BOX_G;
  const int ld = BOX_XIN + BOX_H;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int r = (int)(i % BOX_G);
    const long long l = i / BOX_G;
    float acc = b_ih[r] + b_hh[r];
    for (int k = 0; k < BOX_H; ++k) acc = fmaf(w_ih[(long long)r * ld + BOX_XIN + k], emb[l * BOX_H + k], acc);
    table[i] = acc;
  }
}

OG_API int og_box_label_table(const float* emb, const float* w_ih, const float* b_ih, const float* b_hh, int NL,
                              float* table, cudaStream_t stream) {
  if (NL < 1 || NL > BOX_MAX_LABELS) return (int)cudaErrorInvalidValue;
  box_label_table_kernel<<<tblocks((long long)NL * BOX_G), 256, 0, stream>>>(emb, w_ih, b_ih, b_hh, NL, table);
  OG_RETURN_LAST_ERROR();
}

// ---------------------------------------------------------------------------------------------------------------
// The decoder.  One CTA of 256 threads per tile of TILE samples runs every step of its samples, so the launch needs
// no host between steps.  The gate weights ([xy | wh] columns of W_ih and all of W_hh, 1.4 MB) are read from L2 in
// the transposed packing wt[k][r] (a warp reads 32 consecutive rows), and the label columns come from the label
// table.  Per step:
//   A. the xy / wh embeddings of each sample's inputs (threads k < 100);
//   B. thread j: the four gate pre-activations of unit j for every sample of the tile, one fmaf chain each in the
//      fixed order table, xy/wh columns 0..99, h 0..255; then the cell update (c stays in a register);
//   C. warp s, sample s: the label head (softmax, clamp, argmax), the xy mixture head, its sample, next_xy_embedding
//      of (new x, input y), the wh mixture head and its sample.  Dot products are per-lane fmaf chains in k order.
// Every sample's arithmetic is the same whatever the tile, B or its place in the batch, and no atomics are used, so
// replays are bitwise equal.
// ---------------------------------------------------------------------------------------------------------------
struct BoxDecArgs {
  const float* h0;      // [B][256] encoder h_n with the directions concatenated (forward, backward)
  const float* c0;      // [B][256]
  const float* table;   // [NL][1024]
  const float* wt;      // [356][1024]: rows 0..99 = W_ih[:, 0:100]^T, rows 100..355 = W_hh^T
  const float* xy_w; const float* xy_b;     // xy_embedding (50, 2), (50,)
  const float* wh_w; const float* wh_b;     // wh_embedding
  const float* nxy_w; const float* nxy_b;   // next_xy_embedding
  const float* lout_t; const float* lout_b; // [256][NL], (NL,)
  const float* xyo_t; const float* xyo_b;   // [256 + NL][30], (30,)
  const float* who_t; const float* who_b;   // [256 + NL + 50][30], (30,)
  const float* noise;   // [B][S][6]: u_xy, n1, n2, u_wh, n3, n4
  long long* labels;    // [B][S], -1 after the end
  float* samples;       // [B][S][4]: x, y, w, r (normalised), 0 after the end
  long long* steps;     // [B]
  float* dbg;           // [B][S][NL + 60] or null: p, then the xy and wh mixture parameters (pi, mu_x, mu_y, sigma_x,
                        // sigma_y, rho; sigma before the temperature scaling)
  float x0, y0, w0, r0; // the first step's inputs (the raw means)
  int B, S, NL, sos, eos;
};

// the mixture parameters of raw[30] (get_gmm_params, DecoderRNN.py:373-384) into par[30], and one sample from them
// (sample_next_state, :350-371) with the component chosen by numpy's rule for the uniform u
__device__ void box_gmm_sample(const float* raw, float* par, float u, float n1, float n2, float& x, float& y) {
  float m = raw[0];
  for (int k = 1; k < BOX_K; ++k) m = fmaxf(m, raw[k]);
  float e[BOX_K], s = 0.f;
  for (int k = 0; k < BOX_K; ++k) { e[k] = expf(raw[k] - m); s += e[k]; }
  for (int k = 0; k < BOX_K; ++k) {
    par[k] = e[k] / s;
    par[BOX_K + k] = raw[BOX_K + k];
    par[2 * BOX_K + k] = raw[2 * BOX_K + k];
    par[3 * BOX_K + k] = expf(raw[3 * BOX_K + k]);
    par[4 * BOX_K + k] = expf(raw[4 * BOX_K + k]);
    par[5 * BOX_K + k] = tanhf(raw[5 * BOX_K + k]);
  }
  // adjust_temp in float32: q = exp(log(pi) / T - max), normalised
  float q[BOX_K], qm = -INFINITY;
  for (int k = 0; k < BOX_K; ++k) { q[k] = logf(par[k]) / BOX_TEMP; qm = fmaxf(qm, q[k]); }
  float qs = 0.f;
  for (int k = 0; k < BOX_K; ++k) { q[k] = expf(q[k] - qm); qs += q[k]; }
  // np.random.choice: cdf = cumsum(p) / cdf[-1] in float64, component = searchsorted(cdf, u, side='right')
  double cdf[BOX_K], acc = 0.0;
  for (int k = 0; k < BOX_K; ++k) { acc += (double)(q[k] / qs); cdf[k] = acc; }
  int c = 0;
  for (int k = 0; k < BOX_K; ++k) c += (cdf[k] / cdf[BOX_K - 1] <= (double)u) ? 1 : 0;
  c = c < BOX_K - 1 ? c : BOX_K - 1;
  const float sc = (float)sqrt((double)BOX_TEMP);   // sigma *= np.sqrt(temperature) on a float32 tensor
  const float sx = par[3 * BOX_K + c] * sc, sy = par[4 * BOX_K + c] * sc, rho = par[5 * BOX_K + c];
  x = par[BOX_K + c] + sx * n1;
  y = par[2 * BOX_K + c] + sy * (rho * n1 + sqrtf(1.f - rho * rho) * n2);
}

template <int TILE>
__global__ void __launch_bounds__(BOX_THREADS, 1) box_decode_kernel(BoxDecArgs a) {
  __shared__ float s_x[TILE][BOX_XIN];
  __shared__ float s_h[TILE][BOX_H];
  __shared__ float s_p[TILE][BOX_MAX_LABELS];
  __shared__ float s_raw[TILE][BOX_P];
  __shared__ float s_nxy[TILE][BOX_AUG];
  __shared__ float s_in[TILE][4];          // x, y, w, r fed to the step
  __shared__ float s_par[TILE][BOX_P];
  __shared__ float s_xy[TILE][2];
  __shared__ int s_lab[TILE];
  __shared__ int s_live[TILE];

  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const long long b0 = (long long)blockIdx.x * TILE;
  float c[TILE];
#pragma unroll
  for (int s = 0; s < TILE; ++s) {
    const long long b = b0 + s;
    const bool in = b < a.B;
    c[s] = in ? a.c0[b * BOX_H + tid] : 0.f;
    s_h[s][tid] = in ? a.h0[b * BOX_H + tid] : 0.f;
    if (tid == 0) {
      s_live[s] = in ? 1 : 0;
      s_lab[s] = a.sos;
      s_in[s][0] = a.x0; s_in[s][1] = a.y0; s_in[s][2] = a.w0; s_in[s][3] = a.r0;
    }
    if (in) {                                // the outputs past each sample's end
      for (int t = tid; t < a.S; t += BOX_THREADS) {
        a.labels[b * a.S + t] = -1;
        for (int q = 0; q < 4; ++q) a.samples[(b * a.S + t) * 4 + q] = 0.f;
      }
      if (a.dbg)
        for (long long i = tid; i < (long long)a.S * (a.NL + 2 * BOX_P); i += BOX_THREADS)
          a.dbg[b * a.S * (a.NL + 2 * BOX_P) + i] = 0.f;
    }
  }
  __syncthreads();

  for (int t = 0; t < a.S; ++t) {
    // A. input embeddings
    for (int i = tid; i < TILE * BOX_XIN; i += BOX_THREADS) {
      const int s = i / BOX_XIN, k = i % BOX_XIN;
      if (!s_live[s]) continue;
      const float* w = k < BOX_AUG ? a.xy_w : a.wh_w;
      const float* bb = k < BOX_AUG ? a.xy_b : a.wh_b;
      const int j = k % BOX_AUG;
      const float u = k < BOX_AUG ? s_in[s][0] : s_in[s][2], v = k < BOX_AUG ? s_in[s][1] : s_in[s][3];
      s_x[s][k] = fmaf(w[2 * j + 1], v, fmaf(w[2 * j], u, bb[j]));
    }
    __syncthreads();

    // B. gates and cell of unit tid
    bool live[TILE];
    bool any = false;
#pragma unroll
    for (int s = 0; s < TILE; ++s) { live[s] = s_live[s] != 0; any |= live[s]; }
    if (!any) break;                         // block-uniform
    float acc[TILE][4];
#pragma unroll
    for (int s = 0; s < TILE; ++s) {
      const float* row = a.table + (long long)s_lab[s] * BOX_G + tid;
#pragma unroll
      for (int g = 0; g < 4; ++g) acc[s][g] = live[s] ? __ldg(row + g * BOX_H) : 0.f;
    }
#pragma unroll 4
    for (int k = 0; k < BOX_XIN + BOX_H; ++k) {
      const float* wr = a.wt + (long long)k * BOX_G + tid;
      float w[4];
#pragma unroll
      for (int g = 0; g < 4; ++g) w[g] = __ldg(wr + g * BOX_H);
#pragma unroll
      for (int s = 0; s < TILE; ++s) {
        const float xv = k < BOX_XIN ? s_x[s][k] : s_h[s][k - BOX_XIN];
#pragma unroll
        for (int g = 0; g < 4; ++g) acc[s][g] = fmaf(w[g], xv, acc[s][g]);
      }
    }
    __syncthreads();                         // every thread has read s_h
#pragma unroll
    for (int s = 0; s < TILE; ++s) {
      if (!live[s]) continue;
      const float ig = og_sigmoid(acc[s][0]), fg = og_sigmoid(acc[s][1]);
      const float gg = tanhf(acc[s][2]), og = og_sigmoid(acc[s][3]);
      c[s] = __fadd_rn(__fmul_rn(fg, c[s]), __fmul_rn(ig, gg));
      s_h[s][tid] = og * tanhf(c[s]);
    }
    __syncthreads();

    // C. heads and sampling, warp s for sample s
    if (warp < TILE && s_live[warp]) {
      const int s = warp;
      const long long b = b0 + s;
      const float* h = s_h[s];
      const float* nz = a.noise + (b * a.S + t) * 6;
      float* dbg = a.dbg ? a.dbg + (b * a.S + t) * (long long)(a.NL + 2 * BOX_P) : nullptr;
      // label head: p = softmax(l_out(h)).clamp(1e-5, 1); the label is the first index of max p
      float lg[BOX_MAX_LABELS / 32];
      float m = -INFINITY;
#pragma unroll
      for (int q = 0; q < BOX_MAX_LABELS / 32; ++q) {
        const int r = q * 32 + lane;
        float v = -INFINITY;
        if (r < a.NL) {
          v = a.lout_b[r];
          for (int k = 0; k < BOX_H; ++k) v = fmaf(a.lout_t[k * a.NL + r], h[k], v);
        }
        lg[q] = v;
        m = fmaxf(m, v);
      }
      m = warp_max(m);
      float sum = 0.f;
#pragma unroll
      for (int q = 0; q < BOX_MAX_LABELS / 32; ++q) {
        lg[q] = q * 32 + lane < a.NL ? expf(lg[q] - m) : 0.f;
        sum += lg[q];
      }
      sum = warp_sum(sum);
      float best = -1.f;
      int arg = 0;
#pragma unroll
      for (int q = 0; q < BOX_MAX_LABELS / 32; ++q) {
        const int r = q * 32 + lane;
        if (r < a.NL) {
          const float p = fminf(fmaxf(lg[q] / sum, 1e-5f), 1.f);
          s_p[s][r] = p;
          if (dbg) dbg[r] = p;
          if (p > best) { best = p; arg = r; }
        }
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        const float ob = __shfl_xor_sync(0xffffffffu, best, o);
        const int oa = __shfl_xor_sync(0xffffffffu, arg, o);
        if (ob > best || (ob == best && oa < arg)) { best = ob; arg = oa; }
      }
      __syncwarp();
      // xy head over cat(h, p)
      if (lane < BOX_P) {
        float v = a.xyo_b[lane];
        for (int k = 0; k < BOX_H; ++k) v = fmaf(a.xyo_t[k * BOX_P + lane], h[k], v);
        for (int k = 0; k < a.NL; ++k) v = fmaf(a.xyo_t[(BOX_H + k) * BOX_P + lane], s_p[s][k], v);
        s_raw[s][lane] = v;
      }
      __syncwarp();
      if (lane == 0) {
        float x, y;
        box_gmm_sample(s_raw[s], s_par[s], nz[0], nz[1], nz[2], x, y);
        s_xy[s][0] = x; s_xy[s][1] = y;
      }
      __syncwarp();
      if (dbg && lane < BOX_P) dbg[a.NL + lane] = s_par[s][lane];
      // next_xy_embedding of (the new x, this step's input y), DecoderRNN.py:166-170
      const float xn = s_xy[s][0];
      for (int j = lane; j < BOX_AUG; j += 32)
        s_nxy[s][j] = fmaf(a.nxy_w[2 * j + 1], s_in[s][1], fmaf(a.nxy_w[2 * j], xn, a.nxy_b[j]));
      __syncwarp();
      // wh head over cat(h, p, next_xy)
      if (lane < BOX_P) {
        float v = a.who_b[lane];
        for (int k = 0; k < BOX_H; ++k) v = fmaf(a.who_t[k * BOX_P + lane], h[k], v);
        for (int k = 0; k < a.NL; ++k) v = fmaf(a.who_t[(BOX_H + k) * BOX_P + lane], s_p[s][k], v);
        for (int k = 0; k < BOX_AUG; ++k) v = fmaf(a.who_t[(BOX_H + a.NL + k) * BOX_P + lane], s_nxy[s][k], v);
        s_raw[s][lane] = v;
      }
      __syncwarp();
      if (lane == 0) {
        float w, r;
        box_gmm_sample(s_raw[s], s_par[s], nz[3], nz[4], nz[5], w, r);
        a.labels[b * a.S + t] = arg;
        float* smp = a.samples + (b * a.S + t) * 4;
        smp[0] = s_xy[s][0]; smp[1] = s_xy[s][1]; smp[2] = w; smp[3] = r;
        s_in[s][0] = s_xy[s][0]; s_in[s][1] = s_xy[s][1]; s_in[s][2] = w; s_in[s][3] = r;
        s_lab[s] = arg;
        if (arg == a.eos || t == a.S - 1) {
          s_live[s] = 0;
          a.steps[b] = t + 1;
        }
      }
      __syncwarp();
      if (dbg && lane < BOX_P) dbg[a.NL + BOX_P + lane] = s_par[s][lane];
    }
    __syncthreads();
  }
}

template <int TILE>
static int box_decode_launch(const BoxDecArgs& a, cudaStream_t stream) {
  box_decode_kernel<TILE><<<og_cdiv(a.B, TILE), BOX_THREADS, 0, stream>>>(a);
  OG_RETURN_LAST_ERROR();
}

OG_API int og_box_decode(const float* h0, const float* c0, const float* table, const float* wt, const float* xy_w,
                         const float* xy_b, const float* wh_w, const float* wh_b, const float* nxy_w,
                         const float* nxy_b, const float* lout_t, const float* lout_b, const float* xyo_t,
                         const float* xyo_b, const float* who_t, const float* who_b, const float* noise, int B, int S,
                         int NL, int sos, int eos, float x0, float y0, float w0, float r0, long long* labels,
                         float* samples, long long* steps, float* dbg, cudaStream_t stream) {
  if (B < 0 || S < 1 || NL < 1 || NL > BOX_MAX_LABELS || sos < 0 || sos >= NL || eos < 0 || eos >= NL)
    return (int)cudaErrorInvalidValue;
  if (B == 0) return 0;
  BoxDecArgs a;
  a.h0 = h0; a.c0 = c0; a.table = table; a.wt = wt;
  a.xy_w = xy_w; a.xy_b = xy_b; a.wh_w = wh_w; a.wh_b = wh_b; a.nxy_w = nxy_w; a.nxy_b = nxy_b;
  a.lout_t = lout_t; a.lout_b = lout_b; a.xyo_t = xyo_t; a.xyo_b = xyo_b; a.who_t = who_t; a.who_b = who_b;
  a.noise = noise; a.labels = labels; a.samples = samples; a.steps = steps; a.dbg = dbg;
  a.x0 = x0; a.y0 = y0; a.w0 = w0; a.r0 = r0;
  a.B = B; a.S = S; a.NL = NL; a.sos = sos; a.eos = eos;
  // one sample per CTA while that fills at most a quarter of the SMs; larger batches share the weight reads of a step
  // between the samples of a tile
  if (B <= 32) return box_decode_launch<1>(a, stream);
  if (B <= 64) return box_decode_launch<2>(a, stream);
  if (B <= 128) return box_decode_launch<4>(a, stream);
  return box_decode_launch<8>(a, stream);
}

// ---------------------------------------------------------------------------------------------------------------
// Samples to layout, one thread per sample (at most S <= BOXES_NUM + 1 steps): de-normalise in float64, keep the
// steps with x, y, w, h > 0, drop the last kept one (or keep nothing when only one is kept), drop boxes with a
// special label, cap each class at max(trunc(mu + sigma * n), 2) boxes in order, centre -> corner and clip to the
// 256-pixel frame, the boxes.txt round trip int(float('%.2f' % v)), the ROI_MIN_SIZE filter and the three scales.
// ---------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ double box_txt_int(double v) {
  // v > 0 here.  '%.2f' rounds the exact binary value to two decimals, so it reaches the next integer exactly when
  // the fraction is at least 0.995; the double 0.995 lies just below 0.995 and the next double just above it.
  const double f = floor(v);
  return f + ((v - f) > 0.995 ? 1.0 : 0.0);
}

__global__ void box_layout_kernel(const long long* __restrict__ labels, const float* __restrict__ samples,
                                  const long long* __restrict__ steps, const double* __restrict__ mean_std,
                                  const long long* __restrict__ label_to_class, const double* __restrict__ count_stats,
                                  const float* __restrict__ noise_cnt, int B, int S, int NL, int C, int R,
                                  int min_size, double* __restrict__ rois, double* __restrict__ fm_rois,
                                  long long* __restrict__ roi_cls, long long* __restrict__ num_rois) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  constexpr int MAXS = 16;                 // steps per sample (S <= BOXES_NUM + 1 for the sampler)
  int kept[MAXS], cls[MAXS];
  double box[MAXS][4];
  int n = 0;
  const int st = (int)steps[b];
  for (int t = 0; t < st && t < S; ++t) {
    const float* p = samples + ((long long)b * S + t) * 4;
    // product and sum rounded separately, as numpy does (a contracted fma could move a value across a boundary)
    const double x = __dadd_rn(__dmul_rn((double)p[0], mean_std[1]), mean_std[0]);
    const double y = __dadd_rn(__dmul_rn((double)p[1], mean_std[3]), mean_std[2]);
    const double w = __dadd_rn(__dmul_rn((double)p[2], mean_std[5]), mean_std[4]);
    const double h = __dmul_rn(w, __dadd_rn(__dmul_rn((double)p[3], mean_std[7]), mean_std[6]));
    if (x > 0 && y > 0 && w > 0 && h > 0) {
      box[n][0] = x; box[n][1] = y; box[n][2] = w; box[n][3] = h;
      kept[n++] = t;
    }
  }
  n = n > 1 ? n - 1 : 0;                   // drop the last kept step
  int m = 0;
  for (int i = 0; i < n; ++i) {            // special labels (<pad>, <sos>, <unk>) have no class: drop the box
    const long long l = labels[(long long)b * S + kept[i]];
    const long long c = (l >= 0 && l < NL) ? label_to_class[l] : -1;
    if (c < 0) continue;
    for (int q = 0; q < 4; ++q) box[m][q] = box[i][q];
    cls[m++] = (int)c;
  }
  int out = 0;
  for (int i = 0; i < m; ++i) {
    int before = 0;
    for (int j = 0; j < i; ++j) before += cls[j] == cls[i];
    const double draw = __dadd_rn(count_stats[2 * cls[i]],
                                  __dmul_rn(count_stats[2 * cls[i] + 1], (double)noise_cnt[(long long)b * C + cls[i]]));
    const double thr = fmax(trunc(draw), 2.0);
    if ((double)before >= thr) continue;
    double x = __dsub_rn(box[i][0], __dmul_rn(box[i][2], 0.5));     // x - w / 2.0
    x = fmin(fmax(x, 1.0), 255.0);
    double y = __dsub_rn(box[i][1], __dmul_rn(box[i][3], 0.5));
    y = fmin(fmax(y, 1.0), 255.0);
    const double w = fmin(box[i][2], 256.0 - x), h = fmin(box[i][3], 256.0 - y);
    const double v[4] = {box_txt_int(x), box_txt_int(y), box_txt_int(w), box_txt_int(h)};
    if (v[2] < min_size && v[3] < min_size) continue;
    if (out >= R) break;
    for (int k = 0; k < 3; ++k) {
      double* r = rois + (((long long)k * B + b) * R + out) * 6;
      const double sc = (double)(64 << k) / 256.0;
      for (int q = 0; q < 4; ++q) r[q] = v[q] * sc;
      r[4] = cls[i]; r[5] = 0.0;
    }
    double* f = fm_rois + ((long long)b * R + out) * 6;
    for (int q = 0; q < 4; ++q) f[q] = v[q] * 0.25 / 2.0;
    f[4] = cls[i]; f[5] = 0.0;
    roi_cls[(long long)b * R + out] = cls[i];
    ++out;
  }
  num_rois[b] = out;
  for (int o = out; o < R; ++o) {
    for (int k = 0; k < 3; ++k)
      for (int q = 0; q < 6; ++q) rois[(((long long)k * B + b) * R + o) * 6 + q] = 0.0;
    for (int q = 0; q < 6; ++q) fm_rois[((long long)b * R + o) * 6 + q] = 0.0;
    roi_cls[(long long)b * R + o] = 0;
  }
}

OG_API int og_box_layout(const long long* labels, const float* samples, const long long* steps,
                         const double* mean_std, const long long* label_to_class, const double* count_stats,
                         const float* noise_cnt, int B, int S, int NL, int C, int R, int min_size, double* rois,
                         double* fm_rois, long long* roi_cls, long long* num_rois, cudaStream_t stream) {
  if (B < 0 || S < 1 || S > 16 || NL < 1 || C < 1 || R < 1) return (int)cudaErrorInvalidValue;
  if (B == 0) return 0;
  box_layout_kernel<<<og_cdiv(B, 64), 64, 0, stream>>>(labels, samples, steps, mean_std, label_to_class, count_stats,
                                                       noise_cnt, B, S, NL, C, R, min_size, rois, fm_rois, roi_cls,
                                                       num_rois);
  OG_RETURN_LAST_ERROR();
}
