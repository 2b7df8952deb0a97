// Shape generator stage of box-conditioned sampling: the one-hot box maps SHP_G_NET reads (ref: miscc/load.py:178-189,
// 625-641), its ConvLSTM cell (ref: model.py:818-863) with the bidirectional concat of SHP_G_NET.forward
// (model.py:949-964), the crop by the box feature maps (model.py:969-972), and the heat maps built from generated
// masks (ref: miscc/utils.py:524-584 form_hmaps).  The convolutions around them are the library's conv kernels.
#include "common.cuh"

static int sblocks(long long total) {
  long long b = (total + 255) / 256;
  long long cap = (long long)og_num_sms() * 32;
  return (int)(b < cap ? (b < 1 ? 1 : b) : cap);
}

// ---------------------------------------------------------------------------------------------------------------
// Box maps.  One box edge of the loader: min(int(round(v)), size - 1), round = numpy round-half-to-even on float64
// (rint), then used as a Python slice bound (a negative bound counts from the end).
// ---------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ int box_edge(double v, int size) {
  double r = fmin(rint(v), (double)(size - 1));
  int i = (int)fmax(r, -2.0 * size);
  if (i < 0) i += size;
  return i < 0 ? 0 : i;
}

// maps: NHWC [2][B][R][S][S][Cp] (forward then backward sequence), one float4 of channels per thread
__global__ void bbox_maps_kernel(const double* __restrict__ rois, int rs, const long long* __restrict__ cls,
                                 const long long* __restrict__ num_rois, int B, int boxes, int R, int S, int Cp4,
                                 long long total, float* __restrict__ maps) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int q = (int)(i % Cp4);
    long long r = i / Cp4;
    const int x = (int)(r % S);
    r /= S;
    const int y = (int)(r % S);
    r /= S;                                            // image index over [2][B][R]
    const int t = (int)(r % R);
    const int b = (int)((r / R) % B);
    const int dir = (int)(r / ((long long)R * B));
    const int slot = dir ? boxes - 1 - t : t;          // bbox_maps_bwd = bbox_maps_fwd[::-1] over all slots, then [:R]
    float4 o = make_float4(0.f, 0.f, 0.f, 0.f);
    if (slot >= 0 && slot < (int)num_rois[b]) {
      const double* row = rois + ((long long)b * boxes + slot) * rs;
      const int x0 = box_edge(row[0], S), y0 = box_edge(row[1], S);
      const int x1 = box_edge(row[0] + row[2], S), y1 = box_edge(row[1] + row[3], S);
      const int c = (int)cls[(long long)b * boxes + slot] - 4 * q;
      if (x >= x0 && x < x1 && y >= y0 && y < y1 && c >= 0 && c < 4) {
        if (c == 0) o.x = 1.f;
        else if (c == 1) o.y = 1.f;
        else if (c == 2) o.z = 1.f;
        else o.w = 1.f;
      }
    }
    st4(maps + i * 4, o);
  }
}

// fmaps: [B][R][F][F] from fm_rois / 2 (the 32 -> 16 scale of load.py:637-640)
__global__ void bbox_fmaps_kernel(const double* __restrict__ fm_rois, int fs, const long long* __restrict__ num_rois,
                                  int boxes, int R, int F, long long total, float* __restrict__ fmaps) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int x = (int)(i % F);
    const int y = (int)((i / F) % F);
    const int t = (int)((i / ((long long)F * F)) % R);
    const int b = (int)(i / ((long long)F * F * R));
    float v = 0.f;
    if (t < (int)num_rois[b]) {
      const double* row = fm_rois + ((long long)b * boxes + t) * fs;
      const int x0 = box_edge(row[0] / 2.0, F), y0 = box_edge(row[1] / 2.0, F);
      const int x1 = box_edge(row[0] / 2.0 + row[2] / 2.0, F), y1 = box_edge(row[1] / 2.0 + row[3] / 2.0, F);
      if (x >= x0 && x < x1 && y >= y0 && y < y1) v = 1.f;
    }
    fmaps[i] = v;
  }
}

OG_API int og_form_bbox_maps(const double* rois, int rois_stride, const double* fm_rois, int fm_stride,
                             const long long* cls, const long long* num_rois, int B, int boxes, int R, int ncls, int Cp,
                             int S, int F, float* maps, float* fmaps, cudaStream_t stream) {
  if (Cp % 4 || Cp < ncls || R > boxes) return (int)cudaErrorInvalidValue;
  const long long total = 2LL * B * R * S * S * (Cp / 4);
  if (total == 0) return 0;
  bbox_maps_kernel<<<sblocks(total), 256, 0, stream>>>(rois, rois_stride, cls, num_rois, B, boxes, R, S, Cp / 4, total,
                                                      maps);
  OG_CHECK(cudaGetLastError());
  const long long ftotal = (long long)B * R * F * F;
  bbox_fmaps_kernel<<<sblocks(ftotal), 256, 0, stream>>>(fm_rois, fm_stride, num_rois, boxes, R, F, ftotal, fmaps);
  OG_RETURN_LAST_ERROR();
}

// ---------------------------------------------------------------------------------------------------------------
// ConvLSTM cell, both directions in one launch.  gates = gx[b*R + t] (x-part of Gates with its bias, computed for every
// step up front) + gh[b] (conv(h_{t-1}, W_h); absent at t = 0, where h = 0); chunk order in, remember, out, cell.
// Writes h into the next step's conv operand and straight into the 2*Ch + Cz channel joint buffer of jointConv:
// forward h at slot t, backward h at slot R-1-t (model.py:962).
// ---------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ float lstm_c(float f, float cp, float i, float g) {
  return __fadd_rn(__fmul_rn(f, cp), __fmul_rn(i, g));       // (remember * prev_cell) + (in * cell_gate), unfused
}

__global__ void clstm_cell_kernel(const float* __restrict__ gx_f, const float* __restrict__ gx_b,
                                  const float* __restrict__ gh_f, const float* __restrict__ gh_b, float* c_f, float* c_b,
                                  float* __restrict__ h_f, float* __restrict__ h_b, float* __restrict__ joint, int B,
                                  int R, int t, int HW, int Ch, int Cj, long long per_dir) {
  const int Ch4 = Ch / 4;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < 2 * per_dir;
       i += (long long)gridDim.x * blockDim.x) {
    const int dir = (int)(i / per_dir);
    long long r = i - dir * per_dir;
    const int q = (int)(r % Ch4);
    r /= Ch4;
    const int p = (int)(r % HW);
    const int b = (int)(r / HW);
    const float* gx = (dir ? gx_b : gx_f) + (((long long)b * R + t) * HW + p) * 4 * Ch + q * 4;
    const float* gh = dir ? gh_b : gh_f;
    float* cs = (dir ? c_b : c_f) + ((long long)b * HW + p) * Ch + q * 4;
    float4 a[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) a[k] = ldg4(gx + k * Ch);
    if (gh != nullptr) {
      const float* ghp = gh + ((long long)b * HW + p) * 4 * Ch + q * 4;
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const float4 u = ldg4(ghp + k * Ch);
        a[k].x += u.x; a[k].y += u.y; a[k].z += u.z; a[k].w += u.w;
      }
    }
    const float4 cp = gh != nullptr ? *reinterpret_cast<const float4*>(cs) : make_float4(0.f, 0.f, 0.f, 0.f);
    float4 c, h;
#define OG_LSTM_LANE(L)                                                                       \
    {                                                                                         \
      const float ig = og_sigmoid(a[0].L), fg = og_sigmoid(a[1].L), og = og_sigmoid(a[2].L); \
      const float gg = tanhf(a[3].L);                                                         \
      c.L = lstm_c(fg, cp.L, ig, gg);                                                         \
      h.L = og * tanhf(c.L);                                                                  \
    }
    OG_LSTM_LANE(x) OG_LSTM_LANE(y) OG_LSTM_LANE(z) OG_LSTM_LANE(w)
#undef OG_LSTM_LANE
    st4(cs, c);
    st4((dir ? h_b : h_f) + ((long long)b * HW + p) * Ch + q * 4, h);
    const int slot = dir ? R - 1 - t : t;
    st4(joint + (((long long)b * R + slot) * HW + p) * Cj + dir * Ch + q * 4, h);
  }
}

OG_API int og_clstm_cell(const float* gx_f, const float* gx_b, const float* gh_f, const float* gh_b, float* c_f,
                         float* c_b, float* h_f, float* h_b, float* joint, int B, int R, int t, int HW, int Ch, int Cj,
                         cudaStream_t stream) {
  if (Ch % 4 || Cj % 4 || Cj < 2 * Ch || t < 0 || t >= R || ((gh_f == nullptr) != (gh_b == nullptr)))
    return (int)cudaErrorInvalidValue;
  const long long per_dir = (long long)B * HW * (Ch / 4);
  if (per_dir == 0) return 0;
  clstm_cell_kernel<<<sblocks(2 * per_dir), 256, 0, stream>>>(gx_f, gx_b, gh_f, gh_b, c_f, c_b, h_f, h_b, joint, B, R, t,
                                                            HW, Ch, Cj, per_dir);
  OG_RETURN_LAST_ERROR();
}

// crop (model.py:969-972): out[p][c] = x[p][c] * s[p], s = the box feature map of the pixel's image
__global__ void mul_pixels_kernel(const float* __restrict__ x, const float* __restrict__ s, int C4, long long total,
                                  float* __restrict__ out) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const float v = s[i / C4];
    const float4 a = ldg4(x + i * 4);
    st4(out + i * 4, make_float4(a.x * v, a.y * v, a.z * v, a.w * v));
  }
}
OG_API int og_mul_pixels(const float* x, const float* s, long long P, int C, float* out, cudaStream_t stream) {
  if (C % 4) return (int)cudaErrorInvalidValue;
  const long long total = P * (C / 4);
  if (total == 0) return 0;
  mul_pixels_kernel<<<sblocks(total), 256, 0, stream>>>(x, s, C / 4, total, out);
  OG_RETURN_LAST_ERROR();
}

// ---------------------------------------------------------------------------------------------------------------
// Heat maps from generated masks (form_hmaps).  slots: NHWC [B][P][Cs] (lane t = roi slot t at the largest heat-map
// size), hmap: NHWC [B][P][Cp].  Min / max over a map are exact operations, and the per-CTA partials are combined in a
// fixed order, so results are bitwise repeatable.  Three passes:
//   1. per-slot partial min / max;
//   2. every slot t < num_rois[b] normalised in place ((v - min) / (max - min); a constant map below 0.6 -> 0, a
//      constant map >= 0.6 unchanged); the class map is written (zero, then max over the slots of each class), and
//      the partial min / max of each slot's class channel;
//   3. every present class channel renormalised by the same rule (once per class: the rule is idempotent).
// Slots t >= num_rois[b] keep their raw values (utils.py:542-558 only touches the first num_rois slots).
// ---------------------------------------------------------------------------------------------------------------
constexpr int GH_MAX_SLOTS = 16;
constexpr int GH_THREADS = 256;
constexpr int GH_PIX_PER_CTA = 1024;

__device__ __forceinline__ float norm_rule(float v, float lo, float hi) {
  if (lo != hi) return (v - lo) / (hi - lo);
  return hi < 0.6f ? v * 0.f : v;
}

// reduce per-thread (lo[t], hi[t]) over the CTA and write them to part[t][2]
__device__ void cta_minmax(float (&lo)[GH_MAX_SLOTS], float (&hi)[GH_MAX_SLOTS], int n, float* part) {
  __shared__ float s_lo[GH_THREADS / 32][GH_MAX_SLOTS], s_hi[GH_THREADS / 32][GH_MAX_SLOTS];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
#pragma unroll
  for (int t = 0; t < GH_MAX_SLOTS; ++t) {
    if (t >= n) break;
    float a = lo[t], b = hi[t];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      a = fminf(a, __shfl_xor_sync(0xffffffffu, a, o));
      b = fmaxf(b, __shfl_xor_sync(0xffffffffu, b, o));
    }
    if (lane == 0) { s_lo[warp][t] = a; s_hi[warp][t] = b; }
  }
  __syncthreads();
  if (threadIdx.x < n) {
    float a = INFINITY, b = -INFINITY;
    for (int w = 0; w < GH_THREADS / 32; ++w) { a = fminf(a, s_lo[w][threadIdx.x]); b = fmaxf(b, s_hi[w][threadIdx.x]); }
    part[threadIdx.x * 2] = a;
    part[threadIdx.x * 2 + 1] = b;
  }
}

// final (lo, hi) of slot t from the nblk partials of image b, in block order
__device__ __forceinline__ void final_minmax(const float* part, int nblk, int Cs, int t, float& lo, float& hi) {
  lo = INFINITY; hi = -INFINITY;
  for (int k = 0; k < nblk; ++k) {
    lo = fminf(lo, part[((long long)k * Cs + t) * 2]);
    hi = fmaxf(hi, part[((long long)k * Cs + t) * 2 + 1]);
  }
}

struct GenHmapArgs {
  float* slots;
  float* hmap;
  const long long* cls;
  const long long* num_rois;
  float* part_s;      // [B][nblk][Cs][2]
  float* part_c;      // [B][nblk][Cs][2]
  long long P;
  int Cs, Cp, boxes, ncls, nblk;
};

__device__ __forceinline__ int slot_count(const GenHmapArgs& a, int b) {
  int n = (int)a.num_rois[b];
  n = n < a.Cs ? n : a.Cs;
  return n < a.boxes ? (n < 0 ? 0 : n) : a.boxes;
}

__global__ void __launch_bounds__(GH_THREADS) gen_slot_minmax_kernel(GenHmapArgs a) {
  const int b = blockIdx.y, n = slot_count(a, b);
  float lo[GH_MAX_SLOTS], hi[GH_MAX_SLOTS];
#pragma unroll
  for (int t = 0; t < GH_MAX_SLOTS; ++t) { lo[t] = INFINITY; hi[t] = -INFINITY; }
  const long long p0 = (long long)blockIdx.x * GH_PIX_PER_CTA;
  for (long long p = p0 + threadIdx.x; p < p0 + GH_PIX_PER_CTA && p < a.P; p += GH_THREADS) {
    const float* row = a.slots + ((long long)b * a.P + p) * a.Cs;
#pragma unroll
    for (int t = 0; t < GH_MAX_SLOTS; ++t)
      if (t < n) { const float v = row[t]; lo[t] = fminf(lo[t], v); hi[t] = fmaxf(hi[t], v); }
  }
  cta_minmax(lo, hi, n, a.part_s + ((long long)b * a.nblk + blockIdx.x) * a.Cs * 2);
}

__global__ void __launch_bounds__(GH_THREADS) gen_composite_kernel(GenHmapArgs a) {
  const int b = blockIdx.y, n = slot_count(a, b);
  __shared__ float s_lo[GH_MAX_SLOTS], s_hi[GH_MAX_SLOTS];
  __shared__ int s_cls[GH_MAX_SLOTS];
  if (threadIdx.x < n) {
    final_minmax(a.part_s + (long long)b * a.nblk * a.Cs * 2, a.nblk, a.Cs, threadIdx.x, s_lo[threadIdx.x],
                 s_hi[threadIdx.x]);
    const long long c = a.cls[(long long)b * a.boxes + threadIdx.x];
    s_cls[threadIdx.x] = (c >= 0 && c < a.ncls) ? (int)c : -1;
  }
  __syncthreads();
  float lo[GH_MAX_SLOTS], hi[GH_MAX_SLOTS];
#pragma unroll
  for (int t = 0; t < GH_MAX_SLOTS; ++t) { lo[t] = INFINITY; hi[t] = -INFINITY; }
  const long long p0 = (long long)blockIdx.x * GH_PIX_PER_CTA;
  for (long long p = p0 + threadIdx.x; p < p0 + GH_PIX_PER_CTA && p < a.P; p += GH_THREADS) {
    float* row = a.slots + ((long long)b * a.P + p) * a.Cs;
    float* out = a.hmap + ((long long)b * a.P + p) * a.Cp;
    float v[GH_MAX_SLOTS];
#pragma unroll
    for (int t = 0; t < GH_MAX_SLOTS; ++t)
      if (t < n) { v[t] = norm_rule(row[t], s_lo[t], s_hi[t]); row[t] = v[t]; }
    for (int c = 0; c < a.Cp; c += 4) st4(out + c, make_float4(0.f, 0.f, 0.f, 0.f));
#pragma unroll
    for (int t = 0; t < GH_MAX_SLOTS; ++t) {
      if (t >= n || s_cls[t] < 0) continue;
      float m = 0.f;                                   // raw_gen_hmap starts at zero (utils.py:531)
#pragma unroll
      for (int u = 0; u < GH_MAX_SLOTS; ++u)           // slots in roi order, each max-composited in turn
        if (u < n && s_cls[u] == s_cls[t]) m = fmaxf(v[u], m);
      out[s_cls[t]] = m;
      lo[t] = fminf(lo[t], m);
      hi[t] = fmaxf(hi[t], m);
    }
  }
  cta_minmax(lo, hi, n, a.part_c + ((long long)b * a.nblk + blockIdx.x) * a.Cs * 2);
}

__global__ void __launch_bounds__(GH_THREADS) gen_class_norm_kernel(GenHmapArgs a) {
  const int b = blockIdx.y, n = slot_count(a, b);
  __shared__ float s_lo[GH_MAX_SLOTS], s_hi[GH_MAX_SLOTS];
  __shared__ int s_cls[GH_MAX_SLOTS];
  if (threadIdx.x < n) {
    final_minmax(a.part_c + (long long)b * a.nblk * a.Cs * 2, a.nblk, a.Cs, threadIdx.x, s_lo[threadIdx.x],
                 s_hi[threadIdx.x]);
    const long long c = a.cls[(long long)b * a.boxes + threadIdx.x];
    int k = (c >= 0 && c < a.ncls) ? (int)c : -1;
    for (int u = 0; u < threadIdx.x && k >= 0; ++u)    // a class listed twice is renormalised once
      if (a.cls[(long long)b * a.boxes + u] == c) k = -1;
    s_cls[threadIdx.x] = k;
  }
  __syncthreads();
  const long long p0 = (long long)blockIdx.x * GH_PIX_PER_CTA;
  for (long long p = p0 + threadIdx.x; p < p0 + GH_PIX_PER_CTA && p < a.P; p += GH_THREADS) {
    float* out = a.hmap + ((long long)b * a.P + p) * a.Cp;
#pragma unroll
    for (int t = 0; t < GH_MAX_SLOTS; ++t)
      if (t < n && s_cls[t] >= 0) out[s_cls[t]] = norm_rule(out[s_cls[t]], s_lo[t], s_hi[t]);
  }
}

OG_API int og_gen_hmaps(float* slots, int B, long long P, int Cs, const long long* cls, int boxes,
                        const long long* num_rois, int ncls, int Cp, float* hmap, cudaStream_t stream) {
  if (Cs > GH_MAX_SLOTS || Cp % 4 || Cp < ncls) return (int)cudaErrorInvalidValue;
  if (B == 0 || P == 0) return 0;
  GenHmapArgs a;
  a.slots = slots; a.hmap = hmap; a.cls = cls; a.num_rois = num_rois; a.P = P;
  a.Cs = Cs; a.Cp = Cp; a.boxes = boxes; a.ncls = ncls; a.nblk = og_cdiv(P, GH_PIX_PER_CTA);
  float* work = nullptr;
  OG_CHECK(og_work_alloc(&work, (size_t)2 * B * a.nblk * Cs * 2, stream));
  a.part_s = work;
  a.part_c = work + (size_t)B * a.nblk * Cs * 2;
  const dim3 grid(a.nblk, B);
  gen_slot_minmax_kernel<<<grid, GH_THREADS, 0, stream>>>(a);
  cudaError_t e = cudaGetLastError();
  if (e == cudaSuccess) {
    gen_composite_kernel<<<grid, GH_THREADS, 0, stream>>>(a);
    e = cudaGetLastError();
  }
  if (e == cudaSuccess) {
    gen_class_norm_kernel<<<grid, GH_THREADS, 0, stream>>>(a);
    e = cudaGetLastError();
  }
  const cudaError_t f = cudaFreeAsync(work, stream);
  return (int)(e != cudaSuccess ? e : f);
}
