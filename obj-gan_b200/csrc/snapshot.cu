// The attention-map snapshot canvases of the training and evaluation loops (ref: miscc/utils.py:59-306,
// build_super_images / build_super_shape_images): one uint8 HWC canvas per PNG, everything but the caption glyphs.
//
// Per image i < nvis the canvas holds a caption strip of `strip` rows, then the row [lr image, pad, (map_j, pad) x
// (words+1)] and the row [image, pad, (merged_j, pad) x (words+1)], tiles vis x vis, pads 2 zero columns.  Map 0 is
// the max over the image's maps; maps j > n_i (n_i the image's map count) are zero tiles.
//
// Launches, upscale = vis / att > 1 (skimage 0.14 pyramid_expand(sigma=20), float64 throughout):
//   prep    the word-max map and every map's min / max (the clip bounds of the resize)
//   vblur   bilinear resize (half-pixel centres, numpy-reflect neighbours, clipped to the map's min / max) of a column
//           strip made in shared memory with its 80-pixel apron (scipy reflect), then the vertical 161-tap Gaussian
//   hblur   the horizontal Gaussian in place, one min / max pair per block (no atomics: the partials are reduced in
//           a fixed order by minmax)
//   minmax  the normalisation bounds: per image (starting from min 1, max 0, like the reference) or per map
//   compose image tiles (torch bilinear upsample, fp32), normalised and truncated maps, the 210/255 blend of PIL's
//           paste, pads and strip backgrounds
// With upscale 1 (shape snapshots) vblur / hblur are skipped and the map arithmetic is float32, in the reference's
// operation order with explicit rounding.
#include "common.cuh"

namespace {

constexpr int RADIUS = 80;          // int(4 * sigma + 0.5), sigma = 20 (scipy.ndimage.gaussian_filter, truncate 4)
constexpr int VTX = 8;              // columns per vblur block
constexpr int HRY = 4;              // rows per hblur block
constexpr int NT = 256;

__constant__ unsigned char kColor[20][3] = {
    {128, 64, 128}, {244, 35, 232}, {70, 70, 70},   {102, 102, 156}, {190, 153, 153}, {153, 153, 153}, {250, 170, 30},
    {220, 220, 0},  {107, 142, 35}, {152, 251, 152}, {70, 130, 180}, {220, 20, 60},   {255, 0, 0},     {0, 0, 142},
    {119, 11, 32},  {0, 60, 100},   {0, 80, 100},   {0, 0, 230},     {0, 0, 70},      {0, 0, 0}};

__device__ __forceinline__ int map_count(const long long* lens, int L, int i) {
  return lens ? (int)min((long long)L, lens[i]) : L;
}

// skimage's 'reflect' (numpy reflect: mirror, edge not repeated) for the one-pixel overhang of the bilinear resize
__device__ __forceinline__ int reflect_np(int k, int n) {
  if (n == 1) return 0;
  return k < 0 ? -k : (k > n - 1 ? 2 * (n - 1) - k : k);
}
// scipy.ndimage's 'reflect' (half-sample symmetric) for the Gaussian's apron; n > RADIUS, so one mirror suffices
__device__ __forceinline__ int reflect_half(int k, int n) { return k < 0 ? -k - 1 : (k >= n ? 2 * n - 1 - k : k); }

// exp(-x^2 / (2 sigma^2)) / sum for x = 0..RADIUS (the symmetric half of scipy's _gaussian_kernel1d)
__device__ void gauss_weights(double* w) {
  if (threadIdx.x <= RADIUS) w[threadIdx.x] = exp(-0.5 / 400.0 * (double)(threadIdx.x * threadIdx.x));
  __syncthreads();
  __shared__ double total;
  if (threadIdx.x == 0) {
    double s = w[0];
    for (int k = 1; k <= RADIUS; ++k) s += 2.0 * w[k];
    total = s;
  }
  __syncthreads();
  const double s = total;
  __syncthreads();
  if (threadIdx.x <= RADIUS) w[threadIdx.x] /= s;
  __syncthreads();
}

template <typename T>
__device__ void block_minmax(T& mn, T& mx) {
  __shared__ T smn[NT / 32], smx[NT / 32];
  for (int o = 16; o > 0; o >>= 1) {
    const T a = __shfl_xor_sync(0xffffffffu, mn, o), b = __shfl_xor_sync(0xffffffffu, mx, o);
    mn = a < mn ? a : mn;
    mx = b > mx ? b : mx;
  }
  const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
  if (l == 0) { smn[w] = mn; smx[w] = mx; }
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int k = 1; k < NT / 32; ++k) {
      mn = smn[k] < mn ? smn[k] : mn;
      mx = smx[k] > mx ? smx[k] : mx;
    }
  }
}

__device__ __forceinline__ const float* map_src(const float* maps, const float* maxmap, int L, int P, int i, int j) {
  return j == 0 ? maxmap + (size_t)i * P : maps + ((size_t)i * L + (j - 1)) * P;
}

__global__ void __launch_bounds__(NT) snap_prep_kernel(const float* __restrict__ maps, int L, int P,
                                                       const long long* __restrict__ lens, float* __restrict__ maxmap,
                                                       double* __restrict__ mm0) {
  const int j = blockIdx.x, i = blockIdx.y, M = L + 1;
  const int n = map_count(lens, L, i);
  if (j > n) return;
  float mn = INFINITY, mx = -INFINITY;
  if (j == 0) {
    const float* base = maps + (size_t)i * L * P;
    for (int p = threadIdx.x; p < P; p += NT) {
      float v = n > 0 ? base[p] : 0.f;
      for (int l = 1; l < n; ++l) {
        const float x = base[(size_t)l * P + p];
        v = x > v ? x : v;
      }
      maxmap[(size_t)i * P + p] = v;
      mn = fminf(mn, v);
      mx = fmaxf(mx, v);
    }
  } else {
    const float* src = maps + ((size_t)i * L + (j - 1)) * P;
    for (int p = threadIdx.x; p < P; p += NT) {
      const float v = src[p];
      mn = fminf(mn, v);
      mx = fmaxf(mx, v);
    }
  }
  block_minmax(mn, mx);
  if (threadIdx.x == 0) {
    mm0[((size_t)i * M + j) * 2] = mn;
    mm0[((size_t)i * M + j) * 2 + 1] = mx;
  }
}

// skimage.transform.resize(order=1, mode='reflect', clip=True) of an att x att map at output pixel (y, x), in float64
__device__ __forceinline__ double resized(const float* __restrict__ a, int att, int up, int y, int x, double lo,
                                          double hi) {
  const double sr = __dsub_rn(__ddiv_rn(__dadd_rn((double)y, 0.5), (double)up), 0.5);
  const double sc = __dsub_rn(__ddiv_rn(__dadd_rn((double)x, 0.5), (double)up), 0.5);
  const int r0 = (int)floor(sr), c0 = (int)floor(sc), r1 = (int)ceil(sr), c1 = (int)ceil(sc);
  const double dr = __dsub_rn(sr, (double)r0), dc = __dsub_rn(sc, (double)c0);
  const int R0 = reflect_np(r0, att), R1 = reflect_np(r1, att), C0 = reflect_np(c0, att), C1 = reflect_np(c1, att);
  const double ndc = __dsub_rn(1.0, dc), ndr = __dsub_rn(1.0, dr);
  const double top = __dadd_rn(__dmul_rn(ndc, (double)a[R0 * att + C0]), __dmul_rn(dc, (double)a[R0 * att + C1]));
  const double bot = __dadd_rn(__dmul_rn(ndc, (double)a[R1 * att + C0]), __dmul_rn(dc, (double)a[R1 * att + C1]));
  const double v = __dadd_rn(__dmul_rn(ndr, top), __dmul_rn(dr, bot));
  return fmin(fmax(v, lo), hi);
}

__global__ void __launch_bounds__(NT) snap_vblur_kernel(const float* __restrict__ maps, const float* __restrict__ maxmap,
                                                        int L, int att, const long long* __restrict__ lens, int vis,
                                                        const double* __restrict__ mm0, double* __restrict__ work) {
  extern __shared__ double sm[];
  double* w = sm;                         // RADIUS + 1 weights
  double* col = sm + RADIUS + 1;          // (vis + 2 RADIUS) x VTX
  const int j = blockIdx.y, i = blockIdx.z, M = L + 1, up = vis / att;
  if (j > map_count(lens, L, i)) return;
  gauss_weights(w);
  const float* src = map_src(maps, maxmap, L, att * att, i, j);
  const double lo = mm0[((size_t)i * M + j) * 2], hi = mm0[((size_t)i * M + j) * 2 + 1];
  const int x0 = blockIdx.x * VTX, ext = vis + 2 * RADIUS;
  for (int idx = threadIdx.x; idx < ext * VTX; idx += NT) {
    const int rr = idx / VTX, cx = idx - rr * VTX, x = x0 + cx;
    col[idx] = x < vis ? resized(src, att, up, reflect_half(rr - RADIUS, vis), x, lo, hi) : 0.0;
  }
  __syncthreads();
  double* dst = work + ((size_t)i * M + j) * vis * vis;
  for (int idx = threadIdx.x; idx < vis * VTX; idx += NT) {
    const int y = idx / VTX, cx = idx - y * VTX, x = x0 + cx;
    if (x >= vis) continue;
    const double* c = col + (y + RADIUS) * VTX + cx;
    double acc = w[0] * c[0];
    for (int k = 1; k <= RADIUS; ++k) acc = fma(w[k], c[-k * VTX] + c[k * VTX], acc);
    dst[(size_t)y * vis + x] = acc;
  }
}

__global__ void __launch_bounds__(NT) snap_hblur_kernel(int L, const long long* __restrict__ lens, int vis,
                                                        double* __restrict__ work, double* __restrict__ part) {
  extern __shared__ double sm[];
  double* w = sm;
  double* buf = sm + RADIUS + 1;          // HRY x (vis + 2 RADIUS)
  const int j = blockIdx.y, i = blockIdx.z, M = L + 1, K = gridDim.x;
  if (j > map_count(lens, L, i)) return;
  gauss_weights(w);
  const int y0 = blockIdx.x * HRY, ext = vis + 2 * RADIUS;
  double* plane = work + ((size_t)i * M + j) * vis * vis;
  for (int idx = threadIdx.x; idx < HRY * ext; idx += NT) {
    const int ry = idx / ext, cc = idx - ry * ext;
    buf[idx] = plane[(size_t)(y0 + ry) * vis + reflect_half(cc - RADIUS, vis)];
  }
  __syncthreads();
  double mn = INFINITY, mx = -INFINITY;
  for (int idx = threadIdx.x; idx < HRY * vis; idx += NT) {
    const int ry = idx / vis, x = idx - ry * vis;
    const double* c = buf + ry * ext + x + RADIUS;
    double acc = w[0] * c[0];
    for (int k = 1; k <= RADIUS; ++k) acc = fma(w[k], c[-k] + c[k], acc);
    plane[(size_t)(y0 + ry) * vis + x] = acc;
    mn = fmin(mn, acc);
    mx = fmax(mx, acc);
  }
  block_minmax(mn, mx);
  if (threadIdx.x == 0) {
    part[(((size_t)i * M + j) * K + blockIdx.x) * 2] = mn;
    part[(((size_t)i * M + j) * K + blockIdx.x) * 2 + 1] = mx;
  }
}

// per_map = 0: one (min, max) per image over its maps j <= n_i, from (1, 0) like the reference's minVglobal /
// maxVglobal; per_map = 1: one pair per map.  `src` holds K (min, max) partials per map.
__global__ void __launch_bounds__(NT) snap_minmax_kernel(const double* __restrict__ src, int K, int L,
                                                         const long long* __restrict__ lens, int per_map,
                                                         double* __restrict__ stats) {
  const int i = blockIdx.y, M = L + 1, n = map_count(lens, L, i);
  int j0 = 0, j1 = n;
  if (per_map) {
    j0 = j1 = blockIdx.x;
    if (j0 > n) return;
  }
  double mn = per_map ? INFINITY : 1.0, mx = per_map ? -INFINITY : 0.0;
  const int cnt = (j1 - j0 + 1) * K;
  for (int q = threadIdx.x; q < cnt; q += NT) {
    const double* p = src + (((size_t)i * M + j0) * K + q) * 2;
    mn = fmin(mn, p[0]);
    mx = fmax(mx, p[1]);
  }
  block_minmax(mn, mx);
  if (threadIdx.x == 0) {
    double* o = stats + (per_map ? ((size_t)i * M + j0) * 2 : (size_t)i * 2);
    o[0] = mn;
    o[1] = mx;
  }
}

// np.uint8 of a value: truncation toward zero; NaN (0 / 0 of a constant image) gives 0
__device__ __forceinline__ unsigned char to_u8(double v) {
  if (!(v == v)) return 0;
  return (unsigned char)__double2uint_rz(fmin(fmax(v, 0.0), 255.0));
}

// nn.Upsample(size=vis, mode='bilinear', align_corners=False) of image i at (y, x), channel c, then
// (x + 1) / 2 * 255 in float32 and the truncation of np.uint8
__device__ __forceinline__ unsigned char image_u8(const float* __restrict__ im, int s, int vis, int i, int c, int y,
                                                  int x) {
  const float* p = im + ((size_t)i * 3 + c) * s * s;
  float v;
  if (s == vis) {
    v = p[y * s + x];
  } else {
    const float scale = __fdiv_rn((float)s, (float)vis);
    float ry = fmaxf(__fsub_rn(__fmul_rn(scale, __fadd_rn((float)y, 0.5f)), 0.5f), 0.f);
    float rx = fmaxf(__fsub_rn(__fmul_rn(scale, __fadd_rn((float)x, 0.5f)), 0.5f), 0.f);
    const int y0 = min((int)floorf(ry), s - 1), x0 = min((int)floorf(rx), s - 1);
    const float ly = fminf(fmaxf(__fsub_rn(ry, (float)y0), 0.f), 1.f), lx = fminf(fmaxf(__fsub_rn(rx, (float)x0), 0.f), 1.f);
    const int y1 = y0 + (y0 < s - 1 ? 1 : 0), x1 = x0 + (x0 < s - 1 ? 1 : 0);
    const float wy0 = __fsub_rn(1.f, ly), wx0 = __fsub_rn(1.f, lx);
    const float t0 = __fadd_rn(__fmul_rn(p[y0 * s + x0], wx0), __fmul_rn(p[y0 * s + x1], lx));
    const float t1 = __fadd_rn(__fmul_rn(p[y1 * s + x0], wx0), __fmul_rn(p[y1 * s + x1], lx));
    v = __fadd_rn(__fmul_rn(t0, wy0), __fmul_rn(t1, ly));
  }
  v = __fmul_rn(__fmul_rn(__fadd_rn(v, 1.f), 0.5f), 255.f);
  if (!(v == v)) return 0;
  return (unsigned char)__float2uint_rz(fminf(fmaxf(v, 0.f), 255.f));
}

struct ComposeArgs {
  const float *img, *lr, *maps, *maxmap;
  const long long* lens;
  const double *work, *stats;
  unsigned char* out;
  int img_side, lr_side, L, att, vis, words, strip, per_map, expand, width;
};

__device__ __forceinline__ unsigned char map_u8(const ComposeArgs& a, int i, int j, int y, int x) {
  const int M = a.L + 1;
  const double* st = a.stats + (a.per_map ? ((size_t)i * M + j) * 2 : (size_t)i * 2);
  if (a.expand) {
    const double v = a.work[(((size_t)i * M + j) * a.vis + y) * a.vis + x], mn = st[0], mx = st[1];
    double q = v;
    if (!a.per_map || mx != mn) q = __ddiv_rn(__dsub_rn(v, mn), __dsub_rn(mx, mn));
    return to_u8(__dmul_rn(q, 255.0));
  }
  const float v = map_src(a.maps, a.maxmap, a.L, a.att * a.att, i, j)[y * a.att + x];
  const float mn = (float)st[0], mx = (float)st[1];
  float q = v;
  if (!a.per_map || mx != mn) q = __fdiv_rn(__fsub_rn(v, mn), __fsub_rn(mx, mn));
  q = __fmul_rn(q, 255.f);
  if (!(q == q)) return 0;
  return (unsigned char)__float2uint_rz(fminf(fmaxf(q, 0.f), 255.f));
}

__global__ void __launch_bounds__(NT) snap_compose_kernel(const ComposeArgs a) {
  const int X = blockIdx.x * NT + threadIdx.x, Y = blockIdx.y;
  if (X >= a.width) return;
  const int per = a.strip + 2 * a.vis, i = Y / per, r = Y - i * per, tw = a.vis + 2;
  const int t = X / tw, xx = X - t * tw;
  unsigned char o[3] = {0, 0, 0};
  if (r < a.strip) {
    for (int c = 0; c < 3; ++c) o[c] = t >= 2 ? kColor[t - 2][c] : 1;
  } else if (xx < a.vis) {
    const bool top = r < a.strip + a.vis;
    const int y = top ? r - a.strip : r - a.strip - a.vis;
    if (t == 0) {
      const float* im = top ? a.lr : a.img;
      const int s = top ? a.lr_side : a.img_side;
      for (int c = 0; c < 3; ++c) o[c] = image_u8(im, s, a.vis, i, c, y, xx);
    } else if (t - 1 <= map_count(a.lens, a.L, i)) {
      const unsigned m = map_u8(a, i, t - 1, y, xx);
      for (int c = 0; c < 3; ++c) {
        if (top) {
          o[c] = (unsigned char)m;
        } else {
          // PIL paste(att, mask=L 210) over the image: DIV255(img * 45 + att * 210), DIV255(v) = ((v+128)>>8 + v+128)>>8
          const unsigned v = image_u8(a.img, a.img_side, a.vis, i, c, y, xx) * 45u + m * 210u + 128u;
          o[c] = (unsigned char)(((v >> 8) + v) >> 8);
        }
      }
    }
  }
  unsigned char* p = a.out + ((size_t)Y * a.width + X) * 3;
  p[0] = o[0];
  p[1] = o[1];
  p[2] = o[2];
}

}  // namespace

OG_API int og_snapshot_canvas(const float* img, int img_side, const float* lr, int lr_side, const float* maps, int L,
                              int att, const long long* lens, int nvis, int vis, int words, int strip, int per_map,
                              float* maxmap, double* mm0, double* work, double* part, double* stats,
                              unsigned char* out, cudaStream_t stream) {
  if (nvis <= 0) return 0;
  if (L < 1 || att < 1 || vis % att != 0 || words < 0 || words > 20 || strip < 0) return (int)cudaErrorInvalidValue;
  const int M = L + 1, up = vis / att, expand = up > 1;
  if (expand && (vis % HRY != 0 || vis <= RADIUS || !work || !part)) return (int)cudaErrorInvalidValue;
  snap_prep_kernel<<<dim3(M, nvis), NT, 0, stream>>>(maps, L, att * att, lens, maxmap, mm0);
  int K = 1;
  if (expand) {
    const int ext = vis + 2 * RADIUS;
    const size_t vsm = (size_t)(RADIUS + 1 + ext * VTX) * sizeof(double);
    const size_t hsm = (size_t)(RADIUS + 1 + ext * HRY) * sizeof(double);
    snap_vblur_kernel<<<dim3(og_cdiv(vis, VTX), M, nvis), NT, vsm, stream>>>(maps, maxmap, L, att, lens, vis, mm0,
                                                                              work);
    K = vis / HRY;
    snap_hblur_kernel<<<dim3(K, M, nvis), NT, hsm, stream>>>(L, lens, vis, work, part);
  }
  snap_minmax_kernel<<<dim3(per_map ? M : 1, nvis), NT, 0, stream>>>(expand ? part : mm0, K, L, lens, per_map, stats);
  ComposeArgs a{img, lr ? lr : img, maps, maxmap, lens, work, stats, out, img_side, lr ? lr_side : img_side, L, att,
                vis, words, strip, per_map, expand, (words + 2) * (vis + 2)};
  snap_compose_kernel<<<dim3(og_cdiv(a.width, NT), nvis * (strip + 2 * vis)), NT, 0, stream>>>(a);
  OG_RETURN_LAST_ERROR();
}
