// preprocess.cu — batched input preparation on the GPU: the test-time silhouette crop (util_img.get_bbox + util_img.crop,
// called by every model's preprocess_wrapper) and MarrnetBaseModel.preprocess (models/marrnetbase.py:71-126): the bicubic
// resize to im_size, clamping, binarisation and scaling of the 2.5D maps, and the colour jitter, lighting noise and
// normalisation of rgb.  The reference runs these per sample in float64 numpy and cv2 on the host.
//
// Contract (include/genre_b200.h states it too; tests/preprocess_ref.py restates it in numpy, bit for bit).  All arithmetic
// is fp64 with one rounding per operation and no FMA, except where fp32 is stated; outputs are rounded once to fp32 at the
// end, as the reference's convert_to_float32 does.
//   sources   packed: one byte buffer and desc [B, 4] int64 on the device, (byte offset, H, W, C) per sample, element type
//             uint8 or uint16, the value x / 255.0 or x / 65535.0 in fp64 (np.iinfo(dtype).max);
//             dense: [B, H, W, C] float32 or float64, the value widened to fp64.
//             C in {1, 3, 4}; single-channel keys (mask, depth, silhou) read channel 0, rgb and normal channels 0..2.
//   bbox      get_bbox: the smallest and largest row and column with mask > th (fp64 compare), by integer atomics.  No such
//             pixel: valid = 0 and the sample's crops are NaN (preprocess then gives NaN rgb and, by the binarisation's
//             NaN -> 0, a zero silhou: valid is the mark to rely on).
//   window    crop, with y1, x1, y2, x2 = (min col, min row, max col, max row), so x indexes rows:
//               x_mid = (x1 + x2) / 2, y_mid = (y1 + y2) / 2, l = max(x2 - x1, y2 - y1) * out / (out - 2 * pad),
//               x1' = rint(x_mid - l / 2), x2' = rint(x_mid + l / 2), likewise y (rint: half to even, as np.round).
//             Window row j reads image row clamp(x1' + j, 0, H - 1), likewise columns: the reference's edge padding.
//   linear    cv2 INTER_LINEAR of the window (n_r = x2' - x1' + 1 rows, n_c = y2' - y1' + 1 columns) to out x out:
//               s = (d + 0.5) * (n / out) - 0.5, i = floor(s), f = s - i, taps clamp(i) and clamp(i + 1) into [0, n),
//               h = (1 - f_x) * v0 + f_x * v1 per tap row, then out = (1 - f_y) * h0 + f_y * h1.
//   cubic     cv2 INTER_CUBIC to im_size x im_size (util_img.resize(im, S, 'horizontal'); square sources only), n -> S:
//               fx = (float)((d + 0.5) * (1 / (S / n)) - 0.5), i = floor(fx), fx -= i (fp32);
//               coefficients in fp32 with A = -0.75: c0 = ((A(x+1) - 5A)(x+1) + 8A)(x+1) - 4A,
//               c1 = ((A+2)x - (A+3))x x + 1, c2 = ((A+2)(1-x) - (A+3))(1-x)(1-x) + 1, c3 = 1 - c0 - c1 - c2;
//               taps clamp(i - 1 .. i + 2); h = ((c0 v0 + c1 v1) + c2 v2) + c3 v3 per tap row, then the same over h.
//   depth, normal  clamp to the source's own min and max (normal: over its three channels; no clamp when the source holds a
//             NaN, as numpy's min is then NaN), then * scale_25d.
//   silhou    clamp, then 1 if > 0.999 else 0 (NaN -> 0), then * scale_25d.
//   rgb       test: (x - mean_c) / std_c.  train: the three jitter steps in the drawn order (brightness 0, contrast 1,
//             saturation 2, alpha in the order of the steps), then x_c += noise_c, then normalise, where
//               gray = (0.299 r + 0.587 g) + 0.114 b;  brightness x = a x + (1 - a) * 0;  contrast x = a x + (1 - a) m;
//               saturation x = a x + (1 - a) gray(x);
//             m, the mean of gray at the contrast step, is the one non-local value: p[g][c] = the sum over the rows of
//             group g (PP_GROUP_ROWS rows) of column c, in row order; col[c] = the sum of p[g][c] in group order;
//             m = (the sum of col[c] in column order) / S^2.  Every sum starts from its first term.
// Results depend only on the sample's own inputs (deterministic, batch-equivariant).  Descriptors and jitter orders live on
// the device and are trusted: the Python layer builds and checks them.
//
// Kernels: pp_bbox_kernel and pp_minmax_kernel (per-sample integer atomics), pp_crop_kernel (thread per output pixel:
// window, linear taps of the photo and the mask), pp_cubic_kernel (thread per output pixel: cubic taps and the per-pixel
// finish of every key except train-mode rgb), pp_gray_kernel / pp_mean_kernel / pp_jitter_kernel (train-mode rgb).
#include "common.cuh"

namespace gb {

constexpr int PP_THREADS = 256;
constexpr int PP_STAT_BLOCKS = 64;    // CTAs per sample of the atomic reductions (grid-stride over the sample)
constexpr int PP_GROUP_ROWS = 16;     // rows per partial sum of the contrast mean
constexpr int PP_MAX_OUT = 4096;

enum { PP_U8 = 0, PP_U16 = 1, PP_F32 = 2, PP_F64 = 3 };
enum { PP_RGB = 0, PP_DEPTH = 1, PP_SILHOU = 2, PP_NORMAL = 3 };

struct PpSrc {
  const char *data;
  const long long *desc;   // packed: [B, 4] (byte offset, H, W, C); NULL: dense
  int dtype;
  long long H, W, C;       // dense only
};

struct PpImg {
  const char *p;
  long long H, W, C;
  int dtype;
};

__device__ __forceinline__ PpImg pp_image(const PpSrc &s, int b) {
  PpImg im;
  im.dtype = s.dtype;
  if (s.desc) {
    const long long *d = s.desc + 4 * b;
    im.p = s.data + __ldg(d);
    im.H = __ldg(d + 1);
    im.W = __ldg(d + 2);
    im.C = __ldg(d + 3);
  } else {
    im.H = s.H;
    im.W = s.W;
    im.C = s.C;
    const long long es = s.dtype == PP_U8 ? 1 : s.dtype == PP_U16 ? 2 : s.dtype == PP_F32 ? 4 : 8;
    im.p = s.data + (size_t)b * (size_t)(s.H * s.W * s.C) * (size_t)es;
  }
  return im;
}

// element i (C order) as fp64
__device__ __forceinline__ double pp_load(const PpImg &im, long long i) {
  switch (im.dtype) {
    case PP_U8: return __ddiv_rn((double)__ldg((const unsigned char *)im.p + i), 255.0);
    case PP_U16: return __ddiv_rn((double)__ldg((const unsigned short *)im.p + i), 65535.0);
    case PP_F32: return (double)__ldg((const float *)im.p + i);
    default: return __ldg((const double *)im.p + i);
  }
}

// element i as fp64 for a dtype known at compile time: pp_cubic_kernel is templated on it, which keeps the dtype switch out
// of its 16 taps per channel (228 -> at most 110 registers, two CTAs per SM)
template <int DT>
__device__ __forceinline__ double pp_load_t(const char *p, long long i) {
  if (DT == PP_U8) return __ddiv_rn((double)__ldg((const unsigned char *)p + i), 255.0);
  if (DT == PP_U16) return __ddiv_rn((double)__ldg((const unsigned short *)p + i), 65535.0);
  if (DT == PP_F32) return (double)__ldg((const float *)p + i);
  return __ldg((const double *)p + i);
}

__device__ __forceinline__ double pp_at(const PpImg &im, long long r, long long c, int ch) {
  return pp_load(im, (r * im.W + c) * im.C + ch);
}

__device__ __forceinline__ long long pp_clamp(long long v, long long lo, long long hi) { return v < lo ? lo : v > hi ? hi : v; }

// ---- bbox of mask > th: keys (H - r_min, r_max + 1, W - c_min, c_max + 1), all 0 when empty -------------------------------
__global__ void __launch_bounds__(PP_THREADS)
pp_bbox_kernel(PpSrc mask, double th, int *__restrict__ keys) {
  const int b = blockIdx.y;
  const PpImg im = pp_image(mask, b);
  const long long n = im.H * im.W;
  unsigned k[4] = {0u, 0u, 0u, 0u};
  for (long long i = (long long)blockIdx.x * PP_THREADS + threadIdx.x; i < n; i += (long long)gridDim.x * PP_THREADS) {
    if (pp_load(im, i * im.C) > th) {
      const long long r = i / im.W, c = i - r * im.W;
      k[0] = max(k[0], (unsigned)(im.H - r));
      k[1] = max(k[1], (unsigned)(r + 1));
      k[2] = max(k[2], (unsigned)(im.W - c));
      k[3] = max(k[3], (unsigned)(c + 1));
    }
  }
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const unsigned v = __reduce_max_sync(0xffffffffu, k[j]);
    if ((threadIdx.x & 31) == 0 && v) atomicMax(keys + 4 * b + j, (int)v);
  }
}

// ---- min / max of a source: ordered fp64 keys (min stored complemented), NaN flag --------------------------------------
__device__ __forceinline__ unsigned long long pp_key(double v) {
  const unsigned long long u = (unsigned long long)__double_as_longlong(v);
  return (u >> 63) ? ~u : (u | 0x8000000000000000ull);
}
__device__ __forceinline__ double pp_unkey(unsigned long long k) {
  return __longlong_as_double((long long)((k >> 63) ? (k & 0x7fffffffffffffffull) : ~k));
}

__device__ __forceinline__ unsigned long long pp_warp_max(unsigned long long v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const unsigned long long y = __shfl_xor_sync(0xffffffffu, v, o);
    v = y > v ? y : v;
  }
  return v;
}

// stats[b] = (~min key, max key, NaN seen), zero-initialised; channels 0 .. nch-1 of each pixel
__global__ void __launch_bounds__(PP_THREADS)
pp_minmax_kernel(PpSrc src, int nch, unsigned long long *__restrict__ stats) {
  const int b = blockIdx.y;
  const PpImg im = pp_image(src, b);
  const long long n = im.H * im.W;
  unsigned long long kmin = 0ull, kmax = 0ull, nan = 0ull;   // kmin holds ~key, so larger is smaller
  for (long long i = (long long)blockIdx.x * PP_THREADS + threadIdx.x; i < n; i += (long long)gridDim.x * PP_THREADS) {
    for (int ch = 0; ch < nch; ++ch) {
      const double v = pp_load(im, i * im.C + ch);
      if (v != v) {
        nan = 1ull;
        continue;
      }
      const unsigned long long k = pp_key(v);
      kmin = ~k > kmin ? ~k : kmin;
      kmax = k > kmax ? k : kmax;
    }
  }
  kmin = pp_warp_max(kmin);
  kmax = pp_warp_max(kmax);
  nan = pp_warp_max(nan);
  if ((threadIdx.x & 31) == 0) {
    if (kmin) atomicMax(stats + 3 * b, kmin);
    if (kmax) atomicMax(stats + 3 * b + 1, kmax);
    if (nan) atomicMax(stats + 3 * b + 2, nan);
  }
}

// ---- crop: window of the bbox, linear resize of the photo (3 channels) and the mask (channel 0) -----------------------
struct PpTaps {
  long long i0, i1;   // source indices (image, after the window's edge clamp)
  double w0, w1;
};

__device__ __forceinline__ PpTaps pp_linear_taps(int d, int out, long long lo, long long n, long long size) {
  const double s = __dsub_rn(__dmul_rn(__dadd_rn((double)d, 0.5), __ddiv_rn((double)n, (double)out)), 0.5);
  const double fl = floor(s);
  const long long i = (long long)fl;
  PpTaps t;
  t.w1 = __dsub_rn(s, fl);
  t.w0 = __dsub_rn(1.0, t.w1);
  t.i0 = pp_clamp(lo + pp_clamp(i, 0, n - 1), 0, size - 1);
  t.i1 = pp_clamp(lo + pp_clamp(i + 1, 0, n - 1), 0, size - 1);
  return t;
}

__device__ __forceinline__ double pp_bilinear(const PpImg &im, const PpTaps &ty, const PpTaps &tx, int ch) {
  const double h0 = __dadd_rn(__dmul_rn(tx.w0, pp_at(im, ty.i0, tx.i0, ch)), __dmul_rn(tx.w1, pp_at(im, ty.i0, tx.i1, ch)));
  const double h1 = __dadd_rn(__dmul_rn(tx.w0, pp_at(im, ty.i1, tx.i0, ch)), __dmul_rn(tx.w1, pp_at(im, ty.i1, tx.i1, ch)));
  return __dadd_rn(__dmul_rn(ty.w0, h0), __dmul_rn(ty.w1, h1));
}

// the window bound nearer to or farther from the start: rint(mid -+ l / 2)
__device__ __forceinline__ long long pp_bound(double mid, double half, bool upper) {
  return (long long)rint(upper ? __dadd_rn(mid, half) : __dsub_rn(mid, half));
}

// grid (pixel blocks, B): thread per output pixel of rgb [B, out, out, 3] and silhou [B, out, out] (fp64)
__global__ void __launch_bounds__(PP_THREADS)
pp_crop_kernel(PpSrc img, PpSrc mask, const int *__restrict__ keys, int out, double pad, double *__restrict__ rgb,
               double *__restrict__ silhou, unsigned char *__restrict__ valid) {
  const int b = blockIdx.y;
  const long long p = (long long)blockIdx.x * PP_THREADS + threadIdx.x;
  if (p >= (long long)out * out) return;
  const PpImg im = pp_image(img, b), mk = pp_image(mask, b);
  const int *k = keys + 4 * b;
  const bool ok = k[1] > 0;
  if (p == 0) valid[b] = ok ? 1 : 0;
  const size_t o = (size_t)b * out * out + p;
  if (!ok) {
    const double nan = __longlong_as_double(0x7ff8000000000000ll);
    rgb[3 * o] = rgb[3 * o + 1] = rgb[3 * o + 2] = nan;
    if (silhou) silhou[o] = nan;
    return;
  }
  const long long x1 = mk.H - k[0], x2 = k[1] - 1, y1 = mk.W - k[2], y2 = k[3] - 1;   // x: rows, y: columns
  const double xm = __ddiv_rn((double)(x1 + x2), 2.0), ym = __ddiv_rn((double)(y1 + y2), 2.0);
  const long long ext = max(x2 - x1, y2 - y1);
  const double l = __ddiv_rn((double)(ext * out), __dsub_rn((double)out, __dmul_rn(2.0, pad)));
  const double half = __ddiv_rn(l, 2.0);
  const long long wx1 = pp_bound(xm, half, false), wx2 = pp_bound(xm, half, true);
  const long long wy1 = pp_bound(ym, half, false), wy2 = pp_bound(ym, half, true);
  const int dr = (int)(p / out), dc = (int)(p - (long long)dr * out);
  const PpTaps ty = pp_linear_taps(dr, out, wx1, wx2 - wx1 + 1, im.H);
  const PpTaps tx = pp_linear_taps(dc, out, wy1, wy2 - wy1 + 1, im.W);
#pragma unroll
  for (int ch = 0; ch < 3; ++ch) rgb[3 * o + ch] = pp_bilinear(im, ty, tx, ch);
  if (silhou) silhou[o] = pp_bilinear(mk, ty, tx, 0);
}

// ---- cubic resize and the per-pixel finish ----------------------------------------------------------------------------
struct PpCubic {
  long long i[4];
  double c[4];
};

__device__ __forceinline__ PpCubic pp_cubic_taps(int d, int S, long long n) {
  const double sc = __ddiv_rn(1.0, __ddiv_rn((double)S, (double)n));
  float fx = __double2float_rn(__dsub_rn(__dmul_rn(__dadd_rn((double)d, 0.5), sc), 0.5));
  const float fl = floorf(fx);
  const long long sx = (long long)fl;
  fx = __fsub_rn(fx, fl);
  const float A = -0.75f;
  const float x1 = __fadd_rn(fx, 1.0f), y = __fsub_rn(1.0f, fx);
  const float c0 = __fsub_rn(__fmul_rn(__fadd_rn(__fmul_rn(__fsub_rn(__fmul_rn(A, x1), 5.0f * A), x1), 8.0f * A), x1), 4.0f * A);
  const float c1 = __fadd_rn(__fmul_rn(__fmul_rn(__fsub_rn(__fmul_rn(A + 2.0f, fx), A + 3.0f), fx), fx), 1.0f);
  const float c2 = __fadd_rn(__fmul_rn(__fmul_rn(__fsub_rn(__fmul_rn(A + 2.0f, y), A + 3.0f), y), y), 1.0f);
  const float c3 = __fsub_rn(__fsub_rn(__fsub_rn(1.0f, c0), c1), c2);
  PpCubic t;
  t.c[0] = c0;
  t.c[1] = c1;
  t.c[2] = c2;
  t.c[3] = c3;
#pragma unroll
  for (int j = 0; j < 4; ++j) t.i[j] = pp_clamp(sx - 1 + j, 0, n - 1);
  return t;
}

__device__ __forceinline__ double pp_dot4(const double *c, const double *v) {
  return __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(c[0], v[0]), __dmul_rn(c[1], v[1])), __dmul_rn(c[2], v[2])),
                   __dmul_rn(c[3], v[3]));
}

template <int DT>
__device__ __forceinline__ double pp_bicubic(const PpImg &im, const PpCubic &ty, const PpCubic &tx, int ch) {
  double h[4];
#pragma unroll
  for (int a = 0; a < 4; ++a) {
    const char *row = im.p;
    const long long base = ty.i[a] * im.W;
    double v[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) v[j] = pp_load_t<DT>(row, (base + tx.i[j]) * im.C + ch);
    h[a] = pp_dot4(tx.c, v);
  }
  return pp_dot4(ty.c, h);
}

__constant__ double PP_MEAN[3] = {0.485, 0.456, 0.406};
__constant__ double PP_STD[3] = {0.229, 0.224, 0.225};

// grid (pixel blocks, B): out [B, nch, S, S] fp32 (or fp64 tmp for train-mode rgb); DT = the source's element type
template <int DT>
__global__ void __launch_bounds__(PP_THREADS)
pp_cubic_kernel(PpSrc src, int kind, int S, double scale, const unsigned long long *__restrict__ stats, float *__restrict__ out,
                double *__restrict__ tmp) {
  const int b = blockIdx.y;
  const long long p = (long long)blockIdx.x * PP_THREADS + threadIdx.x;
  const long long plane = (long long)S * S;
  if (p >= plane) return;
  const PpImg im = pp_image(src, b);
  const int dr = (int)(p / S), dc = (int)(p - (long long)dr * S);
  const PpCubic ty = pp_cubic_taps(dr, S, im.H), tx = pp_cubic_taps(dc, S, im.W);
  const int nch = (kind == PP_RGB || kind == PP_NORMAL) ? 3 : 1;
  bool clamp = false;
  double lo = 0.0, hi = 0.0;
  if (kind != PP_RGB) {
    const unsigned long long *st = stats + 3 * b;
    clamp = st[2] == 0ull;
    lo = pp_unkey(~st[0]);
    hi = pp_unkey(st[1]);
  }
  for (int ch = 0; ch < nch; ++ch) {
    double v = pp_bicubic<DT>(im, ty, tx, ch);
    const size_t o = ((size_t)b * nch + ch) * plane + p;
    if (tmp) {
      tmp[o] = v;
      continue;
    }
    if (kind == PP_RGB) {
      v = __ddiv_rn(__dsub_rn(v, PP_MEAN[ch]), PP_STD[ch]);
    } else {
      if (clamp) {
        if (v < lo) v = lo;
        if (v > hi) v = hi;
      }
      if (kind == PP_SILHOU) v = v > 0.999 ? 1.0 : 0.0;
      v = __dmul_rn(v, scale);
    }
    out[o] = __double2float_rn(v);
  }
}

// ---- train-mode rgb: jitter chain, contrast mean, lighting noise --------------------------------------------------------
__device__ __forceinline__ double pp_gray(const double *x) {
  return __dadd_rn(__dadd_rn(__dmul_rn(0.299, x[0]), __dmul_rn(0.587, x[1])), __dmul_rn(0.114, x[2]));
}

// the jitter steps k0 .. k1-1 of sample b's order; m is used by a contrast step only
__device__ __forceinline__ void pp_jitter(double *x, const int *order, const double *alpha, int k0, int k1, double m) {
  for (int k = k0; k < k1; ++k) {
    const double a = alpha[k], a1 = __dsub_rn(1.0, a);
    const int step = order[k];
    if (step == 0) {
      const double z = __dmul_rn(a1, 0.0);
#pragma unroll
      for (int c = 0; c < 3; ++c) x[c] = __dadd_rn(__dmul_rn(a, x[c]), z);
    } else if (step == 1) {
      const double z = __dmul_rn(a1, m);
#pragma unroll
      for (int c = 0; c < 3; ++c) x[c] = __dadd_rn(__dmul_rn(a, x[c]), z);
    } else if (step == 2) {
      const double z = __dmul_rn(a1, pp_gray(x));
#pragma unroll
      for (int c = 0; c < 3; ++c) x[c] = __dadd_rn(__dmul_rn(a, x[c]), z);
    }
  }
}

__device__ __forceinline__ int pp_contrast_step(const int *order) {
  return order[0] == 1 ? 0 : order[1] == 1 ? 1 : 2;
}

// grid (column blocks, row groups, B): part[b][g][c] = sum over the group's rows of gray at the contrast step
__global__ void __launch_bounds__(PP_THREADS)
pp_gray_kernel(const double *__restrict__ tmp, int S, const int *__restrict__ order, const double *__restrict__ alpha,
               double *__restrict__ part) {
  const int b = blockIdx.z, g = blockIdx.y;
  const int c = blockIdx.x * PP_THREADS + threadIdx.x;
  if (c >= S) return;
  int o[3];
  double a[3];
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    o[k] = __ldg(order + 3 * b + k);
    a[k] = __ldg(alpha + 3 * b + k);
  }
  const int kc = pp_contrast_step(o);
  const size_t plane = (size_t)S * S;
  const double *t = tmp + (size_t)b * 3 * plane;
  const int r0 = g * PP_GROUP_ROWS, r1 = min(r0 + PP_GROUP_ROWS, S);
  double acc = 0.0;
  for (int r = r0; r < r1; ++r) {
    const size_t q = (size_t)r * S + c;
    double x[3] = {__ldg(t + q), __ldg(t + plane + q), __ldg(t + 2 * plane + q)};
    pp_jitter(x, o, a, 0, kc, 0.0);
    const double gv = pp_gray(x);
    acc = r == r0 ? gv : __dadd_rn(acc, gv);
  }
  part[((size_t)b * gridDim.y + g) * S + c] = acc;
}

// one CTA per sample: m[b] = (sum over c of (sum over g of part[b][g][c])) / S^2, every sum in index order
__global__ void __launch_bounds__(PP_THREADS)
pp_mean_kernel(const double *__restrict__ part, int S, int G, double *__restrict__ mean) {
  extern __shared__ double s_col[];
  const int b = blockIdx.x;
  const double *pb = part + (size_t)b * G * S;
  for (int c = threadIdx.x; c < S; c += PP_THREADS) {
    double acc = pb[c];
    for (int g = 1; g < G; ++g) acc = __dadd_rn(acc, pb[(size_t)g * S + c]);
    s_col[c] = acc;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    double acc = s_col[0];
    for (int c = 1; c < S; ++c) acc = __dadd_rn(acc, s_col[c]);
    mean[b] = __ddiv_rn(acc, (double)S * (double)S);
  }
}

// grid (pixel blocks, B): the whole chain, lighting noise, normalisation, fp32 NCHW
__global__ void __launch_bounds__(PP_THREADS)
pp_jitter_kernel(const double *__restrict__ tmp, int S, const int *__restrict__ order, const double *__restrict__ alpha,
                 const double *__restrict__ noise, const double *__restrict__ mean, float *__restrict__ out) {
  const int b = blockIdx.y;
  const long long p = (long long)blockIdx.x * PP_THREADS + threadIdx.x;
  const size_t plane = (size_t)S * S;
  if (p >= (long long)plane) return;
  int o[3];
  double a[3];
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    o[k] = __ldg(order + 3 * b + k);
    a[k] = __ldg(alpha + 3 * b + k);
  }
  const size_t base = (size_t)b * 3 * plane + p;
  double x[3] = {__ldg(tmp + base), __ldg(tmp + base + plane), __ldg(tmp + base + 2 * plane)};
  pp_jitter(x, o, a, 0, 3, __ldg(mean + b));
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const double v = __dadd_rn(x[c], __ldg(noise + 3 * b + c));
    out[base + c * plane] = __double2float_rn(__ddiv_rn(__dsub_rn(v, PP_MEAN[c]), PP_STD[c]));
  }
}

// ---- host side --------------------------------------------------------------------------------------------------------
static size_t pp_align(size_t x) { return (x + 255) & ~(size_t)255; }
static unsigned pp_blocks(long long n) { return (unsigned)((n + PP_THREADS - 1) / PP_THREADS); }
static int pp_groups(int S) { return (S + PP_GROUP_ROWS - 1) / PP_GROUP_ROWS; }

struct PpLayout {
  size_t stats, tmp, part, mean, total;
};

static bool pp_layout(int kind, int train, int64_t B, int S, PpLayout *L) {
  if (B < 1 || B > 65535 || S < 1 || S > PP_MAX_OUT || kind < PP_RGB || kind > PP_NORMAL) return false;
  const bool chain = kind == PP_RGB && train;
  L->stats = 0;
  L->tmp = pp_align((size_t)B * 3 * sizeof(unsigned long long));
  const size_t plane = (size_t)S * S;
  L->part = L->tmp + (chain ? pp_align((size_t)B * 3 * plane * sizeof(double)) : 0);
  L->mean = L->part + (chain ? pp_align((size_t)B * pp_groups(S) * S * sizeof(double)) : 0);
  L->total = L->mean + pp_align((size_t)B * sizeof(double));
  return true;
}

static bool pp_dtype_ok(int dtype, bool packed) {
  return packed ? (dtype == PP_U8 || dtype == PP_U16) : (dtype == PP_F32 || dtype == PP_F64);
}

static int pp_check_src(const char *what, const void *data, const int64_t *desc, int dtype, int64_t H, int64_t W, int64_t C) {
  GB_REQUIRE(data, GENRE_B200_EINVAL, "%s: null pointer", what);
  GB_REQUIRE(pp_dtype_ok(dtype, desc != nullptr), GENRE_B200_EINVAL,
             "%s: dtype %d unsupported (packed: 0 uint8, 1 uint16; dense: 2 float32, 3 float64)", what, dtype);
  if (!desc) {
    GB_REQUIRE(H >= 1 && W >= 1 && H <= (1 << 16) && W <= (1 << 16) && (C == 1 || C == 3 || C == 4), GENRE_B200_EINVAL,
               "%s: dense H=%lld W=%lld C=%lld out of range (1..65536, C in {1, 3, 4})", what, (long long)H, (long long)W,
               (long long)C);
  }
  return 0;
}

}  // namespace gb

using namespace gb;

extern "C" size_t genre_b200_crop_to_render_workspace_bytes(int64_t B) {
  return (B >= 1 && B <= 65535) ? pp_align((size_t)B * 4 * sizeof(int)) : 0;
}

extern "C" int genre_b200_crop_to_render(const void *img, const int64_t *img_desc, int img_dtype, const void *mask,
                                         const int64_t *mask_desc, int mask_dtype, int64_t B, int out_size, double pad,
                                         double th, double *rgb, double *silhou, uint8_t *valid, void *workspace,
                                         size_t workspace_bytes, void *stream) {
  GB_REQUIRE(img && img_desc && mask && mask_desc && rgb && valid && workspace, GENRE_B200_EINVAL,
             "crop_to_render: null pointer");
  GB_REQUIRE(B >= 1 && B <= 65535, GENRE_B200_EINVAL, "crop_to_render: B=%lld out of range [1, 65535]", (long long)B);
  GB_REQUIRE(pp_dtype_ok(img_dtype, true) && pp_dtype_ok(mask_dtype, true), GENRE_B200_EINVAL,
             "crop_to_render: dtype %d / %d unsupported (packed images: 0 uint8, 1 uint16)", img_dtype, mask_dtype);
  GB_REQUIRE(out_size >= 1 && out_size <= PP_MAX_OUT, GENRE_B200_EINVAL, "crop_to_render: out_size=%d out of range [1, %d]",
             out_size, PP_MAX_OUT);
  GB_REQUIRE(pad >= 0.0 && 2.0 * pad < (double)out_size, GENRE_B200_EINVAL,
             "crop_to_render: pad=%g must satisfy 0 <= 2 * pad < out_size", pad);
  GB_REQUIRE(th == th, GENRE_B200_EINVAL, "crop_to_render: threshold is NaN");
  const size_t need = genre_b200_crop_to_render_workspace_bytes(B);
  GB_REQUIRE(workspace_bytes >= need && aligned16(workspace), GENRE_B200_EWORKSPACE,
             "crop_to_render: workspace too small or misaligned (%zu bytes needed, 16-byte aligned)", need);
  cudaStream_t st = as_stream(stream);
  int *keys = (int *)workspace;
  const cudaError_t e = cudaMemsetAsync(keys, 0, (size_t)B * 4 * sizeof(int), st);
  if (e != cudaSuccess) {
    set_error("crop_to_render: memset: %s", cudaGetErrorString(e));
    return (int)e;
  }
  const PpSrc si{(const char *)img, (const long long *)img_desc, img_dtype, 0, 0, 0};
  const PpSrc sm{(const char *)mask, (const long long *)mask_desc, mask_dtype, 0, 0, 0};
  pp_bbox_kernel<<<dim3(PP_STAT_BLOCKS, (unsigned)B), PP_THREADS, 0, st>>>(sm, th, keys);
  if (int rc = check_launch("crop_to_render bbox kernel")) return rc;
  pp_crop_kernel<<<dim3(pp_blocks((long long)out_size * out_size), (unsigned)B), PP_THREADS, 0, st>>>(
      si, sm, keys, out_size, pad, rgb, silhou, valid);
  return check_launch("crop_to_render crop kernel");
}

extern "C" size_t genre_b200_preprocess_workspace_bytes(int kind, int train, int64_t B, int im_size) {
  PpLayout L{};
  return pp_layout(kind, train, B, im_size, &L) ? L.total : 0;
}

extern "C" int genre_b200_preprocess(int kind, int train, const void *src, const int64_t *desc, int dtype, int64_t B,
                                     int64_t H, int64_t W, int64_t C, int im_size, double scale_25d, const int32_t *order,
                                     const double *alpha, const double *noise, float *out, void *workspace,
                                     size_t workspace_bytes, void *stream) {
  GB_REQUIRE(kind >= PP_RGB && kind <= PP_NORMAL, GENRE_B200_EINVAL,
             "preprocess: kind=%d unsupported (0 rgb, 1 depth, 2 silhou, 3 normal)", kind);
  GB_REQUIRE(out && workspace, GENRE_B200_EINVAL, "preprocess: null pointer");
  if (int rc = pp_check_src("preprocess", src, desc, dtype, H, W, C)) return rc;
  GB_REQUIRE(desc || H == W, GENRE_B200_EINVAL, "preprocess: dense source is %lldx%lld; only square images are resized",
             (long long)H, (long long)W);
  GB_REQUIRE(desc || kind == PP_DEPTH || kind == PP_SILHOU || C == 3, GENRE_B200_EINVAL,
             "preprocess: rgb and normal need C = 3 (got %lld)", (long long)C);
  GB_REQUIRE(B >= 1 && B <= 65535, GENRE_B200_EINVAL, "preprocess: B=%lld out of range [1, 65535]", (long long)B);
  GB_REQUIRE(im_size >= 1 && im_size <= PP_MAX_OUT, GENRE_B200_EINVAL, "preprocess: im_size=%d out of range [1, %d]",
             im_size, PP_MAX_OUT);
  const bool chain = kind == PP_RGB && train;
  GB_REQUIRE(!chain || (order && alpha && noise), GENRE_B200_EINVAL,
             "preprocess: train-mode rgb needs the jitter order, alpha and noise");
  PpLayout L{};
  pp_layout(kind, train, B, im_size, &L);
  GB_REQUIRE(workspace_bytes >= L.total && aligned16(workspace), GENRE_B200_EWORKSPACE,
             "preprocess: workspace too small or misaligned (%zu bytes needed, 16-byte aligned)", L.total);
  cudaStream_t st = as_stream(stream);
  char *ws = (char *)workspace;
  unsigned long long *stats = (unsigned long long *)(ws + L.stats);
  const PpSrc s{(const char *)src, (const long long *)desc, dtype, H, W, C};
  const dim3 grid(pp_blocks((long long)im_size * im_size), (unsigned)B);
  if (kind != PP_RGB) {
    const cudaError_t e = cudaMemsetAsync(stats, 0, (size_t)B * 3 * sizeof(unsigned long long), st);
    if (e != cudaSuccess) {
      set_error("preprocess: memset: %s", cudaGetErrorString(e));
      return (int)e;
    }
    pp_minmax_kernel<<<dim3(PP_STAT_BLOCKS, (unsigned)B), PP_THREADS, 0, st>>>(s, kind == PP_NORMAL ? 3 : 1, stats);
    if (int rc = check_launch("preprocess min/max kernel")) return rc;
  }
  double *tmp = chain ? (double *)(ws + L.tmp) : nullptr;
  switch (dtype) {
    case PP_U8: pp_cubic_kernel<PP_U8><<<grid, PP_THREADS, 0, st>>>(s, kind, im_size, scale_25d, stats, out, tmp); break;
    case PP_U16: pp_cubic_kernel<PP_U16><<<grid, PP_THREADS, 0, st>>>(s, kind, im_size, scale_25d, stats, out, tmp); break;
    case PP_F32: pp_cubic_kernel<PP_F32><<<grid, PP_THREADS, 0, st>>>(s, kind, im_size, scale_25d, stats, out, tmp); break;
    default: pp_cubic_kernel<PP_F64><<<grid, PP_THREADS, 0, st>>>(s, kind, im_size, scale_25d, stats, out, tmp); break;
  }
  if (int rc = check_launch("preprocess cubic kernel")) return rc;
  if (!chain) return 0;
  double *part = (double *)(ws + L.part), *mean = (double *)(ws + L.mean);
  const int G = pp_groups(im_size);
  pp_gray_kernel<<<dim3(pp_blocks(im_size), (unsigned)G, (unsigned)B), PP_THREADS, 0, st>>>(tmp, im_size, order, alpha, part);
  if (int rc = check_launch("preprocess gray kernel")) return rc;
  pp_mean_kernel<<<(unsigned)B, PP_THREADS, (size_t)im_size * sizeof(double), st>>>(part, im_size, G, mean);
  if (int rc = check_launch("preprocess mean kernel")) return rc;
  pp_jitter_kernel<<<grid, PP_THREADS, 0, st>>>(tmp, im_size, order, alpha, noise, mean, out);
  return check_launch("preprocess jitter kernel");
}
