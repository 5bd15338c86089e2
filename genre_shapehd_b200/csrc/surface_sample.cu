// surface_sample.cu — area-weighted uniform point sampling of batched triangle meshes on the GPU: the step between
// marching cubes and the Chamfer / F-score evaluation of predicted voxel grids (the reference's nndistance op is the metric;
// it had no device path from a mesh to points).  n points per sample, so every output is dense and no host synchronisation
// is needed.
//
// Contract (include/genre_b200.h states it too; tests/surface_sample_ref.py restates it in numpy, bit for bit):
//   meshes  the packed format of genre_b200_isosurface_*: verts [sum V, 3] fp32, faces [sum F, 3] int32 with indices local to
//           the sample, vert_off / face_off [N+1] int64 on the device.  Indices lie in [0, V_n).  F (the total) < 2^31.
//   weight  per face, in fp64 from the fp32 vertices a, b, c, one rounding per operation, no contraction:
//             e1 = b - a, e2 = c - a (per axis);
//             nx = e1y*e2z - e1z*e2y, ny = e1z*e2x - e1x*e2z, nz = e1x*e2y - e1y*e2x;
//             s = sqrt((nx*nx + ny*ny) + nz*nz);   a non-finite s (a non-finite vertex) counts as 0.
//           smax_b = the largest s of sample b (integer atomicMax on the fp64 bits: s >= 0, so the bits are monotone; exact and
//           deterministic).  w_f = floor(ldexp(s_f / smax_b, 32)) as uint64, and w_f = 0 for every face when smax_b = 0.
//   scan    P_f = the inclusive prefix sum of w within the sample, T_b = its last value (0 for a sample without faces).
//           w_f <= 2^32 and F < 2^31, so every sum is exact in uint64 and independent of the order of the additions.
//   point i of sample b (uint64 arithmetic wraps; GOLDEN = 0x9E3779B97F4A7C15):
//             r_j = splitmix64(seed_b + (3i + j + 1) * GOLDEN), j = 0, 1, 2, with splitmix64's output function
//             z ^= z >> 30; z *= 0xBF58476D1CE4E5B9; z ^= z >> 27; z *= 0x94D049BB133111EB; z ^= z >> 31;
//             face f = the smallest f with P_f > mulhi64(r_0, T_b) (the high 64 bits of the 128-bit product), so face f is
//             chosen with probability w_f / T_b up to 2^-64, and a face of weight 0 never;
//             U = r_1 >> 40, V = r_2 >> 40 (24-bit integers); if U + V > 2^24 then U = 2^24 - U, V = 2^24 - V;
//             u = U * 2^-24, v = V * 2^-24 (exact in fp32);
//             per axis p = fl(fl(a + fl(u * fl(b - a))) + fl(v * fl(c - a))), no FMA.
//   output  points [N, n, 3] fp32, face [N, n] int32 local to the sample.  A sample with T_b = 0 (no faces, or all of zero
//           area) gets NaN points and face -1.  A point depends only on (seed_b, i) and its own mesh: results are
//           deterministic and batch-equivariant.
//
// Kernels: ss_weight_kernel (thread per face: s, the per-sample maximum), ss_scan_kernel (one CTA per sample: quantise and
// scan in tiles of SS_SCAN_THREADS x SS_SCAN_ITEMS faces with a running carry), ss_sample_kernel (thread per point: three
// splitmix64 draws, a binary search in P, the barycentric point).
//
// Backward (genre_b200_surface_sample_backward): the gradient of the points with respect to the vertices, with the drawn faces
// and barycentric draws held fixed (the reparameterised sampling gradient; nothing flows through the area weights).  Point i
// of sample b redraws (u, v) from (seed_b, i) with the forward's helper and reads its face from the forward's face output;
// dp/da = 1 - u - v, dp/db = u, dp/dc = v, exact in fp32.  ss_sample_backward_kernel (thread per point) adds each
// fl32(w * g) to grad_verts by fp32 atomicAdd after a memset: the order of the additions is unspecified, so the result is
// not bitwise reproducible.  Points with face -1 contribute nothing.
#include "common.cuh"

namespace gb {

constexpr int SS_THREADS = 256;
constexpr int SS_SCAN_THREADS = 1024;
constexpr int SS_SCAN_ITEMS = 8;
constexpr unsigned long long SS_GOLDEN = 0x9E3779B97F4A7C15ull;
constexpr int64_t SS_MAX_FACES = (int64_t)1 << 31;   // exclusive
constexpr int64_t SS_MAX_POINTS = (int64_t)1 << 30;  // per sample, inclusive

__device__ __forceinline__ unsigned long long ss_splitmix64(unsigned long long z) {
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  return z ^ (z >> 31);
}

// the barycentric draw (u, v) of point i of a sample with seed `seed`: r_1, r_2 and the U + V > 2^24 fold
__device__ __forceinline__ void ss_barycentric(unsigned long long seed, long long i, float &u, float &v) {
  const unsigned long long k = 3ull * (unsigned long long)i;
  const unsigned long long r1 = ss_splitmix64(seed + (k + 2ull) * SS_GOLDEN);
  const unsigned long long r2 = ss_splitmix64(seed + (k + 3ull) * SS_GOLDEN);
  unsigned U = (unsigned)(r1 >> 40), V = (unsigned)(r2 >> 40);
  if (U + V > (1u << 24)) {
    U = (1u << 24) - U;
    V = (1u << 24) - V;
  }
  u = __fmul_rn((float)U, 0x1p-24f);
  v = __fmul_rn((float)V, 0x1p-24f);
}

// largest n with off[n] <= i (empty samples are skipped over)
__device__ __forceinline__ int ss_sample_of(const long long *__restrict__ off, int N, long long i) {
  int lo = 0, hi = N - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (__ldg(off + mid) <= i) lo = mid;
    else hi = mid - 1;
  }
  return lo;
}

__device__ __forceinline__ double ss_face_weight(const float *__restrict__ a, const float *__restrict__ b,
                                                 const float *__restrict__ c) {
  double e1[3], e2[3];
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    const double ak = (double)__ldg(a + k);
    e1[k] = __dsub_rn((double)__ldg(b + k), ak);
    e2[k] = __dsub_rn((double)__ldg(c + k), ak);
  }
  const double nx = __dsub_rn(__dmul_rn(e1[1], e2[2]), __dmul_rn(e1[2], e2[1]));
  const double ny = __dsub_rn(__dmul_rn(e1[2], e2[0]), __dmul_rn(e1[0], e2[2]));
  const double nz = __dsub_rn(__dmul_rn(e1[0], e2[1]), __dmul_rn(e1[1], e2[0]));
  const double s = __dsqrt_rn(__dadd_rn(__dadd_rn(__dmul_rn(nx, nx), __dmul_rn(ny, ny)), __dmul_rn(nz, nz)));
  return s <= 1.7976931348623157e308 ? s : 0.0;   // NaN and inf -> 0
}

// thread per face: the fp64 bits of s into P[f], the per-sample maximum into smax (warp-reduced when the warp is one sample)
__global__ void __launch_bounds__(SS_THREADS)
ss_weight_kernel(const float *__restrict__ verts, const int *__restrict__ faces, long long F,
                 const long long *__restrict__ vert_off, const long long *__restrict__ face_off, int N,
                 unsigned long long *__restrict__ P, unsigned long long *__restrict__ smax) {
  const long long f = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const bool ok = f < F;
  const int n = ok ? ss_sample_of(face_off, N, f) : -1;
  unsigned long long bits = 0;
  if (ok) {
    const float *vb = verts + 3 * __ldg(vert_off + n);
    const double s = ss_face_weight(vb + 3 * __ldg(faces + 3 * f), vb + 3 * __ldg(faces + 3 * f + 1),
                                    vb + 3 * __ldg(faces + 3 * f + 2));
    bits = (unsigned long long)__double_as_longlong(s);
    P[f] = bits;
  }
  const int n0 = __shfl_sync(0xffffffffu, n, 0);
  if (__all_sync(0xffffffffu, n == n0 || n < 0)) {
    if (n0 < 0) return;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const unsigned long long y = __shfl_xor_sync(0xffffffffu, bits, o);
      bits = y > bits ? y : bits;
    }
    if ((threadIdx.x & 31) == 0) atomicMax(smax + n0, bits);
  } else if (ok) {
    atomicMax(smax + n, bits);
  }
}

__device__ __forceinline__ unsigned long long ss_quantise(unsigned long long sbits, double smax) {
  if (!(smax > 0.0)) return 0ull;
  const double q = __ddiv_rn(__longlong_as_double((long long)sbits), smax);   // in [0, 1]
  return __double2ull_rz(__dmul_rn(q, 4294967296.0));                          // floor of a non-negative value
}

// one CTA per sample: P[f] (s bits on entry) -> the inclusive prefix sum of the quantised weights
__global__ void __launch_bounds__(SS_SCAN_THREADS)
ss_scan_kernel(const long long *__restrict__ face_off, const unsigned long long *__restrict__ smax,
               unsigned long long *__restrict__ P) {
  __shared__ unsigned long long s_warp[SS_SCAN_THREADS / 32];
  const int b = blockIdx.x;
  const long long fb = face_off[b], nf = face_off[b + 1] - fb;
  const double mx = __longlong_as_double((long long)smax[b]);
  unsigned long long *p = P + fb;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  unsigned long long carry = 0;
  for (long long base = 0; base < nf; base += SS_SCAN_THREADS * SS_SCAN_ITEMS) {
    const long long i0 = base + (long long)threadIdx.x * SS_SCAN_ITEMS;
    unsigned long long w[SS_SCAN_ITEMS];
#pragma unroll
    for (int k = 0; k < SS_SCAN_ITEMS; ++k) w[k] = i0 + k < nf ? ss_quantise(p[i0 + k], mx) : 0ull;
#pragma unroll
    for (int k = 1; k < SS_SCAN_ITEMS; ++k) w[k] += w[k - 1];
    const unsigned long long total = w[SS_SCAN_ITEMS - 1];
    unsigned long long inc = total;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const unsigned long long y = __shfl_up_sync(0xffffffffu, inc, o);
      if (lane >= o) inc += y;
    }
    if (lane == 31) s_warp[warp] = inc;
    __syncthreads();
    if (warp == 0) {
      const unsigned long long wt = s_warp[lane];
      unsigned long long wi = wt;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const unsigned long long y = __shfl_up_sync(0xffffffffu, wi, o);
        if (lane >= o) wi += y;
      }
      s_warp[lane] = wi;   // inclusive over warps
    }
    __syncthreads();
    const unsigned long long before = carry + (warp ? s_warp[warp - 1] : 0ull) + (inc - total);
#pragma unroll
    for (int k = 0; k < SS_SCAN_ITEMS; ++k)
      if (i0 + k < nf) p[i0 + k] = before + w[k];
    carry += s_warp[SS_SCAN_THREADS / 32 - 1];
    __syncthreads();   // s_warp is rewritten by the next tile
  }
}

// grid (point blocks, N): thread per (point, sample)
__global__ void __launch_bounds__(SS_THREADS)
ss_sample_kernel(const float *__restrict__ verts, const int *__restrict__ faces, const long long *__restrict__ vert_off,
                 const long long *__restrict__ face_off, const unsigned long long *__restrict__ seeds,
                 const unsigned long long *__restrict__ P, long long n, float *__restrict__ points, int *__restrict__ face) {
  const int b = blockIdx.y;
  const long long i = (long long)blockIdx.x * SS_THREADS + threadIdx.x;
  if (i >= n) return;
  const size_t o = (size_t)b * n + i;
  const long long fb = __ldg(face_off + b), nf = __ldg(face_off + b + 1) - fb;
  const unsigned long long *p = P + fb;
  const unsigned long long T = nf > 0 ? p[nf - 1] : 0ull;
  if (T == 0ull) {
    points[3 * o] = points[3 * o + 1] = points[3 * o + 2] = __int_as_float(0x7fc00000);
    face[o] = -1;
    return;
  }
  const unsigned long long seed = __ldg(seeds + b);
  const unsigned long long r0 = ss_splitmix64(seed + (3ull * (unsigned long long)i + 1ull) * SS_GOLDEN);
  const unsigned long long x = __umul64hi(r0, T);
  long long lo = 0, hi = nf - 1;   // P[nf - 1] = T > x: the answer exists
  while (lo < hi) {
    const long long mid = (lo + hi) >> 1;
    if (p[mid] > x) hi = mid;
    else lo = mid + 1;
  }
  float u, v;
  ss_barycentric(seed, i, u, v);
  const int *fp = faces + 3 * (fb + lo);
  const float *vb = verts + 3 * __ldg(vert_off + b);
  const float *A = vb + 3 * __ldg(fp), *B = vb + 3 * __ldg(fp + 1), *C = vb + 3 * __ldg(fp + 2);
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    const float va = __ldg(A + a);
    points[3 * o + a] = __fadd_rn(__fadd_rn(va, __fmul_rn(u, __fsub_rn(__ldg(B + a), va))), __fmul_rn(v, __fsub_rn(__ldg(C + a), va)));
  }
  face[o] = (int)lo;
}

// grid (point blocks, N): thread per (point, sample); grad_verts zeroed beforehand
__global__ void __launch_bounds__(SS_THREADS)
ss_sample_backward_kernel(const int *__restrict__ faces, const long long *__restrict__ vert_off,
                          const long long *__restrict__ face_off, const unsigned long long *__restrict__ seeds, long long n,
                          const int *__restrict__ face, const float *__restrict__ grad_points, float *__restrict__ grad_verts) {
  const int b = blockIdx.y;
  const long long i = (long long)blockIdx.x * SS_THREADS + threadIdx.x;
  if (i >= n) return;
  const size_t o = (size_t)b * n + i;
  const int f = __ldg(face + o);
  if (f < 0) return;
  float u, v;
  ss_barycentric(__ldg(seeds + b), i, u, v);
  const float w[3] = {__fsub_rn(__fsub_rn(1.0f, u), v), u, v};   // exact: u, v are multiples of 2^-24 with u + v <= 1
  const int *fp = faces + 3 * (__ldg(face_off + b) + f);
  float *gv = grad_verts + 3 * __ldg(vert_off + b);
  const float g[3] = {__ldg(grad_points + 3 * o), __ldg(grad_points + 3 * o + 1), __ldg(grad_points + 3 * o + 2)};
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    float *dst = gv + 3 * (size_t)__ldg(fp + c);
#pragma unroll
    for (int a = 0; a < 3; ++a) atomicAdd(dst + a, __fmul_rn(w[c], g[a]));
  }
}

struct SsLayout {
  size_t smax, P, total;   // byte offsets into the workspace
};

static size_t ss_align(size_t x) { return (x + 255) & ~(size_t)255; }

static bool ss_layout(int64_t N, int64_t F, SsLayout *L) {
  if (N < 1 || N > 65535 || F < 0 || F >= SS_MAX_FACES) return false;
  L->smax = 0;
  L->P = ss_align((size_t)N * sizeof(unsigned long long));
  L->total = L->P + ss_align((size_t)F * sizeof(unsigned long long));
  return true;
}

static unsigned ss_blocks(long long n, int threads) { return (unsigned)((n + threads - 1) / threads); }

}  // namespace gb

using namespace gb;

extern "C" size_t genre_b200_surface_sample_workspace_bytes(int64_t N, int64_t F) {
  SsLayout L{};
  return ss_layout(N, F, &L) ? L.total : 0;
}

extern "C" int genre_b200_surface_sample(const float *verts, int64_t V, const int32_t *faces, int64_t F,
                                         const int64_t *vert_off, const int64_t *face_off, int64_t N, const uint64_t *seeds,
                                         int64_t n, float *points, int32_t *face, void *workspace, size_t workspace_bytes,
                                         void *stream) {
  GB_REQUIRE(vert_off && face_off && seeds && points && face && workspace && (verts || V == 0) && (faces || F == 0),
             GENRE_B200_EINVAL, "surface_sample: null pointer");
  GB_REQUIRE(N >= 1 && N <= 65535, GENRE_B200_EINVAL, "surface_sample: N=%lld out of range [1, 65535]", (long long)N);
  GB_REQUIRE(V >= 0 && V <= ((int64_t)1 << 40) && F >= 0 && F < SS_MAX_FACES, GENRE_B200_EINVAL,
             "surface_sample: V=%lld, F=%lld out of range (F < 2^31)", (long long)V, (long long)F);
  GB_REQUIRE(n >= 1 && n <= SS_MAX_POINTS, GENRE_B200_EINVAL, "surface_sample: n=%lld out of range [1, 2^30]", (long long)n);
  SsLayout L{};
  ss_layout(N, F, &L);
  GB_REQUIRE(workspace_bytes >= L.total && aligned16(workspace), GENRE_B200_EWORKSPACE,
             "surface_sample: workspace too small or misaligned (%zu bytes needed, 16-byte aligned)", L.total);
  cudaStream_t st = as_stream(stream);
  char *ws = (char *)workspace;
  unsigned long long *smax = (unsigned long long *)(ws + L.smax), *P = (unsigned long long *)(ws + L.P);
  const long long *vo = (const long long *)vert_off, *fo = (const long long *)face_off;
  if (F > 0) {
    const cudaError_t e = cudaMemsetAsync(smax, 0, (size_t)N * sizeof(unsigned long long), st);
    if (e != cudaSuccess) {
      set_error("surface_sample: memset: %s", cudaGetErrorString(e));
      return (int)e;
    }
    ss_weight_kernel<<<ss_blocks(F, SS_THREADS), SS_THREADS, 0, st>>>(verts, faces, F, vo, fo, (int)N, P, smax);
    if (int rc = check_launch("surface_sample weight kernel")) return rc;
    ss_scan_kernel<<<(unsigned)N, SS_SCAN_THREADS, 0, st>>>(fo, smax, P);
    if (int rc = check_launch("surface_sample scan kernel")) return rc;
  }
  ss_sample_kernel<<<dim3(ss_blocks(n, SS_THREADS), (unsigned)N), SS_THREADS, 0, st>>>(
      verts, faces, vo, fo, (const unsigned long long *)seeds, P, n, points, face);
  return check_launch("surface_sample kernel");
}

extern "C" int genre_b200_surface_sample_backward(const int32_t *faces, int64_t F, const int64_t *vert_off,
                                                  const int64_t *face_off, int64_t N, const uint64_t *seeds, int64_t n,
                                                  const int32_t *face, const float *grad_points, int64_t V, float *grad_verts,
                                                  void *stream) {
  GB_REQUIRE(vert_off && face_off && seeds && face && grad_points && (faces || F == 0) && (grad_verts || V == 0),
             GENRE_B200_EINVAL, "surface_sample_backward: null pointer");
  GB_REQUIRE(N >= 1 && N <= 65535, GENRE_B200_EINVAL, "surface_sample_backward: N=%lld out of range [1, 65535]", (long long)N);
  GB_REQUIRE(V >= 0 && V <= ((int64_t)1 << 40) && F >= 0 && F < SS_MAX_FACES, GENRE_B200_EINVAL,
             "surface_sample_backward: V=%lld, F=%lld out of range (F < 2^31)", (long long)V, (long long)F);
  GB_REQUIRE(n >= 1 && n <= SS_MAX_POINTS, GENRE_B200_EINVAL, "surface_sample_backward: n=%lld out of range [1, 2^30]",
             (long long)n);
  if (V == 0) return 0;   // no vertex: no face was drawn either
  cudaStream_t st = as_stream(stream);
  const cudaError_t e = cudaMemsetAsync(grad_verts, 0, (size_t)V * 3 * sizeof(float), st);
  if (e != cudaSuccess) {
    set_error("surface_sample_backward: memset: %s", cudaGetErrorString(e));
    return (int)e;
  }
  ss_sample_backward_kernel<<<dim3(ss_blocks(n, SS_THREADS), (unsigned)N), SS_THREADS, 0, st>>>(
      faces, (const long long *)vert_off, (const long long *)face_off, (const unsigned long long *)seeds, n, face, grad_points,
      grad_verts);
  return check_launch("surface_sample backward kernel");
}
