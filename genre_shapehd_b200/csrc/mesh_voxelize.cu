// mesh_voxelize.cu — conservative voxelisation of batched triangle meshes on the GPU: the inverse of marching cubes, so that
// ground-truth meshes (ShapeNet, Pix3D) can be scored by voxel_iou and made into training grids without a CPU tool.
//
// Contract (include/genre_b200.h states it too; tests/mesh_voxelize_ref.py restates it in numpy, bit for bit):
//   meshes  the packed format of genre_b200_isosurface_*: verts [sum V, 3] fp32, faces [sum F, 3] int32 with indices local to
//           the sample, vert_off / face_off [N+1] int64 on the device.  Indices lie in [0, V_n) (trusted).  F < 2^31.
//   frame   voxel (i0, i1, i2) of the (n0, n1, n2) = (D, H, W) grid is the closed cube [i_a/n_a - 0.5, (i_a+1)/n_a - 0.5] per
//           axis, axis 0 = vertex coordinate 0 = the first array axis.  Everything below is fp64 from the fp32 vertices, one
//           rounding per operation, no contraction, in the order written.  Grid units: g_a = (p_a + 0.5) * n_a, so the voxel
//           is the box [i_a, i_a + 1].
//   skip    a face with a non-finite vertex coordinate, or whose normal e1 x e2 (e1 = b - a, e2 = c - a, components as in
//           csrc/surface_sample.cu: nx = e1y*e2z - e1z*e2y, ...) is exactly 0 in all three components (common.cuh's
//           mesh_face_kept, shared with csrc/winding.cu).
//   test    a voxel is set iff the closed triangle and the closed cube intersect, by the separating-axis test in grid units
//           (touching is overlap: a separation needs a strict inequality):
//             box axes   voxel i_a lies in [max(ceil(min_k g_ka) - 1, 0), min(floor(max_k g_ka), n_a - 1)] on every axis;
//             translate  v_ka = g_ka - (i_a + 0.5);
//             normal     f0 = g1 - g0, f1 = g2 - g1, f2 = g0 - g2, e = g2 - g0 (per axis); m = f0 x e in the order above;
//                        separated iff |(m0*v00 + m1*v01) + m2*v02| > 0.5 * ((|m0| + |m1|) + |m2|);
//             edges      for j = 0, 1, 2 and the box axes 0, 1, 2, the axis (A on axis s, B on axis t, s < t) =
//                        (-f_j2 on 1, f_j1 on 2), (f_j2 on 0, -f_j0 on 2), (-f_j1 on 0, f_j0 on 1); per vertex
//                        p_k = A*v_ks + B*v_kt, r = 0.5 * (|A| + |B|); separated iff min_k p_k > r or max_k p_k < -r.
//   output  out [N, D, H, W] fp32: 1.0 for a set voxel, 0.0 elsewhere, written once and dense.  Deterministic and
//           batch-equivariant; nothing is copied to the host, so a call can be captured in a CUDA graph.
//
// Kernels: mv_count_kernel (thread per face: its columns, the grid-clipped box in the two axes other than the normal's
// dominant one, ties to the lowest axis), mv_scan_kernel (one CTA per sample: inclusive int64 prefix sums of the counts),
// mv_column_kernel (a fixed grid per sample strides over the sample's columns, read on the device; a binary search finds the
// column's face; the voxels of the column that pass the normal's test form one interval, found from an estimate and
// corrected exactly, and each of them takes the nine edge tests; hits go by atomicOr into a bit-packed [N][D][H][ceil(W/32)]
// grid, which is order-free), mv_expand_kernel (thread per output voxel).
//
// Why the column walk drops nothing that the full test accepts: along the dominant axis d only v_0d changes with the layer i,
// and fl(g_0d - (i + 0.5)), the product with m_d and the two sums are each monotone in i, so the normal's rounded value is
// monotone in i and the layers where it passes are one interval.  The walk finds exactly that interval inside the box.
#include "common.cuh"

namespace gb {

constexpr int MV_THREADS = 256;
constexpr int MV_SCAN_THREADS = 1024;
constexpr int MV_SCAN_ITEMS = 8;
constexpr int MV_MAX_DIM = 512;
constexpr int64_t MV_MAX_FACES = (int64_t)1 << 31;   // exclusive

// largest n with off[n] <= i (empty samples are skipped over)
__device__ __forceinline__ int mv_sample_of(const long long *__restrict__ off, int N, long long i) {
  int lo = 0, hi = N - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (__ldg(off + mid) <= i) lo = mid;
    else hi = mid - 1;
  }
  return lo;
}

struct MvFace {
  double g[3][3];     // [vertex][axis], grid units
  double m[3];        // f0 x e, grid units
  int lo[3], hi[3];   // the grid-clipped box, inclusive
  int d, u, v;        // dominant axis of m; column axes u < v
};

// false: the face is skipped or its box misses the grid
__device__ __forceinline__ bool mv_face(const float *__restrict__ vb, const int *__restrict__ fp, const int (&dims)[3],
                                        MvFace &F) {
  float p[3][3];
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    const float *q = vb + 3 * __ldg(fp + k);
#pragma unroll
    for (int a = 0; a < 3; ++a) p[k][a] = __ldg(q + a);
  }
  if (!mesh_face_kept(p)) return false;
#pragma unroll
  for (int k = 0; k < 3; ++k)
#pragma unroll
    for (int a = 0; a < 3; ++a) F.g[k][a] = __dmul_rn(__dadd_rn((double)p[k][a], 0.5), (double)dims[a]);
  bool empty = false;
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    const double mn = fmin(fmin(F.g[0][a], F.g[1][a]), F.g[2][a]);
    const double mx = fmax(fmax(F.g[0][a], F.g[1][a]), F.g[2][a]);
    const double lo = fmax(__dsub_rn(ceil(mn), 1.0), 0.0), hi = fmin(floor(mx), (double)(dims[a] - 1));
    empty = empty || lo > hi;
    F.lo[a] = lo > hi ? 0 : (int)lo;
    F.hi[a] = lo > hi ? -1 : (int)hi;
  }
  if (empty) return false;
  double f0[3], e[3];
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    f0[a] = __dsub_rn(F.g[1][a], F.g[0][a]);
    e[a] = __dsub_rn(F.g[2][a], F.g[0][a]);
  }
  F.m[0] = __dsub_rn(__dmul_rn(f0[1], e[2]), __dmul_rn(f0[2], e[1]));
  F.m[1] = __dsub_rn(__dmul_rn(f0[2], e[0]), __dmul_rn(f0[0], e[2]));
  F.m[2] = __dsub_rn(__dmul_rn(f0[0], e[1]), __dmul_rn(f0[1], e[0]));
  const double a0 = fabs(F.m[0]), a1 = fabs(F.m[1]), a2 = fabs(F.m[2]);
  const int d = a1 > a0 ? (a2 > a1 ? 2 : 1) : (a2 > a0 ? 2 : 0);   // ties to the lowest axis
  F.d = d;
  F.u = d == 0 ? 1 : 0;
  F.v = d == 2 ? 1 : 2;
  return true;
}

// x[i] by selects, so that a run-time axis keeps the face in registers
template <typename T>
__device__ __forceinline__ T mv_sel(const T (&x)[3], int i) {
  return i == 0 ? x[0] : (i == 1 ? x[1] : x[2]);
}

__device__ __forceinline__ long long mv_columns(const MvFace &F) {
  return (long long)(mv_sel(F.hi, F.u) - mv_sel(F.lo, F.u) + 1) * (mv_sel(F.hi, F.v) - mv_sel(F.lo, F.v) + 1);
}

// separated along the axis with A on component s and B on component t of the translated vertices
__device__ __forceinline__ bool mv_separated(double A, double B, double s0, double t0, double s1, double t1, double s2,
                                             double t2) {
  const double p0 = __dadd_rn(__dmul_rn(A, s0), __dmul_rn(B, t0));
  const double p1 = __dadd_rn(__dmul_rn(A, s1), __dmul_rn(B, t1));
  const double p2 = __dadd_rn(__dmul_rn(A, s2), __dmul_rn(B, t2));
  const double r = __dmul_rn(0.5, __dadd_rn(fabs(A), fabs(B)));
  return fmin(fmin(p0, p1), p2) > r || fmax(fmax(p0, p1), p2) < -r;
}

// the nine edge axes for the voxel whose centre is c
__device__ __forceinline__ bool mv_edges_overlap(const MvFace &F, const double (&c)[3]) {
  double v[3][3];
#pragma unroll
  for (int k = 0; k < 3; ++k)
#pragma unroll
    for (int a = 0; a < 3; ++a) v[k][a] = __dsub_rn(F.g[k][a], c[a]);
#pragma unroll
  for (int j = 0; j < 3; ++j) {
    const int k1 = j == 2 ? 0 : j + 1;
    const double f0 = __dsub_rn(F.g[k1][0], F.g[j][0]), f1 = __dsub_rn(F.g[k1][1], F.g[j][1]),
                 f2 = __dsub_rn(F.g[k1][2], F.g[j][2]);
    if (mv_separated(-f2, f1, v[0][1], v[0][2], v[1][1], v[1][2], v[2][1], v[2][2])) return false;
    if (mv_separated(f2, -f0, v[0][0], v[0][2], v[1][0], v[1][2], v[2][0], v[2][2])) return false;
    if (mv_separated(-f1, f0, v[0][0], v[0][1], v[1][0], v[1][1], v[2][0], v[2][1])) return false;
  }
  return true;
}

// thread per face: its column count into P[f]
__global__ void __launch_bounds__(MV_THREADS)
mv_count_kernel(const float *__restrict__ verts, const int *__restrict__ faces, long long F,
                const long long *__restrict__ vert_off, const long long *__restrict__ face_off, int N, int D, int H, int W,
                long long *__restrict__ P) {
  const long long f = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= F) return;
  const int n = mv_sample_of(face_off, N, f);
  const int dims[3] = {D, H, W};
  MvFace face;
  P[f] = mv_face(verts + 3 * __ldg(vert_off + n), faces + 3 * f, dims, face) ? mv_columns(face) : 0ll;
}

// one CTA per sample: P[f] (counts on entry) -> their inclusive prefix sum within the sample
__global__ void __launch_bounds__(MV_SCAN_THREADS)
mv_scan_kernel(const long long *__restrict__ face_off, long long *__restrict__ P) {
  __shared__ long long s_warp[MV_SCAN_THREADS / 32];
  const int b = blockIdx.x;
  const long long fb = face_off[b], nf = face_off[b + 1] - fb;
  long long *p = P + fb;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  long long carry = 0;
  for (long long base = 0; base < nf; base += MV_SCAN_THREADS * MV_SCAN_ITEMS) {
    const long long i0 = base + (long long)threadIdx.x * MV_SCAN_ITEMS;
    long long w[MV_SCAN_ITEMS];
#pragma unroll
    for (int k = 0; k < MV_SCAN_ITEMS; ++k) w[k] = i0 + k < nf ? p[i0 + k] : 0ll;
#pragma unroll
    for (int k = 1; k < MV_SCAN_ITEMS; ++k) w[k] += w[k - 1];
    const long long total = w[MV_SCAN_ITEMS - 1];
    long long inc = total;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const long long y = __shfl_up_sync(0xffffffffu, inc, o);
      if (lane >= o) inc += y;
    }
    if (lane == 31) s_warp[warp] = inc;
    __syncthreads();
    if (warp == 0) {
      long long wi = s_warp[lane];
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const long long y = __shfl_up_sync(0xffffffffu, wi, o);
        if (lane >= o) wi += y;
      }
      s_warp[lane] = wi;   // inclusive over warps
    }
    __syncthreads();
    const long long before = carry + (warp ? s_warp[warp - 1] : 0ll) + (inc - total);
#pragma unroll
    for (int k = 0; k < MV_SCAN_ITEMS; ++k)
      if (i0 + k < nf) p[i0 + k] = before + w[k];
    carry += s_warp[MV_SCAN_THREADS / 32 - 1];
    __syncthreads();   // s_warp is rewritten by the next tile
  }
}

// the normal's rounded signed distance from the voxel centre c, times the sign of m_d (non-increasing in the layer)
__device__ __forceinline__ double mv_plane(const MvFace &F, const double (&c)[3], double sgn) {
  const double d = __dadd_rn(__dadd_rn(__dmul_rn(F.m[0], __dsub_rn(F.g[0][0], c[0])), __dmul_rn(F.m[1], __dsub_rn(F.g[0][1], c[1]))),
                             __dmul_rn(F.m[2], __dsub_rn(F.g[0][2], c[2])));
  return sgn * d;
}

// grid (blocks per sample, N): threads stride over the sample's columns
__global__ void __launch_bounds__(MV_THREADS)
mv_column_kernel(const float *__restrict__ verts, const int *__restrict__ faces, const long long *__restrict__ vert_off,
                 const long long *__restrict__ face_off, int D, int H, int W, const long long *__restrict__ P,
                 unsigned *__restrict__ bits) {
  const int b = blockIdx.y;
  const long long fb = __ldg(face_off + b), nf = __ldg(face_off + b + 1) - fb;
  if (nf == 0) return;
  const long long *p = P + fb;
  const long long T = p[nf - 1];
  const int dims[3] = {D, H, W};
  const int W32 = (W + 31) >> 5;
  const float *vb = verts + 3 * __ldg(vert_off + b);
  unsigned *grid = bits + (size_t)b * D * H * W32;
  for (long long col = (long long)blockIdx.x * MV_THREADS + threadIdx.x; col < T;
       col += (long long)gridDim.x * MV_THREADS) {
    long long lo = 0, hi = nf - 1;   // the smallest f with P_f > col: P[nf - 1] = T > col
    while (lo < hi) {
      const long long mid = (lo + hi) >> 1;
      if (p[mid] > col) hi = mid;
      else lo = mid + 1;
    }
    MvFace F;
    mv_face(vb, faces + 3 * (fb + lo), dims, F);   // true: the face has columns
    const long long local = col - (lo > 0 ? p[lo - 1] : 0ll);
    const int d = F.d, blo = mv_sel(F.lo, d), bhi = mv_sel(F.hi, d);
    const int nv = mv_sel(F.hi, F.v) - mv_sel(F.lo, F.v) + 1;
    const double cu = (double)(mv_sel(F.lo, F.u) + (int)(local / nv)) + 0.5;
    const double cv = (double)(mv_sel(F.lo, F.v) + (int)(local % nv)) + 0.5;
    const double md = mv_sel(F.m, d);
    const double r = __dmul_rn(0.5, __dadd_rn(__dadd_rn(fabs(F.m[0]), fabs(F.m[1])), fabs(F.m[2])));
    int l0 = blo, l1 = bhi;
    double sgn = 1.0;
    if (md != 0.0) {
      // estimate: the plane's d-coordinate over the column's centre; the touching layers lie within 2 of it
      sgn = md > 0.0 ? 1.0 : -1.0;
      const double z = mv_sel(F.g[0], d) - (mv_sel(F.m, F.u) * (cu - mv_sel(F.g[0], F.u)) +
                                            mv_sel(F.m, F.v) * (cv - mv_sel(F.g[0], F.v))) / md;
      const double zf = floor(z);
      if (zf == zf) {
        l0 = (int)fmin(fmax(zf - 2.0, (double)blo), (double)bhi);
        l1 = (int)fmin(fmax(zf + 2.0, (double)blo), (double)bhi);
      }
    }  // else m = 0 (a sliver below fp64 resolution in grid units): the normal passes every layer
    // the voxel centre of layer i in this column, axes in array order (u < v are the two axes other than d)
    auto centre = [&](int i, double (&c)[3]) {
      const double cd = (double)i + 0.5;
      c[0] = d == 0 ? cd : cu;
      c[1] = d == 0 ? cu : (d == 1 ? cd : cv);
      c[2] = d == 2 ? cd : cv;
    };
    double c[3];
    // exact correction: l0 = the first layer with q <= r, l1 = the last with q >= -r (q non-increasing)
    for (;;) {
      if (l0 <= blo) break;
      centre(l0 - 1, c);
      if (mv_plane(F, c, sgn) > r) break;
      --l0;
    }
    for (; l0 <= bhi; ++l0) {
      centre(l0, c);
      if (mv_plane(F, c, sgn) <= r) break;
    }
    for (;;) {
      if (l1 >= bhi) break;
      centre(l1 + 1, c);
      if (mv_plane(F, c, sgn) < -r) break;
      ++l1;
    }
    for (; l1 >= blo; --l1) {
      centre(l1, c);
      if (mv_plane(F, c, sgn) >= -r) break;
    }
    for (int i = l0; i <= l1; ++i) {
      centre(i, c);
      if (!mv_edges_overlap(F, c)) continue;
      const int i0 = (int)c[0], i1 = (int)c[1], i2 = (int)c[2];
      atomicOr(grid + ((size_t)i0 * H + i1) * W32 + (i2 >> 5), 1u << (i2 & 31));
    }
  }
}

// thread per output voxel
__global__ void __launch_bounds__(MV_THREADS)
mv_expand_kernel(const unsigned *__restrict__ bits, long long total, int W, float *__restrict__ out) {
  const int W32 = (W + 31) >> 5;
  for (long long o = (long long)blockIdx.x * MV_THREADS + threadIdx.x; o < total; o += (long long)gridDim.x * MV_THREADS) {
    const long long row = o / W;
    const int x = (int)(o - row * W);
    out[o] = (__ldg(bits + row * W32 + (x >> 5)) >> (x & 31)) & 1u ? 1.0f : 0.0f;
  }
}

struct MvLayout {
  size_t bits, bits_bytes, P, total;   // byte offsets and sizes in the workspace
};

static size_t mv_align(size_t x) { return (x + 255) & ~(size_t)255; }

static bool mv_layout(int64_t N, int64_t F, int D, int H, int W, MvLayout *L) {
  if (N < 1 || N > 65535 || F < 0 || F >= MV_MAX_FACES || D < 1 || D > MV_MAX_DIM || H < 1 || H > MV_MAX_DIM || W < 1 ||
      W > MV_MAX_DIM)
    return false;
  L->bits = 0;
  L->bits_bytes = (size_t)N * D * H * ((W + 31) / 32) * sizeof(unsigned);
  L->P = mv_align(L->bits_bytes);
  L->total = L->P + mv_align((size_t)F * sizeof(long long));
  return true;
}

}  // namespace gb

using namespace gb;

extern "C" size_t genre_b200_mesh_voxelize_workspace_bytes(int64_t N, int64_t F, int D, int H, int W) {
  MvLayout L{};
  return mv_layout(N, F, D, H, W, &L) ? L.total : 0;
}

extern "C" int genre_b200_mesh_voxelize(const float *verts, int64_t V, const int32_t *faces, int64_t F,
                                        const int64_t *vert_off, const int64_t *face_off, int64_t N, int D, int H, int W,
                                        float *out, void *workspace, size_t workspace_bytes, void *stream) {
  GB_REQUIRE(vert_off && face_off && out && workspace && (verts || V == 0) && (faces || F == 0), GENRE_B200_EINVAL,
             "mesh_voxelize: null pointer");
  GB_REQUIRE(N >= 1 && N <= 65535, GENRE_B200_EINVAL, "mesh_voxelize: N=%lld out of range [1, 65535]", (long long)N);
  GB_REQUIRE(V >= 0 && V <= ((int64_t)1 << 40) && F >= 0 && F < MV_MAX_FACES, GENRE_B200_EINVAL,
             "mesh_voxelize: V=%lld, F=%lld out of range (F < 2^31)", (long long)V, (long long)F);
  GB_REQUIRE(D >= 1 && D <= MV_MAX_DIM && H >= 1 && H <= MV_MAX_DIM && W >= 1 && W <= MV_MAX_DIM, GENRE_B200_EINVAL,
             "mesh_voxelize: grid %dx%dx%d out of range (every dimension in [1, 512])", D, H, W);
  MvLayout L{};
  mv_layout(N, F, D, H, W, &L);
  GB_REQUIRE(workspace_bytes >= L.total && aligned16(workspace), GENRE_B200_EWORKSPACE,
             "mesh_voxelize: workspace too small or misaligned (%zu bytes needed, 16-byte aligned)", L.total);
  cudaStream_t st = as_stream(stream);
  char *ws = (char *)workspace;
  unsigned *bits = (unsigned *)(ws + L.bits);
  long long *P = (long long *)(ws + L.P);
  const long long *vo = (const long long *)vert_off, *fo = (const long long *)face_off;
  const cudaError_t e = cudaMemsetAsync(bits, 0, L.bits_bytes, st);
  if (e != cudaSuccess) {
    set_error("mesh_voxelize: memset: %s", cudaGetErrorString(e));
    return (int)e;
  }
  if (F > 0) {
    mv_count_kernel<<<(unsigned)((F + MV_THREADS - 1) / MV_THREADS), MV_THREADS, 0, st>>>(verts, faces, F, vo, fo, (int)N, D,
                                                                                           H, W, P);
    if (int rc = check_launch("mesh_voxelize count kernel")) return rc;
    mv_scan_kernel<<<(unsigned)N, MV_SCAN_THREADS, 0, st>>>(fo, P);
    if (int rc = check_launch("mesh_voxelize scan kernel")) return rc;
    // a fixed grid (the column totals stay on the device): about 8 CTAs per SM over the whole batch
    const int per_sample = (int)((8LL * sm_count() + N - 1) / N);
    mv_column_kernel<<<dim3((unsigned)per_sample, (unsigned)N), MV_THREADS, 0, st>>>(verts, faces, vo, fo, D, H, W, P, bits);
    if (int rc = check_launch("mesh_voxelize column kernel")) return rc;
  }
  const long long total = (long long)N * D * H * W;
  const long long blocks = (total + MV_THREADS - 1) / MV_THREADS;
  const unsigned grid = (unsigned)(blocks < 16LL * sm_count() ? blocks : 16LL * sm_count());
  mv_expand_kernel<<<grid, MV_THREADS, 0, st>>>(bits, total, W, out);
  return check_launch("mesh_voxelize expand kernel");
}
