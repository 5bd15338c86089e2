// raycast.cu — first-hit ray casting of batched triangle meshes on the GPU (SURVEY 8f-4): the trimesh call of the published
// test path (util/util_sph.py:7-18, mesh.ray.intersects_id(..., multiple_hits=False)) for a whole batch on the device.
//
// Contract (include/genre_b200.h states it too; oracle_ray/raycast_oracle.c restates it in scalar C, bit for bit):
//   meshes  the packed format of genre_b200_isosurface_*: verts [sum V, 3] fp32, faces [sum F, 3] int32 with indices local to
//           the sample, vert_off / face_off [N+1] int64 on the device.  Vertices are finite; indices lie in [0, V_n).
//   rays    origin o, direction d (not necessarily unit).  A ray with a non-finite component or d = 0 misses everything.
//   face    DEGENERATE iff its fp32 normal is zero: e1 = v1 - v0, e2 = v2 - v0, n = (e1y*e2z - e1z*e2y, ...), every product and
//           difference rounded once.  Degenerate faces never hit (marching cubes emits them where a value equals the level).
//   hit     Woop-Benthin-Wald watertight test, two-sided, in fp32 with one rounding per step (__f*_rn, no contraction):
//             kz = the axis of the largest |d_a| (the lowest on ties), kx = kz+1, ky = kx+1 (mod 3), swapped if d_kz < 0;
//             Sx = d_kx / d_kz, Sy = d_ky / d_kz, Sz = 1 / d_kz;
//             for each vertex P: p = P - o (per axis), px = p_kx - Sx*p_kz, py = p_ky - Sy*p_kz, pz = Sz*p_kz;
//             U = Cx*By - Cy*Bx, V = Ax*Cy - Ay*Cx, W = Bx*Ay - By*Ax   (A, B, C the sheared v0, v1, v2);
//             miss if (U<0 || V<0 || W<0) && (U>0 || V>0 || W>0);  det = (U + V) + W, miss if det == 0;
//             T = (U*Az + V*Bz) + W*Cz;  t = T / det;  hit iff 0 < t < +inf.
//           A shared edge is evaluated from the same two sheared vertices in both faces, and its edge function comes out
//           exactly negated, so a ray through an edge or a vertex of a closed mesh cannot slip between its faces.
//   result  per (sample, ray): the hit with the smallest t, ties to the smallest face index; t = +inf and face = -1 on a miss.
//           face is local to the sample.  It equals a loop over all of the sample's faces for every grid resolution G.
//
// Acceleration (no effect on the result): a uniform G^3 grid per sample over the vertex box padded by eta = 2^-12 * M (M the
// largest coordinate magnitude of the box) on every side.
//   count : box by order-preserving integer atomics (deterministic); per sample the largest face extent along each axis; every
//           non-degenerate face is binned into all cells that meet its box padded by eta; the per-cell counts and their sum
//           refs[n] are written.
//   build : per sample exclusive scan of the cell counts, then the face ids go into their cells (any order within a cell).
//   first_hit: thread per (ray, sample).  Clip the ray to the padded box, walk the cells with a 3D-DDA (boundary parameters
//           recomputed from the planes at each step, no accumulation), test every face of each cell, keep the best (t, face)
//           lexicographically — so the order of the lists and faces seen twice do not matter.
// Why the walk finds the brute-force answer.  Let g be any face the test accepts with t_g.  Because U, V, W share det's sign
// and T is the same weighted sum, t_g is (to a few ulps) a convex combination of Az, Bz, Cz: the ray point at t_g has its kz
// coordinate inside g's kz range.  The accepted ray also passes (to a few ulps) through g at some t*, whose kz coordinate is in
// the same range, so |t_g - t*| <= ext_kz(g) / |d_kz| <= E = (maxext_kz + 4 eta) / |d_kz| * (1 + 2^-10).  All rounding errors
// of the clip, the DDA planes, the cell indices and the test are a few ulps of max(M, |o|) <= 2^-14 M when |o| <= 2^6 M, i.e.
// below eta / 4; so the DDA's cell at t* lies within eta of g's box and g is in its list.  The walk stops after a cell only when
// best_t + E <= t_exit (rounded up): any face that could beat or tie the best has t* <= t_exit, hence sits in a visited cell.
// A ray with |o|_inf > 2^6 M loops over all faces instead (no error argument needed).  Hence the result does not depend on G.
#include "common.cuh"

namespace gb {

constexpr int RC_THREADS = 128;
constexpr int RC_SCAN_THREADS = 1024;
constexpr int RC_MAX_GRID = 256;

struct RcGrid {          // per sample, written by rc_grid_kernel
  float lo[3], hi[3];    // padded box
  float cell[3], inv[3]; // cell edge and its reciprocal per axis
  float eta, mag;        // binning margin, largest coordinate magnitude of the box
  int empty;             // no vertices, or all equal: every face is degenerate
  int pad_;
};

__device__ __forceinline__ unsigned rc_ord(float f) {
  const unsigned u = __float_as_uint(f);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float rc_unord(unsigned u) { return __uint_as_float((u & 0x80000000u) ? (u & 0x7fffffffu) : ~u); }

// largest n with off[n] <= i (empty samples are skipped over)
__device__ __forceinline__ int rc_sample(const long long *__restrict__ off, int N, long long i) {
  int lo = 0, hi = N - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (__ldg(off + mid) <= i) lo = mid;
    else hi = mid - 1;
  }
  return lo;
}

__device__ __forceinline__ void rc_load3(const float *__restrict__ p, float (&v)[3]) {
  v[0] = __ldg(p);
  v[1] = __ldg(p + 1);
  v[2] = __ldg(p + 2);
}

__device__ __forceinline__ bool rc_degenerate(const float (&a)[3], const float (&b)[3], const float (&c)[3]) {
  const float e1x = __fsub_rn(b[0], a[0]), e1y = __fsub_rn(b[1], a[1]), e1z = __fsub_rn(b[2], a[2]);
  const float e2x = __fsub_rn(c[0], a[0]), e2y = __fsub_rn(c[1], a[1]), e2z = __fsub_rn(c[2], a[2]);
  const float nx = __fsub_rn(__fmul_rn(e1y, e2z), __fmul_rn(e1z, e2y));
  const float ny = __fsub_rn(__fmul_rn(e1z, e2x), __fmul_rn(e1x, e2z));
  const float nz = __fsub_rn(__fmul_rn(e1x, e2y), __fmul_rn(e1y, e2x));
  return nx == 0.0f && ny == 0.0f && nz == 0.0f;
}

struct RcRay {
  float o[3];
  int kx, ky, kz;
  float Sx, Sy, Sz;
};

// false: the ray misses everything (non-finite component or zero direction)
__device__ __forceinline__ bool rc_ray_setup(const float (&o)[3], const float (&d)[3], RcRay &r) {
#pragma unroll
  for (int a = 0; a < 3; ++a)
    if (!isfinite(o[a]) || !isfinite(d[a])) return false;
  const float ax = fabsf(d[0]), ay = fabsf(d[1]), az = fabsf(d[2]);
  const int kz = ax >= ay ? (ax >= az ? 0 : 2) : (ay >= az ? 1 : 2);
  if (d[kz] == 0.0f) return false;
  int kx = kz == 2 ? 0 : kz + 1, ky = kx == 2 ? 0 : kx + 1;
  if (d[kz] < 0.0f) {
    const int s = kx;
    kx = ky;
    ky = s;
  }
  r.kx = kx;
  r.ky = ky;
  r.kz = kz;
  r.Sx = __fdiv_rn(d[kx], d[kz]);
  r.Sy = __fdiv_rn(d[ky], d[kz]);
  r.Sz = __fdiv_rn(1.0f, d[kz]);
#pragma unroll
  for (int a = 0; a < 3; ++a) r.o[a] = o[a];
  return true;
}

__device__ __forceinline__ float rc_pick(const float (&p)[3], int k) { return k == 0 ? p[0] : k == 1 ? p[1] : p[2]; }

// the contract's test; updates (best_t, best_f) lexicographically
__device__ __forceinline__ void rc_test(const RcRay &r, const float (&v0)[3], const float (&v1)[3], const float (&v2)[3], int f,
                                        float &best_t, int &best_f) {
  float A[3], B[3], C[3];
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    A[a] = __fsub_rn(v0[a], r.o[a]);
    B[a] = __fsub_rn(v1[a], r.o[a]);
    C[a] = __fsub_rn(v2[a], r.o[a]);
  }
  const float Akz = rc_pick(A, r.kz), Bkz = rc_pick(B, r.kz), Ckz = rc_pick(C, r.kz);
  const float Ax = __fsub_rn(rc_pick(A, r.kx), __fmul_rn(r.Sx, Akz)), Ay = __fsub_rn(rc_pick(A, r.ky), __fmul_rn(r.Sy, Akz));
  const float Bx = __fsub_rn(rc_pick(B, r.kx), __fmul_rn(r.Sx, Bkz)), By = __fsub_rn(rc_pick(B, r.ky), __fmul_rn(r.Sy, Bkz));
  const float Cx = __fsub_rn(rc_pick(C, r.kx), __fmul_rn(r.Sx, Ckz)), Cy = __fsub_rn(rc_pick(C, r.ky), __fmul_rn(r.Sy, Ckz));
  const float U = __fsub_rn(__fmul_rn(Cx, By), __fmul_rn(Cy, Bx));
  const float V = __fsub_rn(__fmul_rn(Ax, Cy), __fmul_rn(Ay, Cx));
  const float W = __fsub_rn(__fmul_rn(Bx, Ay), __fmul_rn(By, Ax));
  if ((U < 0.0f || V < 0.0f || W < 0.0f) && (U > 0.0f || V > 0.0f || W > 0.0f)) return;
  const float det = __fadd_rn(__fadd_rn(U, V), W);
  if (det == 0.0f) return;
  const float Az = __fmul_rn(r.Sz, Akz), Bz = __fmul_rn(r.Sz, Bkz), Cz = __fmul_rn(r.Sz, Ckz);
  const float T = __fadd_rn(__fadd_rn(__fmul_rn(U, Az), __fmul_rn(V, Bz)), __fmul_rn(W, Cz));
  const float t = __fdiv_rn(T, det);
  if (!(t > 0.0f && t < INFINITY)) return;
  if (t < best_t || (t == best_t && f < best_f)) {
    best_t = t;
    best_f = f;
  }
}

__device__ __forceinline__ int rc_cell(float x, float lo, float inv, int G) {
  const float c = floorf(__fmul_rn(__fsub_rn(x, lo), inv));
  return (int)fminf(fmaxf(c, 0.0f), (float)(G - 1));   // NaN -> 0
}

// thread per vertex: per-sample box as order-preserving unsigned min [N][3] then max [N][3] (warp-reduced when the warp is one
// sample)
__global__ void __launch_bounds__(256)
rc_bbox_kernel(const float *__restrict__ verts, long long V, const long long *__restrict__ vert_off, int N,
               unsigned *__restrict__ bbox) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const bool ok = i < V;
  const int n = ok ? rc_sample(vert_off, N, i) : -1;
  unsigned u[3] = {0xffffffffu, 0xffffffffu, 0xffffffffu}, w[3] = {0u, 0u, 0u};
  if (ok)
#pragma unroll
    for (int a = 0; a < 3; ++a) u[a] = w[a] = rc_ord(__ldg(verts + 3 * i + a));
  const int n0 = __shfl_sync(0xffffffffu, n, 0);
  if (__all_sync(0xffffffffu, n == n0 || n < 0)) {
    if (n0 < 0) return;
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      const unsigned mn = __reduce_min_sync(0xffffffffu, u[a]), mx = __reduce_max_sync(0xffffffffu, w[a]);
      if ((threadIdx.x & 31) == 0) {
        atomicMin(bbox + 3 * n0 + a, mn);
        atomicMax(bbox + 3 * (N + n0) + a, mx);
      }
    }
  } else if (ok) {
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      atomicMin(bbox + 3 * n + a, u[a]);
      atomicMax(bbox + 3 * (N + n) + a, w[a]);
    }
  }
}

// thread per sample: the padded grid
__global__ void rc_grid_kernel(const unsigned *__restrict__ bbox, const long long *__restrict__ vert_off, int N, int G,
                               RcGrid *__restrict__ grids) {
  const int n = blockIdx.x * blockDim.x + threadIdx.x;
  if (n >= N) return;
  RcGrid g;
  float lo[3], hi[3], emax = 0.0f, mag = 0.0f;
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    lo[a] = rc_unord(bbox[3 * n + a]);
    hi[a] = rc_unord(bbox[3 * (N + n) + a]);
    emax = fmaxf(emax, __fsub_rn(hi[a], lo[a]));
    mag = fmaxf(mag, fmaxf(fabsf(lo[a]), fabsf(hi[a])));
  }
  g.empty = (vert_off[n + 1] == vert_off[n] || !(emax > 0.0f)) ? 1 : 0;
  g.mag = mag;
  g.eta = __fmul_rn(mag, 1.0f / 4096.0f);
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    g.lo[a] = __fsub_rn(lo[a], g.eta);
    g.hi[a] = __fadd_rn(hi[a], g.eta);
    g.cell[a] = __fdiv_rn(__fsub_rn(g.hi[a], g.lo[a]), (float)G);
    g.inv[a] = __fdiv_rn(1.0f, g.cell[a]);
  }
  g.pad_ = 0;
  grids[n] = g;
}

struct RcFace {
  int n, local;
  int c0[3], c1[3];   // inclusive cell range
};

// false: empty sample or degenerate face (binned nowhere)
__device__ __forceinline__ bool rc_face_cells(const float *__restrict__ verts, const int *__restrict__ faces,
                                              const long long *__restrict__ vert_off, const long long *__restrict__ face_off,
                                              const RcGrid *__restrict__ grids, int N, int G, long long f, RcFace &rf,
                                              float (&ext)[3]) {
  rf.n = rc_sample(face_off, N, f);
  rf.local = (int)(f - face_off[rf.n]);
  const RcGrid &g = grids[rf.n];
  if (g.empty) return false;
  const long long vb = vert_off[rf.n];
  float v[3][3];
#pragma unroll
  for (int k = 0; k < 3; ++k) rc_load3(verts + 3 * (vb + __ldg(faces + 3 * f + k)), v[k]);
  if (rc_degenerate(v[0], v[1], v[2])) return false;
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    const float mn = fminf(fminf(v[0][a], v[1][a]), v[2][a]), mx = fmaxf(fmaxf(v[0][a], v[1][a]), v[2][a]);
    ext[a] = __fsub_rn(mx, mn);
    rf.c0[a] = rc_cell(__fsub_rn(mn, g.eta), g.lo[a], g.inv[a], G);
    rf.c1[a] = rc_cell(__fadd_rn(mx, g.eta), g.lo[a], g.inv[a], G);
  }
  return true;
}

// thread per face: per-cell counts, refs[n], largest face extent per axis
__global__ void __launch_bounds__(256)
rc_count_kernel(const float *__restrict__ verts, const int *__restrict__ faces, long long F,
                const long long *__restrict__ vert_off, const long long *__restrict__ face_off, int N, int G,
                const RcGrid *__restrict__ grids, unsigned *__restrict__ cnt, unsigned *__restrict__ maxext,
                unsigned long long *__restrict__ refs) {
  const long long f = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= F) return;
  RcFace rf;
  float ext[3];
  if (!rc_face_cells(verts, faces, vert_off, face_off, grids, N, G, f, rf, ext)) return;
  const size_t G3 = (size_t)G * G * G;
  unsigned *c = cnt + (size_t)rf.n * G3;
  for (int x = rf.c0[0]; x <= rf.c1[0]; ++x)
    for (int y = rf.c0[1]; y <= rf.c1[1]; ++y)
      for (int z = rf.c0[2]; z <= rf.c1[2]; ++z) atomicAdd(c + ((size_t)x * G + y) * G + z, 1u);
#pragma unroll
  for (int a = 0; a < 3; ++a) atomicMax(maxext + 3 * rf.n + a, __float_as_uint(ext[a]));   // ext >= 0: bits are monotone
  const unsigned long long k = (unsigned long long)(rf.c1[0] - rf.c0[0] + 1) * (rf.c1[1] - rf.c0[1] + 1) * (rf.c1[2] - rf.c0[2] + 1);
  atomicAdd(refs + rf.n, k);
}

// one CTA per sample: cur = exclusive prefix of cnt within the sample (each thread owns a contiguous chunk)
__global__ void __launch_bounds__(RC_SCAN_THREADS)
rc_scan_kernel(const unsigned *__restrict__ cnt, unsigned *__restrict__ cur, int G3) {
  __shared__ unsigned s_warp[RC_SCAN_THREADS / 32];
  const size_t base = (size_t)blockIdx.x * G3;
  const int chunk = (G3 + RC_SCAN_THREADS - 1) / RC_SCAN_THREADS;
  const int b = min(G3, threadIdx.x * chunk), e = min(G3, b + chunk);
  unsigned sum = 0;
  for (int i = b; i < e; ++i) sum += cnt[base + i];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  unsigned inc = sum;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const unsigned y = __shfl_up_sync(0xffffffffu, inc, o);
    if (lane >= o) inc += y;
  }
  if (lane == 31) s_warp[warp] = inc;
  __syncthreads();
  if (warp == 0) {
    const unsigned w = s_warp[lane];
    unsigned wi = w;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const unsigned y = __shfl_up_sync(0xffffffffu, wi, o);
      if (lane >= o) wi += y;
    }
    s_warp[lane] = wi - w;
  }
  __syncthreads();
  unsigned run = s_warp[warp] + inc - sum;
  for (int i = b; i < e; ++i) {
    cur[base + i] = run;
    run += cnt[base + i];
  }
}

// thread per face: the face id into every cell of its range; cur ends as the cell's end
__global__ void __launch_bounds__(256)
rc_fill_kernel(const float *__restrict__ verts, const int *__restrict__ faces, long long F,
               const long long *__restrict__ vert_off, const long long *__restrict__ face_off, int N, int G,
               const RcGrid *__restrict__ grids, unsigned *__restrict__ cur, const long long *__restrict__ ref_off,
               int *__restrict__ ref_ids) {
  const long long f = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= F) return;
  RcFace rf;
  float ext[3];
  if (!rc_face_cells(verts, faces, vert_off, face_off, grids, N, G, f, rf, ext)) return;
  const size_t G3 = (size_t)G * G * G;
  unsigned *c = cur + (size_t)rf.n * G3;
  int *ids = ref_ids + ref_off[rf.n];
  for (int x = rf.c0[0]; x <= rf.c1[0]; ++x)
    for (int y = rf.c0[1]; y <= rf.c1[1]; ++y)
      for (int z = rf.c0[2]; z <= rf.c1[2]; ++z) ids[atomicAdd(c + ((size_t)x * G + y) * G + z, 1u)] = rf.local;
}

struct RcMesh {
  const float *verts;
  const int *faces;
  long long vb, fb;   // the sample's first vertex and face
};

__device__ __forceinline__ void rc_test_face(const RcMesh &m, const RcRay &r, int lf, float &best_t, int &best_f) {
  const int *fp = m.faces + 3 * (m.fb + lf);
  float v0[3], v1[3], v2[3];
  rc_load3(m.verts + 3 * (m.vb + __ldg(fp)), v0);
  rc_load3(m.verts + 3 * (m.vb + __ldg(fp + 1)), v1);
  rc_load3(m.verts + 3 * (m.vb + __ldg(fp + 2)), v2);
  rc_test(r, v0, v1, v2, lf, best_t, best_f);
}

// grid (ray blocks, N): thread per (ray, sample)
__global__ void __launch_bounds__(RC_THREADS)
rc_first_hit_kernel(const float *__restrict__ verts, const int *__restrict__ faces, const long long *__restrict__ vert_off,
                    const long long *__restrict__ face_off, int G, const RcGrid *__restrict__ grids,
                    const unsigned *__restrict__ cnt, const unsigned *__restrict__ cur, const unsigned *__restrict__ maxext,
                    const long long *__restrict__ ref_off, const int *__restrict__ ref_ids, const float *__restrict__ origins,
                    const float *__restrict__ dirs, long long R, long long ray_stride, float *__restrict__ t_out,
                    int *__restrict__ face_out) {
  const int n = blockIdx.y;
  const long long ray = (long long)blockIdx.x * RC_THREADS + threadIdx.x;
  if (ray >= R) return;
  float o[3], d[3];
  rc_load3(origins + (size_t)n * ray_stride + 3 * ray, o);
  rc_load3(dirs + (size_t)n * ray_stride + 3 * ray, d);
  float best_t = INFINITY;
  int best_f = -1;
  RcRay r;
  const RcGrid &g = grids[n];
  const RcMesh m{verts, faces, vert_off[n], face_off[n]};
  const int nf = (int)(face_off[n + 1] - m.fb);
  if (nf > 0 && !g.empty && rc_ray_setup(o, d, r)) {
    const float mo = fmaxf(fmaxf(fabsf(o[0]), fabsf(o[1])), fabsf(o[2]));
    if (!(mo <= 64.0f * g.mag)) {
      for (int lf = 0; lf < nf; ++lf) {   // far origin: every face, degenerate ones excluded as in the binning
        const int *fp = faces + 3 * (m.fb + lf);
        float v0[3], v1[3], v2[3];
        rc_load3(verts + 3 * (m.vb + __ldg(fp)), v0);
        rc_load3(verts + 3 * (m.vb + __ldg(fp + 1)), v1);
        rc_load3(verts + 3 * (m.vb + __ldg(fp + 2)), v2);
        if (!rc_degenerate(v0, v1, v2)) rc_test(r, v0, v1, v2, lf, best_t, best_f);
      }
    } else {
      float invd[3], tn = 0.0f, tf = INFINITY;
      bool hit_box = true;
#pragma unroll
      for (int a = 0; a < 3; ++a) {
        invd[a] = __fdiv_rn(1.0f, d[a]);
        if (d[a] != 0.0f) {
          const float t0 = __fmul_rn(__fsub_rn(g.lo[a], o[a]), invd[a]), t1 = __fmul_rn(__fsub_rn(g.hi[a], o[a]), invd[a]);
          tn = fmaxf(tn, fminf(t0, t1));
          tf = fminf(tf, fmaxf(t0, t1));
        } else if (o[a] < g.lo[a] || o[a] > g.hi[a]) {
          hit_box = false;
        }
      }
      if (hit_box && tn <= tf) {
        int idx[3], step[3];
#pragma unroll
        for (int a = 0; a < 3; ++a) {
          idx[a] = rc_cell(__fadd_rn(o[a], __fmul_rn(tn, d[a])), g.lo[a], g.inv[a], G);
          step[a] = d[a] > 0.0f ? 1 : d[a] < 0.0f ? -1 : 0;
        }
        const float E = __fmul_ru(__fmul_ru(__fadd_ru(__uint_as_float(maxext[3 * n + r.kz]), 4.0f * g.eta), fabsf(invd[r.kz])),
                                  1.0f + 1.0f / 1024.0f);
        const size_t G3 = (size_t)G * G * G;
        const unsigned *cn = cnt + (size_t)n * G3, *cu = cur + (size_t)n * G3;
        const int *ids = ref_ids + ref_off[n];
        for (int it = 0; it < 3 * G; ++it) {
          const size_t c = ((size_t)idx[0] * G + idx[1]) * G + idx[2];
          const unsigned end = cu[c], beg = end - cn[c];
          for (unsigned j = beg; j < end; ++j) rc_test_face(m, r, __ldg(ids + j), best_t, best_f);
          float tnext[3];
#pragma unroll
          for (int a = 0; a < 3; ++a) {
            const float plane = __fadd_rn(g.lo[a], __fmul_rn((float)(idx[a] + (step[a] > 0 ? 1 : 0)), g.cell[a]));
            tnext[a] = step[a] ? __fmul_rn(__fsub_rn(plane, o[a]), invd[a]) : INFINITY;
          }
          const int a = tnext[0] <= tnext[1] ? (tnext[0] <= tnext[2] ? 0 : 2) : (tnext[1] <= tnext[2] ? 1 : 2);
          if (best_f >= 0 && __fadd_ru(best_t, E) <= tnext[a]) break;
          idx[a] += step[a];
          if (idx[a] < 0 || idx[a] >= G || step[a] == 0) break;
        }
      }
    }
  }
  t_out[(size_t)n * R + ray] = best_t;
  face_out[(size_t)n * R + ray] = best_f;
}

struct RcLayout {
  size_t bbox, maxext, grids, cnt, cur, total;   // byte offsets into the workspace
};

static size_t rc_align(size_t x) { return (x + 255) & ~(size_t)255; }

static bool rc_layout(int64_t N, int G, RcLayout *L) {
  if (N < 1 || N > 65535 || G < 1 || G > RC_MAX_GRID) return false;
  const size_t G3 = (size_t)G * G * G;
  L->bbox = 0;
  L->maxext = rc_align((size_t)N * 6 * sizeof(unsigned));
  L->grids = L->maxext + rc_align((size_t)N * 3 * sizeof(unsigned));
  L->cnt = L->grids + rc_align((size_t)N * sizeof(RcGrid));
  L->cur = L->cnt + rc_align((size_t)N * G3 * sizeof(unsigned));
  L->total = L->cur + rc_align((size_t)N * G3 * sizeof(unsigned));
  return true;
}

static int rc_check(const char *fn, const float *verts, int64_t V, const int32_t *faces, int64_t F, const int64_t *vert_off,
                    const int64_t *face_off, int64_t N, int G, void *workspace, size_t workspace_bytes, RcLayout *L) {
  GB_REQUIRE(vert_off && face_off && workspace && (verts || V == 0) && (faces || F == 0), GENRE_B200_EINVAL,
             "%s: null pointer", fn);
  GB_REQUIRE(N >= 1 && N <= 65535, GENRE_B200_EINVAL, "%s: N=%lld out of range [1, 65535]", fn, (long long)N);
  GB_REQUIRE(V >= 0 && F >= 0 && V <= ((int64_t)1 << 40) && F <= ((int64_t)1 << 40), GENRE_B200_EINVAL,
             "%s: V=%lld, F=%lld out of range", fn, (long long)V, (long long)F);
  GB_REQUIRE(G >= 1 && G <= RC_MAX_GRID, GENRE_B200_EINVAL, "%s: grid G=%d out of range [1, %d]", fn, G, RC_MAX_GRID);
  rc_layout(N, G, L);
  GB_REQUIRE(workspace_bytes >= L->total && aligned16(workspace), GENRE_B200_EWORKSPACE,
             "%s: workspace too small or misaligned (%zu bytes needed, 16-byte aligned)", fn, L->total);
  return 0;
}

static unsigned rc_blocks(long long n, int threads) { return (unsigned)((n + threads - 1) / threads); }

}  // namespace gb

using namespace gb;

extern "C" size_t genre_b200_raycast_workspace_bytes(int64_t N, int G) {
  RcLayout L{};
  return rc_layout(N, G, &L) ? L.total : 0;
}

extern "C" int genre_b200_raycast_count(const float *verts, int64_t V, const int32_t *faces, int64_t F, const int64_t *vert_off,
                                        const int64_t *face_off, int64_t N, int G, int64_t *refs, void *workspace,
                                        size_t workspace_bytes, void *stream) {
  GB_REQUIRE(refs, GENRE_B200_EINVAL, "raycast_count: null pointer");
  RcLayout L{};
  if (int rc = rc_check("raycast_count", verts, V, faces, F, vert_off, face_off, N, G, workspace, workspace_bytes, &L))
    return rc;
  cudaStream_t st = as_stream(stream);
  char *ws = (char *)workspace;
  cudaError_t e = cudaMemsetAsync(ws + L.bbox, 0xff, (size_t)N * 3 * sizeof(unsigned), st);
  if (e == cudaSuccess) e = cudaMemsetAsync(ws + L.bbox + (size_t)N * 3 * sizeof(unsigned), 0, (size_t)N * 3 * sizeof(unsigned), st);
  if (e == cudaSuccess) e = cudaMemsetAsync(ws + L.maxext, 0, (size_t)N * 3 * sizeof(unsigned), st);
  if (e == cudaSuccess) e = cudaMemsetAsync(ws + L.cnt, 0, L.cur - L.cnt, st);
  if (e == cudaSuccess) e = cudaMemsetAsync(refs, 0, (size_t)N * sizeof(int64_t), st);
  if (e != cudaSuccess) {
    set_error("raycast_count: memset: %s", cudaGetErrorString(e));
    return (int)e;
  }
  unsigned *bbox = (unsigned *)(ws + L.bbox);
  RcGrid *grids = (RcGrid *)(ws + L.grids);
  const long long *vo = (const long long *)vert_off, *fo = (const long long *)face_off;
  if (V > 0) {
    rc_bbox_kernel<<<rc_blocks(V, 256), 256, 0, st>>>(verts, V, vo, (int)N, bbox);
    if (int rc = check_launch("raycast bbox kernel")) return rc;
  }
  rc_grid_kernel<<<rc_blocks(N, 128), 128, 0, st>>>(bbox, vo, (int)N, G, grids);
  if (int rc = check_launch("raycast grid kernel")) return rc;
  if (F > 0) {
    rc_count_kernel<<<rc_blocks(F, 256), 256, 0, st>>>(verts, faces, F, vo, fo, (int)N, G, grids, (unsigned *)(ws + L.cnt),
                                                       (unsigned *)(ws + L.maxext), (unsigned long long *)refs);
    if (int rc = check_launch("raycast count kernel")) return rc;
  }
  return 0;
}

extern "C" int genre_b200_raycast_build(const float *verts, int64_t V, const int32_t *faces, int64_t F, const int64_t *vert_off,
                                        const int64_t *face_off, int64_t N, int G, const int64_t *ref_off, int32_t *ref_ids,
                                        void *workspace, size_t workspace_bytes, void *stream) {
  GB_REQUIRE(ref_off, GENRE_B200_EINVAL, "raycast_build: null pointer");
  RcLayout L{};
  if (int rc = rc_check("raycast_build", verts, V, faces, F, vert_off, face_off, N, G, workspace, workspace_bytes, &L))
    return rc;
  cudaStream_t st = as_stream(stream);
  char *ws = (char *)workspace;
  rc_scan_kernel<<<(unsigned)N, RC_SCAN_THREADS, 0, st>>>((const unsigned *)(ws + L.cnt), (unsigned *)(ws + L.cur), G * G * G);
  if (int rc = check_launch("raycast scan kernel")) return rc;
  if (F > 0) {
    GB_REQUIRE(ref_ids, GENRE_B200_EINVAL, "raycast_build: null pointer");
    rc_fill_kernel<<<rc_blocks(F, 256), 256, 0, st>>>(verts, faces, F, (const long long *)vert_off, (const long long *)face_off,
                                                      (int)N, G, (const RcGrid *)(ws + L.grids), (unsigned *)(ws + L.cur),
                                                      (const long long *)ref_off, ref_ids);
    if (int rc = check_launch("raycast fill kernel")) return rc;
  }
  return 0;
}

extern "C" int genre_b200_raycast_first_hit(const float *verts, int64_t V, const int32_t *faces, int64_t F,
                                            const int64_t *vert_off, const int64_t *face_off, int64_t N, int G,
                                            const int64_t *ref_off, const int32_t *ref_ids, const float *origins,
                                            const float *dirs, int64_t R, int64_t ray_batch_stride, float *t, int32_t *face,
                                            void *workspace, size_t workspace_bytes, void *stream) {
  GB_REQUIRE(ref_off && origins && dirs && t && face, GENRE_B200_EINVAL, "raycast_first_hit: null pointer");
  RcLayout L{};
  if (int rc = rc_check("raycast_first_hit", verts, V, faces, F, vert_off, face_off, N, G, workspace, workspace_bytes, &L))
    return rc;
  GB_REQUIRE(R >= 1 && R <= ((int64_t)1 << 36), GENRE_B200_EINVAL, "raycast_first_hit: R=%lld out of range", (long long)R);
  GB_REQUIRE(ray_batch_stride == 0 || ray_batch_stride == 3 * R, GENRE_B200_EINVAL,
             "raycast_first_hit: ray_batch_stride must be 0 (shared rays) or 3*R, got %lld", (long long)ray_batch_stride);
  cudaStream_t st = as_stream(stream);
  char *ws = (char *)workspace;
  rc_first_hit_kernel<<<dim3(rc_blocks(R, RC_THREADS), (unsigned)N), RC_THREADS, 0, st>>>(
      verts, faces, (const long long *)vert_off, (const long long *)face_off, G, (const RcGrid *)(ws + L.grids),
      (const unsigned *)(ws + L.cnt), (const unsigned *)(ws + L.cur), (const unsigned *)(ws + L.maxext),
      (const long long *)ref_off, ref_ids, origins, dirs, R, ray_batch_stride, t, face);
  return check_launch("raycast first-hit kernel");
}
