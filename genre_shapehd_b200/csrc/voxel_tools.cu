// voxel_tools.cu — batched voxel-grid utilities: the reference's per-sample CPU toolkit util/util_voxel.py (fill :167-238,
// transform / transform_by_matrix :107-161, find_bound :31-52, downsample :10-28, translate :64-90) for batches resident on
// the device.
//
// Conventions (as isosurface.cu and raycast.cu): dense fp32 volumes [N, D, H, W], every dimension in [2, 512],
// 1 <= N <= 65535; the caller owns every buffer and workspace; the library allocates nothing, never synchronises, and
// reports argument errors before any launch.
//
// fill       exterior fill by union-find connected-component labelling of the EMPTY voxels (v > threshold is occupied, so NaN
//            is empty).  Each sample has its own label space in the workspace: node 0 is the OUTSIDE, a virtual empty shell
//            around the grid, and voxel p (linear index (i*H + j)*W + k) is node p + 1.  Every union links the larger root
//            under the smaller one, so the outside is always the root of its component.
//              local : 8^3 tiles, one thread per voxel; union-find in shared memory over the tile's empty voxels and their
//                      in-tile forward neighbours (3 directions for 6-connectivity, 13 for 26), then every voxel stores the
//                      global node of its tile root (occupied voxels store FILL_OCC).
//              merge : the forward neighbours across tile faces (an edge or corner neighbour only when no face step towards
//                      it is empty), and every empty voxel on the grid's border with node 0: atomic-CAS union on the global
//                      labels, path halving on the way to the roots.
//              final : out = occupied || root != 0.
//            Three passes whatever the shape: no loop runs "until nothing changes", so a maze costs about what a sphere
//            costs.  The result is a set membership (is the voxel's component the outside's?), so it is the same whatever
//            order the unions happen in: deterministic.
// transform  one thread per output voxel; fp64 coordinates in the order the header states, scipy's RegularGridInterpolator
//            'linear' sum (corners in C order, weight ((w0*w1)*w2), value * weight added to 0 in turn) in fp64, one rounding
//            to fp32 (or the threshold compared in fp64).
// stats      a grid-stride pass per sample over pool^3 cells: the box of a > th_a and, with b, the pooled IoU counts (pooled
//            values compared in fp64, as the reference thresholds its fp64 downsample output); block
//            reductions, then one integer atomic per block and quantity.  Init and finalize kernels around it.
// downsample / translate   one thread per output voxel.
#include "common.cuh"

namespace gb {

constexpr int VT_MAX_DIM = 512;
constexpr int VT_THREADS = 256;
constexpr int FILL_TILE = 8;
constexpr int FILL_THREADS = FILL_TILE * FILL_TILE * FILL_TILE;
constexpr unsigned FILL_OCC = 0xffffffffu;

// the 13 forward neighbour offsets (di, dj, dk) > 0 lexicographically; the first 3 are the face neighbours
__device__ constexpr int kFwd[13][3] = {{0, 0, 1}, {0, 1, 0}, {1, 0, 0},   {0, 1, -1}, {0, 1, 1},  {1, -1, -1}, {1, -1, 0},
                                        {1, -1, 1}, {1, 0, -1}, {1, 0, 1}, {1, 1, -1}, {1, 1, 0}, {1, 1, 1}};

// ---- fill ---------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ int s_find(volatile int *s, int x) {
  int p;
  while ((p = s[x]) != x) x = p;
  return x;
}

__device__ __forceinline__ void s_unite(volatile int *s, int a, int b) {
  a = s_find(s, a);
  b = s_find(s, b);
  while (a != b) {
    if (a > b) {
      const int t = a;
      a = b;
      b = t;
    }
    const int old = atomicCAS((int *)&s[b], b, a);
    if (old == b) return;
    b = s_find(s, old);   // b was linked meanwhile: continue from its new root
    a = s_find(s, a);
  }
}

// root of node x; halves the path on the way.  Only a non-root's entry is written, and always with one of its ancestors,
// which a concurrent union (a CAS that expects a root) never races with.
__device__ __forceinline__ unsigned g_find(unsigned *L, unsigned x) {
  while (true) {
    const unsigned p = __ldcg(L + x);
    if (p == x) return x;
    const unsigned gp = __ldcg(L + p);
    if (gp == p) return p;
    __stcg(L + x, gp);
    x = gp;
  }
}

__device__ __forceinline__ void g_unite(unsigned *L, unsigned a, unsigned b) {
  a = g_find(L, a);
  b = g_find(L, b);
  while (a != b) {
    if (a > b) {
      const unsigned t = a;
      a = b;
      b = t;
    }
    const unsigned old = atomicCAS(L + b, b, a);
    if (old == b) return;
    b = g_find(L, old);
    a = g_find(L, a);
  }
}

struct FillTile {
  int i, j, k;      // voxel coordinates
  int tz, ty, tx;   // coordinates inside the tile
  bool valid;
};

__device__ __forceinline__ FillTile fill_tile(int D, int H, int W) {
  const int tk = (W + FILL_TILE - 1) / FILL_TILE, tj = (H + FILL_TILE - 1) / FILL_TILE;
  const int b = blockIdx.x;
  FillTile t;
  t.tx = threadIdx.x & 7;
  t.ty = (threadIdx.x >> 3) & 7;
  t.tz = threadIdx.x >> 6;
  t.k = (b % tk) * FILL_TILE + t.tx;
  t.j = ((b / tk) % tj) * FILL_TILE + t.ty;
  t.i = (b / (tk * tj)) * FILL_TILE + t.tz;
  t.valid = t.i < D && t.j < H && t.k < W;
  return t;
}

// grid (tiles, N)
__global__ void __launch_bounds__(FILL_THREADS)
fill_local_kernel(const float *__restrict__ vol, int D, int H, int W, float threshold, int ndir, unsigned *__restrict__ labels) {
  __shared__ int s[FILL_THREADS];
  const int n = blockIdx.y;
  const long long P = (long long)D * H * W;
  const FillTile t = fill_tile(D, H, W);
  const long long p = ((long long)t.i * H + t.j) * W + t.k;
  const int me = threadIdx.x;
  const bool empty = t.valid && !(__ldg(vol + (size_t)n * P + p) > threshold);
  s[me] = empty ? me : -1;
  __syncthreads();
  if (empty) {
    for (int d = 0; d < ndir; ++d) {
      const int z = t.tz + kFwd[d][0], y = t.ty + kFwd[d][1], x = t.tx + kFwd[d][2];
      if (z >= FILL_TILE || y < 0 || y >= FILL_TILE || x < 0 || x >= FILL_TILE) continue;
      const int q = (z * FILL_TILE + y) * FILL_TILE + x;
      if (s[q] >= 0) s_unite(s, me, q);
    }
  }
  __syncthreads();
  unsigned *L = labels + (size_t)n * (P + 1);
  if (blockIdx.x == 0 && me == 0) L[0] = 0u;   // the outside
  if (!t.valid) return;
  unsigned lab = FILL_OCC;
  if (empty) {
    const int r = s_find(s, me);
    const long long rp = ((long long)(t.i - t.tz + (r >> 6)) * H + (t.j - t.ty + ((r >> 3) & 7))) * W + (t.k - t.tx + (r & 7));
    lab = (unsigned)(rp + 1);
  }
  L[p + 1] = lab;
}

__global__ void __launch_bounds__(FILL_THREADS)
fill_merge_kernel(int D, int H, int W, int ndir, unsigned *__restrict__ labels) {
  const int n = blockIdx.y;
  const long long P = (long long)D * H * W;
  const FillTile t = fill_tile(D, H, W);
  if (!t.valid) return;
  unsigned *L = labels + (size_t)n * (P + 1);
  const long long p = ((long long)t.i * H + t.j) * W + t.k;
  if (__ldcg(L + p + 1) == FILL_OCC) return;
  if (t.i == 0 || t.j == 0 || t.k == 0 || t.i == D - 1 || t.j == H - 1 || t.k == W - 1) g_unite(L, 0u, (unsigned)(p + 1));
  for (int d = 0; d < ndir; ++d) {
    const int z = t.tz + kFwd[d][0], y = t.ty + kFwd[d][1], x = t.tx + kFwd[d][2];
    if (z < FILL_TILE && y >= 0 && y < FILL_TILE && x >= 0 && x < FILL_TILE) continue;   // done by the local pass
    const int i = t.i + kFwd[d][0], j = t.j + kFwd[d][1], k = t.k + kFwd[d][2];
    if (i >= D || j < 0 || j >= H || k < 0 || k >= W) continue;
    const long long q = ((long long)i * H + j) * W + k;
    if (__ldcg(L + q + 1) == FILL_OCC) continue;
    // an edge or corner neighbour is skipped when a face step from p towards it is empty: p joins that voxel m, and m joins
    // q through a pair with fewer non-zero offsets, which is united or skipped by the same rule, down to face pairs
    bool covered = false;
    const long long stride[3] = {(long long)H * W, W, 1};
    for (int a = 0; a < 3 && d >= 3; ++a)
      if (kFwd[d][a] != 0) covered |= __ldcg(L + p + kFwd[d][a] * stride[a] + 1) != FILL_OCC;
    if (!covered) g_unite(L, (unsigned)(p + 1), (unsigned)(q + 1));
  }
}

// grid (ceil(P / VT_THREADS), N)
__global__ void __launch_bounds__(VT_THREADS)
fill_final_kernel(long long P, unsigned *__restrict__ labels, unsigned char *__restrict__ out) {
  const int n = blockIdx.y;
  const long long p = (long long)blockIdx.x * VT_THREADS + threadIdx.x;
  if (p >= P) return;
  unsigned *L = labels + (size_t)n * (P + 1);
  const unsigned lab = __ldcg(L + p + 1);
  out[(size_t)n * P + p] = (unsigned char)(lab == FILL_OCC || g_find(L, (unsigned)(p + 1)) != 0u);
}

// ---- transform ----------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(VT_THREADS)
transform_kernel(const float *__restrict__ vol, int D, int H, int W, const double *__restrict__ params, unsigned flags,
                 double lo, double hi, double threshold, void *__restrict__ out) {
  const int n = blockIdx.y;
  const long long P = (long long)D * H * W;
  const long long p = (long long)blockIdx.x * VT_THREADS + threadIdx.x;
  if (p >= P) return;
  const int k = (int)(p % W), j = (int)((p / W) % H), i = (int)(p / ((long long)H * W));
  const int dim[3] = {D, H, W};
  const double c[3] = {0.5 * D, 0.5 * H, 0.5 * W};   // exact
  const double u[3] = {__dsub_rn((double)i, c[0]), __dsub_rn((double)j, c[1]), __dsub_rn((double)k, c[2])};
  const double *m = params + 12 * (size_t)n;
  int i0[3];
  double y[3];
  bool inside = true;
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    double x = __dadd_rn(__dmul_rn(__ldg(m + 3 * a), u[0]), __dmul_rn(__ldg(m + 3 * a + 1), u[1]));
    x = __dadd_rn(x, __dmul_rn(__ldg(m + 3 * a + 2), u[2]));
    x = __dadd_rn(__dadd_rn(x, c[a]), __ldg(m + 9 + a));
    inside &= x >= 0.0 && x <= (double)(dim[a] - 1);   // NaN: outside
    i0[a] = inside ? min((int)floor(x), dim[a] - 2) : 0;
    y[a] = __dsub_rn(x, (double)i0[a]);
  }
  double val = 0.0;
  if (inside) {
    const float *v = vol + (size_t)n * P + ((long long)i0[0] * H + i0[1]) * W + i0[2];
#pragma unroll
    for (int corner = 0; corner < 8; ++corner) {
      const int b0 = corner >> 2, b1 = (corner >> 1) & 1, b2 = corner & 1;
      const double w0 = b0 ? y[0] : __dsub_rn(1.0, y[0]);
      const double w1 = b1 ? y[1] : __dsub_rn(1.0, y[1]);
      const double w2 = b2 ? y[2] : __dsub_rn(1.0, y[2]);
      const double w = __dmul_rn(__dmul_rn(w0, w1), w2);
      const float f = __ldg(v + (b0 * (long long)H + b1) * W + b2);
      val = __dadd_rn(val, __dmul_rn((double)f, w));
    }
  }
  if (flags & GENRE_B200_VOXEL_CLAMP) val = val < lo ? lo : (val > hi ? hi : val);   // np.clip: NaN stays NaN
  if (flags & GENRE_B200_VOXEL_THRESHOLD)
    ((unsigned char *)out)[(size_t)n * P + p] = (unsigned char)(val > threshold);
  else
    ((float *)out)[(size_t)n * P + p] = __double2float_rn(val);
}

// ---- stats --------------------------------------------------------------------------------------------------------------
constexpr int STATS_CELLS_PER_THREAD = 4;

__global__ void stats_init_kernel(int N, int *__restrict__ bounds, unsigned long long *__restrict__ counts) {
  const int n = blockIdx.x * blockDim.x + threadIdx.x;
  if (n >= N) return;
  if (bounds) {
    for (int a = 0; a < 3; ++a) {
      bounds[6 * n + a] = 0x7fffffff;
      bounds[6 * n + 3 + a] = -1;
    }
  }
  if (counts)
    for (int a = 0; a < 3; ++a) counts[3 * n + a] = 0ull;
}

// empty samples get zeros; the upper bound becomes exclusive
__global__ void stats_finalize_kernel(int N, int *__restrict__ bounds) {
  const int n = blockIdx.x * blockDim.x + threadIdx.x;
  if (n >= N) return;
  const bool empty = bounds[6 * n + 3] < 0;
  for (int a = 0; a < 3; ++a) {
    bounds[6 * n + a] = empty ? 0 : bounds[6 * n + a];
    bounds[6 * n + 3 + a] = empty ? 0 : bounds[6 * n + 3 + a] + 1;
  }
}

__device__ __forceinline__ float pool_max(float m, float v) { return (v > m || v != v) ? v : m; }   // NaN propagates, as np.max

// grid (blocks, N): a grid-stride loop over the sample's ceil(D/pool) x ceil(H/pool) x ceil(W/pool) cells
__global__ void __launch_bounds__(VT_THREADS)
stats_kernel(const float *__restrict__ a, const float *__restrict__ b, int D, int H, int W, int pool, int mean, double th_a,
             double th_b, int *__restrict__ bounds, unsigned long long *__restrict__ counts) {
  // fp32 voxels compare with the thresholds rounded to fp32 (as numpy and torch compare an fp32 grid with a Python float);
  // pooled values, as the reference's fp64 downsample output, compare in fp64
  const float fa = __double2float_rn(th_a), fb = __double2float_rn(th_b);
  const int n = blockIdx.y;
  const long long P = (long long)D * H * W;
  const int cD = (D + pool - 1) / pool, cH = (H + pool - 1) / pool, cW = (W + pool - 1) / pool;
  const int fD = D / pool, fH = H / pool, fW = W / pool;   // complete cells (the remainder is not pooled)
  const long long cells = (long long)cD * cH * cW;
  const float *va = a + (size_t)n * P;
  const float *vb = b ? b + (size_t)n * P : nullptr;
  const double cell = (double)pool * pool * pool;
  int lo[3] = {0x7fffffff, 0x7fffffff, 0x7fffffff}, hi[3] = {-1, -1, -1};
  unsigned ca = 0, cb = 0, cab = 0;
  for (long long c = (long long)blockIdx.x * VT_THREADS + threadIdx.x; c < cells; c += (long long)gridDim.x * VT_THREADS) {
    const int ck = (int)(c % cW), cj = (int)((c / cW) % cH), ci = (int)(c / ((long long)cW * cH));
    const bool whole = vb && ci < fD && cj < fH && ck < fW;
    float ma = -INFINITY, mb = -INFINITY;
    double sa = 0.0, sb = 0.0;
    for (int di = 0; di < pool; ++di) {
      const int i = ci * pool + di;
      if (i >= D) break;
      for (int dj = 0; dj < pool; ++dj) {
        const int j = cj * pool + dj;
        if (j >= H) break;
        for (int dk = 0; dk < pool; ++dk) {
          const int k = ck * pool + dk;
          if (k >= W) break;
          const long long q = ((long long)i * H + j) * W + k;
          const float x = __ldg(va + q);
          if (bounds && x > fa) {
            lo[0] = min(lo[0], i), lo[1] = min(lo[1], j), lo[2] = min(lo[2], k);
            hi[0] = max(hi[0], i), hi[1] = max(hi[1], j), hi[2] = max(hi[2], k);
          }
          if (whole) {
            const float z = __ldg(vb + q);
            if (mean) {
              sa = __dadd_rn(sa, (double)x);
              sb = __dadd_rn(sb, (double)z);
            } else {
              ma = pool_max(ma, x);
              mb = pool_max(mb, z);
            }
          }
        }
      }
    }
    if (whole) {
      bool ia, ib;
      if (pool == 1) {
        ia = (mean ? __double2float_rn(sa) : ma) > fa;   // the voxels themselves: sa = 0 + x is exact
        ib = (mean ? __double2float_rn(sb) : mb) > fb;
      } else {
        ia = (mean ? __ddiv_rn(sa, cell) : (double)ma) > th_a;
        ib = (mean ? __ddiv_rn(sb, cell) : (double)mb) > th_b;
      }
      ca += ia;
      cb += ib;
      cab += ia && ib;
    }
  }
  // block reduction: warps, then warp 0; one atomic per block and quantity
  __shared__ int s_b[VT_THREADS / 32][6];
  __shared__ unsigned s_c[VT_THREADS / 32][3];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  int r[6];
  unsigned rc[3];
  for (int x = 0; x < 3; ++x) {
    r[x] = __reduce_min_sync(0xffffffffu, lo[x]);
    r[3 + x] = __reduce_max_sync(0xffffffffu, hi[x]);
  }
  rc[0] = __reduce_add_sync(0xffffffffu, ca);
  rc[1] = __reduce_add_sync(0xffffffffu, cb);
  rc[2] = __reduce_add_sync(0xffffffffu, cab);
  if (lane == 0) {
    for (int x = 0; x < 6; ++x) s_b[warp][x] = r[x];
    for (int x = 0; x < 3; ++x) s_c[warp][x] = rc[x];
  }
  __syncthreads();
  if (threadIdx.x != 0) return;
  for (int w = 1; w < VT_THREADS / 32; ++w) {
    for (int x = 0; x < 3; ++x) {
      r[x] = min(r[x], s_b[w][x]);
      r[3 + x] = max(r[3 + x], s_b[w][3 + x]);
      rc[x] += s_c[w][x];
    }
  }
  if (bounds && r[3] >= 0) {
    for (int x = 0; x < 3; ++x) {
      atomicMin(bounds + 6 * n + x, r[x]);
      atomicMax(bounds + 6 * n + 3 + x, r[3 + x]);
    }
  }
  if (counts)
    for (int x = 0; x < 3; ++x)
      if (rc[x]) atomicAdd(counts + 3 * n + x, (unsigned long long)rc[x]);
}

// ---- downsample / translate ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(VT_THREADS)
downsample_kernel(const float *__restrict__ vol, int R, int times, int use_max, float *__restrict__ out) {
  const int n = blockIdx.y;
  const int d = R / times;
  const long long Q = (long long)d * d * d;
  const long long o = (long long)blockIdx.x * VT_THREADS + threadIdx.x;
  if (o >= Q) return;
  const int z = (int)(o % d), y = (int)((o / d) % d), x = (int)(o / ((long long)d * d));
  const float *v = vol + (size_t)n * R * R * R;
  float m = -INFINITY;
  double s = 0.0;
  for (int di = 0; di < times; ++di)
    for (int dj = 0; dj < times; ++dj)
      for (int dk = 0; dk < times; ++dk) {
        const float f = __ldg(v + ((long long)(x * times + di) * R + (y * times + dj)) * R + (z * times + dk));
        if (use_max) m = pool_max(m, f);
        else s = __dadd_rn(s, (double)f);
      }
  out[(size_t)n * Q + o] = use_max ? m : __double2float_rn(__ddiv_rn(s, (double)times * times * times));
}

__global__ void __launch_bounds__(VT_THREADS)
translate_kernel(const float *__restrict__ vol, int D, int H, int W, const int *__restrict__ bounds,
                 const int *__restrict__ offsets, float *__restrict__ out) {
  const int n = blockIdx.y;
  const long long P = (long long)D * H * W;
  const long long p = (long long)blockIdx.x * VT_THREADS + threadIdx.x;
  if (p >= P) return;
  const int pos[3] = {(int)(p / ((long long)H * W)), (int)((p / W) % H), (int)(p % W)};
  const int dim[3] = {D, H, W};
  bool in = true;
  int src[3];
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    src[a] = pos[a] - __ldg(offsets + 3 * n + a);
    in &= src[a] >= __ldg(bounds + 6 * n + a) && src[a] < __ldg(bounds + 6 * n + 3 + a) && src[a] >= 0 && src[a] < dim[a];
  }
  out[(size_t)n * P + p] = in ? __ldg(vol + (size_t)n * P + ((long long)src[0] * H + src[1]) * W + src[2]) : 0.0f;
}

// ---- host side ----------------------------------------------------------------------------------------------------------
static bool vt_shape_ok(int64_t N, int D, int H, int W) {
  return N >= 1 && N <= 65535 && D >= 2 && H >= 2 && W >= 2 && D <= VT_MAX_DIM && H <= VT_MAX_DIM && W <= VT_MAX_DIM;
}

static int vt_check(const char *fn, int64_t N, int D, int H, int W) {
  GB_REQUIRE(N >= 1 && N <= 65535, GENRE_B200_EINVAL, "%s: N=%lld out of range [1, 65535]", fn, (long long)N);
  GB_REQUIRE(vt_shape_ok(N, D, H, W), GENRE_B200_EINVAL, "%s: volume %dx%dx%d unsupported (every dimension in [2, %d])", fn,
             D, H, W, VT_MAX_DIM);
  return 0;
}

static unsigned vt_blocks(long long P) { return (unsigned)((P + VT_THREADS - 1) / VT_THREADS); }

}  // namespace gb

using namespace gb;

extern "C" size_t genre_b200_voxel_fill_workspace_bytes(int64_t N, int D, int H, int W) {
  if (!vt_shape_ok(N, D, H, W)) return 0;
  return (size_t)N * ((size_t)D * H * W + 1) * sizeof(unsigned);
}

extern "C" int genre_b200_voxel_fill(const float *vol, int64_t N, int D, int H, int W, float threshold, int connectivity,
                                     uint8_t *out, void *workspace, size_t workspace_bytes, void *stream) {
  GB_REQUIRE(vol && out && workspace, GENRE_B200_EINVAL, "voxel_fill: null pointer");
  if (int rc = vt_check("voxel_fill", N, D, H, W)) return rc;
  GB_REQUIRE(connectivity == 6 || connectivity == 26, GENRE_B200_EINVAL, "voxel_fill: connectivity %d (6 or 26)", connectivity);
  GB_REQUIRE(threshold == threshold, GENRE_B200_EINVAL, "voxel_fill: threshold is NaN");
  const size_t need = genre_b200_voxel_fill_workspace_bytes(N, D, H, W);
  GB_REQUIRE(workspace_bytes >= need && aligned16(workspace), GENRE_B200_EWORKSPACE,
             "voxel_fill: workspace too small or misaligned (%zu bytes needed, 16-byte aligned)", need);
  cudaStream_t st = as_stream(stream);
  const int ndir = connectivity == 6 ? 3 : 13;
  const unsigned tiles = (unsigned)(((D + FILL_TILE - 1) / FILL_TILE) * ((H + FILL_TILE - 1) / FILL_TILE) *
                                    ((W + FILL_TILE - 1) / FILL_TILE));
  unsigned *labels = (unsigned *)workspace;
  fill_local_kernel<<<dim3(tiles, (unsigned)N), FILL_THREADS, 0, st>>>(vol, D, H, W, threshold, ndir, labels);
  if (int rc = check_launch("voxel_fill local kernel")) return rc;
  fill_merge_kernel<<<dim3(tiles, (unsigned)N), FILL_THREADS, 0, st>>>(D, H, W, ndir, labels);
  if (int rc = check_launch("voxel_fill merge kernel")) return rc;
  const long long P = (long long)D * H * W;
  fill_final_kernel<<<dim3(vt_blocks(P), (unsigned)N), VT_THREADS, 0, st>>>(P, labels, out);
  return check_launch("voxel_fill final kernel");
}

extern "C" int genre_b200_voxel_transform(const float *vol, int64_t N, int D, int H, int W, const double *params,
                                          unsigned flags, double clamp_lo, double clamp_hi, double threshold, void *out,
                                          void *stream) {
  GB_REQUIRE(vol && params && out, GENRE_B200_EINVAL, "voxel_transform: null pointer");
  if (int rc = vt_check("voxel_transform", N, D, H, W)) return rc;
  GB_REQUIRE((flags & ~(GENRE_B200_VOXEL_CLAMP | GENRE_B200_VOXEL_THRESHOLD)) == 0, GENRE_B200_EINVAL,
             "voxel_transform: unknown flags 0x%x", flags);
  GB_REQUIRE(!(flags & GENRE_B200_VOXEL_CLAMP) || clamp_lo <= clamp_hi, GENRE_B200_EINVAL,
             "voxel_transform: clamp range [%g, %g] is empty or NaN", clamp_lo, clamp_hi);
  GB_REQUIRE(!(flags & GENRE_B200_VOXEL_THRESHOLD) || threshold == threshold, GENRE_B200_EINVAL,
             "voxel_transform: threshold is NaN");
  const long long P = (long long)D * H * W;
  transform_kernel<<<dim3(vt_blocks(P), (unsigned)N), VT_THREADS, 0, as_stream(stream)>>>(vol, D, H, W, params, flags,
                                                                                          clamp_lo, clamp_hi, threshold, out);
  return check_launch("voxel_transform kernel");
}

extern "C" int genre_b200_voxel_stats(const float *a, const float *b, int64_t N, int D, int H, int W, int pool, int pool_mode,
                                      double th_a, double th_b, int32_t *bounds, int64_t *counts, void *stream) {
  GB_REQUIRE(a && (bounds || counts), GENRE_B200_EINVAL, "voxel_stats: null pointer (a, and bounds or counts, are needed)");
  GB_REQUIRE(!counts || b, GENRE_B200_EINVAL, "voxel_stats: null pointer (counts need b)");
  if (int rc = vt_check("voxel_stats", N, D, H, W)) return rc;
  GB_REQUIRE(pool >= 1 && pool <= D && pool <= H && pool <= W, GENRE_B200_EINVAL,
             "voxel_stats: pool %d out of range [1, min(D, H, W)]", pool);
  GB_REQUIRE(pool_mode == GENRE_B200_POOL_MAX || pool_mode == GENRE_B200_POOL_MEAN, GENRE_B200_EINVAL,
             "voxel_stats: pool_mode %d unknown", pool_mode);
  GB_REQUIRE(th_a == th_a && th_b == th_b, GENRE_B200_EINVAL, "voxel_stats: threshold is NaN");
  cudaStream_t st = as_stream(stream);
  const unsigned nb = (unsigned)((N + 255) / 256);
  stats_init_kernel<<<nb, 256, 0, st>>>((int)N, bounds, (unsigned long long *)counts);
  if (int rc = check_launch("voxel_stats init kernel")) return rc;
  const long long cells = (long long)((D + pool - 1) / pool) * ((H + pool - 1) / pool) * ((W + pool - 1) / pool);
  const unsigned blocks = (unsigned)((cells + VT_THREADS * STATS_CELLS_PER_THREAD - 1) / (VT_THREADS * STATS_CELLS_PER_THREAD));
  stats_kernel<<<dim3(blocks, (unsigned)N), VT_THREADS, 0, st>>>(a, b, D, H, W, pool, pool_mode == GENRE_B200_POOL_MEAN, th_a,
                                                                 th_b, bounds, (unsigned long long *)counts);
  if (int rc = check_launch("voxel_stats kernel")) return rc;
  if (!bounds) return 0;
  stats_finalize_kernel<<<nb, 256, 0, st>>>((int)N, bounds);
  return check_launch("voxel_stats finalize kernel");
}

extern "C" int genre_b200_voxel_downsample(const float *vol, int64_t N, int R, int times, int use_max, float *out,
                                           void *stream) {
  GB_REQUIRE(vol && out, GENRE_B200_EINVAL, "voxel_downsample: null pointer");
  if (int rc = vt_check("voxel_downsample", N, R, R, R)) return rc;
  GB_REQUIRE(times >= 1 && times <= R, GENRE_B200_EINVAL, "voxel_downsample: times %d out of range [1, R=%d]", times, R);
  const int d = R / times;
  downsample_kernel<<<dim3(vt_blocks((long long)d * d * d), (unsigned)N), VT_THREADS, 0, as_stream(stream)>>>(
      vol, R, times, use_max ? 1 : 0, out);
  return check_launch("voxel_downsample kernel");
}

extern "C" int genre_b200_voxel_translate(const float *vol, int64_t N, int D, int H, int W, const int32_t *bounds,
                                          const int32_t *offsets, float *out, void *stream) {
  GB_REQUIRE(vol && bounds && offsets && out, GENRE_B200_EINVAL, "voxel_translate: null pointer");
  if (int rc = vt_check("voxel_translate", N, D, H, W)) return rc;
  const long long P = (long long)D * H * W;
  translate_kernel<<<dim3(vt_blocks(P), (unsigned)N), VT_THREADS, 0, as_stream(stream)>>>(vol, D, H, W, bounds, offsets, out);
  return check_launch("voxel_translate kernel");
}
