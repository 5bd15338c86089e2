// isosurface.cu — batched marching cubes on the GPU (SURVEY 8f-3): the iso-surface the reference extracts from every predicted
// voxel grid with skimage.measure.marching_cubes_lewiner (visualize/visualizer.py:160, util/util_sph.py:47).
//
// Contract (include/genre_b200.h states it too; oracle_iso/isosurface_oracle.c restates it in scalar C, bit for bit):
//   input   N dense fp32 volumes [D, H, W], 2 <= D, H, W <= 512.  A grid point is INSIDE iff v > level (NaN is outside).
//   vertices one per grid edge whose ends lie on different sides.  Point p owns its edges to p+e0, p+e1, p+e2; for the edge from
//           p (value v0) to q (value v1) along axis a:  t = fl(fl(level - v0) / fl(v1 - v0)),
//           x_a = fl(fl(fl(p_a + t) * spacing_a) - shift_a),  x_b = fl(fl(p_b * spacing_b) - shift_b) for the other axes.
//           Every step rounds once (__fadd_rn / __fmul_rn / __fdiv_rn; no FMA contraction).  Axis 0 is the array's first axis.
//           Non-finite voxels take the same formula: a finite p and an infinite q give t = +-0 (the vertex is p); a NaN end
//           or an infinite p gives a NaN t and x_a.
//           Order: by sample, grid point linear index (i*H + j)*W + k, then axis.
//   cells   per-cell segment linking, no case table.  On each of the cell's 6 faces, walked counter-clockwise as seen from
//           outside the cell, an edge is an ENTRY (outside -> inside corner) or an EXIT (inside -> outside); every entry is linked
//           to the next exit along the walk.  A face whose inside corners a, d lie on a diagonal (b, c outside) is decided by
//           the asymptotic decider: with x' = fl(x - level), the inside corners are joined through the face iff
//           fl(a'*d') > fl(b'*c') (a tie keeps them apart), and then each entry links to the SECOND exit.  The rule sees only
//           the face's four values, so the two cells sharing a face agree: the mesh is crack-free.  Interior ambiguities
//           (Lewiner's tunnel tests) are not resolved.
//           Every crossing edge has one incoming and one outgoing link, so the links form closed loops of m >= 3 edges;
//           a loop gives the fan (v_s, v_{s+i}, v_{s+i+1}), i = 1 .. m-2 (indices mod m): m - 2 triangles, at most 10 per cell.
//           The apex v_s is the first loop vertex that shares no cell face with a loop vertex other than its two
//           neighbours, else v_0: a fan diagonal inside a face could coincide with one of the neighbouring cell.  Loops
//           through the same face twice with no such vertex (they need ambiguous faces) can still leave a mesh edge with
//           more than two triangles; every edge is always used equally often in both directions.
//   local edge id  an edge along axis a whose offsets along the other axes b < c are ob, oc: 4a + 2*ob + oc.
//   faces   loops by smallest edge id, each walked from that edge (v_0) along its links.  Triangles are counter-clockwise seen from
//           outside (<= level): normals point away from the > level region.  Order: by sample, cell linear index (the index of
//           its lowest corner), loop, fan position.  int32 indices into the sample's own vertex block.
//
// Kernels (tile = 256 consecutive grid points of one sample; a thread per point):
//   count : the point's 3-bit crossing mask and the triangle count of the cell it is the lowest corner of -> one byte per point
//           in the workspace ("code" = mask | ntri << 3); the CTA sums vertices and triangles into its tile's packed total.
//   scan  : one CTA per sample turns the tile totals into exclusive offsets and writes counts[n] = {vertices, faces}.
//   vertex: block scan of popc(mask) + tile offset = the point's vertex base, kept in the workspace; writes the coordinates.
//   face  : block scan of ntri + tile offset; re-links the cell's nonempty faces and writes the fans.  The vertex of local edge
//           e is base[owner] + popc(mask[owner] & ((1 << axis) - 1)).
// The volume is read once by count (neighbour reads hit L1/L2) and again only around crossings by the emit kernels.
//
// Backward (genre_b200_isosurface_backward): the gradient of the vertex coordinates with respect to the volume.  Only x_a of
// the vertex on the edge p -> q = p + e_a depends on the volume, through t; with g = grad_verts[v][a] (the other two
// components are ignored), in fp64 from the fp32 operands, one rounding per operation, in this order:
//           d = v1 - v0,  k = (g * s_a) / (d * d),  c0 = k * (level - v1) goes to p,  c1 = k * (v0 - level) goes to q.
//           An edge with a non-finite end contributes 0.
//   grad  : a gather, thread per grid point on the count kernel's tiling: the point sums its own crossing edges a = 0, 1, 2
//           (their c0), then the incoming edges from p - e_a, a = 0, 1, 2 (their c1), in fp64 from 0, rounded once to fp32.
//           The vertex of edge (owner, a) is vbase[owner] + popc(code[owner] & 7 & ((1 << a) - 1)), read only where the mask
//           bit is set (vbase is written only there).  No atomics: deterministic.
#include "common.cuh"

namespace gb {

constexpr int ISO_THREADS = 256;
constexpr int ISO_SCAN_THREADS = 1024;
constexpr int ISO_MAX_DIM = 512;

// the 6 cell faces: corners (c = 4*o0 + 2*o1 + o2) counter-clockwise seen from outside, and the local edge id from corner
// [i] to corner [i+1]
__device__ constexpr int kFaceCorner[6][4] = {{0, 1, 3, 2}, {4, 6, 7, 5}, {0, 4, 5, 1}, {2, 3, 7, 6}, {0, 2, 6, 4}, {1, 5, 7, 3}};
__device__ constexpr int kFaceEdge[6][4] = {{8, 5, 9, 4}, {6, 11, 7, 10}, {0, 10, 1, 8}, {9, 3, 11, 2}, {4, 2, 6, 0}, {1, 7, 3, 5}};
// corners at the two ends of each local edge (low end first)
__device__ constexpr int kEdgeLo[12] = {0, 1, 2, 3, 0, 1, 4, 5, 0, 2, 4, 6};
__device__ constexpr int kEdgeHi[12] = {4, 5, 6, 7, 2, 3, 6, 7, 1, 3, 5, 7};

// exclusive block scan; *total gets the block's sum.  Every thread of the block must call it.
template <int NT, typename T>
__device__ __forceinline__ T iso_block_scan(T x, T *total) {
  __shared__ T s_warp[NT / 32];
  __shared__ T s_total;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  T inc = x;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const T y = __shfl_up_sync(0xffffffffu, inc, o);
    if (lane >= o) inc += y;
  }
  if (lane == 31) s_warp[warp] = inc;
  __syncthreads();
  if (warp == 0) {
    const T w = lane < NT / 32 ? s_warp[lane] : T(0);
    T wi = w;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const T y = __shfl_up_sync(0xffffffffu, wi, o);
      if (lane >= o) wi += y;
    }
    if (lane < NT / 32) s_warp[lane] = wi - w;
    if (lane == NT / 32 - 1) s_total = wi;
  }
  __syncthreads();
  const T excl = s_warp[warp] + inc - x;
  *total = s_total;
  __syncthreads();  // the shared slots are reused by the next call
  return excl;
}

// directed links of the cell's crossing edges, 4 bits per local edge (next edge of its loop); `in` = inside mask of the 8 corners
__device__ __forceinline__ unsigned long long iso_links(const float (&v)[8], unsigned in, float level) {
  unsigned long long links = 0;
#pragma unroll
  for (int f = 0; f < 6; ++f) {
    unsigned q = 0;  // inside bits in walk order
#pragma unroll
    for (int i = 0; i < 4; ++i) q |= ((in >> kFaceCorner[f][i]) & 1u) << i;
    if (q == 0u || q == 15u) continue;
    bool joined = false;
    if (q == 5u || q == 10u) {
      const float x0 = __fsub_rn(v[kFaceCorner[f][0]], level), x1 = __fsub_rn(v[kFaceCorner[f][1]], level);
      const float x2 = __fsub_rn(v[kFaceCorner[f][2]], level), x3 = __fsub_rn(v[kFaceCorner[f][3]], level);
      const float p02 = __fmul_rn(x0, x2), p13 = __fmul_rn(x1, x3);
      joined = q == 5u ? p02 > p13 : p13 > p02;
    }
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const bool entry = !((q >> i) & 1u) && ((q >> ((i + 1) & 3)) & 1u);
      if (!entry) continue;
      int skip = joined ? 1 : 0, target = -1;
#pragma unroll
      for (int s = 1; s < 4; ++s) {
        const int j = (i + s) & 3;
        const bool exit = ((q >> j) & 1u) && !((q >> ((j + 1) & 3)) & 1u);
        if (exit && target < 0) {
          if (skip == 0) target = kFaceEdge[f][j];
          else --skip;
        }
      }
      links |= (unsigned long long)target << (4 * kFaceEdge[f][i]);
    }
  }
  return links;
}

__device__ __forceinline__ unsigned iso_crossings(unsigned in) {
  unsigned cross = 0;
#pragma unroll
  for (int e = 0; e < 12; ++e) cross |= (((in >> kEdgeLo[e]) ^ (in >> kEdgeHi[e])) & 1u) << e;
  return cross;
}

__device__ __forceinline__ int iso_next(unsigned long long links, int e) { return (int)((links >> (4 * e)) & 15u); }

// bit 2*f + s for the two cell faces (normal to axis f, side s) local edge e lies on
__device__ __forceinline__ unsigned iso_edge_faces(int e) {
  const int a = e >> 2, b = a == 0 ? 1 : 0, c = a == 2 ? 1 : 2;
  return 1u << (2 * b + ((e >> 1) & 1)) | 1u << (2 * c + (e & 1));
}

// fan apex: the first loop position whose vertex shares no cell face with a loop vertex other than its two neighbours, else 0
__device__ __forceinline__ int iso_fan_apex(unsigned long long loop, int m) {
  for (int s = 0; s < m; ++s) {
    const unsigned fs = iso_edge_faces((int)((loop >> (4 * s)) & 15u));
    bool ok = true;
    for (int t = 2; t + 1 < m; ++t) ok &= !(fs & iso_edge_faces((int)((loop >> (4 * ((s + t) % m))) & 15u)));
    if (ok) return s;
  }
  return 0;
}

// the 8 corners of the cell whose lowest corner is p (all in range)
__device__ __forceinline__ void iso_load_cell(const float *__restrict__ v, long long p, int HW, int W, float (&c)[8]) {
#pragma unroll
  for (int o = 0; o < 8; ++o) c[o] = __ldg(v + p + ((o >> 2) & 1) * (long long)HW + ((o >> 1) & 1) * W + (o & 1));
}

__device__ __forceinline__ unsigned iso_inside(const float (&c)[8], float level) {
  unsigned in = 0;
#pragma unroll
  for (int o = 0; o < 8; ++o) in |= (c[o] > level ? 1u : 0u) << o;
  return in;
}

// grid (tiles, N): codes[n][p] and the tile's packed total (vertices << 32 | triangles)
__global__ void __launch_bounds__(ISO_THREADS)
iso_count_kernel(const float *__restrict__ vol, int D, int H, int W, float level, unsigned char *__restrict__ codes,
                 unsigned long long *__restrict__ tiles_ws, int tiles) {
  const int n = blockIdx.y;
  const long long P = (long long)D * H * W;
  const int HW = H * W;
  const long long p = (long long)blockIdx.x * ISO_THREADS + threadIdx.x;
  const float *v = vol + (size_t)n * P;
  unsigned nv = 0, nt = 0;
  if (p < P) {
    const int k = (int)(p % W), j = (int)((p / W) % H), i = (int)(p / HW);
    const bool ci = i + 1 < D, cj = j + 1 < H, ck = k + 1 < W;
    const float v0 = __ldg(v + p);
    const bool in0 = v0 > level;
    unsigned mask = 0;
    if (ci) mask |= (unsigned)((__ldg(v + p + HW) > level) != in0) << 0;
    if (cj) mask |= (unsigned)((__ldg(v + p + W) > level) != in0) << 1;
    if (ck) mask |= (unsigned)((__ldg(v + p + 1) > level) != in0) << 2;
    if (ci && cj && ck) {
      float c[8];
      iso_load_cell(v, p, HW, W, c);
      const unsigned in = iso_inside(c, level);
      if (in != 0u && in != 255u) {
        const unsigned long long links = iso_links(c, in, level);
        const unsigned cross = iso_crossings(in);
        unsigned left = cross, loops = 0;
        while (left) {
          const int s = __ffs(left) - 1;
          int e = s;
          do {
            left &= ~(1u << e);
            e = iso_next(links, e);
          } while (e != s);
          ++loops;
        }
        nt = __popc(cross) - 2 * loops;
      }
    }
    nv = __popc(mask);
    codes[(size_t)n * P + p] = (unsigned char)(mask | nt << 3);
  }
  unsigned long long tot;
  iso_block_scan<ISO_THREADS, unsigned long long>((unsigned long long)nv << 32 | nt, &tot);
  if (threadIdx.x == 0) tiles_ws[(size_t)n * tiles + blockIdx.x] = tot;
}

// one CTA per sample: packed tile totals -> exclusive packed offsets; counts[n] = {vertices, faces}.  Per-sample totals fit
// in 32 bits (3*D*H*W and 10*(D-1)(H-1)(W-1) at 512^3), so the low half never carries into the high half.
__global__ void __launch_bounds__(ISO_SCAN_THREADS)
iso_scan_kernel(unsigned long long *__restrict__ tiles_ws, int tiles, long long *__restrict__ counts) {
  const int n = blockIdx.x;
  unsigned long long *t = tiles_ws + (size_t)n * tiles;
  unsigned long long carry = 0;
  for (int base = 0; base < tiles; base += ISO_SCAN_THREADS) {
    const int idx = base + threadIdx.x;
    const unsigned long long x = idx < tiles ? t[idx] : 0ull;
    unsigned long long tot;
    const unsigned long long excl = iso_block_scan<ISO_SCAN_THREADS, unsigned long long>(x, &tot);
    if (idx < tiles) t[idx] = carry + excl;
    carry += tot;
  }
  if (threadIdx.x == 0) {
    counts[2 * n] = (long long)(carry >> 32);
    counts[2 * n + 1] = (long long)(carry & 0xffffffffull);
  }
}

__global__ void __launch_bounds__(ISO_THREADS)
iso_vertex_kernel(const float *__restrict__ vol, int D, int H, int W, float level, float3 spacing, float3 shift,
                  const unsigned char *__restrict__ codes, const unsigned long long *__restrict__ tiles_ws, int tiles,
                  unsigned *__restrict__ vbase, const long long *__restrict__ vert_off, float *__restrict__ verts) {
  const int n = blockIdx.y;
  const long long P = (long long)D * H * W;
  const int HW = H * W;
  const long long p = (long long)blockIdx.x * ISO_THREADS + threadIdx.x;
  const unsigned mask = p < P ? codes[(size_t)n * P + p] & 7u : 0u;
  unsigned tot;
  const unsigned excl = iso_block_scan<ISO_THREADS, unsigned>(__popc(mask), &tot);
  if (!mask) return;
  const unsigned base = (unsigned)(tiles_ws[(size_t)n * tiles + blockIdx.x] >> 32) + excl;
  vbase[(size_t)n * P + p] = base;
  const float *v = vol + (size_t)n * P;
  const int k = (int)(p % W), j = (int)((p / W) % H), i = (int)(p / HW);
  const float pos[3] = {(float)i, (float)j, (float)k};
  const float sp[3] = {spacing.x, spacing.y, spacing.z}, sh[3] = {shift.x, shift.y, shift.z};
  const long long stride[3] = {HW, W, 1};
  float grid[3];
#pragma unroll
  for (int b = 0; b < 3; ++b) grid[b] = __fsub_rn(__fmul_rn(pos[b], sp[b]), sh[b]);
  const float v0 = __ldg(v + p);
  float *out = verts + 3 * (size_t)(vert_off[n] + base);
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    if (!((mask >> a) & 1u)) continue;
    const float v1 = __ldg(v + p + stride[a]);
    const float t = __fdiv_rn(__fsub_rn(level, v0), __fsub_rn(v1, v0));
    const float x = __fsub_rn(__fmul_rn(__fadd_rn(pos[a], t), sp[a]), sh[a]);
#pragma unroll
    for (int b = 0; b < 3; ++b) out[b] = b == a ? x : grid[b];
    out += 3;
  }
}

__global__ void __launch_bounds__(ISO_THREADS)
iso_face_kernel(const float *__restrict__ vol, int D, int H, int W, float level, const unsigned char *__restrict__ codes,
                const unsigned long long *__restrict__ tiles_ws, int tiles, const unsigned *__restrict__ vbase,
                const long long *__restrict__ face_off, int *__restrict__ faces) {
  const int n = blockIdx.y;
  const long long P = (long long)D * H * W;
  const int HW = H * W;
  const long long p = (long long)blockIdx.x * ISO_THREADS + threadIdx.x;
  const unsigned nt = p < P ? codes[(size_t)n * P + p] >> 3 : 0u;
  unsigned tot;
  const unsigned excl = iso_block_scan<ISO_THREADS, unsigned>(nt, &tot);
  if (!nt) return;
  const unsigned fbase = (unsigned)(tiles_ws[(size_t)n * tiles + blockIdx.x] & 0xffffffffull) + excl;
  const float *v = vol + (size_t)n * P;
  const unsigned char *cd = codes + (size_t)n * P;
  const unsigned *vb = vbase + (size_t)n * P;
  float c[8];
  iso_load_cell(v, p, HW, W, c);
  const unsigned in = iso_inside(c, level);
  const unsigned long long links = iso_links(c, in, level);
  const unsigned cross = iso_crossings(in);
  // vertex id of local edge e: owner = p + offsets of the edge's low corner; rank of axis e/4 in the owner's mask
  auto vid = [&](int e) -> int {
    const int lo = e < 4 ? (e & 3) : e < 8 ? (((e >> 1) & 1) << 2 | (e & 1)) : (((e >> 1) & 1) << 2 | (e & 1) << 1);
    const long long q = p + ((lo >> 2) & 1) * (long long)HW + ((lo >> 1) & 1) * W + (lo & 1);
    return (int)(vb[q] + __popc(cd[q] & 7u & ((1u << (e >> 2)) - 1u)));
  };
  int *out = faces + 3 * (size_t)(face_off[n] + fbase);
  unsigned left = cross;
  while (left) {
    const int s0 = __ffs(left) - 1;
    unsigned long long loop = 0;  // the loop's edges in walk order, 4 bits each
    int m = 0, e = s0;
    do {
      left &= ~(1u << e);
      loop |= (unsigned long long)e << (4 * m++);
      e = iso_next(links, e);
    } while (e != s0);
    const int s = iso_fan_apex(loop, m);
    auto at = [&](int t) { return (int)((loop >> (4 * ((s + t) % m))) & 15u); };
    const int a = vid(at(0));
    int b = vid(at(1));
    for (int t = 2; t < m; ++t) {
      const int d = vid(at(t));
      out[0] = a;
      out[1] = b;
      out[2] = d;
      out += 3;
      b = d;
    }
  }
}

// x is finite (not NaN, not +-inf)
__device__ __forceinline__ bool iso_finite(float x) { return fabsf(x) <= 3.402823466e38f; }

// the contribution of edge (owner, a) to one of its ends: c0 (to the owner, lo = true) or c1 (to the far end)
__device__ __forceinline__ double iso_edge_grad(float v0, float v1, float level, float g, float s, bool lo) {
  if (!iso_finite(v0) || !iso_finite(v1)) return 0.0;
  const double d = __dsub_rn((double)v1, (double)v0);
  const double k = __ddiv_rn(__dmul_rn((double)g, (double)s), __dmul_rn(d, d));
  return lo ? __dmul_rn(k, __dsub_rn((double)level, (double)v1)) : __dmul_rn(k, __dsub_rn((double)v0, (double)level));
}

// grid (tiles, N): thread per grid point; grad_vol fully written
__global__ void __launch_bounds__(ISO_THREADS)
iso_grad_kernel(const float *__restrict__ vol, int D, int H, int W, float level, float3 spacing,
                const unsigned char *__restrict__ codes, const unsigned *__restrict__ vbase,
                const long long *__restrict__ vert_off, const float *__restrict__ grad_verts, float *__restrict__ grad_vol) {
  const int n = blockIdx.y;
  const long long P = (long long)D * H * W;
  const int HW = H * W;
  const long long p = (long long)blockIdx.x * ISO_THREADS + threadIdx.x;
  if (p >= P) return;
  const float *v = vol + (size_t)n * P;
  const unsigned char *cd = codes + (size_t)n * P;
  const unsigned *vb = vbase + (size_t)n * P;
  const float *gv = grad_verts + 3 * (size_t)__ldg(vert_off + n);
  const int k = (int)(p % W), j = (int)((p / W) % H), i = (int)(p / HW);
  const float vp = __ldg(v + p);
  double sum = 0.0;
  const unsigned own = cd[p] & 7u;
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    const long long stride = a == 0 ? HW : a == 1 ? W : 1;
    const float s = a == 0 ? spacing.x : a == 1 ? spacing.y : spacing.z;
    if ((own >> a) & 1u) {
      const unsigned vid = vb[p] + __popc(own & ((1u << a) - 1u));
      sum = __dadd_rn(sum, iso_edge_grad(vp, __ldg(v + p + stride), level, __ldg(gv + 3 * (size_t)vid + a), s, true));
    }
  }
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    const long long stride = a == 0 ? HW : a == 1 ? W : 1;
    const float s = a == 0 ? spacing.x : a == 1 ? spacing.y : spacing.z;
    if ((a == 0 ? i : a == 1 ? j : k) > 0) {
      const long long o = p - stride;
      const unsigned m = cd[o] & 7u;
      if ((m >> a) & 1u) {
        const unsigned vid = vb[o] + __popc(m & ((1u << a) - 1u));
        sum = __dadd_rn(sum, iso_edge_grad(__ldg(v + o), vp, level, __ldg(gv + 3 * (size_t)vid + a), s, false));
      }
    }
  }
  grad_vol[(size_t)n * P + p] = __double2float_rn(sum);
}

struct IsoLayout {
  long long P;
  int tiles;
  size_t codes, vbase, tiles_ws, total;   // byte offsets into the workspace
};

static size_t iso_align(size_t x) { return (x + 255) & ~(size_t)255; }

static bool iso_layout(int64_t N, int D, int H, int W, IsoLayout *L) {
  if (N < 1 || N > 65535 || D < 2 || H < 2 || W < 2 || D > ISO_MAX_DIM || H > ISO_MAX_DIM || W > ISO_MAX_DIM) return false;
  L->P = (long long)D * H * W;
  L->tiles = (int)((L->P + ISO_THREADS - 1) / ISO_THREADS);
  L->codes = 0;
  L->vbase = iso_align((size_t)N * L->P);
  L->tiles_ws = L->vbase + iso_align((size_t)N * L->P * sizeof(unsigned));
  L->total = L->tiles_ws + iso_align((size_t)N * L->tiles * sizeof(unsigned long long));
  return true;
}

static int iso_check(const char *fn, const float *vol, int64_t N, int D, int H, int W, float level, void *workspace,
                     size_t workspace_bytes, IsoLayout *L) {
  GB_REQUIRE(vol && workspace, GENRE_B200_EINVAL, "%s: null pointer", fn);
  GB_REQUIRE(N >= 1 && N <= 65535, GENRE_B200_EINVAL, "%s: N=%lld out of range [1, 65535]", fn, (long long)N);
  GB_REQUIRE(D >= 2 && H >= 2 && W >= 2 && D <= ISO_MAX_DIM && H <= ISO_MAX_DIM && W <= ISO_MAX_DIM, GENRE_B200_EINVAL,
             "%s: volume %dx%dx%d unsupported (every dimension in [2, %d])", fn, D, H, W, ISO_MAX_DIM);
  GB_REQUIRE(level == level, GENRE_B200_EINVAL, "%s: level is NaN", fn);
  iso_layout(N, D, H, W, L);
  GB_REQUIRE(workspace_bytes >= L->total && aligned16(workspace), GENRE_B200_EWORKSPACE,
             "%s: workspace too small or misaligned (%zu bytes needed, 16-byte aligned)", fn, L->total);
  return 0;
}

}  // namespace gb

using namespace gb;

extern "C" size_t genre_b200_isosurface_workspace_bytes(int64_t N, int D, int H, int W) {
  IsoLayout L;
  return iso_layout(N, D, H, W, &L) ? L.total : 0;
}

extern "C" int genre_b200_isosurface_count(const float *vol, int64_t N, int D, int H, int W, float level, int64_t *counts,
                                           void *workspace, size_t workspace_bytes, void *stream) {
  GB_REQUIRE(counts, GENRE_B200_EINVAL, "isosurface_count: null pointer");
  IsoLayout L;
  if (int rc = iso_check("isosurface_count", vol, N, D, H, W, level, workspace, workspace_bytes, &L)) return rc;
  cudaStream_t st = as_stream(stream);
  char *ws = (char *)workspace;
  unsigned long long *tws = (unsigned long long *)(ws + L.tiles_ws);
  iso_count_kernel<<<dim3((unsigned)L.tiles, (unsigned)N), ISO_THREADS, 0, st>>>(vol, D, H, W, level,
                                                                                  (unsigned char *)(ws + L.codes), tws, L.tiles);
  if (int rc = check_launch("isosurface count kernel")) return rc;
  iso_scan_kernel<<<(unsigned)N, ISO_SCAN_THREADS, 0, st>>>(tws, L.tiles, (long long *)counts);
  return check_launch("isosurface scan kernel");
}

extern "C" int genre_b200_isosurface_emit(const float *vol, int64_t N, int D, int H, int W, float level, float sx, float sy,
                                          float sz, float shx, float shy, float shz, const int64_t *vert_off,
                                          const int64_t *face_off, float *verts, int32_t *faces, void *workspace,
                                          size_t workspace_bytes, void *stream) {
  GB_REQUIRE(vert_off && face_off && verts && faces, GENRE_B200_EINVAL, "isosurface_emit: null pointer");
  IsoLayout L;
  if (int rc = iso_check("isosurface_emit", vol, N, D, H, W, level, workspace, workspace_bytes, &L)) return rc;
  cudaStream_t st = as_stream(stream);
  char *ws = (char *)workspace;
  const unsigned char *codes = (const unsigned char *)(ws + L.codes);
  unsigned *vbase = (unsigned *)(ws + L.vbase);
  const unsigned long long *tws = (const unsigned long long *)(ws + L.tiles_ws);
  const dim3 grid((unsigned)L.tiles, (unsigned)N);
  iso_vertex_kernel<<<grid, ISO_THREADS, 0, st>>>(vol, D, H, W, level, make_float3(sx, sy, sz), make_float3(shx, shy, shz),
                                                  codes, tws, L.tiles, vbase, (const long long *)vert_off, verts);
  if (int rc = check_launch("isosurface vertex kernel")) return rc;
  iso_face_kernel<<<grid, ISO_THREADS, 0, st>>>(vol, D, H, W, level, codes, tws, L.tiles, vbase, (const long long *)face_off,
                                                faces);
  return check_launch("isosurface face kernel");
}

extern "C" int genre_b200_isosurface_backward(const float *vol, int64_t N, int D, int H, int W, float level, float sx, float sy,
                                              float sz, const int64_t *vert_off, const float *grad_verts, float *grad_vol,
                                              void *workspace, size_t workspace_bytes, void *stream) {
  GB_REQUIRE(vert_off && grad_verts && grad_vol, GENRE_B200_EINVAL, "isosurface_backward: null pointer");
  IsoLayout L;
  if (int rc = iso_check("isosurface_backward", vol, N, D, H, W, level, workspace, workspace_bytes, &L)) return rc;
  const char *ws = (const char *)workspace;
  iso_grad_kernel<<<dim3((unsigned)L.tiles, (unsigned)N), ISO_THREADS, 0, as_stream(stream)>>>(
      vol, D, H, W, level, make_float3(sx, sy, sz), (const unsigned char *)(ws + L.codes), (const unsigned *)(ws + L.vbase),
      (const long long *)vert_off, grad_verts, grad_vol);
  return check_launch("isosurface backward kernel");
}
