/* isosurface_oracle.c — scalar C restatement of the marching-cubes contract of genre_b200_isosurface_* (include/genre_b200.h,
 * genre_shapehd_b200/csrc/isosurface.cu).  TEST INFRASTRUCTURE: the GPU tests require the device output to equal this one bit
 * for bit.  Built with -ffp-contract=off: every float operation below rounds once, as __fadd_rn / __fmul_rn / __fdiv_rn do.
 *
 * The cube tables are not written out here: they are derived from the rules at first use, so a slip in the kernel's
 * hand-written tables shows up as a mismatch.
 *   corners   c = 4*o0 + 2*o1 + o2 for the offsets (o0, o1, o2) of the cell's lowest point
 *   edge id   an edge along axis a whose offsets along the other axes b < c are ob, oc: 4a + 2*ob + oc
 *   faces     the face normal to axis f at side s, its corners walked counter-clockwise seen from outside the cell
 */
#include <stdint.h>
#include <stdlib.h>

#define EXPORT __attribute__((visibility("default")))

static int face_corner[6][4], face_edge[6][4], edge_lo[12], edge_hi[12];
static int tables_ready;

static void other_axes(int a, int *b, int *c) {
  *b = a == 0 ? 1 : 0;
  *c = a == 2 ? 1 : 2;
}

static int corner(const int o[3]) { return 4 * o[0] + 2 * o[1] + o[2]; }

static int edge_between(int c1, int c2) {
  int o[3] = {(c1 >> 2) & 1, (c1 >> 1) & 1, c1 & 1}, a = 0, b, c;
  for (int x = 0; x < 3; ++x)
    if (((c1 ^ c2) >> (2 - x)) & 1) a = x;
  other_axes(a, &b, &c);
  return 4 * a + 2 * o[b] + o[c];
}

static void init_tables(void) {
  /* e_b x e_c = sgn[f] * e_f for the two other axes b < c; the outward normal of side s is (2s - 1) * e_f.  The walk
   * (0,0) (1,0) (1,1) (0,1) in (o_b, o_c) is counter-clockwise about e_b x e_c. */
  static const int sgn[3] = {1, -1, 1};
  static const int ccw[4][2] = {{0, 0}, {1, 0}, {1, 1}, {0, 1}};
  for (int f = 0; f < 3; ++f)
    for (int s = 0; s < 2; ++s) {
      const int face = 2 * f + s, fwd = sgn[f] * (2 * s - 1) > 0;
      int b, c;
      other_axes(f, &b, &c);
      for (int i = 0; i < 4; ++i) {
        const int *st = ccw[fwd ? i : (4 - i) & 3];
        int o[3];
        o[f] = s;
        o[b] = st[0];
        o[c] = st[1];
        face_corner[face][i] = corner(o);
      }
      for (int i = 0; i < 4; ++i) face_edge[face][i] = edge_between(face_corner[face][i], face_corner[face][(i + 1) & 3]);
    }
  for (int e = 0; e < 12; ++e) {
    const int a = e / 4;
    int b, c, o[3];
    other_axes(a, &b, &c);
    o[b] = (e >> 1) & 1;
    o[c] = e & 1;
    o[a] = 0;
    edge_lo[e] = corner(o);
    o[a] = 1;
    edge_hi[e] = corner(o);
  }
  tables_ready = 1;
}

/* the cell's directed links (next[e], -1 where edge e has no crossing); returns the crossing mask */
static unsigned cell_links(const float v[8], float level, int next[12]) {
  int in[8];
  unsigned cross = 0;
  for (int o = 0; o < 8; ++o) in[o] = v[o] > level;
  for (int e = 0; e < 12; ++e) {
    next[e] = -1;
    if (in[edge_lo[e]] != in[edge_hi[e]]) cross |= 1u << e;
  }
  for (int f = 0; f < 6; ++f) {
    int q[4];
    for (int i = 0; i < 4; ++i) q[i] = in[face_corner[f][i]];
    int joined = 0;
    if (q[0] == q[2] && q[1] == q[3] && q[0] != q[1]) {
      /* asymptotic decider: the inside corners a, d are joined iff fl(a' d') > fl(b' c'), x' = fl(x - level) */
      const float x0 = v[face_corner[f][0]] - level, x1 = v[face_corner[f][1]] - level;
      const float x2 = v[face_corner[f][2]] - level, x3 = v[face_corner[f][3]] - level;
      const float p02 = x0 * x2, p13 = x1 * x3;
      joined = q[0] ? p02 > p13 : p13 > p02;
    }
    for (int i = 0; i < 4; ++i) {
      if (q[i] || !q[(i + 1) & 3]) continue;  /* not an entry */
      int want = joined ? 2 : 1;
      for (int s = 1; s < 4; ++s) {
        const int j = (i + s) & 3;
        if (q[j] && !q[(j + 1) & 3] && --want == 0) {
          next[face_edge[f][i]] = face_edge[f][j];
          break;
        }
      }
    }
  }
  return cross;
}

/* bit 2*f + s for each of the two cell faces (normal to axis f, side s) local edge e lies on */
static int edge_faces(int e) {
  int b, c;
  other_axes(e / 4, &b, &c);
  return 1 << (2 * b + ((e >> 1) & 1)) | 1 << (2 * c + (e & 1));
}

/* position of the fan apex in a loop: the first vertex that shares no cell face with any loop vertex other than its two
 * neighbours (so that no fan diagonal lies in a face the neighbouring cell may also triangulate), else the first vertex */
static int fan_apex(const int *loop, int m) {
  for (int s = 0; s < m; ++s) {
    int ok = 1;
    for (int t = 2; t + 1 < m && ok; ++t) ok = !(edge_faces(loop[s]) & edge_faces(loop[(s + t) % m]));
    if (ok) return s;
  }
  return 0;
}

/* (i, j, k) offsets of the low end of local edge e */
static void edge_owner(int e, int d[3]) {
  const int lo = edge_lo[e];
  d[0] = (lo >> 2) & 1;
  d[1] = (lo >> 1) & 1;
  d[2] = lo & 1;
}

static void load_cell(const float *vol, int H, int W, int i, int j, int k, float v[8]) {
  for (int o = 0; o < 8; ++o)
    v[o] = vol[((int64_t)(i + ((o >> 2) & 1)) * H + (j + ((o >> 1) & 1))) * W + (k + (o & 1))];
}

static int point_mask(const float *vol, int D, int H, int W, int i, int j, int k, float level) {
  const int64_t p = ((int64_t)i * H + j) * W + k;
  const int in0 = vol[p] > level;
  int m = 0;
  if (i + 1 < D && (vol[p + (int64_t)H * W] > level) != in0) m |= 1;
  if (j + 1 < H && (vol[p + W] > level) != in0) m |= 2;
  if (k + 1 < W && (vol[p + 1] > level) != in0) m |= 4;
  return m;
}

/* one volume [D, H, W]: vertex and face counts */
EXPORT void oracle_isosurface_count(const float *vol, int D, int H, int W, float level, int64_t *nverts, int64_t *nfaces) {
  if (!tables_ready) init_tables();
  int64_t nv = 0, nf = 0;
  for (int i = 0; i < D; ++i)
    for (int j = 0; j < H; ++j)
      for (int k = 0; k < W; ++k) {
        const int m = point_mask(vol, D, H, W, i, j, k, level);
        nv += (m & 1) + ((m >> 1) & 1) + ((m >> 2) & 1);
        if (i + 1 == D || j + 1 == H || k + 1 == W) continue;
        float v[8];
        int next[12], seen = 0;
        load_cell(vol, H, W, i, j, k, v);
        const unsigned cross = cell_links(v, level, next);
        for (int e = 0; e < 12; ++e) {
          if (!((cross >> e) & 1) || ((seen >> e) & 1)) continue;
          int m_loop = 0, x = e;
          do {
            seen |= 1 << x;
            ++m_loop;
            x = next[x];
          } while (x != e);
          nf += m_loop - 2;
        }
      }
  *nverts = nv;
  *nfaces = nf;
}

/* one volume: verts [V, 3], faces [F, 3] in the contract's order (V, F from oracle_isosurface_count) */
EXPORT int oracle_isosurface(const float *vol, int D, int H, int W, float level, const float *spacing, const float *shift,
                             float *verts, int32_t *faces) {
  if (!tables_ready) init_tables();
  const int64_t P = (int64_t)D * H * W;
  int32_t *base = (int32_t *)malloc(sizeof(int32_t) * P);
  unsigned char *mask = (unsigned char *)malloc(P);
  if (!base || !mask) {
    free(base);
    free(mask);
    return -1;
  }
  int32_t nv = 0;
  for (int i = 0; i < D; ++i)
    for (int j = 0; j < H; ++j)
      for (int k = 0; k < W; ++k) {
        const int64_t p = ((int64_t)i * H + j) * W + k;
        const int m = point_mask(vol, D, H, W, i, j, k, level);
        const int pos[3] = {i, j, k};
        const int64_t step[3] = {(int64_t)H * W, W, 1};
        base[p] = nv;
        mask[p] = (unsigned char)m;
        for (int a = 0; a < 3; ++a) {
          if (!((m >> a) & 1)) continue;
          const float v0 = vol[p], v1 = vol[p + step[a]];
          const float t = (level - v0) / (v1 - v0);
          for (int b = 0; b < 3; ++b) {
            const float x = b == a ? (float)pos[b] + t : (float)pos[b];
            verts[3 * (int64_t)nv + b] = x * spacing[b] - shift[b];
          }
          ++nv;
        }
      }
  int64_t nf = 0;
  for (int i = 0; i + 1 < D; ++i)
    for (int j = 0; j + 1 < H; ++j)
      for (int k = 0; k + 1 < W; ++k) {
        float v[8];
        int next[12], id[12], seen = 0;
        load_cell(vol, H, W, i, j, k, v);
        const unsigned cross = cell_links(v, level, next);
        if (!cross) continue;
        for (int e = 0; e < 12; ++e) {
          if (!((cross >> e) & 1)) continue;
          int d[3];
          edge_owner(e, d);
          const int64_t q = ((int64_t)(i + d[0]) * H + (j + d[1])) * W + (k + d[2]);
          int rank = 0;
          for (int a = 0; a < e / 4; ++a) rank += (mask[q] >> a) & 1;
          id[e] = base[q] + rank;
        }
        for (int e = 0; e < 12; ++e) {
          if (!((cross >> e) & 1) || ((seen >> e) & 1)) continue;
          int loop[12], m = 0, x = e;
          do {
            seen |= 1 << x;
            loop[m++] = x;
            x = next[x];
          } while (x != e);
          const int s = fan_apex(loop, m);
          for (int t = 1; t + 1 < m; ++t) {
            faces[3 * nf + 0] = id[loop[s]];
            faces[3 * nf + 1] = id[loop[(s + t) % m]];
            faces[3 * nf + 2] = id[loop[(s + t + 1) % m]];
            ++nf;
          }
        }
      }
  free(base);
  free(mask);
  return 0;
}
