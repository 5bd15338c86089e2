/* raycast_oracle.c — scalar C restatement of the ray-casting contract (include/genre_b200.h, csrc/raycast.cu header):
 * for every ray, a loop over every face of its mesh.  TEST INFRASTRUCTURE ONLY.  Built with -ffp-contract=off, so every
 * float operation below rounds once, as the kernel's __f*_rn intrinsics do. */
#include <math.h>
#include <stdint.h>

#define ORACLE_API __attribute__((visibility("default")))

static int degenerate(const float *a, const float *b, const float *c) {
  float e1[3], e2[3];
  for (int k = 0; k < 3; ++k) {
    e1[k] = b[k] - a[k];
    e2[k] = c[k] - a[k];
  }
  float nx = e1[1] * e2[2] - e1[2] * e2[1];
  float ny = e1[2] * e2[0] - e1[0] * e2[2];
  float nz = e1[0] * e2[1] - e1[1] * e2[0];
  return nx == 0.0f && ny == 0.0f && nz == 0.0f;
}

/* verts [V,3], faces [F,3] (indices into verts), rays o, d [R,3] -> t [R] (+inf on a miss), face [R] (-1 on a miss) */
ORACLE_API void oracle_raycast(const float *verts, const int32_t *faces, int64_t F, const float *orig, const float *dirs,
                               int64_t R, float *t_out, int32_t *f_out) {
  for (int64_t r = 0; r < R; ++r) {
    const float *o = orig + 3 * r, *d = dirs + 3 * r;
    float best_t = INFINITY;
    int32_t best_f = -1;
    int ok = 1;
    for (int k = 0; k < 3; ++k) ok &= isfinite(o[k]) && isfinite(d[k]);
    float ad[3] = {fabsf(d[0]), fabsf(d[1]), fabsf(d[2])};
    int kz = ad[0] >= ad[1] ? (ad[0] >= ad[2] ? 0 : 2) : (ad[1] >= ad[2] ? 1 : 2);
    if (ok && d[kz] != 0.0f) {
      int kx = (kz + 1) % 3, ky = (kx + 1) % 3;
      if (d[kz] < 0.0f) {
        int s = kx;
        kx = ky;
        ky = s;
      }
      float Sx = d[kx] / d[kz], Sy = d[ky] / d[kz], Sz = 1.0f / d[kz];
      for (int64_t f = 0; f < F; ++f) {
        const float *v[3] = {verts + 3 * (int64_t)faces[3 * f], verts + 3 * (int64_t)faces[3 * f + 1],
                             verts + 3 * (int64_t)faces[3 * f + 2]};
        if (degenerate(v[0], v[1], v[2])) continue;
        float sx[3], sy[3], sz[3];
        for (int i = 0; i < 3; ++i) {
          float p[3] = {v[i][0] - o[0], v[i][1] - o[1], v[i][2] - o[2]};
          sx[i] = p[kx] - Sx * p[kz];
          sy[i] = p[ky] - Sy * p[kz];
          sz[i] = p[kz];
        }
        float U = sx[2] * sy[1] - sy[2] * sx[1];
        float V = sx[0] * sy[2] - sy[0] * sx[2];
        float W = sx[1] * sy[0] - sy[1] * sx[0];
        if ((U < 0.0f || V < 0.0f || W < 0.0f) && (U > 0.0f || V > 0.0f || W > 0.0f)) continue;
        float det = (U + V) + W;
        if (det == 0.0f) continue;
        float Az = Sz * sz[0], Bz = Sz * sz[1], Cz = Sz * sz[2];
        float T = (U * Az + V * Bz) + W * Cz;
        float t = T / det;
        if (!(t > 0.0f && t < INFINITY)) continue;
        if (t < best_t || (t == best_t && f < best_f)) {
          best_t = t;
          best_f = (int32_t)f;
        }
      }
    }
    t_out[r] = best_t;
    f_out[r] = best_f;
  }
}
