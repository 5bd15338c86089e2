// winding.cu — generalized winding numbers of batched triangle meshes (Jacobson, Kavan & Sorkine-Hornung 2013), the exact
// sum over every face: w(q) = sum_f Omega_f(q) / 4 pi, 1 inside and 0 outside a closed, consistently oriented mesh, and close
// to that across holes and self-intersections, so |w| > 0.5 fills the meshes that voxel_fill leaks through.
//
// The arithmetic is stated in include/genre_b200.h and restated in fp64, with a derived per-query bound on this fp32 order,
// by tests/winding_ref.py.  Per (face, query) pair, with n = (v1 - v0) x (v2 - v0) computed once per face:
//   a, b, c = v0 - q, v1 - q, v2 - q;  det = a . n (= a . (b x c), without the cancellation of three long vectors);
//   den = la lb lc + (a.b) lc + (b.c) la + (c.a) lb;  term = atan2f(det, den) = Omega / 2, 0 when det == 0.
// The terms of a query are added in fp64, in face order, on one thread: the result is bitwise repeatable and independent of
// the batch, of P and of the tiling.
//
// Launch: one CTA of WN_THREADS queries of one sample, one query per thread, grid (ceil(Q / WN_THREADS), N).  The sample's
// faces pass through shared memory in tiles of WN_THREADS: each thread gathers one face (its vertices through `faces`),
// applies the skip rule and writes (v0, v1, v2, n) as three float4; a skipped face becomes all zeros, so its det is 0 and
// its term 0.  Every thread then reads the same face: shared-memory broadcasts.
#include "common.cuh"

namespace gb {

constexpr int WN_THREADS = 256;
constexpr int WN_MAX_DIM = 512;
constexpr int64_t WN_MAX_FACES = (int64_t)1 << 31;   // exclusive
constexpr double WN_INV_2PI = 0.15915494309189535;   // the fp64 value nearest 1 / 2 pi

// the fp32 term of one face (v0 = A.xyz, v1 = (A.w, B.x, B.y), v2 = (B.z, B.w, C.x), n = C.yzw) at q, in the header's order
__device__ __forceinline__ float wn_term(const float4 A, const float4 B, const float4 C, float qx, float qy, float qz) {
  const float ax = __fsub_rn(A.x, qx), ay = __fsub_rn(A.y, qy), az = __fsub_rn(A.z, qz);
  const float bx = __fsub_rn(A.w, qx), by = __fsub_rn(B.x, qy), bz = __fsub_rn(B.y, qz);
  const float cx = __fsub_rn(B.z, qx), cy = __fsub_rn(B.w, qy), cz = __fsub_rn(C.x, qz);
  const float det = __fmaf_rn(az, C.w, __fmaf_rn(ay, C.z, __fmul_rn(ax, C.y)));
  const float la = __fsqrt_rn(__fmaf_rn(az, az, __fmaf_rn(ay, ay, __fmul_rn(ax, ax))));
  const float lb = __fsqrt_rn(__fmaf_rn(bz, bz, __fmaf_rn(by, by, __fmul_rn(bx, bx))));
  const float lc = __fsqrt_rn(__fmaf_rn(cz, cz, __fmaf_rn(cy, cy, __fmul_rn(cx, cx))));
  const float ab = __fmaf_rn(az, bz, __fmaf_rn(ay, by, __fmul_rn(ax, bx)));
  const float bc = __fmaf_rn(bz, cz, __fmaf_rn(by, cy, __fmul_rn(bx, cx)));
  const float ca = __fmaf_rn(cz, az, __fmaf_rn(cy, ay, __fmul_rn(cx, ax)));
  const float den = __fmaf_rn(ca, lb, __fmaf_rn(bc, la, __fmaf_rn(ab, lc, __fmul_rn(__fmul_rn(la, lb), lc))));
  return det == 0.0f ? 0.0f : atan2f(det, den);
}

// grid (ceil(Q / WN_THREADS), N); points == nullptr: the queries are the centres of the D x H x W grid
__global__ void __launch_bounds__(WN_THREADS)
winding_kernel(const float *__restrict__ verts, const int *__restrict__ faces, const long long *__restrict__ vert_off,
               const long long *__restrict__ face_off, const float *__restrict__ points, long long pN, long long Q, int D,
               int H, int W, float *__restrict__ out) {
  __shared__ float4 tile[WN_THREADS][3];
  const int b = blockIdx.y;
  const long long q = (long long)blockIdx.x * WN_THREADS + threadIdx.x;
  const bool active = q < Q;
  float qx = 0.0f, qy = 0.0f, qz = 0.0f;
  if (active) {
    if (points) {
      const float *p = points + b * pN + 3 * q;
      qx = __ldg(p);
      qy = __ldg(p + 1);
      qz = __ldg(p + 2);
    } else {
      // c_a = fl(fl(i_a + 0.5) / n_a) - 0.5, voxelize_mesh's frame
      const int i2 = (int)(q % W), i1 = (int)((q / W) % H), i0 = (int)(q / ((long long)W * H));
      qx = __fsub_rn(__fdiv_rn(__fadd_rn((float)i0, 0.5f), (float)D), 0.5f);
      qy = __fsub_rn(__fdiv_rn(__fadd_rn((float)i1, 0.5f), (float)H), 0.5f);
      qz = __fsub_rn(__fdiv_rn(__fadd_rn((float)i2, 0.5f), (float)W), 0.5f);
    }
  }
  const long long fb = __ldg(face_off + b), nf = __ldg(face_off + b + 1) - fb;
  const float *vb = verts + 3 * __ldg(vert_off + b);
  const int *fp = faces + 3 * fb;
  double acc = 0.0;
  for (long long base = 0; base < nf; base += WN_THREADS) {
    const int cnt = (int)min((long long)WN_THREADS, nf - base);
    if (threadIdx.x < cnt) {
      const int *f = fp + 3 * (base + threadIdx.x);
      float v[3][3];
#pragma unroll
      for (int k = 0; k < 3; ++k) {
        const float *s = vb + 3 * __ldg(f + k);
#pragma unroll
        for (int a = 0; a < 3; ++a) v[k][a] = __ldg(s + a);
      }
      float n[3] = {0.0f, 0.0f, 0.0f};
      if (mesh_face_kept(v)) {
        float e1[3], e2[3];
#pragma unroll
        for (int a = 0; a < 3; ++a) {
          e1[a] = __fsub_rn(v[1][a], v[0][a]);
          e2[a] = __fsub_rn(v[2][a], v[0][a]);
        }
        n[0] = __fmaf_rn(e1[1], e2[2], -__fmul_rn(e1[2], e2[1]));
        n[1] = __fmaf_rn(e1[2], e2[0], -__fmul_rn(e1[0], e2[2]));
        n[2] = __fmaf_rn(e1[0], e2[1], -__fmul_rn(e1[1], e2[0]));
      } else {
#pragma unroll
        for (int k = 0; k < 3; ++k)
#pragma unroll
          for (int a = 0; a < 3; ++a) v[k][a] = 0.0f;
      }
      tile[threadIdx.x][0] = make_float4(v[0][0], v[0][1], v[0][2], v[1][0]);
      tile[threadIdx.x][1] = make_float4(v[1][1], v[1][2], v[2][0], v[2][1]);
      tile[threadIdx.x][2] = make_float4(v[2][2], n[0], n[1], n[2]);
    }
    __syncthreads();
    if (active)
      for (int j = 0; j < cnt; ++j)
        acc = __dadd_rn(acc, (double)wn_term(tile[j][0], tile[j][1], tile[j][2], qx, qy, qz));
    __syncthreads();   // the tile is rewritten next
  }
  if (active) out[(long long)b * Q + q] = __double2float_rn(__dmul_rn(acc, WN_INV_2PI));
}

}  // namespace gb

using namespace gb;

extern "C" int genre_b200_winding_number(const float *verts, int64_t V, const int32_t *faces, int64_t F,
                                         const int64_t *vert_off, const int64_t *face_off, int64_t N, const float *points,
                                         int64_t P, int64_t pN, int D, int H, int W, float *out, void *stream) {
  GB_REQUIRE(vert_off && face_off && (verts || V == 0) && (faces || F == 0), GENRE_B200_EINVAL,
             "winding_number: null pointer");
  GB_REQUIRE(N >= 1 && N <= 65535, GENRE_B200_EINVAL, "winding_number: N=%lld out of range [1, 65535]", (long long)N);
  GB_REQUIRE(V >= 0 && V <= ((int64_t)1 << 40) && F >= 0 && F < WN_MAX_FACES, GENRE_B200_EINVAL,
             "winding_number: V=%lld, F=%lld out of range (F < 2^31)", (long long)V, (long long)F);
  long long Q;
  if (points) {
    GB_REQUIRE(P >= 0 && P < ((int64_t)1 << 31), GENRE_B200_EINVAL, "winding_number: P=%lld out of range [0, 2^31)",
               (long long)P);
    GB_REQUIRE(pN == 0 || pN == 3 * P, GENRE_B200_EINVAL,
               "winding_number: the point stride must be 0 (shared points) or 3*P, got %lld", (long long)pN);
    GB_REQUIRE(D == 0 && H == 0 && W == 0, GENRE_B200_EINVAL, "winding_number: points mode takes D = H = W = 0");
    Q = P;
  } else {
    GB_REQUIRE(P == 0 && pN == 0, GENRE_B200_EINVAL, "winding_number: grid mode takes P = pN = 0");
    GB_REQUIRE(D >= 1 && D <= WN_MAX_DIM && H >= 1 && H <= WN_MAX_DIM && W >= 1 && W <= WN_MAX_DIM, GENRE_B200_EINVAL,
               "winding_number: grid %dx%dx%d out of range (every dimension in [1, 512])", D, H, W);
    Q = (long long)D * H * W;
  }
  GB_REQUIRE(out || Q == 0, GENRE_B200_EINVAL, "winding_number: null output");
  GB_REQUIRE((((uintptr_t)verts | (uintptr_t)faces | (uintptr_t)points | (uintptr_t)out) & 3) == 0 &&
                 (((uintptr_t)vert_off | (uintptr_t)face_off) & 7) == 0,
             GENRE_B200_EALIGN, "winding_number: fp32 / int32 buffers must be 4-byte and offsets 8-byte aligned");
  if (Q == 0) return 0;
  const dim3 grid((unsigned)((Q + WN_THREADS - 1) / WN_THREADS), (unsigned)N);
  winding_kernel<<<grid, WN_THREADS, 0, as_stream(stream)>>>(verts, faces, (const long long *)vert_off,
                                                             (const long long *)face_off, points, pN, Q, D, H, W, out);
  return check_launch("winding_number kernel");
}
