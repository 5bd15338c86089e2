// pose_score.cu — scores of candidate camera poses of a grid against observed camera-frame points: the mean squared
// distance (clamped to tau) from the posed points to the grid's surface, read from a precomputed distance field.
//
// One thread per candidate: it moves every point of its sample into the grid frame with its camera and sums the costs in
// point order, so a candidate's score is bitwise the same whatever else the call holds and however it is tiled.  A CTA
// serves 256 candidates of one sample; the sample's points (at most 4096, 48 KB) are staged once in shared memory and read
// as broadcasts.  The field lookups are 8-tap trilinear gathers through the read-only cache; the CTAs of one sample are
// adjacent in the grid, so they share its field in L2.
// The exact arithmetic is stated in include/genre_b200.h and restated in fp64 by tests/pose_score_ref.py.
#include "render.cuh"

namespace gb {

constexpr int PS_THREADS = 256;
constexpr int PS_MAX_POINTS = 4096;
constexpr int PS_MAX_RES = 256;

__global__ void __launch_bounds__(PS_THREADS)
pose_score_kernel(const float *__restrict__ field, int R, const float *__restrict__ points, int P,
                  const int32_t *__restrict__ counts, const float *__restrict__ rot, long long rN, long long rK,
                  const float *__restrict__ eye, long long eN, long long eK, int K, float tau, float *__restrict__ score) {
  extern __shared__ float pts[];                 // [count][3]
  const int n = blockIdx.y;
  const int cnt = __ldg(counts + n);
  const bool ok = cnt >= 1 && cnt <= P;
  if (ok)
    for (int i = threadIdx.x; i < 3 * cnt; i += PS_THREADS) pts[i] = __ldg(points + (size_t)n * P * 3 + i);
  __syncthreads();
  const int k = blockIdx.x * PS_THREADS + threadIdx.x;
  if (k >= K) return;
  float *out = score + (size_t)n * K + k;
  if (!ok) {                                     // the host checks counts; a bad one reads nothing
    *out = __int_as_float(0x7fffffff);
    return;
  }
  const float *r = rot + n * rN + k * rK;
  const float *e = eye + n * eN + k * eK;
  float m[9];
#pragma unroll
  for (int i = 0; i < 9; ++i) m[i] = __ldg(r + i);
  const float ex = __ldg(e), ey = __ldg(e + 1), ez = __ldg(e + 2);
  const float *vol = field + (size_t)n * R * R * R;
  const float Rf = (float)R, hi = (float)(R - 1), tau2 = __fmul_rn(tau, tau);
  const VoxPre pre{1.0f, 0.0f, 0.0f};
  float acc = 0.0f;
  for (int p = 0; p < cnt; ++p) {
    const float px = pts[3 * p], py = pts[3 * p + 1], pz = pts[3 * p + 2];
    // x = rot p + eye, f = (x + 0.5) R - 0.5 per axis
    const float gx = __fadd_rn(fmaf(m[2], pz, fmaf(m[1], py, __fmul_rn(m[0], px))), ex);
    const float gy = __fadd_rn(fmaf(m[5], pz, fmaf(m[4], py, __fmul_rn(m[3], px))), ey);
    const float gz = __fadd_rn(fmaf(m[8], pz, fmaf(m[7], py, __fmul_rn(m[6], px))), ez);
    const float fx = __fsub_rn(__fmul_rn(__fadd_rn(gx, 0.5f), Rf), 0.5f);
    const float fy = __fsub_rn(__fmul_rn(__fadd_rn(gy, 0.5f), Rf), 0.5f);
    const float fz = __fsub_rn(__fmul_rn(__fadd_rn(gz, 0.5f), Rf), 0.5f);
    float c = tau2;
    if (fx >= 0.0f && fx <= hi && fy >= 0.0f && fy <= hi && fz >= 0.0f && fz <= hi) {
      Taps t;
      make_taps_at(fx, fy, fz, R, t);
      const float v = sample_trilinear<false>(vol, t, R, pre);
      c = __fmul_rn(v, v);
    }
    acc = __fadd_rn(acc, c);
  }
  *out = __fdiv_rn(acc, (float)cnt);
}

}  // namespace gb

using namespace gb;

extern "C" int genre_b200_pose_score(const float *field, int64_t N, int res, const float *points, int64_t P,
                                     const int32_t *counts, const float *rot, int64_t rN, int64_t rK, const float *eye,
                                     int64_t eN, int64_t eK, int64_t K, float tau, float *score, void *stream) {
  GB_REQUIRE(field && points && counts && rot && eye && score, GENRE_B200_EINVAL, "pose_score: null pointer");
  GB_REQUIRE(N >= 1 && N <= 65535, GENRE_B200_EINVAL, "pose_score: N=%lld out of range [1, 65535]", (long long)N);
  GB_REQUIRE(res >= 1 && res <= PS_MAX_RES, GENRE_B200_EINVAL, "pose_score: R=%d out of range [1, %d]", res, PS_MAX_RES);
  GB_REQUIRE(P >= 1 && P <= PS_MAX_POINTS, GENRE_B200_EINVAL, "pose_score: P=%lld points out of range [1, %d]",
             (long long)P, PS_MAX_POINTS);
  GB_REQUIRE(K >= 1 && K <= (1ll << 30), GENRE_B200_EINVAL, "pose_score: K=%lld candidates out of range [1, 2^30]",
             (long long)K);
  GB_REQUIRE(rN >= 0 && rK >= 0 && eN >= 0 && eK >= 0, GENRE_B200_EINVAL, "pose_score: negative camera strides");
  GB_REQUIRE(tau > 0.0f && tau <= 3.4e38f, GENRE_B200_EINVAL, "pose_score: tau %g must be positive and finite",
             (double)tau);
  GB_REQUIRE((((uintptr_t)field | (uintptr_t)points | (uintptr_t)counts | (uintptr_t)rot | (uintptr_t)eye |
               (uintptr_t)score) & 3) == 0,
             GENRE_B200_EALIGN, "pose_score: every buffer must be 4-byte aligned");
  const dim3 grid((unsigned)((K + PS_THREADS - 1) / PS_THREADS), (unsigned)N);
  const size_t smem = (size_t)P * 3 * sizeof(float);
  pose_score_kernel<<<grid, PS_THREADS, smem, as_stream(stream)>>>(field, res, points, (int)P, counts, rot, rN, rK, eye,
                                                                   eN, eK, (int)K, tau, score);
  return check_launch("pose_score kernel");
}
