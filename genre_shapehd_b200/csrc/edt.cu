// edt.cu — exact Euclidean distance transform of batched cubic grids: the squared distance, in voxel units, from every
// voxel to the nearest voxel whose value is >= level.  Separable, one pass per axis (Felzenszwalb & Huttenlocher,
// "Distance Transforms of Sampled Functions", Theory of Computing 8, 2012), all three passes in place on the output.
//
//   z pass (the contiguous axis): the input is binary, so the 1-D transform is the squared distance to the nearest set bit
//          of the row.  A warp per row: lane l reads elements 32 j + l (coalesced), a ballot per word gives the row's bits,
//          and each lane finds its element's nearest set bit below and above with __clz / __ffs.
//   y, x passes: the lower envelope of the parabolas q -> f(p) + (q - p)^2 along the axis.  One thread per line, the 32
//          lanes of a warp on 32 consecutive z, so every step of a line's walk reads or writes 32 consecutive floats: all
//          global traffic is coalesced without a transpose.  The envelope (at most R parabolas, each packed as
//          f(p) << 8 | p in one int) lives in shared memory as [k][lane], so every access is conflict-free.
// Values are integers below 2^24 (3 (R-1)^2 at most), exact in fp32, and parabola intersections are compared by int64
// cross-multiplication instead of a division, so the result is exact and does not depend on scheduling.
#include "common.cuh"
#include <math_constants.h>

namespace gb {

constexpr int EDT_MAX_RES = 256;

// z pass: one warp per row (n, x, y); rows_total = N R^2
template <int W>
__global__ void __launch_bounds__(256)
edt_rows_kernel(const float *__restrict__ vox, float *__restrict__ out, int R, float level, long long rows_total) {
  const long long row = (long long)blockIdx.x * 8 + (threadIdx.x >> 5);
  if (row >= rows_total) return;
  const int lane = threadIdx.x & 31;
  const float *src = vox + (size_t)row * R;
  float *dst = out + (size_t)row * R;
  unsigned w[W];
#pragma unroll
  for (int j = 0; j < W; ++j) {
    const int z = 32 * j + lane;
    w[j] = __ballot_sync(0xffffffffu, z < R && __ldg(src + z) >= level);
  }
#pragma unroll
  for (int j = 0; j < W; ++j) {
    const int z = 32 * j + lane;
    // nearest set bit at or below z: this word's bits <= lane, else the highest bit of a lower word
    int lo = -1;
    const unsigned below = w[j] & (0xffffffffu >> (31 - lane));
    if (below) {
      lo = 32 * j + 31 - __clz(below);
    } else {
#pragma unroll
      for (int i = j - 1; i >= 0; --i)
        if (lo < 0 && w[i]) lo = 32 * i + 31 - __clz(w[i]);
    }
    // nearest set bit at or above z: this word's bits >= lane, else the lowest bit of a higher word
    int hi = -1;
    const unsigned above = w[j] & (0xffffffffu << lane);
    if (above) {
      hi = 32 * j + __ffs(above) - 1;
    } else {
#pragma unroll
      for (int i = j + 1; i < W; ++i)
        if (hi < 0 && w[i]) hi = 32 * i + __ffs(w[i]) - 1;
    }
    int d = 0x7fffffff;
    if (lo >= 0) d = z - lo;
    if (hi >= 0) d = min(d, hi - z);
    if (z < R) dst[z] = d == 0x7fffffff ? CUDART_INF_F : (float)(d * d);
  }
}

// y or x pass, in place: line (n, a, z) holds the elements base + q * stride, q = 0 .. R-1, with
// base = n R^3 + a * a_stride + z.  blockIdx.x = z tile of 32, blockIdx.y = a, blockIdx.z = n; one warp per block.
__global__ void __launch_bounds__(32)
edt_lines_kernel(float *__restrict__ out, int R, long long stride, long long a_stride) {
  extern __shared__ int env[];                   // [R][32]: the envelope's parabolas, f << 8 | p
  const int lane = threadIdx.x;
  const int z = blockIdx.x * 32 + lane;
  if (z >= R) return;
  float *line = out + (size_t)blockIdx.z * R * R * R + (size_t)blockIdx.y * a_stride + z;
  int k = -1;                                    // top of the envelope
  int vk = 0, fk = 0, vk1 = 0, fk1 = 0;          // parabolas k and k - 1 (p, f)
  for (int q0 = 0; q0 < R; q0 += 8) {
    float fv[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) fv[i] = q0 + i < R ? line[(size_t)(q0 + i) * stride] : CUDART_INF_F;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      if (fv[i] == CUDART_INF_F) continue;
      const int q = q0 + i, fq = (int)fv[i];
      const long long bq = (long long)fq + (long long)q * q;
      // pop k while the new parabola's intersection with k is at or left of k's intersection with k - 1:
      //   (bq - bk) / (2 (q - vk)) <= (bk - bk1) / (2 (vk - vk1)), both denominators > 0
      while (k >= 1) {
        const long long bk = (long long)fk + (long long)vk * vk, bk1 = (long long)fk1 + (long long)vk1 * vk1;
        if ((bq - bk) * (long long)(vk - vk1) > (bk - bk1) * (long long)(q - vk)) break;
        --k;
        vk = vk1;
        fk = fk1;
        if (k >= 1) {
          const int e = env[(k - 1) * 32 + lane];
          vk1 = e & 0xff;
          fk1 = e >> 8;
        }
      }
      ++k;
      env[k * 32 + lane] = (fq << 8) | q;
      vk1 = vk;
      fk1 = fk;
      vk = q;
      fk = fq;
    }
  }
  if (k < 0) {                                   // no finite value on the line: it stays +inf
    for (int q = 0; q < R; ++q) line[(size_t)q * stride] = CUDART_INF_F;
    return;
  }
  int j = 0;
  int e = env[lane];
  int vj = e & 0xff, fj = e >> 8;
  for (int q = 0; q < R; ++q) {
    // advance while parabola j + 1's intersection with j lies left of q: (b_{j+1} - b_j) < 2 q (v_{j+1} - v_j)
    while (j < k) {
      const int e1 = env[(j + 1) * 32 + lane];
      const int v1 = e1 & 0xff, f1 = e1 >> 8;
      const long long b1 = (long long)f1 + (long long)v1 * v1, b0 = (long long)fj + (long long)vj * vj;
      if (b1 - b0 >= 2ll * q * (v1 - vj)) break;
      ++j;
      vj = v1;
      fj = f1;
    }
    const int d = q - vj;
    line[(size_t)q * stride] = (float)(d * d + fj);
  }
}

}  // namespace gb

using namespace gb;

extern "C" int genre_b200_distance_transform(const float *vox, int64_t N, int res, float level, float *out_sq,
                                             void *stream) {
  GB_REQUIRE(vox && out_sq, GENRE_B200_EINVAL, "distance_transform: null pointer");
  GB_REQUIRE(vox != out_sq, GENRE_B200_EINVAL, "distance_transform: in-place operation is not supported");
  GB_REQUIRE(N >= 1 && N <= 65535, GENRE_B200_EINVAL, "distance_transform: N=%lld out of range [1, 65535]", (long long)N);
  GB_REQUIRE(res >= 1 && res <= EDT_MAX_RES, GENRE_B200_EINVAL, "distance_transform: R=%d out of range [1, %d]", res,
             EDT_MAX_RES);
  GB_REQUIRE(level == level, GENRE_B200_EINVAL, "distance_transform: level is NaN");
  GB_REQUIRE((((uintptr_t)vox | (uintptr_t)out_sq) & 3) == 0, GENRE_B200_EALIGN,
             "distance_transform: vox and out_sq must be 4-byte aligned");
  cudaStream_t st = as_stream(stream);
  const long long rows = (long long)N * res * res;
  const unsigned rgrid = (unsigned)((rows + 7) / 8);
  switch ((res + 31) / 32) {
#define GB_EDT(WW) \
  case WW: edt_rows_kernel<WW><<<rgrid, 256, 0, st>>>(vox, out_sq, res, level, rows); break;
    GB_EDT(1) GB_EDT(2) GB_EDT(3) GB_EDT(4) GB_EDT(5) GB_EDT(6) GB_EDT(7) GB_EDT(8)
#undef GB_EDT
    default: return fail_arg(GENRE_B200_EINVAL, "distance_transform: R=%d unsupported", res);
  }
  if (int rc = check_launch("distance_transform rows kernel")) return rc;
  const dim3 lgrid((unsigned)((res + 31) / 32), (unsigned)res, (unsigned)N);
  const size_t smem = (size_t)res * 32 * sizeof(int);
  const long long R = res;
  edt_lines_kernel<<<lgrid, 32, smem, st>>>(out_sq, res, R, R * R);         // along y: lines (n, x, z)
  if (int rc = check_launch("distance_transform y kernel")) return rc;
  edt_lines_kernel<<<lgrid, 32, smem, st>>>(out_sq, res, R * R, R);         // along x: lines (n, y, z)
  return check_launch("distance_transform x kernel");
}
