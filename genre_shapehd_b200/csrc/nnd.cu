// nnd.cu — Chamfer nearest-neighbour distance (both directions) and its backward.
//
// Reference: toolbox/nndistance/src/nnd_cuda.cu
//   NmDistanceKernel :6-128  fixed <<<(32,16),512>>> grid regardless of problem size, one thread per
//                            query scanning all candidates, legacy default stream (:130-131)
//   NmDistanceGradKernel :143-162, launcher :163-177 (two cudaMemset + two launches, default stream)
// Here one launch covers both directions.  The op is bound by the FP32 issue rate (2*B*N*M pairs x 6 fp32 operations + the
// running minimum), so the kernel spends as few instructions per pair as exact arithmetic allows:
//   * candidates come in pairs (float2: each lane evaluates two candidates per step; each thread carries two queries, so a
//     shared-memory candidate pair (3 x LDS.64 from SoA tiles) feeds four pairs);
//   * only the running MINIMUM is updated per pair (one FMNMX for two candidates); the arg-min is recovered afterwards: each
//     lane remembers the 16-candidate chunk in which its minimum improved ("<": the earliest chunk wins) and re-evaluates that
//     one chunk at the end to find the first index whose distance equals the minimum.
// Hopper has no packed fp32 arithmetic, so a pair costs its scalar instructions; the minimum-only update still halves the rest.  A CTA owns 128 queries; each query is scanned by 4 lanes on interleaved candidate
// pairs and the 4 partial (distance, index) results meet in a 2-step shuffle reduction that keeps the lowest index on ties — the
// reference's semantics (strict '<' on an ascending scan, nnd_cuda.cu:33,120).
// The squared distance is rounded exactly as nvcc contracts the reference expression
// x2*x2+y2*y2+z2*z2 (SASS of oracle/_ref/libref_nnd_cuda.so):  fma(dz,dz, fma(dx,dx, dy*dy)),
// with d* = candidate - query, each operation IEEE-rounded on its own, so distances AND indices are
// bit-identical to the reference kernel.
#include "common.cuh"
#include <math_constants.h>

namespace gb {

constexpr int NND_THREADS = 256;
constexpr int NND_SLICES = 4;                                      // lanes per query pair
constexpr int NND_QUERIES = NND_THREADS / NND_SLICES * 2;          // 128 queries per CTA (2 per thread)
constexpr int NND_TILE = 1024;                                     // candidates per shared-memory tile (SoA, 12 KiB)
constexpr int NND_STEPS = NND_TILE / 2 / NND_SLICES;               // candidate-pair steps per lane and tile (128)
constexpr int NND_CHUNK = 8;                                       // steps per arg-min chunk (16 candidates)
constexpr int NND_CHUNKS = NND_STEPS / NND_CHUNK;                  // 16 chunks per tile
constexpr float NND_FAR = 1e18f;                                   // padding candidates: distance ~1e36, never the minimum

// squared distances of the candidate pair (cx, cy, cz) to the query whose negated coordinates are duplicated in (nx, ny, nz)
__device__ __forceinline__ float2 nnd_dist2(float2 cx, float2 cy, float2 cz, float2 nx, float2 ny, float2 nz) {
  const float2 dx = make_float2(__fadd_rn(cx.x, nx.x), __fadd_rn(cx.y, nx.y));
  const float2 dy = make_float2(__fadd_rn(cy.x, ny.x), __fadd_rn(cy.y, ny.y));
  const float2 dz = make_float2(__fadd_rn(cz.x, nz.x), __fadd_rn(cz.y, nz.y));
  return make_float2(__fmaf_rn(dz.x, dz.x, __fmaf_rn(dx.x, dx.x, __fmul_rn(dy.x, dy.x))),
                     __fmaf_rn(dz.y, dz.y, __fmaf_rn(dx.y, dx.y, __fmul_rn(dy.y, dy.y))));
}
__device__ __forceinline__ float nnd_dist1(float cx, float cy, float cz, float qx, float qy, float qz) {
  const float dx = __fadd_rn(cx, -qx), dy = __fadd_rn(cy, -qy), dz = __fadd_rn(cz, -qz);
  return __fmaf_rn(dz, dz, __fmaf_rn(dx, dx, __fmul_rn(dy, dy)));
}

__global__ void __launch_bounds__(NND_THREADS)
nnd_forward_kernel(const float *__restrict__ xyz1, const float *__restrict__ xyz2, int N, int M,
                   float *__restrict__ dist1, float *__restrict__ dist2, int *__restrict__ idx1,
                   int *__restrict__ idx2) {
  __shared__ __align__(16) float s_x[NND_TILE];
  __shared__ __align__(16) float s_y[NND_TILE];
  __shared__ __align__(16) float s_z[NND_TILE];
  const int b = blockIdx.y;
  const bool fwd = blockIdx.z == 0;  // z = 0: queries from xyz1 against xyz2;  z = 1: the other way round
  const int nq = fwd ? N : M, nc = fwd ? M : N;
  if (blockIdx.x * NND_QUERIES >= nq) return;
  const float *q = (fwd ? xyz1 : xyz2) + (size_t)b * nq * 3;
  const float *cand = (fwd ? xyz2 : xyz1) + (size_t)b * nc * 3;
  float *dist = (fwd ? dist1 : dist2) + (size_t)b * nq;
  int *idx = (fwd ? idx1 : idx2) + (size_t)b * nq;

  const int slice = threadIdx.x & (NND_SLICES - 1);
  const int qi0 = blockIdx.x * NND_QUERIES + (threadIdx.x >> 2) * 2;   // this thread's queries: qi0, qi0 + 1
  float qx[2], qy[2], qz[2];
#pragma unroll
  for (int a = 0; a < 2; ++a) {
    const bool live = qi0 + a < nq;
    qx[a] = live ? q[(qi0 + a) * 3 + 0] : 0.f;
    qy[a] = live ? q[(qi0 + a) * 3 + 1] : 0.f;
    qz[a] = live ? q[(qi0 + a) * 3 + 2] : 0.f;
  }
  const float2 nxA = make_float2(-qx[0], -qx[0]), nyA = make_float2(-qy[0], -qy[0]), nzA = make_float2(-qz[0], -qz[0]);
  const float2 nxB = make_float2(-qx[1], -qx[1]), nyB = make_float2(-qy[1], -qy[1]), nzB = make_float2(-qz[1], -qz[1]);
  const float2 *sx2 = reinterpret_cast<const float2 *>(s_x), *sy2 = reinterpret_cast<const float2 *>(s_y),
               *sz2 = reinterpret_cast<const float2 *>(s_z);

  float best[2] = {CUDART_INF_F, CUDART_INF_F};
  int bestc[2] = {-1, -1};   // chunk id (tile * NND_CHUNKS + chunk) in which the running minimum last improved
  int tile = 0;
  for (int k0 = 0; k0 < nc; k0 += NND_TILE, ++tile) {
    __syncthreads();  // previous tile fully consumed
    for (int j = threadIdx.x; j < NND_TILE; j += NND_THREADS) {
      const bool ok = k0 + j < nc;
      const float *c = cand + (size_t)(k0 + j) * 3;
      s_x[j] = ok ? c[0] : NND_FAR;
      s_y[j] = ok ? c[1] : 0.f;
      s_z[j] = ok ? c[2] : 0.f;
    }
    __syncthreads();
    const int nchunk = min(NND_CHUNKS, (min(NND_TILE, nc - k0) + 2 * NND_SLICES * NND_CHUNK - 1) / (2 * NND_SLICES * NND_CHUNK));
    for (int c = 0; c < nchunk; ++c) {
      float mA = CUDART_INF_F, mB = CUDART_INF_F;
#pragma unroll
      for (int i = 0; i < NND_CHUNK; ++i) {
        const int p = slice + NND_SLICES * (c * NND_CHUNK + i);   // candidates 2p, 2p + 1 of the tile
        const float2 cx = sx2[p], cy = sy2[p], cz = sz2[p];
        const float2 dA = nnd_dist2(cx, cy, cz, nxA, nyA, nzA);
        const float2 dB = nnd_dist2(cx, cy, cz, nxB, nyB, nzB);
        mA = fminf(mA, fminf(dA.x, dA.y));
        mB = fminf(mB, fminf(dB.x, dB.y));
      }
      if (mA < best[0]) { best[0] = mA; bestc[0] = tile * NND_CHUNKS + c; }
      if (mB < best[1]) { best[1] = mB; bestc[1] = tile * NND_CHUNKS + c; }
    }
  }
  // arg-min: re-evaluate the winning chunk of each query in ascending candidate order, first exact match
  int besti[2] = {0, 0};
#pragma unroll
  for (int a = 0; a < 2; ++a) {
    if (bestc[a] < 0) continue;
    const int kt = (bestc[a] / NND_CHUNKS) * NND_TILE, c = bestc[a] % NND_CHUNKS;
    bool found = false;
    for (int i = 0; i < NND_CHUNK && !found; ++i) {
      const int p = slice + NND_SLICES * (c * NND_CHUNK + i);
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int k = kt + 2 * p + e;
        if (!found && k < nc) {
          const float *cc = cand + (size_t)k * 3;
          if (nnd_dist1(cc[0], cc[1], cc[2], qx[a], qy[a], qz[a]) == best[a]) {
            besti[a] = k;
            found = true;
          }
        }
      }
    }
  }
  // combine the 4 slices of a query: smaller distance wins, equal distance -> smaller index
#pragma unroll
  for (int a = 0; a < 2; ++a) {
#pragma unroll
    for (int o = 1; o < NND_SLICES; o <<= 1) {
      const float od = __shfl_xor_sync(0xffffffffu, best[a], o);
      const int oi = __shfl_xor_sync(0xffffffffu, besti[a], o);
      if (od < best[a] || (od == best[a] && oi < besti[a])) {
        best[a] = od;
        besti[a] = oi;
      }
    }
    if (slice == 0 && qi0 + a < nq) {
      dist[qi0 + a] = best[a];
      idx[qi0 + a] = besti[a];
    }
  }
}

// grad_xyz1[j] += 2 g1[j] (x1[j] - x2[idx1[j]]);  grad_xyz2[idx1[j]] -= the same; and symmetrically for g2
__global__ void __launch_bounds__(256)
nnd_backward_kernel(const float *__restrict__ xyz1, const float *__restrict__ xyz2, int N, int M,
                    const float *__restrict__ g1, const float *__restrict__ g2, const int *__restrict__ idx1,
                    const int *__restrict__ idx2, float *__restrict__ grad1, float *__restrict__ grad2) {
  const int b = blockIdx.y;
  const bool fwd = blockIdx.z == 0;
  const int nq = fwd ? N : M, nc = fwd ? M : N;
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= nq) return;
  const float *a = (fwd ? xyz1 : xyz2) + (size_t)b * nq * 3;
  const float *o = (fwd ? xyz2 : xyz1) + (size_t)b * nc * 3;
  float *ga = (fwd ? grad1 : grad2) + (size_t)b * nq * 3;
  float *go = (fwd ? grad2 : grad1) + (size_t)b * nc * 3;
  const int j2 = (fwd ? idx1 : idx2)[(size_t)b * nq + j];
  const float g = (fwd ? g1 : g2)[(size_t)b * nq + j] * 2.0f;
  const float vx = g * (a[j * 3 + 0] - o[j2 * 3 + 0]);
  const float vy = g * (a[j * 3 + 1] - o[j2 * 3 + 1]);
  const float vz = g * (a[j * 3 + 2] - o[j2 * 3 + 2]);
  atomicAdd(ga + j * 3 + 0, vx);
  atomicAdd(ga + j * 3 + 1, vy);
  atomicAdd(ga + j * 3 + 2, vz);
  atomicAdd(go + j2 * 3 + 0, -vx);
  atomicAdd(go + j2 * 3 + 1, -vy);
  atomicAdd(go + j2 * 3 + 2, -vz);
}

static int nnd_check(int64_t B, int64_t N, int64_t M) {
  GB_REQUIRE(B > 0 && B <= 65535, GENRE_B200_EINVAL, "nnd: batch %lld must be in [1, 65535]", (long long)B);
  GB_REQUIRE(N > 0 && M > 0 && N < (1ll << 29) && M < (1ll << 29), GENRE_B200_EINVAL,
             "nnd: point counts (%lld, %lld) must be in [1, 2^29)", (long long)N, (long long)M);
  return 0;
}

}  // namespace gb

using namespace gb;

extern "C" int genre_b200_nnd_forward(const float *xyz1, const float *xyz2, int64_t B, int64_t N, int64_t M,
                                      float *dist1, float *dist2, int32_t *idx1, int32_t *idx2, void *stream) {
  GB_REQUIRE(xyz1 && xyz2 && dist1 && dist2 && idx1 && idx2, GENRE_B200_EINVAL, "nnd forward: null pointer");
  if (int rc = nnd_check(B, N, M)) return rc;
  const int64_t mx = N > M ? N : M;
  dim3 grid((unsigned)((mx + NND_QUERIES - 1) / NND_QUERIES), (unsigned)B, 2);
  nnd_forward_kernel<<<grid, NND_THREADS, 0, as_stream(stream)>>>(xyz1, xyz2, (int)N, (int)M, dist1, dist2, idx1, idx2);
  return check_launch("nnd forward kernel");
}

extern "C" int genre_b200_nnd_backward(const float *xyz1, const float *xyz2, int64_t B, int64_t N, int64_t M,
                                       const float *grad_dist1, const float *grad_dist2, const int32_t *idx1,
                                       const int32_t *idx2, float *grad_xyz1, float *grad_xyz2, void *stream) {
  GB_REQUIRE(xyz1 && xyz2 && grad_dist1 && grad_dist2 && idx1 && idx2 && grad_xyz1 && grad_xyz2, GENRE_B200_EINVAL,
             "nnd backward: null pointer");
  if (int rc = nnd_check(B, N, M)) return rc;
  cudaStream_t st = as_stream(stream);
  cudaError_t e = cudaMemsetAsync(grad_xyz1, 0, (size_t)B * N * 3 * sizeof(float), st);
  if (e == cudaSuccess) e = cudaMemsetAsync(grad_xyz2, 0, (size_t)B * M * 3 * sizeof(float), st);
  if (e != cudaSuccess) {
    set_error("nnd backward: memset: %s", cudaGetErrorString(e));
    return (int)e;
  }
  const int64_t mx = N > M ? N : M;
  dim3 grid((unsigned)((mx + 255) / 256), (unsigned)B, 2);
  nnd_backward_kernel<<<grid, 256, 0, st>>>(xyz1, xyz2, (int)N, (int)M, grad_dist1, grad_dist2, idx1, idx2, grad_xyz1,
                                            grad_xyz2);
  return check_launch("nnd backward kernel");
}
