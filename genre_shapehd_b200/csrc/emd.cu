// emd.cu — earth mover's distance between equal-size point sets: a Jacobi auction with eps-scaling (Bertsekas), one CTA per
// pair.  The contract (cost, bid, tie rules, eps schedule, sum order) is stated in include/genre_b200.h and restated in numpy
// by tests/emd_ref.py, bit for bit.
//
// Layout: the pair's q (the objects), the prices, the assignment both ways, the per-object highest bid and its bidder, each
// bidder's bid and two lists of unassigned persons (this round's, the next one's) live in shared memory, 56 n bytes (224 KiB
// at n = 4096).  p (the persons) stays in global memory: a bidder reads its own three coordinates once per bid, while q is scanned by every bid.
// A round is three passes separated by block barriers:
//   A  every unassigned person bids.  512 threads, 16 warps: with at least 16 bidders one warp serves one bidder at a time;
//      with fewer, a group of G = 16 / cnt warps (rounded down to a power of two) splits one bidder's object scan, so the
//      long tail of rounds with a handful of bidders still uses the whole CTA.  (1024 threads would cap the kernel at 64
//      registers and spill.)  Each lane keeps (best value, its lowest object, second value) over its
//      objects; the merge of two such triples is exact (maxima and an index comparison, no rounding), so the result does not
//      depend on the grouping or the reduction order.  The bid goes to bid[i]; its object, encoded as assign[i] = -2 - j, and
//      a 64-bit atomicMax of the bid's bits (bids are > 0, so bit order is value order) into best[j].
//   B  every bidder whose bid equals best[j] proposes itself by atomicMin into winner[j]: the lowest index wins equal bids.
//   C  the winner of j evicts j's owner (who joins the next list), takes j, sets price[j] and restores best / winner to
//      their idle values; the others rejoin the list.  The list order is scheduling-dependent but nothing reads it in order.
#include "common.cuh"
#include <math_constants.h>

namespace gb {

constexpr int EMD_THREADS = 512;
constexpr int EMD_WARPS = EMD_THREADS / 32;
constexpr int EMD_MAX_N = 4096;
constexpr int EMD_MAX_ROUNDS = 1 << 22;                    // per pair, over all phases: the safety net of the header
constexpr float EMD_COORD_MAX = 4611686018427387904.0f;    // 2^62: |coordinate| above it (or NaN) refuses the pair
constexpr int EMD_IDLE = 0x7fffffff;                       // winner[j] when j has no bid in flight

__host__ __device__ constexpr size_t emd_smem_bytes(int n) { return (size_t)n * (3 * 8 + 3 * 4 + 5 * 4); }

// c_ij: fp32, no contraction, correctly rounded sqrt
__device__ __forceinline__ float emd_cost(float px, float py, float pz, float qx, float qy, float qz) {
  const float dx = __fsub_rn(px, qx), dy = __fsub_rn(py, qy), dz = __fsub_rn(pz, qz);
  return __fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz)));
}

struct Best {
  double v1, v2;   // the best value and the best over every other object
  int j1;          // the lowest object attaining v1
};

// the triple of the union of two disjoint object sets (exact: no rounding)
__device__ __forceinline__ void emd_merge(Best &a, const Best &b) {
  if (b.v1 > a.v1 || (b.v1 == a.v1 && b.j1 < a.j1)) {
    a.v2 = fmax(a.v1, b.v2);
    a.v1 = b.v1;
    a.j1 = b.j1;
  } else {
    a.v2 = fmax(a.v2, b.v1);
  }
}

__device__ __forceinline__ Best emd_warp_merge(Best t) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    Best u;
    u.v1 = __shfl_xor_sync(0xffffffffu, t.v1, o);
    u.v2 = __shfl_xor_sync(0xffffffffu, t.v2, o);
    u.j1 = __shfl_xor_sync(0xffffffffu, t.j1, o);
    emd_merge(t, u);
  }
  return t;
}

// objects lane, lane + stride, ... in ascending order: a later equal value only raises v2
__device__ __forceinline__ Best emd_scan(float px, float py, float pz, const float *qx, const float *qy, const float *qz,
                                         const double *price, int n, int lane, int stride) {
  Best t{-CUDART_INF, -CUDART_INF, EMD_IDLE};
  for (int j = lane; j < n; j += stride) {
    const double v = __dsub_rn(-(double)emd_cost(px, py, pz, qx[j], qy[j], qz[j]), price[j]);
    if (v > t.v1) {
      t.v2 = t.v1;
      t.v1 = v;
      t.j1 = j;
    } else if (v > t.v2) {
      t.v2 = v;
    }
  }
  return t;
}

__device__ __forceinline__ void emd_place_bid(int i, Best t, const double *price, double eps, double *bid, int *assign,
                                              unsigned long long *best) {
  const double v2 = t.v2 == -CUDART_INF ? t.v1 : t.v2;   // n = 1: no second object, the bid is price + eps
  const double x = __dadd_rn(__dadd_rn(price[t.j1], __dsub_rn(t.v1, v2)), eps);
  bid[i] = x;
  assign[i] = -2 - t.j1;
  atomicMax(best + t.j1, (unsigned long long)__double_as_longlong(x));
}

__global__ void __launch_bounds__(EMD_THREADS, 1)
emd_auction_kernel(const float *__restrict__ p_all, const float *__restrict__ q_all, int n, double eps_user,
                   int32_t *__restrict__ match, double *__restrict__ emd, int32_t *__restrict__ counters) {
  extern __shared__ __align__(16) unsigned char emd_smem[];
  double *price = reinterpret_cast<double *>(emd_smem);
  double *bid = price + n;
  unsigned long long *best = reinterpret_cast<unsigned long long *>(bid + n);
  float *qx = reinterpret_cast<float *>(best + n), *qy = qx + n, *qz = qy + n;
  int *assign = reinterpret_cast<int *>(qz + n), *owner = assign + n, *winner = owner + n;
  int *list0 = winner + n;   // the two lists: list0 and list0 + n
  __shared__ float s_lo[3][EMD_WARPS], s_hi[3][EMD_WARPS];
  __shared__ int s_bad[EMD_WARPS];
  __shared__ Best s_part[EMD_WARPS];
  __shared__ double s_eps[2];   // the first phase's eps, the effective eps
  __shared__ int s_cnt[2];

  const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const float *p = p_all + (size_t)b * n * 3, *q = q_all + (size_t)b * n * 3;

  // q into shared memory, the pair's bounding box, and the refusal of non-finite or huge coordinates
  float lo[3] = {CUDART_INF_F, CUDART_INF_F, CUDART_INF_F}, hi[3] = {-CUDART_INF_F, -CUDART_INF_F, -CUDART_INF_F};
  int bad = 0;
  for (int k = tid; k < n; k += EMD_THREADS) {
    const float a[3] = {__ldg(q + 3 * k), __ldg(q + 3 * k + 1), __ldg(q + 3 * k + 2)};
    const float c[3] = {__ldg(p + 3 * k), __ldg(p + 3 * k + 1), __ldg(p + 3 * k + 2)};
    qx[k] = a[0];
    qy[k] = a[1];
    qz[k] = a[2];
#pragma unroll
    for (int d = 0; d < 3; ++d) {
      bad |= !(fabsf(a[d]) <= EMD_COORD_MAX) | !(fabsf(c[d]) <= EMD_COORD_MAX);
      lo[d] = fminf(lo[d], fminf(a[d], c[d]));
      hi[d] = fmaxf(hi[d], fmaxf(a[d], c[d]));
    }
    price[k] = 0.0;
    best[k] = 0ull;
    winner[k] = EMD_IDLE;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    bad |= __shfl_xor_sync(0xffffffffu, bad, o);
#pragma unroll
    for (int d = 0; d < 3; ++d) {
      lo[d] = fminf(lo[d], __shfl_xor_sync(0xffffffffu, lo[d], o));
      hi[d] = fmaxf(hi[d], __shfl_xor_sync(0xffffffffu, hi[d], o));
    }
  }
  if (lane == 0) {
    s_bad[warp] = bad;
#pragma unroll
    for (int d = 0; d < 3; ++d) {
      s_lo[d][warp] = lo[d];
      s_hi[d][warp] = hi[d];
    }
  }
  __syncthreads();
  if (tid == 0) {
    int any = 0;
    float l[3] = {CUDART_INF_F, CUDART_INF_F, CUDART_INF_F}, h[3] = {-CUDART_INF_F, -CUDART_INF_F, -CUDART_INF_F};
    for (int w = 0; w < EMD_WARPS; ++w) {
      any |= s_bad[w];
#pragma unroll
      for (int d = 0; d < 3; ++d) {
        l[d] = fminf(l[d], s_lo[d][w]);
        h[d] = fmaxf(h[d], s_hi[d][w]);
      }
    }
    s_bad[0] = any;
    // D = sqrt((ex*ex + ey*ey) + ez*ez), e = (double)hi - (double)lo, fp64 without contraction
    const double ex = __dsub_rn((double)h[0], (double)l[0]), ey = __dsub_rn((double)h[1], (double)l[1]),
                 ez = __dsub_rn((double)h[2], (double)l[2]);
    const double D = __dsqrt_rn(__dadd_rn(__dadd_rn(__dmul_rn(ex, ex), __dmul_rn(ey, ey)), __dmul_rn(ez, ez)));
    const double eps_eff = fmax(eps_user, ldexp(D, -32));
    s_eps[0] = fmax(__dmul_rn(D, 0.25), eps_eff);
    s_eps[1] = eps_eff;
  }
  __syncthreads();
  const bool refused = s_bad[0] != 0;
  const double eps_eff = s_eps[1];
  double eps = s_eps[0];
  int rounds = 0, phases = 0;
  bool ok = !refused;

  while (ok) {
    // a phase: the assignment resets, the prices carry over.  The barrier keeps s_cnt[0] until every thread has read the
    // last phase's final count.
    __syncthreads();
    for (int k = tid; k < n; k += EMD_THREADS) {
      assign[k] = -1;
      owner[k] = -1;
      list0[k] = k;
    }
    if (tid == 0) s_cnt[0] = n;
    ++phases;
    int cur = 0;
    __syncthreads();
    for (;;) {
      const int cnt = s_cnt[cur];
      const int *list = list0 + cur * n;
      int *next = list0 + (cur ^ 1) * n;
      // A: bids
      if (tid == 0) s_cnt[cur ^ 1] = 0;
      if (cnt >= EMD_WARPS) {
        for (int k = warp; k < cnt; k += EMD_WARPS) {
          const int i = list[k];
          const Best t = emd_warp_merge(emd_scan(__ldg(p + 3 * i), __ldg(p + 3 * i + 1), __ldg(p + 3 * i + 2), qx, qy, qz,
                                                 price, n, lane, 32));
          if (lane == 0) emd_place_bid(i, t, price, eps, bid, assign, best);
        }
      } else {
        int G = 1;
        while (2 * G * cnt <= EMD_WARPS) G *= 2;
        const int group = warp / G, sub = warp % G;
        const int i = group < cnt ? list[group] : -1;
        if (i >= 0) {
          const Best t = emd_warp_merge(emd_scan(__ldg(p + 3 * i), __ldg(p + 3 * i + 1), __ldg(p + 3 * i + 2), qx, qy, qz,
                                                 price, n, sub * 32 + lane, G * 32));
          if (lane == 0) s_part[warp] = t;
        }
        __syncthreads();
        if (i >= 0 && sub == 0 && lane == 0) {
          Best t = s_part[warp];
          for (int w = 1; w < G; ++w) emd_merge(t, s_part[warp + w]);
          emd_place_bid(i, t, price, eps, bid, assign, best);
        }
      }
      __syncthreads();
      // B: the highest bid on an object, then the lowest bidder among equal bids
      for (int k = tid; k < cnt; k += EMD_THREADS) {
        const int i = list[k], j = -2 - assign[i];
        if ((unsigned long long)__double_as_longlong(bid[i]) == best[j]) atomicMin(winner + j, i);
      }
      __syncthreads();
      // C: winners take their objects, evicted owners and losers form the next list
      for (int k = tid; k < cnt; k += EMD_THREADS) {
        const int i = list[k], j = -2 - assign[i];
        if (winner[j] == i) {
          const int old = owner[j];
          if (old >= 0) {
            assign[old] = -1;
            next[atomicAdd(s_cnt + (cur ^ 1), 1)] = old;
          }
          owner[j] = i;
          assign[i] = j;
          price[j] = bid[i];
          best[j] = 0ull;
          winner[j] = EMD_IDLE;
        } else {
          assign[i] = -1;
          next[atomicAdd(s_cnt + (cur ^ 1), 1)] = i;
        }
      }
      __syncthreads();
      cur ^= 1;
      ++rounds;
      if (s_cnt[cur] == 0) break;
      if (rounds >= EMD_MAX_ROUNDS) {
        ok = false;
        break;
      }
    }
    if (!ok || eps == eps_eff) break;
    eps = fmax(__dmul_rn(eps, 0.25), eps_eff);
  }

  if (tid == 0) {
    counters[2 * b] = rounds;
    counters[2 * b + 1] = phases;
  }
  int32_t *m = match + (size_t)b * n;
  if (!ok) {
    for (int k = tid; k < n; k += EMD_THREADS) m[k] = -1;
    if (tid == 0) emd[b] = CUDART_NAN;
    return;
  }
  // emd: the matched costs widened to fp64, zero-padded to the next power of two N2 and summed by halving
  // (a[i] += a[i + N2/2^s]), then divided by n.  price serves as the scratch.
  int h = 1;
  while (h < n) h *= 2;
  h /= 2;
  for (int k = tid; k < n; k += EMD_THREADS) m[k] = assign[k];
  if (n == 1) {
    if (tid == 0) emd[b] = (double)emd_cost(p[0], p[1], p[2], qx[assign[0]], qy[assign[0]], qz[assign[0]]);
    return;
  }
  for (int k = tid; k < h; k += EMD_THREADS) {
    double a = (double)emd_cost(p[3 * k], p[3 * k + 1], p[3 * k + 2], qx[assign[k]], qy[assign[k]], qz[assign[k]]);
    const int k2 = k + h;
    if (k2 < n)
      a = __dadd_rn(a, (double)emd_cost(p[3 * k2], p[3 * k2 + 1], p[3 * k2 + 2], qx[assign[k2]], qy[assign[k2]],
                                         qz[assign[k2]]));
    bid[k] = a;
  }
  __syncthreads();
  while (h > 1) {
    h /= 2;
    for (int k = tid; k < h; k += EMD_THREADS) bid[k] = __dadd_rn(bid[k], bid[k + h]);
    __syncthreads();
  }
  if (tid == 0) emd[b] = __ddiv_rn(bid[0], (double)n);
}

static bool emd_shape_ok(int64_t B, int64_t n) { return B >= 1 && B <= 65535 && n >= 1 && n <= EMD_MAX_N; }

}  // namespace gb

using namespace gb;

extern "C" size_t genre_b200_emd_workspace_bytes(int64_t B, int64_t n) {
  return emd_shape_ok(B, n) ? (size_t)((B * 2 * sizeof(int32_t) + 15) / 16 * 16) : 0;
}

extern "C" int genre_b200_emd_forward(const float *p, const float *q, int64_t B, int64_t n, double eps, int32_t *match,
                                      double *emd, void *workspace, size_t workspace_bytes, void *stream) {
  GB_REQUIRE(p && q && match && emd && workspace, GENRE_B200_EINVAL, "emd: null pointer");
  GB_REQUIRE(B >= 1 && B <= 65535, GENRE_B200_EINVAL, "emd: B=%lld out of range [1, 65535]", (long long)B);
  GB_REQUIRE(n >= 1 && n <= EMD_MAX_N, GENRE_B200_EINVAL, "emd: n=%lld points per set out of range [1, %d]", (long long)n,
             EMD_MAX_N);
  GB_REQUIRE(eps > 0.0 && eps <= 1.7976931348623157e308, GENRE_B200_EINVAL, "emd: eps=%g must be finite and > 0", eps);
  const size_t need = genre_b200_emd_workspace_bytes(B, n);
  GB_REQUIRE(workspace_bytes >= need && aligned16(workspace), GENRE_B200_EWORKSPACE,
             "emd: workspace too small or misaligned (%zu bytes needed, 16-byte aligned)", need);
  const size_t smem = emd_smem_bytes((int)n);
  cudaError_t e = cudaFuncSetAttribute(emd_auction_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) {
    set_error("emd: shared memory attribute: %s", cudaGetErrorString(e));
    return (int)e;
  }
  emd_auction_kernel<<<(unsigned)B, EMD_THREADS, smem, as_stream(stream)>>>(p, q, (int)n, eps, match, emd,
                                                                          (int32_t *)workspace);
  return check_launch("emd auction kernel");
}
