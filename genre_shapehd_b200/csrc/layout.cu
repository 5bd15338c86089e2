// layout.cu — NCDHW <-> channel-blocked activation layouts for the wgmma convolution kernels (convt3d.cu).
//
// The reference's nets (networks/networks.py) exchange NCDHW fp32 tensors; the kernels want 16 bytes per position and
// channel group ([B*D][C/g][H][W][g], g = 4 fp32 or 8 fp16) so that a tap shift is an address offset.  These are the
// boundary crossings, each ONE pass over the data: every warp load is a contiguous run along x of one channel plane,
// every store is 16 bytes per thread, contiguous across the warp.  Pure HBM-bound byte moves.
//   to_blocked    : [B,C,D,H,W] fp32            -> [B*D][C/g][H][W][g]                      (cast to fp16 when g = 8)
//   s2d_blocked   : [B,C,D,H,W] fp32 (even ext) -> [B*D/2][8C/g][H/2][W/2][g], channel = ((c*2+pz)*2+py)*2+px
//   s2d_sources   : [B,C,D,H,W] fp32 (even ext) -> [B*D/2][8*cpad/g][H/2][W/2][g], the 8 parity sub-volumes one after
//                   the other along the channel-group axis, each zero-padded from C to cpad channels
//   s4d_blocked   : [B,C,D,H,W] fp32 (ext % 4)   -> [B*D/4][64C/g][H/4][W/4][g], channel = ((c*4+rz)*4+ry)*4+rx
//   from_blocked  : [B*D][cg][H][W][4] fp32     -> [B,C,D,H,W] fp32 (drops channel padding)
#include <cuda_fp16.h>

#include "common.cuh"

namespace gb {

constexpr int LY_THREADS = 256;

template <int G>
__device__ __forceinline__ void store_unit(void *dst, size_t unit_index, const float (&x)[G]) {
  if (G == 4) {
    reinterpret_cast<float4 *>(dst)[unit_index] = make_float4(x[0], x[1], x[2], x[3]);
  } else {
    const __half2 a = __floats2half2_rn(x[0], x[1]), b = __floats2half2_rn(x[2], x[3]);
    const __half2 c = __floats2half2_rn(x[4 % G], x[5 % G]), d = __floats2half2_rn(x[6 % G], x[7 % G]);
    uint4 u;
    u.x = *reinterpret_cast<const unsigned *>(&a);
    u.y = *reinterpret_cast<const unsigned *>(&b);
    u.z = *reinterpret_cast<const unsigned *>(&c);
    u.w = *reinterpret_cast<const unsigned *>(&d);
    reinterpret_cast<uint4 *>(dst)[unit_index] = u;
  }
}

// X2 output (the fp32-accurate conv mode's operand): [r][2 parts][CG][plane] units of 8 fp16, part 0 = hi = fp16(a), part 1 =
// lo' = fp16((a - hi) * 2^11).  `u` is the unit index in the single-part layout [r][CG][plane]; units_per_r = CG * plane.
__device__ __forceinline__ void store_unit_x2(void *dst, size_t u, size_t r, size_t units_per_r, const float (&x)[8]) {
  uint4 ph, pl;
  split_hi_lo8(x, ph, pl);
  uint4 *o = reinterpret_cast<uint4 *>(dst) + u + r * units_per_r;
  o[0] = ph;
  o[units_per_r] = pl;
}
template <int G, bool X2>
__device__ __forceinline__ void store_out(void *dst, size_t u, size_t r, size_t units_per_r, const float (&x)[G]) {
  if constexpr (X2) {
    static_assert(G == 8, "the hi/lo operand has 8 channels per unit");
    store_unit_x2(dst, u, r, units_per_r, x);
  } else {
    store_unit<G>(dst, u, x);
  }
}

template <int G, bool X2 = false>
__global__ void __launch_bounds__(LY_THREADS)
to_blocked_kernel(const float *__restrict__ src, void *__restrict__ dst, int C, int D, int H, int W, size_t units) {
  const int CG = C / G;
  const size_t plane = (size_t)H * W, vol = plane * D;
  for (size_t u = (size_t)blockIdx.x * LY_THREADS + threadIdx.x; u < units; u += (size_t)gridDim.x * LY_THREADS) {
    const size_t hw = u % plane;
    size_t r = u / plane;
    const int cg = (int)(r % CG);
    r /= CG;  // b * D + d
    const size_t b = r / D, d = r - b * D;
    const float *s = src + ((b * C + (size_t)cg * G) * D + d) * plane + hw;
    float x[G];
#pragma unroll
    for (int e = 0; e < G; ++e) x[e] = __ldg(s + e * vol);
    store_out<G, X2>(dst, u, r, (size_t)CG * plane, x);
  }
}

// one thread = one output position (z', y', x') of one input channel c: reads the 2x2x2 cell as four float2
template <int G, bool X2 = false>
__global__ void __launch_bounds__(LY_THREADS)
s2d_blocked_kernel(const float *__restrict__ src, void *__restrict__ dst, int C, int D, int H, int W, size_t cells,
                   int CGo /* channel groups of dst (>= C*8/G; the extra ones were zero-filled by the launcher) */) {
  const int D2 = D / 2, H2 = H / 2, W2 = W / 2;
  for (size_t i = (size_t)blockIdx.x * LY_THREADS + threadIdx.x; i < cells; i += (size_t)gridDim.x * LY_THREADS) {
    const int x2 = (int)(i % W2);
    size_t r = i / W2;
    const int y2 = (int)(r % H2);
    r /= H2;
    const int c = (int)(r % C);
    r /= C;  // b * D2 + z'
    const size_t b = r / D2, z2 = r - b * D2;
    const float *s = src + (((b * C + c) * D + 2 * z2) * H + 2 * y2) * (size_t)W + 2 * x2;
    float v[8];
#pragma unroll
    for (int pz = 0; pz < 2; ++pz)
#pragma unroll
      for (int py = 0; py < 2; ++py) {
        const float2 t = __ldg(reinterpret_cast<const float2 *>(s + ((size_t)pz * H + py) * W));
        v[(pz * 2 + py) * 2] = t.x;
        v[(pz * 2 + py) * 2 + 1] = t.y;
      }
    if (G == 8) {
      float x[G];
#pragma unroll
      for (int e = 0; e < G; ++e) x[e] = v[e % 8];
      store_out<G, X2>(dst, ((r * CGo + c) * H2 + y2) * (size_t)W2 + x2, r, (size_t)CGo * H2 * W2, x);
    } else {
#pragma unroll
      for (int pz = 0; pz < 2; ++pz) {
        float x[G];
#pragma unroll
        for (int e = 0; e < G; ++e) x[e] = v[(pz * 4 + e) % 8];
        store_unit<G>(dst, ((r * CGo + c * 2 + pz) * H2 + y2) * (size_t)W2 + x2, x);
      }
    }
  }
}

// one thread = (z', pz, py, channel group, y', x'): reads G float2 (both x parities), writes the px = 0 and 1 units
template <int G, bool X2 = false>
__global__ void __launch_bounds__(LY_THREADS)
s2d_sources_kernel(const float *__restrict__ src, void *__restrict__ dst, int C, int cpad, int D, int H, int W,
                   size_t items) {
  const int D2 = D / 2, H2 = H / 2, W2 = W / 2, CGs = cpad / G;
  const size_t vol = (size_t)D * H * W;
  for (size_t i = (size_t)blockIdx.x * LY_THREADS + threadIdx.x; i < items; i += (size_t)gridDim.x * LY_THREADS) {
    const int x2 = (int)(i % W2);
    size_t r = i / W2;
    const int y2 = (int)(r % H2);
    r /= H2;
    const int cg = (int)(r % CGs);
    r /= CGs;
    const int pzy = (int)(r & 3);
    r >>= 2;  // b * D2 + z'
    const size_t b = r / D2, z2 = r - b * D2;
    const int pz = pzy >> 1, py = pzy & 1;
    const float *s = src + (((b * C + (size_t)cg * G) * D + 2 * z2 + pz) * H + 2 * y2 + py) * (size_t)W + 2 * x2;
    float x0[G], x1[G];
#pragma unroll
    for (int e = 0; e < G; ++e) {
      float2 t = make_float2(0.f, 0.f);
      if (cg * G + e < C) t = __ldg(reinterpret_cast<const float2 *>(s + e * vol));
      x0[e] = t.x;
      x1[e] = t.y;
    }
    const size_t u = ((r * (8 * CGs) + (size_t)(pzy * 2) * CGs + cg) * H2 + y2) * (size_t)W2 + x2;
    store_out<G, X2>(dst, u, r, (size_t)8 * CGs * H2 * W2, x0);
    store_out<G, X2>(dst, u + (size_t)CGs * H2 * W2, r, (size_t)8 * CGs * H2 * W2, x1);
  }
}

// 4x space-to-depth: one thread = one 16-byte unit = 8/G rows of 4 consecutive x of one (c, rz) plane
template <int G, bool X2 = false>
__global__ void __launch_bounds__(LY_THREADS)
s4d_blocked_kernel(const float *__restrict__ src, void *__restrict__ dst, int C, int D, int H, int W, size_t units) {
  const int D4 = D / 4, H4 = H / 4, W4 = W / 4;
  constexpr int UPP = 16 / G;  // units per (c, rz) plane of 16 (ry, rx) channels
  const int CGo = C * 4 * UPP;
  for (size_t u = (size_t)blockIdx.x * LY_THREADS + threadIdx.x; u < units; u += (size_t)gridDim.x * LY_THREADS) {
    const int x4 = (int)(u % W4);
    size_t r = u / W4;
    const int y4 = (int)(r % H4);
    r /= H4;
    const int cg = (int)(r % CGo);
    r /= CGo;  // b * D4 + z'
    const size_t b = r / D4, z4 = r - b * D4;
    const int h = cg % UPP, crz = cg / UPP, rz = crz & 3, c = crz >> 2;
    const float *s = src + (((b * C + c) * D + 4 * z4 + rz) * H + 4 * y4 + h * (G / 4)) * (size_t)W + 4 * x4;
    float x[G];
#pragma unroll
    for (int row = 0; row < G / 4; ++row) {
      const float4 t = __ldg(reinterpret_cast<const float4 *>(s + (size_t)row * W));
      x[row * 4 + 0] = t.x;
      x[row * 4 + 1] = t.y;
      x[row * 4 + 2] = t.z;
      x[row * 4 + 3] = t.w;
    }
    store_out<G, X2>(dst, u, r, (size_t)CGo * H4 * W4, x);
  }
}

__global__ void __launch_bounds__(LY_THREADS)
from_blocked_kernel(const float4 *__restrict__ src, float *__restrict__ dst, int C, int CG, int D, int H, int W,
                    size_t units) {
  const size_t plane = (size_t)H * W, vol = plane * D;
  for (size_t u = (size_t)blockIdx.x * LY_THREADS + threadIdx.x; u < units; u += (size_t)gridDim.x * LY_THREADS) {
    const size_t hw = u % plane;
    size_t r = u / plane;
    const int cg = (int)(r % CG);
    r /= CG;
    const size_t b = r / D, d = r - b * D;
    const float4 v = __ldg(src + u);
    float *o = dst + ((b * C + (size_t)cg * 4) * D + d) * plane + hw;
    const int c0 = cg * 4;
    if (c0 + 0 < C) o[0] = v.x;
    if (c0 + 1 < C) o[vol] = v.y;
    if (c0 + 2 < C) o[2 * vol] = v.z;
    if (c0 + 3 < C) o[3 * vol] = v.w;
  }
}

// blocked fp32 groups of 4 -> blocked fp16 groups of 8 (channel padding to a multiple of 8 is zero-filled)
__global__ void __launch_bounds__(LY_THREADS)
regroup_f16_kernel(const float4 *__restrict__ src, uint4 *__restrict__ dst, int cg4, int cg8, size_t plane, size_t units) {
  for (size_t u = (size_t)blockIdx.x * LY_THREADS + threadIdx.x; u < units; u += (size_t)gridDim.x * LY_THREADS) {
    const size_t hw = u % plane;
    size_t r = u / plane;
    const int g = (int)(r % cg8);
    r /= cg8;  // b * D + d
    const float4 *s = src + (r * cg4 + 2 * g) * plane + hw;
    const float4 a = __ldg(s);
    const float4 b = 2 * g + 1 < cg4 ? __ldg(s + plane) : make_float4(0.f, 0.f, 0.f, 0.f);
    const float x[8] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w};
    store_unit<8>(dst, u, x);
  }
}

// dst[m][i] = clamp(src[m][i] * scale, lo, hi), dst maps dst_stride floats apart (a channel of a wider tensor)
__global__ void __launch_bounds__(LY_THREADS)
scale_clamp_kernel(const float4 *__restrict__ src, float *__restrict__ dst, size_t n4, size_t dst_stride, size_t total4,
                   float scale, float lo, float hi) {
  for (size_t i = (size_t)blockIdx.x * LY_THREADS + threadIdx.x; i < total4; i += (size_t)gridDim.x * LY_THREADS) {
    const size_t m = i / n4, j = i - m * n4;
    float4 v = __ldg(src + i);
    v.x = fminf(fmaxf(__fmul_rn(v.x, scale), lo), hi);
    v.y = fminf(fmaxf(__fmul_rn(v.y, scale), lo), hi);
    v.z = fminf(fmaxf(__fmul_rn(v.z, scale), lo), hi);
    v.w = fminf(fmaxf(__fmul_rn(v.w, scale), lo), hi);
    st_stream_f4(dst + m * dst_stride + j * 4, v);
  }
}

// fp32 -> (lo, hi, hi) for the 3xTF32 scheme: hi = x rounded to TF32 (10-bit mantissa), lo = x - hi (exact in fp32).
// [BD][CG][H][W][4] -> [BD][3*CG][H][W][4] with the three blocks of CG groups in that order (weights: W_hi | W_lo | W_hi).
__device__ __forceinline__ float tf32_round(float x) {
  unsigned u;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(u) : "f"(x));
  return __uint_as_float(u);
}
__global__ void __launch_bounds__(LY_THREADS)
split3_kernel(const float4 *__restrict__ src, float4 *__restrict__ dst, int CG, size_t plane, size_t units) {
  for (size_t u = (size_t)blockIdx.x * LY_THREADS + threadIdx.x; u < units; u += (size_t)gridDim.x * LY_THREADS) {
    const size_t hw = u % plane;
    size_t r = u / plane;
    const int cg = (int)(r % CG);
    r /= CG;  // b * D + d
    const float4 v = __ldg(src + u);
    const float4 hi = make_float4(tf32_round(v.x), tf32_round(v.y), tf32_round(v.z), tf32_round(v.w));
    const float4 lo = make_float4(v.x - hi.x, v.y - hi.y, v.z - hi.z, v.w - hi.w);
    float4 *o = dst + (r * 3 * CG + cg) * plane + hw;
    o[0] = lo;  // small terms first: the tensor core's fp32 accumulator truncates, so the error of a step scales with
    o[(size_t)CG * plane] = hi;  // the partial sum it is added to; the two cross terms go in while that sum is ~2^-11 of
    o[(size_t)2 * CG * plane] = hi;  // its final size
  }
}

static unsigned ly_grid(size_t n) {
  const size_t blocks = (n + LY_THREADS - 1) / LY_THREADS;
  const size_t cap = (size_t)sm_count() * 8 * 16;  // grid-stride beyond ~16 waves of 8 CTAs per SM
  return (unsigned)(blocks < cap ? (blocks ? blocks : 1) : cap);
}

}  // namespace gb

using namespace gb;

namespace gb {
// fp32 blocked [BD][cg4][H][W][4] -> fp16 [BD][2][cg8][H][W][8]: part 0 = hi = fp16(a) (round to nearest), part 1 = lo' =
// fp16((a - hi) * 2^11): a = hi + lo' * 2^-11 to ~2^-22 |a| (absolute floor ~1.5e-11).  The activation operand of the
// fp32-accurate "f16x2" convolution mode (csrc/convt3d.cu X2).  |a| > 65504 becomes inf (and stays visible in the output).
__global__ void __launch_bounds__(LY_THREADS)
split2_f16_kernel(const float4 *__restrict__ src, uint4 *__restrict__ dst, int cg4, int cg8, size_t plane, size_t units) {
  for (size_t u = (size_t)blockIdx.x * LY_THREADS + threadIdx.x; u < units; u += (size_t)gridDim.x * LY_THREADS) {
    const size_t hw = u % plane;
    size_t r = u / plane;
    const int g = (int)(r % cg8);
    r /= cg8;  // b * D + d
    const float4 *s = src + (r * cg4 + 2 * g) * plane + hw;
    const float4 a = __ldg(s);
    const float4 b = 2 * g + 1 < cg4 ? __ldg(s + plane) : make_float4(0.f, 0.f, 0.f, 0.f);
    const float x[8] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w};
    uint4 ph, pl;
    split_hi_lo8(x, ph, pl);
    uint4 *o = dst + ((r * 2) * cg8 + g) * plane + hw;
    o[0] = ph;
    o[(size_t)cg8 * plane] = pl;
  }
}
}  // namespace gb


// mode 0: to_blocked, 1: s2d_blocked, 2: s2d_sources (cpad = padded channels per sub-volume; ignored otherwise),
// 3: s4d_blocked.
// group 4 -> fp32 units, 8 -> fp16 units.  src is contiguous NCDHW fp32.
extern "C" int genre_b200_ncdhw_to_blocked(const float *src, int64_t B, int64_t C, int64_t D, int64_t H, int64_t W,
                                           int mode, int group_in, int cpad, void *dst, void *stream) {
  int group = group_in;
  GB_REQUIRE(src && dst, GENRE_B200_EINVAL, "to_blocked: null pointer");
  GB_REQUIRE(B > 0 && C > 0 && D > 0 && H > 0 && W > 0, GENRE_B200_EINVAL, "to_blocked: empty tensor");
  GB_REQUIRE(group == 4 || group == 8 || group == 16, GENRE_B200_EINVAL,
             "to_blocked: group must be 4 (fp32), 8 (fp16) or 16 (fp16 hi/lo parts of 8 channels: dst [B*D'][2][cg][H'][W'][8])");
  const bool x2 = group == 16;
  if (x2) group = 8;
  GB_REQUIRE(aligned16(dst), GENRE_B200_EALIGN, "to_blocked: dst must be 16-byte aligned");
  cudaStream_t st = as_stream(stream);
  if (mode == 0) {
    GB_REQUIRE(C % group == 0, GENRE_B200_EINVAL, "to_blocked: C=%lld not a multiple of %d", (long long)C, group);
    const size_t units = (size_t)(B * D * (C / group) * H * W);
    if (group == 4) to_blocked_kernel<4><<<ly_grid(units), LY_THREADS, 0, st>>>(src, dst, (int)C, (int)D, (int)H, (int)W, units);
    else if (x2) to_blocked_kernel<8, true><<<ly_grid(units), LY_THREADS, 0, st>>>(src, dst, (int)C, (int)D, (int)H, (int)W, units);
    else to_blocked_kernel<8><<<ly_grid(units), LY_THREADS, 0, st>>>(src, dst, (int)C, (int)D, (int)H, (int)W, units);
    return check_launch("to_blocked kernel");
  }
  GB_REQUIRE(D % 2 == 0 && H % 2 == 0 && W % 2 == 0, GENRE_B200_EINVAL, "space-to-depth: odd extent");
  GB_REQUIRE(((uintptr_t)src & 7) == 0, GENRE_B200_EALIGN, "space-to-depth: src must be 8-byte aligned");
  if (mode == 1) {
    const size_t cells = (size_t)(B * C * (D / 2) * (H / 2) * (W / 2));
    int cgo = (int)(C * 8 / group);
    if (cpad > C * 8) {  // pad the 8C space-to-depth channels with zero groups up to cpad channels
      GB_REQUIRE(cpad % group == 0, GENRE_B200_EINVAL, "s2d_blocked: cpad=%d not a multiple of %d", cpad, group);
      cgo = cpad / group;
      cudaError_t e = cudaMemsetAsync(dst, 0, (size_t)(B * (D / 2)) * cgo * (size_t)((H / 2) * (W / 2)) * 16 * (x2 ? 2 : 1), st);
      if (e != cudaSuccess) return fail_arg((int)e, "s2d_blocked: memset: %s", cudaGetErrorString(e));
    }
    if (group == 4) s2d_blocked_kernel<4><<<ly_grid(cells), LY_THREADS, 0, st>>>(src, dst, (int)C, (int)D, (int)H, (int)W, cells, cgo);
    else if (x2) s2d_blocked_kernel<8, true><<<ly_grid(cells), LY_THREADS, 0, st>>>(src, dst, (int)C, (int)D, (int)H, (int)W, cells, cgo);
    else s2d_blocked_kernel<8><<<ly_grid(cells), LY_THREADS, 0, st>>>(src, dst, (int)C, (int)D, (int)H, (int)W, cells, cgo);
    return check_launch("s2d_blocked kernel");
  }
  if (mode == 3) {
    GB_REQUIRE(D % 4 == 0 && H % 4 == 0 && W % 4 == 0 && aligned16(src), GENRE_B200_EINVAL,
               "4x space-to-depth: extents must be multiples of 4 and src 16-byte aligned");
    const size_t units = (size_t)(B * C * 64 / group * (D / 4) * (H / 4) * (W / 4));
    if (group == 4) s4d_blocked_kernel<4><<<ly_grid(units), LY_THREADS, 0, st>>>(src, dst, (int)C, (int)D, (int)H, (int)W, units);
    else if (x2) s4d_blocked_kernel<8, true><<<ly_grid(units), LY_THREADS, 0, st>>>(src, dst, (int)C, (int)D, (int)H, (int)W, units);
    else s4d_blocked_kernel<8><<<ly_grid(units), LY_THREADS, 0, st>>>(src, dst, (int)C, (int)D, (int)H, (int)W, units);
    return check_launch("s4d_blocked kernel");
  }
  GB_REQUIRE(mode == 2, GENRE_B200_EINVAL, "to_blocked: unknown mode %d", mode);
  GB_REQUIRE(cpad >= C && cpad % group == 0, GENRE_B200_EINVAL, "s2d_sources: cpad=%d must be >= C and a multiple of %d", cpad, group);
  const size_t items = (size_t)(B * (D / 2) * 4 * (cpad / group) * (H / 2) * (W / 2));
  if (group == 4) s2d_sources_kernel<4><<<ly_grid(items), LY_THREADS, 0, st>>>(src, dst, (int)C, cpad, (int)D, (int)H, (int)W, items);
  else if (x2) s2d_sources_kernel<8, true><<<ly_grid(items), LY_THREADS, 0, st>>>(src, dst, (int)C, cpad, (int)D, (int)H, (int)W, items);
  else s2d_sources_kernel<8><<<ly_grid(items), LY_THREADS, 0, st>>>(src, dst, (int)C, cpad, (int)D, (int)H, (int)W, items);
  return check_launch("s2d_sources kernel");
}

// blocked fp32 [B*D][cg][H][W][4] -> contiguous NCDHW [B,C,D,H,W] (C <= 4*cg)
extern "C" int genre_b200_blocked_to_ncdhw(const float *src, int cg, int64_t B, int64_t C, int64_t D, int64_t H,
                                           int64_t W, float *dst, void *stream) {
  GB_REQUIRE(src && dst, GENRE_B200_EINVAL, "from_blocked: null pointer");
  GB_REQUIRE(B > 0 && C > 0 && D > 0 && H > 0 && W > 0 && cg > 0 && C <= 4 * (int64_t)cg && C > 4 * (int64_t)(cg - 1),
             GENRE_B200_EINVAL, "from_blocked: bad shape (C=%lld, cg=%d)", (long long)C, cg);
  GB_REQUIRE(aligned16(src), GENRE_B200_EALIGN, "from_blocked: src must be 16-byte aligned");
  const size_t units = (size_t)(B * D * cg * H * W);
  from_blocked_kernel<<<ly_grid(units), LY_THREADS, 0, as_stream(stream)>>>((const float4 *)src, dst, (int)C, cg, (int)D,
                                                                           (int)H, (int)W, units);
  return check_launch("from_blocked kernel");
}

// blocked fp32 [BD][cg4][H][W][4] -> blocked fp16 [BD][(cg4+1)/2][H][W][8] (operand of the fp16 tensor-core kernels)
extern "C" int genre_b200_blocked_f32_to_f16(const float *src, int cg4, int64_t BD, int64_t H, int64_t W, void *dst,
                                             void *stream) {
  GB_REQUIRE(src && dst && cg4 > 0 && BD > 0 && H > 0 && W > 0, GENRE_B200_EINVAL, "blocked_f32_to_f16: bad argument");
  GB_REQUIRE(aligned16(src) && aligned16(dst), GENRE_B200_EALIGN, "blocked_f32_to_f16: alignment");
  const int cg8 = (cg4 + 1) / 2;
  const size_t plane = (size_t)(H * W), units = (size_t)BD * cg8 * plane;
  regroup_f16_kernel<<<ly_grid(units), LY_THREADS, 0, as_stream(stream)>>>((const float4 *)src, (uint4 *)dst, cg4, cg8, plane,
                                                                          units);
  return check_launch("regroup_f16 kernel");
}

// dst[m][:] = clamp(src[m][:] * scale, lo, hi) for `maps` maps of n floats, dst maps dst_map_stride floats apart:
// GenRe's `clamp(proj_depth / 50, 1e-5, 1 - 1e-5)` + torch.cat (genre_full_model.py:126-127) as one pass.
extern "C" int genre_b200_scale_clamp_strided(const float *src, int64_t maps, int64_t n, float scale, float lo, float hi,
                                              float *dst, int64_t dst_map_stride, void *stream) {
  GB_REQUIRE(src && dst && maps > 0 && n > 0 && n % 4 == 0 && dst_map_stride >= n && dst_map_stride % 4 == 0,
             GENRE_B200_EINVAL, "scale_clamp: bad argument (n and stride must be multiples of 4)");
  GB_REQUIRE(aligned16(src) && aligned16(dst), GENRE_B200_EALIGN, "scale_clamp: alignment");
  const size_t n4 = (size_t)n / 4, total4 = n4 * (size_t)maps;
  scale_clamp_kernel<<<ly_grid(total4), LY_THREADS, 0, as_stream(stream)>>>((const float4 *)src, dst, n4,
                                                                           (size_t)dst_map_stride, total4, scale, lo, hi);
  return check_launch("scale_clamp kernel");
}

// blocked fp32 [BD][cg][H][W][4] -> [BD][3*cg][H][W][4] = (lo | hi | hi) blocks, hi = TF32-rounded value, lo = the
// remainder: the activation operand of the fp32-accurate "3xTF32" convolution mode (A_lo*W_hi + A_hi*W_lo + A_hi*W_hi)
extern "C" int genre_b200_blocked_split3(const float *src, int cg, int64_t BD, int64_t H, int64_t W, float *dst,
                                         void *stream) {
  GB_REQUIRE(src && dst && cg > 0 && BD > 0 && H > 0 && W > 0, GENRE_B200_EINVAL, "blocked_split3: bad argument");
  GB_REQUIRE(aligned16(src) && aligned16(dst), GENRE_B200_EALIGN, "blocked_split3: alignment");
  const size_t plane = (size_t)(H * W), units = (size_t)BD * cg * plane;
  split3_kernel<<<ly_grid(units), LY_THREADS, 0, as_stream(stream)>>>((const float4 *)src, (float4 *)dst, cg, plane, units);
  return check_launch("split3 kernel");
}

// blocked fp32 [BD][cg4][H][W][4] -> fp16 [BD][2][(cg4+1)/2][H][W][8] = (hi | lo' = (a - hi) * 2^11) parts: the activation
// operand of the fp32-accurate "f16x2" convolution mode (2 MMAs per K step: A_hi x [W_hi | W_lo'] and A_lo' x W_hi)
extern "C" int genre_b200_blocked_split2_f16(const float *src, int cg4, int64_t BD, int64_t H, int64_t W, void *dst,
                                             void *stream) {
  GB_REQUIRE(src && dst && cg4 > 0 && BD > 0 && H > 0 && W > 0, GENRE_B200_EINVAL, "blocked_split2_f16: bad argument");
  GB_REQUIRE(aligned16(src) && aligned16(dst), GENRE_B200_EALIGN, "blocked_split2_f16: alignment");
  const int cg8 = (cg4 + 1) / 2;
  const size_t plane = (size_t)(H * W), units = (size_t)BD * cg8 * plane;
  split2_f16_kernel<<<ly_grid(units), LY_THREADS, 0, as_stream(stream)>>>((const float4 *)src, (uint4 *)dst, cg4, cg8, plane, units);
  return check_launch("split2_f16 kernel");
}
