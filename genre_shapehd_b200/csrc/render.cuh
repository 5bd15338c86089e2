// render.cuh — device helpers shared by the volume renderers (render_sph.cu, render_cam.cu): trilinear taps with zero
// padding, the clamp constants of the stop probabilities, and the warp scans along a ray.
#pragma once
#include "common.cuh"

namespace gb {

struct Taps {
  int base;        // linear index of corner (x0, y0, z0); may be out of range, see masks
  float w[8];      // weights in order (x,y,z) = 000, 001, 010, 011, 100, 101, 110, 111
  unsigned valid;  // bit i set if tap i is inside the volume
};

// taps of the continuous voxel coordinate (fx, fy, fz): voxel i sits at coordinate i, x0 = floor(f)
__device__ __forceinline__ void make_taps_at(float fx, float fy, float fz, int R, Taps &t) {
  const float x0f = floorf(fx), y0f = floorf(fy), z0f = floorf(fz);
  // clamp before the int conversion so far-away samples stay well defined
  const int x0 = (int)fminf(fmaxf(x0f, -2.0f), (float)R), y0 = (int)fminf(fmaxf(y0f, -2.0f), (float)R),
            z0 = (int)fminf(fmaxf(z0f, -2.0f), (float)R);
  const float wx1 = fx - x0f, wx0 = (x0f + 1.0f) - fx;
  const float wy1 = fy - y0f, wy0 = (y0f + 1.0f) - fy;
  const float wz1 = fz - z0f, wz0 = (z0f + 1.0f) - fz;
  t.base = (x0 * R + y0) * R + z0;
  t.w[0] = wx0 * wy0 * wz0; t.w[1] = wx0 * wy0 * wz1; t.w[2] = wx0 * wy1 * wz0; t.w[3] = wx0 * wy1 * wz1;
  t.w[4] = wx1 * wy0 * wz0; t.w[5] = wx1 * wy0 * wz1; t.w[6] = wx1 * wy1 * wz0; t.w[7] = wx1 * wy1 * wz1;
  const unsigned Rm = (unsigned)(R - 1);
  if (((unsigned)x0 < Rm) & ((unsigned)y0 < Rm) & ((unsigned)z0 < Rm)) {  // all 8 taps inside: the common case
    t.valid = 0xFFu;
    return;
  }
  const bool vx0 = (unsigned)x0 < (unsigned)R, vx1 = (unsigned)(x0 + 1) < (unsigned)R;
  const bool vy0 = (unsigned)y0 < (unsigned)R, vy1 = (unsigned)(y0 + 1) < (unsigned)R;
  const bool vz0 = (unsigned)z0 < (unsigned)R, vz1 = (unsigned)(z0 + 1) < (unsigned)R;
  t.valid = (unsigned)(vx0 & vy0 & vz0) | ((unsigned)(vx0 & vy0 & vz1) << 1) | ((unsigned)(vx0 & vy1 & vz0) << 2) |
            ((unsigned)(vx0 & vy1 & vz1) << 3) | ((unsigned)(vx1 & vy0 & vz0) << 4) |
            ((unsigned)(vx1 & vy0 & vz1) << 5) | ((unsigned)(vx1 & vy1 & vz0) << 6) |
            ((unsigned)(vx1 & vy1 & vz1) << 7);
}

__device__ __forceinline__ int tap_offset(int i, int R) {
  return ((i >> 2) & 1) * R * R + ((i >> 1) & 1) * R + (i & 1);
}

// Optional transform of every voxel value as it is fetched: v -> clamp(v * scale, lo, hi).  GenRe renders
// clamp(proj * 50, 1e-5, 1 - 1e-5) (depth_pred_with_sph_inpaint.py:124): applying the two elementwise ops here (same
// fp32 operations, same order) removes two dense passes over the volume.  Out-of-volume taps stay 0 (zero padding).
struct VoxPre {
  float scale, lo, hi;
};
template <bool PRE>
__device__ __forceinline__ float fetch_vox(const float *__restrict__ p, const VoxPre &pre) {
  const float v = __ldg(p);
  return PRE ? fminf(fmaxf(__fmul_rn(v, pre.scale), pre.lo), pre.hi) : v;
}

template <bool PRE>
__device__ __forceinline__ float sample_trilinear(const float *__restrict__ vol, const Taps &t, int R, const VoxPre &pre) {
  float acc = 0.0f;
  if (t.valid == 0xFFu) {  // interior: 4 pairs of z-adjacent taps
#pragma unroll
    for (int i = 0; i < 8; ++i) acc = fmaf(fetch_vox<PRE>(vol + t.base + tap_offset(i, R), pre), t.w[i], acc);
  } else if (t.valid) {
#pragma unroll
    for (int i = 0; i < 8; ++i)
      if (t.valid & (1u << i)) acc = fmaf(fetch_vox<PRE>(vol + t.base + tap_offset(i, R), pre), t.w[i], acc);
  }
  return acc;
}

// sample_trilinear<false>'s raw (the same fmas in the same order, bit for bit) and d raw / d f in voxel units at the
// coordinate (fx, fy, fz) the taps were made from: the derivative of the cell make_taps_at selects (on a voxel face,
// the one-sided derivative of the cell above it).  Out-of-volume taps are 0.
__device__ __forceinline__ float sample_trilinear_grad(const float *__restrict__ vol, const Taps &t, int R, float fx,
                                                       float fy, float fz, float &dx, float &dy, float &dz) {
  float v[8], acc = 0.0f;
  if (t.valid == 0xFFu) {
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      v[i] = __ldg(vol + t.base + tap_offset(i, R));
      acc = fmaf(v[i], t.w[i], acc);
    }
  } else {
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      v[i] = 0.0f;
      if (t.valid & (1u << i)) {
        v[i] = __ldg(vol + t.base + tap_offset(i, R));
        acc = fmaf(v[i], t.w[i], acc);
      }
    }
  }
  const float x0f = floorf(fx), y0f = floorf(fy), z0f = floorf(fz);
  const float wx1 = fx - x0f, wx0 = (x0f + 1.0f) - fx;
  const float wy1 = fy - y0f, wy0 = (y0f + 1.0f) - fy;
  const float wz1 = fz - z0f, wz0 = (z0f + 1.0f) - fz;
  // tap i: bit 2 = x, bit 1 = y, bit 0 = z
  dx = fmaf(v[7] - v[3], wy1 * wz1, fmaf(v[6] - v[2], wy1 * wz0, fmaf(v[5] - v[1], wy0 * wz1, (v[4] - v[0]) * (wy0 * wz0))));
  dy = fmaf(v[7] - v[5], wx1 * wz1, fmaf(v[6] - v[4], wx1 * wz0, fmaf(v[3] - v[1], wx0 * wz1, (v[2] - v[0]) * (wx0 * wz0))));
  dz = fmaf(v[7] - v[6], wx1 * wy1, fmaf(v[5] - v[4], wx1 * wy0, fmaf(v[3] - v[2], wx0 * wy1, (v[1] - v[0]) * (wx0 * wy0))));
  return acc;
}

// sample_trilinear_grad's raw and d raw / d f (the same operations in the same order, bit for bit), and the three mixed
// second partials hxy = d2 raw / df_x df_y, hxz, hyz of the same cell (the interpolant's Hessian in f; its diagonal is
// 0).  Each mixed partial is the cell's second difference across its two axes, weighted along the third.
__device__ __forceinline__ float sample_trilinear_hess(const float *__restrict__ vol, const Taps &t, int R, float fx,
                                                       float fy, float fz, float &dx, float &dy, float &dz, float &hxy,
                                                       float &hxz, float &hyz) {
  float v[8], acc = 0.0f;
  if (t.valid == 0xFFu) {
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      v[i] = __ldg(vol + t.base + tap_offset(i, R));
      acc = fmaf(v[i], t.w[i], acc);
    }
  } else {
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      v[i] = 0.0f;
      if (t.valid & (1u << i)) {
        v[i] = __ldg(vol + t.base + tap_offset(i, R));
        acc = fmaf(v[i], t.w[i], acc);
      }
    }
  }
  const float x0f = floorf(fx), y0f = floorf(fy), z0f = floorf(fz);
  const float wx1 = fx - x0f, wx0 = (x0f + 1.0f) - fx;
  const float wy1 = fy - y0f, wy0 = (y0f + 1.0f) - fy;
  const float wz1 = fz - z0f, wz0 = (z0f + 1.0f) - fz;
  // tap i: bit 2 = x, bit 1 = y, bit 0 = z
  dx = fmaf(v[7] - v[3], wy1 * wz1, fmaf(v[6] - v[2], wy1 * wz0, fmaf(v[5] - v[1], wy0 * wz1, (v[4] - v[0]) * (wy0 * wz0))));
  dy = fmaf(v[7] - v[5], wx1 * wz1, fmaf(v[6] - v[4], wx1 * wz0, fmaf(v[3] - v[1], wx0 * wz1, (v[2] - v[0]) * (wx0 * wz0))));
  dz = fmaf(v[7] - v[6], wx1 * wy1, fmaf(v[5] - v[4], wx1 * wy0, fmaf(v[3] - v[2], wx0 * wy1, (v[1] - v[0]) * (wx0 * wy0))));
  hxy = fmaf((v[7] - v[3]) - (v[5] - v[1]), wz1, ((v[6] - v[2]) - (v[4] - v[0])) * wz0);
  hxz = fmaf((v[7] - v[3]) - (v[6] - v[2]), wy1, ((v[5] - v[1]) - (v[4] - v[0])) * wy0);
  hyz = fmaf((v[7] - v[5]) - (v[6] - v[4]), wx1, ((v[3] - v[1]) - (v[2] - v[0])) * wx0);
  return acc;
}

// exclusive product over the warp's lanes; total = the product of all 32
__device__ __forceinline__ float warp_excl_prod32(float v, float &total) {
  float incl = v;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    const float u = __shfl_up_sync(0xffffffffu, incl, d);
    if ((threadIdx.x & 31) >= d) incl *= u;
  }
  total = __shfl_sync(0xffffffffu, incl, 31);
  float excl = __shfl_up_sync(0xffffffffu, incl, 1);
  if ((threadIdx.x & 31) == 0) excl = 1.0f;
  return excl;
}

// exclusive suffix sum over the warp's lanes; total = the sum of all 32
__device__ __forceinline__ float warp_excl_suffix_sum32(float v, float &total) {
  const int lane = threadIdx.x & 31;
  float incl = v;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    const float u = __shfl_down_sync(0xffffffffu, incl, d);
    if (lane + d < 32) incl += u;
  }
  total = __shfl_sync(0xffffffffu, incl, 0);
  float excl = __shfl_down_sync(0xffffffffu, incl, 1);
  if (lane == 31) excl = 0.0f;
  return excl;
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// the stop probabilities' clamp (spherical_proj.py:66), at the fp32 constants torch.clamp uses on fp32
constexpr float RS_PMIN = 1e-5f;
constexpr float RS_PMAX = (float)(1.0 - 1e-5);

}  // namespace gb
