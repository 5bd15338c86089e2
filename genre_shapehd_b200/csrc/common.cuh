// common.cuh — shared helpers for libgenre_b200 (sm_90a only; no torch, no CPU fallback).
#pragma once
#include <cuda_runtime.h>
#include <cuda_fp16.h>
#include <stdint.h>
#include <stddef.h>
#include <stdio.h>
#include <stdarg.h>
#include "../../include/genre_b200.h"

namespace gb {

// ---- error reporting (thread-local message behind genre_b200_last_error) -------------------------
void set_error(const char *fmt, ...);
int fail_arg(int code, const char *fmt, ...);
int check_launch(const char *what);  // cudaPeekAtLastError -> 0 or the cudaError_t (message recorded)
const char *last_error();

// streaming multiprocessors of the current device (cached per device): grid sizes that aim at whole waves use it
int sm_count();

#define GB_REQUIRE(cond, code, ...)                      \
  do {                                                   \
    if (!(cond)) return gb::fail_arg((code), __VA_ARGS__); \
  } while (0)

static inline bool aligned16(const void *p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }
static inline cudaStream_t as_stream(void *s) { return reinterpret_cast<cudaStream_t>(s); }

// ---- device helpers --------------------------------------------------------------------------------
// FLOOR_I of the reference (back_projection_kernel.cu:36-37): truncation, minus one for negatives.
// Not a true floor for negative integers; kept because it decides which points are in bounds.
__device__ __forceinline__ int floor_i_ref(float a) { return a < 0.0f ? (int)a - 1 : (int)a; }

// streaming 16-byte store: written once, never re-read by this kernel -> do not allocate in L1
__device__ __forceinline__ void st_stream_f4(float *p, float4 v) {
  asm volatile("st.global.cs.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(p), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w)
               : "memory");
}
__device__ __forceinline__ void st_stream_f1(float *p, float v) {
  asm volatile("st.global.cs.f32 [%0], %1;" ::"l"(p), "f"(v) : "memory");
}

// 8 fp16 -> one 16-byte unit
__device__ __forceinline__ uint4 pack_half8(const __half (&h)[8]) {
  uint32_t w[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) w[i] = (uint32_t)__half_as_ushort(h[2 * i]) | ((uint32_t)__half_as_ushort(h[2 * i + 1]) << 16);
  return make_uint4(w[0], w[1], w[2], w[3]);
}

// 8 fp32 -> one 16-byte unit of 8 fp16, each rounded to nearest (the operand of the single-pass f16 mode)
__device__ __forceinline__ uint4 pack_f16x8(const float (&x)[8]) {
  __half h[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) h[i] = __float2half_rn(x[i]);
  return pack_half8(h);
}

// The activation operand of the fp32-accurate f16x2 convolution mode for 8 channels: hi = fp16(a), lo' = fp16((a - hi) * 2^11),
// a = hi + lo' * 2^-11 to 2^-22 |a| while |a| >= 2^-14 (fp16's smallest normal).  Below that, fp16's subnormal spacing (2^-24)
// in lo' makes the error an absolute floor instead: |a - hi - lo' * 2^-11| <= 2^-22 |a| + 2^-36 for every finite |a| < 65520.
// Every producer of this operand (the layout kernels and the convolution epilogues) calls this
// function: the intrinsics are never contracted into an FMA with the code that computed `a`, so the same fp32 value gives the
// same bits wherever it is split.  |a| >= 65520 rounds hi to inf (and stays visible in the output); up to there hi is finite.
__device__ __forceinline__ void split_hi_lo8(const float (&x)[8], uint4 &hi, uint4 &lo) {
  __half h[8], l[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    h[i] = __float2half_rn(x[i]);
    l[i] = __float2half_rn(__fmul_rn(__fsub_rn(x[i], __half2float(h[i])), 2048.0f));
  }
  hi = pack_half8(h);
  lo = pack_half8(l);
}

// The face rule of genre_b200_mesh_voxelize and genre_b200_winding_number: a face (p[0], p[1], p[2]) is kept iff every
// vertex coordinate is finite and its fp64 normal e1 x e2 (e1 = p1 - p0, e2 = p2 - p0 from the fp32 vertices, one rounding
// per operation, nx = e1y*e2z - e1z*e2y, ...: genre_b200_surface_sample's weight order) is not exactly 0.  A skipped face
// contributes nothing.
__device__ __forceinline__ bool mesh_face_kept(const float (&p)[3][3]) {
  bool finite = true;
#pragma unroll
  for (int k = 0; k < 3; ++k)
#pragma unroll
    for (int a = 0; a < 3; ++a) finite = finite && isfinite(p[k][a]);
  if (!finite) return false;
  double e1[3], e2[3];
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    e1[a] = __dsub_rn((double)p[1][a], (double)p[0][a]);
    e2[a] = __dsub_rn((double)p[2][a], (double)p[0][a]);
  }
  const double nx = __dsub_rn(__dmul_rn(e1[1], e2[2]), __dmul_rn(e1[2], e2[1]));
  const double ny = __dsub_rn(__dmul_rn(e1[2], e2[0]), __dmul_rn(e1[0], e2[2]));
  const double nz = __dsub_rn(__dmul_rn(e1[0], e2[1]), __dmul_rn(e1[1], e2[0]));
  return !(nx == 0.0 && ny == 0.0 && nz == 0.0);
}

__device__ __forceinline__ unsigned lanemask_lt() {
  unsigned m;
  asm("mov.u32 %0, %%lanemask_lt;" : "=r"(m));
  return m;
}

}  // namespace gb
