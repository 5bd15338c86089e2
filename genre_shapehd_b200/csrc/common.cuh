// common.cuh — shared helpers for libgenre_b200 (sm_90a only; no torch, no CPU fallback).
#pragma once
#include <cuda_runtime.h>
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

__device__ __forceinline__ unsigned lanemask_lt() {
  unsigned m;
  asm("mov.u32 %0, %%lanemask_lt;" : "=r"(m));
  return m;
}

}  // namespace gb
