// convt_c1_wgrad.cu — weight gradient of ConvTranspose3d(Cin -> 1, k=4, s=2, p=1), the last layer of every decoder
// (Unet_3D.dec6 networks/networks.py:167-168, VoxelDecoder main.17 :57, VoxelGenerator :98).
//
//   out[b, 2i - 1 + k] += x[b, ci, i] * W[ci, k]      =>      dW[ci, k] = sum_{b, i} x[b, ci, i] * gy[b, 2i - 1 + k]
//
// i.e. a [Cin x P] x [P x 64] product with P = B*D*H*W input positions (1 M at B=4, 64^3) and the right operand an
// im2col of the ONE-channel output gradient.  cuDNN answers this shape with `wgrad2d_grouped_direct_kernel`: 40.7 ms of a
// 60 ms Unet_3D training step at B=4 (profiles/r01_train_unet_launches.csv).  It is 2.7 GMAC over 200 MB: anything
// reasonable is a thousand times faster.  Here a CTA owns (b, z, 8 rows): the 4 x 18 x (2W+2) window of gy and the
// Cin x 8 x W slab of x sit in shared memory; thread (tap k, channel lane) keeps Cin/4 partial sums in registers over the
// slab's positions (x reads are warp broadcasts), CTAs are persistent over slabs, and the partials go to a workspace
// that a second kernel reduces in a fixed order: the result is bitwise reproducible.
#include "common.cuh"

namespace gb {

// CTAs of a weight-gradient launch, two per SM: the workspace holds one partial sum per CTA, so its size and the grid
// come from this one value
static int wgrad_max_ctas() { return 2 * sm_count(); }

constexpr int WG_THREADS = 256;   // 64 taps x 4 channel lanes
constexpr int WG_ROWS = 8;        // input rows per slab
constexpr int WG_MAX_CPT = 16;    // channels per thread (Cin <= 64)

// gy window geometry in shared memory: 4 planes x (2*ROWS+2) rows x (2W+2) columns with a 1-voxel halo; the row pitch is
// padded to 4 (mod 32) words and the plane pitch to 16 (mod 32) so that the 64 taps (kz,ky,kx) of one position fall into
// distinct banks (bank = 16 kz + 4 ky + kx for 32 consecutive taps)
struct GyWindow {
  int rows, pitch, plane;
};
__host__ __device__ inline GyWindow gy_window(int W) {
  GyWindow g;
  g.rows = 2 * WG_ROWS + 2;
  int p = 2 * W + 2;
  while ((p & 31) != 4) ++p;
  g.pitch = p;
  int pl = g.rows * p;
  while ((pl & 31) != 16) ++pl;
  g.plane = pl;
  return g;
}

template <int CPT>
__global__ void __launch_bounds__(WG_THREADS)
convt_c1_wgrad_kernel(const float *__restrict__ x, const float *__restrict__ gy, int Cin, int D, int H, int W, int n_slabs,
                      float *__restrict__ partial /* [gridDim.x][Cin][64] */) {
  extern __shared__ float smem[];
  const GyWindow gw = gy_window(W);
  const int GW = 2 * W + 2, GR = gw.rows;
  float *s_g = smem;                               // [4][plane]: rows of `pitch` words
  float *s_x = smem + 4 * gw.plane;                // [Cin][WG_ROWS * W]
  const int tid = threadIdx.x, k = tid & 63, lane = tid >> 6;
  const int kz = k >> 4, ky = (k >> 2) & 3, kx = k & 3;
  const int Do = 2 * D, Ho = 2 * H, Wo = 2 * W;
  const int slabs_per_map = D * (H / WG_ROWS);
  float acc[CPT];
#pragma unroll
  for (int j = 0; j < CPT; ++j) acc[j] = 0.0f;

  for (int slab = blockIdx.x; slab < n_slabs; slab += gridDim.x) {
    const int b = slab / slabs_per_map, r = slab - b * slabs_per_map;
    const int z = r / (H / WG_ROWS), y0 = (r - z * (H / WG_ROWS)) * WG_ROWS;
    __syncthreads();  // previous slab fully consumed
    // gy window: planes 2z-1 .. 2z+2, rows 2y0-1 .. 2y0+2*ROWS, columns -1 .. 2W
    const float *gmap = gy + (size_t)b * Do * Ho * Wo;
    for (int i = tid; i < 4 * GR * GW; i += WG_THREADS) {
      const int c = i % GW, rr = (i / GW) % GR, pl = i / (GW * GR);
      const int oz = 2 * z - 1 + pl, oy = 2 * y0 - 1 + rr, ox = c - 1;
      const bool ok = (oz >= 0) & (oz < Do) & (oy >= 0) & (oy < Ho) & (ox >= 0) & (ox < Wo);
      s_g[pl * gw.plane + rr * gw.pitch + c] = ok ? __ldg(gmap + ((size_t)oz * Ho + oy) * Wo + ox) : 0.0f;
    }
    const int npos = WG_ROWS * W;
    for (int i = tid; i < Cin * npos; i += WG_THREADS) {
      const int ci = i / npos, p = i - ci * npos;
      s_x[i] = __ldg(x + ((((size_t)b * Cin + ci) * D + z) * H + y0) * (size_t)W + p);
    }
    __syncthreads();
    const float *gk = s_g + kz * gw.plane + ky * gw.pitch + kx;  // tap k of position (yy, xx): gk[2*yy*pitch + 2*xx]
    for (int yy = 0; yy < WG_ROWS; ++yy) {
      const float *grow = gk + 2 * yy * gw.pitch;
      const float *xrow = s_x + yy * W;
      for (int xx = 0; xx < W; ++xx) {
        const float g = grow[2 * xx];
#pragma unroll
        for (int j = 0; j < CPT; ++j) {
          const int ci = lane + 4 * j;
          if (ci < Cin) acc[j] = fmaf(xrow[ci * npos + xx], g, acc[j]);
        }
      }
    }
  }
  float *out = partial + (size_t)blockIdx.x * Cin * 64;
#pragma unroll
  for (int j = 0; j < CPT; ++j) {
    const int ci = lane + 4 * j;
    if (ci < Cin) out[ci * 64 + k] = acc[j];
  }
}

__global__ void __launch_bounds__(256)
convt_c1_wgrad_reduce_kernel(const float *__restrict__ partial, int n_parts, int n_out, float *__restrict__ dW) {
  const int i = blockIdx.x * 256 + threadIdx.x;
  if (i >= n_out) return;
  float s = 0.0f;
  for (int p = 0; p < n_parts; ++p) s += partial[(size_t)p * n_out + i];  // fixed order
  dW[i] = s;
}

// input gradient of the same layer: dx[b, ci, i] = sum_k W[ci, k] * gy[b, 2i - 1 + k]  (a Conv3d(1 -> Cin, k4, s2, p1) of
// gy; cuDNN: 2.5 ms at B=4).  Same slab and gy window; a thread owns 2 positions, keeps their 64 taps of gy in registers
// and walks the channels with broadcast reads of W from shared memory; stores are coalesced along x.
__global__ void __launch_bounds__(WG_THREADS)
convt_c1_dgrad_kernel(const float *__restrict__ gy, const float *__restrict__ weight /* [Cin][64] */, int Cin, int D, int H,
                      int W, float *__restrict__ dx) {
  extern __shared__ float smem[];
  const GyWindow gw = gy_window(W);
  const int GW = 2 * W + 2, GR = gw.rows;
  float *s_g = smem;
  float *s_w = smem + 4 * gw.plane;  // [Cin][64]
  const int tid = threadIdx.x;
  const int Do = 2 * D, Ho = 2 * H, Wo = 2 * W;
  const int slabs_per_map = D * (H / WG_ROWS);
  const int slab = blockIdx.x;
  const int b = slab / slabs_per_map, r = slab - b * slabs_per_map;
  const int z = r / (H / WG_ROWS), y0 = (r - z * (H / WG_ROWS)) * WG_ROWS;
  const float *gmap = gy + (size_t)b * Do * Ho * Wo;
  for (int i = tid; i < 4 * GR * GW; i += WG_THREADS) {
    const int c = i % GW, rr = (i / GW) % GR, pl = i / (GW * GR);
    const int oz = 2 * z - 1 + pl, oy = 2 * y0 - 1 + rr, ox = c - 1;
    const bool ok = (oz >= 0) & (oz < Do) & (oy >= 0) & (oy < Ho) & (ox >= 0) & (ox < Wo);
    s_g[pl * gw.plane + rr * gw.pitch + c] = ok ? __ldg(gmap + ((size_t)oz * Ho + oy) * Wo + ox) : 0.0f;
  }
  for (int i = tid; i < Cin * 64; i += WG_THREADS) s_w[i] = __ldg(weight + i);
  __syncthreads();
  const int npos = WG_ROWS * W;
  for (int p = tid; p < npos; p += WG_THREADS) {
    const int yy = p / W, xx = p - yy * W;
    float g[64];
#pragma unroll
    for (int kz = 0; kz < 4; ++kz)
#pragma unroll
      for (int ky = 0; ky < 4; ++ky)
#pragma unroll
        for (int kx = 0; kx < 4; ++kx)
          g[(kz * 4 + ky) * 4 + kx] = s_g[kz * gw.plane + (2 * yy + ky) * gw.pitch + 2 * xx + kx];
    float *o = dx + ((((size_t)b * Cin) * D + z) * H + y0) * (size_t)W + p;
    const size_t cstride = (size_t)D * H * W;
    for (int ci = 0; ci < Cin; ++ci) {
      const float4 *w4 = reinterpret_cast<const float4 *>(s_w + ci * 64);
      float a = 0.0f;
#pragma unroll
      for (int q = 0; q < 16; ++q) {
        const float4 wv = w4[q];
        a = fmaf(wv.x, g[4 * q], a);
        a = fmaf(wv.y, g[4 * q + 1], a);
        a = fmaf(wv.z, g[4 * q + 2], a);
        a = fmaf(wv.w, g[4 * q + 3], a);
      }
      o[ci * cstride] = a;
    }
  }
}

}  // namespace gb

using namespace gb;

extern "C" size_t genre_b200_convt_c1_wgrad_workspace_bytes(int cin) { return (size_t)wgrad_max_ctas() * (size_t)cin * 64 * sizeof(float); }

// x [B][Cin][D][H][W] fp32 contiguous (the concatenated input), gy [B][1][2D][2H][2W] fp32 contiguous,
// dW [Cin][1][4][4][4] (fully written).  H % 8 == 0, Cin <= 64, workspace of genre_b200_convt_c1_wgrad_workspace_bytes(Cin).
extern "C" int genre_b200_convt_c1_wgrad(const float *x, const float *gy, int64_t B, int64_t Cin, int64_t D, int64_t H,
                                         int64_t W, float *dW, void *workspace, size_t workspace_bytes, void *stream) {
  GB_REQUIRE(x && gy && dW && workspace, GENRE_B200_EINVAL, "convt_c1_wgrad: null pointer");
  GB_REQUIRE(B > 0 && Cin > 0 && Cin <= 4 * WG_MAX_CPT && D > 0 && H > 0 && H % WG_ROWS == 0 && W > 0, GENRE_B200_EINVAL,
             "convt_c1_wgrad: unsupported shape (Cin <= 64, H %% 8 == 0)");
  GB_REQUIRE(workspace_bytes >= genre_b200_convt_c1_wgrad_workspace_bytes((int)Cin), GENRE_B200_EWORKSPACE,
             "convt_c1_wgrad: workspace too small");
  const size_t smem = ((size_t)4 * gy_window((int)W).plane + (size_t)Cin * WG_ROWS * W) * sizeof(float);
  GB_REQUIRE(smem <= 200 * 1024, GENRE_B200_EINVAL, "convt_c1_wgrad: slab does not fit shared memory (W=%lld, Cin=%lld)",
             (long long)W, (long long)Cin);
  const int64_t n_slabs = B * D * (H / WG_ROWS);
  GB_REQUIRE(n_slabs < (1ll << 31), GENRE_B200_EINVAL, "convt_c1_wgrad: too many slabs");
  const int grid = (int)(n_slabs < wgrad_max_ctas() ? n_slabs : wgrad_max_ctas());
  cudaStream_t st = as_stream(stream);
  const int cpt = (int)((Cin + 3) / 4);
#define GB_WG(CPT)                                                                                                   \
  do {                                                                                                               \
    auto kern = convt_c1_wgrad_kernel<CPT>;                                                                          \
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);              \
    if (e != cudaSuccess) return fail_arg((int)e, "convt_c1_wgrad: cudaFuncSetAttribute: %s", cudaGetErrorString(e)); \
    kern<<<grid, WG_THREADS, smem, st>>>(x, gy, (int)Cin, (int)D, (int)H, (int)W, (int)n_slabs, (float *)workspace);  \
  } while (0)
  if (cpt <= 4) GB_WG(4);
  else if (cpt <= 8) GB_WG(8);
  else if (cpt <= 10) GB_WG(10);
  else GB_WG(16);
#undef GB_WG
  if (int rc = check_launch("convt_c1_wgrad kernel")) return rc;
  const int n_out = (int)Cin * 64;
  convt_c1_wgrad_reduce_kernel<<<(n_out + 255) / 256, 256, 0, st>>>((const float *)workspace, grid, n_out, dW);
  return check_launch("convt_c1_wgrad reduce kernel");
}

// gy [B][1][2D][2H][2W], weight [Cin][1][4][4][4] -> dx [B][Cin][D][H][W] (fully written).  H % 8 == 0, Cin <= 192.
extern "C" int genre_b200_convt_c1_dgrad(const float *gy, const float *weight, int64_t B, int64_t Cin, int64_t D, int64_t H,
                                         int64_t W, float *dx, void *stream) {
  GB_REQUIRE(gy && weight && dx, GENRE_B200_EINVAL, "convt_c1_dgrad: null pointer");
  GB_REQUIRE(B > 0 && Cin > 0 && Cin <= 192 && D > 0 && H > 0 && H % WG_ROWS == 0 && W > 0, GENRE_B200_EINVAL,
             "convt_c1_dgrad: unsupported shape (H %% 8 == 0)");
  const size_t smem = ((size_t)4 * gy_window((int)W).plane + (size_t)Cin * 64) * sizeof(float);
  GB_REQUIRE(smem <= 200 * 1024, GENRE_B200_EINVAL, "convt_c1_dgrad: slab does not fit shared memory");
  const int64_t n_slabs = B * D * (H / WG_ROWS);
  GB_REQUIRE(n_slabs < (1ll << 31), GENRE_B200_EINVAL, "convt_c1_dgrad: too many slabs");
  cudaError_t e = cudaFuncSetAttribute(convt_c1_dgrad_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return fail_arg((int)e, "convt_c1_dgrad: cudaFuncSetAttribute: %s", cudaGetErrorString(e));
  convt_c1_dgrad_kernel<<<(unsigned)n_slabs, WG_THREADS, smem, as_stream(stream)>>>(gy, weight, (int)Cin, (int)D, (int)H,
                                                                                  (int)W, dx);
  return check_launch("convt_c1_dgrad kernel");
}

// ------------------------------------------------------------------------------------------------------------------
// Weight gradient of Conv3d(Cin <= 2, Cout <= 20, k=8, s=2, p=3): Unet_3D.enc1 (networks/networks.py:151), the layer whose
// cuDNN wgrad (`wgrad2d_grouped_direct_kernel`) is 40.7 ms of a 60 ms training step at B=4.
//     dW[co, ci, kz, ky, kx] = sum_{b, o} gy[b, co, o] * x[b, ci, 2o - 3 + k]          (20480 sums over 1 M positions)
// CTA = slab (b, oz, 8 output rows, all ox); gy slab [Cout][8*Wo] and ONE input plane (z = 2 oz - 3 + kz) per kz step in
// shared memory.  Thread = (ky, kx pair) x ci x channel lane: 2 taps x 5 output channels x 8 kz = 80 register partial
// sums; per position one 8-byte x read and 5 broadcast gy reads feed 10 FMAs.  Persistent CTAs, per-CTA partials, and a
// fixed-order second pass: bitwise reproducible.
namespace gb {

constexpr int W8_ROWS = 8;
constexpr int W8_CI = 2, W8_COL = 4, W8_CPL = 5;  // input channels, channel lanes, output channels per lane (Cout <= 20)

__global__ void __launch_bounds__(256)
conv_k8s2_wgrad_kernel(const float *__restrict__ x, const float *__restrict__ gy, int Cin, int Cout, int D, int H, int W,
                       int n_slabs, float *__restrict__ partial /* [gridDim.x][20][2][512] */) {
  extern __shared__ float smem[];
  const int Do = D / 2, Ho = H / 2, Wo = W / 2;
  const int XR = 2 * W8_ROWS + 6;             // input rows a slab touches per plane
  int pitch = W + 6;                          // columns -3 .. W+2
  while ((pitch & 31) != 8) ++pitch;          // ky rows 8 banks apart, kx pairs 2 apart
  const int xplane = XR * pitch;
  float *s_x = smem;                          // [2][XR][pitch]
  float *s_g = smem + W8_CI * xplane;         // [20][W8_ROWS * Wo]
  const int tid = threadIdx.x;
  const int pair = tid & 31, ky = pair >> 2, kx0 = (pair & 3) * 2, ci = (tid >> 5) & 1, col = tid >> 6;
  const int npos = W8_ROWS * Wo;
  const int slabs_per_map = Do * (Ho / W8_ROWS);
  float acc[8][W8_CPL][2];
#pragma unroll
  for (int a = 0; a < 8; ++a)
#pragma unroll
    for (int j = 0; j < W8_CPL; ++j) acc[a][j][0] = acc[a][j][1] = 0.0f;

  for (int slab = blockIdx.x; slab < n_slabs; slab += gridDim.x) {
    const int b = slab / slabs_per_map, r = slab - b * slabs_per_map;
    const int oz = r / (Ho / W8_ROWS), oy0 = (r - oz * (Ho / W8_ROWS)) * W8_ROWS;
    __syncthreads();
    for (int i = tid; i < 20 * npos; i += 256) {
      const int co = i / npos, p = i - co * npos;
      s_g[i] = co < Cout ? __ldg(gy + ((((size_t)b * Cout + co) * Do + oz) * Ho + oy0) * (size_t)Wo + p) : 0.0f;
    }
#pragma unroll
    for (int kz = 0; kz < 8; ++kz) {
      const int z = 2 * oz - 3 + kz;
      if (kz) __syncthreads();  // previous plane consumed (uniform: z depends only on the slab)
      const bool zin = z >= 0 && z < D;
      for (int i = tid; i < W8_CI * XR * (W + 6); i += 256) {
        const int c = i % (W + 6), rr = (i / (W + 6)) % XR, cc = i / ((W + 6) * XR);
        const int yy = 2 * oy0 - 3 + rr, xx = c - 3;
        const bool ok = zin & (cc < Cin) & (yy >= 0) & (yy < H) & (xx >= 0) & (xx < W);
        s_x[cc * xplane + rr * pitch + c] = ok ? __ldg(x + ((((size_t)b * Cin + cc) * D + z) * H + yy) * (size_t)W + xx) : 0.0f;
      }
      __syncthreads();
      if (!zin) continue;
      const float *xk = s_x + ci * xplane + ky * pitch + kx0;  // taps (ky, kx0), (ky, kx0+1) of output (yy, xx): xk[2yy*pitch + 2xx]
      for (int yy = 0; yy < W8_ROWS; ++yy) {
        const float *xr = xk + 2 * yy * pitch;
        const float *gr = s_g + yy * Wo;
        for (int xx = 0; xx < Wo; ++xx) {
          const float2 xv = *reinterpret_cast<const float2 *>(xr + 2 * xx);
#pragma unroll
          for (int j = 0; j < W8_CPL; ++j) {
            const float g = gr[(col + W8_COL * j) * npos + xx];
            acc[kz][j][0] = fmaf(g, xv.x, acc[kz][j][0]);
            acc[kz][j][1] = fmaf(g, xv.y, acc[kz][j][1]);
          }
        }
      }
    }
  }
  float *out = partial + (size_t)blockIdx.x * 20 * 2 * 512;
#pragma unroll
  for (int kz = 0; kz < 8; ++kz)
#pragma unroll
    for (int j = 0; j < W8_CPL; ++j) {
      const int co = col + W8_COL * j;
      float *o = out + ((size_t)(co * 2 + ci) * 8 + kz) * 64 + ky * 8 + kx0;
      o[0] = acc[kz][j][0];
      o[1] = acc[kz][j][1];
    }
}

// partial [n_parts][20][2][512] -> dW [Cout][Cin][512]
__global__ void __launch_bounds__(256)
conv_k8s2_wgrad_reduce_kernel(const float *__restrict__ partial, int n_parts, int Cin, int Cout, float *__restrict__ dW) {
  const int i = blockIdx.x * 256 + threadIdx.x;
  if (i >= Cout * Cin * 512) return;
  const int k = i & 511, ci = (i >> 9) % Cin, co = (i >> 9) / Cin;
  const size_t src = ((size_t)co * 2 + ci) * 512 + k;
  float s = 0.0f;
  for (int p = 0; p < n_parts; ++p) s += partial[(size_t)p * 20480 + src];
  dW[i] = s;
}

}  // namespace gb

extern "C" size_t genre_b200_conv_k8s2_wgrad_workspace_bytes(void) { return (size_t)wgrad_max_ctas() * 20480 * sizeof(float); }

// x [B][Cin][D][H][W], gy [B][Cout][D/2][H/2][W/2] (fp32, contiguous) -> dW [Cout][Cin][8][8][8] (fully written).
// Cin <= 2, Cout <= 20, even extents, (H/2) % 8 == 0, W <= 128.
extern "C" int genre_b200_conv_k8s2_wgrad(const float *x, const float *gy, int64_t B, int64_t Cin, int64_t Cout, int64_t D,
                                          int64_t H, int64_t W, float *dW, void *workspace, size_t workspace_bytes,
                                          void *stream) {
  GB_REQUIRE(x && gy && dW && workspace, GENRE_B200_EINVAL, "conv_k8s2_wgrad: null pointer");
  GB_REQUIRE(B > 0 && Cin > 0 && Cin <= W8_CI && Cout > 0 && Cout <= 20 && D > 0 && D % 2 == 0 && H > 0 && H % (2 * W8_ROWS) == 0 &&
                 W > 0 && W % 2 == 0 && W <= 128,
             GENRE_B200_EINVAL, "conv_k8s2_wgrad: unsupported shape (Cin <= 2, Cout <= 20, H %% 16 == 0, W <= 128 even)");
  GB_REQUIRE(workspace_bytes >= genre_b200_conv_k8s2_wgrad_workspace_bytes(), GENRE_B200_EWORKSPACE,
             "conv_k8s2_wgrad: workspace too small");
  int pitch = (int)W + 6;
  while ((pitch & 31) != 8) ++pitch;
  const size_t smem = ((size_t)W8_CI * (2 * W8_ROWS + 6) * pitch + (size_t)20 * W8_ROWS * (W / 2)) * sizeof(float);
  GB_REQUIRE(smem <= 200 * 1024, GENRE_B200_EINVAL, "conv_k8s2_wgrad: slab does not fit shared memory");
  const int64_t n_slabs = B * (D / 2) * ((H / 2) / W8_ROWS);
  GB_REQUIRE(n_slabs < (1ll << 31), GENRE_B200_EINVAL, "conv_k8s2_wgrad: too many slabs");
  const int grid = (int)(n_slabs < wgrad_max_ctas() ? n_slabs : wgrad_max_ctas());
  cudaStream_t st = as_stream(stream);
  cudaError_t e = cudaFuncSetAttribute(conv_k8s2_wgrad_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return fail_arg((int)e, "conv_k8s2_wgrad: cudaFuncSetAttribute: %s", cudaGetErrorString(e));
  conv_k8s2_wgrad_kernel<<<grid, 256, smem, st>>>(x, gy, (int)Cin, (int)Cout, (int)D, (int)H, (int)W, (int)n_slabs,
                                                  (float *)workspace);
  if (int rc = check_launch("conv_k8s2_wgrad kernel")) return rc;
  const int n_out = (int)(Cout * Cin * 512);
  conv_k8s2_wgrad_reduce_kernel<<<(n_out + 255) / 256, 256, 0, st>>>((const float *)workspace, grid, (int)Cin, (int)Cout, dW);
  return check_launch("conv_k8s2_wgrad reduce kernel");
}
