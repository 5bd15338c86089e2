// convt_c1.cu — ConvTranspose3d(Cin -> 1, k=4, s=2, p=1) forward: the last layer of every decoder in networks.py
// (Unet_3D.dec6 networks.py:167-168 = cat(dec5, enc1) -> ConvT(40 -> 1); VoxelDecoder main.17 :57; VoxelGenerator :98).
//
// With one output channel this is a 320-MAC stencil per output voxel, not a GEMM: tensor cores have nothing to chew on
// (N = 1), so it runs on the FP32 pipe.  Inputs arrive in the channel-blocked layout the wgmma kernels write
// ([B*D][C/4][H][W][4]), so one 16-byte load brings 4 channels of a position and one 16-byte broadcast load brings the
// matching 4 weights: 118 loads per 1024 FMAs.  A thread owns 4 input-aligned cells along x = 32 outputs (4 cells x 8
// parities), needs the 3 x 3 x 6 neighbourhood per channel group, and writes eight 16-byte stores into the NCDHW
// output.  The two halves of the skip concatenation are two source tensors (never concatenated).
//   out[2j+p] = bias + sum_c sum_t in[c, j + base_p - t] * W[c, k0_p + 2t],  k0_p = (p+1)%2, base_p = p
#include "common.cuh"

namespace gb {

constexpr int C1_TX = 16, C1_TY = 8, C1_TZ = 2;       // threads; each handles 4 cells along x
constexpr int C1_CELLS = 4;

__global__ void __launch_bounds__(C1_TX *C1_TY *C1_TZ)
convt_c1_kernel(const float4 *__restrict__ src0, int cg0, const float4 *__restrict__ src1, int cg1, int D, int H, int W,
                const float *__restrict__ weight /* [Cin][64] */, float bias, int act_sigmoid,
                float *__restrict__ out /* [B][2D][2H][2W] */) {
  extern __shared__ float4 s_w[];  // [cg][64 taps] float4 over the 4 channels of the group
  const int ncg = cg0 + cg1;
  for (int i = threadIdx.x + C1_TX * (threadIdx.y + C1_TY * threadIdx.z); i < ncg * 64; i += C1_TX * C1_TY * C1_TZ) {
    const int cg = i >> 6, k = i & 63;
    s_w[i] = make_float4(weight[(cg * 4 + 0) * 64 + k], weight[(cg * 4 + 1) * 64 + k], weight[(cg * 4 + 2) * 64 + k],
                         weight[(cg * 4 + 3) * 64 + k]);
  }
  __syncthreads();
  const int x0 = (blockIdx.x * C1_TX + threadIdx.x) * C1_CELLS;
  const int y = blockIdx.y * C1_TY + threadIdx.y;
  const int zb = blockIdx.z * C1_TZ + threadIdx.z;  // b * D + z
  const int b = zb / D, z = zb - b * D;
  if (x0 >= W || y >= H || b < 0) return;

  float acc[C1_CELLS][8];
#pragma unroll
  for (int c = 0; c < C1_CELLS; ++c)
#pragma unroll
    for (int p = 0; p < 8; ++p) acc[c][p] = 0.0f;

  for (int cg = 0; cg < ncg; ++cg) {
    const float4 *src = cg < cg0 ? src0 : src1;
    const int lcg = cg < cg0 ? cg : cg - cg0, ncgs = cg < cg0 ? cg0 : cg1;
    const float4 *w = s_w + cg * 64;
    // one z-plane of the neighbourhood at a time (keeps the register footprint at 3 x 6 float4): plane dz serves the
    // (parity, tap) pairs with pz - tz + 1 == dz.  Parity p (per dim), tap t: input offset d = p - t in {-1,0,+1},
    // kernel index k = (p+1)%2 + 2t.
#pragma unroll
    for (int dz = 0; dz < 3; ++dz) {
      const int zz = z + dz - 1;
      float4 in[3][C1_CELLS + 2];
#pragma unroll
      for (int dy = 0; dy < 3; ++dy) {
        const int yy = y + dy - 1;
        const bool okzy = (zz >= 0) & (zz < D) & (yy >= 0) & (yy < H);
        const float4 *row = src + ((((size_t)b * D + (okzy ? zz : 0)) * ncgs + lcg) * H + (okzy ? yy : 0)) * (size_t)W;
#pragma unroll
        for (int dx = 0; dx < C1_CELLS + 2; ++dx) {
          const int xx = x0 + dx - 1;
          in[dy][dx] = (okzy & (xx >= 0) & (xx < W)) ? __ldg(row + xx) : make_float4(0.f, 0.f, 0.f, 0.f);
        }
      }
#pragma unroll
      for (int pz = 0; pz < 2; ++pz)
#pragma unroll
        for (int tz = 0; tz < 2; ++tz) {
          if (pz - tz + 1 != dz) continue;
#pragma unroll
          for (int py = 0; py < 2; ++py)
#pragma unroll
            for (int ty = 0; ty < 2; ++ty)
#pragma unroll
              for (int px = 0; px < 2; ++px)
#pragma unroll
                for (int tx = 0; tx < 2; ++tx) {
                  const int kz = ((pz + 1) & 1) + 2 * tz, ky = ((py + 1) & 1) + 2 * ty, kx = ((px + 1) & 1) + 2 * tx;
                  const float4 wv = w[(kz * 4 + ky) * 4 + kx];
                  const int dy = py - ty + 1, dxo = px - tx + 1;
#pragma unroll
                  for (int c = 0; c < C1_CELLS; ++c) {
                    const float4 v = in[dy][c + dxo];
                    float a = acc[c][(pz * 2 + py) * 2 + px];
                    a = fmaf(v.x, wv.x, a);
                    a = fmaf(v.y, wv.y, a);
                    a = fmaf(v.z, wv.z, a);
                    a = fmaf(v.w, wv.w, a);
                    acc[c][(pz * 2 + py) * 2 + px] = a;
                  }
                }
        }
    }
  }
  const int Ho = 2 * H, Wo = 2 * W, Do = 2 * D;
#pragma unroll
  for (int pz = 0; pz < 2; ++pz)
#pragma unroll
    for (int py = 0; py < 2; ++py) {
      float o[2 * C1_CELLS];
#pragma unroll
      for (int c = 0; c < C1_CELLS; ++c)
#pragma unroll
        for (int px = 0; px < 2; ++px) {
          float v = acc[c][(pz * 2 + py) * 2 + px] + bias;
          if (act_sigmoid) v = 1.0f / (1.0f + __expf(-v));
          o[2 * c + px] = v;
        }
      float *dst = out + (((size_t)b * Do + (2 * z + pz)) * Ho + (2 * y + py)) * (size_t)Wo + 2 * x0;
      st_stream_f4(dst, make_float4(o[0], o[1], o[2], o[3]));
      st_stream_f4(dst + 4, make_float4(o[4], o[5], o[6], o[7]));
    }
}

}  // namespace gb

using namespace gb;

// ConvTranspose3d(4*(cg0+cg1) -> 1, kernel 4, stride 2, padding 1) on channel-blocked fp32 inputs.
//   src0 [B*D][cg0][H][W][4], src1 [B*D][cg1][H][W][4] or NULL;  weight [Cin][4*4*4] (the module's [Cin,1,4,4,4]);
//   out [B][2D][2H][2W] fp32 (NCDHW with C = 1);  act_sigmoid: apply the generator's final Sigmoid.  W % 4 == 0.
extern "C" int genre_b200_convt_c1_forward(const float *src0, int cg0, const float *src1, int cg1, int64_t B, int64_t D,
                                           int64_t H, int64_t W, const float *weight, float bias, int act_sigmoid,
                                           float *out, void *stream) {
  GB_REQUIRE(src0 && weight && out, GENRE_B200_EINVAL, "convt_c1: null pointer");
  GB_REQUIRE(cg0 > 0 && cg1 >= 0 && (cg1 == 0 || src1), GENRE_B200_EINVAL, "convt_c1: bad channel groups");
  GB_REQUIRE(B > 0 && D > 0 && H > 0 && W > 0 && W % C1_CELLS == 0, GENRE_B200_EINVAL, "convt_c1: bad extent");
  GB_REQUIRE(aligned16(src0) && aligned16(out) && (!src1 || aligned16(src1)), GENRE_B200_EALIGN, "convt_c1: alignment");
  GB_REQUIRE((cg0 + cg1) * 64 * 16 <= 48 * 1024, GENRE_B200_EINVAL, "convt_c1: too many input channels (max 192)");
  dim3 block(C1_TX, C1_TY, C1_TZ);
  dim3 grid((unsigned)((W / C1_CELLS + C1_TX - 1) / C1_TX), (unsigned)((H + C1_TY - 1) / C1_TY),
            (unsigned)((B * D + C1_TZ - 1) / C1_TZ));
  GB_REQUIRE(grid.z <= 65535 && grid.y <= 65535, GENRE_B200_EINVAL, "convt_c1: grid too large");
  convt_c1_kernel<<<grid, block, (size_t)(cg0 + cg1) * 64 * sizeof(float4), as_stream(stream)>>>(
      (const float4 *)src0, cg0, (const float4 *)src1, cg1, (int)D, (int)H, (int)W, weight, bias, act_sigmoid, out);
  return check_launch("convt_c1 kernel");
}
