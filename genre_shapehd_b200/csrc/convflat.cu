// convflat.cu — the stride-2 3D convolutions of the SMALL volumes (<= 8^3 on the coarse side) as a wgmma implicit GEMM over a
// flattened, zero-separated volume.
//
// Reference layers: networks/networks.py:157-165 (Unet_3D.enc4, enc5 = Conv3d(k 4, s 2, p 1) -> BatchNorm3d -> LeakyReLU on
// 16^3 / 8^3; dec2, dec3 = cat(x, skip) -> ConvTranspose3d(k 4, s 2, p 1) -> BatchNorm3d -> ReLU on 4^3 / 8^3), and the 4^3 / 8^3
// stages of VoxelDecoder / VoxelGenerator / VoxelDiscriminator (:40-57, :79-97, :253-256).  These layers hold 1% of the
// refiner's FLOPs but a quarter of its time on the big-volume kernel's fallbacks: their planes are too small for the
// (16 y-rows x 8 x) tiles of convt3d.cu, and their channel counts (80-640) exceed its N <= 64.
//
// Formulation.  Pad every dimension of the coarse volume by ONE zero separator (x = W, y = H, z = D) and flatten batch and
// volume into one axis: position q = ((b*(D+1) + z)*(H+1) + y)*(W+1) + x.  Every tap of a k=4, s=2, p=1 convolution (either
// direction, after the parity split) moves by at most one voxel per dimension, so it is a SHIFT of q by
// dz*(H+1)*(W+1) + dy*(W+1) + dx, and every out-of-volume neighbour lands on a separator: the zero padding is in the data.
//     GEMM per class:  M = all positions q (the separators' rows are computed and dropped),  N = Cout,  K = 8 taps * Cin
// With the operand stored as [part][channel group of 8 fp16][position][16 B], the rows of an M-tile are CONTIGUOUS 16-byte
// units: the K-major no-swizzle operand of ANY tap is the same shared-memory array at a different 16-byte offset, and the
// array itself (tile + the largest shift on both sides) arrives with ONE cp.async.bulk per channel group.
//   transposed conv: 8 output parity classes (blockIdx.z), class (pz,py,px) tap t reads shift d = (p ? 1 - t : -t) per dim;
//   strided conv   : the K range is the 8 parity sub-volumes of the fine input (sub-volume s = channels [s*Cin, (s+1)*Cin)),
//                    sub-volume parity p, tap t reads shift d = 1 - p - t.
// OP 1: fp16 operands; OP 2: the fp32-accurate fp16 hi/lo split of convt3d.cu (2 MMAs per K step, see ConvTCfg there).
// CTA = MT M-tiles of 128 positions x NPAD output channels (x 2 accumulator halves in OP 2) of one class; warps 0-3:
// warp 0 lane 0 issues the bulk copies, then all four run the epilogue (scale/shift = bias + folded BatchNorm, LeakyReLU,
// NCDHW fp32 store) from a shared-memory image of the accumulators; warps 4-11: two consumer warpgroups, warpgroup wg
// issuing the m64 wgmma of rows [64 wg, 64 wg + 64) of every M-tile with its accumulators in registers (MT * NACC <= 256).
// A stage = one K step (16 channels) x 8 taps.
#include <cuda_fp16.h>
#include "common.cuh"
#include "tc_ptx.cuh"

namespace gb {

constexpr int CF_THREADS = 384;
constexpr int CF_CONSUMER_WARPS = 8;
constexpr int CF_TAPS = 8;
constexpr int CF_MAX_STAGES = 6;

struct ConvFlatParams {
  const __half *act;    // [parts][cgs][P][8]: flattened zero-separated operand; position q sits at index lead + q
  int cgs;              // channel groups of 8 (even)
  long long P;          // positions per channel group array
  int lead;             // >= halo
  int halo;             // largest |shift| = (H+1)*(W+1) + (W+1) + 1
  int B, D, H, W;       // coarse volume
  long long M;          // B*(D+1)*(H+1)*(W+1) GEMM rows
  const __half *wpack;  // [class][ntile][K step][8 taps][2 kcore][NACC/8][8][8]
  int ntiles, ksteps;
  int cgs_per_group;    // 0: the shift row is the class (transposed conv); else: the sub-volume of the K step = 2*kstep / this
  int shift[8][CF_TAPS];
  int up;               // 1: output at 2*j + parity of the class (transposed conv); 0: output at j
  const float *scale, *shift_c;  // [ntiles*NPAD]
  float slope;
  float *out;           // NCDHW fp32 [B][Cout][Do][Ho][Wo]
  int Cout;
  int stages, a_cg_stride, stage_bytes, ring_bytes;   // shared-memory plan (host)
};

template <int NPAD, int MT, int OP>
__global__ void __launch_bounds__(CF_THREADS, 1) convflat_kernel(const ConvFlatParams p) {
  constexpr bool X2 = OP == 2;
  constexpr int PARTS = X2 ? 2 : 1;
  constexpr int NACC = PARTS * NPAD;
  constexpr int B_TAP_BYTES = 2 * (NACC / 8) * 128;
  constexpr int B_BYTES = CF_TAPS * B_TAP_BYTES;
  constexpr int ACC_LD = NPAD + 4;   // accumulator image [MT][128 rows][ACC_LD] fp32, over the drained ring
  static_assert(MT * NACC <= 256 && NACC <= 256 && NPAD % 16 == 0, "accumulator shape");
  extern __shared__ __align__(128) uint8_t smem[];
  uint8_t *stages = smem;
  uint64_t *full = reinterpret_cast<uint64_t *>(smem + (size_t)p.ring_bytes);
  uint64_t *empty = full + CF_MAX_STAGES;
  float *acc_img = reinterpret_cast<float *>(smem);

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const long long q0 = (long long)blockIdx.x * (128 * MT);   // first position of this CTA
  const int ntile = blockIdx.y, cls = blockIdx.z;
  const int a_bytes = PARTS * 2 * p.a_cg_stride;
  const int a_cg_bytes = (128 * MT + 2 * p.halo) * 16;

  if (tid == 0) {
    for (int s = 0; s < p.stages; ++s) {
      mbar_init(&full[s], 1);
      mbar_init(&empty[s], CF_CONSUMER_WARPS);
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if (warp < 4) {
    if (tid == 0) {
      // ===================== producer: per K step, 2*PARTS operand arrays + the weights of its 8 taps ===================
      const __half *wbase = p.wpack + ((size_t)cls * p.ntiles + ntile) * (size_t)p.ksteps * (B_BYTES / 2);
      for (int ks = 0; ks < p.ksteps; ++ks) {
        const int s = ks % p.stages, use = ks / p.stages;
        if (use > 0) mbar_wait(&empty[s], (use - 1) & 1);
        uint8_t *sa = stages + (size_t)s * p.stage_bytes;
        mbar_arrive_expect_tx(&full[s], (uint32_t)(B_BYTES + PARTS * 2 * a_cg_bytes));
        bulk_g2s(sa + a_bytes, wbase + (size_t)ks * (B_BYTES / 2), B_BYTES, &full[s]);
#pragma unroll
        for (int part = 0; part < PARTS; ++part) {
#pragma unroll
          for (int c = 0; c < 2; ++c) {
            const __half *src = p.act + (((size_t)part * p.cgs + (size_t)(ks * 2 + c)) * p.P + (size_t)(p.lead + q0 - p.halo)) * 8;
            bulk_g2s(sa + (part * 2 + c) * p.a_cg_stride, src, (uint32_t)a_cg_bytes, &full[s]);
          }
        }
      }
    }
  } else {
    // ===================== consumers ============================================================================
    const int wg = (warp - 4) >> 2;
    float acc[MT][NACC / 2];
#pragma unroll
    for (int mt = 0; mt < MT; ++mt)
#pragma unroll
      for (int j = 0; j < NACC / 2; ++j) acc[mt][j] = 0.0f;
    for (int ks = 0; ks < p.ksteps; ++ks) {
      const int s = ks % p.stages, use = ks / p.stages;
      mbar_wait(&full[s], use & 1);
      wgmma_fence();
      const uint32_t sa = smem_u32(stages + (size_t)s * p.stage_bytes);
      const uint32_t sb = sa + a_bytes;
      const int grp = p.cgs_per_group ? ((ks * 2) / p.cgs_per_group) & 7 : cls;
#pragma unroll
      for (int t = 0; t < CF_TAPS; ++t) {
        const uint64_t bdesc = gmma_desc(sb + t * B_TAP_BYTES, (NACC / 8) * 128, 128);
        const int sh = p.shift[grp][t];
#pragma unroll
        for (int mt = 0; mt < MT; ++mt) {
          const uint32_t a0 = sa + (uint32_t)((p.halo + sh + 128 * mt + 64 * wg) * 16);
          const uint64_t adesc = gmma_desc(a0, p.a_cg_stride, 128);
          wgmma_f16<NACC>(acc[mt], adesc, bdesc);
          if constexpr (X2) {
            const uint64_t adesc_lo = gmma_desc(a0 + 2 * p.a_cg_stride, p.a_cg_stride, 128);
            wgmma_f16<NPAD>(acc[mt] + NPAD / 2, adesc_lo, bdesc);
          }
        }
      }
      wgmma_commit();
      wgmma_wait<0>();
      __syncwarp();
      if (lane == 0) mbar_arrive(&empty[s]);
    }
    // every stage has been consumed: the ring becomes the accumulator image
    asm volatile("bar.sync 1, 256;" ::: "memory");   // ... by BOTH consumer warpgroups: the other one may still be reading it
#pragma unroll
    for (int mt = 0; mt < MT; ++mt) store_acc_tile<NPAD, X2>(acc[mt], acc_img + ((size_t)mt * 128 + 64 * wg) * ACC_LD, ACC_LD);
  }
  __syncthreads();
  if (warp < 4) {
    // ===================== epilogue ===========================================================================
    const int Wp = p.W + 1, Hp = p.H + 1, Dp = p.D + 1;
    const int Do = p.up ? 2 * p.D : p.D, Ho = p.up ? 2 * p.H : p.H, Wo = p.up ? 2 * p.W : p.W;
    const int pz = p.up ? (cls >> 2) & 1 : 0, py = p.up ? (cls >> 1) & 1 : 0, px = p.up ? cls & 1 : 0;
    const size_t ovol = (size_t)Do * Ho * Wo;
#pragma unroll
    for (int mt = 0; mt < MT; ++mt) {
      const long long q = q0 + mt * 128 + warp * 32 + lane;
      long long r = q;
      const int x = (int)(r % Wp); r /= Wp;
      const int y = (int)(r % Hp); r /= Hp;
      const int z = (int)(r % Dp);
      const long long b = r / Dp;
      const bool valid = q < p.M && x < p.W && y < p.H && z < p.D;
      const int oz = p.up ? 2 * z + pz : z, oy = p.up ? 2 * y + py : y, ox = p.up ? 2 * x + px : x;
      float *orow = p.out + (size_t)b * p.Cout * ovol + ((size_t)oz * Ho + oy) * Wo + ox;
      const float *arow = acc_img + ((size_t)mt * 128 + warp * 32 + lane) * ACC_LD;
#pragma unroll 1
      for (int nb = 0; nb < NPAD / 16; ++nb) {
        if (valid) {
          float v[16];
          ld_row<16>(arow + nb * 16, v);
#pragma unroll
          for (int i = 0; i < 16; ++i) {
            const int n = ntile * NPAD + nb * 16 + i;
            if (n < p.Cout) {
              const float t = fmaf(v[i], __ldg(p.scale + n), __ldg(p.shift_c + n));
              orow[(size_t)n * ovol] = t > 0.0f ? t : t * p.slope;
            }
          }
        }
      }
    }
  }
}

// ---- operand construction: NCDHW fp32 -> [part][cg][P][8 fp16], separators / lead / tail zero ------------------------------
// subvol = 0: the volume itself, channel group cg of the source lands at group cg_off + cg;
// subvol = 1: the 8 parity sub-volumes of the (2D, 2H, 2W) source as 8 channel blocks, group (s*C/8 + cg).
// src == nullptr: zero-fill groups [cg_off, cg_off + ncg).
template <int PARTS>
__global__ void __launch_bounds__(256)
flat_pack_kernel(const float *__restrict__ src, int C, int B, int D, int H, int W, int subvol, __half *__restrict__ dst, int cg_off,
                 int ncg, int cgs, long long P, int lead) {
  const long long idx = (long long)blockIdx.x * 256 + threadIdx.x;
  if (idx >= (long long)ncg * P) return;
  const int cg = (int)(idx / P);
  const long long pos = idx - (long long)cg * P;
  const int Wp = W + 1, Hp = H + 1, Dp = D + 1;
  long long r = pos - lead;
  uint4 hi = make_uint4(0, 0, 0, 0), lo = make_uint4(0, 0, 0, 0);
  if (src != nullptr && r >= 0 && r < (long long)B * Dp * Hp * Wp) {
    const int x = (int)(r % Wp); r /= Wp;
    const int y = (int)(r % Hp); r /= Hp;
    const int z = (int)(r % Dp);
    const int b = (int)(r / Dp);
    if (x < W && y < H && z < D) {
      int c0 = cg * 8, sz = z, sy = y, sx = x, SD = D, SH = H, SW = W;
      if (subvol) {
        const int sv = c0 / C;
        c0 -= sv * C;
        SD = 2 * D; SH = 2 * H; SW = 2 * W;
        sz = 2 * z + ((sv >> 2) & 1); sy = 2 * y + ((sv >> 1) & 1); sx = 2 * x + (sv & 1);
      }
      const size_t cstride = (size_t)SD * SH * SW;
      const float *s = src + ((size_t)b * C + c0) * cstride + ((size_t)sz * SH + sy) * SW + sx;
      __half h[8], l[8];
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        const float a = c0 + e < C ? __ldg(s + e * cstride) : 0.0f;
        h[e] = __float2half_rn(a);
        l[e] = __float2half_rn((a - __half2float(h[e])) * 2048.0f);
      }
      hi = *reinterpret_cast<uint4 *>(h);
      lo = *reinterpret_cast<uint4 *>(l);
    }
  }
  uint4 *d = reinterpret_cast<uint4 *>(dst);
  d[((size_t)(cg_off + cg)) * P + pos] = hi;
  if (PARTS == 2) d[((size_t)cgs + cg_off + cg) * P + pos] = lo;
}

template <int NPAD, int MT, int OP>
static int launch_convflat(ConvFlatParams &p, int classes, cudaStream_t st) {
  constexpr int PARTS = OP == 2 ? 2 : 1, NACC = PARTS * NPAD;
  if constexpr (MT > 1 && MT * NACC > 256) {   // register budget of the consumers
    return launch_convflat<NPAD, MT / 2, OP>(p, classes, st);
  } else {
    const int acc_bytes = MT * 128 * (NPAD + 4) * 4;
    constexpr int B_BYTES = CF_TAPS * 2 * (NACC / 8) * 128;
    const int a_cg_bytes = (128 * MT + 2 * p.halo) * 16;
    p.a_cg_stride = (a_cg_bytes + 127) / 128 * 128;
    p.stage_bytes = PARTS * 2 * p.a_cg_stride + B_BYTES;
    int stages = (224 * 1024) / p.stage_bytes;
    if (stages > CF_MAX_STAGES) stages = CF_MAX_STAGES;
    if (stages > p.ksteps) stages = p.ksteps < 1 ? 1 : p.ksteps;
    GB_REQUIRE(stages >= 2 || p.ksteps == 1, GENRE_B200_EINVAL, "convflat: a stage of %d bytes does not fit twice", p.stage_bytes);
    p.stages = stages;
    p.ring_bytes = stages * p.stage_bytes > acc_bytes ? stages * p.stage_bytes : acc_bytes;
    const size_t smem = (size_t)p.ring_bytes + 256;
    auto kern = convflat_kernel<NPAD, MT, OP>;
    static bool configured[64] = {};
    int dev = 0;
    cudaGetDevice(&dev);
    if (!configured[dev & 63]) {
      if (cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024) != cudaSuccess)
        return check_launch("convflat: cudaFuncSetAttribute");
      configured[dev & 63] = true;
    }
    const long long mtiles = (p.M + 128 * MT - 1) / (128 * MT);
    dim3 grid((unsigned)mtiles, (unsigned)p.ntiles, (unsigned)classes);
    kern<<<grid, CF_THREADS, smem, st>>>(p);
    return check_launch("convflat kernel");
  }
}

}  // namespace gb

using namespace gb;

// positions per channel-group array of the operand of a (B, D, H, W) coarse volume, and the index of position 0
extern "C" int64_t genre_b200_convflat_positions(int64_t B, int D, int H, int W, int *lead_out) {
  if (B <= 0 || D <= 0 || H <= 0 || W <= 0) return 0;
  const int halo = (H + 1) * (W + 1) + (W + 1) + 1;
  const int lead = (halo + 7) / 8 * 8;
  const long long M = (long long)B * (D + 1) * (H + 1) * (W + 1);
  if (lead_out) *lead_out = lead;
  return lead + (M + 255) / 256 * 256 + lead;
}

// NCDHW fp32 source -> channel groups [cg_off, cg_off + ceil(C'/8)) of the operand (C' = C, or 8*C for subvol), see flat_pack_kernel.
//   B, D, H, W: the COARSE volume (the source is [B, C, 2D, 2H, 2W] when subvol = 1); parts 1 (fp16) or 2 (hi | lo')
//   src == NULL: zero `zero_groups` groups from cg_off (the padding of an odd group count)
extern "C" int genre_b200_convflat_pack(const float *src, int C, int64_t B, int D, int H, int W, int subvol, void *operand, int cg_off,
                                        int cgs, int parts, int zero_groups, void *stream) {
  GB_REQUIRE(operand && B > 0 && D > 0 && H > 0 && W > 0 && cgs > 0 && cg_off >= 0, GENRE_B200_EINVAL, "convflat_pack: bad arguments");
  GB_REQUIRE(parts == 1 || parts == 2, GENRE_B200_EINVAL, "convflat_pack: parts must be 1 or 2");
  int lead = 0;
  const long long P = genre_b200_convflat_positions(B, D, H, W, &lead);
  int ncg;
  if (src) {
    GB_REQUIRE(C > 0 && (!subvol || C % 8 == 0), GENRE_B200_EINVAL, "convflat_pack: sub-volume sources need C %% 8 == 0 (C=%d)", C);
    ncg = subvol ? C : (C + 7) / 8;
  } else {
    ncg = zero_groups;
  }
  GB_REQUIRE(ncg > 0 && cg_off + ncg <= cgs, GENRE_B200_EINVAL, "convflat_pack: groups [%d, %d) exceed %d", cg_off, cg_off + ncg, cgs);
  const long long total = (long long)ncg * P;
  const unsigned grid = (unsigned)((total + 255) / 256);
  cudaStream_t st = as_stream(stream);
  if (parts == 2)
    flat_pack_kernel<2><<<grid, 256, 0, st>>>(src, C, (int)B, D, H, W, subvol, (__half *)operand, cg_off, ncg, cgs, P, lead);
  else
    flat_pack_kernel<1><<<grid, 256, 0, st>>>(src, C, (int)B, D, H, W, subvol, (__half *)operand, cg_off, ncg, cgs, P, lead);
  return check_launch("convflat_pack kernel");
}

// out[B, Cout, Do, Ho, Wo] = act(scale * conv(operand) + shift), NCDHW fp32.
//   operand: genre_b200_convflat_pack's [parts][cgs][P][8 fp16] of the coarse (B, D, H, W) volume, cgs even
//   transposed = 1: ConvTranspose3d(k 4, s 2, p 1), K = 8*cgs input channels, output (2D, 2H, 2W);
//   transposed = 0: Conv3d(k 4, s 2, p 1) of the (2D, 2H, 2W) input given as 8 sub-volume blocks of cgs/8 groups, output (D, H, W)
//   wpack: [classes][ntiles][cgs/2][8 taps][2][parts*npad/8][8][8] fp16 (ops_conv.pack_flat_*), npad 64 or 80, op 1 (fp16) / 2 (hi/lo)
extern "C" int genre_b200_convflat_forward(const void *operand, int cgs, int64_t B, int D, int H, int W, int transposed,
                                           const void *wpack, int npad, int op, const float *scale, const float *shift, float slope,
                                           float *out, int Cout, void *stream) {
  GB_REQUIRE(operand && wpack && scale && shift && out, GENRE_B200_EINVAL, "convflat: null pointer");
  GB_REQUIRE(B > 0 && D > 0 && H > 0 && W > 0 && D <= 16 && H <= 16 && W <= 16, GENRE_B200_EINVAL,
             "convflat: coarse volume %dx%dx%d unsupported (each dimension 1..16)", D, H, W);
  GB_REQUIRE(cgs > 0 && cgs % 2 == 0 && Cout > 0, GENRE_B200_EINVAL, "convflat: cgs=%d must be even, Cout=%d", cgs, Cout);
  GB_REQUIRE(transposed || (cgs % 16 == 0), GENRE_B200_EINVAL, "convflat: a strided conv needs 8 sub-volume blocks of an even group count");
  GB_REQUIRE(op == 1 || op == 2, GENRE_B200_EINVAL, "convflat: op %d (1 = fp16, 2 = fp16 hi/lo)", op);
  GB_REQUIRE(npad == 64 || npad == 80, GENRE_B200_EINVAL, "convflat: npad %d (64 or 80)", npad);
  GB_REQUIRE(aligned16(operand) && aligned16(wpack), GENRE_B200_EALIGN, "convflat: operands must be 16-byte aligned");
  ConvFlatParams p{};
  p.act = (const __half *)operand;
  p.cgs = cgs;
  p.P = genre_b200_convflat_positions(B, D, H, W, &p.lead);
  p.halo = (H + 1) * (W + 1) + (W + 1) + 1;
  p.B = (int)B; p.D = D; p.H = H; p.W = W;
  p.M = (long long)B * (D + 1) * (H + 1) * (W + 1);
  p.wpack = (const __half *)wpack;
  p.ntiles = (Cout + npad - 1) / npad;
  p.ksteps = cgs / 2;
  p.cgs_per_group = transposed ? 0 : cgs / 8;
  const int sz = (H + 1) * (W + 1), sy = W + 1;
  for (int g = 0; g < 8; ++g)
    for (int t = 0; t < 8; ++t) {
      int d[3];
      for (int k = 0; k < 3; ++k) {
        const int par = (g >> (2 - k)) & 1, tt = (t >> (2 - k)) & 1;
        d[k] = transposed ? (par ? 1 - tt : -tt) : 1 - par - tt;
      }
      p.shift[g][t] = d[0] * sz + d[1] * sy + d[2];
    }
  p.up = transposed ? 1 : 0;
  p.scale = scale; p.shift_c = shift; p.slope = slope;
  p.out = out; p.Cout = Cout;
  const int classes = transposed ? 8 : 1;
  // two M-tiles per CTA halve the weight traffic per output; one keeps more CTAs in flight on the smallest layers
  const long long ctas2 = ((p.M + 255) / 256) * p.ntiles * classes;
  const bool mt2 = ctas2 >= 120;
  cudaStream_t st = as_stream(stream);
#define GB_CF(NP, OPV)                                                         \
  if (npad == NP && op == OPV) return mt2 ? launch_convflat<NP, 2, OPV>(p, classes, st) : launch_convflat<NP, 1, OPV>(p, classes, st);
  GB_CF(64, 1) GB_CF(64, 2) GB_CF(80, 1) GB_CF(80, 2)
#undef GB_CF
  return fail_arg(GENRE_B200_EINVAL, "convflat: no kernel for npad=%d op=%d", npad, op);
}
