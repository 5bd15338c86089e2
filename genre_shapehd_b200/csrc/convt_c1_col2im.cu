// convt_c1_col2im.cu — ConvTranspose3d(Cin -> 1, k 4, s 2, p 1) on 64-wide volumes as a wgmma GEMM over the 64 kernel taps
// followed by a shared-memory col2im: the last layer of every decoder at full size.
//
// Reference layers: networks/networks.py:167-168 (Unet_3D.dec6 = cat(dec5, enc1) -> ConvTranspose3d(2 nf -> 1) on 64^3),
// :57 (VoxelDecoder main.17: 32 -> 1 on 64^3), :98 (VoxelGenerator: 64 -> 1).
//
// With ONE output channel the usual implicit GEMM has N = 8 parity classes: 3% of an MMA's width (convt3d.cu MODE 4), and the
// exact FP32 stencil (convt_c1.cu) is bound by shared-memory / L1 operand traffic at 22% of the FP32 peak.  Transposing the
// roles of taps and outputs gives a real GEMM:
//     P[j, k] = sum_c x[c, j] * W[c, k]          M = input positions j,  N = 64 taps k = (kz,ky,kx),  K = Cin
//     out[2j - 1 + k] += P[j, k]                 col2im: every output voxel is the sum of 8 entries of P
// The A operand of the GEMM is the channel-blocked activation itself (no halo, no im2col): 128 consecutive positions of one
// (plane, channel group) are 128 contiguous 16-byte units = the K-major no-swizzle operand, fetched with plain bulk copies.
//
// CTA = one (sample, band of 2 input rows), sweeping z.  Per z step: 128 positions (one M-tile of 2 rows x 64) x 64 taps are
// accumulated in the registers of one consumer warpgroup (fp16 operands; OP 2 = the fp32-accurate hi/lo split of convt3d.cu:
// columns [0,64) hi*hi, [64,128) the 2^11-scaled cross terms: 128 fp32 registers per thread, which is what bounds the band),
// which stores hi + 2^-11 cross to a shared-memory image; 4 epilogue warps (one thread per position) then add the image into
// a ring of four output planes in shared memory while the consumers accumulate the next step.  Along x the two contributions of an output are summed in registers (warp shuffles; the two lanes at a warp
// seam exchange through a scratch), and the taps are processed in 4 phases (kz>>1, ky>>1): within a phase a position adds one
// float2 (outputs 2x, 2x+1) to each of 4 (kz, ky) rows and different positions hit different cells, so the adds are race-free
// without atomics; a barrier separates phases (shared-memory traffic: 1/4 of a per-tap scatter, and conflict-free).  Output
// planes 2z-1 and 2z are complete after step z (their other contributions came from step z-1, carried in the ring) and leave
// with 16-byte stores.  Only the two output rows on each side of a band are shared with the neighbouring band's CTA: those are
// added with red.global.add.v4.f32 onto zeroed rows (two commutative contributions: deterministic), zeroed by one strided
// memset before the launch.  The bias is added by exactly one contributor of every output.
#include <cuda_fp16.h>
#include "common.cuh"
#include "tc_ptx.cuh"

namespace gb {

constexpr int CI_W = 64;             // input width (positions per row)
constexpr int CI_ROWS = 2;           // input rows per band
constexpr int CI_POS = CI_W * CI_ROWS;   // positions per z step = 1 M-tile
constexpr int CI_MT = 1;
constexpr int CI_EPI_WARPS = 4 * CI_MT;   // one warp per (M-tile, 32-row quarter): a thread owns one input position per z step
constexpr int CI_THREADS = (CI_EPI_WARPS + 5) * 32;   // + consumer warpgroup + producer warp
constexpr int CI_ACC_LD = 64 + 4;        // accumulator image [CI_POS rows][CI_ACC_LD] fp32
constexpr int CI_MAX_STAGES = 6;
constexpr int CI_UY = 2 * CI_ROWS + 2;   // output rows touched by a band
constexpr int CI_PITCH = 136;            // floats per ring row: column ux + 3 holds output x = ux - 1 (x = 0 is 16-byte aligned)
constexpr int CI_PLANE = CI_UY * CI_PITCH;

struct ColParams {
  const __half *src0, *src1;   // blocked [B*D][parts*cg][H][64][8 fp16]
  int cg0, cg1;                // channel groups of 8 per part
  int B, D, H;
  const __half *wpack;         // [ksteps][2 kcore][NACC/8][8][8]
  int ksteps, stages;
  const float *bias;           // 1 value
  float *out;                  // [B][2D][2H][128]
};

__device__ __forceinline__ void named_bar_sync(int id, int count) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(count) : "memory"); }

__device__ __forceinline__ void red_add_v4(float *p, float4 v) {
  asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(p), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w) : "memory");
}

template <int OP>
__global__ void __launch_bounds__(CI_THREADS, 1) convt_c1_col2im_kernel(const ColParams p) {
  constexpr bool X2 = OP == 2;
  constexpr int PARTS = X2 ? 2 : 1;
  constexpr int NACC = PARTS * 64;
  constexpr int CG_BYTES = CI_POS * 16;                  // one channel group of one part: CI_ROWS rows x 64 positions x 16 B
  constexpr int STAGE_BYTES = PARTS * 2 * CG_BYTES;      // one K step (16 channels)
  constexpr int W_KSTEP_BYTES = 2 * (NACC / 8) * 128;
  extern __shared__ __align__(128) uint8_t smem[];
  uint8_t *stages = smem;
  uint8_t *sw = smem + (size_t)p.stages * STAGE_BYTES;
  float *ring = reinterpret_cast<float *>(sw + (size_t)p.ksteps * W_KSTEP_BYTES);
  float *acc_img = ring + 4 * CI_PLANE;
  uint64_t *full = reinterpret_cast<uint64_t *>(acc_img + CI_POS * CI_ACC_LD);
  uint64_t *empty = full + CI_MAX_STAGES;
  uint64_t *wbar = empty + CI_MAX_STAGES;
  uint64_t *acc_full = wbar + 1;     // the consumers have stored step z's accumulators to the image
  uint64_t *acc_empty = acc_full + 1;   // the epilogue has read them

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int band = blockIdx.x, nbands = gridDim.x, b = blockIdx.y;
  const int y0 = band * CI_ROWS;

  if (tid == 0) {
    for (int s = 0; s < p.stages; ++s) {
      mbar_init(&full[s], 1);
      mbar_init(&empty[s], 4);    // the 4 consumer warps
    }
    mbar_init(wbar, 1);
    mbar_init(acc_full, 128);
    mbar_init(acc_empty, CI_EPI_WARPS * 32);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if (warp == CI_EPI_WARPS + 4) {
    // ===================== producer =============================================================================
    if (lane == 0) {
      mbar_arrive_expect_tx(wbar, (uint32_t)(p.ksteps * W_KSTEP_BYTES));
      bulk_g2s(sw, p.wpack, (uint32_t)(p.ksteps * W_KSTEP_BYTES), wbar);
      int it = 0;
      for (int z = 0; z < p.D; ++z) {
        const size_t bd = (size_t)b * p.D + z;
        for (int ks = 0; ks < p.ksteps; ++ks, ++it) {
          const int s = it % p.stages, use = it / p.stages;
          if (use > 0) mbar_wait(&empty[s], (use - 1) & 1);
          uint8_t *sa = stages + (size_t)s * STAGE_BYTES;
          mbar_arrive_expect_tx(&full[s], (uint32_t)STAGE_BYTES);
#pragma unroll
          for (int part = 0; part < PARTS; ++part) {
#pragma unroll
            for (int c = 0; c < 2; ++c) {
              int cg = ks * 2 + c;
              const __half *src = p.src0;
              int ncg = p.cg0;
              if (cg >= p.cg0) { cg -= p.cg0; src = p.src1; ncg = p.cg1; }
              const __half *g = src + ((((bd * PARTS + part) * ncg + cg) * p.H + y0) * (size_t)CI_W) * 8;
              bulk_g2s(sa + (part * 2 + c) * CG_BYTES, g, (uint32_t)CG_BYTES, &full[s]);
            }
          }
        }
      }
    }
  } else if (warp >= CI_EPI_WARPS) {
    // ===================== consumers: the two m64 halves of the M-tile, accumulators in registers =====================
    static_assert(CI_MT == 1, "one consumer warpgroup holds one M-tile");
    mbar_wait(wbar, 0);
    int it = 0;
    for (int z = 0; z < p.D; ++z) {
      float acc[2][NACC / 2];
#pragma unroll
      for (int h = 0; h < 2; ++h)
#pragma unroll
        for (int j = 0; j < NACC / 2; ++j) acc[h][j] = 0.0f;
      for (int ks = 0; ks < p.ksteps; ++ks, ++it) {
        const int s = it % p.stages, use = it / p.stages;
        mbar_wait(&full[s], use & 1);
        wgmma_fence();
        const uint32_t sa = smem_u32(stages + (size_t)s * STAGE_BYTES);
        const uint64_t bdesc = gmma_desc(smem_u32(sw) + ks * W_KSTEP_BYTES, (NACC / 8) * 128, 128);
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const uint32_t a0 = sa + h * 64 * 16;
          wgmma_f16<NACC>(acc[h], gmma_desc(a0, CG_BYTES, 128), bdesc);
          if constexpr (X2) wgmma_f16<64>(acc[h] + 32, gmma_desc(a0 + 2 * CG_BYTES, CG_BYTES, 128), bdesc);
        }
        wgmma_commit();
        wgmma_wait<0>();
        __syncwarp();
        if (lane == 0) mbar_arrive(&empty[s]);
      }
      if (z > 0) mbar_wait(acc_empty, (z - 1) & 1);   // the epilogue has read step z-1's accumulators
#pragma unroll
      for (int h = 0; h < 2; ++h) store_acc_tile<64, X2>(acc[h], acc_img + h * 64 * CI_ACC_LD, CI_ACC_LD);
      mbar_arrive(acc_full);
    }
  } else {
    // ===================== epilogue: accumulator image -> scatter-add into the plane ring -> global ======================
    const int etid = tid;                                 // 0..CI_EPI_WARPS*32 - 1
    const int quarter = warp & 3, mt = warp >> 2;         // 32-row quarter of this warp; its M-tile
    const int row = quarter * 32 + lane;                  // accumulator row within the M-tile: input row (row >> 6), x = row & 63
    const int x = row & 63;
    const int yl = 2 * mt + (row >> 6);                   // input row of this thread within the band
    for (int i = etid; i < 4 * CI_PLANE; i += CI_EPI_WARPS * 32) ring[i] = 0.0f;
    named_bar_sync(1, CI_EPI_WARPS * 32);
    const float bias = __ldg(p.bias);
    const int Ho = 2 * p.H, Do = 2 * p.D;
    constexpr int Wo = 2 * CI_W;
    const float *arow = acc_img + (size_t)(mt * 128 + row) * CI_ACC_LD;
    // ring cell of output column ox = 2x of this thread's two input rows (column ox + 4: even, so an (ox, ox + 1) pair is one float2)
    float *base = ring + (2 * yl) * CI_PITCH + 2 * x + 4;
    const int xhalf = quarter & 1, ysub = quarter >> 1;
    // taps kx = 3 of x = 31 and kx = 0 of x = 32 belong to cells of the neighbouring warp: exchanged through this scratch
    float *scr = reinterpret_cast<float *>(acc_empty + 1);   // [2 buffers][M-tile: 4 slots, CI_MT used][2 rows][2 directions][4 (rz,ry)]

    auto flush_plane = [&](int slot, int oz) {   // complete plane -> global, ring slot back to zero
      float *pl = ring + slot * CI_PLANE;
      for (int i = etid; i < CI_UY * (Wo / 4); i += CI_EPI_WARPS * 32) {
        const int uy = i / (Wo / 4), q = i - uy * (Wo / 4);
        float4 *sp = reinterpret_cast<float4 *>(pl + uy * CI_PITCH + 4 + 4 * q);
        float4 v = *sp;
        *sp = make_float4(0.f, 0.f, 0.f, 0.f);
        const int oy = 2 * y0 - 1 + uy;
        if (oy < 0 || oy >= Ho) continue;
        if (uy >= 2 || band == 0) { v.x += bias; v.y += bias; v.z += bias; v.w += bias; }
        float *dst = p.out + (((size_t)b * Do + oz) * Ho + oy) * (size_t)Wo + 4 * q;
        const bool shared_row = (uy <= 1 && band > 0) || (uy >= CI_UY - 2 && band < nbands - 1);
        if (shared_row) red_add_v4(dst, v);
        else st_stream_f4(dst, v);
      }
    };

    for (int z = 0; z < p.D; ++z) {
      mbar_wait(acc_full, z & 1);
      const int zs = (2 * z) & 3;   // ring slot of tap kz = 0 (output plane 2z - 1); tap kz uses (zs + kz) & 3
      // 4 phases (tz, ty): the 16 taps (rz, ry, kx = 0..3) of a position.  Along x the two contributions of an output are
      // summed in registers first (ox = 2x: kx = 1 of x and kx = 3 of x - 1; ox = 2x + 1: kx = 2 of x and kx = 0 of x + 1, via
      // warp shuffles), so a position adds ONE float2 per (kz, ky) to the ring: distinct cells for distinct positions.
      // The 4 ring cells are loaded before any of them is touched (no load-add-store chains).
      float *pb[4];   // this position's cell row in the ring plane of tap kz
#pragma unroll
      for (int k = 0; k < 4; ++k) pb[k] = base + ((zs + k) & 3) * CI_PLANE;
#pragma unroll
      for (int ph = 0; ph < 4; ++ph) {
        const int tz = ph >> 1, ty = ph & 1;
        float v[16];   // index tx * 8 + rz * 4 + ry * 2 + rx, kx = 2 tx + rx
        ld_row<16>(arow + ph * 16, v);
        if (ph == 3) mbar_arrive(acc_empty);   // the last read of this step's image: the consumers may overwrite it
        float *sb = scr + (ph & 1) * 64 + (mt * 2 + ysub) * 8;
        if (lane == 31 && xhalf == 0) {
#pragma unroll
          for (int j = 0; j < 4; ++j) sb[j] = v[8 + 2 * j + 1];       // kx = 3 of x = 31
        }
        if (lane == 0 && xhalf == 1) {
#pragma unroll
          for (int j = 0; j < 4; ++j) sb[4 + j] = v[2 * j];           // kx = 0 of x = 32
        }
        named_bar_sync(1, CI_EPI_WARPS * 32);   // scratch visible; the previous phase's adds are done
        float2 a[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) {           // j = rz * 2 + ry
          const int kz = 2 * tz + (j >> 1), ky = 2 * ty + (j & 1);
          a[j] = *reinterpret_cast<const float2 *>(pb[kz] + ky * CI_PITCH);
        }
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          float up = __shfl_up_sync(0xffffffffu, v[8 + 2 * j + 1], 1), dn = __shfl_down_sync(0xffffffffu, v[2 * j], 1);
          if (lane == 0) up = xhalf ? sb[j] : 0.0f;          // x = 0: output -1 does not exist
          if (lane == 31) dn = xhalf ? 0.0f : sb[4 + j];     // x = 63: output 128 does not exist
          a[j].x += v[2 * j + 1] + up;      // ox = 2x:     kx = 1 here + kx = 3 of x - 1
          a[j].y += v[8 + 2 * j] + dn;      // ox = 2x + 1: kx = 2 here + kx = 0 of x + 1
        }
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const int kz = 2 * tz + (j >> 1), ky = 2 * ty + (j & 1);
          *reinterpret_cast<float2 *>(pb[kz] + ky * CI_PITCH) = a[j];
        }
      }
      named_bar_sync(1, CI_EPI_WARPS * 32);     // all adds of this step are in the ring
      // planes 2z - 1 (tap kz = 0) and 2z (kz = 1) have received everything
      if (z > 0) flush_plane(zs, 2 * z - 1);
      else {      // output plane -1 does not exist: drop what tap kz = 0 of the first step scattered
        float *pl = ring + zs * CI_PLANE;
        for (int i = etid; i < CI_PLANE; i += CI_EPI_WARPS * 32) pl[i] = 0.0f;
      }
      flush_plane((zs + 1) & 3, 2 * z);
      named_bar_sync(1, CI_EPI_WARPS * 32);
    }
    // the last step's tap kz = 2 plane (output 2D - 1) has no later contributor; its kz = 3 plane (output 2D) is dropped
    flush_plane((2 * (p.D - 1) + 2) & 3, Do - 1);
  }
}

template <int OP>
static int launch_col2im(ColParams &p, cudaStream_t st) {
  constexpr int PARTS = OP == 2 ? 2 : 1, NACC = PARTS * 64;
  constexpr int STAGE_BYTES = PARTS * 2 * CI_POS * 16;
  // weights + plane ring + accumulator image + barriers and exchange scratch
  const int fixed = p.ksteps * 2 * (NACC / 8) * 128 + 4 * CI_PLANE * 4 + CI_POS * CI_ACC_LD * 4 + 1024;
  int stages = (226 * 1024 - fixed) / STAGE_BYTES;
  if (stages > CI_MAX_STAGES) stages = CI_MAX_STAGES;
  GB_REQUIRE(stages >= 2, GENRE_B200_EINVAL, "convt_c1_col2im: %d K steps of weights leave no room for the pipeline", p.ksteps);
  p.stages = stages;
  const size_t smem = (size_t)stages * STAGE_BYTES + fixed;
  auto kern = convt_c1_col2im_kernel<OP>;
  static bool configured[64] = {};
  int dev = 0;
  cudaGetDevice(&dev);
  if (!configured[dev & 63]) {
    if (cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024) != cudaSuccess)
      return check_launch("convt_c1_col2im: cudaFuncSetAttribute");
    configured[dev & 63] = true;
  }
  dim3 grid((unsigned)(p.H / CI_ROWS), (unsigned)p.B);
  kern<<<grid, CI_THREADS, smem, st>>>(p);
  return check_launch("convt_c1_col2im kernel");
}

}  // namespace gb

using namespace gb;

// ConvTranspose3d(8*(cg0+cg1) -> 1, kernel 4, stride 2, padding 1) on channel-blocked fp16 operands of a [B, C, D, H, 64] volume.
//   src0 [B*D][parts*cg0][H][64][8 fp16], src1 likewise with cg1 groups or NULL (the second half of a skip concatenation);
//   parts = 1 (op 1: fp16 operands) or 2 (op 2: hi | lo' = (a - hi) * 2^11 parts: fp32-accurate); cg0 + cg1 even; H % 8 == 0;
//   wpack [(cg0+cg1)/2][2][parts*8][8][8] fp16: row n = t*8 + r holds tap k = 2t + r per dimension (ops_conv.pack_convt_c1_col2im_weights);
//   bias: 1 float on the device;  out [B][2D][2H][128] fp32, fully overwritten.
extern "C" int genre_b200_convt_c1_col2im_forward(const void *src0, int cg0, const void *src1, int cg1, int64_t B, int64_t D, int64_t H,
                                                  int64_t W, const void *wpack, int op, const float *bias, float *out, void *stream) {
  GB_REQUIRE(src0 && wpack && bias && out, GENRE_B200_EINVAL, "convt_c1_col2im: null pointer");
  GB_REQUIRE(cg0 > 0 && cg1 >= 0 && (cg1 == 0 || src1) && (cg0 + cg1) % 2 == 0, GENRE_B200_EINVAL, "convt_c1_col2im: bad channel groups");
  GB_REQUIRE(B > 0 && B <= 65535 && D > 0 && H > 0 && H % CI_ROWS == 0 && W == CI_W, GENRE_B200_EINVAL,
             "convt_c1_col2im: extent %lldx%lldx%lld unsupported (W = 64, H %% 8 == 0)", (long long)D, (long long)H, (long long)W);
  GB_REQUIRE(op == 1 || op == 2, GENRE_B200_EINVAL, "convt_c1_col2im: op %d (1 = fp16, 2 = fp16 hi/lo)", op);
  GB_REQUIRE(aligned16(src0) && aligned16(wpack) && aligned16(out) && (!src1 || aligned16(src1)), GENRE_B200_EALIGN, "convt_c1_col2im: alignment");
  ColParams p{};
  p.src0 = (const __half *)src0; p.src1 = (const __half *)src1;
  p.cg0 = cg0; p.cg1 = cg1;
  p.B = (int)B; p.D = (int)D; p.H = (int)H;
  p.wpack = (const __half *)wpack;
  p.ksteps = (cg0 + cg1) / 2;
  p.bias = bias;
  p.out = out;
  cudaStream_t st = as_stream(stream);
  // zero the output rows two bands share (rows 2 R j - 1, 2 R j of every plane, R = CI_ROWS: pairs of adjacent rows at a pitch
  // of 2 R rows)
  const int64_t Wo = 2 * W, Ho = 2 * H, Do = 2 * D, nbands = H / CI_ROWS;
  const int64_t pairs = B * Do * nbands - 1;
  if (nbands > 1 && pairs > 0) {
    if (cudaMemset2DAsync(out + (2 * CI_ROWS - 1) * Wo, (size_t)2 * CI_ROWS * Wo * sizeof(float), 0, (size_t)2 * Wo * sizeof(float),
                          (size_t)pairs, st) != cudaSuccess)
      return check_launch("convt_c1_col2im: memset");
  }
  (void)Ho;
  return op == 2 ? launch_col2im<2>(p, st) : launch_col2im<1>(p, st);
}
