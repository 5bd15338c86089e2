// convt3d.cu — stride-2 ConvTranspose3d forward as a wgmma (Hopper warpgroup tensor core) implicit GEMM, TF32 in / FP32 out.
//
// Reference layers: networks/networks.py:162-167 (Unet_3D.dec2..dec6 = Deconv3d_skip: cat(x, skip) ->
// ConvTranspose3d(k, s=2, p) [-> BatchNorm3d -> LeakyReLU]), :253-256,:40-57 (VoxelDecoder / VoxelGenerator
// deconv3d_2x).  The dominant one, dec5 = ConvT(80 -> 20, k=8, s=2, p=3) on 32^3, is 53.7 of Unet_3D's 78 GFLOP.
//
// Formulation.  o = 2 i - p + k splits the output into 8 parity classes (o = 2 j + par); class `par` only sees
// the taps k = k0 + 2 t, t < T = K/2, at input positions i = j + base - t: a stride-1 T^3-tap convolution.
//     GEMM per class:  M = B * D*H*W positions,  N = Cout (padded to NPAD),  K = T^3 * Cin
// Activations are kept channel-BLOCKED: [B*D][C/4][H][W][4] (16 bytes per position and channel group), so
//   * a shared-memory halo [cg][y][x][4] is exactly wgmma's canonical K-major NO-SWIZZLE operand layout
//     (core matrix = 8 consecutive x positions x 16 B; next y row = SBO; next channel group = LBO), and
//   * the operand of ANY tap is the same halo at a different 16-byte-aligned start address: one halo load feeds
//     T*T (y,x) taps and MT M-tiles, which is what keeps the kernel off the L2 bandwidth wall at N = 20.
// The two sources of the skip concatenation are two tensors walked one after the other along K (the cat is never
// materialised).  Weights are pre-packed on the host into the exact shared-memory image of each (parity, z-tap,
// K-chunk) stage and arrive with ONE cp.async.bulk per stage.
//
// CTA = one (b, z, 16 y-rows, 8*MT x-columns) output slab of one parity class: MT M-tiles of 128 rows.  Warps 0-3: one
// thread issues the halo tensor copies (out-of-range elements zero-filled = padding) and the weight copy of every stage, then
// all four run the epilogue (shared-memory accumulator image -> scale/shift/LeakyReLU -> blocked store).  Warps 4-11: two
// consumer warpgroups, each issuing the m64 wgmma of one half (8 y-rows) of every M-tile and holding its MT x NACC / 2 fp32
// accumulators in registers, so MT * NACC <= 256 (launch_convt_impl narrows the x tile until it fits).  After the last K
// step they store the accumulators to shared memory (over the drained pipeline ring) for the epilogue warps.  MODE 5 in the
// hi/lo split runs three consumer warpgroups (warps 4-15) on 192-position M-tiles (template parameter CW).
// Pipeline: STAGES-deep ring of (halo chunk, weight chunk) with full/empty mbarriers; every consumer warp arrives on a slot's
// empty barrier once its wgmma that read the slot have completed.  With 3 or more stages a stage's MMAs stay in flight while
// the next stage is awaited and issued (wgmma.wait_group 1): its slot is released after the next stage's MMAs are committed.
#include <cuda.h>   // CUtensorMap + the cuTensorMapEncodeTiled prototype (the entry point is resolved through the runtime: no -lcuda)
#include <cstring>
#include "common.cuh"
#include "tc_ptx.cuh"

namespace gb {

constexpr int CT_ACC_COLS = 256;      // accumulator columns per CTA (MT * NACC): 128 fp32 registers per consumer thread
constexpr int CT_BY = 16;             // y rows per CTA (16 core-matrix groups of 8 x positions = M 128)
constexpr int CT_KCG = 2;             // channel groups (of 4) per stage = one K=8 TF32 MMA per tap and M-tile

struct ConvTParams {
  const float *src0, *src1;  // blocked activations [B*D][cg][H][W][16 bytes]; src1 may be null (cg1 = 0).
                             // A channel group is 16 bytes per position: 4 fp32 (TF32 path) or 8 fp16 (F16 path).
  int cg0, cg1;
  int B, D, H, W;            // input extent
  const float *wpack;        // [8 parity][T ztap][nchunk][T*T taps][2 kcore][NPAD/8][8][4]
  const float *scale, *shift;  // per output channel (NPAD entries): y = act(acc * scale + shift)
  float slope;               // LeakyReLU slope (1 = identity)
  float *out;                // blocked [B*2D][cgo][2H][2W][4]
  int cgo;                   // output channel groups
  int base[2];               // input index = j + base[par] - t
  int xtiles;                // the CTA tile is 8*MT positions wide; W = xtiles * 8 * MT (set by the launcher)
  int act_sigmoid = 0;       // MODE 4: apply a sigmoid after the bias
  int srcpar_cgs;            // 0, or: the K range is 8 parity sub-volumes of srcpar_cgs channel groups each (strided
                             // Conv3d k=4 s=2 p=1 after space-to-depth); sub-volume s = (pz,py,px) uses base 1 - p per dim
  // fp16 modes: the epilogue writes the fp16 operand(s) of the next layers instead of `out` when odst[0] is set (OP_PLAIN or
  // OP_PARITY layout, ocg groups of 8 channels, oparts parts: 2 = hi | lo' of split_hi_lo8, 1 = fp16).  Channels >= 4 * cgo
  // are written as zeros.
  uint4 *odst[2] = {nullptr, nullptr};
  int olayout[2] = {0, 0};
  int ocg[2] = {0, 0};
  int oparts = 0;
  // Unet_3D.enc1 in split-z MODE 2 over fp16 groups of 8 (conv3d_k8s2_s4d, npad 80): K chunk kc holds the 16 space-to-depth
  // channels (c, rz) = (kc >> 2, kc & 3), and z tap tz of z class pz reads kernel tap 7 - 4 tz + rz - 2 pz, so the stages
  // where that lies outside [0, 8) carry only zero weights and are skipped (a third of them)
  int s4d_zskip = 0;
};
// operand output layouts (Do, Ho, Wo: the output extent)
//   OP_PLAIN   [B*Do][oparts][ocg][Ho][Wo][8 fp16]: the blocked operand of a following ConvTranspose3d
//   OP_PARITY  [B*Do/2][oparts][8 s][ocg][Ho/2][Wo/2][8 fp16], s = ((z&1)*2 + (y&1))*2 + (x&1): the parity sub-volumes of a
//              following Conv3d(k 4, s 2, p 1) (genre_b200_ncdhw_to_blocked mode 2, cpad = 8 * ocg)
constexpr int OP_PLAIN = 1, OP_PARITY = 2;

// one 8-channel group k of output position (b, oz, oy, ox) into every operand destination that has a group k
__device__ __forceinline__ void store_operand(const ConvTParams &p, int k, int b, int oz, int oy, int ox, int Do, int Ho, int Wo,
                                              const float (&v)[8]) {
  uint4 u[2];
  if (p.oparts == 2) split_hi_lo8(v, u[0], u[1]);
  else u[0] = pack_f16x8(v);
#pragma unroll
  for (int d = 0; d < 2; ++d) {
    if (p.odst[d] == nullptr || k >= p.ocg[d]) continue;
    size_t idx, pstride;
    if (p.olayout[d] == OP_PLAIN) {
      pstride = (size_t)p.ocg[d] * Ho * Wo;
      idx = ((size_t)(b * Do + oz) * p.oparts * p.ocg[d] + k) * ((size_t)Ho * Wo) + (size_t)oy * Wo + ox;
    } else {
      const int H2 = Ho >> 1, W2 = Wo >> 1, s = ((oz & 1) * 2 + (oy & 1)) * 2 + (ox & 1);
      pstride = (size_t)8 * p.ocg[d] * H2 * W2;
      idx = (((size_t)(b * (Do >> 1) + (oz >> 1)) * p.oparts * 8 + s) * p.ocg[d] + k) * ((size_t)H2 * W2) + (size_t)(oy >> 1) * W2 + (ox >> 1);
    }
    p.odst[d][idx] = u[0];
    if (p.oparts == 2) p.odst[d][idx + pstride] = u[1];
  }
}

// ---- the kernel ----------------------------------------------------------------------------------------------
// T: taps per dimension of a parity class (K/2: 2 for k=4, 4 for k=8); NPAD: padded Cout (32 or 64); MT = W/8.
// X2: the fp32-accurate fp16 hi/lo operand split.  Activations arrive as [B*D][2 parts: hi, lo'][cg][H][W][8 fp16] with
// lo' = (a - hi) * 2^11, weights as [W_hi | W_lo'] side by side along N (lo' = (w - hi) * 2^11).  Per K step and tap,
// three N = NPAD MMAs, in this order:
//     A_hi  x W_hi   ->  accumulator columns [0, NPAD)        (acc_hi)
//     A_hi  x W_lo'  ->  accumulator columns [NPAD, 2*NPAD)   (acc_cross)
//     A_lo' x W_hi   ->  accumulator columns [NPAD, 2*NPAD)   (acc_cross)
// so the hi*hi products and the 2^11-scaled cross terms keep separate accumulators (the tensor core's fp32 accumulator
// truncates: a step's error scales with the partial sum it joins, and the cross terms would otherwise ride on the big one),
// and the epilogue returns acc_hi + 2^-11 * acc_cross.  The first two could be one N = 2*NPAD MMA, but the third would then
// write into half of its registers, which makes ptxas serialize every wgmma of the kernel.
// The halo of a channel group arrives as ONE cp.async.bulk.tensor (5-D tiled tensor map over [plane][cg][H][W][16 B], box
// [1][1][PY][PX][16 B], out-of-bounds elements zero-filled = the convolution's padding); each channel group starts on a
// 128-byte boundary of shared memory (the LBO of the A descriptor is that padded stride).
// PW > 0: the paired form of MODE 5 over an input PW wide.  Its halo is flattened: rows of pitch PX = PW + 2 (input x from
// -2, the two columns past the right edge of a row are the zero columns of the next), PY rows = enough for MT * M
// consecutive positions starting anywhere in a row plus the 3 rows and 3 columns the taps reach (see the kernel).
// CW: consumer warpgroups, each issuing the m64 MMAs of 64 rows of every M-tile, so an M-tile is M = 64 * CW rows.  Only the
// paired form takes CW = 3 (its positions are a flat run; the other modes' 128-row tiles are 16 y-rows x 8 x-columns).
template <int T, int NPAD, int MT, bool X2 = false, int PW = 0, int CW = 2>
struct ConvTCfg {
  static constexpr int M = 64 * CW;
  static constexpr int W = 8 * MT;
  static constexpr int PY = PW ? (M * MT + (T + 1) * (PW + 2) + 1) / (PW + 2) : CT_BY + T - 1;   // halo extent
  static constexpr int PX = PW ? PW + 2 : W + T - 1;
  static constexpr int PARTS = X2 ? 2 : 1;
  static constexpr int NACC = PARTS * NPAD;                    // accumulator columns per M-tile = width of the B operand
  static constexpr int A_CG_BYTES = PY * PX * 16;              // one channel group of the halo
  static constexpr int A_CG_STRIDE = ((A_CG_BYTES + 127) / 128) * 128;   // its pitch in shared memory = LBO of A
  static constexpr int A_BYTES = PARTS * CT_KCG * A_CG_STRIDE; // [part][channel group][halo]
  static constexpr int A_TX_BYTES = PARTS * CT_KCG * A_CG_BYTES;  // bytes the tensor copies of one stage deliver
  static constexpr int B_TAP_BYTES = 2 * (NACC / 8) * 128;     // one (y,x) tap: [2 kcore][NACC/8][8 rows][16 B]
  // A stage holds the halo of one (z tap, K chunk) and the weights of ROWS of its T tap rows; YS = T / ROWS (rounded up)
  // stages walk the same halo when all T*T taps do not fit twice into shared memory (X2 with 5x5 union taps: 128 KB).
  // dec5's union form (MODE 2, X2) keeps 2 stages of 3 + 2 tap rows: 3 stages of 2 + 2 + 1 rows would let its MMAs stay in
  // flight across stages (the kernel's INFLIGHT), but load each halo three times, and measured 5.40 ms per call against 4.97
  // (H100 80GB HBM3, 700 W).  Its paired form (MODE 5, X2: 16 taps, 97 KB per stage) takes all 4 tap rows in one stage,
  // a 2-stage ring that loads each halo once: 3.75 ms per call, against 4.25 ms for 2 + 2 rows in a 3-stage ring with MMAs
  // in flight and every halo loaded twice (H100 80GB HBM3, 700 W, SM clock 1.92-1.98 GHz, B = 16).  With CW = 3 (192
  // positions, 10 halo rows at W = 32) a stage is 101 KB and the ring still holds 2.
  static constexpr int stage_bytes(int ys) { return ((A_BYTES + ((T + ys - 1) / ys) * T * B_TAP_BYTES + 127) / 128) * 128; }
  static constexpr int pick_ys() {
    for (int ys = 1; ys < T; ++ys)
      if (2 * stage_bytes(ys) <= 218 * 1024) return ys;
    return T;
  }
  static constexpr int YS = pick_ys();
  static constexpr int ROWS = (T + YS - 1) / YS;
  static constexpr int rows_of(int ys) { return (ys + 1) * ROWS <= T ? ROWS : T - ys * ROWS; }   // tap rows of stage ys
  static constexpr int B_BYTES = ROWS * T * B_TAP_BYTES;
  static constexpr int STAGE_BYTES = stage_bytes(YS);
  // one CTA per SM (the accumulators take half the register file): the whole 227 KB of shared memory serves the ring
  static constexpr int STAGES = (218 * 1024) / STAGE_BYTES > 6 ? 6 : (218 * 1024) / STAGE_BYTES;
  // epilogue image of the accumulators, [M rows][MT * NPAD (+ 4 pad) columns] fp32, over the drained ring
  static constexpr int ACC_LD = MT * NPAD + 4;
  static constexpr int ACC_BYTES = M * ACC_LD * 4;
  static constexpr int RING_BYTES = STAGES * STAGE_BYTES > ACC_BYTES ? STAGES * STAGE_BYTES : ACC_BYTES;
  static constexpr size_t SMEM = (size_t)RING_BYTES + 256;
  static_assert(STAGES >= 2, "stage too large");
  static_assert(MT * NACC <= CT_ACC_COLS, "accumulators exceed the register budget");
  static_assert(SMEM <= 227 * 1024, "shared memory");
  static_assert(NACC <= 256 && NACC % 16 == 0 && NPAD % 16 == 0 || !X2, "X2: MMA N must be a multiple of 16, at most 256");
  static_assert(PW == 0 || (T == 4 && PY <= 256 && PX <= 256), "paired form: 4 taps per dimension, tensor-copy box <= 256");
  static_assert(CW == 2 || (CW == 3 && PW > 0), "three consumer warpgroups: the paired form only");
};

// MODE 0: 8 parity classes (blockIdx.y), output at 2*j + parity (ConvTranspose3d stride 2); TZ = T = K/2 taps
// MODE 1: one class, output at j (stride-1 tap convolution; strided Conv3d arrives here after space-to-depth)
// MODE 2: ConvTranspose3d stride 2 with the four (y,x) parity classes MERGED along N (blockIdx.y = z parity): the
//         classes read the same halo at offsets that overlap in all but one tap per dimension, so one MMA over the
//         union of T = K/2 + 1 taps with N = 4 * Cout columns (n = (py*2+px)*Cout + co, zero weights where a class
//         does not use a tap) replaces four N = Cout MMAs.  An M128 MMA costs about the same 64+ cycles for any
//         N <= 128 (the A operand streams from shared memory at a fixed rate), so this is ~2.5x fewer tensor cycles.
//         TZ = K/2 z taps of the CTA's z parity.
// MODE 3: a stride-1 T-tap convolution whose N columns are the 8 output classes of a 2x upsampled grid
//         (n = ((qz*2+qy)*2+qx)*Cout + co, written to output position 2*j + q): a strided Conv3d(k 8, s 2, p 3) on
//         a 4x space-to-depth input (Unet_3D.enc1: 2 -> 128 channels, 3 taps, N = 8 x 20) - the same "few wide
//         MMAs instead of many narrow ones" trade as MODE 2, for a forward convolution.
// MODE 4: ConvTranspose3d(k 4, s 2, p 1) to ONE output channel (the last layer of every decoder): MODE 3's geometry with
//         N = 16 columns of which 8 are the output classes; the epilogue adds the bias (shift[0]), optionally applies
//         the sigmoid, and writes the NCDHW fp32 volume directly.
// MODE 5: MODE 2 with PAIRED classes (ConvTranspose3d k 8, s 2, p 3; the fp16 operand modes).  Output 2j (y parity 0 of
//         coarse j) and output 2j - 1 (parity 1 of coarse j - 1) read the same four inputs j + 1 - t, t < 4, with their own
//         tap t each, so coarse position j computes the pair (2j - 1, 2j) per dimension: 4 x 4 (y,x) taps, N = 4 * Cout, no
//         zero columns (MODE 2 walks the 5 x 5 union, 9 of its 25 taps zero for some class).  Coarse j then runs over
//         [0, H] x [0, W], which the 16 x 8 tiles cannot cover, so M is flattened per plane: position q = y * PX + x over a
//         halo of pitch PX = W + 2 starting at input x = -2.  Tap (ty, tx) is the same shared-memory array shifted by
//         ((3 - ty) * PX + 3 - tx) * 16 bytes; reads past a row's right edge land on the next row's two leading columns,
//         which are input x = -2, -1: zeros, the padding they need.  The A operand's 8-row core groups are 8 consecutive
//         positions (SBO = 128 B).  CTA = one (b, z parity, z plane, run of MT * M positions of the (H+1) x PX plane); the
//         epilogue drops x = W + 1 (the pitch's spare column), y > H and outputs -1 and 2H / 2W.  Per output the MMAs that
//         carry non-zero weights come in MODE 2's order (z tap, K chunk, y tap, x tap), and MODE 2's others add exact
//         zeros, so the two modes give bit-identical results.
// OP: operand type: 0 = TF32 (fp32 storage), 1 = fp16, 2 = fp16 hi/lo split (X2, see ConvTCfg), 3 = TF32 operands of the
//     3xTF32 split (lo | hi | hi along K) with a two-level accumulator: the tensor core's fp32 accumulator truncates, so a
//     step's error scales with the partial sum it joins, and over the thousands of K steps of a k=8 layer (Unet_3D.dec5's
//     input gradient: 3 x 1280) that bias grows past 1e-4 of the result.  OP 3 hands each stage's MMA partial sums to a
//     second register set with round-to-nearest fp32 adds and restarts the MMA accumulator from 0; the two sets take the
//     register budget of twice the columns (launch_convt_impl narrows the tile as for X2).
// PW: the input width of MODE 5 (its halo pitch is compile-time), 0 otherwise.
// CW: consumer warpgroups (ConvTCfg).  MODE 5 in the hi/lo split runs CW = 3: M-tiles of 192 positions, so every stage's
// weights (80 KB) serve 192 positions instead of 128.  The accumulators of one M-tile (80 registers per thread) leave room
// for a third warpgroup within the 128 registers per thread of a 512-thread CTA.
template <int TZ, int T, int NPAD, int MT, int MODE, int OP, int PW = 0, int CW = 2>
__global__ void __launch_bounds__(128 + 128 * CW, 1)
convt3d_s2_kernel(const ConvTParams p, const __grid_constant__ CUtensorMap tmap0, const __grid_constant__ CUtensorMap tmap1) {
  constexpr bool F16 = OP == 1 || OP == 2, X2 = OP == 2, FLUSH = OP == 3;
  using Cfg = ConvTCfg<T, NPAD, MT, X2, PW, CW>;
  constexpr int NACC = Cfg::NACC;
  static_assert(!FLUSH || 2 * MT * NACC <= CT_ACC_COLS, "two-level accumulators exceed the register budget");
  constexpr bool PAR = MODE == 0, MERGE = MODE == 2, MERGE8 = MODE == 3, C1 = MODE == 4, PAIR = MODE == 5;
  static_assert(PAIR == (PW > 0), "MODE 5 and only MODE 5 takes an input width");
  // a stage's MMAs stay in flight while the next stage is issued (its slot is released one stage late) only with a ring of 3
  // or more, where the producer still has a slot to fill meanwhile; OP 3 reads its accumulators after every stage
  constexpr int INFLIGHT = Cfg::STAGES >= 3 && !FLUSH ? 1 : 0;
  extern __shared__ __align__(128) uint8_t smem[];
  uint8_t *stages = smem;
  uint64_t *full = reinterpret_cast<uint64_t *>(smem + (size_t)Cfg::RING_BYTES);
  uint64_t *empty = full + Cfg::STAGES;
  float *acc_img = reinterpret_cast<float *>(smem);   // after the main loop: [M rows][ACC_LD]

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int par = blockIdx.y;  // parity class: bit 2 = z, bit 1 = y, bit 0 = x
  const int pz = MERGE || PAIR ? par : (par >> 2) & 1, py = (par >> 1) & 1, px = par & 1;
  const int ytiles = PAIR ? 1 : p.H / CT_BY;
  const int xt = blockIdx.x % p.xtiles;   // MODE 5: the run of positions within the plane
  const int tile = blockIdx.x / p.xtiles;
  const int yt = tile % ytiles;
  const int zj = (tile / ytiles) % p.D;
  const int b = tile / (ytiles * p.D);
  const int y0 = yt * CT_BY, x0 = xt * Cfg::W;
  // MODE 5: the CTA's first position q0, the plane row yq0 it lies in and its offset in that row; halo row r holds input row
  // yq0 - 2 + r, so position q under tap (ty, tx) reads halo element q - yq0 * PX + (3 - ty) * PX + 3 - tx
  const int q0 = xt * Cfg::M * MT, yq0 = q0 / Cfg::PX, qoff = q0 - yq0 * Cfg::PX;
  const int nchunk = (p.cg0 + p.cg1) / CT_KCG;

  // (z tap, K chunk) enumeration shared by the producer and the MMA issuer: qq = tz * nchunk + kc, skipped when the z tap
  // plane of that K chunk lies outside the input (it contributes nothing), and with s4d_zskip when its weights are all zero
  // (an MMA whose products are all zero leaves the accumulator's value as it is).  Each qq is YS stages, stage ys holding the
  // tap rows [ys * ROWS, min(T, ys * ROWS + ROWS)): an unrolled loop, so every stage's MMA sequence has a compile-time
  // shape (a runtime bound on the tap rows makes ptxas serialize every wgmma).  The per-dimension base offset of a chunk
  // is uniform (parity class / plain convolution) or a function of the chunk's source sub-volume (strided conv).
  auto stage_of = [&](int qq, int &tz, int &kc, int &bz, int &by, int &bx) -> bool {
    tz = qq / nchunk;
    kc = qq - tz * nchunk;
    if (p.srcpar_cgs) {
      const int sv = ((kc * CT_KCG) / p.srcpar_cgs) & 7;  // & 7: the K range may hold several blocks of 8 sub-volumes (3xTF32)
      bz = 1 - ((sv >> 2) & 1);
      by = 1 - ((sv >> 1) & 1);
      bx = 1 - (sv & 1);
    } else {
      bz = p.base[pz];
      by = MERGE ? T / 2 : p.base[py];
      bx = MERGE ? T / 2 : p.base[px];
    }
    if (MERGE && p.s4d_zskip) {
      const int kz = 7 - 4 * tz + (kc & 3) - 2 * pz;
      if (kz < 0 || kz >= 8) return false;
    }
    const int zi = zj + bz - tz;
    return zi >= 0 && zi < p.D;
  };
  const int n_qq = TZ * nchunk;

  if (tid == 0) {
    for (int s = 0; s < Cfg::STAGES; ++s) {
      mbar_init(&full[s], 1);                    // the producer's expect_tx arrival (halo + weight bytes)
      mbar_init(&empty[s], 4 * CW);              // every consumer warp
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if (warp < 4) {
    // ===================== producer: ONE thread issues the tensor copies (halo) and the bulk copy (weights) of every stage ====
    if (tid == 0) {
      int it = 0;
      for (int qq = 0; qq < n_qq; ++qq) {
        int tz, kc, bz, by, bx;
        if (!stage_of(qq, tz, kc, bz, by, bx)) continue;
#pragma unroll
        for (int ys = 0; ys < Cfg::YS; ++ys) {
          const int s = it % Cfg::STAGES, use = it / Cfg::STAGES;
          ++it;
          if (use > 0) mbar_wait(&empty[s], (use - 1) & 1);
          uint8_t *sa = stages + (size_t)s * Cfg::STAGE_BYTES;
          // weights of tap rows [ys*ROWS, ...) of this (class, z tap, K chunk): a contiguous slice of its T*T-tap block
          const uint32_t wbytes = (uint32_t)(Cfg::rows_of(ys) * T * Cfg::B_TAP_BYTES);
          const float *wsrc = p.wpack + ((((size_t)par * TZ + tz) * nchunk + kc) * (size_t)(T * T * Cfg::B_TAP_BYTES / 4)) +
                              (size_t)ys * Cfg::ROWS * T * (Cfg::B_TAP_BYTES / 4);
          mbar_arrive_expect_tx(&full[s], wbytes + (uint32_t)Cfg::A_TX_BYTES);
          bulk_g2s(sa + Cfg::A_BYTES, wsrc, wbytes, &full[s]);
          const int zi = zj + bz - tz;
          const int gy0 = PAIR ? yq0 - 2 : y0 + by - (T - 1), gx0 = PAIR ? -2 : x0 + bx - (T - 1);  // halo row r = input row gy0 + r
#pragma unroll
          for (int part = 0; part < Cfg::PARTS; ++part) {
#pragma unroll
            for (int c = 0; c < CT_KCG; ++c) {
              int cg = kc * CT_KCG + c;
              const CUtensorMap *tm = &tmap0;
              if (cg >= p.cg0) { cg -= p.cg0; tm = &tmap1; }
              tma_load_5d(sa + (part * CT_KCG + c) * Cfg::A_CG_STRIDE, tm, gx0, gy0, cg, (b * p.D + zi) * Cfg::PARTS + part, &full[s]);
            }
          }
        }
      }
    }
  } else {
    // ===================== consumers: warpgroup wg issues the wgmma of rows [64 wg, 64 wg + 64) of every M-tile ===========
    const int wg = (warp - 4) >> 2;
    float acc[MT][NACC / 2];
    float tot[FLUSH ? MT : 1][FLUSH ? NACC / 2 : 1];   // OP 3: the round-to-nearest sum of the stages' MMA partial sums
#pragma unroll
    for (int mt = 0; mt < MT; ++mt)
#pragma unroll
      for (int j = 0; j < NACC / 2; ++j) acc[mt][j] = 0.0f;
    if constexpr (FLUSH) {
#pragma unroll
      for (int mt = 0; mt < MT; ++mt)
#pragma unroll
        for (int j = 0; j < NACC / 2; ++j) tot[mt][j] = 0.0f;
    }
    // frees a slot: this warp's wgmma that read it are done
    auto release = [&](int slot) {
      __syncwarp();
      if (lane == 0) mbar_arrive(&empty[slot]);
    };
    int it = 0;
    int held = -1;   // the slot of the last committed stage, whose MMAs may still be running
    for (int qq = 0; qq < n_qq; ++qq) {
      int tz, kc, bz, by, bx;
      if (!stage_of(qq, tz, kc, bz, by, bx)) continue;
#pragma unroll
      for (int ys = 0; ys < Cfg::YS; ++ys) {
        const int s = it % Cfg::STAGES, use = it / Cfg::STAGES;
        ++it;
        mbar_wait(&full[s], use & 1);
        wgmma_fence();
        const uint32_t sa = smem_u32(stages + (size_t)s * Cfg::STAGE_BYTES);
        const uint32_t sb = sa + Cfg::A_BYTES;
#pragma unroll
        for (int r = 0; r < Cfg::rows_of(ys); ++r) {
          const int ty = ys * Cfg::ROWS + r;
#pragma unroll
          for (int tx = 0; tx < T; ++tx) {
            const uint32_t btap = sb + (r * T + tx) * Cfg::B_TAP_BYTES;
            const uint64_t bdesc = gmma_desc(btap, (NACC / 8) * 128, 128);
#pragma unroll
            for (int mt = 0; mt < MT; ++mt) {
              // rows of this M-tile under tap (ty,tx): halo row (T-1-ty) + y, column (T-1-tx) + 8*mt + x; this warpgroup's
              // 64 rows are y = 8 wg .. 8 wg + 7.  MODE 5: positions q0 + M mt + 64 wg + [0, 64), consecutive in the
              // flattened halo, so an 8-row core group is 8 consecutive 16-byte positions
              constexpr uint32_t SBO = PAIR ? 128 : Cfg::PX * 16;
              const uint32_t a0 = PAIR ? sa + (qoff + Cfg::M * mt + 64 * wg + (T - 1 - ty) * Cfg::PX + (T - 1 - tx)) * 16
                                       : sa + (((T - 1 - ty + 8 * wg) * Cfg::PX) + (T - 1 - tx) + 8 * mt) * 16;
              const uint64_t adesc = gmma_desc(a0, Cfg::A_CG_STRIDE, SBO);
              if constexpr (X2) {
                // A_hi x W_hi into the hi accumulator, then the cross terms A_hi x W_lo' and A_lo' x W_hi, in that order,
                // into the cross accumulator: three N = NPAD MMAs on disjoint registers (an MMA that writes into part of
                // another's accumulator registers makes ptxas serialize every wgmma)
                const uint64_t adesc_lo = gmma_desc(a0 + CT_KCG * Cfg::A_CG_STRIDE, Cfg::A_CG_STRIDE, SBO);
                wgmma_f16<NPAD>(acc[mt], adesc, bdesc);
                wgmma_f16<NPAD>(acc[mt] + NPAD / 2, adesc, gmma_desc(btap + (NPAD / 8) * 128, (NACC / 8) * 128, 128));
                wgmma_f16<NPAD>(acc[mt] + NPAD / 2, adesc_lo, bdesc);
              } else if constexpr (F16) {
                wgmma_f16<NACC>(acc[mt], adesc, bdesc);
              } else {
                wgmma_tf32<NACC>(acc[mt], adesc, bdesc);
              }
            }
          }
        }
        wgmma_commit();
        if constexpr (!INFLIGHT) {
          wgmma_wait<0>();
          if constexpr (FLUSH) {
#pragma unroll
            for (int mt = 0; mt < MT; ++mt)
#pragma unroll
              for (int j = 0; j < NACC / 2; ++j) {
                tot[mt][j] += acc[mt][j];
                acc[mt][j] = 0.0f;
              }
          }
          release(s);
        } else {
          // keep this stage's MMAs in flight while the next stage's operands are awaited: only the previous stage's
          // must be done before its slot is handed back
          wgmma_wait<1>();
          if (held >= 0) release(held);
          held = s;
        }
      }
    }
    wgmma_wait<0>();
    if (held >= 0) release(held);
    // every stage has been consumed, so no copy can still land in the ring: it becomes the accumulator image
    asm volatile("bar.sync 1, %0;" ::"n"(128 * CW) : "memory");   // ... by EVERY consumer warpgroup: another may still read it
#pragma unroll
    for (int mt = 0; mt < MT; ++mt) {
      if constexpr (FLUSH) store_acc_tile<NPAD, X2>(tot[mt], acc_img + (size_t)(64 * wg) * Cfg::ACC_LD + mt * NPAD, Cfg::ACC_LD);
      else store_acc_tile<NPAD, X2>(acc[mt], acc_img + (size_t)(64 * wg) * Cfg::ACC_LD + mt * NPAD, Cfg::ACC_LD);
    }
  }
  __syncthreads();
  if (tid < Cfg::M) {
    // ===================== epilogue: accumulator image -> act(acc*scale+shift) -> blocked global store ===============
    // one accumulator row per thread: the 4 producer warps, joined by the first 2 consumer warps when CW = 3
    const int m = tid;
    const float *arow = acc_img + (size_t)m * Cfg::ACC_LD;
    const int yy = m >> 3, xx = m & 7;
    constexpr bool UP = PAR || MERGE || MERGE8 || C1 || PAIR;
    const int Ho = UP ? 2 * p.H : p.H, Wo = UP ? 2 * p.W : p.W, Do = UP ? 2 * p.D : p.D;
    const int oz_plain = UP ? 2 * zj + pz : zj, oy = PAR ? 2 * (y0 + yy) + py : y0 + yy;
    auto act = [&](float a, int n) {
      const float t = fmaf(a, __ldg(p.scale + n), __ldg(p.shift + n));
      return t > 0.0f ? t : t * p.slope;
    };
    // operand outputs: groups of 8 channels past those the accumulators hold are the destinations' zero padding
    const bool to_operands = F16 && p.odst[0] != nullptr;
    auto store_zero_groups = [&](int k0, int oz, int oyy, int ox) {
      const int kmax = max(p.ocg[0], p.odst[1] ? p.ocg[1] : 0);
      const float z[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
      for (int k = k0; k < kmax; ++k) store_operand(p, k, b, oz, oyy, ox, Do, Ho, Wo, z);
    };
    if constexpr (C1) {
      const float bias = __ldg(p.shift);
#pragma unroll
      for (int mt = 0; mt < MT; ++mt) {
        float v[8];
        ld_row<8>(arow + mt * NPAD, v);
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          v[i] += bias;
          if (p.act_sigmoid) v[i] = 1.0f / (1.0f + __expf(-v[i]));
        }
        const int oxb = 2 * (x0 + 8 * mt + xx);
#pragma unroll
        for (int qzy = 0; qzy < 4; ++qzy) {
          float *dst = p.out + (((size_t)b * Do + 2 * zj + (qzy >> 1)) * Ho + 2 * (y0 + yy) + (qzy & 1)) * (size_t)Wo + oxb;
          *reinterpret_cast<float2 *>(dst) = make_float2(v[qzy * 2], v[qzy * 2 + 1]);
        }
      }
    } else if constexpr (PAIR) {
      constexpr int CP = NPAD / 4;            // output channels per (y,x) class
      static_assert(CP % 4 == 0, "merged classes must be whole channel groups");
      const int oz = 2 * zj + pz;
#pragma unroll
      for (int mt = 0; mt < MT; ++mt) {
        const int q = q0 + Cfg::M * mt + m, y = q / Cfg::PX, x = q - y * Cfg::PX;
        if (y > p.H || x > p.W) continue;     // past the plane, or the pitch's spare column x = W + 1
#pragma unroll
        for (int qy = 0; qy < 2; ++qy) {
          const int oyy = 2 * y - qy;         // class y parity 1 is output 2y - 1, parity 0 is 2y
          if (oyy < 0 || oyy >= Ho) continue;
#pragma unroll
          for (int qx = 0; qx < 2; ++qx) {
            const int ox = 2 * x - qx;
            if (ox < 0 || ox >= Wo) continue;
            const float *cls = arow + mt * NPAD + (qy * 2 + qx) * CP;   // the CP channels of class (qy, qx)
            if (to_operands) {
#pragma unroll
              for (int k = 0; k < (CP + 7) / 8; ++k) {
                float v[8];
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                  const int c0 = 8 * k + 4 * h;
                  float v4[4] = {0.f, 0.f, 0.f, 0.f};
                  if (c0 < CP) ld_row<4>(cls + c0, v4);
#pragma unroll
                  for (int e = 0; e < 4; ++e) v[4 * h + e] = c0 < CP && c0 + e < 4 * p.cgo ? act(v4[e], c0 + e) : 0.0f;
                }
                store_operand(p, k, b, oz, oyy, ox, Do, Ho, Wo, v);
              }
              store_zero_groups((CP + 7) / 8, oz, oyy, ox);
              continue;
            }
#pragma unroll
            for (int cgo = 0; cgo < CP / 4; ++cgo) {
              if (cgo >= p.cgo) continue;  // uniform across the CTA
              float v4[4];
              ld_row<4>(cls + cgo * 4, v4);
              float4 o;
              float *po = &o.x;
#pragma unroll
              for (int e = 0; e < 4; ++e) po[e] = act(v4[e], cgo * 4 + e);
              *reinterpret_cast<float4 *>(p.out + (((((size_t)b * Do + oz) * p.cgo + cgo) * Ho + oyy) * (size_t)Wo + ox) * 4) = o;
            }
          }
        }
      }
    } else if constexpr (MERGE || MERGE8) {
      constexpr int NZ = MERGE8 ? 2 : 1;      // z classes held by this CTA's accumulators
      constexpr int CP = NPAD / (4 * NZ);     // output channels per class
      static_assert(CP % 4 == 0, "merged classes must be whole channel groups");
#pragma unroll
      for (int mt = 0; mt < MT; ++mt) {
        const int oxb = 2 * (x0 + 8 * mt + xx);
#pragma unroll
        for (int qzy = 0; qzy < 2 * NZ; ++qzy) {
          const int qz = MERGE8 ? qzy >> 1 : 0, qy = qzy & 1;
          const int oyy = 2 * (y0 + yy) + qy;
          const int oz = MERGE8 ? 2 * zj + qz : 2 * zj + pz;
          if (to_operands) {
#pragma unroll
            for (int qx = 0; qx < 2; ++qx) {
              const float *cls = arow + mt * NPAD + (qzy * 2 + qx) * CP;   // the CP channels of class (qz, qy, qx)
#pragma unroll
              for (int k = 0; k < (CP + 7) / 8; ++k) {
                float v[8];
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                  const int c0 = 8 * k + 4 * h;
                  float v4[4] = {0.f, 0.f, 0.f, 0.f};
                  if (c0 < CP) ld_row<4>(cls + c0, v4);
#pragma unroll
                  for (int e = 0; e < 4; ++e) v[4 * h + e] = c0 < CP && c0 + e < 4 * p.cgo ? act(v4[e], c0 + e) : 0.0f;
                }
                store_operand(p, k, b, oz, oyy, oxb + qx, Do, Ho, Wo, v);
              }
              store_zero_groups((CP + 7) / 8, oz, oyy, oxb + qx);
            }
            continue;
          }
#pragma unroll
          for (int cgo = 0; cgo < CP / 4; ++cgo) {
            if (cgo >= p.cgo) continue;  // uniform across the CTA
            float v[8], v4[4];
            ld_row<4>(arow + mt * NPAD + (qzy * 2) * CP + cgo * 4, v4);
#pragma unroll
            for (int i = 0; i < 4; ++i) v[i] = v4[i];
            ld_row<4>(arow + mt * NPAD + (qzy * 2 + 1) * CP + cgo * 4, v4);
#pragma unroll
            for (int i = 0; i < 4; ++i) v[4 + i] = v4[i];
            float4 o[2];
#pragma unroll
            for (int qx = 0; qx < 2; ++qx) {
              float *po = &o[qx].x;
#pragma unroll
              for (int e = 0; e < 4; ++e) {
                const int n = cgo * 4 + e;
                const float t = fmaf(v[qx * 4 + e], __ldg(p.scale + n), __ldg(p.shift + n));
                po[e] = t > 0.0f ? t : t * p.slope;
              }
            }
            float *dst = p.out + (((((size_t)b * Do + oz) * p.cgo + cgo) * Ho + oyy) * (size_t)Wo + oxb) * 4;
            *reinterpret_cast<float4 *>(dst) = o[0];
            *reinterpret_cast<float4 *>(dst + 4) = o[1];
          }
        }
      }
    } else {
#pragma unroll
    for (int mt = 0; mt < MT; ++mt) {
      const int ox = PAR ? 2 * (x0 + 8 * mt + xx) + px : x0 + 8 * mt + xx;
      if (to_operands) {
#pragma unroll
        for (int nb = 0; nb < NPAD / 32; ++nb) {
          float v[32];
          ld_row<32>(arow + mt * NPAD + nb * 32, v);
#pragma unroll
          for (int k8 = 0; k8 < 4; ++k8) {
            float g[8];
#pragma unroll
            for (int e = 0; e < 8; ++e) {
              const int n = nb * 32 + k8 * 8 + e;
              g[e] = n < 4 * p.cgo ? act(v[k8 * 8 + e], n) : 0.0f;
            }
            store_operand(p, nb * 4 + k8, b, oz_plain, oy, ox, Do, Ho, Wo, g);
          }
        }
        store_zero_groups(NPAD / 8, oz_plain, oy, ox);
        continue;
      }
#pragma unroll
      for (int nb = 0; nb < NPAD / 32; ++nb) {
        float v[32];
        ld_row<32>(arow + mt * NPAD + nb * 32, v);
#pragma unroll
        for (int g4 = 0; g4 < 8; ++g4) {
          const int cgo = nb * 8 + g4;
          if (cgo < p.cgo) {
            float4 o;
            float *po = &o.x;
#pragma unroll
            for (int e = 0; e < 4; ++e) {
              const int n = cgo * 4 + e;
              float t = fmaf(v[g4 * 4 + e], __ldg(p.scale + n), __ldg(p.shift + n));
              po[e] = t > 0.0f ? t : t * p.slope;
            }
            float *dst = p.out + (((((size_t)b * Do + oz_plain) * p.cgo + cgo) * Ho + oy) * (size_t)Wo + ox) * 4;
            *reinterpret_cast<float4 *>(dst) = o;
          }
        }
      }
    }
    }
  }
}


// ---- tensor maps of the activation operands (host) ------------------------------------------------------------------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *, const cuuint64_t *,
                                  const cuuint32_t *, const cuuint32_t *, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static EncodeTiledFn tmap_encoder() {
  static EncodeTiledFn fn = nullptr;
  static bool tried = false;
  if (!tried) {
    tried = true;
    void *p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess && q == cudaDriverEntryPointSuccess)
      fn = (EncodeTiledFn)p;
    cudaGetLastError();
  }
  return fn;
}
// blocked activations [planes][ncg][H][W][16 B] as a 5-D map of 4-byte elements (4, W, H, ncg, planes); box = one channel
// group's halo (4, PX, PY, 1, 1); elements outside [0,W) x [0,H) are delivered as zeros
static bool make_halo_tmap(CUtensorMap *m, const void *base, long long planes, int ncg, int H, int W, int PX, int PY) {
  EncodeTiledFn enc = tmap_encoder();
  if (!enc || !base || ncg <= 0) return false;
  const cuuint64_t gdim[5] = {4, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)ncg, (cuuint64_t)planes};
  const cuuint64_t gstr[4] = {16, (cuuint64_t)W * 16, (cuuint64_t)H * W * 16, (cuuint64_t)ncg * H * W * 16};
  const cuuint32_t box[5] = {4, (cuuint32_t)PX, (cuuint32_t)PY, 1, 1};
  const cuuint32_t estr[5] = {1, 1, 1, 1, 1};
  return enc(m, CU_TENSOR_MAP_DATA_TYPE_UINT32, 5, const_cast<void *>(base), gdim, gstr, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
             CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

template <int TZ, int T, int NPAD, int MT, int MODE, int OP, int PW = 0, int CW = 2>
static int launch_convt_variant(const ConvTParams &p, cudaStream_t st) {
  using Cfg = ConvTCfg<T, NPAD, MT, OP == 2, PW, CW>;
  auto kern = convt3d_s2_kernel<TZ, T, NPAD, MT, MODE, OP, PW, CW>;
  static bool configured[64] = {};
  int dev = 0;
  cudaGetDevice(&dev);
  if (!configured[dev & 63]) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)Cfg::SMEM);
    if (e != cudaSuccess) {
      set_error("convt3d: cudaFuncSetAttribute(%zu bytes): %s", Cfg::SMEM, cudaGetErrorString(e));
      return (int)e;
    }
    configured[dev & 63] = true;
  }
  ConvTParams q = p;
  if constexpr (PW > 0) {
    if (p.W != PW) return fail_arg(GENRE_B200_EINVAL, "convt3d: the paired kernel for W=%d got W=%d", PW, p.W);
    q.xtiles = ((p.H + 1) * Cfg::PX + Cfg::M * MT - 1) / (Cfg::M * MT);   // runs of MT * M positions per (H+1) x PX plane
  } else {
    q.xtiles = p.W / Cfg::W;
    if (q.xtiles < 1 || q.xtiles * Cfg::W != p.W) return fail_arg(GENRE_B200_EINVAL, "convt3d: W=%d is not a multiple of the %d-wide tile", p.W, Cfg::W);
  }
  if (!tmap_encoder())
    return fail_arg(GENRE_B200_EINVAL, "convt3d: the driver entry point cuTensorMapEncodeTiled could not be resolved (the halo "
                                       "loads are tensor copies)");
  CUtensorMap tm0, tm1;
  memset(&tm0, 0, sizeof(tm0));
  memset(&tm1, 0, sizeof(tm1));
  const long long planes = (long long)p.B * p.D * Cfg::PARTS;
  if (!make_halo_tmap(&tm0, p.src0, planes, p.cg0, p.H, p.W, Cfg::PX, Cfg::PY))
    return fail_arg(GENRE_B200_EINVAL, "convt3d: cuTensorMapEncodeTiled failed for the first operand");
  if (p.cg1 > 0 && !make_halo_tmap(&tm1, p.src1, planes, p.cg1, p.H, p.W, Cfg::PX, Cfg::PY))
    return fail_arg(GENRE_B200_EINVAL, "convt3d: cuTensorMapEncodeTiled failed for the second operand");
  dim3 grid((unsigned)(p.B * p.D * (PW ? 1 : p.H / CT_BY) * q.xtiles), MODE == 0 ? 8 : MODE == 2 || MODE == 5 ? 2 : 1);
  kern<<<grid, 128 + 128 * CW, Cfg::SMEM, st>>>(q, tm0, tm1);
  return check_launch("convt3d_s2 kernel");
}

template <int TZ, int T, int NPAD, int MT, int MODE, int OP, int PW = 0>
static int launch_convt_impl(const ConvTParams &p, cudaStream_t st) {
  // narrower x tiles (more CTAs, each with fewer M-tiles) until the accumulators fit the consumers' registers
  if constexpr (MT > 1 && MT * (OP >= 2 ? 2 : 1) * NPAD > CT_ACC_COLS) {
    return launch_convt_impl<TZ, T, NPAD, MT / 2, MODE, OP, PW>(p, st);
  } else {
    return launch_convt_variant<TZ, T, NPAD, MT, MODE, OP, PW>(p, st);
  }
}

// X2 doubles the accumulator columns (launch_convt_impl narrows the tile to fit them)
template <int TZ, int T, int NPAD, int MT, int MODE>
static int launch_convt_x2(const ConvTParams &p, cudaStream_t st) {
  if constexpr (NPAD % 16 != 0 || 2 * NPAD > 256) {
    return fail_arg(GENRE_B200_EINVAL, "convt3d: the fp16 hi/lo mode needs N = %d to be a multiple of 16, at most 128", NPAD);
  } else {
    return launch_convt_impl<TZ, T, NPAD, MT, MODE, 2>(p, st);
  }
}
// op: the operand type of the entry point's f16 argument, 0 TF32, 1 fp16, 2 fp16 hi/lo, 3 3xTF32 (two-level accumulator)
template <int TZ, int T, int NPAD, int MT, int MODE>
static int launch_convt_op(const ConvTParams &p, int op, cudaStream_t st) {
  if (op == 2) return launch_convt_x2<TZ, T, NPAD, MT, MODE>(p, st);
  if (op == 3) {
    if constexpr (2 * NPAD > CT_ACC_COLS)   // N > 128: no room for the second register set, one-level accumulation
      return launch_convt_impl<TZ, T, NPAD, MT, MODE, 0>(p, st);
    else
      return launch_convt_impl<TZ, T, NPAD, MT, MODE, 3>(p, st);
  }
  return op == 1 ? launch_convt_impl<TZ, T, NPAD, MT, MODE, 1>(p, st) : launch_convt_impl<TZ, T, NPAD, MT, MODE, 0>(p, st);
}
template <int T, int NPAD, int MT, bool PAR>
static int launch_convt(const ConvTParams &p, int op, cudaStream_t st) {
  return launch_convt_op<T, T, NPAD, MT, PAR ? 0 : 1>(p, op, st);
}
template <int TZ, int T, int NPAD, int MT>
static int launch_convt_merged(const ConvTParams &p, int op, cudaStream_t st) {
  return launch_convt_op<TZ, T, NPAD, MT, 2>(p, op, st);
}
// MODE 5, the fp16 operand modes, N = 80: three M-tiles of 128 positions per CTA in fp16 (240 accumulator columns); in the
// hi/lo split (160 columns) one M-tile of 192 positions on three consumer warpgroups
template <int PW>
static int launch_convt_paired(const ConvTParams &p, int op, cudaStream_t st) {
  return op == 2 ? launch_convt_variant<4, 4, 80, 1, 5, 2, PW, 3>(p, st) : launch_convt_impl<4, 4, 80, 3, 5, 1, PW>(p, st);
}
// the operand destinations dst0, layout0, cpad0, dst1, layout1, cpad1 of an entry point
struct OperandOut {
  void *dst[2];
  int layout[2], cpad[2];
};
static int set_operand_outputs(ConvTParams &p, const OperandOut &o, int f16, int64_t Do, int64_t Ho, int64_t Wo, const char *who) {
  GB_REQUIRE(f16 == 1 || f16 == 2, GENRE_B200_EINVAL, "%s: operand outputs need fp16 operands (f16 = 1 or 2), not %d", who, f16);
  for (int d = 0; d < 2; ++d) {
    if (!o.dst[d]) continue;
    GB_REQUIRE(o.layout[d] == OP_PLAIN || o.layout[d] == OP_PARITY, GENRE_B200_EINVAL,
               "%s: operand layout %d unknown (1 = plain blocked, 2 = parity sub-volumes)", who, o.layout[d]);
    GB_REQUIRE(o.cpad[d] % 8 == 0 && o.cpad[d] >= 4 * p.cgo, GENRE_B200_EINVAL,
               "%s: operand cpad %d must be a multiple of 8 and cover the %d output channels", who, o.cpad[d], 4 * p.cgo);
    GB_REQUIRE(o.layout[d] == OP_PLAIN || (Do % 2 == 0 && Ho % 2 == 0 && Wo % 2 == 0), GENRE_B200_EINVAL,
               "%s: parity sub-volumes of an odd output extent", who);
    GB_REQUIRE(aligned16(o.dst[d]), GENRE_B200_EALIGN, "%s: operand destinations must be 16-byte aligned", who);
    p.odst[d] = reinterpret_cast<uint4 *>(o.dst[d]);
    p.olayout[d] = o.layout[d];
    p.ocg[d] = o.cpad[d] / 8;
  }
  p.oparts = f16 == 2 ? 2 : 1;
  return 0;
}
// The checks every entry point of the halo kernel shares, and the ConvTParams they fill (the entry point sets base and
// its own fields).  `who` prefixes the messages.  Exactly one of out and ops.dst[0] is set; the operand destinations are
// those of an output extent `up` (1 or 2) times the input's.  out_align: the alignment the epilogue's stores to out need.
static int halo_params(ConvTParams &p, const char *who, const void *src0, int cg0, const void *src1, int cg1, int64_t B,
                       int64_t D, int64_t H, int64_t W, const void *wpack, int f16, const float *scale, const float *shift,
                       float slope, float *out, int cgo, const OperandOut &ops, int up, int out_align = 16) {
  GB_REQUIRE(src0 && wpack && scale && shift, GENRE_B200_EINVAL, "%s: null pointer", who);
  GB_REQUIRE(out || ops.dst[0], GENRE_B200_EINVAL, "%s: null pointer (out, or the first operand destination)", who);
  GB_REQUIRE(!(out && ops.dst[0]), GENRE_B200_EINVAL, "%s: both out and an operand destination given (one or the other)", who);
  GB_REQUIRE(H % CT_BY == 0 && H > 0 && D > 0 && B > 0, GENRE_B200_EINVAL, "%s: bad extent", who);
  GB_REQUIRE(cg0 > 0 && cg1 >= 0 && (cg0 + cg1) % CT_KCG == 0 && (cg1 == 0 || src1), GENRE_B200_EINVAL,
             "%s: channel groups (%d + %d) must be even in total", who, cg0, cg1);
  GB_REQUIRE(B * D * (H / CT_BY) < (1ll << 31), GENRE_B200_EINVAL, "%s: grid too large", who);
  GB_REQUIRE(aligned16(src0) && aligned16(wpack) && (!src1 || aligned16(src1)) && ((uintptr_t)out & (out_align - 1)) == 0,
             GENRE_B200_EALIGN, "%s: buffers must be 16-byte aligned, out %d-byte aligned", who, out_align);
  p.src0 = (const float *)src0; p.src1 = (const float *)src1; p.cg0 = cg0; p.cg1 = cg1;
  p.B = (int)B; p.D = (int)D; p.H = (int)H; p.W = (int)W;
  p.wpack = (const float *)wpack; p.scale = scale; p.shift = shift; p.slope = slope; p.out = out; p.cgo = cgo;
  p.srcpar_cgs = 0;
  return ops.dst[0] ? set_operand_outputs(p, ops, f16, up * D, up * H, up * W, who) : 0;
}

template <int MT>
static int launch_convt_c1(const ConvTParams &p, int op, cudaStream_t st) {
  if (op == 2)   // not routed (ops_conv.convt_c1_tc): the exact FP32-pipe stencil serves the fp32-accurate modes
    return fail_arg(GENRE_B200_EINVAL, "convt_c1_tc: the fp16 hi/lo operand mode is not supported for the 1-channel layer");
  return op == 1 ? launch_convt_impl<3, 3, 16, MT, 4, 1>(p, st) : launch_convt_impl<3, 3, 16, MT, 4, 0>(p, st);
}
template <int T, int NPAD, int MT>
static int launch_conv_merged8(const ConvTParams &p, int op, cudaStream_t st) {
  return launch_convt_op<T, T, NPAD, MT, 3>(p, op, st);
}

}  // namespace gb

using namespace gb;

// ConvTranspose3d(kernel K in {4, 8}, stride 2, padding K/2 - 1) forward on channel-blocked activations.
//   src0 [B*D][cg0][H][W][4], src1 [B*D][cg1][H][W][4] or NULL: the two halves of the channel concatenation
//   wpack: weights packed by genre_shapehd_b200.ops_conv.pack_convt_weights (layout in the kernel header)
//   scale, shift [npad]: per-channel affine applied to the accumulator (bias and folded eval-mode BatchNorm),
//   slope: LeakyReLU slope (1 = none).   out [B*2D][cgo][2H][2W][4], or the operand destinations (OP_PLAIN / OP_PARITY)
// Supported: W in {16, 32}, H % 16 == 0, cg0 + cg1 even, 4*cgo <= npad, npad in {32, 64}.
extern "C" int genre_b200_convt3d_s2_forward(const void *src0, int cg0, const void *src1, int cg1, int64_t B, int64_t D,
                                             int64_t H, int64_t W, const void *wpack, int ksize, int npad, int f16,
                                             const float *scale, const float *shift, float slope, float *out, int cgo,
                                             void *dst0, int layout0, int cpad0, void *dst1, int layout1, int cpad1,
                                             void *stream) {
  ConvTParams p;
  const int rc = halo_params(p, "convt3d", src0, cg0, src1, cg1, B, D, H, W, wpack, f16, scale, shift, slope, out, cgo,
                             {{dst0, dst1}, {layout0, layout1}, {cpad0, cpad1}}, 2);
  if (rc) return rc;
  GB_REQUIRE(ksize == 4 || ksize == 8, GENRE_B200_EINVAL, "convt3d: kernel size %d unsupported (4 or 8)", ksize);
  GB_REQUIRE(npad == 32 || npad == 64, GENRE_B200_EINVAL, "convt3d: npad %d unsupported (32 or 64)", npad);
  GB_REQUIRE(W == 16 || W == 32, GENRE_B200_EINVAL, "convt3d: input width %lld unsupported (16 or 32)", (long long)W);
  GB_REQUIRE(cgo > 0 && 4 * cgo <= npad, GENRE_B200_EINVAL, "convt3d: %d output channels exceed npad %d", 4 * cgo, npad);
  const int pad = ksize / 2 - 1;
  for (int par = 0; par < 2; ++par) {
    const int k0 = (par + pad) % 2;
    p.base[par] = (par + pad - k0) / 2;
  }
  cudaStream_t st = as_stream(stream);
  const int T = ksize / 2;
#define GB_CT(TT, NN, MM) return launch_convt<TT, NN, MM, true>(p, f16, st)
  if (T == 4 && npad == 32 && W == 32) GB_CT(4, 32, 4);
  if (T == 4 && npad == 32 && W == 16) GB_CT(4, 32, 2);
  if (T == 2 && npad == 32 && W == 32) GB_CT(2, 32, 4);
  if (T == 2 && npad == 32 && W == 16) GB_CT(2, 32, 2);
  if (T == 2 && npad == 64 && W == 32) GB_CT(2, 64, 4);
  if (T == 2 && npad == 64 && W == 16) GB_CT(2, 64, 2);
  if (T == 4 && npad == 64 && W == 32) GB_CT(4, 64, 4);
  if (T == 4 && npad == 64 && W == 16) GB_CT(4, 64, 2);
#undef GB_CT
  return fail_arg(GENRE_B200_EINVAL, "convt3d: no kernel instance for k=%d npad=%d W=%lld", ksize, npad, (long long)W);
}

// ConvTranspose3d(kernel 8, stride 2, padding 3) with the four (y,x) output parity classes merged along N (kernel MODE 2):
// the layer that dominates Unet_3D, dec5 = ConvT(80 -> 20) on 32^3 (networks/networks.py:166).  Same operands as
// genre_b200_convt3d_s2_forward except
//   wpack, npad = 4 * cpad columns ordered n = (py*2+px)*cpad + co;  scale, shift [cpad]:
//     paired = 1 (fp16 operands f16 = 1, 2 and W in {16, 32} only): paired classes (kernel MODE 5)
//         [2 z-parity][4 z-tap][Cin chunk][4*4 taps][2][npad/8][8][8]  (ops_conv.pack_convt_paired_weights)
//     paired = 0: the 5 x 5 union of the classes' taps (kernel MODE 2)
//         [2 z-parity][4 z-tap][Cin chunk][5*5 union taps][2][npad/8][8][g]  (ops_conv.pack_convt_merged_weights)
// Supported: ksize 8, npad = 80 (Cout <= 20), W = 16 or a multiple of 32, H % 16 == 0.
extern "C" int genre_b200_convt3d_s2_merged_forward(const void *src0, int cg0, const void *src1, int cg1, int64_t B,
                                                    int64_t D, int64_t H, int64_t W, const void *wpack, int ksize,
                                                    int npad, int f16, int paired, const float *scale, const float *shift,
                                                    float slope, float *out, int cgo, void *dst0, int layout0, int cpad0,
                                                    void *dst1, int layout1, int cpad1, void *stream) {
  ConvTParams p;
  const int rc = halo_params(p, "convt3d_merged", src0, cg0, src1, cg1, B, D, H, W, wpack, f16, scale, shift, slope, out, cgo,
                             {{dst0, dst1}, {layout0, layout1}, {cpad0, cpad1}}, 2);
  if (rc) return rc;
  GB_REQUIRE(ksize == 8, GENRE_B200_EINVAL, "convt3d_merged: kernel size %d unsupported (8)", ksize);
  GB_REQUIRE(npad == 80, GENRE_B200_EINVAL, "convt3d_merged: npad %d unsupported (80 = 4 classes x 20 channels)", npad);
  GB_REQUIRE(W == 16 || (W > 0 && W % 32 == 0), GENRE_B200_EINVAL,
             "convt3d_merged: input width %lld unsupported (16, or a multiple of 32 walked in 32-wide tiles)", (long long)W);
  GB_REQUIRE(cgo > 0 && 16 * cgo <= npad, GENRE_B200_EINVAL, "convt3d_merged: %d output channels exceed npad/4", 4 * cgo);
  GB_REQUIRE(paired == 0 || paired == 1, GENRE_B200_EINVAL,
             "convt3d_merged: paired = %d unknown (1 = paired classes, 0 = the union of their taps)", paired);
  GB_REQUIRE(!paired || ((f16 == 1 || f16 == 2) && (W == 16 || W == 32)), GENRE_B200_EINVAL,
             "convt3d_merged: the paired classes need fp16 operands (f16 = 1 or 2) and W = 16 or 32, not f16 = %d, W = %lld",
             f16, (long long)W);
  const int pad = ksize / 2 - 1;
  for (int par = 0; par < 2; ++par) {
    const int k0 = (par + pad) % 2;
    p.base[par] = (par + pad - k0) / 2;
  }
  cudaStream_t st = as_stream(stream);
  if (paired) return W == 32 ? launch_convt_paired<32>(p, f16, st) : launch_convt_paired<16>(p, f16, st);
  if (W % 32 == 0) return launch_convt_merged<4, 5, 80, 4>(p, f16, st);  // 32-wide x tiles
  return launch_convt_merged<4, 5, 80, 2>(p, f16, st);
}

// Conv3d(kernel 8, stride 2, padding 3), few input channels, Cout <= 20, on a 4x space-to-depth input (kernel MODE 3):
// Unet_3D.enc1 = Conv3d(2 -> 20) on 128^3 (networks/networks.py:151).
//   src [B*D][cg][H][W][16 B]: D,H,W = input extent / 4, channels ((c*4+rz)*4+ry)*4+rx (genre_b200_ncdhw_to_blocked mode 3)
//   wpack [3 z-tap][chunk][9 taps][2][npad/8][8][g], npad = 160 columns n = ((qz*2+qy)*2+qx)*20 + co
//         (ops_conv.pack_conv_k8s2_s4d_weights);  scale, shift [20];  out [B*2D][cgo][2H][2W][4] fp32
// Supported: W % 16 == 0, H % 16 == 0, cg even.  The operand outputs of enc1 are those of enc2 (OP_PARITY: output class q at
// coarse position j IS sub-volume q at j) and dec6.
extern "C" int genre_b200_conv3d_k8s2_s4d_forward(const void *src, int cg, int64_t B, int64_t D, int64_t H, int64_t W,
                                                  const void *wpack, int npad, int f16, const float *scale,
                                                  const float *shift, float slope, float *out, int cgo, void *dst0, int layout0,
                                                  int cpad0, void *dst1, int layout1, int cpad1, void *stream) {
  ConvTParams p;
  const int rc = halo_params(p, "conv3d_k8s2_s4d", src, cg, nullptr, 0, B, D, H, W, wpack, f16, scale, shift, slope, out, cgo,
                             {{dst0, dst1}, {layout0, layout1}, {cpad0, cpad1}}, 2);
  if (rc) return rc;
  GB_REQUIRE(npad == 160 || npad == 80, GENRE_B200_EINVAL,
             "conv3d_k8s2_s4d: npad %d unsupported (160 = 8 classes x 20 channels, or 80 = 4 (y,x) classes per z class)", npad);
  GB_REQUIRE(W > 0 && W % 16 == 0, GENRE_B200_EINVAL, "conv3d_k8s2_s4d: bad extent");
  GB_REQUIRE(cgo > 0 && cgo <= 5, GENRE_B200_EINVAL, "conv3d_k8s2_s4d: too many output channels");
  GB_REQUIRE(B * D * (H / CT_BY) * (W / 16) < (1ll << 31), GENRE_B200_EINVAL, "conv3d_k8s2_s4d: grid too large");
  p.base[0] = p.base[1] = 1;  // input cell = j + 1 - t
  // npad 80: the z class moves to blockIdx.y (MODE 2 with 3 z taps per class; wpack [2 qz][3][chunk][9][2][10][8][g]):
  // twice the MMAs of the 8-class form, but half the accumulator columns and weight bytes per stage.  In the fp16 operand
  // modes (groups of 8 channels: K chunk = (c, rz)) the z class's all-zero (z tap, K chunk) stages are skipped
  if (npad == 80) {
    p.s4d_zskip = f16 == 1 || f16 == 2;
    return launch_convt_merged<3, 3, 80, 2>(p, f16, as_stream(stream));
  }
  return launch_conv_merged8<3, 160, 2>(p, f16, as_stream(stream));
}

// ConvTranspose3d(Cin -> 1, k 4, s 2, p 1) on the tensor cores (kernel MODE 4): the last layer of every decoder
// (Unet_3D.dec6 networks/networks.py:167-168, VoxelDecoder main.17 :57, VoxelGenerator :98).  3 union taps per dimension,
// the 8 output classes as N columns.
//   src0/src1 blocked operands [B*D][cg][H][W][16 B] (two halves of a skip concatenation; src1 may be NULL)
//   wpack [3][chunk][9][2][2][8][g] (ops_conv.pack_convt_c1_tc_weights), bias, act_sigmoid;  out [B][2D][2H][2W] fp32
// Supported: W in {16, 32, 64}, H % 16 == 0, cg0 + cg1 even.
extern "C" int genre_b200_convt_c1_tc_forward(const void *src0, int cg0, const void *src1, int cg1, int64_t B, int64_t D,
                                              int64_t H, int64_t W, const void *wpack, int f16, const float *bias,
                                              int act_sigmoid, float *out, void *stream) {
  ConvTParams p;   // out takes float2 stores: 8-byte aligned
  const int rc = halo_params(p, "convt_c1_tc", src0, cg0, src1, cg1, B, D, H, W, wpack, f16, bias, bias, 1.0f, out, 1,
                             OperandOut{}, 2, 8);
  if (rc) return rc;
  GB_REQUIRE(W == 16 || W == 32 || W == 64, GENRE_B200_EINVAL, "convt_c1_tc: input width %lld unsupported", (long long)W);
  p.act_sigmoid = act_sigmoid;
  p.base[0] = p.base[1] = 1;
  cudaStream_t st = as_stream(stream);
  if (W == 64) return launch_convt_c1<8>(p, f16, st);
  if (W == 32) return launch_convt_c1<4>(p, f16, st);
  return launch_convt_c1<2>(p, f16, st);
}

// Stride-1 convolution with T taps per dimension on channel-blocked activations (same kernel, one output class):
//     out[b, z, y, x, n] = act(scale[n] * sum_{tz,ty,tx,c} in[b, z + base - tz, y + base - ty, x + base - tx, c] * Wt[...] + shift[n])
// A strided Conv3d reaches this form through space-to-depth (genre_shapehd_b200/ops_conv.py): Unet_3D.enc1 =
// Conv3d(2 -> 20, k=8, s=2, p=3) (networks/networks.py:151) is a 5-tap stride-1 convolution over the 16 s2d channels.
//   wpack [T z-tap][C/8 chunk][T*T taps][2][npad/8][8][4];  out [B*D][cgo][H][W][4]
// Supported: T in {3, 5}, W in {16, 32, 64}, H % 16 == 0, npad = 32 (or 64 with T = 3, 96 with T = 5).
extern "C" int genre_b200_conv3d_taps_forward(const void *src0, int cg0, const void *src1, int cg1, int64_t B,
                                              int64_t D, int64_t H, int64_t W, const void *wpack, int taps, int base,
                                              int npad, int f16, const float *scale, const float *shift, float slope,
                                              float *out, int cgo, void *stream) {
  ConvTParams p;
  const int rc = halo_params(p, "conv3d_taps", src0, cg0, src1, cg1, B, D, H, W, wpack, f16, scale, shift, slope, out, cgo,
                             OperandOut{}, 1);
  if (rc) return rc;
  GB_REQUIRE(taps == 3 || taps == 5, GENRE_B200_EINVAL, "conv3d_taps: %d taps unsupported (3 or 5)", taps);
  GB_REQUIRE(npad == 32 || (npad == 64 && taps == 3) || (npad == 96 && taps == 5), GENRE_B200_EINVAL,
             "conv3d_taps: npad %d unsupported (32; 64 with 3 taps; 96 with 5 taps)", npad);
  GB_REQUIRE(W == 16 || W == 32 || W == 64, GENRE_B200_EINVAL, "conv3d_taps: width %lld unsupported", (long long)W);
  GB_REQUIRE(cgo > 0 && 4 * cgo <= npad, GENRE_B200_EINVAL, "conv3d_taps: too many output channels");
  p.base[0] = p.base[1] = base;
  cudaStream_t st = as_stream(stream);
  // 3 taps, N = 64: Conv3d(1 -> 64, k4, s2, p1) over the 2x space-to-depth input (VoxelDiscriminator's first layer)
  if (taps == 3 && npad == 64) {
    if (W % 32 == 0) return launch_convt<3, 64, 4, false>(p, f16, st);
    return launch_convt<3, 64, 2, false>(p, f16, st);
  }
  // 5 taps, N = 96: Conv3d(20 -> 80, k8, s2, p3) over the 2x space-to-depth input = the input gradient of Unet_3D.dec5
  // (ConvTranspose3d 80 -> 20)
  if (taps == 5 && npad == 96) {
    if (W % 32 == 0) return launch_convt<5, 96, 4, false>(p, f16, st);
    return launch_convt<5, 96, 2, false>(p, f16, st);
  }
#define GB_CV(TT, MM) return launch_convt<TT, 32, MM, false>(p, f16, st)
  if (taps == 5 && W == 64) GB_CV(5, 8);
  if (taps == 5 && W == 32) GB_CV(5, 4);
  if (taps == 5 && W == 16) GB_CV(5, 2);
  if (taps == 3 && W == 64) GB_CV(3, 8);
  if (taps == 3 && W == 32) GB_CV(3, 4);
  if (taps == 3 && W == 16) GB_CV(3, 2);
#undef GB_CV
  return fail_arg(GENRE_B200_EINVAL, "conv3d_taps: no kernel instance");
}

// Conv3d(kernel 4, stride 2, padding 1) forward (VoxelDiscriminator networks/networks.py:247-250 conv3d_half, Unet_3D
// enc2..enc5 :152-155) on the same kernel: the input arrives as its 8 parity sub-volumes in ONE channel-blocked tensor
//   src [B*D'][8*cgs][H'][W'][16 B]   (D' = D/2 ...; channel group index = s*cgs + c, s = (pz*2+py)*2+px)
// and sub-volume s is a K range with 2 taps per dimension: in[2(o+delta)+p] with delta = (1-p) - t, k = 3 - 2t - p.
//   wpack [2 z-tap][kblocks*8*cgs/2 chunk][4 taps][2][npad/8][8][g];  out [B*D'][cgo][H'][W'][4] fp32
//   kblocks (1, or 3 for the hi|lo|hi operand of the 3xTF32 mode): how many such 8-sub-volume blocks the K range holds
// Supported: W' in {16, 32}, H' % 16 == 0, cgs even, npad in {32, 64, 96, 128}.
extern "C" int genre_b200_conv3d_k4s2_forward(const void *src, int cgs, int kblocks, int64_t B, int64_t D, int64_t H, int64_t W,
                                              const void *wpack, int npad, int f16, const float *scale, const float *shift,
                                              float slope, float *out, int cgo, void *dst0, int layout0, int cpad0, void *dst1,
                                              int layout1, int cpad1, void *stream) {
  ConvTParams p;
  const int rc = halo_params(p, "conv3d_k4s2", src, 8 * cgs * (kblocks > 0 ? kblocks : 1), nullptr, 0, B, D, H, W, wpack, f16,
                             scale, shift, slope, out, cgo, {{dst0, dst1}, {layout0, layout1}, {cpad0, cpad1}}, 1);
  if (rc) return rc;
  GB_REQUIRE(npad == 32 || npad == 64 || npad == 96 || npad == 128, GENRE_B200_EINVAL, "conv3d_k4s2: npad %d", npad);
  GB_REQUIRE(W == 16 || W == 32, GENRE_B200_EINVAL, "conv3d_k4s2: output width %lld unsupported (16 or 32)", (long long)W);
  GB_REQUIRE(cgs > 0 && cgs % CT_KCG == 0, GENRE_B200_EINVAL, "conv3d_k4s2: channel groups per sub-volume must be even");
  GB_REQUIRE(cgo > 0 && 4 * cgo <= npad, GENRE_B200_EINVAL, "conv3d_k4s2: too many output channels");
  p.srcpar_cgs = cgs;
  p.base[0] = p.base[1] = 0;
  cudaStream_t st = as_stream(stream);
#define GB_CS(NN, MM) return launch_convt<2, NN, MM, false>(p, f16, st)
  if (W == 32) {
    if (npad == 32) GB_CS(32, 4);
    if (npad == 64) GB_CS(64, 4);
    if (npad == 96) GB_CS(96, 4);
    if (npad == 128) GB_CS(128, 4);
  } else {
    if (npad == 32) GB_CS(32, 2);
    if (npad == 64) GB_CS(64, 2);
    if (npad == 96) GB_CS(96, 2);
    if (npad == 128) GB_CS(128, 2);
  }
#undef GB_CS
  return fail_arg(GENRE_B200_EINVAL, "conv3d_k4s2: no kernel instance");
}
