"""The shapes the convolution routes of ops_conv accept, as plain data: one case per predicate edge, and the kernel instance
each (case, operand mode) must launch.

A case gives the module (networks.Conv3d / ConvTranspose3d / Conv3d_block / Deconv3d_skip or a FusedSequential slice
with eval BatchNorm and an activation where the route fuses them), the source shapes, the library entry point the route
calls, the kernel family and kappa per operand mode (tests/infer_ref.py's terms).  instance_of(case, mode) restates the
launch: the arguments ops_conv passes (npad, tile width, op) and the C++ dispatch of csrc/convt3d.cu (launch_convt_impl's
MT narrowing, op 3 falling back to one-level accumulation above N = 128, MODE 5's (PW, CW)), csrc/convflat.cu (one or two
M-tiles per CTA, narrowed to the register budget) and csrc/convt_c1_col2im.cu.  abi_instances() enumerates every
instance those dispatchers can reach through the C ABI; ABI_ONLY lists the ones neither this table nor the gradient
table (tests/conv_grad_domain.py) reaches, each with why and which test runs it.  tests/test_conv_domain_cpu.py checks the
ledger against the built library, and tests/test_gpu_conv_domain_fp64.py runs every case against fp64.

MMA steps per output (kappa): fp16 operands take K steps of 16 channels (one m64nNk16 wgmma), the fp32 operand modes
(tf32, the 3xTF32 split) steps of 8 channels (CT_KCG = 2 groups of 4, m64nNk8).  A halo kernel's output sums
z taps x ceil(K / step) x (y, x) taps of its configuration: T x T per parity class (MODE 0 / 1), the 5 x 5 union
(MODE 2), the 4 x 4 paired taps (MODE 5), 3 x 3 over space-to-depth (MODE 3 and the taps forms).
"""
import infer_ref as R
from genre_shapehd_b200.ops_conv import PARITY, PLAIN

MODES_HALO = ("f16x2", "f16", "fp32x3", "tf32")
MODES_FP16 = ("f16x2", "f16")
MODES_C1TC = ("f16", "tf32")
MODES_SKINNY = ("f16x2",)            # FP32 FMA chains: the operand mode does not reach them
MODES_STENCIL = ("f16x2", "f16")     # the FP32 stencil, where neither col2im nor convt_c1_tc takes the width
OP = {"tf32": 0, "f16": 1, "f16x2": 2, "fp32x3": 3}
ACC_COLS = 256                       # CT_ACC_COLS / the flat kernel's register budget: MT * accumulator columns


def kstep(mode):
    """channels per MMA K step: fp16 groups of 8 x 2, fp32 groups of 4 x 2"""
    return 16 if mode in ("f16", "f16x2") else 8


def _halo_steps(mode, tz, kchan, yx):
    return tz * -(-kchan // kstep(mode)) * yx


class Case:
    """kind: conv | convt (bare module), seq (FusedSequential slice: conv [, bn], act), block (Conv3d_block),
    skip (Deconv3d_skip).  geometry: dict(cin, cout, k, s, p, bias, bn, act) of the module; shapes: source shapes;
    route: the halo / flat configuration instance_of needs"""

    def __init__(self, name, kind, geometry, shapes, entry, family, modes, route, kappa, straddle=False):
        self.name, self.kind, self.geometry, self.shapes = name, kind, geometry, [tuple(s) for s in shapes]
        self.entry, self.family, self.modes, self.route, self._kappa = entry, family, modes, route, kappa
        self.straddle = straddle

    def kappa(self, mode):
        return self._kappa(mode)

    @property
    def batch(self):
        return self.shapes[0][0]

    @property
    def cin(self):
        return sum(s[1] for s in self.shapes)

    def __repr__(self):
        return "Case(%s)" % self.name


def _g(cin, cout, k, s=2, p=1, bias=True, bn=False, act=None):
    return dict(cin=cin, cout=cout, k=k, s=s, p=p, bias=bias, bn=bn, act=act)


# ---- kappa per configuration ------------------------------------------------------------------------------------------
def _kappa_convt(cin, t, yx=None, x3_yx=None):
    """ConvTranspose3d k = 2t (MODE 0: t z taps x t x t), or the merged / paired classes (yx (y,x) taps per z tap)"""
    yx = t * t if yx is None else yx

    def k(mode):
        if mode == "fp32x3":
            return R.kappa_x3(R.stages_x3(t, cin, t if x3_yx is None else x3_yx))
        return R.kappa_tc(mode, _halo_steps(mode, t, cin, yx))
    return k


def _kappa_merged(cin):
    """Cout <= 20 k8: paired MODE 5 (4 x 4) in the fp16 modes, the 5 x 5 union (MODE 2) in the fp32 ones"""
    def k(mode):
        if mode == "fp32x3":
            return R.kappa_x3(R.stages_x3(4, cin, 5))
        return R.kappa_tc(mode, _halo_steps(mode, 4, cin, 16 if mode in MODES_FP16 else 25))
    return k


def _cpad_k4s2(cin, mode):
    g = 8 if mode in MODES_FP16 else 4
    return -(-cin // (2 * g)) * 2 * g


def _kappa_k4s2(cin):
    def k(mode):
        kc = 8 * _cpad_k4s2(cin, mode)
        if mode == "fp32x3":
            return R.kappa_x3(R.stages_x3(2, kc, 2))
        return R.kappa_tc(mode, _halo_steps(mode, 2, kc, 4))
    return k


def _kappa_taps(taps, kchan):
    """stride-1 taps over a space-to-depth input of kchan channels (zero-padded to whole K steps)"""
    def k(mode):
        if mode == "fp32x3":
            return R.kappa_x3(R.stages_x3(taps, -(-kchan // 8) * 8, taps))
        return R.kappa_tc(mode, _halo_steps(mode, taps, kchan, taps * taps))
    return k


def _kappa_s4d(cin):
    return _kappa_taps(3, 64 * cin)


def _kappa_flat(cin_total, transposed):
    return lambda mode: R.kappa_tc(mode, R.steps_flat(cin_total, transposed))


def _kappa_c1_tc(cin_padded):
    return lambda mode: R.kappa_tc(mode, _halo_steps(mode, 3, cin_padded, 9))


def _kappa_col2im(cin_padded):
    return lambda mode: R.kappa_col2im(mode, -(-cin_padded // 16))


def _kappa_skinny(transposed, k):
    return lambda mode: R.kappa_skinny(transposed, k)


# ---- the table ----------------------------------------------------------------------------------------------------------
E_CONVT = "genre_b200_convt3d_s2_forward"
E_MERGED = "genre_b200_convt3d_s2_merged_forward"
E_K4S2 = "genre_b200_conv3d_k4s2_forward"
E_S4D = "genre_b200_conv3d_k8s2_s4d_forward"
E_TAPS = "genre_b200_conv3d_taps_forward"
E_C1TC = "genre_b200_convt_c1_tc_forward"
E_COL2IM = "genre_b200_convt_c1_col2im_forward"
E_FLAT = "genre_b200_convflat_forward"
E_SKINNY = "genre_b200_skinny_gemm"
E_C1 = "genre_b200_convt_c1_forward"

CASES = [
    # ConvTranspose3d k4 s2 on the halo kernel (MODE 0): W in {16, 32}, H % 16, Cout <= 64 in npad 32 / 64
    Case("convt_k4 B1 D1 16x16 c16->4 npad32", "convt", _g(16, 4, 4), [(1, 16, 1, 16, 16)], E_CONVT, "halo", MODES_HALO,
         dict(T=2, npad=32, W=16), _kappa_convt(16, 2)),
    Case("convt_k4 B3 D3 32x32 c32->33 npad64 BN ReLU", "seq", _g(32, 33, 4, bn=True, act="relu"), [(3, 32, 3, 32, 32)],
         E_CONVT, "halo", MODES_HALO, dict(T=2, npad=64, W=32), _kappa_convt(32, 2)),
    Case("convt_k4 B3 D2 48x16 skip 8+24->32 npad32 BN LReLU", "skip", _g(32, 32, 4, bn=True, act="lrelu"),
         [(3, 8, 2, 48, 16), (3, 24, 2, 48, 16)], E_CONVT, "halo", MODES_HALO, dict(T=2, npad=32, W=16),
         _kappa_convt(32, 2), straddle=True),
    Case("convt_k4 B1 D1 16x16 c16->64 npad64 BN LReLU", "seq", _g(16, 64, 4, bn=True, act="lrelu"), [(1, 16, 1, 16, 16)],
         E_CONVT, "halo", MODES_HALO, dict(T=2, npad=64, W=16), _kappa_convt(16, 2)),
    Case("convt_k4 B1 D2 16x32 c16->32 npad32", "convt", _g(16, 32, 4), [(1, 16, 2, 16, 32)], E_CONVT, "halo", MODES_HALO,
         dict(T=2, npad=32, W=32), _kappa_convt(16, 2)),
    # k8 with Cout > 20: the non-merged T = 4 kernels
    Case("convt_k8 B1 D1 16x16 c16->21 npad32", "convt", _g(16, 21, 8, p=3), [(1, 16, 1, 16, 16)], E_CONVT, "halo",
         MODES_HALO, dict(T=4, npad=32, W=16), _kappa_convt(16, 4)),
    Case("convt_k8 B3 D1 16x32 c16->40 npad64", "convt", _g(16, 40, 8, p=3), [(3, 16, 1, 16, 32)], E_CONVT, "halo",
         MODES_HALO, dict(T=4, npad=64, W=32), _kappa_convt(16, 4)),
    Case("convt_k8 B1 D1 16x32 c16->32 npad32", "convt", _g(16, 32, 8, p=3), [(1, 16, 1, 16, 32)], E_CONVT, "halo",
         MODES_HALO, dict(T=4, npad=32, W=32), _kappa_convt(16, 4)),
    Case("convt_k8 B1 D1 16x16 c16->64 npad64", "convt", _g(16, 64, 8, p=3), [(1, 16, 1, 16, 16)], E_CONVT, "halo",
         MODES_HALO, dict(T=4, npad=64, W=16), _kappa_convt(16, 4)),
    # k8 with Cout <= 20: the four (y, x) classes merged in N = 80 (paired MODE 5 in the fp16 modes, MODE 2 otherwise)
    Case("convt_k8 merged B1 D1 16x32 skip 8+8->20", "skip", _g(16, 20, 8, p=3, bn=True, act="lrelu"),
         [(1, 8, 1, 16, 32), (1, 8, 1, 16, 32)], E_MERGED, "halo", MODES_HALO, dict(W=32), _kappa_merged(16),
         straddle=True),
    Case("convt_k8 merged B3 D3 32x16 c16->5", "convt", _g(16, 5, 8, p=3), [(3, 16, 3, 32, 16)], E_MERGED, "halo",
         MODES_HALO, dict(W=16), _kappa_merged(16)),
    # Conv3d k4 s2 over parity sub-volumes: Cin >= 8 (zero-padded to whole K chunks per sub-volume), Cout <= 128, W' in {16, 32}
    Case("k4s2 B1 D2 32x32 c8->32 npad32", "block", _g(8, 32, 4, bn=True, act="lrelu"), [(1, 8, 2, 32, 32)], E_K4S2,
         "halo", MODES_HALO, dict(npad=32, W=16), _kappa_k4s2(8)),
    Case("k4s2 B1 D2 32x64 c16->12 npad32", "conv", _g(16, 12, 4), [(1, 16, 2, 32, 64)], E_K4S2, "halo", MODES_HALO,
         dict(npad=32, W=32), _kappa_k4s2(16)),
    Case("k4s2 B1 D2 32x32 c8->64 npad64", "conv", _g(8, 64, 4), [(1, 8, 2, 32, 32)], E_K4S2, "halo", MODES_HALO,
         dict(npad=64, W=16), _kappa_k4s2(8)),
    Case("k4s2 B3 D6 32x64 c20->33 npad64", "block", _g(20, 33, 4, bn=True, act="lrelu"), [(3, 20, 6, 32, 64)], E_K4S2,
         "halo", MODES_HALO, dict(npad=64, W=32), _kappa_k4s2(20)),
    Case("k4s2 B1 D2 32x64 c24->96 npad96", "conv", _g(24, 96, 4), [(1, 24, 2, 32, 64)], E_K4S2, "halo", MODES_HALO,
         dict(npad=96, W=32), _kappa_k4s2(24)),
    Case("k4s2 B3 D2 32x32 c16->97 npad128", "block", _g(16, 97, 4, bn=True, act="lrelu"), [(3, 16, 2, 32, 32)], E_K4S2,
         "halo", MODES_HALO, dict(npad=128, W=16), _kappa_k4s2(16)),
    # Conv3d k8 s2, Cin in {2, 4, 6, 8}: the 4x space-to-depth form (Cout <= 20, extents % 64 / 4) ...
    Case("k8s2 s4d B1 D4 64x64 c2->20", "block", _g(2, 20, 8, p=3, bn=True, act="lrelu"), [(1, 2, 4, 64, 64)], E_S4D,
         "halo", MODES_HALO, dict(W=16), _kappa_s4d(2)),
    Case("k8s2 s4d B3 D4 64x128 c8->5", "conv", _g(8, 5, 8, p=3), [(3, 8, 4, 64, 128)], E_S4D, "halo", MODES_HALO,
         dict(W=32), _kappa_s4d(8)),
    # ... else the 5-tap form over the 2x space-to-depth input (Cout <= 32)
    Case("k8s2 taps5 B1 D2 32x32 c2->8", "conv", _g(2, 8, 8, p=3), [(1, 2, 2, 32, 32)], E_TAPS, "halo", MODES_HALO,
         dict(T=5, npad=32, W=16), _kappa_taps(5, 16)),
    Case("k8s2 taps5 B3 D2 32x64 c6->32 BN LReLU", "block", _g(6, 32, 8, p=3, bn=True, act="lrelu"), [(3, 6, 2, 32, 64)],
         E_TAPS, "halo", MODES_HALO, dict(T=5, npad=32, W=32), _kappa_taps(5, 48)),
    Case("k8s2 taps5 B1 D2 32x128 c4->24", "conv", _g(4, 24, 8, p=3), [(1, 4, 2, 32, 128)], E_TAPS, "halo", MODES_HALO,
         dict(T=5, npad=32, W=64), _kappa_taps(5, 32)),
    # Conv3d k4 s2 on 1 or 2 channels, 32 < Cout <= 64: 3 taps over the 2x space-to-depth input
    Case("k4s2 s2d B1 D2 32x32 c1->33", "conv", _g(1, 33, 4), [(1, 1, 2, 32, 32)], E_TAPS, "halo", MODES_HALO,
         dict(T=3, npad=64, W=16), _kappa_taps(3, 8)),
    Case("k4s2 s2d B3 D4 32x128 c2->64 LReLU", "seq", _g(2, 64, 4, act="lrelu"), [(3, 2, 4, 32, 128)], E_TAPS, "halo",
         MODES_HALO, dict(T=3, npad=64, W=64), _kappa_taps(3, 16)),
    # the 1-channel ConvTranspose3d on the tensor cores (MODE 4): W in {16, 32, 64}, the sigmoid epilogue
    Case("c1_tc B1 D1 16x16 c16->1", "convt", _g(16, 1, 4), [(1, 16, 1, 16, 16)], E_C1TC, "halo", MODES_C1TC,
         dict(W=16), _kappa_c1_tc(16)),
    Case("c1_tc B3 D3 16x32 skip 8+24->1", "skip", _g(32, 1, 4), [(3, 8, 3, 16, 32), (3, 24, 3, 16, 32)], E_C1TC, "halo",
         MODES_C1TC, dict(W=32), _kappa_c1_tc(32), straddle=True),
    Case("c1_tc B1 D2 16x64 c16->1 sigmoid", "seq", _g(16, 1, 4, act="sigmoid"), [(1, 16, 2, 16, 64)], E_C1TC, "halo",
         MODES_C1TC, dict(W=64), _kappa_c1_tc(16)),
    # the 1-channel ConvTranspose3d on 64-wide volumes: tap GEMM + col2im
    Case("col2im B1 D1 8x64 c16->1", "convt", _g(16, 1, 4), [(1, 16, 1, 8, 64)], E_COL2IM, "col2im", MODES_FP16, {},
         _kappa_col2im(16)),
    Case("col2im B3 D3 16x64 skip 8+40->1", "skip", _g(48, 1, 4), [(3, 8, 3, 16, 64), (3, 40, 3, 16, 64)], E_COL2IM,
         "col2im", MODES_FP16, {}, _kappa_col2im(48), straddle=True),
    # the accepted edges of col2im's K-step limit (ops_conv.C2I_MAX_KSTEPS): 40 steps in the hi/lo split, 85 in f16
    Case("col2im B1 D1 8x64 c640->1 (40 K steps)", "convt", _g(640, 1, 4), [(1, 640, 1, 8, 64)], E_COL2IM, "col2im", ("f16x2",),
         {}, _kappa_col2im(640)),
    Case("col2im B1 D1 8x64 c1360->1 (85 K steps)", "convt", _g(1360, 1, 4), [(1, 1360, 1, 8, 64)], E_COL2IM, "col2im", ("f16",),
         {}, _kappa_col2im(1360)),
    # the FP32-pipe 1-channel stencil (csrc/convt_c1.cu): Cin % 4, Cin <= 48, W % 4; odd B x D (a partial last z block of
    # two planes), partial x blocks (64 input columns per block) and y blocks (8 rows)
    Case("c1 stencil B3 D1 5x20 c12->1", "convt", _g(12, 1, 4), [(3, 12, 1, 5, 20)], E_C1, "c1", MODES_STENCIL, {},
         lambda mode: R.kappa_c1_stencil(12)),
    Case("c1 stencil B1 D3 8x68 skip 24+24->1", "skip", _g(48, 1, 4), [(1, 24, 3, 8, 68), (1, 24, 3, 8, 68)], E_C1, "c1",
         MODES_STENCIL, {}, lambda mode: R.kappa_c1_stencil(48), straddle=True),
    Case("c1 stencil B5 D1 16x32 c4->1", "convt", _g(4, 1, 4), [(5, 4, 1, 16, 32)], E_C1, "c1", ("f16x2",), {},
         lambda mode: R.kappa_c1_stencil(4)),
    # the flattened-volume kernel: extents <= 8 (16 for the strided conv), non-cubic, 1 - 3 N tiles of 64 or 80
    Case("flat convt B1 1^3 c16->8", "convt", _g(16, 8, 4), [(1, 16, 1, 1, 1)], E_FLAT, "flat", MODES_FP16, dict(transposed=True),
         _kappa_flat(16, True)),
    Case("flat convt B3 3x5x8 c24->150 (2 x 80) BN ReLU", "seq", _g(24, 150, 4, bn=True, act="relu"), [(3, 24, 3, 5, 8)],
         E_FLAT, "flat", MODES_FP16, dict(transposed=True), _kappa_flat(24, True)),
    Case("flat convt B5 4^3 skip 8+24->161 (3 x 64) BN LReLU", "skip", _g(32, 161, 4, bn=True, act="lrelu"),
         [(5, 8, 4, 4, 4), (5, 24, 4, 4, 4)], E_FLAT, "flat", MODES_FP16, dict(transposed=True), _kappa_flat(32, True), straddle=True),
    Case("flat convt B5 8^3 c16->64 (two M tiles)", "convt", _g(16, 64, 4), [(5, 16, 8, 8, 8)], E_FLAT, "flat",
         MODES_FP16, dict(transposed=True), _kappa_flat(16, True)),
    Case("flat convt B5 8^3 c16->80 (two M tiles)", "convt", _g(16, 80, 4), [(5, 16, 8, 8, 8)], E_FLAT, "flat",
         MODES_FP16, dict(transposed=True), _kappa_flat(16, True)),
    Case("flat conv B1 2^3 c16->8", "conv", _g(16, 8, 4), [(1, 16, 2, 2, 2)], E_FLAT, "flat", MODES_FP16, dict(transposed=False),
         _kappa_flat(16, False)),
    Case("flat conv B3 4x8x16 c32->200 (3 x 80) BN LReLU", "block", _g(32, 200, 4, bn=True, act="lrelu"),
         [(3, 32, 4, 8, 16)], E_FLAT, "flat", MODES_FP16, dict(transposed=False), _kappa_flat(32, False)),
    Case("flat conv B15 16^3 c16->192 (3 x 64, two M tiles)", "conv", _g(16, 192, 4), [(15, 16, 16, 16, 16)], E_FLAT,
         "flat", MODES_FP16, dict(transposed=False), _kappa_flat(16, False)),
    # weight-streaming FP32 products: a Conv3d whose kernel is its input (non-cubic too), a ConvTranspose3d of a 1^3 input
    Case("skinny conv B1 k(2,3,4) c8->6", "conv", _g(8, 6, (2, 3, 4), s=1, p=0), [(1, 8, 2, 3, 4)], E_SKINNY, "skinny",
         MODES_SKINNY, {}, _kappa_skinny(False, 8 * 24)),
    Case("skinny conv B3 k4 c40->12 BN LReLU", "block", _g(40, 12, 4, s=1, p=0, bn=True, act="lrelu"), [(3, 40, 4, 4, 4)],
         E_SKINNY, "skinny", MODES_SKINNY, {}, _kappa_skinny(False, 40 * 64)),
    Case("skinny convt B5 1^3 k(2,3,4) c24->6", "convt", _g(24, 6, (2, 3, 4), s=1, p=0), [(5, 24, 1, 1, 1)], E_SKINNY,
         "skinny", MODES_SKINNY, {}, _kappa_skinny(True, 24)),
    Case("skinny convt B3 1^3 skip 160+160->8 BN LReLU", "skip", _g(320, 8, 4, s=1, p=0, bn=True, act="lrelu"),
         [(3, 160, 1, 1, 1), (3, 160, 1, 1, 1)], E_SKINNY, "skinny", MODES_SKINNY, {}, _kappa_skinny(True, 320)),
]
CASE_IDS = [c.name for c in CASES]


def case(name):
    return next(c for c in CASES if c.name == name)


# ---- route boundaries: the nearest shapes each predicate rejects -------------------------------------------------------
BOUNDARIES = [   # (name, transposed, cin, cout, k, s, p, input shape, modes)
    ("convt_k4 W = 48", True, 16, 8, 4, 2, 1, (1, 16, 1, 16, 48), MODES_FP16),
    ("convt_k4 H = 24", True, 16, 8, 4, 2, 1, (1, 16, 1, 24, 16), MODES_FP16),
    ("convt_k4 Cout 65", True, 16, 65, 4, 2, 1, (1, 16, 1, 16, 16), MODES_FP16),
    ("convt_k8 Cout 65", True, 16, 65, 8, 2, 3, (1, 16, 1, 16, 16), MODES_FP16),
    ("k4s2 Cin 7", False, 7, 32, 4, 2, 1, (1, 7, 2, 32, 32), MODES_FP16),
    ("k4s2 Cout 129", False, 16, 129, 4, 2, 1, (1, 16, 2, 32, 32), MODES_FP16),
    ("k4s2 W' = 64", False, 16, 32, 4, 2, 1, (1, 16, 2, 32, 128), MODES_FP16),
    ("k8s2 Cin 10", False, 10, 8, 8, 2, 3, (1, 10, 2, 32, 32), MODES_FP16),
    ("k8s2 Cout 33", False, 2, 33, 8, 2, 3, (1, 2, 2, 32, 32), MODES_FP16),
    ("k4s2 s2d Cout 65", False, 1, 65, 4, 2, 1, (1, 1, 2, 32, 32), MODES_FP16),
    ("k4s2 s2d Cin 3", False, 3, 64, 4, 2, 1, (1, 3, 2, 32, 32), MODES_FP16),
    ("flat convt extent 9", True, 16, 8, 4, 2, 1, (1, 16, 2, 2, 9), MODES_FP16),
    ("flat conv extent 18", False, 16, 8, 4, 2, 1, (1, 16, 2, 2, 18), MODES_FP16),
    ("flat conv Cin 8", False, 8, 8, 4, 2, 1, (1, 8, 4, 4, 4), MODES_FP16),
    ("flat convt Cout 7", True, 16, 7, 4, 2, 1, (1, 16, 4, 4, 4), MODES_FP16),
    ("col2im Cin 656 (41 K steps)", True, 656, 1, 4, 2, 1, (1, 656, 1, 8, 64), ("f16x2",)),
    ("col2im Cin 1376 (86 K steps)", True, 1376, 1, 4, 2, 1, (1, 1376, 1, 8, 64), ("f16",)),
    ("c1_tc W = 128 Cin 56", True, 56, 1, 4, 2, 1, (1, 56, 1, 16, 128), MODES_FP16),
    ("col2im H = 12 Cin 56", True, 56, 1, 4, 2, 1, (1, 56, 1, 12, 64), MODES_FP16),
    ("convt_c1 Cin 52", True, 52, 1, 4, 2, 1, (1, 52, 1, 8, 20), MODES_FP16),
    ("convt_c1 Cin 6", True, 6, 1, 4, 2, 1, (1, 6, 1, 8, 20), MODES_FP16),
    ("convt_c1 W = 18", True, 8, 1, 4, 2, 1, (1, 8, 1, 8, 18), MODES_FP16),
    ("skinny K % 4", False, 3, 4, 1, 1, 0, (1, 3, 1, 1, 1), MODES_FP16),
    ("skinny kernel < input", False, 8, 4, 4, 1, 0, (1, 8, 5, 5, 5), MODES_FP16),
]

# ---- operand outputs off the nets' shapes ------------------------------------------------------------------------------
# (name, producer, module arguments, source shapes, requested operands): two shapes per producer at odd B and depths
# Unet_3D does not use; D odd where the layout allows it (a Conv3d k4 s2 output; the parity layout needs even extents)
OPERAND_CASES = [
    ("s4d B3 D4 64x64 c2->12", "block", (2, 12, 8, 2, 3), [(3, 2, 4, 64, 64)], [(PARITY, 16), (PLAIN, 16)]),
    ("s4d B5 D8 64x128 c4->20", "block", (4, 20, 8, 2, 3), [(5, 4, 8, 64, 128)], [(PLAIN, 24), (PARITY, 32)]),
    ("k4s2 B3 D6 32x64 c20->40 (output D 3)", "block", (20, 40, 4, 2, 1), [(3, 20, 6, 32, 64)], [(PLAIN, 40)]),
    ("k4s2 B5 D4 32x32 c24->36", "block", (24, 36, 4, 2, 1), [(5, 24, 4, 32, 32)], [(PARITY, 48), (PLAIN, 40)]),
    ("convt_k4 B3 D3 16x16 skip 16+16->24", "skip", (32, 24, 4, 2, 1), [(3, 16, 3, 16, 16)] * 2,
     [(PLAIN, 24), (PARITY, 32)]),
    ("convt_k4 B5 D1 32x32 skip 16+16->33", "skip", (32, 33, 4, 2, 1), [(5, 16, 1, 32, 32)] * 2,
     [(PARITY, 48), (PLAIN, 40)]),
    ("convt_k8 paired B3 D3 16x32 skip 8+8->20", "skip", (16, 20, 8, 2, 3), [(3, 8, 3, 16, 32)] * 2,
     [(PLAIN, 24), (PARITY, 32)]),
    ("convt_k8 paired B5 D1 32x16 skip 8+8->7", "skip", (16, 7, 8, 2, 3), [(5, 8, 1, 32, 16)] * 2,
     [(PLAIN, 8), (PARITY, 16)]),
]


# ---- the C++ dispatch, restated -----------------------------------------------------------------------------------------
HALO = "convt3d_s2_kernel"
FLAT = "convflat_kernel"
COL2IM = "convt_c1_col2im_kernel"


def _impl(tz, t, npad, mt, mode_, op, pw=0):
    """launch_convt_impl: narrow the x tile until MT x (2 in the split modes) x NPAD accumulator columns fit"""
    while mt > 1 and mt * (2 if op >= 2 else 1) * npad > ACC_COLS:
        mt //= 2
    return (tz, t, npad, mt, mode_, op, pw, 2)


def _op(tz, t, npad, mt, mode_, op):
    """launch_convt_op: op 2 needs N % 16 == 0 and 2 N <= 256 (None: the launch fails); op 3 above N = 128 accumulates
    on one level (OP 0)"""
    if op == 2:
        return None if npad % 16 or 2 * npad > ACC_COLS else _impl(tz, t, npad, mt, mode_, 2)
    if op == 3:
        return _impl(tz, t, npad, mt, mode_, 0 if 2 * npad > ACC_COLS else 3)
    return _impl(tz, t, npad, mt, mode_, 1 if op == 1 else 0)


def _paired(pw, op):
    return (4, 4, 80, 1, 5, 2, pw, 3) if op == 2 else _impl(4, 4, 80, 3, 5, 1, pw)


def halo_instance(entry, op, **a):
    """the convt3d_s2_kernel template arguments an entry point launches for op and its arguments (the dispatch of
    csrc/convt3d.cu); None where it fails"""
    w = a["W"]
    if entry == E_CONVT:                                  # MODE 0, MT = W / 8
        return _op(a["T"], a["T"], a["npad"], w // 8, 0, op)
    if entry == E_MERGED:
        if a.get("paired"):
            return _paired(w, op) if op in (1, 2) else None
        return _op(4, 5, 80, 4 if w % 32 == 0 else 2, 2, op)
    if entry == E_S4D:                                    # npad 80: z class on blockIdx.y (MODE 2); 160: MODE 3
        return _op(3, 3, 80, 2, 2, op) if a["npad"] == 80 else _op(3, 3, 160, 2, 3, op)
    if entry == E_C1TC:
        mt = {64: 8, 32: 4, 16: 2}[w]
        return None if op == 2 else _impl(3, 3, 16, mt, 4, 1 if op == 1 else 0)
    if entry == E_TAPS:                                   # MODE 1
        t, npad = a["T"], a["npad"]
        if npad in (64, 96):
            return _op(t, t, npad, 4 if w % 32 == 0 else 2, 1, op)
        return _op(t, t, 32, {64: 8, 32: 4, 16: 2}[w], 1, op)
    if entry == E_K4S2:
        return _op(2, 2, a["npad"], 4 if w == 32 else 2, 1, op)
    raise ValueError(entry)


def flat_npad(cout):
    return 64 if -(-cout // 64) * 64 < -(-cout // 80) * 80 else 80


def flat_instance(npad, op, b, d, h, w, ntiles, transposed):
    """genre_b200_convflat_forward: two M-tiles per CTA when the grid has >= 120 CTAs at MT 2, narrowed until
    MT x NPAD x parts fit 256 accumulator columns"""
    m = b * (d + 1) * (h + 1) * (w + 1)
    mt = 2 if -(-m // 256) * ntiles * (8 if transposed else 1) >= 120 else 1
    while mt > 1 and mt * npad * (2 if op == 2 else 1) > ACC_COLS:
        mt //= 2
    return (npad, mt, op)


def instance_of(c, mode):
    """(kernel, template arguments) the case launches in `mode`, or None for skinny_gemm (not a template)"""
    op = OP[mode]
    g = c.geometry
    if c.family in ("skinny", "c1"):           # not templates: no instance to tell apart
        return None
    if c.family == "col2im":
        return (COL2IM, (op,))
    if c.family == "flat":
        transposed = c.route["transposed"]
        b, _, d, h, w = c.shapes[0]
        if not transposed:
            d, h, w = d // 2, h // 2, w // 2
        npad = flat_npad(g["cout"])
        return (FLAT, flat_instance(npad, op, b, d, h, w, -(-g["cout"] // npad), transposed))
    a = dict(c.route)
    if c.entry == E_MERGED:
        a["paired"] = mode in MODES_FP16 and a["W"] in (16, 32)      # ops_conv._paired_classes
    if c.entry == E_S4D:
        a["npad"] = 80 if mode in ("f16x2", "fp32x3") else 160         # split_z in the doubled-column modes
    return (HALO, halo_instance(c.entry, op, **a))


def abi_instances():
    """every (kernel, template arguments) the C dispatchers can launch, over all their accepted arguments"""
    out = set()
    ops = (0, 1, 2, 3)

    def add(inst):
        if inst is not None:
            out.add((HALO, inst))
    for op in ops:
        for t in (2, 4):
            for npad in (32, 64):
                for w in (16, 32):
                    add(halo_instance(E_CONVT, op, T=t, npad=npad, W=w))
        for w in (16, 32, 64):
            add(halo_instance(E_MERGED, op, W=w, paired=False))
            add(halo_instance(E_C1TC, op, W=w))
            for t, npad in ((5, 32), (3, 32), (3, 64), (5, 96)):
                add(halo_instance(E_TAPS, op, T=t, npad=npad, W=w))
        for w in (16, 32):
            add(halo_instance(E_MERGED, op, W=w, paired=True))
            for npad in (32, 64, 96, 128):
                add(halo_instance(E_K4S2, op, npad=npad, W=w))
        for npad in (80, 160):
            add(halo_instance(E_S4D, op, npad=npad, W=16))
    for npad in (64, 80):
        for op in (1, 2):
            for mt in (1, 2):
                inst = (npad, mt, op)
                while inst[1] > 1 and inst[1] * npad * (2 if op == 2 else 1) > ACC_COLS:
                    inst = (npad, inst[1] // 2, op)
                out.add((FLAT, inst))
    out |= {(COL2IM, (1,)), (COL2IM, (2,))}
    return out


def table_instances():
    """{(kernel, args): [(case name, mode)]} over the table"""
    out = {}
    for c in CASES:
        for mode in c.modes:
            inst = instance_of(c, mode)
            if inst is not None:
                out.setdefault(inst, []).append((c.name, mode))
    return out


# Instances the C ABI reaches that no case of the table does: (kernel, args) -> (why no route of ops_conv takes it in the
# table's modes, the tests that do run it)
_NONE = "none: reachable only through the C ABI"
_PAIRED = "test_gpu_convt_paired / test_gpu_k8_stream (paired = 0, bit-equal to the paired walk)"
_SPLITZ = "test_gpu_conv_k8_tiles / test_gpu_k8_stream (S4D_SPLIT_Z = True)"
_TAPS3 = "conv3d_taps with 3 taps and npad 32: ops_conv issues 3 taps only at npad 64 (the space-to-depth Conv3d k4 s2)"
_DGRAD16 = "dgrad_convt_k8s2 (N = 96) runs under _forced_mode('tf32'): never with fp16 operands"
ABI_ONLY = {
    (HALO, (3, 3, 32, 2, 1, 0, 0, 2)): (_TAPS3, _NONE),
    (HALO, (3, 3, 32, 2, 1, 1, 0, 2)): (_TAPS3, _NONE),
    (HALO, (3, 3, 32, 2, 1, 2, 0, 2)): (_TAPS3, _NONE),
    (HALO, (3, 3, 32, 2, 1, 3, 0, 2)): (_TAPS3, _NONE),
    (HALO, (3, 3, 32, 4, 1, 0, 0, 2)): (_TAPS3, _NONE),
    (HALO, (3, 3, 32, 4, 1, 1, 0, 2)): (_TAPS3, _NONE),
    (HALO, (3, 3, 32, 4, 1, 2, 0, 2)): (_TAPS3, _NONE),
    (HALO, (3, 3, 32, 4, 1, 3, 0, 2)): (_TAPS3, _NONE),
    (HALO, (3, 3, 32, 8, 1, 0, 0, 2)): (_TAPS3, _NONE),
    (HALO, (3, 3, 32, 8, 1, 1, 0, 2)): (_TAPS3, _NONE),
    (HALO, (3, 3, 80, 2, 2, 0, 0, 2)): ("enc1's split-z form in tf32: S4D_SPLIT_Z is off by default (npad 160 is taken)", _NONE),
    (HALO, (3, 3, 80, 2, 2, 1, 0, 2)): ("enc1's split-z form in f16: S4D_SPLIT_Z is off by default (npad 160 is taken)", _SPLITZ),
    (HALO, (4, 5, 80, 1, 2, 2, 0, 2)): ("merged MODE 2 in the fp16 hi/lo split: ops_conv pairs the classes at W in {16, 32}, "
                                        "the only widths _convt_supported accepts", _PAIRED),
    (HALO, (4, 5, 80, 2, 2, 1, 0, 2)): ("merged MODE 2 with fp16 operands: as above", _PAIRED),
    (HALO, (5, 5, 96, 1, 1, 2, 0, 2)): (_DGRAD16, _NONE),
    (HALO, (5, 5, 96, 2, 1, 1, 0, 2)): (_DGRAD16, _NONE),
}
