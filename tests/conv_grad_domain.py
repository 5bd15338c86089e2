"""The shapes the gradient convolutions of ops_conv accept, as plain data: one case per predicate edge of the tensor-core
input gradients of the k=8 layers (dgrad_convt_k8s2, dgrad_conv_k8s2), the WGAN-GP double backward's grad-of-grad
convolution (_ConvInputGrad.backward -> conv3d(ggx, m), layers with a bias) on each route it takes, and the nearest
shapes the predicates reject.

Both paths run inside ops_conv._forced_mode("tf32"), so they see two effective operand modes:
  tf32    base mode f16 or tf32 with torch.backends.cudnn.allow_tf32 on: single-pass TF32 operands (op 0)
  fp32x3  base mode exact, f16x2 or fp32x3, or allow_tf32 off: the 3xTF32 split (op 3)
The base mode still decides the forward under autograd: in the fp16 modes (f16, f16x2) a ConvTranspose3d needs
Cin % 16 == 0 to run custom, and a layer whose forward falls back to cuDNN has no custom backward either.

A case gives the layer, the forward's input shape x (the output gradient has the forward's output shape), how the
gradient is reached (autograd, or a direct call of the dgrad function for shapes autograd cannot reach), the entry point
and conv_domain.halo_instance arguments of the kernel it must launch, and kappa per effective mode from the
configuration terms of conv_domain's forward cases:
  dgrad_convt_k8s2   the input gradient of ConvTranspose3d(Cin_t -> Cout_t, k8 s2 p3) is the 5-tap form over the 2x
                     space-to-depth of gy (8 Cout_t channels, N = 96 columns, conv3d_taps_forward)
  dgrad_conv_k8s2    that of Conv3d(Cin -> Cout, k8 s2 p3) the merged MODE 2 classes (4 z taps x the 5 x 5 union) over
                     Cout zero-padded to whole K chunks of 8
  double backward    conv3d's own route for the layer: k4s2, the space-to-depth s2d, enc1's s4d or 5-tap form
tests/test_gpu_conv_grad_fp64.py runs the table against fp64; tests/test_conv_domain_cpu.py counts its kernel instances
in the ledger.
"""
import torch

import conv_domain as D
from genre_shapehd_b200.networks import networks as nets

EFFECTIVE = ("tf32", "fp32x3")
# id -> (ops_conv.PRECISION, cudnn.allow_tf32, the forward's operand mode, the gradient convolutions' effective mode)
SETTINGS = {
    "tf32": ("tf32", True, "tf32", "tf32"),
    "f16": ("f16", True, "f16", "tf32"),
    "exact": ("exact", True, "f16x2", "fp32x3"),
    "fp32x3": ("fp32x3", True, "fp32x3", "fp32x3"),
    "exact tf32 off": ("exact", False, "f16x2", "fp32x3"),
}


class GradCase:
    """kind: dgrad_convt (ConvTranspose3d k8 s2 p3) | dgrad_conv (Conv3d k8 s2 p3) | double (Conv3d with a bias: the
    grad-of-grad convolution).  x: the forward's input shape; via: autograd | direct; entry, route: the entry point and
    halo_instance arguments (a dict value is per effective mode), entry None for a rejected neighbour"""

    def __init__(self, name, kind, cin, cout, k, x, via, entry, route, kappa):
        self.name, self.kind, self.cin, self.cout, self.k, self.x = name, kind, cin, cout, k, tuple(x)
        self.via, self.entry, self.route, self._kappa = via, entry, route, kappa
        self.p = 3 if k == 8 else 1

    @property
    def transposed(self):
        return self.kind == "dgrad_convt"

    @property
    def gy(self):
        """the forward's output shape"""
        b, _, d, h, w = self.x
        if self.transposed:
            return (b, self.cout, 2 * d, 2 * h, 2 * w)
        return (b, self.cout, d // 2, h // 2, w // 2)

    @property
    def products(self):
        """products per output of the gradient convolution (interior): dx of a ConvTranspose3d k8 s2 reads all 8^3 taps
        of gy, dx of a Conv3d k8 s2 the 4^3 of one parity class, the double backward is the forward convolution"""
        if self.kind == "dgrad_convt":
            return self.cout * 512
        if self.kind == "dgrad_conv":
            return self.cout * 64
        return self.cin * self.k ** 3

    def runs_custom(self, fwd_mode):
        """does the gradient run on the entry point with the forward in fwd_mode?"""
        if self.entry is None:
            return False
        if self.kind == "dgrad_convt" and self.via == "autograd":      # ops_conv._convt_supported: Cin % (2 groups)
            return self.cin % (16 if fwd_mode in D.MODES_FP16 else 8) == 0
        return True

    def kappa(self, mode):
        return self._kappa(mode)

    def instance(self, mode):
        a = {k: (v[mode] if isinstance(v, dict) else v) for k, v in self.route.items()}
        if self.entry == D.E_MERGED:
            a["paired"] = False                      # dgrad_conv_k8s2 walks the union of the classes' taps
        return (D.HALO, D.halo_instance(self.entry, D.OP[mode], **a))

    def __repr__(self):
        return "GradCase(%s)" % self.name


def _convt(name, cin, cout, x, via="autograd", entry=D.E_TAPS):
    """ConvTranspose3d(cin -> cout, 8, 2, 3): dx = the 5-tap form over the space-to-depth of gy, W' = x's width"""
    return GradCase(name, "dgrad_convt", cin, cout, 8, x, via, entry, dict(T=5, npad=96, W=x[4]), D._kappa_taps(5, 8 * cout))


def _conv(name, cin, cout, x, via="autograd", entry=D.E_MERGED):
    """Conv3d(cin -> cout, 8, 2, 3): dx = the merged MODE 2 classes over gy (W = gy's width), Cout padded to 8"""
    return GradCase(name, "dgrad_conv", cin, cout, 8, x, via, entry, dict(W=x[4] // 2), D._kappa_merged(-(-cout // 8) * 8))


def _double(name, cin, cout, k, x, entry, route, kappa):
    return GradCase(name, "double", cin, cout, k, x, "autograd", entry, route, kappa)


CASES = [
    # dgrad_convt_k8s2: Cin_t <= 96 (cgo <= 24 of N = 96), any Cout_t (K = 8 Cout_t), gy width 2W with W in {16, 32, 64}
    _convt("convt 80->20 B1 D2 16x16 (dec5's channels, W' 16)", 80, 20, (1, 80, 2, 16, 16)),
    _convt("convt 96->20 B3 D1 16x32 (N edge)", 96, 20, (3, 96, 1, 16, 32)),
    _convt("convt 8->2 B1 D3 48x16 (K 16, three row tiles)", 8, 2, (1, 8, 3, 48, 16)),
    _convt("convt 16->64 B2 D2 16x32 (K 512, non-merged forward)", 16, 64, (2, 16, 2, 16, 32)),
    _convt("convt 5->7 B1 D2 16x64 direct (W' 64, partial group)", 5, 7, (1, 5, 2, 16, 64), via="direct"),
    _convt("convt 112->20 B1 D1 16x16 (Cin_t past 96: cuDNN)", 112, 20, (1, 112, 1, 16, 16), entry=None),
    _convt("convt 16->8 B1 D1 16x24 direct (W 24: rejected)", 16, 8, (1, 16, 1, 16, 24), via="direct", entry=None),
    # dgrad_conv_k8s2: Cin <= 20 (cgo <= 5 of N = 80 / 4 classes), gy height % 16, gy width 16 or a multiple of 32
    _conv("conv 2->20 B1 D2 32x32 (gy one plane, 16 wide)", 2, 20, (1, 2, 2, 32, 32)),
    _conv("conv 8->32 B3 D6 32x64 (Cin limit, Cout unpadded, odd gy depth)", 8, 32, (3, 8, 6, 32, 64)),
    _conv("conv 4->7 B1 D4 64x128 (Cout padded by 1, gy 64 wide)", 4, 7, (1, 4, 4, 64, 128)),
    _conv("conv 2->1 B2 D2 32x32 (one K chunk, 7 of 8 padding)", 2, 1, (2, 2, 2, 32, 32)),
    _conv("conv 20->12 B1 D2 32x64 direct (N edge)", 20, 12, (1, 20, 2, 32, 64), via="direct"),
    _conv("conv 5->3 B3 D4 32x32 direct (Cin 5)", 5, 3, (3, 5, 4, 32, 32), via="direct"),
    _conv("conv 4->8 B1 D2 32x192 direct (gy 96 wide)", 4, 8, (1, 4, 2, 32, 192), via="direct"),
    _conv("conv 21->8 B1 D2 32x32 direct (Cin 21: rejected)", 21, 8, (1, 21, 2, 32, 32), via="direct", entry=None),
    _conv("conv 4->8 B1 D2 32x96 direct (gy 48 wide: rejected)", 4, 8, (1, 4, 2, 32, 96), via="direct", entry=None),
    # the double backward: conv3d(ggx, m) without the bias, on the layer's inference route
    _double("double s2d 1->64 B3 D4 32x32 (critic main.0)", 1, 64, 4, (3, 1, 4, 32, 32), D.E_TAPS,
            dict(T=3, npad=64, W=16), D._kappa_taps(3, 8)),
    _double("double s2d 2->33 B3 D2 32x128 (Cout > 32 edge, widest)", 2, 33, 4, (3, 2, 2, 32, 128), D.E_TAPS,
            dict(T=3, npad=64, W=64), D._kappa_taps(3, 16)),
    _double("double k4s2 8->128 B3 D2 32x64 (Cin and Cout limits)", 8, 128, 4, (3, 8, 2, 32, 64), D.E_K4S2,
            dict(npad=128, W=32), D._kappa_k4s2(8)),
    _double("double k4s2 64->64 B3 D4 32x32", 64, 64, 4, (3, 64, 4, 32, 32), D.E_K4S2, dict(npad=64, W=16), D._kappa_k4s2(64)),
    _double("double k8s2 s4d 2->20 B3 D4 64x64", 2, 20, 8, (3, 2, 4, 64, 64), D.E_S4D,
            dict(npad={"tf32": 160, "fp32x3": 80}, W=16), D._kappa_s4d(2)),
    _double("double k8s2 taps5 2->32 B3 D2 32x32", 2, 32, 8, (3, 2, 2, 32, 32), D.E_TAPS, dict(T=5, npad=32, W=16),
            D._kappa_taps(5, 16)),
]
CASE_IDS = [c.name for c in CASES]


def case(name):
    return next(c for c in CASES if c.name == name)


def module(c):
    """the case's layer on the CPU, PyTorch's default initialisation (the bias included) under a per-case seed"""
    torch.manual_seed(c.cin * 131 + c.cout)
    return (nets.ConvTranspose3d if c.transposed else nets.Conv3d)(c.cin, c.cout, c.k, 2, c.p)


def table_instances():
    """{(kernel, args): [(case name, effective mode)]} over the cases that run a kernel"""
    out = {}
    for c in CASES:
        if c.entry is None:
            continue
        for mode in EFFECTIVE:
            out.setdefault(c.instance(mode), []).append((c.name, mode))
    return out
