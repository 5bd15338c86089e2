"""The route functions of ops_conv (_conv_route, _convt_route) on shapes alone, without a device.

They must name the kernel each convolution runs, as the GPU suites observe it:
  - every case of conv_domain.CASES in each of its operand modes: the entry point and kernel family the case launches;
  - every conv_domain.BOUNDARIES shape: no kernel;
  - every conv_domain.OPERAND_CASES producer: a route that writes operand outputs;
  - the forward and gradient routes of conv_grad_domain.CASES;
  - LAYERS: per layer, the entry point of each ops_conv call recorded on an H100 80GB HBM3 (test_gpu_infer_fp64._calls) in one
    eval forward of Unet_3D at bench.py's B = 16 in the default and the f16 mode, one eval forward each of VoxelDecoder,
    VoxelGenerator and VoxelDiscriminator at the WGAN-GP batch of 8, one Unet_3D training step at B = 4 and one WGAN-GP
    gradient-penalty step of VoxelDiscriminator at B = 2, with the operand-layout answers of the Unet_3D runs (LAYOUTS).
"""
import pytest
import torch

import conv_domain as D
import conv_grad_domain as G
from genre_shapehd_b200 import ops_conv
from genre_shapehd_b200.networks import networks as nets


@pytest.fixture(autouse=True)
def _defaults(monkeypatch):
    monkeypatch.setattr(ops_conv, "PRECISION", "exact")
    monkeypatch.setattr(ops_conv, "POLICY", set(ops_conv._default_policy))
    monkeypatch.setattr(torch.backends.cudnn, "allow_tf32", True)


def route_of(entry, m):
    """the route an entry point (genre_b200_ prefix optional) is launched from, for layer m"""
    e = entry.replace("genre_b200_", "").replace("[operands]", "")
    k8 = m.kernel_size[0] == 8
    return {"convt3d_s2_forward": "convt_k8" if k8 else "convt_k4", "convt3d_s2_merged_forward": "convt_k8",
            "conv3d_k4s2_forward": "conv_k4s2", "conv3d_k8s2_s4d_forward": "conv_k8s2",
            "conv3d_taps_forward": "conv_k8s2" if k8 else "conv_k4s2_s2d", "convt_c1_tc_forward": "convt_c1_tc",
            "convt_c1_col2im_forward": "convt_c1_col2im", "convflat_forward": "flat", "skinny_gemm": "skinny",
            "convt_c1_forward": "convt_c1"}[e]


def _check_form(entry, m, shape):
    """the k8 s2 Conv3d launches the 4x space-to-depth form through conv3d_k8s2_s4d_forward, the 5-tap one otherwise"""
    if route_of(entry, m) == "conv_k8s2":
        assert ops_conv._conv_k8s2_s4d_form(shape, m) == ("s4d" in entry), (entry, shape)


def _bn(state):
    return None if state is None else torch.nn.BatchNorm3d(1).train(state == "batch")


def _route(m, srcs, bn=None, slope=False, grad=False, sigmoid=False):
    if isinstance(m, torch.nn.ConvTranspose3d):
        return ops_conv._convt_route(m, srcs, bn, slope, grad, sigmoid)
    return None if sigmoid else ops_conv._conv_route(m, srcs[0], bn, slope, grad)


# ---- conv_domain ---------------------------------------------------------------------------------------------------------
def _case_module(transposed, cin, cout, k, s, p, bias=True):
    with torch.device("meta"):
        return (nets.ConvTranspose3d if transposed else nets.Conv3d)(cin, cout, k, s, p, bias=bias)


@pytest.mark.parametrize("name,mode", [(c.name, mode) for c in D.CASES for mode in c.modes])
def test_domain_case_route(name, mode):
    c = D.case(name)
    g = c.geometry
    transposed = c.kind in ("convt", "skip") or c.entry in (D.E_CONVT, D.E_C1TC) or bool(c.route.get("transposed"))
    m = _case_module(transposed, g["cin"], g["cout"], g["k"], g["s"], g["p"], g["bias"])
    srcs = [(s, "plain") for s in c.shapes]
    bn = _bn("eval" if g["bn"] else None)
    with ops_conv.precision(mode), torch.no_grad():
        got = _route(m, srcs, bn, g["act"] in ("relu", "lrelu"), sigmoid=g["act"] == "sigmoid")
        assert got == route_of(c.entry, m), (name, mode, got)
        _check_form(c.entry, m, c.shapes[0])


@pytest.mark.parametrize("spec,mode", [(b, mode) for b in D.BOUNDARIES for mode in b[-1]], ids=lambda v: str(v)[:40])
def test_boundary_shape_has_no_route(spec, mode):
    name, transposed, cin, cout, k, s, p, shape, _ = spec
    m = _case_module(transposed, cin, cout, k, s, p)
    with ops_conv.precision(mode), torch.no_grad():
        assert _route(m, [(shape, "plain")]) is None, name


@pytest.mark.parametrize("mode", ["f16x2", "f16"])
@pytest.mark.parametrize("spec", D.OPERAND_CASES, ids=[o[0] for o in D.OPERAND_CASES])
def test_operand_producer_route_writes_operands(spec, mode):
    name, kind, (cin, cout, k, s, p), shapes, _ = spec
    m = _case_module(kind == "skip", cin, cout, k, s, p)
    with ops_conv.precision(mode), torch.no_grad():
        got = _route(m, [(sh, "plain") for sh in shapes], _bn("eval"), True)
        assert got in ("conv_k4s2", "conv_k8s2", "convt_k4", "convt_k8"), (name, got)
        if got == "conv_k8s2":
            assert ops_conv._conv_k8s2_s4d_form(shapes[0], m)
        if got == "convt_k8":
            assert ops_conv.MERGE_PARITIES and cout <= 20 and ops_conv._paired_classes(8, shapes[0][4])


# ---- conv_grad_domain ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("setting", list(G.SETTINGS))
@pytest.mark.parametrize("name", G.CASE_IDS)
def test_gradient_case_routes(name, setting, monkeypatch):
    c = G.case(name)
    precision, tf32, fwd_mode, _ = G.SETTINGS[setting]
    monkeypatch.setattr(ops_conv, "PRECISION", precision)
    monkeypatch.setattr(torch.backends.cudnn, "allow_tf32", tf32)
    m = G.module(c)
    assert ops_conv._mode() == fwd_mode
    fwd = _route(m, [(c.x, "plain")], grad=True)
    if c.kind == "dgrad_convt" and c.via == "autograd":
        assert (fwd == "train_forward") == (c.cin % (16 if fwd_mode in D.MODES_FP16 else 8) == 0), fwd
    elif c.via == "autograd":
        assert fwd == "train_forward", fwd
    if c.kind == "double":
        with ops_conv._forced_mode("tf32"), torch.no_grad():
            assert _route(m, [(c.x, "plain")]) == route_of(c.entry, m)
            _check_form(c.entry, m, c.x)
    else:
        assert ops_conv._tc_dgrad_supported(c.gy, m) == (c.entry is not None)


# ---- the nets' layers, as recorded on the GPU ----------------------------------------------------------------------------
# (run, ops_conv call, layer, sources ((shape, kind), ...), BatchNorm (None | eval | batch), slope / act, needs_grad, mode,
#  convolution entry points called)  for forward calls;
# (run, backward, layer, (gy shape, x shape), needs_input_grad[:2], None, grad enabled, mode, entry points)  for backward ones
LAYERS = [
    ('unet_eval_b16', 'conv3d', 'enc1.net.0', (((16, 2, 128, 128, 128), 'plain'),), 'eval', 'slope', False, 'f16x2', ('conv3d_k8s2_s4d_forward[operands]',)),
    ('unet_eval_b16', 'conv3d', 'enc2.net.0', (((16, 20, 64, 64, 64), 'operand'),), 'eval', 'slope', False, 'f16x2', ('conv3d_k4s2_forward[operands]',)),
    ('unet_eval_b16', 'conv3d', 'enc3.net.0', (((16, 40, 32, 32, 32), 'operand'),), 'eval', 'slope', False, 'f16x2', ('conv3d_k4s2_forward',)),
    ('unet_eval_b16', 'conv3d', 'enc4.net.0', (((16, 80, 16, 16, 16), 'twin'),), 'eval', 'slope', False, 'f16x2', ('convflat_forward',)),
    ('unet_eval_b16', 'conv3d', 'enc5.net.0', (((16, 160, 8, 8, 8), 'plain'),), 'eval', 'slope', False, 'f16x2', ('convflat_forward',)),
    ('unet_eval_b16', 'conv3d', 'enc6.net.0', (((16, 320, 4, 4, 4), 'plain'),), 'eval', 'slope', False, 'f16x2', ('skinny_gemm',)),
    ('unet_eval_b16', 'deconv_skip', 'dec1.net.0', (((16, 640, 1, 1, 1), 'plain'), ((16, 640, 1, 1, 1), 'plain')), 'eval', 'slope', False, 'f16x2', ('skinny_gemm',)),
    ('unet_eval_b16', 'deconv_skip', 'dec2.net.0', (((16, 320, 4, 4, 4), 'plain'), ((16, 320, 4, 4, 4), 'plain')), 'eval', 'slope', False, 'f16x2', ('convflat_forward',)),
    ('unet_eval_b16', 'deconv_skip', 'dec3.net.0', (((16, 160, 8, 8, 8), 'plain'), ((16, 160, 8, 8, 8), 'plain')), 'eval', 'slope', False, 'f16x2', ('convflat_forward',)),
    ('unet_eval_b16', 'deconv_skip', 'dec4.net.0', (((16, 80, 16, 16, 16), 'plain'), ((16, 80, 16, 16, 16), 'twin')), 'eval', 'slope', False, 'f16x2', ('convt3d_s2_forward[operands]',)),
    ('unet_eval_b16', 'deconv_skip', 'dec5.net.0', (((16, 40, 32, 32, 32), 'operand'), ((16, 40, 32, 32, 32), 'operand')), 'eval', 'slope', False, 'f16x2', ('convt3d_s2_merged_forward[operands]',)),
    ('unet_eval_b16', 'deconv_skip', 'dec6.net', (((16, 20, 64, 64, 64), 'operand'), ((16, 20, 64, 64, 64), 'operand')), None, None, False, 'f16x2', ('convt_c1_col2im_forward',)),
    ('unet_eval_b16_f16', 'conv3d', 'enc1.net.0', (((16, 2, 128, 128, 128), 'plain'),), 'eval', 'slope', False, 'f16', ('conv3d_k8s2_s4d_forward[operands]',)),
    ('unet_eval_b16_f16', 'conv3d', 'enc2.net.0', (((16, 20, 64, 64, 64), 'operand'),), 'eval', 'slope', False, 'f16', ('conv3d_k4s2_forward[operands]',)),
    ('unet_eval_b16_f16', 'conv3d', 'enc3.net.0', (((16, 40, 32, 32, 32), 'operand'),), 'eval', 'slope', False, 'f16', ('conv3d_k4s2_forward',)),
    ('unet_eval_b16_f16', 'conv3d', 'enc4.net.0', (((16, 80, 16, 16, 16), 'twin'),), 'eval', 'slope', False, 'f16', ('convflat_forward',)),
    ('unet_eval_b16_f16', 'conv3d', 'enc5.net.0', (((16, 160, 8, 8, 8), 'plain'),), 'eval', 'slope', False, 'f16', ('convflat_forward',)),
    ('unet_eval_b16_f16', 'conv3d', 'enc6.net.0', (((16, 320, 4, 4, 4), 'plain'),), 'eval', 'slope', False, 'f16', ('skinny_gemm',)),
    ('unet_eval_b16_f16', 'deconv_skip', 'dec1.net.0', (((16, 640, 1, 1, 1), 'plain'), ((16, 640, 1, 1, 1), 'plain')), 'eval', 'slope', False, 'f16', ('skinny_gemm',)),
    ('unet_eval_b16_f16', 'deconv_skip', 'dec2.net.0', (((16, 320, 4, 4, 4), 'plain'), ((16, 320, 4, 4, 4), 'plain')), 'eval', 'slope', False, 'f16', ('convflat_forward',)),
    ('unet_eval_b16_f16', 'deconv_skip', 'dec3.net.0', (((16, 160, 8, 8, 8), 'plain'), ((16, 160, 8, 8, 8), 'plain')), 'eval', 'slope', False, 'f16', ('convflat_forward',)),
    ('unet_eval_b16_f16', 'deconv_skip', 'dec4.net.0', (((16, 80, 16, 16, 16), 'plain'), ((16, 80, 16, 16, 16), 'twin')), 'eval', 'slope', False, 'f16', ('convt3d_s2_forward[operands]',)),
    ('unet_eval_b16_f16', 'deconv_skip', 'dec5.net.0', (((16, 40, 32, 32, 32), 'operand'), ((16, 40, 32, 32, 32), 'operand')), 'eval', 'slope', False, 'f16', ('convt3d_s2_merged_forward[operands]',)),
    ('unet_eval_b16_f16', 'deconv_skip', 'dec6.net', (((16, 20, 64, 64, 64), 'operand'), ((16, 20, 64, 64, 64), 'operand')), None, None, False, 'f16', ('convt_c1_col2im_forward',)),
    ('unet_train_b4', 'conv3d', 'enc1.net.0', (((4, 2, 128, 128, 128), 'plain'),), 'batch', 'slope', True, 'f16x2', ()),
    ('unet_train_b4', 'conv3d', 'enc1.net.0', (((4, 2, 128, 128, 128), 'plain'),), None, None, True, 'f16x2', ('conv3d_k8s2_s4d_forward',)),
    ('unet_train_b4', 'conv3d', 'enc2.net.0', (((4, 20, 64, 64, 64), 'plain'),), 'batch', 'slope', True, 'f16x2', ()),
    ('unet_train_b4', 'conv3d', 'enc2.net.0', (((4, 20, 64, 64, 64), 'plain'),), None, None, True, 'f16x2', ('conv3d_k4s2_forward',)),
    ('unet_train_b4', 'conv3d', 'enc3.net.0', (((4, 40, 32, 32, 32), 'plain'),), 'batch', 'slope', True, 'f16x2', ()),
    ('unet_train_b4', 'conv3d', 'enc3.net.0', (((4, 40, 32, 32, 32), 'plain'),), None, None, True, 'f16x2', ('conv3d_k4s2_forward',)),
    ('unet_train_b4', 'conv3d', 'enc4.net.0', (((4, 80, 16, 16, 16), 'plain'),), 'batch', 'slope', True, 'f16x2', ()),
    ('unet_train_b4', 'conv3d', 'enc4.net.0', (((4, 80, 16, 16, 16), 'plain'),), None, None, True, 'f16x2', ()),
    ('unet_train_b4', 'conv3d', 'enc5.net.0', (((4, 160, 8, 8, 8), 'plain'),), 'batch', 'slope', True, 'f16x2', ()),
    ('unet_train_b4', 'conv3d', 'enc5.net.0', (((4, 160, 8, 8, 8), 'plain'),), None, None, True, 'f16x2', ()),
    ('unet_train_b4', 'conv3d', 'enc6.net.0', (((4, 320, 4, 4, 4), 'plain'),), 'batch', 'slope', True, 'f16x2', ()),
    ('unet_train_b4', 'conv3d', 'enc6.net.0', (((4, 320, 4, 4, 4), 'plain'),), None, None, True, 'f16x2', ()),
    ('unet_train_b4', 'deconv_skip', 'dec1.net.0', (((4, 640, 1, 1, 1), 'plain'), ((4, 640, 1, 1, 1), 'plain')), 'batch', 'slope', True, 'f16x2', ()),
    ('unet_train_b4', 'conv_transpose3d', 'dec1.net.0', (((4, 1280, 1, 1, 1), 'plain'),), None, None, True, 'f16x2', ()),
    ('unet_train_b4', 'deconv_skip', 'dec2.net.0', (((4, 320, 4, 4, 4), 'plain'), ((4, 320, 4, 4, 4), 'plain')), 'batch', 'slope', True, 'f16x2', ()),
    ('unet_train_b4', 'conv_transpose3d', 'dec2.net.0', (((4, 640, 4, 4, 4), 'plain'),), None, None, True, 'f16x2', ()),
    ('unet_train_b4', 'deconv_skip', 'dec3.net.0', (((4, 160, 8, 8, 8), 'plain'), ((4, 160, 8, 8, 8), 'plain')), 'batch', 'slope', True, 'f16x2', ()),
    ('unet_train_b4', 'conv_transpose3d', 'dec3.net.0', (((4, 320, 8, 8, 8), 'plain'),), None, None, True, 'f16x2', ()),
    ('unet_train_b4', 'deconv_skip', 'dec4.net.0', (((4, 80, 16, 16, 16), 'plain'), ((4, 80, 16, 16, 16), 'plain')), 'batch', 'slope', True, 'f16x2', ()),
    ('unet_train_b4', 'conv_transpose3d', 'dec4.net.0', (((4, 160, 16, 16, 16), 'plain'),), None, None, True, 'f16x2', ('convt3d_s2_forward',)),
    ('unet_train_b4', 'deconv_skip', 'dec5.net.0', (((4, 40, 32, 32, 32), 'plain'), ((4, 40, 32, 32, 32), 'plain')), 'batch', 'slope', True, 'f16x2', ()),
    ('unet_train_b4', 'conv_transpose3d', 'dec5.net.0', (((4, 80, 32, 32, 32), 'plain'),), None, None, True, 'f16x2', ('convt3d_s2_merged_forward',)),
    ('unet_train_b4', 'deconv_skip', 'dec6.net', (((4, 20, 64, 64, 64), 'plain'), ((4, 20, 64, 64, 64), 'plain')), None, None, True, 'f16x2', ()),
    ('unet_train_b4', 'conv_transpose3d', 'dec6.net', (((4, 40, 64, 64, 64), 'plain'),), None, None, True, 'f16x2', ('convt_c1_forward',)),
    ('unet_train_b4', '_ConvForward.backward', 'dec5.net.0', ((4, 20, 64, 64, 64), (4, 80, 32, 32, 32)), (True, True), None, False, 'f16x2', ('conv3d_taps_forward',)),
    ('unet_train_b4', '_ConvForward.backward', 'dec4.net.0', ((4, 40, 32, 32, 32), (4, 160, 16, 16, 16)), (True, True), None, False, 'f16x2', ()),
    ('unet_train_b4', '_ConvForward.backward', 'enc3.net.0', ((4, 80, 16, 16, 16), (4, 40, 32, 32, 32)), (True, True), None, False, 'f16x2', ()),
    ('unet_train_b4', '_ConvForward.backward', 'enc2.net.0', ((4, 40, 32, 32, 32), (4, 20, 64, 64, 64)), (True, True), None, False, 'f16x2', ()),
    ('unet_train_b4', '_ConvForward.backward', 'enc1.net.0', ((4, 20, 64, 64, 64), (4, 2, 128, 128, 128)), (False, True), None, False, 'f16x2', ('conv_k8s2_wgrad',)),
    ('vdec_eval_b8', 'fused_block', 'main.0', (((8, 200, 1, 1, 1), 'plain'),), 'eval', 'ReLU', False, 'f16x2', ('skinny_gemm',)),
    ('vdec_eval_b8', 'fused_block', 'main.3', (((8, 512, 4, 4, 4), 'plain'),), 'eval', 'ReLU', False, 'f16x2', ('convflat_forward',)),
    ('vdec_eval_b8', 'fused_block', 'main.8', (((8, 256, 8, 8, 8), 'plain'),), 'eval', 'ReLU', False, 'f16x2', ('convflat_forward',)),
    ('vdec_eval_b8', 'fused_block', 'main.11', (((8, 128, 16, 16, 16), 'plain'),), 'eval', 'ReLU', False, 'f16x2', ('convt3d_s2_forward',)),
    ('vdec_eval_b8', 'fused_block', 'main.14', (((8, 64, 32, 32, 32), 'twin'),), 'eval', 'ReLU', False, 'f16x2', ('convt3d_s2_forward',)),
    ('vdec_eval_b8', 'conv_transpose3d', 'main.17', (((8, 32, 64, 64, 64), 'twin'),), None, None, False, 'f16x2', ('convt_c1_col2im_forward',)),
    ('vgen_eval_b8', 'fused_block', 'main.0', (((8, 200, 1, 1, 1), 'plain'),), 'eval', 'ReLU', False, 'f16x2', ('skinny_gemm',)),
    ('vgen_eval_b8', 'fused_block', 'main.3', (((8, 512, 4, 4, 4), 'plain'),), 'eval', 'ReLU', False, 'f16x2', ('convflat_forward',)),
    ('vgen_eval_b8', 'fused_block', 'main.6', (((8, 256, 8, 8, 8), 'plain'),), 'eval', 'ReLU', False, 'f16x2', ('convflat_forward',)),
    ('vgen_eval_b8', 'fused_block', 'main.9', (((8, 128, 16, 16, 16), 'plain'),), 'eval', 'ReLU', False, 'f16x2', ('convt3d_s2_forward',)),
    ('vgen_eval_b8', 'fused_block', 'main.12', (((8, 64, 32, 32, 32), 'twin'),), 'eval', 'ReLU', False, 'f16x2', ('convt3d_s2_forward',)),
    ('vgen_eval_b8', 'fused_block', 'main.15', (((8, 64, 64, 64, 64), 'twin'),), None, 'Sigmoid', False, 'f16x2', ()),
    ('vgen_eval_b8', 'conv_transpose3d', 'main.15', (((8, 64, 64, 64, 64), 'twin'),), None, None, False, 'f16x2', ('convt_c1_col2im_forward',)),
    ('vdis_eval_b8', 'fused_block', 'main.0', (((8, 1, 128, 128, 128), 'plain'),), None, 'LeakyReLU', False, 'f16x2', ('conv3d_taps_forward',)),
    ('vdis_eval_b8', 'fused_block', 'main.2', (((8, 64, 64, 64, 64), 'twin'),), None, 'LeakyReLU', False, 'f16x2', ('conv3d_k4s2_forward',)),
    ('vdis_eval_b8', 'fused_block', 'main.4', (((8, 64, 32, 32, 32), 'twin'),), None, 'LeakyReLU', False, 'f16x2', ('conv3d_k4s2_forward',)),
    ('vdis_eval_b8', 'fused_block', 'main.6', (((8, 128, 16, 16, 16), 'twin'),), None, 'LeakyReLU', False, 'f16x2', ('convflat_forward',)),
    ('vdis_eval_b8', 'fused_block', 'main.8', (((8, 256, 8, 8, 8), 'plain'),), None, 'LeakyReLU', False, 'f16x2', ('convflat_forward',)),
    ('vdis_eval_b8', 'conv3d', 'main.10', (((8, 512, 4, 4, 4), 'plain'),), None, None, False, 'f16x2', ('skinny_gemm',)),
    ('vdis_gp_b2', 'fused_block', 'main.0', (((2, 1, 128, 128, 128), 'plain'),), None, 'LeakyReLU', True, 'f16x2', ()),
    ('vdis_gp_b2', 'conv3d', 'main.0', (((2, 1, 128, 128, 128), 'plain'),), None, None, True, 'f16x2', ('conv3d_taps_forward',)),
    ('vdis_gp_b2', 'fused_block', 'main.2', (((2, 64, 64, 64, 64), 'plain'),), None, 'LeakyReLU', True, 'f16x2', ()),
    ('vdis_gp_b2', 'conv3d', 'main.2', (((2, 64, 64, 64, 64), 'plain'),), None, None, True, 'f16x2', ('conv3d_k4s2_forward',)),
    ('vdis_gp_b2', 'fused_block', 'main.4', (((2, 64, 32, 32, 32), 'plain'),), None, 'LeakyReLU', True, 'f16x2', ()),
    ('vdis_gp_b2', 'conv3d', 'main.4', (((2, 64, 32, 32, 32), 'plain'),), None, None, True, 'f16x2', ('conv3d_k4s2_forward',)),
    ('vdis_gp_b2', 'fused_block', 'main.6', (((2, 128, 16, 16, 16), 'plain'),), None, 'LeakyReLU', True, 'f16x2', ()),
    ('vdis_gp_b2', 'conv3d', 'main.6', (((2, 128, 16, 16, 16), 'plain'),), None, None, True, 'f16x2', ()),
    ('vdis_gp_b2', 'fused_block', 'main.8', (((2, 256, 8, 8, 8), 'plain'),), None, 'LeakyReLU', True, 'f16x2', ()),
    ('vdis_gp_b2', 'conv3d', 'main.8', (((2, 256, 8, 8, 8), 'plain'),), None, None, True, 'f16x2', ()),
    ('vdis_gp_b2', 'conv3d', 'main.10', (((2, 512, 4, 4, 4), 'plain'),), None, None, True, 'f16x2', ()),
    ('vdis_gp_b2', '_ConvForward.backward', 'main.4', ((2, 128, 16, 16, 16), (2, 64, 32, 32, 32)), (True, True), None, True, 'f16x2', ()),
    ('vdis_gp_b2', '_ConvForward.backward', 'main.2', ((2, 64, 32, 32, 32), (2, 64, 64, 64, 64)), (True, True), None, True, 'f16x2', ()),
    ('vdis_gp_b2', '_ConvForward.backward', 'main.0', ((2, 64, 64, 64, 64), (2, 1, 128, 128, 128)), (True, True), None, True, 'f16x2', ()),
    ('vdis_gp_b2', '_ConvInputGrad.backward', 'main.0', ((2, 1, 128, 128, 128), None), (True, True), None, False, 'f16x2', ('conv3d_taps_forward',)),
    ('vdis_gp_b2', '_ConvInputGrad.backward', 'main.2', ((2, 64, 64, 64, 64), None), (True, True), None, False, 'f16x2', ('conv3d_k4s2_forward',)),
    ('vdis_gp_b2', '_ConvInputGrad.backward', 'main.4', ((2, 64, 32, 32, 32), None), (True, True), None, False, 'f16x2', ('conv3d_k4s2_forward',)),
    ('vdis_gp_b2', '_ConvForward.backward', 'main.4', ((2, 128, 16, 16, 16), (2, 64, 32, 32, 32)), (True, True), None, False, 'f16x2', ()),
    ('vdis_gp_b2', '_ConvForward.backward', 'main.2', ((2, 64, 32, 32, 32), (2, 64, 64, 64, 64)), (True, True), None, False, 'f16x2', ()),
    ('vdis_gp_b2', '_ConvForward.backward', 'main.0', ((2, 64, 64, 64, 64), (2, 1, 128, 128, 128)), (True, True), None, False, 'f16x2', ()),
]
# (run, block, operand_layout arguments, mode, answer)
LAYOUTS = [
    ('unet_eval_b16', 'enc2', ((16, 20, 64, 64, 64),), 'f16x2', (2, 32)),
    ('unet_eval_b16', 'dec6', ((16, 20, 64, 64, 64), (16, 20, 64, 64, 64)), 'f16x2', (1, 24)),
    ('unet_eval_b16', 'enc3', ((16, 40, 32, 32, 32),), 'f16x2', (2, 48)),
    ('unet_eval_b16', 'dec5', ((16, 40, 32, 32, 32), (16, 40, 32, 32, 32)), 'f16x2', (1, 40)),
    ('unet_eval_b16', 'enc4', ((16, 80, 16, 16, 16),), 'f16x2', None),
    ('unet_eval_b16', 'dec4', ((16, 80, 16, 16, 16), (16, 80, 16, 16, 16)), 'f16x2', (1, 80)),
    ('unet_eval_b16', 'enc5', ((16, 160, 8, 8, 8),), 'f16x2', None),
    ('unet_eval_b16', 'dec3', ((16, 160, 8, 8, 8), (16, 160, 8, 8, 8)), 'f16x2', None),
    ('unet_eval_b16', 'enc6', ((16, 320, 4, 4, 4),), 'f16x2', None),
    ('unet_eval_b16', 'dec2', ((16, 320, 4, 4, 4), (16, 320, 4, 4, 4)), 'f16x2', None),
    ('unet_eval_b16_f16', 'enc2', ((16, 20, 64, 64, 64),), 'f16', (2, 32)),
    ('unet_eval_b16_f16', 'dec6', ((16, 20, 64, 64, 64), (16, 20, 64, 64, 64)), 'f16', (1, 24)),
    ('unet_eval_b16_f16', 'enc3', ((16, 40, 32, 32, 32),), 'f16', (2, 48)),
    ('unet_eval_b16_f16', 'dec5', ((16, 40, 32, 32, 32), (16, 40, 32, 32, 32)), 'f16', (1, 40)),
    ('unet_eval_b16_f16', 'enc4', ((16, 80, 16, 16, 16),), 'f16', None),
    ('unet_eval_b16_f16', 'dec4', ((16, 80, 16, 16, 16), (16, 80, 16, 16, 16)), 'f16', (1, 80)),
    ('unet_eval_b16_f16', 'enc5', ((16, 160, 8, 8, 8),), 'f16', None),
    ('unet_eval_b16_f16', 'dec3', ((16, 160, 8, 8, 8), (16, 160, 8, 8, 8)), 'f16', None),
    ('unet_eval_b16_f16', 'enc6', ((16, 320, 4, 4, 4),), 'f16', None),
    ('unet_eval_b16_f16', 'dec2', ((16, 320, 4, 4, 4), (16, 320, 4, 4, 4)), 'f16', None),
    ('unet_train_b4', 'enc2', ((4, 20, 64, 64, 64),), 'f16x2', None),
    ('unet_train_b4', 'dec6', ((4, 20, 64, 64, 64), (4, 20, 64, 64, 64)), 'f16x2', None),
    ('unet_train_b4', 'enc3', ((4, 40, 32, 32, 32),), 'f16x2', None),
    ('unet_train_b4', 'dec5', ((4, 40, 32, 32, 32), (4, 40, 32, 32, 32)), 'f16x2', None),
    ('unet_train_b4', 'enc4', ((4, 80, 16, 16, 16),), 'f16x2', None),
    ('unet_train_b4', 'dec4', ((4, 80, 16, 16, 16), (4, 80, 16, 16, 16)), 'f16x2', None),
    ('unet_train_b4', 'enc5', ((4, 160, 8, 8, 8),), 'f16x2', None),
    ('unet_train_b4', 'dec3', ((4, 160, 8, 8, 8), (4, 160, 8, 8, 8)), 'f16x2', None),
    ('unet_train_b4', 'enc6', ((4, 320, 4, 4, 4),), 'f16x2', None),
    ('unet_train_b4', 'dec2', ((4, 320, 4, 4, 4), (4, 320, 4, 4, 4)), 'f16x2', None),
]
_NETS = {"unet": nets.Unet_3D, "vdec": nets.VoxelDecoder, "vgen": lambda: nets.VoxelGenerator(res=128),
         "vdis": lambda: nets.VoxelDiscriminator(res=128)}


def _net(run):
    with torch.device("meta"):
        return _NETS[run.split("_")[0]]()


@pytest.mark.parametrize("run", sorted({r[0] for r in LAYERS}))
def test_layer_routes_reproduce_the_recorded_entry_points(run):
    mods = dict(_net(run).named_modules())
    for _, fn, layer, srcs, bn, act, grad, mode, entries in (r for r in LAYERS if r[0] == run):
        m = mods[layer]
        with ops_conv.precision(mode):
            if fn.endswith(".backward"):
                gy, x = srcs
                if fn == "_ConvInputGrad.backward":      # the grad-of-grad convolution: conv3d(ggx, m) in TF32 or better
                    with ops_conv._forced_mode("tf32"):
                        got = _route(m, [(gy, "plain")])
                    assert len(entries) == 1 and got == route_of(entries[0], m), (layer, got, entries)
                    continue
                dx, dw = bn
                wgrad = dw and not grad and ops_conv._k8_wgrad_supported(x, m)
                dgrad = dx and not grad and ops_conv.TC_BACKWARD and ops_conv._tc_dgrad_supported(gy, m)
                assert ("conv_k8s2_wgrad" in entries) == wgrad, (layer, entries)
                assert len(entries) - wgrad == dgrad, (layer, entries)
                continue
            got = _route(m, list(srcs), _bn(bn), act in ("slope", "ReLU", "LeakyReLU"), grad, act == "Sigmoid")
            if grad and got in ("train_forward", "convt_c1_train"):
                with torch.no_grad():                    # the custom forward of _ConvForward / _ConvTC1Train
                    inner = _route(m, list(srcs))
                got = "convt_c1" if got == "convt_c1_train" else inner
            if not entries:
                assert got is None, (run, layer, fn, got)
                continue
            assert len(entries) == 1 and got == route_of(entries[0], m), (run, layer, fn, got, entries)
            _check_form(entries[0], m, srcs[0][0])
            if entries[0].endswith("[operands]"):
                assert got in ("conv_k4s2", "conv_k8s2", "convt_k4", "convt_k8"), (layer, got)


@pytest.mark.parametrize("run", sorted({r[0] for r in LAYOUTS}))
def test_operand_layouts_reproduce_the_recorded_answers(run):
    net = _net(run).train(run.startswith("unet_train"))
    for _, block, shapes, mode, answer in (r for r in LAYOUTS if r[0] == run):
        with ops_conv.precision(mode), torch.set_grad_enabled(run.startswith("unet_train")):
            assert getattr(net, block).operand_layout(*shapes) == answer, (block, shapes)
