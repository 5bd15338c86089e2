"""Operand outputs on CPU: the address map of the convolution epilogue's fp16 operand destinations (csrc/convt3d.cu
store_operand), the routing decision that lets Unet_3D's layers write them (ops_conv.conv_operand_layout /
deconv_operand_layout), and the rule that an ops_conv.OperandActivation never reaches a layer that needs fp32."""
import pytest
import torch

from genre_shapehd_b200 import ops_conv
from genre_shapehd_b200.networks import networks as nets


def store_operand_index(layout, part, parts, ocg, k, b, oz, oy, ox, do, ho, wo):
    """csrc/convt3d.cu store_operand: 16-byte unit of channel group k, part `part` of output position (b, oz, oy, ox)"""
    if layout == ops_conv.PLAIN:
        return ((b * do + oz) * parts * ocg + k) * ho * wo + oy * wo + ox + part * ocg * ho * wo
    h2, w2 = ho // 2, wo // 2
    s = ((oz & 1) * 2 + (oy & 1)) * 2 + (ox & 1)
    return (((b * (do // 2) + oz // 2) * parts * 8 + s) * ocg + k) * h2 * w2 + (oy // 2) * w2 + ox // 2 + part * 8 * ocg * h2 * w2


def _epilogue_image(x, layout, cpad, parts):
    """what the epilogue writes for the NCDHW values x: unit index -> the 8 channel values of group k (zero padded); the
    lo' part is filled with a marker so that a part mix-up shows"""
    b, c, d, h, w = x.shape
    ocg = cpad // 8
    xp = torch.nn.functional.pad(x, (0, 0, 0, 0, 0, 0, 0, cpad - c))
    units = b * d * h * w * ocg * parts
    img = torch.full((units, 8), float("nan"))
    for bb in range(b):
        for z in range(d):
            for y in range(h):
                for xx in range(w):
                    for k in range(ocg):
                        for part in range(parts):
                            u = store_operand_index(layout, part, parts, ocg, k, bb, z, y, xx, d, h, w)
                            assert torch.isnan(img[u]).all(), "two positions map to one unit"
                            img[u] = xp[bb, 8 * k:8 * k + 8, z, y, xx] if part == 0 else -1.0
    assert not torch.isnan(img).any(), "a unit of the destination is never written"
    return img


@pytest.mark.parametrize("c,cpad", [(20, 32), (40, 48), (8, 8)])
def test_parity_destination_map_is_the_space_to_depth_sources_layout(c, cpad):
    x = torch.randn(2, c, 4, 6, 4)
    for parts in (1, 2):
        img = _epilogue_image(x, ops_conv.PARITY, cpad, parts)
        ref = ops_conv.space_to_depth_sources(x, cpad, 8, None)          # [B*D/2, 8*cpad/8, H/2, W/2, 8], part 0 only
        hi = img.view(2 * 2, parts, 8 * (cpad // 8), 3, 2, 8)[:, 0]
        assert torch.equal(hi, ref)


@pytest.mark.parametrize("c,cpad", [(20, 24), (40, 40)])
def test_plain_destination_map_is_the_blocked_layout(c, cpad):
    x = torch.randn(2, c, 3, 4, 5)
    xp = torch.nn.functional.pad(x, (0, 0, 0, 0, 0, 0, 0, cpad - c))
    for parts in (1, 2):
        img = _epilogue_image(x, ops_conv.PLAIN, cpad, parts)
        hi = img.view(2 * 3, parts, cpad // 8, 4, 5, 8)[:, 0]
        assert torch.equal(hi, ops_conv.to_blocked(xp, 8))


def _unet_layouts(net, b=2):
    """(consumer -> layout) at Unet_3D's 128^3 shapes, as Unet_3D.forward asks"""
    s = lambda c, r: torch.Size((b, c, r, r, r))
    return {"enc2": net.enc2.operand_layout(s(20, 64)), "enc3": net.enc3.operand_layout(s(40, 32)),
            "enc4": net.enc4.operand_layout(s(80, 16)), "dec4": net.dec4.operand_layout(s(80, 16), s(80, 16)),
            "dec5": net.dec5.operand_layout(s(40, 32), s(40, 32)), "dec6": net.dec6.operand_layout(s(20, 64), s(20, 64))}


def test_unet_operand_layouts_follow_the_routing(monkeypatch):
    net = nets.Unet_3D().eval()
    with torch.no_grad(), ops_conv.precision("f16x2"):
        got = _unet_layouts(net)
    assert got == {"enc2": (ops_conv.PARITY, 32), "enc3": (ops_conv.PARITY, 48), "enc4": None,
                   "dec4": (ops_conv.PLAIN, 80), "dec5": (ops_conv.PLAIN, 40), "dec6": (ops_conv.PLAIN, 24)}
    with torch.no_grad(), ops_conv.precision("f16"):
        assert _unet_layouts(net) == got
    # fp32 wanted: the fp32-accurate 3xTF32 and the TF32 modes, autograd, batch statistics, a layer off its kernel
    for mode in ("fp32x3", "tf32"):
        with torch.no_grad(), ops_conv.precision(mode):
            assert set(_unet_layouts(net).values()) == {None}
    with ops_conv.precision("f16x2"):
        assert set(_unet_layouts(net).values()) == {None}              # grad enabled, parameters require it
    net.train()
    with torch.no_grad(), ops_conv.precision("f16x2"):
        assert _unet_layouts(net)["enc2"] is None and _unet_layouts(net)["dec5"] is None
    net.eval()
    monkeypatch.setattr(ops_conv, "POLICY", ops_conv.POLICY - {"conv_k4s2", "convt_c1_col2im"})
    with torch.no_grad(), ops_conv.precision("f16x2"):
        got = _unet_layouts(net)
    assert got["enc2"] is None and got["enc3"] is None and got["dec6"] is None and got["dec5"] == (ops_conv.PLAIN, 40)


def test_operand_activation_is_refused_where_fp32_is_needed():
    act = ops_conv.OperandActivation((2, 20, 4, 4, 4))
    act.operands[ops_conv.PLAIN] = (torch.zeros(1), 24)
    assert tuple(act.shape) == (2, 20, 4, 4, 4) and act.dim() == 5 and act.size(1) == 20 and not act.requires_grad
    assert act.operand(ops_conv.PLAIN, 24)[1] == 24
    with pytest.raises(RuntimeError, match="fp32"):
        act.operand(ops_conv.PARITY)
    with pytest.raises(RuntimeError, match="another operand"):
        act.operand(ops_conv.PLAIN, 32)
    with pytest.raises(RuntimeError, match="fp32"):
        ops_conv._blocked_f32(act)
    with pytest.raises(RuntimeError):
        with ops_conv.precision("fp32x3" if act.mode != "fp32x3" else "f16"):   # written in another mode: refused too
            act.operand(ops_conv.PLAIN)


def _d(v=4096):
    """a fake, 16-byte aligned device address: argument checks come before any launch and never dereference it"""
    import ctypes
    return ctypes.c_void_p(v)


@pytest.mark.parametrize("call,code,needle", [
    (lambda L: L.genre_b200_convt3d_s2_forward(_d(), 2, None, 0, 1, 2, 16, 16, _d(), 4, 32, 0, _d(), _d(), 1.0, None, 5,
                                               _d(), 1, 24, None, 0, 0, None), -1, b"fp16"),
    (lambda L: L.genre_b200_convt3d_s2_forward(_d(), 2, None, 0, 1, 2, 16, 16, _d(), 4, 32, 2, _d(), _d(), 1.0, None, 5,
                                               None, 1, 24, None, 0, 0, None), -1, b"null"),
    (lambda L: L.genre_b200_convt3d_s2_forward(_d(), 2, None, 0, 1, 2, 16, 16, _d(), 4, 32, 2, _d(), _d(), 1.0, _d(), 5,
                                               _d(), 1, 24, None, 0, 0, None), -1, b"both"),
    (lambda L: L.genre_b200_convt3d_s2_merged_forward(_d(), 2, None, 0, 1, 2, 16, 16, _d(), 8, 80, 2, 1, _d(), _d(), 1.0, None,
                                                      5, _d(), 3, 24, None, 0, 0, None), -1, b"layout"),
    (lambda L: L.genre_b200_convt3d_s2_merged_forward(_d(), 2, None, 0, 1, 2, 16, 16, _d(), 8, 80, 2, 1, _d(), _d(), 1.0, None,
                                                      5, None, 0, 0, None, 0, 0, None), -1, b"first operand destination"),
    (lambda L: L.genre_b200_conv3d_k8s2_s4d_forward(_d(), 2, 1, 2, 16, 16, _d(), 80, 2, _d(), _d(), 1.0, None, 5,
                                                    _d(), 2, 32, _d(), 1, 16, None), -1, b"cpad"),
    (lambda L: L.genre_b200_conv3d_k8s2_s4d_forward(_d(), 2, 1, 2, 16, 16, _d(), 80, 2, _d(), _d(), 1.0, _d(), 5,
                                                    _d(), 2, 32, None, 0, 0, None), -1, b"both"),
    (lambda L: L.genre_b200_conv3d_k4s2_forward(_d(), 2, 1, 1, 2, 16, 16, _d(), 64, 2, _d(), _d(), 1.0, None, 10,
                                                _d(), 2, 48, _d(4104), 1, 40, None), -3, b"aligned"),
    (lambda L: L.genre_b200_conv3d_k4s2_forward(_d(), 2, 1, 1, 2, 16, 16, _d(), 64, 2, _d(), _d(), 1.0, None, 10,
                                                None, 0, 0, None, 0, 0, None), -1, b"first operand destination"),
])
def test_operand_outputs_validate_before_launching(call, code, needle):
    from genre_shapehd_b200 import _lib
    lib = _lib.load()
    rc = call(lib)
    msg = lib.genre_b200_last_error()
    assert rc == code, (rc, msg)
    assert needle.lower() in msg.lower(), msg
