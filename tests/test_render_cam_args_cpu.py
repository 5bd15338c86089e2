"""The camera renderer's entry points reject every unsupported size, null and misaligned pointer before launching (fake
device addresses, never dereferenced), and the Python functions refuse CPU and non-fp32 tensors."""
import ctypes

import pytest
import torch

from genre_shapehd_b200 import _lib, postprocess


def _d(v=4096):
    return ctypes.c_void_p(v)


def _render(L, vox=_d(), N=1, R=16, H=8, W=8, Z=16, fl=_d(), cd=_d(), out=_d()):
    return L.genre_b200_render_camera_forward(vox, N, R, H, W, Z, fl, 0, cd, 0, 0.0, out, _d(), None)


def _loss_bwd(L, obs=_d(), g=_d(), gv=_d(), Z=16):
    return L.genre_b200_ray_consistency_backward(_d(), 1, 16, 8, 8, Z, _d(), 0, _d(), 0, obs, 64, 8, 1, 1.0, g, gv, None)


@pytest.mark.parametrize("call,code,needle", [
    (lambda L: _render(L, vox=None), -1, b"null"),
    (lambda L: _render(L, out=None), -1, b"null"),
    (lambda L: _render(L, R=1), -1, b"resolution"),
    (lambda L: _render(L, R=1025), -1, b"resolution"),
    (lambda L: _render(L, H=0), -1, b"image size"),
    (lambda L: _render(L, W=16385), -1, b"image size"),
    (lambda L: _render(L, Z=0), -1, b"z_res"),
    (lambda L: _render(L, Z=4097), -1, b"z_res"),
    (lambda L: _render(L, N=0), -1, b"batch"),
    (lambda L: _render(L, N=1 << 40), -1, b"batch"),
    (lambda L: _render(L, vox=_d(4098)), -3, b"aligned"),
    (lambda L: _render(L, out=_d(4097)), -3, b"aligned"),
    (lambda L: L.genre_b200_render_camera_backward(_d(), 1, 16, 8, 8, 16, _d(), 0, _d(), 0, 0.0, _d(), None, _d(), None),
     -1, b"null"),
    (lambda L: L.genre_b200_ray_consistency_forward(_d(), 1, 16, 8, 8, 16, _d(), 0, _d(), 0, None, 64, 8, 1, 1.0, _d(), None),
     -1, b"null"),
    (lambda L: _loss_bwd(L, obs=_d(4099)), -3, b"aligned"),
    (lambda L: _loss_bwd(L, gv=None), -1, b"null"),
    (lambda L: _loss_bwd(L, Z=5000), -1, b"z_res"),
])
def test_entry_points_validate_before_launching(call, code, needle):
    lib = _lib.load()
    rc = call(lib)
    msg = lib.genre_b200_last_error()
    assert rc == code, (rc, msg)
    assert needle.lower() in msg.lower(), msg


def test_python_layer_refuses_cpu_and_non_fp32():
    with pytest.raises(RuntimeError):
        postprocess.render_depth(torch.zeros(1, 1, 8, 8, 8))
    with pytest.raises(RuntimeError):
        postprocess.ray_consistency_loss(torch.zeros(1, 1, 8, 8, 8), torch.zeros(1, 1, 4, 4))


def test_default_z_res():
    assert postprocess.default_z_res(128) == 445
    assert postprocess.default_z_res(2) == 8
