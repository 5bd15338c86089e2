"""networks/networks.py drop-in: state_dict layout, parameters under a fixed seed and forward outputs must equal the
reference's (digests recorded from the reference module by tests/golden/make_golden_networks.py)."""
import hashlib
import json
import os

import numpy as np
import pytest
import torch

import networks.networks as nets

G = json.load(open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "networks_digest.json")))


def build(name):
    case = G["cases"][name]
    torch.manual_seed(1234)
    net = getattr(nets, name.split("_res")[0])(**case["kwargs"])
    torch.manual_seed(99)
    shape = case["input_shape"]
    x = torch.rand(*shape) if "Discriminator" in name or name == "Unet_3D" else torch.randn(*shape)
    return case, net, x


def signature(t, n=64):
    flat = t.detach().reshape(-1).double().cpu()
    idx = torch.linspace(0, flat.numel() - 1, n).long()
    return float(flat.sum()), float(flat.abs().sum()), flat[idx].numpy()


@pytest.mark.parametrize("name", list(G["cases"]))
def test_state_dict_layout_and_seeded_parameters_match_reference(name):
    case, net, _ = build(name)
    sd = net.state_dict()
    assert [[k, list(v.shape)] for k, v in sd.items()] == case["state_dict"]
    h = hashlib.sha256()
    for k, v in sd.items():
        h.update(k.encode())
        h.update(np.ascontiguousarray(v.numpy()).tobytes())
    assert h.hexdigest() == case["params_sha256"], "same seed must give the reference's parameters (creation order)"
    assert sum(p.numel() for p in net.parameters()) == case["n_params"]


@pytest.mark.parametrize("name", ["VoxelDecoder", "VoxelGenerator_res64", "VoxelDiscriminator_res64", "VoxelDiscriminator"])
def test_forward_matches_reference_on_cpu(name):
    """torch path of the drop-in (the reference is pure torch.nn): eval and train mode signatures."""
    case, net, x = build(name)
    for mode in ("eval", "train"):
        getattr(net, mode)()
        with torch.no_grad():
            y = net(x)
        s, a, samples = signature(y)
        ref = case[mode]
        assert list(y.shape) == ref["shape"]
        np.testing.assert_allclose(samples, ref["samples"], rtol=2e-4, atol=2e-5 * max(1.0, ref["abs_sum"] / y.numel()))
        assert abs(a - ref["abs_sum"]) <= 1e-4 * max(1.0, ref["abs_sum"])


def test_helpers_and_import_surface():
    for name in ("Unet_3D", "VoxelGenerator", "VoxelDiscriminator", "ImageEncoder", "VoxelDecoder", "ViewAsLinear",
                 "Conv3d_block", "Deconv3d_skip", "conv3d_half", "deconv3d_2x", "conv3d_minus3", "deconv3d_add3",
                 "batchnorm3d", "batchnorm", "batchnorm1d", "fc", "relu", "relu_leaky", "maxpool", "dropout"):
        assert hasattr(nets, name), name
    assert nets.ViewAsLinear.forward(torch.zeros(3, 4, 5)).shape == (3, 20)
    assert nets.relu_leaky().negative_slope == 0.2
    with pytest.raises(NotImplementedError):
        nets.VoxelGenerator(res=32)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["Unet_3D", "VoxelDecoder", "VoxelGenerator", "VoxelDiscriminator"])
@pytest.mark.parametrize("mode", ["exact", "f16"])
def test_forward_matches_reference_on_gpu(name, mode):
    """CUDA path against the reference digests (recorded on CPU fp32).
    exact (the DEFAULT mode, under PyTorch's default allow_tf32 = True): the custom kernels run their fp32-accurate operand-split
          scheme and the layers without a custom kernel run ops_conv.exact_fallback's 3xTF32 split on cuDNN: whole-net outputs
          within 1e-4 (north_star) with the fp16 hi/lo split,
          3e-4 with the older 3xTF32 scheme (its accumulator truncation error grows with 3x the MMA steps);
    f16   (opt-in): single-pass fp16 operands, with the tolerance a 10-bit mantissa allows through a 12-layer network."""
    from genre_shapehd_b200 import ops_conv
    torch.backends.cudnn.allow_tf32 = True     # PyTorch's default: in the exact mode the layers left to cuDNN must still run fp32
    torch.backends.cuda.matmul.allow_tf32 = False
    try:
        case, net, x = build(name)
        net = net.cuda()
        x = x.cuda()
        with ops_conv.precision(mode):
            for phase in ("eval", "train"):
                getattr(net, phase)()
                with torch.no_grad():
                    y = net(x)
                s, a, samples = signature(y)
                ref = case[phase]
                assert list(y.shape) == ref["shape"]
                scale = max(1e-3, ref["abs_sum"] / y.numel())
                tol = 2e-2 if mode == "f16" else 1e-4 if ops_conv.EXACT_IMPL == "f16x2" else 3e-4
                np.testing.assert_allclose(samples, ref["samples"], rtol=tol, atol=tol * scale)
                assert abs(a - ref["abs_sum"]) <= tol * max(1.0, ref["abs_sum"])
    finally:
        torch.backends.cudnn.allow_tf32 = True
