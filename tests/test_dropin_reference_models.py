"""The reference's FROZEN model files import, build and RUN on top of this package's toolbox / nndistance / networks.

The frozen callers come from $GENRE_REF, else <repo>/baseline/_ref (an unmodified copy staged by
__graft_entry__.build() from a checkout; git-ignored).  Without one these tests skip: the reference's model files
are not part of this repository.  The GPU tests (``-m gpu``) run ``Net.forward`` of models/genre_full_model.py:116-132 (BASELINE configs[2]) and one training
step of models/shapehd.py:113-118 on CUDA and check every hot-path tensor against the CPU oracle / torch fp32.
"""
import argparse
import os
import sys
import types

import numpy as np
import pytest
import torch

from genre_shapehd_b200 import compat

REF = compat.find_reference()
needs_ref = pytest.mark.skipif(REF is None, reason="no reference checkout and no staged baseline/_ref")


@pytest.fixture(scope="module")
def ref_root():
    from conftest import REPO
    if REF is None:
        pytest.skip("no reference checkout")
    root = compat.bootstrap(REF)
    yield root, REPO


def _mine(obj, repo):
    mod = sys.modules[obj.__module__]
    return os.path.abspath(mod.__file__).startswith(os.path.join(repo, "genre_shapehd_b200"))


def genre_opt(joint_train=False):
    return argparse.Namespace(joint_train=joint_train, padding_margin=16, inpaint_path=None, pred_depth_minmax=True,
                              net1_path=None, load_offline=False)


@needs_ref
def test_frozen_models_import_on_top_of_this_package(ref_root):
    root, repo = ref_root
    import models.genre_full_model as gfm
    import models.shapehd as shd
    import models.wgangp as wg
    import models.marrnet2 as m2
    import models.depth_pred_with_sph_inpaint as dpi
    assert os.path.abspath(gfm.__file__).startswith(os.path.abspath(root))   # the caller is the reference's file, unchanged
    assert _mine(gfm.Camera_back_projection_layer, repo)
    assert _mine(gfm.SphericalBackProjection, repo)
    assert _mine(gfm.Unet_3D, repo)
    assert gfm.gen_sph_grid.__module__ == "toolbox.spherical_proj" and _mine(gfm.gen_sph_grid, repo)
    assert _mine(dpi.render_spherical, repo)
    assert _mine(wg.VoxelGenerator, repo) and _mine(wg.VoxelDiscriminator, repo)
    assert _mine(m2.VoxelDecoder, repo)
    assert shd is not None


@needs_ref
def test_staged_callers_are_unmodified_copies(ref_root):
    """baseline/_ref holds byte-identical copies of the reference files (checked where both trees exist)."""
    root, repo = ref_root
    staged = os.path.join(repo, "baseline", "_ref")
    import __graft_entry__
    checkout = __graft_entry__.REFERENCE        # the checkout build() stages from
    if not (checkout and os.path.isdir(os.path.join(staged, "models"))):
        pytest.skip("needs both a reference checkout and the staged copy")
    for rel in ("models/genre_full_model.py", "models/depth_pred_with_sph_inpaint.py", "models/shapehd.py", "models/wgangp.py",
                "models/netinterface.py", "networks/uresnet.py", "networks/revresnet.py", "util/util_sph.py"):
        assert open(os.path.join(staged, rel), "rb").read() == open(os.path.join(checkout, rel), "rb").read(), rel


@needs_ref
def test_genre_net_builds_with_reference_constructor(ref_root):
    root, repo = ref_root
    import models.genre_full_model as gfm
    net = gfm.Net(genre_opt(), gfm.Model)
    assert _mine(net.refine_net, repo) and _mine(net.proj_depth, repo)
    keys = list(net.state_dict().keys())
    assert "grid" in keys and any(k.startswith("refine_net.enc1.net.0.") for k in keys)
    assert any(k.startswith("depth_and_inpaint.render_spherical.") or "depth_weight" in k for k in keys)


@needs_ref
def test_fold_batchnorm2d_eval_keeps_the_2d_nets_outputs(ref_root):
    """compat.fold_batchnorm2d_eval (the 2D nets' cheap win used by bench.py): every BatchNorm2d of the reference's U-ResNets
    disappears into its convolution and the outputs move only at rounding level"""
    import models.genre_full_model as gfm
    from genre_shapehd_b200.synth_genre import init_genre_net_for_bench
    torch.manual_seed(0)
    net = gfm.Net(genre_opt(), gfm.Model)
    init_genre_net_for_bench(net)
    net.eval()
    dn = net.depth_and_inpaint
    x = types.SimpleNamespace(rgb=torch.randn(1, 3, 256, 256))      # the min/max head needs the 8x8 encoder output of a 256^2 image
    s = torch.rand(1, 1, 160, 160)
    with torch.no_grad():
        a1, a2 = dn.net1(x), dn.net2(s)
        n = compat.fold_batchnorm2d_eval(dn.net1) + compat.fold_batchnorm2d_eval(dn.net2)
        b1, b2 = dn.net1(x), dn.net2(s)
    assert n == 124 and not any(isinstance(m, torch.nn.BatchNorm2d) for m in list(dn.net1.modules()) + list(dn.net2.modules()))
    for a, b in ((a1, b1), (a2, b2)):
        for k in a:
            assert (a[k] - b[k]).abs().max().item() <= 1e-5 * max(1.0, a[k].abs().max().item()), k
    assert compat.fold_batchnorm2d_eval(dn.net1) == 0            # idempotent


# ---- on the GPU: the frozen callers RUN on the drop-in -----------------------------------------------------------------
def genre_inputs(batch, device, seed=0):
    """C3 inputs (SURVEY 8d): rgb ~ N(0,1), silhou = 100 * disc mask (scale_25d, marrnetbase.py:17)"""
    g = torch.Generator().manual_seed(seed)
    rgb = torch.randn(batch, 3, 256, 256, generator=g)
    yy, xx = torch.meshgrid(torch.arange(256.0), torch.arange(256.0), indexing="ij")
    sil = torch.stack([(((yy - 127.5) ** 2 + (xx - 127.5) ** 2) < (70.0 + 6 * i) ** 2).float() for i in range(batch)])[:, None] * 100
    return types.SimpleNamespace(rgb=rgb.to(device), silhou=sil.to(device))


@pytest.mark.gpu
def test_genre_full_model_forward_runs_on_cuda_and_matches_the_oracle(ref_root, oracle):
    """models/genre_full_model.py:116-132 Net.forward, B=2, eval, random init, on CUDA through the drop-in ops; every
    hot-path tensor it returns is recomputed from ITS OWN inputs by the CPU oracle (toolbox ops) / fp32 cuDNN (Unet_3D)."""
    import models.genre_full_model as gfm
    from genre_shapehd_b200 import _lib, ops_conv
    from genre_shapehd_b200.synth_genre import init_genre_net_for_bench
    torch.manual_seed(0)
    dev = torch.device("cuda:0")
    net = gfm.Net(genre_opt(), gfm.Model)
    init_genre_net_for_bench(net)
    net = net.to(dev).eval()
    captured = {}
    net.depth_and_inpaint.proj_depth.register_forward_pre_hook(lambda m, a: captured.__setitem__("depth", a[0].detach().clone()))
    n0 = _lib.launch_count
    tf32 = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = False          # fp32 semantics of the reference: the conv kernels run their fp32-accurate mode
    try:
        with torch.no_grad():
            out = net(genre_inputs(2, dev))
            torch.cuda.synchronize()
            assert _lib.launch_count - n0 >= 10, "the frozen Net did not run on this library's kernels"
            depth = captured["depth"]
            assert depth.shape == (2, 1, 256, 256) and not depth.is_contiguous()     # permuted + flipped view (depth_pred...:140-141)
            # cam_bp (a1, a3)
            tdf_o, cnt_o = oracle.cam_bp_forward(depth.cpu().numpy(), 418.3, 2.2, 128, shift=True)
            assert (cnt_o > 0).sum() > 2000, "the synthetic depth must hit the voxel grid (bench init of the minmax head)"
            proj = (out["proj_depth"] / 50).cpu().numpy()
            assert np.array_equal(proj != 0, cnt_o > 0)
            assert np.abs(proj - tdf_o).max() < 1e-5
            # render_spherical + sph_pad (a9, a10), full size, against the independent oracle
            rs = net.depth_and_inpaint.render_spherical
            vox = np.clip(tdf_o * np.float32(50), np.float32(1e-5), np.float32(1 - 1e-5))
            sph_o = oracle.render_spherical(vox, rs.grid.cpu().numpy(), rs.depth_weight.cpu().numpy())
            from toolbox.spherical_proj import sph_pad
            sph_o = sph_pad(torch.from_numpy(sph_o), 16).numpy()
            assert np.abs(out["pred_sph_partial"].cpu().numpy() - sph_o).max() < 1e-4
            # spherical back-projection glue (a4, a6)
            full = out["pred_sph_full"]
            crop = (1 - full[:, :, 16:144, 16:144]).cpu().numpy()
            from toolbox.spherical_proj import gen_sph_grid
            tdf_s, cnt_s = oracle.sph_bp_forward(crop, gen_sph_grid().numpy()[0], 128)
            want = (-tdf_s + np.float32(1 / 128)) * np.float32(128) * np.clip(cnt_s, 0, 1)
            got = out["pred_proj_sph_full"].cpu().numpy()
            assert np.array_equal(got != 0, want != 0) or np.abs(got - want).max() < 1e-4
            assert np.abs(got - want).max() < 1e-4
            # Unet_3D (a12): same module, same input, custom kernels off -> cuDNN fp32
            refine_in = torch.cat((out["pred_proj_sph_full"], out["pred_proj_depth"]), dim=1)
            enabled = ops_conv.ENABLED
            ops_conv.ENABLED = False
            try:
                ref = net.refine_net(refine_in)
            finally:
                ops_conv.ENABLED = enabled
            pv = out["pred_voxel"]
            assert pv.shape == (2, 1, 128, 128, 128) and torch.isfinite(pv).all()
            err = (pv - ref).abs().max().item()
            assert err <= 1e-4 * max(1.0, ref.abs().max().item()), "Unet_3D logits differ from cuDNN fp32 by %g" % err
            occ = (torch.sigmoid(pv) - torch.sigmoid(ref)).abs().max().item()
            assert occ <= 1e-4, "occupancies differ by %g" % occ
    finally:
        torch.backends.cudnn.allow_tf32 = tf32


@pytest.mark.gpu
def test_shapehd_training_step_runs_on_cuda(ref_root):
    """models/shapehd.py:113-118 Net.forward + the loss of :67-79 + backward + Adam step (BASELINE configs[3], B=2), on CUDA
    through the drop-in 3D nets; loss and the decoder's gradients are compared with the same step on cuDNN fp32."""
    import models.shapehd as shd
    from genre_shapehd_b200 import ops_conv
    dev = torch.device("cuda:0")
    torch.manual_seed(1)
    net = shd.Net().to(dev)
    net.train()
    g = torch.Generator().manual_seed(2)
    B = 2

    def batch():
        sil = (torch.rand(B, 1, 256, 256, generator=g) > 0.4).float()
        return types.SimpleNamespace(depth=torch.rand(B, 1, 256, 256, generator=g).to(dev), normal=torch.rand(B, 3, 256, 256, generator=g).to(dev),
                                     silhou=sil.to(dev))
    gt = (torch.rand(B, 1, 128, 128, 128, generator=g) < 0.05).float().to(dev)
    crit = torch.nn.BCEWithLogitsLoss()
    state = {k: v.clone() for k, v in net.state_dict().items()}
    inp = batch()

    def step(custom):
        net.load_state_dict(state)
        enabled = ops_conv.ENABLED
        ops_conv.ENABLED = custom
        tf32 = torch.backends.cudnn.allow_tf32
        torch.backends.cudnn.allow_tf32 = False
        try:
            opt = torch.optim.Adam(net.marrnet2.parameters(), lr=1e-3)
            opt.zero_grad()
            x = types.SimpleNamespace(depth=inp.depth.clone(), normal=inp.normal.clone(), silhou=inp.silhou.clone())
            pred = net(x)
            loss = crit(pred["voxel"], gt) + 1e-3 * (-pred["is_real"].mean())
            loss.backward()
            grads = {n: p.grad.detach().clone() for n, p in net.marrnet2.decoder.named_parameters() if p.grad is not None}
            opt.step()
            torch.cuda.synchronize()
            return loss.item(), grads
        finally:
            ops_conv.ENABLED = enabled
            torch.backends.cudnn.allow_tf32 = tf32
    loss_c, g_c = step(True)
    loss_r, g_r = step(False)
    assert np.isfinite(loss_c) and abs(loss_c - loss_r) <= 1e-4 * max(1.0, abs(loss_r))
    assert g_c.keys() == g_r.keys() and len(g_c) >= 10
    overall = max(v.abs().max().item() for v in g_r.values())
    for name in g_c:
        scale = g_r[name].abs().max().item()
        # two fp32 implementations with different summation orders, through training-mode BatchNorm at batch 2 and the BCE's
        # cancellation: weight gradients agree to a few 1e-3 of their scale.  The bias of a convolution that feeds a
        # training-mode BatchNorm has an exactly-zero gradient (the mean is subtracted): both sides hold rounding noise there,
        # hence the absolute floor.
        assert (g_c[name] - g_r[name]).abs().max().item() <= 1e-2 * scale + 1e-6 * overall, name
    for p in net.d.parameters():
        assert p.grad is None            # D stays frozen (shapehd.py:104-105)


@pytest.mark.gpu
def test_fused_batched_forward_equals_the_frozen_forward(ref_root):
    """genre_shapehd_b200.fused.genre_forward_fused (SURVEY 8f-1 / 8f-4: the batched, mesh-free stand-in for
    forward_with_trimesh) returns the tensors of the frozen Net.forward"""
    import models.genre_full_model as gfm
    from genre_shapehd_b200.fused import genre_forward_fused
    from genre_shapehd_b200.synth_genre import init_genre_net_for_bench
    torch.manual_seed(0)
    dev = torch.device("cuda:0")
    net = gfm.Net(genre_opt(), gfm.Model)
    init_genre_net_for_bench(net)
    net = net.to(dev).eval()
    x = genre_inputs(3, dev, seed=4)
    # The back-projections bin points into voxels: a 1e-7 change of a depth value can move a point across a voxel boundary.
    # cuDNN does not promise bitwise-identical results between two calls of the 2D nets, so both forwards are fed the SAME
    # 2D-net outputs (computed once, replayed): what is compared is the 3D path.
    dn = net.depth_and_inpaint
    cache = {}

    def replay(name, mod):
        orig = mod.forward

        def fwd(inp):
            if name not in cache:
                cache[name] = {k: v.clone() for k, v in orig(inp).items()}
            return {k: v.clone() for k, v in cache[name].items()}
        mod.forward = fwd
    replay("net1", dn.net1)
    replay("net2", dn.net2)
    with torch.no_grad():
        a = net(types.SimpleNamespace(rgb=x.rgb.clone(), silhou=x.silhou.clone()))
        b = genre_forward_fused(net, types.SimpleNamespace(rgb=x.rgb.clone(), silhou=x.silhou.clone()))
    for key in ("proj_depth", "pred_sph_partial", "pred_sph_full", "pred_proj_sph_full", "pred_proj_depth", "pred_voxel"):
        assert a[key].shape == b[key].shape, key
        scale = max(1.0, a[key].abs().max().item())
        assert (a[key] - b[key]).abs().max().item() <= 2e-4 * scale, key
    assert (a["pred_voxel"] - b["pred_voxel"]).abs().max().item() <= 1e-4 * max(1.0, a["pred_voxel"].abs().max().item())
