"""The reference's CPU path of the GenRe forward (BASELINE configs[2]) — BASELINE INFRASTRUCTURE, see cpu_toolbox/README.md.

build_cpu_genre_net() returns the frozen models/genre_full_model.Net (the reference's file, from $GENRE_REF or
baseline/_ref) on CPU with
    toolbox.*            -> oracle/cpu_toolbox (the CUDA-only ops restated on the CPU oracle, maps in parallel)
    networks.*           -> the reference's own networks/networks.py, uresnet.py, revresnet.py on torch CPU
Must run in a process that never called genre_shapehd_b200.install() (bench.py --impl reference is such a process).
"""
import argparse
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(HERE)


def build_cpu_genre_net(ref_root=None):
    import torch
    for name in ("toolbox", "networks", "nndistance"):
        if name in sys.modules:
            raise RuntimeError("%s is already imported (from %s): the CPU reference path needs its own process"
                               % (name, getattr(sys.modules[name], "__file__", "?")))
    if REPO not in sys.path:
        sys.path.insert(0, REPO)
    from genre_shapehd_b200 import compat
    from genre_shapehd_b200.synth_genre import init_genre_net_for_bench
    ref_root = ref_root or compat.find_reference()
    if ref_root is None:
        raise FileNotFoundError("no staged reference callers (baseline/_ref): run __graft_entry__.build() where a reference checkout is found")
    sys.path.insert(0, ref_root)                                    # models, util, networks (the reference's own, CPU torch)
    sys.path.insert(0, os.path.join(HERE, "cpu_toolbox"))           # toolbox -> CPU oracle stand-ins
    compat.stub_optional_modules()
    import models.genre_full_model as gfm
    import toolbox
    assert os.path.abspath(toolbox.__file__).startswith(os.path.join(HERE, "cpu_toolbox"))
    assert os.path.abspath(gfm.Unet_3D.__module__ and sys.modules[gfm.Unet_3D.__module__].__file__).startswith(os.path.abspath(ref_root))
    opt = argparse.Namespace(joint_train=False, padding_margin=16, inpaint_path=None, pred_depth_minmax=True,
                             net1_path=None, load_offline=False)
    torch.manual_seed(0)
    net = gfm.Net(opt, gfm.Model)
    init_genre_net_for_bench(net)
    return net.eval()
