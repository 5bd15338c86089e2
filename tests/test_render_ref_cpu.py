"""CPU checks of tests/render_ref.py: the fp64 renderer against the CPU oracle and the fp64 torch composition, its backward
against gradcheck and autograd, the per-voxel bounds against a brute-force loop, the negative controls' distance from
the reference, and the stop-probability reference against the oracle."""
import math

import numpy as np
import pytest
import torch

import render_ref as RR
from toolbox.spherical_proj import render_spherical


def _vol(n, res, seed, lo=0.0, hi=1.0, sparse=None):
    g = torch.Generator().manual_seed(seed)
    v = torch.rand(n, 1, res, res, res, generator=g) * (hi - lo) + lo
    if sparse is not None:
        v = torch.where(torch.rand(v.shape, generator=g) < sparse, v, torch.full_like(v, RR.PMIN))
    return v


def test_taps_are_the_kernels_order_and_sum_to_one():
    f = torch.tensor([[1.25, 2.5, 0.75], [-0.5, 3.0, 3.5], [4.0, 4.0, 4.0]], dtype=torch.float32)
    idx, w, valid = RR.taps64(f, 5)
    assert torch.allclose(w[0].sum(), torch.tensor(1.0, dtype=torch.float64))
    # tap 0 is (x0, y0, z0), tap 1 is z0 + 1, tap 4 is x0 + 1
    assert idx[0, 0].item() == (1 * 5 + 2) * 5 + 0 and idx[0, 1].item() == idx[0, 0].item() + 1
    assert idx[0, 4].item() == idx[0, 0].item() + 25
    assert abs(w[0, 0].item() - 0.75 * 0.5 * 0.25) < 1e-15
    assert not valid[1, 0] and valid[1, 4]           # x0 = -1 is outside, x0 + 1 = 0 inside
    assert valid[2].sum().item() == 1 and w[2, 0].item() == 1.0   # on the last grid point: one tap, weight 1


@pytest.mark.parametrize("res,s,z", [(8, 6, 20), (12, 5, 37), (9, 4, 1), (10, 7, 2)])
def test_forward_vs_oracle_and_fp64_composition(oracle, res, s, z):
    m = render_spherical(sph_res=s, z_res=z)
    vox = _vol(2, res, res + z, sparse=0.5)
    ref = RR.render64(vox, m.grid, m.depth_weight)
    o = torch.from_numpy(oracle.render_spherical(vox.numpy(), m.grid.numpy(), m.depth_weight.numpy()))
    # the oracle is fp32 with the kernel's trilinear expression and a sequential product: within the plain kernel's rule
    assert RR.bound_ratio(o, ref["out"], RR.fwd_bound(ref, RR.kappa_plain(z))) <= 1.0
    comp = RR.composition64(vox, m.grid, m.depth_weight)
    assert (comp - ref["out"]).abs().max().item() <= 1e-14


def test_forward_pre_transform_is_applied_in_fp32_before_sampling():
    m = render_spherical(sph_res=5, z_res=30)
    raw = _vol(1, 8, 3, 0.0, 0.03)
    pre = (50.0, 1e-5, 1 - 1e-5)
    a = RR.render64(raw, m.grid, m.depth_weight, pre=pre)["out"]
    b = RR.render64(torch.clamp(raw * 50, 1e-5, 1 - 1e-5), m.grid, m.depth_weight)["out"]
    assert torch.equal(a, b)


class _Render64(torch.autograd.Function):
    @staticmethod
    def forward(ctx, vox, grid, dw, g):
        ctx.save_for_backward(vox, grid, dw)
        return RR.render64(vox, grid, dw)["out"]

    @staticmethod
    def backward(ctx, gout):
        vox, grid, dw = ctx.saved_tensors
        r = RR.render64(vox, grid, dw, g=gout.contiguous())
        assert r["amb"].abs().max().item() == 0.0
        return r["grad"], None, None, None


def test_backward_vs_gradcheck_at_a_tiny_size():
    m = render_spherical(sph_res=3, z_res=12)
    vox = _vol(1, 5, 1, 0.05, 0.9).double().requires_grad_(True)
    assert torch.autograd.gradcheck(lambda v: _Render64.apply(v, m.grid, m.depth_weight, None), (vox,), eps=1e-6,
                                    atol=1e-8, rtol=1e-6)


@pytest.mark.parametrize("z", [40, 33])
def test_backward_vs_autograd_of_the_fp64_composition(z):
    m = render_spherical(sph_res=8, z_res=z)
    vox = _vol(2, 10, z, 0.02, 0.95)
    vox[:, :, 3:6, 3:6, 3:6] = 0.97
    g = torch.randn(2, 1, 8, 8, generator=torch.Generator().manual_seed(z), dtype=torch.float64)
    ref = RR.render64(vox, m.grid, m.depth_weight, g=g)
    assert ref["amb"].abs().max().item() == 0.0
    x = vox.double().requires_grad_(True)
    (RR.composition64(x, m.grid, m.depth_weight) * g).sum().backward()
    scale = x.grad.abs().max().item()
    assert (x.grad - ref["grad"]).abs().max().item() <= 1e-12 * scale


def test_bounds_and_term_counts_vs_a_brute_force_loop():
    """A_v, B_v, A_amb,v, F_v and n_v of render64 against scalar loops over rays, samples and taps"""
    res, s, z = 4, 3, 9
    m = render_spherical(sph_res=s, z_res=z)
    vox = _vol(1, res, 5, 0.0, 1.0)
    vox[0, 0, :2] = RR.PMIN             # exactly 1e-5: ambiguous samples
    vox[0, 0, 2, 2, 2] = 1.5            # clamped at the top
    g = torch.randn(1, 1, s, s, generator=torch.Generator().manual_seed(2), dtype=torch.float64)
    ref = RR.render64(vox, m.grid, m.depth_weight, g=g)
    v = vox.double()[0, 0]
    w = m.depth_weight.double()
    f = RR.coords32(m.grid, res).double()
    acc = {k: np.zeros((res, res, res)) for k in ("grad", "Av", "Bv", "amb", "floor", "n")}
    tol = RR.K_I * RR.U
    n_amb = 0
    for a in range(s):
        for b in range(s):
            gg = g[0, 0, a, b].item()
            taps, raw, I = [], [], []
            for k in range(z):
                x = f[a, b, k]
                x0 = [math.floor(c) for c in x.tolist()]
                fr = [c - c0 for c, c0 in zip(x.tolist(), x0)]
                tk, r, ii = [], 0.0, 0.0
                for cx in (0, 1):
                    for cy in (0, 1):
                        for cz in (0, 1):
                            pos = (x0[0] + cx, x0[1] + cy, x0[2] + cz)
                            wt = ((fr[0] if cx else 1 - fr[0]) * (fr[1] if cy else 1 - fr[1]) * (fr[2] if cz else 1 - fr[2]))
                            if all(0 <= q < res for q in pos):
                                tk.append((pos, wt))
                                r += v[pos].item() * wt
                                ii += abs(v[pos].item() * wt)
                taps.append(tk)
                raw.append(r)
                I.append(ii)
            p = [min(max(r, RR.PMIN), RR.PMAX) for r in raw]
            T = [1.0]
            for k in range(z):
                T.append(T[-1] * (1 - p[k]))
            TZ = T[z]
            s_ = [p[k] * T[k] for k in range(z)]
            amb = [abs(raw[k] - RR.PMIN) <= tol * I[k] or abs(raw[k] - RR.PMAX) <= tol * I[k] for k in range(z)]
            mk = [RR.PMIN - tol * I[k] <= raw[k] <= RR.PMAX + tol * I[k] for k in range(z)]
            psi = max(I[k] * mk[k] / p[k] for k in range(z)) + 2 * sum(I[k] * mk[k] / (1 - p[k]) for k in range(z))
            for k in range(z):
                Ak = sum(w[j].item() * s_[j] for j in range(k + 1, z))
                D = T[k] * w[k].item() - (Ak + TZ) / (1 - p[k])
                dabs = abs(gg) * (T[k] * abs(w[k].item()) + (Ak + TZ) / (1 - p[k]))
                passing = not amb[k] and RR.PMIN <= raw[k] <= RR.PMAX
                n_amb += amb[k]
                for pos, wt in taps[k]:
                    if passing:
                        acc["grad"][pos] += gg * D * wt
                    if passing or amb[k]:
                        acc["Av"][pos] += dabs * wt
                        acc["Bv"][pos] += dabs * RR.K_I * psi * wt
                        acc["floor"][pos] += abs(gg) * (z + 8) * RR.TINY / (1 - p[k]) * wt
                        acc["n"][pos] += wt != 0
                    if amb[k]:
                        acc["amb"][pos] += abs(gg * D) * wt
    assert n_amb > 0
    for k, a in acc.items():
        np.testing.assert_allclose(ref[k][0, 0].numpy(), a, rtol=1e-12, atol=1e-300, err_msg=k)


def _controls_case():
    m = render_spherical(sph_res=16, z_res=64)
    vox = _vol(1, 16, 9, sparse=0.05)
    vox[0, 0, 5:10, 5:10, 5:10] = 0.6
    return m, vox


@pytest.mark.parametrize("control", RR.FWD_CONTROLS)
def test_forward_controls_are_far_outside_the_rule(control):
    m, vox = _controls_case()
    ref = RR.render64(vox, m.grid, m.depth_weight)
    brick = RR.occupied_brick(vox, m.grid)
    c = RR.render64(vox, m.grid, m.depth_weight, control=control, brick=brick)
    kappa = max(RR.kappa_plain(64), RR.kappa_skip(64))
    r = RR.bound_ratio(c["out"], ref["out"], RR.fwd_bound(ref, kappa, RR.skip_table_term(m.depth_weight, 64)))
    assert r > 10.0, (control, r)


@pytest.mark.parametrize("control", RR.BWD_CONTROLS)
def test_backward_controls_are_far_outside_the_rule(control):
    m, vox = _controls_case()
    vox[0, 0, 11:13, 11:13, 11:13] = 1.5        # clamped at the top
    g = torch.randn(1, 1, 16, 16, generator=torch.Generator().manual_seed(4), dtype=torch.float64)
    ref = RR.render64(vox, m.grid, m.depth_weight, g=g)
    c = RR.render64(vox, m.grid, m.depth_weight, g=g, control=control)
    r = RR.bound_ratio(c["grad"], ref["grad"], RR.bwd_bound(ref, RR.kappa_bwd(64)))
    assert r > 10.0, (control, r)


@pytest.mark.parametrize("shape", [(2, 1, 4, 4, 64), (1, 1, 3, 3, 37), (1, 1, 2, 2, 300)])
def test_calc_prob_reference_vs_oracle(oracle, shape):
    rng = np.random.RandomState(sum(shape))
    p = np.clip(rng.rand(*shape), 1e-5, 1 - 1e-5).astype(np.float32)
    p[0, 0, 0, 0, 3:12] = 1 - 1e-5
    g = rng.randn(*shape).astype(np.float32)
    z = shape[-1]
    ref = RR.calc_prob64(torch.from_numpy(p), torch.from_numpy(g))
    s_o = oracle.calc_prob_forward(p)
    assert RR.bound_ratio(torch.from_numpy(s_o), ref["s"], RR.U * RR.kappa_cp_fwd(z) * ref["A"] + ref["floor"]) <= 1.0
    # the oracle's backward takes the fp32 weighted stop probabilities, as the op does
    gr_o = torch.from_numpy(oracle.calc_prob_backward(p, s_o * g))
    assert RR.bound_ratio(gr_o, ref["grad"], RR.U * RR.kappa_cp_bwd(z) * ref["Ag"] + ref["floorg"]) <= 1.0
    for ctl, key in (("inclusive transmittance", "s"), ("suffix includes own term", "grad"), ("second term dropped", "grad")):
        c = RR.calc_prob64(torch.from_numpy(p), torch.from_numpy(g), control=ctl)
        A, fl, k = (ref["A"], ref["floor"], RR.kappa_cp_fwd(z)) if key == "s" else (ref["Ag"], ref["floorg"], RR.kappa_cp_bwd(z))
        assert RR.bound_ratio(c[key], ref[key], RR.U * k * A + fl) > 10.0, ctl
