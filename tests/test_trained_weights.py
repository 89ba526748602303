"""CPU: the trained-like parameters of scene.perturb_networks carry what the geometric init zeroes (Fourier columns,
weight-norm scales, hidden biases) while the SDF stays a surface that renders.  If one of these properties is lost the
kernel conformance tests on these weights (tests/test_gpu_networks.py) become vacuous again, so each is asserted."""
import numpy as np
import pytest
import torch

from oracle import port
from multiply_b200 import scene as S


@pytest.fixture(scope="module")
def trained():
    return S.make_scene(P=2, S=64, seed=42, weights="trained")


def _f64(sd):
    return {k: v.double() for k, v in sd.items()}


def _sdf_grad(sd, x, cond):
    x = x.detach().clone().requires_grad_(True)
    y = port.implicit_forward(sd, x, cond.double(), 6)
    return y[:, 0].detach(), torch.autograd.grad(y[:, 0].sum(), x)[0]


def _near_surface(person, sd, n=40000, band=0.03):
    """Canonical points near the body whose fp64 |sdf| < band."""
    g = torch.Generator().manual_seed(3)
    vc = person["verts_c"].double()
    x = vc[torch.randint(0, vc.shape[0], (n,), generator=g)] + 0.05 * torch.randn(n, 3, generator=g, dtype=torch.float64)
    sdf, _ = _sdf_grad(sd, x, person["cond"])
    return x[sdf.abs() < band]


def _without_fourier(sd):
    """The same effective weights with the Fourier columns of lin0 / lin4 zeroed (g rescaled so that the remaining
    columns keep their values)."""
    out = dict(sd)
    for l, cols in ((0, slice(3, 39)), (4, slice(-36, None))):
        v = sd[f"lin{l}.weight_v"].clone()
        v[:, cols] = 0
        out[f"lin{l}.weight_v"] = v
        out[f"lin{l}.weight_g"] = sd[f"lin{l}.weight_g"] * v.norm(dim=1, keepdim=True) / \
            sd[f"lin{l}.weight_v"].norm(dim=1, keepdim=True)
    return out


def test_deterministic(trained):
    again = S.make_scene(P=2, S=64, seed=42, weights="trained")
    for p in range(2):
        for k in ("implicit", "render"):
            for name, v in trained["persons"][p][k].items():
                assert torch.equal(v, again["persons"][p][k][name]), (p, k, name)
    for name, v in trained["bg_implicit"].items():
        assert torch.equal(v, again["bg_implicit"][name]), name


def test_weight_norm_scales(trained):
    """(a) g / ||v||_row differs from 1 by more than 0.2 on most rows of every weight-norm layer."""
    for person in trained["persons"]:
        for net in ("implicit", "render"):
            sd = person[net]
            r = torch.cat([sd[k].double()[:, 0] / sd[k.replace("weight_g", "weight_v")].double().norm(dim=1)
                           for k in sd if k.endswith(".weight_g")])
            frac = float(((r - 1).abs() > 0.2).double().mean())
            assert frac > 0.6, (net, frac)


def test_parameters_not_degenerate(trained):
    geo = S.make_scene(P=2, S=64, seed=42)
    for person, p0 in zip(trained["persons"], geo["persons"]):
        sd = person["implicit"]
        assert float(sd["lin0.weight_v"][:, 3:39].abs().min()) > 0
        assert float(sd["lin4.weight_v"][:, -36:].abs().min()) > 0
        for l in range(8):
            assert float(sd[f"lin{l}.bias"].abs().mean()) > 0.02, l
        assert float((sd["lin8.bias"][1:] - p0["implicit"]["lin8.bias"][1:]).abs().mean()) > 0.02
        assert not torch.equal(person["render"]["lin_pose.weight"], p0["render"]["lin_pose.weight"])
        assert not torch.equal(person["render"]["lin_pose.bias"], p0["render"]["lin_pose.bias"])
    assert not torch.equal(trained["bg_implicit"]["lin0.weight"], geo["bg_implicit"]["lin0.weight"])
    assert not torch.equal(trained["bg_render"]["lin0.weight"], geo["bg_render"]["lin0.weight"])


@pytest.mark.parametrize("p", [0, 1])
def test_fourier_share_and_gradient_norm(trained, p):
    """(b) on near-surface points the Fourier columns carry >= 10 % of the fp64 grad sdf at the median;
    (c) |grad sdf| stays within roughly [0.2, 5] there."""
    person = trained["persons"][p]
    sd = _f64(person["implicit"])
    x = _near_surface(person, sd)
    assert x.shape[0] > 200
    _, g = _sdf_grad(sd, x, person["cond"])
    _, g0 = _sdf_grad(_without_fourier(sd), x, person["cond"])
    share = (g - g0).norm(dim=1) / g.norm(dim=1)
    assert float(share.median()) >= 0.10, float(share.median())
    n = g.norm(dim=1).numpy()
    lo, hi = np.quantile(n, [0.05, 0.95])
    assert 0.2 <= lo and hi <= 5.0, (float(lo), float(hi))
    assert 0.03 < n.min() and n.max() < 10.0


def test_renders_surfaces():
    """(d) a 'boxes' ray batch still hits surfaces: acc_map > 0.5 on a sizeable fraction of the rays."""
    sc = S.make_scene(P=2, S=16, seed=42, weights="trained")
    inp = S.make_rays(sc, 64, seed=5, region="boxes")
    o = port.multiply_forward(sc, inp, S.make_hit_lists(sc, inp))
    assert float((o["acc_map"] > 0.5).float().mean()) > 0.2
    assert bool(torch.isfinite(o["rgb_values"]).all())
