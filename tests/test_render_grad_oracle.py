"""CPU: the differentiable restatement of the compositing stages (oracle/render_grad.py), which the GPU backward tests use
as their fp64 reference.  Its values in float32 reproduce oracle/port.py; its gradients match the reference's own
autograd (LaplaceDensity, Multiply.bg_volume_rendering) stored in tests/golden/render_grad.npz; gradcheck holds away
from the kinks; and at the kinks it takes torch's conventions (sign(0) = 0)."""
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from oracle import port, render_grad as RG      # noqa: E402

GOLD = os.path.join(ROOT, "tests", "golden", "render_grad.npz")


def _persons(seed, P, R, n, dtype=torch.float64):
    rng = np.random.RandomState(seed)
    out = []
    for p in range(P):
        idx = np.flatnonzero(rng.random_sample(R) < 0.7).astype(np.int64)
        Rp = idx.size
        z = np.sort(rng.uniform(0.5, 3.5, (Rp, n + 1)), 1).astype(np.float32)
        sdf = rng.uniform(-0.3, 0.3, (Rp, n)).astype(np.float32)
        sdf[np.abs(sdf) < 0.02] = 0.05
        out.append(dict(idx=idx, z=torch.tensor(z, dtype=dtype), sdf=torch.tensor(sdf, dtype=dtype),
                        rgb=torch.tensor(rng.random_sample((Rp, n, 3)), dtype=dtype),
                        nrm=torch.tensor(rng.uniform(-1, 1, (Rp, n, 3)), dtype=dtype)))
    return out


def test_fp32_values_match_port():
    """composite / bg_volume_rendering / blend in float32 against port.composite_nerfacc, port.bg_volume_rendering."""
    P, R, n, bp = 3, 14, 9, 0.05
    ps = _persons(1, P, R, n, torch.float32)
    beta = port.get_beta(bp)
    got = RG.composite(ps, R, n, beta)
    want = port.composite_nerfacc([torch.from_numpy(d["idx"]) for d in ps], [d["z"][:, :-1] for d in ps],
                                  [d["z"][:, -1] for d in ps], [d["sdf"] for d in ps], [d["rgb"] for d in ps],
                                  [d["nrm"] for d in ps], list(range(P)), R, bp)
    for g, w in zip(got, want):
        assert g.dtype == torch.float32
        assert float((g - w).abs().max()) < 1e-6
    z = torch.from_numpy(RG.bg_depths(R, 3.0, np.random.RandomState(2).random_sample((R, 32))))
    s = torch.from_numpy(np.random.RandomState(3).uniform(-2, 2, (R, 32)).astype(np.float32))
    assert torch.equal(RG.bg_volume_rendering(z, s), port.bg_volume_rendering(z, s.reshape(-1, 1)))
    rgb, fgv = RG.blend(got[0], got[4], torch.ones(R, 3))
    assert torch.equal(rgb, fgv)


def test_matches_reference_density_gradients():
    """LaplaceDensity's autograd through beta = |beta_param| + beta_min, at sdf = 0, +-1e-9, and beta_param <= 0."""
    g = np.load(GOLD)
    sdf = torch.from_numpy(g["density_sdf"]).double()
    u = torch.from_numpy(g["density_u"]).double()
    for k, bp in enumerate(g["density_beta_params"]):
        p = torch.tensor(float(bp), dtype=torch.float64, requires_grad=True)
        s = sdf.clone().requires_grad_(True)
        sigma = RG.laplace_density(s, p.abs() + 1e-4)
        (sigma * u).sum().backward()
        want_s = g["density_grad_sdf"][k].astype(np.float64)
        assert np.allclose(sigma.detach().numpy(), g["density_sigma"][k], rtol=1e-5, atol=1e-6 * np.abs(g["density_sigma"][k]).max())
        assert np.allclose(s.grad.numpy(), want_s, rtol=2e-5, atol=1e-6 * np.abs(want_s).max())
        assert np.all(s.grad.numpy()[sdf.numpy() == 0] == 0) and np.all(want_s[sdf.numpy() == 0] == 0)
        wb = float(g["density_grad_beta_param"][k])
        assert abs(float(p.grad) - wb) <= 2e-5 * max(abs(wb), 1.0), (bp, float(p.grad), wb)


@pytest.mark.parametrize("mode", ["eval", "train"])
def test_matches_reference_bg_gradients(mode):
    """Multiply.bg_volume_rendering + the sum of multiply.py:539: d bg_sdf (0 and |s| ~ 1e-9 on the 1e10 interval) and
    d per-sample colour."""
    g = np.load(GOLD)
    z = torch.from_numpy(g[f"bg_{mode}_z"]).double()
    assert np.array_equal(g[f"bg_{mode}_z"], RG.bg_depths(z.shape[0], 3.0, g["bg_t_rand"] if mode == "train" else None))
    s = torch.from_numpy(g[f"bg_{mode}_sdf"]).double().requires_grad_(True)
    c = torch.from_numpy(g[f"bg_{mode}_rgb"]).double().requires_grad_(True)
    _, v = RG.bg_volume_rendering(z, s, c)
    (v * torch.from_numpy(g[f"bg_{mode}_u"]).double()).sum().backward()
    assert np.allclose(v.detach().numpy(), g[f"bg_{mode}_values"], atol=2e-6)
    for got, want in ((s.grad.numpy(), g[f"bg_{mode}_grad_sdf"]), (c.grad.numpy(), g[f"bg_{mode}_grad_rgb"])):
        # float32 reference: relative to the row scale (the 1e10 interval makes last-sample entries ~1e9)
        scale = np.abs(want).reshape(want.shape[0], -1).max(1) + 1e-6
        err = np.abs(got - want).reshape(want.shape[0], -1).max(1)
        assert np.all(err <= 5e-4 * scale), (err / scale).max()
    assert np.all(s.grad.numpy()[g[f"bg_{mode}_sdf"] == 0] == 0)


def test_matches_stored_foreground_gradients():
    """The restated foreground block's float64 gradients on the stored 3-person input (no live ties)."""
    g = np.load(GOLD)
    P = 3
    n = g["fg_sdf_0"].shape[1]
    R = g["fg_d_acc"].shape[0]
    beta = torch.tensor(float(g["fg_beta"]), dtype=torch.float64, requires_grad=True)
    tp = [dict(idx=g[f"fg_idx_{p}"], **{k: torch.from_numpy(g[f"fg_{k}_{p}"]).requires_grad_(k != "z")
                                        for k in ("z", "sdf", "rgb", "nrm")}) for p in range(P)]
    outs = RG.composite(tp, R, n, beta)
    loss = sum((o * torch.from_numpy(g["fg_" + k])).sum() for o, k in zip(outs, ("d_fg", "d_nrm", "d_acc", "d_accp", "d_bgT")))
    loss.backward()
    assert abs(float(beta.grad) - float(g["fg_grad_beta"])) <= 1e-10 * max(1.0, abs(float(g["fg_grad_beta"])))
    for p in range(P):
        for k in ("sdf", "rgb", "nrm"):
            assert np.allclose(tp[p][k].grad.numpy(), g[f"fg_grad_{k}_{p}"], rtol=1e-10, atol=1e-12)


def test_gradcheck_away_from_kinks():
    """torch.autograd.gradcheck of the three stages on small float64 cases (no sdf near 0, distinct t_end)."""
    P, R, n = 2, 5, 4
    ps = _persons(9, P, R, n)
    beta = torch.tensor(0.2, dtype=torch.float64, requires_grad=True)
    leaves = [beta] + [d[k].requires_grad_(True) for d in ps for k in ("sdf", "rgb", "nrm")]

    def f(*args):
        b = args[0]
        it = iter(args[1:])
        qs = [dict(idx=d["idx"], z=d["z"], sdf=next(it), rgb=next(it), nrm=next(it)) for d in ps]
        return RG.composite(qs, R, n, b)
    assert torch.autograd.gradcheck(f, leaves, eps=1e-6, atol=1e-6, rtol=1e-5)
    z = torch.from_numpy(RG.bg_depths(3, 3.0)).double()
    s = torch.from_numpy(np.random.RandomState(4).uniform(0.1, 2.0, (3, 32)) *
                         np.sign(np.random.RandomState(5).uniform(-1, 1, (3, 32)))).requires_grad_(True)
    c = torch.rand(3, 32, 3, dtype=torch.float64, requires_grad=True)
    assert torch.autograd.gradcheck(lambda a, b: RG.bg_volume_rendering(z, a, b)[1], (s, c), eps=1e-7, atol=1e-6)
    fg = torch.rand(4, 3, dtype=torch.float64, requires_grad=True)
    t = torch.rand(4, dtype=torch.float64, requires_grad=True)
    bg = torch.rand(4, 3, dtype=torch.float64, requires_grad=True)
    assert torch.autograd.gradcheck(RG.blend, (fg, t, bg))


def test_zero_sdf_has_zero_gradient():
    """At sdf == 0 exactly, d/d sdf is 0 in both the foreground (Laplace) and the background (|s|) restatements."""
    P, R, n = 2, 4, 6
    ps = _persons(12, P, R, n)
    for d in ps:
        d["sdf"][:, ::2] = 0.0
        d["sdf"].requires_grad_(True)
    fg, nrm, acc, accp, bgT = RG.composite(ps, R, n, torch.tensor(0.01, dtype=torch.float64))
    (fg.sum() + acc.sum() + bgT.sum()).backward()
    for d in ps:
        assert torch.all(d["sdf"].grad[:, ::2] == 0)
        assert torch.any(d["sdf"].grad[:, 1::2] != 0)
    z = torch.from_numpy(RG.bg_depths(2, 3.0)).double()
    s = torch.zeros(2, 32, dtype=torch.float64, requires_grad=True)
    RG.bg_volume_rendering(z, s, torch.rand(2, 32, 3, dtype=torch.float64))[1].sum().backward()
    assert torch.all(s.grad == 0)
