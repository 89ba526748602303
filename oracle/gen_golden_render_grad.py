"""TEST INFRASTRUCTURE ONLY — generate tests/golden/render_grad.npz: autograd gradients of the reference's own compositing
pieces, which pin the differentiable restatement oracle/render_grad.py.

    python -m oracle.gen_golden_render_grad

Runs only where the reference tree is present (oracle/ref_shim.py).  What it stores:
  * LaplaceDensity (lib/model/density.py:15-29), the UNMODIFIED reference module: sigma and torch autograd's gradients
    w.r.t. sdf and the `beta` parameter of a weighted sum of sigma, for beta_param in {0.1, 1e-3, -0.05, 0, -1e-4} and sdf
    values that include 0, +-1e-3 and +-1e-9;
  * Multiply.bg_volume_rendering (multiply.py:682-696, called unbound on a shell object with the reference AbsDensity) and
    the weighted sum of :539: gradients w.r.t. bg_sdf and the per-sample colours, on eval and jittered depths, with
    exact zeros and |s| ~ 1e-9 on the 1e10-long last interval;
  * the foreground block restated by oracle/render_grad.composite in float64 on a seeded 3-person input without live
    ties: gradients w.r.t. sdf / rgb / normals per person and beta for random upstream gradients of every output.
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)

from oracle import ref_shim, render_grad as RG      # noqa: E402

GOLD = os.path.join(ROOT, "tests", "golden")
BETA_PARAMS = (0.1, 1e-3, -0.05, 0.0, -1e-4)


def density_case(ref, out):
    g = torch.Generator().manual_seed(3)
    sdf = torch.cat([torch.tensor([0.0, 1e-3, -1e-3, 1e-9, -1e-9, 0.0]), (torch.rand(58, generator=g) - 0.5) * 0.4])
    u = torch.randn(sdf.shape[0], generator=g)
    out["density_sdf"], out["density_u"] = sdf.numpy(), u.numpy()
    out["density_beta_params"] = np.array(BETA_PARAMS, np.float32)
    sig, gs, gb = [], [], []
    for bp in BETA_PARAMS:
        dens = ref.density.LaplaceDensity(params_init={"beta": bp}, beta_min=0.0001)
        s = sdf.clone().requires_grad_(True)
        sigma = dens(s)
        (sigma * u).sum().backward()
        sig.append(sigma.detach().numpy())
        gs.append(s.grad.numpy())
        gb.append(float(dens.beta.grad))
    out["density_sigma"], out["density_grad_sdf"] = np.stack(sig), np.stack(gs)
    out["density_grad_beta_param"] = np.array(gb, np.float32)


def bg_case(ref, out):
    Multiply = ref.multiply.Multiply
    m = Multiply.__new__(Multiply)
    torch.nn.Module.__init__(m)
    m.bg_density = ref.density.AbsDensity()
    g = torch.Generator().manual_seed(4)
    R = 24
    t_rand = torch.rand(R, 32, generator=g)
    for name, tr in (("eval", None), ("train", t_rand.numpy())):
        z = torch.from_numpy(RG.bg_depths(R, 3.0, tr))
        sdf = (torch.rand(R, 32, generator=g) - 0.5) * 2.0
        sdf[0, :] = 0.0
        sdf[1, 5] = 0.0
        sdf[2:8, -1] = torch.tensor([1e-9, -1e-9, 3e-10, -2e-9, 0.0, 1e-8])
        sdf[8:12, :-1] = 1e-4 * sdf[8:12, :-1]                     # nearly empty rays: the last interval decides
        sdf[8:12, -1] = torch.tensor([1e-9, -5e-10, 2e-10, 1e-10])
        rgb = torch.rand(R, 32, 3, generator=g)
        u = torch.randn(R, 3, generator=g)
        s = sdf.clone().requires_grad_(True)
        c = rgb.clone().requires_grad_(True)
        w = Multiply.bg_volume_rendering(m, z, s.reshape(-1, 1))
        bgv = torch.sum(w.unsqueeze(-1) * c, 1)                     # multiply.py:539
        (bgv * u).sum().backward()
        out.update({f"bg_{name}_z": z.numpy(), f"bg_{name}_sdf": sdf.numpy(), f"bg_{name}_rgb": rgb.numpy(),
                    f"bg_{name}_u": u.numpy(), f"bg_{name}_values": bgv.detach().numpy(),
                    f"bg_{name}_grad_sdf": s.grad.numpy(), f"bg_{name}_grad_rgb": c.grad.numpy()})
    out["bg_t_rand"] = t_rand.numpy()


def fg_case(out):
    """3 persons, n = 17, R = 12; rows are strictly increasing and distinct between persons (no live ties)."""
    rng = np.random.RandomState(8)
    P, R, n = 3, 12, 17
    persons = []
    for p in range(P):
        idx = np.flatnonzero(rng.random_sample(R) < 0.7).astype(np.int64)
        if idx.size == 0:
            idx = np.array([0], np.int64)
        Rp = idx.size
        z = np.sort(rng.uniform(0.5, 3.5, (Rp, n + 1)), 1)
        zm = 0.5 * (z[:, :-1] + z[:, 1:])
        sdf = np.clip((rng.uniform(1.0, 3.0, (Rp, 1)) - zm) * rng.uniform(1, 10, (Rp, 1)), -1, 1)
        sdf[rng.random_sample(sdf.shape) < 0.05] = 0.0
        persons.append(dict(idx=idx, z=z, sdf=sdf, rgb=rng.random_sample((Rp, n, 3)), nrm=rng.uniform(-1, 1, (Rp, n, 3))))
    ups = dict(d_fg=rng.randn(R, 3), d_nrm=rng.randn(R, 3), d_acc=rng.randn(R), d_accp=rng.randn(R, P), d_bgT=rng.randn(R))
    beta = torch.tensor(0.05, dtype=torch.float64, requires_grad=True)
    tp = [dict(idx=d["idx"], **{k: torch.tensor(d[k], requires_grad=(k != "z")) for k in ("z", "sdf", "rgb", "nrm")})
          for d in persons]
    outs = RG.composite(tp, R, n, beta)
    loss = sum((o * torch.from_numpy(ups[k])).sum() for o, k in zip(outs, ("d_fg", "d_nrm", "d_acc", "d_accp", "d_bgT")))
    loss.backward()
    out["fg_beta"] = np.array(0.05)
    out["fg_grad_beta"] = np.array(float(beta.grad))
    for k, v in ups.items():
        out["fg_" + k] = v
    for p, (d, t) in enumerate(zip(persons, tp)):
        for k in ("idx", "z", "sdf", "rgb", "nrm"):
            out[f"fg_{k}_{p}"] = d[k]
        for k in ("sdf", "rgb", "nrm"):
            out[f"fg_grad_{k}_{p}"] = t[k].grad.numpy()


def main():
    torch.set_default_dtype(torch.float32)
    ref = ref_shim.load()
    out = {}
    density_case(ref, out)
    bg_case(ref, out)
    fg_case(out)
    os.makedirs(GOLD, exist_ok=True)
    np.savez_compressed(os.path.join(GOLD, "render_grad.npz"), **out)
    print("wrote render_grad", {k: np.asarray(v).shape for k, v in out.items()})


if __name__ == "__main__":
    main()
