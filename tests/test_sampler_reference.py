"""CPU: the float64 sampler reference of tests/test_gpu_sampler.py and tests/_sampler_ref.py -- oracle/port.error_bound_get_z_vals with ``dtype``,
``ray_sdf_fn`` and ``trace`` -- states the same algorithm as the float32 port that the goldens of the reference pin."""
import os

import numpy as np
import pytest
import torch

from multiply_b200 import scene as S
from oracle import port
import _sampler_ref as ref


def _rays(sc, R, seed, region, p=0):
    inp = S.make_rays(sc, R, seed=seed, region=region)
    dirs, cam = port.get_camera_params(inp["uv"], inp["pose"], inp["intrinsics"])
    cam = cam.unsqueeze(1).repeat(1, dirs.shape[1], 1).reshape(-1, 3)
    dirs = dirs.reshape(-1, 3)
    return inp, dirs, cam


@pytest.mark.parametrize("name,Sn,R,region", [("forward_S64_R48", 64, 48, "boxes"), ("forward_S16_R96", 16, 96, "image")])
def test_float32_trace_bit_equal_and_golden(golden_dir, name, Sn, R, region):
    """In float32 the traced path (dtype, ray_sdf_fn, trace) is bit-equal to the plain call, and both stay within the
    tolerances of tests/test_oracle_golden.py against the reference's own sampler output."""
    g = np.load(os.path.join(golden_dir, name + ".npz"))
    sc = S.make_scene(P=2, S=Sn, seed=42)
    inp, dirs, cam = _rays(sc, R, 1234, region)
    assert np.array_equal(inp["uv"].numpy(), g["uv"])
    for p in range(2):
        idx = torch.from_numpy(g[f"hits_{p}"])
        if idx.numel() == 0:
            idx = torch.tensor([0])
        person = sc["persons"][p]
        z, zb = port.error_bound_get_z_vals(dirs[idx], cam[idx], person, sc["cfg"], sc["beta_param"])
        tr, st = {}, {}
        fn = lambda o, zz, d: port.sdf_func_with_smpl_deformer(
            (o.unsqueeze(1) + zz.unsqueeze(2) * d.unsqueeze(1)).reshape(-1, 3), person, sc["cfg"])[0]
        z2, zb2 = port.error_bound_get_z_vals(dirs[idx], cam[idx], person, sc["cfg"], sc["beta_param"], stats=st,
                                              dtype=torch.float32, ray_sdf_fn=fn, trace=tr)
        assert torch.equal(z, z2) and torch.equal(zb, zb2)
        assert len(tr["trips"]) == st["trips"] == int(g["trips"][p])
        assert all(t["final"] == (i == st["trips"] - 1) for i, t in enumerate(tr["trips"]))
        assert np.abs(z2[:, :-1].numpy() - g[f"z_vals_{p}"]).max() < 2e-4


def test_float32_training_trace_golden(golden_dir):
    """Training mode (recorded draws of the reference) with the trace on: bit-equal to the plain call, and within the
    tolerances of test_oracle_golden.test_sampler_training_mode."""
    g = np.load(os.path.join(golden_dir, "sampler_train.npz"))
    sc = S.make_scene(P=2, S=16, seed=42)
    inp, dirs, cam = _rays(sc, 40, 21, "boxes")
    idx = torch.from_numpy(g["hits"])
    rng = {k: torch.from_numpy(g[k]) for k in ("t_rand", "u_final", "extra_perm", "eik_idx", "t_rand_bg")}
    a = port.error_bound_get_z_vals(dirs[idx], cam[idx], sc["persons"][0], sc["cfg"], sc["beta_param"], rng=rng)
    tr = {}
    b = port.error_bound_get_z_vals(dirs[idx], cam[idx], sc["persons"][0], sc["cfg"], sc["beta_param"], rng=rng,
                                    dtype=torch.float32, trace=tr)
    for x, y in zip(a, b):
        assert torch.equal(x, y)
    assert len(tr["trips"]) * sc["cfg"]["N_samples_eval"] == g["extra_perm"].shape[0]
    dz = np.abs(b[0].numpy() - g["z_vals"])
    assert np.median(dz) < 1e-6 and dz.max() < 5e-3
    assert np.abs(b[1].numpy() - g["z_bg"]).max() < 1e-7


class _Analytic:
    """ray_sdf_fn of an analytic SDF, evaluated in the caller's dtype; no point is near an outlier radius."""

    def __init__(self, f):
        self.f, self.dist = f, []

    def __call__(self, o, z, d):
        x = (o.unsqueeze(1) + z.unsqueeze(2) * d.unsqueeze(1)).reshape(-1, 3)
        self.dist.append(torch.full(z.shape, 1e3, dtype=torch.float64))
        return self.f(x)[:, None]


ANALYTIC = {
    "sphere": lambda x: (x - x.new_tensor([0.0, 0.1, 0.0])).norm(dim=1) - 0.3,
    "plane": lambda x: x @ x.new_tensor([0.0, 0.0, 1.0]) - 0.05,
    "constant": lambda x: torch.full_like(x[:, 0], 0.02),
}


@pytest.mark.parametrize("shape", sorted(ANALYTIC))
@pytest.mark.parametrize("E,S_,X,T,eps", [(32, 16, 8, 5, 0.1), (64, 32, 16, 3, 1e-3), (33, 33, 1, 1, 0.1)])
def test_float64_against_float32_analytic(shape, E, S_, X, T, eps):
    """The float64 port against the float32 port on a sphere, a plane and a constant SDF, through the comparison the GPU
    tests use (equal trips, batch flag off its tie, per-sample bound with the recorded masks)."""
    sc = S.make_scene(P=1, S=16, seed=42)
    _, dirs, cam = _rays(sc, 64, 5, "boxes")
    d, o = dirs[:20], cam[:20]
    cfg = ref.cfg_of(E, S_, X, T, eps=eps)
    st = {}
    z32, _ = port.error_bound_get_z_vals(d, o, None, cfg, cfg["beta_param"], stats=st, ray_sdf_fn=_Analytic(
        ANALYTIC[shape]))
    cb = _Analytic(ANALYTIC[shape])
    tr, st64 = {}, {}
    port.error_bound_get_z_vals(d.double(), o.double(), None, cfg, cfg["beta_param"], stats=st64, dtype=torch.float64,
                                ray_sdf_fn=cb, trace=tr)
    tr["n_trips"] = st64["trips"]
    assert tr["trips"][0]["z"].dtype == torch.float64 and tr["trips"][-1]["cdf"].dtype == torch.float64
    ref.compare("cpu " + shape, cfg, d, o, z32, st["trips"], tr, cb.dist)
