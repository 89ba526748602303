"""CPU: the restatements of tests/test_gpu_frame_geometry.py (lbs, the camera lift, sphere bounds, depth2pts_outside)
against oracle/port.py and the goldens of the reference, so that the float64 references the GPU tests use state the same
operations."""
import importlib.util
import os

import numpy as np
import torch

from multiply_b200 import scene as S
from oracle import port

_spec = importlib.util.spec_from_file_location(
    "_frame_geometry_gpu_tests", os.path.join(os.path.dirname(os.path.abspath(__file__)), "test_gpu_frame_geometry.py"))
G = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(G)


def test_lbs_reference_matches_port_and_golden(golden_dir):
    """lbs_ref in float32 against port.lbs (the reference's lbs.py run in float32) and in float64 against smpl_lbs.npz;
    SMPLServer's scale / translation / canonical inverse against port.smpl_server_forward."""
    g = np.load(os.path.join(golden_dir, "smpl_lbs.npz"))
    sm = S.make_smpl_model(300)
    model = G.model_np(sm)
    betas, pose = g["betas"][0], g["pose"][0]
    v_p, A_p = port.lbs(torch.from_numpy(betas), torch.from_numpy(pose), sm)
    o32 = G.lbs_ref(model, betas, pose, dtype=np.float32)
    assert o32["verts"].dtype == np.float32
    assert np.abs(o32["verts"] - v_p.numpy()).max() < 2e-6
    assert np.abs(o32["tfs"] - A_p.numpy()).max() < 2e-6
    o64 = G.lbs_ref(model, betas, pose)
    assert np.abs(o64["verts"] - g["verts"]).max() < 2e-6
    assert np.abs(o64["tfs"] - g["A"]).max() < 2e-6
    # the magnitudes bound the values
    assert (o64["M_verts"] >= np.abs(o64["verts"])).all() and (o64["M_tfs"] >= np.abs(o64["tfs"]) - 1e-12).all()
    tinv, _ = port.smpl_canonical_tfs_inv(sm, torch.zeros(10))
    _, cano = G.canonical_ref(model, np.zeros(10, np.float32))
    assert np.abs(cano[0] - tinv.numpy()).max() < 5e-5
    ref = port.smpl_server_forward(sm, tinv, torch.tensor([0.5]), torch.tensor([0.3, 0.1, -0.2]),
                                   torch.from_numpy(pose), torch.from_numpy(betas))
    o = G.lbs_ref(model, betas, pose, 0.5, (0.3, 0.1, -0.2), absolute=False, cinv=cano)
    assert np.abs(o["verts"] - ref["smpl_verts"].numpy()).max() < 5e-6
    assert np.abs(o["tfs"] - ref["smpl_tfs"].numpy()).max() < 5e-5


def test_rodrigues_reference_matches_port():
    """rodrigues_ref in float32 against port.batch_rodrigues on every pose of the GPU test (theta = 0, tiny angles, pi,
    up to 4 pi)."""
    for name, th in G.smpl_poses().items():
        r32, _ = G.rodrigues_ref(th, np.float32)
        rp = port.batch_rodrigues(torch.from_numpy(th).view(-1, 3)).numpy()
        assert np.abs(r32 - rp).max() < 4e-6, name
        r64, _ = G.rodrigues_ref(th)
        assert np.abs(r64 - rp).max() < 1e-5, name


def test_lift_and_sphere_reference_match_port_and_golden(golden_dir):
    """lift_ref / sphere_ref against rays.npz (float64) and port.get_camera_params / get_sphere_intersections on the
    skewed camera of the GPU test (float32)."""
    g = np.load(os.path.join(golden_dir, "rays.npz"))
    d, cam, _ = G.lift_ref(g["uv"][0], g["pose"][0], g["intrinsics"][0])
    assert np.abs(d - g["ray_dirs"][0]).max() < 1e-6
    assert np.array_equal(cam.astype(np.float32), g["cam_loc"][0])
    nf, under, _ = G.sphere_ref(np.broadcast_to(g["cam_loc"][0], d.shape), g["ray_dirs"][0], 3.0)
    assert (under > 0).all() and np.abs(nf - g["near_far"]).max() < 2e-5
    K, pose = G.skew_camera()
    uv = G._uv(700, 1)
    d32, _, _ = G.lift_ref(uv, pose, K, np.float32)
    dp, cp = port.get_camera_params(torch.from_numpy(uv)[None], torch.from_numpy(pose)[None], torch.from_numpy(K)[None])
    assert np.abs(d32 - dp[0].numpy()).max() < 4e-7
    d64, _, _ = G.lift_ref(uv, pose, K)
    assert np.abs(d64 - dp[0].numpy()).max() < 1e-6
    cam = np.broadcast_to(cp[0].numpy(), (700, 3))
    nf64, _, _ = G.sphere_ref(cam, dp[0].numpy(), 3.0)
    nfp = port.get_sphere_intersections(torch.from_numpy(np.ascontiguousarray(cam)), dp[0], 3.0).numpy()
    assert np.abs(nf64 - nfp).max() < 2e-6


def test_depth2pts_reference_matches_port():
    """depth2pts_ref against port.depth2pts_outside on the GPU test's background rays and the grid_rays(res=24) frame,
    wherever the latter is finite.  The rays through the sphere's centre are skipped explicitly: there the port (as the
    reference) divides 0 by 0 and gives NaN, and the restatement gives the limit p_sphere / |p_sphere|."""
    o, d = G.bg_rays()
    K, pose = S.make_camera(res=24)
    gd, gc = port.get_camera_params(S.grid_rays(res=24)["uv"], pose, K)
    o = np.concatenate([o, np.broadcast_to(gc[0].numpy(), (576, 3))]).astype(np.float32)
    d = np.concatenate([d, gd[0].numpy()]).astype(np.float32)
    R = o.shape[0]
    centre = [0, 1, 2, 7 + 250 + 12 * 24 + 12]
    z = G.RG.bg_depths(R, 3.0)
    want = port.depth2pts_outside(torch.from_numpy(o)[:, None].expand(-1, 32, -1).double(),
                                  torch.from_numpy(d)[:, None].expand(-1, 32, -1).double(),
                                  torch.from_numpy(z).double(), 3.0).numpy()
    got = G.depth2pts_ref(o, d, z, 3.0)
    bad = ~np.isfinite(want).all((1, 2))
    assert np.array_equal(np.flatnonzero(bad), centre)
    assert np.abs(got[~bad] - want[~bad]).max() < 1e-9
    assert np.isfinite(got).all()
    for i in centre:
        o64, d64 = o[i].astype(np.float64), d[i].astype(np.float64)
        odd = d64 @ o64
        ps = o64 + (np.sqrt(odd * odd - (o64 @ o64 - 9.0)) - odd) * d64
        assert np.allclose(got[i, :, :3], ps / np.linalg.norm(ps), rtol=0, atol=1e-15)
        assert np.array_equal(got[i, :, 3], z[i].astype(np.float64))
