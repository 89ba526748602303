"""CPU: pin oracle/port.py against the outputs of the UNMODIFIED reference modules
(tests/golden/*.npz, produced by oracle/gen_golden.py in the build container)."""
import os
import numpy as np
import pytest
import torch

from oracle import port
from multiply_b200 import scene as S


def _g(golden_dir, name):
    return np.load(os.path.join(golden_dir, name + ".npz"))


@pytest.fixture(scope="module")
def scene64():
    return S.make_scene(P=2, S=64, seed=42)


def test_implicit_fg(golden_dir, scene64):
    g = _g(golden_dir, "implicit_fg")
    p0 = scene64["persons"][0]
    with torch.no_grad():
        y = port.implicit_forward(p0["implicit"], torch.from_numpy(g["x"]), p0["cond"], 6)
    assert np.abs(y.numpy() - g["out"]).max() < 2e-6


def test_implicit_fg_grad(golden_dir, scene64):
    g = _g(golden_dir, "implicit_fg_grad")
    p0 = scene64["persons"][0]
    x = torch.from_numpy(g["x"]).requires_grad_(True)
    y = port.implicit_forward(p0["implicit"], x, p0["cond"], 6)
    gr = torch.autograd.grad(y[:, 0].sum(), x)[0]
    assert np.abs(gr.numpy() - g["grad"]).max() < 2e-6


def test_render_fg(golden_dir, scene64):
    g = _g(golden_dir, "render_fg")
    p0 = scene64["persons"][0]
    with torch.no_grad():
        rgb = port.rendering_forward(p0["render"], "pose_no_view", torch.from_numpy(g["x"]),
                                     torch.from_numpy(g["normals"]), None, p0["cond"], torch.from_numpy(g["feat"]))
    assert np.abs(rgb.numpy() - g["rgb"]).max() < 1e-6


def test_bg_nets(golden_dir, scene64):
    g = _g(golden_dir, "bg_nets")
    with torch.no_grad():
        y = port.implicit_forward(scene64["bg_implicit"], torch.from_numpy(g["x"]), scene64["frame_code"], 10,
                                  weight_norm=False)
        rgb = port.rendering_forward(scene64["bg_render"], "nerf_frame_encoding", None, None,
                                     torch.from_numpy(g["view"]), None, y[:, 1:],
                                     frame_latent_code=scene64["frame_code"], weight_norm=False, multires_view=4)
    assert np.abs(y.numpy() - g["out"]).max() < 2e-6
    assert np.abs(rgb.numpy() - g["rgb"]).max() < 1e-6


def test_density(golden_dir, scene64):
    g = _g(golden_dir, "density")
    beta = port.get_beta(scene64["beta_param"])
    assert float(beta) == float(g["beta"])
    s = port.laplace_density(torch.from_numpy(g["sdf"]), beta)
    assert np.array_equal(s.numpy(), g["sigma"])
    s = port.laplace_density(torch.from_numpy(g["sdf"]), torch.tensor(0.013))
    assert np.array_equal(s.numpy(), g["sigma_b"])


def test_deformer(golden_dir, scene64):
    g = _g(golden_dir, "deformer")
    p0 = scene64["persons"][0]
    xc, outl = port.deform_inverse(torch.from_numpy(g["pts"]), p0)
    assert np.array_equal(outl.numpy(), g["outlier"])
    assert np.abs(xc.numpy() - g["x_c"]).max() < 1e-6
    w, _ = port.query_skinning_weights(xc[None], p0["verts_c"], p0["weights"][None])
    xd = port.skinning(xc[None], w, p0["tfs"][None], inverse=False)[0]
    assert np.abs(xd.numpy() - g["x_d"]).max() < 1e-6


@pytest.mark.parametrize("name,P,Sn,R,region,seed", [("forward_S64_R48", 2, 64, 48, "boxes", 42),
                                                     ("forward_S16_R96", 2, 16, 96, "image", 42),
                                                     ("forward_P3_S32_R40", 3, 32, 40, "boxes", 7)])
def test_forward(golden_dir, name, P, Sn, R, region, seed):
    g = _g(golden_dir, name)
    sc = S.make_scene(P=P, S=Sn, seed=seed)
    inp = S.make_rays(sc, R, seed=1234, region=region)
    assert np.array_equal(inp["uv"].numpy(), g["uv"]), "synthetic input drifted from the golden's"
    hits = S.make_hit_lists(sc, inp)
    for p in range(P):
        assert np.array_equal(hits[p].numpy(), g[f"hits_{p}"])
    st = {}
    o = port.multiply_forward(sc, inp, hits, stats=st, return_samples=True)
    assert list(st["trips"]) == list(g["trips"])
    for k in ("rgb_values", "fg_rgb_values", "normal_values", "acc_map", "acc_person_list"):
        assert np.abs(o[k].numpy() - g[k]).max() < 1e-5, k
    for p in range(P):
        assert np.abs(o["_z_vals"][p].numpy() - g[f"z_vals_{p}"]).max() < 2e-4
        assert np.abs(o["_sdf"][p].numpy() - g[f"sdf_{p}"]).max() < 1e-4


def test_smpl_lbs(golden_dir):
    """oracle/port.lbs against the reference's lib/smpl/lbs.py:lbs (run unmodified by gen_golden)."""
    g = _g(golden_dir, "smpl_lbs")
    sm = S.make_smpl_model(300)
    verts, A = port.lbs(torch.from_numpy(g["betas"])[0], torch.from_numpy(g["pose"])[0], sm)
    assert np.abs(verts.numpy() - g["verts"]).max() < 2e-6
    assert np.abs(A.numpy() - g["A"]).max() < 2e-6


def test_rays(golden_dir):
    """port.get_camera_params / get_sphere_intersections against the reference's rend_util (skewed intrinsics,
    rotated camera)."""
    g = _g(golden_dir, "rays")
    dirs, cam = port.get_camera_params(torch.from_numpy(g["uv"]), torch.from_numpy(g["pose"]),
                                       torch.from_numpy(g["intrinsics"]))
    assert np.abs(dirs.numpy() - g["ray_dirs"]).max() < 1e-7
    assert np.abs(cam.numpy() - g["cam_loc"]).max() == 0.0
    cam_r = cam.unsqueeze(1).repeat(1, 300, 1).reshape(-1, 3)
    nf = port.get_sphere_intersections(cam_r, dirs.reshape(-1, 3), r=3.0)
    assert np.abs(nf.numpy() - g["near_far"]).max() < 1e-6


def test_sdf_grid(golden_dir, scene64):
    """port.sdf_grid (generate_mesh lattice + query_oc) against the reference's Multiply.query_oc."""
    g = _g(golden_dir, "sdf_grid")
    p1 = scene64["persons"][1]
    vals, pts = port.sdf_grid(p1, dict(scene64["cfg"], multires=6), p1["verts_c"], int(g["res"]))
    assert np.array_equal(pts, g["points"])
    assert np.abs(vals.numpy().reshape(-1) - g["occ"]).max() < 2e-6


def test_sampler_training_mode(golden_dir):
    """port.error_bound_get_z_vals in TRAINING mode (random draws fed in as tensors) against the reference's
    ErrorBoundSampler.get_z_vals with model.training set: sample depths, jittered inverse-sphere depths, eikonal pick."""
    g = _g(golden_dir, "sampler_train")
    sc = S.make_scene(P=2, S=16, seed=42)
    inputs = dict(S.make_rays(sc, 40, seed=21, region="boxes"))
    assert np.array_equal(inputs["uv"].numpy(), g["uv"])
    dirs, cam = port.get_camera_params(inputs["uv"], inputs["pose"], inputs["intrinsics"])
    cam = cam.unsqueeze(1).repeat(1, dirs.shape[1], 1).reshape(-1, 3)
    dirs = dirs.reshape(-1, 3)
    idx = torch.from_numpy(g["hits"])
    rng = {k: torch.from_numpy(g[k]) for k in ("t_rand", "u_final", "extra_perm", "eik_idx", "t_rand_bg")}
    st = {}
    z, z_bg, z_eik = port.error_bound_get_z_vals(dirs[idx], cam[idx], sc["persons"][0], sc["cfg"], sc["beta_param"],
                                                 stats=st, rng=rng)
    assert st["trips"] * sc["cfg"]["N_samples_eval"] == g["extra_perm"].shape[0]
    assert np.abs(z_bg.numpy() - g["z_bg"]).max() < 1e-7
    dz = np.abs(z.numpy() - g["z_vals"])
    assert np.median(dz) < 1e-6 and dz.max() < 5e-3          # coarse 16/32/8 sampler: see test_forward_golden_coarse
    assert np.abs(z_eik.numpy() - g["z_eik"]).max() < 5e-3


def _train_inputs(g, sc):
    """The `train` argument of port.multiply_forward / Renderer.render from the recorded draws of the reference."""
    rng, eik = [], []
    for p in range(2):
        rng.append({"t_rand": torch.from_numpy(g[f"t_rand_{p}"]), "u_final": torch.from_numpy(g[f"u_final_{p}"]),
                    "extra_perm": torch.from_numpy(g[f"extra_perm_{p}"]), "eik_idx": torch.from_numpy(g[f"eik_idx_{p}"]),
                    "t_rand_bg": torch.from_numpy(g[f"t_rand_bg_sampler_{p}"])})
        vc = sc["persons"][p]["verts_c"]
        idx = torch.from_numpy(g[f"eik_perm_{p}"])[:512]
        eik.append(vc[idx] + torch.from_numpy(g[f"eik_noise_{p}"])[0] * 0.01)        # sampler.py:100-103, local_sigma 0.01
    return dict(rng=rng, eik_points=eik, t_rand_bg=torch.from_numpy(g["t_rand_bg"]))


def test_forward_training_mode(golden_dir):
    """port.multiply_forward(train=...) — the VALUES of Multiply.forward's training branch (stochastic sampling, no
    outlier clamp, eikonal gradients, jittered background depths) — against the reference's own objects driven through
    that branch with the same random draws."""
    g = _g(golden_dir, "forward_train")
    sc = S.make_scene(P=2, S=16, seed=42)
    inputs = S.make_rays(sc, 40, seed=33, region="boxes")
    assert np.array_equal(inputs["uv"].numpy(), g["uv"])
    hits = [torch.from_numpy(g[f"hits_{p}"]) for p in range(2)]
    st = {}
    out = port.multiply_forward(sc, inputs, hits, stats=st, return_samples=True, train=_train_inputs(g, sc))
    assert [t * sc["cfg"]["N_samples_eval"] for t in st["trips"]] == [g[f"extra_perm_{p}"].shape[0] for p in range(2)]
    assert np.abs(out["grad_theta"].numpy() - g["grad_theta"]).max() < 2e-6
    for p in range(2):
        dz = np.abs(out["_z_vals"][p].numpy() - g[f"z_vals_{p}"])
        assert np.median(dz) < 1e-6 and dz.max() < 5e-3
    # coarse 16/32/8 sampler: pixels inherit the depth jitter of the inverse-CDF step (see test_forward_golden_coarse)
    for k, tol in (("rgb_values", 1e-5), ("acc_map", 1e-5), ("normal_values", 5e-4), ("acc_person_list", 1e-5)):
        d = np.abs(out[k].numpy() - g[k])
        assert np.median(d) < 1e-5 and d.max() < tol, (k, float(d.max()))


def test_implicit_fg_trained(golden_dir):
    """oracle/port.py in float64 against the reference modules at trained-like parameters (scene.perturb_networks):
    anchors the fp64 oracle of tests/test_gpu_networks.py -- weight-norm semantics (g != ||v||_row), the embedding
    order for d = 3 (non-zero Fourier columns), the skip layer and the hidden biases -- to the reference."""
    g = _g(golden_dir, "implicit_fg_trained")
    p0 = S.make_scene(P=2, S=64, seed=42, weights="trained")["persons"][0]
    imp = {k: v.double() for k, v in p0["implicit"].items()}
    ren = {k: v.double() for k, v in p0["render"].items()}
    cond = p0["cond"].double()
    x = torch.from_numpy(g["x"]).double().requires_grad_(True)
    y = port.implicit_forward(imp, x, cond, 6)
    gr = torch.autograd.grad(y[:, 0].sum(), x)[0]
    # the fixture is the reference in float32: the bounds are its rounding (measured 2.6e-6 / 1.3e-6 / 9e-8); a port
    # that ignored weight_g would be off by 3
    assert np.abs(y.detach().numpy() - g["out"]).max() < 5e-6
    assert np.abs(gr.numpy() - g["grad"]).max() < 5e-6
    with torch.no_grad():
        rgb = port.rendering_forward(ren, "pose_no_view", x.detach(), torch.from_numpy(g["normals"]).double(), None, cond,
                                     torch.from_numpy(g["out"][:, 1:]).double())
    assert np.abs(rgb.numpy() - g["rgb"]).max() < 1e-6
