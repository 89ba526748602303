"""TEST INFRASTRUCTURE ONLY — generate tests/golden/*.npz by running the UNMODIFIED reference
modules (imported from /root/reference/code under oracle/ref_shim.py) on seeded synthetic
inputs.  Runs only in the build container (the GPU box has no /root/reference); the
outputs are committed so that every other machine can pin oracle/port.py and the CUDA
path against what the reference itself computes.

    python -m oracle.gen_golden            # rewrites tests/golden/

What is executed from the reference, unmodified:
  lib.model.networks.ImplicitNet / RenderingNet   (forward)
  lib.model.density.LaplaceDensity / AbsDensity
  lib.model.ray_sampler.ErrorBoundSampler.get_z_vals
  lib.model.deformer.SMPLDeformer.forward / forward_skinning / query_skinning_weights_smpl_multi, skinning
  lib.model.multiply.Multiply.sdf_func_with_smpl_deformer / get_rbg_value / forward_gradient /
      depth2pts_outside / bg_volume_rendering          (called as unbound methods on a shell object)
  lib.utils.rend_util.get_camera_params / get_sphere_intersections
and, because Multiply.forward itself needs trimesh (host ray/box test) which is absent, a
line-for-line driver of its eval branch (multiply.py:223-232, 254-310, 393-418, 425-484,
514-545, 589-598) that calls those reference objects.
"""
import os
import sys
import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)

from oracle import ref_shim, port          # noqa: E402
from multiply_b200 import scene as S       # noqa: E402

GOLD = os.path.join(ROOT, "tests", "golden")


def ref_opts(A):
    imp = A(dict(feature_vector_size=256, d_in=3, d_out=1, dims=[256] * 8, init="geometry", bias=0.6,
                 skip_in=[4], weight_norm=True, embedder_mode="fourier", multires=6, cond="smpl",
                 number_person=2, scene_bounding_sphere=3.0))
    ren = A(dict(feature_vector_size=256, mode="pose_no_view", d_in=14, d_out=3, dims=[256] * 4,
                 weight_norm=True, multires_view=-1))
    bgi = A(dict(feature_vector_size=256, d_in=4, d_out=1, dims=[256] * 8, init="none", bias=0.0,
                 skip_in=[4], weight_norm=False, embedder_mode="fourier", multires=10, cond="frame"))
    bgr = A(dict(feature_vector_size=256, mode="nerf_frame_encoding", d_in=3, d_out=3, dims=[128],
                 weight_norm=False, multires_view=4))
    return imp, ren, bgi, bgr


def build_ref_model(ref, scene):
    """A shell ``Multiply`` object populated with reference sub-modules carrying the synthetic
    scene's parameters (Multiply.__init__ needs SMPL pkl / betas.npy / smpl_init .pth)."""
    A = ref.AttrDict
    imp_o, ren_o, bgi_o, bgr_o = ref_opts(A)
    Multiply = ref.multiply.Multiply
    m = Multiply.__new__(Multiply)
    torch.nn.Module.__init__(m)
    m.using_nerfacc = True
    m.use_person_encoder = False
    m.with_bkgd = True
    m.sdf_bounding_sphere = 3.0
    m.foreground_implicit_network_list = torch.nn.ModuleList()
    m.foreground_rendering_network_list = torch.nn.ModuleList()
    m.deformer_list = torch.nn.ModuleList()
    for person in scene["persons"]:
        net = ref.networks.ImplicitNet(imp_o)
        net.load_state_dict(person["implicit"], strict=True)
        m.foreground_implicit_network_list.append(net)
        rn = ref.networks.RenderingNet(ren_o)
        rn.load_state_dict(person["render"], strict=True)
        m.foreground_rendering_network_list.append(rn)
        D = ref.deformer.SMPLDeformer
        d = D.__new__(D)
        torch.nn.Module.__init__(d)
        d.max_dist, d.K = 0.05, 1
        d.smpl_verts = person["verts_c"][None]
        d.smpl_weights = person["weights"][None]
        m.deformer_list.append(d)
    m.bg_implicit_network = ref.networks.ImplicitNet(bgi_o)
    m.bg_implicit_network.load_state_dict(scene["bg_implicit"], strict=True)
    m.bg_rendering_network = ref.networks.RenderingNet(bgr_o)
    m.bg_rendering_network.load_state_dict(scene["bg_render"], strict=True)
    m.density = ref.density.LaplaceDensity(params_init={"beta": scene["beta_param"]}, beta_min=0.0001)
    m.bg_density = ref.density.AbsDensity()
    c = scene["cfg"]
    m.ray_sampler = ref.ray_sampler.ErrorBoundSampler(
        3.0, inverse_sphere_bg=True, near=c["near"], N_samples=c["N_samples"],
        N_samples_eval=c["N_samples_eval"], N_samples_extra=c["N_samples_extra"], eps=c["eps"],
        beta_iters=c["beta_iters"], max_total_iters=c["max_total_iters"],
        N_samples_inverse_sphere=32, add_tiny=c["add_tiny"])
    m.eval()
    return m


def ref_forward(ref, m, scene, inputs, hit_lists):
    """Eval branch of Multiply.forward driven with the reference's own objects."""
    Multiply = ref.multiply.Multiply
    torch.set_grad_enabled(True)
    ray_dirs, cam_loc = ref.rend_util.get_camera_params(inputs["uv"], inputs["pose"], inputs["intrinsics"])
    _, num_pixels, _ = ray_dirs.shape
    cam_loc = cam_loc.unsqueeze(1).repeat(1, num_pixels, 1).reshape(-1, 3)
    ray_dirs = ray_dirs.reshape(-1, 3)
    P = len(scene["persons"])
    fg_rgb_list, normal_values_list, sdf_output_list, z_vals_list, person_id_list, z_max_list = [], [], [], [], [], []
    index_ray_box_list = []
    trips = []
    # count sampler trips by wrapping the sdf function
    for person_id in range(P):
        person = scene["persons"][person_id]
        index_ray_box = hit_lists[person_id]
        if len(index_ray_box) == 0:
            index_ray_box = torch.tensor([0])
        index_ray_box = index_ray_box.long()
        cam_i, dir_i = cam_loc[index_ray_box], ray_dirs[index_ray_box]
        index_ray_box_list.append(index_ray_box)
        cond = {"smpl": person["smpl_pose"][:, 3:] / np.pi}
        smpl_tfs = person["tfs"][None]
        smpl_verts = person["verts_p"][None]
        calls = [0]
        orig = Multiply.sdf_func_with_smpl_deformer

        def counting(self, *a, **k):
            calls[0] += 1
            return orig(self, *a, **k)
        m.sdf_func_with_smpl_deformer = counting.__get__(m)
        z_vals, _ = m.ray_sampler.get_z_vals(dir_i, cam_i, m, cond, smpl_tfs, eval_mode=True,
                                             smpl_verts=smpl_verts, person_id=person_id)
        del m.sdf_func_with_smpl_deformer
        m.eval()        # the sampler leaves the implicit net in train(); no numeric effect (SURVEY §8c)
        trips.append(calls[0])
        z_vals, z_vals_bg = z_vals
        z_max = z_vals[:, -1]
        z_vals = z_vals[:, :-1]
        N_samples = z_vals.shape[1]
        npx = cam_i.shape[0]
        points = cam_i.unsqueeze(1) + z_vals.unsqueeze(2) * dir_i.unsqueeze(1)
        points_flat = points.reshape(-1, 3)
        dirs = dir_i.unsqueeze(1).repeat(1, N_samples, 1)
        sdf_output, canonical_points, feature_vectors = m.sdf_func_with_smpl_deformer(
            points_flat, cond, smpl_tfs, smpl_verts=smpl_verts, person_id=person_id)
        differentiable_points = canonical_points.reshape(npx, N_samples, 3).reshape(-1, 3)
        sdf_output = sdf_output.reshape(npx, N_samples, 1).reshape(-1, 1)
        sdf_output_list.append(sdf_output.reshape(npx, N_samples).detach())
        view = -dirs.reshape(-1, 3)
        fg_rgb_flat, others = m.get_rbg_value(points_flat, differentiable_points, view, cond, smpl_tfs,
                                              feature_vectors=feature_vectors, person_id=person_id,
                                              is_training=False)
        fg_rgb_list.append(fg_rgb_flat.detach().reshape(-1, N_samples, 3))
        normal_values_list.append(others["normals"].detach().reshape(-1, N_samples, 3))
        z_max_list.append(z_max)
        z_vals_list.append(z_vals)
        person_id_list.append(torch.ones(npx, N_samples) * person_id)

    # multiply.py:427-480 with the nerfacc restatements of oracle/port.py
    fg_rgb, normal, acc, acc_p, bg_T = port.composite_nerfacc(
        index_ray_box_list, z_vals_list, z_max_list, sdf_output_list, fg_rgb_list, normal_values_list,
        list(range(P)), cam_loc.shape[0], scene["beta_param"])
    # multiply.py:482-484, 514-539
    z_vals_bg = m.ray_sampler.inverse_sphere_sampler.get_z_vals(ray_dirs, cam_loc, m)
    z_vals_bg = z_vals_bg * (1. / m.ray_sampler.scene_bounding_sphere)
    N_bg = z_vals_bg.shape[1]
    z_vals_bg = torch.flip(z_vals_bg, dims=[-1, ])
    bg_dirs = ray_dirs.unsqueeze(1).repeat(1, N_bg, 1)
    bg_locs = cam_loc.unsqueeze(1).repeat(1, N_bg, 1)
    bg_points = m.depth2pts_outside(bg_locs, bg_dirs, z_vals_bg)
    frame_latent_code = scene["frame_code"]
    with torch.no_grad():
        bg_output = m.bg_implicit_network(bg_points.reshape(-1, 4), {"frame": frame_latent_code})[0]
        bg_sdf = bg_output[:, :1]
        bg_feat = bg_output[:, 1:]
        bg_ro = m.bg_rendering_network(None, None, bg_dirs.reshape(-1, 3), None, bg_feat, frame_latent_code)
        bg_rgb = bg_ro.reshape(-1, N_bg, 3)
        bg_weights = m.bg_volume_rendering(z_vals_bg, bg_sdf)
        bg_rgb_values = torch.sum(bg_weights.unsqueeze(-1) * bg_rgb, 1)
    rgb_values = fg_rgb + bg_T.unsqueeze(-1) * bg_rgb_values
    return dict(acc_map=acc, acc_person_list=acc_p, rgb_values=rgb_values,
                fg_rgb_values=fg_rgb + bg_T.unsqueeze(-1) * torch.ones_like(fg_rgb),
                normal_values=normal, bg_T=bg_T, bg_rgb=bg_rgb_values,
                z_vals=z_vals_list, sdf=sdf_output_list, rgb=fg_rgb_list, normals=normal_values_list,
                trips=trips)


def save(name, **arrs):
    out = {}
    for k, v in arrs.items():
        if isinstance(v, torch.Tensor):
            v = v.detach().numpy()
        out[k] = np.asarray(v)
    os.makedirs(GOLD, exist_ok=True)
    np.savez_compressed(os.path.join(GOLD, name + ".npz"), **out)
    print("wrote", name, {k: v.shape for k, v in out.items()})


def main():
    torch.set_num_threads(8)
    ref = ref_shim.load()
    A = ref.AttrDict
    scene = S.make_scene(P=2, S=64, seed=42)
    m = build_ref_model(ref, scene)
    g = torch.Generator().manual_seed(5)

    # ---- op-level vectors -----------------------------------------------------------
    p0 = scene["persons"][0]
    x = (torch.rand(256, 3, generator=g) - 0.5) * 2.0
    cond = {"smpl": p0["cond"]}
    with torch.no_grad():
        y = m.foreground_implicit_network_list[0](x, cond, person_id=0)[0]
    save("implicit_fg", x=x, out=y)

    xg = x[:64].clone().requires_grad_(True)
    out = m.foreground_implicit_network_list[0](xg, cond, person_id=0)[0]
    grad = torch.autograd.grad(out[:, 0].sum(), xg)[0]
    save("implicit_fg_grad", x=x[:64], grad=grad)

    nrm = torch.nn.functional.normalize(torch.randn(256, 3, generator=g), dim=1)
    with torch.no_grad():
        rgb = m.foreground_rendering_network_list[0](x, nrm, None, p0["cond"], y[:, 1:], person_id=0)
    save("render_fg", x=x, normals=nrm, feat=y[:, 1:], rgb=rgb)

    x4 = torch.nn.functional.normalize(torch.randn(256, 3, generator=g), dim=1)
    x4 = torch.cat([x4, torch.rand(256, 1, generator=g) / 3.0], 1)
    vd = torch.nn.functional.normalize(torch.randn(256, 3, generator=g), dim=1)
    with torch.no_grad():
        yb = m.bg_implicit_network(x4, {"frame": scene["frame_code"]})[0]
        rb = m.bg_rendering_network(None, None, vd, None, yb[:, 1:], scene["frame_code"])
    save("bg_nets", x=x4, view=vd, out=yb, rgb=rb)

    sdfv = torch.linspace(-0.5, 4.0, 200)
    save("density", sdf=sdfv, sigma=m.density(sdfv).detach(),
         sigma_b=m.density(sdfv, beta=torch.tensor(0.013)).detach(), beta=m.density.get_beta().detach())

    # deformer: points around the posed body
    vp = p0["verts_p"]
    pts = vp[torch.randint(0, vp.shape[0], (512,), generator=g)] + 0.06 * torch.randn(512, 3, generator=g)
    xc, outl = m.deformer_list[0].forward(pts, p0["tfs"][None], return_weights=False, inverse=True,
                                          smpl_verts=vp[None])
    xd = m.deformer_list[0].forward_skinning(xc[None], None, p0["tfs"][None])[0]
    save("deformer", pts=pts, x_c=xc, outlier=outl, x_d=xd)

    # ---- SMPL linear blend skinning: the reference's own lib/smpl/lbs.py on a synthetic SMPL-shaped model ----
    sm = S.make_smpl_model(300)
    betas = 0.5 * torch.randn(1, 10, generator=g)
    pose = 0.3 * torch.randn(1, 72, generator=g)
    verts, _, _, _, A = ref.lbs.lbs(betas, pose, sm["v_template"][None], sm["shapedirs"], sm["posedirs"],
                                    sm["J_regressor"], sm["parents"], sm["lbs_weights"], dtype=torch.float32)
    save("smpl_lbs", betas=betas, pose=pose, verts=verts[0], A=A[0])

    # ---- sampler + full forward -----------------------------------------------------
    for case in FORWARD_CASES:
        forward_case(ref, *case)
    rays_case(ref)
    grid_case(ref)
    train_sampler_case(ref)
    train_forward_case(ref)
    trained_case(ref)


def trained_case(ref):
    """ImplicitNet forward (sdf, features), its autograd grad sdf and RenderingNet RGB of the unmodified reference
    modules at the trained-like parameters of scene.perturb_networks (non-zero Fourier columns, g != ||v||_row, hidden
    biases), on points over the canonical box and near the body."""
    sc = S.make_scene(P=2, S=64, seed=42, weights="trained")
    m = build_ref_model(ref, sc)
    p0 = sc["persons"][0]
    g = torch.Generator().manual_seed(11)
    vc = p0["verts_c"]
    x = torch.cat([(torch.rand(128, 3, generator=g) - 0.5) * 2.0,
                   vc[torch.randint(0, vc.shape[0], (128,), generator=g)] + 0.03 * torch.randn(128, 3, generator=g)])
    xg = x.clone().requires_grad_(True)
    out = m.foreground_implicit_network_list[0](xg, {"smpl": p0["cond"]}, person_id=0)[0]
    grad = torch.autograd.grad(out[:, 0].sum(), xg)[0]
    nrm = torch.nn.functional.normalize(grad, dim=1)
    with torch.no_grad():
        rgb = m.foreground_rendering_network_list[0](x, nrm, None, p0["cond"], out[:, 1:].detach(), person_id=0)
    save("implicit_fg_trained", x=x, out=out, grad=grad, normals=nrm, rgb=rgb)


def train_sampler_case(ref):
    """ErrorBoundSampler.get_z_vals in TRAINING mode (model.training: stratified start samples, random final
    abscissae, randperm extras, randint eikonal pick, jittered inverse-sphere samples; ray_sampler.py:32-40,171,202,
    212-218; the SDF callback does not clamp outliers, multiply.py:142).  Every random tensor the reference draws is
    recorded in draw order so that the port and the CUDA sampler can be fed the same numbers."""
    sc = S.make_scene(P=2, S=16, seed=42)
    m = build_ref_model(ref, sc)
    m.train()
    inputs = S.make_rays(sc, 40, seed=21, region="boxes")
    hits = S.make_hit_lists(sc, inputs)
    ray_dirs, cam_loc = ref.rend_util.get_camera_params(inputs["uv"], inputs["pose"], inputs["intrinsics"])
    cam_loc = cam_loc.unsqueeze(1).repeat(1, ray_dirs.shape[1], 1).reshape(-1, 3)
    ray_dirs = ray_dirs.reshape(-1, 3)
    pid = 0
    person = sc["persons"][pid]
    idx = hits[pid].long()
    draws = []
    orig = (torch.rand, torch.randperm, torch.randint)

    def rec(fn, tag):
        def w(*a, **k):
            out = fn(*a, **k)
            draws.append((tag, out.clone()))
            return out
        return w
    torch.rand, torch.randperm, torch.randint = rec(orig[0], "rand"), rec(orig[1], "randperm"), rec(orig[2], "randint")
    try:
        torch.manual_seed(1234)
        (z_vals, z_bg), z_eik = m.ray_sampler.get_z_vals(ray_dirs[idx], cam_loc[idx], m, {"smpl": person["cond"]},
                                                         person["tfs"][None], eval_mode=False,
                                                         smpl_verts=person["verts_p"][None], person_id=pid)
    finally:
        torch.rand, torch.randperm, torch.randint = orig
    tags = [t for t, _ in draws]
    assert tags == ["rand", "rand", "randperm", "randint", "rand"], tags
    save("sampler_train", hits=idx, t_rand=draws[0][1], u_final=draws[1][1], extra_perm=draws[2][1],
         eik_idx=draws[3][1], t_rand_bg=draws[4][1], z_vals=z_vals, z_bg=z_bg, z_eik=z_eik, uv=inputs["uv"])


def train_forward_case(ref):
    """The TRAINING branch of Multiply.forward (multiply.py:174-598 with self.training, shipped loss weights, epoch >= 250)
    driven line by line with the reference's own objects, as ref_forward does for the eval branch: per person
    get_z_vals(training) -> sdf_func_with_smpl_deformer (no outlier clamp) -> eikonal samples and gradients
    (:320-331) -> get_rbg_value(is_training=True); then the nerfacc block, the second inverse-sphere draw (:482) and
    the background.  Every random tensor drawn on the way is recorded in draw order."""
    Multiply = ref.multiply.Multiply
    sc = S.make_scene(P=2, S=16, seed=42)
    m = build_ref_model(ref, sc)
    m.train()
    inputs = S.make_rays(sc, 40, seed=33, region="boxes")
    hits = S.make_hit_lists(sc, inputs)
    ray_dirs, cam_loc = ref.rend_util.get_camera_params(inputs["uv"], inputs["pose"], inputs["intrinsics"])
    R = ray_dirs.shape[1]
    cam_loc = cam_loc.unsqueeze(1).repeat(1, R, 1).reshape(-1, 3)
    ray_dirs = ray_dirs.reshape(-1, 3)
    draws = []
    orig = (torch.rand, torch.randperm, torch.randint, torch.randn_like)

    def rec(fn, tag):
        def w(*a, **k):
            out = fn(*a, **k)
            draws.append((tag, out.clone()))
            return out
        return w
    torch.rand, torch.randperm, torch.randint, torch.randn_like = (rec(orig[0], "rand"), rec(orig[1], "randperm"),
                                                                  rec(orig[2], "randint"), rec(orig[3], "randn_like"))
    out = {}
    try:
        torch.manual_seed(4321)
        torch.set_grad_enabled(True)
        fg_rgb_list, nrm_list, sdf_list, z_list, zmax_list, idx_list, grad_theta_list, z_eik_list = [], [], [], [], [], [], [], []
        for pid in range(2):
            person = sc["persons"][pid]
            idx = hits[pid].long()
            cam_i, dir_i = cam_loc[idx], ray_dirs[idx]
            cond = {"smpl": person["smpl_pose"][:, 3:] / np.pi}
            smpl_tfs, smpl_verts = person["tfs"][None], person["verts_p"][None]
            (z_vals, _), z_eik = m.ray_sampler.get_z_vals(dir_i, cam_i, m, cond, smpl_tfs, eval_mode=False,
                                                          smpl_verts=smpl_verts, person_id=pid)
            z_max, z_vals = z_vals[:, -1], z_vals[:, :-1]
            N = z_vals.shape[1]
            npx = cam_i.shape[0]
            pts = (cam_i.unsqueeze(1) + z_vals.unsqueeze(2) * dir_i.unsqueeze(1)).reshape(-1, 3)
            sdf_output, canonical_points, feature_vectors = m.sdf_func_with_smpl_deformer(pts, cond, smpl_tfs,
                                                                                         smpl_verts=smpl_verts, person_id=pid)
            # multiply.py:320-331 (smpl_server_list[pid].verts_c = the deformer's canonical vertices)
            smpl_verts_c = person["verts_c"][None]
            indices = torch.randperm(smpl_verts_c.shape[1])[:512]
            verts_c = torch.index_select(smpl_verts_c, 1, indices)
            sample = ref.sampler_cls().get_points(verts_c, global_ratio=0.)
            sample.requires_grad_()
            local_pred = m.foreground_implicit_network_list[pid](sample, cond, person_id=pid)[..., 0:1]
            grad_theta_list.append(Multiply_gradient(ref, sample, local_pred).detach())
            dirs = dir_i.unsqueeze(1).repeat(1, N, 1)
            fg_rgb_flat, others = m.get_rbg_value(pts, canonical_points.reshape(-1, 3), -dirs.reshape(-1, 3), cond, smpl_tfs,
                                                  feature_vectors=feature_vectors, person_id=pid, is_training=True)
            fg_rgb_list.append(fg_rgb_flat.detach().reshape(-1, N, 3))
            nrm_list.append(others["normals"].detach().reshape(-1, N, 3))
            sdf_list.append(sdf_output.detach().reshape(npx, N))
            z_list.append(z_vals)
            zmax_list.append(z_max)
            idx_list.append(idx)
            z_eik_list.append(z_eik)
        fg_rgb, normal, acc, acc_p, bg_T = port.composite_nerfacc(idx_list, z_list, zmax_list, sdf_list, fg_rgb_list, nrm_list,
                                                                 [0, 1], R, sc["beta_param"])
        z_vals_bg = m.ray_sampler.inverse_sphere_sampler.get_z_vals(ray_dirs, cam_loc, m)          # multiply.py:482
        z_vals_bg = z_vals_bg * (1. / m.ray_sampler.scene_bounding_sphere)
        z_vals_bg = torch.flip(z_vals_bg, dims=[-1, ])
        N_bg = z_vals_bg.shape[1]
        bg_dirs = ray_dirs.unsqueeze(1).repeat(1, N_bg, 1)
        bg_locs = cam_loc.unsqueeze(1).repeat(1, N_bg, 1)
        bg_points = m.depth2pts_outside(bg_locs, bg_dirs, z_vals_bg)
        with torch.no_grad():
            bg_output = m.bg_implicit_network(bg_points.reshape(-1, 4), {"frame": sc["frame_code"]})[0]
            bg_ro = m.bg_rendering_network(None, None, bg_dirs.reshape(-1, 3), None, bg_output[:, 1:], sc["frame_code"])
            bg_weights = m.bg_volume_rendering(z_vals_bg, bg_output[:, :1])
            bg_rgb_values = torch.sum(bg_weights.unsqueeze(-1) * bg_ro.reshape(-1, N_bg, 3), 1)
        rgb_values = fg_rgb + bg_T.unsqueeze(-1) * bg_rgb_values
        out = dict(rgb_values=rgb_values, normal_values=normal, acc_map=acc, acc_person_list=acc_p,
                   grad_theta=torch.cat(grad_theta_list, dim=1), uv=inputs["uv"])
        for pid in range(2):
            out[f"hits_{pid}"] = idx_list[pid]
            out[f"z_vals_{pid}"] = z_list[pid]
            out[f"sdf_{pid}"] = sdf_list[pid]
            out[f"z_eik_{pid}"] = z_eik_list[pid]
    finally:
        torch.rand, torch.randperm, torch.randint, torch.randn_like = orig
    tags = [t for t, _ in draws]
    per = ["rand", "rand", "randperm", "randint", "rand", "randperm", "randn_like", "rand"]
    assert tags == per + per + ["rand"], tags
    for pid in range(2):
        d = draws[8 * pid: 8 * pid + 8]
        out[f"t_rand_{pid}"], out[f"u_final_{pid}"], out[f"extra_perm_{pid}"] = d[0][1], d[1][1], d[2][1]
        out[f"eik_idx_{pid}"], out[f"t_rand_bg_sampler_{pid}"] = d[3][1], d[4][1]
        out[f"eik_perm_{pid}"], out[f"eik_noise_{pid}"] = d[5][1], d[6][1]
    out["t_rand_bg"] = draws[16][1]
    save("forward_train", **out)


def Multiply_gradient(ref, inputs, outputs):
    """multiply.py:728-738 (module-level `gradient`)."""
    return ref.multiply.gradient(inputs, outputs)


def grid_case(ref):
    """Multiply.query_oc (multiply.py:169-172) on the dense lattice of generate_mesh (lib/utils/mesh.py:78-105; the
    point mapping of :92-95 is restated here because generate_mesh itself needs the compiled MISE extension)."""
    sc = S.make_scene(P=2, S=64, seed=42)
    m = build_ref_model(ref, sc)
    p1 = sc["persons"][1]
    res = 12
    center, extent, scale = port.mesh_bounds(p1["verts_c"])
    idx = np.stack(np.meshgrid(np.arange(res + 1), np.arange(res + 1), np.arange(res + 1), indexing="ij"), -1).reshape(-1, 3)
    pts = idx.astype(np.float32)
    pts = (pts / res - 0.5) * scale
    pts = pts * extent + center
    with torch.no_grad():
        occ = ref.multiply.Multiply.query_oc(m, torch.tensor(pts).float(), {"smpl": p1["cond"]}, 1)["occ"]
    save("sdf_grid", res=np.array(res), center=center, extent=np.array(extent), points=pts, occ=occ[:, 0])


def rays_case(ref):
    """rend_util.get_camera_params (:45-72, quaternion and matrix poses are both 4x4 here) with a skewed, off-centre
    intrinsic matrix and a rotated camera, and get_sphere_intersections (:131-147) at r = 3 (multiply.py:85)."""
    g = torch.Generator().manual_seed(77)
    R = 300
    uv = torch.rand(1, R, 2, generator=g) * 512.0
    K = torch.eye(4)[None].clone()
    K[0, 0, 0], K[0, 1, 1], K[0, 0, 2], K[0, 1, 2], K[0, 0, 1] = 880.0, 910.0, 250.0, 262.0, 3.5
    ax = torch.nn.functional.normalize(torch.randn(3, generator=g), dim=0)
    ang = 0.4
    Kx = torch.tensor([[0, -ax[2], ax[1]], [ax[2], 0, -ax[0]], [-ax[1], ax[0], 0]])
    Rm = torch.eye(3) + np.sin(ang) * Kx + (1 - np.cos(ang)) * (Kx @ Kx)
    pose = torch.eye(4)[None].clone()
    pose[0, :3, :3] = Rm
    pose[0, :3, 3] = torch.tensor([0.3, -0.2, 2.2])
    dirs, cam = ref.rend_util.get_camera_params(uv, pose, K)
    cam_r = cam.unsqueeze(1).repeat(1, R, 1).reshape(-1, 3)
    nf = ref.rend_util.get_sphere_intersections(cam_r, dirs.reshape(-1, 3), r=3.0)
    save("rays", uv=uv, pose=pose, intrinsics=K, ray_dirs=dirs, cam_loc=cam, near_far=nf)


# (name, persons, N_samples, rays, ray region, scene seed)
FORWARD_CASES = (("forward_S64_R48", 2, 64, 48, "boxes", 42), ("forward_S16_R96", 2, 16, 96, "image", 42),
                 ("forward_P3_S32_R40", 3, 32, 40, "boxes", 7))


def forward_case(ref, name, P, Sn, R, region, seed):
    """The reference's own sampler / deformer / networks / density objects driven through the eval branch of
    Multiply.forward on a synthetic scene; everything the parity tests compare is stored."""
    sc = S.make_scene(P=P, S=Sn, seed=seed)
    mm = build_ref_model(ref, sc)
    inputs = S.make_rays(sc, R, seed=1234, region=region)
    hits = S.make_hit_lists(sc, inputs)
    o = ref_forward(ref, mm, sc, inputs, hits)
    flat = {k: v for k, v in o.items() if isinstance(v, torch.Tensor)}
    for p in range(P):
        flat[f"z_vals_{p}"] = o["z_vals"][p]
        flat[f"sdf_{p}"] = o["sdf"][p]
        flat[f"rgb_{p}"] = o["rgb"][p]
        flat[f"normals_{p}"] = o["normals"][p]
        flat[f"hits_{p}"] = hits[p]
    flat["trips"] = np.array(o["trips"])
    flat["uv"] = inputs["uv"]
    save(name, **flat)


if __name__ == "__main__":
    import sys
    if len(sys.argv) > 2 and sys.argv[1] == "--only":      # regenerate single forward fixtures, e.g. --only forward_P3_S32_R40
        torch.set_num_threads(8)
        _ref = ref_shim.load()
        for case in FORWARD_CASES:
            if case[0] in sys.argv[2:]:
                forward_case(_ref, *case)
        if "rays" in sys.argv[2:]:
            rays_case(_ref)
        if "sdf_grid" in sys.argv[2:]:
            grid_case(_ref)
        if "sampler_train" in sys.argv[2:]:
            train_sampler_case(_ref)
        if "forward_train" in sys.argv[2:]:
            train_forward_case(_ref)
        if "implicit_fg_trained" in sys.argv[2:]:
            trained_case(_ref)
    else:
        main()
