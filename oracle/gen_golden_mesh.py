"""TEST INFRASTRUCTURE ONLY — generate tests/golden/forward_train_early.npz: the reference's training branch at
current_epoch < 250, where Multiply.forward tests every canonical sample against the person's canonical mesh
(check_off_in_surface_points_cano_mesh, multiply.py:153-167, :313-316) and merges the flags (:549-560).  Runs only in
the build container (the GPU box has no /root/reference).

    python -m oracle.gen_golden_mesh

Everything else is gen_golden.py's: the reference modules load under oracle/ref_shim.py and the training branch is
driven line by line (Multiply.forward itself needs trimesh and the SMPL pkl).  kaolin is absent, so its two functions
in the shim's stub modules are bound to the definitions of oracle/mesh_port.py before the reference calls them; the
reference's own check_off_in_surface_points_cano_mesh (sqrt, sign, reshape, min, the two comparisons) runs unmodified.

The fixture holds everything forward_train.npz holds, the canonical points of each person's main pass, the per-ray
minimum of the signed distance per person (which rays sit on a threshold), the per-person flags and the merged
index_off_surface / index_in_surface.
"""
import sys

import numpy as np
import torch

from oracle import mesh_port, port, ref_shim
from oracle.gen_golden import build_ref_model, save, Multiply_gradient
from multiply_b200 import scene as S


def load_ref():
    """The reference modules with kaolin's point_to_mesh_distance / check_sign / index_vertices_by_faces bound to
    oracle/mesh_port.py (the stub modules of ref_shim have no implementations)."""
    ref = ref_shim.load()
    sys.modules["kaolin.metrics.trianglemesh"].point_to_mesh_distance = mesh_port.point_to_mesh_distance
    sys.modules["kaolin.ops.mesh"].check_sign = mesh_port.check_sign
    sys.modules["kaolin.ops.mesh"].index_vertices_by_faces = mesh_port.index_vertices_by_faces
    ref.multiply.index_vertices_by_faces = mesh_port.index_vertices_by_faces     # imported by name, multiply.py:18
    return ref


def train_early_case(ref, name="forward_train_early", epoch=137, ray_seed=35, torch_seed=4322):
    """The TRAINING branch of Multiply.forward (multiply.py:174-598 with self.training, shipped loss weights) at an epoch
    < 250 driven line by line with the reference's own objects, as gen_golden.train_forward_case does at epoch >= 250:
    per person get_z_vals(training) -> sdf_func_with_smpl_deformer (no outlier clamp) -> the reference's
    check_off_in_surface_points_cano_mesh on the canonical points (:313-316) -> eikonal samples and gradients
    (:320-331) -> get_rbg_value(is_training=True); then the nerfacc block, the second inverse-sphere draw (:482), the
    background and the merge of the surface flags (:549-560).  Every random tensor drawn on the way is recorded in draw
    order.  The canonical meshes are scene.make_body_mesh's (the SMPL pkl's faces are licence-gated), assigned to the
    model's mesh_*_list as Multiply.__init__ does (:118-121).  137 is neither < 20 nor a multiple of 20, so the pose
    conditioning is not zeroed (:271-273)."""
    assert epoch < 250
    import kaolin          # the stub module of ref_shim, its functions bound by load_ref
    sc = S.make_scene(P=2, S=16, seed=42)
    m = build_ref_model(ref, sc)
    m.train()
    m.threshold = 0.05
    m.mesh_v_cano_list, m.mesh_f_cano_list, m.mesh_face_vertices_list = [], [], []
    for pid in range(2):
        v, f = S.make_body_mesh(100 + pid)
        m.mesh_v_cano_list.append(v[None])
        m.mesh_f_cano_list.append(f)
        m.mesh_face_vertices_list.append(mesh_port.index_vertices_by_faces(v[None], f))
    off_list, in_list = [], []
    inputs = S.make_rays(sc, 40, seed=ray_seed, region="boxes")
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
        torch.manual_seed(torch_seed)
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
            o_p, i_p = m.check_off_in_surface_points_cano_mesh(canonical_points, N, person_id=pid,
                                                               threshold=m.threshold)
            off_list.append(o_p)
            in_list.append(i_p)
            # the minimum signed distance per ray, the same lines (:155-164) spelled out: which rays sit on a
            # threshold
            xc = canonical_points.detach()
            dist, _, _ = kaolin.metrics.trianglemesh.point_to_mesh_distance(xc.unsqueeze(0).contiguous(), m.mesh_face_vertices_list[pid])
            sgn = 1 - 2 * kaolin.ops.mesh.check_sign(m.mesh_v_cano_list[pid], m.mesh_f_cano_list[pid], xc.unsqueeze(0)).float()
            out[f"min_signed_{pid}"] = torch.min((sgn * torch.sqrt(dist)).reshape(npx, N, 1), 1)[0][:, 0]
            out[f"x_cano_{pid}"] = xc
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
        out.update(rgb_values=rgb_values, normal_values=normal, acc_map=acc, acc_person_list=acc_p,
                   grad_theta=torch.cat(grad_theta_list, dim=1), uv=inputs["uv"])
        index_off_surface = torch.tensor(np.ones((R, 2)), dtype=torch.bool)  # multiply.py:549-560 (using_nerfacc)
        index_in_surface = torch.tensor(np.zeros((R, 2)), dtype=torch.bool)
        for p, (ray_index, index_off, index_in) in enumerate(zip(idx_list, off_list, in_list)):
            index_off_surface[ray_index, p] = index_off
            index_in_surface[ray_index, p] = index_in
            out[f"off_{p}"], out[f"in_{p}"] = index_off, index_in
        out["index_off_surface"] = torch.all(index_off_surface, dim=1)
        out["index_in_surface"] = torch.any(index_in_surface, dim=1)
        out["epoch"] = np.array(epoch)
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
    save(name, **out)




if __name__ == "__main__":
    torch.set_num_threads(8)
    train_early_case(load_ref())
