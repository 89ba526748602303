"""TEST INFRASTRUCTURE ONLY — generate tests/golden/opt_depth.npz: opt_depth's two geometric losses and their vertex
gradients, computed by the reference's own code in float64, which pin oracle/opt_depth.py (and, through it, what the
device drop-ins are asked to reproduce).

    python -m oracle.gen_golden_opt_depth

Runs only where the reference tree is present.  What runs:
  * the camera: MultiplyModel.get_renderer's lines (multiply_model.py:553-571) with cv2.decomposeProjectionMatrix on a
    Hi4D-style P = world_mat @ scale_mat, smpl scale s = 1 / scale_mat[0,0];
  * MultiplyModel.get_interpenetration_loss (multiply_model.py:521-551), the function itself, taken from
    multiply_model.py with ``ast`` (importing the file needs Lightning), with kaolin.ops.mesh.check_sign bound to
    oracle/mesh_port.py and pytorch3d.ops.knn_points to oracle/port.py, ``.cuda()`` as the identity, in float64 with
    autograd; its randperm draws come from torch.manual_seed(PERM_SEED) and are stored;
  * the depth-order block of opt_depth (multiply_model.py:399-469), driven line by line as the reference writes it, on
    float64 depth maps of oracle/raster.py:depth_map (the renderer's layer 0, pytorch3d absent).
Two persons: scene.make_body_mesh(step=0.1) and the same mesh moved into it (they interpenetrate), seen by a camera
whose 48 x 64 image holds both.  Stored: the inputs, the camera (K, R, T as cv2 gives them), both losses and their
gradients with respect to every vertex of both persons.
"""
import ast
import os
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)

from multiply_b200 import scene as S      # noqa: E402
from oracle import mesh_port, port, raster as RA      # noqa: E402

REF = "/root/reference/code/multiply_model.py"
GOLD = os.path.join(ROOT, "tests", "golden", "opt_depth.npz")
H, W = 48, 64
PERM_SEED = 7
SAM_SEED = 3


def hi4d_P():
    """world_mat (K [R|t], 4x4) and scale_mat (diag(sc, sc, sc, 1) with a centre offset), as Hi4D's cameras.npz has."""
    K = np.array([[70.0, 0.4, 31.3], [0.0, 71.5, 24.6], [0.0, 0.0, 1.0]])
    th = 0.2
    R = np.array([[np.cos(th), 0, np.sin(th)], [0, 1, 0], [-np.sin(th), 0, np.cos(th)]]) @ np.diag([1.0, -1.0, -1.0])
    t = np.array([0.05, 0.1, 3.4])
    world = np.eye(4)
    world[:3, :4] = K @ np.concatenate([R, t[:, None]], 1)
    scale_mat = np.eye(4)
    scale_mat[:3, :3] *= 1.7
    scale_mat[:3, 3] = [0.02, -0.01, 0.03]
    return world, scale_mat


def get_renderer_camera(P, scale):
    """multiply_model.py:555-570 with cv2 (the Renderer construction at :573-576 needs pytorch3d)."""
    import cv2
    P_norm = np.eye(4)
    P_norm[:, :] = P[:, :]
    scale_eye = np.eye(4)
    scale_eye[0, 0] = scale
    scale_eye[1, 1] = scale
    scale_eye[2, 2] = scale
    P_norm = P_norm @ scale_eye
    out = cv2.decomposeProjectionMatrix(P_norm[:3, :])
    cam_intrinsics = out[0]
    render_R = out[1]
    cam_center = out[2]
    cam_center = (cam_center[:3] / cam_center[3])[:, 0]
    render_T = -render_R @ cam_center
    return cam_intrinsics, render_R, render_T


def reference_interpenetration_loss():
    """get_interpenetration_loss as the reference defines it, bound to the CPU definitions."""
    tree = ast.parse(open(REF).read())
    fn = next(n for n in ast.walk(tree) if isinstance(n, ast.FunctionDef) and n.name == "get_interpenetration_loss")
    mod = ast.Module(body=[fn], type_ignores=[])
    kaolin = types.SimpleNamespace(ops=types.SimpleNamespace(mesh=types.SimpleNamespace(check_sign=mesh_port.check_sign)))
    ops = types.SimpleNamespace(knn_points=port.knn_points)
    ns = dict(torch=torch, kaolin=kaolin, ops=ops)
    exec(compile(mod, REF, "exec"), ns)
    return lambda vertex_list, face_list: ns["get_interpenetration_loss"](None, vertex_list, face_list)


def sam_logits():
    g = torch.Generator().manual_seed(SAM_SEED)
    who = torch.randint(2, (H, W), generator=g)
    lg = torch.where(torch.stack([who == 0, who == 1], -1), 3.0, -4.0).double()
    lg[torch.rand(H, W, generator=g) < 0.1] = 3.0
    lg[..., 1] += 0.5 * (lg[..., 0] == lg[..., 1])
    return (lg + 0.1 * torch.randn(H, W, 2, generator=g, dtype=torch.float64))[None]


def reference_depth_block(renderer_depth_map, org_sam_mask):
    """multiply_model.py:399-469, line by line (the visualisation at :431-451 and the weights left out)."""
    sigmoid = torch.nn.Sigmoid()
    reshape_depth_map_list = []
    for map_id, depth_map_i in enumerate(renderer_depth_map):
        depth_map_i = depth_map_i[0, :, :, 0]
        reshape_depth_map_list.append(depth_map_i)
    max_depth_map_list = []
    max_depth = 999
    for map_id, depth_map_i in enumerate(reshape_depth_map_list):
        depth_map_processed = depth_map_i.clone()
        no_interaction = depth_map_processed < 0
        depth_map_processed[no_interaction] = max_depth
        max_depth_map_list.append(depth_map_processed)
    max_depth_map = torch.stack(max_depth_map_list, dim=-1)
    front_depth_map, _ = torch.min(max_depth_map, dim=-1)
    valid_mask = front_depth_map < max_depth
    sam_mask = org_sam_mask
    sam_mask = sigmoid(sam_mask)
    sam_mask = sam_mask.squeeze(0)
    valid_mask = torch.logical_and(valid_mask, sam_mask.sum(dim=-1) <= (1 + 1e-2))
    valid_mask = torch.logical_and(valid_mask, sam_mask.sum(dim=-1) >= (0.7))
    sam_mask_idx = torch.argmax(sam_mask, dim=-1)
    sam_mask_idx = sam_mask_idx.unsqueeze(-1)
    gt_depth_map = torch.gather(max_depth_map, dim=-1, index=sam_mask_idx)
    gt_depth_map = gt_depth_map.squeeze(-1)
    valid_mask = torch.logical_and(valid_mask, gt_depth_map < max_depth)
    valid_mask = valid_mask.flatten()
    gt_depth_map = gt_depth_map.flatten()[valid_mask]
    front_depth_map = front_depth_map.flatten()[valid_mask]
    exclude_mask = ~(gt_depth_map == front_depth_map)
    loss = torch.log(1 + torch.exp(gt_depth_map[exclude_mask] - front_depth_map[exclude_mask])).sum()
    return loss, int(exclude_mask.sum())


def main():
    assert os.path.exists(REF), "the reference tree is needed to generate this fixture"
    world, scale_mat = hi4d_P()
    P = world @ scale_mat
    s = 1.0 / scale_mat[0, 0]
    K, R, T = get_renderer_camera(P, s)
    cam = RA.camera_record(R, T, K)
    v0, f = S.make_body_mesh(step=0.1)
    v0 = torch.as_tensor(v0, dtype=torch.float32)
    v1 = v0 + torch.tensor([0.21, 0.03, 0.09])
    f = torch.as_tensor(f, dtype=torch.int64)
    verts = [v0, v1]
    faces = [f, f]
    logits = sam_logits()

    old_cuda, old_dtype = torch.Tensor.cuda, torch.get_default_dtype()
    torch.Tensor.cuda = lambda self, *a, **k: self
    torch.set_default_dtype(torch.float64)
    try:
        vl = [v.double()[None].requires_grad_(True) for v in verts]
        torch.manual_seed(PERM_SEED)
        i_loss = reference_interpenetration_loss()(vl, [x[None] for x in faces])
        i_grad = torch.autograd.grad(i_loss.sum(), vl)
        torch.manual_seed(PERM_SEED)
        perms = [torch.randperm(v.shape[0]) for v in verts]
        vd = [v.double().requires_grad_(True) for v in verts]
        dm = [RA.depth_map(cam, v, fc, H, W) for v, fc in zip(vd, faces)]
        d_loss, n_excl = reference_depth_block(dm, logits)
        d_grad = torch.autograd.grad(d_loss, vd)
    finally:
        torch.Tensor.cuda = old_cuda
        torch.set_default_dtype(old_dtype)
    assert n_excl > 0 and float(i_loss.detach()) > 0, n_excl
    np.savez_compressed(
        GOLD, P=P, scale=np.array([s]), K=K, R=R, T=T, H=np.array([H]), W=np.array([W]),
        verts0=v0.numpy(), verts1=v1.numpy(), faces=f.numpy().astype(np.int32), sam_logits=logits.numpy(),
        perm0=perms[0].numpy().astype(np.int32), perm1=perms[1].numpy().astype(np.int32),
        interp_loss=np.array([float(i_loss)]), interp_grad0=i_grad[0][0].numpy(), interp_grad1=i_grad[1][0].numpy(),
        depth_loss=np.array([float(d_loss)]), depth_n=np.array([n_excl]), depth_grad0=d_grad[0].numpy(),
        depth_grad1=d_grad[1].numpy())
    print("wrote %s: interpenetration %.6g, depth order %.6g over %d pixels" % (GOLD, float(i_loss.detach()), float(d_loss),
                                                                               n_excl))


if __name__ == "__main__":
    main()
