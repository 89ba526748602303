"""Times opt_depth's geometric-loss operators on the GPU with CUDA events after warm-up (DESIGN.md §3.8):

  * the depth map (mp_depth_raster) and its backward (mp_depth_raster_backward) at 1280 x 940 for two persons, with
    scene.make_body_mesh meshes at the default step (about 1.3 x 10^4 faces) and at step 0.005 (about 6 x 10^5);
  * the K=1 nearest-vertex search (mp_knn1) and its backward for 5120 queries against both partner sizes;
  * one whole geometric-loss step: two make_smpl_scene persons, SMPL forward -> posed canonical meshes -> depth maps,
    check_sign and knn_points -> oracle/opt_depth.py's two losses -> backward to scale, transl, thetas and betas.

    python scripts/bench_opt_depth.py [--iters 50]

Prints the card name and power limit with the numbers, one JSON line at the end."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from multiply_b200 import engine, scene as S                   # noqa: E402
from multiply_b200.model.render import Renderer                 # noqa: E402
from multiply_b200.utils import kaolin_ops, pytorch3d_ops       # noqa: E402
from oracle import opt_depth as OD                               # noqa: E402

H, W = 1280, 940


def timed(fn, iters):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:                # noqa: BLE001
        q = "%s (nvidia-smi: %s)" % (torch.cuda.get_device_name(0), e)
    return q


def camera(centre):
    K = np.array([[1400.0, 0.0, W / 2], [0.0, 1400.0, H / 2], [0.0, 0.0, 1.0]])
    r = Renderer(img_size=[H, W], cam_intrinsic=K)
    r.set_camera(torch.eye(3)[None], torch.tensor(-np.asarray(centre) + np.array([0.0, 0.0, 3.2]))[None].float())
    return r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a GPU"
    torch.cuda.set_device(0)
    info = card()
    print("card:", info)
    res = {"card": info}

    for step in (0.033, 0.005):
        v, f = S.make_body_mesh(step=step)
        v0, f0 = torch.as_tensor(v).cuda(), torch.as_tensor(f).cuda()
        persons = [(v0, f0), (v0 + torch.tensor([0.18, 0.02, 0.12], device="cuda"), f0)]
        r = camera(v0.mean(0).cpu().numpy())
        vs = [p[0].clone().requires_grad_(True) for p in persons]
        fwd = timed(lambda: [engine.DepthRaster.apply(r.cam, H, W, x.device, x.detach(), ff) for x, (_, ff) in
                             zip(vs, persons)], args.iters)
        outs = [engine.DepthRaster.apply(r.cam, H, W, x.device, x, ff)[0] for x, (_, ff) in zip(vs, persons)]
        covered = sum(int((o >= 0).sum()) for o in outs)
        g = [torch.randn(H, W, device="cuda") for _ in outs]
        bwd = timed(lambda: torch.autograd.grad(outs, vs, g, retain_graph=True), args.iters)
        key = "depth_F%d" % f0.shape[0]
        res[key] = dict(faces=int(f0.shape[0]), persons=2, covered_pixels=covered, forward_ms=fwd, backward_ms=bwd)
        print("depth map 2 persons x %d faces at %dx%d (%d pixels covered): forward %.3f ms, backward %.3f ms"
              % (f0.shape[0], H, W, covered, fwd, bwd))
        q = persons[0][0][torch.randperm(v0.shape[0], device="cuda")[:5120]][None].clone().requires_grad_(True)
        p2 = persons[1][0][None].clone().requires_grad_(True)
        kf = timed(lambda: pytorch3d_ops.knn_points(q.detach(), p2.detach()), args.iters)
        d, _, nn = pytorch3d_ops.knn_points(q, p2)
        gd, gn = torch.randn_like(d), torch.randn_like(nn)
        kb = timed(lambda: torch.autograd.grad([d, nn], [q, p2], [gd, gn], retain_graph=True), args.iters)
        res["knn_5120_N%d" % v0.shape[0]] = dict(forward_ms=kf, backward_ms=kb)
        print("knn K=1: 5120 queries x %d vertices: forward %.3f ms, backward %.3f ms" % (v0.shape[0], kf, kb))

    # one geometric-loss step of opt_depth
    sc, model, inp = S.make_smpl_scene(P=2)
    trans = inp["smpl_trans"].clone()
    trans[0, 1] = trans[0, 0] + torch.tensor([0.12, 0.03, 0.08])
    servers = model.smpl_server_list
    cano = [torch.as_tensor(s.mesh_verts_c, dtype=torch.float32).cuda() for s in servers]
    faces = [torch.as_tensor(s.faces, dtype=torch.int64).reshape(-1, 3).cuda() for s in servers]
    leaves = dict(scale=inp["smpl_params"][0, 0, 0].reshape(1).cuda().requires_grad_(True))
    for p in range(2):
        leaves["transl%d" % p] = trans[0, p].reshape(1, 3).cuda().requires_grad_(True)
        leaves["thetas%d" % p] = inp["smpl_pose"][0, p].reshape(1, 72).cuda().requires_grad_(True)
        leaves["betas%d" % p] = torch.zeros(1, 10, device="cuda", requires_grad=True)
    logits = torch.randn(1, H, W, 2, device="cuda") * 3
    with torch.no_grad():
        centre = torch.cat([servers[p](leaves["scale"], leaves["transl%d" % p], leaves["thetas%d" % p],
                                       leaves["betas%d" % p])["smpl_verts"][0] for p in range(2)]).mean(0)
        r = camera((centre / leaves["scale"]).cpu().numpy())
    perms = [torch.randperm(c.shape[0]) for c in cano]

    def step():
        vs = []
        for p, srv in enumerate(servers):
            o = srv(leaves["scale"], leaves["transl%d" % p], leaves["thetas%d" % p], leaves["betas%d" % p])
            xd = model.get_deformed_mesh_fast_mode_multiple_person(cano[p], o["smpl_tfs"], p)
            vs.append((1 / leaves["scale"].squeeze()) * xd)
        dm = r.render_multiple_depth_map(vs, [f[None] for f in faces])
        d_loss, _ = OD.depth_order_loss(dm, logits)
        i_loss = OD.interpenetration_loss(vs, faces, kaolin_ops.check_sign, pytorch3d_ops.knn_points, perms)
        loss = 0.005 * d_loss + 0.0005 * i_loss.sum()
        torch.autograd.grad(loss, list(leaves.values()))
    st = timed(step, max(5, args.iters // 5))
    res["geometric_loss_step_ms"] = st
    res["geometric_loss_step_faces"] = [int(f.shape[0]) for f in faces]
    print("opt_depth geometric-loss step (2 persons, %s faces, %dx%d): %.3f ms" % ([int(f.shape[0]) for f in faces], H,
                                                                                   W, st))
    print(json.dumps(res))


if __name__ == "__main__":
    main()
