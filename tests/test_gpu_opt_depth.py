"""GPU: the K=1 nearest-vertex search (csrc/raster.cu, mp_knn1 / mp_knn1_backward) against oracle/port.py:knn_points'
definition, and opt_depth's geometric losses end to end on the device against the float64 port chain.

knn: raster.cu computes d2 = (dx*dx + dy*dy) + dz*dz in fp32 with every step rounded and keeps the lowest index on
ties, as the definition does, so dists and idx are compared bit for bit (the definition runs as torch ops on the
device here: at N1 = 10^5 x N2 = 3 x 10^5 the CPU would take minutes).  Its backward is a scatter of fp64 terms summed
per vertex in a fixed order: |err| <= C 2^-24 M per component with C = 4, M the sum of the |terms|.

End to end: two scene.make_smpl_scene persons translated into each other, their canonical body meshes posed by
Multiply.get_deformed_mesh_fast_mode_multiple_person, divided by the scale (multiply_model.py:390-393), through the new
Renderer, kaolin_ops.check_sign and pytorch3d_ops.knn_points into oracle/opt_depth.py's two losses, on a seeded SAM
logit map and seeded randperm draws.  The float64 port chain (port.smpl_server_forward, forward skinning with the
nearest canonical vertex's weights, oracle/raster.py:depth_map) runs the same loss code with the device's discrete
decisions (pix_to_face, inside, nearest vertex) held fixed, as the backward holds them, and its posed vertices carried
at the device's values (the depth loss's vertex gradients move by ~10^3 2^-24 when the vertices move by one fp32
rounding, so vertices that differ in the last bit cannot meet a tight gate; the posed vertices themselves are checked
against the float64 chain).  Gate: test_gpu_body_grad.py's SMPL gate, |err| <= 19 2^-24 max|want|, on the posed
vertices and on each loss's value and gradients.
"""
import numpy as np
import pytest
import torch

from multiply_b200 import _lib as L, scene as S
from oracle import opt_depth as OD, port, raster as RA

from _abi import padded, same, take
from _setups import dirty_workspace

gpu = pytest.mark.gpu
EPS = 2.0 ** -24
C_GATE = 4.0
C_SMPL = 19.0


def nearest_def(p1, p2):
    """port.knn_points' definition as torch ops on the device: (d2 [N1] fp32, idx [N1] int64)."""
    x, v = p1.cuda().float(), p2.cuda().float()
    d2 = torch.empty(x.shape[0], device="cuda")
    out = torch.empty(x.shape[0], dtype=torch.int64, device="cuda")
    ar = torch.arange(v.shape[0], device="cuda")
    step = max(1, (1 << 27) // max(v.shape[0], 1))
    for s in range(0, x.shape[0], step):
        xs = x[s:s + step]
        dx, dy, dz = xs[:, 0:1] - v[None, :, 0], xs[:, 1:2] - v[None, :, 1], xs[:, 2:3] - v[None, :, 2]
        d = dx * dx
        d = d + dy * dy
        d = d + dz * dz
        m = d.min(1, keepdim=True).values
        d2[s:s + step] = m[:, 0]
        out[s:s + step] = torch.where(d == m, ar[None], v.shape[0]).min(1).values
    return d2.cpu(), out.cpu()


def knn(p1, p2, ws=None):
    a, b = p1.float().cuda().contiguous(), p2.float().cuda().contiguous()
    N1, N2 = a.shape[0], b.shape[0]
    nb = L.call("mp_knn1_workspace_bytes", N1)
    ws = dirty_workspace(nb) if ws is None else ws
    d, i, nn = padded(N1), padded(N1, torch.int64), padded((N1, 3))
    L.call("mp_knn1", a, N1, b, N2, d, i, nn, ws, nb)
    return take(d, N1, "dists"), take(i, N1, "idx"), take(nn, (N1, 3), "nn")


def check_knn(p1, p2, what):
    d, i, nn = knn(p1, p2)
    rd, ri = nearest_def(p1, p2)
    print("%s: N1 = %d, N2 = %d" % (what, p1.shape[0], p2.shape[0]))
    assert same(d, rd), "%s: dists differ at %d queries" % (what, int((d != rd).sum()))
    assert torch.equal(i, ri), "%s: idx differs at %d queries" % (what, int((i != ri).sum()))
    assert same(nn, p2.float()[ri])
    return d, i, nn


@gpu
@pytest.mark.parametrize("N1,N2", [(1, 1), (5120, 10475), (5120, 300000), (100000, 300000), (37, 1025)])
def test_knn_random(N1, N2):
    g = torch.Generator().manual_seed(N1 + N2)
    p2 = torch.randn(N2, 3, generator=g) * 0.3
    p1 = p2[torch.randint(N2, (N1,), generator=g)] + 0.01 * torch.randn(N1, 3, generator=g)
    check_knn(p1, p2, "random")


@gpu
def test_knn_ties_and_duplicates():
    """Queries equidistant from several vertices (lattice points, dyadic coordinates), duplicate vertices across tile and
    chunk boundaries, queries equal to vertices, and a cloud where every query has many exact ties."""
    g = torch.Generator().manual_seed(3)
    lat = torch.stack(torch.meshgrid(*[torch.arange(12.0)] * 3, indexing="ij"), -1).reshape(-1, 3) * 0.25
    p2 = torch.cat([lat, lat[torch.randperm(lat.shape[0], generator=g)[:700]], lat])      # duplicates, later indices
    p1 = torch.cat([lat[:500] + 0.125, lat[:500], lat[:300] + torch.tensor([0.125, 0.0, 0.0]),
                    torch.rand(400, 3, generator=g) * 3])
    _, i, _ = check_knn(p1, p2, "ties")
    assert (i < lat.shape[0]).all()                                      # the first copy wins
    check_knn(torch.zeros(50, 3), torch.zeros(3000, 3), "all equal")


@gpu
def test_knn_workspace_and_refusals():
    p1, p2 = torch.randn(1000, 3), torch.randn(4000, 3)
    a = knn(p1, p2)
    b = knn(p1, p2, ws=torch.zeros(max(L.call("mp_knn1_workspace_bytes", 1000), 1), dtype=torch.uint8, device="cuda"))
    assert all(same(x, y) for x, y in zip(a, b))
    nb = L.call("mp_knn1_workspace_bytes", 1000)
    x, y = p1.cuda(), p2.cuda()
    d = torch.empty(1000, device="cuda")
    ws = dirty_workspace(nb + 256)
    with pytest.raises(L.MpError, match="workspace too small"):
        L.call("mp_knn1", x, 1000, y, 4000, d, None, None, ws, nb - 1)
    with pytest.raises(L.MpError, match="not 256-byte aligned"):
        L.call("mp_knn1", x, 1000, y, 4000, d, None, None, ws[4:], nb)
    with pytest.raises(L.MpError, match="N2 >= 1"):
        L.call("mp_knn1", x, 1000, y, 0, d, None, None, ws, nb)
    nbb = L.call("mp_knn1_backward_workspace_bytes", 1000, 4000)
    wsb = dirty_workspace(nbb)
    i = a[1].cuda()
    with pytest.raises(L.MpError, match="workspace too small"):
        L.call("mp_knn1_backward", x, 1000, y, 4000, i, d, None, torch.empty_like(x), torch.empty_like(y), wsb, nbb - 1)


def knn_backward(p1, p2, idx, d_d, d_nn):
    a, b = p1.float().cuda().contiguous(), p2.float().cuda().contiguous()
    N1, N2 = a.shape[0], b.shape[0]
    nb = L.call("mp_knn1_backward_workspace_bytes", N1, N2)
    ws = dirty_workspace(nb)
    g1, g2 = padded((N1, 3)), padded((N2, 3))
    L.call("mp_knn1_backward", a, N1, b, N2, idx.cuda(), None if d_d is None else d_d.float().cuda().contiguous(),
           None if d_nn is None else d_nn.float().cuda().contiguous(), g1, g2, ws, nb)
    return take(g1, (N1, 3), "d_p1"), take(g2, (N2, 3), "d_p2")


@gpu
@pytest.mark.parametrize("shared", [False, True])
def test_knn_backward(shared):
    g = torch.Generator().manual_seed(17)
    N2 = 20000
    p2 = torch.randn(N2, 3, generator=g) * 0.3
    N1 = 5120
    if shared:      # many queries share one nearest vertex: a tight cluster around p2[7] and p2[N2 - 1]
        p1 = torch.cat([p2[7] + 1e-4 * torch.randn(N1 // 2, 3, generator=g),
                        p2[N2 - 1] + 1e-4 * torch.randn(N1 - N1 // 2, 3, generator=g)])
    else:
        p1 = p2[torch.randint(N2, (N1,), generator=g)] + 0.01 * torch.randn(N1, 3, generator=g)
    _, idx, _ = knn(p1, p2)
    d_d, d_nn = torch.randn(N1, generator=g), torch.randn(N1, 3, generator=g)
    for dd, dn in ((d_d, d_nn), (d_d, None), (None, d_nn)):
        g1, g2 = knn_backward(p1, p2, idx, dd, dn)
        x = p1.double().requires_grad_(True)
        v = p2.double().requires_grad_(True)
        nn = v[idx]
        dist = ((x - nn) ** 2).sum(1)
        t1 = torch.zeros(N1, 3, dtype=torch.float64)
        t2 = torch.zeros(N1, 3, dtype=torch.float64)                  # each query's term to its vertex
        if dd is not None:
            t1 += 2 * (x - nn).detach() * dd.double()[:, None]
            t2 -= 2 * (x - nn).detach() * dd.double()[:, None]
        if dn is not None:
            t2 += dn.double()
        L_ = (0 if dd is None else (dist * dd.double()).sum()) + (0 if dn is None else (nn * dn.double()).sum())
        L_.backward()
        mag2 = torch.zeros(N2, 3, dtype=torch.float64).index_add_(0, idx, t2.abs())
        gx = torch.zeros_like(x) if x.grad is None else x.grad
        assert ((g1.double() - gx).abs() <= C_GATE * EPS * t1.abs()).all()
        err2 = (g2.double() - v.grad).abs()
        print("knn backward shared=%s: worst |err| / (2^-24 M) = %.3f" % (
            shared, float((err2 / mag2.clamp_min(1e-300))[mag2 > 0].max()) / EPS if (mag2 > 0).any() else 0.0))
        assert (err2 <= C_GATE * EPS * mag2).all()
        assert (g2[(mag2 == 0).all(1)] == 0).all()
        assert same(g2, knn_backward(p1, p2, idx, dd, dn)[1])


@gpu
def test_knn_points_dropin_shapes_and_autograd():
    from multiply_b200.utils.pytorch3d_ops import knn_points
    p1 = torch.randn(1, 300, 3, device="cuda", requires_grad=True)
    p2 = torch.randn(1, 2000, 3, device="cuda", requires_grad=True)
    d, i, nn = knn_points(p1, p2, K=1, return_nn=True)
    assert d.shape == (1, 300, 1) and i.shape == (1, 300, 1) and i.dtype == torch.int64 and nn.shape == (1, 300, 1, 3)
    rd, ri = nearest_def(p1[0].detach(), p2[0].detach())
    assert same(d[0, :, 0].detach().cpu(), rd) and torch.equal(i[0, :, 0].cpu(), ri)
    (d.sum() + nn.sum()).backward()
    assert p1.grad.shape == p1.shape and p2.grad.shape == p2.shape
    with pytest.raises(NotImplementedError):
        knn_points(p1, p2, K=2)


# ---------------------------------------------------------------------------------------------
# end to end: posed meshes -> depth maps + nearest vertices -> losses -> SMPL-parameter gradients
# ---------------------------------------------------------------------------------------------

H_E2E, W_E2E = 1280, 940


def e2e_camera(centre):
    """A camera 3.2 units in front of the persons' centre (R = I, looking along +z), Hi4D-like intrinsics."""
    K = np.array([[1400.0, 0.0, W_E2E / 2 + 2.3], [0.0, 1400.0, H_E2E / 2 - 4.7], [0.0, 0.0, 1.0]])
    T = -np.asarray(centre, dtype=np.float64) + np.array([0.0, 0.0, 3.2])
    return K, np.eye(3), T


def test_e2e_chain_runs_on_cpu_definitions():
    """The float64 port chain and oracle/opt_depth.py run on the CPU definitions alone (nothing here needs a GPU)."""
    v, f = S.make_body_mesh(step=0.066)
    v = torch.as_tensor(v).double()
    f = torch.as_tensor(f)
    K, R, T = e2e_camera(v.mean(0).numpy())
    cam = RA.camera_record(R, T, K)
    H, W = 96, 72
    cam["fx"], cam["fy"], cam["cx"], cam["cy"] = 100.0, 100.0, 36.0, 48.0
    dm = [RA.depth_map(cam, v, f, H, W), RA.depth_map(cam, v + 0.05, f, H, W)]
    logits = torch.randn(1, H, W, 2, generator=torch.Generator().manual_seed(0), dtype=torch.float64) * 4
    loss, n = OD.depth_order_loss(dm, logits)
    assert n > 0 and torch.isfinite(loss)


@gpu
def test_opt_depth_losses_end_to_end():
    from multiply_b200.model.render import Renderer
    from multiply_b200.utils import kaolin_ops, pytorch3d_ops
    from oracle import mesh_port
    from _body_grad_port import float64, model64, _t
    P = 2
    sc, model, inp = S.make_smpl_scene(P=P)
    trans = inp["smpl_trans"].clone()
    trans[0, 1] = trans[0, 0] + torch.tensor([0.12, 0.03, 0.08])          # translated into each other
    scale = inp["smpl_params"][0, 0, 0].reshape(1)
    params = [dict(transl=trans[0, p].reshape(1, 3), thetas=inp["smpl_pose"][0, p].reshape(1, 72),
                   betas=torch.from_numpy(np.random.RandomState(60 + p).normal(0, 0.5, (1, 10)).astype(np.float32)))
              for p in range(P)]
    servers = model.smpl_server_list
    cano = [torch.as_tensor(srv.mesh_verts_c, dtype=torch.float32) for srv in servers]
    faces = [torch.as_tensor(srv.faces, dtype=torch.int64).reshape(-1, 3) for srv in servers]
    gperm = torch.Generator().manual_seed(11)
    perms = [torch.randperm(c.shape[0], generator=gperm) for c in cano]

    # device: the reference's lines with the three drop-ins
    sp = scale.clone().cuda().requires_grad_(True)
    dp = [{k: v.clone().cuda().requires_grad_(True) for k, v in pr.items()} for pr in params]
    verts_gpu = []
    for p, srv in enumerate(servers):
        o = srv(sp, dp[p]["transl"], dp[p]["thetas"], dp[p]["betas"])
        xd = model.get_deformed_mesh_fast_mode_multiple_person(cano[p].cuda(), o["smpl_tfs"], p)
        verts_gpu.append((1 / sp.squeeze()) * xd)
    centre = torch.cat([v[0] for v in verts_gpu]).detach().mean(0).cpu().numpy()
    K, R, T = e2e_camera(centre)
    r = Renderer(img_size=[H_E2E, W_E2E], cam_intrinsic=K)
    r.set_camera(torch.tensor(R)[None].float(), torch.tensor(T)[None].float())
    dm_gpu = r.render_multiple_depth_map(verts_gpu, [f.cuda()[None] for f in faces])
    logits = sam_logits(H_E2E, W_E2E, 5)
    d_loss, n_excl = OD.depth_order_loss(dm_gpu, logits.cuda())
    i_loss = OD.interpenetration_loss(verts_gpu, [f.cuda() for f in faces], kaolin_ops.check_sign,
                                      pytorch3d_ops.knn_points, perms)
    assert n_excl > 100 and float(i_loss.detach()) > 0, n_excl
    leaves = [sp] + [dp[p][k] for p in range(P) for k in ("transl", "thetas", "betas")]
    got = {}
    for name, loss in (("depth", d_loss), ("interp", i_loss)):
        g = torch.autograd.grad(loss.sum(), leaves, retain_graph=True, allow_unused=True)
        got[name] = [float(loss.detach().sum())] + [np.zeros(x.numel()) if gi is None else gi.cpu().double().numpy().reshape(-1)
                                     for gi, x in zip(g, leaves)]

    # the device's discrete decisions, held fixed in the port chain
    cam = RA.camera_record(R, T, K)
    p2f = [engine_p2f(r, v[0], f) for v, f in zip(verts_gpu, faces)]
    for p in range(P):
        assert torch.equal(p2f[p], RA.rasterize(cam, verts_gpu[p][0].detach().cpu(), faces[p], H_E2E, W_E2E)["pix_to_face"])
    inside = {}
    nearest = {}
    for p in range(P):
        pts = verts_gpu[p][0].detach()[perms[p][:5120].cuda()]
        for q in range(P):
            if q != p:
                inside[p, q] = kaolin_ops.check_sign(verts_gpu[q].detach(), faces[q].cuda(), pts[None])[0].cpu()
                pen = pts[inside[p, q].cuda()]
                if pen.shape[0]:
                    nearest[p, q] = pytorch3d_ops.knn_points(pen[None], verts_gpu[q].detach())[1][0, :, 0].cpu()

    # float64 port chain, its posed vertices carried at the device's values (straight through: the depth loss's vertex
    # gradients change by ~10^3 2^-24 under one fp32 rounding of the vertices, so only equal vertices compare at the
    # SMPL gate); the forward chain is checked separately against them
    want = {}
    v_gpu = [v[0].detach().cpu().double() for v in verts_gpu]
    with float64():
        def posed(s, tr):
            out = []
            for p, srv in enumerate(servers):
                sm = S.make_smpl_model(300 + p, body_seed=100 + p)
                o = port.smpl_server_forward(model64(sm), _t(srv.tfs_c_inv.cpu().numpy()), s, *tr[p])
                idx = _nearest_cano(cano[p], srv.verts_c[0])
                Wt = _t(srv.weights[0].cpu().numpy())[idx]
                Tm = torch.einsum("pn,nij->pij", Wt, o["smpl_tfs"])
                xd = torch.einsum("pij,pj->pi", Tm[:, :3, :3], cano[p].double()) + Tm[:, :3, 3]
                out.append((1 / s[0]) * xd)
            return out

        s0, h = float(scale), 1e-6
        for name in ("depth", "interp"):
            tr = [tuple(_t(params[p][k].numpy().reshape(-1), True) for k in ("transl", "thetas", "betas"))
                  for p in range(P)]
            vs = []
            for p, v64 in enumerate(posed(torch.full((1,), s0), tr)):
                c = float((v64.detach() - v_gpu[p]).abs().max()) / (EPS * float(v64.detach().abs().max()))
                print("posed vertices of person %d: device vs float64 C = %.2f" % (p, c))
                assert c < C_SMPL, (p, c)
                vs.append((v64 + (v_gpu[p] - v64).detach())[None])
                vs[-1].retain_grad()
            if name == "depth":
                dm = [depth_map_at(cam, v[0], f, pf) for v, f, pf in zip(vs, faces, p2f)]
                lv = OD.depth_order_loss(dm, logits.double())[0]
            else:
                order = iter([(p, q) for p in range(P) for q in range(P) if q != p])
                cur = {}

                def check_sign(verts, f, pts):          # the loss asks person by person, partner by partner
                    cur["pq"] = next(order)
                    return inside[cur["pq"]][None]

                def knn_points(p1, p2, K=1, return_nn=True):
                    idx = nearest[cur["pq"]]
                    return None, idx[None, :, None], p2[0][idx][None, :, None, :]
                lv = OD.interpenetration_loss(vs, faces, check_sign, knn_points, perms)
            lv.sum().backward()
            with torch.no_grad():       # scale: port.smpl_server_forward scales in place, so d/ds by central differences
                fd = [(a - b) / (2 * h) for a, b in zip(posed(torch.full((1,), s0 + h), tr),
                                                        posed(torch.full((1,), s0 - h), tr))]
                d_s = sum(float((v.grad[0] * d).sum()) for v, d in zip(vs, fd))
            want[name] = [float(lv.detach().sum()), np.array([d_s])] + \
                [x.grad.numpy().reshape(-1) for t3 in tr for x in t3]
    for name in want:
        M = max(np.abs(np.asarray(w)).max() for w in want[name][1:])
        c_val = abs(got[name][0] - want[name][0]) / (EPS * abs(want[name][0]))
        c_grad = max(float(np.abs(gg - np.asarray(ww).reshape(-1)).max()) for gg, ww in
                     zip(got[name][1:], want[name][1:])) / (EPS * M)
        print("%s loss: value %.6g (C = %.2f), gradients C = %.2f (gate %g)" % (name, want[name][0], c_val, c_grad,
                                                                              C_SMPL))
        assert c_val < C_SMPL and c_grad < C_SMPL, (name, c_val, c_grad)


def sam_logits(H, W, seed):
    """A seeded SAM logit map [1,H,W,2]: per pixel one person at +3 and the other at -4 (sigmoid sum 0.97: valid), or
    both at +3 on a tenth of the pixels (sum 1.9: invalid), plus noise of 0.1.  No pixel sits near the 0.7 / 1.01
    thresholds or an argmax tie, so fp32 and fp64 decide alike."""
    g = torch.Generator().manual_seed(seed)
    who = torch.randint(2, (H, W), generator=g)
    lg = torch.where(torch.stack([who == 0, who == 1], -1), 3.0, -4.0)
    lg[torch.rand(H, W, generator=g) < 0.1] = 3.0
    lg[..., 1] += 0.5 * (lg[..., 0] == lg[..., 1])                     # no argmax ties
    return (lg + 0.1 * torch.randn(H, W, 2, generator=g))[None]


def engine_p2f(renderer, verts, faces):
    from multiply_b200 import engine
    H, W = renderer.image_size
    _, p2f = engine.DepthRaster.apply(renderer.cam, H, W, verts.device, verts.detach(), faces.cuda())
    return p2f.cpu()


def depth_map_at(cam, verts, faces, p2f):
    """oracle/raster.py:depth_map with the device's pix_to_face: [1,H,W,1] fp64 with gradients."""
    H, W = p2f.shape
    p = p2f.reshape(-1)
    hit = torch.nonzero(p >= 0).reshape(-1)
    px, py = (hit % W).double() + 0.5, (hit // W).double() + 0.5
    z = RA.face_depth(verts[faces[p[hit]]], px, py, cam)
    return torch.full((H * W,), -1.0, dtype=verts.dtype).index_put((hit,), z).reshape(1, H, W, 1)


def _nearest_cano(x, verts):
    return nearest_def(x, verts.detach().cpu())[1]
