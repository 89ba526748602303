"""GPU: the depth map of posed meshes (csrc/raster.cu, mp_depth_raster / mp_depth_raster_backward) against
oracle/raster.py's float64 definition.

raster.cu claims the oracle's rounding (fp64 on the fp32 inputs, no FMA contraction, the same operation order) and a
schedule-independent nearest-face choice (atomicMin on fp32 depth bits, then face index).  So the forward comparisons
are exact on every pixel: zbuf bit for bit and pix_to_face equal, with no pixels masked near an edge or a depth tie.
The oracle's decision margins are printed so a reader sees how close the cases come to a flip.

The backward is compared with float64 autograd of the closed form (oracle/raster.py:face_depth) at the GPU's own
pix_to_face: per vertex component |err| <= C 2^-24 M with C = 4, M the sum over the pixel terms the vertex receives of
each term's largest |component| (the device sums in fp64 and rounds once, so the bound is one fp32 rounding of a sum no
larger than M plus fp64 noise).
"""
import numpy as np
import pytest
import torch

from multiply_b200 import _lib as L, engine, scene as S
from oracle import raster as RA

from _abi import padded, same, take
from _setups import dirty_workspace

gpu = pytest.mark.gpu
C_GATE = 4.0


def cam_of(R, T, fx, fy, cx, cy):
    K = np.array([[fx, 0, cx], [0, fy, cy], [0, 0, 1.0]])
    return RA.camera_record(R, T, K), engine.camera(R, T, fx, fy, cx, cy)


def raster(cam_c, verts, faces, H, W, ws=None):
    v = verts.float().cuda().contiguous()
    f = faces.long().cuda().contiguous().reshape(-1, 3)
    V, F = v.shape[0], f.shape[0]
    nb = L.call("mp_depth_raster_workspace_bytes", H, W, F)
    ws = dirty_workspace(nb) if ws is None else ws
    zb, pf = padded(H * W), padded(H * W, torch.int64)
    L.call("mp_depth_raster", cam_c, v if V else None, V, f if F else None, F, H, W, zb, pf, ws, nb)
    return take(zb, (H, W), "zbuf"), take(pf, (H, W), "pix_to_face")


def check_exact(cam, cam_c, verts, faces, H, W, what):
    ref = RA.rasterize(cam, verts, faces, H, W)
    zb, pf = raster(cam_c, verts, faces, H, W)
    covered = int((ref["pix_to_face"] >= 0).sum())
    m = ref["edge_margin"][ref["pix_to_face"] >= 0]
    g = ref["depth_gap"][torch.isfinite(ref["depth_gap"])]
    print("%s: %d x %d, F = %d, %d pixels covered, smallest inside margin %.3g, smallest depth gap %.3g"
          % (what, H, W, faces.reshape(-1, 3).shape[0], covered, float(m.min()) if m.numel() else float("inf"),
             float(g.min()) if g.numel() else float("inf")))
    assert same(zb, ref["zbuf"]), "%s: zbuf differs at %d pixels" % (what, int((zb.view(torch.int32) != ref["zbuf"].view(torch.int32)).sum()))
    assert torch.equal(pf, ref["pix_to_face"]), "%s: pix_to_face differs at %d pixels" % (what, int((pf != ref["pix_to_face"]).sum()))
    return zb, pf, ref


def random_scene(F, seed, H, W, spread=1.0):
    g = torch.Generator().manual_seed(seed)
    centres = (torch.rand(F, 1, 3, generator=g) * 2 - 1) * torch.tensor([1.2, 1.2, 0.0]) * spread
    centres[..., 2] = 2.0 + 2.0 * torch.rand(F, 1, generator=g)
    tri = centres + 0.3 * (torch.rand(F, 3, 3, generator=g) * 2 - 1)
    verts = tri.reshape(-1, 3)
    faces = torch.arange(3 * F).reshape(F, 3)
    return verts, faces


# ---------------------------------------------------------------------------------------------
# forward, exact
# ---------------------------------------------------------------------------------------------

@gpu
@pytest.mark.parametrize("H,W", [(1, 1), (1, 37), (17, 33), (1280, 940)])
def test_random_faces_at_every_image_size(H, W):
    R = np.array([[0.96, -0.28, 0.0], [0.28, 0.96, 0.0], [0.0, 0.0, 1.0]])
    cam, cam_c = cam_of(R, [0.05, -0.02, 0.3], 0.9 * max(H, W), 0.9 * max(H, W), W / 2 + 0.25, H / 2 - 0.125)
    verts, faces = random_scene(400, 11 + H + W, H, W)
    check_exact(cam, cam_c, verts, faces, H, W, "random")


@gpu
def test_no_faces_and_skipped_faces():
    H, W = 17, 33
    cam, cam_c = cam_of(np.eye(3), [0, 0, 0], 20.0, 20.0, W / 2, H / 2)
    zb, pf = raster(cam_c, torch.zeros(0, 3), torch.zeros(0, 3, dtype=torch.int64), H, W)
    assert (zb == -1).all() and (pf == -1).all()
    v = torch.tensor([
        [100.0, 0, 2], [101, 0, 2], [100, 1, 2],             # off-screen
        [-0.2, -0.2, -1], [0.2, -0.2, -1], [0, 0.2, -1],      # behind the camera
        [-0.2, -0.2, 0], [0.2, -0.2, 2], [0, 0.2, 2],         # a vertex at Z = 0
        [-0.2, -0.2, 2], [0.2, 0.2, 2], [0.4, 0.4, 2],        # collinear: zero area
        [0.1, 0.1, 2], [0.1, 0.1, 2], [0.1, 0.1, 2],          # a point
    ])
    f = torch.arange(15).reshape(5, 3)
    zb, pf = raster(cam_c, v, f, H, W)
    assert (zb == -1).all() and (pf == -1).all()
    check_exact(cam, cam_c, v, f, H, W, "skipped")


@gpu
def test_faces_straddling_every_border_and_covering_no_centre():
    H, W = 17, 33
    cam, cam_c = cam_of(np.eye(3), [0, 0, 0], 1.0, 1.0, 0.0, 0.0)       # u = X / Z: Z = 1 puts vertices in pixels
    tris = []
    for cx_, cy_ in [(0, 8), (33, 8), (16, 0), (16, 17), (0, 0), (33, 17), (0, 17), (33, 0)]:
        tris.append([[cx_ - 3.3, cy_ - 2.7, 1], [cx_ + 2.9, cy_ - 3.1, 1], [cx_ + 0.2, cy_ + 3.6, 1]])
    tris.append([[5.6, 5.6, 1], [5.9, 5.6, 1], [5.7, 5.9, 1]])           # inside one pixel, holds no centre
    tris.append([[-150, -150, 3], [240, -120, 3], [30, 270, 3]])          # covers the whole image (Z = 3: / 3)
    v = torch.tensor(tris, dtype=torch.float32).reshape(-1, 3)
    f = torch.arange(v.shape[0]).reshape(-1, 3)
    zb, pf, ref = check_exact(cam, cam_c, v, f, H, W, "borders")
    assert (pf >= 0).all()                                                # the whole-image face is behind the others
    assert not (pf == 8).any()


@gpu
def test_pixel_centres_on_shared_edges_and_vertices():
    """A lattice of squares split along alternating diagonals with every vertex on a pixel centre (fx = 1, Z = 1), and
    the same lattice duplicated behind at equal depth: edges and vertices pass through centres, duplicates tie."""
    H, W = 24, 40
    n = 8
    cam, cam_c = cam_of(np.eye(3), [0, 0, 0], 1.0, 1.0, 0.0, 0.0)
    xs = np.arange(n + 1) * 4 + 2.5
    ys = np.arange(n + 1) * 3 + 0.5
    X, Y = np.meshgrid(xs, ys, indexing="ij")
    verts = torch.tensor(np.stack([X, Y, np.ones_like(X)], -1).reshape(-1, 3), dtype=torch.float32)
    faces = []
    for i in range(n):
        for j in range(n):
            a, b, c, d = i * (n + 1) + j, (i + 1) * (n + 1) + j, (i + 1) * (n + 1) + j + 1, i * (n + 1) + j + 1
            faces += [[a, b, c], [a, c, d]] if (i + j) % 2 else [[a, b, d], [b, c, d]]
    faces = torch.tensor(faces)
    faces = torch.cat([faces.flip(1), faces])                           # both windings; the first copy wins ties
    zb, pf, _ = check_exact(cam, cam_c, verts, faces, H, W, "shared edges")
    assert ((pf < faces.shape[0] // 2) | (pf == -1)).all()
    cam2, cam2_c = cam_of(np.eye(3), [0, 0, 1.0], 2.0, 2.0, 0.0, 0.0)  # Z = 2: u = 2 X / 2, still exact
    check_exact(cam2, cam2_c, verts, faces, H, W, "shared edges, Z = 2")


def hi4d_camera(H=1280, W=940):
    """A Hi4D-style camera looking at the body meshes (which stand along y around the origin) from z = -3.2."""
    R = np.array([[1.0, 0, 0], [0, -1.0, 0], [0, 0, -1.0]])
    th = 0.1
    Ry = np.array([[np.cos(th), 0, np.sin(th)], [0, 1, 0], [-np.sin(th), 0, np.cos(th)]])
    return cam_of(R @ Ry, [0.03, 0.25, 3.2], 1480.0, 1480.0, W / 2 + 3.3, H / 2 - 7.1)


def two_persons(step):
    v, f = S.make_body_mesh(step=step)
    v = torch.as_tensor(v)
    f = torch.as_tensor(f)
    v2 = v + torch.tensor([0.18, 0.02, 0.12])                          # interpenetrating partner
    return [(v, f), (v2, f)]


@gpu
@pytest.mark.parametrize("step", [0.033, 0.005])
def test_two_interpenetrating_persons_full_size(step):
    H, W = 1280, 940
    cam, cam_c = hi4d_camera(H, W)
    persons = two_persons(step)
    for p, (v, f) in enumerate(persons):
        check_exact(cam, cam_c, v, f, H, W, "person %d, step %g" % (p, step))
    v = torch.cat([persons[0][0], persons[1][0]])
    f = torch.cat([persons[0][1], persons[1][1] + persons[0][0].shape[0]])
    check_exact(cam, cam_c, v, f, H, W, "both persons as one mesh, step %g" % step)


@gpu
def test_reruns_workspace_and_size_query():
    H, W = 1280, 940
    cam, cam_c = hi4d_camera(H, W)
    (v, f), _ = two_persons(0.033)
    a = raster(cam_c, v, f, H, W)
    b = raster(cam_c, v, f, H, W, ws=torch.zeros(L.call("mp_depth_raster_workspace_bytes", H, W, f.shape[0]),
                                                  dtype=torch.uint8, device="cuda"))
    assert same(a[0], b[0]) and same(a[1], b[1])
    nb = L.call("mp_depth_raster_workspace_bytes", H, W, f.shape[0])
    ws = dirty_workspace(nb + 256)
    vv, ff = v.cuda(), f.cuda()
    zb, pf = torch.empty(H * W, device="cuda"), torch.empty(H * W, dtype=torch.int64, device="cuda")
    with pytest.raises(L.MpError, match="workspace too small"):
        L.call("mp_depth_raster", cam_c, vv, vv.shape[0], ff, ff.shape[0], H, W, zb, pf, ws, nb - 1)
    with pytest.raises(L.MpError, match="not 256-byte aligned"):
        L.call("mp_depth_raster", cam_c, vv, vv.shape[0], ff, ff.shape[0], H, W, zb, pf, ws[8:], nb)
    with pytest.raises(L.MpError, match="need H, W >= 1"):
        L.call("mp_depth_raster", cam_c, vv, vv.shape[0], ff, ff.shape[0], 0, W, zb, pf, ws, nb)
    with pytest.raises(L.MpError, match="need V, F >= 0"):
        L.call("mp_depth_raster", cam_c, vv, -1, ff, ff.shape[0], H, W, zb, pf, ws, nb)
    L.call("mp_depth_raster", cam_c, vv, vv.shape[0], ff, ff.shape[0], H, W, zb, pf, ws, nb)
    assert same(zb.reshape(H, W).cpu(), a[0])
    nbb = L.call("mp_depth_raster_backward_workspace_bytes", H, W, vv.shape[0])
    wsb = dirty_workspace(nbb)
    dv = torch.empty(vv.shape[0], 3, device="cuda")
    with pytest.raises(L.MpError, match="workspace too small"):
        L.call("mp_depth_raster_backward", cam_c, vv, vv.shape[0], ff, ff.shape[0], H, W, pf, zb, dv, wsb, nbb - 1)


# ---------------------------------------------------------------------------------------------
# backward
# ---------------------------------------------------------------------------------------------

def raster_backward(cam_c, verts, faces, H, W, p2f, d_zbuf):
    v = verts.float().cuda().contiguous()
    f = faces.long().cuda().contiguous().reshape(-1, 3)
    V, F = v.shape[0], f.shape[0]
    nb = L.call("mp_depth_raster_backward_workspace_bytes", H, W, V)
    ws = dirty_workspace(nb)
    dv = padded((V, 3))
    L.call("mp_depth_raster_backward", cam_c, v, V, f if F else None, F, H, W, p2f.cuda().contiguous(),
           d_zbuf.float().cuda().contiguous(), dv, ws, nb)
    return take(dv, (V, 3), "d_verts")


def reference_backward(cam, verts, faces, H, W, p2f, d_zbuf):
    """float64 autograd of face_depth per covered pixel: (sum of terms, M) per vertex component, M = the sum over the
    vertex's pixel terms of each term's largest |component|.  (A component that vanishes in exact arithmetic, such as
    the motion of a vertex within a plane parallel to the view, is computed as the cancellation of the term's other
    components, so its fp64 noise scales with them, not with itself.)"""
    faces = faces.long().reshape(-1, 3)
    p = p2f.reshape(-1)
    hit = torch.nonzero(p >= 0).reshape(-1)
    fv = faces[p[hit]]                                                    # [N,3]
    tri = verts.double()[fv].clone().requires_grad_(True)
    px, py = (hit % W).double() + 0.5, (hit // W).double() + 0.5
    g = d_zbuf.reshape(-1)[hit].double()
    z = RA.face_depth(tri, px, py, cam)
    (z * g).sum().backward()
    terms = tri.grad                                                      # [N,3,3], one pixel each
    V = verts.shape[0]
    ref = torch.zeros(V, 3, dtype=torch.float64).index_add_(0, fv.reshape(-1), terms.reshape(-1, 3))
    big = terms.abs().amax(2, keepdim=True).expand(-1, -1, 3)
    mag = torch.zeros(V, 3, dtype=torch.float64).index_add_(0, fv.reshape(-1), big.reshape(-1, 3))
    return ref, mag


def check_backward(cam, cam_c, verts, faces, H, W, seed, what):
    zb, pf = raster(cam_c, verts, faces, H, W)
    g = torch.Generator().manual_seed(seed)
    d = torch.randn(H, W, generator=g)
    d[torch.rand(H, W, generator=g) < 0.1] = 0.0
    dv = raster_backward(cam_c, verts, faces, H, W, pf, d)
    ref, mag = reference_backward(cam, verts, faces, H, W, pf, d)
    err = (dv.double() - ref).abs()
    bound = C_GATE * 2.0 ** -24 * mag
    ratio = float((err / mag.clamp_min(1e-300))[mag > 0].max()) / 2.0 ** -24 if (mag > 0).any() else 0.0
    print("%s: worst |err| / (2^-24 M) = %.3f (C = %g), %d vertices touched" % (what, ratio, C_GATE,
                                                                                  int((mag > 0).any(1).sum())))
    assert (err <= bound).all(), what
    assert (dv[(mag == 0).all(1)] == 0).all(), "%s: an untouched vertex got a gradient" % what
    dv2 = raster_backward(cam_c, verts, faces, H, W, pf, d)
    assert same(dv, dv2), "%s: rerun differs" % what
    return dv


@gpu
@pytest.mark.parametrize("H,W", [(1, 37), (17, 33), (1280, 940)])
def test_backward_random_faces(H, W):
    cam, cam_c = cam_of(np.eye(3), [0.05, -0.02, 0.3], 0.9 * max(H, W), 0.9 * max(H, W), W / 2 + 0.25, H / 2)
    verts, faces = random_scene(400, 23 + H, H, W)
    check_backward(cam, cam_c, verts, faces, H, W, 5, "random %dx%d" % (H, W))


@gpu
@pytest.mark.parametrize("step", [0.033, 0.005])
def test_backward_body_meshes(step):
    H, W = 1280, 940
    cam, cam_c = hi4d_camera(H, W)
    (v, f), _ = two_persons(step)
    check_backward(cam, cam_c, v, f, H, W, 7, "body step %g" % step)


@gpu
def test_backward_thousands_of_pixels_on_one_face():
    H, W = 256, 300
    cam, cam_c = cam_of(np.eye(3), [0, 0, 0], 200.0, 210.0, 150.0, 128.0)
    v = torch.tensor([[-2.0, -2.0, 2.0], [3.0, -1.5, 2.6], [-0.5, 2.5, 3.1], [0.1, 0.1, 1.5], [0.4, 0.1, 1.6],
                      [0.2, 0.5, 1.4], [9.0, 9.0, 9.0]])                  # the last vertex is in no face
    f = torch.tensor([[0, 1, 2], [3, 4, 5]])
    dv = check_backward(cam, cam_c, v, f, H, W, 9, "one large face")
    assert (dv[6] == 0).all()


@gpu
def test_autograd_node_and_renderer():
    from multiply_b200.model.render import Renderer
    H, W = 64, 48
    K = np.array([[60.0, 0.3, 24.5], [0, 61.0, 31.5], [0, 0, 1.0]])
    r = Renderer(img_size=[H, W], cam_intrinsic=K)
    R = torch.tensor([[[1.0, 0, 0], [0, 1.0, 0], [0, 0, 1.0]]])
    T = torch.tensor([[0.0, 0.0, 0.5]])
    r.set_camera(R, T)
    verts, faces = random_scene(60, 3, H, W, spread=0.5)
    v = verts.cuda()[None].requires_grad_(True)
    (dm,) = r.render_multiple_depth_map([v], [faces.cuda()[None]])
    assert dm.shape == (1, H, W, 1) and dm.device == v.device
    cam = RA.camera_record(R[0].numpy(), T[0].numpy(), K)
    ref = RA.rasterize(cam, verts, faces, H, W)
    assert same(dm[0, :, :, 0].detach().cpu(), ref["zbuf"])
    d = torch.randn(1, H, W, 1, device="cuda")
    (dm * d).sum().backward()
    ref_g, mag = reference_backward(cam, verts, faces, H, W, ref["pix_to_face"], d.cpu()[0, :, :, 0])
    assert ((v.grad[0].cpu().double() - ref_g).abs() <= C_GATE * 2.0 ** -24 * mag).all()
    with pytest.raises(NotImplementedError):
        r.softrender_multiple_meshes([v], [faces], None)
