"""CPU: the definitions behind opt_depth's geometric losses — oracle/opt_depth.py against the reference's own code
(tests/golden/opt_depth.npz), the camera extraction against cv2, and exact properties of oracle/raster.py's depth map."""
import numpy as np
import pytest
import torch

from multiply_b200.model.render import Renderer, camera_from_projection
from multiply_b200.utils import pytorch3d_ops
from oracle import mesh_port, opt_depth as OD, port, raster as RA


@pytest.fixture(scope="module")
def gold(golden_dir):
    import os
    return dict(np.load(os.path.join(golden_dir, "opt_depth.npz")))


def test_losses_and_gradients_match_the_reference(gold):
    H, W = int(gold["H"][0]), int(gold["W"][0])
    cam = RA.camera_record(gold["R"], gold["T"], gold["K"])
    f = torch.from_numpy(gold["faces"]).long()
    verts = [torch.from_numpy(gold["verts0"]), torch.from_numpy(gold["verts1"])]
    perms = [torch.from_numpy(gold["perm0"]).long(), torch.from_numpy(gold["perm1"]).long()]

    vl = [v.double()[None].requires_grad_(True) for v in verts]
    i_loss = OD.interpenetration_loss(vl, [f, f], mesh_port.check_sign, port.knn_points, perms)
    gi = torch.autograd.grad(i_loss.sum(), vl)
    np.testing.assert_allclose(float(i_loss.detach()), gold["interp_loss"][0], rtol=1e-12)
    for p in range(2):
        np.testing.assert_allclose(gi[p][0].numpy(), gold["interp_grad%d" % p], rtol=1e-10, atol=1e-14)

    vd = [v.double().requires_grad_(True) for v in verts]
    dm = [RA.depth_map(cam, v, f, H, W) for v in vd]
    d_loss, n = OD.depth_order_loss(dm, torch.from_numpy(gold["sam_logits"]))
    gd = torch.autograd.grad(d_loss, vd)
    assert n == int(gold["depth_n"][0])
    np.testing.assert_allclose(float(d_loss.detach()), gold["depth_loss"][0], rtol=1e-12)
    for p in range(2):
        np.testing.assert_allclose(gd[p].numpy(), gold["depth_grad%d" % p], rtol=1e-10, atol=1e-14)


def test_camera_extraction_matches_cv2(gold):
    cv2 = pytest.importorskip("cv2")
    K, R, T = camera_from_projection(gold["P"], float(gold["scale"][0]))
    np.testing.assert_allclose(K, gold["K"], rtol=1e-12, atol=1e-12)
    np.testing.assert_allclose(R, gold["R"], rtol=1e-12, atol=1e-12)
    np.testing.assert_allclose(T, gold["T"], rtol=1e-12, atol=1e-12)
    rng = np.random.RandomState(0)
    for k in range(20):
        A = rng.normal(size=(3, 3))
        Kt = np.array([[800 + 100 * rng.rand(), 3 * rng.randn(), 400.0], [0, 820.0, 300.0], [0, 0, 1.0]])
        q, _ = np.linalg.qr(A)
        q *= np.sign(np.linalg.det(q))
        P = Kt @ np.concatenate([q, rng.normal(size=(3, 1))], 1) * (3.0 if k % 2 else 1.0)   # K[2,2] = 3: kept
        s = 0.5 + rng.rand()
        Kc, Rc, c = cv2.decomposeProjectionMatrix((P @ np.diag([s, s, s, 1.0]))[:3])[:3]
        Tc = -Rc @ (c[:3] / c[3])[:, 0]
        K2, R2, T2 = camera_from_projection(P, s)
        np.testing.assert_allclose(K2, Kc, rtol=1e-9, atol=1e-9)
        np.testing.assert_allclose(R2, Rc, atol=1e-10)
        np.testing.assert_allclose(T2, Tc, rtol=1e-9, atol=1e-9)


def _cam(fx=100.0, cx=32.0, cy=24.0, T=(0.0, 0.0, 0.0)):
    return RA.camera_record(np.eye(3), T, np.array([[fx, 0, cx], [0, fx, cy], [0, 0, 1.0]]))


def test_plane_facing_the_camera_gives_its_depth_exactly():
    for Z in (0.5, 2.0, 3.25, 7.0):
        v = torch.tensor([[-5.0, -5.0, Z], [5.0, -5.0, Z], [5.0, 5.0, Z], [-5.0, 5.0, Z]])
        o = RA.rasterize(_cam(), v, torch.tensor([[0, 1, 2], [0, 2, 3]]), 48, 64)
        assert (o["zbuf"] == Z).all() and (o["pix_to_face"] >= 0).all()


def test_cube_shows_its_front_faces():
    c = torch.tensor([[x, y, z] for x in (-0.5, 0.5) for y in (-0.5, 0.5) for z in (-0.5, 0.5)]) + torch.tensor([0, 0, 3.0])
    quads = [(0, 1, 3, 2), (4, 6, 7, 5), (0, 4, 5, 1), (2, 3, 7, 6), (0, 2, 6, 4), (1, 5, 7, 3)]
    faces = torch.tensor([t for a, b, cc, d in quads for t in ((a, b, cc), (a, cc, d))])
    o = RA.rasterize(_cam(), c, faces, 48, 64)
    hit = o["pix_to_face"] >= 0
    assert hit.sum() > 0
    front = {i for i, tri in enumerate(faces.tolist()) if all(c[k, 2] == 2.5 for k in tri)}
    assert set(o["pix_to_face"][hit].unique().tolist()) <= front
    assert (o["zbuf"][hit] == 2.5).all()


def test_duplicate_faces_resolve_to_the_lower_index():
    v = torch.tensor([[-1.0, -1.0, 2.0], [1.0, -1.0, 2.5], [0.0, 1.0, 3.0]])
    faces = torch.tensor([[0, 1, 2], [2, 1, 0], [1, 2, 0], [0, 1, 2]])
    o = RA.rasterize(_cam(), v, faces, 48, 64)
    hit = o["pix_to_face"] >= 0
    assert hit.sum() > 100
    # the cyclic rotation [1, 2, 0] rounds the same depth the same way only when its terms are summed in the same
    # order; either way the winner is the lowest index among the faces at the smallest fp32 depth
    assert (o["pix_to_face"][hit] <= 2).all()
    o2 = RA.rasterize(_cam(), v, faces[[3, 0]], 48, 64)
    assert (o2["pix_to_face"][o2["pix_to_face"] >= 0] == 0).all()


def test_face_covering_no_pixel_centre_leaves_minus_one():
    # inside pixel (5, 5) (centre (5.5, 5.5)) without holding it; fx = 1, Z = 1: screen = world
    v = torch.tensor([[5.6, 5.1, 1.0], [5.9, 5.1, 1.0], [5.7, 5.45, 1.0]])
    o = RA.rasterize(_cam(fx=1.0, cx=0.0, cy=0.0), v, torch.tensor([[0, 1, 2]]), 12, 12)
    assert (o["pix_to_face"] == -1).all() and (o["zbuf"] == -1).all()
    # a face whose edge passes exactly through a centre covers it (closed triangle), from both windings
    v = torch.tensor([[5.5, 2.0, 1.0], [5.5, 9.0, 1.0], [9.0, 5.0, 1.0]])
    for f in ([0, 1, 2], [2, 1, 0]):
        o = RA.rasterize(_cam(fx=1.0, cx=0.0, cy=0.0), v, torch.tensor([f]), 12, 12)
        assert o["pix_to_face"][5, 5] == 0


def test_skipped_faces_and_empty_meshes():
    v = torch.tensor([[-0.1, -0.1, -1.0], [0.1, -0.1, 2.0], [0.0, 0.1, 2.0], [0.0, 0.0, 2.0]])
    o = RA.rasterize(_cam(), v, torch.tensor([[0, 1, 2], [3, 3, 3], [1, 2, 2]]), 48, 64)
    assert (o["pix_to_face"] == -1).all()
    o = RA.rasterize(_cam(), v, torch.zeros(0, 3, dtype=torch.int64), 1, 1)
    assert o["zbuf"].shape == (1, 1) and float(o["zbuf"]) == -1.0


def test_dropins_refuse_what_they_do_not_provide():
    r = Renderer(img_size=[48, 64], cam_intrinsic=np.array([[100.0, 0, 32], [0, 100.0, 24], [0, 0, 1]]))
    with pytest.raises(NotImplementedError, match="soft silhouette"):
        r.softrender_multiple_meshes([], [], [])
    with pytest.raises(NotImplementedError):
        r.render_multiple_meshes([], [], [])
    with pytest.raises(NotImplementedError, match="K = 1"):
        pytorch3d_ops.knn_points(torch.zeros(1, 2, 3), torch.zeros(1, 3, 3), K=2)


def test_size_queries_are_host_calls_and_refuse_bad_shapes():
    """The four workspace queries answer on the host (no launch, no device), grow with the problem, and answer 0 for
    shapes their calls refuse."""
    from multiply_b200 import _lib as L
    n0 = L.call("mp_launch_count", 0)
    for name, small, large in (("mp_depth_raster_workspace_bytes", (1, 1, 0), (1280, 940, 600000)),
                               ("mp_depth_raster_backward_workspace_bytes", (1, 1, 0), (1280, 940, 300000)),
                               ("mp_knn1_workspace_bytes", (1,), (100000,)),
                               ("mp_knn1_backward_workspace_bytes", (1, 1), (5120, 300000))):
        assert 0 < L.call(name, *small) <= L.call(name, *large), name
    assert L.call("mp_launch_count", 0) == n0
    assert L.call("mp_depth_raster_workspace_bytes", 0, 5, 1) == 0
    assert L.call("mp_depth_raster_workspace_bytes", 5, 5, -1) == 0
    assert L.call("mp_depth_raster_backward_workspace_bytes", 5, 0, 3) == 0
    assert L.call("mp_knn1_backward_workspace_bytes", 5, 0) == 0
    assert L.call("mp_knn1_workspace_bytes", 0) == 0
