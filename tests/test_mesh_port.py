"""CPU: the kaolin definitions of oracle/mesh_port.py (point_to_mesh_distance, check_sign), the synthetic canonical mesh
(scene.make_body_mesh) and the training forward at current_epoch < 250 against the reference
(tests/golden/forward_train_early.npz)."""
import math
import os
import numpy as np
import pytest
import torch

from oracle import mesh_port as port
from multiply_b200 import scene as S


def _volume(v, f):
    v = v.double()
    return float((v[f[:, 0]] * torch.cross(v[f[:, 1]], v[f[:, 2]], dim=1)).sum() / 6)


def _winding(v, f, pts):
    """Generalised winding number (sum of the faces' signed solid angles / 4 pi, Van Oosterom & Strackee), fp64."""
    v = v.double()
    out = torch.empty(pts.shape[0], dtype=torch.float64)
    for s in range(0, pts.shape[0], 128):
        p = pts[s:s + 128].double()[:, None]
        a, b, c = v[f[:, 0]][None] - p, v[f[:, 1]][None] - p, v[f[:, 2]][None] - p
        la, lb, lc = a.norm(dim=-1), b.norm(dim=-1), c.norm(dim=-1)
        num = (a * torch.cross(b, c, dim=-1)).sum(-1)
        den = la * lb * lc + (a * b).sum(-1) * lc + (b * c).sum(-1) * la + (c * a).sum(-1) * lb
        out[s:s + 128] = (2 * torch.atan2(num, den)).sum(1) / (4 * math.pi)
    return out


def make_torus(R=0.5, r=0.18, nu=48, nv=24):
    """Closed torus (a hole through it) around the z axis, outward-oriented."""
    u = torch.arange(nu, dtype=torch.float64) * 2 * math.pi / nu
    w = torch.arange(nv, dtype=torch.float64) * 2 * math.pi / nv
    U, W = torch.meshgrid(u, w, indexing="ij")
    v = torch.stack([(R + r * torch.cos(W)) * torch.cos(U), (R + r * torch.cos(W)) * torch.sin(U), r * torch.sin(W)], -1)
    i, j = torch.meshgrid(torch.arange(nu), torch.arange(nv), indexing="ij")
    a, b = i * nv + j, ((i + 1) % nu) * nv + j
    c, d = ((i + 1) % nu) * nv + (j + 1) % nv, i * nv + (j + 1) % nv
    f = torch.cat([torch.stack([a, b, c], -1).reshape(-1, 3), torch.stack([a, c, d], -1).reshape(-1, 3)])
    return v.reshape(-1, 3).float(), f.long()


@pytest.fixture(scope="module")
def body_mesh():
    return S.make_body_mesh(100)


def test_distance_regions_hand_computed():
    """One point in each of the 7 regions of the triangle (0,0,0), (1,0,0), (0,1,0)."""
    tri = torch.tensor([[[0., 0, 0], [1, 0, 0], [0, 1, 0]]])[None]
    pts = torch.tensor([[0.2, 0.2, 0.5], [-1, -1, 0.3], [2, -0.5, 0], [-0.5, 2, 1], [0.5, -1, 0], [1, 1, 0],
                        [-1, 0.5, 0]])
    want_d2 = [0.25, 2 + 0.09, 1 + 0.25, 0.25 + 1 + 1, 1.0, 0.5, 1.0]
    want_t = [0, 1, 2, 3, 4, 5, 6]
    d2, idx, typ = port.point_to_mesh_distance(pts[None], tri)
    assert d2.shape == (1, 7) and d2.dtype == torch.float32
    assert idx.dtype == torch.int64 and typ.dtype == torch.int32
    assert np.allclose(d2[0].numpy(), want_d2, rtol=1e-7, atol=0)
    assert typ[0].tolist() == want_t and idx[0].tolist() == [0] * 7


def test_distance_against_dense_sampling():
    """Never above the distance to a dense sampling of the triangles, and within its resolution of it."""
    g = torch.Generator().manual_seed(3)
    tris = (torch.rand(6, 3, 3, generator=g) - 0.5).double()
    pts = (torch.rand(300, 3, generator=g) - 0.5).double() * 1.6
    k = 200
    i, j = torch.meshgrid(torch.arange(k + 1), torch.arange(k + 1), indexing="ij")
    m = (i + j) <= k
    bu, bv = (i[m].double() / k), (j[m].double() / k)
    samples = (tris[:, None, 0] + bu[None, :, None] * (tris[:, None, 1] - tris[:, None, 0])
               + bv[None, :, None] * (tris[:, None, 2] - tris[:, None, 0])).reshape(-1, 3)
    edge = max(float((tris[:, a] - tris[:, b]).norm(dim=-1).max()) for a, b in ((0, 1), (1, 2), (2, 0)))
    res = edge / k                      # every point of a triangle lies within this of a sample
    d2, _ = port._closest_point_triangle(pts[:, None], tris[None, :, 0], tris[None, :, 1], tris[None, :, 2])
    exact = d2.min(1)[0].sqrt()
    sampled = torch.cdist(pts, samples).min(1)[0]
    assert bool((exact <= sampled + 1e-9).all())
    assert bool((sampled <= exact + res + 1e-9).all())


def _sign_agrees(v, f, pts):
    inside = port.check_sign(v[None], f, pts[None])[0]
    d2, _, _ = port.point_to_mesh_distance(pts[None], port.index_vertices_by_faces(v[None], f))
    far = d2[0].double().sqrt() > 1e-4
    wn = _winding(v, f, pts) > 0.5
    assert int(far.sum()) > 0.9 * pts.shape[0]
    assert torch.equal(inside[far], wn[far])
    return inside[far]


def test_sign_synthetic_meshes(body_mesh):
    g = torch.Generator().manual_seed(8)
    for v, f in (body_mesh, S.make_body_mesh(101)):
        lo, hi = v.min(0)[0], v.max(0)[0]
        pts = lo - 0.05 + (hi - lo + 0.1) * torch.rand(1500, 3, generator=g)
        # plus points on the lattice of the mesh's own vertices' x / y (rays through vertices and edges)
        pts = torch.cat([pts, v[::37] + torch.tensor([0.0, 0.0, 0.01])])
        ins = _sign_agrees(v, f, pts)
        assert 0 < int(ins.sum()) < ins.numel()


def test_sign_torus():
    v, f = make_torus()
    g = torch.Generator().manual_seed(9)
    pts = (torch.rand(3000, 3, generator=g) - 0.5) * torch.tensor([1.6, 1.6, 0.5])
    pts = torch.cat([pts, torch.tensor([[0.0, 0.0, 0.0], [0.0, 0.0, -0.1], [0.5, 0.0, 0.0], [0.0, -0.5, 0.05]])])
    ins = _sign_agrees(v, f, pts)
    assert not bool(ins[-4]) and not bool(ins[-3]) and bool(ins[-2]) and bool(ins[-1])      # the hole is outside


def test_body_mesh_watertight_oriented_deterministic(body_mesh):
    v, f = body_mesh
    assert v.dtype == torch.float32 and f.dtype == torch.int64
    assert 10000 < f.shape[0] < 20000            # of the order of SMPL's 13 776
    e = torch.cat([f[:, [0, 1]], f[:, [1, 2]], f[:, [2, 0]]]).tolist()
    directed = set(map(tuple, e))
    assert len(directed) == len(e)               # no directed edge twice
    assert all((b, a) in directed for a, b in e)     # every edge once in each direction
    assert _volume(v, f) > 0.03
    v2, f2 = S.make_body_mesh(100)
    assert torch.equal(v, v2) and torch.equal(f, f2)
    # non-convex: the mesh's volume is well below its convex hull's bounding box
    ext = (v.max(0)[0] - v.min(0)[0]).double()
    assert _volume(v, f) < 0.3 * float(ext.prod())


def _train_inputs(g, sc):
    rng, eik = [], []
    for p in range(2):
        rng.append({"t_rand": torch.from_numpy(g[f"t_rand_{p}"]), "u_final": torch.from_numpy(g[f"u_final_{p}"]),
                    "extra_perm": torch.from_numpy(g[f"extra_perm_{p}"]), "eik_idx": torch.from_numpy(g[f"eik_idx_{p}"]),
                    "t_rand_bg": torch.from_numpy(g[f"t_rand_bg_sampler_{p}"])})
        vc = sc["persons"][p]["verts_c"]
        idx = torch.from_numpy(g[f"eik_perm_{p}"])[:512]
        eik.append(vc[idx] + torch.from_numpy(g[f"eik_noise_{p}"])[0] * 0.01)
    return dict(rng=rng, eik_points=eik, t_rand_bg=torch.from_numpy(g["t_rand_bg"]))


def flag_mismatches(got, want, ref_min, thr=0.05, eps=1e-6):
    """Rows where two flag vectors differ, and how many of them are NOT on a boundary (reference minimum within eps of
    0 or thr): returns (exempt rows, unexplained mismatches)."""
    got, want, ref_min = np.asarray(got).astype(bool), np.asarray(want).astype(bool), np.asarray(ref_min)
    edge = (np.abs(ref_min) <= eps) | (np.abs(ref_min - thr) <= eps)
    return int(edge.sum()), int(((got != want) & ~edge).sum())


def ray_on_boundary(g, R, thr=0.05, eps=1e-6):
    """[R] bool: some person's reference row minimum of this ray lies within eps of 0 or thr."""
    edge = np.zeros(R, dtype=bool)
    for p in range(2):
        m = g[f"min_signed_{p}"]
        edge[g[f"hits_{p}"]] |= (np.abs(m) <= eps) | (np.abs(m - thr) <= eps)
    return edge


def test_forward_training_early_epoch(golden_dir):
    """mesh_port.multiply_forward(train=..., epoch=137, meshes=...) against the reference's training branch at epoch 137
    (check_off_in_surface_points_cano_mesh and the merge of multiply.py:549-560)."""
    g = np.load(os.path.join(golden_dir, "forward_train_early.npz"))
    sc = S.make_scene(P=2, S=16, seed=42)
    inputs = S.make_rays(sc, 40, seed=35, region="boxes")
    assert np.array_equal(inputs["uv"].numpy(), g["uv"]) and int(g["epoch"]) == 137
    hits = [torch.from_numpy(g[f"hits_{p}"]) for p in range(2)]
    meshes = [S.make_body_mesh(100 + p) for p in range(2)]
    out = port.multiply_forward(sc, inputs, hits, train=_train_inputs(g, sc), epoch=137, meshes=meshes)
    n_edge = 0
    for p in range(2):
        e, bad = flag_mismatches(out["_off_p"][p], g[f"off_{p}"], g[f"min_signed_{p}"])
        n_edge += e
        assert bad == 0
        e, bad = flag_mismatches(out["_in_p"][p], g[f"in_{p}"], g[f"min_signed_{p}"])
        assert bad == 0
        # the flags of the reference's own canonical points are exactly the port's definition
        o, i, mn = port.check_off_in_surface(torch.from_numpy(g[f"x_cano_{p}"]), 25, *meshes[p])
        assert np.array_equal(o.numpy(), g[f"off_{p}"]) and np.array_equal(i.numpy(), g[f"in_{p}"])
        assert np.array_equal(mn.numpy(), g[f"min_signed_{p}"])
    edge = ray_on_boundary(g, 40)
    for k in ("index_off_surface", "index_in_surface"):
        assert not bool(((out[k].numpy() != g[k]) & ~edge).any()), k
    assert n_edge <= 2
    assert np.abs(out["grad_theta"].numpy() - g["grad_theta"]).max() < 2e-6
    for k, tol in (("rgb_values", 1e-5), ("acc_map", 1e-5), ("normal_values", 5e-4), ("acc_person_list", 1e-5)):
        d = np.abs(out[k].numpy() - g[k])
        assert np.median(d) < 1e-5 and d.max() < tol, (k, float(d.max()))


def test_forward_training_late_epoch_has_no_flags():
    sc = S.make_scene(P=2, S=16, seed=42)
    g = np.load(os.path.join(os.path.dirname(__file__), "golden", "forward_train.npz"))
    inputs = S.make_rays(sc, 40, seed=33, region="boxes")
    hits = [torch.from_numpy(g[f"hits_{p}"]) for p in range(2)]
    out = port.multiply_forward(sc, inputs, hits, train=_train_inputs(g, sc), epoch=251)
    assert out["index_off_surface"] is None and out["index_in_surface"] is None
