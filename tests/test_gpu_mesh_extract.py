"""GPU: mesh extraction (generate_mesh, lib/utils/mesh.py:78-132) — device MISE against the reference's own compiled
MISE driven by the mirror's Multiply.query_oc, device marching cubes and component selection against
oracle/mesh_extract.py, the posed mesh against the oracle's forward_skinning, and rejected inputs."""
import ctypes as C

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from multiply_b200 import engine, scene as S, _lib as L
from multiply_b200.utils import mesh as umesh
from oracle import build_ref, mesh_extract as M


@pytest.fixture(scope="module")
def model():
    engine.set_engine("tc")
    sc = S.make_scene(P=2, S=16, seed=42, weights="trained")
    return sc, S.mirror_model(sc)


def _values_at(m, pid, cond, R, center, extent):
    def f(idx):
        pts = torch.from_numpy(umesh.lattice_points(np.asarray(idx), R, center, extent)).cuda()
        occ = torch.cat([m.query_oc(b, cond, pid)["occ"] for b in torch.split(pts, 5000, dim=0)])
        return occ[:, 0].double().cpu().numpy()
    return f


@pytest.mark.parametrize("pid,res_init,depth,level", [(0, 8, 2, 0.0), (1, 8, 2, 0.0), (0, 32, 2, 0.0), (1, 32, 2, 0.0),
                                                      (0, 32, 3, 0.0), (1, 32, 3, 0.02), (1, 32, 4, 0.0)])
def test_mise_matches_reference(model, pid, res_init, depth, level):
    mod = build_ref.load_mise()
    if mod is None:
        pytest.skip("oracle/_ref has no compiled reference MISE (python -m oracle.build_ref with the reference tree)")
    sc, m = model
    person = sc["persons"][pid]
    cond = {"smpl": person["cond"].cuda()}
    center, extent, pad = umesh.bounds(person["verts_c"])
    R = res_init << depth
    f = m._ensure_renderer(torch.device("cuda", torch.cuda.current_device())).fields[pid]
    f.set_cond(cond["smpl"])
    grid, n, ev = f.mise(center, extent, res_init, depth, level, pad, want_evaluated=True)
    g_ref, ev_ref, rounds = M.reference_mise(mod, _values_at(m, pid, cond, R, center, extent), res_init, depth, level)
    assert n == sum(len(r) for r in rounds)
    assert np.array_equal(ev.cpu().numpy(), ev_ref)
    assert np.array_equal(grid.cpu().numpy().astype(np.float64), g_ref)
    assert 0 < n < (R + 1) ** 3 or depth == 0


def _sphere(R, r, c=(0.5, 0.5, 0.5)):
    x = np.arange(R + 1) / R
    X, Y, Z = np.meshgrid(x, x, x, indexing="ij")
    return (np.sqrt((X - c[0]) ** 2 + (Y - c[1]) ** 2 + (Z - c[2]) ** 2) - r).astype(np.float32)


def _torus(R, a=0.3, b=0.1):
    x = np.arange(R + 1) / R - 0.5
    X, Y, Z = np.meshgrid(x, x, x, indexing="ij")
    return (np.sqrt((np.sqrt(X ** 2 + Y ** 2) - a) ** 2 + Z ** 2) - b).astype(np.float32)


def _random(R, seed, quant=False):
    rng = np.random.default_rng(seed)
    g = rng.standard_normal((R + 1,) * 3).astype(np.float32)
    if quant:
        g = np.round(g * 2).astype(np.float32) / 2          # exact ties: values on the level, decider ties
    g[0], g[-1], g[:, 0], g[:, -1], g[:, :, 0], g[:, :, -1] = 1, 1, 1, 1, 1, 1
    return g


GRIDS = {
    "sphere1": lambda: _sphere(1, 0.6),
    "sphere2": lambda: _sphere(2, 0.3),
    "sphere37": lambda: _sphere(37, 0.31),
    "torus64": lambda: _torus(64),
    "sphere128": lambda: _sphere(128, 0.27, (0.47, 0.52, 0.5)),
    "random9": lambda: _random(9, 1),
    "random20q": lambda: _random(20, 2, quant=True),
    "random33": lambda: _random(33, 3),
}


@pytest.mark.parametrize("name", sorted(GRIDS))
@pytest.mark.parametrize("level", [0.0, 0.125])
def test_marching_cubes_matches_oracle(name, level):
    g = GRIDS[name]()
    R = g.shape[0] - 1
    center, extent, pad = (0.1, -0.2, 0.3), 1.7, 1.1
    v, f = engine.marching_cubes(torch.from_numpy(g).cuda(), level, center, extent, pad)
    vr, fr = M.marching_cubes(g, level, center, extent, pad)
    assert np.array_equal(v.cpu().numpy(), vr)
    assert np.array_equal(f.cpu().numpy(), fr)
    v2, f2 = engine.largest_component(v, f)
    vc, fc = M.largest_component(vr, fr)
    assert np.array_equal(v2.cpu().numpy(), vc) and np.array_equal(f2.cpu().numpy(), fc)


def test_marching_cubes_on_mise_grid(model):
    sc, m = model
    person = sc["persons"][0]
    center, extent, pad = umesh.bounds(person["verts_c"])
    f = m._ensure_renderer(torch.device("cuda", torch.cuda.current_device())).fields[0]
    f.set_cond(person["cond"].cuda())
    grid, _ = f.mise(center, extent, 32, 2, 0.0, pad)
    v, fc = engine.marching_cubes(grid, 0.0, center, extent, pad)
    vr, fr = M.marching_cubes(grid.cpu().numpy(), 0.0, center, extent, pad)
    assert len(fr) > 1000
    assert np.array_equal(v.cpu().numpy(), vr) and np.array_equal(fc.cpu().numpy(), fr)
    v2, f2 = engine.largest_component(v, fc)
    vc, fcc = M.largest_component(vr, fr)
    assert np.array_equal(v2.cpu().numpy(), vc) and np.array_equal(f2.cpu().numpy(), fcc)


@pytest.mark.parametrize("R", [512, 1024])
def test_marching_cubes_large_sphere(R):
    """At the res_up=4 size and the limit: a closed 2-manifold, Euler characteristic 2, volume within O(h^2)."""
    r = 0.3
    x = torch.arange(R + 1, device="cuda", dtype=torch.float32) / R - 0.5
    g = (x[:, None, None] ** 2 + x[None, :, None] ** 2 + x[None, None, :] ** 2).sqrt_().sub_(r)
    v, f = engine.marching_cubes(g, 0.0, (0.0, 0.0, 0.0), 1.0, 1.0)
    del g
    F = f.shape[0]
    e = torch.cat([f[:, [0, 1]], f[:, [1, 2]], f[:, [2, 0]]])                  # directed edges
    key = e[:, 0] * v.shape[0] + e[:, 1]
    assert torch.unique(key).numel() == 3 * F                                  # every directed edge once
    rkey = e[:, 1] * v.shape[0] + e[:, 0]
    assert bool(torch.isin(rkey, key).all())                                   # ... and its reverse once
    assert v.shape[0] - 3 * F // 2 + F == 2
    vd = v.double()
    vol = float((vd[f[:, 0]] * torch.cross(vd[f[:, 1]], vd[f[:, 2]], dim=1)).sum()) / 6.0
    exact = 4.0 / 3.0 * np.pi * r ** 3
    assert vol > 0 and abs(vol - exact) < 2.0 / R ** 2


def test_components_multi_tie_empty():
    R = 40
    two = np.minimum(_sphere(R, 0.12, (0.25, 0.5, 0.5)), _sphere(R, 0.18, (0.7, 0.5, 0.5)))
    many = _random(12, 5)
    for g in (two, many, _sphere(R, 2.0), np.ones((R + 1,) * 3, np.float32)):
        v, f = engine.marching_cubes(torch.from_numpy(g).cuda(), 0.0)
        vr, fr = M.marching_cubes(g, 0.0)
        v2, f2 = engine.largest_component(v, f)
        vc, fc = M.largest_component(vr, fr)
        assert np.array_equal(v2.cpu().numpy(), vc) and np.array_equal(f2.cpu().numpy(), fc)
    v, f = engine.largest_component(*engine.marching_cubes(torch.from_numpy(two).cuda(), 0.0))
    assert float(v[:, 0].min()) > 0.4 * R                                       # the larger sphere
    # three triangles of area exactly 0.5: the one holding face 0 is kept, whatever its vertices' order
    verts = torch.tensor([[0, 0, 0], [1, 0, 0], [0, 1, 0], [5, 0, 0], [6, 0, 0], [5, 1, 0], [9, 0, 0], [10, 0, 0],
                          [9, 1, 0]], dtype=torch.float32, device="cuda")
    faces = torch.tensor([[3, 4, 5], [0, 1, 2], [6, 7, 8]], dtype=torch.int64, device="cuda")
    v, f = engine.largest_component(verts, faces)
    assert torch.equal(v, verts[3:6]) and f.tolist() == [[0, 1, 2]]
    vc, fc = M.largest_component(verts.cpu().numpy(), faces.cpu().numpy())
    assert np.array_equal(v.cpu().numpy(), vc) and np.array_equal(f.cpu().numpy(), fc)
    v, f = engine.largest_component(verts[:0], faces[:0])
    assert v.shape == (0, 3) and f.shape == (0, 3)


def test_generate_mesh_end_to_end_and_rerun(model):
    """generate_mesh is the largest component of marching cubes on the MISE grid and reruns bit-identically; that
    surface -> set_canonical_mesh -> check_sign on lattice points with |sdf| > 2h agrees with the grid's sign (all
    components: points inside a dropped component are inside the grid's surface but not the kept mesh); the posed mesh
    matches the oracle's forward_skinning."""
    from oracle import port
    sc, m = model
    pid = 1
    person = sc["persons"][pid]
    cond = {"smpl": person["cond"].cuda()}
    v, f = umesh.generate_mesh(m, pid, cond, person["verts_c"], res_init=32, res_up=2)
    v2, f2 = umesh.generate_mesh(m, pid, cond, person["verts_c"], res_init=32, res_up=2)
    assert torch.equal(v, v2) and torch.equal(f, f2) and f.shape[0] > 1000
    center, extent, pad = umesh.bounds(person["verts_c"])
    fld = m._ensure_renderer(torch.device("cuda", torch.cuda.current_device())).fields[pid]
    fld.set_cond(cond["smpl"])
    grid, _ = fld.mise(center, extent, 32, 2, 0.0, pad)
    va, fa = engine.marching_cubes(grid, 0.0, center, extent, pad)
    vk, fk = engine.largest_component(va, fa)
    assert vk.shape == v.shape and fk.shape == f.shape
    assert torch.equal(fk, f) and float((vk - v).abs().max()) == 0.0
    m.set_canonical_mesh(pid, va, fa)
    R = 128
    h = float(pad * extent / R)
    idx = torch.nonzero(grid.abs() > 2 * h)
    idx = idx[torch.randperm(idx.shape[0], generator=torch.Generator().manual_seed(0))[:20000].cuda()]
    pts = torch.from_numpy(umesh.lattice_points(idx.cpu().numpy(), R, center, extent)).cuda()
    inside = m._canonical_mesh(pid, pts.device).check_sign(pts)
    want = grid[idx[:, 0], idx[:, 1], idx[:, 2]] < 0
    agree = float((inside == want).float().mean())
    b = torch.cat([grid[0].flatten(), grid[-1].flatten(), grid[:, 0].flatten(), grid[:, -1].flatten(),
                   grid[:, :, 0].flatten(), grid[:, :, -1].flatten()])
    print("check_sign vs grid sign: %.6f of %d points; boundary points below the level: %d"
          % (agree, idx.shape[0], int((b < 0).sum())))
    if not bool((b < 0).any()):          # the surface is closed only if it does not reach the lattice's boundary
        assert agree > 0.999
    m.set_canonical_mesh(pid, v, f)
    # posed mesh (multiply.py:129-134)
    xd = m.get_deformed_mesh_fast_mode_multiple_person(v[None], person["tfs"].cuda()[None], pid)
    ref, _ = port.forward_skinning(v.cpu().double(), dict(person, verts_c=person["verts_c"].double(),
                                                              weights=person["weights"].double(),
                                                              tfs=person["tfs"].double()))
    assert xd.shape == (1, v.shape[0], 3)
    assert float((xd[0].cpu().double() - ref).abs().max()) < 1e-5


def test_rejected_inputs(model):
    sc, m = model
    f = m._ensure_renderer(torch.device("cuda", torch.cuda.current_device())).fields[0]
    c = L.vec3(C.c_float, (0.0, 0.0, 0.0))
    n = C.c_longlong(0)
    g = torch.zeros(9 ** 3, device="cuda")

    def rejected(text, name, *args):
        with pytest.raises(L.MpError, match=r"failed \(-\d+\): .*" + text):
            L.call(name, *args)

    ws = L.workspace(L.call("mp_mise_workspace_bytes", 4, 1), "cuda")
    rejected("res_init", "mp_mise", f.handle, c, 1.0, 1.1, 4, 9, 0.0, g, None, C.byref(n), ws, ws.numel())
    rejected("", "mp_mise", f.handle, c, 1.0, 1.1, 4, 1, float("nan"), g, None, None, ws, ws.numel())
    rejected("", "mp_mise", f.handle, c, 1.0, 1.1, 4, 1, 0.0, None, None, None, ws, ws.numel())
    rejected("workspace", "mp_mise", f.handle, c, 1.0, 1.1, 4, 1, 0.0, g, None, None, ws, 16)
    V, F = C.c_longlong(0), C.c_longlong(0)
    mws = L.workspace(L.call("mp_marching_cubes_workspace_bytes", 8), "cuda")
    rejected("", "mp_marching_cubes_count", g, 0, 0.0, C.byref(V), C.byref(F), mws, mws.numel())
    rejected("", "mp_marching_cubes_count", g, 1025, 0.0, C.byref(V), C.byref(F), mws, mws.numel())
    rejected("", "mp_marching_cubes_count", g, 8, float("nan"), C.byref(V), C.byref(F), mws, mws.numel())
    rejected("", "mp_marching_cubes_count", None, 8, 0.0, C.byref(V), C.byref(F), mws, mws.numel())
    rejected("", "mp_marching_cubes_count", g, 8, 0.0, C.byref(V), C.byref(F), mws, 64)
    verts = torch.zeros(3, 3, device="cuda")
    faces = torch.tensor([[0, 1, 5]], dtype=torch.int64, device="cuda")
    cws = L.workspace(L.call("mp_largest_component_workspace_bytes", 3, 1), "cuda")
    Vo, Fo = C.c_int(0), C.c_int(0)
    rejected("outside", "mp_largest_component", verts, 3, faces, 1, verts, faces, C.byref(Vo), C.byref(Fo), cws,
             cws.numel())
    rejected("", "mp_largest_component", verts, 3, faces, 1, verts, faces, C.byref(Vo), C.byref(Fo), cws, 8)
    torch.cuda.synchronize()
