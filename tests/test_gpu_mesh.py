"""GPU: the canonical-mesh kernels (csrc/mesh.cu) against oracle/mesh_port.py's kaolin definitions, the surface flags fused
into mp_render_rays, and Multiply.forward in training at current_epoch < 250 against the reference
(tests/golden/forward_train_early.npz)."""
import os
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from multiply_b200 import scene as S                                              # noqa: E402
from oracle import mesh_port as port                                              # noqa: E402

from _setups import flags_from_taps, fused_setup, mirror_inputs, render_train, train  # noqa: E402


@pytest.fixture(scope="module")
def meshes():
    return {"default": S.make_body_mesh(100), "large": S.make_body_mesh(100, step=0.007)}


def _query_points(v, n, seed):
    """Near-surface band, inside points, far points out to the bounding sphere (r = 3), points outside the grid."""
    g = torch.Generator().manual_seed(seed)
    lo, hi = v.min(0)[0], v.max(0)[0]
    k = n // 4
    band = v[torch.randint(0, v.shape[0], (k,), generator=g)] + 0.03 * torch.randn(k, 3, generator=g)
    box = lo + (hi - lo) * torch.rand(k, 3, generator=g)
    d = torch.nn.functional.normalize(torch.randn(k, 3, generator=g), dim=1)
    far = d * 3.0 * torch.rand(k, 1, generator=g)
    out = lo - 0.5 + (hi - lo + 1.0) * torch.rand(n - 3 * k, 3, generator=g)
    return torch.cat([band, box, far, out]).contiguous()


@pytest.mark.parametrize("which,n", [("default", 100000), ("large", 12000)])
def test_mesh_distance_and_sign_vs_port(meshes, which, n):
    from multiply_b200 import engine
    v, f = meshes[which]
    m = engine.CanonicalMesh(v, f)
    pts = _query_points(v, n, 5)
    d2, fi, dt = m.distance(pts.cuda())
    ins = m.check_sign(pts.cuda())
    torch.cuda.synchronize()
    fv = port.index_vertices_by_faces(v[None], f).cuda()
    rd2, rfi, rdt, second = port.point_to_mesh_distance(pts[None].cuda(), fv, return_second=True)
    rd2, rfi, rdt = rd2[0].double(), rfi[0], rdt[0]
    err = (d2.double() - rd2).abs()
    assert bool((err <= torch.maximum(1e-6 * rd2, torch.full_like(rd2, 1e-9))).all()), float(err.max())
    # the nearest face is defined where it is not a near tie (a closest point on a shared vertex or edge is an exact tie)
    clear = (second - rd2) > torch.maximum(1e-6 * rd2, torch.full_like(rd2, 1e-9))
    assert int(clear.sum()) > 0.2 * n
    assert torch.equal(fi[clear], rfi[clear])
    same = fi == rfi
    assert torch.equal(dt[same], rdt[same])
    rins = port.check_sign(v[None].cuda(), f.cuda(), pts[None].cuda())[0]
    far = rd2.sqrt() > 1e-4
    assert torch.equal(ins[far], rins[far])
    assert 0 < int(ins.sum()) < n


def _flags_vs_port(m, v, f, x, n_samples, thr=0.05):
    off, inn = m.surface_flags(x.cuda(), n_samples, thr)
    ro, ri, rmin = port.check_off_in_surface(x.cuda(), n_samples, v.cuda(), f.cuda(), thr)
    edge = (rmin.abs() <= 1e-6) | ((rmin - thr).abs() <= 1e-6)
    assert not bool(((off != ro) & ~edge).any()) and not bool(((inn != ri) & ~edge).any())
    return off, inn, int(edge.sum())


def test_mesh_surface_flags_vs_port(meshes):
    from multiply_b200 import engine
    v, f = meshes["default"]
    m = engine.CanonicalMesh(v, f)
    g = torch.Generator().manual_seed(11)
    rows, ns = 512, 97
    # rays of samples through the body's box: every row crosses some of the band around the surface
    lo, hi = v.min(0)[0], v.max(0)[0]
    o = lo + (hi - lo) * torch.rand(rows, 1, 3, generator=g)
    d = torch.nn.functional.normalize(torch.randn(rows, 1, 3, generator=g), dim=-1)
    t = torch.linspace(-0.3, 0.3, ns)[None, :, None] * torch.rand(rows, 1, 1, generator=g)
    x = (o + t * d).reshape(-1, 3)
    off, inn, n_edge = _flags_vs_port(m, v, f, x, ns)
    assert n_edge <= 2
    assert 0 < int(off.sum()) < rows and 0 < int(inn.sum()) < rows


# ---- fused path and mirror -----------------------------------------------------------------------------------------

def test_forward_training_early_epoch_mirror(golden_dir):
    """Multiply.forward in .train() at current_epoch = 137 against the reference's training branch (flags of
    check_off_in_surface_points_cano_mesh merged as multiply.py:549-560, and every other output)."""
    from multiply_b200 import engine
    engine.set_engine("tc")
    g = np.load(os.path.join(golden_dir, "forward_train_early.npz"))
    sc = S.make_scene(P=2, S=16, seed=42)
    inp = S.make_rays(sc, 40, seed=35, region="boxes")
    assert np.array_equal(inp["uv"].numpy(), g["uv"])
    m = S.mirror_model(sc)
    out = train(m, mirror_inputs(inp, 2, [torch.from_numpy(g[f"hits_{p}"]).cuda() for p in range(2)], epoch=137), 4322)
    edge = np.zeros(40, dtype=bool)
    for p in range(2):
        mn = g[f"min_signed_{p}"]
        edge[g[f"hits_{p}"]] |= (np.abs(mn) <= 1e-6) | (np.abs(mn - 0.05) <= 1e-6)
    assert int(edge.sum()) <= 2
    for k in ("index_off_surface", "index_in_surface"):
        got = out[k].cpu().numpy()
        assert out[k].dtype == torch.bool and got.shape == (40,)
        assert not bool(((got != g[k]) & ~edge).any()), k
    assert float(np.abs(out["grad_theta"].cpu().numpy() - g["grad_theta"]).max()) < 1e-4
    for k, tol in (("rgb_values", 1e-4), ("acc_map", 1e-4), ("acc_person_list", 1e-4), ("normal_values", 1e-3)):
        d = np.abs(out[k].cpu().numpy() - g[k])
        assert np.median(d) < 1e-5 and d.max() < tol, (k, float(d.max()))


@pytest.mark.parametrize("case", ["both", "single", "empty"])
def test_fused_flags_match_standalone(case):
    """Flags of mp_render_rays == mp_mesh_surface_flags on the same canonical points, for both persons, a single
    rendered person (id = p: one column) and a person with an empty hit list (the ray-0 substitute); flags on or off
    leave every pixel output bit-identical."""
    sc, r, inp, hits, meshes, rngs, tb = fused_setup(empty_person1=(case == "empty"))
    plist = [1] if case == "single" else [0, 1]
    hl = [hits[p] for p in plist]
    rg = [rngs[p] for p in plist]
    ms = [meshes[p] for p in plist]
    on = render_train(r, inp, hl, rg, tb, ms, persons=plist)
    off_ = render_train(r, inp, hl, rg, tb, None, persons=plist)
    for k in ("rgb_values", "fg_rgb_values", "normal_values", "acc_map", "acc_person_list"):
        assert torch.equal(on[k], off_[k]), k
    assert "index_off_surface" not in off_
    want_off, want_in = flags_from_taps(sc, r, inp, hits, ms, on, plist)
    assert torch.equal(on["index_off_surface"], want_off)
    assert torch.equal(on["index_in_surface"], want_in)
    if case == "empty":
        assert bool(on["index_off_surface"][1:][~torch.isin(torch.arange(1, inp["uv"].shape[1]).cuda(),
                                                             hits[0].cuda())].all())


def test_set_canonical_mesh_and_missing_mesh(golden_dir):
    """set_canonical_mesh replaces a person's mesh between two calls (flags follow the new mesh); a person without a
    mesh raises the documented error."""
    from multiply_b200 import engine
    engine.set_engine("tc")
    g = np.load(os.path.join(golden_dir, "forward_train_early.npz"))
    sc = S.make_scene(P=2, S=16, seed=42)
    inp = S.make_rays(sc, 40, seed=35, region="boxes")
    m = S.mirror_model(sc)
    hits = [torch.from_numpy(g[f"hits_{p}"]).cuda() for p in range(2)]
    a = train(m, mirror_inputs(inp, 2, hits, epoch=137), 4322)
    # a much larger mesh: every canonical sample lies inside it
    v, f = S.make_body_mesh(100)
    m.set_canonical_mesh(0, v * 20.0, f)
    m.set_canonical_mesh(1, v * 20.0, f)
    b = train(m, mirror_inputs(inp, 2, hits, epoch=137), 4322)
    hit_any = torch.zeros(40, dtype=torch.bool)
    for h in hits:
        hit_any[h.cpu()] = True
    assert torch.equal(b["index_in_surface"].cpu(), hit_any)
    assert not bool(b["index_off_surface"].cpu()[hit_any].any())
    assert torch.equal(a["rgb_values"], b["rgb_values"])
    x = torch.rand(64, 3, device="cuda") * 0.1
    o, i = m.check_off_in_surface_points_cano_mesh(x, 8, 0)
    assert o.shape == (8,) and bool(i.all()) and not bool(o.any())
    m.mesh_f_cano_list[1] = None
    m._cano_meshes.pop(1, None)
    with pytest.raises(ValueError, match="set_canonical_mesh"):
        train(m, mirror_inputs(inp, 2, hits, epoch=137), 4322)
    late = train(m, mirror_inputs(inp, 2, hits, epoch=251), 4322)
    assert late["index_off_surface"] is None and late["index_in_surface"] is None


def test_kaolin_ops_shapes_and_values(meshes):
    from multiply_b200.utils import kaolin_ops as K
    v, f = meshes["default"]
    pts = _query_points(v, 4000, 21)[None].cuda()
    fv = K.index_vertices_by_faces(v[None].cuda(), f.cuda())
    assert fv.shape == (1, f.shape[0], 3, 3)
    d, i, t = K.point_to_mesh_distance(pts, fv)
    s = K.check_sign(v[None].cuda(), f.cuda(), pts)
    assert d.shape == (1, 4000) and d.dtype == torch.float32
    assert i.shape == (1, 4000) and i.dtype == torch.int64
    assert t.shape == (1, 4000) and t.dtype == torch.int32
    assert s.shape == (1, 4000) and s.dtype == torch.bool
    rd, ri, rt, second = port.point_to_mesh_distance(pts, fv, return_second=True)
    rs = port.check_sign(v[None].cuda(), f.cuda(), pts)
    assert float(((d - rd).abs() / rd.clamp_min(1e-9)).max()) < 1e-6
    clear = (second - rd[0].double()) > 1e-6 * rd[0].double()
    assert torch.equal(i[0][clear], ri[0][clear]) and torch.equal(t[0][clear], rt[0][clear])
    far = rd[0].double().sqrt() > 1e-4
    assert torch.equal(s[0][far], rs[0][far])
