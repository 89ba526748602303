"""GPU: the deformer kernels (csrc/deform.cu) against a brute-force nearest vertex and a float64 restatement of
SMPLDeformer's closed-form skinning (deformer.py:19-50, 72-89), at the inputs where the grid search can go wrong.

The kernel claims an EXACT nearest vertex: the arg-min of d2 = (dx*dx + dy*dy) + dz*dz in fp32 with ties going to the
lowest index (oracle/port.py:knn_points).  So the outlier flags must match the brute force bit for bit, and x_c, x_d and
Jinv must match the fp64 skinning at the brute-force vertex within c * kappa * 2^-24 * scale, where kappa is the fp64
2-norm condition number of the blended 3x3 of that vertex and `scale` the magnitude of the terms each output sums.
Neighbouring vertices get clearly different skinning weights, so a wrong pick moves the geometry far outside that bound.

Bodies: the synthetic person at scale 0.5 and at scale 2 (where the posed and canonical grids must grow their cells to
stay within kMaxCells), tiny bodies (V = 1, 2, 33), a dyadic lattice whose vertex indices fall with x, y, z (every
midpoint is an exact tie, and the lower-index vertex often sits in the +1 cell that scan_block visits last), a flat body
(all z equal) and a body with duplicate vertex positions.  The hand-built bodies blend two joints 170-180 degrees apart
on every vertex, so their blended 3x3 has kappa up to ~1e3.

Queries: near-surface and uniform points, points exactly on cell faces, edges and corners of the posed and canonical
grids (rebuilt on the host with the kernel's fp32 operations), exact ties, points 0.1 +- a few ulps from their nearest
vertex, points in the empty border cells and beyond the clamp, far points (~1e3), and points whose nearest vertex lies
just outside the first search block while a farther vertex lies inside it (what the proof radius guards)."""
import os
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from multiply_b200 import scene as S          # noqa: E402
from oracle import port                       # noqa: E402

from _abi import padded, rows, take           # noqa: E402

U = 2.0 ** -24
POSED_CELL = np.float32(0.05005)   # mp_body_set_pose
R0 = 2
MAX_CELLS = 32768                  # kMaxCells (common.cuh)
SIZES = (0, 1, 127, 128, 129)
# Gate on c of the kappa-scaled bound.  Measured on one H100 80GB HBM3 at a 400 W power limit: worst c = 3.6 on the
# synthetic persons (kappa ~ 1.1) for x_c, x_d and Jinv; on the near-singular hand-built blends c grows with kappa
# (x_c: <= 35 for kappa < 1e3, 81 at kappa ~ 1150; Jinv: 19 and 53; x_d: 0.3).  The closed-form (adjugate) 3x3
# inverse is not backward stable when two singular values are small (a blend of two rotations ~180 degrees apart is
# close to a rank-1 projection), so its error grows faster than kappa * u there.  A wrong vertex moves x_c by O(1)
# relative, far above 128 * kappa * 2^-24 ~ 1e-2 even at kappa = 1e3.
C_GATE = 128.0
MEASURED = {}


# ---------------------------------------------------------------------------------------------
# host restatements of the grid (grid_build_kernel / nearest_vertex, fp32 operation by operation)
# ---------------------------------------------------------------------------------------------

def host_grid(verts, cell):
    """(lo, h, inv_h, dim, cells at the first h, growth steps) as grid_build_kernel computes them."""
    v = np.asarray(verts, np.float32)
    vlo, vhi = v.min(0), v.max(0)
    h = np.float32(cell)
    pad = 2 * R0
    n_first, steps = None, 0
    while True:
        dim = np.array([int(np.floor(np.float32(vhi[a] - vlo[a]) / h)) + 1 + 2 * pad for a in range(3)])
        n = int(np.prod(dim.astype(np.int64)))
        if n_first is None:
            n_first = n
        if n <= MAX_CELLS:
            break
        h = np.float32(h * np.float32(1.25))
        steps += 1
    lo = (vlo - np.float32(pad) * h).astype(np.float32)
    return dict(lo=lo, h=h, inv_h=np.float32(np.float32(1.0) / h), dim=dim, n_first=n_first, steps=steps)


def query_cells(g, p):
    f = ((np.asarray(p, np.float32) - g["lo"]) * g["inv_h"]).astype(np.float32)
    f = np.minimum(np.maximum(f, np.float32(-4.0)), (g["dim"] + 4).astype(np.float32))
    return np.floor(f).astype(np.int64)


def vertex_cells(g, v):
    f = ((np.asarray(v, np.float32) - g["lo"]) * g["inv_h"]).astype(np.float32)
    return np.clip(np.floor(f).astype(np.int64), 0, g["dim"] - 1)


def snap_to_boundary(g, x, axis):
    """fp32 coordinates x[:] moved onto the nearest cell boundary of `axis`, such that (x - lo) * inv_h is an exact
    integer in fp32 where a neighbour within 3 ulps allows it."""
    lo, h, inv_h = g["lo"][axis], g["h"], g["inv_h"]
    k = np.round((x.astype(np.float64) - lo) / float(h))
    x0 = (np.float64(lo) + k * np.float64(h)).astype(np.float32)
    cands, up, dn = [x0], x0, x0
    for _ in range(3):
        up = np.nextafter(up, np.float32(np.inf))
        dn = np.nextafter(dn, np.float32(-np.inf))
        cands += [dn, up]
    cands = np.stack(cands)                                               # [7, n]
    f = ((cands - lo) * inv_h).astype(np.float32)
    ok = f == k.astype(np.float32)[None]
    pick = np.where(ok.any(0), ok.argmax(0), 0)
    return cands[pick, np.arange(x.shape[0])]


# ---------------------------------------------------------------------------------------------
# bodies
# ---------------------------------------------------------------------------------------------

def _rot(axis, ang):
    axis = axis / np.linalg.norm(axis)
    return S._rodrigues((axis * ang)[None])[0]


def near_singular_rig(rng, V):
    """tfs [24,4,4] and weights [V,24]: joint 0 is a translation, joints 1..23 rotations by 170-179.9 degrees about
    random axes (plus translations); vertex v blends joint 0 with joint 1 + v % 23 at 0.5 +- eps, so the blended 3x3
    ranges from kappa ~ 10 to ~ 1e3.  Neighbouring indices get different joints and eps: different transforms."""
    tfs = np.zeros((24, 4, 4))
    tfs[:, 3, 3] = 1.0
    tfs[0, :3, :3] = np.eye(3)
    tfs[0, :3, 3] = rng.uniform(-0.2, 0.2, 3)
    ang = np.deg2rad(np.concatenate([[179.9, 179.8, 179.5, 179.0, 178.0, 177.0, 175.0, 170.0],
                                     rng.uniform(170.0, 179.9, 15)]))
    for j in range(1, 24):
        tfs[j, :3, :3] = _rot(rng.normal(size=3), ang[j - 1])
        tfs[j, :3, 3] = rng.uniform(-0.3, 0.3, 3)
    W = np.zeros((V, 24))
    eps = rng.uniform(-0.05, 0.05, V)
    eps[(rng.random(V) < 0.5) | (np.arange(V) % 23 < 4)] = 0.0     # joints 1-4: kappa 115 ... 1146
    W[:, 0] = 0.5 + eps
    W[np.arange(V), 1 + np.arange(V) % 23] = 0.5 - eps
    return tfs.astype(np.float32), W.astype(np.float32)


def _lattice(n, step, origin):
    axes = [origin[a] + step * np.arange(n[a]) for a in range(3)]
    X, Y, Z = np.meshgrid(*axes, indexing="ij")
    return np.stack([X, Y, Z], -1).reshape(-1, 3)


def _hand_body(name, verts, seed, cano_cell=0.2):
    rng = np.random.RandomState(seed)
    tfs, W = near_singular_rig(rng, verts.shape[0])
    v = np.ascontiguousarray(verts.astype(np.float32))
    return dict(name=name, verts_c=v, verts_p=v, weights=W, tfs=tfs, cano_cell=cano_cell, n_query=12000)


def make_body(name):
    if name in ("person", "person_x2"):
        scale = 0.5 if name == "person" else 2.0
        p = S.make_person(0, 1, scale=scale)
        vc = p["verts_c"].numpy() * np.float32(scale / 0.5)
        return dict(name=name, verts_c=np.ascontiguousarray(vc.astype(np.float32)), verts_p=p["verts_p"].numpy(),
                    weights=p["weights"].numpy(), tfs=p["tfs"].numpy(), cano_cell=0.2 if scale == 0.5 else 0.1,
                    n_query=40000)
    rng = np.random.RandomState(7)
    if name.startswith("tiny"):
        V = int(name[4:])
        return _hand_body(name, rng.uniform(-0.25, 0.25, (V, 3)), 10 + V)
    if name == "lattice":
        # dyadic lattice (exact midpoints and distances); indices fall with x, then y, then z
        v = _lattice((14, 11, 9), 2.0 ** -5, (0.25, -0.5, 0.125))
        v = v[np.lexsort((-v[:, 2], -v[:, 1], -v[:, 0]))]
        return _hand_body(name, v, 21, cano_cell=0.1)
    if name == "flat":
        v = _lattice((20, 16, 1), 2.0 ** -5, (-0.25, 0.0, 0.0625))
        return _hand_body(name, v[rng.permutation(v.shape[0])], 22)
    if name == "duplicates":
        base = rng.uniform(-0.3, 0.3, (300, 3)).astype(np.float32)
        v = np.concatenate([base, base[rng.choice(300, 150, replace=False)], base[rng.choice(300, 60, replace=False)]])
        return _hand_body(name, v[rng.permutation(v.shape[0])], 23)
    raise KeyError(name)


BODIES = ["person", "person_x2", "tiny1", "tiny2", "tiny33", "lattice", "flat", "duplicates"]


# ---------------------------------------------------------------------------------------------
# queries
# ---------------------------------------------------------------------------------------------

def _f32(a):
    return np.ascontiguousarray(np.asarray(a, np.float32).reshape(-1, 3))


def tie_points(v, g):
    """Exact ties: midpoints of lattice-neighbour pairs and centres of lattice squares / cubes.  Returns (points,
    number of pair midpoints whose lower-index vertex lies in the query's +1 cell)."""
    step = np.float32(2.0 ** -5)
    key = {tuple(p): i for i, p in enumerate(v.tolist())}
    pts, plus1 = [], 0
    for a in range(3):
        e = np.zeros(3, np.float32)
        e[a] = step
        for i, p in enumerate(v):
            j = key.get(tuple((p + e).tolist()))
            if j is None:
                continue
            m = p + e / np.float32(2)
            lo_i = min(i, j)
            cq, cl = query_cells(g, m[None])[0, a], vertex_cells(g, v[lo_i][None])[0, a]
            plus1 += int(cl == cq + 1)
            pts.append(m)
    centres = v + step / np.float32(2)
    return _f32(np.concatenate([np.array(pts), centres])), plus1


def proof_radius_points(rng, v, g, n_cand=200000):
    """Points whose nearest vertex lies outside the (2 R0 + 1)^3 block around the query's cell while the best vertex
    inside the block is farther than the first proof radius R0 * 0.999 h but within twice that."""
    span_lo, span_hi = v.min(0) - 0.15, v.max(0) + 0.15
    x = rng.uniform(span_lo, span_hi, (n_cand, 3)).astype(np.float32)
    cq = query_cells(g, x)
    inside = ((cq >= 0) & (cq < g["dim"])).all(1)
    cv = vertex_cells(g, v)
    inblk = (np.abs(cq[:, None, :] - cv[None, :, :]) <= R0).all(-1)                 # [n, V]
    d = x[:, None, :] - v[None, :, :]
    d2 = (d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]) + d[..., 2] * d[..., 2]
    near = d2.argmin(1)
    rr = np.float32(R0) * np.float32(g["h"] * np.float32(0.999))
    blk_best = np.where(inblk, d2, np.inf).min(1)
    sel = inside & ~inblk[np.arange(n_cand), near] & (blk_best > rr * rr) & (blk_best <= np.float32(4) * rr * rr)
    return x[sel][:4000]


def make_queries(body, verts, g, seed):
    """~n_query points of every kind for one grid (posed or canonical); returns (points, coverage counts)."""
    rng = np.random.RandomState(seed)
    v = np.asarray(verts, np.float32)
    V = v.shape[0]
    n = body["n_query"]
    vlo, vhi = v.min(0), v.max(0)
    parts, cov = [], {}
    # near the surface and uniform in the inflated bounding box
    parts.append(v[rng.randint(0, V, n // 4)] + rng.normal(0, 0.03, (n // 4, 3)))
    parts.append(rng.uniform(vlo - 0.3, vhi + 0.3, (n // 5, 3)))
    # on cell faces, edges and corners: 1, 2 or 3 coordinates snapped to a cell boundary
    m = n // 5
    base = (v[rng.randint(0, V, m)] + rng.uniform(-1.5, 1.5, (m, 3)) * g["h"]).astype(np.float32)
    k = rng.randint(1, 4, m)
    order = np.argsort(rng.random((m, 3)), 1)
    snap = order < k[:, None]
    for a in range(3):
        base[snap[:, a], a] = snap_to_boundary(g, base[snap[:, a], a], a)
    f = ((base - g["lo"]) * g["inv_h"]).astype(np.float32)
    cov["on_boundary"] = int(((f == np.floor(f)) & snap).any(1).sum())
    parts.append(base)
    # 0.1 +- 3 ulps from an extreme vertex along each axis direction (the outlier radius, deformer.py:49)
    r = [np.float32(0.1)]
    for _ in range(3):
        r = [np.nextafter(r[0], np.float32(0))] + r + [np.nextafter(r[-1], np.float32(1))]
    r = np.array(r, np.float32)
    for a in range(3):
        for sgn in (-1.0, 1.0):
            ext = v[np.argsort(sgn * v[:, a])[-min(V, 20):]]
            q = np.repeat(ext, r.size, 0)
            q[:, a] = q[:, a] + np.float32(sgn) * np.tile(r, ext.shape[0])
            parts.append(q)
    # the empty border cells and beyond the clamp of nearest_vertex (-4 .. dim + 4 cells)
    glo, ghi = g["lo"], g["lo"] + g["dim"] * g["h"]
    q = rng.uniform(glo - 6 * g["h"], ghi + 6 * g["h"], (n // 5, 3)).astype(np.float32)
    c = query_cells(g, q)
    border = ((c < 2 * R0) | (c > g["dim"] - 1 - 2 * R0)).any(1)
    parts.append(q[border])
    cov["border"] = int(border.sum())
    cov["border_cell_R0"] = int(((c == R0) | (c == g["dim"] - 1 - R0)).any(1).sum())
    # far away
    parts.append(rng.uniform(-1e3, 1e3, (256, 3)))
    parts.append(np.array([[1e3, 0, 0], [-1e3, 0, 0], [0, 1e3, 0], [0, -1e3, 0], [0, 0, 1e3], [0, 0, -1e3]]))
    if body["name"] == "lattice":
        t, plus1 = tie_points(v, g)
        parts.append(t)
        cov["ties"], cov["ties_plus1"] = t.shape[0], plus1
    if body["name"] == "duplicates":
        parts.append(v[rng.randint(0, V, 2000)] + rng.normal(0, 0.01, (2000, 3)))
    if body["name"] in ("tiny2", "tiny33"):
        pr = proof_radius_points(rng, v, g)
        parts.append(pr)
        cov["proof_radius"] = pr.shape[0]
    x = _f32(np.concatenate([np.asarray(p, np.float32) for p in parts]))
    return x[rng.permutation(x.shape[0])], cov


# ---------------------------------------------------------------------------------------------
# references
# ---------------------------------------------------------------------------------------------

def brute_force(x, verts):
    """(index, outlier) of port.knn_points in fp32 (the definition the kernel claims), as deformer.py:41-49 uses it."""
    d2, idx, _ = port.knn_points(torch.from_numpy(x)[None], torch.from_numpy(np.asarray(verts, np.float32))[None],
                                 return_nn=False)
    d = torch.sqrt(torch.clamp(d2[0, :, 0], max=4))
    return idx[0, :, 0].numpy(), (d > 0.1).numpy()


def _blend(W, tfs, idx):
    w = W[idx].astype(np.float64)
    T = np.einsum("pj,jab->pab", w, tfs.astype(np.float64))
    Tabs = np.einsum("pj,jab->pab", np.abs(w), np.abs(tfs.astype(np.float64)))
    return T, Tabs


def ref_inverse(x, idx, W, tfs):
    """x_c in fp64 (deformer.py:81-86 with the 4x4 inverse), kappa of the 3x3 block, and the x_c error scale."""
    T, _ = _blend(W, tfs, idx)
    xh = np.concatenate([x.astype(np.float64), np.ones((x.shape[0], 1))], 1)
    xc = np.einsum("pij,pj->pi", np.linalg.inv(T), xh)[:, :3]
    A = T[:, :3, :3]
    I = np.linalg.inv(A)
    kappa = np.linalg.cond(A)
    c = T[:, :3, 3] / T[:, 3, 3:4]
    scale = (np.abs(I) @ np.ones(3) * (np.abs(x).max(1) + np.abs(c).max(1))[:, None]).max(1)
    return xc, kappa, scale


def ref_forward(x, idx, W, tfs):
    """x_d and Jinv in fp64 (deformer.py:31-35 and the inverse of its 3x3 block), kappa and the error scales."""
    T, Tabs = _blend(W, tfs, idx)
    A = T[:, :3, :3]
    xd = np.einsum("pij,pj->pi", A, x.astype(np.float64)) + T[:, :3, 3]
    I = np.linalg.inv(A)
    kappa = np.linalg.cond(A)
    s_xd = (np.einsum("pij,pj->pi", Tabs[:, :3, :3], np.abs(x.astype(np.float64))) + Tabs[:, :3, 3]).max(1)
    s_J = np.abs(I).sum(2).max(1)
    return xd, I.reshape(-1, 9), kappa, s_xd, s_J


def c_of(err, kappa, scale):
    """Per-point c of err <= c * kappa * 2^-24 * scale."""
    return err / (kappa * U * np.maximum(scale, 1e-30))


# ---------------------------------------------------------------------------------------------
# calls through the C ABI into sentinel-padded buffers
# ---------------------------------------------------------------------------------------------

class DevBody:
    def __init__(self, body):
        from multiply_b200 import engine
        self.b = engine.Body(torch.from_numpy(body["verts_c"]), torch.from_numpy(body["weights"]),
                             cano_cell=body["cano_cell"])
        self.set_pose(body["verts_p"], body["tfs"])

    def set_pose(self, verts_p, tfs):
        self.b.set_pose(torch.from_numpy(np.asarray(verts_p, np.float32)), torch.from_numpy(np.asarray(tfs, np.float32)))

    def inverse(self, x, N, exact_far):
        from multiply_b200 import _lib as L
        xc, out = padded((N, 3)), padded(N, torch.uint8)
        L.call("mp_deform_inverse", self.b.handle, rows(torch.from_numpy(x), N), N, xc, out, int(exact_far))
        torch.cuda.synchronize()
        return take(xc, (N, 3), "x_c").numpy(), take(out, N, "outlier").numpy().astype(bool)

    def forward_jac(self, x, N):
        from multiply_b200 import _lib as L
        xd, J = padded((N, 3)), padded((N, 9))
        L.call("mp_deform_forward_jac", self.b.handle, rows(torch.from_numpy(x), N), N, xd, J)
        torch.cuda.synchronize()
        return take(xd, (N, 3), "x_d").numpy(), take(J, (N, 9), "Jinv").numpy()


_CASES = {}


def case(name):
    """Body, device body, both query sets and their references (cached per module)."""
    if name not in _CASES:
        body = make_body(name)
        gp = host_grid(body["verts_p"], POSED_CELL)
        gc = host_grid(body["verts_c"], np.float32(body["cano_cell"]) * np.float32(0.5))
        xq, cov_p = make_queries(body, body["verts_p"], gp, 1)
        xf, cov_c = make_queries(body, body["verts_c"], gc, 2)
        ip, op = brute_force(xq, body["verts_p"])
        ic, _ = brute_force(xf, body["verts_c"])
        _CASES[name] = dict(body=body, gp=gp, gc=gc, xq=xq, xf=xf, cov_p=cov_p, cov_c=cov_c, idx_p=ip, out_p=op,
                            idx_c=ic, inv=ref_inverse(xq, ip, body["weights"], body["tfs"]),
                            fwd=ref_forward(xf, ic, body["weights"], body["tfs"]), dev=DevBody(body))
    return _CASES[name]


def _record(name, what, c, kappa):
    MEASURED[(name, what)] = (float(c.max()) if c.size else 0.0, float(kappa.max()) if kappa.size else 0.0)
    bins = []
    for lo, hi in ((1, 10), (10, 100), (100, 1000), (1000, np.inf)):
        m = (kappa >= lo) & (kappa < hi)
        bins.append("kappa<%g: %s" % (hi, "%.2f" % c[m].max() if m.any() else "-"))
    print("DEFORMER %-10s %-4s worst c = %.3f  (kappa max %.3g, N = %d; %s)" % (
        name, what, MEASURED[(name, what)][0], MEASURED[(name, what)][1], c.size, ", ".join(bins)))


# ---------------------------------------------------------------------------------------------
# tests
# ---------------------------------------------------------------------------------------------

def test_host_grid_growth():
    """The scale-2 person needs more than kMaxCells cells at h = 0.05005 (posed) and 0.05 (canonical), so the kernel's
    grid-growth loop runs; at scale 0.5 it does not."""
    big, small = make_body("person_x2"), make_body("person")
    gp, gc = host_grid(big["verts_p"], POSED_CELL), host_grid(big["verts_c"], np.float32(0.1) * np.float32(0.5))
    assert gp["n_first"] > MAX_CELLS and gp["steps"] >= 1 and gp["h"] > POSED_CELL
    assert gc["n_first"] > MAX_CELLS and gc["steps"] >= 1
    assert host_grid(small["verts_p"], POSED_CELL)["steps"] == 0


@pytest.mark.parametrize("name", BODIES)
def test_inverse(name):
    """mp_deform_inverse: outlier flags bit-exact against the brute force, x_c within the kappa-scaled fp64 bound at
    the brute-force vertex, reruns bit-identical, and the grid-only mode (exact_far = 0) equal to the exact one on
    non-outliers with the same flags everywhere."""
    cs = case(name)
    x, N = cs["xq"], cs["xq"].shape[0]
    cov = cs["cov_p"]
    assert cov["on_boundary"] > 0.5 * (cs["body"]["n_query"] // 5)
    assert cov["border"] > 100 and cov["border_cell_R0"] > 10
    if name == "lattice":
        assert cov["ties_plus1"] >= 200
    if name == "tiny33":
        assert cov["proof_radius"] >= 1000, cov
    xc, out = cs["dev"].inverse(x, N, True)
    assert np.array_equal(out, cs["out_p"]), "outlier flags differ from the brute force at %d points" % int(
        (out != cs["out_p"]).sum())
    ref, kappa, scale = cs["inv"]
    c = c_of(np.abs(xc.astype(np.float64) - ref).max(1), kappa, scale)
    _record(name, "x_c", c, kappa)
    bad = c > C_GATE
    assert not bad.any(), "x_c off at %d points, first %s: got %s want %s (kappa %.3g)" % (
        int(bad.sum()), x[bad][0], xc[bad][0], ref[bad][0], kappa[bad][0])
    if name in ("lattice", "flat", "duplicates", "tiny33"):
        assert (kappa > 100).sum() > 50 and kappa.max() > 500
    xc2, out2 = cs["dev"].inverse(x, N, True)
    assert np.array_equal(xc2.view(np.uint32), xc.view(np.uint32)) and np.array_equal(out2, out)
    # grid-only search: deformer.py's outlier flags everywhere, the exact result wherever a vertex is within 0.1
    xg, og = cs["dev"].inverse(x, N, False)
    assert np.array_equal(og, cs["out_p"]), "grid-only outlier flags differ at %d points" % int((og != cs["out_p"]).sum())
    keep = ~og
    assert np.array_equal(xg[keep].view(np.uint32), xc[keep].view(np.uint32))


@pytest.mark.parametrize("name", BODIES)
def test_forward_jac(name):
    """mp_deform_forward_jac: x_d and Jinv (row-major inverse of the blended 3x3 of the nearest CANONICAL vertex)
    within the kappa-scaled fp64 bound; reruns bit-identical."""
    cs = case(name)
    x, N = cs["xf"], cs["xf"].shape[0]
    assert cs["cov_c"]["on_boundary"] > 0.5 * (cs["body"]["n_query"] // 5)
    xd, J = cs["dev"].forward_jac(x, N)
    rxd, rJ, kappa, s_xd, s_J = cs["fwd"]
    c_xd = c_of(np.abs(xd.astype(np.float64) - rxd).max(1), kappa, s_xd)
    c_J = c_of(np.abs(J.astype(np.float64) - rJ).max(1), kappa, s_J)
    _record(name, "x_d", c_xd, kappa)
    _record(name, "Jinv", c_J, kappa)
    for what, c, got, want in (("x_d", c_xd, xd, rxd), ("Jinv", c_J, J, rJ)):
        bad = c > C_GATE
        assert not bad.any(), "%s off at %d points, first %s: got %s want %s (kappa %.3g)" % (
            what, int(bad.sum()), x[bad][0], got[bad][0], want[bad][0], kappa[bad][0])
    xd2, J2 = cs["dev"].forward_jac(x, N)
    assert np.array_equal(xd2.view(np.uint32), xd.view(np.uint32)) and np.array_equal(J2.view(np.uint32),
                                                                                       J.view(np.uint32))


@pytest.mark.parametrize("name", ["person", "person_x2", "tiny1", "lattice"])
def test_sizes(name):
    """N = 0, 1, 127, 128, 129 (around the 128-thread block) and the whole set: row k of a call on the first N rows is
    bit-identical to row k of the call on every row, and nothing is written past N."""
    cs = case(name)
    xq, xf = cs["xq"], cs["xf"]
    full_c, full_o = cs["dev"].inverse(xq, xq.shape[0], True)
    full_d, full_J = cs["dev"].forward_jac(xf, xf.shape[0])
    for N in SIZES:
        for ef in (True, False):
            xc, o = cs["dev"].inverse(xq, N, ef)
            if ef:
                assert np.array_equal(xc.view(np.uint32), full_c[:N].view(np.uint32)) and np.array_equal(o, full_o[:N])
            else:
                assert np.array_equal(o, cs["out_p"][:N])
        xd, J = cs["dev"].forward_jac(xf, N)
        assert np.array_equal(xd.view(np.uint32), full_d[:N].view(np.uint32))
        assert np.array_equal(J.view(np.uint32), full_J[:N].view(np.uint32))


def test_set_pose_large_then_small():
    """A body posed at scale 2 (grown grid, more vertices per cell) and then at scale 0.5 answers bit for bit like a
    fresh body posed only at scale 0.5: no grid header, cell table or vertex-transform state survives a pose."""
    small = case("person")
    big = make_body("person_x2")
    body = small["body"]
    reused = DevBody(body)
    reused.set_pose(big["verts_p"], big["tfs"])
    reused.inverse(small["xq"][:4096], 4096, True)        # query the large pose once
    reused.forward_jac(small["xf"][:4096], 4096)
    reused.set_pose(body["verts_p"], body["tfs"])
    x, N = small["xq"], small["xq"].shape[0]
    for ef in (True, False):
        a, ao = reused.inverse(x, N, ef)
        b, bo = small["dev"].inverse(x, N, ef)
        assert np.array_equal(ao, bo) and np.array_equal(a.view(np.uint32), b.view(np.uint32))
    a, aJ = reused.forward_jac(small["xf"], small["xf"].shape[0])
    b, bJ = small["dev"].forward_jac(small["xf"], small["xf"].shape[0])
    assert np.array_equal(a.view(np.uint32), b.view(np.uint32)) and np.array_equal(aJ.view(np.uint32),
                                                                                   bJ.view(np.uint32))
