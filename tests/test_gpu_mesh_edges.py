"""GPU: the canonical-mesh kernels (csrc/mesh.cu) at the inputs where a grid search, a crossing test or a threshold
goes wrong, against oracle/mesh_port.py's brute-force definitions run on the GPU and against an independent analytic
inside test.

mesh.cu claims the same rounding as mesh_port (fp64 without FMA contraction, the same operation order), ties to the
lowest face index, a watertight +z crossing test and flags equal to the reference's `min` tests for every threshold.
So every comparison here is exact (torch.equal): dist2 (fp32), face_idx, dist_type, inside and the flags, with no
masks for near ties or near-surface points.

Meshes:
- voxel unions on a dyadic lattice (boundary squares split into two triangles, shared vertices merged, outward
  orientation): a box, an E with two overhangs (+z rays cross up to six times), a ring with a through-hole and a box with
  a cavity.  Queried on the lattice and at half- and quarter-lattice offsets, +z rays run through vertices, along edges,
  along vertical walls and across the split diagonals; `inside` is checked against the analytic point-in-voxel-set
  answer.  "Aligned" variants pad the face list with degenerate faces so that the grid's cells are the lattice's cells
  halved (lattice planes are cell boundaries), and add random fp32 points whose rounded crossing heights fall on either
  side of a cell boundary.
- tie meshes on a grid with h = 1/4 exactly (asserted from the plan): equidistant faces in different cells and rings
  with the lower index visited last, a fan whose faces all tie at their shared apex, points on cell faces, edges and
  corners, outside the grid in all 26 directions and far away.
- grid-shape edges (F = 1, flat, needle, margin 0 / larger than the mesh, unused / duplicate vertices and degenerate
  faces, one face over the whole grid, an offset of ~100, two far-apart components, a marching-cubes-scale body), each
  with the plan's invariants restated on the host.
Flags: thresholds 0.05, 0.0625, 0, -1e-3 and -0.05, points at, just below and just above the threshold distance in fp32
and just past the capped query's radius, rows all inside / all outside / mixed, standalone and fused into mp_render_rays.
"""
import ctypes as C

import numpy as np
import pytest
import torch

from multiply_b200 import scene as S
from oracle import mesh_port as port

from _abi import padded, take
from _setups import flags_from_taps, fused_setup, render_train

gpu = pytest.mark.gpu

THRESHOLDS = (0.05, 0.0625, 0.0, -1e-3, -0.05)


# ---------------------------------------------------------------------------------------------
# mesh builders (host, numpy)
# ---------------------------------------------------------------------------------------------

def voxel_mesh(occ, origin, step):
    """Boundary of the union of the occupied cells of occ [nx,ny,nz] (cell (i,j,k) spans origin + step * [i, i+1] x
    [j, j+1] x [k, k+1]): every square between an occupied and an empty (or outside) cell, split into two triangles
    (the diagonal alternates with the square's lattice parity), shared vertices merged, counter-clockwise seen from
    outside.  Returns (verts [V,3] fp32, faces [F,3] int64); coordinates must be exact in fp32."""
    occ = np.asarray(occ, bool)
    pad = np.pad(occ, 1)
    origin, step = np.asarray(origin, np.float64), np.broadcast_to(np.asarray(step, np.float64), (3,))
    vid, tris = {}, []

    def vert(q):
        return vid.setdefault(tuple(int(x) for x in q), len(vid))

    for a in range(3):
        u, v = (a + 1) % 3, (a + 2) % 3          # (u, v, a) right-handed: the quad (0,0) (1,0) (1,1) (0,1) faces +a
        for sgn in (1, -1):
            empty = ~np.roll(pad, -sgn, axis=a)
            for c in np.argwhere(pad & empty) - 1:
                base = c.copy()
                base[a] += 1 if sgn > 0 else 0
                q = []
                for du, dv in ((0, 0), (1, 0), (1, 1), (0, 1)):
                    x = base.copy()
                    x[u] += du
                    x[v] += dv
                    q.append(vert(x))
                if sgn < 0:
                    q = q[::-1]
                if int(base.sum()) & 1:
                    tris += [(q[0], q[1], q[2]), (q[0], q[2], q[3])]
                else:
                    tris += [(q[0], q[1], q[3]), (q[1], q[2], q[3])]
    lat = np.array(sorted(vid, key=vid.get), np.float64)
    v64 = origin + step * lat
    v = v64.astype(np.float32)
    assert np.array_equal(v.astype(np.float64), v64), "voxel coordinates must be exact in fp32"
    return torch.from_numpy(v), torch.tensor(tris, dtype=torch.int64)


def voxel_inside(occ, origin, step, pts):
    """Analytic point-in-voxel-set for points not on the union's boundary: the cell holding the point (every cell
    touching a point off the boundary has the same occupancy)."""
    occ = np.asarray(occ, bool)
    c = np.floor((np.asarray(pts, np.float64) - origin) / step).astype(np.int64)
    ok = np.all((c >= 0) & (c < np.array(occ.shape)), axis=1)
    out = np.zeros(len(c), bool)
    out[ok] = occ[c[ok, 0], c[ok, 1], c[ok, 2]]
    return out


def _shape(name):
    if name == "box":
        return np.ones((3, 2, 2), bool)
    if name == "e_overhang":      # spine at x = 0, slabs at z = 0, 2, 4: two overhangs
        e = np.zeros((5, 3, 5), bool)
        e[:, :, 0] = e[:, :, 2] = e[:, :, 4] = True
        e[0] = True
        return e
    if name == "ring_hole":       # a 2 x 2 through-hole along z
        r = np.ones((4, 4, 3), bool)
        r[1:3, 1:3, :] = False
        return r
    if name == "cavity":          # an inner, inward-facing component
        c = np.ones((4, 3, 4), bool)
        c[1:3, 1, 1:3] = False
        return c
    raise KeyError(name)


VOXEL_SHAPES = ("box", "e_overhang", "ring_hole", "cavity")
VOX_ORIGIN = np.array([-0.25, -0.125, -0.375])
ALIGNED_ORIGIN = np.array([-0.25, -0.125, 0.0])     # the grid's lo: cell_of(z) = floor(z / h) keeps z's rounding
VOX_STEP = 0.125


def degenerate_pad(v, f, F_target):
    """Pads the face list to F_target faces with degenerate faces (all three corners vertex f[0, 0]): they never cross
    a ray (zero area) and tie at that vertex only with the real faces around it, which have lower indices."""
    n = F_target - f.shape[0]
    assert n >= 0
    return v, torch.cat([f, f[:1, :1].expand(n, 3)])


def aligned_voxel_mesh(name):
    """The voxel mesh at ALIGNED_ORIGIN with margin 0 and a face count that makes the grid cell the lattice cell halved
    j times (h = step / 2^j): the lattice planes are cell boundaries.  Returns (v, f, h)."""
    occ = _shape(name)
    v, f = voxel_mesh(occ, ALIGNED_ORIGIN, VOX_STEP)
    cells = int(np.prod(occ.shape))
    j = 0
    while cells * 8 ** j < f.shape[0]:
        j += 1
    v, f = degenerate_pad(v, f, cells * 8 ** j)
    return v, f, VOX_STEP / 2 ** j


def watertight(f):
    """Every edge used by exactly two faces, in opposite directions."""
    f = np.asarray(f)
    e = np.concatenate([f[:, [0, 1]], f[:, [1, 2]], f[:, [2, 0]]])
    directed = {}
    for a, b in map(tuple, e):
        directed[(a, b)] = directed.get((a, b), 0) + 1
    return all(n == 1 and directed.get((b, a), 0) == 1 for (a, b), n in directed.items())


def signed_volume(v, f):
    t = np.asarray(v, np.float64)[np.asarray(f)]
    return float(np.einsum("ij,ij->i", t[:, 0], np.cross(t[:, 1], t[:, 2])).sum() / 6.0)


def tri_soup(*tris):
    """(verts, faces) of separate triangles given as 3x3 corner lists."""
    v = np.asarray(tris, np.float64).reshape(-1, 3)
    assert np.array_equal(v.astype(np.float32).astype(np.float64), v)
    return torch.from_numpy(v.astype(np.float32)), torch.arange(v.shape[0], dtype=torch.int64).reshape(-1, 3)


def cat_meshes(*meshes):
    vs, fs, off = [], [], 0
    for v, f in meshes:
        vs.append(v)
        fs.append(f + off)
        off += v.shape[0]
    return torch.cat(vs), torch.cat(fs)


def lattice(lo, hi, step):
    axes = [np.arange(lo[k], hi[k] + step / 2, step) for k in range(3)]
    g = np.stack(np.meshgrid(*axes, indexing="ij"), -1).reshape(-1, 3)
    return torch.from_numpy(g.astype(np.float32))


# ---------------------------------------------------------------------------------------------
# CPU: the builders
# ---------------------------------------------------------------------------------------------

@pytest.mark.parametrize("name", VOXEL_SHAPES)
def test_voxel_builder_watertight(name):
    occ = _shape(name)
    v, f = voxel_mesh(occ, VOX_ORIGIN, VOX_STEP)
    assert watertight(f)
    assert len(set(map(tuple, v.numpy().tolist()))) == v.shape[0], "vertices are merged"
    assert np.unique(f.numpy()).size == v.shape[0], "no unused vertices"
    assert signed_volume(v, f) == pytest.approx(occ.sum() * VOX_STEP ** 3, rel=1e-12), "outward orientation"
    # the analytic inside test agrees with the brute-force crossing parity at cell centres (never on the surface)
    c = lattice(VOX_ORIGIN - VOX_STEP / 2, VOX_ORIGIN + VOX_STEP * (np.array(occ.shape) + 0.5), VOX_STEP)
    ins = port.check_sign(v[None], f, c[None])[0].numpy()
    assert np.array_equal(ins, voxel_inside(occ, VOX_ORIGIN, VOX_STEP, c.numpy()))
    assert 0 < ins.sum() < len(ins)


def test_voxel_builder_cpu_sanity():
    """The E has columns with six crossings, the ring columns through its hole none, the cavity an inner shell."""
    v, f = voxel_mesh(_shape("e_overhang"), VOX_ORIGIN, VOX_STEP)
    p = torch.tensor([[VOX_ORIGIN[0] + 2.5 * VOX_STEP, VOX_ORIGIN[1] + 1.5 * VOX_STEP, VOX_ORIGIN[2] - 1.0]])
    fv = v.double()[f]
    t = port._ray_z_crossing(p.double()[:, None], fv[None, :, 0], fv[None, :, 1], fv[None, :, 2])
    assert int((t > 0).sum()) == 6
    v, f = voxel_mesh(_shape("cavity"), VOX_ORIGIN, VOX_STEP)
    assert f.shape[0] == 2 * (2 * (4 * 3 + 3 * 4 + 4 * 4) + 2 * (2 * 1 + 1 * 2 + 2 * 2))


# ---------------------------------------------------------------------------------------------
# GPU helpers
# ---------------------------------------------------------------------------------------------

def _engine():
    from multiply_b200 import engine
    return engine


def _L():
    from multiply_b200 import _lib as L
    return L


def host_plan_check(m, v, f, margin):
    """The plan's invariants, restated on the host: lo = bounds - margin, dims in 1..1024, ncell <= 4 max(F, 1), and
    n_refs = sum over faces of the cells of the face's fp32 bounding box under cell_of's fp64 formula."""
    p = m.plan
    vn = v.numpy().astype(np.float32)
    fn = f.numpy()
    F = fn.shape[0]
    lo = np.array(p.lo[:])
    dim = np.array(p.dim[:])
    assert np.array_equal(lo, vn.min(0).astype(np.float64) - np.float64(np.float32(margin)))
    assert ((dim >= 1) & (dim <= 1024)).all(), dim
    assert int(np.prod(dim.astype(np.int64))) <= 4 * max(min(F, 1 << 21), 1)
    inv_h = 1.0 / p.h
    tri = vn[fn]                                                     # [F,3,3]
    n = np.ones(F, np.int64)
    for k in range(3):
        def cell_of(x):
            t = np.floor((x.astype(np.float64) - lo[k]) * inv_h)
            return np.clip(t, 0, dim[k] - 1).astype(np.int64)
        n *= cell_of(tri[:, :, k].max(1)) - cell_of(tri[:, :, k].min(1)) + 1
    assert int(n.sum()) == p.n_refs
    assert p.V == v.shape[0] and p.F == F
    return p


def parity(m, v, f, pts):
    """dist2, face_idx, dist_type and inside equal the brute force bit for bit; returns (dist2, inside) of the port."""
    pts = pts.reshape(-1, 3).float().contiguous()
    pc = pts.cuda()
    d2, fi, dt = m.distance(pc)
    ins = m.check_sign(pc)
    fv = port.index_vertices_by_faces(v[None].cuda(), f.cuda())
    rd2, rfi, rdt = port.point_to_mesh_distance(pc[None], fv)
    rins = port.check_sign(v[None].cuda(), f.cuda(), pc[None])[0]
    torch.cuda.synchronize()
    for name, a, b in (("dist2", d2, rd2[0]), ("face_idx", fi, rfi[0]), ("dist_type", dt, rdt[0]),
                       ("inside", ins, rins)):
        bad = (a != b).nonzero()[:, 0]
        assert bad.numel() == 0, (name, bad.numel(), pts[bad[:4].cpu()].tolist(), a[bad[:4]].tolist(),
                                  b[bad[:4]].tolist())
    return rd2[0], rins


def _mesh(v, f, margin=0.01):
    return _engine().CanonicalMesh(v, f, margin=margin)


def _dyadic_queries(occ, extra=3, origin=VOX_ORIGIN):
    """The lattice and its half- and quarter-offsets over the shape's box plus `extra` quarter steps around it."""
    lo = origin - extra * VOX_STEP / 4
    hi = origin + VOX_STEP * np.array(occ.shape) + extra * VOX_STEP / 4
    return lattice(lo, hi, VOX_STEP / 4)


def _random_queries(occ, n, seed, origin=VOX_ORIGIN):
    """fp32 points over the shape's box, reaching well below it: +z rays from there cross the horizontal faces with
    crossing heights p.z + t whose rounding error (~ulp(t)) exceeds ulp(z), so they can round below a face's z."""
    g = torch.Generator().manual_seed(seed)
    ext = VOX_STEP * np.array(occ.shape, np.float64)
    lo = torch.tensor(origin - np.array([0.1, 0.1, ext[2] + 2.0]))
    hi = torch.tensor(origin + ext + 0.1)
    return (lo + (hi - lo) * torch.rand(n, 3, generator=g, dtype=torch.float64)).float()


# ---------------------------------------------------------------------------------------------
# 1-2: voxel meshes, exact parity and the analytic inside test
# ---------------------------------------------------------------------------------------------

@gpu
@pytest.mark.parametrize("aligned", [False, True], ids=["margin", "aligned"])
@pytest.mark.parametrize("name", VOXEL_SHAPES)
def test_voxel_mesh_parity_and_inside(name, aligned):
    occ = _shape(name)
    origin = ALIGNED_ORIGIN if aligned else VOX_ORIGIN
    if aligned:
        v, f, h = aligned_voxel_mesh(name)
        m = _mesh(v, f, margin=0.0)
        assert m.plan.h == h, ("the grid cell must be the halved lattice cell", m.plan.h, h)
    else:
        v, f = voxel_mesh(occ, origin, VOX_STEP)
        m = _mesh(v, f)
    host_plan_check(m, v, f, 0.0 if aligned else 0.01)
    pts = torch.cat([_dyadic_queries(occ, origin=origin), _random_queries(occ, 40000, 3, origin=origin)])
    rd2, rins = parity(m, v, f, pts)
    off_surface = (rd2 > 0).cpu().numpy()
    want = voxel_inside(occ, origin, VOX_STEP, pts.numpy())
    got = rins.cpu().numpy()
    bad = np.nonzero((got != want) & off_surface)[0]
    assert bad.size == 0, pts[bad[:4]].tolist()
    on = ~off_surface
    assert on.sum() > 300 and 0 < want[off_surface].sum() < off_surface.sum()


# ---------------------------------------------------------------------------------------------
# 3: ties and cell boundaries on a grid with h = 1/4
# ---------------------------------------------------------------------------------------------

TIE_F = 64          # with the bounds [0, 1]^3 and margin 0: h = cbrt(1 / 64) = 1/4, 4 x 4 x 4 cells


def _tie_mesh(*tris):
    """The given triangles first (lowest indices), then degenerate anchors at (0,0,0) and (1,1,1) that fix the bounds
    to [0, 1]^3, padded to TIE_F faces."""
    v, f = tri_soup(*tris, [[0, 0, 0]] * 3, [[1, 1, 1]] * 3)
    return degenerate_pad(v, f, TIE_F)


def _axis_tri(a, x, lo, hi):
    """A right triangle in the plane coordinate[a] = x whose other two coordinates span [lo, hi] (legs along them)."""
    u, w = (a + 1) % 3, (a + 2) % 3
    out = []
    for cu, cw in ((lo, lo), (hi, lo), (lo, hi)):
        c = [0.0, 0.0, 0.0]
        c[a], c[u], c[w] = x, cu, cw
        out.append(c)
    return out


def _at(a, x, rest):
    c = [rest, rest, rest]
    c[a] = x
    return c


def tie_cases():
    """(name, mesh, query points) of the tie scenarios."""
    cases = []
    lo, hi = 0.53125, 0.734375            # the triangle's projection holds (0.625, 0.625) in its interior
    for a in range(3):
        # equality at the ring bound: the query sits 1/16 below the boundary 0.5 in cell 1; the higher-index face is
        # in the same cell at 1/16, the lower-index one lies in the boundary plane (cell 2, ring 1): the ring bound and
        # the cell's box distance equal the best distance exactly
        cases.append(("ring_bound_eq_%d" % a, _tie_mesh(_axis_tri(a, 0.5, lo, hi), _axis_tri(a, 0.375, lo, hi)),
                      [_at(a, 0.4375, 0.625)]))
        # the same the other way: the query at 0.5625 in cell 2, the lower-index face in cell 1 at 1/8
        cases.append(("ring_below_%d" % a, _tie_mesh(_axis_tri(a, 0.4375, lo, hi), _axis_tri(a, 0.6875, lo, hi)),
                      [_at(a, 0.5625, 0.625)]))
        # ring 2 against ring 1: the lower-index face in cell 3 (two rings away) ties with one in cell 0
        cases.append(("ring2_%d" % a, _tie_mesh(_axis_tri(a, 0.75, lo, hi), _axis_tri(a, 0.0, lo, hi)),
                      [_at(a, 0.375, 0.625)]))
    # a fan of four faces around the apex (0.5, 0.5, 0.5), a cell corner; the apex is vertex a, b, c, a of its faces
    apex, z0 = [0.5, 0.5, 0.5], 0.375
    base = [[0.625, 0.5 - 0.125, z0], [0.625, 0.625, z0], [0.375, 0.625, z0], [0.375, 0.375, z0]]
    fan = []
    for k in range(4):
        tri = [apex, base[k], base[(k + 1) % 4]]
        r = k % 3
        fan.append(tri[r:] + tri[:r])
    apex_q = [[0.5, 0.5, 0.5 + j / 32] for j in range(0, 9)] + [[0.5, 0.5, 0.75]]
    cases.append(("fan", _tie_mesh(*fan), apex_q))
    cases.append(("fan_rev", _tie_mesh(*fan[::-1]), apex_q))
    cases.append(("fan_rot", _tie_mesh(*(fan[1:] + fan[:1])), apex_q))       # face 0 has the apex as vertex c
    return cases


def _cell_lattice_queries():
    """Every point of spacing 1/32 over [-1/4, 5/4]^3 (cell faces, edges and corners of the 1/4 grid, and outside it in
    all 26 directions), and far points in the 26 directions."""
    pts = [lattice([-0.25] * 3, [1.25] * 3, 1 / 32)]
    d = np.array([(i, j, k) for i in (-1, 0, 1) for j in (-1, 0, 1) for k in (-1, 0, 1) if (i, j, k) != (0, 0, 0)])
    for s in (3.0, 1e3, 1e5):
        pts.append(torch.from_numpy((0.5 + s * d).astype(np.float32)))
    return torch.cat(pts)


@gpu
def test_tie_meshes_exact():
    cells = _cell_lattice_queries()
    for name, (v, f), q in tie_cases():
        m = _mesh(v, f, margin=0.0)
        p = host_plan_check(m, v, f, 0.0)
        assert p.h == 0.25 and tuple(p.dim) == (4, 4, 4), (name, p.h, tuple(p.dim))
        q = torch.tensor(q, dtype=torch.float32)
        parity(m, v, f, torch.cat([q, cells]))
        # the scenario's queries resolve to the lowest-index face, at an exact tie
        d2, fi, dt = m.distance(q.cuda())
        fv = v[f]
        all_d2, _ = port._closest_point_triangle(q.double()[:, None], fv[None, :, 0].double(), fv[None, :, 1].double(),
                                                 fv[None, :, 2].double())
        if name.startswith("fan"):
            assert bool((all_d2[:, :4] == all_d2[:, :1]).all()), name
            assert torch.equal(fi.cpu(), torch.zeros(len(q), dtype=torch.int64)), name
        else:
            assert bool((all_d2[:, 0] == all_d2[:, 1]).all()) and torch.equal(fi.cpu(), torch.zeros(1, dtype=torch.int64))


@gpu
def test_sparse_two_components_long_ring_search():
    """Two small dense components at opposite corners of a large box: queries near neither walk many empty rings."""
    v, f = S.make_body_mesh(100)
    v = v * 0.02
    v, f = cat_meshes((v, f), (v + 1.0, f))
    m = _mesh(v, f)
    host_plan_check(m, v, f, 0.01)
    assert min(m.plan.dim) >= 16, tuple(m.plan.dim)
    g = torch.Generator().manual_seed(9)
    pts = torch.cat([-0.2 + 1.4 * torch.rand(3000, 3, generator=g),
                     torch.tensor([[0.5, 0.5, 0.5], [0.25, 0.75, 0.5], [1.2, -0.2, 0.5], [0.5, 0.5, 40.0]])])
    parity(m, v, f, pts)


# ---------------------------------------------------------------------------------------------
# 4: grid-shape edges
# ---------------------------------------------------------------------------------------------

def _flat(z=0.3, n=8):
    """A planar triangulated square (all z equal)."""
    xs = np.linspace(-0.5, 0.5, n + 1)
    X, Y = np.meshgrid(xs, xs, indexing="ij")
    v = np.stack([X, Y, np.full_like(X, z)], -1).reshape(-1, 3).astype(np.float32)
    idx = lambda i, j: i * (n + 1) + j
    f = []
    for i in range(n):
        for j in range(n):
            f += [(idx(i, j), idx(i + 1, j), idx(i + 1, j + 1)), (idx(i, j), idx(i + 1, j + 1), idx(i, j + 1))]
    return torch.from_numpy(v), torch.tensor(f, dtype=torch.int64)


def _needle(n=64, r=4e-4):
    """A thin triangular tube along x: extent ratio 1 / r > 1024."""
    xs = np.linspace(0.0, 1.0, n + 1)
    ring = np.array([[0.0, 0.0], [r, 0.0], [0.0, r]])
    v = np.concatenate([np.column_stack([np.full(3, x), ring]) for x in xs]).astype(np.float32)
    f = []
    for i in range(n):
        for k in range(3):
            a, b, c, d = 3 * i + k, 3 * i + (k + 1) % 3, 3 * (i + 1) + k, 3 * (i + 1) + (k + 1) % 3
            f += [(a, b, d), (a, d, c)]
    return torch.from_numpy(v), torch.tensor(f, dtype=torch.int64)


def _messy():
    """The E with unused vertices (one far off, which widens the grid), duplicated vertices taken by some faces, and
    degenerate faces: collinear corners along an edge, and three equal corners."""
    v, f = voxel_mesh(_shape("e_overhang"), VOX_ORIGIN, VOX_STEP)
    V = v.shape[0]
    v = torch.cat([v, torch.tensor([[2.0, 2.0, 2.0], [0.0, 0.0, 0.0]]), v[:16]])
    f = f.clone()
    f[::5] = torch.where(f[::5] < 16, f[::5] + V + 2, f[::5])          # faces on the duplicates
    e = f[0]
    mid = v[e[:2]].mean(0, keepdim=True)
    v = torch.cat([v, mid])
    f = torch.cat([f, torch.tensor([[int(e[0]), v.shape[0] - 1, int(e[1])], [int(e[2])] * 3])])
    return v, f


def _whole_grid_face():
    """A small dense mesh plus one face across its whole box (binned into every cell of its plane's band)."""
    v, f = voxel_mesh(_shape("ring_hole"), VOX_ORIGIN, VOX_STEP)
    lo, hi = v.min(0)[0], v.max(0)[0]
    big = torch.stack([lo, torch.tensor([hi[0], lo[1], hi[2]]), hi])
    return cat_meshes((v, f), (big, torch.tensor([[0, 1, 2]])))


def grid_edge_meshes():
    e = voxel_mesh(_shape("e_overhang"), VOX_ORIGIN, VOX_STEP)
    return {
        "single_face": (tri_soup([[0.0, 0.0, 0.0], [0.5, 0.125, 0.0], [0.25, 0.375, 0.25]]), 0.01),
        "flat": (_flat(), 0.01),
        "flat_margin0": (_flat(), 0.0),
        "needle": (_needle(), 0.0),
        "margin0": (e, 0.0),
        "margin_huge": (e, 2.0),
        "messy": (_messy(), 0.01),
        "whole_grid_face": (_whole_grid_face(), 0.01),
        "offset_100": ((e[0] + torch.tensor([100.0, -100.0, 100.25]), e[1]), 0.01),
        "body_offset_100": ((S.make_body_mesh(101)[0] + torch.tensor([100.0, 99.5, -100.0]), S.make_body_mesh(101)[1]),
                            0.01),
    }


def _around(v, n, seed, spread=0.1):
    """Near-vertex, box and outside points, plus the vertices and the edge midpoints' lattice-free neighbours."""
    g = torch.Generator().manual_seed(seed)
    lo, hi = v.min(0)[0].double(), v.max(0)[0].double()
    ext = (hi - lo).clamp_min(1e-3)
    k = n // 3
    near = v[torch.randint(0, v.shape[0], (k,), generator=g)].double() + spread * ext.max() * torch.randn(k, 3,
                                                                                                         generator=g,
                                                                                                         dtype=torch.float64)
    box = lo + ext * torch.rand(k, 3, generator=g, dtype=torch.float64)
    out = lo - ext + 3 * ext * torch.rand(n - 2 * k, 3, generator=g, dtype=torch.float64)
    return torch.cat([near, box, out, v.double()]).float()


@gpu
@pytest.mark.parametrize("name", ["single_face", "flat", "flat_margin0", "needle", "margin0", "margin_huge", "messy",
                                  "whole_grid_face", "offset_100", "body_offset_100"])
def test_grid_shape_edges(name):
    (v, f), margin = grid_edge_meshes()[name]
    m = _mesh(v, f, margin=margin)
    p = host_plan_check(m, v, f, margin)
    if name == "needle":
        ext = v.max(0)[0] - v.min(0)[0]
        assert float(ext.max() / ext.min()) > 1024 and max(p.dim) == 1024
    if name.startswith("flat"):
        assert p.dim[2] == 1
    if name == "whole_grid_face":
        assert p.n_refs >= p.dim[0] * p.dim[1] * p.dim[2]
    pts = _around(v, 6000, 17)
    if name in ("margin0", "margin_huge", "messy", "whole_grid_face", "offset_100"):
        base = _dyadic_queries(_shape("e_overhang"))
        pts = torch.cat([pts, base + (torch.tensor([100.0, -100.0, 100.25]) if name == "offset_100" else 0.0)])
    parity(m, v, f, pts)


@gpu
def test_marching_cubes_scale_body():
    v, f = S.make_body_mesh(100, step=0.005)
    assert f.shape[0] > 3e5
    m = _mesh(v, f)
    host_plan_check(m, v, f, 0.01)
    parity(m, v, f, _around(v, 900, 23, spread=0.01)[:1000])


# ---------------------------------------------------------------------------------------------
# 5: surface flags at the threshold
# ---------------------------------------------------------------------------------------------

Z_TOP = -(2.0 ** -40)      # the slab's top face: distances above / below it are not fp32 numbers themselves


def slab_mesh():
    """The box [-1, 1]^2 x [-1, Z_TOP]: points over (0.1, 0.2) within 0.8 of the top face are nearest to its interior."""
    return voxel_mesh(np.ones((1, 1, 1), bool), [-1.0, -1.0, -1.0], [2.0, 2.0, 1.0 + Z_TOP])


def threshold_points(thr, n_ulps=24):
    """fp32 points above (outside) and below (inside) the slab's top face near the distance |thr|, chosen so that
    sqrtf(float(d2)) falls just below, on and just above |thr| in fp32, and points just past the capped query's radius
    |thr| (1 + 1e-6) and on the surface.  Returns (points [N,3], d [N] fp32 as the reference computes it)."""
    t = abs(np.float32(thr))
    zs = []
    for side in (1, -1):
        z0 = np.float32(Z_TOP + side * float(t))
        z = z0
        for _ in range(n_ulps):
            z = np.nextafter(z, np.float32(-np.inf))
        for _ in range(2 * n_ulps + 1):
            zs.append(z)
            z = np.nextafter(z, np.float32(np.inf))
        cap = float(t) * (1.0 + 1e-6)
        for k in range(4):
            zs.append(np.nextafter(np.float32(Z_TOP + side * cap), np.float32(side * np.inf)) if k == 0 else
                      np.float32(Z_TOP + side * cap * (1 + k * 1e-7)))
    zs += [np.float32(Z_TOP), np.float32(0.0), np.nextafter(np.float32(Z_TOP), np.float32(-1))]
    z = np.array(zs, np.float32)
    pts = np.column_stack([np.full_like(z, 0.1), np.full_like(z, 0.2), z])
    delta = z.astype(np.float64) - Z_TOP
    d = np.sqrt((delta * delta).astype(np.float32))
    return torch.from_numpy(pts), torch.from_numpy(d), delta


def _flags_exact(m, v, f, x, n, thr):
    off, inn = m.surface_flags(x.cuda(), n, thr)
    ro, ri, rmin = port.check_off_in_surface(x.cuda(), n, v.cuda(), f.cuda(), thr)
    torch.cuda.synchronize()
    for name, a, b in (("off", off, ro), ("in", inn, ri)):
        bad = (a != b).nonzero()[:, 0]
        assert bad.numel() == 0, (name, thr, bad.numel(), rmin[bad[:4]].tolist())
    return off, inn, rmin


@gpu
@pytest.mark.parametrize("thr", THRESHOLDS)
def test_flags_at_threshold_distance(thr):
    v, f = slab_mesh()
    m = _mesh(v, f)
    pts, d, delta = threshold_points(thr)
    t = np.float32(abs(thr))
    dn = d.numpy()
    if thr != 0:
        # the set straddles |thr| in fp32, and holds points whose exact distance exceeds |thr| while their fp32 distance
        # equals it (inside the cap), and points past the cap
        assert (dn < t).any() and (dn == t).any() and (dn > t).any()
        assert ((dn == t) & (np.abs(delta) > float(t))).any()
        assert (np.abs(delta) > float(t) * (1 + 1e-6)).any()
    assert (dn == 0).any()
    off, inn, rmin = _flags_exact(m, v, f, pts, 1, thr)
    s = rmin.cpu().numpy()
    assert (s == np.float32(thr)).any() or thr == 0.0 and (s == 0).any()
    # pairs of samples per row: every combination of two points in rows of N_samples = 2
    k = pts.shape[0]
    i, j = np.meshgrid(np.arange(k), np.arange(k), indexing="ij")
    pairs = pts[torch.from_numpy(np.stack([i.ravel(), j.ravel()], 1).ravel())]
    _flags_exact(m, v, f, pairs, 2, thr)


def _ray_samples(v, rows, ns, seed, scale=0.3):
    """Rows of ns samples along random segments through the mesh's box (rows that stay inside, stay outside or cross)."""
    g = torch.Generator().manual_seed(seed)
    lo, hi = v.min(0)[0], v.max(0)[0]
    o = lo + (hi - lo) * torch.rand(rows, 1, 3, generator=g)
    d = torch.nn.functional.normalize(torch.randn(rows, 1, 3, generator=g), dim=-1)
    t = torch.linspace(-1.0, 1.0, ns)[None, :, None] * scale * torch.rand(rows, 1, 1, generator=g)
    return (o + t * d).reshape(-1, 3)


@gpu
@pytest.mark.parametrize("thr", THRESHOLDS)
def test_flags_rows_body_and_voxels(thr):
    """Rows of N_samples = 1, 2 and 97 on the body mesh and on the voxel meshes (whose lattice queries sit at the dyadic
    threshold 0.0625 from the surface, on it, and 0.03125 from it), with rows all inside, all outside and mixed."""
    v, f = S.make_body_mesh(100)
    m = _mesh(v, f)
    offs, ins = [], []
    for rows, ns, seed in ((1, 1, 1), (3, 2, 2), (2000, 1, 3), (1500, 2, 4), (400, 97, 5), (1, 97, 6)):
        x = _ray_samples(v, rows, ns, seed, scale=0.05 if ns == 97 else 0.3)
        off, inn, _ = _flags_exact(m, v, f, x, ns, thr)
        offs.append(off)
        ins.append(inn)
    off, inn = torch.cat(offs), torch.cat(ins)
    assert 0 < int(off.sum()) < off.numel() and 0 < int(inn.sum()) < inn.numel()
    for name in VOXEL_SHAPES:
        occ = _shape(name)
        vv, ff = voxel_mesh(occ, VOX_ORIGIN, VOX_STEP)
        mm = _mesh(vv, ff)
        q = _dyadic_queries(occ)
        _flags_exact(mm, vv, ff, q, 1, thr)
        n = (q.shape[0] // 97) * 97
        _flags_exact(mm, vv, ff, q[:n], 97, thr)
        ins = torch.from_numpy(voxel_inside(occ, VOX_ORIGIN, VOX_STEP, q.numpy()))
        deep = q[ins][: (int(ins.sum()) // 2) * 2]           # all-inside rows of two
        _flags_exact(mm, vv, ff, deep, 2, thr)
        outside = q[~ins][: (int((~ins).sum()) // 2) * 2]     # rows of two outside (or on the surface)
        _flags_exact(mm, vv, ff, outside, 2, thr)


@gpu
def test_flags_negative_threshold_inside_depth():
    """With thr < 0 an inside sample at depth d < |thr| keeps off (s = -d > thr), one at depth > |thr| clears it; an
    outside sample never clears it.  (Before the fix every inside sample cleared off.)"""
    v, f = slab_mesh()
    m = _mesh(v, f)
    x = torch.tensor([[0.1, 0.2, Z_TOP - 0.01], [0.1, 0.2, Z_TOP - 0.2], [0.1, 0.2, 0.3], [0.1, 0.2, Z_TOP]])
    off, inn = m.surface_flags(x.cuda(), 1, -0.05)
    assert off.tolist() == [True, False, True, True]       # on the top face: outside, s = +0 > thr
    assert inn.tolist() == [True, True, False, True]
    _flags_exact(m, v, f, x, 1, -0.05)
    off, _ = m.surface_flags(x.cuda(), 1, float("-inf"))
    assert off.tolist() == [True, True, True, True]
    off, _ = m.surface_flags(x.cuda(), 1, float("inf"))
    assert off.tolist() == [False] * 4


@gpu
def test_flags_nan_threshold_rejected():
    L = _L()
    v, f = slab_mesh()
    m = _mesh(v, f)
    x = torch.zeros(4, 3, device="cuda")
    with pytest.raises(L.MpError, match="NaN"):
        m.surface_flags(x, 2, float("nan"))


@gpu
@pytest.mark.parametrize("thr", [-0.05, -1e-3, 0.05])
def test_fused_flags_threshold(thr):
    """mp_render_rays' fused flags at thr equal mp_mesh_surface_flags on the main pass's canonical points and the
    brute-force flags of those points; a NaN threshold is an error."""
    sc, r, inp, hits, meshes, rngs, tb = fused_setup()
    on = render_train(r, inp, hits, rngs, tb, meshes, persons=[0, 1], thr=thr)
    xcs = []
    want_off, want_in = flags_from_taps(sc, r, inp, hits, meshes, on, [0, 1], thr=thr, xc_out=xcs)
    assert torch.equal(on["index_off_surface"], want_off)
    assert torch.equal(on["index_in_surface"], want_in)
    for p, (h, xc) in enumerate(xcs):
        v, f = S.make_body_mesh(100 + p)
        o, i = meshes[p].surface_flags(xc, r.n, thr)
        ro, ri, _ = port.check_off_in_surface(xc, r.n, v.cuda(), f.cuda(), thr)
        assert torch.equal(o, ro) and torch.equal(i, ri)
    if thr == -0.05:
        # the threshold matters: some ray keeps off only because of inside samples shallower than |thr|
        o0, _ = flags_from_taps(sc, r, inp, hits, meshes, on, [0, 1], thr=0.0)
        assert bool((want_off & ~o0).any())
    L = _L()
    with pytest.raises(L.MpError, match="NaN"):
        render_train(r, inp, hits, rngs, tb, meshes, persons=[0, 1], thr=float("nan"))


# ---------------------------------------------------------------------------------------------
# 6: ABI hygiene
# ---------------------------------------------------------------------------------------------

def _body():
    return S.make_body_mesh(100)


@gpu
def test_abi_null_outputs_zero_n_and_padding():
    L = _L()
    v, f = _body()
    m = _mesh(v, f)
    pts = _around(v, 300, 31).cuda()
    d2, fi, dt = m.distance(pts)
    ins = m.check_sign(pts)
    for N in (0, 1, 127, 128, 129):
        o, oi, ot, ou = padded(N), padded(N, torch.int64), padded(N, torch.int32), padded(N, torch.uint8)
        L.call("mp_mesh_distance", m.handle, pts, N, o, oi, ot)
        L.call("mp_mesh_check_sign", m.handle, pts, N, ou)
        torch.cuda.synchronize()
        assert torch.equal(take(o, N, "sq_dist"), d2[:N].cpu()) and torch.equal(take(oi, N, "face_idx"), fi[:N].cpu())
        assert torch.equal(take(ot, N, "dist_type"), dt[:N].cpu())
        assert torch.equal(take(ou, N, "inside").bool(), ins[:N].cpu())
        # NULL face_idx / dist_type
        o2 = padded(N)
        L.call("mp_mesh_distance", m.handle, pts, N, o2, None, None)
        torch.cuda.synchronize()
        assert torch.equal(o2, o)
        # flags: rows = N of 2 samples
        x = pts[:2].repeat(N + 1, 1)[: 2 * N].contiguous() if N else pts
        fo, fn = padded(N, torch.uint8), padded(N, torch.uint8)
        L.call("mp_mesh_surface_flags", m.handle, x, N, 2, 0.05, fo, fn)
        torch.cuda.synchronize()
        fo, fn = take(fo, N, "off_surface"), take(fn, N, "in_surface")
        if N:
            ro, ri = m.surface_flags(x, 2, 0.05)
            assert torch.equal(fo.bool(), ro.cpu()) and torch.equal(fn.bool(), ri.cpu())


@gpu
def test_abi_reruns_two_handles_and_rebuild():
    v, f = _body()
    ve, fe = voxel_mesh(_shape("e_overhang"), VOX_ORIGIN, VOX_STEP)
    pts = torch.cat([_around(v, 3000, 41), _dyadic_queries(_shape("e_overhang"))[:3000]])
    pts = pts[: pts.shape[0] // 2 * 2].cuda()
    a = _mesh(v, f)
    ra = a.distance(pts) + (a.check_sign(pts), a.surface_flags(pts, 2, 0.05))
    b = _mesh(ve, fe)
    rb = b.distance(pts) + (b.check_sign(pts), b.surface_flags(pts, 2, 0.05))
    for _ in range(2):     # interleaved reruns on both live handles are bit-identical
        for m, want in ((a, ra), (b, rb)):
            got = m.distance(pts) + (m.check_sign(pts), m.surface_flags(pts, 2, 0.05))
            for x, y in zip(got[:4], want[:4]):
                assert torch.equal(x, y)
            assert all(torch.equal(x, y) for x, y in zip(got[4], want[4]))
    # a mesh built after another one was freed (its storage is reused) answers as the one built while both lived
    del a
    torch.cuda.synchronize()
    c = _mesh(ve, fe)
    rc = c.distance(pts) + (c.check_sign(pts),)
    for x, y in zip(rc, rb[:4]):
        assert torch.equal(x, y)
    parity(c, ve, fe, pts.cpu())


@gpu
def test_abi_errors_leave_nothing_behind():
    L = _L()
    v, f = voxel_mesh(_shape("box"), VOX_ORIGIN, VOX_STEP)
    V = v.shape[0]
    vd, fd = v.cuda(), f.cuda()
    scratch = L.workspace(L.MP_MESH_PLAN_SCRATCH_BYTES, "cuda")

    def rejected(msg, faces, Vn, Fn, margin):
        p = L.MeshPlan()
        p.V, p.F, p.n_refs, p.storage_bytes = -5, -5, -5, 12345
        with pytest.raises(L.MpError, match=r"failed \(-\d+\): .*" + msg):
            L.call("mp_mesh_plan", vd, Vn, faces, Fn, margin, scratch, p)
        assert (p.V, p.F, p.n_refs, p.storage_bytes) == (-5, -5, -5, 12345), "no plan is written"

    for (row, col), bad in (((len(f) // 2, 1), -1), ((len(f) // 2, 1), V), ((0, 0), V)):
        fb = f.clone()
        fb[row, col] = bad
        rejected("outside", fb.cuda(), V, f.shape[0], 0.01)
    for Vn, Fn, margin, msg in ((2, f.shape[0], 0.01, "V >= 3"), (V, 0, 0.01, "F >= 1"), (V, f.shape[0], -0.01, "margin")):
        rejected(msg, fd, Vn, Fn, margin)
    # storage one byte short: an error and no handle
    p = L.MeshPlan()
    L.call("mp_mesh_plan", vd, V, fd, f.shape[0], 0.01, scratch, p)
    storage = L.workspace(p.storage_bytes, "cuda")
    h = L.Handle("mp_mesh_free")
    with pytest.raises(L.MpError, match=r"failed \(-\d+\): .*storage"):
        L.call("mp_mesh_create", p, vd, fd, storage, p.storage_bytes - 1, C.byref(h))
    assert h.value is None
    L.call("mp_mesh_create", p, vd, fd, storage, p.storage_bytes, C.byref(h))
    assert h.value is not None
