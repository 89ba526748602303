"""float64 references for mesh extraction (DESIGN §3.7) that do not restate its triangulation: the vertex rule, face
locality and per-cube counts, directed-edge balance, components and their signed volumes, areas and Euler
characteristics, and the largest component.  numpy / scipy on the grid and the mesh only; shared by the GPU invariant
tests and the CPU test that keeps these references honest against oracle/mesh_extract.py."""
import math

import numpy as np
from scipy.sparse import coo_matrix
from scipy.sparse.csgraph import connected_components


def crossings(g, level):
    """[R+1]^3 x 3 bool: the lattice edge from point p along axis a has exactly one end with (double)v < level."""
    below = np.asarray(g, np.float32).astype(np.float64) < float(level)
    n1 = below.shape[0]
    c = np.zeros((n1, n1, n1, 3), bool)
    c[:-1, :, :, 0] = below[:-1] != below[1:]
    c[:, :-1, :, 1] = below[:, :-1] != below[:, 1:]
    c[:, :, :-1, 2] = below[:, :, :-1] != below[:, :, 1:]
    return c


def vertex_rule(g, level, center=None, extent=None, pad=1.1):
    """The vertices marching cubes must emit: (verts [V,3] fp32, edge ids [V] = 3 * lattice index + axis, ascending).
    t = (level - v0) / (v1 - v0) along the edge from its lower end, mapped by ((p / R - 0.5) * pad) * extent + centre
    in fp64 and rounded to fp32 once; extent=None is the lattice form (centre R/2, extent R, pad 1)."""
    v = np.asarray(g, np.float32).astype(np.float64)
    R = v.shape[0] - 1
    if extent is None:
        center, extent, pad = (R / 2.0,) * 3, float(R), 1.0
    eid = np.flatnonzero(crossings(g, level))      # C order over (x, y, z, axis) is edge-id order
    idx, axis = np.divmod(eid, 3)
    p = np.stack(np.unravel_index(idx, v.shape), axis=1)
    flat = v.reshape(-1)
    v0 = flat[idx]
    v1 = flat[idx + np.array([(R + 1) ** 2, R + 1, 1])[axis]]
    c = p.astype(np.float64)
    c[np.arange(len(c)), axis] += (float(level) - v0) / (v1 - v0)
    verts = (((c / float(R) - 0.5) * float(pad)) * float(extent) + np.asarray(center, np.float64)).astype(np.float32)
    return verts, eid


def _edge_points(eid, R):
    idx, axis = np.divmod(np.asarray(eid, np.int64), 3)
    return np.stack(np.unravel_index(idx, (R + 1,) * 3), axis=1), axis


def face_cubes(g, level, faces, eid):
    """Locality and per-cube counts.  Every face has three distinct vertices whose lattice edges belong to one cube;
    faces come in non-decreasing cube order; in every cube with E crossed edges and T triangles, T = 0 iff E = 0,
    E - T is even with (E - T) / 2 polygons in [1, 4], and every crossed edge is used by one of its triangles.
    A triangle whose three edges lie in one cube face belongs to either cube of that face; it takes the cube of a
    neighbouring face in the list, or, between two cubes, the one its polygon count needs.  Returns each face's cube
    (x-major index)."""
    R = np.asarray(g).shape[0] - 1
    F = len(faces)
    faces = np.asarray(faces, np.int64).reshape(-1, 3)
    assert F == 0 or (faces.min() >= 0 and faces.max() < len(eid))
    assert np.all((faces[:, 0] != faces[:, 1]) & (faces[:, 1] != faces[:, 2]) & (faces[:, 0] != faces[:, 2]))
    p, a = _edge_points(eid, R)
    # cubes holding edge (p, a): q_a = p_a, q_k in {p_k - 1, p_k} otherwise, inside [0, R-1]
    lo = np.clip(p - (np.arange(3)[None] != a[:, None]), 0, R - 1)
    hi = np.clip(p, 0, R - 1)
    flo = lo[faces].max(axis=1)
    fhi = hi[faces].min(axis=1)
    assert np.all(flo <= fhi), "a face whose edges share no cube"
    n_cand = np.prod(fhi - flo + 1, axis=1)
    assert np.all(n_cand <= 2)
    key = lambda q: (q[..., 0] * R + q[..., 1]) * R + q[..., 2]
    ca, cb = key(flo), key(fhi)
    cube = np.where(n_cand == 1, ca, -1)
    cross = crossings(g, level)
    E = np.zeros((R, R, R), np.int64)
    for ax in range(3):
        for d1, d2 in ((0, 0), (0, 1), (1, 0), (1, 1)):
            s = [slice(0, R)] * 3
            k1, k2 = [k for k in range(3) if k != ax]
            s[k1], s[k2] = slice(d1, d1 + R), slice(d2, d2 + R)
            E += cross[s[0], s[1], s[2], ax]
    E = E.reshape(-1)
    pending = []
    for i in np.flatnonzero(n_cand == 2):      # ca < cb; the neighbours' cubes bound it by the order
        prev = cube[i - 1] if i > 0 else -1
        nxt = cube[i + 1] if i + 1 < F else -1
        if prev == cb[i] or (nxt == cb[i] and prev != ca[i]):
            cube[i] = cb[i]
        elif nxt == ca[i] or (prev == ca[i] and nxt not in (cb[i], -1)):
            cube[i] = ca[i]
        else:
            pending.append(i)
    T = np.bincount(cube[cube >= 0], minlength=R ** 3)
    for i in pending:                          # between its two cubes: the one whose E - T is odd without it
        cube[i] = ca[i] if (E[ca[i]] - T[ca[i]]) % 2 else cb[i]
        T[cube[i]] += 1
    assert np.all(cube >= 0)
    assert np.all(np.diff(cube) >= 0), "faces out of cube order"
    T = np.bincount(cube, minlength=R ** 3)
    assert np.array_equal(T == 0, E == 0)
    assert np.all((E - T) % 2 == 0)
    P = (E - T) // 2
    assert np.all((P[E > 0] >= 1) & (P[E > 0] <= 4))
    used = np.unique(cube[:, None] * len(eid) + faces)
    assert np.array_equal(np.bincount(used // max(len(eid), 1), minlength=R ** 3), E)
    return cube


def edge_use(faces, V):
    """(undirected edges [U,2] a < b, their use counts, count(a->b), count(b->a))."""
    faces = np.asarray(faces, np.int64).reshape(-1, 3)
    a = faces.reshape(-1)
    b = faces[:, [1, 2, 0]].reshape(-1)
    und, inv = np.unique(np.minimum(a, b) * V + np.maximum(a, b), return_inverse=True)
    fwd = np.bincount(inv, weights=(a < b), minlength=len(und)).astype(np.int64)
    rev = np.bincount(inv, weights=(a > b), minlength=len(und)).astype(np.int64)
    return np.stack([und // V, und % V], axis=1), fwd + rev, fwd, rev


def balance(g, faces, eid, closed):
    """Closure and consistent winding: count(a->b) = count(b->a) for every undirected edge, used by 2 or 4 faces.  On a
    grid whose boundary holds points below the level, the unbalanced edges are segments in one boundary face of the
    lattice.  Returns the number of unbalanced edges."""
    R = np.asarray(g).shape[0] - 1
    edges, use, fwd, rev = edge_use(faces, len(eid))
    bad = fwd != rev
    if closed:
        assert not bad.any(), "%d unbalanced edges" % int(bad.sum())
        assert np.all((use == 2) | (use == 4))
        return 0
    p, a = _edge_points(eid, R)
    planes = np.zeros(len(eid), np.int64)          # bit 2k + side: the edge lies in the boundary plane x_k = side * R
    for k in range(3):
        off = a != k
        planes |= ((p[:, k] == 0) & off).astype(np.int64) << (2 * k)
        planes |= ((p[:, k] == R) & off).astype(np.int64) << (2 * k + 1)
    e = edges[bad]
    assert np.all(planes[e[:, 0]] & planes[e[:, 1]]), "an unbalanced edge off the lattice's boundary"
    assert np.all(np.abs(fwd - rev)[bad] == 1)
    return int(bad.sum())


def components(V, faces):
    """scipy's connected components of the face-vertex graph: (count, label of every vertex)."""
    faces = np.asarray(faces, np.int64).reshape(-1, 3)
    r = np.concatenate([faces[:, 0], faces[:, 1]])
    c = np.concatenate([faces[:, 1], faces[:, 2]])
    return connected_components(coo_matrix((np.ones(len(r)), (r, c)), shape=(V, V)), directed=False)


def _per_component(values, comp, n):
    order = np.argsort(comp, kind="stable")
    cuts = np.searchsorted(comp[order], np.arange(n + 1))
    vs = values[order]
    return np.array([math.fsum(vs[cuts[k]:cuts[k + 1]]) for k in range(n)])


def geometry(verts, faces):
    """Per component (scipy labels): signed enclosed volume (fsum of a . (b x c) / 6), Euler characteristic
    V - E + F with an edge used by 2k faces counted k times (a fan diagonal in a cube face may be shared by four
    triangles, two in each direction), and face count.  Returns a list of (volume, euler, faces) by increasing volume."""
    v = np.asarray(verts, np.float64)
    faces = np.asarray(faces, np.int64).reshape(-1, 3)
    n, lab = components(len(v), faces)
    fc = lab[faces[:, 0]]
    a, b, c = v[faces[:, 0]], v[faces[:, 1]], v[faces[:, 2]]
    vol = _per_component(np.einsum("ij,ij->i", a, np.cross(b, c)) / 6.0, fc, n)
    edges, use, _, _ = edge_use(faces, len(v))
    assert np.all(use % 2 == 0)
    ne = np.bincount(lab[edges[:, 0]], weights=use // 2, minlength=n)
    nv = np.bincount(lab[np.unique(faces)], minlength=n)
    nf = np.bincount(fc, minlength=n)
    out = [(float(vol[k]), int(nv[k] - ne[k] + nf[k]), int(nf[k])) for k in range(n) if nf[k]]
    return sorted(out)


def face_areas(verts, faces):
    v = np.asarray(verts, np.float64)
    faces = np.asarray(faces, np.int64).reshape(-1, 3)
    a, b, c = v[faces[:, 0]], v[faces[:, 1]], v[faces[:, 2]]
    return 0.5 * np.linalg.norm(np.cross(b - a, c - a), axis=1)


NEAR_TIE = 2.0 ** -40


def largest_component(verts, faces):
    """The components (scipy labels) of largest fsum area: every one within NEAR_TIE relative of the largest, in order
    of their lowest face index, and the compaction of each (its vertices and faces in original order, re-indexed).
    Returns a list of (verts, faces)."""
    verts = np.asarray(verts, np.float32).reshape(-1, 3)
    faces = np.asarray(faces, np.int64).reshape(-1, 3)
    if len(faces) == 0:
        return [(np.zeros((0, 3), np.float32), np.zeros((0, 3), np.int64))]
    n, lab = components(len(verts), faces)
    fc = lab[faces[:, 0]]
    area = _per_component(face_areas(verts, faces), fc, n)
    best = area.max()
    near = np.flatnonzero(area >= best * (1.0 - NEAR_TIE))
    first = np.array([np.flatnonzero(fc == k)[0] for k in near])
    out = []
    for k in near[np.argsort(first)]:
        vk = lab == k
        new = np.cumsum(vk) - 1
        out.append((verts[vk], new[faces[fc == k]]))
    return out
