"""CPU restatement of generate_mesh's extraction steps (lib/utils/mesh.py:78-132) as the device implements them
(csrc/mesh_extract.cu, DESIGN §3.7): MISE (lib/libmise/mise.pyx), the marching-cubes definition, the component rule.
numpy, fp64 where the kernels are fp64, written for clarity rather than speed.

Also ``reference_mise``: the reference's own MISE module (compiled by oracle/build_ref.py) driven the way
generate_mesh drives it (:87-109)."""
import itertools

import numpy as np


# ---- MISE ------------------------------------------------------------------------------------------------------------

def mise(values_at, res_init, depth, level):
    """values_at(idx [N,3] int64 lattice coordinates, lattice order) -> values [N].  Returns (grid [(R+1)^3] float64 =
    to_dense(), evaluated [(R+1)^3] bool, list of the index arrays evaluated per round)."""
    R = res_init << depth
    n1 = R + 1
    added = np.zeros((n1,) * 3, bool)
    known = np.zeros((n1,) * 3, bool)
    val = np.zeros((n1,) * 3, np.float64)
    s0 = 1 << depth
    added[::s0, ::s0, ::s0] = True
    # leaf level of each voxel of level depth-1 (depth once it is split into finest leaves)
    Rh = R >> 1
    leaf = np.zeros((Rh,) * 3, np.int64) if depth > 0 else None
    rounds = []
    while True:
        pend = added & ~known
        idx = np.argwhere(pend)
        if len(idx) == 0:
            break
        rounds.append(idx)
        val[pend] = np.asarray(values_at(idx), np.float64)
        known |= pend
        if depth == 0:
            continue
        pos = np.zeros(leaf.shape, bool)
        neg = np.zeros(leaf.shape, bool)
        kidx = np.argwhere(known)
        kv = val[known]
        for d in itertools.product((-1, 0), repeat=3):
            c = kidx + np.array(d)
            ok = np.all((c >= 0) & (c < R), axis=1)
            v = c[ok] >> 1
            L = leaf[v[:, 0], v[:, 1], v[:, 2]]
            m = L < depth
            v, L, vv = v[m], L[m], kv[ok][m]
            sh = (depth - 1 - L)[:, None]
            a = (v >> sh) << sh
            p, q = vv >= level, vv <= level
            pos[a[p, 0], a[p, 1], a[p, 2]] = True
            neg[a[q, 0], a[q, 1], a[q, 2]] = True
        vox = np.argwhere(leaf < depth)
        L = leaf[vox[:, 0], vox[:, 1], vox[:, 2]]
        sh = (depth - 1 - L)[:, None]
        a = (vox >> sh) << sh
        split = pos[a[:, 0], a[:, 1], a[:, 2]] & neg[a[:, 0], a[:, 1], a[:, 2]]
        anchors = np.all(vox == a, axis=1) & split
        for (x, y, z), l in zip(vox[anchors], L[anchors]):
            cs = 1 << (depth - l - 1)
            added[2 * x:2 * x + 2 * cs + 1:cs, 2 * y:2 * y + 2 * cs + 1:cs, 2 * z:2 * z + 2 * cs + 1:cs] = True
        sv = vox[split]
        leaf[sv[:, 0], sv[:, 1], sv[:, 2]] += 1
    return _to_dense(np.where(known, val, np.nan)), known, rounds


def _to_dense(g):
    g = g.copy()
    for axis in range(3):
        h = np.moveaxis(g, axis, 0)
        for i in range(1, h.shape[0]):
            h[i] = np.where(np.isnan(h[i]), h[i - 1], h[i])
    return g


def reference_mise(mise_module, values_at, res_init, depth, level):
    """The reference's MISE (compiled mise.pyx) in generate_mesh's loop (:87-109).  Returns (to_dense() grid,
    evaluated mask, list of the query() arrays)."""
    m = mise_module.MISE(res_init, depth, level)
    R = m.resolution
    ev = np.zeros((R + 1,) * 3, bool)
    rounds = []
    pts = m.query()
    while pts.shape[0] != 0:
        rounds.append(pts)
        ev[pts[:, 0], pts[:, 1], pts[:, 2]] = True
        m.update(pts, np.asarray(values_at(pts), np.float64))
        pts = m.query()
    return m.to_dense(), ev, rounds


# ---- marching cubes ----------------------------------------------------------------------------------------------------

CORNERS = [(dx, dy, dz) for dx in (0, 1) for dy in (0, 1) for dz in (0, 1)]      # corner c = 4 dx + 2 dy + dz
# cube edges (lower corner, axis) sorted by lattice-edge id 3 * lattice index + axis
EDGES = sorted([(c, a) for c, (dx, dy, dz) in enumerate(CORNERS) for a in range(3) if (dx, dy, dz)[a] == 0],
               key=lambda e: (CORNERS[e[0]], e[1]))
EDGE_ID = {e: i for i, e in enumerate(EDGES)}


def _edge(c0, c1):
    lo, hi = min(c0, c1), max(c0, c1)
    a = [i for i in range(3) if CORNERS[lo][i] != CORNERS[hi][i]]
    return EDGE_ID[(lo, a[0])]


def _faces():
    """Each cube face: its corners counter-clockwise seen from outside (right-hand rule about the outward normal)."""
    out = []
    for axis in range(3):
        for side in (0, 1):
            cs = [c for c in range(8) if CORNERS[c][axis] == side]
            n = np.zeros(3)
            n[axis] = 1 if side else -1
            ctr = np.mean([CORNERS[c] for c in cs], axis=0)
            u = np.array(CORNERS[cs[0]]) - ctr
            w = np.cross(n, u)
            ang = [np.arctan2(np.dot(np.array(CORNERS[c]) - ctr, w), np.dot(np.array(CORNERS[c]) - ctr, u)) for c in cs]
            out.append([cs[i] for i in np.argsort(ang)])
    return out


FACES = _faces()


def cube_triangles(below, fv):
    """below: 8 bools, fv: 8 fp64 values - level.  Triangles as local edge triples, DESIGN §3.7."""
    nxt = {}
    for q in FACES:
        e = [_edge(q[j], q[(j + 1) % 4]) for j in range(4)]
        starts = [j for j in range(4) if not below[q[j]] and below[q[(j + 1) % 4]]]
        ends = [j for j in range(4) if below[q[j]] and not below[q[(j + 1) % 4]]]
        if len(starts) == 1:
            nxt[e[starts[0]]] = e[ends[0]]
        elif len(starts) == 2:
            p02, p13 = fv[q[0]] * fv[q[2]], fv[q[1]] * fv[q[3]]
            sep_below = (p13 >= p02) if below[q[0]] else (p02 >= p13)
            for j in starts:
                nxt[e[j]] = e[(j + 1) % 4] if sep_below else e[(j + 3) % 4]
    tris, seen = [], set()
    for e0 in sorted(nxt):
        if e0 in seen:
            continue
        poly = [e0]
        while nxt[poly[-1]] != e0:
            poly.append(nxt[poly[-1]])
        seen.update(poly)
        for i in range(1, len(poly) - 1):
            tris.append((e0, poly[i], poly[i + 1]))
    return tris


_CACHE = {}


def marching_cubes(grid, level=0.0, center=None, extent=None, pad=1.1):
    """grid [(R+1)^3] (x-major) -> (verts [V,3] fp32, faces [F,3] int64) by the definition of DESIGN §3.7.
    extent=None: lattice coordinates (centre R/2, extent R, pad 1)."""
    g = np.asarray(grid, np.float32)
    R = g.shape[0] - 1
    n1 = R + 1
    if extent is None:
        center, extent, pad = (R / 2.0,) * 3, float(R), 1.0
    level = float(level)
    below = g.astype(np.float64) < level
    # vertices: crossing lattice edges in id order 3 * index + axis
    eid, pos = [], []
    for a in range(3):
        sl0 = [slice(None)] * 3
        sl1 = [slice(None)] * 3
        sl0[a], sl1[a] = slice(0, R), slice(1, n1)
        cr = below[tuple(sl0)] != below[tuple(sl1)]
        p = np.argwhere(cr)
        v0 = g[tuple(sl0)][cr].astype(np.float64)
        v1 = g[tuple(sl1)][cr].astype(np.float64)
        t = (level - v0) / (v1 - v0)
        c = p.astype(np.float64)
        c[:, a] = c[:, a] + t
        eid.append((p[:, 0] * n1 + p[:, 1]) * n1 + p[:, 2])
        pos.append(c)
        eid[-1] = eid[-1] * 3 + a
    eid = np.concatenate(eid)
    c = np.concatenate(pos)
    o = np.argsort(eid, kind="stable")
    eid, c = eid[o], c[o]
    ctr = np.asarray(center, np.float64)
    verts = (((c / float(R) - 0.5) * float(pad)) * float(extent) + ctr[None]).astype(np.float32)
    # faces: every cube with a crossing, in cube order
    fvals = g.astype(np.float64) - level
    mask = np.zeros((R, R, R), np.int64)
    for ci, (dx, dy, dz) in enumerate(CORNERS):
        mask |= below[dx:dx + R, dy:dy + R, dz:dz + R].astype(np.int64) << ci
    cubes = np.argwhere((mask != 0) & (mask != 255))
    faces = []
    for x, y, z in cubes:
        fv = [fvals[x + dx, y + dy, z + dz] for dx, dy, dz in CORNERS]
        b = [bool(below[x + dx, y + dy, z + dz]) for dx, dy, dz in CORNERS]
        for tri in cube_triangles(b, fv):
            ids = []
            for e in tri:
                ci, a = EDGES[e]
                dx, dy, dz = CORNERS[ci]
                ids.append((((x + dx) * n1 + (y + dy)) * n1 + (z + dz)) * 3 + a)
            faces.append(ids)
    faces = np.asarray(faces, np.int64).reshape(-1, 3)
    faces = np.searchsorted(eid, faces).astype(np.int64) if len(faces) else faces
    return verts, faces


# ---- largest component -------------------------------------------------------------------------------------------------

AREA_CHUNK = 256


def face_areas(verts, faces):
    v = np.asarray(verts, np.float32).astype(np.float64)
    a, b, c = v[faces[:, 0]], v[faces[:, 1]], v[faces[:, 2]]
    e1, e2 = b - a, c - a
    cx = e1[:, 1] * e2[:, 2] - e1[:, 2] * e2[:, 1]
    cy = e1[:, 2] * e2[:, 0] - e1[:, 0] * e2[:, 2]
    cz = e1[:, 0] * e2[:, 1] - e1[:, 1] * e2[:, 0]
    return 0.5 * np.sqrt(cx * cx + cy * cy + cz * cz)


def components(V, faces):
    """Component label of every vertex (its lowest vertex index) through faces sharing vertices."""
    parent = np.arange(V)

    def find(x):
        while parent[x] != x:
            parent[x] = parent[parent[x]]
            x = parent[x]
        return x

    for f in faces:
        for k in (1, 2):
            a, b = find(f[0]), find(f[k])
            if a != b:
                parent[max(a, b)] = min(a, b)
    return np.array([find(v) for v in range(V)], np.int64)


def largest_component(verts, faces):
    """Keep the component of largest area (fp64, summed in the order of DESIGN §3.7); equal areas: the one holding the
    lowest face index.  Returns (verts, faces) compacted in order and re-indexed; empty input -> empty output."""
    verts = np.asarray(verts, np.float32).reshape(-1, 3)
    faces = np.asarray(faces, np.int64).reshape(-1, 3)
    if len(verts) == 0 or len(faces) == 0:
        return np.zeros((0, 3), np.float32), np.zeros((0, 3), np.int64)
    lab = components(len(verts), faces)
    key = lab[faces[:, 0]]
    order = np.argsort(key, kind="stable")
    ks = key[order]
    ar = face_areas(verts, faces)[order]
    F = len(faces)
    best = None
    i = 0
    while i < F:
        j = i
        while j < F and ks[j] == ks[i]:
            j += 1
        total, k = 0.0, i
        while k < j:                      # chunks: cut at every multiple of AREA_CHUNK
            e = min(j, (k // AREA_CHUNK + 1) * AREA_CHUNK)
            s = 0.0
            for m in range(k, e):
                s += ar[m]
            total += s
            k = e
        cand = (total, -int(order[i]), int(ks[i]))
        if best is None or cand[:2] > best[:2]:
            best = cand
        i = j
    w = best[2]
    vkeep = lab == w
    fkeep = key == w
    new = np.cumsum(vkeep) - 1
    return verts[vkeep], new[faces[fkeep]].astype(np.int64)


# ---- checks ------------------------------------------------------------------------------------------------------------

def edge_use(faces):
    """(undirected edge -> number of faces using it, directed edge -> number of faces using it)"""
    und, dire = {}, {}
    for f in faces:
        for k in range(3):
            a, b = int(f[k]), int(f[(k + 1) % 3])
            dire[(a, b)] = dire.get((a, b), 0) + 1
            u = (min(a, b), max(a, b))
            und[u] = und.get(u, 0) + 1
    return und, dire


def euler(verts, faces):
    und, _ = edge_use(faces)
    return len(np.unique(faces)) - len(und) + len(faces)


def volume(verts, faces):
    """Signed enclosed volume (positive when the normals point outward)."""
    v = np.asarray(verts, np.float64)
    a, b, c = v[faces[:, 0]], v[faces[:, 1]], v[faces[:, 2]]
    return float(np.sum(np.einsum("ij,ij->i", a, np.cross(b, c)))) / 6.0
