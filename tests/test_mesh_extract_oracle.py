"""CPU: oracle/mesh_extract.py — its MISE against the reference's compiled MISE (oracle/_ref, built by
oracle/build_ref.py), its marching cubes against the properties DESIGN §3.7 promises, and the component rule."""
import itertools

import numpy as np
import pytest

from oracle import build_ref, mesh_extract as M

import _mesh_ref as X
from _setups import MESH_SHAPES, mesh_grid


@pytest.fixture(scope="module")
def ref_mise():
    mod = build_ref.load_mise()
    if mod is None:
        pytest.skip("oracle/_ref has no compiled reference MISE (python -m oracle.build_ref with the reference tree)")
    return mod


def _world(idx, R):
    return (np.asarray(idx, np.float64) / R - 0.5) * 1.1       # generate_mesh's padded box [-0.55, 0.55]^3


def sphere(R, r=0.3, c=(0.0, 0.0, 0.0)):
    return lambda idx: np.linalg.norm(_world(idx, R) - np.array(c), axis=1) - r


def two_spheres(R):
    return lambda idx: np.minimum(sphere(R, 0.2, (-0.25, 0, 0))(idx), sphere(R, 0.15, (0.28, 0.05, 0))(idx))


def slab(R, res_init):
    s = 1.1 / res_init                                        # coarse cell; x = 0 is a coarse lattice plane
    return lambda idx: np.abs(_world(idx, R)[:, 0] - (0.5 * s + 0.0017)) - 0.15 * s


def on_level(R, level):
    # values exactly equal to the level on many lattice points (a quantised plane)
    return lambda idx: np.round((np.asarray(idx)[:, 0] + np.asarray(idx)[:, 1] - R) / 4.0) + level


FIELDS = {"sphere": sphere, "two_spheres": two_spheres, "slab": None, "on_level": None}


@pytest.mark.parametrize("res_init,depth", [(4, 2), (8, 3), (32, 2)])
@pytest.mark.parametrize("field", sorted(FIELDS))
@pytest.mark.parametrize("level", [0.0, 0.05])
def test_mise_matches_compiled_reference(ref_mise, res_init, depth, field, level):
    R = res_init << depth
    fn = {"sphere": lambda: sphere(R), "two_spheres": lambda: two_spheres(R), "slab": lambda: slab(R, res_init),
          "on_level": lambda: on_level(R, level)}[field]()
    g_ref, ev_ref, rounds_ref = M.reference_mise(ref_mise, fn, res_init, depth, level)
    g, ev, rounds = M.mise(fn, res_init, depth, level)
    assert np.array_equal(g, g_ref)
    assert np.array_equal(ev, ev_ref)
    assert len(rounds) == len(rounds_ref)
    for a, b in zip(rounds, rounds_ref):          # the same points per round (the reference's order is its own)
        assert np.array_equal(a, b[np.lexsort(b.T[::-1])])


def test_mise_misses_a_thin_slab(ref_mise):
    """A slab thinner than a coarse cell between coarse lattice points is never refined: MISE's grid differs from the
    dense grid there (the reference behaves the same way)."""
    res_init, depth = 8, 3
    R = res_init << depth
    fn = slab(R, res_init)
    g, ev, _ = M.mise(fn, res_init, depth, 0.0)
    idx = np.argwhere(np.ones((R + 1,) * 3, bool))
    dense = fn(idx).reshape((R + 1,) * 3)
    assert (dense < 0).any() and not (g < 0).any()
    assert ev.sum() == (res_init + 1) ** 3


def _grid_sphere(R, r, c=(0.5, 0.5, 0.5)):
    x = np.arange(R + 1) / R
    X, Y, Z = np.meshgrid(x, x, x, indexing="ij")
    return (np.sqrt((X - c[0]) ** 2 + (Y - c[1]) ** 2 + (Z - c[2]) ** 2) - r).astype(np.float32)


def _grid_torus(R, a=0.3, b=0.12):
    x = np.arange(R + 1) / R - 0.5
    X, Y, Z = np.meshgrid(x, x, x, indexing="ij")
    return (np.sqrt((np.sqrt(X ** 2 + Y ** 2) - a) ** 2 + Z ** 2) - b).astype(np.float32)


def _check_closed(v, f):
    und, dire = M.edge_use(f)
    assert set(und.values()) == {2}
    assert set(dire.values()) == {1}


def _check_on_edges(g, level, v, f):
    """Every vertex lies on a lattice edge whose ends are on opposite sides of the level."""
    R = g.shape[0] - 1
    for p in v:
        lo = np.floor(p).astype(int)
        frac = p - lo
        axes = np.nonzero(frac)[0]
        assert len(axes) <= 1
        if len(axes) == 1:
            a = axes[0]
            hi = lo.copy()
            hi[a] += 1
            assert (g[tuple(lo)] < level) != (g[tuple(hi)] < level)
        else:        # t = 0: the vertex is the lower corner itself, which is not below
            assert lo.max() <= R


@pytest.mark.parametrize("R", [16, 40])
def test_marching_cubes_sphere(R):
    r = 0.3
    g = _grid_sphere(R, r)
    v, f = M.marching_cubes(g, 0.0)
    _check_closed(v, f)
    _check_on_edges(g, 0.0, v, f)
    assert M.euler(v, f) == 2
    vol = M.volume(v, f) / R ** 3
    exact = 4.0 / 3.0 * np.pi * r ** 3
    assert vol > 0 and abs(vol - exact) < 2.0 / R ** 2


def test_marching_cubes_torus():
    R = 48
    g = _grid_torus(R)
    v, f = M.marching_cubes(g, 0.0)
    _check_closed(v, f)
    assert M.euler(v, f) == 0
    vol = M.volume(v, f) / R ** 3
    exact = 2 * np.pi ** 2 * 0.3 * 0.12 ** 2
    assert vol > 0 and abs(vol - exact) < 3.0 / R ** 2


@pytest.mark.parametrize("seed,quant", [(0, False), (1, False), (2, True), (3, True)])
def test_marching_cubes_random_grids(seed, quant):
    rng = np.random.default_rng(seed)
    g = rng.standard_normal((11, 11, 11)).astype(np.float32)
    if quant:
        g = np.round(g).astype(np.float32)        # values on the level, decider ties
    g[0], g[-1], g[:, 0], g[:, -1], g[:, :, 0], g[:, :, -1] = 1, 1, 1, 1, 1, 1
    v, f = M.marching_cubes(g, 0.0)
    # closed and consistently oriented: every undirected edge is used by an even number of faces, half in each
    # direction.  A few edges are used by 4: a fan diagonal that lies in a cube face on both sides of it (DESIGN §3.7).
    und, dire = M.edge_use(f)
    assert set(und.values()) <= {2, 4}
    assert all(dire.get((a, b), 0) == dire.get((b, a), 0) == n // 2 for (a, b), n in und.items())
    assert sum(n == 4 for n in und.values()) < 0.01 * len(und)
    _check_on_edges(g, 0.0, v, f)
    assert M.volume(v, f) > 0


def test_marching_cubes_all_corner_patterns_with_ties():
    """Every one of the 256 corner patterns of a cube padded by an outside layer, with the ambiguous faces' decider at
    a tie (|values| all 1): closed, consistently oriented, on sign-change edges, positive volume."""
    for case in range(256):
        g = np.ones((4, 4, 4), np.float32)
        for c, (dx, dy, dz) in enumerate(M.CORNERS):
            if (case >> c) & 1:
                g[1 + dx, 1 + dy, 1 + dz] = -1.0
        v, f = M.marching_cubes(g, 0.0)
        if case == 0:
            assert len(f) == 0
            continue
        _check_closed(v, f)
        _check_on_edges(g, 0.0, v, f)
        assert M.volume(v, f) > 0


def test_cube_faces_are_counter_clockwise_from_outside():
    for q in M.FACES:
        p = [np.array(M.CORNERS[c], float) for c in q]
        ctr = np.mean(p, axis=0)
        n = np.cross(p[1] - p[0], p[2] - p[1])
        assert np.dot(n, ctr - 0.5) > 0


def test_largest_component_rule():
    R = 32
    g = np.minimum(_grid_sphere(R, 0.12, (0.25, 0.5, 0.5)), _grid_sphere(R, 0.18, (0.7, 0.5, 0.5)))
    v, f = M.marching_cubes(g, 0.0)
    assert len(np.unique(M.components(len(v), f))) == 2
    vk, fk = M.largest_component(v, f)
    assert vk[:, 0].min() > 0.4 * R
    _check_closed(vk, fk)
    assert fk.max() == len(vk) - 1
    # equal areas: the component holding face 0
    verts = np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0], [5, 0, 0], [6, 0, 0], [5, 1, 0]], np.float32)
    vk, fk = M.largest_component(verts, np.array([[3, 4, 5], [0, 1, 2]]))
    assert np.array_equal(vk, verts[3:]) and fk.tolist() == [[0, 1, 2]]
    vk, fk = M.largest_component(verts, np.array([[0, 1, 2], [3, 4, 5]]))
    assert np.array_equal(vk, verts[:3])
    # no sign change: empty
    v, f = M.marching_cubes(np.ones((5, 5, 5), np.float32), 0.0)
    vk, fk = M.largest_component(v, f)
    assert vk.shape == (0, 3) and fk.shape == (0, 3)


def test_edges_table():
    ids = [3 * ((dx * 2 + dy) * 2 + dz) + a for (c, a) in M.EDGES for dx, dy, dz in [M.CORNERS[c]]]
    assert ids == sorted(ids) and len(M.EDGES) == 12
    assert all(sum(1 for q in M.FACES for j in range(4) if M._edge(q[j], q[(j + 1) % 4]) == e) == 2
               for e in range(12))
    assert list(itertools.chain(*M.FACES)).count(0) == 3


@pytest.mark.parametrize("name", sorted(MESH_SHAPES) + ["quantised", "random"])
def test_invariant_references_agree_with_the_oracle(name):
    """tests/_mesh_ref.py's vertex rule equals the oracle's vertices in both calling forms, and its locality, count and
    balance checks accept the oracle's faces, on small closed and open grids at every level the GPU tests use."""
    world = ((0.1, -0.2, 0.3), 1.7, 1.1)
    for R in (1, 2, 3, 9, 14):
        for level in (0.0, 0.125, -0.0625, -0.0):
            for variant in ("closed", "open"):
                g = mesh_grid(name, R, level, variant)
                v, f = M.marching_cubes(g, level)
                vr, eid = X.vertex_rule(g, level)
                assert np.array_equal(v, vr)
                assert np.array_equal(M.marching_cubes(g, level, *world)[0], X.vertex_rule(g, level, *world)[0])
                X.face_cubes(g, level, f, eid)
                assert (X.balance(g, f, eid, variant == "closed") > 0) == (variant == "open" and len(f) > 0)


def test_invariant_references_reject_broken_meshes():
    """The checks fail on what they exist to catch (one face reversed, a vertex id moved to the next crossed edge,
    faces out of cube order), and the largest-component reference picks the oracle's component."""
    g = mesh_grid("quantised", 9, 0.0)
    v, f = M.marching_cubes(g, 0.0)
    _, eid = X.vertex_rule(g, 0.0)
    X.face_cubes(g, 0.0, f, eid)
    X.balance(g, f, eid, True)
    bad = f.copy()
    bad[len(f) // 2] = bad[len(f) // 2, ::-1]
    with pytest.raises(AssertionError):
        X.balance(g, bad, eid, True)
    moved = f.copy()
    moved[0, 0] = (moved[0, 0] + 1) % len(eid)
    with pytest.raises(AssertionError):
        X.face_cubes(g, 0.0, moved, eid)
        X.balance(g, moved, eid, True)
    with pytest.raises(AssertionError):
        X.face_cubes(g, 0.0, f[::-1], eid)
    vk, fk = X.largest_component(v, f)[0]
    vc, fc = M.largest_component(v, f)
    assert np.array_equal(vk, vc) and np.array_equal(fk, fc)
