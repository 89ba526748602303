"""GPU: every library call's outputs are independent of what its workspace, its output buffers and the storage of its
persistent objects held before the call.

Production code reuses device memory: the caching allocator hands a workspace, an output or a handle's storage the bytes
of whatever used them last, and the epoch-end mesh extraction runs every person's extraction back to back.  So each
entry point runs input B twice, once on zero-filled buffers and once on the very buffers a call on input A (same sizes,
different data) has just used, and the outputs must be bit-identical; A is checked the same way with the roles swapped.
Stale contents are thus values a legitimate call wrote, in range for the shapes, never synthetic poison.

Also here: the largest component on a mesh whose union-find trees are deep (the labelling race that dropped a vertex
from the kept component), the epoch-end sequence of generate_mesh calls, and calls on a non-default caller stream whose
outputs are read on that stream without a host synchronisation."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from multiply_b200 import engine, scene as S, _lib as L     # noqa: E402
from multiply_b200.utils import mesh as umesh               # noqa: E402
from oracle import mesh_extract as M                        # noqa: E402

import _calls as calls                                                              # noqa: E402
from _abi import same, snap                                                         # noqa: E402
from _setups import Smpl, geo, mirror_inputs, points, posed_body, pts, train, trained  # noqa: E402,F401


# ---------------------------------------------------------------------------------------------
# fresh versus reused buffers
# ---------------------------------------------------------------------------------------------

def _zeroed(case):
    """Zero-filled output buffers and workspace of a call."""
    o = {k: torch.zeros(shape, dtype=dtype, device="cuda") for k, (shape, dtype) in case.outs.items()}
    return o, torch.zeros(max(int(case.query()), 1), dtype=torch.uint8, device="cuda")


def check_reuse(case, a, b):
    """B on zeroed buffers, then A on other zeroed buffers, then B on A's buffers and A on B's (outputs and workspace):
    both reused runs must equal the fresh ones bit for bit, and A and B must differ (else the reuse proves nothing).
    Returns (A, B) fresh outputs."""
    s1, s2 = _zeroed(case), _zeroed(case)
    b_fresh = snap(case.call(b, *s1))
    a_fresh = snap(case.call(a, *s2))
    b_reused = snap(case.call(b, *s2))
    a_reused = snap(case.call(a, *s1))
    for tag, want, got in (("B", b_fresh, b_reused), ("A", a_fresh, a_reused)):
        for k in want:
            assert same(want[k], got[k]), "%s: output %s differs when its buffers held another call's bytes" % (tag, k)
    assert any(not same(a_fresh[k], b_fresh[k]) for k in a_fresh), "A and B give identical outputs"
    return a_fresh, b_fresh


# ---------------------------------------------------------------------------------------------
# scenes
# ---------------------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def mise_grids(trained):
    """Both persons' MISE grids at res_init 32, depth 2 (R = 128)."""
    sc, fields, _ = trained
    out = []
    for pid in range(2):
        f, center, extent, pad = calls.person_box(sc, fields, pid)
        out.append(f.mise(center, extent, 32, 2, 0.0, pad)[0])
    torch.cuda.synchronize()
    return out


# ---------------------------------------------------------------------------------------------
# mesh extraction
# ---------------------------------------------------------------------------------------------

@pytest.mark.parametrize("res_init,depth", [(32, 2), (32, 3), (64, 4)])
def test_mise_reuse(trained, res_init, depth):
    """MISE of person 0 (A) and person 1 (B).  At 32/3 the two persons evaluate under 2^20 points in all (0.75 M and
    0.98 M), so every round fits one 2^20-point slab; 64/4 (R = 1024) is there for the slab loop: each
    person evaluates more than 5 * 2^20 points over its rounds, most of them in the last."""
    sc, fields, _ = trained
    c = calls.mise(sc, fields, res_init, depth)
    a, b = check_reuse(c, c.inputs(0), c.inputs(1))
    print("MISE %d/%d: %d and %d points evaluated" % (res_init, depth, a["n"], b["n"]))
    if depth == 4:
        assert min(a["n"], b["n"]) > (depth + 1) << 20


def test_marching_cubes_reuse(mise_grids):
    """Count and emit on one workspace (emit reads the count's offsets), persons 0 and 1's MISE grids; outputs sized for
    the larger mesh, each compared over the rows its call writes.  The fresh meshes equal the oracle's."""
    R = mise_grids[0].shape[0] - 1
    sizes = [engine.marching_cubes(g, 0.0) for g in mise_grids]
    Vm, Fm = max(v.shape[0] for v, _ in sizes), max(f.shape[0] for _, f in sizes)
    outs = check_reuse(calls.marching_cubes(R, Vm, Fm), mise_grids[0], mise_grids[1])
    for g, o in zip(mise_grids, outs):
        vr, fr = M.marching_cubes(g.cpu().numpy(), 0.0)
        assert np.array_equal(o["v"].cpu().numpy().reshape(-1, 3), vr)
        assert np.array_equal(o["f"].cpu().numpy().reshape(-1, 3), fr)


def test_largest_component_reuse(mise_grids):
    """A: marching cubes of person 0's grid; B: the same V and F with the faces relabelled by a vertex permutation, so
    every component, root and sort key differs.  Both fresh results equal the oracle's."""
    v, f = engine.marching_cubes(mise_grids[0], 0.0)
    V, F = v.shape[0], f.shape[0]
    perm = torch.randperm(V, generator=torch.Generator().manual_seed(3)).cuda()
    fb = perm[f].contiguous()
    outs = check_reuse(calls.largest_component(V, F), (v, f), (v, fb))
    for (vi, fi), o in zip(((v, f), (v, fb)), outs):
        vc, fc = M.largest_component(vi.cpu().numpy(), fi.cpu().numpy())
        assert o["V"] == len(vc) and o["F"] == len(fc)
        assert np.array_equal(o["v"].cpu().numpy().reshape(-1, 3), vc)
        assert np.array_equal(o["f"].cpu().numpy().reshape(-1, 3), fc)


def test_largest_component_deep_union_find():
    """Two interleaved triangle strips, faces (k, k+2, k+4) in order: the concurrent unions link long chains, so the
    labelling pass runs while many threads compress the same paths.  A compression that lands on a vertex after its
    own thread labelled it must not change its label: the kept component is the whole longer strip (even vertices),
    every vertex and face of it, in order."""
    n = 1 << 20                                     # vertices of the long strip (even ids); the short one has n / 4
    h = 2.0 ** -10
    j = torch.arange(n, dtype=torch.float64)
    pos = torch.stack([torch.div(j, 2, rounding_mode="floor") * h, (j % 2) * h, torch.zeros(n, dtype=torch.float64)], 1)
    verts = torch.empty(2 * n, 3, dtype=torch.float64)
    verts[0::2] = pos
    verts[1::2] = pos + torch.tensor([0.0, 0.0, 1.0], dtype=torch.float64)
    verts = verts.float()
    k = torch.arange(n - 2, dtype=torch.int64)
    long_strip = torch.stack([2 * k, 2 * k + 2, 2 * k + 4], 1)
    ks = torch.arange(n // 4 - 2, dtype=torch.int64)
    short_strip = torch.stack([2 * ks + 1, 2 * ks + 3, 2 * ks + 5], 1)
    faces = torch.cat([long_strip, short_strip])
    vd, fd = verts.cuda(), faces.cuda()
    lc = calls.largest_component(2 * n, faces.shape[0])
    o = lc.call((vd, fd), *_zeroed(lc))
    torch.cuda.synchronize()
    assert (o["V"], o["F"]) == (n, n - 2), "kept %d vertices and %d faces of the %d / %d of the long strip" % (
        o["V"], o["F"], n, n - 2)
    assert torch.equal(o["v"].cpu().reshape(-1, 3), verts[0::2])
    assert torch.equal(o["f"].cpu().reshape(-1, 3), torch.stack([k, k + 1, k + 2], 1))


def test_sdf_grid_reuse(trained):
    sc, fields, _ = trained
    c = calls.sdf_grid(sc, fields, 64)
    check_reuse(c, c.inputs(0), c.inputs(1))


# ---------------------------------------------------------------------------------------------
# networks, background, sampler
# ---------------------------------------------------------------------------------------------

@pytest.mark.parametrize("N", [1, 127, 129])
@pytest.mark.parametrize("grad", [False, True])
def test_implicit_forward_reuse(trained, N, grad):
    c = calls.implicit_forward(trained[1][0], N, grad)
    check_reuse(c, c.inputs(10 + N), c.inputs(20 + N))


@pytest.mark.parametrize("N", [1, 127, 129])
def test_bg_nets_forward_reuse(trained, N):
    c = calls.bg_nets_forward(trained[2], N)
    check_reuse(c, c.inputs(30 + N), c.inputs(40 + N))


@pytest.mark.parametrize("N", [1, 129, 32769])
@pytest.mark.parametrize("net", ["implicit", "bg_implicit", "render"])
def test_network_backward_reuse(trained, net, N):
    """N = 32769: two chunks, the second run in the workspace the first left."""
    f = trained[2] if net == "bg_implicit" else trained[1][0]
    c = calls.render_backward(f, N) if net == "render" else calls.implicit_backward(f, N)
    check_reuse(c, c.inputs(50 + N), c.inputs(60 + N))


def test_background_reuse(trained):
    """Rays from cameras inside the r = 3 sphere, R = 301 (not a multiple of the 8 rays per block)."""
    c = calls.background(trained[2], 301)
    check_reuse(c, c.inputs(50), c.inputs(60))


@pytest.mark.parametrize("train", [False, True])
def test_sample_rays_reuse(geo, train):
    """The eval and the training sampler on person 0's rays (A: one ray set and draws, B: another)."""
    sc, f, body = geo
    c = calls.sample_rays(sc, f, body, 300, train)
    check_reuse(c, c.inputs(5), c.inputs(6))


# ---------------------------------------------------------------------------------------------
# compositor and its backward
# ---------------------------------------------------------------------------------------------

def test_composite_reuse():
    c = calls.composite()
    check_reuse(c, c.inputs(11), c.inputs(12))


def test_composite_backward_reuse():
    """Gradient buffers hold R rows per person (hit lists differ between A and B); each is compared over its rows."""
    c = calls.composite_backward()
    check_reuse(c, c.inputs(11), c.inputs(12))


# ---------------------------------------------------------------------------------------------
# SMPL server and deformer backward
# ---------------------------------------------------------------------------------------------

def test_smpl_backward_reuse():
    c = calls.smpl_backward(Smpl(S.make_smpl_model(300)))
    check_reuse(c, c.inputs(1), c.inputs(2))


@pytest.mark.parametrize("N", [1, 4097])
def test_deform_backward_reuse(N):
    body, _ = posed_body()
    c = calls.deform_inverse_backward(body, N)
    check_reuse(c, c.inputs(71), c.inputs(72))
    c = calls.deform_forward_jac_backward(body, N)
    check_reuse(c, c.inputs(73), c.inputs(74))


# ---------------------------------------------------------------------------------------------
# persistent stores: a handle built in storage that held another handle's bytes
# ---------------------------------------------------------------------------------------------

def _built_in(monkeypatch, src, build):
    """build() with every ``_lib.workspace`` it asks for holding the leading bytes of ``src`` (zeros past them; src
    None: all zeros)."""
    def ws(nbytes, device):
        b = torch.zeros(max(int(nbytes), 1), dtype=torch.uint8, device=device)
        if src is not None:
            n = min(b.numel(), src.numel())
            b[:n] = src[:n]
        return b
    with monkeypatch.context() as m:
        m.setattr(L, "workspace", ws)
        obj = build()
    torch.cuda.synchronize()
    return obj


def _stores_agree(monkeypatch, old_storage, build, first_call):
    fresh = _built_in(monkeypatch, None, build)
    stale = _built_in(monkeypatch, old_storage, build)
    want, got = snap(first_call(fresh)), snap(first_call(stale))
    for k in want:
        assert same(want[k], got[k]), "%s differs when the handle was built in another handle's storage" % k


def test_field_store_reuse(monkeypatch, trained):
    sc, fields, bg = trained
    p1 = sc["persons"][1]
    x = pts(129, 3, 80)
    nrm = pts(129, 3, 81)

    def first(f):
        f.set_cond(p1["cond"])
        sdf, feat, grad = f.implicit_forward(x, want_grad=True)
        return dict(sdf=sdf, feat=feat, grad=grad, rgb=f.render_forward(x, nrm, feat))

    _stores_agree(monkeypatch, fields[0].storage, lambda: engine.Field(p1["implicit"], p1["render"]), first)

    def first_bg(f):
        f.set_cond(sc["frame_code"])
        sdf, rgb = f.bg_forward(pts(129, 4, 82), nrm / nrm.norm(dim=1, keepdim=True))
        return dict(sdf=sdf, rgb=rgb)

    _stores_agree(monkeypatch, fields[0].storage,
                  lambda: engine.Field(sc["bg_implicit"], sc["bg_render"], background=True), first_bg)


def test_body_store_reuse(monkeypatch, trained):
    sc, _, _ = trained
    p0, p1 = sc["persons"]
    old = engine.Body(p0["verts_c"], p0["weights"], cano_cell=0.1001 / p0["scale"])
    old.set_pose(p0["verts_p"], p0["tfs"])
    torch.cuda.synchronize()
    x = points(4097, p1["verts_p"], 90).cuda()

    def first(b):
        b.set_pose(p1["verts_p"], p1["tfs"])
        xc, out = b.deform_inverse(x)
        xd, J = b.forward_jac(xc)
        return dict(xc=xc, out=out, xd=xd, J=J)

    _stores_agree(monkeypatch, old.storage,
                  lambda: engine.Body(p1["verts_c"], p1["weights"], cano_cell=0.1001 / p1["scale"]), first)


def test_smpl_store_reuse(monkeypatch):
    old = Smpl(S.make_smpl_model(300))
    model = S.make_smpl_model(301)
    rng = np.random.RandomState(4)
    args = (1.1, rng.normal(0, 0.3, 3), rng.normal(0, 0.4, 72), rng.normal(0, 1, 10))

    def first(s):
        v, t = s.forward(*args, absolute=False)
        return dict(cinv=torch.from_numpy(s.cinv), v=v, t=t)

    _stores_agree(monkeypatch, old.storage, lambda: Smpl(model), first)


def test_mesh_store_reuse(monkeypatch):
    old = engine.CanonicalMesh(*S.make_body_mesh(100))
    v, f = S.make_body_mesh(101)
    g = torch.Generator().manual_seed(5)
    vt = torch.as_tensor(v).float()
    pts = (vt[torch.randint(vt.shape[0], (6000,), generator=g)] + 0.05 * torch.randn(6000, 3, generator=g)).cuda()

    def first(m):
        d2, fi, dt = m.distance(pts)
        off, ins = m.surface_flags(pts, 8)
        return dict(d2=d2, fi=fi, dt=dt, sign=m.check_sign(pts), off=off, ins=ins)

    _stores_agree(monkeypatch, old.storage, lambda: engine.CanonicalMesh(v, f), first)


# ---------------------------------------------------------------------------------------------
# the epoch-end sequence, and calls on a caller's own stream
# ---------------------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def mirror():
    engine.set_engine("tc")
    sc = S.make_scene(P=2, S=16, seed=42, weights="trained")
    return sc, S.mirror_model(sc)


def _cond(sc, pid):
    return {"smpl": sc["persons"][pid]["cond"].cuda()}


def test_epoch_end_mesh_sequence(mirror):
    """generate_mesh for person 0, person 1, person 0 with no cleanup in between: person 0's two meshes are
    bit-identical and every mesh equals the oracle's marching cubes and largest component on the same MISE grid.  Then
    both meshes go to set_canonical_mesh and a training step's surface flags equal those of a model that only ever saw
    the final meshes."""
    sc, m = mirror
    meshes = []
    for pid in (0, 1, 0):
        meshes.append(umesh.generate_mesh(m, pid, _cond(sc, pid), sc["persons"][pid]["verts_c"], res_init=32, res_up=2))
    assert torch.equal(meshes[0][0], meshes[2][0]) and torch.equal(meshes[0][1], meshes[2][1])
    fields = m._ensure_renderer(torch.device("cuda", torch.cuda.current_device())).fields
    for pid, (v, f) in zip((0, 1), meshes[1:][::-1]):
        center, extent, pad = umesh.bounds(sc["persons"][pid]["verts_c"])
        fields[pid].set_cond(_cond(sc, pid)["smpl"])
        grid, _ = fields[pid].mise(center, extent, 32, 2, 0.0, pad)
        vr, fr = M.largest_component(*M.marching_cubes(grid.cpu().numpy(), 0.0, center, extent, pad))
        assert f.shape[0] > 1000
        assert np.array_equal(v.cpu().numpy(), vr) and np.array_equal(f.cpu().numpy(), fr), "person %d" % pid
    final = {0: meshes[2], 1: meshes[1]}
    for pid, (v, f) in final.items():
        m.set_canonical_mesh(pid, v, f)
    fresh = S.mirror_model(sc)
    for pid, (v, f) in final.items():
        fresh.set_canonical_mesh(pid, v.clone(), f.clone())
    inp = S.make_rays(sc, 256, seed=35, region="boxes")
    hits = [h.cuda() for h in S.make_hit_lists(sc, inp)]
    got = train(m, mirror_inputs(inp, 2, hits, epoch=137), 4322)
    want = train(fresh, mirror_inputs(inp, 2, hits, epoch=137), 4322)
    for k in ("index_off_surface", "index_in_surface", "rgb_values"):
        assert torch.equal(got[k], want[k]), k


def test_generate_mesh_on_caller_stream(mirror):
    """Person 0's mesh extracted on a non-default stream equals the default stream's."""
    sc, m = mirror
    v0, f0 = umesh.generate_mesh(m, 0, _cond(sc, 0), sc["persons"][0]["verts_c"], res_init=32, res_up=2)
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        v, f = umesh.generate_mesh(m, 0, _cond(sc, 0), sc["persons"][0]["verts_c"], res_init=32, res_up=2)
        assert torch.equal(v, v0) and torch.equal(f, f0)


PIXELS = ("rgb_values", "fg_rgb_values", "normal_values", "acc_map", "acc_person_list")


def test_render_on_caller_stream(trained):
    """The caller's current stream is a non-default stream: set_cond (which rewrites the field's folded first-layer bias
    in place) right after a render that read the field on its branch streams, host inputs (device copies made for the
    call and released on return), and the outputs read on that stream with no host synchronisation.  Both renders equal
    the same renders on the default stream."""
    sc, _, _ = trained
    r = engine.Renderer(sc)
    inp = S.make_rays(sc, 512, seed=9, region="boxes")
    hits = S.make_hit_lists(sc, inp)
    conds = [sc["persons"][0]["cond"], sc["persons"][1]["cond"]]
    want = []
    for c in conds:
        r.fields[0].set_cond(c)
        o = r.render(inp, hits)
        torch.cuda.synchronize()
        want.append({k: o[k].clone() for k in PIXELS})
    assert not torch.equal(want[0]["rgb_values"], want[1]["rgb_values"])
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        got = []
        for c in conds:
            r.fields[0].set_cond(c)
            got.append(r.render(inp, hits))
        for w, g in zip(want, got):
            for k in PIXELS:
                assert same(w[k], g[k]), k
    r.fields[0].set_cond(conds[0])
    torch.cuda.synchronize()
