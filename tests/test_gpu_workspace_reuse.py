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
import ctypes as C

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from multiply_b200 import engine, scene as S, _lib as L     # noqa: E402
from multiply_b200.utils import mesh as umesh               # noqa: E402
from oracle import mesh_extract as M                        # noqa: E402


# ---------------------------------------------------------------------------------------------
# fresh versus reused buffers
# ---------------------------------------------------------------------------------------------

def _bits(t):
    """The bytes of a tensor (NaNs compare by bit pattern), or a host value as is."""
    if not torch.is_tensor(t):
        return t
    t = t.detach().contiguous().reshape(-1)
    return t.to(torch.uint8) if t.dtype == torch.bool else t.view(torch.uint8)


def _same(a, b):
    a, b = _bits(a), _bits(b)
    return torch.equal(a, b) if torch.is_tensor(a) else a == b


def _snap(out):
    torch.cuda.synchronize()
    return {k: v.clone() if torch.is_tensor(v) else v for k, v in out.items()}


def check_reuse(run, a, b, bufs):
    """run(inp, bufs) -> dict of outputs (views of ``bufs`` or host values).  ``bufs``: name -> tensor giving the shape
    and dtype of every buffer the call writes (workspace included).  B on zeroed buffers, then A on other zeroed
    buffers, then B on A's buffers and A on B's: both reused runs must equal the fresh ones bit for bit, and A and B
    must differ (else the reuse proves nothing).  Returns (A, B) fresh outputs."""
    zero = lambda: {k: torch.zeros_like(v) for k, v in bufs.items()}          # noqa: E731
    s1, s2 = zero(), zero()
    b_fresh = _snap(run(b, s1))
    a_fresh = _snap(run(a, s2))
    b_reused = _snap(run(b, s2))
    a_reused = _snap(run(a, s1))
    for tag, want, got in (("B", b_fresh, b_reused), ("A", a_fresh, a_reused)):
        for k in want:
            assert _same(want[k], got[k]), "%s: output %s differs when its buffers held another call's bytes" % (tag, k)
    assert any(not _same(a_fresh[k], b_fresh[k]) for k in a_fresh), "A and B give identical outputs"
    return a_fresh, b_fresh


# ---------------------------------------------------------------------------------------------
# scenes
# ---------------------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def trained():
    """The trained-like scene: both persons' fields with their own cond, and the background field."""
    engine.set_engine("tc")
    sc = S.make_scene(P=2, S=16, seed=42, weights="trained")
    fields = []
    for p in sc["persons"]:
        f = engine.Field(p["implicit"], p["render"])
        f.set_cond(p["cond"])
        fields.append(f)
    bg = engine.Field(sc["bg_implicit"], sc["bg_render"], background=True)
    bg.set_cond(sc["frame_code"])
    return sc, fields, bg


@pytest.fixture(scope="module")
def geo():
    """Person 0 of the geometric scene the sampler tests use: field, posed body."""
    engine.set_engine("tc")
    sc = S.make_scene(P=2, S=16, seed=42)
    p = sc["persons"][0]
    f = engine.Field(p["implicit"], p["render"])
    f.set_cond(p["cond"])
    b = engine.Body(p["verts_c"], p["weights"], cano_cell=0.1001 / p["scale"])
    b.set_pose(p["verts_p"], p["tfs"])
    return sc, f, b


def _person_box(sc, fields, pid):
    center, extent, pad = umesh.bounds(sc["persons"][pid]["verts_c"])
    return fields[pid], center, extent, pad


@pytest.fixture(scope="module")
def mise_grids(trained):
    """Both persons' MISE grids at res_init 32, depth 2 (R = 128)."""
    sc, fields, _ = trained
    out = []
    for pid in range(2):
        f, center, extent, pad = _person_box(sc, fields, pid)
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
    n1 = (res_init << depth) + 1

    def run(inp, b):
        f, center, extent, pad = inp
        n = C.c_longlong(0)
        L.call("mp_mise", f.handle, L.vec3(C.c_float, center), float(extent), float(pad), res_init, depth, 0.0, b["grid"],
               b["ev"], C.byref(n), b["ws"], b["ws"].numel())
        return dict(grid=b["grid"], ev=b["ev"], n=n.value)

    bufs = dict(grid=torch.empty(n1 ** 3, device="cuda"), ev=torch.empty(n1 ** 3, dtype=torch.uint8, device="cuda"),
                ws=L.workspace(L.call("mp_mise_workspace_bytes", res_init, depth), "cuda"))
    a, b = check_reuse(run, _person_box(sc, fields, 0), _person_box(sc, fields, 1), bufs)
    print("MISE %d/%d: %d and %d points evaluated" % (res_init, depth, a["n"], b["n"]))
    if depth == 4:
        assert min(a["n"], b["n"]) > (depth + 1) << 20


def test_marching_cubes_reuse(mise_grids):
    """Count and emit on one workspace (emit reads the count's offsets), persons 0 and 1's MISE grids; outputs sized for
    the larger mesh, each compared over the rows its call writes.  The fresh meshes equal the oracle's."""
    R = mise_grids[0].shape[0] - 1
    sizes = [engine.marching_cubes(g, 0.0) for g in mise_grids]
    Vm, Fm = max(v.shape[0] for v, _ in sizes), max(f.shape[0] for _, f in sizes)

    def run(g, b):
        V, F = C.c_longlong(0), C.c_longlong(0)
        L.call("mp_marching_cubes_count", g, R, 0.0, C.byref(V), C.byref(F), b["ws"], b["ws"].numel())
        L.call("mp_marching_cubes_emit", g, R, 0.0, L.vec3(C.c_double, (R / 2.0,) * 3), float(R), 1.0, b["v"], b["f"],
               b["ws"], b["ws"].numel())
        return dict(V=V.value, F=F.value, v=b["v"][:3 * V.value], f=b["f"][:3 * F.value])

    bufs = dict(ws=L.workspace(L.call("mp_marching_cubes_workspace_bytes", R), "cuda"),
                v=torch.empty(3 * Vm, device="cuda"), f=torch.empty(3 * Fm, dtype=torch.int64, device="cuda"))
    outs = check_reuse(run, mise_grids[0], mise_grids[1], bufs)
    for g, o in zip(mise_grids, outs):
        vr, fr = M.marching_cubes(g.cpu().numpy(), 0.0)
        assert np.array_equal(o["v"].cpu().numpy().reshape(-1, 3), vr)
        assert np.array_equal(o["f"].cpu().numpy().reshape(-1, 3), fr)


def _lc_run(b, inp):
    v, f = inp
    V, F = v.shape[0], f.shape[0]
    Vo, Fo = C.c_int(0), C.c_int(0)
    L.call("mp_largest_component", v, V, f, F, b["v"], b["f"], C.byref(Vo), C.byref(Fo), b["ws"], b["ws"].numel())
    return dict(V=Vo.value, F=Fo.value, v=b["v"][:3 * Vo.value], f=b["f"][:3 * Fo.value])


def _lc_bufs(V, F):
    return dict(ws=L.workspace(L.call("mp_largest_component_workspace_bytes", V, F), "cuda"),
                v=torch.empty(3 * V, device="cuda"), f=torch.empty(3 * F, dtype=torch.int64, device="cuda"))


def test_largest_component_reuse(mise_grids):
    """A: marching cubes of person 0's grid; B: the same V and F with the faces relabelled by a vertex permutation, so
    every component, root and sort key differs.  Both fresh results equal the oracle's."""
    v, f = engine.marching_cubes(mise_grids[0], 0.0)
    V, F = v.shape[0], f.shape[0]
    perm = torch.randperm(V, generator=torch.Generator().manual_seed(3)).cuda()
    fb = perm[f].contiguous()
    outs = check_reuse(lambda inp, b: _lc_run(b, inp), (v, f), (v, fb), _lc_bufs(V, F))
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
    o = _lc_run(_lc_bufs(2 * n, faces.shape[0]), (vd, fd))
    torch.cuda.synchronize()
    assert (o["V"], o["F"]) == (n, n - 2), "kept %d vertices and %d faces of the %d / %d of the long strip" % (
        o["V"], o["F"], n, n - 2)
    assert torch.equal(o["v"].cpu().reshape(-1, 3), verts[0::2])
    assert torch.equal(o["f"].cpu().reshape(-1, 3), torch.stack([k, k + 1, k + 2], 1))


def test_sdf_grid_reuse(trained):
    sc, fields, _ = trained
    res = 64

    def run(inp, b):
        f, center, extent, pad = inp
        L.call("mp_sdf_grid", f.handle, L.vec3(C.c_float, center), float(extent), float(pad), res, b["vals"], b["ws"],
               b["ws"].numel())
        return dict(vals=b["vals"])

    bufs = dict(vals=torch.empty((res + 1) ** 3, device="cuda"),
                ws=L.workspace(L.call("mp_sdf_grid_workspace_bytes", res), "cuda"))
    check_reuse(run, _person_box(sc, fields, 0), _person_box(sc, fields, 1), bufs)


# ---------------------------------------------------------------------------------------------
# networks, background, sampler
# ---------------------------------------------------------------------------------------------

def _pts(N, d, seed, lo=-1.0, hi=1.0):
    g = torch.Generator().manual_seed(seed)
    return (lo + (hi - lo) * torch.rand(N, d, generator=g)).cuda()


def _mlp_ws(N):
    return L.workspace(L.call("mp_mlp_workspace_bytes", N), "cuda")


@pytest.mark.parametrize("N", [1, 127, 129])
@pytest.mark.parametrize("grad", [False, True])
def test_implicit_forward_reuse(trained, N, grad):
    _, fields, _ = trained
    f = fields[0]

    def run(x, b):
        if grad:
            L.call("mp_implicit_forward_grad", f.handle, x, N, b["sdf"], b["feat"], b["grad"], b["ws"], b["ws"].numel())
            return dict(sdf=b["sdf"], feat=b["feat"], grad=b["grad"])
        L.call("mp_implicit_forward", f.handle, x, N, b["sdf"], b["feat"], b["ws"], b["ws"].numel())
        return dict(sdf=b["sdf"], feat=b["feat"])

    bufs = dict(sdf=torch.empty(N, device="cuda"), feat=torch.empty(N, 256, device="cuda"), ws=_mlp_ws(N))
    if grad:
        bufs["grad"] = torch.empty(N, 3, device="cuda")
    check_reuse(run, _pts(N, 3, 10 + N), _pts(N, 3, 20 + N), bufs)


@pytest.mark.parametrize("N", [1, 127, 129])
def test_bg_nets_forward_reuse(trained, N):
    _, _, bg = trained

    def run(inp, b):
        pts, view = inp
        L.call("mp_bg_nets_forward", bg.handle, pts, view, N, b["sdf"], b["rgb"], b["ws"], b["ws"].numel())
        return dict(sdf=b["sdf"], rgb=b["rgb"])

    def inp(seed):
        view = _pts(N, 3, seed + 1)
        return _pts(N, 4, seed, -1.0, 1.0), (view / view.norm(dim=1, keepdim=True)).contiguous()

    bufs = dict(sdf=torch.empty(N, device="cuda"), rgb=torch.empty(N, 3, device="cuda"), ws=_mlp_ws(N))
    check_reuse(run, inp(30 + N), inp(40 + N), bufs)


def test_background_reuse(trained):
    """Rays from cameras inside the r = 3 sphere, R = 301 (not a multiple of the 8 rays per block)."""
    _, _, bg = trained
    R = 301

    def inp(seed):
        d = _pts(R, 3, seed)
        return (d / d.norm(dim=1, keepdim=True)).contiguous(), _pts(R, 3, seed + 1, -1.5, 1.5)

    def run(rays, b):
        d, c = rays
        L.call("mp_background", bg.handle, d, c, R, 3.0, b["rgb"], b["ws"], b["ws"].numel())
        return dict(rgb=b["rgb"])

    bufs = dict(rgb=torch.empty(R, 3, device="cuda"),
                ws=L.workspace(L.call("mp_background_workspace_bytes", R), "cuda"))
    check_reuse(run, inp(50), inp(60), bufs)


@pytest.mark.parametrize("train", [False, True])
def test_sample_rays_reuse(geo, train):
    """The eval and the training sampler on person 0's rays (A: one ray set and draws, B: another)."""
    from test_gpu_sampler import rays, train_rng
    sc, f, body = geo
    cfg = dict(sc["cfg"], beta_param=sc["beta_param"])
    c = engine.sampler_cfg(cfg, cfg["beta_param"])
    R = 300
    n = cfg["N_samples"] + cfg["N_samples_extra"] + 2

    def inp(seed):
        d, o = rays(sc, R, seed=seed)
        return d.cuda(), o.cuda(), train_rng(cfg, R, seed=seed)

    def run(x, b):
        d, o, rng = x
        if not train:
            L.call("mp_sample_rays", c, body.handle, f.handle, d, o, R, b["z"], b["z_bg"], b["trips"], b["ws"],
                   b["ws"].numel())
            return dict(z=b["z"], z_bg=b["z_bg"], trips=b["trips"])
        r, keep = engine.sampler_rng_struct(rng, torch.device("cuda"))
        L.call("mp_sample_rays_train", c, body.handle, f.handle, d, o, R, r, b["z"], b["z_bg"], b["z_eik"], b["trips"],
               b["ws"], b["ws"].numel())
        torch.cuda.synchronize()        # the draws in ``keep`` are read by the kernels
        return dict(z=b["z"], z_bg=b["z_bg"], z_eik=b["z_eik"], trips=b["trips"])

    bufs = dict(z=torch.empty(R, n, device="cuda"), z_bg=torch.empty(R, 32, device="cuda"),
                z_eik=torch.empty(R, device="cuda"), trips=torch.empty(1, dtype=torch.int32, device="cuda"),
                ws=L.workspace(L.call("mp_sampler_workspace_bytes", c, R), "cuda"))
    check_reuse(run, inp(5), inp(6), bufs)


# ---------------------------------------------------------------------------------------------
# compositor and its backward
# ---------------------------------------------------------------------------------------------

P_C, R_C, N_C, BETA_C = 3, 300, 33, 0.1


def _composite_inputs(seed):
    from test_gpu_composite import make_inputs, person_samples
    persons = make_inputs(seed, P_C, R_C, N_C)
    arr, keep = person_samples(persons)
    rng = np.random.RandomState(seed + 100)
    ups = {k: torch.from_numpy(rng.standard_normal(s).astype(np.float32)).cuda()
           for k, s in (("d_fg", (R_C, 3)), ("d_nrm", (R_C, 3)), ("d_acc", R_C), ("d_accp", (R_C, P_C)), ("d_bgT", R_C))}
    return dict(arr=arr, keep=keep, rows=[d["idx"].size for d in persons], ups=ups)


def test_composite_reuse():
    def run(x, b):
        L.call("mp_composite", x["arr"], P_C, R_C, N_C, BETA_C, b["fg"], b["nrm"], b["acc"], b["accp"], b["bgT"], b["ws"],
               b["ws"].numel())
        return {k: b[k] for k in ("fg", "nrm", "acc", "accp", "bgT")}

    bufs = dict(fg=torch.empty(R_C, 3, device="cuda"), nrm=torch.empty(R_C, 3, device="cuda"),
                acc=torch.empty(R_C, device="cuda"), accp=torch.empty(R_C, P_C, device="cuda"),
                bgT=torch.empty(R_C, device="cuda"),
                ws=L.workspace(L.call("mp_composite_workspace_bytes", R_C, P_C), "cuda"))
    check_reuse(run, _composite_inputs(11), _composite_inputs(12), bufs)


def test_composite_backward_reuse():
    """Gradient buffers hold R rows per person (hit lists differ between A and B); each is compared over its rows."""
    def run(x, b):
        gr = (L.PersonSampleGrads * P_C)()
        for p in range(P_C):
            gr[p].d_sdf, gr[p].d_rgb, gr[p].d_normal = (L.ptr(b["%s%d" % (k, p)]) for k in ("sdf", "rgb", "nrm"))
        u = x["ups"]
        L.call("mp_composite_backward", x["arr"], P_C, R_C, N_C, BETA_C, u["d_fg"], u["d_nrm"], u["d_acc"], u["d_accp"],
               u["d_bgT"], gr, b["d_beta"], b["ws"], b["ws"].numel())
        out = {"d_beta": b["d_beta"]}
        for p, rows in enumerate(x["rows"]):
            out["sdf%d" % p] = b["sdf%d" % p][:rows]
            out["rgb%d" % p] = b["rgb%d" % p][:rows]
            out["nrm%d" % p] = b["nrm%d" % p][:rows]
        return out

    bufs = dict(d_beta=torch.empty(1, device="cuda"),
                ws=L.workspace(L.call("mp_composite_backward_workspace_bytes", R_C, P_C), "cuda"))
    for p in range(P_C):
        bufs["sdf%d" % p] = torch.empty(R_C, N_C, device="cuda")
        bufs["rgb%d" % p] = torch.empty(R_C, N_C, 3, device="cuda")
        bufs["nrm%d" % p] = torch.empty(R_C, N_C, 3, device="cuda")
    check_reuse(run, _composite_inputs(11), _composite_inputs(12), bufs)


# ---------------------------------------------------------------------------------------------
# SMPL server and deformer backward
# ---------------------------------------------------------------------------------------------

def test_smpl_backward_reuse():
    from test_gpu_body_grad import Smpl
    sm = Smpl(S.make_smpl_model(300))
    V = sm.V

    def inp(seed):
        rng = np.random.RandomState(seed)
        args = Smpl._args(1.0 + 0.1 * rng.rand(), rng.normal(0, 0.3, 3), rng.normal(0, 0.4, 72), rng.normal(0, 1, 10))
        dv = torch.from_numpy(rng.standard_normal((V, 3)).astype(np.float32)).cuda()
        dt = torch.from_numpy(rng.standard_normal((24, 4, 4)).astype(np.float32)).cuda()
        return args, dv, dt

    def run(x, b):
        args, dv, dt = x
        L.call("mp_smpl_backward", sm.h, *args, 0, dv, dt, b["scale"], b["transl"], b["thetas"], b["betas"], b["ws"],
               b["ws"].numel())
        return {k: b[k] for k in ("scale", "transl", "thetas", "betas")}

    bufs = dict(scale=torch.empty(1, device="cuda"), transl=torch.empty(3, device="cuda"),
                thetas=torch.empty(72, device="cuda"), betas=torch.empty(10, device="cuda"),
                ws=L.workspace(L.call("mp_smpl_backward_workspace_bytes", V), "cuda"))
    check_reuse(run, inp(1), inp(2), bufs)


@pytest.mark.parametrize("N", [1, 4097])
def test_deform_backward_reuse(N):
    from test_gpu_body_grad import _points, _posed_body
    body, _ = _posed_body()

    def inp(seed):
        u = torch.from_numpy(np.random.RandomState(seed).randn(N, 3).astype(np.float32)).cuda()
        uj = torch.from_numpy(np.random.RandomState(seed + 1).randn(N, 9).astype(np.float32)).cuda()
        return _points(N, body.verts_p, seed).cuda(), u, uj

    def run_inv(x, b):
        p, u, _ = x
        L.call("mp_deform_inverse_backward", body.handle, p, N, 1, u, b["d_tfs"], b["d_x"], b["xc"], b["ws"],
               b["ws"].numel())
        return {k: b[k] for k in ("d_tfs", "d_x", "xc")}

    def run_fwd(x, b):
        p, u, uj = x
        L.call("mp_deform_forward_jac_backward", body.handle, p, N, u, uj, b["d_tfs"], b["d_x"], b["ws"],
               b["ws"].numel())
        return {k: b[k] for k in ("d_tfs", "d_x")}

    bufs = dict(d_tfs=torch.empty(24, 4, 4, device="cuda"), d_x=torch.empty(N, 3, device="cuda"),
                xc=torch.empty(N, 3, device="cuda"),
                ws=L.workspace(L.call("mp_deform_backward_workspace_bytes", N), "cuda"))
    check_reuse(run_inv, inp(71), inp(72), bufs)
    del bufs["xc"]
    check_reuse(run_fwd, inp(73), inp(74), bufs)


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
    want, got = _snap(first_call(fresh)), _snap(first_call(stale))
    for k in want:
        assert _same(want[k], got[k]), "%s differs when the handle was built in another handle's storage" % k


def test_field_store_reuse(monkeypatch, trained):
    sc, fields, bg = trained
    p1 = sc["persons"][1]
    x = _pts(129, 3, 80)
    nrm = _pts(129, 3, 81)

    def first(f):
        f.set_cond(p1["cond"])
        sdf, feat, grad = f.implicit_forward(x, want_grad=True)
        return dict(sdf=sdf, feat=feat, grad=grad, rgb=f.render_forward(x, nrm, feat))

    _stores_agree(monkeypatch, fields[0].storage, lambda: engine.Field(p1["implicit"], p1["render"]), first)

    def first_bg(f):
        f.set_cond(sc["frame_code"])
        sdf, rgb = f.bg_forward(_pts(129, 4, 82), nrm / nrm.norm(dim=1, keepdim=True))
        return dict(sdf=sdf, rgb=rgb)

    _stores_agree(monkeypatch, fields[0].storage,
                  lambda: engine.Field(sc["bg_implicit"], sc["bg_render"], background=True), first_bg)


def test_body_store_reuse(monkeypatch, trained):
    sc, _, _ = trained
    p0, p1 = sc["persons"]
    old = engine.Body(p0["verts_c"], p0["weights"], cano_cell=0.1001 / p0["scale"])
    old.set_pose(p0["verts_p"], p0["tfs"])
    torch.cuda.synchronize()
    from test_gpu_body_grad import _points
    x = _points(4097, p1["verts_p"], 90).cuda()

    def first(b):
        b.set_pose(p1["verts_p"], p1["tfs"])
        xc, out = b.deform_inverse(x)
        xd, J = b.forward_jac(xc)
        return dict(xc=xc, out=out, xd=xd, J=J)

    _stores_agree(monkeypatch, old.storage,
                  lambda: engine.Body(p1["verts_c"], p1["weights"], cano_cell=0.1001 / p1["scale"]), first)


def test_smpl_store_reuse(monkeypatch):
    from test_gpu_body_grad import Smpl
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
    from test_gpu_mirror import _build
    engine.set_engine("tc")
    sc = S.make_scene(P=2, S=16, seed=42, weights="trained")
    return sc, _build(sc)


def _cond(sc, pid):
    return {"smpl": sc["persons"][pid]["cond"].cuda()}


def test_epoch_end_mesh_sequence(mirror):
    """generate_mesh for person 0, person 1, person 0 with no cleanup in between: person 0's two meshes are
    bit-identical and every mesh equals the oracle's marching cubes and largest component on the same MISE grid.  Then
    both meshes go to set_canonical_mesh and a training step's surface flags equal those of a model that only ever saw
    the final meshes."""
    from test_gpu_mirror import _build
    from test_gpu_mesh import _inputs, _train
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
    fresh = _build(sc)
    for pid, (v, f) in final.items():
        fresh.set_canonical_mesh(pid, v.clone(), f.clone())
    inp = S.make_rays(sc, 256, seed=35, region="boxes")
    hits = [h.cuda() for h in S.make_hit_lists(sc, inp)]
    got = _train(m, _inputs(sc, inp, hits, 137), 4322)
    want = _train(fresh, _inputs(sc, inp, hits, 137), 4322)
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
                assert _same(w[k], g[k]), k
    r.fields[0].set_cond(conds[0])
    torch.cuda.synchronize()
