"""Every workspace and storage query reports exactly the bytes its call needs, and the call writes none beyond them.

Each `*_bytes` query returns the size of the layout its call carves.  For every query/call pair the call runs with its
buffer placed at the front of a larger allocation whose tail holds a sentinel:
- with exactly the query's bytes it succeeds, leaves the tail untouched and gives outputs bit-identical to a run with a
  generously oversized buffer;
- with one byte less it is refused ("too small") before it enqueues anything: no launch, outputs untouched;
- with a base 16 bytes past a 256-byte boundary it is refused.
The MLP operator query (mp_mlp_workspace_bytes, and the MLP share of every layout that nests it) is the largest layout
of both engines and all their programs, because the engine can change between the query and the call.  Every call runs
under both engines.  A call whose own layout is that largest one (the gradient chains, and every layout that nests the
MLP query) is refused one byte less under at least one engine; any other call must write nothing past that byte."""
import ctypes as C
from contextlib import contextmanager

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from multiply_b200 import engine, scene as S, _lib as L     # noqa: E402
from multiply_b200.utils import mesh as umesh               # noqa: E402
from test_gpu_workspace_reuse import geo, trained, _composite_inputs, _pts, P_C, R_C, N_C, BETA_C  # noqa: F401

TAIL = 4096 + 256
SENT = 0xA5
SPARE = 1 << 20         # the generously oversized run


def _launches():
    return L.call("mp_launch_count", 0)


@contextmanager
def placed(monkeypatch, names, mode, pos=-2):
    """Every call of one of ``names`` made through ``_lib.call`` in the block gets, instead of its buffer argument
    (args[pos]; its byte count at args[pos + 1], which callers size by the query), the front of a sentinel-filled
    allocation: the query's bytes ("exact"), one byte less ("short"), SPARE more ("generous"), or the query's bytes
    16 bytes past an aligned base ("misaligned").  Calls that share a buffer share its replacement.  The allocations
    outlive the block (a handle built in one keeps using it).  A call that returns must have written nothing past the
    bytes it got; a refused one must have launched nothing."""
    real = L.call
    bigs = {}
    seen = []

    def call(fname, *args):
        if fname not in names:
            return real(fname, *args)
        args = list(args)
        buf, need = args[pos], int(args[pos + 1])
        key = buf.data_ptr()
        if key not in bigs:
            bigs[key] = torch.full((need + SPARE + TAIL,), SENT, dtype=torch.uint8, device="cuda")
        big = bigs[key]
        off = 16 if mode == "misaligned" else 0
        got = {"exact": need, "short": need - 1, "generous": need + SPARE, "misaligned": need}[mode]
        args[pos], args[pos + 1] = big[off:], got
        seen.append(need)
        n0 = _launches()
        try:
            r = real(fname, *args)
        except L.MpError:
            assert _launches() == n0, "%s launched kernels before it refused its buffer" % fname
            raise
        torch.cuda.synchronize()
        bad = int((big[off + got:] != SENT).sum())
        assert bad == 0, "%s wrote %d bytes past the %d it was given (query %d)" % (fname, bad, got, need)
        return r

    with monkeypatch.context() as m:
        m.setattr(L, "call", call)
        yield seen
    placed.keep.append(bigs)


placed.keep = []


@pytest.fixture(autouse=True)
def _release():
    yield
    placed.keep.clear()


def _bits(v):
    if not torch.is_tensor(v):
        return v
    v = v.detach().contiguous().reshape(-1)
    return v.to(torch.uint8) if v.dtype == torch.bool else v.view(torch.uint8).clone()


def _snap(out):
    torch.cuda.synchronize()
    return {k: _bits(v) for k, v in out.items()}


def _equal(a, b):
    return torch.equal(a, b) if torch.is_tensor(a) else a == b


def check_bounds(monkeypatch, name, run, outs=dict, pos=-2, refuse=True):
    """name: the entry point, or a tuple of entry points that share one buffer.  run(o) makes the calls (``o = outs()``,
    output buffers filled with sentinels) and returns a dict of outputs.  refuse=False: the call may accept one byte
    less (see the module docstring).  Returns whether it refused."""
    names = name if isinstance(name, tuple) else (name,)
    with placed(monkeypatch, names, "generous", pos):
        want = _snap(run(outs()))
    with placed(monkeypatch, names, "exact", pos) as seen:
        got = _snap(run(outs()))
    assert seen, "%s was not called" % name
    for k in want:
        assert _equal(want[k], got[k]), "%s: output %s differs with exactly the query's bytes" % (name, k)
    o = outs()
    before = _snap(o)
    refused = True
    try:
        with placed(monkeypatch, names, "short", pos):
            run(o)
        refused = False
    except L.MpError as e:
        assert "too small" in str(e), str(e)
    if refused:
        after = _snap(o)
        for k in before:
            assert _equal(before[k], after[k]), "%s: output %s written by a refused call" % (name, k)
    assert refused or not refuse, "%s accepted one byte less than its query" % name
    with pytest.raises(L.MpError, match="256-byte aligned"):
        with placed(monkeypatch, names, "misaligned", pos):
            run(outs())
    return refused


def check_engines(monkeypatch, name, run, outs=dict, need_refusal=True):
    """check_bounds under both MLP engines; need_refusal: the call's layout is the query's, so one engine refuses one
    byte less."""
    refused = []
    try:
        for eng in ("tc", "simt"):
            engine.set_engine(eng)
            refused.append(check_bounds(monkeypatch, name, run, outs, refuse=False))
    finally:
        engine.set_engine("tc")
    assert any(refused) or not need_refusal, "%s: neither engine refused one byte less" % name


def _full(shape, dtype=torch.float32):
    shape = shape if isinstance(shape, tuple) else (shape,)
    v = -1234.5 if dtype.is_floating_point else (0xA5 if dtype == torch.uint8 else -7)
    return torch.full(shape, v, dtype=dtype, device="cuda")


def _mlp_ws(N):
    return L.workspace(L.call("mp_mlp_workspace_bytes", N), "cuda")


# ---------------------------------------------------------------------------------------------
# networks, lattice SDF, deformer SDF, background
# ---------------------------------------------------------------------------------------------

EDGES = [1, 127, 129, 32767, 32769]


@pytest.mark.parametrize("N", EDGES)
@pytest.mark.parametrize("grad", [False, True])
def test_implicit_forward_bounds(monkeypatch, trained, N, grad):
    f = trained[1][0]
    x = _pts(N, 3, 10 + N)
    name = "mp_implicit_forward_grad" if grad else "mp_implicit_forward"

    def outs():
        return dict(sdf=_full(N), feat=_full((N, 256)), grad=_full((N, 3)))

    def run(o):
        ws = _mlp_ws(N)
        if grad:
            L.call(name, f.handle, x, N, o["sdf"], o["feat"], o["grad"], ws, ws.numel())
        else:
            L.call(name, f.handle, x, N, o["sdf"], o["feat"], ws, ws.numel())
        return o

    check_engines(monkeypatch, name, run, outs, need_refusal=grad)


@pytest.mark.parametrize("N", [1, 129, 65537])
def test_render_forward_bounds(monkeypatch, trained, N):
    f = trained[1][0]
    x, nrm, feat = _pts(N, 3, 1), _pts(N, 3, 2), _pts(N, 256, 3)

    def run(o):
        ws = _mlp_ws(N)
        L.call("mp_render_forward", f.handle, x, nrm, feat, N, o["rgb"], ws, ws.numel())
        return o

    check_engines(monkeypatch, "mp_render_forward", run, lambda: dict(rgb=_full((N, 3))), need_refusal=False)


@pytest.mark.parametrize("N", [1, 127, 129])
def test_bg_nets_forward_bounds(monkeypatch, trained, N):
    bg = trained[2]
    pts, view = _pts(N, 4, 5), _pts(N, 3, 6)
    view = (view / view.norm(dim=1, keepdim=True)).contiguous()

    def run(o):
        ws = _mlp_ws(N)
        L.call("mp_bg_nets_forward", bg.handle, pts, view, N, o["sdf"], o["rgb"], ws, ws.numel())
        return o

    check_engines(monkeypatch, "mp_bg_nets_forward", run, lambda: dict(sdf=_full(N), rgb=_full((N, 3))),
                  need_refusal=False)


@pytest.mark.parametrize("res", [8, 101])
def test_sdf_grid_bounds(monkeypatch, trained, res):
    """res 101: (res + 1)^3 > 2^20, two slabs."""
    sc, fields, _ = trained
    center, extent, pad = umesh.bounds(sc["persons"][0]["verts_c"])

    def run(o):
        ws = L.workspace(L.call("mp_sdf_grid_workspace_bytes", res), "cuda")
        L.call("mp_sdf_grid", fields[0].handle, L.vec3(C.c_float, center), float(extent), float(pad), res, o["v"], ws,
               ws.numel())
        return o

    check_engines(monkeypatch, "mp_sdf_grid", run, lambda: dict(v=_full((res + 1) ** 3)))


@pytest.mark.parametrize("N", [1, 129, 32769])
def test_sdf_with_deformer_bounds(monkeypatch, geo, N):
    sc, f, body = geo
    x = _pts(N, 3, 7, -0.8, 0.8)

    def run(o):
        ws = L.workspace(L.call("mp_sdf_with_deformer_workspace_bytes", N), "cuda")
        L.call("mp_sdf_with_deformer", body.handle, f.handle, x, N, o["sdf"], o["xc"], o["feat"], ws, ws.numel())
        return o

    check_engines(monkeypatch, "mp_sdf_with_deformer", run,
                  lambda: dict(sdf=_full(N), xc=_full((N, 3)), feat=_full((N, 256))))


@pytest.mark.parametrize("R", [1, 301])
def test_background_bounds(monkeypatch, trained, R):
    bg = trained[2]
    d = _pts(R, 3, 8)
    d = (d / d.norm(dim=1, keepdim=True)).contiguous()
    c = _pts(R, 3, 9, -1.5, 1.5)

    def run(o):
        ws = L.workspace(L.call("mp_background_workspace_bytes", R), "cuda")
        L.call("mp_background", bg.handle, d, c, R, 3.0, o["rgb"], ws, ws.numel())
        return o

    check_engines(monkeypatch, "mp_background", run, lambda: dict(rgb=_full((R, 3))))


# ---------------------------------------------------------------------------------------------
# sampler, compositor, SMPL and deformer backward
# ---------------------------------------------------------------------------------------------

@pytest.mark.parametrize("R", [1, 129])
@pytest.mark.parametrize("train", [False, True])
def test_sample_rays_bounds(monkeypatch, geo, R, train):
    from test_gpu_sampler import rays, train_rng
    sc, f, body = geo
    cfg = dict(sc["cfg"], beta_param=sc["beta_param"])
    c = engine.sampler_cfg(cfg, cfg["beta_param"])
    n = cfg["N_samples"] + cfg["N_samples_extra"] + 2
    d, o_ = (t.cuda() for t in rays(sc, R, seed=4))
    rng, keep = engine.sampler_rng_struct(train_rng(cfg, R, seed=4), torch.device("cuda"))
    name = "mp_sample_rays_train" if train else "mp_sample_rays"

    def outs():
        return dict(z=_full((R, n)), z_bg=_full((R, 32)), z_eik=_full(R), trips=_full(1, torch.int32))

    def run(o):
        ws = L.workspace(L.call("mp_sampler_workspace_bytes", c, R), "cuda")
        if train:
            L.call(name, c, body.handle, f.handle, d, o_, R, rng, o["z"], o["z_bg"], o["z_eik"], o["trips"], ws,
                   ws.numel())
        else:
            L.call(name, c, body.handle, f.handle, d, o_, R, o["z"], o["z_bg"], o["trips"], ws, ws.numel())
        return o

    check_engines(monkeypatch, name, run, outs)


def test_composite_bounds(monkeypatch):
    x = _composite_inputs(11)

    def outs():
        return dict(fg=_full((R_C, 3)), nrm=_full((R_C, 3)), acc=_full(R_C), accp=_full((R_C, P_C)), bgT=_full(R_C))

    def run(o):
        ws = L.workspace(L.call("mp_composite_workspace_bytes", R_C, P_C), "cuda")
        L.call("mp_composite", x["arr"], P_C, R_C, N_C, BETA_C, o["fg"], o["nrm"], o["acc"], o["accp"], o["bgT"], ws,
               ws.numel())
        return o

    check_bounds(monkeypatch, "mp_composite", run, outs)


def test_composite_backward_bounds(monkeypatch):
    x = _composite_inputs(12)
    u = x["ups"]

    def outs():
        o = dict(d_beta=_full(1))
        for p in range(P_C):
            for k in ("sdf", "rgb", "nrm"):
                o["%s%d" % (k, p)] = _full((R_C, N_C, 3 if k != "sdf" else 1))
        return o

    def run(o):
        gr = (L.PersonSampleGrads * P_C)()
        for p in range(P_C):
            gr[p].d_sdf, gr[p].d_rgb, gr[p].d_normal = (L.ptr(o["%s%d" % (k, p)]) for k in ("sdf", "rgb", "nrm"))
        ws = L.workspace(L.call("mp_composite_backward_workspace_bytes", R_C, P_C), "cuda")
        L.call("mp_composite_backward", x["arr"], P_C, R_C, N_C, BETA_C, u["d_fg"], u["d_nrm"], u["d_acc"], u["d_accp"],
               u["d_bgT"], gr, o["d_beta"], ws, ws.numel())
        return o

    check_bounds(monkeypatch, "mp_composite_backward", run, outs)


def test_smpl_backward_bounds(monkeypatch):
    from test_gpu_body_grad import Smpl
    sm = Smpl(S.make_smpl_model(300))
    rng = np.random.RandomState(1)
    args = Smpl._args(1.05, rng.normal(0, 0.3, 3), rng.normal(0, 0.4, 72), rng.normal(0, 1, 10))
    dv = torch.from_numpy(rng.standard_normal((sm.V, 3)).astype(np.float32)).cuda()
    dt = torch.from_numpy(rng.standard_normal((24, 4, 4)).astype(np.float32)).cuda()

    def run(o):
        ws = L.workspace(L.call("mp_smpl_backward_workspace_bytes", sm.V), "cuda")
        L.call("mp_smpl_backward", sm.h, *args, 0, dv, dt, o["scale"], o["transl"], o["thetas"], o["betas"], ws,
               ws.numel())
        return o

    check_bounds(monkeypatch, "mp_smpl_backward", run,
                 lambda: dict(scale=_full(1), transl=_full(3), thetas=_full(72), betas=_full(10)))


@pytest.mark.parametrize("N", [1, 4097])
def test_deform_backward_bounds(monkeypatch, N):
    from test_gpu_body_grad import _points, _posed_body
    body, _ = _posed_body()
    p = _points(N, body.verts_p, 71).cuda()
    u = torch.from_numpy(np.random.RandomState(1).randn(N, 3).astype(np.float32)).cuda()
    uj = torch.from_numpy(np.random.RandomState(2).randn(N, 9).astype(np.float32)).cuda()

    def outs():
        return dict(d_tfs=_full((24, 4, 4)), d_x=_full((N, 3)), xc=_full((N, 3)))

    def run_inv(o):
        ws = L.workspace(L.call("mp_deform_backward_workspace_bytes", N), "cuda")
        L.call("mp_deform_inverse_backward", body.handle, p, N, 1, u, o["d_tfs"], o["d_x"], o["xc"], ws, ws.numel())
        return o

    def run_fwd(o):
        ws = L.workspace(L.call("mp_deform_backward_workspace_bytes", N), "cuda")
        L.call("mp_deform_forward_jac_backward", body.handle, p, N, u, uj, o["d_tfs"], o["d_x"], ws, ws.numel())
        return o

    check_bounds(monkeypatch, "mp_deform_inverse_backward", run_inv, outs)
    check_bounds(monkeypatch, "mp_deform_forward_jac_backward", run_fwd, outs)


# ---------------------------------------------------------------------------------------------
# mesh extraction
# ---------------------------------------------------------------------------------------------

@pytest.mark.parametrize("res_init,depth", [(4, 1), (16, 2)])
def test_mise_bounds(monkeypatch, trained, res_init, depth):
    sc, fields, _ = trained
    center, extent, pad = umesh.bounds(sc["persons"][0]["verts_c"])
    n1 = (res_init << depth) + 1

    def run(o):
        n = C.c_longlong(0)
        ws = L.workspace(L.call("mp_mise_workspace_bytes", res_init, depth), "cuda")
        L.call("mp_mise", fields[0].handle, L.vec3(C.c_float, center), float(extent), float(pad), res_init, depth, 0.0,
               o["grid"], o["ev"], C.byref(n), ws, ws.numel())
        return dict(o, n=n.value)

    check_engines(monkeypatch, "mp_mise", run, lambda: dict(grid=_full(n1 ** 3), ev=_full(n1 ** 3, torch.uint8)))


@pytest.fixture(scope="module")
def grid64(trained):
    sc, fields, _ = trained
    center, extent, pad = umesh.bounds(sc["persons"][0]["verts_c"])
    g = fields[0].mise(center, extent, 16, 2, 0.0, pad)[0]
    torch.cuda.synchronize()
    return g


def test_marching_cubes_bounds(monkeypatch, grid64):
    """Count and emit share one workspace (emit reads the count's offsets)."""
    R = grid64.shape[0] - 1
    v0, f0 = engine.marching_cubes(grid64, 0.0)
    V, F = v0.shape[0], f0.shape[0]

    def run(o):
        ws = L.workspace(L.call("mp_marching_cubes_workspace_bytes", R), "cuda")
        nv, nf = C.c_longlong(0), C.c_longlong(0)
        L.call("mp_marching_cubes_count", grid64, R, 0.0, C.byref(nv), C.byref(nf), ws, ws.numel())
        L.call("mp_marching_cubes_emit", grid64, R, 0.0, L.vec3(C.c_double, (R / 2.0,) * 3), float(R), 1.0, o["v"],
               o["f"], ws, ws.numel())
        return dict(o, V=nv.value, F=nf.value)

    check_bounds(monkeypatch, ("mp_marching_cubes_count", "mp_marching_cubes_emit"), run,
                 lambda: dict(v=_full(3 * V), f=_full(3 * F, torch.int64)))


def test_largest_component_bounds(monkeypatch, grid64):
    v, f = engine.marching_cubes(grid64, 0.0)
    V, F = v.shape[0], f.shape[0]

    def run(o):
        ws = L.workspace(L.call("mp_largest_component_workspace_bytes", V, F), "cuda")
        nv, nf = C.c_int(0), C.c_int(0)
        L.call("mp_largest_component", v, V, f, F, o["v"], o["f"], C.byref(nv), C.byref(nf), ws, ws.numel())
        return dict(o, V=nv.value, F=nf.value)

    check_bounds(monkeypatch, "mp_largest_component", run, lambda: dict(v=_full(3 * V), f=_full(3 * F, torch.int64)))


# ---------------------------------------------------------------------------------------------
# persistent stores: body, SMPL server, canonical mesh
# ---------------------------------------------------------------------------------------------

def test_body_storage_bounds(monkeypatch, trained):
    p = trained[0]["persons"][1]
    from test_gpu_body_grad import _points
    x = _points(4097, p["verts_p"], 90).cuda()

    def run(o):
        b = engine.Body(p["verts_c"], p["weights"], cano_cell=0.1001 / p["scale"])
        b.set_pose(p["verts_p"], p["tfs"])
        xc, out = b.deform_inverse(x)
        return dict(xc=xc, out=out)

    check_bounds(monkeypatch, "mp_body_create", run, pos=-3)


def test_smpl_storage_bounds(monkeypatch):
    from test_gpu_body_grad import Smpl
    model = S.make_smpl_model(301)
    rng = np.random.RandomState(4)
    args = (1.1, rng.normal(0, 0.3, 3), rng.normal(0, 0.4, 72), rng.normal(0, 1, 10))

    def run(o):
        s = Smpl(model)
        v, t = s.forward(*args, absolute=False)
        return dict(cinv=torch.from_numpy(s.cinv), v=v, t=t)

    check_bounds(monkeypatch, "mp_smpl_create", run, pos=-3)


def test_mesh_storage_bounds(monkeypatch):
    v, f = S.make_body_mesh(101)
    g = torch.Generator().manual_seed(5)
    vt = torch.as_tensor(v).float()
    pts = (vt[torch.randint(vt.shape[0], (6000,), generator=g)] + 0.05 * torch.randn(6000, 3, generator=g)).cuda()

    def run(o):
        m = engine.CanonicalMesh(v, f)
        d2, fi, dt = m.distance(pts)
        return dict(d2=d2, fi=fi, dt=dt, sign=m.check_sign(pts))

    check_bounds(monkeypatch, "mp_mesh_create", run, pos=-3)


def test_pack_and_plan_refuse_a_misaligned_base(monkeypatch, trained):
    """The two buffers outside the query rule, mp_field_pack's storage (sized by an upper bound) and mp_mesh_plan's
    fixed scratch, follow the alignment rule too."""
    p = trained[0]["persons"][0]
    with pytest.raises(L.MpError, match="mp_field_pack: storage base .* not 256-byte aligned"):
        with placed(monkeypatch, ("mp_field_pack",), "misaligned", pos=-3):
            engine.Field(p["implicit"], p["render"])
    v, f = S.make_body_mesh(100)
    vd, fd = torch.as_tensor(v).float().cuda(), torch.as_tensor(f).long().cuda()
    scratch = L.workspace(L.MP_MESH_PLAN_SCRATCH_BYTES + 16, "cuda")
    plan = L.MeshPlan()
    n0 = _launches()
    with pytest.raises(L.MpError, match="mp_mesh_plan: scratch base .* not 256-byte aligned"):
        L.call("mp_mesh_plan", vd, vd.shape[0], fd, fd.shape[0], 0.01, scratch[16:], plan)
    assert _launches() == n0
    L.call("mp_mesh_plan", vd, vd.shape[0], fd, fd.shape[0], 0.01, scratch, plan)
    assert plan.storage_bytes > 0


def test_zero_size_calls_take_the_query_with_a_null_buffer(trained, geo):
    """At N = 0 the deformer backward's layout is empty: its query answers 0 and the call takes (NULL, 0), still
    writing d_tfs = 0.  The calls that return before their carve at a zero size take (NULL, their query) as well, and
    write nothing."""
    from test_gpu_body_grad import _posed_body
    body, _ = _posed_body()
    assert L.call("mp_deform_backward_workspace_bytes", 0) == 0
    for P in (1, 3):
        assert L.call("mp_composite_workspace_bytes", 0, P) == 0
        assert L.call("mp_composite_backward_workspace_bytes", 0, P) == 0
    one, u = _pts(1, 3, 1), _pts(1, 9, 2)
    for name, args in (("mp_deform_inverse_backward", (body.handle, None, 0, 1, None)),
                       ("mp_deform_forward_jac_backward", (body.handle, None, 0, None, None))):
        d_tfs = _full((24, 4, 4))
        if name == "mp_deform_inverse_backward":
            L.call(name, *args, d_tfs, None, None, None, 0)
        else:
            L.call(name, *args, d_tfs, None, None, 0)
        torch.cuda.synchronize()
        assert torch.equal(d_tfs, torch.zeros_like(d_tfs)), name
    sc, f, b = geo
    bg = trained[2]
    o = _full(8)
    L.call("mp_implicit_forward", f.handle, one, 0, o, None, None, L.call("mp_mlp_workspace_bytes", 0))
    L.call("mp_implicit_forward_grad", f.handle, one, 0, o, None, o, None, L.call("mp_mlp_workspace_bytes", 0))
    L.call("mp_render_forward", trained[1][0].handle, one, one, u, 0, o, None, L.call("mp_mlp_workspace_bytes", 0))
    L.call("mp_bg_nets_forward", bg.handle, one, one, 0, o, o, None, L.call("mp_mlp_workspace_bytes", 0))
    L.call("mp_sdf_with_deformer", b.handle, f.handle, one, 0, o, o, None, None,
           L.call("mp_sdf_with_deformer_workspace_bytes", 0))
    L.call("mp_background", bg.handle, one, one, 0, 3.0, o, None, L.call("mp_background_workspace_bytes", 0))
    cfg = dict(sc["cfg"], beta_param=sc["beta_param"])
    c = engine.sampler_cfg(cfg, cfg["beta_param"])
    L.call("mp_sample_rays", c, b.handle, f.handle, one, one, 0, o, None, None, None,
           L.call("mp_sampler_workspace_bytes", c, 0))
    torch.cuda.synchronize()
    assert torch.equal(o, _full(8))


# ---------------------------------------------------------------------------------------------
# the fused render
# ---------------------------------------------------------------------------------------------

PIXELS = (("rgb_values", 3), ("fg_rgb_values", 3), ("normal_values", 3), ("acc_map", 0), ("acc_person_list", 2))


@pytest.fixture(scope="module")
def render_setup():
    engine.set_engine("tc")
    sc = S.make_scene(P=2, S=16, seed=42)
    r = engine.Renderer(sc)
    inp = S.make_rays(sc, 300, seed=9, region="boxes")
    hits = S.make_hit_lists(sc, inp)
    meshes = [engine.CanonicalMesh(*S.make_body_mesh(100 + p)) for p in range(2)]
    return sc, r, inp, hits, meshes


@pytest.mark.parametrize("mode", ["eval", "device_counts", "train", "train_meshes"])
def test_render_rays_bounds(monkeypatch, render_setup, mode):
    from test_gpu_sampler import train_rng
    sc, r, inp, hits, meshes = render_setup
    R = inp["uv"].shape[1]
    hl = [h.cuda() for h in hits]
    if mode == "device_counts":
        hl = [(h, torch.tensor([h.numel()], dtype=torch.int32, device="cuda")) for h in hl]
    train = None
    if mode.startswith("train"):
        g = torch.Generator().manual_seed(3)
        train = dict(rng=[train_rng(r.cfg, h.numel(), seed=20 + k) for k, h in enumerate(hl)],
                     t_rand_bg=torch.rand(R, 32, generator=g))
        if mode == "train_meshes":
            train["meshes"] = meshes

    def outs():
        return {k: _full((R, w) if w else (R,)) for k, w in PIXELS}

    def run(o):
        r._ws = None
        res = r.render(inp, hl, out=o, train=train)
        return {k: res[k] for k in res if torch.is_tensor(res[k])}

    check_bounds(monkeypatch, "mp_render_rays", run, outs)
