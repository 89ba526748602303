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
MLP query) is refused one byte less under at least one engine; any other call must write nothing past that byte.
The one buffer outside this rule is mp_mesh_plan's fixed scratch (MP_MESH_PLAN_SCRATCH_BYTES), which follows the
alignment rule."""
import ctypes as C
import re
from contextlib import contextmanager

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from multiply_b200 import engine, scene as S, _lib as L     # noqa: E402
from multiply_b200.utils import mesh as umesh               # noqa: E402

import _calls as calls                                                              # noqa: E402
from _abi import same, sentinel, snap                                               # noqa: E402
from _setups import (Smpl, field_descs, geo, points, posed_body, pts, refused_fields, train_rng,   # noqa: E402,F401
                     trained)

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


def check_bounds(monkeypatch, name, run, outs=dict, pos=-2, refuse=True):
    """name: the entry point, or a tuple of entry points that share one buffer.  run(o) makes the calls (``o = outs()``,
    output buffers filled with sentinels) and returns a dict of outputs.  refuse=False: the call may accept one byte
    less (see the module docstring).  Returns whether it refused."""
    names = name if isinstance(name, tuple) else (name,)
    with placed(monkeypatch, names, "generous", pos):
        want = snap(run(outs()))
    with placed(monkeypatch, names, "exact", pos) as seen:
        got = snap(run(outs()))
    assert seen, "%s was not called" % name
    for k in want:
        assert same(want[k], got[k]), "%s: output %s differs with exactly the query's bytes" % (name, k)
    o = outs()
    before = snap(o)
    refused = True
    try:
        with placed(monkeypatch, names, "short", pos):
            run(o)
        refused = False
    except L.MpError as e:
        assert "too small" in str(e), str(e)
    if refused:
        after = snap(o)
        for k in before:
            assert same(before[k], after[k]), "%s: output %s written by a refused call" % (name, k)
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
    return torch.full(shape, sentinel(dtype), dtype=dtype, device="cuda")


def _case(case, x):
    """check_bounds' (name, run, outs) for a call case on inputs x: sentinel-filled outputs, a workspace of the query's
    bytes, and every output buffer compared whole."""
    def run(o):
        return {**case.call(x, o, L.workspace(case.query(), "cuda")), **o}
    return case.name, run, lambda: {k: _full(shape, dtype) for k, (shape, dtype) in case.outs.items()}


# ---------------------------------------------------------------------------------------------
# networks, lattice SDF, deformer SDF, background
# ---------------------------------------------------------------------------------------------

EDGES = [1, 127, 129, 32767, 32769]


@pytest.mark.parametrize("N", EDGES)
@pytest.mark.parametrize("grad", [False, True])
def test_implicit_forward_bounds(monkeypatch, trained, N, grad):
    c = calls.implicit_forward(trained[1][0], N, grad)
    check_engines(monkeypatch, *_case(c, c.inputs(10 + N)), need_refusal=grad)


@pytest.mark.parametrize("N", [1, 129, 65537])
def test_render_forward_bounds(monkeypatch, trained, N):
    f = trained[1][0]
    x, nrm, feat = pts(N, 3, 1), pts(N, 3, 2), pts(N, 256, 3)

    def run(o):
        ws = L.workspace(L.call("mp_mlp_workspace_bytes", N), "cuda")
        L.call("mp_render_forward", f.handle, x, nrm, feat, N, o["rgb"], ws, ws.numel())
        return o

    check_engines(monkeypatch, "mp_render_forward", run, lambda: dict(rgb=_full((N, 3))), need_refusal=False)


@pytest.mark.parametrize("N", [1, 127, 129])
def test_bg_nets_forward_bounds(monkeypatch, trained, N):
    c = calls.bg_nets_forward(trained[2], N)
    check_engines(monkeypatch, *_case(c, c.inputs(5)), need_refusal=False)


@pytest.mark.parametrize("res", [8, 101])
def test_sdf_grid_bounds(monkeypatch, trained, res):
    """res 101: (res + 1)^3 > 2^20, two slabs."""
    sc, fields, _ = trained
    c = calls.sdf_grid(sc, fields, res)
    check_engines(monkeypatch, *_case(c, c.inputs(0)))


@pytest.mark.parametrize("N", [1, 129, 32769])
def test_sdf_with_deformer_bounds(monkeypatch, geo, N):
    sc, f, body = geo
    x = pts(N, 3, 7, -0.8, 0.8)

    def run(o):
        ws = L.workspace(L.call("mp_sdf_with_deformer_workspace_bytes", N), "cuda")
        L.call("mp_sdf_with_deformer", body.handle, f.handle, x, N, o["sdf"], o["xc"], o["feat"], ws, ws.numel())
        return o

    check_engines(monkeypatch, "mp_sdf_with_deformer", run,
                  lambda: dict(sdf=_full(N), xc=_full((N, 3)), feat=_full((N, 256))))


@pytest.mark.parametrize("N", EDGES)
@pytest.mark.parametrize("net", ["implicit", "bg_implicit", "render"])
def test_network_backward_bounds(monkeypatch, trained, net, N):
    """The networks' backward runs on the tensor cores only (it has no SIMT path), and its layout holds one chunk of
    32768 points at most: N = 32769 runs two chunks in it."""
    f = trained[2] if net == "bg_implicit" else trained[1][0]
    c = calls.render_backward(f, N) if net == "render" else calls.implicit_backward(f, N)
    check_bounds(monkeypatch, *_case(c, c.inputs(30 + N)))


@pytest.mark.parametrize("R", [1, 301])
def test_background_bounds(monkeypatch, trained, R):
    c = calls.background(trained[2], R)
    check_engines(monkeypatch, *_case(c, c.inputs(8)))


# ---------------------------------------------------------------------------------------------
# sampler, compositor, SMPL and deformer backward
# ---------------------------------------------------------------------------------------------

@pytest.mark.parametrize("R", [1, 129])
@pytest.mark.parametrize("train", [False, True])
def test_sample_rays_bounds(monkeypatch, geo, R, train):
    sc, f, body = geo
    c = calls.sample_rays(sc, f, body, R, train)
    check_engines(monkeypatch, *_case(c, c.inputs(4)))


def test_composite_bounds(monkeypatch):
    c = calls.composite()
    check_bounds(monkeypatch, *_case(c, c.inputs(11)))


def test_composite_backward_bounds(monkeypatch):
    c = calls.composite_backward()
    check_bounds(monkeypatch, *_case(c, c.inputs(12)))


def test_smpl_backward_bounds(monkeypatch):
    c = calls.smpl_backward(Smpl(S.make_smpl_model(300)))
    check_bounds(monkeypatch, *_case(c, c.inputs(1)))


@pytest.mark.parametrize("N", [1, 4097])
def test_deform_backward_bounds(monkeypatch, N):
    body, _ = posed_body()
    for c in (calls.deform_inverse_backward(body, N), calls.deform_forward_jac_backward(body, N)):
        check_bounds(monkeypatch, *_case(c, c.inputs(71)))


# ---------------------------------------------------------------------------------------------
# mesh extraction
# ---------------------------------------------------------------------------------------------

@pytest.mark.parametrize("res_init,depth", [(4, 1), (16, 2)])
def test_mise_bounds(monkeypatch, trained, res_init, depth):
    sc, fields, _ = trained
    c = calls.mise(sc, fields, res_init, depth)
    check_engines(monkeypatch, *_case(c, c.inputs(0)))


@pytest.fixture(scope="module")
def grid64(trained):
    sc, fields, _ = trained
    center, extent, pad = umesh.bounds(sc["persons"][0]["verts_c"])
    g = fields[0].mise(center, extent, 16, 2, 0.0, pad)[0]
    torch.cuda.synchronize()
    return g


def test_marching_cubes_bounds(monkeypatch, grid64):
    """Count and emit share one workspace (emit reads the count's offsets)."""
    v0, f0 = engine.marching_cubes(grid64, 0.0)
    c = calls.marching_cubes(grid64.shape[0] - 1, v0.shape[0], f0.shape[0])
    check_bounds(monkeypatch, *_case(c, grid64))


def test_largest_component_bounds(monkeypatch, grid64):
    v, f = engine.marching_cubes(grid64, 0.0)
    c = calls.largest_component(v.shape[0], f.shape[0])
    check_bounds(monkeypatch, *_case(c, (v, f)))


# ---------------------------------------------------------------------------------------------
# persistent stores: body, SMPL server, canonical mesh
# ---------------------------------------------------------------------------------------------

def test_body_storage_bounds(monkeypatch, trained):
    p = trained[0]["persons"][1]
    x = points(4097, p["verts_p"], 90).cuda()

    def run(o):
        b = engine.Body(p["verts_c"], p["weights"], cano_cell=0.1001 / p["scale"])
        b.set_pose(p["verts_p"], p["tfs"])
        xc, out = b.deform_inverse(x)
        return dict(xc=xc, out=out)

    check_bounds(monkeypatch, "mp_body_create", run, pos=-3)


def test_smpl_storage_bounds(monkeypatch):
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


def test_field_storage_bounds(monkeypatch, geo, trained):
    """mp_field_pack's storage: foreground fields on geometric and trained weights, the background field, and the
    mirror's fields whose partner network is a zero stand-in without weight norm (weight_g NULL).  Every field is
    evaluated by implicit_forward with and without the gradient and render_forward, or bg_forward, under both engines."""
    from multiply_b200.model import networks
    N = 129
    x, nrm, feat, x4 = pts(N, 3, 1), pts(N, 3, 2), pts(N, 256, 3), pts(N, 4, 4)
    view = pts(N, 3, 5)
    view = (view / view.norm(dim=1, keepdim=True)).contiguous()

    def mirror(cls, opt, sd):
        net = cls(S.MODEL_OPT[opt])
        net.load_state_dict(sd, strict=True)
        return net.field("cuda")

    def run(o):
        fields = []
        for sc in (geo[0], trained[0]):
            p = sc["persons"][0]
            fields += [("fg", engine.Field(p["implicit"], p["render"]), p["cond"])]
        sc, p = trained[0], trained[0]["persons"][0]
        fields += [("bg", engine.Field(sc["bg_implicit"], sc["bg_render"], background=True), sc["frame_code"]),
                   ("fg", mirror(networks.ImplicitNet, "implicit_network", p["implicit"]), p["cond"]),
                   ("fg", mirror(networks.RenderingNet, "rendering_network", p["render"]), p["cond"]),
                   ("bg", mirror(networks.ImplicitNet, "bg_implicit_network", sc["bg_implicit"]), sc["frame_code"]),
                   ("bg", mirror(networks.RenderingNet, "bg_rendering_network", sc["bg_render"]), sc["frame_code"])]
        out = {}
        try:
            for eng in ("tc", "simt"):
                engine.set_engine(eng)
                for i, (kind, f, cond) in enumerate(fields):
                    f.set_cond(cond)
                    if kind == "bg":
                        out.update({f"{i}/{eng}/bg/{k}": v for k, v in zip(("sdf", "rgb"), f.bg_forward(x4, view))})
                        continue
                    out.update({f"{i}/{eng}/fwd/{k}": v for k, v in zip(("sdf", "feat"), f.implicit_forward(x))})
                    out.update({f"{i}/{eng}/grad/{k}": v
                                for k, v in zip(("sdf", "feat", "grad"), f.implicit_forward(x, want_grad=True))})
                    out[f"{i}/{eng}/rgb"] = f.render_forward(x, nrm, feat)
        finally:
            engine.set_engine("tc")
        return out

    check_bounds(monkeypatch, "mp_field_pack", run, pos=-3)


def test_pack_refuses_unsupported_networks_before_any_launch(geo):
    """Every kind of network pair mp_field_pack refuses is refused with its message before anything is enqueued: no
    launch, the storage untouched, and no handle."""
    storage = torch.full((32 << 20,), SENT, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    for what, (isd, rsd, background, imp), msg in refused_fields(geo[0]):
        d, r, keep = field_descs(isd, rsd, background, "cuda", **imp)
        h = L.Handle("mp_field_free")
        n0 = _launches()
        with pytest.raises(L.MpError, match=re.escape("mp_field_pack failed") + ".*" + re.escape(msg)):
            L.call("mp_field_pack", d, r, int(background), storage, storage.numel(), C.byref(h))
        assert _launches() == n0, what
        assert not h.value, what
    torch.cuda.synchronize()
    assert bool((storage == SENT).all())


def test_mesh_plan_refuses_a_misaligned_scratch():
    """mp_mesh_plan's fixed scratch, the one buffer outside the query rule, follows the alignment rule."""
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
    body, _ = posed_body()
    assert L.call("mp_deform_backward_workspace_bytes", 0) == 0
    for P in (1, 3):
        assert L.call("mp_composite_workspace_bytes", 0, P) == 0
        assert L.call("mp_composite_backward_workspace_bytes", 0, P) == 0
    one, u = pts(1, 3, 1), pts(1, 9, 2)
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
