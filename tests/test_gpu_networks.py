"""GPU: conformance of the MLP kernels (both engines) against oracle/port.py evaluated in float64 on the CPU, on the
geometric-init weights and on the trained-like weights of scene.perturb_networks.

The geometric init zeroes the Fourier columns, makes weight norm the identity and zeroes the hidden biases, so on it
the chain rule through sin / cos, the weight-norm fold and the bias loads of the epilogues are never exercised with
non-zero data.  Every operator entry point of the networks is checked here on both weight sets:
  - at sizes around the warp, warpgroup and 128-row tile edges and around T = 128 x SMs (one tile per CTA), N = 0
    included, through the C ABI with output buffers padded by a sentinel tail that must survive the call;
  - for row-position invariance: f(x)[k:] == f(x[k:]) bit for bit (rows are independent and the reduction order is
    fixed, so any difference is an indexing or layout bug);
  - for grid invariance: the tensor-core chain run with 1 and 3 persistent CTAs (many tiles per CTA: mbarrier phase
    wrap, scratch reuse) must give bit-identical outputs to the default grid;
  - in the precision modes of the tensor-core engine;
and the fused render (per-sample debug taps included) and the Multiply mirror are compared with the oracle."""
import ctypes as C
import os
import subprocess
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
from _setups import mirror_inputs             # noqa: E402

ENGINES = ["simt", "tc"]
WEIGHTS = ["geometric", "trained"]
# the network tolerances of tests/test_gpu_parity.py (gradients get twice that), here measured against fp64
TOL_NET = {"simt": 1e-5, "tc": 2e-5}
TOL_GATE = 1e-4               # BASELINE.json north_star: RGB / SDF / normals
SHIFTS = (1, 8, 16, 64, 127)  # moves rows across warp (8 rows per quad group), warpgroup (64) and tile (128) boundaries


# ---------------------------------------------------------------------------------------------
# inputs and fp64 references
# ---------------------------------------------------------------------------------------------

def _tile_points():
    from multiply_b200 import _lib as L
    return 128 * int(L.call("mp_device_sm_count"))


def _sizes(T):
    return [0, 1, 63, 64, 65, 127, 128, 129, 255, 257, T - 1, T, T + 1, 3 * T + 77]


def _scene(weights):
    return S.make_scene(P=2, S=64, seed=42, weights=weights)


def _fg_points(person, n, seed=1):
    """Canonical points: half over the [-1, 1]^3 box, half within ~0.05 of the body surface, interleaved."""
    g = torch.Generator().manual_seed(seed)
    vc = person["verts_c"]
    box = (torch.rand(n, 3, generator=g) - 0.5) * 2.0
    near = vc[torch.randint(0, vc.shape[0], (n,), generator=g)] + 0.05 * torch.randn(n, 3, generator=g)
    pick = torch.rand(n, generator=g) < 0.5
    return torch.where(pick[:, None], near, box).contiguous()


def _bg_points(n, seed=2):
    g = torch.Generator().manual_seed(seed)
    x4 = torch.nn.functional.normalize(torch.randn(n, 3, generator=g), dim=1)
    x4 = torch.cat([x4, torch.rand(n, 1, generator=g) / 3.0], 1).contiguous()
    vd = torch.nn.functional.normalize(torch.randn(n, 3, generator=g), dim=1).contiguous()
    return x4, vd


def _f64(sd):
    return {k: v.double() for k, v in sd.items()}


def _ref_fg(person, x, chunk=8192):
    """fp64 ImplicitNet: (out [N,257], grad sdf [N,3])."""
    sd, cond = _f64(person["implicit"]), person["cond"].double()
    outs, grads = [], []
    for s in range(0, x.shape[0], chunk):
        xs = x[s:s + chunk].double().requires_grad_(True)
        y = port.implicit_forward(sd, xs, cond, 6)
        grads.append(torch.autograd.grad(y[:, 0].sum(), xs)[0])
        outs.append(y.detach())
    return torch.cat(outs), torch.cat(grads)


def _ref_render(person, x, nrm, feat):
    with torch.no_grad():
        return port.rendering_forward(_f64(person["render"]), "pose_no_view", x.double(), nrm.double(), None,
                                      person["cond"].double(), feat.double())


def _ref_bg(sc, pts, view, chunk=8192):
    code = sc["frame_code"].double()
    sdf, rgb = [], []
    with torch.no_grad():
        for s in range(0, pts.shape[0], chunk):
            y = port.implicit_forward(_f64(sc["bg_implicit"]), pts[s:s + chunk].double(), code, 10, weight_norm=False)
            rgb.append(port.rendering_forward(_f64(sc["bg_render"]), "nerf_frame_encoding", None, None,
                                              view[s:s + chunk].double(), None, y[:, 1:], frame_latent_code=code,
                                              weight_norm=False, multires_view=4))
            sdf.append(y[:, 0])
    return torch.cat(sdf), torch.cat(rgb)


class _Case:
    """One weight set: packed fields, inputs of the largest size and their fp64 references."""

    def __init__(self, weights, nmax):
        from multiply_b200 import engine
        self.sc = _scene(weights)
        self.person = self.sc["persons"][0]
        self.field = engine.Field(self.person["implicit"], self.person["render"])
        self.field.set_cond(self.person["cond"])
        self.bg = engine.Field(self.sc["bg_implicit"], self.sc["bg_render"], background=True)
        self.bg.set_cond(self.sc["frame_code"])
        self.x = _fg_points(self.person, nmax)
        self.out64, self.grad64 = _ref_fg(self.person, self.x)
        g = torch.Generator().manual_seed(3)
        self.nrm = torch.nn.functional.normalize(torch.randn(nmax, 3, generator=g), dim=1).contiguous()
        self.feat = self.out64[:, 1:].float().contiguous()          # the colour net's input, identical on both sides
        self.rgb64 = _ref_render(self.person, self.x, self.nrm, self.feat)
        self.pts4, self.view = _bg_points(nmax)
        self.bg_sdf64, self.bg_rgb64 = _ref_bg(self.sc, self.pts4, self.view)


@pytest.fixture(scope="module")
def T():
    return _tile_points()


@pytest.fixture(scope="module")
def cases(T):
    return {w: _Case(w, 3 * T + 77) for w in WEIGHTS}


# ---------------------------------------------------------------------------------------------
# the C ABI with sentinel-padded outputs
# ---------------------------------------------------------------------------------------------

def _ws(N):
    from multiply_b200 import _lib as L
    return L.workspace(L.call("mp_mlp_workspace_bytes", N), "cuda")


def call_implicit(field, x, N, want_feat=True, want_grad=False):
    from multiply_b200 import _lib as L
    xd = rows(x, N)
    sdf = padded(N)
    feat = padded((N, 256)) if want_feat else None
    ws = _ws(N)
    if want_grad:
        grad = padded((N, 3))
        L.call("mp_implicit_forward_grad", field.handle, xd, N, sdf, feat, grad, ws, ws.numel())
    else:
        L.call("mp_implicit_forward", field.handle, xd, N, sdf, feat, ws, ws.numel())
    torch.cuda.synchronize()
    o = {"sdf": take(sdf, N, "sdf")}
    if want_feat:
        o["feat"] = take(feat, (N, 256), "feat")
    if want_grad:
        o["grad"] = take(grad, (N, 3), "grad")
    return o


def call_render(field, x, nrm, feat, N):
    from multiply_b200 import _lib as L
    rgb = padded((N, 3))
    ws = _ws(N)
    L.call("mp_render_forward", field.handle, rows(x, N), rows(nrm, N), rows(feat, N), N, rgb, ws, ws.numel())
    torch.cuda.synchronize()
    return {"rgb": take(rgb, (N, 3), "rgb")}


def call_bg(field, pts, view, N, want_sdf=True):
    from multiply_b200 import _lib as L
    sdf = padded(N) if want_sdf else None
    rgb = padded((N, 3))
    ws = _ws(N)
    L.call("mp_bg_nets_forward", field.handle, rows(pts, N), rows(view, N), N, sdf, rgb, ws, ws.numel())
    torch.cuda.synchronize()
    o = {"rgb": take(rgb, (N, 3), "bg rgb")}
    if want_sdf:
        o["sdf"] = take(sdf, N, "bg sdf")
    return o


def _err(a, b):
    if a.numel() == 0:
        return 0.0
    return float((a.double() - b.double()).abs().max())


def _lattice(person, res, scale=1.1):
    """generate_mesh's lattice (lib/utils/mesh.py:92-95) as port.sdf_grid builds it: (centre, extent, points [n,3])."""
    center, extent, scale = port.mesh_bounds(person["verts_c"], scale)
    idx = np.stack(np.meshgrid(np.arange(res + 1), np.arange(res + 1), np.arange(res + 1), indexing="ij"),
                   -1).reshape(-1, 3)
    pts = (idx.astype(np.float32) / res - 0.5) * scale
    return center, extent, torch.from_numpy(pts * extent + center)


def call_sdf_grid(field, person, res):
    from multiply_b200 import _lib as L
    center, extent, _ = _lattice(person, res)
    n = (res + 1) ** 3
    vals = padded(n)
    ws = L.workspace(L.call("mp_sdf_grid_workspace_bytes", res), "cuda")
    L.call("mp_sdf_grid", field.handle, L.vec3(C.c_float, center), float(extent), 1.1, int(res), vals, ws, ws.numel())
    torch.cuda.synchronize()
    return take(vals, n, "sdf grid")


# ---------------------------------------------------------------------------------------------
# every entry point, every size, both weight sets, against fp64
# ---------------------------------------------------------------------------------------------

@pytest.mark.parametrize("weights", WEIGHTS)
@pytest.mark.parametrize("eng", ENGINES)
def test_implicit_forward(cases, T, eng, weights):
    """mp_implicit_forward with features (forward program) and without (sdf-only program)."""
    from multiply_b200 import engine
    engine.set_engine(eng)
    c = cases[weights]
    worst = {"sdf": 0.0, "feat": 0.0, "sdf_only": 0.0}
    for N in _sizes(T):
        o = call_implicit(c.field, c.x, N)
        worst["sdf"] = max(worst["sdf"], _err(o["sdf"], c.out64[:N, 0]))
        worst["feat"] = max(worst["feat"], _err(o["feat"], c.out64[:N, 1:]))
        o2 = call_implicit(c.field, c.x, N, want_feat=False)
        worst["sdf_only"] = max(worst["sdf_only"], _err(o2["sdf"], c.out64[:N, 0]))
        for k, v in worst.items():
            assert v < TOL_NET[eng], (k, N, v)
    print("\n[%s/%s] mp_implicit_forward fp64 L-inf: %s" % (eng, weights, {k: "%.2e" % v for k, v in worst.items()}))


@pytest.mark.parametrize("weights", WEIGHTS)
@pytest.mark.parametrize("eng", ENGINES)
def test_implicit_forward_grad(cases, T, eng, weights):
    """mp_implicit_forward_grad: sdf, features and d sdf / d x (the reverse sweep through sin / cos of the embedding)."""
    from multiply_b200 import engine
    engine.set_engine(eng)
    c = cases[weights]
    worst = {"sdf": 0.0, "feat": 0.0, "grad": 0.0}
    for N in _sizes(T):
        o = call_implicit(c.field, c.x, N, want_grad=True)
        worst["sdf"] = max(worst["sdf"], _err(o["sdf"], c.out64[:N, 0]))
        worst["feat"] = max(worst["feat"], _err(o["feat"], c.out64[:N, 1:]))
        worst["grad"] = max(worst["grad"], _err(o["grad"], c.grad64[:N]))
        assert worst["sdf"] < TOL_NET[eng] and worst["feat"] < TOL_NET[eng], (N, worst)
        assert worst["grad"] < 2 * TOL_NET[eng], (N, worst)
    print("\n[%s/%s] mp_implicit_forward_grad fp64 L-inf: %s" % (eng, weights,
                                                                  {k: "%.2e" % v for k, v in worst.items()}))


@pytest.mark.parametrize("weights", WEIGHTS)
@pytest.mark.parametrize("eng", ENGINES)
def test_render_forward(cases, T, eng, weights):
    from multiply_b200 import engine
    engine.set_engine(eng)
    c = cases[weights]
    worst = 0.0
    for N in _sizes(T):
        o = call_render(c.field, c.x, c.nrm, c.feat, N)
        worst = max(worst, _err(o["rgb"], c.rgb64[:N]))
        assert worst < TOL_NET[eng], (N, worst)
    print("\n[%s/%s] mp_render_forward fp64 L-inf: rgb %.2e" % (eng, weights, worst))


@pytest.mark.parametrize("weights", WEIGHTS)
@pytest.mark.parametrize("eng", ENGINES)
def test_bg_nets_forward(cases, T, eng, weights):
    from multiply_b200 import engine
    engine.set_engine(eng)
    c = cases[weights]
    worst = {"sdf": 0.0, "rgb": 0.0}
    for N in _sizes(T):
        o = call_bg(c.bg, c.pts4, c.view, N)
        worst["sdf"] = max(worst["sdf"], _err(o["sdf"], c.bg_sdf64[:N]))
        worst["rgb"] = max(worst["rgb"], _err(o["rgb"], c.bg_rgb64[:N]))
        o2 = call_bg(c.bg, c.pts4, c.view, N, want_sdf=False)
        assert torch.equal(o2["rgb"], o["rgb"]), N
        assert max(worst.values()) < TOL_NET[eng], (N, worst)
    print("\n[%s/%s] mp_bg_nets_forward fp64 L-inf: %s" % (eng, weights, {k: "%.2e" % v for k, v in worst.items()}))


@pytest.mark.parametrize("weights", WEIGHTS)
@pytest.mark.parametrize("eng", ENGINES)
def test_sdf_grid(cases, eng, weights):
    """mp_sdf_grid: lattices of 5^3, 8^3, 13^3, 26^3 (past one tile per CTA) and 102^3 (two 2^20-point slabs).  The
    values equal mp_implicit_forward at numpy's lattice points bit for bit, and fp64 on a sample (every point of the
    small lattices; 4096 points plus the slab seam of the large one)."""
    from multiply_b200 import engine
    engine.set_engine(eng)
    c = cases[weights]
    worst = 0.0
    for res in (4, 7, 12, 25, 101):
        vals = call_sdf_grid(c.field, c.person, res)
        _, _, pts = _lattice(c.person, res)
        direct = call_implicit(c.field, pts, pts.shape[0], want_feat=False)["sdf"]
        assert torch.equal(vals, direct), res
        n = pts.shape[0]
        if n <= 20000:
            idx = torch.arange(n)
        else:
            g = torch.Generator().manual_seed(res)
            seam = torch.arange((1 << 20) - 300, (1 << 20) + 300)
            idx = torch.cat([torch.randint(0, n, (4096,), generator=g), seam, torch.arange(n - 64, n)])
        out64, _ = _ref_fg(c.person, pts[idx])
        worst = max(worst, _err(vals[idx], out64[:, 0]))
        assert worst < TOL_NET[eng], (res, worst)
    print("\n[%s/%s] mp_sdf_grid fp64 L-inf: %.2e" % (eng, weights, worst))


# ---------------------------------------------------------------------------------------------
# layout invariances
# ---------------------------------------------------------------------------------------------

def _all_outputs(c, N, x=None, nrm=None, feat=None, pts4=None, view=None):
    """Every network output for the first N rows of the given inputs (the case's by default)."""
    x = c.x if x is None else x
    o = {}
    for k, v in call_implicit(c.field, x, N).items():
        o["fwd_" + k] = v
    o["sdf_only"] = call_implicit(c.field, x, N, want_feat=False)["sdf"]
    for k, v in call_implicit(c.field, x, N, want_grad=True).items():
        o["grad_" + k] = v
    o["rgb"] = call_render(c.field, x, c.nrm if nrm is None else nrm, c.feat if feat is None else feat, N)["rgb"]
    for k, v in call_bg(c.bg, c.pts4 if pts4 is None else pts4, c.view if view is None else view, N).items():
        o["bg_" + k] = v
    return o


@pytest.mark.parametrize("weights", WEIGHTS)
@pytest.mark.parametrize("eng", ENGINES)
def test_row_shift_invariance(cases, eng, weights):
    """f(x)[k:] == f(x[k:]) bit for bit for shifts across warp, warpgroup and tile boundaries."""
    from multiply_b200 import engine
    engine.set_engine(eng)
    c = cases[weights]
    N = 1000
    full = _all_outputs(c, N)
    for k in SHIFTS:
        sh = _all_outputs(c, N - k, x=c.x[k:N], nrm=c.nrm[k:N], feat=c.feat[k:N], pts4=c.pts4[k:N],
                          view=c.view[k:N])
        for name, v in full.items():
            bad = (v[k:] != sh[name]).reshape(N - k, -1).any(1)
            assert not bool(bad.any()), "%s: shift %d changes %d rows (first %d)" % (
                name, k, int(bad.sum()), int(bad.nonzero()[0, 0]))


def _grid_sweep(path):
    """The tensor-core outputs of every entry point on the trained-like weights at sizes that leave a ragged last tile
    and several tiles per CTA, written to ``path`` (npz).  Run in this process and in subprocesses with MP_TC_GRID."""
    from multiply_b200 import engine
    engine.set_engine("tc")
    T = _tile_points()
    c = _Case.__new__(_Case)
    c.sc = _scene("trained")
    c.person = c.sc["persons"][0]
    c.field = engine.Field(c.person["implicit"], c.person["render"])
    c.field.set_cond(c.person["cond"])
    c.bg = engine.Field(c.sc["bg_implicit"], c.sc["bg_render"], background=True)
    c.bg.set_cond(c.sc["frame_code"])
    nmax = 3 * T + 77
    c.x = _fg_points(c.person, nmax)
    g = torch.Generator().manual_seed(3)
    c.nrm = torch.nn.functional.normalize(torch.randn(nmax, 3, generator=g), dim=1).contiguous()
    c.feat = torch.randn(nmax, 256, generator=g).contiguous()
    c.pts4, c.view = _bg_points(nmax)
    res = {}
    for N in (1, 129, T + 1, nmax):
        for k, v in _all_outputs(c, N).items():
            res["%s_%d" % (k, N)] = v.numpy()
    res["grid_25"] = call_sdf_grid(c.field, c.person, 25).numpy()
    np.savez(path, **res)


@pytest.mark.parametrize("grid", [1, 3])
def test_grid_invariance(tmp_path, grid):
    """MP_TC_GRID (read once per process) caps the persistent CTAs of the tensor-core chain: with 1 or 3 CTAs every
    CTA runs many tiles, so its mbarrier phases wrap and its scratch is reused.  The outputs must be bit-identical to
    the default grid's."""
    ref_path, sub_path = tmp_path / "default.npz", tmp_path / ("grid%d.npz" % grid)
    _grid_sweep(ref_path)
    env = dict(os.environ, MP_TC_GRID=str(grid))
    env["PYTHONPATH"] = ROOT + os.pathsep + env.get("PYTHONPATH", "")
    p = subprocess.run([sys.executable, os.path.abspath(__file__), "--grid-sweep", str(sub_path)], env=env, cwd=ROOT,
                       capture_output=True, text=True, timeout=900)
    assert p.returncode == 0, p.stdout[-2000:] + p.stderr[-4000:]
    a, b = np.load(ref_path), np.load(sub_path)
    assert sorted(a.files) == sorted(b.files)
    for k in a.files:
        assert np.array_equal(a[k], b[k]), "%s: %d values differ with MP_TC_GRID=%d" % (
            k, int((a[k] != b[k]).sum()), grid)


# ---------------------------------------------------------------------------------------------
# precision modes of the tensor-core engine on trained-like weights
# ---------------------------------------------------------------------------------------------

def test_precision_modes_trained(cases, T):
    """'colour1' leaves SDF, features and grad sdf bit-identical to 'parity' and keeps RGB within 1e-4 of fp64;
    'throughput' is finite and within 2e-2."""
    from multiply_b200 import engine
    engine.set_engine("tc")
    c = cases["trained"]
    N = T + 1
    outs = {}
    try:
        for mode in ("parity", "colour1", "throughput"):
            engine.set_precision(mode)
            o = {"fg_" + k: v for k, v in call_implicit(c.field, c.x, N, want_grad=True).items()}
            o.update({"bg_" + k: v for k, v in call_bg(c.bg, c.pts4, c.view, N).items()})
            outs[mode] = o
    finally:
        engine.set_precision("parity")
    for k in ("fg_sdf", "fg_feat", "fg_grad", "bg_sdf"):
        assert torch.equal(outs["colour1"][k], outs["parity"][k]), k
    for mode in ("parity", "colour1"):
        assert _err(outs[mode]["bg_rgb"], c.bg_rgb64[:N]) < TOL_GATE, mode
    t = outs["throughput"]
    assert all(bool(torch.isfinite(v).all()) for v in t.values())
    assert _err(t["bg_rgb"], c.bg_rgb64[:N]) < 2e-2
    assert _err(t["fg_sdf"], c.out64[:N, 0]) < 2e-2 and _err(t["bg_sdf"], c.bg_sdf64[:N]) < 2e-2
    print("\n[tc/trained] bg rgb fp64 L-inf: parity %.2e colour1 %.2e throughput %.2e" % tuple(
        _err(outs[m]["bg_rgb"], c.bg_rgb64[:N]) for m in ("parity", "colour1", "throughput")))


# ---------------------------------------------------------------------------------------------
# render level on trained-like weights
# ---------------------------------------------------------------------------------------------

def _render_trained(eng, mode="parity"):
    from multiply_b200 import engine
    engine.set_engine(eng)
    sc = _scene("trained")
    inp = S.make_rays(sc, 256, seed=5, region="boxes")
    hits = S.make_hit_lists(sc, inp)
    try:
        engine.set_precision(mode)
        o = engine.Renderer(sc).render(inp, hits, debug=True)
        torch.cuda.synchronize()
    finally:
        engine.set_precision("parity")
    return sc, inp, hits, o


@pytest.fixture(scope="module")
def oracle_trained():
    sc = _scene("trained")
    inp = S.make_rays(sc, 256, seed=5, region="boxes")
    hits = S.make_hit_lists(sc, inp)
    st = {}
    ref = port.multiply_forward(sc, inp, hits, stats=st, return_samples=True)
    return ref, st["trips"]


def _per_sample_errors(o, ref, p):
    """Per-sample sdf / rgb / normal errors where both sides sampled the same depth and the sample is not an outlier."""
    z = o[f"z_vals_{p}"].cpu().numpy()[:, :-1]
    m = (np.abs(z - ref["_z_vals"][p].numpy()) < 1e-6) & (ref["_sdf"][p].numpy() != 4.0)
    assert m.sum() >= 1000, int(m.sum())        # outliers (sdf = 4) are most samples of a box ray
    e = {"sdf": np.abs(o[f"sdf_{p}"].cpu().numpy() - ref["_sdf"][p].numpy())[m].max()}
    for k in ("rgb", "normals"):
        e[k] = np.abs(o[f"{k}_{p}"].cpu().numpy() - ref["_" + k][p].numpy())[m].max()
    return e


@pytest.mark.parametrize("eng", ENGINES)
def test_render_vs_oracle_trained(oracle_trained, eng):
    """Renderer.render, shipped sampler sizes (64/128/32), 256 rays, trained-like weights, against
    port.multiply_forward: trip counts equal, every output within the gates, and per sample sdf / rgb / normals
    (the debug taps of the fused shade program) within 1e-4 of the oracle's."""
    ref, trips = oracle_trained
    _, _, _, o = _render_trained(eng)
    assert list(o["trips"].cpu().numpy()) == list(trips)
    errs = {k: _err(o[k].cpu(), ref[k]) for k in ("rgb_values", "fg_rgb_values", "normal_values", "acc_map",
                                                   "acc_person_list")}
    for p in range(2):
        for k, v in _per_sample_errors(o, ref, p).items():
            errs[f"{k}_{p}"] = float(v)
    print("\n[%s/trained] render vs oracle L-inf: %s" % (eng, {k: "%.2e" % v for k, v in errs.items()}))
    for k, v in errs.items():
        assert v < TOL_GATE, (k, v)


def test_render_precision_modes_trained(oracle_trained):
    """The fused render in 'colour1': per-sample SDF and normals bit-identical to 'parity', pixels and per-sample RGB
    within 1e-4 of the oracle; 'throughput': finite, RGB within 3e-2."""
    ref, _ = oracle_trained
    _, _, _, par = _render_trained("tc")
    _, _, _, c1 = _render_trained("tc", "colour1")
    _, _, _, thr = _render_trained("tc", "throughput")
    for p in range(2):
        assert torch.equal(c1[f"sdf_{p}"], par[f"sdf_{p}"]) and torch.equal(c1[f"normals_{p}"], par[f"normals_{p}"])
        assert _per_sample_errors(c1, ref, p)["rgb"] < TOL_GATE
    assert _err(c1["rgb_values"].cpu(), ref["rgb_values"]) < TOL_GATE
    assert bool(torch.isfinite(thr["rgb_values"]).all())
    # plain fp16 operands everywhere: 2.05e-2 measured on these weights at the pixel level (on an H100), against 7e-5
    # for the background network alone; the bound of test_precision_modes on the geometric init is 2e-2
    assert _err(thr["rgb_values"].cpu(), ref["rgb_values"]) < 3e-2


def test_mirror_checkpoint_trained():
    """The route a real checkpoint takes: Multiply.load_reference_checkpoint with a Lightning-style state dict of
    trained-like weights, then Multiply.forward with the reference's input dict, against the oracle."""
    from multiply_b200 import engine
    from multiply_b200.model.multiply import Multiply
    engine.set_engine("tc")
    sc = _scene("trained")
    P = 2
    m = Multiply(S.model_opt(sc["cfg"]), smpl_server_list=[S.SyntheticSMPLServer(p, P) for p in range(P)])
    sd = {"model." + k: v for k, v in S.mirror_state_dict(sc).items()}
    res = m.load_reference_checkpoint(sd, strict=True)
    assert not res.missing_keys and not res.unexpected_keys
    m = m.cuda().eval()
    inp = S.make_rays(sc, 96, seed=11, region="boxes")
    hits = S.make_hit_lists(sc, inp)
    ref = port.multiply_forward(sc, inp, hits)
    out = m(mirror_inputs(inp, P, [h.cuda() for h in hits]))
    torch.cuda.synchronize()
    for k in ("rgb_values", "fg_rgb_values", "acc_map", "acc_person_list", "normal_values"):
        assert _err(out[k].cpu(), ref[k]) < TOL_GATE, k


if __name__ == "__main__":
    if len(sys.argv) == 3 and sys.argv[1] == "--grid-sweep":
        _grid_sweep(sys.argv[2])
