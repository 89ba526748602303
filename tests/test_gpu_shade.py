"""GPU: the fused shade pass of mp_render_rays (deform -> work list -> forward Jacobian -> one launch of the full shade
program: SDF, reverse sweep, normal epilogue, colour net) checked sample by sample against float64 at the sampler's
own depths.

The inputs are the render's own samples: every debug tap's depth z rebuilds its point x = cam + z d exactly as
deform_rays_kernel does (fp32, the product and the sum rounded separately), so the points are bit-exact.  Each sample
is then compared with two references, both oracle/port.py evaluated in float64 on the GPU:

  (a) independent, from z alone: inverse LBS with the nearest posed vertex, the 0.1 outlier flag, the forward
      Jacobian with the nearest canonical vertex of x_c, ImplicitNet and d sdf / d x_c, normalize(g . J^-1) then
      normalize(., eps=1e-6) (multiply.py:661, :606), RenderingNet 'pose_no_view'.  A nearest-vertex choice that fp32
      cannot resolve (the fp64 gap between the two nearest vertices, or the distance's gap to 0.1, within what fp32
      rounding of the distance or of x_c can bridge) is never masked: both candidates are evaluated and either is
      accepted.  Those samples are counted and must stay under 0.1 % of all samples; no other sample is excluded.
  (b) the shade program in isolation: x_c and the outlier flags from the renderer's own bodies (the device functions
      the main pass calls), J^-1 from forward_jac, fp64 evaluated at those float32 inputs.  Against the operators the
      fused taps are bit-identical where the same fp32 operations run (see test_bench_case).

Gates.  sdf and rgb: absolute error; normals: |n - n64|_inf * |g64 J64^-1| / ||J64^-1||_2 (a normal's error is the
gradient's error amplified by ||J^-1|| / |g J^-1|).  Samples with |g64 J64^-1| / ||J64^-1||_2 < COND_SMALL carry an
ill-conditioned normal: their rgb error is taken net of the term the normal error carries into rgb
(max_k sum_j |d rgb_k / d n_j| * |n - n64|_inf).  Every gate is 4x the worst value measured on one H100 (printed as
MEASURED at the end of the module); in addition reference (b) must stay within 2x the operator tolerance TOL_NET, and
every sample of reference (a) within the 1e-4 north star, ill-conditioned normals by their scaled measure."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
for _p in (ROOT, HERE):
    if _p not in sys.path:
        sys.path.insert(0, _p)

from multiply_b200 import engine, scene as S          # noqa: E402
from oracle import port                               # noqa: E402

from _abi import same                                 # noqa: E402

ENGINES = ["simt", "tc"]
TOL_NET = {"simt": 1e-5, "tc": 2e-5}     # operator-level fp64 tolerance of test_gpu_networks.py (gradients: twice)
TOL_GATE = 1e-4                          # BASELINE.json north star: RGB / SDF / normals
COND_SMALL = 0.1                         # |g J^-1| / ||J^-1|| below which a normal counts as ill-conditioned
TIE_REL = 2.0 ** -20                     # fp32 rounding of a squared distance: < 5 * 2^-24 relative each
TIE_FRAC = 1e-3                          # tie-margin samples allowed, over every sample the module compares
BENCH_RAYS, BENCH_S = 4096, 128          # bench.py: 2 persons, 4096 'boxes' rays, S/E/X = 128/256/64 (n = 193)
DEV = "cuda"                             # the fp64 references run on the GPU

# 4x the worst measured on one H100 80GB HBM3 at a 700 W power limit, per (reference, class, engine); rgb1 is the
# 'colour1' precision mode of the tensor-core engine.  Measured: a/sdf 6.29e-6 simt, 7.95e-6 tc; a/rgb 5.64e-7, 5.57e-7;
# a/nrm 5.97e-6, 8.51e-6; b/sdf 5.85e-6, 7.10e-6; b/rgb 5.63e-7, 5.61e-7; b/nrm 4.43e-6, 9.24e-6; rgb1 8.38e-5 (both)
GATE = {
    ("a", "sdf", "simt"): 2.52e-5, ("a", "rgb", "simt"): 2.26e-6, ("a", "nrm", "simt"): 2.39e-5,
    ("a", "sdf", "tc"): 3.18e-5, ("a", "rgb", "tc"): 2.23e-6, ("a", "nrm", "tc"): 3.41e-5,
    ("b", "sdf", "simt"): 2.34e-5, ("b", "rgb", "simt"): 2.26e-6, ("b", "nrm", "simt"): 1.78e-5,
    ("b", "sdf", "tc"): 2.84e-5, ("b", "rgb", "tc"): 2.25e-6, ("b", "nrm", "tc"): 3.70e-5,
    ("a", "rgb1", "tc"): 3.36e-4, ("b", "rgb1", "tc"): 3.36e-4,
}
MEASURED = {}
COUNTS = {}
TIES = dict(ties=0, samples=0)           # tie-margin samples and all samples compared in this session


@pytest.fixture(scope="module", autouse=True)
def _print_measured():
    yield
    for k in sorted(MEASURED):
        print("MEASURED %s/%s/%s %.3g (gate %.3g)" % (k + (MEASURED[k], GATE[k])))
    for k in sorted(COUNTS):
        print("COUNT %s %s" % (k, COUNTS[k]))


def _note_count(key, **kw):
    COUNTS[key] = kw
    print("%s: %s" % (key, kw))


# ---------------------------------------------------------------------------------------------
# renders
# ---------------------------------------------------------------------------------------------

def _L():
    from multiply_b200 import _lib as L
    return L


def _sm_count():
    return int(_L().call("mp_device_sm_count"))


def _render(sc, inp, hits, eng, mode="parity", train=None, r=None):
    """(Renderer, debug outputs) of one render under engine ``eng`` and precision ``mode``."""
    engine.set_engine(eng)
    engine.set_precision(mode)
    try:
        r = engine.Renderer(sc) if r is None else r
        o = r.render(inp, hits, debug=True, train=train)
        torch.cuda.synchronize()
    finally:
        engine.set_precision("parity")
    return r, o


def _taps(o, P):
    return {f"{k}_{p}": o[f"{k}_{p}"].clone() for p in range(P) for k in ("z_vals", "sdf", "rgb", "normals")}


def _bench_scene(weights):
    sc = S.make_scene(P=2, S=BENCH_S, seed=42, weights=weights)
    inp = S.make_rays(sc, BENCH_RAYS, seed=1234, region="boxes")
    return sc, inp, S.make_hit_lists(sc, inp)


def _points(inp, hits, o, k, n):
    """The main pass's points of rendered person k: x = cam + z d with two separately rounded fp32 ops, as
    deform_rays_kernel forms them (deform.cu: __fadd_rn(cam, __fmul_rn(z, d)))."""
    from multiply_b200.model import rend_util
    dirs, cam = rend_util.camera_rays(inp["uv"].cuda(), inp["pose"], inp["intrinsics"])
    h = engine.hit_list(hits[k], "cuda")
    z = o[f"z_vals_{k}"][:, :n]
    zd = z[..., None] * dirs[h][:, None]
    return (cam[h][:, None] + zd).reshape(-1, 3)


# ---------------------------------------------------------------------------------------------
# float64 references
# ---------------------------------------------------------------------------------------------

def _p64(person):
    d = lambda t: torch.as_tensor(t).double().to(DEV)
    return dict(implicit={k: d(v) for k, v in person["implicit"].items()},
                render={k: d(v) for k, v in person["render"].items()}, cond=d(person["cond"]).reshape(1, -1),
                verts_p=d(person["verts_p"]).reshape(-1, 3), verts_c=d(person["verts_c"]).reshape(-1, 3),
                weights=d(person["weights"]).reshape(-1, 24), tfs=d(person["tfs"]).reshape(24, 4, 4))


def _nearest2(pts, verts, chunk=2048):
    """fp64 squared distances and indices of the nearest and second-nearest vertex: d2 = (dx^2 + dy^2) + dz^2."""
    out = [[], [], [], []]
    for s in range(0, pts.shape[0], chunk):
        p = pts[s:s + chunk]
        d = (p[:, None, 0] - verts[None, :, 0]) ** 2
        d += (p[:, None, 1] - verts[None, :, 1]) ** 2
        d += (p[:, None, 2] - verts[None, :, 2]) ** 2
        v, i = torch.topk(d, 2, dim=1, largest=False, sorted=True)
        for o, t in zip(out, (v[:, 0], i[:, 0], v[:, 1], i[:, 1])):
            o.append(t)
    if pts.shape[0] == 0:
        e = torch.zeros(0, dtype=torch.float64, device=pts.device)
        return e, e.long(), e, e.long()
    return tuple(torch.cat(o) for o in out)


def _inverse_skin(P64, x, vi):
    """deformer.py:19-30 with the weights of vertex vi (K = 1: conf = 1): x_c = (sum_j w_j tfs_j)^-1 [x; 1]."""
    return port.skinning(x[None], P64["weights"][vi][None], P64["tfs"][None], inverse=True)[0]


def _jinv(P64, vi):
    """Inverse of the forward-skinning Jacobian (multiply.py:640-650) with the weights of canonical vertex vi."""
    A = torch.einsum("pn,nij->pij", P64["weights"][vi], P64["tfs"])[:, :3, :3]
    return torch.linalg.inv(A)


def _shade64(P64, xc, Jinv, chunk=32768):
    """fp64 sdf, rgb, normal and the normal's condition |g J^-1| / ||J^-1||_2 at x_c; for the ill-conditioned ones also
    the rgb sensitivity max_k sum_j |d rgb_k / d n_j| (0 elsewhere)."""
    res = {k: [] for k in ("sdf", "rgb", "nrm", "cond", "sens")}
    for s in range(0, xc.shape[0], chunk):
        xs = xc[s:s + chunk].detach().clone().requires_grad_(True)
        J = Jinv[s:s + chunk]
        y = port.implicit_forward(P64["implicit"], xs, P64["cond"], 6)
        g = torch.autograd.grad(y[:, 0].sum(), xs)[0]
        with torch.no_grad():
            v = torch.einsum("bi,bij->bj", g, J)
            n = F.normalize(F.normalize(v, dim=1), dim=-1, eps=1e-6)
            feat = y[:, 1:].detach()
            rgb = port.rendering_forward(P64["render"], "pose_no_view", xs.detach(), n, None, P64["cond"], feat)
            cond = v.norm(dim=1) / torch.linalg.matrix_norm(J, ord=2)
        sens = torch.zeros_like(cond)
        ill = cond < COND_SMALL
        if bool(ill.any()):
            nl = n[ill].clone().requires_grad_(True)
            c = port.rendering_forward(P64["render"], "pose_no_view", xs.detach()[ill], nl, None, P64["cond"], feat[ill])
            rows = [torch.autograd.grad(c[:, k].sum(), nl, retain_graph=k < 2)[0].abs().sum(1) for k in range(3)]
            sens[ill] = torch.stack(rows, 1).max(1)[0]
        for k, t in zip(res, (y[:, 0].detach(), rgb, n, cond, sens)):
            res[k].append(t)
    if xc.shape[0] == 0:
        z = torch.zeros(0, dtype=torch.float64, device=DEV)
        return dict(sdf=z, rgb=z.reshape(0, 3), nrm=z.reshape(0, 3), cond=z, sens=z)
    return {k: torch.cat(v) for k, v in res.items()}


def _errors(sdf, rgb, nrm, ref):
    """Per-sample error of each class against one fp64 evaluation (see the module docstring)."""
    dn = (nrm.double() - ref["nrm"]).abs().max(1)[0]
    drgb = (rgb.double() - ref["rgb"]).abs().max(1)[0]
    ill = ref["cond"] < COND_SMALL
    return dict(sdf=(sdf.double() - ref["sdf"]).abs(), rgb=torch.where(ill, (drgb - ref["sens"] * dn).clamp(min=0), drgb),
                nrm=dn * ref["cond"], dn=dn, drgb=drgb, ill=ill, cond=ref["cond"])


def _ref_a(P64, x, listed, xc32):
    """Reference (a) at the fp32 points x of one person: dict(outlier, tie_outlier, tie, and the fp64 x_c / J^-1 of every
    nearest-vertex candidate as (rows, x_c, J^-1)).  Candidates: the nearest posed vertex, plus the second one where
    fp32 rounding of the squared distance (relative TIE_REL) can reorder them; for each resulting x_c the nearest
    canonical vertex, plus the second where the gap is within TIE_REL or within what the distance of the deformer's
    fp32 x_c (xc32) from the fp64 one can bridge.  A tie counts where it can change what
    the shade program wrote: the outlier flag of any sample, the vertices of the listed ones."""
    x64 = x.double()
    d1, i1, d2, i2 = _nearest2(x64, P64["verts_p"])
    tie_p = ((d2 - d1) <= TIE_REL * d1) & listed
    dist = d1.clamp(max=4.0).sqrt()
    tie_o = (dist - 0.1).abs() <= TIE_REL * 0.1
    tie = tie_p | tie_o
    tie_c_any = torch.zeros_like(tie)
    cands = []
    for pv, rows in ((i1, listed.nonzero()[:, 0]), (i2, tie_p.nonzero()[:, 0])):
        xc = _inverse_skin(P64, x64[rows], pv[rows])
        c1, j1, c2, j2 = _nearest2(xc, P64["verts_c"])
        # the gap |x - v2|^2 - |x - v1|^2 is linear in x: moving x by delta moves it by at most 2 delta |v1 - v2|
        delta = 1.25 * (xc32[rows].double() - xc).norm(dim=1) + 1e-8
        sep = (P64["verts_c"][j1] - P64["verts_c"][j2]).norm(dim=1)
        tie_c = (c2 - c1) <= TIE_REL * c1 + 2 * delta * sep
        tie_c_any[rows[tie_c]] = True
        tr = tie_c.nonzero()[:, 0]
        cands += [(rows, xc, _jinv(P64, j1)), (rows[tr], xc[tr], _jinv(P64, j2[tr]))]
    kinds = dict(posed=int(tie_p.sum()), outlier=int(tie_o.sum()), canonical=int(tie_c_any.sum()))
    return dict(outlier=dist > 0.1, tie_outlier=tie_o, tie=tie | tie_c_any, kinds=kinds, cands=cands)


def _compare_a(P64, ra, sdf, rgb, nrm, listed, sdf_rows):
    """Per-sample errors of reference (a): the minimum over the nearest-vertex candidates of each sample.  listed: the
    samples whose rgb / normal the shade program wrote; sdf_rows: those whose sdf it wrote."""
    N = listed.shape[0]
    inf = torch.full((N,), float("inf"), dtype=torch.float64, device=DEV)
    best = {k: inf.clone() for k in ("sdf", "rgb", "nrm", "dn", "drgb")}
    cond = torch.ones(N, dtype=torch.float64, device=DEV)
    ill = torch.zeros(N, dtype=torch.bool, device=DEV)
    for rows, xc, J in ra["cands"]:
        if rows.numel() == 0:
            continue
        e = _errors(sdf[rows], rgb[rows], nrm[rows], _shade64(P64, xc, J))
        first = bool(torch.isinf(best["sdf"][rows]).all())
        for k in best:
            best[k][rows] = torch.minimum(best[k][rows], e[k])
        if first:
            cond[rows], ill[rows] = e["cond"], e["ill"]
    best["sdf"] = torch.where(sdf_rows, best["sdf"], torch.zeros_like(best["sdf"]))
    for k in best:
        best[k] = torch.where(listed, best[k], torch.zeros_like(best[k]))
    best.update(cond=cond, ill=ill & listed)
    return best


def _epilogue(g, J):
    """normalize(normalize(g . J^-1), eps=1e-6) in fp64 from the fp32 operands, and the amplification
    |(|g| |J^-1|)| / |g J^-1| of their rounding."""
    g, J = g.double(), J.double().reshape(-1, 3, 3)
    v = torch.einsum("bi,bij->bj", g, J)
    amp = torch.einsum("bi,bij->bj", g.abs(), J.abs()).norm(dim=1) / v.norm(dim=1).clamp(min=1e-300)
    return F.normalize(F.normalize(v, dim=1), dim=-1, eps=1e-6), amp


# ---------------------------------------------------------------------------------------------
# one person's checks
# ---------------------------------------------------------------------------------------------

def _check_person(tag, eng, r, p, k, person, inp, hits, o, pruned, train=False, rgb_class="rgb", mode="parity",
                  strict=True):
    """Every check of rendered person k (scene person p, fp64 parameters ``person``) of a render under engine ``eng``
    and precision ``mode``; returns the worst error of each (reference, class).  strict=False (a mode outside the
    gates): the bit-identities only, no gate, nothing recorded as MEASURED."""
    n = r.n
    x = _points(inp, hits, o, k, n)
    N = x.shape[0]
    sdf, rgb, nrm = o[f"sdf_{k}"].reshape(N), o[f"rgb_{k}"].reshape(N, 3), o[f"normals_{k}"].reshape(N, 3)
    body, field = r.bodies[p], r.fields[p]
    # ---- reference (b): the renderer's own deformer, forward Jacobian and operators -------------------------------
    xc32, outl = body.deform_inverse(x, exact_far=not pruned)
    listed = ~outl if pruned else torch.ones_like(outl)
    sdf_rows = listed if train else listed & ~outl
    if not train:    # sdf 4 where the deformer flags an outlier (pruned: in the deformer; else after the shade launch)
        assert bool((sdf[outl] == 4.0).all()), tag
    if pruned:       # pruned samples: rgb / normals left at the memset's +0.0
        z3 = torch.zeros_like(rgb[outl])
        assert same(rgb[outl], z3) and same(nrm[outl], z3), tag
    # sigmoid > 0: every listed sample was written, the last row of a ragged tile and of a SIMT chunk included
    miss = ~(rgb[listed] > 0).all(1)
    assert not bool(miss.any()), "%s: %d listed samples the shade program did not write" % (tag, int(miss.sum()))
    L_ = listed.nonzero()[:, 0]
    if L_.numel() == 0:      # nothing shaded (a device count of 0): the taps above and the flags are all there is
        ra = _ref_a(person, x, listed, xc32)
        assert not bool(((outl != ra["outlier"]) & ~ra["tie_outlier"]).any()), tag
        return {}
    engine.set_engine(eng)
    engine.set_precision(mode)
    try:
        _, Jl = body.forward_jac(xc32[L_])
        op_sdf, _, op_grad = field.implicit_forward(xc32[L_], want_feat=False, want_grad=True)
        torch.cuda.synchronize()
    finally:
        engine.set_precision("parity")
    # sdf: the fused program and mp_implicit_forward_grad run the same steps L0..L7 on independent rows: bit-identical
    srows = sdf_rows[L_]
    bad = sdf[L_][srows].view(torch.int32) != op_sdf[srows].view(torch.int32)
    assert not bool(bad.any()), "%s: %d sdf taps differ from mp_implicit_forward_grad at the deformer's x_c" % (
        tag, int(bad.sum()))
    # normals: the epilogue evaluated in fp64 from the operator's fp32 grad and forward_jac's J^-1.  Within a few ulp,
    # not bitwise: both engines' kernels are built with FMA contraction, so their fp32 dot products g . J^-1 and sums
    # of squares round differently from any sequence of torch ops; the bound scales with the cancellation in g . J^-1
    n_epi, amp = _epilogue(op_grad, Jl)
    ulp = ((nrm[L_].double() - n_epi).abs().max(1)[0] / (2.0 ** -24 * (1 + amp))).max().item() if L_.numel() else 0.0
    assert ulp <= 16, "%s: normal taps %.1f ulp from the epilogue of mp_implicit_forward_grad's grad" % (tag, ulp)
    eb = _errors(sdf[L_], rgb[L_], nrm[L_], _shade64(person, xc32[L_].double(), Jl.double().reshape(-1, 3, 3)))
    eb["sdf"] = torch.where(srows, eb["sdf"], torch.zeros_like(eb["sdf"]))
    # ---- reference (a): from z alone --------------------------------------------------------------------------------
    ra = _ref_a(person, x, listed, xc32)
    disagree = (outl != ra["outlier"]) & ~ra["tie_outlier"]
    assert not bool(disagree.any()), "%s: %d outlier flags differ from fp64" % (tag, int(disagree.sum()))
    ea = _compare_a(person, ra, sdf, rgb, nrm, listed, sdf_rows)
    ties = int(ra["tie"].sum())
    _note_count("%s p%d" % (tag, k), samples=N, shaded=int(listed.sum()), tie_margin=ties, tie_kinds=ra["kinds"],
                ill_normals=int(ea["ill"].sum()),
                ill_cond=["%.2e" % v for v in ea["cond"][ea["ill"]].sort()[0][:8].tolist()],
                epilogue_ulp="%.2f" % ulp)
    TIES["ties"] += ties
    TIES["samples"] += N
    worst = {}
    for ref, e in (("a", ea), ("b", eb)):
        for cls in ("sdf", "rgb", "nrm"):
            worst[(ref, rgb_class if cls == "rgb" else cls, eng)] = float(e[cls].max()) if e[cls].numel() else 0.0
    print("%s p%d worst: %s" % (tag, k, {"%s/%s" % kk[:2]: "%.2e" % vv for kk, vv in worst.items()}))
    if not strict:
        return worst
    for key, v in worst.items():
        MEASURED[key] = max(MEASURED.get(key, 0.0), v)
    # north star on (a), every sample: ill-conditioned normals by their scaled measure, their rgb net of the normal's
    for name, v in (("sdf", ea["sdf"]), ("rgb", torch.where(ea["ill"], ea["rgb"], ea["drgb"])),
                    ("nrm", torch.where(ea["ill"], ea["nrm"], ea["dn"]))):
        w = float(v.max()) if v.numel() else 0.0
        assert w < TOL_GATE, "%s: reference (a) %s %.3g at sample %d" % (tag, name, w, int(v.argmax()) if v.numel() else -1)
    for key, v in worst.items():
        assert v <= GATE[key], "%s: %s %.3g over the gate %.3g" % (tag, key, v, GATE[key])
        if key[0] == "b" and key[1] != "rgb1":
            assert v <= 2 * (2 if key[1] == "nrm" else 1) * TOL_NET[eng], (tag, key, v)
    return worst


def _check_render(tag, eng, sc, inp, hits, o, r, pruned, train=False, **kw):
    persons = [_p64(p) for p in sc["persons"]]
    return [_check_person(tag, eng, r, p, p, persons[p], inp, hits, o, pruned, train, **kw) for p in range(len(hits))]


# ---------------------------------------------------------------------------------------------
# the benchmark's case
# ---------------------------------------------------------------------------------------------

_BENCH = {}


def _bench(eng, weights):
    if (eng, weights) not in _BENCH:
        sc, inp, hits = _bench_scene(weights)
        r, o = _render(sc, inp, hits, eng)
        _BENCH[(eng, weights)] = (sc, inp, hits, r, _taps(o, 2))
    return _BENCH[(eng, weights)]


@pytest.mark.parametrize("weights", ["trained", "geometric"])
@pytest.mark.parametrize("eng", ENGINES)
def test_bench_case(eng, weights):
    """bench.py's workload: P = 2, 4096 'boxes' rays, S/E/X = 128/256/64, beta_param 0.1 (outliers pruned).  The work
    list runs to ~1e5-1e6 points: many tiles per persistent CTA, a ragged last tile whose length only the device
    knows, SIMT chunk seams on a device-side count.  Bit-identities against the operators at the deformer's x_c, then
    references (b) and (a)."""
    sc, inp, hits, r, o = _bench(eng, weights)
    _check_render("bench/%s/%s" % (eng, weights), eng, sc, inp, hits, o, r, pruned=True)


def test_bench_case_colour1():
    """'colour1' (single-term colour layers, tensor cores): sdf and normals bit-identical to 'parity' (the colour layers
    follow them), rgb per sample under its own gate."""
    sc, inp, hits, r, par = _bench("tc", "trained")
    _, o = _render(sc, inp, hits, "tc", mode="colour1", r=r)
    for p in range(2):
        for k in ("z_vals", "sdf", "normals"):
            assert same(o[f"{k}_{p}"], par[f"{k}_{p}"]), (p, k)
    _check_render("bench/tc/colour1", "tc", sc, inp, hits, o, r, pruned=True, rgb_class="rgb1", mode="colour1")




def test_throughput_exceeds_gates():
    """The same comparison under 'throughput' (one fp16 term in every layer) exceeds the parity gates on sdf, for both
    references: the gates tell a wrong chain from a right one.  (The bit-identities against the operators hold in
    every mode.)"""
    sc, inp, hits, r, _ = _bench("tc", "trained")
    _, o = _render(sc, inp, hits, "tc", mode="throughput", r=r)
    w = _check_render("bench/tc/throughput", "tc", sc, inp, hits, o, r, pruned=True, mode="throughput", strict=False)
    for ref in ("a", "b"):
        v = max(ww[(ref, "sdf", "tc")] for ww in w)
        print("throughput: reference (%s) sdf %.3g, parity gate %.3g" % (ref, v, GATE[(ref, "sdf", "tc")]))
        assert v > GATE[(ref, "sdf", "tc")], ref


# ---------------------------------------------------------------------------------------------
# exact caps: every sample shaded, work lists of chosen lengths
# ---------------------------------------------------------------------------------------------

def _cap_targets(T):
    """(name, base, offset): list lengths at the last-tile, persistent-grid and SIMT-chunk (32768) edges."""
    return [("1", 0, 1), ("127", 128, -1), ("128", 128, 0), ("129", 128, 1), ("128T-1", 128 * T, -1),
            ("128T", 128 * T, 0), ("128T+1", 128 * T, 1), ("32767", 32768, -1), ("32768", 32768, 0),
            ("32769", 32768, 1), ("65537", 65536, 1)]


def _cap_layout(base, offset, max_rows, n_lo=2, n_hi=260):
    """(R_p, S, X, E) with R_p * (S + X + 1) = base + offset, or the nearest length on the same side of ``base``
    (offset 0: exactly base) that factorises with n = S + X + 1 in [n_lo, n_hi] and R_p <= max_rows."""
    tgt = base + offset
    for d in range(0, 64):
        for v in (tgt + d, tgt - d) if offset else (tgt,):
            if v < 1 or (offset > 0 and v <= base) or (offset < 0 and v >= base):
                continue
            for n in range(n_hi, n_lo - 1, -1):
                if v % n == 0 and v // n <= max_rows:
                    X = (n - 1) // 3
                    S_ = n - 1 - X
                    return v // n, S_, X, max(S_, 2)
    raise AssertionError("no layout for %d" % tgt)


_CAP = {}


def _cap_scene():
    if "sc" not in _CAP:
        sc = S.make_scene(P=2, S=16, seed=42, beta=0.3, weights="trained")
        inp = S.make_rays(sc, 2048, seed=21, region="boxes")
        _CAP["sc"] = (sc, inp, S.make_hit_lists(sc, inp))
    return _CAP["sc"]


def _cap_case(name, T):
    """The beta_param 0.3 scene (beta = 0.3001 >= 0.23: prune_is_exact is false, every sample is shaded, so each
    person's shade launch has count == cap == R_p * n) with its sampler sized for the target list length."""
    sc, inp, hits0 = _cap_scene()
    base, offset = {t[0]: t[1:] for t in _cap_targets(T)}[name]
    R = inp["uv"].shape[1]
    Rp, S_, X, E = _cap_layout(base, offset, R)
    cfg = dict(sc["cfg"], N_samples=S_, N_samples_extra=X, N_samples_eval=E)
    sc2 = dict(sc, cfg=cfg)
    hits = []
    for h in hits0:         # the person's box rays first, then the others, R_p of them in ray order
        rest = torch.from_numpy(np.setdiff1d(np.arange(R), h.numpy()))
        hits.append(torch.cat([h, rest])[:Rp].sort()[0])
    return sc2, inp, hits, Rp * (S_ + X + 1), (Rp, S_, X, E)


@pytest.mark.parametrize("target", [t[0] for t in _cap_targets(1)])
@pytest.mark.parametrize("eng", ENGINES)
def test_exact_cap(eng, target):
    """Work lists of exactly 1 (or 2), 127, 128, 129, 128 T - 1, 128 T, 128 T + 1 (T = SMs), 32767, 32768, 32769 and
    65537 points (or the nearest length on the same side of the edge): a last tile of 1 or 127 rows, one tile per CTA
    plus or minus a row, SIMT chunk seams.  Outliers are shaded too: sdf 4, rgb / normals at the exact-nearest x_c."""
    T = _sm_count()
    sc, inp, hits, cap, lay = _cap_case(target, T)
    print("exact cap %s: R_p * n = %d (R_p, S, X, E = %s)" % (target, cap, lay))
    COUNTS["cap %s/%s" % (target, eng)] = dict(achieved=cap, layout=lay)
    r, o = _render(sc, inp, hits, eng)
    assert r.n * hits[0].numel() == cap
    _check_render("cap%s/%s" % (target, eng), eng, sc, inp, hits, o, r, pruned=False)


# ---------------------------------------------------------------------------------------------
# count 0, eight persons, training mode
# ---------------------------------------------------------------------------------------------

def _solo(sc, p):
    """Person p alone, the body and networks unchanged (the slice parallel.py renders), no background."""
    return dict(sc, persons=[sc["persons"][p]], bg_implicit=None, bg_render=None)


@pytest.mark.parametrize("eng", ENGINES)
def test_count_zero(eng):
    """Person 1's rays all pass more than 0.15 from its posed vertices: every sample is an outlier, its shade launch
    runs on a device count of 0, and its taps are sdf = 4, rgb = normals = 0 exactly.  Person 0's taps are bit-identical
    to a render of person 0 alone, and within the gates."""
    from multiply_b200.model import rend_util
    sc = S.make_scene(P=2, S=64, seed=42, weights="trained")
    inp = S.make_rays(sc, 1024, seed=9, region="boxes")
    hits = S.make_hit_lists(sc, inp)
    dirs, cam = rend_util.get_camera_params_host(inp["uv"], inp["pose"], inp["intrinsics"])
    v = torch.as_tensor(sc["persons"][1]["verts_p"]).double()
    d, c = dirs.double(), cam.double()
    far = []
    for i in range(d.shape[0]):      # distance of the ray's line to every vertex
        w = v - c[i]
        t = (w @ d[i]) / (d[i] @ d[i])
        far.append(bool(((w - t[:, None] * d[i]).norm(dim=1) > 0.15).all()))
    miss = torch.tensor(far).nonzero()[:, 0]
    assert miss.numel() >= 64
    hits[1] = miss[:256].to(torch.int64)
    r, o = _render(sc, inp, hits, eng)
    assert bool((o["sdf_1"] == 4.0).all())
    assert same(o["rgb_1"], torch.zeros_like(o["rgb_1"])) and same(o["normals_1"], torch.zeros_like(o["normals_1"]))
    _, solo = _render(_solo(sc, 0), inp, hits[:1], eng)
    for k in ("z_vals", "sdf", "rgb", "normals"):
        assert same(o[f"{k}_0"], solo[f"{k}_0"]), k
    _check_person("count0/%s" % eng, eng, r, 0, 0, _p64(sc["persons"][0]), inp, hits, o, pruned=True)


@pytest.mark.parametrize("eng", ENGINES)
def test_eight_persons(eng):
    """P = MP_MAX_PERSONS = 8, 512 rays, person 7 reduced to the substituted ray 0 (an empty hit list): per-branch
    workspaces and streams.  Each person's taps are bit-identical to a render of that person alone."""
    sc = S.make_scene(P=8, S=32, seed=42, weights="trained")
    inp = S.make_rays(sc, 512, seed=13, region="boxes")
    hits = S.make_hit_lists(sc, inp)
    hits[7] = torch.zeros(0, dtype=torch.int64)
    r, o = _render(sc, inp, hits, eng)
    assert o["sdf_7"].shape[0] == 1
    for p in range(8):
        _, solo = _render(_solo(sc, p), inp, [hits[p]], eng)
        for k in ("z_vals", "sdf", "rgb", "normals"):
            assert same(o[f"{k}_{p}"], solo[f"{k}_0"]), (p, k)
    _check_person("P8/%s p7" % eng, eng, r, 7, 7, _p64(sc["persons"][7]), inp, hits, o, pruned=True)


@pytest.mark.parametrize("eng", ENGINES)
def test_training(eng):
    """Training mode with recorded draws (P = 2, 1024 rays): prune = 0 and no outlier clamp, so every sample is listed
    and compared, outliers at their un-clamped sdf."""
    from multiply_b200.model.ray_sampler import ErrorBoundSampler
    sc = S.make_scene(P=2, S=64, seed=42, weights="trained")
    inp = S.make_rays(sc, 1024, seed=5, region="boxes")
    hits = S.make_hit_lists(sc, inp)
    smp = ErrorBoundSampler(3.0, inverse_sphere_bg=True, **{k: sc["cfg"][k] for k in (
        "near", "N_samples", "N_samples_eval", "N_samples_extra", "eps", "beta_iters", "max_total_iters", "add_tiny")})
    torch.manual_seed(0)
    rngs = [smp.draw_training_rng(h.numel()) for h in hits]
    rngs = [{k: v for k, v in d.items() if k != "states"} for d in rngs]
    r, o = _render(sc, inp, hits, eng, train=dict(rng=rngs, t_rand_bg=None))
    _check_render("train/%s" % eng, eng, sc, inp, hits, o, r, pruned=False, train=True)


# ---------------------------------------------------------------------------------------------
# invariances (bitwise)
# ---------------------------------------------------------------------------------------------

@pytest.mark.parametrize("eng", ENGINES)
def test_rerun_invariance(eng):
    """Two renders of the benchmark case give bit-identical taps.  The warp-aggregated atomicAdd that builds the pruned
    work list (deform.cu, deform_rays_kernel) may place a sample in another tile and row on the second run, so this
    checks that the shade program's rows are independent of their list position -- but only as far as the atomic
    ordering actually changed between the runs: the list order is not observable through the ABI, so a pass cannot
    prove that a reorder happened."""
    sc, inp, hits, r, first = _bench(eng, "trained")
    _, o = _render(sc, inp, hits, eng, r=r)
    for k, v in first.items():
        assert same(o[k], v), k


@pytest.mark.parametrize("eng", ENGINES)
def test_streams_invariance(eng):
    """mp_set_streams(0) (one stream) and (1) (a stream per person) give bit-identical taps."""
    sc, inp, hits, r, _ = _bench(eng, "trained")
    L = _L()
    out = {}
    try:
        for on in (0, 1):
            L.call("mp_set_streams", on)
            out[on] = _taps(_render(sc, inp, hits, eng, r=r)[1], 2)
    finally:
        L.call("mp_set_streams", int(os.environ.get("MP_RENDER_STREAMS", "1") != "0"))
    for k, v in out[0].items():
        assert same(out[1][k], v), k


def _grid_sweep(path):
    """The taps of the benchmark case and of the 128 T + 1 exact cap, tensor-core engine, written to ``path`` (npz).
    Run in this process and in subprocesses with MP_TC_GRID."""
    res = {}
    sc, inp, hits = _bench_scene("trained")
    _, o = _render(sc, inp, hits, "tc")
    res.update({"bench_" + k: v.cpu().numpy() for k, v in _taps(o, 2).items()})
    sc, inp, hits, _, _ = _cap_case("128T+1", _sm_count())
    _, o = _render(sc, inp, hits, "tc")
    res.update({"cap_" + k: v.cpu().numpy() for k, v in _taps(o, 2).items()})
    np.savez(path, **res)


@pytest.mark.parametrize("grid", [1, 3])
def test_grid_invariance(tmp_path, grid):
    """MP_TC_GRID (read once per process) caps the persistent CTAs of the shade launch: with 1 or 3 CTAs each runs
    hundreds of tiles.  The taps must be bit-identical to the default grid's."""
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
        assert np.array_equal(a[k].view(np.uint32), b[k].view(np.uint32)), "%s: %d values differ with MP_TC_GRID=%d" % (
            k, int((a[k] != b[k]).sum()), grid)


def test_tie_margin_share():
    """Tie-margin samples (the only samples reference (a) does not pin to one nearest-vertex choice) stay under 0.1 % of
    all samples compared above.  Most come from the cases that shade every sample, outliers metres from the body
    included: far from the body many vertices are nearly equidistant.  Runs last; needs the benchmark cases' samples."""
    if TIES["samples"] < 10 ** 6:
        pytest.skip("needs test_bench_case's samples in the same session")
    share = TIES["ties"] / TIES["samples"]
    print("tie-margin samples: %d of %d (%.4f %%)" % (TIES["ties"], TIES["samples"], 100 * share))
    assert share < TIE_FRAC


if __name__ == "__main__":
    if len(sys.argv) == 3 and sys.argv[1] == "--grid-sweep":
        _grid_sweep(sys.argv[2])
