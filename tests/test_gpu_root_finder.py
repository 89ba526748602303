"""GPU: the optional Broyden root finder (mp_deform_broyden, mp_body_set_root_finder and the ROOT = true deform kernels)
against a float64 restatement of the same algorithm (tests/_broyden_ref.py), step by step, and on every path the switch
turns on.

- Each step: for max_steps 1, 2 and 3 the restatement starts from the GPU's own closed-form start (bit-equal to
  mp_deform_inverse) and applies x_{k+1} = x_k - J_k^-1 g_k, forward skinning with the nearest canonical vertex of each
  iterate and the rank-one update of J^-1.  The runs with max_steps 0..K expose the GPU's best iterate after every step,
  so the best-iterate rule is checked exactly: where the float64 residuals clearly order, the GPU moved to the new
  iterate or kept the old one bit for bit.
- Whole runs (max_steps 10 and 64, N from 0 to 1.6 M): converged == residual < thr, steps < max_steps only when
  converged, steps == 0 exactly when the closed-form residual is < thr (and then x_c is the closed form), residual never
  above the closed form's, residual == float64 |forward_skinning(x_c) - x|, reruns bit-identical, finite outputs.
- Threshold and geometry edges, non-finite and overflowing inputs (no nearest vertex: the rules of DESIGN §3.2), every
  switched path (mp_deform_inverse, mp_sdf_with_deformer, the main pass of mp_render_rays) bit for bit, rejections.

Gates are per element, err <= C * 2^-24 * M with M the float64 sum of |terms| behind the element (_broyden_ref.py);
C is 4x the worst measured on one H100 (printed as MEASURED).  A nearest-vertex choice fp32 cannot resolve is never
masked: both vertices are evaluated and either is accepted; such points are counted and their share capped."""
import itertools
import math
import os
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from multiply_b200 import engine, scene as S          # noqa: E402

import _broyden_ref as R                              # noqa: E402
from _abi import padded, same, take                   # noqa: E402
from _setups import dirty_workspace, points, posed_body  # noqa: E402

EPS = R.EPS
THR = 1e-5                   # the mirror's default threshold
THR_MIN = 2.0 ** -126        # below every nonzero residual: every step is taken
# 4x the worst measured on one H100 80GB HBM3 at a 700 W power limit: 1.95 (every step, max_steps 1-3), 2.15 (residual
# of whole runs, at 1.6 M points)
C_GATE = dict(step=7.8, resid=8.6)
TIE_FRAC = 0.05              # points with a tie-margin lookup, of one step test's points (measured 0.06 %, 0.3 %, 3.2 %)
RESID_TIE_FRAC = 0.02        # of the points of one whole run whose residual check accepts either vertex (measured
                             # 0.58 % at 1.6 M points, 1 of 129 at N = 129)
BOUNDARY_TIE_FRAC = 0.5      # the same for points built to start on canonical Voronoi boundaries (measured 40 %)
MEASURED = {}
TIES = dict(ties=0, points=0)
RTIES = dict(ties=0, points=0)


@pytest.fixture(scope="module", autouse=True)
def _print_measured():
    yield
    for k in sorted(MEASURED):
        print("MEASURED %s C=%.3g (gate %.3g)" % (k, MEASURED[k], C_GATE[k]))
    print("TIES %d of %d points (steps), %d of %d points (whole-run residuals)" % (
        TIES["ties"], TIES["points"], RTIES["ties"], RTIES["points"]))


def _note(key, c):
    MEASURED[key] = max(MEASURED.get(key, 0.0), float(c))


def _L():
    from multiply_b200 import _lib as L
    return L


def _c(err, M):
    """err / (2^-24 M) per element; 0 / 0 = 0, err / 0 = inf."""
    err = err.abs()
    return torch.where(M > 0, err / (EPS * torch.where(M > 0, M, torch.ones_like(M))),
                       torch.where(err == 0, torch.zeros_like(err), torch.full_like(err, math.inf)))


def _broyden(b, x, K, thr):
    """mp_deform_broyden into sentinel-padded buffers: dict(x_c, residual, converged, outlier, steps) on the GPU."""
    N = x.shape[0]
    o = dict(x_c=padded((N, 3)), residual=padded(N), converged=padded(N, torch.uint8), outlier=padded(N, torch.uint8),
             steps=padded(N, torch.int32))
    _L().call("mp_deform_broyden", b.handle, x, N, int(K), float(thr), o["x_c"], o["residual"], o["converged"],
              o["outlier"], o["steps"])
    torch.cuda.synchronize()
    shapes = dict(x_c=(N, 3), residual=N, converged=N, outlier=N, steps=N)
    return {k: take(o[k], shapes[k], k).cuda() for k in o}


def _fresh_body():
    """A body of posed_body()'s data that never had the root finder switched on."""
    b, _ = posed_body()
    f = engine.Body(b.verts_c, b.weights, cano_cell=0.1001)
    f.set_pose(b.verts_p, b.tfs)
    return f


_B64 = {}


def _b64():
    if "b" not in _B64:
        _B64["b"] = R.Body64(posed_body()[0])
    return _B64["b"]


def _pts(N, seed, **kw):
    b, _ = posed_body()
    return points(N, b.verts_p, seed, **kw).cuda()


# ---------------------------------------------------------------------------------------------
# each step against float64
# ---------------------------------------------------------------------------------------------

@pytest.mark.parametrize("K", [1, 2, 3])
def test_steps_against_float64(K):
    """max_steps K: every step's iterate and residual, and the best-iterate choice after every step."""
    b, _ = posed_body()
    B = _b64()
    x = _pts(20000, seed=40 + K, far_frac=0.2)
    runs = [_broyden(b, x, j, THR_MIN) for j in range(K + 1)]
    xc0, _ = b.deform_inverse(x, exact_far=True)
    assert same(runs[0]["x_c"], xc0), "the closed-form start differs from mp_deform_inverse"
    nz = runs[0]["residual"] > 0
    for j in range(1, K + 1):   # a step is taken exactly while the best residual so far is nonzero
        go = runs[j - 1]["residual"] > 0
        assert same(runs[j]["steps"], torch.where(go, torch.full_like(runs[j]["steps"], j), runs[j - 1]["steps"])), j
    p, x0 = x.double(), runs[0]["x_c"].double()
    # the GPU's switches: after step j it holds iterate j exactly when its x_c changed
    sw = [None] + [(runs[j]["x_c"] != runs[j - 1]["x_c"]).any(1) for j in range(1, K + 1)]
    for j in range(1, K + 1):   # x_c and residual move together: a switch means rn < best
        assert same(sw[j], runs[j]["residual"] != runs[j - 1]["residual"]), "x_c and residual did not move together"
    best = torch.full((x.shape[0],), math.inf, dtype=torch.float64, device="cuda")
    tie_any = torch.zeros(x.shape[0], dtype=torch.bool, device="cuda")
    for combo in itertools.product((0, 1), repeat=K + 1):
        ch = torch.tensor(combo, device="cuda").expand(x.shape[0], K + 1)
        ref = R.run(B, p, x0, K, THR_MIN, ch)
        tie_any |= ref["tie"]
        idx = torch.zeros(x.shape[0], dtype=torch.long, device="cuda")
        c = torch.zeros(x.shape[0], dtype=torch.float64, device="cuda")
        ar = torch.arange(x.shape[0], device="cuda")
        for j in range(K + 1):
            if j:
                rb, mrb = ref["r"][idx, ar], ref["mr"][idx, ar]
                rj, mrj = ref["r"][j], ref["mr"][j]
                m = C_GATE["step"] * EPS * (mrb + mrj)
                better, worse = rj < rb - m, rj > rb + m
                bad = (better & ~sw[j]) | (worse & sw[j])
                c = torch.where(bad & nz, torch.full_like(c, math.inf), c)
                idx = torch.where(sw[j], torch.full_like(idx, j), idx)
            xr, mx = ref["x"][idx, ar], ref["mx"][idx, ar]
            cx = _c(runs[j]["x_c"].double() - xr, mx).max(1)[0]
            cr = _c(runs[j]["residual"].double() - ref["r"][idx, ar], ref["mr"][idx, ar])
            c = torch.maximum(c, torch.maximum(cx, cr))
        best = torch.minimum(best, c)
    ties = int(tie_any.sum())
    TIES["ties"] += ties
    TIES["points"] += x.shape[0]
    worst = float(best.max())
    _note("step", worst)
    print("steps K=%d: worst C %.3g, %d tie-margin points of %d" % (K, worst, ties, x.shape[0]))
    if worst > C_GATE["step"]:
        i = int(best.argmax())
        ref = R.run(B, p[i:i + 1], x0[i:i + 1], K, THR_MIN)
        print("point %d: x %s, GPU x_c %s, residuals %s, switches %s; float64 iterates %s, residuals %s (M %s), tie %s" % (
            i, x[i].tolist(), [o["x_c"][i].tolist() for o in runs], [float(o["residual"][i]) for o in runs],
            [bool(s[i]) for s in sw[1:]], ref["x"][:, 0].tolist(), ref["r"][:, 0].tolist(), ref["mr"][:, 0].tolist(),
            bool(ref["tie"][0])))
    assert worst <= C_GATE["step"], "K=%d: point %d off by C=%.3g" % (K, int(best.argmax()), worst)
    assert ties <= TIE_FRAC * x.shape[0], (ties, x.shape[0])


# ---------------------------------------------------------------------------------------------
# whole runs
# ---------------------------------------------------------------------------------------------

def _resid_c(b, x, xc, res):
    """(C, tie-margin points) of the reported residual against float64 |forward_skinning(x_c) - x|, either vertex where
    fp32 cannot resolve the nearest one."""
    B = _b64()
    worst, ties = 0.0, 0
    for s in range(0, x.shape[0], 1 << 18):
        p, xcd = x[s:s + (1 << 18)].double(), xc[s:s + (1 << 18)].double()
        cs = []
        for choice in (0, 1):
            vi, tie = R.lookup(B, xcd, torch.zeros_like(xcd), torch.full((p.shape[0],), choice, device="cuda"))
            r64, mr = R.residual(B, p, xcd, vi)
            cs.append(_c(res[s:s + (1 << 18)].double() - r64, mr))
        worst = max(worst, float(torch.minimum(*cs).max()))
        ties += int(tie.sum())
    return worst, ties


def _invariants(b, x, K, thr, tie_frac=RESID_TIE_FRAC):
    """Every whole-run invariant of one call on finite points; returns (outputs, number of points the no-vertex rule
    ended).  tie_frac caps the share of points whose residual check accepts either of two vertices."""
    o = _broyden(b, x, K, thr)
    o2 = _broyden(b, x, K, thr)
    for k in o:
        assert same(o[k], o2[k]), "rerun differs: %s" % k
    N = x.shape[0]
    if N == 0:
        return o, 0
    c0 = _broyden(b, x, 0, thr)
    xc0, out0 = b.deform_inverse(x, exact_far=True)
    assert same(c0["x_c"], xc0) and same(o["outlier"], out0.to(torch.uint8))
    res, steps, conv = o["residual"], o["steps"], o["converged"].bool()
    assert same(conv, res < thr), "converged != residual < thr"
    assert bool(((steps >= 0) & (steps <= K)).all())
    ended = (steps < K) & ~conv          # only the no-vertex rule ends an iteration early without convergence
    zero = steps == 0
    assert same(zero & ~ended, c0["residual"] < thr), "steps == 0 differs from closed-form residual < thr"
    assert same(o["x_c"][zero], xc0[zero]) and same(res[zero & ~ended], c0["residual"][zero & ~ended])
    assert bool((res <= c0["residual"]).all()), "a residual above the closed form's"
    # an iteration can only return an iterate it skinned, so finite points give finite outputs whatever path they took
    assert bool(torch.isfinite(o["x_c"]).all() and torch.isfinite(res).all()), "non-finite output"
    c, ties = _resid_c(b, x, o["x_c"], res)
    _note("resid", c)
    RTIES["ties"] += ties
    RTIES["points"] += N
    print("residual check: C %.3g, %d tie-margin points of %d" % (c, ties, N))
    assert c <= C_GATE["resid"], c
    assert ties <= tie_frac * N, (ties, N)
    return o, int(ended.sum())


@pytest.mark.parametrize("N", [0, 1, 127, 128, 129, 1600000])
@pytest.mark.parametrize("K", [10, 64])
def test_whole_run_invariants(K, N):
    b, _ = posed_body()
    if N == 0:      # null pointers throughout; a real output buffer stays untouched
        _L().call("mp_deform_broyden", b.handle, None, 0, K, THR, None, None, None, None, None)
        xc = padded((0, 3))
        _L().call("mp_deform_broyden", b.handle, None, 0, K, THR, xc, None, None, None, None)
        torch.cuda.synchronize()
        take(xc, (0, 3), "x_c")
        return
    x = _pts(N, seed=N + K)
    o, ended = _invariants(b, x, K, THR)
    print("N=%d K=%d: %d converged, %d refined, %d ended by the no-vertex rule" % (
        N, K, int(o["converged"].sum()), int((o["steps"] > 0).sum()), ended))
    assert ended == 0


# ---------------------------------------------------------------------------------------------
# threshold edges
# ---------------------------------------------------------------------------------------------

def test_threshold_edges():
    b, _ = posed_body()
    x = _pts(50000, seed=11)
    # below every residual: every point takes max_steps unless its residual is exactly 0
    for K in (3, 10):
        o, _ = _invariants(b, x, K, THR_MIN)
        assert bool(((o["steps"] == K) | (o["residual"] == 0)).all())
    # above every residual: nothing moves
    o = _broyden(b, x, 10, 1e30)
    xc0, _ = b.deform_inverse(x, exact_far=True)
    assert bool((o["steps"] == 0).all()) and same(o["x_c"], xc0) and bool(o["converged"].all())
    # equal to a point's exact closed-form residual: the loop tests best >= thr, so that point iterates
    c0 = _broyden(b, x, 0, THR)
    r0 = c0["residual"]
    cand = ((r0 > 1e-4) & (r0 < 1e-2)).nonzero()[:, 0][:8]
    assert cand.numel() == 8
    for i in cand.tolist():
        t = float(r0[i])
        o, _ = _invariants(b, x, 10, t)
        assert int(o["steps"][i]) >= 1, "a point at residual == thr did not iterate"
        assert bool(o["converged"][i]) == bool(o["residual"][i] < t)


def test_fold_exact():
    """A two-vertex body whose forward map folds: translations only, so every quantity is a small dyadic rational and the
    fp32 iteration is exact.  The start (0.75, 0, 0) maps to 1.75, iterate 1 (-0.25) to -1.25: equal residuals 1, so the
    best iterate stays the start; then J^-1 = 0.5 and iterate 2 (0.25) has residual 0.5."""
    vc = torch.tensor([[0.0, 0.0, 0.0], [1.0, 0.0, 0.0]], device="cuda")
    W = torch.zeros(2, 24, device="cuda")
    W[0, 0] = W[1, 1] = 1.0
    tfs = torch.eye(4, device="cuda").repeat(24, 1, 1)
    tfs[1, 0, 3] = 1.0
    vp = vc + torch.tensor([[0.0, 0.0, 0.0], [1.0, 0.0, 0.0]], device="cuda")
    b = engine.Body(vc, W, cano_cell=0.1001)
    b.set_pose(vp, tfs)
    x = torch.tensor([[0.75, 0.0, 0.0]], device="cuda")
    o = _broyden(b, x, 0, THR)
    assert o["x_c"].tolist() == [[0.75, 0.0, 0.0]] and float(o["residual"]) == 1.0
    o = _broyden(b, x, 1, THR)
    assert o["x_c"].tolist() == [[0.75, 0.0, 0.0]] and float(o["residual"]) == 1.0 and int(o["steps"]) == 1
    o = _broyden(b, x, 2, THR)
    assert o["x_c"].tolist() == [[0.25, 0.0, 0.0]] and float(o["residual"]) == 0.5 and int(o["steps"]) == 2
    # thr == the closed-form residual 1.0 exactly: iterates; converged only below it
    o = _broyden(b, x, 2, 1.0)
    assert int(o["steps"]) == 2 and bool(o["converged"]) and float(o["residual"]) == 0.5
    o = _broyden(b, x, 1, 1.0)
    assert int(o["steps"]) == 1 and not bool(o["converged"])


# ---------------------------------------------------------------------------------------------
# geometry edges
# ---------------------------------------------------------------------------------------------

def _d2_f32(p, v):
    """The kernel's squared distance, (dx*dx + dy*dy) + dz*dz with every operation rounded to fp32."""
    d = (p[:, None, :] - v[None, :, :]).float()
    return (d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]) + d[..., 2] * d[..., 2]


def test_geometry_edges():
    b, _ = posed_body()
    B = _b64()
    vp = b.verts_p
    rng = np.random.RandomState(3)
    # points on posed vertices
    on = vp[torch.from_numpy(rng.randint(0, vp.shape[0], 4000)).cuda()].contiguous()
    _invariants(b, on, 10, THR)
    # midpoints of posed vertex pairs: exact fp32 ties must resolve to the lower index
    i = torch.from_numpy(rng.randint(0, vp.shape[0], 4000)).cuda()
    d = _d2_f32(vp[i], vp).float()
    d[torch.arange(i.numel()), i] = math.inf
    j = d.argmin(1)
    mid = ((vp[i] + vp[j]) * 0.5).contiguous()
    _invariants(b, mid, 10, THR)
    dm = _d2_f32(mid, vp)
    lo, hi = torch.minimum(i, j), torch.maximum(i, j)
    ar = torch.arange(i.numel(), device="cuda")
    tie = (dm[ar, lo] == dm[ar, hi]) & (dm[ar, lo] == dm.min(1)[0])
    xc0, _ = b.deform_inverse(mid, exact_far=True)
    t = tie.nonzero()[:, 0]
    p = mid[t].double()
    x_lo = torch.einsum("nij,nj->ni", B.Mi[lo[t]], p - _tau(b, lo[t]))
    x_hi = torch.einsum("nij,nj->ni", B.Mi[hi[t]], p - _tau(b, hi[t]))
    dist = (x_lo - x_hi).norm(dim=1) > 1e-4      # ties whose two closed forms tell the vertices apart
    print("exact posed ties among %d midpoints: %d, %d with distinct closed forms" % (
        i.numel(), t.numel(), int(dist.sum())))
    assert int(dist.sum()) >= 10, "too few exact posed ties to check the lowest-index rule"
    e_lo = (xc0[t].double() - x_lo).norm(dim=1)
    assert bool((e_lo[dist] < 1e-5).all()), "a posed tie did not take the lowest index"
    # canonical Voronoi boundaries: forward-skin midpoints of canonical neighbours, so starts and iterates land on them
    vc = b.verts_c
    i = torch.from_numpy(rng.randint(0, vc.shape[0], 4000)).cuda()
    dc = _d2_f32(vc[i], vc).float()
    dc[torch.arange(i.numel()), i] = math.inf
    j = dc.argmin(1)
    mc = ((vc[i] + vc[j]) * 0.5).double()
    A = B.A[i]
    xd = (torch.einsum("nij,nj->ni", A[:, :, :3], mc) + A[:, :, 3]).float().contiguous()
    _invariants(b, xd, 10, THR, tie_frac=BOUNDARY_TIE_FRAC)
    # points 1-5 units from the body: outliers, which mp_deform_broyden refines (the ROOT paths do not)
    for dist_ in (1.0, 2.5, 5.0):
        xf = _pts(4000, seed=int(dist_ * 10), far_frac=1.0, far=-dist_)
        o, ended = _invariants(b, xf, 10, THR)
        moved = (o["x_c"] != b.deform_inverse(xf, exact_far=True)[0]).any(1) & o["outlier"].bool()
        print("far %.1f: %d outliers, %d of them refined, %d ended by the no-vertex rule" % (
            dist_, int(o["outlier"].sum()), int(moved.sum()), ended))
        assert bool(moved.any()), "mp_deform_broyden did not refine any outlier"
        assert ended == 0


def _tau(b, vi):
    """t / s of vertex vi's blended transform in float64 (the inverse's translation)."""
    W, tfs = b.weights.double()[vi], b.tfs.double().reshape(24, 4, 4)
    A = torch.einsum("vn,nij->vij", W, tfs)
    return A[:, :3, 3] / A[:, 3, 3:4]


# ---------------------------------------------------------------------------------------------
# no nearest vertex: non-finite and overflowing inputs
# ---------------------------------------------------------------------------------------------

BAD = [[float("nan"), 0.0, 0.0], [0.0, 0.0, float("inf")], [-float("inf"), 1.0, 1.0], [1e20, 0.0, 0.0],
       [0.0, -1e20, 0.0], [1e20, 1e20, 1e20], [float("nan")] * 3]


def _mixed(N, seed):
    """N normal points with the BAD rows at spread positions: (mixed batch, bad positions, the batch without them)."""
    x = _pts(N, seed)
    pos = torch.linspace(0, N + len(BAD) - 1, len(BAD)).long().cuda()
    keep = torch.ones(N + len(BAD), dtype=torch.bool, device="cuda")
    keep[pos] = False
    m = torch.empty(N + len(BAD), 3, device="cuda")
    m[keep] = x
    m[pos] = torch.tensor(BAD, device="cuda")
    return m.contiguous(), keep, x


def test_no_vertex_broyden():
    b, _ = posed_body()
    m, keep, x = _mixed(3000, 21)
    for K in (1, 10, 64):
        o = _broyden(b, m, K, THR)
        ref = _broyden(b, x, K, THR)
        for k in o:
            assert same(o[k][keep], ref[k]), (K, k)
        bad = ~keep
        assert same(o["x_c"][bad], m[bad]), "a point without a vertex must keep x_c = x"
        assert bool(torch.isnan(o["residual"][bad]).all() and (o["steps"][bad] == 0).all())
        assert not bool(o["converged"][bad].any()) and bool(o["outlier"][bad].all())
    # the switched paths: those points are outliers and keep x_c = x
    f = _fresh_body()
    f.set_root_finder(10, THR)
    xc, out = f.deform_inverse(m, exact_far=True)
    ref, _ = f.deform_inverse(x, exact_far=True)
    assert same(xc[keep], ref) and same(xc[~keep], m[~keep]) and bool(out[~keep].all())


def _overflow_body():
    """Three canonical vertices, one bone each: c0 = 0 (identity), c1 = (0.1, 0, 0) (x scaled by s = 2^-70, translated by
    (0.08, 5, 0)), c2 = (0.08, -5, 0) (translated by (1, 2.5, 0)).  J^-1 at c1 is diag(2^70, 1, 1), so any x residual
    there sends the next iterate beyond 2^64, where every fp32 squared distance overflows."""
    s = 2.0 ** -70
    vc = torch.tensor([[0.0, 0.0, 0.0], [0.1, 0.0, 0.0], [0.08, -5.0, 0.0]], device="cuda")
    W = torch.zeros(3, 24, device="cuda")
    W[0, 0] = W[1, 1] = W[2, 2] = 1.0
    tfs = torch.eye(4, device="cuda").repeat(24, 1, 1)
    tfs[1, 0, 0], tfs[1, 0, 3], tfs[1, 1, 3] = s, 0.08, 5.0
    tfs[2, 0, 3], tfs[2, 1, 3] = 1.0, 2.5
    vp = torch.einsum("vij,vj->vi", tfs[:3, :3, :3], vc) + tfs[:3, :3, 3]
    b = engine.Body(vc, W, cano_cell=0.1001)
    b.set_pose(vp.contiguous(), tfs)
    return b


def test_no_vertex_iterate_ends_iteration():
    """An iterate without a nearest vertex ends that point's iteration: the best iterate so far and its residual come
    back, steps counts the steps taken.  Both points start at x (nearest posed vertex c0, within 0.1: not outliers) in
    c1's canonical cell.
    - (0.055, 0, 0): residual (0.025, 5, 0); step 1 moves x by -0.025 * 2^70 and has no vertex: x_c = x, steps 1.
    - (0.08, 0, 0): residual (0, 5, 0); step 1 lands on c2 with a smaller residual (1, -2.5, 0); after the rank-one
      update step 2 moves x by about -2^70 * 2/3 and has no vertex: x_c = iterate 1 = (0.08, -5, 0), steps 2."""
    b = _overflow_body()
    x = torch.tensor([[0.055, 0.0, 0.0], [0.08, 0.0, 0.0]], device="cuda")
    c0 = _broyden(b, x, 0, THR)
    assert same(c0["x_c"], x) and not bool(c0["outlier"].any())
    assert abs(float(c0["residual"][0]) - math.hypot(0.025, 5.0)) < 1e-5 and float(c0["residual"][1]) == 5.0
    o1 = _broyden(b, x, 1, THR)
    x1 = torch.tensor([0.08, -5.0, 0.0], device="cuda")
    assert o1["steps"].tolist() == [1, 1]
    assert same(o1["x_c"][0], x[0]) and same(o1["residual"][0], c0["residual"][0])
    assert same(o1["x_c"][1], x1) and float(o1["residual"][1]) < float(c0["residual"][1])
    assert abs(float(o1["residual"][1]) - math.hypot(1.0, 2.5)) < 1e-5
    for K in (2, 10, 64):
        o = _broyden(b, x, K, THR)
        assert o["steps"].tolist() == [1, 2], (K, o["steps"].tolist())
        assert same(o["x_c"], o1["x_c"]) and same(o["residual"], o1["residual"]), K
        assert not bool(o["converged"].any())
    # the ROOT path stops the same way
    b.set_root_finder(10, THR)
    xc, out = b.deform_inverse(x, exact_far=True)
    assert same(xc, o1["x_c"]) and not bool(out.any())
    b.set_root_finder(0)
    # the overflowing iterates themselves: no vertex, so forward_jac writes NaN
    xd, J = b.forward_jac(torch.tensor([[0.055 - 0.025 * 2.0 ** 70, 0.0, 0.0]], device="cuda"))
    assert bool(torch.isnan(xd).all() and torch.isnan(J).all())


def test_no_vertex_forward_jac():
    b, _ = posed_body()
    m, keep, x = _mixed(3000, 22)
    xc, _ = b.deform_inverse(x, exact_far=True)
    mc = torch.empty_like(m)
    mc[keep] = xc
    mc[~keep] = m[~keep]
    xd, J = b.forward_jac(mc)
    xd0, J0 = b.forward_jac(xc)
    assert same(xd[keep], xd0) and same(J[keep], J0)
    assert bool(torch.isnan(xd[~keep]).all() and torch.isnan(J[~keep]).all())
    # the backward: NaN d_x_c, nothing to d_tfs (the reference batch carries a good point with zero cotangents there)
    rng = np.random.RandomState(4)
    u = torch.from_numpy(rng.randn(m.shape[0], 3).astype(np.float32)).cuda()
    uj = torch.from_numpy(rng.randn(m.shape[0], 9).astype(np.float32)).cuda()
    dxc, dtfs = b.forward_jac_backward(mc, u, uj)
    rc = mc.clone()
    rc[~keep] = xc[0]
    ru, ruj = u.clone(), uj.clone()
    ru[~keep] = 0.0
    ruj[~keep] = 0.0
    dxc0, dtfs0 = b.forward_jac_backward(rc, ru, ruj)
    assert same(dxc[keep], dxc0[keep]) and same(dtfs, dtfs0)
    assert bool(torch.isnan(dxc[~keep]).all())
    # appended after the batch: d_tfs and d_x_c bit-identical to the batch without them
    n = xc.shape[0]
    app = torch.cat([xc, m[~keep]]).contiguous()
    dxa, dta = b.forward_jac_backward(app, u[:app.shape[0]].contiguous(), uj[:app.shape[0]].contiguous())
    dx1, dt1 = b.forward_jac_backward(xc, u[:n].contiguous(), uj[:n].contiguous())
    assert same(dta, dt1) and same(dxa[:n], dx1) and bool(torch.isnan(dxa[n:]).all())
    # with only d_x_d, only d_Jinv
    for a, bb in ((u, None), (None, uj)):
        if a is None:
            a = torch.zeros_like(u)
        d1, t1 = b.forward_jac_backward(mc, a, bb)
        ra = a.clone()
        ra[~keep] = 0.0
        rb = None if bb is None else ruj
        d2, t2 = b.forward_jac_backward(rc, ra, rb)
        assert same(t1, t2) and same(d1[keep], d2[keep])


# ---------------------------------------------------------------------------------------------
# every switched path
# ---------------------------------------------------------------------------------------------

@pytest.mark.parametrize("K", [3, 10])
def test_switched_inverse_and_sdf(K):
    from multiply_b200 import _lib as L
    engine.set_engine("tc")
    sc = S.make_scene(P=2, S=16, seed=42, weights="trained")
    p = sc["persons"][0]
    f = engine.Field(p["implicit"], p["render"])
    f.set_cond(p["cond"])
    b = engine.Body(p["verts_c"], p["weights"], cano_cell=0.1001 / p["scale"])
    b.set_pose(p["verts_p"], p["tfs"])
    x = points(20000, b.verts_p, 17, far_frac=0.2).cuda()
    plain = {e: b.deform_inverse(x, exact_far=e) for e in (False, True)}
    br = _broyden(b, x, K, THR)
    b.set_root_finder(K, THR)
    try:
        for e in (False, True):
            xc, out = b.deform_inverse(x, exact_far=e)
            assert same(out, plain[e][1])
            assert same(xc[~out], br["x_c"][~out]), "non-outliers differ from mp_deform_broyden (exact_far %d)" % e
            assert same(xc[out], plain[e][0][out]), "outliers left the closed form (exact_far %d)" % e
        N = x.shape[0]
        sdf, xcs = torch.empty(N, device="cuda"), torch.empty(N, 3, device="cuda")
        ws = dirty_workspace(L.call("mp_sdf_with_deformer_workspace_bytes", N))
        L.call("mp_sdf_with_deformer", b.handle, f.handle, x, N, sdf, xcs, None, ws, ws.numel())
        xc, out = b.deform_inverse(x, exact_far=True)
        assert same(xcs, xc)
        op, _ = f.implicit_forward(xc, want_feat=False)
        torch.cuda.synchronize()
        assert same(sdf[~out], op[~out]) and bool((sdf[out] == 4.0).all())
    finally:
        b.set_root_finder(0)
    for e in (False, True):
        xc, out = b.deform_inverse(x, exact_far=e)
        assert same(xc, plain[e][0]) and same(out, plain[e][1])


def test_switch_off_restores_default():
    x = _pts(20000, seed=23)
    f, g = _fresh_body(), _fresh_body()
    f.set_root_finder(10, THR)
    f.deform_inverse(x)
    f.set_root_finder(0)
    for e in (False, True):
        a, b_ = f.deform_inverse(x, exact_far=e), g.deform_inverse(x, exact_far=e)
        assert same(a[0], b_[0]) and same(a[1], b_[1])
    assert same(f.forward_jac(x)[1], g.forward_jac(x)[1])


def _main_points(inp, hits, o, k, n):
    """The main pass's points of person k: x = cam + z d with two separately rounded fp32 ops (deform_rays_kernel)."""
    from multiply_b200.model import rend_util
    dirs, cam = rend_util.camera_rays(inp["uv"].cuda(), inp["pose"], inp["intrinsics"])
    h = engine.hit_list(hits[k], "cuda")
    z = o[f"z_vals_{k}"][:, :n]
    return (cam[h][:, None] + z[..., None] * dirs[h][:, None]).reshape(-1, 3)


def _epilogue_ulp(nrm, g, J):
    """ulp distance of the normal taps from normalize(normalize(g . J^-1), eps=1e-6) in float64, scaled by the
    amplification of the dot product's rounding (test_gpu_shade.py's bound)."""
    import torch.nn.functional as F
    g, J = g.double(), J.double().reshape(-1, 3, 3)
    v = torch.einsum("bi,bij->bj", g, J)
    amp = torch.einsum("bi,bij->bj", g.abs(), J.abs()).norm(dim=1) / v.norm(dim=1).clamp(min=1e-300)
    n = F.normalize(F.normalize(v, dim=1), dim=-1, eps=1e-6)
    return float(((nrm.double() - n).abs().max(1)[0] / (EPS * (1 + amp))).max()) if n.numel() else 0.0


@pytest.mark.parametrize("train", [False, True])
@pytest.mark.parametrize("eng", ["simt", "tc"])
def test_switched_render_main_pass(eng, train):
    """mp_render_rays with every body's root finder on: the main pass's sdf taps are mp_implicit_forward_grad at the
    Broyden x_c bit for bit (the closed form at outliers), its normals the epilogue with forward_jac's J^-1 there."""
    from multiply_b200.model.ray_sampler import ErrorBoundSampler
    engine.set_engine(eng)
    sc = S.make_scene(P=2, S=16, seed=42, weights="trained")
    inp = S.make_rays(sc, 256, seed=9, region="boxes")
    hits = S.make_hit_lists(sc, inp)
    r = engine.Renderer(sc)
    for b in r.bodies:
        b.set_root_finder(10, THR)
    tr = None
    if train:
        smp = ErrorBoundSampler(3.0, inverse_sphere_bg=True, **{k: sc["cfg"][k] for k in (
            "near", "N_samples", "N_samples_eval", "N_samples_extra", "eps", "beta_iters", "max_total_iters",
            "add_tiny")})
        torch.manual_seed(0)
        rngs = [smp.draw_training_rng(h.numel()) for h in hits]
        tr = dict(rng=[{k: v for k, v in d.items() if k != "states"} for d in rngs], t_rand_bg=None)
    o = r.render(inp, hits, debug=True, train=tr)
    torch.cuda.synchronize()
    pruned = not train       # beta 0.1: eval prunes outliers exactly, training lists every sample
    for k in range(len(hits)):
        body, field = r.bodies[k], r.fields[k]
        x = _main_points(inp, hits, o, k, r.n)
        N = x.shape[0]
        sdf, nrm = o[f"sdf_{k}"].reshape(N), o[f"normals_{k}"].reshape(N, 3)
        xc, out = body.deform_inverse(x, exact_far=not pruned)
        br = _broyden(body, x, 10, THR)
        assert same(xc[~out], br["x_c"][~out]), "main-pass x_c differs from mp_deform_broyden"
        listed = ~out if pruned else torch.ones_like(out)
        L_ = listed.nonzero()[:, 0]
        # some shaded samples sit at a refined x_c, not at the closed form
        refined = (xc[L_] != _broyden(body, x, 0, THR)["x_c"][L_]).any(1)
        assert int(refined.sum()) > 0, "no shaded sample was refined"
        _, J = body.forward_jac(xc[L_])
        op, _, grad = field.implicit_forward(xc[L_], want_feat=False, want_grad=True)
        torch.cuda.synchronize()
        rows = listed[L_] if train else ~out[L_]
        assert same(sdf[L_][rows], op[rows]), "%s/%s p%d: sdf taps differ at the Broyden x_c" % (eng, train, k)
        if not train:
            assert bool((sdf[out] == 4.0).all())
        ulp = _epilogue_ulp(nrm[L_], grad, J)
        print("%s train=%s p%d: %d samples, %d refined listed, normal taps %.2f ulp" % (
            eng, train, k, N, int(refined.sum()), ulp))
        assert ulp <= 16, ulp


# ---------------------------------------------------------------------------------------------
# rejections
# ---------------------------------------------------------------------------------------------

@pytest.mark.parametrize("K,thr", [(-1, THR), (65, THR), (10, 0.0), (10, -1.0), (10, float("nan"))])
def test_rejections(K, thr):
    L = _L()
    b = _fresh_body()
    x = _pts(300, seed=2)
    N = x.shape[0]
    o = [padded((N, 3)), padded(N), padded(N, torch.uint8), padded(N, torch.uint8), padded(N, torch.int32)]
    with pytest.raises(L.MpError):
        L.call("mp_deform_broyden", b.handle, x, N, K, thr, *o)
    torch.cuda.synchronize()
    for buf, s in zip(o, ((0, 3), 0, 0, 0, 0)):
        take(buf, s, "output")      # nothing written: the whole buffer still holds the sentinel
    with pytest.raises(L.MpError):
        L.call("mp_body_set_root_finder", b.handle, K, thr)
    xc, out = b.deform_inverse(x)
    g = _fresh_body()
    assert same(xc, g.deform_inverse(x)[0])     # the rejected switch left the body as it was
