"""GPU: the backward of the compositing stages (csrc/composite.cu: mp_composite_backward, mp_final_compose_backward;
csrc/background.cu: mp_bg_composite_backward), the background taps of mp_render_rays, and the differentiable training
forward of the mirror (Multiply.set_render_grad), against float64 autograd of oracle/render_grad.py.

Gate.  Every gradient is compared per ray with a bound c * 2^-24 * (sum of |terms| of the ray), where the terms are those
the kernel adds: for d(sigma delta)_k they are |g_j| over the ray's samples plus |bg_T dbg_T| (T, w <= 1), scaled by the
local factor |delta_k dsigma/dsdf_k| for d sdf; for d rgb / d normal the upstream |d fg| resp. |d normal| of the ray; for
d_beta the same over all samples with |delta_k dsigma/dbeta_k|.  Transmittances and local factors below 2^-102 count
as 2^-102 (an absolute floor of c * 2^-126: fp32 goes subnormal there).

Measured on one H100 80GB HBM3 at a 400 W power limit: worst c = 76.7 (the mirror at P = 3), 53.8 for
mp_composite_backward alone (P = 5, n = 193, beta = 0.1), 7.6 on the tie case, 2.1 for the background; the reversed tie
order is off by c = 5.3e6.  C_MEASURED is the worst c over all cases of this file
(printed as "c=" by each test); the gate is C_GATE = 4 * C_MEASURED."""
import os
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
for p in (ROOT, HERE):
    if p not in sys.path:
        sys.path.insert(0, p)

from oracle import render_grad as RG                            # noqa: E402
from _abi import SENTINEL, padded, take                         # noqa: E402
from _setups import make_inputs, mirror_inputs, person_samples, wpc_of  # noqa: E402

EPS = 2.0 ** -24
TINY = 2.0 ** -102
C_MEASURED = 77.0
C_GATE = 4 * C_MEASURED
WORST = {}


def _g(t):
    """.grad as numpy, zeros where autograd left it None (no path to the loss)."""
    return t.grad.numpy() if t.grad is not None else np.zeros(tuple(t.shape))


def _note(what, c):
    WORST["all"] = max(WORST.get("all", 0.0), c)
    print("c=%.3g %s (worst so far %.3g)" % (c, what, WORST["all"]))


# ---------------------------------------------------------------------------------------------
# reference: float64 autograd of the restatement
# ---------------------------------------------------------------------------------------------

def _ups(seed, R, P, null=()):
    rng = np.random.RandomState(seed)
    u = dict(d_fg=rng.randn(R, 3), d_nrm=rng.randn(R, 3), d_acc=rng.randn(R), d_accp=rng.randn(R, P), d_bgT=rng.randn(R))
    u = {k: v.astype(np.float32) for k, v in u.items()}
    for k in null:
        u[k] = None
    return u


def gate_scales(persons, R, n, beta, ups, bgT):
    """Per person: M [R_p,1] = sum over the ray's samples of |g_k| plus |bg_T dbg_T| (the terms of d(sigma delta)),
    ds / db = |delta dsigma/dsdf| / |delta dsigma/dbeta| per sample, and the ray's max |d fg| / |d normal|."""
    P = len(persons)
    z = lambda k, shp: np.zeros(shp) if ups[k] is None else np.asarray(ups[k], np.float64)   # noqa: E731
    dfg, dn, dacc, daccp, dbgT = z("d_fg", (R, 3)), z("d_nrm", (R, 3)), z("d_acc", R), z("d_accp", (R, P)), z("d_bgT", R)
    # values below 2^-102 count as 2^-102: the kernels' fp32 transmittances and exponentials go subnormal there, so the
    # bound keeps an absolute floor of c * 2^-126 times the local factors
    M = np.abs(dbgT) * np.maximum(np.asarray(bgT, np.float64), TINY)
    out = []
    for p, d in enumerate(persons):
        g = np.abs(np.einsum("rc,rnc->rn", dfg[d["idx"]], d["rgb"].astype(np.float64))) + \
            np.abs(np.einsum("rc,rnc->rn", dn[d["idx"]], d["nrm"].astype(np.float64))) + \
            np.abs(dacc[d["idx"]] + daccp[d["idx"], p])[:, None]
        np.add.at(M, d["idx"], g.sum(1))
        s = d["sdf"].astype(np.float64)
        delta = d["z"][:, 1:].astype(np.float64) - d["z"][:, :-1]
        e = np.exp(-np.abs(s) / beta)
        sig = (1 / beta) * (0.5 + 0.5 * np.sign(s) * np.expm1(-np.abs(s) / beta))
        out.append(dict(ds=np.abs(delta) * np.maximum(e / (2 * beta * beta), TINY),
                        db=np.abs(delta) * np.maximum(np.abs(sig) / beta + np.abs(s) * e / (2 * beta ** 3), TINY),
                        dfg=np.abs(dfg[d["idx"]]).max(1)[:, None, None] + 1e-30,
                        dn=np.abs(dn[d["idx"]]).max(1)[:, None, None] + 1e-30))
    for p, d in enumerate(persons):
        out[p]["M"] = M[d["idx"]][:, None]
    return out


def ref_backward(persons, R, n, beta, ups, reverse=False):
    """fp64 gradients of sum(outputs * upstream) and the gate scales."""
    b = torch.tensor(float(np.float32(beta)), dtype=torch.float64, requires_grad=True)
    tp = [dict(idx=d["idx"], z=torch.from_numpy(d["z"]).double(),
               **{k: torch.from_numpy(d[k]).double().requires_grad_(True) for k in ("sdf", "rgb", "nrm")})
          for d in persons]
    outs = RG.composite(tp, R, n, b, reverse=reverse)
    loss = 0
    for o, k in zip(outs, ("d_fg", "d_nrm", "d_acc", "d_accp", "d_bgT")):
        if ups[k] is not None:
            loss = loss + (o * torch.from_numpy(ups[k]).double()).sum()
    loss.backward()
    grads = [dict(sdf=_g(t["sdf"]), rgb=_g(t["rgb"]), nrm=_g(t["nrm"])) for t in tp]
    return grads, float(b.grad), gate_scales(persons, R, n, float(b.detach()), ups, outs[4].detach().numpy())


def worst_c(persons, got, want, wbeta, got_beta, sc):
    """max over every gradient of |got - want| / (2^-24 * scale)."""
    worst, db_scale = 0.0, abs(wbeta)
    for p, d in enumerate(persons):
        if d["idx"].size == 0:
            continue
        s = sc[p]
        c_sdf = np.abs(got[p]["sdf"] - want[p]["sdf"]) / (EPS * (s["ds"] * s["M"] + np.abs(want[p]["sdf"])) + 1e-300)
        c_rgb = np.abs(got[p]["rgb"] - want[p]["rgb"]) / (EPS * s["dfg"])
        c_nrm = np.abs(got[p]["nrm"] - want[p]["nrm"]) / (EPS * s["dn"])
        worst = max(worst, float(c_sdf.max()), float(c_rgb.max()), float(c_nrm.max()))
        db_scale += float((s["db"] * s["M"]).sum())
    return max(worst, abs(got_beta - wbeta) / (EPS * db_scale + 1e-300))


# ---------------------------------------------------------------------------------------------
# the C ABI with sentinel-padded gradient buffers
# ---------------------------------------------------------------------------------------------

def grad_outputs(persons, n):
    """Per person padded d sdf / d rgb / d normal buffers, and d_beta."""
    return [dict(sdf=padded((d["idx"].size, n)), rgb=padded((d["idx"].size, n, 3)), nrm=padded((d["idx"].size, n, 3)))
            for d in persons], padded(1)


def call_backward(persons, R, n, beta, ups, P_arg=None, ws_delta=0, null_grad=None, out=None):
    """(gradient buffers, d_beta) as ``grad_outputs`` makes them (or ``out``), after the call."""
    from multiply_b200 import _lib as L
    P = len(persons)
    arr, keep = person_samples(persons)
    bufs, d_beta = grad_outputs(persons, n) if out is None else out
    gr = (L.PersonSampleGrads * P)()
    for p, b in enumerate(bufs):
        gr[p].d_sdf, gr[p].d_rgb, gr[p].d_normal = (L.ptr(b[k]) for k in ("sdf", "rgb", "nrm"))
        if null_grad == p:
            gr[p].d_rgb = None
    up = {k: (torch.from_numpy(v).cuda() if v is not None else None) for k, v in ups.items()}
    ws_bytes = L.call("mp_composite_backward_workspace_bytes", R, P) + ws_delta
    ws = L.workspace(ws_bytes, "cuda")
    L.call("mp_composite_backward", arr, P if P_arg is None else P_arg, R, n, float(beta), up["d_fg"], up["d_nrm"],
           up["d_acc"], up["d_accp"], up["d_bgT"], gr, d_beta, ws, ws_bytes)
    torch.cuda.synchronize()
    return bufs, d_beta


def check_against(persons, R, n, beta, ups, bufs, d_beta, reverse=False, assert_ok=True, tag=""):
    """Worst c of (sdf, rgb, normal, beta) against the fp64 reference (optionally the reversed tie order)."""
    want, wbeta, sc = ref_backward(persons, R, n, beta, ups, reverse=reverse)
    got = [{k: take(bufs[p][k], shp, "%s p%d" % (k, p)).numpy() for k, shp in
            (("sdf", (d["idx"].size, n)), ("rgb", (d["idx"].size, n, 3)), ("nrm", (d["idx"].size, n, 3)))}
           for p, d in enumerate(persons)]
    worst = worst_c(persons, got, want, wbeta, float(take(d_beta, 1, "d_beta")[0]), sc)
    if assert_ok:
        _note(tag or "composite_backward", worst)
        assert worst < C_GATE, (worst, tag)
    return worst


# (P, n, beta): P = 1..8, n = 1, 31, 32, 33, 97, 193, both betas
CASES = [(1, 1, 0.1), (1, 97, 1e-4), (2, 31, 0.1), (2, 193, 1e-4), (3, 33, 0.1), (3, 1, 1e-4), (4, 32, 1e-4),
         (4, 97, 0.1), (5, 193, 0.1), (5, 33, 1e-4), (6, 31, 1e-4), (6, 97, 0.1), (7, 32, 0.1), (7, 193, 1e-4),
         (8, 1, 0.1), (8, 33, 1e-4), (8, 193, 0.1)]
NULLS = [(), ("d_nrm",), ("d_acc", "d_bgT"), ("d_fg", "d_accp"), ("d_fg", "d_nrm", "d_acc", "d_accp")]


@pytest.mark.parametrize("P,n,beta", CASES, ids=["P%d-n%d-b%g" % c for c in CASES])
def test_composite_backward_vs_fp64(P, n, beta):
    """Every gradient against fp64 autograd at R = 1 and around the rays-per-block edge, with persons missing rays
    (rays with K = 0), zero-length intervals, sdf == 0, T underflow at beta = 1e-4, identical z rows of two persons,
    and random or partly NULL upstream gradients; nothing is written outside [R_p, n]; a rerun is bit-identical."""
    wpc = wpc_of(P, n)
    for j, R in enumerate(sorted({1, max(1, wpc - 1), wpc, wpc + 1, 2 * wpc + 1})):
        persons = make_inputs(77 * P + n + R, P, R, n, substitute=(R % 2 == 1))
        ups = _ups(R + n, R, P, NULLS[(j + P) % len(NULLS)])
        bufs, d_beta = call_backward(persons, R, n, beta, ups)
        check_against(persons, R, n, beta, ups, bufs, d_beta, tag="composite P=%d n=%d b=%g R=%d" % (P, n, beta, R))
        bufs2, d_beta2 = call_backward(persons, R, n, beta, ups)
        for a, b in zip(bufs, bufs2):
            for k in a:
                assert torch.equal(a[k].view(torch.int32), b[k].view(torch.int32)), k
        assert torch.equal(d_beta.view(torch.int32), d_beta2.view(torch.int32))


def test_zero_sdf_gives_zero_gradient():
    """sdf == 0 exactly: d sdf is exactly 0 (torch's sign(0) = 0), while its neighbours are not."""
    P, n, R, beta = 2, 33, 5, 0.1
    persons = make_inputs(5, P, R, n, ties=False)
    for d in persons:
        d["sdf"][:, ::3] = 0.0
    bufs, _ = call_backward(persons, R, n, beta, _ups(1, R, P))
    for p, d in enumerate(persons):
        g = take(bufs[p]["sdf"], d["sdf"].shape, "sdf").numpy()
        assert np.all(g[:, ::3] == 0) and np.any(g[:, 1::3] != 0)


def test_tie_order_backward():
    """Identical z rows of two persons with large sigma delta: the kernel's gradients match the (t_end, person, sample)
    order within the gate and differ from the reversed order by more than the gate."""
    P, n, R, beta = 3, 33, wpc_of(3, 33) + 1, 0.1
    persons = make_inputs(7, P, R, n)
    for p, d in enumerate(persons):
        row = int(np.searchsorted(d["idx"], 0))
        d["sdf"][row] = 1.0
        d["sdf"][row, -1] = -0.1 - 0.3 * p
    ups = _ups(3, R, P)
    bufs, d_beta = call_backward(persons, R, n, beta, ups)
    check_against(persons, R, n, beta, ups, bufs, d_beta, tag="tie order")
    c_rev = check_against(persons, R, n, beta, ups, bufs, d_beta, reverse=True, assert_ok=False)
    print("reversed order c=%.3g" % c_rev)
    assert c_rev > C_GATE


def test_rejected_calls_leave_outputs_untouched():
    """Bad P, a short workspace and a NULL required gradient buffer: negative status, mp_last_error text, nothing
    written."""
    from multiply_b200 import _lib as L
    persons = make_inputs(4, 2, 5, 8)
    ups = _ups(2, 5, 2)

    def rejected(text, **kw):
        bufs, d_beta = out = grad_outputs(persons, 8)
        with pytest.raises(L.MpError, match=r"failed \(-\d+\): .*" + text):
            call_backward(persons, 5, 8, 0.1, ups, out=out, **kw)
        assert all(bool((b == SENTINEL).all()) for bb in bufs for b in bb.values())
        assert bool((d_beta == SENTINEL).all())

    for bad_P in (0, 9):
        rejected("bad person list", P_arg=bad_P)
    rejected("workspace too small", ws_delta=-1)
    rejected("null argument", null_grad=1)


# ---------------------------------------------------------------------------------------------
# background and final blend
# ---------------------------------------------------------------------------------------------

@pytest.mark.parametrize("mode", ["eval", "train"])
def test_bg_composite_backward(mode):
    """mp_bg_composite_backward on eval and jittered depths (sdf with exact zeros, |s| ~ 1e-9 on the 1e10 interval):
    d bg_sdf per ray within c * 2^-24 * sum_j (|h_j| dist_j) (1e10 for the last sample), d bg_rgb samples within
    c * 2^-24 * |d bg_rgb|."""
    from multiply_b200 import _lib as L
    R, bound = 1029, 3.0
    rng = np.random.RandomState(21)
    t_rand = rng.random_sample((R, 32)).astype(np.float32) if mode == "train" else None
    sdf = rng.uniform(-2, 2, (R, 32)).astype(np.float32)
    sdf[::5, 3] = 0.0
    sdf[::7, -1] = rng.choice(np.float32([1e-9, -1e-9, 3e-10, 0.0]), len(range(0, R, 7)))
    sdf[::11, :-1] *= np.float32(1e-4)
    rgb = rng.random_sample((R, 32, 3)).astype(np.float32)
    d_out = rng.randn(R, 3).astype(np.float32)
    dv = {k: torch.from_numpy(v).cuda() for k, v in (("sdf", sdf), ("rgb", rgb), ("d", d_out))}
    tr = torch.from_numpy(t_rand).cuda() if t_rand is not None else None
    g_sdf, g_rgb = padded((R, 32)), padded((R, 32, 3))
    L.call("mp_bg_composite_backward", dv["sdf"], dv["rgb"], R, bound, tr, dv["d"], g_sdf, g_rgb)
    torch.cuda.synchronize()
    got_s, got_c = take(g_sdf, (R, 32), "d_bg_sdf").numpy(), take(g_rgb, (R, 32, 3), "d_bg_rgb").numpy()
    z = torch.from_numpy(RG.bg_depths(R, bound, t_rand)).double()
    s = torch.from_numpy(sdf).double().requires_grad_(True)
    c = torch.from_numpy(rgb).double().requires_grad_(True)
    _, v = RG.bg_volume_rendering(z, s, c)
    (v * torch.from_numpy(d_out).double()).sum().backward()
    h = np.abs(np.einsum("rc,rjc->rj", d_out.astype(np.float64), rgb))
    dist = np.concatenate([z[:, :-1].numpy() - z[:, 1:].numpy(), np.full((R, 1), 1e10)], 1)
    fe = dist * np.abs(sdf)
    scale_s = (h.sum(1, keepdims=True) * (1 + fe.sum(1, keepdims=True))) * dist + np.abs(s.grad.numpy())
    c_s = float((np.abs(got_s - s.grad.numpy()) / (EPS * scale_s)).max())
    c_c = float((np.abs(got_c - c.grad.numpy()) / (EPS * (np.abs(d_out).max(1)[:, None, None] + 1e-30))).max())
    _note("bg_" + mode, max(c_s, c_c))
    assert max(c_s, c_c) < C_GATE
    assert np.all(got_s[sdf == 0] == 0)


@pytest.mark.parametrize("with_bg,with_fgv", [(True, True), (False, True), (True, False), (False, False)])
def test_final_compose_backward(with_bg, with_fgv):
    """d fg = d rgb + d fg_values; d bg_T = sum_c (d rgb_c bg_c + d fg_values_c); d bg = bg_T d rgb -- bit for bit as the
    fp32 expressions in that order, with NULL bg_rgb (white) and NULL d fg_rgb_values."""
    from multiply_b200 import _lib as L
    R = 1029
    rng = np.random.RandomState(13)
    bgT, bg = rng.random_sample(R).astype(np.float32), rng.random_sample((R, 3)).astype(np.float32)
    d_rgb, d_fgv = rng.randn(R, 3).astype(np.float32), rng.randn(R, 3).astype(np.float32)
    t = {k: torch.from_numpy(v).cuda() for k, v in (("bgT", bgT), ("bg", bg), ("d_rgb", d_rgb), ("d_fgv", d_fgv))}
    o_fg, o_T, o_bg = padded((R, 3)), padded(R), padded((R, 3))
    L.call("mp_final_compose_backward", t["bgT"], t["bg"] if with_bg else None, R, t["d_rgb"],
           t["d_fgv"] if with_fgv else None, o_fg, o_T, o_bg)
    torch.cuda.synchronize()
    dv = d_fgv if with_fgv else np.zeros_like(d_fgv)
    b = bg if with_bg else np.ones_like(bg)
    want_fg = (d_rgb + dv).astype(np.float32)
    acc = np.zeros(R, np.float32)
    for c in range(3):
        acc = (acc + ((d_rgb[:, c] * b[:, c]).astype(np.float32) + dv[:, c]).astype(np.float32)).astype(np.float32)
    want_bg = (bgT[:, None] * d_rgb).astype(np.float32)
    assert np.array_equal(take(o_fg, (R, 3), "d_fg").numpy().view(np.uint32), want_fg.view(np.uint32))
    assert np.array_equal(take(o_T, (R,), "d_bgT").numpy().view(np.uint32), acc.view(np.uint32))
    assert np.array_equal(take(o_bg, (R, 3), "d_bg").numpy().view(np.uint32), want_bg.view(np.uint32))


# ---------------------------------------------------------------------------------------------
# fused render taps and the mirror's differentiable training forward
# ---------------------------------------------------------------------------------------------

def test_render_taps_leave_pixels_unchanged():
    """mp_render_rays with the background taps requested gives bit-identical pixels; the bg_rgb tap equals
    mp_background's output on the same rays, and the per-sample taps reproduce it through the restated blend."""
    from multiply_b200 import engine, scene as S
    from multiply_b200.model import rend_util
    sc = S.make_scene(P=2, S=16, seed=42, weights="trained")
    inp = S.make_rays(sc, 96, seed=5, region="image")
    hits = S.make_hit_lists(sc, inp)
    r = engine.Renderer(sc)
    base = r.render(inp, hits)
    beta = torch.tensor(float(np.float32(abs(np.float32(r.beta_param))) + np.float32(r.beta_min)), device="cuda")
    from multiply_b200.model.ray_sampler import ErrorBoundSampler
    smp = ErrorBoundSampler(3.0, inverse_sphere_bg=True, **{k: sc["cfg"][k] for k in
                            ("near", "N_samples", "N_samples_eval", "N_samples_extra", "eps", "beta_iters",
                             "max_total_iters", "add_tiny")})
    torch.manual_seed(0)
    rngs = [smp.draw_training_rng(h.numel()) for h in hits]
    rngs = [{k: v for k, v in d.items() if k != "states"} for d in rngs]
    tr = dict(rng=rngs, t_rand_bg=None)
    off = r.render(inp, hits, train=tr)
    on = r.render(inp, hits, train=dict(tr, beta=beta))
    for k in ("rgb_values", "fg_rgb_values", "normal_values", "acc_map", "acc_person_list"):
        assert torch.equal(off[k].view(torch.int32), on[k].detach().view(torch.int32)), k
        assert not off[k].requires_grad and on[k].requires_grad
    # bg_rgb tap == mp_background on the eval depths
    R = inp["uv"].shape[1]
    dirs, cam = rend_util.camera_rays(inp["uv"].cuda(), inp["pose"], inp["intrinsics"])
    r.bg.set_cond(sc["frame_code"])
    bg = r.bg.bg_pixels(dirs, cam, 3.0)
    ev = r.render(inp, hits, train=dict(rng=rngs, t_rand_bg=None, beta=beta))
    torch.cuda.synchronize()
    assert torch.equal(ev["samples_bg"]["bg_rgb"].view(torch.int32), bg.view(torch.int32))
    sb = ev["samples_bg"]
    from_taps = RG.bg_volume_rendering(torch.from_numpy(RG.bg_depths(R, 3.0)).double(), sb["sdf"].detach().cpu().double(),
                                       sb["rgb"].detach().cpu().double())[1]
    assert float((from_taps - bg.cpu().double()).abs().max()) < 1e-5


OPT_TRAIN_LOSS_EPS = 1e-6


def _loss(rgb, acc, accp, gt, mask):
    """loss.py:30-57: L1(rgb) + BCE(acc_map) + L1(acc_person, mask)."""
    l_rgb = (rgb - gt).abs().mean()
    e = OPT_TRAIN_LOSS_EPS
    bce = -1 * (acc * (acc + e).log() + (1 - acc) * (1 - acc + e).log()).mean() * 2
    return l_rgb + bce + (accp - mask).abs().mean()


def _mirror_case(P, seed=33):
    from multiply_b200 import scene as S
    sc = S.make_scene(P=P, S=16, seed=42, weights="trained")
    inp = S.make_rays(sc, 40, seed=seed, region="boxes")
    hits = [h.cuda() for h in S.make_hit_lists(sc, inp)]
    return S.mirror_model(sc), mirror_inputs(inp, P, hits, epoch=251)


def _run_mirror(m, inputs, pid, grad_on, streams=1):
    from multiply_b200 import _lib as L
    L.call("mp_set_streams", streams)
    m.set_render_grad(grad_on)
    m.train()
    try:
        torch.manual_seed(4321)
        out = m(inputs, id=pid)
    finally:
        m.eval()
        L.call("mp_set_streams", 1)
    return out


@pytest.mark.parametrize("P,pid", [(2, -1), (2, 1), (3, -1)])
def test_mirror_training_backward(P, pid):
    """Multiply in .train() with set_render_grad(True): loss = L1(rgb) + BCE(acc_map) + L1(acc_person, mask);
    backward gives density.beta.grad and every render_samples .grad within the gate of fp64 autograd of the restatement
    fed the same taps; the gradients are bit-identical with mp_set_streams(0) and (1); with the switch off the outputs
    are the same bits and carry no graph."""
    m, inputs = _mirror_case(P)
    R = inputs["uv"].shape[1]
    Pn = P if pid == -1 else 1
    g = torch.Generator().manual_seed(P)
    gt = torch.rand(R, 3, generator=g).cuda()
    mask = torch.rand(R, Pn, generator=g).cuda()
    runs = []
    for streams in (1, 0):
        m.density.beta.grad = None
        out = _run_mirror(m, inputs, pid, True, streams)
        loss = _loss(out["rgb_values"], out["acc_map"], out["acc_person_list"], gt, mask)
        loss.backward()
        torch.cuda.synchronize()
        runs.append((out, float(m.density.beta.grad)))
    (out, gbeta), (out0, gbeta0) = runs
    assert np.float32(gbeta) == np.float32(gbeta0)
    rs, rs0 = out["render_samples"], out0["render_samples"]
    for a, b in zip(rs["persons"], rs0["persons"]):
        for k in ("sdf", "rgb", "normal"):
            assert torch.equal(a[k].grad.view(torch.int32), b[k].grad.view(torch.int32)), k
    for k in ("sdf", "rgb"):
        assert torch.equal(rs["bg"][k].grad.view(torch.int32), rs0["bg"][k].grad.view(torch.int32)), k
    off = _run_mirror(m, inputs, pid, False)
    for k in ("rgb_values", "acc_map", "acc_person_list", "normal_values"):
        assert torch.equal(off[k].view(torch.int32), out[k].detach().view(torch.int32)), k
        assert off[k].grad_fn is None and not off[k].requires_grad
    assert "render_samples" not in off
    # fp64 restatement fed the taps; the upstream gradients of the gate are the loss's own, read from the restatement
    bp = torch.tensor(float(m.density.beta.detach()), dtype=torch.float64, requires_grad=True)
    b32 = float(np.float32(abs(np.float32(float(bp)))) + np.float32(m.density.beta_min))    # the fp32 beta of the render
    beta = bp.abs() + (b32 - abs(float(bp)))
    persons = [dict(idx=d["ray_index"].cpu().numpy(), z=d["z_vals"].cpu().numpy(), sdf=d["sdf"].detach().cpu().numpy(),
                    rgb=d["rgb"].detach().cpu().numpy(), nrm=d["normal"].detach().cpu().numpy()) for d in rs["persons"]]
    tp = [dict(idx=d["idx"], z=torch.from_numpy(d["z"]).double(),
               **{k: torch.from_numpy(d[k]).double().requires_grad_(True) for k in ("sdf", "rgb", "nrm")})
          for d in persons]
    n = persons[0]["sdf"].shape[1]
    outs = RG.composite(tp, R, n, beta)
    for o in outs:
        o.retain_grad()
    fg, nrm, acc, accp, bgT = outs
    bgd = rs["bg"]
    bsdf = bgd["sdf"].detach().cpu().double().requires_grad_(True)
    brgb = bgd["rgb"].detach().cpu().double().requires_grad_(True)
    zb = torch.from_numpy(RG.bg_depths(R, 3.0, bgd["t_rand"].cpu().numpy())).double()
    _, bg = RG.bg_volume_rendering(zb, bsdf, brgb)
    bg.retain_grad()
    rgb, _ = RG.blend(fg, bgT, bg)
    assert float((rgb - out["rgb_values"].detach().cpu().double()).abs().max()) < 1e-5
    # the loss's gradients w.r.t. the pixels, taken at the render's own (fp32) pixel values: BCE near acc = 1 is too
    # ill-conditioned to take them at the restated values
    px = [out[k].detach().cpu().double().requires_grad_(True) for k in ("rgb_values", "acc_map", "acc_person_list")]
    _loss(*px, gt.cpu().double(), mask.cpu().double()).backward()
    ((rgb * px[0].grad).sum() + (acc * px[1].grad).sum() + (accp * px[2].grad).sum()).backward()
    ups = dict(zip(("d_fg", "d_nrm", "d_acc", "d_accp", "d_bgT"), (_g(o) for o in outs)))
    sc = gate_scales(persons, R, n, float(beta), ups, bgT.detach().numpy())
    got = [dict(sdf=d["sdf"].grad.cpu().numpy(), rgb=d["rgb"].grad.cpu().numpy(), nrm=d["normal"].grad.cpu().numpy())
           for d in rs["persons"]]
    want = [dict(sdf=_g(t["sdf"]), rgb=_g(t["rgb"]), nrm=_g(t["nrm"])) for t in tp]
    worst = worst_c(persons, got, want, float(bp.grad), gbeta, sc)
    # background: d sdf within c 2^-24 sum_j |h_j| dist_j (1 + total optical depth), d rgb within c 2^-24 |d bg_rgb|
    h = np.abs(np.einsum("rc,rjc->rj", bg.grad.numpy(), brgb.detach().numpy()))
    dist = np.concatenate([(zb[:, :-1] - zb[:, 1:]).numpy(), np.full((R, 1), 1e10)], 1)
    fe = dist * np.abs(bsdf.detach().numpy())
    scale_s = h.sum(1, keepdims=True) * (1 + fe.sum(1, keepdims=True)) * dist + np.abs(bsdf.grad.numpy())
    worst = max(worst, float((np.abs(bgd["sdf"].grad.cpu().numpy() - bsdf.grad.numpy()) / (EPS * scale_s)).max()))
    dscale = np.abs(bg.grad.numpy()).max(1)[:, None, None] + 1e-30
    worst = max(worst, float((np.abs(bgd["rgb"].grad.cpu().numpy() - brgb.grad.numpy()) / (EPS * dscale)).max()))
    _note("mirror P=%d id=%d" % (P, pid), worst)
    assert worst < C_GATE
