"""GPU: the multi-person compositor (csrc/composite.cu: mp_composite, mp_final_compose) against a float64 restatement of
multiply.py:427-480 at person-count, sample-count, block and tie edges.

The kernel merges the P per-person lists of a ray by rank (binary searches: upper_bound for earlier persons, lower_bound
for later ones, so equal t_end values keep (person, sample) order), scans sigma * delta in chunks per lane and takes bg_T
from the exclusive prefix of the ray's last merged sample.  Whole renders only ever tie on the shared `far` where
sigma ~ 0, so the tie order and the prefix there are checked here on synthetic inputs where they matter: identical z
rows of two persons on one ray, zero-length intervals inside one list, and the shared far with a negative sdf on the
last sample.  Sizes: P = 1 .. 8 (MP_MAX_PERSONS), n around the warp (1, 31, 32, 33, 193, 385) and the largest n whose
12 P n bytes of shared memory per warp fit the kernel's 200 KB cap at P = 8; R = 1 and around the rays-per-block edge."""
import os
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from _abi import SENTINEL, padded, take                                     # noqa: E402
from _setups import SMEM_CAP, make_inputs, person_samples, wpc_of           # noqa: E402

N_MAX_P8 = SMEM_CAP // (12 * 8)         # 2133: the largest n with 12 * P * n <= 200 KB at P = 8
# fp64 comparison gate of every output (fg_rgb, normal, acc, acc_person, bg_T); the measured worst values are quoted in
# the docstring of test_composite_vs_fp64
TOL = 1e-5
MEASURED = {}


# ---------------------------------------------------------------------------------------------
# float64 (or float32) restatement of multiply.py:427-480
# ---------------------------------------------------------------------------------------------

def composite_ref(persons, R, n, beta, dtype=np.float64, reverse=False):
    """Flatten every person's samples, sort by (ray, t_end, person, sample) -- (ray, t_end, -person, -sample) with
    `reverse` --, Laplace sigma (density.py:20-25), exclusive per-ray prefix of sigma * delta, w = T * alpha, and
    bg_T = T at the start of the ray's last merged sample (1 for rays no person hits).
    persons: list of dict(idx [R_p] int64, z [R_p, n+1], sdf [R_p, n], rgb / nrm [R_p, n, 3]).
    Returns fg_rgb [R,3], normal [R,3], acc [R], acc_person [R,P], bg_T [R] in `dtype`."""
    P = len(persons)
    cols = {k: [] for k in ("ray", "pid", "smp", "ts", "te", "sdf", "rgb", "nrm")}
    for p, d in enumerate(persons):
        Rp = d["idx"].shape[0]
        cols["ray"].append(np.repeat(np.asarray(d["idx"], np.int64), n))
        cols["pid"].append(np.full(Rp * n, p))
        cols["smp"].append(np.tile(np.arange(n), Rp))
        cols["ts"].append(d["z"][:, :-1].reshape(-1))
        cols["te"].append(d["z"][:, 1:].reshape(-1))
        cols["sdf"].append(d["sdf"].reshape(-1))
        cols["rgb"].append(d["rgb"].reshape(-1, 3))
        cols["nrm"].append(d["nrm"].reshape(-1, 3))
    c = {k: np.concatenate(v) for k, v in cols.items()}
    sg = -1 if reverse else 1
    o = np.lexsort((sg * c["smp"], sg * c["pid"], c["te"], c["ray"]))
    c = {k: v[o] for k, v in c.items()}
    # sigma and the exponentials with torch's operations in the order of oracle/port.py (in float32, 1 - exp and the
    # 0.5 + 0.5 * expm1 of a positive sdf cancel, so another library's expm1 would move them by an ulp of 0.5 / beta)
    td = torch.float64 if dtype == np.float64 else torch.float32
    ts, te, sdf = (torch.from_numpy(c[k].astype(dtype)) for k in ("ts", "te", "sdf"))
    b = torch.tensor(beta, dtype=td)
    sigma = (1 / b) * (0.5 + 0.5 * sdf.sign() * torch.expm1(-sdf.abs() / b))
    sd_t = sigma * (te - ts)
    sd = sd_t.numpy()
    ray = c["ray"]
    starts = np.flatnonzero(np.r_[True, ray[1:] != ray[:-1]]) if ray.size else np.zeros(0, np.int64)
    ends = np.r_[starts[1:], ray.size]
    excl = np.zeros_like(sd)
    for s, e in zip(starts, ends):             # per-ray sequential exclusive scan (nerfacc's definition)
        excl[s + 1:e] = np.cumsum(sd[s:e - 1], dtype=dtype)
    T = torch.exp(-torch.from_numpy(excl)).numpy()
    w = (torch.from_numpy(T) * (1 - torch.exp(-sd_t))).numpy()
    fg, nrm = np.zeros((R, 3), dtype), np.zeros((R, 3), dtype)
    acc, accp = np.zeros(R, dtype), np.zeros((R, P), dtype)
    np.add.at(fg, ray, w[:, None] * c["rgb"].astype(dtype))
    np.add.at(nrm, ray, w[:, None] * c["nrm"].astype(dtype))
    np.add.at(acc, ray, w)
    np.add.at(accp, (ray, c["pid"]), w)
    bgT = np.ones(R, dtype)
    if ray.size:
        bgT[ray[ends - 1]] = T[ends - 1]
    return fg, nrm, acc, accp, bgT


# ---------------------------------------------------------------------------------------------
# synthetic inputs
# ---------------------------------------------------------------------------------------------

def subset(persons, rays):
    """The same samples composited for the rays `rays` only (sorted), renumbered 0 .. len(rays) - 1."""
    out = []
    for d in persons:
        keep = np.isin(d["idx"], rays)
        out.append(dict(idx=np.searchsorted(rays, d["idx"][keep]).astype(np.int64),
                        **{k: np.ascontiguousarray(d[k][keep]) for k in ("z", "sdf", "rgb", "nrm")}))
    return out


# ---------------------------------------------------------------------------------------------
# the C ABI with sentinel-padded outputs
# ---------------------------------------------------------------------------------------------

def outputs(R, P):
    return dict(fg=padded((R, 3)), nrm=padded((R, 3)), acc=padded(R), accp=padded((R, P)), bgT=padded(R))


def call_composite(persons, R, n, beta, P_arg=None, ws_delta=0, bufs=None):
    """The five outputs on the host, read from ``bufs`` (fresh ``outputs`` by default)."""
    from multiply_b200 import _lib as L
    P = len(persons)
    arr, keep = person_samples(persons)
    bufs = outputs(R, P) if bufs is None else bufs
    ws_bytes = L.call("mp_composite_workspace_bytes", R, P) + ws_delta
    ws = L.workspace(ws_bytes, "cuda")
    L.call("mp_composite", arr, P if P_arg is None else P_arg, R, n, float(beta), bufs["fg"], bufs["nrm"], bufs["acc"],
           bufs["accp"], bufs["bgT"], ws, ws_bytes)
    torch.cuda.synchronize()
    return tuple(take(bufs[k], shp, name).numpy() for k, shp, name in (
        ("fg", (R, 3), "fg_rgb"), ("nrm", (R, 3), "normal"), ("acc", R, "acc"), ("accp", (R, P), "acc_person"),
        ("bgT", R, "bg_T")))


NAMES = ("fg_rgb", "normal", "acc", "acc_person", "bg_T")


def _errs(got, want):
    return {k: float(np.abs(np.asarray(g, np.float64) - w).max()) if g.size else 0.0
            for k, g, w in zip(NAMES, got, want)}


# (P, n, beta): every P in 1..8, every n of the docstring, both betas; beta = 1e-4 makes T underflow after one sample
CASES = [(1, 1, 0.1), (1, 32, 1e-4), (1, 385, 0.1), (2, 31, 0.1), (2, 33, 1e-4), (3, 193, 0.1), (3, 1, 1e-4),
         (4, 32, 0.1), (4, 385, 1e-4), (5, 33, 0.1), (6, 193, 1e-4), (7, 31, 0.1), (7, 385, 0.1), (8, 1, 0.1),
         (8, 33, 1e-4), (8, 193, 0.1), (8, N_MAX_P8, 0.1), (8, N_MAX_P8, 1e-4)]


@pytest.mark.parametrize("P,n,beta", CASES, ids=["P%d-n%d-b%g" % c for c in CASES])
def test_composite_vs_fp64(P, n, beta):
    """Every output against the fp64 restatement, at R = 1 and around the rays-per-block edge; nothing written past R;
    and a subset of the rays composited alone (hit lists remapped) gives bit-identical results for those rays.

    Measured on one H100 80GB HBM3 at a 400 W power limit: worst error over all cases and outputs 3.1e-6 (P = 7,
    n = 385, beta = 0.1); the fp32 sigma of a positive sdf (0.5 + 0.5 * expm1 cancels) and the fp32 prefix sums over up
    to 17 064 samples per ray account for it."""
    wpc = wpc_of(P, n)
    Rs = sorted({1, max(1, wpc - 1), wpc, wpc + 1, 2 * wpc + 1, 3 * wpc + 5})
    for R in Rs:
        persons = make_inputs(1000 * P + n + R, P, R, n, substitute=(R % 2 == 1))
        got = call_composite(persons, R, n, beta)
        want = composite_ref(persons, R, n, np.float32(beta))
        e = _errs(got, want)
        key = (P, n, beta, R)
        MEASURED[key] = max(e.values())
        print("COMPOSITE P=%d n=%d beta=%g R=%d wpc=%d errors %s" % (P, n, beta, R, wpc,
                                                                   " ".join("%s=%.2e" % kv for kv in e.items())))
        assert max(e.values()) < TOL, e
        if R >= 3:
            rays = np.arange(0, R, 2)
            part = call_composite(subset(persons, rays), rays.size, n, beta)
            for k, a, b in zip(NAMES, part, got):
                assert np.array_equal(a.view(np.uint32), b[rays].view(np.uint32)), k


def test_tie_order():
    """Equal t_end values merge in (person, sample) order.  A case where that order and the reversed one differ by
    more than 1e-3 in the weights or bg_T: the kernel matches the first and not the second."""
    P, n, R, beta = 3, 33, wpc_of(3, 33) + 1, 0.1
    persons = make_inputs(7, P, R, n)
    for p, d in enumerate(persons):        # ray 0 (every person hits it): nearly empty up to a dense last sample
        row = int(np.searchsorted(d["idx"], 0))
        d["sdf"][row] = 1.0
        d["sdf"][row, -1] = -0.1 - 0.3 * p
    fwd = composite_ref(persons, R, n, np.float32(beta))
    rev = composite_ref(persons, R, n, np.float32(beta), reverse=True)
    gap = max(float(np.abs(a - b).max()) for a, b in zip(fwd, rev))
    assert gap > 1e-3
    got = call_composite(persons, R, n, beta)
    assert max(_errs(got, fwd).values()) < TOL
    assert max(_errs(got, rev).values()) > 1e-3 - TOL
    # in particular on bg_T, where the shared far with a negative sdf decides which sample is last
    assert float(np.abs(fwd[4] - rev[4]).max()) > 1e-3
    assert float(np.abs(got[4] - fwd[4]).max()) < TOL


def test_rejected_calls_leave_outputs_untouched():
    """An over-cap P * n, a P outside [1, 8] and a short workspace each return a negative status with the expected
    mp_last_error() text, and no output is written (the checks run on the host before any kernel writes)."""
    from multiply_b200 import _lib as L

    def rejected(text, persons, R, n, **kw):
        bufs = outputs(R, len(persons))
        with pytest.raises(L.MpError, match=r"failed \(-\d+\): .*" + text):
            call_composite(persons, R, n, 0.1, bufs=bufs, **kw)
        assert all(bool((b == SENTINEL).all()) for b in bufs.values())

    rejected("too large for shared memory", make_inputs(3, 8, 5, N_MAX_P8 + 1, ties=False), 5, N_MAX_P8 + 1)
    persons = make_inputs(4, 2, 5, 8)
    for bad_P in (0, 9):
        rejected("bad person list", persons, 5, 8, P_arg=bad_P)
    rejected("workspace too small", persons, 5, 8, ws_delta=-1)
    # the largest n that fits still runs
    persons = make_inputs(5, 8, 2, N_MAX_P8, ties=False)
    call_composite(persons, 2, N_MAX_P8, 0.1)


@pytest.mark.parametrize("with_bg,with_fg_out", [(True, True), (False, True), (True, False), (False, False)])
def test_final_compose(with_bg, with_fg_out):
    """rgb = fg + bg_T * bg (bg NULL: white) and fg_rgb_values = fg + bg_T (may be NULL), bit for bit as fp32."""
    from multiply_b200 import _lib as L
    R = 1029
    rng = np.random.RandomState(11)
    fg = rng.random_sample((R, 3)).astype(np.float32)
    bgT = rng.random_sample(R).astype(np.float32)
    bgT[::7] = 1.0
    bgT[::11] = 0.0
    bg = rng.random_sample((R, 3)).astype(np.float32)
    d_fg, d_T, d_bg = (torch.from_numpy(a).cuda() for a in (fg, bgT, bg))
    rgb = padded((R, 3))
    fgo = padded((R, 3)) if with_fg_out else None
    L.call("mp_final_compose", d_fg, d_T, d_bg if with_bg else None, R, rgb, fgo)
    torch.cuda.synchronize()
    b = bg if with_bg else np.ones_like(bg)
    want = (fg + (bgT[:, None] * b).astype(np.float32)).astype(np.float32)
    assert np.array_equal(take(rgb, (R, 3), "rgb").numpy().view(np.uint32), want.view(np.uint32))
    if with_fg_out:
        want_fg = (fg + bgT[:, None]).astype(np.float32)
        assert np.array_equal(take(fgo, (R, 3), "fg_rgb_values").numpy().view(np.uint32), want_fg.view(np.uint32))
