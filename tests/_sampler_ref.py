"""The float64 comparison of the error-bound sampler shared by tests/test_gpu_sampler.py (GPU against float64) and
tests/test_sampler_reference.py (float32 port against float64): per-sample bounds from the decision trace of
oracle/port.error_bound_get_z_vals(dtype=torch.float64, trace=...).

Per sample the bound is |dz| <= K 2^-24 s, s = |z| + M (b1 - b0) / max(denom, 1e-5) (the first-order sensitivity of the
inverse CDF to the cdf's M-term sums) plus the s of its two bins, accumulated over trips.  Discrete decisions inside fp32
resolution do not mask their ray; they widen the bound by what the other outcome can do:
- searchsorted or the denom cutoff within MARGIN 2^-24: the sample lies in its bin or a neighbouring one;
- a line-search test `err <= eps` within MARGIN_ERR M 2^-24 (relative): from that step on the two sides may bisect
  different halves, so beta is known only within that step's bracket; the trip's resampling is rerun at both ends of
  it and the samples' largest move is added to their s;
- the sample at u = 1 lands in whichever bin the rounding of the cdf's tail against 1 picks (cdf[M-1] <= 1 gives z[M-1];
  above 1 it lies inside the last bins, which the 1e-5 pdf floor keeps below the denom cutoff).  The reference's own
  fp32 cumsum lands on either side, so depths from the first such bin on are held to the exact invariants only; at most
  TAIL_MAX values per row.
A ray is masked only when one of its points lies within MARGIN (s + 3) 2^-24 of the 0.1 outlier radius (the SDF jumps
to 4 there), s the point's first-order sensitivity: a sample widened to its neighbouring bins is bounded where it lands,
but the SDF the next trips see there is first-order only.  Trip counts must be equal, and the batch flag's own margin must exceed FLAG_MIN.

Constants were measured on one H100 80GB HBM3 at a 700 W power limit (GPU against float64; the float32 port against
float64 on the CPU is inside the same bounds)."""
import torch

from oracle import port

EPS = 2.0 ** -24
MEASURED = {}

# K of the per-sample bound: the worst measured is 1256 (list edges); 635 on the trip edges, 37 on the geometry edges,
# 5.4 in training mode
K_Z = 2048.0
MARGIN = 16.0
MARGIN_ERR = 4.0
# masked fraction (rays with a point at the outlier radius) allowed per case: measured 0 on single-trip, geometry,
# slow-ray and training cases.  Over several trips a point's first-order s grows with M / max(denom, 1e-5), so more
# points sit inside MARGIN (s + 3) 2^-24 of the radius: measured at most 0.25 (4 of 16 rays) with E <= 64, 0.667
# (4 of 6 rays) at E = 512 with 8 trips (M = 4096)
MASK_MAX = 0.05
MASK_MAX_TRIPS = 0.3
MASK_MAX_M4096 = 0.75
# output values per row past the u = 1 tail cutoff: far, the extra at z[M-1], the u = 1 sample and one neighbour
TAIL_MAX = 4
# share of samples whose searchsorted / denom decision is inside MARGIN 2^-24, allowed per trip: measured at most 0.83
# (the 1e-5 pdf floor puts every empty bin of the final set 1e-5 M 1e-5 below the denom cutoff)
AMB_MAX = 0.9
# share of rays whose line search has a test inside MARGIN_ERR M 2^-24, allowed per trip: measured at most 0.5 (M = 4096)
LS_MAX = 0.75
# the batch flag's float64 margin must exceed this for the case to be deterministic
FLAG_MIN = 1e-3


def note(key, v):
    MEASURED[key] = max(MEASURED.get(key, 0.0), float(v))


def report():
    for k in sorted(MEASURED):
        print("MEASURED %s = %.4g" % (k, MEASURED[k]))


def cfg_of(E, S_, X, iters, eps=0.1, beta_iters=10, near=0.0, beta=0.1):
    return dict(scene_bounding_sphere=3.0, near=near, N_samples=S_, N_samples_eval=E, N_samples_extra=X, eps=eps,
                beta_iters=beta_iters, max_total_iters=iters, add_tiny=1e-6, beta_param=beta)


def far_of(d, o, r=3.0):
    return port.get_sphere_intersections(o, d, r=r)[:, 1]


def sensitivities(name, cfg, tr, dist, d, o, extra_idx=None):
    """Per ray: the float64 final set, sorted, with the sensitivity s of each value (units of 2^-24, widened over
    neighbours the sort may swap), the mask and the tail cutoff.  dist: per trip the float64 distance of the trip's new
    points to the nearest vertex (None: no outlier radius); extra_idx: the list positions of the extras (training mode's
    randperm(M)[:X]; default linspace(0, M-1, X))."""
    X = cfg["N_samples_extra"]
    beta0 = port.get_beta(cfg["beta_param"]).double()
    z0 = tr["trips"][0]["z"]
    s_list = z0.abs().clone()
    R = z0.shape[0]
    masked = torch.zeros(R, dtype=torch.bool)
    cut = torch.full((R,), float("inf"), dtype=torch.float64)
    s_new = s_pt = s_first = s_list      # s_first: first-order only, never widened
    for t, tp in enumerate(tr["trips"]):
        M = tp["z"].shape[1]
        if dist is not None:
            masked |= ((dist[t] - 0.1).abs() < MARGIN * EPS * (s_pt + 3.0)).any(1)
        if bool((tp["u"][:, -1] == 1).any()):
            # tail bins the u = 1 sample can fall into: from bin k-1 (k the first cdf entry within MARGIN 2^-24 of 1)
            # on; only a bin whose pdf is below the 1e-5 denom cutoff puts it a whole bin away
            cdf, res = tp["cdf"], MARGIN * EPS
            k = (cdf >= 1 - res).double().argmax(1)
            i = torch.arange(M - 1)[None]
            low = (i >= (k - 1)[:, None]) & ((cdf[:, 1:] - cdf[:, :-1]) < 1e-5 + res)
            first = low.double().argmax(1)
            cut = torch.where(low.any(1), torch.minimum(cut, tp["z"].gather(1, first[:, None])[:, 0]), cut)
        b0, b1 = tp["z"].gather(1, tp["below"]), tp["z"].gather(1, tp["above"])
        s_new = tp["samples"].abs() + M * (b1 - b0).abs() / tp["denom_raw"].clamp_min(1e-5) + \
            torch.maximum(s_list.gather(1, tp["below"]), s_list.gather(1, tp["above"]))
        s_pt = tp["samples"].abs() + M * (b1 - b0).abs() / tp["denom_raw"].clamp_min(1e-5) + \
            torch.maximum(s_first.gather(1, tp["below"]), s_first.gather(1, tp["above"]))
        amb = (tp["u_margin"] < MARGIN * EPS) | (tp["denom_margin"] < MARGIN * EPS)
        lo = tp["z"].gather(1, (tp["below"] - 1).clamp_min(0))
        hi = tp["z"].gather(1, (tp["above"] + 1).clamp_max(M - 1))
        s_new = torch.where(amb, torch.maximum(s_new, (hi - lo) / EPS), s_new)
        note("ambiguous cdf decisions " + name, float(amb.double().mean()))
        assert float(amb.double().mean()) <= AMB_MAX, (name, t, float(amb.double().mean()))
        # line search: beta is known within the bracket of its first test inside MARGIN_ERR M 2^-24
        close = tp["err_steps"].abs() < MARGIN_ERR * M * EPS
        has = close.any(1)
        note("line-search widened rays " + name, float(has.double().mean()))
        assert float(has.double().mean()) <= LS_MAX, (name, t, float(has.double().mean()))
        if bool(has.any()):
            dbeta = torch.where(has, tp["brackets"].gather(1, close.double().argmax(1)[:, None])[:, 0], 0.0)
            lo_b = torch.minimum(beta0.expand(R), tp["beta_init"])
            hi_b = torch.maximum(beta0.expand(R), tp["beta_init"])
            move = torch.zeros_like(s_new)
            for b in ((tp["beta"] - dbeta).clamp(lo_b, hi_b), (tp["beta"] + dbeta).clamp(lo_b, hi_b)):
                alt = port._inverse_cdf_step(tp["z"], tp["sdf"], tp["d_star"], b, not tp["final"], tp["u"],
                                             cfg["add_tiny"])["samples"]
                move = torch.maximum(move, (alt - tp["samples"]).abs())
            s_new = s_new + move / EPS
        if not tp["final"]:
            s_list = torch.cat([s_list, s_new], 1).gather(1, tp["order"])
            s_first = torch.cat([s_first, s_pt], 1).gather(1, tp["order"])
    last = tr["trips"][-1]
    M = last["z"].shape[1]
    far = far_of(d.double(), o.double())
    idx = torch.linspace(0, M - 1, X).long() if extra_idx is None else extra_idx.long()
    near = torch.full((R, 1), cfg["near"], dtype=torch.float64)
    vals = torch.cat([last["samples"], near, far[:, None], last["z"][:, idx]], 1)
    sens = torch.cat([s_new, torch.zeros_like(near), far.abs()[:, None], s_list[:, idx]], 1)
    srt, order = torch.sort(vals, dim=1, stable=True)
    ss = sens.gather(1, order)
    # sorting is 1-Lipschitz; a value can swap with neighbours inside its own uncertainty: take the window max
    win = ss.clone()
    for k in (1, 2):
        win[:, k:] = torch.maximum(win[:, k:], ss[:, :-k])
        win[:, :-k] = torch.maximum(win[:, :-k], ss[:, k:])
    return srt, win, masked, cut


def compare(name, cfg, d, o, z, trips, tr, dist, extra_idx=None, mask_max=MASK_MAX):
    """Trip count equal, batch flag off its tie, masked and tail shares within their bounds, and |dz| <= K 2^-24 s on
    every unmasked value below the tail cutoff."""
    for t, tp in enumerate(tr["trips"]):
        assert tp["flag_margin"] > FLAG_MIN, "%s: batch flag of trip %d within %.2g of its tie" % (
            name, t, tp["flag_margin"])
    assert trips == tr["n_trips"], (name, trips, tr["n_trips"])
    srt, win, masked, cut = sensitivities(name, cfg, tr, dist, d, o, extra_idx)
    z = z.double()
    head = srt < cut[:, None]
    ratio = torch.where(head, (z - srt).abs() / (EPS * win.clamp_min(1e-30)), torch.zeros_like(z)).max(1)[0]
    frac, tail = float(masked.double().mean()), int((~head).sum(1).max())
    note("K_z " + name, float(ratio[~masked].max()) if bool((~masked).any()) else 0.0)
    note("masked " + name, frac)
    note("tail values per row " + name, tail)
    assert frac <= mask_max, "%s: %.3f of the rays masked" % (name, frac)
    assert tail <= TAIL_MAX, "%s: %d values of a row past the u = 1 tail cutoff" % (name, tail)
    bad = (~masked) & (ratio > K_Z)
    assert not bool(bad.any()), "%s: %d rays over K = %g (worst %.3g)" % (name, int(bad.sum()), K_Z,
                                                                           float(ratio[~masked].max()))
