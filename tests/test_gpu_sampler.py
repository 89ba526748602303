"""GPU: the error-bound ray sampler (csrc/sampler.cu: mp_sample_rays, mp_sample_rays_train) at list, trip, tie and batch
edges.

Exact checks, no tolerance, wherever the algorithm is deterministic:
- every output slot is written (sentinel outputs, a workspace of 0xFF bytes = NaN floats / -1 ints), and the outputs are
  bit-equal to a run on a zeroed workspace, also after a call with another configuration on the same workspace;
- per-ray outputs do not depend on which warp, block or SM runs the ray (permuted and 33x replicated batches);
- a field whose SDF is exact on both MLP engines gives bit-equal samples on SIMT and tensor cores;
- rows are sorted, finite, inside [near, far] and hold near and far;
- training mode picks the row of its per-trip draws for the trip count the loop ended on;
- invalid configurations are rejected through the ABI and write nothing.

Float64 comparisons elsewhere (tests/_sampler_ref.py states the bound, the widenings and the masks):
oracle/port.error_bound_get_z_vals in float64 with the draws of the GPU run, its SDF callback the GPU's own deformer and
field at the fp32 points the kernels form, so both sides sample one function."""
import os
import re
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from multiply_b200 import scene as S          # noqa: E402  (CPU-only module)
from oracle import port                       # noqa: E402

from _abi import SENTINEL, SENTINEL_INT, padded, take                                            # noqa: E402
from _sampler_ref import EPS, MASK_MAX_M4096, MASK_MAX_TRIPS, cfg_of, compare, far_of, report      # noqa: E402
from _setups import rays, train_rng                                                              # noqa: E402


@pytest.fixture(scope="module", autouse=True)
def _print_measured():
    yield
    report()


# ---------------------------------------------------------------------------------------------
# set-up: one person of the synthetic scene, its rays, and the sampler ABI
# ---------------------------------------------------------------------------------------------

def c_cfg(cfg):
    from multiply_b200 import engine
    return engine.sampler_cfg(cfg, cfg["beta_param"])


@pytest.fixture(scope="module")
def scene():
    return S.make_scene(P=2, S=16, seed=42)


@pytest.fixture(scope="module")
def person(scene):
    from multiply_b200 import engine
    p = scene["persons"][0]
    f = engine.Field(p["implicit"], p["render"])
    f.set_cond(p["cond"])
    b = engine.Body(p["verts_c"], p["weights"], cano_cell=0.1001 / p["scale"])
    b.set_pose(p["verts_p"], p["tfs"])
    return dict(p=p, field=f, body=b)


def const_field(p, c):
    """ImplicitNet with weight_g = 0 on every layer and last bias c: SDF = c on every non-outlier, exactly, on both
    engines (every layer's weight is 0 * v / |v|)."""
    from multiply_b200 import engine
    imp = {k: (torch.zeros_like(v) if k.endswith("weight_g") else v.clone()) for k, v in p["implicit"].items()}
    imp["lin8.bias"] = torch.zeros_like(imp["lin8.bias"])
    imp["lin8.bias"][0] = c
    f = engine.Field(imp, p["render"])
    f.set_cond(p["cond"])
    return f


def run(cfg, body, field, d, o, rng=None, ws=None, fill=None):
    """One sampler call through the ABI.  Returns dict(err, z, z_bg, z_eik, trips) on the host -- err: the error text of
    a rejected call, else None -- and the workspace it used; fill: byte value written into the workspace first."""
    from multiply_b200 import _lib as L, engine
    c = c_cfg(cfg)
    R = d.shape[0]
    n = cfg["N_samples"] + cfg["N_samples_extra"] + 2
    need = L.call("mp_sampler_workspace_bytes", c, R)
    if ws is None or ws.numel() < need:
        ws = L.workspace(need, "cuda")
    if fill is not None:
        ws.fill_(fill)
    dd, oo = d.cuda().contiguous(), o.cuda().contiguous()
    z, z_bg, z_eik, trips = padded((R, n)), padded((R, 32)), padded(R), padded(1, torch.int32)
    err = None
    try:
        if rng is None:
            L.call("mp_sample_rays", c, body.handle, field.handle, dd, oo, R, z, z_bg, trips, ws, ws.numel())
        else:
            r, keep = engine.sampler_rng_struct(rng, torch.device("cuda"))
            L.call("mp_sample_rays_train", c, body.handle, field.handle, dd, oo, R, r, z, z_bg, z_eik, trips, ws,
                   ws.numel())
    except L.MpError as e:
        err = str(e)
    torch.cuda.synchronize()
    out = dict(err=err, z=take(z, (R, n), "z_vals"), z_bg=take(z_bg, (R, 32), "z_bg"), z_eik=take(z_eik, R, "z_eik"),
               trips=int(take(trips, 1, "trips")[0]))
    return out, ws


def check_rows(out, cfg, d, o, train=False):
    """Exact invariants of every output row: no sentinel, finite, sorted, inside [near, far], near and far present."""
    z = out["z"]
    assert out["err"] is None, out["err"]
    assert not bool((z == SENTINEL).any()), "%d slots of z_vals unwritten" % int((z == SENTINEL).sum())
    assert not bool((out["z_bg"] == SENTINEL).any())
    assert bool(torch.isfinite(z).all())
    assert bool((z[:, 1:] >= z[:, :-1]).all()), "a row is not sorted"
    near = cfg["near"]
    assert bool((z[:, 0] == near).all()), "near is not the first sample"
    # every sample lies in [z[0], z[M-1]] = [near, far]: far is the row's last value (the host's fp32 far may differ
    # from the kernel's by the summation order of d . o)
    far = far_of(d, o).to(torch.float32)
    assert bool(((z[:, -1] - far).abs() <= 8 * EPS * far.abs().clamp_min(1.0)).all()), "far is not the last sample"
    if train:
        assert not bool((out["z_eik"] == SENTINEL).any())


# ---------------------------------------------------------------------------------------------
# float64 reference driven by the GPU's own SDF
# ---------------------------------------------------------------------------------------------

def gpu_callback(body, field, verts_p):
    """ray_sdf_fn of port.error_bound_get_z_vals: the points o + z d formed in fp32 with separate roundings (as
    deform_rays_kernel does), evaluated by mp_sdf_with_deformer (outliers -> 4); the float64 nearest-vertex distance of
    each point is kept per call, to know the points near the 0.1 outlier radius."""
    from multiply_b200 import _lib as L
    dist = []
    v64 = verts_p.double()

    def fn(o, z, d):
        o32, z32, d32 = o.float(), z.float(), d.float()
        x = (o32.unsqueeze(1) + (z32.unsqueeze(2) * d32.unsqueeze(1))).reshape(-1, 3).contiguous()
        N = x.shape[0]
        xg = x.cuda()
        sdf = torch.empty(N, device="cuda")
        xc = torch.empty(N, 3, device="cuda")
        ws = L.workspace(L.call("mp_sdf_with_deformer_workspace_bytes", N), "cuda")
        L.call("mp_sdf_with_deformer", body.handle, field.handle, xg, N, sdf, xc, None, ws, ws.numel())
        d2, _, _ = port.knn_points(x.double()[None], v64[None], return_nn=False)
        dist.append(d2[0, :, 0].sqrt().reshape(z.shape))
        return sdf.cpu().double()[:, None]

    fn.dist = dist
    return fn


def reference(cfg, person, d, o, rng=None):
    """float64 port run with the GPU callback; returns (z_out, z_bg, z_eik or None, trace, callback)."""
    cb = gpu_callback(person["body"], person["field"], person["p"]["verts_p"])
    tr, st = {}, {}
    out = port.error_bound_get_z_vals(d.double(), o.double(), None, cfg, cfg["beta_param"], stats=st, rng=rng,
                                      dtype=torch.float64, ray_sdf_fn=cb, trace=tr)
    tr["n_trips"] = st["trips"]
    return out, tr, cb


# ---------------------------------------------------------------------------------------------
# exact checks
# ---------------------------------------------------------------------------------------------

def test_rejects_invalid_configs(scene, person):
    """Unsupported configurations fail through the ABI with an error and write nothing: E < 2, S > E, S < 1, X < 0,
    max_total_iters 0 or > 8, and -- training mode only -- N_samples_extra > N_samples_eval (the reference's
    randperm(M)[:X] has only min(X, M) entries after one trip)."""
    d, o = rays(scene, 8)
    bad = [cfg_of(1, 1, 0, 2), cfg_of(16, 17, 4, 2), cfg_of(16, 0, 4, 2), cfg_of(16, 8, -1, 2), cfg_of(16, 8, 4, 0),
           cfg_of(16, 8, 4, 9)]
    for cfg in bad:
        for rng in (None, "train"):
            r = train_rng(dict(cfg, N_samples=max(cfg["N_samples"], 1), N_samples_extra=max(cfg["N_samples_extra"], 0),
                               max_total_iters=min(max(cfg["max_total_iters"], 1), 8)), 8) if rng else None
            out, _ = run(cfg, person["body"], person["field"], d, o, rng=r)
            assert re.search(r"failed \(-\d+\): .*sampler", out["err"] or ""), (cfg, out["err"])
            assert bool((out["z"] == SENTINEL).all()) and out["trips"] == SENTINEL_INT
    cfg = cfg_of(16, 8, 17, 2)
    out, _ = run(cfg, person["body"], person["field"], d, o, rng=train_rng(cfg, 8))
    assert re.search(r"failed \(-\d+\): .*N_samples_extra", out["err"] or ""), out["err"]
    assert bool((out["z"] == SENTINEL).all()) and bool((out["z_eik"] == SENTINEL).all())
    # the same configuration is valid in eval mode (the extras come from linspace(0, M-1, X))
    out, _ = run(cfg, person["body"], person["field"], d, o)
    check_rows(out, cfg, d, o)
    cfg = cfg_of(16, 8, 16, 2)      # X == E is accepted in training mode
    out, _ = run(cfg, person["body"], person["field"], d, o, rng=train_rng(cfg, 8))
    check_rows(out, cfg, d, o, train=True)


@pytest.mark.parametrize("train", [False, True])
def test_every_slot_written_and_workspace_independent(scene, person, train):
    """Outputs prefilled with a sentinel and a workspace of 0xFF bytes: no sentinel survives, and the outputs are
    bit-equal to a run on a zeroed workspace; again after a call with another configuration on the same workspace
    (stale SamplerState, tables and lists).  The u = 0 sample equals near in every eval row, so a merge that sends two
    values to one slot leaves a sentinel here."""
    d, o = rays(scene, 37)
    a = cfg_of(32, 16, 8, 5)
    b = cfg_of(64, 7, 33 if not train else 20, 3, eps=0.05)
    big = cfg_of(64, 64, 64, 8)
    for cfg in (a, b):
        rng = train_rng(cfg, 37, edges=True) if train else None
        ref, ws = run(big, person["body"], person["field"], d, o, rng=train_rng(big, 37) if train else None)
        check_rows(ref, big, d, o, train)
        zero, _ = run(cfg, person["body"], person["field"], d, o, rng=rng, fill=0)
        check_rows(zero, cfg, d, o, train)
        # straight after the other configuration on its workspace, nothing refilled: its SamplerState, tables and lists
        stale, _ = run(cfg, person["body"], person["field"], d, o, rng=rng, ws=ws)
        ff, _ = run(cfg, person["body"], person["field"], d, o, rng=rng, ws=ws, fill=0xFF)
        for out in (stale, ff):
            check_rows(out, cfg, d, o, train)
            assert out["trips"] == zero["trips"]
            for k in ("z", "z_bg") + (("z_eik",) if train else ()):
                assert torch.equal(out[k], zero[k]), k


@pytest.mark.parametrize("R", [1, 7, 8, 9, 31, 33, 63, 65])
def test_ray_order_and_replication(scene, person, R):
    """Per-ray outputs depend on the ray alone: the batch permuted, and replicated 33x so that it spans every SM (and
    block tails of 8 warps), gives bit-equal rows, z_bg and trip count (the set of rays, hence the batch flag, is the
    same)."""
    d, o = rays(scene, R, seed=11)
    cfg = cfg_of(64, 32, 16, 5)
    base, _ = run(cfg, person["body"], person["field"], d, o)
    check_rows(base, cfg, d, o)
    g = torch.Generator().manual_seed(R)
    perm = torch.randperm(R, generator=g)
    pout, _ = run(cfg, person["body"], person["field"], d[perm], o[perm])
    assert pout["trips"] == base["trips"]
    assert torch.equal(pout["z"], base["z"][perm]) and torch.equal(pout["z_bg"], base["z_bg"][perm])
    rep = torch.randperm(33 * R, generator=g)
    src = torch.arange(R).repeat(33)[rep]
    rout, _ = run(cfg, person["body"], person["field"], d[src], o[src])
    assert rout["trips"] == base["trips"]
    assert torch.equal(rout["z"], base["z"][src]) and torch.equal(rout["z_bg"], base["z_bg"][src])


@pytest.mark.parametrize("c", [0.0, -0.02])
def test_engines_bit_equal_on_exact_field(scene, person, c):
    """SDF = c on non-outliers and 4 on outliers, exact on both MLP engines: SIMT and tensor cores give bit-equal
    samples.  c = 0: sign(0) = 0, so d* = 0 everywhere; c = -0.02: the sign changes at the 0.1 shell."""
    from multiply_b200 import engine
    d, o = rays(scene, 70, seed=3)
    f = const_field(person["p"], c)
    outs = {}
    try:
        for eng in ("simt", "tc"):
            engine.set_engine(eng)
            for cfg in (cfg_of(64, 32, 16, 5), cfg_of(33, 33, 1, 8, eps=0.01)):
                out, _ = run(cfg, person["body"], f, d, o)
                check_rows(out, cfg, d, o)
                outs[(eng, cfg["N_samples_eval"])] = out
    finally:
        engine.set_engine("tc")
    for E in (64, 33):
        a, b = outs[("simt", E)], outs[("tc", E)]
        assert a["trips"] == b["trips"] and torch.equal(a["z"], b["z"]) and torch.equal(a["z_bg"], b["z_bg"])


def test_field_sdf_independent_of_row(scene, person):
    """The float64 comparisons evaluate the SDF of each point through mp_sdf_with_deformer, while the sampler evaluates
    its compacted list, so a point sits at another row of the MLP tiles: the tensor-core SDF of a point must not depend
    on its row (checked by evaluating the same points at shifted offsets of a batch)."""
    from multiply_b200 import engine
    engine.set_engine("tc")
    g = torch.Generator().manual_seed(1)
    x = (torch.rand(1000, 3, generator=g) - 0.5) * 0.6
    f = person["field"]
    base, _ = f.implicit_forward(x, want_feat=False)
    for shift in (1, 31, 64, 127):
        pad = (torch.rand(shift, 3, generator=g) - 0.5) * 0.6
        s, _ = f.implicit_forward(torch.cat([pad, x]), want_feat=False)
        assert torch.equal(s[shift:], base), shift


# ---------------------------------------------------------------------------------------------
# float64 comparisons
# ---------------------------------------------------------------------------------------------

LIST_CASES = [(E, S_, X) for E in (2, 3, 31, 32, 33, 64, 128, 256, 512)
              for S_ in sorted({1, max(1, E // 2), E}) for X in (0, 1, 32)]


@pytest.mark.parametrize("E,S_,X", LIST_CASES)
def test_list_and_lane_edges_vs_float64(scene, person, E, S_, X):
    """One trip (max_total_iters = 1: the final set is drawn from the uniform list) at every list size around the 32-lane
    chunking, S in {1, E/2, E}, X in {0, 1, 32}; E = 2, 3 with X = 32 make X + 2 > M, so the shared-memory stride is
    set by X.  Against the float64 port on the GPU's SDF."""
    from multiply_b200 import engine
    engine.set_engine("tc")
    R = 24
    d, o = rays(scene, R, seed=E + S_ + X)
    cfg = cfg_of(E, S_, X, 1)
    gpu, _ = run(cfg, person["body"], person["field"], d, o)
    check_rows(gpu, cfg, d, o)
    _, tr, cb = reference(cfg, person, d, o)
    compare("list", cfg, d, o, gpu["z"], gpu["trips"], tr, cb.dist)


TRIP_CASES = [(32, 16, 8, 1, 0.1), (32, 16, 8, 2, 0.1), (32, 16, 8, 5, 0.1), (32, 16, 8, 8, 0.1),
              (64, 32, 16, 8, 0.1), (64, 32, 16, 5, 1e-3), (64, 32, 16, 8, 1e-3), (128, 64, 32, 5, 10.0),
              (512, 64, 32, 8, 1e-3)]


@pytest.mark.parametrize("E,S_,X,T,eps", TRIP_CASES)
def test_trip_edges_vs_float64(scene, person, E, S_, X, T, eps):
    """Trip caps 1, 2, 5, 8 with eps that converges mid-run (0.1), never (1e-3) and at the first trip (10); E = 512 with
    8 trips reaches M = 4096, the largest per-warp shared-memory footprint.  Also runs the same batch with every cap
    1..T: each cap exposes that trip's state through the final set."""
    from multiply_b200 import engine
    engine.set_engine("tc")
    R = 16 if E < 512 else 6
    d, o = rays(scene, R, seed=100 + E + T)
    caps = range(1, T + 1) if E <= 64 else (T,)
    for cap in caps:
        cfg = cfg_of(E, S_, X, cap, eps=eps)
        gpu, _ = run(cfg, person["body"], person["field"], d, o)
        check_rows(gpu, cfg, d, o)
        _, tr, cb = reference(cfg, person, d, o)
        if eps >= 10.0:
            assert tr["n_trips"] == 1
        if eps <= 1e-3:
            assert tr["n_trips"] == cap
        big = E * cap >= 4096
        compare("trips M=4096" if big else "trips", cfg, d, o, gpu["z"], gpu["trips"], tr, cb.dist,
                mask_max=MASK_MAX_M4096 if big else MASK_MAX_TRIPS)


def test_single_slow_ray_keeps_batch_going(scene, person):
    """Rays that miss the body (SDF 4 everywhere: converged at trip 1) batched with one ray through the body: the slow
    ray's flag keeps every ray going, and the fast rays' later trips must still match float64."""
    from multiply_b200 import engine
    engine.set_engine("tc")
    d, o = rays(scene, 1, seed=7)
    miss_d = torch.tensor([[0.0, 0.0, 1.0], [0.0, 1.0, 0.0], [1.0, 0.0, 0.0], [-0.6, 0.8, 0.0]])
    miss_d = miss_d / miss_d.norm(dim=1, keepdim=True)
    dd = torch.cat([miss_d, d, miss_d])
    oo = o.repeat(dd.shape[0], 1)
    cfg = cfg_of(32, 16, 8, 5)
    gpu, _ = run(cfg, person["body"], person["field"], dd, oo)
    check_rows(gpu, cfg, dd, oo)
    alone, _ = run(cfg, person["body"], person["field"], miss_d, o.repeat(miss_d.shape[0], 1))
    assert alone["trips"] == 1 and gpu["trips"] > 1
    _, tr, cb = reference(cfg, person, dd, oo)
    compare("slow ray", cfg, dd, oo, gpu["z"], gpu["trips"], tr, cb.dist)


def test_geometry_edges(scene, person):
    """Rays that graze the bounding sphere (far ~ near: cameras just inside the r = 3 sphere looking out), a camera outside
    the sphere whose ray line meets it only behind the camera (far clamped to 0: every interval 0), and rays that miss
    the body shell."""
    from multiply_b200 import engine
    engine.set_engine("tc")
    oo, dd = [], []
    for gap in (1e-4, 1e-3, 1e-2):
        for tilt in (0.0, 0.3):
            oo.append(torch.tensor([0.0, 0.0, 3.0 - gap]))
            v = torch.tensor([tilt * gap, 0.0, 1.0])
            dd.append(v / v.norm())
    oo += [torch.tensor([0.0, 0.0, 2.5])] * 2
    dd += [torch.tensor([0.0, 0.0, -1.0]), torch.tensor([0.0, 1.0, 0.0])]
    oo, dd = torch.stack(oo), torch.stack(dd)
    far = far_of(dd.double(), oo.double())
    assert bool((far[:6] < 2e-2).all()) and bool((far[:6] > 0).all()), far
    cfg = cfg_of(32, 16, 8, 5)
    gpu, _ = run(cfg, person["body"], person["field"], dd, oo)
    check_rows(gpu, cfg, dd, oo)
    _, tr, cb = reference(cfg, person, dd, oo)
    compare("geometry", cfg, dd, oo, gpu["z"], gpu["trips"], tr, cb.dist)
    # outside the sphere, looking away from it: under > 0 but both roots behind the camera -> far = 0
    oo2 = torch.tensor([[0.0, 0.0, 5.0]]).repeat(3, 1)
    dd2 = torch.tensor([[0.0, 0.0, 1.0], [0.0, 0.1, 0.995], [0.1, 0.0, 0.995]])
    dd2 = dd2 / dd2.norm(dim=1, keepdim=True)
    out, _ = run(cfg, person["body"], person["field"], dd2, oo2)
    assert out["err"] is None and not bool((out["z"] == SENTINEL).any())
    assert bool((out["z"] == 0).all()), "far clamped to 0 must give a row of zeros"


# ---------------------------------------------------------------------------------------------
# training mode
# ---------------------------------------------------------------------------------------------

@pytest.mark.parametrize("T", [1, 2, 3, 5, 8])
def test_training_rows_of_the_trip_count(scene, person, T):
    """Distinct draws in every per-trip row, the trip count forced by the cap (eps = 1e-3 never converges): z_bg must be
    bit-equal to the jittered inverse-sphere depths of row T-1, and z_eik to z_vals[eik_idx[T-1]].  t_rand / u_final
    hold exact 0 and 1 - 2^-24, so stratified samples tie with near and with each other (the rank sort's tie rule), and
    eik_idx = S + X + 1 picks the last slot."""
    R = 21
    d, o = rays(scene, R, seed=40 + T)
    cfg = cfg_of(32, 16, 8, T, eps=1e-3)
    rng = train_rng(cfg, R, seed=T, edges=True)
    out, _ = run(cfg, person["body"], person["field"], d, o, rng=rng)
    check_rows(out, cfg, d, o, train=True)
    assert out["trips"] == T
    row = T - 1
    tb = torch.linspace(0., 1., steps=32)
    z_bg = torch.zeros(R, 1) * (1. - tb) + torch.ones(R, 1) * tb
    mids = .5 * (z_bg[..., 1:] + z_bg[..., :-1])
    upper = torch.cat([mids, z_bg[..., -1:]], -1)
    lower = torch.cat([z_bg[..., :1], mids], -1)
    z_bg = (lower + (upper - lower) * rng["t_rand_bg"][row]) * (1. / 3.0)
    assert torch.equal(out["z_bg"], z_bg)
    eik = out["z"].gather(1, rng["eik_idx"][row].long()[:, None])[:, 0]
    assert torch.equal(out["z_eik"], eik)
    # ties: t_rand = 0 at sample 0 makes the first stratified sample equal near; u_final = 0 draws z[0] again
    z = out["z"]
    assert bool((z[:, 1] == 0).all()), "the tied samples at near must all be kept"


def train_callback(body, field):
    """ray_sdf_fn of the training sampler: fp32 points as deform_rays_kernel forms them, the exact inverse deformer and
    the field's SDF, no outlier clamp (multiply.py:142 is eval-only)."""
    def fn(o, z, d):
        o32, z32, d32 = o.float(), z.float(), d.float()
        x = (o32.unsqueeze(1) + (z32.unsqueeze(2) * d32.unsqueeze(1))).reshape(-1, 3).contiguous()
        xc, _ = body.deform_inverse(x.cuda(), exact_far=True)
        sdf, _ = field.implicit_forward(xc, want_feat=False)
        return sdf.cpu().double()[:, None]
    return fn


@pytest.mark.parametrize("T", [1, 2, 3, 5])
@pytest.mark.parametrize("edges", [False, True])
def test_training_vs_float64(scene, person, T, edges):
    """Training-mode z_vals against the float64 port fed the draws of row T-1 (the trip count forced by the cap): the
    extras are z[:, extra_perm[T-1][:X]] of the float64 list, so a wrong row or stride of the per-trip draws moves them
    by whole intervals.  With edges, t_rand / u_final hold exact 0 and 1 - 2^-24."""
    from multiply_b200 import engine
    engine.set_engine("tc")
    R = 16
    d, o = rays(scene, R, seed=60 + T)
    cfg = cfg_of(32, 16, 8, T, eps=1e-3)
    rng = train_rng(cfg, R, seed=10 + T, edges=edges)
    out, _ = run(cfg, person["body"], person["field"], d, o, rng=rng)
    check_rows(out, cfg, d, o, train=True)
    row = T - 1
    perm = rng["extra_perm"][row, :T * cfg["N_samples_eval"]]
    rng64 = dict(t_rand=rng["t_rand"], u_final=rng["u_final"], extra_perm=perm, eik_idx=rng["eik_idx"][row],
                 t_rand_bg=rng["t_rand_bg"][row])
    tr, st = {}, {}
    port.error_bound_get_z_vals(d.double(), o.double(), None, cfg, cfg["beta_param"], stats=st, rng=rng64,
                                dtype=torch.float64, ray_sdf_fn=train_callback(person["body"], person["field"]), trace=tr)
    tr["n_trips"] = st["trips"]
    assert st["trips"] == T
    compare("train", cfg, d, o, out["z"], out["trips"], tr, None, extra_idx=perm[:cfg["N_samples_extra"]])
