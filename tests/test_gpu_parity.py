"""GPU parity tests: the CUDA path (through the C ABI) against the golden outputs of the
unmodified reference (tests/golden) and against the CPU oracle on the same seeded inputs.
Tolerance: 1e-4 L-inf on RGB / SDF (BASELINE.json north_star), stated per assertion."""
import os
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from multiply_b200 import scene as S


def _g(golden_dir, name):
    return np.load(os.path.join(golden_dir, name + ".npz"))


ENGINES = ["simt", "tc"]
# Network-level tolerance (absolute, outputs are O(1)): the fp32 SIMT engine agrees with the CPU
# reference to rounding; the tensor-core engine (fp16 hi/lo operands, fp32 accumulation inside the tensor
# core, whose round-toward-zero is compensated in the epilogue, mlp_tc.cu:kRzPerMma) to ~2e-6 — both far
# inside the 1e-4 gate of north_star.
TOL_NET = {"simt": 1e-5, "tc": 2e-5}
# Rendered normals (an output of Multiply.forward, multiply.py:597): 1e-4 on both engines.  They amplify the
# gradient error by 1 / |grad sdf . J^-1|, which is what the uncompensated tensor-core engine of round 1 failed
# on (4.8e-4); with the compensation the measured value is 3e-6.
TOL_NORMAL = {"simt": 1e-4, "tc": 1e-4}


@pytest.fixture(scope="module")
def scene64():
    return S.make_scene(P=2, S=64, seed=42)


@pytest.fixture(scope="module")
def field0(scene64):
    from multiply_b200 import engine
    p0 = scene64["persons"][0]
    f = engine.Field(p0["implicit"], p0["render"])
    f.set_cond(p0["cond"])
    return f


def _maxabs(a, b):
    return float(np.abs(np.asarray(a, dtype=np.float64) - np.asarray(b, dtype=np.float64)).max())


@pytest.mark.parametrize("eng", ENGINES)
def test_implicit_forward(golden_dir, field0, eng):
    from multiply_b200 import engine
    engine.set_engine(eng)
    g = _g(golden_dir, "implicit_fg")
    sdf, feat = field0.implicit_forward(torch.from_numpy(g["x"]))
    torch.cuda.synchronize()
    tol = TOL_NET[eng]
    assert _maxabs(sdf.cpu().numpy(), g["out"][:, 0]) < tol
    assert _maxabs(feat.cpu().numpy(), g["out"][:, 1:]) < tol
    sdf2, _ = field0.implicit_forward(torch.from_numpy(g["x"]), want_feat=False)
    assert _maxabs(sdf2.cpu().numpy(), g["out"][:, 0]) < tol


@pytest.mark.parametrize("eng", ENGINES)
def test_implicit_grad(golden_dir, field0, eng):
    from multiply_b200 import engine
    engine.set_engine(eng)
    g = _g(golden_dir, "implicit_fg_grad")
    _, _, grad = field0.implicit_forward(torch.from_numpy(g["x"]), want_grad=True)
    assert _maxabs(grad.cpu().numpy(), g["grad"]) < 2 * TOL_NET[eng]


def test_camera_rays_and_sphere(golden_dir):
    """a1 / a2 at the operator level: mp_camera_rays and mp_sphere_intersections against what the reference's own
    rend_util.get_camera_params / get_sphere_intersections computed (skewed off-centre intrinsics, rotated camera)."""
    from multiply_b200.model import rend_util
    g = _g(golden_dir, "rays")
    dirs, cam = rend_util.get_camera_params(torch.from_numpy(g["uv"]).cuda(), torch.from_numpy(g["pose"]).cuda(),
                                            torch.from_numpy(g["intrinsics"]).cuda())
    assert dirs.shape == (1, 300, 3) and cam.shape == (1, 3)
    assert _maxabs(dirs.cpu().numpy(), g["ray_dirs"]) < 2e-7
    assert _maxabs(cam.cpu().numpy(), g["cam_loc"]) == 0.0
    cam_r = cam.expand(300, 3).contiguous()
    nf = rend_util.get_sphere_intersections(cam_r, torch.from_numpy(g["ray_dirs"][0]).cuda(), r=3.0)
    assert _maxabs(nf.cpu().numpy(), g["near_far"]) < 2e-6
    # a camera outside the sphere: the reference exits (rend_util.py:140-142), the mirror raises
    with pytest.raises(RuntimeError):
        rend_util.get_sphere_intersections(cam_r + torch.tensor([50.0, 0.0, 0.0], device="cuda"),
                                           torch.from_numpy(g["ray_dirs"][0]).cuda(), r=3.0)


@pytest.mark.parametrize("eng", ENGINES)
def test_background_nets(golden_dir, scene64, eng):
    """a12 at the operator level: bg ImplicitNet (d_in 4, multires 10, frame cond) + bg RenderingNet
    ('nerf_frame_encoding') through mp_bg_nets_forward against the reference modules' outputs."""
    from multiply_b200 import engine
    engine.set_engine(eng)
    g = _g(golden_dir, "bg_nets")
    f = engine.Field(scene64["bg_implicit"], scene64["bg_render"], background=True)
    f.set_cond(scene64["frame_code"])
    sdf, rgb = f.bg_forward(torch.from_numpy(g["x"]), torch.from_numpy(g["view"]))
    torch.cuda.synchronize()
    assert _maxabs(sdf.cpu().numpy(), g["out"][:, 0]) < TOL_NET[eng]
    assert _maxabs(rgb.cpu().numpy(), g["rgb"]) < TOL_NET[eng]
    sdf2, feat = f.implicit_forward(torch.from_numpy(g["x"]))
    assert _maxabs(sdf2.cpu().numpy(), g["out"][:, 0]) < TOL_NET[eng]
    assert _maxabs(feat.cpu().numpy(), g["out"][:, 1:]) < TOL_NET[eng]


@pytest.mark.parametrize("eng", ENGINES)
def test_sdf_grid(golden_dir, scene64, eng):
    """f3: canonical SDF on the dense lattice of generate_mesh (mp_sdf_grid: points generated on the device, streamed
    through the sdf-only program) against the reference's Multiply.query_oc on the same lattice; the lattice points
    themselves are bit-equal to numpy's (checked through a second query at the golden points)."""
    from multiply_b200 import engine
    engine.set_engine(eng)
    g = _g(golden_dir, "sdf_grid")
    p1 = scene64["persons"][1]
    f = engine.Field(p1["implicit"], p1["render"])
    f.set_cond(p1["cond"])
    res = int(g["res"])
    vals = f.sdf_grid(g["center"], float(g["extent"]), res)
    torch.cuda.synchronize()
    assert vals.shape == (res + 1,) * 3
    assert _maxabs(vals.cpu().numpy().reshape(-1), g["occ"]) < TOL_NET[eng]
    direct, _ = f.implicit_forward(torch.from_numpy(g["points"]), want_feat=False)
    assert torch.equal(direct, vals.reshape(-1))           # same points bit for bit -> same SDF bit for bit


def test_sphere_status_flag():
    """mp_render_rays reports a camera outside the bounding sphere through mp_render_out_t.status; the Renderer raises
    where the reference exits."""
    from multiply_b200 import engine
    engine.set_engine("tc")
    sc = S.make_scene(P=1, S=16, seed=42)
    inp = S.make_rays(sc, 16, seed=2, region="boxes")
    hits = S.make_hit_lists(sc, inp)
    r = engine.Renderer(sc)
    r.render(inp, hits, check=True)
    far = dict(inp, pose=inp["pose"].clone())
    far["pose"][0, 0, 3] = 10.0            # camera moved sideways: its rays pass the r = 3 sphere by
    with pytest.raises(RuntimeError, match="BOUNDING SPHERE"):
        r.render(far, hits, check=True)


def test_render_forward(golden_dir, field0):
    g = _g(golden_dir, "render_fg")
    rgb = field0.render_forward(torch.from_numpy(g["x"]), torch.from_numpy(g["normals"]), torch.from_numpy(g["feat"]))
    assert _maxabs(rgb.cpu().numpy(), g["rgb"]) < 1e-5


def test_deformer(golden_dir, scene64):
    from multiply_b200 import engine
    g = _g(golden_dir, "deformer")
    p0 = scene64["persons"][0]
    b = engine.Body(p0["verts_c"], p0["weights"], cano_cell=0.2)
    b.set_pose(p0["verts_p"], p0["tfs"])
    xc, outl = b.deform_inverse(torch.from_numpy(g["pts"]))
    assert np.array_equal(outl.cpu().numpy(), g["outlier"])
    assert _maxabs(xc.cpu().numpy(), g["x_c"]) < 1e-5
    xd, J = b.forward_jac(torch.from_numpy(g["x_c"]))
    assert _maxabs(xd.cpu().numpy(), g["x_d"]) < 1e-5
    # grid path == brute force (exact_far) on non-outliers when the far scan is disabled
    xc2, outl2 = b.deform_inverse(torch.from_numpy(g["pts"]), exact_far=False)
    m = ~g["outlier"]
    assert np.array_equal(outl2.cpu().numpy(), g["outlier"])
    assert _maxabs(xc2.cpu().numpy()[m], g["x_c"][m]) < 1e-5


def test_deform_broyden(scene64):
    """Row f4 (non-default; the reference has no root finder): mp_deform_broyden against oracle/port.py:deform_broyden."""
    from multiply_b200 import engine
    from oracle import port
    p1 = scene64["persons"][1]
    g = torch.Generator().manual_seed(0)
    v = p1["verts_p"]
    x = v[torch.randint(0, v.shape[0], (6000,), generator=g)] + 0.04 * torch.randn(6000, 3, generator=g)
    b = engine.Body(p1["verts_c"], p1["weights"], cano_cell=0.2)
    b.set_pose(p1["verts_p"], p1["tfs"])
    xc0, outl0 = b.deform_inverse(x)
    o = b.deform_broyden(x, 10, 1e-5)
    ref_xc, ref_res, ref_conv, ref_out = port.deform_broyden(x, p1, 10, 1e-5)
    assert torch.equal(o["outlier"].cpu(), ref_out) and torch.equal(outl0.cpu(), ref_out)
    # the reported residual is the residual of the returned point (forward skinning on the device)
    xd, _ = b.forward_jac(o["x_c"])
    assert float(((xd - x.cuda()).norm(dim=-1) - o["residual"]).abs().max()) < 2e-6
    # consistent points (closed-form residual below the threshold) take no step and are bit-equal to mp_deform_inverse
    still = o["steps"] == 0
    assert 0.3 < float(still.float().mean()) < 0.95
    assert torch.equal(o["x_c"][still], xc0[still])
    assert bool((o["residual"][still] < 1e-5).all())
    # against the CPU statement: same verdicts, same roots
    conv = o["converged"].cpu()
    assert float((conv == ref_conv).float().mean()) > 0.995
    both = conv & ref_conv
    assert float(both.float().mean()) > 0.85
    assert float((o["x_c"].cpu()[both] - ref_xc[both]).abs().max()) < 1e-4
    assert float((o["x_c"].cpu() - ref_xc).abs().max(dim=-1)[0].gt(1e-4).float().mean()) < 0.01
    # the switch: every inverse-deformer call refines non-outliers, outliers keep the closed form
    b.set_root_finder(10, 1e-5)
    xc1, outl1 = b.deform_inverse(x)
    m = ~outl1
    assert torch.equal(outl1, outl0)
    assert torch.equal(xc1[m], o["x_c"][m]) and torch.equal(xc1[~m], xc0[~m])
    b.set_root_finder(0)
    assert torch.equal(b.deform_inverse(x)[0], xc0)


@pytest.mark.parametrize("eng", ENGINES)
def test_forward_with_root_finder(eng):
    """The whole path with the root finder switched on for every body (sampler, main pass, normals at the refined
    canonical points) against the oracle with the same switch."""
    from multiply_b200 import engine
    from oracle import port
    engine.set_engine(eng)
    sc = S.make_scene(P=2, S=16, seed=42)
    inp = S.make_rays(sc, 128, seed=9, region="boxes")
    hits = S.make_hit_lists(sc, inp)
    sc_ref = dict(sc, persons=[dict(p, root_finder=(10, 1e-5)) for p in sc["persons"]])
    ref = port.multiply_forward(sc_ref, inp, hits)
    plain = port.multiply_forward(sc, inp, hits)
    r = engine.Renderer(sc)
    for b in r.bodies:
        b.set_root_finder(10, 1e-5)
    o = r.render(inp, hits)
    torch.cuda.synchronize()
    assert _maxabs(ref["rgb_values"].numpy(), plain["rgb_values"].numpy()) > 1e-3      # the switch matters here
    for k in ("rgb_values", "acc_map", "normal_values"):
        d = np.abs(o[k].cpu().numpy() - ref[k].numpy()).reshape(128, -1).max(1)
        assert (d > 1e-4).mean() < 0.03, (k, float(d.max()), float((d > 1e-4).mean()))
        assert np.median(d) < 1e-5, k


def test_density(golden_dir):
    from multiply_b200 import _lib as L
    g = _g(golden_dir, "density")
    s = torch.from_numpy(g["sdf"]).cuda()
    out = torch.empty_like(s)
    L.call("mp_laplace_density", s, s.numel(), float(g["beta"]), out)
    assert _maxabs(out.cpu().numpy(), g["sigma"]) < 1e-6 * max(1.0, float(np.abs(g["sigma"]).max()))


def _check_forward(o, g, eng, tol=1e-4):
    for k in ("rgb_values", "fg_rgb_values", "acc_map", "acc_person_list"):
        assert _maxabs(o[k].cpu().numpy(), g[k]) < tol, k
    assert _maxabs(o["normal_values"].cpu().numpy(), g["normal_values"]) < TOL_NORMAL[eng]
    for p in range(2):
        z = o[f"z_vals_{p}"].cpu().numpy()[:, :-1]
        assert _maxabs(z, g[f"z_vals_{p}"]) < 1e-3
        m = np.abs(z - g[f"z_vals_{p}"]) < 1e-6          # SDF is comparable where both sampled the same depth
        assert m.mean() > 0.5
        assert float(np.abs(o[f"sdf_{p}"].cpu().numpy() - g[f"sdf_{p}"])[m].max()) < 1e-4


def _render_golden(eng, name, Sn, R, region, golden_dir):
    from multiply_b200 import engine
    engine.set_engine(eng)
    g = _g(golden_dir, name)
    sc = S.make_scene(P=2, S=Sn, seed=42)
    inp = S.make_rays(sc, R, seed=1234, region=region)
    hits = S.make_hit_lists(sc, inp)
    r = engine.Renderer(sc)
    o = r.render(inp, hits, debug=True)
    torch.cuda.synchronize()
    assert list(o["trips"].cpu().numpy()) == list(g["trips"])
    return o, g


@pytest.mark.parametrize("eng", ENGINES)
def test_forward_golden(golden_dir, eng):
    """End-to-end Multiply.forward (eval, shipped sampler sizes 64/128/32) against what the unmodified
    reference computed: RGB / acc / per-sample SDF within 1e-4."""
    o, g = _render_golden(eng, "forward_S64_R48", 64, 48, "boxes", golden_dir)
    _check_forward(o, g, eng)


@pytest.mark.parametrize("eng", ENGINES)
def test_forward_golden_coarse_sampler(golden_dir, eng):
    """Stress case S/E/X = 16/32/8, five Algorithm-1 trips.  With 32 coarse bins the inverse-CDF step divides by
    cdf differences of ~1e-5, which amplifies 1e-7 rounding differences to ~1e-3 in z (the CPU restatement and
    the reference themselves differ by 3e-5 in z here, tests/test_oracle_golden.py), and a sample that lands on
    the 0.1 outlier radius (deformer.py:49) flips between sdf = 4 and the network value.  The discontinuity
    is the reference's; the test therefore bounds the bulk: trip counts equal, >= 90 % of the rays within 1e-4
    and nothing wildly off."""
    o, g = _render_golden(eng, "forward_S16_R96", 16, 96, "image", golden_dir)
    err = np.abs(o["rgb_values"].cpu().numpy() - g["rgb_values"]).max(1)
    assert (err < 1e-4).mean() >= 0.90, float((err < 1e-4).mean())
    assert err.max() < 5e-2
    for p in range(2):
        dz = np.abs(o[f"z_vals_{p}"].cpu().numpy()[:, :-1] - g[f"z_vals_{p}"])
        assert np.median(dz) < 1e-5 and dz.max() < 5e-3


def _sdf_where_z_agrees(o, ref, p):
    """Per-sample SDF is only comparable where both sides sampled the same depth."""
    z = o[f"z_vals_{p}"].cpu().numpy()[:, :-1]
    zr = ref["_z_vals"][p].numpy()
    m = np.abs(z - zr) < 1e-6
    assert m.mean() > 0.5
    return float(np.abs(o[f"sdf_{p}"].cpu().numpy() - ref["_sdf"][p].numpy())[m].max())


@pytest.mark.parametrize("eng", ENGINES)
def test_forward_vs_oracle(eng):
    """Shipped sampler sizes (S/E/X = 64/128/32), 256 rays, against the CPU oracle (oracle/port.py) run on
    this machine: every output of Multiply.forward within 1e-4."""
    from multiply_b200 import engine
    from oracle import port
    engine.set_engine(eng)
    sc = S.make_scene(P=2, S=64, seed=42)
    inp = S.make_rays(sc, 256, seed=5, region="boxes")
    hits = S.make_hit_lists(sc, inp)
    st = {}
    ref = port.multiply_forward(sc, inp, hits, stats=st, return_samples=True)
    r = engine.Renderer(sc)
    o = r.render(inp, hits, debug=True)
    torch.cuda.synchronize()
    assert list(o["trips"].cpu().numpy()) == list(st["trips"])
    for k in ("rgb_values", "fg_rgb_values", "normal_values", "acc_map", "acc_person_list"):
        assert _maxabs(o[k].cpu().numpy(), ref[k].numpy()) < 1e-4, k
    for p in range(2):
        assert _sdf_where_z_agrees(o, ref, p) < 1e-4


def test_forward_config1_scale():
    """BASELINE configs[1] sampler sizes (S/E/X = 128/256/64, n = 193 main-pass samples, 2 persons) on 512 rays of
    the benchmark batch against the CPU oracle: trips equal, every output of Multiply.forward within 1e-4, per-sample
    SDF within 1e-4 wherever both sides sampled the same depth."""
    from multiply_b200 import engine
    from oracle import port
    engine.set_engine("tc")
    torch.set_num_threads(min(32, os.cpu_count() or 8))
    sc = S.make_scene(P=2, S=128, seed=42)
    full = S.make_rays(sc, 4096, seed=1234, region="boxes")
    inp = dict(uv=full["uv"][:, :512].contiguous(), pose=full["pose"], intrinsics=full["intrinsics"])
    hits = S.make_hit_lists(sc, inp)
    st = {}
    ref = port.multiply_forward(sc, inp, hits, stats=st, return_samples=True)
    o = engine.Renderer(sc).render(inp, hits, debug=True)
    torch.cuda.synchronize()
    assert list(o["trips"].cpu().numpy()) == list(st["trips"])
    for k in ("rgb_values", "fg_rgb_values", "acc_map", "acc_person_list"):
        assert _maxabs(o[k].cpu().numpy(), ref[k].numpy()) < 1e-4, k
    assert _maxabs(o["normal_values"].cpu().numpy(), ref["normal_values"].numpy()) < TOL_NORMAL["tc"]
    for p in range(2):
        assert _sdf_where_z_agrees(o, ref, p) < 1e-4


@pytest.mark.parametrize("eng", ENGINES)
def test_forward_vs_oracle_coarse(eng):
    """S/E/X = 32/64/16 (five trips): RGB still within 1e-4; the opacity / normal maps inherit the ~1e-3
    depth jitter of the coarse inverse-CDF step (see test_forward_golden_coarse_sampler) and get 5e-4."""
    from multiply_b200 import engine
    from oracle import port
    engine.set_engine(eng)
    sc = S.make_scene(P=2, S=32, seed=42)
    inp = S.make_rays(sc, 384, seed=77, region="boxes")
    hits = S.make_hit_lists(sc, inp)
    st = {}
    ref = port.multiply_forward(sc, inp, hits, stats=st, return_samples=True)
    o = engine.Renderer(sc).render(inp, hits, debug=True)
    torch.cuda.synchronize()
    assert list(o["trips"].cpu().numpy()) == list(st["trips"])
    assert _maxabs(o["rgb_values"].cpu().numpy(), ref["rgb_values"].numpy()) < 1e-4
    for k in ("fg_rgb_values", "normal_values", "acc_map", "acc_person_list"):
        assert _maxabs(o[k].cpu().numpy(), ref[k].numpy()) < 5e-4, k


def test_precision_modes():
    """mp_set_precision: 'colour1' (single-term colour layers) leaves SDF / normals bit-identical to the parity mode and
    keeps RGB inside the 1e-4 gate; 'throughput' (plain fp16 operands everywhere) is outside the gate but sane."""
    from multiply_b200 import engine
    from oracle import port
    engine.set_engine("tc")
    sc = S.make_scene(P=2, S=64, seed=42)
    inp = S.make_rays(sc, 256, seed=5, region="boxes")
    hits = S.make_hit_lists(sc, inp)
    ref = port.multiply_forward(sc, inp, hits)
    r = engine.Renderer(sc)
    try:
        outs = {}
        for mode in ("parity", "colour1", "throughput"):
            engine.set_precision(mode)
            outs[mode] = {k: v.clone() for k, v in r.render(inp, hits, debug=True).items()}
            torch.cuda.synchronize()
    finally:
        engine.set_precision("parity")
    for p in range(2):
        assert torch.equal(outs["colour1"][f"sdf_{p}"], outs["parity"][f"sdf_{p}"])
        assert torch.equal(outs["colour1"][f"normals_{p}"], outs["parity"][f"normals_{p}"])
    for mode in ("parity", "colour1"):
        assert _maxabs(outs[mode]["rgb_values"].cpu().numpy(), ref["rgb_values"].numpy()) < 1e-4, mode
        assert _maxabs(outs[mode]["acc_map"].cpu().numpy(), ref["acc_map"].numpy()) < 1e-4, mode
    t = outs["throughput"]
    assert bool(torch.isfinite(t["rgb_values"]).all())
    assert _maxabs(t["rgb_values"].cpu().numpy(), ref["rgb_values"].numpy()) < 2e-2


def test_empty_hit_list_and_single_person():
    """Edge cases of multiply.py:262-263 (empty hit list -> ray 0) vs the oracle."""
    from multiply_b200 import engine
    from oracle import port
    engine.set_engine("simt")
    sc = S.make_scene(P=2, S=16, seed=42)
    inp = S.make_rays(sc, 64, seed=5, region="image")
    hits = S.make_hit_lists(sc, inp)
    hits[1] = torch.zeros(0, dtype=torch.int64)
    ref = port.multiply_forward(sc, inp, hits)
    o = engine.Renderer(sc).render(inp, hits)
    torch.cuda.synchronize()
    for k in ("rgb_values", "normal_values", "acc_map", "acc_person_list"):
        assert _maxabs(o[k].cpu().numpy(), ref[k].numpy()) < 1e-4, k


@pytest.mark.parametrize("P,Sn,R", [(3, 256, 40), (6, 32, 64)])
def test_more_persons_and_samples(P, Sn, R):
    """BASELINE configs 3 and 5 shapes at test size: 3 persons with 256 samples/ray (S/E/X = 256/512/128,
    n = 385) and 6 persons; all rays hit every person (worst case of SURVEY.md §8d)."""
    from multiply_b200 import engine
    from oracle import port
    engine.set_engine("tc")
    torch.set_num_threads(min(32, torch.get_num_threads()))
    sc = S.make_scene(P=P, S=Sn, seed=42)
    inp = S.make_rays(sc, R, seed=9, region="boxes")
    hits = S.make_hit_lists(sc, inp, all_hit=True)
    st = {}
    ref = port.multiply_forward(sc, inp, hits, stats=st)
    o = engine.Renderer(sc).render(inp, hits, debug=True)
    torch.cuda.synchronize()
    assert list(o["trips"].cpu().numpy()) == list(st["trips"])
    assert o["acc_person_list"].shape == (R, P)
    tol = 1e-4 if Sn >= 64 else 5e-4
    for k in ("rgb_values", "fg_rgb_values", "acc_map", "acc_person_list"):
        assert _maxabs(o[k].cpu().numpy(), ref[k].numpy()) < tol, k


def test_branch_streams_match_single_stream():
    """mp_render_rays runs persons and background on their own streams (joined before the compositor); the result
    must be bit-identical to the single-stream schedule, call after call (workspace reuse across calls)."""
    from multiply_b200 import engine, _lib as L
    engine.set_engine("tc")
    sc = S.make_scene(P=3, S=64, seed=7)
    inp = S.make_rays(sc, 300, seed=3, region="boxes")
    hits = S.make_hit_lists(sc, inp)
    r = engine.Renderer(sc)
    try:
        L.call("mp_set_streams", 0)
        ref = {k: v.clone() for k, v in r.render(inp, hits).items()}
        torch.cuda.synchronize()
        L.call("mp_set_streams", 1)
        for _ in range(3):
            o = r.render(inp, hits)
            torch.cuda.synchronize()
            for k in ("rgb_values", "fg_rgb_values", "normal_values", "acc_map", "acc_person_list"):
                assert torch.equal(o[k], ref[k]), k
    finally:
        L.call("mp_set_streams", 1)


def test_edge_cases_single_ray_and_no_hits():
    """R = 1, and a batch in which no ray hits any box (every hit list empty -> ray 0, multiply.py:262-263):
    the outputs equal the oracle's and untouched rays are pure background (acc 0, bg_T 1)."""
    from multiply_b200 import engine
    from oracle import port
    engine.set_engine("tc")
    sc = S.make_scene(P=2, S=16, seed=42)
    one = S.make_rays(sc, 1, seed=2, region="boxes")
    hits = S.make_hit_lists(sc, one)
    ref = port.multiply_forward(sc, one, hits)
    o = engine.Renderer(sc).render(one, hits)
    torch.cuda.synchronize()
    assert _maxabs(o["rgb_values"].cpu().numpy(), ref["rgb_values"].numpy()) < 1e-4
    # rays in an image corner miss both boxes
    K, pose = S.make_camera()
    uv = torch.rand(1, 33, 2, generator=torch.Generator().manual_seed(4)) * 6.0
    inp = dict(uv=uv, pose=pose, intrinsics=K)
    hits = S.make_hit_lists(sc, inp)
    assert all(h.numel() == 0 for h in hits)
    ref = port.multiply_forward(sc, inp, hits)
    o = engine.Renderer(sc).render(inp, hits, debug=True)
    torch.cuda.synchronize()
    for k in ("rgb_values", "fg_rgb_values", "acc_map", "acc_person_list"):
        assert _maxabs(o[k].cpu().numpy(), ref[k].numpy()) < 1e-4, k
    assert float(o["acc_map"][1:].abs().max()) == 0.0 and float((o["bg_T"][1:] - 1).abs().max()) == 0.0


def test_abi_reports_errors():
    """Error convention of the C ABI: negative status + mp_last_error(), nothing thrown, nothing written."""
    import ctypes as C
    from multiply_b200 import _lib as L, engine
    lib = L.lib()
    sc = S.make_scene(P=1, S=16, seed=42)
    r = engine.Renderer(sc)
    c = engine.sampler_cfg(sc["cfg"], 0.1)
    d = torch.zeros(8, 3, device="cuda")
    z = torch.zeros(8, 16 + 8 + 2, device="cuda")
    tiny = torch.empty(64, dtype=torch.uint8, device="cuda")
    rc = lib.mp_sample_rays(C.byref(c), r.bodies[0].handle, r.fields[0].handle, d.data_ptr(), d.data_ptr(), 8, z.data_ptr(),
                            None, None, tiny.data_ptr(), tiny.numel(), L.stream_ptr())
    assert rc != 0 and b"workspace too small" in lib.mp_last_error()
    rc = lib.mp_sample_rays(C.byref(c), None, r.fields[0].handle, d.data_ptr(), d.data_ptr(), 8, z.data_ptr(), None, None,
                            tiny.data_ptr(), tiny.numel(), L.stream_ptr())
    assert rc != 0 and b"null argument" in lib.mp_last_error()
    with pytest.raises(L.MpError):
        L.check(rc, "mp_sample_rays")


def test_call_refuses_a_strided_tensor():
    """``_lib.call`` checks every tensor before the library is entered: a transposed (non-contiguous) CUDA tensor raises
    MpError naming the function and the argument, and nothing is enqueued."""
    from multiply_b200 import _lib as L
    s = torch.rand(4, 6, device="cuda").t()
    out = torch.empty(24, device="cuda")
    before = L.call("mp_launch_count", 0)
    with pytest.raises(L.MpError, match="mp_laplace_density, argument 0: expected a contiguous tensor"):
        L.call("mp_laplace_density", s, 24, 0.1, out)
    assert L.call("mp_launch_count", 0) == before
    L.call("mp_laplace_density", s.contiguous(), 24, 0.1, out)
    assert L.call("mp_launch_count", 0) > before
