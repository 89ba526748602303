"""GPU: the host-side mirror of the reference operator surface (multiply_b200/model) — same class names,
constructor options, state-dict keys and forward signatures as /root/reference/code/lib/model — checked
against the CPU oracle and against the fused Renderer."""
import math
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from multiply_b200 import scene as S     # noqa: E402

from _setups import mirror_inputs       # noqa: E402

@pytest.mark.parametrize("pid", [-1, 0, 1])
@pytest.mark.parametrize("device_culling", [False, True])
def test_multiply_forward_drop_in(pid, device_culling):
    """Multiply.forward(input, id) with the reference's input dict (SURVEY.md §8b) == oracle.  id = -1 renders both
    persons, id = p only person p (multiply.py:244-247: person_list = [id], acc_person_list is [R,1]); with
    device_culling the hit lists are not passed in but computed on the GPU (box, slab test, compaction, empty-list
    rule) with the count left on the device."""
    from multiply_b200 import engine
    from oracle import port
    engine.set_engine("tc")
    sc = S.make_scene(P=2, S=16, seed=42)
    inp = S.make_rays(sc, 96, seed=11, region="boxes")
    hits = S.make_hit_lists(sc, inp)
    plist = [0, 1] if pid == -1 else [pid]
    sub = dict(sc, persons=[sc["persons"][p] for p in plist])
    ref = port.multiply_forward(sub, inp, [hits[p] for p in plist])
    m = S.mirror_model(sc)
    inputs = mirror_inputs(inp, 2, None if device_culling else [h.cuda() for h in hits])
    out = m(inputs, id=pid)
    torch.cuda.synchronize()
    assert set(out) == {"acc_map", "acc_person_list", "rgb_values", "fg_rgb_values", "normal_values"}
    assert out["acc_person_list"].shape == (96, len(plist))
    for k in ("rgb_values", "fg_rgb_values", "acc_map", "acc_person_list"):
        assert float((out[k].cpu() - ref[k]).abs().max()) < 1e-4, k
    # a second call (cached renderer, new pose upload) gives the same pixels
    out2 = m(inputs, id=pid)
    torch.cuda.synchronize()
    assert torch.equal(out2["rgb_values"], out["rgb_values"])


def test_multiply_forward_canonical_pose():
    """canonical_pose=True (multiply.py:196-201): bodies at zero translation in the canonical hip pose, the pose
    conditioning of the networks still from smpl_pose (:270)."""
    from multiply_b200 import engine
    from oracle import port
    engine.set_engine("tc")
    sc = S.make_scene(P=2, S=16, seed=42)
    m = S.mirror_model(sc)
    P = 2
    cpose = torch.zeros(1, 72)
    cpose[0, 5], cpose[0, 8] = math.pi / 6, -math.pi / 6
    persons = []
    for p in range(P):
        o = S.SyntheticSMPLServer(p, P)(torch.tensor([0.5]), torch.zeros(1, 3), cpose, torch.zeros(1, 10))
        persons.append(dict(sc["persons"][p], verts_p=o["smpl_verts"][0], tfs=o["smpl_tfs"][0]))
    csc = dict(sc, persons=persons)
    inp = S.make_rays(csc, 80, seed=13, region="boxes")
    hits = S.make_hit_lists(csc, inp)
    assert sum(h.numel() for h in hits) > 40
    ref = port.multiply_forward(csc, inp, hits)
    out = m(mirror_inputs(inp, P, [h.cuda() for h in hits]), canonical_pose=True)
    torch.cuda.synchronize()
    for k in ("rgb_values", "fg_rgb_values", "acc_map", "acc_person_list"):
        assert float((out[k].cpu() - ref[k]).abs().max()) < 1e-4, k


def test_device_culling_matches_host():
    """mp_ray_aabb_hits (box from the posed vertices on the device, fp64 slab test, ordered compaction, empty -> ray 0)
    against the host slab test of scene.make_hit_lists on 5000 rays; count stays on the device."""
    from multiply_b200 import engine
    from multiply_b200.model import rend_util
    sc = S.make_scene(P=2, S=16, seed=42)
    inp = S.make_rays(sc, 5000, seed=3, region="image")
    dirs, cam = rend_util.get_camera_params_host(inp["uv"], inp["pose"], inp["intrinsics"])
    ref = S.make_hit_lists(sc, inp)
    for p, person in enumerate(sc["persons"]):
        idx, cnt = engine.ray_aabb_hits(cam.cuda(), dirs.cuda(), person["verts_p"].cuda(), 1.2)
        n = int(cnt.item())
        assert torch.equal(idx[:n].cpu(), ref[p])
    # rays in an image corner miss the box: the list becomes [0] on the device (multiply.py:262-263)
    uv = torch.rand(1, 33, 2, generator=torch.Generator().manual_seed(4)) * 6.0
    K, pose = S.make_camera()
    dirs, cam = rend_util.get_camera_params_host(uv, pose, K)
    idx, cnt = engine.ray_aabb_hits(cam.cuda(), dirs.cuda(), sc["persons"][0]["verts_p"].cuda(), 1.2)
    assert int(cnt.item()) == 1 and int(idx[0].item()) == 0


def test_query_oc_and_dense_grid(golden_dir):
    """Multiply.query_oc (multiply.py:169-172) through the mirror, batch by batch as generate_mesh calls it
    (lib/utils/mesh.py:97-100), and utils.mesh.dense_sdf_grid in one call: both equal the reference's values."""
    import os
    from multiply_b200 import engine
    from multiply_b200.utils import mesh
    engine.set_engine("tc")
    g = np.load(os.path.join(golden_dir, "sdf_grid.npz"))
    sc = S.make_scene(P=2, S=64, seed=42)
    m = S.mirror_model(sc)
    p1 = sc["persons"][1]
    cond = {"smpl": p1["cond"].cuda()}
    pts = torch.from_numpy(g["points"]).cuda()
    occ = torch.cat([m.query_oc(b, cond, 1)["occ"] for b in torch.split(pts, 500, dim=0)])
    assert occ.shape == (pts.shape[0], 1)
    assert float(np.abs(occ[:, 0].cpu().numpy() - g["occ"]).max()) < 5e-5
    dense = mesh.dense_sdf_grid(m, 1, cond, p1["verts_c"], res=int(g["res"]))
    assert torch.equal(dense.reshape(-1), occ[:, 0])


def test_sampler_training_mode(golden_dir):
    """f1, forward half: ErrorBoundSampler.get_z_vals with model.training (stratified start samples, random final
    abscissae, randperm extras, eikonal pick, jittered inverse-sphere depths, no outlier clamp in the SDF callback)
    against the reference's own sampler in training mode — (a) with the recorded random draws passed in
    (mp_sample_rays_train), (b) through the mirror with the same torch.manual_seed, which replays the reference's
    random stream."""
    import os
    from multiply_b200 import engine, _lib as L
    from multiply_b200.model.ray_sampler import ErrorBoundSampler
    from multiply_b200.model import rend_util
    engine.set_engine("tc")
    g = np.load(os.path.join(golden_dir, "sampler_train.npz"))
    sc = S.make_scene(P=2, S=16, seed=42)
    inputs = S.make_rays(sc, 40, seed=21, region="boxes")
    dirs, cam = rend_util.get_camera_params_host(inputs["uv"], inputs["pose"], inputs["intrinsics"])
    idx = torch.from_numpy(g["hits"])
    d, o = dirs[idx].cuda(), cam[idx].cuda()
    R = idx.numel()
    p0 = sc["persons"][0]
    m = S.mirror_model(sc)
    cfg = sc["cfg"]
    smp = ErrorBoundSampler(3.0, cfg["near"], cfg["N_samples"], cfg["N_samples_eval"], cfg["N_samples_extra"], cfg["eps"],
                            cfg["beta_iters"], cfg["max_total_iters"], inverse_sphere_bg=True, add_tiny=cfg["add_tiny"])
    T, E = cfg["max_total_iters"], cfg["N_samples_eval"]
    trips_ref = g["extra_perm"].shape[0] // E
    rng = smp.draw_training_rng(R)
    rng.pop("states")
    rng["t_rand"], rng["u_final"] = torch.from_numpy(g["t_rand"]), torch.from_numpy(g["u_final"])
    rng["extra_perm"][trips_ref - 1, :trips_ref * E] = torch.from_numpy(g["extra_perm"]).to(torch.int32)
    rng["eik_idx"][trips_ref - 1] = torch.from_numpy(g["eik_idx"]).to(torch.int32)
    rng["t_rand_bg"][trips_ref - 1] = torch.from_numpy(g["t_rand_bg"])

    def check(z, z_bg, z_eik, trips):
        assert int(trips.item()) == trips_ref
        assert float(np.abs(z_bg.cpu().numpy() - g["z_bg"]).max()) < 1e-6
        dz = np.abs(z.cpu().numpy() - g["z_vals"])
        assert np.median(dz) < 1e-5 and dz.max() < 5e-3         # coarse 16/32/8 sampler: see test_forward_golden_coarse
        assert float(np.abs(z_eik.cpu().numpy() - g["z_eik"]).max()) < 5e-3

    m.train()
    try:
        # (a) recorded draws
        lib = L.lib()
        c = engine.sampler_cfg(smp.cfg, float(m.density.beta.detach()), float(m.density.beta_min))
        body = m.deformer_list[0].body(d.device)
        body.set_pose(p0["verts_p"].cuda(), p0["tfs"].cuda())
        field = m.field_list[0]
        field.set_cond(p0["cond"].cuda())
        z = torch.empty(R, cfg["N_samples"] + cfg["N_samples_extra"] + 2, device="cuda")
        z_bg = torch.empty(R, 32, device="cuda")
        trips = torch.zeros(1, dtype=torch.int32, device="cuda")
        smp._ws = L.workspace(L.call("mp_sampler_workspace_bytes", c, R), "cuda")
        (z, z_bg), z_eik = smp._get_z_vals_training(lib, c, body, field, d.contiguous(), o.contiguous(), R, z, z_bg, trips,
                                                    d.device, rng=rng)
        torch.cuda.synchronize()
        check(z, z_bg, z_eik, trips)
        # (b) the mirror draws the reference's random stream itself
        torch.manual_seed(1234)
        (z2, z_bg2), z_eik2 = smp.get_z_vals(d, o, m, {"smpl": p0["cond"].cuda()}, p0["tfs"][None].cuda(), False,
                                              p0["verts_p"][None].cuda(), 0)
        torch.cuda.synchronize()
        check(z2, z_bg2, z_eik2, smp.last_trips)
        assert torch.equal(z2, z) and torch.equal(z_eik2, z_eik)
    finally:
        m.eval()


def test_forward_training_values(golden_dir):
    """f1, forward half: Multiply.forward with model.training (values of the training branch: stochastic sampling, no
    outlier clamp, eikonal gradients, jittered background) against the reference's own objects driven through that
    branch (tests/golden/forward_train.npz) — the mirror replays the reference's random stream from the same seed."""
    import os
    from multiply_b200 import engine
    engine.set_engine("tc")
    g = np.load(os.path.join(golden_dir, "forward_train.npz"))
    sc = S.make_scene(P=2, S=16, seed=42)
    inp = S.make_rays(sc, 40, seed=33, region="boxes")
    assert np.array_equal(inp["uv"].numpy(), g["uv"])
    m = S.mirror_model(sc)
    inputs = mirror_inputs(inp, 2, [torch.from_numpy(g[f"hits_{p}"]).cuda() for p in range(2)], epoch=251)
    m.train()
    try:
        torch.manual_seed(4321)
        out = m(inputs)
        torch.cuda.synchronize()
    finally:
        m.eval()
    assert out["index_off_surface"] is None and out["grad_theta"].shape == (1, 1024, 3)
    assert abs(float(out["temporal_loss"]) - 1e-4) < 1e-6
    assert float(np.abs(out["grad_theta"].cpu().numpy() - g["grad_theta"]).max()) < 1e-4
    for k, tol in (("rgb_values", 1e-4), ("acc_map", 1e-4), ("acc_person_list", 1e-4), ("normal_values", 1e-3)):
        d = np.abs(out[k].cpu().numpy() - g[k])
        assert np.median(d) < 1e-5 and d.max() < tol, (k, float(d.max()))


def test_load_reference_checkpoint_keys():
    """A Lightning checkpoint of the reference (keys 'model.*', plus smpl_server_list / deformer_list buffers and
    MultiplyModel's body_model_list, train.py:16-22) loads through load_reference_checkpoint with strict=True."""
    sc = S.make_scene(P=2, S=16, seed=42)
    m = S.mirror_model(sc)
    sd = {"model." + k: v for k, v in m.state_dict().items()}
    sd["model.smpl_server_list.0.smpl.v_template"] = torch.zeros(6890, 3)
    sd["model.deformer_list.1.smpl.smpl.lbs_weights"] = torch.zeros(6890, 24)
    sd["body_model_list.0.betas.weight"] = torch.zeros(1, 10)
    res = m.load_reference_checkpoint(sd, strict=True)
    assert not res.missing_keys and not res.unexpected_keys


def test_operator_mirrors():
    """ImplicitNet / RenderingNet / LaplaceDensity / SMPLDeformer / ErrorBoundSampler called the way the
    reference calls them (networks.py:126, :263; density.py:11; deformer.py:19; ray_sampler.py:66)."""
    from multiply_b200 import engine
    from multiply_b200.model import networks, density, deformer
    from oracle import port
    engine.set_engine("tc")
    sc = S.make_scene(P=2, S=16, seed=42)
    p0 = sc["persons"][0]
    net = networks.ImplicitNet(S.MODEL_OPT["implicit_network"])
    net.load_state_dict(p0["implicit"], strict=True)
    net = net.cuda().eval()
    x = (torch.rand(300, 3, generator=torch.Generator().manual_seed(1)) - 0.5)
    y = net(x.cuda(), {"smpl": p0["cond"].cuda()})
    with torch.no_grad():
        ref = port.implicit_forward(p0["implicit"], x, p0["cond"], 6)
    assert y.shape == (1, 300, 257)
    assert float((y[0].cpu() - ref).abs().max()) < 5e-5
    rn = networks.RenderingNet(S.MODEL_OPT["rendering_network"])
    rn.load_state_dict(p0["render"], strict=True)
    rn = rn.cuda().eval()
    nrm = torch.nn.functional.normalize(torch.randn(300, 3, generator=torch.Generator().manual_seed(2)), dim=1)
    rgb = rn(x.cuda(), nrm.cuda(), None, p0["cond"].cuda(), ref[:, 1:].cuda())
    with torch.no_grad():
        rref = port.rendering_forward(p0["render"], "pose_no_view", x, nrm, None, p0["cond"], ref[:, 1:])
    assert float((rgb.cpu() - rref).abs().max()) < 1e-5
    dens = density.LaplaceDensity(params_init={"beta": 0.1}, beta_min=1e-4).cuda()
    s = torch.linspace(-0.5, 4.0, 100)
    assert float((dens(s.cuda()).cpu() - port.laplace_density(s, port.get_beta(0.1))).abs().max()) < 1e-5
    d = deformer.SMPLDeformer(smpl_verts=p0["verts_c"], smpl_weights=p0["weights"], scale=0.5)
    pts = p0["verts_p"][:400] + 0.03
    xc, outl = d.forward(pts.cuda(), p0["tfs"][None].cuda(), return_weights=False, inverse=True,
                         smpl_verts=p0["verts_p"][None].cuda())
    xr, orf = port.deform_inverse(pts, p0)
    assert bool((outl.cpu() == orf).all()) and float((xc.cpu() - xr).abs().max()) < 1e-5
    assert net(x[:0].cuda(), {"smpl": p0["cond"].cuda()}).shape[1] == 0      # zero-size early return


def test_sdf_func_with_smpl_deformer_mirror():
    """Multiply.sdf_func_with_smpl_deformer (multiply.py:137-151) through the mirror class, against the oracle."""
    from multiply_b200 import engine
    from oracle import port
    engine.set_engine("tc")
    sc = S.make_scene(P=2, S=16, seed=42)
    m = S.mirror_model(sc)
    p1 = sc["persons"][1]
    g = torch.Generator().manual_seed(3)
    pts = torch.cat([p1["verts_p"][:300] + 0.02 * torch.randn(300, 3, generator=g),       # near the body
                     p1["verts_p"][:100] + 0.5])                                          # outliers
    sdf, xc, feat = m.sdf_func_with_smpl_deformer(pts.cuda(), {"smpl": p1["cond"].cuda()}, p1["tfs"][None].cuda(),
                                                  p1["verts_p"][None].cuda(), 1)
    with torch.no_grad():
        rs, rx, rf = port.sdf_func_with_smpl_deformer(pts, p1, sc["cfg"])
    assert sdf.shape == (400, 1) and xc.shape == (400, 3) and feat.shape == (400, 256)
    assert float((sdf.cpu() - rs).abs().max()) < 5e-5
    assert float((xc.cpu() - rx).abs().max()) < 1e-5
    assert float((feat.cpu() - rf).abs().max()) < 5e-5
    assert bool(((sdf.cpu() == 4.0) == (rs == 4.0)).all()) and bool((rs[300:] == 4.0).any())


def test_smpl_server_and_culling(golden_dir):
    """SMPLServer (lbs) against the reference's lbs.py output (golden) and the oracle's SMPLServer.forward;
    GPU ray/box culling against the host slab test."""
    import os
    from multiply_b200 import engine
    from multiply_b200.model.smpl import SMPLServer
    from multiply_b200.model import rend_util
    from oracle import port
    g = np.load(os.path.join(golden_dir, "smpl_lbs.npz"))
    sm = S.make_smpl_model(300)
    srv = SMPLServer(model=sm)
    betas, pose = torch.from_numpy(g["betas"]), torch.from_numpy(g["pose"])
    out = srv(torch.ones(1), torch.zeros(1, 3), pose, betas, absolute=True)
    torch.cuda.synchronize()
    assert float(np.abs(out["smpl_verts"][0].cpu().numpy() - g["verts"]).max()) < 5e-6
    assert float(np.abs(out["smpl_tfs"][0].cpu().numpy() - g["A"]).max()) < 5e-6
    # SMPLServer.forward with scale / translation / canonical inverse vs the oracle (smpl.py:50-95)
    tinv, vc = port.smpl_canonical_tfs_inv(sm, torch.zeros(10))
    assert float((srv.verts_c[0].cpu() - vc).abs().max()) < 5e-6
    assert float((srv.tfs_c_inv.cpu() - tinv).abs().max()) < 5e-5
    ref = port.smpl_server_forward(sm, tinv, torch.tensor([0.5]), torch.tensor([0.3, 0.1, -0.2]), pose[0], betas[0])
    out = srv(torch.tensor([0.5]), torch.tensor([[0.3, 0.1, -0.2]]), pose, betas)
    torch.cuda.synchronize()
    assert float((out["smpl_verts"][0].cpu() - ref["smpl_verts"]).abs().max()) < 5e-6
    assert float((out["smpl_tfs"][0].cpu() - ref["smpl_tfs"]).abs().max()) < 5e-5
    # culling
    sc = S.make_scene(P=2, S=16, seed=42)
    inp = S.make_rays(sc, 5000, seed=3, region="image")
    dirs, cam = rend_util.get_camera_params_host(inp["uv"], inp["pose"], inp["intrinsics"])
    for person in sc["persons"]:
        c, h = S.person_box(person)
        ref_hits = S.ray_box_hits(cam, dirs, c, h)
        got = engine.ray_box_hits(cam.cuda(), dirs.cuda(), c.tolist(), h.tolist())
        assert torch.equal(got.cpu(), ref_hits)


def test_sequence_directory_drives_forward(tmp_path):
    """f2: a preprocessed sequence directory (the files Hi4D.py:119-146 reads) -> utils.data.SequenceData -> the input
    dict -> Multiply.forward through the chunked full-frame loop of test_step (idr_utils.render_full_frame).  The same
    frame rendered in one call from hand-built inputs (camera K / pose, smpl_params) must agree: the reader recovers the
    camera from P = world_mat @ scale_mat by RQ decomposition like cv2.decomposeProjectionMatrix."""
    import struct, zlib
    from multiply_b200 import engine
    from multiply_b200.utils import data as D, idr_utils
    engine.set_engine("tc")
    P, res = 2, 24
    sc = S.make_scene(P=P, S=16, seed=42)
    model = S.mirror_model(sc)
    K, pose = S.make_camera(f=900.0 * res / 512, res=res)         # same field of view as the 512 x 512 test camera
    base = mirror_inputs(dict(S.grid_rays(res=res), intrinsics=K, pose=pose), P)

    Rm = pose[0, :3, :3].double().numpy().T                       # world -> camera
    c = pose[0, :3, 3].double().numpy()
    scale_mat = np.diag([2.0, 2.0, 2.0, 1.0])                      # scale = 0.5, as smpl_scene_inputs
    world = np.eye(4)
    world[:3, :4] = K[0, :3, :3].double().numpy() @ np.concatenate([Rm, (-Rm @ (2.0 * c))[:, None]], 1)
    np.save(tmp_path / "mean_shape.npy", np.zeros((P, 10), np.float32))
    np.save(tmp_path / "poses.npy", base["smpl_pose"].cpu().numpy().repeat(5, 0))
    np.save(tmp_path / "normalize_trans.npy", base["smpl_trans"].cpu().numpy().repeat(5, 0))
    np.savez(tmp_path / "cameras_normalize.npz",
             **{"scale_mat_%d" % i: scale_mat for i in range(5)}, **{"world_mat_%d" % i: world for i in range(5)})
    seq = D.SequenceData(str(tmp_path), start_frame=0, end_frame=5, img_size=(res, res))
    frame = seq.frame(3, device="cuda")
    assert torch.allclose(frame["pose"].cpu(), pose, atol=1e-5)
    assert torch.allclose(frame["intrinsics"][0, :3, :3].cpu(), K[0, :3, :3], rtol=1e-5, atol=1e-3)
    assert torch.equal(frame["uv"].cpu(), base["uv"].cpu())
    assert torch.allclose(frame["smpl_params"][..., 0].cpu(), base["smpl_params"][..., 0].cpu(), atol=1e-7)
    for k in ("smpl_pose", "smpl_trans", "smpl_shape"):
        assert torch.allclose(frame[k].cpu(), base[k].cpu(), atol=1e-7), k

    whole = model(frame)
    chunks = idr_utils.render_full_frame(model, frame, seq.total_pixels, n_pixels=seq.total_pixels)
    ref = model(dict(base, idx=torch.tensor([3]).cuda()))
    torch.cuda.synchronize()
    assert float(whole["acc_map"].max()) > 0.5                     # the persons are in the frame
    for k in ("rgb_values", "normal_values", "acc_map"):
        assert torch.isfinite(whole[k]).all()
        assert torch.equal(chunks[k].reshape(whole[k].shape), whole[k]), k
        bad = ((whole[k] - ref[k]).abs().reshape(res * res, -1).max(1)[0] > 1e-3).float().mean()
        assert float(bad) < 0.01, (k, float(bad))                  # camera recovered to ~1e-6: same picture


def test_multiply_root_finder_switch():
    """Row f4 through the mirror: Multiply.set_root_finder(10) == oracle with the same switch; (0) restores the
    reference's closed-form path bit for bit."""
    from multiply_b200 import engine
    from oracle import port
    engine.set_engine("tc")
    sc = S.make_scene(P=2, S=16, seed=42)
    inp = S.make_rays(sc, 96, seed=11, region="boxes")
    hits = S.make_hit_lists(sc, inp)
    m = S.mirror_model(sc)
    inputs = mirror_inputs(inp, 2, [h.cuda() for h in hits])
    plain = {k: v.clone() for k, v in m(inputs).items()}
    m.set_root_finder(10, 1e-5)
    on = {k: v.clone() for k, v in m(inputs).items()}
    m.set_root_finder(0)
    off = m(inputs)
    torch.cuda.synchronize()
    ref = port.multiply_forward(dict(sc, persons=[dict(p, root_finder=(10, 1e-5)) for p in sc["persons"]]), inp, hits)
    assert float((on["rgb_values"] - plain["rgb_values"]).abs().max()) > 1e-3
    for k in ("rgb_values", "normal_values", "acc_map"):
        assert torch.equal(off[k], plain[k]), k
        d = (on[k].cpu() - ref[k]).abs().reshape(96, -1).max(1)[0]
        assert float((d > 1e-4).float().mean()) < 0.03 and float(d.median()) < 1e-5, (k, float(d.max()))


def test_oriented_box_culling():
    """culling='obb' (multiply.py:208-214: oriented box of the posed mesh, extents x1.2, built on the host): the device
    ray test against that box equals a float64 slab test in the box frame, and the forward runs on those lists and
    equals the oracle fed with the same lists."""
    from multiply_b200 import engine
    from multiply_b200.model import rend_util
    from multiply_b200.utils import obb
    from oracle import port
    engine.set_engine("tc")
    sc = S.make_scene(P=2, S=16, seed=42)
    inp = S.make_rays(sc, 160, seed=21, region="image")
    P = 2
    servers = [S.SyntheticSMPLServer(p, P) for p in range(P)]
    m = S.mirror_model(sc, servers, culling="obb")
    inputs = mirror_inputs(inp, P)
    out = m(inputs)
    torch.cuda.synchronize()
    # the same lists on the host
    dirs, cam = rend_util.get_camera_params_host(inp["uv"], inp["pose"], inp["intrinsics"])
    cam = cam.reshape(-1, 3)[:1]
    d64, c64 = dirs.double().numpy(), cam.double().numpy()
    hits, persons = [], []
    for p in range(P):
        o = servers[p](inputs["smpl_params"][:, p, 0].cpu(), inputs["smpl_trans"][:, p].cpu(), inputs["smpl_pose"][:, p].cpu(),
                       inputs["smpl_shape"][:, p].cpu())
        v = o["smpl_verts"][0]
        persons.append(dict(sc["persons"][p], verts_p=v, tfs=o["smpl_tfs"][0]))
        c, h, rot = obb.culling_box(v.numpy(), 1.2)
        o_l = (c64 - c) @ rot.T
        d_l = d64 @ rot.T
        with np.errstate(divide="ignore", invalid="ignore"):
            t1, t2 = (-h - o_l) / d_l, (h - o_l) / d_l
        tn, tf = np.minimum(t1, t2).max(1), np.maximum(t1, t2).min(1)
        ids = np.nonzero((tn <= tf) & (tf >= 0))[0]
        dev_ids = engine.ray_box_hits(cam.expand(160, 3).contiguous().cuda(), dirs.cuda(), c, h, rot)
        assert np.array_equal(dev_ids.cpu().numpy(), ids)
        assert 0 < len(ids) < 160                                 # a real cull: some rays hit, some miss
        hits.append(torch.from_numpy(ids if len(ids) else np.array([0])).long())
    ref = port.multiply_forward(dict(sc, persons=persons), inp, hits)
    for k in ("rgb_values", "acc_map", "acc_person_list"):
        assert float((out[k].cpu() - ref[k]).abs().max()) < 1e-4, k
