"""TEST INFRASTRUCTURE ONLY — CPU oracle for the MultiPly volume-rendering hot path.

A plain-PyTorch (CPU, fp32) restatement of the reference's eval-mode
``Multiply.forward`` and every operator it calls.  It exists to CHECK the CUDA
path; it is never imported by the product package (only by tests/, bench.py's
``cpu_baseline`` / ``--impl reference`` legs and ``__graft_entry__.smoke``).

Pinning: the reference ships no tests / golden vectors for this path
(SURVEY.md §0-2).  This file is pinned instead against the *unmodified reference
modules* run on CPU under the shims of ``oracle/ref_shim.py``:
``oracle/gen_golden.py`` executes both on the same seeded inputs and commits the
reference's outputs as ``tests/golden/*.npz``; ``tests/test_oracle_golden.py``
re-checks this port against them on every run.  The third-party kernels the
reference calls (pytorch3d ``knn_points``, nerfacc ``render_weight_from_density`` /
``pack_info`` / ``accumulate_along_rays``, trimesh ray-box hits) are absent and
unpinned upstream; their restatements below are definitions ("parity unpinned" at
that boundary, see DESIGN.md).

All ``file:line`` cites are relative to /root/reference/code.
"""
import math
import numpy as np
import torch
import torch.nn.functional as F

# --------------------------------------------------------------------------------------
# third-party restatements (SURVEY.md Appendix C)
# --------------------------------------------------------------------------------------


def knn_points(p1, p2, K=1, return_nn=True, chunk=8192):
    """pytorch3d.ops.knn_points for K=1 (call site lib/model/deformer.py:39).

    Squared L2 distance, arg-min over p2.  Definition used by both oracle and CUDA
    kernel: d2 = (dx*dx + dy*dy) + dz*dz with every product/sum rounded separately
    (no FMA), ties resolved to the lowest vertex index.
    p1 [1,N,3], p2 [1,V,3] -> (d2 [1,N,1], idx [1,N,1] int64, nn [1,N,1,3])
    """
    assert K == 1 and p1.shape[0] == 1 and p2.shape[0] == 1
    x, v = p1[0], p2[0]
    N = x.shape[0]
    d2 = torch.empty(N, dtype=x.dtype)
    idx = torch.empty(N, dtype=torch.int64)
    vx, vy, vz = v[:, 0][None], v[:, 1][None], v[:, 2][None]
    for s in range(0, N, chunk):
        xs = x[s:s + chunk]
        dx = xs[:, 0:1] - vx
        dy = xs[:, 1:2] - vy
        dz = xs[:, 2:3] - vz
        d = dx * dx
        d = d + dy * dy
        d = d + dz * dz
        m, i = torch.min(d, dim=1)      # torch.min returns the first minimal index on CPU
        d2[s:s + chunk] = m
        idx[s:s + chunk] = i
    nn = v[idx] if return_nn else None
    return d2[None, :, None], idx[None, :, None], (nn[None, :, None, :] if return_nn else None)


def pack_info(ray_indices, n_rays):
    """nerfacc.pack_info (call site lib/model/multiply.py:456): [n_rays,2]=(start,count)."""
    cnt = torch.bincount(ray_indices, minlength=n_rays)
    start = torch.cumsum(cnt, 0) - cnt
    return torch.stack([start, cnt], dim=1)


def render_weight_from_density(t_starts, t_ends, sigmas, ray_indices=None, n_rays=None):
    """nerfacc.render_weight_from_density (call site lib/model/multiply.py:455).

    alpha = 1-exp(-sigma*dt); T = exp(-exclusive per-ray prefix sum of sigma*dt); w = T*alpha.
    Rows are sorted by ray.  Returns (weights, transmittance, alphas)."""
    sd = sigmas * (t_ends - t_starts)
    alphas = 1.0 - torch.exp(-sd)
    info = pack_info(ray_indices, n_rays)
    # per-ray sequential exclusive scan (association independent of the other rays)
    sd_np = sd.detach().numpy()
    out = np.zeros_like(sd_np)
    st = info[:, 0].numpy()
    ct = info[:, 1].numpy()
    for r in range(n_rays):
        c = ct[r]
        if c <= 1:
            continue
        s = st[r]
        out[s + 1:s + c] = np.cumsum(sd_np[s:s + c - 1], dtype=np.float32)
    trans = torch.exp(-torch.from_numpy(out))
    return trans * alphas, trans, alphas


def accumulate_along_rays(weights, values=None, ray_indices=None, n_rays=None):
    """nerfacc.accumulate_along_rays (call sites lib/model/multiply.py:465-478)."""
    if values is None:
        src = weights[:, None]
    else:
        src = weights[:, None] * values
    out = torch.zeros(n_rays, src.shape[1], dtype=src.dtype)
    out.index_add_(0, ray_indices, src)
    return out


# --------------------------------------------------------------------------------------
# networks (lib/model/networks.py, embedders.py, density.py)
# --------------------------------------------------------------------------------------


def embed(x, multires):
    """lib/model/embedders.py:8-34: [x, sin(2^0 x), cos(2^0 x), ..., sin(2^(L-1) x), cos(2^(L-1) x)]."""
    outs = [x]
    freqs = 2.0 ** torch.linspace(0.0, multires - 1, multires)
    for f in freqs:
        outs.append(torch.sin(x * f))
        outs.append(torch.cos(x * f))
    return torch.cat(outs, -1)


def _lin(sd, l, weight_norm):
    """weight-normed linear (networks.py:82-83 / 257-258): W = g * v / ||v||_row."""
    if weight_norm:
        w = torch._weight_norm(sd[f"lin{l}.weight_v"], sd[f"lin{l}.weight_g"], 0)
    else:
        w = sd[f"lin{l}.weight"]
    return w, sd[f"lin{l}.bias"]


def softplus100(x):
    return F.softplus(x, beta=100)


def implicit_forward(sd, x, cond, multires, skip_in=(4,), weight_norm=True, n_lin=9):
    """ImplicitNet.forward, lib/model/networks.py:126-208 (cond in {'smpl','frame'}).

    x [N,d_in], cond [1,C] -> [N,257]."""
    N = x.shape[0]
    if N == 0:
        return x
    inp = embed(x, multires) if multires > 0 else x
    input_cond = cond.expand(N, -1)
    h = inp
    for l in range(n_lin):
        w, b = _lin(sd, l, weight_norm)
        if l == 0:
            h = torch.cat([h, input_cond], -1)
        if l in skip_in:
            h = torch.cat([h, inp], 1) / np.sqrt(2)
        h = F.linear(h, w, b)
        if l < n_lin - 1:
            h = softplus100(h)
    return h


def rendering_forward(sd, mode, points, normals, view_dirs, body_pose, feature_vectors,
                      frame_latent_code=None, weight_norm=True, multires_view=-1):
    """RenderingNet.forward, lib/model/networks.py:263-312, modes 'pose_no_view' and
    'nerf_frame_encoding'."""
    if mode == "pose_no_view":
        n = points.shape[0]
        bp = body_pose.unsqueeze(1).expand(-1, n, -1).reshape(n, -1)
        bp = F.linear(bp, sd["lin_pose.weight"], sd["lin_pose.bias"])
        h = torch.cat([points, normals, bp, feature_vectors], -1)
    elif mode == "nerf_frame_encoding":
        vd = embed(view_dirs, multires_view)
        fl = frame_latent_code.expand(vd.shape[0], -1)
        h = torch.cat([vd, fl, feature_vectors], -1)
    else:
        raise NotImplementedError(mode)
    n_lin = len([k for k in sd if k.startswith("lin") and k.endswith("bias") and "pose" not in k])
    for l in range(n_lin):
        w, b = _lin(sd, l, weight_norm)
        h = F.linear(h, w, b)
        if l < n_lin - 1:
            h = torch.relu(h)
    return torch.sigmoid(h)


def laplace_density(sdf, beta):
    """LaplaceDensity.density_func, lib/model/density.py:20-25."""
    alpha = 1 / beta
    return alpha * (0.5 + 0.5 * sdf.sign() * torch.expm1(-sdf.abs() / beta))


def get_beta(beta_param, beta_min=1e-4):
    """LaplaceDensity.get_beta, lib/model/density.py:27-29."""
    return torch.tensor(beta_param, dtype=torch.float32).abs() + torch.tensor(beta_min, dtype=torch.float32)


# --------------------------------------------------------------------------------------
# deformer (lib/model/deformer.py)
# --------------------------------------------------------------------------------------


def query_skinning_weights(pts, smpl_verts, smpl_weights):
    """SMPLDeformer.query_skinning_weights_smpl_multi, deformer.py:37-50 (K=1).
    pts [1,N,3], smpl_verts [V,3], smpl_weights [1,V,24] -> weights [1,N,24], outlier [N]."""
    d2, idx, _ = knn_points(pts, smpl_verts.unsqueeze(0), K=1, return_nn=True)
    d2 = torch.clamp(d2, max=4)
    conf = torch.exp(-d2)
    d = torch.sqrt(d2)
    conf = conf / conf.sum(-1, keepdim=True)
    idx = idx[0]
    w = smpl_weights[:, idx, :]
    w = torch.sum(w * conf.unsqueeze(-1), dim=-2).detach()
    outlier = (d[..., 0] > 0.1)[0]
    return w, outlier


def skinning(x, w, tfs, inverse=False):
    """skinning(), deformer.py:72-89."""
    x_h = F.pad(x, (0, 1), value=1.0)
    if inverse:
        w_tf = torch.einsum("bpn,bnij->bpij", w, tfs)
        x_h = torch.einsum("bpij,bpj->bpi", w_tf.inverse(), x_h)
    else:
        x_h = torch.einsum("bpn,bnij,bpj->bpi", w, tfs, x_h)
    return x_h[:, :, :3]


def deform_inverse(x, person):
    """SMPLDeformer.forward(inverse=True, return_weights=False), deformer.py:19-30."""
    w, outlier = query_skinning_weights(x[None], person["verts_p"], person["weights"][None])
    xc = skinning(x.unsqueeze(0), w, person["tfs"][None], inverse=True).squeeze(0)
    rf = person.get("root_finder")          # row f4 (non-default, not in the reference): see deform_broyden
    if rf and x.shape[0] > 0:
        keep = ~outlier
        if bool(keep.any()):
            xr, _, _, _ = deform_broyden(x[keep], dict(person, root_finder=None), rf[0], rf[1])
            xc = xc.clone()
            xc[keep] = xr
    return xc, outlier


def forward_skinning(x_c, person):
    """SMPLDeformer.forward_skinning, deformer.py:31-35: weights of the nearest CANONICAL vertex, forward LBS.
    Returns (x_d [N,3], A [N,3,3] = upper-left block of the blended transform)."""
    w, _ = query_skinning_weights(x_c[None], person["verts_c"], person["weights"][None])
    T = torch.einsum("bpn,bnij->bpij", w, person["tfs"][None])[0]
    x_d = torch.einsum("pij,pj->pi", T[:, :3, :3], x_c) + T[:, :3, 3]
    return x_d, T[:, :3, :3]


def deform_broyden(x, person, max_steps=10, cvg_threshold=1e-5):
    """Row f4 — NOT a restatement of reference code: the reference has no root finder (SURVEY.md fact 0-1).  This is
    the CPU statement of the algorithm mp_deform_broyden implements, anchored on the two reference maps it connects:
    start = the closed-form inverse (deformer.py:19-30), residual g(x_c) = forward_skinning(x_c) - x
    (deformer.py:31-35).  Broyden's method with J^-1 initialised to the inverse blended 3x3 at the start point,
    Sherman-Morrison rank-one updates, lowest-residual iterate kept.  Returns (x_c, residual, converged, outlier)."""
    xc, outlier = deform_inverse(x, person)
    xc = xc.clone()
    f, A = forward_skinning(xc, person)
    Ji = torch.linalg.inv(A)
    g = f - x
    best = g.norm(dim=-1)
    cur = xc.clone()
    for _ in range(max_steps):
        act = best >= cvg_threshold
        if not bool(act.any()):
            break
        idx = act.nonzero()[:, 0]
        dx = -torch.einsum("pij,pj->pi", Ji[idx], g[idx])
        xn = cur[idx] + dx
        fn, _ = forward_skinning(xn, person)
        gn = fn - x[idx]
        dg = gn - g[idx]
        u = torch.einsum("pij,pj->pi", Ji[idx], dg)
        vt = torch.einsum("pi,pij->pj", dx, Ji[idx])
        den = (dx * u).sum(-1)
        ok = den.abs() > 1e-20
        upd = (dx - u)[:, :, None] * vt[:, None, :] / torch.where(ok, den, torch.ones_like(den))[:, None, None]
        Ji[idx] = Ji[idx] + torch.where(ok[:, None, None], upd, torch.zeros_like(upd))
        cur[idx] = xn
        g[idx] = gn
        rn = gn.norm(dim=-1)
        better = rn < best[idx]
        bi = idx[better]
        best[bi] = rn[better]
        xc[bi] = xn[better]
    return xc, best, best < cvg_threshold, outlier


def sdf_func_with_smpl_deformer(x, person, cfg, chunk=65536, training=False):
    """Multiply.sdf_func_with_smpl_deformer, lib/model/multiply.py:137-151 (eval: outliers forced to 4, :142-143;
    training: the network value everywhere)."""
    sdfs, xcs, feats = [], [], []
    for s in range(0, max(x.shape[0], 1), chunk):
        xs = x[s:s + chunk]
        x_c, outlier = deform_inverse(xs, person)
        out = implicit_forward(person["implicit"], x_c, person["cond"], cfg["multires"])
        sdf = out[:, 0:1].clone()
        if not training:
            sdf[outlier] = 4.0
        sdfs.append(sdf)
        xcs.append(x_c)
        feats.append(out[:, 1:])
    return torch.cat(sdfs), torch.cat(xcs), torch.cat(feats)


# --------------------------------------------------------------------------------------
# SMPL server (lib/model/smpl.py:50-95 -> lib/smpl/body_models.py:278-364 -> lib/smpl/lbs.py:136-229)
# --------------------------------------------------------------------------------------


def batch_rodrigues(rot_vecs):
    """lib/smpl/lbs.py:276-307."""
    n = rot_vecs.shape[0]
    angle = torch.norm(rot_vecs + 1e-8, dim=1, keepdim=True)
    rot_dir = rot_vecs / angle
    cos = torch.unsqueeze(torch.cos(angle), dim=1)
    sin = torch.unsqueeze(torch.sin(angle), dim=1)
    rx, ry, rz = torch.split(rot_dir, 1, dim=1)
    zeros = torch.zeros((n, 1))
    K = torch.cat([zeros, -rz, ry, rz, zeros, -rx, -ry, rx, zeros], dim=1).view((n, 3, 3))
    ident = torch.eye(3).unsqueeze(dim=0)
    return ident + sin * K + (1 - cos) * torch.bmm(K, K)


def batch_rigid_transform(rot_mats, joints, parents):
    """lib/smpl/lbs.py:323-378 (batch 1): returns (posed_joints [J,3], rel_transforms A [J,4,4])."""
    J = joints.shape[0]
    rel = joints.clone()
    rel[1:] = rel[1:] - joints[parents[1:]]
    T = torch.zeros(J, 4, 4)
    T[:, :3, :3] = rot_mats
    T[:, :3, 3] = rel
    T[:, 3, 3] = 1
    chain = [T[0]]
    for i in range(1, J):
        chain.append(torch.matmul(chain[int(parents[i])], T[i]))
    G = torch.stack(chain, dim=0)
    jh = F.pad(joints, [0, 1]).unsqueeze(-1)
    A = G - F.pad(torch.matmul(G, jh), [3, 0, 0, 0, 0, 0])
    return G[:, :3, 3], A


def lbs(betas, pose, model):
    """lib/smpl/lbs.py:136-229 (batch 1, pose2rot, pose_blend): betas [10], pose [72] ->
    (verts [V,3], A [24,4,4])."""
    v_shaped = model["v_template"] + torch.einsum('l,mkl->mk', betas, model["shapedirs"])
    J = torch.einsum('ik,ji->jk', v_shaped, model["J_regressor"])
    rot = batch_rodrigues(pose.view(-1, 3))
    pose_feature = (rot[1:] - torch.eye(3)).reshape(1, -1)
    v_posed = v_shaped + torch.matmul(pose_feature, model["posedirs"]).view(-1, 3)
    _, A = batch_rigid_transform(rot, J, model["parents"])
    T = torch.matmul(model["lbs_weights"], A.view(24, 16)).view(-1, 4, 4)
    vh = torch.cat([v_posed, torch.ones(v_posed.shape[0], 1)], dim=1)
    verts = torch.matmul(T, vh.unsqueeze(-1))[:, :3, 0]
    return verts, A


def smpl_server_forward(model, tfs_c_inv, scale, transl, thetas, betas, absolute=False):
    """SMPLServer.forward, lib/model/smpl.py:50-95: scale [1], transl [3], thetas [72], betas [10] ->
    dict(smpl_verts [V,3], smpl_tfs [24,4,4])."""
    verts, A = lbs(betas, thetas, model)
    out_verts = verts * scale + transl * scale
    tf = A.clone()
    tf[:, :3, :] = tf[:, :3, :] * scale
    tf[:, :3, 3] = tf[:, :3, 3] + transl * scale
    if not absolute:
        tf = torch.einsum('nij,njk->nik', tf, tfs_c_inv)
    return {"smpl_verts": out_verts, "smpl_tfs": tf}


def smpl_canonical_tfs_inv(model, betas):
    """SMPLServer.__init__, smpl.py:35-47: canonical pose (hips +-pi/6 about z), absolute transforms, inverted."""
    th = torch.zeros(72)
    th[5] = np.pi / 6
    th[8] = -np.pi / 6
    out = smpl_server_forward(model, None, torch.ones(1), torch.zeros(3), th, betas, absolute=True)
    return out["smpl_tfs"].inverse(), out["smpl_verts"]


# --------------------------------------------------------------------------------------
# rays (lib/utils/rend_util.py)
# --------------------------------------------------------------------------------------


def get_camera_params(uv, pose, intrinsics):
    """rend_util.get_camera_params + lift, rend_util.py:45-87 (4x4 pose branch)."""
    cam_loc = pose[:, :3, 3]
    p = pose
    b, n, _ = uv.shape
    x = uv[:, :, 0].view(b, -1)
    y = uv[:, :, 1].view(b, -1)
    z = torch.ones((b, n))
    fx = intrinsics[:, 0, 0]
    fy = intrinsics[:, 1, 1]
    cx = intrinsics[:, 0, 2]
    cy = intrinsics[:, 1, 2]
    sk = intrinsics[:, 0, 1]
    x_lift = (x - cx.unsqueeze(-1) + cy.unsqueeze(-1) * sk.unsqueeze(-1) / fy.unsqueeze(-1)
              - sk.unsqueeze(-1) * y / fy.unsqueeze(-1)) / fx.unsqueeze(-1) * z
    y_lift = (y - cy.unsqueeze(-1)) / fy.unsqueeze(-1) * z
    pts = torch.stack((x_lift, y_lift, z, torch.ones_like(z)), dim=-1).permute(0, 2, 1)
    world = torch.bmm(p, pts).permute(0, 2, 1)[:, :, :3]
    dirs = F.normalize(world - cam_loc[:, None, :], dim=2)
    return dirs, cam_loc


def get_sphere_intersections(cam_loc, ray_directions, r=1.0):
    """rend_util.get_sphere_intersections, rend_util.py:131-147."""
    dot = torch.bmm(ray_directions.view(-1, 1, 3), cam_loc.view(-1, 3, 1)).squeeze(-1)
    under = dot ** 2 - (cam_loc.norm(2, 1, keepdim=True) ** 2 - r ** 2)
    if (under <= 0).sum() > 0:
        raise RuntimeError("BOUNDING SPHERE PROBLEM!")   # reference calls exit()
    out = torch.sqrt(under) * torch.tensor([-1.0, 1.0]) - dot
    return out.clamp_min(0.0)


# --------------------------------------------------------------------------------------
# sampler (lib/model/ray_sampler.py), eval mode
# --------------------------------------------------------------------------------------


def _error_bound(beta, sdf, z_vals, dists, d_star):
    """ErrorBoundSampler.get_error_bound, ray_sampler.py:222-230."""
    density = laplace_density(sdf.reshape(z_vals.shape), beta)
    shifted = torch.cat([torch.zeros(dists.shape[0], 1, dtype=dists.dtype), dists * density[:, :-1]], dim=-1)
    integral = torch.cumsum(shifted, dim=-1)
    eps_sec = torch.exp(-d_star / beta) * (dists ** 2.) / (4 * beta ** 2)
    err_int = torch.cumsum(eps_sec, dim=-1)
    bound = (torch.clamp(torch.exp(err_int), max=1.e6) - 1.0) * torch.exp(-integral[:, :-1])
    return bound.max(-1)[0]


def _inverse_cdf_step(z_vals, sdf, d_star, beta, cont, u, add_tiny):
    """One trip's resampling after the line search, ray_sampler.py:124-186: the error-bound pdf (cont, :141-155) or the
    weights' pdf (final set, :157-165), the cdf and the inverse CDF at abscissae u."""
    dtype = z_vals.dtype
    dists = z_vals[:, 1:] - z_vals[:, :-1]
    density = laplace_density(sdf.reshape(z_vals.shape), beta.unsqueeze(-1))
    dists = torch.cat([dists, torch.tensor([1e10], dtype=dtype).unsqueeze(0).repeat(dists.shape[0], 1)], -1)
    free_energy = dists * density
    shifted = torch.cat([torch.zeros(dists.shape[0], 1, dtype=dtype), free_energy[:, :-1]], dim=-1)
    alpha = 1 - torch.exp(-free_energy)
    transmittance = torch.exp(-torch.cumsum(shifted, dim=-1))
    weights = alpha * transmittance
    if cont:
        eps_sec = torch.exp(-d_star / beta.unsqueeze(-1)) * (dists[:, :-1] ** 2.) / (4 * beta.unsqueeze(-1) ** 2)
        err_int = torch.cumsum(eps_sec, dim=-1)
        bound_opacity = (torch.clamp(torch.exp(err_int), max=1.e6) - 1.0) * transmittance[:, :-1]
        pdf = bound_opacity + add_tiny
    else:
        pdf = weights[..., :-1]
        pdf = pdf + 1e-5
    pdf = pdf / torch.sum(pdf, -1, keepdim=True)
    cdf = torch.cumsum(pdf, -1)
    cdf = torch.cat([torch.zeros_like(cdf[..., :1]), cdf], -1)
    bins = z_vals
    inds = torch.searchsorted(cdf, u, right=True)
    below = torch.max(torch.zeros_like(inds - 1), inds - 1)
    above = torch.min((cdf.shape[-1] - 1) * torch.ones_like(inds), inds)
    inds_g = torch.stack([below, above], -1)
    matched = [inds_g.shape[0], inds_g.shape[1], cdf.shape[-1]]
    cdf_g = torch.gather(cdf.unsqueeze(1).expand(matched), 2, inds_g)
    bins_g = torch.gather(bins.unsqueeze(1).expand(matched), 2, inds_g)
    denom_raw = cdf_g[..., 1] - cdf_g[..., 0]
    denom = torch.where(denom_raw < 1e-5, torch.ones_like(denom_raw), denom_raw)
    t = (u - cdf_g[..., 0]) / denom
    samples = bins_g[..., 0] + t * (bins_g[..., 1] - bins_g[..., 0])
    return dict(pdf=pdf, cdf=cdf, below=below, above=above, denom_raw=denom_raw, denom=denom, samples=samples)


def error_bound_get_z_vals(ray_dirs, cam_loc, person, cfg, beta_param, sdf_fn=None, stats=None, rng=None,
                           dtype=torch.float32, ray_sdf_fn=None, trace=None):
    """ErrorBoundSampler.get_z_vals (inverse_sphere_bg=True), ray_sampler.py:66-220.

    Eval mode (``rng is None``): returns (z_vals [R,S+X+2], z_bg [R,32]).
    Training mode (``model.training``): every random draw of the reference is an INPUT (``rng``), in the order the
    reference draws them —
      t_rand [R,E]   stratified jitter of the uniform start samples      ray_sampler.py:32-40
      u_final [R,S]  the inverse-CDF abscissae of the final sample set   :171
      extra_perm [M] torch.randperm(M) whose first X entries pick the extra samples (M = trips * E)   :202
      eik_idx [R]    torch.randint(S+X+2, (R,)) for z_samples_eik         :212-213
      t_rand_bg [R,32]  jitter of the inverse-sphere samples (the UniformSampler sees model.training too)   :216
    — the SDF callback does not clamp outliers (multiply.py:142 is eval-only) and the return is
    (z_vals, z_bg, z_samples_eik [R,1]).  ``stats`` (dict) receives 'trips'.

    ``dtype``: the floating type of every tensor the sampler creates (the reference's is float32; float64 gives a
    high-precision restatement of the same algorithm).  ``ray_sdf_fn(cam_loc [R,3], z [R,N], ray_dirs [R,3]) -> sdf
    [R*N,1]`` replaces ``sdf_fn`` when the caller builds the sample points itself.  ``trace`` (dict) receives
    ``trips``, one dict per trip with the state after its line search and the margin of every discrete decision:
      z, sdf [R,M], beta [R]      the sorted list, its SDF and the beta of the line search
      err0 [R]                    the error bound at beta0 (get_error_bound, :222-230)
      err_margin [R]              min over the line search's tests `err <= eps` of |err - eps| / eps
      flag, flag_margin           the batch test beta.max() > beta0 (:137), and |max(err0) - eps| / eps: how far the
                                  slowest ray's error is from eps
      final                       whether this trip drew the final set
      cdf [R,M]; u, below, above, denom_raw, denom, samples [R,N]   the inverse CDF (:166-186)
      u_margin [R,N]              distance of each abscissa to the nearest cdf entry that can decide it: cdf[0] = 0 is
                                  exact on every side and is left out; u = 1 gets inf, its bin is decided by how the
                                  cdf's tail rounds against 1 (see cdf_last, pdf_last)
      denom_margin [R,N]          |cdf[above] - cdf[below] - 1e-5|, the `denom < 1e-5` test
      cdf_last [R]                cdf[M-1] - 1: at u = 1 this decides whether the sample is z[M-1] (cdf[M-1] <= 1) or
                                  lies inside the last bin
      pdf_last [R]                the last bin's normalised pdf: below 1e-5 the sample in the last bin is b0 + (1 -
                                  cdf[M-2]) (b1 - b0), a whole interval from z[M-1]
      merge_margin [R,N]          distance of each new sample to the nearest list value it is merged with (0 = tie)
      order [R,M+N]               the sort index of cat([z, samples]) (non-final trips)."""
    S, E, X = cfg["N_samples"], cfg["N_samples_eval"], cfg["N_samples_extra"]
    eps, beta_iters, max_iters = cfg["eps"], cfg["beta_iters"], cfg["max_total_iters"]
    add_tiny, bound_r = cfg["add_tiny"], cfg["scene_bounding_sphere"]
    near_v = cfg.get("near", 0.0)
    training = rng is not None
    if sdf_fn is None:
        sdf_fn = lambda pts: sdf_func_with_smpl_deformer(pts, person, cfg, training=training)[0]
    if ray_sdf_fn is None:
        ray_sdf_fn = lambda o, z, d: sdf_fn((o.unsqueeze(1) + z.unsqueeze(2) * d.unsqueeze(1)).reshape(-1, 3))
    if trace is not None:
        trace["trips"] = []
    ray_dirs, cam_loc = ray_dirs.to(dtype), cam_loc.to(dtype)
    R = ray_dirs.shape[0]
    beta0 = get_beta(beta_param).to(dtype)

    # UniformSampler.get_z_vals, ray_sampler.py:21-42 (take_sphere_intersection=True, eval)
    si = get_sphere_intersections(cam_loc, ray_dirs, r=bound_r)
    near = near_v * torch.ones(R, 1, dtype=dtype)
    far = si[:, 1:]
    t_vals = torch.linspace(0., 1., steps=E, dtype=dtype)
    z_vals = near * (1. - t_vals) + far * t_vals
    if training:      # ray_sampler.py:32-40
        mids = .5 * (z_vals[..., 1:] + z_vals[..., :-1])
        upper = torch.cat([mids, z_vals[..., -1:]], -1)
        lower = torch.cat([z_vals[..., :1], mids], -1)
        z_vals = lower + (upper - lower) * rng["t_rand"].to(dtype)
    samples, samples_idx = z_vals, None

    dists = z_vals[:, 1:] - z_vals[:, :-1]
    bound = (1.0 / (4.0 * torch.log(torch.tensor(eps + 1.0, dtype=dtype)))) * (dists ** 2.).sum(-1)
    beta = torch.sqrt(bound)

    total_iters, not_converge = 0, True
    sdf = None
    while not_converge and total_iters < max_iters:
        with torch.no_grad():
            samples_sdf = ray_sdf_fn(cam_loc, samples, ray_dirs).to(dtype)
        if samples_idx is not None:
            sdf_merge = torch.cat([sdf.reshape(-1, z_vals.shape[1] - samples.shape[1]),
                                   samples_sdf.reshape(-1, samples.shape[1])], -1)
            sdf = torch.gather(sdf_merge, 1, samples_idx).reshape(-1, 1)
        else:
            sdf = samples_sdf

        d = sdf.reshape(z_vals.shape)
        dists = z_vals[:, 1:] - z_vals[:, :-1]
        a, b, c = dists, d[:, :-1].abs(), d[:, 1:].abs()
        first_cond = a.pow(2) + b.pow(2) <= c.pow(2)
        second_cond = a.pow(2) + c.pow(2) <= b.pow(2)
        d_star = torch.zeros(z_vals.shape[0], z_vals.shape[1] - 1, dtype=dtype)
        d_star[first_cond] = b[first_cond]
        d_star[second_cond] = c[second_cond]
        s = (a + b + c) / 2.0
        area_before_sqrt = s * (s - a) * (s - b) * (s - c)
        mask = ~first_cond & ~second_cond & (b + c - a > 0)
        d_star[mask] = (2.0 * torch.sqrt(area_before_sqrt[mask])) / (a[mask])
        d_star = (d[:, 1:].sign() * d[:, :-1].sign() == 1) * d_star

        curr_error = _error_bound(beta0, sdf, z_vals, dists, d_star)
        if trace is not None:
            # the test at beta0 picks beta0 or the bisection result, which lies between beta0 and the start beta
            tr = dict(z=z_vals.clone(), sdf=d.clone(), d_star=d_star, err0=curr_error.clone(), beta_init=beta.clone(),
                      err_steps=[(curr_error - eps) / eps], brackets=[(beta - beta0).abs()])
        beta[curr_error <= eps] = beta0
        beta_min, beta_max = beta0.unsqueeze(0).repeat(z_vals.shape[0]), beta
        for _ in range(beta_iters):
            beta_mid = (beta_min + beta_max) / 2.
            curr_error = _error_bound(beta_mid.unsqueeze(-1), sdf, z_vals, dists, d_star)
            if trace is not None:
                tr["err_steps"].append((curr_error - eps) / eps)
                tr["brackets"].append((beta_max - beta_min).abs())
            beta_max[curr_error <= eps] = beta_mid[curr_error <= eps]
            beta_min[curr_error > eps] = beta_mid[curr_error > eps]
        beta = beta_max

        total_iters += 1
        not_converge = bool(beta.max() > beta0)
        cont = not_converge and total_iters < max_iters
        if cont or not training:      # ray_sampler.py:166-170
            u = torch.linspace(0., 1., steps=E if cont else S, dtype=dtype).unsqueeze(0).repeat(R, 1).contiguous()
        else:
            u = rng["u_final"].to(dtype).contiguous()
        st_ = _inverse_cdf_step(z_vals, sdf, d_star, beta, cont, u, add_tiny)
        cdf, pdf, below, above, denom_raw, denom, samples = (st_[k] for k in (
            "cdf", "pdf", "below", "above", "denom_raw", "denom", "samples"))

        if trace is not None:
            gap = (u.unsqueeze(-1) - cdf[:, 1:].unsqueeze(1)).abs()
            gap = torch.where((u == 1).unsqueeze(-1), torch.full_like(gap, math.inf), gap)
            # a ray raises the batch flag (beta.max() > beta0 after the line search) iff err0 > eps and its start beta
            # exceeds beta0; the flag's margin is that of its most robust raiser, or of its least robust non-raiser
            raise_m = torch.minimum((tr["err0"] - eps) / eps, (tr["beta_init"] - beta0) / beta0)
            tr.update(beta=beta.clone(), flag=not_converge, final=not cont,
                      flag_margin=float(raise_m.max() if not_converge else -raise_m.max()),
                      err_steps=torch.stack(tr["err_steps"], 1), brackets=torch.stack(tr["brackets"], 1),
                      cdf=cdf, u=u, below=below, above=above, denom_raw=denom_raw, denom=denom, samples=samples,
                      u_margin=gap.min(-1)[0], denom_margin=(denom_raw - 1e-5).abs(), cdf_last=cdf[:, -1] - 1,
                      pdf_last=pdf[:, -1],
                      merge_margin=(samples.unsqueeze(-1) - z_vals.unsqueeze(1)).abs().min(-1)[0])
            trace["trips"].append(tr)

        if cont:
            z_vals, samples_idx = torch.sort(torch.cat([z_vals, samples], -1), -1)
            if trace is not None:
                tr["order"] = samples_idx

    if stats is not None:
        stats["trips"] = total_iters
        stats["beta"] = beta.clone()
    z_samples = samples
    near = near_v * torch.ones(R, 1, dtype=dtype)
    far = get_sphere_intersections(cam_loc, ray_dirs, r=bound_r)[:, 1:]
    if X > 0:
        if training:
            assert rng["extra_perm"].shape[0] == z_vals.shape[1], "randperm(M) was drawn for another trip count"
            sampling_idx = rng["extra_perm"][:X].long()
        else:
            sampling_idx = torch.linspace(0, z_vals.shape[1] - 1, X).long()
        z_extra = torch.cat([near, far, z_vals[:, sampling_idx]], -1)
    else:
        z_extra = torch.cat([near, far], -1)
    z_out, _ = torch.sort(torch.cat([z_samples, z_extra], -1), -1)

    # inverse-sphere background samples: UniformSampler(1.0, 0.0, 32, False, far=1.0), ray_sampler.py:215-218
    tb = torch.linspace(0., 1., steps=32, dtype=dtype)
    z_bg = torch.zeros(R, 1, dtype=dtype) * (1. - tb) + torch.ones(R, 1, dtype=dtype) * tb
    if training:
        z_eik = torch.gather(z_out, 1, rng["eik_idx"].long().unsqueeze(-1))      # ray_sampler.py:212-213
        mids = .5 * (z_bg[..., 1:] + z_bg[..., :-1])
        upper = torch.cat([mids, z_bg[..., -1:]], -1)
        lower = torch.cat([z_bg[..., :1], mids], -1)
        z_bg = lower + (upper - lower) * rng["t_rand_bg"].to(dtype)
        return z_out, z_bg * (1. / bound_r), z_eik
    return z_out, z_bg * (1. / bound_r)


# --------------------------------------------------------------------------------------
# colour / normals (lib/model/multiply.py:600-661)
# --------------------------------------------------------------------------------------


def forward_gradient(pnts_c, person, cfg):
    """Multiply.forward_gradient (eval), multiply.py:620-661: returns (normal_dir, feature)."""
    pnts_c = pnts_c.detach().clone().requires_grad_(True)
    w, _ = query_skinning_weights(pnts_c.detach()[None], person["verts_c"], person["weights"][None])
    pnts_d = skinning(pnts_c.unsqueeze(0), w, person["tfs"][None], inverse=False).squeeze(0)
    grads = []
    for i in range(3):
        d_out = torch.zeros_like(pnts_d)
        d_out[:, i] = 1
        g = torch.autograd.grad(pnts_d, pnts_c, d_out, retain_graph=True)[0]
        grads.append(g)
    grads = torch.stack(grads, dim=-2)
    grads_inv = grads.inverse()
    out = implicit_forward(person["implicit"], pnts_c, person["cond"], cfg["multires"])
    sdf = out[:, :1]
    feature = out[:, 1:]
    gradients = torch.autograd.grad(sdf, pnts_c, torch.ones_like(sdf))[0]
    nrm = F.normalize(torch.einsum('bi,bij->bj', gradients, grads_inv), dim=1)
    return nrm.detach(), feature.detach()


def get_rbg_value(pnts_c, person, cfg, chunk=32768):
    """Multiply.get_rbg_value (eval, pose_no_view), multiply.py:600-618."""
    rgbs, nrms = [], []
    for s in range(0, max(pnts_c.shape[0], 1), chunk):
        pc = pnts_c[s:s + chunk]
        g, feat = forward_gradient(pc, person, cfg)
        normals = F.normalize(g, dim=-1, eps=1e-6)
        rgb = rendering_forward(person["render"], "pose_no_view", pc, normals, None, person["cond"], feat)
        rgbs.append(rgb[:, :3])
        nrms.append(normals)
    return torch.cat(rgbs), torch.cat(nrms)


# --------------------------------------------------------------------------------------
# canonical SDF grid queries (multiply.py:169-172, lib/utils/mesh.py:78-105)
# --------------------------------------------------------------------------------------


def mesh_bounds(verts, scale=1.1):
    """generate_mesh, lib/utils/mesh.py:80-86: centre / longest side of the tight vertex box, padding factor."""
    v = verts.detach().cpu().numpy().reshape(-1, 3)
    bbox = np.stack([v.min(axis=0), v.max(axis=0)], axis=0)
    return (bbox[0] + bbox[1]) * 0.5, (bbox[1] - bbox[0]).max(), scale


def query_oc(x, person, cfg):
    """Multiply.query_oc, multiply.py:169-172: canonical SDF at x [N,3] -> [N,1]."""
    with torch.no_grad():
        return implicit_forward(person["implicit"], x.reshape(-1, 3), person["cond"], cfg["multires"])[:, :1]


def sdf_grid(person, cfg, verts, res, scale=1.1):
    """The dense (res+1)^3 lattice of generate_mesh (:92-95 point mapping, numpy fp32) through query_oc."""
    center, extent, scale = mesh_bounds(verts, scale)
    idx = np.stack(np.meshgrid(np.arange(res + 1), np.arange(res + 1), np.arange(res + 1), indexing="ij"), -1).reshape(-1, 3)
    pts = idx.astype(np.float32)
    pts = (pts / res - 0.5) * scale
    pts = pts * extent + center
    return query_oc(torch.tensor(pts).float(), person, cfg)[:, 0].reshape(res + 1, res + 1, res + 1), pts


# --------------------------------------------------------------------------------------
# background (multiply.py:514-539, 682-726)
# --------------------------------------------------------------------------------------


def depth2pts_outside(ray_o, ray_d, depth, bound_r):
    """Multiply.depth2pts_outside, multiply.py:698-726."""
    o_dot_d = torch.sum(ray_d * ray_o, dim=-1)
    under_sqrt = o_dot_d ** 2 - ((ray_o ** 2).sum(-1) - bound_r ** 2)
    d_sphere = torch.sqrt(under_sqrt) - o_dot_d
    p_sphere = ray_o + d_sphere.unsqueeze(-1) * ray_d
    p_mid = ray_o - o_dot_d.unsqueeze(-1) * ray_d
    p_mid_norm = torch.norm(p_mid, dim=-1)
    rot_axis = torch.cross(ray_o, p_sphere, dim=-1)
    rot_axis = rot_axis / torch.norm(rot_axis, dim=-1, keepdim=True)
    phi = torch.asin(p_mid_norm / bound_r)
    theta = torch.asin(p_mid_norm * depth)
    rot_angle = (phi - theta).unsqueeze(-1)
    p_new = p_sphere * torch.cos(rot_angle) + \
        torch.cross(rot_axis, p_sphere, dim=-1) * torch.sin(rot_angle) + \
        rot_axis * torch.sum(rot_axis * p_sphere, dim=-1, keepdim=True) * (1. - torch.cos(rot_angle))
    p_new = p_new / torch.norm(p_new, dim=-1, keepdim=True)
    return torch.cat((p_new, depth.unsqueeze(-1)), dim=-1)


def bg_volume_rendering(z_vals_bg, bg_sdf):
    """Multiply.bg_volume_rendering with AbsDensity, multiply.py:682-696."""
    dens = torch.abs(bg_sdf).reshape(-1, z_vals_bg.shape[1])
    d = z_vals_bg[:, :-1] - z_vals_bg[:, 1:]
    d = torch.cat([d, torch.tensor([1e10]).unsqueeze(0).repeat(d.shape[0], 1)], -1)
    fe = d * dens
    sh = torch.cat([torch.zeros(d.shape[0], 1), fe[:, :-1]], dim=-1)
    alpha = 1 - torch.exp(-fe)
    T = torch.exp(-torch.cumsum(sh, dim=-1))
    return alpha * T


def background_rgb(ray_dirs, cam_loc, scene, z_bg):
    """multiply.py:514-539 (eval, no shadow channel)."""
    cfg = scene["cfg"]
    nb = z_bg.shape[1]
    zb = torch.flip(z_bg, dims=[-1])
    bg_dirs = ray_dirs.unsqueeze(1).repeat(1, nb, 1)
    bg_locs = cam_loc.unsqueeze(1).repeat(1, nb, 1)
    pts = depth2pts_outside(bg_locs, bg_dirs, zb, cfg["scene_bounding_sphere"]).reshape(-1, 4)
    out = implicit_forward(scene["bg_implicit"], pts, scene["frame_code"], cfg["bg_multires"],
                           weight_norm=False)
    bg_sdf = out[:, :1]
    feat = out[:, 1:]
    rgb = rendering_forward(scene["bg_render"], "nerf_frame_encoding", None, None, bg_dirs.reshape(-1, 3),
                            None, feat, frame_latent_code=scene["frame_code"], weight_norm=False,
                            multires_view=cfg["bg_multires_view"]).reshape(-1, nb, 3)
    w = bg_volume_rendering(zb, bg_sdf)
    return torch.sum(w.unsqueeze(-1) * rgb, 1)


# --------------------------------------------------------------------------------------
# composite (multiply.py:425-480)
# --------------------------------------------------------------------------------------


def composite_nerfacc(index_ray_box_list, z_vals_list, z_max_list, sdf_list, rgb_list, nrm_list,
                      person_list, n_rays, beta_param):
    """The flatten / sort / nerfacc block, multiply.py:427-480.

    Tie order: the reference's first sort (multiply.py:443) is unstable; here ties on t_end
    keep (person, sample) order (stable) — ties only occur on zero-density intervals
    (SURVEY.md §7 'tie hazards')."""
    N = z_vals_list[0].shape[1]
    ray = torch.cat([ix.unsqueeze(1).repeat(1, N).flatten() for ix in index_ray_box_list]).float().unsqueeze(-1)
    zm = [torch.cat([z, m.unsqueeze(-1)], dim=1) for z, m in zip(z_vals_list, z_max_list)]
    zs = torch.cat([z[:, :-1].flatten() for z in zm]).unsqueeze(-1)
    ze = torch.cat([z[:, 1:].flatten() for z in zm]).unsqueeze(-1)
    sdf = torch.cat([s.flatten() for s in sdf_list]).unsqueeze(-1)
    rgb = torch.cat([c.reshape(-1, 3) for c in rgb_list])
    nrm = torch.cat([c.reshape(-1, 3) for c in nrm_list])
    pid = torch.cat([torch.full((z.shape[0] * N,), float(p)) for z, p in zip(z_vals_list, person_list)]).unsqueeze(-1)
    tab = torch.cat([ray, zs, ze, sdf, rgb, nrm, pid], dim=1)
    _, si = torch.sort(tab[:, 2], descending=False, dim=0, stable=True)
    tab = tab[si]
    _, ri = torch.sort(tab[:, 0], descending=False, dim=0, stable=True)
    tab = tab[ri]
    ray_indices = tab[:, 0].long()
    t_s, t_e = tab[:, 1], tab[:, 2]
    sig = laplace_density(tab[:, 3], get_beta(beta_param))
    weights, trans, _ = render_weight_from_density(t_s, t_e, sig, ray_indices=ray_indices, n_rays=n_rays)
    info = pack_info(ray_indices, n_rays)
    valid = info[info[:, 1] != 0]
    last = valid[1:, 0].long() - 1
    last = torch.cat([last, torch.tensor([weights.shape[0] - 1])], dim=0)
    bg_T = torch.ones(n_rays)
    bg_T[ray_indices[last]] = trans[last]
    acc_rgb = accumulate_along_rays(weights, tab[:, 4:7], ray_indices, n_rays)
    acc_nrm = accumulate_along_rays(weights, tab[:, 7:10], ray_indices, n_rays)
    acc_w = accumulate_along_rays(weights, None, ray_indices, n_rays).reshape(-1)
    acc_p = []
    for p in person_list:
        m = tab[:, 10] == p
        acc_p.append(accumulate_along_rays(weights[m], None, ray_indices[m], n_rays).reshape(-1))
    return acc_rgb, acc_nrm, acc_w, torch.stack(acc_p, dim=1), bg_T


# --------------------------------------------------------------------------------------
# the whole eval forward (multiply.py:174-598, eval branch, using_nerfacc=True)
# --------------------------------------------------------------------------------------


def eikonal_gradients(person, cfg, sample):
    """multiply.py:326-331 + gradient() (:728-738): d sdf / d x at the eikonal sample points [N,3] -> [N,3]."""
    x = sample.detach().clone().requires_grad_(True)
    out = implicit_forward(person["implicit"], x, person["cond"], cfg["multires"])
    return torch.autograd.grad(out[:, :1], x, torch.ones_like(out[:, :1]))[0].detach()


def multiply_forward(scene, inputs, hit_lists, with_bg=True, stats=None, return_samples=False, train=None):
    """Multiply.forward: eval branch, or — with ``train`` — the VALUES of the training branch for the shipped loss weights
    at current_epoch >= 250 (multiply.py:312-331, 393-484, 548-588; no smpl-surface / zero-pose / kaolin terms).
    ``train`` = dict(rng=[per person draws of get_z_vals, see error_bound_get_z_vals], eik_points=[per person [N,3]
    eikonal sample points, i.e. verts_c[randperm[:512]] + randn * 0.01, multiply.py:322-326 / sampler.py:100-103],
    t_rand_bg=[R,32] the draw of the second inverse-sphere call (:482)); adds 'grad_theta' [1, sum N, 3] and
    '_z_eik' to the output.

    scene: dict(cfg, persons=[dict(implicit, render, verts_p, verts_c, weights, tfs, cond)],
                bg_implicit, bg_render, frame_code, beta_param)
    inputs: dict(uv [1,R,2], pose [1,4,4], intrinsics [1,4,4])
    hit_lists: per person int64 tensor of ray indices (the reference computes these with
               trimesh on the host, multiply.py:256-263; they are an input here)."""
    cfg = scene["cfg"]
    ray_dirs, cam_loc = get_camera_params(inputs["uv"], inputs["pose"], inputs["intrinsics"])
    R = ray_dirs.shape[1]
    cam_loc = cam_loc.unsqueeze(1).repeat(1, R, 1).reshape(-1, 3)
    ray_dirs = ray_dirs.reshape(-1, 3)
    P = len(scene["persons"])
    zs, zmaxs, sdfs, rgbs, nrms, idxs = [], [], [], [], [], []
    trips, z_eiks, grad_theta = [], [], []
    for p in range(P):
        person = scene["persons"][p]
        idx = hit_lists[p]
        if idx.numel() == 0:
            idx = torch.tensor([0], dtype=torch.int64)          # multiply.py:262-263
        co, do = cam_loc[idx], ray_dirs[idx]
        st = {}
        if train is not None:
            z_vals, _, z_eik = error_bound_get_z_vals(do, co, person, cfg, scene["beta_param"], stats=st,
                                                      rng=train["rng"][p])
            z_eiks.append(z_eik)
            grad_theta.append(eikonal_gradients(person, cfg, train["eik_points"][p]))
        else:
            z_vals, _ = error_bound_get_z_vals(do, co, person, cfg, scene["beta_param"], stats=st)
        trips.append(st["trips"])
        z_max = z_vals[:, -1]
        z_vals = z_vals[:, :-1]
        n = z_vals.shape[1]
        pts = (co.unsqueeze(1) + z_vals.unsqueeze(2) * do.unsqueeze(1)).reshape(-1, 3)
        sdf, x_c, _ = sdf_func_with_smpl_deformer(pts, person, cfg, training=train is not None)
        rgb, nrm = get_rbg_value(x_c, person, cfg)
        zs.append(z_vals)
        zmaxs.append(z_max)
        sdfs.append(sdf.reshape(-1, n))
        rgbs.append(rgb.reshape(-1, n, 3))
        nrms.append(nrm.reshape(-1, n, 3))
        idxs.append(idx)
    fg_rgb, normal, acc, acc_p, bg_T = composite_nerfacc(idxs, zs, zmaxs, sdfs, rgbs, nrms, list(range(P)), R,
                                                         scene["beta_param"])
    if with_bg:
        tb = torch.linspace(0., 1., steps=32)
        z_bg = torch.zeros(R, 1) * (1. - tb) + torch.ones(R, 1) * tb
        if train is not None:      # the inverse-sphere UniformSampler sees model.training (ray_sampler.py:32-40)
            mids = .5 * (z_bg[..., 1:] + z_bg[..., :-1])
            upper = torch.cat([mids, z_bg[..., -1:]], -1)
            lower = torch.cat([z_bg[..., :1], mids], -1)
            z_bg = lower + (upper - lower) * train["t_rand_bg"]
        z_bg = z_bg * (1. / cfg["scene_bounding_sphere"])
        bg_rgb = background_rgb(ray_dirs, cam_loc, scene, z_bg)
    else:
        bg_rgb = torch.ones_like(fg_rgb)
    rgb_values = fg_rgb + bg_T.unsqueeze(-1) * bg_rgb
    out = {
        "acc_map": acc,
        "acc_person_list": acc_p,
        "rgb_values": rgb_values,
        "fg_rgb_values": fg_rgb + bg_T.unsqueeze(-1) * torch.ones_like(fg_rgb),
        "normal_values": normal,
    }
    if train is not None:
        out["grad_theta"] = torch.cat(grad_theta, 0).unsqueeze(0)       # multiply.py:564 (cat over persons, dim 1)
        out["_z_eik"] = z_eiks
    if stats is not None:
        stats["trips"] = trips
    if return_samples:
        out["_z_vals"] = zs
        out["_sdf"] = sdfs
        out["_rgb"] = rgbs
        out["_normals"] = nrms
        out["_bg_T"] = bg_T
    return out
