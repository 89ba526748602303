"""Synthetic stand-in scenes for the MultiPly hot path (SURVEY.md §8d).

The SMPL model files, the demo sequence and the pretrained init are licence-gated /
absent offline, so benchmarks and tests run on a synthetic scene with the same
shapes: a 6890-vertex capsule body on the SMPL kinematic tree, skinning weights,
bone transforms built exactly the way ``SMPLServer.forward`` builds them
(/root/reference/code/lib/model/smpl.py:50-95), geometric-init networks with the
shipped YAML dimensions (confs/model/taichi01_model.yaml:17-58).

Everything here is plain CPU torch/numpy and deterministic in its seeds; the CUDA
path and the oracle are fed the identical tensors.
"""
import math
import numpy as np
import torch

# SMPL kinematic tree (kintree_table of the SMPL pkl, read at lib/smpl/body_models.py:243)
PARENTS = [-1, 0, 0, 0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 9, 9, 12, 13, 14, 16, 17, 18, 19, 20, 21]

# approximate SMPL rest-pose joint locations (metres, T-pose)
_J = np.array([
    [0.00, 0.00, 0.00], [0.07, -0.09, 0.00], [-0.07, -0.09, 0.00], [0.00, 0.11, 0.00],
    [0.10, -0.47, 0.00], [-0.10, -0.47, 0.00], [0.00, 0.25, 0.00], [0.09, -0.87, -0.03],
    [-0.09, -0.87, -0.03], [0.00, 0.30, 0.00], [0.11, -0.93, 0.09], [-0.11, -0.93, 0.09],
    [0.00, 0.52, -0.02], [0.08, 0.43, -0.01], [-0.08, 0.43, -0.01], [0.00, 0.60, 0.02],
    [0.18, 0.46, -0.02], [-0.18, 0.46, -0.02], [0.44, 0.45, -0.03], [-0.44, 0.45, -0.03],
    [0.69, 0.45, -0.03], [-0.69, 0.45, -0.03], [0.77, 0.44, -0.03], [-0.77, 0.44, -0.03]], dtype=np.float64)
_RADIUS = np.array([0.13, 0.08, 0.08, 0.13, 0.065, 0.065, 0.13, 0.05, 0.05, 0.13, 0.04, 0.04,
                    0.06, 0.07, 0.07, 0.10, 0.06, 0.06, 0.045, 0.045, 0.04, 0.04, 0.035, 0.035])

DEFAULT_CFG = dict(
    # ray_sampler (confs/model/taichi01_model.yaml:67-76)
    near=0.0, N_samples=64, N_samples_eval=128, N_samples_extra=32, eps=0.1, beta_iters=10,
    max_total_iters=5, add_tiny=1.0e-6,
    scene_bounding_sphere=3.0,          # lib/model/multiply.py:85
    multires=6, bg_multires=10, bg_multires_view=4, dim_frame_encoding=32,
)


def make_cfg(S=64):
    """Sampler sizes scale 1:2:1/2 like the shipped 64/128/32 (SURVEY.md §8a size table)."""
    c = dict(DEFAULT_CFG)
    c.update(N_samples=S, N_samples_eval=2 * S, N_samples_extra=S // 2)
    return c


def _rodrigues(aa):
    """lib/smpl/lbs.py:276-307 (batch_rodrigues) in float64."""
    angle = np.linalg.norm(aa + 1e-8, axis=1, keepdims=True)
    d = aa / angle
    c, s = np.cos(angle)[:, :, None], np.sin(angle)[:, :, None]
    K = np.zeros((aa.shape[0], 3, 3))
    K[:, 0, 1], K[:, 0, 2] = -d[:, 2], d[:, 1]
    K[:, 1, 0], K[:, 1, 2] = d[:, 2], -d[:, 0]
    K[:, 2, 0], K[:, 2, 1] = -d[:, 1], d[:, 0]
    return np.eye(3)[None] + s * K + (1 - c) * (K @ K)


def _rigid_transform(rot, joints):
    """lib/smpl/lbs.py:323-378 (batch_rigid_transform): relative 4x4 transforms A [24,4,4]."""
    n = joints.shape[0]
    rel = joints.copy()
    rel[1:] -= joints[PARENTS[1:]]
    T = np.zeros((n, 4, 4))
    T[:, :3, :3] = rot
    T[:, :3, 3] = rel
    T[:, 3, 3] = 1
    chain = [T[0]]
    for i in range(1, n):
        chain.append(chain[PARENTS[i]] @ T[i])
    G = np.stack(chain)
    jh = np.concatenate([joints, np.zeros((n, 1))], 1)[:, :, None]
    corr = np.zeros((n, 4, 4))
    corr[:, :, 3:] = G @ jh
    return G - corr


def _capsules():
    """The body's capsules in the rest pose: end points a [25,3], b [25,3], radii [25]."""
    # bones: (parent joint -> joint) for j>=1, plus a head blob at joint 15 and a pelvis blob at 0
    seg_a = [_J[PARENTS[j]] for j in range(1, 24)] + [_J[15], _J[0]]
    seg_b = [_J[j] for j in range(1, 24)] + [_J[15] + np.array([0, 0.12, 0.0]), _J[0] + np.array([0, 0.02, 0])]
    seg_r = [_RADIUS[j] for j in range(1, 24)] + [0.10, 0.13]
    return np.array(seg_a), np.array(seg_b), np.array(seg_r)


def _skin_weights(verts):
    """Normalised Gaussian of the distance to the bone segment of each joint: [N,24]."""
    W = np.zeros((verts.shape[0], 24))
    for j in range(24):
        a = _J[PARENTS[j]] if j > 0 else _J[0]
        b = _J[j] if j > 0 else _J[0] + np.array([0, 0.05, 0])
        ab = b - a
        t = np.clip(((verts - a) @ ab) / (ab @ ab + 1e-12), 0, 1)
        d = np.linalg.norm(verts - (a + t[:, None] * ab), axis=1)
        W[:, j] = np.exp(-(d / 0.06) ** 2)
    W[W < 1e-4 * W.max(1, keepdims=True)] = 0
    W /= W.sum(1, keepdims=True)
    return W


def make_body(seed, V=6890):
    """Capsule body: rest verts [V,3], skinning weights [V,24] (row-sum 1)."""
    rng = np.random.RandomState(seed)
    seg_a, seg_b, seg_r = _capsules()
    length = np.linalg.norm(seg_b - seg_a, axis=1)
    area = 2 * math.pi * seg_r * (length + 2 * seg_r)
    counts = np.floor(area / area.sum() * V).astype(int)
    counts[0] += V - counts.sum()
    verts = []
    for a, b, r, c in zip(seg_a, seg_b, seg_r, counts):
        ax = b - a
        L = np.linalg.norm(ax)
        ax = ax / (L + 1e-12)
        t = rng.uniform(-r, L + r, size=c)
        dirs = rng.normal(size=(c, 3))
        dirs -= (dirs @ ax)[:, None] * ax[None]
        dirs /= np.linalg.norm(dirs, axis=1, keepdims=True) + 1e-12
        tc = np.clip(t, 0, L)
        over = t - tc                       # hemispherical caps
        rad = np.sqrt(np.maximum(r * r - over * over, 0.0))
        p = a[None] + (tc + over)[:, None] * ax[None] + rad[:, None] * dirs
        verts.append(p)
    verts = np.concatenate(verts, 0)[:V]
    return verts, _skin_weights(verts)


def _canonical_A():
    """Bone transforms of the canonical pose (hips +-pi/6 about z, lib/model/smpl.py:38-39)."""
    theta_c = np.zeros((24, 3))
    theta_c[1, 2] = math.pi / 6
    theta_c[2, 2] = -math.pi / 6
    return _rigid_transform(_rodrigues(theta_c), _J)


# Freudenthal split of a cube (corner bit 1 = +x, 2 = +y, 4 = +z) into 6 tetrahedra around the 0-7 diagonal; the same
# split in every cube, so the tetrahedra of neighbouring cubes share faces exactly
_TETS = np.array([[0, 1, 3, 7], [0, 1, 5, 7], [0, 2, 3, 7], [0, 2, 6, 7], [0, 4, 5, 7], [0, 4, 6, 7]])


def make_body_mesh(body_seed=100, step=0.033):
    """Triangle mesh of the capsule union of ``make_body`` in the canonical pose: (verts [V,3] fp32, faces [F,3] int64).

    Marching tetrahedra of the union's signed distance on a lattice of spacing ``step``: one vertex per lattice edge
    the surface crosses (shared by every tetrahedron around that edge), triangles oriented so that their normal points
    from the inside corners of their tetrahedron to the outside ones.  The result is watertight (every edge in exactly
    two faces, in opposite directions), consistently oriented (positive volume) and non-convex.  The canonical capsules
    are the rest-pose ones with their end points moved by the canonical pose's skinning (the weights of make_body).
    ``body_seed`` only shifts the lattice by a sub-step offset (no lattice point lies on the surface); the default step
    gives a face count of the order of SMPL's 13 776, step 0.005 about 3 x 10^5.  Deterministic."""
    seg_a, seg_b, seg_r = _capsules()
    A_c = _canonical_A()
    seg_a = lbs_np(seg_a, _skin_weights(seg_a), A_c)
    seg_b = lbs_np(seg_b, _skin_weights(seg_b), A_c)
    off = step * (0.25 + 0.5 * ((body_seed * 0.6180339887498949) % 1.0)) * np.array([1.0, 0.7548776662, 0.5698402910])
    pad = 3 * step
    lo = np.minimum(seg_a, seg_b).min(0) - seg_r.max() - pad - off
    hi = np.maximum(seg_a, seg_b).max(0) + seg_r.max() + pad
    n = np.ceil((hi - lo) / step).astype(int) + 1
    axes = [lo[k] + step * np.arange(n[k]) for k in range(3)]
    sdf = np.full(tuple(n), np.inf)
    for a, b, r in zip(seg_a, seg_b, seg_r):     # each capsule inside its own box (+ 2 steps): exact near every surface
        blo = np.maximum(np.floor((np.minimum(a, b) - r - 2 * step - lo) / step).astype(int), 0)
        bhi = np.minimum(np.ceil((np.maximum(a, b) + r + 2 * step - lo) / step).astype(int) + 1, n)
        X, Y, Z = np.meshgrid(*[axes[k][blo[k]:bhi[k]] for k in range(3)], indexing="ij")
        P = np.stack([X, Y, Z], -1)
        ab = b - a
        t = np.clip(((P - a) @ ab) / (ab @ ab + 1e-12), 0.0, 1.0)
        d = np.linalg.norm(P - (a + t[..., None] * ab), axis=-1) - r
        sl = tuple(slice(blo[k], bhi[k]) for k in range(3))
        sdf[sl] = np.minimum(sdf[sl], d)
    sdf[sdf == 0.0] = 1e-12
    # cubes with a sign change
    inside = sdf < 0
    corners = [(i & 1, (i >> 1) & 1, (i >> 2) & 1) for i in range(8)]
    cnt = sum(inside[dx:n[0] - 1 + dx, dy:n[1] - 1 + dy, dz:n[2] - 1 + dz].astype(np.int8) for dx, dy, dz in corners)
    cx, cy, cz = np.nonzero((cnt > 0) & (cnt < 8))
    gid = lambda x, y, z: (x * n[1] + y) * n[2] + z
    cid = np.stack([gid(cx + dx, cy + dy, cz + dz) for dx, dy, dz in corners], 1)      # [C,8]
    tv = cid[:, _TETS].reshape(-1, 4)                                                  # [T,4] lattice ids
    flat = sdf.reshape(-1)
    ts = flat[tv]
    tin = ts < 0
    k = tin.sum(1)
    keep = (k > 0) & (k < 4)
    tv, ts, tin, k = tv[keep], ts[keep], tin[keep], k[keep]
    order = np.argsort(~tin, axis=1, kind="stable")               # inside corners first
    tv = np.take_along_axis(tv, order, 1)
    tris = []
    for kk, pairs in ((1, [[(0, 1), (0, 2), (0, 3)]]), (3, [[(0, 3), (1, 3), (2, 3)]]),
                      (2, [[(0, 2), (0, 3), (1, 3)], [(0, 2), (1, 3), (1, 2)]])):
        sel = tv[k == kk]
        for tri in pairs:
            e = np.stack([np.sort(np.stack([sel[:, i], sel[:, j]], 1), 1) for i, j in tri], 1)     # [n,3,2]
            tris.append((e, sel, kk))
    edges = np.concatenate([e.reshape(-1, 2) for e, _, _ in tris], 0)
    uniq, inv = np.unique(edges, axis=0, return_inverse=True)
    inv = inv.reshape(-1)

    def pos(ids):
        x = ids // (n[1] * n[2])
        y = (ids // n[2]) % n[1]
        z = ids % n[2]
        return np.stack([axes[0][x], axes[1][y], axes[2][z]], -1)
    pa, pb = pos(uniq[:, 0]), pos(uniq[:, 1])
    sa, sb = flat[uniq[:, 0]], flat[uniq[:, 1]]
    verts = pa + (sa / (sa - sb))[:, None] * (pb - pa)
    faces, o = [], 0
    for e, sel, kk in tris:
        m = e.shape[0]
        f = inv[o:o + 3 * m].reshape(m, 3)
        o += 3 * m
        # orient: normal from the inside corners of the tetrahedron towards its outside corners
        pc = pos(sel)
        din = pc[:, :kk].mean(1)
        dout = pc[:, kk:].mean(1)
        v = verts[f]
        nrm = np.cross(v[:, 1] - v[:, 0], v[:, 2] - v[:, 0])
        flip = (nrm * (dout - din)).sum(1) < 0
        f[flip] = f[flip][:, [0, 2, 1]]
        faces.append(f)
    faces = np.concatenate(faces, 0)
    # canonical order: faces sorted by their vertex ids (independent of numpy's traversal)
    faces = faces[np.lexsort(faces.T[::-1])]
    return (torch.from_numpy(np.ascontiguousarray(verts.astype(np.float32))),
            torch.from_numpy(np.ascontiguousarray(faces.astype(np.int64))))


def lbs_np(verts, W, A):
    T = np.einsum("vj,jab->vab", W, A)
    vh = np.concatenate([verts, np.ones((verts.shape[0], 1))], 1)
    return np.einsum("vab,vb->va", T, vh)[:, :3]


def make_person(p, P, pose_std=0.2, scale=0.5):
    """Person p: canonical verts, posed verts, weights, bone transforms, pose conditioning.

    Mirrors SMPLServer.forward (lib/model/smpl.py:50-95): verts_p = s*(LBS(theta)+t);
    tfs = diag(s)-scaled A(theta) with t*s added, right-multiplied by A(theta_cano)^-1."""
    verts_t, W = make_body(100 + p)
    rng = np.random.RandomState(200 + p)
    # canonical pose: hips +-pi/6 about z (lib/model/smpl.py:38-39)
    theta_c = np.zeros((24, 3))
    theta_c[1, 2] = math.pi / 6
    theta_c[2, 2] = -math.pi / 6
    A_c = _rigid_transform(_rodrigues(theta_c), _J)
    verts_c = lbs_np(verts_t, W, A_c)
    theta = rng.normal(0, pose_std, size=(24, 3))
    theta[0] = rng.normal(0, 0.1, size=3)
    A_p = _rigid_transform(_rodrigues(theta), _J)
    transl = np.array([0.8 * (p - (P - 1) / 2.0), 0.15, 0.3 * p])
    verts_p = scale * lbs_np(verts_t, W, A_p) + transl * scale
    tf = A_p.copy()
    tf[:, :3, :] *= scale
    tf[:, :3, 3] += transl * scale
    tfs = np.einsum("nij,njk->nik", tf, np.linalg.inv(A_c))
    f32 = lambda a: torch.from_numpy(np.ascontiguousarray(a.astype(np.float32)))
    return dict(verts_c=f32(verts_c), verts_p=f32(verts_p), weights=f32(W), tfs=f32(tfs),
                smpl_pose=f32(theta.reshape(1, 72)),
                cond=f32(theta.reshape(1, 72)[:, 3:] / math.pi), scale=scale)


# ------------------------------------------------------------------------------------
# network parameter init (state-dict layout of lib/model/networks.py)
# ------------------------------------------------------------------------------------


def _wn(sd, name, w, b):
    """store as weight-norm pair (nn.utils.weight_norm, networks.py:82-83): g = ||v||_row, v = w."""
    sd[f"{name}.weight_g"] = w.norm(dim=1, keepdim=True).clone()
    sd[f"{name}.weight_v"] = w.clone()
    sd[f"{name}.bias"] = b.clone()


def init_implicit_fg(gen):
    """ImplicitNet geometric init, networks.py:55-76, dims of taichi01_model.yaml:17-30."""
    d0 = 39
    dims = [d0] + [256] * 8 + [257]
    sd = {}
    for l in range(9):
        out_dim = dims[l + 1] - d0 if (l + 1) == 4 else dims[l + 1]
        in_dim = dims[l] + (69 if l == 0 else 0)
        w = torch.empty(out_dim, in_dim)
        b = torch.zeros(out_dim)
        if l == 8:
            w.normal_(math.sqrt(math.pi) / math.sqrt(dims[l]), 0.0001, generator=gen)
            b.fill_(-0.6)
        elif l == 0:
            w.zero_()
            w[:, :3].normal_(0.0, math.sqrt(2) / math.sqrt(out_dim), generator=gen)
        elif l == 4:
            w.normal_(0.0, math.sqrt(2) / math.sqrt(out_dim), generator=gen)
            w[:, -(d0 - 3):] = 0.0
        else:
            w.normal_(0.0, math.sqrt(2) / math.sqrt(out_dim), generator=gen)
        if l == 0:
            # a trained net conditions on pose; give the cond columns small weights so the
            # folded bias path is exercised
            w[:, 39:].normal_(0.0, 0.02, generator=gen)
        _wn(sd, f"lin{l}", w, b)
    return sd


def _default_linear(out_dim, in_dim, gen):
    k = 1.0 / math.sqrt(in_dim)
    w = (torch.rand(out_dim, in_dim, generator=gen) * 2 - 1) * k
    b = (torch.rand(out_dim, generator=gen) * 2 - 1) * k
    return w, b


def init_render_fg(gen):
    """RenderingNet 'pose_no_view', networks.py:223-262, taichi01_model.yaml:31-38."""
    sd = {}
    w, b = _default_linear(8, 69, gen)
    sd["lin_pose.weight"], sd["lin_pose.bias"] = w, b
    dims = [270, 256, 256, 256, 256, 3]
    for l in range(5):
        w, b = _default_linear(dims[l + 1], dims[l], gen)
        if l == 4:
            w = w * 8.0      # spread the colours over (0,1) so RGB parity is a meaningful test
        _wn(sd, f"lin{l}", w, b)
    return sd


def init_implicit_bg(gen):
    """bg ImplicitNet (d_in 4, multires 10, cond 'frame', no weight-norm), yaml:39-50."""
    d0 = 84
    dims = [d0] + [256] * 8 + [257]
    sd = {}
    for l in range(9):
        out_dim = dims[l + 1] - d0 if (l + 1) == 4 else dims[l + 1]
        in_dim = dims[l] + (32 if l == 0 else 0)
        w, b = _default_linear(out_dim, in_dim, gen)
        sd[f"lin{l}.weight"], sd[f"lin{l}.bias"] = w, b
    return sd


def init_render_bg(gen):
    """bg RenderingNet 'nerf_frame_encoding' (315 -> 128 -> 3), yaml:51-58."""
    sd = {}
    dims = [315, 128, 3]
    for l in range(2):
        w, b = _default_linear(dims[l + 1], dims[l], gen)
        if l == 1:
            w = w * 6.0
        sd[f"lin{l}.weight"], sd[f"lin{l}.bias"] = w, b
    return sd


def make_scene(P=2, S=64, seed=42, beta=0.1, weights="geometric"):
    """weights: 'geometric' (the networks' initialisation) or 'trained' (perturb_networks(scene, seed) of it)."""
    gen = torch.Generator().manual_seed(seed)
    persons = []
    for p in range(P):
        d = make_person(p, P)
        d["implicit"] = init_implicit_fg(gen)
        d["render"] = init_render_fg(gen)
        persons.append(d)
    scene = dict(cfg=make_cfg(S), persons=persons,
                 bg_implicit=init_implicit_bg(gen), bg_render=init_render_bg(gen),
                 frame_code=torch.randn(1, 32, generator=torch.Generator().manual_seed(7)),
                 beta_param=beta)
    if weights == "trained":
        return perturb_networks(scene, seed)
    assert weights == "geometric", weights
    return scene


# ------------------------------------------------------------------------------------
# trained-like parameters
# ------------------------------------------------------------------------------------
# The geometric init zeroes or trivialises exactly what the MLP kernels treat specially: the Fourier columns of lin0 /
# lin4 are zero (no sin / cos term reaches the SDF or its gradient), weight_g = ||v||_row (the weight-norm fold is the
# identity) and the hidden biases are zero.  A trained checkpoint has none of this; perturb_networks makes parameters
# that look like one while the SDF stays a smooth surface around the body.

FOURIER_AMP = 0.2         # Fourier column noise of lin0 / lin4, relative to the xyz columns' std, times 2^-frequency
REL_NOISE = 0.1           # weight noise of every other layer, relative to the layer's weight std
HIDDEN_BIAS_STD = 0.05    # biases of lin0..lin7 (zero in the geometric init)


def _embed_freq(k, d=3):
    """Frequency index f of embedding column k ([x, sin(2^0 x), cos(2^0 x), sin(2^1 x), ...], embedders.py:8-34); -1
    for x itself."""
    return -1 if k < d else (k - d) // (2 * d)


def _noise(shape, std, gen):
    return torch.randn(*shape, generator=gen, dtype=torch.float64) * std


def _store_weight(sd, name, w, gen):
    """Effective weight w stored as a weight-norm pair whose g / ||v||_row = u ~ U(0.5, 2): v = w / u, g = ||v|| u."""
    u = 0.5 + 1.5 * torch.rand(w.shape[0], 1, generator=gen, dtype=torch.float64)
    v = w / u
    sd[f"{name}.weight_v"] = v.float()
    sd[f"{name}.weight_g"] = (v.norm(dim=1, keepdim=True) * u).float()


def _effective(sd, name):
    if f"{name}.weight_v" in sd:
        v = sd[f"{name}.weight_v"].double()
        return sd[f"{name}.weight_g"].double() * v / v.norm(dim=1, keepdim=True)
    return sd[f"{name}.weight"].double()


def _sdf64(sd, x, cond, multires=6):
    """fp64 SDF of a foreground ImplicitNet state dict at x [N,3] (networks.py:126-208); used to keep the surface in
    place when the parameters are perturbed."""
    emb = [x] + [f(x * 2.0 ** i) for i in range(multires) for f in (torch.sin, torch.cos)]
    emb = torch.cat(emb, -1)
    h = torch.cat([emb, cond.double().expand(x.shape[0], -1)], -1)
    for l in range(9):
        if l == 4:
            h = torch.cat([h, emb], -1) / math.sqrt(2)
        h = torch.nn.functional.linear(h, _effective(sd, f"lin{l}"), sd[f"lin{l}.bias"].double())
        if l < 8:
            h = torch.nn.functional.softplus(h, beta=100)
    return h[:, 0]


def _perturb_implicit_fg(sd, gen, d=3, multires=6, anchor=None):
    """anchor = (x [N,3], cond): lin8's sdf bias is shifted so that the median SDF at x is the unperturbed one's."""
    d0 = d * (1 + 2 * multires)
    out = {}
    for l in range(9):
        w = _effective(sd, f"lin{l}")
        b = sd[f"lin{l}.bias"].double().clone()
        if l in (0, 4):
            # columns of the input embedding: in lin0 the first d0, in lin4 (the skip input [h3, embed]) the last d0
            off = 0 if l == 0 else w.shape[1] - d0
            s_xyz = float(w[:, off:off + d].std())
            w[:, off:off + d] += _noise((w.shape[0], d), REL_NOISE * s_xyz, gen)
            for k in range(d, d0):
                w[:, off + k] = _noise((w.shape[0],), FOURIER_AMP * s_xyz * 2.0 ** -_embed_freq(k, d), gen)
            if l == 0:        # the pose-cond columns
                w[:, d0:] += _noise((w.shape[0], w.shape[1] - d0), REL_NOISE * float(w[:, d0:].std()), gen)
            else:             # the hidden part of lin4
                w[:, :off] += _noise((w.shape[0], off), REL_NOISE * float(w[:, :off].std()), gen)
        elif l == 8:
            # the geometric init gives every output row the same mean weight: spread the feature rows
            w[0] += _noise((w.shape[1],), 0.2 * float(w[0].mean()), gen)
            w[1:] += _noise((w.shape[0] - 1, w.shape[1]), float(w[1:].mean()), gen)
            b[1:] += _noise((b.shape[0] - 1,), 0.1, gen)
        else:
            w += _noise(w.shape, REL_NOISE * float(w.std()), gen)
        if l < 8:
            b += _noise(b.shape, HIDDEN_BIAS_STD, gen)
        _store_weight(out, f"lin{l}", w, gen)
        out[f"lin{l}.bias"] = b.float()
    if anchor is not None:
        # softplus is convex: noise on the pre-activations raises every hidden mean and with it the SDF; then scale the
        # SDF row so that the median |grad sdf| near the surface is 1, as the eikonal loss of a training run makes it
        x, cond = anchor
        shift = (_sdf64(out, x, cond) - _sdf64(sd, x, cond)).median()
        out["lin8.bias"][0] -= float(shift)
        x = x.clone().requires_grad_(True)
        y = _sdf64(out, x, cond)
        g = torch.autograd.grad(y.sum(), x)[0].norm(dim=1)
        c = 1.0 / float(g[y.detach().abs() < 0.05].median())
        out["lin8.weight_g"][0] *= c
        out["lin8.bias"][0] *= c
    return out


def _perturb_render_fg(sd, gen):
    out = {}
    n = len([k for k in sd if k.startswith("lin") and k.endswith(".bias") and "pose" not in k])
    for l in range(n):
        w = _effective(sd, f"lin{l}")
        w += _noise(w.shape, REL_NOISE * float(w.std()), gen)
        _store_weight(out, f"lin{l}", w, gen)
        out[f"lin{l}.bias"] = sd[f"lin{l}.bias"].clone()
    w = sd["lin_pose.weight"].double()
    out["lin_pose.weight"] = (w + _noise(w.shape, 0.5 * float(w.std()), gen)).float()
    b = sd["lin_pose.bias"].double()
    out["lin_pose.bias"] = (b + _noise(b.shape, 0.5 * float(b.std()), gen)).float()
    return out


def _perturb_plain(sd, gen):
    """Networks without weight norm (background): relative noise on every weight."""
    out = {}
    for k, v in sd.items():
        if k.endswith(".weight"):
            w = v.double()
            out[k] = (w + _noise(w.shape, REL_NOISE * float(w.std()), gen)).float()
        else:
            out[k] = v.clone()
    return out


def perturb_networks(scene, seed=0):
    """A copy of ``scene`` whose networks carry trained-like parameters, deterministic in ``seed``:
      - every weight gets noise, the zero Fourier columns of the foreground lin0 / lin4 included (their noise falls as
        2^-frequency, so the SDF stays smooth while sin / cos carry a good share of its gradient);
      - every weight-norm layer stores g = ||v||_row * U(0.5, 2) (the effective weight is the perturbed one);
      - lin0..lin7 of the foreground ImplicitNet get non-zero biases, the feature part of lin8's bias is perturbed;
      - the RenderingNet's lin_pose is perturbed as well;
      - lin8's SDF row is shifted and scaled so that the median SDF at the canonical body vertices is the unperturbed
        one's and the median |grad sdf| near the surface is 1.
    Bodies, cameras and the sampler configuration are shared with ``scene``."""
    gen = torch.Generator().manual_seed(10007 + seed)
    persons = []
    for person in scene["persons"]:
        anchor = (person["verts_c"].double(), person["cond"])
        persons.append(dict(person, implicit=_perturb_implicit_fg(person["implicit"], gen, anchor=anchor),
                            render=_perturb_render_fg(person["render"], gen)))
    return dict(scene, persons=persons, bg_implicit=_perturb_plain(scene["bg_implicit"], gen),
                bg_render=_perturb_plain(scene["bg_render"], gen))


# ------------------------------------------------------------------------------------
# camera, rays, hit lists
# ------------------------------------------------------------------------------------


def make_camera(f=900.0, res=512, cam_z=2.5):
    K = torch.eye(4)
    K[0, 0] = K[1, 1] = f
    K[0, 2] = K[1, 2] = res / 2
    pose = torch.eye(4)
    pose[1, 1] = -1.0
    pose[2, 2] = -1.0      # camera +z looks along world -z, image y points down
    pose[2, 3] = cam_z
    return K[None], pose[None]


def person_box(person, inflate=1.2):
    """Axis-aligned stand-in for trimesh's oriented box x1.2 (lib/model/multiply.py:208-214):
    returns (center[3], half_extent[3])."""
    v = person["verts_p"]
    lo, hi = v.min(0)[0], v.max(0)[0]
    return (lo + hi) / 2, (hi - lo) / 2 * inflate


def ray_box_hits(cam_loc, ray_dirs, center, half):
    """Slab test; returns sorted int64 ray indices (the list the reference gets from
    trimesh RayMeshIntersector.intersects_id, multiply.py:256-263)."""
    o = cam_loc.double() - center.double()
    d = ray_dirs.double()
    inv = 1.0 / torch.where(d.abs() < 1e-12, torch.full_like(d, 1e-12), d)
    t1 = (-half.double() - o) * inv
    t2 = (half.double() - o) * inv
    tmin = torch.minimum(t1, t2).max(1)[0]
    tmax = torch.maximum(t1, t2).min(1)[0]
    hit = (tmax >= torch.clamp(tmin, min=0.0))
    return torch.nonzero(hit).flatten()


def make_rays(scene, R, seed=1234, region="boxes", res=512):
    """uv [1,R,2] pixel coords.  region='image': uniform over the frame; 'boxes': uniform over
    the image-space bounding rectangle of all persons' boxes (the reference's training
    sampler concentrates rays on the human bounding box, lib/datasets/Hi4D.py:56)."""
    K, pose = make_camera(res=res)
    g = torch.Generator().manual_seed(seed)
    if region == "image":
        lo = torch.tensor([0.0, 0.0])
        hi = torch.tensor([float(res), float(res)])
    else:
        pts = []
        for person in scene["persons"]:
            c, h = person_box(person)
            for sx in (-1, 1):
                for sy in (-1, 1):
                    for sz in (-1, 1):
                        pts.append(c + h * torch.tensor([sx, sy, sz], dtype=torch.float32))
        pts = torch.stack(pts)
        w2c = torch.inverse(pose[0])
        pc = (w2c[:3, :3] @ pts.T + w2c[:3, 3:]).T
        u = K[0, 0, 0] * pc[:, 0] / pc[:, 2] + K[0, 0, 2]
        v = K[0, 1, 1] * pc[:, 1] / pc[:, 2] + K[0, 1, 2]
        lo = torch.stack([u.min(), v.min()]).clamp(0, res)
        hi = torch.stack([u.max(), v.max()]).clamp(0, res)
    uv = lo + (hi - lo) * torch.rand(R, 2, generator=g)
    return dict(uv=uv[None].contiguous(), pose=pose, intrinsics=K)


def grid_rays(res=512, start=0, count=None):
    """Full-frame mgrid pixels (lib/datasets/Hi4D.py:254-255: uv = (x, y))."""
    K, pose = make_camera(res=res)
    ys, xs = torch.meshgrid(torch.arange(res), torch.arange(res), indexing="ij")
    uv = torch.stack([xs.flatten(), ys.flatten()], -1).float()
    if count is not None:
        uv = uv[start:start + count]
    return dict(uv=uv[None].contiguous(), pose=pose, intrinsics=K)


def make_hit_lists(scene, inputs, all_hit=False):
    """Per-person hit lists, computed once on the host and fed to both oracle and CUDA path."""
    from .model import rend_util
    dirs, cam = rend_util.get_camera_params_host(inputs["uv"], inputs["pose"], inputs["intrinsics"])
    R = dirs.shape[0]
    out = []
    for person in scene["persons"]:
        if all_hit:
            out.append(torch.arange(R, dtype=torch.int64))
        else:
            c, h = person_box(person)
            out.append(ray_box_hits(cam, dirs, c, h))
    return out


def make_smpl_model(seed=300, body_seed=100):
    """Synthetic stand-in for the licence-gated SMPL pkl: the arrays lib/smpl/body_models.py:SMPL registers
    (v_template, shapedirs, posedirs, J_regressor, parents, lbs_weights), with SMPL's shapes."""
    rng = np.random.RandomState(seed)
    verts_t, W = make_body(body_seed)
    V = verts_t.shape[0]
    shapedirs = 0.01 * rng.randn(V, 3, 10)
    posedirs = 0.004 * rng.randn(207, V * 3)
    Jr = np.zeros((24, V))
    for j in range(24):
        d = np.linalg.norm(verts_t - _J[j], axis=1)
        idx = np.argsort(d)[:64]
        w = np.exp(-(d[idx] / 0.08) ** 2) + 1e-6
        Jr[j, idx] = w / w.sum()
    f32 = lambda a: torch.from_numpy(np.ascontiguousarray(a.astype(np.float32)))
    return dict(v_template=f32(verts_t), shapedirs=f32(shapedirs), posedirs=f32(posedirs), J_regressor=f32(Jr),
                parents=torch.tensor(PARENTS, dtype=torch.int64), lbs_weights=f32(W))


class SyntheticSMPLServer:
    """Offline stand-in for lib/model/smpl.py:SMPLServer (needs the licence-gated SMPL pkl): same call
    signature and output keys; the body is the capsule model above.  ``forward`` ignores betas (the
    capsule body has no shape space) and applies scale / translation / pose exactly as smpl.py:50-95."""

    def __init__(self, person_index=0, P=2):
        self.p, self.P = person_index, P
        verts_t, W = make_body(100 + person_index)
        self._verts_t, self._W = verts_t, W
        theta_c = np.zeros((24, 3))
        theta_c[1, 2] = math.pi / 6
        theta_c[2, 2] = -math.pi / 6
        self._A_c = _rigid_transform(_rodrigues(theta_c), _J)
        self._A_c_inv = np.linalg.inv(self._A_c)
        f32 = lambda a: torch.from_numpy(np.ascontiguousarray(a.astype(np.float32)))
        self.verts_c = f32(lbs_np(verts_t, W, self._A_c))[None]
        self.weights = f32(W)[None]
        self.scale = 1.0
        # canonical triangle mesh of the same capsules (the SMPL pkl's `f` over verts_c in the reference,
        # multiply.py:118-121); its own vertices, since verts_c here is a point cloud
        self.mesh_verts_c, self.faces = make_body_mesh(100 + person_index)

    def canonical_output(self):
        return self(torch.ones(1), torch.zeros(1, 3), torch.zeros(1, 72), torch.zeros(1, 10))

    def __call__(self, scale, transl, thetas, betas, absolute=False):
        s = float(scale.reshape(-1)[0])
        self.scale = s
        t = transl.detach().cpu().double().numpy().reshape(3)
        th = thetas.detach().cpu().double().numpy().reshape(24, 3)
        A_p = _rigid_transform(_rodrigues(th), _J)
        verts = s * lbs_np(self._verts_t, self._W, A_p) + t * s
        tf = A_p.copy()
        tf[:, :3, :] *= s
        tf[:, :3, 3] += t * s
        if not absolute:
            tf = np.einsum("nij,njk->nik", tf, self._A_c_inv)
        f32 = lambda a: torch.from_numpy(np.ascontiguousarray(a.astype(np.float32)))
        dev = thetas.device
        return {"smpl_verts": f32(verts)[None].to(dev), "smpl_tfs": f32(tf)[None].to(dev),
                "smpl_weights": self.weights.to(dev)}


# ------------------------------------------------------------------------------------
# drop-in scene: bodies produced by the DEVICE SMPL server (model.smpl.SMPLServer / mp_smpl_forward), so that
# Multiply.forward(input_dict) and the resident-input Renderer see the same scene (bench.py, tests)
# ------------------------------------------------------------------------------------

MODEL_OPT = dict(
    with_bkgd=True, num_training_frames=75, dim_frame_encoding=32,
    implicit_network=dict(feature_vector_size=256, d_in=3, d_out=1, dims=[256] * 8, init="geometry", bias=0.6,
                          skip_in=[4], weight_norm=True, embedder_mode="fourier", multires=6, cond="smpl"),
    rendering_network=dict(feature_vector_size=256, mode="pose_no_view", d_in=14, d_out=3, dims=[256] * 4,
                           weight_norm=True, multires_view=-1),
    bg_implicit_network=dict(feature_vector_size=256, d_in=4, d_out=1, dims=[256] * 8, init="none", bias=0.0,
                             skip_in=[4], weight_norm=False, embedder_mode="fourier", multires=10, cond="frame"),
    bg_rendering_network=dict(feature_vector_size=256, mode="nerf_frame_encoding", d_in=3, d_out=3, dims=[128],
                              weight_norm=False, multires_view=4),
    density=dict(params_init={"beta": 0.1}, beta_min=0.0001),
)


def smpl_scene_inputs(P, frame_index=3, pose_std=0.2, scale=0.5):
    """The SMPL entries of the reference's input dict for the synthetic P-person scene (SURVEY.md 8b)."""
    smpl_pose = torch.zeros(1, P, 72)
    smpl_trans = torch.zeros(1, P, 3)
    for p in range(P):
        rng = np.random.RandomState(200 + p)
        theta = rng.normal(0, pose_std, size=(24, 3))
        theta[0] = rng.normal(0, 0.1, size=3)
        smpl_pose[0, p] = torch.from_numpy(theta.reshape(72).astype(np.float32))
        smpl_trans[0, p] = torch.tensor([0.8 * (p - (P - 1) / 2.0), 0.15, 0.3 * p])
    smpl_params = torch.zeros(1, P, 86)
    smpl_params[:, :, 0] = scale
    return dict(smpl_params=smpl_params, smpl_pose=smpl_pose, smpl_shape=torch.zeros(1, P, 10),
                smpl_trans=smpl_trans, idx=torch.tensor([frame_index]))


def smpl_scene_networks(P, S, seed):
    """Networks / sampler config of the drop-in scene (everything but the bodies): returns (per-person net dicts, rest)."""
    gen = torch.Generator().manual_seed(seed)
    nets = [dict(implicit=init_implicit_fg(gen), render=init_render_fg(gen)) for _ in range(P)]
    rest = dict(cfg=make_cfg(S), bg_implicit=init_implicit_bg(gen), bg_render=init_render_bg(gen),
                frame_code=torch.randn(1, 32, generator=torch.Generator().manual_seed(7)), beta_param=0.1)
    return nets, rest


def model_opt(cfg):
    """The mirror ``Multiply``'s options: MODEL_OPT with the ray sampler of the scene config ``cfg``."""
    return dict(MODEL_OPT, ray_sampler=dict({k: v for k, v in cfg.items()
                                             if k in ("near", "N_samples", "N_samples_eval", "N_samples_extra", "eps",
                                                      "beta_iters", "max_total_iters", "add_tiny")},
                                            N_samples_inverse_sphere=32))


def mirror_state_dict(scene, frame_index=3):
    """The mirror ``Multiply``'s state dict for a make_scene-style dict: every person's foreground nets, the background
    nets, density.beta, and the frame latent, whose row ``frame_index`` holds the scene's frame code."""
    sd = {}
    for p, person in enumerate(scene["persons"]):
        for k, v in person["implicit"].items():
            sd[f"foreground_implicit_network_list.{p}.{k}"] = v
        for k, v in person["render"].items():
            sd[f"foreground_rendering_network_list.{p}.{k}"] = v
    for k, v in scene["bg_implicit"].items():
        sd["bg_implicit_network." + k] = v
    for k, v in scene["bg_render"].items():
        sd["bg_rendering_network." + k] = v
    sd["density.beta"] = torch.tensor(scene["beta_param"])
    fw = torch.zeros(75, 32)
    fw[frame_index] = scene["frame_code"][0]
    sd["frame_latent_encoder.weight"] = fw
    return sd


def mirror_model(scene, servers=None, culling="aabb", device="cuda", frame_index=3):
    """The mirror ``Multiply`` (eval, on ``device``) holding the weights of a make_scene-style dict; its SMPL servers
    are ``servers``, by default one SyntheticSMPLServer per person."""
    from .model.multiply import Multiply
    P = len(scene["persons"])
    if servers is None:
        servers = [SyntheticSMPLServer(p, P) for p in range(P)]
    model = Multiply(model_opt(scene["cfg"]), smpl_server_list=servers, culling=culling)
    model.load_state_dict(mirror_state_dict(scene, frame_index), strict=True)
    return model.to(device).eval()


def make_smpl_scene(P=2, S=64, seed=42, device="cuda", frame_index=3, pose_std=0.2, scale=0.5):
    """Returns (scene, model, smpl_inputs): `scene` is a make_scene-style dict (CPU tensors) whose persons are the
    outputs of the device SMPL servers for `smpl_inputs` (smpl_params / smpl_pose / smpl_shape / smpl_trans / idx, the
    reference's input-dict entries, SURVEY.md 8b); `model` is the mirror ``Multiply`` (eval, on `device`) holding the
    same weights and servers."""
    from .model.smpl import SMPLServer
    servers = [SMPLServer(model=make_smpl_model(300 + p, body_seed=100 + p), device=device) for p in range(P)]
    for p, srv in enumerate(servers):          # canonical mesh of the capsules (SyntheticSMPLServer)
        srv.mesh_verts_c, srv.faces = make_body_mesh(100 + p)
    smpl_inputs = smpl_scene_inputs(P, frame_index, pose_std, scale)
    smpl_params, smpl_pose, smpl_trans = smpl_inputs["smpl_params"], smpl_inputs["smpl_pose"], smpl_inputs["smpl_trans"]
    nets, rest = smpl_scene_networks(P, S, seed)
    persons = []
    for p in range(P):
        o = servers[p](smpl_params[:, p, 0], smpl_trans[:, p], smpl_pose[:, p], torch.zeros(1, 10))
        torch.cuda.synchronize()
        servers[p].scale = scale
        persons.append(dict(verts_c=servers[p].verts_c[0].cpu(), weights=servers[p].weights[0].cpu(),
                            verts_p=o["smpl_verts"][0].cpu(), tfs=o["smpl_tfs"][0].cpu(),
                            smpl_pose=smpl_pose[:, p].clone(), cond=smpl_pose[:, p, 3:] / math.pi, scale=scale,
                            implicit=nets[p]["implicit"], render=nets[p]["render"]))
    scene = dict(rest, persons=persons)
    model = mirror_model(scene, servers, device=device, frame_index=frame_index)
    return scene, model, smpl_inputs
