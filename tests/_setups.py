"""Set-ups the GPU tests share: scenes and their handles, mp_field_pack's network descriptors (and the pairs it
refuses, which the CPU size-query test uses too), the mirror's input dict, SMPL handles, points, rays, the
sampler's training draws, the compositor's synthetic inputs and the fused render with canonical meshes."""
import ctypes as C

import numpy as np
import pytest
import torch

from multiply_b200 import engine, scene as S, _lib as L

from _abi import padded, take


# ---------------------------------------------------------------------------------------------
# scenes
# ---------------------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def trained():
    """The trained-like scene: both persons' fields with their own cond, and the background field."""
    engine.set_engine("tc")
    sc = S.make_scene(P=2, S=16, seed=42, weights="trained")
    fields = []
    for p in sc["persons"]:
        f = engine.Field(p["implicit"], p["render"])
        f.set_cond(p["cond"])
        fields.append(f)
    bg = engine.Field(sc["bg_implicit"], sc["bg_render"], background=True)
    bg.set_cond(sc["frame_code"])
    return sc, fields, bg


def field_descs(implicit_sd, render_sd, background, device=None, **imp):
    """mp_field_pack's (implicit, render) descriptors of a state-dict pair, laid out as engine.Field lays them out, and
    the device tensors they point to; ``imp`` overrides descriptor fields (multires, skip_layer).  device None: every
    weight pointer NULL and lin_pose, where the state dict has it, a dummy address, since the size query reads only the
    dimensions and whether lin_pose is given."""
    keep = []

    def put(t):
        if device is None:
            return None
        keep.append(L.dev(t, device))
        return L.ptr(keep[-1])

    def stack(sd):
        st = L.LinearStack()
        st.n_layers = len([k for k in sd if k.startswith("lin") and k.endswith(".bias") and "pose" not in k])
        for l in range(st.n_layers):
            v = sd[f"lin{l}.weight_v"] if f"lin{l}.weight_v" in sd else sd[f"lin{l}.weight"]
            st.weight_v[l], st.weight_g[l], st.bias[l] = put(v), put(sd.get(f"lin{l}.weight_g")), put(sd[f"lin{l}.bias"])
            st.out_dim[l], st.in_dim[l] = v.shape
        return st

    d = L.ImplicitDesc(stack(implicit_sd), 4 if background else 3, 10 if background else 6, 32 if background else 69, 4)
    for k, v in imp.items():
        setattr(d, k, v)
    r = L.RenderDesc(stack(render_sd), 1 if background else 0, 4 if background else -1)
    if "lin_pose.weight" in render_sd:
        r.lin_pose_weight = put(render_sd["lin_pose.weight"]) if device else 256
        r.lin_pose_bias = put(render_sd["lin_pose.bias"]) if device else 256
    return d, r, keep


def _resized(sd, l, out, inp):
    """sd with layer l at out x inp (zero weights)."""
    sd = dict(sd)
    v = f"lin{l}.weight_v" if f"lin{l}.weight_v" in sd else f"lin{l}.weight"
    sd[v], sd[f"lin{l}.bias"] = torch.zeros(out, inp), torch.zeros(out)
    if f"lin{l}.weight_g" in sd:
        sd[f"lin{l}.weight_g"] = torch.ones(out, 1)
    return sd


def refused_fields(sc):
    """Every kind of network pair mp_field_pack refuses, made from scene ``sc``'s: (what, field_descs arguments, the
    message it is refused with)."""
    p = sc["persons"][0]
    fi, fr, bi, br = p["implicit"], p["render"], sc["bg_implicit"], sc["bg_render"]
    e7 = 3 * (1 + 2 * 7)       # multires 7: 15 embedding columns per axis, one more than the final-gradient step keeps
    return [
        ("layer count", ({k: v for k, v in fi.items() if not k.startswith("lin8.")}, fr, False, {}),
         "ImplicitNet must have 9 linear layers (got 8)"),
        ("skip layer", (fi, fr, False, dict(skip_layer=3)), "skip_in must be [4]"),
        ("implicit shape", (_resized(fi, 2, 255, 256), fr, False, {}), "implicit layer 2 has unsupported shape 255x256"),
        ("pose_no_view width", (fi, _resized(fr, 0, 256, 271), False, {}),
         "pose_no_view colour net must take 270 inputs and carry lin_pose"),
        ("nerf_frame_encoding width", (bi, _resized(br, 0, 128, 316), True, {}),
         "nerf_frame_encoding colour net has unsupported input width 316"),
        ("no lin_pose", (fi, {k: v for k, v in fr.items() if not k.startswith("lin_pose")}, False, {}),
         "pose_no_view colour net must take 270 inputs and carry lin_pose"),
        ("multires 7", (_resized(_resized(fi, 0, 256, e7 + 69), 3, 256 - e7, 256), fr, False, dict(multires=7)),
         "the final-gradient step keeps 1 + 2 * multires <= 14 embedding columns per axis"),
    ]


@pytest.fixture(scope="module")
def geo():
    """Person 0 of the geometric scene the sampler tests use: field, posed body."""
    engine.set_engine("tc")
    sc = S.make_scene(P=2, S=16, seed=42)
    p = sc["persons"][0]
    f = engine.Field(p["implicit"], p["render"])
    f.set_cond(p["cond"])
    b = engine.Body(p["verts_c"], p["weights"], cano_cell=0.1001 / p["scale"])
    b.set_pose(p["verts_p"], p["tfs"])
    return sc, f, b


# ---------------------------------------------------------------------------------------------
# the mirror
# ---------------------------------------------------------------------------------------------

def mirror_inputs(rays, P, hits=None, epoch=None):
    """The reference's input dict for the synthetic P-person scene, on the GPU: the rays' uv / pose / intrinsics and
    scene.smpl_scene_inputs(P); ``hits``: index_ray_box_list; ``epoch``: the training entries current_epoch and
    smpl_pose_last (the pose 0.01 off)."""
    d = dict(uv=rays["uv"], pose=rays["pose"], intrinsics=rays["intrinsics"], **S.smpl_scene_inputs(P))
    d = {k: v.cuda() for k, v in d.items()}
    if hits is not None:
        d["index_ray_box_list"] = hits
    if epoch is not None:
        d["current_epoch"] = epoch
        d["smpl_pose_last"] = d["smpl_pose"] + 0.01
    return d


def train(m, inputs, seed, id=-1):
    """Multiply.forward in .train() with torch's random stream at ``seed``."""
    m.train()
    try:
        torch.manual_seed(seed)
        out = m(inputs, id=id)
        torch.cuda.synchronize()
    finally:
        m.eval()
    return out


# ---------------------------------------------------------------------------------------------
# SMPL server and deformer
# ---------------------------------------------------------------------------------------------

def dirty_workspace(nbytes):
    """A workspace of ``nbytes`` (at least one) filled with 0xFF bytes: NaN floats, -1 ints."""
    return torch.full((max(int(nbytes), 1),), 0xFF, dtype=torch.uint8, device="cuda")


class Smpl:
    def __init__(self, model):
        self.model, self.V = model, model["v_template"].shape[0]
        self.d = {k: torch.as_tensor(np.ascontiguousarray(np.asarray(model[k]), np.float32)).cuda()
                  for k in ("v_template", "shapedirs", "posedirs", "J_regressor", "lbs_weights")}
        pa = (C.c_int * 24)(*[max(int(p), 0) for p in model["parents"]])
        self.storage = L.workspace(L.call("mp_smpl_bytes", self.V), "cuda")
        self.h = L.Handle("mp_smpl_free")
        d = self.d
        L.call("mp_smpl_create", d["v_template"], d["shapedirs"], d["posedirs"], d["J_regressor"], pa, d["lbs_weights"],
               self.V, None, self.storage, self.storage.numel(), C.byref(self.h))
        ti = torch.empty(24, 4, 4, device="cuda")
        L.call("mp_smpl_canonical", self.h, None, ti)
        self.cinv = ti.cpu().numpy()

    @staticmethod
    def _args(scale, transl, theta, betas):
        return [torch.from_numpy(np.asarray(a, np.float32).reshape(-1)).cuda() for a in ((scale,), transl, theta, betas)]

    def forward(self, scale, transl, theta, betas, absolute):
        v, t = torch.empty(self.V, 3, device="cuda"), torch.empty(24, 4, 4, device="cuda")
        L.call("mp_smpl_forward", self.h, *self._args(scale, transl, theta, betas), int(absolute), v, t)
        return v, t

    def backward(self, scale, transl, theta, betas, absolute, u_v, u_t):
        dv = None if u_v is None else torch.from_numpy(np.asarray(u_v, np.float32)).cuda()
        dt = None if u_t is None else torch.from_numpy(np.asarray(u_t, np.float32)).cuda()
        outs = [padded(n) for n in (1, 3, 72, 10)]
        ws = dirty_workspace(L.call("mp_smpl_backward_workspace_bytes", self.V))
        L.call("mp_smpl_backward", self.h, *self._args(scale, transl, theta, betas), int(absolute), dv, dt, *outs, ws,
               ws.numel())
        torch.cuda.synchronize()
        return [take(o, n, "d_" + k).numpy() for o, n, k in zip(outs, (1, 3, 72, 10), ("scale", "transl", "thetas", "betas"))]


def small_model(V, seed=301, dense=False):
    """scene.make_smpl_model's construction at V vertices (the first V of the capsule body); dense: every vertex
    regresses every joint (positive weights, rows summing to 1)."""
    rng = np.random.RandomState(seed)
    verts_t, W = S.make_body(100, V=V)
    V = verts_t.shape[0]
    Jr = np.zeros((24, V))
    if dense:
        Jr = rng.uniform(0.5, 1.5, (24, V))
        Jr /= Jr.sum(1, keepdims=True)
    else:
        for j in range(24):
            d = np.linalg.norm(verts_t - S._J[j], axis=1)
            idx = np.argsort(d)[:min(64, V)]
            w = np.exp(-(d[idx] / 0.08) ** 2) + 1e-6
            Jr[j, idx] = w / w.sum()
    f32 = lambda a: np.ascontiguousarray(a.astype(np.float32))
    return dict(v_template=f32(verts_t), shapedirs=f32(0.01 * rng.randn(V, 3, 10)),
                posedirs=f32(0.004 * rng.randn(207, V * 3)), J_regressor=f32(Jr),
                parents=np.array(S.PARENTS, np.int64), lbs_weights=f32(W))


_BODY = {}


def posed_body():
    """(engine.Body, SMPLServer) of make_smpl_model(300) at a random pose and shape, built once."""
    if "b" not in _BODY:
        from multiply_b200.model.smpl import SMPLServer
        sm = S.make_smpl_model(300)
        srv = SMPLServer(model=sm)
        rng = np.random.RandomState(7)
        o = srv(torch.ones(1), torch.zeros(1, 3), torch.from_numpy(rng.normal(0, 0.3, (1, 72)).astype(np.float32)),
                torch.from_numpy(rng.normal(0, 1, (1, 10)).astype(np.float32)))
        b = engine.Body(srv.verts_c[0], srv.weights[0], cano_cell=0.1001)
        b.set_pose(o["smpl_verts"][0], o["smpl_tfs"][0])
        _BODY["b"] = (b, srv)
    return _BODY["b"]


def points(N, verts, seed, far_frac=0.1, far=0.3):
    """Points within 0.09 of a vertex (inside the 0.1 outlier radius, where the grid search is exact either way), the first
    far_frac of them moved by far * a random direction: ~N(0, far) per axis, or (far < 0) exactly |far| away, beyond the
    grid's reach."""
    rng = np.random.RandomState(seed)
    v = verts.cpu().numpy()
    off = rng.normal(0, 0.03, (N, 3))
    n = np.linalg.norm(off, axis=1, keepdims=True)
    off = np.where(n > 0.09, off * (0.09 / np.maximum(n, 1e-30)), off)
    p = v[rng.randint(0, v.shape[0], N)] + off
    nf = int(N * far_frac)
    if nf:
        d = rng.normal(0, 1, (nf, 3))
        p[:nf] += d * far if far > 0 else -far * d / np.linalg.norm(d, axis=1, keepdims=True)
    return torch.from_numpy(p.astype(np.float32))


def pts(N, d, seed, lo=-1.0, hi=1.0):
    """N points uniform in [lo, hi)^d on the GPU."""
    g = torch.Generator().manual_seed(seed)
    return (lo + (hi - lo) * torch.rand(N, d, generator=g)).cuda()


# ---------------------------------------------------------------------------------------------
# sampler
# ---------------------------------------------------------------------------------------------

def rays(scene, R, seed=5):
    """R rays of person 0's box (repeated if the box has fewer hits), as float32 (dirs, cam) on the host."""
    from oracle import port
    inp = S.make_rays(scene, max(4 * R, 64), seed=seed, region="boxes")
    dirs, cam = port.get_camera_params(inp["uv"], inp["pose"], inp["intrinsics"])
    dirs = dirs.reshape(-1, 3)
    cam = cam.unsqueeze(1).repeat(1, dirs.shape[0] // cam.shape[0], 1).reshape(-1, 3)
    idx = S.make_hit_lists(scene, inp)[0]
    idx = idx.repeat((R + idx.numel() - 1) // idx.numel())[:R]
    return dirs[idx].contiguous(), cam[idx].contiguous()


def train_rng(cfg, R, seed=0, edges=False):
    """Draws of mp_sample_rays_train with distinct per-trip rows.  edges: t_rand / u_final hold exact 0 and 1 - 2^-24
    (stratified samples tie with near and with each other) and eik_idx hits S+X+1."""
    E, S_, X, T = cfg["N_samples_eval"], cfg["N_samples"], cfg["N_samples_extra"], cfg["max_total_iters"]
    g = torch.Generator().manual_seed(seed)
    t_rand, u_final = torch.rand(R, E, generator=g), torch.rand(R, S_, generator=g)
    if edges:
        top = 1.0 - 2.0 ** -24
        t_rand[:, 0::3] = 0.0
        t_rand[:, 1::5] = top
        u_final[:, 0::4] = 0.0
        u_final[:, 1::4] = top
    perm = torch.zeros(T, T * E, dtype=torch.int32)
    for t in range(T):
        perm[t, :(t + 1) * E] = torch.randperm((t + 1) * E, generator=g).to(torch.int32)
    eik = torch.randint(S_ + X + 2, (T, R), generator=g, dtype=torch.int32)
    if edges:
        eik[:, 0::2] = S_ + X + 1
    bg = torch.rand(T, R, 32, generator=g)
    return dict(t_rand=t_rand, u_final=u_final, extra_perm=perm, eik_idx=eik, t_rand_bg=bg)


# ---------------------------------------------------------------------------------------------
# compositor
# ---------------------------------------------------------------------------------------------

SMEM_CAP = 200 * 1024                   # launch_composite: dynamic shared memory of one block


def wpc_of(P, n):
    """Rays per block of launch_composite."""
    return max(1, min(8, SMEM_CAP // (12 * P * n)))


def make_inputs(seed, P, R, n, substitute=False, ties=True):
    """Per-person hit lists and sample rows.  Ray 0 is hit by every person, ray 1 by none, ray 2 by person 0 only, the
    rest by random subsets; with `substitute` the last person's list is the single ray 0 (multiply.py:262-263).  Rows
    are sorted z with a per-ray `far` shared by all persons as the last column; sdf spreads over [-1, 1] with exact
    zeros.  With `ties`: persons 0 and 1 share one z row on ray 0 (and on every third ray both hit), some rows carry
    zero-length intervals, and half of the rays end with a negative sdf on the last sample."""
    rng = np.random.RandomState(seed)
    H = rng.random_sample((P, R)) < 0.6
    H[:, 0] = True
    if R > 1:
        H[:, 1] = False
    if R > 2:
        H[:, 2] = False
        H[0, 2] = True
    if substitute and P > 1:
        H[P - 1] = False
        H[P - 1, 0] = True
    far = rng.uniform(3.0, 4.0, R).astype(np.float32)
    neg_last = rng.random_sample(R) < 0.5
    persons = []
    for p in range(P):
        idx = np.flatnonzero(H[p]).astype(np.int64)
        Rp = idx.size
        near = rng.uniform(0.5, 1.5, Rp)
        u = np.sort(rng.random_sample((Rp, n - 1)), 1) if n > 1 else np.zeros((Rp, 0))
        z = np.concatenate([near[:, None], near[:, None] + u * (far[idx] - near)[:, None], far[idx][:, None]], 1)
        z = z.astype(np.float32)
        z[:, -1] = far[idx]
        zm = 0.5 * (z[:, :-1] + z[:, 1:])
        surf = rng.uniform(0.8, 3.5, (Rp, 1))
        k = rng.uniform(1.0, 20.0, (Rp, 1))
        sdf = np.clip((surf - zm) * k + rng.normal(0, 0.05, zm.shape), -1, 1)
        noisy = rng.random_sample(Rp) < 0.3
        sdf[noisy] = rng.uniform(-1, 1, (int(noisy.sum()), n))
        sdf[rng.random_sample(sdf.shape) < 0.05] = 0.0
        sdf = sdf.astype(np.float32)
        if ties:
            if n > 2:        # zero-length intervals: z[i + 1] = z[i] on some rows
                rows = rng.random_sample(Rp) < 0.3
                cols = rng.randint(1, n - 1, int(rows.sum()))
                z[np.flatnonzero(rows), cols + 1] = z[np.flatnonzero(rows), cols]
            last_neg = neg_last[idx]
            sdf[last_neg, -1] = -np.abs(sdf[last_neg, -1]) - np.float32(0.25)
        persons.append(dict(idx=idx, z=np.ascontiguousarray(z), sdf=np.ascontiguousarray(sdf),
                            rgb=rng.random_sample((Rp, n, 3)).astype(np.float32),
                            nrm=rng.uniform(-1, 1, (Rp, n, 3)).astype(np.float32)))
    if ties and P > 1:      # persons 0 and 1: identical z rows (and a negative-sdf stretch) on shared rays
        a, b = persons[0], persons[1]
        shared = np.intersect1d(a["idx"], b["idx"])
        shared = shared[(shared % 3) == 0]
        ra, rb = np.searchsorted(a["idx"], shared), np.searchsorted(b["idx"], shared)
        b["z"][rb] = a["z"][ra]
        b["sdf"][rb, : max(1, n // 2)] = -0.05
        a["sdf"][ra, : max(1, n // 2)] = -0.02
    return persons


def person_samples(persons):
    """(mp_person_samples_t array, the device tensors it points to); a person without rays gets one-element
    placeholders, so that every pointer is valid."""
    keep = []
    for d in persons:
        if d["idx"].size:
            keep.append([torch.from_numpy(np.ascontiguousarray(d[k])).cuda() for k in ("idx", "z", "sdf", "rgb", "nrm")])
        else:
            keep.append([torch.zeros(1, dtype=torch.int64, device="cuda")] + [torch.zeros(1, device="cuda")] * 4)
    return engine.person_samples([t + [int(d["idx"].size)] for t, d in zip(keep, persons)]), keep


# ---------------------------------------------------------------------------------------------
# the fused render with canonical meshes (training surface flags)
# ---------------------------------------------------------------------------------------------

def fused_setup(R=256, empty_person1=False):
    """The geometric two-person scene's Renderer, R rays, their hit lists (person 1's empty on request), both canonical
    meshes, per-person training draws and bg jitter."""
    from multiply_b200.model.ray_sampler import ErrorBoundSampler
    engine.set_engine("tc")
    sc = S.make_scene(P=2, S=16, seed=42)
    r = engine.Renderer(sc)
    inp = S.make_rays(sc, R, seed=77, region="boxes")
    hits = S.make_hit_lists(sc, inp)
    if empty_person1:
        hits[1] = torch.zeros(0, dtype=torch.int64)
    meshes = [engine.CanonicalMesh(*S.make_body_mesh(100 + p)) for p in range(2)]
    smp = ErrorBoundSampler(3.0, inverse_sphere_bg=True, **{k: sc["cfg"][k] for k in (
        "near", "N_samples", "N_samples_eval", "N_samples_extra", "eps", "beta_iters", "max_total_iters", "add_tiny")})
    torch.manual_seed(5)
    rngs = [smp.draw_training_rng(max(h.numel(), 1)) for h in hits]
    rngs = [{k: v for k, v in rg.items() if k != "states"} for rg in rngs]
    return sc, r, inp, hits, meshes, rngs, torch.rand(R, 32)


def render_train(r, inp, hits, rngs, t_rand_bg, meshes, persons=None, thr=0.05):
    tr = dict(rng=rngs, t_rand_bg=t_rand_bg)
    if meshes is not None:
        tr.update(meshes=meshes, threshold=thr)
    out = r.render(inp, hits, debug=True, persons=persons, train=tr)
    torch.cuda.synchronize()
    return out


def flags_from_taps(sc, r, inp, hits, meshes, out, plist, thr=0.05, xc_out=None):
    """The flags recomputed with mp_mesh_surface_flags from the main pass's canonical points (z taps -> samples ->
    mp_deform_inverse), merged on the host as multiply.py:549-560.  xc_out (a list) receives each person's (rows,
    canonical points)."""
    from multiply_b200.model import rend_util
    dirs, cam = rend_util.get_camera_params(inp["uv"].cuda(), inp["pose"].cuda(), inp["intrinsics"].cuda())
    dirs = dirs[0]
    R = dirs.shape[0]
    cam = cam.expand(R, 3)
    n = r.n
    off = torch.ones(R, len(plist), dtype=torch.bool, device="cuda")
    inn = torch.zeros(R, len(plist), dtype=torch.bool, device="cuda")
    for k, p in enumerate(plist):
        h = hits[p] if hits[p].numel() else torch.zeros(1, dtype=torch.int64)
        h = h.cuda()
        z = out[f"z_vals_{k}"][:, :n]
        x = (cam[h][:, None] + z[..., None] * dirs[h][:, None]).reshape(-1, 3)
        xc, _ = r.bodies[p].deform_inverse(x, exact_far=True)
        o, i = meshes[k].surface_flags(xc, n, thr)
        if xc_out is not None:
            xc_out.append((h, xc))
        off[h, k] = o
        inn[h, k] = i
    return off.all(1), inn.any(1)


# ---------------------------------------------------------------------------------------------
# mesh-extraction grids
# ---------------------------------------------------------------------------------------------
#
# Analytic shapes on the (R+1)^3 lattice of the unit cube (x-major, point i at i / R), stored as MESH_SCALE x their
# signed distance so that a level l moves every surface outward by l / MESH_SCALE: levels up to 0.125 keep each shape
# and its holes well inside the cube.  "surfaces" gives, for that offset, each closed surface's signed enclosed volume
# (negative for a surface that bounds a cavity) and Euler characteristic, in increasing order of volume; "min_R" is the
# smallest R at which the shape's thinnest part spans enough cells for its topology and volume to hold.

MESH_SCALE = 4.0


def _unit_lattice(R):
    u = np.arange(R + 1, dtype=np.float64) / R
    return np.meshgrid(u, u, u, indexing="ij")


def _ball(X, Y, Z, c, r):
    return np.sqrt((X - c[0]) ** 2 + (Y - c[1]) ** 2 + (Z - c[2]) ** 2) - r


def _ring(X, Y, Z, c, a, b):
    """Solid torus about the z axis through c: major radius a, minor radius b."""
    return np.sqrt((np.sqrt((X - c[0]) ** 2 + (Y - c[1]) ** 2) - a) ** 2 + (Z - c[2]) ** 2) - b


def _ball_volume(r):
    return 4.0 / 3.0 * np.pi * r ** 3


_RING_VOLUME = {}


def _two_rings_volume(a, b, d):
    """Volume of the union of two coplanar solid tori (a, b) whose centres lie 2d apart: twice a torus less their
    overlap, integrated over the plane as 2 min(h1, h2), h the half-height of each solid torus (scipy dblquad)."""
    key = (a, b, d)
    if key not in _RING_VOLUME:
        from scipy import integrate

        def h(x, y, cx):
            r = np.hypot(x - cx, y) - a
            return np.sqrt(max(b * b - r * r, 0.0))

        ov, _ = integrate.dblquad(lambda y, x: 2.0 * min(h(x, y, -d), h(x, y, d)), 0.0, a + b - d, 0.0, a + b,
                                  epsabs=1e-10, epsrel=1e-10)
        _RING_VOLUME[key] = 2.0 * (2.0 * np.pi ** 2 * a * b * b) - 4.0 * ov
    return _RING_VOLUME[key]


_ELL_C, _ELL_A = (0.45, 0.53, 0.52), (0.32, 0.22, 0.16)
_DT_C, _DT_A, _DT_B, _DT_D = (0.5, 0.503, 0.497), 0.15, 0.07, 0.17
_TS = ((0.25, 0.5, 0.49), 0.13), ((0.69, 0.52, 0.51), 0.19)
_SH_C, _SH_R1, _SH_R2 = (0.51, 0.5, 0.49), 0.18, 0.34

MESH_SHAPES = {
    "sphere": dict(
        sdf=lambda X, Y, Z: _ball(X, Y, Z, (0.48, 0.51, 0.505), 0.3),
        surfaces=lambda o: [(_ball_volume(0.3 + o), 2)], min_R=37),
    "ellipsoid": dict(      # min(axes) x (ellipsoidal radius - 1): the level scales the ellipsoid by 1 + o / 0.16
        sdf=lambda X, Y, Z: _ELL_A[2] * (np.sqrt(((X - _ELL_C[0]) / _ELL_A[0]) ** 2 + ((Y - _ELL_C[1]) / _ELL_A[1]) ** 2
                                                 + ((Z - _ELL_C[2]) / _ELL_A[2]) ** 2) - 1.0),
        surfaces=lambda o: [(_ball_volume(1.0) * np.prod(_ELL_A) * (1.0 + o / _ELL_A[2]) ** 3, 2)], min_R=37),
    "torus": dict(
        sdf=lambda X, Y, Z: _ring(X, Y, Z, (0.5, 0.49, 0.51), 0.28, 0.1),
        surfaces=lambda o: [(2.0 * np.pi ** 2 * 0.28 * (0.1 + o) ** 2, 0)], min_R=64),
    "double_torus": dict(   # two tori side by side whose tubes merge between them: genus 2
        sdf=lambda X, Y, Z: np.minimum(_ring(X, Y, Z, (_DT_C[0] - _DT_D, _DT_C[1], _DT_C[2]), _DT_A, _DT_B),
                                       _ring(X, Y, Z, (_DT_C[0] + _DT_D, _DT_C[1], _DT_C[2]), _DT_A, _DT_B)),
        surfaces=lambda o: [(_two_rings_volume(_DT_A, _DT_B + o, _DT_D), -2)], min_R=64),
    "two_spheres": dict(
        sdf=lambda X, Y, Z: np.minimum(_ball(X, Y, Z, *_TS[0]), _ball(X, Y, Z, *_TS[1])),
        surfaces=lambda o: [(_ball_volume(_TS[0][1] + o), 2), (_ball_volume(_TS[1][1] + o), 2)], min_R=37),
    "shell": dict(          # below between r1 and r2: the inner surface faces the centre and encloses -V(r1)
        sdf=lambda X, Y, Z: np.maximum(_SH_R1 - np.sqrt((X - _SH_C[0]) ** 2 + (Y - _SH_C[1]) ** 2 + (Z - _SH_C[2]) ** 2),
                                       np.sqrt((X - _SH_C[0]) ** 2 + (Y - _SH_C[1]) ** 2 + (Z - _SH_C[2]) ** 2) - _SH_R2),
        surfaces=lambda o: [(-_ball_volume(_SH_R1 - o), 2), (_ball_volume(_SH_R2 + o), 2)], min_R=37),
}


def lattice_boundary(R):
    b = np.zeros((R + 1,) * 3, bool)
    b[0], b[-1], b[:, 0], b[:, -1], b[:, :, 0], b[:, :, -1] = True, True, True, True, True, True
    return b


def mesh_grid(name, R, level, variant="closed"):
    """An fp32 grid [R+1]^3 at ``level``: an entry of MESH_SHAPES, "random" (standard normal noise) or "quantised"
    (level + multiples of 0.5: values on the level, t = 0 / 1 vertices, asymptotic-decider ties).  "closed": no
    boundary point below the level (those of a coarse shape or of noise are lifted to level + 1); "open": a shape's
    closed grid with a patch of the x = 0 face set below the level, or the noise as drawn."""
    if name in MESH_SHAPES:
        g = (MESH_SCALE * MESH_SHAPES[name]["sdf"](*_unit_lattice(R))).astype(np.float32)
    else:
        rng = np.random.default_rng(1000 * R + {"random": 1, "quantised": 2}[name])
        g = rng.standard_normal((R + 1,) * 3).astype(np.float32)
        if name == "quantised":
            g = np.float32(level) + np.round(g * 2).astype(np.float32) / np.float32(2)
        if variant == "open":
            return g
    lift = lattice_boundary(R) & (g.astype(np.float64) < level)
    g[lift] = np.float32(level + 1.0)
    if variant == "open":
        h = R // 2 + 1
        g[0, :h, :h] = np.float32(level - 1.0)
    return g
