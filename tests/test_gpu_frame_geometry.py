"""GPU: the kernels that build every frame's geometry against float64 restatements, at the shapes and values where they
break.

- SMPL server (csrc/smpl.cu: mp_smpl_create / _forward / _canonical): lbs with Rodrigues' +1e-8 bias, the kinematic
  chain, the pose blend, skinning, SMPLServer's scale / translation / canonical inverse (smpl.py:35-95).  Models with
  V = 1, 127, 128, 129 (the 128-thread skin blocks' tail), 6890, and one with a dense J_regressor (every vertex in the
  32-lane joint regression); poses at theta = 0, tiny angles, pi and pi +- 1e-3, up to 4 pi, random and canonical.
- Camera rays and sphere bounds (csrc/rays.cu: mp_camera_rays, mp_sphere_intersections) around the 256-thread block
  tails, with exact tangency, cameras outside the sphere and the OR-ed status flag.
- Ray culling (mp_ray_box_hits, mp_ray_aabb_hits, mp_hit_list_finalize): ids in order and exactly those of a float64
  slab test with the same 1e-12 clamp, around the 32-lane and 1024-ray tile edges.
- Background (csrc/background.cu: mp_background and the bg taps of mp_render_rays) against float64 depth2pts_outside,
  float64 background networks and float64 bg_volume_rendering, on both engines; the ray through the sphere's centre
  gets the limit p_sphere / |p_sphere| (the reference's NaN).

Gates are per element, err <= C * 2^-24 * M, M the float64 sum of |terms| behind the element; C is 4x the worst
measured on one H100 80GB HBM3 at a 400 W power limit (quoted in each test's docstring)."""
import ctypes as C
import os
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from multiply_b200 import scene as S          # noqa: E402  (CPU-only module)
from oracle import render_grad as RG          # noqa: E402

from _abi import SENTINEL_INT, padded, take     # noqa: E402
from _setups import small_model                 # noqa: E402

EPS = 2.0 ** -24
MEASURED = {}

# gates in units of 2^-24 * M: 4x the worst measured on one H100 80GB HBM3 at a 400 W power limit (each test's docstring)
C_SMPL = 8.2
C_RAYS = 2.1
C_PORT = 16.0
C_SPHERE = 5.2
C_BG = {"simt": 34.0, "tc": 28.0}
C_BG_TAP = 7.3


def _note(key, c):
    MEASURED[key] = max(MEASURED.get(key, 0.0), float(c))


def _report(prefix):
    for k in sorted(MEASURED):
        if k.startswith(prefix):
            print("MEASURED %s C=%.3g" % (k, MEASURED[k]))


@pytest.fixture(scope="module", autouse=True)
def _print_measured():
    yield
    _report("")


def _ratio(err, M):
    """err / (2^-24 M) elementwise, where M = 0 demands err = 0."""
    err, M = np.asarray(err, np.float64), np.asarray(M, np.float64)
    return np.where(M > 0, err / (EPS * np.where(M > 0, M, 1.0)), np.where(err == 0, 0.0, np.inf))


# ---------------------------------------------------------------------------------------------
# SMPL: float64 restatement of lbs.py:136-378 and smpl.py:35-95, with the magnitudes M of every output
# ---------------------------------------------------------------------------------------------

def rodrigues_ref(theta, dtype=np.float64):
    """batch_rodrigues (lbs.py:276-307): angle = |theta + 1e-8|, axis = theta / angle.  Returns (R [J,3,3], M): M bounds
    the terms of I + sin K + (1 - cos) K K (1 - cos cancels: its terms are 1 and cos) plus the sensitivity to the
    rounding of the angle."""
    th = np.asarray(theta, dtype).reshape(-1, 3)
    a = th + dtype(1e-8)
    ang = np.sqrt((a * a).sum(1, dtype=dtype))[:, None, None].astype(dtype)
    d = th / ang[:, :, 0]
    c, s = np.cos(ang).astype(dtype), np.sin(ang).astype(dtype)
    K = np.zeros((th.shape[0], 3, 3), dtype)
    K[:, 0, 1], K[:, 0, 2] = -d[:, 2], d[:, 1]
    K[:, 1, 0], K[:, 1, 2] = d[:, 2], -d[:, 0]
    K[:, 2, 0], K[:, 2, 1] = -d[:, 1], d[:, 0]
    KK = K @ K
    I = np.eye(3, dtype=dtype)[None]
    R = I + s * K + (dtype(1) - c) * KK
    aK, aKK = np.abs(K), np.abs(K) @ np.abs(K)
    M = I + np.abs(s) * aK + (1 + np.abs(c)) * aKK + ang * (np.abs(c) * aK + np.abs(s) * aKK)
    return R, M


def lbs_ref(model, betas, theta, scale=1.0, transl=(0.0, 0.0, 0.0), absolute=True, cinv=None, dtype=np.float64):
    """SMPLServer.forward (smpl.py:50-95) over lbs (lbs.py:136-229) in `dtype`.  model: numpy arrays (v_template [V,3],
    shapedirs [V,3,10], posedirs [207,3V], J_regressor [24,V], lbs_weights [V,24], parents [24]); cinv = (tfs_c_inv,
    its M) when not absolute.  Returns dict(verts [V,3], tfs [24,4,4], A [24,4,4] scaled/translated, and their M)."""
    f = lambda a: np.asarray(a, np.float32).astype(dtype)
    vt, sd, pd, Jr, W = (f(model[k]) for k in ("v_template", "shapedirs", "posedirs", "J_regressor", "lbs_weights"))
    par = [int(p) for p in model["parents"]]
    b, th = f(betas).reshape(10), f(theta).reshape(24, 3)
    s, t = dtype(np.float32(scale)), f(transl).reshape(3)
    V = vt.shape[0]
    v_shaped = vt + sd @ b
    M_vs = np.abs(vt) + np.abs(sd) @ np.abs(b)
    J = Jr @ v_shaped
    M_J = np.abs(Jr) @ M_vs
    R, M_R = rodrigues_ref(th, dtype)
    I = np.eye(3, dtype=dtype)
    pf = (R[1:] - I).reshape(207)
    M_pf = M_R[1:].reshape(207)
    pb = (pf @ pd).reshape(V, 3)
    M_pb = (M_pf @ np.abs(pd)).reshape(V, 3)
    x, M_x = v_shaped + pb, M_vs + M_pb
    G, M_G = np.zeros((24, 4, 4), dtype), np.zeros((24, 4, 4), dtype)
    for i in range(24):
        T, MT = np.zeros((4, 4), dtype), np.zeros((4, 4), dtype)
        T[:3, :3], MT[:3, :3] = R[i], M_R[i]
        T[:3, 3] = J[i] if i == 0 else J[i] - J[par[i]]
        MT[:3, 3] = M_J[i] if i == 0 else M_J[i] + M_J[par[i]]
        T[3, 3] = MT[3, 3] = 1
        if i == 0:
            G[0], M_G[0] = T, MT
        else:
            G[i], M_G[i] = G[par[i]] @ T, M_G[par[i]] @ MT
    A, M_A = G.copy(), M_G.copy()
    A[:, :, 3] -= np.einsum("jrc,jc->jr", G[:, :, :3], J)
    M_A[:, :, 3] += np.einsum("jrc,jc->jr", M_G[:, :, :3], M_J)
    A[:, :3, :] *= s
    M_A[:, :3, :] *= abs(s)
    A[:, :3, 3] += t * s
    M_A[:, :3, 3] += np.abs(t * s)
    if absolute:
        tfs, M_tfs = A, M_A
    else:
        ci, M_ci = cinv
        tfs = A @ ci
        M_tfs = M_A @ np.abs(ci) + np.abs(A) @ M_ci
    Tv = W @ A.reshape(24, 16)
    M_Tv = np.abs(W) @ M_A.reshape(24, 16)
    verts = np.stack([(Tv[:, 4 * r:4 * r + 3] * x).sum(1) + Tv[:, 4 * r + 3] for r in range(3)], 1)
    M_v = np.stack([(M_Tv[:, 4 * r:4 * r + 3] * M_x).sum(1) + M_Tv[:, 4 * r + 3] for r in range(3)], 1)
    return dict(verts=verts, tfs=tfs, A=A, M_verts=M_v, M_tfs=M_tfs, M_A=M_A)


CANONICAL_THETA = np.zeros(72, np.float32)
CANONICAL_THETA[5], CANONICAL_THETA[8] = np.pi / 6, -np.pi / 6       # smpl.py:38-39, hips +-pi/6 about z


def canonical_ref(model, betas_c):
    """smpl.py:35-47: the canonical pose's absolute transforms (scale 1, no translation), their inverse and its M
    (first order: |A^-1| M_A |A^-1|, plus the inverse's own rounding)."""
    o = lbs_ref(model, betas_c, CANONICAL_THETA)
    ci = np.linalg.inv(o["A"])
    a = np.abs(ci)
    return o, (ci, a @ o["M_A"] @ a + a)


def model_np(m):
    return {k: (v.numpy() if torch.is_tensor(v) else np.asarray(v)) for k, v in m.items()}


def get_model(name):
    if name == "smpl6890":
        return model_np(S.make_smpl_model(300))
    if name == "dense6890":
        m = model_np(S.make_smpl_model(300))
        return dict(m, J_regressor=small_model(6890, seed=302, dense=True)["J_regressor"])
    return small_model(int(name[1:]))


class SmplHandle:
    """mp_smpl_create / _forward / _canonical through the C ABI with sentinel-padded outputs."""

    def __init__(self, model, betas_c=None):
        from multiply_b200 import _lib as L
        self.L = L
        self.V = model["v_template"].shape[0]
        self.d = {k: torch.from_numpy(np.ascontiguousarray(model[k], np.float32)).cuda()
                  for k in ("v_template", "shapedirs", "posedirs", "J_regressor", "lbs_weights")}
        self.bc = None if betas_c is None else torch.from_numpy(np.asarray(betas_c, np.float32)).cuda()
        pa = (C.c_int * 24)(*[max(int(p), 0) for p in model["parents"]])
        self.storage = L.workspace(L.call("mp_smpl_bytes", self.V), "cuda")
        self.h = L.Handle("mp_smpl_free")
        d = self.d
        L.call("mp_smpl_create", d["v_template"], d["shapedirs"], d["posedirs"], d["J_regressor"], pa, d["lbs_weights"],
               self.V, self.bc, self.storage, self.storage.numel(), C.byref(self.h))

    def canonical(self):
        vc, ti = padded((self.V, 3)), padded((24, 4, 4))
        self.L.call("mp_smpl_canonical", self.h, vc, ti)
        torch.cuda.synchronize()
        return take(vc, (self.V, 3), "verts_c").numpy(), take(ti, (24, 4, 4), "tfs_c_inv").numpy()

    def forward(self, scale, transl, theta, betas, absolute):
        args = [torch.from_numpy(np.asarray(a, np.float32).reshape(-1)).cuda() for a in ((scale,), transl, theta, betas)]
        v, t = padded((self.V, 3)), padded((24, 4, 4))
        self.L.call("mp_smpl_forward", self.h, *args, int(absolute), v, t)
        torch.cuda.synchronize()
        return take(v, (self.V, 3), "smpl_verts").numpy(), take(t, (24, 4, 4), "smpl_tfs").numpy()


_U = np.array([0.36, -0.48, 0.8])          # a unit axis with no zero component


def smpl_poses():
    """name -> theta [72] float32: zero, one joint at tiny angles, pi and pi +- 1e-3 on the global orient (0) and a leaf
    joint (23), angles up to 4 pi, random, canonical."""
    rng = np.random.RandomState(17)
    P = {"zero": np.zeros((24, 3))}
    for m in (1e-7, 1e-4, 1e-2):
        th = np.zeros((24, 3))
        th[7] = m * _U
        P["j7_%g" % m] = th
    for j in (0, 23):
        for name, m in (("pi", np.pi), ("pi-", np.pi - 1e-3), ("pi+", np.pi + 1e-3)):
            th = rng.normal(0, 0.2, (24, 3))
            th[j] = m * _U
            P["j%d_%s" % (j, name)] = th
    ax = rng.normal(size=(24, 3))
    ax /= np.linalg.norm(ax, axis=1, keepdims=True)
    th = ax * rng.uniform(np.pi, 4 * np.pi, (24, 1))
    th[0] = 4 * np.pi * _U
    th[23] = 4 * np.pi * ax[23]
    P["large"] = th
    P["random_a"] = rng.normal(0, 0.3, (24, 3))
    P["random_b"] = rng.normal(0, 0.5, (24, 3))
    P["canonical"] = CANONICAL_THETA.reshape(24, 3)
    return {k: v.reshape(72).astype(np.float32) for k, v in P.items()}


def _betas(v, seed):
    sg = np.where(np.random.RandomState(seed).rand(10) < 0.5, -1.0, 1.0)
    return (v * sg).astype(np.float32) if seed else np.full(10, v, np.float32)


# (betas, scale, transl, absolute)
PLACEMENTS = [(_betas(0.0, 0), 1.0, (0.0, 0.0, 0.0), 1), (_betas(3.0, 0), 0.25, (0.3, -0.2, 0.1), 0),
              (_betas(-3.0, 0), 2.0, (-1.5, 0.7, 2.0), 1), (_betas(5.0, 3), 1.0, (0.05, 0.1, -0.02), 0),
              (_betas(-5.0, 0), 2.0, (0.4, -1.1, 0.6), 0), (_betas(3.0, 5), 0.25, (0.0, 0.0, 0.0), 1)]
MODELS = ["V1", "V127", "V128", "V129", "smpl6890", "dense6890"]


def _smpl_case(hd, model, cano, theta, placement):
    betas, scale, transl, absolute = placement
    want = lbs_ref(model, betas, theta, scale, transl, bool(absolute), cinv=cano)
    v, t = hd.forward(scale, transl, theta, betas, absolute)
    cv = _ratio(np.abs(v - want["verts"]), want["M_verts"]).max()
    ct = _ratio(np.abs(t - want["tfs"]), want["M_tfs"]).max()
    return max(cv, ct), (cv, ct)


@pytest.mark.parametrize("name", MODELS)
def test_smpl_server_vs_fp64(name):
    """verts_c, tfs_c_inv and every pose x placement of the docstring, with betas_canonical NULL and given, against the
    float64 restatement: per element err <= C_SMPL 2^-24 M (M: the chain's |products| for the transforms,
    |T| (|v_shaped| + |pose blend|) + |t| for the vertices, |A^-1| M |A^-1| for the canonical inverse); nothing
    written past V or the 24 transforms.  Measured worst C: 2.04 (smpl6890), 2.01 (dense J_regressor), 1.8 (V = 1 ..
    129); 0.81 on verts_c / tfs_c_inv."""
    model = get_model(name)
    poses = smpl_poses()
    bc_given = _betas(1.5, 11)
    for bc in (None, bc_given):
        hd = SmplHandle(model, bc)
        o, cano = canonical_ref(model, np.zeros(10, np.float32) if bc is None else bc)
        vc, ti = hd.canonical()
        c = max(_ratio(np.abs(vc - o["verts"]), o["M_verts"]).max(), _ratio(np.abs(ti - cano[0]), cano[1]).max())
        _note("smpl_canonical/" + name, c)
        assert c < C_SMPL, (name, bc is not None, c)
        for pn, theta in poses.items():
            for k, pl in enumerate(PLACEMENTS):
                c, parts = _smpl_case(hd, model, cano, theta, pl)
                _note("smpl/%s/%s" % (name, pn), c)
                _note("smpl/" + name, c)
                assert c < C_SMPL, (name, pn, k, bc is not None, parts)


def test_smpl_handle_state_does_not_leak():
    """Pose A, then B (other betas, scale, translation, absolute flag), then A on one handle: the first and third
    outputs are bit-equal (pose_feature and A_abs are per-handle scratch, rewritten by every call)."""
    model = get_model("smpl6890")
    poses = smpl_poses()
    hd = SmplHandle(model)
    a = (0.5, (0.3, 0.1, -0.2), poses["random_a"], _betas(3.0, 7), 0)
    b = (2.0, (-1.0, 0.4, 0.9), poses["large"], _betas(-5.0, 8), 1)
    v1, t1 = hd.forward(*a)
    v2, t2 = hd.forward(*b)
    v3, t3 = hd.forward(*a)
    assert not np.array_equal(v1, v2)
    assert np.array_equal(v1.view(np.uint32), v3.view(np.uint32))
    assert np.array_equal(t1.view(np.uint32), t3.view(np.uint32))


# ---------------------------------------------------------------------------------------------
# camera rays and sphere bounds: float64 restatement of rend_util.py:45-87, :131-147
# ---------------------------------------------------------------------------------------------

def skew_camera():
    """A skewed, off-centre K and a rotated, translated camera-to-world pose (float32 [4,4] each)."""
    K = np.eye(4, dtype=np.float32)
    K[0, 0], K[0, 1], K[0, 2], K[1, 1], K[1, 2] = 612.3, 3.7, 301.9, 598.1, 244.6
    R, _ = rodrigues_ref(np.array([0.4, -0.9, 0.25]))
    pose = np.eye(4, dtype=np.float32)
    pose[:3, :3] = R[0]
    pose[:3, 3] = (0.3, -0.2, 2.4)
    return K, pose


def lift_ref(uv, pose, K, dtype=np.float64):
    """get_camera_params + lift (4x4 pose branch) in `dtype`: (dirs [R,3], cam_loc [3], M [R]).  M bounds the direction's
    rounding: the lift's |terms| through |pose|, over |world - cam_loc|."""
    uv, P, K = (np.asarray(a, np.float32).astype(dtype) for a in (uv, pose, K))
    fx, sk, cx, fy, cy = K[0, 0], K[0, 1], K[0, 2], K[1, 1], K[1, 2]
    x, y = uv[:, 0], uv[:, 1]
    xl = (x - cx + cy * sk / fy - sk * y / fy) / fx
    yl = (y - cy) / fy
    pts = np.stack([xl, yl, np.ones_like(xl), np.ones_like(xl)], 0)
    world = (P @ pts).T[:, :3]
    cam = P[:3, 3]
    d = world - cam
    n = np.maximum(np.sqrt((d * d).sum(1)), 1e-12)
    M_xl = (np.abs(x) + abs(cx) + abs(cy * sk / fy) + np.abs(sk * y / fy)) / abs(fx)
    M_yl = (np.abs(y) + abs(cy)) / abs(fy)
    aP = np.abs(P)
    M_d = (aP[:3, 0][None] * M_xl[:, None] + aP[:3, 1][None] * M_yl[:, None] + aP[:3, 2][None] + 2 * aP[:3, 3][None])
    return d / n[:, None], cam, M_d.max(1) / n


def sphere_ref(cam, dirs, r, dtype=np.float64):
    """get_sphere_intersections in `dtype`: (near_far [R,2] clamped at 0, under [R], M [R])."""
    o, d = np.asarray(cam, np.float32).astype(dtype), np.asarray(dirs, np.float32).astype(dtype)
    dot = (d * o).sum(1)
    oo = (o * o).sum(1)
    under = dot * dot - (oo - dtype(r) * dtype(r))
    s = np.sqrt(np.maximum(under, 0))
    nf = np.maximum(np.stack([-s - dot, s - dot], 1), 0)
    M_dot = (np.abs(d) * np.abs(o)).sum(1)
    M_under = dot * dot + 2 * np.abs(dot) * M_dot + 2 * oo + r * r
    M = s + M_dot + M_under / (2 * np.maximum(s, 1e-30))
    return nf, under, M


def call_camera_rays(uv, pose, K):
    from multiply_b200 import _lib as L
    R = uv.shape[0]
    t = [torch.from_numpy(np.ascontiguousarray(a, np.float32).reshape(-1)).cuda() for a in (uv, pose, K)]
    dirs, cam = padded((R, 3)), padded((R, 3))
    L.call("mp_camera_rays", *t, R, dirs, cam)
    torch.cuda.synchronize()
    return take(dirs, (R, 3), "ray_dirs").numpy(), take(cam, (R, 3), "cam_loc").numpy()


def call_sphere(cam, dirs, r, flag0=0):
    from multiply_b200 import _lib as L
    R = cam.shape[0]
    c, d = (torch.from_numpy(np.ascontiguousarray(a, np.float32).reshape(-1)).cuda() for a in (cam, dirs))
    nf = padded((R, 2))
    flag = torch.full((1,), flag0, dtype=torch.int32, device="cuda")
    L.call("mp_sphere_intersections", c, d, R, float(r), nf, flag)
    torch.cuda.synchronize()
    return take(nf, (R, 2), "near_far").numpy(), int(flag.item())


def _ordered(a):
    i = np.asarray(a, np.float32).view(np.int32).astype(np.int64)
    return np.where(i < 0, -(2 ** 31) - i, i)


def ulp_diff(a, b):
    return np.abs(_ordered(a) - _ordered(b))


def _uv(R, seed):
    rng = np.random.RandomState(seed)
    uv = np.stack([rng.uniform(0, 640, R), rng.uniform(0, 480, R)], 1)
    uv[:min(R, 4)] = np.array([[0, 0], [639.5, 479.5], [301.9, 244.6], [301, 244]])[:min(R, 4)]
    return uv.astype(np.float32)


@pytest.mark.parametrize("R", [1, 255, 256, 257, 4097])
def test_camera_rays(R):
    """mp_camera_rays on a skewed, off-centre K and a rotated pose against the float64 lift: per component
    err <= C_RAYS 2^-24 M; cam_loc is the pose's translation exactly; and against oracle/port.get_camera_params, the
    float32 statement of the reference, within C_PORT 2^-24 on the unit vectors.  Measured worst C 0.515 against
    float64; against the port 4 x 2^-24, which is up to 15 ulp on small components: the two agree neither exactly nor
    to 1 ulp, because world - cam_loc cancels and torch's CPU bmm rounds the four-term sums of `world` in its own
    order."""
    from oracle import port
    K, pose = skew_camera()
    uv = _uv(R, R)
    dirs, cam = call_camera_rays(uv, pose, K)
    want, cam64, M = lift_ref(uv, pose, K)
    c = _ratio(np.abs(dirs - want), M[:, None]).max()
    _note("camera_rays", c)
    assert c < C_RAYS, c
    assert np.array_equal(cam, np.broadcast_to(pose[:3, 3], (R, 3)))
    pd, _ = port.get_camera_params(torch.from_numpy(uv)[None], torch.from_numpy(pose)[None], torch.from_numpy(K)[None])
    pd = pd[0].numpy()
    _note("camera_rays_vs_port_ulp", ulp_diff(dirs, pd).max())
    c = float(np.abs(dirs - pd).max()) / EPS
    _note("camera_rays_vs_port", c)
    assert c < C_PORT, c


def test_sphere_bounds():
    """mp_sphere_intersections against float64: rays from a camera inside the r = 3 sphere (R around the 256-thread
    block), cameras outside it looking at it and away from it (near and far clamp to 0); per element
    err <= C_SPHERE 2^-24 M.  The flag: 0 after an all-hit batch, stays 1 when pre-set (the kernel ORs), and set by rays
    whose `under` is exactly 0 in fp32 (tangent: the reference's `under <= 0`) placed in the last block's tail.
    Measured worst C 1.3."""
    K, pose = skew_camera()
    worst = 0.0
    for R in (1, 255, 256, 257, 1029):
        dirs, cam = call_camera_rays(_uv(R, 100 + R), pose, K)
        nf, flag = call_sphere(cam, dirs, 3.0)
        want, under, M = sphere_ref(cam, dirs, 3.0)
        assert flag == 0 and (under > 0).all()
        worst = max(worst, _ratio(np.abs(nf - want), M[:, None]).max())
        _, flag = call_sphere(cam, dirs, 3.0, flag0=1)
        assert flag == 1
    # cameras outside the sphere: towards it (near > 0) and away from it (the line meets the sphere behind the camera)
    rng = np.random.RandomState(3)
    o = rng.normal(size=(300, 3))
    o = (o / np.linalg.norm(o, axis=1, keepdims=True) * rng.uniform(3.5, 6.0, (300, 1))).astype(np.float32)
    tgt = rng.uniform(-1.5, 1.5, (300, 3))
    d = tgt - o
    d[150:] = -d[150:]
    d = (d / np.linalg.norm(d, axis=1, keepdims=True)).astype(np.float32)
    nf, flag = call_sphere(o, d, 3.0)
    want, under, M = sphere_ref(o, d, 3.0)
    assert flag == 0 and (under > 0).all()
    assert (nf[:150] > 0).all() and (nf[150:] == 0).all() and (want[150:] == 0).all()
    worst = max(worst, _ratio(np.abs(nf - want), M[:, None]).max())
    _note("sphere", worst)
    assert worst < C_SPHERE, worst
    # exact tangency in fp32: |o| = 5, o . d = -4, r = 3 -> under = 16 - (25 - 9) = 0
    tang_o = np.float32([[0, 3, -4], [3, 0, -4], [0, -3, 4], [4, 3, 0]])
    tang_d = np.float32([[0, 0, 1], [0, 0, 1], [0, 0, -1], [-1, 0, 0]])
    dirs, cam = call_camera_rays(_uv(257, 9), pose, K)
    for k in range(4):
        c2, d2 = cam.copy(), dirs.copy()
        c2[-1], d2[-1] = tang_o[k], tang_d[k]
        _, under, _ = sphere_ref(c2, d2, 3.0)
        assert under[-1] == 0
        nf, flag = call_sphere(c2, d2, 3.0)
        assert flag == 1, k
        assert nf[-1, 0] == nf[-1, 1] == 4.0
    # a ray that misses sets it too
    c2, d2 = cam.copy(), dirs.copy()
    c2[-1], d2[-1] = (0, 3.5, -4), (0, 0, 1)
    assert call_sphere(c2, d2, 3.0)[1] == 1


# ---------------------------------------------------------------------------------------------
# culling: float64 slab test with the kernel's 1e-12 clamp (scene.ray_box_hits), optionally in a rotated box frame
# ---------------------------------------------------------------------------------------------

def slab_hits_ref(cam, dirs, c, h, rot=None):
    """Sorted ids of the rays that hit the box (centre c, half extents h, rows of rot = its axes), in float64 with the
    kernel's rounding order: o = cam - c ; o_a = rot_a . o ; |d_a| < 1e-12 -> 1e-12 ; t = (+-h - o_a) * (1 / d_a)."""
    o = np.asarray(cam, np.float32).astype(np.float64) - np.asarray(c, np.float64)
    d = np.asarray(dirs, np.float32).astype(np.float64)
    Rm = np.eye(3) if rot is None else np.asarray(rot, np.float64).reshape(3, 3)
    tmin = np.full(o.shape[0], -1e300)
    tmax = np.full(o.shape[0], 1e300)
    for a in range(3):
        oa = Rm[a, 0] * o[:, 0] + Rm[a, 1] * o[:, 1] + Rm[a, 2] * o[:, 2]
        da = Rm[a, 0] * d[:, 0] + Rm[a, 1] * d[:, 1] + Rm[a, 2] * d[:, 2]
        da = np.where(np.abs(da) < 1e-12, 1e-12, da)
        inv = 1.0 / da
        t1, t2 = (-h[a] - oa) * inv, (h[a] - oa) * inv
        tmin = np.maximum(tmin, np.minimum(t1, t2))
        tmax = np.minimum(tmax, np.maximum(t1, t2))
    return np.flatnonzero(tmax >= np.maximum(tmin, 0.0))


def call_box_hits(cam, dirs, c, h, rot=None):
    from multiply_b200 import _lib as L
    R = cam.shape[0]
    cc, dd = (torch.from_numpy(np.ascontiguousarray(a, np.float32).reshape(-1)).cuda() for a in (cam, dirs))
    rot_d = None if rot is None else torch.from_numpy(np.asarray(rot, np.float64).reshape(9)).cuda()
    idx = padded(R, torch.int64)
    cnt = torch.full((1,), -1, dtype=torch.int32, device="cuda")
    L.call("mp_ray_box_hits", cc, dd, R, L.vec3(C.c_double, c), L.vec3(C.c_double, h), rot_d, idx, cnt)
    torch.cuda.synchronize()
    n = int(cnt.item())
    assert 0 <= n <= R
    return take(idx, n, "hit ids").numpy(), idx, cnt


BOX_C, BOX_H = (0.25, -0.5, 0.75), (0.5, 0.25, 0.375)     # exactly representable: faces at c +- h are float32


def pattern_rays(mask, seed, c=BOX_C, h=BOX_H, rot=None):
    """Rays from origins 3-6 away from the box: those in `mask` aim at a point well inside it, the others point
    directly away from it."""
    rng = np.random.RandomState(seed)
    R = mask.size
    Rm = np.eye(3) if rot is None else np.asarray(rot).reshape(3, 3)
    o = rng.normal(size=(R, 3))
    o = o / np.linalg.norm(o, axis=1, keepdims=True) * rng.uniform(3, 6, (R, 1)) + np.asarray(c)
    tgt = np.asarray(c) + (rng.uniform(-0.5, 0.5, (R, 3)) * np.asarray(h)) @ Rm
    d = np.where(mask[:, None], tgt - o, o - np.asarray(c))
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    return o.astype(np.float32), d.astype(np.float32)


def _pattern(name, R):
    m = np.zeros(R, bool)
    if name == "all":
        m[:] = True
    elif name == "alternate":
        m[::2] = True
    elif name == "last_tile":
        m[(R - 1) // 1024 * 1024:] = True
    elif name == "last_ray":
        m[-1] = True
    return m


CULL_R = [1, 31, 32, 33, 1023, 1024, 1025, 2048, 5000]


@pytest.mark.parametrize("R", CULL_R)
def test_ray_box_hits_patterns(R):
    """Hit patterns none / all / alternate / only the last partial tile / only ray R-1, axis-aligned and in an oriented
    box (rot_dev): the ids equal the float64 slab test's, in ascending order, nothing written past the count; an empty
    list is finalised by mp_hit_list_finalize to [0] with count 1, a non-empty one is left alone."""
    from multiply_b200 import _lib as L
    rot, _ = rodrigues_ref(np.array([0.3, 0.7, -0.5]))
    for rname, rm in (("aligned", None), ("oriented", rot[0])):
        for pname in ("none", "all", "alternate", "last_tile", "last_ray"):
            mask = _pattern(pname, R)
            cam, dirs = pattern_rays(mask, R + len(pname), rot=rm)
            want = slab_hits_ref(cam, dirs, BOX_C, BOX_H, rm)
            assert np.array_equal(want, np.flatnonzero(mask)), (rname, pname)
            got, idx, cnt = call_box_hits(cam, dirs, BOX_C, BOX_H, rm)
            assert np.array_equal(got, want), (rname, pname, got[:8], want[:8])
            L.call("mp_hit_list_finalize", idx, cnt)
            torch.cuda.synchronize()
            n = int(cnt.item())
            if want.size == 0:
                assert n == 1 and int(idx[0].item()) == 0 and bool((idx[1:] == SENTINEL_INT).all())
            else:
                assert n == want.size and np.array_equal(idx[:n].cpu().numpy(), want)


def test_ray_box_hits_axis_parallel_and_special_cameras():
    """Axis-parallel rays take the 1e-12 clamp: origins inside, outside and exactly on each slab face (on the +h face
    the slab's t range ends at 0, on the -h face it starts there); a camera inside the box hits with every ray; a box
    behind the camera is hit by none."""
    c, h = BOX_C, BOX_H
    cam, dirs = [], []
    for a in range(3):                        # ray along axis a, from outside the box on that axis
        for sgn in (1.0, -1.0):
            d = np.zeros(3)
            d[a] = sgn
            for b in range(3):
                if b == a:
                    continue
                for off in (0.0, 0.5 * h[b], -0.5 * h[b], h[b], -h[b], 1.5 * h[b], -1.5 * h[b], 1e-7, -h[b] - 1e-7):
                    o = np.array(c, np.float64)
                    o[a] -= sgn * 2.0
                    o[b] += off
                    cam.append(o)
                    dirs.append(d.copy())
    cam, dirs = np.float32(cam), np.float32(dirs)
    # the faces are exactly representable: the origin lies on them bit for bit
    assert ((cam.astype(np.float64) - np.asarray(c)) == np.asarray(h)).any(1).sum() > 0
    want = slab_hits_ref(cam, dirs, c, h)
    assert 0 < want.size < cam.shape[0]
    got, _, _ = call_box_hits(cam, dirs, c, h)
    assert np.array_equal(got, want)
    rng = np.random.RandomState(4)
    R = 1500
    d = rng.normal(size=(R, 3))
    d = (d / np.linalg.norm(d, axis=1, keepdims=True)).astype(np.float32)
    inside = np.broadcast_to(np.float32(c) + np.float32([0.1, -0.05, 0.2]), (R, 3)).copy()
    got, _, _ = call_box_hits(inside, d, c, h)
    assert np.array_equal(got, np.arange(R)) and np.array_equal(slab_hits_ref(inside, d, c, h), np.arange(R))
    cam0 = np.broadcast_to(np.float32([0, 0, 2.5]), (R, 3)).copy()
    fwd = np.float32([0, 0, -1]) + 0.2 * rng.uniform(-1, 1, (R, 3)).astype(np.float32)
    fwd = (fwd / np.linalg.norm(fwd, axis=1, keepdims=True)).astype(np.float32)
    behind = (0.0, 0.0, 4.0)
    got, _, _ = call_box_hits(cam0, fwd, behind, (0.5, 0.5, 0.5))
    assert got.size == 0 and slab_hits_ref(cam0, fwd, behind, (0.5, 0.5, 0.5)).size == 0


@pytest.mark.parametrize("V", [1, 31, 1025, 6890])
def test_ray_aabb_hits(V):
    """mp_ray_aabb_hits: box_ws holds the float64 centre ((lo + hi) / 2) and inflated half extents ((hi - lo) / 2 * 1.2)
    of the float32 bounds bit for bit; the ids equal the slab test's on that box, and the list comes out finalised
    (empty -> [0], count 1)."""
    from multiply_b200 import _lib as L
    rng = np.random.RandomState(V)
    verts = (rng.normal(size=(V, 3)) * np.float32([0.3, 0.8, 0.2]) + np.float32([0.1, 0.2, -0.1])).astype(np.float32)
    K, pose = S.make_camera(f=60.0, res=64)
    for R in (33, 1025):
        uv = rng.uniform(0, 64, (R, 2)).astype(np.float32)
        dirs, cam = call_camera_rays(uv, pose[0].numpy(), K[0].numpy())
        vd, cd, dd = (torch.from_numpy(np.ascontiguousarray(a).reshape(-1)).cuda() for a in (verts, cam, dirs))
        idx = padded(R, torch.int64)
        cnt = torch.full((1,), -1, dtype=torch.int32, device="cuda")
        box = padded(6, torch.float64)
        L.call("mp_ray_aabb_hits", cd, dd, R, vd, V, 1.2, idx, cnt, box)
        torch.cuda.synchronize()
        lo, hi = verts.min(0).astype(np.float64), verts.max(0).astype(np.float64)
        ctr, half = (lo + hi) / 2.0, (hi - lo) / 2.0 * 1.2
        b = take(box, 6, "box_ws").numpy()
        assert np.array_equal(b[:3], ctr) and np.array_equal(b[3:6], half)
        want = slab_hits_ref(cam, dirs, ctr, half)
        if want.size == 0:
            want = np.zeros(1, np.int64)
        n = int(cnt.item())
        assert n == want.size
        assert np.array_equal(take(idx, n, "aabb ids").numpy(), want)


# ---------------------------------------------------------------------------------------------
# background: float64 depth2pts_outside (multiply.py:698-726), networks and bg_volume_rendering (:682-696)
# ---------------------------------------------------------------------------------------------

def depth2pts_ref(o, d, depth, r, dtype=np.float64):
    """depth2pts_outside in `dtype` for rays o, d [R,3] and depths [R,n]: [R,n,4].  Where cross(o, p_sphere) = 0 (a ray
    through the centre) the rotation angle is 0 and the point is the limit p_sphere / |p_sphere|."""
    o, d = np.asarray(o, np.float32).astype(dtype), np.asarray(d, np.float32).astype(dtype)
    depth = np.asarray(depth, np.float32).astype(dtype)
    odd = (d * o).sum(-1)
    under = odd * odd - ((o * o).sum(-1) - dtype(r) * dtype(r))
    dsph = np.sqrt(under) - odd
    ps = o + dsph[:, None] * d
    pm = o - odd[:, None] * d
    pmn = np.sqrt((pm * pm).sum(-1))
    ax = np.cross(o, ps)
    an = np.sqrt((ax * ax).sum(-1))
    ax = np.where(an[:, None] > 0, ax / np.where(an > 0, an, 1)[:, None], 0)
    ang = (np.arcsin(pmn / dtype(r))[:, None] - np.arcsin(pmn[:, None] * depth))[:, :, None]
    ca, sa = np.cos(ang), np.sin(ang)
    psn, axn = ps[:, None, :], ax[:, None, :]
    pn = psn * ca + np.cross(axn, psn) * sa + axn * (axn * psn).sum(-1, keepdims=True) * (1 - ca)
    pn = pn / np.sqrt((pn * pn).sum(-1, keepdims=True))
    return np.concatenate([pn, depth[:, :, None]], -1)


def bg_nets_ref(sc, pts4, view):
    """The background ImplicitNet / RenderingNet of oracle/port.py on the state dicts cast to float64."""
    from oracle import port
    f64 = lambda sd: {k: v.double() for k, v in sd.items()}
    code = sc["frame_code"].double()
    with torch.no_grad():
        out = port.implicit_forward(f64(sc["bg_implicit"]), torch.from_numpy(pts4), code, 10, weight_norm=False)
        rgb = port.rendering_forward(f64(sc["bg_render"]), "nerf_frame_encoding", None, None, torch.from_numpy(view),
                                     None, out[:, 1:], frame_latent_code=code, weight_norm=False, multires_view=4)
    return out[:, 0].numpy(), rgb.numpy()


def background_ref(sc, cam, dirs, r=3.0):
    """(bg_rgb [R,3], sdf [R,32], rgb samples [R,32,3]) in float64 on the kernel's float32 depths (flipped order)."""
    R = cam.shape[0]
    z = RG.bg_depths(R, r)
    pts = depth2pts_ref(cam, dirs, z, r)
    view = np.repeat(np.asarray(dirs, np.float32).astype(np.float64), 32, 0)
    sdf, rgb = bg_nets_ref(sc, pts.reshape(-1, 4), view)
    sdf, rgb = sdf.reshape(R, 32), rgb.reshape(R, 32, 3)
    z = z.astype(np.float64)
    dist = np.concatenate([z[:, :-1] - z[:, 1:], np.full((R, 1), 1e10)], 1)
    fe = dist * np.abs(sdf)
    T = np.exp(-np.concatenate([np.zeros((R, 1)), np.cumsum(fe[:, :-1], 1)], 1))
    w = (1 - np.exp(-fe)) * T
    return (w[:, :, None] * rgb).sum(1), sdf, rgb


def bg_rays(n_random=250, seed=8):
    """Ray 0: through the centre towards it, 1: through it away from it, 2: on a diagonal through it, 3-5: |p_mid| =
    1e-6, 1e-4, 1e-2, 6: near-grazing (|p_mid| = 2.99 of r = 3), then random rays from cameras inside the sphere."""
    o = [[0, 0, 2.5], [2.2, 0, 0], [0.5, 0.5, 0]]
    d = [[0, 0, -1], [1, 0, 0], [-np.sqrt(0.5), -np.sqrt(0.5), 0]]
    for pm in (1e-6, 1e-4, 1e-2):
        o.append([0, 0, 2.5])
        a = pm / 2.5
        d.append([a, 0, -np.sqrt(1 - a * a)])
    o.append([0, 2.99, 0])
    d.append([1, 0, 0])
    rng = np.random.RandomState(seed)
    cams = np.array([[0, 0, 2.5], [0.7, -0.4, 1.9], [-1.2, 0.9, -2.1], [0.1, 0.05, -0.02], [2.6, 1.0, 0.8]])
    oc = cams[rng.randint(0, len(cams), n_random)]
    dr = rng.normal(size=(n_random, 3))
    dr /= np.linalg.norm(dr, axis=1, keepdims=True)
    o = np.concatenate([np.array(o, np.float64), oc]).astype(np.float32)
    d = np.concatenate([np.array(d, np.float64), dr]).astype(np.float32)
    return o, d


_SCENE = {}


def bg_scene():
    if "sc" not in _SCENE:
        _SCENE["sc"] = S.make_scene(P=2, S=16, seed=42, weights="trained")
    return _SCENE["sc"]


def call_background(eng, cam, dirs, r=3.0):
    from multiply_b200 import engine, _lib as L
    engine.set_engine(eng)
    sc = bg_scene()
    key = "field_" + eng
    if key not in _SCENE:
        _SCENE[key] = engine.Field(sc["bg_implicit"], sc["bg_render"], background=True)
        _SCENE[key].set_cond(sc["frame_code"])
    R = cam.shape[0]
    c, d = (torch.from_numpy(np.ascontiguousarray(a, np.float32).reshape(-1)).cuda() for a in (cam, dirs))
    out = padded((R, 3))
    ws = L.workspace(L.call("mp_background_workspace_bytes", R), "cuda")
    L.call("mp_background", _SCENE[key].handle, d, c, R, float(r), out, ws, ws.numel())
    torch.cuda.synchronize()
    return take(out, (R, 3), "bg_rgb").numpy()


@pytest.mark.parametrize("eng", ["simt", "tc"])
def test_background_vs_fp64(eng):
    """mp_background on rays through the centre, at |p_mid| from 1e-6 to near-grazing and from cameras inside the
    sphere, R around the 8-rays-per-block edge: bg_rgb (in [0, 1], so M = 1) within C_BG[eng] 2^-24 of float64; every
    value finite.  The prefixes of one ray set are run, so ray 0 (the exact centre ray) is in every batch.  Measured
    worst C: 8.43 (simt), 6.8 (tc); a swapped depth flip gives 7.9e4, a last interval of 1 instead of 1e10 8.8e6."""
    o, d = bg_rays()
    want, _, _ = background_ref(bg_scene(), o, d)
    worst = 0.0
    for R in (1, 7, 8, 9, 257):
        got = call_background(eng, o[:R], d[:R])
        assert np.isfinite(got).all(), R
        worst = max(worst, float(np.abs(got - want[:R]).max()) / EPS)
    _note("bg/" + eng, worst)
    assert worst < C_BG[eng], worst


def _render_frame(r, inp, hits):
    o = r.render(inp, hits)
    torch.cuda.synchronize()
    return {k: o[k].cpu().numpy() for k in ("rgb_values", "fg_rgb_values", "normal_values", "acc_map")}


def test_centre_ray_background_is_the_limit():
    """The centre pixel (12, 12) of grid_rays(res=24) looks through the sphere's centre.  Its background is finite and
    equals the float64 limit p_sphere / |p_sphere| (within the bg gate), through mp_background on both engines and
    through mp_render_rays (hit lists without that ray, so rgb there is the background itself); every other pixel is
    bit-identical to the same frame rendered without the centre ray."""
    from multiply_b200 import engine
    sc = bg_scene()
    res, ctr = 24, 12 * 24 + 12
    inp = S.grid_rays(res=res)
    R = res * res
    dirs, cam = call_camera_rays(inp["uv"][0].numpy(), inp["pose"][0].numpy(), inp["intrinsics"][0].numpy())
    assert np.array_equal(dirs[ctr], np.float32([0, 0, -1])) and np.array_equal(cam[ctr], np.float32([0, 0, 2.5]))
    want, _, _ = background_ref(sc, cam[ctr:ctr + 1], dirs[ctr:ctr + 1])
    keep = np.arange(R) != ctr
    for eng in ("simt", "tc"):
        full = call_background(eng, cam, dirs)
        part = call_background(eng, cam[keep], dirs[keep])
        assert np.isfinite(full).all()
        assert np.array_equal(full[keep].view(np.uint32), part.view(np.uint32)), eng
        assert float(np.abs(full[ctr] - want[0]).max()) / EPS < C_BG[eng], (eng, full[ctr], want[0])
    engine.set_engine("tc")
    r = engine.Renderer(sc)
    hits = [h[h != ctr] for h in S.make_hit_lists(sc, inp)]
    full = _render_frame(r, inp, hits)
    inp2 = dict(inp, uv=inp["uv"][:, torch.from_numpy(keep)].contiguous())
    hits2 = [h - (h > ctr).to(h.dtype) for h in hits]
    part = _render_frame(r, inp2, hits2)
    for k in full:
        assert np.isfinite(full[k]).all(), k
        assert np.array_equal(full[k][keep].view(np.uint32), part[k].view(np.uint32)), k
    assert float(np.abs(full["rgb_values"][ctr] - want[0]).max()) / EPS < C_BG["tc"]


def test_background_taps_sample_order():
    """The per-sample taps of mp_render_rays (bg_sdf [R,32], bg_rgb_samples [R,32,3], in the flipped depth order the
    networks see) against float64 on the grid_rays(res=24) frame, centre ray included: per sample
    err <= C_BG_TAP 2^-24 (1 + |value|), and the bg_rgb tap within C_BG["tc"] 2^-24.  Measured worst C 1.82 per sample,
    6.56 on bg_rgb; a swapped flip gives 1.3e5 per sample."""
    from multiply_b200 import engine
    from multiply_b200.model.ray_sampler import ErrorBoundSampler
    sc = bg_scene()
    inp = S.grid_rays(res=24)
    engine.set_engine("tc")
    r = engine.Renderer(sc)
    hits = S.make_hit_lists(sc, inp)
    smp = ErrorBoundSampler(3.0, inverse_sphere_bg=True, **{k: sc["cfg"][k] for k in
                            ("near", "N_samples", "N_samples_eval", "N_samples_extra", "eps", "beta_iters",
                             "max_total_iters", "add_tiny")})
    torch.manual_seed(0)
    rngs = [{k: v for k, v in smp.draw_training_rng(h.numel()).items() if k != "states"} for h in hits]
    beta = torch.tensor(float(np.float32(abs(np.float32(r.beta_param))) + np.float32(r.beta_min)), device="cuda")
    o = r.render(inp, hits, train=dict(rng=rngs, t_rand_bg=None, beta=beta))
    torch.cuda.synchronize()
    sb = o["samples_bg"]
    sdf, rgb, bg = (t.detach().cpu().numpy() for t in (sb["sdf"], sb["rgb"], sb["bg_rgb"]))
    dirs, cam = call_camera_rays(inp["uv"][0].numpy(), inp["pose"][0].numpy(), inp["intrinsics"][0].numpy())
    want_bg, want_sdf, want_rgb = background_ref(sc, cam, dirs)
    assert np.isfinite(sdf).all() and np.isfinite(rgb).all() and np.isfinite(bg).all()
    c = max(_ratio(np.abs(sdf - want_sdf), 1 + np.abs(want_sdf)).max(),
            _ratio(np.abs(rgb - want_rgb), 1 + np.abs(want_rgb)).max())
    _note("bg_taps", c)
    assert c < C_BG_TAP, c
    cb = float(np.abs(bg - want_bg).max()) / EPS
    _note("bg_taps_rgb", cb)
    assert cb < C_BG["tc"], cb
