"""GPU: the backward of the SMPL server and the deformer (mp_smpl_backward, mp_deform_inverse_backward,
mp_deform_forward_jac_backward) and the mirror's autograd through them, against the float64 autograd of oracle/port.py's
restatements (pinned to the reference's own code by test_body_grad_golden.py) and against tests/golden/body_grad.npz.

Gates are per element, err <= C * 2^-24 * M.  M is the float64 sum of |terms| behind the element where the backward is one
reduction over points (d_tfs: sum_i w_ij |dL/dA_i|; d_x: |A^-T| |g|); for the SMPL parameters, whose terms pass through the
whole chain, M is the largest |gradient| among the four parameter outputs of the call.  C is 4x the worst measured on
one H100 (printed as MEASURED)."""
import os
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from multiply_b200 import scene as S                 # noqa: E402
from oracle import gen_golden_body_grad as G          # noqa: E402
from oracle import port                               # noqa: E402

from _abi import padded, take                         # noqa: E402
from _body_grad_port import port_smpl_grads, float64  # noqa: E402
from _setups import Smpl, dirty_workspace, points, posed_body, small_model  # noqa: E402

EPS = 2.0 ** -24
MEASURED = {}
# 4x the worst measured on one H100 80GB HBM3 at a 700 W power limit: 4.69 (SMPL parameters, mirror chains included),
# 44.7 (d_x / d_x_c, at 1.6 M points), 98.5 (d_tfs, at 1.6 M points: 1.6 M terms per bone)
C_SMPL = 19.0
C_DX = 179.0
C_TFS = 394.0


def _note(key, c):
    MEASURED[key] = max(MEASURED.get(key, 0.0), float(c))
    return c


@pytest.fixture(scope="module", autouse=True)
def _print_measured():
    yield
    for k in sorted(MEASURED):
        print("MEASURED %s C=%.3g" % (k, MEASURED[k]))


def _c(err, M):
    err, M = np.abs(np.asarray(err, np.float64)), np.asarray(M, np.float64)
    r = np.where(M > 0, err / (EPS * np.where(M > 0, M, 1.0)), np.where(err == 0, 0.0, np.inf))
    return float(r.max()) if r.size else 0.0


def _L():
    from multiply_b200 import _lib as L
    return L


def _bits(*arrs):
    return [np.asarray(a, np.float32).view(np.uint32).copy() for a in arrs]


# ---------------------------------------------------------------------------------------------
# SMPL server
# ---------------------------------------------------------------------------------------------

def _poses():
    rng = np.random.RandomState(21)
    u = np.array([0.36, -0.48, 0.8])
    large = rng.normal(0, 0.3, (24, 3))
    large[0], large[5], large[23] = (np.pi - 1e-3) * u, (np.pi + 1e-3) * u, np.pi * u
    return {"zero": np.zeros(72), "canonical": G.CANONICAL.copy(), "random": rng.normal(0, 0.4, 72),
            "large": large.reshape(72)}


SMPL_MODELS = ["V1", "V127", "V128", "V129", "smpl6890"]
MODES = ["verts", "tfs", "both"]


@pytest.mark.parametrize("name", SMPL_MODELS)
def test_smpl_backward_vs_port(name):
    """Every pose x (absolute, placement) x upstream mode against the port's float64 autograd; outputs padded, a 0xFF
    workspace, two runs bit-identical."""
    model = G.model64() if name == "smpl6890" else small_model(int(name[1:]))
    model = {k: (v.numpy() if torch.is_tensor(v) else np.asarray(v)) for k, v in model.items()}
    model = {k: (v.astype(np.float32) if k != "parents" else v) for k, v in model.items()}
    hd = Smpl(model)
    V = hd.V
    rng = np.random.RandomState(5)
    for pn, theta in _poses().items():
        theta = theta.astype(np.float32)
        for absolute, scale, transl in ((0, 1.0, (0.0, 0.0, 0.0)), (1, 1.0, (0.0, 0.0, 0.0)), (0, 0.7, (0.3, -0.2, 1.1)),
                                        (1, 1.6, (-0.5, 0.4, 0.2))):
            betas = rng.normal(0, 1, 10).astype(np.float32)
            u_v, u_t = rng.randn(V, 3).astype(np.float32), rng.randn(24, 4, 4).astype(np.float32)
            for mode in MODES:
                uv = u_v if mode != "tfs" else None
                ut = u_t if mode != "verts" else None
                want = port_smpl_grads(model, hd.cinv, np.float32(scale), transl, theta, betas, absolute, False,
                                       np.zeros((V, 3)) if uv is None else uv, np.zeros((24, 4, 4)) if ut is None else ut)
                got = hd.backward(scale, transl, theta, betas, absolute, uv, ut)
                again = hd.backward(scale, transl, theta, betas, absolute, uv, ut)
                for a, b in zip(_bits(*got), _bits(*again)):
                    assert np.array_equal(a, b), (name, pn, mode)
                M = max(np.abs(want[k]).max() for k in ("scale", "transl", "thetas", "betas"))
                for g, key in zip(got, ("scale", "transl", "thetas", "betas")):
                    w = want[key].reshape(-1)
                    c = _note("smpl/%s/%s" % (key, name), _c(g - w, np.full(w.shape, M)))
                    assert c < C_SMPL, (name, pn, absolute, mode, key, c)


def test_smpl_backward_matches_golden(golden_dir):
    gold = dict(np.load(os.path.join(golden_dir, "body_grad.npz")))
    model = {k: (v.numpy().astype(np.float32) if torch.is_tensor(v) and v.is_floating_point() else
                 (v.numpy() if torch.is_tensor(v) else v)) for k, v in S.make_smpl_model(G.MODEL_SEED).items()}
    hd = Smpl(model)
    for k, name in enumerate(G.SMPL_CASES):
        g = lambda key: gold[f"smpl_{name}_{key}"]
        u_v, u_t = G.cotangents(100 + k, (hd.V, 3), (24, 4, 4))
        betas = np.zeros(10) if bool(g("v_template")) else g("betas")
        got = hd.backward(g("scale"), g("transl"), g("theta"), betas, int(g("absolute")), u_v, u_t)
        M = max(np.abs(g("grad_" + k)).max() for k in ("scale", "transl", "thetas", "betas"))
        for gv, key in zip(got, ("scale", "transl", "thetas", "betas")):
            w = g("grad_" + key).reshape(-1)
            if bool(g("v_template")) and key == "betas":
                continue              # the mirror discards them (test_mirror_smpl_v_template_betas)
            c = _note("golden_smpl/" + key, _c(gv - w, np.full(w.shape, M)))
            assert c < C_SMPL, (name, key, c)


def test_smpl_backward_ignores_later_forward():
    """forward(A), forward(B), backward(A) equals backward(A) alone, bit for bit."""
    model = {k: (v.numpy() if torch.is_tensor(v) else v) for k, v in S.make_smpl_model(300).items()}
    hd = Smpl(model)
    rng = np.random.RandomState(3)
    a = (0.8, (0.1, 0.2, 0.3), rng.normal(0, 0.4, 72), rng.normal(0, 1, 10), 0)
    b = (1.5, (-1.0, 0.4, 0.9), rng.normal(0, 1.0, 72), rng.normal(0, 2, 10), 1)
    u_v, u_t = rng.randn(hd.V, 3), rng.randn(24, 4, 4)
    alone = hd.backward(*a, u_v, u_t)
    hd.forward(*a)
    hd.forward(*b)
    after = hd.backward(*a, u_v, u_t)
    for x, y in zip(_bits(*alone), _bits(*after)):
        assert np.array_equal(x, y)


# ---------------------------------------------------------------------------------------------
# deformer
# ---------------------------------------------------------------------------------------------

def _nearest(x, verts):
    """port.knn_points' definition on the device: d2 = (dx*dx + dy*dy) + dz*dz in fp32, lowest index on ties."""
    x, v = x.cuda().float(), verts.cuda().float()
    out = torch.empty(x.shape[0], dtype=torch.int64, device="cuda")
    ar = torch.arange(v.shape[0], device="cuda")
    for s in range(0, x.shape[0], 8192):
        xs = x[s:s + 8192]
        dx, dy, dz = xs[:, 0:1] - v[None, :, 0], xs[:, 1:2] - v[None, :, 1], xs[:, 2:3] - v[None, :, 2]
        d = dx * dx
        d = d + dy * dy
        d = d + dz * dz
        m = d.min(1, keepdim=True).values
        out[s:s + 8192] = torch.where(d == m, ar[None], v.shape[0]).min(1).values
    return out


def _ref_inverse(x, idx, W, tfs, u, keep=None):
    """port.skinning(inverse=True) in float64 on the device with the weights of vertex idx: (x_c, d_x, d_tfs, M_x, M_tfs).
    keep: points whose bone terms count (the others have no vertex on the GPU)."""
    xv = x.cuda().double().requires_grad_(True)
    tv = tfs.cuda().double().requires_grad_(True)
    w = W.cuda().double()[idx][None]
    A = torch.einsum("bpn,bnij->bpij", w, tv[None])
    A.retain_grad()
    xh = torch.nn.functional.pad(xv[None], (0, 1), value=1.0)
    xc = torch.einsum("bpij,bpj->bpi", A.inverse(), xh)[0, :, :3]
    (xc * u.cuda().double()).sum().backward()
    dA = A.grad[0]
    wk = w[0] if keep is None else w[0] * keep.cuda().double()[:, None]
    M_tfs = torch.einsum("pn,pij->nij", wk, dA.abs())
    inv = A.detach()[0].inverse()[:, :3, :3]
    M_x = torch.einsum("pji,pj->pi", inv.abs(), u.cuda().double().abs())
    d_tfs = torch.einsum("pn,pij->nij", wk, dA)
    return xc.detach(), xv.grad, d_tfs, M_x, M_tfs


def _inv_backward(b, x, u, exact_far):
    L = _L()
    N = x.shape[0]
    xd, ud = x.cuda().contiguous(), u.cuda().float().contiguous()
    d_tfs, d_x, xc = padded((24, 4, 4)), padded((N, 3)), padded((N, 3))
    ws = dirty_workspace(L.call("mp_deform_backward_workspace_bytes", N))
    L.call("mp_deform_inverse_backward", b.handle, xd if N else None, N, int(exact_far), ud if N else None, d_tfs, d_x, xc,
           ws, ws.numel())
    torch.cuda.synchronize()
    return take(d_tfs, (24, 4, 4), "d_tfs"), take(d_x, (N, 3), "d_x"), take(xc, (N, 3), "x_c")


WAVE = 1024 * 256
INV_SIZES = [0, 1, 255, 256, 257, WAVE - 1, WAVE + 1, 2 * WAVE - 1, 2 * WAVE + 1, 1600000]


@pytest.mark.parametrize("N", INV_SIZES)
@pytest.mark.parametrize("exact_far", [1, 0])
def test_deform_inverse_backward(N, exact_far):
    """d_x, the full 4x4 d_tfs (bottom row included) and the recomputed x_c (bit-equal to mp_deform_inverse's) against
    the port's float64 autograd; with exact_far = 0 the points are near the body or 5 away from it (no vertex:
    d_x = d_x_c, nothing to the bones).  Padded outputs, a 0xFF workspace, reruns bit-identical."""
    b, _ = posed_body()
    far = 0.3 if exact_far else -5.0
    x = points(N, b.verts_p, 11 + N, far=far)
    u = torch.from_numpy(np.random.RandomState(N).randn(N, 3).astype(np.float32))
    d_tfs, d_x, xc = _inv_backward(b, x, u, exact_far)
    d_tfs2, d_x2, xc2 = _inv_backward(b, x, u, exact_far)
    assert torch.equal(d_tfs.view(torch.int32), d_tfs2.view(torch.int32)) and torch.equal(d_x.view(torch.int32),
                                                                                          d_x2.view(torch.int32))
    if N == 0:
        assert not d_tfs.any()
        return
    xf, _ = b.deform_inverse(x.cuda(), exact_far=bool(exact_far))
    assert torch.equal(xc.view(torch.int32), xf.cpu().view(torch.int32))
    idx = _nearest(x, b.verts_p)
    keep = None
    if not exact_far:
        none = (xf.cpu() == x).all(1)             # no vertex within reach: x_c = x
        keep = ~none
        assert torch.equal(d_x[none].view(torch.int32), u[none].view(torch.int32))
    _, want_dx, want_tfs, M_x, M_tfs = _ref_inverse(x, idx, b.weights, b.tfs, u, keep)
    sel = slice(None) if keep is None else keep.cuda()
    c = _note("inverse/d_x", _c((d_x.cuda().double() - want_dx)[sel].cpu(), M_x[sel].cpu()))
    assert c < C_DX, c
    c = _note("inverse/d_tfs", _c(d_tfs.double() - want_tfs.cpu(), M_tfs.cpu()))
    assert c < C_TFS, c


def test_deform_inverse_backward_ties():
    """Points at exact midpoints of lattice vertices (fp32 ties): the recomputed x_c is bit-equal to the forward's and
    the gradients follow the lowest-index vertex."""
    from multiply_b200 import engine
    g = np.arange(6) / 32.0
    V = np.stack(np.meshgrid(g, g, g, indexing="ij"), -1).reshape(-1, 3).astype(np.float32)
    W = np.random.RandomState(1).dirichlet(np.ones(24) * 0.3, V.shape[0]).astype(np.float32)
    b = engine.Body(torch.from_numpy(V), torch.from_numpy(W), cano_cell=0.1001)
    _, srv = posed_body()
    o = srv(torch.ones(1), torch.zeros(1, 3), torch.from_numpy(np.random.RandomState(2).normal(0, 0.3, (1, 72)).astype(
        np.float32)), torch.zeros(1, 10))
    b.set_pose(torch.from_numpy(V), o["smpl_tfs"][0])
    x = torch.from_numpy((V[:-1] + np.array([1.0 / 64, 0, 0], np.float32)).astype(np.float32))
    u = torch.from_numpy(np.random.RandomState(3).randn(x.shape[0], 3).astype(np.float32))
    d_tfs, d_x, xc = _inv_backward(b, x, u, 1)
    xf, _ = b.deform_inverse(x.cuda(), exact_far=True)
    assert torch.equal(xc.view(torch.int32), xf.cpu().view(torch.int32))
    idx = _nearest(x, torch.from_numpy(V))
    _, want_dx, want_tfs, M_x, M_tfs = _ref_inverse(x, idx, torch.from_numpy(W), b.tfs, u)
    assert _note("ties/d_x", _c(d_x.double() - want_dx.cpu(), M_x.cpu())) < C_DX
    assert _note("ties/d_tfs", _c(d_tfs.double() - want_tfs.cpu(), M_tfs.cpu())) < C_TFS


def test_deform_inverse_backward_refuses_root_finder():
    from multiply_b200 import _lib as L
    b, _ = posed_body()
    b.set_root_finder(5)
    try:
        with pytest.raises(L.MpError, match="root finder"):
            b.deform_inverse_backward(torch.zeros(4, 3, device="cuda"), torch.ones(4, 3, device="cuda"))
    finally:
        b.set_root_finder(0)


def _fwd_backward(b, xc, u_xd, u_J):
    L = _L()
    N = xc.shape[0]
    d_tfs, d_xc = padded((24, 4, 4)), padded((N, 3))
    ws = dirty_workspace(L.call("mp_deform_backward_workspace_bytes", N))
    dxd = None if u_xd is None else u_xd.cuda().float().contiguous()
    dJ = None if u_J is None else u_J.cuda().float().reshape(N, 9).contiguous()
    L.call("mp_deform_forward_jac_backward", b.handle, xc.cuda().contiguous(), N, dxd, dJ, d_tfs, d_xc, ws, ws.numel())
    torch.cuda.synchronize()
    return take(d_tfs, (24, 4, 4), "d_tfs"), take(d_xc, (N, 3), "d_x_c")


def _ref_forward(xc, idx, W, tfs, u_xd, u_J):
    """port.forward_skinning + the inverse Jacobian in float64 on the device with the weights of vertex idx."""
    xv = xc.cuda().double().requires_grad_(True)
    tv = tfs.cuda().double().requires_grad_(True)
    w = W.cuda().double()[idx]
    T = torch.einsum("pn,nij->pij", w, tv)
    T.retain_grad()
    x_d = torch.einsum("pij,pj->pi", T[:, :3, :3], xv) + T[:, :3, 3]
    Ji = torch.linalg.inv(T[:, :3, :3])
    loss = 0.0
    if u_xd is not None:
        loss = loss + (x_d * u_xd.cuda().double()).sum()
    if u_J is not None:
        loss = loss + (Ji * u_J.cuda().double().reshape(-1, 3, 3)).sum()
    loss.backward()
    M_tfs = torch.einsum("pn,pij->nij", w, T.grad.abs())
    Mx = torch.zeros_like(xv) if u_xd is None else torch.einsum("pij,pi->pj", T.detach()[:, :3, :3].abs(),
                                                                u_xd.cuda().double().abs())
    gx = torch.zeros_like(xv) if xv.grad is None else xv.grad
    return gx, torch.einsum("pn,pij->nij", w, T.grad), Mx, M_tfs


_MESH = {}


def _cano_mesh_sizes():
    """Vertex counts of generate_mesh's canonical meshes (MISE + marching cubes + largest component) of both persons of
    scene.make_scene(weights='trained')."""
    if "v" not in _MESH:
        from multiply_b200 import engine
        from multiply_b200.utils import mesh as umesh
        sc = S.make_scene(P=2, S=16, seed=42, weights="trained")
        vs = []
        for p in sc["persons"]:
            f = engine.Field(p["implicit"], p["render"])
            f.set_cond(p["cond"])
            center, extent, pad = umesh.bounds(p["verts_c"])
            v, _, _ = f.extract_mesh(center, extent, 32, 3, 0.0, pad)
            vs.append(v.cpu())
        _MESH["v"] = vs
    return _MESH["v"]


@pytest.mark.parametrize("mode", ["x_d", "Jinv", "both"])
def test_forward_jac_backward(mode):
    """On generate_mesh's canonical-mesh vertices (and N = 1, 257): d_x_c and d_tfs (bottom row 0) against the port's
    float64 autograd, d_x_d alone, d_Jinv alone and both; padded outputs, 0xFF workspace, reruns bit-identical."""
    b, _ = posed_body()
    sets = [v for v in _cano_mesh_sizes()] + [points(1, b.verts_c, 1), points(257, b.verts_c, 2, far_frac=0.0)]
    for k, xc in enumerate(sets):
        N = xc.shape[0]
        rng = np.random.RandomState(k)
        u_xd = torch.from_numpy(rng.randn(N, 3).astype(np.float32)) if mode != "Jinv" else None
        u_J = torch.from_numpy(rng.randn(N, 9).astype(np.float32)) if mode != "x_d" else None
        d_tfs, d_xc = _fwd_backward(b, xc, u_xd, u_J)
        d_tfs2, d_xc2 = _fwd_backward(b, xc, u_xd, u_J)
        assert torch.equal(d_tfs.view(torch.int32), d_tfs2.view(torch.int32))
        assert torch.equal(d_xc.view(torch.int32), d_xc2.view(torch.int32))
        assert not d_tfs[:, 3, :].any()
        idx = _nearest(xc, b.verts_c)
        gx, gt, Mx, Mt = _ref_forward(xc, idx, b.weights, b.tfs, u_xd, u_J)
        c = _note("forward_jac/%s/d_x_c" % mode, _c(d_xc.double() - gx.cpu(), Mx.cpu()))
        assert c < C_DX, (k, N, c)
        c = _note("forward_jac/%s/d_tfs" % mode, _c(d_tfs.double() - gt.cpu(), Mt.cpu()))
        assert c < C_TFS, (k, N, c)


def test_deformer_backward_matches_golden(golden_dir):
    gold = dict(np.load(os.path.join(golden_dir, "body_grad.npz")))
    from multiply_b200 import engine
    W = S.make_smpl_model(G.MODEL_SEED)["lbs_weights"]
    b = engine.Body(torch.from_numpy(gold["fwd_verts_c"].astype(np.float32)), W, cano_cell=0.1001)
    b.set_pose(torch.from_numpy(gold["inv_verts_p"].astype(np.float32)), torch.from_numpy(gold["inv_tfs"].astype(np.float32)))
    N = gold["inv_x"].shape[0]
    u_xc, = G.cotangents(200, (N, 3))
    d_tfs, d_x, _ = _inv_backward(b, torch.from_numpy(gold["inv_x"].astype(np.float32)), torch.from_numpy(u_xc), 1)
    w = gold["inv_grad_x"]
    assert _note("golden/inverse/d_x", _c(d_x.numpy() - w, np.abs(w).max())) < C_DX
    w = gold["inv_grad_tfs"]
    assert _note("golden/inverse/d_tfs", _c(d_tfs.numpy() - w, np.abs(w).max())) < C_TFS
    u_xd, u_J = G.cotangents(201, (N, 3), (N, 3, 3))
    d_tfs, d_xc = _fwd_backward(b, torch.from_numpy(gold["fwd_x_c"].astype(np.float32)), torch.from_numpy(u_xd),
                                torch.from_numpy(u_J))
    w = gold["fwd_grad_x_c"]
    assert _note("golden/forward_jac/d_x_c", _c(d_xc.numpy() - w, np.abs(w).max())) < C_DX
    w = gold["fwd_grad_tfs"]
    assert _note("golden/forward_jac/d_tfs", _c(d_tfs.numpy() - w, np.abs(w).max())) < C_TFS


# ---------------------------------------------------------------------------------------------
# mirror: torch.autograd through SMPLServer -> deformer, against the same chains in the float64 port
# ---------------------------------------------------------------------------------------------

def _mirror_setup():
    from multiply_b200.model.smpl import SMPLServer
    from multiply_b200.model.deformer import SMPLDeformer
    sm = S.make_smpl_model(300)
    srv = SMPLServer(model=sm)
    dfm = SMPLDeformer(smpl_verts=srv.verts_c, smpl_weights=srv.weights)
    rng = np.random.RandomState(31)
    params = dict(scale=torch.tensor([0.9]), transl=torch.tensor([[0.1, -0.2, 0.3]]),
                  thetas=torch.from_numpy(rng.normal(0, 0.3, (1, 72)).astype(np.float32)),
                  betas=torch.from_numpy(rng.normal(0, 1, (1, 10)).astype(np.float32)))
    return sm, srv, dfm, params


def _port_chain(sm, srv, params, tail):
    """SMPLServer (port.smpl_server_forward, d_scale by linearity as in _body_grad_port) -> tail(verts, tfs) -> loss, in
    float64 on the CPU; returns the gradients of scale, transl, thetas, betas."""
    from _body_grad_port import model64, _t
    m = model64(sm)
    cinv = _t(srv.tfs_c_inv.cpu().numpy())
    with float64():
        t, th, b = (_t(params[k].numpy().reshape(-1), True) for k in ("transl", "thetas", "betas"))

        def loss_at(s):
            o = port.smpl_server_forward(m, cinv, s, t, th, b)
            return tail(o["smpl_verts"], o["smpl_tfs"], s)
        s0 = float(params["scale"])
        loss_at(torch.full((1,), s0)).backward()
        with torch.no_grad():
            h = 1e-6
            ds = (loss_at(torch.full((1,), s0 + h)) - loss_at(torch.full((1,), s0 - h))) / (2 * h)
        return dict(scale=np.array([float(ds)]), transl=t.grad.numpy(), thetas=th.grad.numpy(), betas=b.grad.numpy())


def _mirror_grads(srv, params, tail_gpu):
    p = {k: v.clone().cuda().requires_grad_(True) for k, v in params.items()}
    o = srv(p["scale"], p["transl"], p["thetas"], p["betas"])
    loss = tail_gpu(o)
    g = torch.autograd.grad(loss, [p["scale"], p["transl"], p["thetas"], p["betas"]])
    return {k: x.cpu().numpy().reshape(-1) for k, x in zip(("scale", "transl", "thetas", "betas"), g)}


def _compare(key, got, want):
    M = max(np.abs(w).max() for w in want.values())
    for k in got:
        w = want[k].reshape(-1)
        c = _note("mirror/%s/%s" % (key, k), _c(got[k] - w, np.full(w.shape, M)))
        assert c < C_SMPL, (key, k, c)


def test_mirror_opt_depth_chain():
    """SMPLServer -> Multiply.get_deformed_mesh_fast_mode_multiple_person -> (1/scale) verts -> a seeded loss: the
    opt_depth chain (multiply_model.py:230-487) to scale, transl, thetas, betas."""
    from multiply_b200.model.multiply import Multiply
    sm, srv, dfm, params = _mirror_setup()
    m = Multiply.__new__(Multiply)
    torch.nn.Module.__init__(m)
    m.deformer_list = [dfm]
    verts = _cano_mesh_sizes()[0][:3000]
    u = torch.from_numpy(np.random.RandomState(4).randn(verts.shape[0], 3).astype(np.float32))
    W = srv.weights[0].cpu().double()
    idx = _nearest(verts, srv.verts_c[0]).cpu()

    def tail_gpu(o):
        xd = m.get_deformed_mesh_fast_mode_multiple_person(verts.cuda()[None], o["smpl_tfs"], 0)
        return ((1.0 / o_scale[0]) * xd[0] * u.cuda()).sum()

    def tail_port(verts_p, tfs, s):
        T = torch.einsum("pn,nij->pij", W[idx], tfs)
        xd = torch.einsum("pij,pj->pi", T[:, :3, :3], verts.double()) + T[:, :3, 3]
        return ((1.0 / s[0]) * xd * u.double()).sum()

    p = {k: v.clone().cuda().requires_grad_(True) for k, v in params.items()}
    o_scale = p["scale"]
    o = srv(p["scale"], p["transl"], p["thetas"], p["betas"])
    g = torch.autograd.grad(tail_gpu(o), [p["scale"], p["transl"], p["thetas"], p["betas"]])
    got = {k: x.cpu().numpy().reshape(-1) for k, x in zip(("scale", "transl", "thetas", "betas"), g)}
    _compare("opt_depth", got, _port_chain(sm, srv, params, tail_port))


def test_mirror_inverse_deformer_chain():
    """SMPLServer -> SMPLDeformer.forward(inverse=True, smpl_verts) -> a seeded loss on x_c, gradients to the SMPL
    parameters and to x; none to smpl_verts."""
    sm, srv, dfm, params = _mirror_setup()
    with torch.no_grad():
        o0 = srv(params["scale"], params["transl"], params["thetas"], params["betas"])
    x = points(2000, o0["smpl_verts"][0], 8, far_frac=0.0)
    u = torch.from_numpy(np.random.RandomState(5).randn(2000, 3).astype(np.float32))
    idx = _nearest(x, o0["smpl_verts"][0]).cpu()
    W = srv.weights[0].cpu().double()

    def tail_gpu(o):
        xc, _ = dfm.forward(xg, o["smpl_tfs"], return_weights=False, inverse=True, smpl_verts=o["smpl_verts"])
        return (xc * u.cuda()).sum()

    def tail_port(verts_p, tfs, s):
        xc = port.skinning(x.double()[None], W[idx][None], tfs[None], inverse=True)[0]
        return (xc * u.double()).sum()

    xg = x.cuda().requires_grad_(True)
    got = _mirror_grads(srv, params, tail_gpu)
    _compare("inverse", got, _port_chain(sm, srv, params, tail_port))
    p = {k: v.cuda() for k, v in params.items()}
    o = srv(p["scale"], p["transl"], p["thetas"], p["betas"])
    vp = o["smpl_verts"].clone().requires_grad_(True)
    xc, _ = dfm.forward(xg, o["smpl_tfs"], return_weights=False, inverse=True, smpl_verts=vp)
    (xc * u.cuda()).sum().backward()
    assert xg.grad is not None and vp.grad is None


def test_mirror_forward_skinning_chain():
    """SMPLServer -> forward_skinning + jacobian_inverse (the transforms the body is posed with) -> a seeded loss; a
    different transform tensor is refused."""
    sm, srv, dfm, params = _mirror_setup()
    xc = points(1500, srv.verts_c[0], 9, far_frac=0.0)
    u_x = torch.from_numpy(np.random.RandomState(6).randn(1500, 3).astype(np.float32))
    u_J = torch.from_numpy(np.random.RandomState(7).randn(1500, 3, 3).astype(np.float32))
    idx = _nearest(xc, srv.verts_c[0]).cpu()
    W = srv.weights[0].cpu().double()

    def tail_gpu(o):
        dfm.forward(torch.zeros(1, 3, device="cuda"), o["smpl_tfs"].detach(), return_weights=False, inverse=True,
                    smpl_verts=o["smpl_verts"].detach())
        xd = dfm.forward_skinning(xc.cuda()[None], None, o["smpl_tfs"])
        J = dfm.jacobian_inverse(xc.cuda(), o["smpl_tfs"])
        return (xd[0] * u_x.cuda()).sum() + (J * u_J.cuda()).sum()

    def tail_port(verts_p, tfs, s):
        T = torch.einsum("pn,nij->pij", W[idx], tfs)
        xd = torch.einsum("pij,pj->pi", T[:, :3, :3], xc.double()) + T[:, :3, 3]
        return (xd * u_x.double()).sum() + (torch.linalg.inv(T[:, :3, :3]) * u_J.double()).sum()

    got = _mirror_grads(srv, params, tail_gpu)
    _compare("forward_skinning", got, _port_chain(sm, srv, params, tail_port))
    other = torch.eye(4, device="cuda").repeat(1, 24, 1, 1).requires_grad_(True)
    with pytest.raises(ValueError):
        dfm.forward_skinning(xc.cuda()[None], None, other)


def test_mirror_no_grad_unchanged():
    """Without requires_grad (and under no_grad) the outputs are bit-equal to the plain forward and carry no grad_fn."""
    sm, srv, dfm, params = _mirror_setup()
    p = {k: v.cuda() for k, v in params.items()}
    a = srv(p["scale"], p["transl"], p["thetas"], p["betas"])
    q = {k: v.clone().requires_grad_(True) for k, v in p.items()}
    with torch.no_grad():
        b = srv(q["scale"], q["transl"], q["thetas"], q["betas"])
    c = srv(q["scale"], q["transl"], q["thetas"], q["betas"])
    for k in ("smpl_verts", "smpl_tfs"):
        assert a[k].grad_fn is None and b[k].grad_fn is None and c[k].grad_fn is not None
        assert torch.equal(a[k], b[k]) and torch.equal(a[k], c[k].detach())
    x = points(500, a["smpl_verts"][0], 3).cuda()
    xc0, o0 = dfm.forward(x, a["smpl_tfs"], return_weights=False, inverse=True, smpl_verts=a["smpl_verts"])
    xc1, o1 = dfm.forward(x, c["smpl_tfs"], return_weights=False, inverse=True, smpl_verts=c["smpl_verts"])
    assert xc0.grad_fn is None and xc1.grad_fn is not None
    assert torch.equal(xc0, xc1.detach()) and torch.equal(o0, o1)


def test_mirror_smpl_v_template_betas():
    """A server built with v_template ignores betas (smpl.py:65-66): their gradient is exactly 0."""
    from multiply_b200.model.smpl import SMPLServer
    sm = S.make_smpl_model(300)
    srv = SMPLServer(model=sm, v_template=sm["v_template"].numpy() * 1.01)
    b = torch.randn(1, 10, device="cuda", requires_grad=True)
    th = (0.2 * torch.randn(1, 72, device="cuda")).requires_grad_(True)
    o = srv(torch.ones(1, device="cuda"), torch.zeros(1, 3, device="cuda"), th, b)
    (o["smpl_verts"].sum() + o["smpl_tfs"].sum()).backward()
    assert b.grad is not None and not b.grad.any() and th.grad.abs().sum() > 0
