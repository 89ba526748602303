"""GPU: the first-order backward of ImplicitNet and RenderingNet 'pose_no_view' (mp_implicit_backward,
mp_render_backward, engine.ImplicitFunction / engine.RenderFunction behind the mirror modules) against float64 torch
autograd through oracle/port.py's implicit_forward / rendering_forward (evaluated on the device in float64).

Every gradient tensor must satisfy max|g - g_ref| <= 1e-4 max|g_ref|, on the geometric-init and the trained-like weights
(scene.perturb_networks), with weight norm (foreground) and without (background), at sizes around the 64-row and
128-point tile edges, at 3 x 128 x SMs + 77 points and at a size that spans three internal chunks of 32768 points."""
import pytest
import torch

from multiply_b200 import engine, scene as S, _lib as L
from multiply_b200.model import networks
from oracle import port

from _abi import same
from _setups import dirty_workspace

pytestmark = pytest.mark.gpu

TOL = 1e-4
WEIGHTS = ["geometric", "trained"]
CHUNKS3 = 2 * 32768 + 5


def _sizes():
    T = 128 * int(L.call("mp_device_sm_count"))
    return [1, 127, 128, 129, 3 * T + 77, CHUNKS3]


@pytest.fixture(scope="module")
def scenes():
    engine.set_engine("tc")
    out = {}
    for w in WEIGHTS:
        sc = S.make_scene(P=1, S=16, seed=42, weights=w)
        p = sc["persons"][0]
        fg = engine.Field(p["implicit"], p["render"])
        bg = engine.Field(sc["bg_implicit"], sc["bg_render"], background=True)
        out[w] = dict(sc=sc, fg=fg, bg=bg, fg_cond=p["cond"], bg_cond=sc["frame_code"])
    return out


def _inputs(n, d, seed, lo=-1.0, hi=1.0):
    g = torch.Generator().manual_seed(seed)
    return (lo + (hi - lo) * torch.rand(n, d, generator=g)).cuda()


def _randn(shape, seed):
    return torch.randn(*shape, generator=torch.Generator().manual_seed(seed)).cuda()


def _effective_leaves(sd, n_lin):
    """float64 leaves lin{l}.weight (the applied W: g v / ||v|| where weight-normed) and lin{l}.bias."""
    leaves = {}
    for l in range(n_lin):
        if f"lin{l}.weight_v" in sd:
            w = torch._weight_norm(sd[f"lin{l}.weight_v"].double(), sd[f"lin{l}.weight_g"].double(), 0)
        else:
            w = sd[f"lin{l}.weight"].double()
        leaves[f"lin{l}.weight"] = w.detach().cuda().requires_grad_(True)
        leaves[f"lin{l}.bias"] = sd[f"lin{l}.bias"].double().cuda().requires_grad_(True)
    return leaves


def _ref_implicit(sd, x, cond, multires, d_sdf, d_feat):
    leaves = _effective_leaves(sd, 9)
    xs = x.double().requires_grad_(True)
    c = cond.reshape(1, -1).double().cuda().requires_grad_(True)
    y = port.implicit_forward(leaves, xs, c, multires, weight_norm=False)
    loss = (y[:, 0] * (0 if d_sdf is None else d_sdf.double())).sum()
    loss = loss + (y[:, 1:] * (0 if d_feat is None else d_feat.double())).sum()
    params = [leaves[f"lin{l}.{k}"] for l in range(9) for k in ("weight", "bias")]
    g = torch.autograd.grad(loss, [xs, c] + params, allow_unused=True)
    return dict(d_x=g[0], d_cond=g[1].reshape(-1), d_weight=list(g[2::2]), d_bias=list(g[3::2]))


def _ref_render(sd, pts, nrm, feat, body_pose, d_rgb):
    leaves = _effective_leaves(sd, 5)
    leaves["lin_pose.weight"] = sd["lin_pose.weight"].double().cuda().requires_grad_(True)
    leaves["lin_pose.bias"] = sd["lin_pose.bias"].double().cuda().requires_grad_(True)
    p, n, f = (t.double().requires_grad_(True) for t in (pts, nrm, feat))
    bp = body_pose.reshape(1, -1).double().cuda().requires_grad_(True)
    rgb = port.rendering_forward(leaves, "pose_no_view", p, n, None, bp, f, weight_norm=False)
    params = [leaves[f"lin{l}.{k}"] for l in range(5) for k in ("weight", "bias")]
    g = torch.autograd.grad((rgb * d_rgb.double()).sum(),
                            [p, n, f, bp, leaves["lin_pose.weight"], leaves["lin_pose.bias"]] + params)
    return dict(d_points=g[0], d_normals=g[1], d_feat=g[2], d_body_pose=g[3].reshape(-1), d_lin_pose_weight=g[4],
                d_lin_pose_bias=g[5], d_weight=list(g[6::2]), d_bias=list(g[7::2]))


# a pre-activation this close to 0 may round to the other side in fp32: the ReLU derivative is ambiguous there
KINK = 1e-6


def _relu_margin(sd, pts, nrm, feat, body_pose):
    """Each point's smallest |pre-activation| over the colour net's ReLU layers, in float64.  Where it is below KINK,
    relu' (0 or 1) of an fp32 evaluation may differ from the float64 one, and so may that point's whole contribution to
    every gradient, a whole term rather than a rounding error."""
    leaves = _effective_leaves(sd, 4)
    with torch.no_grad():
        bp = body_pose.reshape(1, -1).double().cuda()
        pf = torch.nn.functional.linear(bp, sd["lin_pose.weight"].double().cuda(), sd["lin_pose.bias"].double().cuda())
        h = torch.cat([pts.double(), nrm.double(), pf.expand(pts.shape[0], -1), feat.double()], -1)
        margin = torch.full((pts.shape[0],), float("inf"), dtype=torch.float64, device=pts.device)
        for l in range(4):
            z = torch.nn.functional.linear(h, leaves[f"lin{l}.weight"], leaves[f"lin{l}.bias"])
            margin = torch.minimum(margin, z.abs().min(1).values)
            h = torch.relu(z)
    return margin


def _check(got, ref, what):
    """max|g - g_ref| <= TOL max|g_ref| for every tensor; returns the worst relative error."""
    worst = 0.0
    for k, r in ref.items():
        gs, rs = (got[k], r) if isinstance(r, list) else ([got[k]], [r])
        for i, (g, rr) in enumerate(zip(gs, rs)):
            name = "%s %s%s" % (what, k, "[%d]" % i if isinstance(r, list) else "")
            assert g is not None and g.shape == rr.shape, name
            assert bool(torch.isfinite(g).all()), name + ": not finite"
            if rr.numel() == 0:
                continue
            scale = float(rr.abs().max())
            err = float((g.double() - rr).abs().max())
            assert err <= TOL * scale, "%s: max error %.3e, %.2e of max|ref| %.3e" % (name, err, err / max(scale, 1e-300),
                                                                                    scale)
            worst = max(worst, err / scale if scale > 0 else 0.0)
    return worst


# ---------------------------------------------------------------------------------------------
# operator level, against float64
# ---------------------------------------------------------------------------------------------

@pytest.mark.parametrize("N", _sizes())
@pytest.mark.parametrize("kind", ["fg", "bg"])
@pytest.mark.parametrize("weights", WEIGHTS)
def test_implicit_backward(scenes, weights, kind, N):
    c = scenes[weights]
    f, cond = c[kind], c[kind + "_cond"]
    sd = c["sc"]["persons"][0]["implicit"] if kind == "fg" else c["sc"]["bg_implicit"]
    x = _inputs(N, 3, 10 + N) if kind == "fg" else torch.cat([_inputs(N, 3, 10 + N), _inputs(N, 1, 11, 0, 1 / 3)], 1)
    d_sdf, d_feat = _randn((N,), 20 + N), _randn((N, 256), 30 + N)
    f.set_cond(cond)
    got = f.implicit_backward(x, d_sdf, d_feat)
    ref = _ref_implicit(sd, x, cond, 6 if kind == "fg" else 10, d_sdf, d_feat)
    worst = _check(got, ref, "%s/%s/N=%d" % (weights, kind, N))
    print("\n[%s/%s N=%d] implicit backward worst relative error %.2e" % (weights, kind, N, worst))


@pytest.mark.parametrize("which", ["sdf", "feat"])
@pytest.mark.parametrize("seed", [1, 2])
@pytest.mark.parametrize("weights", WEIGHTS)
def test_implicit_backward_one_upstream(scenes, weights, seed, which):
    """d_sdf only, or d_feat only: the other is passed as NULL."""
    c = scenes[weights]
    N = 3 * 128 * int(L.call("mp_device_sm_count")) + 77
    x = _inputs(N, 3, 100 + seed)
    d_sdf = _randn((N,), 200 + seed) if which == "sdf" else None
    d_feat = _randn((N, 256), 300 + seed) if which == "feat" else None
    c["fg"].set_cond(c["fg_cond"])
    got = c["fg"].implicit_backward(x, d_sdf, d_feat)
    ref = _ref_implicit(c["sc"]["persons"][0]["implicit"], x, c["fg_cond"], 6, d_sdf, d_feat)
    _check(got, ref, "%s/%s-only/seed %d" % (weights, which, seed))


@pytest.mark.parametrize("N", _sizes())
@pytest.mark.parametrize("weights", WEIGHTS)
def test_render_backward(scenes, weights, N):
    c = scenes[weights]
    f, bp = c["fg"], c["fg_cond"]
    pts = _inputs(N, 3, 40 + N)
    nrm = torch.nn.functional.normalize(_randn((N, 3), 50 + N), dim=1).contiguous()
    feat = _randn((N, 256), 60 + N) * 0.5
    sd = c["sc"]["persons"][0]["render"]
    # points where a ReLU sits at its kink get no upstream gradient, on both sides
    keep = _relu_margin(sd, pts, nrm, feat, bp) >= KINK
    assert int((~keep).sum()) <= 2 + N // 20, "%d of %d points at a ReLU kink" % (int((~keep).sum()), N)
    d_rgb = (_randn((N, 3), 70 + N) * keep[:, None]).contiguous()
    f.set_cond(bp)
    got = f.render_backward(pts, nrm, feat, d_rgb)
    ref = _ref_render(sd, pts, nrm, feat, bp, d_rgb)
    worst = _check(got, ref, "%s/render/N=%d" % (weights, N))
    print("\n[%s N=%d] render backward worst relative error %.2e (%d points at a ReLU kink)" % (
        weights, N, worst, int((~keep).sum())))


def _flat(r):
    out = []
    for v in r.values():
        out += v if isinstance(v, list) else [v]
    return out


@pytest.mark.parametrize("kind", ["fg", "bg", "render"])
def test_upstream_scale_is_exact(scenes, kind):
    """A VJP is linear in its upstream gradient: with the upstream multiplied by 2^k (k = -20, 12), every output is
    exactly 2^k times the unscaled one (the operands are scaled to fp16's range by powers of two, which is exact), and
    meets the gate against float64 at that scale.  N spans two chunks, whose operand scales differ."""
    c = scenes["trained"]
    N = 3 * 128 * int(L.call("mp_device_sm_count")) + 77
    if kind == "render":
        f, cond, sd = c["fg"], c["fg_cond"], c["sc"]["persons"][0]["render"]
        pts, feat = _inputs(N, 3, 40), _randn((N, 256), 41) * 0.5
        nrm = torch.nn.functional.normalize(_randn((N, 3), 42), dim=1).contiguous()
        keep = _relu_margin(sd, pts, nrm, feat, cond) >= KINK
        up = [(_randn((N, 3), 43) * keep[:, None]).contiguous()]
        run = lambda u: f.render_backward(pts, nrm, feat, u[0])                      # noqa: E731
        ref = lambda u: _ref_render(sd, pts, nrm, feat, cond, u[0])                  # noqa: E731
    else:
        f, cond = c[kind], c[kind + "_cond"]
        sd = c["sc"]["persons"][0]["implicit"] if kind == "fg" else c["sc"]["bg_implicit"]
        x = _inputs(N, 3, 44) if kind == "fg" else torch.cat([_inputs(N, 3, 44), _inputs(N, 1, 45, 0, 1 / 3)], 1)
        up = [_randn((N,), 46), _randn((N, 256), 47)]
        run = lambda u: f.implicit_backward(x, u[0], u[1])                           # noqa: E731
        ref = lambda u: _ref_implicit(sd, x, cond, 6 if kind == "fg" else 10, u[0], u[1])   # noqa: E731
    f.set_cond(cond)
    base = _flat(run(up))
    for k in (-20, 12):
        scaled = [u * 2.0 ** k for u in up]
        got = run(scaled)
        bad = [i for i, (a, b) in enumerate(zip(_flat(got), base)) if not torch.equal(a, b * 2.0 ** k)]
        assert not bad, "%s: outputs %s are not exactly 2^%d times the unscaled ones" % (kind, bad, k)
        _check(got, ref(scaled), "%s upstream x 2^%d" % (kind, k))


# ---------------------------------------------------------------------------------------------
# through the mirror modules' autograd
# ---------------------------------------------------------------------------------------------

def _module(cls, opt, sd):
    m = cls(S.MODEL_OPT[opt])
    m.load_state_dict(sd, strict=True)
    return m.cuda()


def _wn_leaves(sd):
    return {k: v.double().cuda().requires_grad_(True) for k, v in sd.items()}


@pytest.mark.parametrize("kind", ["fg", "bg"])
@pytest.mark.parametrize("weights", WEIGHTS)
def test_implicit_net_autograd(scenes, weights, kind):
    c = scenes[weights]
    sc = c["sc"]
    sd, opt, key = ((sc["persons"][0]["implicit"], "implicit_network", "smpl") if kind == "fg" else
                    (sc["bg_implicit"], "bg_implicit_network", "frame"))
    net = _module(networks.ImplicitNet, opt, sd)
    N = 1000
    x = _inputs(N, 3 if kind == "fg" else 4, 5).requires_grad_(True)
    cond = c[kind + "_cond"].cuda().requires_grad_(True)
    w = _randn((1, N, 257), 6)
    y = net(x, {key: cond})
    names = [n for n, _ in net.named_parameters()]
    g = torch.autograd.grad((y * w).sum(), [x, cond] + list(net.parameters()))
    leaves = _wn_leaves(sd)
    x64, c64 = x.detach().double().requires_grad_(True), cond.detach().double().requires_grad_(True)
    y64 = port.implicit_forward(leaves, x64, c64, 6 if kind == "fg" else 10, weight_norm=(kind == "fg"))
    g64 = torch.autograd.grad((y64 * w[0].double()).sum(), [x64, c64] + [leaves[n] for n in names])
    _check(dict(zip(["x", "cond"] + names, g)), dict(zip(["x", "cond"] + names, g64)), "%s/%s mirror" % (weights, kind))
    y2 = net(x, {key: cond})
    with pytest.raises(NotImplementedError, match="second-order"):
        torch.autograd.grad((y2 * w).sum(), x, create_graph=True)


@pytest.mark.parametrize("weights", WEIGHTS)
def test_rendering_net_autograd(scenes, weights):
    c = scenes[weights]
    sd = c["sc"]["persons"][0]["render"]
    net = _module(networks.RenderingNet, "rendering_network", sd)
    N = 1000
    pts = _inputs(N, 3, 7).requires_grad_(True)
    nrm = torch.nn.functional.normalize(_randn((N, 3), 8), dim=1).detach().requires_grad_(True)
    feat = (_randn((N, 256), 9) * 0.5).requires_grad_(True)
    bp = c["fg_cond"].cuda().requires_grad_(True)
    w = _randn((N, 3), 10)
    rgb = net(pts, nrm, None, bp, feat)
    names = [n for n, _ in net.named_parameters()]
    g = torch.autograd.grad((rgb * w).sum(), [pts, nrm, feat, bp] + list(net.parameters()))
    leaves = _wn_leaves(sd)
    ins = [t.detach().double().requires_grad_(True) for t in (pts, nrm, feat, bp)]
    rgb64 = port.rendering_forward(leaves, "pose_no_view", ins[0], ins[1], None, ins[3], ins[2])
    g64 = torch.autograd.grad((rgb64 * w.double()).sum(), ins + [leaves[n] for n in names])
    keys = ["points", "normals", "feature_vectors", "body_pose"] + names
    _check(dict(zip(keys, g)), dict(zip(keys, g64)), "%s/render mirror" % weights)
    rgb2 = net(pts, nrm, None, bp, feat)
    with pytest.raises(NotImplementedError, match="second-order"):
        torch.autograd.grad((rgb2 * w).sum(), pts, create_graph=True)


@pytest.mark.parametrize("weights", WEIGHTS)
def test_mean_loss_through_the_mirror(scenes, weights):
    """A loss averaged over points, the usual case: per-point upstream gradients of about 1 / (N x 257) and 1 / (N x 3)."""
    c = scenes[weights]
    p = c["sc"]["persons"][0]
    N = 1000
    net = _module(networks.ImplicitNet, "implicit_network", p["implicit"])
    x = _inputs(N, 3, 15).requires_grad_(True)
    cond = c["fg_cond"].cuda().requires_grad_(True)
    names = [n for n, _ in net.named_parameters()]
    g = torch.autograd.grad(net(x, {"smpl": cond}).mean(), [x, cond] + list(net.parameters()))
    leaves = _wn_leaves(p["implicit"])
    x64, c64 = x.detach().double().requires_grad_(True), cond.detach().double().requires_grad_(True)
    g64 = torch.autograd.grad(port.implicit_forward(leaves, x64, c64, 6).mean(), [x64, c64] + [leaves[n] for n in names])
    _check(dict(zip(["x", "cond"] + names, g)), dict(zip(["x", "cond"] + names, g64)), "%s implicit .mean()" % weights)
    rn = _module(networks.RenderingNet, "rendering_network", p["render"])
    nrm = torch.nn.functional.normalize(_randn((N, 3), 16), dim=1).contiguous()
    feat = _randn((N, 256), 17) * 0.5
    keep = _relu_margin(p["render"], x.detach(), nrm, feat, c["fg_cond"]) >= KINK
    pts, nrm, feat = (t.detach()[keep].contiguous().requires_grad_(True) for t in (x, nrm, feat))
    bp = c["fg_cond"].cuda().requires_grad_(True)
    names = [n for n, _ in rn.named_parameters()]
    g = torch.autograd.grad(rn(pts, nrm, None, bp, feat).mean(), [pts, nrm, feat, bp] + list(rn.parameters()))
    leaves = _wn_leaves(p["render"])
    ins = [t.detach().double().requires_grad_(True) for t in (pts, nrm, feat, bp)]
    g64 = torch.autograd.grad(port.rendering_forward(leaves, "pose_no_view", ins[0], ins[1], None, ins[3], ins[2]).mean(),
                              ins + [leaves[n] for n in names])
    keys = ["points", "normals", "feature_vectors", "body_pose"] + names
    _check(dict(zip(keys, g)), dict(zip(keys, g64)), "%s render .mean()" % weights)


def test_no_grad_modules_run_the_plain_forward(scenes):
    """With no gradient wanted the modules issue exactly the plain forward's launches and return its values."""
    c = scenes["trained"]
    p = c["sc"]["persons"][0]
    net = _module(networks.ImplicitNet, "implicit_network", p["implicit"])
    rn = _module(networks.RenderingNet, "rendering_network", p["render"])
    x = _inputs(777, 3, 3)
    cond = p["cond"].cuda()
    nrm = torch.nn.functional.normalize(_randn((777, 3), 4), dim=1).contiguous()
    f, fr = net.field(x.device), rn.field(x.device)
    torch.cuda.synchronize()
    n0 = L.call("mp_launch_count", 0)
    f.set_cond(cond)
    sdf, feat = f.implicit_forward(x)
    n1 = L.call("mp_launch_count", 0)
    fr.set_cond(cond)
    rgb = fr.render_forward(x, nrm, feat)
    n2 = L.call("mp_launch_count", 0)
    with torch.no_grad():
        y = net(x, {"smpl": cond})
        n3 = L.call("mp_launch_count", 0)
        rgb2 = rn(x, nrm, None, cond, y[0, :, 1:].contiguous())
    n4 = L.call("mp_launch_count", 0)
    assert (n3 - n2, n4 - n3) == (n1 - n0, n2 - n1)
    assert same(y[0, :, 0], sdf) and same(y[0, :, 1:].contiguous(), feat) and same(rgb2, rgb)
    for prm in list(net.parameters()) + list(rn.parameters()):     # grad mode on, but nothing requires grad
        prm.requires_grad_(False)
    y3 = net(x, {"smpl": cond})
    assert L.call("mp_launch_count", 0) - n4 == n1 - n0
    assert same(y3, y) and y3.grad_fn is None


# ---------------------------------------------------------------------------------------------
# determinism, workspace, refusals
# ---------------------------------------------------------------------------------------------

def _abi_implicit(f, x, d_sdf, d_feat, ws, nbytes=None):
    N = x.shape[0]
    d_x = torch.full((N, f.d_in), float("nan"), device="cuda")
    d_cond = torch.full((f.cond_dim,), float("nan"), device="cuda")
    g = L.LinearGrads()
    dW = [torch.full((o, i), float("nan"), device="cuda") for o, i in f.imp_shapes]
    db = [torch.full((o,), float("nan"), device="cuda") for o, _ in f.imp_shapes]
    for l in range(9):
        g.d_weight[l], g.d_bias[l] = L.ptr(dW[l]), L.ptr(db[l])
    L.call("mp_implicit_backward", f.handle, x if N else None, N, d_sdf if N else None, d_feat if N else None,
           d_x if N else None, g, d_cond, ws, ws.numel() if nbytes is None else nbytes)
    torch.cuda.synchronize()
    return [d_x, d_cond] + dW + db


def _abi_render(f, x, nrm, feat, d_rgb, ws):
    N = x.shape[0]
    outs = [torch.full(s, float("nan"), device="cuda") for s in ((N, 3), (N, 3), (N, 256), (8, 69), (8,), (69,))]
    g = L.LinearGrads()
    dW = [torch.full((o, i), float("nan"), device="cuda") for o, i in f.ren_shapes]
    db = [torch.full((o,), float("nan"), device="cuda") for o, _ in f.ren_shapes]
    for l in range(len(dW)):
        g.d_weight[l], g.d_bias[l] = L.ptr(dW[l]), L.ptr(db[l])
    nz = (lambda t: t) if N else (lambda t: None)
    L.call("mp_render_backward", f.handle, nz(x), nz(nrm), nz(feat), N, nz(d_rgb), nz(outs[0]), nz(outs[1]),
           nz(outs[2]), g, outs[3], outs[4], outs[5], ws, ws.numel())
    torch.cuda.synchronize()
    return outs + dW + db


def test_deterministic_and_independent_of_workspace(scenes):
    c = scenes["trained"]
    f = c["fg"]
    f.set_cond(c["fg_cond"])
    N = 40000
    x, d_sdf, d_feat = _inputs(N, 3, 1), _randn((N,), 2), _randn((N, 256), 3)
    nb = L.call("mp_implicit_backward_workspace_bytes", N)
    a = _abi_implicit(f, x, d_sdf, d_feat, L.workspace(nb, "cuda"))
    b = _abi_implicit(f, x, d_sdf, d_feat, L.workspace(nb, "cuda"))
    d = _abi_implicit(f, x, d_sdf, d_feat, dirty_workspace(nb))
    assert all(same(u, v) for u, v in zip(a, b)), "two calls differ"
    assert all(same(u, v) for u, v in zip(a, d)), "a NaN-filled workspace changes the result"
    pts, feat = _inputs(N, 3, 4), _randn((N, 256), 5)
    nrm = torch.nn.functional.normalize(_randn((N, 3), 6), dim=1).contiguous()
    d_rgb = _randn((N, 3), 7)
    nr = L.call("mp_render_backward_workspace_bytes", N)
    a = _abi_render(f, pts, nrm, feat, d_rgb, L.workspace(nr, "cuda"))
    b = _abi_render(f, pts, nrm, feat, d_rgb, L.workspace(nr, "cuda"))
    d = _abi_render(f, pts, nrm, feat, d_rgb, dirty_workspace(nr))
    assert all(same(u, v) for u, v in zip(a, b)), "two render calls differ"
    assert all(same(u, v) for u, v in zip(a, d)), "a NaN-filled workspace changes the render result"
    assert all(bool(torch.isfinite(t).all()) for t in a + d)


def test_workspace_refusals_before_any_launch(scenes):
    c = scenes["trained"]
    f, bg = c["fg"], c["bg"]
    f.set_cond(c["fg_cond"])
    N = 300
    x, d_sdf, d_feat = _inputs(N, 3, 1), _randn((N,), 2), _randn((N, 256), 3)
    nb = L.call("mp_implicit_backward_workspace_bytes", N)
    exact = _abi_implicit(f, x, d_sdf, d_feat, L.workspace(nb, "cuda"))
    assert all(bool(torch.isfinite(t).all()) for t in exact)
    big = L.workspace(nb + 256, "cuda")
    for ws, n, msg in ((big, nb - 1, "too small"), (big[1:], nb, "not 256-byte aligned")):
        torch.cuda.synchronize()
        n0 = L.call("mp_launch_count", 0)
        with pytest.raises(L.MpError, match=msg):
            _abi_implicit(f, x, d_sdf, d_feat, ws, nbytes=n)
        assert L.call("mp_launch_count", 0) == n0
    pts, nrm, feat, d_rgb = _inputs(N, 3, 4), _inputs(N, 3, 5), _randn((N, 256), 6), _randn((N, 3), 7)
    nr = L.call("mp_render_backward_workspace_bytes", N)
    n0 = L.call("mp_launch_count", 0)
    with pytest.raises(L.MpError, match="too small"):
        L.call("mp_render_backward", f.handle, pts, nrm, feat, N, d_rgb, None, None, None, L.LinearGrads(), None, None,
               None, L.workspace(nr, "cuda"), nr - 1)
    with pytest.raises(L.MpError, match="not a foreground"):
        _abi_render(bg, pts, nrm, feat, d_rgb, L.workspace(nr, "cuda"))
    assert L.call("mp_launch_count", 0) == n0


def test_zero_points(scenes):
    c = scenes["trained"]
    for f in (c["fg"], c["bg"]):
        assert L.call("mp_implicit_backward_workspace_bytes", 0) == 0
        out = _abi_implicit(f, torch.zeros(0, f.d_in, device="cuda"), None, None, None, nbytes=0)
        assert all(bool((t == 0).all()) for t in out[1:])
    assert L.call("mp_render_backward_workspace_bytes", 0) == 0
    z = torch.zeros(0, 3, device="cuda")
    out = _abi_render(c["fg"], z, z, torch.zeros(0, 256, device="cuda"), z, L.workspace(0, "cuda"))
    assert all(bool((t == 0).all()) for t in out[3:])
