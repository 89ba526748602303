"""GPU: the networks' first-order backward (mp_implicit_backward, mp_render_backward and the mirror modules' autograd
through them) element by element against float64, at chunk, scale and partial-output edges and across optimizer steps.

Every gradient keeps test_gpu_network_grad.py's per-tensor gate (max|g - g_ref| <= 1e-4 max|g_ref|) and must also meet
a per-element one, |g - g_ref| <= C 2^-24 M, with M the float64 magnitude backward of tests/_network_grad_ref.py.  The
per-tensor gate alone lets a row or column whose values lie below 1e-4 of the tensor's largest be wholly wrong (dW8's
sdf row, lin0's cond columns, d_cond, the lin_pose chain).  C is 4x the worst measured per output kind on one H100
(printed as MEASURED).  Points whose colour-net pre-activation lies within 1e-6 of a ReLU kink get no upstream
gradient (test_gpu_network_grad.py)."""
import pytest
import torch

from multiply_b200 import engine, scene as S, _lib as L
from multiply_b200.model import networks

import _network_grad_ref as R
from _abi import padded, same, sentinel, take

pytestmark = pytest.mark.gpu

TOL = 1e-4
WEIGHTS = ["geometric", "trained"]
CHUNK = R.CHUNK
# 4x the worst measured per output kind on one H100 80GB HBM3 at a 700 W power limit.  Implicit: 59.6 (d_bias), 58.0
# (d_weight), both at N = 1 where nothing averages; 7.08 (d_cond), 4.21 (d_x).  The geometric-init foreground's d_x has its
# own, 1.1e3: its lin0 reads x alone (the embedding's other weights are 0), and at points where lin0's G cancels the
# error G carries from the layers above it dominates G's own terms (float32 autograd shows the same at 30).  Render:
# 21.8 (d_weight), 19.4 (d_bias), 5.01 (d_feat), 4.30 (d_points), 4.13 (d_normals), 1.19 / 1.17 (lin_pose weight /
# bias), 0.625 (d_body_pose).
C = {"implicit": dict(d_x=17.0, d_cond=29.0, d_weight=232.0, d_bias=240.0),
     "render": dict(d_points=17.2, d_normals=16.5, d_feat=20.0, d_weight=87.0, d_bias=78.0, d_body_pose=2.5,
                    d_lin_pose_weight=4.8, d_lin_pose_bias=4.7)}
C["implicit geometric fg"] = dict(C["implicit"], d_x=4400.0)
MEASURED = {}


@pytest.fixture(scope="module", autouse=True)
def _print_measured():
    yield
    for k in sorted(MEASURED):
        print("MEASURED %s C=%.3g" % (k, MEASURED[k]))


def _tiles():
    return 128 * int(L.call("mp_device_sm_count"))


def _sizes():
    return [1, 127, 128, 129, 3 * _tiles() + 77, CHUNK - 1, CHUNK, CHUNK + 1, 2 * CHUNK, 2 * CHUNK + 1]


@pytest.fixture(scope="module")
def scenes():
    engine.set_engine("tc")
    out = {}
    for w in WEIGHTS:
        sc = S.make_scene(P=1, S=16, seed=42, weights=w)
        p = sc["persons"][0]
        out[w] = dict(weights=w, sc=sc, p=p, fg=engine.Field(p["implicit"], p["render"]),
                      bg=engine.Field(sc["bg_implicit"], sc["bg_render"], background=True))
    return out


def _gen(seed):
    return torch.Generator().manual_seed(seed)


def _fg_points(person, n, seed):
    """Canonical points: interleaved, half over the [-1, 1]^3 box and half within ~0.05 of the body; every eighth point
    is replaced by one with |x| up to 3 (outside the box, where the embedding's high frequencies are far from 0)."""
    g = _gen(seed)
    vc = torch.as_tensor(person["verts_c"]).float()
    box = (torch.rand(n, 3, generator=g) - 0.5) * 2.0
    near = vc[torch.randint(0, vc.shape[0], (n,), generator=g)] + 0.05 * torch.randn(n, 3, generator=g)
    far = (torch.rand(n, 3, generator=g) - 0.5) * 6.0
    x = torch.where((torch.rand(n, generator=g) < 0.5)[:, None], near, box)
    x[::8] = far[::8]
    return x.contiguous().cuda()


def _bg_points(n, seed):
    """As the background sampler makes them: a unit direction and 1/r in (0, 1/3]."""
    g = _gen(seed)
    d = torch.nn.functional.normalize(torch.randn(n, 3, generator=g), dim=1)
    inv_r = (1.0 - torch.rand(n, 1, generator=g)) / 3.0
    return torch.cat([d, inv_r], 1).contiguous().cuda()


def _randn(shape, seed):
    return torch.randn(*shape, generator=_gen(seed)).cuda()


class Imp:
    """One ImplicitNet case: the field, its state dict, cond and multires, points and upstreams."""

    def __init__(self, c, kind, N, seed, d_sdf=None, d_feat=None):
        self.kind, self.f = kind, c[kind]
        self.net = "implicit geometric fg" if (c["weights"], kind) == ("geometric", "fg") else "implicit"
        self.sd = c["p"]["implicit"] if kind == "fg" else c["sc"]["bg_implicit"]
        self.cond = c["p"]["cond"] if kind == "fg" else c["sc"]["frame_code"]
        self.L = 6 if kind == "fg" else 10
        self.x = _fg_points(c["p"], N, seed) if kind == "fg" else _bg_points(N, seed)
        self.d_sdf = _randn((N,), seed + 1) if d_sdf is None else d_sdf
        self.d_feat = _randn((N, 256), seed + 2) if d_feat is None else d_feat

    def run(self, **want):
        self.f.set_cond(self.cond)
        return self.f.implicit_backward(self.x, self.d_sdf, self.d_feat, **want)

    def ref(self):
        return R.ref_implicit(self.sd, self.x, self.cond, self.L, self.d_sdf, self.d_feat)

    def mag(self):
        return R.implicit_magnitude(self.sd, self.x, self.cond, self.L, self.d_sdf, self.d_feat)


class Ren:
    """One RenderingNet case; points at a ReLU kink get no upstream."""

    def __init__(self, c, N, seed, scale=None):
        self.f, self.sd, self.cond = c["fg"], c["p"]["render"], c["p"]["cond"]
        self.pts = _fg_points(c["p"], N, seed)
        self.nrm = torch.nn.functional.normalize(_randn((N, 3), seed + 1), dim=1).contiguous()
        self.feat = _randn((N, 256), seed + 2) * 0.5
        keep = R.relu_margin(self.sd, self.pts, self.nrm, self.feat, self.cond) >= R.KINK
        assert int((~keep).sum()) <= 2 + N // 20
        up = _randn((N, 3), seed + 3) * keep[:, None]
        self.d_rgb = (up if scale is None else up * scale[:, None]).contiguous()

    def run(self, **want):
        self.f.set_cond(self.cond)
        return self.f.render_backward(self.pts, self.nrm, self.feat, self.d_rgb, **want)

    def ref(self):
        return R.ref_render(self.sd, self.pts, self.nrm, self.feat, self.cond, self.d_rgb)

    def mag(self):
        return R.render_magnitude(self.sd, self.pts, self.nrm, self.feat, self.cond, self.d_rgb)


def _tensor_gate(got, ref, what):
    for name, _, g in R.items(got):
        if g is None:
            continue
        r = dict((n, t) for n, _, t in R.items(ref))[name]
        assert g.shape == r.shape and bool(torch.isfinite(g).all()), "%s %s" % (what, name)
        if r.numel():
            err, scale = float((g.double() - r).abs().max()), float(r.abs().max())
            assert err <= TOL * scale, "%s %s: max error %.3e of max|ref| %.3e" % (what, name, err, scale)


def _element_gate(net, got, ref, mag, what):
    worst = R.element_c(got, ref, mag)
    print("\n[%s] C %s" % (what, " ".join("%s=%.3g" % kv for kv in sorted(worst.items()))))
    for k, c in worst.items():
        MEASURED["%s %s" % (net, k)] = max(MEASURED.get("%s %s" % (net, k), 0.0), c)
        assert c <= C[net][k], "%s %s: an element needs C = %.3g > %g" % (what, k, c, C[net][k])
    return worst


def _gate(net, got, ref, mag, what):
    _tensor_gate(got, ref, what)
    return _element_gate(net, got, ref, mag, what)


def _check(case, what):
    net = "render" if isinstance(case, Ren) else case.net
    got = case.run()
    return got, _gate(net, got, case.ref(), case.mag(), what)


# ---------------------------------------------------------------------------------------------
# sizes, upstream imbalance, chunk scales, zero and sparse upstreams
# ---------------------------------------------------------------------------------------------

@pytest.mark.parametrize("N", _sizes())
@pytest.mark.parametrize("kind", ["fg", "bg"])
@pytest.mark.parametrize("weights", WEIGHTS)
def test_implicit_sizes(scenes, weights, kind, N):
    _check(Imp(scenes[weights], kind, N, 10 + N), "%s/%s N=%d" % (weights, kind, N))


@pytest.mark.parametrize("N", _sizes())
@pytest.mark.parametrize("weights", WEIGHTS)
def test_render_sizes(scenes, weights, N):
    _check(Ren(scenes[weights], N, 20 + N), "%s/render N=%d" % (weights, N))


@pytest.mark.parametrize("k", [20, -20])
@pytest.mark.parametrize("kind", ["fg", "bg"])
@pytest.mark.parametrize("weights", WEIGHTS)
def test_upstream_imbalance(scenes, weights, kind, k):
    """d_sdf and d_feat come from different loss terms in training: d_sdf at 2^k times d_feat's scale."""
    N = 3 * _tiles() + 77
    _check(Imp(scenes[weights], kind, N, 30, d_sdf=_randn((N,), 31) * 2.0 ** k),
           "%s/%s d_sdf x 2^%d" % (weights, kind, k))


def _rows(d, lo, hi):
    """The per-point outputs of a result dict, rows [lo, hi)."""
    return {k: v[lo:hi] for k, v in d.items() if k in ("d_x", "d_points", "d_normals", "d_feat") and v is not None}


@pytest.mark.parametrize("small", [0, 1])
@pytest.mark.parametrize("kind", ["fg", "bg", "render"])
def test_chunk_scales(scenes, kind, small):
    """Two chunks whose upstreams differ by 2^24: chunk ``small``'s is scaled by 2^-24.  Each chunk's layer inputs and G
    are scaled by their own maxima, so each chunk's points meet the gate on their own, and so do the parameters."""
    c = scenes["trained"]
    N = 2 * CHUNK
    s = torch.ones(N, device="cuda")
    s[small * CHUNK:(small + 1) * CHUNK] = 2.0 ** -24
    if kind == "render":
        case, net = Ren(c, N, 40, scale=s), "render"
    else:
        case, net = Imp(c, kind, N, 40), "implicit"
        case.d_sdf, case.d_feat = case.d_sdf * s, (case.d_feat * s[:, None]).contiguous()
    got = case.run()
    ref, mag = case.ref(), case.mag()
    _tensor_gate({k: v for k, v in got.items() if k not in ("d_x", "d_points", "d_normals", "d_feat")}, ref, kind)
    for ch in range(2):
        lo, hi = ch * CHUNK, (ch + 1) * CHUNK
        _tensor_gate(_rows(got, lo, hi), _rows(ref, lo, hi), "%s chunk %d" % (kind, ch))
        _element_gate(net, _rows(got, lo, hi), _rows(ref, lo, hi), _rows(mag, lo, hi), "%s chunk %d" % (kind, ch))
    _element_gate(net, got, ref, mag, kind)


@pytest.mark.parametrize("kind", ["fg", "bg", "render"])
def test_zero_upstream(scenes, kind):
    """An all-zero upstream over two chunks: every output is exactly 0."""
    c = scenes["trained"]
    N = CHUNK + 1
    if kind == "render":
        case = Ren(c, N, 50, scale=torch.zeros(N, device="cuda"))
    else:
        case = Imp(c, kind, N, 50, d_sdf=torch.zeros(N, device="cuda"), d_feat=torch.zeros(N, 256, device="cuda"))
    for name, _, t in R.items(case.run()):
        assert bool((t == 0).all()), "%s: %s is not all zero" % (kind, name)


@pytest.mark.parametrize("kind", ["fg", "bg", "render"])
def test_sparse_upstream(scenes, kind):
    """1 % of the points carry an upstream, as the sampler's samples do: the others' input gradients are exactly 0, and
    every output meets the gate."""
    c = scenes["trained"]
    N = CHUNK + 1
    live = (torch.rand(N, generator=_gen(61)) < 0.01).cuda()
    if kind == "render":
        case, net = Ren(c, N, 60, scale=live.float()), "render"
    else:
        case, net = Imp(c, kind, N, 60), "implicit"
        case.d_sdf, case.d_feat = case.d_sdf * live, (case.d_feat * live[:, None]).contiguous()
    got = case.run()
    for k, v in _rows(got, 0, N).items():
        assert bool((v[~live] == 0).all()), "%s: %s is not 0 at a point without upstream" % (kind, k)
    _gate(net, got, case.ref(), case.mag(), "%s sparse" % kind)


# ---------------------------------------------------------------------------------------------
# NULL outputs at the C ABI
# ---------------------------------------------------------------------------------------------

def _imp_shapes(f, N):
    s = {"d_x": (N, f.d_in), "d_cond": (f.cond_dim,)}
    for l, (o, i) in enumerate(f.imp_shapes):
        s["d_weight[%d]" % l], s["d_bias[%d]" % l] = (o, i), (o,)
    return s


def _ren_shapes(f, N):
    s = {"d_points": (N, 3), "d_normals": (N, 3), "d_feat": (N, 256), "d_lin_pose_weight": (8, 69),
         "d_lin_pose_bias": (8,), "d_body_pose": (69,)}
    for l, (o, i) in enumerate(f.ren_shapes):
        s["d_weight[%d]" % l], s["d_bias[%d]" % l] = (o, i), (o,)
    return s


def _abi_call(case, want):
    """The call with the outputs in ``want`` given (sentinel-padded buffers) and the rest NULL: the outputs written,
    checked for writes past their ends, and the launches it made.  The NULL outputs' buffers stay all sentinel."""
    imp = isinstance(case, Imp)
    f = case.f
    N = (case.x if imp else case.pts).shape[0]
    shapes = _imp_shapes(f, N) if imp else _ren_shapes(f, N)
    bufs = {k: padded(s) for k, s in shapes.items()}
    given = {k: (bufs[k] if k in want else None) for k in shapes}
    g = L.LinearGrads()
    for l in range(len(f.imp_shapes if imp else f.ren_shapes)):
        g.d_weight[l], g.d_bias[l] = L.ptr(given["d_weight[%d]" % l]), L.ptr(given["d_bias[%d]" % l])
    f.set_cond(case.cond)
    if imp:
        nb = L.call("mp_implicit_backward_workspace_bytes", N)
        ws = L.workspace(nb, "cuda")
        torch.cuda.synchronize()
        n0 = L.call("mp_launch_count", 0)
        L.call("mp_implicit_backward", f.handle, case.x, N, case.d_sdf, case.d_feat, given["d_x"], g, given["d_cond"],
               ws, nb)
    else:
        nb = L.call("mp_render_backward_workspace_bytes", N)
        ws = L.workspace(nb, "cuda")
        torch.cuda.synchronize()
        n0 = L.call("mp_launch_count", 0)
        L.call("mp_render_backward", f.handle, case.pts, case.nrm, case.feat, N, case.d_rgb, given["d_points"],
               given["d_normals"], given["d_feat"], g, given["d_lin_pose_weight"], given["d_lin_pose_bias"],
               given["d_body_pose"], ws, nb)
    n = L.call("mp_launch_count", 0) - n0
    torch.cuda.synchronize()
    out = {}
    for k, s in shapes.items():
        if k in want:
            out[k] = take(bufs[k], s, k)
        else:
            assert bool((bufs[k] == sentinel(torch.float32)).all()), "%s written though NULL" % k
    return out, n


def _params(net_shapes):
    return {"d_weight[%d]" % l for l in range(len(net_shapes))} | {"d_bias[%d]" % l for l in range(len(net_shapes))}


IMP_SUBSETS = {
    "x": lambda p: {"d_x"}, "cond": lambda p: {"d_cond"}, "w0": lambda p: {"d_weight[0]"},
    "b0": lambda p: {"d_bias[0]"}, "params": lambda p: p, "x+params": lambda p: p | {"d_x"},
    "x+cond": lambda p: {"d_x", "d_cond"}, "params+cond": lambda p: p | {"d_cond"}}
REN_SUBSETS = {
    "inputs": lambda p: {"d_points", "d_normals", "d_feat"}, "points": lambda p: {"d_points"},
    "feat": lambda p: {"d_feat"}, "body_pose": lambda p: {"d_body_pose"},
    "lin_pose": lambda p: {"d_lin_pose_weight", "d_lin_pose_bias"}, "b0": lambda p: {"d_bias[0]"},
    "params": lambda p: p, "inputs+params": lambda p: p | {"d_points", "d_normals", "d_feat"},
    "inputs+pose": lambda p: {"d_points", "d_normals", "d_feat", "d_body_pose", "d_lin_pose_weight",
                              "d_lin_pose_bias"},
    "params+pose": lambda p: p | {"d_body_pose", "d_lin_pose_weight", "d_lin_pose_bias"}}


@pytest.fixture(scope="module")
def full_calls(scenes):
    """Every output of both calls at N = 32769 (two chunks): (case, outputs, launches), keyed fg / bg / render."""
    c = scenes["trained"]
    out = {}
    for kind in ("fg", "bg", "render"):
        case = Ren(c, CHUNK + 1, 70) if kind == "render" else Imp(c, kind, CHUNK + 1, 70)
        f = case.f
        names = set(_imp_shapes(f, 1) if kind != "render" else _ren_shapes(f, 1))
        out[kind] = (case,) + _abi_call(case, names)
    return out


def _check_subset(full_calls, kind, want):
    case, full, n_full = full_calls[kind]
    got, n = _abi_call(case, want)
    assert set(got) == want
    for k in want:
        assert same(got[k], full[k]), "%s: %s differs from the all-outputs call's" % (kind, k)
    # the launches the omitted products save, per chunk (two here): a weight-gradient GEMM and its reduction per layer;
    # the first layer's input-gradient GEMM and the input's backward (the embedding's, or the colour input's)
    layers = len(case.f.imp_shapes if kind != "render" else case.f.ren_shapes)
    saved = 0
    if not any(k.startswith("d_weight") for k in want):
        saved += 2 * layers * 2
    if not want & {"d_x", "d_points", "d_normals", "d_feat"}:
        saved += 2 * 2
    assert n <= n_full - saved, "%s: %d launches with outputs %s, %d with all; %d should be skipped" % (
        kind, n, sorted(want), n_full, saved)
    return got


@pytest.mark.parametrize("subset", list(IMP_SUBSETS))
@pytest.mark.parametrize("kind", ["fg", "bg"])
def test_implicit_null_outputs(full_calls, kind, subset):
    """Each subset of outputs the engine can request (want_x / want_params / want_cond) and single outputs: what is
    written equals the all-outputs call bit for bit, NULL outputs are untouched and their products are not launched."""
    f = full_calls[kind][0].f
    _check_subset(full_calls, kind, IMP_SUBSETS[subset](_params(f.imp_shapes)))


@pytest.mark.parametrize("subset", list(REN_SUBSETS))
def test_render_null_outputs(full_calls, subset):
    f = full_calls["render"][0].f
    _check_subset(full_calls, "render", REN_SUBSETS[subset](_params(f.ren_shapes)))


# ---------------------------------------------------------------------------------------------
# through the mirror modules
# ---------------------------------------------------------------------------------------------

def _module(cls, opt, sd):
    m = cls(S.MODEL_OPT[opt])
    m.load_state_dict(sd, strict=True)
    return m.cuda()


def _imp_module(c, kind):
    return (_module(networks.ImplicitNet, "implicit_network", c["p"]["implicit"]) if kind == "fg" else
            _module(networks.ImplicitNet, "bg_implicit_network", c["sc"]["bg_implicit"]))


def _module_refs(net, inputs, upstream):
    """float64 gradients and their M for a mirror module at its current parameters: dict name -> (ref, M) over the
    inputs (x, cond / points, normals, body_pose, feature_vectors) and the named parameters."""
    sd = {k: v.detach() for k, v in net.state_dict().items()}
    out = {}
    if isinstance(net, networks.ImplicitNet):
        x, cond = inputs
        L_ = net.multires
        ref = R.ref_implicit(sd, x, cond, L_, upstream[:, 0].contiguous(), upstream[:, 1:].contiguous())
        mag = R.implicit_magnitude(sd, x, cond, L_, upstream[:, 0], upstream[:, 1:])
        out["x"], out["cond"] = (ref["d_x"], mag["d_x"]), (ref["d_cond"].reshape(cond.shape),
                                                           mag["d_cond"].reshape(cond.shape))
        n = 9
    else:
        pts, nrm, bp, feat = inputs
        ref = R.ref_render(sd, pts, nrm, feat, bp, upstream)
        mag = R.render_magnitude(sd, pts, nrm, feat, bp, upstream)
        for k, r in (("points", "d_points"), ("normals", "d_normals"), ("feature_vectors", "d_feat")):
            out[k] = (ref[r], mag[r])
        out["body_pose"] = (ref["d_body_pose"].reshape(bp.shape), mag["d_body_pose"].reshape(bp.shape))
        out["lin_pose.weight"] = (ref["d_lin_pose_weight"], mag["d_lin_pose_weight"])
        out["lin_pose.bias"] = (ref["d_lin_pose_bias"], mag["d_lin_pose_bias"])
        n = 5
    for l in range(n):
        out["lin%d.bias" % l] = (ref["d_bias"][l], mag["d_bias"][l])
        if "lin%d.weight_v" % l in sd:
            v, g = sd["lin%d.weight_v" % l].double(), sd["lin%d.weight_g" % l].double()
            nv = v.norm(dim=1, keepdim=True)
            dW = ref["d_weight"][l]
            dg = (dW * v / nv).sum(1, keepdim=True)
            dv = g / nv * (dW - dg * v / nv)
            mv, mg = R.weight_norm_magnitude(mag["d_weight"][l], v, g)
            out["lin%d.weight_v" % l], out["lin%d.weight_g" % l] = (dv, mv), (dg, mg)
        else:
            out["lin%d.weight" % l] = (ref["d_weight"][l], mag["d_weight"][l])
    return out


def _gate_module(net, got, refs, what):
    """got: name -> gradient (None: not requested) against _module_refs' (ref, M), summed where refs is a list."""
    refs = refs if isinstance(refs, list) else [refs]
    kind = "implicit" if isinstance(net, networks.ImplicitNet) else "render"
    for name, g in got.items():
        r = sum(rs[name][0] for rs in refs)
        m = sum(rs[name][1] for rs in refs)
        _tensor_gate({name: g}, {name: r}, what)
        k = {"x": "d_x", "cond": "d_x", "points": "d_points", "normals": "d_normals", "feature_vectors": "d_feat",
             "body_pose": "d_body_pose", "lin_pose.weight": "d_lin_pose_weight",
             "lin_pose.bias": "d_lin_pose_bias"}.get(name, "d_bias" if name.endswith("bias") else "d_weight")
        if kind == "implicit" and name == "cond":
            k = "d_cond"
        c = R.ratio(g.double() - r, m)
        MEASURED["%s %s" % (kind, k)] = max(MEASURED.get("%s %s" % (kind, k), 0.0), c)
        assert c <= C[kind][k], "%s %s: an element needs C = %.3g > %g" % (what, name, c, C[kind][k])


def _imp_inputs(c, kind, N, seed, cond=None):
    x = _fg_points(c["p"], N, seed) if kind == "fg" else _bg_points(N, seed)
    cond = (c["p"]["cond"] if kind == "fg" else c["sc"]["frame_code"]) if cond is None else cond
    return x, cond.reshape(1, -1).cuda().clone()


def _ren_inputs(c, N, seed, bp=None):
    pts = _fg_points(c["p"], N, seed)
    nrm = torch.nn.functional.normalize(_randn((N, 3), seed + 1), dim=1).contiguous()
    feat = _randn((N, 256), seed + 2) * 0.5
    bp = (c["p"]["cond"] if bp is None else bp).reshape(1, -1).cuda().clone()
    keep = R.relu_margin(c["p"]["render"], pts, nrm, feat, bp) >= R.KINK
    return (pts, nrm, bp, feat), keep


def _imp_forward(net, kind, x, cond):
    return net(x, {"smpl" if kind == "fg" else "frame": cond})[0]


@pytest.mark.parametrize("kind", ["fg", "bg", "render"])
def test_autograd_partial_requests(scenes, kind):
    """Modules where only some tensors require grad (frozen parameters, a detached input, cond or body_pose): every
    gradient is bit-identical to the one the all-requiring run gives, and None where nothing requires it."""
    c = scenes["trained"]
    N = 3000
    if kind == "render":
        net = _module(networks.RenderingNet, "rendering_network", c["p"]["render"])
        ins, keep = _ren_inputs(c, N, 80)
        w = _randn((N, 3), 84) * keep[:, None]
        names_in = ["points", "normals", "body_pose", "feature_vectors"]
        fwd = lambda t: net(t[0], t[1], None, t[2], t[3])                              # noqa: E731
    else:
        net = _imp_module(c, kind)
        ins = _imp_inputs(c, kind, N, 80)
        w = _randn((N, 257), 84)
        names_in = ["x", "cond"]
        fwd = lambda t: _imp_forward(net, kind, t[0], t[1])                          # noqa: E731
    params = dict(net.named_parameters())

    def run(req_in, req_par):
        for n, p in params.items():
            p.requires_grad_(n in req_par)
            p.grad = None
        leaves = [t.detach().clone().requires_grad_(n in req_in) for n, t in zip(names_in, ins)]
        (fwd(leaves) * w).sum().backward()
        got = {n: t.grad for n, t in zip(names_in, leaves)}
        got.update({n: p.grad for n, p in params.items()})
        return got

    full = run(set(names_in), set(params))
    pose = {"lin_pose.weight", "lin_pose.bias"}
    cases = [(set(names_in), set()), (set(), set(params)), ({names_in[0]}, set()), ({names_in[-1]}, set(params)),
             (set(names_in) - {"cond", "body_pose"}, set(params) - pose), ({names_in[0]}, {"lin0.bias"})]
    if kind == "render":
        cases += [({"body_pose"}, set()), (set(), pose), ({"body_pose"}, pose)]
    try:
        for req_in, req_par in cases:
            got = run(req_in, req_par)
            for n, g in got.items():
                if n in req_in or n in req_par:
                    assert g is not None and same(g, full[n]), "%s: %s differs (requested %s)" % (
                        kind, n, sorted(req_in | req_par))
                else:
                    assert g is None, "%s: %s has a gradient it did not request" % (kind, n)
    finally:
        for p in params.values():
            p.requires_grad_(True)


@pytest.mark.parametrize("kind", ["fg", "render"])
def test_two_conds_in_one_graph(scenes, kind):
    """One module evaluated with cond A, then with cond B, and one backward of the summed loss: each node's backward
    runs with its own forward's cond."""
    c = scenes["trained"]
    N = 2000
    cond_b = c["p"]["cond"] + 0.3 * torch.randn(c["p"]["cond"].shape, generator=_gen(91))
    if kind == "render":
        net = _module(networks.RenderingNet, "rendering_network", c["p"]["render"])
        (pts, nrm, bpa, feat), ka = _ren_inputs(c, N, 90)
        bpb = cond_b.reshape(1, -1).cuda()
        kb = R.relu_margin(c["p"]["render"], pts, nrm, feat, bpb) >= R.KINK
        keep = ka & kb
        wa, wb = _randn((N, 3), 92) * keep[:, None], _randn((N, 3), 93) * keep[:, None]
        leaves = [t.detach().clone().requires_grad_(True) for t in (pts, nrm, feat)]
        bps = [bpa.requires_grad_(True), bpb.clone().requires_grad_(True)]
        loss = (net(leaves[0], leaves[1], None, bps[0], leaves[2]) * wa).sum() + \
            (net(leaves[0], leaves[1], None, bps[1], leaves[2]) * wb).sum()
        loss.backward()
        ra = _module_refs(net, (pts, nrm, bpa.detach(), feat), wa)
        rb = _module_refs(net, (pts, nrm, bpb, feat), wb)
        got = {n: p.grad for n, p in net.named_parameters()}
        got.update(points=leaves[0].grad, normals=leaves[1].grad, feature_vectors=leaves[2].grad)
        _gate_module(net, got, [ra, rb], "render two conds")
        _gate_module(net, {"body_pose": bps[0].grad}, ra, "render cond A")
        _gate_module(net, {"body_pose": bps[1].grad}, rb, "render cond B")
        return
    net = _imp_module(c, "fg")
    x, ca = _imp_inputs(c, "fg", N, 90)
    cb = cond_b.reshape(1, -1).cuda()
    wa, wb = _randn((N, 257), 92), _randn((N, 257), 93)
    xl = x.clone().requires_grad_(True)
    cl = [ca.clone().requires_grad_(True), cb.clone().requires_grad_(True)]
    ((_imp_forward(net, "fg", xl, cl[0]) * wa).sum() + (_imp_forward(net, "fg", xl, cl[1]) * wb).sum()).backward()
    ra, rb = _module_refs(net, (x, ca), wa), _module_refs(net, (x, cb), wb)
    got = {n: p.grad for n, p in net.named_parameters()}
    got["x"] = xl.grad
    _gate_module(net, got, [ra, rb], "implicit two conds")
    _gate_module(net, {"cond": cl[0].grad}, ra, "implicit cond A")
    _gate_module(net, {"cond": cl[1].grad}, rb, "implicit cond B")


@pytest.mark.parametrize("kind", ["fg", "render"])
def test_sgd_steps(scenes, kind):
    """Three SGD steps on a mirror module: at every step the gradients meet the gates against float64 at the module's
    own current parameters (the field is repacked after each step)."""
    c = scenes["trained"]
    N = 2000
    if kind == "render":
        net = _module(networks.RenderingNet, "rendering_network", c["p"]["render"])
        (pts, nrm, bp, feat), keep = _ren_inputs(c, N, 100)
        w = _randn((N, 3), 101) * keep[:, None] / N
    else:
        net = _imp_module(c, "fg")
        x, cond = _imp_inputs(c, "fg", N, 100)
        w = _randn((N, 257), 101) / N
    opt = torch.optim.SGD(net.parameters(), lr=1e-2)
    before = {n: p.detach().clone() for n, p in net.named_parameters()}
    for step in range(3):
        opt.zero_grad()
        if kind == "render":
            (net(pts, nrm, None, bp, feat) * w).sum().backward()
            refs = _module_refs(net, (pts, nrm, bp, feat), w)
        else:
            (_imp_forward(net, "fg", x, cond) * w).sum().backward()
            refs = _module_refs(net, (x, cond), w)
        _gate_module(net, {n: p.grad for n, p in net.named_parameters()}, refs, "%s SGD step %d" % (kind, step))
        opt.step()
    assert any(not torch.equal(before[n], p) for n, p in net.named_parameters())


def _adam(kw):
    return lambda ps: torch.optim.Adam(ps, lr=1e-3, **kw)


UPDATES = ["adam", "adam_foreach", "adam_fused", "load_state_dict", "data"]


@pytest.mark.parametrize("how", UPDATES)
@pytest.mark.parametrize("kind", ["fg", "render"])
def test_update_repacks_the_field(scenes, kind, how):
    """After an optimizer step (Adam: default, foreach, fused), load_state_dict or ``p.data = t``, the next forward and
    backward equal those of a module freshly built from the same state_dict, bit for bit."""
    c = scenes["trained"]
    N = 1000
    if kind == "render":
        make = lambda: _module(networks.RenderingNet, "rendering_network", c["p"]["render"])   # noqa: E731
        (pts, nrm, bp, feat), keep = _ren_inputs(c, N, 110)
        w = _randn((N, 3), 111) * keep[:, None]
        fwd = lambda m: m(pts, nrm, None, bp, feat)                                         # noqa: E731
    else:
        make = lambda: _imp_module(c, "fg")                                                 # noqa: E731
        x, cond = _imp_inputs(c, "fg", N, 110)
        w = _randn((N, 257), 111)
        fwd = lambda m: _imp_forward(m, "fg", x, cond)                                      # noqa: E731
    net = make()
    (fwd(net) * w).sum().backward()           # packs and uses the field
    if how.startswith("adam"):
        kw = {"adam": {}, "adam_foreach": dict(foreach=True), "adam_fused": dict(fused=True)}[how]
        _adam(kw)(net.parameters()).step()
    elif how == "load_state_dict":
        sd = {k: v + 1e-3 * torch.randn(v.shape, generator=_gen(112)).cuda() for k, v in net.state_dict().items()}
        net.load_state_dict(sd)
    else:
        for p in net.parameters():
            p.data = p.data * 1.01
    net.zero_grad()
    y = fwd(net)
    (y * w).sum().backward()
    fresh = make()
    fresh.load_state_dict(net.state_dict())
    y2 = fwd(fresh)
    (y2 * w).sum().backward()
    assert same(y, y2), "%s after %s: the forward differs from a fresh module's" % (kind, how)
    for (n, p), (_, q) in zip(net.named_parameters(), fresh.named_parameters()):
        assert same(p.grad, q.grad), "%s after %s: d %s differs from a fresh module's" % (kind, how, n)


def test_backward_on_caller_stream(scenes):
    """Both calls on a non-default stream, read there without a host synchronisation: the same bits as on the default
    stream."""
    c = scenes["trained"]
    cases = [Imp(c, "fg", CHUNK + 1, 120), Imp(c, "bg", 5000, 121), Ren(c, CHUNK + 1, 122)]
    want = [{k: v.clone() for k, _, v in R.items(case.run())} for case in cases]
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for case, w in zip(cases, want):
            got = {k: v for k, _, v in R.items(case.run())}
            for k in w:
                assert same(got[k], w[k]), k
