"""References of the networks' first-order backward (mp_implicit_backward, mp_render_backward) and the per-element error
model their gates use.

Reference values are torch autograd through oracle/port.py's implicit_forward / rendering_forward on the effective
weights (W = g v / ||v|| where weight-normed), evaluated in float64 on the device of the inputs (float32 for the CPU
check of the bound).

Error model.  Every gradient element g must satisfy |g - g_ref| <= C 2^-24 M.  M is a float64 *magnitude backward*
written layer by layer over the structure of DESIGN.md §3.9, with every weight and input replaced by its absolute value.
M is the magnitude of the terms of the operation that produced the element, taken from the float64 values of its
operands, plus the error those operands carry from the operation before them.  For a layer l with activation s, input
A_{l-1}, pre-activation Z_l and upstream dA_l:
    M_Z_l      = |W_l| |A_{l-1}| + |b_l|                        the fp32 recompute of Z
    M_A_l      = |A_l| + |s'(Z_l)| M_Z_l                        the recomputed activation, with Z's error
    M_dA_l     = |G_{l+1}| |W_{l+1}|                            the input-gradient product
    M_G_l      = M_dA_l |s'(Z_l)| + |dA_l| (|s''(Z_l)| M_Z_l + 2^-102)
                                                                G = dA s'(Z) at the recomputed Z (softplus with beta
                                                                100 has s'' up to 25); 2^-102 = 2^-126 / 2^-24 is s'
                                                                underflowing fp32 far below a kink
    M_dW_l     = M_G_l^T M_A_{l-1},  M_db_l = sum over points of M_G_l,  the input gradient out of the first layer
                 M_G_0 |W_0|
An error enters M through one operation, not again in the next layer's terms (M_dA takes |G|, not M_G).  A bound that
carried every earlier error's full magnitude through |W| would grow by the row sum of |W| (about 10 here) per layer,
10^8 over the stack, and gate nothing; the errors the layers pass on average out in the next sum as the values do, and C
covers them.  (LEVELS is the number of operations an error is carried through.)
ImplicitNet's skip layer takes [h3, embedding] with the skip's 1/sqrt(2) in its weight, and its input gradient splits
between h3 and the embedding; the embedding's backward is sum_f 2^f (|cos(2^f x)| M_sin + |sin(2^f x)| M_cos) plus the
identity columns.  lin0's cond columns are M_db0 (x) |cond| and M_dcond = |W0[:, E:]|^T M_db0.  RenderingNet's pose
features lin_pose(body_pose) enter its input with the magnitude |Wp| |body_pose| + |bp|, and the lin_pose chain is
M_dpf = |W0[:, 6:14]|^T M_db0, M_dWp = M_dpf (x) |body_pose|, M_dbp = M_dpf, M_dbody_pose = |Wp|^T M_dpf.

Operand floor.  The kernel scales each operand of a product so that its largest magnitude lies in [2^13, 2^14), then
splits every element into fp16 hi + lo.  Below about 2^-17 of that maximum lo falls onto fp16's subnormal grid and the
element keeps fewer bits than the split's 22.  So in every product each staged operand element counts as
max(|a|, 2^-17 amax), with amax the operand's largest |value|: per chunk of 32768 points for the layer inputs and G, per
call for the weights (lin0: its embedding columns, the part the product reads).  The bias sums, the cond columns, the
lin_pose chain and the embedding's backward are not staged products and take no floor."""
import math

import torch
import torch.nn.functional as F

from oracle import port

EPS = 2.0 ** -24
FLOOR = 2.0 ** -17
CHUNK = 32768
BETA = 100.0
LEVELS = 1
TINY = 2.0 ** -102      # fp32's smallest normal, 2^-126, as a multiple of EPS

# a pre-activation this close to 0 may round to the other side in fp32: the ReLU derivative is ambiguous there
KINK = 1e-6


# ---------------------------------------------------------------------------------------------
# reference values: torch autograd of the port
# ---------------------------------------------------------------------------------------------

def effective_leaves(sd, n_lin, dtype=torch.float64, device="cuda"):
    """Leaves lin{l}.weight (the applied W: g v / ||v|| where weight-normed) and lin{l}.bias, in ``dtype``."""
    leaves = {}
    for l in range(n_lin):
        if f"lin{l}.weight_v" in sd:
            w = torch._weight_norm(sd[f"lin{l}.weight_v"].double(), sd[f"lin{l}.weight_g"].double(), 0)
        else:
            w = sd[f"lin{l}.weight"].double()
        leaves[f"lin{l}.weight"] = w.detach().to(device, dtype).requires_grad_(True)
        leaves[f"lin{l}.bias"] = sd[f"lin{l}.bias"].to(device, dtype).requires_grad_(True)
    return leaves


def _up(t, dtype):
    return 0 if t is None else t.to(dtype)


def ref_implicit(sd, x, cond, multires, d_sdf, d_feat, dtype=torch.float64):
    """VJP of ImplicitNet at x [N, d_in] with cond: dict(d_x, d_cond, d_weight [9], d_bias [9])."""
    leaves = effective_leaves(sd, 9, dtype, x.device)
    xs = x.to(dtype).requires_grad_(True)
    c = cond.reshape(1, -1).to(x.device, dtype).requires_grad_(True)
    y = port.implicit_forward(leaves, xs, c, multires, weight_norm=False)
    loss = (y[:, 0] * _up(d_sdf, dtype)).sum() + (y[:, 1:] * _up(d_feat, dtype)).sum()
    params = [leaves[f"lin{l}.{k}"] for l in range(9) for k in ("weight", "bias")]
    g = torch.autograd.grad(loss, [xs, c] + params, allow_unused=True)
    return dict(d_x=g[0], d_cond=g[1].reshape(-1), d_weight=list(g[2::2]), d_bias=list(g[3::2]))


def ref_render(sd, pts, nrm, feat, body_pose, d_rgb, dtype=torch.float64):
    """VJP of RenderingNet 'pose_no_view': dict(d_points, d_normals, d_feat, d_body_pose, d_lin_pose_weight,
    d_lin_pose_bias, d_weight [5], d_bias [5])."""
    dev = pts.device
    leaves = effective_leaves(sd, 5, dtype, dev)
    leaves["lin_pose.weight"] = sd["lin_pose.weight"].to(dev, dtype).requires_grad_(True)
    leaves["lin_pose.bias"] = sd["lin_pose.bias"].to(dev, dtype).requires_grad_(True)
    p, n, f = (t.to(dtype).requires_grad_(True) for t in (pts, nrm, feat))
    bp = body_pose.reshape(1, -1).to(dev, dtype).requires_grad_(True)
    rgb = port.rendering_forward(leaves, "pose_no_view", p, n, None, bp, f, weight_norm=False)
    params = [leaves[f"lin{l}.{k}"] for l in range(5) for k in ("weight", "bias")]
    g = torch.autograd.grad((rgb * d_rgb.to(dtype)).sum(),
                            [p, n, f, bp, leaves["lin_pose.weight"], leaves["lin_pose.bias"]] + params)
    return dict(d_points=g[0], d_normals=g[1], d_feat=g[2], d_body_pose=g[3].reshape(-1), d_lin_pose_weight=g[4],
                d_lin_pose_bias=g[5], d_weight=list(g[6::2]), d_bias=list(g[7::2]))


def relu_margin(sd, pts, nrm, feat, body_pose):
    """Each point's smallest |pre-activation| over the colour net's ReLU layers, in float64.  Where it is below KINK,
    relu' of an fp32 evaluation may differ from the float64 one, and so may that point's whole contribution to every
    gradient: a whole term, not a rounding error."""
    dev = pts.device
    leaves = effective_leaves(sd, 4, torch.float64, dev)
    with torch.no_grad():
        bp = body_pose.reshape(1, -1).to(dev, torch.float64)
        pf = F.linear(bp, sd["lin_pose.weight"].to(dev, torch.float64), sd["lin_pose.bias"].to(dev, torch.float64))
        h = torch.cat([pts.double(), nrm.double(), pf.expand(pts.shape[0], -1), feat.double()], -1)
        margin = torch.full((pts.shape[0],), float("inf"), dtype=torch.float64, device=dev)
        for l in range(4):
            z = F.linear(h, leaves[f"lin{l}.weight"], leaves[f"lin{l}.bias"])
            margin = torch.minimum(margin, z.abs().min(1).values)
            h = torch.relu(z)
    return margin


# ---------------------------------------------------------------------------------------------
# the magnitude backward
# ---------------------------------------------------------------------------------------------

def _weights(sd, n_lin, device):
    leaves = effective_leaves(sd, n_lin, torch.float64, device)
    return ([leaves[f"lin{l}.weight"].detach() for l in range(n_lin)],
            [leaves[f"lin{l}.bias"].detach() for l in range(n_lin)])


def _staged(m, a):
    """An operand of a product as staged: max(m, 2^-17 amax), amax = max |a| over each chunk of CHUNK points (rows)."""
    out = m.clone()
    for s in range(0, m.shape[0], CHUNK):
        am = float(a[s:s + CHUNK].abs().max()) if a[s:s + CHUNK].numel() else 0.0
        out[s:s + CHUNK].clamp_(min=FLOOR * am)
    return out


def _staged_w(w):
    """|W| as staged: max(|W|, 2^-17 max|W|) (the weights are scaled once per call)."""
    a = w.abs()
    return a.clamp(min=FLOOR * float(a.max()))


def _softplus(z):
    """softplus(beta=100, threshold=20) and its first two derivatives."""
    bz = BETA * z
    lin = bz > 20.0
    s = torch.where(lin, z, torch.log1p(torch.exp(bz.clamp(max=20.0))) / BETA)
    d1 = torch.where(lin, torch.ones_like(z), torch.sigmoid(bz))
    d2 = torch.where(lin, torch.zeros_like(z), BETA * torch.sigmoid(bz) * torch.sigmoid(-bz))
    return s, d1, d2


def _up64(t, shape, device):
    return torch.zeros(shape, dtype=torch.float64, device=device) if t is None else t.double().reshape(shape)


def implicit_magnitude(sd, x, cond, multires, d_sdf, d_feat):
    """M of every output of mp_implicit_backward (module docstring), float64 on x's device, keyed as ref_implicit."""
    dev = x.device
    W, b = _weights(sd, 9, dev)
    N, d = x.shape
    E = d * (1 + 2 * multires)
    skip = 4
    r2 = math.sqrt(2.0)
    with torch.no_grad():
        x64 = x.double()
        emb = port.embed(x64, multires)
        c = cond.reshape(-1).to(dev, torch.float64)
        Wk = [w.clone() for w in W]            # the weights the kernel's products read
        Wk[0] = W[0][:, :E]
        Wk[skip] = W[skip] / r2
        Ws = [_staged_w(w) for w in Wk]
        b0 = b[0] + W[0][:, E:] @ c
        mb0 = b[0].abs() + W[0][:, E:].abs() @ c.abs()
        # forward: each layer's input A and its M_A, the pre-activation Z, M_Z and s', s'' at Z
        A, MA, MZ, D1, D2 = [], [], [], [], []
        a, ma = emb, emb.abs()
        for l in range(9):
            if l == skip:
                a, ma = torch.cat([a, emb], 1), torch.cat([ma, emb.abs()], 1)
            A.append(a)
            MA.append(ma)
            if l == 8:
                break
            z = a @ Wk[l].T + (b0 if l == 0 else b[l])
            mz = _staged(a.abs(), a) @ Ws[l].T + (mb0 if l == 0 else b[l].abs())
            s, d1, d2 = _softplus(z)
            MZ.append(mz)
            D1.append(d1)
            D2.append(d2)
            a, ma = s, s.abs() + d1 * mz
        # backward: G and M_G of layer l
        g = torch.cat([_up64(d_sdf, (N, 1), dev), _up64(d_feat, (N, 256), dev)], 1)
        mg = [g.abs()] * (LEVELS + 1)
        MW, MB = [None] * 9, [None] * 9
        m_emb = torch.zeros(N, E, dtype=torch.float64, device=dev)
        for l in range(8, -1, -1):
            MW[l] = _staged(mg[-1], g).T @ _staged(MA[l], A[l])
            MB[l] = mg[-1].sum(0)
            da, mda = g @ Wk[l], [_staged(m, g) @ Ws[l] for m in mg]
            if l == skip:
                MW[l] = MW[l] / r2
                m_emb = m_emb + mda[-1][:, -E:]
                da, mda = da[:, :-E], [m[:, :-E] for m in mda]
            if l == 0:
                m_emb = m_emb + mda[-1]
                break
            g = da * D1[l - 1]
            mg = [g.abs()] + [m * D1[l - 1] + da.abs() * (D2[l - 1] * MZ[l - 1] + TINY) for m in mda[:-1]]
        MW[0] = torch.cat([MW[0], MB[0][:, None] * c.abs()[None, :]], 1)
        m_cond = W[0][:, E:].abs().T @ MB[0]
        m_x = m_emb[:, :d].clone()
        for f in range(multires):
            t = x64 * 2.0 ** f
            ms, mc = m_emb[:, d + 2 * f * d: d + (2 * f + 1) * d], m_emb[:, d + (2 * f + 1) * d: d + (2 * f + 2) * d]
            m_x += 2.0 ** f * (t.cos().abs() * ms + t.sin().abs() * mc)
    return dict(d_x=m_x, d_cond=m_cond, d_weight=MW, d_bias=MB)


def render_magnitude(sd, pts, nrm, feat, body_pose, d_rgb):
    """M of every output of mp_render_backward (module docstring), float64 on pts' device, keyed as ref_render."""
    dev = pts.device
    W, b = _weights(sd, 5, dev)
    Ws = [_staged_w(w) for w in W]
    with torch.no_grad():
        Wp = sd["lin_pose.weight"].to(dev, torch.float64)
        bpb = sd["lin_pose.bias"].to(dev, torch.float64)
        bp = body_pose.reshape(-1).to(dev, torch.float64)
        N = pts.shape[0]
        pf = (Wp @ bp + bpb).expand(N, -1)
        mpf = (Wp.abs() @ bp.abs() + bpb.abs()).expand(N, -1)
        a = torch.cat([pts.double(), nrm.double(), pf, feat.double()], 1)
        ma = torch.cat([pts.double().abs(), nrm.double().abs(), mpf, feat.double().abs()], 1)
        A, MA, Z, MZ = [], [], [], []
        for l in range(5):
            A.append(a)
            MA.append(ma)
            z = a @ W[l].T + b[l]
            mz = _staged(ma if l == 0 else a.abs(), a) @ Ws[l].T + b[l].abs()
            Z.append(z)
            MZ.append(mz)
            on = (z > 0).double()
            a, ma = z * on, mz * on
        y = torch.sigmoid(Z[4])
        d1 = y * (1 - y)
        d2 = d1 * (1 - 2 * y)
        up = d_rgb.double()
        g = up * d1
        mg = [up.abs() * (d1 + d2.abs() * MZ[4] + TINY)] * (LEVELS + 1)
        MW, MB = [None] * 5, [None] * 5
        for l in range(4, -1, -1):
            MW[l] = _staged(mg[-1], g).T @ _staged(MA[l], A[l])
            MB[l] = mg[-1].sum(0)
            da, mda = g @ W[l], [_staged(m, g) @ Ws[l] for m in mg]
            if l == 0:
                break
            on = (Z[l - 1] > 0).double()
            g = da * on
            mg = [g.abs()] + [m * on for m in mda[:-1]]
        m_pf = W[0][:, 6:14].abs().T @ MB[0]
        mda = mda[-1]
    return dict(d_points=mda[:, 0:3], d_normals=mda[:, 3:6], d_feat=mda[:, 14:], d_body_pose=Wp.abs().T @ m_pf,
                d_lin_pose_weight=m_pf[:, None] * bp.abs()[None, :], d_lin_pose_bias=m_pf, d_weight=MW, d_bias=MB)


def weight_norm_magnitude(m_dw, v, g):
    """M of d weight_v and d weight_g from M of d W, W = g v / ||v|| (rows): dg = dW . v^, dv = g / ||v|| (dW - dg v^)."""
    v, g = v.double().to(m_dw.device), g.double().to(m_dw.device)
    nv = v.norm(dim=1, keepdim=True)
    vh = (v / nv).abs()
    m_dg = (m_dw * vh).sum(1, keepdim=True)
    return g.abs() / nv * (m_dw + vh * m_dg), m_dg


# ---------------------------------------------------------------------------------------------
# gates
# ---------------------------------------------------------------------------------------------

def items(d):
    """(name, kind, tensor) of every output in a result dict; list entries are named k[i] and share the kind k."""
    for k, v in d.items():
        if isinstance(v, list):
            for i, t in enumerate(v):
                yield "%s[%d]" % (k, i), k, t
        else:
            yield k, k, v


def ratio(err, M):
    """max over elements of |err| / (2^-24 M): the C an element needs; inf where M = 0 and err != 0."""
    err, M = err.abs().double(), M.double()
    r = torch.where(M > 0, err / (EPS * torch.where(M > 0, M, torch.ones_like(M))),
                    torch.where(err == 0, torch.zeros_like(M), torch.full_like(M, math.inf)))
    return float(r.max()) if r.numel() else 0.0


def element_c(got, ref, mag):
    """kind -> the largest C any element of that kind needs (|g - g_ref| <= C 2^-24 M); outputs that are None in
    ``got`` are skipped."""
    out = {}
    mags = {name: m for name, _, m in items(mag)}
    refs = {name: r for name, _, r in items(ref)}
    for name, kind, g in items(got):
        if g is None:
            continue
        r, m = refs[name], mags[name]
        assert g.shape == r.shape == m.shape, (name, g.shape, r.shape, m.shape)
        out[kind] = max(out.get(kind, 0.0), ratio(g.double().to(r.device) - r.double(), m))
    return out
