"""Float64 restatement of mp_deform_broyden on the GPU, for tests/test_gpu_root_finder.py.

Every quantity carries, next to its float64 value, a first-order magnitude M: the float64 sum of |terms| behind it,
propagated through the same operations the kernel performs (a sum adds its operands' M and its own |result|, a product
scales each operand's M by the other's |value|, 1 / d adds M_d / d^2, the 2-norm adds |M_g|).  An fp32 result
then sits within C * 2^-24 * M of the float64 one for a C that depends only on the depth of the expression, which is
what the tests gate on.

The nearest canonical vertex is taken in float64.  Where the two nearest vertices are so close in distance that fp32
rounding of the squared distance or the fp32 iterate's own error could reorder them, the lookup is a tie: a run given
``choice`` = 1 at that lookup takes the second vertex, so that the tests can evaluate both and accept either."""
import torch

EPS = 2.0 ** -24
TIE_REL = 2.0 ** -20         # fp32 rounding of a squared distance: < 5 * 2^-24 relative
TIE_C = 16.0                 # a tie where the fp32 iterate, within TIE_C * 2^-24 * M of float64, could reorder the two


class Body64:
    """A posed engine.Body in float64: canonical vertices, the blended [3,4] transform of every vertex and its M, the
    inverse 3x3 and its M."""

    def __init__(self, body):
        self.vc = body.verts_c.double().reshape(-1, 3)
        W, tfs = body.weights.double().reshape(-1, 24), body.tfs.double().reshape(24, 4, 4)
        self.A = torch.einsum("vn,nij->vij", W, tfs)[:, :3, :].contiguous()
        self.Am = torch.einsum("vn,nij->vij", W.abs(), tfs.abs())[:, :3, :].contiguous()
        M = self.A[:, :, :3]
        self.Mi = torch.linalg.inv(M)
        Ia = self.Mi.abs()
        self.Mim = Ia @ self.Am[:, :, :3] @ Ia + Ia


def nearest2(pts, verts, chunk=4096):
    """fp64 squared distances and indices of the nearest and second-nearest vertex: d2 = (dx^2 + dy^2) + dz^2."""
    out = [[], [], [], []]
    for s in range(0, pts.shape[0], chunk):
        p = pts[s:s + chunk]
        d = (p[:, None, 0] - verts[None, :, 0]) ** 2
        d += (p[:, None, 1] - verts[None, :, 1]) ** 2
        d += (p[:, None, 2] - verts[None, :, 2]) ** 2
        v, i = torch.topk(d, 2, dim=1, largest=False, sorted=True)
        for o, t in zip(out, (v[:, 0], i[:, 0], v[:, 1], i[:, 1])):
            o.append(t)
    if pts.shape[0] == 0:
        e = torch.zeros(0, dtype=torch.float64, device=pts.device)
        return e, e.long(), e, e.long()
    return tuple(torch.cat(o) for o in out)


def lookup(B, x, mx, choice=None):
    """(vertex, tie) of the nearest canonical vertex of x (float64 [n,3], magnitude mx [n,3]); choice [n] of 0 / 1
    picks the second vertex at ties."""
    d1, i1, d2, i2 = nearest2(x, B.vc)
    sep = (B.vc[i1] - B.vc[i2]).norm(dim=1)
    # the gap |x - v2|^2 - |x - v1|^2 is linear in x: moving x by delta moves it by at most 2 delta |v1 - v2|; the
    # fp32 differences x - v round by up to 2^-24 |x| even where x itself is exact
    delta = TIE_C * EPS * (mx.norm(dim=1) + x.norm(dim=1))
    tie = (d2 - d1) <= TIE_REL * d1 + 2 * delta * sep
    vi = i1 if choice is None else torch.where(tie & (choice == 1), i2, i1)
    return vi, tie


def mv(A, x):
    return torch.einsum("nij,nj->ni", A, x)


def skin(B, x, mx, vi):
    """forward_skinning with vertex vi's weights, f = M x + t, and its magnitude."""
    A, Am = B.A[vi], B.Am[vi]
    f = mv(A[:, :, :3], x) + A[:, :, 3]
    mf = mv(Am[:, :, :3], x.abs()) + Am[:, :, 3] + mv(A[:, :, :3].abs(), mx)
    return f, mf


def norm(g, mg):
    """|g| and its M: |delta |g|| <= |delta g|_2 also where g is 0."""
    r = g.norm(dim=1)
    return r, mg.norm(dim=1) + r


def residual(B, p, x, vi):
    """|forward_skinning(x) - p| at the fp32 points x (exact in float64) with vertex vi, and its magnitude."""
    f, mf = skin(B, x, torch.zeros_like(x), vi)
    g = f - p
    return norm(g, mf + g.abs())


def run(B, p, x0, K, thr, choice=None):
    """mp_deform_broyden restated: from the start x0 (the GPU's closed form, exact in float64) at most K steps while the
    best residual is >= thr.  choice [n, K + 1] (or None): per lookup, 0 / 1 = first / second vertex at a tie.
    Returns dict(x [K+1,n,3], mx, r [K+1,n], mr (iterates and residuals), active [K+1,n] (step j was taken),
    tie [n] (some lookup was a tie)."""
    n = p.shape[0]
    x, mx = x0.clone(), torch.zeros_like(x0)
    ch = (lambda j: None) if choice is None else (lambda j: choice[:, j])
    vi, tie = lookup(B, x, mx, ch(0))
    f, mf = skin(B, x, mx, vi)
    g = f - p
    mg = mf + g.abs()
    Ji, mJi = B.Mi[vi].clone(), B.Mim[vi].clone()
    r, mr = norm(g, mg)
    best = r.clone()
    xs, mxs, rs, mrs = [x.clone()], [mx.clone()], [r], [mr]
    act = [torch.zeros(n, dtype=torch.bool, device=p.device)]
    for k in range(K):
        a = best >= thr
        dx = -mv(Ji, g)
        mdx = mv(Ji.abs(), mg) + mv(mJi, g.abs()) + mv(Ji.abs(), g.abs())
        xn = x + dx
        mxn = mx + mdx + xn.abs()
        vi, t = lookup(B, xn, mxn, ch(k + 1))
        tie = tie | (t & a)
        fn, mfn = skin(B, xn, mxn, vi)
        gn = fn - p
        mgn = mfn + gn.abs()
        dg = gn - g
        mdg = mgn + mg + dg.abs()
        u = mv(Ji, dg)
        mu = mv(Ji.abs(), mdg) + mv(mJi, dg.abs()) + mv(Ji.abs(), dg.abs())
        vt = torch.einsum("ni,nij->nj", dx, Ji)
        mvt = torch.einsum("ni,nij->nj", mdx, Ji.abs()) + torch.einsum("ni,nij->nj", dx.abs(), mJi + Ji.abs())
        den = (dx * u).sum(1)
        mden = (mdx * u.abs() + dx.abs() * mu + (dx * u).abs()).sum(1)
        upd = den.abs() > 1e-20
        iden = 1.0 / torch.where(upd, den, torch.ones_like(den))
        miden = mden * iden * iden + iden.abs()
        av = dx - u
        mav = mdx + mu + av.abs()
        T = av[:, :, None] * vt[:, None, :] * iden[:, None, None]
        mT = (mav[:, :, None] * vt.abs()[:, None, :] * iden.abs()[:, None, None]
              + av.abs()[:, :, None] * mvt[:, None, :] * iden.abs()[:, None, None]
              + av.abs()[:, :, None] * vt.abs()[:, None, :] * miden[:, None, None] + T.abs())
        Jn = Ji + torch.where(upd[:, None, None], T, torch.zeros_like(T))
        mJn = mJi + torch.where(upd[:, None, None], mT, torch.zeros_like(mT)) + Jn.abs()
        rn, mrn = norm(gn, mgn)
        A3 = a[:, None]
        x, mx = torch.where(A3, xn, x), torch.where(A3, mxn, mx)
        g, mg = torch.where(A3, gn, g), torch.where(A3, mgn, mg)
        Ji, mJi = torch.where(a[:, None, None], Jn, Ji), torch.where(a[:, None, None], mJn, mJi)
        best = torch.where(a & (rn < best), rn, best)
        xs.append(xn)
        mxs.append(mxn)
        rs.append(rn)
        mrs.append(mrn)
        act.append(a)
    return dict(x=torch.stack(xs), mx=torch.stack(mxs), r=torch.stack(rs), mr=torch.stack(mrs), active=torch.stack(act),
                tie=tie)
