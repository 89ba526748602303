"""Float64 autograd through oracle/port.py's restatements of the SMPL server and the deformer: the reference gradients of
test_body_grad_golden.py (pinned there to the reference's own code) and test_gpu_body_grad.py (any size)."""
import contextlib

import numpy as np
import torch

from oracle import port


@contextlib.contextmanager
def float64():
    old = torch.get_default_dtype()
    torch.set_default_dtype(torch.float64)
    try:
        yield
    finally:
        torch.set_default_dtype(old)


def _t(a, grad=False):
    return torch.tensor(np.asarray(a, np.float64), requires_grad=grad)


def model64(model):
    return {k: (torch.as_tensor(np.asarray(v)).double() if k != "parents" else torch.as_tensor(np.asarray(v)).long())
            for k, v in model.items() if k in ("v_template", "shapedirs", "posedirs", "J_regressor", "lbs_weights",
                                               "parents")}


def port_smpl_grads(model, tfs_c_inv, scale, transl, theta, betas, absolute, v_template, u_v, u_t):
    """Gradients of <u_v, smpl_verts> + <u_t, smpl_tfs> through port.smpl_server_forward in float64 w.r.t. transl, thetas,
    betas (autograd) and scale.  port.smpl_server_forward writes the scale in place (as smpl.py:86-88 does), which
    autograd refuses to differentiate w.r.t. scale; the outputs are linear in scale, so d_scale = <u, out(1) - out(0)>."""
    m = model64(model)
    with float64():
        cinv = _t(tfs_c_inv)
        s = _t(np.reshape(scale, 1))
        t, th, b = _t(np.reshape(transl, 3), True), _t(np.reshape(theta, 72), True), _t(np.reshape(betas, 10), True)
        bb = torch.zeros_like(b) if v_template else b
        uv, ut = _t(u_v), _t(u_t)
        o = port.smpl_server_forward(m, cinv, s, t, th, bb, absolute=bool(absolute))
        ((o["smpl_verts"] * uv).sum() + (o["smpl_tfs"] * ut).sum()).backward()
        with torch.no_grad():
            lin = [port.smpl_server_forward(m, cinv, torch.full((1,), v), t, th, bb, absolute=bool(absolute))
                   for v in (1.0, 0.0)]
            ds = sum(((a[k] - z[k]) * u).sum() for a, z in [lin] for k, u in (("smpl_verts", uv), ("smpl_tfs", ut)))
        grad = lambda x: np.zeros(x.shape) if x.grad is None else x.grad.numpy()
        return dict(verts=o["smpl_verts"].detach().numpy(), tfs=o["smpl_tfs"].detach().numpy(), scale=np.array([float(ds)]),
                    transl=grad(t), thetas=grad(th), betas=grad(b))


def port_inverse_grads(x, verts_p, weights, tfs, u_xc):
    """deformer.py:19-30 in float64 (port.query_skinning_weights + port.skinning(inverse=True)): -> x_c, gradients of
    <u_xc, x_c> w.r.t. x and tfs, the nearest posed vertex of every point and the per-point dL/dA [N,4,4]."""
    with float64():
        xv, tv = _t(x, True), _t(tfs, True)
        w, _ = port.query_skinning_weights(xv.detach()[None], _t(verts_p), _t(weights)[None])
        A = torch.einsum("bpn,bnij->bpij", w, tv[None])
        A.retain_grad()
        x_h = torch.nn.functional.pad(xv[None], (0, 1), value=1.0)
        xc = torch.einsum("bpij,bpj->bpi", A.inverse(), x_h)[0, :, :3]
        (xc * _t(u_xc)).sum().backward()
        assert np.allclose(xc.detach().numpy(), port.skinning(xv.detach()[None], w, tv.detach()[None], inverse=True)[0])
        return dict(x_c=xc.detach().numpy(), x=xv.grad.numpy(), tfs=tv.grad.numpy(), w=w[0].numpy(),
                    dA=A.grad[0].numpy(), A=A.detach()[0].numpy())


def port_forward_grads(x_c, verts_c, weights, tfs, u_xd=None, u_J=None):
    """deformer.py:31-35 and multiply.py:625-641 in float64 (port.forward_skinning, Jinv = A^-1): gradients of
    <u_xd, x_d> + <u_J, Jinv> w.r.t. x_c and tfs, plus the per-point dL/dT [N,3,4] and the weights used."""
    with float64():
        xv, tv = _t(x_c, True), _t(tfs, True)
        person = dict(verts_c=_t(verts_c), weights=_t(weights), tfs=tv)
        x_d, A = port.forward_skinning(xv, person)
        Jinv = torch.linalg.inv(A)
        loss = 0.0
        if u_xd is not None:
            loss = loss + (x_d * _t(u_xd)).sum()
        if u_J is not None:
            loss = loss + (Jinv * _t(np.reshape(u_J, (-1, 3, 3)))).sum()
        loss.backward()
        w, _ = port.query_skinning_weights(xv.detach()[None], _t(verts_c), _t(weights)[None])
        return dict(x_d=x_d.detach().numpy(), Jinv=Jinv.detach().numpy(), A=A.detach().numpy(),
                    x_c=np.zeros(np.shape(x_c)) if xv.grad is None else xv.grad.numpy(), tfs=tv.grad.numpy(),
                    w=w[0].numpy())
