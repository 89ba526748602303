"""Mirror of /root/reference/code/lib/model/deformer.py (SMPLDeformer, skinning)."""
import torch

from .. import engine


class SMPLDeformer(torch.nn.Module):
    """deformer.py:6-54.  The reference builds its canonical vertices / skinning weights from the SMPL model
    files (licence-gated, absent offline); here they are passed in explicitly (``smpl_verts`` [1,V,3],
    ``smpl_weights`` [1,V,24]) — everything else keeps the reference's signatures."""

    def __init__(self, max_dist=0.05, K=1, gender="male", betas=None, smpl_verts=None, smpl_weights=None, scale=1.0):
        super().__init__()
        if K != 1:
            raise NotImplementedError("K must be 1 (the only value the reference uses, deformer.py:7)")
        if smpl_verts is None or smpl_weights is None:
            raise ValueError("SMPL model files are not available: pass the canonical smpl_verts / smpl_weights")
        self.max_dist, self.K = max_dist, K
        self.smpl_verts = smpl_verts.reshape(1, -1, 3)
        self.smpl_weights = smpl_weights.reshape(1, -1, 24)
        self._scale = float(scale)
        self._body = None
        self._root_finder = (0, 1e-5)

    def set_root_finder(self, max_steps, cvg_threshold=1e-5):
        """Not in the reference (SURVEY.md §8 row f4): max_steps > 0 refines the closed-form inverse with Broyden
        iterations on forward_skinning(x_c) = x (engine.Body.set_root_finder); 0 = reference behaviour (default)."""
        self._root_finder = (int(max_steps), float(cvg_threshold))
        if self._body is not None:
            self._body.set_root_finder(*self._root_finder)

    def body(self, device):
        if self._body is None or self._body.device != torch.device(device):
            self._body = engine.Body(self.smpl_verts[0], self.smpl_weights[0], cano_cell=0.1001 / max(self._scale, 1e-3),
                                     device=device)
            if self._root_finder[0] > 0:
                self._body.set_root_finder(*self._root_finder)
        return self._body

    def forward(self, x, smpl_tfs, return_weights=True, inverse=False, smpl_verts=None):
        if x.shape[0] == 0:
            return x                                   # deformer.py:20
        if return_weights or not inverse or smpl_verts is None:
            raise NotImplementedError("only the hot-path call forward(x, tfs, return_weights=False, inverse=True, "
                                      "smpl_verts=posed) is provided (multiply.py:139)")
        b = self.body(x.device)
        tfs = smpl_tfs[0] if smpl_tfs.ndim == 4 else smpl_tfs
        b.set_pose(smpl_verts[0], tfs)
        if torch.is_grad_enabled() and (x.requires_grad or smpl_tfs.requires_grad):
            # gradients to x and smpl_tfs; none to smpl_verts (the weights are detached, deformer.py:47)
            return engine.DeformInverse.apply(b, True, x, tfs)
        return b.deform_inverse(x, exact_far=True)

    def _posed_tfs(self, b, smpl_tfs):
        """The [24,4,4] view of ``smpl_tfs``, which must be the transforms the body is posed with: the gradient goes to
        exactly that tensor, never to other transforms."""
        tfs = smpl_tfs.reshape(24, 4, 4)
        if not torch.equal(b.tfs, tfs.detach().to(device=b.tfs.device, dtype=b.tfs.dtype)):
            raise ValueError("smpl_tfs differs from the transforms the body is posed with (forward(...) of this frame)")
        return tfs

    def forward_skinning(self, xc, cond, smpl_tfs):
        """deformer.py:31-35 — returns x_d [1,N,3]; the Jacobian used for normals comes from ``jacobian_inverse``.
        With grad mode on, gradients go to ``xc`` and ``smpl_tfs`` when either requires grad."""
        b = self.body(xc.device)
        if getattr(b, "tfs", None) is None:
            raise RuntimeError("call forward(...) (which sets the frame's pose) first")
        if torch.is_grad_enabled() and (xc.requires_grad or torch.is_tensor(smpl_tfs) and smpl_tfs.requires_grad):
            xd, _ = engine.ForwardJac.apply(b, xc.reshape(-1, 3), self._posed_tfs(b, smpl_tfs))
            return xd[None]
        xd, _ = b.forward_jac(xc.reshape(-1, 3))
        return xd[None]

    def jacobian_inverse(self, xc, smpl_tfs=None):
        """Inverse Jacobian of forward skinning at xc (multiply.py:625-641) -> [N,3,3].  Given ``smpl_tfs`` (the
        transforms the body is posed with) and grad mode on, gradients go to it; Jinv is piecewise constant in xc."""
        b = self.body(xc.device)
        if smpl_tfs is not None and torch.is_grad_enabled() and smpl_tfs.requires_grad:
            _, J = engine.ForwardJac.apply(b, xc.reshape(-1, 3), self._posed_tfs(b, smpl_tfs))
            return J.reshape(-1, 3, 3)
        _, J = b.forward_jac(xc.reshape(-1, 3))
        return J.reshape(-1, 3, 3)
