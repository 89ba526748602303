"""Mirror of /root/reference/code/lib/model/smpl.py: ``SMPLServer`` on the device (mp_smpl_forward).

The reference loads the licence-gated SMPL pkl through ``lib.smpl.body_models.SMPL`` (smpl.py:12); here the
model arrays are passed in (``model=dict(v_template, shapedirs, posedirs, J_regressor, parents, lbs_weights)`` —
exactly the buffers body_models.py registers), so the real pkl can be plugged in when available and
``scene.make_smpl_model`` stands in offline."""
import ctypes as C
import numpy as np
import torch

from .. import _lib as L
from .. import engine


class SMPLServer(torch.nn.Module):
    def __init__(self, gender="neutral", betas=None, v_template=None, model=None, device="cuda"):
        super().__init__()
        if model is None:
            raise ValueError("SMPL model files are licence-gated: pass model=dict(v_template, shapedirs, ...)")
        dev = torch.device(device)
        self._arr = {k: L.dev(model[k], dev) for k in ("v_template", "shapedirs", "posedirs", "J_regressor", "lbs_weights")}
        self._ignore_betas = v_template is not None        # smpl.py:65-66: betas are zeroed when v_template is given
        if v_template is not None:
            self._arr["v_template"] = L.dev(torch.as_tensor(v_template), dev)
        self.V = self._arr["v_template"].shape[0]
        par = [int(p) for p in model["parents"]]
        par[0] = -1
        self.bone_parents = np.array(par)
        self.betas = L.dev(torch.as_tensor(betas), dev) if betas is not None else None
        pa = (C.c_int * 24)(*[max(p, 0) for p in par])
        self._storage = L.workspace(L.call("mp_smpl_bytes", self.V), dev)
        self.handle = L.Handle("mp_smpl_free")
        a = self._arr
        L.call("mp_smpl_create", a["v_template"], a["shapedirs"], a["posedirs"], a["J_regressor"], pa, a["lbs_weights"],
               self.V, self.betas.reshape(-1) if self.betas is not None and v_template is None else None,
               self._storage, self._storage.numel(), C.byref(self.handle))
        self.device = dev
        vc = torch.empty(self.V, 3, device=dev)
        ti = torch.empty(24, 4, 4, device=dev)
        L.call("mp_smpl_canonical", self.handle, vc, ti)
        self.verts_c = vc[None]                      # smpl.py:45
        self.tfs_c_inv = ti                          # smpl.py:47
        self.weights = a["lbs_weights"][None]
        self.scale = 1.0
        # the pkl's triangles over verts_c (multiply.py:118-121), when the model dict carries them (optional `faces`)
        self.faces = torch.as_tensor(model["faces"]).to(torch.int64) if model.get("faces") is not None else None

    def forward(self, scale, transl, thetas, betas, absolute=False):
        """smpl.py:50-95: scale [1], transl [1,3], thetas [1,72], betas [1,10] -> dict.  When grad mode is on and any of
        the four requires grad, smpl_verts / smpl_tfs carry gradients to them (mp_smpl_backward)."""
        if torch.is_grad_enabled() and any(torch.is_tensor(x) and x.requires_grad for x in (scale, transl, thetas, betas)):
            verts, tfs = engine.SmplFunction.apply(self, bool(absolute), scale, transl, thetas, betas)
        else:
            verts, tfs, _ = self._run(scale, transl, thetas, betas, absolute)
        return {"smpl_verts": verts[None], "smpl_tfs": tfs[None], "smpl_weights": self.weights}

    def _run(self, scale, transl, thetas, betas, absolute):
        dev = self.device
        s, t, th, b = (L.dev(x.reshape(-1), dev) for x in (scale, transl, thetas, betas))
        if self._ignore_betas:
            b = torch.zeros_like(b)
        verts = torch.empty(self.V, 3, device=dev)
        tfs = torch.empty(24, 4, 4, device=dev)
        L.call("mp_smpl_forward", self.handle, s, t, th, b, int(absolute), verts, tfs)
        self._keep = (s, t, th, b)
        return verts, tfs, (s, t, th, b)

    def _backward(self, inputs, absolute, d_verts, d_tfs):
        """mp_smpl_backward at the inputs ``_run`` saw: -> (d_scale [1], d_transl [3], d_thetas [72], d_betas [10])."""
        dev = self.device
        s, t, th, b = inputs
        d_verts, d_tfs = L.dev(d_verts, dev), L.dev(d_tfs, dev)
        out = [torch.empty(n, device=dev) for n in (1, 3, 72, 10)]
        ws = L.workspace(L.call("mp_smpl_backward_workspace_bytes", self.V), dev)
        L.call("mp_smpl_backward", self.handle, s, t, th, b, int(absolute), d_verts, d_tfs, *out, ws, ws.numel())
        if self._ignore_betas:
            out[3] = torch.zeros_like(out[3])
        return tuple(out)

    def canonical_output(self):
        th = torch.zeros(1, 72)
        th[0, 5], th[0, 8] = np.pi / 6, -np.pi / 6
        b = self.betas.reshape(1, 10) if self.betas is not None else torch.zeros(1, 10)
        return self(torch.ones(1), torch.zeros(1, 3), th, b)
