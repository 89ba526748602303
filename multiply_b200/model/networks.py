"""Mirror of /root/reference/code/lib/model/networks.py: ``ImplicitNet`` and ``RenderingNet`` with the
reference's constructor options, parameter names (``lin{l}.weight_g / weight_v / bias``, ``lin_pose.*``)
and forward signatures, so reference checkpoints load unchanged.  ``forward`` runs on the C-ABI library — there is no
PyTorch fallback.  When grad mode is on and an input or a parameter requires grad, it runs as one autograd node
(engine.ImplicitFunction / engine.RenderFunction: the same forward call, a first-order backward on the device);
otherwise it issues exactly the plain forward's launches."""
import math
import numpy as np
import torch
import torch.nn as nn
from torch.optim.optimizer import register_optimizer_step_post_hook

from .. import engine


class _Lin(nn.Module):
    """nn.Linear / weight-normed nn.Linear parameter holder (networks.py:50-83, 254-259)."""

    def __init__(self, in_dim, out_dim, weight_norm):
        super().__init__()
        w = torch.empty(out_dim, in_dim)
        nn.init.kaiming_uniform_(w, a=math.sqrt(5))
        bound = 1 / math.sqrt(in_dim)
        b = torch.empty(out_dim).uniform_(-bound, bound)
        self.bias = nn.Parameter(b)
        if weight_norm:
            self.weight_g = nn.Parameter(w.norm(dim=1, keepdim=True))
            self.weight_v = nn.Parameter(w)
        else:
            self.weight = nn.Parameter(w)

    def set_weight(self, w, b):
        with torch.no_grad():
            if hasattr(self, "weight_v"):
                self.weight_v.copy_(w)
                self.weight_g.copy_(w.norm(dim=1, keepdim=True))
            else:
                self.weight.copy_(w)
            self.bias.copy_(b)


def _wants_grad(module, *inputs):
    """Grad mode is on and an input or a parameter requires grad: the forward goes through the autograd function."""
    return torch.is_grad_enabled() and (any(t.requires_grad for t in inputs if torch.is_tensor(t)) or
                                        any(p.requires_grad for p in module.parameters()))


def _effective(module):
    """W_0, b_0, W_1, b_1, ... of the module's lin{l}: the weight the layer applies (torch._weight_norm(v, g, 0) where
    weight-normed, as nn.utils.weight_norm computes it) and the bias."""
    out = []
    for l in range(module.num_layers - 1):
        lin = getattr(module, "lin%d" % l)
        w = torch._weight_norm(lin.weight_v, lin.weight_g, 0) if hasattr(lin, "weight_v") else lin.weight
        out += [w, lin.bias]
    return out


# Optimizer steps taken in this process.  A fused optimizer step (torch.optim.Adam(fused=True)) updates the parameters
# in place without bumping their version counters, so the packed field's cache key also holds this count, bumped after
# every step by a hook; it is read on the host, so keeping it costs no synchronisation.
_optimizer_steps = 0


def _count_step(optimizer, args, kwargs):
    global _optimizer_steps
    _optimizer_steps += 1


register_optimizer_step_post_hook(_count_step)


def _field_key(module, device):
    """When a mirror module's packed field is stale: a parameter changed in place (its version), was replaced
    (``p.data = t``: its storage), or an optimizer stepped.  An in-place change that bumps no version counter outside an
    optimizer step, such as ``p.data.mul_(2)``, is not seen: rebuild the module's field by hand after one
    (``module._field = None``)."""
    return (str(device), _optimizer_steps, tuple((int(p._version), p.data_ptr()) for p in module.parameters()))


def _get(opt, k, default=None):
    if isinstance(opt, dict):
        return opt.get(k, default)
    return getattr(opt, k, default) if not hasattr(opt, "get") else opt.get(k, default)


class ImplicitNet(nn.Module):
    """networks.py:7-208.  Supported options: cond in {'smpl','frame'}, skip_in == [4], 8 hidden layers of
    256 — the shipped configurations (confs/model/*.yaml:17-50)."""

    def __init__(self, opt, betas=None):
        super().__init__()
        self.opt = opt
        self.d_in = _get(opt, "d_in")
        self.multires = _get(opt, "multires")
        self.cond = _get(opt, "cond")
        self.skip_in = list(_get(opt, "skip_in"))
        dims_h = list(_get(opt, "dims"))
        if self.cond not in ("smpl", "frame") or self.skip_in != [4] or dims_h != [256] * 8:
            raise NotImplementedError("ImplicitNet: only the shipped configuration family is supported "
                                      "(cond smpl|frame, skip_in [4], dims 8x256)")
        self.cond_dim = 69 if self.cond == "smpl" else 32
        d0 = self.d_in * (1 + 2 * self.multires)
        dims = [d0] + dims_h + [_get(opt, "d_out") + _get(opt, "feature_vector_size")]
        self.num_layers = len(dims)
        wn = bool(_get(opt, "weight_norm"))
        for l in range(self.num_layers - 1):
            out_dim = dims[l + 1] - dims[0] if (l + 1) in self.skip_in else dims[l + 1]
            in_dim = dims[l] + (self.cond_dim if l == 0 else 0)
            lin = _Lin(in_dim, out_dim, wn)
            if _get(opt, "init") == "geometry":      # networks.py:55-76
                w = torch.empty(out_dim, in_dim)
                b = torch.zeros(out_dim)
                if l == self.num_layers - 2:
                    w.normal_(np.sqrt(np.pi) / np.sqrt(dims[l]), 0.0001)
                    b.fill_(-_get(opt, "bias"))
                elif l == 0:
                    w.zero_()
                    w[:, :3].normal_(0.0, np.sqrt(2) / np.sqrt(out_dim))
                elif l in self.skip_in:
                    w.normal_(0.0, np.sqrt(2) / np.sqrt(out_dim))
                    w[:, -(dims[0] - 3):] = 0.0
                else:
                    w.normal_(0.0, np.sqrt(2) / np.sqrt(out_dim))
                lin.set_weight(w, b)
            setattr(self, "lin" + str(l), lin)
        self._field = None
        self._field_key = None

    def _dummy_render_sd(self):
        bg = self.cond == "frame"
        sd = {}
        dims = [315, 128, 3] if bg else [270, 256, 256, 256, 256, 3]
        for l in range(len(dims) - 1):
            sd[f"lin{l}.weight"] = torch.zeros(dims[l + 1], dims[l])
            sd[f"lin{l}.bias"] = torch.zeros(dims[l + 1])
        if not bg:
            sd["lin_pose.weight"] = torch.zeros(8, 69)
            sd["lin_pose.bias"] = torch.zeros(8)
        return sd

    def field(self, device):
        key = _field_key(self, device)
        if self._field is None or self._field_key != key:
            self._field = engine.Field({k: v.detach() for k, v in self.state_dict().items()}, self._dummy_render_sd(),
                                       background=(self.cond == "frame"), device=device)
            self._field_key = key
        return self._field

    def forward(self, input, cond, current_epoch=None, person_id=-1):
        if input.ndim == 2:
            input = input.unsqueeze(0)
        nb, npnt, nd = input.shape
        if nb * npnt == 0:
            return input                       # networks.py:131
        assert nb == 1, "the hot path always runs with batch size 1 (multiply.py:208)"
        f = self.field(input.device)
        if _wants_grad(self, input, cond[self.cond]):
            out = engine.ImplicitFunction.apply(f, input.reshape(-1, nd), cond[self.cond], *_effective(self))
            return out.reshape(nb, npnt, -1)
        f.set_cond(cond[self.cond])
        sdf, feat = f.implicit_forward(input.reshape(-1, nd))
        return torch.cat([sdf[:, None], feat], 1).reshape(nb, npnt, -1)


class RenderingNet(nn.Module):
    """networks.py:223-312, modes 'pose_no_view' (foreground) and 'nerf_frame_encoding' (background)."""

    def __init__(self, opt, triplane=None):
        super().__init__()
        self.mode = _get(opt, "mode")
        if self.mode not in ("pose_no_view", "nerf_frame_encoding"):
            raise NotImplementedError("RenderingNet mode %s" % self.mode)
        dims = [_get(opt, "d_in") + _get(opt, "feature_vector_size")] + list(_get(opt, "dims")) + [_get(opt, "d_out")]
        self.multires_view = _get(opt, "multires_view")
        if self.multires_view > 0:
            dims[0] += 3 * 2 * self.multires_view
        if self.mode == "nerf_frame_encoding":
            dims[0] += 32
        if self.mode == "pose_no_view":
            self.lin_pose = nn.Linear(69, 8)
        self.num_layers = len(dims)
        wn = bool(_get(opt, "weight_norm"))
        for l in range(self.num_layers - 1):
            setattr(self, "lin" + str(l), _Lin(dims[l], dims[l + 1], wn))
        self._field = None
        self._field_key = None

    def _dummy_implicit_sd(self):
        bg = self.mode == "nerf_frame_encoding"
        d0, c = (84, 32) if bg else (39, 69)
        dims = [d0] + [256] * 8 + [257]
        sd = {}
        for l in range(9):
            o = dims[l + 1] - d0 if l + 1 == 4 else dims[l + 1]
            i = dims[l] + (c if l == 0 else 0)
            sd[f"lin{l}.weight"] = torch.zeros(o, i)
            sd[f"lin{l}.bias"] = torch.zeros(o)
        return sd

    def field(self, device):
        key = _field_key(self, device)
        if self._field is None or self._field_key != key:
            self._field = engine.Field(self._dummy_implicit_sd(), {k: v.detach() for k, v in self.state_dict().items()},
                                       background=(self.mode == "nerf_frame_encoding"), device=device)
            self._field_key = key
        return self._field

    def forward(self, points, normals, view_dirs, body_pose, feature_vectors, frame_latent_code=None,
                id_latent_code=None, person_id=-1, tri_feat=None):
        if self.mode != "pose_no_view":
            raise NotImplementedError("standalone background colour net: use Multiply.forward / mp_background")
        f = self.field(points.device)
        if _wants_grad(self, points, normals, body_pose, feature_vectors):
            return engine.RenderFunction.apply(f, points, normals, body_pose, feature_vectors, *_effective(self),
                                               self.lin_pose.weight, self.lin_pose.bias)
        f.set_cond(body_pose)
        return f.render_forward(points, normals, feature_vectors)
