"""Mirror of /root/reference/code/lib/model/density.py (LaplaceDensity, AbsDensity)."""
import torch
import torch.nn as nn

from .. import _lib as L


class Density(nn.Module):
    """density.py:4-12: every entry of ``params_init`` becomes a scalar parameter of that name (``beta``); calling the
    module evaluates ``density_func``."""

    def __init__(self, params_init=None):
        super().__init__()
        for name, value in dict(params_init or {}).items():
            self.register_parameter(name, nn.Parameter(torch.as_tensor(float(value), dtype=torch.float32)))

    def forward(self, sdf, beta=None):
        return self.density_func(sdf, beta=beta)


class LaplaceDensity(Density):
    """density.py:15-29: alpha * Laplace(0, beta).cdf(-sdf)."""

    def __init__(self, params_init=None, beta_min=0.0001):
        super().__init__(params_init=params_init)
        self.beta_min = float(beta_min)

    def get_beta(self):
        return self.beta.abs() + self.beta_min

    def density_func(self, sdf, beta=None):
        if beta is None:
            beta = self.get_beta()
        if torch.is_tensor(beta) and beta.numel() > 1:
            raise NotImplementedError("per-ray beta lives inside the fused sampler (mp_sample_rays)")
        b = float(beta.detach()) if torch.is_tensor(beta) else float(beta)
        s = L.dev(sdf, sdf.device)
        out = torch.empty_like(s)
        L.call("mp_laplace_density", s, s.numel(), b, out)
        return out.reshape(sdf.shape)


class AbsDensity(Density):
    """density.py:32-34 (background): |sdf|, a single elementwise op that only occurs fused inside mp_background."""

    def density_func(self, sdf, beta=None):
        return torch.abs(sdf)
