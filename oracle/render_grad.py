"""Differentiable restatement of the compositing stages of Multiply.forward, for gradient checks.

    composite(...)            the flatten / sort / nerfacc block, multiply.py:427-480
    bg_volume_rendering(...)  Multiply.bg_volume_rendering with AbsDensity, multiply.py:682-696, and the sum of :539
    blend(...)                rgb_values / fg_rgb_values, multiply.py:544-545, :590

Everything is torch, in the dtype of the inputs (float64 for the references of the GPU tests), so torch autograd gives
the gradient definition, kinks included: sign(0) = 0, d|s|/ds = sign(s); expm1's derivative is exp (see _expm1).  Tie order on equal t_end is (person,
sample) ascending, as oracle/port.py and the kernels use.  nerfacc's exclusive scan (render_weight_from_density) becomes
a per-ray cumsum over a [rays, max samples] table padded with zeros; its backward is a definition, unpinned upstream
like its forward.  oracle/port.py stays the value reference; tests/test_render_grad_oracle.py checks that this restatement
run in float32 reproduces its values.
"""
import numpy as np
import torch


def _expm1(x):
    """torch.expm1 whose derivative is exp(x).  torch's own backward is expm1(x) + 1, which is exactly 0 once expm1(x)
    rounds to -1 (|sdf| / beta > 37 in float64, > 17 in float32): this restatement keeps the analytic tail the
    kernels compute instead of that rounding artefact."""
    x0 = x.detach()
    return torch.expm1(x0) + torch.exp(x0) * (x - x0)


def laplace_density(sdf, beta):
    """LaplaceDensity.density_func, lib/model/density.py:20-25 (beta: a tensor, differentiable)."""
    alpha = 1 / beta
    return alpha * (0.5 + 0.5 * sdf.sign() * _expm1(-sdf.abs() / beta))


def merged_order(persons, n, reverse=False):
    """Flattened samples of every person sorted by (ray, t_end, person, sample) -- (ray, t_end, -person, -sample) with
    `reverse`.  persons: list of dict(idx [R_p] int64, z [R_p, n+1] (numpy or tensor)).  Returns the dict of numpy
    columns ray / pid / row / smp in merged order."""
    cols = {k: [] for k in ("ray", "pid", "row", "smp", "te")}
    for p, d in enumerate(persons):
        idx = np.asarray(d["idx"], np.int64)
        Rp = idx.shape[0]
        z = d["z"].detach().cpu().numpy() if torch.is_tensor(d["z"]) else np.asarray(d["z"])
        cols["ray"].append(np.repeat(idx, n))
        cols["pid"].append(np.full(Rp * n, p))
        cols["row"].append(np.repeat(np.arange(Rp), n))
        cols["smp"].append(np.tile(np.arange(n), Rp))
        cols["te"].append(z[:, 1:].reshape(-1).astype(np.float64))
    c = {k: np.concatenate(v) for k, v in cols.items()}
    sg = -1 if reverse else 1
    o = np.lexsort((sg * c["smp"], sg * c["pid"], c["te"], c["ray"]))
    return {k: v[o] for k, v in c.items()}


def composite(persons, R, n, beta, reverse=False):
    """multiply.py:427-480.  persons: list of dict(idx [R_p] int64, z [R_p, n+1], sdf [R_p, n], rgb / nrm [R_p, n, 3])
    with z / sdf / rgb / nrm torch tensors of one dtype (any may require grad); beta a 0-d tensor.
    Returns fg_rgb [R,3], normal [R,3], acc [R], acc_person [R,P], bg_T [R] (bg_T = 1 for rays no person hits)."""
    P = len(persons)
    dt = persons[0]["sdf"].dtype
    c = merged_order(persons, n, reverse)
    M = c["ray"].size
    counts = np.bincount(c["ray"], minlength=R) if M else np.zeros(R, np.int64)
    starts = np.cumsum(counts) - counts
    pos = np.arange(M) - starts[c["ray"]]
    Kmax = max(int(counts.max()) if R else 0, 1)
    # every per-sample tensor in merged order: flat index of (person, row, sample) in the concatenated person tables
    base = np.cumsum([0] + [d["sdf"].numel() for d in persons])[:-1]
    fi = torch.from_numpy(base[c["pid"]] + c["row"] * n + c["smp"])

    def gather(key, width):
        return torch.cat([d[key].reshape(-1, width) for d in persons], 0)[fi]
    ts = torch.cat([d["z"][:, :-1].reshape(-1) for d in persons])[fi]
    te = torch.cat([d["z"][:, 1:].reshape(-1) for d in persons])[fi]
    sdf = gather("sdf", 1)[:, 0]
    rgb, nrm = gather("rgb", 3), gather("nrm", 3)
    sd = laplace_density(sdf, beta) * (te - ts)
    ray_t, pos_t = torch.from_numpy(c["ray"]), torch.from_numpy(pos)
    X = torch.zeros(R, Kmax, dtype=dt).index_put((ray_t, pos_t), sd)
    E = torch.cat([torch.zeros(R, 1, dtype=dt), torch.cumsum(X[:, :-1], 1)], 1)      # exclusive per-ray prefix
    T = torch.exp(-E)
    W = T * (1 - torch.exp(-X))
    w = W[ray_t, pos_t]
    fg = torch.zeros(R, 3, dtype=dt).index_add(0, ray_t, w[:, None] * rgb)
    normal = torch.zeros(R, 3, dtype=dt).index_add(0, ray_t, w[:, None] * nrm)
    acc = torch.zeros(R, dtype=dt).index_add(0, ray_t, w)
    accp = torch.zeros(R * P, dtype=dt).index_add(0, ray_t * P + torch.from_numpy(c["pid"]), w).reshape(R, P)
    last = torch.from_numpy(np.maximum(counts - 1, 0))
    bgT = torch.where(torch.from_numpy(counts > 0), T[torch.arange(R), last], torch.ones(R, dtype=dt))
    return fg, normal, acc, accp, bgT


def bg_linspace32():
    """torch.linspace(0, 1, 32) in fp32 (ATen's two-sided fma form, as mp_linspace_host / bg_linspace32)."""
    step = np.float32(1.0) / np.float32(31.0)
    i = np.arange(32)
    lo = (np.float64(step) * i).astype(np.float32)              # fma(step, i, 0): one rounding
    hi = (1.0 - np.float64(step) * (31 - i)).astype(np.float32)  # fma(-step, 31 - i, 1): one rounding
    return np.where(i < 16, lo, hi).astype(np.float32)


def bg_depths(R, bound, t_rand=None):
    """Inverse-sphere depths of the background pass in the flipped order the networks see (multiply.py:482-484, :516;
    ray_sampler.py:215-218 with the jittered UniformSampler when t_rand [R,32] is given), float32 [R,32], rounded step by
    step as the kernels' bg_depth."""
    z = np.broadcast_to(bg_linspace32(), (R, 32)).astype(np.float32)
    if t_rand is not None:
        t = np.asarray(t_rand, np.float32).reshape(R, 32)
        zl = bg_linspace32()
        mid = (np.float32(0.5) * (zl[1:] + zl[:-1])).astype(np.float32)
        lower = np.concatenate([zl[:1], mid]).astype(np.float32)
        upper = np.concatenate([mid, zl[-1:]]).astype(np.float32)
        z = (lower + ((upper - lower) * t).astype(np.float32)).astype(np.float32)
    inv = np.float32(1.0 / bound)
    return np.ascontiguousarray((z * inv).astype(np.float32)[:, ::-1])


def bg_volume_rendering(z_bg, bg_sdf, bg_rgb_samples=None):
    """multiply.py:682-696 with AbsDensity (density.py:32-34): z_bg [R,32] flipped depths, bg_sdf [R,32] -> weights
    [R,32]; with bg_rgb_samples [R,32,3] also the bg_rgb_values [R,3] of :539."""
    dt = bg_sdf.dtype
    dens = torch.abs(bg_sdf)
    d = z_bg[:, :-1] - z_bg[:, 1:]
    d = torch.cat([d, torch.full((d.shape[0], 1), 1e10, dtype=dt)], -1)
    fe = d * dens
    sh = torch.cat([torch.zeros(d.shape[0], 1, dtype=dt), fe[:, :-1]], -1)
    w = (1 - torch.exp(-fe)) * torch.exp(-torch.cumsum(sh, -1))
    if bg_rgb_samples is None:
        return w
    return w, torch.sum(w.unsqueeze(-1) * bg_rgb_samples, 1)


def blend(fg_rgb, bg_T, bg_rgb=None):
    """multiply.py:540-545, :590: (rgb_values, fg_rgb_values); bg_rgb None -> white."""
    b = torch.ones_like(fg_rgb) if bg_rgb is None else bg_rgb
    return fg_rgb + bg_T.unsqueeze(-1) * b, fg_rgb + bg_T.unsqueeze(-1) * torch.ones_like(fg_rgb)
