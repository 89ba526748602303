"""Timings of the canonical-mesh kernels (csrc/mesh.cu, multiply.py:153-167) on the GPU; prints one JSON line.

    python scripts/bench_mesh.py [--steps 10]

Times the surface-flag kernel at the training workload (512 rays x 97 samples x 2 persons, confs/dataset num_sample and
the 64 + 32 + 1 samples per ray), the exact distance and inside test on 1 M points against the default (SMPL-sized)
and a large synthetic mesh, and what the flags add to a training-forward step (the same step without a mesh), and
records the card's name and power limit read in the same run.  Writes nothing to disk.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def _card():
    """Name and power limit of the card the timings ran on (read in the same run)."""
    name = torch.cuda.get_device_name()
    try:
        idx = torch.cuda.current_device()
        out = subprocess.run(["nvidia-smi", "-i", str(idx), "--query-gpu=power.limit", "--format=csv,noheader,nounits"],
                             capture_output=True, text=True, timeout=10).stdout.strip()
        limit = float(out)
    except Exception:
        limit = None
    return {"card": name, "power_limit_w": limit}


def mesh_query(dev, steps=10):
    """The timing record (milliseconds per call, CUDA events; grid builds by host clock including the size read-back)."""
    from multiply_b200 import engine, scene as S
    from multiply_b200.model.ray_sampler import ErrorBoundSampler
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)

    def timed(fn, n):
        fn()
        torch.cuda.synchronize()
        e0.record()
        for _ in range(n):
            fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / n

    rec = _card()
    g = torch.Generator().manual_seed(0)
    meshes = {}
    for name, step in (("default", 0.033), ("large", 0.007)):
        v, f = S.make_body_mesh(100, step=step)
        t0 = time.time()
        m = engine.CanonicalMesh(v, f, device=dev)
        torch.cuda.synchronize()
        build_ms = (time.time() - t0) * 1000.0
        meshes[name] = m
        lo, hi = v.min(0)[0], v.max(0)[0]
        n = 1 << 20
        band = v[torch.randint(0, v.shape[0], (n // 2,), generator=g)] + 0.03 * torch.randn(n // 2, 3, generator=g)
        box = lo - 0.1 + (hi - lo + 0.2) * torch.rand(n - n // 2, 3, generator=g)
        pts = torch.cat([band, box]).to(dev)
        rec[name] = {"faces": f.shape[0], "grid": list(m.grid_dims), "build_ms_host_clock": build_ms,
                     "points": n, "distance_ms": timed(lambda: m.distance(pts), 5),
                     "check_sign_ms": timed(lambda: m.check_sign(pts), 5)}
    # surface flags at the training workload: samples along 512 rays through the canonical body, per person
    v, _ = S.make_body_mesh(100)
    lo, hi = v.min(0)[0], v.max(0)[0]
    o = lo + (hi - lo) * torch.rand(512, 1, 3, generator=g)
    d = torch.nn.functional.normalize(torch.randn(512, 1, 3, generator=g), dim=-1)
    x = (o + torch.linspace(-0.6, 0.6, 97)[None, :, None] * d).reshape(-1, 3).to(dev)
    rec["surface_flags_ms_2_persons"] = timed(lambda: [meshes["default"].surface_flags(x, 97) for _ in range(2)], 20)
    # training-forward step with and without the flags (S = 64: 97 samples per ray, 512 rays, 2 persons)
    sc = S.make_scene(P=2, S=64, seed=42)
    r = engine.Renderer(sc, device=dev)
    inp = S.make_rays(sc, 512, seed=3, region="boxes")
    hits = S.make_hit_lists(sc, inp)
    smp = ErrorBoundSampler(3.0, inverse_sphere_bg=True, **{k: sc["cfg"][k] for k in (
        "near", "N_samples", "N_samples_eval", "N_samples_extra", "eps", "beta_iters", "max_total_iters", "add_tiny")})
    torch.manual_seed(1)
    rngs = [{k: v for k, v in smp.draw_training_rng(h.numel()).items() if k != "states"} for h in hits]
    tb = torch.rand(512, 32)
    cano = [engine.CanonicalMesh(*S.make_body_mesh(100 + p), device=dev) for p in range(2)]
    base = dict(rng=rngs, t_rand_bg=tb)
    flags = dict(base, meshes=cano, threshold=0.05)
    t_off, t_on = [], []
    for _ in range(3):              # alternate the two variants
        t_off.append(timed(lambda: r.render(inp, hits, train=base), steps))
        t_on.append(timed(lambda: r.render(inp, hits, train=flags), steps))
    rec["train_step_ms_without_mesh"] = float(np.median(t_off))
    rec["train_step_ms_with_flags"] = float(np.median(t_on))
    rec["flags_add_ms"] = rec["train_step_ms_with_flags"] - rec["train_step_ms_without_mesh"]
    return rec


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "bench_mesh.py times GPU kernels and needs a GPU"
    torch.cuda.set_device(0)
    print(json.dumps({"mesh_query": mesh_query(torch.device("cuda", 0), a.steps)}))
