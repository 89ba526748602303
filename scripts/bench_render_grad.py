"""Timings of the compositing backward (csrc/composite.cu: mp_composite_backward, mp_final_compose_backward;
csrc/background.cu: mp_bg_composite_backward) against the forward compositor mp_composite; prints one JSON line.

    python scripts/bench_render_grad.py [--steps 20]

Two workloads: the training step (2 persons x 512 rays x 97 samples) and BASELINE configs[1] (2 x 4096 x 193).  Every
ray is hit by both persons (the worst case of the merge); sdf, colours and upstream gradients are seeded random data.
Milliseconds per call from CUDA events around `steps` back-to-back calls after warm-up; the card's name and power limit
are read in the same run.  Writes nothing to disk.
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def _card():
    name = torch.cuda.get_device_name()
    try:
        out = subprocess.run(["nvidia-smi", "-i", str(torch.cuda.current_device()), "--query-gpu=power.limit",
                              "--format=csv,noheader,nounits"], capture_output=True, text=True, timeout=10).stdout.strip()
        limit = float(out)
    except Exception:
        limit = None
    return {"card": name, "power_limit_w": limit}


def _time(fn, steps):
    for _ in range(3):
        fn()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(steps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / steps


def workload(P, R, n, steps):
    from multiply_b200 import _lib as L, engine
    g = torch.Generator(device="cuda").manual_seed(R + n)
    dev = "cuda"
    gr = (L.PersonSampleGrads * P)()
    keep = []
    for p in range(P):
        z = torch.sort(torch.rand(R, n + 1, device=dev, generator=g) * 3 + 0.5, 1)[0]
        t = dict(idx=torch.arange(R, device=dev), z=z.contiguous(),
                 sdf=(torch.rand(R, n, device=dev, generator=g) - 0.5) * 0.4,
                 rgb=torch.rand(R, n, 3, device=dev, generator=g), nrm=torch.rand(R, n, 3, device=dev, generator=g),
                 d_sdf=torch.empty(R, n, device=dev), d_rgb=torch.empty(R, n, 3, device=dev),
                 d_nrm=torch.empty(R, n, 3, device=dev))
        keep.append(t)
        gr[p].d_sdf, gr[p].d_rgb, gr[p].d_normal = (L.ptr(t[k]) for k in ("d_sdf", "d_rgb", "d_nrm"))
    arr = engine.person_samples([(t["idx"], t["z"], t["sdf"], t["rgb"], t["nrm"], R) for t in keep])
    o = {k: torch.empty(*s, device=dev) for k, s in (("fg", (R, 3)), ("nrm", (R, 3)), ("acc", (R,)), ("accp", (R, P)),
                                                     ("bgT", (R,)))}
    u = {k: torch.randn(*v.shape, device=dev, generator=g) for k, v in o.items()}
    u["rgb"] = torch.randn(R, 3, device=dev, generator=g)
    bg_rgb = torch.rand(R, 3, device=dev, generator=g)
    bg_sdf = (torch.rand(R, 32, device=dev, generator=g) - 0.5) * 4
    bg_rgb_s = torch.rand(R, 32, 3, device=dev, generator=g)
    d_bg_sdf, d_bg_rgb_s = torch.empty(R, 32, device=dev), torch.empty(R, 32, 3, device=dev)
    d_fg, d_bgT, d_bg = torch.empty(R, 3, device=dev), torch.empty(R, device=dev), torch.empty(R, 3, device=dev)
    d_beta = torch.empty(1, device=dev)
    ws = L.workspace(L.call("mp_composite_workspace_bytes", R, P), dev)
    wsb = L.workspace(L.call("mp_composite_backward_workspace_bytes", R, P), dev)
    beta = 0.1

    def fwd():
        L.call("mp_composite", arr, P, R, n, beta, o["fg"], o["nrm"], o["acc"], o["accp"], o["bgT"], ws, ws.numel())

    def blend_bwd():
        L.call("mp_final_compose_backward", o["bgT"], bg_rgb, R, u["rgb"], u["fg"], d_fg, d_bgT, d_bg)

    def comp_bwd():
        L.call("mp_composite_backward", arr, P, R, n, beta, d_fg, u["nrm"], u["acc"], u["accp"], d_bgT, gr, d_beta, wsb,
               wsb.numel())

    def bg_bwd():
        L.call("mp_bg_composite_backward", bg_sdf, bg_rgb_s, R, 3.0, None, d_bg, d_bg_sdf, d_bg_rgb_s)

    def all_bwd():
        blend_bwd()
        comp_bwd()
        bg_bwd()
    return {"persons": P, "rays": R, "samples": n,
            "ms_composite_forward": _time(fwd, steps), "ms_final_compose_backward": _time(blend_bwd, steps),
            "ms_composite_backward": _time(comp_bwd, steps), "ms_bg_composite_backward": _time(bg_bwd, steps),
            "ms_backward_total": _time(all_bwd, steps)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    a = ap.parse_args()
    import __graft_entry__  # noqa: F401  (repository root on sys.path)
    torch.cuda.set_device(0)
    rec = dict(_card())
    rec["training_step"] = workload(2, 512, 97, a.steps)
    rec["configs1"] = workload(2, 4096, 193, a.steps)
    print(json.dumps(rec))


if __name__ == "__main__":
    main()
