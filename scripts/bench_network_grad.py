"""Timings of the networks' first-order backward (csrc/mlp_grad.cu: mp_implicit_backward, mp_render_backward) against
their forward calls (mp_implicit_forward, mp_render_forward); prints one JSON line.

    python scripts/bench_network_grad.py [--n 1048576] [--steps 5]

Three networks at N = 2^20 points on trained-like weights (scene.perturb_networks): the foreground ImplicitNet, the
RenderingNet 'pose_no_view' and the background ImplicitNet.  Milliseconds per call from CUDA events around `steps`
back-to-back calls after warm-up.  The algorithmic FLOP count comes from the layer shapes: the forward's products are
2 out in per point and layer; the backward counts the recompute plus twice that (input and weight gradients).  The card's
name, power limit and SM clock are read in the same run.  Writes nothing to disk.
"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def _card():
    info = {"card": torch.cuda.get_device_name()}
    try:
        out = subprocess.run(["nvidia-smi", "-i", str(torch.cuda.current_device()),
                              "--query-gpu=power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader,nounits"],
                             capture_output=True, text=True, timeout=10).stdout.strip().split(",")
        info.update(power_limit_w=float(out[0]), sm_clock_mhz=float(out[1]), sm_clock_max_mhz=float(out[2]))
    except Exception:
        info.update(power_limit_w=None, sm_clock_mhz=None, sm_clock_max_mhz=None)
    return info


def _time(fn, steps):
    for _ in range(2):
        fn()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(steps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / steps


def _forward_flops(shapes, first_k=None):
    """2 out in per point over the layers (layer 0 over first_k inputs when the cond is folded into its bias)."""
    return sum(2 * o * (first_k if (l == 0 and first_k) else i) for l, (o, i) in enumerate(shapes))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=1 << 20)
    ap.add_argument("--steps", type=int, default=5)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_network_grad: no CUDA device")
    from multiply_b200 import engine, scene as S, _lib as L
    engine.set_engine("tc")
    N, dev = a.n, "cuda"
    sc = S.make_scene(P=1, S=16, seed=42, weights="trained")
    p = sc["persons"][0]
    fg = engine.Field(p["implicit"], p["render"])
    fg.set_cond(p["cond"])
    bg = engine.Field(sc["bg_implicit"], sc["bg_render"], background=True)
    bg.set_cond(sc["frame_code"])
    g = torch.Generator(device=dev).manual_seed(0)
    x3 = torch.rand(N, 3, device=dev, generator=g) * 2 - 1
    x4 = torch.cat([x3, torch.rand(N, 1, device=dev, generator=g) / 3], 1).contiguous()
    d_sdf, d_feat = torch.randn(N, device=dev, generator=g), torch.randn(N, 256, device=dev, generator=g)
    nrm = torch.nn.functional.normalize(torch.randn(N, 3, device=dev, generator=g), dim=1).contiguous()
    feat = torch.randn(N, 256, device=dev, generator=g) * 0.5
    d_rgb = torch.randn(N, 3, device=dev, generator=g)
    rows = {}

    def implicit(name, f, x, E):
        ws_f = L.workspace(L.call("mp_mlp_workspace_bytes", N), dev)
        sdf, ft = torch.empty(N, device=dev), torch.empty(N, 256, device=dev)
        fwd = _time(lambda: L.call("mp_implicit_forward", f.handle, x, N, sdf, ft, ws_f, ws_f.numel()), a.steps)
        del ws_f
        bwd = _time(lambda: f.implicit_backward(x, d_sdf, d_feat), a.steps)
        flops = _forward_flops(f.imp_shapes, E) * N
        rows[name] = dict(forward_ms=fwd, backward_ms=bwd, forward_tflops=flops / fwd * 1e-9,
                          backward_tflops=3 * flops / bwd * 1e-9)

    implicit("implicit_fg", fg, x3, 39)
    torch.cuda.empty_cache()
    ws_r = L.workspace(L.call("mp_mlp_workspace_bytes", N), dev)
    rgb = torch.empty(N, 3, device=dev)
    fwd = _time(lambda: L.call("mp_render_forward", fg.handle, x3, nrm, feat, N, rgb, ws_r, ws_r.numel()), a.steps)
    del ws_r
    bwd = _time(lambda: fg.render_backward(x3, nrm, feat, d_rgb), a.steps)
    flops = _forward_flops(fg.ren_shapes) * N
    rows["render_fg"] = dict(forward_ms=fwd, backward_ms=bwd, forward_tflops=flops / fwd * 1e-9,
                             backward_tflops=3 * flops / bwd * 1e-9)
    torch.cuda.empty_cache()
    implicit("implicit_bg", bg, x4, 84)
    print(json.dumps(dict(metric="network_backward", n=N, steps=a.steps, **_card(), **rows)))


if __name__ == "__main__":
    main()
