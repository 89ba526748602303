"""Times the body-model backward calls against their forwards, and the same backward as torch fp32 autograd of
oracle/port.py's restatement on the same GPU, with CUDA events after warm-up:

  * mp_deform_inverse vs mp_deform_inverse_backward at 1e5 and 1.6e6 points (a training step's samples, BASELINE configs[1]);
  * mp_deform_forward_jac vs mp_deform_forward_jac_backward at 1e5 and 3e5 canonical-mesh-sized point sets;
  * mp_smpl_forward vs mp_smpl_backward at V = 6890 (d_verts and d_tfs).

    python scripts/bench_body_grad.py [--iters 50]

Prints the card name and power limit with the numbers, one JSON line at the end."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from multiply_b200 import engine, scene as S          # noqa: E402
from multiply_b200.model.smpl import SMPLServer        # noqa: E402


def timed(fn, iters):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:                # noqa: BLE001
        q = "%s (nvidia-smi: %s)" % (torch.cuda.get_device_name(0), e)
    return q


def torch_inverse_backward(x, W, tfs, idx, u):
    """port.skinning(inverse=True) in fp32 torch autograd with the nearest-vertex weights given."""
    tv = tfs.detach().clone().requires_grad_(True)
    xv = x.detach().clone().requires_grad_(True)
    w = W[idx][None]
    A = torch.einsum("bpn,bnij->bpij", w, tv[None])
    xh = torch.nn.functional.pad(xv[None], (0, 1), value=1.0)
    xc = torch.einsum("bpij,bpj->bpi", A.inverse(), xh)[0, :, :3]
    torch.autograd.grad((xc * u).sum(), [xv, tv])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a GPU"
    torch.cuda.set_device(0)
    info = card()
    print("card:", info)
    res = {"card": info}
    sm = S.make_smpl_model(300)
    srv = SMPLServer(model=sm)
    rng = np.random.RandomState(0)
    p = dict(scale=torch.tensor([1.0], device="cuda"), transl=torch.zeros(1, 3, device="cuda"),
             thetas=torch.from_numpy(rng.normal(0, 0.3, (1, 72)).astype(np.float32)).cuda(),
             betas=torch.from_numpy(rng.normal(0, 1, (1, 10)).astype(np.float32)).cuda())
    o = srv(**p)
    body = engine.Body(srv.verts_c[0], srv.weights[0], cano_cell=0.1001)
    body.set_pose(o["smpl_verts"][0], o["smpl_tfs"][0])
    verts_p = o["smpl_verts"][0]
    for N in (100_000, 1_600_000):
        x = verts_p[torch.randint(0, verts_p.shape[0], (N,), device="cuda")] + 0.05 * torch.randn(N, 3, device="cuda")
        u = torch.randn(N, 3, device="cuda")
        f = timed(lambda: body.deform_inverse(x), args.iters)
        bwd = timed(lambda: body.deform_inverse_backward(x, u), args.iters)
        idx = torch.randint(0, verts_p.shape[0], (N,), device="cuda")
        tb = timed(lambda: torch_inverse_backward(x, body.weights, body.tfs, idx, u), max(5, args.iters // 5))
        res["inverse_%d" % N] = dict(forward_ms=f, backward_ms=bwd, ratio=bwd / f, torch_fp32_autograd_ms=tb)
        print("deform_inverse N=%d: forward %.3f ms, backward %.3f ms (x%.2f), torch fp32 autograd %.3f ms (weights given)"
              % (N, f, bwd, bwd / f, tb))
    vc = srv.verts_c[0]
    for N in (100_000, 300_000):
        xc = vc[torch.randint(0, vc.shape[0], (N,), device="cuda")] + 0.01 * torch.randn(N, 3, device="cuda")
        u, uj = torch.randn(N, 3, device="cuda"), torch.randn(N, 9, device="cuda")
        f = timed(lambda: body.forward_jac(xc), args.iters)
        bwd = timed(lambda: body.forward_jac_backward(xc, u, uj), args.iters)
        res["forward_jac_%d" % N] = dict(forward_ms=f, backward_ms=bwd, ratio=bwd / f)
        print("forward_jac N=%d: forward %.3f ms, backward %.3f ms (x%.2f)" % (N, f, bwd, bwd / f))
    dv, dt = torch.randn(srv.V, 3, device="cuda"), torch.randn(24, 4, 4, device="cuda")
    ins = tuple(t.reshape(-1).contiguous() for t in (p["scale"], p["transl"], p["thetas"], p["betas"]))
    f = timed(lambda: srv._run(*ins, False), args.iters)
    bwd = timed(lambda: srv._backward(ins, False, dv, dt), args.iters)
    res["smpl_6890"] = dict(forward_ms=f, backward_ms=bwd, ratio=bwd / f)
    print("smpl V=6890: forward %.3f ms, backward %.3f ms (x%.2f)" % (f, bwd, bwd / f))
    print(json.dumps(res))


if __name__ == "__main__":
    main()
