"""CTA time per tile of the MLP chain kernel (csrc/mlp_tc.cu: tc_chain_kernel) on the benchmark workload, at the default
grid and at a reduced one; prints one JSON line.

    python scripts/bench_tc_chain.py [--steps 20] [--grids default,66]

The workload is bench.py's resident-input render (configs[1]: 2 persons, 4096 rays x 128 samples) on the single-stream
schedule, with the kernel's per-launch CUDA events (mp_profile_enable / mp_profile_read) as bench.py's `roofline`
uses them, and the same 256 MB L2 flush between steps.  MP_TC_GRID is read once per process, so every grid runs in a
subprocess of its own.  For each program kind the record gives the kernel time per step and the CTA time per tile,
kernel_ms x grid / tiles (tiles = points / 128): at a fixed per-SM rate it does not depend on the grid, so a lower
value at the reduced grid means the CTAs contend for a shared resource (L2 / HBM bandwidth).  The partial last round of
a launch weighs more at the larger grid, and launches with fewer tiles than CTAs (the sampler's sdf-only lists)
overstate it.  The card's name, power limit and maximum SM clock are read in the same run.  Writes nothing to disk.
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

KINDS = ("sdf_only", "forward", "shade", "background")


def _card():
    try:
        out = subprocess.run(["nvidia-smi", "-i", str(torch.cuda.current_device()),
                              "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader,nounits"],
                             capture_output=True, text=True, timeout=10).stdout.strip().split(",")
        return {"card": out[0].strip(), "power_limit_w": float(out[1]), "sm_max_mhz": float(out[2])}
    except Exception:
        return {"card": torch.cuda.get_device_name(), "power_limit_w": None, "sm_max_mhz": None}


def _grid():
    """Persistent CTAs of a launch with at least as many tiles (csrc/mlp_tc.cu tc_launch): one per SM, capped by
    MP_TC_GRID.  A launch with fewer tiles than that runs one CTA per tile, which this figure does not account for."""
    from multiply_b200 import _lib as L
    g = L.call("mp_device_sm_count")
    env = int(os.environ.get("MP_TC_GRID", "0") or 0)
    return min(g, env) if env > 0 else g


def measure(steps):
    from multiply_b200 import engine, scene as S, _lib as L
    torch.cuda.set_device(0)
    dev = torch.device("cuda", 0)
    engine.set_engine("tc")
    sc, _, _ = S.make_smpl_scene(P=2, S=128, seed=42, device=dev)
    inp = S.make_rays(sc, 4096, seed=1234, region="boxes")
    hits = S.make_hit_lists(sc, inp)
    r = engine.Renderer(sc, device=dev)
    d_inp = {k: v.to(dev) for k, v in inp.items()}
    d_hits = [h.to(dev) for h in hits]
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    L.call("mp_set_streams", 0)
    for _ in range(3):
        r.render(d_inp, d_hits)
    torch.cuda.synchronize()
    L.call("mp_profile_enable", 1)
    for i in range(steps):
        flush.fill_(i & 0xFF)
        r.render(d_inp, d_hits)
    torch.cuda.synchronize()
    L.call("mp_profile_enable", 0)
    pms, pl, pp = (C.c_double * 4)(), (C.c_longlong * 4)(), (C.c_double * 4)()
    L.call("mp_profile_read", pms, pl, pp, 1)
    grid = _grid()
    rec = {"MP_TC_GRID": os.environ.get("MP_TC_GRID"), "grid": grid, "steps": steps,
           "kernel_ms_per_step": sum(pms) / steps}
    for k, name in enumerate(KINDS):
        tiles = pp[k] / 128.0
        rec[name] = {"kernel_ms_per_step": pms[k] / steps, "launches_per_step": pl[k] / steps,
                     "tiles_per_step": tiles / steps,
                     "cta_us_per_tile": 1000.0 * pms[k] * grid / tiles if tiles > 0 else None}
    return rec


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--grids", default="default,66", help="comma-separated MP_TC_GRID values ('default': unset)")
    ap.add_argument("--child", action="store_true", help=argparse.SUPPRESS)
    a = ap.parse_args()
    if a.child:
        print(json.dumps(measure(a.steps)))
        return
    torch.cuda.set_device(0)
    rec = dict(_card())
    rec["workload"] = "bench.py resident-input render, configs[1], single-stream schedule"
    rec["runs"] = []
    for g in a.grids.split(","):
        env = dict(os.environ)
        env.pop("MP_TC_GRID", None)
        if g != "default":
            env["MP_TC_GRID"] = g
        p = subprocess.run([sys.executable, os.path.abspath(__file__), "--child", "--steps", str(a.steps)], env=env,
                           cwd=ROOT, capture_output=True, text=True)
        if p.returncode != 0:
            raise RuntimeError("grid %s failed:\n%s" % (g, p.stdout[-2000:] + p.stderr[-4000:]))
        rec["runs"].append(json.loads(p.stdout.strip().splitlines()[-1]))
    print(json.dumps(rec))


if __name__ == "__main__":
    main()
