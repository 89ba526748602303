"""Mesh extraction timing (generate_mesh, lib/utils/mesh.py:78-132) per person on trained-like weights.

    python scripts/bench_mesh_extract.py [--reps 5] [--res-up 2 3 4]

Per person and res_up (res_init 32): the device call (MISE + marching cubes + largest component; host clock around a
synchronised call, warmed up, median of --reps), the points MISE evaluated against (R+1)^3, the dense alternative
(mp_sdf_grid + device marching cubes on the whole lattice), and the reference's compiled MISE loop driven by the
mirror's Multiply.query_oc (oracle/_ref, when built).  skimage and trimesh are not available, so the reference's
marching cubes and component steps have no timing.  Prints the card's name and power limit with the numbers.
"""
import argparse
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from multiply_b200 import engine, scene as S          # noqa: E402
from multiply_b200.utils import mesh as umesh         # noqa: E402
from oracle import build_ref, mesh_extract as M       # noqa: E402


def timed(fn, reps):
    fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        t = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        ts.append(time.perf_counter() - t)
    return float(np.median(ts))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--res-up", type=int, nargs="+", default=[2, 3, 4])
    ap.add_argument("--no-reference", action="store_true")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "needs a GPU"
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    print("card: %s" % q.stdout.strip())
    engine.set_engine("tc")
    sc = S.make_scene(P=2, S=16, seed=42, weights="trained")
    m = S.mirror_model(sc)
    mod = None if a.no_reference else build_ref.load_mise()
    for pid, person in enumerate(sc["persons"]):
        cond = person["cond"].cuda()
        center, extent, pad = umesh.bounds(person["verts_c"])
        f = m._ensure_renderer(torch.device("cuda", 0)).fields[pid]
        f.set_cond(cond)
        for up in a.res_up:
            R = 32 << up
            out = {}
            t_dev = timed(lambda: out.setdefault("r", f.extract_mesh(center, extent, 32, up, 0.0, pad)), a.reps)
            v, fc, n = f.extract_mesh(center, extent, 32, up, 0.0, pad)
            t_dense = timed(lambda: engine.marching_cubes(f.sdf_grid(center, extent, R, pad), 0.0, center, extent, pad),
                            a.reps)
            line = ("person %d res_up %d (R=%d): device %.1f ms | evaluated %d of %d (%.2f %%) | dense sdf_grid + "
                    "marching cubes %.1f ms | V %d F %d" % (pid, up, R, 1e3 * t_dev, n, (R + 1) ** 3,
                                                            100.0 * n / (R + 1) ** 3, 1e3 * t_dense, v.shape[0],
                                                            fc.shape[0]))
            if mod is not None:
                def values_at(idx):
                    pts = torch.from_numpy(umesh.lattice_points(np.asarray(idx), R, center, extent)).cuda()
                    occ = torch.cat([m.query_oc(b, {"smpl": cond}, pid)["occ"] for b in torch.split(pts, 5000, dim=0)])
                    return occ[:, 0].double().cpu().numpy()
                t = time.perf_counter()
                M.reference_mise(mod, values_at, 32, up, 0.0)
                line += " | reference MISE loop %.1f ms" % (1e3 * (time.perf_counter() - t))
            print(line, flush=True)


if __name__ == "__main__":
    main()
