"""Where the MLP chain kernel (csrc/mlp_tc.cu: tc_chain_kernel) spends its cycles on the benchmark workload: clocks per
tile by phase, for each program, at the default grid and at a reduced one; prints one JSON line.

    python scripts/tc_stalls.py [--steps 20] [--grids default,66]

The workload is the one scripts/bench_tc_chain.py times: bench.py's resident-input render (configs[1]: 2 persons, 4096
rays x 128 samples) on the single-stream schedule, with the same 256 MB L2 flush between steps.  mp_profile_enable(2)
runs the kernel's stall-accounting build, in which lane 0 of every consumer warp and the weight loader's lane sum
clock64 intervals per step kind and phase (include/multiply_b200.h, mp_profile_read_stalls).  For each program the
record gives, per tile (points / 128), the clocks a consumer warp spends (mean over the consumer warps of a CTA):
  full      blocked on the next weight slot (including the drain of a held slot before that wait)
  wgmma     in wgmma waits after a commit, before the extra K-block and at the end of a step
  barrier   in the warpgroup's named barriers
  epilogue  the step's epilogue
  issue     the rest of the steps: MMA issue, descriptors, the extra K-block's staging
  prologue  the tile prologue (embedding)
  elapsed   the warp's whole run, per tile
and for the loader lane its clocks blocked on a free ring position, and the same split per step kind.  The counters
add a few instructions per wait, so the kernel times of this build (also in the record) run slightly above the default
build's.  MP_TC_GRID is read once per process, so every grid runs in a subprocess of its own.  The card's name, power
limit and maximum SM clock are read in the same run.  Writes nothing to disk.
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
HERE = os.path.dirname(os.path.abspath(__file__))
if HERE not in sys.path:
    sys.path.insert(0, HERE)

from bench_tc_chain import KINDS, _card, _grid     # noqa: E402

STEP_KINDS = ("softplus", "softplus_save", "seed", "features", "reverse", "final_grad", "relu")
PHASES = ("step", "full", "wgmma", "barrier", "epilogue", "empty")


def measure(steps):
    from multiply_b200 import engine, scene as S, _lib as L
    torch.cuda.set_device(0)
    dev = torch.device("cuda", 0)
    engine.set_engine("tc")
    # the counters' workspace block is sized only while the stall build is selected: select it before the renderer
    # sizes its workspaces
    L.call("mp_profile_enable", 2)
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
    W, NW = L.MP_STALL_WORDS, L.MP_STALL_WARPS
    clocks = (C.c_ulonglong * (4 * NW * W))()
    pms, pl, pp = (C.c_double * 4)(), (C.c_longlong * 4)(), (C.c_double * 4)()
    L.call("mp_profile_read", pms, pl, pp, 1)
    L.call("mp_profile_read_stalls", clocks, 1)
    for i in range(steps):
        flush.fill_(i & 0xFF)
        r.render(d_inp, d_hits)
    torch.cuda.synchronize()
    L.call("mp_profile_read", pms, pl, pp, 1)
    L.call("mp_profile_read_stalls", clocks, 1)
    L.call("mp_profile_enable", 0)
    grid = _grid()
    rec = {"MP_TC_GRID": os.environ.get("MP_TC_GRID"), "grid": grid, "steps": steps,
           "kernel_ms_per_step_stall_build": sum(pms) / steps}
    P = L.MP_STALL_PHASES
    for k, name in enumerate(KINDS):
        tiles = pp[k] / 128.0
        if tiles == 0:
            continue
        base = k * NW * W

        def word(w, i):
            return clocks[base + w * W + i]

        cons = range(1, NW)

        def mean_cons(i):
            return sum(word(w, i) for w in cons) / len(cons) / tiles

        by_kind = {}
        tot = {ph: 0.0 for ph in PHASES}
        for sk, sname in enumerate(STEP_KINDS):
            d = {ph: mean_cons(sk * P + j) for j, ph in enumerate(PHASES[:5])}
            d["empty"] = word(0, sk * P + 5) / tiles
            if d["step"] == 0 and d["empty"] == 0:
                continue
            d["issue"] = d["step"] - d["full"] - d["wgmma"] - d["barrier"] - d["epilogue"]
            by_kind[sname] = {ph: round(v) for ph, v in d.items()}
            for ph in PHASES:
                tot[ph] += d[ph]
        rec[name] = {"tiles_per_step": tiles / steps, "kernel_ms_per_step_stall_build": pms[k] / steps,
                     "clocks_per_tile": {"full": round(tot["full"]), "wgmma": round(tot["wgmma"]),
                                         "barrier": round(tot["barrier"]), "epilogue": round(tot["epilogue"]),
                                         "issue": round(tot["step"] - tot["full"] - tot["wgmma"] - tot["barrier"]
                                                        - tot["epilogue"]),
                                         "prologue": round(mean_cons(L.MP_STALL_PROLOGUE)),
                                         "elapsed": round(mean_cons(L.MP_STALL_ELAPSED)),
                                         "loader_empty": round(tot["empty"]),
                                         "loader_elapsed": round(word(0, L.MP_STALL_ELAPSED) / tiles)},
                     "by_step_kind": by_kind}
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
    rec["workload"] = "bench.py resident-input render, configs[1], single-stream schedule, stall-accounting build"
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
