"""GPU diagnostic: where does the rendered-normal error of the tensor-core engine come from?
(1) per-point sdf / gradient of mp_implicit_forward_grad (tc, simt) against the fp64 evaluation of the same
    weights (scripts/numerics_study.py) on points around the surface and near the canonical origin;
(2) per-sample normals of a rendered batch against the oracle, worst samples listed with |grad|."""
import os, sys, json
import numpy as np
import torch
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "scripts"))
import numerics_study as ns
from multiply_b200 import scene as S, engine
from oracle import port

out = {}
sc = S.make_scene(P=2, S=64, seed=42)
person, cfg = sc["persons"][0], dict(sc["cfg"], multires=6)
g = torch.Generator().manual_seed(5)
dirs = torch.nn.functional.normalize(torch.randn(4096, 3, generator=g), dim=1)
xs = dirs * (0.6 + 0.1 * (torch.rand(4096, 1, generator=g) * 2 - 1))
xo = (torch.rand(4096, 3, generator=g) * 2 - 1) * 0.3
f = engine.Field(person["implicit"], person["render"]); f.set_cond(person["cond"])
for tag, x in (("surface", xs), ("origin", xo)):
    t = ns.chain(person, cfg, x, "fp64")
    t32 = ns.chain(person, cfg, x, "fp32")
    for eng in ("simt", "tc"):
        engine.set_engine(eng)
        sdf, feat, grad = f.implicit_forward(x, want_grad=True)
        torch.cuda.synchronize()
        es = float((sdf.cpu().double() - t["sdf"]).abs().max())
        eg = (grad.cpu().double() - t["grad"]).abs().max(1)[0]
        rel = eg / t["grad"].norm(dim=1)
        out["%s_%s" % (tag, eng)] = dict(sdf=es, grad=float(eg.max()), grad_rel=float(rel.max()), grad_mean=float(eg.mean()))
        print(tag, eng, out["%s_%s" % (tag, eng)])
    e32 = (t32["grad"] - t["grad"]).abs().max(1)[0]
    print(tag, "torch fp32", float((t32["sdf"] - t["sdf"]).abs().max()), float(e32.max()), float(e32.mean()))

# rendered batch: per-sample normals vs the oracle
sc = S.make_scene(P=2, S=128, seed=42)
inp = S.make_rays(sc, 4096, seed=1234, region="boxes")
sub = dict(uv=inp["uv"][:, :48].contiguous(), pose=inp["pose"], intrinsics=inp["intrinsics"])
hits = S.make_hit_lists(sc, sub)
ref = port.multiply_forward(sc, sub, hits, return_samples=True)
for eng in ("simt", "tc"):
    engine.set_engine(eng)
    o = engine.Renderer(sc).render(sub, hits, debug=True)
    torch.cuda.synchronize()
    print(eng, "rendered normal linf", float((o["normal_values"].cpu() - ref["normal_values"]).abs().max()),
          "rgb", float((o["rgb_values"].cpu() - ref["rgb_values"]).abs().max()))
    for p in range(2):
        z = o["z_vals_%d" % p].cpu()[:, :-1]
        same = (z - ref["_z_vals"][p]).abs() < 1e-6
        keys = [k for k in ref if k.startswith("_")]
        if p == 0 and eng == "simt":
            print("oracle sample keys", keys)
        if "_normals" in ref:
            dn = (o["normals_%d" % p].cpu() - ref["_normals"][p].reshape(z.shape[0], -1, 3)).abs().max(-1)[0]
            same = same & (ref["_sdf"][p].reshape(z.shape) != 4.0)
            dn = torch.where(same, dn, torch.zeros_like(dn))
            print(eng, "person", p, "per-sample normal max", float(dn.max()), "mean", float(dn.mean()),
                  "count>1e-4", int((dn > 1e-4).sum()), "of", int(same.sum()))
os.makedirs(os.path.join(ROOT, "profiles"), exist_ok=True)
json.dump(out, open(os.path.join(ROOT, "profiles", "normal_diag_%s.json" % os.environ.get("MP_TC_RZ_SCALE", "default")), "w"), indent=1)
