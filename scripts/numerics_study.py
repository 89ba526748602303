"""CPU numerics study of the tensor-core MLP chain (no GPU needed).

Emulates the operand formats of csrc/mlp_tc.cu in torch: every layer product A.W^T is evaluated from
fp16 (or bf16) hi/lo pairs of A and of 2^s W with a chosen subset of the four cross terms, products
exact (fp64 matmul of the rounded operands), result rounded to fp32.  Compares SDF, d sdf/d x, the
normal and RGB of one foreground field against (a) the fp64 evaluation of the same network ("truth")
and (b) the fp32 torch evaluation (what the reference / oracle computes).

    python scripts/numerics_study.py            # prints a table, writes profiles/numerics.json
"""
import json
import os
import sys
import numpy as np
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from multiply_b200 import scene as S      # noqa: E402
from oracle import port                    # noqa: E402


def split(x, dt, n):
    """x (fp64/fp32) -> list of n terms of dtype dt (as fp64) with x ~= sum(terms)."""
    out, r = [], x.double()
    for _ in range(n):
        h = r.to(torch.float32).to(dt).double()
        out.append(h)
        r = r - h
    return out


def wscale(W):
    mx = float(W.abs().max())
    ex = int(np.floor(np.log2(mx))) + 1 if mx > 0 else 0      # mx = f 2^ex, f in [0.5,1)
    return 2.0 ** (14 - ex)


def mm(A, W, mode, dt):
    """A [N,K] fp32, W [out,K] fp32 -> A.W^T fp32 under precision `mode`."""
    if mode == "fp32":
        return (A.float() @ W.float().t())
    if mode == "fp64":
        return A.double() @ W.double().t()
    sc = wscale(W) if dt == torch.float16 else 1.0
    nA = 2 if ("l" in mode.split("+")[0] or any(t[0] == "l" for t in mode.split("+"))) else 1
    nW = 2 if any(t[1] == "l" for t in mode.split("+")) else 1
    a = split(A, dt, max(nA, 1))
    w = split(W.double() * sc, dt, max(nW, 1))
    acc = torch.zeros(A.shape[0], W.shape[0], dtype=torch.float64)
    for t in mode.split("+"):
        ai = 0 if t[0] == "h" else 1
        wi = 0 if t[1] == "h" else 1
        acc = acc + a[ai] @ w[wi].t()
    return (acc / sc).float()


def chain(person, cfg, x, mode, dt=torch.float16, sig16=False, gscale=1.0):
    """SDF forward, analytic reverse sweep, normal (identity skinning Jacobian), colour.  Returns dict."""
    hp = torch.float64 if mode == "fp64" else torch.float32
    sd = person["implicit"]
    x = x.to(hp)
    emb = port.embed(x.double(), cfg["multires"]).to(hp) if mode == "fp64" else port.embed(x.float(), cfg["multires"])
    cond = person["cond"].to(hp).expand(x.shape[0], -1)
    Ws, bs = [], []
    for l in range(9):
        w, b = port._lin({k: v.double() for k, v in sd.items()}, l, True)
        Ws.append(w.to(hp))
        bs.append(b.to(hp))
    E = emb.shape[1]
    h = emb
    sig = []
    for l in range(8):
        W, b = Ws[l], bs[l]
        if l == 0:
            beff = b + cond @ W[:, E:].t()          # cond folded into the bias (constant per call)
            z = mm(h, W[:, :E], mode, dt).to(hp) + beff
        else:
            if l == 4:
                h = torch.cat([h, emb], 1) / np.sqrt(2)
            z = mm(h, W, mode, dt).to(hp) + b
        h = F.softplus(z, beta=100)
        s = torch.sigmoid(100 * z)
        if sig16:
            s = torch.round(s * 65535.0) / 65535.0
        sig.append(s)
    out8 = mm(h, Ws[8], "fp64" if mode == "fp64" else ("fp32" if mode == "fp32" else mode), dt).to(hp) + bs[8]
    sdf = out8[:, 0]
    feat = out8[:, 1:]
    # reverse sweep
    g = (Ws[8][0][None, :] * sig[7]) * gscale
    gemb = torch.zeros_like(emb)
    for l in range(7, 0, -1):
        gin = mm(g, Ws[l].t().contiguous(), mode, dt).to(hp)       # [N, in_l]
        if l == 4:
            gin = gin / np.sqrt(2)
            gemb = gemb + gin[:, 256 - E:]
            gin = gin[:, :256 - E]
        g = gin * sig[l - 1]
    gemb = gemb + mm(g, Ws[0][:, :E].t().contiguous(), mode, dt).to(hp)
    gemb = gemb / gscale
    d = 3
    gx = gemb[:, :d].clone()
    for f in range(cfg["multires"]):
        sn = emb[:, d + 2 * f * d: d + 2 * f * d + d]
        cs = emb[:, d + (2 * f + 1) * d: d + (2 * f + 1) * d + d]
        gx = gx + (2.0 ** f) * (cs * gemb[:, d + 2 * f * d: d + 2 * f * d + d] - sn * gemb[:, d + (2 * f + 1) * d: d + (2 * f + 1) * d + d])
    nrm = F.normalize(gx, dim=1)
    # colour
    rd = {k: v.double() for k, v in person["render"].items()}
    bp = F.linear(person["cond"].double(), rd["lin_pose.weight"], rd["lin_pose.bias"]).to(hp).expand(x.shape[0], -1)
    hcol = torch.cat([x, nrm, bp, feat], -1)
    for l in range(5):
        w, b = port._lin(rd, l, True)
        hcol = mm(hcol, w.to(hp), mode, dt).to(hp) + b.to(hp)
        if l < 4:
            hcol = torch.relu(hcol)
    rgb = torch.sigmoid(hcol)
    return dict(sdf=sdf.double(), grad=gx.double(), nrm=nrm.double(), rgb=rgb.double())


def main():
    torch.manual_seed(0)
    sc = S.make_scene(P=2, S=64, seed=42)
    person, cfg = sc["persons"][0], sc["cfg"]
    cfg = dict(cfg, multires=6)
    g = torch.Generator().manual_seed(5)
    # points around the geometric-init surface (r ~ 0.6) and in the near band the sampler concentrates on
    dirs = F.normalize(torch.randn(4096, 3, generator=g), dim=1)
    r = 0.6 + 0.1 * (torch.rand(4096, 1, generator=g) * 2 - 1)
    x = dirs * r
    truth = chain(person, cfg, x, "fp64")
    rows = []

    def report(name, o):
        e = {k: float((o[k] - truth[k]).abs().max()) for k in ("sdf", "grad", "nrm", "rgb")}
        rows.append(dict(mode=name, **e))
        print("%-34s sdf %.2e  grad %.2e  normal %.2e  rgb %.2e" % (name, e["sdf"], e["grad"], e["nrm"], e["rgb"]))

    report("torch fp32 (reference arithmetic)", chain(person, cfg, x, "fp32"))
    for mode in ("hh+lh+hl", "hh+lh", "hh+hl", "hh"):
        report("fp16 " + mode, chain(person, cfg, x, mode))
    report("fp16 hh+lh+hl, sigma' u16", chain(person, cfg, x, "hh+lh+hl", sig16=True))
    report("fp16 hh+lh+hl, grad x256", chain(person, cfg, x, "hh+lh+hl", gscale=256.0))
    report("fp16 hh+lh+hl, grad x256, sig u16", chain(person, cfg, x, "hh+lh+hl", gscale=256.0, sig16=True))
    for mode in ("hh+lh+hl", "hh"):
        report("bf16 " + mode, chain(person, cfg, x, mode, dt=torch.bfloat16))
    os.makedirs(os.path.join(ROOT, "profiles"), exist_ok=True)
    json.dump(dict(points=4096, truth="fp64 evaluation of the same weights", rows=rows),
              open(os.path.join(ROOT, "profiles", "numerics.json"), "w"), indent=1)


if __name__ == "__main__":
    main()
