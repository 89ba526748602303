"""Not collected by pytest (could not be run on a GPU before the round closed): Multiply.sdf_func_with_smpl_deformer
through the mirror class against the oracle.  `PYTHONPATH=. python scripts/check_sdf_func_mirror.py` on a GPU box."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from multiply_b200 import scene as S


def check_sdf_func_with_smpl_deformer_mirror():
    """Multiply.sdf_func_with_smpl_deformer (multiply.py:137-151) through the mirror class, against the oracle."""
    from multiply_b200 import engine
    from oracle import port
    engine.set_engine("tc")
    sc = S.make_scene(P=2, S=16, seed=42)
    m = S.mirror_model(sc)
    p1 = sc["persons"][1]
    g = torch.Generator().manual_seed(3)
    pts = torch.cat([p1["verts_p"][:300] + 0.02 * torch.randn(300, 3, generator=g),       # near the body
                     p1["verts_p"][:100] + 0.5])                                          # outliers
    sdf, xc, feat = m.sdf_func_with_smpl_deformer(pts.cuda(), {"smpl": p1["cond"].cuda()}, p1["tfs"][None].cuda(),
                                                  p1["verts_p"][None].cuda(), 1)
    with torch.no_grad():
        rs, rx, rf = port.sdf_func_with_smpl_deformer(pts, p1, sc["cfg"])
    assert sdf.shape == (400, 1) and xc.shape == (400, 3) and feat.shape == (400, 256)
    assert float((sdf.cpu() - rs).abs().max()) < 5e-5
    assert float((xc.cpu() - rx).abs().max()) < 1e-5
    assert float((feat.cpu() - rf).abs().max()) < 5e-5
    assert bool(((sdf.cpu() == 4.0) == (rs == 4.0)).all()) and bool((rs[300:] == 4.0).any())




if __name__ == "__main__":
    check_sdf_func_with_smpl_deformer_mirror()
    print("OK")
