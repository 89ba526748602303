"""GPU: the stall-accounting build of the MLP chain kernel (mp_profile_enable(2)) against the default build.

The accounting build reads clock64 around the kernel's waits and adds the totals to a per-CTA block of the workspace;
it must not change what the kernel computes.  For the four programs (sdf-only, sdf + features, the full shade chain,
the background) in the three precision modes, at counts around one tile and around one tile per CTA (1, 127, 128, 129,
128 x SMs, 3 x 128 x SMs + 77: fewer tiles than CTAs, exactly one per CTA, several per CTA with a partial last one),
both builds must give bit-identical outputs, and the shade pass of a render (per-sample sdf, rgb, normals) too.  The
totals of every warp must be consistent: each phase of a step kind within that kind's step time, and the steps plus
the tile prologues within the warp's whole run (a negative interval would wrap the unsigned total and break this)."""
import ctypes as C
import os
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from multiply_b200 import engine, scene as S     # noqa: E402

MODES = ["parity", "colour1", "throughput"]


def _L():
    from multiply_b200 import _lib as L
    return L


def _counts():
    T = 128 * int(_L().call("mp_device_sm_count"))
    return [1, 127, 128, 129, T, 3 * T + 77]


@pytest.fixture(scope="module")
def case():
    sc = S.make_scene(P=2, S=64, seed=42, weights="trained")
    person = sc["persons"][0]
    field = engine.Field(person["implicit"], person["render"])
    field.set_cond(person["cond"])
    bg = engine.Field(sc["bg_implicit"], sc["bg_render"], background=True)
    bg.set_cond(sc["frame_code"])
    n = max(_counts())
    g = torch.Generator().manual_seed(7)
    x = ((torch.rand(n, 3, generator=g) - 0.5) * 2.0).cuda()
    x4 = torch.cat([torch.nn.functional.normalize(torch.randn(n, 3, generator=g), dim=1),
                    torch.rand(n, 1, generator=g) / 3.0], 1).contiguous().cuda()
    view = torch.nn.functional.normalize(torch.randn(n, 3, generator=g), dim=1).contiguous().cuda()
    return dict(sc=sc, field=field, bg=bg, x=x, x4=x4, view=view)


def _programs(c, N):
    """Outputs of the four programs on the first N points (workspaces sized under the current profile setting)."""
    L = _L()
    ws = L.workspace(L.call("mp_mlp_workspace_bytes", N), "cuda")
    f32 = dict(dtype=torch.float32, device="cuda")
    o = {}
    sdf = torch.empty(N, **f32)
    L.call("mp_implicit_forward", c["field"].handle, c["x"][:N], N, sdf, None, ws, ws.numel())
    o["sdf_only.sdf"] = sdf
    sdf, feat = torch.empty(N, **f32), torch.empty(N, 256, **f32)
    L.call("mp_implicit_forward", c["field"].handle, c["x"][:N], N, sdf, feat, ws, ws.numel())
    o["forward.sdf"], o["forward.feat"] = sdf, feat
    sdf, grad = torch.empty(N, **f32), torch.empty(N, 3, **f32)
    L.call("mp_implicit_forward_grad", c["field"].handle, c["x"][:N], N, sdf, None, grad, ws, ws.numel())
    o["full.sdf"], o["full.grad"] = sdf, grad
    sdf, rgb = torch.empty(N, **f32), torch.empty(N, 3, **f32)
    L.call("mp_bg_nets_forward", c["bg"].handle, c["x4"][:N], c["view"][:N], N, sdf, rgb, ws, ws.numel())
    o["background.sdf"], o["background.rgb"] = sdf, rgb
    torch.cuda.synchronize()
    return {k: v.cpu() for k, v in o.items()}


def _shade(c):
    """Per-sample taps of one render: the full shade program's sdf, rgb and normals."""
    sc = c["sc"]
    inp = S.make_rays(sc, 256, seed=5, region="boxes")
    hits = S.make_hit_lists(sc, inp)
    o = engine.Renderer(sc).render(inp, hits, debug=True)
    torch.cuda.synchronize()
    return {f"shade.{k}_{p}": o[f"{k}_{p}"].cpu() for p in range(2) for k in ("sdf", "rgb", "normals")}


def _run(c, stalls, mode):
    L = _L()
    engine.set_engine("tc")
    engine.set_precision(mode)
    L.call("mp_profile_enable", 2 if stalls else 0)
    try:
        out = {N: _programs(c, N) for N in _counts()}
        out["render"] = _shade(c)
    finally:
        L.call("mp_profile_enable", 0)
        engine.set_precision("parity")
    return out


@pytest.mark.parametrize("mode", MODES)
def test_stall_build_is_bit_identical(case, mode):
    ref = _run(case, False, mode)
    got = _run(case, True, mode)
    for key, outs in ref.items():
        for name, a in outs.items():
            b = got[key][name]
            assert torch.equal(a.view(torch.int32), b.view(torch.int32)), "%s at %s: %d values differ" % (
                name, key, int((a != b).sum()))


def test_stall_totals_are_consistent(case):
    L = _L()
    W, NW, P = L.MP_STALL_WORDS, L.MP_STALL_WARPS, L.MP_STALL_PHASES
    clocks = (C.c_ulonglong * (4 * NW * W))()
    L.call("mp_profile_read_stalls", clocks, 1)
    _run(case, True, "parity")
    L.call("mp_profile_read_stalls", clocks, 1)
    tot = np.frombuffer(clocks, dtype=np.uint64).reshape(4, NW, W).astype(np.float64)
    for prog in range(4):
        assert tot[prog, :, L.MP_STALL_ELAPSED].min() > 0, "program %d: a warp recorded no run" % prog
        for w in range(NW):
            rec = tot[prog, w]
            steps = rec[:L.MP_STALL_PROLOGUE].reshape(-1, P)
            if w == 0:
                assert (steps[:, 5] <= steps[:, 0]).all(), "program %d loader: empty waits exceed step time" % prog
            else:
                assert (steps[:, 1:5].sum(1) <= steps[:, 0]).all(), "program %d warp %d: phases exceed steps" % (prog, w)
                assert (steps[:, 5] == 0).all()
            assert steps[:, 0].sum() + rec[L.MP_STALL_PROLOGUE] <= rec[L.MP_STALL_ELAPSED], \
                "program %d warp %d: steps exceed the run" % (prog, w)
            assert steps[:, 0].sum() > 0
