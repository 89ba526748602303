"""One case per workspace-taking entry point that the workspace bounds and reuse tests both drive, so that each call's
argument list is written once.

A case holds the entry point (or the tuple of entry points that share one workspace), its workspace query, the shape
and dtype of every output buffer, ``call(x, o, ws)``, which makes the call on inputs ``x`` with output buffers ``o`` and
workspace ``ws`` through ``_lib.call`` and returns the outputs it wrote (views of ``o``, host counts), and, where the
inputs come from a seed, ``inputs(seed)``."""
import ctypes as C
from typing import Callable, NamedTuple, Optional

import numpy as np
import torch

from multiply_b200 import engine, _lib as L
from multiply_b200.utils import mesh as umesh

from _setups import Smpl, make_inputs, person_samples, points, pts, rays, train_rng


class Case(NamedTuple):
    name: object                    # entry point, or a tuple of entry points sharing the workspace
    query: Callable[[], int]        # the workspace bytes
    outs: dict                      # output buffer name -> (shape, dtype)
    call: Callable                  # call(x, o, ws) -> dict of outputs
    inputs: Optional[Callable] = None   # inputs(seed) -> x


F32, I32, I64, U8 = torch.float32, torch.int32, torch.int64, torch.uint8


def _mlp_query(N):
    return lambda: L.call("mp_mlp_workspace_bytes", N)


# ---------------------------------------------------------------------------------------------
# networks, lattice SDF, background
# ---------------------------------------------------------------------------------------------

def implicit_forward(field, N, grad):
    """mp_implicit_forward(_grad) on N points; inputs(seed): uniform in [-1, 1)^3."""
    outs = dict(sdf=(N, F32), feat=((N, 256), F32))
    if grad:
        outs["grad"] = ((N, 3), F32)

    def call(x, o, ws):
        if grad:
            L.call("mp_implicit_forward_grad", field.handle, x, N, o["sdf"], o["feat"], o["grad"], ws, ws.numel())
            return dict(sdf=o["sdf"], feat=o["feat"], grad=o["grad"])
        L.call("mp_implicit_forward", field.handle, x, N, o["sdf"], o["feat"], ws, ws.numel())
        return dict(sdf=o["sdf"], feat=o["feat"])

    name = "mp_implicit_forward_grad" if grad else "mp_implicit_forward"
    return Case(name, _mlp_query(N), outs, call, lambda seed: pts(N, 3, seed))


def bg_nets_forward(bg, N):
    """mp_bg_nets_forward on N points; inputs(seed): points in [-1, 1)^4, unit view directions."""
    def inputs(seed):
        view = pts(N, 3, seed + 1)
        return pts(N, 4, seed, -1.0, 1.0), (view / view.norm(dim=1, keepdim=True)).contiguous()

    def call(x, o, ws):
        p, view = x
        L.call("mp_bg_nets_forward", bg.handle, p, view, N, o["sdf"], o["rgb"], ws, ws.numel())
        return dict(sdf=o["sdf"], rgb=o["rgb"])

    return Case("mp_bg_nets_forward", _mlp_query(N), dict(sdf=(N, F32), rgb=((N, 3), F32)), call, inputs)


def _grads(shapes, o):
    """mp_linear_grads_t on the output buffers dW{l} / db{l}."""
    g = L.LinearGrads()
    for l in range(len(shapes)):
        g.d_weight[l], g.d_bias[l] = L.ptr(o["dW%d" % l]), L.ptr(o["db%d" % l])
    return g


def _param_outs(shapes):
    outs = {}
    for l, (o, i) in enumerate(shapes):
        outs["dW%d" % l], outs["db%d" % l] = ((o, i), F32), (o, F32)
    return outs


def implicit_backward(field, N):
    """mp_implicit_backward of a foreground or background field on N points, every output wanted; inputs(seed): points
    in [-1, 1)^d_in and upstreams d_sdf, d_feat in [-1, 1)."""
    outs = dict(d_x=((N, field.d_in), F32), d_cond=(field.cond_dim, F32), **_param_outs(field.imp_shapes))

    def call(x, o, ws):
        p, d_sdf, d_feat = x
        L.call("mp_implicit_backward", field.handle, p, N, d_sdf, d_feat, o["d_x"], _grads(field.imp_shapes, o),
               o["d_cond"], ws, ws.numel())
        return dict(o)

    return Case("mp_implicit_backward", lambda: L.call("mp_implicit_backward_workspace_bytes", N), outs, call,
                lambda seed: (pts(N, field.d_in, seed), pts(N, 1, seed + 1).reshape(N), pts(N, 256, seed + 2)))


def render_backward(field, N):
    """mp_render_backward of a foreground field on N points, every output wanted; inputs(seed): points, normals,
    features and d_rgb in [-1, 1)."""
    outs = dict(d_points=((N, 3), F32), d_normals=((N, 3), F32), d_feat=((N, 256), F32), d_lpw=((8, 69), F32),
                d_lpb=(8, F32), d_bp=(69, F32), **_param_outs(field.ren_shapes))

    def call(x, o, ws):
        p, n, f, d_rgb = x
        L.call("mp_render_backward", field.handle, p, n, f, N, d_rgb, o["d_points"], o["d_normals"], o["d_feat"],
               _grads(field.ren_shapes, o), o["d_lpw"], o["d_lpb"], o["d_bp"], ws, ws.numel())
        return dict(o)

    return Case("mp_render_backward", lambda: L.call("mp_render_backward_workspace_bytes", N), outs, call,
                lambda seed: (pts(N, 3, seed), pts(N, 3, seed + 1), pts(N, 256, seed + 2), pts(N, 3, seed + 3)))


def person_box(sc, fields, pid):
    """Person pid's field and the lattice box of generate_mesh around its canonical body."""
    center, extent, pad = umesh.bounds(sc["persons"][pid]["verts_c"])
    return fields[pid], center, extent, pad


def sdf_grid(sc, fields, res):
    """mp_sdf_grid at res; inputs(pid): person pid's field and box."""
    def call(x, o, ws):
        f, center, extent, pad = x
        L.call("mp_sdf_grid", f.handle, L.vec3(C.c_float, center), float(extent), float(pad), res, o["vals"], ws,
               ws.numel())
        return dict(vals=o["vals"])

    return Case("mp_sdf_grid", lambda: L.call("mp_sdf_grid_workspace_bytes", res), dict(vals=((res + 1) ** 3, F32)),
                call, lambda pid: person_box(sc, fields, pid))


def background(bg, R):
    """mp_background on R rays; inputs(seed): unit directions, cameras in [-1.5, 1.5)^3 (inside the r = 3 sphere)."""
    def inputs(seed):
        d = pts(R, 3, seed)
        return (d / d.norm(dim=1, keepdim=True)).contiguous(), pts(R, 3, seed + 1, -1.5, 1.5)

    def call(x, o, ws):
        d, c = x
        L.call("mp_background", bg.handle, d, c, R, 3.0, o["rgb"], ws, ws.numel())
        return dict(rgb=o["rgb"])

    return Case("mp_background", lambda: L.call("mp_background_workspace_bytes", R), dict(rgb=((R, 3), F32)), call,
                inputs)


def mise(sc, fields, res_init, depth):
    """mp_mise at res_init / depth; inputs(pid): person pid's field and box."""
    n1 = (res_init << depth) + 1

    def call(x, o, ws):
        f, center, extent, pad = x
        n = C.c_longlong(0)
        L.call("mp_mise", f.handle, L.vec3(C.c_float, center), float(extent), float(pad), res_init, depth, 0.0,
               o["grid"], o["ev"], C.byref(n), ws, ws.numel())
        return dict(grid=o["grid"], ev=o["ev"], n=n.value)

    return Case("mp_mise", lambda: L.call("mp_mise_workspace_bytes", res_init, depth),
                dict(grid=(n1 ** 3, F32), ev=(n1 ** 3, U8)), call, lambda pid: person_box(sc, fields, pid))


def marching_cubes(R, V, F):
    """mp_marching_cubes_count and _emit on one workspace (emit reads the count's offsets), on an (R + 1)^3 grid, into
    outputs of V vertices and F faces; the outputs are the rows the call writes."""
    def call(g, o, ws):
        nv, nf = C.c_longlong(0), C.c_longlong(0)
        L.call("mp_marching_cubes_count", g, R, 0.0, C.byref(nv), C.byref(nf), ws, ws.numel())
        L.call("mp_marching_cubes_emit", g, R, 0.0, L.vec3(C.c_double, (R / 2.0,) * 3), float(R), 1.0, o["v"], o["f"],
               ws, ws.numel())
        return dict(V=nv.value, F=nf.value, v=o["v"][:3 * nv.value], f=o["f"][:3 * nf.value])

    return Case(("mp_marching_cubes_count", "mp_marching_cubes_emit"),
                lambda: L.call("mp_marching_cubes_workspace_bytes", R), dict(v=(3 * V, F32), f=(3 * F, I64)), call)


def largest_component(V, F):
    """mp_largest_component of a mesh (v, f) with V vertices and F faces; the outputs are the rows the call writes."""
    def call(x, o, ws):
        v, f = x
        nv, nf = C.c_int(0), C.c_int(0)
        L.call("mp_largest_component", v, V, f, F, o["v"], o["f"], C.byref(nv), C.byref(nf), ws, ws.numel())
        return dict(V=nv.value, F=nf.value, v=o["v"][:3 * nv.value], f=o["f"][:3 * nf.value])

    return Case("mp_largest_component", lambda: L.call("mp_largest_component_workspace_bytes", V, F),
                dict(v=(3 * V, F32), f=(3 * F, I64)), call)


# ---------------------------------------------------------------------------------------------
# sampler
# ---------------------------------------------------------------------------------------------

def sample_rays(sc, field, body, R, train):
    """mp_sample_rays(_train) on R rays of person 0's box; inputs(seed): those rays and the training draws."""
    cfg = dict(sc["cfg"], beta_param=sc["beta_param"])
    c = engine.sampler_cfg(cfg, cfg["beta_param"])
    n = cfg["N_samples"] + cfg["N_samples_extra"] + 2

    def inputs(seed):
        d, o = rays(sc, R, seed=seed)
        return d.cuda(), o.cuda(), train_rng(cfg, R, seed=seed)

    def call(x, o, ws):
        d, cam, rng = x
        if not train:
            L.call("mp_sample_rays", c, body.handle, field.handle, d, cam, R, o["z"], o["z_bg"], o["trips"], ws,
                   ws.numel())
            return dict(z=o["z"], z_bg=o["z_bg"], trips=o["trips"])
        r, keep = engine.sampler_rng_struct(rng, torch.device("cuda"))
        L.call("mp_sample_rays_train", c, body.handle, field.handle, d, cam, R, r, o["z"], o["z_bg"], o["z_eik"],
               o["trips"], ws, ws.numel())
        torch.cuda.synchronize()        # the draws in ``keep`` are read by the kernels
        return dict(z=o["z"], z_bg=o["z_bg"], z_eik=o["z_eik"], trips=o["trips"])

    return Case("mp_sample_rays_train" if train else "mp_sample_rays",
                lambda: L.call("mp_sampler_workspace_bytes", c, R),
                dict(z=((R, n), F32), z_bg=((R, 32), F32), z_eik=(R, F32), trips=(1, I32)), call, inputs)


# ---------------------------------------------------------------------------------------------
# compositor and its backward
# ---------------------------------------------------------------------------------------------

P_C, R_C, N_C, BETA_C = 3, 300, 33, 0.1


def composite_inputs(seed):
    """make_inputs' samples of P_C persons on R_C rays, N_C samples each, and upstream gradients."""
    persons = make_inputs(seed, P_C, R_C, N_C)
    arr, keep = person_samples(persons)
    rng = np.random.RandomState(seed + 100)
    ups = {k: torch.from_numpy(rng.standard_normal(s).astype(np.float32)).cuda() for k, s in (
        ("d_fg", (R_C, 3)), ("d_nrm", (R_C, 3)), ("d_acc", R_C), ("d_accp", (R_C, P_C)), ("d_bgT", R_C))}
    return dict(arr=arr, keep=keep, rows=[d["idx"].size for d in persons], ups=ups)


def composite():
    def call(x, o, ws):
        L.call("mp_composite", x["arr"], P_C, R_C, N_C, BETA_C, o["fg"], o["nrm"], o["acc"], o["accp"], o["bgT"], ws,
               ws.numel())
        return {k: o[k] for k in ("fg", "nrm", "acc", "accp", "bgT")}

    return Case("mp_composite", lambda: L.call("mp_composite_workspace_bytes", R_C, P_C),
                dict(fg=((R_C, 3), F32), nrm=((R_C, 3), F32), acc=(R_C, F32), accp=((R_C, P_C), F32), bgT=(R_C, F32)),
                call, composite_inputs)


def composite_backward():
    """Gradient buffers hold R rows per person; the outputs are the rows of each person's hit list."""
    def call(x, o, ws):
        gr = (L.PersonSampleGrads * P_C)()
        for p in range(P_C):
            gr[p].d_sdf, gr[p].d_rgb, gr[p].d_normal = (L.ptr(o["%s%d" % (k, p)]) for k in ("sdf", "rgb", "nrm"))
        u = x["ups"]
        L.call("mp_composite_backward", x["arr"], P_C, R_C, N_C, BETA_C, u["d_fg"], u["d_nrm"], u["d_acc"], u["d_accp"],
               u["d_bgT"], gr, o["d_beta"], ws, ws.numel())
        out = {"d_beta": o["d_beta"]}
        for p, rows in enumerate(x["rows"]):
            for k in ("sdf", "rgb", "nrm"):
                out["%s%d" % (k, p)] = o["%s%d" % (k, p)][:rows]
        return out

    outs = dict(d_beta=(1, F32))
    for p in range(P_C):
        outs.update({"sdf%d" % p: ((R_C, N_C), F32), "rgb%d" % p: ((R_C, N_C, 3), F32),
                     "nrm%d" % p: ((R_C, N_C, 3), F32)})
    return Case("mp_composite_backward", lambda: L.call("mp_composite_backward_workspace_bytes", R_C, P_C), outs, call,
                composite_inputs)


# ---------------------------------------------------------------------------------------------
# SMPL server and deformer backward
# ---------------------------------------------------------------------------------------------

def smpl_backward(sm):
    """mp_smpl_backward of the Smpl handle ``sm``; inputs(seed): parameters and upstream gradients."""
    def inputs(seed):
        rng = np.random.RandomState(seed)
        args = Smpl._args(1.0 + 0.1 * rng.rand(), rng.normal(0, 0.3, 3), rng.normal(0, 0.4, 72), rng.normal(0, 1, 10))
        dv = torch.from_numpy(rng.standard_normal((sm.V, 3)).astype(np.float32)).cuda()
        dt = torch.from_numpy(rng.standard_normal((24, 4, 4)).astype(np.float32)).cuda()
        return args, dv, dt

    def call(x, o, ws):
        args, dv, dt = x
        L.call("mp_smpl_backward", sm.h, *args, 0, dv, dt, o["scale"], o["transl"], o["thetas"], o["betas"], ws,
               ws.numel())
        return {k: o[k] for k in ("scale", "transl", "thetas", "betas")}

    return Case("mp_smpl_backward", lambda: L.call("mp_smpl_backward_workspace_bytes", sm.V),
                dict(scale=(1, F32), transl=(3, F32), thetas=(72, F32), betas=(10, F32)), call, inputs)


def _deform_inputs(body, N):
    def inputs(seed):
        u = torch.from_numpy(np.random.RandomState(seed).randn(N, 3).astype(np.float32)).cuda()
        uj = torch.from_numpy(np.random.RandomState(seed + 1).randn(N, 9).astype(np.float32)).cuda()
        return points(N, body.verts_p, seed).cuda(), u, uj
    return inputs


def deform_inverse_backward(body, N):
    """mp_deform_inverse_backward (exact_far) of N points near the posed body; inputs(seed): points, upstream."""
    def call(x, o, ws):
        p, u, _ = x
        L.call("mp_deform_inverse_backward", body.handle, p, N, 1, u, o["d_tfs"], o["d_x"], o["xc"], ws, ws.numel())
        return {k: o[k] for k in ("d_tfs", "d_x", "xc")}

    return Case("mp_deform_inverse_backward", lambda: L.call("mp_deform_backward_workspace_bytes", N),
                dict(d_tfs=((24, 4, 4), F32), d_x=((N, 3), F32), xc=((N, 3), F32)), call, _deform_inputs(body, N))


def deform_forward_jac_backward(body, N):
    """mp_deform_forward_jac_backward of N points near the posed body; inputs(seed): points, upstream."""
    def call(x, o, ws):
        p, u, uj = x
        L.call("mp_deform_forward_jac_backward", body.handle, p, N, u, uj, o["d_tfs"], o["d_x"], ws, ws.numel())
        return {k: o[k] for k in ("d_tfs", "d_x")}

    return Case("mp_deform_forward_jac_backward", lambda: L.call("mp_deform_backward_workspace_bytes", N),
                dict(d_tfs=((24, 4, 4), F32), d_x=((N, 3), F32)), call, _deform_inputs(body, N))
