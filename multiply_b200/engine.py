"""Device-side scene objects on top of the C ABI: packed fields, posed bodies, the fused renderer.

PyTorch is used for device memory and streams only; every computation is a call into
libmultiply_b200.so (see _lib.py).  No fallback path exists.
"""
import ctypes as C
import functools
import math

import numpy as np
import torch

from . import _lib as L


def set_engine(name):
    """'tc' = wgmma split-fp16 tensor-core engine (default), 'simt' = fp32 validation engine."""
    L.call("mp_set_engine", {"simt": 0, "tc": 1}[name])


def set_precision(mode):
    """Tensor-core engine precision: 'parity' (default, three split terms), 'colour1' (single-term colour layers),
    'throughput' (single fp16 term everywhere; outside the 1e-4 gate)."""
    L.call("mp_set_precision", {"parity": 0, "colour1": 1, "throughput": 2}[mode])


def get_engine():
    return {0: "simt", 1: "tc"}[L.call("mp_get_engine")]


def _stack(sd, n_layers, dev, keep):
    st = L.LinearStack()
    st.n_layers = n_layers
    for l in range(n_layers):
        if f"lin{l}.weight_v" in sd:
            v = L.dev(sd[f"lin{l}.weight_v"], dev)
            g = L.dev(sd[f"lin{l}.weight_g"], dev)
        else:
            v, g = L.dev(sd[f"lin{l}.weight"], dev), None
        b = L.dev(sd[f"lin{l}.bias"], dev)
        keep += [v, g, b]
        st.weight_v[l], st.weight_g[l], st.bias[l] = L.ptr(v), L.ptr(g), L.ptr(b)
        st.out_dim[l], st.in_dim[l] = v.shape
    return st


class Field:
    """Packed ImplicitNet + RenderingNet pair (mp_field_pack)."""

    def __init__(self, implicit_sd, render_sd, background=False, device="cuda"):
        self.device = torch.device(device)
        keep = []
        imp = L.ImplicitDesc()
        imp.lin = _stack(implicit_sd, 9, self.device, keep)
        imp.d_in = 4 if background else 3
        imp.multires = 10 if background else 6
        imp.cond_dim = 32 if background else 69
        imp.skip_layer = 4
        ren = L.RenderDesc()
        n_ren = len([k for k in render_sd if k.startswith("lin") and k.endswith(".bias") and "pose" not in k])
        ren.lin = _stack(render_sd, n_ren, self.device, keep)
        ren.mode = 1 if background else 0
        ren.multires_view = 4 if background else -1
        if not background:
            pw, pb = L.dev(render_sd["lin_pose.weight"], self.device), L.dev(render_sd["lin_pose.bias"], self.device)
            keep += [pw, pb]
            ren.lin_pose_weight, ren.lin_pose_bias = L.ptr(pw), L.ptr(pb)
        self.storage = L.workspace(L.call("mp_field_pack_bytes", imp, ren, int(background)), self.device)
        self.handle = L.Handle("mp_field_free")
        L.call("mp_field_pack", imp, ren, int(background), self.storage, self.storage.numel(), C.byref(self.handle))
        torch.cuda.current_stream().synchronize()   # raw parameter tensors may be released now
        self.background = background
        self.d_in, self.cond_dim = imp.d_in, imp.cond_dim
        self.imp_shapes = [(imp.lin.out_dim[l], imp.lin.in_dim[l]) for l in range(imp.lin.n_layers)]
        self.ren_shapes = [(ren.lin.out_dim[l], ren.lin.in_dim[l]) for l in range(ren.lin.n_layers)]

    def set_cond(self, cond):
        c = L.dev(cond.reshape(-1), self.device)
        L.call("mp_field_set_cond", self.handle, c)
        self._cond = c

    # operator-level entry points ------------------------------------------------------
    def implicit_forward(self, x, want_feat=True, want_grad=False):
        x = L.dev(x, self.device)
        N = x.shape[0]
        sdf = torch.empty(N, device=self.device)
        feat = torch.empty(N, 256, device=self.device) if want_feat else None
        ws = L.workspace(L.call("mp_mlp_workspace_bytes", N), self.device)
        if want_grad:
            grad = torch.empty(N, 3, device=self.device)
            L.call("mp_implicit_forward_grad", self.handle, x, N, sdf, feat, grad, ws, ws.numel())
            return sdf, feat, grad
        L.call("mp_implicit_forward", self.handle, x, N, sdf, feat, ws, ws.numel())
        return sdf, feat

    def sdf_grid(self, center, extent, res, pad=1.1):
        """Canonical SDF on the (res+1)^3 lattice of generate_mesh (lib/utils/mesh.py:78-105): returns [res+1]*3 fp32."""
        n1 = res + 1
        vals = torch.empty(n1, n1, n1, device=self.device)
        ws = L.workspace(L.call("mp_sdf_grid_workspace_bytes", res), self.device)
        L.call("mp_sdf_grid", self.handle, L.vec3(C.c_float, center), float(extent), float(pad), int(res), vals, ws,
               ws.numel())
        return vals

    def mise(self, center, extent, res_init, depth, level=0.0, pad=1.1, want_evaluated=False):
        """MISE of generate_mesh (lib/utils/mesh.py:87-109, lib/libmise/mise.pyx) on the device: returns (grid
        [R+1]*3 fp32 = to_dense(), number of points evaluated[, evaluated [R+1]*3 bool]), R = res_init << depth."""
        n1 = (int(res_init) << int(depth)) + 1
        grid = torch.empty(n1, n1, n1, device=self.device)
        ev = torch.empty(n1, n1, n1, dtype=torch.uint8, device=self.device) if want_evaluated else None
        ws = L.workspace(L.call("mp_mise_workspace_bytes", int(res_init), int(depth)), self.device)
        n = C.c_longlong(0)
        L.call("mp_mise", self.handle, L.vec3(C.c_float, center), float(extent), float(pad), int(res_init), int(depth),
               float(level), grid, ev, C.byref(n), ws, ws.numel())
        return (grid, n.value, ev.bool()) if want_evaluated else (grid, n.value)

    def extract_mesh(self, center, extent, res_init=32, depth=3, level=0.0, pad=1.1):
        """generate_mesh (lib/utils/mesh.py:78-132) for this field: MISE -> marching cubes -> largest component.
        Returns (verts [V,3] fp32, faces [F,3] int64, number of points evaluated); device tensors."""
        grid, n = self.mise(center, extent, res_init, depth, level, pad)
        v, f = marching_cubes(grid, level, center, extent, pad)
        v, f = largest_component(v, f)
        return v, f, n

    def bg_forward(self, pts, view_dirs):
        """Background pair at given points (multiply.py:523-526): pts [N,4], view_dirs [N,3] -> (sdf [N], rgb [N,3])."""
        pts, view_dirs = L.dev(pts, self.device), L.dev(view_dirs, self.device)
        N = pts.shape[0]
        sdf = torch.empty(N, device=self.device)
        rgb = torch.empty(N, 3, device=self.device)
        ws = L.workspace(L.call("mp_mlp_workspace_bytes", N), self.device)
        L.call("mp_bg_nets_forward", self.handle, pts, view_dirs, N, sdf, rgb, ws, ws.numel())
        return sdf, rgb

    def bg_pixels(self, ray_dirs, cam_loc, bound_r):
        """The background pixel of every ray (mp_background: inverse-sphere samples -> background pair -> volume
        rendering, multiply.py:482-539): ray_dirs [R,3], cam_loc [R,3] -> bg_rgb [R,3]."""
        ray_dirs, cam_loc = L.dev(ray_dirs, self.device), L.dev(cam_loc, self.device)
        R = ray_dirs.shape[0]
        rgb = torch.empty(R, 3, device=self.device)
        ws = L.workspace(L.call("mp_background_workspace_bytes", R), self.device)
        L.call("mp_background", self.handle, ray_dirs, cam_loc, R, float(bound_r), rgb, ws, ws.numel())
        return rgb

    def render_forward(self, points, normals, feat):
        points, normals, feat = (L.dev(t, self.device) for t in (points, normals, feat))
        N = points.shape[0]
        rgb = torch.empty(N, 3, device=self.device)
        ws = L.workspace(L.call("mp_mlp_workspace_bytes", N), self.device)
        L.call("mp_render_forward", self.handle, points, normals, feat, N, rgb, ws, ws.numel())
        return rgb

    def _grads(self, shapes, want):
        g = L.LinearGrads()
        dW = [torch.empty(o, i, device=self.device) if want else None for o, i in shapes]
        db = [torch.empty(o, device=self.device) if want else None for o, _ in shapes]
        for l in range(len(shapes)):
            g.d_weight[l], g.d_bias[l] = L.ptr(dW[l]), L.ptr(db[l])
        return g, dW, db

    def implicit_backward(self, x, d_sdf=None, d_feat=None, want_x=True, want_params=True, want_cond=True):
        """VJP of ImplicitNet.forward at x [N,d_in] with the current cond (mp_implicit_backward): d_sdf [N] and d_feat
        [N,256] (None: zero) -> dict(d_x [N,d_in], d_weight [9 x [out,in]] of the effective weights, d_bias, d_cond
        [cond_dim]); what is not wanted is None."""
        x = L.dev(x, self.device)
        N = x.shape[0]
        d_sdf, d_feat = L.dev(d_sdf, self.device), L.dev(d_feat, self.device)
        d_x = torch.empty(N, self.d_in, device=self.device) if want_x else None
        d_cond = torch.empty(self.cond_dim, device=self.device) if want_cond else None
        g, dW, db = self._grads(self.imp_shapes, want_params)
        ws = L.workspace(L.call("mp_implicit_backward_workspace_bytes", N), self.device)
        L.call("mp_implicit_backward", self.handle, x if N else None, N, d_sdf if N else None,
               d_feat if N else None, d_x if N else None, g, d_cond, ws, ws.numel())
        return dict(d_x=d_x, d_weight=dW, d_bias=db, d_cond=d_cond)

    def render_backward(self, points, normals, feat, d_rgb, want_inputs=True, want_params=True, want_pose=True):
        """VJP of RenderingNet.forward 'pose_no_view' with the current cond as body_pose (mp_render_backward): d_rgb
        [N,3] -> dict(d_points, d_normals [N,3], d_feat [N,256], d_weight / d_bias of lin0.., d_lin_pose_weight [8,69],
        d_lin_pose_bias [8], d_body_pose [69]); what is not wanted is None."""
        points, normals, feat, d_rgb = (L.dev(t, self.device) for t in (points, normals, feat, d_rgb))
        N = points.shape[0]
        e = lambda *s: torch.empty(*s, device=self.device)      # noqa: E731
        d_p, d_n, d_f = (e(N, 3), e(N, 3), e(N, 256)) if want_inputs else (None, None, None)
        d_lpw, d_lpb, d_bp = (e(8, 69), e(8), e(69)) if want_pose else (None, None, None)
        g, dW, db = self._grads(self.ren_shapes, want_params)
        ws = L.workspace(L.call("mp_render_backward_workspace_bytes", N), self.device)
        nz = lambda t: t if N else None                          # noqa: E731
        L.call("mp_render_backward", self.handle, nz(points), nz(normals), nz(feat), N, nz(d_rgb), nz(d_p), nz(d_n),
               nz(d_f), g, d_lpw, d_lpb, d_bp, ws, ws.numel())
        return dict(d_points=d_p, d_normals=d_n, d_feat=d_f, d_weight=dW, d_bias=db, d_lin_pose_weight=d_lpw,
                    d_lin_pose_bias=d_lpb, d_body_pose=d_bp)


class Body:
    """Canonical SMPL vertices + skinning weights (SMPLDeformer state) and the per-frame pose."""

    def __init__(self, verts_cano, weights, cano_cell=0.2, device="cuda"):
        self.device = torch.device(device)
        self.verts_c = L.dev(verts_cano, self.device)
        self.weights = L.dev(weights, self.device)
        self.V = self.verts_c.shape[0]
        self.storage = L.workspace(L.call("mp_body_bytes", self.V), self.device)
        self.handle = L.Handle("mp_body_free")
        L.call("mp_body_create", self.verts_c, self.weights, self.V, float(cano_cell), self.storage, self.storage.numel(),
               C.byref(self.handle))

    def set_pose(self, verts_posed, tfs):
        self.verts_p = L.dev(verts_posed, self.device)
        self.tfs = L.dev(tfs.reshape(24, 4, 4), self.device)
        L.call("mp_body_set_pose", self.handle, self.verts_p, self.tfs)

    def deform_inverse(self, x, exact_far=True):
        x = L.dev(x, self.device)
        N = x.shape[0]
        xc = torch.empty(N, 3, device=self.device)
        out = torch.empty(N, dtype=torch.uint8, device=self.device)
        L.call("mp_deform_inverse", self.handle, x, N, xc, out, int(exact_far))
        return xc, out.bool()

    def deform_broyden(self, x, max_steps=10, cvg_threshold=1e-5):
        """Root of forward_skinning(x_c) = x by Broyden's method from the closed-form inverse (row f4, not in the
        reference): returns dict(x_c, residual, converged, outlier, steps)."""
        x = L.dev(x, self.device)
        N = x.shape[0]
        xc = torch.empty(N, 3, device=self.device)
        res = torch.empty(N, device=self.device)
        conv = torch.empty(N, dtype=torch.uint8, device=self.device)
        out = torch.empty(N, dtype=torch.uint8, device=self.device)
        steps = torch.empty(N, dtype=torch.int32, device=self.device)
        L.call("mp_deform_broyden", self.handle, x, N, int(max_steps), float(cvg_threshold), xc, res, conv, out, steps)
        return dict(x_c=xc, residual=res, converged=conv.bool(), outlier=out.bool(), steps=steps)

    def set_root_finder(self, max_steps, cvg_threshold=1e-5):
        """max_steps > 0: every inverse-deformer call on this body refines its non-outlier points with Broyden
        iterations (mp_body_set_root_finder); 0 restores the reference's closed-form inverse."""
        L.call("mp_body_set_root_finder", self.handle, int(max_steps), float(cvg_threshold))

    def forward_jac(self, xc):
        xc = L.dev(xc, self.device)
        N = xc.shape[0]
        xd = torch.empty(N, 3, device=self.device)
        J = torch.empty(N, 9, device=self.device)
        L.call("mp_deform_forward_jac", self.handle, xc, N, xd, J)
        return xd, J

    def deform_inverse_backward(self, x, d_xc, exact_far=True, want_x_c=False):
        """VJP of ``deform_inverse`` at the current pose (mp_deform_inverse_backward): x [N,3], d_xc [N,3] ->
        (d_x [N,3], d_tfs [24,4,4]) and, with ``want_x_c``, the recomputed canonical points."""
        x, d = L.dev(x, self.device), L.dev(d_xc, self.device)
        N = x.shape[0]
        d_x = torch.empty(N, 3, device=self.device)
        d_tfs = torch.empty(24, 4, 4, device=self.device)
        xc = torch.empty(N, 3, device=self.device) if want_x_c else None
        ws = L.workspace(L.call("mp_deform_backward_workspace_bytes", N), self.device)
        L.call("mp_deform_inverse_backward", self.handle, x, N, int(exact_far), d, d_tfs, d_x, xc, ws, ws.numel())
        return (d_x, d_tfs, xc) if want_x_c else (d_x, d_tfs)

    def forward_jac_backward(self, xc, d_xd=None, d_Jinv=None):
        """VJP of ``forward_jac`` at the current pose (mp_deform_forward_jac_backward): xc [N,3], d_xd [N,3] and
        d_Jinv [N,9] (None: zero) -> (d_xc [N,3], d_tfs [24,4,4])."""
        xc = L.dev(xc, self.device)
        N = xc.shape[0]
        d_xd = L.dev(d_xd, self.device)
        d_J = None if d_Jinv is None else L.dev(d_Jinv.reshape(N, 9), self.device)
        d_xc = torch.empty(N, 3, device=self.device)
        d_tfs = torch.empty(24, 4, 4, device=self.device)
        ws = L.workspace(L.call("mp_deform_backward_workspace_bytes", N), self.device)
        L.call("mp_deform_forward_jac_backward", self.handle, xc, N, d_xd, d_J, d_tfs, d_xc, ws, ws.numel())
        return d_xc, d_tfs

    def posed_as(self, pose):
        """Context for a backward: the body posed with ``pose`` = (verts_p, tfs) as a forward saw it, the pose it had
        before restored afterwards (a later frame may have re-posed it in between)."""
        return _Posed(self, pose)


class _Posed:
    def __init__(self, body, pose):
        self.body, self.pose = body, pose

    def __enter__(self):
        b = self.body
        self.prev = (b.verts_p, b.tfs)
        if self.prev[0] is not self.pose[0] or self.prev[1] is not self.pose[1]:
            b.set_pose(*self.pose)
        else:
            self.prev = None
        return b

    def __exit__(self, *exc):
        if self.prev is not None:
            self.body.set_pose(*self.prev)
        return False


class CanonicalMesh:
    """A triangle mesh on the device with its grid of face references (mp_mesh_plan / mp_mesh_create): the canonical
    mesh of one person (multiply.py:118-121, replaced by multiply_model.py:504-506), queried by kaolin's
    point_to_mesh_distance / check_sign (multiply.py:155,158) and the per-ray surface flags (:153-167).  Building it
    reads the grid size back once (one synchronisation); the queries do not synchronise."""

    def __init__(self, verts, faces, margin=0.01, device="cuda"):
        self.device = torch.device(device)
        with torch.cuda.device(self.device):
            v = L.dev(verts.reshape(-1, 3), self.device)
            f = L.dev(torch.as_tensor(faces).reshape(-1, 3), self.device, torch.int64)
            self.V, self.F = v.shape[0], f.shape[0]
            scratch = L.workspace(L.MP_MESH_PLAN_SCRATCH_BYTES, self.device)
            self.plan = L.MeshPlan()
            L.call("mp_mesh_plan", v, self.V, f, self.F, float(margin), scratch, self.plan)
            self.storage = L.workspace(self.plan.storage_bytes, self.device)
            self.handle = L.Handle("mp_mesh_free")
            L.call("mp_mesh_create", self.plan, v, f, self.storage, self.plan.storage_bytes, C.byref(self.handle))
            self._src = (v, f)        # read by the build kernels enqueued above

    @property
    def grid_dims(self):
        return tuple(self.plan.dim)

    def distance(self, pts):
        """pts [N,3] -> (dist2 [N] fp32 squared distance, face_idx [N] int64, dist_type [N] int32), kaolin's
        convention: 0 face interior, 1/2/3 vertex 0/1/2, 4/5/6 edge 01/12/20; ties go to the lowest face index."""
        with torch.cuda.device(self.device):
            p = L.dev(pts.reshape(-1, 3), self.device)
            N = p.shape[0]
            d2 = torch.empty(N, device=self.device)
            fi = torch.empty(N, dtype=torch.int64, device=self.device)
            dt = torch.empty(N, dtype=torch.int32, device=self.device)
            L.call("mp_mesh_distance", self.handle, p, N, d2, fi, dt)
            return d2, fi, dt

    def check_sign(self, pts):
        """pts [N,3] -> inside [N] bool: odd number of crossings of the ray p + t (0,0,1), t > 0."""
        with torch.cuda.device(self.device):
            p = L.dev(pts.reshape(-1, 3), self.device)
            N = p.shape[0]
            ins = torch.empty(N, dtype=torch.uint8, device=self.device)
            L.call("mp_mesh_check_sign", self.handle, p, N, ins)
            return ins.bool()

    def surface_flags(self, x_c, N_samples, threshold=0.05):
        """check_off_in_surface_points_cano_mesh (multiply.py:153-167): x_c [rows*N_samples,3] ->
        (index_off_surface [rows], index_in_surface [rows]) bool."""
        with torch.cuda.device(self.device):
            x = L.dev(x_c.reshape(-1, 3), self.device)
            rows = x.shape[0] // int(N_samples)
            assert rows * int(N_samples) == x.shape[0], "x_c must hold rows * N_samples points"
            off = torch.empty(rows, dtype=torch.uint8, device=self.device)
            ins = torch.empty(rows, dtype=torch.uint8, device=self.device)
            L.call("mp_mesh_surface_flags", self.handle, x, rows, int(N_samples), float(threshold), off, ins)
            return off.bool(), ins.bool()


def camera(R, T, fx, fy, cx, cy):
    """mp_camera_t of a world-to-camera R [3,3], T [3] (OpenCV convention) and the intrinsics, all rounded to fp32."""
    c = L.Camera()
    c.R[:] = [float(x) for x in np.asarray(R, dtype=np.float32).reshape(9)]
    c.T[:] = [float(x) for x in np.asarray(T, dtype=np.float32).reshape(3)]
    c.fx, c.fy, c.cx, c.cy = (float(np.float32(x)) for x in (fx, fy, cx, cy))
    return c


class DepthRaster(torch.autograd.Function):
    """Layer 0 of pytorch3d's hard rasteriser (render.py:135-157) as one autograd node (mp_depth_raster): input verts
    [V,3] (any device; faces [F,3] and the camera are constants), outputs zbuf [H,W] fp32 (-1 where no face covers the
    pixel) and pix_to_face [H,W] int64 (not differentiable), on the device of ``device``.  The backward
    (mp_depth_raster_backward) holds each pixel's face fixed and returns d verts."""

    @staticmethod
    def forward(ctx, cam, H, W, device, verts, faces):
        dev = torch.device(device)
        with torch.cuda.device(dev):
            v = L.dev(verts.reshape(-1, 3), dev)
            f = L.dev(faces.reshape(-1, 3), dev, torch.int64)
            V, F = v.shape[0], f.shape[0]
            ws = L.workspace(L.call("mp_depth_raster_workspace_bytes", H, W, F), dev)
            zbuf = torch.empty(H, W, device=dev)
            p2f = torch.empty(H, W, dtype=torch.int64, device=dev)
            L.call("mp_depth_raster", cam, v if V else None, V, f if F else None, F, H, W, zbuf, p2f, ws, ws.numel())
        ctx.cam, ctx.H, ctx.W, ctx.dev, ctx.verts_in = cam, H, W, dev, verts
        ctx.save_for_backward(v, f, p2f)
        ctx.mark_non_differentiable(p2f)
        return zbuf, p2f

    @staticmethod
    def backward(ctx, d_zbuf, _d_p2f):
        if d_zbuf is None:
            return None, None, None, None, None, None
        v, f, p2f = ctx.saved_tensors
        V, F, dev = v.shape[0], f.shape[0], ctx.dev
        with torch.cuda.device(dev):
            g = L.dev(d_zbuf, dev)
            ws = L.workspace(L.call("mp_depth_raster_backward_workspace_bytes", ctx.H, ctx.W, V), dev)
            d_v = torch.empty(V, 3, device=dev)
            L.call("mp_depth_raster_backward", ctx.cam, v if V else None, V, f if F else None, F, ctx.H, ctx.W, p2f, g,
                   d_v if V else None, ws, ws.numel())
        return None, None, None, None, _grad_like(d_v, ctx.verts_in), None


class Knn1(torch.autograd.Function):
    """pytorch3d.ops.knn_points(p1, p2, K=1, return_nn=True) (multiply_model.py:539) as one autograd node (mp_knn1):
    inputs p1 [N1,3], p2 [N2,3] (N2 >= 1), outputs dists [N1] (squared), idx [N1] int64 (not differentiable) and nn
    [N1,3] = p2[idx], on p1's device.  The backward (mp_knn1_backward) returns d p1 and d p2."""

    @staticmethod
    def forward(ctx, p1, p2):
        dev = p1.device
        with torch.cuda.device(dev):
            a = L.dev(p1.reshape(-1, 3), dev)
            b = L.dev(p2.reshape(-1, 3), dev)
            N1, N2 = a.shape[0], b.shape[0]
            ws = L.workspace(L.call("mp_knn1_workspace_bytes", N1), dev)
            dists = torch.empty(N1, device=dev)
            idx = torch.empty(N1, dtype=torch.int64, device=dev)
            nn = torch.empty(N1, 3, device=dev)
            L.call("mp_knn1", a, N1, b, N2, dists, idx, nn, ws, ws.numel())
        ctx.inputs = (p1, p2)
        ctx.save_for_backward(a, b, idx)
        ctx.mark_non_differentiable(idx)
        return dists, idx, nn

    @staticmethod
    def backward(ctx, d_dists, _d_idx, d_nn):
        a, b, idx = ctx.saved_tensors
        N1, N2, dev = a.shape[0], b.shape[0], a.device
        with torch.cuda.device(dev):
            ws = L.workspace(L.call("mp_knn1_backward_workspace_bytes", N1, N2), dev)
            d_a = torch.empty(N1, 3, device=dev)
            d_b = torch.empty(N2, 3, device=dev)
            L.call("mp_knn1_backward", a, N1, b, N2, idx, L.dev(d_dists, dev), L.dev(d_nn, dev), d_a, d_b, ws,
                   ws.numel())
        p1, p2 = ctx.inputs
        return _grad_like(d_a, p1), _grad_like(d_b, p2)


def marching_cubes(grid, level=0.0, center=(0.0, 0.0, 0.0), extent=None, pad=1.1):
    """Marching cubes (DESIGN §3.7) on a device grid [R+1]*3 (x-major): returns (verts [V,3] fp32 in world space
    ((p / R - 0.5) * pad) * extent + centre, faces [F,3] int64).  extent=None: lattice coordinates (pad 1, extent R,
    centre R/2)."""
    g = L.dev(grid, grid.device)
    R = g.shape[0] - 1
    if extent is None:
        center, extent, pad = (R / 2.0,) * 3, float(R), 1.0
    with torch.cuda.device(g.device):
        ws = L.workspace(L.call("mp_marching_cubes_workspace_bytes", R), g.device)
        V, F = C.c_longlong(0), C.c_longlong(0)
        L.call("mp_marching_cubes_count", g, R, float(level), C.byref(V), C.byref(F), ws, ws.numel())
        verts = torch.empty(V.value, 3, device=g.device)
        faces = torch.empty(F.value, 3, dtype=torch.int64, device=g.device)
        L.call("mp_marching_cubes_emit", g, R, float(level), L.vec3(C.c_double, center), float(extent), float(pad),
               verts if V.value else None, faces if F.value else None, ws, ws.numel())
        return verts, faces


def largest_component(verts, faces):
    """The connected component of largest area (generate_mesh :122-130): (verts [V,3], faces [F,3] int64) of that
    component, in their original order and re-indexed.  No faces: empty tensors."""
    dev = verts.device
    v = L.dev(verts.reshape(-1, 3), dev)
    f = L.dev(faces.reshape(-1, 3), dev, torch.int64)
    V, F = v.shape[0], f.shape[0]
    with torch.cuda.device(dev):
        ws = L.workspace(L.call("mp_largest_component_workspace_bytes", V, F), dev)
        vo = torch.empty(max(V, 1), 3, device=dev)
        fo = torch.empty(max(F, 1), 3, dtype=torch.int64, device=dev)
        Vo, Fo = C.c_int(0), C.c_int(0)
        L.call("mp_largest_component", v if V else None, V, f if F else None, F, vo, fo, C.byref(Vo), C.byref(Fo), ws,
               ws.numel())
        return vo[:Vo.value], fo[:Fo.value]


BETA_MIN = 1e-4      # LaplaceDensity's default (density.py:24)


def sampler_beta(beta_param, beta_min=BETA_MIN):
    """The sampler's and the compositor's beta: |beta_param| + beta_min in fp32, as mp_render_rays forms it."""
    return float(np.float32(abs(np.float32(beta_param))) + np.float32(beta_min))


def samples_per_ray(cfg):
    """n, the samples per ray after the sampler (multiply.py:290-292)."""
    return cfg["N_samples"] + cfg["N_samples_extra"] + 1


def hit_list(ids, device=None):
    """A person's ray ids (tensor or sequence) as a contiguous int64 tensor on ``device`` (default: where they are);
    an empty list becomes ray 0 (multiply.py:262-263)."""
    h = torch.as_tensor(ids, dtype=torch.int64).reshape(-1)
    return (h if h.numel() else torch.zeros(1, dtype=torch.int64)).to(device).contiguous()


def sampler_cfg(cfg, beta_param, beta_min=BETA_MIN):
    c = L.SamplerCfg()
    c.scene_bounding_sphere = cfg["scene_bounding_sphere"]
    c.near = cfg.get("near", 0.0)
    c.N_samples = cfg["N_samples"]
    c.N_samples_eval = cfg["N_samples_eval"]
    c.N_samples_extra = cfg["N_samples_extra"]
    c.eps = cfg["eps"]
    c.beta_iters = cfg["beta_iters"]
    c.max_total_iters = cfg["max_total_iters"]
    c.add_tiny = cfg["add_tiny"]
    c.beta_param = beta_param
    c.beta_min = beta_min
    return c


class Renderer:
    """The fused eval forward (mp_render_rays) over a scene dict as produced by scene.make_scene
    (or assembled from a checkpoint by model.multiply.Multiply)."""

    def __init__(self, scene, device="cuda"):
        self.device = torch.device(device)
        if self.device.index is None:
            self.device = torch.device("cuda", torch.cuda.current_device())
        device = self.device
        self.cfg = scene["cfg"]
        self.beta_param = float(scene["beta_param"])
        self.beta_min = float(scene.get("beta_min", BETA_MIN))
        self.P = len(scene["persons"])
        self.fields, self.bodies = [], []
        with torch.cuda.device(self.device):
            self._build(scene, device)
        self._ws = None
        self._status = None
        self.n = samples_per_ray(self.cfg)

    def _build(self, scene, device):
        for person in scene["persons"]:
            f = Field(person["implicit"], person["render"], background=False, device=device)
            f.set_cond(person["cond"])
            scale = float(person.get("scale", 1.0))
            b = Body(person["verts_c"], person["weights"], cano_cell=0.1001 / max(scale, 1e-3), device=device)
            b.set_pose(person["verts_p"], person["tfs"])
            self.fields.append(f)
            self.bodies.append(b)
        self.bg = None
        if scene.get("bg_implicit") is not None:
            self.bg = Field(scene["bg_implicit"], scene["bg_render"], background=True, device=device)
            self.bg.set_cond(scene["frame_code"])

    def update_person(self, p, person):
        """New pose for person p (per-frame update): cond, posed vertices, bone transforms."""
        with torch.cuda.device(self.device):
            self.fields[p].set_cond(person["cond"])
            self.bodies[p].set_pose(person["verts_p"], person["tfs"])

    def check_status(self):
        """Raises if the last render saw a ray that misses the bounding sphere — where the reference prints
        'BOUNDING SPHERE PROBLEM!' and exits (rend_util.py:140-142).  Reads one device int (synchronises)."""
        if self._status is not None and int(self._status.item()) & 1:
            raise RuntimeError("BOUNDING SPHERE PROBLEM! (a camera ray misses the r=%g scene sphere)"
                               % self.cfg["scene_bounding_sphere"])

    def render(self, inputs, hit_lists, debug=False, persons=None, check=False, out=None, train=None):
        """inputs: uv [1,R,2], pose [1,4,4], intrinsics [1,4,4] (CUDA or CPU tensors);
        hit_lists: per rendered person either an int64 tensor of ray ids (empty -> ray 0, multiply.py:262-263) or a
        pair (ids [R] int64 on the device, count [1] int32 on the device) as produced by ``ray_aabb_hits`` — the
        count then never visits the host;
        persons: indices of the persons to render (default: all; ``Multiply.forward(input, id=p)`` passes [p],
        multiply.py:244-247) — ``acc_person_list`` has one column per rendered person;
        check: read the bounding-sphere status flag after the call (synchronises) and raise like the reference;
        out: optional dict of preallocated contiguous output tensors (e.g. ``parallel.PixelBuffer.views``);
        train: training-mode VALUES (mp_train_t): dict(rng=[per rendered person the tabled draws of
        ``ErrorBoundSampler.draw_training_rng``], t_rand_bg=[R,32] or None) — stochastic sampling, no outlier clamp,
        jittered background depths; adds ``z_eik_{k}`` [R_k] per person.  With ``meshes=[CanonicalMesh per rendered
        person]`` (current_epoch < 250, multiply.py:313-316) and ``threshold`` (default 0.05) it also returns
        ``index_off_surface`` / ``index_in_surface`` [R] bool, merged over persons as multiply.py:549-560.  With
        ``beta=<0-d tensor>`` (the LaplaceDensity beta, equal to the fp32 |beta_param| + beta_min the sampler uses) the
        five pixel outputs are attached to beta's graph through ``RenderComposite``: ``out["samples"]`` is a list of
        per-person dicts of leaf tensors (sdf [R_k,n], rgb / normal [R_k,n,3], which require grad; plus z_vals [R_k,n+1]
        and ray_index [R_k]) and, when a background is rendered, ``out["samples_bg"]`` holds its leaves (sdf [R,32],
        rgb [R,32,3] in the flipped depth order; plus t_rand, the jitter of its depths or None, and bg_rgb [R,3]).  Backward fills their ``.grad``
        and beta's; the networks, deformer and SMPL inputs stay outside the graph.
        Returns the eval output dict of Multiply.forward (multiply.py:589-598)."""
        with torch.cuda.device(self.device):
            return self._render(inputs, hit_lists, debug, persons, check, out, train)

    def _render(self, inputs, hit_lists, debug, persons, check, out_bufs=None, train=None):
        dev = self.device
        uv = L.dev(inputs["uv"].reshape(-1, 2), dev)
        pose = L.dev(inputs["pose"].reshape(4, 4), dev)
        K = L.dev(inputs["intrinsics"].reshape(4, 4), dev)
        R = uv.shape[0]
        plist = list(range(self.P)) if persons is None else [int(p) for p in persons]
        Pn = len(plist)
        assert len(hit_lists) == Pn, "one hit list per rendered person"
        sc = L.Scene()
        sc.sampler = sampler_cfg(self.cfg, self.beta_param, self.beta_min)
        sc.P = Pn
        hits = []
        dev_counts = False
        for k, p in enumerate(plist):
            h = hit_lists[k]
            cnt = None
            if isinstance(h, (tuple, list)):
                h, cnt = h
                assert h.is_cuda and cnt.is_cuda and h.dtype == torch.int64 and cnt.dtype == torch.int32
                dev_counts = True
                h = h.to(dev).contiguous()
            else:
                h = hit_list(h, dev)
            hits.append((h, cnt))
            sc.body[k] = self.bodies[p].handle
            sc.field[k] = self.fields[p].handle
            sc.hit_index[k] = L.ptr(h)
            sc.hit_count[k] = h.numel()
            sc.hit_count_dev[k] = L.ptr(cnt)
        sc.bg_field = self.bg.handle if self.bg is not None else None
        keep_train = []
        z_eik = {}
        flags = {}
        beta = train.get("beta") if train is not None else None
        grad_on = beta is not None
        if grad_on:
            assert torch.is_tensor(beta) and beta.numel() == 1, "train['beta'] must be a 0-d tensor"
            want = sampler_beta(self.beta_param, self.beta_min)
            assert np.float32(float(beta.detach())) == want, \
                "train['beta'] = %r differs from the sampler's beta %r" % (float(beta.detach()), want)
            assert not dev_counts, "render gradients need host-side hit counts"
        if train is not None:
            assert not dev_counts, "training mode needs host-side hit counts"
            tr = L.Train()
            for k in range(Pn):
                rs, kp = sampler_rng_struct(train["rng"][k], dev)
                keep_train += [rs, kp]
                tr.rng[k] = C.pointer(rs)
                z_eik[k] = torch.empty(hits[k][0].numel(), device=dev)
                tr.z_eik[k] = L.ptr(z_eik[k])
            tb = L.dev(train.get("t_rand_bg"), dev)
            keep_train.append(tb)
            tr.t_rand_bg = L.ptr(tb)
            meshes = train.get("meshes")
            if meshes is not None:
                assert len(meshes) == Pn and all(m is not None for m in meshes), "one canonical mesh per rendered person"
                for k, m in enumerate(meshes):
                    tr.cano_mesh[k] = m.handle
                keep_train.append(list(meshes))
                tr.surface_threshold = float(train.get("threshold", 0.05))
                flags = {"index_off_surface": torch.empty(R, dtype=torch.uint8, device=dev),
                         "index_in_surface": torch.empty(R, dtype=torch.uint8, device=dev)}
                tr.index_off_surface = L.ptr(flags["index_off_surface"])
                tr.index_in_surface = L.ptr(flags["index_in_surface"])
            keep_train.append(tr)
            sc.train = C.pointer(tr)
        need = L.call("mp_render_workspace_bytes", sc, R)
        if self._ws is None or self._ws.numel() < need:
            self._ws = L.workspace(need, dev)
        if self._status is None:
            self._status = torch.zeros(1, dtype=torch.int32, device=dev)
        out = L.RenderOut()
        shapes = {"rgb_values": (R, 3), "fg_rgb_values": (R, 3), "normal_values": (R, 3), "acc_map": (R,),
                  "acc_person_list": (R, Pn)}
        if out_bufs is not None:
            res = {k: out_bufs[k] for k in shapes}
            for k, shp in shapes.items():
                assert res[k].dtype == torch.float32 and tuple(res[k].shape) == shp, k
        else:
            res = {k: torch.empty(*shp, device=dev) for k, shp in shapes.items()}
        for k, v in res.items():
            setattr(out, k, L.ptr(v))
        out.status = L.ptr(self._status)
        taps = {}
        if debug or grad_on:       # per-sample taps: debug outputs and the compositor's inputs for RenderComposite
            n = self.n
            taps["bg_T"] = torch.empty(R, device=dev)
            out.bg_T = L.ptr(taps["bg_T"])
            for k in range(Pn):
                Rp = hits[k][0].numel()
                for name, shp in (("z_vals", (Rp, n + 1)), ("sdf", (Rp, n)), ("rgb", (Rp, n, 3)), ("normals", (Rp, n, 3))):
                    taps[f"{name}_{k}"] = torch.empty(*shp, device=dev)
                    getattr(out, name)[k] = L.ptr(taps[f"{name}_{k}"])
        dbg = {}
        if debug:
            assert not dev_counts, "debug taps need host-side hit counts"
            dbg = {"trips": torch.zeros(Pn, dtype=torch.int32, device=dev), **taps}
            out.trips = L.ptr(dbg["trips"])
        if grad_on and self.bg is not None:
            for name, shp in (("bg_rgb", (R, 3)), ("bg_sdf", (R, 32)), ("bg_rgb_samples", (R, 32, 3))):
                taps[name] = torch.empty(*shp, device=dev)
                setattr(out, name, L.ptr(taps[name]))
        L.call("mp_render_rays", sc, uv, pose, K, R, out, self._ws, self._ws.numel())
        self._keep = (uv, pose, K, hits, keep_train)
        for k, v in z_eik.items():
            dbg[f"z_eik_{k}"] = v
        for k, v in flags.items():
            res[k] = v.bool()
        if check:
            self.check_status()
        if grad_on:
            res.update(self._attach_graph(res, taps, hits, beta, train.get("t_rand_bg"), R, Pn))
        res.update(dbg)
        return res

    def _attach_graph(self, res, taps, hits, beta, t_rand_bg, R, Pn):
        dev = self.device
        samples = [dict(sdf=taps[f"sdf_{k}"].clone().requires_grad_(True), rgb=taps[f"rgb_{k}"].clone().requires_grad_(True),
                        normal=taps[f"normals_{k}"].clone().requires_grad_(True), z_vals=taps[f"z_vals_{k}"], ray_index=hits[k][0])
                   for k in range(Pn)]
        leaves = [t for d in samples for t in (d["sdf"], d["rgb"], d["normal"])]
        extra = {}
        info = dict(n=self.n, R=R, P=Pn, beta=float(beta.detach()), hits=[h[0] for h in hits], z=[d["z_vals"] for d in samples],
                    bg_T=taps["bg_T"], bound=float(self.cfg["scene_bounding_sphere"]), device=dev, bg=None)
        if self.bg is not None:
            t_rand = L.dev(t_rand_bg, dev)
            bg = dict(sdf=taps["bg_sdf"].clone().requires_grad_(True),
                      rgb=taps["bg_rgb_samples"].clone().requires_grad_(True), t_rand=t_rand, bg_rgb=taps["bg_rgb"])
            leaves += [bg["sdf"], bg["rgb"]]
            info["bg"] = dict(rgb=taps["bg_rgb"], t_rand=t_rand)
            extra["samples_bg"] = bg
        names = ("rgb_values", "fg_rgb_values", "normal_values", "acc_map", "acc_person_list")
        outs = RenderComposite.apply(info, tuple(res[k] for k in names), beta, *leaves)
        extra.update(zip(names, outs))
        extra["samples"] = samples
        return extra


class RenderComposite(torch.autograd.Function):
    """The compositing stages of Multiply.forward as one autograd node: inputs beta (0-d) and the per-sample leaves
    (per rendered person sdf, rgb, normal; then the background's sdf and rgb when one is rendered), outputs rgb_values,
    fg_rgb_values, normal_values, acc_map, acc_person_list.  The forward returns the pixels the fused render already
    produced (nothing is recomputed); the backward runs mp_final_compose_backward, mp_composite_backward and
    mp_bg_composite_backward on the current stream.  d_beta is dL/dbeta of beta itself; the |beta_param| + beta_min
    chain is ordinary torch on the parameter."""

    @staticmethod
    def forward(ctx, info, pixels, beta, *leaves):
        ctx.info = info
        ctx.beta_shape = beta.shape
        ctx.save_for_backward(*leaves)
        return tuple(p.detach() for p in pixels)

    @staticmethod
    def backward(ctx, d_rgb, d_fgv, d_nrm, d_acc, d_accp):
        info = ctx.info
        leaves = ctx.saved_tensors
        dev, R, P, n = info["device"], info["R"], info["P"], info["n"]
        d_rgb, d_fgv, d_nrm, d_acc, d_accp = (L.dev(t, dev) for t in (d_rgb, d_fgv, d_nrm, d_acc, d_accp))
        with torch.cuda.device(dev):
            if d_rgb is None:
                d_rgb = torch.zeros(R, 3, device=dev)
            bg = info["bg"]
            d_fg = torch.empty(R, 3, device=dev)
            d_bgT = torch.empty(R, device=dev)
            d_bg = torch.empty(R, 3, device=dev) if bg is not None else None
            L.call("mp_final_compose_backward", info["bg_T"], bg["rgb"] if bg else None, R, d_rgb, d_fgv, d_fg, d_bgT, d_bg)
            arr = person_samples([(info["hits"][k], info["z"][k], *leaves[3 * k: 3 * k + 3], info["hits"][k].numel())
                                  for k in range(P)])
            gr = (L.PersonSampleGrads * P)()
            grads = []
            for k in range(P):
                gk = tuple(torch.empty_like(t) for t in leaves[3 * k: 3 * k + 3])
                gr[k].d_sdf, gr[k].d_rgb, gr[k].d_normal = (L.ptr(t) for t in gk)
                grads += gk
            d_beta = torch.empty(1, device=dev)
            ws = L.workspace(L.call("mp_composite_backward_workspace_bytes", R, P), dev)
            L.call("mp_composite_backward", arr, P, R, n, info["beta"], d_fg, d_nrm, d_acc, d_accp, d_bgT, gr, d_beta, ws,
                   ws.numel())
            if bg is not None:
                b_sdf, b_rgb = leaves[3 * P], leaves[3 * P + 1]
                d_bsdf, d_brgb = torch.empty_like(b_sdf), torch.empty_like(b_rgb)
                L.call("mp_bg_composite_backward", b_sdf, b_rgb, R, info["bound"], bg["t_rand"], d_bg, d_bsdf, d_brgb)
                grads += [d_bsdf, d_brgb]
        return (None, None, d_beta.reshape(ctx.beta_shape)) + tuple(grads)


def _grad_like(g, t):
    """A gradient computed on the device, in the shape, dtype and device of the input ``t`` it belongs to."""
    return g.reshape(t.shape).to(device=t.device, dtype=t.dtype)


def _first_order(name):
    """Refuses a backward that builds a graph (create_graph=True): the networks' backward is first order only."""
    def wrap(fn):
        @functools.wraps(fn)
        def backward(ctx, *grads):
            if torch.is_grad_enabled():
                raise NotImplementedError("%s: second-order gradients (create_graph=True) are not implemented; the "
                                          "networks' backward is first order (DESIGN.md §7)" % name)
            return fn(ctx, *grads)
        return backward
    return wrap


class ImplicitFunction(torch.autograd.Function):
    """ImplicitNet.forward on a packed ``Field`` as one autograd node: inputs x [N,d_in], cond [cond_dim] (any shape of
    that size) and the effective parameters W_0, b_0, ..., W_8, b_8 (W = g v / ||v|| where weight-normed, so autograd
    carries dW to g and v); output [N,257] = (sdf | feature), from the field's forward call.  The backward runs
    mp_implicit_backward on the current stream with the cond of this forward."""

    @staticmethod
    def forward(ctx, field, x, cond, *params):
        field.set_cond(cond)
        sdf, feat = field.implicit_forward(x)
        ctx.field, ctx.inputs = field, (x, cond) + params
        ctx.save_for_backward(L.dev(x, field.device), L.dev(cond, field.device))
        return torch.cat([sdf[:, None], feat], 1)

    @staticmethod
    @_first_order("ImplicitFunction")
    @torch.autograd.function.once_differentiable
    def backward(ctx, d_out):
        x, cond = ctx.saved_tensors
        f, need = ctx.field, ctx.needs_input_grad
        with torch.cuda.device(f.device):
            f.set_cond(cond)         # a later forward may have conditioned the field differently
            d = L.dev(d_out, f.device)
            r = f.implicit_backward(x, d[:, 0].contiguous(), d[:, 1:].contiguous(), want_x=need[1],
                                    want_params=any(need[3:]), want_cond=need[2])
        grads = [None, None if r["d_x"] is None else _grad_like(r["d_x"], ctx.inputs[0]),
                 None if r["d_cond"] is None else _grad_like(r["d_cond"], ctx.inputs[1])]
        for l in range(len(f.imp_shapes)):
            for g, t in ((r["d_weight"][l], ctx.inputs[2 + 2 * l]), (r["d_bias"][l], ctx.inputs[3 + 2 * l])):
                grads.append(None if g is None else _grad_like(g, t))
        return tuple(grads)


class RenderFunction(torch.autograd.Function):
    """RenderingNet.forward 'pose_no_view' on a packed ``Field`` as one autograd node: inputs points [N,3], normals
    [N,3], body_pose [69] (any shape of that size), feature_vectors [N,256] and the parameters W_0, b_0, ..., W_4, b_4
    (effective weights), lin_pose.weight [8,69], lin_pose.bias [8]; output rgb [N,3] from the field's forward call.  The
    backward runs mp_render_backward on the current stream with the body_pose of this forward."""

    @staticmethod
    def forward(ctx, field, points, normals, body_pose, feat, *params):
        field.set_cond(body_pose)
        rgb = field.render_forward(points, normals, feat)
        ctx.field, ctx.inputs = field, (points, normals, body_pose, feat) + params
        ctx.save_for_backward(*(L.dev(t, field.device) for t in (points, normals, body_pose, feat)))
        return rgb

    @staticmethod
    @_first_order("RenderFunction")
    @torch.autograd.function.once_differentiable
    def backward(ctx, d_rgb):
        points, normals, body_pose, feat = ctx.saved_tensors
        f, need = ctx.field, ctx.needs_input_grad
        with torch.cuda.device(f.device):
            f.set_cond(body_pose)
            r = f.render_backward(points, normals, feat, d_rgb, want_inputs=any(need[1:3]) or need[4],
                                  want_params=any(need[5:-2]), want_pose=need[3] or any(need[-2:]))
        n = len(f.ren_shapes)
        outs = [r["d_points"], r["d_normals"], r["d_body_pose"], r["d_feat"]]
        for l in range(n):
            outs += [r["d_weight"][l], r["d_bias"][l]]
        outs += [r["d_lin_pose_weight"], r["d_lin_pose_bias"]]
        return (None,) + tuple(None if g is None or not nd else _grad_like(g, t)
                               for g, t, nd in zip(outs, ctx.inputs, need[1:]))


class SmplFunction(torch.autograd.Function):
    """SMPLServer.forward (mp_smpl_forward) as one autograd node: inputs scale [1], transl [3], thetas [72], betas [10]
    (any shapes with those sizes, on any device), outputs smpl_verts [V,3], smpl_tfs [24,4,4].  ``server`` provides
    ``_run(s, t, th, b, absolute)`` -> (verts, tfs, device inputs) and ``_backward(inputs, absolute, d_verts, d_tfs)``
    -> (d_scale, d_transl, d_thetas, d_betas), the latter mp_smpl_backward on the current stream."""

    @staticmethod
    def forward(ctx, server, absolute, scale, transl, thetas, betas):
        verts, tfs, dev_inputs = server._run(scale, transl, thetas, betas, absolute)
        ctx.server, ctx.absolute = server, absolute
        ctx.inputs = (scale, transl, thetas, betas)
        ctx.save_for_backward(*dev_inputs)
        return verts, tfs

    @staticmethod
    def backward(ctx, d_verts, d_tfs):
        grads = ctx.server._backward(ctx.saved_tensors, ctx.absolute, d_verts, d_tfs)
        return (None, None) + tuple(None if g is None else _grad_like(g, t) for g, t in zip(grads, ctx.inputs))


class DeformInverse(torch.autograd.Function):
    """SMPLDeformer.forward(x, smpl_tfs, inverse=True) on a posed ``Body`` (mp_deform_inverse) as an autograd node:
    inputs x [N,3] and the smpl_tfs [24,4,4] the body is posed with; outputs x_c [N,3] and the outlier mask (not
    differentiable).  The backward runs mp_deform_inverse_backward on the current stream, at the pose of the forward."""

    @staticmethod
    def forward(ctx, body, exact_far, x, tfs):
        xc, outlier = body.deform_inverse(x, exact_far=exact_far)
        ctx.body, ctx.exact_far, ctx.pose = body, exact_far, (body.verts_p, body.tfs)
        ctx.inputs = (x, tfs)
        ctx.save_for_backward(L.dev(x, body.device))
        ctx.mark_non_differentiable(outlier)
        return xc, outlier

    @staticmethod
    def backward(ctx, d_xc, _d_outlier):
        x_in, tfs_in = ctx.inputs
        if d_xc is None:
            return None, None, None, None
        (x,) = ctx.saved_tensors
        with ctx.body.posed_as(ctx.pose) as b:
            d_x, d_tfs = b.deform_inverse_backward(x, d_xc, exact_far=ctx.exact_far)
        return None, None, _grad_like(d_x, x_in), _grad_like(d_tfs, tfs_in)


class ForwardJac(torch.autograd.Function):
    """SMPLDeformer.forward_skinning and the inverse Jacobian of Multiply.forward_gradient on a posed ``Body``
    (mp_deform_forward_jac) as one autograd node: inputs x_c [N,3] and the smpl_tfs [24,4,4] the body is posed with;
    outputs x_d [N,3] and Jinv [N,9].  The backward runs mp_deform_forward_jac_backward on the current stream."""

    @staticmethod
    def forward(ctx, body, xc, tfs):
        xd, J = body.forward_jac(xc)
        ctx.body, ctx.pose = body, (body.verts_p, body.tfs)
        ctx.inputs = (xc, tfs)
        ctx.save_for_backward(L.dev(xc, body.device))
        return xd, J

    @staticmethod
    def backward(ctx, d_xd, d_J):
        xc_in, tfs_in = ctx.inputs
        (xc,) = ctx.saved_tensors
        with ctx.body.posed_as(ctx.pose) as b:
            d_xc, d_tfs = b.forward_jac_backward(xc, d_xd, d_J)
        return None, _grad_like(d_xc, xc_in), _grad_like(d_tfs, tfs_in)


def person_samples(persons):
    """mp_person_samples_t array from per-person (ray_index, z_vals, sdf, rgb, normal, n_rows); the caller keeps the
    tensors alive while the array is in use."""
    arr = (L.PersonSamples * len(persons))()
    for a, (idx, z, sdf, rgb, nrm, n_rows) in zip(arr, persons):
        a.ray_index, a.z_vals, a.sdf, a.rgb, a.normal = (L.ptr(t) for t in (idx, z, sdf, rgb, nrm))
        a.n_rows = n_rows
    return arr


def sampler_rng_struct(rng, dev):
    """mp_sampler_rng_t from the tabled draws of ``ErrorBoundSampler.draw_training_rng`` (t_rand [R,E], u_final [R,S],
    extra_perm [T,T*E] int32, eik_idx [T,R] int32, t_rand_bg [T,R,32]); returns (struct, tensors to keep alive)."""
    keep = {k: L.dev(rng[k], dev, torch.int32 if k in ("extra_perm", "eik_idx") else torch.float32)
            for k in ("t_rand", "u_final", "extra_perm", "eik_idx", "t_rand_bg")}
    r = L.SamplerRng()
    for k, v in keep.items():
        setattr(r, k, L.ptr(v))
    return r, keep


class GraphedRender:
    """One eval forward captured in a CUDA graph and replayed: the ~60 kernel launches, memsets and the stream fork/join
    of mp_render_rays become a single graph launch (the sampler trips and the MLP tile counts are read from device
    memory, so nothing in the launch configuration depends on the data).  The input tensors are static device buffers —
    write new rays / camera into ``uv`` / ``pose`` / ``intrinsics`` (and new hit ids / counts into the hit-list
    tensors given at capture) and ``replay()``; poses are updated as usual through ``Renderer.update_person``."""

    def __init__(self, renderer, inputs, hit_lists, persons=None):
        self.r = renderer
        dev = renderer.device
        self.inputs = {k: L.dev(inputs[k], dev).clone() for k in ("uv", "pose", "intrinsics")}
        self.hits = [tuple(t.to(dev) for t in h) if isinstance(h, (tuple, list)) else h.to(dev).clone() for h in hit_lists]
        self.persons = persons
        with torch.cuda.device(dev):
            side = torch.cuda.Stream()
            side.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(side):
                for _ in range(2):                      # warm-up outside the capture: lazy resources, workspace size
                    renderer.render(self.inputs, self.hits, persons=persons)
            torch.cuda.current_stream().wait_stream(side)
            torch.cuda.synchronize()
            self.graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(self.graph):
                self.out = renderer.render(self.inputs, self.hits, persons=persons)

    def replay(self):
        self.graph.replay()
        return self.out


def ray_aabb_hits(cam_loc, ray_dirs, verts, inflate=1.2):
    """Device-side culling against the x`inflate` axis-aligned box of `verts` [V,3] (multiply.py:208-214 uses trimesh's
    oriented box; see INTEGRATION.md): returns (ids [R] int64, count [1] int32), both on the device, the list already
    finalised (empty -> ray 0, multiply.py:262-263).  No host synchronisation: feed the pair to ``Renderer.render``."""
    dev = cam_loc.device
    cam, d, v = L.dev(cam_loc, dev), L.dev(ray_dirs, dev), L.dev(verts.reshape(-1, 3), dev)
    R = cam.shape[0]
    with torch.cuda.device(dev):
        idx = torch.empty(R, dtype=torch.int64, device=dev)
        cnt = torch.zeros(1, dtype=torch.int32, device=dev)
        box = torch.empty(8, dtype=torch.float64, device=dev)
        L.call("mp_ray_aabb_hits", cam, d, R, v, v.shape[0], float(inflate), idx, cnt, box)
    return idx, cnt


def ray_box_hits(cam_loc, ray_dirs, center, half_extent, rot=None, device_count=False):
    """Device-side ray / box culling (mp_ray_box_hits): sorted int64 ray ids that hit the box.  One scalar
    device->host read for the count — the reference pays a full `.cpu()` round trip plus trimesh here
    (multiply.py:256).  ``device_count=True`` returns (ids [R], count [1]) with the count left on the device and the
    list finalised (empty -> ray 0, mp_hit_list_finalize), the form ``Renderer.render`` takes without a host read."""
    dev = cam_loc.device
    cam, d = L.dev(cam_loc, dev), L.dev(ray_dirs, dev)
    R = cam.shape[0]
    with torch.cuda.device(dev):
        idx = torch.empty(R, dtype=torch.int64, device=dev)
        cnt = torch.zeros(1, dtype=torch.int32, device=dev)
        rot_d = None if rot is None else L.dev(torch.as_tensor(rot).reshape(9), dev, torch.float64)
        L.call("mp_ray_box_hits", cam, d, R, L.vec3(C.c_double, center), L.vec3(C.c_double, half_extent), rot_d, idx, cnt)
        if device_count:
            L.call("mp_hit_list_finalize", idx, cnt)
            return idx, cnt
    return idx[: int(cnt.item())]
