"""TEST INFRASTRUCTURE ONLY — CPU definitions of the kaolin mesh queries the reference's training branch calls, and
the training forward at current_epoch < 250 on top of oracle/port.py.

kaolin 0.13.0 (README of the reference): ``point_to_mesh_distance`` / ``check_sign`` / ``index_vertices_by_faces``,
called by Multiply.check_off_in_surface_points_cano_mesh (multiply.py:153-167) and
MultiplyModel.get_interpenetration_loss (multiply_model.py:532).  kaolin is absent and unpinned, so the functions here
are the DEFINITIONS the CUDA kernels (multiply_b200/csrc/mesh.cu) are checked against ("parity unpinned" at that
boundary, like port.py's knn_points / nerfacc restatements): fp64 brute force over all faces, each step written in the
order mesh.cu performs it (mesh.cu is compiled without FMA contraction), so that both round identically.  Every
function runs on the device of its ``points`` argument (CPU in the CPU tests, CUDA in the GPU tests).

All ``file:line`` cites are relative to /root/reference/code.
"""
import torch

from . import port


def index_vertices_by_faces(vertices_features, faces):
    """kaolin.ops.mesh.index_vertices_by_faces: [B,V,D], [F,3] -> [B,F,3,D]."""
    return vertices_features[:, faces.long()]


def _dot(a, b):
    return a[..., 0] * b[..., 0] + a[..., 1] * b[..., 1] + a[..., 2] * b[..., 2]


def _closest_point_triangle(p, a, b, c):
    """Squared distance from p [...,3] to triangle (a, b, c) [...,3] (fp64) and the region of the closest point
    (Ericson, Real-Time Collision Detection 5.1.5): 0 face interior, 1/2/3 vertex a/b/c, 4/5/6 edge ab/bc/ca.  The
    first matching case of the sequence wins, as in mesh.cu:point_triangle_d2."""
    ab, ac, ap = b - a, c - a, p - a
    d1, d2 = _dot(ab, ap), _dot(ac, ap)
    bp = p - b
    d3, d4 = _dot(ab, bp), _dot(ac, bp)
    vc = d1 * d4 - d3 * d2
    cp = p - c
    d5, d6 = _dot(ab, cp), _dot(ac, cp)
    vb = d5 * d2 - d1 * d6
    va = d3 * d6 - d5 * d4
    e43, e56 = d4 - d3, d5 - d6
    den = 1.0 / (va + vb + vc)
    q0 = (a + (vb * den)[..., None] * ab) + (vc * den)[..., None] * ac
    q4 = a + (d1 / (d1 - d3))[..., None] * ab
    q6 = a + (d2 / (d2 - d6))[..., None] * ac
    q5 = b + (e43 / (e43 + e56))[..., None] * (c - b)
    cases = [(d1 <= 0) & (d2 <= 0), (d3 >= 0) & (d4 <= d3), (vc <= 0) & (d1 >= 0) & (d3 <= 0), (d6 >= 0) & (d5 <= d6),
             (vb <= 0) & (d2 >= 0) & (d6 <= 0), (va <= 0) & (e43 >= 0) & (e56 >= 0)]
    pts = [a.expand_as(q0), b.expand_as(q0), q4, c.expand_as(q0), q6, q5]
    types = [1, 2, 4, 3, 6, 5]
    q, t = q0, torch.zeros(q0.shape[:-1], dtype=torch.int32, device=q0.device)
    for cond, qq, tt in zip(cases[::-1], pts[::-1], types[::-1]):      # last assignment = first matching case
        q = torch.where(cond[..., None], qq, q)
        t = torch.where(cond, torch.full_like(t, tt), t)
    d = p - q
    return _dot(d, d), t


def point_to_mesh_distance(points, face_vertices, chunk_pairs=1 << 22, return_second=False):
    """kaolin.metrics.trianglemesh.point_to_mesh_distance: points [1,N,3], face_vertices [1,F,3,3] ->
    (distance [1,N] fp32 SQUARED distance to the nearest face, face_idx [1,N] int64, dist_type [1,N] int32).

    dist_type follows kaolin's documented convention: 0 = the closest point is inside the face, 1/2/3 = vertex 0/1/2,
    4/5/6 = edge 01/12/20.  kaolin is not installed here, so which of its outputs break exact ties, and how it labels
    a point equidistant from two regions, are unconfirmed: this definition takes the lowest face index and the first
    region of the sequence 1, 2, 4, 3, 6, 5, 0 (Ericson's case order).  Arithmetic: fp64 on the fp32 inputs, squared
    distance rounded to fp32 at the end.  return_second: also the second-smallest squared distance over the other faces
    (fp64, [N]) — where the two are close the nearest face is ambiguous.  Runs on the device of ``points``."""
    assert points.shape[0] == 1 and face_vertices.shape[0] == 1
    x = points[0].double()
    fv = face_vertices[0].double().to(x.device)
    N, Fn = x.shape[0], fv.shape[0]
    a, b, c = fv[None, :, 0], fv[None, :, 1], fv[None, :, 2]
    step = max(1, chunk_pairs // max(Fn, 1))
    d2 = torch.empty(N, dtype=torch.float64, device=x.device)
    second = torch.empty(N, dtype=torch.float64, device=x.device)
    idx = torch.empty(N, dtype=torch.int64, device=x.device)
    typ = torch.empty(N, dtype=torch.int32, device=x.device)
    for s in range(0, N, step):
        p = x[s:s + step, None]
        d, t = _closest_point_triangle(p, a, b, c)
        # a (near-)degenerate face can reach the face-interior case with va + vb + vc == 0 and get a NaN distance: it
        # has no distance and is skipped, as mesh.cu's comparisons skip it (its edges are other faces' edges)
        d = torch.where(torch.isnan(d), torch.full_like(d, float("inf")), d)
        m = d.min(1)[0]
        i = (d == m[:, None]).int().argmax(1)          # lowest index among exact ties
        d2[s:s + step], idx[s:s + step] = m, i
        typ[s:s + step] = t.gather(1, i[:, None])[:, 0]
        if return_second:
            second[s:s + step] = d.scatter(1, i[:, None], float("inf")).min(1)[0] if Fn > 1 else float("inf")
    out = (d2.float()[None], idx[None], typ[None])
    return out + (second,) if return_second else out


def _ray_z_crossing(p, fa, fb, fc):
    """Crossing parameter t of the ray p + t (0,0,1) with triangle (a, b, c), or -1 (t <= 0 or no crossing); p [...,3],
    corners [...,3] fp64.  Edge functions U (b->c), V (c->a), W (a->b) of the corners relative to p; a zero edge
    function counts only for the edge that points up or exactly left in counter-clockwise order (so of two faces that
    share an edge from opposite sides exactly one counts a ray through it).  mesh.cu:ray_z_crossing."""
    a, b, c = fa - p, fb - p, fc - p
    U = b[..., 0] * c[..., 1] - b[..., 1] * c[..., 0]
    V = c[..., 0] * a[..., 1] - c[..., 1] * a[..., 0]
    W = a[..., 0] * b[..., 1] - a[..., 1] * b[..., 0]
    den = U + V + W
    s = torch.where(den > 0, 1.0, -1.0).to(den.dtype)
    U, V, W = U * s, V * s, W * s

    def owns(dx, dy):
        return (dy > 0) | ((dy == 0) & (dx < 0))
    ok = (den != 0) & (U >= 0) & (V >= 0) & (W >= 0)
    ok &= (U != 0) | owns(s * (c[..., 0] - b[..., 0]), s * (c[..., 1] - b[..., 1]))
    ok &= (V != 0) | owns(s * (a[..., 0] - c[..., 0]), s * (a[..., 1] - c[..., 1]))
    ok &= (W != 0) | owns(s * (b[..., 0] - a[..., 0]), s * (b[..., 1] - a[..., 1]))
    t = (U * a[..., 2] + V * b[..., 2] + W * c[..., 2]) / (s * den)
    return torch.where(ok & (t > 0), t, torch.full_like(t, -1.0))


def check_sign(verts, faces, points, chunk_pairs=1 << 22):
    """kaolin.ops.mesh.check_sign: verts [1,V,3], faces [F,3], points [1,N,3] -> inside [1,N] bool.

    Definition: inside iff the ray p + t (0,0,1), t > 0, crosses the mesh an odd number of times (fp64 edge functions
    on the fp32 inputs, a crossing exactly on a shared edge or vertex counted once, _ray_z_crossing).  kaolin casts its
    own ray; for a watertight mesh the parity does not depend on the direction away from the surface.  Like kaolin's,
    the result is meaningful for watertight meshes only.  Runs on the device of ``points``."""
    assert verts.shape[0] == 1 and points.shape[0] == 1
    x = points[0].double()
    fv = verts[0].double().to(x.device)[faces.long().to(x.device)]
    N, Fn = x.shape[0], fv.shape[0]
    a, b, c = fv[None, :, 0], fv[None, :, 1], fv[None, :, 2]
    step = max(1, chunk_pairs // max(Fn, 1))
    out = torch.empty(N, dtype=torch.bool, device=x.device)
    for s in range(0, N, step):
        t = _ray_z_crossing(x[s:s + step, None], a, b, c)
        out[s:s + step] = ((t > 0).sum(1) % 2) == 1
    return out[None]


def check_off_in_surface(x_cano, N_samples, verts, faces, threshold=0.05):
    """Multiply.check_off_in_surface_points_cano_mesh (multiply.py:153-167) on the definitions above:
    x_cano [rows*N_samples,3] -> (index_off_surface [rows], index_in_surface [rows]) bool and the per-row minimum of
    the signed distance [rows] (fp32)."""
    distance, _, _ = point_to_mesh_distance(x_cano.unsqueeze(0).contiguous(), index_vertices_by_faces(verts[None], faces))
    distance = torch.sqrt(distance)
    sign = check_sign(verts[None], faces, x_cano.unsqueeze(0)).float()
    sign = 1 - 2 * sign
    signed_distance = sign * distance
    batch_size = x_cano.shape[0] // N_samples
    signed_distance = signed_distance.reshape(batch_size, N_samples, 1)
    minimum = torch.min(signed_distance, 1)[0]
    return (minimum > threshold).squeeze(1), (minimum <= 0.).squeeze(1), minimum.squeeze(1)


def multiply_forward(scene, inputs, hit_lists, train, epoch, meshes=None, threshold=0.05, **kw):
    """port.multiply_forward(train=...) — the values of Multiply.forward's training branch — plus, at epoch < 250, the
    surface flags of multiply.py:313-316 (``check_off_in_surface_points_cano_mesh`` on every person's canonical samples)
    merged over persons as :549-560.  ``meshes`` = per person (verts [V,3], faces [F,3]) of the canonical mesh.
    Adds 'index_off_surface' / 'index_in_surface' ([R] bool, None at epoch >= 250) and, at epoch < 250, the per-person
    rows of the person's hit list: '_off_p' / '_in_p' (bool) and '_min_p' (the row minimum of the signed distance)."""
    out = port.multiply_forward(scene, inputs, hit_lists, train=train, **dict(kw, return_samples=True))
    out["index_off_surface"] = out["index_in_surface"] = None
    if epoch >= 250:
        return out
    P = len(scene["persons"])
    assert meshes is not None and len(meshes) == P, "epoch < 250 needs one canonical mesh per person"
    ray_dirs, cam_loc = port.get_camera_params(inputs["uv"], inputs["pose"], inputs["intrinsics"])
    R = ray_dirs.shape[1]
    cam_loc = cam_loc.unsqueeze(1).repeat(1, R, 1).reshape(-1, 3)
    ray_dirs = ray_dirs.reshape(-1, 3)
    off = torch.ones(R, P, dtype=torch.bool)
    inn = torch.zeros(R, P, dtype=torch.bool)
    out["_off_p"], out["_in_p"], out["_min_p"] = [], [], []
    for p in range(P):
        idx = hit_lists[p]
        if idx.numel() == 0:
            idx = torch.tensor([0], dtype=torch.int64)                  # multiply.py:262-263
        co, do = cam_loc[idx], ray_dirs[idx]
        z_vals = out["_z_vals"][p]
        n = z_vals.shape[1]
        # the main pass's samples and canonical points, exactly as port.multiply_forward forms them (multiply.py:295-308)
        pts = (co.unsqueeze(1) + z_vals.unsqueeze(2) * do.unsqueeze(1)).reshape(-1, 3)
        _, x_c, _ = port.sdf_func_with_smpl_deformer(pts, scene["persons"][p], scene["cfg"], training=True)
        o, i, mn = check_off_in_surface(x_c, n, meshes[p][0], meshes[p][1], threshold)       # multiply.py:313-316
        off[idx, p] = o                                                 # multiply.py:549-560
        inn[idx, p] = i
        out["_off_p"].append(o)
        out["_in_p"].append(i)
        out["_min_p"].append(mn)
    out["index_off_surface"] = torch.all(off, dim=1)
    out["index_in_surface"] = torch.any(inn, dim=1)
    return out
