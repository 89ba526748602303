"""TEST INFRASTRUCTURE ONLY — CPU definition of the hard depth map opt_depth reads from pytorch3d's rasteriser.

Renderer.render_multiple_depth_map (lib/model/render.py:135-157) rasterises each person's posed mesh with
RasterizationSettings(faces_per_pixel=10, blur_radius=0) (render.py:65-66) and returns zbuf; opt_depth reads only layer
0 (multiply_model.py:396-401).  pytorch3d is absent and unpinned, so this restatement is the DEFINITION the CUDA
kernels (multiply_b200/csrc/raster.cu) are checked against ("parity unpinned" at that boundary, DESIGN §3.8):

  * camera: (X, Y, Z) = R v + T, u = fx X / Z + cx, v = fy Y / Z + cy (OpenCV's projection, which the flips of
    set_camera, render.py:73-78, turn into pytorch3d's convention and back);
  * pixel (r, c) samples (c + 0.5, r + 0.5) (pytorch3d's pixel centres);
  * a face with a vertex at Z <= 0 or of zero projected area is skipped (pytorch3d differs only for faces crossing the
    camera plane, which posed bodies in front of the camera never do);
  * a face covers a sample when the sample lies in the closed projected triangle (edge functions, signed by the area,
    >= 0: blur radius 0 keeps signed distance <= 0, so edge pixels count);
  * depth z = 1 / (b0 / Z0 + b1 / Z1 + b2 / Z2) with the screen barycentrics (perspective-correct), fp64 on the fp32
    inputs, rounded to fp32 once; zbuf = the smallest fp32 depth, ties to the lowest face index; -1 where no face
    covers the pixel, pix_to_face likewise.

Every step is written in the order raster.cu performs it (raster.cu is compiled without FMA contraction), so both round
identically.  Each face enumerates only the pixels of its clipped screen box, which keeps full-size images with 3 x 10^5
faces fast on the CPU.

All ``file:line`` cites are relative to /root/reference/code.
"""
import numpy as np
import torch


def camera_record(R, T, K):
    """The fp32 camera the renderer holds: R [3,3], T [3] (render_R / render_T of get_renderer, cast to float as
    multiply_model.py:570-571 does) and fx, fy, cx, cy = K[0,0], K[1,1], K[0,2], K[1,2] (render.py:38-42)."""
    f32 = lambda x: torch.as_tensor(np.asarray(x, dtype=np.float64)).float()
    K = np.asarray(K, dtype=np.float64)
    return dict(R=f32(R).reshape(3, 3), T=f32(T).reshape(3),
                fx=float(np.float32(K[0, 0])), fy=float(np.float32(K[1, 1])),
                cx=float(np.float32(K[0, 2])), cy=float(np.float32(K[1, 2])))


def project(cam, verts):
    """verts [...,3] (fp32 values) -> X, Y, Z, u, v (fp64), rounded step by step as raster.cu:tri_setup."""
    R, T = cam["R"].double(), cam["T"].double()
    x, y, z = verts[..., 0].double(), verts[..., 1].double(), verts[..., 2].double()
    X = ((R[0, 0] * x + R[0, 1] * y) + R[0, 2] * z) + T[0]
    Y = ((R[1, 0] * x + R[1, 1] * y) + R[1, 2] * z) + T[1]
    Z = ((R[2, 0] * x + R[2, 1] * y) + R[2, 2] * z) + T[2]
    u = (cam["fx"] * X) / Z + cam["cx"]
    v = (cam["fy"] * Y) / Z + cam["cy"]
    return X, Y, Z, u, v


def _edge(u, v, i, px, py):
    j, k = (i + 1) % 3, (i + 2) % 3
    return (u[..., j] - px) * (v[..., k] - py) - (v[..., j] - py) * (u[..., k] - px)


def face_depth(tri, px, py, cam):
    """Differentiable fp64 closed form of one face's depth at samples: tri [N,3,3] world-space vertices (fp64, any
    autograd graph), px, py [N] -> z [N] (not rounded).  The depth backward of raster.cu is its exact derivative."""
    _, _, Z, u, v = project(cam, tri)
    A = (u[:, 1] - u[:, 0]) * (v[:, 2] - v[:, 0]) - (v[:, 1] - v[:, 0]) * (u[:, 2] - u[:, 0])
    b = [_edge(u, v, i, px, py) / A for i in range(3)]
    s = (b[0] / Z[:, 0] + b[1] / Z[:, 1]) + b[2] / Z[:, 2]
    return 1.0 / s


def rasterize(cam, verts, faces, H, W):
    """verts [V,3] fp32, faces [F,3] int -> dict of zbuf [H,W] fp32, pix_to_face [H,W] int64 and the decisions'
    margins: ``edge_margin`` [H,W] fp64, the smallest |edge function / area| over every (face, pixel) pair whose box
    holds the pixel and whose other two edges pass (the distance of the inside test from flipping, in barycentric
    units; +inf where no face's box holds the pixel), and ``depth_gap`` [H,W] fp64, the fp64 depth of the second
    nearest covering face minus the nearest's (+inf with fewer than two)."""
    verts = torch.as_tensor(verts).float()
    faces = torch.as_tensor(faces).long().reshape(-1, 3)
    V, F = verts.shape[0], faces.shape[0]
    n = H * W
    zbuf = torch.full((n,), -1.0, dtype=torch.float32)
    p2f = torch.full((n,), -1, dtype=torch.int64)
    margin = torch.full((n,), float("inf"), dtype=torch.float64)
    gap = torch.full((n,), float("inf"), dtype=torch.float64)
    out = dict(zbuf=zbuf.reshape(H, W), pix_to_face=p2f.reshape(H, W), edge_margin=margin.reshape(H, W),
               depth_gap=gap.reshape(H, W))
    if F == 0:
        return out
    valid = ((faces >= 0) & (faces < V)).all(1)
    fv = verts[faces.clamp(0, max(V - 1, 0))]                           # [F,3,3]
    X, Y, Z, u, v = project(cam, fv)
    A = (u[:, 1] - u[:, 0]) * (v[:, 2] - v[:, 0]) - (v[:, 1] - v[:, 0]) * (u[:, 2] - u[:, 0])
    valid &= (Z > 0).all(1) & (A.abs() > 0)
    ulo = torch.minimum(torch.minimum(u[:, 0], u[:, 1]), u[:, 2])
    uhi = torch.maximum(torch.maximum(u[:, 0], u[:, 1]), u[:, 2])
    vlo = torch.minimum(torch.minimum(v[:, 0], v[:, 1]), v[:, 2])
    vhi = torch.maximum(torch.maximum(v[:, 0], v[:, 1]), v[:, 2])
    c0 = torch.clamp(torch.ceil(ulo - 0.5), min=0.0)
    c1 = torch.clamp(torch.floor(uhi - 0.5), max=float(W - 1))
    r0 = torch.clamp(torch.ceil(vlo - 0.5), min=0.0)
    r1 = torch.clamp(torch.floor(vhi - 0.5), max=float(H - 1))
    valid &= (c0 <= c1) & (r0 <= r1)
    f_ok = torch.nonzero(valid).reshape(-1)
    if f_ok.numel() == 0:
        return out
    c0, c1, r0, r1 = (t[f_ok].long() for t in (c0, c1, r0, r1))
    nc, nr = c1 - c0 + 1, r1 - r0 + 1
    cnt = nc * nr
    fi = torch.repeat_interleave(torch.arange(f_ok.numel()), cnt)       # (face, pixel) pairs, face by face
    start = torch.cumsum(cnt, 0) - cnt
    q = torch.arange(int(cnt.sum())) - start[fi]
    r = r0[fi] + q // nc[fi]
    c = c0[fi] + q % nc[fi]
    px, py = c.double() + 0.5, r.double() + 0.5
    uu, vv, ZZ, AA = u[f_ok][fi], v[f_ok][fi], Z[f_ok][fi], A[f_ok][fi]
    e = [_edge(uu, vv, i, px, py) for i in range(3)]
    pos = AA > 0
    inside_i = [torch.where(pos, ei >= 0, ei <= 0) for ei in e]
    inside = inside_i[0] & inside_i[1] & inside_i[2]
    pix = r * W + c
    # margin of the inside decision: |b_i| of an edge whose two partners pass (flipping it alone flips the decision)
    b_abs = [(ei / AA).abs() for ei in e]
    m = torch.full_like(px, float("inf"))
    for i in range(3):
        others = inside_i[(i + 1) % 3] & inside_i[(i + 2) % 3]
        m = torch.where(others, torch.minimum(m, b_abs[i]), m)
    margin.scatter_reduce_(0, pix, m, reduce="amin")
    s = (e[0] / AA / ZZ[:, 0] + e[1] / AA / ZZ[:, 1]) + e[2] / AA / ZZ[:, 2]
    z64 = 1.0 / s
    z32 = z64.float()
    face = f_ok[fi]
    key = z32.view(torch.int32).long() * (1 << 32) + face       # positive fp32 depths order like their bits
    key = torch.where(inside, key, torch.full_like(key, torch.iinfo(torch.int64).max))
    best = torch.full((n,), torch.iinfo(torch.int64).max, dtype=torch.int64)
    best.scatter_reduce_(0, pix, key, reduce="amin")
    hit = best != torch.iinfo(torch.int64).max
    zbuf[hit] = (best[hit] >> 32).to(torch.int32).view(torch.float32)
    p2f[hit] = best[hit] & 0xFFFFFFFF
    # depth gap: the second smallest fp64 depth among covering faces
    zin = torch.where(inside, z64, torch.full_like(z64, float("inf")))
    first = torch.full((n,), float("inf"), dtype=torch.float64).scatter_reduce_(0, pix, zin, reduce="amin")
    won = inside & (face == p2f[pix])
    rest = torch.where(won, torch.full_like(zin, float("inf")), zin)
    second = torch.full((n,), float("inf"), dtype=torch.float64).scatter_reduce_(0, pix, rest, reduce="amin")
    gap.copy_(torch.where(hit, second - first, gap))
    return out


def depth_map(cam, verts, faces, H, W):
    """The float64 depth map with gradients: verts [V,3] (fp64, any autograd graph) -> [1,H,W,1], the nearest face's
    unrounded depth face_depth where rasterize (on verts rounded to fp32) finds one, -1 elsewhere.  Faces are chosen
    as the device chooses them and held fixed, as the depth backward holds them."""
    faces = torch.as_tensor(faces).long().reshape(-1, 3)
    p2f = rasterize(cam, verts.detach().float(), faces, H, W)["pix_to_face"].reshape(-1)
    hit = torch.nonzero(p2f >= 0).reshape(-1)
    px, py = (hit % W).double() + 0.5, (hit // W).double() + 0.5
    z = face_depth(verts[faces[p2f[hit]]], px, py, cam)
    out = torch.full((H * W,), -1.0, dtype=verts.dtype).index_put((hit,), z)
    return out.reshape(1, H, W, 1)
