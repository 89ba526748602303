"""Mirror of /root/reference/code/lib/utils/mesh.py:generate_mesh (:78-132).

The reference extracts a canonical mesh by letting the MISE octree (lib/libmise, Cython, host) ask
``func(points) -> {'occ': sdf}`` for batches of lattice points (``Multiply.query_oc``, multiply.py:169-172), then runs
skimage's marching cubes and keeps trimesh's connected component of largest area.  ``generate_mesh`` here runs all of
it on the device (mp_mise, mp_marching_cubes_*, mp_largest_component; DESIGN §3.7 states the marching-cubes tiling and
how it differs from skimage's).  ``dense_sdf_grid`` evaluates the whole (res+1)^3 lattice of the finest MISE level in
one call (mp_sdf_grid), and ``lattice_points`` reproduces generate_mesh's point mapping for callers that keep the
octree loop and call ``Multiply.query_oc`` batch by batch."""
import numpy as np
import torch


def bounds(verts, scale=1.1):
    """generate_mesh:80-86: centre, longest side of the tight SMPL box, padding factor."""
    v = verts.detach().cpu().numpy().reshape(-1, 3)
    bbox = np.stack([v.min(axis=0), v.max(axis=0)], axis=0)
    return (bbox[0] + bbox[1]) * 0.5, (bbox[1] - bbox[0]).max(), scale


def lattice_points(idx, resolution, center, extent, scale=1.1):
    """generate_mesh:92-95 for integer lattice coordinates idx [N,3] -> fp32 points [N,3] (numpy arithmetic)."""
    p = idx.astype(np.float32)
    p = (p / resolution - 0.5) * scale
    return p * extent + center


def _field(model, person_id, cond):
    dev = next(model.parameters()).device
    f = model._ensure_renderer(dev).fields[person_id]
    c = cond["smpl"] if isinstance(cond, dict) else cond
    return dev, f, c


def dense_sdf_grid(model, person_id, cond, verts, res=256, scale=1.1):
    """SDF of person ``person_id`` on the dense (res+1)^3 lattice around ``verts`` (the canonical SMPL vertices the
    reference passes, multiply_model.py:941-945).  ``model``: model.multiply.Multiply mirror.  Returns a device tensor
    [res+1, res+1, res+1]."""
    center, extent, pad = bounds(verts, scale)
    dev, f, c = _field(model, person_id, cond)
    with torch.cuda.device(dev):
        f.set_cond(c.detach())
        return f.sdf_grid(center, extent, res, pad)


def generate_mesh(model, person_id, cond, verts, level_set=0, res_init=32, res_up=3):
    """generate_mesh(func, verts, level_set, res_init, res_up) with func = person ``person_id``'s canonical SDF under
    ``cond`` (what the reference's ``lambda x: model.query_oc(x, cond, person_id)`` evaluates): MISE on the
    (res_init << res_up)^3 lattice around ``verts``, marching cubes, largest component.  Returns (verts [V,3] fp32,
    faces [F,3] int64) as device tensors, the input of ``Multiply.set_canonical_mesh``; an SDF without a sign change
    gives V = F = 0 (the reference returns None there)."""
    center, extent, pad = bounds(verts)
    dev, f, c = _field(model, person_id, cond)
    with torch.cuda.device(dev):
        f.set_cond(c.detach())
        v, fc, _ = f.extract_mesh(center, extent, int(res_init), int(res_up), float(level_set), pad)
        return v, fc
