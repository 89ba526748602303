"""Mirror of /root/reference/code/lib/utils/rend_util.py (the two functions on the hot path)."""
import torch
import torch.nn.functional as F

from .. import _lib as L


def get_camera_params_host(uv, pose, intrinsics):
    """Host (CPU) evaluation of get_camera_params (rend_util.py:45-87) used only to build
    ray/box hit lists, which the reference also computes on the host (multiply.py:256).
    Returns (ray_dirs [R,3], cam_loc [R,3])."""
    pose = pose_matrix(pose)
    cam_loc = pose[:, :3, 3]
    b, n, _ = uv.shape
    x = uv[:, :, 0].view(b, -1)
    y = uv[:, :, 1].view(b, -1)
    z = torch.ones((b, n))
    fx, fy = intrinsics[:, 0, 0], intrinsics[:, 1, 1]
    cx, cy, sk = intrinsics[:, 0, 2], intrinsics[:, 1, 2], intrinsics[:, 0, 1]
    xl = (x - cx[:, None] + cy[:, None] * sk[:, None] / fy[:, None] - sk[:, None] * y / fy[:, None]) / fx[:, None] * z
    yl = (y - cy[:, None]) / fy[:, None] * z
    pts = torch.stack((xl, yl, z, torch.ones_like(z)), dim=-1).permute(0, 2, 1)
    world = torch.bmm(pose, pts).permute(0, 2, 1)[:, :, :3]
    dirs = F.normalize(world - cam_loc[:, None, :], dim=2)
    return dirs.reshape(-1, 3), cam_loc[:, None, :].expand(-1, n, -1).reshape(-1, 3)


def pose_matrix(pose):
    """The two pose forms rend_util.get_camera_params accepts (rend_util.py:46-54): a [B,4,4] camera-to-world matrix is
    returned as is; a [B,7] vector (unit-normalised quaternion w,x,y,z | camera centre) is expanded with the rotation of
    ``quat_to_rot`` (:88-105).  A handful of scalar operations on the host side of the call."""
    if pose.dim() == 3:
        return pose
    if tuple(pose.shape) == (4, 4):
        return pose[None]
    if pose.dim() != 2 or pose.shape[1] != 7:
        raise ValueError("pose must be [B,4,4] or [B,7] (quaternion | centre), got %s" % (tuple(pose.shape),))
    q = F.normalize(pose[:, :4].float(), dim=1)
    w, x, y, z = q[:, 0], q[:, 1], q[:, 2], q[:, 3]
    rows = [1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + w * y),
            2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w),
            2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]
    out = torch.eye(4, device=pose.device, dtype=torch.float32).repeat(pose.shape[0], 1, 1)
    out[:, :3, :3] = torch.stack(rows, dim=1).reshape(-1, 3, 3)
    out[:, :3, 3] = pose[:, 4:].float()
    return out


def camera_rays(uv, pose, intrinsics):
    """mp_camera_rays on uv's device: uv [R,2] (or [1,R,2]), pose and intrinsics as ``get_camera_params`` takes them ->
    (ray_dirs [R,3], cam_loc [R,3], the camera centre once per ray)."""
    dev = uv.device
    u, p, k = (L.dev(t, dev) for t in (uv.reshape(-1, 2), pose_matrix(pose).reshape(4, 4), intrinsics.reshape(4, 4)))
    R = u.shape[0]
    dirs = torch.empty(R, 3, device=dev)
    cam = torch.empty(R, 3, device=dev)
    L.call("mp_camera_rays", u, p, k, R, dirs, cam)
    return dirs, cam


def get_camera_params(uv, pose, intrinsics):
    """rend_util.get_camera_params (rend_util.py:45-72) on the device: uv [1,R,2], pose [1,4,4] (or [1,7] quaternion
    form), intrinsics [1,4,4] -> (ray_dirs [1,R,3], cam_loc [1,3])."""
    dirs, cam = camera_rays(uv, pose, intrinsics)
    return dirs[None], cam[:1]


def get_sphere_intersections(cam_loc, ray_directions, r=1.0):
    """rend_util.get_sphere_intersections (rend_util.py:131-147): [R,3],[R,3] -> [R,2]; raises where the reference
    calls exit() (a ray missing the bounding sphere)."""
    dev = cam_loc.device
    c, d = L.dev(cam_loc, dev), L.dev(ray_directions, dev)
    R = c.shape[0]
    out = torch.empty(R, 2, device=dev)
    flag = torch.zeros(1, dtype=torch.int32, device=dev)
    L.call("mp_sphere_intersections", c, d, R, float(r), out, flag)
    if int(flag.item()):
        raise RuntimeError("BOUNDING SPHERE PROBLEM!")
    return out
