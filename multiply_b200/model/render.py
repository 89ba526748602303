"""lib/model/render.py:Renderer for opt_depth's depth maps (multiply_model.py:393-401), on the device kernels of
csrc/raster.cu (engine.DepthRaster).

Only the hard depth map is provided: ``render_multiple_depth_map`` returns layer 0 of pytorch3d's zbuf, the one layer
opt_depth reads (:396-401), with gradients to the vertices.  The shaded and soft renderers (render.py:104-133) are not
provided: the soft silhouette term runs only on the ``depth_end: False`` path, at weight 0 in every shipped config.
The definition the kernels follow is oracle/raster.py's (DESIGN §3.8)."""
import numpy as np
import torch

from .. import engine
from ..utils.data import decompose_projection


def camera_from_projection(P, scale):
    """MultiplyModel.get_renderer's camera (multiply_model.py:553-576) without cv2: P [3,4] or [4,4] and the SMPL scale
    s -> (K [3,3], R [3,3], T [3]) in float64, with K, R, c = decomposeProjectionMatrix((P @ diag(s, s, s, 1))[:3])
    (K not normalised by K[2,2], as cv2 returns it) and T = -R c[:3] / c[3]."""
    P_norm = np.eye(4)
    P = np.asarray(P, dtype=np.float64)
    P_norm[:P.shape[0], :] = P
    P_norm = P_norm @ np.diag([scale, scale, scale, 1.0])
    K, R, c = decompose_projection(P_norm[:3, :])
    T = -R @ (c[:3] / c[3])
    return K, R, T


class Renderer:
    """render.py:Renderer.  ``cam_intrinsic`` [3,3] gives fx, fy, cx, cy (K[0,0], K[1,1], K[0,2], K[1,2], the skew and
    K[2,2] ignored, render.py:38-42); ``img_size`` = (H, W) of the depth maps (render.py:65); ``focal_length`` and
    ``principal_point`` are ignored as the reference ignores them.  The camera starts at R = I, T = 0 (OpenCV
    convention; the reference's default pytorch3d R = diag(-1, -1, 1) is that camera)."""

    def __init__(self, focal_length=None, principal_point=None, img_size=None, cam_intrinsic=None):
        K = np.asarray(cam_intrinsic, dtype=np.float64)
        self.cam_intrinsic = cam_intrinsic
        self.image_size = (int(img_size[0]), int(img_size[1]))
        self.intrinsics = (K[0, 0], K[1, 1], K[0, 2], K[1, 2])
        self.set_camera(torch.eye(3)[None], torch.zeros(1, 3))

    def set_camera(self, R, T):
        """R [1,3,3], T [1,3]: world-to-camera rotation and translation in OpenCV's convention (get_renderer's
        render_R / render_T, multiply_model.py:567-574); set_camera's flips (render.py:73-78) only translate them into
        pytorch3d's convention, so they are applied as given."""
        R = torch.as_tensor(R).detach().float().cpu().reshape(3, 3).numpy()
        T = torch.as_tensor(T).detach().float().cpu().reshape(3).numpy()
        self.cam = engine.camera(R, T, *self.intrinsics)

    def render_multiple_depth_map(self, verts_list, faces_list, verts_colors_list=None):
        """render.py:135-157: per person, verts [1,V,3] and faces [1,F,3] -> depth map [1,H,W,1] (layer 0 of zbuf: the
        nearest face's view-space depth, -1 where no face covers the pixel), differentiable in verts, on the vertices'
        device.  verts_colors_list is accepted and unused, as for the depth map in the reference."""
        H, W = self.image_size
        out = []
        for v, f in zip(verts_list, faces_list):
            zbuf, _ = engine.DepthRaster.apply(self.cam, H, W, v.device, v, f)
            out.append(zbuf[None, :, :, None])
        return out

    def render_multiple_meshes(self, verts_list, faces_list, verts_colors_list):
        raise NotImplementedError("Renderer provides the hard depth map of opt_depth only (render_multiple_depth_map); "
                                  "the shaded renderer is not implemented")

    def softrender_multiple_meshes(self, verts_list, faces_list, verts_colors_list):
        raise NotImplementedError("Renderer provides the hard depth map of opt_depth only (render_multiple_depth_map); "
                                  "the soft silhouette renderer (depth_end: False, weight 0 in the shipped configs) is "
                                  "not implemented")
