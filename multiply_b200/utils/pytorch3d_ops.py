"""Drop-in for the pytorch3d.ops call of the reference's interpenetration loss, on the device kernels of csrc/raster.cu
(engine.Knn1):

    pytorch3d.ops.knn_points(p1, p2, K=1, return_nn=True)      multiply_model.py:539

Shapes and return conventions are pytorch3d's (batch size 1).  The definition the kernels follow is
oracle/port.py:knn_points: squared distance (dx*dx + dy*dy) + dz*dz in fp32, ties to the lowest index."""
from .. import engine


def knn_points(p1, p2, K=1, return_nn=True):
    """p1 [1,N1,3], p2 [1,N2,3] (CUDA, N2 >= 1) -> (dists [1,N1,1] squared distances, idx [1,N1,1] int64, nn [1,N1,1,3]
    = p2[idx] or None), differentiable in p1 and p2 through dists and nn.  Only K = 1 is provided."""
    if K != 1:
        raise NotImplementedError("knn_points: only K = 1 is provided (the interpenetration loss's use)")
    assert p1.dim() == 3 and p1.shape[0] == 1 and p2.dim() == 3 and p2.shape[0] == 1, "p1, p2 must be [1,N,3]"
    dists, idx, nn = engine.Knn1.apply(p1[0], p2[0])
    return dists[None, :, None], idx[None, :, None], (nn[None, :, None, :] if return_nn else None)
