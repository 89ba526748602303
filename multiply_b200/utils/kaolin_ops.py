"""Drop-ins for the kaolin calls of the reference, on the device kernels of csrc/mesh.cu (engine.CanonicalMesh):

    kaolin.metrics.trianglemesh.point_to_mesh_distance   multiply.py:155
    kaolin.ops.mesh.check_sign                            multiply.py:158, multiply_model.py:532
    kaolin.ops.mesh.index_vertices_by_faces               multiply.py:121

Shapes and return conventions are kaolin's (batch size 1).  Each call builds the mesh's grid (one synchronisation);
callers that query one mesh repeatedly keep an ``engine.CanonicalMesh`` instead.  The definitions the kernels are
checked against are oracle/mesh_port.py's."""
import torch

from .. import engine


def index_vertices_by_faces(vertices_features, faces):
    """[B,V,D], [F,3] -> [B,F,3,D]."""
    return vertices_features[:, faces.long()]


def point_to_mesh_distance(points, face_vertices):
    """points [1,N,3], face_vertices [1,F,3,3] (CUDA) -> (squared distance [1,N] fp32, face index [1,N] int64,
    distance type [1,N] int32: 0 face interior, 1/2/3 vertex 0/1/2, 4/5/6 edge 01/12/20).  Ties go to the lowest
    face index."""
    assert points.dim() == 3 and points.shape[0] == 1, "points must be [1,N,3]"
    assert face_vertices.dim() == 4 and face_vertices.shape[0] == 1 and face_vertices.shape[2:] == (3, 3)
    F = face_vertices.shape[1]
    dev = points.device
    verts = face_vertices[0].reshape(-1, 3)
    faces = torch.arange(3 * F, dtype=torch.int64, device=dev).reshape(F, 3)
    m = engine.CanonicalMesh(verts, faces, device=dev)
    d2, idx, typ = m.distance(points[0])
    return d2[None], idx[None], typ[None]


def check_sign(verts, faces, points):
    """verts [1,V,3], faces [F,3], points [1,N,3] (CUDA) -> inside [1,N] bool: odd number of crossings of the ray
    p + t (0,0,1), t > 0, with the mesh.  Meaningful for watertight meshes only, as kaolin's."""
    assert verts.dim() == 3 and verts.shape[0] == 1 and points.dim() == 3 and points.shape[0] == 1
    m = engine.CanonicalMesh(verts[0], faces, device=points.device)
    return m.check_sign(points[0])[None]
