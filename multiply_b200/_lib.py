"""ctypes binding of libmultiply_b200.so (the C ABI declared in include/multiply_b200.h).

There is no fallback: if the shared library is missing the import of anything that needs it
raises, and every entry point raises ``MpError`` with the library's error text on failure.

The product package reaches the library through ``call`` alone: it refuses a tensor the kernels could not read (host
memory, a strided view) before anything is enqueued, and names the failing function from the table, not from the caller.
"""
import ctypes as C
import os

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("MP_LIB") or os.path.join(HERE, "libmultiply_b200.so")     # MP_LIB: A/B builds (scripts/)

MP_MAX_LAYERS = 12
MP_MAX_PERSONS = 8
# layout of mp_profile_read_stalls' array: [4 program kinds][MP_STALL_WARPS][MP_STALL_WORDS]
MP_STALL_PHASES, MP_STALL_PROLOGUE, MP_STALL_ELAPSED, MP_STALL_WORDS, MP_STALL_WARPS = 6, 42, 43, 44, 9

c_float_p = C.POINTER(C.c_float)
c_int_p = C.POINTER(C.c_int)


class MpError(RuntimeError):
    pass


class LinearStack(C.Structure):
    _fields_ = [("n_layers", C.c_int),
                ("weight_v", C.c_void_p * MP_MAX_LAYERS),
                ("weight_g", C.c_void_p * MP_MAX_LAYERS),
                ("bias", C.c_void_p * MP_MAX_LAYERS),
                ("in_dim", C.c_int * MP_MAX_LAYERS),
                ("out_dim", C.c_int * MP_MAX_LAYERS)]


class ImplicitDesc(C.Structure):
    _fields_ = [("lin", LinearStack), ("d_in", C.c_int), ("multires", C.c_int), ("cond_dim", C.c_int),
                ("skip_layer", C.c_int)]


class RenderDesc(C.Structure):
    _fields_ = [("lin", LinearStack), ("mode", C.c_int), ("multires_view", C.c_int),
                ("lin_pose_weight", C.c_void_p), ("lin_pose_bias", C.c_void_p)]


class LinearGrads(C.Structure):
    _fields_ = [("d_weight", C.c_void_p * MP_MAX_LAYERS), ("d_bias", C.c_void_p * MP_MAX_LAYERS)]


class SamplerCfg(C.Structure):
    _fields_ = [("scene_bounding_sphere", C.c_float), ("near", C.c_float), ("N_samples", C.c_int),
                ("N_samples_eval", C.c_int), ("N_samples_extra", C.c_int), ("eps", C.c_float),
                ("beta_iters", C.c_int), ("max_total_iters", C.c_int), ("add_tiny", C.c_float),
                ("beta_param", C.c_float), ("beta_min", C.c_float)]


class SamplerRng(C.Structure):
    _fields_ = [("t_rand", C.c_void_p), ("u_final", C.c_void_p), ("extra_perm", C.c_void_p), ("eik_idx", C.c_void_p),
                ("t_rand_bg", C.c_void_p)]


class PersonSamples(C.Structure):
    _fields_ = [("n_rows", C.c_int), ("ray_index", C.c_void_p), ("z_vals", C.c_void_p), ("sdf", C.c_void_p),
                ("rgb", C.c_void_p), ("normal", C.c_void_p)]


class Train(C.Structure):
    _fields_ = [("rng", C.POINTER(SamplerRng) * MP_MAX_PERSONS), ("z_eik", C.c_void_p * MP_MAX_PERSONS),
                ("t_rand_bg", C.c_void_p),
                ("cano_mesh", C.c_void_p * MP_MAX_PERSONS), ("surface_threshold", C.c_float),
                ("index_off_surface", C.c_void_p), ("index_in_surface", C.c_void_p)]


MP_MESH_PLAN_SCRATCH_BYTES = 1024


class MeshPlan(C.Structure):
    _fields_ = [("V", C.c_int), ("F", C.c_int), ("lo", C.c_double * 3), ("h", C.c_double), ("dim", C.c_int * 3),
                ("n_refs", C.c_longlong), ("storage_bytes", C.c_size_t)]


class Camera(C.Structure):
    _fields_ = [("R", C.c_float * 9), ("T", C.c_float * 3), ("fx", C.c_float), ("fy", C.c_float), ("cx", C.c_float),
                ("cy", C.c_float)]


class Scene(C.Structure):
    _fields_ = [("sampler", SamplerCfg), ("P", C.c_int),
                ("body", C.c_void_p * MP_MAX_PERSONS), ("field", C.c_void_p * MP_MAX_PERSONS),
                ("bg_field", C.c_void_p),
                ("hit_index", C.c_void_p * MP_MAX_PERSONS), ("hit_count", C.c_int * MP_MAX_PERSONS),
                ("hit_count_dev", C.c_void_p * MP_MAX_PERSONS), ("train", C.POINTER(Train))]


class RenderOut(C.Structure):
    _fields_ = [("rgb_values", C.c_void_p), ("fg_rgb_values", C.c_void_p), ("normal_values", C.c_void_p),
                ("acc_map", C.c_void_p), ("acc_person_list", C.c_void_p),
                ("z_vals", C.c_void_p * MP_MAX_PERSONS), ("sdf", C.c_void_p * MP_MAX_PERSONS),
                ("rgb", C.c_void_p * MP_MAX_PERSONS), ("normals", C.c_void_p * MP_MAX_PERSONS),
                ("trips", C.c_void_p), ("bg_T", C.c_void_p), ("status", C.c_void_p),
                ("bg_rgb", C.c_void_p), ("bg_sdf", C.c_void_p), ("bg_rgb_samples", C.c_void_p)]


class PersonSampleGrads(C.Structure):
    _fields_ = [("d_sdf", C.c_void_p), ("d_rgb", C.c_void_p), ("d_normal", C.c_void_p)]


# Two markers stand in the table for a C type and tell ``call`` what the header's convention is:
STATUS = "int: 0, or an error code with its text in mp_last_error()"      # every other restype is a value
STREAM = "void* stream, the last parameter: the current stream unless the caller passes one"
_CTYPE = {STATUS: C.c_int, STREAM: C.c_void_p}

# name -> (restype, argtypes) ; mirrors include/multiply_b200.h one to one
_VP, _I, _F, _SZ = C.c_void_p, C.c_int, C.c_float, C.c_size_t
SIGNATURES = {
    "mp_version": (_I, []),
    "mp_last_error": (C.c_char_p, []),
    "mp_device_sm_count": (_I, []),
    "mp_linspace_host": (STATUS, [_F, _F, _I, c_float_p]),
    "mp_launch_count": (C.c_longlong, [_I]),
    "mp_field_pack_bytes": (_SZ, [C.POINTER(ImplicitDesc), C.POINTER(RenderDesc), _I]),
    "mp_field_pack": (STATUS, [C.POINTER(ImplicitDesc), C.POINTER(RenderDesc), _I, _VP, _SZ, C.POINTER(_VP), STREAM]),
    "mp_field_free": (None, [_VP]),
    "mp_field_set_cond": (STATUS, [_VP, _VP, STREAM]),
    "mp_set_engine": (STATUS, [_I]),
    "mp_get_engine": (_I, []),
    "mp_set_precision": (STATUS, [_I]),
    "mp_get_precision": (_I, []),
    "mp_profile_enable": (STATUS, [_I]),
    "mp_set_streams": (STATUS, [_I]),
    "mp_profile_read": (STATUS, [C.POINTER(C.c_double), C.POINTER(C.c_longlong), C.POINTER(C.c_double), _I]),
    "mp_profile_read_stalls": (STATUS, [C.POINTER(C.c_ulonglong), _I]),
    "mp_implicit_forward": (STATUS, [_VP, _VP, _I, _VP, _VP, _VP, _SZ, STREAM]),
    "mp_implicit_forward_grad": (STATUS, [_VP, _VP, _I, _VP, _VP, _VP, _VP, _SZ, STREAM]),
    "mp_render_forward": (STATUS, [_VP, _VP, _VP, _VP, _I, _VP, _VP, _SZ, STREAM]),
    "mp_mlp_workspace_bytes": (_SZ, [_I]),
    "mp_bg_nets_forward": (STATUS, [_VP, _VP, _VP, _I, _VP, _VP, _VP, _SZ, STREAM]),
    "mp_implicit_backward_workspace_bytes": (_SZ, [_I]),
    "mp_implicit_backward": (STATUS, [_VP, _VP, _I, _VP, _VP, _VP, C.POINTER(LinearGrads), _VP, _VP, _SZ, STREAM]),
    "mp_render_backward_workspace_bytes": (_SZ, [_I]),
    "mp_render_backward": (STATUS, [_VP, _VP, _VP, _VP, _I, _VP, _VP, _VP, _VP, C.POINTER(LinearGrads), _VP, _VP, _VP,
                                    _VP, _SZ, STREAM]),
    "mp_sdf_grid_workspace_bytes": (_SZ, [_I]),
    "mp_sdf_grid": (STATUS, [_VP, c_float_p, _F, _F, _I, _VP, _VP, _SZ, STREAM]),
    "mp_body_bytes": (_SZ, [_I]),
    "mp_body_create": (STATUS, [_VP, _VP, _I, _F, _VP, _SZ, C.POINTER(_VP), STREAM]),
    "mp_body_free": (None, [_VP]),
    "mp_body_set_pose": (STATUS, [_VP, _VP, _VP, STREAM]),
    "mp_deform_inverse": (STATUS, [_VP, _VP, _I, _VP, _VP, _I, STREAM]),
    "mp_deform_forward_jac": (STATUS, [_VP, _VP, _I, _VP, _VP, STREAM]),
    "mp_deform_backward_workspace_bytes": (_SZ, [_I]),
    "mp_deform_inverse_backward": (STATUS, [_VP, _VP, _I, _I, _VP, _VP, _VP, _VP, _VP, _SZ, STREAM]),
    "mp_deform_forward_jac_backward": (STATUS, [_VP, _VP, _I, _VP, _VP, _VP, _VP, _VP, _SZ, STREAM]),
    "mp_deform_broyden": (STATUS, [_VP, _VP, _I, _I, _F, _VP, _VP, _VP, _VP, _VP, STREAM]),
    "mp_body_set_root_finder": (STATUS, [_VP, _I, _F]),
    "mp_laplace_density": (STATUS, [_VP, _I, _F, _VP, STREAM]),
    "mp_camera_rays": (STATUS, [_VP, _VP, _VP, _I, _VP, _VP, STREAM]),
    "mp_sphere_intersections": (STATUS, [_VP, _VP, _I, _F, _VP, _VP, STREAM]),
    "mp_ray_box_hits": (STATUS, [_VP, _VP, _I, C.POINTER(C.c_double), C.POINTER(C.c_double), _VP, _VP, _VP, STREAM]),
    "mp_hit_list_finalize": (STATUS, [_VP, _VP, STREAM]),
    "mp_ray_aabb_hits": (STATUS, [_VP, _VP, _I, _VP, _I, C.c_double, _VP, _VP, _VP, STREAM]),
    "mp_smpl_bytes": (_SZ, [_I]),
    "mp_smpl_create": (STATUS, [_VP, _VP, _VP, _VP, C.POINTER(C.c_int), _VP, _I, _VP, _VP, _SZ, C.POINTER(_VP),
                                STREAM]),
    "mp_smpl_free": (None, [_VP]),
    "mp_smpl_canonical": (STATUS, [_VP, _VP, _VP, STREAM]),
    "mp_smpl_forward": (STATUS, [_VP, _VP, _VP, _VP, _VP, _I, _VP, _VP, STREAM]),
    "mp_smpl_backward_workspace_bytes": (_SZ, [_I]),
    "mp_smpl_backward": (STATUS, [_VP, _VP, _VP, _VP, _VP, _I, _VP, _VP, _VP, _VP, _VP, _VP, _VP, _SZ, STREAM]),
    "mp_sampler_workspace_bytes": (_SZ, [C.POINTER(SamplerCfg), _I]),
    "mp_sample_rays": (STATUS, [C.POINTER(SamplerCfg), _VP, _VP, _VP, _VP, _I, _VP, _VP, _VP, _VP, _SZ, STREAM]),
    "mp_sample_rays_train": (STATUS, [C.POINTER(SamplerCfg), _VP, _VP, _VP, _VP, _I, C.POINTER(SamplerRng), _VP, _VP, _VP,
                                      _VP, _VP, _SZ, STREAM]),
    "mp_sdf_with_deformer_workspace_bytes": (_SZ, [_I]),
    "mp_sdf_with_deformer": (STATUS, [_VP, _VP, _VP, _I, _VP, _VP, _VP, _VP, _SZ, STREAM]),
    "mp_composite_workspace_bytes": (_SZ, [_I, _I]),
    "mp_composite": (STATUS, [C.POINTER(PersonSamples), _I, _I, _I, _F, _VP, _VP, _VP, _VP, _VP, _VP, _SZ, STREAM]),
    "mp_final_compose": (STATUS, [_VP, _VP, _VP, _I, _VP, _VP, STREAM]),
    "mp_composite_backward_workspace_bytes": (_SZ, [_I, _I]),
    "mp_composite_backward": (STATUS, [C.POINTER(PersonSamples), _I, _I, _I, _F, _VP, _VP, _VP, _VP, _VP,
                                       C.POINTER(PersonSampleGrads), _VP, _VP, _SZ, STREAM]),
    "mp_bg_composite_backward": (STATUS, [_VP, _VP, _I, _F, _VP, _VP, _VP, _VP, STREAM]),
    "mp_final_compose_backward": (STATUS, [_VP, _VP, _I, _VP, _VP, _VP, _VP, _VP, STREAM]),
    "mp_background_workspace_bytes": (_SZ, [_I]),
    "mp_background": (STATUS, [_VP, _VP, _VP, _I, _F, _VP, _VP, _SZ, STREAM]),
    "mp_mesh_plan": (STATUS, [_VP, _I, _VP, _I, _F, _VP, C.POINTER(MeshPlan), STREAM]),
    "mp_mesh_create": (STATUS, [C.POINTER(MeshPlan), _VP, _VP, _VP, _SZ, C.POINTER(_VP), STREAM]),
    "mp_mesh_free": (None, [_VP]),
    "mp_mesh_distance": (STATUS, [_VP, _VP, _I, _VP, _VP, _VP, STREAM]),
    "mp_mesh_check_sign": (STATUS, [_VP, _VP, _I, _VP, STREAM]),
    "mp_mesh_surface_flags": (STATUS, [_VP, _VP, _I, _I, _F, _VP, _VP, STREAM]),
    "mp_depth_raster_workspace_bytes": (_SZ, [_I, _I, _I]),
    "mp_depth_raster": (STATUS, [C.POINTER(Camera), _VP, _I, _VP, _I, _I, _I, _VP, _VP, _VP, _SZ, STREAM]),
    "mp_depth_raster_backward_workspace_bytes": (_SZ, [_I, _I, _I]),
    "mp_depth_raster_backward": (STATUS, [C.POINTER(Camera), _VP, _I, _VP, _I, _I, _I, _VP, _VP, _VP, _VP, _SZ, STREAM]),
    "mp_knn1_workspace_bytes": (_SZ, [_I]),
    "mp_knn1": (STATUS, [_VP, _I, _VP, _I, _VP, _VP, _VP, _VP, _SZ, STREAM]),
    "mp_knn1_backward_workspace_bytes": (_SZ, [_I, _I]),
    "mp_knn1_backward": (STATUS, [_VP, _I, _VP, _I, _VP, _VP, _VP, _VP, _VP, _VP, _SZ, STREAM]),
    "mp_mise_workspace_bytes": (_SZ, [_I, _I]),
    "mp_mise": (STATUS, [_VP, c_float_p, _F, _F, _I, _I, C.c_double, _VP, _VP, C.POINTER(C.c_longlong), _VP, _SZ,
                         STREAM]),
    "mp_marching_cubes_workspace_bytes": (_SZ, [_I]),
    "mp_marching_cubes_count": (STATUS, [_VP, _I, C.c_double, C.POINTER(C.c_longlong), C.POINTER(C.c_longlong), _VP,
                                         _SZ, STREAM]),
    "mp_marching_cubes_emit": (STATUS, [_VP, _I, C.c_double, C.POINTER(C.c_double), C.c_double, C.c_double, _VP, _VP,
                                        _VP, _SZ, STREAM]),
    "mp_largest_component_workspace_bytes": (_SZ, [_I, _I]),
    "mp_largest_component": (STATUS, [_VP, _I, _VP, _I, _VP, _VP, c_int_p, c_int_p, _VP, _SZ, STREAM]),
    "mp_render_workspace_bytes": (_SZ, [C.POINTER(Scene), _I]),
    "mp_render_rays": (STATUS, [C.POINTER(Scene), _VP, _VP, _VP, _I, C.POINTER(RenderOut), _VP, _SZ, STREAM]),
}

_lib = None


def lib():
    """Loads the shared library (once).  Fails loudly when it has not been built."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise MpError("libmultiply_b200.so is missing (%s): run `python -m multiply_b200.build` — there is "
                          "no CPU / PyTorch fallback" % LIB_PATH)
        h = C.CDLL(LIB_PATH)
        for name, (res, args) in SIGNATURES.items():
            fn = getattr(h, name)
            fn.restype = _CTYPE.get(res, res)
            fn.argtypes = [_CTYPE.get(a, a) for a in args]
        _lib = h
    return _lib


def check(rc, what=""):
    if rc != 0:
        raise MpError("%s failed (%d): %s" % (what, rc, lib().mp_last_error().decode()))


def ptr(t):
    """Device pointer of a CUDA tensor (or None)."""
    if t is None:
        return None
    if not t.is_cuda:
        raise MpError("expected a CUDA tensor (the library has no CPU path)")
    if not t.is_contiguous():
        raise MpError("expected a contiguous tensor")
    return t.data_ptr()


def stream_ptr():
    return torch.cuda.current_stream().cuda_stream


def call(name, *args):
    """Calls library function ``name``.  A tensor argument becomes its device pointer through ``ptr``; a structure is
    passed by reference where the parameter is a pointer to it; everything else (None, numbers, handles, ctypes arrays,
    ``byref`` objects) is ctypes' to convert.  The trailing stream of a function that takes one may be left out: it is
    the current stream.  A non-zero status raises ``MpError`` with the library's message; a value is returned."""
    res, params = SIGNATURES[name]
    fn = getattr(lib(), name)
    own_stream = len(args) == len(params) - 1 and params[-1] is STREAM
    if len(args) + own_stream != len(params):
        raise MpError("%s takes %d arguments, got %d" % (name, len(params), len(args)))
    conv = []
    for i, (a, p) in enumerate(zip(args, params)):
        if isinstance(a, torch.Tensor):
            try:
                a = ptr(a)
            except MpError as e:
                raise MpError("%s, argument %d: %s" % (name, i, e)) from None
        elif isinstance(a, C.Structure) and p is C.POINTER(type(a)):
            a = C.byref(a)
        conv.append(a)
    if own_stream:
        conv.append(stream_ptr())
    out = fn(*conv)
    if res is not STATUS:
        return out
    check(out, name)


def dev(t, device, dtype=torch.float32):
    """``t`` (or None) detached, on ``device``, of ``dtype`` and contiguous: the form every tensor the library reads has."""
    return None if t is None else t.detach().to(device=device, dtype=dtype).contiguous()


def workspace(nbytes, device):
    """Uninitialised device bytes for a ``*_bytes`` query's answer; never empty, so its pointer is always valid."""
    return torch.empty(max(int(nbytes), 1), dtype=torch.uint8, device=device)


def vec3(ctype, v):
    """A host [3] array of ``ctype`` (a centre, half extents)."""
    return (ctype * 3)(*[float(x) for x in v])


class Handle(C.c_void_p):
    """An object the library built in caller storage (the ``out`` of mp_field_pack / mp_*_create); passes wherever a
    ``void*`` does.  Dropping it calls the ``mp_*_free`` named at construction."""

    def __init__(self, free):
        super().__init__()
        self.free = free

    def __del__(self):
        try:
            if self.value:
                call(self.free, self)
        except Exception:       # interpreter shutdown: the library or this module may already be gone
            pass
