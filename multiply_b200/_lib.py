"""ctypes binding of libmultiply_b200.so (the C ABI declared in include/multiply_b200.h).

There is no fallback: if the shared library is missing the import of anything that needs it
raises, and every entry point raises ``MpError`` with the library's error text on failure.
"""
import ctypes as C
import os

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("MP_LIB") or os.path.join(HERE, "libmultiply_b200.so")     # MP_LIB: A/B builds (scripts/)

MP_MAX_LAYERS = 12
MP_MAX_PERSONS = 8

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


# name -> (restype, argtypes) ; mirrors include/multiply_b200.h one to one
_VP, _I, _F, _SZ = C.c_void_p, C.c_int, C.c_float, C.c_size_t
SIGNATURES = {
    "mp_version": (_I, []),
    "mp_last_error": (C.c_char_p, []),
    "mp_device_sm_count": (_I, []),
    "mp_linspace_host": (_I, [_F, _F, _I, c_float_p]),
    "mp_launch_count": (C.c_longlong, [_I]),
    "mp_field_pack_bytes": (_SZ, []),
    "mp_field_pack": (_I, [C.POINTER(ImplicitDesc), C.POINTER(RenderDesc), _I, _VP, _SZ, C.POINTER(_VP), _VP]),
    "mp_field_free": (None, [_VP]),
    "mp_field_set_cond": (_I, [_VP, _VP, _VP]),
    "mp_set_engine": (_I, [_I]),
    "mp_get_engine": (_I, []),
    "mp_set_precision": (_I, [_I]),
    "mp_get_precision": (_I, []),
    "mp_profile_enable": (_I, [_I]),
    "mp_set_streams": (_I, [_I]),
    "mp_profile_read": (_I, [C.POINTER(C.c_double), C.POINTER(C.c_longlong), C.POINTER(C.c_double), _I]),
    "mp_implicit_forward": (_I, [_VP, _VP, _I, _VP, _VP, _VP, _SZ, _VP]),
    "mp_implicit_forward_grad": (_I, [_VP, _VP, _I, _VP, _VP, _VP, _VP, _SZ, _VP]),
    "mp_render_forward": (_I, [_VP, _VP, _VP, _VP, _I, _VP, _VP, _SZ, _VP]),
    "mp_mlp_workspace_bytes": (_SZ, [_I]),
    "mp_bg_nets_forward": (_I, [_VP, _VP, _VP, _I, _VP, _VP, _VP, _SZ, _VP]),
    "mp_sdf_grid_workspace_bytes": (_SZ, [_I]),
    "mp_sdf_grid": (_I, [_VP, c_float_p, _F, _F, _I, _VP, _VP, _SZ, _VP]),
    "mp_body_bytes": (_SZ, [_I]),
    "mp_body_create": (_I, [_VP, _VP, _I, _F, _VP, _SZ, C.POINTER(_VP), _VP]),
    "mp_body_free": (None, [_VP]),
    "mp_body_set_pose": (_I, [_VP, _VP, _VP, _VP]),
    "mp_deform_inverse": (_I, [_VP, _VP, _I, _VP, _VP, _I, _VP]),
    "mp_deform_forward_jac": (_I, [_VP, _VP, _I, _VP, _VP, _VP]),
    "mp_deform_broyden": (_I, [_VP, _VP, _I, _I, _F, _VP, _VP, _VP, _VP, _VP, _VP]),
    "mp_body_set_root_finder": (_I, [_VP, _I, _F]),
    "mp_laplace_density": (_I, [_VP, _I, _F, _VP, _VP]),
    "mp_camera_rays": (_I, [_VP, _VP, _VP, _I, _VP, _VP, _VP]),
    "mp_sphere_intersections": (_I, [_VP, _VP, _I, _F, _VP, _VP, _VP]),
    "mp_ray_box_hits": (_I, [_VP, _VP, _I, C.POINTER(C.c_double), C.POINTER(C.c_double), _VP, _VP, _VP, _VP]),
    "mp_hit_list_finalize": (_I, [_VP, _VP, _VP]),
    "mp_ray_aabb_hits": (_I, [_VP, _VP, _I, _VP, _I, C.c_double, _VP, _VP, _VP, _VP]),
    "mp_smpl_bytes": (_SZ, [_I]),
    "mp_smpl_create": (_I, [_VP, _VP, _VP, _VP, C.POINTER(C.c_int), _VP, _I, _VP, _VP, _SZ, C.POINTER(_VP), _VP]),
    "mp_smpl_free": (None, [_VP]),
    "mp_smpl_canonical": (_I, [_VP, _VP, _VP, _VP]),
    "mp_smpl_forward": (_I, [_VP, _VP, _VP, _VP, _VP, _I, _VP, _VP, _VP]),
    "mp_sampler_workspace_bytes": (_SZ, [C.POINTER(SamplerCfg), _I]),
    "mp_sample_rays": (_I, [C.POINTER(SamplerCfg), _VP, _VP, _VP, _VP, _I, _VP, _VP, _VP, _VP, _SZ, _VP]),
    "mp_sample_rays_train": (_I, [C.POINTER(SamplerCfg), _VP, _VP, _VP, _VP, _I, C.POINTER(SamplerRng), _VP, _VP, _VP, _VP,
                                  _VP, _SZ, _VP]),
    "mp_sdf_with_deformer": (_I, [_VP, _VP, _VP, _I, _VP, _VP, _VP, _VP, _SZ, _VP]),
    "mp_composite_workspace_bytes": (_SZ, [_I, _I]),
    "mp_composite": (_I, [C.POINTER(PersonSamples), _I, _I, _I, _F, _VP, _VP, _VP, _VP, _VP, _VP, _SZ, _VP]),
    "mp_final_compose": (_I, [_VP, _VP, _VP, _I, _VP, _VP, _VP]),
    "mp_composite_backward_workspace_bytes": (_SZ, [_I, _I]),
    "mp_composite_backward": (_I, [C.POINTER(PersonSamples), _I, _I, _I, _F, _VP, _VP, _VP, _VP, _VP,
                                   C.POINTER(PersonSampleGrads), _VP, _VP, _SZ, _VP]),
    "mp_bg_composite_backward": (_I, [_VP, _VP, _I, _F, _VP, _VP, _VP, _VP, _VP]),
    "mp_final_compose_backward": (_I, [_VP, _VP, _I, _VP, _VP, _VP, _VP, _VP, _VP]),
    "mp_background_workspace_bytes": (_SZ, [_I]),
    "mp_background": (_I, [_VP, _VP, _VP, _I, _F, _VP, _VP, _SZ, _VP]),
    "mp_mesh_plan": (_I, [_VP, _I, _VP, _I, _F, _VP, C.POINTER(MeshPlan), _VP]),
    "mp_mesh_create": (_I, [C.POINTER(MeshPlan), _VP, _VP, _VP, _SZ, C.POINTER(_VP), _VP]),
    "mp_mesh_free": (None, [_VP]),
    "mp_mesh_distance": (_I, [_VP, _VP, _I, _VP, _VP, _VP, _VP]),
    "mp_mesh_check_sign": (_I, [_VP, _VP, _I, _VP, _VP]),
    "mp_mesh_surface_flags": (_I, [_VP, _VP, _I, _I, _F, _VP, _VP, _VP]),
    "mp_mise_workspace_bytes": (_SZ, [_I, _I]),
    "mp_mise": (_I, [_VP, c_float_p, _F, _F, _I, _I, C.c_double, _VP, _VP, C.POINTER(C.c_longlong), _VP, _SZ, _VP]),
    "mp_marching_cubes_workspace_bytes": (_SZ, [_I]),
    "mp_marching_cubes_count": (_I, [_VP, _I, C.c_double, C.POINTER(C.c_longlong), C.POINTER(C.c_longlong), _VP, _SZ,
                                     _VP]),
    "mp_marching_cubes_emit": (_I, [_VP, _I, C.c_double, C.POINTER(C.c_double), C.c_double, C.c_double, _VP, _VP, _VP,
                                    _SZ, _VP]),
    "mp_largest_component_workspace_bytes": (_SZ, [_I, _I]),
    "mp_largest_component": (_I, [_VP, _I, _VP, _I, _VP, _VP, c_int_p, c_int_p, _VP, _SZ, _VP]),
    "mp_render_workspace_bytes": (_SZ, [C.POINTER(Scene), _I]),
    "mp_render_rays": (_I, [C.POINTER(Scene), _VP, _VP, _VP, _I, C.POINTER(RenderOut), _VP, _SZ, _VP]),
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
            fn.restype = res
            fn.argtypes = args
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
    import torch
    return torch.cuda.current_stream().cuda_stream
