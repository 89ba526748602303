"""CPU: host-side logic of the C ABI that needs no GPU — the library loads, exports every
symbol include/multiply_b200.h declares, and its torch-exact linspace matches torch."""
import ctypes as C
import os
import re
import numpy as np
import torch

from multiply_b200 import _lib as L, scene as S

from _setups import field_descs

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_library_exports_every_declared_symbol():
    hdr = open(os.path.join(ROOT, "include", "multiply_b200.h")).read()
    declared = set(re.findall(r"\b(mp_[a-z0-9_]+)\s*\(", hdr))
    lib = L.lib()
    missing = [n for n in sorted(declared) if not hasattr(lib, n)]
    assert not missing, missing
    assert declared == set(L.SIGNATURES), (declared ^ set(L.SIGNATURES))
    assert lib.mp_version() >= 100


def test_linspace_matches_torch():
    lib = L.lib()
    for (a, b, n) in [(0, 1, 128), (0, 1, 64), (0, 1, 256), (0, 1, 512), (0, 1, 32), (0, 1, 16),
                      (0, 127, 32), (0, 255, 32), (0, 639, 32), (0, 1279, 64), (0, 2559, 128), (0, 31, 8),
                      (0, 159, 8), (0, 383, 64)]:
        buf = (C.c_float * n)()
        assert lib.mp_linspace_host(a, b, n, buf) == 0
        assert np.array_equal(np.array(buf, dtype=np.float32), torch.linspace(float(a), float(b), n).numpy()), (a, b, n)


def test_errors_are_reported_not_thrown():
    lib = L.lib()
    assert lib.mp_linspace_host(0.0, 1.0, 0, None) != 0
    assert b"mp_linspace_host" in lib.mp_last_error()
    assert lib.mp_set_engine(7) != 0
    assert lib.mp_set_engine(1) == 0 and lib.mp_get_engine() == 1


def test_workspace_and_storage_queries_are_pure_host():
    """The queries answer from shapes alone; mp_field_pack_bytes from the two network descriptors, whose weight pointers
    are NULL here."""
    lib = L.lib()
    c = L.SamplerCfg(3.0, 0.0, 64, 128, 32, 0.1, 10, 5, 1e-6, 0.1, 1e-4)
    a = lib.mp_sampler_workspace_bytes(C.byref(c), 512)
    b = lib.mp_sampler_workspace_bytes(C.byref(c), 1024)
    assert 0 < a < b
    assert lib.mp_body_bytes(6890) > 6890 * 16 * 2
    sc = S.make_scene(P=1, S=16, seed=42)
    p = sc["persons"][0]
    fg_imp, fg_ren, _ = field_descs(p["implicit"], p["render"], False)
    bg_imp, bg_ren, _ = field_descs(sc["bg_implicit"], sc["bg_render"], True)
    fg = lib.mp_field_pack_bytes(C.byref(fg_imp), C.byref(fg_ren), 0)
    bg = lib.mp_field_pack_bytes(C.byref(bg_imp), C.byref(bg_ren), 1)
    assert fg > bg > 0


def test_product_path_has_no_oracle_import():
    """The product package must never import the oracle (no CPU fallback)."""
    pkg = os.path.join(ROOT, "multiply_b200")
    for dp, _, fs in os.walk(pkg):
        for f in fs:
            if f.endswith(".py"):
                src = open(os.path.join(dp, f)).read()
                assert not re.search(r"^\s*(from|import)\s+oracle", src, re.M), f
                assert "import_module(\"oracle" not in src and "__import__(\"oracle" not in src, f


def test_quaternion_pose_form():
    """rend_util.get_camera_params accepts pose as [B,7] = quaternion (w,x,y,z) | centre (rend_util.py:46-50, quat_to_rot
    :88-105): the mirror expands it to the same matrix scipy's Rotation gives, and the host ray builder agrees with the
    matrix form."""
    import numpy as np
    import torch
    from scipy.spatial.transform import Rotation
    from multiply_b200.model import rend_util
    rng = np.random.default_rng(0)
    q = rng.standard_normal((5, 4))
    c = rng.standard_normal((5, 3))
    pose7 = torch.tensor(np.concatenate([q * 3.0, c], 1), dtype=torch.float32)        # un-normalised on purpose
    M = rend_util.pose_matrix(pose7)
    qn = q / np.linalg.norm(q, axis=1, keepdims=True)
    R = Rotation.from_quat(qn[:, [1, 2, 3, 0]]).as_matrix()                            # scipy wants x,y,z,w
    assert np.allclose(M[:, :3, :3].numpy(), R, atol=1e-6)
    assert np.allclose(M[:, :3, 3].numpy(), c, atol=1e-7)
    assert np.allclose(M[:, 3].numpy(), np.tile([0, 0, 0, 1.0], (5, 1)))
    m44 = torch.eye(4)[None]
    assert rend_util.pose_matrix(m44) is m44
    K = torch.eye(4)[None].clone()
    K[0, 0, 0] = K[0, 1, 1] = 500.0
    K[0, 0, 2] = K[0, 1, 2] = 128.0
    uv = torch.tensor(rng.random((1, 7, 2)) * 256, dtype=torch.float32)
    d7, c7 = rend_util.get_camera_params_host(uv, pose7[:1], K)
    d4, c4 = rend_util.get_camera_params_host(uv, M[:1], K)
    assert torch.equal(d7, d4) and torch.equal(c7, c4)
