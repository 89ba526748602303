"""CPU: the one call path of the binding (``_lib.call``) — what it refuses before the library is entered, how it names
a failure, and that its table states the header's conventions.  Nothing here reaches a kernel."""
import ctypes as C
import os
import re

import pytest
import torch

from multiply_b200 import _lib as L, scene as S

from _setups import field_descs, refused_fields

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
# the int-returning functions whose int is an answer, not a status
INT_VALUES = {"mp_version", "mp_get_engine", "mp_get_precision", "mp_device_sm_count"}


def test_host_tensor_is_refused_before_the_library_is_entered(monkeypatch):
    entered = []
    monkeypatch.setattr(L.lib(), "mp_laplace_density", lambda *a: entered.append(a) or 0)
    ok = torch.zeros(8)
    with pytest.raises(L.MpError, match=r"mp_laplace_density, argument 0: expected a CUDA tensor"):
        L.call("mp_laplace_density", ok, 8, 0.1, None)
    with pytest.raises(L.MpError, match=r"mp_laplace_density, argument 3: expected a CUDA tensor"):
        L.call("mp_laplace_density", None, 8, 0.1, ok, None)
    with pytest.raises(L.MpError, match=r"mp_laplace_density takes 5 arguments, got 2"):
        L.call("mp_laplace_density", None, 8)
    assert entered == []


def test_status_raises_with_the_tables_name_and_value_returns():
    with pytest.raises(L.MpError) as e:
        L.call("mp_set_engine", 7)
    assert "mp_set_engine failed (" in str(e.value) and "engine must be 0" in str(e.value)
    assert L.call("mp_set_engine", 1) is None
    assert L.call("mp_get_engine") == 1                       # 1 is an answer here, not a failure
    assert L.call("mp_version") == L.lib().mp_version()
    assert L.call("mp_mlp_workspace_bytes", 1024) == L.lib().mp_mlp_workspace_bytes(1024) > 0
    c = L.SamplerCfg(3.0, 0.0, 64, 128, 32, 0.1, 10, 5, 1e-6, 0.1, 1e-4)      # a structure goes by reference
    assert L.call("mp_sampler_workspace_bytes", c, 512) == L.lib().mp_sampler_workspace_bytes(C.byref(c), 512)


def test_table_states_the_headers_status_and_stream_conventions():
    hdr = open(os.path.join(ROOT, "include", "multiply_b200.h")).read()
    hdr = re.sub(r"/\*.*?\*/", "", hdr, flags=re.S)
    decl = {m.group(2): (m.group(1).strip(), m.group(3))
            for m in re.finditer(r"([\w ]+?[\s*]+)(mp_[a-z0-9_]+)\s*\(([^;{}]*?)\)\s*;", hdr)}
    assert set(decl) == set(L.SIGNATURES)
    for name, (res, params) in L.SIGNATURES.items():
        ret, plist = decl[name]
        assert (res is L.STATUS) == (ret == "int" and name not in INT_VALUES), name
        assert res is not L.STREAM and L.STREAM not in params[:-1], name
        takes_stream = re.search(r"void\s*\*\s*stream\s*$", plist) is not None
        assert (bool(params) and params[-1] is L.STREAM) == takes_stream, name
        assert len(params) == (0 if plist.strip() == "void" else plist.count(",") + 1), name
    for name in ("mp_last_error", "mp_launch_count", "mp_field_pack_bytes", "mp_render_workspace_bytes") + tuple(INT_VALUES):
        assert L.SIGNATURES[name][0] not in (L.STATUS, None), name


def test_size_queries_are_host_calls():
    """Every workspace and storage query answers on the host: no launch, no device needed (on a machine without a GPU
    the SM count is taken as 132), and a query of a larger problem never asks for less.  mp_field_pack_bytes reads only
    the descriptors' dimensions (every weight pointer here is NULL): the background pair's storage is the smaller, and a
    pair the pack refuses is answered 0."""
    n0 = L.call("mp_launch_count", 0)
    c = L.SamplerCfg(3.0, 0.0, 64, 128, 32, 0.1, 10, 5, 1e-6, 0.1, 1e-4)
    sc = S.make_scene(P=1, S=16, seed=42)
    p = sc["persons"][0]
    fg = field_descs(p["implicit"], p["render"], False)[:2] + (0,)
    bg = field_descs(sc["bg_implicit"], sc["bg_render"], True)[:2] + (1,)
    for name, small, large in (("mp_mlp_workspace_bytes", (1,), (32769,)),
                               ("mp_sdf_with_deformer_workspace_bytes", (1,), (129,)),
                               ("mp_sdf_grid_workspace_bytes", (8,), (101,)),
                               ("mp_background_workspace_bytes", (1,), (301,)),
                               ("mp_sampler_workspace_bytes", (c, 1), (c, 129)),
                               ("mp_composite_workspace_bytes", (1, 1), (300, 3)),
                               ("mp_composite_backward_workspace_bytes", (1, 1), (300, 3)),
                               ("mp_deform_backward_workspace_bytes", (1,), (4097,)),
                               ("mp_smpl_backward_workspace_bytes", (300,), (6890,)),
                               ("mp_body_bytes", (3,), (6890,)),
                               ("mp_smpl_bytes", (300,), (6890,)),
                               ("mp_mise_workspace_bytes", (4, 1), (16, 2)),
                               ("mp_marching_cubes_workspace_bytes", (8,), (64,)),
                               ("mp_largest_component_workspace_bytes", (3, 1), (1000, 2000)),
                               ("mp_field_pack_bytes", bg, fg)):
        assert 0 < L.call(name, *small) <= L.call(name, *large), name
    for what, (isd, rsd, background, imp), _ in refused_fields(sc):
        assert L.call("mp_field_pack_bytes", *field_descs(isd, rsd, background, **imp)[:2], int(background)) == 0, what
    assert L.call("mp_launch_count", 0) == n0
