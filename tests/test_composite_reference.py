"""CPU: the compositing restatement of tests/test_gpu_composite.py, run in float32, against oracle/port.py's
composite_nerfacc (the restatement the golden renders were checked with), so that the fp64 reference the GPU tests use
states the same operation."""
import importlib.util
import os

import numpy as np
import pytest
import torch

from oracle import port

_spec = importlib.util.spec_from_file_location(
    "_composite_gpu_tests", os.path.join(os.path.dirname(os.path.abspath(__file__)), "test_gpu_composite.py"))
G = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(G)


@pytest.mark.parametrize("P,n,R,beta_param,ties", [(1, 1, 3, 0.1, True), (2, 33, 9, 0.1, True), (3, 16, 7, 0.05, True),
                                                   (4, 31, 12, 0.0, False), (8, 5, 6, 0.1, True)])
def test_reference_matches_port(P, n, R, beta_param, ties):
    persons = G.make_inputs(P * 100 + n, P, R, n, substitute=True, ties=ties)
    beta = np.float32(port.get_beta(beta_param).item())
    got = G.composite_ref(persons, R, n, beta, dtype=np.float32)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a))
    want = port.composite_nerfacc([t(d["idx"]) for d in persons], [t(d["z"][:, :-1]) for d in persons],
                                  [t(d["z"][:, -1]) for d in persons], [t(d["sdf"]) for d in persons],
                                  [t(d["rgb"]) for d in persons], [t(d["nrm"]) for d in persons], list(range(P)), R,
                                  beta_param)
    for name, a, b in zip(G.NAMES, got, want):
        assert a.dtype == np.float32
        assert float(np.abs(a - b.numpy().reshape(a.shape)).max()) < 1e-6, name
    # and the fp64 statement agrees with both to float32 rounding
    ref64 = G.composite_ref(persons, R, n, beta)
    for name, a, b in zip(G.NAMES, got, ref64):
        assert float(np.abs(a - b).max()) < 1e-5, name
