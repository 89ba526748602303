"""CPU: the float64 autograd of oracle/port.py's SMPL and deformer restatements (lbs, smpl_server_forward, skinning,
forward_skinning) against tests/golden/body_grad.npz, the float64 autograd of the reference's own lbs, SMPLServer lines,
deformer.skinning and Multiply.forward_gradient's Jacobian (oracle/gen_golden_body_grad.py).  The GPU tests
(test_gpu_body_grad.py) use the port as their reference at any size."""
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from oracle import gen_golden_body_grad as G      # noqa: E402
from _body_grad_port import port_smpl_grads, port_inverse_grads, port_forward_grads   # noqa: E402

GOLD = os.path.join(ROOT, "tests", "golden", "body_grad.npz")


@pytest.fixture(scope="module")
def gold():
    return dict(np.load(GOLD))


@pytest.fixture(scope="module")
def model():
    return G.model64()


def _close(a, b, what):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    scale = max(np.abs(b).max(), 1e-300)
    err = np.abs(a - b).max() / scale
    assert err < 1e-10, (what, err)


@pytest.mark.parametrize("name", list(G.SMPL_CASES))
def test_port_smpl_grads_match_reference(gold, model, name):
    k = list(G.SMPL_CASES).index(name)
    V = model["v_template"].shape[0]
    u_v, u_t = G.cotangents(100 + k, (V, 3), (24, 4, 4))
    g = lambda key: gold[f"smpl_{name}_{key}"]
    got = port_smpl_grads(model, gold["smpl_tfs_c_inv"], g("scale"), g("transl"), g("theta"), g("betas"),
                          int(g("absolute")), bool(g("v_template")), u_v, u_t)
    _close(got["tfs"], g("tfs"), name + "/tfs")
    for key in ("scale", "transl", "thetas", "betas"):
        _close(got[key], g("grad_" + key), name + "/" + key)
    if bool(g("v_template")):
        assert not np.any(got["betas"]) and not np.any(g("grad_betas"))


def test_port_inverse_deformer_grads_match_reference(gold, model):
    N = gold["inv_x"].shape[0]
    u_xc, = G.cotangents(200, (N, 3))
    got = port_inverse_grads(gold["inv_x"], gold["inv_verts_p"], model["lbs_weights"].numpy(), gold["inv_tfs"], u_xc)
    _close(got["x_c"], gold["inv_x_c"], "x_c")
    _close(got["x"], gold["inv_grad_x"], "d_x")
    _close(got["tfs"], gold["inv_grad_tfs"], "d_tfs")


def test_port_forward_skinning_grads_match_reference(gold, model):
    N = gold["fwd_x_c"].shape[0]
    u_xd, u_J = G.cotangents(201, (N, 3), (N, 3, 3))
    got = port_forward_grads(gold["fwd_x_c"], gold["fwd_verts_c"], model["lbs_weights"].numpy(), gold["inv_tfs"], u_xd,
                             u_J)
    _close(got["x_d"], gold["fwd_x_d"], "x_d")
    _close(got["Jinv"], gold["fwd_Jinv"], "Jinv")
    _close(got["x_c"], gold["fwd_grad_x_c"], "d_x_c")
    _close(got["tfs"], gold["fwd_grad_tfs"], "d_tfs")
