"""Person-sharded rendering (multiply_b200/parallel.py: PersonShardedRenderer) against the fused single-GPU forward.
In one process (world 1) the per-person pass, mp_composite, mp_background and mp_final_compose are driven separately
through the C ABI; the frame must equal mp_render_rays bit for bit.  The 2-rank exchange is covered on CPU
(tests/test_parallel_gloo.py) and on two GPUs by scripts/person_shard_check.py."""
import pytest
import torch

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("P,empty,beta_min", [pytest.param(2, None, None, id="2-None"),
                                               pytest.param(3, 1, None, id="3-1"),
                                               pytest.param(2, None, 1e-3, id="2-None-beta_min1e-3")])
def test_person_sharded_equals_fused_forward(P, empty, beta_min):
    from multiply_b200 import engine, parallel, scene as S
    engine.set_engine("tc")
    sc = S.make_scene(P=P, S=64, seed=11)
    if beta_min is not None:                                  # a density.beta_min other than LaplaceDensity's default
        sc["beta_min"] = beta_min
    inp = S.make_rays(sc, 257, seed=2, region="boxes")
    hits = S.make_hit_lists(sc, inp)
    if empty is not None:
        hits[empty] = torch.zeros(0, dtype=torch.int64)       # multiply.py:262-263: ray 0 stands in
    ref = engine.Renderer(sc).render(inp, hits)
    out = parallel.PersonShardedRenderer(sc).render(inp, hits)
    torch.cuda.synchronize()
    for k in parallel.PIXEL_KEYS:
        assert torch.equal(out[k], ref[k]), k
