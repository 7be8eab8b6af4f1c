"""The launch plan of the benchmarked batch (512 pairs of 640x480, 5 levels) on an H100 (132 SMs x 2 CTAs): level 0 runs in
three slices of the pair index with squads of 2, 4 and 8 CTAs (pairs 0-333, 334-452, 453-511).  Results do not depend on
the plan: both sides of every slice boundary equal single alignments, and the batch under the previous default squad size
(g = 3: slices of 3, 6 and 12 CTAs) returns the same bits."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

B = 512


def _same(a, b):
    return (np.array_equal(a.transformation, b.transformation) and np.array_equal(a.information, b.information)
            and a.log_likelihood == b.log_likelihood and a.levels == b.levels)


def test_batch_512_plan_does_not_change_results(engine, monkeypatch):
    import torch
    from dvo_slam_b200 import synth
    from dvo_slam_b200.engine import Config

    dev = torch.device("cuda", 0)
    scfg = synth.SceneConfig()
    H, W = scfg.height, scfg.width
    I = np.empty((2 * B, H, W), np.float32)
    Z = np.empty((2 * B, H, W), np.float32)
    for i in range(B):                      # the bench's seeds
        p = synth.make_pair(i, scfg, device=dev)
        I[i] = p["I_ref"].cpu().numpy(); Z[i] = p["Z_ref"].cpu().numpy()
        I[B + i] = p["I_cur"].cpu().numpy(); Z[B + i] = p["Z_cur"].cpu().numpy()
    pyrs = engine.pyramid_batch(I, Z, synth.FR1_INTRINSICS, 5)
    refs, curs = pyrs[:B], pyrs[B:]
    cfg = Config(first_level=4, last_level=0, max_iterations_per_level=50, precision=1e-4)
    res = engine.match_batch(refs, curs, cfg)
    for i in (0, 333, 334, 452, 453, 511):
        assert _same(res[i], engine.match(refs[i], curs[i], cfg)), i
    monkeypatch.setenv("DVO_B200_FINE_G", "3")
    old = engine.match_batch(refs, curs, cfg)
    assert all(_same(res[i], old[i]) for i in range(B))
