"""The metric's second half: pose AUC@5/10/20 of the engine EQUALS the CPU oracle's on the same synthetic units
(same weights, same inputs) -- eval_multi_view.py:53-87 / eval_pairs.py:262-277.  32 units with the full layer stack at
a reduced keypoint count (the oracle restates the reference's dense (6+3n)^2 two-view BA, minutes per pair at 1024);
a score-driven confidence head (synthetic.py) keeps the AUC away from 0."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize('config', ['cfg3', 'cfg2'])
def test_pose_auc_engine_equals_oracle(config):
    import bench
    from e2e_multi_view_matching_b200.models.multi_view_matcher import MultiViewMatcher
    cfg = bench.CONFIGS[config]
    sd = bench.make_weights(cfg)
    model = MultiViewMatcher({'GNN_layers': cfg['layers'], 'multi_frame_matching': cfg['kind'] == 'tuple'}).eval()
    model.load_state_dict({k: torch.from_numpy(np.asarray(v)) for k, v in sd.items()})
    model = model.cuda()
    torch.set_num_threads(bench.cpu_threads())
    r = bench.pose_auc_parity(cfg, model, sd, torch.device('cuda'), n_units=32)
    print(config, r)
    assert r['oracle'][2] > 30.0, 'the synthetic setup should give a meaningful AUC'
    # Two-view path: equal to 0.1 pt (measured 3e-4 pt).  Multi-view path: the global LM bundle adjustment of a tuple whose
    # problem is poorly conditioned (free scale gauge) stops after a different number of iterations in the two
    # implementations (same cost to 0.5 %, poses up to ~2 deg apart on 5 of 32 tuples; tools/auc_diag.py)
    # -- unpinned against Ceres' exact iterates on both sides (DESIGN.md §5): 0.5 pt, and the
    # median pair must agree to 0.01 deg.
    assert r['max_abs_diff_pt'] <= (0.1 if config == 'cfg2' else 0.5), r
    assert r['median_abs_pose_error_diff_deg'] < 1e-2, r
