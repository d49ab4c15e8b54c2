"""CPU: the float64 oracles the two-view pose sweep (tests/test_two_view_pose_shapes_gpu.py) compares against.

- oracle.pose.run_bundle_adjust_2_view_schur (3x3 point blocks eliminated) against the dense (6+3n)^2 oracle,
  run_bundle_adjust_2_view, at n <= 150: the same trace and the same best pose, with and without Jacobi scaling,
  and the same exclusion of items with <= 6 valid matches.
- oracle.ba_init.ba_initialize_edges: the edge rule and the disconnected-graph fallback.
- The scene generators: rotations past 120 deg, pure forward motion, near-collinear centres, a corrupted edge."""
import numpy as np
import pytest


def _w8pt_items(seeds, n, **kw):
    from oracle import pose as P
    out = []
    for s in seeds:
        sc = P.make_two_view_scene(s, n, outlier_frac=0.2, **kw)
        f = {k: v.astype(np.float64) for k, v in sc.items() if k != 'outlier'}
        T, info = P.estimate_relative_pose_w8pt(f['kpts0'], f['kpts1'], f['intr'], f['intr'], f['conf'],
                                                determine_inliers=True)
        cn = info['confidence'].copy()
        cn[~info['pos_depth_mask']] = 0
        out.append((info['kpts0_norm'], info['kpts1_norm'], cn, T))
    return [np.concatenate(x, 0) for x in zip(*out)]


@pytest.mark.parametrize('jacobi', [True, False], ids=['jacobi', 'no_jacobi'])
@pytest.mark.parametrize('n,kw', [(12, {}), (40, {}), (150, {}), (60, {'motion': 'forward', 'rot_deg': (0, 0)}),
                                  (60, {'motion': 'orbit', 'rot_deg': (130, 179)})],
                         ids=['n12', 'n40', 'n150', 'forward', 'orbit'])
def test_schur_equals_dense(n, kw, jacobi):
    from oracle import pose as P
    k0, k1, cn, T = _w8pt_items((3, 4), n, **kw)
    cn[1, :7] = np.where(cn[1, :7] > 0, cn[1, :7], 0.05)
    cn[1, 7:] = 0                                    # second item: exactly 7 valid matches
    if n > 12:
        cn[0, ::5] = 0
    worst = [0.0, 0.0]
    for it in (0, 1, 10):
        ed, vd, trd = P.run_bundle_adjust_2_view(k0, k1, cn, T, it, return_trace=True, jacobi_precond=jacobi)
        es, vs, trs = P.run_bundle_adjust_2_view_schur(k0, k1, cn, T, it, jacobi_precond=jacobi)
        assert vd.tolist() == vs.tolist() == [True, True]
        for b in range(2):
            trs_b = trs[b]
            assert trs_b.shape == (it + 1,)
            worst[0] = max(worst[0], float((np.abs(trs_b - trd[b]) / np.maximum(trs_b, trs_b[0])).max()))
            worst[1] = max(worst[1], float(np.abs(es[b] - ed[b]).max()))
    print('trace err / max(trace, trace[0]) %.1e, pose err %.1e' % tuple(worst))
    # Two solvers of the same steps, both in float64: they differ by the rounding of the two linear solves, which
    # the 7-match item (a nearly singular problem whose residual grows once lambda is small) amplifies to ~1e-9
    assert worst[0] <= 1e-8 and worst[1] <= 1e-8, worst
    # 6 valid matches: excluded, T_init comes back
    cn[0, 6:] = 0
    es, vs, trs = P.run_bundle_adjust_2_view_schur(k0, k1, cn, T, 10, jacobi_precond=jacobi)
    assert vs.tolist() == [False, True] and trs[0] is None
    np.testing.assert_array_equal(es[0], T[0])


def test_ba_initialize_edge_rule_and_fallback():
    from oracle import ba_init as BI
    extr, rel = BI.make_pose_graph(3, 4)
    pairs = [(a, b) for b in range(4) for a in range(b)]
    Trel = np.array([rel[p] for p in pairs])
    tree = extr.copy()
    tree[1:, :3, 3] += 0.01
    n_pad = 64
    inl = np.zeros((len(pairs), n_pad), np.uint8)
    inl[:, :20] = 1
    succ = np.ones(len(pairs), np.uint8)
    on = np.zeros(len(pairs), np.uint8)
    out, ne = BI.ba_initialize_edges(4, pairs, tree, Trel, succ, on, inl)
    assert ne == 6
    np.testing.assert_allclose(out, extr, atol=1e-6)          # exact relative poses: the ground truth back
    inl[:, 19] = 0                                            # 19 inliers everywhere: only tree edges remain
    on[[0, 1, 3]] = 1                                         # (0,1) (0,2) (0,3)
    succ[1] = 0                                               # a failed pair is never an edge, on the tree or not
    out, ne = BI.ba_initialize_edges(4, pairs, tree, Trel, succ, on, inl)
    assert ne == 2
    assert (out == tree).all()                                # view 2 unreachable: the tree poses unchanged
    inl[1, 40:61] = 1                                         # 21 inliers counted over n_pad, but pair failed
    inl[4, 40:61] = 1                                         # (1,3): 21 inliers, off the tree
    out, ne = BI.ba_initialize_edges(4, pairs, tree, Trel, succ, on, inl)
    assert ne == 3 and (out == tree).all()
    inl[2, 40:60] = 1                                         # (1,2): exactly 20 = min_inliers connects view 2
    out, ne = BI.ba_initialize_edges(4, pairs, tree, Trel, succ, on, inl)
    assert ne == 4
    np.testing.assert_allclose(out, extr, atol=1e-6)


def test_scene_generators():
    from oracle import pose as P
    from oracle import ba_init as BI
    for s in range(4):
        sc = P.make_two_view_scene(s, 50, motion='orbit', rot_deg=(130, 179), outlier_frac=0.0)
        R = sc['T_021'][0, :3, :3].astype(np.float64)
        assert np.trace(R) < -0.28                            # > 130 deg
        sc = P.make_two_view_scene(s, 50, motion='forward', rot_deg=(0, 0))
        T = sc['T_021'][0].astype(np.float64)
        assert (T[:3, :3] == np.eye(3)).all() and T[0, 3] == 0 and T[1, 3] == 0 and T[2, 3] < 0
    extr, rel = BI.make_pose_graph(1, 5, rot_deg=(130, 179))
    for (a, b), T in rel.items():
        if a == 0:
            assert np.trace(T[:3, :3]) < -0.28
    extr, rel = BI.make_pose_graph(2, 5, collinear=0.01)
    c = np.array([-E[:3, :3].T @ E[:3, 3] for E in extr])
    assert np.abs(c[:, 1:]).max() <= 0.01 + 1e-12
    _, rel_c = BI.make_pose_graph(2, 5, collinear=0.01, corrupt=(1, 3))
    for k in rel:
        assert np.allclose(rel[k], rel_c[k]) == (k != (1, 3))


def test_degenerate_triangulation_rule():
    """A match at the principal point of both images under pure forward motion: the DLT matrix has zero z and w
    columns, the SVD returns the camera centre (depth 0), the rule returns (0, 0, 1).  Every other match
    triangulates as triangulate_points does."""
    from oracle import pose as P
    rng = np.random.default_rng(0)
    x0 = rng.uniform(-0.5, 0.5, (20, 2))
    x1 = rng.uniform(-0.5, 0.5, (20, 2))
    x0[3] = x1[3] = 0.0
    T = np.eye(4)
    T[2, 3] = -0.3
    X = P.triangulate_points_first_view_identity(T, x0, x1)
    ref = P.triangulate_points(np.eye(4)[:3][None], T[None, :3], x0[None], x1[None])[0]
    np.testing.assert_array_equal(ref[3], [0.0, 0.0, 0.0])
    np.testing.assert_array_equal(X[3], [0.0, 0.0, 1.0])
    keep = np.arange(20) != 3
    np.testing.assert_array_equal(X[keep], ref[keep])
    T[0, 3] = 0.1                                     # not along the optical axis: the point is unique again
    X = P.triangulate_points_first_view_identity(T, x0, x1)
    ref = P.triangulate_points(np.eye(4)[:3][None], T[None, :3], x0[None], x1[None])[0]
    np.testing.assert_array_equal(X, ref)
