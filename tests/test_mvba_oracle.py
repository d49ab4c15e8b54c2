"""CPU: the multi-view BA oracle (oracle/mvba.py) reproduces the reference's own known-answer tests
(pose_optimization/multi_view/bundle_adjustment/problem/test/test_ba_problem.cpp:165-184), with the
same scene, the same glibc rand() noise stream and the same tolerances."""
import numpy as np
import pytest

from oracle import mvba as M

EXPECTED = [0.3, -0.2, 0.5, 0.3, -0.4, 0.5]


@pytest.mark.parametrize('name,args,tol', [('Perfect2Cams5Pts', (0., 0., 0.), 1e-6),
                                           ('Noisy2Cams5Pts', (0.1, 10., 0.2), 9e-2),
                                           ('MoreNoisy2Cams5Pts', (0.2, 0., 0.3), 4e-2)])
def test_gtest_known_answers(name, args, tol):
    pb = M.gtest_problem(EXPECTED, *args)
    cams, pts, info = M.solve(pb)
    assert np.abs(cams[0]).max() < 1e-6                    # camera 0 stays fixed (:152-156)
    assert np.abs(cams[1] - np.array(EXPECTED)).max() < tol, (name, cams[1])
    assert info['final_cost'] <= info['initial_cost'] + 1e-30


def test_angle_axis_jacobian_and_roundtrip():
    rng = np.random.default_rng(0)
    for _ in range(5):
        w, p = rng.standard_normal(3) * 0.8, rng.standard_normal(3)
        J = M.d_rotated_point_d_angle_axis(w, p)
        eps = 1e-6
        Jn = np.stack([(M.angle_axis_to_R(w + eps * np.eye(3)[i]) @ p - M.angle_axis_to_R(w - eps * np.eye(3)[i]) @ p)
                       / (2 * eps) for i in range(3)], 1)
        assert np.abs(J - Jn).max() < 1e-8
        assert np.abs(M.R_to_angle_axis(M.angle_axis_to_R(w)) - w).max() < 1e-12


def _scene_digest(sc):
    import hashlib
    h = hashlib.sha256()
    for k in sc['kpts']:
        h.update(np.ascontiguousarray(k).tobytes())
    h.update(sc['K'].tobytes())
    h.update(sc['poses'].tobytes())
    for key in sorted(sc['matches']):
        h.update(sc['matches'][key].tobytes())
        h.update(sc['conf'][key].tobytes())
    return h.hexdigest()[:16]


@pytest.mark.parametrize('args,kw,digest', [((1, 3, 60), dict(outlier_frac=0.0), '6e8f9b6c84a7385e'),
                                            ((2, 5, 100), dict(outlier_frac=0.1), 'aa84f8b954d1d014'),
                                            ((7, 4, 120), dict(outlier_frac=0.0, noise_px=0.0), '1ae23e0574359342')])
def test_scene_generator_is_unchanged(args, kw, digest):
    """The scenes the GPU parity tests use are pinned: the ragged-view and empty-pair options of
    make_multi_view_scene leave the default scene (and its random draws) exactly as before, and
    spelling the defaults out gives the same scene."""
    assert _scene_digest(M.make_multi_view_scene(*args, **kw)) == digest
    assert _scene_digest(M.make_multi_view_scene(*args, view_counts=[args[2]] * args[1], empty_pairs=(), **kw)) == digest


def test_scene_ragged_views_and_empty_pairs():
    sc = M.make_multi_view_scene(5, 4, 300, view_counts=[300, 200, 7, 256], empty_pairs=[(1, 3)])
    assert [k.shape[0] for k in sc['kpts']] == [300, 200, 7, 256]
    for (a, b), m in sc['matches'].items():
        assert m.shape == sc['conf'][(a, b)].shape == (sc['kpts'][a].shape[0],)
        assert m.max() < sc['kpts'][b].shape[0]
        assert (m < 0).all() == ((a, b) == (1, 3))


def test_pipeline_recovers_poses():
    sc = M.make_multi_view_scene(3, 4, 80, outlier_frac=0.0, noise_px=0.2)
    out = M.multi_view_pipeline(sc)
    from oracle.pose import compute_pose_error
    for b in range(1, 4):
        gt = sc['poses'][b] @ np.linalg.inv(sc['poses'][0])
        pr = out['extr'][b] @ np.linalg.inv(out['extr'][0])
        et, er = compute_pose_error(gt, pr[:3, :3], pr[:3, 3])
        # translations inherit the per-pair scale ambiguity of the spanning-tree chain (the Theia
        # position-averaging step that resolves it is SURVEY.md f-1, not restated): rotations only
        assert er < 1.5, (b, et, er)
