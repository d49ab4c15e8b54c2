"""CPU: the RANSAC oracle (tests/ransac_oracle.py) pinned to OpenCV 4.13, the library the reference's estimate_pose
calls: the five-point solution sets, the float-rounded inlier test, recoverPose with its in-place mask, the estimate_pose
loop over stacked solutions, and the statistics of the RANSAC itself (cv2's samples cannot be reproduced)."""
import subprocess
import sys

import numpy as np
import pytest

cv2 = pytest.importorskip('cv2')

from oracle import pose as P
from tests import ransac_oracle as RO


def _five(rng, kind):
    R = P.rodrigues(rng.standard_normal(3) * 0.3)
    t = rng.standard_normal(3) * (0.01 if kind == 'small_baseline' else 1.0)
    X = np.column_stack([rng.uniform(-1, 1, 5), rng.uniform(-1, 1, 5), rng.uniform(2, 6, 5)])
    if kind == 'near_planar':
        X[:, 2] = 4.0 + 1e-3 * rng.standard_normal(5)
    X2 = X @ R.T + t
    return X[:, :2] / X[:, 2:], X2[:, :2] / X2[:, 2:]


def _essential_residual(E, x1, x2):
    return max(np.abs(RO.epipolar_rows(x1, x2) @ E.reshape(9)).max(),
               np.abs(2 * E @ E.T @ E - np.trace(E @ E.T) * E).max())


def test_five_point_solution_sets_match_cv2():
    """Same number of solutions and the same unit-norm, sign-fixed E to 1e-8 on generic configurations.  The two
    solvers lose accuracy differently on ill-conditioned sets (both small-baseline and near-planar ones and the odd
    generic set with close roots): every solution that differs by more than 1e-8 is reported with the root
    separation of the degree-10 polynomial and both solvers' constraint residuals; on generic sets at most 2 % may
    differ, none by more than 1e-5."""
    rng = np.random.default_rng(0)
    report = []
    n_sol = 0
    for trial in range(240):
        kind = ['generic', 'generic', 'small_baseline', 'near_planar'][trial % 4]
        x1, x2 = _five(rng, kind)
        E, _ = cv2.findEssentialMat(x1, x2, np.eye(3), method=cv2.RANSAC, threshold=1e-3)
        cvs = [RO.normalize_E(E[3 * k:3 * k + 3]) for k in range(len(E) // 3)] if E is not None else []
        ours = RO.five_point(x1, x2)
        Q = RO.epipolar_rows(x1, x2)
        roots = RO.real_roots(RO.det_polynomial(RO.hidden_variable_matrix(
            RO.gauss_jordan(RO.constraint_matrix(RO.null_space_householder(Q))))))
        sep = float(np.diff(roots).min()) if len(roots) > 1 else np.inf
        if len(cvs) != len(ours):
            report.append((trial, kind, 'count', len(cvs), len(ours), sep))
            assert kind != 'generic', report[-1]
            continue
        for e in cvs:
            n_sol += 1
            d = min(np.abs(e - o).max() for o in ours)
            if d > 1e-8:
                o = min(ours, key=lambda o: np.abs(e - o).max())
                report.append((trial, kind, 'E', d, sep, _essential_residual(o, x1, x2), _essential_residual(e, x1, x2)))
                if kind == 'generic':
                    assert d < 1e-5, report[-1]
    n_generic_off = sum(1 for r in report if r[1] == 'generic')
    print('solutions compared: %d; differing by more than 1e-8: %d (generic: %d)' % (n_sol, len(report), n_generic_off))
    for r in report:
        print(r)
    assert n_sol > 700
    assert n_generic_off <= 0.02 * n_sol / 2


def _scene(seed, n, outlier, noise=1.0):
    sc = P.make_two_view_scene(seed, n, outlier_frac=outlier, noise_px=noise)
    K = sc['intr'][0].astype(np.float64)
    return sc, K, RO.normalize_kpts(sc['kpts0'][0], K), RO.normalize_kpts(sc['kpts1'][0], K)


@pytest.mark.parametrize('outlier', [0.3, 0.6])
def test_float_rounded_inlier_test_reproduces_cv2_mask(outlier):
    for seed in range(4):
        sc, K, x1, x2 = _scene(seed, 1024, outlier)
        thr = RO.norm_threshold(K, K, 1.0)
        E, mask = cv2.findEssentialMat(x1, x2, np.eye(3), threshold=thr, prob=0.99999, method=cv2.RANSAC)
        np.testing.assert_array_equal(RO.inlier_mask(E[:3], x1, x2, thr), mask.ravel() > 0)


def test_recover_pose_matches_cv2_including_the_in_place_mask():
    """recoverPose called exactly as estimate_pose calls it, `cv2.recoverPose(E, x1, x2, np.eye(3), 1e9, mask=mask)`:
    the positional 1e9 is the R output of the (E, p1, p2, K[, R[, t[, mask]]]) overload (the call returns four values),
    so OpenCV's fixed distance threshold of 50 applies, which the oracle's default reproduces.  20 scenes, for cv2's E
    with its mask and for the true E with random masks over the true matches."""
    rng = np.random.default_rng(3)
    for seed in range(20):
        sc, K, x1, x2 = _scene(seed, 1024, 0.3)
        thr = RO.norm_threshold(K, K, 1.0)
        E, mask = cv2.findEssentialMat(x1, x2, np.eye(3), threshold=thr, prob=0.99999, method=cv2.RANSAC)
        T = sc['T_021'][0].astype(np.float64)
        E_true = P.hat(T[:3, 3]) @ T[:3, :3]
        rand = ((rng.uniform(size=1024) < 0.5) & ~sc['outlier'][0]).astype(np.uint8)[:, None]
        for Ek, mk in ((E[:3], mask), (E_true, rand)):
            m_cv = mk.copy()
            ret = cv2.recoverPose(Ek, x1, x2, np.eye(3), 1e9, mask=m_cv)
            assert len(ret) == 4
            n_cv, R_cv, t_cv, _ = ret
            n, R, t, m = RO.recover_pose(Ek, x1, x2, mk.ravel() > 0)
            assert n == n_cv, seed
            np.testing.assert_allclose(R, R_cv, atol=1e-9)
            np.testing.assert_allclose(t, t_cv[:, 0], atol=1e-9)
            np.testing.assert_array_equal(m, m_cv.ravel() > 0)


def _reference_flow_on(E, mask, x1, x2):
    """models/models/utils.py:300-312 restated with cv2."""
    best, ret = 0, None
    for _E in np.split(E, len(E) / 3):
        n, R, t, _ = cv2.recoverPose(_E, x1, x2, np.eye(3), 1e9, mask=mask)
        if n > best:
            best, ret = n, (R, t[:, 0], mask.ravel() > 0)
    return ret


def test_five_point_estimate_pose_loop_matches_reference_flow():
    """With five matches estimate_pose runs recoverPose on every stacked solution, each call seeing the mask the
    previous one left.  Fed cv2's solutions in cv2's order, the oracle's loop returns what the reference's does (the
    order of the solutions is the solver's: this project's is ascending in the hidden variable)."""
    rng = np.random.default_rng(1)
    checked, differ = 0, []
    for trial in range(120):
        x1, x2 = _five(rng, 'generic')
        E, mask = cv2.findEssentialMat(x1, x2, np.eye(3), method=cv2.RANSAC, threshold=1e-3)
        if E is None:
            continue
        ref = _reference_flow_on(E, mask.copy(), x1, x2)
        got = RO.recover_pose_loop(E, x1, x2, mask.ravel() > 0)
        assert (ref is None) == (got is None)
        # a tie between two candidates of the chosen call is decided by the R1 / R2 labels, which depend on the sign
        # conventions of the SVD (OpenCV's own vs LAPACK's): only untied calls are compared
        n0, _, _, _, good = RO.recover_pose(E[:3], x1, x2, mask.ravel() > 0, return_counts=True)
        if ref is not None and good.count(n0) == 1:
            same = (np.abs(got[0] - ref[0]).max() < 1e-9 and np.abs(got[1] - ref[1]).max() < 1e-9
                    and np.array_equal(got[2], ref[2]))
            if not same:
                differ.append((trial, good, got[2].astype(int).tolist(), ref[2].astype(int).tolist()))
            checked += 1
    print('untied five-point cases: %d, differing from the reference flow: %d' % (checked, len(differ)))
    for d in differ:
        print(d)
    assert checked > 80 and len(differ) <= 0.05 * checked


def _auc(errors):
    return np.array(P.pose_auc(np.array(errors), [5, 10, 20])) * 100


def test_ransac_statistics_comparable_to_cv2():
    """cv2's RANSAC is deterministic; its spread under permutations of the input order is the yardstick for the
    oracle's own samples.  32 pairs x 256 matches per outlier level."""
    for outlier in (0.3, 0.6):
        errs_cv = [[] for _ in range(3)]
        errs_or = []
        for seed in range(32):
            sc, K, x1, x2 = _scene(1000 + seed, 256, outlier)
            T = sc['T_021'][0].astype(np.float64)
            thr = RO.norm_threshold(K, K, 1.0)
            for p in range(3):
                perm = np.random.default_rng(seed * 7 + p).permutation(256) if p else np.arange(256)
                E, mask = cv2.findEssentialMat(x1[perm], x2[perm], np.eye(3), threshold=thr, prob=0.99999,
                                               method=cv2.RANSAC)
                ret = _reference_flow_on(E, mask, x1[perm], x2[perm]) if E is not None else None
                errs_cv[p].append(np.inf if ret is None else max(P.compute_pose_error(T, ret[0], ret[1])))
            ret = RO.estimate_pose(sc['kpts0'][0], sc['kpts1'][0], K, K, 1.0, seed=seed)
            errs_or.append(np.inf if ret is None else max(P.compute_pose_error(T, ret[0], ret[1])))
        cv = np.array([_auc(e) for e in errs_cv])
        ours = _auc(errs_or)
        lo, hi = cv.min(0), cv.max(0)
        spread = hi - lo
        print('outliers %.1f: cv2 AUC@5/10/20 %s .. %s, oracle %s' % (outlier, lo.round(1), hi.round(1), ours.round(1)))
        assert (ours >= lo - 2 * spread - 5).all() and (ours <= hi + 2 * spread + 5).all()


def test_package_import_does_not_import_cv2():
    code = ('import sys; import e2e_multi_view_matching_b200, e2e_multi_view_matching_b200.models.utils, '
            'e2e_multi_view_matching_b200.pipeline, e2e_multi_view_matching_b200.eval_pairs; '
            'assert "cv2" not in sys.modules')
    subprocess.run([sys.executable, '-c', code], check=True, cwd=RO.__file__.rsplit('/tests/', 1)[0])
