"""Device-resident pose stage of the multi-view pipeline: what eval_multi_view.eval_bundle_adjust
(eval_multi_view.py:21-68) does through numpy, two subprocesses and four CSV files, as five
stream-ordered kernel launches with no host synchronisation:

  mvm_gather_matches     valid-match compaction            (bundle_adjust_io.py:66-98)
  mvm_w8pt               per pair w8pt + inlier test       (bundle_adjust_io.py:12-23 -> estimate_relative_pose.py:84)
  mvm_ba2view            per pair two-view LM BA           (bundle_adjust_io.py:19-22)
  mvm_spanning_tree_init maximum spanning tree + chaining  (bundle_adjust_io.py:135-172)
  mvm_multi_view_ba      global BA, camera 0 fixed         (ba_problem.cpp:115-157)

  mvm_ba_initialize      rotation averaging + LUD positions (ba_init.cpp:77-91, the `ba_initializer` binary)
between the spanning tree and the global BA (six launches in total).
"""
import ctypes as C

import torch

from ... import _lib


def _intr4(intr):
    return torch.stack([intr[..., 0, 0], intr[..., 1, 1], intr[..., 0, 2], intr[..., 1, 2]], -1).float()


class MultiViewPoseEngine:
    def __init__(self, conf_thresh=0.0, n_iterations_2view=10, max_iterations_ba=50, use_ba_init=True,
                 min_inliers=20, ransac_thresh=1.0, ransac_conf=0.99999, ransac_max_iters=1000, ransac_seed=0):
        self.conf_thresh = conf_thresh
        self.ransac_thresh = ransac_thresh           # pixels (eval_pairs.py:229)
        self.ransac_conf = ransac_conf               # estimate_pose's conf (models/models/utils.py:288)
        self.ransac_max_iters = ransac_max_iters     # OpenCV's findEssentialMat default
        self.ransac_seed = ransac_seed
        self.n_it2 = n_iterations_2view
        self.max_it = max_iterations_ba
        self.use_ba_init = use_ba_init
        self.min_inliers = min_inliers
        self._ws = None

    def _pair_index(self, pair_ids, dev):
        """Device index tensors (view a / view b of every pair), built once per pair list: indexing with a Python
        list would stage a pageable host->device copy every call, which blocks the host until the matcher's
        kernels have drained (measured: host enqueue time == GPU step time, tools/step_gaps.py)."""
        key = (tuple(pair_ids), str(dev))
        if getattr(self, '_pair_index_key', None) != key:
            self._pair_index_val = (torch.tensor([a for a, _ in pair_ids], dtype=torch.int64, device=dev),
                                    torch.tensor([b for _, b in pair_ids], dtype=torch.int64, device=dev))
            self._pair_index_key = key
        return self._pair_index_val

    def _gather(self, lib, state, mk0, mk1, mconf, n_valid, sp):
        """Valid-match compaction of every (tuple, pair); a ragged batch (state['slot_counts']) bounds each tuple by its
        device counts."""
        kp, T, P, B = state['kpts'], state['n_views'], len(state['pair_ids']), state['batch']
        cnt = (C.c_int * T)(*state['counts'])
        _lib.check(lib.mvm_gather_matches_ragged(_lib.ptr(kp), T, state['n_pad'], cnt,
                                                 _lib.ptr(state.get('slot_counts')), state['pairs'], P, B,
                                                 float(self.conf_thresh), _lib.ptr(mk0), _lib.ptr(mk1), _lib.ptr(mconf),
                                                 _lib.ptr(n_valid), sp), 'mvm_gather_matches_ragged')

    def run(self, state, intr, global_ba=True, rel_pose_method='w8pt_ba'):
        """state: MatcherEngine.last of the matcher call; intr: list (per view) of [B,3,3]/[B,4,4]
        intrinsics.  Returns dict with pairwise poses and (if global_ba) absolute extrinsics.
        rel_pose_method: 'w8pt' / 'w8pt_ba' (the same launches: w8pt, then the two-view BA) or the two-view RANSAC
        modes 'ransac' / 'ransac_ba' (eval_pairs.py:228-243; pairwise poses only, global_ba must be False)."""
        if rel_pose_method not in ('w8pt', 'w8pt_ba', 'ransac', 'ransac_ba'):
            raise ValueError('rel_pose_method must be one of w8pt, w8pt_ba, ransac, ransac_ba, not %r' % (rel_pose_method,))
        if rel_pose_method.startswith('ransac'):
            if global_ba:
                raise ValueError('rel_pose_method=%r computes pairwise poses only: call run(..., global_ba=False)'
                                 % rel_pose_method)
            return self._run_ransac(state, intr, rel_pose_method == 'ransac_ba')
        lib = _lib.lib()
        kp, n_pad = state['kpts'], state['n_pad']
        pairs, pair_ids = state['pairs'], state['pair_ids']
        B, T, P = state['batch'], state['n_views'], len(state['pair_ids'])
        dev = kp.device
        f32 = dict(dtype=torch.float32, device=dev)
        mk0 = torch.empty(B, P, n_pad, 2, **f32)
        mk1 = torch.empty(B, P, n_pad, 2, **f32)
        mconf = torch.empty(B, P, n_pad, **f32)
        n_valid = torch.empty(B, P, dtype=torch.int32, device=dev)
        sp = _lib.stream_ptr()
        with torch.cuda.device(dev):
            self._gather(lib, state, mk0, mk1, mconf, n_valid, sp)
            i4 = torch.stack([_intr4(k.to(dev)) for k in intr], 1)                    # [B,T,4]
            ia_idx, ib_idx = self._pair_index(pair_ids, dev)
            ia = i4.index_select(1, ia_idx)                                           # [B,P,4]
            ib = i4.index_select(1, ib_idx)
            BP = B * P
            T_w8 = torch.empty(B, P, 4, 4, **f32)
            k0n = torch.empty(B, P, n_pad, 2, **f32)
            k1n = torch.empty(B, P, n_pad, 2, **f32)
            cn = torch.empty(B, P, n_pad, **f32)
            pos = torch.empty(B, P, n_pad, dtype=torch.uint8, device=dev)
            inl = torch.empty(B, P, n_pad, dtype=torch.uint8, device=dev)
            succ = torch.empty(B, P, dtype=torch.uint8, device=dev)
            _lib.check(lib.mvm_w8pt(_lib.ptr(mk0), _lib.ptr(mk1), _lib.ptr(ia), _lib.ptr(ib), _lib.ptr(mconf), BP,
                                    n_pad, None, 0, 1, _lib.ptr(T_w8), _lib.ptr(k0n), _lib.ptr(k1n), _lib.ptr(cn),
                                    _lib.ptr(pos), _lib.ptr(inl), None, _lib.ptr(n_valid), _lib.ptr(succ), sp),
                       'mvm_w8pt')
            T_ba = torch.empty(B, P, 4, 4, **f32)
            valid = torch.empty(B, P, dtype=torch.uint8, device=dev)
            pts = torch.empty(BP * n_pad * 3, dtype=torch.float64, device=dev)
            _lib.check(lib.mvm_ba2view(_lib.ptr(k0n), _lib.ptr(k1n), _lib.ptr(cn), _lib.ptr(T_w8), BP, n_pad,
                                       int(self.n_it2), _lib.ptr(T_ba), _lib.ptr(valid), _lib.ptr(pts), None,
                                       _lib.ptr(n_valid), _lib.ptr(pos), sp), 'mvm_ba2view')
            out = {'T_w8pt': T_w8, 'T_pair': T_ba, 'success': succ.bool(), 'valid_ba': valid.bool(),
                   'n_matches': n_valid, 'inliers': inl, 'pos_depth_mask': pos}
            if not global_ba:
                return out
            pa = (C.c_int * P)(*[a for a, _ in pair_ids])
            pb = (C.c_int * P)(*[b for _, b in pair_ids])
            extr0 = torch.empty(B, T, 4, 4, dtype=torch.float64, device=dev)
            on_tree = torch.empty(B, P, dtype=torch.uint8, device=dev)
            _lib.check(lib.mvm_spanning_tree_init(pa, pb, T, P, B, _lib.ptr(T_ba), _lib.ptr(n_valid), _lib.ptr(succ),
                                                  _lib.ptr(extr0), _lib.ptr(on_tree), sp), 'mvm_spanning_tree_init')
            extr_tree = extr0
            if self.use_ba_init:
                extr0 = torch.empty(B, T, 4, 4, dtype=torch.float64, device=dev)
                _lib.check(lib.mvm_ba_initialize(pa, pb, T, P, B, n_pad, _lib.ptr(extr_tree), _lib.ptr(T_ba),
                                                 _lib.ptr(succ), _lib.ptr(on_tree), _lib.ptr(inl), int(self.min_inliers),
                                                 _lib.ptr(extr0), None, sp), 'mvm_ba_initialize')
            nbytes = lib.mvm_mvba_workspace_bytes(T, P, B, n_pad)
            if self._ws is None or self._ws.numel() < nbytes or self._ws.device != dev:
                self._ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
            extr = torch.empty(B, T, 4, 4, **f32)
            iters = torch.empty(B, dtype=torch.int32, device=dev)
            cost = torch.empty(B, 2, dtype=torch.float64, device=dev)
            _lib.check(lib.mvm_multi_view_ba(pa, pb, T, P, B, n_pad, _lib.ptr(k0n), _lib.ptr(k1n), _lib.ptr(mconf),
                                             _lib.ptr(n_valid), _lib.ptr(extr0), _lib.ptr(extr), int(self.max_it),
                                             _lib.ptr(iters), _lib.ptr(cost), _lib.ptr(self._ws), nbytes, sp),
                       'mvm_multi_view_ba')
            out.update({'extrinsics_tree': extr_tree, 'extrinsics_init': extr0, 'extrinsics': extr, 'ba_iterations': iters, 'ba_cost': cost,
                        'kpts_norm_a': k0n, 'kpts_norm_b': k1n, 'mconf': mconf})
        return out

    def _run_ransac(self, state, intr, refine):
        """eval_pairs.py:228-243: estimate_pose (RANSAC + recoverPose) on the valid matches of every pair, then, with
        refine, the two-view BA on the inliers of that pose weighted by the raw match confidences."""
        lib = _lib.lib()
        kp, n_pad = state['kpts'], state['n_pad']
        pairs, pair_ids = state['pairs'], state['pair_ids']
        B, T, P = state['batch'], state['n_views'], len(state['pair_ids'])
        dev = kp.device
        f32 = dict(dtype=torch.float32, device=dev)
        i32 = dict(dtype=torch.int32, device=dev)
        u8 = dict(dtype=torch.uint8, device=dev)
        BP = B * P
        mk0 = torch.empty(B, P, n_pad, 2, **f32)
        mk1 = torch.empty(B, P, n_pad, 2, **f32)
        mconf = torch.empty(B, P, n_pad, **f32)
        n_valid = torch.empty(B, P, **i32)
        sp = _lib.stream_ptr()
        with torch.cuda.device(dev):
            self._gather(lib, state, mk0, mk1, mconf, n_valid, sp)
            i4 = torch.stack([_intr4(k.to(dev)) for k in intr], 1)
            ia_idx, ib_idx = self._pair_index(pair_ids, dev)
            ia = i4.index_select(1, ia_idx).contiguous()
            ib = i4.index_select(1, ib_idx).contiguous()
            T_r = torch.empty(B, P, 4, 4, **f32)
            k0n = torch.empty(B, P, n_pad, 2, **f32)
            k1n = torch.empty(B, P, n_pad, 2, **f32)
            inl = torch.empty(B, P, n_pad, **u8)
            n_inl = torch.empty(B, P, **i32)
            E = torch.empty(B, P, 10, 9, dtype=torch.float64, device=dev)
            n_mod = torch.empty(B, P, **i32)
            iters = torch.empty(B, P, **i32)
            succ = torch.empty(B, P, **u8)
            _lib.check(lib.mvm_ransac_essential(_lib.ptr(mk0), _lib.ptr(mk1), _lib.ptr(ia), _lib.ptr(ib), BP, n_pad,
                                                _lib.ptr(n_valid), float(self.ransac_thresh), float(self.ransac_conf),
                                                int(self.ransac_max_iters), int(self.ransac_seed), _lib.ptr(T_r),
                                                _lib.ptr(k0n), _lib.ptr(k1n), _lib.ptr(inl), _lib.ptr(n_inl), _lib.ptr(E),
                                                _lib.ptr(n_mod), _lib.ptr(iters), _lib.ptr(succ), sp),
                       'mvm_ransac_essential')
            out = {'T_ransac': T_r, 'T_pair': T_r, 'success': succ.bool(), 'n_matches': n_valid, 'inliers': inl,
                   'n_inliers': n_inl, 'ransac_iterations': iters, 'E': E, 'n_models': n_mod,
                   'kpts_a': mk0, 'kpts_b': mk1, 'mconf': mconf, 'kpts_norm_a': k0n, 'kpts_norm_b': k1n}
            if refine:
                T_ba = torch.empty(B, P, 4, 4, **f32)
                valid = torch.empty(B, P, **u8)
                pts = torch.empty(BP * n_pad * 3, dtype=torch.float64, device=dev)
                _lib.check(lib.mvm_ba2view(_lib.ptr(k0n), _lib.ptr(k1n), _lib.ptr(mconf), _lib.ptr(T_r), BP, n_pad,
                                           int(self.n_it2), _lib.ptr(T_ba), _lib.ptr(valid), _lib.ptr(pts), None,
                                           _lib.ptr(n_valid), _lib.ptr(inl), sp), 'mvm_ba2view')
                out.update({'T_pair': T_ba, 'valid_ba': valid.bool()})
        return out


def relative_from_extrinsics(extr, a, b):
    """T_a->b = extr[b] @ inv(extr[a]) (eval_multi_view.py:58)."""
    return extr[:, b] @ torch.linalg.inv(extr[:, a])
