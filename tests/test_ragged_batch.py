"""Host side of ragged batches (no GPU): the C ABI declares and binds the ragged entry points and refuses bad arguments
before any launch, split_ragged_result cuts padded outputs, and MultiViewPipeline routes an image batch with ragged
counts (tuples with keypoints in every view as one ragged batch, tuples with an empty view alone)."""
import ctypes as C
import os
import re
import types

import torch

from e2e_multi_view_matching_b200 import _lib
from e2e_multi_view_matching_b200.models.multi_view_matcher import split_ragged_result, slot_counts_of
from e2e_multi_view_matching_b200.pipeline import MultiViewPipeline

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NEW = ('mvm_matcher_forward_ragged', 'mvm_pack_views_ragged', 'mvm_gather_matches_ragged')


def test_header_declares_and_lib_binds_ragged_entries():
    header = open(os.path.join(ROOT, 'include', 'mvm_b200.h')).read()
    L = _lib.lib()
    for name in NEW:
        assert re.search(r'\bint %s\(' % name, header), name
        assert getattr(L, name).argtypes is not None, name
    assert 'const int* slot_counts' in header


def test_forward_ragged_refuses_unsupported_options_and_null_pointers():
    L = _lib.lib()
    fake = C.c_void_p(0x1000)      # never dereferenced: the host checks fail first
    cnt = (C.c_int * 2)(64, 64)
    wh = (C.c_float * 4)(640, 480, 640, 480)
    pairs = (_lib.PairIO * 1)()
    for mode, score in ((0, 1), (1, 1), (3, 0)):
        o = _lib.MatcherOptions()
        L.mvm_matcher_options_default(C.byref(o))
        o.math_mode, o.score_kernel = mode, score
        rc = L.mvm_matcher_forward_ragged(None, 1, 2, 64, cnt, fake, fake, fake, fake, wh, 100, 0.0, pairs, 1, fake, 1 << 30,
                                          C.byref(o), None)
        assert rc == 1, (mode, score)
    rc = L.mvm_matcher_forward_ragged(None, 1, 2, 64, cnt, fake, fake, fake, fake, wh, 100, 0.0, pairs, 1, fake, 1 << 30,
                                      None, None)
    assert rc == 1


def test_pack_and_gather_ragged_refuse_bad_arguments():
    L = _lib.lib()
    fake = C.c_void_p(0x1000)
    cnt = (C.c_int * 2)(64, 64)
    ptrs = (C.c_void_p * 2)(0x1000, 0x1000)
    assert L.mvm_pack_views_ragged(ptrs, ptrs, ptrs, cnt, fake, 1, 2, 64, None, fake, fake, None) == 1
    assert L.mvm_pack_views_ragged(ptrs, ptrs, ptrs, (C.c_int * 2)(65, 64), fake, 1, 2, 64, fake, fake, fake, None) == 1
    pairs = (_lib.PairIO * 1)()
    pairs[0].view_a, pairs[0].view_b = 0, 1
    assert L.mvm_gather_matches_ragged(None, 2, 64, cnt, fake, pairs, 1, 1, 0.0, fake, fake, fake, fake, None) == 1
    pairs[0].matches_a, pairs[0].conf = 0x1000, 0x1000
    pairs[0].view_b = 2                # no slot 2 in a 2-view batch: its count would be read out of bounds
    assert L.mvm_gather_matches_ragged(fake, 2, 64, cnt, fake, pairs, 1, 1, 0.0, fake, fake, fake, fake, None) == 1


def test_split_ragged_result_cuts_each_tuple():
    B, caps = 3, [7, 5, 6]
    counts = [[7, 2, 4], [1, 5, 3], [6, 6, 0]]        # per view id, [B]
    res = {'matches0_0_1': torch.arange(B * 7).view(B, 7), 'matches1_0_1': torch.arange(B * 5).view(B, 5),
           'matching_scores2_0_2': torch.rand(B, 6), 'scores_1_2': torch.rand(B, 6, 7),
           'conf_scores_0_2': torch.rand(B, 7, 1), 'keypoints1': torch.rand(B, 5, 2), 'scores2': torch.rand(B, 6),
           'descriptors0': torch.rand(B, 256, 7), 'counts0': torch.tensor(counts[0]), 'intr0': torch.rand(B, 3, 3),
           'conf_scores_1_2': None, 'ids': [0, 1, 2]}
    out = split_ragged_result(res, [torch.tensor(c) for c in counts])
    assert len(out) == B
    for b in range(B):
        n = [counts[i][b] for i in range(3)]
        d = out[b]
        assert 'counts0' not in d and 'conf_scores_1_2' not in d and d['ids'] == [0, 1, 2]
        assert torch.equal(d['matches0_0_1'], res['matches0_0_1'][b:b + 1, :n[0]])
        assert torch.equal(d['matches1_0_1'], res['matches1_0_1'][b:b + 1, :n[1]])
        assert torch.equal(d['matching_scores2_0_2'], res['matching_scores2_0_2'][b:b + 1, :n[2]])
        assert torch.equal(d['scores_1_2'], res['scores_1_2'][b:b + 1, :n[1] + 1, :n[2] + 1])
        assert torch.equal(d['conf_scores_0_2'], res['conf_scores_0_2'][b:b + 1, :n[0]])
        assert torch.equal(d['keypoints1'], res['keypoints1'][b:b + 1, :n[1]])
        assert torch.equal(d['scores2'], res['scores2'][b:b + 1, :n[2]])
        assert torch.equal(d['descriptors0'], res['descriptors0'][b:b + 1, :, :n[0]])
        assert torch.equal(d['intr0'], res['intr0'][b:b + 1])
    assert caps == [max(c) for c in counts]


def test_slot_counts_of():
    assert slot_counts_of({'keypoints0': None}, [0, 1]) is None
    d = {'counts0': torch.tensor([3, 4]), 'counts2': torch.tensor([5, 6], dtype=torch.int64)}
    s = slot_counts_of(d, [0, 2])
    assert s.dtype == torch.int32 and s.tolist() == [[3, 5], [4, 6]]


class FakeMatcher:
    config = {'multi_frame_matching': True, 'conf_mlp': True}

    def __init__(self):
        self.calls = []
        self._engine = types.SimpleNamespace(last=None)

    def __call__(self, data):
        T = len(data['ids'])
        B = data['keypoints0'].shape[0]
        self.calls.append({'B': B, 'widths': [data['keypoints%d' % i].shape[1] for i in range(T)],
                           'counts': [data['counts%d' % i].tolist() for i in range(T)] if 'counts0' in data else None,
                           'tag': data['intr0'][:, 0, 0].tolist()})
        self._engine.last = {'view_ids': list(range(T))}
        return {'matches0_0_1': torch.zeros(B, data['keypoints0'].shape[1], dtype=torch.int64)}


class FakePose:
    def run(self, state, intr, global_ba=True):
        return {'extrinsics': torch.stack([k[:, 0, 0] for k in intr], 1)}


def test_pipeline_routes_ragged_image_batch():
    T, B, K = 3, 5, 8
    host = [[8, 3, 5, 0, 6], [2, 8, 4, 7, 1], [5, 5, 5, 5, 0]]   # [T][B]: tuples 3 and 4 have an empty view
    counts = torch.tensor(host, dtype=torch.int32)
    feats = {'keypoints': torch.rand(T, B, K, 2), 'scores': torch.rand(T, B, K), 'descriptors': torch.rand(T, B, 256, K)}
    data = {'ids': list(range(T))}
    for i in range(T):
        data['intr%d' % i] = torch.arange(B, dtype=torch.float32).view(B, 1, 1).expand(B, 3, 3).contiguous()
        data['image%d' % i] = torch.zeros(B, 1, 16, 16)
    matcher = FakeMatcher()
    pipe = MultiViewPipeline(matcher)
    pipe.pose = FakePose()
    out = pipe._run_ragged(data, (host, counts, feats), True)
    assert len(out) == B
    results, poses = [r for r, _ in out], [p for _, p in out]
    alone = [c for c in matcher.calls if c['counts'] is None]
    ragged = [c for c in matcher.calls if c['counts'] is not None]
    assert [c['tag'] for c in alone] == [[3.0], [4.0]]
    assert all(c['B'] == 1 for c in alone)
    assert alone[0]['widths'] == [0, 7, 5] and alone[1]['widths'] == [6, 1, 0]
    assert len(ragged) == 1 and ragged[0]['B'] == 3 and ragged[0]['tag'] == [0.0, 1.0, 2.0]
    assert ragged[0]['widths'] == [8, 8, 5]
    assert ragged[0]['counts'] == [[8, 3, 5], [2, 8, 4], [5, 5, 5]]
    for b in range(B):
        assert poses[b]['extrinsics'].tolist() == [[float(b)] * T]
        assert results[b]['keypoints1'].shape == (1, host[1][b], 2)
        assert torch.equal(results[b]['keypoints1'][0], feats['keypoints'][1, b, :host[1][b]])


def test_pipeline_batch_of_one_with_keypoints_is_unchanged():
    matcher = FakeMatcher()
    pipe = MultiViewPipeline(matcher)
    pipe.pose = FakePose()
    data = {'ids': [0, 1], 'keypoints0': torch.rand(1, 4, 2), 'keypoints1': torch.rand(1, 6, 2),
            'intr0': torch.ones(1, 3, 3), 'intr1': torch.ones(1, 3, 3)}
    res, pose = pipe(data)
    assert isinstance(res, dict) and matcher.calls == [{'B': 1, 'widths': [4, 6], 'counts': None, 'tag': [1.0]}]


class FakeSuperPoint:
    """forward_batch / forward with fixed per-image counts ([T * B], view-major like the batch it gets)."""

    def __init__(self, K, counts):
        self.config = {'max_keypoints': K, 'fill_with_random_keypoints': False}
        self.counts = counts
        self.calls = []

    def forward_batch(self, images):
        n, K = images.shape[0], self.config['max_keypoints']
        self.calls.append(('forward_batch', n))
        return {'keypoints': torch.rand(n, K, 2), 'scores': torch.rand(n, K), 'descriptors': torch.rand(n, 256, K),
                'counts': torch.tensor(self.counts[:n], dtype=torch.int32)}

    def __call__(self, data):
        n = sum(x.shape[0] for x in data['image'])
        self.calls.append(('forward', n))
        return {'keypoints': [torch.rand(5, 2) for _ in range(n)], 'scores': [torch.rand(5) for _ in range(n)],
                'descriptors': [torch.rand(256, 5) for _ in range(n)]}


def image_batch(T, B, size=16):
    d = {'ids': list(range(T))}
    for i in range(T):
        d['image%d' % i] = torch.zeros(B, 1, size, size)
        d['intr%d' % i] = torch.arange(B, dtype=torch.float32).view(B, 1, 1).expand(B, 3, 3).contiguous()
    return d


def test_pipeline_call_routes_by_batch_and_counts(monkeypatch):
    monkeypatch.setattr(torch.Tensor, 'cuda', lambda self, *a, **k: self)      # the fakes run on the CPU
    T, K = 3, 8

    def pipe_with(counts, k=K):
        matcher = FakeMatcher()
        pipe = MultiViewPipeline(matcher, superpoint=FakeSuperPoint(k, counts))
        pipe.pose = FakePose()
        return pipe, matcher

    # B = 1: the existing path (run_super_point), the matcher sees the tuple cut to its counts
    pipe, matcher = pipe_with([8, 3, 6])
    res, pose = pipe(image_batch(T, 1))
    assert isinstance(res, dict) and matcher.calls[0]['B'] == 1 and matcher.calls[0]['widths'] == [8, 3, 6]
    assert matcher.calls[0]['counts'] is None and pipe.superpoint.calls == [('forward_batch', 3)]
    # B > 1, every image at max_keypoints: one batched call, no device counts; run_tuples splits it
    pipe, matcher = pipe_with([K] * 6)
    res, pose = pipe(image_batch(T, 2))
    assert isinstance(res, dict) and matcher.calls == [{'B': 2, 'widths': [K] * T, 'counts': None, 'tag': [0.0, 1.0]}]
    tuples = pipe.run_tuples(image_batch(T, 2))
    assert len(tuples) == 2 and tuples[1][0]['keypoints2'].shape == (1, K, 2)
    assert tuples[1][1]['extrinsics'].tolist() == [[1.0] * T]
    # B > 1 with ragged counts: __call__ refuses (one tensor per output cannot hold them), run_tuples runs them ragged
    counts = [8, 3, 6, 2, 7, 5]            # view-major: view 0 of tuples 0, 1, view 1 of tuples 0, 1, ...
    pipe, matcher = pipe_with(counts)
    try:
        pipe(image_batch(T, 2))
        raise AssertionError('a ragged image batch must not come back as one batch')
    except ValueError as e:
        assert 'run_tuples' in str(e)
    pipe, matcher = pipe_with(counts)
    tuples = pipe.run_tuples(image_batch(T, 2))
    assert len(matcher.calls) == 1 and matcher.calls[0]['counts'] == [[8, 3], [6, 2], [7, 5]]
    assert matcher.calls[0]['widths'] == [8, 6, 7]
    assert [t[0]['keypoints1'].shape[1] for t in tuples] == [6, 2]
    # SuperPoint.forward_batch does not serve max_keypoints > pixels of the score map: run_super_point's other path
    pipe, matcher = pipe_with([], k=16 * 16 + 1)
    res, pose = pipe(image_batch(T, 2))
    assert pipe.superpoint.calls == [('forward', 6)] and matcher.calls[0]['widths'] == [5] * T
