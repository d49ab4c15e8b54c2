"""Ragged batches: tuples whose views have different keypoint counts, the counts on the device (counts{i}), matched and
posed in one batch (mvm_matcher_forward_ragged, mvm_gather_matches_ragged).  Tuple b of a ragged batch must be what a
batch-of-one call on its cut tensors gives: bitwise at the same capacities, within the matcher's tolerances at its own."""
import ctypes as C

import numpy as np
import pytest
import torch

from e2e_multi_view_matching_b200 import _lib
from e2e_multi_view_matching_b200.models.multi_view_matcher import MultiViewMatcher, split_ragged_result
from e2e_multi_view_matching_b200.pose_optimization.multi_view.pose_engine import MultiViewPoseEngine
from e2e_multi_view_matching_b200.synthetic import make_scene_tuple_inputs, make_state_dict
from tests.test_sinkhorn_shapes_gpu import CASES as SINKHORN_SHAPES
from tests.util import compare_matcher_outputs

pytestmark = pytest.mark.gpu

MV_LAYERS = ['self', 'cross'] * 3
PAIR_LAYERS = ['self', 'cross'] * 2
OUT_KEYS = ('matches', 'matching_scores', 'scores_', 'conf_scores_')


def make_matcher(layers, multi=True, seed=3):
    sd = make_state_dict(len(layers), seed=seed, final_proj_gain=12.0, conf_head='score')
    m = MultiViewMatcher({'GNN_layers': layers, 'multi_frame_matching': multi}).eval()
    m.load_state_dict({k: torch.from_numpy(np.asarray(v)) for k, v in sd.items()})
    return m.cuda()


@pytest.fixture(scope='module')
def mv():
    return make_matcher(MV_LAYERS)


@pytest.fixture(scope='module')
def pair():
    return make_matcher(PAIR_LAYERS, multi=False)


def scene(seed, T, cap, B):
    d = make_scene_tuple_inputs(seed, T, cap, batch=B)
    return {k: (torch.from_numpy(v).cuda() if isinstance(v, np.ndarray) and not k.startswith('image')
                else (torch.empty(v.shape, device='meta') if isinstance(v, np.ndarray) else v)) for k, v in d.items()}


def with_counts(data, counts, pad=None):
    """counts [B][T] host ints -> data with counts{i}; pad (a float) overwrites the caller's rows past each count."""
    d = dict(data)
    T = len(counts[0])
    for i in range(T):
        d['counts%d' % i] = torch.tensor([c[i] for c in counts], dtype=torch.int32, device='cuda')
        if pad is not None:
            k, s, de = d['keypoints%d' % i].clone(), d['scores%d' % i].clone(), d['descriptors%d' % i].clone()
            for b, c in enumerate(counts):
                k[b, c[i]:] = pad
                s[b, c[i]:] = pad
                de[b, :, c[i]:] = pad
            d['keypoints%d' % i], d['scores%d' % i], d['descriptors%d' % i] = k, s, de
    return d


def select(data, idx, T, cuts=None):
    """Tuples idx of a batch (cuts: per view, the width to keep)."""
    sel = torch.tensor(idx, device='cuda')
    B = data['keypoints0'].shape[0]
    d = {k: (v.index_select(0, sel) if torch.is_tensor(v) and v.device.type == 'cuda' and v.shape[0] == B else v)
         for k, v in data.items()}
    if cuts is not None:
        for i in range(T):
            d['keypoints%d' % i] = d['keypoints%d' % i][:, :cuts[i]]
            d['scores%d' % i] = d['scores%d' % i][:, :cuts[i]]
            d['descriptors%d' % i] = d['descriptors%d' % i][:, :, :cuts[i]].contiguous()
    return d


def outputs(res):
    return {k: v for k, v in res.items() if k.startswith(OUT_KEYS) and v is not None}


def assert_bitwise(a, b, keys=None):
    for k in (keys or a):
        assert torch.equal(a[k], b[k]), k


def tuple_outputs(res, b, n):
    """Tuple b's outputs; n: its counts per view slot.  Score entries outside its block are never written."""
    out = {}
    for k, v in outputs(res).items():
        if k.startswith('scores_'):
            a, c = (int(x) for x in k[7:].split('_'))
            out[k] = v[b, :n[a] + 1, :n[c] + 1]
        else:
            out[k] = v[b]
    return out


POSE_KEYS = ('T_w8pt', 'T_pair', 'success', 'n_matches', 'extrinsics')


def run_pose(matcher, data, T, **kw):
    res = matcher(data)
    state = matcher._engine.last
    pose = MultiViewPoseEngine().run(state, [data['intr%d' % i] for i in state['view_ids']], **kw)
    return res, pose


def ragged_counts(rng, B, T, cap, lo=32):
    return [[int(rng.integers(lo, cap + 1)) for _ in range(T)] for _ in range(B)]


# 1. uniform counts through the ragged entry: bitwise the existing entry, poses included
def test_uniform_counts_bitwise_equal_existing_entry(mv, pair):
    T, cap, B = 5, 256, 3
    data = scene(11, T, cap, B)
    r0, p0 = run_pose(mv, data, T)
    r1, p1 = run_pose(mv, with_counts(data, [[cap] * T] * B), T)
    assert_bitwise(outputs(r0), outputs(r1))
    assert_bitwise(p0, p1, POSE_KEYS)
    d2 = scene(12, 2, cap, B)
    r0, p0 = run_pose(pair, d2, 2, global_ba=False, rel_pose_method='ransac_ba')
    r1, p1 = run_pose(pair, with_counts(d2, [[cap] * 2] * B), 2, global_ba=False, rel_pose_method='ransac_ba')
    assert_bitwise(outputs(r0), outputs(r1))
    assert_bitwise(p0, p1, ('T_ransac', 'T_pair', 'success', 'n_matches', 'n_inliers'))


# 2. batch independence and permutation
def test_tuple_alone_and_permuted_bitwise(mv):
    T, cap, B = 5, 320, 4
    rng = np.random.default_rng(0)
    counts = ragged_counts(rng, B, T, cap)
    data = with_counts(scene(21, T, cap, B), counts)
    rb, pb = run_pose(mv, data, T)
    rb, pb = [tuple_outputs(rb, b, counts[b]) for b in range(B)], {k: pb[k] for k in POSE_KEYS}
    for b in range(B):
        ra, pa = run_pose(mv, select(data, [b], T), T)
        assert_bitwise(tuple_outputs(ra, 0, counts[b]), rb[b])
        for k in POSE_KEYS:
            assert torch.equal(pa[k][0], pb[k][b]), (b, k)
    perm = [2, 0, 3, 1]
    rp, pp = run_pose(mv, select(data, perm, T), T)
    for i, b in enumerate(perm):
        assert_bitwise(tuple_outputs(rp, i, counts[b]), rb[b])
    for k in POSE_KEYS:
        assert torch.equal(pp[k], pb[k][perm]), k


def check_against_cut(matcher, data, counts, T, pose=True):
    """3. every tuple against the existing batch-of-one call on its tensors cut to the counts."""
    res = matcher(data)
    if pose:
        state = matcher._engine.last
        pr = MultiViewPoseEngine().run(state, [data['intr%d' % i] for i in state['view_ids']])
    split = split_ragged_result(outputs(res), [[c[i] for c in counts] for i in range(T)])
    for b, c in enumerate(counts):
        one = select(data, [b], T, cuts=c)
        for i in range(T):
            del one['counts%d' % i]
        ref = matcher(one)
        ref_np = {k: v.cpu().numpy() for k, v in outputs(ref).items()}
        got_np = {k: v.cpu().numpy() for k, v in split[b].items()}
        assert set(ref_np) == set(got_np)
        for k in ref_np:
            assert ref_np[k].shape == got_np[k].shape, (b, k)
        # the share of stable rows is a statistic of larger problems: a tuple with a handful of keypoints may have none
        compare_matcher_outputs(ref_np, got_np, tau=2e-3, score_tol=(3e-4, 3e-5), min_stable=0.9 if min(c) >= 32 else 0.0)
        if pose:
            state = matcher._engine.last
            p1 = MultiViewPoseEngine().run(state, [one['intr%d' % i] for i in state['view_ids']])
            np.testing.assert_allclose(pr['extrinsics'][b].cpu().numpy(), p1['extrinsics'][0].cpu().numpy(), atol=2e-3)


def test_ragged_agrees_with_per_tuple_call(mv):
    T, cap, B = 5, 384, 4
    counts = ragged_counts(np.random.default_rng(1), B, T, cap, lo=100)
    check_against_cut(mv, with_counts(scene(31, T, cap, B), counts), counts, T)


def test_ragged_agrees_with_oracle(mv):
    """Each tuple of a ragged batch against oracle/matcher_torch on its cut tensors, at the golden tolerances: the
    reference's fp32 run (on the CPU), with the score tolerance set by its distance to a float64 run."""
    from oracle.matcher_torch import matcher_forward
    T, cap, B = 5, 384, 3
    counts = ragged_counts(np.random.default_rng(5), B, T, cap, lo=60)
    data = with_counts(scene(33, T, cap, B), counts)
    split = split_ragged_result(outputs(mv(data)), [[c[i] for c in counts] for i in range(T)])
    sd = make_state_dict(len(MV_LAYERS), seed=3, final_proj_gain=12.0, conf_head='score')
    cfg = {'GNN_layers': MV_LAYERS, 'multi_frame_matching': True}
    for b, c in enumerate(counts):
        one = select(data, [b], T, cuts=c)
        np32 = {k: (v.cpu().numpy() if torch.is_tensor(v) and not v.is_meta else v) for k, v in one.items()
                if not k.startswith('counts')}
        ref = matcher_forward(sd, cfg, np32)
        ref64 = matcher_forward({k: np.asarray(v, dtype=np.float64) for k, v in sd.items()}, cfg,
                                {k: (v.astype(np.float64) if isinstance(v, np.ndarray) else v) for k, v in np32.items()},
                                device='cuda')
        noise = max(float(np.abs(ref[k].astype(np.float64) - ref64[k]).max()) for k in ref if k.startswith('scores_'))
        got = {k: v.cpu().numpy() for k, v in split[b].items()}
        compare_matcher_outputs({k: v for k, v in ref.items() if k in got}, got, tau=2e-3,
                                score_tol=(max(3e-4, 4.0 * noise), 3e-5), min_stable=0.9)


# 4. count edges under one capacity.  The Sinkhorn kernel and its cluster size follow the capacity: 64 / 128 / 256 / 512 /
# 1024 give clusters of 1 / 2 / 4 / 8 / 16 CTAs, 2048 the multi-CTA kernel.  Under each, the (m, n) shapes of the Sinkhorn
# shape suite that fit and the tile and slice edges.
EDGES = [1, 63, 64, 65, 127, 128, 129, 255, 256, 257, 511, 513, 1023, 1024, 1025, 1500, 2047]


@pytest.mark.parametrize('cap', [64, 128, 256, 512, 1024, 2048])
def test_count_edges(pair, cap):
    shapes = sorted({(m, n) for _, m, n, *_ in SINKHORN_SHAPES if m <= cap and n <= cap})
    edges = [e for e in EDGES if e <= cap] + [cap]
    counts = [list(mn) for mn in shapes] + [[edges[i], edges[(3 * i + 1) % len(edges)]] for i in range(len(edges))]
    data = with_counts(scene(41 + cap, 2, cap, len(counts)), counts)
    check_against_cut(pair, data, counts, 2, pose=False)


# 5. the caller's padding never enters; entries past the counts are -1 / 0 / 0
@pytest.mark.parametrize('pad', [float('nan'), 1e30, -1e30])
def test_caller_padding_ignored(mv, pad):
    T, cap, B = 4, 256, 3
    counts = ragged_counts(np.random.default_rng(2), B, T, cap)
    data = scene(51, T, cap, B)
    r0 = outputs(mv(with_counts(data, counts, pad=0.0)))
    r1 = outputs(mv(with_counts(data, counts, pad=pad)))
    for k, v in r0.items():
        if k.startswith('scores_'):
            a, c = (int(x) for x in k[7:].split('_'))
            for b, n in enumerate(counts):
                assert torch.equal(v[b, :n[a] + 1, :n[c] + 1], r1[k][b, :n[a] + 1, :n[c] + 1]), (k, b)
            continue
        assert torch.equal(v, r1[k]), k
        x = int(k[len('matches' if k.startswith('matches') else 'matching_scores' if k.startswith('matching')
                      else 'conf_scores_'):].split('_')[0])
        for b, n in enumerate(counts):
            tail = v[b, n[x]:]
            assert (tail == (-1 if k.startswith('matches') else 0)).all(), (k, b)


def run_abi(mv, data, counts, T, cap, fill):
    """mvm_pack_views_ragged + mvm_matcher_forward_ragged on caller-allocated outputs whose score buffers hold `fill`."""
    B = len(counts)
    lib, dev = _lib.lib(), data['keypoints0'].device
    packed = mv._pack(dev)
    n_pad = (cap + 63) // 64 * 64
    slot = torch.tensor(counts, dtype=torch.int32, device=dev)
    kp = torch.empty(B, T, n_pad, 2, device=dev)
    sc = torch.empty(B, T, n_pad, device=dev)
    de = torch.empty(B, T, 256, n_pad, device=dev)
    ptrs = [(C.c_void_p * T)(*[data[k % i].data_ptr() for i in range(T)])
            for k in ('keypoints%d', 'scores%d', 'descriptors%d')]
    cnt = (C.c_int * T)(*[cap] * T)
    sp = _lib.stream_ptr()
    assert lib.mvm_pack_views_ragged(ptrs[0], ptrs[1], ptrs[2], cnt, _lib.ptr(slot), B, T, n_pad, _lib.ptr(kp),
                                     _lib.ptr(sc), _lib.ptr(de), sp) == 0
    pair_ids = [(a, b) for b in range(T) for a in range(b)]
    pairs = (_lib.PairIO * len(pair_ids))()
    outs = []
    for p, (a, b) in enumerate(pair_ids):
        o = {'matches_a': torch.empty(B, cap, dtype=torch.int64, device=dev),
             'matches_b': torch.empty(B, cap, dtype=torch.int64, device=dev),
             'mscores_a': torch.empty(B, cap, device=dev), 'mscores_b': torch.empty(B, cap, device=dev),
             'scores': torch.full((B, cap + 1, cap + 1), fill, device=dev),
             'conf': torch.empty(B, cap, 1, device=dev)}
        outs.append(o)
        pairs[p].view_a, pairs[p].view_b = a, b
        for k in ('matches_a', 'matches_b', 'mscores_a', 'mscores_b', 'scores', 'conf'):
            setattr(pairs[p], k, o[k].data_ptr())
    nbytes = lib.mvm_matcher_workspace_bytes(B, T, n_pad, len(pair_ids), 1)
    ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
    h, w = data['image0'].shape[-2:]
    wh = (C.c_float * (2 * T))(*[float(w), float(h)] * T)
    assert lib.mvm_matcher_forward_ragged(C.byref(packed.struct), B, T, n_pad, cnt, _lib.ptr(slot), _lib.ptr(kp),
                                          _lib.ptr(sc), _lib.ptr(de), wh, 100, 0.0, pairs, len(pair_ids), _lib.ptr(ws),
                                          nbytes, None, sp) == 0
    torch.cuda.synchronize()
    return dict(zip(pair_ids, outs))


def test_scores_outside_each_block_not_written(mv):
    """Score buffers filled by the caller: every entry outside a tuple's [m_b + 1, n_b + 1] block keeps its sentinel, and
    the outputs are bitwise those of buffers filled with zeros (so nothing outside the blocks is read either)."""
    T, cap, B, sentinel = 3, 192, 3, 12345.5
    counts = ragged_counts(np.random.default_rng(6), B, T, cap)
    data = scene(55, T, cap, B)
    got = run_abi(mv, data, counts, T, cap, sentinel)
    zero = run_abi(mv, data, counts, T, cap, 0.0)
    for (a, c), o in got.items():
        z = o['scores']
        for b, n in enumerate(counts):
            inside = torch.zeros_like(z[b], dtype=torch.bool)
            inside[:n[a] + 1, :n[c] + 1] = True
            assert (z[b][~inside] == sentinel).all(), ((a, c), b)
            assert torch.equal(z[b][inside], zero[(a, c)]['scores'][b][inside]), ((a, c), b)
        for k in ('matches_a', 'matches_b', 'mscores_a', 'mscores_b', 'conf'):
            assert torch.equal(o[k], zero[(a, c)][k]), ((a, c), k)


# 6. a tuple with a zero-count view leaves every other tuple bitwise unchanged
def test_zero_count_view_isolated(mv):
    T, cap, B = 4, 256, 3
    counts = ragged_counts(np.random.default_rng(3), B, T, cap)
    data = scene(61, T, cap, B)
    r0 = mv(with_counts(data, counts))
    r0 = [tuple_outputs(r0, b, counts[b]) for b in range(B)]
    bad = [list(c) for c in counts]
    bad[1][2] = 0
    r1 = mv(with_counts(data, bad))
    for b in (0, 2):
        assert_bitwise(r0[b], tuple_outputs(r1, b, counts[b]))
    # tuple 1 has no keypoints in view 2: every pair with view 2, on either side, has no match and no match score
    for a, c in ((0, 2), (1, 2), (2, 3)):
        for x in (a, c):
            assert (r1['matches%d_%d_%d' % (x, a, c)][1] == -1).all(), (x, a, c)
            assert (r1['matching_scores%d_%d_%d' % (x, a, c)][1] == 0).all(), (x, a, c)


# 7. one CUDA graph of matcher + pose stage serves any device counts at the same capacities
def test_cuda_graph_replay_with_new_counts(mv):
    T, cap, B = 4, 256, 3
    rng = np.random.default_rng(4)
    c0, c1 = ragged_counts(rng, B, T, cap), ragged_counts(rng, B, T, cap)
    data = with_counts(scene(71, T, cap, B), c0)
    pe = MultiViewPoseEngine()

    def step():
        res = mv(data)
        state = mv._engine.last
        return res, pe.run(state, [data['intr%d' % i] for i in state['view_ids']])

    step()
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        step()
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        gres, gpose = step()
    for counts in (c1, c0):
        for i in range(T):
            data['counts%d' % i].copy_(torch.tensor([c[i] for c in counts], dtype=torch.int32))
        g.replay()
        torch.cuda.synchronize()
        eres, epose = step()
        for b in range(B):
            assert_bitwise(tuple_outputs(eres, b, counts[b]), tuple_outputs(gres, b, counts[b]))
        assert_bitwise(epose, gpose, POSE_KEYS)


# 8. MultiViewPipeline on an image batch with ragged SuperPoint counts; eval with --image_batch
def test_pipeline_image_batch_matches_per_tuple():
    from e2e_multi_view_matching_b200.models.superpoint import SuperPoint
    from e2e_multi_view_matching_b200.pipeline import MultiViewPipeline
    from e2e_multi_view_matching_b200.synthetic import make_superpoint_state_dict, render_tuple_images
    # threshold 0.65 leaves 300-400 keypoints per rendered image with these weights: every view's count differs
    sp = SuperPoint({'max_keypoints': 512, 'keypoint_threshold': 0.65, 'nms_radius': 4, 'remove_borders': 4}).eval()
    sp.load_state_dict({k: torch.from_numpy(v) for k, v in make_superpoint_state_dict(0).items()})
    pipe = MultiViewPipeline(make_matcher(MV_LAYERS), superpoint=sp.cuda())
    T, B = 5, 4
    parts = [render_tuple_images(make_scene_tuple_inputs(300 + i, T, 512, batch=1, noise_px=0.0), seed=300 + i)
             for i in range(B)]
    data = {k: (torch.from_numpy(np.concatenate([p[k] for p in parts])).cuda() if isinstance(v, np.ndarray) else v)
            for k, v in parts[0].items() if not k.startswith(('keypoints', 'scores', 'descriptors'))}
    with pytest.raises(ValueError, match='run_tuples'):
        pipe(data)
    out = pipe.run_tuples(data)
    assert len(out) == B
    results, poses = [r for r, _ in out], [p for _, p in out]
    assert len({tuple(results[b]['keypoints%d' % i].shape) for b in range(B) for i in range(T)}) > 1
    for b in range(B):
        one = {k: (v[b:b + 1] if torch.is_tensor(v) else v) for k, v in data.items()}
        r1, p1 = pipe(one)
        for i in range(T):
            assert torch.equal(r1['keypoints%d' % i], results[b]['keypoints%d' % i])
        ref = {k: v.cpu().numpy() for k, v in outputs(r1).items()}
        got = {k: v.cpu().numpy() for k, v in outputs(results[b]).items()}
        # rendered scenes with seeded weights leave many near-tied rows: matches are compared on the stable ones only
        compare_matcher_outputs(ref, got, tau=2e-3, score_tol=(3e-4, 3e-5), min_stable=0.0)
        np.testing.assert_allclose(poses[b]['extrinsics'][0].cpu().numpy(), p1['extrinsics'][0].cpu().numpy(),
                                   atol=2e-3)


def test_eval_image_batch_auc_matches_batch_of_one():
    from e2e_multi_view_matching_b200.eval_multi_view import main
    args = ['--images', '--n_tuples', '8', '--max_keypoints', '512', '--keypoint_threshold', '0.65']
    a = main(args + ['--image_batch', '1'])
    b = main(args + ['--image_batch', '4'])
    assert max(a.values()) >= 5.0, a          # the comparison says nothing when every AUC is near 0
    for k in a:
        assert abs(a[k] - b[k]) <= 0.5, (k, a[k], b[k])
