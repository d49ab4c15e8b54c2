"""run_super_point (helpers.py:83-96) and the image-in routing of train_step, validation_step and MultiViewPipeline,
without a GPU: the SuperPoint front-end is a stub with SuperPoint's interface (forward / forward_batch / config), and
tensors stay on the CPU.  The reshaping and key naming are checked against the reference's own helpers.run_super_point
where the reference sources can be imported (oracle/ref_shim.py)."""
import importlib
import os
import types

import numpy as np
import pytest
import torch

T_VIEWS, H, W, K = 3, 24, 32, 5


class StubSuperPoint:
    """SuperPoint's interface on the CPU.  Image i of a call gets keypoints / scores / descriptors derived from the
    image's first pixel, so results can be traced back to the image they came from; `short` images get fewer than
    max_keypoints keypoints from forward (and a smaller count from forward_batch)."""

    def __init__(self, max_keypoints=K, fill=False, short=()):
        self.config = {'max_keypoints': max_keypoints, 'fill_with_random_keypoints': fill}
        self.short = set(short)
        self.calls = []

    def _one(self, img):
        tag = float(img.reshape(-1)[0])
        n = K - 2 if int(tag) in self.short else K
        kp = torch.arange(2 * n, dtype=torch.float32).reshape(n, 2) + tag
        return kp, torch.full((n,), tag), torch.full((256, n), tag)

    def __call__(self, data):
        self.calls.append(('forward', [tuple(b.shape) for b in data['image']]))
        out = {'keypoints': [], 'scores': [], 'descriptors': []}
        for batch in data['image']:
            for img in batch:
                for k, v in zip(out, self._one(img)):
                    out[k].append(v)
        return out

    def forward_batch(self, images):
        self.calls.append(('forward_batch', tuple(images.shape)))
        kp, sc, de, counts = [], [], [], []
        for img in images:
            a, b, c = self._one(img)
            n = a.shape[0]
            counts.append(K if self.config['fill_with_random_keypoints'] else n)
            kp.append(torch.cat([a, torch.zeros(K - n, 2)]))
            sc.append(torch.cat([b, torch.zeros(K - n)]))
            de.append(torch.cat([c, torch.zeros(256, K - n)], 1))
        return {'keypoints': torch.stack(kp), 'scores': torch.stack(sc), 'descriptors': torch.stack(de),
                'counts': torch.tensor(counts, dtype=torch.int32)}


def _images(batch):
    """image{m} [batch,1,H,W] whose first pixel is the image's running number m * batch + b."""
    data = {'ids': list(range(T_VIEWS))}
    for m in range(T_VIEWS):
        img = torch.rand(batch, 1, H, W)
        img[:, 0, 0, 0] = torch.arange(batch, dtype=torch.float32) + m * batch
        data['image%d' % m] = img
    return data


@pytest.fixture
def on_cpu(monkeypatch):
    """The reference and run_super_point move the images with .cuda(): keep them where they are."""
    monkeypatch.setattr(torch.Tensor, 'cuda', lambda self, *a, **k: self)


def _reference_helpers():
    from oracle import ref_shim
    if not os.path.isdir(ref_shim.REF):
        pytest.skip('the reference sources are not available')
    ref_shim.load()
    try:
        return importlib.import_module('helpers')
    except ImportError as e:
        pytest.skip('the reference helpers do not import here: %s' % e)


def _same(a, b):
    assert sorted(a) == sorted(b)
    for k in a:
        if torch.is_tensor(a[k]):
            assert a[k].shape == b[k].shape and torch.equal(a[k], b[k]), k
        else:
            assert a[k] == b[k], k


@pytest.mark.parametrize('batch', [1, 3])
@pytest.mark.parametrize('merge', [True, False])
def test_run_super_point_matches_reference_helpers(on_cpu, batch, merge):
    from e2e_multi_view_matching_b200.training import run_super_point
    helpers = _reference_helpers()
    opt = types.SimpleNamespace(batch_size=batch)
    ours, ref = _images(batch), _images(batch)
    for m in range(T_VIEWS):
        ref['image%d' % m] = ours['image%d' % m].clone()
    run_super_point(opt, ours, StubSuperPoint(fill=True), merge=merge)
    helpers.run_super_point(opt, ref, StubSuperPoint(fill=True), merge=merge)
    _same(ours, ref)


@pytest.mark.parametrize('batch', [1, 3])
def test_run_super_point_layout(on_cpu, batch):
    """keypoints{m} [B,K,2], scores{m} [B,K], descriptors{m} [B,256,K] of image b of view m, from one forward_batch
    over the T*B merged images; no other key is added."""
    from e2e_multi_view_matching_b200.training import run_super_point
    data = _images(batch)
    sp = StubSuperPoint(fill=True)
    run_super_point(types.SimpleNamespace(batch_size=batch), data, sp)
    assert sp.calls == [('forward_batch', (T_VIEWS * batch, 1, H, W))]
    assert sorted(data) == sorted(['ids'] + ['%s%d' % (k, m) for k in ('image', 'keypoints', 'scores', 'descriptors')
                                             for m in range(T_VIEWS)])
    for m in range(T_VIEWS):
        assert data['keypoints%d' % m].shape == (batch, K, 2)
        assert data['scores%d' % m].shape == (batch, K)
        assert data['descriptors%d' % m].shape == (batch, 256, K)
        assert data['scores%d' % m][:, 0].tolist() == [float(m * batch + b) for b in range(batch)]


def test_run_super_point_routing(on_cpu):
    from e2e_multi_view_matching_b200.training import run_super_point
    opt = types.SimpleNamespace(batch_size=1)
    # every image reaches max_keypoints without fill: the batched path
    sp = StubSuperPoint()
    run_super_point(opt, _images(1), sp)
    assert [c[0] for c in sp.calls] == ['forward_batch']
    # an image short of max_keypoints without fill: still one batched call (one dense pass); each image's valid
    # entries become the per-image lists forward gives, batch size 1 -> per-image tensors with a leading 1
    sp = StubSuperPoint(short={1})
    data = _images(1)
    run_super_point(opt, data, sp)
    assert [c[0] for c in sp.calls] == ['forward_batch']
    assert data['keypoints1'].shape == (1, K - 2, 2) and data['keypoints0'].shape == (1, K, 2)
    assert data['descriptors1'].shape == (1, 256, K - 2) and data['descriptors1'].is_contiguous()
    lists = _images(1)
    run_super_point(opt, lists, StubSuperPoint(short={1}), merge=False)
    for k in ('keypoints', 'scores', 'descriptors'):
        for m in range(T_VIEWS):
            assert torch.equal(data[k + str(m)], lists[k + str(m)]), (k, m)
    # merge=False, max_keypoints = -1 and max_keypoints above the score map's pixel count never take the batched path
    for kw, mk in (({'merge': False}, K), ({}, -1), ({}, H * W + 1)):
        sp = StubSuperPoint(max_keypoints=mk)
        run_super_point(opt, _images(1), sp, **kw)
        assert [c[0] for c in sp.calls] == ['forward']


def _training_case():
    from oracle.make_train_backward_golden import build, CASES
    case = CASES[0]
    data_np, sd = build(case)
    return case, data_np, sd


class _FrontEndFromData(StubSuperPoint):
    """forward_batch hands back the keypoints / scores / descriptors of a keypoint-in batch, view-major as
    run_super_point merges the images."""

    def __init__(self, data):
        super().__init__(max_keypoints=data['keypoints0'].shape[1], fill=True)
        self.data = data

    def forward_batch(self, images):
        self.calls.append(('forward_batch', tuple(images.shape)))
        n = len(self.data['ids'])
        out = {k: torch.cat([self.data[k + str(m)] for m in range(n)]) for k in ('keypoints', 'scores', 'descriptors')}
        out['counts'] = torch.full((images.shape[0],), self.config['max_keypoints'], dtype=torch.int32)
        return out


def test_train_step_routes_images_through_super_point(monkeypatch, on_cpu):
    """train_step on a batch with images and no keypoints == train_step on the batch with the front-end's keypoints
    (loss and every gradient, bitwise), with the matcher's stages on the float64 stand-ins; a batch that has
    keypoints never calls the front-end."""
    from tests import emul_ops
    from tests.test_train_host_logic import PATCHED, match_loss
    from e2e_multi_view_matching_b200 import ops, _lib, training
    from e2e_multi_view_matching_b200.models.multi_view_matcher import MultiViewMatcher
    for f in PATCHED:
        monkeypatch.setattr(ops, f, getattr(emul_ops, f))
    monkeypatch.setattr(_lib, 'require_cuda', lambda device, what: None)
    monkeypatch.setattr(training, 'compute_match_loss', match_loss)
    case, data_np, sd = _training_case()
    full = {k: (torch.from_numpy(v) if isinstance(v, np.ndarray) else v) for k, v in data_np.items()}
    opt = types.SimpleNamespace(pose_loss=False, batch_size=case['batch'])

    def step(data, sp):
        model = MultiViewMatcher({'multi_frame_matching': True, 'GNN_layers': case['layers'], 'conf_mlp': False,
                                  'full_output': False})
        model.load_state_dict({k: torch.from_numpy(np.asarray(v)) for k, v in sd.items() if not k.startswith('conf_mlp')})
        model.train()
        optimizer = torch.optim.SGD(model.parameters(), lr=1e-3)
        loss, _ = training.train_step(opt, data, model, optimizer, n_pairs=3, super_point=sp)
        return loss, [p.detach().clone() for p in model.parameters()]

    sp_unused = _FrontEndFromData(full)
    loss_kp, params_kp = step(dict(full), sp_unused)
    assert sp_unused.calls == []
    image_in = {k: v for k, v in full.items() if not k.startswith(('keypoints', 'scores', 'descriptors'))}
    sp = _FrontEndFromData(full)
    loss_img, params_img = step(dict(image_in), sp)
    assert [c[0] for c in sp.calls] == ['forward_batch']
    assert torch.equal(loss_kp, loss_img)
    assert all(torch.equal(a, b) for a, b in zip(params_kp, params_img))
    with pytest.raises(ValueError):
        step(dict(image_in), None)


def test_validation_step_routes_images_through_super_point(monkeypatch, on_cpu):
    from e2e_multi_view_matching_b200 import training
    seen = []

    def fake_run_matcher(opt, data, matcher):
        seen.append(sorted(data))
        z = data['keypoints0'].sum().reshape(1)
        return {'match_loss': z, 'rot_loss': z * 0, 'transl_loss': z * 0}, {}

    monkeypatch.setattr(training, 'run_matcher', fake_run_matcher)
    case, data_np, _ = _training_case()
    full = {k: (torch.from_numpy(v) if isinstance(v, np.ndarray) else v) for k, v in data_np.items()}
    opt = types.SimpleNamespace(pose_loss=False, batch_size=case['batch'], rot_weight=0.0, trans_weight=0.0)
    sp = _FrontEndFromData(full)
    v_kp, _ = training.validation_step(opt, dict(full), None, 3, 0.0, super_point=sp)
    assert sp.calls == []
    image_in = {k: v for k, v in full.items() if not k.startswith(('keypoints', 'scores', 'descriptors'))}
    v_img, _ = training.validation_step(opt, dict(image_in), None, 3, 0.0, super_point=sp)
    assert [c[0] for c in sp.calls] == ['forward_batch']
    assert seen[0] == seen[1] and torch.equal(v_kp, v_img)
    with pytest.raises(ValueError):
        training.validation_step(opt, dict(image_in), None, 3, 0.0)


def test_multi_view_pipeline_routes_images_through_super_point(on_cpu):
    from e2e_multi_view_matching_b200.pipeline import MultiViewPipeline
    seen = []

    class FakeMatcher:
        config = {'multi_frame_matching': True, 'conf_mlp': True}
        _engine = types.SimpleNamespace(last=None)

        def __call__(self, data):
            seen.append(dict(data))
            return {'scores_0_1': torch.zeros(1)}

    data = _images(2)
    sp = StubSuperPoint(fill=True)
    result, pose = MultiViewPipeline(FakeMatcher(), superpoint=sp)(data)
    assert pose is None and [c[0] for c in sp.calls] == ['forward_batch']
    assert 'keypoints0' not in data                                     # the caller's dict is left as it is
    for m in range(T_VIEWS):
        for k in ('keypoints', 'scores', 'descriptors'):
            assert torch.equal(result[k + str(m)], seen[0][k + str(m)])
    # keypoints given: the front-end is not run, the matcher gets the caller's tensors
    sp2 = StubSuperPoint(fill=True)
    MultiViewPipeline(FakeMatcher(), superpoint=sp2)(seen[0])
    assert sp2.calls == [] and all(seen[1][k] is seen[0][k] for k in seen[0])
    # views of different sizes run one batch per view
    data = _images(1)
    data['image2'] = torch.rand(1, 1, H + 8, W)
    data['image2'][0, 0, 0, 0] = 2.0
    sp3 = StubSuperPoint(fill=True)
    MultiViewPipeline(FakeMatcher(), superpoint=sp3)(data)
    assert [c[0] for c in sp3.calls] == ['forward']
    with pytest.raises(ValueError):
        MultiViewPipeline(FakeMatcher())(_images(1))
