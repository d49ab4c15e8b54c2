"""SuperGlue with the upstream/reference forward(data) contract (models/models/superglue.py:179-285):
keys keypoints0/1, scores0/1, descriptors0/1, image0/1 -> matches0/1, matching_scores0/1 with
match_threshold (default 0.2).  Same state-dict keys as upstream (kenc, gnn, final_proj,
bin_score); computes in libmvm_b200.so through the same engine as MultiViewMatcher."""
import torch
from torch import nn

from .. import _lib
from ..packing import PackedMatcher
from .multi_view_matcher import KeypointEncoder, AttentionalGNN, MatcherEngine, image_wh, slot_counts_of


class SuperGlue(nn.Module):
    default_config = {
        'descriptor_dim': 256,
        'weights': 'indoor',
        'keypoint_encoder': [32, 64, 128, 256],
        'GNN_layers': ['self', 'cross'] * 9,
        'sinkhorn_iterations': 100,
        'match_threshold': 0.2,
    }

    def __init__(self, config):
        super().__init__()
        self.config = {**self.default_config, **config}
        d = self.config['descriptor_dim']
        self.kenc = KeypointEncoder(d, list(self.config['keypoint_encoder']))
        self.gnn = AttentionalGNN(d, self.config['GNN_layers'])
        self.final_proj = nn.Conv1d(d, d, kernel_size=1, bias=True)
        self.register_parameter('bin_score', torch.nn.Parameter(torch.tensor(1.)))
        # The reference unconditionally loads weights/superglue_<indoor|outdoor>.pth
        # (superglue.py:223-226); that file is an external download, so a path may be given
        # via config['weights_path'], otherwise the caller load_state_dict()s.
        path = self.config.get('weights_path')
        if path is not None:
            self.load_state_dict(torch.load(str(path), map_location='cpu'))
        self._engine = MatcherEngine()
        self._packed = None
        self._packed_key = None

    def _pack(self, device):
        key = (str(device),) + tuple((p.data_ptr(), p._version) for p in self.parameters()) + \
            tuple((b.data_ptr(), b._version) for b in self.buffers())
        if self._packed is None or key != self._packed_key:
            self._packed = PackedMatcher(self.state_dict(), self.config['GNN_layers'],
                                         conf_mlp=False, device=device)
            self._packed_key = key
        return self._packed

    def forward(self, data):
        kpts0, kpts1 = data['keypoints0'], data['keypoints1']
        if kpts0.shape[1] == 0 or kpts1.shape[1] == 0:  # no keypoints (superglue.py:235-242)
            shape0, shape1 = kpts0.shape[:-1], kpts1.shape[:-1]
            return {
                'matches0': kpts0.new_full(shape0, -1, dtype=torch.int),
                'matches1': kpts1.new_full(shape1, -1, dtype=torch.int),
                'matching_scores0': kpts0.new_zeros(shape0),
                'matching_scores1': kpts1.new_zeros(shape1),
            }
        if kpts0.device.type != 'cuda':
            raise _lib.MvmError('SuperGlue needs CUDA tensors (no CPU fallback)')
        packed = self._pack(kpts0.device)
        views = [(data['keypoints%d' % i].float(), data['scores%d' % i].float(),
                  data['descriptors%d' % i].float()) for i in (0, 1)]
        with torch.no_grad():
            # each view normalised by its own image (superglue.py:245-246)
            o = self._engine.run(packed, views, [image_wh(data, 0), image_wh(data, 1)], [(0, 1)],
                                 self.config['sinkhorn_iterations'], self.config['match_threshold'],
                                 slot_counts_of(data, [0, 1]))[(0, 1)]
        return {
            'matches0': o['matches_a'],
            'matches1': o['matches_b'],
            'matching_scores0': o['mscores_a'],
            'matching_scores1': o['mscores_b'],
        }
