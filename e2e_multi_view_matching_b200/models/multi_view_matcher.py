"""MultiViewMatcher with the reference's constructor, config keys, state-dict keys and
forward(data) -> dict contract (models/models/multi_view_matcher.py:103-332), computing in
libmvm_b200.so.  The nn.Modules below exist only to own parameters/buffers under the
reference's key names (load_state_dict / DataParallel / checkpoints keep working); forward
never runs them -- it repacks the weights (packing.py) and makes one C-ABI call per tuple
batch (mvm_matcher_forward).  Eval mode only: the training branch is SURVEY.md §8 f-2.
"""
import ctypes as C

import torch
from torch import nn

from .. import _lib
from ..packing import PackedMatcher


def MLP(channels, do_bn=True, last_layer=True):
    """Parameter container with the reference's Sequential indices (multi_view_matcher.py:8-22)."""
    n = len(channels)
    layers = []
    for i in range(1, n):
        layers.append(nn.Conv1d(channels[i - 1], channels[i], kernel_size=1, bias=True))
        if i < (n - 1 if last_layer else n):
            if do_bn:
                layers.append(nn.BatchNorm1d(channels[i]))
            layers.append(nn.ReLU())
    return nn.Sequential(*layers)


class KeypointEncoder(nn.Module):
    def __init__(self, feature_dim, layers):
        super().__init__()
        self.encoder = MLP([3] + layers + [feature_dim])
        nn.init.constant_(self.encoder[-1].bias, 0.0)


class MultiHeadedAttention(nn.Module):
    def __init__(self, num_heads, d_model):
        super().__init__()
        self.merge = nn.Conv1d(d_model, d_model, kernel_size=1)
        self.proj = nn.ModuleList([nn.Conv1d(d_model, d_model, kernel_size=1) for _ in range(3)])


class AttentionalPropagation(nn.Module):
    def __init__(self, feature_dim, num_heads):
        super().__init__()
        self.attn = MultiHeadedAttention(num_heads, feature_dim)
        self.mlp = MLP([feature_dim * 2, feature_dim * 2, feature_dim])
        nn.init.constant_(self.mlp[-1].bias, 0.0)


class AttentionalGNN(nn.Module):
    def __init__(self, feature_dim, layer_names):
        super().__init__()
        self.layers = nn.ModuleList([AttentionalPropagation(feature_dim, 4) for _ in layer_names])
        self.names = layer_names


class ConfidenceMLP(nn.Module):
    def __init__(self, feature_dim, in_dim, out_dim=1):
        super().__init__()
        self.layers_f = MLP([feature_dim * 2, feature_dim * 2, feature_dim], last_layer=False)
        self.layers_c = MLP([in_dim, feature_dim, feature_dim], last_layer=False)
        self.layers = MLP([feature_dim, out_dim])
        nn.init.constant_(self.layers[-1].bias, 0.0)


def _round_up(x, m):
    return (x + m - 1) // m * m


def image_wh(data, i):
    """(width, height) of data['image{i}'], the size normalize_keypoints divides by (superglue.py:65-72)."""
    h, w = data['image' + str(i)].shape[-2:]
    return w, h


class MatcherEngine:
    """Shape-keyed workspaces + the C-ABI call.  Shared by MultiViewMatcher and SuperGlue."""

    def __init__(self):
        self._ws = {}
        self.last = None

    def workspace(self, nbytes, device):
        key = str(device)
        buf = self._ws.get(key)
        if buf is None or buf.numel() < nbytes:
            buf = torch.empty(nbytes, dtype=torch.uint8, device=device)
            self._ws[key] = buf
        return buf

    def run(self, packed, views, view_wh, pair_ids, sinkhorn_iters, match_threshold):
        """views: list (per view slot) of (kpts [B,n,2], scores [B,n], desc [B,256,n]) CUDA tensors; view_wh: list (per
        view slot) of the (width, height) its keypoints are normalised by.
        Returns {pair: dict of output tensors} following the reference's shapes/dtypes."""
        lib = _lib.lib()
        T = len(views)
        assert len(view_wh) == T
        B = views[0][0].shape[0]
        dev = views[0][0].device
        counts = [int(v[0].shape[1]) for v in views]
        n_pad = max(64, _round_up(max(counts), 64))
        kp = torch.empty(B, T, n_pad, 2, dtype=torch.float32, device=dev)
        sc = torch.empty(B, T, n_pad, dtype=torch.float32, device=dev)
        de = torch.empty(B, T, 256, n_pad, dtype=torch.float32, device=dev)
        # one pack launch (zero padding included) instead of three fills + three strided copies per view
        views = [tuple(x.contiguous() for x in v) for v in views]
        for k, s, d in views:
            assert k.dtype == s.dtype == d.dtype == torch.float32 and d.shape[1] == 256
        ptrs = [(C.c_void_p * T)(*[v[i].data_ptr() for v in views]) for i in range(3)]
        cnt_pack = (C.c_int * T)(*counts)
        with torch.cuda.device(dev):
            _lib.check(lib.mvm_pack_views(ptrs[0], ptrs[1], ptrs[2], cnt_pack, B, T, n_pad, _lib.ptr(kp), _lib.ptr(sc),
                                          _lib.ptr(de), _lib.stream_ptr()), 'mvm_pack_views')
        n_pairs = len(pair_ids)
        pairs = (_lib.PairIO * n_pairs)()
        outs = {}
        for p, (a, b) in enumerate(pair_ids):
            m, n = counts[a], counts[b]
            o = {
                'matches_a': torch.empty(B, m, dtype=torch.int64, device=dev),
                'matches_b': torch.empty(B, n, dtype=torch.int64, device=dev),
                'mscores_a': torch.empty(B, m, dtype=torch.float32, device=dev),
                'mscores_b': torch.empty(B, n, dtype=torch.float32, device=dev),
                'scores': torch.empty(B, m + 1, n + 1, dtype=torch.float32, device=dev),
                'conf': (torch.empty(B, m, 1, dtype=torch.float32, device=dev)
                         if packed.has_conf else None),
            }
            outs[(a, b)] = o
            pairs[p].view_a, pairs[p].view_b = a, b
            pairs[p].matches_a = o['matches_a'].data_ptr()
            pairs[p].matches_b = o['matches_b'].data_ptr()
            pairs[p].mscores_a = o['mscores_a'].data_ptr()
            pairs[p].mscores_b = o['mscores_b'].data_ptr()
            pairs[p].scores = o['scores'].data_ptr()
            pairs[p].conf = o['conf'].data_ptr() if o['conf'] is not None else None
        nbytes = lib.mvm_matcher_workspace_bytes(B, T, n_pad, n_pairs, int(packed.has_conf))
        ws = self.workspace(nbytes, dev)
        cnt = (C.c_int * T)(*counts)
        wh = [(float(w), float(h)) for w, h in view_wh]
        with torch.cuda.device(dev):
            if len(set(wh)) == 1:
                # one image size for every view: the plain entry point (the same arithmetic, bit for bit)
                rc = lib.mvm_matcher_forward(
                    C.byref(packed.struct), B, T, n_pad, cnt, _lib.ptr(kp), _lib.ptr(sc), _lib.ptr(de),
                    wh[0][0], wh[0][1], int(sinkhorn_iters), float(match_threshold),
                    pairs, n_pairs, _lib.ptr(ws), nbytes, _lib.stream_ptr())
            else:
                table = (C.c_float * (2 * T))(*[x for pair in wh for x in pair])
                rc = lib.mvm_matcher_forward_views(
                    C.byref(packed.struct), B, T, n_pad, cnt, _lib.ptr(kp), _lib.ptr(sc), _lib.ptr(de),
                    table, int(sinkhorn_iters), float(match_threshold),
                    pairs, n_pairs, _lib.ptr(ws), nbytes, None, _lib.stream_ptr())
        _lib.check(rc, 'mvm_matcher_forward')
        # device-resident state the pose stage continues from (no host round trip)
        self.last = {'kpts': kp, 'counts': counts, 'n_pad': n_pad, 'pairs': pairs, 'pair_ids': list(pair_ids),
                     'outs': outs, 'batch': B, 'n_views': T}
        return outs


class MultiViewMatcher(nn.Module):
    """Multi-view feature matcher (drop-in for models/models/multi_view_matcher.py:103)."""
    default_config = {
        'descriptor_dim': 256,
        'weights': 'none',
        'keypoint_encoder': [32, 64, 128, 256],
        'GNN_layers': ['self', 'cross'] * 9,
        'sinkhorn_iterations': 100,
        'multi_frame_matching': True,
        'full_output': False,
        'conf_mlp': True,
        # not a reference key: in train mode with full_output, conf_scores_* carry a graph into the confidence head and
        # the matcher (training.run_matcher sets it with pose_loss); the eval path does not read it
        'conf_grad': False,
    }

    def __init__(self, config):
        super().__init__()
        self.config = {**self.default_config, **config}
        d = self.config['descriptor_dim']
        assert d == 256 and list(self.config['keypoint_encoder']) == [32, 64, 128, 256], \
            'libmvm_b200 kernels are specialised for descriptor_dim 256 / encoder [32,64,128,256]'
        self.kenc = KeypointEncoder(d, list(self.config['keypoint_encoder']))
        self.gnn = AttentionalGNN(d, self.config['GNN_layers'])
        self.final_proj = nn.Conv1d(d, d, kernel_size=1, bias=True)
        self.register_parameter('bin_score', torch.nn.Parameter(torch.tensor(1.)))
        assert self.config['weights'] in ['indoor', 'outdoor', 'none']
        if self.config['weights'] != 'none':
            raise FileNotFoundError('pretrained superglue_%s.pth is an external download that is '
                                    'not available offline; load a checkpoint with '
                                    'load_state_dict instead' % self.config['weights'])
        if self.config['conf_mlp']:
            self.conf_mlp = ConfidenceMLP(d, 1)
        self._engine = MatcherEngine()
        self._packed = None
        self._packed_key = None
        self.match_threshold = 0.0   # multi_view_matcher.py:297

    # ---- weight repacking (cached; invalidated when parameters change) ----
    def _pack(self, device):
        key = (str(device),) + tuple((p.data_ptr(), p._version) for p in self.parameters()) + \
            tuple((b.data_ptr(), b._version) for b in self.buffers())
        if self._packed is None or key != self._packed_key:
            # 'fold_merge' is not a reference key: False keeps attn.merge as its own GEMM (A/B of the offline fold)
            self._packed = PackedMatcher(self.state_dict(), self.config['GNN_layers'],
                                         conf_mlp=self.config['conf_mlp'], device=device,
                                         fold_merge=self.config.get('fold_merge', True))
            self._packed_key = key
        return self._packed

    @staticmethod
    def _empty_pair(result, kpts0, kpts1, id0, id1):
        shape0, shape1 = kpts0.shape[:-1], kpts1.shape[:-1]
        result['matches{}_{}_{}'.format(id0, id0, id1)] = kpts0.new_full(shape0, -1, dtype=torch.int)
        result['matches{}_{}_{}'.format(id1, id0, id1)] = kpts1.new_full(shape1, -1, dtype=torch.int)
        result['matching_scores{}_{}_{}'.format(id0, id0, id1)] = kpts0.new_zeros(shape0)
        result['matching_scores{}_{}_{}'.format(id1, id0, id1)] = kpts1.new_zeros(shape1)

    def _publish(self, result, outs, ids_map):
        for (a, b), o in outs.items():
            id0, id1 = ids_map[a], ids_map[b]
            result['matches{}_{}_{}'.format(id0, id0, id1)] = o['matches_a']
            result['matches{}_{}_{}'.format(id1, id0, id1)] = o['matches_b']
            result['matching_scores{}_{}_{}'.format(id0, id0, id1)] = o['mscores_a']
            result['matching_scores{}_{}_{}'.format(id1, id0, id1)] = o['mscores_b']
            result['scores_{}_{}'.format(id0, id1)] = o['scores']
            result['conf_scores_{}_{}'.format(id0, id1)] = o['conf']

    def _view(self, data, i):
        return (data['keypoints' + str(i)].float(), data['scores' + str(i)].float(),
                data['descriptors' + str(i)].float())

    def forward(self, data):
        if self.training:
            # batch-statistics BatchNorm cannot be folded into the packed weights: the train branch sequences the stage
            # kernels (models/train_forward.py); with autograd enabled the `scores_*` outputs carry the graph of
            # MatcherTrainFn, so loss.backward() fills the parameters' .grad like the reference's autograd does.
            from .train_forward import train_forward
            if self.config['multi_frame_matching']:
                return train_forward(self, data)
            result = {}
            for id1 in range(len(data['ids'])):
                for id0 in range(id1):
                    result.update(train_forward(self, data, view_ids=[id0, id1]))
            return result
        tuple_size = len(data['ids'])
        dev = data['keypoints0'].device
        if dev.type != 'cuda':
            raise _lib.MvmError('MultiViewMatcher needs CUDA tensors (no CPU fallback)')
        packed = self._pack(dev)
        result = {}
        iters = self.config['sinkhorn_iterations']
        self._engine.last = None        # the pose stage must never continue from a previous call's state
        with torch.no_grad():
            if not self.config['multi_frame_matching']:
                # pairwise `match` for every id0 < id1 (multi_view_matcher.py:325-329)
                for id1 in range(tuple_size):
                    for id0 in range(id1):
                        k0, k1 = data['keypoints' + str(id0)], data['keypoints' + str(id1)]
                        if k0.shape[1] == 0 or k1.shape[1] == 0:
                            self._empty_pair(result, k0, k1, id0, id1)
                            continue
                        # each view normalised by its own image (multi_view_matcher.py:165-166)
                        outs = self._engine.run(packed, [self._view(data, id0), self._view(data, id1)],
                                                [image_wh(data, id0), image_wh(data, id1)], [(0, 1)], iters,
                                                self.match_threshold)
                        self._engine.last['view_ids'] = [id0, id1]
                        self._publish(result, outs, {0: id0, 1: id1})
                return result
            # multi_match (multi_view_matcher.py:217-320), eval branch
            with_kpts = [i for i in range(tuple_size) if data['keypoints' + str(i)].shape[1] > 0]
            for id1 in range(tuple_size):
                for id0 in range(id1):
                    if id0 not in with_kpts or id1 not in with_kpts:
                        self._empty_pair(result, data['keypoints' + str(id0)],
                                         data['keypoints' + str(id1)], id0, id1)
            if len(with_kpts) >= 2:
                wh = image_wh(data, 0)   # "assume all images have the same size" (:264)
                slot = {i: s for s, i in enumerate(with_kpts)}
                pair_ids = [(slot[i0], slot[i1]) for i1 in with_kpts for i0 in with_kpts if i0 < i1]
                outs = self._engine.run(packed, [self._view(data, i) for i in with_kpts], [wh] * len(with_kpts),
                                        pair_ids, iters, self.match_threshold)
                self._engine.last['view_ids'] = list(with_kpts)     # slot -> view id of the caller's data dict
                self._publish(result, outs, {s: i for i, s in slot.items()})
        return result
