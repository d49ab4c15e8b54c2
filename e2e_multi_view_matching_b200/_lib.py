"""ctypes binding of libmvm_b200.so (C ABI declared in include/mvm_b200.h).

There is no CPU fallback: if the shared library is missing or a call returns a non-zero
status this module raises.  Build it with ``python -m e2e_multi_view_matching_b200.build``
(nvcc, sm_90a) -- __graft_entry__.build() does that.
"""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, 'libmvm_b200.so')

MVM_MAX_LAYERS = 64
MVM_MAX_VIEWS = 8
MVM_SUPERPOINT_MAX_SELECT = 16384
MVM_CONF_MAX_PAIRS = 28

_fp = C.c_void_p  # device pointers travel as integers


class LayerWeights(C.Structure):
    _fields_ = [('w_qkv', _fp), ('b_qkv', _fp), ('w_merge', _fp), ('b_merge', _fp),
                ('w_mlp0', _fp), ('b_mlp0', _fp), ('w_mlp1', _fp), ('b_mlp1', _fp),
                ('is_cross', C.c_int)]


class MatcherWeights(C.Structure):
    _fields_ = [('n_layers', C.c_int), ('hi_offset', C.c_longlong), ('lo_offset', C.c_longlong),
                ('kenc_w', _fp * 5), ('kenc_b', _fp * 5),
                ('layers', LayerWeights * MVM_MAX_LAYERS),
                ('w_final', _fp), ('b_final', _fp),
                ('bin_score', C.c_float),
                ('has_conf', C.c_int),
                ('conf_wf0', _fp), ('conf_bf0', _fp),
                ('conf_wf1', _fp), ('conf_bf1', _fp),
                ('conf_wc0', _fp), ('conf_bc0', _fp),
                ('conf_wc1', _fp), ('conf_bc1', _fp),
                ('conf_wl', _fp), ('conf_bl', C.c_float),
                ('flat_base', _fp), ('w16_hi', _fp), ('w16_lo', _fp), ('w16_scale', C.c_float)]


class PairIO(C.Structure):
    _fields_ = [('view_a', C.c_int), ('view_b', C.c_int),
                ('matches_a', _fp), ('matches_b', _fp),
                ('mscores_a', _fp), ('mscores_b', _fp),
                ('scores', _fp), ('conf', _fp)]


class MatcherOptions(C.Structure):
    _fields_ = [('math_mode', C.c_int), ('score_kernel', C.c_int), ('gemm_tile', C.c_int), ('gemm_kernel', C.c_int),
                ('sinkhorn_variant', C.c_int), ('attention_split', C.c_int), ('gemm_split', C.c_int)]


class SuperPointWeights(C.Structure):
    _fields_ = [('w', _fp * 10), ('b', _fp * 10), ('w_pb', _fp), ('b_pb', _fp), ('w_db', _fp), ('b_db', _fp)]


class MvmError(RuntimeError):
    pass


_STATUS = {1: 'invalid argument', 2: 'kernel launch failure', 3: 'workspace too small'}
_lib = None


def lib():
    """Load the shared library once; fail loudly when it is absent."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise MvmError(
            'libmvm_b200.so not found at %s -- the CUDA extension is required (no CPU fallback). '
            'Build it with: python -m e2e_multi_view_matching_b200.build' % LIB_PATH)
    L = C.CDLL(LIB_PATH)
    L.mvm_version.restype = C.c_char_p
    L.mvm_matcher_workspace_bytes.restype = C.c_size_t
    L.mvm_matcher_workspace_bytes.argtypes = [C.c_int] * 5
    L.mvm_matcher_forward.restype = C.c_int
    L.mvm_matcher_forward.argtypes = [
        C.POINTER(MatcherWeights), C.c_int, C.c_int, C.c_int, C.POINTER(C.c_int), _fp, _fp, _fp,
        C.c_float, C.c_float, C.c_int, C.c_float, C.POINTER(PairIO), C.c_int, _fp, C.c_size_t, _fp]
    L.mvm_gt_matches_workspace_bytes.restype = C.c_size_t
    L.mvm_gt_matches_workspace_bytes.argtypes = [C.c_int, C.c_int]
    L.mvm_gt_matches_pair.restype = C.c_int
    L.mvm_gt_matches_pair.argtypes = [_fp] * 7 + [C.c_int] * 4 + [C.c_float, C.c_float, _fp, _fp, _fp, C.c_size_t, _fp]
    I, F = C.c_int, C.c_float
    L.mvm_batchnorm_train.restype = I
    L.mvm_batchnorm_train.argtypes = [_fp, _fp, I, I, I, I, I, I, I, _fp, _fp, F, I, _fp, _fp, F, _fp, _fp, _fp]
    L.mvm_batchnorm_train_backward.restype = I
    L.mvm_batchnorm_train_backward.argtypes = [_fp, _fp, _fp, I, I, I, I, I, I, I, _fp, _fp, I, _fp, _fp, I, _fp, _fp]
    L.mvm_colsum.restype = I
    L.mvm_colsum.argtypes = [_fp, I, I, I, _fp, I, _fp, _fp]
    L.mvm_conf_backward_ws_doubles.restype = C.c_size_t
    L.mvm_conf_backward_ws_doubles.argtypes = [I]
    L.mvm_debug_set_conf_i0_check.restype = None
    L.mvm_debug_set_conf_i0_check.argtypes = [I]
    L.mvm_conf_tail_backward.restype = I
    L.mvm_conf_tail_backward.argtypes = [_fp, _fp, _fp, _fp, I, _fp, _fp, _fp, _fp, C.c_size_t, _fp]
    L.mvm_conf_gather_backward.restype = I
    L.mvm_conf_gather_backward.argtypes = [_fp] * 5 + [I] * 5 + [C.POINTER(I), C.POINTER(I)] + [_fp] * 4 + [C.c_size_t, _fp]
    L.mvm_transpose_split.restype = I
    L.mvm_transpose_split.argtypes = [_fp, I, I, I, _fp, _fp, _fp, C.c_longlong, _fp]
    L.mvm_attention_backward.restype = I
    L.mvm_attention_backward.argtypes = [_fp, _fp, _fp, _fp, _fp, I, I, I, C.POINTER(C.c_int), I, _fp]
    L.mvm_linear_tc_presplit_splitk.restype = I
    L.mvm_linear_tc_presplit_splitk.argtypes = [_fp, I, _fp, _fp, I, _fp, I, I, I, I, F, I, _fp, _fp]
    L.mvm_debug_set_attention_backward_variant.restype = I
    L.mvm_debug_set_attention_backward_variant.argtypes = [I]
    L.mvm_sinkhorn_train_pot_floats.restype = C.c_size_t
    L.mvm_sinkhorn_train_pot_floats.argtypes = [I, I, I, I]
    L.mvm_sinkhorn_train_forward.restype = I
    L.mvm_sinkhorn_train_forward.argtypes = [_fp, C.c_longlong, C.c_longlong, _fp, I, I, I, I, _fp, _fp, _fp]
    L.mvm_sinkhorn_train_backward.restype = I
    L.mvm_sinkhorn_train_backward.argtypes = [_fp, C.c_longlong, C.c_longlong, _fp, _fp, I, I, I, I, _fp, _fp, _fp]
    L.mvm_pair_scores.restype = I
    L.mvm_pair_scores.argtypes = [_fp, _fp, _fp, I, I, I, I, C.POINTER(I), C.POINTER(I), C.POINTER(I), C.POINTER(I),
                                  C.POINTER(C.c_void_p), F, _fp]
    L.mvm_pack_views.restype = C.c_int
    L.mvm_pack_views.argtypes = [C.POINTER(C.c_void_p), C.POINTER(C.c_void_p), C.POINTER(C.c_void_p), C.POINTER(C.c_int),
                                 C.c_int, C.c_int, C.c_int, _fp, _fp, _fp, _fp]
    L.mvm_matcher_options_default.restype = None
    L.mvm_matcher_options_default.argtypes = [C.POINTER(MatcherOptions)]
    L.mvm_matcher_forward_ex.restype = C.c_int
    L.mvm_matcher_forward_ex.argtypes = [
        C.POINTER(MatcherWeights), C.c_int, C.c_int, C.c_int, C.POINTER(C.c_int), _fp, _fp, _fp,
        C.c_float, C.c_float, C.c_int, C.c_float, C.POINTER(PairIO), C.c_int, _fp, C.c_size_t,
        C.POINTER(MatcherOptions), _fp]
    L.mvm_matcher_forward_views.restype = C.c_int
    L.mvm_matcher_forward_views.argtypes = [
        C.POINTER(MatcherWeights), C.c_int, C.c_int, C.c_int, C.POINTER(C.c_int), _fp, _fp, _fp,
        C.POINTER(C.c_float), C.c_int, C.c_float, C.POINTER(PairIO), C.c_int, _fp, C.c_size_t,
        C.POINTER(MatcherOptions), _fp]
    for name in ('mvm_debug_set_score_kernel', 'mvm_debug_set_gemm_tile', 'mvm_debug_set_gemm_kernel',
                 'mvm_debug_set_attention_split', 'mvm_debug_set_gemm_split', 'mvm_debug_set_attention_h3_variant'):
        getattr(L, name).restype = None
        getattr(L, name).argtypes = [C.c_int]
    for name in ('mvm_debug_set_attention_timing', 'mvm_debug_set_sinkhorn_timing', 'mvm_debug_set_mvba_timing'):
        getattr(L, name).restype = None
        getattr(L, name).argtypes = [_fp]
    L.mvm_linear.restype = C.c_int
    L.mvm_linear.argtypes = [_fp, C.c_int, _fp, C.c_int, C.c_int, _fp, C.c_int, _fp, _fp, C.c_int,
                             _fp, C.c_int, C.c_int, C.c_int, C.c_int, C.c_float, C.c_int, _fp]
    L.mvm_linear_tc_presplit.restype = C.c_int
    L.mvm_linear_tc_presplit.argtypes = [_fp, C.c_int, _fp, C.c_int, C.c_int, _fp, _fp, C.c_int, _fp, _fp, C.c_int,
                                         _fp, C.c_int, C.c_int, C.c_int, C.c_int, C.c_float, C.c_int, _fp]
    L.mvm_linear_tc_h16.restype = C.c_int
    L.mvm_linear_tc_h16.argtypes = [_fp, C.c_int, _fp, C.c_int, C.c_int, _fp, _fp, C.c_float, C.c_int, _fp, _fp, C.c_int,
                                    _fp, C.c_int, C.c_int, C.c_int, C.c_int, C.c_float, C.c_int, _fp]
    L.mvm_qkv_projection.restype = C.c_int
    L.mvm_qkv_projection.argtypes = [_fp, _fp, _fp, _fp, _fp, C.c_float, _fp, _fp, C.c_int, C.c_int, C.c_int,
                                     _fp, _fp, _fp, _fp, _fp]
    L.mvm_linear_tc.restype = C.c_int
    L.mvm_linear_tc.argtypes = [_fp, C.c_int, _fp, C.c_int, C.c_int, _fp, C.c_int, _fp, _fp, C.c_int,
                                _fp, C.c_int, C.c_int, C.c_int, C.c_int, C.c_float, C.c_int, C.c_int, _fp]
    L.mvm_set_math_mode.restype = C.c_int
    L.mvm_set_math_mode.argtypes = [C.c_int]
    L.mvm_get_math_mode.restype = C.c_int
    L.mvm_attention_tc.restype = C.c_int
    L.mvm_attention_tc.argtypes = [_fp, _fp, _fp, C.c_int, C.c_int, C.c_int, C.POINTER(C.c_int), C.c_int, C.c_int, _fp,
                                   _fp, _fp]
    L.mvm_attention_h3.restype = C.c_int
    L.mvm_attention_h3.argtypes = [_fp, _fp, _fp, _fp, _fp, _fp, C.c_int, C.c_int, C.c_int, C.POINTER(C.c_int), C.c_int, _fp]
    L.mvm_attention.restype = C.c_int
    L.mvm_attention.argtypes = [_fp, _fp, C.c_int, C.c_int, C.c_int, C.POINTER(C.c_int), C.c_int, _fp]
    L.mvm_sinkhorn_workspace_floats.restype = C.c_size_t
    L.mvm_sinkhorn_workspace_floats.argtypes = [C.c_int, C.c_int, C.c_int]
    for name in ('mvm_log_optimal_transport', 'mvm_log_optimal_transport_ref', 'mvm_log_optimal_transport_logdomain'):
        f = getattr(L, name)
        f.restype = C.c_int
        f.argtypes = [_fp, C.c_int, C.c_int, C.c_int, C.c_float, C.c_int, _fp, _fp]
    L.mvm_log_optimal_transport_ex.restype = C.c_int
    L.mvm_log_optimal_transport_ex.argtypes = [_fp, C.c_int, C.c_int, C.c_int, C.c_float, C.c_int, _fp, C.c_int, _fp]
    L.mvm_sinkhorn_max_active_clusters.restype = C.c_int
    L.mvm_sinkhorn_max_active_clusters.argtypes = [C.c_int, C.c_int]
    L.mvm_extract_matches.restype = C.c_int
    L.mvm_extract_matches.argtypes = [_fp, C.c_int, C.c_int, C.c_int, C.c_float, _fp, _fp, _fp,
                                      _fp, _fp, _fp]
    L.mvm_w8pt.restype = C.c_int
    L.mvm_w8pt.argtypes = [_fp, _fp, _fp, _fp, _fp, C.c_int, C.c_int, _fp, C.c_int, C.c_int, _fp,
                           _fp, _fp, _fp, _fp, _fp, _fp, _fp, _fp, _fp]
    L.mvm_w8pt_backward.restype = C.c_int
    L.mvm_w8pt_backward.argtypes = [_fp, _fp, _fp, _fp, _fp, C.c_int, C.c_int, _fp, C.c_int, _fp, _fp, _fp, _fp, _fp]
    L.mvm_ransac_essential.restype = C.c_int
    L.mvm_ransac_essential.argtypes = [_fp, _fp, _fp, _fp, C.c_int, C.c_int, _fp, C.c_float, C.c_double, C.c_int,
                                       C.c_ulonglong, _fp, _fp, _fp, _fp, _fp, _fp, _fp, _fp, _fp, _fp]
    L.mvm_ba2view.restype = C.c_int
    L.mvm_ba2view.argtypes = [_fp, _fp, _fp, _fp, C.c_int, C.c_int, C.c_int, _fp, _fp, _fp, _fp, _fp, _fp, _fp]
    L.mvm_gather_matches.restype = C.c_int
    L.mvm_gather_matches.argtypes = [_fp, C.c_int, C.c_int, C.POINTER(C.c_int), C.POINTER(PairIO), C.c_int,
                                     C.c_int, C.c_float, _fp, _fp, _fp, _fp, _fp]
    L.mvm_spanning_tree_init.restype = C.c_int
    L.mvm_spanning_tree_init.argtypes = [C.POINTER(C.c_int), C.POINTER(C.c_int), C.c_int, C.c_int, C.c_int,
                                         _fp, _fp, _fp, _fp, _fp, _fp]
    L.mvm_ba_initialize.restype = C.c_int
    L.mvm_ba_initialize.argtypes = [C.POINTER(C.c_int), C.POINTER(C.c_int), C.c_int, C.c_int, C.c_int, C.c_int,
                                    _fp, _fp, _fp, _fp, _fp, C.c_int, _fp, _fp, _fp]
    L.mvm_mvba_workspace_bytes.restype = C.c_size_t
    L.mvm_mvba_workspace_bytes.argtypes = [C.c_int] * 4
    L.mvm_multi_view_ba.restype = C.c_int
    L.mvm_multi_view_ba.argtypes = [C.POINTER(C.c_int), C.POINTER(C.c_int), C.c_int, C.c_int, C.c_int, C.c_int,
                                    _fp, _fp, _fp, _fp, _fp, _fp, C.c_int, _fp, _fp, _fp, C.c_size_t, _fp]
    L.mvm_multi_view_ba_ex.restype = C.c_int
    L.mvm_multi_view_ba_ex.argtypes = [C.POINTER(C.c_int), C.POINTER(C.c_int), C.c_int, C.c_int, C.c_int, C.c_int,
                                       _fp, _fp, _fp, _fp, _fp, _fp, C.c_int, _fp, _fp, C.c_int, _fp, _fp, _fp,
                                       C.c_size_t, _fp]
    L.mvm_multi_view_ba_obs.restype = C.c_int
    L.mvm_multi_view_ba_obs.argtypes = [C.POINTER(C.c_int), C.POINTER(C.c_int), C.c_int, C.c_int, C.c_int, C.c_int,
                                        _fp, _fp, _fp, _fp, _fp, _fp, _fp, C.c_int, _fp, _fp, C.c_int, _fp, _fp, _fp,
                                        C.c_size_t, _fp]
    L.mvm_triangulate_pairs.restype = C.c_int
    L.mvm_triangulate_pairs.argtypes = [C.POINTER(C.c_int), C.POINTER(C.c_int), C.c_int, C.c_int, C.c_int, C.c_int,
                                        _fp, _fp, _fp, _fp, _fp, _fp]
    L.mvm_superpoint_workspace_bytes.restype = C.c_size_t
    L.mvm_superpoint_workspace_bytes.argtypes = [C.c_int, C.c_int, C.c_int]
    L.mvm_superpoint_dense.restype = C.c_int
    L.mvm_superpoint_dense.argtypes = [C.POINTER(SuperPointWeights), _fp, C.c_int, C.c_int, C.c_int, C.c_int, _fp, _fp, _fp,
                                       C.c_size_t, _fp]
    L.mvm_superpoint_sample.restype = C.c_int
    L.mvm_superpoint_sample.argtypes = [_fp, _fp, C.c_int, C.c_int, C.c_int, _fp, _fp]
    L.mvm_superpoint_select.restype = C.c_int
    L.mvm_superpoint_select.argtypes = [_fp, C.c_int, C.c_int, C.c_int, C.c_float, C.c_int, C.c_int, _fp, _fp, _fp, _fp]
    L.mvm_superpoint_sample_batch.restype = C.c_int
    L.mvm_superpoint_sample_batch.argtypes = [_fp, _fp, _fp, C.c_int, C.c_int, C.c_int, C.c_int, _fp, _fp]
    L.mvm_match_loss_forward.restype = C.c_int
    L.mvm_match_loss_forward.argtypes = [_fp, _fp, _fp, C.c_int, C.c_int, _fp, _fp, _fp]
    L.mvm_match_loss_backward.restype = C.c_int
    L.mvm_match_loss_backward.argtypes = [_fp, _fp, _fp, C.c_int, C.c_int, _fp, _fp]
    L.mvm_launch_count.restype = C.c_ulonglong
    L.mvm_profile_enable.argtypes = [C.c_int]
    L.mvm_profile_collect.restype = C.c_int
    L.mvm_profile_collect.argtypes = [C.POINTER(C.c_double), C.POINTER(C.c_int), C.c_int]
    _lib = L
    return L


def check(status, what):
    if status != 0:
        raise MvmError('%s failed: %s (status %d)' % (what, _STATUS.get(status, 'unknown'), status))


def require_cuda(device, what):
    """There is no CPU fallback: every entry point refuses non-CUDA tensors."""
    if device.type != 'cuda':
        raise MvmError('%s needs CUDA tensors (no CPU fallback)' % what)


def device_ctx(device):
    """Context that makes `device` the current CUDA device for the launches inside it."""
    import contextlib
    import torch
    return torch.cuda.device(device) if device.type == 'cuda' else contextlib.nullcontext()


def stream_ptr():
    import torch
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def ptr(t):
    """Device pointer of a CUDA tensor (or NULL for None)."""
    if t is None:
        return C.c_void_p(0)
    assert t.is_cuda and t.is_contiguous(), 'libmvm_b200 needs contiguous CUDA tensors'
    return C.c_void_p(t.data_ptr())


PROFILE_TAGS = ['gemm', 'attention', 'sinkhorn', 'score_gemm', 'match', 'conf', 'kenc', 'w8pt', 'ba2',
                'mvba', 'misc']


def profile_collect():
    """-> {tag: (milliseconds, scopes)} since the last collect (needs mvm_profile_enable(1))."""
    n = len(PROFILE_TAGS)
    ms = (C.c_double * n)()
    cnt = (C.c_int * n)()
    lib().mvm_profile_collect(ms, cnt, n)
    return {PROFILE_TAGS[i]: (ms[i], cnt[i]) for i in range(n)}
