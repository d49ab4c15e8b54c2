"""H100-native (sm_90a) engine for the hot path of barbararoessle/e2e_multi_view_matching.

Host-side mirror of the reference's Python interface for that path:
  models.multi_view_matcher.MultiViewMatcher   (models/models/multi_view_matcher.py:103)
  models.superglue.SuperGlue                   (models/models/superglue.py:179)
  models.matching.Matching                     (upstream SuperGlue shim)
  pose_optimization.two_view.*                 (pose_optimization/two_view/*.py)
  pose_optimization.multi_view.*               (pose_optimization/multi_view/*)
Everything computes in libmvm_b200.so (hand-written CUDA, C ABI in include/mvm_b200.h);
there is no CPU fallback.
"""
__version__ = '0.1'


def set_math_mode(mode):
    """Math mode of the matcher's GEMMs/attention: 0 = fp32 CUDA cores, 3 = 3xTF32 on the tensor cores
    (fp32-faithful), 1 = single-pass TF32."""
    from . import _lib
    _lib.check(_lib.lib().mvm_set_math_mode(int(mode)), 'mvm_set_math_mode')


def get_math_mode():
    from . import _lib
    return int(_lib.lib().mvm_get_math_mode())
