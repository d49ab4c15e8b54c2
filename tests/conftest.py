import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line('markers', 'gpu: needs a CUDA device (an H100)')


@pytest.fixture(scope='session')
def golden_dir():
    return os.path.join(ROOT, 'tests', 'golden')


@pytest.fixture(autouse=True)
def _default_math_mode(request):
    """Every GPU test starts from the library default (3xTF32 on the tensor cores) regardless of what ran before."""
    if request.node.get_closest_marker('gpu') is not None:
        import e2e_multi_view_matching_b200 as pkg
        pkg.set_math_mode(3)
        from e2e_multi_view_matching_b200 import _lib
        _lib.lib().mvm_debug_set_attention_split(1)
        _lib.lib().mvm_debug_set_gemm_split(1)
    yield
