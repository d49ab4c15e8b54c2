"""CPU: mvm_superpoint_select / mvm_superpoint_sample_batch refuse invalid arguments before any launch, and their kernels
compile for sm_90a without register spills.  The refusals use no real device memory: every call below is rejected by
the argument checks, which run before anything touches a pointer."""
import ctypes
import os
import re
import subprocess

import pytest

from tests.test_sinkhorn_codegen import _build_module, _tool, PKG

FAKE = ctypes.c_void_p(256)          # never dereferenced: the calls are refused first
NULL = ctypes.c_void_p(0)


@pytest.fixture(scope='module')
def lib():
    from e2e_multi_view_matching_b200 import build, _lib
    build.build()
    return _lib.lib()


def _select(lib, batch=2, height=64, width=64, thr=0.005, border=4, k=16, ptrs=(FAKE,) * 4):
    sc, kp, out, cnt = ptrs
    return lib.mvm_superpoint_select(sc, batch, height, width, thr, border, k, kp, out, cnt, NULL)


@pytest.mark.parametrize('kw', [dict(batch=0), dict(batch=-1), dict(height=0), dict(width=-8), dict(height=12),
                                dict(width=20), dict(border=-1), dict(k=0), dict(k=-5), dict(k=64 * 64 + 1),
                                dict(height=256, width=256, k=16385), dict(thr=float('nan')),
                                dict(ptrs=(NULL, FAKE, FAKE, FAKE)), dict(ptrs=(FAKE, NULL, FAKE, FAKE)),
                                dict(ptrs=(FAKE, FAKE, NULL, FAKE)), dict(ptrs=(FAKE, FAKE, FAKE, NULL)),
                                dict(ptrs=(ctypes.c_void_p(260), FAKE, FAKE, FAKE))],
                         ids=lambda kw: ','.join('%s=%s' % (k, 'ptrs' if k == 'ptrs' else v) for k, v in kw.items()))
def test_select_refuses(lib, kw):
    assert _select(lib, **kw) == 1


@pytest.mark.parametrize('args', [(FAKE, FAKE, FAKE, 0, 8, 4, 4, FAKE), (FAKE, FAKE, FAKE, 2, 0, 4, 4, FAKE),
                                  (FAKE, FAKE, FAKE, 2, 8, 0, 4, FAKE), (FAKE, FAKE, FAKE, 2, 8, 4, -1, FAKE),
                                  (NULL, FAKE, FAKE, 2, 8, 4, 4, FAKE), (FAKE, NULL, FAKE, 2, 8, 4, 4, FAKE),
                                  (FAKE, FAKE, NULL, 2, 8, 4, 4, FAKE), (FAKE, FAKE, FAKE, 2, 8, 4, 4, NULL)])
def test_sample_batch_refuses(lib, args):
    assert lib.mvm_superpoint_sample_batch(*args, NULL) == 1


def test_select_and_sample_kernels_do_not_spill(tmp_path):
    b = _build_module()
    nvcc = b.NVCC if os.path.exists(b.NVCC) else None
    if not nvcc or not _tool('cuobjdump', nvcc):
        pytest.skip('nvcc not available')
    r = subprocess.run([nvcc] + b.FLAGS + ['-Xptxas', '-v', '-c', os.path.join(PKG, 'csrc', 'superpoint.cu'), '-o',
                        str(tmp_path / 'sp.o')], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    for name in ('sp_select_kernel', 'sp_sample_batch_kernel', 'sp_sample_kernel'):
        m = re.search(r"Compiling entry function '[^']*%s[^']*'.*?(\d+) bytes stack frame, (\d+) bytes spill stores, "
                      r"(\d+) bytes spill loads.*?Used (\d+) registers" % name, r.stderr, re.S)
        assert m, (name, r.stderr)
        assert m.group(2) == m.group(3) == '0', (name, m.group(0))
        if name == 'sp_select_kernel':
            assert int(m.group(4)) <= 64, m.group(0)          # 1024 threads per CTA
