"""CPU: mvm_superpoint_dense / _sample / _select / _sample_batch refuse invalid arguments before any launch, and the
SuperPoint kernels compile for sm_90a without register spills.  The refusals use no real device memory: every call below is rejected by
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


def _dense(lib, weights=True, image=FAKE, batch=2, height=16, width=16, r=4, scores=FAKE, dense=FAKE, ws=FAKE,
           ws_bytes=None):
    from e2e_multi_view_matching_b200 import _lib
    w = ctypes.byref(_lib.SuperPointWeights()) if weights else None
    if ws_bytes is None:
        ws_bytes = lib.mvm_superpoint_workspace_bytes(batch, height, width)
    return lib.mvm_superpoint_dense(w, image, batch, height, width, r, scores, dense, ws, ws_bytes, NULL)


@pytest.mark.parametrize('kw', [dict(weights=False), dict(image=NULL), dict(scores=NULL), dict(dense=NULL),
                                dict(ws=NULL), dict(batch=0), dict(batch=-3), dict(height=15), dict(width=15),
                                dict(height=0), dict(r=-1)],
                         ids=lambda kw: ','.join('%s=%s' % (k, 'NULL' if v is NULL else v) for k, v in kw.items()))
def test_dense_refuses(lib, kw):
    assert _dense(lib, **kw) == 1


@pytest.mark.parametrize('shape', [(1, 16, 16), (3, 17, 23), (40, 480, 640)])
def test_dense_refuses_short_workspace(lib, shape):
    B, H, W = shape
    need = lib.mvm_superpoint_workspace_bytes(B, H, W)
    assert need >= (2 * 64 + 5) * B * H * W * 4            # two 64-channel activations + five score-map planes
    assert _dense(lib, batch=B, height=H, width=W, ws_bytes=need - 1) == 3       # MVM_ERR_WORKSPACE


@pytest.mark.parametrize('args', [(FAKE, FAKE, -1, 4, 4, FAKE), (FAKE, FAKE, 8, 0, 4, FAKE), (FAKE, FAKE, 8, 4, 0, FAKE),
                                  (FAKE, FAKE, 8, -1, 4, FAKE), (NULL, FAKE, 8, 4, 4, FAKE),
                                  (FAKE, FAKE, 8, 4, 4, NULL), (FAKE, NULL, 8, 4, 4, FAKE), (FAKE, NULL, 1, 4, 4, FAKE)])
def test_sample_refuses(lib, args):
    assert lib.mvm_superpoint_sample(*args, NULL) == 1


def test_sample_of_no_keypoints_is_ok_without_a_launch(lib):
    """n == 0 returns before any launch: the fake pointers are never touched and no device is needed."""
    assert lib.mvm_superpoint_sample(FAKE, NULL, 0, 4, 4, FAKE, NULL) == 0
    assert lib.mvm_superpoint_sample(FAKE, FAKE, 0, 1, 1, FAKE, NULL) == 0


def test_select_and_sample_kernels_do_not_spill(tmp_path):
    b = _build_module()
    nvcc = b.NVCC if os.path.exists(b.NVCC) else None
    if not nvcc or not _tool('cuobjdump', nvcc):
        pytest.skip('nvcc not available')
    r = subprocess.run([nvcc] + b.FLAGS + ['-Xptxas', '-v', '-c', os.path.join(PKG, 'csrc', 'superpoint.cu'), '-o',
                        str(tmp_path / 'sp.o')], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    for name in ('sp_select_kernel', 'sp_sample_batch_kernel', 'sp_sample_kernel', 'sp_conv3x3_kernel',
                 'sp_scores_kernel'):
        m = re.search(r"Compiling entry function '[^']*%s[^']*'.*?(\d+) bytes stack frame, (\d+) bytes spill stores, "
                      r"(\d+) bytes spill loads.*?Used (\d+) registers" % name, r.stderr, re.S)
        assert m, (name, r.stderr)
        assert m.group(2) == m.group(3) == '0', (name, m.group(0))
        if name == 'sp_select_kernel':
            assert int(m.group(4)) <= 64, m.group(0)          # 1024 threads per CTA
