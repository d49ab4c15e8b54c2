"""Code generation of the staged GEMM epilogue (csrc/gemm_tc.cu), checked without a GPU.

- The persistent instances, fp16x3 <128, 3, W_F16> and tf32x3 <128, 3, W_TF32>, store their output tiles by TMA from
  shared memory: their SASS holds UTMASTG.2D, the sm_90a TMA store.
- Every instance's dynamic shared memory (the ring, the two 16 KB staging buffers of the staged instances, alignment
  slack and barriers) stays within the 232,448 bytes an sm_90 CTA may opt in to.  The launch requests Cfg::SMEM_BYTES,
  which a translation unit that includes the kernel source checks with static_asserts: compiling it is the test.
"""
import importlib.util
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, 'e2e_multi_view_matching_b200')
SRC = os.path.join(PKG, 'csrc', 'gemm_tc.cu')
SM90_SMEM_OPTIN = 232448

# <BN, NPASS, WM, SCORE>: WM 0 = raw W, 1 = tf32 planes, 2 = fp16 planes
INSTANCES = [(128, 3, 2, 0), (128, 3, 1, 0), (128, 3, 1, 1), (128, 3, 0, 0), (128, 1, 0, 0), (256, 3, 1, 0),
             (256, 1, 0, 0)]
STAGED = [(128, 3, 2, 0), (128, 3, 1, 0)]

# Cfg<BN, NPASS, WM>::SMEM_BYTES of every instance against the opt-in limit, and the staged instances' layout: the ring,
# two 16 KB staging buffers, 1024 bytes of alignment slack and 256 of barriers
HARNESS = r'''
#include "gemm_tc.cu"
constexpr int LIMIT = %d;
static_assert(Cfg<128, 3, W_F16>::SMEM_BYTES <= LIMIT && Cfg<128, 3, W_TF32>::SMEM_BYTES <= LIMIT &&
              Cfg<128, 3, W_RAW>::SMEM_BYTES <= LIMIT && Cfg<128, 1, W_RAW>::SMEM_BYTES <= LIMIT &&
              Cfg<256, 3, W_TF32>::SMEM_BYTES <= LIMIT && Cfg<256, 1, W_RAW>::SMEM_BYTES <= LIMIT, "over the opt-in");
static_assert(Cfg<128, 3, W_F16>::SMEM_BYTES == 3 * 65536 + 2 * 16384 + 1024 + 256, "fp16x3 layout");
static_assert(Cfg<128, 3, W_TF32>::SMEM_BYTES == 4 * 49152 + 2 * 16384 + 1024 + 256, "tf32x3 layout");
''' % SM90_SMEM_OPTIN


def mangled(inst):
    return 'gemm_wg_kernelILi%dELi%dELi%dELb%dE' % inst


def _build_module():
    # build.py on its own: importing the package would load the CUDA library
    spec = importlib.util.spec_from_file_location('_mvm_build', os.path.join(PKG, 'build.py'))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def _tools():
    b = _build_module()
    nvcc = b.NVCC if os.path.exists(b.NVCC) else shutil.which('nvcc')
    cuobjdump = os.path.join(os.path.dirname(nvcc), 'cuobjdump') if nvcc else None
    if not nvcc or not cuobjdump or not os.path.exists(cuobjdump):
        pytest.skip('nvcc / cuobjdump not available')
    return b, nvcc, cuobjdump


@pytest.fixture(scope='module')
def sass(tmp_path_factory):
    b, nvcc, cuobjdump = _tools()
    obj = str(tmp_path_factory.mktemp('gemm_tma_codegen') / 'gemm_tc.o')
    r = subprocess.run([nvcc] + b.FLAGS + ['-c', SRC, '-o', obj], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    return subprocess.run([cuobjdump, '-sass', obj], capture_output=True, text=True, check=True).stdout


def sass_function(sass, inst):
    hits = [f for f in re.split(r'\n\s*Function : ', sass)[1:] if mangled(inst) in f.split('\n', 1)[0]]
    assert len(hits) == 1, (inst, len(hits))
    return hits[0]


@pytest.mark.parametrize('inst', STAGED, ids=mangled)
def test_staged_instance_stores_by_tma(sass, inst):
    assert 'UTMASTG.2D' in sass_function(sass, inst)


def test_every_instance_fits_the_shared_memory_opt_in(tmp_path):
    b, nvcc, _ = _tools()
    src = tmp_path / 'smem.cu'
    src.write_text(HARNESS)
    # host code only: the static_asserts are checked in the host pass
    r = subprocess.run([nvcc] + b.FLAGS + ['-I', os.path.join(PKG, 'csrc'), '--cuda', str(src), '-o',
                                           str(tmp_path / 'smem.ii')], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
