"""Code generation of the tensor-core GEMM (csrc/gemm_tc.cu), checked without a GPU.

- No instance of gemm_wg_kernel spills.  Every instance runs 384 threads with setmaxnreg (232 registers per consumer
  thread); the 256-column instances once ran 288 threads, which ptxas budgets as 384 at 168 registers each, and spilled
  up to 124 bytes with their wgmma serialised.
- The 128-column instances keep the pipelined mainloop: the wgmma of k-block kt are retired by a wait<1> while those of
  kt + 1 are in flight (WARPGROUP.DEPBAR.LE gsb0, 0x1).  An in-order mainloop has only waits for 0 groups.
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

# <BN, NPASS, WM, SCORE>: WM 0 = raw W, 1 = tf32 planes, 2 = fp16 planes
INSTANCES = [(128, 3, 2, 0), (128, 3, 1, 0), (128, 3, 1, 1), (128, 3, 0, 0), (128, 1, 0, 0), (256, 3, 1, 0),
             (256, 1, 0, 0)]


def mangled(inst):
    return 'gemm_wg_kernelILi%dELi%dELi%dELb%dE' % inst


def _build_module():
    # build.py on its own: importing the package would load the CUDA library
    spec = importlib.util.spec_from_file_location('_mvm_build', os.path.join(PKG, 'build.py'))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


@pytest.fixture(scope='module')
def compiled(tmp_path_factory):
    b = _build_module()
    nvcc = b.NVCC if os.path.exists(b.NVCC) else shutil.which('nvcc')
    cuobjdump = shutil.which('cuobjdump') if not nvcc else os.path.join(os.path.dirname(nvcc), 'cuobjdump')
    if not nvcc or not cuobjdump or not os.path.exists(cuobjdump):
        pytest.skip('nvcc / cuobjdump not available')
    obj = str(tmp_path_factory.mktemp('gemm_codegen') / 'gemm_tc.o')
    r = subprocess.run([nvcc] + b.FLAGS + ['-Xptxas', '-v', '-c', SRC, '-o', obj], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    sass = subprocess.run([cuobjdump, '-sass', obj], capture_output=True, text=True, check=True).stdout
    return r.stderr, sass


def ptxas_entry(log, inst):
    """The ptxas -v lines of one instance: from its 'Compiling entry function' to the next one."""
    parts = re.split(r"ptxas info\s+: Compiling entry function ", log)
    hits = [p for p in parts[1:] if mangled(inst) in p.split('\n', 1)[0]]
    assert len(hits) == 1, (inst, len(hits))
    return hits[0]


def sass_function(sass, inst):
    hits = [f for f in re.split(r'\n\s*Function : ', sass)[1:] if mangled(inst) in f.split('\n', 1)[0]]
    assert len(hits) == 1, (inst, len(hits))
    return hits[0]


def test_every_instance_is_compiled(compiled):
    log, _ = compiled
    found = set(re.findall(r'gemm_wg_kernelILi(\d+)ELi(\d+)ELi(\d+)ELb(\d)E', log))
    assert found == {tuple(str(x) for x in i) for i in INSTANCES}, found


@pytest.mark.parametrize('inst', INSTANCES, ids=mangled)
def test_gemm_instance_does_not_spill(compiled, inst):
    log, _ = compiled
    entry = ptxas_entry(log, inst)
    m = re.search(r'(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads', entry)
    assert m, entry
    assert m.groups() == ('0', '0', '0'), (inst, m.group(0))
    # C7512: "wgmma.mma_async instructions are serialized due to insufficient register resources"
    serialised = [l for l in log.splitlines() if 'C7512' in l and mangled(inst) in l]
    assert not serialised, serialised


@pytest.mark.parametrize('inst', [(128, 3, 2, 0), (128, 3, 1, 0)], ids=mangled)
def test_pipelined_mainloop_waits_for_one_group(compiled, inst):
    _, sass = compiled
    f = sass_function(sass, inst)
    waits = re.findall(r'WARPGROUP\.DEPBAR\.LE gsb0, (0x[0-9a-f]+)', f)
    assert waits.count('0x1') >= 2, waits       # one per k-block of the two-k-block trip
