"""Code generation of the production Sinkhorn (csrc/sinkhorn_cl.cu), checked without a GPU.

Every iteration of the default instance sinkhorn_cl_kernel<8, 2, false> (and of its phase-timing twin <8, 2, true>)
must run from registers and shared memory only: a local-memory access inside the iteration loop is a dependent trip
through L1 on the critical path of all 100 iterations.  The test asserts that no LDL / STL lies between the loop head
and its back edge in the SASS.  It does not ask for a 0-byte stack frame: the frame that remains holds a few row
pointers of the initial pass that ptxas keeps for the output pass, stored once before the loop and reloaded once after
it, which costs nothing per iteration.
"""
import importlib.util
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, 'e2e_multi_view_matching_b200')
SRC = os.path.join(PKG, 'csrc', 'sinkhorn_cl.cu')


def _build_module():
    # build.py on its own: importing the package would load the CUDA library
    spec = importlib.util.spec_from_file_location('_mvm_build', os.path.join(PKG, 'build.py'))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def _tool(name, nvcc):
    p = os.path.join(os.path.dirname(nvcc), name)
    return p if os.path.exists(p) else shutil.which(name)


@pytest.fixture(scope='module')
def compiled(tmp_path_factory):
    b = _build_module()
    nvcc = b.NVCC if os.path.exists(b.NVCC) else shutil.which('nvcc')
    cuobjdump = _tool('cuobjdump', nvcc) if nvcc else None
    if not nvcc or not cuobjdump:
        pytest.skip('nvcc / cuobjdump not available')
    obj = str(tmp_path_factory.mktemp('sinkhorn_codegen') / 'sinkhorn_cl.o')
    r = subprocess.run([nvcc] + b.FLAGS + ['-Xptxas', '-v', '-c', SRC, '-o', obj], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    sass = subprocess.run([cuobjdump, '-sass', obj], capture_output=True, text=True, check=True).stdout
    return r.stderr, sass


def _function(sass, mangled):
    for f in re.split(r'\n\s*Function : ', sass)[1:]:
        if mangled in f.split('\n', 1)[0]:
            return [(int(a, 16), t.strip()) for a, t in re.findall(r'/\*([0-9a-f]{4,})\*/\s+([^;]*);', f)]
    raise AssertionError('%s not in the SASS' % mangled)


def iteration_loop(ins):
    """The instructions of the Sinkhorn iteration loop: the innermost loop (backward branch) around the CTA-wide
    vote on column re-absorption (__syncthreads_or -> BAR.RED.OR), which every iteration executes once."""
    votes = [a for a, t in ins if 'BAR.RED.OR' in t]
    assert len(votes) == 1, votes
    loops = []
    for a, t in ins:
        m = re.search(r'\bBRA(?:\.\w+)*\s+(0x[0-9a-f]+)', t)
        if m and int(m.group(1), 16) <= votes[0] < a:
            loops.append((int(m.group(1), 16), a))
    assert loops, 'no loop around the absorb vote'
    lo, hi = min(loops, key=lambda x: x[1] - x[0])
    return [(a, t) for a, t in ins if lo <= a <= hi]


@pytest.mark.parametrize('timing', [False, True])
def test_production_sinkhorn_iteration_has_no_local_memory(compiled, timing):
    log, sass = compiled
    ins = _function(sass, 'sinkhorn_cl_kernelILi8ELi2ELb%dE' % int(timing))
    body = iteration_loop(ins)
    assert sum(1 for _, t in body if re.search(r'\bFFMA\b', t)) >= 64     # the row and column passes are in it
    local = [(hex(a), t) for a, t in body if re.search(r'\b(LDL|STL)\b', t)]
    assert not local, local


def test_production_sinkhorn_fits_one_cta_per_sm(compiled):
    log, _ = compiled
    # ptxas -v: "Compiling entry function '<mangled>'" ... "Used N registers" for each instance
    for timing in (0, 1):
        m = re.search(r"sinkhorn_cl_kernelILi8ELi2ELb%dE[^\n]*'.*?Used (\d+) registers" % timing, log, re.S)
        assert m, log
        assert int(m.group(1)) <= 128      # 512 threads x 128 registers = the register file of one SM
