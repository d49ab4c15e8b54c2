"""Code generation of the tensor-core attention (attention_wg_kernel in csrc/attention_wg.cuh, instantiated by
csrc/attention_h3.cu for fp16x3 and csrc/attention_tc.cu for single-pass tf32 and 3xTF32), checked without a GPU.

- No instance spills or keeps a stack frame, and ptxas serialises no wgmma (C7512).  Every instance runs 384 threads with
  setmaxnreg (232 registers per consumer thread); at 288 threads ptxas capped every thread at 168 registers and the
  3xTF32 instance spilled 72 bytes.
- The fp16x3 instance keeps its pipelined schedule: the S of a key tile is retired by a wait<1> while the P V of the
  previous tile is in flight (WARPGROUP.DEPBAR.LE gsb0, 0x1).
- In the fp16x3 instance S = Q K^T takes Q from registers: no wgmma of that kernel has two shared-memory descriptors.
"""
import os
import re
import shutil
import subprocess

import pytest

from tests.test_gemm_codegen import _build_module

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, 'e2e_multi_view_matching_b200', 'csrc')
SOURCES = {16: 'attention_h3.cu', 1: 'attention_tc.cu', 3: 'attention_tc.cu'}


def mangled(mode):
    return '_ZN7attn_wg19attention_wg_kernelILi%dEEEv' % mode


@pytest.fixture(scope='module')
def compiled(tmp_path_factory):
    b = _build_module()
    nvcc = b.NVCC if os.path.exists(b.NVCC) else shutil.which('nvcc')
    cuobjdump = os.path.join(os.path.dirname(nvcc), 'cuobjdump') if nvcc else None
    if not nvcc or not os.path.exists(cuobjdump):
        pytest.skip('nvcc / cuobjdump not available')
    tmp = tmp_path_factory.mktemp('attention_codegen')
    out = {}
    for src in sorted(set(SOURCES.values())):
        obj = str(tmp / (src[:-3] + '.o'))
        r = subprocess.run([nvcc] + b.FLAGS + ['-Xptxas', '-v', '-c', os.path.join(CSRC, src), '-o', obj],
                           capture_output=True, text=True)
        assert r.returncode == 0, r.stderr
        sass = subprocess.run([cuobjdump, '-sass', obj], capture_output=True, text=True, check=True).stdout
        ptx = subprocess.run([nvcc] + b.FLAGS + ['-ptx', os.path.join(CSRC, src), '-o', '-'], capture_output=True,
                             text=True, check=True).stdout
        out[src] = (r.stderr, sass, ptx)
    return out


def ptxas_entry(log, mode):
    """The ptxas -v lines of one instance: from its 'Compiling entry function' to the next one."""
    parts = re.split(r"ptxas info\s+: Compiling entry function ", log)
    hits = [p for p in parts[1:] if mangled(mode) in p.split('\n', 1)[0]]
    assert len(hits) == 1, (mode, len(hits))
    return hits[0]


@pytest.mark.parametrize('mode', sorted(SOURCES))
def test_attention_instance_does_not_spill(compiled, mode):
    log, _, _ = compiled[SOURCES[mode]]
    entry = ptxas_entry(log, mode)
    m = re.search(r'(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads', entry)
    assert m, entry
    assert m.groups() == ('0', '0', '0'), (mode, m.group(0))
    # C7512: "wgmma.mma_async instructions are serialized due to insufficient register resources"
    serialised = [l for l in log.splitlines() if 'C7512' in l and mangled(mode) in l]
    assert not serialised, serialised


def test_fp16x3_keeps_the_pipelined_wait(compiled):
    _, sass, _ = compiled[SOURCES[16]]
    hits = [f for f in re.split(r'\n\s*Function : ', sass)[1:] if mangled(16) in f.split('\n', 1)[0]]
    assert len(hits) == 1, len(hits)
    waits = re.findall(r'WARPGROUP\.DEPBAR\.LE gsb0, (0x[0-9a-f]+)', hits[0])
    assert '0x1' in waits, waits


def test_fp16x3_reads_q_from_registers(compiled):
    _, _, ptx = compiled[SOURCES[16]]
    body = ptx.split('.entry ' + mangled(16), 1)[1].split('.entry ', 1)[0]
    mmas = re.findall(r'wgmma\.mma_async[^;]*;', body, re.S)
    assert len(mmas) >= 24, len(mmas)                          # 12 for S, 12 for P V (pipelined body)
    # operands: {d...}, a, b-desc, ...  -- the A operand of a register form is a brace-enclosed list
    both_desc = [m for m in mmas if re.search(r'\}\s*,\s*%rd\d+\s*,\s*%rd\d+', m)]
    assert not both_desc, both_desc[:1]
