"""The GEMM argument predicate (gemm_desc_valid in csrc/kernels.cuh), checked on the CPU.

Every GEMM launch path (launch_gemm_tc, launch_gemm_tc_persist, which serves mvm_linear_tc_h16 and the split-K entry,
and launch_gemm_simt) refuses a descriptor this predicate rejects before any CUDA call.  A misaligned C or R cannot be
tried on a GPU without risking a fault if the check regressed, so the predicate itself is compiled into a small host
program and run over good and bad descriptors here.  Pointers are plain integers: the predicate never dereferences them.
"""
import importlib.util
import os
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, 'e2e_multi_view_matching_b200')

HARNESS = r'''
#include <cstdio>
#include "kernels.cuh"
int main() {
  int ops, M, N, K, K1, batch, lda, lda2, ldw, ldc, ldr;
  unsigned long long A, A2, W, Whi, Wlo, Whi16, Wlo16, C, R;
  float wscale;
  while (scanf("%d %d %d %d %d %d %llu %d %llu %d %llu %llu %llu %llu %llu %d %f %llu %d %llu %d", &ops, &M, &N, &K,
               &K1, &batch, &A, &lda, &A2, &lda2, &W, &Whi, &Wlo, &Whi16, &Wlo16, &ldw, &wscale, &C, &ldc, &R,
               &ldr) == 21) {
    GemmDesc d = {};
    d.A = (const float*)A; d.lda = lda; d.A2 = (const float*)A2; d.lda2 = lda2; d.K1 = K1;
    d.W = (const float*)W; d.ldw = ldw; d.Whi = (const float*)Whi; d.Wlo = (const float*)Wlo;
    d.Whi16 = (const void*)Whi16; d.Wlo16 = (const void*)Wlo16; d.wscale = wscale;
    d.R = (const float*)R; d.ldr = ldr; d.C = (float*)C; d.ldc = ldc;
    d.M = M; d.N = N; d.K = K; d.alpha = 1.f; d.batch = batch;
    printf("%d\n", gemm_desc_valid(d, ops) ? 1 : 0);
  }
  return 0;
}
'''

FIELDS = ('ops', 'M', 'N', 'K', 'K1', 'batch', 'A', 'lda', 'A2', 'lda2', 'W', 'Whi', 'Wlo', 'Whi16', 'Wlo16', 'ldw',
          'wscale', 'C', 'ldc', 'R', 'ldr')
SIMT, TF32, F16 = 0, 1, 2
BASE = 1 << 20          # a 1 MiB-aligned fake address; + a byte offset gives any alignment


def good(ops):
    d = dict(ops=ops, M=1000, N=256, K=256, K1=256, batch=1, A=BASE, lda=256, A2=0, lda2=0, W=BASE + 0x10000,
             Whi=0, Wlo=0, Whi16=0, Wlo16=0, ldw=256, wscale=0.0, C=BASE + 0x20000, ldc=256, R=0, ldr=0)
    if ops == TF32:
        d.update(Whi=BASE + 0x30000, Wlo=BASE + 0x40000)
    if ops == F16:
        d.update(W=0, Whi16=BASE + 0x30000, Wlo16=BASE + 0x40000, wscale=64.0)
    return d


def variant(ops, **kw):
    d = good(ops)
    d.update(kw)
    return d


def cases():
    """(id, descriptor, expected)"""
    out = []
    for ops, name in ((SIMT, 'simt'), (TF32, 'tf32'), (F16, 'f16')):
        bk = {SIMT: 16, TF32: 32, F16: 64}[ops]
        tc = ops != SIMT
        ok = [
            ('plain', {}),
            ('M1', dict(M=1)),
            ('one_kblock', dict(K=bk, K1=bk, lda=bk, ldw=bk)),
            ('wide_lds', dict(lda=260, ldw=264, ldc=264, R=BASE + 0x50000, ldr=268)),
            ('concat', dict(K=512, K1=bk, A2=BASE + 0x60000, lda2=512 - bk, ldw=512)),
            ('residual_in_place', dict(R=BASE + 0x20000, ldr=256)),
            ('A_16B_offset', dict(A=BASE + 16)),
            ('C_R_8B', dict(C=BASE + 0x20000 + 8, R=BASE + 0x50000 + 8, ldr=256)),
            ('no_bias_no_R', dict(R=0, ldr=0)),
        ]
        if ops == SIMT:
            ok += [('batch3', dict(batch=3)), ('N_ragged', dict(N=100)), ('C_4B', dict(C=BASE + 4, R=BASE + 0x50004, ldr=7)),
                   ('ldc_odd', dict(ldc=257))]
        if ops == TF32:
            ok += [('raw_W_only', dict(Whi=0, Wlo=0)), ('planes_only', dict(W=0))]
        bad = [
            ('M0', dict(M=0)), ('M_negative', dict(M=-5)), ('N0', dict(N=0)),
            ('K0', dict(K=0, K1=0)), ('K_half_kblock', dict(K=bk // 2, K1=bk // 2)),
            ('K_not_multiple', dict(K=256 + bk // 2, K1=256 + bk // 2)),
            ('K1_not_multiple', dict(K=512, K1=bk + bk // 2, A2=BASE + 0x60000, lda2=512)),
            ('K1_ne_K_without_A2', dict(K1=256 - bk)),
            ('concat_K1_0', dict(K=512, K1=0, A2=BASE + 0x60000, lda2=512)),
            ('concat_K1_eq_K', dict(K=512, K1=512, A2=BASE + 0x60000, lda2=512, lda=512, ldw=512)),
            ('A_null', dict(A=0)), ('C_null', dict(C=0)),
            ('A_8B', dict(A=BASE + 8)), ('A_4B', dict(A=BASE + 4)),
            ('A2_8B', dict(K=512, K1=256, A2=BASE + 0x60008, lda2=256, ldw=512)),
            ('lda_odd', dict(lda=258)), ('lda2_odd', dict(K=512, K1=256, A2=BASE + 0x60000, lda2=258, ldw=512)),
            ('ldw_odd', dict(ldw=258)),
        ]
        if ops == SIMT:
            bad += [('W_null', dict(W=0)), ('W_8B', dict(W=BASE + 0x10008)), ('batch0', dict(batch=0))]
        if ops == TF32:
            bad += [('no_W', dict(W=0, Whi=0, Wlo=0)), ('half_planes', dict(W=0, Wlo=0)),
                    ('W_8B', dict(W=BASE + 0x10008)), ('Whi_8B', dict(Whi=BASE + 0x30008)),
                    ('Wlo_4B', dict(Wlo=BASE + 0x40004))]
        if ops == F16:
            bad += [('no_planes', dict(Whi16=0)), ('no_lo_plane', dict(Wlo16=0)), ('wscale0', dict(wscale=0.0)),
                    ('Whi16_8B', dict(Whi16=BASE + 0x30008)), ('Wlo16_2B', dict(Wlo16=BASE + 0x40002)),
                    ('ldw_4_not_8', dict(ldw=260))]
        if tc:
            bad += [('N_not_128', dict(N=192)), ('batch2', dict(batch=2)),
                    ('C_4B', dict(C=BASE + 0x20004)), ('R_4B', dict(R=BASE + 0x50004, ldr=256)),
                    ('ldc_odd', dict(ldc=258)), ('ldr_odd', dict(R=BASE + 0x50000, ldr=258))]
        out += [('%s-ok-%s' % (name, n), variant(ops, **kw), 1) for n, kw in ok]
        out += [('%s-bad-%s' % (name, n), variant(ops, **kw), 0) for n, kw in bad]
    return out


CASES = cases()


def _build_module():
    spec = importlib.util.spec_from_file_location('_mvm_build', os.path.join(PKG, 'build.py'))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


@pytest.fixture(scope='module')
def verdicts(tmp_path_factory):
    b = _build_module()
    nvcc = b.NVCC if os.path.exists(b.NVCC) else shutil.which('nvcc')
    if not nvcc:
        pytest.skip('nvcc not available')
    d = tmp_path_factory.mktemp('gemm_args')
    src, exe = d / 'harness.cu', d / 'harness'
    src.write_text(HARNESS)
    r = subprocess.run([nvcc, '-std=c++17', '-I', os.path.join(PKG, 'csrc'), str(src), '-o', str(exe)],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    lines = '\n'.join(' '.join(str(c[1][f]) for f in FIELDS) for c in CASES) + '\n'
    out = subprocess.run([str(exe)], input=lines, capture_output=True, text=True, check=True).stdout.split()
    assert len(out) == len(CASES)
    return {c[0]: int(v) for c, v in zip(CASES, out)}


@pytest.mark.parametrize('name,expected', [(c[0], c[2]) for c in CASES], ids=[c[0] for c in CASES])
def test_gemm_desc_valid(verdicts, name, expected):
    assert verdicts[name] == expected, name
