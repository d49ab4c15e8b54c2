"""Build libmvm_b200.so (all CUDA kernels + the C ABI) for sm_90a with nvcc, in-tree.

Usage: python -m e2e_multi_view_matching_b200.build [--force]
The shared library is written next to this file so that it travels to the GPU box with the
repo snapshot.  No torch headers are involved: the boundary is a plain C ABI (include/mvm_b200.h).
"""
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, 'csrc')
LIB = os.path.join(HERE, 'libmvm_b200.so')
NVCC = os.environ.get('NVCC', '/usr/local/cuda/bin/nvcc')
FLAGS = ['-gencode', 'arch=compute_90a,code=sm_90a', '-O3', '-lineinfo', '-std=c++17',
         '-Xcompiler', '-fPIC', '--expt-relaxed-constexpr']


def _sources():
    return sorted(f for f in os.listdir(CSRC) if f.endswith('.cu'))


def _needs_build():
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    deps = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if not f.endswith('.o') and f != 'cli']
    deps.append(os.path.join(os.path.dirname(HERE), 'include', 'mvm_b200.h'))
    return any(os.path.getmtime(d) > t for d in deps)


def _compile(src, verbose):
    obj = os.path.join(CSRC, src[:-3] + '.o')
    cmd = [NVCC] + FLAGS + (['-Xptxas', '-v'] if verbose else []) + ['-c', os.path.join(CSRC, src), '-o', obj]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError('nvcc failed for %s:\n%s\n%s' % (src, r.stdout, r.stderr))
    return obj, r.stderr


BIN = os.path.join(HERE, 'bin')
CLI_SRC = os.path.join(CSRC, 'cli', 'ba_cli.cpp')
CLI = {'bundle_adjuster': [], 'ba_initializer': ['-DMVM_CLI_BA_INIT']}


def build_cli(force=False):
    """The two CLI-compatible binaries (same names and file protocol as the reference's
    bundle_adjustment/build/{bundle_adjuster,ba_initializer}) on top of libmvm_b200.so."""
    os.makedirs(BIN, exist_ok=True)
    for name, defs in CLI.items():
        out = os.path.join(BIN, name)
        if not force and os.path.exists(out) and os.path.getmtime(out) > max(os.path.getmtime(CLI_SRC), os.path.getmtime(LIB)):
            continue
        cmd = [NVCC, '-O2', '-std=c++17'] + defs + ['-o', out, CLI_SRC, '-L' + HERE, '-lmvm_b200',
                                                     '-Xlinker', '-rpath', '-Xlinker', '$ORIGIN/..']
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError('CLI build failed for %s:\n%s\n%s' % (name, r.stdout, r.stderr))
    return BIN


def build(force=False, verbose=False):
    if not force and not _needs_build():
        build_cli()
        return LIB
    srcs = _sources()
    with ThreadPoolExecutor(max_workers=min(8, len(srcs))) as ex:
        results = list(ex.map(lambda s: _compile(s, verbose), srcs))
    if verbose:
        for (_, log), s in zip(results, srcs):
            print('==', s)
            print(log)
    objs = [o for o, _ in results]
    cmd = [NVCC, '-shared', '-gencode', 'arch=compute_90a,code=sm_90a', '-o', LIB] + objs + ['-lcuda']
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError('link failed:\n%s\n%s' % (r.stdout, r.stderr))
    build_cli(force=True)
    return LIB


if __name__ == '__main__':
    print(build(force='--force' in sys.argv, verbose='-v' in sys.argv))
