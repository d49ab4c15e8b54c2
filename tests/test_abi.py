"""CPU: the C-ABI shared library loads and exports every function include/*.h declares."""
import ctypes
import glob
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def declared_functions():
    names = []
    for h in glob.glob(os.path.join(ROOT, 'include', '*.h')):
        src = open(h).read()
        src = re.sub(r'/\*.*?\*/', '', src, flags=re.S)
        names += re.findall(r'\b(mvm_[a-z0-9_]+)\s*\(', src)
    return sorted(set(names))


def test_library_exports_declared_symbols():
    from e2e_multi_view_matching_b200 import build, _lib
    build.build()
    lib = ctypes.CDLL(_lib.LIB_PATH)
    names = declared_functions()
    assert len(names) >= 8
    for n in names:
        assert hasattr(lib, n), 'missing symbol %s' % n
    lib.mvm_version.restype = ctypes.c_char_p
    assert b'sm_90a' in lib.mvm_version()


def test_struct_layout_matches_header():
    """sizeof of the ctypes mirrors must equal what the C compiler computes."""
    import subprocess, tempfile
    from e2e_multi_view_matching_b200 import _lib
    src = '#include <stdio.h>\n#include "mvm_b200.h"\nint main(){printf("%zu %zu %zu\\n", sizeof(mvm_layer_weights), sizeof(mvm_matcher_weights), sizeof(mvm_pair_io));return 0;}\n'
    with tempfile.TemporaryDirectory() as d:
        c = os.path.join(d, 'a.c')
        open(c, 'w').write(src)
        exe = os.path.join(d, 'a.out')
        subprocess.check_call(['gcc', '-I', os.path.join(ROOT, 'include'), c, '-o', exe])
        sizes = [int(x) for x in subprocess.check_output([exe]).split()]
    assert sizes == [ctypes.sizeof(_lib.LayerWeights), ctypes.sizeof(_lib.MatcherWeights),
                     ctypes.sizeof(_lib.PairIO)]


def test_product_never_imports_oracle():
    """The oracle is test infrastructure: nothing under the package may import it."""
    pkg = os.path.join(ROOT, 'e2e_multi_view_matching_b200')
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if f.endswith('.py'):
                src = open(os.path.join(dirpath, f)).read()
                assert not re.search(r'^\s*(from|import)\s+oracle\b', src, flags=re.M), f
