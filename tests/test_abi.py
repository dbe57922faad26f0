"""C-ABI checks that need no GPU: the library loads, exports every symbol include/rih_b200.h declares, and the
header is in sync with the RIH_API definitions in csrc/ (tools/gen_header.py)."""
import ctypes
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_header_matches_sources():
    sys.path.insert(0, os.path.join(ROOT, 'tools'))
    import gen_header
    from renderih_b200 import _lib
    protos = _lib.parse_header()
    defs = {name: params for _, _, _, name, params in gen_header.extract()}
    assert set(protos) == set(defs), set(protos) ^ set(defs)
    for name, params in defs.items():
        n = 0 if params.strip() in ('', 'void') else len(params.split(','))
        assert n == len(protos[name][1]), name


def test_library_builds_and_exports_all_symbols():
    from renderih_b200 import _build, _lib
    path = _build.build()
    assert os.path.exists(path)
    lib = ctypes.CDLL(path)
    for name in _lib.parse_header():
        assert hasattr(lib, name), 'missing export %s' % name
    lib.rih_version.restype = ctypes.c_int
    assert lib.rih_version() >= 100
    out = subprocess.run(['nm', '-D', '--defined-only', path], stdout=subprocess.PIPE).stdout.decode()
    exported = set(re.findall(r' T (rih_\w+)', out))
    assert exported == set(_lib.parse_header()), exported ^ set(_lib.parse_header())


def test_sass_is_sm90a():
    from renderih_b200 import _build
    out = subprocess.run(['cuobjdump', '-lelf', _build.build()], stdout=subprocess.PIPE).stdout.decode()
    assert 'sm_90a' in out, out[:400]


def test_product_never_imports_oracle():
    for pkg in (os.path.join(ROOT, 'renderih_b200'), os.path.join(ROOT, 'tools')):     # only tests/, smoke() and bench.py's CPU legs may use oracle/
        for dirpath, _, files in os.walk(pkg):
            for f in files:
                if f.endswith('.py'):
                    text = open(os.path.join(dirpath, f)).read()
                    assert not re.search(r'^\s*(from|import)\s+oracle', text, re.M), f
