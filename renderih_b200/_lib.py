"""ctypes binding of the C-ABI CUDA library `librih_b200.so`; signatures are parsed from include/rih_b200.h.

There is NO fallback: if the library is missing or a call fails, a RuntimeError is raised.
"""
import ctypes
import os
import re

from . import _build

HEADER = os.path.join(os.path.dirname(os.path.abspath(__file__)), '..', 'include', 'rih_b200.h')
_PROTO_RE = re.compile(r'^\s*((?:const\s+)?[\w ]+?\*?)\s*\b(rih_\w+)\s*\(([^)]*)\)\s*;', re.M)


def _ctype(param):
    p = param.strip()
    if p in ('void', ''):
        return None
    if '*' in p:
        return ctypes.c_void_p
    t = ' '.join(p.split()[:-1])  # drop the parameter name
    t = t.replace('const ', '').strip()
    table = {'int': ctypes.c_int, 'float': ctypes.c_float, 'double': ctypes.c_double, 'long long': ctypes.c_longlong,
             'unsigned long long': ctypes.c_ulonglong, 'size_t': ctypes.c_size_t, 'cudaStream_t': ctypes.c_void_p,
             'unsigned int': ctypes.c_uint, 'uint32_t': ctypes.c_uint32}
    if t not in table:
        raise RuntimeError('rih_b200.h: unknown parameter type %r' % p)
    return table[t]


def parse_header(path=HEADER):
    """-> {name: (restype_str, [ctypes types])} for every prototype in the header."""
    text = open(path).read()
    text = re.sub(r'/\*.*?\*/', '', text, flags=re.S)
    text = re.sub(r'//[^\n]*', '', text)
    protos = {}
    for m in _PROTO_RE.finditer(text):
        ret, name, params = m.group(1).strip(), m.group(2), m.group(3)
        args = [_ctype(p) for p in params.split(',')]
        protos[name] = (ret, [a for a in args if a is not None])
        if params.split(',')[-1].strip().startswith('cudaStream_t'):
            STREAM_LAST.add(name)
    return protos


PDL_DEFAULT = '0'     # flipped to '1' once validated on hardware (A/B in bench.py)
STREAM_LAST = set()   # entry points whose last parameter is the CUDA stream to launch on (every kernel-launching one)
TRACE = None          # measurement hook (bench.py): when set to a list, every launching call is bracketed by CUDA events recorded on ITS stream
_lib = None
CALLS = [0]   # number of C-ABI kernel-launching calls issued by this process (bench.py reports it as gpu_launches)


def lib_path():
    return _build.LIB_PATH


def load():
    """Load (building first if the sources changed and nvcc is present). Raises if impossible."""
    global _lib
    if _lib is not None:
        return _lib
    path = _build.LIB_PATH
    if _build.needs_build():
        if _build.have_nvcc():
            _build.build()          # compile / link errors propagate: never run a stale library against a newer header
        elif not os.path.exists(path):
            raise RuntimeError('renderih_b200: CUDA library is not built and nvcc is not available here')
        # no nvcc (e.g. a deployment box): a prebuilt library is accepted only if its embedded source digest matches, checked below
    if not os.path.exists(path):
        raise RuntimeError('renderih_b200: %s missing -- run `python -m renderih_b200._build`' % path)
    lib = ctypes.CDLL(path)
    for name, (ret, args) in parse_header().items():
        if not hasattr(lib, name):
            raise RuntimeError('renderih_b200: %s does not export %s (stale library? rebuild with `python -m renderih_b200._build --force`)' % (path, name))
        fn = getattr(lib, name)  # AttributeError here == header/library mismatch: fail loudly
        fn.restype = ctypes.c_char_p if 'char' in ret else ctypes.c_int
        fn.argtypes = args
    _lib = lib
    # programmatic dependent launch for every kernel (csrc/common.cuh); RIH_PDL=0 selects plain stream-ordered launches
    lib.rih_set_pdl(1 if os.environ.get('RIH_PDL', PDL_DEFAULT) != '0' else 0)
    return lib


def call(name, *args):
    """Invoke a C-ABI entry point; raise RuntimeError(rih_last_error()) on a non-zero status."""
    lib = _lib if _lib is not None else load()
    CALLS[0] += 1
    if TRACE is not None and name in STREAM_LAST:
        import torch
        st = torch.cuda.ExternalStream(args[-1]) if args[-1] else torch.cuda.default_stream()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(st)
        rc = getattr(lib, name)(*args)
        e1.record(st)
        TRACE.append((name, args, e0, e1))
    else:
        rc = getattr(lib, name)(*args)
    if rc != 0:
        raise RuntimeError('%s failed (status %d): %s' % (name, rc, lib.rih_last_error().decode()))
