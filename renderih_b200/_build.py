"""In-tree build of the C-ABI CUDA library (sm_90a only).  `python -m renderih_b200._build` or `build()`.

The shared object is written next to this file (`renderih_b200/librih_b200.so`): it is git-ignored
but travels to the GPU box with the gpurun snapshot.  nvcc cross-compiles without a GPU.
"""
import hashlib
import os
import shutil
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, 'csrc')
LIB_PATH = os.path.join(HERE, 'librih_b200.so')
STAMP_PATH = os.path.join(HERE, 'csrc', '.build_stamp')
ARCH_FLAGS = ['-gencode', 'arch=compute_90a,code=sm_90a']


def _sources():
    return sorted(f for f in os.listdir(CSRC) if f.endswith('.cu'))


def _digest():
    h = hashlib.sha256()
    for f in sorted(os.listdir(CSRC)):
        if f.endswith(('.cu', '.cuh', '.h')):
            h.update(f.encode())
            with open(os.path.join(CSRC, f), 'rb') as fh:
                h.update(fh.read())
    inc = os.path.join(HERE, '..', 'include', 'rih_b200.h')
    if os.path.exists(inc):
        with open(inc, 'rb') as fh:
            h.update(fh.read())
    return h.hexdigest()


def needs_build():
    if not os.path.exists(LIB_PATH) or not os.path.exists(STAMP_PATH):
        return True
    with open(STAMP_PATH) as f:
        return f.read().strip() != _digest()


def have_nvcc():
    return os.path.exists(shutil.which('nvcc') or '/usr/local/cuda/bin/nvcc')


def build(force=False, verbose=False):
    """Compile every .cu under csrc/ into one shared library.  Returns the library path.
    Concurrent callers (the ranks of a torchrun launch) serialise on a file lock; the library is moved into place with an atomic rename."""
    if not force and not needs_build():
        return LIB_PATH
    import fcntl
    os.makedirs(os.path.join(HERE, 'csrc', 'build'), exist_ok=True)
    with open(os.path.join(HERE, 'csrc', 'build', '.lock'), 'w') as lock:
        fcntl.flock(lock, fcntl.LOCK_EX)
        try:
            if not force and not needs_build():      # another rank built it while we waited
                return LIB_PATH
            return _build_locked(verbose)
        finally:
            fcntl.flock(lock, fcntl.LOCK_UN)


def _build_locked(verbose):
    nvcc = shutil.which('nvcc') or '/usr/local/cuda/bin/nvcc'
    if not os.path.exists(nvcc):
        raise RuntimeError('nvcc not found: cannot build renderih_b200 CUDA library')
    objdir = os.path.join(HERE, 'csrc', 'build')
    os.makedirs(objdir, exist_ok=True)
    common = [nvcc] + ARCH_FLAGS + ['-O3', '-lineinfo', '-std=c++17', '-Xcompiler', '-fPIC,-fvisibility=hidden',
                                    '-I', CSRC, '-I', os.path.join(HERE, '..', 'include')]
    procs = []
    objs = []
    for src in _sources():
        obj = os.path.join(objdir, src[:-3] + '.o')
        objs.append(obj)
        cmd = common + ['-c', os.path.join(CSRC, src), '-o', obj]
        procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT)))
    for src, p in procs:
        out, _ = p.communicate()
        if verbose and out:
            sys.stderr.write(out.decode())
        if p.returncode != 0:
            raise RuntimeError('nvcc failed on %s:\n%s' % (src, out.decode()))
    tmp = LIB_PATH + '.tmp.%d' % os.getpid()
    cmd = [nvcc] + ARCH_FLAGS + ['-shared', '-o', tmp] + objs + ['-lcuda']
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT)
    if r.returncode != 0:
        raise RuntimeError('link failed:\n%s' % r.stdout.decode())
    os.replace(tmp, LIB_PATH)
    with open(STAMP_PATH, 'w') as f:
        f.write(_digest())
    return LIB_PATH


if __name__ == '__main__':
    print(build(force='--force' in sys.argv, verbose=True))
