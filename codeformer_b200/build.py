"""Build libcfb200.so in-tree with nvcc for sm_90a (SASS only: wgmma needs the arch-specific target)."""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, 'csrc')
LIB = os.environ.get('CFB_BUILD_OUT') or os.path.join(HERE, 'libcfb200.so')
SOURCES = ['simt_kernels.cu', 'conv_tc.cu', 'runtime.cu', 'pasteback.cu', 'detection.cu', 'yolo.cu', 'arcface.cu', 'bisenet.cu', 'metrics.cu', 'lpips.cu', 'degrade.cu', 'fid.cu']
NVCC = os.environ.get('NVCC', '/usr/local/cuda/bin/nvcc')
FLAGS = ['-gencode', 'arch=compute_90a,code=sm_90a', '-O3', '-lineinfo', '-std=c++17', '-Xcompiler', '-fPIC',
         '-Wno-deprecated-gpu-targets', '-Xptxas', '-v' if os.environ.get('CFB_PTXAS_V') else '-O3'] + \
        os.environ.get('CFB_NVCC_EXTRA', '').split()       # e.g. -DCFB_TC_STAMPS=1


def needs_build():
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    deps = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith(('.cu', '.cuh'))] + \
           [os.path.join(HERE, '..', 'include', 'cfb200.h'), __file__]
    return any(os.path.getmtime(d) > t for d in deps)


def build(force=False, verbose=False):
    """Compile the translation units and link libcfb200.so.  Safe to call from several processes at once: the build
    runs under an exclusive file lock, objects go to a per-process directory and the library is published with os.replace
    (a concurrent CDLL never sees a half-written file)."""
    import fcntl
    import shutil
    import tempfile
    if not force and not needs_build():
        return LIB
    with open(os.path.join(HERE, '.build.lock'), 'w') as lock:
        fcntl.flock(lock, fcntl.LOCK_EX)
        try:
            if not force and not needs_build():      # another process built it while we waited for the lock
                return LIB
            tmp = tempfile.mkdtemp(prefix='cfb_build_', dir=CSRC)
            try:
                return _build_locked(tmp, verbose)
            finally:
                shutil.rmtree(tmp, ignore_errors=True)
        finally:
            fcntl.flock(lock, fcntl.LOCK_UN)


def _build_locked(objdir, verbose):
    objs = []
    procs = []
    for s in SOURCES:
        o = os.path.join(objdir, s.replace('.cu', '.o'))
        cmd = [NVCC] + FLAGS + ['-c', os.path.join(CSRC, s), '-o', o]
        if verbose:
            print(' '.join(cmd), flush=True)
        procs.append((s, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
        objs.append(o)
    fail = False
    for s, p in procs:
        out, _ = p.communicate()
        if p.returncode != 0 or verbose or os.environ.get('CFB_PTXAS_V'):
            print(out)
        fail = fail or p.returncode != 0
    if fail:
        raise RuntimeError('nvcc failed')
    staged = os.path.join(objdir, 'libcfb200.so')
    cmd = [NVCC, '-shared', '-Wno-deprecated-gpu-targets', '-o', staged] + objs + ['-lcudart']
    subprocess.check_call(cmd)
    os.replace(staged, LIB)
    return LIB


if __name__ == '__main__':
    print(build(force='--force' in sys.argv, verbose=True))
