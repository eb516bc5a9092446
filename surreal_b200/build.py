"""Build libsurreal_b200.so in-tree with nvcc for sm_90a (no torch headers: pure C-ABI)."""
import glob
import hashlib
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, 'csrc')
LIB = os.path.join(HERE, 'libsurreal_b200.so')
STAMP = LIB + '.stamp'      # source digest the .so was built from: git-ignored, travels with the .so to the GPU box
NVCC = os.environ.get('NVCC', '/usr/local/cuda/bin/nvcc')
FLAGS = ['-gencode', 'arch=compute_90a,code=sm_90a', '-lineinfo', '-O3', '-std=c++17',
         '-Xcompiler', '-fPIC', '--expt-relaxed-constexpr', '-Xptxas', '-v']


def _sources():
    return sorted(glob.glob(os.path.join(CSRC, '*.cu')))


def _digest():
    h = hashlib.sha256()
    files = _sources() + sorted(glob.glob(os.path.join(CSRC, '*.cuh'))) + \
        [os.path.join(HERE, '..', 'include', 'surreal_b200.h'), os.path.abspath(__file__)]
    for f in files:
        with open(f, 'rb') as fp:
            h.update(fp.read())
    return h.hexdigest()


def build(force=False, verbose=False):
    """Compile every .cu into objects (parallel) and link one shared library.  Returns the .so path."""
    dig = _digest()
    if not force and os.path.exists(LIB) and os.path.exists(STAMP) and open(STAMP).read().strip() == dig:
        return LIB
    if not os.path.exists(NVCC):
        raise RuntimeError('nvcc not found at %s: cannot build libsurreal_b200.so' % NVCC)
    objdir = os.path.join(HERE, 'build')
    os.makedirs(objdir, exist_ok=True)
    procs = []
    for src in _sources():
        obj = os.path.join(objdir, os.path.basename(src)[:-3] + '.o')
        cmd = [NVCC] + FLAGS + ['-c', src, '-o', obj]
        procs.append((src, obj, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
    objs, log = [], []
    for src, obj, pr in procs:
        out, _ = pr.communicate()
        log.append('== %s\n%s' % (os.path.basename(src), out))
        if pr.returncode != 0:
            sys.stderr.write(out)
            raise RuntimeError('nvcc failed on %s' % src)
        objs.append(obj)
    with open(os.path.join(objdir, 'ptxas.log'), 'w') as fp:
        fp.write('\n'.join(log))
    if verbose:
        print('\n'.join(log))
    subprocess.check_call([NVCC, '-shared'] + FLAGS[:2] + ['-o', LIB] + objs + ['-lcudart'])
    with open(STAMP, 'w') as fp:
        fp.write(dig)
    return LIB


if __name__ == '__main__':
    print(build(force='--force' in sys.argv, verbose='-v' in sys.argv))
