"""Builds libpgt_b200.so (all hand-written sm_90a kernels + the C ABI) in-tree with nvcc.

nvcc cross-compiles without a GPU; the .so is git-ignored and rebuilt whenever a source, the
header or the flags change.  `python -m pgtformer_b200.build [--force]`.
"""
import hashlib
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, 'csrc')
LIB_DIR = os.path.join(HERE, 'lib')
LIB_PATH = os.path.join(LIB_DIR, 'libpgt_b200.so')
STAMP = os.path.join(LIB_DIR, 'build.stamp')
NVCC = os.environ.get('NVCC', '/usr/local/cuda/bin/nvcc')
ARCH = ['-gencode', 'arch=compute_90a,code=sm_90a']          # H100 (Hopper): wgmma, TMA, mbarrier
FLAGS = ARCH + ['-lineinfo', '-O3', '-std=c++17',
         '-Xcompiler', '-fPIC', '--expt-relaxed-constexpr']


TORCH_SRC = os.path.join(HERE, 'csrc_torch', 'pgt_torch_ops.cpp')
TORCH_LIB_PATH = os.path.join(LIB_DIR, 'libpgt_torch.so')
TORCH_STAMP = os.path.join(LIB_DIR, 'build_torch.stamp')


def build_torch_shim(force=False):
    """Builds lib/libpgt_torch.so: the TORCH_LIBRARY shim (`torch.ops.pgt.*`) over the C ABI.  Plain g++ — the shim
    contains no device code — against the installed PyTorch's headers, linked to libpgt_b200.so next to it."""
    import sysconfig

    import torch
    from torch.utils import cpp_extension as ce
    h = hashlib.sha256()
    for f in (TORCH_SRC, os.path.join(os.path.dirname(HERE), 'include', 'pgt_b200.h')):
        with open(f, 'rb') as fh:
            h.update(fh.read())
    h.update(torch.__version__.encode())
    fp = h.hexdigest()
    if not force and os.path.exists(TORCH_LIB_PATH) and os.path.exists(TORCH_STAMP) and open(TORCH_STAMP).read() == fp:
        return TORCH_LIB_PATH
    cxx = os.environ.get('CXX', 'g++')
    import shutil
    if shutil.which(cxx) is None:
        if os.path.exists(TORCH_LIB_PATH):
            return TORCH_LIB_PATH
        raise RuntimeError('no C++ compiler for the TORCH_LIBRARY shim')
    inc = ce.include_paths() + [sysconfig.get_paths()['include'], '/usr/local/cuda/include']
    cmd = [cxx, '-O2', '-std=c++17', '-fPIC', '-shared', '-D_GLIBCXX_USE_CXX11_ABI=%d' % int(torch._C._GLIBCXX_USE_CXX11_ABI),
           TORCH_SRC, '-o', TORCH_LIB_PATH]
    for i in inc:
        cmd += ['-I', i]
    for lp in ce.library_paths():
        cmd += ['-L', lp, '-Wl,-rpath,' + lp]
    cmd += ['-L', LIB_DIR, '-Wl,-rpath,$ORIGIN', '-lpgt_b200', '-lc10', '-lc10_cuda', '-ltorch_cpu', '-ltorch_cuda', '-ltorch']
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if r.returncode != 0:
        raise RuntimeError('TORCH_LIBRARY shim build failed:\n' + r.stdout[-4000:])
    with open(TORCH_STAMP, 'w') as fh:
        fh.write(fp)
    return TORCH_LIB_PATH


def _sources():
    return sorted(os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith('.cu'))


def _fingerprint():
    h = hashlib.sha256()
    inc = os.path.join(os.path.dirname(HERE), 'include', 'pgt_b200.h')
    for f in sorted(os.listdir(CSRC)):
        with open(os.path.join(CSRC, f), 'rb') as fh:
            h.update(f.encode() + fh.read())
    with open(inc, 'rb') as fh:
        h.update(fh.read())
    h.update(' '.join(FLAGS).encode())
    return h.hexdigest()


def build(force=False, verbose=False):
    os.makedirs(LIB_DIR, exist_ok=True)
    fp = _fingerprint()
    if not force and os.path.exists(LIB_PATH) and os.path.exists(STAMP) and open(STAMP).read() == fp:
        return LIB_PATH
    if not os.path.exists(NVCC):
        # a library from other sources or flags must not be loaded in place of these kernels
        raise RuntimeError('nvcc not found at %s and %s is missing or was built from other sources' % (NVCC, LIB_PATH))
    objs = []
    procs = []
    for src in _sources():
        obj = os.path.join(LIB_DIR, os.path.basename(src)[:-3] + '.o')
        objs.append(obj)
        cmd = [NVCC] + FLAGS + (['-Xptxas', '-v'] if verbose else []) + ['-c', src, '-o', obj]
        procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
    for src, p in procs:
        out, _ = p.communicate()
        if p.returncode != 0:
            raise RuntimeError('nvcc failed for %s:\n%s' % (src, out))
        if verbose:
            sys.stderr.write(out)
    link = [NVCC, '-shared', '-o', LIB_PATH] + objs + ARCH + ['-lcudart']
    r = subprocess.run(link, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if r.returncode != 0:
        raise RuntimeError('link failed:\n' + r.stdout)
    for o in objs:
        os.remove(o)
    with open(STAMP, 'w') as fh:
        fh.write(fp)
    return LIB_PATH


if __name__ == '__main__':
    print(build(force='--force' in sys.argv, verbose='-v' in sys.argv))
    if '--torch' in sys.argv:
        print(build_torch_shim(force='--force' in sys.argv))
