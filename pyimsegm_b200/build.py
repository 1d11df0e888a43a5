"""
Build the CUDA extension ``libimsegm_b200.so`` in-tree with nvcc for sm_90a (H100).

The library exports the C-ABI of ``include/imsegm_b200.h``; Python binds it with ctypes (``_lib.py``).
``python -m pyimsegm_b200.build`` or ``__graft_entry__.build()``.
"""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, 'csrc')
LIB = os.path.join(HERE, 'libimsegm_b200.so')

ARCH = ['-gencode', 'arch=compute_90a,code=sm_90a']
# -fmad=false: the SLIC sources must reproduce the oracle's IEEE double arithmetic bit for bit
FLAGS = ['-O3', '-lineinfo', '-std=c++17', '-Xcompiler', '-fPIC', '-fmad=false']


def sources():
    return sorted(os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith('.cu'))


def needs_build():
    if not os.path.isfile(LIB):
        return True
    t = os.path.getmtime(LIB)
    deps = [os.path.join(CSRC, f) for f in os.listdir(CSRC)] + [os.path.join(HERE, '..', 'include', 'imsegm_b200.h')]
    return any(os.path.getmtime(d) > t for d in deps)


def build(force=False, verbose=False):
    if not force and not needs_build():
        return LIB
    nvcc = os.environ.get('NVCC', 'nvcc')
    objs = []
    build_dir = os.path.join(HERE, 'build')
    os.makedirs(build_dir, exist_ok=True)
    procs = []
    # any source may include any header, so an object is stale once it is older than its .cu or than the newest header
    headers = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith('.cuh')] + [os.path.join(HERE, '..', 'include', 'imsegm_b200.h')]
    newest_header = max(os.path.getmtime(h) for h in headers)
    for src in sources():
        obj = os.path.join(build_dir, os.path.basename(src)[:-3] + '.o')
        objs.append(obj)
        if (not force) and os.path.isfile(obj) and os.path.getmtime(obj) > max(os.path.getmtime(src), newest_header):
            continue
        cmd = [nvcc] + ARCH + FLAGS + (['-Xptxas', '-v'] if verbose else []) + ['-c', src, '-o', obj]
        procs.append((cmd, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT)))
    for cmd, p in procs:
        out, _ = p.communicate()
        if p.returncode != 0:
            sys.stderr.write(out.decode())
            raise RuntimeError('nvcc failed: %s' % ' '.join(cmd))
        if verbose:
            sys.stderr.write(out.decode())
    cmd = [nvcc] + ARCH + ['-shared', '-o', LIB] + objs + ['-lcudart']
    subprocess.check_call(cmd)
    return LIB


if __name__ == '__main__':
    print(build(force='--force' in sys.argv, verbose='-v' in sys.argv))
