"""Builds libvp_b200.so (hand-written sm_90a kernels + C ABI) in-tree with nvcc.

The .so and its object files are git-ignored build products; the product path never falls back
to anything else when the library is missing (video_prediction_b200/lib.py raises)."""
from __future__ import annotations

import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
CSRC = os.path.join(HERE, 'csrc')
LIB_PATH = os.path.join(HERE, 'libvp_b200.so')
SOURCES = ['api.cu', 'igemm.cu', 'pack.cu', 'elementwise.cu', 'backward.cu', 'discrim.cu', 'planes.cu', 'd0_layer.cu']
ARCH = ['-gencode', 'arch=compute_90a,code=sm_90a']
NVCC_FLAGS = ARCH + ['-O3', '-lineinfo', '-std=c++17',
                     '-Xcompiler', '-fPIC', '--use_fast_math', '-Xptxas', '-v',
                     '-I', os.path.join(ROOT, 'include'), '-I', CSRC]


def _nvcc():
    for cand in (os.environ.get('NVCC'), '/usr/local/cuda/bin/nvcc', 'nvcc'):
        if cand and (os.path.isabs(cand) and os.path.exists(cand) or not os.path.isabs(cand)):
            return cand
    return 'nvcc'


HASH_PATH = os.path.join(HERE, 'libvp_b200.srchash')


def source_hash():
    """Content hash of everything the library is built from (mtimes do not survive the snapshot copy to a GPU box)."""
    import hashlib
    h = hashlib.sha256(' '.join(NVCC_FLAGS[:-4]).encode())
    deps = sorted(os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith(('.cu', '.cuh', '.h')))
    deps.append(os.path.join(ROOT, 'include', 'vp_b200.h'))
    for d in deps:
        h.update(os.path.basename(d).encode())
        with open(d, 'rb') as f:
            h.update(f.read())
    return h.hexdigest()


def needs_build():
    if not os.path.exists(LIB_PATH) or not os.path.exists(HASH_PATH):
        return True
    with open(HASH_PATH) as f:
        return f.read().strip() != source_hash()


def _compile(s):
    o = s[:-3] + '.o'
    cmd = [_nvcc()] + NVCC_FLAGS + ['-c', s, '-o', o]
    return s, o, subprocess.run(cmd, capture_output=True, text=True)


def build(force=False, verbose=False):
    if not force and not needs_build():
        return LIB_PATH
    from concurrent.futures import ThreadPoolExecutor
    srcs = [os.path.join(CSRC, s) for s in SOURCES if os.path.exists(os.path.join(CSRC, s))]
    objs = []
    with ThreadPoolExecutor(max_workers=min(8, len(srcs))) as ex:
        for s, o, r in ex.map(_compile, srcs):
            if verbose or r.returncode:
                sys.stderr.write(r.stdout + r.stderr)
            if r.returncode:
                raise RuntimeError('nvcc failed on %s' % s)
            objs.append(o)
    cmd = [_nvcc(), '-shared', '-o', LIB_PATH] + objs + ARCH
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode:
        sys.stderr.write(r.stdout + r.stderr)
        raise RuntimeError('link failed')
    with open(HASH_PATH, 'w') as f:
        f.write(source_hash())
    return LIB_PATH


if __name__ == '__main__':
    print(build(force='--force' in sys.argv, verbose=True))
