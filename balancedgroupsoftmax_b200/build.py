"""Build libbags_b200.so in-tree with nvcc for sm_90a (H100; cross-compiles without a GPU).

    python -m balancedgroupsoftmax_b200.build [--force] [--verbose]
"""
from __future__ import annotations

import os
import shutil
import subprocess
import sys

_HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(_HERE, 'csrc')
OUT = os.path.join(_HERE, 'libbags_b200.so')
SOURCES = [os.path.join(CSRC, 'bags_api.cu')]
HEADERS = [os.path.join(CSRC, f) for f in ('bags_ptx.cuh', 'bags_wgmma.cuh', 'bags_gemm.cuh', 'bags_kernels.cuh', 'bags_fused_fwd.cuh', 'bags_allreduce.cuh', 'bags_nms.cuh', 'bags_box.cuh', 'bags_mask.cuh', 'bags_segm.cuh', 'bags_mask_target.cuh')] + [
    os.path.join(os.path.dirname(_HERE), 'include', 'bags_b200.h')]

NVCC_FLAGS = [
    '-gencode', 'arch=compute_90a,code=sm_90a', '-lineinfo', '-O3', '-std=c++17',
    '-shared', '-Xcompiler', '-fPIC',
]


def _nvcc() -> str:
    for cand in (os.environ.get('NVCC', ''), shutil.which('nvcc') or '', '/usr/local/cuda/bin/nvcc'):
        if cand and os.path.isfile(cand):
            return cand
    raise RuntimeError('nvcc not found (set $NVCC)')


def is_stale() -> bool:
    if not os.path.isfile(OUT):
        return True
    t = os.path.getmtime(OUT)
    return any(os.path.getmtime(f) > t for f in SOURCES + HEADERS)


def build(force: bool = False, verbose: bool = False) -> str:
    if not force and not is_stale():
        return OUT
    cmd = [_nvcc()] + NVCC_FLAGS + (['-Xptxas', '-v'] if verbose else []) + ['-o', OUT] + SOURCES
    if verbose:
        print(' '.join(cmd))
    res = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if res.returncode != 0:
        raise RuntimeError('nvcc failed:\n' + res.stdout)
    if verbose:
        print(res.stdout)
    return OUT


if __name__ == '__main__':
    path = build(force='--force' in sys.argv, verbose='--verbose' in sys.argv)
    print(path)
