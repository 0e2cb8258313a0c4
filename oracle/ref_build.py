"""Compile the reference's own CUDA NMS op (mmdet/ops/nms/src/nms_cuda.cpp + nms_kernel.cu) for sm_90a into
oracle/_ref/ -- TEST INFRASTRUCTURE.

The sources are compiled where they lie in the reference checkout (see ref_shim.reference_dir()); nothing is copied.
They were written against the THC runtime of torch 1.x, so oracle/ref_include/THC/ supplies the few THC names they
use on top of the CUDA runtime, and ``AT_CHECK`` is mapped to ``TORCH_CHECK``.  The result,
oracle/_ref/ref_nms_cuda*.so, is what oracle/ref_nms.py loads; it needs no reference checkout at run time.

    python -m oracle.ref_build
"""
from __future__ import annotations

import glob
import os
from typing import Optional

_HERE = os.path.dirname(os.path.abspath(__file__))
OUT_DIR = os.path.join(_HERE, '_ref')
INCLUDE = os.path.join(_HERE, 'ref_include')
NAME = 'ref_nms_cuda'


def built_library() -> Optional[str]:
    libs = sorted(glob.glob(os.path.join(OUT_DIR, NAME + '*.so')))
    return libs[0] if libs else None


def build(verbose: bool = False) -> Optional[str]:
    """Compile the reference NMS op; returns the library's path, or None when no reference checkout is reachable
    (an existing oracle/_ref/ is then left as it is)."""
    from oracle import ref_shim
    root = ref_shim.reference_dir()
    if root is None:
        return None
    src = os.path.join(root, 'mmdet', 'ops', 'nms', 'src')
    os.makedirs(OUT_DIR, exist_ok=True)
    from torch.utils import cpp_extension
    saved = os.environ.get('TORCH_CUDA_ARCH_LIST')
    os.environ['TORCH_CUDA_ARCH_LIST'] = '9.0a'
    try:
        cpp_extension.load(
            name=NAME, sources=[os.path.join(src, 'nms_cuda.cpp'), os.path.join(src, 'nms_kernel.cu')],
            extra_include_paths=[INCLUDE], extra_cflags=['-O2', '-DAT_CHECK=TORCH_CHECK'],
            extra_cuda_cflags=['-O2', '-DAT_CHECK=TORCH_CHECK'], build_directory=OUT_DIR, verbose=verbose,
            is_python_module=False)
    finally:
        if saved is None:
            os.environ.pop('TORCH_CUDA_ARCH_LIST', None)
        else:
            os.environ['TORCH_CUDA_ARCH_LIST'] = saved
    path = built_library()
    assert path is not None, 'reference NMS op did not build into %s' % OUT_DIR
    return path


if __name__ == '__main__':
    print(build(verbose=True))
