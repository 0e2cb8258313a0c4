"""The reference's own CUDA RoIAlign op (mmdet/ops/roi_align/src/roi_align_cuda.cpp + roi_align_kernel.cu), compiled
for sm_90a into oracle/_ref/ref_roi_align_cuda*.so, and its loader -- TEST INFRASTRUCTURE.

build() compiles the sources where they lie in the reference checkout (ref_shim.reference_dir()), as
oracle/ref_build.py does for the NMS op: the THC shim of oracle/ref_include and ``AT_CHECK`` mapped to
``TORCH_CHECK``.  The kernel uses ``THCudaCheck`` without including THC/THC.h, so that header is force-included into
it (its THC/THCAtomics.cuh still ships with torch).  The loader reads nothing but oracle/_ref/, so it works without a
reference checkout.

The op launches on the legacy default stream, not torch's current stream: the wrappers synchronise around it.

    forward(features, rois, out_h, out_w, spatial_scale, sample_num) -> [k, C, out_h, out_w]  (roi_align_cuda.forward)
    backward(gout, rois, spatial_scale, sample_num, feature_shape)   -> [B, C, H, W]          (roi_align_cuda.backward)

    python -m oracle.ref_roi_align
"""
from __future__ import annotations

import glob
import importlib.machinery
import importlib.util
import os
from typing import Optional

NAME = 'ref_roi_align_cuda'
_mod = None


def _path() -> Optional[str]:
    from oracle.ref_build import OUT_DIR
    libs = sorted(glob.glob(os.path.join(OUT_DIR, NAME + '*.so')))
    return libs[0] if libs else None


def build(verbose: bool = False) -> Optional[str]:
    """Compile the reference RoIAlign op; returns the library's path, or None when no reference checkout is reachable
    (an existing oracle/_ref/ is then left as it is)."""
    from oracle import ref_shim
    from oracle.ref_build import INCLUDE, OUT_DIR
    root = ref_shim.reference_dir()
    if root is None:
        return None
    src = os.path.join(root, 'mmdet', 'ops', 'roi_align', 'src')
    os.makedirs(OUT_DIR, exist_ok=True)
    from torch.utils import cpp_extension
    saved = os.environ.get('TORCH_CUDA_ARCH_LIST')
    os.environ['TORCH_CUDA_ARCH_LIST'] = '9.0a'
    try:
        cpp_extension.load(
            name=NAME, sources=[os.path.join(src, 'roi_align_cuda.cpp'), os.path.join(src, 'roi_align_kernel.cu')],
            extra_include_paths=[INCLUDE], extra_cflags=['-O2', '-DAT_CHECK=TORCH_CHECK'],
            extra_cuda_cflags=['-O2', '-DAT_CHECK=TORCH_CHECK', '-include', 'THC/THC.h'], build_directory=OUT_DIR,
            verbose=verbose, is_python_module=False)
    finally:
        if saved is None:
            os.environ.pop('TORCH_CUDA_ARCH_LIST', None)
        else:
            os.environ['TORCH_CUDA_ARCH_LIST'] = saved
    path = _path()
    assert path is not None, 'reference RoIAlign op did not build into %s' % OUT_DIR
    return path


def available() -> bool:
    return _path() is not None


def _load():
    global _mod
    if _mod is None:
        import torch  # noqa: F401  (the extension links against libtorch)
        path = _path()
        if path is None:
            raise RuntimeError('reference RoIAlign op not built (python -m oracle.ref_roi_align)')
        loader = importlib.machinery.ExtensionFileLoader('ref_roi_align_cuda', path)
        spec = importlib.util.spec_from_file_location('ref_roi_align_cuda', path, loader=loader)
        mod = importlib.util.module_from_spec(spec)
        loader.exec_module(mod)
        _mod = mod
    return _mod


def forward(features, rois, out_h: int, out_w: int, spatial_scale: float, sample_num: int):
    """RoIAlignFunction.forward (mmdet/ops/roi_align/roi_align.py): fp32 contiguous CUDA features [B, C, H, W] and
    rois [k, 5] -> [k, C, out_h, out_w]."""
    import torch
    out = features.new_zeros(rois.shape[0], features.shape[1], out_h, out_w)
    if rois.shape[0] == 0:
        return out
    torch.cuda.synchronize()
    _load().forward(features, rois, out_h, out_w, float(spatial_scale), int(sample_num), out)
    torch.cuda.synchronize()
    return out


def backward(gout, rois, spatial_scale: float, sample_num: int, feature_shape):
    """RoIAlignFunction.backward: the op's atomicAdd scatter of gout [k, C, out_h, out_w] into zeros of
    ``feature_shape``."""
    import torch
    grad = torch.zeros(tuple(feature_shape), dtype=torch.float32, device=gout.device)
    if rois.shape[0] == 0:
        return grad
    torch.cuda.synchronize()
    _load().backward(gout.contiguous(), rois, gout.shape[2], gout.shape[3], float(spatial_scale), int(sample_num), grad)
    torch.cuda.synchronize()
    return grad


if __name__ == '__main__':
    print(build(verbose=True))
