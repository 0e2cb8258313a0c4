"""The reference's compiled CUDA NMS op (mmdet/ops/nms), as oracle/ref_build.py left it in oracle/_ref/ -- TEST
INFRASTRUCTURE.  Reads nothing but oracle/_ref/, so it works without a reference checkout.

    nms(dets, iou_thr) -> kept indices (int64, CPU), ascending -- what ``nms_cuda.nms`` returns
    nms_wrapper_op(dets, iou_thr) -> (dets[inds], inds)          -- what bbox_nms.py calls as ``nms_wrapper.nms``
"""
from __future__ import annotations

import importlib.machinery
import importlib.util
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
_mod = None


def _path():
    from oracle.ref_build import built_library
    return built_library()


def available() -> bool:
    return _path() is not None


def _load():
    global _mod
    if _mod is None:
        import torch  # noqa: F401  (the extension links against libtorch)
        path = _path()
        if path is None:
            raise RuntimeError('reference NMS op not built (python -m oracle.ref_build)')
        loader = importlib.machinery.ExtensionFileLoader('ref_nms_cuda', path)
        spec = importlib.util.spec_from_file_location('ref_nms_cuda', path, loader=loader)
        mod = importlib.util.module_from_spec(spec)
        loader.exec_module(mod)
        _mod = mod
    return _mod


def nms(dets, iou_thr: float):
    """dets [n, 5] fp32 CUDA (x1, y1, x2, y2, score) -> indices of the kept rows, ascending (the op's own order)."""
    return _load().nms(dets, float(iou_thr))


def nms_wrapper_op(dets, iou_thr: float):
    """mmdet/ops/nms/nms_wrapper.py:nms for a CUDA tensor: (dets[inds], inds)."""
    import torch
    inds = dets.new_zeros(0, dtype=torch.long) if dets.shape[0] == 0 else nms(dets, iou_thr)
    return dets[inds.to(dets.device), :], inds
