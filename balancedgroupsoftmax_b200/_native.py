"""ctypes binding of libbags_b200.so (C ABI declared in include/bags_b200.h).

There is no fallback: if the shared library is missing, or the device is not a
H100 (sm_90), every op raises.  Build it with ``python -m
balancedgroupsoftmax_b200.build`` (or ``__graft_entry__.build()``).
"""
from __future__ import annotations

import ctypes as C
import os
import threading
from typing import Optional

_HERE = os.path.dirname(os.path.abspath(__file__))
# BAGS_LIB: development hook to A/B two builds of the same ABI inside one GPU session
LIB_PATH = os.environ.get('BAGS_LIB') or os.path.join(_HERE, 'libbags_b200.so')

ABI_VERSION = 2
DTYPE_F32 = 0
DTYPE_BF16 = 1
WEIGHTS_U8 = 0
WEIGHTS_F32 = 1
MAX_BINS = 8
MASK_TILE = 64          # BAGS_MASK_TILE: pixels per tile of bags_mask_fwd's rsum scratch

_lib = None
_lock = threading.Lock()

_vp, _ll, _i, _sz = C.c_void_p, C.c_longlong, C.c_int, C.c_size_t

# symbol -> (restype, argtypes); mirrors include/bags_b200.h one to one
SIGNATURES = {
    'bags_abi_version': (_i, []),
    'bags_last_error': (C.c_char_p, []),
    'bags_workspace_bytes': (_sz, []),
    'bags_sample_others': (_i, [_vp, _vp, _i, _i, _i, C.c_double, C.c_uint64, _vp, _vp, _vp, _vp]),
    'bags_mask_avg': (_i, [_vp, _i, _i, _vp, _vp]),
    'bags_group_ce': (_i, [_vp, _ll, _vp, _vp, _vp, _vp, _i, _vp, _i, _i, _i, _i, _vp, _vp, _vp, _ll, _i, _vp,
                           _vp, _sz, _vp]),
    'bags_fused_eligible': (_i, [_vp, _i, _i]),
    'bags_fwd': (_i, [_vp, _ll, _vp, _ll, _vp, _vp, _vp, _vp, _vp, _i, _vp, _i, _i, _i, _i, _i, _i, _vp, _ll,
                      _vp, _vp, _vp, _ll, _vp, _i, _vp, _sz, _vp, _sz, _vp]),
    'bags_ce_fwd': (_i, [_vp, _ll, _vp, _ll, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _vp, _vp, _vp, _ll, _vp, _i, _vp, _sz,
                         _vp, _sz, _vp]),
    'bags_focal_fwd': (_i, [_vp, _ll, _vp, _ll, _vp, _vp, _vp, _vp, C.c_float, C.c_float, C.c_float, _i, _i, _i, _i,
                            _vp, _vp, _vp, _ll, _vp, _i, _vp, _sz, _vp, _sz, _vp]),
    'bags_box_fwd': (_i, [_vp, _ll, _i, _vp, _ll, _vp, _vp, _vp, _vp, C.c_float, C.c_float, _i, _i, _i, _vp, _vp, _vp,
                          _vp, _vp, _sz, _vp]),
    'bags_box_bwd': (_i, [_vp, _vp, _vp, _ll, _i, _vp, _ll, _vp, _vp, _i, _i, _i, _vp, _ll, _vp, _vp, _ll, _vp]),
    'bags_mask_fwd': (_i, [_vp, _i, _vp, _ll, _vp, _vp, _vp, _i, _i, _i, _i, _vp, _vp, _vp, _sz, _vp, _vp, _sz,
                           _vp]),
    'bags_mask_bwd': (_i, [_vp, _vp, _vp, _i, _vp, _ll, _vp, _vp, _i, _i, _i, _i, _vp, _ll, _vp, _vp, _vp]),
    'bags_mask_logits': (_i, [_vp, _i, _vp, _ll, _vp, _vp, _i, _i, _i, _i, _vp, _vp]),
    'bags_reweight': (_i, [_vp, _vp, _vp, _vp, _i, _i, _i, _i, _vp, _vp, _vp]),
    'bags_bwd_scratch_bytes': (_sz, [_i, _ll, _i]),
    'bags_bwd': (_i, [_vp, _ll, _vp, _ll, _vp, _ll, _vp, _vp, _vp, _i, _vp, _ll, _vp, _vp, _ll, _vp, _sz, _i, _i,
                      _i, _i, _i, _i, _vp]),
    'bags_merge_scores': (_i, [_vp, _ll, _vp, _vp, _i, _i, _i, _i, _vp, _ll, _vp]),
    'bags_grad_allreduce_flag_bytes': (_sz, [_i]),
    'bags_grad_allreduce_status_offset': (_ll, [_i]),
    'bags_grad_allreduce': (_i, [_vp, _vp, _ll, _ll, _i, _i, C.c_float, _i, _vp]),
    'bags_class_nms_dense': (_i, [_vp, _i, _vp, _vp, _i, _i, C.c_float, _vp, _vp, _vp]),
    'bags_segm_rle': (_i, [_vp, _i, _i, _i, _vp, _vp, _i, _i, C.c_double, _vp, _vp, _vp]),
    'bags_mask_target': (_i, [_vp, _vp, _vp, _vp, _i, _i, _i, _vp, _vp]),
    'bags_roi_align_fwd': (_i, [_vp, _vp, _vp, _i, _i, _i, _vp, _vp, _i, _i, _i, _i, C.c_float, _vp, _vp, _vp]),
    'bags_roi_align_bwd': (_i, [_vp, _vp, _vp, _vp, _i, _i, _i, _vp, _vp, _i, _i, _i, _i, C.c_float, _vp]),
    'bags_rpn_proposals': (_i, [_vp, _vp, _vp, _vp, _i, _i, _vp, _i, _i, _i, C.c_float, C.c_float, _vp, _vp, _vp, _sz,
                                _vp, _vp, _vp]),
    'bags_rpn_scratch_bytes': (_i, [_vp, _i, _i, _i, _i, _vp]),
    'bags_anchor_target': (_i, [_vp, _vp, _i, _i, _vp, _vp, _i, C.c_float, _i, C.c_float, C.c_float, C.c_float, _i,
                                C.c_double, _i, C.c_double, C.c_double, C.c_float, _vp, _vp, C.c_uint64, _vp, _vp,
                                _sz, _vp, _vp, _vp, _vp, _vp, _vp]),
    'bags_anchor_target_scratch_bytes': (_i, [_vp, _i, _i, _i, _vp]),
    'bags_debug_spin': (_i, [_i, _i, _i, _vp]),
    'bags_cast_bf16': (_i, [_vp, _ll, _vp, _ll, _i, _i, _vp]),
    'bags_linear_act_fwd': (_i, [_vp, _ll, _vp, _ll, _vp, _vp, _ll, _i, _i, _i, _i, _i, _i, _vp]),
    'bags_linear_act_splits': (_i, [_i, _i, _i, _i]),
    'bags_linear_act_fwd_splitk': (_i, [_vp, _ll, _vp, _ll, _vp, _vp, _ll, _i, _i, _i, _i, _i, _i, _vp, _ll, _i, _vp]),
    'bags_act_bwd': (_i, [_vp, _ll, _i, _vp, _ll, _i, _vp, _ll, _i, _i, _i, _vp]),
    'bags_debug_set_timing': (_i, [_vp]),
    'bags_reload_env': (_i, []),
    'bags_gemm_probe': (_i, [_vp, _ll, _i, _vp, _ll, _i, _vp, _ll, _i, _i, _i, _i, _i, _i, _i, _vp]),
}


class BagsNativeError(RuntimeError):
    pass


def lib():
    """Load (once) and return the ctypes handle.  Raises if the library is absent."""
    global _lib
    if _lib is not None:
        return _lib
    with _lock:
        if _lib is not None:
            return _lib
        if not os.path.isfile(LIB_PATH):
            raise BagsNativeError(
                'libbags_b200.so not found at %s -- the BAGS head has no CPU/PyTorch fallback; '
                'build the CUDA extension first (python -m balancedgroupsoftmax_b200.build)' % LIB_PATH)
        handle = C.CDLL(LIB_PATH)
        for name, (res, args) in SIGNATURES.items():
            fn = getattr(handle, name)
            fn.restype = res
            fn.argtypes = args
        ver = handle.bags_abi_version()
        if ver != ABI_VERSION:
            raise BagsNativeError('libbags_b200.so ABI version %d != expected %d' % (ver, ABI_VERSION))
        _lib = handle
        return _lib


def reload_env() -> None:
    """Make the library re-read its BAGS_* environment switches (they are cached after first use)."""
    lib().bags_reload_env()


def check(rc: int, what: str) -> None:
    if rc != 0:
        msg = lib().bags_last_error()
        raise BagsNativeError('%s failed (code %d): %s' % (what, rc, msg.decode('utf-8', 'replace') if msg else ''))


def ptr(t) -> Optional[int]:
    """Device pointer of a torch tensor (None -> NULL)."""
    return None if t is None else t.data_ptr()


def int32_array(values):
    arr = (C.c_int32 * len(values))(*[int(v) for v in values])
    return arr
