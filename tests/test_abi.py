"""CPU: the C-ABI shared library loads and exports every symbol include/bags_b200.h declares;
argument validation that needs no GPU returns error codes + messages (never throws)."""
import ctypes as C
import os
import re

import pytest

from balancedgroupsoftmax_b200 import _native as nat

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, 'include', 'bags_b200.h')


def _declared():
    src = open(HEADER).read()
    src = re.sub(r'/\*.*?\*/', '', src, flags=re.S)
    return sorted(set(re.findall(r'\b(bags_[a-z0-9_]+)\s*\(', src)))


def test_header_symbols_exported():
    lib = nat.lib()
    names = _declared()
    assert len(names) >= 12
    for n in names:
        assert hasattr(lib, n), n
    assert sorted(nat.SIGNATURES.keys()) == names, 'ctypes SIGNATURES out of sync with the header'


def test_abi_version_2_and_workspace():
    lib = nat.lib()
    assert lib.bags_abi_version() == nat.ABI_VERSION == 2
    assert lib.bags_workspace_bytes() >= 4096


def test_invalid_arguments_return_error_codes():
    """Bad shapes, dtypes, workspaces and bin tables through the single-entry-point signatures: error codes and
    messages, never exceptions."""
    lib = nat.lib()
    # NULL operands
    rc = lib.bags_linear_act_fwd(None, 0, None, 0, None, None, 0, 4, 8, 8, nat.DTYPE_BF16, nat.DTYPE_F32, 0, None)
    assert rc == -1 and b'NULL' in lib.bags_last_error()
    # bad dtype
    buf = (C.c_char * 64)()
    p = C.addressof(buf)
    rc = lib.bags_linear_act_fwd(p, 8, p, 8, None, p, 8, 4, 8, 8, 7, nat.DTYPE_F32, 0, None)
    assert rc == -1 and b'dtype' in lib.bags_last_error()
    # group_ce: workspace too small / C not multiple of 4 / bad slices
    sl = nat.int32_array([0, 2, 2, 6])
    rc = lib.bags_group_ce(p, 8, p, p, sl, None, nat.WEIGHTS_U8, None, 1, 8, 2, 4, p, None, None, 0, 0, None, p, 16, None)
    assert rc == -1 and b'workspace' in lib.bags_last_error()
    ws = lib.bags_workspace_bytes()
    rc = lib.bags_group_ce(p, 8, p, p, sl, None, nat.WEIGHTS_U8, None, 1, 6, 2, 4, p, None, None, 0, 0, None, p, ws, None)
    assert rc == -1 and b'multiple of 4' in lib.bags_last_error()
    bad = nat.int32_array([0, 2, 1, 6])   # overlapping slices
    rc = lib.bags_group_ce(p, 8, p, p, bad, None, nat.WEIGHTS_U8, None, 1, 8, 2, 4, p, None, None, 0, 0, None, p, ws, None)
    assert rc == -1 and b'pred_slice' in lib.bags_last_error()
    # too many bins
    rc = lib.bags_sample_others(p, p, 4, 9, 4, 8.0, 1, None, p, p, None)
    assert rc == -1
    with pytest.raises(nat.BagsNativeError):
        nat.check(rc, 'bags_sample_others')


def test_unknown_weights_dtype_is_rejected():
    """weights_dtype other than BAGS_WEIGHTS_U8 / BAGS_WEIGHTS_F32 is a bad argument, reported before any launch."""
    lib = nat.lib()
    buf = (C.c_char * 64)()
    p = C.addressof(buf)
    sl = nat.int32_array([0, 2, 2, 6])
    ws = lib.bags_workspace_bytes()
    rc = lib.bags_group_ce(p, 8, p, p, sl, p, 2, None, 1, 8, 2, 4, p, None, None, 0, 0, None, p, ws, None)
    assert rc == -1 and b'weights dtype 2' in lib.bags_last_error()

def test_ops_refuse_cpu_tensors():
    """No CPU fallback: handing the product a CPU tensor is an error, not a slow path."""
    import torch
    from balancedgroupsoftmax_b200 import ops
    x = torch.zeros(4, 8)
    with pytest.raises(nat.BagsNativeError):
        ops.linear_fwd(x, x, None)
    with pytest.raises(nat.BagsNativeError):
        ops.merge_scores(torch.zeros(4, 8), None)


def test_product_does_not_import_oracle():
    pkg = os.path.join(ROOT, 'balancedgroupsoftmax_b200')
    for fn in os.listdir(pkg):
        if fn.endswith('.py'):
            src = open(os.path.join(pkg, fn)).read()
            assert 'oracle' not in src.replace('# oracle', ''), '%s references the oracle' % fn


def test_grad_allreduce_argument_validation():
    """bags_grad_allreduce: layout / rank / alignment errors are reported before anything touches a device."""
    lib = nat.lib()
    assert lib.bags_grad_allreduce_flag_bytes(2) > lib.bags_grad_allreduce_status_offset(2) > 0
    assert lib.bags_grad_allreduce_flag_bytes(8) > lib.bags_grad_allreduce_flag_bytes(2)
    assert lib.bags_grad_allreduce_flag_bytes(8) % 4 == 0
    buf = (C.c_char * 4096)()
    base = (C.addressof(buf) + 255) // 256 * 256
    peers = (C.c_void_p * 2)(base, base + 1024)
    # NULL peer table
    rc = lib.bags_grad_allreduce(None, None, 1024, 16, 0, 2, 0.5, 0, None)
    assert rc == -1 and b'peer_bufs_host' in lib.bags_last_error()
    # rank outside the world / too many ranks
    assert lib.bags_grad_allreduce(peers, None, 1024, 16, 2, 2, 0.5, 0, None) == -1
    assert lib.bags_grad_allreduce(peers, None, 1024, 16, 0, 17, 0.5, 0, None) == -1
    # count not a multiple of 4 floats
    rc = lib.bags_grad_allreduce(peers, None, 1024, 10, 0, 2, 0.5, 0, None)
    assert rc == -1 and b'multiple of 4' in lib.bags_last_error()
    # flags overlapping the data
    rc = lib.bags_grad_allreduce(peers, None, 32, 16, 0, 2, 0.5, 0, None)
    assert rc == -1 and b'flag' in lib.bags_last_error()
    # misaligned peer mapping
    bad = (C.c_void_p * 2)(base, base + 1028)
    rc = lib.bags_grad_allreduce(bad, None, 1024, 16, 0, 2, 0.5, 0, None)
    assert rc != 0
    with pytest.raises(nat.BagsNativeError):
        nat.check(rc, 'bags_grad_allreduce')
