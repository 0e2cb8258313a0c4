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

def test_fwd_invalid_arguments_return_error_codes():
    """bags_fwd's argument rules on both routes (fused: logits NULL; materialised: a logits buffer), reported before
    anything touches a device -- the fused route shares them with bags_ce_fwd and bags_focal_fwd."""
    lib = nat.lib()
    buf = (C.c_char * 256)()
    base = (C.addressof(buf) + 15) // 16 * 16
    ws = lib.bags_workspace_bytes()
    tiles = nat.int32_array([0, 4, 4, 4])   # two bins tiling C = 8: eligible for the fused kernel
    assert lib.bags_fused_eligible(tiles, 2, 8) == 1

    def call(slices=tiles, l2b=base, wdt=nat.WEIGHTS_U8, N=4, K=8, dtype=nat.DTYPE_BF16, bias=None, logits=None,
             dz=None, ldd=0, colsum=None, ntiles=0, wsb=ws, clear=None, clear_bytes=0, x=base, ldx=None, w=base,
             ldw=None):
        return lib.bags_fwd(x, K if ldx is None else ldx, w, K if ldw is None else ldw, bias, base, l2b, slices, None,
                            wdt, None, N, K, 8, 2, 4, dtype, logits, 8 if logits else 0, base, None, dz, ldd, colsum,
                            ntiles, base, wsb, clear, clear_bytes, None)

    gap = nat.int32_array([0, 2, 4, 4])     # columns 2 and 3 lie in no bin
    assert lib.bags_fused_eligible(gap, 2, 8) == 0
    assert call(slices=gap) == -1 and b'eligible' in lib.bags_last_error()
    assert call(wdt=2) == -1 and b'weights dtype 2' in lib.bags_last_error()
    assert call(dtype=7) == -1 and b'dtype' in lib.bags_last_error()
    assert call(l2b=None) == -1 and b'NULL' in lib.bags_last_error()
    assert call(K=0) == -1 and b'bad shape' in lib.bags_last_error()
    assert call(bias=base + 4) == -1 and b'bias' in lib.bags_last_error()
    assert call(dz=base, ldd=12) == -1 and b'ldd' in lib.bags_last_error()     # not a multiple of 8
    assert call(dz=base, ldd=0) == -1 and b'ldd' in lib.bags_last_error()      # < C
    assert call(colsum=base, ntiles=2) == -1 and b'colsum' in lib.bags_last_error()   # ceil(4/128) = 1 row tile
    assert call(clear=base + 4, clear_bytes=16) == -1 and b'clear' in lib.bags_last_error()
    assert call(clear=base, clear_bytes=8) == -1 and b'clear' in lib.bags_last_error()
    assert call(wsb=16) == -1 and b'workspace' in lib.bags_last_error()
    check_fused_operand_rules(lib, 'bags_fwd', call, base)
    # the materialised route keeps the rules it shares with the fused one
    assert call(logits=base, colsum=base, ntiles=0) == -1 and b'colsum' in lib.bags_last_error()
    assert call(logits=base, clear=base + 4, clear_bytes=16) == -1 and b'clear' in lib.bags_last_error()


def check_fused_operand_rules(lib, who, call, base):
    """The fused route's operand rules in both operand dtypes, reported with the entry point's name before anything
    touches a device: ldx >= K and ldw >= K, x and W 16-byte aligned, row strides whole multiples of 16 bytes.
    ``call(dtype=, K=, x=, ldx=, w=, ldw=)`` is the entry point with otherwise valid arguments (x = W = ``base``, 16-byte
    aligned, ldx = ldw = K by default).  Shared with test_reweight_head_cpu.py and test_focal_cpu.py."""
    for dtype, a in ((nat.DTYPE_BF16, 8), (nat.DTYPE_F32, 4)):   # a: elements per 16 bytes
        K = 2 * a
        for kw in (dict(ldx=K - a), dict(ldw=K - a), dict(ldx=K - a, ldw=K - a)):
            assert call(dtype=dtype, K=K, **kw) == -1, (dtype, kw)
            msg = lib.bags_last_error()
            assert who.encode() in msg and b'>= K' in msg, msg
        for kw in (dict(ldx=K + 1), dict(ldw=K + 2), dict(ldx=K + a // 2)):   # >= K, rows not whole 16-byte pieces
            assert call(dtype=dtype, K=K, **kw) == -1, (dtype, kw)
            msg = lib.bags_last_error()
            assert who.encode() in msg and b'multiples of 16 bytes' in msg, msg
        for name in ('x', 'w'):
            for off in (4, 8):
                assert call(dtype=dtype, K=K, **{name: base + off}) == -1, (dtype, name, off)
                msg = lib.bags_last_error()
                assert who.encode() in msg and b'16-byte aligned' in msg, msg


def test_bwd_invalid_arguments_return_error_codes():
    """bags_bwd's operand rules for each requested output, reported before anything touches a device."""
    lib = nat.lib()
    buf = (C.c_char * 256)()
    base = (C.addressof(buf) + 15) // 16 * 16
    slices = nat.int32_array([0, 4, 4, 4])

    def call(x=base, w=base, dW=None, dX=None, colsum=None, ntiles=0, db=None):
        return lib.bags_bwd(base, 8, x, 8, w, 8, None, slices, colsum, ntiles, dW, 8, db, dX, 8, None, 0, 4, 8, 8, 2,
                            nat.DTYPE_BF16, 0, None)

    assert call(w=None, dX=base) == -1 and b'w is NULL' in lib.bags_last_error()
    assert call(x=None, dW=base) == -1 and b'x is NULL' in lib.bags_last_error()
    assert call(dX=base + 4) == -1 and b'dX not 16-byte aligned' in lib.bags_last_error()
    assert call(db=base, colsum=base, ntiles=0) == -1 and b'colsum_tiles' in lib.bags_last_error()


def test_cast_bf16_rejects_misaligned_pointers():
    """bags_cast_bf16 reads float4 from src and writes 8-byte groups to dst: a misaligned pointer is a bad argument,
    reported before any launch."""
    lib = nat.lib()
    buf = (C.c_char * 256)()
    base = (C.addressof(buf) + 15) // 16 * 16
    rc = lib.bags_cast_bf16(base + 4, 4, base + 128, 4, 1, 4, None)   # src 4 bytes past a 16-byte boundary
    assert rc == -1 and b'aligned' in lib.bags_last_error()
    rc = lib.bags_cast_bf16(base, 4, base + 130, 4, 1, 4, None)       # dst 2 bytes past an 8-byte boundary
    assert rc == -1 and b'aligned' in lib.bags_last_error()


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
