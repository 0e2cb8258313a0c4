"""The merged backward's schedule (pipelined mainloop, early start under the preparation kernel, split-K work list):
the full call (dW, db and dX in one launch) against the split pair that the data-parallel schedule issues (dW + db,
then dX alone), and each of them against float64.

Random normal operands at the bench shape's C = 1236 and K = 1024, 4096 RoIs and ragged row counts.  dX and db must be
bit-identical between the two: both contract the same operands in the same k-block order, and db is summed in a fixed
order by the preparation kernel.  dW is a split-K red.add whose summation order depends on the split factor and on
timing, so it is bounded by fp32 rounding against S = |gout dz|^T |x|, one rounding per wgmma k-step and split.  Against
float64 each output gets the same kind of bound, plus the rounding of the operands (TF32 products, a bf16 W') and of a
bf16 dX.  The cases cover a uniform gout (the kernel reads W itself and starts without waiting) and a non-uniform gout
or a gapped bin table (it reads the scaled copy W' that the preparation kernel writes), with dW zeroed by the caller or
by the preparation kernel.  Eager calls and CUDA-graph replays must give bit-identical dX and db.
"""
from __future__ import annotations

import contextlib
import os

import numpy as np
import pytest
import torch

from balancedgroupsoftmax_b200 import _native as nat

pytestmark = pytest.mark.gpu

DEV = torch.device('cuda', 0)
C, K = 1236, 1024
GAPS = [(0, 100), (108, 21), (129, 1), (140, 500), (700, C - 712)]


@contextlib.contextmanager
def _env(**switches):
    old = {k: os.environ.get(k) for k in switches}
    try:
        for k, v in switches.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = str(v)
        nat.reload_env()
        yield
    finally:
        for k, v in old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v
        nat.reload_env()


def _tables(name):
    from balancedgroupsoftmax_b200 import ops
    if name == 'synthetic':
        from balancedgroupsoftmax_b200.tables import synthetic_tables
        t = synthetic_tables()
        assert t.num_logits == C
        slices = [tuple(int(v) for v in r) for r in t.pred_slice]
    else:
        slices = GAPS
    G = len(slices)
    dt = ops.DeviceTables(G, 1, C, torch.zeros(G, 1, dtype=torch.int32, device=DEV),
                          torch.zeros(1, dtype=torch.int32, device=DEV),
                          nat.int32_array([v for sl in slices for v in sl]), np.array(slices, dtype=np.int64))
    return dt, slices


def _col_scale(slices, gout):
    s = torch.zeros(C, dtype=torch.float32, device=DEV)
    for (st, ln), g in zip(slices, gout.tolist()):
        s[st:st + ln] = g
    return s


def _operands(N, dtype, seed):
    from balancedgroupsoftmax_b200 import ops
    g = torch.Generator(device=DEV).manual_seed(seed)
    dz = torch.zeros((N, ops.pad_cols(C, 8)), dtype=dtype, device=DEV)   # ldd = 1240, as the fused forward writes it
    dz[:, :C] = (torch.randn(N, C, generator=g, device=DEV) * 1e-2).to(dtype)
    x = torch.relu(torch.randn(N, K, generator=g, device=DEV)).to(dtype)
    w = (torch.randn(C, K, generator=g, device=DEV) * 0.05).to(dtype)
    return dz, x, w


def _bwd(dz, x, w, gout, dt, prezeroed, out=None, split=False):
    """fused_bwd into the given (or fresh) buffers; a prezeroed dW is zeroed here, as the forward's clear hook does.
    split: two calls, dW + db and then dX alone, as the data-parallel schedule issues them."""
    from balancedgroupsoftmax_b200 import ops
    N = x.shape[0]
    if out is None:
        out = dict(dW=torch.full((C, K), float('nan'), device=DEV), db=torch.empty(C, device=DEV),
                   dX=torch.empty((N, K), dtype=x.dtype, device=DEV), ws=ops.bwd_scratch(w))
    if prezeroed:
        out['dW'].zero_()
    if split:
        ops.fused_bwd(dz, x, w, gout, dt, None, need_dx=False, dW=out['dW'], wscratch=out['ws'], db=out['db'],
                      dw_prezeroed=prezeroed)
        ops.fused_bwd(dz, x, w, gout, dt, None, need_dw=False, need_db=False, dX=out['dX'], wscratch=out['ws'])
    else:
        ops.fused_bwd(dz, x, w, gout, dt, None, dW=out['dW'], dX=out['dX'], wscratch=out['ws'], db=out['db'],
                      dw_prezeroed=prezeroed)
    return out


def _check_routes(new, ref, dz, x, gout, slices, what):
    assert torch.equal(new['dX'], ref['dX']), '%s: dX differs' % what
    assert torch.equal(new['db'], ref['db']), '%s: db differs' % what
    s = _col_scale(slices, gout)
    S = (dz[:, :C].float().abs() * s.abs()).t() @ x.float().abs()
    err = (new['dW'] - ref['dW']).abs()
    bound = (_ksteps(x.shape[0], x.dtype) + 16) * 2.0 ** -23 * S + 1e-30
    bad = err > bound
    assert not bool(bad.any()), '%s: dW differs by %.3e beyond fp32 summation-order rounding (bound %.3e)' % (
        what, err[bad].max().item(), bound[bad].min().item())


def _ksteps(length, dtype):
    """wgmma k-steps of a contraction over `length`: 4 per k-block of 64 bf16 / 32 fp32 elements"""
    return 4 * -(-length // (64 if dtype == torch.bfloat16 else 32))


def _float64_refs(dz, x, w, gout, slices):
    """(dW, db, dX) in float64 and each one's bound: one fp32 rounding per wgmma k-step, per split-K partial and per
    scaling against S = |gout dz|^T |x| (dW), |gout dz| |W| (dX) and sum |gout dz| (db), plus 2^-8 S for the operand
    roundings (TF32 products; dX's bf16 W' = bf16(gout W)) and 2^-8 |dX| for a bf16 dX."""
    dzs = dz[:, :C].double() * _col_scale(slices, gout).double()
    xd, wd = x.double(), w.double()
    f32 = x.dtype == torch.float32
    ref_dw, ref_db, ref_dx = dzs.t() @ xd, dzs.sum(0), dzs @ wd
    S = dzs.abs().t() @ xd.abs()
    tol_dw = ((_ksteps(x.shape[0], x.dtype) + 16) * 2.0 ** -23 + (2.0 ** -8 if f32 else 0.0)) * S
    tol_db = (x.shape[0] + 16) * 2.0 ** -23 * dzs.abs().sum(0)
    S = dzs.abs() @ wd.abs()
    tol_dx = ((_ksteps(C, x.dtype) + 16) * 2.0 ** -23 + 2.0 ** -8) * S + (0.0 if f32 else 2.0 ** -8 * ref_dx.abs())
    return dict(dW=(ref_dw, tol_dw), db=(ref_db, tol_db), dX=(ref_dx, tol_dx))


def _check_float64(got, refs, what):
    for name, (ref, tol) in refs.items():
        err = (got[name].double() - ref).abs()
        bad = err > tol + 1e-30
        assert not bool(bad.any()), '%s: %s is %.3e from float64 (bound %.3e)' % (
            what, name, err[bad].max().item(), tol[bad].min().item())


CASES = [
    # N, dtype, table, gout, dW zeroed by the caller
    (4096, torch.bfloat16, 'synthetic', 'ones', True),      # bench.py's one-GPU schedule
    (4096, torch.bfloat16, 'synthetic', 'varied', False),   # W' and the dW zeroing from the preparation kernel
    (4096, torch.float32, 'synthetic', 'ones', True),
    (4173, torch.bfloat16, 'gaps', 'ones', False),          # gaps: W' even with a uniform gout
    (8525, torch.bfloat16, 'synthetic', 'varied', True),
    (8525, torch.float32, 'gaps', 'varied', False),
    (131072 + 77, torch.bfloat16, 'synthetic', 'ones', True),
]


def _case_id(c):
    N, dtype, table, gout, prez = c
    return 'N%d-%s-%s-%s-%s' % (N, 'bf16' if dtype == torch.bfloat16 else 'fp32', table, gout,
                                'prezeroed' if prez else 'dirty')


@pytest.mark.parametrize('case', CASES, ids=[_case_id(c) for c in CASES])
def test_merged_matches_unmerged(case):
    """The full call against the split pair, for the default and forced dW split counts."""
    N, dtype, table, gout_mode, prez = case
    dt, slices = _tables(table)
    dz, x, w = _operands(N, dtype, seed=N + len(slices))
    G = len(slices)
    gout = torch.ones(G, device=DEV) if gout_mode == 'ones' else torch.linspace(0.5, 1.5, G, device=DEV)
    refs = _float64_refs(dz, x, w, gout, slices)
    for splits in (None, 1, 16):
        what = '%s splits=%s' % (_case_id(case), splits)
        with _env(BAGS_DW_SPLITS=splits):
            full = _bwd(dz, x, w, gout, dt, prez)
            pair = _bwd(dz, x, w, gout, dt, prez, split=True)
        torch.cuda.synchronize()
        _check_routes(full, pair, dz, x, gout, slices, what + ' full call vs split pair')
        _check_float64(full, refs, what + ' full call')
        _check_float64(pair, refs, what + ' split pair')


@pytest.mark.parametrize('gout_mode', ['ones', 'varied'])
def test_graph_replay_matches_eager(gout_mode):
    """The bench shape's backward captured in a CUDA graph: every replay gives the eager call's dX and db bits."""
    N, dtype = 4096, torch.bfloat16
    dt, slices = _tables('synthetic')
    dz, x, w = _operands(N, dtype, seed=11)
    G = len(slices)
    gout = torch.ones(G, device=DEV) if gout_mode == 'ones' else torch.linspace(0.5, 1.5, G, device=DEV)
    eager = _bwd(dz, x, w, gout, dt, True)
    eager = {k: v.clone() for k, v in eager.items() if k != 'ws'}
    out = _bwd(dz, x, w, gout, dt, True)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph, stream=s):
            for _ in range(3):
                _bwd(dz, x, w, gout, dt, True, out=out)
    torch.cuda.current_stream().wait_stream(s)
    for r in range(3):
        out['dX'].zero_()
        out['db'].zero_()
        graph.replay()
        torch.cuda.synchronize()
        assert torch.equal(out['dX'], eager['dX']), 'replay %d: dX differs from the eager call' % r
        assert torch.equal(out['db'], eager['db']), 'replay %d: db differs from the eager call' % r
        _check_routes(out, eager, dz, x, gout, slices, 'replay %d' % r)
