"""Bring-up probe: every kernel checked in its own subprocess with a timeout.

    python tests/gpu_probe.py            # run all cases, print a table, write gpurun_out/probe.json
    python tests/gpu_probe.py --case X   # run one case in-process

Not collected by pytest (no test_ prefix); the pytest parity suite is tests/test_gpu_*.py.
"""
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def _setup():
    import numpy as np
    import torch
    from balancedgroupsoftmax_b200 import ops
    from balancedgroupsoftmax_b200.tables import synthetic_tables
    from oracle import bags_oracle as O
    torch.manual_seed(0)
    np.random.seed(0)
    return np, torch, ops, synthetic_tables, O


def rel(a, b):
    a = a.double()
    b = b.double()
    return ((a - b).norm() / b.norm().clamp_min(1e-30)).item()


def _problem(N, K=1024, seed=0, wstd=0.05):
    np, torch, ops, synthetic_tables, O = _setup()
    t = synthetic_tables()
    g = torch.Generator().manual_seed(seed)
    x = torch.relu(torch.randn(N, K, generator=g))
    W = torch.randn(t.num_logits, K, generator=g) * wstd
    b = torch.randn(t.num_logits, generator=g) * 0.1
    labels = torch.zeros(N, dtype=torch.long)
    npos = max(1, N // 4)
    labels[:npos] = torch.randint(1, t.num_classes, (npos,), generator=g)
    l2b = torch.from_numpy(t.label2binlabel)
    ps = torch.from_numpy(t.pred_slice)
    np.random.seed(seed)
    remapped = O.remap_labels(labels, l2b, 8.0)
    return t, x, W, b, labels, l2b, ps, remapped


def case_group_ce(name):
    np, torch, ops, _, O = _setup()
    out = {}
    for N in (1, 37, 512):
        t, x, W, b, labels, l2b, ps, remapped = _problem(N)
        z = O.fc_cls(x, W, b)
        ref = O.bags_loss(z, labels, l2b, ps, remapped=remapped)
        dz_ref, _, db_ref, _ = O.closed_form_grads(x, W, b, labels, l2b, ps, remapped)
        dt = ops.DeviceTables.from_tables(t, 'cuda')
        wmask = torch.stack([w.to(torch.uint8) for w in remapped[1]]).cuda()
        avg = ops.mask_avg(wmask)
        assert avg.cpu().tolist() == [float(a) for a in remapped[2]], (avg.cpu().tolist(), remapped[2])
        for dzt in (torch.float32, torch.bfloat16):
            loss, lse, dz, colsum = ops.group_ce(z.cuda(), labels.cuda(), dt, wmask, avg, want_dz=True,
                                                 dz_dtype=dzt, want_lse=True)
            torch.cuda.synchronize()
            lr = max(abs(loss[g].item() - ref['loss_cls_bin%d' % g].item()) /
                     max(abs(ref['loss_cls_bin%d' % g].item()), 1e-3) for g in range(dt.G))
            dr = rel(dz[:, :t.num_logits].float().cpu(), dz_ref)
            cr = rel(colsum.sum(0).cpu(), db_ref)
            out['N%d.%s' % (N, str(dzt)[6:])] = dict(loss=lr, dz=dr, colsum=cr)
            assert lr < 1e-5, lr
            assert dr < (1e-5 if dzt == torch.float32 else 4e-3), dr
            assert cr < 1e-4, cr
    return out


def case_sampler(name):
    np, torch, ops, _, O = _setup()
    out = {}
    for N in (1, 100, 512, 4096, 5000):
        t, x, W, b, labels, l2b, ps, remapped = _problem(N)
        dt = ops.DeviceTables.from_tables(t, 'cuda')
        wmask, avg = ops.sample_others(labels.cuda(), dt, 8.0, seed=1234 + N)
        wmask2, _ = ops.sample_others(labels.cuda(), dt, 8.0, seed=1234 + N)
        wmask3, _ = ops.sample_others(labels.cuda(), dt, 8.0, seed=99)
        torch.cuda.synchronize()
        wm = wmask.cpu()
        assert torch.equal(wm, wmask2.cpu()), 'sampler not deterministic for a fixed seed'
        for g in range(dt.G):
            tg = l2b[g][labels]
            fg = tg > 0
            F = int(fg.sum())
            Oth = N - F
            k = int(F * 8.0)
            w = wm[g].bool()
            if g == 0:
                exp_sum = N
            elif F == 0:
                exp_sum = 0
            elif k >= Oth:
                exp_sum = N
            else:
                exp_sum = F + k
                assert bool(w[fg].all()), 'in-bin rows must be kept'
            assert int(w.sum()) == exp_sum, (g, int(w.sum()), exp_sum)
            assert avg[g].item() == max(float(exp_sum), 1.0)
        out['N%d' % N] = dict(avg=avg.cpu().tolist(), differs_by_seed=bool((wm != wmask3.cpu()).any()))
    return out


def case_merge(name):
    np, torch, ops, _, O = _setup()
    t, x, W, b, labels, l2b, ps, remapped = _problem(1000)
    z = O.fc_cls(x, W * 4, b)
    ref = O.merge_score(z, ps, [torch.from_numpy(s) for s in t.fg_splits], t.num_classes)
    dt = ops.DeviceTables.from_tables(t, 'cuda')
    got = ops.merge_scores(z.cuda(), dt).cpu()
    err = (got - ref).abs().max().item()
    am = bool((got.argmax(1) == ref.argmax(1)).all())
    am_fg = bool((got[:, 1:].argmax(1) == ref[:, 1:].argmax(1)).all())
    assert err < 1e-6 and am and am_fg, (err, am, am_fg)
    return dict(max_abs=err, argmax_equal=am, fg_argmax_equal=am_fg)


def case_fused(name):
    np, torch, ops, _, O = _setup()
    _, dts = name.split('.')
    cdt = torch.bfloat16 if dts == 'bf16' else torch.float32
    out = {}
    for N in (512, 200, 4096):
        t, x, W, b, labels, l2b, ps, remapped = _problem(N)
        gout = [1.0, 0.5, 0.25, 2.0, 1.5]
        if cdt == torch.bfloat16:
            xo, Wo = x.bfloat16().float(), W.bfloat16().float()   # oracle fed the same rounded operands
        else:
            xo, Wo = x, W
        z = O.fc_cls(xo, Wo, b)
        ref = O.bags_loss(z, labels, l2b, ps, remapped=remapped)
        _, dW_ref, db_ref, dX_ref = O.closed_form_grads(xo, Wo, b, labels, l2b, ps, remapped, gout=gout)
        dt = ops.DeviceTables.from_tables(t, 'cuda')
        wmask = torch.stack([w.to(torch.uint8) for w in remapped[1]]).cuda()
        avg = ops.mask_avg(wmask)
        xc, wc = x.cuda().to(cdt), W.cuda().to(cdt)
        loss, logits, _, dz, colsum = ops.fused_fwd(xc, wc, b.cuda(), labels.cuda(), dt, wmask, avg, materialize=True)
        dW, db, dX = ops.fused_bwd(dz, xc, wc, torch.tensor(gout, device='cuda'), dt, colsum)
        torch.cuda.synchronize()
        lr = max(abs(loss[g].item() - ref['loss_cls_bin%d' % g].item()) / abs(ref['loss_cls_bin%d' % g].item())
                 for g in range(dt.G))
        res = dict(loss=lr, logits=rel(logits.cpu(), z), dW=rel(dW.cpu(), dW_ref), db=rel(db.cpu(), db_ref),
                   dX=rel(dX.float().cpu(), dX_ref))
        out['N%d' % N] = res
        tol = dict(loss=1e-3, logits=2e-3, dW=5e-3, db=1e-3, dX=5e-3) if cdt == torch.bfloat16 else \
            dict(loss=1e-3, logits=1e-3, dW=1e-3, db=1e-3, dX=1e-3)
        for k_, v in res.items():
            assert v < tol[k_], (k_, v, tol[k_])
    return out



def case_fusedk(name):
    """fused forward kernel (logits stay on chip) vs the oracle, incl. ragged N and lse output"""
    np, torch, ops, _, O = _setup()
    _, dts = name.split('.')
    cdt = torch.bfloat16 if dts == 'bf16' else torch.float32
    out = {}
    for N in (1, 77, 128, 512, 1000, 4096):
        t, x, W, b, labels, l2b, ps, remapped = _problem(N, seed=N)
        if cdt == torch.bfloat16:
            xo, Wo = x.bfloat16().float(), W.bfloat16().float()
        else:
            xo, Wo = x, W
        z = O.fc_cls(xo, Wo, b)
        ref = O.bags_loss(z, labels, l2b, ps, remapped=remapped)
        dz_ref, dW_ref, db_ref, dX_ref = O.closed_form_grads(xo, Wo, b, labels, l2b, ps, remapped)
        dt = ops.DeviceTables.from_tables(t, 'cuda')
        assert ops.fused_eligible(dt)
        wmask = torch.stack([w.to(torch.uint8) for w in remapped[1]]).cuda()
        avg = ops.mask_avg(wmask)
        xc, wc = x.cuda().to(cdt), W.cuda().to(cdt)
        loss, logits, lse, dz, colsum = ops.fused_fwd(xc, wc, b.cuda(), labels.cuda(), dt, wmask, avg, want_lse=True,
                                                      want_colsum=True)
        assert logits is None
        torch.cuda.synchronize()
        lr = max(abs(loss[g].item() - ref['loss_cls_bin%d' % g].item()) / max(abs(ref['loss_cls_bin%d' % g].item()), 1e-2)
                 for g in range(dt.G))
        lse_ref = torch.stack([torch.logsumexp(z[:, int(ps[g, 0]):int(ps[g, 0]) + int(ps[g, 1])], 1) for g in range(5)], 1)
        res = dict(loss=lr, lse=rel(lse.cpu(), lse_ref), dz=rel(dz[:, :t.num_logits].float().cpu(), dz_ref),
                   colsum=rel(colsum.sum(0).cpu(), db_ref) if db_ref.norm() > 0 else 0.0)
        dW, db, dX = ops.fused_bwd(dz, xc, wc, None, dt, colsum)
        torch.cuda.synchronize()
        res['dW'] = rel(dW.cpu(), dW_ref)
        out['N%d' % N] = res
        tol = dict(loss=1e-4, lse=1e-5, dz=4e-3, colsum=2e-3, dW=3e-3) if cdt == torch.bfloat16 else \
            dict(loss=1e-3, lse=1e-3, dz=2e-3, colsum=1e-3, dW=1e-3 if N >= 64 else 2e-3)
        for k_, v in res.items():
            assert v < tol[k_], (N, k_, v, tol[k_])
    return out


def case_timing(name):
    """rough CUDA-event timings of each launch at the benchmark shape (not a bench number)"""
    np, torch, ops, _, O = _setup()
    N = 4096
    t, x, W, b, labels, l2b, ps, remapped = _problem(N)
    dt = ops.DeviceTables.from_tables(t, 'cuda')
    xc, wc = x.cuda().bfloat16(), W.cuda().bfloat16()
    bc, lc = b.cuda(), labels.cuda()
    gout = torch.ones(5, device='cuda')
    res = {}

    def timeit(fn, iters=50):
        for _ in range(5):
            fn()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(iters):
            fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / iters * 1e3  # us

    wmask, avg = ops.sample_others(lc, dt, 8.0, 1)
    logits = torch.empty(N, t.num_logits, device='cuda')
    res['sample_us'] = timeit(lambda: ops.sample_others(lc, dt, 8.0, 1))
    res['linear_fwd_us'] = timeit(lambda: ops.linear_fwd(xc, wc, bc, out=logits))
    res['group_ce_us'] = timeit(lambda: ops.group_ce(logits, lc, dt, wmask, avg))
    loss, _, _, dz, colsum = ops.fused_fwd(xc, wc, bc, lc, dt, wmask, avg, logits=logits)
    dW = torch.empty(t.num_logits, 1024, device='cuda')
    dX = torch.empty(N, 1024, device='cuda', dtype=torch.bfloat16)
    ws = ops.bwd_scratch(wc)
    res['bwd_all_us'] = timeit(lambda: ops.fused_bwd(dz, xc, wc, gout, dt, colsum, dW=dW, dX=dX, wscratch=ws))
    res['bwd_dw_only_us'] = timeit(lambda: ops.fused_bwd(dz, xc, wc, gout, dt, colsum, need_dx=False, dW=dW))
    res['bwd_dx_only_us'] = timeit(lambda: ops.fused_bwd(dz, xc, wc, None, dt, colsum, need_dw=False, need_db=False, dX=dX))
    res['fwd_unfused_us'] = timeit(lambda: ops.fused_fwd(xc, wc, bc, lc, dt, wmask, avg, logits=logits))
    res['fwd_fused_us'] = timeit(lambda: ops.fused_fwd(xc, wc, bc, lc, dt, wmask, avg))
    # torch reference pieces on the same device for scale
    res['torch_matmul_bf16_us'] = timeit(lambda: torch.matmul(xc, wc.t()))
    # library yardstick: the three plain GEMMs of a step (no softmax, no loss) through cuBLAS, replayed from a CUDA
    # graph so that host launch gaps do not count
    try:
        dzc = dz[:, :t.num_logits].contiguous()
        st = torch.cuda.Stream()
        with torch.cuda.stream(st):
            def three():
                z = torch.matmul(xc, wc.t())
                gw = torch.matmul(dzc.t(), xc)
                gx = torch.matmul(dzc, wc)
                return z, gw, gx
            for _ in range(3):
                three()
            st.synchronize()
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g, stream=st):
                for _ in range(10):
                    three()
            g.replay()
            st.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(st)
            for _ in range(10):
                g.replay()
            e1.record(st)
            st.synchronize()
        res['cublas_three_gemms_graph_us'] = e0.elapsed_time(e1) / 100 * 1e3
    except Exception as ex:  # pragma: no cover
        res['cublas_three_gemms_graph_us'] = repr(ex)
    return res


CASES = {
    'group_ce': case_group_ce, 'sampler': case_sampler, 'merge': case_merge,
    'fused.bf16': case_fused, 'fused.f32': case_fused, 'fusedk.bf16': case_fusedk, 'fusedk.f32': case_fusedk,
    'timing': case_timing,
}


def main():
    if '--case' in sys.argv:
        name = sys.argv[sys.argv.index('--case') + 1]
        res = CASES[name](name)
        print('RESULT ' + json.dumps(res))
        return 0
    only = [a for a in sys.argv[1:] if not a.startswith('-')]
    summary = {}
    for name in CASES:
        if only and not any(name.startswith(o) for o in only):
            continue
        t0 = time.time()
        try:
            p = subprocess.run([sys.executable, os.path.abspath(__file__), '--case', name], capture_output=True,
                               text=True, timeout=240)
            ok = p.returncode == 0
            res = None
            for line in p.stdout.splitlines():
                if line.startswith('RESULT '):
                    res = json.loads(line[7:])
            tail = (p.stdout + p.stderr)[-1500:] if not ok else ''
        except subprocess.TimeoutExpired as e:
            ok, res = False, None
            tail = 'TIMEOUT ' + str((e.stdout or b'')[-500:]) + str((e.stderr or b'')[-500:])
        summary[name] = dict(ok=ok, secs=round(time.time() - t0, 1), result=res, tail=tail)
        print('%-18s %s %5.1fs %s' % (name, 'OK  ' if ok else 'FAIL', time.time() - t0,
                                     json.dumps(res) if ok else tail.replace('\n', ' | ')[-700:]), flush=True)
    os.makedirs(os.path.join(ROOT, 'gpurun_out'), exist_ok=True)
    with open(os.path.join(ROOT, 'gpurun_out', 'probe.json'), 'w') as f:
        json.dump(summary, f, indent=1)
    return 0 if all(v['ok'] for v in summary.values()) else 1


if __name__ == '__main__':
    sys.exit(main())
