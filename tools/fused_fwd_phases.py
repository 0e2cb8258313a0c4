#!/usr/bin/env python
"""Where the fused forward's time goes: per-CTA phase times of bags_fwd_fused_kernel at the bench.py shape.

    python tools/fused_fwd_phases.py [--rois 4096] [--dtype bf16] [--runs 20] [--no-clear]

Points the library's debug timeline (bags_debug_set_timing) at a device buffer, runs the fused forward (4096 RoIs x
1024 features -> 1236 logits in 5 bins, dW zeroed by the kernel as in bench.py's default schedule) once per run with
a device synchronise in between, and reads thread 0's %globaltimer stamps of every CTA.  For each phase it prints the
median and the maximum across CTAs (each the median over the runs), in microseconds:

  start skew     CTA start - earliest CTA start
  mainloop       TMA + wgmma of the row tile
  pass A         per-bin row maxima
  pass B         exponentials and per-bin sums
  exchange wait  publish the partials, wait for the group's other three CTAs
  lse + pass C   combine the partials, dz (and column sums)
  tail           column sums to HBM, dW clear, loss bookkeeping
  CTA total      start to end of the CTA
  kernel span    earliest start to latest end (one value per run)

It also times the forward per call in a CUDA graph of 20 back-to-back forwards (CUDA events, stamps off), and prints
the GPU name and its power limit.  Refuses to run without a GPU.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

PHASES = ['start skew', 'mainloop', 'pass A', 'pass B', 'exchange wait', 'lse + pass C', 'tail', 'CTA total']
MAX_CTAS = 256   # the fused forward's grid is at most 4 CTAs x 64 groups


def _gpu_info(index):
    try:
        out = subprocess.run(['nvidia-smi', '-i', str(index), '--query-gpu=name,power.limit,clocks.sm',
                              '--format=csv,noheader,nounits'], stdout=subprocess.PIPE, stderr=subprocess.DEVNULL,
                             text=True, timeout=20).stdout.strip()
        name, power, clock = [f.strip() for f in out.splitlines()[0].split(',')]
        return name, float(power), float(clock)
    except Exception:
        return None, None, None


def _phases(stamps):
    """stamps: [ctas, 8] int64 ns -> {phase: per-CTA values in us}"""
    s = stamps.double() / 1e3
    d = {
        'start skew': s[:, 0] - s[:, 0].min(),
        'mainloop': s[:, 1] - s[:, 0],
        'pass A': s[:, 2] - s[:, 1],
        'pass B': s[:, 3] - s[:, 2],
        'exchange wait': s[:, 4] - s[:, 3],
        'lse + pass C': s[:, 5] - s[:, 4],
        'tail': s[:, 6] - s[:, 5],
        'CTA total': s[:, 6] - s[:, 0],
    }
    return d, (s[:, 6].max() - s[:, 0].min()).item()


def main() -> int:
    ap = argparse.ArgumentParser()
    ap.add_argument('--rois', type=int, default=4096)
    ap.add_argument('--dtype', default='bf16', choices=['bf16', 'fp32'])
    ap.add_argument('--runs', type=int, default=20)
    ap.add_argument('--no-clear', action='store_true', help='do not let the kernel zero a dW-sized buffer')
    ap.add_argument('--json', default='', help='also write the results to this file')
    args = ap.parse_args()

    import torch
    if not torch.cuda.is_available():
        print('fused_fwd_phases: needs a CUDA GPU (H100); refusing to run without one', file=sys.stderr)
        return 2
    from balancedgroupsoftmax_b200 import _native as nat
    from balancedgroupsoftmax_b200 import ops
    from balancedgroupsoftmax_b200.tables import synthetic_tables

    dev = torch.device('cuda', torch.cuda.current_device())
    mode = torch.bfloat16 if args.dtype == 'bf16' else torch.float32
    N, K = args.rois, 1024
    t = synthetic_tables(1231, seed=0)
    dt = ops.DeviceTables.from_tables(t, dev)
    g = torch.Generator(device=dev).manual_seed(0)
    x = torch.relu(torch.randn(N, K, generator=g, device=dev)).to(mode)
    w = (torch.randn(t.num_logits, K, generator=g, device=dev) * 0.05).to(mode)
    b = torch.randn(t.num_logits, generator=g, device=dev) * 0.1
    labels = torch.zeros(N, dtype=torch.long, device=dev)
    labels[:N // 4] = torch.randint(1, t.num_classes, (N // 4,), generator=g, device=dev)
    wmask, avg = ops.sample_others(labels, dt, 8.0, 1)
    dW = None if args.no_clear else torch.empty(t.num_logits, K, device=dev)
    assert ops.fused_eligible(dt)

    def fwd():
        return ops.fused_fwd(x, w, b, labels, dt, wmask, avg, clear=dW)

    for _ in range(3):
        fwd()
    torch.cuda.synchronize()

    timing = torch.zeros(MAX_CTAS * 8, dtype=torch.int64, device=dev)
    lib = nat.lib()
    per_run, spans = {p: [] for p in PHASES}, []
    nat.check(lib.bags_debug_set_timing(timing.data_ptr()), 'bags_debug_set_timing')
    try:
        for _ in range(args.runs):
            timing.zero_()
            torch.cuda.synchronize()
            fwd()
            torch.cuda.synchronize()
            st = timing.view(MAX_CTAS, 8).cpu()
            st = st[st[:, 0] != 0]
            ph, span = _phases(st)
            spans.append(span)
            for p in PHASES:
                per_run[p].append((ph[p].median().item(), ph[p].max().item()))
    finally:
        nat.check(lib.bags_debug_set_timing(None), 'bags_debug_set_timing')
    ctas = int(st.shape[0])

    # per call in a CUDA graph of 20 back-to-back forwards (no stamps)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        fwd()
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph, stream=s):
            for _ in range(20):
                fwd()
        for _ in range(3):
            graph.replay()
        a, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(s)
        for _ in range(20):
            graph.replay()
        e.record(s)
    s.synchronize()
    graph20_us = a.elapsed_time(e) / (20 * 20) * 1e3

    def med(v):
        v = sorted(v)
        return v[len(v) // 2]

    name, power, clock = _gpu_info(dev.index)
    print('GPU: %s, power limit %s W, SM clock %s MHz (after the runs)' % (name, power, clock))
    print('fused forward, %d RoIs, %s, %d CTAs, %d runs%s' % (N, args.dtype, ctas, args.runs,
                                                            '' if args.no_clear else ', dW cleared by the kernel'))
    print('%-14s %10s %10s' % ('phase (us)', 'median', 'max'))
    res = dict(gpu=name, power_limit_w=power, rois=N, dtype=args.dtype, ctas=ctas, runs=args.runs,
               clear=not args.no_clear, phases_us={})
    for p in PHASES:
        m, x_ = med([r[0] for r in per_run[p]]), med([r[1] for r in per_run[p]])
        res['phases_us'][p] = dict(median=round(m, 3), max=round(x_, 3))
        print('%-14s %10.2f %10.2f' % (p, m, x_))
    res['kernel_span_us'] = round(med(spans), 3)
    res['graph20_us_per_call'] = round(graph20_us, 3)
    print('%-14s %10.2f' % ('kernel span', res['kernel_span_us']))
    print('per call in a graph of 20 forwards: %.2f us' % graph20_us)
    print(json.dumps(res))
    if args.json:
        with open(args.json, 'w') as f:
            json.dump(res, f, indent=1)
    return 0


if __name__ == '__main__':
    raise SystemExit(main())
