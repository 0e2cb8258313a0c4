#!/usr/bin/env python
"""Where the backward's time goes: per-CTA phase times of bwd_prep_kernel + bags_bwd_merged_kernel at the bench.py shape.

    python tools/bwd_phases.py [--rois 4096] [--dtype bf16] [--runs 20] [--gout ones|varied]

Points the library's debug timeline (bags_debug_set_timing) at a device buffer, captures bench.py's one-GPU step in a
CUDA graph and replays it once per run with a device synchronise in between: the fused forward (4096 RoIs x 1024 features -> 1236 logits in 5 bins,
dW zeroed by the forward), then the backward (dW, db, dX; gout = ones, no column sums from the forward).  It reads the
first consumer thread's %globaltimer stamps of every merged-kernel CTA and thread 0's stamps of every preparation
CTA.  For each phase it prints the median and the maximum across CTAs (each the median over the runs), in
microseconds:

  start skew       merged CTA start - earliest merged CTA start
  wait             CTA start to griddepcontrol.wait returned (the consumers' wait)
  mainloop uI      TMA + wgmma of the CTA's unit I (from its start, or from the wait if that came later)
  epilogue uI      the unit's stores / red.add (from the end of its mainloop, or from the wait if that came later)
  dW/dX us/kblock  mainloop time over the unit's k-blocks, per unit kind
  epilogue share   all epilogues over the CTA's span
  CTA total        merged CTA start to its last epilogue end

and per run (median over runs):

  prep span        earliest preparation CTA start to latest end
  prep to load     merged kernel's first operand load - latest preparation CTA end (negative: it started earlier)
  merged span      earliest merged CTA start to latest end
  backward span    earliest preparation CTA start to latest merged end

It also times the backward per call in a CUDA graph of 20 back-to-back backwards (CUDA events, stamps off), and prints
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

ROWS = 4096          # timeline rows: the merged kernel stamps rows [1024, 1024 + 2 grid), the preparation [2048, 4096)
MERGED_ROW, PREP_ROW = 1024, 2048
UNITS = 3            # units per CTA with stamps
PHASES = (['start skew', 'wait'] + ['%s u%d' % (k, i) for i in range(UNITS) for k in ('mainloop', 'epilogue')] +
          ['dW us/kblock', 'dX us/kblock', 'epilogue share', 'CTA total'])
SPANS = ['prep span', 'prep to load', 'merged span', 'backward span']


def _gpu_info(index):
    try:
        out = subprocess.run(['nvidia-smi', '-i', str(index), '--query-gpu=name,power.limit,clocks.sm',
                              '--format=csv,noheader,nounits'], stdout=subprocess.PIPE, stderr=subprocess.DEVNULL,
                             text=True, timeout=20).stdout.strip()
        name, power, clock = [f.strip() for f in out.splitlines()[0].split(',')]
        return name, float(power), float(clock)
    except Exception:
        return None, None, None


def _phases(timing):
    """timing: [ROWS, 8] int64 ns -> ({phase: list of per-CTA values in us}, {span: us})"""
    t = timing.double() / 1e3
    merged = [(t[MERGED_ROW + 2 * c], timing[MERGED_ROW + 2 * c + 1]) for c in range((PREP_ROW - MERGED_ROW) // 2)]
    merged = [(s, m) for s, m in merged if s[0] != 0]
    prep = t[PREP_ROW:ROWS]
    prep = prep[prep[:, 0] != 0]
    t0 = min(s[0].item() for s, _ in merged)
    d = {p: [] for p in PHASES}
    ends = []
    for s, m in merged:
        s = s.tolist()
        d['start skew'].append(s[0] - t0)
        d['wait'].append(s[1] - s[0])
        prev, epi, last = s[0], 0.0, s[0]
        for i in range(UNITS):
            kb = int(m[i])
            if kb == 0:
                break
            ml_end, ep_end = s[2 + 2 * i], s[3 + 2 * i]
            ml = ml_end - max(prev, s[1]) if i == 0 and s[1] < ml_end else ml_end - prev
            ep = ep_end - max(ml_end, s[1])
            d['mainloop u%d' % i].append(ml)
            d['epilogue u%d' % i].append(ep)
            d['dW us/kblock' if kb > 0 else 'dX us/kblock'].append(ml / abs(kb))
            epi += ep
            prev = last = ep_end
        d['CTA total'].append(last - s[0])
        d['epilogue share'].append(epi / max(last - s[0], 1e-9))
        ends.append(last)
    first_load = min(timing[MERGED_ROW + 2 * c + 1, 7].item() for c in range(len(merged))) / 1e3
    spans = {'merged span': max(ends) - t0}
    if prep.shape[0] > 0:
        spans['prep span'] = (prep[:, 2].max() - prep[:, 0].min()).item()
        spans['prep to load'] = first_load - prep[:, 2].max().item()
        spans['backward span'] = max(ends) - prep[:, 0].min().item()
    return d, spans, len(merged), int(prep.shape[0])


def main() -> int:
    ap = argparse.ArgumentParser()
    ap.add_argument('--rois', type=int, default=4096)
    ap.add_argument('--dtype', default='bf16', choices=['bf16', 'fp32'])
    ap.add_argument('--runs', type=int, default=20)
    ap.add_argument('--gout', default='ones', choices=['ones', 'varied'],
                    help="'ones' as bench.py; 'varied' makes the preparation kernel build the scaled copy W'")
    ap.add_argument('--json', default='', help='also write the results to this file')
    args = ap.parse_args()

    import torch
    if not torch.cuda.is_available():
        print('bwd_phases: needs a CUDA GPU (H100); refusing to run without one', file=sys.stderr)
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
    gout = torch.ones(dt.G, device=dev) if args.gout == 'ones' else torch.linspace(0.5, 1.5, dt.G, device=dev)
    dW = torch.empty(t.num_logits, K, device=dev)
    db = torch.empty(t.num_logits, device=dev)
    dX = torch.empty(N, K, device=dev, dtype=mode)
    wscratch = ops.bwd_scratch(w)

    def fwd():
        return ops.fused_fwd(x, w, b, labels, dt, wmask, avg, clear=dW)[3]

    def bwd(dz):
        ops.fused_bwd(dz, x, w, gout, dt, None, dW=dW, dX=dX, wscratch=wscratch, db=db, dw_prezeroed=True)

    for _ in range(3):
        bwd(fwd())
    torch.cuda.synchronize()

    # the stamped step is a captured graph, as bench.py runs it: eager launches would put the host's launch latency
    # between the preparation kernel and the merged kernel
    timing = torch.zeros(ROWS * 8, dtype=torch.int64, device=dev)
    lib = nat.lib()
    per_run, spans = {p: [] for p in PHASES}, {s: [] for s in SPANS}
    nat.check(lib.bags_debug_set_timing(timing.data_ptr()), 'bags_debug_set_timing')
    try:
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            step = torch.cuda.CUDAGraph()
            with torch.cuda.graph(step, stream=s):
                bwd(fwd())
        torch.cuda.current_stream().wait_stream(s)
    finally:
        nat.check(lib.bags_debug_set_timing(None), 'bags_debug_set_timing')
    for _ in range(2):
        step.replay()
    for _ in range(args.runs):
        timing.zero_()
        torch.cuda.synchronize()
        step.replay()
        torch.cuda.synchronize()
        ph, sp, ctas, prep_ctas = _phases(timing.view(ROWS, 8).cpu())
        for p in PHASES:
            if ph[p]:
                v = sorted(ph[p])
                per_run[p].append((v[len(v) // 2], v[-1]))
        for sname in SPANS:
            if sname in sp:
                spans[sname].append(sp[sname])

    # per call in a CUDA graph of 20 back-to-back backwards (no stamps)
    dz = fwd()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        bwd(dz)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph, stream=s):
            for _ in range(20):
                bwd(dz)
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
    print('backward (prep + merged), %d RoIs, %s, gout %s, %d merged CTAs, %d preparation CTAs, %d runs'
          % (N, args.dtype, args.gout, ctas, prep_ctas, args.runs))
    print('%-16s %10s %10s' % ('phase (us)', 'median', 'max'))
    res = dict(gpu=name, power_limit_w=power, rois=N, dtype=args.dtype, gout=args.gout, ctas=ctas,
               prep_ctas=prep_ctas, runs=args.runs, phases_us={}, spans_us={})
    for p in PHASES:
        if not per_run[p]:
            continue
        m, x_ = med([r[0] for r in per_run[p]]), med([r[1] for r in per_run[p]])
        res['phases_us'][p] = dict(median=round(m, 3), max=round(x_, 3))
        print('%-16s %10.3f %10.3f' % (p, m, x_))
    for sname in SPANS:
        if spans[sname]:
            res['spans_us'][sname] = round(med(spans[sname]), 3)
            print('%-16s %10.2f' % (sname, res['spans_us'][sname]))
    res['graph20_us_per_call'] = round(graph20_us, 3)
    print('per call in a graph of 20 backwards: %.2f us' % graph20_us)
    print(json.dumps(res))
    if args.json:
        with open(args.json, 'w') as f:
            json.dump(res, f, indent=1)
    return 0


if __name__ == '__main__':
    raise SystemExit(main())
