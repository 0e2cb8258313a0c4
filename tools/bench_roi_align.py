"""Time the FPN RoI extractor, native against the reference's, alternated in one run:

    native     SingleRoIExtractor (balancedgroupsoftmax_b200.roi_extractor): one bags_roi_align_fwd launch, one
               bags_roi_align_bwd launch
    reference  mmdet's SingleRoIExtractor.forward loop over levels (tests/roi_align_oracle.py:extractor) on the
               reference's own RoIAlign op built into oracle/_ref/, with its host syncs; its backward is the op's
               atomicAdd scatter once per level.  The op launches on the legacy default stream.
    torchvision  torchvision.ops.roi_align on one level, aligned=False: timing only, it computes something else

at three shapes: the Faster R-CNN bbox extractor (2 images padded to 800 x 1344, 1024 RoIs, 7 x 7, 256 channels), the
Mask R-CNN mask extractor (256 positives, 14 x 14) and HTC's semantic extractor (one stride-8 level, 14 x 14, 512
RoIs).  Forward and forward + backward; milliseconds per call from CUDA events over ``--reps`` calls after a warm-up,
median of ``--rounds`` rounds.

    python tools/bench_roi_align.py [--reps 20] [--rounds 5] [--json out.json]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, 'tests')]

from balancedgroupsoftmax_b200.roi_extractor import SingleRoIExtractor  # noqa: E402

STRIDES = [4, 8, 16, 32]
SHAPES = {
    'faster_bbox_7x7': dict(out=7, k=1024, strides=STRIDES),
    'mask_14x14': dict(out=14, k=256, strides=STRIDES),
    'htc_semantic_14x14': dict(out=14, k=512, strides=[8]),
}


def _gpu_info():
    name = torch.cuda.get_device_name(0)
    try:
        out = subprocess.run(['nvidia-smi', '--query-gpu=power.limit', '--format=csv,noheader', '-i', '0'],
                             stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        out = 'unknown'
    return name, out or 'unknown'


def _inputs(cfg, gen):
    feats = [torch.randn(2, 256, 800 // s, 1344 // s, generator=gen).cuda() for s in cfg['strides']]
    k = cfg['k']
    size = torch.exp(torch.empty(k, 2).uniform_(np.log(16), np.log(800), generator=gen))
    ctr = torch.rand(k, 2, generator=gen) * torch.tensor([1344., 800.])
    b = torch.arange(2).repeat_interleave(k // 2).float()[:, None]
    rois = torch.cat([b, ctr - size / 2, ctr + size / 2], 1).cuda().contiguous()
    return feats, rois


class _RefFn(torch.autograd.Function):
    """The reference op as its RoIAlignFunction wraps it."""

    @staticmethod
    def forward(ctx, feat, rois, out, scale, sample_num):
        from oracle import ref_roi_align as REF
        ctx.save_for_backward(rois)
        ctx.args = (scale, sample_num, feat.shape)
        return REF.forward(feat, rois, out, out, scale, sample_num)

    @staticmethod
    def backward(ctx, gout):
        from oracle import ref_roi_align as REF
        scale, sample_num, shape = ctx.args
        return REF.backward(gout, ctx.saved_tensors[0], scale, sample_num, shape), None, None, None, None


def _events(fn, reps):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    fn()
    torch.cuda.synchronize()
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=20)
    ap.add_argument('--rounds', type=int, default=5)
    ap.add_argument('--json', default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), 'bench_roi_align needs a GPU'
    import roi_align_oracle as R
    from oracle import ref_roi_align as REF
    from torchvision.ops import roi_align as tv_roi_align
    name, power = _gpu_info()
    print('GPU: %s, power limit %s' % (name, power))
    gen = torch.Generator().manual_seed(0)
    results = {}
    for shape, cfg in SHAPES.items():
        ext = SingleRoIExtractor(dict(type='RoIAlign', out_size=cfg['out'], sample_num=2), 256, cfg['strides'])
        feats, rois = _inputs(cfg, gen)
        feats = [f.requires_grad_(True) for f in feats]
        gout = torch.randn(cfg['k'], 256, cfg['out'], cfg['out'], generator=gen).cuda()

        def ref_op(feat, r, oh, ow, scale, sample_num):
            return _RefFn.apply(feat, r.contiguous(), oh, scale, sample_num)

        def run(which, backward):
            def fn():
                for f in feats:
                    f.grad = None
                if which == 'native':
                    out = ext(feats, rois)
                elif which == 'reference':
                    out = R.extractor(ref_op, feats, rois, (cfg['out'], cfg['out']), cfg['strides'], 2, 56, 256)
                else:
                    out = tv_roi_align(feats[0], rois, (cfg['out'], cfg['out']), 1 / cfg['strides'][0], 2)
                if backward:
                    out.backward(gout)
            return fn

        with torch.no_grad():
            same = torch.equal(ext(feats, rois),
                               R.extractor(REF.forward, [f.detach() for f in feats], rois, (cfg['out'], cfg['out']),
                                           cfg['strides'], 2, 56, 256))
        times = {}
        for _ in range(args.rounds):
            for which in ('native', 'reference', 'torchvision'):
                for bwd in (False, True):
                    key = '%s_%s' % (which, 'fwd_bwd' if bwd else 'fwd')
                    times.setdefault(key, []).append(_events(run(which, bwd), args.reps))
        med = {k: float(np.median(v)) for k, v in times.items()}
        results[shape] = dict(bitwise_equal=same, ms=med)
        print('%-20s bitwise=%s  ' % (shape, same) + '  '.join('%s %.3f' % (k, v) for k, v in med.items()))
        print('%-20s speed-up fwd %.2fx  fwd+bwd %.2fx' % (
            '', med['reference_fwd'] / med['native_fwd'], med['reference_fwd_bwd'] / med['native_fwd_bwd']))
        del feats
    print(json.dumps(dict(gpu=name, power_limit=power, results=results)))
    if args.json:
        with open(args.json, 'w') as f:
            json.dump(dict(gpu=name, power_limit=power, results=results), f, indent=1)


if __name__ == '__main__':
    main()
