"""Time the mask heads' training targets (FCNMaskHead.get_target -> mask_target) on its routes, alternated in one run:

    host     numpy gt masks: the host loop (boxes and gt indices to the host, cv2.resize per RoI, one upload)
    numpy    numpy gt masks through ops.mask_targets: all masks of the call uploaded from one pinned buffer, one launch
    cuda     gt masks already on the GPU (uint8 tensors): one launch, no host sync

Workloads: Mask R-CNN (2 images x 128 positives, one call per step) and HTC (1 image x 128 positives, three calls per
step with the same gt masks; its numpy route uploads them once per step), masks of 800 x 1344, num_gt in {3, 15, 100}.

    python tools/bench_mask_target.py [--reps 20] [--json out.json]

Per workload and route: host wall time of the targets of one step ending in a device synchronise (median), the
device time of the bags_mask_target launches from CUDA events, the bytes and device time of the numpy route's upload,
and a whole FCNMaskHead training step (get_target -> forward -> loss -> backward; 4 convs, 256 channels, 1231 classes)
per route.  All routes' targets are compared bitwise before anything is timed.
"""
import argparse
import json
import os
import subprocess
import sys
import time
from types import SimpleNamespace

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from balancedgroupsoftmax_b200 import mask_head as MH  # noqa: E402
from balancedgroupsoftmax_b200 import ops  # noqa: E402

H, W, POS, CLASSES = 800, 1344, 128, 1231
CFG = dict(mask_size=28)


def _gpu_info():
    name = torch.cuda.get_device_name(0)
    try:
        out = subprocess.run(['nvidia-smi', '--query-gpu=power.limit', '--format=csv,noheader', '-i', '0'],
                             stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        out = 'unknown'
    return name, out


def _inputs(images, num_gt, seed=0):
    dev = torch.device('cuda', 0)
    rng = np.random.default_rng(seed)
    samp, masks = [], []
    for _ in range(images):
        x1, y1 = rng.random(POS) * W * 0.8, rng.random(POS) * H * 0.8
        bw, bh = 8 + rng.random(POS) * W * 0.3, 8 + rng.random(POS) * H * 0.3
        boxes = np.stack([x1, y1, x1 + bw, y1 + bh], 1).astype(np.float32)
        samp.append(SimpleNamespace(pos_bboxes=torch.from_numpy(boxes).to(dev),
                                    pos_assigned_gt_inds=torch.from_numpy(rng.integers(0, num_gt, POS)).to(dev)))
        m = np.zeros((num_gt, H, W), np.uint8)
        for k in range(num_gt):
            y0, x0 = rng.integers(0, H - 50), rng.integers(0, W - 50)
            m[k, y0:y0 + rng.integers(20, 400), x0:x0 + rng.integers(20, 600)] = 1
        masks.append(m)
    return samp, masks


def _targets(route, head, samp, masks, calls):
    """The targets of one step: ``calls`` get_target calls on the route's masks."""
    if route == 'host':
        return [head.get_target(samp, masks, CFG) for _ in range(calls)]
    if route == 'numpy':
        dev_masks = ops.upload_masks(masks, samp[0].pos_bboxes.device)      # once per step, for every call
    else:
        dev_masks = masks
    return [head.get_target(samp, dev_masks, CFG) for _ in range(calls)]


def _wall(fn, reps):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return out, time.perf_counter() - t0


def _events(fn, reps):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    fn()
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=20)
    ap.add_argument('--json', default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), 'bench_mask_target needs a GPU'
    name, power = _gpu_info()
    print('GPU: %s, power limit %s' % (name, power))
    dev = torch.device('cuda', 0)
    torch.manual_seed(0)
    head = MH.FCNMaskHead(num_convs=4, in_channels=256, conv_out_channels=256, num_classes=CLASSES)
    head.init_weights()
    head = head.to(dev).train()
    results = []
    for wl, images, calls in (('mask_rcnn', 2, 1), ('htc', 1, 3)):
        for num_gt in (3, 15, 100):
            samp, masks = _inputs(images, num_gt, seed=num_gt)
            cuda_masks = [torch.from_numpy(m).to(dev) for m in masks]
            route_masks = dict(host=masks, numpy=masks, cuda=cuda_masks)
            want = _targets('host', head, samp, masks, 1)[0]
            for r in ('numpy', 'cuda'):
                assert torch.equal(_targets(r, head, samp, route_masks[r], 1)[0], want), r
            # targets of one step per route, alternated
            times = {r: [] for r in route_masks}
            for _ in range(args.reps):
                for r in route_masks:
                    times[r].append(_wall(lambda: _targets(r, head, samp, route_masks[r], calls), args.reps)[1])
            kernel_ms = _events(lambda: ops.mask_targets([s.pos_bboxes for s in samp],
                                                         [s.pos_assigned_gt_inds for s in samp], cuda_masks, 28),
                                args.reps)
            upload_bytes = sum(m.nbytes for m in masks)
            upload_dev_ms = _events(lambda: ops.upload_masks(masks, dev), max(args.reps // 4, 3))
            _, upload_wall = min((_wall(lambda: ops.upload_masks(masks, dev), 1) for _ in range(5)),
                                 key=lambda p: p[1])
            # a whole FCNMaskHead training step per route, alternated
            x = torch.randn(images * POS, 256, 14, 14, device=dev)
            labels = torch.randint(0, CLASSES - 1, (images * POS,), device=dev)

            def step(r):
                head.zero_grad()
                ts = _targets(r, head, samp, route_masks[r], calls)
                loss = sum(head.loss(head(x), t, labels)['loss_mask'].sum() for t in ts)
                loss.backward()

            steps = {r: [] for r in route_masks}
            for r in route_masks:
                step(r)
            for _ in range(args.reps):
                for r in route_masks:
                    steps[r].append(_wall(lambda: step(r), 1)[1])
            row = dict(workload=wl, images=images, calls=calls, num_gt=num_gt,
                       targets_ms={r: 1e3 * float(np.median(v)) for r, v in times.items()},
                       step_ms={r: 1e3 * float(np.median(v)) for r, v in steps.items()},
                       kernel_ms=kernel_ms, upload_bytes=upload_bytes, upload_device_ms=upload_dev_ms,
                       upload_wall_ms=1e3 * upload_wall)
            results.append(row)
            print('%-9s num_gt=%3d  targets/step: host %7.2f ms  numpy %7.2f ms  cuda %6.3f ms | kernel %6.3f ms | '
                  'upload %6.1f MB: device %6.2f ms, wall %6.2f ms | head step: host %7.2f  numpy %7.2f  cuda %7.2f ms'
                  % (wl, num_gt, row['targets_ms']['host'], row['targets_ms']['numpy'], row['targets_ms']['cuda'],
                     kernel_ms, upload_bytes / 1e6, upload_dev_ms, row['upload_wall_ms'], row['step_ms']['host'],
                     row['step_ms']['numpy'], row['step_ms']['cuda']))
    if args.json:
        with open(args.json, 'w') as f:
            json.dump(dict(gpu=name, power_limit=power, results=results), f, indent=1)


if __name__ == '__main__':
    main()
