"""Time the mask heads' test path per image, from the mask head's forward to the segm result: the label-only route
(an eval MaskPredHandle: bags_mask_logits computes each detection's channel) against the dense route (the same calls
handed conv_logits' [n, 1231, 28, 28] logits), alternated in one run.

    python tools/bench_mask_eval.py [--reps 10] [--json out.json]      (prints the results as one JSON line)

Sequences, at n = 100 and 300 detections (max_per_img of the LVIS mask configs is 300) on an 800 x 1333 image, with
fp32 RoI features [n, 256, 14, 14] as the configs run them:
  maskrcnn  one FCNMaskHead (4 convs, deconv, 1231 classes), get_seg_masks (fcn_mask_head.py:125-181)
  htc       three HTCMaskHeads with mask_info_flow, each stage's mask_pred.gather(1, labels), the sigmoids averaged
            on the host (merge_aug_masks' np.mean) and get_seg_masks_without (htc.py:403-421)
Reported per case and route: the wall time ending in a device synchronise (median of the reps) and the peak memory
above what is live before the forward; per n, the CUDA-event time of conv_logits (cuDNN, the default TF32 setting)
against bags_mask_logits on the same y, in fp32 and bf16; the card's name and power limit, read in this run.
Before anything is timed, both routes' outputs are compared with TF32 off (both then multiply in fp32 and differ only
in summation order): the label-channel logits (asserted within 1e-5 of the largest), and the RLE results (equal, or
how many masks and pixels differ: a pixel whose resized probability lies within a rounding of the threshold can flip).
"""
import argparse
import json
import os
import subprocess
import sys
import time
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))

from balancedgroupsoftmax_b200 import mask_head as MH  # noqa: E402
from balancedgroupsoftmax_b200 import ops  # noqa: E402

CLASSES = 1231
CFG = dict(mask_thr_binary=0.5)
IMG = (800, 1333)
DEV = torch.device('cuda', 0)


def _encoder():
    """pycocotools for the host loop of a box that leaves the image (none does here), else the tests' restatement."""
    try:
        import pycocotools.mask  # noqa: F401
        return 'pycocotools'
    except ImportError:
        import segm_oracle as SO
        mod = types.ModuleType('pycocotools.mask')
        mod.encode = SO.encode
        pkg = types.ModuleType('pycocotools')
        pkg.mask = mod
        sys.modules['pycocotools'], sys.modules['pycocotools.mask'] = pkg, mod
        return 'tests/segm_oracle.py (pycocotools not installed)'


def _gpu_info():
    name = torch.cuda.get_device_name(0)
    try:
        out = subprocess.run(['nvidia-smi', '--query-gpu=power.limit', '--format=csv,noheader', '-i', '0'],
                             stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        out = 'unknown'
    return name, out


def _detections(n, seed):
    img_h, img_w = IMG
    rng = np.random.default_rng(seed)
    w, h = rng.integers(8, img_w // 2, n), rng.integers(8, img_h // 2, n)
    x0, y0 = rng.integers(0, img_w - w), rng.integers(0, img_h - h)
    det = np.stack([x0, y0, x0 + w - 1, y0 + h - 1, rng.random(n)], 1).astype(np.float32)
    labels = torch.from_numpy(rng.integers(0, CLASSES - 1, n)).long()
    return torch.from_numpy(det).to(DEV), labels.to(DEV)


def _heads(cls, count):
    out = []
    for i in range(count):
        torch.manual_seed(i)
        head = cls(num_convs=4, in_channels=256, conv_out_channels=256, num_classes=CLASSES)
        head.init_weights()
        out.append(head.to(DEV).eval())
    return out


def maskrcnn(heads, feats, det, labels, dense):
    """(segm result, [n, 1, 28, 28] label-channel logits)."""
    head = heads[0]
    pred = head(feats)
    if dense:
        pred = pred.tensor()
        chan = pred[torch.arange(pred.shape[0], device=DEV), labels + 1][:, None]
    else:
        chan = pred.channel_logits(labels + 1)
    return head.get_seg_masks(pred, det, labels, CFG, IMG + (3,), 1.0, True), chan


def htc(heads, feats, det, labels, dense):
    """(segm result, the last stage's gathered logits)."""
    index = (labels.unsqueeze(1) + 1).unsqueeze(2).unsqueeze(3).expand(-1, -1, 28, 28)
    aug, last_feat = [], None
    for head in heads:
        pred, last_feat = head(feats, last_feat)
        g = (pred.tensor() if dense else pred).gather(1, index)
        aug.append(g.sigmoid().cpu().numpy())
    merged = np.mean(aug, axis=0)
    return heads[-1].get_seg_masks_without(merged, det, labels, CFG, IMG + (3,), 1.0, True), g


def _rle_diff(got, want):
    """(masks, pixels) that differ between two segm results of the same detections: a logit that moves by a rounding
    can cross the threshold after the resize."""
    import segm_oracle as SO
    masks = pixels = 0
    for g_list, w_list in zip(got, want):
        for g, w in zip(g_list, w_list):
            if g != w:
                masks += 1
                pixels += int((SO.decode(g) != SO.decode(w)).sum())
    return masks, pixels


def _timed(fn, *args):
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    t0 = time.perf_counter()
    with torch.no_grad():
        fn(*args)
    torch.cuda.synchronize()
    return time.perf_counter() - t0, torch.cuda.max_memory_allocated() - base


def _event_ms(fn, reps=20):
    with torch.no_grad():
        for _ in range(3):
            fn()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(reps):
            fn()
        b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=10)
    ap.add_argument('--json', default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), 'bench_mask_eval needs a GPU'
    encoder = _encoder()
    name, power = _gpu_info()
    print('GPU: %s, power limit %s; host-loop encoder: %s' % (name, power, encoder))
    seqs = dict(maskrcnn=(maskrcnn, _heads(MH.FCNMaskHead, 1)), htc=(htc, _heads(MH.HTCMaskHead, 3)))
    results, kernels = [], []
    for n in (100, 300):
        det, labels = _detections(n, seed=n)
        feats = torch.relu(torch.randn(n, 256, 14, 14, device=DEV, generator=torch.Generator(DEV).manual_seed(n)))
        for seq, (fn, heads) in seqs.items():
            # equal outputs first, TF32 off so that both routes multiply in fp32
            tf32 = torch.backends.cudnn.allow_tf32
            torch.backends.cudnn.allow_tf32 = False
            try:
                with torch.no_grad():
                    got, zg = fn(heads, feats, det, labels, False)
                    want, zw = fn(heads, feats, det, labels, True)
            finally:
                torch.backends.cudnn.allow_tf32 = tf32
            assert zg.shape == zw.shape == (n, 1, 28, 28), (zg.shape, zw.shape)
            zdiff = ((zg.double() - zw.double()).abs().max() / zw.double().abs().max()).item()
            assert zdiff < 1e-5, ('label-channel logits differ', seq, n, zdiff)
            rle_equal = got == want
            diff_masks, diff_pixels = _rle_diff(got, want)
            times, peaks = {False: [], True: []}, {False: 0, True: 0}
            for dense in (False, True):          # warm-up of both routes
                _timed(fn, heads, feats, det, labels, dense)
            for _ in range(args.reps):
                for dense in (False, True):
                    t, peak = _timed(fn, heads, feats, det, labels, dense)
                    times[dense].append(t)
                    peaks[dense] = max(peaks[dense], peak)
            row = dict(seq=seq, n=n, label_only_ms=1e3 * float(np.median(times[False])),
                       dense_ms=1e3 * float(np.median(times[True])), label_only_peak_mb=peaks[False] / 2 ** 20,
                       dense_peak_mb=peaks[True] / 2 ** 20, dense_logits_mb=n * CLASSES * 28 * 28 * 4 / 2 ** 20,
                       rle_equal_without_tf32=rle_equal, differing_masks_without_tf32=diff_masks,
                       differing_pixels_without_tf32=diff_pixels, logits_max_rel_diff_without_tf32=zdiff)
            results.append(row)
            print('%-8s n=%3d  label-only %8.2f ms (peak %7.1f MB)  dense %8.2f ms (peak %7.1f MB)  RLE equal %s '
                  '(%d masks, %d pixels differ)  logits rel diff %.1e' % (
                      seq, n, row['label_only_ms'], row['label_only_peak_mb'], row['dense_ms'], row['dense_peak_mb'],
                      rle_equal, diff_masks, diff_pixels, zdiff))
        conv = seqs['maskrcnn'][1][0].conv_logits
        ch = labels + 1
        for dtype in (torch.float32, torch.bfloat16):
            y = torch.relu(torch.randn(n, 256, 28, 28, device=DEV)).to(dtype)
            conv_d = torch.nn.Conv2d(256, CLASSES, 1).to(DEV, dtype)
            conv_d.load_state_dict(conv.state_dict())
            row = dict(n=n, dtype=str(dtype).replace('torch.', ''),
                       conv_logits_ms=_event_ms(lambda: conv_d(y)),
                       mask_logits_ms=_event_ms(lambda: ops.mask_channel_logits(y, conv.weight, conv.bias, ch)),
                       y_mb=y.numel() * y.element_size() / 2 ** 20)
            kernels.append(row)
            print('kernels n=%3d %-8s conv_logits %7.3f ms  bags_mask_logits %7.3f ms  (y %.0f MB)' % (
                n, row['dtype'], row['conv_logits_ms'], row['mask_logits_ms'], row['y_mb']))
    summary = dict(gpu=name, power_limit=power, encoder=encoder, tf32=torch.backends.cudnn.allow_tf32,
                   results=results, kernels=kernels)
    print(json.dumps(summary))
    if args.json:
        with open(args.json, 'w') as f:
            json.dump(summary, f, indent=1)


if __name__ == '__main__':
    main()
