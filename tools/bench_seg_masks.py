"""Time FCNMaskHead.get_seg_masks per image: the host loop (BAGS_SEGM_NATIVE=0) against the native route, alternated in
one run, on LVIS-sized inputs (1231 classes, 28 x 28 logits, n = 100 and 300 detections -- max_per_img of the mask
configs is 300 -- on 480 x 640 and 800 x 1333 images).

    python tools/bench_seg_masks.py [--reps 5] [--json out.json]

Per case and route: wall time of the call ending in a device synchronise (median of the reps), the kernel time of the
two bags_segm_rle launches from CUDA events (native route only), and the bytes each route copies device to host.  The
host loop needs pycocotools; without it, the loop's encoder is tests/segm_oracle.py's restatement (named in the output).
Both routes' outputs are compared before anything is timed.
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

from balancedgroupsoftmax_b200 import _native as nat  # noqa: E402
from balancedgroupsoftmax_b200 import mask_head as MH  # noqa: E402
from balancedgroupsoftmax_b200 import ops  # noqa: E402

CLASSES = 1231


def _encoder():
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


def _inputs(n, img_h, img_w, seed=0):
    dev = torch.device('cuda', 0)
    rng = np.random.default_rng(seed)
    w = rng.integers(8, img_w // 2, n)
    h = rng.integers(8, img_h // 2, n)
    x0, y0 = rng.integers(0, img_w - w), rng.integers(0, img_h - h)
    det = np.stack([x0, y0, x0 + w - 1, y0 + h - 1, rng.random(n)], 1).astype(np.float32)
    g = torch.Generator(dev).manual_seed(seed)
    logits = torch.randn(n, CLASSES, 28, 28, generator=g, device=dev) * 3
    labels = torch.randint(0, CLASSES - 1, (n,), generator=g, device=dev)
    return torch.from_numpy(det).to(dev), labels, logits


def _gpu_info():
    name = torch.cuda.get_device_name(0)
    try:
        out = subprocess.run(['nvidia-smi', '--query-gpu=power.limit', '--format=csv,noheader', '-i', '0'],
                             stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        out = 'unknown'
    return name, out


class _KernelTimer:
    """CUDA events around every bags_segm_rle launch (wraps the ctypes function ops.seg_masks_rle calls)."""

    def __init__(self):
        self.pairs = []
        self._fn = None

    def __enter__(self):
        lib = nat.lib()
        self._fn = fn = lib.bags_segm_rle

        def timed(*args):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            rc = fn(*args)
            b.record()
            self.pairs.append((a, b))
            return rc
        lib.bags_segm_rle = timed
        return self

    def __exit__(self, *exc):
        nat.lib().bags_segm_rle = self._fn

    def ms(self):
        torch.cuda.synchronize()
        return sum(a.elapsed_time(b) for a, b in self.pairs)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=5)
    ap.add_argument('--json', default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), 'bench_seg_masks needs a GPU'
    encoder = _encoder()
    name, power = _gpu_info()
    print('GPU: %s, power limit %s; host-loop encoder: %s' % (name, power, encoder))
    head = MH.FCNMaskHead(num_convs=1, in_channels=4, conv_out_channels=4, num_classes=CLASSES)
    cfg = dict(mask_thr_binary=0.5)
    results = []
    for img_h, img_w in ((480, 640), (800, 1333)):
        for n in (100, 300):
            det, labels, logits = _inputs(n, img_h, img_w)
            call = (logits, det, labels, cfg, (img_h, img_w, 3), 1.0, True)

            def run(native):
                os.environ['BAGS_SEGM_NATIVE'] = '1' if native else '0'
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                out = head.get_seg_masks(*call)
                torch.cuda.synchronize()
                return out, time.perf_counter() - t0

            ref, _ = run(False)
            got, _ = run(True)
            assert got == ref, 'native and host masks differ'
            times = {False: [], True: []}
            kernel_ms = []
            for _ in range(args.reps):
                for native in (False, True):
                    if native:
                        with _KernelTimer() as kt:
                            _, t = run(True)
                        kernel_ms.append(kt.ms())
                    else:
                        _, t = run(False)
                    times[native].append(t)
            bytes_native = 16 * n + 8 * n + 8 * n + sum(len(r['counts']) for v in got for r in v)
            row = dict(img=[img_h, img_w], n=n, host_ms=1e3 * float(np.median(times[False])),
                       native_ms=1e3 * float(np.median(times[True])), kernel_ms=float(np.median(kernel_ms)),
                       d2h_bytes_host=n * CLASSES * 28 * 28 * 4 + 20 * n + 8 * n, d2h_bytes_native=bytes_native)
            results.append(row)
            print('%4d x %4d  n=%3d  host %8.1f ms  native %7.2f ms  (bags_segm_rle kernels %6.3f ms)  '
                  'D2H bytes host %d  native %d' % (img_h, img_w, n, row['host_ms'], row['native_ms'],
                                                      row['kernel_ms'], row['d2h_bytes_host'],
                                                      row['d2h_bytes_native']))
    os.environ.pop('BAGS_SEGM_NATIVE', None)
    if args.json:
        with open(args.json, 'w') as f:
            json.dump(dict(gpu=name, power_limit=power, encoder=encoder, results=results), f, indent=1)


if __name__ == '__main__':
    main()
