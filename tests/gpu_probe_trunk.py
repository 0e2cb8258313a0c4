"""Timing of the head's trunk layers on this library's tcgen05 GEMMs vs torch (cuBLAS) on the same GPU:
python tests/gpu_probe_trunk.py    -> one JSON line (CUDA events, rotating buffers > L2 are not needed: the 25 MB weight of
shared_fcs.0 plus activations are re-read from L2 / HBM alike in both arms)."""
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from balancedgroupsoftmax_b200 import ops  # noqa: E402


def timed(fn, reps=20):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps * 1e3


def main():
    dev = torch.device('cuda', 0)
    peak = 1698.5
    try:
        peak = float(json.load(open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))),
                                                 'MEASURED_PEAKS.json')))['bf16_tflops'])
    except Exception:
        pass
    out = {'peak_bf16_tflops_burst': peak, 'layers': {}}
    g = torch.Generator().manual_seed(0)
    for name, (N, K, C, relu) in {'shared_fcs.0 (1024 RoIs x 12544 -> 1024, ReLU)': (1024, 12544, 1024, True),
                                  'shared_fcs.1 (1024 x 1024 -> 1024, ReLU)': (1024, 1024, 1024, True),
                                  'fc_reg (1024 x 1024 -> 4924)': (1024, 1024, 4924, False)}.items():
        x = torch.randn(N, K, generator=g).to(dev).bfloat16().requires_grad_(True)
        W = torch.nn.Parameter((torch.randn(C, K, generator=g) / K ** 0.5).to(dev))
        b = torch.nn.Parameter(torch.zeros(C, device=dev))
        od = torch.bfloat16 if relu else torch.float32
        dy = torch.randn(N, C, generator=g).to(dev).to(od)
        flops = 2.0 * N * K * C

        def ours_fwd():
            return ops.LinearActFunction.apply(x, W, b, relu, torch.bfloat16, od)

        def ours_fb():
            x.grad = W.grad = b.grad = None
            ours_fwd().backward(dy)

        lin = torch.nn.Linear(K, C).to(dev)
        with torch.no_grad():
            lin.weight.copy_(W)

        def torch_fwd():
            with torch.autocast('cuda', dtype=torch.bfloat16):
                y = lin(x)
                return torch.relu(y) if relu else y

        def torch_fb():
            x.grad = None
            lin.zero_grad(set_to_none=True)
            y = torch_fwd()
            y.backward(dy.to(y.dtype))

        r = {'ours_fwd_us': timed(ours_fwd), 'ours_fwd_bwd_us': timed(ours_fb), 'torch_bf16_autocast_fwd_us': timed(torch_fwd),
             'torch_bf16_autocast_fwd_bwd_us': timed(torch_fb)}
        r['ours_fwd_tflops'] = flops / (r['ours_fwd_us'] * 1e-6) / 1e12
        r['ours_fwd_frac_of_burst_peak'] = r['ours_fwd_tflops'] / peak
        r['ours_fwd_bwd_tflops'] = 3 * flops / (r['ours_fwd_bwd_us'] * 1e-6) / 1e12
        out['layers'][name] = {k: round(v, 3) for k, v in r.items()}
    print(json.dumps(out))


if __name__ == '__main__':
    main()
