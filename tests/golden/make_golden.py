"""Generate tests/golden/*.npz by executing the REFERENCE'S OWN source (through
oracle/ref_shim.py) on CPU.  Run in the build container where /root/reference exists:

    python tests/golden/make_golden.py

The reference ships no golden vectors for this path; these fixtures are the
pinning: inputs + the reference's outputs (per-bin losses, sampled masks, avg factors, grads,
merged scores).  They travel to the GPU box, where /root/reference does not exist.

Fixture shapes are small on the K (feature) axis so the files stay tiny; the logit axis keeps
the full 1236-wide, 5-bin structure.
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from balancedgroupsoftmax_b200.tables import synthetic_tables  # noqa: E402
from oracle import ref_shim  # noqa: E402

OUT = os.path.dirname(os.path.abspath(__file__))


def make_case(name, N, K, npos, seed, wstd, ratio=8.0, gout=None, zipf=False):
    tables = synthetic_tables(1231, seed=0)
    head = ref_shim.build_reference_head(tables, others_sample_ratio=ratio, fc_out_channels=K)
    torch.manual_seed(seed)
    np.random.seed(seed)
    with torch.no_grad():
        head.fc_cls.weight.normal_(0, wstd)
        head.fc_cls.bias.normal_(0, 0.1)
    x = torch.relu(torch.randn(N, K))
    labels = torch.zeros(N, dtype=torch.long)
    if npos > 0:
        if zipf:
            r = np.random.zipf(1.3, size=npos)
            labels[:npos] = torch.from_numpy(((r - 1) % 1230) + 1)
        else:
            labels[:npos] = torch.randint(1, 1231, (npos,))
    rec = {}
    orig = head._remap_labels

    def wrap(l):
        r = orig(l)
        rec['r'] = r
        return r

    head._remap_labels = wrap
    xr = x.clone().requires_grad_(True)
    z = head.fc_cls(xr)
    losses = head.loss(z, None, labels, None, None, None)
    g = [1.0] * 5 if gout is None else gout
    total = sum(gi * losses['loss_cls_bin%d' % i] for i, gi in enumerate(g))
    total.backward()
    merged = head._merge_score(z.detach())
    new_labels, new_weights, new_avg = rec['r']
    np.savez_compressed(
        os.path.join(OUT, name + '.npz'),
        x=x.numpy(), weight=head.fc_cls.weight.detach().numpy(), bias=head.fc_cls.bias.detach().numpy(),
        labels=labels.numpy(), ratio=np.float64(ratio), gout=np.asarray(g, dtype=np.float32),
        logits_sample=z.detach()[:, ::29].numpy(),
        losses=np.asarray([losses['loss_cls_bin%d' % i].item() for i in range(5)], dtype=np.float64),
        bin_labels=np.stack([t.numpy() for t in new_labels]).astype(np.int16),
        wmask=np.stack([w.numpy() for w in new_weights]).astype(np.uint8),
        avg=np.asarray(new_avg, dtype=np.float64),
        dW=head.fc_cls.weight.grad.numpy(), db=head.fc_cls.bias.grad.numpy(), dX=xr.grad.numpy(),
        merged_argmax=merged.argmax(1).numpy().astype(np.int16),
        merged_fg_argmax=(merged[:, 1:].argmax(1) + 1).numpy().astype(np.int16),
        merged_rowsum=merged.sum(1).numpy(), merged_sample=merged[:, ::37].numpy(),
        seed=np.int64(seed),
    )
    print(name, 'losses', [round(losses['loss_cls_bin%d' % i].item(), 5) for i in range(5)], 'avg', new_avg)


if __name__ == '__main__':
    assert ref_shim.available(), 'reference checkout not reachable'
    make_case('ref_n96_k64', N=96, K=64, npos=24, seed=1, wstd=0.3)
    make_case('ref_n257_k64_cascade', N=257, K=64, npos=70, seed=2, wstd=0.2, gout=[1.0, 0.5, 0.25, 0.5, 1.0])
    make_case('ref_n64_k32_allbg', N=64, K=32, npos=0, seed=3, wstd=0.3)
    make_case('ref_n48_k32_allfg', N=48, K=32, npos=48, seed=4, wstd=0.3, zipf=True)
    # known-answer numbers of the weighted_loss doctest (mmdet/models/losses/utils.py:66-83), evaluated by
    # the reference's own decorator
    ns = ref_shim.load()

    @ns.weighted_loss
    def l1_loss(pred, target):
        return (pred - target).abs()

    pred, target, weight = torch.Tensor([0, 2, 3]), torch.Tensor([1, 1, 1]), torch.Tensor([1, 0, 1])
    np.savez(os.path.join(OUT, 'weighted_loss_kat.npz'),
             mean=l1_loss(pred, target).item(), weighted=l1_loss(pred, target, weight).item(),
             none=l1_loss(pred, target, reduction='none').numpy(),
             avg2=l1_loss(pred, target, weight, avg_factor=2).item())
