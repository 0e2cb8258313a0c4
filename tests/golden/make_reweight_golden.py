"""Regenerate tests/golden/reweight_head_ref_n256.npz: what the reference's own ReweightBBoxHead (run in place on CPU
through oracle/ref_shim.py) returns for the seeded head and inputs of tests/reweight_oracle.fixture_inputs():
loss_cls, acc, loss_bbox, and the gradients of their sum (acc excluded) w.r.t. fc_cls.weight (every 4th row),
fc_cls.bias and the RoI features.  Needs a reference checkout:

    python tests/golden/make_reweight_golden.py
"""
import os
import sys
import tempfile

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(HERE))

import reweight_oracle as R  # noqa: E402


def main():
    inp = R.fixture_inputs()
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, 'cls_weight.pt')
        torch.save(inp['cls_weight'], path)
        head = R.build_reference_reweight_bbox_head(path, num_classes=R.FIX_C, in_channels=R.FIX_IN,
                                                    fc_out_channels=R.FIX_FC, roi_feat_size=R.FIX_ROI)
    missing, unexpected = head.load_state_dict(inp['params'], strict=True)
    assert not missing and not unexpected
    head.train()
    feats = inp['feats'].clone().requires_grad_(True)
    cls_score, bbox_pred = head(feats)
    losses = head.loss(cls_score, bbox_pred, inp['labels'], inp['label_weights'], inp['bbox_targets'],
                       inp['bbox_weights'])
    (losses['loss_cls'] + losses['loss_bbox']).backward()
    out = dict(loss_cls=losses['loss_cls'].detach().numpy(), acc=losses['acc'].detach().numpy(),
               loss_bbox=losses['loss_bbox'].detach().numpy(),
               dW4=head.fc_cls.weight.grad.numpy()[::4],   # every 4th class row keeps the file small
               db=head.fc_cls.bias.grad.numpy(), dX=feats.grad.numpy())
    np.savez_compressed(R.FIXTURE, **{k: np.asarray(v, dtype=np.float32) for k, v in out.items()})
    print({k: (v.shape, float(np.abs(v).max())) for k, v in out.items()})
    print('wrote', R.FIXTURE)


if __name__ == '__main__':
    main()
