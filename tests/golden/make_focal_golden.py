"""Regenerate tests/golden/focal_head_ref_n256.npz: what the reference's own heads with a sigmoid FocalLoss return,
run in place on CPU through oracle/ref_shim.py with the focal-loss op replaced by its float64 restatement
(tests/focal_oracle.py), for the seeded head and inputs of tests/focal_oracle.fixture_inputs():

  shared_*  SharedFCBBoxHead, the block of configs/transferred/faster_rcnn_r50_fpn_1x_lvis_focalloss{,_all}.py
  bfocal_*  ReweightBBoxHead, the block of faster_rcnn_r50_fpn_1x_lvis_reweighthead_bfocal.py ('bf' class weights)

each with loss_cls, acc, loss_bbox and the gradients of loss_cls + loss_bbox w.r.t. fc_cls.weight (every 4th row),
fc_cls.bias and the RoI features.  Needs a reference checkout:

    python tests/golden/make_focal_golden.py
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

import focal_oracle as FO  # noqa: E402


def main():
    inp = FO.fixture_inputs()
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, 'cls_weight_bf.pt')
        torch.save(inp['cls_weight'], path)
        heads = FO.build_reference_heads(path, **FO.fixture_sizes())
    out = {}
    for key, head in heads.items():
        for name, v in FO.run_head(head, inp).items():
            out['%s_%s' % (key, name)] = v.numpy()
    np.savez_compressed(FO.FIXTURE, **{k: np.asarray(v, dtype=np.float32) for k, v in out.items()})
    print({k: (v.shape, float(np.abs(v).max())) for k, v in out.items()})
    print('wrote', FO.FIXTURE)


if __name__ == '__main__':
    main()
