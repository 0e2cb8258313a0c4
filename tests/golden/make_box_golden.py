"""Regenerate tests/golden/box_loss_ref_n256.npz: what the reference's own class-specific heads return for the box term,
run on CPU in float64 through oracle/ref_shim.py, for the seeded parameters and inputs of tests/box_oracle.fixture_inputs():

  gs_*        GSBBoxHeadWith0 (synthetic 1231-class tables), the head of configs/bags/gs_faster_rcnn_*
  reweight_*  ReweightBBoxHead, the head of the re-weighting baselines

each with loss_bbox and the gradients of loss_bbox w.r.t. fc_reg.weight (every 7th row), fc_reg.bias and the RoI
features.  Needs a reference checkout:

    python tests/golden/make_box_golden.py
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

import box_oracle as BO  # noqa: E402


def reference_heads(tmpdir):
    """The reference's GSBBoxHeadWith0 and ReweightBBoxHead at the fixture's sizes (CPU)."""
    import reweight_oracle as R
    from balancedgroupsoftmax_b200.tables import synthetic_tables
    from oracle import ref_shim
    sizes = dict(in_channels=BO.FIX_IN, fc_out_channels=BO.FIX_FC, roi_feat_size=BO.FIX_ROI)
    gs = ref_shim.build_reference_head(synthetic_tables(), tmpdir=tmpdir, **sizes)
    path = os.path.join(tmpdir, 'cls_weight.pt')
    torch.save(torch.ones(1231), path)
    rw = R.build_reference_reweight_bbox_head(path, num_classes=1231, **sizes)
    return {'gs': gs, 'reweight': rw}


def main():
    inp = BO.fixture_inputs()
    out = {}
    with tempfile.TemporaryDirectory() as d:
        for key, head in reference_heads(d).items():
            for name, v in BO.run_box_loss(head, inp, dtype=torch.float64).items():
                out['%s_%s' % (key, name)] = v.numpy()
    np.savez_compressed(BO.FIXTURE, **{k: np.asarray(v, dtype=np.float32) for k, v in out.items()})
    print({k: (v.shape, float(np.abs(v).max())) for k, v in out.items()})
    print('wrote', BO.FIXTURE)


if __name__ == '__main__':
    main()
