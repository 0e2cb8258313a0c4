"""Regenerate tests/golden/mask_loss_ref_p12.npz: what the reference's own mask heads return for the mask term, run on
CPU in float64 through oracle/ref_shim.py (tests/mask_oracle.reference()), for the seeded parameters and inputs of
tests/mask_oracle.fixture_inputs():

  fcn_*  FCNMaskHead with 1231 classes, the head of configs/bags/gs_mask_rcnn_r50_fpn_1x_lvis.py
  htc_*  HTCMaskHead with class_agnostic=True (one logits channel, label 0 for every RoI), fed a res_feat

each with loss_mask and the gradients of loss_mask w.r.t. conv_logits.weight (every 5th row), conv_logits.bias and the
input of conv_logits (dY).  Needs a reference checkout:

    python tests/golden/make_mask_golden.py
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(HERE))

import mask_oracle as MO  # noqa: E402


def reference_heads():
    ref = MO.reference()
    return {'fcn': ref.FCNMaskHead(**MO.head_kwargs('fcn')), 'htc': ref.HTCMaskHead(**MO.head_kwargs('htc'))}


def main():
    inp = MO.fixture_inputs()
    out = {}
    for key, head in reference_heads().items():
        for name, v in MO.run_mask_loss(head, inp, key, dtype=torch.float64).items():
            if name != 'y':
                out['%s_%s' % (key, name)] = v.numpy()
    np.savez_compressed(MO.FIXTURE, **{k: np.asarray(v, dtype=np.float32) for k, v in out.items()})
    print({k: (v.shape, float(np.abs(v).max())) for k, v in out.items()})
    print('wrote', MO.FIXTURE)


if __name__ == '__main__':
    main()
