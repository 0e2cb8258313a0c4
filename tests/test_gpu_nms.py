"""GPU: the device-side class-aware NMS (ops.multiclass_nms -> bags_class_nms_dense) against the oracle's restatement of
the reference's per-class loop (mmdet/core/post_processing/bbox_nms.py:6-66, pinned to the reference's own file in
tests/test_oracle_vs_reference.py)."""
import os

import pytest
import torch

from oracle import bags_oracle as O

pytestmark = [pytest.mark.gpu]


@pytest.mark.parametrize('n,classes,per_class_boxes', [(60, 9, False), (300, 40, True), (1000, 6, False), (5, 3, True)])
def test_class_nms_matches_oracle(n, classes, per_class_boxes):
    from balancedgroupsoftmax_b200 import ops
    g = torch.Generator().manual_seed(n + classes)
    xy = torch.rand(n, 2, generator=g) * 200
    wh = torch.rand(n, 2, generator=g) * 80 + 2
    b4 = torch.cat([xy, xy + wh], 1)
    boxes = (b4[:, None, :] + torch.rand(n, classes, 4, generator=g)).reshape(n, classes * 4) if per_class_boxes else b4
    scores = torch.rand(n, classes, generator=g) ** 2
    for thr, iou, k in ((0.05, 0.5, 100), (0.0, 0.3, 300), (0.999999, 0.5, 10), (0.3, 0.7, -1), (0.3, 0.5, 0), (0.2, 0.5, -2)):
        want_b, want_l = O.multiclass_nms(boxes, scores, thr, iou, k)
        got_b, got_l = ops.multiclass_nms(boxes.cuda(), scores.cuda(), thr, iou, k)
        assert got_b.shape == want_b.shape
        # same detections; order inside equal scores may differ
        key_w = sorted(zip(want_l.tolist(), [tuple(r) for r in want_b.tolist()]))
        key_g = sorted(zip(got_l.cpu().tolist(), [tuple(r) for r in got_b.cpu().tolist()]))
        assert key_w == key_g


def test_get_det_bboxes_runs_native_nms_at_lvis_shape():
    """1000 proposals x 1231 classes, score_thr = 0.0, iou 0.5, max_per_img = 300 (configs/bags/*.py:115-117) through
    GSBBoxHeadWith0.get_det_bboxes(cfg=...) -- the detections equal the oracle loop's on the same merged scores."""
    from balancedgroupsoftmax_b200.head import GSBBoxHeadWith0
    from balancedgroupsoftmax_b200.tables import synthetic_tables
    t = synthetic_tables(1231, seed=0)
    head = GSBBoxHeadWith0(num_fcs=2, in_channels=8, fc_out_channels=64, roi_feat_size=2, num_classes=1231,
                           reg_class_agnostic=True,
                           gs_config=dict(tables=t, others_sample_ratio=8.0, num_bins=5,
                                          loss_bin=dict(type='CrossEntropyLoss', use_sigmoid=False, loss_weight=1.0)))
    head = head.cuda().eval()
    g = torch.Generator().manual_seed(3)
    n = 1000
    z = (torch.randn(n, t.num_logits, generator=g) * 3).cuda()
    xy = torch.rand(n, 2, generator=g) * 600
    wh = torch.rand(n, 2, generator=g) * 200 + 4
    rois = torch.cat([torch.zeros(n, 1), xy, xy + wh], 1).cuda()
    cfg = dict(score_thr=0.0, nms=dict(type='nms', iou_thr=0.5), max_per_img=300)
    with torch.no_grad():
        dets, labels = head.get_det_bboxes(rois, z, None, (800, 1333, 3), 1.0, rescale=False, cfg=cfg)
        boxes, scores = head.get_det_bboxes(rois, z, None, (800, 1333, 3), 1.0, rescale=False, cfg=None)
    want_b, want_l = O.multiclass_nms(boxes.cpu(), scores.cpu(), 0.0, 0.5, 300)
    assert dets.shape == want_b.shape == (300, 5)
    # the cut at max_per_img falls between distinct scores, so the kept detections agree exactly, in score order
    assert torch.equal(labels.cpu(), want_l)
    assert torch.equal(dets.cpu(), want_b)
    assert (dets[1:, 4] < dets[:-1, 4]).all()
