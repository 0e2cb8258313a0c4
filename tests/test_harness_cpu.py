"""CPU: the detector harness up to the head's inputs -- trunk (torchvision, frozen), RoI assignment +
sampling, RoIAlign features, targets -- i.e. the caller side of the hot path.  The head's loss itself needs an H100."""
import pytest
import torch

from balancedgroupsoftmax_b200.harness import BagsDetectorHarness, box_iou_plus1, sample_rois, synthetic_batch
from balancedgroupsoftmax_b200.tables import synthetic_tables

torchvision = pytest.importorskip('torchvision')


def test_iou_plus1_and_sampler_semantics():
    a = torch.tensor([[0., 0., 9., 9.]])
    b = torch.tensor([[0., 0., 9., 9.], [5., 0., 14., 9.], [20., 20., 29., 29.]])
    iou = box_iou_plus1(a, b)
    assert torch.allclose(iou, torch.tensor([[1.0, 50.0 / 150.0, 0.0]]))
    g = torch.Generator().manual_seed(3)
    gt = torch.tensor([[10., 10., 60., 60.], [100., 100., 180., 160.]])
    gl = torch.tensor([7, 1200])
    jit = (torch.rand(300, 4, generator=g) - 0.5) * 8
    props = torch.cat([gt[0] + jit[:150], gt[1] + jit[150:], torch.rand(700, 4, generator=g) * 20 + 300], 0)
    props[:, 2:] = torch.max(props[:, 2:], props[:, :2] + 1)
    s = sample_rois(props, gt, gl, num=512, pos_fraction=0.25, generator=g)
    assert s.pos_bboxes.size(0) == 128 and s.neg_bboxes.size(0) == 384          # 25 % positives, filled with negatives
    assert set(s.pos_gt_labels.tolist()) <= {7, 1200}
    assert (box_iou_plus1(s.pos_bboxes, gt).max(1).values >= 0.5).all()
    assert (box_iou_plus1(s.neg_bboxes, gt).max(1).values < 0.5).all()
    assert s.pos_is_gt.sum() <= 2 and s.pos_is_gt.dtype == torch.uint8
    # no ground truth: everything is negative, at most `num`
    s0 = sample_rois(props, gt[:0], gl[:0], num=512, generator=g)
    assert s0.pos_bboxes.size(0) == 0 and s0.neg_bboxes.size(0) == 512 and s0.pos_gt_labels.numel() == 0


@pytest.mark.timeout(300)
@pytest.mark.parametrize('stages', [1, 3])
def test_harness_produces_head_inputs_and_stops_at_the_gpu_boundary(stages):
    from balancedgroupsoftmax_b200._native import BagsNativeError
    t = synthetic_tables()
    torch.manual_seed(0)
    weights = (1.0,) if stages == 1 else (1.0, 0.5, 0.25)
    h = BagsDetectorHarness(t, num_stages=stages, stage_loss_weights=weights, rois_per_image=64, fc_out_channels=32,
                            min_size=160, max_size=224, proposals_per_image=200)
    assert not any(p.requires_grad for p in h.trunk.parameters()) and len(h.head_parameters()) == 8 * stages
    assert h.heads[0].fc_cls.weight.shape == (t.num_logits, 32)
    imgs, gb, gl = synthetic_batch(2, 120, 200, gts_per_image=4, generator=torch.Generator().manual_seed(1))
    feats, proposals, sizes, scales = h.trunk(imgs)
    assert len(proposals) == 2 and proposals[0].shape[1] == 4
    gbs = [g * s for g, s in zip(gb, scales)]
    x, sampling, boxes = h.head_inputs(feats, proposals, gbs, gl, sizes)
    n = sum(b.size(0) for b in boxes)
    assert x.shape == (n, 256, 7, 7) and 0 < n <= 128
    head = h.heads[0]
    labels, lw, bt, bw = head.get_target(sampling, gbs, gl, h.rcnn_cfg)
    assert labels.shape == (n,) and labels.dtype == torch.long and labels.max() < t.num_classes
    npos = [s.pos_bboxes.size(0) for s in sampling]
    assert all(k <= 16 for k in npos) and (labels > 0).sum().item() == sum(npos)
    assert bt.shape == (n, 4) and (bw.sum(1) > 0).sum().item() == sum(npos)
    # positives come first inside every image's block (what bench.py's synthetic labels imitate)
    off = 0
    for s, b in zip(sampling, boxes):
        k = s.pos_bboxes.size(0)
        assert (labels[off:off + k] > 0).all() and (labels[off + k:off + b.size(0)] == 0).all()
        off += b.size(0)
    h.train()
    assert not h.trunk.training
    cls_score, bbox_pred = head(x)                       # lazy handle: the fc_cls GEMM is fused into the loss
    assert cls_score.shape == (n, t.num_logits) and bbox_pred.shape[0] == n
    with pytest.raises(BagsNativeError):                 # the hot path itself has no CPU fallback
        h.forward_train(imgs, gb, gl)
