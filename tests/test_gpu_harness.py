"""GPU: the detector harness end to end -- frozen torchvision trunk -> RoI sampling -> BAGS head(s)
forward / get_target / loss / backward -> SGD step, at a small image size; losses finite, head gradients non-zero."""
import math

import pytest
import torch

torchvision = pytest.importorskip('torchvision')
pytestmark = pytest.mark.gpu


@pytest.mark.timeout(600)
@pytest.mark.parametrize('stages', [1, 3])
def test_harness_trains_on_synthetic_images(stages):
    from balancedgroupsoftmax_b200.harness import BagsDetectorHarness, synthetic_batch
    from balancedgroupsoftmax_b200.tables import synthetic_tables
    dev = torch.device('cuda', 0)
    t = synthetic_tables(1231, seed=0)
    weights = (1.0,) if stages == 1 else (1.0, 0.5, 0.25)
    torch.manual_seed(0)
    model = BagsDetectorHarness(t, num_stages=stages, stage_loss_weights=weights, rois_per_image=128,
                                min_size=256, max_size=320, proposals_per_image=300).to(dev)
    model.train()
    params = model.head_parameters()
    opt = torch.optim.SGD(params, lr=0.01)
    g = torch.Generator().manual_seed(5)
    first = None
    for it in range(2):
        imgs, gb, gl = synthetic_batch(2, 256, 320, gts_per_image=6, device=dev, generator=g)
        opt.zero_grad(set_to_none=True)
        losses = model.forward_train(imgs, gb, gl)
        per_stage = 6   # loss_cls_bin0..4 + loss_bbox
        assert len(losses) == stages * per_stage
        total = sum(losses.values())
        assert math.isfinite(total.item()), {k: v.item() for k, v in losses.items()}
        total.backward()
        for h in model.heads:
            assert h.fc_cls.weight.grad is not None and torch.isfinite(h.fc_cls.weight.grad).all()
            assert h.fc_cls.weight.grad.abs().sum().item() > 0
            assert h.shared_fcs[0].weight.grad is not None and h.shared_fcs[0].weight.grad.abs().sum().item() > 0
        opt.step()
        first = total.item() if first is None else first
