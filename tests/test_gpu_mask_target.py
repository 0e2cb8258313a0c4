"""GPU: the mask heads' training targets on the device (bags_mask_target, ops.mask_targets, mask_head.mask_target).

Every check is torch.equal against the host loop (mask_target_single: cv2.resize per RoI), except the NaN rows the
native route gives where the host loop raises:
  * LVIS-sized 800 x 1344 masks, boxes of every size, sub-pixel boxes, boxes ending on or past the mask edge, crops
    of exactly the target size and of twice it, 1-pixel-wide and 1-pixel-high crops, non-binary masks;
  * images without positives and a batch with none; num_gt from 1 to 200; numpy and CUDA masks; mask sizes 28, 14
    and (28, 14);
  * with CUDA masks: no host sync, and get_target + the fused mask loss captured in one CUDA graph and replayed on new
    boxes, equal to eager;
  * FCNMaskHead and HTCMaskHead get_target -> loss -> backward: bitwise the same loss_mask and gradients on both routes.
"""
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from balancedgroupsoftmax_b200 import mask_head as MH
from balancedgroupsoftmax_b200 import ops

pytestmark = pytest.mark.gpu
DEV = 'cuda'
H_LVIS, W_LVIS = 800, 1344


def _masks(num_gt, H, W, rng, binary=True):
    if binary:
        m = np.zeros((num_gt, H, W), np.uint8)
        for k in range(num_gt):                     # a blob per instance, some noise around it
            y0, x0 = rng.integers(0, H), rng.integers(0, W)
            m[k, y0:y0 + rng.integers(1, H), x0:x0 + rng.integers(1, W)] = 1
            m[k] ^= (rng.random((H, W)) < 0.01).astype(np.uint8)
        return m
    return rng.integers(0, 256, (num_gt, H, W)).astype(np.uint8)


def _boxes(n, H, W, rng, out_hw=(28, 28)):
    """n random boxes of every size plus the edge cases (float32 [m, 4])."""
    x1, y1 = rng.random(n) * W, rng.random(n) * H
    bw, bh = rng.random(n) ** 2 * W, rng.random(n) ** 2 * H
    rand = np.stack([x1, y1, x1 + bw, y1 + bh], 1)
    oh, ow = out_hw
    edge = [
        (0, 0, W - 1, H - 1), (W - 1, H - 1, W - 1, H - 1), (W - 30.5, 10, W - 1, 40), (5, H - 20, 50, H - 0.25),
        (W - 10, H - 10, W + 40, H + 40),                                # past the edges: a smaller crop
        (10.2, 20.7, 10.9, 21.1), (100.6, 50.1, 100.3, 50.05),           # sub-pixel, inverted
        (30, 40, 30 + ow - 1, 40 + oh - 1), (31.9, 40.5, 31.9 + ow - 1, 40.5 + oh - 1),   # exactly the target size
        (30, 40, 30 + 2 * ow - 1, 40 + 2 * oh - 1),                      # exactly twice it
        (30, 40, 30 + 2 * ow - 1, 40 + oh - 1),                          # twice on one axis only
        (7, 3, 7, 300), (7, 3, 500, 3), (7, 3, 7.9, 3.9),                # 1 pixel wide, 1 pixel high, 1 pixel
        (-0.7, -0.2, 60, 70),                                            # truncates to 0
    ]
    return np.concatenate([rand, np.array(edge, np.float64)]).astype(np.float32)


def _batch(npos, num_gt, H=H_LVIS, W=W_LVIS, seed=0, binary=True, out_hw=(28, 28)):
    rng = np.random.default_rng(seed)
    props, gts, masks = [], [], []
    for i, p in enumerate(npos):
        ng = num_gt[i] if isinstance(num_gt, (list, tuple)) else num_gt
        b = _boxes(p, H, W, rng, out_hw)[:p] if p < 15 else _boxes(p - 15, H, W, rng, out_hw)
        props.append(torch.from_numpy(b).to(DEV))
        gts.append(torch.from_numpy(rng.integers(0, max(ng, 1), len(b))).to(DEV))
        masks.append(_masks(ng, H, W, rng, binary))
    return props, gts, masks


def _host(props, gts, masks, mask_size):
    return MH.mask_target(props, gts, masks, dict(mask_size=mask_size))      # numpy masks: the host loop


def _native(props, gts, masks, mask_size):
    cuda_masks = [torch.from_numpy(m).to(DEV) for m in masks]
    assert MH._native_mask_target(props, cuda_masks)
    return MH.mask_target(props, gts, cuda_masks, dict(mask_size=mask_size))


@pytest.mark.parametrize('mask_size', [28, 14, (28, 14)], ids=['28', '14', '28x14'])
@pytest.mark.parametrize('binary', [True, False], ids=['binary', 'uint8'])
def test_lvis_masks_match_host_loop(mask_size, binary):
    out_hw = (mask_size, mask_size) if isinstance(mask_size, int) else mask_size
    props, gts, masks = _batch([128, 128], 15, seed=1, binary=binary, out_hw=out_hw)
    want = _host(props, gts, masks, mask_size)
    got = _native(props, gts, masks, mask_size)
    assert got.dtype == want.dtype == torch.float32 and got.shape == want.shape == (256,) + out_hw
    assert torch.equal(got, want)
    assert torch.equal(ops.mask_targets(props, gts, masks, out_hw), want)      # numpy masks, uploaded


@pytest.mark.parametrize('num_gt', [1, 2, 15, 100, 200])
def test_num_gt(num_gt):
    props, gts, masks = _batch([64, 3, 40], num_gt, H=257, W=301, seed=num_gt)
    want = _host(props, gts, masks, 28)
    assert torch.equal(_native(props, gts, masks, 28), want)
    assert torch.equal(ops.mask_targets(props, gts, masks, 28), want)


def test_every_box_size():
    """Every crop width and height up to 130 and a spread beyond, on one 1344-wide mask."""
    rng = np.random.default_rng(4)
    masks = [_masks(3, 400, W_LVIS, rng, binary=False)]
    sizes = list(range(1, 131)) + [200, 399, 400, 700, 1343, 1344]
    boxes = np.array([(3.5, 1.25, 3.5 + w - 1, 1.25 + sizes[(i * 7) % len(sizes)] - 1) for i, w in enumerate(sizes)] +
                     [(0.0, 0.0, sizes[(i * 5) % len(sizes)] - 1, h - 1) for i, h in enumerate(sizes)], np.float32)
    props = [torch.from_numpy(boxes).to(DEV)]
    gts = [torch.from_numpy(rng.integers(0, 3, len(boxes))).to(DEV)]
    for ms in (28, 14, (28, 14)):
        assert torch.equal(_native(props, gts, masks, ms), _host(props, gts, masks, ms)), ms


def test_images_without_positives():
    props, gts, masks = _batch([0, 37, 0, 5, 0], [3, 4, 0, 2, 1], H=200, W=300, seed=6)
    want = _host(props, gts, masks, 28)
    assert torch.equal(_native(props, gts, masks, 28), want)
    props, gts, masks = _batch([0, 0], 3, H=50, W=60, seed=7)
    got, want = _native(props, gts, masks, 28), _host(props, gts, masks, 28)
    assert got.shape == want.shape == (0, 28, 28) and got.dtype == want.dtype


def test_nan_rows_where_host_loop_raises():
    props, gts, masks = _batch([40, 30], 5, H=200, W=300, seed=8)
    bad = {0: [3, 17], 1: [0, 29]}
    props[0][3] = torch.tensor([10.0, 10.0, 20.0, 20.0], device=DEV)
    gts[0][3] = 5                                                          # gt index == num_gt
    props[0][17] = torch.tensor([310.0, 10.0, 320.0, 20.0], device=DEV)  # starts right of the mask: empty crop
    gts[1][0] = -1
    props[1][29] = torch.tensor([5.0, 205.0, 20.0, 220.0], device=DEV)   # starts below the mask
    got = _native(props, gts, masks, 28)
    offs = [0, 40]
    for i in (0, 1):
        keep = [r for r in range(props[i].shape[0]) if r not in bad[i]]
        want = _host([props[i][keep]], [gts[i][keep]], [masks[i]], 28)
        rows = got[offs[i]:offs[i] + props[i].shape[0]]
        assert torch.equal(rows[keep], want)
        assert torch.isnan(rows[bad[i]]).all()


def test_no_host_sync_with_cuda_masks():
    props, gts, masks = _batch([128, 128], 15, seed=9)
    cuda_masks = [torch.from_numpy(m).to(DEV) for m in masks]
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode('error')
    try:
        out = MH.mask_target(props, gts, cuda_masks, dict(mask_size=28))
    finally:
        torch.cuda.set_sync_debug_mode('default')
    assert torch.equal(out, _host(props, gts, masks, 28))


def test_get_target_and_fused_loss_in_one_cuda_graph():
    props, gts, masks = _batch([128, 128], 15, seed=10)
    cuda_masks = [torch.from_numpy(m).to(DEV) for m in masks]
    samp = [SimpleNamespace(pos_bboxes=p, pos_assigned_gt_inds=g) for p, g in zip(props, gts)]
    head = MH.FCNMaskHead(num_convs=1, in_channels=16, conv_out_channels=16, num_classes=1231).to(DEV)
    cfg = dict(mask_size=28)
    g = torch.Generator().manual_seed(0)
    y = torch.randn(256, 16, 28, 28, generator=g).to(DEV)
    labels = torch.randint(0, 1231, (256,), generator=g).to(DEV)
    W, b = head.conv_logits.weight.detach().reshape(1231, 16).contiguous(), head.conv_logits.bias.detach()

    def step():
        t = head.get_target(samp, cuda_masks, cfg)
        loss, gr, rsum, index = ops.mask_fwd(y, W, b, labels, t / 255.0)
        return (t, loss, gr) + ops.mask_bwd(gr, rsum, None, W, labels, index, tuple(y.shape), y.dtype)

    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        step()
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph, stream=s):
            static = step()
    torch.cuda.current_stream().wait_stream(s)
    new_props, _, _ = _batch([128, 128], 15, seed=11)
    for p, q in zip(props, new_props):
        p.copy_(q)
    graph.replay()
    torch.cuda.synchronize()
    eager = step()
    assert torch.equal(static[0], _host(props, gts, masks, 28))
    for a, e in zip(static, eager):
        assert torch.equal(a, e)


def _head(cls):
    torch.manual_seed(3)
    h = cls(num_convs=2, in_channels=32, conv_out_channels=32, num_classes=1231)
    h.init_weights()
    return h.to(DEV).train()


@pytest.mark.parametrize('kind', ['fcn', 'htc'])
def test_head_step_is_bitwise_on_both_routes(kind):
    cls = MH.HTCMaskHead if kind == 'htc' else MH.FCNMaskHead
    head = _head(cls)
    props, gts, masks = _batch([128, 128], 15, seed=12)
    samp = [SimpleNamespace(pos_bboxes=p, pos_assigned_gt_inds=g) for p, g in zip(props, gts)]
    cuda_masks = [torch.from_numpy(m).to(DEV) for m in masks]
    g = torch.Generator().manual_seed(1)
    x = torch.randn(256, 32, 14, 14, generator=g).to(DEV)
    labels = torch.randint(0, 1230, (256,), generator=g).to(DEV)
    cfg = dict(mask_size=28)
    results = []
    for gt_masks in (masks, cuda_masks):                 # host loop, native route
        head.zero_grad()
        xr = x.clone().requires_grad_(True)
        t = head.get_target(samp, gt_masks, cfg)
        pred = head(xr, return_feat=False) if kind == 'htc' else head(xr)
        loss = head.loss(pred, t, labels)['loss_mask']
        loss.sum().backward()
        results.append([t, loss.detach(), xr.grad] + [p.grad.clone() for p in head.parameters() if p.grad is not None])
    assert len(results[0]) == len(results[1])
    for a, b in zip(*results):
        assert torch.equal(a, b)
