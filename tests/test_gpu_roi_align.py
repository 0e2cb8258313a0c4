"""GPU: the FPN RoI extractor (bags_roi_align_fwd / _bwd) against the reference's own RoIAlign op, built from its
sources into oracle/_ref/ (oracle/ref_roi_align.py), and against the float64 restatement of tests/roi_align_oracle.py.

Forward: bit for bit, both the op on one level and the whole extractor against the reference's loop over levels.
Backward: per element within C_BOUND * 2^-24 * sum|terms| + TINY of the float64 scatter, where the terms are the
gout w / count the reference adds with atomicAdd; the reference op's own backward is held to the same bound.
"""
import numpy as np
import pytest
import torch

import roi_align_oracle as R
from balancedgroupsoftmax_b200 import _native as nat
from balancedgroupsoftmax_b200 import ops
from balancedgroupsoftmax_b200.roi_extractor import SingleRoIExtractor
from oracle import ref_roi_align as REF

pytestmark = pytest.mark.gpu

C_BOUND = 32.0       # fp32 sums of the terms in any order, with random-sign gout
TINY = 1e-30
STRIDES = [4, 8, 16, 32]


@pytest.fixture(scope='module', autouse=True)
def _need_oracle():
    if not REF.available():
        pytest.skip('reference RoIAlign op not built (python -m oracle.ref_roi_align)')


def _same_bits(a, b):
    a, b = a.contiguous(), b.contiguous()
    assert a.shape == b.shape
    same = (a.view(torch.int32) == b.view(torch.int32)) | (torch.isnan(a) & torch.isnan(b))
    bad = (~same).nonzero()
    assert bad.numel() == 0, ('%d differing elements, first %s: %r vs %r'
                              % (bad.shape[0], bad[0].tolist(), a[tuple(bad[0])].item(), b[tuple(bad[0])].item()))


def _native_one(feat, rois, out, scale, sample_num):
    return ops.roi_align_fwd([feat], rois, ops.RoIAlignSpec(out, (float(scale),), sample_num))


def _crafted_rois(H, W, B, gen):
    """RoIs whose samples sit at -1, 0, H - 1, H and one ulp either side (single samples of two-pixel RoIs at
    scale 1), inside / straddling / outside the map, zero and inverted sizes, and random ones."""
    rows = []
    nxt = lambda v, d: float(np.nextafter(np.float32(v), np.float32(d)))   # noqa: E731
    for b in range(B):
        for t in (-1.0, 0.0, H - 1.0, float(H), W - 1.0, float(W)):
            for v in (t, nxt(t, -1e9), nxt(t, 1e9)):
                rows.append([b, v - 1, v - 1, v, v])
                rows.append([b, 0.5, v - 1, 1.5, v])
                rows.append([b, v - 1, 0.25, v, 1.25])
        rows += [[b, 1, 1, 0, 0], [b, 2, 2, 1, 3], [b, 3, 1, -4, 5], [b, -5, -5, -1, -1], [b, W + 2, H + 2, W + 9, H + 5],
                 [b, -3, -2, W + 3, H + 4], [b, 0, 0, W - 1, H - 1], [b, 0.5, 0.5, 0.5, 0.5]]
    rnd = torch.rand(64, 4, generator=gen) * torch.tensor([W + 4., H + 4., W + 4., H + 4.]) - 2
    rnd[:, 2:] = rnd[:, :2] + (rnd[:, 2:] - rnd[:, :2]).abs() * 0.7
    b = torch.randint(0, B, (64, 1), generator=gen).float()
    return torch.cat([torch.tensor(rows, dtype=torch.float32), torch.cat([b, rnd], 1)]).cuda().contiguous()


@pytest.mark.parametrize('out', [(7, 7), (14, 14), (7, 14)], ids=['7', '14', '7x14'])
@pytest.mark.parametrize('sample_num', [0, 1, 2, 3])
def test_op_bitwise_at_crafted_edges(out, sample_num):
    gen = torch.Generator().manual_seed(sample_num * 100 + out[1])
    for (H, W) in ((1, 1), (1, 9), (2, 2), (13, 17)):
        B = 2
        feat = torch.randn(B, 3, H, W, generator=gen).cuda()
        rois = _crafted_rois(H, W, B, gen)
        for scale in (1.0, 0.5):
            _same_bits(_native_one(feat, rois, out, scale, sample_num), REF.forward(feat, rois, *out, scale, sample_num))


@pytest.mark.parametrize('channels', [1, 3, 255, 256, 257])
def test_op_bitwise_channels_and_counts(channels):
    gen = torch.Generator().manual_seed(channels)
    B, H, W = 3, 50, 84
    feat = torch.randn(B, channels, H, W, generator=gen).cuda()
    for k in (0, 1, 4096 if channels in (256, 257) else 300):
        xy = torch.rand(k, 2, generator=gen) * torch.tensor([W * 8., H * 8.])
        wh = torch.rand(k, 2, generator=gen) * 300
        rois = torch.cat([torch.randint(0, B, (k, 1), generator=gen).float(), xy, xy + wh], 1).cuda().contiguous()
        for sample_num in (0, 2):
            nat_out = _native_one(feat, rois, (7, 7), 1 / 8, sample_num)
            assert nat_out.shape == (k, channels, 7, 7)
            _same_bits(nat_out, REF.forward(feat, rois, 7, 7, 1 / 8, sample_num))


def test_batch_index_outside_is_a_zero_row():
    feat = torch.randn(2, 4, 10, 10).cuda()
    rois = torch.tensor([[2, 0, 0, 5, 5], [-1, 0, 0, 5, 5], [1, 0, 0, 5, 5], [1.7, 0, 0, 5, 5]]).cuda()
    out = _native_one(feat, rois, (7, 7), 1.0, 2)
    assert torch.all(out[:2] == 0)
    _same_bits(out[2:], REF.forward(feat, rois[2:].contiguous(), 7, 7, 1.0, 2))
    feats = [feat.clone().requires_grad_(True)]
    o = ops.roi_align_apply(feats, rois, ops.RoIAlignSpec((7, 7), (1.0,), 2))
    o.backward(torch.ones_like(o))
    g_valid = REF.backward(torch.ones_like(o[2:]), rois[2:].contiguous(), 1.0, 2, feat.shape)
    assert torch.allclose(feats[0].grad, g_valid, rtol=1e-5, atol=1e-6)


def _levels_rois():
    """w = h around 112, 224 and 448 (the level boundaries at finest_scale 56), exact and an ulp or two either
    side, plus dense products around them, tiny and NaN scales."""
    rows = []
    for S in (112.0, 224.0, 448.0):
        for d in range(-3, 4):
            s = float(np.float32(S))
            for _ in range(abs(d)):
                s = float(np.nextafter(np.float32(s), np.float32(S + d)))
            rows.append([0, 0, 0, s - 1, s - 1])
            rows.append([0, 10, 20, 10 + s - 1, 20 + S - 1])
        for h in np.linspace(S * S / 120, S * S / 100, 400):
            rows.append([0, 0, 0, 119, h - 1])
    rows += [[0, 0, 0, -1, -1], [0, 5, 5, 5, 5], [0, 0, 0, 1e-30, 1e-30], [0, 0, 0, -1 + 1e-7, -1 + 1e-7],
             [0, 0, 0, -5, 5], [0, 3, 0, 1, 4], [0, 0, 0, float('nan'), 3], [0, 0, 0, float('inf'), 3],
             [0, 0, 0, 1e30, 1e30]]
    return torch.tensor(rows, dtype=torch.float32).cuda()


def test_level_mapping_matches_torch_on_cuda():
    rois = _levels_rois()
    feats = [torch.zeros(1, 1, 4, 4).cuda() for _ in STRIDES]
    spec = ops.RoIAlignSpec((7, 7), tuple(1 / s for s in STRIDES), 2, 56.0)
    _, levels = ops.roi_align_fwd(feats, rois, spec, want_levels=True)
    ref = R.map_roi_levels(rois, len(STRIDES), 56)
    in_range = (ref >= 0) & (ref < len(STRIDES))
    assert torch.equal(levels.long()[in_range], ref[in_range])
    assert torch.all(levels[~in_range] == -1)
    # the NaN scales are the ones outside every level, and there are some
    nan = torch.isnan(torch.sqrt((rois[:, 3] - rois[:, 1] + 1) * (rois[:, 4] - rois[:, 2] + 1)))
    assert nan.sum() >= 2 and torch.equal(~in_range, nan)
    # each boundary is crossed by the sampled products
    assert set(levels.tolist()) == {-1, 0, 1, 2, 3}


def _fpn(B, Cc, H0, W0, gen, levels=4):
    return [torch.randn(B, Cc, -(-H0 // 2 ** i), -(-W0 // 2 ** i), generator=gen).cuda() for i in range(levels)]


def _proposals(k, B, img_h, img_w, gen):
    """Boxes as the sampler hands them to the extractor: log-uniform sizes from 8 to 800 pixels, anywhere in the
    padded image, a quarter of them clipped to it, in image order."""
    size = torch.exp(torch.empty(k, 2).uniform_(np.log(8), np.log(800), generator=gen))
    ctr = torch.rand(k, 2, generator=gen) * torch.tensor([img_w, img_h])
    boxes = torch.cat([ctr - size / 2, ctr + size / 2], 1)
    clip = torch.rand(k, generator=gen) < 0.25
    boxes[clip, 0::2] = boxes[clip, 0::2].clamp(0, img_w - 1)
    boxes[clip, 1::2] = boxes[clip, 1::2].clamp(0, img_h - 1)
    b = torch.arange(B).repeat_interleave(k // B)
    return torch.cat([b[:, None].float(), boxes], 1).cuda().contiguous()


def _ref_extractor(ext, feats, rois, roi_scale_factor=None):
    layer = ext.roi_layers[0]
    return R.extractor(REF.forward, feats, rois, layer.out_size, ext.featmap_strides, layer.sample_num,
                       ext.finest_scale, ext.out_channels, roi_scale_factor, ext.roi_rescale)


def test_extractor_bitwise_at_faster_rcnn_training_shape():
    gen = torch.Generator().manual_seed(0)
    ext = SingleRoIExtractor(dict(type='RoIAlign', out_size=7, sample_num=2), 256, STRIDES)
    feats = _fpn(2, 256, 200, 336, gen)
    rois = _proposals(1024, 2, 800, 1344, gen)
    out = ext(feats, rois)
    assert out.shape == (1024, 256, 7, 7)
    _same_bits(out, _ref_extractor(ext, feats, rois))


def test_extractor_bitwise_with_roi_scale_factor():
    gen = torch.Generator().manual_seed(1)
    ext = SingleRoIExtractor(dict(type='RoIAlign', out_size=14, sample_num=2), 32, STRIDES)
    feats = _fpn(2, 32, 100, 168, gen)
    rois = _proposals(256, 2, 400, 672, gen)
    for factor in (1.5, 0.8):
        _same_bits(ext(feats, rois, roi_scale_factor=factor), _ref_extractor(ext, feats, rois, factor))


def test_extractor_bitwise_single_level_semantic():
    gen = torch.Generator().manual_seed(2)
    ext = SingleRoIExtractor(dict(type='RoIAlign', out_size=14, sample_num=2), 256, [8])
    feat = torch.randn(2, 256, 100, 168, generator=gen).cuda()
    rois = _proposals(512, 2, 800, 1344, gen)
    _same_bits(ext([feat], rois), _ref_extractor(ext, [feat], rois))


def _check_grad(name, g, g64, absum):
    g = g.double().cpu().numpy()
    err = np.abs(g - g64)
    lim = C_BOUND * 2.0 ** -24 * absum + TINY
    bad = err > lim
    assert not bad.any(), '%s: %d elements outside the bound, worst ratio %.3g' % (
        name, bad.sum(), (err / np.maximum(absum * 2.0 ** -24, TINY)).max())


def _scatter64(gout, rois, levels, feats, ext):
    """float64 gradient of every level and the sums of |terms|, each level from the RoIs mapped to it."""
    res = []
    for i, f in enumerate(feats):
        layer = ext.roi_layers[i]
        sel = (levels == i).cpu().numpy() if len(feats) > 1 else np.ones(rois.shape[0], bool)
        res.append(R.backward(gout.double().cpu().numpy()[sel], rois.cpu().numpy()[sel], layer.spatial_scale,
                              layer.sample_num, tuple(f.shape)))
    return res


def _ref_grads(gout, rois, levels, feats, ext):
    layer = ext.roi_layers[0]
    out = []
    for i, f in enumerate(feats):
        sel = (levels == i) if len(feats) > 1 else torch.ones(rois.shape[0], dtype=torch.bool, device=rois.device)
        out.append(REF.backward(gout[sel].contiguous(), rois[sel].contiguous(), 1 / ext.featmap_strides[i],
                                layer.sample_num, tuple(f.shape)))
    return out


@pytest.mark.parametrize('case', ['fpn7', 'fpn14_adaptive', 'single_large_adaptive'])
def test_backward_within_bound_of_float64(case):
    gen = torch.Generator().manual_seed(3)
    if case == 'single_large_adaptive':
        # adaptive samples at stride 4: RoIs over 504 pixels have more than 128 samples per axis (the fallback),
        # the others stay in the tables
        ext = SingleRoIExtractor(dict(type='RoIAlign', out_size=7, sample_num=0), 4, [4])
        feats = [torch.randn(2, 4, 150, 168, generator=gen).cuda()]
        rois = _proposals(8, 2, 600, 672, gen)
        rois[rois[:, 3] - rois[:, 1] > 300, 3] -= 300
        rois[:2, 1:] = torch.tensor([[-20., 10., 590., 540.], [30., -5., 560., 300.]]).cuda()
    else:
        size = 7 if case == 'fpn7' else 14
        ext = SingleRoIExtractor(dict(type='RoIAlign', out_size=size, sample_num=2 if case == 'fpn7' else 0), 8,
                                 STRIDES)
        feats = _fpn(2, 8, 48, 64, gen)
        rois = _proposals(64, 2, 192, 256, gen)
    feats = [f.requires_grad_(True) for f in feats]
    out = ext(feats, rois)
    _same_bits(out.detach(), _ref_extractor(ext, [f.detach() for f in feats], rois))
    gout = torch.randn(out.shape, generator=gen).cuda()
    out.backward(gout)
    levels = R.map_roi_levels(rois, len(feats), ext.finest_scale)
    exp = _scatter64(gout, rois, levels, feats, ext)
    refg = _ref_grads(gout, rois, levels, [f.detach() for f in feats], ext)
    for i, f in enumerate(feats):
        g64, absum = exp[i]
        _check_grad('native level %d' % i, f.grad, g64, absum)
        _check_grad('reference op level %d' % i, refg[i], g64, absum)


def test_levels_without_grad_get_none_and_frozen_trunk_runs_no_backward():
    gen = torch.Generator().manual_seed(4)
    ext = SingleRoIExtractor(dict(type='RoIAlign', out_size=7, sample_num=2), 8, STRIDES)
    feats = _fpn(2, 8, 48, 64, gen)
    rois = _proposals(64, 2, 192, 256, gen)
    feats[1].requires_grad_(True)
    feats[3].requires_grad_(True)
    out = ext(feats, rois)
    out.sum().backward()
    assert feats[0].grad is None and feats[2].grad is None
    assert feats[1].grad is not None and feats[3].grad is not None
    frozen = ext([f.detach() for f in feats], rois)
    assert not frozen.requires_grad
    # half features: cast to fp32 for the op, gradient back through the cast
    half = [f.detach().half().requires_grad_(True) for f in feats]
    o = ext(half, rois)
    assert o.dtype == torch.float32
    _same_bits(o, ext([h.detach().float() for h in half], rois))
    o.sum().backward()
    assert all(h.grad is not None and h.grad.dtype == torch.float16 for h in half)


def test_empty_batch_of_rois():
    ext = SingleRoIExtractor(dict(type='RoIAlign', out_size=7, sample_num=2), 8, STRIDES)
    feats = [f.requires_grad_(True) for f in _fpn(1, 8, 32, 32, torch.Generator().manual_seed(5))]
    out = ext(feats, torch.zeros(0, 5).cuda())
    assert out.shape == (0, 8, 7, 7)
    out.sum().backward()
    assert all(torch.count_nonzero(f.grad) == 0 for f in feats)


def _head_case(kind, gen):
    if kind == 'bbox':
        from balancedgroupsoftmax_b200.head import GSBBoxHeadWith0
        from balancedgroupsoftmax_b200.tables import synthetic_tables
        tables = synthetic_tables()
        head = GSBBoxHeadWith0(
            num_fcs=2, in_channels=256, fc_out_channels=1024, roi_feat_size=7, num_classes=tables.num_classes,
            gs_config=dict(tables=tables, others_sample_ratio=8.0, num_bins=tables.num_bins,
                           loss_bin=dict(type='CrossEntropyLoss', use_sigmoid=False, loss_weight=1.0)))
        ext = SingleRoIExtractor(dict(type='RoIAlign', out_size=7, sample_num=2), 256, STRIDES)
        labels = torch.zeros(128, dtype=torch.int64)
        labels[:32] = torch.randint(1, tables.num_classes, (32,), generator=gen)

        def loss(h, x):
            cls_score, _ = h(x)
            return sum(h.loss(cls_score, None, labels.cuda(), None, None, None).values())
    else:
        from balancedgroupsoftmax_b200.mask_head import FCNMaskHead
        head = FCNMaskHead(num_convs=1, in_channels=256, conv_out_channels=256, num_classes=81)
        ext = SingleRoIExtractor(dict(type='RoIAlign', out_size=14, sample_num=2), 256, STRIDES)
        labels = torch.randint(1, 81, (128,), generator=gen)
        targets = (torch.rand(128, 28, 28, generator=gen) > 0.5).float()

        def loss(h, x):
            return sum(h.loss(h(x), targets.cuda(), labels.cuda()).values())
    head.init_weights()
    return head.cuda().train(), ext, loss


@pytest.mark.parametrize('kind', ['bbox', 'mask'])
def test_whole_stack_gradient(kind):
    """extractor -> head -> loss -> backward: the FPN features' gradient is the float64 scatter of the head's
    gradient within the bound, as is the reference op's scatter of the same gradient; the pooled features equal the
    reference loop's bit for bit."""
    gen = torch.Generator().manual_seed(6)
    head, ext, loss = _head_case(kind, gen)
    feats = [f.requires_grad_(True) for f in _fpn(2, 256, 64, 96, gen)]
    rois = _proposals(128, 2, 256, 384, gen)
    x = ext(feats, rois)
    _same_bits(x.detach(), _ref_extractor(ext, [f.detach() for f in feats], rois))
    x.retain_grad()
    loss(head, x).backward()
    gout = x.grad.detach()
    levels = R.map_roi_levels(rois, 4, ext.finest_scale)
    exp = _scatter64(gout, rois, levels, feats, ext)
    refg = _ref_grads(gout, rois, levels, [f.detach() for f in feats], ext)
    for i, f in enumerate(feats):
        _check_grad('native level %d' % i, f.grad, *exp[i])
        _check_grad('reference op level %d' % i, refg[i], *exp[i])


def test_cuda_graph_replay_equals_eager():
    gen = torch.Generator().manual_seed(7)
    ext = SingleRoIExtractor(dict(type='RoIAlign', out_size=7, sample_num=2), 16, STRIDES)
    feats = [f.requires_grad_(True) for f in _fpn(2, 16, 64, 96, gen)]
    rois = _proposals(256, 2, 256, 384, gen)
    gout = torch.randn(256, 16, 7, 7, generator=gen).cuda()

    def step():
        for f in feats:
            f.grad = None
        out = ext(feats, rois)
        out.backward(gout)
        return out

    eager = step().detach().clone()
    eager_g = [f.grad.clone() for f in feats]
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        step()
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    for f in feats:
        f.grad = None
    with torch.cuda.graph(graph):
        out = ext(feats, rois)
        out.backward(gout)
    graph.replay()
    torch.cuda.synchronize()
    _same_bits(out, eager)
    for f, g in zip(feats, eager_g):
        assert torch.allclose(f.grad, g, rtol=1e-5, atol=1e-6)


def test_invalid_arguments_raise():
    feat = torch.zeros(1, 4, 8, 8).cuda()
    rois = torch.zeros(1, 5).cuda()
    with pytest.raises(nat.BagsNativeError, match='out size'):
        ops.roi_align_fwd([feat], rois, ops.RoIAlignSpec((65, 7), (1.0,), 2))
    with pytest.raises(nat.BagsNativeError, match='levels'):
        ops.roi_align_fwd([feat] * 9, rois, ops.RoIAlignSpec((7, 7), (1.0,) * 9, 2))
    with pytest.raises(nat.BagsNativeError, match='rois'):
        ops.roi_align_fwd([feat], torch.zeros(1, 4).cuda(), ops.RoIAlignSpec((7, 7), (1.0,), 2))
