"""GPU: RPN proposal generation (bags_rpn_proposals via ops.rpn_proposals and RPNHead.get_bboxes) against torch's own
sigmoid and the reference's delta2bbox op sequence, and end to end against the reference's per-image loop
(tests/rpn_oracle.py) with the reference's compiled NMS op from oracle/_ref/ (oracle.ref_nms) or, for tied inputs,
the greedy stand-in with the pinned tie rule.  Equality is bit for bit throughout."""
import numpy as np
import pytest
import torch

import rpn_oracle as O
from balancedgroupsoftmax_b200 import ops
from balancedgroupsoftmax_b200.rpn_head import AnchorGenerator, RPNHead
from oracle import ref_nms as REF

pytestmark = pytest.mark.gpu

STRIDES = [4, 8, 16, 32, 64]
GEN3 = [AnchorGenerator(s, [8], [0.5, 1.0, 2.0]) for s in STRIDES]
RPN_CFG = dict(type='RPNHead', in_channels=256, feat_channels=256, anchor_scales=[8], anchor_ratios=[0.5, 1.0, 2.0],
               anchor_strides=[4, 8, 16, 32, 64], target_means=[.0, .0, .0, .0], target_stds=[1.0, 1.0, 1.0, 1.0],
               loss_cls=dict(type='CrossEntropyLoss', use_sigmoid=True, loss_weight=1.0),
               loss_bbox=dict(type='SmoothL1Loss', beta=1.0 / 9.0, loss_weight=1.0))
TRAIN = dict(nms_pre=2000, nms_post=2000, max_num=2000, nms_thr=0.7, min_bbox_size=0)
TEST = dict(nms_pre=1000, nms_post=1000, max_num=1000, nms_thr=0.7, min_bbox_size=0)


def _need_ref():
    if not REF.available():
        pytest.skip('reference NMS op not built (python -m oracle.ref_build)')


def _same(a, b, what=''):
    a, b = a.detach().float().cpu().contiguous(), b.detach().float().cpu().contiguous()
    assert a.shape == b.shape, (what, a.shape, b.shape)
    same = (a.view(torch.int32) == b.view(torch.int32)) | (torch.isnan(a) & torch.isnan(b))
    bad = (~same).nonzero()
    assert bad.numel() == 0, ('%s: %d differing elements, first %s: %r vs %r'
                              % (what, bad.shape[0], bad[0].tolist(), a[tuple(bad[0])].item(), b[tuple(bad[0])].item()))


def _native(scores, deltas, gens, strides, shapes, cfg, means=(0., 0., 0., 0.), stds=(1., 1., 1., 1.)):
    out, counts = ops.rpn_proposals(scores, deltas, [g.base_anchors for g in gens], strides, shapes, cfg['nms_pre'],
                                    cfg['nms_post'], cfg['max_num'], cfg['nms_thr'], cfg['min_bbox_size'], means,
                                    stds)
    counts = counts.cpu().tolist()
    for b, c in enumerate(counts):
        assert torch.all(out[b, c:] == 0), 'rows after the count are not zero'
    return [out[b, :c] for b, c in enumerate(counts)]


def _oracle(scores, deltas, gens, strides, shapes, cfg, nms, means=(0., 0., 0., 0.), stds=(1., 1., 1., 1.)):
    return O.get_bboxes(scores, deltas, [g.base_anchors for g in gens], strides, shapes, cfg, nms, means, stds)


def _distinct_logits(sizes, B, gen, A=3, lo=-4.0, hi=4.0):
    """[B, A, H, W] logits per level whose sigmoids are distinct in fp32 across the whole batch."""
    total = B * A * sum(h * w for h, w in sizes)
    vals = torch.linspace(lo, hi, total, dtype=torch.float64).float()
    vals = vals[torch.randperm(total, generator=gen)]
    assert torch.unique(vals.sigmoid()).numel() == total
    out, o = [], 0
    for h, w in sizes:
        n = B * A * h * w
        out.append(vals[o:o + n].view(B, A, h, w).cuda())
        o += n
    return out


def _deltas(sizes, B, gen, A=3, scale=0.5):
    return [(torch.randn(B, 4 * A, h, w, generator=gen) * scale).cuda() for h, w in sizes]


def _fpn_sizes(H, W, levels=5):
    return [((H + s - 1) // s, (W + s - 1) // s) for s in STRIDES[:levels]]


# ----------------------------------------------------------------------------------------------------------- scores
def _score_sweep():
    x = np.concatenate([np.linspace(-120, 120, 2500, dtype=np.float32),
                        np.linspace(-1e-3, 1e-3, 600, dtype=np.float32),
                        np.array([0.0, -0.0, np.inf, -np.inf, 1e-45, -1e-45, 1e-38, -1e-38, 88.7, -88.7, 103.9,
                                  -103.9, 16.6, 17.0, -17.0], dtype=np.float32)])
    return torch.from_numpy(x)


@pytest.mark.parametrize('with_nan', [False, True])
def test_scores_equal_torch_sigmoid(with_nan):
    x = _score_sweep()
    if with_nan:
        x = torch.cat([x, torch.tensor([float('nan')])])
    n = x.numel()
    logits = x.view(1, 1, 1, n).cuda()
    deltas = torch.zeros(1, 4, 1, n).cuda()
    gen = [AnchorGenerator(4, [1], [1.0])]
    cfg = dict(nms_pre=-1, nms_post=n, max_num=n, nms_thr=1.0, min_bbox_size=0)
    got = _native([logits], [deltas], gen, [4], [(8, 4 * n + 8)], cfg)[0]
    want = torch.sort(torch.sigmoid(logits.view(-1)), descending=True, stable=True)[0]
    assert got.shape[0] == n
    _same(got[:, 4], want, 'scores')


@pytest.mark.parametrize('quantised', [False, True])
def test_selected_scores_are_the_top_k(quantised):
    """A P2-sized level (201,600 anchors) split over a cluster: the kept scores are the 2000 largest sigmoids."""
    gen = torch.Generator().manual_seed(1)
    logits = torch.randn(1, 3, 200, 336, generator=gen) * 3
    if quantised:
        logits = (logits * 4).round() / 4
    logits = logits.cuda()
    deltas = torch.zeros(1, 12, 200, 336).cuda()
    cfg = dict(nms_pre=2000, nms_post=2000, max_num=2000, nms_thr=1.0, min_bbox_size=0)
    got = _native([logits], [deltas], GEN3[:1], [4], [(800, 1344)], cfg)[0]
    flat = logits[0].permute(1, 2, 0).reshape(-1)
    want = torch.sort(torch.sigmoid(flat), descending=True, stable=True)[0][:2000]
    _same(got[:, 4], want, 'top-k scores')
    if not quantised:   # tie-free: the boxes too
        exp = _oracle([logits], [deltas], GEN3[:1], [4], [(800, 1344)], cfg, O.greedy_nms)[0]
        _same(got, exp, 'proposals')


# ------------------------------------------------------------------------------------------------------------ boxes
def _crafted_deltas(n, gen):
    mr = float(np.float32(abs(np.log(16 / 1000))))
    vals = [0.0, mr, -mr, float(np.nextafter(np.float32(mr), np.float32(10))), -10.0, 10.0, 50.0, -50.0,
            float('nan'), float('inf'), float('-inf'), 1e-30, -1e-30, 0.3, -0.7, 3.9, 4.2]
    d = torch.randn(n, 4, generator=gen) * 2
    for i, v in enumerate(vals):
        for c in range(4):
            d[(4 * i + c) % n, c] = v
            d[(4 * i + c + 1) % n, (c + 2) % 4] = v
    return d


@pytest.mark.parametrize('means,stds', [((0., 0., 0., 0.), (1., 1., 1., 1.)),
                                        ((0.1, -0.2, 0.05, -0.3), (0.1, 0.1, 0.2, 0.2))], ids=['default', 'norm'])
def test_boxes_equal_reference_delta2bbox(means, stds):
    """Every anchor comes out (nms_thr = 1, max_num = anchors): the boxes equal delta2bbox's own op sequence (with
    addcmul) per image, each image with its own img_shape, including clamped and NaN / inf deltas and boxes past
    every image edge."""
    gen = torch.Generator().manual_seed(2)
    B, H, W, stride = 3, 12, 20, 16
    A, n = 3, 3 * 12 * 20
    g = [AnchorGenerator(stride, [8], [0.5, 1.0, 2.0])]
    logits = _distinct_logits([(H, W)], B, gen)[0]
    deltas = []
    for b in range(B):
        d = _crafted_deltas(n, gen)   # rows in flat order (h W + w) A + a
        deltas.append(d.view(H, W, A, 4).permute(2, 3, 0, 1).reshape(4 * A, H, W))
    deltas = torch.stack(deltas).cuda()
    shapes = [(150, 250), (200, 320), (37, 400)]
    cfg = dict(nms_pre=-1, nms_post=n, max_num=n, nms_thr=1.0, min_bbox_size=0)
    got = _native([logits], [deltas], g, [stride], shapes, cfg, means, stds)
    anchors = O.grid_anchors(g[0].base_anchors, H, W, stride, 'cuda')
    for b in range(B):
        s = logits[b].permute(1, 2, 0).reshape(-1).sigmoid()
        d = deltas[b].permute(1, 2, 0).reshape(-1, 4)
        order = torch.sort(s, descending=True, stable=True)[1]
        exp = torch.cat([O.delta2bbox(anchors, d, means, stds, shapes[b]), s[:, None]], 1)[order]
        assert got[b].shape[0] == n
        _same(got[b], exp, 'image %d' % b)


def test_addcmul_against_split_rounding():
    """Records which rounding torch's addcmul has on this build (the kernel pins one fma): on a sweep where the two
    differ, torch.addcmul(px, pw, dx) equals fma(pw, dx, px)."""
    gen = torch.Generator().manual_seed(3)
    px = (torch.rand(1 << 16, generator=gen) * 1000).cuda()
    pw = (torch.rand(1 << 16, generator=gen) * 300 + 1).cuda()
    dx = torch.randn(1 << 16, generator=gen).cuda()
    ref = torch.addcmul(px, pw, dx, value=1)
    split = px + pw * dx
    fused = (px.double() + pw.double() * dx.double()).float()
    assert not torch.equal(split, fused), 'the sweep does not separate the two roundings'
    _same(ref, fused, 'addcmul vs single rounding')


# ------------------------------------------------------------------------------------------------------- end to end
@pytest.mark.parametrize('case', ['train', 'test', 'b1', 'b3', 'b8', 'one_level'])
def test_end_to_end_against_reference_op(case):
    _need_ref()
    gen = torch.Generator().manual_seed(['train', 'test', 'b1', 'b3', 'b8', 'one_level'].index(case) + 10)
    if case in ('train', 'test'):
        B, (H, W), cfg, L = 2 if case == 'train' else 1, (800, 1344), TRAIN if case == 'train' else TEST, 5
    elif case == 'one_level':
        B, (H, W), cfg, L = 2, (320, 480), TEST, 1
    else:
        B, (H, W), cfg, L = int(case[1:]), (256, 384), TRAIN, 5
    sizes = _fpn_sizes(H, W, L)
    logits = _distinct_logits(sizes, B, gen)
    deltas = _deltas(sizes, B, gen)
    shapes = [(H - 13 * b, W - 29 * b) for b in range(B)]
    got = _native(logits, deltas, GEN3[:L], STRIDES[:L], shapes, cfg)
    exp = _oracle(logits, deltas, GEN3[:L], STRIDES[:L], shapes, cfg, REF.nms_wrapper_op)
    for b in range(B):
        _same(got[b], exp[b], '%s image %d' % (case, b))


def test_tied_logits_follow_the_pinned_rule():
    gen = torch.Generator().manual_seed(4)
    B, sizes = 2, _fpn_sizes(256, 384)
    logits = [((torch.randn(B, 3, h, w, generator=gen) * 2 * 4).round() / 4).cuda() for h, w in sizes]
    deltas = _deltas(sizes, B, gen)
    cfg = dict(nms_pre=1000, nms_post=600, max_num=1500, nms_thr=0.7, min_bbox_size=0)
    shapes = [(256, 384), (250, 380)]
    got = _native(logits, deltas, GEN3, STRIDES, shapes, cfg)
    exp = _oracle(logits, deltas, GEN3, STRIDES, shapes, cfg, O.greedy_nms)
    for b in range(B):
        _same(got[b], exp[b], 'image %d' % b)


def test_iou_exactly_at_the_threshold_is_kept():
    """Two 10 x 10 anchors five pixels apart (zero deltas keep them): IoU 50 / 150 in the op's fp32 arithmetic.  At
    nms_thr equal to it both stay; one fp32 step below, the lower-scored one is suppressed."""
    from oracle.bags_oracle import iou_plus1_fp32
    g = [AnchorGenerator(10, [1], [1.0])]
    iou = iou_plus1_fp32(np.array([0, 0, 9, 9]), np.array([5, 0, 14, 9]))
    logits = torch.tensor([1.0, 0.0]).view(1, 1, 1, 2).cuda()
    deltas = torch.zeros(1, 4, 1, 2).cuda()
    for thr, n in ((float(iou), 2), (float(np.nextafter(iou, np.float32(0))), 1)):
        cfg = dict(nms_pre=-1, nms_post=10, max_num=10, nms_thr=thr, min_bbox_size=0)
        got = _native([logits], [deltas], g, [5], [(100, 100)], cfg)[0]
        assert got.shape[0] == n, (thr, got)
        _same(got[0], torch.cat([torch.tensor([0., 0., 9., 9.]).cuda(), torch.sigmoid(logits.view(-1)[:1])]), 'row')


@pytest.mark.parametrize('case', ['nms_post_cut', 'anchor_order', 'pre_covers_all', 'max_num_above', 'one_anchor',
                                  'min_bbox', 'min_bbox_one'])
def test_quirks_and_limits(case):
    gen = torch.Generator().manual_seed(5)
    B, sizes, gens, strides = 2, [(24, 30), (12, 15), (6, 8)], GEN3[:3], STRIDES[:3]
    cfg = dict(nms_pre=1000, nms_post=1000, max_num=1000, nms_thr=0.5, min_bbox_size=0)
    scale = 0.5
    if case == 'nms_post_cut':
        cfg.update(nms_post=40)
    elif case == 'anchor_order':        # no level is selected: the nms_post cut takes survivors in anchor order
        cfg.update(nms_pre=5000, nms_post=25, max_num=60)
    elif case == 'pre_covers_all':
        cfg.update(nms_pre=2160)
    elif case == 'max_num_above':
        cfg.update(max_num=4000)
    elif case == 'one_anchor':
        sizes, gens, strides = [(24, 30), (1, 1)], [GEN3[0], AnchorGenerator(64, [8], [1.0])], [4, 64]
    elif case == 'min_bbox':
        cfg.update(min_bbox_size=24)
        scale = 1.0
    elif case == 'min_bbox_one':
        cfg.update(min_bbox_size=8, nms_thr=1.0, nms_pre=5000)
    A = [g.num_base_anchors for g in gens]
    logits = [_distinct_logits([s], B, gen, A=a)[0] for s, a in zip(sizes, A)]
    deltas = [_deltas([s], B, gen, A=a, scale=scale)[0] for s, a in zip(sizes, A)]
    if case == 'min_bbox_one':   # every box under 2 px but the first anchor's (its own), per level and image
        for d in deltas:
            d[:, 2::4] = -10.0
            d[:, 3::4] = -10.0
            d[:, 0:4, 0, 0] = 0.0
    shapes = [(96, 120), (90, 111)]
    got = _native(logits, deltas, gens, strides, shapes, cfg)
    exp = _oracle(logits, deltas, gens, strides, shapes, cfg, O.greedy_nms)
    for b in range(B):
        _same(got[b], exp[b], '%s image %d' % (case, b))
        if case == 'min_bbox_one':
            assert got[b].shape[0] == len(sizes)


# ------------------------------------------------------------------------------------------------------ CUDA graph
def test_cuda_graph_replay_equals_eager_without_sync():
    gen = torch.Generator().manual_seed(6)
    B, sizes = 2, _fpn_sizes(256, 384)
    logits = _distinct_logits(sizes, B, gen)
    deltas = _deltas(sizes, B, gen)
    base = [g.base_anchors for g in GEN3]
    args = (logits, deltas, base, STRIDES, [(256, 384), (240, 300)], 1000, 1000, 1000, 0.7, 0.0)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode('error')
    try:
        eager, ecounts = ops.rpn_proposals(*args)
    finally:
        torch.cuda.set_sync_debug_mode('default')
    eager, ecounts = eager.clone(), ecounts.clone()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        ops.rpn_proposals(*args)
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out, counts = ops.rpn_proposals(*args)
    out.zero_()
    graph.replay()
    torch.cuda.synchronize()
    _same(out, eager, 'replay')
    assert torch.equal(counts, ecounts)


# ------------------------------------------------------------------------------------------------------ full stack
def test_rpn_head_into_the_bbox_head():
    from balancedgroupsoftmax_b200.head import GSBBoxHeadWith0, _as_tensor
    from balancedgroupsoftmax_b200.registry import build_head
    from balancedgroupsoftmax_b200.roi_extractor import SingleRoIExtractor
    from balancedgroupsoftmax_b200.tables import synthetic_tables
    torch.manual_seed(7)
    rpn = build_head(dict(RPN_CFG))
    rpn.init_weights()
    rpn = rpn.cuda().eval()
    B, H, W = 2, 256, 384
    feats = [torch.randn(B, 256, h, w).cuda() for h, w in _fpn_sizes(H, W)]
    metas = [dict(img_shape=(H, W, 3), scale_factor=1.0, pad_shape=(H, W, 3)),
             dict(img_shape=(240, 360, 3), scale_factor=1.0, pad_shape=(H, W, 3))]
    with torch.no_grad():
        cls_scores, bbox_preds = rpn(feats)
        props = rpn.get_bboxes(cls_scores, bbox_preds, metas, TEST)
        exp = _oracle(cls_scores, bbox_preds, GEN3, STRIDES, [m['img_shape'] for m in metas], TEST, O.greedy_nms)
        for b in range(B):
            _same(props[b], exp[b], 'image %d' % b)
        single = rpn.get_bboxes_single([c[1] for c in cls_scores], [p[1] for p in bbox_preds], None,
                                       metas[1]['img_shape'], 1.0, TEST)
        _same(single, props[1], 'get_bboxes_single')
        rois = torch.cat([torch.cat([p.new_full((p.shape[0], 1), float(b)), p[:, :4]], 1)
                          for b, p in enumerate(props)]).contiguous()
        ext = SingleRoIExtractor(dict(type='RoIAlign', out_size=7, sample_num=2), 256, STRIDES[:4])
        x = ext(feats[:4], rois)
        tables = synthetic_tables()
        head = GSBBoxHeadWith0(
            num_fcs=2, in_channels=256, fc_out_channels=1024, roi_feat_size=7, num_classes=tables.num_classes,
            gs_config=dict(tables=tables, others_sample_ratio=8.0, num_bins=tables.num_bins,
                           loss_bin=dict(type='CrossEntropyLoss', use_sigmoid=False, loss_weight=1.0)))
        head.init_weights()
        head = head.cuda().eval()
        cls_score, bbox_pred = head(x)
    assert x.shape == (rois.shape[0], 256, 7, 7)
    assert torch.isfinite(_as_tensor(bbox_pred)).all() and _as_tensor(cls_score).shape[0] == rois.shape[0]
