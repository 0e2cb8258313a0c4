"""CPU: the oracle (and the host-side mirror of the head) against what the reference's OWN source returned for the same
seeded inputs, stored in tests/golden/reference_outputs.npz by tests/golden/make_ref_golden.py (the reference run in place
through oracle/ref_shim.py).  Large outputs are compared on the stored row / column sample."""
import os
import sys

import numpy as np
import pytest
import torch

from balancedgroupsoftmax_b200.tables import synthetic_tables
from oracle import bags_oracle as O

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden'))
import make_ref_golden as MG  # noqa: E402

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'reference_outputs.npz')


@pytest.fixture(scope='module')
def ref():
    return synthetic_tables(1231, seed=0), np.load(GOLD)


def _rel(a, b):
    a, b = torch.as_tensor(a).double(), torch.as_tensor(b).double()
    return ((a - b).norm() / b.norm().clamp_min(1e-20)).item()


@pytest.mark.parametrize('N,npos,seed', MG.LOSS_CASES)
def test_loss_and_grads_match_reference(ref, N, npos, seed):
    t, d = ref
    l2b, ps = torch.from_numpy(t.label2binlabel), torch.from_numpy(t.pred_slice)
    W, b, x, labels = MG.loss_case_inputs(N, npos, seed, t.num_logits)
    np.random.seed(seed)   # same numpy state => identical sampled masks
    lo, dW, db, dX = O.head_step(x, W, b, labels, l2b, ps, 8.0)
    key = 'loss_%d_%d_%d_' % (N, npos, seed)
    want = d[key + 'losses']
    for g in range(5):
        got = lo['loss_cls_bin%d' % g].item()
        assert abs(got - want[g]) <= 1e-6 * max(1.0, abs(want[g])), g
    assert _rel(dW[::MG.DW_ROWS], d[key + 'dW']) < 1e-6
    assert _rel(db, d[key + 'db']) < 1e-6
    assert _rel(dX[::MG.DX_ROWS], d[key + 'dX']) < 1e-6


def test_merge_score_matches_reference(ref):
    t, d = ref
    ps = torch.from_numpy(t.pred_slice)
    torch.manual_seed(7)
    for i in range(3):
        z = torch.randn(200, t.num_logits) * 3
        b = O.merge_score(z, ps, [torch.from_numpy(s) for s in t.fg_splits], t.num_classes)
        assert np.array_equal(b[:, ::MG.MERGE_COLS].numpy(), d['merge_%d_sample' % i])
        assert np.array_equal(b.argmax(1).numpy(), d['merge_%d_argmax' % i])


def test_tables_load_into_reference_head(ref):
    """The tables the reference's constructor read from the files tables.save_reference_files wrote
    (gs_bbox_head_with0.py:37-49), as stored when the golden file was made, equal synthetic_tables().  Without the
    reference the files themselves no longer pass through its constructor here: a change of the file format is caught
    only when tests/golden/make_ref_golden.py is run again against a reference checkout."""
    t, d = ref
    l2b = d['tables_label2binlabel']
    assert l2b.dtype == np.int64 and l2b.shape == (5, 1231)
    assert np.array_equal(l2b, t.label2binlabel)
    assert np.array_equal(d['tables_pred_slice'], t.pred_slice)
    lens = d['tables_fg_split_lens']
    assert len(lens) == 4 == len(t.fg_splits)
    for a, n, b in zip(np.split(d['tables_fg_splits'], np.cumsum(lens)[:-1]), lens, t.fg_splits):
        assert len(a) == n and np.array_equal(a, b)
    assert int(d['tables_out_features']) == 1236


def test_host_mirror_numpy_sampler_is_the_reference_sampler(ref):
    """GSBBoxHeadWith0(sampler='numpy')._sample_others_numpy draws the same masks as the reference."""
    from balancedgroupsoftmax_b200.head import GSBBoxHeadWith0
    t, d = ref
    mine = GSBBoxHeadWith0(num_fcs=2, in_channels=4, fc_out_channels=128, roi_feat_size=2, num_classes=1231,
                           gs_config=dict(tables=t, others_sample_ratio=8.0, num_bins=5, sampler='numpy',
                                          loss_bin=dict(type='CrossEntropyLoss', use_sigmoid=False, loss_weight=1.0)))
    labels = torch.zeros(400, dtype=torch.long)
    labels[:90] = torch.randint(1, 1231, (90,), generator=torch.Generator().manual_seed(3))
    np.random.seed(11)
    for g in range(1, 5):
        w = mine._sample_others_numpy(mine.label2binlabel[g][labels])
        assert np.array_equal(w.numpy(), d['sampler_w%d' % g])


def test_get_target_matches_reference_bbox_target(ref):
    """The head's standalone target generator against the reference's bbox_target.py / transforms.py."""
    from oracle.ref_shim import AttrDict
    from balancedgroupsoftmax_b200.head import GSBBoxHeadWith0, bbox2delta, bbox_target
    _, d = ref
    imgs = MG.bbox_inputs()
    means, stds = MG.MEANS, MG.STDS
    assert np.array_equal(bbox2delta(imgs[0].pos_bboxes, imgs[0].pos_gt_bboxes, means, stds).numpy(), d['bbox2delta'])
    for pos_weight in (-1, 2.5):
        cfg = AttrDict(pos_weight=pos_weight)
        args = ([r.pos_bboxes for r in imgs], [r.neg_bboxes for r in imgs], [r.pos_gt_bboxes for r in imgs],
                [r.pos_gt_labels for r in imgs], cfg)
        got = bbox_target(*args, reg_classes=1231, target_means=means, target_stds=stds)
        for i, a in enumerate(got):
            b = d['bbox_target_%s_%d' % (pos_weight, i)]
            assert a.numpy().dtype == b.dtype and np.array_equal(a.numpy(), b)
        # not concatenated
        got = bbox_target(*args, target_means=means, target_stds=stds, concat=False)
        for i, la in enumerate(got):
            for j, a in enumerate(la):
                assert np.array_equal(a.numpy(), d['bbox_target_%s_split_%d_%d' % (pos_weight, i, j)])
            assert 'bbox_target_%s_split_%d_%d' % (pos_weight, i, len(la)) not in d
    # through the head method
    t = synthetic_tables()
    head = GSBBoxHeadWith0(num_fcs=1, in_channels=4, fc_out_channels=16, roi_feat_size=1, num_classes=t.num_classes,
                           target_means=means, target_stds=stds,
                           gs_config=dict(tables=t, others_sample_ratio=8.0, num_bins=5,
                                          loss_bin=dict(type='CrossEntropyLoss', use_sigmoid=False, loss_weight=1.0)))
    got = head.get_target(imgs, None, None, AttrDict(pos_weight=-1))
    assert all(np.array_equal(a.numpy(), d['bbox_target_-1_%d' % i]) for i, a in enumerate(got))
    assert got[0].dtype == torch.long and got[0][:5].tolist() == imgs[0].pos_gt_labels.tolist() and got[0][5:25].sum() == 0


def test_multiclass_nms_oracle_matches_reference_loop_in_op_order(ref):
    """The oracle's multiclass_nms against the reference's bbox_nms.py (its compiled NMS op replaced by the oracle's
    greedy "+1" NMS): thresholds, labels, class order, the op's ascending index order inside a class when nothing is
    cut, and the top-k rule."""
    _, d = ref
    boxes4, boxes_pc, scores = MG.nms_inputs()
    for bi, mb in enumerate((boxes4, boxes_pc)):
        for si, (thr, iou, k) in enumerate(MG.NMS_SETTINGS):
            got = O.multiclass_nms(mb, scores.clone(), thr, iou, k)
            assert np.array_equal(got[0].numpy(), d['nms_%d_%d_dets' % (bi, si)])
            assert np.array_equal(got[1].numpy(), d['nms_%d_%d_labels' % (bi, si)])


def test_reweight_variant_matches_reference(ref):
    """Reweight head variant (gs_bbox_head_with0_reweight.py): the oracle's weights / normalisers / per-bin losses
    against the reference class."""
    t, d = ref
    cls_weights = MG.reweight_weights(t)
    l2b, ps = torch.from_numpy(t.label2binlabel), torch.from_numpy(t.pred_slice)
    for N, npos, seed in MG.REWEIGHT_CASES:
        W, b, x, labels = MG.loss_case_inputs(N, npos, seed, t.num_logits, K=64)
        z = torch.nn.functional.linear(x, W, b)
        np.random.seed(seed)
        remapped = O.remap_labels_reweight(labels, l2b, 8.0, cls_weights)
        key = 'reweight_%d_' % seed
        for g, a in enumerate(remapped[1]):
            assert np.array_equal(a.float().numpy(), d[key + 'w%d' % g])
        assert [float(a) for a in remapped[2]] == d[key + 'avg'].tolist()
        got = O.bags_loss(z, labels, l2b, ps, remapped=remapped)
        want = d[key + 'losses']
        for g in range(5):
            k = 'loss_cls_bin%d' % g
            assert abs(got[k].item() - want[g]) <= 1e-6 * max(1.0, abs(want[g])), (k, got[k], want[g])
