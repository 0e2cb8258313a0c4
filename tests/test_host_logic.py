"""CPU: the host-side mirror of the reference's BBoxHead API (registry, config build, state dict,
decorators, sampler host logic).  No kernels run here."""
import numpy as np
import pytest
import torch

from balancedgroupsoftmax_b200 import registry
from balancedgroupsoftmax_b200.fp16 import auto_fp16, force_fp32
from balancedgroupsoftmax_b200.head import ClsScoreHandle, GSBBoxHead, GSBBoxHeadWith0, delta2bbox
from balancedgroupsoftmax_b200.losses import CrossEntropyLoss, SmoothL1Loss
from balancedgroupsoftmax_b200.tables import save_reference_files, synthetic_tables


class ConfigDict(dict):
    __getattr__ = dict.__getitem__


def bags_cfg(paths, attr_style):
    """bbox_head block of configs/bags/gs_faster_rcnn_r50_fpn_1x_lvis_with0_bg8.py:34-59."""
    mk = ConfigDict if attr_style else dict
    return dict(
        type='GSBBoxHeadWith0', num_fcs=2, in_channels=256, fc_out_channels=1024,
        gs_config=mk(label2binlabel=paths['label2binlabel'], pred_slice=paths['pred_slice'],
                     fg_split=paths['fg_split'], others_sample_ratio=8.0,
                     loss_bg=dict(type='CrossEntropyLoss', use_sigmoid=False, loss_weight=1.0), num_bins=5,
                     loss_bin=dict(type='CrossEntropyLoss', use_sigmoid=False, loss_weight=1.0)),
        roi_feat_size=7, num_classes=1231, target_means=[0., 0., 0., 0.], target_stds=[0.1, 0.1, 0.2, 0.2],
        reg_class_agnostic=False,
        loss_cls=dict(type='CrossEntropyLoss', use_sigmoid=False, loss_weight=1.0),
        loss_bbox=dict(type='SmoothL1Loss', beta=1.0, loss_weight=1.0))


@pytest.fixture(scope='module')
def table_files(tmp_path_factory):
    d = tmp_path_factory.mktemp('tables')
    return save_reference_files(synthetic_tables(1231, seed=0), str(d))


@pytest.mark.parametrize('attr_style', [False, True])
def test_builds_from_reference_config_block(table_files, attr_style):
    head = registry.build_head(bags_cfg(table_files, attr_style))
    assert isinstance(head, GSBBoxHeadWith0)
    assert head.fc_cls.in_features == 1024 and head.fc_cls.out_features == 1236
    assert head.fc_reg.out_features == 4 * 1231
    assert head.num_classes == 1231 and head.fp16_enabled is False and head.reg_class_agnostic is False
    assert head.others_sample_ratio == 8.0 and len(head.loss_bins) == 5
    sd = head.state_dict()
    assert {k: tuple(v.shape) for k, v in sd.items()} == {
        'shared_fcs.0.weight': (1024, 12544), 'shared_fcs.0.bias': (1024,),
        'shared_fcs.1.weight': (1024, 1024), 'shared_fcs.1.bias': (1024,),
        'fc_cls.weight': (1236, 1024), 'fc_cls.bias': (1236,),
        'fc_reg.weight': (4924, 1024), 'fc_reg.bias': (4924,)}
    assert all(v.dtype == torch.float32 for v in sd.values())
    # tables are plain attributes, not in the state dict (gs_bbox_head_with0.py:37-49)
    assert head.label2binlabel.dtype == torch.int64 and len(head.fg_splits) == 4


def test_registry_contract():
    assert registry.HEADS.get('GSBBoxHeadWith0') is GSBBoxHeadWith0
    assert registry.HEADS.get('GSBBoxHead') is GSBBoxHead
    assert registry.HEADS.get('SharedFCBBoxHead') is not None
    assert registry.LOSSES.get('CrossEntropyLoss') is CrossEntropyLoss
    with pytest.raises(KeyError):
        registry.build_from_cfg(dict(type='Nope'), registry.HEADS)
    with pytest.raises(TypeError):
        registry.build_from_cfg(dict(type=3), registry.HEADS)
    r = registry.Registry('x')

    @r.register_module
    class A(object):
        pass

    assert r.get('A') is A
    with pytest.raises(KeyError):
        r.register_module(A)
    obj = registry.build_from_cfg(dict(type='SmoothL1Loss'), registry.LOSSES, default_args=dict(beta=0.5))
    assert isinstance(obj, SmoothL1Loss) and obj.beta == 0.5


def test_init_weights_like_reference():
    t = synthetic_tables()
    head = GSBBoxHeadWith0(num_fcs=2, in_channels=8, fc_out_channels=64, roi_feat_size=2, num_classes=1231,
                           gs_config=dict(tables=t, others_sample_ratio=8.0, num_bins=5,
                                          loss_bin=dict(type='CrossEntropyLoss', use_sigmoid=False, loss_weight=1.0)))
    torch.manual_seed(0)
    head.init_weights()
    assert abs(head.fc_cls.weight.std().item() - 0.01) < 1e-3 and head.fc_cls.bias.abs().sum().item() == 0
    assert abs(head.fc_reg.weight.std().item() - 0.001) < 1e-4


def test_training_forward_returns_lazy_handle_and_cpu_loss_raises():
    from balancedgroupsoftmax_b200._native import BagsNativeError
    t = synthetic_tables()
    head = GSBBoxHeadWith0(num_fcs=2, in_channels=4, fc_out_channels=64, roi_feat_size=2, num_classes=1231,
                           gs_config=dict(tables=t, others_sample_ratio=8.0, num_bins=5,
                                          loss_bin=dict(type='CrossEntropyLoss', use_sigmoid=False, loss_weight=1.0)))
    head.train()
    cls_score, bbox_pred = head(torch.randn(10, 4, 2, 2))
    assert isinstance(cls_score, ClsScoreHandle)
    assert tuple(cls_score.shape) == (10, 1236) and cls_score.size(1) == 1236 and cls_score.dim() == 2
    assert tuple(bbox_pred.shape) == (10, 4 * 1231)
    labels = torch.zeros(10, dtype=torch.long)
    with pytest.raises(BagsNativeError):          # no CPU fallback for the hot path
        head.loss(cls_score, None, labels, None, None, None)
    with pytest.raises(BagsNativeError):
        head.eval()(torch.randn(10, 4, 2, 2))


def test_bbox_loss_branch_matches_reference_formula():
    t = synthetic_tables()
    head = GSBBoxHeadWith0(num_fcs=1, in_channels=4, fc_out_channels=32, roi_feat_size=1, num_classes=1231,
                           reg_class_agnostic=True,
                           gs_config=dict(tables=t, others_sample_ratio=8.0, num_bins=5,
                                          loss_bin=dict(type='CrossEntropyLoss', use_sigmoid=False, loss_weight=1.0)))
    labels = torch.tensor([3, 0, 7, 0])
    bbox_pred = torch.tensor([[0.1, 0.2, 2.0, -3.0]] * 4)
    targets = torch.zeros(4, 4)
    weights = torch.ones(4, 4)
    out = head.loss(None, bbox_pred, labels, None, targets, weights)
    # smooth-l1(beta=1): 0.005 + 0.02 + 1.5 + 2.5 per positive row, 2 positives, avg_factor = 4 rows
    assert abs(out['loss_bbox'].item() - 2 * (0.005 + 0.02 + 1.5 + 2.5) / 4) < 1e-6
    assert list(out.keys()) == ['loss_bbox']


def test_fp16_decorators():
    class M(torch.nn.Module):
        def __init__(self):
            super().__init__()
            self.fp16_enabled = False

        @force_fp32(apply_to=('a', ))
        def f(self, a, b):
            return a.dtype, b.dtype

        @force_fp32(apply_to=('cls_score'))     # bare string: substring membership, as the reference relies on
        def g(self, cls_score, other):
            return cls_score.dtype, other.dtype

        @auto_fp16(apply_to=('a', ), out_fp32=True)
        def h(self, a):
            return a

    m = M()
    h, f = torch.zeros(2).half(), torch.zeros(2)
    assert m.f(h, h) == (torch.float16, torch.float16)          # disabled -> untouched
    m.fp16_enabled = True
    assert m.f(h, h) == (torch.float32, torch.float16)
    assert m.f(a=h, b=h) == (torch.float32, torch.float16)
    assert m.g(h, h) == (torch.float32, torch.float16)
    assert m.h(f).dtype == torch.float32
    with pytest.raises(TypeError):
        force_fp32()(lambda x: x)(3)


def test_delta2bbox_doctest_values():
    """mmdet/core/bbox/transforms.py:63-76 known answers."""
    rois = torch.Tensor([[0., 0., 1., 1.], [0., 0., 1., 1.], [0., 0., 1., 1.], [5., 5., 5., 5.]])
    deltas = torch.Tensor([[0., 0., 0., 0.], [1., 1., 1., 1.], [0., 0., 2., -1.], [0.7, -1.9, -0.5, 0.3]])
    out = delta2bbox(rois, deltas, max_shape=(32, 32))
    exp = torch.tensor([[0.0000, 0.0000, 1.0000, 1.0000], [0.2817, 0.2817, 4.7183, 4.7183],
                        [0.0000, 0.6321, 7.3891, 0.3679], [5.8967, 2.9251, 5.5033, 3.2749]])
    assert torch.allclose(out, exp, atol=1e-4)


def test_loss_modules_semantics():
    ce = CrossEntropyLoss(loss_weight=2.0)
    z = torch.tensor([[2.0, 0.0], [0.0, 0.0]])
    y = torch.tensor([0, 1])
    w = torch.tensor([1, 0])
    per = torch.nn.functional.cross_entropy(z, y, reduction='none')
    assert torch.allclose(ce(z, y, w, avg_factor=4.0), 2.0 * (per * w.float()).sum() / 4.0)
    assert torch.allclose(ce(z, y, reduction_override='none'), 2.0 * per)
    with pytest.raises(ValueError):
        ce(z, y, w, avg_factor=2.0, reduction_override='sum')


def test_hostmem_cpulist_and_affinity_restore():
    """NUMA staging helpers: cpulist parsing; the affinity / thread-count context always restores the caller's state
    (and degrades to a no-op when the GPU topology cannot be read, as in this container)."""
    import os
    import torch
    from balancedgroupsoftmax_b200 import hostmem
    assert hostmem._parse_cpulist('0-3,8,10-11\n') == {0, 1, 2, 3, 8, 10, 11}
    assert hostmem._parse_cpulist('') == set()
    aff, nt = os.sched_getaffinity(0), torch.get_num_threads()
    with hostmem.gpu_local_affinity(0) as cpus:
        assert cpus is None or cpus <= aff
        assert torch.get_num_threads() == 1
    assert os.sched_getaffinity(0) == aff and torch.get_num_threads() == nt


def test_load_reference_checkpoint_roundtrip(tmp_path):
    """A checkpoint laid out like the reference's (mmcv dict, 'bbox_head.' prefix, optional 'module.') loads into the
    head; shape mismatches and missing prefixes are refused."""
    import torch
    from balancedgroupsoftmax_b200.head import GSBBoxHeadWith0
    from balancedgroupsoftmax_b200.tables import synthetic_tables
    t = synthetic_tables()
    mk = lambda: GSBBoxHeadWith0(num_fcs=2, in_channels=4, fc_out_channels=32, roi_feat_size=2, num_classes=t.num_classes,
                                 gs_config=dict(tables=t, others_sample_ratio=8.0, num_bins=5,
                                                loss_bin=dict(type='CrossEntropyLoss', use_sigmoid=False, loss_weight=1.0)))
    src, dst = mk(), mk()
    src.init_weights()
    with torch.no_grad():
        src.fc_cls.bias.uniform_(-1, 1)
    sd = {'module.bbox_head.' + k: v.clone() for k, v in src.state_dict().items()}
    sd['module.backbone.conv1.weight'] = torch.zeros(3)
    path = tmp_path / 'epoch_12.pth'
    torch.save({'meta': {}, 'state_dict': sd}, str(path))
    missing, unexpected = dst.load_reference_checkpoint(str(path))
    assert not missing and not unexpected
    assert dst.fc_cls.weight.shape == (t.num_logits, 32)
    for k, v in src.state_dict().items():
        assert torch.equal(dst.state_dict()[k], v)
    import pytest
    with pytest.raises(KeyError):
        dst.load_reference_checkpoint({'state_dict': sd}, prefix='bbox_head.2.')
    bad = dict(sd)
    bad['module.bbox_head.fc_cls.weight'] = torch.zeros(1231, 32)
    with pytest.raises(ValueError):
        dst.load_reference_checkpoint({'state_dict': bad})


def test_get_target_known_values():
    """bbox_target / bbox2delta restatement on hand-checkable boxes (mmdet/core/bbox/bbox_target.py:36-63,
    transforms.py:6-31): positives first with their labels, negatives label 0, '+1' box widths."""
    import math
    from types import SimpleNamespace
    import torch
    from balancedgroupsoftmax_b200.head import bbox2delta, bbox_target
    p = torch.tensor([[0., 0., 9., 9.]])          # 10 x 10, centre 4.5
    gt = torch.tensor([[2., 0., 21., 9.]])        # 20 x 10, centre (11.5, 4.5)
    d = bbox2delta(p, gt, (0, 0, 0, 0), (0.1, 0.1, 0.2, 0.2))
    assert torch.allclose(d, torch.tensor([[7.0, 0.0, math.log(2.0) / 0.2, 0.0]]), atol=1e-6)
    neg = torch.tensor([[1., 1., 2., 2.], [3., 3., 4., 4.]])
    labels, lw, bt, bw = bbox_target([p], [neg], [gt], [torch.tensor([17])], dict(pos_weight=-1),
                                     target_stds=(0.1, 0.1, 0.2, 0.2))
    assert labels.tolist() == [17, 0, 0] and labels.dtype == torch.long
    assert lw.tolist() == [1.0, 1.0, 1.0]
    assert torch.allclose(bt[0], d[0]) and bt[1:].abs().sum() == 0
    assert bw.tolist() == [[1, 1, 1, 1], [0, 0, 0, 0], [0, 0, 0, 0]]
    _, lw2, _, _ = bbox_target([p], [neg], [gt], [torch.tensor([17])], SimpleNamespace(pos_weight=3.0))
    assert lw2.tolist() == [3.0, 1.0, 1.0]
    # an image without positives, one without negatives
    e = torch.zeros(0, 4)
    labels, lw, bt, bw = bbox_target([e, p], [neg, e], [e, gt], [torch.zeros(0, dtype=torch.long), torch.tensor([5])],
                                     dict(pos_weight=-1))
    assert labels.tolist() == [0, 0, 5] and lw.tolist() == [1.0, 1.0, 1.0] and bw[:, 0].tolist() == [0, 0, 1]


def test_graphed_step_refuses_cpu_parameters():
    """No CPU fallback for the graph-captured step either."""
    import pytest
    import torch
    from balancedgroupsoftmax_b200._native import BagsNativeError
    from balancedgroupsoftmax_b200.api import GraphedHeadStep
    from balancedgroupsoftmax_b200.tables import synthetic_tables
    w = torch.nn.Parameter(torch.zeros(1236, 64))
    with pytest.raises(BagsNativeError):
        GraphedHeadStep(w, None, synthetic_tables(), 32)


def test_reweight_head_variant_construction(tmp_path):
    """GSBBoxHeadWith0Reweight: registered, reads bin_cls_weight in the reference's pickle format, validates lengths."""
    import pickle
    import numpy as np
    import pytest
    import torch
    from balancedgroupsoftmax_b200.head import GSBBoxHeadWith0Reweight
    from balancedgroupsoftmax_b200.registry import HEADS, build_from_cfg
    from balancedgroupsoftmax_b200.tables import save_reference_files, synthetic_tables
    t = synthetic_tables()
    paths = save_reference_files(t, str(tmp_path))
    ws = [np.linspace(0.5, 1.5, int(t.pred_slice[g, 1])).astype(np.float32) for g in range(1, 5)]
    wfile = tmp_path / 'bin_cls_weight.pkl'
    with open(wfile, 'wb') as f:
        pickle.dump(ws, f)
    cfg = dict(type='GSBBoxHeadWith0Reweight', num_fcs=2, in_channels=4, fc_out_channels=32, roi_feat_size=2,
               num_classes=1231,
               gs_config=dict(label2binlabel=paths['label2binlabel'], pred_slice=paths['pred_slice'],
                              fg_split=paths['fg_split'], others_sample_ratio=8.0, num_bins=5,
                              bin_cls_weight=str(wfile),
                              loss_bin=dict(type='CrossEntropyLoss', use_sigmoid=False, loss_weight=1.0)))
    head = build_from_cfg(cfg, HEADS)
    assert isinstance(head, GSBBoxHeadWith0Reweight) and len(head.cls_weights) == 4
    tab = head._cls_weight_table
    assert tab.shape == (5, max(len(w) for w in ws)) and torch.all(tab[0] == 1)
    for g, w in enumerate(ws, start=1):
        assert torch.allclose(tab[g, :len(w)], torch.from_numpy(w)) and torch.all(tab[g, len(w):] == 1)
    bad = dict(cfg)
    bad['gs_config'] = dict(cfg['gs_config'], cls_weights=[w[:-1] for w in ws])
    with pytest.raises(AssertionError):
        build_from_cfg(bad, HEADS)


def test_head_reports_kernel_limits_at_construction():
    """Bin tables the native kernels cannot take (ADVICE r1: 3 bins -> 1234 logits, 9 bins) are rejected when the head is
    built, not at the first loss / merge call; a non-'mean' loss_bin reduction likewise."""
    from balancedgroupsoftmax_b200.tables import GroupTables

    def fake_tables(num_bins, num_classes=1231):
        # bin 0 = {bg, fg}; foreground classes dealt round-robin to bins 1..num_bins-1
        l2b = np.zeros((num_bins, num_classes), dtype=np.int64)
        l2b[0, 1:] = 1
        counts = [2]
        splits = []
        for g in range(1, num_bins):
            ids = np.arange(g, num_classes, num_bins - 1)
            ids = ids[ids >= 1]
            l2b[g, ids] = np.arange(1, len(ids) + 1)
            counts.append(len(ids) + 1)
            splits.append(ids.astype(np.int64))
        starts = np.concatenate([[0], np.cumsum(counts)[:-1]])
        ps = np.stack([starts, np.array(counts)], 1).astype(np.int64)
        return GroupTables(l2b, ps, splits)

    def build(tables, **over):
        cfg = dict(tables=tables, others_sample_ratio=8.0, num_bins=tables.num_bins,
                   loss_bin=dict(type='CrossEntropyLoss', use_sigmoid=False, loss_weight=1.0))
        cfg.update(over)
        return GSBBoxHeadWith0(num_fcs=1, in_channels=4, fc_out_channels=16, roi_feat_size=1, num_classes=1231, gs_config=cfg)

    t3 = fake_tables(3)
    assert t3.num_logits == 1231 + 3
    with pytest.raises(ValueError, match='multiple of 4'):
        build(t3)
    with pytest.raises(ValueError, match='at most 8'):
        build(fake_tables(9))
    with pytest.raises(ValueError, match='reduction'):
        build(synthetic_tables(1231, seed=0), loss_bin=dict(type='CrossEntropyLoss', use_sigmoid=False, loss_weight=1.0,
                                                             reduction='sum'))
    build(synthetic_tables(1231, seed=0))     # the 5-bin LVIS-shaped tables are fine


def test_cls_score_handle_works_with_torch_functions():
    """The lazy cls_score of the training forward behaves like the reference's plain tensor for callers that hand it
    to torch functions (torch.cat, softmax, ...): __torch_function__ materialises the logits."""
    class FakeHead(object):
        class fc_cls(object):
            out_features = 6

        def _fc_cls_logits(self, x):
            return x @ torch.arange(24, dtype=torch.float32).view(6, 4).t()
    x = torch.randn(5, 4)
    h = ClsScoreHandle(FakeHead(), x)
    z = FakeHead()._fc_cls_logits(x)
    assert tuple(h.shape) == (5, 6) and h.size(1) == 6 and h.dim() == 2 and h.pending
    assert torch.equal(torch.cat([h, z], 0), torch.cat([z, z], 0)) and not h.pending
    assert torch.allclose(torch.softmax(h, 1), torch.softmax(z, 1))
    assert torch.equal(h.argmax(1), z.argmax(1)) and torch.equal(h[:, 1:3], z[:, 1:3])
    assert torch.equal(torch.stack((h, h)).sum(0), 2 * z)
