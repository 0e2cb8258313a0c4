"""CPU: the RPN proposal restatement (tests/rpn_oracle.py) against the reference's own RPNHead.get_bboxes_single and
anchor_generator.py, executed in place through oracle/ref_shim with a CPU greedy stand-in for its NMS op; RPNHead's
construction from every LVIS config's rpn_head dict; the settings the native route refuses; and the argument rules
of bags_rpn_proposals / bags_rpn_scratch_bytes, which are checked before anything touches a device."""
import ctypes as C
import glob
import os
import runpy
import sys
import types

import numpy as np
import pytest
import torch

import rpn_oracle as O
from balancedgroupsoftmax_b200 import _native as nat
from balancedgroupsoftmax_b200.registry import HEADS, build_from_cfg
from balancedgroupsoftmax_b200.rpn_head import AnchorGenerator, RPNHead
from oracle import ref_shim

STATE_KEYS = ['rpn_conv.weight', 'rpn_conv.bias', 'rpn_cls.weight', 'rpn_cls.bias', 'rpn_reg.weight', 'rpn_reg.bias']
RPN_DICT = dict(type='RPNHead', in_channels=256, feat_channels=256, anchor_scales=[8], anchor_ratios=[0.5, 1.0, 2.0],
                anchor_strides=[4, 8, 16, 32, 64], target_means=[.0, .0, .0, .0], target_stds=[1.0, 1.0, 1.0, 1.0],
                loss_cls=dict(type='CrossEntropyLoss', use_sigmoid=True, loss_weight=1.0),
                loss_bbox=dict(type='SmoothL1Loss', beta=1.0 / 9.0, loss_weight=1.0))
_ref = None


def _reference():
    """The reference's anchor_generator.py, transforms.py and RPNHead (rpn_head.py over anchor_head.py), executed in
    place with stubs for what they import from outside that path; its NMS op is rpn_oracle.greedy_nms."""
    global _ref
    if _ref is not None:
        return _ref
    if not ref_shim.available():
        pytest.skip('no reference checkout')
    ns = ref_shim.load()
    ref_shim.load_bbox_target()
    md = os.path.join(ref_shim.reference_dir(), 'mmdet')
    cnn = types.ModuleType('mmcv.cnn')
    cnn.normal_init = lambda m, mean=0, std=1, bias=0: (torch.nn.init.normal_(m.weight, mean, std),
                                                        torch.nn.init.constant_(m.bias, bias))
    sys.modules['mmcv.cnn'] = cnn
    sys.modules['mmcv'].cnn = cnn
    core = sys.modules['mmdet.core']
    core.delta2bbox = sys.modules['mmdet.core.bbox.transforms'].delta2bbox
    core.multi_apply = sys.modules['mmdet.core.utils'].multi_apply
    core.anchor_target = core.multiclass_nms = None
    ag = ref_shim._exec('mmdet.core.anchor.anchor_generator', os.path.join(md, 'core', 'anchor', 'anchor_generator.py'))
    core.AnchorGenerator = ag.AnchorGenerator
    ops_pkg = sys.modules.get('mmdet.ops') or ref_shim._shell('mmdet.ops', os.path.join(md, 'ops'))
    ops_pkg.nms = O.greedy_nms
    ref_shim._shell('mmdet.models.anchor_heads', os.path.join(md, 'models', 'anchor_heads'))
    HEADS_ = sys.modules['mmdet.models.registry'].HEADS
    for name in ('AnchorHead', 'RPNHead'):
        HEADS_._module_dict.pop(name, None)
    ref_shim._exec('mmdet.models.anchor_heads.anchor_head', os.path.join(md, 'models', 'anchor_heads', 'anchor_head.py'))
    rpn = ref_shim._exec('mmdet.models.anchor_heads.rpn_head', os.path.join(md, 'models', 'anchor_heads', 'rpn_head.py'))
    _ref = types.SimpleNamespace(AnchorGenerator=ag.AnchorGenerator, RPNHead=rpn.RPNHead, AttrDict=ns.AttrDict)
    return _ref


def _rpn_dicts():
    """Every rpn_head dict of the reference's configs, where a checkout is reachable."""
    root = ref_shim.reference_dir()
    if root is None:
        return []
    found = []
    for path in sorted(glob.glob(os.path.join(root, 'configs', '**', '*.py'), recursive=True)):
        try:
            model = runpy.run_path(path).get('model')
        except Exception:
            continue
        if isinstance(model, dict) and isinstance(model.get('rpn_head'), dict):
            found.append((os.path.relpath(path, root), model['rpn_head']))
    return found


# ------------------------------------------------------------------------------------------------- the restatement
def test_greedy_nms_keeps_ascending_indices_and_suppresses_above_threshold():
    dets = torch.tensor([[0, 0, 9, 9, 0.5], [0, 0, 9, 9, 0.9], [20, 20, 29, 29, 0.7], [5, 0, 14, 9, 0.8]])
    kept, inds = O.greedy_nms(dets, 0.3)
    assert inds.tolist() == [1, 2]   # 3 overlaps 1 at IoU 1/3 > 0.3; 0 is 1's duplicate
    kept, inds = O.greedy_nms(dets, float(np.float32(50 / 150)))
    assert inds.tolist() == [1, 2, 3]
    assert O.greedy_nms(dets[:0], 0.5)[1].numel() == 0


def test_ties_are_broken_by_index():
    s = torch.tensor([0.5, 0.7, 0.5, 0.7, float('nan')])
    assert O._desc(s).tolist() == [4, 1, 3, 0, 2]


def _inputs(sizes, A, gen, scale=0.5):
    total = A * sum(h * w for h, w in sizes)
    vals = torch.linspace(-4, 4, total, dtype=torch.float64).float()[torch.randperm(total, generator=gen)]
    scores, deltas, o = [], [], 0
    for h, w in sizes:
        scores.append(vals[o:o + A * h * w].view(A, h, w))
        deltas.append(torch.randn(4 * A, h, w, generator=gen) * scale)
        o += A * h * w
    return scores, deltas


@pytest.mark.parametrize('case', ['selected', 'anchor_order', 'nms_post', 'max_num', 'min_bbox', 'norm'])
def test_reference_get_bboxes_single_equals_the_oracle(case):
    ref = _reference()
    gen = torch.Generator().manual_seed(['selected', 'anchor_order', 'nms_post', 'max_num', 'min_bbox',
                                         'norm'].index(case))
    cfg = dict(nms_across_levels=False, nms_pre=300, nms_post=300, max_num=500, nms_thr=0.7, min_bbox_size=0)
    means, stds = (.0, .0, .0, .0), (1.0, 1.0, 1.0, 1.0)
    if case == 'anchor_order':
        cfg.update(nms_pre=5000, nms_post=20)
    elif case == 'nms_post':
        cfg.update(nms_post=30)
    elif case == 'max_num':
        cfg.update(max_num=70)
    elif case == 'min_bbox':
        cfg.update(min_bbox_size=20)
    elif case == 'norm':
        means, stds = (0.1, -0.1, 0.05, 0.0), (0.1, 0.1, 0.2, 0.2)
    sizes, strides = [(16, 20), (8, 10), (4, 5)], [4, 8, 16]
    head = ref.RPNHead(in_channels=8, feat_channels=8, anchor_scales=[8], anchor_ratios=[0.5, 1.0, 2.0],
                       anchor_strides=strides, target_means=means, target_stds=stds)
    scores, deltas = _inputs(sizes, 3, gen, 1.0 if case == 'min_bbox' else 0.5)
    anchors = [g.grid_anchors(s, st, device='cpu') for g, s, st in zip(head.anchor_generators, sizes, strides)]
    img_shape = (60, 75, 3)
    want = head.get_bboxes_single(scores, deltas, anchors, img_shape, 1.0, ref.AttrDict(cfg))
    got = O.get_bboxes_single(scores, deltas, anchors, img_shape, cfg, O.greedy_nms, means, stds)
    assert want.shape[0] > 0 and torch.equal(got, want)
    if case == 'anchor_order':   # the cut took survivors in anchor order: not the 20 best of each level
        assert want.shape[0] == 60


def test_reference_anchors_of_every_config():
    ref = _reference()
    found = _rpn_dicts()
    assert len(found) >= 10
    for path, d in found:
        for base in d.get('anchor_base_sizes') or d['anchor_strides']:
            mine = AnchorGenerator(base, d['anchor_scales'], d['anchor_ratios'])
            theirs = ref.AnchorGenerator(base, d['anchor_scales'], d['anchor_ratios'])
            assert torch.equal(mine.base_anchors, theirs.base_anchors), (path, base)
            assert torch.equal(mine.grid_anchors((5, 7), base, 'cpu'), theirs.grid_anchors((5, 7), base, 'cpu'))
            assert torch.equal(O.grid_anchors(mine.base_anchors, 5, 7, base), theirs.grid_anchors((5, 7), base, 'cpu'))
            assert torch.equal(mine.valid_flags((5, 7), (3, 6), 'cpu'), theirs.valid_flags((5, 7), (3, 6), 'cpu'))


# ------------------------------------------------------------------------------------------------------ the module
def _check_built(d, head):
    assert isinstance(head, RPNHead)
    assert head.in_channels == d['in_channels'] and head.feat_channels == d['feat_channels']
    assert head.anchor_scales == d['anchor_scales'] and head.anchor_ratios == d['anchor_ratios']
    assert head.anchor_strides == d['anchor_strides'] and head.num_anchors == 3
    assert head.use_sigmoid_cls and head.cls_out_channels == 1 and head.sampling
    assert list(head.state_dict().keys()) == STATE_KEYS
    assert head.rpn_cls.out_channels == 3 and head.rpn_reg.out_channels == 12
    head.init_weights()


def test_rpn_dict_builds():
    assert HEADS.get('RPNHead') is RPNHead
    _check_built(RPN_DICT, build_from_cfg(dict(RPN_DICT), HEADS))


def test_every_reference_config_rpn_head_builds_with_the_reference_keys():
    found = _rpn_dicts()
    if not found:
        pytest.skip('no reference checkout')
    ref = _reference()
    for path, d in found:
        _check_built(d, build_from_cfg(dict(d), HEADS))
        args = dict(d)
        args.pop('type')
        theirs = ref.RPNHead(**args)
        assert list(theirs.state_dict().keys()) == STATE_KEYS, path
        assert [tuple(v.shape) for v in theirs.state_dict().values()] == \
            [tuple(v.shape) for v in build_from_cfg(dict(d), HEADS).state_dict().values()]


@pytest.mark.parametrize('setting', ['softmax', 'across', 'cap'])
def test_settings_without_a_native_route_raise(setting, monkeypatch):
    # without mmdet (the reference loaded in place by other tests would otherwise stand in for it)
    from balancedgroupsoftmax_b200 import rpn_head
    monkeypatch.setattr(rpn_head, '_mmdet_rpn_get_bboxes_single', lambda: None)
    d = dict(RPN_DICT)
    cfg = dict(nms_across_levels=False, nms_pre=1000, nms_post=1000, max_num=1000, nms_thr=0.7, min_bbox_size=0)
    if setting == 'softmax':
        d['loss_cls'] = dict(type='CrossEntropyLoss', use_sigmoid=False, loss_weight=1.0)
    elif setting == 'across':
        cfg['nms_across_levels'] = True
    else:
        cfg['nms_pre'] = 5000
    head = build_from_cfg(d, HEADS)
    A = head.num_anchors * head.cls_out_channels
    cls = [torch.zeros(1, A, 80, 80), torch.zeros(1, A, 40, 40)]
    reg = [torch.zeros(1, 12, 80, 80), torch.zeros(1, 12, 40, 40)]
    match = {'softmax': 'use_sigmoid=False', 'across': 'nms_across_levels', 'cap': 'candidates'}[setting]
    with pytest.raises(NotImplementedError, match=match):
        head.get_bboxes(cls, reg, [dict(img_shape=(320, 320, 3), scale_factor=1.0)], cfg)


def test_loss_needs_mmdet_and_cpu_inputs_raise(monkeypatch):
    from balancedgroupsoftmax_b200 import rpn_head
    monkeypatch.setattr(rpn_head, '_mmdet_core', lambda name: None)
    monkeypatch.setattr(rpn_head, '_mmdet_rpn_get_bboxes_single', lambda: None)
    head = build_from_cfg(dict(RPN_DICT), HEADS)
    with pytest.raises(NotImplementedError, match='anchor_target'):
        head.loss([torch.zeros(1, 3, 4, 4)], [torch.zeros(1, 12, 4, 4)], [torch.zeros(1, 4)], [{}], {})
    cfg = dict(nms_pre=10, nms_post=10, max_num=10, nms_thr=0.7, min_bbox_size=0)
    with pytest.raises(NotImplementedError, match='CPU tensors'):
        head.get_bboxes([torch.zeros(1, 3, 4, 4)], [torch.zeros(1, 12, 4, 4)], [dict(img_shape=(16, 16, 3))], cfg)


@pytest.mark.parametrize('setting', ['softmax', 'across', 'cpu'])
def test_drop_in_falls_back_to_the_reference_loop(setting):
    """Under the drop-in, this package's RPNHead is the one registered in mmdet's HEADS and mmdet's rpn_head module has
    not been imported.  A setting without a native route imports that module (whose own registration would collide)
    and runs its get_bboxes_single: the proposals are the reference's, and the registered RPNHead stays this one."""
    ref = _reference()
    name = 'mmdet.models.anchor_heads.rpn_head'
    registry = sys.modules['mmdet.models.registry'].HEADS
    saved_mod, saved_cls = sys.modules.pop(name), registry._module_dict.pop('RPNHead', None)
    registry._module_dict['RPNHead'] = RPNHead   # what the drop-in's import registers
    try:
        d = dict(RPN_DICT, in_channels=8, feat_channels=8, anchor_strides=[4, 8, 16])
        cfg = ref.AttrDict(nms_across_levels=setting == 'across', nms_pre=300, nms_post=300, max_num=400, nms_thr=0.7,
                           min_bbox_size=0)
        if setting == 'softmax':
            d['loss_cls'] = dict(type='CrossEntropyLoss', use_sigmoid=False, loss_weight=1.0)
        head = registry.get('RPNHead')(**{k: v for k, v in d.items() if k != 'type'})
        assert type(head) is RPNHead
        gen = torch.Generator().manual_seed(11)
        sizes = [(16, 20), (8, 10), (4, 5)]
        scores, deltas = _inputs(sizes, 3 * head.cls_out_channels, gen)
        deltas = [torch.randn(12, h, w, generator=gen) * 0.5 for h, w in sizes]
        metas = [dict(img_shape=(60, 75, 3), scale_factor=1.0), dict(img_shape=(50, 70, 3), scale_factor=1.0)]
        batch_s = [torch.stack([s, s.flip(0)]) for s in scores]
        batch_d = [torch.stack([x, -x]) for x in deltas]
        got = head.get_bboxes(batch_s, batch_d, metas, cfg)
        assert registry.get('RPNHead') is RPNHead
        theirs = sys.modules[name].RPNHead(**{k: v for k, v in d.items() if k != 'type'})
        anchors = [g.grid_anchors(s, st, device='cpu') for g, s, st in zip(theirs.anchor_generators, sizes, [4, 8, 16])]
        for b in range(2):
            want = theirs.get_bboxes_single([s[b] for s in batch_s], [x[b] for x in batch_d], anchors,
                                            metas[b]['img_shape'], 1.0, cfg)
            assert want.shape[0] > 0 and torch.equal(got[b], want), (setting, b)
    finally:
        sys.modules[name] = saved_mod
        registry._module_dict.pop('RPNHead', None)
        if saved_cls is not None:
            registry._module_dict['RPNHead'] = saved_cls


# ----------------------------------------------------------------------------------------- the C ABI's rules
def _levels(*rows):
    return np.ascontiguousarray(np.array(rows, dtype=np.int32).reshape(-1, 4))


def _abi_call(levels=None, L=None, B=1, nms_pre=1000, nms_post=1000, max_num=1000, ptrs=True, scratch=True,
              scratch_bytes=1 << 30, out=True, shapes=((64, 64),)):
    lib = nat.lib()
    levels = _levels((16, 16, 3, 4)) if levels is None else levels
    L = levels.shape[0] if L is None else L
    buf = (C.c_char * 4096)()
    base = (C.addressof(buf) + 255) // 256 * 256
    n = max(L, 1)
    lp = (C.c_void_p * n)(*([base if ptrs else None] * n))
    anchors = (C.c_float * (4 * 16 * 8))()
    shp = nat.int32_array([v for s in list(shapes) + [(64, 64)] * max(0, B - len(shapes)) for v in s])
    ms = (C.c_float * 4)(0, 0, 0, 0)
    sd = (C.c_float * 4)(1, 1, 1, 1)
    o = base if out else None
    return lib.bags_rpn_proposals(lp, lp, levels.ctypes.data, anchors, L, B, shp, nms_pre, nms_post, max_num, 0.7,
                                  0.0, ms, sd, base if scratch else None, scratch_bytes, o, o, None)


def test_rpn_abi_rejects_bad_arguments():
    lib = nat.lib()
    bad = [dict(L=0), dict(L=9), dict(B=0), dict(B=33), dict(levels=_levels((16, 16, 17, 4))),
           dict(levels=_levels((16, 16, 0, 4))), dict(levels=_levels((-1, 16, 3, 4))),
           dict(levels=_levels((16, 16, 3, 0))), dict(max_num=0), dict(nms_post=0),
           dict(levels=_levels((40, 40, 3, 4)), nms_pre=-1), dict(levels=_levels((40, 40, 3, 4)), nms_pre=5000),
           dict(nms_pre=4097, levels=_levels((40, 40, 3, 4))), dict(ptrs=False), dict(scratch=False),
           dict(out=False), dict(scratch_bytes=16)]
    for kw in bad:
        assert _abi_call(**kw) == -1, kw
        assert b'bags_rpn_proposals' in lib.bags_last_error(), (kw, lib.bags_last_error())


def test_rpn_scratch_bytes():
    lib = nat.lib()
    out = C.c_size_t(0)
    lv = _levels((200, 336, 3, 4), (100, 168, 3, 8), (50, 84, 3, 16), (25, 42, 3, 32), (13, 21, 3, 64))
    assert lib.bags_rpn_scratch_bytes(lv.ctypes.data, 5, 2, 2000, 2000, C.byref(out)) == 0
    one = C.c_size_t(0)
    assert lib.bags_rpn_scratch_bytes(lv.ctypes.data, 5, 1, 2000, 2000, C.byref(one)) == 0
    # per image: four levels of 2000 candidates and one of 819, each a candidate list, a bit matrix and survivors
    words = lambda k: (k + 63) // 64   # noqa: E731
    r = lambda x: (x + 255) // 256 * 256   # noqa: E731
    per = 4 * (r(24 * 2000) + r(2000 * words(2000) * 8) + r(20 * 2000)) + r(24 * 819) + r(819 * words(819) * 8) + \
        r(20 * 819)
    assert out.value - one.value == per
    assert lib.bags_rpn_scratch_bytes(lv.ctypes.data, 5, 2, -1, 2000, C.byref(out)) == -1   # P2 without selection
    assert lib.bags_rpn_scratch_bytes(lv.ctypes.data, 5, 2, 2000, 2000, None) == -1
