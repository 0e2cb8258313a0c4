"""CPU: the RPN target restatement (tests/anchor_target_oracle.py) against the reference's own anchor_target,
MaxIoUAssigner, RandomSampler and bbox2delta, executed in place through oracle/ref_shim with np.random.seed fixed and
the same draw injected; the host decisions of RPNHead's native route (inside anchors, no gt, config parsing); the
statistics of the native selection rule; and the argument rules of bags_anchor_target, which are checked before
anything touches a device."""
import ctypes as C
import glob
import os
import runpy
import sys
import types

import numpy as np
import pytest
import torch

import anchor_target_oracle as O
from anchor_target_cases import EDGE_BASE, RPN_CFG, _boxes, _cfg, _head_bases, cases, edge_gts
import sampler_oracle as S
from balancedgroupsoftmax_b200 import _native as nat
from balancedgroupsoftmax_b200.registry import HEADS, build_from_cfg
from oracle import ref_shim

RPN_DICT = dict(type='RPNHead', in_channels=8, feat_channels=8, anchor_scales=[8], anchor_ratios=[0.5, 1.0, 2.0],
                anchor_strides=[4, 8, 16, 32, 64])
_ref = None


def _reference():
    """The reference's anchor_target.py, assign_sampling.py, MaxIoUAssigner, RandomSampler / PseudoSampler and
    transforms.py executed in place; the stubs: mmcv.runner.obj_from_dict and multi_apply."""
    global _ref
    if _ref is not None:
        return _ref
    if not ref_shim.available():
        pytest.skip('no reference checkout')
    ns = ref_shim.load()
    ref_shim.load_bbox_target()
    md = os.path.join(ref_shim.reference_dir(), 'mmdet')
    bd = os.path.join(md, 'core', 'bbox')

    def obj_from_dict(info, parent=None, default_args=None):   # mmcv/runner/utils.py
        args = dict(info)
        obj_type = args.pop('type')
        for k, v in (default_args or {}).items():
            args.setdefault(k, v)
        return getattr(parent, obj_type)(**args)
    runner = types.ModuleType('mmcv.runner')
    runner.obj_from_dict = obj_from_dict
    sys.modules['mmcv.runner'] = runner
    sys.modules['mmcv'].runner = runner
    bbox = sys.modules['mmdet.core.bbox']
    ref_shim._exec('mmdet.core.bbox.geometry', os.path.join(bd, 'geometry.py'))
    asg = ref_shim._shell('mmdet.core.bbox.assigners', os.path.join(bd, 'assigners'))
    for name in ('base_assigner', 'assign_result', 'max_iou_assigner'):
        ref_shim._exec('mmdet.core.bbox.assigners.' + name, os.path.join(bd, 'assigners', name + '.py'))
    asg.MaxIoUAssigner = sys.modules['mmdet.core.bbox.assigners.max_iou_assigner'].MaxIoUAssigner
    asg.BaseAssigner = sys.modules['mmdet.core.bbox.assigners.base_assigner'].BaseAssigner
    smp = ref_shim._shell('mmdet.core.bbox.samplers', os.path.join(bd, 'samplers'))
    for name in ('sampling_result', 'base_sampler', 'random_sampler', 'pseudo_sampler'):
        ref_shim._exec('mmdet.core.bbox.samplers.' + name, os.path.join(bd, 'samplers', name + '.py'))
    smp.RandomSampler = sys.modules['mmdet.core.bbox.samplers.random_sampler'].RandomSampler
    smp.PseudoSampler = sys.modules['mmdet.core.bbox.samplers.pseudo_sampler'].PseudoSampler
    smp.BaseSampler = sys.modules['mmdet.core.bbox.samplers.base_sampler'].BaseSampler
    bbox.assigners, bbox.samplers = asg, smp
    asn = ref_shim._exec('mmdet.core.bbox.assign_sampling', os.path.join(bd, 'assign_sampling.py'))
    bbox.assign_and_sample, bbox.build_assigner = asn.assign_and_sample, asn.build_assigner
    bbox.PseudoSampler = smp.PseudoSampler
    bbox.bbox2delta = sys.modules['mmdet.core.bbox.transforms'].bbox2delta
    ref_shim._shell('mmdet.core.anchor', os.path.join(md, 'core', 'anchor'))
    at = ref_shim._exec('mmdet.core.anchor.anchor_target', os.path.join(md, 'core', 'anchor', 'anchor_target.py'))
    _ref = types.SimpleNamespace(anchor_target=at.anchor_target, AttrDict=ns.AttrDict)
    return _ref


CASES = cases()


def _flatten(levels, B):
    return torch.cat(levels, dim=0 if B == 1 else 1).reshape(B, -1, *levels[0].shape[(1 if B == 1 else 2):])


def _equal(a, b):
    return a.shape == b.shape and a.dtype == b.dtype and torch.equal(torch.nan_to_num(a, nan=12345.), torch.nan_to_num(
        b, nan=12345.)) and torch.equal(torch.isnan(a) if a.is_floating_point() else a, torch.isnan(b)
                                        if b.is_floating_point() else b)


@pytest.mark.parametrize('case', CASES, ids=[c[0] for c in CASES])
def test_reference_anchor_target_equals_the_oracle(case):
    ref = _reference()
    name, bases, sizes, strides, metas, gts, cfg, means, stds = case
    B = len(gts)
    acfg = ref.AttrDict(assigner=dict(cfg['assigner']), sampler=dict(cfg['sampler']),
                        allowed_border=cfg['allowed_border'], pos_weight=cfg['pos_weight'])
    anchor_list, flag_list = [], []
    for m in metas:
        per_a, per_f = [], []
        for base, (H, W), s in zip(bases, sizes, strides):
            per_a.append(O.grid_anchors(base, H, W, s, 'cpu'))
            per_f.append(O.valid_flags(H, W, base.shape[0], min(int(np.ceil(m['pad_shape'][0] / s)), H),
                                       min(int(np.ceil(m['pad_shape'][1] / s)), W), 'cpu'))
        anchor_list.append(per_a)
        flag_list.append(per_f)
    np.random.seed(17)
    want = ref.anchor_target(anchor_list, flag_list, [g.clone() for g in gts], metas, means, stds, acfg)
    np.random.seed(17)
    got = O.anchor_target(bases, sizes, strides, gts, metas, means, stds, cfg, O.numpy_shuffle, 'cpu')
    assert want is not None and got is not None
    (labels, lw, bt, bw), (npos, nneg) = got
    for i, mine in enumerate((labels, lw, bt, bw)):
        assert _equal(_flatten(want[i], B), mine), (name, i)
    assert (want[4], want[5]) == (npos, nneg), name
    if name.startswith('iou_edge'):   # anchor 0 sits at the threshold: positive from float32(0.7) up, negative below 0.3
        want_edge = [(0, 0.), (1, 1.), (1, 1.), (0, 1.), (0, 0.), (0, 0.)][int(name[-1])]
        assert (labels[0, 0].item(), lw[0, 0].item()) == want_edge, name


def test_crafted_ious_sit_at_the_thresholds():
    a0 = EDGE_BASE[0][None]
    ious = [O.bbox_overlaps(g[None], a0)[0, 0].item() for g in edge_gts()]
    for t, got in ((0.7, ious[:3]), (0.3, ious[3:])):
        t32 = np.float32(t)
        assert got == [float(np.nextafter(t32, np.float32(0))), float(t32), float(np.nextafter(t32, np.float32(1)))]
    # torch compares with python floats in fp32: float32(0.7) counts as >= 0.7 and float32(0.3) is not < 0.3
    assert bool(torch.tensor([ious[1]]) >= 0.7) and not bool(torch.tensor([ious[4]]) < 0.3)


def test_the_cpu_route_above_50_gts_equals_the_device_route_on_the_cpu():
    gen = torch.Generator().manual_seed(3)
    anchors = O.grid_anchors(_head_bases()[0], 16, 24, 4, 'cpu')
    gts = _boxes(gen, 80, 90, 60, 2, 40)
    a = dict(RPN_CFG['assigner'])
    assert torch.equal(O.assign(anchors, gts, a), O.assign(anchors, gts, dict(a, cpu_above=None)))


# ------------------------------------------------------------------------------------------------- the head's host side
def test_inside_anchor_decision_matches_the_flags():
    head = build_from_cfg(dict(RPN_DICT, anchor_strides=[4, 8, 16]), HEADS)
    sizes = [(16, 24), (8, 12), (4, 6)]
    bases = [g.base_anchors for g in head.anchor_generators]
    shapes = [((60, 90, 3), (64, 96, 3)), ((1, 1, 3), (4, 4, 3)), ((8, 8, 3), (8, 8, 3)), ((20, 20, 3), (0, 0, 3)),
              ((30, 30, 3), (32, 32, 3)), ((2, 300, 3), (4, 320, 3))]
    for (img, pad) in shapes:
        meta = dict(img_shape=img, pad_shape=pad)
        anchors, valid = O.multi_level(bases, sizes, [4, 8, 16], pad, 'cpu')
        for ab in (-1, 0, 3, 16):
            want = bool(O.inside_flags(anchors, valid, img, ab).any())
            assert head._has_inside_anchor(sizes, meta, ab) == want, (img, pad, ab)


def _train_cfgs():
    root = ref_shim.reference_dir()
    found = []
    for path in sorted(glob.glob(os.path.join(root or '/nonexistent', 'configs', '**', '*.py'), recursive=True)):
        try:
            tc = runpy.run_path(path).get('train_cfg')
        except Exception:
            continue
        if isinstance(tc, dict) and isinstance(tc.get('rpn'), dict):
            found.append((os.path.relpath(path, root), tc['rpn']))
    return found


def test_every_config_train_cfg_rpn_takes_the_native_route():
    found = _train_cfgs()
    if not found:
        pytest.skip('no reference checkout')
    assert len(found) >= 10
    head = build_from_cfg(dict(RPN_DICT), HEADS)
    cuda = types.SimpleNamespace(is_cuda=True, numel=lambda: 0)
    for path, rpn in found:
        assert head._targets_unsupported(rpn, [cuda] * 5, [cuda, cuda], None, 2) is None, path


@pytest.mark.parametrize('setting', ['focal', 'assigner', 'sampler', 'add_gt', 'ignore', 'cpu'])
def test_settings_without_a_native_route_raise_naming_them(setting, monkeypatch):
    from balancedgroupsoftmax_b200 import rpn_head
    monkeypatch.setattr(rpn_head, '_mmdet_core', lambda name: None)
    d = dict(RPN_DICT, anchor_strides=[4])
    cfg = _cfg()
    cuda = types.SimpleNamespace(is_cuda=True, numel=lambda: 3)
    ignore = None
    if setting == 'focal':
        d['loss_cls'] = dict(type='FocalLoss', use_sigmoid=True, gamma=2.0, alpha=0.25, loss_weight=1.0)
    elif setting == 'assigner':
        cfg['assigner']['type'] = 'ApproxMaxIoUAssigner'
    elif setting == 'sampler':
        cfg['sampler']['type'] = 'OHEMSampler'
    elif setting == 'add_gt':
        cfg['sampler']['add_gt_as_proposals'] = True
    elif setting == 'ignore':
        cfg['assigner']['ignore_iof_thr'] = 0.5
        ignore = [cuda]
    head = build_from_cfg(d, HEADS)
    match = {'focal': 'sampling=False', 'assigner': 'ApproxMaxIoUAssigner', 'sampler': 'OHEMSampler',
             'add_gt': 'add_gt_as_proposals', 'ignore': 'ignore_iof_thr', 'cpu': 'CPU tensors'}[setting]
    if setting != 'cpu':
        assert match in head._targets_unsupported(cfg, [cuda], [cuda], ignore, 1)
    with pytest.raises(NotImplementedError, match=match):
        head.loss([torch.zeros(1, 3, 4, 4)], [torch.zeros(1, 12, 4, 4)], [torch.zeros(1, 4)],
                  [dict(img_shape=(16, 16, 3), pad_shape=(16, 16, 3))], cfg, gt_bboxes_ignore=ignore)


# ------------------------------------------------------------------------------------ the selection rule's statistics
def _inclusion(seeds, img, flat, k):
    hits = np.zeros(len(flat))
    pos = {f: i for i, f in enumerate(flat.tolist())}
    for s in seeds:
        for f in O.native_select(s, img, flat, k).tolist():
            hits[pos[f]] += 1
    return hits


def test_selection_is_exact_k_and_uniform():
    flat = np.sort(np.random.RandomState(0).choice(268569, 400, replace=False))
    k, R = 40, 3000
    seeds = [S.effective_seed(0x1234, r) for r in range(R)]
    for s in seeds[:50]:
        chosen = O.native_select(s, 1, flat, k)
        assert len(set(chosen.tolist())) == k and set(chosen.tolist()) <= set(flat.tolist())
    hits = _inclusion(seeds, 1, flat, k)
    p = k / len(flat)
    z = (hits - R * p) / np.sqrt(R * p * (1 - p))
    assert np.abs(z).max() < 5, np.abs(z).max()
    chi = (z ** 2).sum()   # chi-square with n - 1 degrees of freedom, within 5 sigma
    n = len(flat)
    assert abs(chi - (n - 1)) < 5 * np.sqrt(2 * (n - 1)), chi


@pytest.mark.parametrize('pair', ['images', 'seeds', 'high_word', 'steps'])
def test_selection_is_independent(pair):
    """The overlap of two draws of k of n is hypergeometric (mean k^2 / n) when they are independent: summed over R
    trials, within 5 sigma."""
    flat = np.arange(0, 3000, 7)
    n, k, R = len(flat), 60, 1500
    total = 0
    for r in range(R):
        s = (0x9E3779B97F4A7C15 * (r + 1)) & S.MASK64
        if pair == 'images':
            a, b = O.native_select(s, 0, flat, k), O.native_select(s, 1, flat, k)
        elif pair == 'seeds':
            a, b = O.native_select(s, 0, flat, k), O.native_select((s + 1) & S.MASK64, 0, flat, k)
        elif pair == 'high_word':
            a, b = O.native_select(s, 0, flat, k), O.native_select(s ^ (1 << 40), 0, flat, k)
        else:
            a, b = O.native_select(S.effective_seed(s, r), 0, flat, k), \
                O.native_select(S.effective_seed(s, r + 1), 0, flat, k)
        total += len(np.intersect1d(a, b))
    mean = k * k / n
    var = k * (k / n) * ((n - k) / n) * ((n - k) / (n - 1))
    assert abs(total - R * mean) < 5 * np.sqrt(R * var), (total, R * mean)


def test_sixty_four_bit_keys_are_distinct():
    """The index in the key's low half makes the keys distinct by construction.  The hash half alone already is for
    one (seed, image): sample_key's last step, mix32(h ^ n), is a bijection of n, so it has no collision to break."""
    flat = np.arange(268569)
    for seed in (7, (1 << 63) + 5):
        h = S.keys(seed, 1, flat)
        key = (h.astype(np.uint64) << np.uint64(32)) | flat.astype(np.uint64)
        assert len(np.unique(key)) == len(flat) and len(np.unique(h)) == len(flat)


# ----------------------------------------------------------------------------------------- the C ABI's rules
def _levels(*rows):
    return np.ascontiguousarray(np.array(rows, dtype=np.int32).reshape(-1, 4))


def _abi_call(levels=None, L=None, B=1, images=None, total=1, num=256, pos_fraction=0.5, scratch_bytes=1 << 30,
              outs=True, gts_off=0, ab=0.0):
    lib = nat.lib()
    levels = _levels((16, 16, 3, 4)) if levels is None else levels
    L = levels.shape[0] if L is None else L
    buf = (C.c_char * 4096)()
    base = (C.addressof(buf) + 255) // 256 * 256
    anchors = (C.c_float * (4 * 16 * 8))()
    cols = 4 + 2 * max(L, 1)
    if images is None:
        images = [64, 64, 0, 1] + [4, 4] * max(L, 1)
        images = images * B
    img = nat.int32_array(images[:cols * B] if len(images) >= cols * B else images + [0] * (cols * B - len(images)))
    ms = (C.c_float * 4)(0, 0, 0, 0)
    sd = (C.c_float * 4)(1, 1, 1, 1)
    o = base if outs else None
    return lib.bags_anchor_target(levels.ctypes.data, anchors, L, B, img, base + gts_off, total, 0.7, 1, 0.0, 0.3,
                                  0.3, 1, ab, num, pos_fraction, -1.0, -1.0, ms, sd, 1, None, base, scratch_bytes,
                                  o, o, o, o, o, None)


def test_anchor_target_abi_rejects_bad_arguments():
    lib = nat.lib()
    bad = [dict(L=0), dict(L=9), dict(B=0), dict(B=33), dict(levels=_levels((16, 16, 17, 4))),
           dict(levels=_levels((16, 16, 0, 4))), dict(levels=_levels((-1, 16, 3, 4))),
           dict(levels=_levels((16, 16, 3, 0))), dict(levels=_levels((0, 16, 3, 4))),
           dict(images=[64, 64, 0, 0, 4, 4]), dict(images=[64, 64, 1, 1, 4, 4], total=2),
           dict(images=[0, 64, 0, 1, 4, 4]), dict(images=[64, 64, 0, 1, 17, 4]), dict(images=[64, 64, 0, 1, 4, -1]),
           dict(total=2), dict(B=2, total=1), dict(num=-1), dict(pos_fraction=1.5), dict(pos_fraction=-0.1),
           dict(scratch_bytes=16), dict(outs=False), dict(gts_off=4), dict(ab=float('nan'))]
    for kw in bad:
        assert _abi_call(**kw) == -1, kw
        assert b'bags_anchor_target' in lib.bags_last_error(), (kw, lib.bags_last_error())


def test_anchor_target_scratch_bytes():
    lib = nat.lib()
    lv = _levels((200, 336, 3, 4), (100, 168, 3, 8), (50, 84, 3, 16), (25, 42, 3, 32), (13, 21, 3, 64))
    out = C.c_size_t(0)
    assert lib.bags_anchor_target_scratch_bytes(lv.ctypes.data, 5, 2, 600, C.byref(out)) == 0
    r = lambda x: (x + 255) // 256 * 256   # noqa: E731
    N = 3 * (200 * 336 + 100 * 168 + 50 * 84 + 25 * 42 + 13 * 21)
    assert N == 268569
    assert out.value == r(2 * 2 * 4) + r(600 * 8) + r(2 * 4 * 8) + r(2 * N * 4)
    assert lib.bags_anchor_target_scratch_bytes(lv.ctypes.data, 5, 2, 1, C.byref(out)) == -1   # fewer gts than images
    assert lib.bags_anchor_target_scratch_bytes(lv.ctypes.data, 5, 2, 600, None) == -1
