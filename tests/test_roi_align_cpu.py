"""CPU: the RoIAlign restatement (tests/roi_align_oracle.py) on hand-worked cases, the extractor's construction from
every LVIS config's extractor dict, and the argument rules of bags_roi_align_fwd / _bwd, which are checked before
anything touches a device."""
import ctypes as C
import glob
import os
import runpy

import numpy as np
import pytest
import torch

import roi_align_oracle as R
from balancedgroupsoftmax_b200 import _native as nat
from balancedgroupsoftmax_b200.registry import ROI_EXTRACTORS, build_roi_extractor
from balancedgroupsoftmax_b200.roi_extractor import RoIAlign, SingleRoIExtractor
from oracle import ref_shim

F = np.arange(16, dtype=np.float64).reshape(1, 1, 4, 4)   # F[y, x] = 4 y + x


def _one(roi, out=(1, 1), sample_num=1, scale=1.0, feat=F):
    return R.forward(feat, np.array([roi], dtype=np.float32), out[0], out[1], scale, sample_num)[0, 0]


def test_sample_at_pixel_centre_of_the_grid():
    # x1 = y1 = 0, x2 = y2 = 1: the RoI spans [0, 2), one sample at (1, 1)
    assert _one([0, 0, 0, 1, 1])[0, 0] == F[0, 0, 1, 1]


def test_bilinear_weights():
    # x in [0, 1) -> one sample at 0.5 between columns 0 and 1, y likewise: the mean of the 2 x 2 corner
    assert _one([0, 0, 0, 0, 0])[0, 0] == (0 + 1 + 4 + 5) / 4


@pytest.mark.parametrize('x1,expect', [
    (-2.0, 'col0'),       # sample at exactly -1: inside, clamped to column 0
    (-2.5, 'zero'),       # sample at -1.5: outside
    (-1.0, 'col0'),       # sample at exactly 0
    (2.0, 'col3'),        # sample at exactly W - 1: the last column
    (3.0, 'col3'),        # sample at exactly W: inside, clamped
    (3.5, 'zero'),        # sample at W + 0.5: outside
])
def test_samples_at_the_edges(x1, expect):
    # a RoI two pixels wide (x2 = x1 + 1) has its single x sample at x1 + 1; y sample at 1 (row 1)
    v = _one([0, x1, 0, x1 + 1, 1])[0, 0]
    want = {'col0': F[0, 0, 1, 0], 'col3': F[0, 0, 1, 3], 'zero': 0.0}[expect]
    assert v == want, (x1, v, want)


def test_one_ulp_inside_minus_one_is_kept():
    x = np.float32(-1.0)
    below = np.nextafter(x, np.float32(-2))
    ok, lo, hi, l, h = R.axis_sample(np.float32(-1.0), np.float32(0.0), 0, 0, 1, 4)
    assert ok and (lo, hi, l, h) == (0, 1, 0, 1)
    assert not R.axis_sample(below, np.float32(0.0), 0, 0, 1, 4)[0]


def test_one_pixel_and_one_row_maps():
    one = np.array([[[[7.0]]]])
    assert _one([0, 0, 0, 0, 0], feat=one)[0, 0] == 7.0
    row = np.arange(5, dtype=np.float64).reshape(1, 1, 1, 5)
    # y sample at 0.5 on a single row: lo = hi = 0; x sample at 2.5
    assert _one([0, 2, 0, 2, 0], feat=row)[0, 0] == 2.5


@pytest.mark.parametrize('width', [0.0, -3.0])
def test_zero_and_inverted_widths(width):
    # x2 + 1 - x1 <= 0: the RoI collapses to its start; fixed samples all sit at x1
    x1 = 1.0
    v = _one([0, x1, 0, x1 - 1 + width, 1], out=(1, 2), sample_num=2)
    assert np.all(v == F[0, 0, 1, 1])
    # adaptive: ceil(0) = 0 samples per bin on that axis, and the reference divides 0 by 0
    assert np.all(np.isnan(_one([0, x1, 0, x1 - 1 + width, 1], out=(1, 2), sample_num=0)))


def test_adaptive_sample_counts():
    ys, xs, cnt = R.roi_samples(np.float32([0, 0, 0, 9, 2]), 1.0, 2, 2, 0, 16, 16)
    # roi 10 wide, 3 high over 2 x 2 bins: bins of 5 x 1.5 -> 5 and 2 samples per bin
    assert [len(b) for b in xs] == [5, 5] and [len(b) for b in ys] == [2, 2] and cnt == 10


def test_batch_index_outside_gives_zero_row():
    feat = np.ones((2, 1, 4, 4))
    rois = np.array([[2, 0, 0, 1, 1], [-1, 0, 0, 1, 1], [1, 0, 0, 1, 1]], dtype=np.float32)
    out = R.forward(feat, rois, 2, 2, 1.0, 2)
    assert np.all(out[:2] == 0) and np.allclose(out[2], 1)


def test_backward_is_the_adjoint_of_forward():
    rng = np.random.default_rng(0)
    feat = rng.standard_normal((2, 3, 9, 11))
    rois = np.array([[0, 0.3, 1.2, 6.1, 7.7], [1, -1.5, -0.5, 10.6, 9.0], [1, 4, 4, 4, 4]], dtype=np.float32)
    for sample_num in (0, 2):
        out = R.forward(feat, rois, 3, 2, 1.0, sample_num)
        gout = rng.standard_normal(out.shape)
        grad, absum = R.backward(gout, rois, 1.0, sample_num, feat.shape)
        assert np.isclose((out * gout).sum(), (feat * grad).sum())
        assert np.all(absum >= np.abs(grad))


def test_fma32_rounds_once():
    # a * b + c with a product needing more than fp32's precision
    a, b, c = np.float32(1 + 2 ** -23), np.float32(1 + 2 ** -23), np.float32(-1)
    assert R.fma32(a, b, c) == np.float32(2 ** -22 + 2 ** -46)


# ----------------------------------------------------------------------------------------- the module layer
EXTRACTOR_DICTS = [
    dict(type='SingleRoIExtractor', roi_layer=dict(type='RoIAlign', out_size=7, sample_num=2), out_channels=256,
         featmap_strides=[4, 8, 16, 32]),
    dict(type='SingleRoIExtractor', roi_layer=dict(type='RoIAlign', out_size=14, sample_num=2), out_channels=256,
         featmap_strides=[4, 8, 16, 32]),
    dict(type='SingleRoIExtractor', roi_layer=dict(type='RoIAlign', out_size=14, sample_num=2), out_channels=256,
         featmap_strides=[8]),
]


def _config_dicts():
    """Every *_roi_extractor dict of the reference's configs, where a checkout is reachable."""
    root = ref_shim.reference_dir()
    if root is None:
        return []
    found = []
    for path in sorted(glob.glob(os.path.join(root, 'configs', '**', '*.py'), recursive=True)):
        try:
            model = runpy.run_path(path).get('model')
        except Exception:
            continue
        if isinstance(model, dict):
            for key in ('bbox_roi_extractor', 'mask_roi_extractor', 'semantic_roi_extractor'):
                for d in (model.get(key) if isinstance(model.get(key), list) else [model.get(key)]):
                    if isinstance(d, dict):
                        found.append((os.path.relpath(path, root), key, d))
    return found


def _check_built(d, ext):
    assert isinstance(ext, SingleRoIExtractor)
    assert ext.out_channels == d['out_channels'] and ext.featmap_strides == d['featmap_strides']
    assert ext.finest_scale == d.get('finest_scale', 56) and ext.num_inputs == len(d['featmap_strides'])
    assert ext.fp16_enabled is False
    assert isinstance(ext.roi_layers, torch.nn.ModuleList) and len(ext.roi_layers) == len(d['featmap_strides'])
    size = d['roi_layer']['out_size']
    for layer, s in zip(ext.roi_layers, d['featmap_strides']):
        assert isinstance(layer, RoIAlign)
        assert layer.out_size == (size, size) and layer.spatial_scale == 1 / s
        assert layer.sample_num == d['roi_layer']['sample_num'] and layer.use_torchvision is False
    ext.init_weights()


@pytest.mark.parametrize('d', EXTRACTOR_DICTS, ids=['bbox7', 'mask14', 'semantic14'])
def test_extractor_dicts_build(d):
    assert ROI_EXTRACTORS.get('SingleRoIExtractor') is SingleRoIExtractor
    _check_built(d, build_roi_extractor(dict(d)))


def test_every_reference_config_extractor_builds():
    found = _config_dicts()
    if not found:
        pytest.skip('no reference checkout')
    assert len(found) >= 50
    for path, key, d in found:
        _check_built(d, build_roi_extractor(dict(d)))


def test_roi_layer_repr_and_unknown_type():
    layer = RoIAlign(7, 0.25, 2)
    assert repr(layer) == 'RoIAlign(out_size=(7, 7), spatial_scale=0.25, sample_num=2, use_torchvision=False)'
    with pytest.raises(NotImplementedError, match='RoIPool'):
        SingleRoIExtractor(dict(type='RoIPool', out_size=7), 256, [4, 8])


def test_map_roi_levels_and_rescale():
    ext = SingleRoIExtractor(dict(type='RoIAlign', out_size=7, sample_num=2), 256, [4, 8, 16, 32])
    rois = torch.tensor([[0, 0, 0, 10, 10], [0, 0, 0, 111, 111], [0, 0, 0, 223, 223], [0, 5, 5, 2000, 900],
                         [1, 3, 4, 50.5, 90.25]])
    assert torch.equal(ext.map_roi_levels(rois, 4), R.map_roi_levels(rois, 4, 56))
    assert ext.map_roi_levels(rois, 4).tolist() == [0, 1, 2, 3, 0]
    out = ext.roi_rescale(rois, 1.5)
    w = rois[:, 3] - rois[:, 1] + 1
    assert torch.allclose(out[:, 3] - out[:, 1] + 1, w * 1.5)
    assert torch.equal(out[:, 0], rois[:, 0])
    assert torch.allclose((out[:, 1] + out[:, 3]) / 2, (rois[:, 1] + rois[:, 3]) / 2)


def test_cpu_tensors_raise():
    ext = SingleRoIExtractor(dict(type='RoIAlign', out_size=7, sample_num=2), 8, [4, 8])
    feats = [torch.zeros(1, 8, 16, 16), torch.zeros(1, 8, 8, 8)]
    rois = torch.tensor([[0, 0, 0, 10, 10.]])
    with pytest.raises(nat.BagsNativeError):
        ext(feats, rois)
    with pytest.raises(nat.BagsNativeError):
        ext(feats[:1], rois)
    with pytest.raises(nat.BagsNativeError):
        RoIAlign(7, 0.25, 2)(feats[0], rois)


# ----------------------------------------------------------------------------------------- the C ABI's rules
def _abi_call(bwd=False, L=2, B=1, Cc=4, k=1, oh=7, ow=7, sample_num=2, finest=56.0, sizes=(8, 8, 4, 4),
              bufs=True, rois=True, out=True, misalign=0):
    lib = nat.lib()
    buf = (C.c_char * 4096)()
    base = (C.addressof(buf) + 15) // 16 * 16
    ptrs = (C.c_void_p * max(L, 1))(*([base + misalign if bufs else None] * max(L, 1)))
    sz = nat.int32_array(list(sizes) + [1] * max(0, 2 * L - len(sizes)))
    sc = (C.c_float * max(L, 1))(*([0.25] * max(L, 1)))
    r = base if rois else None
    o = base if out else None
    if bwd:
        return lib.bags_roi_align_bwd(o, ptrs, sz, sc, L, B, Cc, r, r, k, oh, ow, sample_num, finest, None)
    return lib.bags_roi_align_fwd(ptrs, sz, sc, L, B, Cc, r, r, k, oh, ow, sample_num, finest, o, None, None)


@pytest.mark.parametrize('bwd', [False, True], ids=['fwd', 'bwd'])
def test_roi_align_abi_rejects_bad_arguments(bwd):
    lib = nat.lib()
    who = b'bags_roi_align_bwd' if bwd else b'bags_roi_align_fwd'
    bad = [dict(L=0), dict(L=9), dict(B=0), dict(Cc=0), dict(k=-1), dict(oh=0), dict(ow=65), dict(finest=0.0),
           dict(finest=float('inf')), dict(sizes=(0, 8, 4, 4)), dict(sizes=(8, 8, 4, 0)), dict(rois=False),
           dict(out=False), dict(misalign=2)]
    if not bwd:
        bad.append(dict(bufs=False))
    for kw in bad:
        assert _abi_call(bwd=bwd, **kw) == -1, kw
        assert who in lib.bags_last_error(), (kw, lib.bags_last_error())
    # nothing to do: no device needed
    assert _abi_call(bwd=bwd, k=0, rois=False, out=False) == 0
    if bwd:
        assert _abi_call(bwd=True, bufs=False) == 0   # no level takes a gradient
