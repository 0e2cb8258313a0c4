"""BAGS group tables: label2binlabel / pred_slice / fg_splits.

The reference generates these once from ``lvis_v0.5_train.json`` with
``tools/lvis_analyse.py:get_cate_gs`` (:11-58) and ``get_split`` (:60-98) and
ships them as ``label2binlabel.pt``, ``pred_slice_with0.pt`` and
``valsplit.pkl``.  The annotation file is not available offline, so this module
restates the same algorithm over an arbitrary ``{category_id: instance_count}``
mapping (iteration order = category order, as ``lvis_train.cats`` gives it) and
can synthesise a long-tailed count vector for benchmarks and tests.

Semantics kept bit-exact (integer tables):
  * row 0 of label2binlabel is [0, 1, 1, ..., 1]           (lvis_analyse.py:20)
  * row g>=1 holds the 1-based index of category cid inside bin g, else 0
    ("others")                                             (:23-36)
  * bins by instance count: <10, <100, <1000, >=1000       (:24-36)
  * pred_slice rows are running (start, count), counts 2, n_1+1, ...  (:45-50)
  * fg_splits[g-1] lists the category ids of bin g in iteration order (:76-91)
"""
from __future__ import annotations

import os
import pickle
from dataclasses import dataclass
from typing import Dict, List, Mapping, Sequence

import numpy as np

DEFAULT_THRESHOLDS = (10, 100, 1000)
# keys the reference head hard-codes (gs_bbox_head_with0.py:46-49)
SPLIT_KEYS_5BIN = ('(0, 10)', '[10, 100)', '[100, 1000)', '[1000, ~)')


@dataclass
class GroupTables:
    label2binlabel: np.ndarray      # [G, num_classes] int64
    pred_slice: np.ndarray          # [G, 2] int64 (start, len)
    fg_splits: List[np.ndarray]     # G-1 arrays of category ids, int64

    @property
    def num_bins(self) -> int:
        return int(self.label2binlabel.shape[0])

    @property
    def num_classes(self) -> int:
        return int(self.label2binlabel.shape[1])

    @property
    def num_logits(self) -> int:
        return int(self.pred_slice[:, 1].sum())

    def cls2col(self) -> np.ndarray:
        """Logit column feeding each merged class score (-1: none).

        Restates the scatter of ``_merge_score`` (gs_bbox_head_with0.py:260-268):
        class 0 <- column start_0; class fg_splits[g-1][j-1] <- column start_g + j.
        """
        out = np.full((self.num_classes,), -1, dtype=np.int32)
        out[0] = int(self.pred_slice[0, 0])
        for g in range(1, self.num_bins):
            start = int(self.pred_slice[g, 0])
            split = self.fg_splits[g - 1]
            for j, cid in enumerate(split.tolist(), start=1):
                if cid >= 1:  # merge[:, 1:] = fg_merge[:, 1:] drops class 0
                    out[cid] = start + j
        return out


def build_group_tables(instance_counts: Mapping[int, int], num_classes: int = 1231,
                       thresholds: Sequence[int] = DEFAULT_THRESHOLDS) -> GroupTables:
    """Restatement of get_cate_gs + get_split for len(thresholds)+2 bins."""
    num_bins = len(thresholds) + 2
    binlabel_count = [1] * num_bins
    label2binlabel = np.zeros((num_bins, num_classes), dtype=np.int64)
    label2binlabel[0, 1:] = binlabel_count[0]
    binlabel_count[0] += 1
    splits: List[List[int]] = [[] for _ in range(num_bins - 1)]
    for cid, ins_count in instance_counts.items():
        b = len(thresholds)
        for i, thr in enumerate(thresholds):
            if ins_count < thr:
                b = i
                break
        g = b + 1
        label2binlabel[g, cid] = binlabel_count[g]
        binlabel_count[g] += 1
        splits[b].append(cid)
    pred_slice = np.zeros((num_bins, 2), dtype=np.int64)
    start = 0
    for i, c in enumerate(binlabel_count):
        pred_slice[i, 0] = start
        pred_slice[i, 1] = c
        start += c
    return GroupTables(label2binlabel, pred_slice, [np.array(s, dtype=np.int64) for s in splits])


def synthetic_instance_counts(num_fg: int = 1230, seed: int = 0, lo: float = 1.0,
                              hi: float = 3.0e4) -> Dict[int, int]:
    """Seeded long-tailed (log-uniform) per-category training instance counts."""
    rng = np.random.RandomState(seed)
    counts = np.exp(rng.uniform(np.log(lo), np.log(hi), size=num_fg)).astype(np.int64)
    counts = np.maximum(counts, 1)
    return {cid: int(c) for cid, c in zip(range(1, num_fg + 1), counts)}


def synthetic_tables(num_classes: int = 1231, seed: int = 0) -> GroupTables:
    return build_group_tables(synthetic_instance_counts(num_classes - 1, seed), num_classes)


def save_reference_files(tables: GroupTables, directory: str) -> Dict[str, str]:
    """Write the three files in the reference's on-disk formats
    (torch.save'd int64 tensors + pickled dict keyed like valsplit.pkl)."""
    import torch
    os.makedirs(directory, exist_ok=True)
    paths = {
        'label2binlabel': os.path.join(directory, 'label2binlabel.pt'),
        'pred_slice': os.path.join(directory, 'pred_slice_with0.pt'),
        'fg_split': os.path.join(directory, 'valsplit.pkl'),
    }
    torch.save(torch.from_numpy(tables.label2binlabel), paths['label2binlabel'])
    torch.save(torch.from_numpy(tables.pred_slice), paths['pred_slice'])
    splits = {}
    if tables.num_bins == 5:
        for k, s in zip(SPLIT_KEYS_5BIN, tables.fg_splits):
            splits[k] = s
    else:
        for i, s in enumerate(tables.fg_splits):
            splits['bin%d' % (i + 1)] = s
    splits['normal'] = np.arange(1, tables.num_classes)
    splits['background'] = np.zeros((1,), dtype=np.int64)
    splits['all'] = np.arange(tables.num_classes)
    with open(paths['fg_split'], 'wb') as f:
        pickle.dump(splits, f)
    return paths


def load_reference_files(label2binlabel: str, pred_slice: str, fg_split: str) -> GroupTables:
    """Load the reference's files (gs_bbox_head_with0.py:37-49)."""
    import torch
    l2b = torch.load(label2binlabel, map_location='cpu')
    ps = torch.load(pred_slice, map_location='cpu')
    l2b = np.asarray(l2b, dtype=np.int64)
    ps = np.asarray(ps, dtype=np.int64)
    with open(fg_split, 'rb') as f:
        split = pickle.load(f)
    num_bins = l2b.shape[0]
    if all(k in split for k in SPLIT_KEYS_5BIN) and num_bins == 5:
        fg = [np.asarray(split[k], dtype=np.int64) for k in SPLIT_KEYS_5BIN]
    else:
        fg = [np.asarray(split['bin%d' % (i + 1)], dtype=np.int64) for i in range(num_bins - 1)]
    return GroupTables(l2b, ps, fg)


def instance_counts_from_annotations(ann_file: str) -> Dict[int, int]:
    """Per-category training instance counts from an LVIS-style annotation json: what ``LVIS(ann).cats`` gives
    tools/lvis_analyse.py:13-15 (``categories[*].id`` -> ``categories[*].instance_count``), in file order (the
    reference iterates the dict in insertion order, and local bin indices follow that order, :23-36).  When a
    category carries no ``instance_count`` the annotations are counted instead."""
    import json
    with open(ann_file) as f:
        data = json.load(f)
    cats = data['categories']
    if all('instance_count' in c for c in cats):
        return {int(c['id']): int(c['instance_count']) for c in cats}
    counts = {int(c['id']): 0 for c in cats}
    for a in data.get('annotations', []):
        counts[int(a['category_id'])] += 1
    return counts


CLS_WEIGHT_FILES = {'inv': 'cls_weight.pt', 'bf': 'cls_weight_bf.pt', 'bours': 'cls_weight_bours.pt'}


def class_weights(instance_counts: Mapping[int, int], num_classes: int = 1231, kind: str = 'inv') -> np.ndarray:
    """Per-class loss weights of ReweightBBoxHead, float64 [num_classes] (index 0 = background), restating
    tools/lvis_analyse.py with its quirks:

      'inv'   get_cate_weight (:338-365): 1 / count with the background count set to 1, divided by the foreground
              mean, background weight 1, clipped to [0.1, 5]                                  -> cls_weight.pt
      'bf'    get_cate_weight_bf (:370-405): class-balanced (1 - beta) / (1 - beta^count), beta = 0.999, with the
              background count 3 x the foreground total, divided by the mean over all classes, not clipped
                                                                                              -> cls_weight_bf.pt
      'bours' get_cate_weight_bours (:409-445): class-balanced weights of the foreground only, divided by their mean,
              background weight 1, clipped to [0.1, 5]                                        -> cls_weight_bours.pt

    A category with no instance gets an infinite raw weight, as in the reference (clipped to 5 where it clips)."""
    counts = np.zeros((num_classes,), dtype=np.float64)
    for cid, c in instance_counts.items():
        counts[cid] = c
    beta = 0.999
    with np.errstate(divide='ignore', invalid='ignore'):
        if kind == 'inv':
            counts[0] = 1
            weight = np.ones_like(counts) / counts
            weight = weight / weight[1:].mean()
            weight[0] = 1
        elif kind == 'bf':
            counts[0] = np.sum(counts[1:]) * 3
            tmp = np.ones_like(counts)
            weight = (tmp - beta) / (tmp - np.power(beta, counts))
            return weight / np.mean(weight)
        elif kind == 'bours':
            fg = counts[1:]
            tmp = np.ones_like(fg)
            w = (tmp - beta) / (tmp - np.power(beta, fg))
            weight = np.ones((num_classes,), dtype=np.float64)
            weight[1:] = w / np.mean(w)
        else:
            raise ValueError('unknown class-weight kind %r (inv, bf, bours)' % (kind,))
    weight = np.where(weight > 5, 5, weight)
    return np.where(weight < 0.1, 0.1, weight)


def save_class_weights(weight: np.ndarray, directory: str, kind: str) -> str:
    """torch.save the float64 weight tensor under the file name the reference's configs load."""
    import torch
    os.makedirs(directory, exist_ok=True)
    path = os.path.join(directory, CLS_WEIGHT_FILES[kind])
    torch.save(torch.from_numpy(np.asarray(weight, dtype=np.float64)), path)
    return path


def main(argv=None) -> int:
    """python -m balancedgroupsoftmax_b200.tables --ann lvis_v0.5_train.json --out data/lvis
    Writes label2binlabel.pt, pred_slice_with0.pt and valsplit.pkl in the reference's formats
    (tools/lvis_analyse.py: get_cate_gs + get_split; --thresholds generalises the 5-bin split).
    With --cls-weight it writes the class-weight files of the re-weighting baselines instead
    (get_cate_weight / _bf / _bours: cls_weight.pt, cls_weight_bf.pt, cls_weight_bours.pt)."""
    import argparse
    ap = argparse.ArgumentParser(description=main.__doc__)
    ap.add_argument('--ann', help='LVIS-style training annotation json (categories with instance_count)')
    ap.add_argument('--synthetic', type=int, default=None, metavar='SEED',
                    help='no annotation file: seeded long-tailed synthetic counts')
    ap.add_argument('--num-classes', type=int, default=None, help='labels incl. background (default: max id + 1)')
    ap.add_argument('--thresholds', type=int, nargs='+', default=list(DEFAULT_THRESHOLDS))
    ap.add_argument('--cls-weight', nargs='+', choices=sorted(CLS_WEIGHT_FILES), default=None,
                    help='write the per-class weight file(s) of ReweightBBoxHead instead of the group tables')
    ap.add_argument('--out', required=True)
    args = ap.parse_args(argv)
    if args.ann:
        counts = instance_counts_from_annotations(args.ann)
    elif args.synthetic is not None:
        counts = synthetic_instance_counts((args.num_classes or 1231) - 1, args.synthetic)
    else:
        ap.error('give --ann or --synthetic')
    num_classes = args.num_classes or (max(counts) + 1)
    if args.cls_weight:
        for kind in args.cls_weight:
            w = class_weights(counts, num_classes, kind)
            path = save_class_weights(w, args.out, kind)
            print('%s: min %.4g max %.4g -> %s' % (kind, float(w.min()), float(w.max()), path))
        return 0
    tables = build_group_tables(counts, num_classes, args.thresholds)
    paths = save_reference_files(tables, args.out)
    print('bins: %s' % ', '.join('%d+1' % len(s) if i else '2' for i, s in enumerate([None] + tables.fg_splits)))
    print('pred_slice:', tables.pred_slice.tolist())
    for k, v in paths.items():
        print('%s -> %s' % (k, v))
    return 0


if __name__ == '__main__':
    raise SystemExit(main())
