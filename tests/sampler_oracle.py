"""Plain numpy restatement of the loss-weight stage -- the device "others" sampler (sample_others_kernel), the reweight
head's per-class weights (reweight_kernel) and the mask normaliser (mask_avg_kernel) -- TEST INFRASTRUCTURE, NOT
PRODUCT CODE.

``sample`` replaces the reference's GSBBoxHeadWith0._sample_others / _remap_labels (gs_bbox_head_with0.py:63-112)
with the device sampler's own deterministic rule, so that a GPU test can compare the kernel's masks byte for byte:

  * bin 0 is all ones, avg_0 = max(N, 1);
  * row n is in bin g >= 1 when 0 <= labels[n] < classes and label2bin[g, labels[n]] > 0; every other row is an
    "other"; F = #in-bin rows, O = N - F, k = int(F * ratio) in float64;
  * F == 0: all zeros, avg 1; k >= O: all ones, avg max(N, 1); k == 0: the in-bin rows only; otherwise the in-bin
    rows plus the k others with the smallest sample_key(seed, g, n); avg_g = max(F + min(k, O), 1).

Where it deliberately differs from the reference:
  * the k others are not np.random.choice's draw but the k smallest counter-based keys (a uniform k-subset for a
    random seed: tests/test_sampler_cpu.py checks it statistically);
  * a label outside [0, classes) is an "other" (the reference would index its table with it);
  * an infinite or huge ratio means "all others" (the reference's int(F * inf) raises).
For a fixed (seed, g) the keys of distinct rows are distinct (the last step, mix32(h ^ n), is a bijection of uint32),
so "the k smallest keys" needs no tie-break.
"""
from __future__ import annotations

import math

import numpy as np

U32 = np.uint32
MASK64 = (1 << 64) - 1
STEP_MUL = 0x9E3779B97F4A7C15      # the seed_step multiplier (odd: the step -> seed map is a bijection mod 2^64)


def mix32(x):
    """murmur3's 32-bit finaliser, elementwise on uint32."""
    x = np.array(x, dtype=np.uint32, copy=True)
    with np.errstate(over='ignore'):
        x ^= x >> U32(16)
        x *= U32(0x85EBCA6B)
        x ^= x >> U32(13)
        x *= U32(0xC2B2AE35)
        x ^= x >> U32(16)
    return x


def keys(seed, g, n):
    """sample_key(seed, g, n) of the kernel for every row in ``n`` (uint32 array); ``seed`` is taken mod 2^64."""
    seed = int(seed) & MASK64
    h = mix32((seed & 0xFFFFFFFF) ^ 0x9E3779B9)
    h = mix32(h ^ U32(seed >> 32))
    h = mix32(h ^ U32((int(g) * 0x632BE5AB + 0x7F4A7C15) & 0xFFFFFFFF))
    return mix32(h ^ np.asarray(n, dtype=np.int64).astype(np.uint32))


def effective_seed(seed, step):
    """The seed the kernel uses with a device step counter: seed + step * 0x9E3779B97F4A7C15 mod 2^64, with the
    int64 step read as an unsigned 64-bit value (-1 wraps to 2^64 - 1)."""
    if step is None:
        return int(seed) & MASK64
    return (int(seed) + (int(step) & MASK64) * STEP_MUL) & MASK64


def in_bin(labels, label2bin, g):
    """[N] bool: 0 <= label < classes and label2bin[g, label] > 0."""
    labels = np.asarray(labels, dtype=np.int64)
    table = np.asarray(label2bin)
    classes = table.shape[1]
    ok = (labels >= 0) & (labels < classes)
    out = np.zeros(labels.shape, dtype=bool)
    out[ok] = table[g, labels[ok]] > 0
    return out


def count_k(F, ratio, O):
    """k = int(F * ratio) in float64, saturated at O (an infinite or huge product means "all others")."""
    x = float(F) * float(ratio)
    if math.isnan(x):
        raise ValueError('NaN sample count')
    if not math.isfinite(x) or x >= O:
        return O
    return int(x)


def bin_counts(labels, label2bin, ratio, g):
    """(F, O, k, mode) of bin g >= 1; mode 0 zeros, 1 ones, 2 in-bin only, 3 in-bin plus k sampled others."""
    fg = in_bin(labels, label2bin, g)
    N = fg.size
    F = int(fg.sum())
    O = N - F
    if F == 0:                                  # before k: 0 * inf is NaN
        return F, O, 0, 0
    k = count_k(F, ratio, O)
    if k >= O:
        return F, O, O, 1
    if k == 0:
        return F, O, 0, 2
    return F, O, k, 3


def sample(labels, label2bin, ratio, seed, step=None):
    """(wmask [G, N] uint8, avg [G] float32) of the device sampler; ``step`` is the device step counter (None: the
    seed as given)."""
    labels = np.asarray(labels, dtype=np.int64).reshape(-1)
    table = np.asarray(label2bin)
    G, N = table.shape[0], labels.size
    s = effective_seed(seed, step)
    wmask = np.zeros((G, N), dtype=np.uint8)
    avg = np.zeros(G, dtype=np.float32)
    wmask[0] = 1
    avg[0] = max(N, 1)
    for g in range(1, G):
        fg = in_bin(labels, table, g)
        F, O, k, mode = bin_counts(labels, table, ratio, g)
        if mode == 0:
            avg[g] = 1.0
            continue
        if mode == 1:
            wmask[g] = 1
            avg[g] = max(N, 1)
            continue
        wmask[g, fg] = 1
        if mode == 3:
            others = np.nonzero(~fg)[0]
            kk = keys(s, g, others)
            wmask[g, others[np.argpartition(kk, k - 1)[:k]]] = 1
        avg[g] = max(F + k, 1)
    return wmask, avg


def reweight(labels, label2bin, wmask, table):
    """(wfloat [G, N], avg [G]) in float64 of the reweight head's weights: w[g, n] = wmask[g, n] (its byte value;
    1 where ``wmask`` is None) times, for g >= 1, table[g, t] with t = label2bin[g, label] for a label in
    [0, classes) and 0 otherwise, and t outside [0, wstride) read as 0 (the "others" weight); avg = max(sum_n w, 1)."""
    labels = np.asarray(labels, dtype=np.int64).reshape(-1)
    l2b = np.asarray(label2bin, dtype=np.int64)
    tab = np.asarray(table, dtype=np.float64)
    G, classes = l2b.shape
    wstride = tab.shape[1]
    N = labels.size
    w = np.ones((G, N)) if wmask is None else np.asarray(wmask, dtype=np.float64).reshape(G, N).copy()
    ok = (labels >= 0) & (labels < classes)
    for g in range(1, G):
        t = np.zeros(N, dtype=np.int64)
        t[ok] = l2b[g, labels[ok]]
        t = np.where((t >= 0) & (t < wstride), t, 0)
        w[g] *= tab[g, t]
    return w, np.maximum(w.sum(1), 1.0)


def mask_avg(wmask):
    """avg [G] = max(sum_n wmask[g, n], 1) as an exact integer (the float32 rounding is the caller's)."""
    w = np.asarray(wmask)
    return np.maximum(w.astype(np.int64).sum(1), 1)
