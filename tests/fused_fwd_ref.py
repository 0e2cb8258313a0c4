"""Float64 references of the fused fc_cls forward (bags_fwd's fused route, bags_ce_fwd, bags_focal_fwd) -- TEST
INFRASTRUCTURE, NOT PRODUCT CODE.

Plain torch on whatever device the inputs live on, never this library.  tests/test_gpu_fused_fwd_vs_float64.py
bounds the kernels against these functions; tests/test_fused_fwd_ref_cpu.py checks them against
oracle/bags_oracle.py and tests/reweight_oracle.py, so that the GPU tests do not rest on an unchecked reference.
The focal loss's per-element reference is tests/focal_oracle.py.
"""
from __future__ import annotations

import math

import torch

U = 2.0 ** -24   # unit roundoff of fp32
LOG_FLT_MIN = math.log(2.0 ** -126)


def bin_targets(labels, l2b, slices, classes):
    """In-bin target column of every (bin, row), [G, N] int64, as the fused kernel scores it (the rule of
    bags_group_ce): l2b[g, label] (the label itself when ``l2b`` is None), and in-bin column 0 where the label lies
    outside [0, classes) or the table entry outside [0, len_g)."""
    lab_ok = (labels >= 0) & (labels < classes)
    labc = labels.clamp(0, classes - 1)
    out = []
    for g, (_, ln) in enumerate(slices):
        t = l2b[g].long()[labc] if l2b is not None else labc
        t = torch.where(lab_ok, t, torch.zeros_like(t))
        out.append(torch.where((t >= 0) & (t < ln), t, torch.zeros_like(t)))
    return torch.stack(out)


def softmax_ce(z, slices, targets, coef):
    """The grouped softmax CE of exact logits z [N, C] (float64) over bins ``slices`` [(start, len)], with in-bin
    targets [G, N] and coef [G, N] = w / avg.  Returns
      dz [N, C]        coef * (softmax - onehot) per bin, 0 in columns outside every bin
      lse [N, G]       logsumexp of each bin
      loss [G]         sum_n coef * (lse - z[target])
      coef_col [N, C]  coef of each column's bin (0 outside every bin)
      terms [N, G]     |coef * (lse - z[target])|, the loss's addends."""
    N, C = z.shape
    G = len(slices)
    dz = torch.zeros(N, C, dtype=torch.float64, device=z.device)
    coef_col = torch.zeros_like(dz)
    lse = torch.empty(N, G, dtype=torch.float64, device=z.device)
    terms = torch.empty_like(lse)
    loss = torch.empty(G, dtype=torch.float64, device=z.device)
    for g, (s, ln) in enumerate(slices):
        zs = z[:, s:s + ln]
        lse[:, g] = torch.logsumexp(zs, 1)
        t = targets[g]
        term = coef[g] * (lse[:, g] - zs.gather(1, t[:, None])[:, 0])
        loss[g] = term.sum()
        terms[:, g] = term.abs()
        onehot = torch.nn.functional.one_hot(t, ln).to(torch.float64)
        dz[:, s:s + ln] = coef[g][:, None] * (torch.softmax(zs, 1) - onehot)
        coef_col[:, s:s + ln] = coef[g][:, None]
    return dz, lse, loss, coef_col, terms


def top1_count(z, labels):
    """#{n : 0 <= labels[n] < C and z[n, labels[n]] == max_c z[n, c]}: mmdet's top-1 accuracy count, with a tie with
    the row maximum counted as correct (exact logits make ties exact)."""
    C = z.shape[1]
    ok = (labels >= 0) & (labels < C)
    zl = z.gather(1, labels.clamp(0, C - 1)[:, None])[:, 0]
    return int((ok & (zl == z.max(1).values)).sum())


def colsum_fp32(dz_stored, N):
    """Per-128-row-tile column sums [ceil(N/128), C] as the kernel forms them: the stored dz values (rows [0, N)) in
    fp32, added in row order to 0.0, one fp32 addition per row; rows >= N of the last tile add 0."""
    tiles = (N + 127) // 128
    C = dz_stored.shape[1]
    d = torch.zeros(tiles * 128, C, dtype=torch.float32, device=dz_stored.device)
    d[:N] = dz_stored[:N].float()
    d = d.view(tiles, 128, C)
    acc = torch.zeros(tiles, C, dtype=torch.float32, device=dz_stored.device)
    for r in range(128):
        acc = acc + d[:, r]
    return acc


def eps_softmax(Z):
    """eps(Z) = (24 Z + 192) 2^-24: the bound, relative to w/avg, of the kernel's dz and lse error on exact logits
    with |z| <= Z (derivation: tests/test_gpu_fused_fwd_vs_float64.py)."""
    return (24.0 * Z + 192.0) * U


def focal(z, t, gamma, alpha):
    """The sigmoid focal loss's per-element loss l and the op's analytic gradient g [N, C] in float64, for the op's
    targets t [N] (read as int32: column t - 1 positive, every other column negative, t < 0 ignores the row).  The
    formulas of tests/focal_oracle.py, with p and 1 - p both formed from e = exp(-|z|): the oracle's 1 - p loses all
    its digits once p rounds to 1 in float64 (z > 37), where the kernel's fp32 q = e / (1 + e) stays exact to a few
    ulp, so an elementwise bound needs this form."""
    z = z.to(torch.float64)
    t = t.to(torch.int32).to(torch.int64).reshape(-1, 1)
    cols = torch.arange(z.shape[1], device=z.device).reshape(1, -1)
    pos = t == cols + 1
    neg = (t >= 0) & ~pos
    e = torch.exp(-z.abs())
    r = 1.0 / (1.0 + e)
    p = torch.where(z >= 0, r, e * r)
    q = torch.where(z >= 0, e * r, r)
    lg = torch.log1p(e)
    log1m = -z.clamp_min(0.0) - lg
    logp = (z.clamp_max(0.0) - lg).clamp_min(LOG_FLT_MIN)
    qg, pg = torch.pow(q, gamma), torch.pow(p, gamma)
    l = torch.where(pos, -alpha * qg * logp, torch.where(neg, -(1.0 - alpha) * pg * log1m, torch.zeros_like(z)))
    g = torch.where(pos, -alpha * qg * (q - gamma * p * logp),
                    torch.where(neg, -(1.0 - alpha) * pg * (gamma * q * log1m - p), torch.zeros_like(z)))
    return l, g
