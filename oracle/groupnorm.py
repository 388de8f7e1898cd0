"""fp64 references of the GroupNorm kernels in their ABI layouts (test infrastructure only): ds_channel_stats and
ds_groupnorm_apply / ds_groupnorm_silu (include/dsengine.h) on channels-last bf16 tensors [B, HW, C].

Written from the module maths they replace (nn.GroupNorm with a biased variance, then nn.SiLU), not from the kernels.
The channel concatenation [x1 | x2] of the up blocks is formed explicitly here.  Each returns ``(ref, absref)`` in
fp64 on the operands' device; ``absref`` is what tests/groupnorm_check.py scales its error terms with."""
from __future__ import annotations

import torch

f64 = torch.float64


def channel_stats(x):
    """{sum x, sum x^2} per (sample, channel) of x [B, ..., C] -> [B, C, 2], and absref = {sum |x|, sum x^2}."""
    B, C = x.shape[0], x.shape[-1]
    xd = x.to(f64).reshape(B, -1, C)
    ref = torch.stack([xd.sum(1), (xd * xd).sum(1)], -1)
    absref = torch.stack([xd.abs().sum(1), (xd * xd).sum(1)], -1)
    return ref, absref


def group_moments(stats, HW, groups, biased=True):
    """(mean, var) [B, groups] in fp64 from per-channel fp64 {sum, sum of squares} [B, C, 2]."""
    B, C = stats.shape[0], stats.shape[1]
    n = HW * (C // groups)
    s = stats.to(f64).reshape(B, groups, C // groups, 2).sum(2)
    mean = s[..., 0] / n
    var = s[..., 1] / n - mean * mean
    if not biased:
        var = var * n / (n - 1)
    return mean, var.clamp_min(0.0)


def groupnorm(x1, gamma, beta, groups, eps, silu, x2=None, stats=None, biased=True):
    """GroupNorm(+SiLU) of [x1 | x2] (channels last, [B, ..., C1 (+ C2)]) with gamma / beta [C].

    ``stats`` [B, C, 2] replaces the exact channel sums (a test passes perturbed ones).  Returns (ref, absref, pre):
    ref the output, absref = (|x| + |mean|) rstd |gamma| (the size of the two terms x sc and mean rstd gamma that the
    kernel's x * sc + sf cancels), pre the value before the SiLU (= ref without it)."""
    x = x1 if x2 is None else torch.cat([x1, x2], -1)
    B, C = x.shape[0], x.shape[-1]
    xd = x.to(f64).reshape(B, -1, C)
    HW = xd.shape[1]
    if stats is None:
        stats = channel_stats(x)[0]
    mean, var = group_moments(stats, HW, groups, biased)
    rstd = 1.0 / torch.sqrt(var + eps)
    cpg = C // groups
    mc = mean.repeat_interleave(cpg, 1)[:, None, :]                            # per channel [B, 1, C]
    rc = rstd.repeat_interleave(cpg, 1)[:, None, :]
    g, b = gamma.to(f64).to(x.device), beta.to(f64).to(x.device)
    pre = (xd - mc) * rc * g + b
    ref = pre * torch.sigmoid(pre) if silu else pre
    absref = (xd.abs() + mc.abs()) * rc * g.abs()
    shape = x.shape
    return ref.reshape(shape), absref.reshape(shape), pre.reshape(shape)
