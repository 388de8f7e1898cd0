"""fp64 reference of the wgmma GEMM and the implicit-GEMM 3x3 conv in the kernels' ABI layout (test infrastructure
only): ds_gemm_bf16 (include/dsengine.h) and ds_conv3x3_nhwc, epilogue included.

Every function returns ``(ref, absref)`` in fp64 on the operands' device: ``ref`` the operation, ``absref`` the same
expression with every operand in absolute value (sum |a||w| + |bias| + |rowbias| + |residual|, passed through the
activation's Lipschitz constant), the size of the terms an output element is summed from.  tests/gemm_check.py turns
the two into a per-element bound.

Weights are taken in diffusers / OIHW layout wherever the kernels' packing is exact (``weights.pack_geglu``,
``weights.pack_conv3x3``), so the packers are under test too.  Where packing rounds (``weights.fold_layernorm``,
``weights.pack_conv3x3_up2``) there are two forms: the packed arithmetic restated exactly (``ln_fold=``,
``conv3x3_up2_phases_abi``) and the unpacked module maths (``ln=``, ``conv3x3_abi(upsample2=True)``).
"""
from __future__ import annotations

import math

import torch
import torch.nn.functional as F

f64 = torch.float64
EPILOGUES = ("none", "gelu", "silu", "quickgelu", "geglu")
# max |d act / dx|: erf-GELU 1.1289 (at x = 2.45); x sigmoid(x) 1.0998; x sigmoid(1.702 x) the same in 1.702 x
LIPSCHITZ = {"none": 1.0, "gelu": 1.13, "silu": 1.1, "quickgelu": 1.1, "geglu": 1.13}


def act(x, epilogue: str):
    """The exact activation: erf-GELU, x sigmoid(x), x sigmoid(1.702 x)."""
    if epilogue == "gelu" or epilogue == "geglu":
        return 0.5 * x * (1.0 + torch.erf(x / math.sqrt(2.0)))
    if epilogue == "silu":
        return x * torch.sigmoid(x)
    if epilogue == "quickgelu":
        return x * torch.sigmoid(1.702 * x)
    return x


def _d(t, dev):
    return None if t is None else t.to(device=dev, dtype=f64)


def row_index(M: int, rows_per_batch: int, dev):
    """The row-bias row of each output row: row // rows_per_batch."""
    return torch.arange(M, device=dev) // rows_per_batch


def _linear_terms(a, w, bias, epilogue, rowbias, rows_per_batch, ln, ln_fold, a2):
    """(acc + bias + rowbias, the same in absolute values) of gemm_abi, fp64 [M, N], columns in w's order."""
    dev = a.device
    a2d = a.reshape(-1, a.shape[-1]).to(dev, f64)
    if a2 is not None:
        a2d = torch.cat([a2d, a2.reshape(a2d.shape[0], -1).to(dev, f64)], 1)
    M = a2d.shape[0]
    wd, bd = _d(w, dev), _d(bias, dev)
    if ln is not None:
        gamma, beta, eps = ln
        g, b = _d(gamma, dev), _d(beta, dev)
        xhat = F.layer_norm(a2d, (a2d.shape[1],), eps=eps)
        acc = (xhat * g + b) @ wd.T
        absacc = ((xhat * g).abs() + b.abs()) @ wd.abs().T
    elif ln_fold is not None:
        colsum, eps = _d(ln_fold[0], dev), ln_fold[1]
        st = _d(ln_fold[2], dev).reshape(M, 2) if len(ln_fold) > 2 else torch.stack([a2d.sum(1), (a2d * a2d).sum(1)], 1)
        K = a2d.shape[1]
        mean = st[:, :1] / K
        rstd = ((st[:, 1:] / K - mean * mean).clamp_min(0) + eps).rsqrt()
        acc = rstd * (a2d @ wd.T - mean * colsum)
        absacc = rstd * (a2d.abs() @ wd.abs().T + mean.abs() * colsum.abs())
    else:
        acc = a2d @ wd.T
        absacc = a2d.abs() @ wd.abs().T
    if bd is not None:
        acc, absacc = acc + bd, absacc + bd.abs()
    if rowbias is not None:
        rb = _d(rowbias, dev)[row_index(M, rows_per_batch, dev)]
        if epilogue == "geglu":      # packed order [value block ; gate block] per 256 columns -> natural [value ; gate]
            n = rb.shape[1] // 2
            rb = rb.reshape(M, n // 128, 2, 128).transpose(1, 2).reshape(M, 2 * n)
        acc, absacc = acc + rb, absacc + rb.abs()
    return acc, absacc


def gemm_abi(a, w, bias=None, *, epilogue: str = "none", residual=None, rowbias=None, rows_per_batch: int = 0,
             out_scale: float = 1.0, ln=None, ln_fold=None, a2=None, dtype=f64):
    """ds_gemm_bf16's operation on a [M, K1] (+ a2 [M, K - K1] along K) and w [N, K]:

        out = (act(acc + bias + rowbias[row // rows_per_batch]) + residual) * out_scale

    ``epilogue="geglu"``: w / bias in diffusers GEGLU.proj layout [value(N/2) ; gate(N/2)], out = value * gelu(gate)
    (the kernel takes them through ``weights.pack_geglu``); the row bias is in the kernel's packed column order.
    ``ln=(gamma, beta, eps)``: acc = LayerNorm(a) @ w^T, the module maths (F.layer_norm -> F.linear).
    ``ln_fold=(colsum, eps)`` or ``(colsum, eps, stats)``: the kernel's folded arithmetic on weights already folded by
    ``weights.fold_layernorm``: acc = rstd * (a @ w'^T - mean * colsum), mean / rstd from ``stats`` [M, 2] fp64
    {sum, sum of squares} of a's rows (default: exact, of ``a``); absref = rstd * (sum |a||w'| + |mean||colsum|).
    Returns (ref, absref) [M, n_out] in ``dtype``."""
    acc, absacc = _linear_terms(a, w, bias, epilogue, rowbias, rows_per_batch, ln, ln_fold, a2)
    M, dev = acc.shape[0], acc.device
    if epilogue == "geglu":
        n = acc.shape[1] // 2
        v, g, ev, eg = acc[:, :n], acc[:, n:], absacc[:, :n], absacc[:, n:]
        out = v * act(g, "gelu")
        absout = act(g, "gelu").abs() * ev + LIPSCHITZ["gelu"] * v.abs() * eg
    else:
        out, absout = act(acc, epilogue), LIPSCHITZ[epilogue] * absacc
    if residual is not None:
        r = residual.reshape(M, -1).to(dev, f64)
        out, absout = out + r, absout + r.abs()
    if out_scale != 1.0:
        out, absout = out * out_scale, absout * abs(out_scale)
    return out.to(dtype), absout.to(dtype)


def pre_activation(a, w, bias=None, *, epilogue: str = "none", rowbias=None, rows_per_batch: int = 0, ln_fold=None,
                   a2=None):
    """acc + bias + rowbias of gemm_abi (for GEGLU: the gate half), fp64 [M, n_out]: where the activation is
    evaluated, for the bound's approximation term."""
    acc, _ = _linear_terms(a, w, bias, epilogue, rowbias, rows_per_batch, None, ln_fold, a2)
    return acc[:, acc.shape[1] // 2:] if epilogue == "geglu" else acc


def _nchw(x, dev):
    return x.to(dev, f64).permute(0, 3, 1, 2)


def _conv_epilogue(out, absout, bias, rowbias, residual, dev):
    """NCHW fp64 conv sums -> NHWC with bias, the per-image time-embedding row bias and the residual added."""
    out, absout = out.permute(0, 2, 3, 1), absout.permute(0, 2, 3, 1)
    if bias is not None:
        b = _d(bias, dev)
        out, absout = out + b, absout + b.abs()
    if rowbias is not None:
        rb = _d(rowbias, dev)[:, None, None, :]
        out, absout = out + rb, absout + rb.abs()
    if residual is not None:
        r = _d(residual, dev)
        out, absout = out + r, absout + r.abs()
    return out.contiguous(), absout.contiguous()


def conv3x3_abi(x, w, bias=None, *, stride: int = 1, rowbias=None, residual=None, pad_bottom_right: bool = False,
                upsample2: bool = False, padding_mode: str = "constant", pads=None):
    """ds_conv3x3_nhwc's operation on NHWC x [B, H, W, Cin] and OIHW w [Cout, Cin, 3, 3] -> NHWC (ref, absref):
    conv2d(x, w, stride, padding 1) + bias + rowbias[b] + residual.
    ``pad_bottom_right`` (stride 2): F.pad(x, (0, 1, 0, 1)) then no padding, the VAE encoder's Downsample2D.
    ``upsample2``: conv2d(F.interpolate(x, scale_factor=2, mode="nearest"), w, padding=1), the module maths of
    Upsample2D (the kernel runs it on the bf16-rounded phase sums of ``weights.pack_conv3x3_up2``: see
    conv3x3_up2_phases_abi for the exact restatement).
    ``padding_mode`` ("replicate") and ``pads`` (left, right, top, bottom; the output keeps the operation's size)
    exist for perturbed references: edge replication instead of zero padding, a stride-2 window moved by a pixel."""
    dev = x.device
    xn, wd = _nchw(x, dev), _d(w, dev)
    if upsample2:
        xn = F.interpolate(xn, scale_factor=2.0, mode="nearest")
    H, W = xn.shape[2], xn.shape[3]
    if pad_bottom_right:
        p, Ho, Wo = (0, 1, 0, 1), H // 2, W // 2
    else:
        p, Ho, Wo = (1, 1, 1, 1), (H - 1) // stride + 1, (W - 1) // stride + 1
    xp = F.pad(xn, pads or p, mode=padding_mode)
    out = F.conv2d(xp, wd, stride=stride)[:, :, :Ho, :Wo]
    absout = F.conv2d(xp.abs(), wd.abs(), stride=stride)[:, :, :Ho, :Wo]
    return _conv_epilogue(out, absout, bias, rowbias, residual, dev)


UP2_OFFSETS = {0: -1, 1: 0}   # output parity -> offset of the 2x2 window's first low-resolution tap


def conv3x3_up2_phases_abi(x, w_phases, bias=None, phase_order=(0, 1, 2, 3)):
    """The fused nearest-x2 upsample conv as the kernel computes it: output pixel (2i + a, 2j + b) is the 2x2
    convolution of x with phase kernel w_phases[2a + b] ([4, Cout, 2, 2, Cin], ``weights.pack_conv3x3_up2``, taken
    as given) over low-resolution pixels (i + off(a) + u, j + off(b) + v), zero outside.  ``phase_order`` permutes the
    phase kernels (for a perturbed reference)."""
    dev = x.device
    xn = _nchw(x, dev)
    B, _, H, W = xn.shape
    wp = _d(w_phases, dev)
    xp = F.pad(xn, (1, 1, 1, 1))
    out = torch.empty(B, wp.shape[1], 2 * H, 2 * W, dtype=f64, device=dev)
    absout = torch.empty_like(out)
    for a in (0, 1):
        for b in (0, 1):
            k = wp[phase_order[2 * a + b]].permute(0, 3, 1, 2)          # [Cout, Cin, 2, 2]
            y0, x0 = 1 + UP2_OFFSETS[a], 1 + UP2_OFFSETS[b]
            win = xp[:, :, y0:y0 + H + 1, x0:x0 + W + 1]
            out[:, :, a::2, b::2] = F.conv2d(win, k)
            absout[:, :, a::2, b::2] = F.conv2d(win.abs(), k.abs())
    return _conv_epilogue(out, absout, bias, None, None, dev)


def conv_in_abi(x, w, bias=None):
    """ds_conv_in_3x3 / im2col_latent + GEMM: 3x3 / pad 1 conv of the 4-channel NHWC latent, OIHW w [Cout, 4, 3, 3]."""
    return conv3x3_abi(x, w, bias)
