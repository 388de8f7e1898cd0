"""The tiny VAE decoder's kernels on the H100 against an fp64 reference on every element: ``ds_tiny_conv64`` (every
epilogue combination, plain and ``upsample2``), ``ds_tiny_latent_in`` and ``ds_tiny_conv_out``, at 1 x 1, sizes that
are not tile multiples and 128 x 128, batch 1 and 3 — and each row of a batch-3 launch ``torch.equal`` to the same row
launched alone.

Bound per element: one bf16 rounding of the output (2^-8 |ref|: half a bf16 ulp at the bottom of the value's binade,
the largest relative rounding error) plus the fp32 accumulation, (K + 3) * 2^-23 * S with S the fp64 sum of the magnitudes of every
term (K products, the bias and the residual) and K = 576 (3 x 3 x 64), 256 for an upsample phase, 36 for the first
layer (whose clamp, tanhf, adds a few fp32 ulps of the input, inside the same bound)."""
import itertools

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
bf16, f32, f64 = torch.bfloat16, torch.float32, torch.float64
DEV = "cuda"
SHAPES = [(1, 1), (7, 17), (33, 9), (128, 128)]


def _bound(ref, absum, k):
    return ref.abs() * 2.0 ** -8 + (k + 3) * 2.0 ** -23 * absum


def _check(got, ref, absum, k, what):
    err = (got.double() - ref).abs()
    tol = _bound(ref, absum, k)
    worst = float((err / tol).max())
    print(f"{what}: max |err| {float(err.max()):.3e}, worst err / bound {worst:.3f}")
    assert torch.isfinite(got).all() and (err <= tol).all(), what


def _conv_ref(x, w_oihw, bias, residual, relu):
    """fp64 conv3x3 / pad 1 of NHWC x with an OIHW filter; returns (NHWC result, NHWC sum of term magnitudes)."""
    xn = x.permute(0, 3, 1, 2).double()
    y = F.conv2d(xn, w_oihw.double(), padding=1)
    s = F.conv2d(xn.abs(), w_oihw.double().abs(), padding=1)
    y, s = y.permute(0, 2, 3, 1), s.permute(0, 2, 3, 1)
    if bias is not None:
        y, s = y + bias.double(), s + bias.double().abs()
    if residual is not None:
        y, s = y + residual.double(), s + residual.double().abs()
    return (y.clamp_min(0) if relu else y), s


def _up2_ref(x, w_up, bias, residual, relu):
    """fp64 conv3x3(nearest_x2(x)) as the kernel computes it: the four 2 x 2 phase filters of pack_conv3x3_up2 (bf16)
    over x; phase (a, b) reads rows i - 1 + a .. i + a and writes pixel (2i + a, 2j + b)."""
    B, H, W, C = x.shape
    xp = F.pad(x.permute(0, 3, 1, 2).double(), (1, 1, 1, 1))
    y = torch.zeros(B, C, 2 * H, 2 * W, dtype=f64, device=x.device)
    s = torch.zeros_like(y)
    for a, b in itertools.product((0, 1), (0, 1)):
        k = w_up[2 * a + b].permute(0, 3, 1, 2).double()             # [Cout, Cin, 2, 2]
        y[:, :, a::2, b::2] = F.conv2d(xp, k)[:, :, a:a + H, b:b + W]
        s[:, :, a::2, b::2] = F.conv2d(xp.abs(), k.abs())[:, :, a:a + H, b:b + W]
    y, s = y.permute(0, 2, 3, 1), s.permute(0, 2, 3, 1)
    if bias is not None:
        y, s = y + bias.double(), s + bias.double().abs()
    if residual is not None:
        y, s = y + residual.double(), s + residual.double().abs()
    return (y.clamp_min(0) if relu else y), s


def _weights(seed, cout=64):
    g = torch.Generator().manual_seed(seed)
    w = (torch.randn(cout, 64, 3, 3, generator=g) / 24).to(bf16).float()
    b = 0.3 * torch.randn(cout, generator=g)
    return w.to(DEV), b.to(DEV)


@pytest.mark.parametrize("up2", [False, True])
@pytest.mark.parametrize("bias,res,relu", list(itertools.product((False, True), repeat=3)))
@pytest.mark.parametrize("H,W", SHAPES)
@pytest.mark.parametrize("B", [1, 3])
def test_conv64_matches_fp64(B, H, W, bias, res, relu, up2):
    from diffsensei_b200 import ops
    from diffsensei_b200.weights import pack_conv3x3, pack_conv3x3_up2
    g = torch.Generator().manual_seed(H * 1000 + W * 10 + B)
    x = torch.randn(B, H, W, 64, generator=g).to(bf16).to(DEV)
    w, b = _weights(H + W)
    Ho, Wo = (2 * H, 2 * W) if up2 else (H, W)
    r = torch.randn(B, Ho, Wo, 64, generator=g).to(bf16).to(DEV) if res else None
    bb = b if bias else None
    wp = pack_conv3x3_up2(w) if up2 else pack_conv3x3(w)
    got = ops.tiny_conv64(x, wp, bb, residual=r, relu=relu, upsample2=up2)
    if up2:
        ref, s = _up2_ref(x, wp, bb, r, relu)
    else:
        ref, s = _conv_ref(x, w, bb, r, relu)
    assert got.shape == (B, Ho, Wo, 64)
    _check(got, ref, s, 256 if up2 else 576, f"conv64 B={B} {H}x{W} bias={bias} res={res} relu={relu} up2={up2}")
    if B == 3:                                               # batch invariance: each row alone gives the same bits
        for i in range(B):
            ri = None if r is None else r[i:i + 1].contiguous()
            one = ops.tiny_conv64(x[i:i + 1].contiguous(), wp, bb, residual=ri, relu=relu, upsample2=up2)
            assert torch.equal(one, got[i:i + 1]), i


@pytest.mark.parametrize("H,W", SHAPES)
@pytest.mark.parametrize("B", [1, 3])
def test_latent_in_matches_fp64(B, H, W):
    from diffsensei_b200 import ops
    g = torch.Generator().manual_seed(H * 7 + W + B)
    lat = (4 * torch.randn(B, 4, H, W, generator=g)).to(DEV)        # wide enough for the clamp to bite
    w = (torch.randn(64, 4, 3, 3, generator=g) / 6).to(DEV)
    b = (0.3 * torch.randn(64, generator=g)).to(DEV)
    inv = 1.0 / 0.13025
    got = ops.tiny_latent_in(lat, w.permute(0, 2, 3, 1).contiguous(), b, inv)
    z = torch.tanh(lat.double() * inv / 3) * 3
    ref = F.conv2d(z, w.double(), b.double(), padding=1).clamp_min(0).permute(0, 2, 3, 1)
    s = (F.conv2d(z.abs(), w.double().abs(), padding=1) + b.double().abs()[:, None, None]).permute(0, 2, 3, 1)
    assert got.shape == (B, H, W, 64) and got.dtype == bf16
    _check(got, ref, s, 36, f"latent_in B={B} {H}x{W}")
    if B == 3:
        for i in range(B):
            assert torch.equal(ops.tiny_latent_in(lat[i:i + 1].contiguous(), w.permute(0, 2, 3, 1).contiguous(), b,
                                                  inv), got[i:i + 1])


@pytest.mark.parametrize("H,W", SHAPES)
@pytest.mark.parametrize("B", [1, 3])
def test_conv_out_matches_fp64(B, H, W):
    from diffsensei_b200 import ops
    from diffsensei_b200.weights import pack_conv3x3
    g = torch.Generator().manual_seed(H * 5 + W + B)
    x = torch.randn(B, H, W, 64, generator=g).to(bf16).to(DEV)
    w, b = _weights(H * 3 + W, cout=3)
    w8 = torch.cat([w, torch.zeros(5, 64, 3, 3, device=DEV)])
    got = ops.tiny_conv_out(x, pack_conv3x3(w8), b)
    ref, s = _conv_ref(x, w, b, None, False)
    assert got.shape == (B, H, W, 3)
    _check(got, ref, s, 576, f"conv_out B={B} {H}x{W}")
    if B == 3:
        for i in range(B):
            assert torch.equal(ops.tiny_conv_out(x[i:i + 1].contiguous(), pack_conv3x3(w8), b), got[i:i + 1])


def test_wrapper_checks():
    from diffsensei_b200 import ops
    from diffsensei_b200.weights import pack_conv3x3
    x = torch.zeros(1, 8, 8, 64, dtype=bf16, device=DEV)
    w = pack_conv3x3(torch.zeros(64, 64, 3, 3, device=DEV))
    with pytest.raises(ops.DsEngineError, match="64 channels"):
        ops.tiny_conv64(torch.zeros(1, 8, 8, 32, dtype=bf16, device=DEV), w)
    with pytest.raises(ops.DsEngineError, match="w must be"):
        ops.tiny_conv64(x, w, upsample2=True)
    with pytest.raises(ops.DsEngineError, match="residual"):
        ops.tiny_conv64(x, w, residual=torch.zeros(1, 8, 8, 32, dtype=bf16, device=DEV))
    with pytest.raises(ops.DsEngineError, match="dtype"):
        ops.tiny_conv64(x.float(), w)
    with pytest.raises(ops.DsEngineError, match="aligned"):
        ops.tiny_conv64(torch.zeros(1 * 8 * 8 * 64 + 1, dtype=bf16, device=DEV)[1:].view(1, 8, 8, 64), w)
