"""Parity of every C-ABI kernel against the CPU oracle / a plain fp32 torch restatement of the same op,
on the same seeded inputs (bf16-rounded where the kernel takes bf16).  Tolerances: the kernels round ONCE to
bf16 at the output (relative 2^-8 = 3.9e-3), so per-op rel-L2 must be <= 1e-2 (BASELINE.md §3); index / mask
work must be bit-exact."""
import os

import pytest
import torch
import torch.nn.functional as F

from conftest import GOLDEN, rel_l2


def launch_count():
    from diffsensei_b200._lib import launch_count as lc
    return lc()

pytestmark = pytest.mark.gpu

bf16, f32 = torch.bfloat16, torch.float32
DEV = "cuda"


def _r(*shape, seed=0, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(*shape, generator=g) * scale).to(bf16)


@pytest.fixture(scope="module")
def ops():
    from diffsensei_b200 import ops as o
    return o


# ---------------------------------------------------------------------------------------------- norms
@pytest.mark.parametrize("B,H,W,C,silu,eps", [(2, 16, 24, 64, True, 1e-5), (2, 7, 9, 320, True, 1e-5),
                                              (1, 32, 32, 1280, False, 1e-6), (3, 5, 3, 960, True, 1e-5),
                                              (2, 64, 64, 640, True, 1e-5), (1, 1, 1, 64, True, 1e-5)])
def test_groupnorm_silu(ops, B, H, W, C, silu, eps):
    x = _r(B, H, W, C, seed=1) * 1.7 + 0.3
    gamma, beta = torch.randn(C) * 0.2 + 1, torch.randn(C) * 0.1
    want = F.group_norm(x.float().permute(0, 3, 1, 2), 32, gamma, beta, eps)
    want = (F.silu(want) if silu else want).permute(0, 2, 3, 1)
    got = ops.groupnorm_silu(x.to(DEV), gamma.to(DEV), beta.to(DEV), 32, eps, silu)
    assert rel_l2(got.float(), want) < 6e-3
    inplace = x.to(DEV).clone()
    ops.groupnorm_silu(inplace, gamma.to(DEV), beta.to(DEV), 32, eps, silu, out=inplace)
    assert torch.equal(inplace, got)


@pytest.mark.parametrize("rows,C", [(77, 128), (300, 640), (64, 1280), (5, 2048), (33, 256)])
def test_layernorm(ops, rows, C):
    x = _r(rows, C, seed=2) * 2 + 0.5
    gamma, beta = torch.randn(C) * 0.2 + 1, torch.randn(C) * 0.1
    want = F.layer_norm(x.float(), (C,), gamma, beta, 1e-5)
    got = ops.layernorm(x.to(DEV), gamma.to(DEV), beta.to(DEV), 1e-5)
    assert rel_l2(got.float(), want) < 6e-3


# ---------------------------------------------------------------------------------------------- bbox kernels
def test_dialog_embed_matches_executed_reference(ops):
    for case in torch.load(os.path.join(GOLDEN, "dialog_embed.pt"), weights_only=False):
        is_bf16 = case["sample"].dtype == bf16
        sample = case["sample"].to(bf16).permute(0, 2, 3, 1).contiguous().to(DEV)
        got = ops.dialog_embed_add_(sample, case["emb"].float().to(DEV), case["dialog_bbox"].float().to(DEV), is_bf16)
        want = case["out"].float().permute(0, 2, 3, 1)
        if is_bf16:      # identical dtype path: bit-exact, including int(bf16(0.9)*152) = 137
            assert torch.equal(got.float().cpu(), want)
        else:            # fp32 reference vs bf16 storage: the SET of touched pixels must be identical
            base = case["sample"].float().permute(0, 2, 3, 1)
            assert torch.equal((got.float().cpu() - base.to(bf16).float()).abs().sum(-1) > 0,
                               (want - base).abs().sum(-1) > 0)


def test_ip_mask_bit_exact_vs_reference_kats_and_all_buckets(ops):
    from oracle import attention as A
    for kat in torch.load(os.path.join(GOLDEN, "ip_mask_kats.pt"), weights_only=False):
        got = ops.ip_mask(kat["bbox"].to(DEV), kat["N"], kat["aspect_ratio"], 16, 16)
        assert torch.equal(got.cpu() == 0, kat["open"])
        assert set(got.unique().tolist()) <= {0.0, -10000.0}
    bb = torch.tensor([[[.05, .10, .50, .95], [.50, .15, .95, .90], [.30, .55, .70, 1.0], [0.0, 0.0, .30, .40]],
                       [[0.0] * 4] * 4, [[1 / 3, 0.25, 2 / 3, 0.75], [0.5, 0.5, 0.5, 0.5], [0, 0, 1, 1], [.2, 0, .2, 1]]])
    tab = torch.load(os.path.join(GOLDEN, "derived_hw_table.pt"), weights_only=False)
    for bh, bw, _d, fh, fw, _dh, _dw in tab.tolist():      # every (bucket, level) shape incl. the 5 quirk cases
        n, ar = fh * fw, (bh // 8) / (bw // 8)
        got = ops.ip_mask(bb.to(DEV), n, ar, 16, 16)
        assert torch.equal(got.cpu() == 0, A.ip_open_mask(bb, n, ar, 16, 16)), (bh, bw, n)


# ---------------------------------------------------------------------------------------------- GEMM / conv
@pytest.mark.parametrize("M,N,K", [(77, 256, 128), (300, 200, 72), (1024, 640, 320), (16, 1280, 2816), (4096, 320, 64)])
def test_gemm_bias_residual(ops, M, N, K):
    a, w = _r(M, K, seed=3), _r(N, K, seed=4, scale=K ** -0.5)
    bias, res = torch.randn(N) * 0.3, _r(M, N, seed=5)
    want = F.linear(a.float(), w.float(), bias) + res.float()
    got = ops.gemm(a.to(DEV), w.to(DEV), bias.to(DEV), residual=res.to(DEV))
    assert rel_l2(got.float(), want) < 5e-3
    got32 = ops.gemm(a.to(DEV), w.to(DEV), bias.to(DEV), residual=res.to(DEV), out_fp32=True)
    assert rel_l2(got32, want) < 1e-5


def test_gemm_geglu_matches_diffusers_feedforward(ops):
    from diffsensei_b200.weights import pack_geglu
    c, M = 128, 333
    x = _r(M, c, seed=6)
    w, b = _r(8 * c, c, seed=7, scale=c ** -0.5), torch.randn(8 * c) * 0.2
    val, gate = F.linear(x.float(), w.float(), b).chunk(2, dim=-1)
    want = val * F.gelu(gate)
    wp, bp = pack_geglu(w.float(), b)
    got = ops.gemm(x.to(DEV), wp.to(DEV), bp.to(DEV), epilogue=ops.EPI_GEGLU)
    assert got.shape == (M, 4 * c) and rel_l2(got.float(), want) < 6e-3


def test_gemm_activations_and_rowbias(ops):
    a, w = _r(512, 192, seed=8), _r(256, 192, seed=9, scale=192 ** -0.5)
    rb = torch.randn(4, 1000)[:, 100:356]
    base = F.linear(a.float(), w.float()) + rb.repeat_interleave(128, 0)
    rbd = torch.randn(4, 1000)
    rbd[:, 100:356] = rb
    got = ops.gemm(a.to(DEV), w.to(DEV), rowbias=rbd.to(DEV)[:, 100:356], rows_per_batch=128)   # strided table slice
    assert rel_l2(got.float(), base) < 5e-3
    assert rel_l2(ops.gemm(a.to(DEV), w.to(DEV), epilogue=ops.EPI_SILU).float(), F.silu(F.linear(a.float(), w.float()))) < 6e-3
    assert rel_l2(ops.gemm(a.to(DEV), w.to(DEV), epilogue=ops.EPI_GELU).float(), F.gelu(F.linear(a.float(), w.float()))) < 6e-3


@pytest.mark.parametrize("M,N,K,geglu", [(300, 200, 72, False), (1024, 1920, 640, False), (333, 1024, 128, True),
                                          (4096, 640, 640, False)])
def test_gemm_layernorm_fusion(ops, M, N, K, geglu):
    """BasicTransformerBlock: h = linear(attn) + h ; y = linear2(LayerNorm(h)).  The first GEMM publishes the row
    statistics of h, the second consumes them with LayerNorm folded into its weights (weights.fold_layernorm)."""
    from diffsensei_b200.weights import colsum_bf16, fold_layernorm, pack_geglu
    a0, w0 = _r(M, 96, seed=20), _r(K, 96, seed=21, scale=96 ** -0.5)
    b0, res = torch.randn(K) * 0.3, _r(M, K, seed=22) * 2 + 0.7          # row mean != 0 on purpose
    gamma, beta = torch.randn(K) * 0.2 + 1, torch.randn(K) * 0.1
    w1, b1 = _r(N, K, seed=23, scale=K ** -0.5), torch.randn(N) * 0.2
    stats = torch.full((2 * M,), 7.0, device=DEV, dtype=torch.float64)     # the call must zero it first
    h = ops.gemm(a0.to(DEV), w0.to(DEV), b0.to(DEV), residual=res.to(DEV), row_stats_out=stats)
    hf = h.float().cpu()
    st = stats.cpu().view(M, 2).float()
    h32 = F.linear(a0.float(), w0.float(), b0) + res.float()   # the statistics are taken before the bf16 rounding
    assert torch.allclose(st[:, 0], h32.sum(1), rtol=1e-4, atol=2e-2)
    assert torch.allclose(st[:, 1], (h32 * h32).sum(1), rtol=1e-4, atol=2e-2)
    ln = F.layer_norm(hf, (K,), gamma, beta, 1e-5)
    w2, b2 = fold_layernorm(w1.float(), b1, gamma, beta)
    if geglu:
        val, gate = F.linear(ln, w1.float(), b1).chunk(2, dim=-1)
        want = val * F.gelu(gate)
        wp, bp = pack_geglu(w2, b2)
        got = ops.gemm(h, wp.to(DEV), bp.to(DEV), epilogue=ops.EPI_GEGLU, ln_stats=stats,
                       ln_colsum=colsum_bf16(wp).to(DEV), ln_eps=1e-5)
    else:
        want = F.linear(ln, w1.float(), b1)
        wp = w2.to(bf16)
        got = ops.gemm(h, wp.to(DEV), b2.to(DEV), ln_stats=stats, ln_colsum=colsum_bf16(wp).to(DEV), ln_eps=1e-5)
    assert rel_l2(got.float(), want) < 8e-3
    # buffer rotation without memsets: the consumer clears a third buffer, a later producer accumulates into it
    third = torch.full((2 * M,), 7.0, device=DEV, dtype=torch.float64)
    if not geglu:
        again = ops.gemm(h, wp.to(DEV), b2.to(DEV), ln_stats=stats, ln_colsum=colsum_bf16(wp).to(DEV), ln_eps=1e-5,
                         zero_rows=third)
        assert torch.equal(again, got) and torch.count_nonzero(third).item() == 0
        ops.gemm(a0.to(DEV), w0.to(DEV), b0.to(DEV), residual=res.to(DEV), row_stats_out=third, row_stats_zeroed=True)
        assert torch.equal(third, stats)          # fp64 sums of fp32 partials: exact, hence order-independent


@pytest.mark.parametrize("B,H,W,Cin,Cout,stride", [(2, 16, 24, 64, 128, 1), (2, 19, 13, 128, 64, 1),
                                                   (1, 16, 32, 64, 128, 2), (2, 19, 13, 64, 64, 2),
                                                   (1, 8, 8, 320, 4, 1), (2, 32, 32, 192, 320, 1)])
def test_conv3x3(ops, B, H, W, Cin, Cout, stride):
    from diffsensei_b200.weights import pack_conv3x3
    x = _r(B, H, W, Cin, seed=10)
    w = _r(Cout, Cin, 3, 3, seed=11, scale=(9 * Cin) ** -0.5)
    bias, temb = torch.randn(Cout) * 0.2, torch.randn(B, Cout) * 0.5
    want = F.conv2d(x.float().permute(0, 3, 1, 2), w.float(), bias, stride=stride, padding=1) + temb[:, :, None, None]
    res = _r(*want.permute(0, 2, 3, 1).shape, seed=12)
    want = want.permute(0, 2, 3, 1) + res.float()
    got = ops.conv3x3(x.to(DEV), pack_conv3x3(w.float()).to(DEV), bias.to(DEV), stride=stride, rowbias=temb.to(DEV),
                      residual=res.to(DEV))
    assert got.shape == want.shape and rel_l2(got.float(), want) < 5e-3


def test_conv_in(ops):
    x = _r(2, 17, 23, 4, seed=13)
    w, b = torch.randn(64, 4, 3, 3) * 0.2, torch.randn(64) * 0.1
    want = F.conv2d(x.float().permute(0, 3, 1, 2), w, b, padding=1).permute(0, 2, 3, 1)
    got = ops.conv_in(x.to(DEV), w.permute(0, 2, 3, 1).contiguous().to(DEV), b.to(DEV))
    assert rel_l2(got.float(), want) < 5e-3


# ---------------------------------------------------------------------------------------------- attention
def test_attention_self_vs_executed_reference(ops):
    g = torch.load(os.path.join(GOLDEN, "attn_self.pt"), weights_only=False)
    hs = g["hs"].to(bf16)
    wqkv = torch.cat([g["to_q"], g["to_k"], g["to_v"]], 0).to(bf16)
    qkv = ops.gemm(hs.to(DEV), wqkv.to(DEV))
    a = ops.attention_self(qkv, g["heads"])
    out = ops.gemm(a, g["to_out_w"].to(bf16).to(DEV), g["to_out_b"].to(DEV))
    assert rel_l2(out.float(), g["out"]) < 1.5e-2        # three chained bf16 roundings vs the fp32 reference


def test_attention_cross_ip_vs_executed_reference(ops):
    g = torch.load(os.path.join(GOLDEN, "attn_cross_ip.pt"), weights_only=False)
    hs, ehs = g["hs"].to(bf16).to(DEV), g["ehs"].to(bf16).to(DEV)
    end = ehs.shape[1] - (g["num_ip_tokens"] + g["num_dummy"])
    q = ops.gemm(hs, g["to_q"].to(bf16).to(DEV))
    kv_t = ops.gemm(ehs[:, :end].contiguous(), torch.cat([g["to_k"], g["to_v"]], 0).to(bf16).to(DEV))
    kv_i = ops.gemm(ehs[:, end:].contiguous(), torch.cat([g["to_k_ip"], g["to_v_ip"]], 0).to(bf16).to(DEV))
    a = ops.attention_cross_ip(q, kv_t, kv_i, g["bbox"].to(DEV), g["heads"], g["aspect_ratio"], g["scale"], 16, 16)
    out = ops.gemm(a, g["to_out_w"].to(bf16).to(DEV), g["to_out_b"].to(DEV))
    assert rel_l2(out.float(), g["out"]) < 1.5e-2


def test_engine_processors_follow_the_diffusers_protocol(ops):
    """The nn.Module processors called exactly like diffusers' Attention.forward calls them."""
    import types
    from diffsensei_b200 import AttnProcessor2_0, MaskedIPAttnProcessor2_0
    g = torch.load(os.path.join(GOLDEN, "attn_cross_ip.pt"), weights_only=False)

    def lin(w, b=None):
        m = torch.nn.Linear(w.shape[1], w.shape[0], bias=b is not None)
        m.weight.data, m.bias = w.clone(), (None if b is None else torch.nn.Parameter(b.clone()))
        return m.to(DEV, bf16)

    attn = types.SimpleNamespace(heads=g["heads"], spatial_norm=None, group_norm=None, norm_cross=False,
                                 residual_connection=False, rescale_output_factor=1.0, to_q=lin(g["to_q"]),
                                 to_k=lin(g["to_k"]), to_v=lin(g["to_v"]),
                                 to_out=[lin(g["to_out_w"], g["to_out_b"]), torch.nn.Identity()])
    proc = MaskedIPAttnProcessor2_0(hidden_size=128, cross_attention_dim=64, num_ip_tokens=64, num_dummy_tokens=16)
    proc.load_state_dict({"to_k_ip.weight": g["to_k_ip"], "to_v_ip.weight": g["to_v_ip"]})
    proc = proc.to(DEV, bf16)
    proc.scale = g["scale"]
    out = proc(attn, g["hs"].to(DEV, bf16), encoder_hidden_states=g["ehs"].to(DEV, bf16), bbox=g["bbox"].to(DEV),
               aspect_ratio=g["aspect_ratio"], dialog_bbox=None)
    assert rel_l2(out.float(), g["out"]) < 1.5e-2
    s = torch.load(os.path.join(GOLDEN, "attn_self.pt"), weights_only=False)
    attn1 = types.SimpleNamespace(heads=s["heads"], spatial_norm=None, group_norm=None, norm_cross=False,
                                  residual_connection=False, rescale_output_factor=1.0, to_q=lin(s["to_q"]),
                                  to_k=lin(s["to_k"]), to_v=lin(s["to_v"]),
                                  to_out=[lin(s["to_out_w"], s["to_out_b"]), torch.nn.Identity()])
    out = AttnProcessor2_0()(attn1, s["hs"].to(DEV, bf16), bbox=g["bbox"].to(DEV), aspect_ratio=1.0, dialog_bbox=None)
    assert rel_l2(out.float(), s["out"]) < 1.5e-2
    assert sorted(proc.state_dict()) == ["to_k_ip.weight", "to_v_ip.weight"] and hasattr(proc, "scale")


@pytest.mark.parametrize("B,N,heads", [(1, 128, 1), (2, 200, 2), (1, 1000, 3), (2, 64, 1)])
def test_attention_self_vs_oracle_sdpa(ops, B, N, heads):
    from oracle.attention import sdpa
    C = heads * 64
    qkv = _r(B, N, 3 * C, seed=14, scale=1.5)
    q, k, v = (t.float().view(B, N, heads, 64).transpose(1, 2) for t in qkv.chunk(3, dim=-1))
    want = sdpa(q, k, v).transpose(1, 2).reshape(B, N, C)
    assert rel_l2(ops.attention_self(qkv.to(DEV), heads).float(), want) < 1e-2


# ---------------------------------------------------------------------------------------------- glue
def test_layout_upsample_concat_silu_timestep(ops):
    x = torch.randn(2, 4, 9, 13)
    nhwc = ops.nchw_to_nhwc(x.to(DEV))
    assert torch.equal(nhwc.cpu(), x.to(bf16).permute(0, 2, 3, 1))
    assert torch.equal(ops.nhwc_to_nchw(nhwc, f32).cpu(), x.to(bf16).float())
    y = _r(2, 5, 7, 64, seed=15)
    for (ho, wo) in ((10, 14), (9, 13), (11, 15)):
        want = F.interpolate(y.float().permute(0, 3, 1, 2), size=(ho, wo), mode="nearest").permute(0, 2, 3, 1)
        assert torch.equal(ops.upsample_nearest(y.to(DEV), ho, wo).float().cpu(), want)
    a, b = _r(3, 5, 64, seed=16), _r(3, 5, 192, seed=17)
    assert torch.equal(ops.concat_channels(a.to(DEV), b.to(DEV)).cpu(), torch.cat([a, b], -1))
    assert rel_l2(ops.silu(y.to(DEV)).float(), F.silu(y.float())) < 4e-3
    from oracle.unet import timestep_sinusoid
    t = torch.tensor([981.0, 1.0, 500.0, 1024.0])
    for dim in (320, 256, 64):
        assert (ops.timestep_embedding(t.to(DEV), dim).float().cpu() - timestep_sinusoid(t, dim)).abs().max() < 8e-3


def test_cfg_step_ddim(ops):
    from oracle.ddim import DDIMSchedule
    sch = DDIMSchedule()
    t = sch.set_timesteps(50)[7]
    a_t, a_prev = sch.coefficients(t)
    bs, H, W = 2, 6, 5
    eps, lat = _r(2 * bs, H, W, 4, seed=18), torch.randn(bs, H, W, 4)
    eu, et = eps.float().chunk(2)
    want = sch.step(eu + 7.5 * (et - eu), t, lat)
    latd, mi = lat.to(DEV).clone(), torch.empty(2 * bs, H, W, 4, dtype=bf16, device=DEV)
    ops.cfg_step_(eps.to(DEV), latd, mi, torch.tensor([a_t, a_prev], device=DEV), 7.5, euler=False)
    assert rel_l2(latd, want) < 1e-5
    assert torch.equal(mi[:bs], mi[bs:]) and torch.equal(mi[:bs].cpu(), latd.cpu().to(bf16))


# ---------------------------------------------------------------------------------------------- full-size properties
def test_full_size_properties_cfg2(ops):
    """BASELINE cfg2 shapes, checked through size-independent properties (the oracle is too slow here)."""
    torch.manual_seed(0)
    # GroupNorm without affine/SiLU: every (sample, group) of the output has mean 0, variance 1
    x = (torch.randn(8, 128, 128, 320, device=DEV) * 2 + 1).to(bf16)
    y = ops.groupnorm_silu(x, torch.ones(320, device=DEV), torch.zeros(320, device=DEV), 32, 1e-5, False)
    g = y.float().view(8, 128 * 128, 32, 10)
    assert g.mean(dim=(1, 3)).abs().max() < 2e-3 and (g.var(dim=(1, 3), unbiased=False) - 1).abs().max() < 5e-3
    del x, y, g
    # softmax rows sum to one: with V == const the attention output is that constant
    B, N, heads = 8, 4096, 10
    qkv = torch.randn(B, N, 3 * heads * 64, device=DEV).to(bf16)
    qkv[:, :, 2 * heads * 64:] = 0.75
    out = ops.attention_self(qkv, heads)
    assert (out.float() - 0.75).abs().max() < 1e-2
    # linearity of the conv in its input:  conv(2x) - bias == 2 (conv(x) - bias)
    from diffsensei_b200.weights import pack_conv3x3
    xc = torch.randn(8, 64, 64, 640, device=DEV).to(bf16)
    w = pack_conv3x3(torch.randn(640, 640, 3, 3, device=DEV) * (9 * 640) ** -0.5)
    y1, y2 = ops.conv3x3(xc, w, out_fp32=True), ops.conv3x3(xc * 2, w, out_fp32=True)
    assert rel_l2(y2, 2 * y1) < 1e-6


# ---------------------------------------------------------------------------------------------- round-2 kernels
def _chan_stats_ref(t):          # t: [B, ..., C] -> fp64 [B, C, 2]
    B, C = t.shape[0], t.shape[-1]
    v = t.double().reshape(B, -1, C)
    return torch.stack([v.sum(1), (v * v).sum(1)], dim=-1)


@pytest.mark.parametrize("B,H,W,C", [(2, 16, 24, 64), (3, 7, 9, 320), (1, 64, 64, 1280), (2, 33, 17, 2560)])
def test_channel_stats(ops, B, H, W, C):
    x = _r(B, H, W, C, seed=5) * 1.5 + 0.25
    got = ops.channel_stats(x.to(DEV)).cpu()
    want = _chan_stats_ref(x)
    assert got.shape == (B, C, 2)
    assert torch.allclose(got, want, rtol=1e-5, atol=1e-3)       # fp32 partials over <= a few hundred pixels
    again = ops.channel_stats(x.to(DEV)).cpu()
    assert torch.equal(again, got)                               # fixed-order partials + exact fp64 sums


@pytest.mark.parametrize("B,H,W,C1,C2,silu,eps", [(2, 16, 24, 64, 0, True, 1e-5), (2, 9, 7, 640, 320, True, 1e-5),
                                                 (1, 32, 32, 1280, 640, True, 1e-5), (2, 8, 8, 1280, 1280, True, 1e-5),
                                                 (3, 5, 3, 320, 0, False, 1e-6), (2, 64, 64, 320, 320, True, 1e-5)])
def test_groupnorm_apply_two_sources(ops, B, H, W, C1, C2, silu, eps):
    """GroupNorm(+SiLU) of torch.cat([x1, x2], channel) from per-channel statistics, without the concatenation:
    group boundaries of the result (e.g. 60 channels per group at 1280 + 640) straddle the two tensors."""
    x1 = _r(B, H, W, C1, seed=1) * 1.7 + 0.3
    x2 = (_r(B, H, W, C2, seed=2) * 0.6 - 0.2) if C2 else None
    C = C1 + C2
    gamma, beta = torch.randn(C) * 0.2 + 1, torch.randn(C) * 0.1
    xc = x1 if x2 is None else torch.cat([x1, x2], dim=-1)
    want = F.group_norm(xc.float().permute(0, 3, 1, 2), 32, gamma, beta, eps)
    want = (F.silu(want) if silu else want).permute(0, 2, 3, 1)
    s1 = ops.channel_stats(x1.to(DEV))
    s2 = ops.channel_stats(x2.to(DEV)) if C2 else None
    got = ops.groupnorm_apply(x1.to(DEV), s1, gamma.to(DEV), beta.to(DEV), 32, eps, silu,
                              x2=None if x2 is None else x2.to(DEV), stats2=s2)
    assert got.shape == (B, H, W, C) and rel_l2(got.float(), want) < 6e-3


@pytest.mark.parametrize("M,N,K1,K2", [(512, 320, 640, 320), (1024, 640, 1280, 640), (300, 1280, 2560 - 1280, 1280)])
def test_gemm_two_operand_k_concat(ops, M, N, K1, K2):
    """The 1x1 shortcut of an up-block resnet on torch.cat([hidden, skip], 1): [a | a2] along K from two tensors."""
    a, a2 = _r(M, K1, seed=3), _r(M, K2, seed=4)
    w = _r(N, K1 + K2, seed=5, scale=(K1 + K2) ** -0.5)
    bias = torch.randn(N) * 0.1
    want = F.linear(torch.cat([a, a2], 1).float(), w.float(), bias)
    got = ops.gemm(a.to(DEV), w.to(DEV), bias.to(DEV), a2=a2.to(DEV))
    ref = ops.gemm(torch.cat([a, a2], 1).to(DEV), w.to(DEV), bias.to(DEV))
    assert rel_l2(got.float(), want) < 6e-3 and torch.equal(got, ref)      # same K order -> bit-identical


@pytest.mark.parametrize("B,HW,N,K,res", [(2, 1024, 1280, 256, True), (3, 128, 320, 128, False), (8, 1024, 1280, 64, True),
                                          (2, 256, 640, 192, True)])
def test_gemm_producer_channel_stats(ops, B, HW, N, K, res):
    """chan_stats from the GEMM epilogue == statistics of the bf16 output it wrote (incl. the tail-launch split at
    M = 8192, N = 1280 where the last m-rows run as BN = 128 tiles)."""
    a = _r(B * HW, K, seed=6)
    w = _r(N, K, seed=7, scale=K ** -0.5)
    bias = torch.randn(N) * 0.1
    r = _r(B * HW, N, seed=8) if res else None
    st = torch.zeros(B, N, 2, dtype=torch.float64, device=DEV)
    out = ops.gemm(a.to(DEV), w.to(DEV), bias.to(DEV), residual=None if r is None else r.to(DEV), chan_stats=st,
                   stats_rows_per_sample=HW)
    want = F.linear(a.float(), w.float(), bias) + (0 if r is None else r.float())
    assert rel_l2(out.float(), want) < 6e-3
    ref = _chan_stats_ref(out.cpu().view(B, HW, N))
    assert torch.allclose(st.cpu(), ref, rtol=1e-5, atol=1e-3)
    plain = ops.gemm(a.to(DEV), w.to(DEV), bias.to(DEV), residual=None if r is None else r.to(DEV))
    assert torch.equal(plain, out)                                # the statistics epilogue does not change the output


@pytest.mark.parametrize("B,H,W,Cin,Cout,stride", [(2, 16, 16, 64, 64, 1), (2, 18, 27, 128, 320, 1), (1, 33, 20, 64, 128, 2),
                                                  (8, 32, 32, 128, 1280, 1)])
def test_conv_producer_channel_stats(ops, B, H, W, Cin, Cout, stride):
    """chan_stats from the conv epilogue on ragged maps: pixels of partial 8x16 patches must not be counted."""
    x = _r(B, H, W, Cin, seed=9)
    w = _r(Cout, Cin, 3, 3, seed=10, scale=(9 * Cin) ** -0.5)
    bias = torch.randn(Cout) * 0.1
    from diffsensei_b200.weights import pack_conv3x3
    st = torch.zeros(B, Cout, 2, dtype=torch.float64, device=DEV)
    out = ops.conv3x3(x.to(DEV), pack_conv3x3(w.float()).to(DEV), bias.to(DEV), stride=stride, chan_stats=st)
    want = F.conv2d(x.float().permute(0, 3, 1, 2), w.float(), bias, stride=stride, padding=1).permute(0, 2, 3, 1)
    assert rel_l2(out.float(), want) < 6e-3
    assert torch.allclose(st.cpu(), _chan_stats_ref(out.cpu()), rtol=1e-5, atol=1e-3)


def test_gemm_tail_launch_is_bit_identical_to_wide_tiles(ops):
    """M 8192 x N 1280 is 320 wide tiles on 132 CTAs: the call runs the last m-rows as 128-column units of the same
    launch (mixed-width schedule).  Every output element accumulates the same k-blocks in the same order, so
    those rows must equal the same rows computed on their own (15 wide tiles, no split)."""
    M, N, K = 8192, 1280, 640
    a = _r(M, K, seed=11).to(DEV)
    w = _r(N, K, seed=12, scale=K ** -0.5).to(DEV)
    bias = (torch.randn(N) * 0.1).to(DEV)
    r = _r(M, N, seed=13).to(DEV)
    full = ops.gemm(a, w, bias, residual=r)
    want = F.linear(a.float(), w.float(), bias) + r.float()
    assert rel_l2(full.float(), want) < 6e-3
    tail = ops.gemm(a[M - 768:].contiguous(), w, bias, residual=r[M - 768:].contiguous())
    assert torch.equal(full[M - 768:], tail)
    head = ops.gemm(a[:2048].contiguous(), w, bias, residual=r[:2048].contiguous())
    assert torch.equal(full[:2048], head)


@pytest.mark.parametrize("B,H,W,Cout", [(2, 16, 24, 64), (1, 17, 9, 320), (2, 32, 32, 512)])
def test_conv_in_as_im2col_gemm(ops, B, H, W, Cout):
    """conv_in (Cin = 4) on the tensor cores: ds_im2col_latent + ds_gemm_bf16 with weights.pack_conv_in."""
    from diffsensei_b200.weights import pack_conv_in
    g = torch.Generator().manual_seed(31)
    x = _r(B, H, W, 4, seed=30)
    w = (torch.randn(Cout, 4, 3, 3, generator=g) / 6).to(bf16).float()
    b = torch.randn(Cout, generator=g) * 0.1
    want = F.conv2d(x.float().permute(0, 3, 1, 2), w, b, padding=1).permute(0, 2, 3, 1)
    a = ops.im2col_latent(x.to(DEV))
    assert a.shape == (B * H * W, 64) and torch.count_nonzero(a[:, 36:]).item() == 0
    got = ops.gemm(a, pack_conv_in(w).to(DEV), b.to(DEV)).view(B, H, W, Cout)
    assert rel_l2(got.float(), want) < 6e-3


@pytest.mark.parametrize("B,H,W,Cin,Cout", [(2, 8, 16, 64, 64), (1, 9, 13, 128, 320), (2, 32, 32, 640, 640), (1, 19, 5, 64, 128)])
def test_conv3x3_fused_nearest_upsample(ops, B, H, W, Cin, Cout):
    """Upsample2D: conv3x3(F.interpolate(x, scale_factor=2, mode='nearest')) as four 2x2 phase convolutions of x
    (ds_conv3x3_nhwc upsample2): ragged patches, odd sizes, and the producer statistics accumulated over the 4 launches."""
    from diffsensei_b200.weights import pack_conv3x3_up2
    x = _r(B, H, W, Cin, seed=40)
    w = _r(Cout, Cin, 3, 3, seed=41, scale=(9 * Cin) ** -0.5)
    bias = torch.randn(Cout) * 0.1
    want = F.conv2d(F.interpolate(x.float().permute(0, 3, 1, 2), scale_factor=2.0, mode="nearest"), w.float(), bias,
                    padding=1).permute(0, 2, 3, 1)
    st = torch.zeros(B, Cout, 2, dtype=torch.float64, device=DEV)
    got = ops.conv3x3(x.to(DEV), pack_conv3x3_up2(w.float()).to(DEV), bias.to(DEV), chan_stats=st, upsample2=True)
    assert got.shape == (B, 2 * H, 2 * W, Cout)
    assert rel_l2(got.float(), want) < 8e-3            # + one bf16 rounding of the pre-summed taps
    assert torch.allclose(st.cpu(), _chan_stats_ref(got.cpu()), rtol=1e-5, atol=1e-3)


def _block_links(ops, C, M, seed):
    """The linears of one BasicTransformerBlock between its attention kernels, as (args, kwargs) lists for ops.gemm:
    attn2.to_out (+h, row stats) -> ff.net.0 (LayerNorm folded, GEGLU) -> ff.net.2 (+h, row stats) -> to_qkv (LN)."""
    from diffsensei_b200.weights import colsum_bf16, fold_layernorm, pack_geglu
    g = torch.Generator().manual_seed(seed)

    def lin(n, k, ln=False, geglu=False):
        w, b = torch.randn(n, k, generator=g) * k ** -0.5, torch.randn(n, generator=g) * 0.2
        if ln:
            w, b = fold_layernorm(w, b, torch.randn(k, generator=g) * 0.2 + 1, torch.randn(k, generator=g) * 0.1)
        if geglu:
            w, b = pack_geglu(w, b)
        w = w.to(bf16)
        return w.to(DEV), b.to(DEV), (colsum_bf16(w).to(DEV) if ln else None)

    a = (torch.randn(M, C, generator=g)).to(bf16).to(DEV)
    h0 = (torch.randn(M, C, generator=g) * 2 + 0.5).to(bf16).to(DEV)
    wo, bo, _ = lin(C, C)
    w1, b1, cs1 = lin(8 * C, C, ln=True, geglu=True)
    w2, b2, _ = lin(C, 4 * C)
    wq, bq, csq = lin(3 * C, C, ln=True)

    def build():
        h = h0.clone()
        st = [torch.zeros(2 * M, dtype=torch.float64, device=DEV) for _ in range(3)]
        qkv = torch.empty(M, 3 * C, dtype=bf16, device=DEV)
        links = [((a, wo, bo), dict(residual=h, out=h, row_stats_out=st[0], row_stats_zeroed=True)),
                 ((None, w1, b1), dict(epilogue=ops.EPI_GEGLU, ln_stats=st[0], ln_colsum=cs1, zero_rows=st[2])),
                 ((None, w2, b2), dict(residual=h, out=h, row_stats_out=st[1], row_stats_zeroed=True)),
                 ((None, wq, bq), dict(ln_stats=st[1], ln_colsum=csq, zero_rows=st[0], out=qkv))]
        return links, h, st
    return build


@pytest.mark.parametrize("C,M", [(640, 4096), (1280, 8192), (640, 128 * 5 + 40), (320, 1024)])
def test_gemm_chain_is_bit_identical_to_separate_launches(ops, C, M):
    """ds_gemm_chain: attn2.to_out -> ff.net.0 -> ff.net.2 -> to_qkv as ONE persistent launch with per-row-block
    dependency counters.  Outputs, intermediates and LayerNorm statistics must equal the four-launch sequence bit for
    bit, launch after launch (the kernel hands its counters back zeroed), including odd row-block counts."""
    build = _block_links(ops, C, M, seed=C + M)
    links, h_ref, st_ref = build()
    # the reference: the same four GEMMs as four launches of the same tile geometry (128 x 256 tiles; the row statistics
    # are fp64 sums of per-tile fp32 partials, so they depend — in the last bit — on the tile widths)
    prev, want = None, []
    for args, kw in links:
        n0 = launch_count()
        prev = ops.gemm_chain([((prev,) + args[1:] if args[0] is None else args, kw)], min_links=1)[0]
        assert launch_count() - n0 == 1
        want.append(prev.clone())
    # ... which agrees with the default schedule (mixed-width / 192-column tiles) to rounding
    links_d, h_d, _ = build()
    prev = None
    for args, kw in links_d:
        prev = ops.gemm(*((prev,) + args[1:] if args[0] is None else args), **kw)
    assert rel_l2(prev.float(), want[3].float()) < 2e-3 and rel_l2(h_d.float(), h_ref.float()) < 2e-3
    torch.cuda.synchronize()
    for it in range(6):
        links, h, st = build()
        n0 = launch_count()
        got = ops.gemm_chain(links)
        assert launch_count() - n0 == 1, "the chain must be ONE launch"
        torch.cuda.synchronize()
        assert torch.equal(got[1], want[1]), f"ff.net.0 output differs (iteration {it})"
        assert torch.equal(got[3], want[3]), f"to_qkv output differs (iteration {it})"
        assert torch.equal(h, h_ref), f"residual stream differs (iteration {it})"
        assert torch.equal(st[1], st_ref[1]) and torch.count_nonzero(st[0]).item() == 0
    # two-link chain (attn.to_out -> attn2.to_q) through the same counters
    links, h, st = build()
    two = ops.gemm_chain([links[0], ((None, links[3][0][1], links[3][0][2]),
                                     dict(ln_stats=st[0], ln_colsum=links[3][1]["ln_colsum"], zero_rows=st[2]))])
    links, h2, st2 = build()
    ops.gemm_chain([links[0]], min_links=1)
    ref = ops.gemm_chain([((h2, links[3][0][1], links[3][0][2]),
                           dict(ln_stats=st2[0], ln_colsum=links[3][1]["ln_colsum"]))], min_links=1)[0]
    assert torch.equal(two[1], ref)


def test_gemm_chain_falls_back_for_shapes_it_does_not_take(ops):
    a, w = _r(64, 128, seed=1).to(DEV), _r(128, 128, seed=2, scale=128 ** -0.5).to(DEV)
    n0 = launch_count()
    o = ops.gemm_chain([((a, w), {}), ((None, w), {})])          # M <= 128: two ordinary launches
    assert launch_count() - n0 == 2
    assert torch.equal(o[1], ops.gemm(ops.gemm(a, w), w))
