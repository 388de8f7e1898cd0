"""FreeU without a GPU: the oracle's Fourier filter against a numpy fp64 closed form, what ``apply_freeu`` touches, the
truthiness rule, the oracle forward with FreeU off, and the captured-stepper key."""
import numpy as np
import pytest
import torch

import freeu_oracle as F

SIDES = [1, 2, 3, 5, 12, 17, 64]


def _closed_form(x: np.ndarray, s: float) -> np.ndarray:
    """x - (1 - s) / (HW) Re sum over the DISTINCT frequencies {0, -1 mod H} x {0, -1 mod W} of X e^{+i...}."""
    H, W = x.shape[-2:]
    h = np.arange(H)[:, None]
    w = np.arange(W)[None, :]
    low = np.zeros(x.shape)
    for ky in sorted({0, (-1) % H}):
        for kx in sorted({0, (-1) % W}):
            e = np.exp(2j * np.pi * (ky * h / H + kx * w / W))
            X = (x * np.conj(e)).sum(axis=(-2, -1), keepdims=True)
            low += (X * e).real / (H * W)
    return x - (1 - s) * low


@pytest.mark.parametrize("H", SIDES)
@pytest.mark.parametrize("W", SIDES)
def test_oracle_fourier_filter_equals_the_closed_form(H, W):
    g = torch.Generator().manual_seed(H * 100 + W)
    x = torch.randn(2, 3, H, W, generator=g) + 0.5              # a mean, so the zero frequency matters
    got = F.fourier_filter(x, threshold=1, scale=0.2)
    want = _closed_form(x.double().numpy(), 0.2)
    assert got.dtype == x.dtype
    np.testing.assert_allclose(got.double().numpy(), want, rtol=0, atol=2e-5)
    # a side of 1 is not the identity: the zero frequency is still scaled
    assert not torch.allclose(got, x, atol=1e-3)


def test_fourier_filter_of_bf16_runs_in_fp32_and_casts_back():
    x = torch.randn(1, 4, 8, 8).to(torch.bfloat16)
    got = F.fourier_filter(x, 1, 0.9)
    assert got.dtype == torch.bfloat16
    assert torch.equal(got, F.fourier_filter(x.float(), 1, 0.9).to(torch.bfloat16))


def test_apply_freeu_touches_up_blocks_0_and_1_and_half_the_hidden_channels():
    kw = dict(s1=0.9, s2=0.2, b1=1.3, b2=1.4)
    hid0, skip0 = torch.randn(2, 12, 5, 6), torch.randn(2, 8, 5, 6)
    for idx, b, s in ((0, 1.3, 0.9), (1, 1.4, 0.2)):
        hid, skip = F.apply_freeu(idx, hid0.clone(), skip0, **kw)
        assert torch.equal(hid[:, :6], hid0[:, :6] * b) and torch.equal(hid[:, 6:], hid0[:, 6:])
        assert torch.equal(skip, F.fourier_filter(skip0, 1, s))
    for idx in (2, 3):
        hid, skip = F.apply_freeu(idx, hid0.clone(), skip0, **kw)
        assert torch.equal(hid, hid0) and skip is skip0


def _tiny_oracle():
    import diffsensei_b200 as ds
    from oracle.unet import OracleUNet
    torch.manual_seed(0)
    return ds, OracleUNet(ds.TINY).eval()


def _tiny_inputs(ds, h=16, w=24):
    from test_engine_gpu import _inputs
    lat, ehs, pooled, time_ids, bbox, dialog = _inputs(ds.TINY, 1, h, w)
    return torch.cat([lat] * 2), 741, ehs, pooled, time_ids, bbox, h / w, dialog


def test_oracle_forward_with_freeu_off_is_unchanged():
    ds, oracle = _tiny_oracle()
    args = _tiny_inputs(ds)
    want = oracle(*args)
    with F.freeu(oracle, 0.9, 0.2, 1.3, 1.4):
        on = oracle(*args)
    assert torch.equal(oracle(*args), want)                    # disable_freeu restores the forward
    assert not torch.allclose(on, want, atol=1e-3)
    for zeroed in ((0.0, 0.2, 1.3, 1.4), (0.9, 0, 1.3, 1.4), (0.9, 0.2, 0.0, 1.4), (0.9, 0.2, 1.3, None)):
        with F.freeu(oracle, *zeroed):
            assert torch.equal(oracle(*args), want), zeroed


def test_oracle_freeu_filters_the_six_skips_of_up_blocks_0_and_1(monkeypatch):
    """With the filter recorded and replaced by the identity and b = 1, the wrapped forward is the plain forward bit
    for bit (split / cat): FreeU reaches the oracle only through those six skips."""
    ds, oracle = _tiny_oracle()
    args = _tiny_inputs(ds, 18, 27)
    want = oracle(*args)
    seen = []
    monkeypatch.setattr(F, "fourier_filter", lambda x, threshold, scale: seen.append((tuple(x.shape), scale)) or x)
    with F.freeu(oracle, 0.9, 0.2, 1.0, 1.0):
        got = oracle(*args)
    assert torch.equal(got, want)
    # latent 18 x 27: up-block 0 runs at 5 x 7, up-block 1 at 9 x 14 (the need_size path)
    assert seen == [((2, 256, 5, 7), 0.9), ((2, 256, 5, 7), 0.9), ((2, 128, 5, 7), 0.9),
                    ((2, 128, 9, 14), 0.2), ((2, 128, 9, 14), 0.2), ((2, 64, 9, 14), 0.2)]


def _engine():
    import diffsensei_b200 as ds
    return ds, ds.UNetMangaEngine(ds.TINY, device="cpu")


def test_engine_freeu_truthiness():
    _ds, eng = _engine()
    assert eng.freeu is None
    eng.enable_freeu(0.9, 0.2, 1.3, 1.4)
    assert eng.freeu == (0.9, 0.2, 1.3, 1.4)
    for zeroed in ((0.0, 0.2, 1.3, 1.4), (0.9, 0.2, 1.3, 0), (None, 0.2, 1.3, 1.4)):
        eng.enable_freeu(*zeroed)
        assert eng.freeu is None, zeroed
    eng.enable_freeu(0.9, 0.2, 1.3, 1.4)
    eng.disable_freeu()
    assert eng.freeu is None


def test_freeu_pool_slots_cover_every_site():
    ds, eng = _engine()
    assert eng._freeu_pool_slots() == 6 + 6 + 4 + 4 + 3 + 2        # TINY has SDXL's channel ratios
    sdxl = ds.UNetMangaEngine(ds.SDXL_MANGA, device="cpu")
    assert sdxl._freeu_pool_slots() == 25


def test_stepper_key_holds_the_freeu_values(monkeypatch):
    ds, eng = _engine()
    monkeypatch.setattr(eng, "_ip_weights_version", lambda: 0)
    pipe = ds.DiffSenseiPipeline(eng)
    lat, pe = torch.zeros(1, 4, 16, 24), torch.zeros(2, 157, 128)
    key = lambda: pipe.stepper_key(lat, pe, 16 / 24, None, 4, 7.5)
    off = key()
    pipe.enable_freeu(0.9, 0.2, 1.3, 1.4)
    on = key()
    pipe.enable_freeu(0.9, 0.2, 1.3, 1.5)
    other = key()
    pipe.enable_freeu(0.9, 0.0, 1.3, 1.5)
    assert key() == off
    pipe.enable_freeu(0.9, 0.2, 1.3, 1.4)
    assert key() == on
    pipe.disable_freeu()
    assert key() == off
    assert len({off, on, other}) == 3
