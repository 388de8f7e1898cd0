"""img2img on the H100: the VAE image preprocessing kernel against Pillow bit for bit, the posterior kernel against a
torch fp32 restatement, the encoder's Downsample2D padding, the encoder against the fp32 oracle (oracle/vae_encoder.py)
at TINY and SDXL widths, batch-row independence, ``__call__(image=...)`` against a composition of its public pieces,
``generate_page`` img2img panels against their solo calls, and a short TINY img2img loop against the oracle loop.
Tolerances: encoder ``mean`` rel-L2 <= 3e-2 (bf16 activations, fp32 accumulation / normalisation, BASELINE.md §3);
posterior kernel <= 1e-6 relative (mode() exact)."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from conftest import rel_l2
from test_image_processor_gpu import _tiny_pipeline
from test_img2img_host import SIZES, _diffusers_arith, _image

pytestmark = pytest.mark.gpu
bf16, f32 = torch.bfloat16, torch.float32
DEV = "cuda"


def _encoder_pair(cfg_e, cfg_o, seed=0):
    import diffsensei_b200 as ds
    from diffsensei_b200.weights import random_state_dict, vae_encoder_param_shapes
    from oracle.vae_encoder import OracleVaeEncoder
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    sd = random_state_dict(vae_encoder_param_shapes(cfg_e), seed=seed, device="cpu")
    sd = {k: v.to(bf16).float() for k, v in sd.items()}
    oracle = OracleVaeEncoder(cfg_o).to(DEV).eval()
    oracle.load_state_dict(sd)
    eng = ds.VaeEncoderEngine(cfg_e, DEV)
    eng.load_state_dict(sd)
    return oracle, eng


def _chunked_attention(att):
    """The oracle's mid-block attention, the same fp32 arithmetic in query chunks (no [N, N] buffer at 2048²)."""
    def forward(x):
        b, c, h, w = x.shape
        hs = att.group_norm(x).reshape(b, c, h * w).transpose(1, 2)
        q, k, v = att.to_q(hs), att.to_k(hs), att.to_v(hs)
        o = torch.cat([torch.softmax(q[:, i:i + 4096] @ k.transpose(1, 2) / c ** 0.5, dim=-1) @ v
                       for i in range(0, h * w, 4096)], dim=1)
        return att.to_out[0](o).transpose(1, 2).reshape(b, c, h, w) + x
    att.forward = forward


# ------------------------------------------------------------------------------------------ kernels
@pytest.mark.parametrize("src,dst", SIZES)
def test_preprocess_kernel_equals_pillow(src, dst):
    from diffsensei_b200 import VaeImageProcessor
    im = _image(*src, seed=src[0])
    h, w = dst if dst else (None, None)
    want = torch.from_numpy(_diffusers_arith(im, h, w))
    proc = VaeImageProcessor()
    got = proc.preprocess(im, h, w).cpu()
    assert got.shape == want.shape and torch.equal(got, want)
    x4 = proc.preprocess_nhwc4(im, h, w).cpu()
    assert torch.equal(x4[..., :3], want.permute(0, 2, 3, 1).to(bf16)) and not x4[..., 3].float().any()


@pytest.mark.parametrize("mode", ["L", "RGBA"])
def test_preprocess_kernel_other_modes(mode):
    from diffsensei_b200 import VaeImageProcessor
    im = _image(133, 171, mode, seed=3)
    assert torch.equal(VaeImageProcessor().preprocess(im, 128, 176).cpu(),
                       torch.from_numpy(_diffusers_arith(im, 128, 176)))


def test_preprocess_float_tensors_follow_diffusers_rule():
    from diffsensei_b200 import VaeImageProcessor
    proc = VaeImageProcessor()
    x = torch.rand(1, 3, 64, 40, generator=torch.Generator().manual_seed(0))
    assert torch.equal(proc.preprocess(x).cpu(), 2.0 * x - 1.0)
    y = x * 2 - 1
    assert torch.equal(proc.preprocess(y).cpu(), y)


def test_posterior_kernel_matches_torch():
    from diffsensei_b200 import ops
    g = torch.Generator().manual_seed(1)
    B, h, w, R = 2, 9, 13, 3
    x = torch.randn(B, h, w, 8, generator=g, dtype=torch.float64) * 3
    x[0, 0, 0, 4:] = 40.0                                                  # logvar clamps at both ends
    x[0, 0, 1, 4:] = -50.0
    wq, bq = torch.randn(8, 8, generator=g, dtype=torch.float64) * 0.5, torch.randn(8, generator=g, dtype=torch.float64)
    wq[4:, :] = torch.eye(8, dtype=torch.float64)[4:] * 1.0                 # logvar rows pass the extreme values
    eps = torch.randn(B, 4, h, w, generator=g)
    noise = torch.randn(B * R, 4, h, w, generator=g)
    coef = torch.tensor([0.8, 0.6])
    d = lambda t: t.to(DEV).float().contiguous()
    mean, logvar, out = ops.vae_posterior(d(x), d(wq), d(bq), eps=d(eps), scale=0.13025, noise=d(noise), coef=d(coef),
                                          repeat=R, want_mean=True, want_logvar=True)
    m = torch.einsum("bhwc,kc->bkhw", x.float().double(), wq.float().double()) + bq.float().double()[None, :, None, None]
    mu, lv = m[:, :4], m[:, 4:].clamp(-30, 20)
    assert rel_l2(mean, mu) < 1e-6 and rel_l2(logvar, lv) < 1e-6
    assert float(logvar.max()) == 20.0 and float(logvar.min()) == -30.0
    # from the kernel's own mean / logvar, the rest is torch's fp32 eager arithmetic, bit for bit
    z = 0.13025 * (mean.cpu() + torch.exp(0.5 * logvar.cpu()) * eps)
    zr = torch.cat([z[b:b + 1].repeat(R, 1, 1, 1) for b in range(B)])
    assert rel_l2(out, coef[0] * zr + coef[1] * noise) < 1e-6
    _, _, mode = ops.vae_posterior(d(x), d(wq), d(bq))
    assert torch.equal(mode, mean)


@pytest.mark.parametrize("H,W", [(16, 24), (40, 8), (17, 9)])
def test_downsample_padding_matches_torch(H, W):
    from diffsensei_b200 import ops
    from diffsensei_b200.weights import pack_conv3x3
    g = torch.Generator().manual_seed(H)
    x = torch.randn(2, 64, H, W, generator=g).to(bf16)
    wt, b = (torch.randn(128, 64, 3, 3, generator=g) * 0.05).to(bf16), torch.randn(128, generator=g)
    want = F.conv2d(F.pad(x.float(), (0, 1, 0, 1)), wt.float(), b, stride=2).permute(0, 2, 3, 1)
    got = ops.conv3x3(x.permute(0, 2, 3, 1).contiguous().to(DEV), pack_conv3x3(wt.to(DEV)), b.to(DEV), stride=2,
                      pad_bottom_right=True, out_fp32=True).cpu()
    assert got.shape == want.shape == (2, H // 2, W // 2, 128) and rel_l2(got, want) < 1e-5


# ------------------------------------------------------------------------------------------ encoder
@pytest.mark.parametrize("H,W", [(64, 96), (216, 312)])
def test_tiny_encoder_matches_oracle(H, W):
    import diffsensei_b200 as ds
    from oracle.vae import TINY_VAE
    oracle, eng = _encoder_pair(ds.TINY_VAE, TINY_VAE, seed=1)
    x = (torch.rand(2, 3, H, W, generator=torch.Generator().manual_seed(2)) * 2 - 1).to(bf16).float().to(DEV)
    want = oracle.encode(x)
    got = eng.encode(x).latent_dist
    assert got.mean.shape == (2, 4, H // 8, W // 8)
    assert rel_l2(got.mean, want.mean) < 3e-2 and rel_l2(got.logvar, want.logvar) < 3e-2
    assert torch.equal(got.mode(), got.mean)
    s = got.sample(torch.Generator().manual_seed(4))
    eps = torch.randn(got.mean.shape, generator=torch.Generator().manual_seed(4)).to(DEV)
    assert rel_l2(s, got.mean + got.std * eps) < 1e-6


@pytest.mark.parametrize("H,W", [(512, 512), (216, 312), (2048, 2048)])
def test_sdxl_encoder_matches_oracle(H, W):
    import diffsensei_b200 as ds
    from oracle.vae import SDXL_VAE
    oracle, eng = _encoder_pair(ds.SDXL_VAE, SDXL_VAE, seed=3)
    _chunked_attention(oracle.encoder.mid_block.attentions[0])
    x = (torch.rand(1, 3, H, W, generator=torch.Generator().manual_seed(5)) * 2 - 1).to(bf16).float().to(DEV)
    want = oracle.encode(x).mean
    got = eng.encode(x).latent_dist.mean
    err = rel_l2(got, want)
    print(f"SDXL-size VAE encode {H}x{W} vs fp32 oracle: mean rel-L2 {err:.3e}")
    assert got.shape == (1, 4, H // 8, W // 8) and err < 3e-2


def test_encoder_rows_do_not_depend_on_the_batch():
    import diffsensei_b200 as ds
    from diffsensei_b200.weights import random_state_dict, vae_encoder_param_shapes
    eng = ds.VaeEncoderEngine(ds.SDXL_VAE, DEV)
    eng.load_state_dict(random_state_dict(vae_encoder_param_shapes(ds.SDXL_VAE), 6, DEV))
    g = torch.Generator().manual_seed(7)
    for H, W in ((128, 128), (216, 312)):
        x = (torch.rand(3, H, W, 4, generator=g) * 2 - 1).to(bf16)
        x[..., 3] = 0
        x = x.to(DEV)
        both = eng.moments_nhwc(x)
        for r in range(3):
            assert torch.equal(both[r:r + 1], eng.moments_nhwc(x[r:r + 1].contiguous())), (H, W, r)


# ------------------------------------------------------------------------------------------ pipeline
@pytest.fixture(scope="module")
def pipe(tmp_path_factory):
    import diffsensei_b200 as ds
    from diffsensei_b200.weights import random_state_dict, vae_decoder_param_shapes, vae_encoder_param_shapes
    torch.cuda.set_device(0)
    p, _, _ = _tiny_pipeline(tmp_path_factory.mktemp("tok"))
    vae = ds.VaeDecoderEngine(ds.TINY_VAE, DEV)
    vae.load_state_dict({k: v.to(bf16).float()
                         for k, v in random_state_dict(vae_decoder_param_shapes(ds.TINY_VAE), 2, "cpu").items()})
    enc = ds.VaeEncoderEngine(ds.TINY_VAE, DEV)
    enc.load_state_dict({k: v.to(bf16).float()
                         for k, v in random_state_dict(vae_encoder_param_shapes(ds.TINY_VAE), 3, "cpu").items()})
    p.vae, p.vae_encoder = vae, enc
    return p


@pytest.mark.parametrize("sched", ["ddim", "euler"])
@pytest.mark.parametrize("strength,ns", [(0.6, 1), (0.3, 2), (1.0, 1)])
def test_call_equals_its_public_pieces(pipe, sched, strength, ns):
    import diffsensei_b200 as ds
    pipe.scheduler = ds.EulerDiscreteScheduler() if sched == "euler" else ds.DDIMScheduler()
    im = _image(150, 200, seed=9)
    steps = 5
    rec = {}
    orig = pipe.denoise

    def spy(latents, *a, **k):
        rec.update(lat=latents.clone(), a=a, k=k)
        return orig(latents, *a, **k)
    pipe.denoise = spy
    try:
        out = pipe(prompt="a panel", image=im, strength=strength, num_inference_steps=steps, num_samples=ns,
                   generator=torch.Generator().manual_seed(11))
    finally:
        del pipe.denoise
    t_start, n_run = ds.get_timesteps(steps, strength)
    g = torch.Generator().manual_seed(11)
    sch = pipe.scheduler
    sch.set_timesteps(steps)
    x4 = pipe.vae_image_processor.preprocess_nhwc4(im)
    assert x4.shape == (1, 144, 200, 4)
    init = pipe.vae_encoder.encode_latents(x4, g, ns)                      # first draw
    noise = torch.randn(init.shape, generator=g).to(DEV)                   # second draw
    sch.set_begin_index(t_start)
    lat = sch.add_noise(init, noise, torch.tensor([sch.timesteps[t_start]] * ns))
    assert torch.equal(rec["lat"], lat) and rec["k"]["start_index"] == t_start
    st = pipe.make_stepper(lat, *rec["a"][:-2], num_inference_steps=steps, guidance_scale=rec["a"][-1],
                           use_graph=False, start_index=t_start)
    assert st.timesteps == sch.set_timesteps(steps)[t_start:] and len(st.timesteps) == n_run
    for i in range(n_run):
        st.step(i)
    assert torch.equal(st.latents_nchw(), out.latents)
    assert out.latents.shape == (ns, 4, 18, 25)
    pipe.scheduler = ds.DDIMScheduler()


def test_new_keywords_leave_text_to_image_alone(pipe):
    import diffsensei_b200 as ds
    kw = dict(prompt="a panel", height=128, width=192, num_inference_steps=3, generator=None)
    a = pipe(**{**kw, "generator": torch.Generator().manual_seed(1)}).latents
    enc, pipe.vae_encoder = pipe.vae_encoder, None
    try:
        b = pipe(**{**kw, "generator": torch.Generator().manual_seed(1)}).latents
    finally:
        pipe.vae_encoder = enc
    assert torch.equal(a, b)
    assert isinstance(pipe.scheduler, ds.DDIMScheduler)


def _img_panels():
    gen = lambda s: torch.Generator().manual_seed(s)
    return [
        dict(prompt="one", height=128, width=192, generator=gen(0)),
        dict(prompt="two", image=_image(128, 192, seed=1), generator=gen(1)),
        dict(prompt="three", image=_image(300, 200, seed=2), height=224, width=312, num_samples=2, generator=gen(2)),
        dict(prompt="four", height=224, width=312, generator=gen(3)),
        dict(prompt="five", image=_image(200, 100, seed=4), height=128, width=192, generator=gen(4)),
        dict(prompt="six", image=torch.rand(1, 3, 224, 312, generator=gen(9)), generator=gen(5)),
    ]


@pytest.mark.parametrize("use_graph", [True, False])
def test_page_img2img_panels_equal_their_solo_calls(pipe, use_graph):
    page = dict(num_inference_steps=4, guidance_scale=7.5, output_type="pt", strength=0.6, use_graph=use_graph)
    got = pipe.generate_page(_img_panels(), **page)
    assert [tuple(g.latents.shape) for g in got] == [(1, 4, 16, 24), (1, 4, 16, 24), (2, 4, 28, 39), (1, 4, 28, 39),
                                                     (1, 4, 16, 24), (1, 4, 28, 39)]
    for i, (g, p) in enumerate(zip(got, _img_panels())):
        want = pipe(**p, **page)
        assert torch.equal(g.latents, want.latents) and torch.equal(g.images, want.images), i


def test_page_img2img_with_agent(pipe, monkeypatch):
    import test_page_gpu
    from test_page_gpu import _agent, _result_generation, _stub_tokenizer
    from test_image_processor_host import make_image
    PAGE = dict(test_page_gpu.PAGE, num_inference_steps=4)                  # strength 0.3 of 4 steps: 1 step
    monkeypatch.setattr(test_page_gpu, "PAGE", PAGE)                       # the solo calls of _result_generation
    tok = _stub_tokenizer()
    agent = _agent(tok.SPACE)
    panels = lambda: [dict(prompt="a panel one", height=128, width=192, ip_images=[make_image(180, 260, seed=1)],
                           ip_bbox=[[.1, .1, .5, .9]], generator=torch.Generator().manual_seed(0),
                           image=_image(128, 192, seed=6)),
                      dict(prompt="a panel two", height=128, width=192, generator=torch.Generator().manual_seed(1))]
    got = pipe.generate_page(panels(), agent=agent, tokenizer_mllm=tok, max_new_tokens=67, **PAGE)
    for i, (g, p) in enumerate(zip(got, panels())):
        want = _result_generation(pipe, tok, agent, p, 0.4, 67)
        assert torch.equal(g.latents, want.latents) and torch.equal(g.images, want.images), i


# ------------------------------------------------------------------------------------------ loop vs oracle
@pytest.mark.parametrize("sched", ["ddim", "euler"])
def test_tiny_img2img_loop_matches_oracle(sched):
    """Engine UNet + encoder against the oracle UNet + encoder + img2img restatement over a 4-step loop at strength
    0.75 (3 steps run), within the existing loop bound (final latents rel-L2 <= 3e-2)."""
    import diffsensei_b200 as ds
    from oracle import img2img as oi
    from oracle.ddim import DDIMSchedule
    from oracle.euler import EulerSchedule
    from oracle.unet import OracleUNet
    from oracle.vae import TINY_VAE
    torch.manual_seed(0)
    cfg = ds.TINY
    ounet = OracleUNet(cfg).eval().to(DEV)
    ounet.set_ip_scale(0.6)
    unet = ds.UNetMangaEngine(cfg, DEV)
    unet.load_state_dict({k: v.cpu() for k, v in ounet.state_dict().items()})
    oenc, enc = _encoder_pair(ds.TINY_VAE, TINY_VAE, seed=4)
    pipe = ds.DiffSenseiPipeline(unet, vae_encoder=enc,
                                 scheduler=ds.EulerDiscreteScheduler() if sched == "euler" else None)
    pipe.set_ip_scale(0.6)
    g = torch.Generator().manual_seed(1)
    ehs = torch.randn(2, 77 + 80, cfg.cross_attention_dim, generator=g).to(DEV)
    pooled = torch.randn(2, cfg.pooled_text_dim, generator=g).to(DEV)
    time_ids = torch.tensor([[128.0, 192.0, 0, 0, 128.0, 192.0]] * 2, device=DEV)
    bbox = torch.zeros(2, cfg.max_num_ips, 4, device=DEV)
    steps, strength = 4, 0.75
    t_start, _ = ds.get_timesteps(steps, strength)
    im = _image(128, 192, seed=12)
    # oracle
    x = torch.from_numpy(oi.preprocess(np.array(im))).to(DEV)
    sch = EulerSchedule() if sched == "euler" else DDIMSchedule()
    ts = sch.set_timesteps(steps)
    if sched == "euler":
        add = lambda i, n: oi.euler_add_noise(sch.sigmas.to(DEV), i, n, t_start)
    else:
        add = lambda i, n: oi.ddim_add_noise(sch.alphas_cumprod.to(DEV), i, n, ts[t_start])
    lat_o = oi.prepare_latents(oenc.encode(x.to(bf16).float()), TINY_VAE.scaling_factor, 1, add,
                               torch.Generator().manual_seed(3))
    for t in ts[t_start:]:
        mi = torch.cat([lat_o] * 2)
        if sched == "euler":
            mi = sch.scale_model_input(mi, t)
        eu, et = ounet(mi, t, ehs, pooled, time_ids, bbox, 16 / 24, None).chunk(2)
        lat_o = sch.step(eu + 7.5 * (et - eu), t, lat_o)
    # engine
    pipe.scheduler.set_timesteps(steps)
    lat = enc.encode_latents(pipe.vae_image_processor.preprocess_nhwc4(im), torch.Generator().manual_seed(3), 1,
                             pipe.scheduler.add_noise_coefficients(t_start, DEV))
    got = pipe.denoise(lat, ehs, pooled, time_ids, bbox, 16 / 24, None, steps, 7.5, start_index=t_start)
    err = rel_l2(got, lat_o)
    print(f"TINY img2img {sched} vs oracle: rel-L2 {err:.3e}")
    assert err < 3e-2
