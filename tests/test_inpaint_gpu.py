"""Inpainting on the H100: the mask preprocessing kernel against Pillow bit for bit, the inpaint step kernels against
the plain step kernels and torch eager, ``__call__(image=..., mask_image=...)`` against a composition of its public
pieces, graph replay and a refilled cached stepper, ``generate_page`` inpaint panels against their solo calls, and a
short TINY inpaint loop against the oracle (oracle/inpaint.py) under DDIM and Euler."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from conftest import rel_l2
from test_image_processor_gpu import _tiny_pipeline
from test_img2img_host import _image
from test_inpaint_host import MASK_SIZES, _mask, _pillow_mask

pytestmark = pytest.mark.gpu
bf16, f32, u8 = torch.bfloat16, torch.float32, torch.uint8
DEV = "cuda"


def _mask_processor():
    from diffsensei_b200 import VaeImageProcessor
    return VaeImageProcessor(vae_scale_factor=8, do_normalize=False, do_binarize=True, do_convert_grayscale=True)


# ------------------------------------------------------------------------------------------ mask kernel
@pytest.mark.parametrize("mode", ["L", "RGB"])
@pytest.mark.parametrize("src,dst", MASK_SIZES)
def test_mask_kernel_equals_pillow(src, dst, mode):
    from oracle import inpaint as oi
    im = _mask(*src, mode=mode, seed=src[1])
    h, w = dst if dst else (None, None)
    want = torch.from_numpy(_pillow_mask(im, h, w))
    proc = _mask_processor()
    got = proc.preprocess(im, h, w).cpu()
    assert got.shape == want.shape and torch.equal(got, want)
    assert torch.equal(got, torch.from_numpy(oi.mask_preprocess(np.array(im), h, w)))
    lat = proc.preprocess_latent_mask(im, h, w).cpu()
    assert lat.dtype == u8 and torch.equal(lat[None].float(), oi.latent_mask(want))
    arr = np.array(im)                                              # uint8 arrays / tensors are that PIL mode
    assert torch.equal(proc.preprocess(arr, h, w).cpu(), want)
    assert torch.equal(proc.preprocess(torch.from_numpy(arr).to(DEV), h, w).cpu(), want)


def test_float_masks_are_binarised_at_size():
    proc = _mask_processor()
    x = torch.rand(1, 1, 64, 40, generator=torch.Generator().manual_seed(0))
    x[0, 0, 0, :4] = torch.tensor([0.5, 0.49999997, 0.0, 1.0])
    want = (x >= 0.5).float()
    assert torch.equal(proc.preprocess(x).cpu(), want)
    assert torch.equal(proc.preprocess(x[0, 0].to(DEV), 64, 40).cpu(), want)
    assert torch.equal(proc.preprocess_latent_mask(x).cpu()[None].float(), want[..., ::8, ::8])


# ------------------------------------------------------------------------------------------ step kernels
def _step_inputs(bs, h, w, seed):
    g = torch.Generator().manual_seed(seed)
    eps = (torch.randn(2 * bs, h, w, 4, generator=g)).to(bf16).to(DEV)
    lat = (torch.randn(bs, h, w, 4, generator=g) * 3).to(DEV)
    z = torch.randn(bs, h, w, 4, generator=g).to(DEV)
    n = torch.randn(bs, h, w, 4, generator=g).to(DEV)
    rnd = (torch.rand(bs, h, w, generator=g) < 0.5).to(u8).to(DEV)
    return eps, lat, z, n, rnd


@pytest.mark.parametrize("sched", ["ddim", "euler"])
@pytest.mark.parametrize("bs,h,w", [(1, 9, 13), (2, 16, 19), (3, 40, 37)])
def test_inpaint_step_kernels(sched, bs, h, w):
    import diffsensei_b200 as ds
    s = ds.EulerDiscreteScheduler() if sched == "euler" else ds.DDIMScheduler()
    s.set_timesteps(10)
    tab = s.inpaint_coefficient_table(0, DEV)
    for i in (0, 6, 9):                                             # 9: the last step, {c0, c1} = {1, 0}
        coef = tab[i].contiguous()
        plain_coef = coef[:-2].contiguous()
        eps, lat0, z, n, rnd = _step_inputs(bs, h, w, seed=100 * bs + i)
        lat_p, mi_p = lat0.clone(), torch.zeros(2 * bs, h, w, 4, dtype=bf16, device=DEV)
        s.fused_step_(eps, lat_p, mi_p, plain_coef, 7.5)
        init = coef[-2] * z + coef[-1] * n                          # torch eager add_noise arithmetic
        if i == 9:
            assert torch.equal(init, z)
        div = coef[2] if sched == "euler" else None
        mi_init = (init / div if div is not None else init).to(bf16)
        for name, m in (("ones", torch.ones_like(rnd)), ("zeros", torch.zeros_like(rnd)), ("random", rnd)):
            lat, mi = lat0.clone(), torch.zeros(2 * bs, h, w, 4, dtype=bf16, device=DEV)
            s.fused_inpaint_step_(eps, lat, mi, coef, 7.5, z, n, m)
            keep = m.bool()[..., None]
            want_lat = torch.where(keep, lat_p, init)
            want_mi = torch.where(keep, mi_p[:bs], mi_init)
            assert torch.equal(lat, want_lat), (name, i)
            assert torch.equal(mi[:bs], want_mi) and torch.equal(mi[bs:], want_mi), (name, i)
            if name == "ones":
                assert torch.equal(lat, lat_p) and torch.equal(mi, mi_p)


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


def _composed(pipe, im, mask_im, strength, ns, steps, seed, rec):
    """The inpaint call restated from public pieces: the processors, ``encode_latents`` (draw a), the latent noise
    (draw b), the dropped masked-image draw (c), ``add_noise``, then the PLAIN stepper with the blend and the next UNet
    input redone in torch eager after every step."""
    import diffsensei_b200 as ds
    g = torch.Generator().manual_seed(seed)
    sch = pipe.scheduler
    ts = sch.set_timesteps(steps)
    t_start, n_run = ds.get_timesteps(steps, strength)
    x4 = pipe.vae_image_processor.preprocess_nhwc4(im)
    h, w = x4.shape[1] // 8, x4.shape[2] // 8
    z = pipe.vae_encoder.encode_latents(x4, g, ns)                          # (a)
    noise = torch.randn(z.shape, generator=g).to(DEV)                       # (b)
    torch.randn(1, 4, h, w, generator=g)                                    # (c)
    sch.set_begin_index(t_start)
    lat = noise * sch.init_noise_sigma if strength == 1.0 else \
        sch.add_noise(z, noise, torch.tensor([ts[t_start]] * ns))
    sch.begin_index = None                          # in the loop diffusers' Euler add_noise reads the step index
    mask = pipe.mask_processor.preprocess(mask_im, x4.shape[1], x4.shape[2])
    m = F.interpolate(mask, size=(h, w)).repeat(ns, 1, 1, 1)
    assert torch.equal(rec["lat"], lat) and rec["k"]["start_index"] == t_start
    z_r, n_r, m_r = rec["k"]["inpaint"]
    assert torch.equal(z_r, z) and torch.equal(n_r, noise) and torch.equal(m_r.float(), m[:, 0])
    st = pipe.make_stepper(lat, *rec["a"][:-2], num_inference_steps=steps, guidance_scale=rec["a"][-1],
                           use_graph=False, start_index=t_start)
    for i in range(n_run):
        st.step(i)
        x = st.latents_nchw()
        k = t_start + i
        init = sch.add_noise(z, noise, torch.tensor([ts[k + 1]] * ns)) if i < n_run - 1 else z
        x = (1 - m) * init + m * x
        st.lat.copy_(x.permute(0, 2, 3, 1))
        if i < n_run - 1:
            mi = (x.permute(0, 2, 3, 1) / st.in_div[i + 1]).to(bf16)
            st.model_in[:ns].copy_(mi)
            st.model_in[ns:].copy_(mi)
    return st.latents_nchw(), g


@pytest.mark.parametrize("sched", ["ddim", "euler"])
@pytest.mark.parametrize("strength,ns", [(0.6, 1), (1.0, 1), (0.6, 2)])
def test_call_equals_its_public_pieces(pipe, sched, strength, ns):
    import diffsensei_b200 as ds
    pipe.scheduler = ds.EulerDiscreteScheduler() if sched == "euler" else ds.DDIMScheduler()
    im, mask_im = _image(150, 200, seed=9), _mask(100, 120, mode="RGB", seed=5)
    steps, rec = 5, {}
    orig = pipe.denoise

    def spy(latents, *a, **k):
        rec.update(lat=latents.clone(), a=a, k=k)
        return orig(latents, *a, **k)
    pipe.denoise = spy
    g_call = torch.Generator().manual_seed(11)
    try:
        out = pipe(prompt="a panel", image=im, mask_image=mask_im, strength=strength, num_inference_steps=steps,
                   num_samples=ns, generator=g_call)
    finally:
        del pipe.denoise
    try:
        want, g = _composed(pipe, im, mask_im, strength, ns, steps, 11, rec)
        assert torch.equal(g_call.get_state(), g.get_state())             # the generator ends where diffusers' does
        assert out.latents.shape == (ns, 4, 18, 25) and torch.equal(out.latents, want)
        keep = rec["k"]["inpaint"][2] == 0                                  # unmasked pixels end as the image latents
        z = rec["k"]["inpaint"][0]
        assert keep.any() and torch.equal(out.latents.permute(0, 2, 3, 1)[keep], z.permute(0, 2, 3, 1)[keep])
    finally:
        pipe.scheduler = ds.DDIMScheduler()


def _inpaint_rows(pipe, seed, h=16, w=24):
    g = torch.Generator().manual_seed(seed)
    z, n = torch.randn(2, 4, h, w, generator=g).to(DEV), torch.randn(2, 4, h, w, generator=g).to(DEV)
    m = (torch.rand(2, h, w, generator=g) < 0.4).to(u8).to(DEV)
    return z + n, (z, n, m)


def test_graph_replay_and_refilled_stepper(pipe):
    cfg = pipe.unet.cfg
    g = torch.Generator().manual_seed(3)
    cond = lambda: (torch.randn(4, 77 + 80, cfg.cross_attention_dim, generator=g).to(DEV),
                    torch.randn(4, cfg.pooled_text_dim, generator=g).to(DEV))
    time_ids = torch.tensor([[128.0, 192.0, 0, 0, 128.0, 192.0]] * 4, device=DEV)
    bbox = torch.zeros(4, cfg.max_num_ips, 4, device=DEV)
    pipe._steppers.clear()
    for sched_seed, (lat, inp) in enumerate((_inpaint_rows(pipe, 1), _inpaint_rows(pipe, 2))):
        ehs, pooled = cond()
        args = (ehs, pooled, time_ids, bbox, 16 / 24, None, 4, 7.5)
        graph = pipe.denoise(lat, *args, use_graph=True, start_index=1, inpaint=inp)
        eager = pipe.denoise(lat, *args, use_graph=False, start_index=1, inpaint=inp)
        assert torch.equal(graph, eager), sched_seed
        assert len(pipe._steppers) == 1                                     # the second panel refilled the first
    plain = pipe.denoise(lat, *args, use_graph=True, start_index=1)
    assert len(pipe._steppers) == 2 and not torch.equal(plain, graph)      # the inpaint flag is in the key


def _page_panels():
    gen = lambda s: torch.Generator().manual_seed(s)
    return [
        dict(prompt="one", height=128, width=192, generator=gen(0)),
        dict(prompt="two", image=_image(128, 192, seed=1), mask_image=_mask(64, 96, seed=1), generator=gen(1)),
        dict(prompt="three", image=_image(300, 200, seed=2), height=224, width=312, num_samples=2,
             mask_image=_mask(300, 200, mode="RGB", seed=2), generator=gen(2)),
        dict(prompt="four", image=_image(200, 100, seed=4), height=128, width=192, generator=gen(4)),
        dict(prompt="five", image=_image(128, 192, seed=5), generator=gen(5),
             mask_image=(torch.rand(1, 1, 128, 192, generator=gen(8)) > 0.3).float()),
        dict(prompt="six", height=224, width=312, generator=gen(3)),
        dict(prompt="seven", image=torch.rand(1, 3, 224, 312, generator=gen(9)),
             mask_image=np.array(_mask(224, 312, seed=7)), generator=gen(6)),
    ]


@pytest.mark.parametrize("use_graph", [True, False])
def test_page_inpaint_panels_equal_their_solo_calls(pipe, use_graph):
    page = dict(num_inference_steps=4, guidance_scale=7.5, output_type="pt", strength=0.6, use_graph=use_graph)
    got = pipe.generate_page(_page_panels(), **page)
    assert [tuple(g.latents.shape) for g in got] == [(1, 4, 16, 24), (1, 4, 16, 24), (2, 4, 28, 39), (1, 4, 16, 24),
                                                     (1, 4, 16, 24), (1, 4, 28, 39), (1, 4, 28, 39)]
    for i, (g, p) in enumerate(zip(got, _page_panels())):
        want = pipe(**p, **page)
        assert torch.equal(g.latents, want.latents) and torch.equal(g.images, want.images), i


def test_page_inpaint_with_agent(pipe, monkeypatch):
    import test_page_gpu
    from test_page_gpu import _agent, _result_generation, _stub_tokenizer
    from test_image_processor_host import make_image
    PAGE = dict(test_page_gpu.PAGE, num_inference_steps=4)                  # strength 0.3 of 4 steps: 1 step
    monkeypatch.setattr(test_page_gpu, "PAGE", PAGE)                       # the solo calls of _result_generation
    tok = _stub_tokenizer()
    agent = _agent(tok.SPACE)
    panels = lambda: [dict(prompt="a panel one", height=128, width=192, ip_images=[make_image(180, 260, seed=1)],
                           ip_bbox=[[.1, .1, .5, .9]], generator=torch.Generator().manual_seed(0),
                           image=_image(128, 192, seed=6), mask_image=_mask(128, 192, seed=6)),
                      dict(prompt="a panel two", height=128, width=192, generator=torch.Generator().manual_seed(1))]
    got = pipe.generate_page(panels(), agent=agent, tokenizer_mllm=tok, max_new_tokens=67, **PAGE)
    for i, (g, p) in enumerate(zip(got, panels())):
        want = _result_generation(pipe, tok, agent, p, 0.4, 67)
        assert torch.equal(g.latents, want.latents) and torch.equal(g.images, want.images), i


def test_mask_support_leaves_text_to_image_and_img2img_alone(pipe):
    import diffsensei_b200 as ds
    kw = dict(prompt="a panel", height=128, width=192, num_inference_steps=4)
    im = _image(128, 192, seed=3)
    run = lambda **k: pipe(**kw, **k, generator=torch.Generator().manual_seed(1)).latents
    t2i, i2i = run(), run(image=im, strength=0.6)
    run(image=im, strength=0.6, mask_image=_mask(128, 192, seed=3))         # an inpaint stepper of the same shapes
    assert torch.equal(run(), t2i) and torch.equal(run(image=im, strength=0.6), i2i)
    assert torch.equal(run(image=im, strength=0.6, mask_image=None), i2i)
    proc, pipe.mask_processor = pipe.mask_processor, None
    try:
        assert torch.equal(run(), t2i) and torch.equal(run(image=im, strength=0.6), i2i)
    finally:
        pipe.mask_processor = proc
    assert isinstance(pipe.scheduler, ds.DDIMScheduler)


# ------------------------------------------------------------------------------------------ loop vs oracle
@pytest.mark.parametrize("sched", ["ddim", "euler"])
def test_tiny_inpaint_loop_matches_oracle(sched):
    """Engine UNet + encoder + inpaint step against the oracle UNet + encoder + inpaint restatement over a 4-step
    loop at strength 0.75 (3 steps run), within the existing loop bound (final latents rel-L2 <= 3e-2)."""
    import diffsensei_b200 as ds
    from oracle import img2img as oi2
    from oracle import inpaint as oi
    from oracle.ddim import DDIMSchedule
    from oracle.euler import EulerSchedule
    from oracle.unet import OracleUNet
    from oracle.vae import TINY_VAE
    from test_img2img_gpu import _encoder_pair
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
    im, mask_im = _image(128, 192, seed=12), _mask(128, 192, mode="RGB", seed=12)
    # oracle
    x = torch.from_numpy(oi2.preprocess(np.array(im))).to(DEV)
    m = oi.latent_mask(torch.from_numpy(oi.mask_preprocess(np.array(mask_im)))).to(DEV)
    sch = EulerSchedule() if sched == "euler" else DDIMSchedule()
    ts = sch.set_timesteps(steps)
    if sched == "euler":
        add = lambda z, n, k: oi2.euler_add_noise(sch.sigmas.to(DEV), z, n, k)
        sigma0 = sch.init_noise_sigma
    else:
        add = lambda z, n, k: oi2.ddim_add_noise(sch.alphas_cumprod.to(DEV), z, n, ts[k])
        sigma0 = 1.0
    lat_o, z_o, n_o = oi.prepare_latents(oenc.encode(x.to(bf16).float()), TINY_VAE.scaling_factor, 1, strength,
                                         lambda z, n: add(z, n, t_start), sigma0, torch.Generator().manual_seed(3))
    run = ts[t_start:]
    for i, t in enumerate(run):
        mi = torch.cat([lat_o] * 2)
        if sched == "euler":
            mi = sch.scale_model_input(mi, t)
        eu, et = ounet(mi, t, ehs, pooled, time_ids, bbox, 16 / 24, None).chunk(2)
        lat_o = sch.step(eu + 7.5 * (et - eu), t, lat_o)
        lat_o = oi.blend(lat_o, z_o, n_o, m, i, len(run), lambda z, n, j: add(z, n, t_start + j + 1))
    # engine
    pipe.scheduler.set_timesteps(steps)
    moments = enc.moments_nhwc(pipe.vae_image_processor.preprocess_nhwc4(im))
    eps, noise = pipe._draw_inpaint_noise(16, 24, 1, torch.Generator().manual_seed(3))
    mask = pipe.mask_processor.preprocess_latent_mask(mask_im)
    assert torch.equal(mask[:, None].float(), m)
    lat, inp = pipe._inpaint_start(moments, eps, noise, mask, 1, t_start, strength)
    got = pipe.denoise(lat, ehs, pooled, time_ids, bbox, 16 / 24, None, steps, 7.5, start_index=t_start, inpaint=inp)
    err = rel_l2(got, lat_o)
    print(f"TINY inpaint {sched} vs oracle: rel-L2 {err:.3e}")
    assert err < 3e-2
