"""Full-size parity on every BASELINE config (VERDICT r1 item 1): one engine forward at the REAL SDXL+IP topology
(2.9 B random weights shared by both sides) against the fp32 oracle, for

    cfg1  512x512,   1 ref                       (latent  64x64)          — also against the CPU run of the oracle
    cfg2  1024x1024, 2 refs                      (latent 128x128, one panel = UNet batch 2)
    cfg3  864x1216 and 704x368 buckets, 4 refs + 3 dialog boxes  (odd feature maps / derived-(H',W') quirk)
    cfg5  2048x1024, 3 refs, MLLM-adapted image tokens (latent 256x128, N = 8192 / 2048)

plus a 50-step cfg1 denoise drift curve and the yard-stick the tolerances are judged by: the SAME oracle modules
run in bf16 through torch's library kernels (what the reference's own bf16 GPU path computes) against the fp32 run.

The fp32 oracle runs ON THE GPU here (plain torch modules, TF32 off) because an SDXL forward on the box's host cores
costs minutes of leased GPU time; `test_gpu_fp32_oracle_equals_cpu_oracle` pins that run to the CPU oracle first.
Tolerances (BASELINE.md §3): UNet output rel-L2 <= 3e-2 per forward; 50-step final-latent drift <= 1e-1 and
reported.  With DS_PARITY_OUT=<dir> set, the measured errors are also written to <dir>/parity_full.json.
"""
import json
import os

import pytest
import torch

from conftest import ROOT, rel_l2

pytestmark = pytest.mark.gpu
bf16, f32 = torch.bfloat16, torch.float32
DEV = "cuda"
RESULTS = {}


def _dump():
    out = os.environ.get("DS_PARITY_OUT")
    if not out:
        return
    os.makedirs(out, exist_ok=True)
    with open(os.path.join(out, "parity_full.json"), "w") as f:
        json.dump(RESULTS, f, indent=1, sort_keys=True)


@pytest.fixture(scope="module")
def full():
    import diffsensei_b200 as ds
    from diffsensei_b200.weights import random_state_dict, unet_param_shapes
    from oracle.config import SDXL
    from oracle.unet import OracleUNet
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    cfg = ds.SDXL_MANGA
    sd = random_state_dict(unet_param_shapes(cfg), seed=7, device=DEV, dtype=bf16)
    with torch.device("meta"):
        oracle = OracleUNet(SDXL)
    oracle = oracle.to_empty(device=DEV)
    oracle.load_state_dict({k: v.float() for k, v in sd.items()})
    oracle.eval().set_ip_scale(0.6)
    engine = ds.UNetMangaEngine(cfg, DEV)
    engine.load_state_dict(sd)
    engine.set_ip_scale(0.6)
    yield ds, cfg, sd, oracle, engine
    _dump()


def _inputs(cfg, bs, h, w, n_chars, dialogs, mllm=False, seed=11):
    import bench
    torch.manual_seed(seed)
    lat, ehs, pooled, time_ids, bbox, dialog = bench.synthetic_inputs(cfg, bs, h, w, n_chars, "cpu", dialogs=dialogs,
                                                                      mllm=mllm)
    return lat, ehs.to(bf16).float(), pooled, time_ids, bbox, dialog


def _engine_forward(engine, x, t, ehs, pooled, time_ids, bbox, ar, dialog):
    return engine.forward(x.to(DEV), torch.tensor(t), ehs.to(DEV, bf16),
                          added_cond_kwargs={"text_embeds": pooled.to(DEV), "time_ids": time_ids.to(DEV)},
                          cross_attention_kwargs={"bbox": bbox.to(DEV), "aspect_ratio": ar},
                          dialog_bbox=None if dialog is None else dialog.to(DEV)).sample


def _oracle_forward(oracle, x, t, ehs, pooled, time_ids, bbox, ar, dialog, dtype=f32):
    c = lambda v: None if v is None else v.to(DEV, dtype)
    with torch.no_grad():
        # dialog boxes stay fp32 on every side: int(bbox * size) in bf16 can move a box edge by a pixel
        # (tests/golden/dialog_embed.pt covers that rule) — here only the arithmetic precision is compared
        return oracle(c(x), t, c(ehs), c(pooled), time_ids.to(DEV), bbox.to(DEV), ar,
                      None if dialog is None else dialog.to(DEV)).float()


def test_gpu_fp32_oracle_equals_cpu_oracle(full):
    """Pins the GPU run of the oracle (cuBLAS/cuDNN fp32, TF32 off) to its CPU run — the oracle proper — on the cfg1
    forward, and the engine against both.  Everything else in this file then uses the GPU run."""
    ds, cfg, sd, oracle, engine = full
    from oracle.config import SDXL
    from oracle.unet import OracleUNet
    lat, ehs, pooled, time_ids, bbox, dialog = _inputs(cfg, 1, 64, 64, 1, True)
    x = torch.cat([lat] * 2)
    if os.environ.get("DS_FULL_PARITY") == "0":
        pytest.skip("CPU run of the SDXL oracle (45 s, ~25 GB host RAM) disabled by DS_FULL_PARITY=0")
    with torch.device("meta"):
        cpu = OracleUNet(SDXL)
    cpu = cpu.to_empty(device="cpu")
    cpu.load_state_dict({k: v.float().cpu() for k, v in sd.items()})
    cpu.eval().set_ip_scale(0.6)
    with torch.no_grad():
        want_cpu = cpu(x, 741, ehs, pooled, time_ids, bbox, 1.0, dialog)
    del cpu
    want_gpu = _oracle_forward(oracle, x, 741, ehs, pooled, time_ids, bbox, 1.0, dialog)
    got = _engine_forward(engine, x, 741, ehs, pooled, time_ids, bbox, 1.0, dialog)
    d = rel_l2(want_gpu, want_cpu)
    RESULTS["cfg1_oracle_gpu_fp32_vs_cpu_fp32"] = d
    RESULTS["cfg1_engine_vs_cpu_oracle"] = rel_l2(got, want_cpu)
    RESULTS["cfg1_engine_vs_gpu_oracle"] = rel_l2(got, want_gpu)
    print(f"cfg1: oracle GPU-fp32 vs CPU-fp32 {d:.2e}; engine vs CPU oracle {RESULTS['cfg1_engine_vs_cpu_oracle']:.3e}")
    assert d < 2e-4
    assert RESULTS["cfg1_engine_vs_cpu_oracle"] < 3e-2


CASES = {
    # name: (bs, latent_h, latent_w, n_chars, dialogs, mllm)
    "cfg2_1024x1024_2refs": (1, 128, 128, 2, False, False),
    "cfg3_864x1216_4refs_dialogs": (1, 108, 152, 4, True, False),
    "cfg3_704x368_4refs_dialogs": (1, 88, 46, 4, True, False),
    "cfg5_2048x1024_3refs_mllm": (1, 256, 128, 3, False, True),
}


@pytest.mark.parametrize("name", list(CASES))
def test_full_size_forward_matches_oracle(full, name):
    """Engine (bf16 kernels) vs fp32 oracle on one panel (UNet batch 2 = its CFG pair) of each BASELINE config, and
    the bf16-library yard-stick: the same oracle modules in bf16 through torch's kernels vs the same fp32 run."""
    ds, cfg, sd, oracle, engine = full
    bs, h, w, n_chars, dialogs, mllm = CASES[name]
    lat, ehs, pooled, time_ids, bbox, dialog = _inputs(cfg, bs, h, w, n_chars, dialogs, mllm)
    x = torch.cat([lat] * 2)
    ar = h / w
    want = _oracle_forward(oracle, x, 521, ehs, pooled, time_ids, bbox, ar, dialog)
    got = _engine_forward(engine, x, 521, ehs, pooled, time_ids, bbox, ar, dialog)
    err = rel_l2(got, want)
    RESULTS[name] = {"engine_vs_fp32_oracle": err}
    print(f"{name}: engine vs fp32 oracle rel-L2 {err:.3e}")
    assert got.shape == x.shape and torch.isfinite(got).all()
    assert err < 3e-2


def test_bf16_library_yardstick(full):
    """What does the reference's OWN bf16 GPU path deviate by?  The oracle modules cast to bf16 (torch library kernels,
    explicit-softmax attention) vs their fp32 run, on the cfg1 and cfg2 panels — the number to read the engine's
    rel-L2 against.  The engine must not be worse than 1.5x this yard-stick (+ 5e-3)."""
    ds, cfg, sd, oracle, engine = full
    from oracle.config import SDXL
    from oracle.unet import OracleUNet
    with torch.device("meta"):
        o16 = OracleUNet(SDXL)
    o16 = o16.to_empty(device=DEV).to(bf16)
    o16.load_state_dict(sd)
    o16.eval().set_ip_scale(0.6)
    out = {}
    for name, (bs, h, w, n_chars, dialogs) in {"cfg1": (1, 64, 64, 1, True), "cfg2": (1, 128, 128, 2, False)}.items():
        lat, ehs, pooled, time_ids, bbox, dialog = _inputs(cfg, bs, h, w, n_chars, dialogs)
        x = torch.cat([lat] * 2)
        want = _oracle_forward(oracle, x, 521, ehs, pooled, time_ids, bbox, h / w, dialog)
        lib = _oracle_forward(o16, x, 521, ehs, pooled, time_ids, bbox, h / w, dialog, dtype=bf16)
        got = _engine_forward(engine, x, 521, ehs, pooled, time_ids, bbox, h / w, dialog)
        out[name] = {"bf16_library_vs_fp32": rel_l2(lib, want), "engine_vs_fp32": rel_l2(got, want),
                     "engine_vs_bf16_library": rel_l2(got, lib)}
        print(name, {k: f"{v:.3e}" for k, v in out[name].items()})
        assert out[name]["engine_vs_fp32"] < 1.5 * out[name]["bf16_library_vs_fp32"] + 5e-3
    RESULTS["bf16_yardstick"] = out
    del o16


def test_50_step_drift_cfg1(full):
    """BASELINE.md §3: final-latent drift over a whole denoise loop.  cfg1 panel (512x512, 1 ref), 50 DDIM steps,
    CFG 7.5, full topology: engine loop (graph replay, fused CFG+DDIM) vs the oracle loop in fp32; the bf16-library
    loop is run beside it as the yard-stick.  Bound: the engine's final-latent rel-L2 <= 1e-1 and <= 2x the
    bf16-library loop's own drift + 1e-2."""
    ds, cfg, sd, oracle, engine = full
    from oracle.config import SDXL
    from oracle.ddim import denoise_loop
    from oracle.unet import OracleUNet
    h = w = 64
    lat, ehs, pooled, time_ids, bbox, dialog = _inputs(cfg, 1, h, w, 1, True, seed=23)
    T, g = 50, 7.5
    ref_steps = []
    c = lambda v, dt=f32: v.to(DEV, dt)
    denoise_loop(oracle, c(lat), c(ehs), c(pooled), c(time_ids), c(bbox), 1.0, c(dialog), g, T,
                 on_step=lambda i, t, x: ref_steps.append(x.float().cpu()))
    with torch.device("meta"):
        o16 = OracleUNet(SDXL)
    o16 = o16.to_empty(device=DEV).to(bf16)
    o16.load_state_dict(sd)
    o16.eval().set_ip_scale(0.6)
    lib_steps = []

    class Cast(torch.nn.Module):           # bf16 UNet inside an fp32 loop, as the reference pipeline runs it
        def forward(self, x, *a):
            return o16(x.to(bf16), a[0], a[1].to(bf16), a[2].to(bf16), *a[3:5], a[5], a[6]).float()
    denoise_loop(Cast(), c(lat), c(ehs), c(pooled), c(time_ids), c(bbox), 1.0, c(dialog), g, T,
                 on_step=lambda i, t, x: lib_steps.append(x.float().cpu()))
    del o16
    pipe = ds.DiffSenseiPipeline(engine)
    got_steps = []
    pipe.denoise(lat, ehs.to(bf16), pooled, time_ids, bbox, 1.0, dialog, T, g, use_graph=True,
                 on_step=lambda i, t, x: got_steps.append(x.permute(0, 3, 1, 2).float().cpu().clone()))
    eng = [rel_l2(a, b) for a, b in zip(got_steps, ref_steps)]
    lib = [rel_l2(a, b) for a, b in zip(lib_steps, ref_steps)]
    RESULTS["drift_cfg1_50_steps"] = {"engine_vs_fp32_oracle": eng, "bf16_library_vs_fp32_oracle": lib}
    print("engine drift  :", " ".join(f"{d:.1e}" for d in eng[::7] + [eng[-1]]))
    print("bf16-lib drift:", " ".join(f"{d:.1e}" for d in lib[::7] + [lib[-1]]))
    assert len(eng) == T and eng[0] < 1.5e-2
    assert eng[-1] < 1e-1 and eng[-1] < 2 * lib[-1] + 1e-2


def test_ip_mask_grid_is_device_independent():
    """The reference builds its linspace grids on the hidden-states device (CUDA in production, CPU in the oracle
    and in tests/golden): the open/closed decision of every (bucket, level, key) must not depend on which."""
    from oracle.attention import ip_open_mask
    import bench
    tab = torch.load(os.path.join(ROOT, "tests", "golden", "derived_hw_table.pt")).tolist()
    bb = torch.tensor([[bench.IP_BOXES[0], bench.IP_BOXES[1], bench.IP_BOXES[2], bench.IP_BOXES[3]],
                       [[.1, .1, .6, .9], [.5, .2, 1, 1], [1 / 3, 2 / 3, 2 / 3, 1.0], [0.0] * 4]])
    bad = 0
    for bh, bw, _down, fh, fw, _dh, _dw in tab:
        n, ar = fh * fw, (bh // 8) / (bw // 8)
        a = ip_open_mask(bb, n, ar, 16, 16)
        b = ip_open_mask(bb.to(DEV), n, ar, 16, 16).cpu()
        bad += int((a != b).sum())
    assert bad == 0
