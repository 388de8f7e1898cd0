"""The fused step kernel's output bits, pinned.

``ds_cfg_step`` (the guidance blend, the DDIM or Euler update, the optional inpaint blend and the next UNet input) is
compared with `torch.equal`-strength checks (SHA-256 of the fp32 latents and of the bf16 next UNet input, every chunk)
against tests/golden/step_bits.json.  All eight variants run -- DDIM / Euler, 2 chunks (CFG) / 3 chunks (CFG +
perturbed-attention guidance with an adaptive scale), with / without the inpaint blend under a random mask -- at the
cfg2 latent shape and at two shapes whose pixel count is not a multiple of the 256-thread block, on the first, a
middle and the last step of a 30-step schedule (where sigma_next = 0 and {c0, c1} = {1, 0}).  Inputs come from
seeded CPU generators, so every build sees the same values.  The goldens were written by the eight separate kernels
this one replaced:

    python tests/test_step_bits_gpu.py [OUT.json]     (on an H100; default OUT is tests/golden/step_bits.json)
"""
import hashlib
import json
import os
import sys

import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
GOLDEN_FILE = os.path.join(HERE, "golden", "step_bits.json")

pytestmark = pytest.mark.gpu

bf16, f32 = torch.bfloat16, torch.float32
DEV = "cuda"
T_STEPS = 30
GUIDANCE = 7.5
PAG_SCALE, PAG_ADAPTIVE = 3.0, 0.003      # s_i = 3 - 0.003 (1000 - t_i): nonzero on every step of the schedule
SHAPES = [(4, 128, 128), (2, 17, 23), (3, 6, 5)]   # cfg2 latents, then bs*HW = 782 and 90
STEPS = [0, 14, T_STEPS - 1]
VARIANTS = [(euler, chunks, inpaint) for euler in (False, True) for chunks in (2, 3) for inpaint in (False, True)]


def case_name(euler, chunks, inpaint, shape, step):
    return (f"{'euler' if euler else 'ddim'}_c{chunks}{'_inpaint' if inpaint else ''}_"
            f"{'x'.join(map(str, shape))}_s{step}")


def all_cases():
    return {case_name(*v, shp, st): (*v, shp, st) for v in VARIANTS for shp in SHAPES for st in STEPS}


def coef_row(euler, chunks, inpaint, step):
    """The step's fp32 coefficient row on the host: the update's columns, {c0, c1} with inpaint, s with 3 chunks."""
    from diffsensei_b200.scheduler import DDIMScheduler, EulerDiscreteScheduler, pag_scales
    sch = EulerDiscreteScheduler() if euler else DDIMScheduler()
    ts = sch.set_timesteps(T_STEPS)
    row = [sch.coefficient_table("cpu")[step]]
    if inpaint:
        last = step + 1 == T_STEPS
        row.append(torch.tensor([1.0, 0.0]) if last else sch.add_noise_coefficients(step + 1))
    if chunks == 3:
        row.append(pag_scales(ts, PAG_SCALE, PAG_ADAPTIVE)[step:step + 1])
    return torch.cat(row).to(f32)


def make_inputs(euler, chunks, inpaint, shape, step):
    """(noise_pred bf16 [chunks*bs,H,W,4], latents fp32 [bs,H,W,4], coef, inpaint state or None), all on the host."""
    bs, H, W = shape
    coef = coef_row(euler, chunks, inpaint, step)
    g = torch.Generator().manual_seed(1000 * step + 100 * bs + 10 * chunks + 2 * euler + inpaint)
    eps = torch.randn(chunks * bs, H, W, 4, generator=g).to(bf16)
    lat = torch.randn(bs, H, W, 4, generator=g) * (float(coef[0]) if euler else 1.0)
    inp = None
    if inpaint:
        inp = (torch.randn(bs, H, W, 4, generator=g), torch.randn(bs, H, W, 4, generator=g),
               (torch.rand(bs, H, W, generator=g) < 0.5).to(torch.uint8))
    return eps, lat, coef, inp


def run_case(step_fn, euler, chunks, inpaint, shape, step):
    """Run one case through ``step_fn(noise_pred, latents, model_in, coef, inpaint)``; returns (latents, model_in)."""
    eps, lat, coef, inp = make_inputs(euler, chunks, inpaint, shape, step)
    lat = lat.to(DEV)
    mi = torch.full(eps.shape, float("nan"), dtype=bf16, device=DEV)
    step_fn(eps.to(DEV), lat, mi, coef.to(DEV), None if inp is None else tuple(t.to(DEV) for t in inp))
    torch.cuda.synchronize()
    return lat, mi


def bits(t):
    return hashlib.sha256(t.contiguous().cpu().view(torch.uint8).numpy().tobytes()).hexdigest()


def cfg_step_fn(ops, euler):
    return lambda eps, lat, mi, coef, inp: ops.cfg_step_(eps, lat, mi, coef, GUIDANCE, euler=euler, inpaint=inp)


@pytest.fixture(scope="module")
def golden():
    with open(GOLDEN_FILE) as f:
        return json.load(f)


@pytest.mark.parametrize("name", sorted(all_cases()))
def test_step_bits_match_golden(golden, name):
    from diffsensei_b200 import ops
    euler, chunks, inpaint, shape, step = all_cases()[name]
    lat, mi = run_case(cfg_step_fn(ops, euler), euler, chunks, inpaint, shape, step)
    assert torch.isfinite(lat).all() and torch.isfinite(mi.float()).all()
    assert {"latents": bits(lat), "model_in": bits(mi)} == golden[name]


if __name__ == "__main__":
    sys.path.insert(0, ROOT)
    from diffsensei_b200 import ops as o
    out = {}
    for name, (euler, chunks, inpaint, shape, step) in sorted(all_cases().items()):
        lat, mi = run_case(cfg_step_fn(o, euler), euler, chunks, inpaint, shape, step)
        out[name] = {"latents": bits(lat), "model_in": bits(mi)}
        print(name, out[name], flush=True)
    with open(sys.argv[1] if len(sys.argv) > 1 else GOLDEN_FILE, "w") as f:
        json.dump(out, f, indent=1, sort_keys=True)
        f.write("\n")
