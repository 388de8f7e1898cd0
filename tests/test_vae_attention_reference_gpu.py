"""ds_attention_single_head (vae_attention.cu) against oracle.attention.single_head_attention in fp64 on every element
of every case of tests/vae_attn_check.py, at its bound, with the output filled with a NaN pattern before the launch
(so an unwritten row fails) and guard elements after it; on q / k / v captured from the SDXL-size decoder; on strided
operands.  An image's output must be the same bits at any batch size, and one NaN or +-Inf must change exactly the
outputs it reaches: a Q row its output row, a K row its image, a V element its column of its image.  The module's
teardown prints the worst error as a fraction of the bound per family, the wall time and the device."""
import time

import pytest
import torch

import vae_attn_check as K

pytestmark = pytest.mark.gpu

DEV = "cuda"
bf16 = torch.bfloat16
GUARD = 4096
PATTERN = 0x7FA5                      # a bf16 NaN
WORST = {}
T0 = [0.0]


@pytest.fixture(scope="module")
def ops():
    torch.cuda.set_device(0)
    from diffsensei_b200 import ops as o
    return o


@pytest.fixture(scope="module", autouse=True)
def report():
    T0[0] = time.time()
    yield
    print(f"\n[vae-attn-reference] wall time {time.time() - T0[0]:.1f} s on {torch.cuda.get_device_name()}")
    for fam, w in sorted(WORST.items()):
        print(f"[vae-attn-reference] worst of {fam}: {w:.3f} of the bound")


def bits(t):
    return t.contiguous().view(torch.int16)


def launch(ops, q, k, v):
    """The kernel's output into a NaN-patterned buffer, with GUARD pattern elements after it that must survive."""
    n = q.numel()
    buf = torch.full((n + GUARD,), PATTERN, dtype=torch.int16, device=DEV)
    out = buf[:n].view(bf16).view(q.shape[0], q.shape[1], q.shape[-1])
    ops.attention_single_head(q, k, v, out=out)
    torch.cuda.synchronize()
    assert bool((buf[n:] == PATTERN).all()), "ds_attention_single_head wrote past B * N * D"
    return out


def check(fam, got, ref, absref, muts=()):
    worst, rel = K.measure(got, ref, absref)
    WORST[fam] = max(WORST.get(fam, 0.0), worst)
    assert worst <= 1.0 and rel <= K.REL_L2, f"{fam}: worst {worst:.3f} of the bound, rel-L2 {rel:.2e}"
    for name, mref in dict(muts).items():
        assert not K.passes(got, mref, absref), f"{fam}: the bound accepts the reference with {name}"


@pytest.mark.parametrize("case", K.CASES, ids=K.case_id)
def test_every_element(ops, case):
    D, B, N, num = case
    q, k, v = (t.to(DEV) for t in K.inputs(case))
    got = launch(ops, q, k, v)
    ref, absref = K.references(q, k, v)
    muts = K.mutations(case, q, k, v) if case in K.MUTATION_CASES else {}
    check(f"{num} D={D}", got, ref, absref, muts)


def test_decoder_operands(ops, monkeypatch):
    """q / k / v of the SDXL-size decoder's mid-block attention (seeded weights, latent 64x48: N = 3072, D = 512),
    captured at the engine's call into ops.attention_single_head."""
    import diffsensei_b200 as ds
    from diffsensei_b200.weights import random_state_dict, vae_decoder_param_shapes
    sd = random_state_dict(vae_decoder_param_shapes(ds.SDXL_VAE), seed=3, device="cpu")
    eng = ds.VaeDecoderEngine(ds.SDXL_VAE, DEV)
    eng.load_state_dict({name: w.to(bf16).float() for name, w in sd.items()})
    seen, real = [], ops.attention_single_head

    def spy(q, k, v, out=None):
        seen.append((q.clone(), k.clone(), v.clone()))
        return real(q, k, v, out=out)

    monkeypatch.setattr(ops, "attention_single_head", spy)
    lat = torch.randn(1, 4, 64, 48, generator=torch.Generator().manual_seed(2)) * 0.9
    eng.decode(lat.to(DEV) / ds.SDXL_VAE.scaling_factor)
    monkeypatch.undo()
    assert len(seen) == 1 and seen[0][0].shape == (1, 3072, 512)
    q, k, v = seen[0]
    check("decoder operands D=512", launch(ops, q, k, v), *K.references(q, k, v))


@pytest.mark.parametrize("N", [65, 1092])
@pytest.mark.parametrize("D", [128, 512])
def test_strided_operands(ops, D, N):
    """q / k / v as column slices of one [B, N, 3D + 64] buffer (row stride > D): the bound, and the contiguous
    launch's bits."""
    B = 3
    wide = K.attn_check.randn(N + D, B, N, 3 * D + 64).to(bf16).to(DEV)
    q, k, v = wide[..., :D], wide[..., D:2 * D], wide[..., 2 * D:3 * D]
    got = launch(ops, q, k, v)
    check(f"strided D={D}", got, *K.references(q, k, v))
    assert torch.equal(bits(got), bits(launch(ops, q.contiguous(), k.contiguous(), v.contiguous())))


@pytest.mark.parametrize("D", [128, 512])
def test_batch_invariance(ops, D):
    """Each image of a B = 5 launch at N = 1000 (partial query and key tiles) has the bits it has alone; a repeated
    launch has the same bits."""
    q, k, v = (t.to(DEV) for t in K.inputs((D, 5, 1000, "randn")))
    out = launch(ops, q, k, v)
    assert torch.equal(bits(out), bits(launch(ops, q, k, v)))
    for b in range(5):
        alone = launch(ops, q[b:b + 1].contiguous(), k[b:b + 1].contiguous(), v[b:b + 1].contiguous())
        assert torch.equal(bits(alone[0]), bits(out[b])), b


NONFINITE = [float("nan"), float("inf"), float("-inf")]


def poisoned(ops, D, where, value):
    """(clean, poisoned) outputs of a B = 3, N = 100 launch with ``value`` written by ``where(q, k, v)``."""
    q, k, v = (t.to(DEV) for t in K.inputs((D, 3, 100, "randn")))
    clean = launch(ops, q, k, v)
    q, k, v = q.clone(), k.clone(), v.clone()
    where(q, k, v, value)
    return clean, launch(ops, q, k, v)


@pytest.mark.parametrize("D", [128, 512])
def test_nan_in_a_q_row_poisons_its_output_row(ops, D):
    def put(q, k, v, x):
        q[1, 99, 5] = x
    clean, got = poisoned(ops, D, put, float("nan"))
    hit = torch.zeros(got.shape, dtype=torch.bool, device=DEV)
    hit[1, 99] = True
    assert bool(torch.isnan(got[hit]).all()) and torch.equal(bits(got[~hit]), bits(clean[~hit]))


@pytest.mark.parametrize("j", [0, 99])
@pytest.mark.parametrize("value", NONFINITE, ids=str)
@pytest.mark.parametrize("D", [128, 512])
def test_non_finite_k_row_poisons_its_image(ops, D, value, j):
    """Key row j of image 1 all ``value``: every query's score at key j sums products of both signs (or a NaN), so
    every output of image 1 is non-finite; images 0 and 2 keep their bits (image 1's key 0 is what a 2-D tensor map
    would load into image 0's last, partial key tile)."""
    def put(q, k, v, x):
        k[1, j] = x
    clean, got = poisoned(ops, D, put, value)
    assert not bool(torch.isfinite(got[1]).any())
    assert torch.equal(bits(got[0::2]), bits(clean[0::2]))


@pytest.mark.parametrize("D", [128, 512])
def test_nan_in_a_v_element_poisons_its_column(ops, D):
    def put(q, k, v, x):
        v[1, 99, 7] = x
    clean, got = poisoned(ops, D, put, float("nan"))
    hit = torch.zeros(got.shape, dtype=torch.bool, device=DEV)
    hit[1, :, 7] = True
    assert bool(torch.isnan(got[hit]).all()) and torch.equal(bits(got[~hit]), bits(clean[~hit]))
