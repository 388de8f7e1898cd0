"""The attention kernels' output bits, pinned.

Self-attention, the Resampler's attention and the fused text + masked-IP cross-attention are compared with
`torch.equal`-strength checks (a SHA-256 of the bf16 output bits) against tests/golden/attn_bits.json, at the cfg2
shapes, the cfg3 tail shapes and key sets too long to stay resident in shared memory.  Inputs come from seeded CPU
generators, so every build sees the same values.  The goldens were written by the kernel these replaced:

    python tests/test_attn_bits_gpu.py [OUT.json]     (on an H100; default OUT is tests/golden/attn_bits.json)

Per-sample results must not depend on the batch a sample is launched in: a 2-sample slice of an 8-sample launch is
bit-equal to the 2-sample launch."""
import hashlib
import json
import os
import sys

import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
GOLDEN_FILE = os.path.join(HERE, "golden", "attn_bits.json")

pytestmark = pytest.mark.gpu

bf16 = torch.bfloat16
DEV = "cuda"
BENCH_BOXES = [[.05, .10, .50, .95], [.50, .15, .95, .90], [0.0] * 4, [0.0] * 4]

# (B, N, heads): cfg2 levels 1 and 2, then the cfg3 tail shapes (N not a multiple of the 128-row query tile)
SELF = [(8, 4096, 10), (8, 1024, 20), (2, 4104, 10), (2, 4032, 10), (2, 1012, 10), (2, 1026, 20), (2, 1008, 20),
        (2, 264, 20)]
# (Bc, nq, n_kv, heads): the Resampler's perceiver attention (16 latents against 257 CLIP tokens + magi + latents)
RESAMPLER = [(8, 16, 274, 20)]
# name -> (B, N, heads, n_text, boxes, tokens_per_ip, num_dummy, aspect_ratio)
CROSS = {
    "cfg2_l1": (8, 4096, 10, 77, BENCH_BOXES, 16, 16, 1.0),
    "cfg2_l2": (8, 1024, 20, 77, BENCH_BOXES, 16, 16, 1.0),
    "cfg3_tail": (2, 4104, 10, 77, BENCH_BOXES, 16, 16, 864 / 1216),
    # no dummy keys: rows outside both boxes see no open IP key (every IP score carries the -10000 mask)
    "no_open_ip": (2, 1024, 20, 77, BENCH_BOXES[:2], 32, 0, 1.0),
    # key sets longer than shared memory holds at once
    "long_keys": (2, 1024, 20, 300, BENCH_BOXES, 64, 16, 1.0),
}


def _randn(seed, *shape):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(*shape, generator=g).to(bf16)


def run_self(ops, B, N, h, seed=11):
    qkv = _randn(seed, B, N, 3 * 64 * h)
    return ops.attention_self(qkv.to(DEV), h)


def run_resampler(ops, Bc, nq, n_kv, h, seed=12):
    q = _randn(seed, Bc, nq, 64 * h)
    kv = _randn(seed + 1, Bc, n_kv, 2 * 64 * h)
    return ops.resampler_attn(q.to(DEV), kv.to(DEV), h)


def run_cross(ops, B, N, h, n_text, boxes, tpi, num_dummy, ar, seed=13):
    C = 64 * h
    n_ip = num_dummy + len(boxes) * tpi
    q = _randn(seed, B, N, C)
    kv_t = _randn(seed + 1, B, n_text, 2 * C)
    kv_i = _randn(seed + 2, B, n_ip, 2 * C)
    bbox = torch.tensor([boxes] * B, dtype=torch.float32)
    return ops.attention_cross_ip(q.to(DEV), kv_t.to(DEV), kv_i.to(DEV), bbox.to(DEV), h, ar, 0.6, tpi, num_dummy)


def bits(t):
    return hashlib.sha256(t.contiguous().cpu().view(torch.int16).numpy().tobytes()).hexdigest()


def all_cases():
    cases = {f"self_B{B}_N{N}_h{h}": (run_self, (B, N, h)) for B, N, h in SELF}
    cases.update({f"resampler_B{Bc}_nq{nq}_nkv{nk}_h{h}": (run_resampler, (Bc, nq, nk, h))
                  for Bc, nq, nk, h in RESAMPLER})
    cases.update({f"cross_{name}": (run_cross, args) for name, args in CROSS.items()})
    return cases


@pytest.fixture(scope="module")
def ops():
    from diffsensei_b200 import ops as o
    return o


@pytest.fixture(scope="module")
def golden():
    with open(GOLDEN_FILE) as f:
        return json.load(f)


@pytest.mark.parametrize("name", sorted(all_cases()))
def test_attention_bits_match_golden(ops, golden, name):
    fn, args = all_cases()[name]
    out = fn(ops, *args)
    torch.cuda.synchronize()
    assert torch.isfinite(out.float()).all()
    assert bits(out) == golden[name]


def test_self_attention_batch_invariant(ops):
    qkv = _randn(21, 8, 1024, 3 * 64 * 20).to(DEV)
    full = ops.attention_self(qkv, 20)
    part = ops.attention_self(qkv[2:4].contiguous(), 20)
    assert torch.equal(full[2:4], part)


def test_cross_attention_batch_invariant(ops):
    B, N, h = 8, 1024, 20
    C = 64 * h
    q = _randn(22, B, N, C).to(DEV)
    kv_t = _randn(23, B, 77, 2 * C).to(DEV)
    kv_i = _randn(24, B, 80, 2 * C).to(DEV)
    bbox = torch.tensor([BENCH_BOXES, BENCH_BOXES[:1] + [[0.0] * 4] * 3] * (B // 2), device=DEV)
    full = ops.attention_cross_ip(q, kv_t, kv_i, bbox, h, 1.0, 0.6, 16, 16)
    s = slice(2, 4)
    part = ops.attention_cross_ip(q[s].contiguous(), kv_t[s].contiguous(), kv_i[s].contiguous(),
                                  bbox[s].contiguous(), h, 1.0, 0.6, 16, 16)
    assert torch.equal(full[s], part)


def test_cross_attention_streaming_batch_invariant(ops):
    """300 text keys + 80 IP keys take 7 key tiles, more than stay resident: the streaming kernel."""
    B, N, h = 4, 1000, 4
    C = 64 * h
    q = _randn(25, B, N, C).to(DEV)
    kv_t = _randn(26, B, 300, 2 * C).to(DEV)
    kv_i = _randn(27, B, 80, 2 * C).to(DEV)
    bbox = torch.tensor([BENCH_BOXES, [[0.0] * 4] * 4] * (B // 2), device=DEV)
    full = ops.attention_cross_ip(q, kv_t, kv_i, bbox, h, 0.625, 0.6, 16, 16)
    s = slice(1, 3)
    part = ops.attention_cross_ip(q[s].contiguous(), kv_t[s].contiguous(), kv_i[s].contiguous(),
                                  bbox[s].contiguous(), h, 0.625, 0.6, 16, 16)
    assert torch.equal(full[s], part)


def test_resampler_batch_invariant(ops):
    q = _randn(28, 8, 16, 64 * 20).to(DEV)
    kv = _randn(29, 8, 274, 2 * 64 * 20).to(DEV)
    full = ops.resampler_attn(q, kv, 20)
    part = ops.resampler_attn(q[2:4].contiguous(), kv[2:4].contiguous(), 20)
    assert torch.equal(full[2:4], part)


if __name__ == "__main__":
    sys.path.insert(0, ROOT)
    from diffsensei_b200 import ops as o
    out = {}
    for name, (fn, args) in sorted(all_cases().items()):
        out[name] = bits(fn(o, *args))
        print(name, out[name], flush=True)
    with open(sys.argv[1] if len(sys.argv) > 1 else GOLDEN_FILE, "w") as f:
        json.dump(out, f, indent=1, sort_keys=True)
        f.write("\n")
