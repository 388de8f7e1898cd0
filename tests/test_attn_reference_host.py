"""The fp64 attention reference of oracle/attention.py pinned to the executed reference, and the attention tolerance of
tests/attn_check.py calibrated on the CPU: an emulation of the kernels' roundings passes it at every case the GPU
test runs, and it rejects each plausible kernel mistake (the perturbed references of attn_check.*_mutations)."""
import os

import pytest
import torch
import torch.nn.functional as F

import attn_check as K
from conftest import GOLDEN, rel_l2
from oracle import attention as A

f64 = torch.float64


def _load(name):
    return {k: (v.to(f64) if torch.is_tensor(v) and v.is_floating_point() else v)
            for k, v in torch.load(os.path.join(GOLDEN, name), weights_only=False).items()}


def test_self_reference_reproduces_executed_golden():
    g = _load("attn_self.pt")
    qkv = torch.cat([F.linear(g["hs"], g[w]) for w in ("to_q", "to_k", "to_v")], -1)
    out = F.linear(A.self_attention_abi(qkv, g["heads"]), g["to_out_w"], g["to_out_b"])
    assert rel_l2(out, g["out"]) <= 1e-5


def test_cross_reference_reproduces_executed_golden():
    g = _load("attn_cross_ip.pt")
    end = g["ehs"].shape[1] - (g["num_ip_tokens"] + g["num_dummy"])
    text, ip = g["ehs"][:, :end], g["ehs"][:, end:]
    q = F.linear(g["hs"], g["to_q"])
    kv_t = torch.cat([F.linear(text, g["to_k"]), F.linear(text, g["to_v"])], -1)
    kv_i = torch.cat([F.linear(ip, g["to_k_ip"]), F.linear(ip, g["to_v_ip"])], -1)
    tpi = g["num_ip_tokens"] // g["bbox"].shape[1]
    a = A.cross_ip_attention_abi(q, kv_t, kv_i, g["bbox"].float(), g["heads"], g["aspect_ratio"], g["scale"], tpi,
                                 g["num_dummy"])
    assert rel_l2(F.linear(a, g["to_out_w"], g["to_out_b"]), g["out"]) <= 1e-5


def test_cross_reference_matches_processor_restatement_without_dummy_keys():
    """num_dummy = 0, 7 tokens per IP, 3 boxes incl. an all-zero one: the ABI-layout reference against the
    MaskedIPAttnProcessor2_0 restatement, both in fp64."""
    B, N, ar, heads, nt, tpi, num_ips = 3, 264, 44 / 23, 2, 20, 7, 3
    c, cc = heads * 64, 48
    hs, ehs = K.randn(1, B, N, c).to(f64), K.randn(2, B, nt + tpi * num_ips, cc).to(f64)
    w = {n: K.randn(3 + i, c, c if n in ("q", "o") else cc, scale=0.1).to(f64)
         for i, n in enumerate(("q", "k", "v", "k_ip", "v_ip", "o"))}
    bo = K.randn(9, c).to(f64)
    bbox = K.make_boxes(B, num_ips, N, ar)
    want = A.cross_ip_attention(hs, ehs, bbox, ar, w["q"], w["k"], w["v"], w["k_ip"], w["v_ip"], w["o"], bo, heads,
                                0.6, tpi * num_ips, 0)
    text, ip = ehs[:, :nt], ehs[:, nt:]
    kv_t = torch.cat([F.linear(text, w["k"]), F.linear(text, w["v"])], -1)
    kv_i = torch.cat([F.linear(ip, w["k_ip"]), F.linear(ip, w["v_ip"])], -1)
    a = A.cross_ip_attention_abi(F.linear(hs, w["q"]), kv_t, kv_i, bbox, heads, ar, 0.6, tpi, 0)
    assert rel_l2(F.linear(a, w["o"], bo), want) <= 1e-12


# the GPU test's cases; self-attention at one (batch, head) per shape so that the CPU keeps up
HOST_CASES = [("self", "randn", (1, n, 1)) for _, n, _ in K.SELF_CASES] + \
             [("resampler", "randn", c) for c in K.RESAMPLER_CASES] + \
             [("cross", "randn", c) for c in K.CROSS_CASES] + \
             [(kind, num, (1, case[1], 1) if kind == "self" else case) for kind, num, case in K.NUMERICS] + \
             [(kind, "randn", case) for kind, case in sorted(K.MUTATION_CASES, key=str) if kind == "self"]


@pytest.mark.parametrize("kind,numerics,case", HOST_CASES, ids=str)
def test_emulated_kernel_within_tolerance(kind, numerics, case):
    inputs = K.make_inputs(kind, case, numerics)
    mutations = numerics == "randn" and (kind, case) in K.MUTATION_CASES
    ref, absref, muts = K.references(kind, case, inputs, mutations)
    got = K.emulate(kind, case, inputs)
    worst, rel = K.measure(got, ref, absref)
    print(f"[attn-emulation] {kind} {numerics} {case}: worst {worst:.3f} of the bound, rel-L2 {rel:.2e}")
    assert worst <= 1.0 and rel <= K.REL_L2
    for name, mref in muts.items():
        assert not K.passes(got, mref, absref), f"the tolerance accepts the reference with {name}"


def test_mutation_cases_cover_every_mutation():
    built = set()
    for kind, case in K.MUTATION_CASES:
        built |= set(K.references(kind, case, K.make_inputs(kind, case), mutations=True)[2])
    assert built == {"box_keys_shifted", "dummy_keys_always_open", "half_open_box", "padding_keys_counted",
                     "ip_scale_on_text", "true_feature_map"}


@pytest.mark.parametrize("kind,case", [("self", (1, 1012, 2)), ("resampler", (2, 130, 257, 2)),
                                       ("cross", "long_text_264")], ids=str)
def test_rising_inputs_raise_the_row_max_at_every_key_tile(kind, case):
    inputs = K.make_inputs(kind, case, "rising")
    if kind == "self":
        c = inputs[0].shape[-1] // 3
        q, keys = inputs[0][..., :c], [inputs[0][..., c:2 * c]]
    elif kind == "resampler":
        q, keys = inputs[0], [inputs[1][..., :inputs[0].shape[-1]]]
    else:
        q, keys = inputs[0], [kv[..., :inputs[0].shape[-1]] for kv in inputs[1:3]]
    for k in keys:
        for h in range(q.shape[-1] // 64):
            cols = slice(64 * h, 64 * h + 64)
            s = q[..., cols].double() @ k[..., cols].double().transpose(-1, -2)
            tiles = (s.shape[-1] + 63) // 64
            tile_max = torch.stack([s[..., 64 * t:64 * t + 64].amax(-1) for t in range(tiles)], -1)
            assert tiles > 1 and (tile_max.diff(dim=-1) > 0).all()
