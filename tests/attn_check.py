"""The attention kernels' cases, inputs, tolerance and perturbed references, shared by test_attn_reference_host.py
(the tolerance calibrated on a CPU emulation of the kernels' roundings) and test_attn_reference_gpu.py (the kernels
against the fp64 reference of oracle/attention.py).

Tolerance.  A kernel output element passes when

    |got - ref| <= RTOL * |ref| + ATOL_A * absref        and, over the whole output,  rel-L2(got, ref) <= REL_L2

where ref is the fp64 result and absref the same attention with |V| (for cross-attention: text + |ip_scale| * IP),
i.e. sum_j softmax_j |v_j|, the size of the terms the output is summed from.  The kernels round in two places that
matter: P = exp(S - m) is rounded to bf16 before O += P V (the row sums l take the fp32 P), and the output is rounded
to bf16 once.  With U = 2^-8 the bf16 unit roundoff, the first contributes at most U * absref, the second at most
U * |ref| (+ U^2 * absref).  ATOL_A = 2U leaves U * absref for the fp32 scores, the fp32 -10000 mask (half an ulp of
14427 in the log2 domain: 3.4e-4 relative in P) and the reordered fp32 sums.  emulate_* below reproduces those
roundings on the CPU; test_attn_reference_host.py shows it inside the bound at every case (its worst element at 0.54
of the bound with peaky scores, 0.05-0.35 otherwise) and each perturbation of the reference (*_mutations) rejected.
REL_L2 is twice the worst rel-L2 the emulation shows over the cases (2.5e-3, set by the one final rounding)."""
import math

import torch

from oracle import attention as A

bf16 = torch.bfloat16
U = 2.0 ** -8
RTOL = U
ATOL_A = 2 * U
REL_L2 = 5e-3
HD = 64
KTILE = 64  # keys per kernel tile: keys past a set's end are zero-filled up to the next multiple

# (B, N, heads): 1, 2 and 3 key tiles (attend_set's direct last, even and odd pipelines), partial query tiles, the
# cfg3 tail shapes, then cfg2 levels 1 and 2 and cfg5
SELF_CASES = [(2, n, 2) for n in (1, 2, 63, 64, 65, 127, 128, 129, 192, 264, 1012, 1026, 4104)] + \
             [(8, 4096, 10), (8, 1024, 20), (2, 8192, 10)]
# (Bc, nq, n_kv, heads): the Resampler's 16 latents against 257 CLIP tokens + magi + latents, then edges
RESAMPLER_CASES = [(8, 16, 274, 20), (1, 1, 1, 1), (3, 16, 64, 2), (3, 16, 65, 2), (2, 130, 257, 2), (5, 16, 1000, 4)]
# name -> (B, heads, N, aspect_ratio, n_text, (num_ips, tokens_per_ip, num_dummy), ip_scale).  Key tiles (text + IP)
# <= 4 run attn_cross_kernel with both sets resident, more stream through attn_stream_kernel.
CROSS_CASES = {
    "production_240": (4, 2, 240, 0.6, 77, (4, 16, 16), 0.6),                # 2 + 2 tiles: resident at the limit
    "no_dummy_264_quirk": (4, 2, 264, 44 / 23, 64, (4, 16, 0), 1.0),         # derived 24x11, true map 22x12
    "one_ip_key": (3, 1, 240, 0.6, 1, (1, 1, 0), 0.6),                      # softmax over one key per set
    "tpi7_1012": (4, 2, 1012, 44 / 23, 128, (3, 7, 5), -0.5),                # boxes straddle 64-key tiles
    "tpi13_1012": (4, 3, 1012, 44 / 23, 128, (5, 13, 11), 0.6),              # 2 + 2 tiles, straddling
    "tpi48_stream": (3, 2, 1000, 0.625, 77, (2, 48, 33), 0.6),               # 2 + 3 tiles: streams
    "ips16_4104": (4, 2, 4104, 108 / 152, 300, (16, 4, 0), 0.6),             # 16 boxes in 64 keys; 5 + 1 tiles
    "ips16_272_8192": (2, 2, 8192, 2.0, 1, (16, 16, 16), 0.6),               # 272 IP keys; 1 + 5 tiles
    "persistent_3x7": (3, 7, 1000, 0.625, 77, (4, 16, 16), 0.0),             # 168 items: CTAs cross (b, head)
    "persistent_8x10": (8, 10, 4096, 1.0, 77, (4, 16, 16), 0.6),             # cfg2 level 1, 2560 items
    "long_text_264": (2, 4, 264, 44 / 23, 300, (4, 16, 16), 1.0),            # 5 + 2 tiles
}
PRODUCTION_BOXES = [[.05, .10, .50, .95], [.50, .15, .95, .90]]
# N -> the true feature map where the reference's derived (H', W') differs from it
TRUE_HW = {264: (22, 12)}
# (kernel, numerics, case): scores of std ~50, and a row max that grows at every key tile
NUMERICS = [(kind, numerics, case) for numerics in ("peaky", "rising") for kind, case in
            [("self", (2, 4104, 2)), ("self", (2, 264, 2)), ("resampler", (2, 130, 257, 2)),
             ("resampler", (5, 16, 1000, 4)), ("cross", "production_240"), ("cross", "tpi48_stream"),
             ("cross", "long_text_264")]]
# the cases whose checks must also reject every perturbed reference built for them (together: all six), with the
# "randn" inputs: under "peaky" scores the zero-filled keys' score 0 is negligible, as it should be
MUTATION_CASES = {("self", (2, 65, 2)), ("self", (2, 1012, 2)), ("resampler", (3, 16, 65, 2)),
                  ("resampler", (8, 16, 274, 20)), ("cross", "production_240"), ("cross", "no_dummy_264_quirk"),
                  ("cross", "tpi7_1012")}


def randn(seed, *shape, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(*shape, generator=g) * scale


def peaky(x, seed):
    """Rows scaled by an amplitude in [6, 8]: scores of std ~50, a near one-hot softmax."""
    g = torch.Generator().manual_seed(seed)
    return x * (6.0 + 2.0 * torch.rand(*x.shape[:-1], 1, generator=g))


def rising(q, k, heads, alpha=0.5):
    """Every row's score maximum grows by ~alpha from one 64-key tile to the next, so the running max and the
    rescale of O by corr change at every step: column 64h of q is 8, column 64h of key j is alpha * (j // 64), and the
    other key columns are shrunk to noise of std 0.05 (score noise ~0.05)."""
    q, k = q.clone(), k.clone()
    c = heads * HD
    ramp = alpha * (torch.arange(k.shape[1]) // KTILE).float()
    k[..., :c] *= 0.05
    for h in range(heads):
        q[..., h * HD] = 8.0
        k[..., h * HD] = ramp
    return q, k


def self_inputs(B, N, heads, numerics="randn", seed=11):
    c = heads * HD
    qkv = randn(seed, B, N, 3 * c)
    if numerics == "peaky":
        qkv[..., :2 * c] = peaky(qkv[..., :2 * c], seed + 1)
    elif numerics == "rising":
        q, k = rising(qkv[..., :c], qkv[..., c:2 * c], heads)
        qkv = torch.cat([q, k, qkv[..., 2 * c:]], -1)
    return qkv.to(bf16)


def resampler_inputs(Bc, nq, n_kv, heads, numerics="randn", seed=12):
    c = heads * HD
    q, kv = randn(seed, Bc, nq, c), randn(seed + 1, Bc, n_kv, 2 * c)
    if numerics == "peaky":
        q, kv[..., :c] = peaky(q, seed + 2), peaky(kv[..., :c], seed + 3)
    elif numerics == "rising":
        q, k = rising(q, kv[..., :c], heads)
        kv = torch.cat([k, kv[..., c:]], -1)
    return q.to(bf16), kv.to(bf16)


def grid_points(N, ar):
    H, W = A.derive_hw(N, ar)
    return torch.linspace(0, 1, W), torch.linspace(0, 1, H)


def make_boxes(B, num_ips, N, ar, seed=5):
    """fp32 [B, num_ips, 4], a different mix per batch row: the last row all-zero padding (the CFG negative), row 1
    the production boxes, the others the edge cases below, rotated per row, then random boxes."""
    xs, ys = grid_points(N, ar)
    W, H = len(xs), len(ys)
    g = torch.Generator().manual_seed(seed)
    edge = [
        [0.0, 0.0, 1.0, 1.0],                                                      # the full image
        [xs[W // 4], ys[H // 3], xs[(3 * W) // 4], ys[(2 * H) // 3]],              # edges on linspace points
        [xs[W // 2], 0.1, xs[W // 2], 0.9],                                        # zero width, on a grid column
        [-0.3, -0.2, 0.45, 1.4],                                                   # reaches outside [0, 1]
        [0.3, 0.2, 0.8, 0.7],                                                      # overlaps its neighbours
        [0.2, 0.05, 0.6, 0.6],
    ]
    rows = []
    for b in range(B):
        if b == B - 1 and B > 1:
            row = [[0.0] * 4] * num_ips
        elif b == 1:
            row = (PRODUCTION_BOXES + [[0.0] * 4] * num_ips)[:num_ips]
        else:
            row = []
            for i in range(num_ips):
                if i < len(edge):
                    row.append(edge[(i + b) % len(edge)])
                else:
                    x = torch.rand(2, generator=g).sort().values.tolist()
                    y = torch.rand(2, generator=g).sort().values.tolist()
                    row.append([x[0], y[0], x[1], y[1]])
        rows.append([[float(v) for v in box] for box in row])
    return torch.tensor(rows, dtype=torch.float32)


def cross_inputs(B, heads, N, ar, n_text, layout, numerics="randn", seed=13):
    num_ips, tpi, nd = layout
    c = heads * HD
    q = randn(seed, B, N, c)
    kv_t, kv_i = randn(seed + 1, B, n_text, 2 * c), randn(seed + 2, B, nd + num_ips * tpi, 2 * c)
    if numerics == "peaky":
        q = peaky(q, seed + 3)
        kv_t[..., :c], kv_i[..., :c] = peaky(kv_t[..., :c], seed + 4), peaky(kv_i[..., :c], seed + 5)
    elif numerics == "rising":
        q, kt = rising(q, kv_t[..., :c], heads)
        _, ki = rising(q, kv_i[..., :c], heads)
        kv_t, kv_i = torch.cat([kt, kv_t[..., c:]], -1), torch.cat([ki, kv_i[..., c:]], -1)
    return q.to(bf16), kv_t.to(bf16), kv_i.to(bf16), make_boxes(B, num_ips, N, ar)


def abs_v(kv, c):
    """k | v -> k | |v|: the reference of this is absref."""
    return torch.cat([kv[..., :-c], kv[..., -c:].abs()], -1)


# ---------------------------------------------------------------------------------------------- the check
def measure(got, ref, absref):
    """(worst element's |got - ref| / bound, rel-L2); the check passes when both are <= 1 and <= REL_L2."""
    ref, absref = ref.double(), absref.double()
    got = got.to(ref.device).double()
    err = (got - ref).abs()
    bound = RTOL * ref.abs() + ATOL_A * absref
    worst = float(torch.where(err == 0, 0.0, err / bound).max())
    rel = float((got - ref).norm() / ref.norm().clamp_min(1e-300))
    return worst, rel


def passes(got, ref, absref):
    worst, rel = measure(got, ref, absref)
    return worst <= 1.0 and rel <= REL_L2


# ---------------------------------------------------------------------------------------------- CPU emulation
def emulate_heads(q, k, v, heads, open_mask=None):
    """The kernels' roundings: fp32 scores of the bf16 operands (+ the -10000 mask in fp32), P rounded to bf16 for
    P V, fp32 row sums of the unrounded P.  fp32 [B, Nq, C], before the output rounding."""
    B, n, c = q.shape
    out = torch.empty(B, n, c)
    for b in range(B):
        for h in range(heads):
            cols = slice(h * HD, (h + 1) * HD)
            s = (q[b, :, cols].float() @ k[b, :, cols].float().T) * 0.125
            if open_mask is not None:
                s = s + torch.where(open_mask[b], 0.0, A.MASK_VALUE)
            p = torch.exp(s - s.amax(-1, keepdim=True))
            out[b, :, cols] = (p.to(bf16).float() @ v[b, :, cols].float()) / p.sum(-1, keepdim=True)
    return out


def emulate_self(qkv, heads):
    c = qkv.shape[-1] // 3
    return emulate_heads(qkv[..., :c], qkv[..., c:2 * c], qkv[..., 2 * c:], heads).to(bf16)


def emulate_resampler(q, kv, heads):
    c = q.shape[-1]
    return emulate_heads(q, kv[..., :c], kv[..., c:], heads).to(bf16)


def emulate_cross(q, kv_t, kv_i, bbox, heads, ar, ip_scale, tpi, nd):
    c = q.shape[-1]
    open_ = A.ip_open_mask(bbox, q.shape[1], ar, tpi, nd)
    text = emulate_heads(q, kv_t[..., :c], kv_t[..., c:], heads)
    ip = emulate_heads(q, kv_i[..., :c], kv_i[..., c:], heads, open_)
    return (text + torch.tensor(ip_scale, dtype=torch.float32) * ip).to(bf16)


# ---------------------------------------------------------------------------------------------- perturbed references
def pad_to_tile(kv):
    """kv with its last partial 64-key tile completed by zero keys (what TMA fills in), for the reference that
    counts them in the softmax."""
    pad = -kv.shape[1] % KTILE
    return torch.cat([kv, kv.new_zeros(kv.shape[0], pad, kv.shape[2])], 1)


def shift_box_keys(open_, box, tpi, nd):
    """Box `box`'s key range [lo, lo + tpi) moved to [lo + 1, lo + tpi + 1): key lo closes, key lo + tpi (the next
    box's first key) also opens for the pixels in this box."""
    lo = nd + box * tpi
    inside = open_[..., lo].clone()
    m = open_.clone()
    m[..., lo] = False
    if lo + tpi < m.shape[-1]:
        m[..., lo + tpi] |= inside
    return m


def true_map_aspect(N, H, W):
    """An aspect ratio for which the reference derives exactly (H, W) from N."""
    ar = H / W
    assert A.derive_hw(N, ar) == (H, W)
    return ar


def self_mutations(qkv, heads):
    """Self-attention with the zero-filled keys of the last partial key tile counted in the softmax."""
    c = qkv.shape[-1] // 3
    kv = pad_to_tile(qkv[..., c:])
    return {"padding_keys_counted": A.attention_heads(qkv[..., :c], kv[..., :c], kv[..., c:], heads)}


def resampler_mutations(q, kv, heads):
    c = q.shape[-1]
    kv = pad_to_tile(kv)
    return {"padding_keys_counted": A.attention_heads(q, kv[..., :c], kv[..., c:], heads)}


def cross_mutations(q, kv_t, kv_i, bbox, heads, ar, ip_scale, tpi, nd, true_hw=None):
    """The reference with each of the mistakes a kernel could make, in fp64 on q's device.  Only the mutations that
    change this case's result are built."""
    c = q.shape[-1]
    N = q.shape[1]
    bbox = bbox.cpu()
    open_ = A.ip_open_mask(bbox, N, ar, tpi, nd)
    text = A.attention_heads(q, kv_t[..., :c], kv_t[..., c:], heads)
    ip_k, ip_v = kv_i[..., :c], kv_i[..., c:]
    ip = A.attention_heads(q, ip_k, ip_v, heads, open_)

    def with_mask(m):
        return text + ip_scale * A.attention_heads(q, ip_k, ip_v, heads, m)

    out = {}
    num_ips = bbox.shape[1]
    inside = open_[..., nd::tpi][..., :num_ips]                  # [B, N, num_ips]
    if ip_scale != 0:
        box = int(inside.sum((0, 1)).argmax())
        out["box_keys_shifted"] = with_mask(shift_box_keys(open_, box, tpi, nd))
        if nd > 0:
            m = open_.clone()
            m[..., :nd] = True
            out["dummy_keys_always_open"] = with_mask(m)
        half_open = bbox.clone()
        half_open[..., 2:] = torch.nextafter(half_open[..., 2:], torch.tensor(-math.inf))   # x <= x2' <=> x < x2
        out["half_open_box"] = with_mask(A.ip_open_mask(half_open, N, ar, tpi, nd))
        if true_hw is not None:
            out["true_feature_map"] = with_mask(A.ip_open_mask(bbox, N, true_map_aspect(N, *true_hw), tpi, nd))
    if ip_scale != 1:
        out["ip_scale_on_text"] = ip_scale * (text + ip)
    if kv_t.shape[1] % KTILE:
        kv = pad_to_tile(kv_t)
        out["padding_keys_counted"] = A.attention_heads(q, kv[..., :c], kv[..., c:], heads) + ip_scale * ip
    return out


# ---------------------------------------------------------------------------------------------- one case
def make_inputs(kind, case, numerics="randn"):
    """CPU bf16 operands (and fp32 boxes) of one case, in the kernel's ABI layout."""
    if kind == "self":
        return (self_inputs(*case, numerics=numerics),)
    if kind == "resampler":
        return resampler_inputs(*case, numerics=numerics)
    B, heads, N, ar, n_text, layout, _ = CROSS_CASES[case]
    return cross_inputs(B, heads, N, ar, n_text, layout, numerics=numerics)


def references(kind, case, inputs, mutations=False):
    """(ref, absref, {mutation: perturbed ref}) in fp64 on the operands' device."""
    if kind == "self":
        (qkv,), heads = inputs, case[2]
        c = qkv.shape[-1] // 3
        muts = self_mutations(qkv, heads) if mutations and qkv.shape[1] % KTILE else {}
        return A.self_attention_abi(qkv, heads), A.self_attention_abi(abs_v(qkv, c), heads), muts
    if kind == "resampler":
        (q, kv), heads = inputs, case[3]
        c = q.shape[-1]
        muts = resampler_mutations(q, kv, heads) if mutations and kv.shape[1] % KTILE else {}
        return A.resampler_attention_abi(q, kv, heads), A.resampler_attention_abi(q, abs_v(kv, c), heads), muts
    _, heads, N, ar, _, (_, tpi, nd), s = CROSS_CASES[case]
    q, kv_t, kv_i, bbox = inputs
    c = q.shape[-1]
    ref = A.cross_ip_attention_abi(q, kv_t, kv_i, bbox, heads, ar, s, tpi, nd)
    absref = A.cross_ip_attention_abi(q, abs_v(kv_t, c), abs_v(kv_i, c), bbox, heads, ar, abs(s), tpi, nd)
    muts = cross_mutations(q, kv_t, kv_i, bbox, heads, ar, s, tpi, nd, TRUE_HW.get(N)) if mutations else {}
    return ref, absref, muts


def emulate(kind, case, inputs):
    if kind == "self":
        return emulate_self(inputs[0], case[2])
    if kind == "resampler":
        return emulate_resampler(*inputs, case[3])
    _, heads, _, ar, _, (_, tpi, nd), s = CROSS_CASES[case]
    return emulate_cross(*inputs, heads, ar, s, tpi, nd)
