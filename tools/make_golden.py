#!/usr/bin/env python
"""Generate tests/golden/*.pt by EXECUTING the reference's own torch-only modules (build container only).

The reference (jianzongwu/DiffSensei @ /root/reference) has no tests or golden vectors (SURVEY.md §4).
Two of its hot-path files import nothing but torch, so they run here on CPU:
    src/models/attention_processor.py   (AttnProcessor2_0, MaskedIPAttnProcessor2_0)
    src/models/resampler.py             (Resampler)
and ``UNetMangaModel.encode_dialog_bbox`` (src/models/unet.py:88-114) is a pure-torch method that is lifted
out of its (diffusers-dependent) module with ``ast`` and executed on a stub ``self``.
Nothing is copied into this repository: the reference code is imported/executed from where it lies and only
its seeded inputs and outputs are saved.  /root/reference does not exist on the GPU box, so the fixtures are
committed; re-run this script only in the build container:

    python tools/make_golden.py            # every fixture
    python tools/make_golden.py agent      # tests/golden/agent_generate.pt only
    python tools/make_golden.py mllm       # tests/golden/mllm_inputs.pt only
"""
from __future__ import annotations

import ast
import importlib.util
import os
import sys
import types

import torch

REF = "/root/reference"
OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden")


def load_module(name: str, path: str):
    spec = importlib.util.spec_from_file_location(name, path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def lift_function(path: str, func_name: str, **module_globals):
    """Compile one function definition out of a module that cannot be imported (missing diffusers); the function
    sees ``torch`` and ``module_globals`` as its module's globals."""
    tree = ast.parse(open(path).read())
    for node in ast.walk(tree):
        if isinstance(node, ast.FunctionDef) and node.name == func_name:
            mod = ast.Module(body=[node], type_ignores=[])
            ns = {"torch": torch, **module_globals}
            exec(compile(mod, path, "exec"), ns)
            return ns[func_name]
    raise KeyError(func_name)


class StubAttn:
    """The attributes a processor reads from diffusers' Attention (attention_processor.py:34-94) for SDXL."""

    def __init__(self, dim, kv_dim, heads, gen):
        def lin(i, o, bias):
            m = torch.nn.Linear(i, o, bias=bias)
            with torch.no_grad():
                m.weight.copy_(torch.randn(o, i, generator=gen) / i ** 0.5)
                if bias:
                    m.bias.copy_(torch.randn(o, generator=gen) * 0.1)
            return m

        self.heads = heads
        self.spatial_norm = None
        self.group_norm = None
        self.norm_cross = False
        self.residual_connection = False
        self.rescale_output_factor = 1.0
        self.to_q = lin(dim, dim, False)
        self.to_k = lin(kv_dim, dim, False)
        self.to_v = lin(kv_dim, dim, False)
        self.to_out = [lin(dim, dim, True), torch.nn.Identity()]

    def weights(self):
        return {"to_q": self.to_q.weight.detach().clone(), "to_k": self.to_k.weight.detach().clone(),
                "to_v": self.to_v.weight.detach().clone(), "to_out_w": self.to_out[0].weight.detach().clone(),
                "to_out_b": self.to_out[0].bias.detach().clone()}


def sampled(out: torch.Tensor, n: int = 8192, seed: int = 7):
    """A fixed seeded sample of a large output (flat indices + fp32 values) so every fixture stays far below 1 MB;
    outputs of at most `n` elements are stored whole."""
    out = out.detach().float()
    if out.numel() <= n:
        return out
    idx = torch.randperm(out.numel(), generator=torch.Generator().manual_seed(seed))[:n].sort().values
    return {"shape": tuple(out.shape), "idx": idx.to(torch.int32), "vals": out.reshape(-1)[idx].clone()}


@torch.no_grad()
def main():
    os.makedirs(OUT, exist_ok=True)
    ap = load_module("ref_attention_processor", f"{REF}/src/models/attention_processor.py")
    rs = load_module("ref_resampler", f"{REF}/src/models/resampler.py")

    # ------------------------------------------------------------------ self-attention
    g = torch.Generator().manual_seed(0)
    attn = StubAttn(128, 128, 2, g)
    hs = torch.randn(2, 96, 128, generator=g)
    out = ap.AttnProcessor2_0()(attn, hs)
    torch.save({"hs": hs, "heads": 2, **attn.weights(), "out": out}, f"{OUT}/attn_self.pt")

    # ------------------------------------------------------------------ text + masked-IP cross-attention
    g = torch.Generator().manual_seed(1)
    dim, kv, heads, n_ips, tpi = 128, 64, 2, 4, 16
    H, W = 12, 20                               # feature map; aspect_ratio = H / W as pipeline :272
    attn = StubAttn(dim, kv, heads, g)
    proc = ap.MaskedIPAttnProcessor2_0(hidden_size=dim, cross_attention_dim=kv, num_ip_tokens=n_ips * tpi,
                                       num_dummy_tokens=tpi)
    proc.to_k_ip.weight.copy_(torch.randn(dim, kv, generator=g) / kv ** 0.5)
    proc.to_v_ip.weight.copy_(torch.randn(dim, kv, generator=g) / kv ** 0.5)
    proc.scale = 0.6
    hs = torch.randn(2, H * W, dim, generator=g)
    ehs = torch.randn(2, 77 + 80, kv, generator=g)
    bbox = torch.tensor([[[0.0, 0.0, 0.0, 0.0]] * 4,
                         [[0.05, 0.10, 0.50, 0.95], [0.50, 0.15, 0.95, 0.90], [0.30, 0.55, 0.70, 1.0],
                          [0.0, 0.0, 0.0, 0.0]]])
    out = proc(attn, hs, encoder_hidden_states=ehs, bbox=bbox, aspect_ratio=H / W)
    torch.save({"hs": hs, "ehs": ehs, "bbox": bbox, "aspect_ratio": H / W, "heads": heads, "scale": 0.6,
                "num_ip_tokens": n_ips * tpi, "num_dummy": tpi, **attn.weights(),
                "to_k_ip": proc.to_k_ip.weight.detach().clone(), "to_v_ip": proc.to_v_ip.weight.detach().clone(),
                "out": out}, f"{OUT}/attn_cross_ip.pt")

    # ------------------------------------------------------------------ IP mask known-answer tests
    proc = ap.MaskedIPAttnProcessor2_0(hidden_size=64, cross_attention_dim=64, num_ip_tokens=64, num_dummy_tokens=16)
    kats = []
    # (iii) of SURVEY.md §8c: open fraction 0.2065 at N = 32x32
    bb = torch.tensor([[[0.0] * 4] * 4, [[.1, .1, .6, .9], [.5, .2, 1, 1], [0.0] * 4, [0.0] * 4]])
    for (n, ar, b) in [(1024, 1.0, bb), (24 * 11, 184 / 352, bb), (15 * 5, 136 / 480, bb), (38 * 27, 27 / 38, bb),
                       (64, 1.0, torch.tensor([[[0.5, 0.5, 0.5, 0.5], [0.0, 0.0, 1.0, 1.0], [3 / 7, 0.0, 4 / 7, 1.0],
                                               [0.25, 0.25, 0.75, 0.75]]]))]:
        m = proc.prepare_attention_mask_ip(b, torch.zeros(b.shape[0], n, 64), 1, ar)[:, 0]   # heads identical
        kats.append({"N": n, "aspect_ratio": ar, "bbox": b, "open": (m == 0)})
    torch.save(kats, f"{OUT}/ip_mask_kats.pt")

    # derived (H', W') for every (bucket, level): with bbox [0,0,1,0] only the first row (y == 0) is inside,
    # so the number of open ip-0 keys' pixels equals the derived width.
    try:
        du = load_module("ref_dataset_utils", f"{REF}/src/datasets/utils.py")
        buckets = [b for grp in du.size_buckets for b in grp["buckets"]]
    except Exception as e:  # PIL missing etc.: parse the literal instead
        src = open(f"{REF}/src/datasets/utils.py").read()
        tree = ast.parse(src)
        lit = next(n.value for n in tree.body if isinstance(n, ast.Assign) and n.targets[0].id == "size_buckets")
        buckets = [b for grp in ast.literal_eval(lit) for b in grp["buckets"]]
    rows = []
    row_box = torch.tensor([[[0.0, 0.0, 1.0, 0.0]] + [[0.0] * 4] * 3])
    for (bh, bw, _r) in buckets:
        for down in (16, 32):                       # level-1 and level-2 feature maps (latent/2, latent/4)
            lh, lw = bh // 8, bw // 8               # latent size
            # true feature-map dims after stride-2 convs with padding 1: ceil division
            fh, fw = lh, lw
            for _ in range({16: 1, 32: 2}[down]):
                fh, fw = (fh - 1) // 2 + 1, (fw - 1) // 2 + 1
            n = fh * fw
            ar = lh / lw                            # pipeline_diffsensei.py:272 uses the LATENT aspect ratio
            m = proc.prepare_attention_mask_ip(row_box, torch.zeros(1, n, 64), 1, ar)[0, 0]
            w_derived = int((m[:, 16] == 0).sum())
            rows.append((bh, bw, down, fh, fw, n // w_derived, w_derived))
    torch.save(torch.tensor(rows, dtype=torch.int32), f"{OUT}/derived_hw_table.pt")
    mism = sum(1 for r in rows if (r[3], r[4]) != (r[5], r[6]))
    print(f"derived-(H',W') table: {len(rows)} (bucket, level) rows, {mism} differ from the true feature map")

    # ------------------------------------------------------------------ dialog bbox embedding
    enc = lift_function(f"{REF}/src/models/unet.py", "encode_dialog_bbox")
    g = torch.Generator().manual_seed(2)
    cases = []
    for dtype in (torch.float32, torch.bfloat16):
        stub = types.SimpleNamespace(dialog_bbox_embedding=torch.randn(8, generator=g).to(dtype))
        sample = torch.randn(2, 8, 19, 152, generator=g).to(dtype)
        db = torch.tensor([[[.05, .05, .30, .20], [.70, .05, .95, .22], [.40, .80, .65, .97], [0.0, 0.0, 0.9, 0.5]]
                           + [[0.0] * 4] * 4, [[0.0] * 4] * 8]).to(dtype)
        cases.append({"sample": sample, "dialog_bbox": db, "emb": stub.dialog_bbox_embedding,
                      "out": enc(stub, sample, db)})
    torch.save(cases, f"{OUT}/dialog_embed.pt")

    # ------------------------------------------------------------------ Resampler (tiny config)
    # weights and inputs are regenerated from the seeds on both sides (tests/test_oracle_golden.py::resampler_tiny_case)
    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    from diffsensei_b200.config import RESAMPLER, RESAMPLER_TINY
    from diffsensei_b200.weights import random_state_dict, resampler_param_shapes
    import dataclasses
    kw = dataclasses.asdict(RESAMPLER_TINY)
    model = rs.Resampler(**kw).eval()
    sdt = random_state_dict(resampler_param_shapes(RESAMPLER_TINY), seed=44, device="cpu")
    model.load_state_dict({k: v.to(torch.bfloat16).float() for k, v in sdt.items()})
    gt = torch.Generator().manual_seed(45)
    x = torch.randn(1, 4, 33, 64, generator=gt).to(torch.bfloat16).float()
    magi = torch.randn(1, 4, 32, generator=gt).to(torch.bfloat16).float()
    x[0, 2:] = 0
    magi[0, 2:] = 0
    torch.save({"kwargs": kw, "weight_seed": 44, "input_seed": 45, "n_real": 2, "out": model(x, magi),
                "out_zero": model(torch.zeros_like(x), torch.zeros_like(magi))}, f"{OUT}/resampler_tiny.pt")
    # ------------------------------------------------------------------ Resampler at the SHIPPED config
    # (configs/model/diffsensei.yaml + scripts/demo/gradio_wo_mllm.py:174-185: 83,978,752 params).  The weights
    # (336 MB) and inputs are NOT stored: both sides regenerate them from the seeds below with
    # diffsensei_b200.weights.random_state_dict / torch.Generator (same torch build on the GPU box); only a fixed
    # seeded sample of the reference's outputs is committed (sampled()).
    kwf = dataclasses.asdict(RESAMPLER)
    full = rs.Resampler(**kwf).eval()
    print("Resampler(shipped config) params:", sum(p.numel() for p in full.parameters()))
    sdf = random_state_dict(resampler_param_shapes(RESAMPLER), seed=42, device="cpu")
    sdf = {k: v.to(torch.bfloat16).float() for k, v in sdf.items()}      # bf16-representable on both sides
    full.load_state_dict(sdf)
    gx = torch.Generator().manual_seed(43)
    xf = torch.randn(1, 4, 257, 1280, generator=gx).to(torch.bfloat16).float()
    mf = torch.randn(1, 4, 768, generator=gx).to(torch.bfloat16).float()
    xf[0, 3:] = 0                                                        # 3 real characters, 1 padded (:131-132)
    mf[0, 3:] = 0
    torch.save({"kwargs": kwf, "weight_seed": 42, "input_seed": 43, "n_real": 3, "out": sampled(full(xf, mf)),
                "out_zero": sampled(full(torch.zeros_like(xf), torch.zeros_like(mf)))}, f"{OUT}/resampler_full.pt")
    # ------------------------------------------------------------------ QwenResampler (MLLM adaptor, §8f-4)
    # configs/model/diffsensei.yaml agent.input_resampler / output_resampler + a small one; weights / inputs are
    # regenerated from seeds on both sides (tests/test_oracle_golden.py::qwen_case), only outputs are stored
    qr = load_module("ref_qwen_resampler", f"{REF}/src/models/qwen_resampler.py")
    qcases = {}
    for name, kw in (("tiny", dict(grid_size=4, embed_dim=128, num_heads=2, kv_dim=64)),
                     ("input", dict(grid_size=8, embed_dim=5120, num_heads=32, kv_dim=2048)),
                     ("output", dict(grid_size=8, embed_dim=2048, num_heads=32, kv_dim=5120))):
        m = qr.QwenResampler(**kw).eval()
        gq = torch.Generator().manual_seed(50)
        sdq = {}
        for k, v in m.state_dict().items():
            if k == "pos_embed":
                sdq[k] = v
            elif k.endswith("weight") and v.dim() == 1:
                sdq[k] = (1 + 0.1 * torch.randn(v.shape, generator=gq)).to(torch.bfloat16).float()
            elif k.endswith("bias"):
                sdq[k] = (0.05 * torch.randn(v.shape, generator=gq)).to(torch.bfloat16).float()
            elif k == "query":
                sdq[k] = torch.randn(v.shape, generator=gq).to(torch.bfloat16).float()
            else:
                sdq[k] = (torch.randn(v.shape, generator=gq) * v.shape[-1] ** -0.5).to(torch.bfloat16).float()
        m.load_state_dict(sdq)
        xq = torch.randn(2, kw["grid_size"] ** 2, kw["kv_dim"], generator=gq).to(torch.bfloat16).float()
        qcases[name] = {"kwargs": kw, "seed": 50, "out": sampled(m(xq))}
    torch.save(qcases, f"{OUT}/qwen_resampler.pt")
    for f in sorted(os.listdir(OUT)):
        print(f, os.path.getsize(os.path.join(OUT, f)))


class StubTokenizer:
    """A LlamaTokenizer stand-in for the agent fixture: ``encode`` puts the leading sentencepiece "▁" piece in front
    (what the reference's ``encode(EOI_TOKEN)[1]`` relies on); ``<img>``, ``<img_00000>`` .. and ``</img>`` are single
    ids; any other character is one id."""
    SPACE, BOI, IMG0, EOI = 29, 900, 901, 965
    bos_token_id = 1

    def encode(self, s, add_special_tokens=False):
        ids, i = [self.SPACE], 0
        while i < len(s):
            if s.startswith("<img>", i):
                ids.append(self.BOI); i += 5
            elif s.startswith("</img>", i):
                ids.append(self.EOI); i += 6
            elif s.startswith("<img_", i):
                ids.append(self.IMG0 + int(s[i + 5:i + 10])); i += 11
            else:
                ids.append(100 + ord(s[i]) % 50); i += 1
        return ids

    def decode(self, ids, skip_special_tokens=True):
        return " ".join(str(int(x)) for x in ids)


AGENT_LLAMA = dict(vocab_size=1000, hidden_size=256, intermediate_size=688, num_hidden_layers=2, num_attention_heads=2,
                   max_position_embeddings=512, rms_norm_eps=1e-5, bos_token_id=1, eos_token_id=2, pad_token_id=0)


@torch.no_grad()
def agent_golden():
    """tests/golden/agent_generate.pt: the reference's ContinuousLVLM.generate + AutoImageTokenGenerationProcessor +
    QwenResampler EXECUTED on a seeded tiny transformers LlamaForCausalLM (oracle.agent.seeded_llama regenerates it)."""
    sys.path.insert(0, REF)
    sys.path.insert(1, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    from src.models.mllm.seed_x import ContinuousLVLM
    from src.models.qwen_resampler import QwenResampler
    from oracle.agent import image_token_rule, seeded_llama, seeded_qwen_sd
    tok = StubTokenizer()
    img_ids = tok.encode("<img>" + "".join(f"<img_{i:05d}>" for i in range(64)) + "</img>")
    rkw_in = dict(grid_size=8, embed_dim=256, num_heads=4, kv_dim=64)
    rkw_out = dict(grid_size=8, embed_dim=64, num_heads=4, kv_dim=256)
    cases = []
    # (name, llm seed, prompt text ids, ends in <img>, max_new_tokens, eos override)
    for name, seed, ends_boi, max_new, eos in (("free", 3, False, 120, 2), ("forced", 4, True, 100, 2),
                                                ("max_new", 5, True, 40, 2)):
        llm, _ = seeded_llama(AGENT_LLAMA, seed)
        llm.generation_config.eos_token_id = eos
        torch.manual_seed(seed + 100)
        inp, outp = QwenResampler(**rkw_in).eval(), QwenResampler(**rkw_out).eval()
        g = torch.Generator().manual_seed(seed + 200)
        for m, kw in ((inp, rkw_in), (outp, rkw_out)):
            sd = seeded_qwen_sd(kw, g)
            assert list(sd) == list(m.state_dict()), "state-dict order differs from the restatement"
            m.load_state_dict(sd)
        text = [100 + (7 * k + seed) % 50 for k in range(10)]
        ids = [1] + text + [tok.BOI] + list(range(tok.IMG0, tok.IMG0 + 64)) + [tok.EOI] + [110] + \
            ([tok.BOI] if ends_boi else [120])
        ids = torch.tensor([ids])
        cmp = torch.zeros_like(ids, dtype=torch.bool)
        cmp[0, 12:76] = True
        img = torch.randn(1, 64, 64, generator=g).to(torch.bfloat16).float()
        agent = ContinuousLVLM(llm, inp, outp).eval()
        o = agent.generate(tok, input_ids=ids, image_embeds=img, ids_cmp_mask=cmp, max_new_tokens=max_new,
                           num_img_gen_tokens=64)
        # top-2 margins of the free steps, teacher-forced over the reference's own raw sequence
        emb = llm.get_input_embeddings()(ids).clone()
        emb[cmp] = inp(img).reshape(-1, 256)
        seq_raw = _raw_sequence(llm, ids, emb, img_ids, eos, max_new)
        full = torch.cat([emb, llm.get_input_embeddings()(seq_raw[None, :-1])], 1)
        logits = llm(inputs_embeds=full).logits[0, ids.shape[1] - 1:].float()
        margins, last = {}, int(ids[0, -1])
        for t in range(seq_raw.numel()):
            s = image_token_rule(last, logits[t].clone(), img_ids)
            if last not in img_ids[:-1]:
                top = s.topk(2).values
                margins[t] = float(top[0] - top[1])
            last = int(seq_raw[t])
        cases.append({"name": name, "llm_seed": seed, "llama": AGENT_LLAMA, "resampler_seed": seed + 200,
                      "input_resampler": rkw_in, "output_resampler": rkw_out, "input_ids": ids, "ids_cmp_mask": cmp,
                      "image_embeds": img, "img_ids": img_ids, "eos": eos, "max_new_tokens": max_new,
                      "raw_ids": seq_raw, "output_ids": o["output_ids"].clone(), "ids_gen_mask": o["ids_gen_mask"],
                      "num_gen_imgs": o["num_gen_imgs"], "img_gen_feat": o["img_gen_feat"], "margins": margins})
        print(name, "new tokens", o["output_ids"].numel(), "images", o["num_gen_imgs"],
              "min free margin", min(margins.values()) if margins else None)
    # canned: llm.generate returns fixed sequences / hidden states; EOIs at 30 (< 64: skipped), 100 and 170
    n_new, C = 180, 256
    gc = torch.Generator().manual_seed(9)
    prompt = torch.tensor([[1, 101, 102, 103]])
    new = torch.randint(100, 150, (n_new,), generator=gc)
    for e in (30, 100, 170):
        new[e] = tok.EOI
    hid = [torch.randn(1, prompt.shape[1], C, generator=gc)] + [torch.randn(1, 1, C, generator=gc)
                                                                  for _ in range(n_new - 1)]

    class CannedLLM(torch.nn.Module):
        def __init__(self):
            super().__init__()
            self.emb = torch.nn.Embedding(1000, C)
            self.dtype_ = torch.float32

        @property
        def dtype(self):
            return torch.float32

        def get_input_embeddings(self):
            return self.emb

        def generate(self, input_ids=None, **kw):
            return types.SimpleNamespace(sequences=torch.cat([input_ids, new[None]], 1),
                                         hidden_states=tuple((h,) for h in hid))

    torch.manual_seed(10)
    outp = QwenResampler(**rkw_out).eval()
    agent = ContinuousLVLM(CannedLLM(), QwenResampler(**rkw_in).eval(), outp).eval()
    o = agent.generate(tok, input_ids=prompt, max_new_tokens=n_new, num_img_gen_tokens=64)
    canned = {"prompt": prompt, "new_ids": new, "hidden_seed": 9,
              "img_ids": img_ids, "output_ids": o["output_ids"].clone(), "ids_gen_mask": o["ids_gen_mask"],
              "num_gen_imgs": o["num_gen_imgs"], "text": o["text"],
              "run_feats": torch.stack([torch.cat([h[0] for h in hid], 0)[prompt.shape[1]:][s:s + 64]
                                        for s in (36, 106)])}
    torch.save({"cases": cases, "canned": canned}, f"{OUT}/agent_generate.pt")
    print("agent_generate.pt", os.path.getsize(f"{OUT}/agent_generate.pt"))


def _raw_sequence(llm, ids, emb, img_ids, eos, max_new):
    from oracle.agent import greedy
    return greedy(llm, ids, emb, img_ids, eos, max_new)[0]


MLLM_PROMPTS = ["", "a manga panel", "two girls talk on a rooftop at night,\nwind", "<img> inside a prompt"]


def mllm_golden():
    """tests/golden/mllm_inputs.pt: the demo's ``get_mllm_inputs`` (scripts/demo/gradio.py:36-57, lifted out of the
    gradio module) EXECUTED on ``StubTokenizer`` for ``MLLM_PROMPTS``."""
    get_mllm_inputs = lift_function(f"{REF}/scripts/demo/gradio.py", "get_mllm_inputs", BOI_TOKEN="<img>",
                                    EOI_TOKEN="</img>", IMG_TOKEN="<img_{:05d}>")
    cases = [{"prompt": p, **dict(zip(("input_ids", "ids_cmp_mask"), get_mllm_inputs(p, StubTokenizer())))}
             for p in MLLM_PROMPTS]
    torch.save(cases, f"{OUT}/mllm_inputs.pt")
    print("mllm_inputs.pt", os.path.getsize(f"{OUT}/mllm_inputs.pt"))


if __name__ == "__main__":
    if sys.argv[1:] == ["agent"]:
        sys.exit(agent_golden())
    if sys.argv[1:] == ["mllm"]:
        sys.exit(mllm_golden())
    sys.exit(main())
