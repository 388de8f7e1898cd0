"""Image preprocessing of the reference's character references: the GPU processors (ds_image_preprocess) against
transformers' PIL-backed processors on the host, in one run.

Workloads:
* ``crops4``: four character crops of the sizes a manga page yields (180x260, 400x300, 224x224, 90x500, RGB);
* ``photo``: one 4000x3000 photo (the long-tap case: ~55 bicubic taps per output pixel on each axis).

For each workload, both processors (CLIP + ViT, as prepare_ip_image_embeds runs them):
* ``gpu_call_ms``: ``proc(images=PIL list).pixel_values`` for both, host clock around the call and a device
  synchronise: PIL ``.convert("RGB")``, host-to-device copy, kernels;
* ``gpu_device_us``: both modes on uint8 images already on the device, CUDA events around 200 back-to-back calls
  (the kernels plus any gaps between their launches);
* ``host_pil_ms``: CLIPImageProcessorPil + ViTImageProcessorPil (``return_tensors="pt"``, CPU tensors), host clock.
Medians over ``--reps`` repetitions after ``--warmup`` untimed ones.  The outputs are checked equal (torch.equal) in
the same run.  The GPU's name and power limit come from ``nvidia-smi --query-gpu`` (read only).
Prints one JSON object; ``--out FILE`` also writes it there.

    python tools/image_preprocess_bench.py [--reps 20] [--warmup 3]
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

WORKLOADS = {"crops4": [(180, 260), (400, 300), (224, 224), (90, 500)], "photo": [(4000, 3000)]}   # (width, height)


def gpu_info():
    q = "name,power.limit"
    out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True,
                         timeout=30, check=True).stdout.strip().splitlines()[0]
    return dict(zip(q.split(","), [s.strip() for s in out.split(",")]))


def images_for(sizes, seed=0):
    from PIL import Image
    rng = np.random.default_rng(seed)
    return [Image.fromarray(rng.integers(0, 256, (h, w, 3), dtype=np.uint8)) for w, h in sizes]


def host_ms(fn, reps, warmup, sync=False):
    for _ in range(warmup):
        fn()
    times = []
    for _ in range(reps):
        if sync:
            torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn()
        if sync:
            torch.cuda.synchronize()
        times.append((time.perf_counter() - t0) * 1e3)
    return statistics.median(times), times


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("image_preprocess_bench.py needs an H100: diffsensei_b200 has no CPU path")
    import diffsensei_b200 as ds
    from diffsensei_b200 import ops
    from transformers import CLIPImageProcessorPil, ViTImageProcessorPil
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    info = gpu_info()
    clip, vit = ds.CLIPImageProcessor(), ds.ViTImageProcessor()
    clip_ref, vit_ref = CLIPImageProcessorPil(), ViTImageProcessorPil()
    result = {"gpu": info, "torch_threads": torch.get_num_threads(), "workloads": {}}
    for name, sizes in WORKLOADS.items():
        images = images_for(sizes)
        gpu = lambda: (clip(images=images).pixel_values, vit(images=images).pixel_values)
        host = lambda: (clip_ref(images=images, return_tensors="pt").pixel_values,
                        vit_ref(images=images, return_tensors="pt").pixel_values)
        g, h = gpu(), host()
        equal = all(torch.equal(a.cpu(), b) for a, b in zip(g, h))
        gpu_med, gpu_all = host_ms(gpu, args.reps, args.warmup, sync=True)
        host_med, host_all = host_ms(host, args.reps, args.warmup)

        # the packed uint8 images already on the device, both modes per call
        hwc = [torch.from_numpy(np.array(im)).reshape(-1) for im in images]
        src = torch.cat(hwc).to(dev)
        hw = [(h_, w_) for w_, h_ in sizes]
        outs = {m: torch.empty(len(sizes), 3, 224, 224, device=dev) for m in ("clip", "vit")}
        scr = {m: torch.empty(max(ops.image_preprocess_scratch_bytes(hw, m), 16), dtype=torch.uint8, device=dev)
               for m in ("clip", "vit")}
        call = lambda: [ops.image_preprocess(src, hw, m, out=outs[m], scratch=scr[m]) for m in ("clip", "vit")]
        for _ in range(args.warmup):
            call()
        kern = []
        for _ in range(args.reps):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(200):
                call()
            e1.record()
            e1.synchronize()
            kern.append(e0.elapsed_time(e1) * 1e3 / 200)
        result["workloads"][name] = {
            "sizes_wxh": sizes, "outputs_equal": equal,
            "gpu_call_ms": round(gpu_med, 3), "gpu_call_ms_all": [round(t, 3) for t in gpu_all],
            "gpu_device_us": round(statistics.median(kern), 2), "gpu_device_us_all": [round(t, 2) for t in kern],
            "host_pil_ms": round(host_med, 3), "host_pil_ms_all": [round(t, 3) for t in host_all],
        }
    line = json.dumps(result)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
