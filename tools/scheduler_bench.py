"""DDIM vs Euler on the cfg2 workload (1024x1024, bs 4 -> UNet batch 8, 2 character refs, CFG 7.5), in one run:

* the whole cfg2 step (UNet forward + the scheduler's fused CFG update), graph replay, alternating DDIM and Euler over
  several rounds so that both see the same machine state;
* the two fused update kernels alone (ds_cfg_ddim_step / ds_cfg_euler_step) at the cfg2 latent shape: each op
  captured 100 times in a CUDA graph, rotating over buffer sets larger than the 50 MB L2, timed with CUDA events;
* the GPU's name and power limit, read with `nvidia-smi --query-gpu=name,power.limit` (read only).

Random weights (seed 1234) and bench.py's synthetic cfg2 inputs: the step time does not depend on the values.
Prints one JSON object; ``--out FILE`` also writes it there.

    python tools/scheduler_bench.py [--rounds 4] [--steps 20] [--warmup 3]
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402

bf16, f32 = torch.bfloat16, torch.float32


def gpu_info():
    q = "name,power.limit"
    out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True,
                         timeout=30, check=True).stdout.strip().splitlines()[0]
    return dict(zip(q.split(","), [s.strip() for s in out.split(",")]))


def update_kernels(ds, dev, bs=4, h=128, w=128, sets=16, launches=100, reps=5):
    """us per launch of each fused update at the cfg2 latent shape, and the bytes it must move."""
    n = bs * h * w * 4
    nbytes = 2 * n * 2 + 2 * n * 4 + 2 * n * 2          # read both eps halves, read + write fp32 latents, write model_in
    bufs = [(torch.randn(2 * bs, h, w, 4, device=dev).to(bf16), torch.randn(bs, h, w, 4, device=dev),
             torch.empty(2 * bs, h, w, 4, dtype=bf16, device=dev)) for _ in range(sets)]
    ddim = ds.DDIMScheduler()
    ddim.set_timesteps(bench.T_STEPS)
    euler = ds.EulerDiscreteScheduler()
    euler.set_timesteps(bench.T_STEPS)
    out = {"bytes_per_launch": nbytes, "l2_rotation_bytes": sets * nbytes}
    for name, sch in (("ddim", ddim), ("euler", euler)):
        coef = sch.coefficient_table(dev)[10].contiguous()       # a mid-loop row: same cost for every row
        call = lambda k: sch.fused_step_(bufs[k % sets][0], bufs[k % sets][1], bufs[k % sets][2], coef,
                                         bench.GUIDANCE)
        side = torch.cuda.Stream(device=dev)
        side.wait_stream(torch.cuda.current_stream(dev))
        with torch.cuda.stream(side):
            for k in range(sets):
                call(k)
        torch.cuda.current_stream(dev).wait_stream(side)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            for k in range(launches):
                call(k)
        for _ in range(3):
            graph.replay()
        times = []
        for _ in range(reps):
            times.append(bench.event_time_ms(lambda i: graph.replay(), 10) * 1e3 / launches)
        us = statistics.median(times)
        out[name] = {"us_per_launch": round(us, 3), "GBps": round(nbytes / (us * 1e-6) / 1e9, 1),
                     "us_per_launch_all_reps": [round(t, 3) for t in times]}
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=4)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("scheduler_bench.py needs an H100: diffsensei_b200 has no CPU path")
    import diffsensei_b200 as ds
    from diffsensei_b200.weights import random_state_dict, unet_param_shapes
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    info = gpu_info()

    cfg = ds.SDXL_MANGA
    engine = ds.UNetMangaEngine(cfg, dev)
    sd = random_state_dict(unet_param_shapes(cfg), seed=1234, device=dev, dtype=bf16)
    engine.load_state_dict(sd)
    del sd
    torch.cuda.empty_cache()
    engine.set_ip_scale(bench.IP_SCALE)
    (bs, h, w, nc, dlg, ml), = bench.config_panels("cfg2")
    inp = bench.synthetic_inputs(cfg, bs, h, w, nc, dev, dialogs=dlg, mllm=ml)
    pipe = ds.DiffSenseiPipeline(engine)
    steppers = {}
    for name, sch in (("ddim", ds.DDIMScheduler()), ("euler", ds.EulerDiscreteScheduler())):
        pipe.scheduler = sch
        steppers[name] = pipe.make_stepper(*inp[:5], h / w, inp[5], bench.T_STEPS, bench.GUIDANCE, use_graph=True)
    torch.cuda.synchronize()

    step_ms = {name: [] for name in steppers}
    for _ in range(args.rounds):
        for name, st in steppers.items():
            for i in range(args.warmup):
                st.step(i)
            torch.cuda.synchronize()
            step_ms[name].append(bench.event_time_ms(lambda i: st.step((args.warmup + i) % bench.T_STEPS),
                                                     args.steps))
    kernels = update_kernels(ds, dev)
    result = {
        "gpu": info,
        "workload": f"cfg2: 1024x1024, bs {bs} (UNet batch {2 * bs}), {nc} character refs, CFG {bench.GUIDANCE}, "
                    f"graph replay, {args.steps} timed steps x {args.rounds} alternating rounds",
        "cfg2_step_ms": {name: {"median": round(statistics.median(v), 2), "rounds": [round(x, 2) for x in v]}
                         for name, v in step_ms.items()},
        "update_kernel": kernels,
    }
    line = json.dumps(result)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
