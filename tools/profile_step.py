#!/usr/bin/env python
"""One EAGER (non-graph) denoise step at BASELINE cfg2 for `ncu --metrics gpu__time_duration.sum` launch lists.
Usage on the GPU box:
  ncu --metrics gpu__time_duration.sum --clock-control none --profile-from-start off --csv \
      --log-file gpurun_out/launches.csv python tools/profile_step.py
The profiled range (cudaProfilerStart/Stop) is exactly one step: UNet forward + fused CFG/DDIM update."""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

import bench
import diffsensei_b200 as ds
from diffsensei_b200.weights import random_state_dict, unet_param_shapes

dev = torch.device("cuda:0")
cfg = ds.SDXL_MANGA
engine = ds.UNetMangaEngine(cfg, dev)
engine.load_state_dict(random_state_dict(unet_param_shapes(cfg), 1234, dev, torch.bfloat16))
engine.set_ip_scale(bench.IP_SCALE)
pipe = ds.DiffSenseiPipeline(engine)
lat, ehs, pooled, time_ids, bbox, dialog = bench.synthetic_inputs(cfg, 4, 128, 128, 2, dev)
st = pipe.make_stepper(lat, ehs, pooled, time_ids, bbox, 1.0, dialog, bench.T_STEPS, bench.GUIDANCE, use_graph=False)
st.step(0)
torch.cuda.synchronize()
torch.cuda.cudart().cudaProfilerStart()
st.step(1)
torch.cuda.synchronize()
torch.cuda.cudart().cudaProfilerStop()
print("profiled one eager step")
