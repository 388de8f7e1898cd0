#!/usr/bin/env python
"""The kernel-roofline measurements of bench.py alone (no UNet step): prints one JSON line, with the DS_*
environment switches that were set."""
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

import bench
import diffsensei_b200 as ds

dev = torch.device("cuda:0")
torch.cuda.set_device(dev)
out = bench.kernel_rooflines(ds, bench.measured_peaks(), dev)
out["env"] = {k: v for k, v in os.environ.items() if k.startswith("DS_")}
print(json.dumps(out))
