#!/usr/bin/env python
"""Kernel time per step of `compare` on the benchmark's 10 000-sketch set, from torch.profiler (CUDA activities), in a run
of its own (tracing slows the host, so bench.py is not profiled).  Prints ms per step and launches per step per kernel.

    python scripts/profile_compare_step.py > profiles/h100/compare_step_kernels.txt
"""
import collections
import os
import sys

import torch
from torch.profiler import ProfilerActivity, profile

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bench  # noqa: E402
from sourmash_b200 import batch as B  # noqa: E402

torch.cuda.set_device(0)
B.set_device(0)
s = torch.cuda.current_stream(); B.set_stream(s.cuda_stream)
h, off = bench.compare_workload()
n = len(off) - 1
sset = B.SketchSet.from_host(h, off)
d_out = torch.empty((n, n), dtype=torch.float64, device="cuda")
for _ in range(3):
    B.compare_jaccard_device(sset, d_out.data_ptr())
torch.cuda.synchronize()
STEPS = 5
with profile(activities=[ProfilerActivity.CUDA]) as prof:
    for _ in range(STEPS):
        B.compare_jaccard_device(sset, d_out.data_ptr())
    torch.cuda.synchronize()
tot = collections.defaultdict(float); cnt = collections.Counter()
for e in prof.events():
    if e.device_type == torch.autograd.DeviceType.CUDA:
        tot[e.name] += e.device_time_total / 1e3; cnt[e.name] += 1
rows = sorted(((v / STEPS, cnt[k] / STEPS, k) for k, v in tot.items()), reverse=True)
print("ms per step, launches per step, kernel")
for ms, c, k in rows:
    print("%8.3f %5.1f %s" % (ms, c, k[:150]))
print("sum %.3f ms" % sum(r[0] for r in rows))
print(B.last_compare_plan())
