#!/usr/bin/env python
"""Deformation-MLP forward+backward: the wgmma GEMM chain (utils.time_utils) vs the reference's fp32
PyTorch module (oracle/_ref/refpy/time_utils.py) on the same GPU.  FLOPs per point = 3 124 224
(SURVEY.md 8(d), blender DeformNetworkNormal, fwd+bwd)."""
import importlib
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "dg-mesh_b200"), os.path.join(ROOT, "tests")):
    sys.path.insert(0, p)
import torch  # noqa: E402
import util  # noqa: E402

ref = util.load_reference_pymodules()
tu = importlib.import_module("utils.time_utils")
FLOP_PER_POINT = 3_124_224


def bench(net, x, t, steps=20, warmup=5, train=True):
    def step():
        if train:
            xa = x.detach().requires_grad_(True)
            out = net(xa, t)
            loss = sum(o.sum() for o in out)
            loss.backward()
        else:
            with torch.no_grad():
                net(x, t)
    for _ in range(warmup):
        step()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        step()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps


if "--profile" in sys.argv:      # one warm-up + one step at 100k for `ncu --metrics gpu__time_duration.sum`
    torch.manual_seed(0)
    mine = tu.DeformNetworkNormal(is_blender=True).cuda()
    x = (torch.rand(100_000, 3, device="cuda") * 2 - 1)
    t = torch.full((100_000, 1), 0.37, device="cuda")
    print(bench(mine, x, t, steps=1, warmup=1))
    sys.exit(0)

rows = []
for n in (10_000, 100_000, 200_000):
    torch.manual_seed(0)
    mine = tu.DeformNetworkNormal(is_blender=True).cuda()
    x = (torch.rand(n, 3, device="cuda") * 2 - 1)
    t = torch.full((n, 1), 0.37, device="cuda")
    row = {"points": n}
    for train in (True, False):
        ms = bench(mine, x, t, train=train)
        key = "fwd_bwd" if train else "fwd"
        flops = FLOP_PER_POINT * n if train else FLOP_PER_POINT * n / 3
        row[f"ours_{key}_ms"] = round(ms, 4)
        row[f"ours_{key}_tflops"] = round(flops / (ms * 1e-3) / 1e12, 1)
        if ref is not None:
            theirs = ref.time_utils.DeformNetworkNormal(is_blender=True).cuda()
            theirs.load_state_dict(mine.state_dict())
            ms_r = bench(theirs, x, t, train=train)
            row[f"ref_{key}_ms"] = round(ms_r, 4)
            row[f"speedup_{key}"] = round(ms_r / ms, 2)
    rows.append(row)
    print(json.dumps(row))
