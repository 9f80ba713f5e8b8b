#!/usr/bin/env python
"""Generate golden input/output vectors by running the UNMODIFIED reference rasterizer
(oracle/_ref, built from /root/reference by oracle/build_ref.py) on a GPU:

    gpurun -- 'python tests/golden/make_golden.py gpurun_out/golden'   # then copy *.npz to tests/golden/

The reference ships no fixtures of its own (SURVEY.md section 4), so these pin the CPU oracle
(tests/test_golden_cpu.py) and are a second parity target for the CUDA path.  Inputs are
regenerated from the recorded seeds by tests/util.small_scene (deterministic CPU generator)."""
import json
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
for p in (ROOT, os.path.join(ROOT, "dg-mesh_b200"), os.path.join(ROOT, "tests")):
    sys.path.insert(0, p)
import util  # noqa: E402
from test_raster_gpu import _cam_cuda, _cuda, run_ref  # noqa: E402

CASES = [
    dict(name="raster_sh3", n=1500, W=128, H=80, seed=3, scale=0.05, degree=3, colors=False, cov=False),
    dict(name="raster_sh1_odd", n=1200, W=99, H=70, seed=5, scale=0.08, degree=1, colors=False, cov=False),
    dict(name="raster_precomp", n=1000, W=96, H=64, seed=2, scale=0.05, degree=3, colors=True, cov=True),
]


def main(out_dir):
    os.makedirs(out_dir, exist_ok=True)
    for c in CASES:
        sc, cam = util.small_scene(n=c["n"], W=c["W"], H=c["H"], seed=c["seed"], scale=c["scale"], degree=c["degree"])
        bg = torch.tensor([1.0, 0.5, 0.25])
        dpix = torch.randn(3, c["H"], c["W"], generator=torch.Generator().manual_seed(1))
        r = run_ref(_cuda(sc), _cam_cuda(cam), bg.cuda(), c["degree"], c["colors"], c["cov"], dpix.cuda())
        arr = dict(meta=np.frombuffer(json.dumps(c).encode(), dtype=np.uint8), bg=bg.numpy(), dpix=dpix.numpy(),
                   num_rendered=np.int64(r["R"]))
        for k in ("radii", "tiles_touched", "depths", "means2D", "conic_opacity", "point_list_keys", "point_list",
                  "ranges", "n_contrib", "final_T", "color"):
            arr[k] = r[k].cpu().numpy()
        if not c["colors"]:
            arr["rgb"], arr["clamped"] = r["rgb"].cpu().numpy(), r["clamped"].cpu().numpy()
        if not c["cov"]:
            arr["cov3D"] = r["cov3D"].cpu().numpy()
        for k, g in r["grads"].items():
            if g is not None:
                arr["grad_" + k] = g.cpu().numpy()
        np.savez_compressed(os.path.join(out_dir, c["name"] + ".npz"), **arr)
        print(c["name"], "R =", r["R"])


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else os.path.join(ROOT, "gpurun_out", "golden"))
