#!/usr/bin/env python
"""Text timeline of one step of the bench's 8-frame dynamic batch (forward + backward): when each kernel of each frame reached the
front of its stream and when it finished (dgm_profile_enable(2); CUDA events on the internal streams)."""
import ctypes
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "dg-mesh_b200"), os.path.join(ROOT, "tests")):
    sys.path.insert(0, p)
import torch  # noqa: E402
import bench  # noqa: E402
import _dgm_lib  # noqa: E402
import diff_gaussian_rasterization as dgr  # noqa: E402

NAMES = ["preprocess", "tile_scan", "scatter", "sort_pack", "render_fwd", "render_bwd", "preprocess_bwd", "count"]
dev = torch.device("cuda")
sc, cams, dpix = bench.make_inputs(dev)
deltas = bench.make_deltas(sc, dev)
leaves, gflat, _ = bench.flat_params(sc, dev)
bg = torch.ones(3, device=dev)
settings = bench.batch_settings(dgr, cams, bg, list(range(bench.FRAMES)))
dp = torch.stack([d.to(dev) for d in dpix]).contiguous()


def step():
    gflat.zero_()
    bench.run_batch(dgr, leaves, settings, dp, deltas=deltas)


for _ in range(5):
    step()
torch.cuda.synchronize()
lib = _dgm_lib.lib()
lib.dgm_profile_enable(2)
step()
cap = 512
b, e, ids = (ctypes.c_float * cap)(), (ctypes.c_float * cap)(), (ctypes.c_int * cap)()
n = lib.dgm_timeline_read(b, e, ids, cap)
lib.dgm_profile_enable(0)
seen = {}
rows = []
for i in range(n):
    k = ids[i]
    f = seen.get(k, 0)
    seen[k] = f + 1
    rows.append((b[i], e[i], NAMES[k], f))
print(f"streams={os.environ.get('DGMESH_B200_STREAMS', 'default')}  launches={n}")
for bb, ee, name, f in sorted(rows, key=lambda r: r[1]):
    print(f"  end {ee*1e3:8.1f} us   front-of-stream {bb*1e3:8.1f} us   dur<= {1e3*(ee-bb):7.1f}   {name}[{f}]")
