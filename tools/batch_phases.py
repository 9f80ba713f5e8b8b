#!/usr/bin/env python
"""Where does a frame batch spend its time?  Times the forward and backward halves of the bench's headline
step (the 8-frame dynamic batch: per-frame deformed means / scales / rotations, shared opacity and SH)
separately, with CUDA events and a synchronise between the halves."""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "dg-mesh_b200"), os.path.join(ROOT, "tests")):
    sys.path.insert(0, p)
import torch  # noqa: E402
import bench  # noqa: E402
import diff_gaussian_rasterization as dgr  # noqa: E402

dev = torch.device("cuda")
sc, cams, dpix = bench.make_inputs(dev)
deltas = bench.make_deltas(sc, dev)
leaves, gflat, _ = bench.flat_params(sc, dev)
bg = torch.ones(3, device=dev)
frames = list(range(bench.FRAMES))
settings = bench.batch_settings(dgr, cams, bg, frames)
dp = torch.stack([d.to(dev) for d in dpix]).contiguous()


def ev():
    return torch.cuda.Event(enable_timing=True)


fw, bw = [], []
for it in range(24):
    gflat.zero_()
    torch.cuda.synchronize()
    e0, e1 = ev(), ev()
    e0.record()
    color, radii = dgr.BatchGaussianRasterizer(settings)(
        means3D=leaves["means3D"][None] + deltas["means3D"], means2D=None, opacities=leaves["opacities"],
        shs=leaves["shs"], scales=leaves["scales"][None] + deltas["scales"],
        rotations=leaves["rotations"][None] + deltas["rotations"])
    e1.record()
    torch.cuda.synchronize()
    e1b, e2 = ev(), ev()
    e1b.record()
    color.backward(dp)
    e2.record()
    torch.cuda.synchronize()
    if it >= 4:
        fw.append(e0.elapsed_time(e1))
        bw.append(e1b.elapsed_time(e2))
fw.sort()
bw.sort()
print(f"streams={os.environ.get('DGMESH_B200_STREAMS', 'default')}  {bench.FRAMES} frames: "
      f"forward median {fw[len(fw) // 2]:.3f} ms, backward median {bw[len(bw) // 2]:.3f} ms "
      f"(min {bw[0]:.3f}, max {bw[-1]:.3f}) over {len(bw)} steps")
