#!/usr/bin/env python
"""Host-side overhead probe: tiny scene (GPU time negligible) -> wall time per forward+backward
call through the public API ~= CPU cost of the binding.  Prints ours vs the reference extension.
`--maps` times a call with extra maps instead (forward_surface with normals and camera_grad=True; ours only)."""
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "dg-mesh_b200"), os.path.join(ROOT, "tests")):
    sys.path.insert(0, p)
import torch  # noqa: E402
import synth  # noqa: E402
import util  # noqa: E402
import diff_gaussian_rasterization as dgr  # noqa: E402


def probe(mod, n_iter=300, maps=False):
    dev = torch.device("cuda", 0)
    sc = synth.gaussian_scene(n=256, seed=0, device=dev)
    cam = synth.look_at_camera(width=64, height=64, device=dev)
    bg = torch.ones(3, device=dev)
    leaves = {k: sc[k].clone().requires_grad_(True) for k in ("means3D", "opacities", "scales", "rotations", "shs")}
    dp = torch.randn(3, 64, 64, device=dev)
    rs = synth.raster_settings_for(cam, bg, settings_cls=mod.GaussianRasterizationSettings)
    r = mod.GaussianRasterizer(rs)

    m2d = torch.zeros_like(leaves["means3D"], requires_grad=True)
    normals = torch.nn.functional.normalize(torch.randn(256, 3, device=dev), dim=-1).requires_grad_(True)
    for t in (rs.viewmatrix, rs.projmatrix, rs.campos):
        t.requires_grad_(maps)

    def one():
        kw = dict(means3D=leaves["means3D"], means2D=m2d, opacities=leaves["opacities"], shs=leaves["shs"],
                  scales=leaves["scales"], rotations=leaves["rotations"])
        if maps:
            out = r.forward_surface(normals=normals, camera_grad=True, **kw)
            torch.autograd.backward([out[0], out[5], out[6]], [dp, dp[:1], dp])
        else:
            color, radii = r(**kw)
            color.backward(dp)

    for _ in range(20):
        one()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(n_iter):
        one()
    t1 = time.perf_counter()
    torch.cuda.synchronize()
    t2 = time.perf_counter()
    return (t1 - t0) / n_iter * 1e6, (t2 - t0) / n_iter * 1e6


if "--maps" in sys.argv:
    print("ours, forward_surface(normals, camera_grad): enqueue %.1f us/call, with final sync %.1f us/call"
          % probe(dgr, maps=True))
    sys.exit(0)
print("ours      : enqueue %.1f us/call, with final sync %.1f us/call" % probe(dgr))
ref = util.load_reference_rasterizer()
if ref is not None:
    print("reference : enqueue %.1f us/call, with final sync %.1f us/call" % probe(ref))
