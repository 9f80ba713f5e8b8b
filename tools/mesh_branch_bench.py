"""Cost of DG-Mesh's mesh branch for a frame batch: F = 8 frames, DPSR / marching cubes at G = 288, P = 100k
Gaussians, 800x800 cameras, alternating in one run

  (a) F calls of utils.renderer.mesh_renderer, then the losses and one backward;
  (b) one utils.renderer.mesh_renderer_batch, then the same losses and one backward.

Losses per frame: L1 of the mask and of the image against fixed targets, plus laplace_regularizer_const (called
per frame).  Reported: the step time of each arm (device events, median and range over --rounds rounds of --steps
steps each), the per-stage times of each arm measured on their own (DPSR forward, marching cubes including its
host wait, the two MLPs, rasterisation + interpolate + antialias with their backward), host waits per step,
peak memory per step, and the card's name and power limit read in the same run.

    python tools/mesh_branch_bench.py [--root TREE] [--arms ab] [--rounds 5] [--steps 3] [--no-stages] [--out FILE]

--root runs the package of another tree (e.g. a checkout of an earlier commit, for arm (a) only)."""
import argparse
import importlib
import json
import math
import os
import subprocess
import sys
import time
from types import SimpleNamespace

import numpy as np

ap = argparse.ArgumentParser()
ap.add_argument("--root", default=os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
ap.add_argument("--arms", default="ab")
ap.add_argument("--rounds", type=int, default=5)
ap.add_argument("--steps", type=int, default=3)
ap.add_argument("--frames", type=int, default=8)
ap.add_argument("--no-stages", action="store_true", help="step times only (e.g. for an earlier tree)")
ap.add_argument("--out", default=None)
args = ap.parse_args()
sys.path.insert(0, os.path.join(os.path.abspath(args.root), "dg-mesh_b200"))

import torch  # noqa: E402

import _dgm_lib  # noqa: E402
from diso import DiffMC  # noqa: E402
from nvdiffrast_utils.dpsr import DPSR  # noqa: E402
from nvdiffrast_utils.regularizer import laplace_regularizer_const  # noqa: E402

tu = importlib.import_module("utils.time_utils")
renderer = importlib.import_module("utils.renderer")
F, P, G, H, W, R = args.frames, 100_000, 288, 800, 800, 0.6


def camera(theta):
    c = np.array([3 * math.sin(theta), 0.3, 3 * math.cos(theta)], np.float32)
    z = c / np.linalg.norm(c)
    x = np.cross([0, 1, 0], z)
    x /= np.linalg.norm(x)
    y = np.cross(z, x)
    T = np.eye(4, dtype=np.float32)
    T[:3, 0], T[:3, 1], T[:3, 2], T[:3, 3] = x, y, z, c
    return SimpleNamespace(K=None, FoVx=0.8, FoVy=0.8, image_width=W, image_height=H, orig_transform=T)


torch.manual_seed(0)
d = torch.nn.functional.normalize(torch.randn(P, 3), dim=1).cuda()
xyz = (d * R).requires_grad_(True)
normal = d.clone().requires_grad_(True)
thres = torch.nn.Parameter(torch.tensor(0.0, device="cuda"))
gauss = SimpleNamespace(get_xyz=xyz, get_normal=normal, gaussian_center=torch.zeros(3, device="cuda"),
                        gaussian_scale=torch.tensor([1.0], device="cuda"), density_thres_param=thres,
                        dpsr=DPSR(res=(G, G, G), sig=2.0), diffmc=DiffMC())
back = SimpleNamespace(net=tu.DeformNetworkNormal(is_blender=True).cuda())
back.step = lambda x, t: back.net(x, t)
app = SimpleNamespace(net=tu.AppearanceNetwork(is_blender=True).cuda())
app.step = lambda x, t: app.net(x, t)
d_xyz = (0.03 * torch.randn(F, 1, 3)).cuda().expand(F, P, 3).contiguous()
fids = torch.linspace(0.05, 0.95, F, device="cuda").reshape(F, 1)
cams = [camera(2 * math.pi * k / F) for k in range(F)]
gt_mask = torch.zeros(H, W, 1, device="cuda")
gt_mask[H // 4:3 * H // 4, W // 4:3 * W // 4] = 1
gt_img = torch.rand(3, H, W, generator=torch.Generator().manual_seed(1)).cuda()
params = [xyz, normal, thres] + list(back.net.parameters()) + list(app.net.parameters())

waits = []
lib = _dgm_lib.lib()
_real_wait = lib.dgm_notify_wait


def _wait(h):
    waits.append(1)
    return _real_wait(h)


lib.dgm_notify_wait = _wait


def losses(mask, image, verts, faces):
    return (mask - gt_mask).abs().mean() + (image - gt_img).abs().mean() + laplace_regularizer_const(verts, faces)


def step_a():
    total = 0.0
    for k in range(F):
        m, img, v, f, _ = renderer.mesh_renderer(None, gauss, d_xyz[k], 0.0, fids[k], back, app,
                                                 viewpoint_cam=cams[k])
        total = total + losses(m, img, v, f)
    total.backward()


def step_b():
    m, img, v, f, _ = renderer.mesh_renderer_batch(None, gauss, d_xyz, 0.0, fids, back, app, viewpoint_cams=cams)
    total = sum(losses(m[k], img[k], v[k], f[k]) for k in range(F))
    total.backward()


ARMS = {"a": step_a, "b": step_b}


def zero():
    for p in params:
        p.grad = None


def time_arm(fn, steps):
    zero()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    n0 = len(waits)
    torch.cuda.reset_peak_memory_stats()
    e0.record()
    for _ in range(steps):
        fn()
        zero()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps, (len(waits) - n0) / steps, torch.cuda.max_memory_allocated() / 2 ** 30


def stage_times(arm, reps=3):
    """each stage of one arm's step on its own: device events around reps repetitions"""
    ev = lambda: torch.cuda.Event(enable_timing=True)  # noqa: E731
    out = {}
    with torch.no_grad():
        pts, nrm = renderer._dpsr_inputs(gauss, d_xyz, torch.zeros_like(d_xyz), False)

        def run(name, fn):
            fn()
            torch.cuda.synchronize()
            a, b = ev(), ev()
            a.record()
            for _ in range(reps):
                r = fn()
            b.record()
            torch.cuda.synchronize()
            out[name] = a.elapsed_time(b) / reps
            return r
        if arm == "a":
            psr = run("dpsr_fwd", lambda: [gauss.dpsr.forward_signed(pts[k:k + 1], nrm[k:k + 1], thres)
                                           for k in range(F)])
            mesh = run("mc_incl_wait", lambda: [gauss.diffmc(p) for p in psr])
            vl, fl = [m[0] for m in mesh], [m[1].int() for m in mesh]
            run("mlps", lambda: [app.step(v + back.step(v, fids[k].expand(v.shape[0], 1))[0],
                                          fids[k].expand(v.shape[0], 1)) for k, v in enumerate(vl)])
        else:
            psr = run("dpsr_fwd", lambda: gauss.dpsr.forward_signed(pts, nrm, thres))
            vl, fl = run("mc_incl_wait", lambda: gauss.diffmc.forward_batch(psr))
            fl = [f.int() for f in fl]
            va = torch.cat(vl)
            t = torch.repeat_interleave(fids, torch.tensor([v.shape[0] for v in vl], device="cuda"), dim=0)
            run("mlps", lambda: app.step(va + back.step(va, t)[0], t))
    vcol = [torch.rand(v.shape[0], 3, device="cuda") for v in vl]
    vl = [v.detach().requires_grad_(True) for v in vl]

    def raster_a():
        for k in range(F):
            pose, K, res = renderer._camera(cams[k])
            clip, rast, topo = renderer._raster(None, vl[k], fl[k], pose, K, res)
            m3 = renderer._mask_from(rast, clip, vl[k], fl[k], topo)
            img = renderer._image_from(rast, clip, fl[k], vcol[k], m3, False, topo)
            (m3.mean() + img.mean()).backward()

    def raster_b():
        import nvdiffrast.torch as dr
        cam = [renderer._camera(c) for c in cams]
        pos = torch.cat([renderer._clip(v, p, K, r)[0] for v, (p, K, r) in zip(vl, cam)])
        voff = np.cumsum([0] + [v.shape[0] for v in vl])
        nf = [f.shape[0] for f in fl]
        tri = torch.cat([f + int(o) for f, o in zip(fl, voff)]).int()
        ranges = torch.tensor([[sum(nf[:k]), nf[k]] for k in range(F)], dtype=torch.int32)
        rast, _ = dr.rasterize(None, pos, tri, resolution=[H, W], ranges=ranges)
        topo = dr.edge_opposites(tri, pos.shape[0])
        m3, _ = dr.interpolate(torch.ones(pos.shape[0], 3, device="cuda")[None], rast, tri)
        m3 = dr.antialias(m3, rast, pos, tri, topology_hash=topo)
        img, _ = dr.interpolate(torch.cat(vcol)[None], rast, tri)
        img = dr.antialias(img, rast, pos, tri, topology_hash=topo)
        (m3.mean() + img.mean()).backward()
    run_fn = raster_a if arm == "a" else raster_b
    run_fn()
    torch.cuda.synchronize()
    a, b = ev(), ev()
    a.record()
    for _ in range(reps):
        run_fn()
    b.record()
    torch.cuda.synchronize()
    out["raster_fwd_bwd"] = a.elapsed_time(b) / reps
    out["verts_per_frame"] = int(sum(v.shape[0] for v in vl) / F)
    return out


def main():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip().splitlines()
    res = {"card": q[0] if q else torch.cuda.get_device_name(), "root": os.path.abspath(args.root), "F": F, "P": P,
           "G": G, "HxW": [H, W], "arms": {}}
    arms = [a for a in "ab" if a in args.arms]
    for a in arms:                                   # warm-up: every shape the timed window uses
        ARMS[a]()
        zero()
    times = {a: [] for a in arms}
    for _ in range(args.rounds):                     # alternating rounds
        for a in arms:
            times[a].append(time_arm(ARMS[a], args.steps))
    for a in arms:
        ms = sorted(t[0] for t in times[a])
        res["arms"][a] = {"step_ms_median": ms[len(ms) // 2], "step_ms_range": [ms[0], ms[-1]],
                          "step_ms_all": [t[0] for t in times[a]], "host_waits_per_step": times[a][0][1],
                          "peak_mem_gib": max(t[2] for t in times[a]),
                          "stages_ms": "not measured" if args.no_stages else stage_times(a)}
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "a") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    t0 = time.time()
    main()
    print(f"wall {time.time() - t0:.1f} s", file=sys.stderr)
