"""Dual marching cubes (diso.DiffDMC) against marching cubes (diso.DiffMC) at G = 288, alternating in one run.

Fields: the DPSR field of a synth.py Gaussian scene (P = 100k, the means as points, their normals) and the signed
distance of a sphere joined with a tilted torus.  Per extractor and field:
  - forward (including its one host wait) + backward of L = sum(verts^2), for B = 1 and for a batch of B = 8 grids
    (forward_batch), device-synchronised wall time, median and range over --rounds rounds of --steps steps;
  - V and F, and triangle quality: 1/5/50 % percentiles of the minimum angle, the share of triangles with a minimum
    angle below 10 degrees, and the largest aspect ratio (`quality`).  The same figures from the CPU reference
    meshes (tests/mc_reference.py, tests/dmc_reference.py) are checked to agree;
  - one mesh_renderer_batch step (F = 8 frames at 800x800, 100k Gaussians on a sphere, L1 losses + backward) with
    each extractor as `gaussians.diffmc`.
--profile runs torch.profiler over a few forward + backward calls instead and prints the kernel times.
The card's name and power limit are read in the same run.

    python tools/dmc_bench.py [--rounds 5] [--steps 5] [--profile] [--out FILE]"""
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

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [os.path.join(ROOT, "dg-mesh_b200"), os.path.join(ROOT, "tests")]
ap = argparse.ArgumentParser()
ap.add_argument("--rounds", type=int, default=5)
ap.add_argument("--steps", type=int, default=5)
ap.add_argument("--profile", action="store_true")
ap.add_argument("--renderer-only", action="store_true", help="only the mesh_renderer_batch step times")
ap.add_argument("--out", default=None)
args = ap.parse_args()

import torch  # noqa: E402

from diso import DiffDMC, DiffMC  # noqa: E402
from dmc_reference import dmc_reference  # noqa: E402
from mc_reference import mc_reference  # noqa: E402
from nvdiffrast_utils.dpsr import DPSR  # noqa: E402
import synth  # noqa: E402

G = 288


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip().splitlines()
    return q[torch.cuda.current_device()] if q else torch.cuda.get_device_name()


def fields():
    sc = synth.gaussian_scene(100_000, seed=0, device="cuda")
    pts = (sc["means3D"] / 1.3 * 0.45 + 0.5)[None]
    with torch.no_grad():
        dpsr = DPSR(res=(G, G, G), sig=2.0)(pts, sc["normals"][None])[0].float()
    x = torch.linspace(-1, 1, G, device="cuda")
    X, Y, Z = torch.meshgrid(x, x, x, indexing="ij")
    sph = (X + 0.35) ** 2 + Y ** 2 + Z ** 2
    c, s = math.cos(0.5), math.sin(0.5)
    ty, tz = c * Y - s * Z, s * Y + c * Z
    q = torch.sqrt((X - 0.35) ** 2 + ty ** 2) - 0.4
    tor = torch.sqrt(q * q + tz * tz) - 0.15
    st = torch.minimum(torch.sqrt(sph) - 0.4, tor)
    return {"dpsr": dpsr.contiguous(), "sphere_torus": st.contiguous()}


def quality(v, f):
    """(min-angle 1/5/50 % percentiles in degrees, share of triangles with a minimum angle < 10 degrees, largest
    aspect ratio = longest edge * (sum of edge lengths) / (4 sqrt(3) area), 1 for an equilateral triangle)."""
    p = np.asarray(v, np.float64)[np.asarray(f)]
    e = [p[:, 1] - p[:, 0], p[:, 2] - p[:, 1], p[:, 0] - p[:, 2]]
    ln = np.stack([np.linalg.norm(x, axis=1) for x in e], 1)
    area = 0.5 * np.linalg.norm(np.cross(e[0], -e[2]), axis=1)
    ang = []
    for i in range(3):
        a, b = -e[(i + 2) % 3], e[i]
        cosv = (a * b).sum(1) / np.maximum(ln[:, (i + 2) % 3] * ln[:, i], 1e-300)
        ang.append(np.degrees(np.arccos(np.clip(cosv, -1, 1))))
    mn = np.min(np.stack(ang, 1), 1)
    ar = ln.max(1) * ln.sum(1) / np.maximum(4 * math.sqrt(3) * area, 1e-300)
    return {"min_angle_p1": float(np.percentile(mn, 1)), "min_angle_p5": float(np.percentile(mn, 5)),
            "min_angle_p50": float(np.percentile(mn, 50)), "share_below_10deg": float((mn < 10).mean()),
            "max_aspect": float(ar.max())}


def run(ext, grids, batch):
    g = grids.detach().requires_grad_(True)
    if batch:
        vl, _ = ext.forward_batch(g)
        loss = sum(v.square().sum() for v in vl)
    else:
        v, _ = ext(g[0])
        loss = v.square().sum()
    loss.backward()


def timed(fn):
    out = []
    for _ in range(args.rounds):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(args.steps):
            fn()
        torch.cuda.synchronize()
        out.append((time.perf_counter() - t0) * 1e3 / args.steps)
    return float(np.median(out)), float(min(out)), float(max(out))


def camera(theta, H, W):
    """a camera on a circle of radius 3 around the origin, looking at it (blender / OpenGL pose)"""
    c = np.array([3 * math.sin(theta), 0.3, 3 * math.cos(theta)], np.float32)
    z = c / np.linalg.norm(c)
    x = np.cross([0, 1, 0], z)
    x /= np.linalg.norm(x)
    y = np.cross(z, x)
    T = np.eye(4, dtype=np.float32)
    T[:3, 0], T[:3, 1], T[:3, 2], T[:3, 3] = x, y, z, c
    return SimpleNamespace(K=None, FoVx=0.8, FoVy=0.8, image_width=W, image_height=H, orig_transform=T)


def renderer_arm(ext):
    tu = importlib.import_module("utils.time_utils")
    renderer = importlib.import_module("utils.renderer")
    torch.manual_seed(0)
    n, Fr, H, W, R = 100_000, 8, 800, 800, 0.6
    d = torch.nn.functional.normalize(torch.randn(n, 3), dim=1).cuda()
    xyz, normal = (d * R).requires_grad_(True), d.clone().requires_grad_(True)
    gauss = SimpleNamespace(get_xyz=xyz, get_normal=normal, gaussian_center=torch.zeros(3, device="cuda"),
                            gaussian_scale=torch.tensor([1.0], device="cuda"),
                            density_thres_param=torch.nn.Parameter(torch.tensor(0.0, device="cuda")),
                            dpsr=DPSR(res=(G, G, G), sig=2.0), diffmc=ext)
    back = SimpleNamespace(net=tu.DeformNetworkNormal(is_blender=True).cuda())
    back.step = lambda x, t: back.net(x, t)
    app = SimpleNamespace(net=tu.AppearanceNetwork(is_blender=True).cuda())
    app.step = lambda x, t: app.net(x, t)
    d_xyz = (0.03 * torch.randn(Fr, 1, 3, device="cuda")).expand(Fr, n, 3)
    fids = torch.linspace(0.1, 0.9, Fr, device="cuda")[:, None]
    cams = [camera(0.4 * k, H, W) for k in range(Fr)]

    def step():
        masks, images, _, _, _ = renderer.mesh_renderer_batch(None, gauss, d_xyz, 0.0, fids, back, app,
                                                              viewpoint_cams=cams)
        (masks.mean() + images.mean()).backward()
    return step


def main():
    info = {"card": card(), "G": G}
    print(json.dumps(info), flush=True)
    exts = {"mc": DiffMC(), "dmc": DiffDMC()}
    fl = fields()
    if args.profile:
        from torch.profiler import ProfilerActivity, profile
        for name, phi in fl.items():
            for en, ext in exts.items():
                for _ in range(2):
                    run(ext, phi[None], False)
                with profile(activities=[ProfilerActivity.CUDA]) as prof:
                    for _ in range(5):
                        run(ext, phi[None], False)
                    torch.cuda.synchronize()
                ks = {e.key: round(e.device_time_total / 5 / 1e3, 4) for e in prof.key_averages()
                      if e.device_time_total > 0 and ("mc_" in e.key or "Scan" in e.key or "totals" in e.key)}
                print(json.dumps({"field": name, "extractor": en, "kernel_ms_per_call": ks}), flush=True)
        return
    res = dict(info, fields={})
    for name, phi in ({} if args.renderer_only else fl).items():
        r = res["fields"][name] = {}
        batch = phi[None].expand(8, G, G, G).contiguous()
        for en, ext in exts.items():
            v, f = ext(phi)
            r[en] = {"V": int(v.shape[0]), "F": int(f.shape[0]), **quality(v.cpu().numpy(), f.cpu().numpy())}
        host = phi.cpu().numpy()
        ref = {"mc": mc_reference(host), "dmc": dmc_reference(host)}
        for en in exts:   # the reference gives the same meshes, so the same figures
            q = {"V": len(ref[en].verts), "F": len(ref[en].faces), **quality(ref[en].verts, ref[en].faces)}
            r[en]["reference_agrees"] = q == {k: r[en][k] for k in q}
        for _ in range(2):
            for ext in exts.values():
                run(ext, phi[None], False)
                run(ext, batch, True)
        t = {en: {"B1": [], "B8": []} for en in exts}
        for _ in range(2):   # alternate the arms
            for en, ext in exts.items():
                t[en]["B1"].append(timed(lambda: run(ext, phi[None], False)))
                t[en]["B8"].append(timed(lambda: run(ext, batch, True)))
        for en in exts:
            for b in ("B1", "B8"):
                med = [x[0] for x in t[en][b]]
                r[en][f"fwd_bwd_ms_{b}"] = [round(float(np.median(med)), 3), round(min(x[1] for x in t[en][b]), 3),
                                            round(max(x[2] for x in t[en][b]), 3)]
        print(json.dumps({name: r}), flush=True)
        del batch
    steps = {en: renderer_arm(ext) for en, ext in exts.items()}
    for s in steps.values():
        s()
    tt = {en: [] for en in exts}
    for _ in range(2):
        for en, s in steps.items():
            tt[en].append(timed(s))
    res["mesh_renderer_batch_F8_ms"] = {en: [round(float(np.median([x[0] for x in v])), 2),
                                             round(min(x[1] for x in v), 2), round(max(x[2] for x in v), 2)]
                                        for en, v in tt.items()}
    print(json.dumps(res))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as fh:
            json.dump(res, fh, indent=1)


if __name__ == "__main__":
    main()
