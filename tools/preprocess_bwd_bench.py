#!/usr/bin/env python
"""The per-Gaussian backward (`preprocess_bwd_kernel`) on the bench scene, alone.

    python tools/preprocess_bwd_bench.py [--steps N]          # kernel time (CUDA events, dgm_profile_*), F = 1 and 8
    python tools/preprocess_bwd_bench.py --dump-preprocess-bwd DIR [--snapshot DIR0]
    python tools/preprocess_bwd_bench.py --compare-dumps DIR_A DIR_B

Timing: the one-frame launch (`dgr_backward`) and the 8-frame dynamic batch launch (`dgr_backward_batch`: per-frame
means / scales / rotations, shared opacity and SH), each as the mean of the kernel's own event time over N steps,
set against DESIGN.md's compulsory traffic (643 P bytes for one frame, F 219 P + 388 P for the batch), with the
card's name, power limit and SM clock read in the same run.

Dump: the kernel uses no atomics, so for a fixed `grad_acc` (the moments render_bwd leaves per frame) its outputs
are deterministic.  The dump renders each frame once through the one-frame API and recovers that frame's
`grad_acc` exactly from the gradients the kernel copies out of it (2D mean, conic, opacity, colour); this snapshot
is saved (or loaded from --snapshot DIR0, so that two builds of the library see the same one).  It then writes
the snapshot into the workspaces of a fresh forward, runs the backward with a zero pixel gradient (render_bwd
adds nothing) and saves every output of the per-Gaussian backward for F = 1 and F = 8, on the bench scene
(P = 100 000) and on its first 99 989 Gaussians (P not a multiple of 32).  --compare-dumps checks two such
directories bit for bit."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "dg-mesh_b200"), os.path.join(ROOT, "tests")):
    sys.path.insert(0, p)

FRAMES = 8
SCENES = {"bench": 100_000, "odd": 99_989}


def card():
    import torch
    q = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm",
                        "--format=csv,noheader,nounits"], capture_output=True, text=True).stdout.strip()
    name, plim, sm, smax = [c.strip() for c in q.split(",")] if q.count(",") == 3 else (None,) * 4
    return {"name": torch.cuda.get_device_name(0), "power_limit_w": plim, "sm_mhz": sm, "sm_max_mhz": smax,
            "smi_name": name}


def setup(P):
    import torch
    import bench
    import diff_gaussian_rasterization as dgr
    dev = torch.device("cuda")
    sc, cams, dpix = bench.make_inputs(dev)
    sc = {k: v[:P].contiguous() for k, v in sc.items()}
    deltas = bench.make_deltas(sc, dev)
    bg = torch.ones(3, device=dev)
    settings = bench.batch_settings(dgr, cams, bg, list(range(FRAMES)))
    dpix = torch.stack([d.to(dev) for d in dpix]).contiguous()
    return sc, deltas, settings, dpix


def frame_params(sc, deltas, f):
    return {"means3D": sc["means3D"] + deltas["means3D"][f], "scales": sc["scales"] + deltas["scales"][f],
            "rotations": sc["rotations"] + deltas["rotations"][f]}


def time_kernel(steps, warmup):
    import torch
    import _dgm_lib
    import bench
    import diff_gaussian_rasterization as dgr
    sc, deltas, settings, dpix = setup(SCENES["bench"])
    P = SCENES["bench"]
    leaves = {k: v.clone().requires_grad_(True) for k, v in sc.items()}
    lib = _dgm_lib.lib()

    def one(f):
        fp = frame_params(leaves, deltas, f)
        color, _ = dgr.GaussianRasterizer(settings[f])(means3D=fp["means3D"], means2D=None,
                                                       opacities=leaves["opacities"], shs=leaves["shs"],
                                                       scales=fp["scales"], rotations=fp["rotations"])
        color.backward(dpix[f])

    def batch(_):
        bench.run_batch(dgr, leaves, settings, dpix, deltas=deltas)

    out = {}
    for name, fn, nbytes in (("F1", one, 643 * P), ("F8", batch, FRAMES * 219 * P + 388 * P)):
        for i in range(warmup):
            fn(i % FRAMES)
        torch.cuda.synchronize()
        lib.dgm_profile_enable(1)
        ms = []
        for i in range(steps):
            fn(i % FRAMES)
            ms.append(_dgm_lib.profile_read()["preprocess_bwd"])
        lib.dgm_profile_enable(0)
        t = float(np.mean(ms))
        out[name] = {"ms": t, "ms_median": float(np.median(ms)), "alg_bytes": nbytes, "GBps": nbytes / (t * 1e-3) / 1e9}
    out["card"] = card()
    return out


def grad_acc_view(buf, geom_addr, P):
    """[P,12] float32 view of grad_acc in the per-Gaussian workspace at geom_addr (GeomWS::from's layout: each
    array starts at the next 128-byte boundary)."""
    p = geom_addr
    for nbytes in (4 * P, 3 * P, 4 * P, 8 * P, 24 * P, 16 * P, 12 * P, 4 * P):
        p = (p + 127) // 128 * 128 + nbytes
    import torch
    o = (p + 127) // 128 * 128 - buf.data_ptr()
    return buf[o:o + 48 * P].view(torch.float32).view(P, 12)


def one_frame_backward(P, s, ws, radii, sc, fp, dpix):
    """dgr_backward on the one-frame workspace ws: the nine outputs of the per-Gaussian backward."""
    import torch
    import _dgm_lib
    dev = dpix.device
    e = lambda *shape: torch.empty(shape, device=dev)  # noqa: E731
    o = {"mean2D": e(P, 3), "conic": e(P, 2, 2), "opacity": e(P, 1), "color": e(P, 3), "mean3D": e(P, 3),
         "cov3D": e(P, 6), "sh": e(P, 16, 3), "scale": e(P, 3), "rotation": e(P, 4)}
    p = _dgm_lib.ptr
    rc = _dgm_lib.lib().dgr_backward(
        P, s.sh_degree, 16, p(s.bg), int(s.image_width), int(s.image_height), p(fp["means3D"]), p(sc["shs"]), None,
        p(fp["scales"]), float(s.scale_modifier), p(fp["rotations"]), None, p(s.viewmatrix), p(s.projmatrix),
        p(s.campos), float(s.tanfovx), float(s.tanfovy), p(radii), ws.geom, ws.binning, ws.R_cap, ws.img,
        p(dpix), *[p(o[k]) for k in ("mean2D", "conic", "opacity", "color", "mean3D", "cov3D", "sh", "scale",
                                      "rotation")], _dgm_lib.stream_ptr())
    _dgm_lib.check(rc, "dgr_backward")
    return o


def one_frame_forward(sc, deltas, settings, f):
    import diff_gaussian_rasterization as dgr
    fp = {k: v.detach().requires_grad_(True) for k, v in frame_params(sc, deltas, f).items()}
    color, radii = dgr.GaussianRasterizer(settings[f])(means3D=fp["means3D"], means2D=None,
                                                       opacities=sc["opacities"], shs=sc["shs"],
                                                       scales=fp["scales"], rotations=fp["rotations"])
    return fp, color.grad_fn.ws, radii


def snapshot(P, sc, deltas, settings, dpix):
    """grad_acc of every frame after render_bwd, recovered from the values the kernel copies out of it."""
    import torch
    snap = []
    for f in range(FRAMES):
        fp, ws, radii = one_frame_forward(sc, deltas, settings, f)
        o = one_frame_backward(P, settings[f], ws, radii, sc, fp, dpix[f])
        con = o["conic"].reshape(P, 4)
        z = torch.zeros(P, device=dpix.device)
        snap.append(torch.stack([o["mean2D"][:, 0], o["mean2D"][:, 1], con[:, 0], con[:, 1], con[:, 3],
                                 o["opacity"][:, 0], o["color"][:, 0], o["color"][:, 1], o["color"][:, 2], z, z, z], 1))
    return torch.stack(snap)


def dump(out_dir, snap_dir):
    import torch
    import diff_gaussian_rasterization as dgr
    os.makedirs(out_dir, exist_ok=True)
    report = {}
    for scene, P in SCENES.items():
        sc, deltas, settings, dpix = setup(P)
        path = os.path.join(snap_dir or out_dir, f"snapshot_{scene}.npy")
        if snap_dir:
            snap = torch.from_numpy(np.load(path)).cuda()
        else:
            snap = snapshot(P, sc, deltas, settings, dpix)
            np.save(path, snap.cpu().numpy())
        zero = torch.zeros_like(dpix[0])
        save = lambda name, t: np.save(os.path.join(out_dir, f"{scene}_{name}.npy"),  # noqa: E731
                                       t.detach().float().cpu().numpy())
        # one frame (dgr_backward): frame 0
        fp, ws, radii = one_frame_forward(sc, deltas, settings, 0)
        acc = grad_acc_view(ws.buf, ws.geom, P)
        acc.copy_(snap[0])
        o = one_frame_backward(P, settings[0], ws, radii, sc, fp, zero)
        assert torch.equal(o["mean2D"][:, :2], snap[0][:, :2]), "grad_acc layout / zero-gradient premise"
        assert not acc.any(), "grad_acc not re-zeroed"
        for k, v in o.items():
            save(f"F1_{k}", v)
        # 8-frame dynamic batch (dgr_backward_batch)
        leaves = {k: v.detach().clone().requires_grad_(True) for k, v in sc.items() if k in ("opacities", "shs")}
        pf = {k: torch.stack([frame_params(sc, deltas, f)[k] for f in range(FRAMES)]).detach().requires_grad_(True)
              for k in ("means3D", "scales", "rotations")}
        m2d = torch.zeros(FRAMES, P, 3, device=dpix.device, requires_grad=True)
        color, _ = dgr.BatchGaussianRasterizer(settings)(means3D=pf["means3D"], means2D=m2d, **leaves,
                                                         scales=pf["scales"], rotations=pf["rotations"])
        ws = color.grad_fn.ws
        for f in range(FRAMES):
            grad_acc_view(ws.buf, ws.geom + f * ws.gs, P).copy_(snap[f])
        color.backward(torch.zeros_like(color))
        assert torch.equal(m2d.grad[..., :2], snap[..., :2]), "grad_acc layout / zero-gradient premise"
        for k, v in (("mean2D", m2d), ("mean3D", pf["means3D"]), ("scale", pf["scales"]),
                     ("rotation", pf["rotations"]), ("opacity", leaves["opacities"]), ("sh", leaves["shs"])):
            save(f"F8_{k}", v.grad)
        report[scene] = {"P": P, "visible_frac_frame0": float((snap[0].abs().sum(1) > 0).float().mean())}
    print(json.dumps({"dump": out_dir, "snapshot": snap_dir or out_dir, **report}))


def compare(a, b):
    names = sorted(f for f in os.listdir(b) if f.endswith(".npy") and not f.startswith("snapshot_"))
    assert names, f"no dump in {b}"
    out, ok = {}, True
    for f in names:
        x, y = np.load(os.path.join(a, f)), np.load(os.path.join(b, f))
        same = x.shape == y.shape and bool(np.array_equal(x.view(np.uint32), y.view(np.uint32)))
        out[f] = same
        ok &= same
    print(json.dumps({"bit_identical": ok, "arrays": len(names), "per_array": out}))
    return 0 if ok else 1


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=100)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--dump-preprocess-bwd", metavar="DIR")
    ap.add_argument("--snapshot", metavar="DIR0", help="load the grad_acc snapshots saved by an earlier dump")
    ap.add_argument("--compare-dumps", nargs=2, metavar=("DIR_A", "DIR_B"))
    a = ap.parse_args()
    if a.compare_dumps:
        return compare(*a.compare_dumps)
    import torch
    assert torch.cuda.is_available(), "needs a GPU"
    if a.dump_preprocess_bwd:
        dump(a.dump_preprocess_bwd, a.snapshot)
        return 0
    print(json.dumps(time_kernel(a.steps, a.warmup)))
    return 0


if __name__ == "__main__":
    sys.exit(main())
