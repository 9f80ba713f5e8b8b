#!/usr/bin/env python
"""TEST INFRASTRUCTURE: run the reference's dgmesh/train.py UNMODIFIED (the copy under oracle/_ref/dgmesh,
made by oracle/build_ref.py) for a few dozen iterations on a synthetic D-NeRF-shaped scene, on either stack:

    python tools/train_harness.py --stack ours        # dg-mesh_b200/launch.py resolution order (drop-ins win)
    python tools/train_harness.py --stack reference   # the reference's own modules + its stock CUDA extensions

and print ONE JSON line: per-iteration loss, image checksum, number of Gaussians and ms per iteration, plus
which file every replaced module resolved to.  `--compare a.json b.json` checks two such lines against each
other.  The script is run as `__main__` through runpy, exactly as `python train.py --config ...` would; the
only interventions are (1) stand-ins for third-party packages that are not installed (tools/harness_stubs.py),
(2) observation hooks (the scalar passed to `.backward()`, `render()`'s image, an iteration counter that ends
the run after --iters iterations instead of training 25 000), none of which touches the numerics.

Phases (config keys of the reference): iterations < warm_up render the canonical Gaussians; from warm_up on the
deformation MLPs run; from dpsr_iter on the mesh branch (DPSR -> marching cubes -> mesh rasteriser -> mesh
losses) runs too -- that needs a mesh rasteriser, which only the 'ours' stack has offline (the reference's is
nvdiffrast), so `--dpsr-iter` defaults to "never" for a two-stack comparison."""
import argparse
import json
import math
import os
import runpy
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_TREE = os.path.join(ROOT, "oracle", "_ref", "dgmesh")
sys.path.insert(0, os.path.join(ROOT, "tools"))


def make_dataset(path, n_train=12, n_test=2, size=200, seed=0):
    """A D-NeRF-shaped folder: transforms_{train,test}.json + RGBA PNGs of a few coloured blobs that move with
    time, seen from cameras on a ring (camera_angle_x = 0.6911, radius 4: the D-NeRF intrinsics)."""
    import numpy as np
    from PIL import Image
    os.makedirs(os.path.join(path, "train"), exist_ok=True)
    os.makedirs(os.path.join(path, "test"), exist_ok=True)
    rng = np.random.default_rng(seed)
    fovx = 0.6911112070083618
    focal = 0.5 * size / math.tan(0.5 * fovx)
    centers = rng.uniform(-0.5, 0.5, (6, 3))
    vel = rng.uniform(-0.4, 0.4, (6, 3))
    colors = rng.uniform(0.2, 1.0, (6, 3))
    sigma = rng.uniform(0.12, 0.25, 6)

    def frame(az, el, t):
        # Blender / OpenGL camera-to-world looking at the origin from radius 4
        pos = 4.0 * np.array([math.cos(el) * math.cos(az), math.cos(el) * math.sin(az), math.sin(el)])
        fwd = -pos / np.linalg.norm(pos)
        right = np.cross(fwd, np.array([0.0, 0.0, 1.0]))
        right /= np.linalg.norm(right)
        up = np.cross(right, fwd)
        c2w = np.eye(4)
        c2w[:3, 0], c2w[:3, 1], c2w[:3, 2], c2w[:3, 3] = right, up, -fwd, pos
        w2c = np.linalg.inv(c2w)
        ys, xs = np.mgrid[0:size, 0:size]
        rgb = np.zeros((size, size, 3))
        trans = np.ones((size, size))
        pts = centers + vel * t
        cam = (w2c[:3, :3] @ pts.T).T + w2c[:3, 3]
        for i in np.argsort(cam[:, 2]):             # OpenGL: camera looks down -z, nearest has the largest z
            x, y, z = cam[i]
            u, v = size / 2 + focal * x / -z, size / 2 - focal * y / -z
            s = focal * sigma[i] / -z
            a = 0.95 * np.exp(-((xs + 0.5 - u) ** 2 + (ys + 0.5 - v) ** 2) / (2 * s * s))
            rgb = rgb * (1 - a[..., None]) + colors[i] * a[..., None]   # back-to-front "over"
            trans = trans * (1 - a)
        alpha = 1 - trans
        with np.errstate(invalid="ignore", divide="ignore"):
            straight = np.where(alpha[..., None] > 1e-6, rgb / np.maximum(alpha[..., None], 1e-6), 0.0)
        img = np.concatenate([np.clip(straight, 0, 1), alpha[..., None]], -1)
        return c2w, (img * 255 + 0.5).astype(np.uint8)

    for split, n in (("train", n_train), ("test", n_test)):
        frames = []
        for k in range(n):
            t = k / n
            c2w, img = frame(2 * math.pi * k / n + (0.3 if split == "test" else 0.0), 0.35, t)
            name = f"{split}/r_{k:03d}"
            Image.fromarray(img, "RGBA").save(os.path.join(path, name + ".png"))
            frames.append({"file_path": "./" + name, "rotation": 0.0, "time": t, "transform_matrix": c2w.tolist()})
        with open(os.path.join(path, f"transforms_{split}.json"), "w") as f:
            json.dump({"camera_angle_x": fovx, "frames": frames}, f)


def write_config(path, data_dir, out_dir, a):
    import yaml
    cfg = dict(source_path=data_dir, model_path=out_dir, downsample=1.0, white_background=True, eval=True,
               is_blender=True, iterations=1_000_000, warm_up=a.warm_up,
               # as in the reference's configs (densify_until_iter 15 000 < anchor_iter 16 000): train.py's
               # densification bookkeeping (:489-496) indexes with the pre-anchor visibility mask
               densify_until_iter=min(1_000_000, a.anchor_iter),
               densify_from_iter=a.densify_from, densification_interval=a.densify_every,
               opacity_reset_interval=1_000_000, dpsr_iter=a.dpsr_iter, dpsr_sig=3.0, grid_res=a.grid_res,
               gaussian_ratio=1.2, init_density_threshold=0.0, mask_loss_weight=1.0, mesh_img_loss_weight=1.0,
               laplacian_loss_weight=1.0, use_anchor=1.0 if a.anchor_iter < 1_000_000 else 0.0,
               anchor_iter=a.anchor_iter, anchor_n_1_bs=128, anchor_0_1_bs=128, anchor_search_radius=0.0015,
               anchor_interval=a.anchor_every, normal_warm_up=a.normal_warm_up)
    with open(path, "w") as f:
        yaml.safe_dump(cfg, f)


class _Stop(Exception):
    pass


def run(a):
    import numpy as np
    import torch
    if a.stack == "ours":            # before the stand-ins: `diso`, `simple_knn` ... are real modules on this stack
        sys.path.insert(0, os.path.join(ROOT, "dg-mesh_b200"))
    import harness_stubs
    harness_stubs.install()
    work = a.work or f"/tmp/dgmesh_harness_{a.stack}"
    data, out = os.path.join(work, "data"), os.path.join(work, "out")
    os.makedirs(out, exist_ok=True)
    if not os.path.exists(os.path.join(data, "transforms_train.json")):
        make_dataset(data, size=a.size)
    cfg = os.path.join(work, "cfg.yaml")
    write_config(cfg, data, out, a)
    if not os.path.isdir(REF_TREE):
        print(json.dumps({"unavailable": "oracle/_ref/dgmesh missing: run oracle/build_ref.py"}))
        return 0
    if a.stack == "ours":
        sys.path.insert(0, os.path.join(ROOT, "dg-mesh_b200"))
        import launch
        launch.install(REF_TREE)
        resolved = launch.resolved()
    else:
        # the reference's own stack: its python modules + its stock extensions built for sm_90a
        sys.path.insert(0, REF_TREE)
        sys.path.insert(0, os.path.join(ROOT, "oracle", "_ref"))
        resolved = {}
        for name in ("gaussian_renderer", "utils.time_utils", "utils.loss_utils", "diff_gaussian_rasterization",
                     "simple_knn._C"):
            try:
                resolved[name] = __import__(name, fromlist=["x"]).__file__
            except Exception as e:
                resolved[name] = f"<{type(e).__name__}: {e}>"

    # ---- observation hooks
    rec = {"loss": [], "img_mean": [], "n_gauss": [], "iter_ms": []}
    state = {"n": 0, "ev": None}
    orig_backward = torch.Tensor.backward

    def backward(self, *args, **kw):
        if self.numel() == 1 and self.dim() == 0 and not args and not kw:
            rec["loss"].append(float(self.detach()))
        return orig_backward(self, *args, **kw)

    torch.Tensor.backward = backward
    import gaussian_renderer
    orig_render = gaussian_renderer.render

    def render(*args, **kw):
        pkg = orig_render(*args, **kw)
        if torch.is_grad_enabled():
            rec["img_mean"].append(float(pkg["render"].detach().mean()))
            rec["n_gauss"].append(int(pkg["radii"].shape[0]))
        return pkg

    gaussian_renderer.render = render
    import scene
    gm = scene.GaussianModelDPSRDynamicAnchor
    orig_lr = gm.update_learning_rate

    def update_learning_rate(self, iteration):
        ev = torch.cuda.Event(enable_timing=True)
        ev.record()
        if state["ev"] is not None:
            state["ev"].synchronize()
            ev.synchronize()
            rec["iter_ms"].append(state["ev"].elapsed_time(ev))
        state["ev"] = ev
        state["n"] += 1
        if state["n"] > a.iters:
            raise _Stop()
        return orig_lr(self, iteration)

    gm.update_learning_rate = update_learning_rate
    t0 = time.time()
    real_stdout = sys.stdout          # safe_state(quiet) replaces sys.stdout with a silent writer
    sys.argv = [os.path.join(REF_TREE, "train.py"), "--config", cfg, "--quiet", "--log_every", "100000000"]
    cwd = os.getcwd()
    os.chdir(REF_TREE)
    err = None
    prof = None
    if os.environ.get("HARNESS_CPROFILE"):
        import cProfile
        prof = cProfile.Profile()
        prof.enable()
    try:
        runpy.run_path(os.path.join(REF_TREE, "train.py"), run_name="__main__")
    except _Stop:
        pass
    except BaseException as e:  # reported in the JSON line, with where it happened
        import traceback
        err = f"{type(e).__name__}: {e} @ " + " <- ".join(
            f"{os.path.basename(f.filename)}:{f.lineno}" for f in traceback.extract_tb(e.__traceback__)[-4:])
    finally:
        if prof is not None:
            import pstats
            prof.disable()
            pstats.Stats(prof, stream=sys.stderr).sort_stats("cumulative").print_stats(45)
        os.chdir(cwd)
        sys.stdout = real_stdout
        torch.Tensor.backward = orig_backward
    out_line = {"stack": a.stack, "iters_done": len(rec["loss"]), "error": err, "wall_s": round(time.time() - t0, 1),
                "image": [a.size, a.size], "config": {"warm_up": a.warm_up, "dpsr_iter": a.dpsr_iter,
                                                      "densify_from": a.densify_from, "densify_every": a.densify_every,
                                                      "anchor_iter": a.anchor_iter, "anchor_every": a.anchor_every},
                "loss": rec["loss"], "img_mean": rec["img_mean"], "n_gauss": rec["n_gauss"],
                "iter_ms_median_last_half": (float(np.median(rec["iter_ms"][len(rec["iter_ms"]) // 2:]))
                                             if rec["iter_ms"] else None),
                "resolved": resolved}
    print(json.dumps(out_line))
    return 0 if err is None else 1


def compare(fa, fb, tol):
    a, b = (json.loads(open(f).read().strip().splitlines()[-1]) for f in (fa, fb))
    n = min(len(a["loss"]), len(b["loss"]))
    worst = max(abs(x - y) / max(abs(y), 1e-6) for x, y in zip(a["loss"][:n], b["loss"][:n])) if n else None
    ng = max((abs(x - y) / max(y, 1) for x, y in zip(a["n_gauss"][:n], b["n_gauss"][:n])), default=None)
    res = {"iterations_compared": n, "max_rel_loss_diff": worst,
           "max_rel_gaussian_count_diff": ng, "gaussian_counts_last": [a["n_gauss"][n - 1], b["n_gauss"][n - 1]] if n else None,
           "errors": [a.get("error"), b.get("error")],
           "ms_per_iter": {a["stack"]: a["iter_ms_median_last_half"], b["stack"]: b["iter_ms_median_last_half"]}}
    res["ok"] = bool(n and worst is not None and worst < tol and ng is not None and ng < 0.02 and
                     not a.get("error") and not b.get("error"))
    print(json.dumps(res))
    return 0 if res["ok"] else 1


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--stack", choices=["ours", "reference"], default="ours")
    ap.add_argument("--iters", type=int, default=60)
    ap.add_argument("--size", type=int, default=200)
    ap.add_argument("--warm-up", dest="warm_up", type=int, default=10)
    ap.add_argument("--dpsr-iter", dest="dpsr_iter", type=int, default=1_000_000)
    ap.add_argument("--normal-warm-up", dest="normal_warm_up", type=int, default=10)
    ap.add_argument("--grid-res", dest="grid_res", type=int, default=64)
    ap.add_argument("--anchor-iter", dest="anchor_iter", type=int, default=1_000_000,
                    help="first iteration after which anchor_mesh runs (train.py:288-303); default: never")
    ap.add_argument("--anchor-every", dest="anchor_every", type=int, default=100)
    ap.add_argument("--densify-from", dest="densify_from", type=int, default=20)
    ap.add_argument("--densify-every", dest="densify_every", type=int, default=15)
    ap.add_argument("--work", default=None)
    ap.add_argument("--compare", nargs=2, default=None)
    ap.add_argument("--tol", type=float, default=0.05)
    a = ap.parse_args()
    sys.exit(compare(a.compare[0], a.compare[1], a.tol) if a.compare else run(a))
