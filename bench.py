#!/usr/bin/env python
"""bench.py -- the headline benchmark of BASELINE.json:
raster fwd+bwd frames/s @ 100k Gaussians, 800x800 (configs[1], SURVEY.md 8(d) C2), 1/2/4/8 H100.

  python bench.py --gpus N --steps K --warmup W            # this repo (CUDA path via the C-ABI)
  python bench.py --impl reference --gpus N --steps K ...  # stock diff_gaussian_rasterization (oracle/_ref)
  python bench.py ... --dump-outputs DIR                    # + the last timed step's outputs as DIR/<name>.npy

A "step" is one batch of 8 training frames of a DYNAMIC scene (8 cameras on a ring at times
t_k = k/8, SURVEY C4): every frame renders the canonical Gaussians deformed for its own time --
means3D + d_xyz_k, scales + d_scaling_k, rotations + d_rotation_k, exactly what
gaussian_renderer.render() hands the rasterizer (dgmesh/gaussian_renderer/__init__.py:60-86) -- so the
rasterizer sees per-frame [F,P,.] parameters; opacity and SH are shared.  At N GPUs each rank renders
8/N of the frames forward+backward and, when N > 1, the canonical-Gaussian gradients are combined with
ONE all-reduce over a flat fp32 buffer -- this library's NVSwitch kernel on >= 4 GPUs, NCCL on 2 -- ("scaling": "strong").
  value         frames/s over the whole job, inputs resident in HBM, through `BatchGaussianRasterizer`
                (per-frame-parameter frame batch: one call, binning chains overlapped with blend kernels)
  e2e           the same step fed from pinned HOST buffers every step (cameras + 8-bit ground-truth
                images up, a gradient checksum down), copies inside the timed region
  single_frame  the same 8 frames through the reference's own one-frame API (`GaussianRasterizer`,
                one call per frame), device-timed and e2e -- what an unmodified train.py sees
The reference arm (--impl reference) runs the same frames with the same per-frame parameters through
the stock extension's `GaussianRasterizer`.
"""
import argparse
import json
import math
import os
import subprocess
import sys
import threading
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
for _p in (ROOT, os.path.join(ROOT, "dg-mesh_b200"), os.path.join(ROOT, "tests")):
    if _p not in sys.path:
        sys.path.insert(0, _p)

import torch  # noqa: E402
import torch.distributed as dist  # noqa: E402

N_GAUSS, WIDTH, HEIGHT, FRAMES = 100_000, 800, 800, 8
FRAMES = int(os.environ.get("DGMESH_B200_BENCH_FRAMES", FRAMES))   # 8 is the contract; other values only exercise code paths
METRIC = "raster fwd+bwd frames/s @100k Gauss 800x800"


class ClockSampler:
    """nvidia-smi clocks / throttle reasons sampled DURING the timed region."""
    Q = ("index,clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.active,clocks_event_reasons.hw_slowdown,"
         "clocks_event_reasons.hw_thermal_slowdown,clocks_event_reasons.sw_thermal_slowdown,"
         "clocks_event_reasons.sw_power_cap")

    def __init__(self, gpu_index):
        self.gpu, self.rows, self.proc = gpu_index, [], None

    def start(self):
        try:
            self.proc = subprocess.Popen(["nvidia-smi", f"--id={self.gpu}", f"--query-gpu={self.Q}",
                                          "--format=csv,noheader,nounits", "-lms", "100"],
                                         stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True)
            self.th = threading.Thread(target=self._read, daemon=True)
            self.th.start()
        except Exception:
            self.proc = None

    def _read(self):
        for line in self.proc.stdout:
            self.rows.append([c.strip() for c in line.split(",")])

    def stop(self):
        if self.proc is None:
            return {"sm_mhz": None, "sm_max_mhz": None, "reasons": ["nvidia-smi unavailable"]}
        self.proc.terminate()
        try:
            self.proc.wait(timeout=2)
        except Exception:
            self.proc.kill()
        sm = sorted(float(r[1]) for r in self.rows if len(r) >= 9 and r[1].replace(".", "").isdigit())
        mx = [float(r[2]) for r in self.rows if len(r) >= 9 and r[2].replace(".", "").isdigit()]
        names = ["hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"]
        reasons = [n for i, n in enumerate(names) if any(len(r) >= 9 and r[5 + i].lower().startswith("active")
                                                         for r in self.rows)]
        return {"sm_mhz": sm[len(sm) // 2] if sm else None, "sm_max_mhz": max(mx) if mx else None,
                "reasons": reasons, "samples": len(sm)}


def make_inputs(device):
    import synth
    sc = synth.gaussian_scene(n=N_GAUSS, seed=0, device=device)
    cams = [synth.look_at_camera(azimuth_deg=45.0 * k, elevation_deg=20.0, radius=4.0, width=WIDTH, height=HEIGHT,
                                 fid=k / FRAMES, device=device) for k in range(FRAMES)]
    g = torch.Generator().manual_seed(1)
    dpix = [torch.randn(3, HEIGHT, WIDTH, generator=g) for _ in range(FRAMES)]
    return sc, cams, dpix


class Exchange:
    """The step's one collective over the flat gradient buffer: this library's NVSwitch all-reduce kernel
    (csrc/nvls.cu, buffer in symmetric memory) when the platform has multicast support, else ncclAllReduce."""

    def __init__(self, n, device, world):
        self.kind, self.handle, self.epoch = "nccl", None, 1
        n_pad = (n + 3) // 4 * 4
        self.buf = None
        # on 2 GPUs NCCL's direct peer copy moves less data than a multicast round trip; from 4 GPUs on the
        # multicast exchange sends and receives the buffer once per GPU
        default = "nvls" if world >= 4 else "nccl"
        if world > 1 and os.environ.get("DGMESH_B200_EXCHANGE", default) == "nvls":
            try:
                import torch.distributed._symmetric_memory as symm_mem
                buf = symm_mem.empty(n_pad, dtype=torch.float32, device=device)
                h = symm_mem.rendezvous(buf, dist.group.WORLD)
                if not h.multicast_ptr:
                    raise RuntimeError("no multicast support")
                buf.zero_()
                h.barrier()
                self.buf, self.handle, self.kind = buf, h, "nvls (own kernel, multimem.ld_reduce / multimem.st)"
                self.blocks = dp_blocks()
            except Exception as e:  # recorded in the JSON line
                self.kind = f"nccl (nvls unavailable: {type(e).__name__}: {e})"
        if world > 1:
            # every rank must take the same path: if the symmetric-memory set-up failed anywhere, nobody uses it
            agreed = torch.tensor([1.0 if self.handle is not None else 0.0], device=device)
            dist.all_reduce(agreed, op=dist.ReduceOp.MIN)
            if float(agreed) == 0.0 and self.handle is not None:
                self.handle, self.buf = None, None
                self.kind = "nccl (another rank could not set up symmetric memory)"
        if self.buf is None:
            self.buf = torch.zeros(n_pad, device=device)
        self.flat = self.buf[:n]

    def allreduce(self):
        if self.handle is None:
            dist.all_reduce(self.flat)
            return
        import _dgm_lib
        h = self.handle
        rc = _dgm_lib.lib().dgx_allreduce_nvls(int(h.multicast_ptr), self.buf.numel(), int(h.signal_pad_ptrs_dev),
                                               h.rank, h.world_size, self.epoch, 1.0, self.blocks,
                                               _dgm_lib.stream_ptr())
        _dgm_lib.check(rc, "dgx_allreduce_nvls")
        self.epoch += 2


def dp_blocks():
    import dp
    return dp.NvlsFlatGrad.BLOCKS


DUMP_COLOR_SAMPLES = 4_000_000   # rendered values kept by --dump-outputs (16 MB of the 61 MB batch)


def dump_outputs(out_dir, color, leaves):
    """What the timed path hands its caller after its last step: the rendered batch (the values at a fixed, seeded
    sample of flat positions) and the gradient of every Gaussian parameter, as float32 .npy files."""
    import numpy as np
    os.makedirs(out_dir, exist_ok=True)
    flat = color.detach().reshape(-1)
    g = torch.Generator().manual_seed(123)
    idx = torch.randperm(flat.numel(), generator=g)[:min(DUMP_COLOR_SAMPLES, flat.numel())].sort().values
    np.save(os.path.join(out_dir, "color_sample.npy"), flat[idx.to(flat.device)].float().cpu().numpy())
    for n, p in leaves.items():
        np.save(os.path.join(out_dir, f"grad_{n}.npy"), p.grad.detach().float().cpu().numpy())


def flat_params(sc, device, world=1):
    """Leaves as views of one flat buffer, with .grad views of one flat grad buffer, so the DP
    exchange is a single all-reduce (SURVEY 8(e))."""
    names = ["means3D", "opacities", "scales", "rotations", "shs"]
    sizes = [sc[n].numel() for n in names]
    flat = torch.empty(sum(sizes), device=device)
    ex = Exchange(sum(sizes), device, world)
    gflat = ex.flat
    leaves, off = {}, 0
    for n, s in zip(names, sizes):
        v = flat[off:off + s].view_as(sc[n])
        v.copy_(sc[n])
        p = v.detach().requires_grad_(True)
        p.grad = gflat[off:off + s].view_as(sc[n])
        leaves[n] = p
        off += s
    return leaves, gflat, ex


def make_deltas(sc, device):
    """Per-frame deformation of the canonical Gaussians (what the deformation MLP returns for time
    t_k = k/8): smooth in k, a few per cent of the scene / Gaussian size."""
    g = torch.Generator().manual_seed(11)
    P = sc["means3D"].shape[0]
    base = {"means3D": 0.03 * torch.randn(2, P, 3, generator=g), "scales": 0.001 * torch.randn(2, P, 3, generator=g),
            "rotations": 0.01 * torch.randn(2, P, 4, generator=g)}
    out = {}
    for n, b in base.items():
        ph = [2 * math.pi * k / FRAMES for k in range(FRAMES)]
        out[n] = torch.stack([math.cos(a) * b[0] + math.sin(a) * b[1] for a in ph]).to(device).contiguous()
    return out


def run_frames(dgr, synth, leaves, cams, dpix, bg, frame_ids, staged=None, deltas=None):
    """forward + backward of the given frames through the one-frame public API.  `staged` (e2e leg) maps a
    frame to (event, view, proj, campos, dpix) device tensors filled from pinned host memory by the
    copy stream; the compute stream waits on the frame's event before touching them."""
    last = None
    for k in frame_ids:
        cam = cams[k]
        if staged is not None:
            ev, view, proj, cpos, dp = staged[k]   # dp: callable(color) -> pixel gradient
            torch.cuda.current_stream().wait_event(ev)
        else:
            view, proj, cpos, dp = cam.world_view_transform, cam.full_proj_transform, cam.camera_center, dpix[k]
        rs = dgr.GaussianRasterizationSettings(
            image_height=HEIGHT, image_width=WIDTH, tanfovx=math.tan(cam.FoVx * 0.5), tanfovy=math.tan(cam.FoVy * 0.5),
            bg=bg, scale_modifier=1.0, viewmatrix=view, projmatrix=proj, sh_degree=3, campos=cpos, prefiltered=False,
            debug=False)
        m2d = torch.zeros_like(leaves["means3D"], requires_grad=True)
        if deltas is None:
            m3, sc_, ro = leaves["means3D"], leaves["scales"], leaves["rotations"]
        else:   # the frame's own deformed parameters (render(): means3D = xyz + d_xyz, ...)
            m3 = leaves["means3D"] + deltas["means3D"][k]
            sc_ = leaves["scales"] + deltas["scales"][k]
            ro = leaves["rotations"] + deltas["rotations"][k]
        color, radii = dgr.GaussianRasterizer(rs)(means3D=m3, means2D=m2d, opacities=leaves["opacities"],
                                                  shs=leaves["shs"], scales=sc_, rotations=ro)
        color.backward(dp(color) if callable(dp) else dp)
        last = color
    return last


class HostFeed:
    """e2e leg: every step the frames' cameras (35 floats each) and their ground-truth images (3xHxW
    uint8, as a dataset stores them) are copied from PINNED HOST memory on a side stream into one of TWO
    device staging slots (the prefetch of a training loop's data loader: step i+1's upload runs while step i
    renders; every copy is inside the timed region); the pixel gradient is the L2-loss gradient (render - gt)
    formed on the device; the step's result (a checksum of the accumulated parameter gradient) is copied back
    to the host every step and read one step later (the usual lagged loss read of a training loop), the last
    one after the final synchronise."""

    def __init__(self, cams, frames, dev):
        self.frames = frames
        F = len(frames)
        self.h_cam = torch.stack([torch.cat([cams[k].world_view_transform.cpu().reshape(-1),
                                             cams[k].full_proj_transform.cpu().reshape(-1),
                                             cams[k].camera_center.cpu().reshape(-1)]) for k in frames]).pin_memory()
        g = torch.Generator().manual_seed(7)
        self.h_gt = torch.randint(0, 256, (F, 3, HEIGHT, WIDTH), dtype=torch.uint8, generator=g).pin_memory()
        self.slots = []
        for _ in range(2):
            d_cam = torch.empty_like(self.h_cam, device=dev)
            sl = {"d_cam": d_cam, "d_gt": torch.empty_like(self.h_gt, device=dev),
                  "views": [d_cam[i, 0:16].view(4, 4) for i in range(F)],
                  "projs": [d_cam[i, 16:32].view(4, 4) for i in range(F)],
                  "campos": [d_cam[i, 32:35] for i in range(F)],
                  "ev_cam": torch.cuda.Event(), "ev_gt": torch.cuda.Event(), "consumed": torch.cuda.Event()}
            sl["consumed"].record()
            self.slots.append(sl)
        self.cur = self.slots[0]
        self.copy_stream = torch.cuda.Stream(device=dev)
        self.out_host = torch.zeros(2).pin_memory()
        self.out_ev = [None, None]
        self.n = 0
        self.results = []
        self.h2d_bytes = self.h_cam.numel() * 4 + self.h_gt.numel()

    def upload(self):
        """Start this step's copies into the slot the step before last used; returns the slot."""
        sl = self.cur = self.slots[self.n & 1]
        self.copy_stream.wait_event(sl["consumed"])  # step n-2 no longer reads this slot
        with torch.cuda.stream(self.copy_stream):
            sl["d_cam"].copy_(self.h_cam, non_blocking=True)
            sl["ev_cam"].record(self.copy_stream)
            sl["d_gt"].copy_(self.h_gt, non_blocking=True)
            sl["ev_gt"].record(self.copy_stream)
        return sl

    def pixel_grad(self, color, i=None):
        """d(L2 loss)/d(color) for the whole batch (i is None) or frame slot i."""
        sl = self.cur
        torch.cuda.current_stream().wait_event(sl["ev_gt"])
        gt = sl["d_gt"] if i is None else sl["d_gt"][i]
        return torch.add(color.detach(), gt, alpha=-1.0 / 255.0)   # one kernel: uint8 -> float, scale, subtract

    def finish(self, result):
        self.cur["consumed"].record()
        slot = self.n & 1
        if self.out_ev[slot] is not None:      # the result of step n-2 has long arrived: read it
            self.out_ev[slot].synchronize()
            self.results.append(float(self.out_host[slot]))
        self.out_host[slot:slot + 1].copy_(result.reshape(1), non_blocking=True)
        ev = torch.cuda.Event()
        ev.record()
        self.out_ev[slot] = ev
        self.n += 1

    def drain(self):
        torch.cuda.synchronize()
        for slot in ((self.n & 1), ((self.n + 1) & 1)):
            if self.out_ev[slot] is not None:
                self.results.append(float(self.out_host[slot]))
                self.out_ev[slot] = None
        return self.results


def batch_settings(dgr, cams, bg, frames, views=None, projs=None, campos=None):
    out = []
    for i, k in enumerate(frames):
        c = cams[k]
        out.append(dgr.GaussianRasterizationSettings(
            image_height=HEIGHT, image_width=WIDTH, tanfovx=math.tan(c.FoVx * 0.5), tanfovy=math.tan(c.FoVy * 0.5),
            bg=bg, scale_modifier=1.0, viewmatrix=views[i] if views else c.world_view_transform,
            projmatrix=projs[i] if projs else c.full_proj_transform, sh_degree=3,
            campos=campos[i] if campos else c.camera_center, prefiltered=False, debug=False))
    return out


def run_batch(dgr, leaves, settings, dpix_stacked, wait_fwd=None, deltas=None):
    """forward + backward of a frame batch through BatchGaussianRasterizer (this repo's batched API):
    per-frame deformed means / scales / rotations [F,P,.], shared opacity and SH."""
    if wait_fwd is not None:
        torch.cuda.current_stream().wait_event(wait_fwd)
    if deltas is None:
        m3, sc_, ro = leaves["means3D"], leaves["scales"], leaves["rotations"]
    else:
        m3 = leaves["means3D"][None] + deltas["means3D"]
        sc_ = leaves["scales"][None] + deltas["scales"]
        ro = leaves["rotations"][None] + deltas["rotations"]
    color, radii = dgr.BatchGaussianRasterizer(settings)(
        means3D=m3, means2D=None, opacities=leaves["opacities"], shs=leaves["shs"], scales=sc_, rotations=ro)
    color.backward(dpix_stacked(color) if callable(dpix_stacked) else dpix_stacked)
    return color


def timed(fn, steps, warmup, world):
    for _ in range(warmup):
        fn()
    if world > 1:
        dist.barrier()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    if world > 1:
        dist.barrier()
    ms = torch.tensor([e0.elapsed_time(e1)], device="cuda")
    if world > 1:
        dist.all_reduce(ms, op=dist.ReduceOp.MAX)
    return float(ms)


def cpu_baseline_port():
    """The CPU oracle (C restatement of the reference) timed on this box's host cores on ONE frame
    of the same workload (forward + backward), single thread."""
    import numpy as np
    import synth
    from oracle.oracle import RasterOracle
    os.environ["OMP_NUM_THREADS"] = "1"
    sc = synth.gaussian_scene(n=N_GAUSS, seed=0)
    cam = synth.look_at_camera(azimuth_deg=0.0, elevation_deg=20.0, width=WIDTH, height=HEIGHT)
    import util
    orc = RasterOracle(32)
    dp = np.random.default_rng(1).standard_normal((3, HEIGHT, WIDTH)).astype(np.float32)
    t0 = time.perf_counter()
    o = util.oracle_forward(orc, sc, cam, [1, 1, 1])
    orc.backward(o, dp)
    dt = time.perf_counter() - t0
    return {"value": 1.0 / dt, "unit": "frames/s", "cores": 1, "kind": "port",
            "sample": f"1 frame (fwd+bwd) of the same 100k/800x800 workload, C oracle, 1 thread of {os.cpu_count()}"}


def cpu_paths_baseline():
    """north_star: "its PyTorch-CPU deformation-MLP/KNN path timed on the box's own host cores in the
    same run (core count stated)".  C1 = DeformNetworkNormal(is_blender) fwd+bwd on 10k points with the
    reference's own module (oracle/_ref/refpy) on all host threads; KNN = the k-d-tree restatement of
    distCUDA2 on 100k points (1 thread).  Reported, not optimised."""
    import numpy as np
    import util
    from oracle.oracle import knn_mean_dist2
    out = {"cores": os.cpu_count()}
    ref = util.load_reference_pymodules()
    if ref is not None:
        # all 128 threads of the box make this small problem ~50x SLOWER (measured 9.9 s/step); 16 is what
        # a tuned CPU run would use
        torch.set_num_threads(max(1, min(16, os.cpu_count() or 1)))
        out["torch_threads"] = torch.get_num_threads()
        torch.manual_seed(0)
        net = ref.time_utils.DeformNetworkNormal(is_blender=True)
        g = torch.Generator().manual_seed(0)
        x = (torch.rand(10_000, 3, generator=g) * 2 - 1).requires_grad_(True)
        t = torch.full((10_000, 1), 0.37)

        def step():
            net.zero_grad(set_to_none=True)
            sum(o.sum() for o in net(x, t)).backward()
        step()
        t0 = time.perf_counter()
        for _ in range(3):
            step()
        out["mlp_c1_10k_fwd_bwd_ms"] = (time.perf_counter() - t0) / 3 * 1e3
    pts = np.random.default_rng(0).standard_normal((100_000, 3)) * 0.5
    t0 = time.perf_counter()
    knn_mean_dist2(pts)
    out["knn_100k_ms"] = (time.perf_counter() - t0) * 1e3
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--impl", default="ours", choices=["ours", "reference"])
    ap.add_argument("--no-cpu-baseline", action="store_true")
    ap.add_argument("--graph", choices=["on", "off"], default="off",
                    help="replay the single-GPU step as ONE CUDA graph (the library is capture-safe); "
                         "not used with NCCL: capturing the all-reduce hung in this round's test")
    ap.add_argument("--no-train-step", action="store_true",
                    help="skip the full-train-step leg (BASELINE.json's second metric, N=1 only)")
    ap.add_argument("--dump-outputs", metavar="DIR", default=None,
                    help="after the timed steps, write what the last one computed (rendered colours, sampled; "
                         "parameter gradients) as DIR/<name>.npy (rank 0)")
    a = ap.parse_args()
    a.warmup = max(a.warmup, 3)
    # exactly ONE line may reach stdout (the JSON): libraries that print there (NCCL's version banner)
    # are sent to stderr for the duration of the run
    sys.stdout.flush()
    real_stdout = os.dup(1)
    os.dup2(2, 1)

    rank, world = int(os.environ.get("RANK", 0)), int(os.environ.get("WORLD_SIZE", 1))
    local = int(os.environ.get("LOCAL_RANK", 0))
    if a.impl == "reference" and rank != 0:
        return 0  # the stock rasterizer is single-GPU: rank 0 alone measures it
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    if world > 1 and a.impl == "ours":
        os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
        dist.init_process_group("nccl", device_id=dev)
    else:
        world = 1

    import synth
    if a.impl == "reference":
        import util
        dgr = util.load_reference_rasterizer()
        if dgr is None:
            os.dup2(real_stdout, 1)
            print(json.dumps({"impl": "reference", "unavailable": "oracle/_ref not built in this snapshot"}), flush=True)
            return 0
    else:
        import diff_gaussian_rasterization as dgr
        import _dgm_lib
        _dgm_lib.lib()  # fail loudly when the CUDA library is missing -- there is no fallback

    sc, cams, dpix = make_inputs(dev)
    dpix = [d.to(dev) for d in dpix]
    deltas_all = make_deltas(sc, dev)
    leaves, gflat, exchange = flat_params(sc, dev, world if a.impl == "ours" else 1)
    bg = torch.ones(3, device=dev)
    my_frames = [k for k in range(FRAMES) if k % world == rank]

    ours = a.impl == "ours"
    my_deltas = {n: v[my_frames].contiguous() for n, v in deltas_all.items()}   # this rank's frames, [F_local,P,.]
    if ours:
        dev_settings = batch_settings(dgr, cams, bg, my_frames)
        dpix_stacked = torch.stack([dpix[k] for k in my_frames]).contiguous()

    # a rank that holds ONE frame of the step (8 GPUs) has nothing to batch: it goes through the one-frame API,
    # which is the shorter host path (measured at N = 8: 0.541 vs 0.577 ms per step)
    one = ours and len(my_frames) == 1

    last = {}   # the colour of the step's last render (a graph replay rewrites the captured tensor in place)

    def step():
        gflat.zero_()
        if one:
            last["color"] = run_frames(dgr, synth, leaves, cams, dpix, bg, my_frames, deltas=deltas_all)
        elif ours:
            last["color"] = run_batch(dgr, leaves, dev_settings, dpix_stacked, deltas=my_deltas)
        else:
            last["color"] = run_frames(dgr, synth, leaves, cams, dpix, bg, my_frames, deltas=deltas_all)
        if world > 1:
            exchange.allreduce()  # the one collective of the step (SURVEY 8(e))

    def step_render_only():
        gflat.zero_()
        if one:
            run_frames(dgr, synth, leaves, cams, dpix, bg, my_frames, deltas=deltas_all)
        else:
            run_batch(dgr, leaves, dev_settings, dpix_stacked, deltas=my_deltas)

    def step_single():      # the same frames, one GaussianRasterizer call each (reference-style loop)
        gflat.zero_()
        run_frames(dgr, synth, leaves, cams, dpix, bg, my_frames, deltas=deltas_all)
        if world > 1:
            exchange.allreduce()

    # Optional: capture the step once and replay it as a CUDA graph (parameters, cameras and pixel
    # gradients live at fixed addresses exactly as in a training loop with in-place optimiser updates;
    # the library does no host polling while capturing).  Single GPU only.
    use_graph = ours and a.graph == "on" and world == 1
    timed_step = step
    graph_note = None
    if use_graph:
        for _ in range(3):
            step()          # eager warm-up: sizes the instance workspaces, creates the internal streams
        torch.cuda.synchronize()
        if world > 1:
            dist.barrier()
        try:
            cap_stream = torch.cuda.Stream()
            cap_stream.wait_stream(torch.cuda.current_stream())
            graph = torch.cuda.CUDAGraph()
            with torch.cuda.stream(cap_stream):
                with torch.cuda.graph(graph, stream=cap_stream):
                    step()
            torch.cuda.current_stream().wait_stream(cap_stream)
            torch.cuda.synchronize()
            timed_step = graph.replay
        except Exception as e:  # keep the run alive: measure the eager step instead and say so
            graph_note = f"graph capture failed ({type(e).__name__}: {e}); eager step timed"
            use_graph = False
            torch.cuda.synchronize()

    sampler = ClockSampler(local)
    if rank == 0:
        sampler.start()
    ms = timed(timed_step, a.steps, a.warmup, world)
    clocks = sampler.stop() if rank == 0 else None
    if a.dump_outputs and rank == 0:
        dump_outputs(a.dump_outputs, last["color"], leaves)
    if use_graph:
        # graph replay cannot wait for the status words (no host interaction inside a graph): prove that no frame
        # overflowed its instance workspace by comparing the replayed gradient with an eager step's
        graph.replay()
        torch.cuda.synchronize()
        g_replay = gflat.clone()
        step()
        torch.cuda.synchronize()
        err = float((g_replay - gflat).abs().max() / (gflat.abs().max() + 1e-30))
        graph_note = f"replay vs eager gradient max-norm difference {err:.2e}"
        assert err < 1e-3, graph_note
    value = FRAMES * a.steps / (ms * 1e-3)
    breakdown = None
    if world > 1 and ours:
        nccl_probe = torch.zeros_like(gflat)
        breakdown = {"render_only_ms": timed(step_render_only, a.steps, 2, world) / a.steps,
                     "allreduce_only_ms": timed(exchange.allreduce, a.steps, 2, world) / a.steps,
                     "nccl_allreduce_only_ms": timed(lambda: dist.all_reduce(nccl_probe), a.steps, 2, world) / a.steps,
                     "allreduce_bytes": gflat.numel() * 4, "exchange": exchange.kind}

    # ---- e2e leg: host buffers, copies inside the timed region
    feed = HostFeed(cams, my_frames, dev)
    if ours:
        for sl in feed.slots:
            sl["settings"] = batch_settings(dgr, cams, bg, my_frames, sl["views"], sl["projs"], sl["campos"])

    def step_e2e():
        sl = feed.upload()
        gflat.zero_()
        if ours and not one:
            run_batch(dgr, leaves, sl["settings"], feed.pixel_grad, wait_fwd=sl["ev_cam"], deltas=my_deltas)
        else:
            staged = {k: (sl["ev_cam"], sl["views"][i], sl["projs"][i], sl["campos"][i],
                          (lambda c, i=i: feed.pixel_grad(c, i))) for i, k in enumerate(my_frames)}
            run_frames(dgr, synth, leaves, cams, dpix, bg, my_frames, staged=staged, deltas=deltas_all)
        if world > 1:
            exchange.allreduce()
        feed.finish(gflat.sum())

    e2e_steps = a.steps
    ms_e2e = timed(step_e2e, e2e_steps, 3, world)
    host_results = feed.drain()
    assert len(host_results) == e2e_steps + 3 and all(math.isfinite(v) for v in host_results), host_results
    e2e_value = FRAMES * e2e_steps / (ms_e2e * 1e-3)

    single = None
    if ours:
        # ---- the reference's own one-frame API: device-timed, then fed from the host like e2e
        ms_single = timed(step_single, a.steps, 3, world)
        feed1 = HostFeed(cams, my_frames, dev)

        def step_single_e2e():
            sl = feed1.upload()
            gflat.zero_()
            staged = {k: (sl["ev_cam"], sl["views"][i], sl["projs"][i], sl["campos"][i],
                          (lambda c, i=i: feed1.pixel_grad(c, i))) for i, k in enumerate(my_frames)}
            run_frames(dgr, synth, leaves, cams, dpix, bg, my_frames, staged=staged, deltas=deltas_all)
            if world > 1:
                exchange.allreduce()
            feed1.finish(gflat.sum())

        ms_single_e2e = timed(step_single_e2e, a.steps, 3, world)
        feed1.drain()
        single = {"api": "GaussianRasterizer, one call per frame (reference API)",
                  "value": FRAMES * a.steps / (ms_single * 1e-3), "unit": "frames/s",
                  "ms_per_frame": ms_single / a.steps / len(my_frames),
                  "e2e": {"value": FRAMES * a.steps / (ms_single_e2e * 1e-3), "unit": "frames/s"}}
    h2d = feed.h2d_bytes * world
    d2h = 4 * world

    out = {
        "metric": METRIC, "value": value, "unit": "frames/s", "n_gpus": a.gpus, "steps": a.steps, "warmup": a.warmup,
        "ms_per_step": ms / a.steps, "higher_is_better": True, "scaling": "strong", "vs_baseline": None,
        "dtype": "f32", "data": "synthetic",
        "config": {"workload": "BASELINE.json configs[1]: 100k Gaussians, 800x800, SH degree 3, raster fwd+bwd; "
                               "step = 8-frame batch (8 ring cameras), frames sharded over ranks",
                   "gaussians": N_GAUSS, "width": WIDTH, "height": HEIGHT, "frames_per_step": FRAMES,
                   "parallelism": f"dp{world} over frames" + (
                       (", 1 all-reduce of grads (" + ("own NVSwitch kernel" if exchange.handle is not None else "NCCL") + ")")
                       if world > 1 else ""),
                   "scene": "dynamic: frame k renders xyz + d_xyz_k, scales + d_scaling_k, rotations + d_rotation_k",
                   "api": (("GaussianRasterizer (one frame per rank: nothing to batch)" if one else
                            "BatchGaussianRasterizer (frame batch, per-frame deformed means/scales/rotations)")
                           + (", step replayed as one CUDA graph" if (ours and use_graph) else "")) if ours
                          else "GaussianRasterizer per frame (reference API)",
                   "l2_policy": "inputs larger than L2: per step 8 frames x (~42 MB instance records + 12 MB "
                                "per-Gaussian state + 13 MB pixel state) + 24 MB parameters + 61 MB pixel "
                                "gradients = ~620 MB streamed through the 50 MB L2"},
        "e2e": {"value": e2e_value, "unit": "frames/s", "h2d_bytes_per_step": h2d, "d2h_bytes_per_step": d2h},
        "clocks": clocks,
    }
    if single:
        out["single_frame"] = single
    if breakdown:
        out["breakdown"] = breakdown
    if graph_note:
        out["graph_note"] = graph_note
    if a.impl == "reference":
        out["impl"] = "reference"
        out["n_gpus"] = a.gpus
        out["gpu_launches"] = 0
        out["cpu_baseline"] = {"value": value, "unit": "frames/s", "cores": os.cpu_count(), "kind": "reference",
                               "sample": "stock diff_gaussian_rasterization (unmodified reference sources built for "
                                         "sm_90a) on ONE H100, same 8-frame batch; host threads only launch kernels"}
        out["e2e"] = {"value": value, "unit": "frames/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}
        out["e2e_host_buffers"] = {"value": e2e_value, "unit": "frames/s"}
    else:
        # ---- roofline leg: per-kernel CUDA-event durations on the launching stream
        import _dgm_lib
        _dgm_lib.lib().dgm_profile_enable(1)
        acc, R_sum = {}, 0
        nprof = 3
        for _ in range(nprof):
            for k in my_frames:
                run_frames(dgr, synth, leaves, cams, dpix, bg, [k], deltas=deltas_all)
                for n, v in _dgm_lib.profile_read().items():
                    acc[n] = acc.get(n, 0.0) + v
        _dgm_lib.lib().dgm_profile_enable(0)
        cnt = nprof * len(my_frames)
        kern_ms = {n: v / cnt for n, v in acc.items()}
        # R (tile instances) of each frame defines the algorithmic bytes
        Rs = []
        for k in my_frames:
            c = cams[k]
            rs = synth.raster_settings_for(c, bg, settings_cls=dgr.GaussianRasterizationSettings)
            R, *_ = dgr._C.rasterize_gaussians(bg, sc["means3D"] + deltas_all["means3D"][k], torch.Tensor([]),
                                               sc["opacities"], sc["scales"] + deltas_all["scales"][k],
                                               sc["rotations"] + deltas_all["rotations"][k], 1.0, torch.Tensor([]),
                                               rs.viewmatrix, rs.projmatrix,
                                               rs.tanfovx, rs.tanfovy, HEIGHT, WIDTH, sc["shs"], 3, rs.campos, False,
                                               False)
            Rs.append(R)
        R_mean = sum(Rs) / len(Rs)
        T = ((WIDTH + 15) // 16) * ((HEIGHT + 15) // 16)
        npix = WIDTH * HEIGHT
        alg = {"render_fwd": 40 * R_mean + 20 * npix + 8 * T,
               "render_bwd": 40 * R_mean + 20 * npix + 8 * T + 44 * N_GAUSS}
        dom = max(("render_fwd", "render_bwd"), key=lambda n: kern_ms.get(n, 0.0))
        peaks_path = os.path.join(ROOT, "MEASURED_PEAKS.json")
        if os.path.exists(peaks_path):
            peak, peak_src = float(json.load(open(peaks_path))["hbm_gbs"]), "measured (MEASURED_PEAKS.json hbm_gbs)"
        else:
            peak, peak_src = 3350.0, "H100 SXM data sheet (HBM3, 700 W card)"
        achieved = alg[dom] / (kern_ms[dom] * 1e-3) / 1e9
        traffic = None
        tp = os.path.join(ROOT, "profiles", "traffic.json")
        if os.path.exists(tp):
            traffic = json.load(open(tp)).get(dom)
        out["roofline"] = {"bound": "hbm", "kernel": dom, "achieved": achieved, "peak": peak, "unit": "GB/s",
                           "frac": achieved / peak, "traffic": traffic, "peak_source": peak_src,
                           "algorithmic_bytes_per_launch": alg[dom], "launch_ms": kern_ms[dom],
                           "note": "the blend kernels are ALU/MUFU-bound (256 pixel x Gaussian evaluations per "
                                   "40 B instance record), not HBM-bound: see DESIGN.md 'roofline'"}
        out["kernel_ms"] = kern_ms
        out["num_rendered_mean"] = R_mean
        # this library's kernels per frame: preprocess(+count), tile_scan, scatter, sort_pack, render_fwd,
        # render_bwd, preprocess_bwd (torch's own elementwise kernels around them are not counted)
        out["gpu_launches"] = 7 * len(my_frames) * a.steps * world
        if rank == 0 and not a.no_cpu_baseline:
            out["cpu_baseline"] = cpu_baseline_port()
            try:
                out["cpu_baseline"]["other_paths"] = cpu_paths_baseline()
            except Exception as e:
                out["cpu_baseline"]["other_paths"] = {"error": f"{type(e).__name__}: {e}"}
        if rank == 0 and world == 1 and not a.no_train_step:
            # BASELINE.json's other metric: full train-step ms (config C3, 200k Gaussians), ours and the
            # reference's own modules side by side on this GPU (tools/train_step.py)
            try:
                sys.path.insert(0, os.path.join(ROOT, "tools"))
                import train_step
                out["train_step"] = train_step.measure(steps=5)
            except Exception as e:  # never lose the headline line over the extra leg
                out["train_step"] = {"error": f"{type(e).__name__}: {e}"}
    if world > 1 and ours and not a.no_train_step:
        # ---- BASELINE configs[3] (SURVEY C4): the FULL train step, one frame per rank (camera k on the ring,
        # t_k = k / world), ONE all-reduce of [canonical-Gaussian grads || the five MLPs' grads] through dp.FlatGrad
        try:
            sys.path.insert(0, os.path.join(ROOT, "tools"))
            import dp
            import train_step as ts
            torch.cuda.empty_cache()
            S = ts.build("ours", 200_000, 288, dev, azimuth_deg=360.0 * rank / world)   # same seed: replicated parameters
            try:
                fg = dp.NvlsFlatGrad(S.params)       # this library's NVSwitch all-reduce
                fg_kind = "nvls (own kernel)"
            except Exception as e:
                fg = dp.FlatGrad(S.params)
                fg_kind = f"nccl ({type(e).__name__}: {e})"
            agreed = torch.tensor([1.0 if isinstance(fg, dp.NvlsFlatGrad) else 0.0], device=dev)
            dist.all_reduce(agreed, op=dist.ReduceOp.MIN)          # same path on every rank
            if float(agreed) == 0.0 and isinstance(fg, dp.NvlsFlatGrad):
                fg = dp.FlatGrad(S.params)
                fg_kind = "nccl (another rank could not set up symmetric memory)"

            def dp_step():
                fg.zero()
                ts.full_step(S, t_value=rank / world, clear_grads=False)
                fg.allreduce(average=True)

            def dp_step_local():
                fg.zero()
                ts.full_step(S, t_value=rank / world, clear_grads=False)

            ms_dp = timed(dp_step, 5, 3, world) / 5
            ms_local = timed(dp_step_local, 5, 2, world) / 5
            out["train_step_dp"] = {"config": "C4: full train step (200k Gaussians, grid 288), 1 frame per rank, t_k = k/N",
                                    "ms_per_step": ms_dp, "ms_without_allreduce": ms_local,
                                    "frames_per_s": world / (ms_dp * 1e-3), "allreduce_bytes": fg.flat.numel() * 4,
                                    "exchange": fg_kind,
                                    "scaling": "weak"}
            del S, fg
        except Exception as e:
            out["train_step_dp"] = {"error": f"{type(e).__name__}: {e}"}
    if world > 1:
        dist.destroy_process_group()
    sys.stdout.flush()
    os.dup2(real_stdout, 1)
    if rank == 0:
        print(json.dumps(out), flush=True)
    return 0


if __name__ == "__main__":
    sys.exit(main())
