"""FlexiCubes (flexicubes.FlexiCubes) against dual marching cubes (diso.DiffDMC) at G = 288, alternating in one run.

Fields: the DPSR field of a synth.py Gaussian scene (P = 100k) and the signed distance of a sphere joined with a
tilted torus (tools/dmc_bench.py's two fields).  Arms per field:
  - dmc: DiffDMC;
  - fc_neutral: FlexiCubes with no weights and no offsets;
  - fc_infer / fc_train: FlexiCubes with random raw weights and offsets (deform = 0.3 tanh(randn)), inference mode,
    and training mode with L_dev in the loss;
  - torch_fp32: tests/flexicubes_oracle.py's code run in float32 on the GPU (roughly what a pure-torch FlexiCubes
    costs; its topology comes from dmc_reference on the CPU, which is not timed).
Each arm: forward (including its host waits) + backward of L = sum(verts^2) (+ sum(L_dev) in training mode),
device-synchronised wall time, median and range over --rounds rounds of --steps steps; V, F and the peak memory
of one call.  --profile runs torch.profiler over a few calls of the FlexiCubes arms and prints the kernel split.
The card's name and power limit are read in the same run.

    python tools/flexicubes_bench.py [--rounds 5] [--steps 5] [--profile] [--out FILE]"""
import argparse
import json
import math
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [os.path.join(ROOT, "dg-mesh_b200"), os.path.join(ROOT, "tests")]
ap = argparse.ArgumentParser()
ap.add_argument("--rounds", type=int, default=5)
ap.add_argument("--steps", type=int, default=5)
ap.add_argument("--profile", action="store_true")
ap.add_argument("--out", default=None)
args = ap.parse_args()

import torch  # noqa: E402

from diso import DiffDMC  # noqa: E402
from dmc_reference import dmc_reference  # noqa: E402
from flexicubes import FlexiCubes  # noqa: E402
import flexicubes_oracle  # noqa: E402
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
    return {"dpsr": dpsr.contiguous(), "sphere_torus": torch.minimum(torch.sqrt(sph) - 0.4, tor).contiguous()}


def weights(dev):
    g = torch.Generator().manual_seed(0)
    c = (G - 1,) * 3
    return {"deform": 0.3 * torch.tanh(torch.randn(G, G, G, 3, generator=g)).to(dev),
            "beta": torch.randn(*c, 12, generator=g).to(dev), "alpha": torch.randn(*c, 8, generator=g).to(dev),
            "gamma_f": torch.randn(*c, generator=g).to(dev)}


def arms(phi):
    w = {n: t.requires_grad_(True) for n, t in weights(phi.device).items()}
    p = phi.clone().requires_grad_(True)
    fc, dmc = FlexiCubes(), DiffDMC()
    ref = dmc_reference(phi.cpu().numpy())

    def run_dmc():
        v, f = dmc(p)
        v.square().sum().backward()
        return v, f

    def run_fc(weighted, training):
        def go():
            kw = dict(w) if weighted else {}
            v, f, L = fc(p, **kw, training=training)
            (v.square().sum() + (L.sum() if training else 0.0)).backward()
            return v, f
        return go

    def run_torch_gpu():
        # the oracle's float64 statements in float32 on the GPU: index tensors built once, outside the timing
        v, L = torch_fc(p, w["deform"], w["beta"], w["alpha"])
        (v.square().sum() + L.sum()).backward()
        return v, torch.empty(2 * len(ref.quads), 3)

    torch_fc = _torch_fp32(ref)
    return {"dmc": run_dmc, "fc_neutral": run_fc(False, False), "fc_infer": run_fc(True, False),
            "fc_train": run_fc(True, True), "torch_fp32": run_torch_gpu}


def _torch_fp32(ref):
    """tests/flexicubes_oracle.py's vertex and L_dev statements in float32 on the GPU, for a fixed topology."""
    import numpy as np
    _, pof, edge_lo, _ = flexicubes_oracle.tables()
    cells = np.stack(np.unravel_index(ref.cell, (G, G, G)), 1)
    cs = flexicubes_oracle.cell_cases(ref_phi_inside[0])[tuple(cells.T)]
    member = torch.from_numpy(pof[cs] == ref.patch[:, None]).cuda()
    wc = torch.from_numpy(np.ravel_multi_index(cells.T, (G - 1,) * 3)).cuda()
    ct = torch.from_numpy(cells).cuda()
    ends = []
    for e in range(12):
        a, lo = e >> 2, int(edge_lo[e])
        n0 = ct + torch.tensor([lo & 1, (lo >> 1) & 1, lo >> 2], device="cuda")
        n1 = n0.clone()
        n1[:, a] += 1
        ends.append(((n0[:, 0] * G + n0[:, 1]) * G + n0[:, 2], (n1[:, 0] * G + n1[:, 1]) * G + n1[:, 2], lo,
                     lo + (1 << a)))
    grid = torch.stack(torch.meshgrid(*(torch.arange(G, dtype=torch.float32, device="cuda"),) * 3, indexing="ij"),
                       -1).reshape(-1, 3)
    k = member.sum(1)

    def f(phi, deform, beta, alpha):
        s = phi.reshape(-1)
        x = grid + deform.reshape(-1, 3)
        al = 1 + 0.99 * torch.tanh(alpha.reshape(-1, 8)[wc])
        be = 1 + 0.99 * torch.tanh(beta.reshape(-1, 12)[wc])
        u = []
        for e, (i0, i1, lo, hi) in enumerate(ends):
            w0, w1 = al[:, lo] * s[i0], al[:, hi] * s[i1]
            t = torch.where(member[:, e], w0 / torch.where(member[:, e], w0 - w1, 1.0), 0.0)
            u.append(x[i0] + t[:, None] * (x[i1] - x[i0]))
        u = torch.stack(u, 1)
        bm = torch.where(member, be, 0.0)
        v = (bm[:, :, None] * u).sum(1) / bm.sum(1, keepdim=True)
        d = flexicubes_oracle._safe_norm(u - v[:, None]) / (G - 1)
        mean = torch.where(member, d, 0.0).sum(1) / k
        return v / (G - 1), (d - mean[:, None]).abs()[member]
    return f


ref_phi_inside = [None]


def timed(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(args.steps):
        fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) / args.steps * 1e3


def main():
    out = {"card": card(), "G": G, "fields": {}}
    print(out["card"])
    for name, phi in fields().items():
        ref_phi_inside[0] = (phi < 0).cpu().numpy()
        a = arms(phi)
        res = {}
        for n, fn in a.items():      # warm-up, sizes and peak memory
            torch.cuda.synchronize()
            torch.cuda.reset_peak_memory_stats()
            base = torch.cuda.memory_allocated()
            v, f = fn()
            torch.cuda.synchronize()
            res[n] = {"V": int(v.shape[0]), "F": int(f.shape[0]),
                      "peak_MB": (torch.cuda.max_memory_allocated() - base) / 2 ** 20, "ms": []}
        if args.profile:
            from torch.profiler import ProfilerActivity, profile
            for n in ("fc_neutral", "fc_infer", "fc_train"):
                with profile(activities=[ProfilerActivity.CUDA]) as prof:
                    for _ in range(3):
                        a[n]()
                    torch.cuda.synchronize()
                print(f"--- {name} {n}")
                print(prof.key_averages().table(sort_by="cuda_time_total", row_limit=14))
            continue
        for _ in range(args.rounds):    # alternate the arms round by round
            for n, fn in a.items():
                res[n]["ms"].append(timed(fn))
        for n, r in res.items():
            ms = sorted(r.pop("ms"))
            r.update(median_ms=ms[len(ms) // 2], min_ms=ms[0], max_ms=ms[-1])
            print(f"{name:13s} {n:11s} V={r['V']:8d} F={r['F']:8d} fwd+bwd {r['median_ms']:8.2f} ms "
                  f"[{r['min_ms']:.2f}, {r['max_ms']:.2f}]  peak {r['peak_MB']:8.1f} MB")
        out["fields"][name] = res
    if args.out:
        with open(args.out, "w") as fh:
            json.dump(out, fh, indent=1)


if __name__ == "__main__":
    main()
