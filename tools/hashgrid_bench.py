"""Cost of the hash-grid field at N = 10^5 for one frame and a batch of 8, forward + backward per call:

  * HashGridField at its defaults (four grids, L = 16, Fe = 2, T = 2^19) and with grids=("xyz",);
  * the same default encoding written in torch float32 on the GPU (gather of the 8 corner rows per level and grid,
    index_add_ in the backward through autograd's indexing);
  * HexPlaneField at its defaults and the existing DeformNetwork (wgmma), on the same x and t (the batch as one F N
    call);
  * each hash-grid kernel's time from torch.profiler (a run of its own) against the byte model `bytes_model` below.

    python tools/hashgrid_bench.py [--reps 30] [--out FILE]

Byte model: a corner row is Fe floats and x-neighbours (the first axis, prime 1 when hashed) sit in adjacent slots
(dense: always; hashed: the two slots differ only in the low bits, unless the carry of i_a + 1 runs past them).  A
32-byte sector holds 32 / (4 Fe) rows, so each of a cell's 4 x-pairs touches 1 + 4 Fe / 32 sectors on average:
5 sectors per (point-frame, grid, level) at Fe = 2, 6 at Fe = 4, dense and hashed levels alike.  The backward's
fixed-point adds are counted as 8 bytes per (corner, feature) red.add.u64.

Device events around `reps` calls after warm-up; the card's name and power limit are read in the same run."""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (os.path.join(ROOT, "dg-mesh_b200"), os.path.join(ROOT, "tests")):
    sys.path.insert(0, p)

import hashgrid_oracle as ho  # noqa: E402
from hashgrid import HashGridField  # noqa: E402
from hexplane import HexPlaneField  # noqa: E402

N = 100_000
KERNELS = ("hg_fwd_kernel", "hg_max_kernel", "hg_bwd_kernel", "hg_finish_kernel")


def timed(fn, reps, warmup=3):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps


def bytes_model(f, F):
    """Bytes each kernel moves, by the model in the module docstring."""
    G, L, Fe, T = len(f.grids), f.levels, f.features, 2 ** f.log2_table
    spatial = "xyz" in f.grids
    samples = L * N * ((1 if spatial else 0) + F * (G - spatial))     # (point-frame, grid, level) samples
    sector_bytes = 32 * 4 * (1 + 4 * Fe / 32)
    out = F * N * G * L * Fe * 4
    return {
        "hg_fwd_kernel": 12 * N + 4 * F * N + samples * sector_bytes + out,
        "hg_max_kernel": out,
        "hg_bwd_kernel": 12 * N + 4 * F * N + out + samples * (sector_bytes + 8 * Fe * 8) + 12 * N,
        "hg_finish_kernel": G * L * T * Fe * (8 + 4),
    }


def torch_encoding(f):
    """The same encoding in torch float32 on the device (differentiable in the tables and x)."""
    T = 2 ** f.log2_table
    corners = torch.tensor([[(k >> j) & 1 for j in range(3)] for k in range(8)], device="cuda")

    def enc(x, t):
        F = t.shape[0]
        lo, hi = f.box[0], f.box[1]
        u3 = ((x - lo) / (hi - lo)).clamp(0, 1)
        u = torch.cat([u3[None].expand(F, -1, 3), t.clamp(0, 1)], -1)
        outs = []
        for g, grid in enumerate(f.grids):
            for l, R in enumerate(f.resolutions):
                R3 = [min(R, f.time_resolution) if a == 3 else R for a in ho.AXES[grid]]
                p = torch.stack([u[..., a] * r for a, r in zip(ho.AXES[grid], R3)], -1)
                c = torch.minimum(torch.floor(p.detach()), torch.tensor(R3, device="cuda") - 1)
                w = p - c
                idx = c.long()[..., None, :] + corners
                s = ho.slots(idx, R3, T)
                fac = torch.where(corners.bool(), w[..., None, :], 1 - w[..., None, :])
                wt = fac[..., 0] * fac[..., 1] * fac[..., 2]
                outs.append((wt[..., None] * f.tables[g][l][s]).sum(-2))
        return torch.cat(outs, -1)
    return enc


def kernel_ms(fn, reps=10):
    from torch.profiler import ProfilerActivity, profile
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            fn()
        torch.cuda.synchronize()
    out = {}
    for ev in prof.key_averages():
        key = next((k for k in KERNELS if k in ev.key), "memset" if "emset" in ev.key else None)
        if key is None:
            continue
        t = getattr(ev, "device_time_total", None)
        if t is None:
            t = ev.cuda_time_total
        out[key] = out.get(key, 0.0) + t / 1000.0 / reps
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=30)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a CUDA device"
    dev = torch.device("cuda")
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    res = {"card": card or torch.cuda.get_device_name(), "N": N}
    box = [[-1.0] * 3, [1.0] * 3]
    g = torch.Generator().manual_seed(0)
    torch.manual_seed(0)
    fields = {"hashgrid_default": HashGridField(box).to(dev),
              "hashgrid_xyz": HashGridField(box, grids=("xyz",)).to(dev)}
    hexp = HexPlaneField(box).to(dev)
    from utils.time_utils import DeformNetwork
    mlp = DeformNetwork(is_blender=True).to(dev)
    x = (torch.rand(N, 3, generator=g) * 2 - 1).to(dev).requires_grad_(True)
    for F in (1, 8):
        t = torch.rand(F, N, 1, generator=g).to(dev)
        row = {}
        for name, f in fields.items():
            gout = torch.randn(F, N, f.out_dim, generator=g).to(dev)
            row[f"{name}_fwd_bwd_ms"] = timed(lambda: f(x, t).backward(gout), args.reps)
        fd = fields["hashgrid_default"]
        enc = torch_encoding(fd)
        gout = torch.randn(F, N, fd.out_dim, generator=g).to(dev)
        row["torch_float32_encoding_fwd_bwd_ms"] = timed(lambda: enc(x, t).backward(gout), max(3, args.reps // 10))
        gh = torch.randn(F, N, hexp.out_dim, generator=g).to(dev)
        row["hexplane_fwd_bwd_ms"] = timed(lambda: hexp(x, t).backward(gh), args.reps)
        xf = x.detach()[None].expand(F, N, 3).reshape(-1, 3).contiguous().requires_grad_(True)
        tf = t.reshape(-1, 1)
        row["deform_network_wgmma_fwd_bwd_ms"] = timed(lambda: sum(o.square().sum() for o in mlp(xf, tf)).backward(),
                                                       max(5, args.reps // 5))
        res[f"F{F}"] = row
    # kernel breakdown, a profiled run of its own
    for F in (1, 8):
        t = torch.rand(F, N, 1, generator=g).to(dev)
        for name, f in fields.items():
            gout = torch.randn(F, N, f.out_dim, generator=g).to(dev)
            ms = kernel_ms(lambda: f(x, t).backward(gout))
            by = bytes_model(f, F)
            res[f"F{F}"][f"{name}_kernels"] = {
                k: {"ms": round(v, 4), "bytes": by.get(k), "GB_per_s": round(by[k] / v / 1e6, 1) if k in by else None}
                for k, v in ms.items()}
    line = json.dumps(res, default=lambda v: round(v, 4))
    print(line)
    if args.out:
        with open(args.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
