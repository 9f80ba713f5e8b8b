"""Cost of the HexPlane field at N = 10^5 (C = 32, R = 64 / 128, R_t = 25, the field's defaults), for one frame and
a batch of 8:

  * the encoding forward + backward (csrc/hexplane.cu) and, for comparison, the same encoding written with torch
    F.grid_sample in float32 (tests/hexplane_oracle.py run in float32);
  * the regularisers forward + backward;
  * HexPlaneDeformNetwork forward + backward, with the nn.Linear heads' share measured alone on the same features;
  * the existing DeformNetwork (wgmma) forward + backward on the same x and t (the batch as one F N call);
  * each kernel's time from torch.profiler (a run of its own) and its L2-side bytes from the formulas in
    `l2_bytes` below, so the backward's sort can be set against the rest of it.

    python tools/hexplane_bench.py [--reps 50] [--out FILE]

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

import hexplane_oracle as ho  # noqa: E402
from hexplane import HexPlaneDeformNetwork, HexPlaneField  # noqa: E402

N, C, RES, RT = 100_000, 32, (64, 128), 25


def timed(fn, reps, warmup=5):
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


def l2_bytes(F):
    """Bytes each kernel moves between the SMs and L2 (float32, C channels, S scales; corner reads counted per
    sample, as every sample is a separate line)."""
    S = len(RES)
    E = 3 * S * N * (1 + F)                                  # backward entries: 3 S N spatial + 3 S F N time
    cells = sum(3 * (R - 1) ** 2 + 3 * (R - 1) * (RT - 1) for R in RES)
    texels = sum(3 * R * R + 3 * RT * R for R in RES)
    samples = 3 * S * N + 3 * S * F * N
    fwd = 12 * N + 4 * F * N + samples * 4 * C * 4 + F * N * S * C * 4
    return {
        "hp_fwd_kernel": fwd,
        "hp_bwd_kernel": fwd + 12 * N + E * (4 * C + 8 + 8),   # + dL/dx, staging (dL/dsample, fractions, key, id)
        "DeviceRadixSort": 2 * 2 * E * 8,                       # two passes of keys + ids, read and written
        "hp_cell_kernel": E * (4 + 8 + 4 * C) + cells * 16 * C,
        "hp_texel_kernel": texels * (4 * 4 * C + 4 * C),
        "hp_reg_fwd_kernel": texels * 4 * C,
        "hp_reg_bwd_kernel": texels * 2 * 4 * C,
    }


def kernel_ms(fn, reps=20):
    """{kernel group: ms per call} from torch.profiler."""
    from torch.profiler import ProfilerActivity, profile
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            fn()
        torch.cuda.synchronize()
    out = {}
    for ev in prof.key_averages():
        name = ev.key
        key = next((k for k in l2_bytes(1) if k in name), None)
        if key is None:
            continue
        t = getattr(ev, "device_time_total", None)
        if t is None:
            t = ev.cuda_time_total
        out[key] = out.get(key, 0.0) + t / 1000.0 / reps
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a CUDA device"
    dev = torch.device("cuda")
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    res = {"card": card or torch.cuda.get_device_name(), "N": N, "C": C, "resolutions": RES, "R_t": RT}
    box = [[-1.0] * 3, [1.0] * 3]
    g = torch.Generator().manual_seed(0)
    torch.manual_seed(0)
    net = HexPlaneDeformNetwork(box, channels=C).to(dev)
    field = net.field
    with torch.no_grad():
        for p in field.planes:
            p.add_(0.05 * torch.randn(p.shape, generator=g).to(dev))
    x = (torch.rand(N, 3, generator=g) * 2 - 1).to(dev).requires_grad_(True)
    from utils.time_utils import DeformNetwork
    mlp = DeformNetwork(is_blender=True).to(dev)
    for F in (1, 8):
        t = torch.rand(F, N, 1, generator=g).to(dev)
        gout = torch.randn(F, N, field.out_dim, generator=g).to(dev)

        def enc():
            field(x, t).backward(gout)

        planes32 = list(field.planes)

        def enc_torch():
            ho.field(x, t, field.box, planes32, field.S).backward(gout)

        def network():
            sum(o.square().sum() for o in net(x, t)).backward()

        feats = field(x, t).detach().requires_grad_(True)

        def heads():
            h = net.feature_out(feats)
            sum(getattr(net, n)(h).square().sum() for n, _ in net.heads).backward()

        xf = x.detach()[None].expand(F, N, 3).reshape(-1, 3).contiguous().requires_grad_(True)
        tf = t.reshape(-1, 1)

        def deform_mlp():
            sum(o.square().sum() for o in mlp(xf, tf)).backward()

        res[f"F{F}"] = {
            "encoding_fwd_bwd_ms": timed(enc, args.reps),
            "torch_grid_sample_encoding_fwd_bwd_ms": timed(enc_torch, max(5, args.reps // 5)),
            "network_fwd_bwd_ms": timed(network, args.reps),
            "heads_fwd_bwd_ms": timed(heads, args.reps),
            "deform_network_wgmma_fwd_bwd_ms": timed(deform_mlp, max(5, args.reps // 5)),
        }
    res["regularisers_fwd_bwd_ms"] = timed(lambda: sum(field.regularisers()).backward(), args.reps)
    # kernel breakdown, a profiled run of its own
    for F in (1, 8):
        t = torch.rand(F, N, 1, generator=g).to(dev)
        gout = torch.randn(F, N, field.out_dim, generator=g).to(dev)
        ms = kernel_ms(lambda: field(x, t).backward(gout))
        if F == 1:
            ms.update(kernel_ms(lambda: sum(field.regularisers()).backward()))
        by = l2_bytes(F)
        res[f"F{F}"]["kernels"] = {k: {"ms": round(v, 4), "l2_bytes": by[k], "GB_per_s": round(by[k] / v / 1e6, 1)}
                                   for k, v in ms.items()}
    line = json.dumps(res, default=lambda v: round(v, 4))
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
