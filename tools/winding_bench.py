"""Cost of the generalized winding number (mesh_distance.winding_number, csrc/winding.cu), of signed_distance next
to point_mesh_distance, and of mesh_metrics(iou_points=100_000):

* two shapes, CUDA events around repeated calls after warm-up:
  - a diso.DiffMC mesh of a sphere joined with a torus at G = 288 (about 343k faces), 200 000 queries near it;
  - an icosphere of 5 242 880 faces, 10^6 queries near it;
  each timed as the build alone (one query at beta = 2), winding_number at beta = 2 on all queries and at
  beta = inf on a subset (exact mode costs F solid angles per query), signed_distance and point_mesh_distance
  (forward, and forward + backward) on all queries.  queries/s is over the query part (call minus build);
* at the small shape, the same exact sum as a chunked torch fp32 brute force on a subset of queries;
* mesh_metrics on icospheres of radii 1 and 1.05 at 100 000 points with iou_points = 0 and 100 000;
* the card, its power limit and SM clock, read in the same run, and one JSON line.

Every call includes the Python checks (one host read of the face index range).
Usage: python tools/winding_bench.py [--reps 3] [--runs 2]"""
import argparse
import json
import math
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "dg-mesh_b200"), os.path.join(ROOT, "tests"), os.path.join(ROOT, "tools")):
    if p not in sys.path:
        sys.path.insert(0, p)

import torch  # noqa: E402
from mesh_distance_bench import card, near, timed  # noqa: E402


def brute_force(p, v, f, pairs=1 << 25):
    """The exact winding number as plain torch fp32 statements, in chunks of about `pairs` (query, face) pairs."""
    fl = f.long()
    A, B, C = v[fl[:, 0]], v[fl[:, 1]], v[fl[:, 2]]
    step = max(1, pairs // f.shape[0])
    out = []
    for i in range(0, p.shape[0], step):
        q = p[i:i + step, None]
        a, b, c = A[None] - q, B[None] - q, C[None] - q
        det = (a * torch.linalg.cross(b, c, dim=2)).sum(2)
        la, lb, lc = a.norm(dim=2), b.norm(dim=2), c.norm(dim=2)
        den = la * lb * lc + (a * b).sum(2) * lc + (b * c).sum(2) * la + (c * a).sum(2) * lb
        om = torch.where(det == 0, 0.0, 2 * torch.atan2(det, den))
        out.append(om.double().sum(1) / (4 * math.pi))
    return torch.cat(out).float()


def shapes():
    from test_meshrast_fp64 import _sdf_mesh
    from test_metrics_gpu import _icosphere
    v, f = _sdf_mesh(288)
    v, f = v.cuda(), f.cuda()
    yield "diffmc G=288", v, f, near(v, f, 200_000, 0), 20_000, 2_000
    v, f = _icosphere(1.0, faceting=2e-6)
    yield "large icosphere", v, f.int(), near(v, f, 1_000_000, 2), 2_000, 0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--runs", type=int, default=2, help="repeat every timing this many times to show the spread")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "winding_bench needs a GPU"
    from mesh_distance import point_mesh_distance, signed_distance, winding_number
    info = card()
    print(f"card: {info}")
    rows = []
    for name, v, f, p, q_exact, q_brute in shapes():
        vv, pp = v.clone().requires_grad_(True), p.clone().requires_grad_(True)
        g = torch.ones(p.shape[0], device="cuda")
        pe = p[:q_exact].contiguous()

        def sdf_fwd_bwd():
            signed_distance(pp, vv, f)[0].backward(g)

        def pmd_fwd_bwd():
            point_mesh_distance(pp, vv, f)[0].backward(g)

        r = {"shape": name, "V": v.shape[0], "F": f.shape[0], "Q": p.shape[0], "Q_exact": q_exact, "runs": []}
        for _ in range(args.runs):
            t = {"build_ms": timed(lambda: winding_number(p[:1], v, f), args.reps),
                 "winding_beta2_ms": timed(lambda: winding_number(p, v, f), args.reps),
                 "winding_exact_subset_ms": timed(lambda: winding_number(pe, v, f, math.inf), 1),
                 "signed_distance_ms": timed(lambda: signed_distance(p, v, f), args.reps),
                 "point_mesh_distance_ms": timed(lambda: point_mesh_distance(p, v, f), args.reps),
                 "signed_distance_fwd_bwd_ms": timed(sdf_fwd_bwd, args.reps),
                 "point_mesh_distance_fwd_bwd_ms": timed(pmd_fwd_bwd, args.reps)}
            t["beta2_queries_per_s"] = p.shape[0] / max(t["winding_beta2_ms"] - t["build_ms"], 1e-6) * 1e3
            t["exact_queries_per_s"] = q_exact / max(t["winding_exact_subset_ms"] - t["build_ms"], 1e-6) * 1e3
            t["exact_solid_angles_per_s"] = t["exact_queries_per_s"] * f.shape[0]
            if q_brute:
                pb = p[:q_brute].contiguous()
                t["torch_fp32_brute_force_ms"] = timed(lambda: brute_force(pb, v, f), 1)
                t["torch_fp32_queries_per_s"] = q_brute / t["torch_fp32_brute_force_ms"] * 1e3
                t["torch_fp32_max_diff_to_exact"] = float((brute_force(pb, v, f) -
                                                           winding_number(pb, v, f, math.inf)).abs().max())
            r["runs"].append(t)
        print(json.dumps(r))
        rows.append(r)
        del vv, pp
    from test_metrics_gpu import _icosphere
    from mesh_metrics import mesh_metrics
    m1, m2 = _icosphere(1.0), _icosphere(1.05)
    mm = {}
    for n in (0, 100_000):
        gen = torch.Generator(device="cuda").manual_seed(0)
        mm[f"iou_points={n}"] = [timed(lambda: mesh_metrics(m1, m2, 100_000, thresholds=(0.05,), generator=gen,
                                                            iou_points=n), 2) for _ in range(args.runs)]
    print(f"mesh_metrics at 100 000 points (ms per run): {mm}")
    print(json.dumps({"winding_bench": rows, "mesh_metrics_100k_ms": mm, "card": info}))


if __name__ == "__main__":
    main()
