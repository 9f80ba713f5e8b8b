#!/usr/bin/env python
"""Compare two `bench.py --dump-outputs DIR` directories written by two builds of the library:
    python tools/compare_outputs.py NEW_DIR OLD_DIR
The rendered sample must be bit-identical; every gradient must satisfy max|a - b| / max|b| <= 1e-5 (the bar of
the frame-batch-vs-single-frame tests).  Prints one JSON object with each value and exits 1 on a failure."""
import json
import os
import sys

import numpy as np

GRAD_TOL = 1e-5


def main():
    new_dir, old_dir = sys.argv[1], sys.argv[2]
    names = sorted(f for f in os.listdir(old_dir) if f.endswith(".npy"))
    assert names and "color_sample.npy" in names, f"no dump in {old_dir}"
    out, ok = {}, True
    for f in names:
        a, b = np.load(os.path.join(new_dir, f)), np.load(os.path.join(old_dir, f))
        assert a.shape == b.shape, f
        if f == "color_sample.npy":
            same = bool(np.array_equal(a.view(np.uint32), b.view(np.uint32)))
            out[f] = {"bit_identical": same}
            ok &= same
        else:
            a64, b64 = a.astype(np.float64), b.astype(np.float64)
            e = float(np.abs(a64 - b64).max() / max(np.abs(b64).max(), 1e-30))
            out[f] = {"rel_err": e}
            ok &= e <= GRAD_TOL
    out["ok"] = bool(ok)
    print(json.dumps(out))
    return 0 if ok else 1


if __name__ == "__main__":
    sys.exit(main())
