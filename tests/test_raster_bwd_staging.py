"""Gradients of the blend backward against the CPU oracle on scenes that reach each path of its staged
contraction (csrc/raster_bwd.cu: a warp stages (w, alpha T) of up to CHUNK records, contracts them when the
chunk is full and once more, partially filled, before each batch of RB records is flushed):

* one batch holding more than 2 * CHUNK contributing records of one warp (several full chunks, then a partial one);
* tile lists of several batches;
* an image whose size is not a multiple of the 16x16 tile, so some lanes lie outside the image.

Same bar as test_raster_gpu.test_against_cpu_oracle: integer state equal, image and gradients within 1e-4."""
import numpy as np
import pytest
import torch

import util
from test_raster_gpu import TOL, _cam_cuda, _cuda, run_ours

pytestmark = pytest.mark.gpu
CHUNK = 16   # records a warp stages before it contracts them
RB = 256     # records per batch


def _clustered_scene(n, W, H, seed, opacity_scale):
    """n large, faint Gaussians around the origin: every one covers every pixel and contributes to it."""
    sc, cam = util.small_scene(n=n, W=W, H=H, seed=seed, scale=0.3)
    g = torch.Generator().manual_seed(seed)
    sc["means3D"] = 0.05 * torch.randn(n, 3, generator=g)
    sc["opacities"] = sc["opacities"] * opacity_scale
    return sc, cam


def _contributors_per_warp(o, W, H):
    """Largest number of records with at least one contributing pixel in one warp's 8x4 block (fp64 restatement
    of the forward's tests: power <= 0, alpha >= 1/255, position < n_contrib of the pixel)."""
    m2 = o["means2D"].reshape(-1, 2).astype(np.float64)
    co = o["conic_opacity"].reshape(-1, 4).astype(np.float64)
    nc = o["n_contrib"].reshape(H, W).astype(np.int64)
    gx = (W + 15) // 16
    best = 0
    for t, (a, b) in enumerate(o["ranges"].reshape(-1, 2)):
        if b <= a:
            continue
        ids = o["point_list"][a:b].astype(np.int64)
        pos = np.arange(b - a)[:, None]
        for w in range(8):
            x0, y0 = (t % gx) * 16 + (w & 1) * 8, (t // gx) * 16 + (w >> 1) * 4
            ys, xs = [v.ravel() for v in np.mgrid[y0:y0 + 4, x0:x0 + 8]]
            inside = (xs < W) & (ys < H)
            ncp = np.where(inside, nc[np.minimum(ys, H - 1), np.minimum(xs, W - 1)], 0)
            dx, dy = m2[ids, :1] - xs[None], m2[ids, 1:] - ys[None]
            power = -0.5 * (co[ids, :1] * dx * dx + co[ids, 2:3] * dy * dy) - co[ids, 1:2] * dx * dy
            alpha = np.minimum(0.99, co[ids, 3:] * np.exp(power))
            contrib = (power <= 0) & (alpha >= 1 / 255) & (pos < ncp[None])
            best = max(best, int(contrib.any(1).sum()))
    return best


@pytest.mark.parametrize("scene", ["full_chunks_in_one_batch", "several_batches", "ragged_image"])
def test_blend_backward_against_cpu_oracle(scene):
    from oracle.oracle import RasterOracle
    if scene == "full_chunks_in_one_batch":
        W, H = 32, 32
        sc, cam = _clustered_scene(120, W, H, seed=1, opacity_scale=0.05)
    elif scene == "several_batches":
        W, H = 32, 32
        sc, cam = _clustered_scene(600, W, H, seed=2, opacity_scale=0.02)
    else:
        W, H = 45, 37
        sc, cam = util.small_scene(n=1500, W=W, H=H, seed=4, scale=0.05)
    o = util.oracle_forward(RasterOracle(32), sc, cam, [1, 1, 1])
    lens = (o["ranges"].reshape(-1, 2)[:, 1].astype(np.int64) - o["ranges"].reshape(-1, 2)[:, 0])
    if scene == "full_chunks_in_one_batch":
        assert lens.max() <= RB and _contributors_per_warp(o, W, H) > 2 * CHUNK
    elif scene == "several_batches":
        assert lens.max() > 2 * RB and _contributors_per_warp(o, W, H) > RB
    else:
        assert W % 16 and H % 16 and lens.max() > 0
    dpix = np.random.default_rng(5).standard_normal((3, H, W)).astype(np.float32)
    g = RasterOracle(32).backward(o, dpix)
    a = run_ours(_cuda(sc), _cam_cuda(cam), torch.ones(3, device="cuda"), 3, False, False,
                 torch.from_numpy(dpix).cuda())
    assert np.array_equal(a["radii"].cpu().numpy(), o["radii"])
    assert a["R"] == o["num_rendered"]
    assert np.array_equal(a["n_contrib"].cpu().numpy().astype(np.uint32).ravel(), o["n_contrib"].ravel())
    assert util.rel_err(a["color"].cpu(), o["color"]) < TOL
    names = dict(means3D="dL_dmean3D", opacities="dL_dopacity", scales="dL_dscale", rotations="dL_drot",
                 shs="dL_dsh", means2D="dL_dmean2D")
    for k, gk in names.items():
        ref = torch.from_numpy(g[gk]).reshape(a["grads"][k].shape)
        assert util.rel_err(a["grads"][k].cpu(), ref) < TOL, k
