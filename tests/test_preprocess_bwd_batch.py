"""The per-Gaussian backward of a frame batch runs once for all frames and sums the gradients of shared inputs
over the frames on chip.  A batch must equal F single-frame calls: images and radii identical, per-frame
gradients and summed gradients within the accumulation-order tolerance, for every split of the inputs into
per-frame and shared ones, for SH or precomputed colours, scale/rotation or precomputed covariances, for frame
counts that do and do not fill the frames one block covers, and for a Gaussian count that is not a multiple of
the Gaussians a warp covers."""
import pytest
import torch

import util
from test_raster_gpu import TOL, _cam_cuda, _cuda

pytestmark = pytest.mark.gpu

W, H, P = 128, 80, 2999
PF_ALL = ("means3D", "scales", "rotations", "opacities", "shs", "colors_precomp", "cov3D_precomp")
DGMESH = ("means3D", "scales", "rotations")          # DG-Mesh: deformed per frame; opacity and SH shared


def _inputs(F, per_frame, use_colors=False, use_cov=False, seed=3):
    """Leaves of one batch (per-frame inputs [F,P,.], shared ones [P,.]) and the frames' settings.  The cameras
    circle the scene close up, so each sees part of it: many Gaussians are culled in some frames only."""
    import diff_gaussian_rasterization as dgr
    import synth
    sc, _ = util.small_scene(n=P, W=W, H=H, seed=seed, scale=0.04)
    g = torch.Generator().manual_seed(seed)
    bg = torch.tensor([0.3, 0.6, 0.9], device="cuda")
    cams = [_cam_cuda(synth.look_at_camera(azimuth_deg=10.0 + 360.0 * k / F, elevation_deg=15.0, radius=1.6, width=W,
                                           height=H, fovx=0.6911, fovy=0.6911 * H / W)) for k in range(F)]
    sets = [synth.raster_settings_for(c, bg, settings_cls=dgr.GaussianRasterizationSettings) for c in cams]
    base = {"means3D": sc["means3D"], "opacities": sc["opacities"], "scales": sc["scales"],
            "rotations": sc["rotations"]}
    if use_colors:
        base["colors_precomp"] = sc["shs"][:, 0, :].abs()
    else:
        base["shs"] = sc["shs"]
    # a small per-frame perturbation of each input (what a deformation network adds for the frame's time)
    jitter = {"means3D": lambda x, r: x + 0.02 * r, "scales": lambda x, r: x * torch.exp(0.1 * r),
              "rotations": lambda x, r: x + 0.02 * r, "opacities": lambda x, r: x * (0.9 + 0.05 * r.clamp(-1, 1)),
              "shs": lambda x, r: x + 0.05 * r, "colors_precomp": lambda x, r: x * (0.9 + 0.05 * r.clamp(-1, 1))}
    leaves = {}
    for k, x in base.items():
        if k in per_frame:
            x = torch.stack([jitter[k](x, torch.randn(x.shape, generator=g)) for _ in range(F)])
        leaves[k] = x
    if use_cov:
        sc_, ro = leaves.pop("scales"), leaves.pop("rotations")
        pf_cov = "scales" in per_frame or "rotations" in per_frame or "cov3D_precomp" in per_frame
        if pf_cov:
            sc_ = sc_ if sc_.ndim == 3 else sc_[None].expand(F, -1, -1)
            ro = ro if ro.ndim == 3 else ro[None].expand(F, -1, -1)
            leaves["cov3D_precomp"] = torch.stack([util.cov3d_torch(sc_[f], ro[f]) for f in range(F)])
        else:
            leaves["cov3D_precomp"] = util.cov3d_torch(sc_, ro)
    return {k: v.cuda().contiguous() for k, v in leaves.items()}, sets


def _batch_vs_single_frames(F, leaves, sets):
    import diff_gaussian_rasterization as dgr
    dpix = torch.randn(F, 3, H, W, generator=torch.Generator().manual_seed(7)).cuda()
    lb = {k: v.clone().requires_grad_(True) for k, v in leaves.items()}
    m2d = torch.zeros(F, P, 3, device="cuda", requires_grad=True)
    color, radii = dgr.BatchGaussianRasterizer(sets)(means2D=m2d, **lb)
    color.backward(dpix)
    ls = {k: v.clone().requires_grad_(True) for k, v in leaves.items()}
    for f in range(F):
        m1 = torch.zeros(P, 3, device="cuda", requires_grad=True)
        # per-frame inputs have a leading frame dimension (ndim 3, or 4 for SH)
        kw = {k: (v[f] if v.ndim == (4 if k == "shs" else 3) else v) for k, v in ls.items()}
        c1, r1 = dgr.GaussianRasterizer(sets[f])(means2D=m1, **kw)
        c1.backward(dpix[f])
        assert torch.equal(c1, color[f]) and torch.equal(r1, radii[f]), f
        assert util.rel_err(m2d.grad[f], m1.grad) < TOL, f
    for k in leaves:
        assert lb[k].grad.shape == ls[k].grad.shape, k
        assert util.rel_err(lb[k].grad, ls[k].grad) < TOL, k
    return radii


@pytest.mark.parametrize("F", [1, 3, 8, 11])
@pytest.mark.parametrize("per_frame", [PF_ALL, DGMESH, ("opacities", "shs")], ids=["none_shared", "dgmesh", "opac_color"])
def test_batch_equals_single_frames(F, per_frame):
    leaves, sets = _inputs(F, per_frame)
    radii = _batch_vs_single_frames(F, leaves, sets)
    if F > 1:   # the scene exercises Gaussians that are culled in some frames and visible in others
        assert bool(((radii == 0).any(0) & (radii > 0).any(0)).any())


@pytest.mark.parametrize("per_frame", [(), PF_ALL], ids=["all_shared", "none_shared"])
@pytest.mark.parametrize("use_colors,use_cov", [(True, False), (False, True), (True, True)],
                         ids=["colors_precomp", "cov3D_precomp", "both"])
def test_precomputed_inputs(use_colors, use_cov, per_frame):
    leaves, sets = _inputs(11, per_frame, use_colors, use_cov)
    _batch_vs_single_frames(11, leaves, sets)


@pytest.mark.parametrize("use_colors", [False, True], ids=["shs", "colors_precomp"])
def test_unused_gradients_may_be_null(monkeypatch, use_colors):
    """dgr_backward_batch takes NULL for dL_dcolor when SH colours are given and for dL_dcov3D without
    cov3D_precomp.  Every other output must be what it is when both buffers are given."""
    import _dgm_lib
    import diff_gaussian_rasterization as dgr
    F = 3
    leaves, sets = _inputs(F, DGMESH, use_colors)
    real = _dgm_lib.lib()
    checked = []

    class Spy:
        def __getattr__(self, name):
            return getattr(real, name)

        def dgr_backward_batch(self, *args):
            outs = []
            for null in (False, True):
                bufs = [torch.zeros(F * P * 48, device="cuda") for _ in range(8)]   # [29:37]: the eight outputs
                a = list(args)
                a[29:37] = [b.data_ptr() for b in bufs]
                if null:
                    if args[8] is not None:         # shs given: the colour gradient is scratch
                        a[31] = None
                    if args[13] is None:            # no cov3D_precomp
                        a[33] = None
                assert real.dgr_backward_batch(*a) == 0
                outs.append(bufs)
            torch.cuda.synchronize()
            for i, (x, y) in enumerate(zip(*outs)):
                if i in (2, 4) and (i != 2 or not use_colors):
                    continue
                assert util.rel_err(y, x) < 1e-5, i
            checked.append(True)
            return real.dgr_backward_batch(*args)

    monkeypatch.setattr(_dgm_lib, "lib", lambda: Spy())
    lb = {k: v.clone().requires_grad_(True) for k, v in leaves.items()}
    color, _ = dgr.BatchGaussianRasterizer(sets)(means2D=None, **lb)
    color.backward(torch.randn(color.shape, generator=torch.Generator().manual_seed(1)).cuda())
    assert checked and all(torch.isfinite(v.grad).all() for v in lb.values())
