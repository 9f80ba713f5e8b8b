"""Which C entry points each public method of the rasterizer calls, without a GPU: the library is the recording
stub of test_binding_cpu, tensors live on the CPU.  For every call shape and every differentiable output, a loss on
that output alone is back-propagated, and the test checks the sequence of dgr_* calls, the outputs' order and shapes,
the shape (or None) of every input's gradient, and that the optional gradient pointers the loss does not use reach
the library as NULL.

The entry point is the narrowest one that takes every argument segment in use: forward maps (_aux) < normals (_nrm) <
surface maps (_surf); backward depth / alpha gradients (_aux) < camera (_cam) < normal map (_nrm) < surface maps
(_surf) < absolute screen-space gradient (_abs)."""
import pytest
import torch

import _dgm_lib
import diff_gaussian_rasterization as dgr
import synth
from test_binding_cpu import StubLib

P, W, H, F, C = 16, 32, 24, 2, 5
FWD = ("_aux", "_nrm", "_surf")
BWD = ("_aux", "_cam", "_nrm", "_surf", "_abs")
# argument index of each optional pointer of the backward, (single frame, batch), and the segment that adds it
SLOTS = {"depth": ("_aux", 24, 29), "alpha": ("_aux", 25, 30), "view": ("_cam", 35, 39), "proj": ("_cam", 36, 40),
         "campos": ("_cam", 37, 41), "normal": ("_nrm", 40, 44), "dnormals": ("_nrm", 41, 46),
         "median_depth": ("_surf", 45, 51), "distortion": ("_surf", 46, 52), "abs": ("_abs", 48, 55)}
MAP_CHANNELS = {"color": 3, "depth": 1, "alpha": 1, "median_depth": 1, "distortion": 1, "normal": 3, "features": C}


@pytest.fixture()
def stub(monkeypatch):
    st = StubLib()
    monkeypatch.setattr(_dgm_lib, "lib", lambda: st)
    monkeypatch.setattr(_dgm_lib, "stream_ptr", lambda: 0)
    monkeypatch.setattr(dgr, "_f32c", lambda t, name: None if (t is None or t.numel() == 0) else t.contiguous())
    monkeypatch.setattr(dgr, "_sizes", lambda P, W, H, R: (4096, 60 * R + 128, 8192, 4096,
                                                           (60 * R + 128 + 511) // 512 * 512, 8192))

    class FakeNotify:      # every frame fits: status words all zero
        host_ptr, event = 0x1000, 0x2000

        def __init__(self):
            self.words = [0] * (64 * 8)

        def wait(self):
            pass

    fake = FakeNotify()
    monkeypatch.setattr(dgr._Notify, "get", classmethod(lambda cls, dev: fake))
    monkeypatch.setattr(torch.cuda, "is_current_stream_capturing", lambda: False)
    dgr._Sizing.hint.clear()
    dgr._stacked.clear()
    yield st


def _normals(per_frame=False):
    return torch.rand((F, P, 3) if per_frame else (P, 3), requires_grad=True)


def _features(per_frame=False):
    return torch.rand((F, P, C) if per_frame else (P, C), requires_grad=True)


def _abs(batch):
    return torch.zeros(((F,) if batch else ()) + (P, 3), requires_grad=True)


# (id, batch, method, keyword factory, outputs in the documented order, request: camera_grad, abs, normals, surface,
# features)
CASES = [
    ("depth_alpha", False, "forward_depth_alpha", dict, ("color", "radii", "depth", "alpha"), ""),
    ("camera", False, "forward_with_camera_grad", dict, ("color", "radii"), "cam"),
    ("camera_maps", False, "forward_with_camera_grad", lambda: dict(depth_alpha=True),
     ("color", "radii", "depth", "alpha"), "cam"),
    ("abs", False, "forward_abs_grad", lambda: dict(means2D_abs=_abs(False)), ("color", "radii"), "abs"),
    ("abs_maps_camera", False, "forward_abs_grad",
     lambda: dict(means2D_abs=_abs(False), depth_alpha=True, camera_grad=True),
     ("color", "radii", "depth", "alpha"), "cam abs"),
    ("normal", False, "forward_normal", lambda: dict(normals=_normals()),
     ("color", "radii", "depth", "alpha", "normal"), "nrm"),
    ("normal_camera_abs", False, "forward_normal",
     lambda: dict(normals=_normals(), camera_grad=True, means2D_abs=_abs(False)),
     ("color", "radii", "depth", "alpha", "normal"), "cam abs nrm"),
    ("surface", False, "forward_surface", dict,
     ("color", "radii", "depth", "alpha", "median_depth", "distortion"), "surf"),
    ("surface_normal", False, "forward_surface", lambda: dict(normals=_normals(), near=0.5, far=20.0),
     ("color", "radii", "depth", "alpha", "median_depth", "distortion", "normal"), "nrm surf"),
    ("surface_normal_camera_abs", False, "forward_surface",
     lambda: dict(normals=_normals(), camera_grad=True, means2D_abs=_abs(False)),
     ("color", "radii", "depth", "alpha", "median_depth", "distortion", "normal"), "cam abs nrm surf"),
    ("features", False, "forward_features", lambda: dict(features=_features()),
     ("color", "radii", "depth", "alpha", "features"), "feat"),
    ("features_camera", False, "forward_features", lambda: dict(features=_features(), camera_grad=True),
     ("color", "radii", "depth", "alpha", "features"), "cam feat"),
    ("batch", True, "forward", dict, ("color", "radii"), ""),
    ("batch_abs", True, "forward", lambda: dict(means2D_abs=_abs(True)), ("color", "radii"), "abs"),
    ("batch_depth_alpha", True, "forward_depth_alpha", dict, ("color", "radii", "depth", "alpha"), ""),
    ("batch_depth_alpha_abs", True, "forward_depth_alpha", lambda: dict(means2D_abs=_abs(True)),
     ("color", "radii", "depth", "alpha"), "abs"),
    ("batch_camera", True, "forward_with_camera_grad", dict, ("color", "radii"), "cam"),
    ("batch_camera_maps_abs", True, "forward_with_camera_grad",
     lambda: dict(depth_alpha=True, means2D_abs=_abs(True)), ("color", "radii", "depth", "alpha"), "cam abs"),
    ("batch_normal_shared", True, "forward_normal", lambda: dict(normals=_normals()),
     ("color", "radii", "depth", "alpha", "normal"), "nrm"),
    ("batch_normal_per_frame_camera_abs", True, "forward_normal",
     lambda: dict(normals=_normals(True), camera_grad=True, means2D_abs=_abs(True)),
     ("color", "radii", "depth", "alpha", "normal"), "cam abs nrm"),
    ("batch_surface", True, "forward_surface", dict,
     ("color", "radii", "depth", "alpha", "median_depth", "distortion"), "surf"),
    ("batch_surface_normal_shared_abs", True, "forward_surface",
     lambda: dict(normals=_normals(), means2D_abs=_abs(True)),
     ("color", "radii", "depth", "alpha", "median_depth", "distortion", "normal"), "abs nrm surf"),
    ("batch_surface_normal_per_frame_camera", True, "forward_surface",
     lambda: dict(normals=_normals(True), camera_grad=True),
     ("color", "radii", "depth", "alpha", "median_depth", "distortion", "normal"), "cam nrm surf"),
    ("batch_features", True, "forward_features", lambda: dict(features=_features()),
     ("color", "radii", "depth", "alpha", "features"), "feat"),
    ("batch_features_camera", True, "forward_features", lambda: dict(features=_features(True), camera_grad=True),
     ("color", "radii", "depth", "alpha", "features"), "cam feat"),
    ("batch_features_surface", True, "forward_features", lambda: dict(features=_features(), surface=(0.2, 100.0)),
     ("color", "radii", "depth", "alpha", "features", "median_depth", "distortion"), "feat surf"),
    ("batch_features_normal_surface", True, "forward_features",
     lambda: dict(features=_features(True), normals=_normals(), surface=(0.2, 100.0)),
     ("color", "radii", "depth", "alpha", "features", "median_depth", "distortion", "normal"), "feat nrm surf"),
]
ROWS = [pytest.param(case, loss, id=f"{case[0]}-{loss}") for case in CASES for loss in case[4] if loss != "radii"]


def _widest(base, suffixes, used):
    return base + max((s for s in suffixes if s in used), key=suffixes.index, default="")


@pytest.mark.parametrize("case,loss", ROWS)
def test_dispatch(stub, case, loss):
    label, batch, method, make_kw, outputs, request = case
    request = set(request.split())
    sc = synth.gaussian_scene(n=P, seed=0)
    leaves = {k: sc[k].clone().requires_grad_(True) for k in ("means3D", "opacities", "scales", "rotations", "shs")}
    cams = [synth.look_at_camera(azimuth_deg=30.0 * k, width=W, height=H) for k in range(F if batch else 1)]
    sets = [synth.raster_settings_for(c, torch.ones(3), settings_cls=dgr.GaussianRasterizationSettings) for c in cams]
    cam_leaves = []
    for s in sets:    # every camera tensor could take a gradient: only camera_grad may give it one
        for t in (s.viewmatrix, s.projmatrix, s.campos):
            cam_leaves.append(t.requires_grad_(True))
    lead = (F,) if batch else ()
    m2d = torch.zeros(lead + (P, 3), requires_grad=True)
    kw = make_kw()
    r = dgr.BatchGaussianRasterizer(sets) if batch else dgr.GaussianRasterizer(sets[0])

    out = getattr(r, method)(means2D=m2d, **leaves, **kw)

    assert len(out) == len(outputs)
    for name, o in zip(outputs, out):
        if name == "radii":
            assert o.shape == lead + (P,) and o.dtype == torch.int32
        else:
            assert o.shape == lead + (MAP_CHANNELS[name], H, W), name
    stub.calls.clear()
    out[outputs.index(loss)].sum().backward()

    # the C calls of the backward, in order
    names = [c[0] for c in stub.calls if c[0].startswith(("dgr_backward", "dgr_features_bwd"))]
    base = "dgr_backward_batch" if batch else "dgr_backward"
    used = set()
    if loss in ("depth", "alpha"):
        used.add("_aux")
    if "cam" in request:
        used.add("_cam")
    if loss == "normal":
        used.add("_nrm")
    if loss in ("median_depth", "distortion"):
        used.add("_surf")
    if "abs" in request:
        used.add("_abs")
    sym = _widest(base, BWD, used)
    assert names == (["dgr_features_bwd"] if loss == "features" else []) + [sym]
    args = [c[1] for c in stub.calls if c[0] == sym][0]
    width = BWD.index(sym[len(base):]) if sym != base else -1
    for slot, (seg, i_single, i_batch) in SLOTS.items():
        if BWD.index(seg) > width:
            continue
        want = {"depth": loss == "depth", "alpha": loss == "alpha", "normal": loss == "normal",
                "dnormals": loss == "normal", "median_depth": loss == "median_depth",
                "distortion": loss == "distortion", "abs": "abs" in request}.get(slot, "cam" in request)
        assert bool(args[i_batch if batch else i_single]) == want, slot

    # gradients of every input
    for k, shape in dict(means3D=(P, 3), opacities=(P, 1), scales=(P, 3), rotations=(P, 4), shs=(P, 16, 3)).items():
        assert leaves[k].grad is not None and leaves[k].grad.shape == shape, k
    assert m2d.grad.shape == lead + (P, 3)
    for key, wanted in (("normals", loss == "normal"), ("features", loss == "features"), ("means2D_abs", True)):
        if key in kw:
            assert (kw[key].grad.shape if kw[key].grad is not None else None) == \
                (kw[key].shape if wanted else None), key
    for t in cam_leaves:
        assert (t.grad.shape if t.grad is not None else None) == (t.shape if "cam" in request else None)


@pytest.mark.parametrize("case", [pytest.param(c, id=c[0]) for c in CASES])
def test_forward_dispatch(stub, case):
    """The forward's C calls: the narrowest entry point that writes every requested map, then the feature pass."""
    label, batch, method, make_kw, outputs, request = case
    request = set(request.split())
    sc = synth.gaussian_scene(n=P, seed=0)
    cams = [synth.look_at_camera(azimuth_deg=30.0 * k, width=W, height=H) for k in range(F if batch else 1)]
    sets = [synth.raster_settings_for(c, torch.ones(3), settings_cls=dgr.GaussianRasterizationSettings) for c in cams]
    r = dgr.BatchGaussianRasterizer(sets) if batch else dgr.GaussianRasterizer(sets[0])
    getattr(r, method)(means2D=None, **{k: sc[k] for k in ("means3D", "opacities", "scales", "rotations", "shs")},
                       **make_kw())
    names = [c[0] for c in stub.calls if c[0].startswith(("dgr_forward", "dgr_features_fwd"))]
    used = {s for s, on in (("_aux", "depth" in outputs), ("_nrm", "normal" in outputs),
                            ("_surf", "median_depth" in outputs)) if on}
    sym = _widest("dgr_forward_batch" if batch else "dgr_forward", FWD, used)
    assert names == [sym] + (["dgr_features_fwd"] if "feat" in request else [])
