"""Shared helpers for the parity tests."""
import importlib.util
import math
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_DIR = os.path.join(ROOT, "oracle", "_ref")


def small_scene(n=400, W=96, H=64, seed=0, scale=0.05, degree=3):
    """A tiny scene for oracle-speed tests (torch CPU tensors + camera namespace)."""
    import synth
    sc = synth.gaussian_scene(n=n, seed=seed, sh_degree=degree, scale_median=scale)
    cam = synth.look_at_camera(azimuth_deg=25.0 + 10 * seed, elevation_deg=15.0, radius=4.0, width=W, height=H,
                               fovx=0.6911, fovy=0.6911 * H / W)
    return sc, cam


def oracle_forward(orc, sc, cam, bg, degree=3, use_colors=False, use_cov=False):
    kw = dict(means3D=sc["means3D"].numpy(), opacities=sc["opacities"].numpy(),
              view=cam.world_view_transform.numpy(), proj=cam.full_proj_transform.numpy(),
              campos=cam.camera_center.numpy(), W=cam.image_width, H=cam.image_height,
              tan_fovx=math.tan(cam.FoVx * 0.5), tan_fovy=math.tan(cam.FoVy * 0.5), bg=np.asarray(bg, np.float32))
    if use_colors:
        kw["colors_precomp"] = sc["shs"][:, 0, :].abs().numpy()
    else:
        kw["shs"], kw["degree"] = sc["shs"].numpy(), degree
    if use_cov:
        kw["cov3D_precomp"] = cov3d_torch(sc["scales"], sc["rotations"]).numpy()
    else:
        kw["scales"], kw["rotations"] = sc["scales"].numpy(), sc["rotations"].numpy()
    return orc.forward(**kw)


def cov3d_torch(scales, rots):
    """Sigma = (S R)^T (S R) from un-normalised quaternions (what the kernels compute)."""
    r, x, y, z = rots.unbind(-1)
    R = torch.stack([1 - 2 * (y * y + z * z), 2 * (x * y - r * z), 2 * (x * z + r * y),
                     2 * (x * y + r * z), 1 - 2 * (x * x + z * z), 2 * (y * z - r * x),
                     2 * (x * z - r * y), 2 * (y * z + r * x), 1 - 2 * (x * x + y * y)], -1).reshape(-1, 3, 3)
    # glm columns are the rows written above -> the stacked matrix is R^T in math notation
    Rm = R.transpose(1, 2)
    L = Rm @ torch.diag_embed(scales)
    S = L @ L.transpose(1, 2)
    return torch.stack([S[:, 0, 0], S[:, 0, 1], S[:, 0, 2], S[:, 1, 1], S[:, 1, 2], S[:, 2, 2]], -1).contiguous()


def load_reference_rasterizer():
    """Import the UNMODIFIED reference extension built by oracle/build_ref.py under the
    module name `ref_dgr` (the product drop-in owns the name diff_gaussian_rasterization)."""
    if "ref_dgr" in sys.modules:
        return sys.modules["ref_dgr"]
    pkg = os.path.join(REF_DIR, "diff_gaussian_rasterization")
    init = os.path.join(pkg, "__init__.py")
    if not (os.path.exists(init) and os.path.exists(os.path.join(pkg, "_C.so"))):
        return None
    spec = importlib.util.spec_from_file_location("ref_dgr", init, submodule_search_locations=[pkg])
    mod = importlib.util.module_from_spec(spec)
    sys.modules["ref_dgr"] = mod
    spec.loader.exec_module(mod)
    return mod


def _align(off, a=128):
    return (off + a - 1) // a * a


def parse_ref_buffers(geom, binning, img, P, R, W, H):
    """Views into the reference's three opaque byte tensors, following the obtain()
    sequence of GeometryState / BinningState / ImageState::fromChunk
    (dgr/cuda_rasterizer/rasterizer_impl.cu:155-194; alignment 128 on the ADDRESS)."""
    out = {}

    def take(buf, base, off, count, dtype, shape=None):
        itemsize = torch.tensor([], dtype=dtype).element_size()
        a = _align(base + off) - base
        t = buf[a:a + count * itemsize].view(dtype)
        if shape:
            t = t.view(*shape)
        return t, a + count * itemsize

    b = geom.data_ptr()
    off = 0
    out["depths"], off = take(geom, b, off, P, torch.float32)
    out["clamped"], off = take(geom, b, off, 3 * P, torch.uint8, (P, 3))
    out["internal_radii"], off = take(geom, b, off, P, torch.int32)
    out["means2D"], off = take(geom, b, off, 2 * P, torch.float32, (P, 2))
    out["cov3D"], off = take(geom, b, off, 6 * P, torch.float32, (P, 6))
    out["conic_opacity"], off = take(geom, b, off, 4 * P, torch.float32, (P, 4))
    out["rgb"], off = take(geom, b, off, 3 * P, torch.float32, (P, 3))
    out["tiles_touched"], off = take(geom, b, off, P, torch.int32)
    N = W * H
    b = img.data_ptr()
    off = 0
    out["final_T"], off = take(img, b, off, N, torch.float32)
    out["n_contrib"], off = take(img, b, off, N, torch.int32)
    out["ranges_full"], off = take(img, b, off, 2 * N, torch.int32, (N, 2))
    T = ((W + 15) // 16) * ((H + 15) // 16)
    out["ranges"] = out["ranges_full"][:T]
    if R > 0:
        b = binning.data_ptr()
        off = 0
        out["point_list"], off = take(binning, b, off, R, torch.int32)
        _, off = take(binning, b, off, R, torch.int32)
        out["point_list_keys"], off = take(binning, b, off, R, torch.int64)
    else:
        out["point_list"] = torch.zeros(0, dtype=torch.int32, device=geom.device)
        out["point_list_keys"] = torch.zeros(0, dtype=torch.int64, device=geom.device)
    return out


def rel_err(a, b):
    """max |a-b| / (max|b| + tiny): the 'relative to the tensor's scale' error used for the
    1e-4 fp32 contract (north_star)."""
    a = torch.as_tensor(a, dtype=torch.float64).detach().cpu()
    b = torch.as_tensor(b, dtype=torch.float64).detach().cpu()
    if a.numel() == 0:
        return 0.0
    return float((a - b).abs().max() / (b.abs().max() + 1e-30))


def load_reference_pymodules():
    """The reference's pure-PyTorch modules (copied to oracle/_ref/refpy by oracle/build_ref.py, or read
    from /root/reference when present) as a package `refpy` whose unavailable third-party imports
    (trimesh, open3d, pytorch3d, ...) are replaced by inert stand-ins: only the torch/numpy functions
    of the hot path are exercised.  Returns None when neither location exists."""
    if "refpy" in sys.modules:
        return sys.modules["refpy"]
    refpy = os.path.join(REF_DIR, "refpy")
    if not os.path.isdir(refpy):
        return None
    return _load_refpy(refpy)


def load_reference_networks():
    """The reference's `time_utils` / `rigid_utils` for the MLP parity tests: the reference's own modules where
    oracle/_ref/refpy is built, else the fp32 restatement (tests/ref_time_utils.py, pinned to the reference's
    stored outputs by tests/test_golden_py.py) with this package's rigid_utils."""
    ref = load_reference_pymodules()
    if ref is not None:
        return ref
    import types
    import ref_time_utils
    return types.SimpleNamespace(time_utils=ref_time_utils, rigid_utils=importlib.import_module("utils.rigid_utils"))


def load_reference_dpsr():
    """The reference's `dpsr` for the DPSR parity tests: its own module where oracle/_ref/refpy is built, else the
    restatement tests/ref_dpsr.py (pinned to the reference's stored field and gradients by tests/test_dpsr.py)."""
    ref = load_reference_pymodules()
    if ref is not None:
        return ref
    import types
    import ref_dpsr
    return types.SimpleNamespace(dpsr=ref_dpsr)


def _load_refpy(refpy):
    import types
    from unittest import mock
    for name in ("trimesh", "imageio", "skimage", "skimage.measure", "pytorch3d", "pytorch3d.structures",
                 "pytorch3d.renderer", "igl", "open3d", "plyfile"):
        if name not in sys.modules:
            try:
                __import__(name)
            except Exception:
                sys.modules[name] = mock.MagicMock()
    pkg = types.ModuleType("refpy")
    pkg.__path__ = [refpy]
    sys.modules["refpy"] = pkg
    # the reference's time_utils does `from utils.rigid_utils import exp_se3`: `utils` must resolve OUR
    # modules first (utils.time_utils, utils.renderer) and fall through to the reference copy for the rest
    utils = types.ModuleType("utils")
    utils.__path__ = [os.path.join(ROOT, "dg-mesh_b200", "utils"), refpy]
    sys.modules.setdefault("utils", utils)
    for sub in ("rigid_utils",):
        spec = importlib.util.spec_from_file_location(f"utils.{sub}", os.path.join(refpy, f"{sub}.py"))
        m = importlib.util.module_from_spec(spec)
        sys.modules[f"utils.{sub}"] = m
        spec.loader.exec_module(m)
    for sub in ("dpsr_utils", "dpsr", "time_utils", "graphics_utils", "sh_utils"):
        spec = importlib.util.spec_from_file_location(f"refpy.{sub}", os.path.join(refpy, f"{sub}.py"))
        m = importlib.util.module_from_spec(spec)
        sys.modules[f"refpy.{sub}"] = m
        spec.loader.exec_module(m)
        setattr(pkg, sub, m)
    # the reference modules have bound what they need; from here on `utils.rigid_utils` is this repo's again
    pkg.rigid_utils = sys.modules.pop("utils.rigid_utils")
    return pkg


def rel_l2(a, b):
    """||a - b||_2 / ||b||_2 (the error measure for bf16 gradient tensors: single elements of a bf16
    backward can be off by far more than the tensor as a whole)."""
    a = torch.as_tensor(a, dtype=torch.float64).detach().cpu()
    b = torch.as_tensor(b, dtype=torch.float64).detach().cpu()
    return float((a - b).norm() / (b.norm() + 1e-30))
