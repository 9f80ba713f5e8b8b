"""Golden vectors generated from the reference's own PyTorch modules (tests/golden/make_golden_py.py,
fp32 on the CPU of the build container): they pin (CPU) the numpy DPSR oracle, the bf16 restatement
of the MLPs and the drop-in modules' parameter layout / initialisation order, and are (GPU) a parity
target for the CUDA MLP and DPSR paths that does not need the reference at test time."""
import glob
import importlib
import os

import numpy as np
import pytest
import torch

import util
from oracle.oracle import dpsr_forward_np

GOLD = os.path.join(os.path.dirname(__file__), "golden")
MLP_FILES = sorted(glob.glob(os.path.join(GOLD, "mlp_*.npz")))


def _mlp_case(path, device):
    import sys
    sys.path.insert(0, GOLD)
    from make_golden_py import mlp_inputs, param_checksum
    z = np.load(path)
    cls, blender = os.path.basename(path)[4:-4].rsplit("_", 1)
    seed = int(z["seed"])
    tu = importlib.import_module("utils.time_utils")
    torch.manual_seed(seed)
    net = getattr(tu, cls)(is_blender=bool(int(blender)))
    if cls == "DeformNetworkNormalSep":
        torch.manual_seed(seed + 100)
        torch.nn.init.normal_(net.gaussian_normal.weight, std=0.05)
    x, t, gout = mlp_inputs(257, seed)
    return z, net.to(device), x.to(device), t.to(device), gout.to(device), param_checksum


@pytest.mark.parametrize("path", MLP_FILES, ids=[os.path.basename(f) for f in MLP_FILES])
def test_dropin_modules_initialise_like_the_reference_and_restatement_matches_cpu(path):
    from test_mlp import emulate, heads
    z, net, x, t, gout, checksum = _mlp_case(path, "cpu")
    # same seed + same construction order => the very same parameters as the reference module
    assert abs(checksum(net) - float(z["checksum"])) <= 1e-6 * max(1.0, abs(float(z["checksum"])))
    with torch.no_grad():
        y = torch.cat(heads(net, emulate(net, x, t)), -1)
    assert util.rel_err(y, z["y"]) < 3e-2          # bf16 operands vs the fp32 reference


@pytest.mark.parametrize("path", MLP_FILES, ids=[os.path.basename(f) for f in MLP_FILES])
def test_fp32_network_restatement_matches_reference_golden_cpu(path):
    """tests/ref_time_utils.py (the reference networks where oracle/_ref is not built) reproduces the reference's
    stored fp32 outputs and gradients."""
    import ref_time_utils
    z, mine, x, t, gout, _ = _mlp_case(path, "cpu")
    cls = type(mine).__name__
    net = getattr(ref_time_utils, cls)(is_blender=mine.is_blender)
    net.load_state_dict(mine.state_dict())
    xa = x.clone().requires_grad_(True)
    out = net(xa, t)
    y = torch.cat(out if isinstance(out, tuple) else (out,), -1)
    assert util.rel_l2(y, z["y"]) < 1e-5 and util.rel_err(y, z["y"]) < 1e-4
    (y * gout[:, :y.shape[1]]).sum().backward()
    assert util.rel_l2(xa.grad, z["dx"]) < 1e-4
    for k, p in net.named_parameters():
        key = "g_" + k.replace(".", "__")
        if key in z.files:
            assert util.rel_l2(p.grad, z[key]) < 1e-4, k


def test_numpy_dpsr_oracle_matches_reference_golden_cpu():
    z = np.load(os.path.join(GOLD, "dpsr_g32.npz"))
    phi = dpsr_forward_np(z["V"], z["N"], 32, float(z["sig"]))
    assert util.rel_err(phi, z["phi"]) < 2e-4


@pytest.mark.gpu
@pytest.mark.parametrize("path", MLP_FILES, ids=[os.path.basename(f) for f in MLP_FILES])
def test_cuda_mlp_matches_reference_golden(path):
    z, net, x, t, gout, _ = _mlp_case(path, "cuda")
    xa = x.clone().requires_grad_(True)
    out = net(xa, t)
    y = torch.cat(out if isinstance(out, tuple) else (out,), -1)
    # default precision (bf16x3 forward, bf16 backward) against the reference's fp32 CPU results:
    # outputs <= 1e-4, every gradient <= 3e-2 relative L2 (DESIGN.md "MLP numerics contract")
    assert util.rel_l2(y, z["y"]) < 1e-4 and util.rel_err(y, z["y"]) < 1e-3
    (y * gout[:, :y.shape[1]]).sum().backward()
    assert util.rel_l2(xa.grad, z["dx"]) < 3e-2
    for k, p in net.named_parameters():
        key = "g_" + k.replace(".", "__")
        if key in z.files:
            assert util.rel_l2(p.grad, z[key]) < 3e-2, k


@pytest.mark.gpu
def test_cuda_dpsr_matches_reference_golden():
    from nvdiffrast_utils.dpsr import DPSR
    from test_dpsr import affine_close
    z = np.load(os.path.join(GOLD, "dpsr_g32.npz"))
    V = torch.from_numpy(z["V"]).cuda().requires_grad_(True)
    N = torch.from_numpy(z["N"]).cuda().requires_grad_(True)
    phi = DPSR(res=(32, 32, 32), sig=float(z["sig"]))(V[None], N[None])[0]
    (phi * torch.from_numpy(z["gout"]).cuda()).sum().backward()
    ok, info = affine_close(phi.detach(), z["phi"])
    assert ok, info
    ok, info = affine_close(N.grad, z["dN"], resid_tol=2e-3, scale_tol=1e-2)
    assert ok, ("dN", info)
    ok, info = affine_close(V.grad, z["dV"], resid_tol=2e-3, scale_tol=1e-2)
    assert ok, ("dV", info)


@pytest.mark.parametrize("cls,blender", [("DeformNetwork", True), ("DeformNetworkNormal", True),
                                         ("DeformNetworkNormal", False), ("DeformNetworkNormalSep", True),
                                         ("AppearanceNetwork", True)])
def test_state_dicts_are_interchangeable_with_the_reference_cpu(cls, blender):
    """INTEGRATION.md: reference checkpoints load into the drop-in modules and vice versa (same parameter
    names, shapes and registration order)."""
    ref = util.load_reference_pymodules()
    if ref is None:
        pytest.skip("oracle/_ref/refpy missing")
    tu = importlib.import_module("utils.time_utils")
    torch.manual_seed(3)
    theirs = getattr(ref.time_utils, cls)(is_blender=blender)
    mine = getattr(tu, cls)(is_blender=blender)
    sd_t, sd_m = theirs.state_dict(), mine.state_dict()
    assert list(sd_t.keys()) == list(sd_m.keys())
    assert [tuple(v.shape) for v in sd_t.values()] == [tuple(v.shape) for v in sd_m.values()]
    mine.load_state_dict(sd_t, strict=True)
    theirs.load_state_dict(mine.state_dict(), strict=True)
    for k in sd_t:
        assert torch.equal(mine.state_dict()[k], sd_t[k])
    # constructor surface: unsupported trunk shapes raise; is_6dof has the reference's parameters, in its order
    with pytest.raises(NotImplementedError):
        getattr(tu, "DeformNetwork")(D=4)
    if cls in ("DeformNetwork", "DeformNetworkNormal"):
        torch.manual_seed(3)
        t6 = getattr(ref.time_utils, cls)(is_blender=blender, is_6dof=True)
        torch.manual_seed(3)
        m6 = getattr(tu, cls)(is_blender=blender, is_6dof=True)
        assert list(t6.state_dict().keys()) == list(m6.state_dict().keys())
        for k, v in t6.state_dict().items():
            assert torch.equal(v, m6.state_dict()[k]), k       # same construction order -> same default init
