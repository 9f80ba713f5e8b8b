"""DPSR parity: numpy oracle vs the reference's own PyTorch code (CPU, pins the oracle), and the
CUDA path vs the reference (forward and autograd gradients) on the GPU.  Where oracle/_ref is not built the
reference is its restatement tests/ref_dpsr.py, pinned here to the reference's stored outputs."""
import os

import numpy as np
import pytest
import torch

import util
from oracle.oracle import dpsr_forward_np


def _points(n, seed, spread=0.18):
    g = torch.Generator().manual_seed(seed)
    V = (0.5 + spread * torch.randn(n, 3, generator=g)).clamp(1e-6, 1 - 1e-6)
    N = torch.nn.functional.normalize(torch.randn(n, 3, generator=g), dim=1) + 0.1 * torch.randn(n, 3, generator=g)
    return V, N


def affine_close(a, b, resid_tol=5e-5, scale_tol=5e-3):
    """a ~= alpha * b + beta with alpha ~ 1.  DPSR normalises the field by |phi[0,0,0] - mean_p phi(p)|, a
    difference of two numbers ~100-1000x larger than itself: the reference's fp32 `torch.mean` over the
    points (dpsr.py:61) alone moves that scale by ~1e-4..1e-3 between runs/devices (measured: a 1e-7
    relative perturbation of the normals changes the reference output by 1.5e-5 at G=32), while this
    implementation accumulates the mean in fp64.  So parity is asserted on the field up to that one noisy
    global scale/shift: the residual after the best affine fit must be at fp32 level."""
    a = torch.as_tensor(a, dtype=torch.float64).reshape(-1).cpu()
    b = torch.as_tensor(b, dtype=torch.float64).reshape(-1).cpu()
    A = torch.stack([b, torch.ones_like(b)], 1)
    sol = torch.linalg.lstsq(A, a[:, None]).solution[:, 0]
    alpha, beta = float(sol[0]), float(sol[1])
    resid = float((a - (alpha * b + beta)).abs().max() / (b.abs().max() + 1e-30))
    return abs(alpha - 1) < scale_tol and resid < resid_tol, (alpha, beta, resid)


ref = util.load_reference_dpsr()


def test_dpsr_restatement_matches_reference_golden_cpu():
    """tests/ref_dpsr.py (the reference's DPSR where oracle/_ref is not built) reproduces the reference's stored
    field and autograd gradients."""
    import ref_dpsr
    z = np.load(os.path.join(os.path.dirname(__file__), "golden", "dpsr_g32.npz"))
    V = torch.from_numpy(z["V"]).requires_grad_(True)
    N = torch.from_numpy(z["N"]).requires_grad_(True)
    phi = ref_dpsr.DPSR(res=(32, 32, 32), sig=float(z["sig"]))(V[None], N[None])[0]
    (phi * torch.from_numpy(z["gout"])).sum().backward()
    assert util.rel_err(phi.detach(), z["phi"]) < 1e-5
    assert util.rel_err(V.grad, z["dV"]) < 1e-5 and util.rel_err(N.grad, z["dN"]) < 1e-5


@pytest.mark.parametrize("G,n,sig", [(16, 300, 2.0), (32, 2000, 3.0)])
def test_oracle_matches_reference_dpsr_cpu(G, n, sig):
    V, N = _points(n, G)
    V[:7] = torch.tensor([0.25, 0.5, 0.75])            # points exactly on grid nodes
    phi_ref = ref.dpsr.DPSR(res=(G, G, G), sig=sig)(V[None], N[None])[0].numpy()
    phi = dpsr_forward_np(V.numpy(), N.numpy(), G, sig)
    assert util.rel_err(phi, phi_ref) < 2e-4


@pytest.mark.gpu
@pytest.mark.parametrize("G,n,sig", [(32, 3000, 3.0), (64, 20000, 3.0), (288, 200_000, 3.0)])
def test_cuda_dpsr_matches_reference(G, n, sig):
    from nvdiffrast_utils.dpsr import DPSR
    V, N = _points(n, G + 1)
    V[:5] = torch.tensor([0.25, 0.5, 0.75])
    gout = torch.randn(G, G, G, generator=torch.Generator().manual_seed(3)).cuda()
    Va, Na = V.cuda().requires_grad_(True), N.cuda().requires_grad_(True)
    phi = DPSR(res=(G, G, G), sig=sig)(Va[None], Na[None])
    assert phi.shape == (1, G, G, G)
    (phi[0] * gout).sum().backward()
    Vb, Nb = V.cuda().requires_grad_(True), N.cuda().requires_grad_(True)
    phi_ref = ref.dpsr.DPSR(res=(G, G, G), sig=sig).cuda()(Vb[None], Nb[None])
    (phi_ref[0] * gout).sum().backward()
    ok, info = affine_close(phi.detach(), phi_ref.detach())
    assert ok, info
    assert util.rel_err(phi, phi_ref) < 5e-3
    ok, info = affine_close(Na.grad, Nb.grad, resid_tol=2e-3, scale_tol=1e-2)
    assert ok, ("dN", info)
    ok, info = affine_close(Va.grad, Vb.grad, resid_tol=2e-3, scale_tol=1e-2)
    assert ok, ("dV", info)


@pytest.mark.gpu
def test_cuda_dpsr_signed_variant_matches_mesh_renderer_glue():
    """forward_signed == psr * sign - thres as utils/renderer.py:163-168 computes it (values + grads)."""
    from nvdiffrast_utils.dpsr import DPSR
    G, n = 48, 8000
    V, N = _points(n, 9)
    gout = torch.randn(G, G, G, generator=torch.Generator().manual_seed(4)).cuda()
    th = torch.tensor(0.02, device="cuda", requires_grad=True)
    Va, Na = V.cuda().requires_grad_(True), N.cuda().requires_grad_(True)
    out = DPSR(res=(G, G, G), sig=3.0).forward_signed(Va[None], Na[None], th)
    (out * gout).sum().backward()
    th2 = torch.tensor(0.02, device="cuda", requires_grad=True)
    Vb, Nb = V.cuda().requires_grad_(True), N.cuda().requires_grad_(True)
    psr = ref.dpsr.DPSR(res=(G, G, G), sig=3.0).cuda()(Vb[None], Nb[None])
    sign = -1 if psr[0, 0, 0, 0].detach() < 0 else 1
    ref_out = (psr * sign - th2).squeeze(0)
    (ref_out * gout).sum().backward()
    assert util.rel_err(out, ref_out) < 1e-4
    assert util.rel_err(Na.grad, Nb.grad) < 1e-3 and util.rel_err(Va.grad, Vb.grad) < 1e-3
    assert abs(float(th.grad) - float(th2.grad)) < 1e-3 * abs(float(th2.grad))


@pytest.mark.gpu
def test_cuda_dpsr_against_numpy_oracle_and_errors():
    from nvdiffrast_utils.dpsr import DPSR
    G, n = 24, 1500
    V, N = _points(n, 5)
    phi = DPSR(res=(G, G, G), sig=2.0)(V.cuda()[None], N.cuda()[None])[0].cpu().numpy()
    assert util.rel_err(phi, dpsr_forward_np(V.numpy(), N.numpy(), G, 2.0)) < 2e-4
    with pytest.raises(NotImplementedError):
        DPSR(res=(32, 32), sig=2.0)
    with pytest.raises(ValueError):
        DPSR(res=(G, G, G), sig=2.0)(V[None], N[None])     # CPU tensors: no fallback
