"""Image loss (SURVEY.md 8(f)-3: L1 + SSIM, dgmesh/utils/loss_utils.py:18-76 as composed in
dgmesh/train.py:308-311): the numpy oracle is pinned on the CPU against the reference's own functions and
autograd; the fused CUDA kernels are compared with both on the GPU."""
import importlib.util
import os

import numpy as np
import pytest
import torch

import util
from oracle.oracle import image_loss_np


def _ref_loss_utils():
    """The reference's loss_utils where oracle/_ref is built, else its restatement tests/ref_loss_utils.py (pinned
    to the numpy oracle by test_oracle_matches_reference_loss_and_autograd_cpu)."""
    p = os.path.join(util.REF_DIR, "refpy", "loss_utils.py")
    if os.path.exists(p):
        spec = importlib.util.spec_from_file_location("ref_loss_utils_built", p)
        m = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(m)
        return m
    import ref_loss_utils
    return ref_loss_utils


ref_lu = _ref_loss_utils()


def _images(H, W, seed):
    g = torch.Generator().manual_seed(seed)
    gt = torch.rand(3, H, W, generator=g)
    img = (gt + 0.15 * torch.randn(3, H, W, generator=g)).clamp(0, 1)
    return img, gt


@pytest.mark.parametrize("H,W", [(40, 56), (33, 47), (8, 9)])
def test_oracle_matches_reference_loss_and_autograd_cpu(H, W):
    img, gt = _images(H, W, H * W)
    x = img.clone().requires_grad_(True)
    l1, ss = ref_lu.l1_loss(x, gt), ref_lu.ssim(x, gt)
    loss = (1.0 - 0.2) * l1 + 0.2 * (1.0 - ss)
    loss.backward()
    o_loss, o_l1, o_ss, o_grad = image_loss_np(img.numpy(), gt.numpy(), 0.2)
    assert abs(o_l1 - float(l1)) < 1e-6 and abs(o_ss - float(ss)) < 1e-5 and abs(o_loss - float(loss)) < 1e-5
    assert util.rel_err(o_grad, x.grad) < 1e-4


@pytest.mark.gpu
@pytest.mark.parametrize("H,W", [(800, 800), (67, 45), (16, 16), (1080, 1920)])
def test_cuda_image_loss_matches_reference(H, W):
    import importlib
    lu = importlib.import_module("utils.loss_utils")
    img, gt = _images(H, W, H + W)
    img, gt = img.cuda(), gt.cuda()
    xa = img.clone().requires_grad_(True)
    loss, l1, ss = lu.image_loss(xa, gt, 0.2, return_parts=True)
    (3.0 * loss).backward()
    xb = img.clone().requires_grad_(True)
    rl1, rss = ref_lu.l1_loss(xb, gt), ref_lu.ssim(xb, gt)
    rloss = (1.0 - 0.2) * rl1 + 0.2 * (1.0 - rss)
    (3.0 * rloss).backward()
    assert abs(float(loss) - float(rloss)) < 1e-5 and abs(float(l1) - float(rl1)) < 1e-6
    assert abs(float(ss) - float(rss)) < 1e-5
    assert util.rel_err(xa.grad, xb.grad) < 1e-4
    # the stand-alone ssim() drop-in
    xc = img.clone().requires_grad_(True)
    s = lu.ssim(xc, gt)
    s.backward()
    xd = img.clone().requires_grad_(True)
    ref_lu.ssim(xd, gt).backward()
    assert abs(float(s) - float(rss)) < 1e-5 and util.rel_err(xc.grad, xd.grad) < 1e-4


@pytest.mark.gpu
def test_cuda_image_loss_against_numpy_oracle_and_errors():
    import importlib
    lu = importlib.import_module("utils.loss_utils")
    img, gt = _images(50, 70, 9)
    xa = img.cuda().requires_grad_(True)
    loss = lu.image_loss(xa, gt.cuda(), 0.2)
    loss.backward()
    o_loss, _, _, o_grad = image_loss_np(img.numpy(), gt.numpy(), 0.2)
    assert abs(float(loss) - o_loss) < 1e-5 and util.rel_err(xa.grad, o_grad) < 1e-4
    with pytest.raises(ValueError):
        lu.image_loss(img, gt)                       # CPU tensors: no fallback
    with pytest.raises(NotImplementedError):
        lu.ssim(xa, gt.cuda(), window_size=7)


@pytest.mark.gpu
@pytest.mark.parametrize("sub", [2, 5])
def test_cuda_laplacian_regulariser_matches_reference(sub):
    """nvdiffrast_utils.regularizer.laplace_regularizer_const (regularizer.py:40-59): fused forward / backward
    against the reference's own function (imported unmodified from oracle/_ref/dgmesh; where that is not built,
    its restatement in tests/ref_loss_utils.py) and its autograd."""
    import importlib.util
    import os
    import sys
    ref_file = os.path.join(util.ROOT, "oracle", "_ref", "dgmesh", "nvdiffrast_utils", "regularizer.py")
    built = os.path.exists(ref_file)
    if built:
        sys.path.insert(0, os.path.join(util.ROOT, "tools"))
        import harness_stubs
        harness_stubs.install()
        import launch
        launch.install(os.path.join(util.ROOT, "oracle", "_ref", "dgmesh"))
        spec = importlib.util.spec_from_file_location("nvdiffrast_utils._ref_regularizer_for_test", ref_file)
        refmod = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(refmod)
    else:
        import ref_loss_utils as refmod
    mine = importlib.import_module("nvdiffrast_utils.regularizer")
    assert mine.__file__.startswith(os.path.join(util.ROOT, "dg-mesh_b200"))
    from test_meshrast import icosphere
    v, f = icosphere(sub, 0.7)
    g = torch.Generator().manual_seed(sub)
    v = (v + 0.02 * torch.randn(v.shape, generator=g)).cuda()
    f = f.cuda()
    va, vb = v.clone().requires_grad_(True), v.clone().requires_grad_(True)
    la = mine.laplace_regularizer_const(va, f.long())
    lb = refmod.laplace_regularizer_const(vb, f.long())
    assert abs(float(la) - float(lb)) < 1e-6 * max(1.0, abs(float(lb))) and la.shape == lb.shape
    (la * 3.0).backward()
    (lb * 3.0).backward()
    assert util.rel_err(va.grad, vb.grad) < 1e-5
    if built:
        assert callable(mine.avg_edge_length)    # names this drop-in does not define fall through to the reference
