"""Drop-in `utils.loss_utils` (reference: dgmesh/utils/loss_utils.py): l1_loss, l2_loss, kl_divergence,
ssim with the reference's signatures, plus `image_loss(image, gt, lambda_dssim)` = the composition
dgmesh/train.py:308-311 uses, (1 - l) * l1_loss + l * (1 - ssim), as ONE fused forward kernel and ONE
fused backward kernel (csrc/loss.cu) instead of the reference's ~10 depthwise 11x11 conv2d calls and
~30 elementwise kernels.

`ssim(img1, img2)` is differentiable w.r.t. img1 only (the rendered image); the ground truth never
requires grad in the reference.  CUDA tensors only -- no CPU fallback.
"""
import ctypes
import os
import sys

import torch

_root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if _root not in sys.path:
    sys.path.insert(0, _root)
import _dgm_lib  # noqa: E402


def l1_loss(network_output, gt):
    return torch.abs((network_output - gt)).mean()


def l2_loss(network_output, gt):
    return ((network_output - gt) ** 2).mean()


def kl_divergence(rho, rho_hat):
    rho_hat = torch.mean(torch.sigmoid(rho_hat), 0)
    rho = torch.tensor([rho] * len(rho_hat), device=rho_hat.device)
    return torch.mean(rho * torch.log(rho / (rho_hat + 1e-5)) + (1 - rho) * torch.log((1 - rho) / (1 - rho_hat + 1e-5)))


class _ImageLoss(torch.autograd.Function):
    @staticmethod
    def forward(ctx, img, gt, lam, mode):
        if not img.is_cuda or not gt.is_cuda:
            raise ValueError("loss_utils : CUDA tensors required (no CPU fallback)")
        if img.dim() != 3 or img.shape[0] != 3 or img.shape != gt.shape:
            raise ValueError("expected img and gt of shape [3, H, W]")
        x, y = img.detach().contiguous().float(), gt.detach().contiguous().float()
        H, W = int(x.shape[1]), int(x.shape[2])
        lib = _dgm_lib.lib()
        nbytes = _dgm_lib.c_size_t()
        _dgm_lib.check(lib.dgloss_workspace_size(H, W, ctypes.byref(nbytes)), "dgloss_workspace_size")
        ws = torch.empty((nbytes.value,), dtype=torch.uint8, device=x.device)
        out = torch.empty((3,), dtype=torch.float32, device=x.device)
        _dgm_lib.check(lib.dgloss_forward(H, W, x.data_ptr(), y.data_ptr(), float(lam), int(mode), out.data_ptr(),
                                          ws.data_ptr(), nbytes.value, _dgm_lib.stream_ptr()), "dgloss_forward")
        ctx.save_for_backward(x, y, ws)
        ctx.lam, ctx.mode = float(lam), int(mode)
        return out[0].clone(), out[1].clone(), out[2].clone()

    @staticmethod
    def backward(ctx, g_loss, g_l1, g_ssim):
        x, y, ws = ctx.saved_tensors
        H, W = int(x.shape[1]), int(x.shape[2])
        g = g_loss.contiguous().float().reshape(1)
        dimg = torch.empty_like(x)
        _dgm_lib.check(_dgm_lib.lib().dgloss_backward(H, W, x.data_ptr(), y.data_ptr(), ctx.lam, ctx.mode,
                                                      g.data_ptr(), dimg.data_ptr(), ws.data_ptr(), ws.numel(),
                                                      _dgm_lib.stream_ptr()), "dgloss_backward")
        return dimg, None, None, None


def image_loss(image, gt_image, lambda_dssim=0.2, return_parts=False):
    """(1 - lambda) * L1 + lambda * (1 - SSIM) (dgmesh/train.py:308-311).  Only the returned loss carries
    gradient; `l1` and `ssim` (return_parts=True) are detached values for logging."""
    loss, l1, ss = _ImageLoss.apply(image, gt_image, lambda_dssim, 0)
    return (loss, l1.detach(), ss.detach()) if return_parts else loss


def ssim(img1, img2, window_size=11, size_average=True):
    """Mean SSIM of two [3,H,W] images (loss_utils.py:39-76: window 11, sigma 1.5)."""
    if window_size != 11 or not size_average:
        raise NotImplementedError("loss_utils : window_size=11, size_average=True (what train.py uses) only")
    return _ImageLoss.apply(img1, img2, 1.0, 1)[0]
