"""PyTorch restatement of the reference's image losses (DG-Mesh dgmesh/utils/loss_utils.py: l1_loss, ssim) and of
its Laplacian regulariser (dgmesh/nvdiffrast_utils/regularizer.py: laplace_regularizer_const), the stand-ins for
the reference's files where oracle/_ref has not been built.  tests/test_loss.py pins the losses to the numpy
oracle (oracle/oracle.py: image_loss_np)."""
from math import exp

import torch
import torch.nn.functional as F


def l1_loss(network_output, gt):
    return torch.abs(network_output - gt).mean()


def _gaussian(window_size, sigma):
    g = torch.tensor([exp(-(x - window_size // 2) ** 2 / float(2 * sigma ** 2)) for x in range(window_size)])
    return g / g.sum()


def _window(window_size, channel):
    w1 = _gaussian(window_size, 1.5).unsqueeze(1)
    w2 = w1.mm(w1.t()).float().unsqueeze(0).unsqueeze(0)
    return w2.expand(channel, 1, window_size, window_size).contiguous()


def ssim(img1, img2, window_size=11, size_average=True):
    channel = img1.size(-3)
    window = _window(window_size, channel).to(img1.device).type_as(img1)
    pad = window_size // 2
    mu1 = F.conv2d(img1, window, padding=pad, groups=channel)
    mu2 = F.conv2d(img2, window, padding=pad, groups=channel)
    mu1_sq, mu2_sq, mu1_mu2 = mu1.pow(2), mu2.pow(2), mu1 * mu2
    sigma1_sq = F.conv2d(img1 * img1, window, padding=pad, groups=channel) - mu1_sq
    sigma2_sq = F.conv2d(img2 * img2, window, padding=pad, groups=channel) - mu2_sq
    sigma12 = F.conv2d(img1 * img2, window, padding=pad, groups=channel) - mu1_mu2
    C1, C2 = 0.01 ** 2, 0.03 ** 2
    ssim_map = ((2 * mu1_mu2 + C1) * (2 * sigma12 + C2)) / ((mu1_sq + mu2_sq + C1) * (sigma1_sq + sigma2_sq + C2))
    return ssim_map.mean() if size_average else ssim_map.mean(1).mean(1).mean(1)


def laplace_regularizer_const(v_pos, t_pos_idx):
    term = torch.zeros_like(v_pos)
    norm = torch.zeros_like(v_pos[..., 0:1])
    v0, v1, v2 = v_pos[t_pos_idx[:, 0], :], v_pos[t_pos_idx[:, 1], :], v_pos[t_pos_idx[:, 2], :]
    term.scatter_add_(0, t_pos_idx[:, 0:1].repeat(1, 3), (v1 - v0) + (v2 - v0))
    term.scatter_add_(0, t_pos_idx[:, 1:2].repeat(1, 3), (v0 - v1) + (v2 - v1))
    term.scatter_add_(0, t_pos_idx[:, 2:3].repeat(1, 3), (v0 - v2) + (v1 - v2))
    two = torch.ones_like(v0) * 2.0
    norm.scatter_add_(0, t_pos_idx[:, 0:1], two)
    norm.scatter_add_(0, t_pos_idx[:, 1:2], two)
    norm.scatter_add_(0, t_pos_idx[:, 2:3], two)
    term = term / torch.clamp(norm, min=1.0)
    return torch.mean(term ** 2)
