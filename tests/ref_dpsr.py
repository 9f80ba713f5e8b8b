"""PyTorch restatement of the reference's DPSR (DG-Mesh dgmesh/nvdiffrast_utils/dpsr.py:28-70 with the helpers of
dpsr_utils.py: point_rasterize, fftfreqs, spec_gaussian_filter, grid_interp), batch 1, differentiable w.r.t. the
points and normals -- the stand-in for `refpy.dpsr` where oracle/_ref has not been built.  Same algorithm as the
numpy oracle (oracle/oracle.py: dpsr_forward_np); tests/test_dpsr.py pins it to the reference's stored field and
gradients (tests/golden/dpsr_g32.npz)."""
import math

import torch


class DPSR(torch.nn.Module):
    def __init__(self, res, sig=10, scale=True, shift=True):
        super().__init__()
        self.G, self.sig = res[0], sig

    def forward(self, V, N):
        G = self.G
        V, N = V[0], N[0]
        cs = 1.0 / G
        t = V.detach() / cs
        fl, ce = torch.floor(t), torch.ceil(t)
        i0, i1 = fl.long(), (ce.long() % G)
        w0 = (V - (fl + 1) * cs).abs() / cs      # weight of node i0: distance to the opposite corner
        w1 = (V - fl * cs).abs() / cs
        corners = []
        for a in (0, 1):
            for b in (0, 1):
                for c in (0, 1):
                    ix, iy, iz = (i1 if a else i0)[:, 0], (i1 if b else i0)[:, 1], (i1 if c else i0)[:, 2]
                    w = (w1 if a else w0)[:, 0] * (w1 if b else w0)[:, 1] * (w1 if c else w0)[:, 2]
                    corners.append(((ix * G + iy) * G + iz, w))
        ras = torch.zeros(3, G * G * G, dtype=V.dtype, device=V.device)
        for idx, w in corners:
            ras = ras.index_add(1, idx, (w[:, None] * N).t())
        ras_s = torch.fft.rfftn(ras.view(3, G, G, G), dim=(1, 2, 3))
        fx = torch.fft.fftfreq(G, d=1 / G, device=V.device)
        fz = torch.fft.rfftfreq(G, d=1 / G, device=V.device)
        om = torch.stack(torch.meshgrid(fx, fx, fz, indexing="ij"), -1)
        dis = torch.sqrt((om ** 2).sum(-1))
        filt = torch.exp(-0.5 * ((self.sig * 2 * dis / G) ** 2))
        omega = om * (2 * math.pi)
        Nf = ras_s * filt[None]
        div = sum((-1j * omega[..., c]) * Nf[c] for c in range(3))
        lap = -(omega ** 2).sum(-1)
        Phi = div / (lap + 1e-6)
        keep = torch.ones_like(lap)
        keep[0, 0, 0] = 0
        phi = torch.fft.irfftn(Phi * keep, s=(G, G, G), dim=(0, 1, 2))
        flat = phi.reshape(-1)
        fv = sum(flat[idx] * w for idx, w in corners)
        phi = phi - fv.mean()
        return (-phi / phi[0, 0, 0].abs() * 0.5)[None]
