"""fp32 PyTorch restatement of the reference's deformation / appearance networks (DG-Mesh
dgmesh/utils/time_utils.py), the stand-in for `refpy.time_utils` where oracle/_ref/refpy has not been built.

The classes are the drop-in modules (same parameters, names, construction order and heads, so state dicts move
between the two freely) with the CUDA chain replaced by the reference's fp32 graph: positional encodings
[v, sin(2^k v), cos(2^k v)], the time-net (is_blender), 8 x (Linear + ReLU) with [x_emb, t_emb] concatenated in
front of the activation after layer 4, linear heads (sigmoid for the colour head).
tests/test_golden_py.py pins these modules to the reference's stored outputs and gradients."""
import importlib

import torch

tu = importlib.import_module("utils.time_utils")


def _pe(v, L):
    out = [v]
    for k in range(L):
        out += [torch.sin(v * 2.0 ** k), torch.cos(v * 2.0 ** k)]
    return torch.cat(out, -1)


class _Fp32:
    def _run(self, x, t):
        x_emb = _pe(x, 10)
        t_emb = _pe(t, self.t_multires)
        if self.is_blender:
            t_emb = self.timenet(t_emb)
        h = torch.cat([x_emb, t_emb], -1)
        for i, l in enumerate(self.linear):
            h = torch.relu(l(h))
            if i in self.skips:
                h = torch.cat([x_emb, t_emb, h], -1)
        ps = self._head_params()
        cols = []
        for w, b in zip(ps[0::2], ps[1::2]):
            y = torch.nn.functional.linear(h, w, b)
            cols.append(torch.sigmoid(y) if self.SIGMOID else y)
        return cols


class DeformNetwork(_Fp32, tu.DeformNetwork):
    pass


class DeformNetworkNormal(_Fp32, tu.DeformNetworkNormal):
    pass


class DeformNetworkNormalSep(_Fp32, tu.DeformNetworkNormalSep):
    pass


class AppearanceNetwork(_Fp32, tu.AppearanceNetwork):
    pass
