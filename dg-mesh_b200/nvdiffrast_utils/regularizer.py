"""Drop-in `nvdiffrast_utils.regularizer` (reference: dgmesh/nvdiffrast_utils/regularizer.py):
`laplace_regularizer_const(v_pos, t_pos_idx)` -- the Laplacian term of the mesh branch
(dgmesh/train.py:277-283) -- as one fused forward (face pass + vertex pass) and one fused backward instead of
the reference's 3 gathers + 6 scatter_adds + elementwise chain and its autograd mirror.  Every other name of
the reference module (image_grad, avg_edge_length, normal_consistency: not used by train.py) resolves to the
reference's own file through the merged `nvdiffrast_utils` package path set up by launch.install()."""
import ctypes
import os
import sys

import torch

_root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if _root not in sys.path:
    sys.path.insert(0, _root)
import _dgm_lib  # noqa: E402


class _Laplacian(torch.autograd.Function):
    @staticmethod
    def forward(ctx, v_pos, tri):
        if not v_pos.is_cuda:
            raise ValueError("laplace_regularizer_const : CUDA tensors required (no CPU fallback)")
        v = v_pos.contiguous().float()
        t = tri.to(torch.int32).contiguous()
        V, F = v.shape[0], t.shape[0]
        nb = _dgm_lib.c_size_t()
        _dgm_lib.check(_dgm_lib.lib().dgl_laplacian_workspace(V, ctypes.byref(nb)), "dgl_laplacian_workspace")
        ws = torch.empty((nb.value,), dtype=torch.uint8, device=v.device)
        out = torch.empty((1,), dtype=torch.float32, device=v.device)
        rc = _dgm_lib.lib().dgl_laplacian_forward(V, F, _dgm_lib.ptr(v), _dgm_lib.ptr(t), out.data_ptr(),
                                                  ws.data_ptr(), nb.value, _dgm_lib.stream_ptr())
        _dgm_lib.check(rc, "dgl_laplacian_forward")
        ctx.save_for_backward(t, ws)
        ctx.V = V
        return out.reshape(())

    @staticmethod
    def backward(ctx, g):
        t, ws = ctx.saved_tensors
        V = ctx.V
        dv = torch.empty((V, 3), dtype=torch.float32, device=ws.device)
        gl = g.reshape(1).contiguous().float()
        rc = _dgm_lib.lib().dgl_laplacian_backward(V, t.shape[0], _dgm_lib.ptr(t), gl.data_ptr(), _dgm_lib.ptr(dv),
                                                   ws.data_ptr(), ws.numel(), _dgm_lib.stream_ptr())
        _dgm_lib.check(rc, "dgl_laplacian_backward")
        return dv, None


def laplace_regularizer_const(v_pos, t_pos_idx):
    return _Laplacian.apply(v_pos, t_pos_idx)


def __getattr__(name):
    import importlib.util
    pkg = sys.modules.get("nvdiffrast_utils")
    here = os.path.dirname(os.path.abspath(__file__))
    for d in list(getattr(pkg, "__path__", [])):
        cand = os.path.join(d, "regularizer.py")
        if os.path.abspath(d) != here and os.path.exists(cand):
            mod = sys.modules.get("_reference_nvdiffrast_utils_regularizer")
            if mod is None:
                spec = importlib.util.spec_from_file_location("nvdiffrast_utils._reference_regularizer", cand)
                mod = importlib.util.module_from_spec(spec)
                sys.modules["_reference_nvdiffrast_utils_regularizer"] = mod
                spec.loader.exec_module(mod)
            if hasattr(mod, name):
                return getattr(mod, name)
    raise AttributeError(f"module 'nvdiffrast_utils.regularizer' has no attribute {name!r}")
