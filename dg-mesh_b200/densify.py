"""Adaptive density control on the device (SURVEY.md 8(f)-2).

`densify_and_prune(model, max_grad, min_opacity, extent, max_screen_size)` is a drop-in for
GaussianModelDPSRDynamicAnchor.densify_and_prune
(dgmesh/scene/gaussian_model_dpsr_dynamic_anchor.py:540-551) operating on the reference's own model
object: same attributes (`_xyz`, `_features_dc`, ... , `optimizer` with named param groups,
`xyz_gradient_accum`, `denom`, `max_radii2D`, `percent_dense`), same resulting rows in the same order,
same Adam state, same consumption of the CUDA random generator (one torch.normal of shape
[2 * n_split, 3]).  Where the reference runs clone -> split -> prune as three rounds of torch.cat /
boolean masking over 7 parameters x 3 tensors, this makes ONE plan (dgd_plan), reads four counters,
and writes every surviving row once (dgd_apply).

`install(model_class)` replaces the method on the reference class (the launcher does this)."""
import ctypes
import os
import sys

import torch
from torch import nn

_root = os.path.dirname(os.path.abspath(__file__))
if _root not in sys.path:
    sys.path.insert(0, _root)
import _dgm_lib  # noqa: E402

_ROLE = {"xyz": 1, "scaling": 2}
_ATTR = {"xyz": "_xyz", "f_dc": "_features_dc", "f_rest": "_features_rest", "opacity": "_opacity",
         "scaling": "_scaling", "rotation": "_rotation", "normal": "_normal"}


def densify_and_prune(self, max_grad, min_opacity, extent, max_screen_size):
    lib = _dgm_lib.lib()
    xyz = self._xyz
    if not xyz.is_cuda:
        raise ValueError("densify_and_prune : CUDA tensors required (no CPU fallback)")
    P, dev = xyz.shape[0], xyz.device
    if P == 0:
        return
    st = _dgm_lib.stream_ptr()
    nb = _dgm_lib.c_size_t()
    _dgm_lib.check(lib.dgd_workspace_size(P, ctypes.byref(nb)), "dgd_workspace_size")
    ws = torch.empty((nb.value,), dtype=torch.uint8, device=dev)
    counts = torch.empty((4,), dtype=torch.int32, device=dev)
    acc = self.xyz_gradient_accum.detach().contiguous().float().reshape(-1)
    den = self.denom.detach().contiguous().float().reshape(-1)
    scaling = self._scaling.detach().contiguous()
    opacity = self._opacity.detach().contiguous().reshape(-1)
    rotation = self._rotation.detach().contiguous()
    size_prune = bool(max_screen_size)      # the reference's `if max_screen_size:`
    _dgm_lib.check(lib.dgd_plan(P, acc.data_ptr(), den.data_ptr(), scaling.data_ptr(), opacity.data_ptr(),
                                float(max_grad), float(min_opacity), float(extent), float(self.percent_dense),
                                int(size_prune), float(max_screen_size or 0.0), ws.data_ptr(), nb.value,
                                counts.data_ptr(), st), "dgd_plan")
    n_keep, n_clone, n_split, n_child = (int(v) for v in counts.tolist())       # the one host read
    n_out = n_keep + n_clone + 2 * n_child
    # the split samples: same generator call as the reference (:463-465)
    stds = torch.empty((2 * n_split, 3), dtype=torch.float32, device=dev)
    if n_split:
        _dgm_lib.check(lib.dgd_split_stds(P, scaling.data_ptr(), ws.data_ptr(), nb.value, stds.data_ptr(), st),
                       "dgd_split_stds")
    means = torch.zeros((stds.size(0), 3), device=dev)
    samples = torch.normal(mean=means, std=stds)
    # gather every parameter group the reference touches (gaussian_param_list), with its Adam moments
    groups = [g for g in self.optimizer.param_groups if g["name"] in self.gaussian_param_list]
    fields = (_dgm_lib.DgdField * len(groups))()
    keep, new = [], []
    for k, g in enumerate(groups):
        assert len(g["params"]) == 1
        p = g["params"][0]
        src = p.detach().contiguous()
        width = src.numel() // P
        dst = torch.empty((n_out,) + tuple(src.shape[1:]), dtype=torch.float32, device=dev)
        state = self.optimizer.state.get(p, None)
        f = fields[k]
        f.src, f.dst, f.width, f.role = src.data_ptr(), dst.data_ptr(), width, _ROLE.get(g["name"], 0)
        m1d = m2d = None
        if state is not None and "exp_avg" in state:
            m1, m2 = state["exp_avg"].contiguous(), state["exp_avg_sq"].contiguous()
            m1d, m2d = torch.empty_like(dst), torch.empty_like(dst)
            f.m1_src, f.m2_src, f.m1_dst, f.m2_dst = m1.data_ptr(), m2.data_ptr(), m1d.data_ptr(), m2d.data_ptr()
            keep += [m1, m2]
        keep.append(src)
        new.append((g, p, state, dst, m1d, m2d))
    if n_out:
        _dgm_lib.check(lib.dgd_apply(P, len(groups), fields, rotation.data_ptr(), samples.data_ptr(), ws.data_ptr(),
                                     nb.value, st), "dgd_apply")
    # re-seat parameters and optimiser state the way cat_tensors_to_optimizer / _prune_optimizer do
    for g, p, state, dst, m1d, m2d in new:
        newp = nn.Parameter(dst.requires_grad_(True))
        if state is not None:
            if m1d is not None:
                state["exp_avg"], state["exp_avg_sq"] = m1d, m2d
            del self.optimizer.state[p]
            self.optimizer.state[newp] = state
        g["params"][0] = newp
        setattr(self, _ATTR[g["name"]], newp)
    self.xyz_gradient_accum = torch.zeros((n_out, 1), device=dev)
    self.denom = torch.zeros((n_out, 1), device=dev)
    self.max_radii2D = torch.zeros((n_out,), device=dev)


def install(model_class):
    """Replace `densify_and_prune` on a reference Gaussian-model class; returns the original method."""
    orig = model_class.densify_and_prune
    if orig is densify_and_prune:
        return getattr(model_class, "_reference_densify_and_prune", None)
    model_class._reference_densify_and_prune = orig      # kept for parity tests / fallback inspection
    model_class.densify_and_prune = densify_and_prune
    return orig
