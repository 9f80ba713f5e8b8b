"""`simple_knn._C.distCUDA2` backed by libdgmesh_b200.so (sm_90a).

Mirrors dgmesh/submodules/simple-knn/spatial.cu:15-26 / ext.cpp:15-17:
    distCUDA2(points: cuda float32 [P,3]) -> cuda float32 [P]
(mean of the squared distances to the 3 nearest neighbours).  No host synchronisation, current stream."""
import os
import sys

import torch

_root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if _root not in sys.path:
    sys.path.insert(0, _root)
import _dgm_lib  # noqa: E402


def distCUDA2(points):
    lib = _dgm_lib.lib()
    if not points.is_cuda:
        raise ValueError("distCUDA2: points must be a CUDA tensor")
    pts = points.contiguous().float()
    P = pts.shape[0]
    means = torch.zeros((P,), dtype=torch.float32, device=pts.device)  # reference: torch::full({P}, 0.0)
    if P == 0:
        return means
    nbytes = _dgm_lib.c_size_t()
    _dgm_lib.check(lib.dgk_workspace_size(P, nbytes), "dgk_workspace_size")
    ws = torch.empty((nbytes.value,), dtype=torch.uint8, device=pts.device)
    _dgm_lib.check(lib.dgk_dist2(P, pts.data_ptr(), means.data_ptr(), ws.data_ptr(), nbytes.value,
                                 _dgm_lib.stream_ptr()), "dgk_dist2")
    return means
