"""Frame-batched mesh branch, host side (no GPU needed): every batch entry point of DPSR, marching cubes and the
range-mode mesh rasteriser refuses a batch size outside [1, 64], a NULL pointer and a range past the triangles
before anything touches a device, and the Python layers refuse malformed ranges, mismatched per-frame deltas and
mixed camera resolutions with ValueError."""
import importlib
from types import SimpleNamespace

import numpy as np
import pytest
import torch

D = 1 << 20   # a dummy address: must never be dereferenced


def _lib():
    import _dgm_lib
    return _dgm_lib.lib()


def _err(lib, rc, *words):
    msg = lib.dgm_last_error()
    assert rc == -1, (rc, msg)
    for w in words:
        assert w in msg, (w, msg)


def test_dpsr_batch_argument_errors():
    lib = _lib()
    n = __import__("_dgm_lib").c_size_t()
    for B in (0, 65):
        _err(lib, lib.dgp_batch_workspace_size(D, B, n), b"dgp_batch_workspace_size", b"B out of range")
        _err(lib, lib.dgp_forward_batch(D, B, 10, 2.0, D, D, 0, None, D, D, 1 << 40, None), b"dgp_forward_batch",
             b"B out of range")
        _err(lib, lib.dgp_backward_batch(D, B, 10, D, D, 0, D, D, D, None, D, 1 << 40, None), b"dgp_backward_batch",
             b"B out of range")
    _err(lib, lib.dgp_batch_workspace_size(None, 2, n), b"null")
    _err(lib, lib.dgp_forward_batch(None, 2, 10, 2.0, D, D, 0, None, D, D, 1 << 40, None), b"null")
    _err(lib, lib.dgp_forward_batch(D, 2, 10, 2.0, D, D, 0, None, D, None, 1 << 40, None), b"null")
    _err(lib, lib.dgp_backward_batch(D, 2, 10, D, D, 0, D, D, D, None, None, 1 << 40, None), b"null")


def test_marching_cubes_batch_argument_errors():
    import _dgm_lib
    lib = _lib()
    n = _dgm_lib.c_size_t()
    one, two = _dgm_lib.c_size_t(), _dgm_lib.c_size_t()
    assert lib.dgmc_workspace_size(32, one) == 0 and lib.dgmc_workspace_size_batch(1, 32, two) == 0
    assert one.value == two.value                     # B = 1 is the single-grid workspace
    prev = one.value
    for B in (2, 4, 64):
        assert lib.dgmc_workspace_size_batch(B, 32, n) == 0 and n.value > prev
        prev = n.value
    for B in (0, 65):
        _err(lib, lib.dgmc_workspace_size_batch(B, 32, n), b"B out of range")
        _err(lib, lib.dgmc_count_batch(B, 32, D, 0.0, D, 1 << 40, D, None, None, None), b"dgmc_count_batch",
             b"B out of range")
        _err(lib, lib.dgmc_emit_batch(B, 32, D, 0.0, D, 1 << 40, D, D, 16, D, 16, None), b"dgmc_emit_batch",
             b"B out of range")
        _err(lib, lib.dgmc_backward_batch(B, 32, (_dgm_lib.c_int32 * 65)(), D, 0.0, D, D, D, None),
             b"dgmc_backward_batch", b"B out of range")
    _err(lib, lib.dgmc_count_batch(2, 32, None, 0.0, D, 1 << 40, D, None, None, None), b"dgmc_count_batch")
    _err(lib, lib.dgmc_count_batch(2, 32, D, 0.0, D, 1 << 40, None, None, None, None), b"null totals")
    _err(lib, lib.dgmc_emit_batch(2, 32, D, 0.0, D, 1 << 40, D, None, 16, D, 16, None), b"null output")
    _err(lib, lib.dgmc_emit_batch(2, 32, D, 0.0, D, 1 << 40, D, D, (1 << 29) + 1, D, 16, None), b"capacity")
    _err(lib, lib.dgmc_backward_batch(2, 32, None, D, 0.0, D, D, D, None), b"dgmc_backward_batch")
    counts = (_dgm_lib.c_int32 * 2)(5, 7)
    _err(lib, lib.dgmc_backward_batch(2, 32, counts, D, 0.0, None, D, D, None), b"null vsrc")
    G = 8
    edges = 3 * G * G * (G - 1)
    _err(lib, lib.dgmc_backward_batch(2, G, (_dgm_lib.c_int32 * 2)(5, edges + 1), D, 0.0, D, D, D, None),
         b"V out of range")
    # the whole batch shares the 29-bit vertex packing
    big = (_dgm_lib.c_int32 * 2)(1 << 28, (1 << 28) + 1)
    _err(lib, lib.dgmc_backward_batch(2, 800, big, D, 0.0, D, D, D, None), b"V out of range")


def test_meshrast_batch_argument_errors():
    import _dgm_lib
    lib = _lib()
    ranges = (_dgm_lib.c_int32 * 130)()
    for B in (0, 65):
        _err(lib, lib.dgmr_rasterize_batch(3, 4, B, ranges, 8, 8, D, D, D, D, None), b"B out of range")
        _err(lib, lib.dgmr_rasterize_bwd_batch(B, 8, 8, D, D, D, D, D, None), b"dgmr_rasterize_bwd_batch")
        _err(lib, lib.dgmr_interpolate_batch(B, 8, 8, 3, D, D, D, D, None), b"dgmr_interpolate_batch")
        _err(lib, lib.dgmr_interpolate_bwd_batch(B, 8, 8, 3, D, D, D, D, D, D, None), b"dgmr_interpolate_bwd_batch")
        _err(lib, lib.dgmr_antialias_batch(B, 8, 8, 3, D, D, D, D, D, D, None), b"dgmr_antialias_batch")
        _err(lib, lib.dgmr_antialias_bwd_batch(B, 8, 8, 3, D, D, D, D, D, D, D, D, None), b"dgmr_antialias_bwd_batch")
    _err(lib, lib.dgmr_rasterize_batch(3, 4, 2, None, 8, 8, D, D, D, D, None), b"null ranges")
    for r in ((0, 4, 3, 2), (-1, 2, 0, 0), (0, -1, 0, 0), (0, 5, 0, 0)):   # past F = 4, negative first / count
        _err(lib, lib.dgmr_rasterize_batch(3, 4, 2, (_dgm_lib.c_int32 * 4)(*r), 8, 8, D, D, D, D, None),
             b"runs past F")
    # rast.w holds triangle ids up to 2^29 (nvdiffrast's encoding past 2^24): more triangles are refused
    big = (1 << 29) + 1
    _err(lib, lib.dgmr_rasterize(3, big, 8, 8, D, D, D, D, None), b"2^29")
    _err(lib, lib.dgmr_rasterize_batch(3, big, 1, (_dgm_lib.c_int32 * 2)(0, 2), 8, 8, D, D, D, D, None), b"2^29")
    ok = (_dgm_lib.c_int32 * 4)(0, 2, 2, 2)
    _err(lib, lib.dgmr_rasterize_batch(3, 4, 2, ok, 8, 8, D, D, None, D, None), b"bad argument")
    _err(lib, lib.dgmr_interpolate_batch(2, 8, 8, 3, None, D, D, D, None), b"bad argument")
    _err(lib, lib.dgmr_antialias_batch(2, 8, 8, 3, D, D, D, D, None, D, None), b"bad argument")


def test_range_mode_python_argument_errors():
    import meshrast
    pos, tri = torch.zeros(6, 4), torch.tensor([[0, 1, 2], [3, 4, 5]], dtype=torch.int32)
    bad = (torch.tensor([[0, 1]], dtype=torch.int64),            # not int32
           torch.tensor([0, 1], dtype=torch.int32),              # not [B,2]
           torch.zeros((1, 3), dtype=torch.int32),
           torch.zeros((65, 2), dtype=torch.int32),              # more than 64 images
           torch.tensor([[0, 1], [1, 2]], dtype=torch.int32),    # runs past tri
           torch.tensor([[-1, 1]], dtype=torch.int32),
           [[0, 1]])
    for r in bad:
        with pytest.raises(ValueError):
            meshrast.rasterize(None, pos, tri, [8, 8], ranges=r)
    with pytest.raises(ValueError):                              # range mode takes pos [V,4]
        meshrast.rasterize(None, pos[None], tri, [8, 8], ranges=torch.tensor([[0, 1]], dtype=torch.int32))
    with pytest.raises(ValueError):                              # instanced mode is not supported
        meshrast.rasterize(None, torch.zeros(2, 6, 4), tri, [8, 8])
    with pytest.raises(ValueError):
        meshrast.interpolate(torch.zeros(2, 6, 3), torch.zeros(2, 8, 8, 4), tri)
    with pytest.raises(ValueError):
        meshrast.antialias(torch.zeros(2, 8, 8, 3), torch.zeros(2, 8, 8, 4), torch.zeros(2, 6, 4), tri)
    with pytest.raises(ValueError):                              # color and rast cover different images
        meshrast.antialias(torch.zeros(2, 8, 8, 3), torch.zeros(3, 8, 8, 4), pos, tri)


def _cam(H, W):
    return SimpleNamespace(K=np.array([[W, 0, W / 2], [0, H, H / 2], [0, 0, 1]], dtype=np.float32),
                           orig_transform=np.eye(4, dtype=np.float32), image_height=H, image_width=W,
                           FoVx=1.0, FoVy=1.0)


def test_branch_python_argument_errors():
    renderer = importlib.import_module("utils.renderer")
    n = 16
    gauss = SimpleNamespace(get_xyz=torch.zeros(n, 3), get_normal=torch.zeros(n, 3))
    with pytest.raises(ValueError):                              # 3 frames of d_xyz, 2 of d_normal
        renderer.extract_mesh_batch(gauss, torch.zeros(3, n, 3), torch.zeros(2, n, 3))
    with pytest.raises(ValueError):
        renderer.extract_mesh_batch(gauss, [0.0, 0.0], torch.zeros(3, n, 3))
    with pytest.raises(ValueError):
        renderer.extract_mesh_batch(gauss, torch.zeros(3, n, 3), 0.0, frames=2)
    fids = torch.tensor([[0.1], [0.2]])
    with pytest.raises(ValueError):                              # mixed camera resolutions
        renderer.mesh_renderer_batch(None, gauss, 0.0, 0.0, fids, None, None, viewpoint_cams=[_cam(8, 8), _cam(8, 6)])
    with pytest.raises(ValueError):                              # one camera per frame
        renderer.mesh_renderer_batch(None, gauss, 0.0, 0.0, fids, None, None, viewpoint_cams=[_cam(8, 8)])
    with pytest.raises(ValueError):                              # deltas for 3 frames, 2 times
        renderer.mesh_renderer_batch(None, gauss, torch.zeros(3, n, 3), 0.0, fids, None, None)
