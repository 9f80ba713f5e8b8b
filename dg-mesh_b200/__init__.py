"""dgmesh_b200 -- H100-native (sm_90a) implementation of DG-Mesh's per-iteration hot path.

The package holds the CUDA kernels + C-ABI (`csrc/`, `libdgmesh_b200.so`) and the
host-side mirrors of the reference's Python surface for this path:

    diff_gaussian_rasterization   (GaussianRasterizationSettings, GaussianRasterizer)
    simple_knn._C                 (distCUDA2)
    gaussian_renderer             (render)

Put this directory on PYTHONPATH to use them as drop-ins for the reference's
submodules (see INTEGRATION.md).  There is no CPU fallback: every op raises if the
CUDA library is missing.
"""
__version__ = "0.1"
