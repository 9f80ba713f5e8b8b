"""`nvdiffrast.torch` surface used by dgmesh/utils/renderer.py:33-121 and dgmesh/train.py:71,
implemented by meshrast.py (sm_90a kernels behind the C-ABI)."""
from meshrast import (RasterizeContext, RasterizeCudaContext, RasterizeGLContext, antialias,  # noqa: F401
                      edge_opposites, interpolate, rasterize)
