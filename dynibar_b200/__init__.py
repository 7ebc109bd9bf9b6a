"""dynibar_b200: CUDA-native DynIBaR per-ray volumetric IBR hot path for the H100.

Python/PyTorch host code over a C-ABI shared library of hand-written sm_90a
kernels (`dynibar_b200/csrc`, declared in `include/dynibar_b200.h`).  The
public surface mirrors the reference's: `render_ray.render_rays_mv`,
`render_ray.render_rays_mono`, `projection.Projector`,
`sample_ray.RaySamplerSingleImage`.
"""

__version__ = "0.1.0"
