"""nvdiffrecmc_b200 -- H100-native (sm_90a) replacement for the nvdiffrecmc per-iteration hot path:
environment-light importance sampling + shadow-ray visibility + PBR BSDF (fwd/bwd) + bilateral
denoiser, behind the reference's own `render/optixutils`, `render/renderutils` and `denoiser` APIs.

Sub-packages mirror the reference layout:
    nvdiffrecmc_b200.optixutils   <->  render/optixutils   (OptiXContext, optix_build_bvh, optix_env_shade, bilateral_denoiser)
    nvdiffrecmc_b200.renderutils  <->  render/renderutils  (pbr_bsdf, prepare_shading_normal, ... )
    nvdiffrecmc_b200.denoiser     <->  denoiser/denoiser.py (BilateralDenoiser)
    nvdiffrecmc_b200.light        <->  render/light.py      (EnvironmentLight)
    nvdiffrecmc_b200.dmtet        <->  geometry/dmtet.py    (marching_tets, sdf_reg_loss)
All of them call hand-written CUDA kernels in lib/libmcshade.so through the C ABI in include/mcshade.h.
"""
from . import _lib  # noqa: F401

__all__ = ["optixutils", "renderutils", "denoiser", "light"]
