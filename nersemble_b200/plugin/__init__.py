"""Host-side mirror of the reference's nerfstudio plugin surface for the render hot path.

Same class names, constructor/forward signatures, config dataclasses, output keys and
state_dict keys as /root/reference/src/nersemble/nerfstudio/** (cited per class), with all
arithmetic behind libnsb (CUDA, sm_90a).  NeRSembleNGPModel.get_outputs is differentiable
(fused forward + backward kernels); the stand-alone component modules are forward-only and
raise when called with autograd enabled instead of silently returning graph-less tensors.
"""
from .components import (HashEnsemble, HashEnsembleConfig, SE3DeformationField, SE3DeformationFieldConfig,
                         TCNNHashEncodingConfig, GenericScheduler)
from .field import NeRSembleNeRFactoField
from .sampler import NeRSembleVolumetricSampler, OccGridEstimator
from .model import NeRSembleNGPModel, NeRSembleNGPModelConfig, BaseModelConfig
from .occupancy_filter import filter_occupancy_grid
from .datamanager import DeviceImageCache, DeviceRaySampler, ray_batch

__all__ = ["HashEnsemble", "HashEnsembleConfig", "SE3DeformationField", "SE3DeformationFieldConfig",
           "TCNNHashEncodingConfig", "GenericScheduler", "NeRSembleNeRFactoField", "NeRSembleVolumetricSampler",
           "OccGridEstimator", "NeRSembleNGPModel", "NeRSembleNGPModelConfig", "BaseModelConfig", "filter_occupancy_grid",
           "DeviceImageCache", "DeviceRaySampler", "ray_batch"]
