from .base import (AppliedTransform, IntensityTransform, SpatialTransform, Transform,
                   execution_device, set_execution_device)
from .compose import Compose
from .intensity import BiasField, Blur, Gamma, LabelsToImage, Noise, Normalize, RescaleIntensity, Standardize
from .inverse import apply_inverse_transform, get_inverse_transform
from .neighbours import Crop, CropOrPad, Flip, Pad
from .spatial import Affine, ElasticDeformation, Resample, Spatial

__all__ = [
    "Affine", "AppliedTransform", "BiasField", "Blur", "Compose", "Crop", "CropOrPad", "ElasticDeformation",
    "Flip", "Gamma", "IntensityTransform", "LabelsToImage", "Noise", "Normalize", "Pad", "Resample", "RescaleIntensity", "Spatial",
    "SpatialTransform", "Standardize", "Transform",
    "apply_inverse_transform", "execution_device", "get_inverse_transform",
    "set_execution_device",
]
