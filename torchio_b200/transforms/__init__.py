from .base import (AppliedTransform, IntensityTransform, SpatialTransform, Transform,
                   execution_device, set_execution_device)
from .compose import Compose
from .intensity import BiasField, Blur, Gamma, LabelsToImage, Noise, Normalize, RescaleIntensity, Standardize
from .label import Contour, OneHot, RemapLabels, RemoveLabels, SequentialLabels
from .inverse import apply_inverse_transform, get_inverse_transform
from .neighbours import Crop, CropOrPad, Flip, Pad
from .resolution import Anisotropy, Resize
from .spatial import Affine, ElasticDeformation, Resample, Spatial

__all__ = [
    "Affine", "Anisotropy", "AppliedTransform", "BiasField", "Blur", "Compose", "Contour", "Crop", "CropOrPad", "ElasticDeformation",
    "Flip", "Gamma", "IntensityTransform", "LabelsToImage", "Noise", "Normalize", "OneHot", "Pad", "RemapLabels",
    "RemoveLabels", "Resample", "Resize", "RescaleIntensity", "SequentialLabels", "Spatial",
    "SpatialTransform", "Standardize", "Transform",
    "apply_inverse_transform", "execution_device", "get_inverse_transform",
    "set_execution_device",
]
