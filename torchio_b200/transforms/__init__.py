from .base import (AppliedTransform, IntensityTransform, SpatialTransform, Transform,
                   execution_device, set_execution_device)
from .compose import Compose
from .histogram import HistogramStandardization, compute_histogram_landmarks
from .intensity import (BiasField, Blur, Gamma, LabelsToImage, Noise, Normalize, RescaleIntensity, Standardize,
                        ZNormalization)
from .label import Contour, OneHot, RemapLabels, RemoveLabels, SequentialLabels
from .inverse import apply_inverse_transform, get_inverse_transform
from .neighbours import Crop, CropOrPad, Flip, Pad
from .resolution import Anisotropy, Resize
from .spatial import Affine, ElasticDeformation, Resample, Spatial

__all__ = [
    "Affine", "Anisotropy", "AppliedTransform", "BiasField", "Blur", "Compose", "Contour", "Crop", "CropOrPad", "ElasticDeformation",
    "Flip", "Gamma", "HistogramStandardization", "IntensityTransform", "LabelsToImage", "Noise", "Normalize", "OneHot", "Pad", "RemapLabels",
    "RemoveLabels", "Resample", "Resize", "RescaleIntensity", "SequentialLabels", "Spatial",
    "SpatialTransform", "Standardize", "Transform", "ZNormalization",
    "apply_inverse_transform", "compute_histogram_landmarks", "execution_device", "get_inverse_transform",
    "set_execution_device",
]
