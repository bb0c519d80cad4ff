from .base import (AppliedTransform, IntensityTransform, SpatialTransform, Transform,
                   execution_device, set_execution_device)
from .clamp_mask_swap import Clamp, Mask, Swap
from .compose import Compose
from .histogram import HistogramStandardization, compute_histogram_landmarks
from .intensity import (BiasField, Blur, Gamma, LabelsToImage, Noise, Normalize, RescaleIntensity, Standardize,
                        ZNormalization)
from .label import Contour, KeepLargestComponent, OneHot, RemapLabels, RemoveLabels, SequentialLabels
from .inverse import apply_inverse_transform, get_inverse_transform
from .neighbours import Crop, CropOrPad, Flip, Pad
from .orientation import CopyAffine, EnsureShapeMultiple, Reorient, ToReferenceSpace, Transpose
from .resolution import Anisotropy, Resize
from .spatial import Affine, ElasticDeformation, Resample, Spatial
from .ghosting import Ghosting
from .motion import Motion
from .pca import PCA
from .spike import Spike

__all__ = [
    "Affine", "Anisotropy", "AppliedTransform", "BiasField", "Blur", "Clamp", "Compose", "Contour", "CopyAffine", "Crop", "CropOrPad", "ElasticDeformation", "EnsureShapeMultiple",
    "Flip", "Gamma", "Ghosting", "HistogramStandardization", "IntensityTransform", "KeepLargestComponent", "LabelsToImage", "Mask", "Motion", "Noise", "Normalize", "OneHot", "PCA", "Pad", "RemapLabels",
    "RemoveLabels", "Reorient", "Resample", "Resize", "RescaleIntensity", "SequentialLabels", "Spatial",
    "SpatialTransform", "Spike", "Standardize", "Swap", "ToReferenceSpace", "Transform", "Transpose", "ZNormalization",
    "apply_inverse_transform", "compute_histogram_landmarks", "execution_device", "get_inverse_transform",
    "set_execution_device",
]
