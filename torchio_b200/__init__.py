"""torchio_b200 — CUDA-native 3-D augmentation hot path behind the TorchIO v2 API.

Drop-in for the reference's spatial + intensity augmentation chain
(`Affine`, `ElasticDeformation`, `Spatial`, `LabelsToImage`, `BiasField`, `Blur`,
`Noise`, `Gamma`, `Compose`), the label-map utilities (`RemapLabels`, `RemoveLabels`,
`SequentialLabels`, `OneHot`, `Contour`, `KeepLargestComponent`), the resolution changes (`Anisotropy`,
`Resize`), histogram standardization (`HistogramStandardization`,
`ZNormalization`), `Clamp`, `Mask`, `Swap`, `Spike`, `Ghosting`, `Motion`, `PCA`, the orientation and shape
utilities (`Reorient`, `Transpose`, `EnsureShapeMultiple`, `CopyAffine`, `ToReferenceSpace`) and its patch path (`UniformSampler`, `Queue`,
`SubjectsLoader`, `GridSampler`, `PatchAggregator`) on tensor-backed `Subject` / `SubjectsBatch` data.  The
tensor math runs in hand-written sm_90a (H100) CUDA kernels exposed through the C-ABI
of ``include/tio_b200.h``; see DESIGN.md and INTEGRATION.md.
"""

from .data import (AffineMatrix, Image, ImagesBatch, LabelMap, ScalarImage, StudiesBatch,
                   Subject, SubjectsBatch)
from .ops import differentiable_default, exact_coords_default, set_differentiable, set_exact_coords
from .params import Choice
from .patches import (GridSampler, ImagesLoader, LabelSampler, PatchAggregator, PatchLocation, PatchSampler, Queue,
                      StudiesLoader, SubjectsLoader, UniformSampler, WeightedSampler, collate_images, collate_studies,
                      collate_subjects)
from .transforms import (Affine, Anisotropy, AppliedTransform, BiasField, Blur, Clamp, Compose, Contour, CopyAffine, Crop, CropOrPad,
                         ElasticDeformation, EnsureShapeMultiple, Flip, Gamma, Ghosting, HistogramStandardization, IntensityTransform, KeepLargestComponent, LabelsToImage, Mask, Motion, Noise, Normalize, OneHot, PCA, Pad,
                         RemapLabels, RemoveLabels, Reorient, Resample, RescaleIntensity, Resize, SequentialLabels, Spatial,
                         SpatialTransform, Spike, Swap, Standardize, ToReferenceSpace, Transform, Transpose, ZNormalization,
                         apply_inverse_transform, execution_device, get_inverse_transform,
                         set_execution_device)

__version__ = "0.1.0"

__all__ = [
    "Affine", "AffineMatrix", "Anisotropy", "AppliedTransform", "BiasField", "Blur", "Choice", "Clamp", "Compose", "Contour", "CopyAffine", "Crop", "CropOrPad",
    "ElasticDeformation", "EnsureShapeMultiple", "Flip", "Gamma", "Ghosting", "GridSampler", "HistogramStandardization", "Image", "ImagesBatch", "ImagesLoader", "IntensityTransform",
    "KeepLargestComponent",     "LabelMap", "LabelSampler", "LabelsToImage", "Mask", "Motion", "Noise", "Normalize", "OneHot", "Pad", "PatchAggregator", "PCA", "PatchLocation", "PatchSampler", "Queue", "RemapLabels", "RemoveLabels",
    "Reorient", "Resample", "RescaleIntensity", "Resize", "ScalarImage", "SequentialLabels", "Spatial",
    "SpatialTransform", "Spike", "Standardize", "StudiesBatch", "StudiesLoader", "Subject", "SubjectsBatch",
    "SubjectsLoader", "Swap", "ToReferenceSpace", "Transform", "Transpose", "UniformSampler", "WeightedSampler", "ZNormalization", "apply_inverse_transform", "collate_images",
    "collate_studies", "collate_subjects", "differentiable_default", "exact_coords_default", "execution_device", "get_inverse_transform",
    "set_differentiable", "set_exact_coords", "set_execution_device",
]
