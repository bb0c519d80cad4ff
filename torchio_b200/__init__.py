"""torchio_b200 — CUDA-native 3-D augmentation hot path behind the TorchIO v2 API.

Drop-in for the reference's spatial + intensity augmentation chain
(`Affine`, `ElasticDeformation`, `Spatial`, `LabelsToImage`, `BiasField`, `Blur`,
`Noise`, `Gamma`, `Compose`), the label-map utilities (`RemapLabels`, `RemoveLabels`,
`SequentialLabels`, `OneHot`, `Contour`), the resolution changes (`Anisotropy`,
`Resize`), histogram standardization (`HistogramStandardization`,
`ZNormalization`) and its patch path (`UniformSampler`, `Queue`,
`SubjectsLoader`) on tensor-backed `Subject` / `SubjectsBatch` data.  The
tensor math runs in hand-written sm_90a (H100) CUDA kernels exposed through the C-ABI
of ``include/tio_b200.h``; see DESIGN.md and INTEGRATION.md.
"""

from .data import (AffineMatrix, Image, ImagesBatch, LabelMap, ScalarImage, StudiesBatch,
                   Subject, SubjectsBatch)
from .ops import exact_coords_default, set_exact_coords
from .params import Choice
from .patches import (GridSampler, ImagesLoader, LabelSampler, PatchLocation, PatchSampler, Queue,
                      StudiesLoader, SubjectsLoader, UniformSampler, WeightedSampler, collate_images, collate_studies,
                      collate_subjects)
from .transforms import (Affine, Anisotropy, AppliedTransform, BiasField, Blur, Compose, Contour, Crop, CropOrPad,
                         ElasticDeformation, Flip, Gamma, HistogramStandardization, IntensityTransform, LabelsToImage, Noise, Normalize, OneHot, Pad,
                         RemapLabels, RemoveLabels, Resample, RescaleIntensity, Resize, SequentialLabels, Spatial,
                         SpatialTransform, Standardize, Transform, ZNormalization,
                         apply_inverse_transform, execution_device, get_inverse_transform,
                         set_execution_device)

__version__ = "0.1.0"

__all__ = [
    "Affine", "AffineMatrix", "Anisotropy", "AppliedTransform", "BiasField", "Blur", "Choice", "Compose", "Contour", "Crop", "CropOrPad",
    "ElasticDeformation", "Flip", "Gamma", "GridSampler", "HistogramStandardization", "Image", "ImagesBatch", "ImagesLoader", "IntensityTransform",
    "LabelMap", "LabelSampler", "LabelsToImage", "Noise", "Normalize", "OneHot", "Pad", "PatchLocation", "PatchSampler", "Queue", "RemapLabels", "RemoveLabels",
    "Resample", "RescaleIntensity", "Resize", "ScalarImage", "SequentialLabels", "Spatial",
    "SpatialTransform", "Standardize", "StudiesBatch", "StudiesLoader", "Subject", "SubjectsBatch",
    "SubjectsLoader", "Transform", "UniformSampler", "WeightedSampler", "ZNormalization", "apply_inverse_transform", "collate_images",
    "collate_studies", "collate_subjects", "exact_coords_default", "execution_device", "get_inverse_transform",
    "set_exact_coords", "set_execution_device",
]
