"""KeepLargestComponent test infrastructure: the fixture cases, their seeded inputs, the reference's op
sequence (label/keep_largest.py:63-125 of TorchIO 2.0.0a2) on plain torch tensors with a pluggable
connected-component labeller standing in for SimpleITK, and the two labellers (scipy, and the C
oracle, which needs no scipy).  ``tests/golden/generate_keep_largest.py`` runs the reference's class on
these cases; nothing here is imported by the product.

SimpleITK is not available, so its three calls are restated (`SitkRestatement`) from what ITK
documents, under one assumption that could not be checked against SimpleITK itself:
- ``ConnectedComponent(image, fullyConnected)`` labels the nonzero voxels 1, 2, ... with face (6) or
  full (26) connectivity, numbering the objects in raster order with x, numpy's last axis, fastest
  (``GetImageFromArray`` maps the array's last axis to x).  ``scipy.ndimage.label`` numbers them the
  same way.
- ``RelabelComponent(image, sortByObjectSize=True)`` renumbers them by decreasing size, and
  (ASSUMED) breaks ties by the smaller original number: a stable sort.
So among equal-size components of a label, the one whose first voxel in C order comes first is kept.
"""

from __future__ import annotations

import json
from pathlib import Path

import numpy as np
import torch

GOLDEN = Path(__file__).resolve().parent / "golden"

I8, U8, I16, I32, I64, F32 = torch.int8, torch.uint8, torch.int16, torch.int32, torch.int64, torch.float32

# transforms: [(class name, kwargs)], one Compose when there are several; kind selects the input:
#   blobs       labels (low, high) on a 2x-upsampled random grid, plus `salt` of random voxels
#   voxels      zeros with [(element, (i, j, k), value)] set
#   checker     label 1 + (i + j + k) % 2
#   serpentine  one 1-voxel-wide path of label 1 through the whole volume, plus stray voxels of it
# extra: [(element, value)] written into a 2 x 3 corner block of that element;
# nan / inf: written into one voxel of the given elements; fractional: + 0.5 on a lattice.
KEEP = "KeepLargestComponent"
CASES = [
    dict(name="keep_largest_defaults_i16", transforms=[(KEEP, {})],
         batch=3, shape=(14, 13, 12), dtype=I16, kind="blobs", labels=(0, 5), salt=0.08, seed=301),
    dict(name="keep_largest_six_connected_i16", transforms=[(KEEP, {"fully_connected": False})],
         batch=3, shape=(14, 13, 12), dtype=I16, kind="blobs", labels=(0, 5), salt=0.08, seed=301),
    dict(name="keep_largest_pair_face_u8", transforms=[(KEEP, {"fully_connected": False})],
         batch=1, shape=(6, 6, 6), dtype=U8, kind="voxels",
         voxels=[(0, (1, 1, 1), 1), (0, (1, 1, 2), 1), (0, (4, 4, 4), 1), (0, (0, 5, 5), 2)], seed=302),
    dict(name="keep_largest_pair_edge_six_u8", transforms=[(KEEP, {"fully_connected": False})],
         batch=1, shape=(6, 6, 6), dtype=U8, kind="voxels",
         voxels=[(0, (4, 1, 1), 1), (0, (4, 2, 2), 1), (0, (0, 4, 4), 1), (0, (2, 2, 2), 2)], seed=303),
    dict(name="keep_largest_pair_edge_full_u8", transforms=[(KEEP, {})],
         batch=1, shape=(6, 6, 6), dtype=U8, kind="voxels",
         voxels=[(0, (4, 1, 1), 1), (0, (4, 2, 2), 1), (0, (0, 4, 4), 1), (0, (2, 2, 2), 2)], seed=304),
    dict(name="keep_largest_pair_corner_full_i32", transforms=[(KEEP, {})],
         batch=1, shape=(6, 6, 6), dtype=I32, kind="voxels",
         voxels=[(0, (3, 1, 1), 1), (0, (4, 2, 2), 1), (0, (0, 4, 4), 1), (0, (5, 5, 0), 1)], seed=305),
    dict(name="keep_largest_pair_corner_six_i32", transforms=[(KEEP, {"fully_connected": False})],
         batch=1, shape=(6, 6, 6), dtype=I32, kind="voxels",
         voxels=[(0, (3, 1, 1), 1), (0, (4, 2, 2), 1), (0, (0, 4, 4), 1), (0, (5, 5, 0), 1)], seed=306),
    dict(name="keep_largest_label_subset_i16", transforms=[(KEEP, {"labels": [1, 3]})],
         batch=3, shape=(12, 11, 10), dtype=I16, kind="blobs", labels=(0, 5), salt=0.1, seed=307),
    dict(name="keep_largest_absent_duplicate_labels_i32", transforms=[(KEEP, {"labels": [2, 9, 2, -70000]})],
         batch=2, shape=(12, 11, 10), dtype=I32, kind="blobs", labels=(0, 4), salt=0.1, seed=308),
    dict(name="keep_largest_u8_257_is_1", transforms=[(KEEP, {"labels": [257, 1]})],
         batch=2, shape=(10, 9, 11), dtype=U8, kind="blobs", labels=(0, 4), salt=0.1, seed=309),
    dict(name="keep_largest_background_3_i16", transforms=[(KEEP, {"background_label": 3})],
         batch=2, shape=(12, 10, 11), dtype=I16, kind="blobs", labels=(0, 5), salt=0.08, seed=310),
    dict(name="keep_largest_background_minus1_i16", transforms=[(KEEP, {"background_label": -1})],
         batch=2, shape=(12, 10, 11), dtype=I16, kind="blobs", labels=(-1, 3), salt=0.08, seed=311),
    dict(name="keep_largest_background_minus1_u8", transforms=[(KEEP, {"background_label": -1})],
         batch=2, shape=(12, 10, 11), dtype=U8, kind="blobs", labels=(0, 3), salt=0.08, extra=[(1, 255)],
         seed=312),
    dict(name="keep_largest_background_overflow_i16", transforms=[(KEEP, {"background_label": 70000})],
         batch=2, shape=(8, 9, 10), dtype=I16, kind="blobs", labels=(0, 3), salt=0.05, seed=313),
    dict(name="keep_largest_background_overflow_absent_i16",
         transforms=[(KEEP, {"labels": [7], "background_label": 70000})],
         batch=2, shape=(8, 9, 10), dtype=I16, kind="blobs", labels=(0, 3), salt=0.05, seed=314),
    dict(name="keep_largest_i8", transforms=[(KEEP, {})],
         batch=3, shape=(11, 12, 13), dtype=I8, kind="blobs", labels=(-3, 3), salt=0.1, seed=315),
    dict(name="keep_largest_i64_large_labels", transforms=[(KEEP, {})],
         batch=2, shape=(11, 12, 13), dtype=I64, kind="blobs", labels=(0, 4), salt=0.1, large=True, seed=316),
    dict(name="keep_largest_i64_large_explicit", transforms=[(KEEP, {"labels": [2**24 + 1, 2**40 + 2, 1]})],
         batch=2, shape=(11, 12, 13), dtype=I64, kind="blobs", labels=(0, 4), salt=0.1, large=True, seed=317),
    dict(name="keep_largest_f32_fractional", transforms=[(KEEP, {})],
         batch=3, shape=(12, 11, 10), dtype=F32, kind="blobs", labels=(-1, 4), salt=0.1, fractional=True,
         extra=[(1, -0.0), (2, 0.0)], seed=318),
    dict(name="keep_largest_f32_explicit_labels", transforms=[(KEEP, {"labels": [0, 2, 2.5]})],
         batch=2, shape=(12, 11, 10), dtype=F32, kind="blobs", labels=(-1, 4), salt=0.1, fractional=True,
         extra=[(0, -0.0)], seed=319),
    dict(name="keep_largest_f32_background_2_24", transforms=[(KEEP, {"background_label": 2**24 + 1})],
         batch=2, shape=(10, 11, 9), dtype=F32, kind="blobs", labels=(0, 3), salt=0.1, extra=[(0, 2.0**24)],
         seed=320),
    dict(name="keep_largest_f32_nan_error", transforms=[(KEEP, {})],
         batch=3, shape=(8, 9, 10), dtype=F32, kind="blobs", labels=(0, 3), salt=0.05, nan=[1, 2], inf=[2],
         seed=321),
    dict(name="keep_largest_f32_inf_error", transforms=[(KEEP, {})],
         batch=3, shape=(8, 9, 10), dtype=F32, kind="blobs", labels=(0, 3), salt=0.05, nan=[1], inf=[1, 2],
         seed=322),
    dict(name="keep_largest_f32_nan_explicit", transforms=[(KEEP, {"labels": [1, 2]})],
         batch=3, shape=(8, 9, 10), dtype=F32, kind="blobs", labels=(0, 3), salt=0.05, nan=[0, 2], inf=[1],
         seed=323),
    dict(name="keep_largest_b1_i16", transforms=[(KEEP, {})],
         batch=1, shape=(15, 14, 13), dtype=I16, kind="blobs", labels=(0, 6), salt=0.1, seed=324),
    dict(name="keep_largest_some_elements_i16", transforms=[(KEEP, {"labels": [4, 1]})],
         batch=3, shape=(12, 11, 10), dtype=I16, kind="blobs", labels=(0, 3), salt=0.1, extra=[(1, 4)],
         seed=325),
    dict(name="keep_largest_tie_first_voxel_i16", transforms=[(KEEP, {})],
         batch=1, shape=(8, 8, 8), dtype=I16, kind="voxels",
         voxels=[(0, (5, 0, 0), 1), (0, (5, 0, 1), 1), (0, (6, 0, 0), 1),
                 (0, (0, 6, 6), 1), (0, (0, 6, 7), 1), (0, (0, 7, 7), 1),
                 (0, (2, 2, 7), 2), (0, (2, 3, 7), 2), (0, (2, 2, 0), 2), (0, (3, 2, 0), 2)], seed=326),
    dict(name="keep_largest_tie_six_connected_i16", transforms=[(KEEP, {"fully_connected": False})],
         batch=2, shape=(7, 6, 5), dtype=I16, kind="voxels",
         voxels=[(0, (6, 5, 4), 1), (0, (0, 0, 1), 1), (0, (3, 3, 3), 1), (1, (1, 1, 1), 2), (1, (2, 2, 2), 2),
                 (1, (1, 2, 2), 3)], seed=327),
    dict(name="keep_largest_k1_i16", transforms=[(KEEP, {})],
         batch=2, shape=(13, 12, 1), dtype=I16, kind="blobs", labels=(0, 4), salt=0.1, seed=328),
    dict(name="keep_largest_odd_shape_i32", transforms=[(KEEP, {})],
         batch=2, shape=(37, 29, 23), dtype=I32, kind="blobs", labels=(0, 6), salt=0.02, seed=329),
    dict(name="keep_largest_serpentine_u8", transforms=[(KEEP, {})],
         batch=1, shape=(24, 24, 24), dtype=U8, kind="serpentine", seed=330),
    dict(name="keep_largest_serpentine_six_u8", transforms=[(KEEP, {"fully_connected": False})],
         batch=1, shape=(24, 24, 24), dtype=U8, kind="serpentine", seed=331),
    dict(name="keep_largest_checker_six_i16", transforms=[(KEEP, {"fully_connected": False})],
         batch=1, shape=(7, 6, 5), dtype=I16, kind="checker", seed=332),
    dict(name="keep_largest_checker_full_i16", transforms=[(KEEP, {})],
         batch=1, shape=(7, 6, 5), dtype=I16, kind="checker", seed=333),
    dict(name="keep_largest_two_channels_error", transforms=[(KEEP, {})],
         batch=2, channels=2, shape=(6, 5, 4), dtype=I16, kind="blobs", labels=(0, 3), salt=0.1, seed=334),
    dict(name="keep_largest_p05_i16", transforms=[(KEEP, {"p": 0.5})],
         batch=2, shape=(9, 8, 7), dtype=I16, kind="blobs", labels=(0, 3), salt=0.1, seed=335),
    dict(name="keep_largest_p05_skipped_i16", transforms=[(KEEP, {"p": 0.5})],
         batch=2, shape=(9, 8, 7), dtype=I16, kind="blobs", labels=(0, 3), salt=0.1, seed=337),
    dict(name="keep_largest_compose_cleanup_i16",
         transforms=[("SequentialLabels", {}), ("RemoveLabels", {"labels": [4, 5]}), (KEEP, {"labels": [1]})],
         batch=3, shape=(12, 11, 10), dtype=I16, kind="blobs", labels=(2, 9), salt=0.1, seed=336),
]
CASES_BY_NAME = {c["name"]: c for c in CASES}


def _serpentine(shape) -> torch.Tensor:
    """One path of 1s: along K on the even rows of the even planes, joined at alternating row ends,
    and plane to plane at alternating corners; nothing else touches it, even diagonally."""
    I, J, K = shape
    out = torch.zeros(shape, dtype=torch.int64)
    last_end = None
    for i in range(0, I, 2):
        rows = list(range(0, J, 2))
        if (i // 2) % 2:
            rows.reverse()
        if last_end is not None:
            out[i - 1, last_end[0], last_end[1]] = 1  # joins the planes
        for n, j in enumerate(rows):
            out[i, j, :] = 1
            if n + 1 < len(rows):
                end = K - 1 if n % 2 == 0 else 0
                out[i, (j + rows[n + 1]) // 2, end] = 1
        last_end = (rows[-1], K - 1 if (len(rows) - 1) % 2 == 0 else 0)
    return out


def label_map(case) -> torch.Tensor:
    """(B, C, I, J, K) labels of the case's dtype from its seed."""
    g = torch.Generator().manual_seed(case["seed"] * 7919)
    b, c = case["batch"], case.get("channels", 1)
    shape = case["shape"]
    kind = case["kind"]
    if kind == "blobs":
        lo, hi = case["labels"]
        coarse = torch.randint(lo, hi, (b, c, *((s + 1) // 2 for s in shape)), generator=g)
        data = coarse.repeat_interleave(2, 2).repeat_interleave(2, 3).repeat_interleave(2, 4)
        data = data[:, :, :shape[0], :shape[1], :shape[2]].clone()
        salt = torch.rand(data.shape, generator=g) < case["salt"]
        data[salt] = torch.randint(lo, hi, data.shape, generator=g)[salt]
    elif kind == "voxels":
        data = torch.zeros((b, c, *shape), dtype=torch.int64)
        for element, (i, j, k), value in case["voxels"]:
            data[element, 0, i, j, k] = value
    elif kind == "checker":
        i, j, k = torch.meshgrid(*(torch.arange(s) for s in shape), indexing="ij")
        data = (1 + (i + j + k) % 2).expand(b, c, *shape).clone()
    else:  # serpentine, plus stray voxels away from it
        data = _serpentine(shape).expand(b, c, *shape).clone()
        data[:, :, 1, 1::4, 2] = 1
    if case.get("large"):
        data[:, :, ::2, 1::3] += 2**24 + 1
        data[:, :, 1::2, ::3] += 2**40
    data = data.to(torch.float64 if case["dtype"] == F32 else torch.int64)
    for element, value in case.get("extra", []):
        data[element, 0, :2, :3] = value
    data = data.to(case["dtype"])
    if case.get("fractional"):
        data[:, :, ::3, 1] += 0.5
    for element in case.get("nan", []):
        data[element, 0, 3, 3, 3] = float("nan")
    for n, element in enumerate(case.get("inf", [])):
        data[element, 0, 1, 2, 3] = float("inf") if n % 2 else float("-inf")
    return data


def scalar_image(case) -> torch.Tensor:
    g = torch.Generator().manual_seed(case["seed"] * 31)
    return torch.rand((case["batch"], 1, *case["shape"]), generator=g)


def affines(case) -> list[np.ndarray]:
    return [np.diag([1.0 + 0.25 * b, 1.0, 1.5, 1.0]) for b in range(case["batch"])]


def load_fixture(name) -> dict:
    """{"history", "out_seg", "out_t1", or "error": {"type", "message"} (what the reference raised)}."""
    z = np.load(GOLDEN / f"{name}.npz")
    out = {"history": json.loads(bytes(z["history"]).decode())}
    if "error" in z:
        out["error"] = json.loads(bytes(z["error"]).decode())
    for key in ("out_seg", "out_t1"):
        if key in z:
            out[key] = torch.from_numpy(z[key])
    return out


# ---- labellers: binary (I, J, K) uint8 array -> components numbered 1, 2, ... by decreasing size ---


def _by_size(first_index: np.ndarray, sizes: np.ndarray) -> np.ndarray:
    """New number (1 = largest) of each component given in raster order of first voxels: a stable
    sort by decreasing size."""
    order = np.argsort(-sizes, kind="stable")
    rank = np.empty_like(order)
    rank[order] = np.arange(1, len(order) + 1)
    return rank


def scipy_labeller(binary: np.ndarray, fully_connected: bool) -> np.ndarray:
    from scipy import ndimage

    structure = ndimage.generate_binary_structure(3, 3 if fully_connected else 1)
    labelled, n = ndimage.label(binary, structure=structure)  # numbered in raster order
    if n == 0:
        return labelled
    sizes = np.bincount(labelled.reshape(-1), minlength=n + 1)[1:]
    table = np.concatenate([[0], _by_size(np.arange(n), sizes)])
    return table[labelled]


def c_labeller(binary: np.ndarray, fully_connected: bool) -> np.ndarray:
    from oracle import components as cc_oracle

    values = torch.from_numpy(np.ascontiguousarray(binary))
    roots = cc_oracle.connected_components(values, values != 0, fully_connected).numpy().reshape(-1)
    firsts, inverse, sizes = np.unique(roots[roots >= 0], return_inverse=True, return_counts=True)
    out = np.zeros(roots.shape, dtype=np.int64)
    out[roots >= 0] = _by_size(firsts, sizes)[inverse]
    return out.reshape(binary.shape)


class SitkRestatement:
    """The SimpleITK calls of keep_largest.py:117-120 restated with a labeller (see the module
    docstring for what this assumes)."""

    def __init__(self, labeller=scipy_labeller):
        self.labeller = labeller

    def GetImageFromArray(self, array):  # noqa: N802  (SimpleITK's names)
        return np.asarray(array)

    def ConnectedComponent(self, image, fullyConnected=False):  # noqa: N802, N803
        return ("components", image, bool(fullyConnected))

    def RelabelComponent(self, image, sortByObjectSize=True):  # noqa: N802, N803
        assert sortByObjectSize and image[0] == "components"
        return self.labeller(image[1], image[2])

    def GetArrayFromImage(self, image):  # noqa: N802
        return image


# ---- the reference's op sequence ---------------------------------------------------------------


def keep_largest_element(data, labels, background_label, fully_connected, labeller):
    """_keep_largest_per_label (keep_largest.py:89-125), SimpleITK replaced by ``labeller``."""
    result = data.clone()
    if labels is None:
        unique = data.unique().tolist()
        labels = [int(v) for v in unique if int(v) != background_label]
    for label in labels:
        binary = (data == label).cpu().numpy().astype("uint8")
        if binary.sum() == 0:
            continue
        relabeled = labeller(binary, fully_connected)
        mask = torch.from_numpy((relabeled >= 2).astype("uint8")).to(data.device)
        result[mask.bool()] = background_label
    return result


def keep_largest(data, labels=None, background_label=0, fully_connected=True, labeller=scipy_labeller):
    """KeepLargestComponent.apply_transform (keep_largest.py:63-86) on one label batch, in place."""
    b, c = data.shape[:2]
    if c != 1:
        raise RuntimeError(f"KeepLargestComponent requires single-channel label maps, got {c} channels")
    for i in range(b):
        data[i, 0] = keep_largest_element(data[i, 0], labels=labels, background_label=background_label,
                                          fully_connected=fully_connected, labeller=labeller)
    return data


def reference_output(case, data, labeller=scipy_labeller):
    """(output, history) of the case's transforms on ``data`` for a p=1 pipeline (the coin of a p < 1
    case is the test's business)."""
    import label_map_cases as label_ref

    history = []
    for name, kwargs in case["transforms"]:
        if name == KEEP:
            params = {}
            data = keep_largest(data.clone(), kwargs.get("labels"), kwargs.get("background_label", 0),
                                kwargs.get("fully_connected", True), labeller)
        elif name == "SequentialLabels":
            params = {"remappings": {"seg": label_ref.sequential_params(data)}}
            data = label_ref.renumber(data, params["remappings"]["seg"])
        else:  # RemoveLabels
            params = {}
            data = label_ref.remove(data, kwargs["labels"], kwargs.get("background_label", 0))
        history.append({"name": name, "params": params})
    return data, history
