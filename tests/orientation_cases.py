"""Reorient / Transpose / EnsureShapeMultiple / CopyAffine / ToReferenceSpace test infrastructure: the
fixture cases, their seeded inputs, how a case is run, and a numpy oracle of the voxel moves written
from the definitions (nibabel's apply_orientation: np.flip on the input axes, then transpose; pad and
crop by the recorded amounts).  ``tests/golden/generate_orientation.py`` runs the reference's classes
on these cases; nothing here is imported by the product."""

from __future__ import annotations

import json
from pathlib import Path

import numpy as np
import torch

GOLDEN = Path(__file__).resolve().parent / "golden"

F32, U8, I8, I16, I32, I64 = torch.float32, torch.uint8, torch.int8, torch.int16, torch.int32, torch.int64
SHORT = {U8: "u8", I8: "i8", I16: "i16", I32: "i32", I64: "i64"}


# Inputs: "t1" (ScalarImage, (B, C, *shape) fp32, uniform [-100, 400)) and, with `seg`, a LabelMap
# "seg" (B, 1, *shape) of labels 0..5 of that dtype.  `affine`: one of AFFINES, per element.
def _rotation(axis: int, degrees: float) -> np.ndarray:
    c, s = np.cos(np.radians(degrees)), np.sin(np.radians(degrees))
    r = np.eye(3)
    a, b = [x for x in range(3) if x != axis]
    r[a, a], r[a, b], r[b, a], r[b, b] = c, -s, s, c
    return r


def tilted_affine(b: int) -> np.ndarray:
    """Element 0: RAS tilted by 20° about S; element 1: axes (A, S, R) order, tilted; then alternating."""
    m = np.eye(4)
    direction = _rotation(2, 20.0) @ _rotation(0, -7.0)
    if b % 2 == 1:
        direction = direction[:, [1, 2, 0]] * np.array([1.0, -1.0, 1.0])
    m[:3, :3] = direction * np.array([0.9, 1.1, 1.7])
    m[:3, 3] = [-12.5 + b, 7.25, 3.0 - 2 * b]
    return m


def _diag(*spacing) -> np.ndarray:
    m = np.diag([*spacing, 1.0])
    m[:3, 3] = [1.0, -2.0, 3.5]
    return m


AFFINES = {
    "ras": lambda b: _diag(1.0, 1.0, 1.0),
    "las": lambda b: _diag(-1.0, 1.0, 1.0),
    "aniso": lambda b: _diag(-0.7, 1.3, 2.5),
    "tilted": tilted_affine,
}

REORIENT_CASES = [
    dict(name="reorient_las_b1_f32", batch=1, shape=(9, 8, 7), affine="ras", kwargs=dict(orientation="LAS")),
    dict(name="reorient_ras_from_las_b3_f32", batch=3, shape=(9, 8, 7), affine="las", kwargs=dict(orientation="RAS")),
    dict(name="reorient_ras_identity_b3_f32", batch=3, shape=(9, 8, 7), affine="ras", kwargs=dict()),
    dict(name="reorient_ars_b3_f32", batch=3, shape=(9, 8, 7), affine="ras", kwargs=dict(orientation="ARS")),
    dict(name="reorient_psr_b3_f32", batch=3, shape=(9, 8, 7), affine="ras", kwargs=dict(orientation="PSR")),
    dict(name="reorient_spl_b1_f32", batch=1, shape=(9, 8, 7), affine="ras", kwargs=dict(orientation="SPL")),
    dict(name="reorient_air_b3_f32", batch=3, shape=(9, 8, 7), affine="ras", kwargs=dict(orientation="AIR")),
    dict(name="reorient_lps_b3_f32", batch=3, shape=(9, 8, 7), affine="las", kwargs=dict(orientation="LPS")),
    dict(name="reorient_lowercase_b1_f32", batch=1, shape=(9, 8, 7), affine="las", kwargs=dict(orientation="lps")),
    dict(name="reorient_tilted_b3_f32", batch=3, shape=(9, 8, 7), affine="tilted", seg=I16,
         kwargs=dict(orientation="PSR")),
    dict(name="reorient_aniso_spl_b3_f32", batch=3, shape=(9, 8, 7), affine="aniso", kwargs=dict(orientation="SPL")),
    dict(name="reorient_odd_c2_b1_f32", batch=1, channels=2, shape=(35, 6, 33), affine="tilted",
         kwargs=dict(orientation="SPL")),
    dict(name="reorient_2d_b3_f32", batch=3, shape=(12, 10, 1), affine="ras", kwargs=dict(orientation="ILA")),
    *[dict(name=f"reorient_seg_{SHORT[d]}", batch=3, shape=(9, 8, 7), affine="aniso", seg=d,
           kwargs=dict(orientation="PSR")) for d in (U8, I8, I16, I32, I64)],
    dict(name="reorient_include_seg", batch=3, shape=(9, 8, 7), affine="ras", seg=I16,
         kwargs=dict(orientation="SPL", include=["seg"])),
    dict(name="reorient_exclude_seg", batch=3, shape=(9, 8, 7), affine="ras", seg=I16,
         kwargs=dict(orientation="SPL", exclude=["seg"])),
    dict(name="reorient_p05_applied", batch=3, shape=(9, 8, 7), affine="ras", seed=3,
         kwargs=dict(orientation="AIR", p=0.5)),
    dict(name="reorient_p05_skipped", batch=3, shape=(9, 8, 7), affine="ras", seed=1,
         kwargs=dict(orientation="AIR", p=0.5)),
    dict(name="reorient_error_init_length", batch=1, shape=(2, 2, 2), affine="ras", kwargs=dict(orientation="RA")),
    dict(name="reorient_error_init_letters", batch=1, shape=(2, 2, 2), affine="ras", kwargs=dict(orientation="RAX")),
    dict(name="reorient_error_init_pairs", batch=1, shape=(2, 2, 2), affine="ras", kwargs=dict(orientation="RRS")),
    dict(name="reorient_error_init_type", batch=1, shape=(2, 2, 2), affine="ras", kwargs=dict(orientation=5)),
]

TRANSPOSE_CASES = [
    dict(name="transpose_b3_f32", batch=3, shape=(9, 8, 7), affine="tilted", kwargs=dict()),
    dict(name="transpose_include_t1", batch=3, shape=(9, 8, 7), affine="aniso", seg=I16, kwargs=dict(include=["t1"])),
    dict(name="transpose_2d_b1", batch=1, shape=(12, 10, 1), affine="ras", kwargs=dict()),
]

_MODES = ("constant", "reflect", "replicate", "circular", "mean", "median", "minimum")
ESM_CASES = [
    *[dict(name=f"ensure_multiple_pad_{mode}", batch=3, shape=(9, 8, 7), affine="aniso",
           kwargs=dict(target_multiple=4, padding_mode=mode)) for mode in _MODES],
    dict(name="ensure_multiple_pad_fill", batch=3, shape=(9, 8, 7), affine="ras", seg=I16,
         kwargs=dict(target_multiple=(4, 3, 5), fill=2.5)),
    dict(name="ensure_multiple_crop", batch=3, shape=(9, 8, 7), affine="tilted", seg=U8,
         kwargs=dict(target_multiple=(4, 3, 2), method="crop")),
    dict(name="ensure_multiple_crop_clamp_to_1", batch=1, shape=(9, 8, 20), affine="ras",
         kwargs=dict(target_multiple=16, method="crop")),
    dict(name="ensure_multiple_unchanged", batch=3, shape=(8, 8, 4), affine="ras", kwargs=dict(target_multiple=4)),
    dict(name="ensure_multiple_include_t1", batch=3, shape=(9, 8, 7), affine="ras", seg=I16,
         kwargs=dict(target_multiple=8, include=["t1"])),
    dict(name="ensure_multiple_subject_pad", batch=1, shape=(9, 8, 7), affine="tilted", seg=I16, subject=True,
         kwargs=dict(target_multiple=4, padding_mode="reflect")),
    dict(name="ensure_multiple_subject_crop", batch=1, shape=(9, 8, 7), affine="ras", subject=True,
         kwargs=dict(target_multiple=(2, 3, 4), method="crop")),
    dict(name="ensure_multiple_error_init_zero", batch=1, shape=(2, 2, 2), affine="ras", kwargs=dict(target_multiple=0)),
    dict(name="ensure_multiple_error_init_length", batch=1, shape=(2, 2, 2), affine="ras",
         kwargs=dict(target_multiple=(2, 2))),
    dict(name="ensure_multiple_error_init_value", batch=1, shape=(2, 2, 2), affine="ras",
         kwargs=dict(target_multiple=(2, 0, 2))),
    dict(name="ensure_multiple_error_init_method", batch=1, shape=(2, 2, 2), affine="ras",
         kwargs=dict(target_multiple=2, method="both")),
    dict(name="ensure_multiple_error_init_mode", batch=1, shape=(2, 2, 2), affine="ras",
         kwargs=dict(target_multiple=2, padding_mode="wrap")),
]

COPY_CASES = [
    dict(name="copy_affine_b3", batch=3, shape=(9, 8, 7), affine="tilted", seg=I16, seg_affine="aniso",
         kwargs=dict(target="t1")),
    dict(name="copy_affine_include_t1", batch=3, shape=(9, 8, 7), affine="tilted", seg=I16, seg_affine="aniso",
         kwargs=dict(target="seg", include=["t1"])),
    dict(name="copy_affine_error_missing", batch=3, shape=(9, 8, 7), affine="ras", seg=I16, kwargs=dict(target="brain")),
]

REFERENCE_CASES = [
    dict(name="to_reference_space_b3", batch=3, shape=(9, 8, 7), affine="ras", seg=I16, kwargs=dict()),
    dict(name="to_reference_space_exclude_seg", batch=3, shape=(5, 4, 3), affine="ras", seg=I16,
         kwargs=dict(exclude=["seg"])),
    dict(name="to_reference_space_error_init", batch=1, shape=(2, 2, 2), affine="ras", kwargs=dict()),
]

CASES = {c["name"]: c for c in [*REORIENT_CASES, *TRANSPOSE_CASES, *ESM_CASES, *COPY_CASES, *REFERENCE_CASES]}
for _c in CASES.values():
    _c["kind"] = ("Reorient" if _c["name"].startswith("reorient") else "Transpose" if _c["name"].startswith("transpose")
                  else "EnsureShapeMultiple" if _c["name"].startswith("ensure") else "CopyAffine"
                  if _c["name"].startswith("copy") else "ToReferenceSpace")


def seed(case) -> int:
    return case.get("seed", 700 + sorted(CASES).index(case["name"]))


def reference_tensor() -> torch.Tensor:
    return torch.as_tensor(np.random.default_rng(99).uniform(0, 1, (1, 20, 16, 14)), dtype=torch.float32)


def reference_affine() -> np.ndarray:
    m = tilted_affine(1)
    m[:3, 3] = [4.0, -3.5, 10.25]
    return m


def reference_image(tio=None):
    """ToReferenceSpace's reference image, built with ``tio`` (this package by default)."""
    if tio is None:
        import torchio_b200 as tio
    return tio.ScalarImage(reference_tensor(), affine=reference_affine())


def inputs(case) -> dict[str, tuple[torch.Tensor, list[np.ndarray]]]:
    """name -> ((B, C, I, J, K) tensor, per-element affines)."""
    rng = np.random.default_rng(seed(case))
    b, shape = case["batch"], case["shape"]
    t1 = torch.as_tensor(rng.uniform(-100.0, 400.0, (b, case.get("channels", 1), *shape)), dtype=F32)
    out = {"t1": (t1, [AFFINES[case["affine"]](i) for i in range(b)])}
    if case.get("seg") is not None:
        seg = torch.as_tensor(rng.integers(0, 6, (b, 1, *shape)), dtype=case["seg"])
        out["seg"] = (seg, [AFFINES[case.get("seg_affine", case["affine"])](i) for i in range(b)])
    return out


def subjects(tio, images) -> list:
    b = images["t1"][0].shape[0]
    out = []
    for i in range(b):
        entries = {}
        for key, (data, affines) in images.items():
            cls = tio.ScalarImage if key == "t1" else tio.LabelMap
            entries[key] = cls(data[i].clone(), affine=affines[i].copy())
        out.append(tio.Subject(**entries))
    return out


def batch(case, images, tio=None):
    if tio is None:
        import torchio_b200 as tio
    return tio.SubjectsBatch.from_subjects(subjects(tio, images))


def transform(case, tio=None):
    if tio is None:
        import torchio_b200 as tio
    kwargs = dict(case["kwargs"])
    if case["kind"] == "ToReferenceSpace":
        kwargs["reference"] = reference_tensor() if "error" in case["name"] else reference_image(tio)
    return getattr(tio, case["kind"])(**kwargs)


def apply(case, batch, tio=None):
    """Run the case (the global seed already set): ({name: (data, [affine arrays])}, history)."""
    t = transform(case, tio)
    if case.get("subject"):
        out = t(batch.unbatch()[0])
        images = {k: (out[k].data[None], [np.asarray(out[k].affine.numpy(), dtype=np.float64)]) for k in batch.images}
        return images, list(out.applied_transforms)
    out = t(batch)
    images = {k: (ib.data, [np.asarray(a.numpy(), dtype=np.float64) for a in ib.affines])
              for k, ib in out.images.items()}
    return images, list(out.applied_transforms)


# ---- the numpy oracle -----------------------------------------------------------------------

def _selected(record, key) -> bool:
    include, exclude = record.get("include"), record.get("exclude")
    return (include is None or key in include) and (exclude is None or key not in exclude)


def _reorient(x: np.ndarray, ornt) -> np.ndarray:
    ornt = np.asarray(ornt)
    for ax in range(3):
        if ornt[ax, 1] == -1:
            x = np.flip(x, ax + 2)
    return np.ascontiguousarray(np.transpose(x, (0, 1, *(int(p) + 2 for p in np.argsort(ornt[:, 0])))))


def _pad(x: np.ndarray, padding, mode, fill) -> np.ndarray:
    widths = [(0, 0), (0, 0), (padding[0], padding[1]), (padding[2], padding[3]), (padding[4], padding[5])]
    if mode == "constant":
        return np.pad(x, widths, mode="constant", constant_values=np.asarray(fill).astype(x.dtype))
    if mode in ("reflect", "replicate", "circular"):
        return np.pad(x, widths, mode={"reflect": "reflect", "replicate": "edge", "circular": "wrap"}[mode])
    out = []
    for element in x:
        flat = element.reshape(-1)
        if mode == "median":  # the 0.5 quantile, interpolated in fp32 as torch.lerp does
            s = np.sort(flat).astype(np.float32)
            pos = 0.5 * (flat.size - 1)
            lo = int(np.floor(pos))
            a, b, w = s[lo], s[min(lo + 1, flat.size - 1)], np.float32(pos - lo)
            value = a + w * (b - a) if w < 0.5 else b - (b - a) * (np.float32(1) - w)
        else:
            value = flat.min() if mode == "minimum" else np.float32(flat.astype(np.float64).mean())
        out.append(np.pad(element, widths[1:], mode="constant", constant_values=np.asarray(value).astype(x.dtype)))
    return np.stack(out)


def _crop(x: np.ndarray, cropping) -> np.ndarray:
    i0, i1, j0, j1, k0, k1 = cropping
    return np.ascontiguousarray(x[:, :, i0:x.shape[2] - i1, j0:x.shape[3] - j1, k0:x.shape[4] - k1])


def oracle_output(case, images, history) -> dict[str, tuple[np.ndarray, None]]:
    """The voxels every recorded step leaves, from the definitions.  Statistic padding modes take
    the element's minimum, its fp32 mean and its lower median: the fixtures' ties are the checks."""
    out = {k: (v.numpy().copy(), None) for k, (v, _) in images.items()}
    for record in history:
        name, params = record["name"], record["params"]
        for key in out:
            x = out[key][0]
            if name == "Reorient" and _selected(record, key) and not (
                    np.array_equal(np.asarray(params["ornt"])[:, 0], [0, 1, 2])
                    and np.all(np.asarray(params["ornt"])[:, 1] == 1)):
                x = _reorient(x, params["ornt"])
            elif name == "Transpose":
                x = np.ascontiguousarray(np.transpose(x, (0, 1, 4, 3, 2)))
            elif name == "Pad" and _selected(record, key):
                x = _pad(x, params["padding"], params["padding_mode"], params["fill"])
            elif name == "Crop" and _selected(record, key):
                x = _crop(x, params["cropping"])
            out[key] = (x, None)
    return out


def output_affines(case, batch, params) -> dict[str, list[np.ndarray]]:
    """The affines the transform writes, on the host (no voxel moves)."""
    t = transform(case)
    if case["kind"] == "Reorient":
        from torchio_b200.data import _inv_ornt_aff

        ornt = np.asarray(params["ornt"])
        identity = np.array_equal(ornt[:, 0], [0, 1, 2]) and np.all(ornt[:, 1] == 1)
        selected = t._get_images(batch)
        return {k: [a.numpy() @ _inv_ornt_aff(ornt, ib.data.shape[-3:]) if k in selected and not identity
                    else a.numpy() for a in ib.affines] for k, ib in batch.images.items()}
    if case["kind"] == "Transpose":
        return {k: [a.numpy()[:, [2, 1, 0, 3]] for a in ib.affines] for k, ib in batch.images.items()}
    t.apply_transform(batch, params)  # CopyAffine / ToReferenceSpace touch affines only
    return {k: [a.numpy() for a in ib.affines] for k, ib in batch.images.items()}


def as_stored(t) -> np.ndarray:
    if isinstance(t, torch.Tensor):
        t = t.detach().cpu().contiguous().numpy()
    return np.ascontiguousarray(t)


def same(a, b) -> bool:
    a, b = np.asarray(a), np.asarray(b)
    if a.shape != b.shape or a.dtype != b.dtype:
        return False
    if a.dtype.kind == "f":
        return bool(np.array_equal(a.view(f"u{a.itemsize}"), b.view(f"u{b.itemsize}")))
    return bool(np.array_equal(a, b))


def load_fixture(name: str) -> dict:
    with np.load(GOLDEN / f"orientation_{name}.npz") as z:
        out = {k: z[k] for k in z.files}
    for key in ("history", "error", "hydra", "repr"):
        if key in out:
            out[key] = json.loads(out[key].tobytes().decode())
    return out
