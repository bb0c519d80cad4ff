"""nibabel.orientations for generate_orientation.py: restatements of nibabel's documented algorithms
(io_orientation, axcodes2ornt, ornt_transform, inv_ornt_aff, ornt2axcodes, aff2axcodes), written for
the tests because nibabel is not installed.  The generator installs this module as
``nibabel.orientations`` in place of the ``_shim/`` stub (whose aff2axcodes always answers RAS) before
it imports the reference; the other generators keep the stub.  An "ornt" is a (p, 2) float array:
row = input axis, [output axis, +1 / -1 direction]."""

import numpy as np


def io_orientation(affine, tol=None):
    affine = np.asarray(affine)
    q, p = affine.shape[0] - 1, affine.shape[1] - 1
    rzs = affine[:q, :p]
    zooms = np.sqrt(np.sum(rzs * rzs, axis=0))
    zooms[zooms == 0] = 1
    rs = rzs / zooms
    u, s, vt = np.linalg.svd(rs, full_matrices=False)
    if tol is None:
        tol = s.max() * max(rs.shape) * np.finfo(s.dtype).eps
    keep = s > tol
    r = np.dot(u[:, keep], vt[keep])
    ornt = np.ones((p, 2), dtype=np.int8) * np.nan
    for in_ax in range(p):
        col = r[:, in_ax]
        if not np.allclose(col, 0):
            out_ax = np.argmax(np.abs(col))
            ornt[in_ax, 0] = out_ax
            ornt[in_ax, 1] = -1 if col[out_ax] < 0 else 1
            r[out_ax, :] = 0
    return ornt


def axcodes2ornt(axcodes, labels=None):
    labels = list(zip("LPI", "RAS")) if labels is None else labels
    allowed = sum([list(pair) for pair in labels], []) + [None]
    if not set(axcodes).issubset(allowed):
        raise ValueError(f"Not all axis codes {list(axcodes)} in label set {allowed}")
    ornt = np.ones((len(axcodes), 2), dtype=np.int8) * np.nan
    for code_idx, code in enumerate(axcodes):
        for label_idx, codes in enumerate(labels):
            if code is None:
                continue
            if code in codes:
                ornt[code_idx, :] = [label_idx, -1 if code == codes[0] else 1]
                break
    return ornt


def ornt_transform(start_ornt, end_ornt):
    start_ornt = np.asarray(start_ornt)
    end_ornt = np.asarray(end_ornt)
    if start_ornt.shape != end_ornt.shape:
        raise ValueError("The orientations must have the same shape")
    result = np.empty_like(start_ornt)
    for end_in_idx, (end_out_idx, end_flip) in enumerate(end_ornt):
        for start_in_idx, (start_out_idx, start_flip) in enumerate(start_ornt):
            if end_out_idx == start_out_idx:
                result[start_in_idx, :] = [end_in_idx, 1 if start_flip == end_flip else -1]
                break
        else:
            raise ValueError("Unable to find out axis %d in start_ornt" % end_out_idx)
    return result


def inv_ornt_aff(ornt, shape):
    ornt = np.asarray(ornt)
    if np.any(np.isnan(ornt)):
        raise ValueError("We cannot invert orientation transform")
    p = ornt.shape[0]
    shape = np.array(shape)[:p]
    axis_transpose = [int(v) for v in ornt[:, 0]]
    undo_reorder = np.eye(p + 1)[axis_transpose + [p], :]
    undo_flip = np.diag(list(ornt[:, 1]) + [1.0])
    center_trans = -(shape - 1) / 2.0
    undo_flip[:p, p] = (ornt[:, 1] * center_trans) - center_trans
    return np.dot(undo_flip, undo_reorder)


def ornt2axcodes(ornt, labels=None):
    labels = list(zip("LPI", "RAS")) if labels is None else labels
    axcodes = []
    for axno, direction in np.asarray(ornt):
        if np.isnan(axno):
            axcodes.append(None)
            continue
        axint = int(np.round(axno))
        if axint != axno:
            raise ValueError(f"Non integer axis number {axno:f}")
        if direction == 1:
            axcodes.append(labels[axint][1])
        elif direction == -1:
            axcodes.append(labels[axint][0])
        else:
            raise ValueError("Direction should be -1 or 1")
    return tuple(axcodes)


def aff2axcodes(aff, labels=None, tol=None):
    return ornt2axcodes(io_orientation(aff, tol), labels)
