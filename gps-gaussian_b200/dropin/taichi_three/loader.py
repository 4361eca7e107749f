"""Wavefront OBJ reading with the reference loader's result (prepare_data/taichi_three/loader.py `readobj`)."""
import numpy as np


def _numbers(rest):
    """The float fields of a line's remainder, or None when one of them is not a number."""
    try:
        return [float(tok) for tok in rest.split()]
    except ValueError:
        return None


def _corner(token):
    """'v', 'v/vt', 'v//vn' or 'v/vt/vn' -> zero-based indices, an empty field giving 0."""
    return [int(part) - 1 if part != "" else 0 for part in token.split("/")]


def readobj(path, scale=1):
    """{'vi': [V,k] float32 * scale, 'vt': [T,k] float32, 'vn': [N,3] float32, 'f': [F,3,c] int32}, each None when the
    file has none.  A line is read when it has a keyword and a remainder; `v`, `vt` and `vn` lines whose remainder is not
    all numbers are skipped.  Quads become the triangles (0, 1, 2) and (2, 3, 0); any other corner count is an error."""
    with open(path, "r") as fh:
        lines = fh.readlines()
    vi, vt, vn, faces = [], [], [], []
    heads = []
    for line in lines:
        parts = line.split(maxsplit=1)
        if len(parts) != 2:
            continue
        heads.append(parts)
    for key, rest in heads:
        if key not in ("v", "vt", "vn"):
            continue
        nums = _numbers(rest)
        if nums is None:
            continue
        {"v": vi, "vt": vt, "vn": vn}[key].append(nums)
    for key, rest in heads:
        if key != "f":
            continue
        corners = [_corner(tok) for tok in rest.split()]
        if len(corners) == 3:
            faces.append(corners)
        elif len(corners) == 4:
            faces.append([corners[0], corners[1], corners[2]])
            faces.append([corners[2], corners[3], corners[0]])
        else:
            raise AssertionError(len(corners))
    as_f32 = lambda rows: None if not rows else np.array(rows).astype(np.float32)
    return {"vi": None if not vi else np.array(vi).astype(np.float32) * scale, "vt": as_f32(vt), "vn": as_f32(vn),
            "f": None if not faces else np.array(faces).astype(np.int32)}
