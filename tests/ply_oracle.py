"""NumPy restatement of the plain PLY readers and writers (formats/ply_3dgs.py Ply3DGSFormat, formats/ply_cc.py
PlyCCFormat) and of the header plyfile writes, for sizes the golden fixture (g15) does not reach.  The field mapping runs
as NumPy structured assignments, so the casts are NumPy's own.  read / write raise ValueError exactly where gsx.ply
refuses (see gsx.ply.decode / encode), so a case's expect ("ok" / "refuse") can be checked against it."""
import numpy as np

from gsx.readers import parse_ply_header

ROW_MAX = 1024
TYPES = {"i1": "char", "u1": "uchar", "i2": "short", "u2": "ushort", "i4": "int", "u4": "uint", "f4": "float",
         "f8": "double"}


def std_order(has_rgb):
    names = ["x", "y", "z", "nx", "ny", "nz", "f_dc_0", "f_dc_1", "f_dc_2"] + [f"f_rest_{i}" for i in range(45)]
    names += ["opacity", "scale_0", "scale_1", "scale_2", "rot_0", "rot_1", "rot_2", "rot_3"]
    return names + (["red", "green", "blue"] if has_rgb else [])


def _kind(dt):
    if dt.shape or dt.byteorder not in "=<|" or f"{dt.kind}{dt.itemsize}" not in TYPES:
        raise ValueError(f"type {dt.str}")
    return f"{dt.kind}{dt.itemsize}"


def _check_cast(s, d):
    s, d = _kind(s), _kind(d)
    if not (s == d or d == "u1" or (d == "f4" and (s[0] in "iu" or s == "f8"))):
        raise ValueError(f"no device cast {s} -> {d}")


def vertices(buf: bytes) -> np.ndarray:
    """The vertex array plyfile would return for a binary little-endian PLY holding only `vertex`."""
    els, end = parse_ply_header(buf)
    if list(els) != ["vertex"] or end > len(buf):
        raise ValueError("not a lone, complete vertex element")
    vx = els["vertex"]
    if not vx.dtype.names or vx.dtype.itemsize > ROW_MAX:
        raise ValueError("vertex rows")
    return np.frombuffer(buf, vx.dtype, vx.count, vx.offset)


def read(buf: bytes, flavor: str) -> np.ndarray:
    v = vertices(buf)
    names = v.dtype.names
    if flavor == "3dgs":
        p = "scal_" if "scal_f_dc_0" in names else ""
        if "scalar_f_dc_0" in names:
            p = "scalar_scal_" if "scalar_scal_f_dc_0" in names else "scalar_"
        base = std_order(True)
    else:
        p = "scalar_" if "scalar_f_dc_0" in names else "scalar_scal_" if "scalar_scal_f_dc_0" in names else ""
        base = std_order(True) + ["nx", "ny", "nz"]
    known = set(base) | {p + b for b in base}
    dt = [(f, "f4") for f in std_order(False)] + ([(c, "u1") for c in ("red", "green", "blue")] if "red" in names
                                                  else [])
    for f in names:
        if f in known:
            continue
        g = f[len("scalar_"):] if flavor == "cc" and f.startswith("scalar_") else f
        if g == "":
            raise ValueError("empty name")
        if g not in [d[0] for d in dt]:
            dt.append((g, v.dtype[f].str))
    out = np.zeros(len(v), dt)
    if out.dtype.itemsize > ROW_MAX:
        raise ValueError("array rows")
    for t in out.dtype.names:
        for s in (t, p + t) + ((f"scalar_{t}",) if flavor == "cc" else ()):
            if s in names:
                _check_cast(v.dtype[s], out.dtype[t])
                with np.errstate(all="ignore"):
                    out[t] = v[s]
                break
    return out


def last_nonzero_rest(data: np.ndarray) -> int:
    for i in range(44, -1, -1):
        f = f"f_rest_{i}"
        if f in data.dtype.names and np.any(data[f] != 0):
            return i
    return -1


def write(data: np.ndarray, flavor: str, crop_sh: bool = False) -> np.ndarray:
    """output_data, the array the writer hands to PlyElement.describe."""
    names = data.dtype.names
    for f in names:
        if f in std_order(False) and f.startswith("f_rest_") and data.dtype[f] != np.dtype("<f4"):
            raise ValueError(f"{f} not float32")
    order = std_order("red" in names)
    if crop_sh:
        last = last_nonzero_rest(data)
        order = [f for f in order if not f.startswith("f_rest_") or int(f[7:]) <= last]
    rename = (lambda f: f) if flavor == "3dgs" else (
        lambda f: f if f in {"x", "y", "z", "nx", "ny", "nz", "red", "green", "blue"} else "scalar_" + f)
    dt, copy = [], []
    for f in order:
        if f in names:
            dt.append((rename(f), data.dtype[f].str))
            copy.append((f, rename(f)))
        elif f in ("nx", "ny", "nz") or (f.startswith("f_rest_") and not crop_sh):
            dt.append((f if f[0] == "n" else rename(f), "f4"))
    for f in names:
        if f not in order and f not in std_order(True):
            o = f if flavor == "3dgs" else "scalar_" + f
            dt.append((o, data.dtype[f].str))
            copy.append((f, o))
    out = np.zeros(len(data), dt)
    for f in out.dtype.names:
        _kind(out.dtype[f])
    if data.dtype.itemsize > ROW_MAX or out.dtype.itemsize > ROW_MAX:
        raise ValueError("rows")
    for f, o in copy:
        out[o] = data[f]
    return out


def header(out: np.ndarray) -> bytes:
    """What plyfile's PlyData([PlyElement.describe(out, 'vertex')], byte_order='<').write puts before the body."""
    props = "".join(f"property {TYPES[_kind(out.dtype[f])]} {f}\n" for f in out.dtype.names)
    return f"ply\nformat binary_little_endian 1.0\nelement vertex {len(out)}\n{props}end_header\n".encode("ascii")


def file(out: np.ndarray) -> bytes:
    return header(out) + np.ascontiguousarray(out).tobytes()
