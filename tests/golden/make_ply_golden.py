"""Generate tests/golden/g15_reference_ply_small.npz: the reference's own Ply3DGSFormat and PlyCCFormat read and write
(formats/ply_3dgs.py, formats/ply_cc.py) on small inputs.

    python tests/golden/make_ply_golden.py REFERENCE_ROOT     (a checkout of francescofugazzi/3dgsconverter)

The two modules are loaded by file path with `plyfile` stubbed: the stub's PlyData.read returns the elements parsed
from the file the script also writes (gsx.readers.parse_ply_header, binary little-endian and fixed-size properties only;
files it cannot parse are refused by gsx and the reference is not run), and PlyElement.describe / PlyData(...).write
capture the array the writer builds.  So the reference's own field logic runs for every case.  Reader cases: plain,
RGB as uchar / float / double / ushort, SH degrees 0-2, every prefix, extras of all 8 PLY types, `scalar_` extras and
extras that collide after stripping, integer and double sources, shuffled properties, comments, n = 0 and special
float patterns in every field; writer cases: both flavours with and without RGB, crop_sh at every SH cut-off and a lone
NaN, degree 0, no normals, extras of every type and non-packed input; and refusals.  Each case stores its input, the
result (length, SHA-256 and dtype of the array's bytes, and for writers the header) or the name of the exception, and
`expect`: "ok" where gsx.ply reproduces it, "refuse" where it raises ValueError.  The script asserts that ply_oracle.py
reproduces every case before it writes the fixture.
"""
import importlib.util
import sys
import tempfile
import types
from pathlib import Path

import numpy as np

HERE = Path(__file__).resolve().parent
sys.path[:0] = [str(HERE.parent), str(HERE.parent.parent / "3dgsconverter_b200")]
import ply_oracle as po  # noqa: E402
import splat_codecs_oracle as sco  # noqa: E402
from make_splat_codecs_golden import import_reference_writers  # noqa: E402

from gsx.readers import parse_ply_header  # noqa: E402

TYPE_NAMES = po.TYPES
STD = po.std_order(False)
SPECIAL = np.array([0x7fc00000, 0xffc00001, 0x7f800001, 0x7fa5a5a5, 0x7f800000, 0xff800000, 0x80000000, 0x00000001,
                    0x807fffff, 0x00400000, 0x3f800000, 0xc2fe0000, 0x437f0000, 0x4f000000, 0xcf000001], np.uint32)


def ply(arr, elements=(), comments=(), fmt="binary_little_endian"):
    """A PLY file of `arr` as its vertex element, plus [(name, array)] elements after it."""
    lines = ["ply", f"format {fmt} 1.0"] + [f"comment {c}" for c in comments] + ["obj_info gsx"] * bool(comments)
    body = b""
    for name, a in (("vertex", arr), *elements):
        lines.append(f"element {name} {len(a)}")
        lines += [f"property {TYPE_NAMES[a.dtype[f].str[1:]]} {f}" for f in a.dtype.names]
        body += np.ascontiguousarray(a).tobytes()
    return ("\n".join(lines + ["end_header"]) + "\n").encode() + body


def rand_rows(names_types, n, seed):
    rng = np.random.default_rng(seed)
    a = np.zeros(n, names_types)
    for f in a.dtype.names:
        dt = a.dtype[f]
        if dt.kind == "f":
            a[f] = rng.normal(0, 2, n).astype(dt)
        elif dt.kind == "b":
            a[f] = rng.integers(0, 2, n).astype(bool)
        else:
            a[f] = rng.integers(np.iinfo(dt).min, np.iinfo(dt).max, n, endpoint=True, dtype=dt)
    return a


def std_fields(deg=3, rgb=None, prefix="", spatial_prefix=False):
    nrest = 3 * ((deg + 1) ** 2 - 1)
    out = []
    for f in STD:
        if f.startswith("f_rest_") and int(f[7:]) >= nrest:
            continue
        spatial = f in ("x", "y", "z", "nx", "ny", "nz")
        out.append(((prefix if (spatial_prefix or not spatial) else "") + f, "<f4"))
    if rgb:
        out += [(c, rgb) for c in ("red", "green", "blue")]
    return out


def specials(a, seed):
    """Every float field of `a` cycles through NaN payloads, +-inf, -0.0, subnormals and edges."""
    for k, f in enumerate(a.dtype.names):
        if a.dtype[f] == np.dtype("<f4"):
            a[f][: len(SPECIAL)] = np.roll(SPECIAL, k + seed).view(np.float32)[: len(a)]
    return a


def reader_cases():
    """{name: (flavor, file bytes, expect)}"""
    out = {}
    files = {}
    files["plain"] = ply(specials(rand_rows(std_fields(), 40, 1), 0))
    files["rgb_uchar"] = ply(rand_rows(std_fields(rgb="u1"), 30, 2))
    a = rand_rows(std_fields(rgb="<f4"), 64, 3)
    red = np.array([0, 1, 255, 255.9, 256, 300.5, -1, -1.5, -0.0, 1e10, -1e10, 2147483520.0, -2147483648.0, np.nan,
                    np.inf, -np.inf, 1e-40, 127.5, 128, 65791.25], np.float32)
    a["red"][: len(red)], a["green"][: len(red)], a["blue"][: len(red)] = red, red[::-1], np.roll(red, 7)
    files["rgb_float"] = ply(a)
    d = rand_rows([("x", "<f8"), ("y", "<f4"), ("z", "<f4"), ("red", "<f8"), ("green", "<u2"), ("blue", "<i4")]
                  + std_fields()[3:], 40, 4)
    dv = np.array([np.nan, -np.nan, np.inf, -np.inf, -0.0, 1e-320, 3.5e38, 3.4028235677973366e38, 1e-46, 1.4e-45,
                   0.1, 255.99, -1.0, 4294967296.0, 2147483648.0, -2147483649.0, 1e19], np.float64)
    d["x"][: len(dv)] = dv
    d["x"].view(np.uint64)[len(dv)] = 0x7ff0000000000123   # signalling NaN payload
    d["x"].view(np.uint64)[len(dv) + 1] = 0xfff4000020000001
    d["red"][: len(dv)] = dv[::-1]
    files["double_x_red"] = ply(d)
    i = rand_rows([(f, {"f_dc_0": "<i4", "f_dc_1": "<u4", "f_dc_2": "<i2", "opacity": "u1", "scale_0": "i1",
                        "scale_1": "<u2"}.get(f, "<f4")) for f in STD], 40, 5)
    i["f_dc_0"][:6] = [16777217, -16777217, 2147483647, -2147483648, 16777219, 0]
    i["f_dc_1"][:4] = [4294967295, 16777217, 2147483649, 4294967040]
    files["int_sources"] = ply(i)
    for deg in (0, 1, 2):
        files[f"deg{deg}"] = ply(rand_rows(std_fields(deg), 20, 6 + deg))
    for p in ("scalar_", "scal_", "scalar_scal_"):
        files[f"prefix_{p}"] = ply(rand_rows(std_fields(prefix=p), 20, 9))
    both = std_fields(prefix="scalar_scal_") + [("scalar_f_dc_0", "<f4")]
    files["prefix_both"] = ply(rand_rows(both, 20, 10))
    ex = [(f"e_{t}", "<" + t if t[1] != "1" else t) for t in TYPE_NAMES]
    files["extras"] = ply(rand_rows(std_fields(rgb="u1") + ex + [("scalar_conf", "<f4"), ("scalar_tag", "u1")], 30, 11))
    files["extras_collide"] = ply(rand_rows(std_fields() + [("scalar_dup", "<f4"), ("dup", "u1"), ("tag", "<i2"),
                                                            ("scalar_tag", "<i2")], 30, 12))
    files["extras_collide_cast"] = ply(rand_rows(std_fields() + [("scalar_dup", "<f8"), ("dup", "<i2")], 10, 13))
    cc_x = std_fields(prefix="scalar_")
    cc_x[0] = ("scalar_x", "<f8")
    files["scalar_x_double"] = ply(rand_rows(cc_x, 20, 14))
    sh = rand_rows(std_fields(rgb="u1"), 25, 15)
    perm = np.random.default_rng(16).permutation(len(sh.dtype.names))
    names = [sh.dtype.names[k] for k in perm]
    files["shuffled_comments"] = ply(sh[names].astype(np.dtype([(f, sh.dtype[f]) for f in names])),
                                     comments=("made by gsx", "second comment"))
    files["n0"] = ply(rand_rows(std_fields(rgb="u1"), 0, 17))
    files["only_some"] = ply(rand_rows([("x", "<f4"), ("opacity", "<f4"), ("green", "u1"), ("foo", "<f4")], 9, 18))
    good = files["rgb_uchar"]
    refuse = {"ascii": good.replace(b"binary_little_endian", b"ascii", 1),
              "big_endian": good.replace(b"binary_little_endian", b"binary_big_endian", 1),
              "list_property": good.replace(b"end_header", b"element face 0\nproperty list uchar int vertex_indices\n"
                                            b"end_header", 1),
              "truncated": good[:-7],
              "camera_element": ply(rand_rows(std_fields(), 5, 20), elements=[("camera", rand_rows(
                  [("fx", "<f4"), ("fy", "<f4"), ("w", "<i4")], 1, 21))]),
              "face_element": ply(rand_rows(std_fields(), 5, 22), elements=[("face", rand_rows(
                  [("a", "<i4"), ("b", "<i4"), ("c", "<i4")], 3, 23))]),
              "too_wide": ply(rand_rows(std_fields() + [(f"w{k}", "<f8") for k in range(100)], 5, 24))}
    for tag, blob in files.items():
        for flavor in ("3dgs", "cc"):
            # CC reads `dup` (int16) into the float64 column of `scalar_dup`: a cast gsx does not reproduce
            cast = tag == "extras_collide_cast" and flavor == "cc"
            out[f"read_{flavor}_{tag}"] = (flavor, blob, "refuse" if cast else "ok")
    for tag, blob in refuse.items():
        out[f"read_3dgs_refuse_{tag}"] = ("3dgs", blob, "refuse")
    return out


def writer_cases():
    """{name: (flavor, input array, crop_sh, expect)}"""
    out = {}
    arrays = {}
    arrays["std"] = specials(rand_rows(std_fields(), 40, 31), 3)
    arrays["rgb"] = rand_rows(std_fields(rgb="u1"), 40, 32)
    for last in (-1, 8, 9, 23, 24, 44):
        a = rand_rows(std_fields(), 30, 33)
        for i in range(45):
            if i > last:
                a[f"f_rest_{i}"] = 0.0
        a["f_rest_44"][3] = -0.0 if last < 44 else a["f_rest_44"][3]
        if last >= 0:
            a[f"f_rest_{last}"][:29] = 0.0   # the only non-zero value of the column is in the last row
        arrays[f"crop_{last}"] = a
    a = rand_rows(std_fields(), 30, 34)
    for i in range(45):
        a[f"f_rest_{i}"] = 0.0
    a["f_rest_30"][17] = np.nan
    arrays["crop_lone_nan"] = a
    arrays["deg0"] = rand_rows(std_fields(0, rgb="u1"), 20, 35)
    arrays["no_normals"] = rand_rows([f for f in std_fields(1) if f[0] not in ("ny", "nz")], 20, 36)
    ex = [(f"e_{t}", "<" + t if t[1] != "1" else t) for t in TYPE_NAMES]
    arrays["extras"] = rand_rows(std_fields(rgb="u1") + ex, 20, 37)
    arrays["some_fields"] = rand_rows([("opacity", "<f4"), ("x", "<f4"), ("green", "u1"), ("f_rest_3", "<f4"),
                                       ("bar", "<i2")], 11, 38)
    base = rand_rows(std_fields(rgb="u1") + [("conf", "<f4")], 25, 39)
    nd = base.dtype
    padded = np.dtype({"names": list(nd.names), "formats": [nd[f] for f in nd.names],
                       "offsets": [nd.fields[f][1] + (5 if k > 10 else 0) for k, f in enumerate(nd.names)],
                       "itemsize": nd.itemsize + 12})
    np_ = np.zeros(len(base), padded)
    for f in nd.names:
        np_[f] = base[f]
    arrays["non_packed"] = np_
    arrays["n0"] = rand_rows(std_fields(rgb="u1"), 0, 40)
    for tag, a in arrays.items():
        for flavor in ("3dgs", "cc"):
            crops = (False, True) if tag in ("std", "rgb", "deg0", "extras", "non_packed") or tag.startswith(
                "crop") else (False,)
            for crop in crops:
                out[f"write_{flavor}_{tag}{'_crop' if crop else ''}"] = (flavor, a, crop, "ok")
    refuse = {"bool": rand_rows(std_fields() + [("flag", "?")], 5, 41),
              "int64": rand_rows(std_fields() + [("id", "<i8")], 5, 42),
              "rest_f8": rand_rows([(f, "<f8" if f == "f_rest_2" else t) for f, t in std_fields()], 5, 43),
              "big_endian": rand_rows(std_fields() + [("conf", ">f4")], 5, 44)}
    for tag, a in refuse.items():
        out[f"write_3dgs_refuse_{tag}"] = ("3dgs", a, False, "refuse")
    return out


class Capture:
    file = None       # bytes the stub's PlyData.read parses
    described = None  # the array the writer handed to PlyElement.describe


def plyfile_stub():
    class Element:
        def __init__(self, name, data):
            self.name, self.data = name, data

    class PlyData:
        def __init__(self, elements=(), byte_order="="):
            self.elements = list(elements)
            assert byte_order == "<"

        @staticmethod
        def read(path):
            buf = Capture.file
            els, end = parse_ply_header(buf)
            if end > len(buf):
                raise ValueError("stub: body cut short")
            return PlyData([Element(e.name, np.frombuffer(buf, e.dtype, e.count, e.offset)) for e in els.values()],
                           "<")

        def __contains__(self, k):
            return any(e.name == k for e in self.elements)

        def __getitem__(self, k):
            return next(e for e in self.elements if e.name == k)

        def write(self, path):
            pass

    class PlyElement:
        @staticmethod
        def describe(data, name):
            Capture.described = data.copy()
            return Element(name, data)

    m = types.ModuleType("plyfile")
    m.PlyData, m.PlyElement = PlyData, PlyElement
    return m


def import_reference_ply(ref_root):
    import_reference_writers(ref_root)
    sys.modules["plyfile"] = plyfile_stub()
    ref = Path(ref_root) / "gsconverter" / "formats"
    out = {}
    for mod, cls in (("ply_3dgs", "Ply3DGSFormat"), ("ply_cc", "PlyCCFormat")):
        spec = importlib.util.spec_from_file_location(f"gsconverter.formats.{mod}", ref / f"{mod}.py")
        m = importlib.util.module_from_spec(spec)
        sys.modules[spec.name] = m
        spec.loader.exec_module(m)
        out[{"ply_3dgs": "3dgs", "ply_cc": "cc"}[mod]] = getattr(m, cls)
    return out


def record(out, name, got, raised):
    if raised is not None:
        out[f"{name}_raises"] = np.array(raised)
        return None
    b = np.ascontiguousarray(got).tobytes()
    out[f"{name}_len"] = np.array(len(b))
    out[f"{name}_sha256"] = np.array(sco.digest(b))
    out[f"{name}_dtype"] = np.array(str(got.dtype.descr))
    return b


def main(ref_root):
    ref = import_reference_ply(ref_root)
    out = {}
    with tempfile.TemporaryDirectory() as tmp:
        path = str(Path(tmp) / "f.ply")
        for name, (flavor, blob, expect) in reader_cases().items():
            out[f"{name}_file"] = np.frombuffer(blob, np.uint8)
            out[f"{name}_flavor"], out[f"{name}_expect"] = np.array(flavor), np.array(expect)
            try:
                parse_ply_header(blob)
            except ValueError:
                assert expect == "refuse"
                print(name, "refused by the device, reference not run")
                continue
            Capture.file = blob
            reader = ref[flavor]()
            got, raised = None, None
            try:
                with np.errstate(all="ignore"):
                    got = reader.read(path)
            except Exception as e:  # noqa: BLE001
                raised = type(e).__name__
                assert expect == "refuse", f"{name}: the reference raises {raised}"
            b = record(out, name, got, raised)
            if raised is None and reader.extra_elements:
                assert expect == "refuse", f"{name}: the reference keeps extra elements"
            try:
                want = po.read(blob, flavor)
            except ValueError:
                assert expect == "refuse", f"{name}: the oracle refuses a file gsx decodes"
            else:
                assert expect == "ok", f"{name}: the oracle decodes a file gsx refuses"
                assert np.ascontiguousarray(want).tobytes() == b and str(want.dtype.descr) == str(got.dtype.descr), \
                    f"{name}: the oracle differs"
            print(name, expect, None if b is None else len(b))
        for name, (flavor, a, crop, expect) in writer_cases().items():
            out[f"{name}_in"] = np.frombuffer(np.ascontiguousarray(a).tobytes(), np.uint8)
            dt = a.dtype   # as a dict, so padding between fields survives the round trip
            out[f"{name}_in_dtype"] = np.array(repr({"names": list(dt.names), "formats": [dt[f].str for f in dt.names],
                                                     "offsets": [dt.fields[f][1] for f in dt.names],
                                                     "itemsize": dt.itemsize}))
            out[f"{name}_flavor"], out[f"{name}_expect"] = np.array(flavor), np.array(expect)
            out[f"{name}_crop"] = np.array(crop)
            Capture.described = None
            with np.errstate(all="ignore"):
                ref[flavor]().write(a, path, crop_sh=crop)
            got = Capture.described
            b = record(out, name, got, None)
            try:
                want = po.write(a, flavor, crop)
            except ValueError:
                assert expect == "refuse", f"{name}: the oracle refuses records gsx encodes"
            else:
                assert expect == "ok", f"{name}: the oracle encodes records gsx refuses"
                assert np.ascontiguousarray(want).tobytes() == b and str(want.dtype.descr) == str(got.dtype.descr), \
                    f"{name}: the oracle differs"
                out[f"{name}_header"] = np.frombuffer(po.header(want), np.uint8)
            print(name, expect, len(b))
    np.savez_compressed(HERE / "g15_reference_ply_small.npz", **out)


if __name__ == "__main__":
    main(sys.argv[1])
