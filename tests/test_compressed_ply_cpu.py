"""CPU: the compressed PLY oracle against the reference's own writer output (g10), the stand-alone PLY writer, and the
argument checks of encode() / gsx_cply_pack that run before any device work."""
import ctypes as C
from pathlib import Path

import numpy as np
import pytest

import compressed_ply_oracle as cpo

GOLDEN = Path(__file__).resolve().parent / "golden" / "g10_reference_compressed_ply_small.npz"


def golden_arrays(z, tag):
    sh = z[f"{tag}_sh"] if f"{tag}_sh" in z.files else None
    return z[f"{tag}_chunk"], z[f"{tag}_vertex"], sh


@pytest.mark.parametrize("tag", ["mixed", "deg1"])
def test_oracle_reproduces_reference_golden(tag):
    z = np.load(GOLDEN)
    a = cpo.golden_inputs()[tag]
    assert cpo.digest(a) == str(z[f"{tag}_input_sha256"]), "gsx.synth no longer regenerates the golden input"
    got = cpo.encode(a, z[f"{tag}_order"])
    cpo.assert_packed_equal(got, golden_arrays(z, tag))
    assert list(got[2].dtype.names) == list(z[f"{tag}_sh_names"])


def test_golden_covers_the_edge_cases():
    z = np.load(GOLDEN)
    c = z["mixed_chunk"]
    assert np.any((c["min_x"] == c["max_x"]) & (c["min_y"] == c["max_y"]) & (c["min_z"] == c["max_z"]))
    assert len(z["mixed_sh_names"]) == 45 and len(z["deg1_sh_names"]) == 9
    assert np.any(z["mixed_vertex"]["packed_rotation"] == (512 << 20 | 512 << 10 | 512))   # the zero quaternion


def parse_ply(path):
    """Minimal binary little-endian PLY reader: (header text, {element: structured array})."""
    raw = Path(path).read_bytes()
    end = raw.index(b"end_header\n") + len(b"end_header\n")
    header = raw[:end].decode("ascii")
    types = {"float": "<f4", "uint": "<u4", "uchar": "u1"}
    elements = []
    for line in header.splitlines():
        w = line.split()
        if w[0] == "element":
            elements.append((w[1], int(w[2]), []))
        elif w[0] == "property":
            elements[-1][2].append((w[2], types[w[1]]))
    out, off = {}, end
    for name, count, fields in elements:
        dt = np.dtype(fields)
        out[name] = np.frombuffer(raw, dtype=dt, count=count, offset=off)
        off += count * dt.itemsize
    assert off == len(raw)
    return header, out


def expected_header(nc, nv, sh_names):
    lines = ["ply", "format binary_little_endian 1.0", f"element chunk {nc}"]
    lines += [f"property float {f}" for f in cpo.CHUNK_FIELDS]
    lines += [f"element vertex {nv}"] + [f"property uint {f}" for f in cpo.VERTEX_FIELDS]
    if sh_names:
        lines += [f"element sh {nv}"] + [f"property uchar {f}" for f in sh_names]
    return "\n".join(lines + ["end_header"]) + "\n"


@pytest.mark.parametrize("tag", ["mixed", "deg1", "no_sh"])
def test_write_ply_parses_back(tag, tmp_path, gsx_lib):
    from gsx.compressed_ply import write_ply
    z = np.load(GOLDEN)
    chunk, vertex, sh = golden_arrays(z, "deg1" if tag == "no_sh" else tag)
    if tag == "no_sh":
        sh = None
    write_ply(tmp_path / "out.ply", chunk, vertex, sh)
    header, el = parse_ply(tmp_path / "out.ply")
    assert header == expected_header(len(chunk), len(vertex), sh.dtype.names if sh is not None else ())
    assert np.array_equal(el["chunk"].view(np.uint32), np.ascontiguousarray(chunk).view(np.uint32))
    assert np.array_equal(el["vertex"], vertex)
    if sh is None:
        assert "sh" not in el
    else:
        assert np.array_equal(el["sh"], sh)


def test_write_ply_spelled_out_header(tmp_path, gsx_lib):
    from gsx.compressed_ply import write_ply
    chunk = np.zeros(1, dtype=[(f, "f4") for f in cpo.CHUNK_FIELDS])
    vertex = np.zeros(2, dtype=[(f, "u4") for f in cpo.VERTEX_FIELDS])
    sh = np.zeros(2, dtype=[("f_rest_0", "u1"), ("f_rest_1", "u1")])
    write_ply(tmp_path / "t.ply", chunk, vertex, sh)
    head = (tmp_path / "t.ply").read_bytes()[:1000].split(b"end_header\n")[0].decode()
    assert head == (
        "ply\nformat binary_little_endian 1.0\nelement chunk 1\n"
        "property float min_x\nproperty float min_y\nproperty float min_z\n"
        "property float max_x\nproperty float max_y\nproperty float max_z\n"
        "property float min_scale_x\nproperty float min_scale_y\nproperty float min_scale_z\n"
        "property float max_scale_x\nproperty float max_scale_y\nproperty float max_scale_z\n"
        "property float min_r\nproperty float min_g\nproperty float min_b\n"
        "property float max_r\nproperty float max_g\nproperty float max_b\n"
        "element vertex 2\nproperty uint packed_position\nproperty uint packed_rotation\n"
        "property uint packed_scale\nproperty uint packed_color\n"
        "element sh 2\nproperty uchar f_rest_0\nproperty uchar f_rest_1\n")
    assert len((tmp_path / "t.ply").read_bytes()) == len(head) + len("end_header\n") + 72 + 32 + 4


def test_encode_refuses_missing_fields(gsx_lib):
    import torch
    from gsx import compressed_ply, records
    r = records.DeviceRecords(torch.zeros((4, 3)), ("x", "y", "z"), None)
    with pytest.raises(ValueError, match="opacity"):
        compressed_ply.encode(r)


def test_cply_pack_argument_errors(gsx_lib):
    """Rejected before any device work: fake (aligned, never dereferenced) device pointers are enough."""
    p = C.c_void_p(4096)
    cols = (C.c_int32 * 14)(*range(14))
    rest = (C.c_int32 * 45)(*range(14, 59))

    def call(n, F=62, c14=cols, n_rest=45):
        return gsx_lib.gsx_cply_pack(p, n, F, p, c14, rest, n_rest, p, p, p, p, p, p, p, p, None)

    assert call(1 << 31) == -2                         # n >= 2^31
    assert call(-1) == -2
    assert call(10, F=20) == -2                        # an f_rest column beyond the row
    assert call(10, c14=(C.c_int32 * 14)(*range(13), 62)) == -2   # rot_3 beyond the row
    assert call(10, c14=(C.c_int32 * 14)(-1, *range(1, 14))) == -2
    assert call(10, n_rest=46) == -2
    assert b"out of range" in gsx_lib.gsx_last_error()
    assert call(0) == 0                                # n = 0: nothing to do
    assert gsx_lib.gsx_cply_narrow_sh(p, 10, 9, 10, p, None) == -2   # keep > width
