"""CPU: the NumPy readers oracle against the reference readers' own results (g13), the binary PLY header parser, and
the argument checks of the reader entry points that run before any device work."""
import ctypes as C
from pathlib import Path

import numpy as np
import pytest

import readers_oracle as ro
import splat_codecs_oracle as sco

GOLDEN = Path(__file__).resolve().parent / "golden" / "g13_reference_readers_small.npz"


def golden_cases():
    z = np.load(GOLDEN)
    return sorted(k[: -len("_file")] for k in z.files if k.endswith("_file"))


def meta_repr(m) -> str:
    return repr(m)


@pytest.mark.parametrize("case", golden_cases())
def test_oracle_reproduces_reference_golden(case):
    z = np.load(GOLDEN)
    blob, fmt = z[f"{case}_file"].tobytes(), str(z[f"{case}_format"])
    if str(z[f"{case}_expect"]) == "refuse":
        with pytest.raises(ValueError), np.errstate(all="ignore"):
            ro.READERS[fmt](blob)
        return
    with np.errstate(all="ignore"):
        a, meta = ro.READERS[fmt](blob)
    b = np.ascontiguousarray(a).tobytes()
    assert len(b) == int(z[f"{case}_len"]) and sco.digest(b) == str(z[f"{case}_sha256"])
    assert str(a.dtype.descr) == str(z[f"{case}_dtype"])
    assert meta_repr(meta) == str(z[f"{case}_meta"])


def test_golden_covers_the_edge_cases():
    z = np.load(GOLDEN)
    cases = golden_cases()
    for fmt in ("splat", "ksplat", "spz", "cply"):
        assert any(str(z[f"{c}_format"]) == fmt and str(z[f"{c}_expect"]) == "ok" for c in cases), fmt
        if fmt != "splat":   # every byte string is a .splat file
            assert any(str(z[f"{c}_format"]) == fmt and str(z[f"{c}_expect"]) == "refuse" for c in cases), fmt
    assert str(z["ksplat_no_centres_raises"]) == "TypeError" and str(z["ksplat_bucket_past_centres_raises"]) == "IndexError"
    assert "f_rest_71" in str(z["spz_degree4_dtype"])                       # degree 4: 72 zero SH columns
    assert "'shDegree': 3" in str(z["ksplat_multisection_meta"])
    assert "uint32 packed_position" in z["cply_aliases_file"].tobytes()[:2000].decode("ascii", "replace")


def test_ply_header_parser():
    from gsx.readers import parse_ply_header
    z = np.load(GOLDEN)
    for case in golden_cases():
        if str(z[f"{case}_format"]) != "cply":
            continue
        blob = z[f"{case}_file"].tobytes()
        if case in ("cply_ascii", "cply_big_endian", "cply_duplicate"):
            with pytest.raises(ValueError):
                parse_ply_header(blob)
            continue
        els, end = parse_ply_header(blob)
        if case == "cply_no_chunk":
            assert "chunk" not in els
        elif case == "cply_truncated":
            assert end > len(blob)
        else:
            assert end == len(blob) and els["vertex"].dtype.itemsize == 16 and els["chunk"].dtype.itemsize == 72
            names = els["vertex"].dtype.names
            assert set(names) == {"packed_position", "packed_rotation", "packed_scale", "packed_color"}
    with pytest.raises(ValueError):
        parse_ply_header(b"ply\nformat binary_little_endian 1.0\nelement v 1\nproperty list uchar int i\nend_header\n")


def test_reader_argument_errors(gsx_lib):
    """Rejected before any device work: fake (never dereferenced) device pointers are enough."""
    p = C.c_void_p(4096)
    i32 = lambda *v: (C.c_int32 * len(v))(*v)  # noqa: E731
    assert gsx_lib.gsx_splat_decode(p, 1 << 31, p, p, None) == -4
    assert gsx_lib.gsx_splat_decode(p, -1, p, p, None) == -2
    assert gsx_lib.gsx_splat_decode(None, 0, None, None, None) == 0
    args = lambda **k: dict(dict(n=10, level=1, sh=9, ncent=2, fb=1, bs=8, npart=1, row=4 * 26), **k)  # noqa: E731
    def ks(**k):
        a = args(**k)
        return gsx_lib.gsx_ksplat_decode_section(p, a["n"], a["level"], a["sh"], 1.0, 1.0, p, a["ncent"], a["fb"],
                                                 a["bs"], p, a["npart"], p, a["row"], p, None)
    assert ks(level=3) == -2
    assert ks(sh=10) == -2
    assert ks(row=4 * 20) == -2                                              # too narrow for 9 SH values
    assert ks(ncent=1) == -2                                                 # the last splat's bucket has no centre
    assert ks(npart=0) == -2                                                 # splats past the full buckets
    assert ks(n=1 << 31) == -4
    assert gsx_lib.gsx_spz_decode(p, 10, 4, 0, 12, p, 71, p, None) == -2    # version
    assert gsx_lib.gsx_spz_decode(p, 10, 3, 4, 12, p, 71, p, None) == -2    # sh_dim
    assert gsx_lib.gsx_spz_decode(p, 10, 3, 0, 128, p, 71, p, None) == -2   # 1 << 128
    assert gsx_lib.gsx_spz_decode(p, 10, 3, 3, 12, p, 71, p, None) == -2    # row too narrow for 9 SH values
    coffs, voffs = i32(*range(0, 72, 4)), i32(0, 4, 8, 12)
    assert gsx_lib.gsx_cply_decode(p, 1, 72, coffs, p, 10, 16, voffs, p, 65, i32(*range(65)), 65, p, p, None) == -2
    assert gsx_lib.gsx_cply_decode(p, 1, 72, coffs, p, 10, 16, i32(0, 4, 8, 13), None, 0, None, 0, p, p, None) == -2
    assert gsx_lib.gsx_cply_decode(p, 1, 70, coffs, p, 10, 16, voffs, None, 0, None, 0, p, p, None) == -2
    assert gsx_lib.gsx_cply_decode(p, -1, 72, coffs, p, 10, 16, voffs, None, 0, None, 0, p, p, None) == -2
