"""CPU: the NumPy plain PLY oracle against the reference readers' and writers' own results (g15), the host half of
gsx.ply (dtypes, field tables, header text, refusals) against the same fixture, which cast branch of gsx_ply_transcode
each case reaches, and the argument checks of gsx_ply_transcode that run before any device work."""
import ctypes as C
from pathlib import Path

import numpy as np
import pytest

import ply_oracle as po
import splat_codecs_oracle as sco

GOLDEN = Path(__file__).resolve().parent / "golden" / "g15_reference_ply_small.npz"


def golden_cases(kind=None):
    z = np.load(GOLDEN)
    names = sorted(k[: -len("_expect")] for k in z.files if k.endswith("_expect"))
    return [c for c in names if kind is None or c.startswith(kind)]


def writer_input(z, case) -> np.ndarray:
    dt = np.dtype(eval(str(z[f"{case}_in_dtype"])))  # noqa: S307  (our own fixture's dtype descr)
    return np.frombuffer(z[f"{case}_in"].tobytes(), dt).copy()


def expected(z, case):
    return str(z[f"{case}_expect"])


@pytest.mark.parametrize("case", golden_cases("read_"))
def test_oracle_reader_reproduces_reference_golden(case):
    z = np.load(GOLDEN)
    blob, flavor = z[f"{case}_file"].tobytes(), str(z[f"{case}_flavor"])
    if expected(z, case) == "refuse":
        with pytest.raises(ValueError):
            po.read(blob, flavor)
        return
    a = po.read(blob, flavor)
    b = np.ascontiguousarray(a).tobytes()
    assert len(b) == int(z[f"{case}_len"]) and sco.digest(b) == str(z[f"{case}_sha256"])
    assert str(a.dtype.descr) == str(z[f"{case}_dtype"])


@pytest.mark.parametrize("case", golden_cases("write_"))
def test_oracle_writer_reproduces_reference_golden(case):
    z = np.load(GOLDEN)
    a, flavor, crop = writer_input(z, case), str(z[f"{case}_flavor"]), bool(z[f"{case}_crop"])
    if expected(z, case) == "refuse":
        with pytest.raises(ValueError):
            po.write(a, flavor, crop)
        return
    out = po.write(a, flavor, crop)
    b = np.ascontiguousarray(out).tobytes()
    assert len(b) == int(z[f"{case}_len"]) and sco.digest(b) == str(z[f"{case}_sha256"])
    assert str(out.dtype.descr) == str(z[f"{case}_dtype"])
    assert po.header(out) == z[f"{case}_header"].tobytes()


@pytest.mark.parametrize("case", golden_cases("read_"))
def test_read_plan_matches_golden(case, gsx_lib):
    """gsx.ply.read_plan: the reference's dtype, and a refusal exactly where the fixture expects one."""
    from gsx import ply
    z = np.load(GOLDEN)
    blob, flavor = z[f"{case}_file"].tobytes(), str(z[f"{case}_flavor"])
    if expected(z, case) == "refuse":
        with pytest.raises(ValueError):
            ply.read_plan(blob, flavor)
        return
    vx, dtype, table = ply.read_plan(blob, flavor)
    assert str(dtype.descr) == str(z[f"{case}_dtype"])
    assert len(table) % 4 == 0 and vx.count * dtype.itemsize == int(z[f"{case}_len"])


@pytest.mark.parametrize("case", golden_cases("write_"))
def test_write_plan_and_header_match_golden(case, gsx_lib):
    """gsx.ply.write_plan with the crop_sh cut-off of the host scan, and compressed_ply.ply_header's text."""
    from gsx import ply
    from gsx.compressed_ply import ply_header
    z = np.load(GOLDEN)
    a, flavor, crop = writer_input(z, case), str(z[f"{case}_flavor"]), bool(z[f"{case}_crop"])
    if expected(z, case) == "refuse":
        with pytest.raises(ValueError):
            ply.check_write_input(a.dtype)
            ply.write_plan(a.dtype, flavor, po.last_nonzero_rest(a) if crop else None)
        return
    out, table = ply.write_plan(a.dtype, flavor, po.last_nonzero_rest(a) if crop else None)
    assert str(out.descr) == str(z[f"{case}_dtype"]) and len(table) % 4 == 0
    assert ply_header([("vertex", len(a), out)])[0] == z[f"{case}_header"].tobytes()


def test_golden_covers_the_edge_cases():
    z = np.load(GOLDEN)
    cases = golden_cases()
    for kind in ("read_3dgs", "read_cc", "write_3dgs", "write_cc"):
        assert any(c.startswith(kind) and expected(z, c) == "ok" for c in cases), kind
    for tag in ("ascii", "big_endian", "list_property", "truncated", "camera_element", "face_element", "too_wide"):
        assert expected(z, f"read_3dgs_refuse_{tag}") == "refuse"
    for tag in ("bool", "int64", "rest_f8", "big_endian"):
        assert expected(z, f"write_3dgs_refuse_{tag}") == "refuse"
    for last in (-1, 8, 9, 23, 24, 44):
        assert f"write_cc_crop_{last}_crop" in cases
    assert "scalar_scal_f_dc_0" in str(z["read_3dgs_prefix_scalar_scal__dtype"])   # 3DGS keeps them as extras
    assert str(z["read_3dgs_n0_len"]) == "0"


CAST_BRANCHES = {"identity": lambda s, d: s == d, "int->f4": lambda s, d: s <= 5 and d == 6,
                 "f8->f4": lambda s, d: (s, d) == (7, 6), "int->u1": lambda s, d: s <= 5 and s != 1 and d == 1,
                 "f4->u1": lambda s, d: (s, d) == (6, 1), "f8->u1": lambda s, d: (s, d) == (7, 1)}


def test_golden_cases_reach_every_cast_branch(gsx_lib):
    """Each branch of transcode_one (gsx_ply.cu) is taken by some golden reader case, and identity copies of all 8
    PLY types are among them."""
    from gsx import ply
    z = np.load(GOLDEN)
    seen, identity_types = set(), set()
    for case in golden_cases("read_"):
        if expected(z, case) == "ok":
            table = ply.read_plan(z[f"{case}_file"].tobytes(), str(z[f"{case}_flavor"]))[2]
            for k in range(0, len(table), 4):
                s, d = table[k + 1], table[k + 3]
                seen |= {b for b, hit in CAST_BRANCHES.items() if hit(s, d)}
                if s == d:
                    identity_types.add(s)
    assert seen == set(CAST_BRANCHES), set(CAST_BRANCHES) - seen
    assert identity_types == set(range(8))


def test_transcode_argument_errors(gsx_lib):
    """Rejected before any device work: fake (never dereferenced) device pointers are enough."""
    p = C.c_void_p(4096)
    t = lambda *v: (C.c_int32 * len(v))(*v)  # noqa: E731
    ok = t(0, 6, 0, 6)
    f = gsx_lib.gsx_ply_transcode
    assert f(None, 0, 4, None, 4, ok, 1, None) == 0
    assert f(p, -1, 4, p, 4, ok, 1, None) == -2
    assert f(p, 1 << 31, 4, p, 4, ok, 1, None) == -4
    assert f(p, 10, 1025, p, 4, ok, 1, None) == -2                        # source row over the limit
    assert f(p, 10, 4, p, 1025, ok, 1, None) == -2                        # destination row over the limit
    assert f(p, 10, 0, p, 4, ok, 0, None) == -2
    assert f(p, 10, 4, p, 4, t(0, 6, 0, 7), 1, None) == -2                # float -> double: no such cast
    assert f(p, 10, 4, p, 4, t(0, 1, 0, 2), 1, None) == -2                # uchar -> short: no such cast
    assert f(p, 10, 4, p, 4, t(0, 8, 0, 6), 1, None) == -2                # type 8 does not exist
    assert f(p, 10, 4, p, 4, t(1, 6, 0, 6), 1, None) == -2                # source field past the row
    assert f(p, 10, 4, p, 6, t(0, 6, 3, 6), 1, None) == -2                # destination field past the row
    assert f(p, 10, 8, p, 8, t(0, 6, 0, 6, 4, 6, 2, 6), 2, None) == -2    # overlapping destination fields
    assert f(p, 10, 8, p, 8, None, 1, None) == -2
    assert f(p, 10, 8, p, 8, ok, 1025, None) == -2


def test_encode_and_decode_refuse_on_the_host(gsx_lib, tmp_path):
    from gsx import ply
    with pytest.raises(ValueError):
        ply.read_plan(b"ply\nformat binary_little_endian 1.0\nelement vertex 1\nend_header\n")   # no properties
    with pytest.raises(ValueError):
        ply.read_plan(b"", "3dgs")
    with pytest.raises(ValueError):
        ply.write_plan(np.dtype([("x", "<f4")]), "blender")
    with pytest.raises(ValueError):
        ply.write_plan(np.dtype([("x", "<f4")] + [(f"w{k}", "<f8") for k in range(128)]), "3dgs")   # 1028-byte rows
