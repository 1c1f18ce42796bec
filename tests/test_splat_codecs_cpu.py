"""CPU: the .ksplat / .spz / .splat oracle against the reference writers' own files (g12), and the argument checks of
the codec entry points that run before any device work."""
import ctypes as C
from pathlib import Path

import numpy as np
import pytest

import splat_codecs_oracle as sco

GOLDEN = Path(__file__).resolve().parent / "golden" / "g12_reference_splat_codecs_small.npz"
TAGS = ["mixed3", "content0", "content1", "content2", "fields0", "fields1", "n0", "n1", "n255", "n256", "n257"]


def oracle_files(a):
    out = {sco.ksplat_tag(c): (lambda c=c: sco.ksplat_file(a, *c)) for c in sco.KSPLAT_CASES}
    out["spz"] = lambda: sco.spz_payload(a)
    out["splat"] = lambda: sco.splat_file(a)
    return out


@pytest.mark.parametrize("tag", TAGS)
def test_oracle_reproduces_reference_golden(tag):
    z = np.load(GOLDEN)
    a = sco.golden_inputs()[tag]
    assert sco.digest(a) == str(z[f"{tag}_input_sha256"]), "gsx.synth no longer regenerates the golden input"
    with np.errstate(all="ignore"):
        for name, make in oracle_files(a).items():
            key = f"{tag}_{name}"
            if f"{key}_raises" in z.files:
                with pytest.raises(Exception) as e:
                    make()
                assert type(e.value).__name__ == str(z[f"{key}_raises"])
                continue
            got = make()
            assert len(got) == int(z[f"{key}_len"]), key
            assert sco.digest(got) == str(z[f"{key}_sha256"]), key


def test_golden_covers_the_edge_cases():
    z = np.load(GOLDEN)
    inputs = sco.golden_inputs()
    assert {k[: -len("_input_sha256")] for k in z.files if k.endswith("_input_sha256")} == set(TAGS)
    assert str(z["fields1_spz_raises"]) == "ValueError"                      # the degree-1 field set
    assert int(z["n0_ksplat_l1_shNone_b256_k5.0_len"]) == 5120
    assert int(z["n0_ksplat_l0_shNone_b256_k5.0_len"]) == 5120
    assert [sco.spz_degree(inputs[f"content{d}"]) for d in range(3)] == [0, 1, 2]
    a = inputs["mixed3"]
    assert sco.spz_degree(a) == 3 and np.isnan(a["x"]).any() and np.isnan(a["rot_1"]).any()
    m = -np.exp(a["scale_0"] + a["scale_1"] + a["scale_2"]) / (1 + np.exp(-a["opacity"]))
    assert len(m) - len(np.unique(m[~np.isnan(m)])) > 5                      # exact metric ties
    assert np.any(np.abs(a["x"] * 4096) >= 2 ** 31) and np.any(np.abs(a["x"] * 4096) >= 2 ** 23)


def test_codec_argument_errors(gsx_lib):
    """Rejected before any device work: fake (never dereferenced) device pointers are enough."""
    p = C.c_void_p(4096)
    c14 = (C.c_int32 * 14)(*range(14))
    sh = (C.c_int32 * 45)(*range(14, 59))
    assert gsx_lib.gsx_ksplat_pack(p, 1 << 31, 62, c14, sh, 24, 1, 256, 1.0, p, p, None) == -4   # n >= 2^31
    assert b"2^31" in gsx_lib.gsx_last_error()
    assert gsx_lib.gsx_ksplat_pack(p, 10, 62, c14, sh, 10, 1, 256, 1.0, p, p, None) == -2        # sh_count
    assert gsx_lib.gsx_ksplat_pack(p, 10, 20, c14, sh, 24, 1, 256, 1.0, p, p, None) == -2        # column >= F
    assert gsx_lib.gsx_ksplat_pack(p, 10, 62, c14, sh, 9, 1, 0, 1.0, p, p, None) == -2           # bucket_size
    assert gsx_lib.gsx_ksplat_pack(p, 0, 62, c14, sh, 9, 1, 256, 1.0, p, p, None) == 0
    assert gsx_lib.gsx_spz_pack(p, 1 << 31, 62, c14, sh, 15, p, None) == -4
    assert gsx_lib.gsx_spz_pack(p, 10, 62, c14, sh, 4, p, None) == -2                           # sh_dim
    assert gsx_lib.gsx_splat_pack(p, 1 << 31, 62, p, c14, p, None) == -4
    assert gsx_lib.gsx_splat_sort_keys(p, 10, 5, (C.c_int32 * 4)(0, 1, 2, 5), p, p, None) == -2
    assert gsx_lib.gsx_records_from_bytes(p, 10, 8, (C.c_int32 * 2)(0, 5), 2, p, None) == -2     # field past the row
    assert [gsx_lib.gsx_ksplat_record_bytes(lv, s) for lv, s in ((0, 0), (0, 24), (1, 9), (2, 24), (3, 9))] == \
        [44, 140, 42, 48, 33]


def test_encode_refuses_missing_fields(gsx_lib):
    import torch
    from gsx import ksplat, records, splat, spz
    r = records.DeviceRecords(torch.zeros((4, 3)), ("x", "y", "z"), None)
    for mod in (ksplat, spz, splat):
        with pytest.raises(ValueError, match="opacity"):
            mod.encode(r)
