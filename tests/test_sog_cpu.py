"""CPU: the NumPy SOG oracle (sog_oracle.py) against the reference writer's own output (g11), the chunk schedule, and
gsx.sog.write_sog (member order, meta.json, lossless WebP round trip)."""
import io
import json
import zipfile
from pathlib import Path

import numpy as np
import pytest

import sog_oracle as so

GOLDEN = Path(__file__).resolve().parent / "golden" / "g11_reference_sog_small.npz"
CASES = ("mixed_l0", "mixed_l7", "deg1", "sh1_80", "planar")


@pytest.fixture(scope="module")
def golden():
    return np.load(GOLDEN)


@pytest.fixture(scope="module")
def inputs():
    return so.golden_inputs()


@pytest.mark.parametrize("case", CASES)
def test_oracle_matches_reference_golden(case, golden, inputs):
    a, level, seed = inputs[case]
    assert so.digest(a) == str(golden[f"{case}_input_sha256"])
    want_tex, want_meta = so.golden_case(golden, case)
    has_fit = f"{case}_fit_centres" in golden.files
    np.random.seed(seed)
    got_tex, got_meta, _ = so.encode(a, level, codebook_fit=so.replay_fit(golden, case) if has_fit else None)
    assert so.rng_equal(np.random.get_state(), so.rng_unpack(golden[f"{case}_rng_end"]))
    assert list(got_tex) == list(want_tex)
    for name, want in want_tex.items():
        if isinstance(want, so.Hashed):
            so.check_hashed(got_tex[name], want, name)
        else:
            assert np.array_equal(got_tex[name], want), name
    assert json.dumps(got_meta) == str(golden[f"{case}_meta"])


def test_golden_stays_small():
    assert GOLDEN.stat().st_size < 700_000


def test_golden_covers_the_branches(golden, inputs):
    metas = {c: so.golden_case(golden, c)[1] for c in CASES}
    assert metas["mixed_l0"]["shN"]["bands"] == 3 and metas["deg1"]["shN"]["bands"] == 1
    assert metas["mixed_l0"]["shN"]["count"] > metas["mixed_l7"]["shN"]["count"]
    assert "shN" not in metas["planar"] and metas["planar"]["means"]["mins"][2] == metas["planar"]["means"]["maxs"][2]
    sh1 = metas["sh1_80"]
    assert len(sh1["scales"]["codebook"]) == 240 and len(sh1["sh0"]["codebook"]) == 240 and sh1["shN"]["count"] == 80
    quats = golden["mixed_l0_quats.webp"].reshape(-1, 4)
    assert np.all(quats[:18_000, 3] >= 252) and set(np.unique(quats[:18_000, 3])) == {252, 253, 254, 255}
    # the spliced scale / colour values that sit exactly between two codebook entries keep the right entry
    a = inputs["mixed_l0"][0]
    s = a[np.lexsort((a["z"], a["y"], a["x"]))]
    for fields, key in ((("scale_0", "scale_1", "scale_2"), "scales"), (("f_dc_0", "f_dc_1", "f_dc_2"), "sh0")):
        cb = np.array(metas["mixed_l0"][key]["codebook"], np.float32)
        mid = (cb[:-1] + cb[1:]) / np.float32(2)
        v = np.concatenate([s[f] for f in fields])
        ties = np.isin(v, mid[np.abs(mid - cb[:-1]) == np.abs(mid - cb[1:])])
        assert ties.sum() >= 50, key
        idx = so.quantize_to_codebook(v[ties], cb)
        assert np.all(cb[idx] > v[ties])                      # a tie takes the right-hand entry


def test_chunk_schedule_matches_reference_rule():
    from gsx.sog import chunk_schedule, texture_size
    assert texture_size(1) == (4, 4) and texture_size(80) == (12, 8) and texture_size(18_000) == (136, 136)
    assert chunk_schedule(80) == (80, [(0, 80, 80)])            # official_standard_k = 64.0: target 256, passthrough
    assert chunk_schedule(600) == (600, [(0, 600, 512)])        # 2 ** -1 * 1024 = 512.0
    assert chunk_schedule(1023) == (1023, [(0, 1023, 512)])
    cs, plan = chunk_schedule(18_000)
    assert cs == 1059 and len(plan) == 17 and {k for _, _, k in plan} == {964} and plan[-1][1] == 18_000
    assert chunk_schedule(18_000, 7)[1][0][2] == 241 and chunk_schedule(18_000, "x") == chunk_schedule(18_000, 0)
    cs, plan = chunk_schedule(10_000_000)
    assert len(plan) == 64 and plan[0][2] == 1024


def test_write_sog_members_and_meta(golden, tmp_path):
    from gsx.sog import write_sog
    for case in ("deg1", "sh1_80", "planar"):
        tex, meta = so.golden_case(golden, case)
        path = tmp_path / f"{case}.sog"
        write_sog(path, tex, meta)
        with zipfile.ZipFile(path) as zf:
            assert zf.namelist() == list(tex) + ["meta.json"]
            assert all(i.compress_type == zipfile.ZIP_STORED for i in zf.infolist())
            assert zf.read("meta.json").decode() == str(golden[f"{case}_meta"])


def test_write_sog_webp_is_lossless(golden, tmp_path):
    """Every member decodes to the exact RGBA array, except the RGB of fully transparent pixels: with the reference's
    save arguments (no exact=True) libwebp's lossless mode does not keep them.  That drops the colour indices of splats
    whose opacity byte is 0 and the label padding, in the reference's files as in these."""
    from PIL import Image
    from gsx.sog import write_sog
    tex, meta = so.golden_case(golden, "deg1")
    path = tmp_path / "deg1.sog"
    write_sog(path, tex, meta)
    transparent = 0
    with zipfile.ZipFile(path) as zf:
        for name, want in tex.items():
            img = Image.open(io.BytesIO(zf.read(name)))
            assert img.format == "WEBP" and img.size == (want.shape[1], want.shape[0])
            got = np.asarray(img.convert("RGBA"))
            assert np.array_equal(got[..., 3], want[..., 3]), name
            visible = want[..., 3] > 0
            assert np.array_equal(got[visible], want[visible]), name
            transparent += int((~visible).sum())
    assert transparent > 0
