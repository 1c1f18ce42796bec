"""CPU: the Python restatement of the device VP8L decoder (vp8l_model.py) against Pillow's convert('RGBA'), on Pillow
files, gsx.webp's encoder output (webp_oracle.py), the SOG bundles of g14 and hand-built streams; that each stream
feature was decoded; and the streams the decoder must refuse."""
import io
import zipfile

import numpy as np
import pytest

import vp8l_model as M
import webp_oracle
from test_sog_reader_cpu import GOLDEN, blob_of, golden_cases


def sog_members() -> dict:
    z = np.load(GOLDEN)
    out = {}
    for case in golden_cases():
        if not case.startswith("writer_n300"):
            continue
        with zipfile.ZipFile(io.BytesIO(blob_of(z, case))) as zf:
            for name in zf.namelist():
                if name.endswith(".webp"):
                    out[f"{case}/{name}"] = zf.read(name)
    return out


def gsx_files() -> dict:
    return {name: webp_oracle.encode(a) for name, a in M.images(1).items()}


CASES = {**M.pillow_cases(), **M.built_cases(), **{f"gsx_{k}": v for k, v in gsx_files().items()}, **sog_members()}


@pytest.mark.parametrize("name", sorted(CASES))
def test_model_matches_pillow(name):
    """64-bit chunks: every stream goes through false starts and re-decode rounds."""
    data = CASES[name]
    assert np.array_equal(M.decode(data, chunk_bits=64), M.pillow_rgba(data)), name


def test_every_feature_is_hit():
    M.COUNTERS.clear()
    for data in CASES.values():
        M.decode(data, chunk_bits=64)
    for key in ("predictor", "cross_colour", "subtract_green", "colour_indexing", "cache", "cache_hit",
                "multi_group", "simple_code_1", "simple_code_2", "normal_code", "dist_plane", "dist_long",
                "repeat_before_first") + tuple(f"mode_{m}" for m in range(14)):
        assert M.COUNTERS.get(key, 0) > 0, key


def test_chunked_walk_paths():
    """Tiny chunks force false starts and group mismatches; max_rounds=0 forces the serial fallback."""
    data = CASES["half_m4_q100"]
    st = {}
    M.decode(data, chunk_bits=32, stats=st)
    assert st["false_starts"] + st["group_mismatches"] > 0 and st["rounds"] > 0
    st = {}
    assert np.array_equal(M.decode(data, chunk_bits=32, max_rounds=0, stats=st), M.pillow_rgba(data))
    assert st["serial_fallbacks"] == 1


def test_pillow_alpha_follows_the_vp8l_hint():
    """Pillow opens a VP8L stream whose alpha hint is 0 as RGB, and convert('RGBA') gives alpha 255 whatever the
    stream holds; a VP8X header's alpha flag changes nothing."""
    from PIL import Image
    px = [("lit", 0x40112233), ("lit", 0x00445566)]
    for flags in (None, 0x00, 0x10):
        for hint in (0, 1):
            data = M.riff(M.build(2, 1, px, alpha_hint=hint), flags, 2, 1)
            im = Image.open(io.BytesIO(data))
            assert im.mode == ("RGBA" if hint else "RGB"), (flags, hint)
            assert M.pillow_rgba(data)[0, :, 3].tolist() == ([0x40, 0x00] if hint else [255, 255])


def malformed() -> dict:
    """name -> file the decoder must refuse (Pillow refuses them too)."""
    good = CASES["half_m1_q100"]
    out = {"truncated": good[:len(good) // 2], "truncated_header": M.riff(bytes(M.build(2, 2, [("lit", 1)] * 4)[:6]))}

    def over_subscribed(w):
        w.put(0, 1), w.put(0, 1)                  # no cache, no meta codes
        w.put(0, 1), w.put(0, 4)                  # a normal code, 4 code-length code lengths
        for _ in range(4):
            w.put(1, 3)                           # four codes of length 1

    def empty(w):
        w.put(0, 1), w.put(0, 1)
        w.put(0, 1), w.put(0, 4)
        for v in (0, 0, 1, 0):                    # only length 0 is coded: 0 bits each
            w.put(v, 3)
        w.put(0, 1)

    def cache_bits_12(w):
        w.put(1, 1), w.put(12, 4)

    out["over_subscribed"] = M.riff(M.build(4, 4, [], trailer=over_subscribed))
    out["empty_code"] = M.riff(M.build(4, 4, [], trailer=empty))
    out["cache_bits_12"] = M.riff(M.build(4, 4, [], trailer=cache_bits_12))
    out["distance_before_start"] = M.riff(M.build(16, 2, [("lit", 7), ("copy", 31, 3)]))
    out["copy_past_end"] = M.riff(M.build(4, 2, [("lit", 7), ("copy", 9, 121)]))
    return out


@pytest.mark.parametrize("name", sorted(malformed()))
def test_malformed_streams_are_refused(name):
    data = malformed()[name]
    with pytest.raises(ValueError):
        M.decode(data, chunk_bits=64)
    with pytest.raises(Exception):
        M.pillow_rgba(data)
