"""The .splat, .ksplat and .spz writer kernels (csrc/gsx_splat_codecs.cu), path by path, with NaN, +-inf and the
values on every rounding, clipping and bucketing boundary.

Each case has a seeded builder.  An unmarked CPU test restates the dispatch (the byte alignment of every staged store,
the partial last CTA, the bucket of each splat, the SH degree the mask implies) and checks in NumPy that the case
reaches the branch it is named after.  A `gpu` test asserts byte equality with splat_codecs_oracle (ksplat_file,
spz_payload, splat_order, splat_file), or with the NumPy expression itself where the test calls an entry point
directly (gsx_codec_sh_mask, gsx_ksplat_centres, gsx_ksplat_pack over every float32 bit pattern)."""
import ctypes as C
import struct

import numpy as np
import pytest

import splat_codecs_oracle as sco

ROWS = 128                    # kThreads: rows per CTA of every pack kernel
F32 = np.float32
NAN, INF = F32(np.nan), F32(np.inf)


def f32(bits):
    return np.uint32(bits).view(np.float32)


def assert_same(got: bytes, want: bytes, what: str):
    assert len(got) == len(want), f"{what}: {len(got)} bytes, want {len(want)}"
    d = np.flatnonzero(np.frombuffer(got, np.uint8) != np.frombuffer(want, np.uint8))
    assert d.size == 0, f"{what}: {d.size} bytes differ, first at {d[:8]}"


def device_records(a, cuda):
    from gsx import records
    return records.DeviceRecords.from_structured(a, cuda)


# ------------------------------------------------------------------------------------------------ SPZ sizes
SPZ_NS = [3 * ROWS + r for r in range(16)] + [1, 127, 128, 129]
SPZ_SECTIONS = {"pos": (0, 9), "alpha": (9, 1), "colour": (10, 3), "scale": (13, 3), "rot": (16, 4)}


def spz_sections(n, sh_dim):
    """{section: (byte offset in the body, bytes per splat)}; the body starts 16-byte aligned after the header."""
    out = {k: (n * s, w) for k, (s, w) in SPZ_SECTIONS.items()}
    if sh_dim:
        out["sh"] = (20 * n, 3 * sh_dim)
    return out


def spz_size_case(n, degree):
    from gsx import synth
    return synth.structured(n, "mixed", sh_degree=degree)


@pytest.mark.parametrize("degree", [0, 3])
def test_spz_sizes_reach_every_alignment(degree):
    sh_dim = {0: 0, 3: 15}[degree]
    assert {n % 16 for n in SPZ_NS} == set(range(16))
    seen = {}
    for n in SPZ_NS:
        last = (n - 1) // ROWS * ROWS                              # the last CTA's first row
        for k, (off, w) in spz_sections(n, sh_dim).items():
            seen.setdefault(k, set()).add((off + last * w) % 16)   # where the last CTA's store starts
    for k, (off, w) in spz_sections(16, sh_dim).items():
        step = off // 16                                           # section start = n * step
        assert seen[k] == {(r * step) % 16 for r in range(16)}, k  # every alignment n mod 16 can give it
    assert sum(n % ROWS != 0 for n in SPZ_NS) >= 18 and max(SPZ_NS) > ROWS   # a partial last CTA, several CTAs
    for n in SPZ_NS[:16]:
        assert spz_size_case(n, degree).dtype.names.count("f_rest_44") == (degree == 3)
    if degree == 3:
        assert sco.spz_degree(spz_size_case(SPZ_NS[0], 3)) == 3


@pytest.mark.gpu
@pytest.mark.parametrize("n", SPZ_NS)
@pytest.mark.parametrize("degree", [0, 3])
def test_spz_pack_every_alignment(degree, n, cuda, gsx_lib):
    from gsx import spz
    a = spz_size_case(n, degree)
    enc = spz.encode(device_records(a, cuda))
    assert enc.payload.data_ptr() % 16 == 0 and enc.sh_degree == degree
    with np.errstate(all="ignore"):
        assert_same(enc.to_host(), sco.spz_payload(a), f"spz n={n} degree={degree}")


# ------------------------------------------------------------------------------------------------ SPZ values
SPZ_QUATS = {   # (rot_0 = w, rot_1, rot_2, rot_3)
    "tie2_xy": (0.0, 0.5, 0.5, 0.0), "tie2_neg": (0.5, 0.0, -0.5, 0.0), "tie2_wz": (-0.5, 0.0, 0.0, 0.5),
    "tie4": (0.5, 0.5, 0.5, 0.5), "tie4_signs": (-0.5, 0.5, -0.5, -0.5), "tie3": (0.0, -0.3, 0.3, 0.3),
    "nan_w": (np.nan, 0.1, 0.2, 0.3), "nan_x": (0.1, np.nan, 0.2, 0.3), "nan_y": (0.1, 0.2, np.nan, 0.3),
    "nan_z": (0.1, 0.2, 0.3, np.nan), "zero": (0.0, 0.0, 0.0, 0.0), "neg_zero": (-0.0, 0.0, -0.0, -0.0),
    "tiny": (1e-30, 0.0, 0.0, 0.0), "inf_w": (np.inf, 0.0, 0.0, 0.0), "inf_x": (0.0, -np.inf, 0.0, 0.0),
    "inf_y": (0.0, 0.0, np.inf, 0.5), "inf_z": (0.5, 0.0, 0.0, -np.inf)}   # inf / inf: a NaN in one slot only
SPZ_POSITIONS = [2048.0, -2048.0, 2047.999755859375, -2047.999755859375, 2048.000244140625, -2048.000244140625,
                 4096.0, -4096.0, 524287.9, 524288.0, -524288.0, -524288.25, 1e6, -1e6, 1e30, np.nan, np.inf,
                 -np.inf, 0.5 / 4096, 1.5 / 4096, -0.5 / 4096, -0.0]
SPZ_OPACITIES = [20.0, -20.0, 20.5, -20.5, 19.99, -19.99, 100.0, -100.0, np.nan, np.inf, -np.inf, 0.0, -0.0]


def spz_sh_values():
    """v with v * 128 + 128 = q exactly on both sides of every bucket edge of the 5-bit (8) and 4-bit (16) columns,
    rint ties (q + 0.5) next to them, negatives below the clip and past int32."""
    q = [8 * k - 4 + d for k in range(-1, 34) for d in (-1, 0)] + [16 * k - 8 + d for k in range(-1, 18) for d in (-1, 0)]
    q += [8 * k - 4.5 for k in range(0, 33, 4)] + [16 * k - 8.5 for k in range(0, 17, 3)] + [-1000.0, 300.0]
    v = [(x - 128.0) / 128.0 for x in q] + [1e10, -1e10, np.nan, np.inf, -np.inf, -0.0]
    return np.array(v, np.float32)


SPZ_EDGE_N = 4096


def spz_edge_case():
    """4 096 SH-3 rows: the quaternions above, positions, opacities and SH values in the first rows (well inside the
    vector part of NumPy's casts), the rest random."""
    from gsx import synth
    a = synth.structured(SPZ_EDGE_N, "mixed")
    for k, q in enumerate(SPZ_QUATS.values()):
        for i in range(4):
            a[f"rot_{i}"][k] = q[i]
    for k, v in enumerate(SPZ_POSITIONS):
        a[("x", "y", "z")[k % 3]][40 + k] = v
        a[("x", "y", "z")[(k + 1) % 3]][90 + k] = -v if v == v else v
    a["opacity"][140:140 + len(SPZ_OPACITIES)] = SPZ_OPACITIES
    sh = spz_sh_values()
    for k, v in enumerate(sh):
        for i in range(45):
            a[f"f_rest_{i}"][200 + k] = v
    return a


def spz_sh_byte(v, bs):
    with np.errstate(all="ignore"):
        q = np.round(np.float32(v) * 128.0 + 128.0).astype(np.int32)
        return np.clip((q + bs // 2) // bs * bs, 0, 255).astype(np.uint8)


def test_spz_edge_case_reaches_its_paths():
    a = spz_edge_case()
    assert sco.spz_degree(a) == 3
    sh = spz_sh_values()
    with np.errstate(all="ignore"):
        t = sh * np.float32(128.0) + np.float32(128.0)
    finite = t[np.isfinite(t)]
    for bs in (8, 16):                                             # both sides of an edge of each bucket width
        q = finite[finite == np.round(finite)].astype(np.int64)
        assert ((q + bs // 2) % bs == 0).sum() >= 10 and ((q + bs // 2) % bs == bs - 1).sum() >= 10
    assert (finite - np.floor(finite) == 0.5).sum() >= 10 and (finite < 0).sum() >= 4
    assert not np.array_equal(spz_sh_byte(sh, 8), spz_sh_byte(sh, 16))   # the two widths differ on these values
    q = np.stack([a[f"rot_{i}"] for i in range(4)], 1)[:len(SPZ_QUATS)]
    with np.errstate(all="ignore"):
        r = np.abs(np.stack([q[:, 1], q[:, 2], q[:, 3], q[:, 0]], 1) / np.sqrt((q * q).sum(1) + 1e-9)[:, None])
    ties = [(row == np.nanmax(row)).sum() for row in r if not np.isnan(row).any()]
    assert {2, 3, 4} <= set(ties)                                  # argmax ties: the first maximum wins
    first_nan = [int(np.flatnonzero(np.isnan(row))[0]) for row in r if np.isnan(row).any()]
    assert set(first_nan) == {0, 1, 2, 3} and len(first_nan) == 8  # the first NaN wins, in every slot
    with np.errstate(all="ignore"):
        p = np.round(np.array(SPZ_POSITIONS, np.float32) * 4096)
    assert (p == 2 ** 23).any() and (p == -2 ** 23 - 1).any()      # the 24-bit wrap, both signs
    assert (np.abs(p) >= 2 ** 31).any() and np.isnan(p).any()     # int32 overflow and NaN -> INT32_MIN
    assert ((np.array(SPZ_OPACITIES) == 20) | (np.array(SPZ_OPACITIES) == -20)).sum() == 2
    assert 200 + len(sh) < SPZ_EDGE_N - 64


@pytest.mark.gpu
def test_spz_pack_value_edges(cuda, gsx_lib):
    from gsx import spz
    a = spz_edge_case()
    with np.errstate(all="ignore"):
        assert_same(spz.encode(device_records(a, cuda)).to_host(), sco.spz_payload(a), "spz edges")


# ------------------------------------------------------------------------------------------------ ksplat pack
KSPLAT_LEVELS = [0, 1, 2, 3, 65535]
KSPLAT_CASES = {"bucket1": (1, 1000), "bucket7_whole": (7, 7 * 150), "bucket7_partial": (7, 7 * 150 + 1),
                "bucket256_whole": (256, 1024), "bucket256_partial": (256, 1001), "bucket_past_n": (5000, 1001)}
SF = np.float32(32767 / (5.0 / 2.0))      # sf_inv of the default block size


def tie_offsets():
    """float32 d with d * SF exactly m + 0.5 (round half to even decides), for odd and even m of both signs, and d
    with rint(d * SF) exactly on and one past each clip end (-32767, 32768)."""
    out = []
    for m in list(range(-30001, 30000, 997)) + [-32768, -32767, 32767, 32768]:
        d0 = np.float32((m + 0.5) / float(SF))
        for k in range(-4, 5):
            d = np.float32(d0 + np.float32(k) * np.spacing(d0))
            if d * SF == np.float32(m + 0.5):
                out.append(d)
                break
    for want in (-32768, -32767, 32768, 32769):
        d0 = np.float32(want / float(SF))
        for k in range(-4, 5):
            d = np.float32(d0 + np.float32(k) * np.spacing(d0))
            if np.round(d * SF) == want:
                out.append(d)
                break
    return np.array(out, np.float32)


def ksplat_case(name):
    """SH-2 rows whose buckets span [-10, 10] on every axis, so the centre is 0 and the inner rows sit on rint ties,
    on and past both clip ends; one NaN position; level-2 SH at and past the clip ends."""
    from gsx import synth
    bs, n = KSPLAT_CASES[name]
    a = synth.structured(n, "mixed", sh_degree=2)
    pool = np.concatenate([tie_offsets(), np.array([-10.0, 10.0, -2.5, 2.5, 0.0, -0.0], np.float32)])
    for k, ax in enumerate("xyz"):
        v = np.resize(np.roll(pool, 7 * k), n)
        if bs >= 3:
            starts = np.arange(0, n, bs)
            ends = np.minimum(starts + bs, n) - 1
            many = ends - starts >= 2
            v[starts[many]], v[ends[many]] = -10.0, 10.0
        a[ax] = v
    a["y"][n // 2] = np.nan
    for k, v in enumerate((-2.0, 2.0, -2.01, 2.01, 1e6, -1e6, np.nan, np.inf, -np.inf, 255.5, 256.0, -1.0)):
        a[f"f_rest_{(5 * k) % 24}"][3 * k + 1] = v
    return a, bs


def ksplat_quantised(a, bs):
    """(x - c) * sf of every axis before rint, as the oracle computes it, with its bucket centres."""
    n = len(a)
    starts = np.arange(0, n, bs)
    with np.errstate(all="ignore"):
        out = []
        for ax in "xyz":
            v = a[ax]
            c = ((np.minimum.reduceat(v, starts) + np.maximum.reduceat(v, starts)) / 2.0).astype(np.float32)
            out.append((v - c[np.arange(n) // bs]) * SF)
    return np.concatenate(out)


@pytest.mark.parametrize("name", list(KSPLAT_CASES))
def test_ksplat_case_reaches_its_paths(name):
    a, bs = ksplat_case(name)
    n = len(a)
    assert (n % bs == 0) == name.endswith("whole") or name == "bucket1"
    if name == "bucket_past_n":
        assert bs > n                                              # one partial bucket
    p = ksplat_quantised(a, bs)
    fin = p[np.isfinite(p)]
    q = np.round(fin) + 32767
    if bs > 1:
        half = fin[fin - np.floor(fin) == 0.5]
        assert len(half) >= 20 and (np.floor(half) % 2 == 0).any() and (np.floor(half) % 2 == 1).any()
        assert (q < 0).any() and (q > 65535).any() and (q == 0).any() and (q == 65535).any()
    else:
        assert (q == 32767).all()                                  # each splat is its own bucket's centre
    assert np.isnan(p).any()
    sh = np.stack([a[f"f_rest_{j}"] for j in range(24)], 1)
    with np.errstate(all="ignore"):
        t = (sh - -2.0) / 4.0 * 255
    assert (t == 0).any() and (t == 255).any() and (t < 0).any() and (t > 255).any()
    assert n > 2 * ROWS and n % ROWS != 0 or n % ROWS == 0


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(KSPLAT_CASES))
def test_ksplat_pack_levels_and_buckets(name, cuda, gsx_lib):
    from gsx import ksplat
    a, bs = ksplat_case(name)
    r = device_records(a, cuda)
    recs = {}
    for lv in KSPLAT_LEVELS:
        enc = ksplat.encode(r, lv, None, bs)
        with np.errstate(all="ignore"):
            assert_same(enc.to_host(), sco.ksplat_file(a, lv, None, bs), f"{name} level {lv}")
        recs[lv] = enc.records.cpu().numpy()
    assert np.array_equal(recs[65535], recs[3])


# ------------------------------------------------------------------------------------------------ every float32
EVERY_ROWS = 1 << 24          # rows per launch


def _bits(start, cnt, cuda):
    """The float32 patterns start .. start + cnt - 1 (as uint32) on the device."""
    import torch
    b = torch.arange(start, start + cnt, dtype=torch.int64, device=cuda)
    return torch.where(b < (1 << 31), b, b - (1 << 32)).to(torch.int32).view(torch.float32)


def _astype_threads(x, dtype):
    """x.astype(dtype) in slices on every CPU: NumPy's float32 -> float16 cast is a scalar loop of ~80 ns per value,
    and the cast releases the GIL."""
    import os
    from concurrent.futures import ThreadPoolExecutor
    out = np.empty(len(x), dtype)
    step = 1 << 20

    def cast(s):
        with np.errstate(all="ignore"):
            out[s:s + step] = x[s:s + step].astype(dtype)
    with ThreadPoolExecutor(min(len(os.sched_getaffinity(0)), 32)) as ex:
        list(ex.map(cast, range(0, len(x), step)))
    return out


def _ksplat_pack_raw(rows, n, level, sh_count, centres, out):
    from gsx import _abi
    from gsx._abi import _ptr, _stream
    F = rows.shape[1]
    c14 = (C.c_int32 * 14)(*[k % F for k in range(14)])
    csh = (C.c_int32 * max(sh_count, 1))(*range(sh_count))
    rc = _abi.lib.gsx_ksplat_pack(_ptr(rows), n, F, c14, csh, sh_count, level, EVERY_ROWS, float(SF), _ptr(centres),
                                  _ptr(out), _stream())
    _abi.check(rc, "gsx_ksplat_pack")


def test_every_float32_layouts():
    """The record bytes the two exhaustive tests read: level-1 rotations (4 x float16 at bytes 12..19, stored with no
    arithmetic) and level >= 3 SH (24 x uint8 at bytes 24..47, the raw cast)."""
    l1 = [("pos", "<u2", 3), ("scale", "<f2", 3), ("rot", "<f2", 4), ("color", "u1", 4)]
    assert np.dtype([(k, t, (c,)) for k, t, c in l1]).fields["rot"][1] == 12
    l3 = [("pos", "<u2", 3), ("scale", "<f2", 3), ("rot", "<f2", 4), ("color", "u1", 4), ("sh", "u1", 24)]
    dt = np.dtype([(k, t, (c,)) for k, t, c in l3])
    assert dt.fields["sh"][1] == 24 and dt.itemsize == 48
    x = np.array([f32(0x7F800001), f32(0xFF800001), f32(0x7FC00000), f32(0x7FA00000)] * 8, np.float32)
    assert list(x.astype(np.float16).view(np.uint16)[:4]) == [0x7C01, 0xFC01, 0x7E00, 0x7D00]   # NaN: payload >> 13
    with np.errstate(all="ignore"):
        for n in range(1, 66):                                      # uint8: the low byte of the int32 conversion
            y = np.resize(np.array([np.nan, np.inf, -np.inf, 300.0, -1.0, 3e9, -3e9, 255.9, 65536.5], np.float32), n)
            i32 = np.where(np.isfinite(y) & (np.abs(y) < 2 ** 31), np.nan_to_num(y), -2 ** 31).astype(np.int64)
            assert np.array_equal(y.astype(np.uint8), (i32 & 0xFF).astype(np.uint8)), n


@pytest.mark.gpu
def test_float16_cast_every_float32(cuda, gsx_lib):
    """Every float32 bit pattern through the level-1 rotation fields of gsx_ksplat_pack, 2^24 rows (2^26 values) per
    launch, against astype(np.float16) on the host: NaN payloads included."""
    import torch
    from gsx.hostcopy import to_host
    rows = torch.zeros((EVERY_ROWS, 14), dtype=torch.float32, device=cuda)
    centres = torch.zeros((1, 3), dtype=torch.float32, device=cuda)
    out = torch.empty((EVERY_ROWS, 24), dtype=torch.uint8, device=cuda)
    per = 4 * EVERY_ROWS
    bad, start = 0, 0
    while start < (1 << 32):
        rows[:, 10:14] = _bits(start, per, cuda).view(EVERY_ROWS, 4)
        _ksplat_pack_raw(rows, EVERY_ROWS, 1, 0, centres, out)
        got = to_host(out[:, 12:20].contiguous()).reshape(-1).view(np.uint16)
        x = np.arange(start, start + per, dtype=np.int64).astype(np.uint32).view(np.float32)
        want = _astype_threads(x, np.float16).view(np.uint16)
        bad += int(np.count_nonzero(got != want))
        start += per
    assert bad == 0, f"{bad} of 2^32 float32 -> float16 casts differ from NumPy"


@pytest.mark.gpu
def test_uint8_cast_every_float32(cuda, gsx_lib):
    """Every float32 bit pattern through the 24 raw SH bytes of a level-3 record (gsx_ksplat_pack), 2^24 rows per
    launch, against astype(np.uint8) on the host."""
    import torch
    from gsx.hostcopy import to_host
    rows = torch.zeros((EVERY_ROWS, 24), dtype=torch.float32, device=cuda)
    centres = torch.zeros((1, 3), dtype=torch.float32, device=cuda)
    out = torch.empty((EVERY_ROWS, 48), dtype=torch.uint8, device=cuda)
    bad, start = 0, 0
    while start < (1 << 32):
        cnt = min(24 * EVERY_ROWS, (1 << 32) - start)
        k = -(-cnt // 24)
        flat = rows.view(-1)
        flat[:cnt] = _bits(start, cnt, cuda)
        flat[cnt:24 * k] = 0.0
        _ksplat_pack_raw(rows, k, 3, 24, centres, out)
        got = to_host(out[:k, 24:48].contiguous()).reshape(-1)[:cnt]
        step = 1 << 26
        for s in range(0, cnt, step):                              # the host side in 2^26-value slices
            e = min(s + step, cnt)
            x = np.arange(start + s, start + e, dtype=np.int64).astype(np.uint32).view(np.float32)
            with np.errstate(all="ignore"):
                bad += int(np.count_nonzero(got[s:e] != x.astype(np.uint8)))
        start += cnt
    assert bad == 0, f"{bad} of 2^32 float32 -> uint8 casts differ from NumPy"


# ------------------------------------------------------------------------------------------------ SH column mask
MASK_KINDS = {"nan": NAN, "subnormal": f32(1), "neg_zero": F32(-0.0)}
MASK_PLACES = {"row0": (545, 0), "partial_warp_last": (100, 99), "tail_256k_33": (256 * 3 + 33, 256 * 3 + 32)}
MASK_F = 47
MASK_COLS = (np.arange(45)[::-1] + 2).astype(np.int32)      # f_rest_k lives in row column MASK_COLS[k]


def mask_case(kind, place, col):
    n, row = MASK_PLACES[place]
    rows = np.zeros((n, MASK_F), np.float32)
    rows[:, :2] = 1.0                                          # non-SH columns, never read
    rows[row, MASK_COLS[col]] = MASK_KINDS[kind]
    return rows


def mask_structured(kind, place, col):
    from gsx import synth
    n, row = MASK_PLACES[place]
    a = synth.structured(n, "mixed")
    for i in range(45):
        a[f"f_rest_{i}"] = 0.0
    a[f"f_rest_{col}"][row] = MASK_KINDS[kind]
    return a


def ksplat_degree(a):
    """The SH degree KSplatFormat.write stores (section header byte 40), from the oracle's file."""
    return struct.unpack_from("<H", sco.ksplat_file(a, 0), 4096 + 40)[0]


@pytest.mark.parametrize("place", list(MASK_PLACES))
@pytest.mark.parametrize("kind", list(MASK_KINDS))
def test_mask_case_reaches_its_path(kind, place):
    n, row = MASK_PLACES[place]
    warp0 = row // 32 * 32
    if place == "row0":
        assert row == 0 and n % 256 != 0
    else:
        assert row == n - 1 and n - warp0 < 32                     # the last row of a partial warp
    if place == "tail_256k_33":
        assert n % 256 == 33 and n > 256
    v = MASK_KINDS[kind]
    assert bool(v != 0) == (kind != "neg_zero") and (kind != "subnormal" or (v > 0 and v < np.finfo(F32).tiny))
    want = {"nan": (2, 1), "subnormal": (2, 1), "neg_zero": (0, 0)}[kind]
    for col in (3, 12, 30):                                        # degree by column: ksplat (0..8 | 9..23), SPZ (last)
        a = mask_structured(kind, place, col)
        k, s = ksplat_degree(a), sco.spz_degree(a)
        assert k == (0 if kind == "neg_zero" or col > 8 else 1) and s == {3: want[1], 12: want[0], 30: 3 * want[1]}[col]


@pytest.mark.gpu
@pytest.mark.parametrize("place", list(MASK_PLACES))
@pytest.mark.parametrize("kind", list(MASK_KINDS))
def test_codec_sh_mask_lone_value_per_column(kind, place, cuda, gsx_lib):
    import torch
    from gsx import _abi, ksplat, spz
    from gsx._abi import _ptr, _stream
    n, _ = MASK_PLACES[place]
    cols = (C.c_int32 * 45)(*MASK_COLS.tolist())
    mask = torch.empty(1, dtype=torch.int64, device=cuda)
    for col in range(45):
        rows = torch.from_numpy(mask_case(kind, place, col)).to(cuda)
        _abi.check(_abi.lib.gsx_codec_sh_mask(_ptr(rows), n, MASK_F, cols, 45, _ptr(mask), _stream()), "sh_mask")
        got = int(mask.cpu().numpy().view(np.uint64)[0])
        assert got == (0 if kind == "neg_zero" else 1 << col), (col, hex(got))
        a = mask_structured(kind, place, col)
        r = device_records(a, cuda)
        assert ksplat.encode(r, 0).sh_degree == ksplat_degree(a), col
        assert spz.sh_degree(r) == sco.spz_degree(a), col


# ------------------------------------------------------------------------------------------------ bucket centres
CENTRE_PAIRS = {   # (lo, hi)
    "nan_lo": (f32(0x7FC00123), F32(1.0)), "nan_hi": (F32(1.0), f32(0xFFC00456)),
    "nan_both": (f32(0x7FC00123), f32(0xFFD00456)), "snan_lo_qnan_hi": (f32(0x7F800005), f32(0x7FC00777)),
    "qnan_lo_snan_hi": (f32(0xFFC00009), f32(0x7F800003)), "snan_hi": (F32(-2.0), f32(0xFF800011)),
    "inf_neg_inf": (INF, -INF), "neg_inf_inf": (-INF, INF), "inf": (INF, F32(5.0)),
    "overflow": (F32(3e38), F32(3e38)), "neg_overflow": (F32(-3e38), F32(-3.4e38)),
    "max_neg_max": (F32(3.4028235e38), F32(-3.4028235e38)), "neg_zeros": (F32(-0.0), F32(-0.0)),
    "mixed_zeros": (F32(-0.0), F32(0.0)), "odd_sum": (f32(1), f32(0)), "plain": (F32(-1.25), F32(3.5))}


def centres_case():
    """[64, 3] bounds: every pair above in each of the three axes (rows 0 .. 15, axis k shifted by k rows), the rest
    random."""
    rng = np.random.default_rng(7)
    lo = rng.normal(0, 10, (64, 3)).astype(np.float32)
    hi = lo + rng.uniform(0, 5, (64, 3)).astype(np.float32)
    pairs = list(CENTRE_PAIRS.values())
    for ax in range(3):
        for k, (l, h) in enumerate(pairs):
            lo[(k + ax) % len(pairs), ax], hi[(k + ax) % len(pairs), ax] = l, h
    return lo, hi


def numpy_centres(lo, hi):
    with np.errstate(all="ignore"):
        return ((lo + hi) / 2.0).astype(np.float32)


def test_centres_case_reaches_its_paths():
    lo, hi = centres_case()
    c = numpy_centres(lo, hi).view(np.uint32)[:16, 0]
    names = list(CENTRE_PAIRS)
    bits = lambda k: dict(zip(names, c))[k]   # noqa: E731
    assert bits("nan_both") == 0x7FC00123 and bits("snan_lo_qnan_hi") == 0x7FC00005   # lo's NaN wins, quieted
    assert bits("qnan_lo_snan_hi") == 0xFFC00009 and bits("nan_hi") == 0xFFC00456 and bits("snan_hi") == 0xFFC00011
    assert bits("inf_neg_inf") == 0xFFC00000 and bits("neg_inf_inf") == 0xFFC00000     # x86's default NaN
    assert bits("overflow") == 0x7F800000 and bits("neg_overflow") == 0xFF800000
    assert bits("max_neg_max") == 0 and bits("neg_zeros") == 0x80000000 and bits("odd_sum") == 0


@pytest.mark.gpu
def test_ksplat_centres_nan_and_overflow(cuda, gsx_lib):
    import torch
    from gsx import _abi
    from gsx._abi import _ptr, _stream
    lo, hi = centres_case()
    lt, ht = torch.from_numpy(lo).to(cuda), torch.from_numpy(hi).to(cuda)
    out = torch.full((64, 3), 7.0, dtype=torch.float32, device=cuda)
    _abi.check(_abi.lib.gsx_ksplat_centres(_ptr(lt), _ptr(ht), 64, _ptr(out), _stream()), "gsx_ksplat_centres")
    got, want = out.cpu().numpy().view(np.uint32), numpy_centres(lo, hi).view(np.uint32)
    bad = np.argwhere(got != want)
    assert bad.size == 0, [(tuple(i), hex(got[tuple(i)]), hex(want[tuple(i)])) for i in bad[:6]]


# ------------------------------------------------------------------------------------------------ .splat
SPLAT_N = 3000


def splat_metric_case():
    """Rows whose metric exp(s0 + s1 + s2) * sigmoid(opacity) is 0 from an exp underflow and from a zero sigmoid,
    subnormal, +inf and NaN (inf * 0, NaN scale, NaN opacity), each class tied many times and scattered over the
    cloud; zero-norm, NaN and infinite quaternions."""
    from gsx import synth
    a = synth.structured(SPLAT_N, "mixed", sh_degree=0)
    rng = np.random.default_rng(11)
    rows = rng.permutation(SPLAT_N)
    classes = {"zero_exp": (-60.0, -60.0, 0.0, 0.3), "zero_sigmoid": (0.1, 0.2, 0.3, -200.0),
               "zero_both": (-80.0, -80.0, 0.0, -np.inf), "subnormal": (-45.0, -45.0, -0.5, 0.0),
               "subnormal_tie": (-45.0, -45.0, -0.5, 0.0), "inf": (50.0, 50.0, 0.0, 0.0),
               "inf_opaque": (90.0, 0.0, 0.0, np.inf), "nan_inf_zero": (50.0, 50.0, 0.0, -np.inf),
               "nan_scale": (np.nan, 0.0, 0.0, 0.0), "nan_opacity": (0.0, 0.0, 0.0, np.nan),
               "ties": (-1.0, -2.0, -3.0, 0.25)}
    for k, vals in enumerate(classes.values()):
        sel = rows[40 * k:40 * k + 40]
        for f, v in zip(("scale_0", "scale_1", "scale_2", "opacity"), vals):
            a[f][sel] = v
    for k, q in enumerate(((0, 0, 0, 0), (-0.0, 0, 0, -0.0), (np.nan, 0, 0, 1), (np.inf, 0, 0, 0), (1e-30, 0, 0, 0))):
        sel = rows[1000 + 20 * k:1020 + 20 * k]
        for i in range(4):
            a[f"rot_{i}"][sel] = q[i]
    return a


def splat_metric(a):
    with np.errstate(all="ignore"):
        return np.exp(a["scale_0"] + a["scale_1"] + a["scale_2"]) * (1.0 / (1.0 + np.exp(-a["opacity"])))


def test_splat_metric_case_reaches_its_paths():
    a = splat_metric_case()
    m = splat_metric(a)
    ssum = a["scale_0"] + a["scale_1"] + a["scale_2"]
    zero = m == 0
    assert (zero & (ssum < -104)).sum() >= 40 and (zero & (a["opacity"] < -100)).sum() >= 40
    assert ((-m).view(np.uint32)[zero] == 0x80000000).all()        # -metric of a zero is -0.0: folded onto +0.0
    sub = (m > 0) & (m < np.finfo(np.float32).tiny)
    assert sub.sum() >= 80 and len(np.unique(m[sub])) == 1        # subnormal metrics, all tied
    assert np.isposinf(m).sum() >= 80 and np.isnan(m).sum() >= 120
    with np.errstate(over="ignore"):
        assert (np.isnan(m) & np.isposinf(np.exp(ssum))).sum() >= 40   # inf * 0
    order = sco.splat_order(a)
    assert np.isnan(m[order[-120:]]).all()                         # NaN last, in index order
    r = np.stack([a[f"rot_{i}"] for i in range(4)], 1)
    assert ((r == 0).all(1)).sum() >= 40                            # zero-norm quaternions: 0 / 0


@pytest.mark.gpu
def test_splat_sort_and_pack_special_metrics(cuda, gsx_lib):
    from gsx import splat
    a = splat_metric_case()
    enc = splat.encode(device_records(a, cuda))
    assert np.array_equal(enc.order.cpu().numpy(), sco.splat_order(a))
    with np.errstate(all="ignore"):
        assert_same(enc.to_host(), sco.splat_file(a), "splat")
