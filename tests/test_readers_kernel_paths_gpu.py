"""The .splat, .ksplat, .spz and compressed PLY reader kernels (csrc/gsx_readers.cu), path by path: rows wider than
the staging buffer (store_rows_gap), staged loads and stores at every byte alignment, the .ksplat partial-bucket
search, the float64 rotation clamps, and compressed PLY rows above 48 KB of shared memory per CTA.

Each case has a seeded builder.  An unmarked CPU test restates the dispatch (row_bytes <= 256 stages whole rows, else
store_rows_gap; the alignment of each staged source and destination; i < full or the bucket search; the shared memory
against 48 KB and 200 KB) and checks in NumPy that the case reaches the branch it is named after.  A `gpu` test asserts
byte equality with readers_oracle, which the CPU tests pin to the reference readers' own results (g13)."""
import struct
import sys
from pathlib import Path

import numpy as np
import pytest

import readers_oracle as ro

sys.path.insert(0, str(Path(__file__).resolve().parent / "golden"))
from make_readers_golden import ksplat_file, sec, spz_body  # noqa: E402

ROWS = 128            # kRows: rows per CTA of every reader kernel
STAGE_MAX = 256       # kStageMax: wider rows go through store_rows_gap
SMEM_DEFAULT = 48 * 1024


def gaussian_row_bytes(degree, has_rgb=False):
    from gsx.readers import gaussian_dtype
    return gaussian_dtype(has_rgb=has_rgb, sh_degree=degree).itemsize


def check(fmt, blob, cuda):
    from gsx import compressed_ply, ksplat, splat, spz
    dec = {"splat": splat.decode, "ksplat": ksplat.decode, "spz": spz.decode, "cply": compressed_ply.decode}[fmt]
    got = dec(blob, cuda).to_host()
    with np.errstate(all="ignore"):
        want = ro.READERS[fmt](blob)[0]
    assert got.dtype == want.dtype and len(got) == len(want), fmt
    g = np.frombuffer(got.tobytes(), np.uint8)
    w = np.frombuffer(np.ascontiguousarray(want).tobytes(), np.uint8)
    d = np.flatnonzero(g != w)
    assert d.size == 0, f"{fmt}: {d.size} bytes differ, first at {d[:8]} (rows {d[:4] // got.dtype.itemsize})"
    return got


# ------------------------------------------------------------------------------------------------ .ksplat layout
def ksplat_plan(blob):
    """Per section, as ksplat.decode lays the file out: (n, sh_count, level, record start, centres start, per)."""
    msc = struct.unpack_from("<I", blob, 4)[0]
    level = min(struct.unpack_from("<H", blob, 20)[0], 2)
    off, out = 4096 + 1024 * msc, []
    for i in range(msc):
        s = dict(zip(ro.SECTION_KEYS, struct.unpack_from("<IIIIfHxxIIIIH", blob, 4096 + 1024 * i)))
        sh = {1: 9, 2: 24}.get(s["shDegree"], 0)
        per = 44 + 4 * sh if level == 0 else 24 + (2 if level == 1 else 1) * sh
        npart, nb = s["partiallyFilledBucketCount"], s["bucketCount"]
        out.append(dict(s, sh_count=sh, level=level, rec_at=off + 4 * npart + 12 * nb, centres_at=off + 4 * npart,
                        per=per))
        off += 4 * npart + 12 * nb + s["maxSplatCount"] * per
    return out


KSPLAT_GAP = [(lv, top) for top in (4, 7) for lv in (0, 1, 2)]


def ksplat_gap_file(level, top):
    """1 350 splats in three sections of SH count 0 (header degree `top`), 9 and 24: rows of degree `top`."""
    return ksplat_file(level, [sec(600, 64, deg=top), sec(450, 16, deg=1), sec(300, 7, deg=2, maxn=310)])


@pytest.mark.parametrize("level,top", KSPLAT_GAP)
def test_ksplat_gap_case_reaches_its_path(level, top):
    blob = ksplat_gap_file(level, top)
    row = gaussian_row_bytes(top)
    assert row > STAGE_MAX                                         # store_rows_gap
    plan = ksplat_plan(blob)
    assert [p["sh_count"] for p in plan] == [0, 9, 24] and sum(p["splatCount"] for p in plan) >= 1000
    for p in plan:
        head = 4 * (9 + p["sh_count"])
        assert p["splatCount"] > ROWS and head + 32 < row          # several CTAs, a zero run between head and tail


@pytest.mark.gpu
@pytest.mark.parametrize("level,top", KSPLAT_GAP)
def test_ksplat_decode_gap_rows(level, top, cuda, gsx_lib):
    blob = ksplat_gap_file(level, top)
    got = check("ksplat", blob, cuda)
    row = 0
    for p in ksplat_plan(blob):
        part = got[row:row + p["splatCount"]]
        n_rest = 3 * ((top + 1) ** 2 - 1)
        for k in range(p["sh_count"], n_rest):                     # SH columns this section does not store
            assert not part[f"f_rest_{k}"].view(np.uint32).any(), (p["sh_count"], k)
        row += p["splatCount"]


def ksplat_align_file():
    """16 level-2 sections of 33-byte records (SH count 9); each earlier section's maxSplatCount moves the next
    section's record start to the next residue mod 16."""
    secs = [sec(130 + 3 * k, 16, deg=1) for k in range(16)]
    for k in range(1, 16):
        r0 = ksplat_plan(ksplat_file(2, secs))[0]["rec_at"] % 16
        r = ksplat_plan(ksplat_file(2, secs))[k]["rec_at"] % 16
        secs[k - 1]["maxn"] += ((r0 + k) - r) % 16                   # 33 = 1 mod 16: one more splat, one byte on
    return ksplat_file(2, secs)


def test_ksplat_align_case_reaches_every_alignment():
    plan = ksplat_plan(ksplat_align_file())
    assert {p["per"] for p in plan} == {33}
    assert {p["rec_at"] % 16 for p in plan} == set(range(16))      # every record start alignment of load_staged
    assert len({p["centres_at"] % 4 for p in plan}) == 4           # centres read byte by byte at any offset
    out = np.cumsum([0] + [p["splatCount"] for p in plan])[:-1] * gaussian_row_bytes(1)
    assert len({o % 16 for o in out}) >= 2 and all(p["splatCount"] % ROWS for p in plan)


@pytest.mark.gpu
def test_ksplat_decode_every_record_alignment(cuda, gsx_lib):
    check("ksplat", ksplat_align_file(), cuda)


def _lengths(rng, k, top):
    v = rng.integers(0, top + 1, k)
    v[0] = v[-1] = 0
    return [int(x) for x in v]


def ksplat_bucket_case(name):
    """(level, sections) of a bucket-search case; every section's n is covered exactly by its buckets."""
    rng = np.random.default_rng(len(name))
    if name == "many_partial":           # 1 000 partial buckets of 0..5 splats, zero-length first and last
        p = _lengths(rng, 1000, 5)
        return 1, [sec(3 * 16 + sum(p), 16, deg=1, fb=3, partial=p)]
    if name == "bucket_size_1":
        p = [0, 3, 1, 0, 2, 5, 0]
        return 2, [sec(200 + sum(p), 1, deg=2, fb=200, partial=p)]
    if name == "n_equals_full":          # partial lengths present, never searched
        return 1, [sec(20 * 16, 16, deg=0, fb=20, partial=[4, 2])]
    if name == "spanning":
        p = [10, 0, 33, 64, 1]
        return 2, [sec(5 * 64 + sum(p), 64, deg=1, fb=5, partial=p)]
    if name == "no_full":                # fullBucketCount = 0: every splat through the search
        p = _lengths(rng, 60, 40)
        return 1, [sec(sum(p), 32, deg=2, fb=0, partial=p), sec(300, 8, deg=1, fb=0, partial=[0, 300, 0])]
    raise KeyError(name)


BUCKET_CASES = ["many_partial", "bucket_size_1", "n_equals_full", "spanning", "no_full"]


def bucket_search(ends, j, strict=True):
    """k_ksplat_decode's search: the first partial bucket whose prefix end is > j (>= j with strict=False)."""
    lo, hi = 0, len(ends) - 1
    while lo < hi:
        mid = (lo + hi) >> 1
        if (ends[mid] > j) if strict else (ends[mid] >= j):
            hi = mid
        else:
            lo = mid + 1
    return lo


@pytest.mark.parametrize("name", BUCKET_CASES)
def test_ksplat_bucket_case_reaches_its_path(name):
    level, secs = ksplat_bucket_case(name)
    for s in secs:
        n, full = s["n"], s["fb"] * s["bs"]
        ends = np.cumsum(s["partial"], dtype=np.int64)
        cover = full + (int(ends[-1]) if len(ends) else 0)
        assert cover == n or (name == "n_equals_full" and cover > n)
        j = np.arange(max(n - full, 0))
        got = [bucket_search(ends, x) for x in j]
        assert got == list(np.searchsorted(ends, j, side="right"))   # the restatement is the oracle's bucket
        if name == "n_equals_full":
            assert n == full and len(j) == 0
        else:
            assert len(j) > 0 and got != [bucket_search(ends, x, strict=False) for x in j]
        if name == "many_partial":
            assert len(ends) == 1000 and s["partial"][0] == s["partial"][-1] == 0 and full > 0
        if name == "bucket_size_1":
            assert s["bs"] == 1 and full > ROWS
        if name == "spanning":
            assert full % ROWS != 0 and 0 < full < n                # one CTA holds full and partial splats
        if name == "no_full":
            assert full == 0
    assert level >= 1


@pytest.mark.gpu
@pytest.mark.parametrize("name", BUCKET_CASES)
def test_ksplat_decode_bucket_search(name, cuda, gsx_lib):
    level, secs = ksplat_bucket_case(name)
    check("ksplat", ksplat_file(level, secs), cuda)


# ------------------------------------------------------------------------------------------------ .spz
SPZ_NS = [3 * ROWS + r for r in range(16)]
SPZ_DIM = {0: 0, 3: 15}


def spz_sections(version, n, dim):
    """Body offsets (16-byte aligned after the header) and widths of the planar sections k_spz_decode loads."""
    pb, rb = (6 if version == 1 else 9), (4 if version >= 3 else 3)
    out = {"pos": (0, pb), "alpha": (n * pb, 1), "colour": (n * (pb + 1), 3), "scale": (n * (pb + 4), 3),
           "rot": (n * (pb + 7), rb)}
    if dim:
        out["sh"] = (n * (pb + 7 + rb), 3 * dim)
    return out


@pytest.mark.parametrize("version", [1, 2, 3])
@pytest.mark.parametrize("degree", [0, 3])
def test_spz_sizes_reach_every_alignment(version, degree):
    dim = SPZ_DIM[degree]
    assert gaussian_row_bytes(degree, True) <= STAGE_MAX           # whole rows
    seen = {}
    for n in SPZ_NS:
        for k, (off, w) in spz_sections(version, n, dim).items():
            seen.setdefault(k, set()).add((off + 3 * ROWS * w) % 16)   # the last CTA's load
    for k, (off, _) in spz_sections(version, 16, dim).items():
        assert seen[k] == {(r * (off // 16)) % 16 for r in range(16)}, k
    assert all(n % ROWS for n in SPZ_NS[1:])


@pytest.mark.gpu
@pytest.mark.parametrize("version", [1, 2, 3])
@pytest.mark.parametrize("degree", [0, 3])
def test_spz_decode_every_alignment(version, degree, cuda, gsx_lib):
    for n in SPZ_NS:
        check("spz", spz_body(version, n, degree, seed=n), cuda)


SPZ_GAP = [(v, d) for v in (2, 3) for d in (4, 9)]


@pytest.mark.parametrize("version,degree", SPZ_GAP)
def test_spz_gap_case_reaches_its_path(version, degree):
    assert gaussian_row_bytes(degree, True) > STAGE_MAX and 1000 > 4 * ROWS   # store_rows_gap, several CTAs


@pytest.mark.gpu
@pytest.mark.parametrize("version,degree", SPZ_GAP)
def test_spz_decode_gap_rows(version, degree, cuda, gsx_lib):
    got = check("spz", spz_body(version, 1000, degree, seed=degree), cuda)
    assert not np.stack([got[f"f_rest_{k}"] for k in range(3 * ((degree + 1) ** 2 - 1))]).view(np.uint32).any()


def spz_v3_words():
    """Every largest-component index with every sign pattern and magnitudes 0 and 511 in the three stored slots."""
    out = []
    for big in range(4):
        for signs in range(8):
            for mags in range(8):
                w = big << 30
                for k in range(3):
                    w |= ((signs >> k & 1) << 9 | (511 if mags >> k & 1 else 0)) << (20 - 10 * k)
                out.append(w)
    return np.array(out, np.uint32)


SPZ_ROT_N = 512


def spz_rotation_file(version):
    """SPZ_ROT_N splats: the first rotation entries set (v3: spz_v3_words; v1, v2: every byte triple of 0, 127, 128,
    255), the rest random."""
    body = bytearray(spz_body(version, SPZ_ROT_N, 1, seed=20 + version))
    off = 16 + spz_sections(version, SPZ_ROT_N, 3)["rot"][0]
    if version >= 3:
        w = spz_v3_words()
        body[off:off + 4 * len(w)] = w.astype("<u4").tobytes()
    else:
        t = np.array([(a, b, c) for a in (0, 127, 128, 255) for b in (0, 127, 128, 255) for c in (0, 127, 128, 255)],
                     np.uint8)
        body[off:off + t.size] = t.tobytes()
    return bytes(body)


@pytest.mark.parametrize("version", [1, 2, 3])
def test_spz_rotation_case_reaches_its_paths(version):
    body = spz_rotation_file(version)
    off = 16 + spz_sections(version, SPZ_ROT_N, 3)["rot"][0]
    if version >= 3:
        w = np.frombuffer(body, "<u4", 256, off)
        assert set(w >> 30) == {0, 1, 2, 3}
        sign = np.stack([(w >> (29 - 10 * k)) & 1 for k in range(3)], 1)
        assert len({tuple(s) for s in sign}) == 8
        v = [((w >> (20 - 10 * k) & 0x1FF).astype(np.float32) / 511.0) * 0.707106781186547524401 for k in range(3)]
        s2 = v[0] ** 2 + v[1] ** 2 + v[2] ** 2
    else:
        xyz = np.frombuffer(body, np.uint8, 3 * 64, off).reshape(-1, 3).astype(np.float32) / 127.5 - 1.0
        s2 = (xyz ** 2).sum(1)
    assert (1.0 - s2 < 0).sum() >= 8 and (1.0 - s2 > 0).sum() >= 8   # the max(0, 1 - s^2) clamp, both sides


@pytest.mark.gpu
@pytest.mark.parametrize("version", [1, 2, 3])
def test_spz_decode_rotation_edges(version, cuda, gsx_lib):
    check("spz", spz_rotation_file(version), cuda)


# ------------------------------------------------------------------------------------------------ .splat
SPLAT_NS = [ROWS + 1, (1 << 10) * ROWS + 77]


def splat_file(n):
    rng = np.random.default_rng(n)
    rec = rng.integers(0, 256, (n, 32), dtype=np.uint8)
    rec[::7, 28:32] = 128                                          # a zero quaternion: the 1e-6 norm clamp
    rec[-1, 28:32] = 128
    rec[3::11, 28:32] = (128, 128, 129, 128)
    return rec.tobytes()


@pytest.mark.parametrize("n", SPLAT_NS)
def test_splat_case_reaches_its_paths(n):
    rec = np.frombuffer(splat_file(n), np.uint8).reshape(n, 32)
    assert n % ROWS != 0 and n > ROWS
    q = (rec[:, 28:32].astype(np.float32) - 128) / 128.0
    norm = np.sqrt((q ** 2).sum(1))
    assert (norm < 1e-6).sum() >= n // 8 and norm[-1] < 1e-6


@pytest.mark.gpu
@pytest.mark.parametrize("n", SPLAT_NS)
def test_splat_decode_partial_cta_and_norm_clamp(n, cuda, gsx_lib):
    check("splat", splat_file(n), cuda)


# ------------------------------------------------------------------------------------------------ compressed PLY
PLY_NAMES = {np.dtype("<f4"): "float", np.dtype("<u4"): "uint", np.dtype("u1"): "uchar", np.dtype("<i2"): "short"}


def ply_file(elements, pad=0):
    """A binary little-endian PLY of (name, structured array) elements, its header padded with a comment of `pad`
    bytes."""
    lines = ["ply", "format binary_little_endian 1.0", "comment " + "p" * pad]
    for name, a in elements:
        lines.append(f"element {name} {len(a)}")
        lines += [f"property {PLY_NAMES[a.dtype.fields[f][0]]} {f}" for f in a.dtype.names]
    lines.append("end_header")
    return ("\n".join(lines) + "\n").encode() + b"".join(np.ascontiguousarray(a).tobytes() for _, a in elements)


def cply_case(name, pad=0):
    """(elements, n, nchunk, nsh) of a compressed PLY case."""
    from gsx.compressed_ply import CHUNK_DTYPE, VERTEX_DTYPE
    n, nchunk, nsh, extra, order = {"sh64": (700, 3, 64, [], None), "padded_vertex": (1000, 4, 45, "pad", None),
                                    "permuted_sh": (600, 3, 24, [], "perm"), "fewer_chunks": (700, 2, 9, [], None),
                                    "row1024": (300, 2, 64, "wide", None), "comment_pad": (300, 2, 9, "u1", None)}[name]
    rng = np.random.default_rng(len(name) + pad)
    chunk = np.zeros(nchunk, CHUNK_DTYPE)
    for f in CHUNK_DTYPE.names:
        chunk[f] = rng.uniform(-5, 5, nchunk).astype(np.float32) + (10.0 if f.startswith("max") else 0.0)
    words = rng.integers(0, 1 << 32, (n, 4), dtype=np.uint64).astype(np.uint32)
    if extra == "pad":      # u1 / f4 / i2 properties around the packed words: odd offsets, a 100-byte row
        fields = [("pad_a", "u1"), ("packed_position", "<u4")] + [(f"e{k}", "<f4") for k in range(20)] + \
                 [("packed_rotation", "<u4"), ("pad_b", "u1"), ("pad_c", "<i2"), ("packed_scale", "<u4"),
                  ("packed_color", "<u4")]
    elif extra == "wide":   # a 1 024-byte row
        fields = [(f, "<u4") for f in VERTEX_DTYPE.names] + [(f"e{k}", "<f4") for k in range(252)]
    elif extra == "u1":
        fields = [("pad_a", "u1")] + [(f, "<u4") for f in VERTEX_DTYPE.names]
    else:
        fields = [(f, "<u4") for f in VERTEX_DTYPE.names]
    vertex = np.zeros(n, fields)
    for k, f in enumerate(VERTEX_DTYPE.names):
        vertex[f] = words[:, k]
    for f, t in fields:
        if f not in VERTEX_DTYPE.names:
            vertex[f] = rng.integers(0, 100, n).astype(t)
    names = [f"f_rest_{i}" for i in range(nsh)]
    if order == "perm":
        names = [names[i] for i in rng.permutation(nsh)]
    sh = rng.integers(0, 256, (n, nsh), dtype=np.uint8).view(np.dtype([(f, "u1") for f in names])).reshape(-1)
    return [("chunk", chunk), ("vertex", vertex), ("sh", sh)], n, nchunk, nsh


CPLY_CASES = ["sh64", "padded_vertex", "permuted_sh", "fewer_chunks", "row1024"]


def cply_layout(blob):
    from gsx.compressed_ply import decode_smem_bytes
    from gsx.readers import parse_ply_header
    els, _ = parse_ply_header(blob)
    vx, sh = els["vertex"], els["sh"]
    nsh = len(sh.dtype.names)
    return els, decode_smem_bytes(vx.dtype.itemsize, sh.dtype.itemsize, nsh)


@pytest.mark.parametrize("name", CPLY_CASES)
def test_cply_case_reaches_its_path(name):
    els, n, nchunk, nsh = cply_case(name)
    blob = ply_file(els)
    layout, smem = cply_layout(blob)
    if name in ("sh64", "padded_vertex", "row1024"):
        assert SMEM_DEFAULT < smem <= 200 * 1024                   # cudaFuncSetAttribute before the launch
    if name == "padded_vertex":
        assert layout["vertex"].dtype.itemsize == 100 and layout["vertex"].dtype.fields["packed_position"][1] == 1
    if name == "permuted_sh":
        assert list(layout["sh"].dtype.names) != sorted(layout["sh"].dtype.names, key=lambda f: int(f[7:]))
    if name == "fewer_chunks":
        assert n > nchunk * 256 and n % ROWS != 0                  # rows past nchunk * 256 stay zero
    if name == "row1024":
        assert layout["vertex"].dtype.itemsize == 1024
    assert nsh == len(layout["sh"].dtype.names)


@pytest.mark.gpu
@pytest.mark.parametrize("name", CPLY_CASES)
def test_cply_decode_layouts(name, cuda, gsx_lib):
    els, n, nchunk, nsh = cply_case(name)
    got = check("cply", ply_file(els), cuda)
    if name == "fewer_chunks":
        assert not got[nchunk * 256:].view(np.uint8).any()


def test_cply_comment_pad_reaches_every_alignment():
    starts = {"chunk": set(), "vertex": set(), "sh": set()}
    for pad in range(16):
        els, n, nchunk, _ = cply_case("comment_pad", pad)
        layout, _ = cply_layout(ply_file(els, pad))
        for k in starts:
            starts[k].add(layout[k].offset % 16)
        assert n % ROWS != 0 and layout["vertex"].dtype.itemsize == 17
    assert all(s == set(range(16)) for s in starts.values())


@pytest.mark.gpu
def test_cply_decode_every_element_alignment(cuda, gsx_lib):
    for pad in range(16):
        els, *_ = cply_case("comment_pad", pad)
        check("cply", ply_file(els, pad), cuda)


REFUSED = ["vertex_row", "chunk_row"]


def refused_rows(kind):
    """A compressed PLY whose vertex row is 1 100 bytes, or whose chunk row is 1 072 bytes."""
    els, *_ = cply_case("sh64")
    chunk, vertex, sh = (a for _, a in els)
    if kind == "vertex_row":
        wide = np.zeros(len(vertex), vertex.dtype.descr + [(f"e{k}", "<f4") for k in range(271)])
        for f in vertex.dtype.names:
            wide[f] = vertex[f]
        vertex = wide
    else:
        wide = np.zeros(len(chunk), chunk.dtype.descr + [(f"e{k}", "<f4") for k in range(250)])
        for f in chunk.dtype.names:
            wide[f] = chunk[f]
        chunk = wide
    return ply_file([("chunk", chunk), ("vertex", vertex), ("sh", sh)])


@pytest.mark.parametrize("kind", REFUSED)
def test_cply_decode_refuses_rows_it_cannot_stage(kind, gsx_lib):
    """A ValueError, as decode's docstring promises, raised on the host before anything is uploaded."""
    from gsx import compressed_ply
    blob = refused_rows(kind)
    layout, _ = cply_layout(blob)
    assert layout[kind.split("_")[0]].dtype.itemsize == {"vertex_row": 1100, "chunk_row": 1072}[kind]
    with pytest.raises(ValueError):
        compressed_ply.decode(blob, "cuda")
    # the widest rows decode accepts stay within the kernel's shared-memory bound
    assert compressed_ply.decode_smem_bytes(1024, 64, 64) <= compressed_ply.DECODE_SMEM_MAX


@pytest.mark.gpu
@pytest.mark.parametrize("kind", REFUSED)
def test_cply_decode_refusal_on_the_device(kind, cuda, gsx_lib):
    from gsx import compressed_ply
    with pytest.raises(ValueError):
        compressed_ply.decode(refused_rows(kind), cuda)
