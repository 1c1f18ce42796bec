"""The Parquet writer kernels path by path: gsx_parquet_split, gsx_parquet_dict_insert / gsx_parquet_dictionary /
gsx_parquet_dict_index, gsx_parquet_pages, gsx_parquet_snappy and gsx_parquet_assemble, called directly and compared
byte for byte with tests/parquet_oracle.py's restatement of each kernel; gsx.parquet.encode at 2^31 rows.

Each case has a seeded builder, a CPU test that its data reaches the branch it is for (the oracle's COUNTERS, or the
arithmetic of the launch), and a GPU test.  Outputs start filled with a sentinel, except the buffers the entry points
document as zeroed by the caller.  Every file a test writes is also read back by pyarrow and its values compared with
the input (NaN <=> null), on the CPU for the oracle's file and on the GPU for the device's, so every page form is
checked against an independent reader and not only against the restatement."""
import ctypes as C
import io
import itertools

import numpy as np
import pytest

import parquet_oracle as po
from gsx import parquet as gp

pq = pytest.importorskip("pyarrow.parquet")
pa = pytest.importorskip("pyarrow")

U32 = np.uint32
SENT = 0xA5A5A5A5                                  # what a uint32 output holds before a launch
SENT_I32 = int(np.array(SENT, U32).view(np.int32))
SENT_B = 0x5A
NAN_PATTERNS = [0x7FC00000, 0xFFC00000, 0x7F800001, 0xFFFFFFFF, 0x7FBFFFFF, 0xFF800001, 0x7FC0BEEF]


def _dev():
    from gsx._abi import lib, _ptr, _stream
    return lib, _ptr, _stream


def _full(shape, cuda, value=SENT_I32, dtype=None):
    import torch
    return torch.full(shape, value, dtype=dtype or torch.int32, device=cuda)


def _up(a, cuda):
    from gsx.hostcopy import to_device
    return to_device(np.ascontiguousarray(a), cuda)


def _host(t, dtype=U32):
    from gsx.hostcopy import to_host
    return to_host(t).view(dtype)


def read_back(blob: bytes, a: np.ndarray) -> None:
    """pyarrow reads the file; every column equals the input's field bit for bit, NaN <=> null."""
    t = pq.read_table(io.BytesIO(blob))
    plan = gp.column_plan(a.dtype)
    assert t.num_rows == len(a) and t.column_names == [c.name for c in plan]
    for c in plan:
        col, v = t.column(c.name), np.ascontiguousarray(a[c.source])
        if c.kind == gp.F4:
            valid = ~np.isnan(v)
            assert np.array_equal(np.asarray(col.is_valid()), valid), c.name
            got = col.to_numpy(zero_copy_only=False).astype(np.float32)
            assert np.array_equal(got[valid].view(U32), v[valid].view(U32)), c.name
        else:
            assert col.null_count == 0 and np.array_equal(col.to_numpy(), v), c.name


def _floats(rng, m):
    """m float32 patterns, none NaN."""
    v = rng.integers(0, 1 << 32, m, dtype=np.uint64).astype(U32)
    v[(v & 0x7FFFFFFF) > 0x7F800000] &= 0xBFFFFFFF
    return v


# ============================================================================================================== split
SPLIT_ROWS = [1, 63, 64, 65, 2047, 2048, 2049, (1 << 20) - 1, (1 << 20) + 1, (1 << 20) + 2048]
MIX5 = np.dtype([("x", "<f4"), ("red", "u1"), ("y", "<f4"), ("opacity", "<f4"), ("z", "<f4")])   # 17-byte rows


def _dtype(name):
    """The layouts of the width / column-count cases (unmapped fields keep their names and input order)."""
    if name == "cols1":
        return np.dtype([("x", "<f4")])
    if name == "row1":
        return np.dtype([("red", "u1")])
    if name == "cols2_row5":
        return np.dtype([("x", "<f4"), ("red", "u1")])
    if name == "cols3":
        return np.dtype([("x", "<f4"), ("y", "<f4"), ("green", "u1")])
    if name == "cols5":
        return MIX5
    if name == "cols257":
        return np.dtype([(f"e{i}", "u1") for i in range(200)] + [(f"f{i}", "<f4") for i in range(57)])
    if name == "row251_padded":
        return np.dtype({"names": ["x", "opacity", "red", "w"], "formats": ["<f4", "<f4", "u1", "<f4"],
                         "offsets": [3, 101, 250, 40], "itemsize": 251})
    if name == "row768_padded":
        return np.dtype({"names": [f"f{i}" for i in range(100)] + ["m"], "formats": ["<f4"] * 100 + ["u1"],
                         "offsets": [7 * i + 2 for i in range(100)] + [767], "itemsize": 768})
    if name == "u1x1024":
        return np.dtype([(f"u{i}", "u1") for i in range(1024)])
    raise KeyError(name)


SPLIT_LAYOUTS = ["cols1", "row1", "cols2_row5", "cols3", "cols5", "cols257", "row251_padded", "row768_padded",
                 "u1x1024"]


def fill_values(a, rng, nan_every=0):
    """Random finite float32 fields and uint8 fields (the padding random too: it is never read)."""
    raw = a.view(np.uint8).reshape(len(a), a.dtype.itemsize)
    raw[:] = rng.integers(0, 256, raw.shape, dtype=np.uint8)
    for f in a.dtype.names:
        if a.dtype.fields[f][0] == np.dtype("<f4"):
            a[f] = rng.standard_normal(len(a)).astype(np.float32) * 100
            if nan_every:
                a[f][rng.integers(0, nan_every):: nan_every] = np.nan
    return a


def split_case(name, n):
    a = np.zeros(n, _dtype(name))
    return fill_values(a, np.random.default_rng(n + len(name)), nan_every=5)


def values_case(n=(1 << 20) + 3000):
    """Every special value, with the extremes in lane 0, in the last row and in the partial last tile; all-null tiles,
    an all-null row group and an all-null column."""
    names = ["x", "y", "z", "opacity", "nx", "ny", "nz", "scale_0", "scale_1"]
    a = np.zeros(n, [(f, "<f4") for f in names] + [("red", "u1"), ("green", "u1")])
    rng = np.random.default_rng(11)
    for f in names:
        a[f] = rng.standard_normal(n).astype(np.float32)
    bits = lambda f: a[f].view(U32)
    last_tile = n // 2048 * 2048
    # x: NaN of both signs and several payloads everywhere; the extremes at row 0 (min) and in the last tile (max)
    bits("x")[rng.integers(0, n, 5000)] = rng.choice(NAN_PATTERNS, 5000)
    a["x"][0], a["x"][last_tile + 17] = -np.inf, np.inf
    # y: the extremes in the last row (min) and in lane 0 of the last tile (max); denormals of both signs
    a["y"][n - 1], a["y"][last_tile] = -3e38, 3e38
    bits("y")[100:110] = [1, 0x80000001, 0x007FFFFF, 0x807FFFFF, 0, 0x80000000, 2, 0x80000002, 0x00400000, 0x80400000]
    # z: all +-0 in row group 0 mixed, only -0 in group 1
    a["z"][:] = np.where(rng.random(n) < 0.5, np.float32(-0.0), np.float32(0.0))
    a["z"][gp.ROW_GROUP:] = -0.0
    # opacity: whole tiles null, and all of row group 1
    for t in (0, 3, 100):
        bits("opacity")[t * 2048:(t + 1) * 2048] = 0xFFC00000
    bits("opacity")[gp.ROW_GROUP:] = 0x7F800001
    # nx: an all-null column; ny: only +0; nz: only -0 and NaN; scale_0: only denormals; scale_1: +-inf and NaN
    bits("nx")[:] = rng.choice(NAN_PATTERNS, n)
    a["ny"][:] = 0.0
    a["nz"][:] = -0.0
    a["nz"][::7] = np.nan
    bits("scale_0")[:] = rng.integers(1, 0x007FFFFF, n).astype(U32) | (rng.integers(0, 2, n).astype(U32) << 31)
    a["scale_1"][:] = np.where(rng.random(n) < 0.5, np.float32(np.inf), np.float32(-np.inf))
    bits("scale_1")[::3] = 0xFFFFFFFF
    a["red"] = rng.integers(1, 255, n)
    a["red"][0], a["red"][n - 1] = 255, 0
    a["green"] = rng.integers(1, 255, n)
    a["green"][last_tile + 5], a["green"][2048 * 7] = 0, 255
    return a


def _spec(a):
    return [(a.dtype.fields[f][1], gp.U1 if a.dtype.fields[f][0] == np.dtype("u1") else gp.F4) for f in a.dtype.names]


def _raw(a):
    return np.ascontiguousarray(a).view(np.uint8).reshape(len(a), a.dtype.itemsize)


@pytest.mark.parametrize("name", SPLIT_LAYOUTS)
def test_split_layout_reaches_its_path(name):
    dt = _dtype(name)
    big = po.split_smem(len(dt.names), dt.itemsize) > 48 * 1024
    assert big == (dt.itemsize >= 768), (name, po.split_smem(len(dt.names), dt.itemsize))
    if name == "cols5":
        assert len(dt.names) % 4                                # not a multiple of the 4 column groups of a CTA
    po.COUNTERS.clear()
    a = split_case(name, 5000)
    out, tnull, keys = po.split_kernel(_raw(a), _spec(a))
    assert ("split_smem_over_48k" in po.COUNTERS) == big
    assert out.shape == (len(dt.names), 5000) and tnull.shape[1] == 3 and 5000 % 2048


def test_values_case_reaches_its_edges():
    po.COUNTERS.clear()
    a = values_case()
    out, tnull, keys = po.split_kernel(_raw(a), _spec(a))
    names = list(a.dtype.names)
    c = {f: names.index(f) for f in names}
    pats = set(out[c["x"]].tolist())
    assert {0x7FC00000, 0xFFC00000, 0x7F800001, 0xFFFFFFFF} <= pats
    assert (tnull[c["opacity"], [0, 3, 100]] == 2048).all() and (tnull[c["nx"]][:-1] == 2048).all()
    assert keys[0, c["opacity"], 1] == 0xFFFFFFFF and keys[1, c["opacity"], 1] == 0    # an all-null row group
    assert (keys[0, c["nx"]] == 0xFFFFFFFF).all() and po.COUNTERS["split_chunk_without_value"] == 3
    assert len(a) % 2048 and len(a) > gp.ROW_GROUP
    assert keys[1, c["red"], 0] == 255 and keys[0, c["red"], 1] == 0 and keys[0, c["green"], 1] == 0 and keys[1, c["green"], 0] == 255


@pytest.mark.parametrize("n", SPLIT_ROWS)
def test_split_rows_reach_their_tiles(n):
    T = -(-n // 2048)
    assert (n % 2048 == 0) == (n in (2048, (1 << 20) + 2048)) and (n % 64 == 0) == (n in (64, 2048, (1 << 20) + 2048))
    if n > gp.ROW_GROUP:
        # tiles on both sides of the row-group edge; the last one partial or not
        assert (T - 1) * 2048 >= gp.ROW_GROUP and -(-n // gp.ROW_GROUP) == 2


def _zero_sign_stats(blob, a):
    """The file's statistics turn a zero min into -0.0 and a zero max into +0.0 (file_parts)."""
    facts = po.chunk_facts(pq.read_metadata(io.BytesIO(blob)))
    plan = gp.column_plan(a.dtype)
    seen = 0
    for g, (rows, cols) in enumerate(facts):
        for c, (has, mm, mn, mx, nulls, _) in zip(plan, cols):
            if c.kind != gp.F4 or not mm:
                continue
            v = a[c.source][g * gp.ROW_GROUP:(g + 1) * gp.ROW_GROUP]
            v = v[~np.isnan(v)]
            if v.min() == 0:
                assert mn == 0x80000000, (c.name, g)
                seen += 1
            if v.max() == 0:
                assert mx == 0, (c.name, g)
                seen += 1
    return seen


def test_values_case_oracle_file_reads_back():
    a = values_case()
    blob = po.encode(a)
    read_back(blob, a)
    assert _zero_sign_stats(blob, a) >= 4


@pytest.mark.parametrize("name", SPLIT_LAYOUTS)
def test_split_layout_oracle_file_reads_back(name):
    a = split_case(name, 5000)
    read_back(po.encode(a), a)


def dev_split(rows_ptr_tensor, n, row_bytes, spec, cuda):
    """gsx_parquet_split with sentinel-filled outputs -> (out [C, n], tile_nulls [C, T], keys [2, C, G])."""
    lib, _ptr, _stream = _dev()
    nc, T, G = len(spec), -(-n // 2048), max(1, -(-n // gp.ROW_GROUP))
    out, tn, keys = _full((nc * n + 1,), cuda), _full((nc * T + 1,), cuda), _full((2 * nc * G + 1,), cuda)
    cs = (C.c_int32 * (2 * nc))(*[v for s in spec for v in s])
    assert lib.gsx_parquet_split(_ptr(rows_ptr_tensor), n, row_bytes, cs, nc, _ptr(out), _ptr(tn), _ptr(keys),
                                 _stream()) == 0
    out, tn, keys = _host(out), _host(tn), _host(keys)
    assert out[-1] == SENT and tn[-1] == SENT and keys[-1] == SENT      # nothing written past the outputs
    return out[:-1].reshape(nc, n), tn[:-1].reshape(nc, T), keys[:-1].reshape(2, nc, G)


def _assert_split(got, want):
    for name, g, w in zip(("out", "tile_nulls", "keys"), got, want):
        bad = np.argwhere(g != w)
        assert not len(bad), f"{name}: {len(bad)} differ, first {bad[:4].tolist()}: {g[tuple(bad[0])]} vs {w[tuple(bad[0])]}"


def _encode_and_check(src, a, cuda):
    blob = gp.encode(src, device=cuda).to_host()
    assert blob == po.encode(a)
    read_back(blob, a)
    return blob


@pytest.mark.gpu
@pytest.mark.parametrize("n", SPLIT_ROWS)
def test_split_row_counts(n, cuda, gsx_lib):
    a = split_case("cols5", n)
    raw = _raw(a)
    _assert_split(dev_split(_up(raw, cuda), n, raw.shape[1], _spec(a), cuda), po.split_kernel(raw, _spec(a)))
    if n < (1 << 20) or n == (1 << 20) + 2048:
        _encode_and_check(a, a, cuda)


@pytest.mark.gpu
@pytest.mark.parametrize("name", SPLIT_LAYOUTS)
def test_split_layouts(name, cuda, gsx_lib):
    a = split_case(name, 5000)
    raw = _raw(a)
    _assert_split(dev_split(_up(raw, cuda), len(a), raw.shape[1], _spec(a), cuda), po.split_kernel(raw, _spec(a)))
    _encode_and_check(a, a, cuda)


@pytest.mark.gpu
def test_split_values(cuda, gsx_lib):
    a = values_case()
    raw = _raw(a)
    _assert_split(dev_split(_up(raw, cuda), len(a), raw.shape[1], _spec(a), cuda), po.split_kernel(raw, _spec(a)))
    assert _zero_sign_stats(_encode_and_check(a, a, cuda), a) >= 4


@pytest.mark.gpu
def test_split_unaligned_base(cuda, gsx_lib):
    """Rows that start 1..15 bytes into a larger buffer: load_staged's head through the base pointer."""
    import torch
    from gsx.readers import Decoded
    a = split_case("row251_padded", 3000)
    raw = _raw(a)
    want = po.split_kernel(raw, _spec(a))
    buf = _full((raw.size + 16,), cuda, SENT_B, dtype=torch.uint8)
    for o in range(1, 16):
        buf[o:o + raw.size] = _up(raw.reshape(-1), cuda)
        view = buf[o:o + raw.size].view(len(a), raw.shape[1])
        assert view.data_ptr() % 16 == o
        _assert_split(dev_split(view, len(a), raw.shape[1], _spec(a), cuda), want)
        _encode_and_check(Decoded(view, a.dtype, None), a, cuda)


# ======================================================================================================= dictionaries
DICT_COUNTS = sorted({1, 2} | {1 << k for k in range(1, 19)} | {(1 << k) + 1 for k in range(1, 18)})
DICT_N = 1 << 20


def dict_case():
    """One column per distinct count (every bit width 1..18), 262 144 exactly, 262 145 with nulls mixed in, 2^20
    distinct, -0 / +0 as the two entries of the 2-value column, NaN payloads in every column but the last, and a
    column whose page 2 is all null."""
    rng = np.random.default_rng(3)
    counts = DICT_COUNTS + [(1 << 18) + 1, 1 << 20, 3]
    cols = np.empty((len(counts), DICT_N), U32)
    for c, d in enumerate(counts):
        if d == 1 << 20:
            vals = np.arange(d, dtype=U32) * 3 + 0x3F000000       # distinct patterns, no NaN
        else:
            vals = np.unique(_floats(rng, 2 * d + 64))[:d] if d != 2 else np.array([0x80000000, 0], U32)
        assert len(vals) == d
        idx = np.concatenate([np.arange(d), rng.integers(0, d, DICT_N - d)])
        cols[c] = vals[rng.permutation(idx)]
        if d != 1 << 20:
            cols[c, rng.integers(0, DICT_N, 999)] = rng.choice(NAN_PATTERNS, 999)
            cols[c, :d] = vals                                    # every value stays present
            cols[c] = cols[c, rng.permutation(DICT_N)] if d > 1 else cols[c]
    cols[-1, 2 * gp.PAGE:3 * gp.PAGE] = 0xFFC00000
    return cols, counts


def _f4_array(cols):
    a = np.zeros(cols.shape[1], [(f"v{c}", "<f4") for c in range(len(cols))])
    for c in range(len(cols)):
        a[f"v{c}"] = cols[c].view(np.float32)
    return a


def test_dict_case_reaches_every_width():
    po.COUNTERS.clear()
    cols, counts = dict_case()
    d = po.distinct_counts(cols, [gp.F4] * len(cols))[:, 0]
    assert d.tolist() == counts
    assert gp.DICT_MAX in counts and gp.DICT_MAX + 1 in counts and (1 << 20) in counts
    widths = set()
    for c in range(len(cols)):
        if d[c] <= gp.DICT_MAX:
            dv, ranks = po.dictionary(cols[c], gp.F4)
            widths.add(gp.bit_width(len(dv)))
    assert widths == set(range(1, 19))
    assert set(cols[1][~po.is_null(cols[1], gp.F4)].tolist()) == {0, 0x80000000}     # -0 and +0: two entries
    over = counts.index(gp.DICT_MAX + 1)
    assert po.is_null(cols[0], gp.F4).any() and po.is_null(cols[over], gp.F4).any()
    pr = po.page_ranks(po.dictionary(cols[-1], gp.F4)[1], po.is_null(cols[-1], gp.F4))
    assert pr[0, 2] == 0xFFFFFFFF and po.COUNTERS["index_page_empty"] == 1
    po.page_ranks(po.dictionary(cols[0], gp.F4)[1], po.is_null(cols[0], gp.F4))
    assert po.COUNTERS["index_page_equal"] == 4


def test_dict_case_oracle_file_reads_back():
    cols, _ = dict_case()
    a = _f4_array(cols[[0, 1, 5, 20, -4, -1]])
    read_back(po.encode(a), a)


def dev_dict_run(cols, g0, ng, cuda, select=None, slots=20):
    """insert -> (host picks the chunks: select(distinct) -> bool [C, ng]) -> dictionary -> index, as gsx.parquet.encode
    runs them.  Returns (distinct [C, G], {(c, g): dictionary}, cols after the index, page_idx [2, C, P])."""
    import torch
    lib, _ptr, _stream = _dev()
    nc, n = cols.shape
    G, P = max(1, -(-n // gp.ROW_GROUP)), -(-n // gp.PAGE)
    cd = _up(cols.view(np.int32), cuda)
    table = torch.zeros((ng * nc) << slots, dtype=torch.int64, device=cuda)
    dcount = torch.zeros(nc * G, dtype=torch.int32, device=cuda)
    assert lib.gsx_parquet_dict_insert(_ptr(cd), n, nc, g0, ng, _ptr(table), slots, _ptr(dcount), _stream()) == 0
    distinct = _host(dcount).astype(np.int64).reshape(nc, G)
    sel = select(distinct[:, g0:g0 + ng]) if select else distinct[:, g0:g0 + ng] <= gp.DICT_MAX
    cc, gg = np.nonzero(sel)
    cnt = distinct[cc, g0 + gg]
    first = np.concatenate([[0], np.cumsum(cnt)[:-1]]).astype(np.int64)
    jobs = np.stack([cc + nc * gg, first, first], 1).astype(np.int64)
    nkeys = int(cnt.sum())
    vals = _full((nkeys + 1,), cuda)
    ws = torch.empty(lib.gsx_parquet_dictionary_workspace_bytes(nkeys), dtype=torch.uint8, device=cuda)
    jd = _up(jobs, cuda)
    assert lib.gsx_parquet_dictionary(_ptr(table), slots, _ptr(jd), len(jobs), nkeys, _ptr(ws), ws.numel(), _ptr(vals),
                                      _stream()) == 0
    page_idx = torch.empty((2, nc, P), dtype=torch.int32, device=cuda)
    page_idx[0].fill_(-1)
    page_idx[1].zero_()
    seld = _up(sel.astype(np.int32), cuda)
    assert lib.gsx_parquet_dict_index(_ptr(cd), n, nc, g0, ng, _ptr(table), slots, _ptr(seld), _ptr(page_idx),
                                      _stream()) == 0
    v = _host(vals)
    assert v[-1] == SENT
    dicts = {(c, g0 + g): v[f:f + k] for c, g, f, k in zip(cc.tolist(), gg.tolist(), first.tolist(), cnt.tolist())}
    return distinct, dicts, _host(cd).reshape(nc, n), _host(page_idx).reshape(2, nc, P)


def _check_dict_run(cols, g0, ng, got, kinds=None):
    distinct, dicts, ranked, page_idx = got
    nc, n = cols.shape
    kinds = kinds or [gp.F4] * nc
    want = po.distinct_counts(cols, kinds)
    for c in range(nc):
        for g in range(want.shape[1]):
            if not g0 <= g < g0 + ng:
                assert distinct[c, g] == 0, (c, g)
            elif want[c, g] <= gp.DICT_MAX:
                assert distinct[c, g] == want[c, g], (c, g, distinct[c, g], want[c, g])
            else:
                assert distinct[c, g] > gp.DICT_MAX, (c, g)
    for c in range(nc):
        expect = cols[c].copy()
        pw = np.empty((2, page_idx.shape[2]), U32)
        pw[0], pw[1] = 0xFFFFFFFF, 0
        for g in range(want.shape[1]):
            s = slice(g * gp.ROW_GROUP, (g + 1) * gp.ROW_GROUP)
            if (c, g) not in dicts:
                continue
            dv, ranks = po.dictionary(cols[c, s], kinds[c])
            assert np.array_equal(dicts[(c, g)], dv), (c, g)
            expect[s] = ranks
            pw[:, 4 * g:4 * g + 4] = po.page_ranks(ranks, po.is_null(cols[c, s], kinds[c]))
        assert np.array_equal(ranked[c], expect), c
        assert np.array_equal(page_idx[:, c], pw), c


@pytest.mark.gpu
def test_dictionary_every_width(cuda, gsx_lib):
    cols, counts = dict_case()
    got = dev_dict_run(cols, 0, 1, cuda)
    assert got[0][counts.index(1 << 20), 0] > gp.DICT_MAX
    assert len(got[1]) == len(counts) - 2                       # the two chunks above the limit are not indexed
    _check_dict_run(cols, 0, 1, got)
    a = _f4_array(cols[[0, 1, 5, 20, -4, -1]])
    _encode_and_check(a, a, cuda)


def batch_case(n=3 * (1 << 20) + 12345):
    rng = np.random.default_rng(9)
    cols = np.empty((2, n), U32)
    cols[0] = _floats(rng, 37)[rng.integers(0, 37, n)]
    cols[1] = rng.integers(0, 256, n).astype(U32)
    cols[0, ::11] = 0x7FC00000
    cols[0, 3 * gp.ROW_GROUP + 5:] = cols[0, 3 * gp.ROW_GROUP + 5]  # the last group's pages: all ranks equal
    return cols


def test_batch_case_reaches_a_partial_last_batch():
    cols = batch_case()
    n = cols.shape[1]
    assert -(-n // gp.ROW_GROUP) == 4 and n % gp.ROW_GROUP and (n - 3 * gp.ROW_GROUP) % 256


@pytest.mark.gpu
def test_dictionary_later_batch(cuda, gsx_lib):
    """g0 = 1, ng = 3: row groups 1..3, the last partial; a uint8 column beside a float one; row group 0 untouched."""
    cols = batch_case()
    kinds = [gp.F4, gp.U1]
    sel = lambda d: np.array([[True, False, True], [False, True, True]])
    got = dev_dict_run(cols, 1, 3, cuda, select=sel)
    assert len(got[1]) == 4
    _check_dict_run(cols, 1, 3, got, kinds)


JOB_COUNTS = [1, 2, 3, 4, 5, 1024]


def jobs_case(njobs, n=4096):
    rng = np.random.default_rng(njobs)
    cols = np.empty((njobs, n), U32)
    shared = _floats(rng, 64)
    for c in range(njobs):                                      # the jobs share patterns: a sort that mixed them shows
        d = c % 7 + 2
        cols[c] = shared[(np.arange(n) * (c + 1) + c) % d + (c % 5)]
    return cols


@pytest.mark.parametrize("njobs", JOB_COUNTS)
def test_job_count_sets_end_bit(njobs):
    end_bit = 33
    while (1 << (end_bit - 32)) < njobs:
        end_bit += 1
    assert end_bit == {1: 33, 2: 33, 3: 34, 4: 34, 5: 35, 1024: 42}[njobs]


@pytest.mark.gpu
@pytest.mark.parametrize("njobs", JOB_COUNTS)
def test_dictionary_job_counts(njobs, cuda, gsx_lib):
    cols = jobs_case(njobs)
    got = dev_dict_run(cols, 0, 1, cuda)
    assert len(got[1]) == njobs
    _check_dict_run(cols, 0, 1, got)


@pytest.mark.gpu
def test_dictionary_tables_under_2_20_slots_are_refused(cuda, gsx_lib):
    """Nothing is launched: the entry points refuse 2^19 slots (the resident-thread overshoot could fill it)."""
    import torch
    lib, _ptr, _stream = _dev()
    small = torch.zeros(64, dtype=torch.int64, device=cuda)
    cols = torch.zeros(16, dtype=torch.int32, device=cuda)
    cnt = torch.zeros(4, dtype=torch.int32, device=cuda)
    assert lib.gsx_parquet_dict_insert(_ptr(cols), 16, 1, 0, 1, _ptr(small), 19, _ptr(cnt), _stream()) != 0
    assert lib.gsx_parquet_dictionary(_ptr(small), 19, _ptr(small), 1, 1, _ptr(small), 1 << 20, _ptr(cnt),
                                      _stream()) != 0
    assert lib.gsx_parquet_dict_index(_ptr(cols), 16, 1, 0, 1, _ptr(small), 19, _ptr(cnt), _ptr(cnt), _stream()) != 0
    assert not small.any() and not cols.any() and not cnt.any()


# ========================================================================================================= page bodies
PAGE_NS = [1, 63, 64, 8191, 8192, gp.PAGE, gp.PAGE + 8193]


def page_forms():
    """(width, form, nulls) of each column: PLAIN, and for every width 1..18 bit-packed, RLE-equal (the all-ones value:
    1, 2 or 3 bytes) and empty; one value only at three widths."""
    out = [(0, "plain", False), (0, "plain", True), (0, "empty", True)]
    for w in range(1, 19):
        out += [(w, "packed", False), (w, "packed", True), (w, "rle", False), (w, "rle", True), (w, "empty", True)]
    return out + [(w, "one", True) for w in (1, 9, 17)]


def pages_case(n):
    """Columns [C, n] of float32 patterns: a width-w column takes its values from a 2^w-entry dictionary (w = 1: 2)."""
    rng = np.random.default_rng(n)
    forms = page_forms()
    cols = np.empty((len(forms), n), U32)
    dicts = {}
    r = np.arange(n)
    for c, (w, form, nulls) in enumerate(forms):
        null = (r % 3 == 1) if nulls else np.zeros(n, bool)
        if form == "empty":
            null[:] = True
        if form == "one":
            null[:] = True
            null[r % gp.PAGE == (r[-1] % gp.PAGE) // 2] = False
        if w == 0:
            v = _floats(rng, n)
        else:
            dv = np.sort(rng.choice(1 << 24, 1 << w, replace=False).astype(U32) + 0x3F800000)
            dicts[c] = dv
            ranks = rng.integers(0, 1 << w, n) if form == "packed" else np.full(n, (1 << w) - 1)
            if form == "packed":
                ranks[r % 97 == 5] = (1 << w) - 1
                ranks[r % 97 == 6] = 0
            v = dv[ranks]
        cols[c] = np.where(null, 0x7FC00000 | (r.astype(U32) & 0xFF), v)
    return cols, forms, dicts


def pages_oracle(n):
    """The body buffer gsx.parquet.encode lays out for pages_case(n) with its forced widths, its layout, and the
    arguments gsx_parquet_pages takes; and the file around it."""
    cols, forms, dicts = pages_case(n)
    nc = len(forms)
    width = np.array([[w] for w, _, _ in forms], np.int64)
    plan = [gp.Column(f"c{c}", 4 * c, gp.F4, f"c{c}") for c in range(nc)]
    nulls = np.zeros((nc, -(-n // gp.PAGE)), np.int64)
    distinct = np.zeros((nc, 1), np.int64)
    keys = np.zeros((nc, 1, 2), np.int64)
    ranked, equal, full = cols.copy(), np.zeros(nulls.shape, bool), {}
    for c in range(nc):
        null = po.is_null(cols[c], gp.F4)
        nulls[c] = np.add.reduceat(null, np.arange(0, n, gp.PAGE))
        v = cols[c][~null]
        if len(v):
            k = po.key(v, gp.F4)
            keys[c, 0] = k.min(), k.max()
        if c in dicts:
            distinct[c, 0] = len(dicts[c])
            full[(c, 0)] = dicts[c]
            ranked[c] = np.where(null, cols[c], np.searchsorted(dicts[c], cols[c]))
            for p in range(nulls.shape[1]):
                s = slice(p * gp.PAGE, (p + 1) * gp.PAGE)
                i = ranked[c, s][~null[s]]
                equal[c, p] = len(i) > 0 and (i == i[0]).all()
    lay = gp.layout(n, distinct, nulls, width, equal)
    body = bytearray(int(lay.pages[-1, 3] + (lay.pages[-1, 4] + 15) // 16 * 16))
    for kind, c, p, off, size, _ in lay.pages.tolist():
        if kind:
            b = dicts[c].astype("<u4").tobytes()
        else:
            s = slice(p * gp.PAGE, (p + 1) * gp.PAGE)
            b = po.data_page(cols[c, s], po.is_null(cols[c, s], gp.F4), int(width[c, 0]), ranked[c, s])
        assert len(b) == size
        body[off:off + size] = b
    f = lambda: po.write_file(plan, n, cols, nulls, distinct, keys, full, width)
    return dict(cols=cols, ranked=ranked, nulls=nulls, width=width, equal=equal, lay=lay, body=bytes(body), dicts=dicts,
                file=f, plan=plan)


def test_page_cases_reach_every_form():
    po.COUNTERS.clear()
    for n in PAGE_NS:
        pages_oracle(n)
    k = po.COUNTERS
    for w in range(1, 19):
        for form in ("packed", "rle"):
            for nulls in (False, True):
                assert k.get(("page", form, w, nulls)), (form, w, nulls)
        assert k.get(("page", "empty", w, True)), w
    assert k.get(("page", "plain", 0, False)) and k.get(("page", "plain", 0, True))
    assert {k.get(("rle_value_bytes", b), 0) > 0 for b in (1, 2, 3)} == {True}
    assert {m for m in range(4) if k.get(("packed_start_mod4", m))} == {0, 1, 2, 3}
    rows = {min(gp.PAGE, n - p * gp.PAGE) for n in PAGE_NS for p in range(-(-n // gp.PAGE))}
    assert {63, 64, 8191, 8192, gp.PAGE} <= rows and any(r % 8 for r in rows)


def test_page_cases_oracle_files_read_back():
    for n in PAGE_NS:
        o = pages_oracle(n)
        t = pq.read_table(io.BytesIO(o["file"]()))
        for c in range(len(o["cols"])):
            v = o["cols"][c]
            null = po.is_null(v, gp.F4)
            col = t.column(f"c{c}")
            assert np.array_equal(np.asarray(col.is_valid()), ~null), (n, c)
            got = col.to_numpy(zero_copy_only=False).astype(np.float32).view(U32)
            assert np.array_equal(got[~null], v[~null]), (n, c)


def dev_pages(o, cuda, dict_jobs=None, dict_vals=None, n=None):
    """gsx_parquet_pages over pages_oracle's arguments (body zeroed, as documented) -> the body bytes."""
    import torch
    lib, _ptr, _stream = _dev()
    ranked, nulls, width, equal, lay = o["ranked"], o["nulls"], o["width"], o["equal"], o["lay"]
    nc, n = ranked.shape
    P, T = nulls.shape[1], -(-n // 2048)
    pg = lay.pages
    info = np.zeros((nc, P, 4), np.int64)
    data = pg[pg[:, 0] == 0]
    info[data[:, 1], data[:, 2], 0] = data[:, 3]
    info[:, :, 1] = nulls
    info[:, :, 2] = width
    info[:, :, 3] = equal
    tn = np.stack([np.add.reduceat(po.is_null(o["cols"][c], gp.F4), np.arange(0, n, 2048)) for c in range(nc)])
    dp = pg[pg[:, 0] == 1]
    first = {}
    vals = []
    for c in sorted(o["dicts"]):
        first[c] = sum(len(v) for v in vals)
        vals.append(o["dicts"][c])
    djobs = np.array([(first[c], off, cnt) for _, c, _, off, _, cnt in dp.tolist()], np.int64).reshape(-1, 3)
    body = torch.zeros(len(o["body"]) // 4 + 4, dtype=torch.int32, device=cuda)
    args = [_up(x, cuda) for x in (ranked.view(np.int32), tn.astype(np.int32), info, np.concatenate(vals).view(np.int32),
                                   djobs)]
    assert lib.gsx_parquet_pages(_ptr(args[0]), n, nc, _ptr(args[1]), _ptr(args[2]), _ptr(args[3]), _ptr(args[4]),
                                 len(djobs), int(djobs[:, 2].max()), _ptr(body), _stream()) == 0
    b = _host(body, np.uint8).tobytes()
    assert b[len(o["body"]):] == bytes(16)
    return b[:len(o["body"])]


@pytest.mark.gpu
@pytest.mark.parametrize("n", PAGE_NS)
def test_pages_every_form(n, cuda, gsx_lib):
    o = pages_oracle(n)
    got = dev_pages(o, cuda)
    want = o["body"]
    if got != want:
        bad = np.flatnonzero(np.frombuffer(got, np.uint8) != np.frombuffer(want, np.uint8))
        pages = [p for p in o["lay"].pages.tolist() if p[3] <= bad[0] < p[3] + p[4]]
        raise AssertionError(f"{len(bad)} body bytes differ, first at {bad[0]} in page {pages}")


def test_many_dictionary_jobs_need_the_y_stride():
    assert 70_000 > 65535


@pytest.mark.gpu
def test_pages_more_than_65535_dictionary_jobs(cuda, gsx_lib):
    """70 000 one-entry dictionary pages beside one data page: k_pq_dict_pages' blockIdx.y stride loop."""
    import torch
    lib, _ptr, _stream = _dev()
    nd = 70_000
    rng = np.random.default_rng(1)
    vals = _floats(rng, nd)
    djobs = np.stack([np.arange(nd), 16 + 16 * np.arange(nd), np.ones(nd)], 1).astype(np.int64)
    cols = np.zeros(1, U32)                                         # one PLAIN value at body offset 0
    info = np.array([[[0, 0, 0, 0]]], np.int64)
    body = torch.zeros(4 * (nd + 1), dtype=torch.int32, device=cuda)
    args = [_up(x, cuda) for x in (cols.view(np.int32), np.zeros(1, np.int32), info, vals.view(np.int32), djobs)]
    assert lib.gsx_parquet_pages(_ptr(args[0]), 1, 1, _ptr(args[1]), _ptr(args[2]), _ptr(args[3]), _ptr(args[4]), nd, 1,
                                 _ptr(body), _stream()) == 0
    got = _host(body).reshape(-1, 4)
    head = po.data_page(cols, np.zeros(1, bool), 0, None)
    assert got[0].tobytes() == head + bytes(16 - len(head))
    assert np.array_equal(got[1:, 0], vals) and not got[1:, 1:].any()


# ============================================================================================================ snappy
def plain_bytes(rng, m, before=b""):
    """m bytes none of which equals the byte 1 or 4 before it (no copy can start inside them)."""
    out = bytearray(before)
    k = len(out)
    for x in rng.integers(0, 256, m).tolist():
        while (len(out) >= 1 and x == out[-1]) or (len(out) >= 4 and x == out[-4]):
            x = (x + 1) & 255
        out.append(x)
    return bytes(out[k:])


def build(parts, seed):
    """Bytes from parts ("lit", k) | ("run", k) | ("rep4", k): plain bytes, k equal bytes (a distance-1 copy of k - 1),
    k bytes repeating a 4-byte word (a distance-4 copy of k - 4)."""
    rng = np.random.default_rng(seed)
    out = bytearray()
    for kind, k in parts:
        if kind == "lit":
            out += plain_bytes(rng, k, bytes(out[-4:]))
        elif kind == "run":
            c = next(x for x in range(256) if x not in out[-4:])
            out += bytes([c]) * k
        else:
            word = plain_bytes(rng, 4, bytes(out[-4:]))
            while len(set(word)) < 4:
                word = plain_bytes(rng, 4, bytes(out[-4:]) + bytes([rng.integers(0, 256)]))
            out += (word * (k // 4 + 1))[:k]
    return bytes(out)


def snappy_bodies():
    b = {}
    for L in (1, 60, 61, 256, 257):
        b[f"lit{L}"] = build([("lit", L - 1), ("run", 20), ("lit", 7)], L)
    b["lit65536"] = build([("lit", 1 << 16)], 0)
    for L in (8, 11, 12, 64, 65, 66, 67, 68, 128, 129, 130):
        b[f"copy1_{L}"] = build([("lit", 9), ("run", L + 1), ("lit", 9)], L)
        b[f"copy4_{L}"] = build([("lit", 9), ("rep4", L + 4), ("lit", 9)], L + 1000)
    b["whole_run"] = bytes([7]) * (1 << 16)
    b["end_word"] = build([("lit", 18), ("run", 47), ("lit", 30)], 5)             # the run ends at byte 64
    b["end_piece"] = build([("lit", 30), ("run", 100)], 6)
    b["far"] = build([("lit", 2000), ("run", 20), ("lit", 1500), ("rep4", 30)], 7)
    b["jobs"] = build([("lit", 3), ("run", 9)] * 5500, 8)[:1 << 16]
    rng = np.random.default_rng(12)
    for L in (1, 2, 3, 4, 5, 15, 16, 17, 31, 32, 33, 65535, 65536):
        b[f"len{L}"] = build([("lit", L // 3), ("run", L - L // 3 - L // 6), ("lit", L // 6)], L)[:L]
    b["multi"] = build([("lit", 70000), ("run", 3000), ("rep4", 80000), ("lit", 40000)], 13)
    b["random"] = rng.integers(0, 4, 200_000).astype(np.uint8).tobytes()
    return b


def test_snappy_bodies_reach_every_element():
    po.COUNTERS.clear()
    bodies = snappy_bodies()
    for body in bodies.values():
        po.snappy(body)
    k = po.COUNTERS
    for L in (1, 60, 61, 256, 257, 65536):
        assert k.get(("literal", L)), L
    for L in (8, 11, 12, 64, 65, 66, 67, 68, 128, 129, 130):
        assert k.get(("copy", 1, L)) and k.get(("copy", 4, L)), L
    assert k.get(("copy", 1, 65535)) and {1, 2, 3} <= {L for L in range(1, 4) if k.get(("copy_last", L))}
    assert k.get(("copy_end_word", False)) and k.get(("copy_end_word", True))
    assert k.get("snappy_scan_second_step") and k.get("snappy_walk_rounds")
    for L in (1, 2, 3, 4, 5, 15, 16, 17, 31, 32, 33, 65535, 65536):
        assert k.get(("piece_len", L)), L
    assert len(bodies["multi"]) > 2 * gp.PIECE and not k.get("snappy_tie")


def _decompress(stream: bytes, size: int) -> bytes:
    return pa.decompress(stream, decompressed_size=size, codec="snappy", asbytes=True)


def test_snappy_oracle_streams_decompress():
    for name, body in snappy_bodies().items():
        assert _decompress(po.snappy(body), len(body)) == body, name


def test_snappy_never_ties():
    """Distance 1 and 4 never tie at a chosen copy start: every string of up to 16 bytes over two symbols, and seeded
    random pieces over small alphabets."""
    po.COUNTERS.clear()
    seen = 0
    for m in range(1, 17):
        for s in itertools.product((0, 1), repeat=m):
            po.snappy_piece(np.array(s, np.uint8))
            seen += 1
    rng = np.random.default_rng(0)
    for k in range(300):
        v = rng.integers(0, 2 + k % 3, int(rng.integers(8, 4000)))
        po.snappy_piece(np.repeat(v, rng.integers(1, 6, len(v))).astype(np.uint8))
    assert seen == (1 << 17) - 2 and po.COUNTERS.get(("copy", 1, 8)) and po.COUNTERS.get(("copy", 4, 8))
    assert "snappy_tie" not in po.COUNTERS


def dev_snappy(bodies, cuda):
    """gsx_parquet_snappy on pages `bodies` (each padded to 16 bytes with its last byte) -> (per page the pieces'
    elements, page_csize)."""
    import torch
    lib, _ptr, _stream = _dev()
    buf, pcs = bytearray(), []
    for p, body in enumerate(bodies):
        off = len(buf)
        buf += body + body[-1:] * ((-len(body)) % 16)
        for s in range(0, len(body), gp.PIECE):
            pcs.append((p, off + s, min(gp.PIECE, len(body) - s)))
    pcs = np.array(pcs, np.int64)
    cap = lib.gsx_parquet_piece_bytes()
    scratch = _full((len(pcs) * cap,), cuda, SENT_B, dtype=torch.uint8)
    sizes = _full((len(pcs),), cuda)
    csize = torch.zeros(len(bodies), dtype=torch.int32, device=cuda)
    bd, pd = _up(np.frombuffer(bytes(buf), np.uint8), cuda), _up(pcs, cuda)
    assert lib.gsx_parquet_snappy(_ptr(bd), _ptr(pd), len(pcs), _ptr(scratch), _ptr(sizes), _ptr(csize),
                                  _stream()) == 0
    s, sc = _host(sizes), _host(scratch, np.uint8).reshape(len(pcs), cap)
    out = [[] for _ in bodies]
    for i, (p, _, _) in enumerate(pcs.tolist()):
        assert s[i] <= cap and (sc[i, s[i]:] == SENT_B).all(), i
        out[p].append(sc[i, :s[i]].tobytes())
    return out, _host(csize)


@pytest.mark.gpu
def test_snappy_every_element(cuda, gsx_lib):
    bodies = snappy_bodies()
    names = list(bodies)
    got, csize = dev_snappy([bodies[k] for k in names], cuda)
    for name, pieces, cs in zip(names, got, csize.tolist()):
        body = bodies[name]
        want = [po.snappy_piece(np.frombuffer(body[s:s + gp.PIECE], np.uint8)) for s in range(0, len(body), gp.PIECE)]
        assert pieces == want, name
        assert cs == sum(len(p) for p in pieces), name
        assert _decompress(gp.Thrift.varint(len(body)) + b"".join(pieces), len(body)) == body, name


# ========================================================================================================== assembly
def assemble_case():
    """Pages of one and of many pieces (one of them all zeros: each piece a few bytes), and more than 1024 heads."""
    rng = np.random.default_rng(4)
    bodies = [rng.integers(0, 3, int(rng.integers(1, 3 * gp.PIECE))).astype(np.uint8).tobytes() for _ in range(6)]
    bodies += [bytes(5 * gp.PIECE), plain_bytes(rng, 300), bytes([1]) * 17]
    heads = [rng.integers(0, 256, int(rng.integers(1, 40))).astype(np.uint8).tobytes() for _ in range(1500)]
    return bodies, heads


def test_assemble_case_reaches_its_paths():
    bodies, heads = assemble_case()
    pieces = [-(-len(b) // gp.PIECE) for b in bodies]
    assert len(heads) > 1024 and 1 in pieces and max(pieces) >= 3
    zero = po.snappy(bodies[6])
    assert len(zero) < 5 * 3100                                       # five pieces of 1 024 3-byte copy elements each


@pytest.mark.gpu
def test_assemble(cuda, gsx_lib):
    import torch
    lib, _ptr, _stream = _dev()
    bodies, heads = assemble_case()
    buf, pcs = bytearray(), []
    for p, body in enumerate(bodies):
        off = len(buf)
        buf += body + bytes((-len(body)) % 16)
        for s in range(0, len(body), gp.PIECE):
            pcs.append((p, off + s, min(gp.PIECE, len(body) - s)))
    pcs = np.array(pcs, np.int64)
    cap = lib.gsx_parquet_piece_bytes()
    scratch = torch.empty(len(pcs) * cap, dtype=torch.uint8, device=cuda)
    sizes = torch.zeros(len(pcs), dtype=torch.int32, device=cuda)
    csize = torch.zeros(len(bodies), dtype=torch.int32, device=cuda)
    bd, pd = _up(np.frombuffer(bytes(buf), np.uint8), cuda), _up(pcs, cuda)
    assert lib.gsx_parquet_snappy(_ptr(bd), _ptr(pd), len(pcs), _ptr(scratch), _ptr(sizes), _ptr(csize),
                                  _stream()) == 0
    streams = [po.snappy(b) for b in bodies]
    cs = [len(s) - po._vl(s) for s in streams]
    assert _host(csize).tolist() == cs
    # file: head k before page k (the rest after), pages where the heads leave room
    file, page_dst, hjobs, blob = bytearray(), [], [], bytearray()
    for k, h in enumerate(heads):
        hjobs.append((len(blob), len(file), len(h)))
        blob += h
        file += h
        if k < len(bodies):
            page_dst.append(len(file))
            file += streams[k][po._vl(streams[k]):]
    first = np.concatenate([[0], np.cumsum([-(-len(b) // gp.PIECE) for b in bodies])[:-1]]).astype(np.int64)
    out = _full((len(file) + 16,), cuda, SENT_B, dtype=torch.uint8)
    up = [_up(x, cuda) for x in (first, np.array(page_dst, np.int64), np.frombuffer(bytes(blob), np.uint8),
                                 np.array(hjobs, np.int64))]
    assert lib.gsx_parquet_assemble(_ptr(scratch), _ptr(pd), len(pcs), _ptr(sizes), *[_ptr(t) for t in up], len(hjobs),
                                    _ptr(out), _stream()) == 0
    got = _host(out, np.uint8).tobytes()
    assert got[len(file):] == bytes([SENT_B]) * 16
    assert got[:len(file)] == bytes(file)
    for body, d, c in zip(bodies, page_dst, cs):
        assert _decompress(gp.Thrift.varint(len(body)) + got[d:d + c], len(body)) == body


def heads_case(n=5000):
    """990 uint8 columns (256-entry dictionaries) and two float32 ones (PLAIN): about 2 000 page headers."""
    rng = np.random.default_rng(2)
    a = np.zeros(n, [(f"u{i}", "u1") for i in range(990)] + [("x", "<f4"), ("y", "<f4")])
    raw = a.view(np.uint8).reshape(n, -1)
    raw[:] = rng.integers(0, 256, raw.shape, dtype=np.uint8)
    a["x"], a["y"] = rng.standard_normal(n), np.nan
    return a


def test_heads_case_needs_more_than_1024_heads():
    a = heads_case()
    pages = pq.read_metadata(io.BytesIO(po.encode(a)))
    cc = [pages.row_group(0).column(c) for c in range(pages.num_columns)]
    assert sum(2 if c.has_dictionary_page else 1 for c in cc) + 2 > 1024


@pytest.mark.gpu
def test_encode_more_than_1024_heads(cuda, gsx_lib):
    a = heads_case()
    _encode_and_check(a, a, cuda)


# ============================================================================================================ refusals
def test_encode_refuses_before_upload(gsx_lib):
    big = np.lib.stride_tricks.as_strided(np.zeros(1, [("x", "<f4")]), shape=(gp.MAX_ROWS + 1,), strides=(0,))
    with pytest.raises(ValueError, match="2\\^31"):
        gp.encode(big, device="cpu")
    with pytest.raises(ValueError, match="1025 columns"):
        gp.encode(np.zeros(2, [(f"u{i}", "u1") for i in range(1025)]), device="cpu")
    with pytest.raises(ValueError, match="1028 bytes"):
        gp.encode(np.zeros(2, [(f"f{i}", "<f4") for i in range(257)]), device="cpu")
    wide = np.dtype({"names": ["x"], "formats": ["<f4"], "offsets": [0], "itemsize": 1025})
    with pytest.raises(ValueError, match="1025 bytes"):
        gp.encode(np.zeros(2, wide), device="cpu")


# ======================================================================================================= 2^31 rows
@pytest.mark.gpu
@pytest.mark.slow
def test_encode_max_rows(cuda, gsx_lib):
    """gsx.parquet.encode at MAX_ROWS: one uint8 column (row * 37) % 256 built on the device, so every row group is
    the same 256-entry dictionary chunk of 8-bit bit-packed pages, the body ~2 GiB, bit positions past 2^32."""
    import torch
    from gsx.readers import Decoded
    free, _ = torch.cuda.mem_get_info(cuda)
    if free < 24 << 30:
        pytest.skip(f"{free >> 30} GiB free; encoding 2^31 rows needs about 16 GiB (estimated)")
    n = gp.MAX_ROWS
    rows = torch.empty((n, 1), dtype=torch.uint8, device=cuda)
    step = 1 << 28
    for s in range(0, n, step):
        r = torch.arange(s, s + step, dtype=torch.int64, device=cuda)
        rows[s:s + step, 0] = ((r * 37) % 256).to(torch.uint8)
        del r
    dt = np.dtype([("red", "u1")])
    blob = gp.encode(Decoded(rows, dt, None)).to_host()
    del rows
    torch.cuda.empty_cache()
    g = np.zeros(gp.ROW_GROUP, dt)
    g["red"] = (np.arange(gp.ROW_GROUP) * 37) % 256
    one = po.encode(g)
    m1 = pq.read_metadata(io.BytesIO(one)).row_group(0).column(0)
    want = one[m1.dictionary_page_offset:m1.dictionary_page_offset + m1.total_compressed_size]
    meta = pq.read_metadata(io.BytesIO(blob))
    assert meta.num_rows == n and meta.num_row_groups == n // gp.ROW_GROUP
    for k in range(meta.num_row_groups):
        cc = meta.row_group(k).column(0)
        assert cc.dictionary_page_offset is not None and "RLE_DICTIONARY" in cc.encodings
        got = blob[cc.dictionary_page_offset:cc.dictionary_page_offset + cc.total_compressed_size]
        assert got == want, k
        s = cc.statistics
        assert (s.min, s.max, s.null_count, meta.row_group(k).num_rows) == (0, 255, 0, gp.ROW_GROUP), k
    f = pq.ParquetFile(io.BytesIO(blob))
    for k in (0, meta.num_row_groups - 1):
        v = f.read_row_group(k).column("red").to_numpy()
        assert np.array_equal(v, g["red"]), k
