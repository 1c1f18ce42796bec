"""NumPy restatement of gsx's Parquet writer (gsx/parquet.py + csrc/gsx_parquet.cu): the column split and statistics,
the dictionary choice, the page bodies (RLE / bit-packed hybrid) and the Snappy elements, byte for byte as the
device writes them.  The page headers and the footer come from gsx.parquet's host code (the Thrift compact protocol
of the same file), which the device path uses as well.

    blob = encode(a)            # a: 1-D structured array -> the file's bytes

Each kernel has its restatement here: split_kernel (k_pq_split: the columns, per-tile nulls and min / max keys),
distinct_counts (k_pq_insert), dictionary (k_pq_collect + k_pq_rank), page_ranks (k_pq_index), data_page and the
dictionary page bytes (k_pq_data_pages, k_pq_dict_pages), snappy_piece (k_pq_snappy) and write_file (k_pq_assemble
with the host's headers).  COUNTERS counts the forms they reach, so tests can show that a case hits its path.
"""
from __future__ import annotations

import numpy as np

from gsx import parquet as gp

COUNTERS: dict = {}      # what the calls since the last clear reached


def _count(key, n: int = 1) -> None:
    COUNTERS[key] = COUNTERS.get(key, 0) + n


# ------------------------------------------------------------------------------------------- split and statistics
def split(a: np.ndarray, plan) -> np.ndarray:
    """uint32 [C, n]: each column's 32-bit patterns (float32 bits, or uint8 widened)."""
    raw = np.ascontiguousarray(a).view(np.uint8).reshape(len(a), a.dtype.itemsize)
    cols = np.empty((len(plan), len(a)), np.uint32)
    for c, col in enumerate(plan):
        if col.kind == gp.F4:
            cols[c] = raw[:, col.offset:col.offset + 4].copy().view("<u4").reshape(-1)
        else:
            cols[c] = raw[:, col.offset]
    return cols


def is_null(v: np.ndarray, kind: int) -> np.ndarray:
    return (v & 0x7FFFFFFF) > 0x7F800000 if kind == gp.F4 else np.zeros(v.shape, bool)


def key(v: np.ndarray, kind: int) -> np.ndarray:
    """Order-preserving uint32 key of a pattern: float32 with the sign bit flipped (positives) or all bits (negatives)."""
    if kind != gp.F4:
        return v.astype(np.int64)
    return np.where(v >> 31 == 0, v ^ 0x80000000, ~v & 0xFFFFFFFF).astype(np.int64)


TILE = 2048                  # rows per k_pq_split / k_pq_data_pages CTA
STAGE = 64                   # rows k_pq_split stages in shared memory at a time


def split_smem(ncols: int, row_bytes: int) -> int:
    """k_pq_split's dynamic shared memory (gsx_parquet_split); above 48 KiB the entry point raises the limit."""
    return ncols * 12 + 4 + ncols * 8 + 16 + STAGE * row_bytes + 16


def split_kernel(raw: np.ndarray, spec) -> tuple:
    """gsx_parquet_split on raw uint8 [n, row_bytes] rows and spec [(offset, kind)]: out uint32 [C, n], tile_nulls
    uint32 [C, tiles], keys uint32 [2, C, groups] (least / greatest key of the chunk's non-null values; 0xFFFFFFFF and 0
    for a chunk without one)."""
    n = raw.shape[0]
    G = max(1, -(-n // gp.ROW_GROUP))
    T = -(-n // TILE)
    out = np.empty((len(spec), n), np.uint32)
    tnull = np.zeros((len(spec), T), np.uint32)
    keys = np.empty((2, len(spec), G), np.uint32)
    keys[0], keys[1] = 0xFFFFFFFF, 0
    if split_smem(len(spec), raw.shape[1] if raw.ndim == 2 else 1) > 48 * 1024:
        _count("split_smem_over_48k")
    for c, (off, kind) in enumerate(spec):
        out[c] = raw[:, off] if kind == gp.U1 else raw[:, off:off + 4].copy().view("<u4").reshape(-1)
        null = is_null(out[c], kind)
        tnull[c] = np.add.reduceat(null, np.arange(0, n, TILE)) if n else tnull[c]
        for g in range(G):
            s = slice(g * gp.ROW_GROUP, (g + 1) * gp.ROW_GROUP)
            v = out[c, s][~null[s]]
            if len(v):
                k = key(v, kind)
                keys[0, c, g], keys[1, c, g] = k.min(), k.max()
            elif n:
                _count("split_chunk_without_value")
    return out, tnull, keys


def distinct_counts(cols: np.ndarray, kinds) -> np.ndarray:
    """k_pq_insert: int64 [C, G] distinct non-null patterns of each chunk (the kernel's count is exact up to DICT_MAX
    and only known to be above it otherwise)."""
    n = cols.shape[1]
    G = max(1, -(-n // gp.ROW_GROUP))
    out = np.zeros((len(cols), G), np.int64)
    for c in range(len(cols)):
        for g in range(G):
            v = cols[c, g * gp.ROW_GROUP:(g + 1) * gp.ROW_GROUP]
            out[c, g] = len(np.unique(v[~is_null(v, kinds[c])]))
    return out


def dictionary(v: np.ndarray, kind: int) -> tuple:
    """k_pq_collect + radix sort + k_pq_rank + k_pq_index for one chunk's patterns v: (the dictionary, ascending
    patterns; v with every non-null value replaced by its rank)."""
    null = is_null(v, kind)
    d = np.unique(v[~null])
    _count(("dictionary_width", gp.bit_width(len(d))))
    return d, np.where(null, v, np.searchsorted(d, v)).astype(np.uint32)


def page_ranks(ranks: np.ndarray, null: np.ndarray) -> np.ndarray:
    """k_pq_index's page_idx for one column: uint32 [2, pages] = least and greatest rank of each page, 0xFFFFFFFF and 0
    (what the caller filled) for a page without a value."""
    P = -(-len(ranks) // gp.PAGE)
    out = np.empty((2, P), np.uint32)
    out[0], out[1] = 0xFFFFFFFF, 0
    for p in range(P):
        s = slice(p * gp.PAGE, (p + 1) * gp.PAGE)
        r = ranks[s][~null[s]]
        if len(r):
            out[:, p] = r.min(), r.max()
            _count("index_page_equal" if r.min() == r.max() else "index_page_mixed")
        else:
            _count("index_page_empty")
    return out


# ----------------------------------------------------------------------------------------------------- hybrid runs
def _bitpack(v: np.ndarray, w: int) -> bytes:
    """v as one bit-packed run's payload: ceil(len / 8) groups of 8 values, w bits each, LSB first."""
    m = (len(v) + 7) // 8 * 8
    p = np.zeros(m, np.int64)
    p[:len(v)] = v
    bits = ((p[:, None] >> np.arange(w)) & 1).astype(np.uint8).reshape(-1)
    return np.packbits(bits, bitorder="little").tobytes()


def data_page(v: np.ndarray, null: np.ndarray, w: int, idx) -> bytes:
    rows, nn = len(v), int((~null).sum())
    if null.any():
        g = (rows + 7) // 8
        defs = gp.Thrift.varint(2 * g + 1) + _bitpack((~null).astype(np.int64), 1)
    else:
        defs = gp.Thrift.varint(2 * rows) + b"\x01"
    out = len(defs).to_bytes(4, "little") + defs
    hn = bool(null.any())
    if w == 0:
        _count(("page", "plain", 0, hn))
        return out + v[~null].astype("<u4").tobytes()
    out += bytes([w])
    i = idx[~null]
    if nn == 0:
        _count(("page", "empty", w, hn))
        return out
    if (i == i[0]).all():
        _count(("page", "rle", w, hn))
        _count(("rle_value_bytes", (w + 7) // 8))
        return out + gp.Thrift.varint(2 * nn) + int(i[0]).to_bytes((w + 7) // 8, "little")
    head = gp.Thrift.varint(2 * ((nn + 7) // 8) + 1)
    _count(("page", "packed", w, hn))
    _count(("packed_start_mod4", (len(out) + len(head)) % 4))
    return out + head + _bitpack(i, w)


# ---------------------------------------------------------------------------------------------------------- snappy
def _run_lengths(eq: np.ndarray) -> np.ndarray:
    """L[i] = number of consecutive True from i on."""
    n = len(eq)
    pos = np.where(eq, n, np.arange(n))
    nxt = np.minimum.accumulate(pos[::-1])[::-1]
    return nxt - np.arange(n)


def _literal(b) -> bytes:
    m = len(b) - 1
    _count(("literal", len(b)))
    tag = bytes([m << 2]) if m < 60 else bytes([60 << 2, m]) if m < 256 else bytes([61 << 2, m & 255, m >> 8])
    return tag + bytes(b)


def _copy(d: int, L: int) -> bytes:
    out = bytearray()
    _count(("copy", d, L))
    while L > 64:
        out += bytes([(63 << 2) | 2, d, 0])
        L -= 64
    _count(("copy_last", L))
    if 4 <= L <= 11:
        out += bytes([((L - 4) << 2) | 1, d])
    else:
        out += bytes([((L - 1) << 2) | 2, d, 0])
    return bytes(out)


def snappy_piece(b: np.ndarray) -> bytes:
    """One piece's elements: greedy from the left, a copy where the bytes from i on repeat those 1 or 4 bytes back
    for >= 8 bytes inside the piece (the longer of the two), literals elsewhere.  The two never tie at a chosen start j:
    the bytes j - 1 and j - 2 differ there (else j - 1 was the candidate, or the copy before went on), so where a
    distance-1 copy starts the distance-4 run is at most 2 bytes long (COUNTERS["snappy_tie"] would count one)."""
    n = len(b)
    e1 = np.zeros(n, bool)
    e4 = np.zeros(n, bool)
    e1[1:] = b[1:] == b[:-1]
    e4[4:] = b[4:] == b[:-4]
    L1, L4 = _run_lengths(e1), _run_lengths(e4)
    cand = np.flatnonzero((L1 >= 8) | (L4 >= 8))
    out, i, lit, k, jobs = bytearray(), 0, 0, 0, 0
    _count(("piece_len", n))
    while True:
        k = int(np.searchsorted(cand, i, "left"))
        if k >= len(cand):
            break
        j = int(cand[k])
        if (j >> 5) - (i >> 5) >= 32:
            _count("snappy_scan_second_step")        # warp 0's 32-word scan does not reach j in its first step
        if L1[j] == L4[j]:
            _count("snappy_tie")
        L, d = (int(L1[j]), 1) if L1[j] >= L4[j] else (int(L4[j]), 4)
        if j > lit:
            out += _literal(b[lit:j])
            jobs += 1
        out += _copy(d, L)
        if (j + L) % 32 == 0:
            _count(("copy_end_word", j + L == n))
        i = lit = j + L
    if n > lit:
        out += _literal(b[lit:])
        jobs += 1
    if jobs > 1024:
        _count("snappy_walk_rounds")                 # more literal jobs than one walk round records
    return bytes(out)


def snappy(body: bytes) -> bytes:
    b = np.frombuffer(body, np.uint8)
    return gp.Thrift.varint(len(b)) + b"".join(snappy_piece(b[s:s + gp.PIECE]) for s in range(0, len(b), gp.PIECE))


# ---------------------------------------------------------------------------------------------------------- encode
def kernel_outputs(a: np.ndarray, plan):
    """What the device hands back to the host: per page nulls [C, P], per chunk distinct [C, G] (DICT_MAX + 1 for
    more), min / max keys [C, G, 2]; plus the columns, their dictionaries and indices for the page bodies."""
    n = len(a)
    G, P = gp.shape(n)
    cols = split(a, plan)
    nulls = np.zeros((len(plan), P), np.int64)
    distinct = np.zeros((len(plan), G), np.int64)
    keys = np.zeros((len(plan), G, 2), np.int64)
    dicts = {}
    for c, col in enumerate(plan):
        null = is_null(cols[c], col.kind)
        for p in range(P):
            nulls[c, p] = null[p * gp.PAGE:(p + 1) * gp.PAGE].sum()
        for g in range(G):
            s = slice(g * gp.ROW_GROUP, (g + 1) * gp.ROW_GROUP)
            v = cols[c, s][~null[s]]
            if len(v):
                k = key(v, col.kind)
                keys[c, g] = k.min(), k.max()
            u = np.sort(v)          # np.unique, by sorting: NumPy's hashed unique is far slower on 1 M values
            u = u[np.concatenate([[True], u[1:] != u[:-1]])] if len(u) else u
            distinct[c, g] = len(u) if len(u) <= gp.DICT_MAX else gp.DICT_MAX + 1
            if len(u) <= gp.DICT_MAX:
                dicts[(c, g)] = u
    return cols, nulls, distinct, keys, dicts


def encode(a: np.ndarray) -> bytes:
    plan = gp.column_plan(a.dtype)
    n = len(a)
    if n > gp.MAX_ROWS:
        raise ValueError("parquet: more than 2^31 rows")
    cols, nulls, distinct, keys, dicts = kernel_outputs(a, plan)
    width = gp.choose_dictionary(distinct, gp.page_rows(n)[None, :] - nulls)
    return write_file(plan, n, cols, nulls, distinct, keys, dicts, width)


def write_file(plan, n, cols, nulls, distinct, keys, dicts, width) -> bytes:
    """The file of kernel_outputs' results with the dictionary bit widths `width` [C, G] (0: PLAIN)."""
    G, P = gp.shape(n)
    idx, equal = {}, np.zeros((len(plan), P), bool)
    for c, col in enumerate(plan):
        for g in range(G):
            if width[c, g]:
                s = slice(g * gp.ROW_GROUP, (g + 1) * gp.ROW_GROUP)
                idx[(c, g)] = np.searchsorted(dicts[(c, g)], cols[c, s])
                null = is_null(cols[c, s], col.kind)
                for p in range(4 * g, min(4 * g + 4, P)):
                    q = slice((p - 4 * g) * gp.PAGE, (p - 4 * g + 1) * gp.PAGE)
                    i = idx[(c, g)][q][~null[q]]
                    equal[c, p] = len(i) > 0 and (i == i[0]).all()
    lay = gp.layout(n, distinct, nulls, width, equal)
    bodies = []
    for kind, c, gpg, _, _, _ in lay.pages.tolist():
        if kind:
            bodies.append(dicts[(c, gpg)].astype("<u4").tobytes())
            continue
        g = gpg // 4
        s = slice(gpg * gp.PAGE, (gpg + 1) * gp.PAGE)
        v = cols[c, s]
        i = idx[(c, g)][(gpg - 4 * g) * gp.PAGE:(gpg - 4 * g + 1) * gp.PAGE] if width[c, g] else None
        bodies.append(data_page(v, is_null(v, plan[c].kind), int(width[c, g]), i))
    streams = [snappy(b) for b in bodies]
    blobs, dst, size = gp.file_parts(plan, lay, gp.chunk_nulls(nulls, G), keys,
                                     np.array([len(s) for s in streams], np.int64))
    out = bytearray(size)
    for off, b in blobs:
        out[off:off + len(b)] = b
    for s, d in zip(streams, dst.tolist()):
        body = s[_vl(s):]
        out[d:d + len(body)] = body
    return bytes(out)


def _vl(stream: bytes) -> int:
    """Bytes of the length varint a Snappy stream starts with."""
    k = 0
    while stream[k] & 0x80:
        k += 1
    return k + 1


# ---------------------------------------------------------------------------------------------------------- inputs
STD = (["x", "y", "z", "nx", "ny", "nz", "f_dc_0", "f_dc_1", "f_dc_2"] + [f"f_rest_{i}" for i in range(45)]
       + ["opacity", "scale_0", "scale_1", "scale_2", "rot_0", "rot_1", "rot_2", "rot_3"])
LARGE = "distinct_262145"


def _cloud(n: int, seed: int, names, u1=(), grid=0.0) -> np.ndarray:
    rng = np.random.default_rng(seed)
    a = np.zeros(n, [(f, "<f4") for f in names] + [(f, "u1") for f in u1])
    for f in names:
        v = rng.standard_normal(n)
        a[f] = np.round(v * grid) / grid if grid else v
    for f in u1:
        a[f] = rng.integers(0, 256, n)
    return a


def golden_inputs() -> dict:
    """The fixture's inputs, by name (deterministic)."""
    sh = lambda d: [f for f in STD if not f.startswith("f_rest_") or int(f[7:]) < {0: 0, 1: 9, 2: 24, 3: 45}[d]]
    out = {"std_rgb": _cloud(300, 1, STD, ("red", "green", "blue")), "std": _cloud(300, 2, STD)}
    for d in range(3):
        out[f"sh{d}"] = _cloud(64, 3 + d, sh(d))
    out["no_normals"] = _cloud(50, 6, [f for f in STD if f not in ("nx", "ny", "nz")])
    out["extras"] = _cloud(40, 7, sh(0) + ["scal_w"], ("red", "green", "blue", "mask"))
    f64 = np.zeros(20, [("x", "<f4"), ("y", "<f4"), ("z", "<f4"), ("opacity", "<f4"), ("d", "<f8")])
    i16 = np.zeros(20, [("x", "<f4"), ("opacity", "<f4"), ("k", "<i2")])
    f64["d"] = np.arange(20) / 3
    i16["k"] = np.arange(20) - 7
    out["float64_extra"], out["int16_extra"] = f64, i16
    out["alpha_collision"] = _cloud(10, 8, ["x", "y", "z", "opacity", "alpha"])
    edge = _cloud(1000, 9, sh(3), ("red", "green", "blue"), grid=40.0)
    edge["x"][::97] = np.nan
    edge["y"][:] = np.nan
    edge["z"][:4] = [np.inf, -np.inf, -0.0, 0.0]
    edge["nx"][:] = 0.0
    edge["ny"][:] = 1.25
    edge["nz"][:] = np.where(np.arange(1000) % 2, -0.0, 0.0)
    edge["f_dc_0"][:3] = np.array([1e-45, -1e-45, 1e-40], np.float32)
    edge["f_dc_1"][:] = np.nan
    edge["f_dc_1"][500] = 3.5
    edge["opacity"][:500] = -0.0
    edge["opacity"][500:] = 0.0
    edge["red"][:] = 7
    out["edges_1000"] = edge
    for n in (0, 1, 7):
        out[f"n{n}"] = _cloud(n, 10 + n, STD, ("red", "green", "blue"))
    big = np.zeros(262145, [("x", "<f4"), ("y", "<f4"), ("opacity", "<f4"), ("scale_0", "<f4")])
    r = np.arange(262145)
    big["x"] = (r % 262144) * np.float32(0.5)
    big["y"] = r * np.float32(0.25)
    big["opacity"] = np.where(r % 5 == 0, np.nan, np.round(np.random.default_rng(13).standard_normal(262145) * 8))
    big["scale_0"] = -1.5
    out[LARGE] = big
    return out


def table_digest(table) -> dict:
    """SHA-256 of each column's values (nulls zeroed) and of its validity, as pyarrow reads them."""
    import hashlib
    out = {}
    for name in table.column_names:
        col = table.column(name).combine_chunks()
        valid = np.asarray(col.is_valid())
        vals = np.asarray(col.fill_null(0))
        out[name] = hashlib.sha256(vals.tobytes() + valid.tobytes()).hexdigest()
    return out


def chunk_facts(meta) -> list:
    """Per row group: rows, and per column chunk (has statistics, has_min_max, min and max as bit patterns,
    null_count, codec)."""
    def bits(v):
        return np.float32(v).view(np.uint32).item() if isinstance(v, float) else int(v)
    out = []
    for g in range(meta.num_row_groups):
        rg = meta.row_group(g)
        cols = []
        for c in range(rg.num_columns):
            cc = rg.column(c)
            s = cc.statistics
            if s is None:
                cols.append((False, False, 0, 0, 0, cc.compression))
            else:
                mm = s.has_min_max
                cols.append((True, mm, bits(s.min) if mm else 0, bits(s.max) if mm else 0, s.null_count,
                             cc.compression))
        out.append((rg.num_rows, cols))
    return out
