"""The .parquet writer on the device: ParquetFormat.write (formats/parquet.py:59-112) from device-resident records.

    enc = encode(records)                 # DeviceRecords, readers.Decoded or a structured array -> Encoded
    write_parquet("out.parquet", enc)     # the file's bytes: enc.to_host()

The reference renames the fields, orders the columns and hands the frame to pandas' to_parquet (pyarrow, defaults).
gsx writes a file that holds the same table: the same column names, order and types (float32 -> FLOAT, uint8 ->
INT32 with Int(8, unsigned)), NaN as null, row groups of 1 048 576 rows, per column chunk the same min, max and
null_count, SNAPPY, and a `pandas` footer entry from which pd.read_parquet rebuilds an equal frame.  The bytes are
gsx's own: each column chunk is dictionary-encoded or PLAIN, whichever is smaller for its data, and Snappy matches
only runs and repeated 32-bit values (csrc/gsx_parquet.cu).

Everything here but the kernels is host code that does not import pandas, pyarrow or thrift: the column plan, the
encoding choice, the page layout and the Thrift compact protocol of the page headers and the footer.  The device does
the column split, statistics, dictionaries, page bodies, Snappy and the assembly of the file; what crosses PCIe is
per-chunk counts and statistics, per-page flags and compressed sizes, the headers, and the finished file.
tests/parquet_oracle.py restates the kernels in NumPy, byte for byte.
"""
from __future__ import annotations

import ctypes as C
import json
import struct
from dataclasses import dataclass

import numpy as np

ROW_GROUP = 1 << 20          # rows per row group (pyarrow's default)
PAGE = 1 << 18               # rows per data page: 1 MiB of float32
DICT_MAX = 1 << 18           # distinct values a dictionary may hold: 1 MiB (pyarrow's dictionary page limit)
PIECE = 1 << 16              # Snappy piece, bytes: each is encoded on its own
MAX_ROWS = 1 << 31
MAX_COLS = 1024              # columns and row bytes gsx_parquet_split takes
ROW_MAX = 1024
CREATED_BY = "gsx (3dgsconverter H100 backend)"

F4, U1 = 0, 1                # column kinds, as gsx_parquet_split numbers them
# Parquet enums (parquet.thrift)
T_INT32, T_FLOAT = 1, 4
PLAIN, RLE, RLE_DICTIONARY = 0, 3, 8
SNAPPY = 1
DATA_PAGE, DICTIONARY_PAGE = 0, 2
OPTIONAL = 1
UINT_8 = 11


# ------------------------------------------------------------------------------------------------------ column plan
@dataclass(frozen=True)
class Column:
    source: str      # field of the input rows
    offset: int      # its byte offset in a row
    kind: int        # F4 or U1
    name: str        # the Parquet column


def _rename() -> dict:
    """parquet.py:63-77: the reference's field -> column renaming."""
    m = {"x": "x", "y": "y", "z": "z", "rot_0": "cov_q3", "rot_1": "cov_q0", "rot_2": "cov_q1", "rot_3": "cov_q2",
         "scale_0": "cov_s0", "scale_1": "cov_s1", "scale_2": "cov_s2", "opacity": "alpha",
         "f_dc_0": "r_sh0", "f_dc_1": "g_sh0", "f_dc_2": "b_sh0", "nx": "nx", "ny": "ny", "nz": "nz"}
    for i in range(15):
        m[f"f_rest_{i}"], m[f"f_rest_{15 + i}"], m[f"f_rest_{30 + i}"] = f"r_sh{i + 1}", f"g_sh{i + 1}", f"b_sh{i + 1}"
    return m


RENAME = _rename()


def _order(has_normals: bool) -> list:
    """parquet.py:79-91: the fixed column order."""
    order = ["x", "y", "z"] + (["nx", "ny", "nz"] if has_normals else [])
    order += ["cov_q0", "cov_q1", "cov_q2", "cov_q3", "cov_s0", "cov_s1", "cov_s2", "alpha"]
    return order + [f"{c}_sh{i}" for c in "rgb" for i in range(16)]


def column_plan(dtype: np.dtype) -> list:
    """[Column] in file order, as parquet.py:93-108 selects and orders the renamed frame's columns: the mapped ones
    present in the fixed order (the normals only when `nx` is a field), then every field that maps to no target name,
    in input order.  ValueError (the drop-in then runs the reference) for: two fields that end up with the same column
    name (pandas raises there too), a column that is not float32 or uint8, non-native byte order, subarray fields."""
    names = dtype.names or ()
    if not names:
        raise ValueError("parquet: a structured dtype with fields is needed")
    renamed = [RENAME.get(f, f) for f in names]
    dup = sorted({r for r in renamed if renamed.count(r) > 1})
    if dup:
        raise ValueError(f"parquet: duplicate column names {dup}")
    by_name = dict(zip(renamed, names))
    targets = set(RENAME.values())
    chosen = [c for c in _order("nx" in names) if c in by_name] + [r for r in renamed if r not in targets]
    plan = []
    for col in chosen:
        f = by_name[col]
        t, off = dtype.fields[f][0], dtype.fields[f][1]
        if t.shape or t.byteorder not in "=<|":
            raise ValueError(f"parquet: field {f} is {t.str}; only native scalar fields are written on the device")
        if t == np.dtype("<f4"):
            kind = F4
        elif t == np.dtype("u1"):
            kind = U1
        else:
            raise ValueError(f"parquet: field {f} is {t.str}; only float32 and uint8 are written on the device")
        plan.append(Column(f, off, kind, col))
    return plan


# ------------------------------------------------------------------------------------------------ thrift (compact)
class Thrift:
    """The Thrift compact protocol, writing only: a struct is a list of (field id, type, value), in ascending ids."""
    BOOL, I8, I16, I32, I64, BINARY, LIST, STRUCT = "bool", 3, 4, 5, 6, 8, 9, 12

    @staticmethod
    def varint(v: int) -> bytes:
        out = bytearray()
        while True:
            b = v & 0x7F
            v >>= 7
            if v:
                out.append(b | 0x80)
            else:
                out.append(b)
                return bytes(out)

    @classmethod
    def zigzag(cls, v: int) -> bytes:
        return cls.varint((v << 1) ^ (v >> 63))

    @classmethod
    def value(cls, t, v) -> bytes:
        if t in (cls.I16, cls.I32, cls.I64):
            return cls.zigzag(int(v))
        if t == cls.I8:
            return struct.pack("<b", v)
        if t == cls.BINARY:
            b = v.encode() if isinstance(v, str) else bytes(v)
            return cls.varint(len(b)) + b
        if t == cls.STRUCT:
            return cls.struct(v)
        raise ValueError(f"thrift: no value encoding for type {t}")

    @classmethod
    def struct(cls, fields) -> bytes:
        out, last = bytearray(), 0
        for fid, t, v in fields:
            if v is None:
                continue
            wire = (1 if v else 2) if t == cls.BOOL else (cls.LIST if isinstance(t, tuple) else t)
            d = fid - last
            out += bytes([(d << 4) | wire]) if 0 < d <= 15 else bytes([wire]) + cls.zigzag(fid)
            last = fid
            if isinstance(t, tuple):          # (LIST, element type)
                et, n = t[1], len(v)
                out += bytes([(n << 4) | et]) if n < 15 else bytes([0xF0 | et]) + cls.varint(n)
                for e in v:
                    out += cls.value(et, e)
            elif t != cls.BOOL:
                out += cls.value(t, v)
        out.append(0)
        return bytes(out)


_T = Thrift
_LIST = _T.LIST


def page_header(ptype: int, usize: int, csize: int, num_values: int, encoding: int) -> bytes:
    """PageHeader: a data page v1 (definition levels RLE, no repetition levels) or a dictionary page."""
    if ptype == DATA_PAGE:
        sub = (5, _T.STRUCT, [(1, _T.I32, num_values), (2, _T.I32, encoding), (3, _T.I32, RLE), (4, _T.I32, RLE)])
    else:
        sub = (7, _T.STRUCT, [(1, _T.I32, num_values), (2, _T.I32, encoding)])
    return _T.struct([(1, _T.I32, ptype), (2, _T.I32, usize), (3, _T.I32, csize), sub])


def schema_elements(plan) -> list:
    """SchemaElement structs: the root group, then one optional leaf per column."""
    out = [[(4, _T.BINARY, "schema"), (5, _T.I32, len(plan))]]
    for c in plan:
        if c.kind == F4:
            out.append([(1, _T.I32, T_FLOAT), (3, _T.I32, OPTIONAL), (4, _T.BINARY, c.name)])
        else:
            logical = [(10, _T.STRUCT, [(1, _T.I8, 8), (2, _T.BOOL, False)])]      # LogicalType.INTEGER
            out.append([(1, _T.I32, T_INT32), (3, _T.I32, OPTIONAL), (4, _T.BINARY, c.name),
                        (6, _T.I32, UINT_8), (10, _T.STRUCT, logical)])
    return out


def pandas_metadata(plan, n: int) -> str:
    """The `pandas` key-value entry pyarrow writes for this frame: a range index, the columns Index (pandas 3's str
    dtype) and each column's pandas_type / numpy_type."""
    cols = [{"name": c.name, "field_name": c.name, "pandas_type": "float32" if c.kind == F4 else "uint8",
             "numpy_type": "float32" if c.kind == F4 else "uint8", "metadata": None} for c in plan]
    meta = {"index_columns": [{"kind": "range", "name": None, "start": 0, "stop": n, "step": 1}],
            "column_indexes": [{"name": None, "field_name": None, "pandas_type": "unicode", "numpy_type": "str",
                                "metadata": {"encoding": "UTF-8"}}],
            "columns": cols, "attributes": {}, "creator": {"library": "gsx", "version": "1.0"},
            "pandas_version": "3.0.2"}
    return json.dumps(meta)


# ----------------------------------------------------------------------------------------------------------- layout
def shape(n: int):
    """(row groups, pages per column) of n rows: one empty row group for n = 0; page k covers rows
    [k * PAGE, min((k + 1) * PAGE, n)), and row group g holds pages [4g, 4g + 4)."""
    return max(1, -(-n // ROW_GROUP)), -(-n // PAGE)


def page_rows(n: int) -> np.ndarray:
    P = -(-n // PAGE)
    return np.minimum(PAGE, n - PAGE * np.arange(P, dtype=np.int64))


def bit_width(d: int) -> int:
    """Bits per dictionary index: ceil(log2(d)), and 1 for a one-entry dictionary (as pyarrow writes it)."""
    return max(1, int(d - 1).bit_length())


def vlen(v) -> np.ndarray:
    """Bytes of the ULEB128 varint of each v (>= 0)."""
    v = np.asarray(v, np.int64)
    n = np.ones(v.shape, np.int64)
    for k in range(1, 10):
        n += v >= (1 << (7 * k))
    return n


def choose_dictionary(distinct: np.ndarray, nonnull: np.ndarray) -> np.ndarray:
    """Per column chunk (distinct [C, G]: distinct non-null patterns, or > DICT_MAX; nonnull [C, P] per page):
    the dictionary's bit width where the dictionary page plus each page's bit width byte and packed indices is
    smaller than PLAIN's 4 bytes a value, else 0 (PLAIN)."""
    C_, G = distinct.shape
    w = np.zeros((C_, G), np.int64)
    for c in range(C_):
        for g in range(G):
            d = int(distinct[c, g])
            nn = nonnull[c, 4 * g:4 * g + 4]
            if d < 1 or d > DICT_MAX:
                continue
            b = bit_width(d)
            if 4 * d + int(np.sum(1 + (nn * b + 7) // 8)) < 4 * int(nn.sum()):
                w[c, g] = b
    return w


def data_body_sizes(n: int, nulls: np.ndarray, width: np.ndarray, equal: np.ndarray) -> np.ndarray:
    """Uncompressed body bytes of every data page [C, P]: the 4-byte length and RLE hybrid of the definition levels
    (one RLE run, or one bit-packed run when the page has nulls), then the values: PLAIN, or the bit width byte and
    the indices as one bit-packed run (one RLE run when all of them are equal; nothing when there are none)."""
    rows = page_rows(n)[None, :]
    nn = rows - nulls
    defs = np.where(nulls > 0, vlen(((rows + 7) // 8) * 2 + 1) + (rows + 7) // 8, vlen(rows * 2) + 1)
    w = np.repeat(width, 4, axis=1)[:, :rows.shape[1]]
    packed = vlen(((nn + 7) // 8) * 2 + 1) + (nn + 7) // 8 * w
    run = vlen(nn * 2) + (w + 7) // 8
    vals = np.where(w == 0, 4 * nn, 1 + np.where(nn == 0, 0, np.where(equal, run, packed)))
    return 4 + defs + vals


@dataclass
class Layout:
    """What the host works out from the kernels' counts: the pages in file order and their bodies' place in the
    uncompressed body buffer."""
    n: int
    width: np.ndarray        # [C, G] dictionary bit width, 0 = PLAIN
    distinct: np.ndarray     # [C, G]
    pages: np.ndarray        # int64 [npages, 6]: kind (0 data, 1 dictionary), column, row group / page, body offset,
    #                          body bytes, rows (data) or entries (dictionary)


def layout(n: int, distinct, nulls, width, equal) -> Layout:
    """Pages in file order (row group by row group, column by column: the dictionary page, then the data pages) and
    the offset of each body in the body buffer (16-byte aligned)."""
    G, P = shape(n)
    C_ = width.shape[0]
    dsize = data_body_sizes(n, nulls, width, equal) if P else np.zeros((C_, 0), np.int64)
    rows = page_rows(n)
    pages = []
    for g in range(G):
        for c in range(C_):
            if width[c, g]:
                pages.append((1, c, g, 0, 4 * int(distinct[c, g]), int(distinct[c, g])))
            for p in range(4 * g, min(4 * g + 4, P)):
                pages.append((0, c, p, 0, int(dsize[c, p]), int(rows[p])))
    pg = np.array(pages, np.int64).reshape(-1, 6)
    if len(pg):
        sizes16 = (pg[:, 4] + 15) // 16 * 16
        pg[:, 3] = np.concatenate([[0], np.cumsum(sizes16)[:-1]])
    return Layout(n, width, distinct, pg)


def pieces(lay: Layout) -> np.ndarray:
    """int64 [npieces, 3]: (page, body offset, bytes) of every Snappy piece, page by page."""
    pg = lay.pages
    cnt = (pg[:, 4] + PIECE - 1) // PIECE
    page = np.repeat(np.arange(len(pg), dtype=np.int64), cnt)
    k = np.arange(len(page), dtype=np.int64) - np.repeat(np.cumsum(cnt) - cnt, cnt)
    off = pg[page, 3] + k * PIECE
    return np.stack([page, off, np.minimum(PIECE, pg[page, 4] - k * PIECE)], 1).astype(np.int64).reshape(-1, 3)


def _stat(kind: int, key: int) -> bytes:
    """A column's min or max as Parquet stores it, from the kernels' order-preserving key (float32: the sign bit
    flipped for positives, every bit for negatives)."""
    if kind == U1:
        return struct.pack("<i", key)
    bits = key ^ 0x80000000 if key & 0x80000000 else ~key & 0xFFFFFFFF
    return struct.pack("<I", bits)


def file_parts(plan, lay: Layout, nulls_chunk, keys, csize):
    """(head blobs [(file offset, bytes)] in file order, data offset of each page in the file, file size).
    nulls_chunk [C, G], keys [C, G, 2] (min and max key; ignored when the chunk has no value), csize [npages]: each
    page's compressed bytes (the Snappy stream: length varint and pieces).  The statistics follow Parquet's rule for
    float zeros: a zero minimum is written as -0.0, a zero maximum as +0.0."""
    n, pg = lay.n, lay.pages
    G, _ = shape(n)
    blobs, pos = [(0, b"PAR1")], 4
    dst = np.zeros(len(pg), np.int64)
    chunks = {}
    for i, (kind, c, gp, _, usize, cnt) in enumerate(pg.tolist()):
        g = gp if kind else gp // 4
        cc = chunks.setdefault((g, c), dict(first=pos, dict=None, data=None, u=0, z=0, enc={RLE}))
        enc = PLAIN if kind or not lay.width[c, g] else RLE_DICTIONARY
        cc["enc"].add(enc)
        if kind:
            cc["dict"] = pos
        elif cc["data"] is None:
            cc["data"] = pos
        head = page_header(DICTIONARY_PAGE if kind else DATA_PAGE, usize, int(csize[i]), cnt, enc)
        blobs.append((pos, head + Thrift.varint(usize)))     # the Snappy stream's length varint goes with the header
        cc["u"] += len(head) + usize
        cc["z"] += len(head) + int(csize[i])
        dst[i] = pos + len(head) + len(Thrift.varint(usize))
        pos += len(head) + int(csize[i])
    groups = []
    for g in range(G):
        rows = min(ROW_GROUP, n - g * ROW_GROUP) if n else 0
        cols, tu, tz = [], 0, 0
        for c, col in enumerate(plan):
            cc = chunks.get((g, c), dict(first=pos, dict=None, data=None, u=0, z=0, enc={PLAIN, RLE}))
            nul = int(nulls_chunk[c, g])
            stats = None
            if rows:
                stats = [(3, _T.I64, nul)]
                if nul < rows:
                    lo, hi = int(keys[c, g, 0]), int(keys[c, g, 1])
                    mn, mx = _stat(col.kind, lo), _stat(col.kind, hi)
                    if col.kind == F4:
                        if mn[:3] == b"\0\0\0" and mn[3] & 0x7F == 0:
                            mn = struct.pack("<I", 0x80000000)
                        if mx[:3] == b"\0\0\0" and mx[3] & 0x7F == 0:
                            mx = struct.pack("<I", 0)
                    stats += [(5, _T.BINARY, mx), (6, _T.BINARY, mn)]
            md = [(1, _T.I32, T_FLOAT if col.kind == F4 else T_INT32), (2, (_LIST, _T.I32), sorted(cc["enc"])),
                  (3, (_LIST, _T.BINARY), [col.name]), (4, _T.I32, SNAPPY), (5, _T.I64, rows),
                  (6, _T.I64, cc["u"]), (7, _T.I64, cc["z"]),
                  (9, _T.I64, cc["data"] if cc["data"] is not None else cc["first"]),
                  (11, _T.I64, cc["dict"]), (12, _T.STRUCT, stats)]
            cols.append([(2, _T.I64, 0), (3, _T.STRUCT, md)])
            tu, tz = tu + cc["u"], tz + cc["z"]
        first = min((chunks[(g, c)]["first"] for c in range(len(plan)) if (g, c) in chunks), default=pos)
        groups.append([(1, (_LIST, _T.STRUCT), cols), (2, _T.I64, tu), (3, _T.I64, rows), (5, _T.I64, first),
                       (6, _T.I64, tz), (7, _T.I16, g)])
    kv = [[(1, _T.BINARY, "pandas"), (2, _T.BINARY, pandas_metadata(plan, n))]]
    footer = _T.struct([(1, _T.I32, 1), (2, (_LIST, _T.STRUCT), schema_elements(plan)), (3, _T.I64, n),
                        (4, (_LIST, _T.STRUCT), groups), (5, (_LIST, _T.STRUCT), kv), (6, _T.BINARY, CREATED_BY),
                        (7, (_LIST, _T.STRUCT), [[(1, _T.STRUCT, [])]] * len(plan))])
    blobs.append((pos, footer + struct.pack("<I", len(footer)) + b"PAR1"))
    return blobs, dst, pos + len(footer) + 8


# ----------------------------------------------------------------------------------------------------------- device
@dataclass
class Encoded:
    file: object             # uint8 CUDA tensor: the whole .parquet file
    rows: int

    def to_host(self) -> bytes:
        """The file's bytes (one D2H)."""
        from .hostcopy import to_bytes
        return to_bytes(self.file)


SLOTS_LOG2 = 20              # dictionary table slots per column chunk: load <= 1/2 at 262 144 + the insert overshoot
TABLE_BYTES = 1 << 30        # dictionary tables of one batch of row groups


def encode(src, device="cuda") -> Encoded:
    """ParquetFormat.write's file (parquet.py:59-112), built on the device from `src`: DeviceRecords, readers.Decoded
    or a 1-D structured NumPy array (uploaded once), the inputs gsx.ply.encode takes.  ValueError, before anything is
    uploaded, for what column_plan refuses, for more than 2^31 rows, rows wider than 1024 bytes and more than 1024
    columns."""
    import torch
    from ._abi import lib, check, _ptr, _stream
    from .hostcopy import to_device, to_host
    from .ply import _device_rows
    n, dt = _source_shape(src)
    plan = column_plan(dt)
    if n > MAX_ROWS:
        raise ValueError(f"parquet: {n} rows; at most 2^31 are written on the device")
    if len(plan) > MAX_COLS:
        raise ValueError(f"parquet: {len(plan)} columns; at most {MAX_COLS} are written on the device")
    if dt.itemsize > ROW_MAX:
        raise ValueError(f"parquet: rows of {dt.itemsize} bytes; at most {ROW_MAX} are written on the device")
    rows, dt, _ = _device_rows(src, device)
    dev = rows.device
    nc, (G, P) = len(plan), shape(n)
    T = -(-n // 2048)
    i32, i64 = torch.int32, torch.int64
    with torch.cuda.device(dev):
        st = _stream()
        cols = torch.empty((nc, n), dtype=i32, device=dev)
        tile_nulls = torch.empty((nc, T), dtype=i32, device=dev)
        keys = torch.empty((2, nc, G), dtype=i32, device=dev)
        spec = (C.c_int32 * (2 * nc))(*[v for c in plan for v in (c.offset, c.kind)])
        check(lib.gsx_parquet_split(_ptr(rows), n, dt.itemsize, spec, nc, _ptr(cols), _ptr(tile_nulls), _ptr(keys), st),
              "gsx_parquet_split")
        tn = to_host(tile_nulls).view(np.uint32).astype(np.int64)
        nulls = np.add.reduceat(tn, np.arange(0, T, PAGE // 2048), axis=1) if n else np.zeros((nc, 0), np.int64)
        nonnull = page_rows(n)[None, :] - nulls
        distinct = np.zeros((nc, G), np.int64)
        width = np.zeros((nc, G), np.int64)
        page_idx = torch.empty((2, nc, P), dtype=i32, device=dev)
        page_idx[0].fill_(-1)
        page_idx[1].zero_()
        dvals, dvoff, dsum = [], {}, 0
        if n:
            batch = max(1, min(G, TABLE_BYTES // (nc * (8 << SLOTS_LOG2)), 65535 // nc))
            table = torch.empty((batch * nc) << SLOTS_LOG2, dtype=i64, device=dev)
            dcount = torch.zeros((nc, G), dtype=i32, device=dev)
            for g0 in range(0, G, batch):
                ng = min(batch, G - g0)
                table[:(ng * nc) << SLOTS_LOG2].zero_()
                check(lib.gsx_parquet_dict_insert(_ptr(cols), n, nc, g0, ng, _ptr(table), SLOTS_LOG2, _ptr(dcount), st),
                      "gsx_parquet_dict_insert")
                d = to_host(dcount[:, g0:g0 + ng]).view(np.uint32).astype(np.int64)
                distinct[:, g0:g0 + ng] = np.minimum(d, DICT_MAX + 1)
                w = choose_dictionary(distinct[:, g0:g0 + ng], nonnull[:, 4 * g0:4 * (g0 + ng)])
                width[:, g0:g0 + ng] = w
                cc, gg = np.nonzero(w)
                if not len(cc):
                    continue
                cnt = distinct[cc, g0 + gg]
                first = np.concatenate([[0], np.cumsum(cnt)[:-1]])
                jobs = np.stack([cc + nc * gg, first, first], 1).astype(np.int64)
                nkeys = int(cnt.sum())
                buf = torch.empty(nkeys, dtype=i32, device=dev)
                ws = torch.empty(lib.gsx_parquet_dictionary_workspace_bytes(nkeys), dtype=torch.uint8, device=dev)
                jobs_dev = to_device(jobs, dev)
                check(lib.gsx_parquet_dictionary(_ptr(table), SLOTS_LOG2, _ptr(jobs_dev), len(jobs), nkeys, _ptr(ws),
                                                 ws.numel(), _ptr(buf), st), "gsx_parquet_dictionary")
                for c, g, f in zip(cc.tolist(), gg.tolist(), first.tolist()):
                    dvoff[(c, g0 + g)] = dsum + f
                dvals.append(buf)
                dsum += nkeys
                sel = to_device((w > 0).astype(np.int32), dev)
                check(lib.gsx_parquet_dict_index(_ptr(cols), n, nc, g0, ng, _ptr(table), SLOTS_LOG2, _ptr(sel),
                                                 _ptr(page_idx), st), "gsx_parquet_dict_index")
            del table
        pi = to_host(page_idx)
        equal = pi[0] == pi[1]
        lay = layout(n, distinct, nulls, width, equal)
        pg = lay.pages
        body_bytes = int(pg[-1, 3] + (pg[-1, 4] + 15) // 16 * 16) if len(pg) else 0
        body = torch.zeros(max(body_bytes // 4, 1), dtype=i32, device=dev)
        if n:
            data = pg[pg[:, 0] == 0]
            info = np.zeros((nc, P, 4), np.int64)
            info[data[:, 1], data[:, 2], 0] = data[:, 3]
            info[:, :, 1] = nulls
            info[:, :, 2] = np.repeat(width, 4, axis=1)[:, :P]
            info[:, :, 3] = equal
            dp = pg[pg[:, 0] == 1]
            djobs = np.array([(dvoff[(c, g)], off, cnt) for _, c, g, off, _, cnt in dp.tolist()], np.int64).reshape(-1, 3)
            dv = (dvals[0] if len(dvals) == 1 else torch.cat(dvals)) if dvals else torch.empty(1, dtype=i32, device=dev)
            # every uploaded table stays referenced until its kernel has run: a freed block could be reused (and
            # overwritten by the next upload) before the stream reaches the kernel
            info_dev, djobs_dev = to_device(info, dev), to_device(djobs, dev)
            check(lib.gsx_parquet_pages(_ptr(cols), n, nc, _ptr(tile_nulls), _ptr(info_dev), _ptr(dv), _ptr(djobs_dev),
                                        len(djobs), int(djobs[:, 2].max(initial=1)), _ptr(body), st),
                  "gsx_parquet_pages")
            del cols, dv, dvals
        pcs = pieces(lay)
        cap = lib.gsx_parquet_piece_bytes()
        scratch = torch.empty(max(len(pcs), 1) * cap, dtype=torch.uint8, device=dev)
        sizes = torch.zeros(max(len(pcs), 1), dtype=i32, device=dev)
        pcsize = torch.zeros(max(len(pg), 1), dtype=i32, device=dev)
        pcs_dev = to_device(pcs, dev)
        check(lib.gsx_parquet_snappy(_ptr(body), _ptr(pcs_dev), len(pcs), _ptr(scratch), _ptr(sizes), _ptr(pcsize), st),
              "gsx_parquet_snappy")
        del body
        csize = to_host(pcsize)[:len(pg)].astype(np.int64) + vlen(pg[:, 4])
        blobs, dst, size = file_parts(plan, lay, chunk_nulls(nulls, G), keys_of(to_host(keys)), csize)
        heads = b"".join(b for _, b in blobs)
        hoff = np.concatenate([[0], np.cumsum([len(b) for _, b in blobs])[:-1]])
        hjobs = np.array([(o, f, len(b)) for o, (f, b) in zip(hoff.tolist(), blobs)], np.int64)
        first = np.concatenate([[0], np.cumsum((pg[:, 4] + PIECE - 1) // PIECE)[:-1]]).astype(np.int64)
        out = torch.empty(size, dtype=torch.uint8, device=dev)
        up = [to_device(x if len(x) else np.zeros(1, np.int64), dev) for x in (first, dst)]
        up += [to_device(np.frombuffer(heads, np.uint8), dev), to_device(hjobs, dev)]
        check(lib.gsx_parquet_assemble(_ptr(scratch), _ptr(pcs_dev), len(pcs), _ptr(sizes), *[_ptr(t) for t in up],
                                       len(hjobs), _ptr(out), st), "gsx_parquet_assemble")
    return Encoded(out, n)


def _source_shape(src):
    """(rows, dtype) of an input encode takes, without touching its data."""
    from .readers import Decoded
    from .records import DeviceRecords
    if isinstance(src, DeviceRecords):
        return len(src), np.dtype([(f, "<f4") for f in src.names])
    if isinstance(src, Decoded) or (isinstance(src, np.ndarray) and src.dtype.names and src.ndim == 1):
        return len(src), src.dtype
    raise ValueError("encode takes DeviceRecords, readers.Decoded or a 1-D structured NumPy array")


def chunk_nulls(nulls: np.ndarray, G: int) -> np.ndarray:
    """[C, G] nulls of each column chunk from those of its pages."""
    if nulls.shape[1] == 0:
        return np.zeros((nulls.shape[0], G), np.int64)
    return np.add.reduceat(nulls, np.arange(0, nulls.shape[1], 4), axis=1)


def keys_of(k) -> np.ndarray:
    """gsx_parquet_split's keys [2, C, G] -> [C, G, 2] int64."""
    k = np.asarray(k).view(np.uint32).astype(np.int64)
    return np.stack([k[0], k[1]], -1)


def write_parquet(path, enc: Encoded) -> None:
    with open(path, "wb") as fh:
        fh.write(enc.to_host())


def prepare_write(self, data, *args, **kwargs):
    """ParquetFormat.write(data, path, **kwargs) for gsx.dropin.install_writer: the file built on the device; returns
    the step that writes it to path and then prints the reference's status line."""
    import sys
    if args:
        raise TypeError("ParquetFormat.write takes no positional arguments after path")
    enc = encode(data)
    blob = enc.to_host()

    def finish(path):
        with open(path, "wb") as fh:
            fh.write(blob)
        status = getattr(sys.modules.get(type(self).__module__), "status_print", print)
        status(f"Parquet write completed. {enc.rows} rows.")
    return finish
