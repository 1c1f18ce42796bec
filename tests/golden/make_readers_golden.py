"""Generate tests/golden/g13_reference_readers_small.npz: the reference's own SplatFormat.read, KSplatFormat.read,
SpzFormat.read and CompressedPlyFormat.read (formats/splat.py, ksplat.py, spz.py, compressed_ply.py) on small files.

    python tests/golden/make_readers_golden.py REFERENCE_ROOT     (a checkout of francescofugazzi/3dgsconverter)

The reader modules are loaded by file path as make_splat_codecs_golden.py loads the writers.  compressed_ply.py reads
through plyfile, which is stubbed: its PlyData.read returns the chunk / vertex / sh arrays that this script also
writes into the file with gsx.compressed_ply.write_ply (or with a hand-written header).  Inputs: files of the
reference writers on g12's edge rows, random record bytes at every ksplat level, random SPZ bodies of every version,
hand-assembled multi-section .ksplat files, float16 and int24 edge patterns, compressed PLYs with 0 / 9 / 24 / 45 SH
properties, fewer chunks than splats need and properties out of order, and malformed files.  Each case stores the
file's bytes, the reader's result (length, SHA-256 and dtype of the array's bytes, and the metadata) or the name of
the exception it raises, and `expect`: "ok" where gsx decodes the file, "refuse" where it raises ValueError.  The
script asserts that readers_oracle.py reproduces every case before it writes the fixture.
"""
import gzip
import importlib.util
import struct
import sys
import tempfile
import types
from pathlib import Path

import numpy as np

HERE = Path(__file__).resolve().parent
sys.path[:0] = [str(HERE.parent), str(HERE.parent.parent / "3dgsconverter_b200")]
import readers_oracle as ro  # noqa: E402
import splat_codecs_oracle as sco  # noqa: E402
from make_splat_codecs_golden import import_reference_writers  # noqa: E402

from gsx.compressed_ply import CHUNK_DTYPE, VERTEX_DTYPE, write_ply  # noqa: E402

CLASSES = {"splat": "SplatFormat", "ksplat": "KSplatFormat", "spz": "SpzFormat", "cply": "CompressedPlyFormat"}


def digest(b: bytes) -> str:
    return sco.digest(b)


def meta_repr(m) -> str:
    return repr(m)


# ------------------------------------------------------------------------------------------------------ input files
def ksplat_file(level, sections, version=(0, 1)):
    """A .ksplat of `sections`: dicts with n, maxn, bs, fb, partial (lengths), nb, block, srange, deg and optional
    `records` / `centres` bytes (random when absent)."""
    rng = np.random.default_rng(len(sections) * 7 + level)
    head = bytearray(4096)
    head[0], head[1] = version
    struct.pack_into("<IIII", head, 4, len(sections), len(sections), sum(s["maxn"] for s in sections),
                     sum(s["n"] for s in sections))
    struct.pack_into("<H", head, 20, level)
    struct.pack_into("<ff", head, 36, -2.0, 2.0)
    secs, body = b"", b""
    lv = min(level, 2)
    for s in sections:
        sh_count = {1: 9, 2: 24}.get(s["deg"], 0)
        per = 44 + 4 * sh_count if lv == 0 else 24 + (2 if lv == 1 else 1) * sh_count
        h = bytearray(1024)
        struct.pack_into("<IIIIfH", h, 0, s["n"], s["maxn"], s["bs"], s["nb"], s["block"], 12)
        struct.pack_into("<IIIIH", h, 24, s["srange"], 0, s["fb"], len(s["partial"]), s["deg"])
        secs += bytes(h)
        body += np.asarray(s["partial"], "<u4").tobytes()
        body += s.get("centres", rng.uniform(-50, 50, 3 * s["nb"]).astype("<f4").tobytes())
        body += s.get("records", rng.integers(0, 256, s["maxn"] * per, dtype=np.uint8).tobytes())
    return bytes(head) + secs + body


def sec(n, level_bs=7, deg=0, maxn=None, partial=None, nb=None, srange=0, block=5.0, fb=None):
    fb = n // level_bs if fb is None else fb
    partial = ([n % level_bs] if n % level_bs else []) if partial is None else partial
    nb = fb + len(partial) if nb is None else nb
    return dict(n=n, maxn=n if maxn is None else maxn, bs=level_bs, fb=fb, partial=partial, nb=nb, block=block,
                srange=srange, deg=deg)


def spz_body(version, n, deg, frac=12, seed=0, patterns=None):
    rng = np.random.default_rng(seed)
    dim = {0: 0, 1: 3, 2: 8, 3: 15}.get(deg, 0)
    size = n * ((6 if version == 1 else 9) + 7 + (4 if version >= 3 else 3) + 3 * dim)
    body = bytearray(rng.integers(0, 256, size, dtype=np.uint8).tobytes())
    if patterns is not None:
        body[:len(patterns)] = patterns
    return struct.pack("<IIIBBBB", 0x5053474E, version, n, deg, frac, 0, 0) + bytes(body)


def cply_arrays(n, nchunk, nsh, seed):
    rng = np.random.default_rng(seed)
    chunk = np.zeros(nchunk, CHUNK_DTYPE)
    for f in CHUNK_DTYPE.names:
        chunk[f] = rng.uniform(-5, 5, nchunk).astype(np.float32) + (10.0 if f.startswith("max") else 0.0)
    if nchunk > 1:   # degenerate and non-finite bounds
        chunk["min_x"][0], chunk["max_x"][0] = 1.0, 1.0
        chunk["min_y"][1], chunk["max_y"][1] = -np.inf, np.inf
        chunk["min_r"][1] = chunk["max_r"][1] = np.float32(np.nan)
    vertex = rng.integers(0, 1 << 32, (n, 4), dtype=np.uint64).astype(np.uint32).view(VERTEX_DTYPE).reshape(-1)
    sh = None
    if nsh:
        sh = rng.integers(0, 256, (n, nsh), dtype=np.uint8).view(np.dtype([(f"f_rest_{i}", "u1") for i in range(nsh)]))
        sh = sh.reshape(-1)
    return chunk, vertex, sh


def ply_bytes(path, chunk, vertex, sh, header_types=None, order=None):
    """write_ply's file, or one with a hand-written header: property type names from header_types, vertex properties
    in `order`."""
    if header_types is None and order is None:
        write_ply(path, chunk, vertex, sh)
        return Path(path).read_bytes()
    t = header_types or {"f4": "float", "u4": "uint", "u1": "uchar"}
    if order is not None:
        moved = np.zeros(len(vertex), [(f, "<u4") for f in order])
        for f in order:
            moved[f] = vertex[f]
        vertex = moved
    els = [("chunk", chunk), ("vertex", vertex)] + ([("sh", sh)] if sh is not None else [])
    lines = ["ply", "format binary_little_endian 1.0", "comment gsx"]
    for name, a in els:
        lines.append(f"element {name} {len(a)}")
        for f in a.dtype.names:
            lines.append(f"property {t[a.dtype.fields[f][0].str[1:]]} {f}")
    lines.append("end_header")
    body = b"".join(np.ascontiguousarray(a).tobytes() for _, a in els)
    return ("\n".join(lines) + "\n").encode() + body


def cases(ref, tmp):
    """{name: (format, file bytes, plyfile stub arrays or None, expect)}"""
    out = {}
    inputs = sco.golden_inputs()
    edge = inputs["mixed3"][np.r_[0:30, 40:75, 80:92, 100:105, 120:150]]
    f = Path(tmp) / "w"
    for tag, a in (("edge", edge), ("n0", inputs["n0"]), ("n1", inputs["n1"]), ("n257", inputs["n257"][:257])):
        ref["SplatFormat"]().write(a, f)
        out[f"splat_writer_{tag}"] = ("splat", f.read_bytes(), None, "ok")
        ref["SpzFormat"]().write(a, f, compression_level=1)
        out[f"spz_writer_{tag}"] = ("spz", f.read_bytes(), None, "ok")
        for lv, shl, bs in ((0, None, 256), (1, None, 7), (2, 1, 256), (3, None, 100)):
            if (tag != "edge" and lv in (0, 3)) or tag == "n257":
                continue
            ref["KSplatFormat"]().write(a, f, lv, sh_level=shl, bucket_size=bs)
            out[f"ksplat_writer_{tag}_l{lv}"] = ("ksplat", f.read_bytes(), None, "ok")
    rng = np.random.default_rng(13)
    rec = rng.integers(0, 256, 100 * 32, dtype=np.uint8)
    rec.view("<f4")[3::8][:40] = np.array([np.nan, -np.nan, np.inf, -np.inf, 0.0, -0.0, 1e-7, 1e-6, 1.0000001e-6,
                                           3e38] * 4, np.float32)
    out["splat_random"] = ("splat", rec.tobytes() + b"\x01\x02\x03", None, "ok")
    out["splat_empty"] = ("splat", b"", None, "ok")
    for lv in (0, 1, 2, 3):
        out[f"ksplat_random_l{lv}"] = ("ksplat", ksplat_file(lv, [sec(60, 7, deg=2)]), None, "ok")
    mix = ksplat_file(1, [sec(40, 32, deg=1, maxn=50), sec(37, 10, deg=2, partial=[3, 0, 4], fb=3),
                          sec(0, 7, deg=3, nb=1, partial=[]), sec(20, 8, deg=0, srange=0, block=np.float32(np.nan),
                                                                 partial=[20], fb=0)])
    out["ksplat_multisection"] = ("ksplat", mix, None, "ok")
    out["ksplat_multisection_l0"] = ("ksplat", ksplat_file(0, [sec(40, 7, deg=2), sec(9, 7, deg=3, maxn=12)]), None,
                                     "ok")
    out["ksplat_srange"] = ("ksplat", ksplat_file(2, [sec(50, 16, deg=1, srange=1000, block=3.0)]), None, "ok")
    out["ksplat_nosections"] = ("ksplat", ksplat_file(1, []), None, "ok")
    out["ksplat_version"] = ("ksplat", ksplat_file(0, [sec(5, 7)], version=(0, 2)), None, "refuse")
    out["ksplat_truncated"] = ("ksplat", ksplat_file(1, [sec(30, 7, deg=1)])[:-5], None, "refuse")
    out["ksplat_short_lengths"] = ("ksplat", ksplat_file(1, [sec(30, 7, partial=[1])]), None, "refuse")
    out["ksplat_bucket_past_centres"] = ("ksplat", ksplat_file(1, [sec(30, 7, nb=3)]), None, "refuse")
    out["ksplat_no_centres"] = ("ksplat", ksplat_file(1, [sec(0, 7, nb=0, partial=[], fb=0)]), None, "refuse")
    out["ksplat_short_header"] = ("ksplat", b"\x00\x01" + bytes(100), None, "refuse")
    # float16 patterns through level-1 scales and SH
    f16 = np.arange(65536, dtype=np.uint16)[::251]
    recs = np.zeros((len(f16), 42), np.uint8)
    for k in range(3):
        recs[:, 6 + 2 * k:8 + 2 * k] = np.roll(f16, k).view(np.uint8).reshape(-1, 2)
    for k in range(9):
        recs[:, 24 + 2 * k:26 + 2 * k] = np.roll(f16, 3 + k).view(np.uint8).reshape(-1, 2)
    s = sec(len(f16), 1 << 20, deg=1, fb=0, partial=[len(f16)])
    s["records"] = recs.tobytes()
    out["ksplat_float16"] = ("ksplat", ksplat_file(1, [s]), None, "ok")
    for v in (1, 2, 3):
        for deg in (0, 1, 2, 3):
            out[f"spz_random_v{v}_d{deg}"] = ("spz", spz_body(v, 30 + deg, deg, seed=10 * v + deg), None, "ok")
    out["spz_degree4"] = ("spz", spz_body(3, 3, 4, seed=7), None, "ok")
    out["spz_gzip_v2"] = ("spz", gzip.compress(spz_body(2, 100, 1, frac=20, seed=8), mtime=0), None, "ok")
    i24 = np.array([0x000000, 0x7fffff, 0x800000, 0xffffff, 0x800001, 0x000001, 0x400000, 0xc00000, 0x123456],
                   np.uint32)
    pat = np.stack([i24 & 0xff, i24 >> 8 & 0xff, i24 >> 16 & 0xff], 1).astype(np.uint8).tobytes()
    out["spz_int24"] = ("spz", spz_body(3, 30, 0, frac=0, seed=9, patterns=pat * 3), None, "ok")
    out["spz_int24_frac127"] = ("spz", spz_body(2, 30, 0, frac=127, seed=9, patterns=pat * 3), None, "ok")
    pat16 = np.array([0x7c00, 0xfc00, 0x7c01, 0x7e00, 0xfe01, 0x0001, 0x8001, 0x03ff, 0x7bff], np.uint16).tobytes()
    out["spz_v1_float16"] = ("spz", spz_body(1, 40, 1, seed=11, patterns=pat16 * 6), None, "ok")
    out["spz_bad_magic"] = ("spz", b"\x00" * 16, None, "refuse")
    out["spz_version4"] = ("spz", struct.pack("<IIIBBBB", 0x5053474E, 4, 0, 0, 12, 0, 0), None, "refuse")
    out["spz_truncated"] = ("spz", spz_body(3, 20, 1)[:-1], None, "refuse")
    out["spz_frac128"] = ("spz", spz_body(3, 5, 0, frac=128), None, "refuse")
    # compressed PLY
    p = Path(tmp) / "c.ply"
    for tag, n, nchunk, nsh in (("n0", 0, 0, 0), ("n1", 1, 1, 9), ("n257", 257, 2, 24), ("sh45", 260, 2, 45),
                                ("fewer_chunks", 300, 1, 0), ("more_chunks", 100, 3, 9)):
        arrays = cply_arrays(n, nchunk, nsh, seed=n + nsh)
        out[f"cply_{tag}"] = ("cply", ply_bytes(p, *arrays), arrays, "ok")
    arrays = cply_arrays(260, 2, 9, seed=5)
    out["cply_aliases"] = ("cply", ply_bytes(p, *arrays, header_types={"f4": "float32", "u4": "uint32", "u1": "uint8"}),
                           arrays, "ok")
    order = ("packed_color", "packed_scale", "packed_position", "packed_rotation")
    out["cply_order"] = ("cply", ply_bytes(p, *arrays, order=order), arrays, "ok")
    c, v, s = arrays
    out["cply_sh_short"] = ("cply", ply_bytes(p, c, v, s[:200]), (c, v, s[:200]), "refuse")
    good = out["cply_n1"][1]
    out["cply_ascii"] = ("cply", good.replace(b"binary_little_endian", b"ascii", 1), None, "refuse")
    out["cply_big_endian"] = ("cply", good.replace(b"binary_little_endian", b"binary_big_endian", 1), None, "refuse")
    out["cply_no_chunk"] = ("cply", good.replace(b"element chunk", b"element chonk", 1), None, "refuse")
    out["cply_truncated"] = ("cply", good[:-3], None, "refuse")
    dup = out["cply_n1"][1].replace(b"property uchar f_rest_1\n", b"property uchar f_rest_0\n", 1)
    out["cply_duplicate"] = ("cply", dup, None, "refuse")
    return out


def plyfile_stub(arrays):
    c, v, s = arrays
    els = {"chunk": c, "vertex": v, **({"sh": s} if s is not None else {})}

    class PlyData:
        @staticmethod
        def read(path):
            return PlyData()

        def __contains__(self, k):
            return k in els

        def __getitem__(self, k):
            return types.SimpleNamespace(data=els[k])

    m = types.ModuleType("plyfile")
    m.PlyData = PlyData
    return m


def main(ref_root):
    ref = import_reference_writers(ref_root)
    ref_dir = Path(ref_root) / "gsconverter" / "formats"
    spec = importlib.util.spec_from_file_location("gsconverter.formats.compressed_ply", ref_dir / "compressed_ply.py")
    m = importlib.util.module_from_spec(spec)
    sys.modules[spec.name] = m
    spec.loader.exec_module(m)
    ref["CompressedPlyFormat"] = m.CompressedPlyFormat
    out = {}
    with tempfile.TemporaryDirectory() as tmp:
        path = Path(tmp) / "in"
        for name, (fmt, blob, arrays, expect) in cases(ref, tmp).items():
            path.write_bytes(blob)
            out[f"{name}_file"] = np.frombuffer(blob, np.uint8)
            out[f"{name}_format"] = np.array(fmt)
            out[f"{name}_expect"] = np.array(expect)
            reader = ref[CLASSES[fmt]]()
            if fmt == "cply" and arrays is None:
                print(name, "refused by the device, reference not run")
                continue
            if arrays is not None:
                sys.modules["plyfile"] = plyfile_stub(arrays)
            try:
                with np.errstate(all="ignore"):
                    got = reader.read(str(path))
            except Exception as e:  # noqa: BLE001
                out[f"{name}_raises"] = np.array(type(e).__name__)
                out[f"{name}_expect"] = np.array("refuse")   # where the reference raises, gsx refuses
                print(name, "raises", type(e).__name__)
                continue
            finally:
                sys.modules.pop("plyfile", None)
            meta = getattr(reader, "metadata", None) if fmt in ("ksplat", "cply") else None
            b = np.ascontiguousarray(got).tobytes()
            out[f"{name}_len"] = np.array(len(b))
            out[f"{name}_sha256"] = np.array(digest(b))
            out[f"{name}_dtype"] = np.array(str(got.dtype.descr))
            out[f"{name}_meta"] = np.array(meta_repr(meta))
            try:
                with np.errstate(all="ignore"):
                    want, wmeta = ro.READERS[fmt](blob)
            except ValueError:
                assert expect == "refuse", f"{name}: the oracle refuses a file gsx decodes"
            else:
                assert expect == "ok", f"{name}: the oracle decodes a file gsx refuses"
                assert digest(np.ascontiguousarray(want).tobytes()) == digest(b), f"{name}: the oracle differs"
                assert str(want.dtype.descr) == str(got.dtype.descr) and meta_repr(wmeta) == meta_repr(meta), name
            print(name, expect, len(b))
    np.savez_compressed(HERE / "g13_reference_readers_small.npz", **out)


if __name__ == "__main__":
    main(sys.argv[1])
