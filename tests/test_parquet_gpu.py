"""GPU: gsx.parquet's device writer byte for byte against tests/parquet_oracle.py, on the fixture's inputs and on
large clouds (random SH-3 records and records decoded on the device from gsx's own .spz: dictionary columns), whose
tables are also checked against a pyarrow write of the same frame; the Snappy kernel on pieces of runs, without
runs, and with a run across a 64 KiB piece boundary; the drop-in."""
import io
import json
from pathlib import Path

import numpy as np
import pytest

pd = pytest.importorskip("pandas")
pq = pytest.importorskip("pyarrow.parquet")

pytestmark = pytest.mark.gpu
GOLDEN = Path(__file__).resolve().parent / "golden" / "g16_reference_parquet_small.npz"


def frame(a):
    """The frame ParquetFormat.write hands to to_parquet, built with the oracle's column plan."""
    from gsx import parquet as gp
    plan = gp.column_plan(a.dtype)
    return pd.DataFrame({c.name: a[c.source] for c in plan})


def test_fixture_cases(gsx_lib, cuda):
    import parquet_oracle as po
    from gsx import parquet as gp
    z = np.load(GOLDEN)
    names = sorted({k.split("/")[0] for k in z.files})
    for name in names:
        a = po.golden_inputs()[name]
        assert json.loads(z[f"{name}/dtype"].tobytes()) == json.loads(json.dumps(a.dtype.descr))
        try:
            want = po.encode(a)
        except ValueError:
            with pytest.raises(ValueError):
                gp.encode(a, device=cuda)
            continue
        got = gp.encode(a, device=cuda).to_host()
        assert got == want, name


def _spz_decoded(a, cuda):
    from gsx import spz
    from gsx.records import DeviceRecords
    payload = spz.encode(DeviceRecords.from_structured(a, cuda)).to_host()
    return spz.decode(payload, device=cuda)


@pytest.mark.parametrize("n", [(1 << 20) + 1, 10_000_000])
@pytest.mark.parametrize("kind", ["random", "spz"])
def test_large_clouds(gsx_lib, cuda, kind, n):
    import parquet_oracle as po
    from gsx import parquet as gp, synth
    a = synth.structured(n, "mixed", 3)
    if kind == "spz":
        dec = _spz_decoded(a, cuda)
        enc = gp.encode(dec)
        a = dec.to_host()
    else:
        enc = gp.encode(a, device=cuda)
    got = enc.to_host()
    print(f"\n{kind} {n}: device file {len(got)} bytes", flush=True)
    assert got == po.encode(a)
    print(f"{kind} {n}: oracle equal", flush=True)
    buf = io.BytesIO()
    frame(a).to_parquet(buf)
    ref = buf.getvalue()
    tm, tr = pq.read_table(io.BytesIO(got)), pq.read_table(io.BytesIO(ref))
    assert tm.schema.remove_metadata().equals(tr.schema.remove_metadata())
    assert tm.replace_schema_metadata(None).equals(tr.replace_schema_metadata(None))
    fm, fr = po.chunk_facts(pq.read_metadata(io.BytesIO(got))), po.chunk_facts(pq.read_metadata(io.BytesIO(ref)))
    assert fm == fr
    assert fm[-1][0] == n % gp.ROW_GROUP
    print(f"{kind} {n}: {len(got)} bytes, pyarrow {len(ref)} ({len(got) / len(ref):.4f})", flush=True)
    if kind == "random":   # the .spz-decoded cloud comes out about 0.6 % larger than pyarrow's file (DESIGN 10)
        assert len(got) <= len(ref), (len(got), len(ref))


def _device_snappy(body: bytes, cuda):
    """gsx_parquet_snappy on one page body -> each piece's elements."""
    import torch
    from gsx import parquet as gp
    from gsx._abi import lib, check, _ptr, _stream
    from gsx.hostcopy import to_device, to_host
    b = np.frombuffer(body, np.uint8)
    pad = np.zeros((len(b) + 15) // 16 * 16, np.uint8)
    pad[:len(b)] = b
    starts = np.arange(0, len(b), gp.PIECE)
    pcs = np.stack([np.zeros_like(starts), starts, np.minimum(gp.PIECE, len(b) - starts)], 1).astype(np.int64)
    cap = lib.gsx_parquet_piece_bytes()
    scratch = torch.empty(len(pcs) * cap, dtype=torch.uint8, device=cuda)
    sizes = torch.zeros(len(pcs), dtype=torch.int32, device=cuda)
    page = torch.zeros(1, dtype=torch.int32, device=cuda)
    body_dev, pcs_dev = to_device(pad, cuda), to_device(pcs, cuda)     # both referenced until the kernel has run
    check(lib.gsx_parquet_snappy(_ptr(body_dev), _ptr(pcs_dev), len(pcs), _ptr(scratch), _ptr(sizes), _ptr(page),
                                 _stream()), "gsx_parquet_snappy")
    s, sc = to_host(sizes), to_host(scratch)
    assert int(to_host(page)[0]) == int(s.sum())
    return [sc[i * cap:i * cap + s[i]].tobytes() for i in range(len(pcs))]


def test_snappy_pieces(gsx_lib, cuda):
    import parquet_oracle as po
    from gsx import parquet as gp
    rng = np.random.default_rng(5)
    runs = np.repeat(rng.integers(0, 256, 2000).astype(np.uint8), rng.integers(8, 90, 2000))[:gp.PIECE]
    none = rng.integers(0, 256, gp.PIECE).astype(np.uint8)
    none[1:][none[1:] == none[:-1]] ^= 1
    cross = rng.integers(0, 256, 3 * gp.PIECE - 5).astype(np.uint8)
    cross[gp.PIECE - 20:gp.PIECE + 40] = 9                               # a run across the first piece boundary
    cross[2 * gp.PIECE - 12:2 * gp.PIECE + 12] = np.tile(np.array([1, 2, 3, 4], np.uint8), 6)   # and a 4-byte repeat
    words = np.tile(rng.integers(0, 1 << 32, 3, dtype=np.uint64).astype(np.uint32), 30000).view(np.uint8)
    for body in (runs, none, cross, words, none[:1], runs[:9]):
        want = [po.snappy_piece(body[s:s + gp.PIECE]) for s in range(0, len(body), gp.PIECE)]
        assert _device_snappy(body.tobytes(), cuda) == want
    assert len(po.snappy_piece(none)) == gp.PIECE + 3
    assert len(po.snappy_piece(runs)) < gp.PIECE // 8


def test_one_entry_dictionary_reads_back(gsx_lib, cuda):
    from gsx import parquet as gp
    a = np.zeros(300_000, [("x", "<f4"), ("opacity", "<f4")])
    a["x"] = 2.5
    a["opacity"][::3] = np.nan
    blob = gp.encode(a, device=cuda).to_host()
    meta = pq.read_metadata(io.BytesIO(blob))
    assert "RLE_DICTIONARY" in meta.row_group(0).column(0).encodings
    t = pq.read_table(io.BytesIO(blob))
    assert np.array_equal(t.column("x").to_numpy(), a["x"])
    assert t.column("alpha").null_count == 100_000


def test_dropin_on_a_stand_in_class(gsx_lib, cuda, tmp_path, capsys):
    from gsx import dropin, parquet as gp
    calls = []

    class ParquetFormat:
        def write(self, data, path, **kwargs):
            calls.append((len(data), path, kwargs))

    original = ParquetFormat.write
    dropin.install_writer(ParquetFormat, gp.prepare_write)
    dropin.install_writer(ParquetFormat, gp.prepare_write)
    assert ParquetFormat._gsx_reference_write is original and ParquetFormat.write is not original
    ok = np.zeros(5, [("x", "<f4"), ("opacity", "<f4")])
    ParquetFormat().write(ok, str(tmp_path / "a.parquet"))
    assert not calls and "Parquet write completed. 5 rows." in capsys.readouterr().out
    assert pq.read_table(tmp_path / "a.parquet").column_names == ["x", "alpha"]
    for bad in (np.zeros(3, [("x", "<f4"), ("d", "<f8")]), np.zeros(3, [("opacity", "<f4"), ("alpha", "<f4")])):
        ParquetFormat().write(bad, str(tmp_path / "b.parquet"), flag=1)
        assert calls[-1] == (3, str(tmp_path / "b.parquet"), {"flag": 1})
