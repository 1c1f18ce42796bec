"""CPU: gsx's Parquet writer as restated by tests/parquet_oracle.py against the reference's own files
(tests/golden/g16_reference_parquet_small.npz, made by make_parquet_golden.py): the same table, frame, row groups and
column-chunk statistics; the refusals; the column plan and the Thrift compact encoder on their own."""
import io
import json
from pathlib import Path

import numpy as np
import pytest

pd = pytest.importorskip("pandas")
pq = pytest.importorskip("pyarrow.parquet")

GOLDEN = Path(__file__).resolve().parent / "golden" / "g16_reference_parquet_small.npz"


@pytest.fixture(scope="module")
def golden(gsx_lib):
    z = np.load(GOLDEN)
    return {k: z[k] for k in z.files}


def cases(g):
    return sorted({k.split("/")[0] for k in g})


def case_input(g, name):
    import parquet_oracle as po
    dt = np.dtype([tuple(f) for f in json.loads(g[f"{name}/dtype"].tobytes())])
    if f"{name}/input" in g:
        return g[f"{name}/input"].view(dt)
    a = po.golden_inputs()[name]
    assert a.dtype == dt
    return a


def test_fixture_inputs_are_the_generators(golden):
    import parquet_oracle as po
    ins = po.golden_inputs()
    assert set(cases(golden)) == set(ins)
    for name in cases(golden):
        if f"{name}/input" in golden:
            assert golden[f"{name}/input"].tobytes() == np.ascontiguousarray(ins[name]).view(np.uint8).tobytes(), name


def test_oracle_file_holds_the_reference_table(golden):
    import parquet_oracle as po
    seen = 0
    for name in cases(golden):
        if f"{name}/error" in golden or name == po.LARGE:
            continue
        a = case_input(golden, name)
        try:
            mine = po.encode(a)
        except ValueError:
            assert name in ("float64_extra", "int16_extra"), name
            continue
        ref = golden[f"{name}/file"].tobytes()
        tm, tr = pq.read_table(io.BytesIO(mine)), pq.read_table(io.BytesIO(ref))
        assert tm.schema.remove_metadata().equals(tr.schema.remove_metadata()), name
        assert tm.replace_schema_metadata(None).equals(tr.replace_schema_metadata(None)), name
        pd.testing.assert_frame_equal(pd.read_parquet(io.BytesIO(mine)), pd.read_parquet(io.BytesIO(ref)),
                                      check_exact=True)
        assert po.chunk_facts(pq.read_metadata(io.BytesIO(mine))) == po.chunk_facts(pq.read_metadata(io.BytesIO(ref)))
        if len(a) >= 1000:
            assert len(mine) <= len(ref), (name, len(mine), len(ref))
        seen += 1
    assert seen >= 11


def test_large_case_matches_the_reference_facts(golden):
    import parquet_oracle as po
    facts = json.loads(golden[f"{po.LARGE}/facts"].tobytes())
    mine = po.encode(po.golden_inputs()[po.LARGE])
    assert po.table_digest(pq.read_table(io.BytesIO(mine))) == facts["digest"]
    got = json.loads(json.dumps(po.chunk_facts(pq.read_metadata(io.BytesIO(mine)))))
    assert got == facts["chunks"]
    assert len(mine) <= facts["size"]


def test_dictionary_limit_is_262144_distinct_values(gsx_lib):
    import parquet_oracle as po
    from gsx import parquet as gp
    a = po.golden_inputs()[po.LARGE]
    _, nulls, distinct, _, _ = po.kernel_outputs(a, gp.column_plan(a.dtype))
    assert distinct[0, 0] == gp.DICT_MAX and distinct[1, 0] == gp.DICT_MAX + 1
    assert distinct[2, 0] == 1       # cov_s0, a constant column: a one-entry dictionary


def test_refusals(golden):
    from gsx import parquet as gp
    for name in ("float64_extra", "int16_extra", "alpha_collision"):
        with pytest.raises(ValueError):
            gp.column_plan(case_input(golden, name).dtype)
    assert golden["alpha_collision/error"].tobytes() == b"ValueError"
    with pytest.raises(ValueError):
        gp.column_plan(np.dtype([("x", ">f4")]))
    with pytest.raises(ValueError):
        gp.column_plan(np.dtype([("x", "<f4", (3,))]))


def test_column_plan_restates_the_reference_order(gsx_lib):
    from gsx import parquet as gp
    dt = np.dtype([("red", "u1"), ("f_rest_3", "<f4"), ("opacity", "<f4"), ("rot_0", "<f4"), ("x", "<f4"),
                   ("f_rest_16", "<f4"), ("ny", "<f4"), ("f_dc_2", "<f4"), ("scale_1", "<f4"), ("extra", "<f4"),
                   ("rot_2", "<f4")])
    plan = gp.column_plan(dt)
    # ny without nx is dropped, as the reference's order lists the normals only when nx is a field
    assert [c.name for c in plan] == ["x", "cov_q1", "cov_q3", "cov_s1", "alpha", "r_sh4", "g_sh2", "b_sh0", "red",
                                      "extra"]
    assert [c.source for c in plan][:3] == ["x", "rot_2", "rot_0"]
    assert plan[8].kind == gp.U1 and plan[8].offset == 0 and plan[0].offset == dt.fields["x"][1]
    deg1 = np.dtype([(f"f_rest_{i}", "<f4") for i in range(9)])
    assert [c.name for c in gp.column_plan(deg1)] == [f"r_sh{i}" for i in range(1, 10)]


def test_thrift_compact_encoding(gsx_lib):
    from gsx.parquet import Thrift as T
    assert T.varint(0) == b"\x00" and T.varint(300) == b"\xac\x02"
    assert T.zigzag(-1) == b"\x01" and T.zigzag(1) == b"\x02"
    # field 1 i32 = 3, field 3 binary "ab", field 20 bool true (long form), stop
    assert T.struct([(1, T.I32, 3), (3, T.BINARY, "ab"), (20, T.BOOL, True)]) == b"\x15\x06\x28\x02ab\x01\x28\x00"
    # a list of 16 i32 uses the long list header
    assert T.struct([(1, (T.LIST, T.I32), [0] * 16)])[:3] == b"\x19\xf5\x10"
    assert T.struct([(2, T.STRUCT, [])]) == b"\x2c\x00\x00"


def test_snappy_elements(gsx_lib):
    import parquet_oracle as po
    run = np.full(200, 7, np.uint8)
    assert po.snappy_piece(run) == bytes([0, 7]) + bytes([(63 << 2) | 2, 1, 0]) * 3 + bytes([((7 - 4) << 2) | 1, 1])
    rnd = np.random.default_rng(0).integers(0, 256, 100).astype(np.uint8)
    assert po.snappy_piece(rnd) == bytes([60 << 2, 99]) + rnd.tobytes()
    rep = np.tile(np.array([1, 2, 3, 4], np.uint8), 5)
    assert po.snappy_piece(rep) == bytes([3 << 2, 1, 2, 3, 4]) + bytes([((16 - 1) << 2) | 2, 4, 0])
