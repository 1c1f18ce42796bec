"""GPU: SOG encode on the device (gsx.sog.encode) against the reference writer's own output (g11) and the NumPy
oracle (sog_oracle.py), under the parity contract of sog_oracle.assert_sog_equal, plus the drop-in write."""
import zipfile
from pathlib import Path

import numpy as np
import pytest

import sog_oracle as so

pytestmark = pytest.mark.gpu

GOLDEN = Path(__file__).resolve().parent / "golden" / "g11_reference_sog_small.npz"


def quantile_fit(values):
    """A deterministic stand-in for the SH codebook fit (no RNG, any number of values)."""
    return np.quantile(values.reshape(-1), np.linspace(0, 1, 256)).astype(np.float32)


def device_encode(a, cuda, level=0, fit=None, seed=None):
    from gsx import records, sog
    r = records.DeviceRecords.from_structured(a, cuda)
    if seed is not None:
        np.random.seed(seed)
    enc = sog.encode(r, level, codebook_fit=fit)
    return enc, enc.to_host()


def check_against_oracle(a, cuda, level=0, fit=quantile_fit, seed=5):
    enc, got = device_encode(a, cuda, level, fit, seed)
    end = np.random.get_state()
    np.random.seed(seed)
    want, want_meta, order = so.encode(a, level, codebook_fit=fit)
    assert so.rng_equal(end, np.random.get_state())
    assert np.array_equal(enc.order.cpu().numpy(), order)
    so.assert_sog_equal(got, enc.meta, want, want_meta)
    return enc, got


@pytest.mark.parametrize("case", ["mixed_l0", "mixed_l7", "deg1", "sh1_80", "planar"])
def test_encode_matches_reference_golden(case, cuda, gsx_lib):
    z = np.load(GOLDEN)
    a, level, seed = so.golden_inputs()[case]
    assert so.digest(a) == str(z[f"{case}_input_sha256"])
    fit = so.replay_fit(z, case) if f"{case}_fit_centres" in z.files else None
    enc, got = device_encode(a, cuda, level, fit, seed)
    assert so.rng_equal(np.random.get_state(), so.rng_unpack(z[f"{case}_rng_end"]))
    want, want_meta = so.golden_case(z, case)
    so.assert_sog_equal(got, enc.meta, want, want_meta)


def test_encode_50k_with_scikit_learn_fit(cuda, gsx_lib):
    from gsx import synth
    enc, got = check_against_oracle(synth.structured(50_000, "mixed"), cuda, fit=None, seed=21)
    assert enc.meta["shN"]["bands"] == 3 and enc.meta["shN"]["count"] == 48 * 683


@pytest.mark.parametrize("n", [1, 80, 1023, 1024, 1025, 16_666, 16_667])
def test_encode_sizes(n, cuda, gsx_lib):
    from gsx import synth
    enc, got = check_against_oracle(synth.structured(n, "mixed"), cuda, seed=n)
    assert enc.meta["count"] == n and enc.meta["shN"]["bands"] == 3
    assert len(enc.meta["scales"]["codebook"]) == (3 * n if 3 * n <= 256 else 256)


def test_encode_band_downgrade_and_gaps(cuda, gsx_lib):
    from gsx import synth
    a = synth.structured(2_500, "mixed")
    for i in range(24, 45):
        a[f"f_rest_{i}"] = 0.0
    a["f_rest_30"][::7] = -0.0                                   # -0.0 counts as zero
    enc, _ = check_against_oracle(a, cuda, level=5)
    assert enc.meta["shN"]["bands"] == 2
    # f_rest_40 missing: 44 fields declare 2 bands; content only up to f_rest_8 -> 1 band, whose fields are all there
    keep = [f for f in a.dtype.names if f != "f_rest_40"]
    b = np.zeros(len(a), dtype=[(f, "f4") for f in keep])
    for f in keep:
        b[f] = a[f]
    for i in range(9, 45):
        if f"f_rest_{i}" in keep:
            b[f"f_rest_{i}"] = 0.0
    enc, _ = check_against_oracle(b, cuda)
    assert enc.meta["shN"]["bands"] == 1


def test_gathered_subset_matches_host_subset(cuda, gsx_lib):
    import torch
    from gsx import records, sog, synth
    a = synth.structured(40_000, "mixed")
    r = records.DeviceRecords.from_structured(a, cuda)
    _, op = r.xyz_opacity()
    keep = torch.nonzero(op > -0.5).flatten().to(torch.int32)
    s = keep.cpu().numpy()
    assert 0 < len(s) < len(a)
    np.random.seed(9)
    enc = sog.encode(r.gather(keep), 3, codebook_fit=quantile_fit)
    np.random.seed(9)
    want, want_meta, _ = so.encode(a[s], 3, codebook_fit=quantile_fit)
    so.assert_sog_equal(enc.to_host(), enc.meta, want, want_meta)


def test_refusals_leave_the_rng_alone(cuda, gsx_lib):
    from gsx import records, sog, synth
    np.random.seed(4)
    state = np.random.get_state()
    a = synth.structured(100, "mixed")
    with pytest.raises(ValueError):
        sog.encode(records.DeviceRecords.from_structured(a[:0], cuda))
    b = np.zeros(100, dtype=[(f, "f4") for f in a.dtype.names if f != "rot_3"])
    with pytest.raises(ValueError):
        sog.encode(records.DeviceRecords.from_structured(b, cuda))
    c = np.zeros(100, dtype=[(f, "f4") for f in a.dtype.names if f != "f_rest_3"])   # 3 bands needs f_rest_3
    c["f_rest_20"] = 1.0
    with pytest.raises(ValueError):
        sog.encode(records.DeviceRecords.from_structured(c, cuda))
    assert so.rng_equal(np.random.get_state(), state)


def test_dropin_write_on_stand_in_class(cuda, gsx_lib, tmp_path):
    from gsx import dropin, sog, synth

    class StandIn:
        def __init__(self):
            self.calls = []

        def write(self, data, path, **kwargs):
            self.calls.append(("original", data, path, kwargs, np.random.get_state()))

    original = StandIn.write
    dropin.install_writer(StandIn, sog.prepare_write, webp="host")
    dropin.install_writer(StandIn, sog.prepare_write, webp="host")       # idempotent
    assert StandIn._gsx_reference_write is original and StandIn.write is not original
    a = synth.structured(3_000, "mixed")
    np.random.seed(8)
    StandIn().write(a, tmp_path / "a.sog", compression_level=7)
    end = np.random.get_state()
    np.random.seed(8)
    want, want_meta, _ = so.encode(a, 7)
    assert so.rng_equal(end, np.random.get_state())
    with zipfile.ZipFile(tmp_path / "a.sog") as zf:
        assert zf.namelist() == list(want) + ["meta.json"]
    # u1 colour fields: not packed float32 records -> the original write, RNG untouched
    b = np.zeros(10, dtype=[("x", "f4"), ("y", "f4"), ("z", "f4"), ("red", "u1"), ("green", "u1"), ("blue", "u1")])
    np.random.seed(2)
    state = np.random.get_state()
    w = StandIn()
    w.write(b, "b.sog", compression_level=3)
    assert len(w.calls) == 1 and w.calls[0][1] is b and w.calls[0][3] == {"compression_level": 3}
    assert so.rng_equal(w.calls[0][4], state)
    # packed float32 without the fields SOG needs: gsx refuses, the original write runs with the RNG as it was
    c = np.zeros(10, dtype=[("x", "f4"), ("y", "f4"), ("z", "f4")])
    w = StandIn()
    w.write(c, "c.sog")
    assert [x[0] for x in w.calls] == ["original"] and so.rng_equal(w.calls[0][4], state)
