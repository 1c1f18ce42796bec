"""The compressed PLY packing kernel (k_cply_pack) and the SOG kernels, path by path, with NaN and +-inf inputs.

Each case has a seeded builder.  An unmarked CPU test checks in NumPy the property of the data the case relies on
(the oracle's chunk row is NaN, the largest quaternion component is a NaN, the SH store has a byte tail, a label
wraps past 65 535, ...).  A `gpu` test asserts exact equality with compressed_ply_oracle.encode, np.lexsort,
sog_oracle.encode under assert_sog_equal, or a NumPy restatement of the SOG texture layout."""
import ctypes as C

import numpy as np
import pytest

import compressed_ply_oracle as cpo
import sog_oracle as so

NEG_NAN = np.uint32(0xFFC00000).view(np.float32)          # what inf - inf gives on x86
NAN_PAYLOAD = np.uint32(0x7FC00123).view(np.float32)
NEG_NAN_PAYLOAD = np.uint32(0xFFD00001).view(np.float32)
NONFINITE = {"nan": np.float32(np.nan), "neg_nan": NEG_NAN, "inf": np.float32(np.inf), "neg_inf": np.float32(-np.inf)}

# ------------------------------------------------------------------------------------------------ compressed PLY
CPLY_FIELDS = ["x", "y", "z", "scale_0", "scale_1", "scale_2", "f_dc_0", "f_dc_1", "f_dc_2", "opacity",
               "rot_0", "rot_1", "rot_2", "rot_3", "f_rest_0", "f_rest_44"]
CPLY_N = 2048          # 8 chunks, n % 4 == 0: no NaN falls into the scalar tail of NumPy's cast loop


def cply_nonfinite_case(field):
    """8 chunks; NaN at chunk 0, -NaN at the last row of chunk 2, +inf at the first row of chunk 4, -inf in chunk 6."""
    from gsx import synth
    a = synth.structured(CPLY_N, "mixed")
    for (name, v), row in zip(NONFINITE.items(), (5, 3 * 256 - 1, 4 * 256, 6 * 256 + 100)):
        a[field][row] = v
    return a


QUAT_CASES = {"nan_first": (np.nan, 1, 0, 0), "nan_second": (1, np.nan, 0, 0), "inf_first": (np.inf, 1, 0, 0),
              "inf_second": (1, np.inf, 0, 0), "neg_inf_third": (0.5, 0.5, -np.inf, 0.1)}


def cply_quat_case():
    from gsx import synth
    a = synth.structured(1024, "mixed")
    for k, q in enumerate(QUAT_CASES.values()):
        for i in range(4):
            a[f"rot_{i}"][300 + 11 * k] = q[i]
    return a


def numpy_nan_cast():
    """np.float32 NaN -> uint32 on this NumPy: 0x80000000 in the vector loop, 0 in the scalar remainder"""
    with np.errstate(invalid="ignore"):
        return np.full(8, np.nan, np.float32).astype(np.uint32), np.full(3, np.nan, np.float32).astype(np.uint32)


def test_numpy_nan_to_uint32_cast_is_pinned():
    vec, tail = numpy_nan_cast()
    assert (vec == 0x80000000).all() and (tail == 0).all()


@pytest.mark.parametrize("field", CPLY_FIELDS)
def test_cply_nonfinite_case_reaches_its_path(field):
    a = cply_nonfinite_case(field)
    with np.errstate(all="ignore"):
        chunk, vertex, sh = cpo.encode(a, np.arange(len(a)))
    bad = np.flatnonzero(~np.isfinite(a[field]))
    assert len(bad) == 4 and (bad < len(a) - len(a) % 4).all() and len({b // 256 for b in bad}) == 4
    if field in ("x", "y", "z"):
        assert np.isnan(chunk[f"min_{field}"][0]) and np.isnan(chunk[f"max_{field}"][2])
        if field == "z":          # a NaN z bound sets bit 31 of every position word of the chunk
            assert (vertex["packed_position"][:256] >> 31 == 1).all()
    if field == "opacity":
        assert vertex["packed_color"][5] >> 31 == 1
    if field.startswith("scale_"):
        ax = "xyz"[int(field[-1])]
        assert np.isnan(chunk[f"min_scale_{ax}"][0])            # np.clip keeps the NaN
    if field.startswith("rot_"):
        assert vertex["packed_rotation"][5] == 0x80000000


def test_cply_quat_case_reaches_its_path():
    a = cply_quat_case()
    q = np.stack([a[f"rot_{i}"] for i in range(4)], axis=1)[300::11][:len(QUAT_CASES)]
    with np.errstate(all="ignore"):
        d = np.sqrt((q * q).sum(axis=1, keepdims=True)) + np.float32(1e-10)
        largest = np.argmax(np.abs(q / d), axis=1)
    assert list(largest) == [0, 0, 0, 1, 2]                     # the first NaN wins np.argmax
    assert np.isnan((q / d)[3, 1]) and not np.isnan((q / d)[3, 0])   # (1, inf): only the second is NaN


REST_CASES = [(0, 256 + 12), (9, 512 + 12), (24, 256 + 5), (45, 768 + 12), (45, 3)]


def cply_rest_case(n_rest, n):
    from gsx import synth
    a = synth.structured(n, "mixed", sh_degree={0: 0, 9: 1, 24: 2, 45: 3}[n_rest])
    for k in range(n_rest):
        a[f"f_rest_{k}"][k % n] = (5.0, -5.0, 3.99, -4.01, np.inf, -np.inf)[k % 6]
    return a


@pytest.mark.parametrize("n_rest,n", REST_CASES)
def test_cply_rest_case_reaches_its_path(n_rest, n):
    a = cply_rest_case(n_rest, n)
    rows_here = n - (n - 1) // 256 * 256
    assert rows_here < 16
    names = [f for f in a.dtype.names if f.startswith("f_rest_")]
    assert len(names) == n_rest
    bytes_last = rows_here * n_rest                                # the last chunk's SH bytes
    if n_rest:
        assert bytes_last >> 4 > 0 and bytes_last & 15 > 0       # 16-byte stores and a byte tail


def _cply_device(a, cuda, order):
    import torch
    from gsx import compressed_ply, records
    r = records.DeviceRecords.from_structured(a, cuda)
    enc = compressed_ply.encode(r, None if order is None else torch.from_numpy(np.asarray(order, np.int32)).to(cuda))
    return enc, enc.to_host()


def _cply_check(a, cuda, order):
    enc, got = _cply_device(a, cuda, order)
    o = enc.order.cpu().numpy()
    with np.errstate(all="ignore"):
        want = cpo.encode(a, o)
    cpo.assert_packed_equal(got, want)
    assert list(enc.sh_names) == (list(want[2].dtype.names) if want[2] is not None else [])
    return o


@pytest.mark.gpu
@pytest.mark.parametrize("field", CPLY_FIELDS)
def test_cply_pack_nonfinite_fields(field, cuda, gsx_lib):
    """Each field group with NaN of both signs and +-inf, in a permuted order, against the oracle bit for bit."""
    a = cply_nonfinite_case(field)
    order = np.random.default_rng(len(field)).permutation(len(a))
    keep = np.flatnonzero(~np.isfinite(a[field]))
    order = np.r_[keep, np.setdiff1d(order, keep, assume_unique=True)]   # the non-finite rows open chunk 0
    _cply_check(a, cuda, order)


@pytest.mark.gpu
def test_cply_pack_quaternions_first_nan_wins(cuda, gsx_lib):
    _cply_check(cply_quat_case(), cuda, np.arange(1024))


@pytest.mark.gpu
@pytest.mark.parametrize("n_rest,n", REST_CASES)
def test_cply_pack_rest_vector_and_byte_tail(n_rest, n, cuda, gsx_lib):
    _cply_check(cply_rest_case(n_rest, n), cuda, np.random.default_rng(n).permutation(n))


@pytest.mark.gpu
def test_cply_encode_nan_positions_in_morton_order(cuda, gsx_lib):
    """The whole encode with its own Morton order: NaN positions order as the reference recursion does."""
    from test_sort_morton_paths_gpu import morton_ref
    a = cply_nonfinite_case("y")
    xyz = np.stack([a["x"], a["y"], a["z"]], axis=1)
    want_order, _ = morton_ref(xyz)
    o = _cply_check(a, cuda, None)
    assert np.array_equal(o, want_order)


# ------------------------------------------------------------------------------------------------ SOG lexsort
LEX_AXES = ["x", "y", "z"]


def lexsort_case(axis, n=3001):
    """Rows with ties on every level; NaN of both signs and two payloads, +-inf and +-0 in one axis."""
    rng = np.random.default_rng(ord(axis))
    xyz = np.round(rng.normal(0, 2, (n, 3)).astype(np.float32) * 2) / 2
    col = "xyz".index(axis)
    specials = [np.nan, NEG_NAN, NAN_PAYLOAD, NEG_NAN_PAYLOAD, np.inf, -np.inf, 0.0, -0.0]
    for k, v in enumerate(specials * 12):
        xyz[(37 * k + 11) % n, col] = v
    return np.ascontiguousarray(xyz, np.float32)


@pytest.mark.parametrize("axis", LEX_AXES)
def test_lexsort_case_reaches_its_path(axis):
    xyz = lexsort_case(axis)
    col = xyz[:, "xyz".index(axis)]
    bits = col.view(np.uint32)
    nan = np.isnan(col)
    assert set(np.unique(bits[nan])) == {0x7FC00000, 0xFFC00000, 0x7FC00123, 0xFFD00001}
    assert np.isinf(col).any() and (bits == 0x80000000).any() and (bits == 0).any()
    # the order-preserving bit mapping alone puts a negative NaN first and sorts NaNs by payload: not np.lexsort
    key = np.where(bits >> 31 == 1, ~bits, bits | np.uint32(0x80000000))
    assert not np.array_equal(np.argsort(key, kind="stable"), np.argsort(col, kind="stable"))


@pytest.mark.gpu
@pytest.mark.parametrize("axis", LEX_AXES)
def test_lexsort_nonfinite_matches_numpy(axis, cuda, gsx_lib):
    import torch
    from gsx import sog
    xyz = lexsort_case(axis)
    want = np.lexsort((xyz[:, 2], xyz[:, 1], xyz[:, 0]))
    got = sog.lexsort_zyx(torch.from_numpy(xyz).to(cuda)).cpu().numpy()
    assert np.array_equal(got, want)


# ------------------------------------------------------------------------------------------------ SOG encode
def quantile_fit(values):
    return np.quantile(values.reshape(-1), np.linspace(0, 1, 256)).astype(np.float32)


def sog_nan_case():
    """2 000 SH-3 rows with NaN / -NaN / +-inf positions on every axis, NaN opacities and NaN quaternions.  The
    K-Means inputs (scales, f_dc, f_rest) stay finite."""
    from gsx import synth
    a = synth.structured(2_000, "mixed")
    for k, f in enumerate(("x", "y", "z")):
        a[f][[10 + k, 500 + k, 900 + k]] = (np.nan, NEG_NAN, np.inf)
    a["x"][1500], a["z"][1501] = -np.inf, NAN_PAYLOAD
    a["opacity"][[20, 21]] = (np.nan, NEG_NAN)
    a["rot_1"][30], a["rot_3"][31] = np.nan, np.inf
    return a


def test_sog_nan_case_reaches_its_path():
    a = sog_nan_case()
    order = np.lexsort((a["z"], a["y"], a["x"]))
    nan_rows = np.flatnonzero(np.isnan(a["x"]))
    assert np.array_equal(order[-len(nan_rows):], nan_rows)      # NaN x rows last, in index order
    for f in ("scale_0", "f_dc_0", "f_rest_0"):
        assert np.isfinite(a[f]).all()


@pytest.mark.gpu
def test_sog_encode_with_nan_rows_matches_oracle(cuda, gsx_lib):
    from gsx import records, sog
    a = sog_nan_case()
    r = records.DeviceRecords.from_structured(a, cuda)
    np.random.seed(3)
    enc = sog.encode(r, 0, codebook_fit=quantile_fit)
    got = enc.to_host()
    np.random.seed(3)
    with np.errstate(all="ignore"):
        want, want_meta, order = so.encode(a, 0, codebook_fit=quantile_fit)
    assert np.array_equal(enc.order.cpu().numpy(), order)
    so.assert_sog_equal(got, enc.meta, want, want_meta)


# ------------------------------------------------------------------------------------------------ SOG kernels
SH_GATHER_COLS = [9, 24, 32, 33, 45]
SH_GATHER_N = [1, 13, 1001]


def sh_gather_case(ncols, n):
    rng = np.random.default_rng(ncols * 100 + n)
    F = 62
    rows = rng.normal(0, 1, (n, F)).astype(np.float32)
    cols = rng.choice(F, ncols, replace=False).astype(np.int32)
    rows[:, cols[::3]] = 0.0                                      # zero columns, one of them -0.0
    rows[:, cols[1]] = -0.0
    rows[n // 2, cols[-1]] = np.nan
    order = rng.permutation(n).astype(np.int32)
    return rows, cols, order


@pytest.mark.parametrize("ncols", SH_GATHER_COLS)
def test_sh_gather_case_reaches_its_path(ncols):
    rows, cols, order = sh_gather_case(ncols, 1001)
    assert (ncols > 32) == (ncols in (33, 45))                    # lanes k + 32 carry columns
    nz = (rows[:, cols] != 0).any(axis=0)
    assert not nz.all() and nz.any() and nz[-1]                   # the NaN column counts as non-zero
    assert 1001 % 8 != 0 and 13 % 8 != 0


@pytest.mark.gpu
@pytest.mark.parametrize("n", SH_GATHER_N)
@pytest.mark.parametrize("ncols", SH_GATHER_COLS)
def test_sog_sh_gather_columns_and_mask(ncols, n, cuda, gsx_lib):
    import torch
    from gsx import _abi
    from gsx._abi import _ptr, _stream
    rows, cols, order = sh_gather_case(ncols, n)
    rt, ot = torch.from_numpy(rows).to(cuda), torch.from_numpy(order).to(cuda)
    out = torch.full((n, ncols), 7.0, dtype=torch.float32, device=cuda)
    nz = torch.empty(1, dtype=torch.int64, device=cuda)
    carr = (C.c_int32 * ncols)(*cols.tolist())
    assert _abi.lib.gsx_sog_sh_gather(_ptr(rt), n, rows.shape[1], _ptr(ot), carr, ncols, _ptr(out), _ptr(nz),
                                      _stream()) == 0
    want = rows[order][:, cols]
    assert np.array_equal(out.cpu().numpy().view(np.uint32), want.view(np.uint32))
    mask = int(nz.cpu().numpy().view(np.uint64)[0])
    want_nz = (want != 0).any(axis=0)
    assert mask == sum(1 << k for k in range(ncols) if want_nz[k])


LABEL_CASES = {"near_wrap": ([65_000, 65_530, 65_535], [0, 1, 0]), "all_pass": ([65_535, 0, 65_536], [1, 1, 1]),
               "none_pass": ([1, 65_280, 65_520], [0, 0, 0])}


def labels_case(name, n=3001, chunk=1001):
    offsets, passthrough = LABEL_CASES[name]
    rng = np.random.default_rng(len(name))
    labels = rng.integers(0, 40, n).astype(np.int32)
    width, height = so.texture_size(n)
    want = np.zeros((width * height, 4), np.uint8)
    l16 = np.concatenate([(np.arange(min(chunk, n - c * chunk)) if passthrough[c] else
                           labels[c * chunk:(c + 1) * chunk]) + offsets[c] for c in range(3)]).astype(np.uint16)
    want[:n, 0], want[:n, 1], want[:n, 3] = l16 & 0xFF, l16 >> 8, 255
    return labels, offsets, passthrough, chunk, width * height, want


@pytest.mark.parametrize("name", list(LABEL_CASES))
def test_labels_case_reaches_its_path(name):
    labels, offsets, passthrough, chunk, pixels, want = labels_case(name)
    total = np.concatenate([labels[:chunk] + offsets[0], labels[chunk:] + max(offsets)])
    if name != "all_pass":
        assert (total > 65_535).any() or name == "none_pass"
    assert pixels > len(labels)                                   # padding pixels
    if name == "near_wrap":
        assert passthrough[1] and offsets[1] + chunk > 65_536     # a passthrough chunk wraps past 65 535


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(LABEL_CASES))
def test_sog_labels_passthrough_and_wrap(name, cuda, gsx_lib):
    import torch
    from gsx import _abi
    from gsx._abi import _ptr, _stream
    labels, offsets, passthrough, chunk, pixels, want = labels_case(name)
    lt = torch.from_numpy(labels).to(cuda)
    out = torch.full((pixels, 4), 9, dtype=torch.uint8, device=cuda)
    i3 = lambda v: (C.c_int32 * 3)(*v)
    assert _abi.lib.gsx_sog_labels(_ptr(lt), len(labels), chunk, 3, i3(offsets), i3(passthrough), pixels, _ptr(out),
                                   _stream()) == 0
    assert np.array_equal(out.cpu().numpy(), want)


CENTROID_CASES = [(37, 9), (100, 45), (65, 24), (1, 3)]


def centroids_case(P, coeffs):
    rng = np.random.default_rng(P * 64 + coeffs)
    pal = rng.normal(0, 0.3, (P, coeffs)).astype(np.float32)
    cb = np.sort(rng.normal(0, 0.3, 256).astype(np.float32))
    pal.flat[::17] = cb[rng.integers(0, 256, pal.size)[::17]]      # exact codebook hits
    w_c, h_c = 64 * coeffs, int(np.ceil(P / 64))
    idx = so.quantize_to_codebook(pal.flatten(), cb)
    want = np.full((w_c * h_c, 4), 255, np.uint8)
    pix = idx.reshape(P, 3, coeffs // 3).transpose(0, 2, 1).reshape(-1, 3)
    want[:len(pix), :3] = pix
    return pal, cb, w_c * h_c, want


@pytest.mark.parametrize("P,coeffs", CENTROID_CASES)
def test_centroids_case_reaches_its_path(P, coeffs):
    _, _, pixels, _ = centroids_case(P, coeffs)
    assert (P * (coeffs // 3)) % (64 * coeffs) != 0 and pixels > P * (coeffs // 3)


@pytest.mark.gpu
@pytest.mark.parametrize("P,coeffs", CENTROID_CASES)
def test_sog_centroids_layout(P, coeffs, cuda, gsx_lib):
    import torch
    from gsx import _abi
    from gsx._abi import _ptr, _stream
    pal, cb, pixels, want = centroids_case(P, coeffs)
    pt, ct = torch.from_numpy(pal).to(cuda), torch.from_numpy(cb).to(cuda)
    out = torch.zeros((pixels, 4), dtype=torch.uint8, device=cuda)
    assert _abi.lib.gsx_sog_centroids(_ptr(pt), P, coeffs, _ptr(ct), len(cb), pixels, _ptr(out), _stream()) == 0
    assert np.array_equal(out.cpu().numpy(), want)
