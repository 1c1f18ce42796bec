"""The SOG texture kernels path by path: gsx_sog_means_minmax, gsx_sog_means, gsx_sog_quats, gsx_sog_gather_values
and gsx_sog_scales_sh0, called directly and compared bit for bit with a NumPy restatement of the reference writer's
expressions (formats/sog.py:279-459, as sog_oracle.encode has them).

Each case has a seeded builder, a CPU test that the data reaches the branch it is for, and a GPU test.  Every GPU case
reads its rows through a random permutation `order` and fills its outputs with a sentinel first, so the padding pixels
[n, pixels) are checked too.  The sign of a zero min or max is the one thing not compared: NumPy's own answer depends on
where the zeros sit (test_numpy_min_zero_sign_depends_on_position)."""
import ctypes as C

import numpy as np
import pytest

import sog_oracle as so

F32 = np.float32
U32 = np.uint32
F = 19                                       # row width: the columns below are scattered through it
XYZ = [5, 0, 17]
ROT = [3, 11, 8, 14]
C7 = [1, 9, 2, 16, 4, 12, 7]                 # scale_0..2, f_dc_0..2, opacity
MINMAX_WS = 1024 * 6 * 4                     # gsx_sog_means_minmax's workspace: 6 floats for each of 1024 blocks
SENT = 0x5A                                  # what the texture bytes hold before a launch
SENT_F = np.uint32(0x7FA5A5A5).view(F32)     # a NaN no kernel writes


def ref_log(v):
    """np.sign(v) * np.log(np.abs(v) + 1.0) (sog.py:279-280) in float32."""
    with np.errstate(all="ignore"):
        return np.sign(v) * np.log(np.abs(v) + 1.0)


def ref_minmax(rows):
    ls = [ref_log(rows[:, c]) for c in XYZ]
    return np.array([np.min(v) for v in ls] + [np.max(v) for v in ls], F32)


def ref_means(rows, order, mm, pixels):
    """means_l, means_u (sog.py:289-309) against the bounds mm = (min x, y, z, max x, y, z)."""
    s = rows[order]
    n = len(order)
    lo = np.full((pixels, 4), 255, np.uint8)
    hi = np.full((pixels, 4), 255, np.uint8)
    for i, c in enumerate(XYZ):
        with np.errstate(all="ignore"):
            u = np.clip((ref_log(s[:, c]) - mm[i]) / (mm[3 + i] - mm[i]) * 65535, 0, 65535).astype(np.uint16)
        lo[:n, i], hi[:n, i] = u & 0xFF, u >> 8
    return lo, hi


def ref_quat_bytes(q, sqrt2=np.sqrt(2.0)):
    """(qb [m, 4], max_idx) of sog.py:315-353 for raw quaternion rows q; sqrt2 = np.sqrt(2.0) is a float64 scalar."""
    with np.errstate(all="ignore"):
        qn = q / np.linalg.norm(q, axis=1, keepdims=True)
        max_idx = np.abs(qn).argmax(axis=1)
        qn *= np.sign(np.take_along_axis(qn, max_idx[:, None], axis=1).flatten()).reshape(-1, 1)
        qn *= sqrt2
        qb = np.clip((qn * 0.5 + 0.5) * 255.0, 0, 255).astype(np.uint8)
    return qb, max_idx


def ref_quats(rows, order, pixels):
    n = len(order)
    qb, max_idx = ref_quat_bytes(rows[order][:, ROT])
    keep = np.array([[1, 2, 3], [0, 2, 3], [0, 1, 3], [0, 1, 2]])[max_idx]
    out = np.full((pixels, 4), 255, np.uint8)
    out[:n, :3] = np.take_along_axis(qb, keep, axis=1)
    out[:n, 3] = 252 + max_idx.astype(np.uint8)
    return out


def ref_alpha(opacity):
    """sh0 alpha (sog.py:452-453)."""
    with np.errstate(all="ignore"):
        return np.clip(1.0 / (1.0 + np.exp(-opacity)) * 255, 0, 255).astype(np.uint8)


def ref_scales_sh0(rows, order, scb, ccb, pixels):
    s = rows[order]
    n = len(order)
    scales = np.zeros((pixels, 4), np.uint8)
    sh0 = np.zeros((pixels, 4), np.uint8)
    for i in range(3):
        scales[:n, i] = so.quantize_to_codebook(s[:, C7[i]], scb)
        sh0[:n, i] = so.quantize_to_codebook(s[:, C7[3 + i]], ccb)
    scales[:n, 3] = 255
    sh0[:n, 3] = ref_alpha(s[:, C7[6]])
    return scales, sh0


def base_rows(n, seed):
    rng = np.random.default_rng(seed)
    rows = rng.normal(0, 10, (n, F)).astype(F32)
    return rows, rng.permutation(n).astype(np.int32), rng


def neighbours(v, k):
    """The float32 values within k ulps of each v (v itself included), flattened."""
    v = np.asarray(v, F32).reshape(-1, 1)
    out = [v]
    up, down = v.copy(), v.copy()
    for _ in range(k):
        up, down = np.nextafter(up, F32(np.inf)), np.nextafter(down, F32(-np.inf))
        out += [up, down]
    return np.concatenate(out, axis=1).reshape(-1)


def i32s(v):
    return (C.c_int32 * len(v))(*[int(x) for x in v])


def _dev():
    from gsx import _abi
    from gsx._abi import _ptr, _stream
    return _abi.lib, _ptr, _stream


def _texture(pixels, cuda):
    import torch
    return torch.full((pixels, 4), SENT, dtype=torch.uint8, device=cuda)


def _sentinel_floats(count, cuda):
    import torch
    return torch.from_numpy(np.full(count, SENT_F)).to(cuda)      # bit for bit: a Python float would quiet the NaN


def _assert_texture(name, got, want):
    bad = np.flatnonzero(np.any(got != want, axis=1))
    assert bad.size == 0, f"{name}: {bad.size} pixels differ, first {bad[:8]}: {got[bad[:3]]} vs {want[bad[:3]]}"


# ================================================================================================= means min / max
def grid_stride(sm_count):
    """Rows between a thread's grid-stride steps in k_sog_log_minmax: 256 threads times the clamped grid."""
    return 256 * min(8 * sm_count, 1024)


H100_STRIDE = grid_stride(132)
MINMAX_SIZES = [1, 31, 256, 257, 1000, 300_000]     # 1000 = 3 full blocks + 232 rows; 300 000 > 256 * 1024


def minmax_places(n, stride):
    """Rows for the extremes: lane 0 of block 0, the last row of the last block, and a row that only a thread's second
    grid-stride step reads (the middle row where the grid covers every row in one step)."""
    return [0, n - 1, stride + 77 if n > stride + 77 else n // 2]


def minmax_case(n, stride=H100_STRIDE):
    rows, _, _ = base_rows(n, n)
    places = minmax_places(n, stride)
    for a, c in enumerate(XYZ):
        rows[places[a], c] = -5e4 - a                  # each axis has its minimum and maximum in other places
        rows[places[(a + 1) % 3], c] = 7e4 + a
    return rows


@pytest.mark.parametrize("n", MINMAX_SIZES)
def test_minmax_case_reaches_its_path(n):
    rows = minmax_case(n)
    places = minmax_places(n, H100_STRIDE)
    if n == 300_000:
        assert n > H100_STRIDE and places[2] >= H100_STRIDE and places[2] - H100_STRIDE < 256   # block 0, step 2
    if n == 1000:
        assert n % 256 and n // 256 == 3
    if n > 2:
        assert len(set(places)) == 3
        for a, c in enumerate(XYZ):
            assert np.argmin(rows[:, c]) == places[a] and np.argmax(rows[:, c]) == places[(a + 1) % 3]


MINMAX_VALUES = ["nan", "neg_nan", "inf", "equal"]


def minmax_value_case(name, n=5000):
    rows, _, _ = base_rows(n, 7 + MINMAX_VALUES.index(name))
    if name == "nan":                                  # a lone NaN per axis, each in another place
        for a, r in enumerate((0, n - 1, 2345)):
            rows[r, XYZ[a]] = np.nan
    elif name == "neg_nan":
        for a, r in enumerate((0, n - 1, 2345)):
            rows[r, XYZ[a]] = -np.float32(np.nan)
    elif name == "inf":                                # x: +inf, y: -inf, z: both
        rows[17, XYZ[0]] = np.inf
        rows[n - 1, XYZ[1]] = -np.inf
        rows[0, XYZ[2]], rows[n - 2, XYZ[2]] = np.inf, -np.inf
    else:                                              # x constant, y all zeros of both signs, z normal
        rows[:, XYZ[0]] = 3.25
        rows[:, XYZ[1]] = 0.0
        rows[::3, XYZ[1]] = -0.0
    return rows


@pytest.mark.parametrize("name", MINMAX_VALUES)
def test_minmax_value_case_reaches_its_path(name):
    rows = minmax_value_case(name)
    mm = ref_minmax(rows)
    if name in ("nan", "neg_nan"):
        assert np.isnan(mm).all() and np.isnan(rows[:, XYZ]).sum() == 3
        assert (np.signbit(rows[:, XYZ][np.isnan(rows[:, XYZ])]) == (name == "neg_nan")).all()
    elif name == "inf":
        assert list(mm[[3, 1, 2, 5]]) == [np.inf, -np.inf, -np.inf, np.inf] and np.isfinite(mm[[0, 4]]).all()
    else:
        assert mm[0] == mm[3] and mm[1] == mm[4] == 0 and mm[2] < mm[5]


def test_numpy_min_zero_sign_depends_on_position():
    """What np.min / np.max give for mixed zeros depends on where they sit (NumPy 2.3.5, x86), so the minmax tests
    compare values with ==: the sign of a zero bound is free (a zero bound maps to the same u16 either way)."""
    signs = set()
    for pos in range(8):
        a = np.full(17, 5.0, F32)
        a[pos], a[pos + 1] = -0.0, 0.0
        r = np.min(a)
        assert r == 0
        signs.add(bool(np.signbit(r)))
    assert signs == {False, True}


def dev_minmax(rows, cuda, n=None):
    import torch
    lib, _ptr, _stream = _dev()
    n = len(rows) if n is None else n
    rt = torch.from_numpy(rows).to(cuda)
    ws = _sentinel_floats(MINMAX_WS // 4, cuda)
    mm = _sentinel_floats(8, cuda)
    assert lib.gsx_sog_means_minmax(_ptr(rt), n, F, i32s(XYZ), _ptr(ws), MINMAX_WS, _ptr(mm), _stream()) == 0
    got = mm.cpu().numpy()
    assert (got[6:].view(U32) == SENT_F.view(U32)).all()           # exactly six floats written
    return got[:6]


def _assert_minmax(got, want):
    assert np.array_equal(got, want, equal_nan=True), (got, want)


@pytest.mark.gpu
@pytest.mark.parametrize("n", MINMAX_SIZES)
def test_sog_means_minmax_sizes_and_places(n, cuda, gsx_lib):
    stride = grid_stride(gsx_lib.gsx_device_sm_count())
    if n == 300_000:
        assert n > stride + 77                                     # the clamped grid: threads take a second step
    rows = minmax_case(n, stride)
    _assert_minmax(dev_minmax(rows, cuda), ref_minmax(rows))


@pytest.mark.gpu
@pytest.mark.parametrize("name", MINMAX_VALUES)
def test_sog_means_minmax_values(name, cuda, gsx_lib):
    rows = minmax_value_case(name)
    _assert_minmax(dev_minmax(rows, cuda), ref_minmax(rows))


# ========================================================================================================= means
MEANS_CASES = ["degenerate", "inf_extent", "nan", "nan_rows", "near_integer"]
PIXELS = ["n", "n+1", "texture"]


def near_integer_values(lo, hi, count, seed):
    """float32 v in (lo, hi) whose (l - mn) / (mx - mn) * 65535 in float32 lies within one ulp of an integer, for the
    bounds mn = ref_log(lo), mx = ref_log(hi): float32 neighbours of the exact preimages of integers."""
    mn, mx = ref_log(np.array([lo, hi], F32))
    ks = np.random.default_rng(seed).integers(1, 65535, count)
    l64 = np.float64(mn) + ks * (np.float64(mx) - np.float64(mn)) / 65535
    v = neighbours(np.sign(l64) * np.expm1(np.abs(l64)), 6)
    with np.errstate(all="ignore"):
        t = (ref_log(v) - mn) / (mx - mn) * 65535
    r = np.round(t)
    return v[(np.abs(t - r) <= np.spacing(np.abs(t).astype(F32))) & (v > lo) & (v < hi)]


def means_case(name, n=3001):
    rows, order, rng = base_rows(n, 100 + MEANS_CASES.index(name))
    if name == "degenerate":                           # every x equal: 0/0 on that axis
        rows[:, XYZ[0]] = -2.5
    elif name == "inf_extent":                         # x: both infinities (inf/inf, NaN), y: +inf only
        rows[5, XYZ[0]], rows[6, XYZ[0]] = np.inf, -np.inf
        rows[n - 1, XYZ[1]] = np.inf
    elif name in ("nan", "nan_rows"):                  # NaN positions on every axis
        for a, c in enumerate(XYZ):
            rows[rng.choice(n, 7, replace=False), c] = np.nan if a != 1 else -np.float32(np.nan)
    else:
        for a, c in enumerate(XYZ):
            rows[0, c], rows[1, c] = -60.0 - a, 90.0 + a
            v = near_integer_values(rows[0, c], rows[1, c], 4000, a)[: n - 2]
            rows[2:2 + len(v), c] = v
    return rows, order


def means_bounds(name, rows):
    """The bounds the kernel gets: the reference's own, except for nan_rows, where they are the finite bounds of the
    other rows, so that the NaN rows themselves go through the normalisation."""
    if name != "nan_rows":
        return ref_minmax(rows)
    with np.errstate(all="ignore"):
        ls = [ref_log(rows[:, c]) for c in XYZ]
    return np.array([np.nanmin(v) for v in ls] + [np.nanmax(v) for v in ls], F32)


def means_pixels(kind, n):
    w, h = so.texture_size(n)
    return {"n": n, "n+1": n + 1, "texture": w * h}[kind]


@pytest.mark.parametrize("name", MEANS_CASES)
def test_means_case_reaches_its_path(name):
    rows, order = means_case(name)
    n = len(rows)
    mm = means_bounds(name, rows)
    lo, hi = ref_means(rows, order, mm, n)
    u = lo[:, :3].astype(np.int64) | hi[:, :3].astype(np.int64) << 8
    assert sorted(order) == list(range(n)) and (order != np.arange(n)).any()
    assert means_pixels("texture", n) > n + 1
    if name == "degenerate":
        assert mm[0] == mm[3] and (u[:, 0] == 0).all() and u[:, 1:].max() == 65535
    elif name == "inf_extent":
        assert np.isinf(mm[0]) and np.isinf(mm[3]) and np.isinf(mm[4]) and np.isfinite(mm[1])
        assert (u[:, :2] == 0).all() and u[:, 2].max() == 65535
    elif name == "nan":
        assert np.isnan(mm).all() and (u == 0).all()
    elif name == "nan_rows":
        assert np.isfinite(mm).all() and (u[np.isnan(rows[order][:, XYZ])] == 0).all()
        assert (u.max(axis=0) == 65535).all()
    else:
        with np.errstate(all="ignore"):
            t = np.stack([(ref_log(rows[:, c]) - mm[a]) / (mm[3 + a] - mm[a]) * 65535 for a, c in enumerate(XYZ)], 1)
        r = np.round(t[2:])
        exact, below = t[2:] == r, (t[2:] < r) & (t[2:] >= r - np.spacing(r.astype(F32)))
        assert exact.sum(axis=0).min() > 100 and below.sum(axis=0).min() > 100   # both sides of the truncation


def dev_means(rows, order, mm, pixels, cuda):
    import torch
    lib, _ptr, _stream = _dev()
    rt, ot = torch.from_numpy(rows).to(cuda), torch.from_numpy(order).to(cuda)
    mt = torch.from_numpy(np.asarray(mm, F32)).to(cuda)
    lo, hi = _texture(pixels, cuda), _texture(pixels, cuda)
    assert lib.gsx_sog_means(_ptr(rt), len(order), F, _ptr(ot), i32s(XYZ), _ptr(mt), pixels, _ptr(lo), _ptr(hi),
                             _stream()) == 0
    return lo.cpu().numpy(), hi.cpu().numpy()


@pytest.mark.gpu
@pytest.mark.parametrize("pixels", PIXELS)
@pytest.mark.parametrize("name", MEANS_CASES)
def test_sog_means_edges(name, pixels, cuda, gsx_lib):
    rows, order = means_case(name)
    mm = means_bounds(name, rows)
    p = means_pixels(pixels, len(rows))
    want_lo, want_hi = ref_means(rows, order, mm, p)
    got_lo, got_hi = dev_means(rows, order, mm, p, cuda)
    _assert_texture("means_l", got_lo, want_lo)
    _assert_texture("means_u", got_hi, want_hi)


@pytest.mark.gpu
def test_sog_minmax_and_means_one_million(cuda, gsx_lib):
    """The two kernels back to back on synth.structured(1 000 000, 'mixed'), byte for byte with the reference."""
    from gsx import synth
    a = synth.structured(1_000_000, "mixed")
    n = len(a)
    rows = np.zeros((n, F), F32)
    for f, c in zip("xyz", XYZ):
        rows[:, c] = a[f]
    order = np.random.default_rng(5).permutation(n).astype(np.int32)
    want_mm = ref_minmax(rows)
    got_mm = dev_minmax(rows, cuda)
    _assert_minmax(got_mm, want_mm)
    w, h = so.texture_size(n)
    want_lo, want_hi = ref_means(rows, order, want_mm, w * h)
    got_lo, got_hi = dev_means(rows, order, got_mm, w * h, cuda)
    _assert_texture("means_l", got_lo, want_lo)
    _assert_texture("means_u", got_hi, want_hi)


# ========================================================================================================= quats
SQRT2_F32 = F32(np.sqrt(2.0))


def crafted_sqrt2_rows():
    """Quaternion rows where q * np.sqrt(2.0) in float32 (instead of float64 rounded once) changes a byte: float32
    neighbours of components that land on a quantize_vec byte boundary, rolled so the largest index varies."""
    ks = np.arange(20, 236)
    c = neighbours((2 * ks / 255.0 - 1) / np.sqrt(2.0), 48)   # (c * sqrt2 * 0.5 + 0.5) * 255 == k
    q = np.stack([c, np.full_like(c, 0.1), np.full_like(c, -0.2),
                  np.sqrt(1 - c.astype(np.float64) ** 2 - 0.05).astype(F32)], 1)
    q = np.concatenate([np.roll(q[k::4], k + 1, axis=1) * (-1) ** k for k in range(4)])
    return q[np.any(ref_quat_bytes(q)[0] != ref_quat_bytes(q, SQRT2_F32)[0], axis=1)]


QUAT_CASES = {
    "neg_largest": [(-0.9, 0.1, 0.2, 0.3), (0.1, -0.95, 0.2, -0.1), (0.3, 0.1, -0.8, 0.2), (0.1, 0.2, -0.3, -0.9)],
    "ties": [(0.5, 0.5, 0.5, 0.5), (-0.5, 0.5, -0.5, 0.5), (0.0, 0.6, -0.6, 0.0), (0.1, 0.2, -0.7, 0.7),
             (-0.7, 0.1, 0.1, -0.7)],
    "nan": [(np.nan, 0.9, 0.1, 0.1), (0.9, np.nan, 0.1, 0.1), (0.1, 0.1, np.nan, 0.9), (0.1, 0.9, 0.1, np.nan),
            (0.1, -np.nan, np.nan, 0.5)],
    "zero": [(0, 0, 0, 0), (0.0, -0.0, 0.0, -0.0), (-0.0, -0.0, -0.0, -0.0)],
    "inf": [(np.inf, 1, 0, 0), (1, -np.inf, 0, 0), (0, 1, np.inf, -np.inf), (0.5, 0.5, 0.5, np.inf)],
    "denormal": [(1e-40, 0, 0, 0), (0, -1e-42, 0, 1e-45), (0.6, 1e-39, -1e-41, 0.8), (1e-38, 2e-38, -3e-38, 1e-39)],
    "sqrt2": None,
}


def quats_case(name):
    """(rows, order, k): the case's quaternions are rows[:k], random ones follow."""
    q = crafted_sqrt2_rows() if name == "sqrt2" else np.array(QUAT_CASES[name], F32)
    k = len(q)
    q = np.concatenate([q, np.random.default_rng(3).normal(0, 1, (300, 4)).astype(F32)])
    rows, order, _ = base_rows(len(q), 200 + list(QUAT_CASES).index(name))
    rows[:, ROT] = q
    return rows, order, k


@pytest.mark.parametrize("name", list(QUAT_CASES))
def test_quats_case_reaches_its_path(name):
    rows, order, k = quats_case(name)
    q = rows[:k, ROT]
    qb, L = ref_quat_bytes(q)
    with np.errstate(all="ignore"):
        qn = q / np.linalg.norm(q, axis=1, keepdims=True)
    if name == "neg_largest":
        assert list(L) == [0, 1, 2, 3] and (qn[np.arange(4), L] < 0).all()
    elif name == "ties":
        a = np.abs(qn)
        assert all((a[i] == a[i, L[i]]).sum() >= 2 for i in range(k))             # the first of equals wins
        assert list(L) == [0, 0, 1, 2, 0]
    elif name == "nan":
        assert np.isnan(qn).all() and (L == 0).all()
    elif name == "zero":
        assert np.isnan(qn).all() and (L == 0).all() and (qb[:, :3] == 0).all()
    elif name == "inf":
        assert list(L) == [0, 1, 2, 3] and np.isnan(qn[np.arange(4), L]).all()   # inf / inf: the NaN is the max
    elif name == "denormal":
        sub = (q != 0) & (np.abs(q) < np.finfo(F32).tiny)
        assert sub.any(axis=1).all() and L[0] == 1 and L[2] == 3                  # 1e-40 / 0 = inf, then 0 / 0
        assert np.isinf(qn[0, 0]) and np.isfinite(qn[2]).all() and np.isinf(qn[3]).all()
    else:
        assert k >= 20 and len(set(L)) == 4


def test_crafted_sqrt2_rows_depend_on_float64_product():
    """Every crafted row changes a byte when the np.sqrt(2.0) product is done in float32."""
    q = crafted_sqrt2_rows()
    assert len(q) >= 20
    assert np.any(ref_quat_bytes(q)[0] != ref_quat_bytes(q, SQRT2_F32)[0], axis=1).all()


@pytest.mark.gpu
@pytest.mark.parametrize("pixels", PIXELS)
@pytest.mark.parametrize("name", list(QUAT_CASES))
def test_sog_quats_edges(name, pixels, cuda, gsx_lib):
    lib, _ptr, _stream = _dev()
    import torch
    rows, order, _ = quats_case(name)
    p = means_pixels(pixels, len(rows))
    rt, ot = torch.from_numpy(rows).to(cuda), torch.from_numpy(order).to(cuda)
    out = _texture(p, cuda)
    assert lib.gsx_sog_quats(_ptr(rt), len(rows), F, _ptr(ot), i32s(ROT), p, _ptr(out), _stream()) == 0
    _assert_texture("quats", out.cpu().numpy(), ref_quats(rows, order, p))


# ================================================================================================== gather values
GATHER_F = 62
GATHER_N = 1001
GATHER_CASES = [("all", 1), ("all", 3), ("all", 45), ("seams", 3), ("repeated", 45)]


def gather_case(kind, ncols, n=GATHER_N):
    rng = np.random.default_rng(ncols * 10 + len(kind))
    rows = rng.normal(0, 1, (n, GATHER_F)).astype(F32)
    rows[::7, 3] = -0.0
    rows[n // 3, :] = np.nan
    cols = rng.choice(GATHER_F, ncols, replace=False).astype(np.int32)
    order = rng.permutation(n).astype(np.int32)
    if kind == "all":
        sel = None
    elif kind == "seams":
        sel = np.array([0, n - 1, n, 2 * n - 1, 3 * n - 1, 2 * n, n + 1, 1], np.int64)
    else:
        sel = rng.integers(0, n * ncols, 3000).astype(np.int64)
        sel[1000:1100] = sel[5]
        sel[-1] = n * ncols - 1
    return rows, cols, order, sel


def ref_gather(rows, cols, order, sel):
    v = np.concatenate([rows[order, c] for c in cols])
    return v if sel is None else v[sel]


@pytest.mark.parametrize("kind,ncols", GATHER_CASES)
def test_gather_case_reaches_its_path(kind, ncols):
    rows, cols, order, sel = gather_case(kind, ncols)
    n = len(rows)
    if sel is None:
        assert len(ref_gather(rows, cols, order, sel)) == n * ncols
    elif kind == "seams":
        assert set(sel // n) == {0, 1, 2} and {n - 1, n, 2 * n - 1, 3 * n - 1} <= set(sel.tolist())
    else:
        assert len(np.unique(sel)) < len(sel) and sel.max() == n * ncols - 1


@pytest.mark.gpu
@pytest.mark.parametrize("kind,ncols", GATHER_CASES)
def test_sog_gather_values(kind, ncols, cuda, gsx_lib):
    import torch
    lib, _ptr, _stream = _dev()
    rows, cols, order, sel = gather_case(kind, ncols)
    want = ref_gather(rows, cols, order, sel)
    m = len(want)
    rt, ot = torch.from_numpy(rows).to(cuda), torch.from_numpy(order).to(cuda)
    st = None if sel is None else torch.from_numpy(sel).to(cuda)
    out = _sentinel_floats(m + 5, cuda)
    assert lib.gsx_sog_gather_values(_ptr(rt), len(rows), GATHER_F, _ptr(ot), i32s(cols), ncols, _ptr(st), m,
                                     _ptr(out), _stream()) == 0
    got = out.cpu().numpy().view(U32)
    assert np.array_equal(got[:m], want.view(U32)) and (got[m:] == SENT_F.view(U32)).all()


# ======================================================================================================= scales / sh0
CODEBOOK_SIZES = [(1, 256), (2, 255), (255, 2), (256, 1)]


def codebook(m, seed):
    """An ascending float32 codebook of m entries; from 8 entries on it has duplicates and both zeros."""
    rng = np.random.default_rng(seed)
    if m == 1:
        return np.array([0.125], F32)
    if m == 2:
        return np.array([-0.5, 0.75], F32)
    cb = np.sort(rng.normal(0, 1, m).astype(F32))
    cb[m // 5 + 1] = cb[m // 5]                                # a duplicate pair
    cb[3 * m // 4:3 * m // 4 + 3] = cb[3 * m // 4]             # three equal entries
    z = np.searchsorted(cb, 0)
    cb[max(z - 1, 0)], cb[min(z, m - 1)] = -0.0, 0.0           # -0.0 then +0.0
    assert (np.diff(cb) >= 0).all()
    return cb


def codebook_values(cb):
    """Exact hits, exact midpoints (ties keep the right-hand entry), values beyond both ends, ±0, NaN and ±inf."""
    mid = (cb[:-1] + cb[1:]) / F32(2)
    tie = mid[np.abs(mid - cb[:-1]) == np.abs(mid - cb[1:])]
    return np.concatenate([cb, tie, neighbours(mid, 1), [cb[0] - 1, cb[0] - 1e6, cb[-1] + 1, cb[-1] * 4 + 1e6],
                           [0.0, -0.0, np.nan, -np.float32(np.nan), np.inf, -np.inf]]).astype(F32)


def alpha_opacities():
    """Opacities on both sides of every alpha byte boundary, around and beyond exp's overflow (-op > 88.72) and
    underflow (-op < -103.97) thresholds, and NaN."""
    k = np.arange(1, 255)
    edges = neighbours(np.log(k / (255.0 - k)), 8)
    limits = neighbours([-88.7228394, 103.972084, -87.5, 88.5, 100.0], 4)
    return np.concatenate([edges, limits, [-200, 200, -95, 95, 0.0, -0.0, np.inf, -np.inf, np.nan,
                                           -np.float32(np.nan)]]).astype(F32)


def scales_case(ms, mc):
    scb, ccb = codebook(ms, ms), codebook(mc, mc + 1000)
    sv, cv, ov = codebook_values(scb), codebook_values(ccb), alpha_opacities()
    n = max(len(sv), len(cv), len(ov)) + 13
    rows, order, rng = base_rows(n, ms * 1000 + mc)
    for j, (c, v) in enumerate(zip(C7, [sv, sv, sv, cv, cv, cv, ov])):
        rows[:, c] = np.resize(np.roll(v, 5 * j), n)
    return rows, order, scb, ccb


@pytest.mark.parametrize("ms,mc", CODEBOOK_SIZES)
def test_scales_case_reaches_its_path(ms, mc):
    rows, order, scb, ccb = scales_case(ms, mc)
    assert len(scb) == ms and len(ccb) == mc
    for cb, c in ((scb, C7[0]), (ccb, C7[3])):
        v, m = rows[:, c], len(cb)
        idx = so.quantize_to_codebook(v, cb)
        assert idx[np.isnan(v)].tolist() and (idx[np.isnan(v)] == m - 1).all()
        if m >= 8:
            assert (np.diff(cb) == 0).sum() >= 3 and np.signbit(cb[cb == 0]).tolist() == [True, False]
        if m > 1:
            raw = np.clip(np.searchsorted(cb, v), 0, m - 1)
            with np.errstate(invalid="ignore"):
                tie = np.abs(v - cb[np.maximum(raw - 1, 0)]) == np.abs(v - cb[raw])
            assert (tie & (raw > 0) & (cb[raw] != cb[np.maximum(raw - 1, 0)])).any()   # a tie keeps the right entry
            assert (idx == 0).any() and (idx == m - 1).any() and (v < cb[0]).any() and (v > cb[-1]).any()
    op = rows[:, C7[6]]
    a = ref_alpha(op)
    k = np.arange(1, 255)
    ea = ref_alpha(neighbours(np.log(k / (255.0 - k)), 8).reshape(len(k), -1))
    both = [ea[i].min() == k[i] - 1 and ea[i].max() == k[i] for i in range(len(k))]
    assert sum(both) >= 230                           # the values straddle nearly every byte boundary
    with np.errstate(over="ignore"):
        ex = np.exp(-op)
    assert np.isinf(ex).any() and (ex == 0).any() and (np.isfinite(ex) & (ex > 0) & (-op > 88)).any()
    assert a[np.isnan(op)].tolist() == [0, 0] and len(set(a.tolist())) >= 250 and {0, 255} <= set(a.tolist())


@pytest.mark.gpu
@pytest.mark.parametrize("pixels", PIXELS)
@pytest.mark.parametrize("ms,mc", CODEBOOK_SIZES)
def test_sog_scales_sh0_codebooks_and_alpha(ms, mc, pixels, cuda, gsx_lib):
    import torch
    lib, _ptr, _stream = _dev()
    rows, order, scb, ccb = scales_case(ms, mc)
    p = means_pixels(pixels, len(rows))
    rt, ot = torch.from_numpy(rows).to(cuda), torch.from_numpy(order).to(cuda)
    st, ct = torch.from_numpy(scb).to(cuda), torch.from_numpy(ccb).to(cuda)
    scales, sh0 = _texture(p, cuda), _texture(p, cuda)
    assert lib.gsx_sog_scales_sh0(_ptr(rt), len(rows), F, _ptr(ot), i32s(C7), _ptr(st), ms, _ptr(ct), mc, p,
                                  _ptr(scales), _ptr(sh0), _stream()) == 0
    want_s, want_c = ref_scales_sh0(rows, order, scb, ccb, p)
    _assert_texture("scales", scales.cpu().numpy(), want_s)
    _assert_texture("sh0", sh0.cpu().numpy(), want_c)


# ============================================================================================================ refusals
NULL = None
FAKE = C.c_void_p(4096)                      # aligned and never dereferenced: every call below refuses on the host
ODD = C.c_void_p(4097)                       # an unaligned texture pointer
ARG, WORKSPACE = -2, -3


def _refuse(gsx_lib, rc, text):
    assert rc == ARG or rc == WORKSPACE, rc
    msg = gsx_lib.gsx_last_error()
    assert text.encode() in msg, msg
    return rc


MINMAX_REFUSALS = {
    "n_negative": (dict(n=-1), ARG, "out of range"),
    "n_2_pow_31": (dict(n=1 << 31), ARG, "out of range"),
    "row_width": (dict(F=0), ARG, "bad row width"),
    "no_splats": (dict(n=0), ARG, "no splats"),
    "workspace": (dict(ws_bytes=MINMAX_WS - 1), WORKSPACE, "workspace too small"),
    "column": (dict(cols=[5, 0, F]), ARG, "column 19 out of range"),
    "negative_column": (dict(cols=[-1, 0, 1]), ARG, "column -1 out of range"),
    "null_rows": (dict(rows=NULL), ARG, "null device pointer"),
}


@pytest.mark.parametrize("name", list(MINMAX_REFUSALS))
def test_sog_means_minmax_refuses(name, gsx_lib):
    kw, rc, text = MINMAX_REFUSALS[name]
    a = dict(rows=NULL, n=10, F=F, cols=XYZ, ws=FAKE, ws_bytes=MINMAX_WS, mm=FAKE)
    a.update(kw)
    got = gsx_lib.gsx_sog_means_minmax(a["rows"], a["n"], a["F"], i32s(a["cols"]), a["ws"], a["ws_bytes"], a["mm"],
                                       None)
    assert _refuse(gsx_lib, got, text) == rc


TEXTURE_REFUSALS = {
    "n_negative": (dict(n=-1), "out of range"),
    "n_2_pow_31": (dict(n=1 << 31, pixels=1 << 31), "out of range"),
    "row_width": (dict(F=0), "bad row width"),
    "pixels_below_n": (dict(pixels=9), "pixels < n"),
    "column": (dict(col=F), "column 19 out of range"),
    "unaligned": (dict(rows=FAKE, out=ODD), "null or unaligned device pointer"),
    "null_rows": (dict(rows=NULL), "null or unaligned device pointer"),
}


def _texture_call(gsx_lib, which, a):
    cols = {"means": XYZ, "quats": ROT, "scales_sh0": C7}[which]
    cols = i32s(cols[:-1] + [a["col"]]) if "col" in a else i32s(cols)
    if which == "means":
        return gsx_lib.gsx_sog_means(a["rows"], a["n"], a["F"], a["order"], cols, FAKE, a["pixels"], a["out"], FAKE,
                                     None)
    if which == "quats":
        return gsx_lib.gsx_sog_quats(a["rows"], a["n"], a["F"], a["order"], cols, a["pixels"], a["out"], None)
    return gsx_lib.gsx_sog_scales_sh0(a["rows"], a["n"], a["F"], a["order"], cols, FAKE, a["ms"], FAKE, a["mc"],
                                      a["pixels"], FAKE, a["out"], None)


@pytest.mark.parametrize("name", list(TEXTURE_REFUSALS))
@pytest.mark.parametrize("which", ["means", "quats", "scales_sh0"])
def test_sog_texture_entry_points_refuse(which, name, gsx_lib):
    """Each refusal comes from a host-side check before any CUDA call.  rows is NULL unless a case needs it set, so a
    check that wrongly passed would still end in the null-pointer refusal, never in a launch; the other pointers are
    aligned fakes that are never dereferenced, or the unaligned one the check is for."""
    kw, text = TEXTURE_REFUSALS[name]
    a = dict(rows=NULL, n=10, F=F, order=FAKE, pixels=16, out=FAKE, ms=256, mc=1)
    a.update(kw)
    assert _refuse(gsx_lib, _texture_call(gsx_lib, which, a), text) == ARG


@pytest.mark.parametrize("ms,mc", [(0, 1), (1, 0), (257, 256), (256, 257)])
def test_sog_scales_sh0_refuses_codebook_sizes(ms, mc, gsx_lib):
    a = dict(rows=NULL, n=10, F=F, order=NULL, pixels=16, out=NULL, ms=ms, mc=mc)
    assert _refuse(gsx_lib, _texture_call(gsx_lib, "scales_sh0", a), "codebook sizes") == ARG


GATHER_REFUSALS = {
    "n_negative": (dict(n=-1), "out of range"),
    "n_2_pow_31": (dict(n=1 << 31), "out of range"),
    "row_width": (dict(F=0), "bad row width"),
    "m_negative": (dict(m=-1), "m=-1 out of range"),
    "m_past_the_columns": (dict(m=31), "m=31 out of range"),
    "no_columns": (dict(ncols=0, sel=FAKE), "0 columns"),
    "46_columns": (dict(ncols=46), "46 columns"),
    "column": (dict(col=F), "column 19 out of range"),
    "null_rows": (dict(rows=NULL), "null device pointer"),
    "n_zero_with_sel": (dict(rows=FAKE, n=0, sel=FAKE), "null device pointer or n = 0"),
}


@pytest.mark.parametrize("name", list(GATHER_REFUSALS))
def test_sog_gather_values_refuses(name, gsx_lib):
    kw, text = GATHER_REFUSALS[name]
    a = dict(rows=NULL, n=10, F=F, order=FAKE, ncols=3, sel=NULL, m=30, out=FAKE)
    a.update(kw)
    cols = [1, 2, a.get("col", 3)] + [4] * max(a["ncols"] - 3, 0)
    got = gsx_lib.gsx_sog_gather_values(a["rows"], a["n"], a["F"], a["order"], i32s(cols), a["ncols"], a["sel"], a["m"],
                                        a["out"], None)
    assert _refuse(gsx_lib, got, text) == ARG
