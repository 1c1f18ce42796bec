"""The radix sort, the multi-level scan, the Morton order and the chunk bounds, path by path.

Each case has a seeded builder.  An unmarked CPU test restates the dispatch (radix form, passes, tiles, scan levels,
the Morton level schedule) and checks in NumPy that the case reaches the branch it is named after.  A `gpu` test
compares the device with NumPy exactly: np.argsort(kind="stable") for csrc/gsx_radix.cu, a restatement of
formats/compressed_ply.py:252-297 for csrc/gsx_morton.cu (order, depth, refusal) and np.minimum/maximum.reduceat for
k_chunk_minmax."""
import numpy as np
import pytest

TILE = 4096          # kRsTile: keys per radix tile
SCAN_BLOCK = 2048    # kScanBlock: elements per scan CTA
ONESWEEP_MAX = 1 << 30


# ---------------------------------------------------------------------------------------------------- restatements
def radix_dispatch(n, b0, b1):
    """radix_sort_pairs: the form, the number of 8-bit passes and of 4096-key tiles."""
    return {"form": "onesweep" if n < ONESWEEP_MAX else "three_kernel", "passes": (b1 - b0 + 7) // 8,
            "tiles": -(-n // TILE)}


def scan_levels(m):
    """exclusive_scan_u32 on m elements: block scans on the way down, one per level."""
    levels = 1
    while m > SCAN_BLOCK:
        m = -(-m // SCAN_BLOCK)
        levels += 1
    return levels


def field_of(keys, b0, b1):
    w = b1 - b0
    mask = np.uint64((1 << w) - 1) if w < 64 else np.uint64(0xFFFFFFFFFFFFFFFF)
    return (keys >> np.uint64(b0)) & mask


def _p12(n):
    n = n & 0x000003ff
    n = (n ^ (n << 16)) & 0xff0000ff
    n = (n ^ (n << 8)) & 0x0300f00f
    n = (n ^ (n << 4)) & 0x030c30c3
    n = (n ^ (n << 2)) & 0x09249249
    return n


def morton_ref(xyz, limit=256):
    """compressed_ply.py:252-297 with a stable argsort, as (order, schedule).  schedule[d] lists (position, length) of
    the runs the recursion enters at depth d, in position order: the device's level d.  A run that comes back as one
    run (not flat) would recurse into the same rows for ever; that raises RecursionError here at once."""
    x, y, z = xyz[:, 0], xyz[:, 1], xyz[:, 2]
    idxs = np.arange(len(xyz), dtype=np.int64)
    schedule = []
    morton_ref.groups = []        # lengths of the runs of equal codes at depth 0
    stack = [(0, len(idxs), 0)] if len(idxs) > 1 else []
    while stack:
        b, e, d = stack.pop()
        while len(schedule) <= d:
            schedule.append([])
        schedule[d].append((b, e - b))
        ix = idxs[b:e]
        cx, cy, cz = x[ix], y[ix], z[ix]
        with np.errstate(all="ignore"):
            mx, Mx, my, My, mz, Mz = cx.min(), cx.max(), cy.min(), cy.max(), cz.min(), cz.max()
            xl, yl, zl = Mx - mx, My - my, Mz - mz
            if xl == 0 and yl == 0 and zl == 0:
                continue
            xm = 1024.0 / xl if xl > 0 else 0
            ym = 1024.0 / yl if yl > 0 else 0
            zm = 1024.0 / zl if zl > 0 else 0
            qx = np.clip((cx - mx) * xm, 0, 1023).astype(np.uint32)
            qy = np.clip((cy - my) * ym, 0, 1023).astype(np.uint32)
            qz = np.clip((cz - mz) * zm, 0, 1023).astype(np.uint32)
        codes = (_p12(qz) << 2) | (_p12(qy) << 1) | _p12(qx)
        o = np.argsort(codes, kind="stable")
        idxs[b:e] = ix[o]
        sc = codes[o]
        cut = np.flatnonzero(sc[1:] != sc[:-1]) + 1
        starts, ends = np.r_[0, cut], np.r_[cut, e - b]
        if d == 0:
            morton_ref.groups = list(ends - starts)
        if len(starts) == 1 and e - b > limit:
            raise RecursionError(f"run of {e - b} rows at depth {d} does not split")
        for s, t in zip(starts[::-1], ends[::-1]):
            if t - s > limit:
                stack.append((b + s, b + t, d + 1))
    for lv in schedule:
        lv.sort()
    return idxs, schedule


def seg_bits(nseg):
    b = 1
    while (1 << b) < nseg:
        b += 1
    return b


def level_warps(runs):
    """(uniform, mixed) warp counts of k_mo_bounds at a level with these runs (32 consecutive active elements)."""
    lens = [ln for _, ln in runs]
    off = np.r_[0, np.cumsum(lens)]
    m = int(off[-1])
    seg = np.searchsorted(off, np.arange(m), side="right") - 1
    nw = -(-m // 32)
    uni = sum(1 for w in range(nw) if (w + 1) * 32 <= m and seg[w * 32] == seg[w * 32 + 31])
    return uni, nw - uni


# ---------------------------------------------------------------------------------------------------- radix builders
RADIX_BITS = [(0, 1), (0, 7), (0, 8), (0, 9), (0, 30), (0, 32), (0, 48), (0, 64), (3, 61), (13, 22)]
RADIX_N = [511, 512, 513, 4095, 4096, 4097, 8193]
RADIX_KINDS = ["ties", "top_bit", "all_digits", "one_digit", "descending"]


def radix_keys(n, b0, b1, kind, seed=0):
    """uint64 keys.  ties: few distinct fields, random bits outside [b0, b1); top_bit: bit 63 set on half the keys
    (a field that reaches bit 63 sees it); all_digits: every 4096-key tile holds all 256 values of the first digit;
    one_digit: the first digit is the same everywhere; descending: the fields in strictly falling order where the
    width allows."""
    rng = np.random.default_rng(seed * 1_000_003 + n * 97 + b0 * 7 + b1)
    noise = rng.integers(0, 1 << 63, n, dtype=np.uint64) | (rng.integers(0, 2, n, dtype=np.uint64) << np.uint64(63))
    w = b1 - b0
    fmask = np.uint64((1 << w) - 1) if w < 64 else np.uint64(0xFFFFFFFFFFFFFFFF)
    if kind == "ties":
        f = rng.integers(0, min(1 << min(w, 62), 37), n, dtype=np.uint64)
        f = (f * np.uint64(0x9E3779B97F4A7C15)) & fmask if w > 6 else f & fmask
    elif kind == "top_bit":
        f = rng.integers(0, 1 << 62, n, dtype=np.uint64) | (rng.integers(0, 2, n, dtype=np.uint64) << np.uint64(63))
        f >>= np.uint64(b0)
        f &= fmask
    elif kind == "all_digits":
        f = rng.integers(0, 1 << min(w, 62), n, dtype=np.uint64) & ~np.uint64(0xFF) & fmask
        f |= (np.arange(n, dtype=np.uint64) * np.uint64(151)) % np.uint64(min(256, 1 << min(w, 8)))
    elif kind == "one_digit":
        f = rng.integers(0, 1 << min(w, 62), n, dtype=np.uint64) & ~np.uint64(0xFF) & fmask
        f |= np.uint64(0xA5) & fmask
    elif kind == "descending":
        f = (np.uint64(n) - np.arange(n, dtype=np.uint64)) & fmask
    else:
        raise ValueError(kind)
    outside = noise & ~(fmask << np.uint64(b0)) if w < 64 else np.zeros(n, np.uint64)
    return (f << np.uint64(b0)) | outside


@pytest.mark.parametrize("bits", RADIX_BITS)
@pytest.mark.parametrize("n", RADIX_N)
def test_radix_case_reaches_its_path(n, bits):
    b0, b1 = bits
    d = radix_dispatch(n, b0, b1)
    assert d["form"] == "onesweep" and d["passes"] == (b1 - b0 + 7) // 8
    assert d["tiles"] == {511: 1, 512: 1, 513: 1, 4095: 1, 4096: 1, 4097: 2, 8193: 3}[n]
    assert (n % TILE == 0) == (n == 4096) and (n % 512 == 0) == (n in (512, 4096))
    for kind in RADIX_KINDS:
        k = radix_keys(n, b0, b1, kind)
        f = field_of(k, b0, b1)
        first = (f & np.uint64(0xFF)).astype(np.int64)
        if kind == "ties":
            assert len(np.unique(f)) < n // 4                       # stability is visible
        if kind == "top_bit" and b1 == 64:
            assert (k >> np.uint64(63)).any() and not (k >> np.uint64(63)).all()
        if kind == "all_digits" and b1 - b0 >= 8 and n >= 256:
            assert len(np.unique(first[:min(n, TILE)])) == 256
        if kind == "one_digit":
            assert len(np.unique(first)) == 1
        if kind == "descending" and (b1 - b0) >= 14:
            assert (np.diff(f.astype(np.float64)) < 0).all()
        if b0 > 0 or b1 < 64:                                       # bits outside the range are not all zero
            outside = k & ~(np.uint64((1 << (b1 - b0)) - 1) << np.uint64(b0)) if b1 - b0 < 64 else np.uint64(0)
            assert np.any(outside)


def _to_torch_u64(keys, dev):
    import torch
    return torch.from_numpy(keys.view(np.int64).copy()).to(dev)


@pytest.mark.gpu
@pytest.mark.parametrize("kind", RADIX_KINDS)
@pytest.mark.parametrize("bits", RADIX_BITS)
@pytest.mark.parametrize("n", RADIX_N)
def test_radix_onesweep_pairs_and_keys(n, bits, kind, cuda, gsx_lib):
    """Pairs and bare words through the raw ABI, the workspace exactly gsx_sort_pairs_workspace_bytes(n) (one byte
    less is refused), against np.argsort(kind="stable") of the field, compared as uint64."""
    import torch
    from gsx import _abi
    from gsx._abi import _ptr, _stream
    b0, b1 = bits
    keys = radix_keys(n, b0, b1, kind)
    want = np.argsort(field_of(keys, b0, b1), kind="stable")
    need = int(_abi.lib.gsx_sort_pairs_workspace_bytes(n))
    for pairs in (True, False):
        k = _to_torch_u64(keys, cuda)
        v = torch.arange(n, dtype=torch.int32, device=cuda) if pairs else None
        small = torch.empty(need - 1, dtype=torch.uint8, device=cuda)
        assert _abi.lib.gsx_sort_pairs(_ptr(k), _ptr(v), n, b0, b1, _ptr(small), need - 1, _stream()) != 0
        ws = torch.empty(need, dtype=torch.uint8, device=cuda)
        assert _abi.lib.gsx_sort_pairs(_ptr(k), _ptr(v), n, b0, b1, _ptr(ws), need, _stream()) == 0
        got_k = k.cpu().numpy().view(np.uint64)
        assert np.array_equal(got_k, keys[want]), f"pairs={pairs}: keys differ"
        if pairs:
            assert np.array_equal(v.cpu().numpy(), want.astype(np.int32))


# ---------------------------------------------------------------------------------------------------- three-kernel
BIG_N = (1 << 30) + 4097
BIG_BYTES = BIG_N * (8 + 4) * 2 + (1 << 30)


def test_three_kernel_case_reaches_its_path():
    d = radix_dispatch(BIG_N, 0, 16)
    assert d["form"] == "three_kernel" and d["passes"] == 2 and d["tiles"] == (1 << 18) + 2
    hist = 256 * d["tiles"]
    assert scan_levels(hist) == 3                 # the digit-major matrix needs the third scan level
    assert BIG_BYTES < 40 << 30


def _big_keys(i):
    """key of element i: i above bit 16, a scrambled 16-bit field below (ties every 65 536 elements)"""
    return (i << 16) | ((i * 40503) & 0xFFFF)


@pytest.mark.gpu
def test_radix_three_kernel_two_passes(cuda, gsx_lib):
    """n = 2^30 + 4097 (the three-kernel form, its scan at three levels), bits [0, 16).  Checked on the device: the
    field is non-decreasing, vals rise within equal fields, vals is a permutation and every key moved with its val."""
    import torch
    from gsx import sor
    free, _ = torch.cuda.mem_get_info()
    if free < 40 << 30:
        pytest.skip(f"needs 40 GiB of free device memory, {free / 2**30:.1f} GiB free")
    n, step = BIG_N, 1 << 27
    keys = torch.empty(n, dtype=torch.int64, device=cuda)
    for s in range(0, n, step):
        i = torch.arange(s, min(s + step, n), dtype=torch.int64, device=cuda)
        keys[s:s + len(i)] = _big_keys(i)
    vals = torch.arange(n, dtype=torch.int32, device=cuda)
    sor.sort_pairs(keys, vals, 0, 16)
    seen = torch.zeros(n, dtype=torch.uint8, device=cuda)
    for s in range(0, n, step):
        e = min(s + step + 1, n)
        f = keys[s:e] & 0xFFFF
        v = vals[s:e].long()
        assert bool((f[1:] >= f[:-1]).all()), f"field falls in [{s}, {e})"
        same = f[1:] == f[:-1]
        assert bool((v[1:][same] > v[:-1][same]).all()), f"unstable in [{s}, {e})"
        assert torch.equal(keys[s:e], _big_keys(v)), f"a key did not move with its value in [{s}, {e})"
        seen[v] = 1
    assert int(seen.sum(dtype=torch.int64)) == n


# ---------------------------------------------------------------------------------------------------- Morton builders
def _background(n, seed):
    """uniform rows in the box [-10, 10]^3, its two corners included: a level-0 cell is 20/1024 wide"""
    b = np.random.default_rng(seed).uniform(-10, 10, (n, 3)).astype(np.float32)
    b[0], b[1] = -10.0, 10.0
    return b


def _blob(center, cnt, sigma, seed):
    """cnt rows within sigma of the centre of the level-0 cell that holds `center`"""
    rng = np.random.default_rng(seed)
    c = (np.floor((np.asarray(center, np.float64) + 10) * 51.2) + 0.5) / 51.2 - 10
    return (c.astype(np.float32) + rng.uniform(-sigma, sigma, (cnt, 3))).astype(np.float32)


def morton_case(name):
    """float32 [N, 3] clouds, each aimed at one path of gsx_morton_order."""
    if name.startswith("run_"):                         # one cell of exactly 256 / 257 rows
        cnt = int(name[4:])
        return np.r_[_background(3000, 1), _blob((1.0, 2.0, 3.0), cnt, 1e-4, 2)]
    if name == "mid_warp":                              # level-1 runs of 300 and 290 rows: the second starts mid-warp
        return np.r_[_background(2000, 3), _blob((-5, 5, 1), 300, 1e-4, 4), _blob((5, -5, -1), 290, 1e-4, 5)]
    if name.startswith("nseg_"):                        # nseg level-1 runs
        k = int(name[5:])
        rng = np.random.default_rng(k)
        parts = [_background(1500, 6)]
        for j in range(k):
            parts.append(_blob(rng.uniform(-9, 9, 3), 260 + 7 * j, 1e-4, 100 + j))
        return np.concatenate(parts)
    if name == "dead_next_to_live":                     # a cell of 300 identical rows beside a cell of 300 distinct rows
        return np.r_[_background(1000, 7), _blob((3.0, 3.0, 3.0), 300, 0.0, 8), _blob((3.0, 3.0, 3.03), 300, 1e-4, 8)]
    if name == "ladder":                                # 22 groups of 300 rows at x = 2^(100 - 11 j)
        x = np.repeat(np.float32(2.0) ** (100 - 11 * np.arange(22, dtype=np.float32)), 300)
        return np.c_[x, np.zeros_like(x), np.zeros_like(x)].astype(np.float32)
    if name == "subnormal":                             # 300 distinct rows 2^-149 apart inside a normal cloud
        sub = np.arange(300, dtype=np.uint32).view(np.float32)
        return np.r_[_background(3000, 9), np.c_[sub, np.zeros(300), np.zeros(300)].astype(np.float32)]
    raise ValueError(name)


MORTON_CASES = ["run_256", "run_257", "mid_warp", "nseg_2", "nseg_3", "nseg_4", "nseg_5", "nseg_17",
                "dead_next_to_live", "ladder", "subnormal"]


def nonfinite_case(name):
    """Clouds with NaN (both signs) and +-inf rows; those ending in _refused are the ones the reference never ends."""
    base = _background(5000, 11)
    neg_nan = np.uint32(0xFFC00000).view(np.float32)
    if name == "nan_full_warp":
        base[40, 0] = np.nan
    elif name == "neg_nan_tail_warp":
        base[4999, 1] = neg_nan
    elif name == "inf_full_warp":
        base[70, 2] = np.inf
    elif name == "neg_inf_tail_warp":
        base[4995, 0] = -np.inf
    elif name == "nan_in_level1_run":
        blob = _blob((1.0, 1.0, 1.0), 300, 1e-4, 12)
        blob[150, 2] = neg_nan
        blob[17, 2] = np.nan
        base = np.r_[base, blob]
    elif name == "inf_and_nan_mixed":
        base[5, 0], base[6, 0], base[7, 1], base[4990, 1] = np.inf, -np.inf, np.nan, neg_nan
    elif name == "nan_extent_refused":
        base = np.c_[np.full(300, np.nan), np.ones(300), np.ones(300)].astype(np.float32)
    elif name == "inf_extent_refused":
        base = np.c_[np.tile([np.inf, -np.inf, 1.0], 100), np.ones(300), np.ones(300)].astype(np.float32)
    elif name == "inf_cell_refused":
        base = np.r_[base[:1000], np.tile(np.float32([[np.inf, 0, 0]]), (300, 1))]
    else:
        raise ValueError(name)
    return np.ascontiguousarray(base, dtype=np.float32)


NONFINITE_CASES = ["nan_full_warp", "neg_nan_tail_warp", "inf_full_warp", "neg_inf_tail_warp", "nan_in_level1_run",
                   "inf_and_nan_mixed", "nan_extent_refused", "inf_extent_refused", "inf_cell_refused"]

SCAN_N = [2047, 2048, 4_194_303, 4_194_304, 4_194_305]


@pytest.mark.parametrize("name", MORTON_CASES)
def test_morton_case_reaches_its_path(name):
    xyz = morton_case(name)
    _, sched = morton_ref(xyz)
    depth = len(sched) - 1
    lv1 = sched[1] if depth >= 1 else []
    if name == "run_256":                               # the blob is one run of 256 at level 0, not entered
        assert depth == 0 and max(morton_ref.groups) == 256
    elif name == "run_257":
        assert lv1 == [(lv1[0][0], 257)]
    elif name == "mid_warp":
        assert sorted(ln for _, ln in lv1) == [290, 300]
        uni, mixed = level_warps(lv1)
        assert uni > 0 and mixed > 0 and lv1[0][1] % 32 != 0     # the second run starts mid-warp
    elif name.startswith("nseg_"):
        k = int(name[5:])
        assert len(lv1) == k and seg_bits(k) == {2: 1, 3: 2, 4: 2, 5: 3, 17: 5}[k]
    elif name == "dead_next_to_live":
        assert [ln for _, ln in lv1] == [300, 300] and depth == 1   # both entered; neither has a run > 256 below
    elif name == "ladder":
        assert depth == 21
    elif name == "subnormal":
        assert depth > 16
    assert depth < 16 or name in ("ladder", "subnormal")


@pytest.mark.parametrize("name", NONFINITE_CASES)
def test_nonfinite_case_reaches_its_path(name):
    xyz = nonfinite_case(name)
    bad = ~np.isfinite(xyz)
    assert bad.any()
    rows = np.flatnonzero(bad.any(axis=1))
    if name.endswith("_refused"):
        with pytest.raises(RecursionError):
            morton_ref(xyz)
        return
    _, sched = morton_ref(xyz)
    if "full_warp" in name:
        assert all(r // 32 < len(xyz) // 32 for r in rows)      # inside a warp of 32 active rows at level 0
    if "tail_warp" in name:
        assert all(r >= len(xyz) // 32 * 32 for r in rows)      # in the last, partial warp at level 0
    if name == "nan_in_level1_run":
        assert len(sched) >= 2
    if np.isnan(xyz).any():                                      # the level-0 box is NaN on that axis: codes 0
        with np.errstate(invalid="ignore"):
            assert np.isnan(xyz.min(axis=0)).any()
    neg = np.isnan(xyz) & (xyz.view(np.uint32) >> 31 == 1)
    if name in ("neg_nan_tail_warp", "nan_in_level1_run", "inf_and_nan_mixed"):
        assert neg.any()


@pytest.mark.parametrize("n", SCAN_N)
def test_scan_case_reaches_its_level(n):
    m1 = n + 1                                          # the level-0 flag scan covers m + 1 = n + 1 elements
    assert scan_levels(m1) == {2047: 1, 2048: 2, 4_194_303: 2, 4_194_304: 3, 4_194_305: 3}[n]
    assert (m1 > SCAN_BLOCK ** 2) == (n >= SCAN_BLOCK ** 2)


def _device_morton(xyz, cuda, limit=256):
    import torch
    from gsx import morton
    got, levels = morton.morton_order(torch.from_numpy(np.ascontiguousarray(xyz)).to(cuda), run_limit=limit,
                                      return_levels=True)
    return got.cpu().numpy().astype(np.int64), levels


@pytest.mark.gpu
@pytest.mark.parametrize("name", MORTON_CASES)
def test_morton_paths_match_reference(name, cuda, gsx_lib):
    xyz = morton_case(name)
    want, sched = morton_ref(xyz)
    got, levels = _device_morton(xyz, cuda)
    assert np.array_equal(got, want)
    assert levels == len(sched)


@pytest.mark.gpu
@pytest.mark.parametrize("name", NONFINITE_CASES)
def test_morton_nonfinite_matches_reference_or_refuses(name, cuda, gsx_lib):
    from gsx._abi import GsxError
    xyz = nonfinite_case(name)
    if name.endswith("_refused"):
        with pytest.raises(GsxError, match="did not split"):
            _device_morton(xyz, cuda)
        return
    want, sched = morton_ref(xyz)
    got, levels = _device_morton(xyz, cuda)
    assert np.array_equal(got, want)
    assert levels == len(sched)


@pytest.mark.gpu
@pytest.mark.parametrize("n", SCAN_N)
def test_morton_flag_scan_levels(n, cuda, gsx_lib):
    """The flag scan of level 0 at m + 1 = 2048, 2049, 2048^2, 2048^2 + 1 and 2048^2 + 2 elements."""
    rng = np.random.default_rng(n)
    xyz = rng.uniform(-1, 1, (n, 3)).astype(np.float32)
    xyz[: n // 3] = np.round(xyz[: n // 3] * 64) / 64           # repeated cells: runs of every length at level 0
    want, sched = morton_ref(xyz)
    got, levels = _device_morton(xyz, cuda)
    assert np.array_equal(got, want)
    assert levels == len(sched)


# ---------------------------------------------------------------------------------------------------- chunk bounds
def minmax_ref(v, starts):
    """np.minimum/maximum.reduceat, with the zero sign made definite: -0.0 for a min and +0.0 for a max of mixed zeros
    (which one np.minimum.reduceat returns depends on the element's position among NumPy's SIMD lanes)."""
    with np.errstate(invalid="ignore"):
        lo, hi = np.minimum.reduceat(v, starts), np.maximum.reduceat(v, starts)
    ends = np.r_[starts[1:], len(v)]
    for c, (s, e) in enumerate(zip(starts, ends)):
        z = v[s:e][v[s:e] == 0]
        if lo[c] == 0 and len(z):
            lo[c] = -0.0 if np.signbit(z).any() else 0.0
        if hi[c] == 0 and len(z):
            hi[c] = 0.0 if (~np.signbit(z)).any() else -0.0
    return lo, hi


CHUNKS = [1, 255, 256, 257, 1000]


def chunk_case(chunk, seed=0):
    """rows [N, 8] with N = 3 chunks + 5: one chunk all NaN, NaN of both signs and +-inf in others, a chunk whose
    min mixes -0.0 and +0.0, and large values the clip range cuts."""
    n = 3 * chunk + 5
    rng = np.random.default_rng(chunk * 10 + seed)
    rows = rng.normal(0, 30, (n, 8)).astype(np.float32)
    order = rng.permutation(n).astype(np.int32)
    at = lambda j: order[j]                                          # row that lands at ordered position j
    rows[[at(j) for j in range(chunk, 2 * chunk)], 1] = np.nan       # chunk 1 of column 1: all NaN (ordered)
    rows[at(0), 2] = np.uint32(0xFFC00000).view(np.float32)
    rows[at(n - 1), 3] = np.nan
    rows[at(min(2, n - 1)), 4], rows[at(n - 2), 4] = np.inf, -np.inf
    zc = [at(j) for j in range(2 * chunk, 3 * chunk)]                # chunk 2 of column 5: zeros of both signs at the min
    rows[zc, 5] = np.abs(rows[zc, 5]) + 1
    rows[zc[0], 5], rows[zc[-1], 5] = 0.0, -0.0
    rows[zc[len(zc) // 2], 6] = 0.0
    return rows, order


@pytest.mark.parametrize("chunk", CHUNKS)
def test_chunk_case_reaches_its_path(chunk):
    rows, order = chunk_case(chunk)
    s = rows[order]
    starts = np.arange(0, len(s), chunk)
    assert len(starts) == -(-len(s) // chunk) and (chunk > 256) == (chunk in (257, 1000))   # rows > threads
    with np.errstate(invalid="ignore"):
        lo = np.minimum.reduceat(s, starts, axis=0)
        clo = np.minimum.reduceat(np.clip(s, -20, 20), starts, axis=0)
    assert np.isnan(lo[1, 1]) and np.isnan(clo[1, 1])                # np.clip keeps the NaN
    assert np.isnan(lo[0, 2]) and np.isnan(lo[-1, 3])
    if chunk > 1:
        assert lo[2, 5] == 0 and np.signbit(s[2 * chunk:3 * chunk, 5][s[2 * chunk:3 * chunk, 5] == 0]).any()
    assert (np.abs(s[np.isfinite(s)]) > 20).any()


def test_numpy_reduceat_zero_sign_depends_on_position():
    """What np.minimum.reduceat gives for mixed zeros depends on where they sit (NumPy 2.3.5, x86): the device does
    not follow it and returns -0.0 (min) / +0.0 (max); the values compare equal either way."""
    signs = set()
    for pos in range(8):
        a = np.full(17, 5.0, np.float32)
        a[pos], a[pos + 1] = -0.0, 0.0
        r = np.minimum.reduceat(a, [0])[0]
        assert r == 0
        signs.add(bool(np.signbit(r)))
    assert signs == {False, True}


@pytest.mark.gpu
@pytest.mark.parametrize("with_order", [True, False])
@pytest.mark.parametrize("chunk", CHUNKS)
def test_chunk_minmax_paths(chunk, with_order, cuda, gsx_lib):
    import torch
    from gsx import morton
    rows, order = chunk_case(chunk)
    s = rows[order] if with_order else rows
    starts = np.arange(0, len(s), chunk)
    rt = torch.from_numpy(rows).to(cuda)
    ot = torch.from_numpy(order).to(cuda) if with_order else None
    for ncol in range(1, 9):
        cols = [(3 * k + ncol) % 8 for k in range(ncol)]            # every column, in a scrambled order
        for clip in (None, (-20.0, 20.0)):
            v = s[:, cols] if clip is None else np.clip(s[:, cols], *clip)
            lo, hi = morton.chunk_minmax(rt, cols, ot, chunk, clip=clip)
            lo, hi = lo.cpu().numpy(), hi.cpu().numpy()
            for j in range(ncol):
                wl, wh = minmax_ref(np.ascontiguousarray(v[:, j]), starts)
                for g, w in ((lo[:, j], wl), (hi[:, j], wh)):
                    assert np.array_equal(np.isnan(g), np.isnan(w)), (ncol, cols[j], clip, g, w)
                    fin = ~np.isnan(w)                               # finite and infinite bounds: bit-exact
                    assert np.array_equal(g[fin].view(np.uint32), w[fin].view(np.uint32)), (ncol, cols[j], clip, g, w)
