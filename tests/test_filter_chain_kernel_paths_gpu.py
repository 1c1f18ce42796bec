"""The kernels every conversion runs between the big filter families, path by path: the NumPy-order mean/std (single
GPU and sharded) and the SOR threshold mask, the bbox and alpha masks, the stream compaction after every filter, and
the device-record gather, column extraction and colour transform.

Every case is a builder (a plain seeded function returning the inputs it runs with) and two kinds of test:
  * an unmarked CPU test restating the dispatch of the host entry point (which kernel, which form, how many launches)
    and asserting that the case reaches its branch, plus the property of the data the case relies on, checked with
    NumPy;
  * a `gpu` test asserting exact equality with a plain NumPy reference: the bits of np.mean / np.std, the keep-masks
    of `oracle`, np.flatnonzero for the compaction, fancy indexing for the gather.  Only the colour alpha channel and
    `scale_exp` keep their documented allowance (expf against NumPy's SIMD exp).

Constants these cases are built around:
  * csrc/gsx_stats.cu: NumPy's pairwise tree splits a node of m > 128 elements at m/2 rounded down to a multiple of 8,
    so its depth depends only on n; a leaf (<= 128 elements) is summed by two lanes with float4 loads
    (`k_pw_leaves2`) when the vector is 16-byte aligned, by eight lanes (`k_pw_leaves`, `leaf_sum8`) otherwise; the
    inner levels dmax-1 .. 10 are combined nine at a time by `k_pw_mid` (one launch each group), levels <= 9 and the
    division by `k_pw_top`.  The sharded form always sums its leaves with `leaf_sum8`.
  * csrc/gsx_stats.cu, csrc/gsx_masks.cu: threshold, bbox and alpha run a 4-wide kernel when the input is 16-byte
    aligned and the mask 4-byte aligned.  The 4-wide threshold kernel also covers the last n % 4 rows; the 4-wide
    bbox and alpha kernels cover n/4 groups and the scalar kernel the rest.  An xyz view at row offset r is 16-byte
    aligned iff r % 4 == 0.
  * csrc/gsx_compact.cu: one pass with decoupled look-back (2 048-row tiles, an 8-byte mask load when the group of 8
    rows is whole and 8-byte aligned, look-back over windows of 32 tiles) below 2^30 rows; count -> scan -> scatter
    over 1 024-row blocks from 2^30 rows on; refused from 2^31 rows on (int32 row indices).
  * csrc/gsx_records.cu: one warp per gathered row, lanes striding over the F floats of the row.
"""
import ctypes as C
import functools

import numpy as np
import pytest

import oracle

F32, U32 = np.float32, np.uint32
FMAX = np.finfo(F32).max
# gsx_stats.cu
LEAF = 128
MID_SPAN = 9                    # k_pw_mid: up to nine levels per launch ...
MID_LOW = 10                    # ... down to level 10; k_pw_top combines levels <= 9
HALO = 128                      # the sharded form's spill-over halo per slab
# gsx_stats.cu / gsx_masks.cu
VEC_ROWS, VEC_IN_ALIGN, VEC_MASK_ALIGN = 4, 16, 4
# gsx_compact.cu
ONEPASS_LIMIT = 1 << 30
TILE, GROUP, WINDOW = 2048, 8, 32
BLOCK2 = 1024
LB_VAL = (1 << 30) - 1
COMPACT_ROW_LIMIT = 1 << 31
GSX_ERR_WORKSPACE, GSX_ERR_UNSUPPORTED = -3, -4
TORCH_ALIGN = 256               # the caching allocator hands out at least 256-byte aligned blocks
SENT8 = 0xA5                    # sentinel byte of the mask buffers
SENT32 = 0x7FA5A5A5             # sentinel word of the float / int32 output buffers (a NaN payload)
SLOW_N = 1 << 26


# ------------------------------------------------------------------------------------------------ dispatch, restated
def _split(m):
    n2 = m // 2
    return n2 - n2 % 8


def pairwise_depth(n):
    """pairwise_depth: levels of NumPy's tree below the root."""
    level, d = {n}, 0
    while True:
        nxt = set()
        for m in level:
            if m > LEAF:
                n2 = _split(m)
                nxt.update((n2, m - n2))
        if not nxt:
            return d
        level, d = nxt, d + 1


def first_n_of_depth(d):
    """The smallest n whose tree has depth d (d >= 1)."""
    return (LEAF << (d - 1)) + 1


def pw_leaves(n):
    """NumPy's leaves as (offset, size, depth)."""
    out, todo = [], [(0, n, 0)]
    while todo:
        off, m, d = todo.pop()
        if m <= LEAF:
            out.append((off, m, d))
        else:
            n2 = _split(m)
            todo += [(off + n2, m - n2, d + 1), (off, n2, d + 1)]
    return sorted(out)


def leaf_of(n, p):
    """(offset, size) of the leaf holding element p."""
    off, m = 0, n
    while m > LEAF:
        n2 = _split(m)
        if p < off + n2:
            m = n2
        else:
            off, m = off + n2, m - n2
    return off, m


def leaf_kernel(byte_addr):
    return "k_pw_leaves2" if byte_addr % 16 == 0 else "k_pw_leaves"


def mid_launches(dmax):
    """pairwise_mid_levels: the (dhi, dlo) of every k_pw_mid launch, and the level k_pw_top starts from."""
    out, d = [], dmax - 1
    while d > MID_LOW - 1:
        dlo = max(d - (MID_SPAN - 1), MID_LOW)
        out.append((d, dlo))
        d = dlo - 1
    return out, d


def vec_split(n, in_addr, mask_addr):
    """(rows of the 4-wide kernel, rows of the scalar kernel) of bbox_mask / alpha_mask."""
    n4 = n // VEC_ROWS if in_addr % VEC_IN_ALIGN == 0 and mask_addr % VEC_MASK_ALIGN == 0 else 0
    return VEC_ROWS * n4, n - VEC_ROWS * n4


def threshold_form(in_addr, mask_addr):
    return "vector" if in_addr % VEC_IN_ALIGN == 0 and mask_addr % VEC_MASK_ALIGN == 0 else "scalar"


def compact_form(n):
    if n >= COMPACT_ROW_LIMIT:
        return "refused"
    return "onepass" if n < ONEPASS_LIMIT else "twopass"


def mask_groups(n, mask_addr):
    """k_cmp_onepass: (groups of 8 rows read with one 8-byte load, groups read byte by byte)."""
    vec = sum(1 for i0 in range(0, n, GROUP) if i0 + GROUP <= n and (mask_addr + i0) % 8 == 0)
    return vec, -(-n // GROUP) - vec


def lookback_windows(tile):
    """Windows of 32 predecessors tile `tile` reads when none of them has published its inclusive prefix yet."""
    return -(-tile // WINDOW)


# ------------------------------------------------------------------------------------------------ references
def same_bits(got, want):
    """Equal bits, NaN == NaN: the device writes the canonical NaN, x86 NumPy keeps the payload of the NaN it met."""
    got, want = np.asarray(got, F32), np.asarray(want, F32)
    return bool(np.all((np.isnan(got) & np.isnan(want)) | (got.view(U32) == want.view(U32))))


def np_mean_std(a):
    with np.errstate(all="ignore"):
        return np.array([np.mean(a), np.std(a)], F32)


def ref_threshold(a, mean, std, tf):
    """gpu_ops.py:259-263 in NumPy 2: mean + tf * std in float32 (tf a weak Python float), then a < thresh."""
    with np.errstate(all="ignore"):
        thresh = F32(mean) + F32(tf) * F32(std)
        return a < thresh, thresh


def ref_bbox(xyz, bounds):
    with np.errstate(over="ignore"):   # a bound past FLT_MAX becomes inf, as in gsx.masks
        return oracle.bbox_mask(xyz[:, 0], xyz[:, 1], xyz[:, 2], *bounds)


def ref_colour(f, scale):
    """splat.py:131-133 / spz.py:131: clip((0.5 + scale * f) * 255, 0, 255).astype(uint8) in float32.  NumPy keeps NaN
    through np.clip and the NaN -> uint8 cast is undefined; the device clamps NaN to 0, which is what the reference
    gives on x86."""
    with np.errstate(invalid="ignore"):
        prod = (F32(0.5) + F32(scale) * f) * F32(255)
        out = np.clip(prod, 0, 255).astype(np.uint8)
    out[np.isnan(prod)] = 0
    return out


# ------------------------------------------------------------------------------------------------ builders
def order_sensitive(n, seed):
    """Mixed signs, magnitudes 1e-3 .. 1e7, the values above 1e2 in pairs that cancel: the sum is far smaller than
    its terms, so every summation order gives other bits."""
    rng = np.random.default_rng(seed)
    e = rng.random(n, dtype=F32)
    mag = np.power(F32(10), e * F32(10) - F32(3))
    a = np.where(rng.random(n, dtype=F32) < 0.5, -mag, mag).astype(F32)
    big = np.flatnonzero(e >= F32(0.5))
    h = len(big) // 2
    a[big[h: 2 * h]] = -a[big[:h]]
    return a[rng.permutation(n)]


SWEEP_N = 1100
BOUNDARY_NS = sorted({x for d in range(1, 23) for x in (first_n_of_depth(d) - 1, first_n_of_depth(d))})
DIV_N = (1 << 24) + 5


def nonfinite_cases():
    """(name, vector): NaN / +inf / -inf at the first, middle and last element, and +inf with -inf."""
    out = []
    for n in (1, 7, 8, 129, 1000, 100_003):
        base = order_sensitive(n, n)
        for where in sorted({0, n // 2, n - 1}):
            for v in (np.nan, np.inf, -np.inf):
                a = base.copy()
                a[where] = v
                out.append((f"{n}-{where}-{v}", a))
        if n > 1:
            a = base.copy()
            a[0], a[-1] = np.inf, -np.inf
            out.append((f"{n}-both-inf", a))
    return out


def overflow_vector(n, seed, signs):
    """Magnitudes in [FLT_MAX / 4, FLT_MAX]: sums of two or more overflow inside the tree."""
    rng = np.random.default_rng(seed)
    a = (FMAX * (0.25 + 0.75 * rng.random(n))).astype(F32)
    if signs == "mixed":
        a[rng.random(n) < 0.5] *= F32(-1)
    return a


def subnormal_vector(n, seed, kind):
    """'sub': subnormal values of both signs (their sums stay subnormal or cross into the normals); 'sq': values of
    1e-20 .. 1e-19 whose squared deviations in the std pass are subnormal."""
    rng = np.random.default_rng(seed)
    if kind == "sub":
        bits = rng.integers(1, 0x00800000, n, dtype=np.uint32)
        bits[rng.random(n) < 0.5] |= np.uint32(0x80000000)
        return bits.view(F32)
    return (1e-20 + 9e-20 * rng.random(n)).astype(F32)


def sharded_world8():
    """World 8 with slab sizes 0..20 such that some leaf spills over three or more slabs."""
    rng = np.random.default_rng(8)
    out = [(20,) * 8, (0, 20, 0, 20, 0, 20, 0, 20), (1, 1, 1, 1, 1, 1, 1, 1), (0, 0, 0, 0, 0, 7, 20, 1)]
    while len(out) < 16:
        s = tuple(int(v) for v in rng.integers(0, 21, 8))
        if sum(s) and max_slabs_per_leaf(s) >= 3:
            out.append(s)
    return out


def max_slabs_per_leaf(sizes):
    bases = np.concatenate([[0], np.cumsum(sizes)])
    n = int(bases[-1])
    best = 0
    for off, m, _ in pw_leaves(n):
        first = np.searchsorted(bases, off, side="right") - 1
        last = np.searchsorted(bases, off + m - 1, side="right") - 1
        best = max(best, int(last - first + 1))
    return best


SHARD_EDGE = [(0, 300, 500), (400, 129, 0), (0, 1000, 0), (0, 0, 257, 0), (0, 4097), (4097, 0)]
CUTS = list(range(1, LEAF))
SHARD_SLOW = (22_369_621, 22_369_622, 22_369_622)


def threshold_stats():
    """(name, mean, std, tf): ordinary, tf = 0 / negative / not float32-representable, and non-finite statistics."""
    return [("plain", 1.5, 0.25, 2.0), ("tf0", 1.5, 0.25, 0.0), ("tfneg", 0.75, 0.5, -1.25), ("tf01", 2.0, 3.0, 0.1),
            ("mean_nan", np.nan, 0.5, 1.0), ("std_nan", 1.0, np.nan, 1.0), ("mean_inf", np.inf, 0.5, 1.0),
            ("mean_ninf", -np.inf, 0.5, 1.0), ("std_inf", 1.0, np.inf, 2.0), ("std_inf_tf0", 1.0, np.inf, 0.0),
            ("std_inf_tfneg", 1.0, np.inf, -1.0)]


def threshold_values(mean, std, tf, seed):
    """thresh and one ulp either side, signed zeros, the extremes, and random values around thresh: 4 * 16 + 3."""
    _, t = ref_threshold(np.zeros(1, F32), mean, std, tf)
    rng = np.random.default_rng(seed)
    fixed = [t, np.nextafter(t, F32(-np.inf)), np.nextafter(t, F32(np.inf)), 0.0, -0.0, FMAX, -FMAX, np.inf, -np.inf,
             np.nan]
    centre = t if np.isfinite(t) else F32(1.0)
    rest = centre + rng.normal(0, 1, 67 - len(fixed))
    a = np.r_[np.array(fixed, F32), rest.astype(F32)]
    return rng.permutation(a).astype(F32)


BBOX_CASES = ("lanes_on_bounds", "unrepresentable", "signed_zero", "nonfinite_inf_bounds", "nonfinite_finite_bounds",
              "lo_gt_hi", "overflow_bound")


def bbox_case(name):
    """(xyz float32 [4k + 3, 3], six Python-float bounds lo_x, lo_y, lo_z, hi_x, hi_y, hi_z)."""
    rng = np.random.default_rng(BBOX_CASES.index(name) + 40)
    inf = float("inf")
    if name == "lanes_on_bounds":
        bounds = (-1.0, -2.0, -4.0, 1.0, 2.0, 4.0)
        rows = []
        for b in range(6):                  # each bound ...
            ax, lower = b % 3, b < 3
            on = F32(bounds[b])
            out = np.nextafter(on, F32(-inf if lower else inf))
            for lane in range(4):           # ... on each lane of the uchar4, exactly on it and one ulp outside
                for v in (on, out):
                    g = np.full((4, 3), 0.5, F32)
                    g[lane, ax] = v
                    rows.append(g)
        xyz = np.concatenate(rows + [np.full((3, 3), 0.5, F32)])
    elif name == "unrepresentable":
        bounds = (0.1, -0.7, 1e-3, 0.3, -0.1, 0.2)
        inner = np.array([0.2, -0.4, 0.1], F32)
        rows = []
        for b in range(6):
            c = F32(bounds[b])
            for v in (np.nextafter(c, F32(-inf)), c, np.nextafter(c, F32(inf))):
                r = inner.copy()
                r[b % 3] = v
                rows.append(r)
        xyz = np.array(rows + [inner] * 5, F32)
    elif name == "signed_zero":
        bounds = (-0.0, 0.0, -0.0, 0.0, -0.0, -0.0)
        rows = [[sx * 0.0, sy * 0.0, sz * 0.0] for sx in (1, -1) for sy in (1, -1) for sz in (1, -1)]
        for ax in range(3):
            for v in (1e-45, -1e-45):
                r = [0.0, -0.0, 0.0]
                r[ax] = v
                rows.append(r)
        xyz = np.array(rows + [[-0.0, 0.0, -0.0]] * 9, F32)
    elif name in ("nonfinite_inf_bounds", "nonfinite_finite_bounds"):
        bounds = (-inf, -inf, -inf, inf, inf, inf) if name == "nonfinite_inf_bounds" else (-1.0, -1.0, -1.0, 1.0, 1.0, 1.0)
        rows = []
        for ax in range(3):
            for v in (np.nan, inf, -inf, FMAX, -FMAX):
                r = [0.25, -0.25, 0.5]
                r[ax] = v
                rows.append(r)
        rows += [[inf, inf, inf], [-inf, -inf, -inf], [np.nan] * 3, [0.0, 0.0, 0.0]]
        xyz = np.array(rows + [[0.5, 0.5, 0.5]] * 16, F32)
    elif name == "lo_gt_hi":
        bounds = (1.0, 1.0, 1.0, -1.0, -1.0, -1.0)
        xyz = np.r_[rng.uniform(-2, 2, (40, 3)), [[1, 1, 1], [-1, -1, -1], [0, 0, 0]]].astype(F32)
    elif name == "overflow_bound":
        bounds = (-1e39, -2.0, -1e39, 1e39, 2.0, 3.5e38)
        rows = []
        for ax in (0, 2):
            for v in (FMAX, -FMAX, inf, -inf, np.nan):
                r = [0.0, 0.0, 0.0]
                r[ax] = v
                rows.append(r)
        rows += [[0.0, 2.0, 0.0], [0.0, np.nextafter(F32(2.0), F32(3.0)), 0.0], [0.0, -2.0, 0.0]]
        xyz = np.array(rows + [[1.0, 1.0, 1.0]] * 14, F32)
    else:
        raise KeyError(name)
    assert len(xyz) % 4 == 3
    return np.ascontiguousarray(xyz, F32), bounds


ALPHA_LIMITS = list(range(1, 255))
ALPHA_L = 11                      # values per threshold (n % 4 == 3); the tails run n = 11, 10, 9, 8


def alpha_values(u):
    """f32(t) and its two neighbours, NaN, +-inf, signed zeros and random values around t."""
    from gsx import masks
    t = F32(masks.alpha_logit_threshold(u))
    rng = np.random.default_rng(u)
    fixed = [t, np.nextafter(t, F32(-np.inf)), np.nextafter(t, F32(np.inf)), np.nan, np.inf, -np.inf, 0.0, -0.0]
    a = np.r_[np.array(fixed, F32), (t + rng.normal(0, 2, ALPHA_L - len(fixed))).astype(F32)]
    return rng.permutation(a).astype(F32)


ONEPASS_NS = (2047, 2048, 2049, 32 * TILE - 1, 32 * TILE + 1, 33 * TILE + 1)
MASK_KINDS = ("all", "none", "runs", "last_tile_one", "first_tile", "bytes")


def compact_mask(n, kind):
    rng = np.random.default_rng(n * 7 + MASK_KINDS.index(kind))
    m = np.zeros(n, np.uint8)
    if kind == "all":
        m[:] = 1
    elif kind == "runs":                          # alternating kept / dropped runs of 1 .. 700 rows
        i, keep = 0, bool(rng.integers(2))
        while i < n:
            r = int(rng.integers(1, 701))
            m[i: i + r] = keep
            i, keep = i + r, not keep
    elif kind == "last_tile_one":
        last = (n - 1) // TILE * TILE
        m[int(rng.integers(last, n))] = 1
    elif kind == "first_tile":
        k = min(n, TILE)
        m[:k] = rng.random(k) < 0.5
    elif kind == "bytes":                         # every non-zero byte keeps its row
        m[:] = rng.choice(np.array([0, 1, 2, 0x80, 0xFF], np.uint8), n, p=[0.4, 0.15, 0.15, 0.15, 0.15])
    return m


def compact_inputs(n, seed):
    """xyz and opacity as random bit patterns (NaN payloads, subnormals: the copy must keep every bit), and a chained
    int32 row index."""
    rng = np.random.default_rng(seed)
    xyz = rng.integers(0, 1 << 32, (n, 3), dtype=np.uint32).view(F32)
    op = rng.integers(0, 1 << 32, n, dtype=np.uint32).view(F32)
    idx = np.sort(rng.choice(20 * n, n, replace=False)).astype(np.int32)
    return xyz, op, idx


TWOPASS_N = (1 << 30) + 4099


GATHER_FS = (1, 3, 14, 17, 31, 32, 33, 45, 62, 65)
GATHER_MS = (1, 7, 8, 9, 100_003)


def gather_case(F, m):
    """Rows of random bit patterns and a permuted index with repeats."""
    rng = np.random.default_rng(F * 1000 + m)
    R = max(64, m // 3)
    rows = rng.integers(0, 1 << 32, (R, F), dtype=np.uint32).view(F32)
    idx = rng.integers(0, R, m).astype(np.int32)
    if m > 1:
        idx[1] = idx[0]                           # at least one repeat
    return rows, idx


SH_C0 = 0.28209479177387814
COLOUR_SCALES = (SH_C0, 0.15)


def _walk(f, scale, want, steps=64):
    """f32 values next to f whose product (0.5 + scale * f) * 255 in float32 satisfies want(prod)."""
    out = []
    for k in range(-steps, steps + 1):
        v = F32(f)
        for _ in range(abs(k)):
            v = np.nextafter(v, F32(np.inf if k > 0 else -np.inf))
        p = (F32(0.5) + F32(scale) * v) * F32(255)
        if want(p):
            out.append(v)
    return out


def colour_edges(scale):
    """Colour inputs whose float32 product is exactly 255, just above and just below it, exactly 0 and just either
    side of 0, plus -0.0, NaN and +-inf."""
    hi, lo = 0.5 / scale, -0.5 / scale
    vals = (_walk(hi, scale, lambda p: p == 255)[:2] + _walk(hi, scale, lambda p: 255 < p < 255.0001)[:2] +
            _walk(hi, scale, lambda p: 254.9999 < p < 255)[:2] + _walk(lo, scale, lambda p: p == 0)[:2] +
            _walk(lo, scale, lambda p: -1e-4 < p < 0)[:2] + _walk(lo, scale, lambda p: 0 < p < 1e-4)[:2])
    return np.array(vals + [-0.0, 0.0, np.nan, np.inf, -np.inf, 1e30, -1e30], F32)


def colour_rows(scale, n=1003, F=14):
    """Records of F fields: f_dc in columns 9, 2, 11 (the edges on all three), opacity in 5, scales in 0, 7, 13."""
    rng = np.random.default_rng(int(scale * 1000))
    rows = rng.normal(0, 1, (n, F)).astype(F32)
    e = colour_edges(scale)
    for c in (9, 2, 11):
        rows[: len(e), c] = np.roll(e, c)
    rows[:, 5] = rng.normal(0, 4, n).astype(F32)
    return rows


# ------------------------------------------------------------------------------------------------ device calls
def _lib():
    from gsx._abi import lib, check
    from gsx._abi import _ptr, _stream
    return lib, check, _ptr, _stream


def mean_std_exact(buf, off, n, ws=None, out=None):
    """gsx_mean_std_f32 on buf[off: off + n] with a workspace of exactly gsx_mean_std_workspace_bytes(n)."""
    import torch
    lib, check, _ptr, _stream = _lib()
    wsb = lib.gsx_mean_std_workspace_bytes(n)
    if ws is None:
        ws = torch.empty(wsb, dtype=torch.uint8, device=buf.device)
    if out is None:
        out = torch.empty(2, dtype=torch.float32, device=buf.device)
    check(lib.gsx_mean_std_f32(_ptr(buf[off: off + n]), n, _ptr(out), _ptr(ws), wsb, _stream()), "gsx_mean_std_f32")
    return out


def mean_std_at(a, shift, cuda):
    import torch
    buf = torch.empty(len(a) + 4, dtype=torch.float32, device=cuda)
    buf[shift: shift + len(a)].copy_(torch.from_numpy(a))
    got = mean_std_exact(buf, shift, len(a)).cpu().numpy()
    del buf
    return got


def sharded_mean_std(a, sizes, cuda):
    """gsx_pairwise_leaves_dist per emulated rank, the slot all-reduce as a plain sum, then gsx_pairwise_finish."""
    import torch
    lib, check, _ptr, _stream = _lib()
    n, world = len(a), len(sizes)
    bases = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int64)
    slabs = [torch.from_numpy(a[bases[r]: bases[r + 1]].copy()).to(cuda) for r in range(world)]
    halo = torch.zeros(world * HALO, dtype=torch.float32, device=cuda)
    for r in range(world):
        m = min(HALO, sizes[r])
        if m:
            halo[r * HALO: r * HALO + m] = slabs[r][:m]
    bases_dev = torch.from_numpy(bases).to(cuda)
    nslot = lib.gsx_pairwise_slots(n)
    meanstd = torch.zeros(2, dtype=torch.float32, device=cuda)
    slot = torch.empty(nslot, dtype=torch.float32, device=cuda)
    for sq in (0, 1):
        total = torch.zeros(nslot, dtype=torch.float32, device=cuda)
        for r in range(world):
            check(lib.gsx_pairwise_leaves_dist(_ptr(slabs[r]), int(bases[r]), int(sizes[r]), n, sq, _ptr(meanstd),
                                               _ptr(halo), _ptr(bases_dev), world, _ptr(slot), _stream()),
                  "gsx_pairwise_leaves_dist")
            total += slot
        check(lib.gsx_pairwise_finish(_ptr(total), n, sq, _ptr(meanstd), _stream()), "gsx_pairwise_finish")
    return meanstd.cpu().numpy()


def _guarded_mask(n, off, cuda):
    import torch
    return torch.full((n + 16,), SENT8, dtype=torch.uint8, device=cuda)


def _unguard(mask, off, n):
    m = mask.cpu().numpy()
    assert np.all(m[:off] == SENT8) and np.all(m[off + n:] == SENT8), "mask bytes written outside [off, off + n)"
    return m[off: off + n]


def threshold_raw(a, in_off, mask_off, ms, tf, cuda):
    import torch
    lib, check, _ptr, _stream = _lib()
    n = len(a)
    buf = torch.zeros(n + 8, dtype=torch.float32, device=cuda)
    buf[in_off: in_off + n] = torch.from_numpy(a)
    msd = torch.tensor(np.asarray(ms, F32), device=cuda)
    mask = _guarded_mask(n, mask_off, cuda)
    check(lib.gsx_threshold_mask(_ptr(buf[in_off:]), n, _ptr(msd), float(F32(tf)), _ptr(mask[mask_off:]), _stream()),
          "gsx_threshold_mask")
    return _unguard(mask, mask_off, n)


def bbox_raw(xyz, row_off, mask_off, bounds, cuda):
    import torch
    lib, check, _ptr, _stream = _lib()
    from gsx._abi import f32x
    n = len(xyz)
    buf = torch.zeros((n + 8, 3), dtype=torch.float32, device=cuda)
    buf[row_off: row_off + n] = torch.from_numpy(xyz)
    with np.errstate(over="ignore"):
        lohi = f32x(*[F32(b) for b in bounds])
    mask = _guarded_mask(n, mask_off, cuda)
    check(lib.gsx_bbox_mask(_ptr(buf[row_off:]), n, lohi, _ptr(mask[mask_off:]), _stream()), "gsx_bbox_mask")
    return _unguard(mask, mask_off, n)


def compact_raw(mask_np, mask_off, xyz, op, idx, cuda):
    """gsx_compact_points with the mask at byte offset mask_off and every output pre-filled with a sentinel.
    Returns (count, xyz_out, op_out, idx_out) over the whole output buffers (n + 64 rows) on the host."""
    import torch
    lib, check, _ptr, _stream = _lib()
    n = len(mask_np)
    mbuf = torch.zeros(n + 16, dtype=torch.uint8, device=cuda)
    mbuf[mask_off: mask_off + n] = torch.from_numpy(mask_np)
    x = torch.from_numpy(xyz).to(cuda)
    o = torch.from_numpy(op).to(cuda) if op is not None else None
    i = torch.from_numpy(idx).to(cuda) if idx is not None else None
    full = lambda *shape: torch.full(shape, SENT32, dtype=torch.int32, device=cuda)  # noqa: E731
    xo, oo, io = full(n + 64, 3), (full(n + 64) if op is not None else None), full(n + 64)
    ws = torch.empty(lib.gsx_compact_workspace_bytes(n), dtype=torch.uint8, device=cuda)
    cnt = C.c_int64(-1)
    check(lib.gsx_compact_points(_ptr(mbuf[mask_off:]), n, _ptr(x), _ptr(o), _ptr(i), _ptr(xo), _ptr(oo), _ptr(io),
                                 C.byref(cnt), _ptr(ws), ws.numel(), _stream()), "gsx_compact_points")
    host = lambda t: t.cpu().numpy() if t is not None else None  # noqa: E731
    return cnt.value, host(xo), host(oo), host(io)


def _free_bytes(cuda):
    """Free device memory once this process's cached blocks are returned (earlier tests leave some)."""
    import torch
    torch.cuda.empty_cache()
    return torch.cuda.mem_get_info(cuda)[0]


def _all_equal_chunked(a, b, chunk=1 << 26):
    """torch.equal over row chunks (no full-size temporaries); b may be a callable (start, end) -> tensor."""
    import torch
    for s in range(0, a.shape[0], chunk):
        e = min(a.shape[0], s + chunk)
        want = b(s, e) if callable(b) else b[s:e]
        if not torch.equal(a[s:e], want):
            return False
    return True


# ================================================================================================ CPU: branch checks
def test_sweep_reaches_every_leaf_form():
    """n = 1..1100: depths 0..4, the serial leaf (< 8 elements), every leaf tail m % 8, unbalanced trees (n = 264 has
    leaves at depths 1 and 2); offset 0 of an aligned buffer takes the float4 leaves, offsets 1..3 the 8-lane form."""
    depths, tails, unbalanced, small = set(), set(), [], False
    for n in range(1, SWEEP_N + 1):
        lv = pw_leaves(n)
        assert sum(m for _, m, _ in lv) == n and max(d for _, _, d in lv) == pairwise_depth(n)
        depths.add(pairwise_depth(n))
        tails |= {m % 8 for _, m, _ in lv if m >= 8}
        small |= any(m < 8 for _, m, _ in lv)
        if len({d for _, _, d in lv}) > 1:
            unbalanced.append(n)
        assert mid_launches(pairwise_depth(n)) == ([], pairwise_depth(n) - 1)   # k_pw_top alone combines
    assert depths == {0, 1, 2, 3, 4} and tails == set(range(8)) and small
    assert 264 in unbalanced and {d for _, _, d in pw_leaves(264)} == {1, 2} and len(unbalanced) > 100
    assert [leaf_kernel(TORCH_ALIGN + 4 * s) for s in range(4)] == ["k_pw_leaves2"] + ["k_pw_leaves"] * 3


def test_depth_boundaries_reach_mid_launches():
    """d_min - 1 and d_min of every depth 1..22: the first k_pw_mid launch from 131 073 (depth 11), two launches from
    67 108 865 (depth 20), and at 268 435 457 (depth 22) a second launch spanning three levels."""
    for d in range(1, 23):
        dm = first_n_of_depth(d)
        assert pairwise_depth(dm - 1) == d - 1 and pairwise_depth(dm) == d
        launches, top = mid_launches(d)
        assert top <= MID_LOW - 1 and top == min(d - 1, MID_LOW - 1)
        assert len(launches) == (0 if d <= MID_LOW else 1 if d < 20 else 2)
    assert first_n_of_depth(11) == 131_073 and mid_launches(11) == ([(10, 10)], 9) and mid_launches(10) == ([], 9)
    assert first_n_of_depth(20) == 67_108_865 and mid_launches(20) == ([(19, 11), (10, 10)], 9)
    assert mid_launches(21) == ([(20, 12), (11, 10)], 9)
    assert first_n_of_depth(22) == 268_435_457 and mid_launches(22) == ([(21, 13), (12, 10)], 9)
    assert [n for n in BOUNDARY_NS if n >= SLOW_N] == [67_108_864, 67_108_865, 134_217_728, 134_217_729,
                                                       268_435_456, 268_435_457]


@pytest.mark.parametrize("n", [n for n in BOUNDARY_NS if LEAF < n < SLOW_N])
def test_order_sensitive_vector(n):
    """A sequential float32 sum and a float64 sum both give other bits than NumPy's pairwise sum."""
    a = order_sensitive(n, n)
    s = np.add.reduce(a)
    assert np.cumsum(a, dtype=F32)[-1].view(U32) != s.view(U32)
    assert F32(np.sum(a, dtype=np.float64)).view(U32) != s.view(U32)


def test_mean_std_edge_vectors():
    """Non-finite entries make NaN or inf; near FLT_MAX an inner node overflows; the subnormal vectors stay subnormal
    (the std one in its squared deviations); past 2^24 the float32 division differs from NumPy's float64 one."""
    for name, a in nonfinite_cases():
        ms = np_mean_std(a)
        assert not np.all(np.isfinite(ms)), name
    for signs in ("pos", "mixed"):
        a = overflow_vector(1000, 3, signs)
        with np.errstate(over="ignore", invalid="ignore"):
            assert np.isfinite(a).all() and not np.isfinite(np.add.reduce(a[:256]))
    sub = subnormal_vector(1000, 5, "sub")
    tiny = np.finfo(F32).tiny
    assert np.all(np.abs(sub) < tiny) and np.all(sub != 0)
    sq = subnormal_vector(1000, 6, "sq")
    d = sq - np.mean(sq)
    assert np.any((d * d != 0) & (np.abs(d * d) < tiny))
    a = order_sensitive(DIV_N, 24)
    s, ms = np.add.reduce(a), np_mean_std(a)
    assert pairwise_depth(DIV_N) == 18 and int(F32(DIV_N)) != DIV_N
    assert (s / F32(DIV_N)).view(U32) != ms[0].view(U32)
    assert F32(np.float64(s) / DIV_N).view(U32) == ms[0].view(U32)


def test_sharded_cases_reach_spill_over():
    for s in sharded_world8():
        assert len(s) == 8 and max(s) <= 20 and max_slabs_per_leaf(s) >= 3, s
    for s in SHARD_EDGE:
        assert s[0] == 0 or s[-1] == 0
    for c in CUTS:                      # (c, 128, 128 - c): both leaves of n = 256 cut at offset c
        bases = np.cumsum((0, c, LEAF, LEAF - c))
        assert [(o, m) for o, m, _ in pw_leaves(256)] == [(0, LEAF), (LEAF, LEAF)]
        assert all(o < b < o + LEAF for o, b in zip((0, LEAF), bases[1:3]))
    n = sum(SHARD_SLOW)
    assert n == SLOW_N + 1 and pairwise_depth(n) == 20 and len(mid_launches(20)[0]) == 2
    for b in np.cumsum(SHARD_SLOW)[:2]:
        off, m = leaf_of(n, int(b))
        assert off < b < off + m


@pytest.mark.parametrize("case", threshold_stats(), ids=lambda c: c[0])
def test_threshold_values_straddle(case):
    name, mean, std, tf = case
    a = threshold_values(mean, std, tf, 1)
    want, t = ref_threshold(a, mean, std, tf)
    assert len(a) % 4 == 3
    if np.isfinite(t):
        below, up = np.nextafter(t, F32(-np.inf)), np.nextafter(t, F32(np.inf))
        assert want[a == below].all() and not want[a == t].any() and not want[a == up].any()
    if name == "tf01":
        assert float(F32(0.1)) != 0.1
    if name in ("std_inf_tf0", "mean_nan", "std_nan"):
        assert np.isnan(t) and not want.any()
    assert [threshold_form(TORCH_ALIGN + 4 * i, TORCH_ALIGN + j) for i, j in ((0, 0), (1, 0), (0, 1), (3, 2))] == \
        ["vector", "scalar", "scalar", "scalar"]


@pytest.mark.parametrize("name", BBOX_CASES)
def test_bbox_case_properties(name):
    xyz, bounds = bbox_case(name)
    want = ref_bbox(xyz, bounds)
    with np.errstate(over="ignore"):
        fb = [F32(b) for b in bounds]
    if name == "lanes_on_bounds":         # 6 bounds x 4 lanes x (on, one ulp out)
        g = want[:192].reshape(48, 4)
        for k in range(48):
            lane = (k // 2) % 4
            assert g[k, lane] == (k % 2 == 0) and all(g[k, j] for j in range(4) if j != lane)
    if name == "unrepresentable":         # a float64 compare would decide some of the f32(bound) rows otherwise
        with np.errstate(over="ignore"):
            f64 = oracle.bbox_mask(*(xyz[:, k].astype(np.float64) for k in range(3)), *bounds)
        assert all(float(f) != b for f, b in zip(fb, bounds)) and np.any(f64 != want)
    if name == "signed_zero":
        assert want[:8].all() and not want[8:14].any()
    if name == "nonfinite_inf_bounds":
        assert not want[np.isnan(xyz).any(axis=1)].any() and want[np.isinf(xyz).any(axis=1) & ~np.isnan(xyz).any(axis=1)].all()
    if name == "lo_gt_hi":
        assert not want.any()
    if name == "overflow_bound":
        assert np.isinf(fb[0]) and np.isinf(fb[3]) and np.isinf(fb[5]) and want.any() and not want.all()
    for r in range(5):                    # xyz at row offset r: 16-byte aligned iff r % 4 == 0
        for mo in range(4):
            v4, s = vec_split(len(xyz), TORCH_ALIGN + 12 * r, TORCH_ALIGN + mo)
            assert (v4 > 0) == (r % 4 == 0 and mo == 0) and s == len(xyz) - v4


def test_alpha_thresholds_need_float64():
    """For 127 of the thresholds 1..254 f32(t) < t: a float32 compare keeps the row at f32(t), the reference drops it."""
    from gsx import masks
    below = 0
    for u in ALPHA_LIMITS:
        t = masks.alpha_logit_threshold(u)
        a = alpha_values(u)
        want = oracle.alpha_mask(a, u)
        if float(F32(t)) < t:
            below += 1
            assert not want[a == F32(t)].any() and (a[a == F32(t)] >= F32(t)).all()
        assert not want[np.isnan(a)].any() and want[a == np.inf].all() and not want[a == -np.inf].any()
    assert below == 127
    assert vec_split(ALPHA_L, TORCH_ALIGN, TORCH_ALIGN) == (8, 3) and vec_split(8, TORCH_ALIGN + 4, TORCH_ALIGN) == (0, 8)


def test_alpha_logit_threshold_libm_within_one_ulp(gsx_lib):
    from gsx import masks
    for u in range(256):
        a = np.float64(gsx_lib.gsx_alpha_logit_threshold(float(u)))
        b = np.float64(masks.alpha_logit_threshold(u))
        assert abs(int(a.view(np.int64)) - int(b.view(np.int64))) <= 1, u


@pytest.mark.parametrize("n", ONEPASS_NS)
@pytest.mark.parametrize("kind", MASK_KINDS)
def test_compact_case_reaches_branch(n, kind):
    m = compact_mask(n, kind)
    keep = np.flatnonzero(m)
    tiles = -(-n // TILE)
    assert compact_form(n) == "onepass"
    if kind == "all":
        assert len(keep) == n
    if kind == "none":
        assert len(keep) == 0
    if kind == "runs":
        assert 0 < len(keep) < n and np.any(np.diff(m.astype(np.int8)) != 0)
    if kind == "last_tile_one":
        assert len(keep) == 1 and keep[0] // TILE == tiles - 1
    if kind == "first_tile":
        assert len(keep) > 0 and keep.max() < TILE
    if kind == "bytes":
        assert set(np.unique(m).tolist()) == {0, 1, 2, 0x80, 0xFF}
    for off in range(8):
        vec, scal = mask_groups(n, TORCH_ALIGN + off)
        assert (vec > 0) == (off == 0) and (scal > 0) == (off != 0 or n % GROUP != 0)
    assert (lookback_windows(tiles - 1) >= 2) == (n == 33 * TILE + 1)


def test_compact_large_forms():
    assert compact_form(ONEPASS_LIMIT - 1) == "onepass" and ONEPASS_LIMIT - 1 == LB_VAL
    assert compact_form(TWOPASS_N) == "twopass" and TWOPASS_N % BLOCK2 != 0 and TWOPASS_N % 32 != 0
    assert compact_form(COMPACT_ROW_LIMIT - 1) == "twopass" and compact_form(COMPACT_ROW_LIMIT) == "refused"


def test_compact_refuses_2_pow_31_rows(gsx_lib):
    """From 2^31 rows the int32 row index would wrap: refused before the workspace is looked at, nothing launched."""
    cnt = C.c_int64(-7)
    rc = gsx_lib.gsx_compact_points(None, COMPACT_ROW_LIMIT, None, None, None, None, None, None, C.byref(cnt), None, 0,
                                    None)
    assert rc == GSX_ERR_UNSUPPORTED and cnt.value == -7
    assert b"2^31" in gsx_lib.gsx_last_error()
    rc = gsx_lib.gsx_compact_points(None, COMPACT_ROW_LIMIT - 1, None, None, None, None, None, None, C.byref(cnt), None,
                                    0, None)
    assert rc == GSX_ERR_WORKSPACE and cnt.value == -7


def test_colour_edges_reach_clip():
    for scale in COLOUR_SCALES:
        e = colour_edges(scale)
        with np.errstate(invalid="ignore"):
            p = (F32(0.5) + F32(scale) * e) * F32(255)
        assert np.sum(p == 255) >= 1 and np.any((p > 255) & (p < 256)) and np.any((p > 254) & (p < 255))
        assert np.sum(p == 0) >= 1 and np.any((p < 0) & (p > -1)) and np.any((p > 0) & (p < 1))
        assert np.isnan(p).any() and np.any(np.signbit(e) & (e == 0))
        want = ref_colour(e, scale)
        assert want[p == 255].min() == 255 and want[(p > 254) & (p < 255)].max() == 254


# ================================================================================================ GPU: exact equality
@pytest.mark.gpu
@pytest.mark.parametrize("shift", range(4))
def test_mean_std_every_n_to_1100(shift, cuda, gsx_lib):
    """n = 1..1100 at element offset 0 (float4 leaves) or 1, 2, 3 (8-lane leaves)."""
    import torch
    a = order_sensitive(SWEEP_N, 1100)
    buf = torch.zeros(SWEEP_N + 8, dtype=torch.float32, device=cuda)
    buf[shift: shift + SWEEP_N] = torch.from_numpy(a)
    ws = torch.empty(gsx_lib.gsx_mean_std_workspace_bytes(SWEEP_N), dtype=torch.uint8, device=cuda)
    out = torch.empty((SWEEP_N, 2), dtype=torch.float32, device=cuda)
    for n in range(1, SWEEP_N + 1):
        mean_std_exact(buf, shift, n, ws=ws, out=out[n - 1])
    got = out.cpu().numpy()
    for n in range(1, SWEEP_N + 1):
        want = np_mean_std(a[:n])
        assert same_bits(got[n - 1], want), (n, got[n - 1], want)


@functools.lru_cache(maxsize=1)
def _boundary_case(n):
    a = order_sensitive(n, n)
    return a, np_mean_std(a)


@pytest.mark.gpu
@pytest.mark.parametrize("n,shift", [pytest.param(n, s, marks=[pytest.mark.slow] if n >= SLOW_N else [])
                                     for n in BOUNDARY_NS for s in (0, 1)])
def test_mean_std_depth_boundaries(n, shift, cuda, gsx_lib):
    a, want = _boundary_case(n)
    assert same_bits(mean_std_at(a, shift, cuda), want)


@pytest.mark.gpu
@pytest.mark.parametrize("shift", (0, 1))
def test_mean_std_nonfinite(shift, cuda, gsx_lib):
    for name, a in nonfinite_cases():
        assert same_bits(mean_std_at(a, shift, cuda), np_mean_std(a)), name


@pytest.mark.gpu
@pytest.mark.parametrize("shift", (0, 1))
@pytest.mark.parametrize("n", (9, 1000, 100_003))
@pytest.mark.parametrize("signs", ("pos", "mixed"))
def test_mean_std_overflow(n, signs, shift, cuda, gsx_lib):
    a = overflow_vector(n, n, signs)
    assert same_bits(mean_std_at(a, shift, cuda), np_mean_std(a))


@pytest.mark.gpu
@pytest.mark.parametrize("shift", (0, 1))
@pytest.mark.parametrize("n", (5, 1000, 100_003))
@pytest.mark.parametrize("kind", ("sub", "sq"))
def test_mean_std_subnormal(n, kind, shift, cuda, gsx_lib):
    """No flush to zero anywhere: the build has no -ftz."""
    a = subnormal_vector(n, n, kind)
    assert same_bits(mean_std_at(a, shift, cuda), np_mean_std(a))


@pytest.mark.gpu
@pytest.mark.parametrize("shift", (0, 1))
def test_mean_std_float64_division_past_2_pow_24(shift, cuda, gsx_lib):
    a, want = _boundary_case(DIV_N)
    assert same_bits(mean_std_at(a, shift, cuda), want)


@pytest.mark.gpu
def test_sharded_world8_small_slabs(cuda, gsx_lib):
    for sizes in sharded_world8():
        a = order_sensitive(sum(sizes), sum(sizes) + 8)
        assert same_bits(sharded_mean_std(a, sizes, cuda), np_mean_std(a)), sizes


@pytest.mark.gpu
@pytest.mark.parametrize("sizes", SHARD_EDGE)
def test_sharded_empty_end_slabs(sizes, cuda, gsx_lib):
    a = order_sensitive(sum(sizes), sum(sizes))
    assert same_bits(sharded_mean_std(a, sizes, cuda), np_mean_std(a))


@pytest.mark.gpu
def test_sharded_cut_at_every_leaf_offset(cuda, gsx_lib):
    a = order_sensitive(2 * LEAF, 256)
    want = np_mean_std(a)
    for c in CUTS:
        assert same_bits(sharded_mean_std(a, (c, LEAF, LEAF - c), cuda), want), c


@pytest.mark.gpu
@pytest.mark.slow
def test_sharded_two_mid_launches(cuda, gsx_lib):
    n = sum(SHARD_SLOW)
    a = order_sensitive(n, n)
    assert same_bits(sharded_mean_std(a, SHARD_SLOW, cuda), np_mean_std(a))


FORM_OFFSETS = [(0, 0), (1, 0), (2, 0), (3, 0), (0, 1), (0, 2), (0, 3), (1, 1)]   # (input offset, mask offset)
_form_id = lambda f: f"in{f[0]}-mask{f[1]}"  # noqa: E731


@pytest.mark.gpu
@pytest.mark.parametrize("form", FORM_OFFSETS, ids=_form_id)
@pytest.mark.parametrize("case", threshold_stats(), ids=lambda c: c[0])
def test_threshold_mask_forms(case, form, cuda, gsx_lib):
    """Every n % 4 in the vector form (in0-mask0) or the scalar form (input 1..3 floats or mask 1..3 bytes off
    alignment)."""
    name, mean, std, tf = case
    io, mo = form
    full = threshold_values(mean, std, tf, 1)
    for tail in range(4):
        a = full[: len(full) - tail]
        want, _ = ref_threshold(a, mean, std, tf)
        got = threshold_raw(a, io, mo, (mean, std), tf, cuda)
        assert np.array_equal(got, want.astype(np.uint8)), (len(a), np.flatnonzero(got != want)[:8])


@pytest.mark.gpu
@pytest.mark.parametrize("form", [(r, mo) for r in range(5) for mo in range(4)], ids=lambda f: f"row{f[0]}-mask{f[1]}")
@pytest.mark.parametrize("name", BBOX_CASES)
def test_bbox_mask_forms(name, form, cuda, gsx_lib):
    """xyz at row offset 0..4 (16-byte aligned at 0 and 4), mask at byte offset 0..3, every n % 4."""
    xyz, bounds = bbox_case(name)
    r, mo = form
    for tail in range(4):
        x = xyz[: len(xyz) - tail]
        want = ref_bbox(x, bounds).astype(np.uint8)
        got = bbox_raw(x, r, mo, bounds, cuda)
        assert np.array_equal(got, want), (len(x), np.flatnonzero(got != want)[:8])


@pytest.mark.gpu
@pytest.mark.parametrize("form", FORM_OFFSETS[:7], ids=_form_id)
def test_alpha_mask_every_threshold(form, cuda, gsx_lib):
    """All 254 thresholds in one buffer (row stride 80 bytes, so every row start stays 16-byte aligned), n = 11, 10,
    9, 8."""
    import torch
    from gsx import masks
    lib, check, _ptr, _stream = _lib()
    U, S = len(ALPHA_LIMITS), 20
    io, mo = form
    vals = np.stack([alpha_values(u) for u in ALPHA_LIMITS])
    for tail in range(4):
        n = ALPHA_L - tail
        ops = torch.zeros((U, S), dtype=torch.float32, device=cuda)
        ops[:, io: io + n] = torch.from_numpy(vals[:, :n])
        mask = torch.full((U, 24), SENT8, dtype=torch.uint8, device=cuda)
        for k, u in enumerate(ALPHA_LIMITS):
            check(lib.gsx_alpha_mask(_ptr(ops[k, io:]), n, masks.alpha_logit_threshold(u), _ptr(mask[k, mo:]),
                                     _stream()), "gsx_alpha_mask")
        got = mask.cpu().numpy()
        assert np.all(got[:, :mo] == SENT8) and np.all(got[:, mo + n:] == SENT8), n
        for k, u in enumerate(ALPHA_LIMITS):
            want = oracle.alpha_mask(vals[k, :n], u).astype(np.uint8)
            assert np.array_equal(got[k, mo: mo + n], want), (u, n)


@pytest.mark.gpu
@pytest.mark.parametrize("limit", (0, -3, 1, 5, 128, 254, 255, 300))
def test_dataprocessor_alpha_filter(limit, cuda, gsx_lib):
    """The caller's early-outs (<= 0 keeps all, >= 255 keeps none) and the float64 rule around f32(t)."""
    from gsconverter.processing import DataProcessor
    from gsx import masks, synth
    a = synth.structured(40_003, "mixed")
    for k, u in enumerate((1, 5, 128, 254)):
        t = F32(masks.alpha_logit_threshold(u))
        a["opacity"][4 * k: 4 * k + 3] = [t, np.nextafter(t, F32(-np.inf)), np.nextafter(t, F32(np.inf))]
    want = a[oracle.alpha_mask(a["opacity"], limit)]
    for dev_rec in (False, True):                     # records gathered on the host / on the device
        dp = DataProcessor(a.copy())
        dp.device_records = dev_rec
        dp.apply_alpha_filter(limit)
        got = dp.data
        assert got.dtype == want.dtype and np.array_equal(got, want), dev_rec


@pytest.mark.gpu
@pytest.mark.parametrize("off", range(8))
@pytest.mark.parametrize("n", ONEPASS_NS)
@pytest.mark.parametrize("kind", MASK_KINDS)
def test_compact_onepass(kind, n, off, cuda, gsx_lib):
    """Mask at byte offset 0..7 (8-byte mask loads only at 0); opacity and the chained input index each present or
    absent (by the offset's low bits); nothing written past the count."""
    m = compact_mask(n, kind)
    xyz, op, idx = compact_inputs(n, n)
    keep = np.flatnonzero(m)
    k = len(keep)
    with_op, with_idx = off % 2 == 0, off // 2 % 2 == 0
    cnt, xo, oo, io = compact_raw(m, off, xyz, op if with_op else None, idx if with_idx else None, cuda)
    assert cnt == k
    assert np.array_equal(xo[:k].view(U32), xyz[keep].view(U32))
    assert np.array_equal(io[:k], idx[keep] if with_idx else keep.astype(np.int32))
    assert np.all(xo[k:] == SENT32) and np.all(io[k:] == SENT32)
    if with_op:
        assert np.array_equal(oo[:k].view(U32), op[keep].view(U32)) and np.all(oo[k:] == SENT32)


@pytest.mark.gpu
@pytest.mark.slow
def test_compact_onepass_largest(cuda, gsx_lib):
    """n = 2^30 - 1, all kept: the largest one-pass size, whose count is exactly the 30-bit look-back maximum.  Peak
    device memory 29.5 GiB, measured on an H100 80GB HBM3 (xyz in and out, the index, the mask)."""
    import torch
    lib, check, _ptr, _stream = _lib()
    n = ONEPASS_LIMIT - 1
    if _free_bytes(cuda) < 34 * 2**30:
        pytest.skip("needs 34 GiB of free device memory")
    gen = torch.Generator(device=cuda).manual_seed(30)
    xyz = torch.rand(n, 3, device=cuda, generator=gen)
    mask = torch.ones(n, dtype=torch.uint8, device=cuda)
    xo = torch.empty_like(xyz)
    io = torch.empty(n, dtype=torch.int32, device=cuda)
    ws = torch.empty(lib.gsx_compact_workspace_bytes(n), dtype=torch.uint8, device=cuda)
    cnt = C.c_int64(-1)
    check(lib.gsx_compact_points(_ptr(mask), n, _ptr(xyz), None, None, _ptr(xo), None, _ptr(io), C.byref(cnt),
                                 _ptr(ws), ws.numel(), _stream()), "gsx_compact_points")
    assert cnt.value == n == LB_VAL
    assert _all_equal_chunked(xo, xyz)
    assert _all_equal_chunked(io, lambda s, e: torch.arange(s, e, dtype=torch.int32, device=cuda))


@pytest.mark.gpu
@pytest.mark.slow
def test_compact_twopass_warp_patterns(cuda, gsx_lib):
    """n = 2^30 + 4099 (a partial last block and a partial last warp), opacity present.  Every warp of 32 rows is
    dropped whole, kept whole, keeps one row, or keeps random rows with random non-zero bytes.  Compared on the device
    with torch.nonzero and indexing.  Peak device memory 41.6 GiB, measured on an H100 80GB HBM3: xyz, opacity and the
    mask in, xyz, opacity and the index out, the int64 nonzero list."""
    import torch
    lib, check, _ptr, _stream = _lib()
    n = TWOPASS_N
    if _free_bytes(cuda) < 46 * 2**30:
        pytest.skip("needs 46 GiB of free device memory")
    gen = torch.Generator(device=cuda).manual_seed(31)
    nw = -(-n // 32)
    kind = torch.randint(0, 4, (nw, 1), dtype=torch.uint8, device=cuda, generator=gen)
    lane = torch.randint(0, 32, (nw, 1), dtype=torch.int64, device=cuda, generator=gen)
    m2 = torch.randint(0, 256, (nw, 32), dtype=torch.uint8, device=cuda, generator=gen)
    m2.mul_(m2 >= 128).mul_(kind == 3)                            # kind 3: bytes 128..255 on about half the rows
    m2.masked_fill_(kind == 1, 0xFF)                              # whole warp kept
    single = torch.zeros((nw, 32), dtype=torch.uint8, device=cuda).scatter_(1, lane, 0x80)
    m2.add_(single * (kind == 2))                                 # one row kept
    del single, lane
    mask = m2.view(-1)[:n]
    xyz = torch.rand(n, 3, device=cuda, generator=gen)
    op = torch.randn(n, device=cuda, generator=gen)
    full = lambda *shape: torch.full(shape, SENT32, dtype=torch.int32, device=cuda)  # noqa: E731
    xo, oo, io = full(n, 3), full(n), full(n)
    ws = torch.empty(lib.gsx_compact_workspace_bytes(n), dtype=torch.uint8, device=cuda)
    cnt = C.c_int64(-1)
    check(lib.gsx_compact_points(_ptr(mask), n, _ptr(xyz), _ptr(op), None, _ptr(xo), _ptr(oo), _ptr(io), C.byref(cnt),
                                 _ptr(ws), ws.numel(), _stream()), "gsx_compact_points")
    k = cnt.value
    nz = torch.nonzero(mask).squeeze(1)
    assert k == nz.numel() and 0 < k < n
    counts = [int(v) for v in torch.bincount(kind.view(-1).long(), minlength=4).tolist()]
    assert min(counts) > 0
    assert _all_equal_chunked(io[:k], lambda s, e: nz[s:e].to(torch.int32))
    assert _all_equal_chunked(xo[:k], lambda s, e: xyz[nz[s:e]].view(torch.int32))
    assert _all_equal_chunked(oo[:k], lambda s, e: op[nz[s:e]].view(torch.int32))
    sent = lambda s, e: torch.full((e - s,), SENT32, dtype=torch.int32, device=cuda)  # noqa: E731
    assert _all_equal_chunked(io[k:], sent) and _all_equal_chunked(oo[k:], sent)


@pytest.mark.gpu
@pytest.mark.parametrize("F", GATHER_FS)
def test_gather_rows(F, cuda, gsx_lib):
    import torch
    lib, check, _ptr, _stream = _lib()
    for m in GATHER_MS:
        rows, idx = gather_case(F, m)
        r = torch.from_numpy(rows).to(cuda)
        i = torch.from_numpy(idx).to(cuda)
        out = torch.full(((m + 2) * F,), SENT32, dtype=torch.int32, device=cuda)
        check(lib.gsx_records_gather_rows(_ptr(r), _ptr(i), m, F, _ptr(out), _stream()), "gsx_records_gather_rows")
        got = out.cpu().numpy()
        assert np.array_equal(got[: m * F].view(U32), rows[idx].reshape(-1).view(U32)), (F, m)
        assert np.all(got[m * F:] == SENT32), (F, m)


@pytest.mark.gpu
@pytest.mark.parametrize("cols", ((5, 0, 13, 7), (13, 12, 11, 0), (0, 1, 2, None), (9, 9, 4, None)))
def test_extract_xyz_opacity_columns(cols, cuda, gsx_lib):
    import torch
    lib, check, _ptr, _stream = _lib()
    n, F = 10_007, 14
    rng = np.random.default_rng(sum(c or 0 for c in cols))
    rows = rng.integers(0, 1 << 32, (n, F), dtype=np.uint32).view(F32)
    cx, cy, cz, cop = cols
    r = torch.from_numpy(rows).to(cuda)
    xyz = torch.full((n + 4, 3), SENT32, dtype=torch.int32, device=cuda)
    op = torch.full((n + 4,), SENT32, dtype=torch.int32, device=cuda)
    check(lib.gsx_records_extract_xyz_opacity(_ptr(r), n, F, cx, cy, cz, cop if cop is not None else 0, _ptr(xyz),
                                              _ptr(op) if cop is not None else None, _stream()),
          "gsx_records_extract_xyz_opacity")
    x, o = xyz.cpu().numpy(), op.cpu().numpy()
    assert np.array_equal(x[:n].view(U32), rows[:, [cx, cy, cz]].view(U32)) and np.all(x[n:] == SENT32)
    if cop is None:
        assert np.all(o == SENT32)
    else:
        assert np.array_equal(o[:n].view(U32), rows[:, cop].view(U32)) and np.all(o[n:] == SENT32)


@pytest.mark.gpu
@pytest.mark.parametrize("scale", COLOUR_SCALES)
def test_colour_rgba8_clip_edges(scale, cuda, gsx_lib):
    """Colour channels, alpha and scale_exp bit-exact at the clip edges (the exp is NumPy's float32 exp)."""
    import torch
    lib, check, _ptr, _stream = _lib()
    rows = colour_rows(scale)
    n, F = rows.shape
    r = torch.from_numpy(rows).to(cuda)
    rgba = torch.full(((n + 4) * 4,), SENT8, dtype=torch.uint8, device=cuda)
    check(lib.gsx_records_color_rgba8(_ptr(r), n, F, 9, 2, 11, 5, float(F32(scale)), _ptr(rgba), _stream()),
          "gsx_records_color_rgba8")
    got = rgba.cpu().numpy()
    assert np.all(got[4 * n:] == SENT8)
    got = got[: 4 * n].reshape(n, 4)
    for ch, c in enumerate((9, 2, 11)):
        want = ref_colour(rows[:, c], scale)
        assert np.array_equal(got[:, ch], want), (ch, np.flatnonzero(got[:, ch] != want)[:8])
    with np.errstate(over="ignore"):
        want_a = np.clip((1.0 / (1.0 + np.exp(-rows[:, 5]))) * 255, 0, 255).astype(np.uint8)
    assert np.array_equal(got[:, 3], want_a), np.flatnonzero(got[:, 3] != want_a)[:8]
    sc = torch.empty((n, 3), dtype=torch.float32, device=cuda)
    check(lib.gsx_records_scale_exp(_ptr(r), n, F, 0, 7, 13, _ptr(sc), _stream()), "gsx_records_scale_exp")
    with np.errstate(over="ignore"):
        want_s = np.exp(rows[:, [0, 7, 13]])
    assert np.array_equal(sc.cpu().numpy().view(U32), want_s.view(U32))
