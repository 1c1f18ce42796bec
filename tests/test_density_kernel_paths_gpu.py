"""The density filter kernels path by path: each histogram form, the flush and fallback branches of the shared-memory
tables, the key-width boundary, the two-word same-column branch, voxel faces, each membership form, the staged API
and non-finite rows, each on a cloud built to reach that path at the shipped constants.

Every case is a builder (a plain seeded function returning float32 xyz and the parameters it runs with) and two kinds
of test:
  * an unmarked CPU test restating the dispatch of `density_voxel_count`, `density_member_mask` and
    `density_grid_count` (workspace layout, grid or hash, kernel, key width, bitmap or hash set, vec4 or scalar) and
    asserting that the case reaches its branch, plus the property of the data the case relies on, checked with NumPy;
  * a `gpu` test asserting exact equality with a plain reference: `np.unique` of floor(xyz / f32(voxel)) for the dense
    list, the counts and the number of voxels; `oracle.density_mask` for the keep-mask; NumPy set membership for the
    membership kernels; a NumPy histogram for the staged grid.

Constants these cases are built around (csrc/gsx_density.cu): a voxel box of <= 24 576 cells is counted in shared
memory by persistent 512-thread CTAs (`k_vox_count_smem`, 4 rows per float4 group, ragged tail of < 4 rows read by
block 0, scalar loads when xyz is not 16-byte aligned), a larger box that fits the workspace by `k_vox_count_grid_agg`
(2 048 rows per CTA into a 1 024-slot shared table, eight probes, then one global add per row), a box of 2^32 - 16
cells or more by `k_vox_count<GridTable>`; a box that does not fit the workspace goes to the hash table, with 3 x 21-bit
keys, or two-word keys when an extent reaches 2^21.  The kept voxels are a bitmap when their box has <= 2^27 voxels
and the bitmap fits the workspace, a hash set otherwise.

Rows with a NaN coordinate fall outside the finite box: they are dropped and counted, and min_points or more of them
are refused (the reference would put them in a voxel of their own, which could then be dense).
"""
import ctypes as C
import functools

import numpy as np
import pytest

import oracle

F32 = np.float32
AXIS_LIM = 1 << 21
SMEM_CELLS, SMEM_THREADS = 24 * 1024, 512
AGG_ROWS, AGG_SLOTS = 256 * 8, 1024
PLAIN_CELLS = 0xFFFFFFF0
MAX_KEEP_BITS = 1 << 27
EXTENT_LIM = 1 << 31
H100_SMS = 132
BIG_N = 300_001
COUNT_NS = (1, 2, 3, 4, 5, 2047, 2048, 2049, BIG_N)
E_COUNT = 37                                    # the crafted voxel of the big clouds holds exactly this many rows


# ------------------------------------------------------------------------------------------------ dispatch, restated
def _align(x, a=256):
    return (x + a - 1) // a * a


def workspace_bytes(n, cap):
    """density_workspace_bytes."""
    n, cap = max(n, 1), max(cap, 1)
    slots = 64
    while slots < 2 * n:
        slots <<= 1
    return slots * 12 + 6 * 1024 * 4 + cap * 28 + 8192


def blob_bytes(ws, cap):
    """What the Carver of density_voxel_count leaves for the grid or hash table: every take aligned to 256."""
    off = 0
    for nbytes in (6 * 1024 * 4, 8 * 4, 4 * 8, 3 * cap * 8, cap * 4):
        off = _align(off) + nbytes
    return ws - _align(off)


def voxels(a, voxel):
    """floor(a / f32(voxel)) as int64, NaN -> INT64_MIN (x86, NumPy and the kernels)."""
    with np.errstate(invalid="ignore", over="ignore"):
        return np.floor(np.asarray(a, F32) / F32(voxel)).astype(np.int64)


def box(xyz, voxel):
    """Voxel box of the finite min/max (fminf/fmaxf leave NaN rows out)."""
    lo, hi = np.fmin.reduce(xyz, axis=0), np.fmax.reduce(xyz, axis=0)
    q0, q1 = voxels(lo, voxel), voxels(hi, voxel)
    return q0, q1 - q0 + 1


def cap_of(n, min_points):
    return n // max(min_points, 1) + 1


def count_path(xyz, voxel, min_points, ws=None):
    """Which histogram kernel density_voxel_count launches."""
    n = len(xyz)
    cap = cap_of(n, min_points)
    ws = workspace_bytes(n, cap) if ws is None else ws
    q0, dim = box(xyz, voxel)
    if np.any(dim < 1) or np.any(dim >= EXTENT_LIM):
        return "error"
    cells = float(np.prod(dim.astype(np.float64)))
    if cells * 4.0 <= blob_bytes(ws, cap):
        ncell = int(np.prod(dim))
        return "smem" if ncell <= SMEM_CELLS else "agg" if ncell < PLAIN_CELLS else "plain"
    return "wide" if np.any(dim >= AXIS_LIM) else "hash"


def smem_blocks(n, sms=H100_SMS):
    """Rows [r0, r1) counted by each CTA of k_vox_count_smem (groups of 4 rows; the tail goes to block 0)."""
    n4 = n // 4
    blocks = max(min(2 * sms, (n4 + SMEM_THREADS - 1) // SMEM_THREADS), 1)
    per = -(-n4 // blocks)
    return [(4 * min(b * per, n4), 4 * min(b * per + per, n4)) for b in range(blocks)]


def member_ws(keep):
    """The workspace gsx.density.member_mask allocates."""
    need = max(64, 1 << int(np.ceil(np.log2(max(2 * len(keep), 1))))) * 16 + 256
    bits = int(np.prod((keep.max(axis=0) - keep.min(axis=0) + 1).astype(np.float64)))
    return max(need, bits // 8 + 256) if bits <= MAX_KEEP_BITS else need


def hash_set_bytes(keep):
    o, hi = keep.min(axis=0), keep.max(axis=0)
    slots = 64
    while slots < 2 * len(keep):
        slots <<= 1
    return slots * 8 * (2 if np.any(hi - o >= AXIS_LIM) else 1)


def member_path(keep, ws):
    """Which membership form density_member_mask runs."""
    o, hi = keep.min(axis=0), keep.max(axis=0)
    if np.any(hi - o >= EXTENT_LIM):
        return "error"
    dx, dy, dz = (int(v) for v in hi - o + 1)
    small = dx <= MAX_KEEP_BITS and dy <= MAX_KEEP_BITS and dx * dy <= MAX_KEEP_BITS and dx * dy * dz <= MAX_KEEP_BITS
    if small and (dx * dy * dz + 31) // 32 * 4 <= ws:
        return "bitmap"
    return "hash_wide" if np.any(hi - o >= AXIS_LIM) else "hash"


def member_split(n, xyz_off, mask_off):
    """(rows of the 4-wide kernel, rows of the scalar kernel)."""
    n4 = n // 4 if xyz_off % 16 == 0 and mask_off % 4 == 0 else 0
    return 4 * n4, n - 4 * n4


# ------------------------------------------------------------------------------------------------ references
def ref_dense(xyz, voxel, min_points):
    """np.unique of the voxels of the rows without NaN: (dense voxels, their counts, number of voxels)."""
    q = voxels(xyz, voxel)[~np.isnan(xyz).any(axis=1)]
    u, c = np.unique(q, axis=0, return_counts=True)
    s = c >= max(min_points, 1)
    return u[s], c[s].astype(np.int32), len(u)


def ref_member(xyz, voxel, keep):
    q = voxels(xyz, voxel)
    u, inv = np.unique(np.r_[keep, q], axis=0, return_inverse=True)
    inv = inv.reshape(-1)
    kept = np.zeros(len(u), bool)
    kept[inv[: len(keep)]] = True
    return kept[inv[len(keep):]]


def ref_grid(xyz, voxel, q0, dim):
    """Histogram of the in-box rows over the box, and the number of the others."""
    q = voxels(xyz, voxel)
    inb = np.all((q >= q0) & (q <= q0 + dim - 1), axis=1)
    r = q[inb] - q0
    flat = (r[:, 0] * dim[1] + r[:, 1]) * dim[2] + r[:, 2]
    return np.bincount(flat, minlength=int(np.prod(dim))).astype(np.int32), int((~inb).sum())


# ------------------------------------------------------------------------------------------------ device calls
def _lib():
    from gsx._abi import lib, check
    from gsx._abi import _stream
    return lib, check, _stream


def voxel_count(x, voxel, min_points, extra=0):
    """gsx_density_voxel_count with the workspace dense_voxels() allocates plus `extra` bytes; sorted like np.unique."""
    import torch
    lib, check, stream = _lib()
    n = x.shape[0]
    cap = cap_of(n, min_points)
    ws = torch.empty(workspace_bytes(n, cap) + extra, dtype=torch.uint8, device=x.device)
    vox, cnt = np.empty((cap, 3), np.int64), np.empty(cap, np.int32)
    nd, nv = C.c_int64(0), C.c_int64(0)
    check(lib.gsx_density_voxel_count(C.c_void_p(x.data_ptr()), n, float(F32(voxel)), int(min_points),
                                      vox.ctypes.data_as(C.c_void_p), cnt.ctypes.data_as(C.c_void_p), cap,
                                      C.byref(nd), C.byref(nv), C.c_void_p(ws.data_ptr()), ws.numel(), stream()),
          "gsx_density_voxel_count")
    vox, cnt = vox[: nd.value], cnt[: nd.value]
    order = np.lexsort((vox[:, 2], vox[:, 1], vox[:, 0]))
    return vox[order], cnt[order], nv.value


def member_raw(xbuf, row0, n, voxel, keep, ws_bytes, mask_off=0):
    """gsx_density_member_mask on rows [row0, row0 + n) of xbuf, into a mask at byte offset mask_off of a guarded
    buffer; checks that no byte outside the mask is written."""
    import torch
    lib, check, stream = _lib()
    keep = np.ascontiguousarray(keep, np.int64)
    mask = torch.full((n + 16,), 0x5A, dtype=torch.uint8, device=xbuf.device)
    ws = torch.empty(max(ws_bytes, 1), dtype=torch.uint8, device=xbuf.device)
    check(lib.gsx_density_member_mask(C.c_void_p(xbuf.data_ptr() + 12 * row0), n, float(F32(voxel)),
                                      keep.ctypes.data_as(C.c_void_p), len(keep), C.c_void_p(mask.data_ptr() + mask_off),
                                      C.c_void_p(ws.data_ptr()), ws_bytes, stream()), "gsx_density_member_mask")
    m = mask.cpu().numpy()
    assert np.all(m[:mask_off] == 0x5A) and np.all(m[mask_off + n:] == 0x5A)
    assert np.all(m[mask_off: mask_off + n] <= 1)
    return m[mask_off: mask_off + n].astype(bool)


def _dev(a, cuda):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).to(cuda)


def _shifted(a, cuda):
    """A device view of `a` starting one row (12 bytes) into its buffer: not 16-byte aligned."""
    import torch
    buf = torch.from_numpy(np.r_[np.zeros((1, 3), F32), a]).to(cuda)
    v = buf[1:]
    assert v.data_ptr() % 16 == 12
    return v


def assert_dense(got, want, what=""):
    assert np.array_equal(got[0], want[0]), what
    assert np.array_equal(got[1], want[1]), what
    assert got[2] == want[2], what


def pct_for(n, min_points):
    """A threshold percentage for which density_filter computes exactly this min_points."""
    p = (min_points + 0.5) / n * 100.0
    assert int(n * (p / 100.0)) == min_points
    return p


# ------------------------------------------------------------------------------------------------ builders
def _f32(a):
    a = np.ascontiguousarray(a, dtype=F32)
    a.setflags(write=False)
    return a


def _rows(q, rng):
    """Points strictly inside voxels q (voxel 1.0), at fractions that are exact in float32 up to 2^22."""
    return q + rng.choice(np.array([0.25, 0.5, 0.75]), q.shape)


FORMS = {   # name: (lowest voxel, extent), voxel 1.0
    "smem": ((-16, -16, -12), (32, 32, 24)),             # 24 576 cells: the largest shared-memory histogram
    "smem_next": ((-3, -1755, 0), (7, 3511, 1)),         # 24 577 cells: the smallest box of the aggregation kernel
    "agg": ((100, 100, 100), (40, 50, 60)),
    "hash": ((-50_000, -70_000, -3), (100_001, 140_001, 7)),
    "wide": ((-2, -1_000_000, -2), (5, 2_500_001, 5)),
}
FORM_PATH = {"smem": "smem", "smem_next": "agg", "agg": "agg", "hash": "hash", "wide": "wide"}


def _grid_extra(form):
    """Workspace added so that a grid form reaches its kernel at any n (the default grows with n)."""
    return 0 if FORM_PATH[form] in ("hash", "wide") else int(np.prod(FORMS[form][1])) * 4 + 256


@functools.lru_cache(None)
def form_cloud(form, n):
    """Rows 0 and 1 are the box corners.  Big clouds: 8 hot voxels with 40 % of the rows, one voxel E with exactly
    E_COUNT rows at random positions, the rest uniform over the box.  Small clouds: random voxels, half of them
    repeats of an earlier row's voxel."""
    lo, ext = (np.array(v, np.int64) for v in FORMS[form])
    rng = np.random.default_rng([7, n, len(form), int(ext[1])])
    q = lo + (rng.random((n, 3)) * ext).astype(np.int64)
    q[0] = lo
    if n >= 2:
        q[1] = lo + ext - 1
    if n >= 1000:
        hot = lo + (rng.random((8, 3)) * ext).astype(np.int64)
        rows = rng.permutation(np.arange(2, n))
        nh = int(0.4 * n)
        q[rows[:nh]] = hot[rng.integers(0, 8, nh)]
        e = lo + ext // 3
        q[np.all(q == e, axis=1)] = lo
        q[rows[nh: nh + E_COUNT]] = e
    else:
        for i in range(2, n):
            if rng.random() < 0.5:
                q[i] = q[rng.integers(0, i)]
    return _f32(_rows(q, rng))


def count_mins(n):
    return (0, 1, 2, E_COUNT - 1, E_COUNT, E_COUNT + 1) if n >= 1000 else (0, 1, 2)


COUNT_CASES = [(f, n) for f in FORMS for n in COUNT_NS if n >= 2 or f == "smem"]
FLUSH_N, FLUSH_THR = 40 * AGG_ROWS, 28
FLUSH_BOX = {"smem": (20, 20, 20), "agg": (30, 40, 50)}


@functools.lru_cache(None)
def flush_cloud(form):
    """40 CTAs of 2 048 rows (both kernels cut the cloud so at this n).  Six voxels H get 3 rows in each of 10 CTAs
    (30 rows, so every partial sum is a multiple of 3 and the crossing add of thr = 28 or 29 never lands on it); one
    voxel E gets 2 rows in each of 14 CTAs (exactly 28); the rest is spread over the other voxels."""
    rng = np.random.default_rng(11 + len(form))
    ext = np.array(FLUSH_BOX[form])
    special = [np.array([1, 1, 1]) + i for i in range(7)]           # H0..H5, then E
    q = (rng.random((FLUSH_N, 3)) * ext).astype(np.int64)
    for s in special:
        hit = np.all(q == s, axis=1)
        q[hit] = (q[hit] + [0, 0, 10]) % ext
    q[0], q[1] = 0, ext - 1
    for i, s in enumerate(special):
        per, nb = (3, 10) if i < 6 else (2, 14)
        for b in rng.choice(np.arange(1, 40), nb, replace=False):
            rows = b * AGG_ROWS + rng.choice(AGG_ROWS, per, replace=False)
            q[rows] = s
    return _f32(_rows(q, rng))


FULL_BLOCKS, FULL_DISTINCT = 16, 1_400


@functools.lru_cache(None)
def agg_full_table():
    """Aggregation box of 60 000 cells; each 2 048-row CTA hits 1 400 distinct cells and puts its other 648 rows in
    one hot voxel, in random order: the shared table fills, and rows go to the global fallback."""
    rng = np.random.default_rng(12)
    ext = np.array([30, 40, 50])
    hot = np.array([15, 20, 25])
    blocks = []
    for b in range(FULL_BLOCKS):
        flat = rng.choice(int(np.prod(ext)), FULL_DISTINCT, replace=False)
        cells = np.stack(np.unravel_index(flat, ext), axis=1)
        cells = cells[~np.all(cells == hot, axis=1)]
        blk = np.r_[cells, np.repeat(hot[None], AGG_ROWS - len(cells), axis=0)]
        blocks.append(blk[rng.permutation(AGG_ROWS)])
    q = np.concatenate(blocks)
    q[0], q[-1] = 0, ext - 1
    return _f32(_rows(q, rng))


KEY_EXTENTS = (AXIS_LIM - 1, AXIS_LIM, AXIS_LIM + 1)


@functools.lru_cache(None)
def key_width_cloud(axis, ext):
    """Extent `ext` voxels on y (axis 1) or z (axis 2), 3 on the others.  A = the far end of that axis (5 rows);
    B = the voxel a 21-bit field overflowing from A would alias: (1, 0, 0) for y, (0, 1, 0) for z (3 rows); C = the
    origin (2 rows); 200 random rows."""
    rng = np.random.default_rng([13, axis, ext])
    a = np.zeros(3, np.int64)
    a[axis] = ext - 1
    b = np.zeros(3, np.int64)
    b[axis - 1] = 1
    span = np.array([3, 3, 3])
    span[axis] = ext
    q = np.r_[np.repeat(a[None], 5, 0), np.repeat(b[None], 3, 0), np.zeros((2, 3), np.int64),
              (rng.random((200, 3)) * span).astype(np.int64), span[None] - 1]
    return _f32(_rows(q, rng)), a, b


@functools.lru_cache(None)
def same_column_cloud():
    """Two-word keys: a y extent of 3 000 001 voxels; 24 000 rows in 40 (x, y) columns, 60 z values each, so most
    slot lookups find their own first word with another z."""
    rng = np.random.default_rng(14)
    cols = np.stack([rng.integers(0, 3, 40), rng.integers(0, 3_000_000, 40)], axis=1)
    pick = rng.integers(0, 40, 24_000)
    q = np.c_[cols[pick], rng.integers(0, 60, 24_000)]
    q[0], q[1] = (0, 0, 0), (2, 3_000_000, 59)
    return _f32(_rows(q, rng))


FACE_VOXELS = (0.1, 0.38, 1.1, 1.0, 2.0)
FACE_VARIANTS = ("smem", "agg", "hash")
INEXACT_VOXELS = (0.1, 0.38, 1.1)      # voxels whose reciprocal is not exact in float32


def _face_values(voxel, ks):
    """k * voxel in float32, one ulp below, and the values a few ulp around it whose float32 quotient rounds up to an
    integer although the exact quotient lies below it."""
    v = F32(voxel)
    on = ks.astype(F32) * v
    below = np.nextafter(on, F32(-np.inf))
    near = np.concatenate([on + j * np.spacing(on) for j in range(-4, 5)]).astype(F32)
    with np.errstate(invalid="ignore"):
        up = near[np.floor(near / v) != np.floor(near.astype(np.float64) / np.float64(v))]
    return np.r_[on, below, up, F32(0.0), F32(-0.0)].astype(F32)


@functools.lru_cache(None)
def faces_cloud(voxel, variant):
    """Coordinates on voxel faces: x from k in [-300, 300], y and z from k in [-1, 1] (smem) or [-6, 6]; the hash
    variant adds two far corners."""
    rng = np.random.default_rng([15, int(voxel * 100), len(variant)])
    xs = _face_values(voxel, np.arange(-300, 301))
    yz = _face_values(voxel, np.arange(-1, 2) if variant == "smem" else np.arange(-6, 7))
    n = 30_000
    xyz = np.c_[rng.choice(xs, n), rng.choice(yz, n), rng.choice(yz, n)]
    xyz = np.r_[xyz, [[0.0, -0.0, 0.0], [-0.0, -0.0, -0.0]]]
    if variant == "hash":
        xyz = np.r_[xyz, [[-1e5, -1e5, -1e5], [1e5, 1e5, 1e5]]]
    return _f32(xyz)


@functools.lru_cache(None)
def faces_keep(voxel, variant):
    """Half of the cloud's voxels, at random."""
    u = np.unique(voxels(faces_cloud(voxel, variant), voxel), axis=0)
    return u[np.random.default_rng(19).random(len(u)) < 0.5]


def _face_extra(voxel, variant):
    if variant == "hash":
        return 0
    _, dim = box(faces_cloud(voxel, variant), voxel)
    return int(np.prod(dim)) * 4 + 256


MEMBER_BOXES = {"2^27": (512, 512, 512), "2^27+1": (81, 1_657_009, 1)}     # 81 * 1 657 009 = 2^27 + 1


@functools.lru_cache(None)
def member_box_case(name):
    """Kept voxels: the 8 corners of the box and 300 random voxels in it.  Points: one in each kept voxel, 2 000
    random in the box, one just outside each of the six sides, and one on each face (coordinate k * voxel)."""
    rng = np.random.default_rng(16 + len(name))
    ext = np.array(MEMBER_BOXES[name])
    lo = np.array([-7, 3, -100])
    corners = np.array([[x, y, z] for x in (0, 1) for y in (0, 1) for z in (0, 1)]) * (ext - 1)
    keep = lo + np.r_[corners, (rng.random((300, 3)) * ext).astype(np.int64)]
    q = np.r_[keep, lo + (rng.random((2_000, 3)) * ext).astype(np.int64)]
    mid = lo + ext // 2
    out = []
    for a in range(3):
        for side in (lo[a] - 1, lo[a] + ext[a]):
            p = mid.copy()
            p[a] = side
            out.append(p)
    pts = np.r_[_rows(np.r_[q, out], rng), lo[None] + 0.0, (lo + ext)[None] + 0.0, (lo + ext - 1)[None] + 0.0]
    return _f32(pts), keep.astype(np.int64)


def with_far(keep):
    """The keep set plus one voxel 10^6 away on x and 10^3 on y, where no point lies: its box exceeds 2^27 voxels,
    so the keep set becomes a hash set."""
    return np.r_[keep, keep[:1] + [1_000_000, 1_000, 0]].astype(np.int64)


@functools.lru_cache(None)
def lanes_case():
    """Point i is kept iff bit (i % 4) of (i // 4) % 16 is set: every 4-bit lane pattern occurs, so a permutation of
    the four lanes of a uchar4 store changes the mask.  60 kept voxels spread over a 64^3 box (a 32 KiB bitmap, a
    1 KiB hash set), 60 others."""
    rng = np.random.default_rng(17)
    n = 4 * 16 * 40 + 7
    cand = np.unique((rng.random((200, 3)) * 64).astype(np.int64), axis=0)[rng.permutation(120)]
    keep = np.r_[cand[:60], [[0, 0, 0], [63, 63, 63]]]
    other = cand[60:120]
    want = np.array([((i // 4) % 16 >> (i % 4)) & 1 for i in range(n)], bool)
    q = np.where(want[:, None], keep[rng.integers(0, len(keep), n)], other[rng.integers(0, len(other), n)])
    return _f32(_rows(q, rng)), keep, want


STAGED_VOXEL = {"smem": 1.1, "grid_only": 0.38}     # the slider at 0.5 and at 0.9
STAGED_CUTS = (0, 0, 1, 3, 6, 1_001, 50_003, 100_001)   # slabs of 0, 1, 2, 3 rows, odd row offsets


@functools.lru_cache(None)
def staged_cloud():
    from gsx import synth
    return _f32(synth.xyz(100_001, "mixed"))


NAN_FORMS = ("smem", "agg", "hash", "wide")
NAN_PATTERNS = {"x": (0,), "y": (1,), "xyz": (0, 1, 2)}
NAN_N, NAN_THR = 60_000, 60                        # density_filter at 0.1 %: min_points = 60


@functools.lru_cache(None)
def nan_cloud(form, pattern, n_nan):
    """A dense blob in voxel (0, 0, 0) (around the origin) or in [100, 200]^3 (agg), a spread background, and for the
    hash forms two far corners.  `n_nan` rows get NaN on the pattern's axes; their finite coordinates lie in the blob's
    voxel, the densest kept one, so that a NaN aliased to voxel 0 lands in a kept voxel."""
    rng = np.random.default_rng([18, len(form), len(pattern), n_nan])
    centre = np.array([150.5, 150.5, 150.5]) if form == "agg" else np.array([0.5, 0.5, 0.5])
    spread = 25.0 if form == "agg" else 9.0
    xyz = np.r_[centre + rng.uniform(-0.45, 0.45, (NAN_N // 3, 3)),
                centre + rng.uniform(-spread, spread, (NAN_N - NAN_N // 3, 3))]
    if form == "hash":
        xyz[:2] = [[-1e5, -1e5, -1e5], [1e5, 1e5, 1e5]]
    if form == "wide":
        xyz[:2] = [[-1.0, -1.0, -1.0], [1.0, 3e6, 1.0]]
    rows = rng.choice(np.arange(2, NAN_N), n_nan, replace=False)
    xyz[rows] = np.array([0.5, 0.5, 0.5]) if form != "agg" else centre
    for a in NAN_PATTERNS[pattern]:
        xyz[rows, a] = np.nan
    return _f32(xyz)


def nan_keep(form, pattern):
    """The voxels a NaN row would alias to (NaN replaced by voxel 0) and those of 500 finite rows."""
    xyz = nan_cloud(form, pattern, NAN_THR - 1)
    nan_rows = np.isnan(xyz).any(axis=1)
    alias = voxels(np.nan_to_num(xyz[nan_rows], nan=0.0), 1.0)
    return np.unique(np.r_[alias, voxels(xyz[~nan_rows][2:502], 1.0)], axis=0)


# ------------------------------------------------------------------------------------------------ CPU: branch checks
@pytest.mark.parametrize("form,n", COUNT_CASES)
def test_count_form_reaches_branch(form, n):
    xyz = form_cloud(form, n)
    for mp in count_mins(n):
        cap = cap_of(n, mp)
        assert count_path(xyz, 1.0, mp, workspace_bytes(n, cap) + _grid_extra(form)) == FORM_PATH[form]
    q0, dim = box(xyz, 1.0)
    assert np.array_equal(q0, FORMS[form][0]) and np.array_equal(dim, FORMS[form][1] if n >= 2 else (1, 1, 1))
    if n >= 1000:
        u, c = np.unique(voxels(xyz, 1.0), axis=0, return_counts=True)
        assert np.sum(c == E_COUNT) >= 1 and np.sum((c >= E_COUNT - 1) & (c <= E_COUNT + 1)) <= 10
    if n == BIG_N:
        assert count_path(xyz, 1.0, E_COUNT) == FORM_PATH[form]          # the public API's own workspace
    if form == "smem":
        tail = n - 4 * (n // 4)
        assert smem_blocks(n)[0][0] == 0 and (tail > 0) == (n % 4 != 0)


def test_plain_grid_kernel_threshold():
    """k_vox_count<GridTable> runs for a box of >= 2^32 - 16 cells held as a grid, i.e. blob >= 4 (2^32 - 16) bytes.  The
    blob grows with the hash table of >= 2n slots (12 bytes each), so the smallest n that reaches it is stated here;
    the kernel is not run at that size."""
    n = 1
    while True:
        cap = n // 1 + 1
        if blob_bytes(workspace_bytes(n, cap), cap) >= 4 * PLAIN_CELLS:
            break
        n *= 2
    lo, hi = n // 2, n
    while hi - lo > 1:
        mid = (lo + hi) // 2
        if blob_bytes(workspace_bytes(mid, mid + 1), mid + 1) >= 4 * PLAIN_CELLS:
            hi = mid
        else:
            lo = mid
    assert 200_000_000 < hi < 700_000_000
    cap = hi + 1
    assert blob_bytes(workspace_bytes(hi, cap), cap) >= 4 * PLAIN_CELLS > blob_bytes(workspace_bytes(lo, lo + 1), lo + 1)


@pytest.mark.parametrize("form", ("smem", "agg"))
def test_flush_cloud_reaches_branch(form):
    xyz = flush_cloud(form)
    assert count_path(xyz, 1.0, FLUSH_THR) == form
    assert smem_blocks(FLUSH_N, H100_SMS) == [(b * AGG_ROWS, (b + 1) * AGG_ROWS) for b in range(40)]
    assert smem_blocks(FLUSH_N, 114) == smem_blocks(FLUSH_N, H100_SMS)     # PCIe H100: the same cut
    q = voxels(xyz, 1.0)
    for i in range(7):
        s = np.array([1, 1, 1]) + i
        blk = np.flatnonzero(np.all(q == s, axis=1)) // AGG_ROWS
        per = np.bincount(blk)
        per = per[per > 0]
        if i < 6:   # 10 CTAs x 3: partial sums 3, 6, ..., 30 skip 28 and 29
            assert len(per) == 10 and np.all(per == 3)
        else:       # exactly thr, in 14 CTAs of 2
            assert len(per) == 14 and np.all(per == 2)


def test_agg_full_table_reaches_branch():
    xyz = agg_full_table()
    assert count_path(xyz, 1.0, 2) == "agg"
    _, dim = box(xyz, 1.0)
    q = voxels(xyz, 1.0)
    for b in range(FULL_BLOCKS):
        blk = q[b * AGG_ROWS: (b + 1) * AGG_ROWS]
        assert len(np.unique(blk, axis=0)) > AGG_SLOTS + 300
        assert np.sum(np.all(blk == [15, 20, 25], axis=1)) > 600


@pytest.mark.parametrize("axis", (1, 2))
@pytest.mark.parametrize("ext", KEY_EXTENTS)
def test_key_width_reaches_branch(axis, ext):
    xyz, a, b = key_width_cloud(axis, ext)
    _, dim = box(xyz, 1.0)
    assert dim[axis] == ext
    assert count_path(xyz, 1.0, 4) == ("hash" if ext < AXIS_LIM else "wide")
    # 21-bit fields: A's field on `axis` overflows into the next one up exactly when ext - 1 == 2^21
    pack = lambda r: (int(r[0]) << 42) + (int(r[1]) << 21) + int(r[2])
    assert (pack(a) == pack(b)) == (ext == AXIS_LIM + 1)
    keep = np.array([a, [0, 0, 0]])
    assert member_path(keep, member_ws(keep)) == "bitmap"
    assert member_path(keep, hash_set_bytes(keep)) == ("hash_wide" if ext - 1 >= AXIS_LIM else "hash")


def test_extent_limit_reaches_refusal():
    ok = _f32([[0.0, 0.0, 0.0], [2147483520.0, 0.0, 0.0]])
    bad = _f32([[0.0, 0.0, 0.0], [0.0, 0.0, 2147483648.0]])
    assert box(ok, 1.0)[1][0] == EXTENT_LIM - 127 and count_path(ok, 1.0, 1) == "wide"
    assert box(bad, 1.0)[1][2] == EXTENT_LIM + 1 and count_path(bad, 1.0, 1) == "error"


def test_same_column_reaches_branch():
    xyz = same_column_cloud()
    assert count_path(xyz, 1.0, 5) == "wide"
    q = voxels(xyz, 1.0)
    cols, per_col = np.unique(q[:, :2], axis=0, return_counts=True)
    zs = [len(np.unique(q[np.all(q[:, :2] == c, axis=1), 2])) for c in cols[per_col > 100]]
    assert len(zs) >= 30 and min(zs) >= 50


@pytest.mark.parametrize("voxel", FACE_VOXELS)
@pytest.mark.parametrize("variant", FACE_VARIANTS)
def test_faces_reach_branch(voxel, variant):
    xyz = faces_cloud(voxel, variant)
    n = len(xyz)
    ws = workspace_bytes(n, cap_of(n, 1)) + _face_extra(voxel, variant)
    assert count_path(xyz, voxel, 1, ws) == variant
    v = F32(voxel)
    assert np.any(xyz == 0) and np.any(np.signbit(xyz) & (xyz == 0)) and np.any(xyz < 0)
    on = np.floor(xyz / v) == xyz / v
    assert on.sum() > 1000 and (np.floor(xyz / v) * v == xyz).sum() > 1000
    if voxel in INEXACT_VOXELS:
        f32q = np.floor(xyz / v)
        f64q = np.floor(xyz.astype(np.float64) / np.float64(v))
        assert np.sum(f32q != f64q) >= 50                    # rounds up to an integer: the float32 quotient decides
        recip = np.floor(xyz * (F32(1.0) / v))
        assert np.sum(recip != f32q) >= 10                   # x * (1 / voxel) would put these rows elsewhere
    keep = faces_keep(voxel, variant)
    assert member_path(keep, member_ws(keep)).startswith("hash" if variant == "hash" else "bitmap")
    assert member_path(with_far(keep), member_ws(with_far(keep))).startswith("hash")


@pytest.mark.parametrize("name", MEMBER_BOXES)
def test_member_box_reaches_branch(name):
    xyz, keep = member_box_case(name)
    d = keep.max(axis=0) - keep.min(axis=0) + 1
    assert int(np.prod(d)) == MAX_KEEP_BITS + (name == "2^27+1")
    want = "bitmap" if name == "2^27" else "hash"
    assert member_path(keep, member_ws(keep)) == want
    assert member_path(keep, hash_set_bytes(keep)) == "hash"
    q = voxels(xyz, 1.0)
    lo, hi = keep.min(axis=0), keep.max(axis=0)
    for a in range(3):                                      # outside on all six sides, and on the faces
        assert np.any(q[:, a] == lo[a] - 1) and np.any(q[:, a] == hi[a] + 1)
        assert np.any(q[:, a] == lo[a]) and np.any(q[:, a] == hi[a])


def test_member_lanes_reach_branch():
    xyz, keep, want = lanes_case()
    assert np.array_equal(ref_member(xyz, 1.0, keep), want)
    g = want[: 4 * (len(want) // 4)].reshape(-1, 4)
    assert np.any(g[:, 1] != g[:, 2]) and np.any(g[:, 0] != g[:, 3])
    for n in (1, 2, 3, 4, 5, 6, 7, 1001, 1002, 1003, 1004):
        assert member_split(n, 0, 0) == (4 * (n // 4), n % 4)
        assert member_split(n, 12, 0) == (0, n) and member_split(n, 0, 1) == (0, n)
    assert member_path(keep, member_ws(keep)) == "bitmap" and member_path(keep, hash_set_bytes(keep)) == "hash"


@pytest.mark.parametrize("form", STAGED_VOXEL)
def test_staged_reaches_branch(form):
    xyz = staged_cloud()
    _, dim = box(xyz, STAGED_VOXEL[form])
    ncell = int(np.prod(dim))
    assert (ncell <= SMEM_CELLS) == (form == "smem")
    inner = dim - 4
    assert int(np.prod(inner)) > 0 and ((int(np.prod(inner)) <= SMEM_CELLS) == (form == "smem"))
    cuts = STAGED_CUTS
    assert {cuts[i + 1] - cuts[i] for i in range(len(cuts) - 1)} >= {0, 1, 2, 3}
    assert any(12 * c % 16 for c in cuts)


@pytest.mark.parametrize("form", NAN_FORMS)
@pytest.mark.parametrize("pattern", NAN_PATTERNS)
def test_nan_cloud_reaches_branch(form, pattern):
    xyz = nan_cloud(form, pattern, NAN_THR - 1)
    assert int(NAN_N * (pct_for(NAN_N, NAN_THR) / 100.0)) == NAN_THR
    assert count_path(xyz, 1.0, NAN_THR) == form
    q0, dim = box(xyz, 1.0)
    nan_rows = np.isnan(xyz).any(axis=1)
    assert nan_rows.sum() == NAN_THR - 1
    # voxel 0 in place of the NaN coordinate: where a key field that keeps only the low bits of INT64_MIN - q0 (= -q0)
    # would count these rows without an in-box test
    alias = voxels(np.nan_to_num(xyz[nan_rows], nan=0.0), 1.0)
    alias_in_box = np.all((alias >= q0) & (alias <= q0 + dim - 1), axis=1)
    assert alias_in_box.all() == (form != "agg") and not alias_in_box.any() == (form == "agg")
    with np.errstate(invalid="ignore"):
        want, info = oracle.density_mask(xyz, 1.0, pct_for(NAN_N, NAN_THR), keep_multicluster=True)
    assert info["clusters"] >= 1 and not want[nan_rows].any()
    if form != "agg":   # the aliased voxel is kept by the reference, so an aliasing kernel would keep the NaN rows
        kept_rows = want & np.all(voxels(xyz, 1.0) == alias[0], axis=1)
        assert kept_rows.sum() > 1000
    keep = nan_keep(form, pattern)
    assert member_path(keep, member_ws(keep)) == "bitmap"
    assert member_path(with_far(keep), member_ws(with_far(keep))) == "hash"
    refuse = nan_cloud(form, pattern, NAN_THR)
    nq = voxels(refuse, 1.0)[np.isnan(refuse).any(axis=1)]
    u, c = np.unique(nq, axis=0, return_counts=True)
    assert len(u) == 1 and c[0] == NAN_THR and u[0][NAN_PATTERNS[pattern][0]] == np.iinfo(np.int64).min   # dense


# ------------------------------------------------------------------------------------------------ GPU: exact equality
@pytest.mark.gpu
@pytest.mark.parametrize("form,n", COUNT_CASES)
def test_count_form_gpu(form, n, cuda, gsx_lib):
    from gsx import density
    xyz = form_cloud(form, n)
    x = _dev(xyz, cuda)
    extra = _grid_extra(form)
    for mp in count_mins(n):
        want = ref_dense(xyz, 1.0, mp)
        assert_dense(voxel_count(x, 1.0, mp, extra), want, (form, n, mp))
        if n in (3, 5, 2049, BIG_N):      # unaligned rows: the scalar loop of k_vox_count_smem
            assert_dense(voxel_count(_shifted(xyz, cuda), 1.0, mp, extra), want, (form, n, mp, "shifted"))
    if n == BIG_N:
        vox, cnt, nv, _ = density.dense_voxels(x, 1.0, E_COUNT)
        assert_dense((vox, cnt, nv), ref_dense(xyz, 1.0, E_COUNT))
        for multi in (True, False):
            want, info_o = oracle.density_mask(xyz, 1.0, pct_for(n, E_COUNT), keep_multicluster=multi)
            got, info = density.density_filter(x, 1.0, pct_for(n, E_COUNT), keep_multicluster=multi)
            assert info["clusters"] == info_o["clusters"] and info["max_len"] == info_o["max_len"]
            assert np.array_equal(got.cpu().numpy(), want)


@pytest.mark.gpu
@pytest.mark.parametrize("form", ("smem", "agg"))
def test_flush_crossings_gpu(form, cuda, gsx_lib):
    xyz = flush_cloud(form)
    x = _dev(xyz, cuda)
    for mp in (FLUSH_THR - 1, FLUSH_THR, FLUSH_THR + 1, 2):
        got = voxel_count(x, 1.0, mp)
        assert len(np.unique(got[0], axis=0)) == len(got[0])          # each dense voxel once
        assert_dense(got, ref_dense(xyz, 1.0, mp), mp)


@pytest.mark.gpu
def test_agg_full_table_gpu(cuda, gsx_lib):
    xyz = agg_full_table()
    x = _dev(xyz, cuda)
    for mp in (0, 2, 3, FULL_BLOCKS * 600):
        assert_dense(voxel_count(x, 1.0, mp), ref_dense(xyz, 1.0, mp), mp)


@pytest.mark.gpu
@pytest.mark.parametrize("axis", (1, 2))
@pytest.mark.parametrize("ext", KEY_EXTENTS)
def test_key_width_gpu(axis, ext, cuda, gsx_lib):
    from gsx import density
    xyz, a, b = key_width_cloud(axis, ext)
    x = _dev(xyz, cuda)
    for mp in (0, 2, 4):
        assert_dense(voxel_count(x, 1.0, mp), ref_dense(xyz, 1.0, mp), mp)
    keep = np.array([a, [0, 0, 0]], np.int64)
    want = ref_member(xyz, 1.0, keep)
    assert want.sum() == 7
    assert np.array_equal(density.member_mask(x, 1.0, keep).cpu().numpy(), want)
    assert np.array_equal(member_raw(x, 0, len(xyz), 1.0, keep, hash_set_bytes(keep)), want)


@pytest.mark.gpu
def test_extent_limit_gpu(cuda, gsx_lib):
    from gsx import density
    from gsx._abi import GsxError
    ok = _f32([[0.0, 0.0, 0.0], [2147483520.0, 0.0, 0.0], [0.25, 0.0, 0.0]])
    assert_dense(voxel_count(_dev(ok, cuda), 1.0, 2), ref_dense(ok, 1.0, 2))
    with pytest.raises(GsxError, match="2\\^31"):
        voxel_count(_dev(_f32([[0.0, 0.0, 0.0], [0.0, 0.0, 2147483648.0]]), cuda), 1.0, 1)
    keep = np.array([[0, 0, 0], [0, EXTENT_LIM, 0]], np.int64)
    with pytest.raises(GsxError, match="2\\^31"):
        density.member_mask(_dev(ok, cuda), 1.0, keep)


@pytest.mark.gpu
def test_same_column_gpu(cuda, gsx_lib):
    xyz = same_column_cloud()
    x = _dev(xyz, cuda)
    for mp in (0, 5, 8, 12):
        assert_dense(voxel_count(x, 1.0, mp), ref_dense(xyz, 1.0, mp), mp)


@pytest.mark.gpu
@pytest.mark.parametrize("voxel", FACE_VOXELS)
@pytest.mark.parametrize("variant", FACE_VARIANTS)
def test_faces_gpu(voxel, variant, cuda, gsx_lib):
    from gsx import density
    xyz = faces_cloud(voxel, variant)
    x = _dev(xyz, cuda)
    extra = _face_extra(voxel, variant)
    for mp in (0, 2, 3):
        assert_dense(voxel_count(x, voxel, mp, extra), ref_dense(xyz, voxel, mp), (voxel, mp))
    keep = faces_keep(voxel, variant)
    want = ref_member(xyz, voxel, keep)
    assert np.array_equal(density.member_mask(x, voxel, keep).cpu().numpy(), want)
    assert np.array_equal(density.member_mask(x, voxel, with_far(keep)).cpu().numpy(), want)


@pytest.mark.gpu
@pytest.mark.parametrize("name", MEMBER_BOXES)
def test_member_box_gpu(name, cuda, gsx_lib):
    from gsx import density
    xyz, keep = member_box_case(name)
    x = _dev(xyz, cuda)
    want = ref_member(xyz, 1.0, keep)
    assert 300 < want.sum() < len(xyz) - 1000
    assert np.array_equal(density.member_mask(x, 1.0, keep).cpu().numpy(), want)
    assert np.array_equal(member_raw(x, 0, len(xyz), 1.0, keep, hash_set_bytes(keep)), want)
    assert np.array_equal(member_raw(x, 1, len(xyz) - 1, 1.0, keep, member_ws(keep), 1), want[1:])


@pytest.mark.gpu
def test_member_lanes_and_tails_gpu(cuda, gsx_lib):
    """n % 4 in {0, 1, 2, 3}, n < 4, xyz 16-byte aligned or not, mask 4-byte aligned or not, bitmap and hash set."""
    xyz, keep, want = lanes_case()
    x = _dev(xyz, cuda)
    for ws in (member_ws(keep), hash_set_bytes(keep)):
        assert np.array_equal(member_raw(x, 0, len(xyz), 1.0, keep, ws), want)
        for n in (1, 2, 3, 4, 5, 6, 7, 1001, 1002, 1003, 1004):
            for row0 in (0, 1, 4):
                for mask_off in (0, 1, 4):
                    got = member_raw(x, row0, n, 1.0, keep, ws, mask_off)
                    assert np.array_equal(got, want[row0: row0 + n]), (ws, n, row0, mask_off)


@pytest.mark.gpu
@pytest.mark.parametrize("form", STAGED_VOXEL)
def test_staged_gpu(form, cuda, gsx_lib):
    import torch
    from gsx import density
    xyz = staged_cloud()
    voxel = STAGED_VOXEL[form]
    x = _dev(xyz, cuda)
    q0, dim = box(xyz, voxel)
    q0d, dimd = density.voxel_range(np.r_[np.fmin.reduce(xyz, 0), np.fmax.reduce(xyz, 0)], voxel)
    assert np.array_equal(q0d, q0) and np.array_equal(dimd, dim)
    for bq0, bdim in ((q0, dim), (q0 + 2, dim - 4)):     # the whole box, and one 2 voxels smaller on every side
        grid = torch.zeros(int(np.prod(bdim)), dtype=torch.int32, device=cuda)
        oob = 0
        for a, b in zip(STAGED_CUTS[:-1], STAGED_CUTS[1:]):
            oob += int(density.grid_count(x[a:b], voxel, bq0, bdim, grid).item())
        want_grid, want_oob = ref_grid(xyz, voxel, bq0, bdim)
        assert np.array_equal(grid.cpu().numpy(), want_grid) and oob == want_oob
        assert (want_oob == 0) == (bdim is dim)
        inb = np.all((voxels(xyz, voxel) >= bq0) & (voxels(xyz, voxel) <= bq0 + bdim - 1), axis=1)
        for mp in (0, 1, 50):
            vox, cnt, nv = density.grid_dense(grid, bq0, bdim, mp, len(xyz))
            assert_dense((vox, cnt, nv), ref_dense(xyz[inb], voxel, mp), (mp, oob))


@pytest.mark.gpu
@pytest.mark.parametrize("form", NAN_FORMS)
@pytest.mark.parametrize("pattern", NAN_PATTERNS)
def test_nan_rows_gpu(form, pattern, cuda, gsx_lib):
    import torch
    from gsx import density
    from gsx._abi import GsxError
    xyz = nan_cloud(form, pattern, NAN_THR - 1)
    x = _dev(xyz, cuda)
    nan_rows = np.isnan(xyz).any(axis=1)
    for mp in (NAN_THR, NAN_THR + 1, 1_000):     # below NAN_THR the NaN rows alone are refused
        assert_dense(voxel_count(x, 1.0, mp), ref_dense(xyz, 1.0, mp), mp)
    vox, cnt, nv, _ = density.dense_voxels(x, 1.0, NAN_THR)
    assert_dense((vox, cnt, nv), ref_dense(xyz, 1.0, NAN_THR))
    with np.errstate(invalid="ignore"):
        want, info_o = oracle.density_mask(xyz, 1.0, pct_for(NAN_N, NAN_THR), keep_multicluster=True)
    got, info = density.density_filter(x, 1.0, pct_for(NAN_N, NAN_THR), keep_multicluster=True)
    assert info["clusters"] == info_o["clusters"] and info["max_len"] == info_o["max_len"]
    assert np.array_equal(got.cpu().numpy(), want)
    # membership: a keep set holding the voxel a NaN would alias to (x or y replaced by voxel 0), bitmap and hash set
    keep = nan_keep(form, pattern)
    mwant = ref_member(xyz, 1.0, keep)
    assert not mwant[nan_rows].any()
    assert np.array_equal(density.member_mask(x, 1.0, keep).cpu().numpy(), mwant)
    assert np.array_equal(density.member_mask(x, 1.0, with_far(keep)).cpu().numpy(), mwant)
    # staged: the NaN rows are the out-of-box points
    q0, dim = box(xyz, 1.0)
    if np.prod(dim) <= 1 << 24:
        grid = torch.zeros(int(np.prod(dim)), dtype=torch.int32, device=cuda)
        oob = int(density.grid_count(x, 1.0, q0, dim, grid).item())
        assert oob == NAN_THR - 1 and np.array_equal(grid.cpu().numpy(), ref_grid(xyz, 1.0, q0, dim)[0])
    # refusal: min_points NaN rows in one voxel pattern
    xr = _dev(nan_cloud(form, pattern, NAN_THR), cuda)
    with pytest.raises(GsxError, match="non-finite"):
        density.dense_voxels(xr, 1.0, NAN_THR)
    with pytest.raises(GsxError, match="non-finite"):
        density.density_filter(xr, 1.0, pct_for(NAN_N, NAN_THR))


@pytest.mark.gpu
@pytest.mark.parametrize("value", (np.inf, -np.inf))
@pytest.mark.parametrize("form", ("smem", "hash"))
def test_inf_rows_refused_gpu(value, form, cuda, gsx_lib):
    from gsx import density
    from gsx._abi import GsxError
    xyz = nan_cloud(form, "x", 0).copy()
    xyz[100, 1] = value
    with pytest.raises(GsxError, match="non-finite"):
        density.dense_voxels(_dev(xyz, cuda), 1.0, NAN_THR)
