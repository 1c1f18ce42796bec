"""Chunk-visit model of the SOR grid layout: in-bucket orders by in-cell Morton code, by in-cell Hilbert code (what
gsx_sor_build lays out) and a k-d leaf order.

The query kernel (k_sor_knn) prunes the 32-point chunks of a long hash bucket by their boxes.  For a query, the chunks
of its 27 probed long buckets whose box lower bound is below the final K-th neighbour d^2 must be scanned by any walk,
even one that starts with the final tau.  This script counts them for sampled queries of a seeded cloud, per query
class, under each order:

    python scripts/sor_layout_model.py --n 10000000 --kind mixed --queries 1000

k-d leaf layout: every segment "long bucket (> 64 points) clipped to one aligned 1024-point super" is laid out as a
k-d tree whose leaves are the aligned 32-point chunks.  A node [a, b) that does not lie inside one aligned chunk splits
at the chunk boundary kd_split(a, b) on the axis of its largest extent, and its m - a smallest points along that axis
go left.  Only the order inside a bucket changes, so the query's result (the multiset of the K smallest d^2 over the
probed buckets) would not.  kd_split / kd_segment_order / long_segments / check_kd_leaves state the rule as code.
"""
from __future__ import annotations

import argparse
import sys
import time
from pathlib import Path

import numpy as np

P1, P2, P3 = 73856093, 19349663, 83492791
SMALL_BUCKET = 64     # kSmallBucket: longer buckets are walked by chunk boxes
SUPER = 1024          # points per super box; a k-d segment is a long bucket clipped to one aligned super
CHUNK = 32


def kd_split(a: int, b: int) -> int:
    """The chunk boundary a node [a, b) splits at: the multiple of 32 nearest (a + b) / 2 (halves round up), clamped
    to the boundaries strictly inside (a, b).  The node must not lie inside one aligned chunk."""
    m = ((a + b + 32) >> 6) << 5
    lo, hi = ((a >> 5) + 1) << 5, ((b - 1) >> 5) << 5
    return min(max(m, lo), hi)


def _is_leaf(a: int, b: int) -> bool:
    return (a >> 5) == ((b - 1) >> 5)


def kd_segment_order(pts: np.ndarray, a: int, b: int) -> np.ndarray:
    """Permutation of the float32 points pts (the segment's positions [a, b)) into k-d leaf order: a node splits at
    kd_split on the axis of its largest extent (first of x, y, z on ties), its m - a smallest points go left."""
    out = np.empty(b - a, dtype=np.int64)
    stack = [(a, b, np.arange(b - a))]
    while stack:
        na, nb, ids = stack.pop()
        if _is_leaf(na, nb):
            out[na - a: nb - a] = ids
            continue
        m = kd_split(na, nb)
        q = pts[ids]
        ext = q.max(0) - q.min(0)
        ax = int(np.argmax(ext))
        ids = ids[np.argsort(q[:, ax], kind="stable")]
        stack.append((na, m, ids[: m - na]))
        stack.append((m, nb, ids[m - na:]))
    return out


def long_segments(starts: np.ndarray, ends: np.ndarray):
    """[a, b) of every long bucket (> SMALL_BUCKET points) clipped to each aligned super it overlaps."""
    for s, e in zip(starts.tolist(), ends.tolist()):
        if e - s <= SMALL_BUCKET:
            continue
        a = s
        while a < e:
            b = min(e, (a // SUPER + 1) * SUPER)
            yield a, b
            a = b


def check_kd_leaves(pts: np.ndarray, a: int, b: int) -> bool:
    """True iff the points at positions [a, b) are laid out by the split rule: every node splits at kd_split with
    its m - a smallest points (along an axis of largest extent) on the left.  Ties are accepted either way."""
    stack = [(a, b)]
    while stack:
        na, nb = stack.pop()
        if _is_leaf(na, nb):
            continue
        m = kd_split(na, nb)
        q = pts[na - a: nb - a]
        ext = q.max(0) - q.min(0)
        if not any(ext[ax] == ext.max() and q[: m - na, ax].max() <= q[m - na:, ax].min() for ax in range(3)):
            return False
        stack.append((na, m))
        stack.append((m, nb))
    return True


def bucket_hash(pos: np.ndarray, lo: np.ndarray, cell: float):
    """gi = floor((p - min) / cell) in float32, int64 hash mod n (the build's bucket); also the cell-relative part."""
    fr = (pos - lo) / np.float32(cell)
    fl = np.floor(fr)
    gi = fl.astype(np.int32).astype(np.int64)
    h = ((gi[:, 0] * P1) ^ (gi[:, 1] * P2) ^ (gi[:, 2] * P3)) % len(pos)
    return h, gi, fr - fl


def interleave(x, y, z, bits: int = 5):
    """Bits interleaved x first (bit b of x -> bit 3b + 2): the Morton code of (x, y, z)."""
    code = np.zeros(len(x), np.int64)
    for bt in range(bits):
        for ax, v in enumerate((x, y, z)):
            code |= ((v >> bt) & 1) << (3 * bt + (2 - ax))
    return code


def hilbert_code(s: np.ndarray, bits: int = 5) -> np.ndarray:
    """Hilbert index of integer sub-cells s [N, 3] in [0, 2^bits)^3: Skilling's transpose form, then interleaved
    (hilbert15 in gsx_sor.cu)."""
    x, y, z = (s[:, a].astype(np.int64) for a in range(3))
    q = 1 << (bits - 1)
    while q > 1:
        p = q - 1
        x = np.where(x & q, x ^ p, x)
        for i in (1, 2):
            v = y if i == 1 else z
            t = (x ^ v) & p
            hit = (v & q) != 0
            x, v = np.where(hit, x ^ p, x ^ t), np.where(hit, v, v ^ t)
            if i == 1:
                y = v
            else:
                z = v
        q >>= 1
    y = y ^ x
    z = z ^ y
    t = np.zeros_like(x)
    q = 1 << (bits - 1)
    while q > 1:
        t = np.where(z & q, t ^ (q - 1), t)
        q >>= 1
    return interleave(x ^ t, y ^ t, z ^ t, bits)


def cell_order(pos: np.ndarray, lo: np.ndarray, cell: float, curve: str = "hilbert", bits: int = 5):
    """A build sort order: (bucket, in-cell curve code, original index); curve "hilbert" is what gsx_sor_build sorts
    by (with its 15-bit code, i.e. up to 16.7 M points), "morton" the Z-order code it used before."""
    h, gi, sub = bucket_hash(pos, lo, cell)
    s = np.clip(sub * np.float32(1 << bits), 0, (1 << bits) - 1).astype(np.int64)
    code = hilbert_code(s, bits) if curve == "hilbert" else interleave(s[:, 0], s[:, 1], s[:, 2], bits)
    order = np.lexsort((np.arange(len(pos)), code, h))
    return order, h[order]


def bucket_ranges(sh: np.ndarray):
    """start / end of every occupied bucket of a bucket-sorted hash array."""
    brk = np.flatnonzero(np.diff(sh)) + 1
    starts = np.r_[0, brk]
    ends = np.r_[brk, len(sh)]
    return starts, ends


def kd_layout(sp: np.ndarray, starts: np.ndarray, ends: np.ndarray) -> np.ndarray:
    """Permutation of the Morton-ordered points sp into the k-d leaf layout."""
    perm = np.arange(len(sp))
    for a, b in long_segments(starts, ends):
        if not _is_leaf(a, b):
            perm[a:b] = a + kd_segment_order(sp[a:b], a, b)
    return perm


def chunk_boxes(sp: np.ndarray):
    n = len(sp)
    pad = (-n) % CHUNK
    x = np.concatenate([sp, np.repeat(sp[-1:], pad, 0)]).reshape(-1, CHUNK, 3)
    return x.min(1), x.max(1)


def probe_hash_i32(g: np.ndarray, n: int) -> np.ndarray:
    """gpu_ops.py probe hash with int32 wrapping products (the default hash mode)."""
    g = g.astype(np.int64)
    hv = [((g[:, a] * p) & 0xffffffff) for a, p in enumerate((P1, P2, P3))]
    h = (hv[0] ^ hv[1] ^ hv[2]).astype(np.uint32).view(np.int32).astype(np.int64)
    return h % n


def count_chunks(sp, starts, ends, bucket_of, cbox, q, gi, tau):
    """Chunks of the probed long buckets of query q whose box lower bound is below tau."""
    lo, hi = cbox
    offs = np.array([(dx, dy, dz) for dx in (-1, 0, 1) for dy in (-1, 0, 1) for dz in (-1, 0, 1)])
    hs = probe_hash_i32(gi[None, :] + offs, len(sp))
    cnt = 0
    for h in hs.tolist():
        bi = bucket_of.get(h)
        if bi is None:
            continue
        s, e = int(starts[bi]), int(ends[bi])
        if e - s <= SMALL_BUCKET:
            continue
        c = np.arange(s >> 5, ((e - 1) >> 5) + 1)
        d = np.maximum(np.maximum(lo[c] - q, q - hi[c]), 0.0)
        cnt += int(((d * d).sum(1) < tau).sum())
    return cnt


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--n", type=int, default=10_000_000)
    ap.add_argument("--kind", default="mixed", choices=["mixed", "uniform", "clustered"])
    ap.add_argument("--k", type=int, default=16)
    ap.add_argument("--queries", type=int, default=1000, help="sampled queries per class")
    ap.add_argument("--seed", type=int, default=7)
    a = ap.parse_args(argv)
    root = Path(__file__).resolve().parents[1]
    sys.path[:0] = [str(root), str(root / "3dgsconverter_b200")]
    import oracle
    from gsx import synth
    from scipy.spatial import cKDTree

    t0 = time.time()
    xyz = synth.xyz(a.n, a.kind)
    lo, cell = oracle.sor_cell_size(xyz)
    order, sh = cell_order(xyz, lo, cell, "morton")
    sp = xyz[order]
    starts, ends = bucket_ranges(sh)
    bucket_of = {int(h): i for i, h in enumerate(sh[starts].tolist())}
    t1 = time.time()
    perm = kd_layout(sp, starts, ends)
    sp_kd = sp[perm]
    t2 = time.time()
    hil, _ = cell_order(xyz, lo, cell, "hilbert")       # the same buckets, another order inside each
    boxes = {"morton": chunk_boxes(sp.astype(np.float64)), "hilbert": chunk_boxes(xyz[hil].astype(np.float64)),
             "kd32": chunk_boxes(sp_kd.astype(np.float64))}

    # query classes by the size of the query's own bucket
    own = np.repeat(ends - starts, ends - starts)          # bucket length at every sorted position
    rng = np.random.default_rng(a.seed)
    tree = cKDTree(xyz.astype(np.float64))
    _, gi_all, _ = bucket_hash(sp, lo, cell)
    print(f"n={a.n} kind={a.kind} cell={cell:.5g} buckets={len(starts)} long={(ends - starts > SMALL_BUCKET).sum()} "
          f"long-bucket points={(own > SMALL_BUCKET).mean():.1%}  (sort {t1 - t0:.1f} s, k-d layout {t2 - t1:.1f} s)")
    for name, sel in (("own bucket <= 64", own <= SMALL_BUCKET), ("own bucket > 64", own > SMALL_BUCKET)):
        cand = np.flatnonzero(sel)
        if len(cand) == 0:
            continue
        pick = rng.choice(cand, size=min(a.queries, len(cand)), replace=False)
        q = sp[pick].astype(np.float64)
        d, _ = tree.query(q, k=a.k + 1)
        tau = d[:, -1] ** 2                                 # final K-th neighbour d^2 (self excluded)
        res = {}
        for lay, cb in boxes.items():
            res[lay] = np.mean([count_chunks(sp, starts, ends, bucket_of, cb, q[i], gi_all[pick[i]], tau[i])
                                for i in range(len(pick))])
        rel = lambda lay: f"{res[lay] / res['morton'] - 1:+.1%}" if res["morton"] else "n/a"
        print(f"  {name:18s} share {sel.mean():5.1%}  queries {len(pick):5d}  chunks with lb < final tau: "
              f"morton {res['morton']:7.2f}  hilbert {res['hilbert']:7.2f} ({rel('hilbert')})  "
              f"kd32 {res['kd32']:7.2f} ({rel('kd32')})")


if __name__ == "__main__":
    main()
