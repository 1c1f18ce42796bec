"""A NumPy/float32 emulation of the ALGORITHM of csrc/gsx_sor.cu's query kernel (test infrastructure).

Purpose: fuzz the exactness arguments of DESIGN.md §4.2 on the CPU, with small fan-outs so that the pruned paths
(bucket boxes, super -> chunk -> points walk, seed chunk, duplicate probes, wrapped probe hash) are exercised on
clouds of a few thousand points: nearest-first order, `lb >= tau` pruning with ties, multiplicity of buckets reached
by two probes, selection on d^2 with sqrt of the winners, the 1e10 sentinel.  The result must equal the brute-force
oracle (oracle/gsx_oracle.c) bit for bit.  Every float operation is a float32 NumPy scalar op in the kernel's order.
"""
import numpy as np

f32 = np.float32
P1, P2, P3 = 73856093, 19349663, 83492791
D2LIM = np.uint32(0x60AD78EB).view(np.float32)   # smallest float32 whose sqrt is >= 1e10f


def _probe_hash(nx, ny, nz, n, mode):
    if mode == "i32wrap":
        w = lambda v: ((int(v) + 2**31) % 2**32) - 2**31  # noqa: E731  wrap to int32
        h = w(nx * P1) ^ w(ny * P2) ^ w(nz * P3)
        return h % n                                       # Python modulo == Taichi's
    return ((nx * P1) ^ (ny * P2) ^ (nz * P3)) % n


def _d2(q, c):
    ax, ay, az = f32(q[0] - c[0]), f32(q[1] - c[1]), f32(q[2] - c[2])
    return f32(f32(f32(ax * ax) + f32(ay * ay)) + f32(az * az))


def _lb(q, lo, hi):
    d = [max(max(f32(lo[a] - q[a]), f32(q[a] - hi[a])), f32(0)) for a in range(3)]
    return f32(f32(f32(d[0] * d[0]) + f32(d[1] * d[1])) + f32(d[2] * d[2]))


def emulate(pos, k, mode="i32wrap", chunk=4, fan=4, small_bucket=6, morton_bits=2, flat_supers=0, group=32):
    """final_means float32[N] computed with the kernel's algorithm (chunk = points per chunk, fan = chunks per
    super, small_bucket = largest bucket scanned without box tests, flat_supers = kFlatSupers: a long bucket
    spanning fewer supers than this tests its chunk boxes directly, `group` at a time, without the super level)."""
    pos = np.ascontiguousarray(pos, dtype=np.float32)
    n = len(pos)
    lo = pos.min(0)
    ext = pos.max(0) - lo
    vol = np.prod(ext)
    if vol <= 0:
        vol = 1.0
    avg = max(1e-8, vol / n)
    cell = f32(max(float((avg * 32) ** (1.0 / 3.0)), 1e-4))
    fr = (pos - lo) / cell
    gi = np.floor(fr).astype(np.int32).astype(np.int64)
    h = ((gi[:, 0] * P1) ^ (gi[:, 1] * P2) ^ (gi[:, 2] * P3)) % n
    sub = np.minimum((fr - np.floor(fr)) * (1 << morton_bits), (1 << morton_bits) - 1).astype(np.int64)
    mort = np.zeros(n, np.int64)
    for b in range(morton_bits):
        for a in range(3):
            mort |= ((sub[:, a] >> b) & 1) << (3 * b + (2 - a))
    order = np.lexsort((np.arange(n), mort, h))            # stable sort by (hash, morton)
    sp = pos[order]
    sh = h[order]
    start, end = {}, {}
    for j, hv in enumerate(sh):
        start.setdefault(int(hv), j)
        end[int(hv)] = j + 1
    box = {hv: (sp[start[hv]:end[hv]].min(0), sp[start[hv]:end[hv]].max(0)) for hv in start}
    nchunk = (n + chunk - 1) // chunk
    cbox = [(sp[c * chunk:(c + 1) * chunk].min(0), sp[c * chunk:(c + 1) * chunk].max(0)) for c in range(nchunk)]
    sup = chunk * fan
    nsup = (n + sup - 1) // sup
    sbox = [(sp[s * sup:(s + 1) * sup].min(0), sp[s * sup:(s + 1) * sup].max(0)) for s in range(nsup)]
    K = min(k, 50)
    out = np.zeros(n, np.float32)
    stats = dict(scanned=0, visits=0)
    for i in range(n):
        q = sp[i]
        g = np.floor((q - lo) / cell).astype(np.int32)
        lst = [D2LIM] * K                                   # ascending list of the K best d^2

        def tau():
            return lst[K - 1]

        def scan(j0, j1):                                   # visit candidates [j0, j1)
            nonlocal lst
            for j in range(j0, j1):
                stats["scanned"] += 1
                d2 = _d2(q, sp[j])
                if d2 > f32(1.0e-12) and d2 < tau():
                    lst.append(d2)
                    lst.sort(kind="stable") if isinstance(lst, np.ndarray) else lst.sort()
                    lst = lst[:K]

        probes = []
        for dx in (-1, 0, 1):
            for dy in (-1, 0, 1):
                for dz in (-1, 0, 1):
                    hv = _probe_hash(int(g[0]) + dx, int(g[1]) + dy, int(g[2]) + dz, n, mode)
                    probes.append(hv if hv in start else None)
        stats["visits"] += sum(end[hv] - start[hv] for hv in probes if hv is not None)
        keys = [(_lb(q, *box[hv]) if hv is not None else None) for hv in probes]
        skip_chunk = -1
        h13 = probes[13]
        if h13 is not None and end[h13] - start[h13] > small_bucket and start[h13] <= i < end[h13]:
            skip_chunk = i // chunk
            scan(max(skip_chunk * chunk, start[h13]), min((skip_chunk + 1) * chunk, end[h13]))
        pending = [p for p in range(27) if keys[p] is not None]
        while pending:
            p = min(pending, key=lambda t: (keys[t], t))    # nearest box first, lowest lane on ties
            if not (keys[p] < tau()):
                break
            pending.remove(p)
            hv = probes[p]
            s, e = start[hv], end[hv]
            if e - s <= small_bucket:
                scan(s, e)
                continue
            skip = skip_chunk if p == 13 else -1
            fc, lc = s // chunk, (e - 1) // chunk
            def chunk_group(cands):                          # nearest chunk box first while it can still improve
                chunks = [(c, _lb(q, *cbox[c])) for c in cands if fc <= c <= lc and c != skip]
                chunks = [(c, l) for c, l in chunks if l < tau()]
                while chunks:
                    c, l = min(chunks, key=lambda t: (t[1], t[0]))
                    if not (l < tau()):
                        break
                    chunks.remove((c, l))
                    scan(max(c * chunk, s), min((c + 1) * chunk, e))

            if flat_supers > 0 and lc // fan - fc // fan < flat_supers:
                for cb in range(fc, lc + 1, group):
                    chunk_group(range(cb, cb + group))
                continue
            sups = [(sid, _lb(q, *sbox[sid])) for sid in range(fc // fan, lc // fan + 1)]
            # the kernel evaluates 32 supers at a time against the tau of that moment; emulate group-wise
            for g0 in range(0, len(sups), 32):
                grp = [(sid, lb) for sid, lb in sups[g0:g0 + 32] if lb < tau()]
                while grp:
                    sid, lb = min(grp, key=lambda t: (t[1], t[0]))
                    if not (lb < tau()):
                        break
                    grp.remove((sid, lb))
                    chunk_group(range(sid * fan, sid * fan + fan))
        d = [np.sqrt(v) for v in lst]                        # float32 sqrt of the winners only
        vals = [v for v in d if v < f32(0.9e10)]
        ssum = f32(0)
        for v in vals:
            ssum = f32(ssum + v)
        out[order[i]] = f32(ssum / f32(len(vals))) if vals else f32(0)
    return out, stats
