"""NumPy restatement of the SOG writer (SogFormat.write, formats/sog.py:249-639 of 3dgsconverter) up to the WebP
step, the inputs of tests/golden/g11_reference_sog_small.npz, and the comparison the tests use.

The writer's K-Means calls (gpu_ops.kmeans) go through `kmeans(data, k, max_iter) -> (centroids, labels)`; the default
is the oracle's Lloyd (oracle.kmeans_lloyd) with the reference's own init draw from the global NumPy RNG.  The SH
codebook fit goes through `codebook_fit(values) -> centres` (scikit-learn's MiniBatchKMeans by default, as at
sog.py:561).  Float32 semantics of NumPy 2: Python float constants are weak scalars, np.sqrt(2.0) is a float64 one."""
from __future__ import annotations

import hashlib

import numpy as np

MAIN_FILES = ("means_l.webp", "means_u.webp", "quats.webp", "scales.webp", "sh0.webp")
SHN_FILES = ("shN_centroids.webp", "shN_labels.webp")
SEED = 11


def oracle_kmeans(data, k, max_iter=10):
    import oracle
    c, labels, _ = oracle.kmeans_lloyd(data, k, max_iter)
    return c, labels


def sklearn_codebook_fit(values):
    from sklearn.cluster import MiniBatchKMeans
    return MiniBatchKMeans(n_clusters=256, n_init="auto").fit(values).cluster_centers_


def texture_size(n):
    width = int(np.ceil(np.sqrt(n) / 4) * 4)
    return width, int(np.ceil(n / width / 4) * 4)


def quantize_to_codebook(vals, cb):
    if len(cb) == 1:
        return np.zeros_like(vals, dtype=np.uint8)
    idx = np.clip(np.searchsorted(cb, vals), 0, len(cb) - 1)
    left = np.maximum(idx - 1, 0)
    use_left = np.abs(vals - cb[left]) < np.abs(vals - cb[idx])
    idx[use_left] = left[use_left]
    return idx.astype(np.uint8)


def _codebook_1d(values, kmeans):
    fit = values
    if len(values) > 50000:
        fit = values[np.random.choice(len(values), 50000, replace=False)]
    c, _ = kmeans(fit.reshape(-1, 1), 256, max_iter=20)
    return sorted(c.flatten())


def sh_bands(s, names):
    """sog.py:465-492 on the sorted records s."""
    if "f_rest_0" not in names:
        return 0
    count = sum(f"f_rest_{i}" in names for i in range(45))
    bands = 3 if count >= 45 else 2 if count >= 24 else 1 if count >= 9 else 0
    if bands == 0:
        return 0
    last = -1
    for i in range({3: 44, 2: 23, 1: 8}[bands], -1, -1):
        if f"f_rest_{i}" in names and np.any(s[f"f_rest_{i}"] != 0):
            last = i
            break
    return 3 if last >= 24 else 2 if last >= 9 else 1 if last >= 0 else 0


def encode(a, compression_level=0, codebook_fit=None, kmeans=None):
    """(textures {name: uint8 [h, w, 4]}, meta, order) of SogFormat.write for the records `a`."""
    kmeans = kmeans or oracle_kmeans
    codebook_fit = codebook_fit or sklearn_codebook_fit
    n = len(a)
    width, height = texture_size(n)
    order = np.lexsort((a["z"], a["y"], a["x"]))
    s = a[order]
    tex = {}

    with np.errstate(all="ignore"):
        lxyz = [np.sign(s[f]) * np.log(np.abs(s[f]) + 1.0) for f in "xyz"]
        mins = [np.min(v) for v in lxyz]
        maxs = [np.max(v) for v in lxyz]
        u = [np.clip((v - lo) / (hi - lo) * 65535, 0, 65535).astype(np.uint16) for v, lo, hi in zip(lxyz, mins, maxs)]
    lo_img = np.full((height * width, 4), 255, np.uint8)
    hi_img = np.full((height * width, 4), 255, np.uint8)
    for i in range(3):
        lo_img[:n, i] = u[i] & 0xFF
        hi_img[:n, i] = u[i] >> 8
    tex["means_l.webp"], tex["means_u.webp"] = lo_img, hi_img

    q = np.column_stack([s[f"rot_{i}"] for i in range(4)])
    with np.errstate(all="ignore"):
        qn = q / np.linalg.norm(q, axis=1, keepdims=True)
        max_idx = np.abs(qn).argmax(axis=1)
        qn *= np.sign(np.take_along_axis(qn, max_idx[:, None], axis=1).flatten()).reshape(-1, 1)
        qn *= np.sqrt(2.0)
        qb = np.clip((qn * 0.5 + 0.5) * 255.0, 0, 255).astype(np.uint8)
    keep = np.array([[1, 2, 3], [0, 2, 3], [0, 1, 3], [0, 1, 2]])[max_idx]
    quats = np.full((height * width, 4), 255, np.uint8)
    quats[:n, :3] = np.take_along_axis(qb, keep, axis=1)
    quats[:n, 3] = 252 + max_idx.astype(np.uint8)
    tex["quats.webp"] = quats

    scale_codebook = _codebook_1d(np.concatenate([s["scale_0"], s["scale_1"], s["scale_2"]]), kmeans)
    scb = np.array(scale_codebook)
    scales = np.zeros((height * width, 4), np.uint8)
    for i in range(3):
        scales[:n, i] = quantize_to_codebook(s[f"scale_{i}"], scb)
    scales[:n, 3] = 255
    tex["scales.webp"] = scales

    color_codebook = _codebook_1d(np.concatenate([s["f_dc_0"], s["f_dc_1"], s["f_dc_2"]]), kmeans)
    ccb = np.array(color_codebook)
    sh0 = np.zeros((height * width, 4), np.uint8)
    for i in range(3):
        sh0[:n, i] = quantize_to_codebook(s[f"f_dc_{i}"], ccb)
    with np.errstate(all="ignore"):
        sh0[:n, 3] = np.clip(1.0 / (1.0 + np.exp(-s["opacity"])) * 255, 0, 255).astype(np.uint8)
    tex["sh0.webp"] = sh0
    sizes = {name: (width, height) for name in MAIN_FILES}

    bands = sh_bands(s, a.dtype.names)
    shn = None
    if bands:
        coeffs = [0, 9, 24, 45][bands]
        sh = np.column_stack([s[f"f_rest_{i}"] for i in range(coeffs)]).astype(np.float32)
        try:
            level = int(compression_level)
        except Exception:  # noqa: BLE001
            level = 0
        official_standard_k = min(64, 2 ** int(np.floor(np.log2(n / 1024)))) * 1024
        target_k = min(65536 if level <= 3 else 16384 if level <= 6 else 4096, official_standard_k)
        target_k = max(256, target_k)
        num_chunks = max(1, min(64, n // 1024))
        chunk_size = int(np.ceil(n / num_chunks))
        k_per_chunk = max(16, int(np.ceil(target_k / num_chunks)))
        cents, labels = [], []
        for i in range(num_chunks):
            start, end = i * chunk_size, min((i + 1) * chunk_size, n)
            if start >= end:
                break
            c, lab = kmeans(sh[start:end], min(end - start, k_per_chunk), max_iter=10)
            labels.append(lab + sum(len(x) for x in cents))
            cents.append(c)
        centroids = np.vstack(cents)
        labels = np.concatenate(labels)
        P = len(centroids)
        codebook = sorted(np.asarray(codebook_fit(centroids.flatten().reshape(-1, 1))).flatten())
        idx = quantize_to_codebook(centroids.flatten(), np.array(codebook))
        w_c, h_c = 64 * coeffs, int(np.ceil(P / 64))
        cimg = np.full((w_c * h_c, 4), 255, np.uint8)
        pix = idx.reshape(P, 3, coeffs // 3).transpose(0, 2, 1).reshape(-1, 3)
        cimg[:len(pix), :3] = pix
        limg = np.zeros((height * width, 4), np.uint8)
        l16 = labels.astype(np.uint16)
        limg[:n, 0], limg[:n, 1], limg[:n, 3] = l16 & 0xFF, l16 >> 8, 255
        tex["shN_centroids.webp"], tex["shN_labels.webp"] = cimg, limg
        sizes["shN_centroids.webp"], sizes["shN_labels.webp"] = (w_c, h_c), (width, height)
        shn = {"count": int(P), "bands": int(bands), "codebook": [float(c) for c in codebook],
               "files": list(SHN_FILES)}

    meta = {"version": 2, "asset": {"generator": "gsconverter-sog"}, "count": n,
            "means": {"mins": [float(m) for m in mins], "maxs": [float(m) for m in maxs],
                      "files": ["means_l.webp", "means_u.webp"]},
            "scales": {"codebook": [float(c) for c in scale_codebook], "files": ["scales.webp"]},
            "quats": {"files": ["quats.webp"]},
            "sh0": {"codebook": [float(c) for c in color_codebook], "files": ["sh0.webp"]}}
    if shn:
        meta["shN"] = shn
    tex = {k: v.reshape(sizes[k][1], sizes[k][0], 4) for k, v in tex.items()}
    return tex, meta, order.astype(np.int32)


class Hashed:
    """A texture the golden keeps as SHA-256 and shape only (a large member that must match exactly)."""

    def __init__(self, sha256: str, shape):
        self.sha256, self.shape = sha256, tuple(int(x) for x in shape)


# (case, member) kept by hash: the level-0 / level-7 palettes of 'mixed' are ~1 MB of near-random indices
HASHED_MEMBERS = {("mixed_l0", "shN_centroids.webp"), ("mixed_l7", "shN_centroids.webp")}


def store_case(out: dict, case: str, tex: dict):
    """Put the textures of `case` into the golden dict `out`: by hash for HASHED_MEMBERS, as a reference to an earlier
    case's identical member (key `<case>_<member>_same_as`), or as the array itself."""
    for name, t in tex.items():
        if (case, name) in HASHED_MEMBERS:
            out[f"{case}_{name}_sha256"] = np.array(digest(t))
            out[f"{case}_{name}_shape"] = np.array(t.shape, np.int64)
            continue
        prev = next((k[: -len(name) - 1] for k, v in out.items()
                     if k.endswith("_" + name) and isinstance(v, np.ndarray) and v.dtype == np.uint8
                     and np.array_equal(v, t)), None)
        if prev is not None:
            out[f"{case}_{name}_same_as"] = np.array(prev)
        else:
            out[f"{case}_{name}"] = t


def check_hashed(got: np.ndarray, want: Hashed, name: str):
    assert got.shape == want.shape and got.dtype == np.uint8, (name, got.shape, want.shape)
    assert digest(got) == want.sha256, f"{name} differs from the reference's (SHA-256)"


def assert_sog_equal(got_tex, got_meta, want_tex, want_meta):
    """The parity contract: every texture byte and meta entry exact; meta.means mins/maxs equal in value (NaN equal to
    NaN), the sign of a zero bound being free because NumPy's own depends on where the zeros sit.
    A want_tex member may be a Hashed."""
    assert list(got_tex) == list(want_tex), (list(got_tex), list(want_tex))
    for name, want in want_tex.items():
        if isinstance(want, Hashed):
            check_hashed(got_tex[name], want, name)
            continue
        assert got_tex[name].shape == want.shape and got_tex[name].dtype == np.uint8, name
        g, w = got_tex[name].reshape(-1, 4), want.reshape(-1, 4)
        bad = np.flatnonzero(np.any(g != w, axis=1))
        assert bad.size == 0, f"{name}: {bad.size} pixels differ, first {bad[:10]}: {g[bad[:3]]} vs {w[bad[:3]]}"
    for key in ("mins", "maxs"):
        gv, wv = np.array(got_meta["means"][key]), np.array(want_meta["means"][key])
        assert np.array_equal(gv, wv, equal_nan=True), (key, gv, wv)
    strip = [{**m, "means": {**m["means"], "mins": None, "maxs": None}} for m in (got_meta, want_meta)]
    assert strip[0] == strip[1]


def rng_pack(state) -> np.ndarray:
    """np.random.get_state() as one float64 array (624 keys, pos, has_gauss, cached_gaussian) for an .npz."""
    return np.concatenate([state[1].astype(np.float64), [state[2], state[3], state[4]]])


def rng_unpack(v: np.ndarray):
    return ("MT19937", v[:624].astype(np.uint32), int(v[624]), int(v[625]), float(v[626]))


def rng_equal(a, b) -> bool:
    return a[0] == b[0] and np.array_equal(a[1], b[1]) and tuple(a[2:]) == tuple(b[2:])


def replay_fit(z, case):
    """codebook_fit that replays the fit recorded in the golden for `case`: checks its input and the RNG state it
    is called in, returns the recorded centres and leaves the RNG where MiniBatchKMeans left it."""
    def fit(values):
        assert digest(np.ascontiguousarray(values, np.float32)) == str(z[f"{case}_fit_input_sha256"]), \
            "the palette handed to the codebook fit differs from the reference's"
        assert rng_equal(np.random.get_state(), rng_unpack(z[f"{case}_rng_before_fit"])), \
            "the codebook fit is called in a different RNG state than in the reference"
        np.random.set_state(rng_unpack(z[f"{case}_rng_after_fit"]))
        return z[f"{case}_fit_centres"]
    return fit


def golden_case(z, case):
    """(textures, meta) the reference wrote for `case`, in member order; a member kept by hash is a Hashed."""
    import json
    tex = {}
    for m in (str(x) for x in z[f"{case}_members"]):
        if f"{case}_{m}_sha256" in z.files:
            tex[m] = Hashed(str(z[f"{case}_{m}_sha256"]), z[f"{case}_{m}_shape"])
        elif f"{case}_{m}_same_as" in z.files:
            tex[m] = z[f"{str(z[f'{case}_{m}_same_as'])}_{m}"]
        else:
            tex[m] = z[f"{case}_{m}"]
    return tex, json.loads(str(z[f"{case}_meta"]))


def digest(a: np.ndarray) -> str:
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def _midpoint_edges(a, seed):
    """Put scale and colour values exactly between two neighbouring codebook entries (the left-neighbour tie rule),
    at sorted positions the seeded fit subsample does not draw, so the codebooks stay what they were."""
    n = len(a)
    order = np.lexsort((a["z"], a["y"], a["x"]))
    s = a[order]
    np.random.seed(seed)
    picks = []
    for fields in (("scale_0", "scale_1", "scale_2"), ("f_dc_0", "f_dc_1", "f_dc_2")):
        values = np.concatenate([s[f] for f in fields])
        sel = np.random.choice(len(values), 50000, replace=False)
        cb = np.array(sorted(oracle_kmeans(values[sel].reshape(-1, 1), 256, 20)[0].flatten()))
        mid = (cb[:-1] + cb[1:]) / np.float32(2)
        tie = np.abs(mid - cb[:-1]) == np.abs(mid - cb[1:])
        free = np.setdiff1d(np.arange(len(values)), sel)[: int(tie.sum())]
        picks.append((fields, free, mid[tie]))
    for fields, free, vals in picks:
        for pos, v in zip(free, vals):
            a[fields[pos // n]][order[pos % n]] = v
    return a


def golden_inputs() -> dict:
    """The inputs of g11_reference_sog_small.npz, regenerated from gsx.synth (pinned by SHA-256), keyed by case:
    (records, compression_level, seed).  'mixed' -- 18 000 SH-3 rows (3N > 50 000: the fit subsample is drawn; 17
    chunks) with edge rows spliced in, at levels 0 and 7; 'deg1' -- 3 000 uniform rows whose f_rest_9..44 are zero;
    'sh1_80' -- 80 SH-1 rows (3N <= 256: both codebooks pass the fit data through; the palette is a passthrough);
    'planar' -- a cloud with constant z and no f_rest fields."""
    from gsx import synth
    a = synth.structured(18_000, "mixed")
    quats = [(0, 0, 0, 0), (-0.9, 0.1, 0.2, 0.3), (0.1, -0.2, -0.95, 0.1), (0.5, 0.5, 0.5, 0.5),
             (0.5, -0.5, 0.5, -0.5), (-0.5, 0.5, -0.5, 0.5), (0.0, 0.0, -0.0, -1.0), (3.0, -3.0, 1.0, 0.0),
             (1e-30, 0, 0, 0), (0.0, -0.0, 0.0, -0.0), (-0.6, 0.6, 0.3, 0.1)]
    for k, q in enumerate(quats):
        for i in range(4):
            a[f"rot_{i}"][3000 + 7 * k] = q[i]
    for k, v in enumerate((0.0, -0.0, 0.0, -0.0, 25.0, -25.0)):
        a[f"scale_{k % 3}"][4000 + k] = v
        a[f"f_dc_{k % 3}"][4100 + k] = v
    a["x"][5000:5003], a["y"][5000:5003], a["z"][5000:5003] = (-0.0, 0.0, -0.0), (0.0, -0.0, 0.0), (-0.0, -0.0, 0.0)
    for k, v in enumerate((200.0, -200.0, 88.0, -88.0, 0.0, -0.0)):
        a["opacity"][5100 + k] = v
    a = _midpoint_edges(a, SEED)
    d = synth.structured(3_000, "uniform")
    for i in range(9, 45):
        d[f"f_rest_{i}"] = 0.0
    p = synth.structured(2_000, "mixed", sh_degree=0)
    p["z"] = 1.5
    return {"mixed_l0": (a, 0, SEED), "mixed_l7": (a, 7, SEED), "deg1": (d, 0, SEED + 1),
            "sh1_80": (synth.structured(80, "mixed", sh_degree=1), 0, SEED + 2), "planar": (p, 0, SEED + 3)}
