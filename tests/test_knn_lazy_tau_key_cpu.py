"""CPU: lane-level models of the two forms k_sor_knn's exactness rests on besides DESIGN.md 4.2's pruning argument.

  * TopK::insert without a tau refresh: a scan step inserts every candidate that beat the tau of the step's START, so
    a later candidate may be >= the current K-th best.  The 32 lanes must still hold the 32 smallest values offered, in
    order -- hence the K smallest for every K <= 32 -- and the tau read after the step must be the true rank K-1.
  * the box key (lb & ~31) | lane: one minimum over the keys must name a lane whose box is nearest up to 32 ulp, the
    key's lower bound must never exceed the true one, and an exhausted key must fail `< tau` for every tau.
"""
import numpy as np

f32 = np.float32
D2LIM = np.uint32(0x60AD78EB).view(np.float32)
KEY_NONE = np.uint32(0xFFFFFFFF)


def lane_insert(v, x):
    """TopK<1>::insert: up = shfl_up(v, 1) with 0 entering lane 0; lanes holding more than x take max(up, x)."""
    up = np.concatenate([[f32(0)], v[:-1]])
    return np.where(v > x, np.maximum(up, x), v)


def scan_step(v, k, d2):
    """One serial scan step: the candidates that beat the tau of the step's start, in lane order, no refresh between."""
    tau = v[k - 1]
    for x in d2[(d2 > f32(1e-12)) & (d2 < tau)]:
        v = lane_insert(v, x)
    return v


def test_lazy_tau_keeps_the_32_smallest():
    rng = np.random.default_rng(11)
    for trial in range(300):
        k = int(rng.integers(1, 33))
        v = np.full(32, D2LIM, f32)
        offered = []
        for step in range(int(rng.integers(1, 12))):
            # few candidates per step (the serial path), drawn from a small set so that ties and repeats are common
            d2 = rng.choice(np.array([0.0, 0.25, 0.5, 0.5, 1.0, 2.0, 3.0, 7.0], f32) * f32(rng.integers(1, 4)),
                            int(rng.integers(0, 9))).astype(f32)
            tau = v[k - 1]
            offered += [x for x in d2 if x > f32(1e-12) and x < tau]
            v = scan_step(v, k, d2)
            want = np.sort(np.array(offered + [D2LIM] * 32, f32))[:32]
            assert np.array_equal(v, want), (trial, step, k)
            assert v[k - 1] == want[k - 1]


def knn_key(lb, lane):
    return (np.asarray(lb, f32).view(np.uint32) & ~np.uint32(31)) | np.uint32(lane)


def knn_key_lb(key):
    return (np.asarray(key, np.uint32) & ~np.uint32(31)).view(f32)


def test_truncated_key_is_a_conservative_lower_bound():
    rng = np.random.default_rng(12)
    lb = np.abs(rng.standard_normal(20_000)).astype(f32) ** 2
    lb[:100] = 0
    lb[100:200] = np.inf
    lanes = rng.integers(0, 32, len(lb))
    key = knn_key(lb, lanes)
    klb = knn_key_lb(key)
    assert np.all(klb <= lb) and np.all((key & np.uint32(31)) == lanes)
    assert np.all(lb.view(np.uint32).astype(np.int64) - klb.view(np.uint32).astype(np.int64) < 32)
    with np.errstate(invalid="ignore"):
        assert not np.any(knn_key_lb(KEY_NONE) < np.array([0, 1, D2LIM, np.inf], f32))   # a NaN: never < tau


def test_one_minimum_names_a_nearest_lane():
    rng = np.random.default_rng(13)
    for trial in range(2000):
        base = f32(rng.uniform(0.01, 4.0))
        # lower bounds a few ulp apart (the near-tie case) mixed with clearly different ones and exhausted lanes
        bits = base.view(np.uint32) + rng.integers(0, 80, 32).astype(np.uint32) * rng.integers(0, 2, 32).astype(np.uint32) * 1000
        bits = bits + rng.integers(0, 40, 32).astype(np.uint32)
        lb = bits.view(f32)
        live = rng.random(32) < 0.8
        key = np.where(live, knn_key(lb, np.arange(32)), KEY_NONE)
        m = key.min()
        if not live.any():
            assert m == KEY_NONE
            continue
        lane = int(m & np.uint32(31))
        assert live[lane] and key[lane] == m
        # every other live box is at most 31 ulp nearer than the one picked; ties in the key break by lane
        assert np.all(lb[live].view(np.uint32).astype(np.int64) > int(lb[lane].view(np.uint32)) - 32)
        # pruning at the minimum is safe: if its key bound is >= tau, every live box's true bound is >= tau
        for t in (lb[live].min(), np.nextafter(lb[live].min(), f32(np.inf)), knn_key_lb(m)):
            if not (knn_key_lb(m) < f32(t)):
                assert np.all(lb[live] >= f32(t))
