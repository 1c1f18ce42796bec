"""Generate tests/golden/g9_reference_stand_in_small.npz: a small run of the reference's own filter_sor_gpu and
_kmeans_taichi source under the serial `taichi` stand-in (ti_serial.py), stored with its inputs.

    python tests/golden/make_taichi_golden_g9.py REFERENCE_ROOT     (a checkout of francescofugazzi/3dgsconverter)

The script asserts that the oracle reproduces the reference's outputs before it writes the file.
"""
import sys
from pathlib import Path

import numpy as np

HERE = Path(__file__).resolve().parent
sys.path[:0] = [str(HERE), str(HERE.parent.parent)]
import ti_serial  # noqa: E402
import oracle  # noqa: E402


def main(ref_root):
    ref = ti_serial.import_reference_gpu_ops(ref_root)
    rng = np.random.default_rng(3)
    xyz = np.concatenate([rng.normal(0, 0.05, (250, 3)), rng.uniform(-2, 2, (150, 3))]).astype(np.float32)
    k, sigma = 12, 1.5
    mask = np.asarray(ref.filter_sor_gpu(xyz, k=k, threshold_factor=sigma), bool)
    assert np.array_equal(mask, oracle.sor_taichi_mask(xyz, k, sigma, "i32wrap"))
    X = rng.normal(size=(300, 5)).astype(np.float32)
    K, iters, seed = 7, 3, 11
    np.random.seed(seed)
    C, L = ref._kmeans_taichi(X, K, max_iter=iters)
    np.random.seed(seed)
    Co, Lo, _ = oracle.kmeans_lloyd(X, K, iters, init=X[np.random.choice(len(X), K, replace=False)])
    assert np.array_equal(L, Lo) and np.array_equal(np.asarray(C, np.float32).view(np.uint32), Co.view(np.uint32))
    np.savez_compressed(HERE / "g9_reference_stand_in_small.npz", sor_xyz=xyz, sor_k=np.int64(k),
                        sor_sigma=np.float64(sigma), sor_mask=mask, km_X=X, km_K=np.int64(K), km_iters=np.int64(iters),
                        km_seed=np.int64(seed), km_centroids=np.asarray(C, np.float32),
                        km_labels=np.asarray(L, np.int32))


if __name__ == "__main__":
    main(sys.argv[1])
