"""Is the K-Means result independent of buffer addresses / alignment / launch history?  (diagnostic)"""
import sys
from pathlib import Path
import torch
ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT)); sys.path.insert(0, str(ROOT / "3dgsconverter_b200"))
from gsx import kmeans as gk  # noqa: E402
dev = torch.device("cuda:0")
rows, D, K = 35503, 45, 256
g = torch.Generator(device=dev).manual_seed(556)
proto = torch.randn(1024, D, device=dev, generator=g) * 0.15
X = proto[torch.randint(0, 1024, (rows * 4,), device=dev, generator=g)] + 0.03 * torch.randn(rows * 4, D, device=dev, generator=g)
blk = X[:rows]
ini = X[:K].clone()
res = {}
for mode in ("tensor", "strict"):
    a = gk.kmeans_lloyd_batched(blk, [0, rows], K, 10, ini.reshape(1, K, D), assign=mode)
    b = gk.kmeans_lloyd_batched(blk.clone(), [0, rows], K, 10, ini.clone().reshape(1, K, D), assign=mode)
    big = torch.empty(rows * D + 7, device=dev)
    mis = big[3:3 + rows * D].view(rows, D)      # 12-byte offset: not 16-byte aligned
    mis.copy_(blk)
    c = gk.kmeans_lloyd_batched(mis, [0, rows], K, 10, ini.reshape(1, K, D), assign=mode)
    res[mode] = a
    print(mode, "clone equal:", torch.equal(a[1], b[1]), torch.equal(a[0].view(torch.int32), b[0].view(torch.int32)),
          "misaligned equal:", torch.equal(a[1], c[1]), torch.equal(a[0].view(torch.int32), c[0].view(torch.int32)))
print("tensor vs strict", torch.equal(res["tensor"][1], res["strict"][1]),
      torch.equal(res["tensor"][0].view(torch.int32), res["strict"][0].view(torch.int32)),
      int((res["tensor"][1] != res["strict"][1]).sum()))
# batched (as in bench c5) vs single
nch = 4
offs = [p * rows for p in range(nch + 1)]
init = torch.stack([X[offs[p]:offs[p] + K] for p in range(nch)])
C, L, cnt = gk.kmeans_lloyd_batched(X, offs, K, 10, init)
C1, L1, _ = gk.kmeans_lloyd_batched(X[offs[1]:offs[2]], [0, rows], K, 10, init[1:2])
print("batched chunk1 vs single:", torch.equal(L[offs[1]:offs[2]], L1), torch.equal(C[1].view(torch.int32), C1[0].view(torch.int32)))
