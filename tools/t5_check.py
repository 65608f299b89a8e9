"""wgmma residual block: bitwise batch independence (n = 4 in one call vs four calls of n = 1), run-to-run determinism and
the error pattern against the exact-FMA kernel, by tile row."""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from jukebox_b200._lib import lib, check, ptr, stream_ptr  # noqa: E402

for C, T, dil in ((64, 4096, 3), (64, 32768, 27), (32, 32768, 9), (64, 262144, 243)):
    g = torch.Generator(device="cuda").manual_seed(C + dil)
    n = 4
    x = torch.randn(n, T, C, device="cuda", generator=g)
    w1 = torch.randn(3, C, C, device="cuda", generator=g) / (3 * C) ** 0.5
    w2 = torch.randn(C, C, device="cuda", generator=g) / C ** 0.5
    b1 = torch.randn(C, device="cuda", generator=g) * 0.1
    b2 = torch.randn(C, device="cuda", generator=g) * 0.1

    def run(xx):
        o = torch.empty_like(xx)
        check(lib().jk_resblock_tc(ptr(xx), ptr(o), ptr(w1), ptr(b1), ptr(w2), ptr(b2), xx.shape[0], T, C, dil, 1.0, stream_ptr()))
        torch.cuda.synchronize()
        return o

    a = run(x)
    a2 = run(x)
    b = torch.cat([run(x[i:i + 1].contiguous()) for i in range(n)])
    ex = torch.empty_like(x)
    check(lib().jk_resblock_cl(ptr(x), ptr(ex), None, ptr(w1), ptr(b1), ptr(w2), ptr(b2), n, T, C, C, dil, 1.0, stream_ptr()))
    torch.cuda.synchronize()
    err = (a - ex).abs().amax(-1)                      # [n, T]
    bad_rr = (a != a2).any(-1)
    bad_nb = (a != b).any(-1)
    print(f"C {C} T {T} dil {dil}: max err vs exact {float(err.max()):.2e} (rel {float(err.max() / ex.abs().max()):.1e}); "
          f"run-to-run mismatching rows {int(bad_rr.sum())}, n=4 vs 4 x n=1 mismatching rows {int(bad_nb.sum())}")
    for name, bad in (("run-to-run", bad_rr), ("batch", bad_nb)):
        if bad.any():
            idx = bad.nonzero()[:12].tolist()
            d = float((a - (a2 if name == "run-to-run" else b)).abs().max())
            tiles = sorted({(i, t // 128) for i, t in bad.nonzero().tolist()})[:10]
            print(f"   {name}: first rows {idx}, max |diff| {d:.2e}, tiles {tiles}, rows in tile {sorted({t % 128 for _, t in bad.nonzero().tolist()})[:16]}")
    worst = err.flatten().topk(5)
    print("   worst rows vs exact:", [(int(i) // T, int(i) % T, f"{float(v):.1e}") for v, i in zip(worst.values, worst.indices)])
