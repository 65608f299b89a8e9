"""Per-phase timing of the persistent decode kernel from its own globaltimer stamps (CTA 0).

    python tools/phase_profile.py [--small] [--pos 4000]

Prints the mean time between consecutive grid barriers, grouped by phase type, for a few tokens at
the given position of the 1b_lyrics workload."""
import argparse
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--small", action="store_true")
    ap.add_argument("--pos", type=int, default=4000)
    ap.add_argument("--n", type=int, default=16)
    ap.add_argument("--workload", default="1b_lyrics")
    args = ap.parse_args()
    import contextlib
    with contextlib.redirect_stdout(sys.stderr):
        prior, _ = bench.build_prior(bench.SMALL if args.small else bench.WORKLOADS[args.workload])
    n = args.n
    ca = prior.prior
    eng = ca._engine(n)
    L = ca.input_dims
    toks = torch.randint(0, ca.bins, (n, L), device="cuda")
    lbuf = torch.empty(n, ca.bins, device="cuda")
    yc = torch.randn(n, ca.width, device="cuda") if ca.y_cond else None
    xc = torch.zeros(n, 1, ca.width, device="cuda") if ca.x_cond else None
    lb = None       # x_cond . x_out^T (SamplingWindow computes it once per window for the tensor-core logits product)
    if xc is not None and ca.add_cond_after_transformer and os.environ.get("JK_LOGIT_BIAS", "1") != "0":
        from jukebox_b200.transformer import f32 as _f32
        lb = _f32.linear_nk(xc.reshape(n, ca.width), ca.x_out.weight).view(n, 1, ca.bins) if hasattr(ca, "x_out") else None
    if ca.transformer.encoder_dims:
        eng.set_encoder_kv(torch.randn(n, ca.transformer.encoder_dims, ca.width, device="cuda"))
    depth = ca.transformer.n_depth
    funcs = [l.attn_func for l in ca.transformer._attn_mods]
    pos = min(args.pos, L - 8)
    eng.reset(pos)
    rows, clocks = [], []
    for i in range(6):
        eng.step(n, tokens=toks, y_cond=yc, x_cond=xc, logits=lbuf, logit_bias=lb)
        torch.cuda.synchronize()
        prof = eng.debug_buffer(5).view(torch.int64).cpu().numpy()
        stamps = prof[: 2 + 5 * depth + 1].astype(np.float64)
        if i >= 2:
            rows.append(np.diff(stamps))
            # SM clock of this step: CTA 0 enters the proj Conv1D of layer l (clock64 stamp, slot 3 + 5 l) right after it
            # stamps the end of the attention phase (globaltimer, same slot); the first and the last layer span the step
            p2 = eng.debug_buffer(6).view(torch.int64).cpu().numpy().reshape(-1, 8).astype(np.float64)
            a, b = 3, 3 + 5 * (depth - 1)
            clocks.append((p2[b, 0] - p2[a, 0]) / (stamps[b] - stamps[a]) * 1e3)
    d = np.mean(rows, 0) / 1e3          # us
    mhz = float(np.mean(clocks))
    print(f"position {pos}, n={n}, depth={depth}: kernel total {d.sum():.1f} us")
    print(f"  embed                : {d[0]:8.2f} us")
    names = ["LN+QKV gemm", "attention", "proj gemm", "LN+FC gemm+gelu", "proj2 gemm"]
    per = d[1:1 + 5 * depth].reshape(depth, 5)
    for j, nm in enumerate(names):
        print(f"  {nm:20s} : mean {per[:, j].mean():7.2f} us  min {per[:, j].min():7.2f}  max {per[:, j].max():7.2f}   (x{depth})")
    for f in sorted(set(funcs)):
        sel = [i for i, g in enumerate(funcs) if g == f]
        print(f"     attention attn_func {f}: mean {per[sel, 1].mean():7.2f} us over {len(sel)} layers")
    print(f"  logits + tail        : {d[1 + 5 * depth]:8.2f} us")
    print(f"  per layer            : {per.sum(1).mean():8.2f} us")
    # intra-phase stamps of CTA 0 (SM clock cycles): slot = phase index
    p2 = eng.debug_buffer(6).view(torch.int64).cpu().numpy().reshape(-1, 8).astype(np.float64)
    print(f"  SM clock measured over the step: {mhz:.0f} MHz (min {min(clocks):.0f}, max {max(clocks):.0f} over {len(clocks)} steps)")
    print("  CTA 0, GEMM phases (us): wait+stage | mma+weights | reduce+publish partials | exchange+epilogue")
    for j, nm in ((0, "LN+QKV"), (2, "proj"), (3, "LN+FC"), (4, "proj2")):
        rows = []
        for l in range(depth):
            slot = 1 + 5 * l + j
            s0, s1, s2, s3, s4 = p2[slot, :5]
            rows.append([(s1 - s0), (s2 - s1), (s3 - s2), (s4 - s3)])
        r = np.mean(rows, 0) / mhz
        print(f"     {nm:8s}: {r[0]:6.2f} | {r[1]:6.2f} | {r[2]:6.2f} | {r[3]:6.2f}")
    # the logits GEMM (when the engine plans one) stamps the slots after the last layer, one per pass
    for ip, sl in enumerate(range(1 + 5 * depth, 1 + 5 * depth + 4)):
        if not p2[sl, 4] > p2[sl, 0] > 0:
            break
        s0, s1, s2, s3, s4 = p2[sl, :5]
        print(f"     logits {ip}: {(s1 - s0) / mhz:6.2f} | {(s2 - s1) / mhz:6.2f} | {(s3 - s2) / mhz:6.2f} | {(s4 - s3) / mhz:6.2f}   "
              f"(polled loads in at {(p2[sl, 6] - s0) / mhz:5.2f})")
    print("  CTA 0, staging detail (us from phase entry): statistics ready | own polled loads in | past the statistics barrier | staged + barrier")
    for j, nm in ((0, "LN+QKV"), (2, "proj"), (3, "LN+FC"), (4, "proj2")):
        rows = []
        for l in range(depth):
            slot = 1 + 5 * l + j
            s0 = p2[slot, 0]
            rows.append([p2[slot, 5] - s0, p2[slot, 6] - s0, p2[slot, 7] - s0, p2[slot, 1] - s0])
        r = np.mean(rows, 0) / mhz
        print(f"     {nm:8s}: {r[0]:6.2f} | {r[1]:6.2f} | {r[2]:6.2f} | {r[3]:6.2f}")
    sel = [l for l in range(depth) if funcs[l] in (1, 3) and p2[1 + 5 * l + 1, 3] > 0]
    if sel:
        ar = np.array([[p2[1 + 5 * l + 1, i] for i in (0, 1, 2, 3)] for l in sel]) / mhz
        d_ = np.diff(ar, axis=1).mean(0)
        print(f"     attention block/prev layers, CTA 0 (us): q/k/v poll + tile load {d_[0]:5.2f} | scores {d_[1]:5.2f} | softmax+PV {d_[2]:5.2f}")
    p3 = eng.debug_buffer(7).view(torch.int64).cpu().numpy().reshape(5, 256, 2).astype(np.float64)
    G = torch.cuda.get_device_properties(0).multi_processor_count
    print("  layer 1, all CTAs (globaltimer, us): phase entry spread (min/median/max after the first entry) | time in phase (min/median/max)")
    for j, nm in enumerate(["LN+QKV", "attention", "proj", "LN+FC", "proj2"]):
        arr, ex = p3[j, :G, 0], p3[j, :G, 1]
        a0 = arr.min()
        dur = (ex - arr) / 1e3
        order = np.argsort(ex)
        print(f"     {nm:10s}: entry {0:5.2f} / {np.median(arr - a0) / 1e3:5.2f} / {(arr.max() - a0) / 1e3:5.2f}   "
              f"in phase {dur.min():5.2f} / {np.median(dur):5.2f} / {dur.max():5.2f}   last out {order[-4:].tolist()}")
    print(f"  layer 1 wall (first entry of LN+QKV -> last exit of proj2): {(p3[4, :G, 1].max() - p3[0, :G, 0].min()) / 1e3:6.2f} us")


if __name__ == "__main__":
    main()
