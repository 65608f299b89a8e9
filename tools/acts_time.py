"""Cost of JukeMIR representations at prior_5b geometry (synthetic weights), with the card it ran on.

Width 4800, 72 layers, 8 heads, attn_order 2, 128 blocks, n_ctx 8192, label-conditioned, merged decoder.  The number of
items per engine is the largest of 32 / 16 / 8 / 4 / 2 whose jk_prior_arena_bytes (host arithmetic) fits the memory left
beside the fp32 weights.  After one warm-up of every shape, three rounds alternate:
  truncated - ConditionalAutoregressive2D.layer_acts(fp16=True, layers=(36,)): the prefill cut after layer 36, the rows
              of layer 36 averaged inside it;
  full      - today's closest route: a full-depth prefill with h_out (fp32 [n, 8192, 4800]) and a torch mean;
  fp32      - layer_acts(fp16=False), item by item (2 items per round: it is the slow path).
Reported: ms per call and clips per second, the capture / pool kernel's time (torch.profiler) against one layer's GEMMs,
its bytes over time against the 3.35 TB/s data-sheet HBM3 figure, and max|fp16 - fp32| / max|fp32| of the pooled
features.

    python tools/acts_time.py [--layers N] [--out results.json]
"""
import ctypes as C
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HBM_TBS = 3.35          # H100 SXM data sheet
LAYER = 36


def _arg(name, default):
    return type(default)(sys.argv[sys.argv.index(name) + 1]) if name in sys.argv else default


def timed(fn):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    out = fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1), out


def main():
    assert torch.cuda.is_available(), "acts_time needs a GPU"
    from jukebox_b200 import _lib
    from jukebox_b200.engine import prior_config
    from jukebox_b200.prior.autoregressive import ConditionalAutoregressive2D
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    card = dict(name=torch.cuda.get_device_name(), nvidia_smi=q.stdout.strip().splitlines()[0] if q.stdout else "n/a")
    print("card:", card, flush=True)
    depth, W, n_ctx = _arg("--layers", 72), 4800, 8192
    torch.manual_seed(0)
    with torch.device("cuda"):
        m = ConditionalAutoregressive2D((n_ctx,), 2048, width=W, depth=depth, heads=8, attn_order=2, blocks=128,
                                        init_scale=0.1, x_cond=True, y_cond=True, merged_decoder=True).eval()
    tr = m.transformer
    tr.configure_engine(bins=m.bins, add_cond_after=m.add_cond_after_transformer)
    free = torch.cuda.mem_get_info()[0]
    n, arena = 0, 0
    for cand in (32, 16, 8, 4, 2):
        cfg = prior_config(**tr._engine_kwargs(cand))
        b = C.c_size_t(0)
        if _lib.lib().jk_prior_arena_bytes(C.byref(cfg), C.byref(b)) != 0:
            continue
        # beside the arena: the full route's h_out (fp32) and x_cond, + 4 GB for the fp32 route's caches and workspace
        need = b.value + cand * n_ctx * W * 4 * 2 + (4 << 30)
        if need < free:
            n, arena = cand, b.value
            break
    assert n, f"no engine of 2..32 items fits {free / 2**30:.1f} GB"
    print(f"{depth} layers; {n} items per engine (arena {arena / 2**30:.1f} GB of {free / 2**30:.1f} GB free)", flush=True)
    g = torch.Generator(device="cuda").manual_seed(1)
    tokens = torch.randint(0, m.bins, (n, n_ctx), device="cuda", generator=g)
    yc = torch.randn(n, 1, W, device="cuda", generator=g) * 0.1
    xc = torch.randn(n, n_ctx, W, device="cuda", generator=g) * 0.01
    n32 = min(n, 2)

    def truncated():
        return m.layer_acts(tokens, xc, yc, layers=(LAYER,), fp16=True)[LAYER]

    def full():
        eng = m._engine(n)
        tr.del_cache()
        h = torch.empty(n, n_ctx, W, device="cuda")
        eng.prefill(n, n_ctx, tokens=tokens, y_cond=yc.view(n, W), x_cond=xc, h_out=h)
        tr.del_cache()
        return h.mean(1)

    def fp32():
        return torch.cat([m.layer_acts(tokens[i:i + 1], xc[i:i + 1], yc[i:i + 1], layers=(LAYER,), fp16=False)[LAYER]
                          for i in range(n32)])

    routes = dict(truncated=truncated, full=full, fp32=fp32)
    for fn in routes.values():              # warm-up of every shape
        fn()
    times = {k: [] for k in routes}
    outs = {}
    for _ in range(3):
        for k, fn in routes.items():
            ms, outs[k] = timed(fn)
            times[k].append(ms)
            print(f"  {k}: {ms:.1f} ms", flush=True)
    # the capture / pool kernel against the layer GEMMs, from one profiled truncated call
    from torch.profiler import profile, ProfilerActivity
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        truncated()
        torch.cuda.synchronize()
    act_us = gemm_us = 0.0
    for e in prof.key_averages():
        dev_us = getattr(e, "device_time_total", None)
        if dev_us is None:
            dev_us = e.cuda_time_total
        if "act_rows_kernel" in e.key:
            act_us += dev_us
        elif "gemm" in e.key.lower():
            gemm_us += dev_us
    gemm_per_layer = gemm_us / (LAYER + 1)
    act_bytes = n * n_ctx * W * 2 + n * W * 4                  # the fp16 rows once, the means out (no x_cond: merged)
    e16 = float((outs["truncated"][:n32] - outs["fp32"]).abs().max() / outs["fp32"].abs().max())
    res = dict(card=card, layers=depth, layer=LAYER, items=n, positions=n_ctx, width=W,
               ms=dict((k, [round(v, 2) for v in vs]) for k, vs in times.items()),
               clips_per_s=dict(truncated=round(n * 1e3 / min(times["truncated"]), 2),
                                full=round(n * 1e3 / min(times["full"]), 2),
                                fp32=round(n32 * 1e3 / min(times["fp32"]), 3)),
               pool_kernel_us=round(act_us, 1), gemm_us_per_layer=round(gemm_per_layer, 1),
               pool_over_layer_gemms=round(act_us / gemm_per_layer, 5) if gemm_per_layer else None,
               pool_tb_s=round(act_bytes / (act_us * 1e-6) / 1e12, 3) if act_us else None, hbm_tb_s=HBM_TBS,
               rel_diff_fp16_fp32=e16)
    print(json.dumps(res))
    out = _arg("--out", "")
    if out:
        with open(out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
