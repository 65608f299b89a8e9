"""Time the fp32 path's forward against forward + backward (csrc/f32_grad.cu) per layer and per window.

    python tools/grad_time.py [--reps 3]

One layer of synthetic weights per case, one item, a whole window (1b_lyrics: width 2 048, 8 576 positions, dense and
block layers; upsampler: width 1 920, 8 192 positions).  CUDA events around jk_f32_forward (one layer) and around the
same forward plus jk_f32_backward of that layer; every shape is warmed up first.  Prints the card's name and power limit,
per layer the times, and the achieved FP32 rate of the backward against the data sheet's 67 TFLOP/s (FLOPs counted from
shapes: the GEMMs of the recomputed forward and of dX / dW, attention's score and value products).  A window's time is
the layer time times the prior's depth (72 / 72 layers)."""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from jukebox_b200 import _lib                 # noqa: E402
from oracle.synth import synth_tensor          # noqa: E402

CASES = {"1b dense": (2048, 2, 8576, 64, 384, 0, 72), "1b block": (2048, 2, 8576, 64, 384, 1, 72),
         "up block": (1920, 1, 8192, 128, 0, 1, 72), "up transpose": (1920, 1, 8192, 128, 0, 2, 72)}
NAMES = [("ln0_g", "ln_0.weight", "W"), ("ln0_b", "ln_0.bias", "W"), ("ln1_g", "ln_1.weight", "W"),
         ("ln1_b", "ln_1.bias", "W"), ("c_attn_w", "attn.c_attn.w", "W,3S"), ("c_attn_b", "attn.c_attn.b", "3S"),
         ("c_proj_w", "attn.c_proj.w", "S,W"), ("c_proj_b", "attn.c_proj.b", "W"), ("fc_w", "mlp.c_fc.w", "W,W"),
         ("fc_b", "mlp.c_fc.b", "W"), ("proj2_w", "mlp.c_proj.w", "W,W"), ("proj2_b", "mlp.c_proj.b", "W")]


def keys_attended(af, P, bc, prime):
    p = torch.arange(P, dtype=torch.float64)
    n = {0: p + 1, 1: p % bc + 1, 2: torch.div(p, bc, rounding_mode="floor") + 1,
         7: torch.where(p < prime, p + 1, torch.full_like(p, prime))}[af]
    return float(n.sum())


def case(name, reps):
    W, H, P, blocks, prime_len, af, depth = CASES[name]
    S, bc = W // 4, P // blocks
    prime = (prime_len // blocks + 1) * blocks if prime_len else 0
    dims = {"W": W, "S": S, "3S": 3 * S}
    L, G, keep = _lib.F32Layer(), _lib.F32GradLayer(), []
    for field, nm, shp in NAMES:
        shape = tuple(dims[d] for d in shp.split(","))
        w = torch.from_numpy(synth_tensor(f"_attn_mods.0.{nm}", shape, 5)).cuda()
        g = torch.zeros_like(w)
        keep += [w, g]
        setattr(L, field, w.data_ptr())
        setattr(G, field, g.data_ptr())
    L.attn_func = af
    kc = torch.zeros(1, P, S, device="cuda")
    vc = torch.zeros_like(kc)
    L.k_cache, L.v_cache = kc.data_ptr(), vc.data_ptr()
    x0 = torch.randn(1, P, W, device="cuda")
    dy = torch.randn(1, P, W, device="cuda")
    a = _lib.F32Args(n=1, P=P, p0=0, width=W, n_state=S, mlp_width=W, heads=H, n_ctx=P, blocks=blocks,
                     prime_len=prime_len, encoder_dims=0, depth=1, x=0, encoder_kv=0, work=0)
    f_need, b_need = C.c_size_t(0), C.c_size_t(0)
    _lib.check(_lib.lib().jk_f32_workspace_floats(C.byref(a), C.byref(f_need)))
    _lib.check(_lib.lib().jk_f32_backward_workspace_floats(C.byref(a), C.byref(b_need)))
    fwork = torch.empty(f_need.value, device="cuda")
    bwork = torch.empty(b_need.value, device="cuda")
    ins = (C.c_void_p * 1)(x0.data_ptr())

    def fwd():
        x = x0.clone()
        a.x, a.work = x.data_ptr(), fwork.data_ptr()
        _lib.check(_lib.lib().jk_f32_forward(C.byref(a), C.pointer(L), _lib.stream_ptr()))

    def bwd():
        dx = dy.clone()
        a.work = bwork.data_ptr()
        _lib.check(_lib.lib().jk_f32_backward(C.byref(a), C.pointer(L), C.pointer(G), ins, _lib.ptr(dx), None,
                                              _lib.stream_ptr()))

    def timed(fn):
        fn()
        torch.cuda.synchronize()
        best = []
        for _ in range(reps):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            fn()
            e1.record()
            e1.synchronize()
            best.append(e0.elapsed_time(e1) * 1e3)
        return min(best)

    t_f = timed(fwd)
    t_fb = timed(lambda: (fwd(), bwd()))
    gemm = 2.0 * P * (W * 3 * S + S * W + 2 * W * W)           # one pass of the layer's four Conv1D products
    attn = 2.0 * 2 * keys_attended(af, P, bc, prime) * S          # scores and values
    flops_b = gemm * 3 + attn * 5                                 # recomputed forward, dX, dW; attention fwd + 2 passes
    return dict(case=name, forward_us=t_f, forward_backward_us=t_fb, backward_us=t_fb - t_f,
                window_forward_backward_s=t_fb * depth / 1e6, backward_tflops=flops_b / ((t_fb - t_f) * 1e-6) / 1e12,
                of_67_tflops=flops_b / ((t_fb - t_f) * 1e-6) / 67e12)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    print(json.dumps(dict(card=card)))
    for name in CASES:
        print(json.dumps(case(name, args.reps)))


if __name__ == "__main__":
    main()
