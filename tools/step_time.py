"""Average duration of the decode-step kernel (no profiling stamps) at a few positions of the 1b_lyrics window."""
import contextlib
import sys
import os

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402

with contextlib.redirect_stdout(sys.stderr):
    wl = bench.SMALL if "--small" in sys.argv else bench.WORKLOADS[os.environ.get("JK_WORKLOAD", "1b_lyrics")]
    prior, _ = bench.build_prior(wl)
ca = prior.prior
n = int(os.environ.get("JK_N", "16"))
eng = ca._engine(int(os.environ.get("JK_ENGINE_N", n)))     # JK_ENGINE_N: an engine planned for more samples than it steps
L = ca.input_dims
toks = torch.randint(0, ca.bins, (n, L), device="cuda")
lbuf = torch.empty(n, ca.bins, device="cuda")
yc = torch.randn(n, ca.width, device="cuda") if ca.y_cond else None
xc = torch.zeros(n, 1, ca.width, device="cuda") if ca.x_cond and not os.environ.get("JK_XC_NONE") else None
lb = None       # x_cond . x_out^T (SamplingWindow computes it once per window for the tensor-core logits product)
if xc is not None and ca.add_cond_after_transformer and os.environ.get("JK_LOGIT_BIAS", "1") != "0":
    from jukebox_b200.transformer import f32 as _f32
    lb = _f32.linear_nk(xc.reshape(n, ca.width), ca.x_out.weight).view(n, 1, ca.bins) if hasattr(ca, "x_out") else None
if ca.transformer.encoder_dims:
    eng.set_encoder_kv(torch.randn(n, ca.transformer.encoder_dims, ca.width, device="cuda"))
for pos in (500, 4000, 8000):
    pos = min(pos, L - 60)
    eng.reset(pos)
    for _ in range(5):
        eng.step(n, tokens=toks, y_cond=yc, x_cond=xc, logits=lbuf, logit_bias=lb)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(50):
        eng.step(n, tokens=toks, y_cond=yc, x_cond=xc, logits=lbuf, logit_bias=lb)
    e1.record()
    torch.cuda.synchronize()
    print(f"decode step at position {pos}: {e0.elapsed_time(e1) / 50 * 1000:.1f} us")
