"""GPU diagnostic (not a test): depth-1 .. 16 transformers per attention pattern, comparing what a decode step returns -
the transformer output h (h_out) and the logits h . x_out^T - with the oracle after every token.  On a mismatch it
prints where the error sits: which samples, which columns of h, and whether the values are finite.  The activations
in between travel between SMs as flagged words and are not kept by the engine."""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import transformer_np as O          # noqa: E402
from oracle.synth import synth_state_dict         # noqa: E402
from jukebox_b200.transformer.transformer import Transformer   # noqa: E402


def run(attn_order, n_in, heads, n_ctx, blocks, bs, steps, enc_dims=0, prime_len=None, depth=1, bins=100):
    tr = Transformer(n_in, n_ctx, heads, depth, mask=True, attn_order=attn_order, blocks=blocks,
                     encoder_dims=enc_dims, prime_len=prime_len)
    named = [(k, tuple(v.shape)) for k, v in tr.state_dict().items()]
    sd = synth_state_dict(named, 7)
    tr.load_state_dict({k: torch.from_numpy(v) for k, v in sd.items()})
    tr.configure_engine(bins=bins)                  # the same launch also computes the logits
    tr = tr.cuda().eval()
    orc = O.TransformerOracle(sd, n_in, n_ctx, heads, depth, attn_order, blocks, enc_dims, prime_len)
    rng = np.random.RandomState(0)
    x = rng.standard_normal((bs, steps, n_in)).astype(np.float32)
    enc = rng.standard_normal((bs, enc_dims, n_in)).astype(np.float32) if enc_dims else None
    x_out = (rng.standard_normal((bins, n_in)) * 0.02).astype(np.float32)
    eng = tr.engine(bs)
    eng.set_embeddings(x_out=torch.from_numpy(x_out).cuda())
    if enc is not None:
        eng.set_encoder_kv(torch.from_numpy(enc).cuda())
    eng.reset(0)
    worst = 0.0
    for i in range(steps):
        ref = orc.step(x[:, i], enc, True)
        h = torch.empty(bs, n_in, device="cuda")
        lg = torch.empty(bs, bins, device="cuda")
        eng.step(bs, x_in=torch.from_numpy(x[:, i]).cuda(), h_out=h, logits=lg)
        h, lg = h.cpu().numpy(), lg.cpu().numpy()
        ref_lg = ref.astype(np.float64) @ x_out.astype(np.float64).T
        err = np.abs(h - ref).max() / max(np.abs(ref).max(), 1e-9)
        err_lg = np.abs(lg - ref_lg).max() / max(np.abs(ref_lg).max(), 1e-9)
        worst = max(worst, err, err_lg)
        if max(err, err_lg) > 1e-3 and i < 4:
            d = np.abs(h - ref)
            cols = np.argsort(d.max(0))[::-1][:8]
            print(f"   step {i}: h rel err {err:.3e}  logits rel err {err_lg:.3e}  |ref| {np.abs(ref).max():.3f}  "
                  f"|h| {np.abs(h).max():.3f}  finite h={np.isfinite(h).all()} logits={np.isfinite(lg).all()}")
            print(f"      per-sample max |h - ref|: {np.array2string(d.max(1), precision=3)}")
            print(f"      worst columns of h: {cols.tolist()}  (max |h - ref| {np.array2string(d.max(0)[cols], precision=3)})")
    print(f"attn_funcs={[l.attn_func for l in tr._attn_mods]} n_in={n_in} heads={heads} bs={bs} steps={steps}: "
          f"worst rel err {worst:.3e}")
    return worst


if __name__ == "__main__":
    torch.manual_seed(0)
    print("SMs:", torch.cuda.get_device_properties(0).multi_processor_count)
    run(0, 64, 2, 48, 4, 2, 12)                       # dense
    run(0, 256, 2, 48, 4, 16, 12)                     # dense, bs 16, dh 32
    run(1, 256, 2, 48, 4, 3, 20, depth=1)             # block only
    run(2, 256, 2, 48, 4, 3, 30, depth=3)             # block, transpose, prev
    run(6, 128, 2, 48, 4, 2, 20, enc_dims=10, depth=4)
    run(12, 128, 2, 96, 8, 2, 40, prime_len=12, depth=16)
    run(0, 2048, 2, 600, 4, 16, 300, depth=1)          # 1b width, dense rows > 256 -> split-KV path
    run(2, 1024, 1, 512, 64, 16, 40, depth=3)          # upsampler-like dh 256
