"""Generate tests/golden/grad_*.npz: gradients of a prior's window loss from the UNMODIFIED reference on CPU.

Run in the build container only (needs the reference tree):

    python -m oracle.make_golden_grad

For each tiny geometry the reference model gets the synthetic weights of its existing fixture (oracle/synth.py), the
decoder (`prior.prior`, a ConditionalAutoregressive2D) is made trainable, and the window's z_forward loss is
backpropagated - once with the model in float32 and once in float64.  Stored: the token sequence and the constant
conditioning the decoder reads (x_cond, y_cond, encoder_kv, in float32 as the float32 model saw them), the loss of each
run and the gradient of every decoder parameter in each dtype (g32:<name>, g64:<name>, at the flat indices idx:<name>).  The geometries together
cover the six attention patterns: single_enc_dec (1, 2, 3, 7), sep_enc_dec (1, 2, 3, 6), upsampler (1, 2, 3) and a
plain dense prior (0).
"""
import copy
import os
import sys
import zlib

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)

from oracle.make_golden import GOLDEN, TINY_PRIORS, load_synth, save  # noqa: E402  (imports the reference)
import torch as t                                                       # noqa: E402


def _run(prior, seq, x_cond, y_cond, enc, dtype):
    """z_forward's loss, restated from the decoder's parts so the conditioning stays the stored constant, backpropagated
    through a copy of the decoder in `dtype`.  A separate lyric encoder's prime loss depends on frozen modules only and
    adds nothing to the decoder's gradient."""
    m = copy.deepcopy(prior.prior).to(dtype)
    m.requires_grad_(True)
    cast = lambda v: None if v is None else v.to(dtype)
    total = prior.total_loss_dims
    if prior.single_enc_dec:
        (prime_loss, gen_loss), _ = m(seq, cast(x_cond), cast(y_cond), fp16=False, get_sep_loss=True)
        loss = prior.prime_loss_fraction * prime_loss * prior.prime_loss_dims / total + gen_loss * prior.gen_loss_dims / total
    else:
        gen_loss, _ = m(seq, cast(x_cond), cast(y_cond), cast(enc), fp16=False)
        loss = gen_loss * prior.gen_loss_dims / total
    loss.backward()
    grads = {n: p.grad.detach().double().numpy() for n, p in m.named_parameters()}
    return float(loss), float(gen_loss), grads


def golden_grad_prior(tag, seed=4):
    from jukebox.hparams import setup_hparams
    from jukebox.make_models import make_vqvae, make_prior
    vq_name, vq_over, pr_name, pr_over = TINY_PRIORS[tag]
    vq = make_vqvae(setup_hparams(vq_name, dict(restore_vqvae="", **vq_over)), "cpu")
    prior = make_prior(setup_hparams(pr_name, dict(restore_prior="", **pr_over)), vq, "cpu")
    named = load_synth(prior, seed)
    fx = np.load(os.path.join(GOLDEN, f"prior_{tag}.npz"))
    y = t.from_numpy(fx["y"]) if "y" in fx.files else None
    z_conds = [t.from_numpy(fx["z_cond"])] if "z_cond" in fx.files else None
    tokens = t.from_numpy(fx["tokens"])
    with t.no_grad():
        x_cond, y_cond, lyric = prior.get_cond(z_conds, y)
        enc = None
        if prior.single_enc_dec:
            z = prior.prior_postprocess(tokens.clone())
            seq, x_cond = prior.prior_preprocess([lyric, z], [None, x_cond])
        else:
            seq = tokens
            if prior.n_tokens and prior.use_tokens:
                enc = prior.get_encoder_kv(lyric, fp16=False)
    arrays = dict(seq=seq)
    for k, v in (("x_cond", x_cond), ("y_cond", y_cond), ("encoder_kv", enc)):
        if v is not None:
            arrays[k] = v.float()
    _finish(f"grad_{tag}", dict(tag=tag, kind="prior", seed=seed, vq_name=vq_name, vq_over=vq_over, pr_name=pr_name,
                                pr_over=pr_over, prime_len=int(prior.prime_loss_dims) if prior.single_enc_dec else 0),
            named, arrays, lambda dt: _run(prior, seq, x_cond, y_cond, enc, dt))


def golden_grad_plain(seed=2, bs=2):
    """a dense (attn_func 0) decoder of its own: the loss is CE / ln 2 over the window, as z_forward's for a prior
    without lyrics"""
    from jukebox.prior.autoregressive import ConditionalAutoregressive2D
    cfg = dict(input_dims=48, bins=50, width=64, depth=3, heads=2, attn_order=0, blocks=None)
    m0 = ConditionalAutoregressive2D((cfg["input_dims"],), cfg["bins"], width=cfg["width"], depth=cfg["depth"],
                                     heads=cfg["heads"], attn_order=0, blocks=None)
    m0.eval()
    named = load_synth(m0, seed)
    g = t.Generator().manual_seed(seed)
    seq = t.randint(0, cfg["bins"], (bs, cfg["input_dims"]), generator=g)

    def run(dtype):
        m = copy.deepcopy(m0).to(dtype)
        m.requires_grad_(True)
        loss, _ = m(seq, fp16=False)
        loss.backward()
        return float(loss), float(loss), {n: p.grad.detach().double().numpy() for n, p in m.named_parameters()}

    _finish("grad_plain", dict(cfg, kind="ca2d", seed=seed, prime_len=0), named, dict(seq=seq), run)


SAMPLE = 512       # elements stored per parameter (idx:<name>, flat indices); smaller parameters are stored whole


def _float64_run():
    """The reference upcasts to float32 where its fp16 mode needs it (LayerNorm's input, the attention scores before the
    softmax, the stack's output: Tensor.float()).  For the float64 run only, .float() leaves a float64 tensor as it is,
    so that every operation runs at float64 - the same formulas, one precision higher."""
    import contextlib

    @contextlib.contextmanager
    def patched():
        orig = t.Tensor.float
        t.Tensor.float = lambda self, *a, **k: self if self.dtype == t.float64 else orig(self, *a, **k)
        try:
            yield
        finally:
            t.Tensor.float = orig
    return patched()


def _finish(name, cfg, named, arrays, run):
    l32, gen32, g32 = run(t.float32)
    with _float64_run():
        l64, gen64, g64 = run(t.float64)
    for n in g32:      # a seeded sample of each large parameter's elements keeps the fixture small
        flat32, flat64 = g32[n].reshape(-1), g64[n].reshape(-1)
        idx = np.arange(flat32.size)
        if flat32.size > SAMPLE:
            idx = np.sort(np.random.RandomState(zlib.crc32(n.encode())).choice(flat32.size, SAMPLE, replace=False))
        arrays[f"idx:{n}"] = idx.astype(np.int32)
        arrays[f"g32:{n}"] = flat32[idx].astype(np.float32)
        arrays[f"g64:{n}"] = flat64[idx]
    cfg = dict(cfg, loss32=l32, loss64=l64, gen32=gen32, gen64=gen64, params=sorted(g32))
    save(name, cfg, named, **arrays)


def main():
    for tag in ("single_enc_dec", "sep_enc_dec", "upsampler"):
        golden_grad_prior(tag)
    golden_grad_plain()


if __name__ == "__main__":
    main()
