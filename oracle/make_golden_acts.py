"""Generate tests/golden/acts_*.npz: intermediate-layer activations of the UNMODIFIED reference, on CPU (JukeMIR's recipe).

Run in the build container only (needs the reference tree):

    python -m oracle.make_golden_acts

JukeMIR (Castellon, Donahue & Liang, ISMIR 2021) takes a prior's representations by building the prior with
`prior_depth=L+1`, restoring the checkpoint non-strictly (the first L+1 layers' weights), setting
`prior.prior.only_encode = True` and calling `prior.prior.forward(...)`: the output of layer L + x_cond.  This does that
for every captured layer L of three tiny priors whose every Conv1D K is >= 64 and a multiple of 8 (so that jukebox_b200
takes them on its fp16 prefill), once with fp16=True and once with fp16=False:
  labelled       - a top-level label-conditioned prior (x_cond = the label time signal);
  single_enc_dec - lyric tokens prepended to the codes; the stored rows are the music positions only;
  sep_enc_dec    - a separate lyric encoder, with encoder-decoder layers (attn_func 6) below the captured layer.
Each fixture stores the config, the (name, shape) list of the FULL prior's state_dict, the weight seed (oracle/synth.py),
the inputs (z, y), what the autoregressive model receives (tokens, x_cond, y_cond, encoder keys enc16 / enc32) and per
layer `a16_L` / `a32_L`: fp32 [bs, positions, width].  (The reference's forward takes whole
windows only - pos_emb is added at full length - so shorter windows are checked against a full window's prefix.)
"""
import numpy as np

from oracle.make_golden import load_synth, save  # noqa: E402  (imports the reference)
import torch as t                                 # noqa: E402

ACTS_PRIORS = {
    # tag: (vqvae hps name, vqvae overrides, prior hps name, prior overrides, captured layers)
    "labelled": ("small_vqvae", dict(sample_length=64 * 256), "small_labelled_prior",
                 dict(n_ctx=64, prior_width=256, prior_depth=8, heads=2, blocks=4, level=1, levels=2), (3, 6)),
    "single_enc_dec": ("small_vqvae", dict(sample_length=84 * 256), "small_single_enc_dec_prior",
                       dict(n_ctx=84, prior_width=256, prior_depth=16, heads=2, blocks=8, n_tokens=12, level=1, levels=2),
                       (9, 15)),
    "sep_enc_dec": ("small_vqvae", dict(sample_length=64 * 256), "small_sep_enc_dec_prior",
                    dict(n_ctx=64, prior_width=256, prior_depth=14, heads=2, blocks=4, n_tokens=16, prime_width=256,
                         prime_depth=3, prime_heads=2, prime_blocks=4, level=1, levels=2, merged_decoder=True),
                    (4, 11)),
}

def _acts(prior, z, y, fp16):
    """prior.prior.forward of an only_encode model over the window z: the music positions' rows"""
    x_cond, y_cond, prime = prior.get_cond([], y)
    if prior.single_enc_dec:
        seq, x_cond = prior.prior_preprocess([prime, z], [None, x_cond])
        return prior.prior(seq, x_cond, y_cond, fp16=fp16)[:, prior.prime_loss_dims:].float()
    enc = prior.get_encoder_kv(prime, fp16=fp16)
    return prior.prior(z, x_cond, y_cond, enc, fp16=fp16).float()


def golden_acts(tag, bs=2, seed=6):
    from jukebox.hparams import setup_hparams
    from jukebox.make_models import make_vqvae, make_prior
    vq_name, vq_over, pr_name, pr_over, layers = ACTS_PRIORS[tag]
    vq = make_vqvae(setup_hparams(vq_name, dict(restore_vqvae="", **vq_over)), "cpu")
    hps = setup_hparams(pr_name, dict(restore_prior="", **pr_over))
    full = make_prior(hps, vq, "cpu")
    named = load_synth(full, seed)
    sd = full.state_dict()
    g = t.Generator().manual_seed(seed)
    ys = []
    for i in range(bs):
        lyric = t.randint(0, hps.n_vocab, (hps.n_tokens,), generator=g).tolist() if hps.n_tokens else []
        genres = [int(t.randint(0, hps.y_bins[0], (1,), generator=g))]
        artist = int(t.randint(0, hps.y_bins[1], (1,), generator=g))
        total = int(hps.min_duration * hps.sr * 3)
        ys.append(full.labeller.get_y_from_ids(artist, genres, lyric, total, 1000 * i))
    y = t.from_numpy(np.stack(ys)).long()
    z = t.randint(0, vq.l_bins, (bs, full.n_ctx), generator=g)
    out = {}
    with t.no_grad():
        # what the CA2D receives (for the numpy oracle): tokens, x_cond, y_cond and the encoder's keys per precision
        x_cond, y_cond, prime = full.get_cond([], y)
        tokens = z
        if full.single_enc_dec:
            tokens, x_cond = full.prior_preprocess([prime, z], [None, x_cond])
        conds = dict(tokens=tokens)
        if x_cond is not None:
            conds["x_cond"] = x_cond
        if y_cond is not None:
            conds["y_cond"] = y_cond
        if not full.single_enc_dec and full.n_tokens and full.use_tokens:
            conds["enc16"] = full.get_encoder_kv(prime, fp16=True).float()
            conds["enc32"] = full.get_encoder_kv(prime, fp16=False).float()
        for L in layers:
            cut = make_prior(setup_hparams(pr_name, dict(restore_prior="", **dict(pr_over, prior_depth=L + 1))), vq, "cpu")
            missing, _ = cut.load_state_dict(sd, strict=False)        # the first L+1 layers (JukeMIR's restore)
            assert not missing, missing
            cut.prior.only_encode = True
            cut.eval()
            for fp16 in (True, False):
                key = ("a16_" if fp16 else "a32_") + str(L)
                out[key] = _acts(cut, z, y, fp16)
            d = float((out[f"a16_{L}"] - out[f"a32_{L}"]).abs().max() / out[f"a32_{L}"].abs().max())
            print(f"{tag} layer {L}: {tuple(out[f'a32_{L}'].shape)}, max|ref16 - ref32| / max|ref32| {d:.2e}")
    tr = full.prior.transformer
    cfg = dict(tag=tag, vq_name=vq_name, vq_over=vq_over, pr_name=pr_name, pr_over=pr_over, seed=seed,
               layers=list(layers), n_ctx=int(full.n_ctx), single_enc_dec=bool(full.single_enc_dec),
               attn_funcs=[m.attn_func for m in tr._attn_mods], width=int(full.prior.width), heads=int(tr.n_head),
               input_dims=int(full.prior.input_dims), attn_order=int(hps.attn_order), blocks=int(tr.blocks),
               prime_len=None if full.prior.prime_len is None else int(full.prior.prime_len), encoder_dims=int(full.prior.encoder_dims), start=int(full.prime_loss_dims
                                                                                                    if full.single_enc_dec else 0),
               add_cond_after=bool(full.prior.add_cond_after_transformer))
    save(f"acts_{tag}", cfg, named, z=z, y=y, **conds, **out)


def main():
    for tag in ACTS_PRIORS:
        golden_acts(tag)


if __name__ == "__main__":
    main()
