"""Generate tests/golden/align_*.npz: attention weights the UNMODIFIED reference records for lyric alignment, on CPU.

Run in the build container only (needs the reference tree):

    python -m oracle.make_golden_align

The reference's get_alignment (jukebox/align.py) calls SimplePrior.z_forward(z, [], y, fp16=fp16,
get_attn_weights={alignment_layer}) on every window; this runs that call once in fp16 and once in fp32 on two tiny priors
whose every Conv1D K is >= 64 and a multiple of 8 (so that jukebox_b200 records them in its fp16 prefill):
  single_enc_dec - lyric tokens prepended to the codes, the prime layer (attn_func 7) recorded: music queries x lyric keys;
  sep_enc_dec    - a separate lyric encoder, the encoder-decoder layer (attn_func 6) recorded, head dim 60 (not a
                   multiple of 8, like 5b_lyrics' 150).
Each fixture stores the config, the (name, shape) list of the state_dict, the weight seed (oracle/synth.py), the inputs
(z, y) and both weight sets (`w16`, `w32`, fp32 arrays [bs, heads, queries, keys]).
"""
import numpy as np

from oracle.make_golden import load_synth, save  # noqa: E402  (imports the reference)
import torch as t                                 # noqa: E402

ALIGN_PRIORS = {
    # tag: (vqvae hps name, vqvae overrides, prior hps name, prior overrides, recorded layer)
    "single_enc_dec": ("small_vqvae", dict(sample_length=84 * 256), "small_single_enc_dec_prior",
                       dict(n_ctx=84, prior_width=256, prior_depth=16, heads=2, blocks=8, n_tokens=12, level=1, levels=2),
                       15),
    "sep_enc_dec": ("small_vqvae", dict(sample_length=64 * 256), "small_sep_enc_dec_prior",
                    dict(n_ctx=64, prior_width=960, prior_depth=10, heads=4, blocks=4, n_tokens=16, prime_width=256,
                         prime_depth=3, prime_heads=2, prime_blocks=4, level=1, levels=2, merged_decoder=True),
                    9),
}


def golden_align(tag, bs=2, seed=5):
    from jukebox.hparams import setup_hparams
    from jukebox.make_models import make_vqvae, make_prior
    vq_name, vq_over, pr_name, pr_over, layer = ALIGN_PRIORS[tag]
    vq = make_vqvae(setup_hparams(vq_name, dict(restore_vqvae="", **vq_over)), "cpu")
    hps = setup_hparams(pr_name, dict(restore_prior="", **pr_over))
    prior = make_prior(hps, vq, "cpu")
    named = load_synth(prior, seed)
    want_func = 7 if prior.single_enc_dec else 6
    assert prior.prior.transformer._attn_mods[layer].attn_func == want_func
    g = t.Generator().manual_seed(seed)
    ys = []
    for i in range(bs):
        lyric = t.randint(0, hps.n_vocab, (hps.n_tokens,), generator=g).tolist()
        genres = [int(t.randint(0, hps.y_bins[0], (1,), generator=g))]
        artist = int(t.randint(0, hps.y_bins[1], (1,), generator=g))
        total = int(hps.min_duration * hps.sr * 3)
        ys.append(prior.labeller.get_y_from_ids(artist, genres, lyric, total, 1000 * i))
    y = t.from_numpy(np.stack(ys)).long()
    z = t.randint(0, vq.l_bins, (bs, prior.n_ctx), generator=g)
    out = {}
    with t.no_grad():
        for fp16 in (True, False):
            rows = []
            for i in range(bs):          # item by item, as the reference's get_alignment calls it
                ws = prior.z_forward(z[i:i + 1], [], y[i:i + 1], fp16=fp16, get_attn_weights={layer})
                assert len(ws) == 1
                rows.append(ws[0].float())
            out["w16" if fp16 else "w32"] = t.cat(rows)
    print(f"{tag}: recorded {tuple(out['w16'].shape)}, max|ref16 - ref32| "
          f"{float((out['w16'] - out['w32']).abs().max()):.2e}")
    cfg = dict(tag=tag, vq_name=vq_name, vq_over=vq_over, pr_name=pr_name, pr_over=pr_over, seed=seed, layer=layer,
               n_ctx=int(prior.n_ctx), single_enc_dec=bool(prior.single_enc_dec))
    save(f"align_{tag}", cfg, named, z=z, y=y, **out)


def main():
    for tag in ALIGN_PRIORS:
        golden_align(tag)


if __name__ == "__main__":
    main()
