"""GPU parity of the fp32 transformer path (csrc/f32_path.cu through the C ABI) against the reference's own fp32 outputs:
Transformer.forward(sample=True, fp16=False) per token (`y32`), forward mode over the whole sequence (`yfull32`, and `y32`
again - the reference's check_sample property that both modes agree), ConditionalAutoregressive2D.primed_sample /
forward in fp32 (`preds32`, `preds32_primed`), recorded attention weights, and SimplePrior.z_forward.

Tolerance: fp32 against fp32 with a different summation order - 2e-5 of the output range."""
import numpy as np
import pytest
import torch

from golden_util import Fixture, logit_cols, rel_err
from test_gpu_transformer import build
from test_gpu_prior import _load, _cuda, _make_prior

pytestmark = pytest.mark.gpu

TOL32 = 2e-5


@pytest.mark.parametrize("tag", ["order9", "order6", "order12", "order2_ragged"])
def test_fp32_sampling_mode_matches_reference(tag):
    fx = Fixture(f"transformer_{tag}")
    c = fx.cfg
    tr = build(fx)
    x = torch.from_numpy(fx["x"]).cuda()
    enc = torch.from_numpy(fx["encoder_kv"]).cuda() if "encoder_kv" in fx else None
    ys = []
    with torch.no_grad():
        for i in range(c["n_ctx"]):
            tr.check_cache(x.shape[0], i, False)
            ys.append(tr(x[:, i:i + 1].contiguous(), encoder_kv=enc, sample=True, fp16=False))
        tr.check_cache(x.shape[0], c["n_ctx"], False)
        tr.del_cache()
        tr.check_cache(x.shape[0], 0, False)
        # chunked (reference check_chunks): 7 + 23 + rest
        parts = [tr(x[:, a:b].contiguous(), encoder_kv=enc, sample=True, fp16=False)
                 for a, b in ((0, 7), (7, 30), (30, c["n_ctx"]))]
    y = torch.cat(ys, 1)
    e = rel_err(y.cpu().numpy(), fx["y32"])
    print(f"{tag}: fp32 sampling mode vs reference fp32 {e:.2e}")
    assert e < TOL32
    assert rel_err(torch.cat(parts, 1).cpu().numpy(), fx["y32"]) < TOL32


@pytest.mark.parametrize("tag", ["order9", "order6", "order12", "order2_ragged"])
def test_fp32_forward_mode_matches_reference(tag):
    fx = Fixture(f"transformer_{tag}")
    tr = build(fx)
    x = torch.from_numpy(fx["x"]).cuda()
    enc = torch.from_numpy(fx["encoder_kv"]).cuda() if "encoder_kv" in fx else None
    with torch.no_grad():
        y = tr(x, encoder_kv=enc, sample=False, fp16=False).cpu().numpy()
        y16 = tr(x, encoder_kv=enc, sample=False, fp16=True, fp16_out=True)
    assert y16.dtype == torch.float16
    want = fx["yfull32"] if "yfull32" in fx else fx["y32"]
    e = rel_err(y, want)
    print(f"{tag}: fp32 forward mode vs reference {e:.2e}")
    assert e < TOL32
    assert rel_err(y, fx["y32"]) < TOL32          # forward mode == sampling mode (reference check_sample)


def test_record_attn_rows_are_the_softmax_of_the_pattern():
    """recorded weights: rows sum to 1 over exactly the keys the pattern attends, and reproduce the layer's output"""
    fx = Fixture("transformer_order6")          # block, transpose, prev-block and enc-dec layers
    c = fx.cfg
    tr = build(fx)
    x = torch.from_numpy(fx["x"]).cuda()
    enc = torch.from_numpy(fx["encoder_kv"]).cuda()
    layers = set(range(c["n_depth"]))
    tr.set_record_attn(layers)
    with torch.no_grad():
        y = tr(x, encoder_kv=enc, sample=False, fp16=False)
    assert len(tr.ws) == c["n_depth"]
    n_ctx, bc = c["n_ctx"], c["n_ctx"] // c["blocks"]
    q = torch.arange(n_ctx, device="cuda")[:, None]
    k = torch.arange(n_ctx, device="cuda")[None, :]
    masks = {1: (k // bc == q // bc) & (k <= q), 2: (k % bc == q % bc) & (k <= q), 3: (k // bc == q // bc - 1),
             0: k <= q}
    for i, w in enumerate(tr.ws):
        f = c["attn_funcs"][i]
        assert tr._attn_mods[i].attn.w is w
        if f == 6:
            assert w.shape == (x.shape[0], c["n_head"], n_ctx, c["encoder_dims"])
            assert torch.allclose(w.sum(-1), torch.ones_like(w[..., 0]), atol=1e-5)
            continue
        m = masks[f]
        assert w.shape == (x.shape[0], c["n_head"], n_ctx, n_ctx)
        assert float(w.masked_fill(m, 0).abs().max()) == 0.0, f"layer {i} (attn_func {f}) has mass outside its pattern"
        rows = m.any(-1)
        s = w.sum(-1)
        assert torch.allclose(s[..., rows], torch.ones_like(s[..., rows]), atol=1e-5)
        assert float(s[..., ~rows].abs().max() if (~rows).any() else 0.0) == 0.0
    tr.set_record_attn(False)
    assert tr.ws == [] and all(b.attn.w is None for b in tr._attn_mods)
    with torch.no_grad():
        y2 = tr(x, encoder_kv=enc, sample=False, fp16=False)
    assert torch.equal(y, y2)


@pytest.mark.parametrize("tag", ["xy", "plain", "encdec_merged"])
def test_ca2d_fp32_sampling_and_forward(tag):
    from jukebox_b200.prior.autoregressive import ConditionalAutoregressive2D
    fx = Fixture(f"ca2d_{tag}")
    c = fx.cfg
    m = ConditionalAutoregressive2D((c["input_dims"],), c["bins"], width=c["width"], depth=c["depth"],
                                    heads=c["heads"], attn_order=c["attn_order"], blocks=c["blocks"],
                                    x_cond=c["x_cond"], y_cond=c["y_cond"], encoder_dims=c["encoder_dims"],
                                    prime_len=c["prime_len"], merged_decoder=c["merged_decoder"])
    m = _load(m, fx)
    tokens = _cuda(fx, "tokens")
    bs = tokens.shape[0]
    xc, yc, enc = _cuda(fx, "x_cond"), _cuda(fx, "y_cond"), _cuda(fx, "encoder_kv")
    torch.manual_seed(0)
    x, preds = m.primed_sample(bs, tokens[:, :-1].clone(), xc, yc, enc, fp16=False, get_preds=True, chunk_size=5)
    assert torch.equal(x[:, :-1], tokens[:, :-1])
    e = rel_err(preds.cpu().numpy(), fx["preds32_primed"])
    print(f"ca2d_{tag}: fp32 primed_sample logits vs reference {e:.2e}")
    assert e < TOL32
    assert rel_err(preds.cpu().numpy(), fx["preds32"]) < TOL32
    # whole-sequence forward: same logits, and the loss is the cross entropy of those logits in bits
    loss, p2 = m(tokens, xc, yc, enc, fp16=False, get_preds=True)
    assert rel_err(p2.cpu().numpy(), fx["preds32"]) < TOL32
    want = torch.nn.functional.cross_entropy(torch.from_numpy(fx["preds32"]).view(-1, c["bins"]),
                                             torch.from_numpy(fx["tokens"]).view(-1)) / np.log(2.)
    assert abs(float(loss) - float(want)) < 1e-4 * max(1.0, abs(float(want)))
    loss16, p16 = m(tokens, xc, yc, enc, fp16=True, get_preds=True)
    assert rel_err(p16.cpu().numpy(), fx["preds16"]) < 5e-3
    # ancestral fp32 sampling: deterministic under the seed, in range, partial windows
    torch.manual_seed(1)
    a = m.sample(bs, xc, yc, enc, fp16=False, temp=0.99, sample_tokens=9)
    torch.manual_seed(1)
    b = m.sample(bs, xc, yc, enc, fp16=False, temp=0.99, sample_tokens=9)
    assert torch.equal(a, b) and a.shape == (bs, 9) and int(a.min()) >= 0 and int(a.max()) < c["bins"]


@pytest.mark.parametrize("tag", ["single_enc_dec", "sep_enc_dec", "upsampler"])
def test_simple_prior_z_forward(tag):
    """z_forward: loss / preds of a full window, and the attention weights alignment reads"""
    fx = Fixture(f"prior_{tag}")
    prior = _make_prior(fx)
    c = fx.cfg
    toks = _cuda(fx, "tokens")
    bs = toks.shape[0]
    y = _cuda(fx, "y")
    z_conds = [_cuda(fx, "z_cond")] if "z_cond" in fx else []
    z = _cuda(fx, "z") if "z" in fx else toks
    upto = toks.shape[1]
    if prior.single_enc_dec:
        # a sampled id inside the lyric vocabulary is clamped to code 0 by prior_postprocess (reference prior.py:196-203),
        # so the merged sequence z_forward rebuilds can leave the golden token sequence there: the model is causal,
        # compare the logits up to the first such position
        with torch.no_grad():
            _, _, lyric = prior.get_cond(z_conds, y)
            merged, _ = prior.prior_preprocess([lyric, z], [None, None])
        diff = (merged != toks).any(0).nonzero()
        upto = int(diff[0]) + 1 if diff.numel() else upto
        assert upto > prior.n_tokens
    loss, metrics = prior.z_forward(z, z_conds, y, fp16=False, get_preds=True)
    preds = logit_cols(fx, metrics["preds"].cpu().numpy())
    e = rel_err(preds[:, :upto], fx["preds32"][:, :upto])
    print(f"prior_{tag}: z_forward fp32 logits vs reference {e:.2e}; loss {float(loss):.4f} bits")
    assert e < TOL32
    assert np.isfinite(float(loss)) and float(metrics["gen_loss"]) > 0
    if prior.single_enc_dec or prior.has_lyric_encoder:
        tr = prior.prior.transformer
        layers = {i for i, b in enumerate(tr._attn_mods) if b.attn_func in (6, 7)}
        ws = prior.z_forward(z, z_conds, y, fp16=False, get_attn_weights=layers)
        assert len(ws) == len(layers) and tr.ws == []
        for w in ws:
            assert w.shape[0] == bs and torch.isfinite(w).all()
