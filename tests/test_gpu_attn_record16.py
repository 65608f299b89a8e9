"""Attention weights recorded by the fp16 prefill (jk_prefill_args.record, csrc/prefill.cu attn_record_*): the pass lyric
alignment runs with the sampling fp16 flag (reference sample.py:118-119 -> align.py get_alignment -> z_forward(fp16=True,
get_attn_weights={alignment_layer})).

  pattern   - every layer recorded: mass only on the layer's key set, rows with keys sum to 1, rows without keys are 0;
              tensor-core record kernel (dh 64, dh 150 on the 4-byte staging) and the scalar one (dh 480)
  fp32 path - the same tokens through the fp32 forward-mode path: elementwise agreement within 1.5e-2 (fp16 activations
              through up to 16 layers put the two 3.6e-3 .. 8.9e-3 apart on an H100); this catches wrong keys, scales or
              normalisation, while the rounding points are held by the reference test below
  reference - golden priors (oracle/make_golden_align.py): max|ours16 - ref16| <= max(1e-3, 1.5 max|ref16 - ref32|),
              the tolerance rule of DESIGN section 2
  routing   - z_forward(fp16=True) records on the engine (the fp32 path is never built) unless the window exceeds the
              prefill capacity; recording leaves the loss and logits bit-identical; batched alignment == item by item"""
import numpy as np
import pytest
import torch

from golden_util import Fixture
from test_gpu_prefill import _model
from test_gpu_prior import _make_prior

pytestmark = pytest.mark.gpu


def _masks(n_ctx, bc):
    q = torch.arange(n_ctx, device="cuda")[:, None]
    k = torch.arange(n_ctx, device="cuda")[None, :]
    return {0: k <= q, 1: (k // bc == q // bc) & (k <= q), 2: (k % bc == q % bc) & (k <= q), 3: (k // bc == q // bc - 1)}


def _forward_ws(m, tokens, yc, xc, ekv, fp16):
    tr = m.transformer
    tr.set_record_attn(True)
    m(tokens, xc, yc, ekv, fp16=fp16)
    ws = list(tr.ws)
    tr.set_record_attn(False)
    return ws


PATTERN_CASES = [
    # attn_order, width, depth, heads, n_ctx, blocks, prime_len, encoder_dims
    (12, 256, 16, 2, 96, 8, 24, 0),      # single enc-dec: block / transpose / prev-block / prime / dense, dh 64
    (2, 256, 6, 1, 128, 4, None, 0),     # upsampler pattern
    (0, 256, 3, 4, 80, None, None, 0),   # dense: two 64-query tiles, a ragged key tile
    (6, 256, 8, 2, 64, 4, None, 24),     # separate enc-dec: attn_func 6 reads the encoder's K from the layer cache
    (2, 4800, 3, 8, 64, 4, None, 0),     # dh 150 (5b_lyrics geometry): 4-byte staging
    (2, 1920, 3, 1, 64, 4, None, 0),     # dh 480 (the released upsamplers): scalar record kernel
]


@pytest.mark.parametrize("case", PATTERN_CASES)
def test_recorded_rows_are_the_softmax_of_the_pattern(case):
    from jukebox_b200.prior.autoregressive import ConditionalAutoregressive2D
    from oracle.synth import synth_state_dict
    order, width, depth, heads, n_ctx, blocks, prime_len, enc = case
    if enc:
        m = ConditionalAutoregressive2D((n_ctx,), 64, width=width, depth=depth, heads=heads, attn_order=order,
                                        blocks=blocks, x_cond=False, y_cond=True, encoder_dims=enc)
        sd = m.state_dict()
        w = synth_state_dict([(k, tuple(v.shape)) for k, v in sd.items() if k != "x_out.weight"], 31)
        w["x_out.weight"] = w["x_emb.weight"]
        m.load_state_dict({k: torch.from_numpy(v) for k, v in w.items()}, strict=True)
        m = m.cuda().eval()
    else:
        m, _ = _model(order, width, depth, heads, n_ctx, blocks, prime_len, seed=order + width)
    tr = m.transformer
    n = 3
    g = torch.Generator().manual_seed(order * 7 + width)
    tokens = torch.randint(0, m.bins, (n, n_ctx), generator=g).cuda()
    yc = torch.randn(n, 1, width, generator=g).cuda()
    ekv = torch.randn(n, enc, width, generator=g).cuda() if enc else None
    assert m._engine(n).prefill_capacity >= n_ctx
    ws16 = _forward_ws(m, tokens, yc, None, ekv, True)
    assert tr._f32 is None, "fp16 recording must not build the fp32 path"
    ws32 = _forward_ws(m, tokens, yc, None, ekv, False)
    assert len(ws16) == depth == len(ws32)
    masks = _masks(n_ctx, n_ctx // blocks if blocks else n_ctx)
    worst = 0.0
    for i, (w, w32) in enumerate(zip(ws16, ws32)):
        f = tr._attn_mods[i].attn_func
        assert w.dtype == torch.float16 and w.shape == w32.shape, (i, f, w.dtype, tuple(w.shape), tuple(w32.shape))
        assert torch.isfinite(w).all()
        w = w.float()
        s = w.sum(-1)
        if f == 6:
            assert w.shape == (n, heads, n_ctx, enc)
            assert torch.allclose(s, torch.ones_like(s), atol=1e-3)
        elif f == 7:        # music queries x the first prime_len keys: the rest of the padded prime block is dropped
            assert w.shape == (n, heads, n_ctx - prime_len, prime_len)
            assert float(s.max()) <= 1 + 1e-3
        else:
            mk = masks[f]
            assert w.shape == (n, heads, n_ctx, n_ctx)
            assert float(w.masked_fill(mk, 0).abs().max()) == 0.0, f"layer {i} (attn_func {f}) has mass outside its pattern"
            rows = mk.any(-1)
            assert torch.allclose(s[..., rows], torch.ones_like(s[..., rows]), atol=1e-3)
            if (~rows).any():
                assert float(s[..., ~rows].abs().max()) == 0.0
        d = float((w - w32).abs().max())
        worst = max(worst, d)
    print(f"order {order} width {width} dh {width // 4 // heads}: max |fp16 record - fp32 record| {worst:.2e}")
    assert worst < 1.5e-2


@pytest.mark.parametrize("tag", ["single_enc_dec", "sep_enc_dec"])
def test_recorded_weights_match_the_reference(tag):
    fx = Fixture(f"align_{tag}")
    prior = _make_prior(fx)
    tr = prior.prior.transformer
    layer = fx.cfg["layer"]
    z, y = torch.from_numpy(fx["z"]).cuda(), torch.from_numpy(fx["y"]).cuda()
    ws = prior.z_forward(z, [], y, fp16=True, get_attn_weights={layer})
    assert len(ws) == 1 and tr.ws == [] and tr._f32 is None
    ours = ws[0].float().cpu().numpy()
    ref16, ref32 = fx["w16"], fx["w32"]
    assert ws[0].dtype == torch.float16 and ours.shape == ref16.shape
    e16, e32, floor = (float(np.abs(ours - ref16).max()), float(np.abs(ours - ref32).max()),
                       float(np.abs(ref16 - ref32).max()))
    print(f"align_{tag}: max|ours16 - ref16| {e16:.2e}, max|ours16 - ref32| {e32:.2e}, max|ref16 - ref32| {floor:.2e}")
    assert e16 <= max(1e-3, 1.5 * floor)
    # the fp32 route returns the same shapes
    ws32 = prior.z_forward(z, [], y, fp16=False, get_attn_weights={layer})
    assert ws32[0].dtype == torch.float32 and ws32[0].shape == ws[0].shape


def test_window_beyond_the_prefill_capacity_records_on_the_fp32_path(monkeypatch):
    fx = Fixture("align_sep_enc_dec")
    prior = _make_prior(fx)
    tr = prior.prior.transformer
    layer = fx.cfg["layer"]
    z, y = torch.from_numpy(fx["z"]).cuda(), torch.from_numpy(fx["y"]).cuda()
    monkeypatch.setenv("JK_PREFILL_MAX", str(prior.n_ctx - 1))       # read when a plan is made
    tr.drop_engine()
    assert tr.prefill_capacity(z.shape[0]) == prior.n_ctx - 1
    ws = prior.z_forward(z, [], y, fp16=True, get_attn_weights={layer})
    assert tr._engine is None, "the capacity is known without building the decoder's engine"
    assert ws[0].dtype == torch.float32 and tr._f32 is not None
    assert ws[0].shape == fx["w32"].shape
    s = ws[0].sum(-1)
    assert torch.allclose(s, torch.ones_like(s), atol=1e-5)
    tr.drop_engine()


def test_more_items_than_one_engine_takes_record_on_the_fp32_path():
    """z_forward(fp16=True, get_attn_weights=...) with more than JK_MAX_BATCH items: no engine takes them in one
    prefill, so the pass records on the fp32 path (as before fp16 recording existed) instead of failing"""
    from jukebox_b200._lib import JK_MAX_BATCH
    fx = Fixture("align_single_enc_dec")
    prior = _make_prior(fx)
    tr = prior.prior.transformer
    layer = fx.cfg["layer"]
    reps = JK_MAX_BATCH // 2 + 1
    z = torch.from_numpy(fx["z"]).cuda().repeat(reps, 1)
    y = torch.from_numpy(fx["y"]).cuda().repeat(reps, 1)
    assert z.shape[0] > JK_MAX_BATCH
    ws = prior.z_forward(z, [], y, fp16=True, get_attn_weights={layer})
    assert tr._engine is None and ws[0].dtype == torch.float32
    assert ws[0].shape == (z.shape[0],) + fx["w32"].shape[1:]
    assert float((ws[0][:2].cpu() - torch.from_numpy(fx["w32"])).abs().max()) < 1e-4


@pytest.mark.parametrize("tag", ["single_enc_dec", "sep_enc_dec"])
def test_recording_leaves_the_forward_pass_unchanged(tag):
    fx = Fixture(f"align_{tag}")
    prior = _make_prior(fx)
    tr = prior.prior.transformer
    z, y = torch.from_numpy(fx["z"]).cuda(), torch.from_numpy(fx["y"]).cuda()
    outs = []
    for rec in (False, True, False):
        tr.set_record_attn({fx.cfg["layer"]} if rec else False)
        loss, metrics = prior.z_forward(z, [], y, fp16=True, get_preds=True)
        assert len(tr.ws) == int(rec)
        outs.append((loss.cpu(), metrics["preds"].cpu()))
    tr.set_record_attn(False)
    assert tr._f32 is None
    for loss, preds in outs[1:]:
        assert torch.equal(loss, outs[0][0]) and torch.equal(preds, outs[0][1])


@pytest.mark.parametrize("tag", ["single_enc_dec", "sep_enc_dec"])
def test_batched_alignment_windows_per_prefill_equal_item_by_item(tag, monkeypatch):
    from jukebox_b200 import align
    fx = Fixture(f"align_{tag}")
    prior = _make_prior(fx)
    prior.alignment_layer, prior.alignment_head = fx.cfg["layer"], 1
    z, y = torch.from_numpy(fx["z"]).cuda(), torch.from_numpy(fx["y"]).cuda()
    z = torch.cat([z, z.flip(1), (z + 1) % prior.l_bins])          # 6 items
    y = torch.cat([y, y, y.flip(0)])
    assert prior.prior.items_per_prefill(z.shape[0]) == z.shape[0]
    batched = align.hop_weights(prior, z, y, True)
    w32 = align.hop_weights(prior, z, y, False)
    monkeypatch.setattr(prior.prior, "items_per_prefill", lambda N: 1)
    single = align.hop_weights(prior, z, y, True)
    assert batched.shape == single.shape == w32.shape == (z.shape[0], prior.n_ctx, prior.n_tokens)
    assert np.array_equal(batched, single)
    print(f"align_{tag}: batched fp16 windows bit-identical to item by item; max|fp16 - fp32| "
          f"{float(np.abs(batched - w32).max()):.2e}")
