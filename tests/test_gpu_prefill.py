"""Chunked prefill (jk_prior_prefill: wgmma GEMMs over all given positions) against stepping the same
tokens one by one through the decode kernel - the equality the reference asserts in its own
check_chunks (prior/autoregressive.py:330-338) - and against the oracle."""
import numpy as np
import pytest
import torch

from golden_util import rel_err

pytestmark = pytest.mark.gpu

# widths are 256 so that every GEMM K (width, n_state = width/4, mlp) is a multiple of the GEMM K block;
# the two paths share every fp16 rounding point and differ in fp32 summation order (register accumulator
# over K blocks vs 8 warps x k16 partials), i.e. the noise floor documented in test_gpu_prior.py
TOL = 3e-3


def _model(attn_order, width, depth, heads, n_ctx, blocks, prime_len=None, bins=64, seed=0, x_cond=False, y_cond=True):
    from jukebox_b200.prior.autoregressive import ConditionalAutoregressive2D
    from oracle.synth import synth_state_dict
    single = prime_len is not None
    m = ConditionalAutoregressive2D((n_ctx,), bins, width=width, depth=depth, heads=heads, attn_order=attn_order,
                                    blocks=blocks, x_cond=x_cond, y_cond=y_cond,
                                    prime_len=prime_len, merged_decoder=single)
    sd = m.state_dict()
    tied = m.share_x_emb_x_out
    w = synth_state_dict([(k, tuple(v.shape)) for k, v in sd.items() if not (tied and k == "x_out.weight")], seed)
    if tied and "x_out.weight" in sd:
        w["x_out.weight"] = w["x_emb.weight"]
    m.load_state_dict({k: torch.from_numpy(v) for k, v in w.items()}, strict=True)
    return m.cuda().eval(), w


def _run(m, n, tokens, P, K, yc, xc, use_prefill):
    """logits of positions P..P+K-1 after the first P given tokens"""
    ca = m
    ca.transformer.del_cache()
    eng = ca._engine(n)
    eng.reset(0)
    out = torch.empty(n, K, ca.bins, device="cuda")
    lbuf = torch.empty(n, ca.bins, device="cuda")
    if use_prefill:
        assert eng.prefill_capacity >= P
        eng.prefill(n, P, tokens=tokens, y_cond=yc, x_cond=xc)
    else:
        for _ in range(P):
            eng.step(n, tokens=tokens, y_cond=yc, x_cond=xc)
    assert eng.position == P
    for k in range(K):
        eng.step(n, tokens=tokens, y_cond=yc, x_cond=xc, logits=lbuf)
        out[:, k] = lbuf
    torch.cuda.synchronize()
    return out.cpu().numpy()


CASES = [
    # attn_order, width, depth, heads, n_ctx, blocks, prime_len, P
    (12, 256, 16, 2, 96, 8, 24, 24),    # single enc-dec pattern set (block / transpose / prev / prime), P = prime
    (12, 256, 16, 2, 96, 8, 24, 61),    # given tokens run past the prime and past several blocks (ring layouts)
    (2, 256, 6, 1, 64, 4, None, 33),    # upsampler-like stack, one head
    (0, 256, 3, 4, 48, None, None, 17),  # dense
    (2, 320, 6, 2, 64, 4, None, 33),    # K tail: n_state 80 is not a multiple of the 64-wide GEMM K block (5b: 1200, upsamplers: 480)
    (2, 256, 6, 1, 1024, 8, None, 700),  # a long run of given tokens (continuation windows re-prime thousands)
    (2, 4800, 3, 8, 64, 4, None, 33),   # 5b_lyrics geometry: n_state 1200, head_dim 150 - head rows are not 16-byte aligned
    (0, 1024, 2, 1, 160, None, None, 150),  # head_dim 256, dense: several key tiles per query tile
]


@pytest.mark.parametrize("case", CASES)
def test_prefill_matches_stepping(case):
    order, width, depth, heads, n_ctx, blocks, prime_len, P = case
    m, _ = _model(order, width, depth, heads, n_ctx, blocks, prime_len, seed=P)
    n, K = 5, 6
    g = torch.Generator().manual_seed(order * 100 + P)
    tokens = torch.randint(0, m.bins, (n, n_ctx), generator=g).cuda()
    yc = torch.randn(n, width, generator=g).cuda()
    a = _run(m, n, tokens, P, K, yc, None, use_prefill=False)
    b = _run(m, n, tokens, P, K, yc, None, use_prefill=True)
    e = rel_err(b, a)
    print(f"prefill vs stepping, order {order} P {P}: {e:.2e}")
    assert np.isfinite(b).all() and e < TOL


def test_prefill_against_oracle_and_public_api():
    """primed_sample takes the prefill path (no get_preds); its continuation logits match the oracle fed
    with the same tokens"""
    from oracle.transformer_np import PriorOracle
    order, width, depth, heads, n_ctx, blocks, prime_len = 12, 256, 16, 2, 96, 8, 24
    m, w = _model(order, width, depth, heads, n_ctx, blocks, prime_len, seed=3)
    n, P, K = 3, 24, 4
    g = torch.Generator().manual_seed(7)
    tokens = torch.randint(0, m.bins, (n, n_ctx), generator=g).cuda()
    yc = torch.randn(n, width, generator=g).cuda()
    got = _run(m, n, tokens, P, K, yc, None, use_prefill=True)
    orc = PriorOracle(w, n_ctx, m.bins, width, depth, heads, attn_order=order, blocks=blocks, x_cond=False, y_cond=True,
                      merged_decoder=True, prime_len=prime_len)
    ref = orc.logits(tokens.cpu().numpy(), None, yc.cpu().numpy()[:, None, :], None, True, n_steps=P + K)
    e = rel_err(got, ref[:, P:P + K])
    print(f"prefill + steps vs oracle fp16: {e:.2e}")
    assert e < 5e-3
    # public API: same seed, with and without the prefill, must sample from (numerically) the same
    # distributions - compare the tokens drawn at a low temperature where ties cannot flip
    torch.manual_seed(0)
    z1 = m.primed_sample(n, tokens[:, :P].clone(), None, yc[:, None, :], fp16=True, temp=0.05, sample_tokens=P + 8)
    assert z1.shape == (n, P + 8) and torch.equal(z1[:, :P], tokens[:, :P])


@pytest.mark.parametrize("bins", [77, 2127 % 256 + 8])
def test_logits_gemm_with_ragged_bins_against_oracle(bins):
    """the logits Conv1D (hi / lo fp16 split of the fp32 x_out on the tensor cores, decode_engine.cu) with a vocabulary
    that is not a multiple of the 8-column MMA group (1b_lyrics: 2127 = 2048 + 79): the last group is padded with zero
    weights and its padding columns are never stored; logits against the oracle's fp32 product"""
    from oracle.transformer_np import PriorOracle
    order, width, depth, heads, n_ctx, blocks = 2, 256, 3, 2, 64, 4
    m, w = _model(order, width, depth, heads, n_ctx, blocks, None, bins=bins, seed=bins)
    n, P, K = 5, 9, 4
    g = torch.Generator().manual_seed(bins)
    tokens = torch.randint(0, m.bins, (n, n_ctx), generator=g).cuda()
    yc = torch.randn(n, width, generator=g).cuda()
    got = _run(m, n, tokens, P, K, yc, None, use_prefill=False)
    orc = PriorOracle(w, n_ctx, m.bins, width, depth, heads, attn_order=order, blocks=blocks, x_cond=False, y_cond=True)
    ref = orc.logits(tokens.cpu().numpy(), None, yc.cpu().numpy()[:, None, :], None, True, n_steps=P + K)
    assert got.shape[-1] == bins and np.isfinite(got).all()
    e = rel_err(got, ref[:, P:P + K])
    print(f"bins {bins}: logits vs oracle fp16 {e:.2e}")
    assert e < 5e-3


def test_only_encode_forward_uses_prefill():
    """forward() of an only_encode stack (the lyric encoder of separated priors): prefill h_out vs stepping"""
    from jukebox_b200.prior.autoregressive import ConditionalAutoregressive2D
    m, _ = _model(2, 256, 4, 1, 64, 4, None, seed=11, y_cond=False)
    n, D, W = 4, 64, 256
    g = torch.Generator().manual_seed(5)
    tokens = torch.randint(0, m.bins, (n, D), generator=g).cuda()
    eng = m._engine(n)
    m.transformer.del_cache()
    eng.reset(0)
    a = torch.empty(n, D, W, device="cuda")
    eng.prefill(n, D, tokens=tokens, h_out=a)
    m.transformer.del_cache()
    eng.reset(0)
    b = torch.empty(n, D, W, device="cuda")
    for i in range(D):
        o = torch.empty(n, W, device="cuda")
        eng.step(n, tokens=tokens, h_out=o)
        b[:, i] = o
    e = rel_err(a.cpu().numpy(), b.cpu().numpy())
    print(f"only_encode prefill vs stepping: {e:.2e}")
    assert e < 5e-3


def test_prefill_with_encoder_decoder_layers_and_get_preds(monkeypatch):
    """enc-dec stacks (5b_lyrics: attn_func 6 layers read the lyric encoder's K/V) take the prefill path, and
    primed_sample(get_preds=True) returns the given positions' logits from it: against stepping and the golden"""
    from golden_util import Fixture
    from jukebox_b200.prior.autoregressive import ConditionalAutoregressive2D
    from oracle.synth import synth_state_dict
    n_ctx, width, bins, enc = 64, 256, 64, 24
    m = ConditionalAutoregressive2D((n_ctx,), bins, width=width, depth=8, heads=2, attn_order=6, blocks=4,
                                    x_cond=True, y_cond=True, encoder_dims=enc)
    sd = m.state_dict()
    w = synth_state_dict([(k, tuple(v.shape)) for k, v in sd.items() if k != "x_out.weight"], 21)
    w["x_out.weight"] = w["x_emb.weight"]
    m.load_state_dict({k: torch.from_numpy(v) for k, v in w.items()}, strict=True)
    m = m.cuda().eval()
    assert any(b.attn_func == 6 for b in m.transformer._attn_mods)
    n, P = 3, 41
    g = torch.Generator().manual_seed(9)
    tokens = torch.randint(0, bins, (n, n_ctx), generator=g).cuda()
    yc = torch.randn(n, 1, width, generator=g).cuda()
    xc = (0.1 * torch.randn(n, n_ctx, width, generator=g)).cuda()
    ekv = torch.randn(n, enc, width, generator=g).cuda()
    eng = m._engine(n)
    assert eng.prefill_capacity >= n_ctx - 1
    outs = []
    for cap in (None, 1):          # prefill in one pass / capacity 1 = every given token stepped
        if cap is not None:
            monkeypatch.setattr(type(eng), "prefill_capacity", property(lambda self: 1))
        torch.manual_seed(0)
        x, preds = m.primed_sample(n, tokens[:, :P].clone(), xc, yc, ekv, fp16=True, temp=0.05, get_preds=True,
                                   sample_tokens=P + 6)
        assert torch.equal(x[:, :P], tokens[:, :P])
        outs.append((x.cpu(), preds.cpu().numpy()))
    e = rel_err(outs[0][1], outs[1][1])
    print(f"enc-dec prefill with get_preds vs stepping: logits {e:.2e}")
    assert np.isfinite(outs[0][1]).all() and e < TOL
