"""Host flow of prior evaluation without a GPU: ConditionalAutoregressive2D.logprob / token_stats / layer_acts cut their
items into the pieces one engine takes, with the engine replaced by a fake; SimplePrior.z_forward / score / token_stats /
layer_acts condition a window in one way, with the conditioner, the lyric encoder and the autoregressive model replaced
by recorders."""
import pytest
import torch

from golden_util import Fixture


class FakeEngine:
    """stands in for DecodeEngine: every output row of an item is its first token, so rows show which item they hold"""

    def __init__(self, prefill_capacity):
        self.prefill_capacity = prefill_capacity
        self.prefills, self.steps = [], []
        self.position = 0

    def reset(self, t0=0):
        self.position = t0

    def prefill(self, n, P, tokens=None, h_out=None, n_layers=0, capture=None, **kw):
        self.prefills.append(n)
        first = tokens[:n, :1].float()
        if h_out is not None:
            h_out.copy_(first[:, :, None].expand(h_out.shape))
        for k in (capture or {}).values():
            k.out.copy_(first[:, :, None].expand(k.out.shape) if k.out.dim() == 3 else first.expand(k.out.shape))
        self.position = P

    def step(self, n, tokens=None, h_out=None, **kw):
        self.steps.append(n)
        h_out.copy_(tokens[:n, :1].float().expand(h_out.shape))
        self.position += 1


def _ca2d(monkeypatch, rows_with_prefill):
    """a model whose engines take a prefill up to `rows_with_prefill` items (0: none at any size)"""
    import jukebox_b200.score as score
    from jukebox_b200.prior import autoregressive as ar
    m = ar.ConditionalAutoregressive2D((24,), 64, width=64, depth=3, heads=1, attn_order=0, blocks=None).eval()
    eng = FakeEngine(64 if rows_with_prefill else 0)
    built = []
    monkeypatch.setattr(m, "_engine", lambda n: built.append(n) or eng)
    monkeypatch.setattr(m.transformer, "prefill_capacity", lambda n: 64 if n <= rows_with_prefill else 0)
    # x_out and the score kernels: the first activation of each row
    monkeypatch.setattr(score, "xout_logprob", lambda h, w, targets: h[:, 0].clone())
    monkeypatch.setattr(score, "xout_stats", lambda h, w, targets=None, top_k=0: score.TokenStats(
        h[:, 0].clone(), h[:, 0].clone(), None, None, h[:, 0].clone()))
    return m, eng, built


def _items(N, D=24):
    return (torch.arange(N)[:, None] + torch.zeros(1, D, dtype=torch.long)) % 64       # item i: tokens all i


def test_more_items_than_one_engine_takes_go_in_pieces_in_item_order(monkeypatch):
    """an engine that takes 16 items (5b_lyrics): 20 items are scored as 16, then 4, by every evaluation method"""
    m, eng, built = _ca2d(monkeypatch, rows_with_prefill=16)
    x = _items(20)
    want = torch.arange(20).float()[:, None]
    assert torch.equal(m.logprob(x), want.expand(20, 24))
    assert torch.equal(m.token_stats(x[:, :10]).entropy, want.expand(20, 10))
    acts = m.layer_acts(x, layers=(0, 2), pool=False)
    assert all(torch.equal(a, want[:, :, None].expand(20, 24, 64)) for a in acts.values())
    assert built == [16, 4] * 3 and eng.prefills == [16, 4] * 3 and eng.steps == []


def test_without_a_prefill_pieces_of_up_to_32_items_step_their_tokens(monkeypatch):
    m, eng, built = _ca2d(monkeypatch, rows_with_prefill=0)
    assert m.items_per_prefill(40) == 0
    lp = m.logprob(_items(40))
    assert torch.equal(lp, torch.arange(40).float()[:, None].expand(40, 24))
    assert built == [32, 8] and eng.prefills == [] and eng.steps == [32] * 24 + [8] * 24
    with pytest.raises(RuntimeError, match="prefill capacity 0"):
        m.layer_acts(_items(4), layers=(1,))


# ---- SimplePrior: one conditioning for every evaluation method --------------------------------------------------------
def _prior(tag):
    from jukebox_b200.hparams import setup_hparams
    from jukebox_b200.make_models import make_vqvae, make_prior
    c = Fixture(f"prior_{tag}").cfg
    vq = make_vqvae(setup_hparams(c["vq_name"], dict(restore_vqvae="", **c["vq_over"])), "cpu")
    return make_prior(setup_hparams(c["pr_name"], dict(restore_prior="", **c["pr_over"])), vq, "cpu").eval()


@pytest.mark.parametrize("tag", ["single_enc_dec", "sep_enc_dec", "upsampler"])
def test_every_evaluation_method_conditions_a_window_alike(tag, monkeypatch):
    import jukebox_b200.score as score
    from jukebox_b200.score import TokenStats
    prior = _prior(tag)
    ca = prior.prior
    N, W = 3, ca.width
    z = torch.randint(0, 2, (N, prior.n_ctx))

    def get_cond(z_conds, y):
        g = torch.Generator().manual_seed(int(y.sum()) if y is not None else 0)
        x_cond = torch.randn(N, prior.n_ctx, W, generator=g) if (prior.x_cond or prior.y_cond) else None
        y_cond = torch.randn(N, 1, W, generator=g) if prior.y_cond else None
        lyric = torch.randint(0, 2, (N, prior.n_tokens), generator=g) if prior.n_tokens else None
        return x_cond, y_cond, lyric

    def get_encoder_kv(lyric, fp16=False, sample=False):
        assert not sample
        return None if not prior.has_lyric_encoder else lyric[:, :, None].float().expand(N, lyric.shape[1], W) + fp16

    seen = {}

    def recorder(name, result):
        def call(x, x_cond=None, y_cond=None, encoder_kv=None, fp16=False, t0=0, **kw):
            seen[name] = (x, x_cond, y_cond, encoder_kv, fp16, t0)
            return result(x, kw)
        return call
    monkeypatch.setattr(prior, "get_cond", get_cond)
    monkeypatch.setattr(prior, "get_encoder_kv", get_encoder_kv)
    monkeypatch.setattr(prior, "get_prime_loss", lambda enc, lyric: torch.tensor(0.0))
    monkeypatch.setattr(score, "xout_logprob", lambda h, w, targets: torch.zeros(h.shape[0]))
    zero = torch.tensor(0.0)
    loss = lambda x, kw: ((zero, zero) if kw.get("get_sep_loss") else zero, None)
    monkeypatch.setattr(ca, "forward", recorder("z_forward", loss))
    monkeypatch.setattr(ca, "logprob", recorder("score", lambda x, kw: torch.zeros(x.shape)))
    monkeypatch.setattr(ca, "token_stats", recorder("token_stats", lambda x, kw: TokenStats(
        *(torch.zeros(x.shape) for _ in range(2)), None, None, torch.zeros(x.shape))))
    monkeypatch.setattr(ca, "layer_acts", recorder("layer_acts", lambda x, kw: {}))
    y = torch.ones(N, 4, dtype=torch.long) if prior.y_cond else None
    for fp16 in (False, True):
        seen.clear()
        prior.z_forward(z, [], y, fp16=fp16)
        prior.score(z, [], y, fp16=fp16)
        prior.token_stats(z, [], y, fp16=fp16)
        prior.layer_acts(z, [], y, layers=(1,), fp16=fp16)
        assert sorted(seen) == ["layer_acts", "score", "token_stats", "z_forward"]
        x_cond, y_cond, lyric = get_cond([], y)
        if prior.single_enc_dec:
            want_x, x_cond = prior.prior_preprocess([lyric, z], [None, x_cond])
        else:
            want_x = z
        enc = None if prior.single_enc_dec else get_encoder_kv(lyric, fp16)
        for name, (x, xc, yc, ek, f, t0) in seen.items():
            for got, want in ((x, want_x), (xc, x_cond), (yc, y_cond), (ek, enc)):
                assert (got is None and want is None) or torch.equal(got, want), (tag, name)
            assert f == fp16
            if name == "layer_acts":
                assert t0 == (ca.prime_len if prior.single_enc_dec else 0)
