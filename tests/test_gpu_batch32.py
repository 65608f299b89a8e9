"""GPU parity of the decode engine above 16 samples: the 32-row kernel (two m16 MMA tiles against every weight
fragment) against the oracle and the reference's own outputs, and against the 16-row kernel on the same samples."""
import numpy as np
import pytest
import torch

from golden_util import Fixture, rel_err
from oracle.synth import synth_state_dict, synth_tensor
from oracle.transformer_np import TransformerOracle
from test_gpu_transformer import CASES, TOL, build

pytestmark = pytest.mark.gpu


def _oracle_run(sd, c, x, enc=None):
    orc = TransformerOracle(sd, c["n_in"], c["n_ctx"], c["n_head"], c["n_depth"], c["attn_order"], c["blocks"],
                            c["encoder_dims"], c["prime_len"])
    return np.stack([orc.step(x[:, i], enc, True) for i in range(x.shape[1])], 1)


@pytest.mark.parametrize("tag", CASES)
def test_oracle_agrees_above_16_samples(tag):
    fx = Fixture(f"transformer_{tag}")
    c = fx.cfg
    tr = build(fx)
    for bs in (17, 24, 32):
        rng = np.random.RandomState(100 + bs)
        x = rng.standard_normal((bs, c["n_ctx"], c["n_in"])).astype(np.float32)
        enc = None
        if c["encoder_dims"]:
            enc = rng.standard_normal((bs, c["encoder_dims"], c["n_in"])).astype(np.float32)
        ref = _oracle_run(fx.weights(), c, x, enc)
        run = lambda a, b: tr(torch.from_numpy(x[a:b]).cuda(), encoder_kv=None if enc is None else torch.from_numpy(enc[a:b]).cuda(),
                              sample=True, fp16=True).cpu().numpy()
        with torch.no_grad():
            tr.del_cache()
            y = run(0, bs)
            halves = []
            for a in (0, 16):              # the same samples through the 16-row kernel
                tr.del_cache()
                halves.append(run(a, min(a + 16, bs)))
        e32, e16 = rel_err(y, ref), rel_err(np.concatenate(halves), ref)
        # On these stress weights some seeds put the fp16 order noise of order12 above TOL for the 16-row kernel too
        # (measured: 6.2e-3 at bs 24, all of it in rows 0..15): the 32-row kernel must not be further from the oracle.
        assert e32 < max(TOL, 1.25 * e16), (tag, bs, e32, e16)


def test_eight_heads_at_32_samples():
    """B * H = 256 attention items over the grid: several (sample, head) items per CTA at 32 rows."""
    from jukebox_b200.transformer.transformer import Transformer
    n_in, n_ctx, heads, depth, blocks = 128, 48, 8, 4, 4
    tr = Transformer(n_in, n_ctx, heads, depth, mask=True, attn_order=12, blocks=blocks, prime_len=8)
    sd = synth_state_dict([(k, tuple(v.shape)) for k, v in tr.state_dict().items()], 21)
    tr.load_state_dict({k: torch.from_numpy(v) for k, v in sd.items()})
    tr = tr.cuda().eval()
    c = dict(n_in=n_in, n_ctx=n_ctx, n_head=heads, n_depth=depth, attn_order=12, blocks=blocks, encoder_dims=0,
             prime_len=8)
    x = np.random.RandomState(7).standard_normal((32, n_ctx, n_in)).astype(np.float32)
    ref = _oracle_run(sd, c, x)
    with torch.no_grad():
        y = tr(torch.from_numpy(x).cuda(), sample=True, fp16=True).cpu().numpy()
    assert rel_err(y, ref) < TOL, rel_err(y, ref)


@pytest.mark.parametrize("tag", ["order12", "order2_ragged"])
def test_one_32_row_step_agrees_with_two_16_row_halves(tag):
    fx = Fixture(f"transformer_{tag}")
    c = fx.cfg
    tr = build(fx)
    x = torch.from_numpy(np.random.RandomState(5).standard_normal((32, c["n_ctx"], c["n_in"])).astype(np.float32)).cuda()
    with torch.no_grad():
        y32 = tr(x, sample=True, fp16=True)
        halves = []
        for h in range(2):                 # the engine built for 32 launches the 16-row kernel for 16 samples
            tr.del_cache()
            halves.append(tr(x[16 * h:16 * (h + 1)].contiguous(), sample=True, fp16=True))
    y16 = torch.cat(halves, 0)
    assert tr._engine.max_batch == 32
    # not bitwise: the split-KV partition of the attention follows the CTAs per (sample, head)
    assert rel_err(y32.cpu().numpy(), y16.cpu().numpy()) < TOL


@pytest.mark.parametrize("tag", ["full1b_o12", "full1b_o9", "fullup_o2"])
def test_baseline_geometry_at_32_samples(tag):
    """the fixture's batch tiled to 32 rows: every replica meets the bounds of test_gpu_fullsize_golden.py"""
    from test_gpu_fullsize_golden import build as build_full
    fx = Fixture(tag)
    c = fx.cfg
    tr = build_full(fx)
    bs = c["bs"]
    x = torch.from_numpy(synth_tensor("input.x", (bs, c["n_ctx"], c["n_in"]), c["seed"])).cuda()
    reps = (32 + bs - 1) // bs
    xt = x.repeat(reps, 1, 1)[:32].contiguous()
    probes = c["probes"]
    ys = []
    with torch.no_grad():
        cur = 0
        for p in probes:
            if p > cur:
                tr(xt[:, cur:p].contiguous(), sample=True, fp16=True)
            ys.append(tr(xt[:, p:p + 1].contiguous(), sample=True, fp16=True)[:, 0])
            cur = p + 1
    y = torch.stack(ys, 1).cpu().numpy()
    assert np.isfinite(y).all()
    y16, y32 = fx["y16"], fx["y32"]
    ref1632 = rel_err(y16, y32)
    for r in range(32):
        e16, e32 = rel_err(y[r:r + 1], y16[r % bs:r % bs + 1]), rel_err(y[r:r + 1], y32[r % bs:r % bs + 1])
        # the order-noise bound of test_gpu_fullsize_golden.py, taken at its 3e-3 ceiling (1.5 x the largest measured noise)
        assert e16 <= 3e-3, (tag, r, e16)
        assert e32 <= 1.6 * ref1632 + 1e-4 or e32 <= 1.6 * rel_err(y16[r % bs:r % bs + 1], y32[r % bs:r % bs + 1]) + 1e-4, (tag, r, e32)
