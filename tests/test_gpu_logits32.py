"""GPU check of the logits above 16 samples (the reference's own check_sample property, autoregressive.py:361-387): the
logits a 17- or 32-sample primed, top-k sampling run computes step by step equal those of a whole-sequence forward
over the tokens it sampled.  Run with the tensor-core logits GEMM and with the fp32 FMA logits (JK_NO_LOGITS_MMA), so
both logits paths of the 32-row kernel and the prefill of the prime at M = N * P are covered."""
import numpy as np
import pytest
import torch

from golden_util import rel_err
from oracle.synth import synth_state_dict

pytestmark = pytest.mark.gpu

TOL_LOGITS = 3e-3      # tests/test_gpu_prior.py


@pytest.mark.parametrize("logits", ["gemm", "fma"])
@pytest.mark.parametrize("n", [17, 32])
def test_sampled_logits_match_forward_above_16_samples(n, logits, monkeypatch):
    from jukebox_b200.prior.autoregressive import ConditionalAutoregressive2D
    if logits == "fma":
        monkeypatch.setenv("JK_NO_LOGITS_MMA", "1")       # read when the engine is planned
    D, bins, width, P = 64, 100, 128, 20                  # width 128: K split 2, so the logits GEMM can be planned
    m = ConditionalAutoregressive2D((D,), bins, width=width, depth=4, heads=2, attn_order=2, blocks=8,
                                    x_cond=True, y_cond=True)
    sd = synth_state_dict([(k, tuple(v.shape)) for k, v in m.state_dict().items()], 31)
    m.load_state_dict({k: torch.from_numpy(v) for k, v in sd.items()})
    m = m.cuda().eval()
    rng = np.random.RandomState(n)
    xc = torch.from_numpy(rng.standard_normal((n, D, width)).astype(np.float32) * 0.5).cuda()
    yc = torch.from_numpy(rng.standard_normal((n, 1, width)).astype(np.float32) * 0.5).cuda()
    prime = torch.from_numpy(rng.randint(0, bins, (n, P))).cuda()
    torch.manual_seed(n)
    x, preds = m.primed_sample(n, prime.clone(), xc, yc, None, fp16=True, temp=0.9, top_k=10, get_preds=True)
    assert m._engine(n).has_logits_gemm == (logits == "gemm")
    assert x.shape == (n, D) and torch.equal(x[:, :P], prime)
    assert int(x.min()) >= 0 and int(x.max()) < bins
    _, want = m(x, xc, yc, fp16=True, get_preds=True)
    p, w = preds.cpu().numpy(), want.cpu().numpy()
    assert np.isfinite(p).all()
    e = rel_err(p, w)
    per_row = [rel_err(p[r], w[r]) for r in range(n)]
    print(f"n {n} {logits}: sampled logits vs forward {e:.2e}, rows 16.. {max(per_row[16:]):.2e}")
    assert e < TOL_LOGITS, (e, per_row)
