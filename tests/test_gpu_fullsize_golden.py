"""GPU parity at BASELINE geometry: the decode kernel against outputs of the UNMODIFIED reference
(tests/golden/full*.npz, written by oracle/make_golden_fullsize.py from /root/reference on CPU).

These fixtures reach what the tiny ones cannot: head_dim 256 / 150 (padded 160) / 480, 47-row K/V tiles with
split-KV merge, block_ctx 134, _prime_len 448, the transposed layout at p >> block_ctx, the dense layer at
8576 rows, 512 encoder rows, fp16 Conv1D parameters, and the K-split GEMM groups of width >= 1920.

Tolerance.  The north star asks 1e-3 relative on fp16 outputs.  Two correct fp16 executions of this path differ
by more than that on these stress weights (|h| up to 25: one fp16 ulp at 16 is 6e-4 of the maximum), and the test
MEASURES it instead of arguing it: oracle/transformer_torch.py replays the reference's own torch operators
(addmm / layer_norm / matmul / softmax, the same rounding points) on this GPU in fp16 - what the reference itself
computes on a GPU - and `ref_gpu_order_noise` is its distance to the reference's CPU fp16 output.  (The fixture's
`y16_alt`, the reference's CPU path with another chunking and thread count, turned out bit-identical to `y16`: the
CPU GEMM's blocking does not depend on either.)  Asserted: our error vs the reference's fp16 output
<= max(1e-3, 1.5 x that noise), AND we are not much further from the reference's fp32 output than its own fp16 path is
(x 1.6).  Every number is printed as one JSON line (pytest -s shows them).
"""
import json

import numpy as np
import pytest
import torch

from golden_util import Fixture, rel_err
from oracle.synth import synth_tensor

pytestmark = pytest.mark.gpu

CASES = ["full1b_o12", "full1b_o9", "full5b_o6", "fullup_o2"]


def record(row):
    print(json.dumps(row))


def build(fx):
    from jukebox_b200.transformer.transformer import Transformer
    from jukebox_b200.transformer.ops import _convert_conv_weights_to_fp16
    c = fx.cfg
    tr = Transformer(c["n_in"], c["n_ctx"], c["n_head"], c["n_depth"], mask=True, attn_order=c["attn_order"],
                     blocks=c["blocks"], encoder_dims=c["encoder_dims"] or None, prime_len=c["prime_len"])
    tr.load_state_dict({k: torch.from_numpy(v) for k, v in fx.weights().items()}, strict=True)
    assert [l.attn_func for l in tr._attn_mods] == c["attn_funcs"]
    if c["fp16_params"]:
        tr.apply(_convert_conv_weights_to_fp16)      # make_models.py:174-177
    return tr.cuda().eval()


@pytest.mark.parametrize("tag", CASES)
def test_decode_at_baseline_geometry_matches_reference(tag):
    fx = Fixture(tag)
    c = fx.cfg
    tr = build(fx)
    x = torch.from_numpy(synth_tensor("input.x", (c["bs"], c["n_ctx"], c["n_in"]), c["seed"])).cuda()
    enc = None
    if c["encoder_dims"]:
        enc = torch.from_numpy(synth_tensor("input.encoder_kv", (c["bs"], c["encoder_dims"], c["n_in"]), c["seed"])).cuda()
    probes = c["probes"]
    last = probes[-1] + 1
    ys = []
    with torch.no_grad():
        cur = 0
        for p in probes:                 # every position goes through the decode kernel, one launch each
            if p > cur:
                tr(x[:, cur:p].contiguous(), encoder_kv=enc, sample=True, fp16=True)
            ys.append(tr(x[:, p:p + 1].contiguous(), encoder_kv=enc, sample=True, fp16=True)[:, 0])
            cur = p + 1
        tr.check_cache(c["bs"], last, True)
    y = torch.stack(ys, 1).cpu().numpy()
    del tr
    torch.cuda.empty_cache()
    # the reference's operators on this GPU in fp16: the order noise between two legitimate executions
    from oracle.transformer_torch import TorchDecodeOracle
    orc = TorchDecodeOracle(fx.weights(), c["n_in"], c["n_ctx"], c["n_head"], c["n_depth"], c["attn_order"], c["blocks"],
                            c["encoder_dims"] or None, c["prime_len"], device="cuda", fp16_params=c["fp16_params"])
    yt, want = [], set(probes)
    with torch.no_grad():
        for p in range(last):
            out = orc.step(x[:, p], enc, True)
            if p in want:
                yt.append(out)
    yt = torch.stack(yt, 1).cpu().numpy()
    del orc
    torch.cuda.empty_cache()
    y16, y32, alt = fx["y16"], fx["y32"], fx["y16_alt"]
    e16, e32 = rel_err(y, y16), rel_err(y, y32)
    noise, ref1632 = rel_err(yt, y16), rel_err(y16, y32)
    per_probe = [rel_err(y[:, i], y16[:, i]) for i in range(len(probes))]
    row = dict(fixture=tag, api="Transformer.forward(sample=True, fp16=True), one decode launch per position",
               ours_vs_ref_fp16=e16, ours_vs_ref_fp32=e32, ref_fp16_order_noise=noise, ref_fp16_vs_ref_fp32=ref1632,
               ours_vs_ref_ops_on_gpu=rel_err(y, yt), ref_cpu_alt_chunking_noise=rel_err(alt, y16),
               worst_probe=int(probes[int(np.argmax(per_probe))]), probes=probes,
               per_probe_vs_ref_fp16=[float(f"{v:.3e}") for v in per_probe], max_abs_ref=float(np.abs(y16).max()))
    record(row)
    print(json.dumps(row))
    assert np.isfinite(y).all()
    assert e16 <= max(1e-3, 1.5 * noise), (e16, noise)
    assert e32 <= 1.6 * ref1632 + 1e-4, (e32, ref1632)
