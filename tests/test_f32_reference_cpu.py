"""The float64 layer restatement (oracle/transformer_f64.py) pinned against the reference's own fp32 outputs.

Stacked over the tiny fixtures it must reproduce `y32` (sampling mode, one position per call) and `yfull32` (forward
mode) of the unmodified reference - far inside the 2e-5 the fp32 path is held to, since the only difference left is
the reference's fp32 rounding.  The GPU tests use this restatement as the yardstick of csrc/f32_path.cu at the priors'
real geometry, so it is checked here first, on the CPU."""
import numpy as np
import pytest
import torch

from golden_util import Fixture, rel_err
from oracle.transformer_f64 import attended_keys, layer_f64, block_params, stack_f64
from oracle.transformer_np import prime_len_padded

TOL = 2e-6          # a tenth of the fp32 path's 2e-5


def _stack(fx):
    c = fx.cfg
    bc = c["n_ctx"] // c["blocks"]
    prime = prime_len_padded(c["prime_len"], c["blocks"]) if c["prime_len"] else None
    x = torch.from_numpy(fx["x"]).double()
    enc = torch.from_numpy(fx["encoder_kv"]).double() if "encoder_kv" in fx else None
    return stack_f64(fx.weights(), x, c["attn_funcs"], c["n_head"], bc, prime, enc).numpy()


@pytest.mark.parametrize("tag", ["order9", "order6", "order12", "order2_ragged"])
def test_float64_stack_reproduces_reference_fp32(tag):
    fx = Fixture(f"transformer_{tag}")
    y = _stack(fx)
    e32 = rel_err(y, fx["y32"])
    efull = rel_err(y, fx["yfull32"]) if "yfull32" in fx else e32
    print(f"transformer_{tag}: float64 stack vs reference fp32 sampling {e32:.2e}, forward {efull:.2e}")
    assert e32 <= TOL and efull <= TOL
    # and it is not the fp16 answer
    assert rel_err(y, fx["y16"]) > 10 * TOL


def test_query_subset_and_weights():
    """evaluating a subset of queries gives the same rows as all of them; recorded weights are the pattern's softmax"""
    fx = Fixture("transformer_order12")
    c = fx.cfg
    bc = c["n_ctx"] // c["blocks"]
    prime = prime_len_padded(c["prime_len"], c["blocks"])
    x = torch.from_numpy(fx["x"]).double()
    sd = fx.weights()
    for d in (0, 1, 2, 15):
        af = c["attn_funcs"][d]
        p = block_params(sd, d)
        full = layer_f64(p, x, range(c["n_ctx"]), af, c["n_head"], bc, prime)
        qs = [0, 1, bc - 1, bc, bc + 1, prime - 1, prime, prime + 1, c["n_ctx"] - 1]
        sub = layer_f64(p, x, qs, af, c["n_head"], bc, prime)
        assert torch.allclose(sub["y"], full["y"][:, qs], rtol=0, atol=1e-12)
        for i, q in enumerate(qs):
            rows = attended_keys(af, q, bc, prime, c["n_ctx"])
            w = sub["w"][:, :, i]
            if rows is None:
                assert float(w.abs().max()) == 0.0
                continue
            mask = torch.zeros(c["n_ctx"], dtype=torch.bool)
            mask[torch.as_tensor(rows)] = True
            assert float(w[..., ~mask].abs().max() if (~mask).any() else 0.0) == 0.0
            assert torch.allclose(w.sum(-1), torch.ones_like(w[..., 0]), atol=1e-12)
        # a shifted key set is another answer
        wrong = layer_f64(p, x, qs[1:], af, c["n_head"], bc, prime, shift=bc if af == 3 else 1)
        assert float((wrong["y"] - sub["y"][:, 1:]).abs().amax(-1).min()) > 1e-3


def test_bound_covers_reference_fp32_rounding():
    """the first-order bound of one layer covers the reference's own fp32 execution of that layer (stat model: the
    reference's CPU GEMMs sum in another order, which the worst-case model covers too)"""
    fx = Fixture("transformer_order6")
    c = fx.cfg
    bc = c["n_ctx"] // c["blocks"]
    x = torch.from_numpy(fx["x"]).double()
    enc = torch.from_numpy(fx["encoder_kv"]).double()
    sd = fx.weights()
    qs = list(range(c["n_ctx"]))
    for d in range(c["n_depth"]):
        p = block_params(sd, d)
        af = c["attn_funcs"][d]
        # the same layer in fp32 through torch (another summation order)
        p32 = {k: v.float() for k, v in p.items()}
        y32 = layer_f64(p32, x.float(), qs, af, c["n_head"], bc, None, enc.float())["y"].double()
        ratios = {}
        for model in ("worst", "stat"):
            ref = layer_f64(p, x, qs, af, c["n_head"], bc, None, enc, bound=model)
            ratios[model] = float(((y32 - ref["y"]).abs() / ref["ey"]).max())
        print(f"order6 layer {d} (attn_func {af}): torch fp32 vs float64 / bound: worst-case {ratios['worst']:.2e}, "
              f"stat {ratios['stat']:.3f}")
        assert ratios["worst"] <= ratios["stat"] <= 1.0
        x = ref["y"]
