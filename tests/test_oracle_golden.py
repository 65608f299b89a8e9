"""Pin the oracle (oracle/*.py, numpy) against the reference's own outputs (tests/golden/).

These are the `-m "not gpu"` parity checks: if they pass, the oracle restates the
reference's algorithm, and the GPU tests may use the oracle as their checker at any size."""
import numpy as np
import pytest

from golden_util import Fixture, rel_err
from oracle.transformer_np import TransformerOracle, PriorOracle
from oracle.vqvae_np import VQVAEOracle

TR_CASES = ["order9", "order6", "order12", "order2_ragged"]


@pytest.mark.parametrize("tag", TR_CASES)
@pytest.mark.parametrize("fp16", [False, True])
def test_transformer_decode_matches_reference(tag, fp16):
    fx = Fixture(f"transformer_{tag}")
    c = fx.cfg
    orc = TransformerOracle(fx.weights(), c["n_in"], c["n_ctx"], c["n_head"], c["n_depth"], c["attn_order"],
                            c["blocks"], c["encoder_dims"], c["prime_len"])
    assert orc.attn_funcs == c["attn_funcs"]
    x = fx["x"]
    enc = fx["encoder_kv"] if "encoder_kv" in fx else None
    y = np.stack([orc.step(x[:, i], enc, fp16) for i in range(c["n_ctx"])], 1)
    ref = fx["y16" if fp16 else "y32"]
    # fp32: summation-order noise only.  fp16: the reference's CPU half GEMMs and ours round
    # the same fp32 accumulations, a few results land on the other side of a rounding boundary.
    tol = 2e-3 if fp16 else 2e-5
    assert rel_err(y, ref) < tol, rel_err(y, ref)


@pytest.mark.parametrize("tag", ["order9", "order6", "order2_ragged"])
def test_transformer_forward_mode_matches_reference(tag):
    fx = Fixture(f"transformer_{tag}")
    c = fx.cfg
    orc = TransformerOracle(fx.weights(), c["n_in"], c["n_ctx"], c["n_head"], c["n_depth"], c["attn_order"],
                            c["blocks"], c["encoder_dims"], c["prime_len"])
    enc = fx["encoder_kv"] if "encoder_kv" in fx else None
    y = orc.forward_full(fx["x"], enc, False)
    assert rel_err(y, fx["yfull32"]) < 2e-5


@pytest.mark.parametrize("tag", ["xy", "plain", "encdec_merged"])
@pytest.mark.parametrize("fp16", [False, True])
def test_ca2d_logits_match_reference(tag, fp16):
    fx = Fixture(f"ca2d_{tag}")
    c = fx.cfg
    orc = PriorOracle(fx.weights(), c["input_dims"], c["bins"], c["width"], c["depth"], c["heads"],
                      c["attn_order"], c["blocks"], c["x_cond"], c["y_cond"], c["encoder_dims"],
                      c["merged_decoder"], c["prime_len"])
    get = lambda k: fx[k] if k in fx else None
    out = orc.logits(fx["tokens"], get("x_cond"), get("y_cond"), get("encoder_kv"), fp16)
    ref = fx["preds16" if fp16 else "preds32"]
    assert rel_err(out, ref) < (2e-3 if fp16 else 2e-5), rel_err(out, ref)
    if not fp16:   # the reference's own chunked prefill agrees with its token-by-token path
        assert rel_err(fx["preds32_primed"], fx["preds32"]) < 2e-5


@pytest.mark.parametrize("tag", ["small", "3level"])
def test_vqvae_matches_reference(tag):
    fx = Fixture(f"vqvae_{tag}")
    c = fx.cfg
    orc = VQVAEOracle(fx.weights(), c["levels"], c["downs_t"], c["strides_t"], c["width"], c["depth"],
                      c["growth"], c["cycle"], c["multipliers"], c["reverse"], c["emb_width"])
    lat = orc.encode_latents(fx["x"])
    zs = orc.encode(fx["x"])
    for l in range(c["levels"]):
        assert rel_err(lat[l], fx[f"lat{l}"]) < 1e-4
        assert zs[l].dtype == np.int64 and zs[l].shape == fx[f"z{l}"].shape
        mism = int((zs[l] != fx[f"z{l}"]).sum())
        assert mism == 0, f"level {l}: {mism} index mismatches"
        xd = orc.decode([fx[f"z{l}"]], start_level=l)
        assert xd.shape == fx[f"xd{l}"].shape
        assert rel_err(xd, fx[f"xd{l}"]) < 1e-4


def test_philox_known_answers():
    """Random123 kat_vectors for philox4x32-10 pin the generator behind jk_sample_categorical"""
    from oracle.sampling_np import philox4x32_10
    kat = [([0, 0, 0, 0], [0, 0], [0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8]),
           ([0xffffffff] * 4, [0xffffffff] * 2, [0x408f276d, 0x41c83b0e, 0xa20bc7c6, 0x6d5451fd]),
           ([0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344], [0xa4093822, 0x299f31d0],
            [0xd16cfe09, 0x94fdcceb, 0x5001e420, 0x24126ea1])]
    for ctr, key, out in kat:
        assert philox4x32_10(ctr, key) == out


@pytest.mark.parametrize("tag", TR_CASES)
def test_torch_restatement_is_the_reference_on_the_same_device(tag):
    """oracle/transformer_torch.py (used on the GPU box to measure fp16 order noise) replays the reference's own
    torch operators, so in fp32 it must reproduce the reference's CPU outputs to 2e-6 on any host.  In fp16 the result
    depends on the host's half-precision GEMM blocking: on the host that wrote the fixtures it is bit-identical up to
    5e-4, on another CPU model (this container has been re-created on different hosts) it shows the same 1.4e-3 ...
    2.2e-3 order noise that tests/test_gpu_fullsize_golden.py measures on the GPU - hence the 3e-3 bound here."""
    import torch
    from oracle.transformer_torch import TorchDecodeOracle
    fx = Fixture(f"transformer_{tag}")
    c = fx.cfg
    orc = TorchDecodeOracle(fx.weights(), c["n_in"], c["n_ctx"], c["n_head"], c["n_depth"], c["attn_order"], c["blocks"],
                            c["encoder_dims"], c["prime_len"])
    x = torch.from_numpy(fx["x"])
    enc = torch.from_numpy(fx["encoder_kv"]) if "encoder_kv" in fx else None
    for fp16, key, tol in ((True, "y16", 3e-3), (False, "y32", 2e-6)):
        orc.reset()
        with torch.no_grad():
            y = torch.stack([orc.step(x[:, i], enc, fp16) for i in range(c["n_ctx"])], 1).numpy()
        assert rel_err(y, fx[key]) < tol, (key, rel_err(y, fx[key]))
