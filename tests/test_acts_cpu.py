"""Layer representations without a GPU: the C ABI of the capture (jk_act_capture, jk_prefill_args.n_layers, jk_pool_rows_f32),
the numpy oracle's per-layer outputs (oracle/acts_np.py) against the reference's JukeMIR recipe (tests/golden/acts_*.npz, oracle/
make_golden_acts.py), and the host control flow of ConditionalAutoregressive2D.layer_acts / audio_representations with
the engine replaced by a fake."""
import ctypes
import os
import re
import shutil
import subprocess
import tempfile

import numpy as np
import pytest
import torch

from golden_util import Fixture, rel_err
from oracle.acts_np import layer_outputs
from oracle.transformer_np import TransformerOracle

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TAGS = ["labelled", "single_enc_dec", "sep_enc_dec"]


# ---- C ABI ---------------------------------------------------------------------------------------------------------
@pytest.mark.skipif(shutil.which("gcc") is None, reason="needs gcc")
def test_capture_struct_matches_its_ctypes_mirror():
    from jukebox_b200 import _lib
    header = open(os.path.join(ROOT, "include", "jkb200.h")).read()
    body = re.search(r"typedef struct jk_act_capture \{(.*?)\} jk_act_capture;", header, re.S).group(1)
    fields = [re.search(r"(\w+)\s*$", p.strip()).group(1) for d in body.split(";") if d.strip() for p in d.split(",")]
    lines = ['#include <stdio.h>', '#include <stddef.h>', '#include "jkb200.h"', "int main(void) {",
             'printf("size %zu\\n", sizeof(jk_act_capture));']
    lines += ['printf("%s %%zu\\n", offsetof(jk_act_capture, %s));' % (f, f) for f in fields]
    lines += ["return 0;", "}"]
    with tempfile.TemporaryDirectory() as d:
        src, exe = os.path.join(d, "abi.c"), os.path.join(d, "abi")
        open(src, "w").write("\n".join(lines))
        subprocess.run(["gcc", "-std=c99", "-I", os.path.join(ROOT, "include"), src, "-o", exe], check=True)
        out = dict(l.split() for l in subprocess.run([exe], capture_output=True, text=True, check=True).stdout.splitlines())
    cls = _lib.ActCapture
    assert ctypes.sizeof(cls) == int(out["size"])
    assert [f[0] for f in cls._fields_] == fields
    for f in fields:
        assert getattr(cls, f).offset == int(out[f]), f
    # the prefill arguments carry the table after the fields they had (zero-initialised = as before)
    names = [f[0] for f in _lib.PrefillArgs._fields_]
    assert names[-3:] == ["n_layers", "capture", "n_capture"]
    assert _lib.PrefillArgs().n_layers == 0 and _lib.PrefillArgs().n_capture == 0


def test_pool_symbol_is_declared_exported_and_bound():
    from jukebox_b200 import _lib
    header = open(os.path.join(ROOT, "include", "jkb200.h")).read()
    m = re.search(r"\bjk_pool_rows_f32\s*\(([^)]*)\)", header)
    assert m and len(m.group(1).split(",")) == 10
    res, args = _lib.SIGNATURES["jk_pool_rows_f32"]
    assert res is ctypes.c_int and len(args) == 10
    assert hasattr(ctypes.CDLL(_lib.LIB_PATH), "jk_pool_rows_f32")
    lib = _lib.lib()
    # argument checks run before any device work
    assert lib.jk_pool_rows_f32(None, 1, 4, 8, 0, 4, None, 0, None, None) != 0
    assert b"null argument" in lib.jk_last_error()


# ---- the oracle's captured layers against the reference ----------------------------------------------------------------
def _oracle_acts(fx, fp16):
    """embedding (autoregressive.py:139-147) -> the oracle's forward mode cut after each layer -> + x_cond"""
    c = fx.cfg
    sd = fx.weights("prior.")
    tsd = {k[len("transformer."):]: v for k, v in sd.items() if k.startswith("transformer.")}
    assert TransformerOracle(tsd, c["width"], c["input_dims"], c["heads"], len(c["attn_funcs"]), c["attn_order"],
                             c["blocks"]).attn_funcs == c["attn_funcs"]
    tokens = fx["tokens"]
    N, D = tokens.shape
    x = np.zeros((N, D, c["width"]), np.float32)
    x[:, 1:] = sd["x_emb.weight"][tokens[:, :-1]]
    x[:, 0] = fx["y_cond"].reshape(N, -1) if "y_cond" in fx else sd["start_token"].reshape(-1)
    xc = fx["x_cond"] if "x_cond" in fx else np.zeros((N, 1, c["width"]), np.float32)
    x = x + sd["pos_emb.pos_emb"] + xc
    enc = fx["enc16" if fp16 else "enc32"] if "enc32" in fx else None
    cap = layer_outputs(tsd, c["width"], c["input_dims"], c["heads"], c["attn_order"], c["blocks"], c["encoder_dims"],
                        c["prime_len"], c["layers"], x, enc, fp16)
    return {l: (h + xc if c["add_cond_after"] else h)[:, c["start"]:] for l, h in cap.items()}


@pytest.mark.parametrize("tag", TAGS)
@pytest.mark.parametrize("fp16", [False, True])
def test_oracle_layer_capture_matches_the_reference(tag, fp16):
    fx = Fixture(f"acts_{tag}")
    acts = _oracle_acts(fx, fp16)
    for l, a in acts.items():
        ref = fx[f"a{16 if fp16 else 32}_{l}"]
        assert a.shape == ref.shape
        e = rel_err(a, ref)
        # the bounds of test_oracle_golden.py: fp32 summation-order noise (2e-5); fp16 that of the fp16 restatement of a
        # whole pass (3e-3) - the reference's CPU half products and the oracle's round the same fp32 accumulations and
        # differ by boundary flips that 9 .. 16 layers carry forward (measured 1.3e-3 .. 2.7e-3, as far apart as the
        # reference's own fp16 and fp32 passes)
        assert e < (3e-3 if fp16 else 2e-5), (tag, l, e)
        assert rel_err(a.mean(1), ref.mean(1)) < (3e-3 if fp16 else 2e-5)


def test_oracle_layer_outputs_by_step_equal_forward_mode():
    fx = Fixture("acts_labelled")
    c = fx.cfg
    sd = {k[len("prior.transformer."):]: v for k, v in fx.weights().items() if k.startswith("prior.transformer.")}
    x = np.random.RandomState(0).standard_normal((2, c["input_dims"], c["width"])).astype(np.float32) * 0.3
    args = (sd, c["width"], c["input_dims"], c["heads"], c["attn_order"], c["blocks"], 0, None, c["layers"], x)
    full, step = layer_outputs(*args), layer_outputs(*args, mode="step")
    for l in c["layers"]:
        assert rel_err(step[l], full[l]) < 2e-5


# ---- host control flow ----------------------------------------------------------------------------------------------
class FakeEngine:
    """stands in for DecodeEngine: a capture of layer l receives (the item's first token) * 1000 + l + the mean position"""

    def __init__(self, depth):
        self.prefill_capacity = 64
        self.calls = []
        self.position = 0
        self.depth = depth

    def reset(self, t0=0):
        self.position = t0

    def prefill(self, n, P, tokens=None, n_layers=0, capture=None, **kw):
        self.calls.append((n, P, n_layers, sorted(capture)))
        for l, k in capture.items():
            first = tokens[:, 0].float()                         # identifies the items of this batch
            v = first[:, None] * 1000 + l + (k.t0 + k.t1 - 1) / 2
            if k.pool:
                k.out.copy_(v.expand(n, k.out.shape[1]))
            else:
                k.out.copy_(v[:, :, None].expand(k.out.shape))
        self.position = -1 if 0 < n_layers < self.depth else P


def _ca2d(monkeypatch, per_batch):
    from jukebox_b200.prior import autoregressive as ar
    m = ar.ConditionalAutoregressive2D((24,), 16, width=64, depth=6, heads=1, attn_order=0, blocks=None).eval()
    eng = FakeEngine(6)
    monkeypatch.setattr(m, "_engine", lambda n: eng)
    monkeypatch.setattr(m, "items_per_prefill", lambda N: min(N, per_batch))
    monkeypatch.setattr(m.transformer, "prefill_capacity", lambda n: eng.prefill_capacity)
    return m, eng


def test_layer_acts_batches_items_and_truncates_after_the_deepest_layer(monkeypatch):
    m, eng = _ca2d(monkeypatch, per_batch=2)
    x = torch.arange(5)[:, None].repeat(1, 20) % 16                 # item i: tokens all i
    out = m.layer_acts(x, layers=(4, 1), fp16=True, pool=True, t0=3)
    assert eng.calls == [(2, 20, 5, [1, 4]), (2, 20, 5, [1, 4]), (1, 20, 5, [1, 4])]
    assert sorted(out) == [1, 4]
    for l in (1, 4):
        assert out[l].shape == (5, 64) and out[l].dtype == torch.float32
        want = torch.arange(5).float() * 1000 + l + (3 + 20 - 1) / 2
        assert torch.equal(out[l][:, 0], want)
    rows = m.layer_acts(x, layers=(2,), fp16=True, pool=False, t0=5)[2]
    assert rows.shape == (5, 15, 64)


def test_layer_acts_beyond_the_prefill_capacity_is_an_error(monkeypatch):
    m, eng = _ca2d(monkeypatch, per_batch=4)
    eng.prefill_capacity = 16
    with pytest.raises(RuntimeError, match="prefill capacity 16"):
        m.layer_acts(torch.zeros(2, 20, dtype=torch.long), layers=(1,), fp16=True)
    assert eng.calls == []
    with pytest.raises(AssertionError):
        m.layer_acts(torch.zeros(2, 20, dtype=torch.long), layers=(6,), fp16=True)     # depth 6: layers 0..5


def test_windows_cut_the_codes_into_consecutive_contexts():
    from jukebox_b200.represent import windows
    assert windows(8192, 8192) == [(0, 8192)]
    assert windows(20000, 8192) == [(0, 8192), (8192, 16384), (16384, 20000)]
    assert windows(8193, 8192) == [(0, 8192)]              # a one-code tail has nothing to attend and is dropped
    assert windows(100, 8192) == [(0, 100)]


class FakePrior:
    """a top-level SimplePrior stand-in: encode gives codes 0..T-1 per item; layer_acts gives the window's mean code"""

    def __init__(self, n_ctx, T, labelled):
        self.level, self.n_ctx, self.x_cond, self.y_cond = 1, n_ctx, False, labelled
        self.sample_length = 4096
        self.T = T
        self.calls = []
        self.prior = type("P", (), {"width": 3})()
        from jukebox_b200.data.labels import Labeller
        self.labeller = Labeller(1, 0, self.sample_length, v3=True)

    def encode(self, x, start_level=None, end_level=None, bs_chunks=1):
        assert (start_level, end_level) == (1, 2)
        return [torch.arange(self.T).repeat(x.shape[0], 1) + torch.arange(x.shape[0])[:, None] * 10000]

    def layer_acts(self, z, z_conds=[], y=None, layers=(), fp16=True, pool=True):
        self.calls.append((z.shape[1], None if y is None else y.tolist(), tuple(layers), fp16, pool))
        v = z.double().mean(1, keepdim=True).float()
        return {l: v.expand(z.shape[0], 3) + l for l in layers}


@pytest.mark.parametrize("T", [50, 64, 100, 129])
def test_audio_representations_weight_the_windows_by_length(T):
    from jukebox_b200.represent import audio_representations
    p = FakePrior(32, T, labelled=False)
    feats = audio_representations(p, torch.zeros(2, 7, 1), layers=(0, 5), fp16=False)
    lens = [c[0] for c in p.calls]
    assert sum(lens) == (T if T % 32 != 1 else T - 1) and all(n == 32 for n in lens[:-1])
    assert all(c[1] is None and c[2] == (0, 5) and c[3] is False and c[4] is True for c in p.calls)
    n = sum(lens)
    for l in (0, 5):
        want = (torch.arange(2).double() * 10000 + (n - 1) / 2 + l).float()        # mean over all positions
        assert feats[l].shape == (2, 3)
        assert torch.allclose(feats[l][:, 0], want, rtol=1e-6)


def test_audio_representations_build_jukemirs_label_row_or_take_the_given_one():
    from jukebox_b200.represent import audio_representations
    p = FakePrior(32, 40, labelled=True)
    audio_representations(p, torch.zeros(2, 7, 1), layers=(1,))
    y0 = p.calls[0][1]
    assert len(y0) == 2 and y0[0] == y0[1]
    assert y0[0][:4] == [p.sample_length, 0, p.sample_length, 0] and y0[0][4] == 0    # total, offset 0, unknown artist, genre
    p.calls.clear()
    y = torch.tensor([[1, 2, 3, 4, 5], [6, 7, 8, 9, 10]])
    audio_representations(p, torch.zeros(2, 7, 1), y=y, layers=(1,))
    assert all(c[1] == y.tolist() for c in p.calls)
