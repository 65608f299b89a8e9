"""Prior fine-tuning without a GPU: the golden gradients, the new struct's ctypes mirror, the refusals of loss_grad
(before any launch, .grad untouched) and the gradient kernels' register use."""
import ctypes as C
import json
import math
import os
import re
import shutil
import subprocess
import tempfile

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from golden_util import Fixture

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# ---- a float64 autograd restatement of the decoder matches the reference's float64 gradients ---------------------------
def _ca2d_loss64(m, seq, x_cond, y_cond, enc, w):
    """sum_m w_m CE_m of a ConditionalAutoregressive2D window in float64 autograd: the fp32 path's operators (shifted
    embedding, LayerNorm, Conv1D, the pattern's key sets, quick_gelu, x_out)"""
    from jukebox_b200.transformer.f32 import layer_params
    N, D = seq.shape
    Wd = m.width
    P = {id(p): p.double().detach().requires_grad_(True) for p in m.parameters()}
    q = lambda p: P[id(p)]
    h = q(m.x_emb.weight)[seq]
    h = torch.roll(h, 1, dims=1)
    first = y_cond.double().view(N, 1, Wd) if m.y_cond else q(m.start_token).view(1, 1, Wd).expand(N, 1, Wd)
    h = torch.cat([first, h[:, 1:]], dim=1) + q(m.pos_emb.pos_emb)
    if x_cond is not None:
        h = h + x_cond.double()
    tr = m.transformer
    bc = tr.n_ctx // tr.blocks if tr.blocks else tr.n_ctx
    prime = (tr.prime_len // tr.blocks + 1) * tr.blocks if tr.prime_len else 0
    pos = torch.arange(D)[:, None]
    for blk in tr._attn_mods:
        p = {k: q(v) for k, v in layer_params(blk)}
        af = blk.attn_func
        Lk = tr.encoder_dims if af == 6 else D
        k_ = torch.arange(Lk)[None, :]
        mask = {0: k_ <= pos, 1: (k_ // bc == pos // bc) & (k_ <= pos), 2: (k_ % bc == pos % bc) & (k_ <= pos),
                3: k_ // bc == pos // bc - 1, 6: torch.ones(D, Lk, dtype=torch.bool),
                7: (k_ < prime) & (k_ <= pos)}[af]
        xn0 = F.layer_norm(h, (Wd,), p["ln0_g"], p["ln0_b"], 1e-5)
        if af == 6:
            qq = xn0 @ p["c_attn_w"] + p["c_attn_b"]
            kk, vv = (enc.double() @ p["c_enc_kv_w"] + p["c_enc_kv_b"]).chunk(2, dim=-1)
        else:
            qq, kk, vv = (xn0 @ p["c_attn_w"] + p["c_attn_b"]).chunk(3, dim=-1)
        H = tr.n_head
        dh = qq.shape[-1] // H
        hd = lambda t_: t_.reshape(N, -1, H, dh).transpose(1, 2)
        s = (hd(qq) @ hd(kk).transpose(-1, -2) / math.sqrt(dh)).masked_fill(~mask, float("-inf"))
        pr = torch.where(mask.any(-1, keepdim=True), torch.softmax(s, -1), torch.zeros_like(s))
        a = (pr @ hd(vv)).transpose(1, 2).reshape(N, D, -1)
        x1 = h + a @ p["c_proj_w"] + p["c_proj_b"]
        g = F.layer_norm(x1, (Wd,), p["ln1_g"], p["ln1_b"], 1e-5) @ p["fc_w"] + p["fc_b"]
        h = x1 + (g * torch.sigmoid(1.702 * g)) @ p["proj2_w"] + p["proj2_b"]
    if m.add_cond_after_transformer and x_cond is not None:
        h = h + x_cond.double()
    logits = h @ q(m.x_out.weight).t()
    ce = F.cross_entropy(logits.reshape(N * D, -1), seq.reshape(-1), reduction="none")
    (ce * w.double().reshape(-1)).sum().backward()
    names = {id(p): n for n, p in m.named_parameters()}
    return {names[k]: v.grad for k, v in P.items()}


@pytest.mark.parametrize("tag", ["single_enc_dec", "sep_enc_dec", "upsampler", "plain"])
def test_float64_restatement_matches_the_reference_float64(tag):
    from jukebox_b200.hparams import setup_hparams
    from jukebox_b200.make_models import make_vqvae, make_prior
    fx = Fixture(f"grad_{tag}")
    c = fx.cfg
    sd = {k: torch.from_numpy(v) for k, v in fx.weights().items()}
    if c["kind"] == "ca2d":
        from jukebox_b200.prior.autoregressive import ConditionalAutoregressive2D
        m = ConditionalAutoregressive2D((c["input_dims"],), c["bins"], width=c["width"], depth=c["depth"],
                                        heads=c["heads"], attn_order=c["attn_order"], blocks=c["blocks"])
        m.load_state_dict(sd)
        total, prior = c["input_dims"], None
    else:
        vq = make_vqvae(setup_hparams(c["vq_name"], dict(restore_vqvae="", **c["vq_over"])), "cpu")
        prior = make_prior(setup_hparams(c["pr_name"], dict(restore_prior="", **c["pr_over"])), vq, "cpu")
        prior.load_state_dict(sd)
        m, total = prior.prior, prior.total_loss_dims
    seq = torch.from_numpy(fx["seq"])
    N, D = seq.shape
    get = lambda k: torch.from_numpy(fx[k]) if k in fx else None
    unit = 1.0 / (N * total * math.log(2.0))
    w = torch.full((N, D), unit, dtype=torch.float64)
    if prior is not None and prior.single_enc_dec:
        w[:, :c["prime_len"]] = prior.prime_loss_fraction * unit
    g = _ca2d_loss64(m, seq, get("x_cond"), get("y_cond"), get("encoder_kv"), w)
    worst = 0.0
    for n in c["params"]:
        ours = g[n].reshape(-1)[torch.from_numpy(fx[f"idx:{n}"].astype(np.int64))].numpy()
        g64 = fx[f"g64:{n}"]
        e = float(np.abs(ours - g64).max() / max(np.abs(g64).max(), 1e-300))
        worst = max(worst, e)
        assert e <= 1e-9, (n, e)
    print(json.dumps(dict(tag=tag, worst_rel=worst)))


# ---- the ctypes mirror of jk_f32_grad_layer --------------------------------------------------------------------------
@pytest.mark.skipif(shutil.which("gcc") is None, reason="needs gcc")
def test_grad_layer_mirror_matches_the_header():
    from jukebox_b200 import _lib
    header = open(os.path.join(ROOT, "include", "jkb200.h")).read()
    body = re.search(r"typedef struct jk_f32_grad_layer \{(.*?)\} jk_f32_grad_layer;", header, re.S).group(1)
    fields = [f.strip().lstrip("*") for f in re.sub(r"float|\*|;", " ", body).replace(",", " ").split()]
    lines = ['#include <stdio.h>', '#include <stddef.h>', '#include "jkb200.h"', "int main(void) {",
             'printf("size %zu\\n", sizeof(jk_f32_grad_layer));']
    lines += ['printf("%s %%zu\\n", offsetof(jk_f32_grad_layer, %s));' % (f, f) for f in fields]
    lines += ["return 0;", "}"]
    with tempfile.TemporaryDirectory() as d:
        src, exe = os.path.join(d, "abi.c"), os.path.join(d, "abi")
        open(src, "w").write("\n".join(lines))
        subprocess.run(["gcc", "-std=c99", "-I", os.path.join(ROOT, "include"), src, "-o", exe], check=True)
        out = dict(l.split() for l in subprocess.run([exe], capture_output=True, text=True, check=True).stdout.splitlines())
    cls = _lib.F32GradLayer
    assert C.sizeof(cls) == int(out["size"])
    assert [f[0] for f in cls._fields_] == fields
    for f in fields:
        assert getattr(cls, f).offset == int(out[f]), f
    # the gradient struct mirrors the parameter fields of jk_f32_layer, in the same order
    assert fields == [f[0] for f in _lib.F32Layer._fields_][:len(fields)]


# ---- refusals: before any launch, .grad untouched ------------------------------------------------------------------
def _tiny(**kw):
    from jukebox_b200.prior.autoregressive import ConditionalAutoregressive2D
    args = dict(width=32, depth=2, heads=2, attn_order=2, blocks=4)
    args.update(kw)
    return ConditionalAutoregressive2D((16,), 20, **args)


def _refused(m, x, match):
    before = {n: (None if p.grad is None else p.grad.clone()) for n, p in m.named_parameters()}
    with pytest.raises(ValueError, match=match):
        m.loss_grad(x)
    for n, p in m.named_parameters():
        assert (p.grad is None) == (before[n] is None) and (p.grad is None or torch.equal(p.grad, before[n])), n


def test_refusals_leave_grad_untouched(monkeypatch):
    from jukebox_b200 import _lib
    monkeypatch.setattr(_lib, "lib", lambda: pytest.fail("a refused call reached the library"))
    x = torch.randint(0, 20, (2, 16))
    m = _tiny().requires_grad_(False)
    _refused(m, x, "no parameter")
    m.transformer._attn_mods[1].requires_grad_(True)
    m.transformer._attn_mods[1].ln_0.weight.grad = torch.ones_like(m.transformer._attn_mods[1].ln_0.weight)
    _refused(m, x, "CUDA device")
    _refused(m, x[:, :10], "whole windows")
    h = _tiny()
    h.transformer._attn_mods[0].mlp.c_fc.w.data = h.transformer._attn_mods[0].mlp.c_fc.w.data.half()
    h.requires_grad_(True)
    _refused(h, x, "fp16_params")
    r = _tiny(res_scale=True)
    r.requires_grad_(True)
    _refused(r, x, "res_scale")
    a = _tiny(attn_order=3)          # attn_func 4 (layers 1, 3)
    a.requires_grad_(True)
    _refused(a, x, "attn_func")


# ---- the gradient kernels keep their values in registers ----------------------------------------------------------
@pytest.mark.skipif(shutil.which("nvcc") is None and not os.path.exists("/usr/local/cuda/bin/nvcc"), reason="needs nvcc")
def test_gradient_kernels_do_not_spill():
    from jukebox_b200.build import NVCC_FLAGS, _nvcc
    flags = [f for f in NVCC_FLAGS if f not in ("--shared",)]
    with tempfile.TemporaryDirectory() as d:
        res = subprocess.run([_nvcc()] + flags + ["-Xptxas", "-v", "-c",
                              os.path.join(ROOT, "jukebox_b200", "csrc", "f32_grad.cu"), "-o", os.path.join(d, "g.o")],
                             capture_output=True, text=True, timeout=600)
    assert res.returncode == 0, res.stderr[-2000:]
    kernels = re.findall(r"Compiling entry function '(\w+)'", res.stderr)
    spills = re.findall(r"(\d+) bytes spill stores, (\d+) bytes spill loads", res.stderr)
    assert len(kernels) >= 12 and len(spills) == len(kernels), res.stderr
    for k, (st, ld) in zip(kernels, spills):
        assert st == "0" and ld == "0", f"{k} spills {st} / {ld} bytes"
