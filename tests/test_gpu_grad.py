"""Gradients of a prior's window loss on the fp32 path's backward kernels (csrc/f32_grad.cu, loss_grad).

(a) tiny fixtures (tests/golden/grad_*.npz, oracle/make_golden_grad.py): every decoder parameter's gradient against the
    reference's float64 gradient.  The yardstick is the reference's own float32 distance to float64 (order noise):
    max|ours - g64| <= ORDER * max|g32 - g64| + FLOOR * max|g64| per parameter.
(b) one layer per pattern at the priors' real geometry against float64 autograd on the GPU (see REAL_TOL).
(c) determinism: two calls are bit-identical, a second call doubles .grad exactly.
(d) frozen lower layers keep .grad None and leave the trainable gradients bit-identical.
(e) the loss equals z_forward(fp16=False)'s.
(f) Adam steps lower the window's loss, and fp16 sampling afterwards draws from the updated weights."""
import ctypes as C
import json
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from golden_util import Fixture
from jukebox_b200 import _lib
from oracle.synth import synth_tensor

pytestmark = pytest.mark.gpu

ORDER = 4.0         # our distance to float64, in units of the reference's float32 distance
FLOOR = 2e-7        # ~ 3 u of the gradient's scale, for parameters whose float32 distance happens to be ~0
TAGS = ["single_enc_dec", "sep_enc_dec", "upsampler", "plain"]


def record(row):
    print(json.dumps(row))


def _prior(tag):
    from jukebox_b200.hparams import setup_hparams
    from jukebox_b200.make_models import make_vqvae, make_prior
    fx = Fixture(f"grad_{tag}")
    c = fx.cfg
    if c["kind"] == "ca2d":
        from jukebox_b200.prior.autoregressive import ConditionalAutoregressive2D
        m = ConditionalAutoregressive2D((c["input_dims"],), c["bins"], width=c["width"], depth=c["depth"],
                                        heads=c["heads"], attn_order=c["attn_order"], blocks=c["blocks"])
        m.load_state_dict({k: torch.from_numpy(v) for k, v in fx.weights().items()}, strict=True)
        return fx, None, m.cuda().eval()
    vq = make_vqvae(setup_hparams(c["vq_name"], dict(restore_vqvae="", **c["vq_over"])), "cpu")
    prior = make_prior(setup_hparams(c["pr_name"], dict(restore_prior="", **c["pr_over"])), vq, "cpu")
    prior.load_state_dict({k: torch.from_numpy(v) for k, v in fx.weights().items()}, strict=True)
    prior = prior.cuda().eval()
    return fx, prior, prior.prior


def _decoder_call(fx, prior, m):
    """the fixture's constant conditioning and the per-row weights of z_forward's loss"""
    seq = torch.from_numpy(fx["seq"]).cuda()
    N, D = seq.shape
    kw = {k: (torch.from_numpy(fx[k]).cuda() if k in fx else None) for k in ("x_cond", "y_cond", "encoder_kv")}
    total = D if prior is None else prior.total_loss_dims
    unit = 1.0 / (N * total * math.log(2.0))
    w = torch.full((N, D), unit, device="cuda")
    if prior is not None and prior.single_enc_dec:
        w[:, :fx.cfg["prime_len"]] = prior.prime_loss_fraction * unit
    return seq, kw, w


def _grads(m):
    return {n: p.grad.detach().clone() for n, p in m.named_parameters() if p.grad is not None}


@pytest.mark.parametrize("tag", TAGS)
def test_gradients_against_reference_float64(tag):
    fx, prior, m = _prior(tag)
    m.requires_grad_(True)
    seq, kw, w = _decoder_call(fx, prior, m)
    ce = m.loss_grad(seq, row_weights=w, **kw)
    loss = float((ce.double() * w.double()).sum())
    assert abs(loss - fx.cfg["loss64"]) <= 1e-5 * abs(fx.cfg["loss64"]), (loss, fx.cfg["loss64"])
    got = _grads(m)
    assert sorted(got) == sorted(fx.cfg["params"])
    worst = 0.0
    for n in fx.cfg["params"]:
        idx = torch.from_numpy(fx[f"idx:{n}"].astype(np.int64)).cuda()
        ours = got[n].reshape(-1)[idx].double().cpu().numpy()
        g64, g32 = fx[f"g64:{n}"], fx[f"g32:{n}"].astype(np.float64)
        scale = max(float(np.abs(g64).max()), 1e-30)
        d_ours, d_ref = float(np.abs(ours - g64).max()), float(np.abs(g32 - g64).max())
        ratio = d_ours / (ORDER * d_ref + FLOOR * scale)
        worst = max(worst, ratio)
        assert ratio <= 1.0, f"{tag} {n}: ours {d_ours:.3e}, reference fp32 {d_ref:.3e}, scale {scale:.3e}"
    record(dict(test="fixture", tag=tag, loss=loss, loss64=fx.cfg["loss64"], worst_over_bound=worst))


@pytest.mark.parametrize("tag", ["upsampler", "sep_enc_dec"])
def test_two_calls_bit_identical_and_accumulate(tag):
    fx, prior, m = _prior(tag)
    m.requires_grad_(True)
    seq, kw, w = _decoder_call(fx, prior, m)
    m.loss_grad(seq, row_weights=w, **kw)
    a = _grads(m)
    m.zero_grad(set_to_none=True)
    m.loss_grad(seq, row_weights=w, **kw)
    b = _grads(m)
    m.loss_grad(seq, row_weights=w, **kw)
    c = _grads(m)
    for n in a:
        assert torch.equal(a[n], b[n]), n
        assert torch.equal(c[n], 2 * a[n]), n


def test_frozen_lower_layers():
    fx, prior, m = _prior("single_enc_dec")
    m.requires_grad_(True)
    seq, kw, w = _decoder_call(fx, prior, m)
    m.loss_grad(seq, row_weights=w, **kw)
    full = _grads(m)
    m.zero_grad(set_to_none=True)
    m.requires_grad_(False)
    top = m.depth // 2
    for blk in m.transformer._attn_mods[top:]:
        blk.requires_grad_(True)
    m.loss_grad(seq, row_weights=w, **kw)
    part = _grads(m)
    for n, p in m.named_parameters():
        if p.requires_grad:
            assert torch.equal(part[n], full[n]), n
        else:
            assert p.grad is None, n
    assert len(part) == 12 * (m.depth - top)


@pytest.mark.parametrize("tag", ["single_enc_dec", "sep_enc_dec", "upsampler"])
def test_loss_matches_z_forward(tag):
    pf = Fixture(f"prior_{tag}")
    _, prior, m = _prior(tag)
    y = torch.from_numpy(pf["y"]).cuda() if "y" in pf else None
    z_conds = [torch.from_numpy(pf["z_cond"]).cuda()] if "z_cond" in pf else []
    tokens = torch.from_numpy(pf["tokens"]).cuda()
    z = prior.prior_postprocess(tokens) if prior.single_enc_dec else tokens
    want, mw = prior.z_forward(z, z_conds, y, fp16=False)
    m.requires_grad_(True)
    got, mg = prior.loss_grad(z, z_conds, y)
    for k in ("gen_loss", "prime_loss"):
        assert abs(float(mg[k]) - float(mw[k])) <= 1e-6 * max(abs(float(mw[k])), 1e-30), (k, float(mg[k]), float(mw[k]))
    assert abs(float(got) - float(want)) <= 1e-6 * abs(float(want)), (float(got), float(want))


def test_adam_lowers_the_loss_and_sampling_follows():
    pf = Fixture("prior_upsampler")
    _, prior, m = _prior("upsampler")
    z_conds = [torch.from_numpy(pf["z_cond"]).cuda()]
    z = torch.from_numpy(pf["tokens"]).cuda()
    torch.manual_seed(3)
    prior.sample(2, z_conds=z_conds, fp16=True, sample_tokens=8)     # packs the engine before the updates
    m.requires_grad_(True)
    opt = torch.optim.Adam([p for p in m.parameters() if p.requires_grad], lr=1e-3, betas=(0.9, 0.95))
    losses = []
    for _ in range(20):
        loss, _ = prior.loss_grad(z, z_conds)
        losses.append(float(loss))
        opt.step()
        opt.zero_grad(set_to_none=True)
    final, _ = prior.z_forward(z, z_conds, fp16=False)
    record(dict(test="adam", first=losses[0], last=losses[-1], after=float(final)))
    assert float(final) < 0.8 * losses[0], losses
    torch.manual_seed(11)
    a = prior.sample(2, z_conds=z_conds, fp16=True, sample_tokens=24)
    _, fresh, _ = _prior("upsampler")
    fresh.load_state_dict(prior.state_dict())
    torch.manual_seed(11)
    b = fresh.sample(2, z_conds=z_conds, fp16=True, sample_tokens=24)
    assert torch.equal(a, b)


# ---- (b) one layer at the priors' real geometry against float64 autograd ----------------------------------------------
# REAL_TOL: max|ours - g64| / max|g64| per gradient tensor.  Every gradient here is a chain of fp32 dot products of at
# most K = 8 576 terms (weight gradients sum over the window's rows, attention over its keys or queries); a sequential
# fma chain of K terms carries a relative error of about u sqrt(K) (u = 2^-24, independent rounding signs), and a layer's
# backward chains about ten such products: 10 u sqrt(8 576) = 5.5e-5.
REAL_TOL = 10 * 2.0 ** -24 * math.sqrt(8576)
GEOM = {"1b": (2048, 2, 8576, 64, 384, 0), "5b": (4800, 8, 8192, 128, None, 512), "up": (1920, 1, 8192, 128, None, 0)}
CASES = [(0, "1b"), (1, "1b"), (2, "up"), (3, "5b"), (6, "5b"), (7, "1b")]
NAMES = [("ln0_g", "ln_0.weight"), ("ln0_b", "ln_0.bias"), ("ln1_g", "ln_1.weight"), ("ln1_b", "ln_1.bias"),
         ("c_attn_w", "attn.c_attn.w"), ("c_attn_b", "attn.c_attn.b"), ("c_proj_w", "attn.c_proj.w"),
         ("c_proj_b", "attn.c_proj.b"), ("fc_w", "mlp.c_fc.w"), ("fc_b", "mlp.c_fc.b"), ("proj2_w", "mlp.c_proj.w"),
         ("proj2_b", "mlp.c_proj.b"), ("c_enc_kv_w", "attn.c_enc_kv.w"), ("c_enc_kv_b", "attn.c_enc_kv.b")]


def _mask(af, P, Lk, bc, prime, shift):
    """[P, Lk] bool: the keys of each query (f32_path.cu's key sets), shifted by `shift` rows"""
    p = torch.arange(P, device="cuda")[:, None]
    k = torch.arange(Lk, device="cuda")[None, :]
    if af == 0:
        m = k <= p
    elif af == 1:
        m = (k // bc == p // bc) & (k <= p)
    elif af == 2:
        m = (k % bc == p % bc) & (k <= p)
    elif af == 3:
        m = (k // bc == p // bc - 1)
    elif af == 6:
        m = torch.ones(P, Lk, dtype=torch.bool, device="cuda")
    else:
        m = (k < prime) & (k <= p)
    if shift:
        s = torch.zeros_like(m)
        s[:, shift:] = m[:, :-shift]
        m = s
    return m


def _layer64(p, x, enc, af, H, mask):
    W = x.shape[-1]
    xn0 = F.layer_norm(x, (W,), p["ln_0.weight"], p["ln_0.bias"], 1e-5)
    if af == 6:
        q = xn0 @ p["attn.c_attn.w"] + p["attn.c_attn.b"]
        k, v = (enc @ p["attn.c_enc_kv.w"] + p["attn.c_enc_kv.b"]).chunk(2, dim=-1)
    else:
        q, k, v = (xn0 @ p["attn.c_attn.w"] + p["attn.c_attn.b"]).chunk(3, dim=-1)
    n, P, S = q.shape
    dh = S // H
    heads = lambda t: t.reshape(n, -1, H, dh).transpose(1, 2)
    s = heads(q) @ heads(k).transpose(-1, -2) / math.sqrt(dh)
    s = s.masked_fill(~mask, float("-inf"))
    pr = torch.softmax(s, dim=-1)
    pr = torch.where(mask.any(-1, keepdim=True), pr, torch.zeros_like(pr))      # a query without keys: output 0
    a = (pr @ heads(v)).transpose(1, 2).reshape(n, P, S)
    x1 = x + a @ p["attn.c_proj.w"] + p["attn.c_proj.b"]
    xn1 = F.layer_norm(x1, (W,), p["ln_1.weight"], p["ln_1.bias"], 1e-5)
    g = xn1 @ p["mlp.c_fc.w"] + p["mlp.c_fc.b"]
    g = g * torch.sigmoid(1.702 * g)
    return x1 + g @ p["mlp.c_proj.w"] + p["mlp.c_proj.b"]


def _grads64(p32, x, enc, dy, af, H, mask):
    p = {k: v.double().requires_grad_(True) for k, v in p32.items()}
    x64 = x.double().requires_grad_(True)
    e64 = None if enc is None else enc.double().requires_grad_(True)
    _layer64(p, x64, e64, af, H, mask).backward(dy.double())
    out = {k: v.grad for k, v in p.items()}
    out["dx"] = x64.grad
    if e64 is not None:
        out["d_encoder_kv"] = e64.grad
    return out


@pytest.mark.parametrize("af,g", CASES)
def test_one_layer_backward_at_real_geometry(af, g):
    from jukebox_b200.transformer.f32 import grad_buffer   # noqa: F401  (the package is built)
    W, H, n_ctx, blocks, prime_len, E = GEOM[g]
    E = E if af == 6 else 0
    S, Mw, n, bc = W // 4, W, 1, n_ctx // blocks
    prime = (prime_len // blocks + 1) * blocks if prime_len else 0
    qw = S if af == 6 else 3 * S
    shapes = [("ln_0.weight", (W,)), ("ln_0.bias", (W,)), ("ln_1.weight", (W,)), ("ln_1.bias", (W,)),
              ("attn.c_attn.w", (W, qw)), ("attn.c_attn.b", (qw,)), ("attn.c_proj.w", (S, W)), ("attn.c_proj.b", (W,)),
              ("mlp.c_fc.w", (W, Mw)), ("mlp.c_fc.b", (Mw,)), ("mlp.c_proj.w", (Mw, W)), ("mlp.c_proj.b", (W,))]
    if af == 6:
        shapes += [("attn.c_enc_kv.w", (W, 2 * S)), ("attn.c_enc_kv.b", (2 * S,))]
    p32 = {nm: torch.from_numpy(synth_tensor(f"_attn_mods.0.{nm}", sh, 5)).cuda() for nm, sh in shapes}
    gen = torch.Generator(device="cuda").manual_seed(af * 7 + len(g))
    x = torch.randn(n, n_ctx, W, device="cuda", generator=gen)
    dy = torch.randn(n, n_ctx, W, device="cuda", generator=gen)
    enc = torch.randn(n, E, W, device="cuda", generator=gen) if af == 6 else None
    L, G = _lib.F32Layer(), _lib.F32GradLayer()
    grads = {}
    for field, nm in NAMES:
        if nm in p32:
            setattr(L, field, p32[nm].data_ptr())
            grads[nm] = torch.zeros_like(p32[nm])
            setattr(G, field, grads[nm].data_ptr())
    L.attn_func = af
    a = _lib.F32Args(n=n, P=n_ctx, p0=0, width=W, n_state=S, mlp_width=Mw, heads=H, n_ctx=n_ctx, blocks=blocks,
                     prime_len=prime_len or 0, encoder_dims=E, depth=1, x=0,
                     encoder_kv=0 if enc is None else enc.data_ptr(), work=0)
    need = C.c_size_t(0)
    _lib.check(_lib.lib().jk_f32_backward_workspace_floats(C.byref(a), C.byref(need)))
    work = torch.empty(need.value, device="cuda")
    a.work = work.data_ptr()
    dx = dy.clone()
    d_enc = torch.zeros_like(enc) if enc is not None else None
    ins = (C.c_void_p * 1)(x.data_ptr())
    _lib.check(_lib.lib().jk_f32_backward(C.byref(a), C.pointer(L), C.pointer(G), ins, _lib.ptr(dx), _lib.ptr(d_enc),
                                          _lib.stream_ptr()))
    ours = dict(grads, dx=dx)
    if d_enc is not None:
        ours["d_encoder_kv"] = d_enc
    Lk = E if af == 6 else n_ctx
    want = _grads64(p32, x, enc, dy, af, H, _mask(af, n_ctx, Lk, bc, prime, 0))
    # dK / dV through the cache rows: the key and value column blocks of c_attn's gradient (enc-dec: d_encoder_kv and
    # the c_enc_kv gradient)
    if af != 6:
        for nm in ("attn.c_attn.w", "attn.c_attn.b"):
            for part, sl in (("k", slice(S, 2 * S)), ("v", slice(2 * S, 3 * S))):
                ours[f"{nm}[{part}]"] = ours[nm][..., sl]
                want[f"{nm}[{part}]"] = want[nm][..., sl]
    # scale of each gradient: its own max, or for the key / value column blocks of c_attn the whole tensor's (the key
    # bias gradient is zero in exact arithmetic: a constant added to every score of a row leaves its softmax unchanged)
    scales = {k: float(want[k.split("[")[0]].abs().max()) for k in want}
    rel = lambda k, o, w_: float((o.double() - w_).abs().max()) / max(scales[k], 1e-300)
    errs = {k: rel(k, ours[k], want[k]) for k in want}
    del want
    shift = bc if af == 3 else 1
    wrong = _grads64(p32, x, enc, dy, af, H, _mask(af, n_ctx, Lk, bc, prime, shift))
    if af != 6:
        for nm in ("attn.c_attn.w", "attn.c_attn.b"):
            for part, sl in (("k", slice(S, 2 * S)), ("v", slice(2 * S, 3 * S))):
                wrong[f"{nm}[{part}]"] = wrong[nm][..., sl]
    away = max(rel(k, ours[k], wrong[k]) for k in wrong)
    record(dict(test="real", af=af, geom=g, tol=REAL_TOL, worst=max(errs.values()),
                worst_name=max(errs, key=errs.get), shifted_away=away, errs={k: float(f"{e:.3g}") for k, e in errs.items()}))
    for k, e in errs.items():
        assert e <= REAL_TOL, f"{k}: {e:.3e} > {REAL_TOL:.3e}"
    assert away >= 10 * REAL_TOL, f"the shifted key set is only {away:.3e} away"
