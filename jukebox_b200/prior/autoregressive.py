"""ConditionalAutoregressive2D: the sampling loop around the persistent decode kernel.

Reference surface kept (jukebox/prior/autoregressive.py): constructor signature, parameter names
(x_emb, pos_emb.pos_emb, start_token, transformer.*, x_out), sample(...), primed_sample(...),
preprocess / postprocess.  Per token the host enqueues ONE kernel (embedding gather + whole
transformer + fp32 logits, jukebox_b200/csrc/decode_engine.cu) and one sampling kernel
(temperature + Categorical, csrc/sampling.cu; top-k / top-p keep the reference's torch filter in
front of it) - nothing synchronises with the host inside the loop (the reference's per-token
`assert (0 <= x).all()` is hoisted out).
"""
import math
from typing import NamedTuple

import numpy as np
import torch as t
import torch.nn as nn
import torch.nn.functional as F

from ..transformer.ops import filter_logits_scaled, sample_categorical, sample_categorical_scored, sample_guided
from ..transformer.transformer import Transformer
from ..utils.logger import get_range


def get_normal(*shape, std=0.01):
    w = t.empty(shape)
    nn.init.normal_(w, std=std)
    return w


def split_chunks(length, chunk_size):
    n_passes = (length + chunk_size - 1) // chunk_size
    chunk_sizes = [*[chunk_size] * (n_passes - 1), (length - 1) % chunk_size + 1]
    assert sum(chunk_sizes) == length
    return chunk_sizes


class Guide(NamedTuple):
    """The alternative conditioning of a guided window (sample / primed_sample with guidance_scale): every drawn token
    comes from g = c + (scale - 1) (c - u), c the logits under the window's conditioning and u under this one.  x_cond,
    y_cond and encoder_kv have the shapes of the window's own; x: the alternative given tokens, None for the same ones."""
    scale: float
    x_cond: object = None
    y_cond: object = None
    encoder_kv: object = None
    x: object = None


class PositionEmbedding(nn.Module):
    def __init__(self, input_shape, width, init_scale=1.0, pos_init=False):
        super().__init__()
        assert not pos_init, "pos_init=True (factorised position embeddings) is not used by any named model"
        self.input_shape = input_shape
        self.input_dims = int(np.prod(input_shape))
        self.pos_init = pos_init
        self.pos_emb = nn.Parameter(get_normal(self.input_dims, width, std=0.01 * init_scale))

    def forward(self):
        return self.pos_emb


class ConditionalAutoregressive2D(nn.Module):
    def __init__(self, input_shape, bins, width=128, depth=2, heads=1, attn_dropout=0.0, resid_dropout=0.0,
                 emb_dropout=0.0, mask=True, zero_out=False, init_scale=1.0, res_scale=False, pos_init=False,
                 m_attn=0.25, m_mlp=1, checkpoint_res=0, checkpoint_attn=0, checkpoint_mlp=0, attn_order=0,
                 blocks=None, spread=None, x_cond=False, y_cond=False, encoder_dims=0, only_encode=False,
                 merged_decoder=False, prime_len=None):
        super().__init__()
        assert emb_dropout == 0.0, "dropout is a training feature"
        self.input_shape = input_shape
        self.input_dims = int(np.prod(input_shape))
        self.encoder_dims, self.bins, self.width, self.depth = encoder_dims, bins, width, depth
        self.x_emb = nn.Embedding(bins, width)
        nn.init.normal_(self.x_emb.weight, std=0.02 * init_scale)
        self.y_cond, self.x_cond = y_cond, x_cond
        if not y_cond:
            self.start_token = nn.Parameter(get_normal(1, width, std=0.01 * init_scale))
        self.pos_emb = PositionEmbedding(input_shape=input_shape, width=width, init_scale=init_scale, pos_init=pos_init)
        self.transformer = Transformer(n_in=width, n_ctx=self.input_dims, n_head=heads, n_depth=depth,
                                       attn_dropout=attn_dropout, resid_dropout=resid_dropout, afn='quick_gelu',
                                       scale=True, mask=mask, zero_out=zero_out, init_scale=init_scale,
                                       res_scale=res_scale, m_attn=m_attn, m_mlp=m_mlp,
                                       checkpoint_attn=checkpoint_attn, checkpoint_mlp=checkpoint_mlp,
                                       checkpoint_res=checkpoint_res, attn_order=attn_order, blocks=blocks,
                                       spread=spread, encoder_dims=encoder_dims, prime_len=prime_len)
        self.only_encode = only_encode
        self.prime_len = prime_len
        self.add_cond_after_transformer = not merged_decoder
        self.share_x_emb_x_out = not merged_decoder
        if not only_encode:
            self.x_out = nn.Linear(width, bins, bias=False)
            if self.share_x_emb_x_out:
                self.x_out.weight = self.x_emb.weight

    # ---- token <-> tensor layout (reference :100-112) -------------------------------------------
    def preprocess(self, x):
        return x.view(x.shape[0], -1).long()

    def postprocess(self, x, sample_tokens=None):
        N = x.shape[0]
        assert (0 <= x).all() and (x < self.bins).all()
        if sample_tokens is None or sample_tokens == self.input_dims:
            return x.view(N, *self.input_shape)
        return x.view(N, -1)

    # ---- engine plumbing ------------------------------------------------------------------
    def _configure_engine(self):
        """the engine also computes this model's logits (none for an only_encode model) and adds x_cond where the model
        adds it"""
        self.transformer.configure_engine(bins=0 if self.only_encode else self.bins,
                                          add_cond_after=self.add_cond_after_transformer)

    def _engine(self, n_samples):
        self._configure_engine()
        eng = self.transformer.engine(n_samples)
        x_out = None if self.only_encode else self.x_out.weight
        start = None if self.y_cond else self.start_token
        # the key lives ON the engine object: a freshly built engine (drop_engine after .cuda() /
        # load_state_dict) always starts without embeddings, whatever address CPython gives it.  It holds each
        # tensor's version counter too, so that an in-place update (an optimiser step) reloads them.
        key = tuple(None if p is None else (p.data_ptr(), p._version)
                    for p in (self.x_emb.weight, self.pos_emb.pos_emb, x_out, start))
        if getattr(eng, "_emb_key", None) != key:
            eng.set_embeddings(x_emb=self.x_emb.weight, pos_emb=self.pos_emb.pos_emb, x_out=x_out,
                               start_token=None if start is None else start.view(-1))
            eng._emb_key = key
        return eng

    def _fresh_engine(self, n, encoder_kv):
        """the engine for n items at position 0 with empty caches, and the lyric encoder's keys encoder_kv [n, ...]
        loaded when a layer attends to them (attn_func 6)"""
        eng = self._engine(n)
        tr = self.transformer
        tr.del_cache()
        if any(b.attn_func == 6 for b in tr._attn_mods):
            assert encoder_kv is not None
            eng.set_encoder_kv(encoder_kv)
        return eng

    def _check_conds(self, N, x_cond, y_cond):
        D = self.input_dims
        if self.y_cond:
            assert y_cond is not None
            assert y_cond.shape == (N, 1, self.width)
            y_cond = y_cond.float().contiguous().view(N, self.width)
        else:
            assert y_cond is None
        if self.x_cond:
            assert x_cond is not None
            assert x_cond.shape == (N, D, self.width) or x_cond.shape == (N, 1, self.width), \
                f"Got {x_cond.shape}, expected ({N}, {D}/{1}, {self.width})"
            x_cond = x_cond.float().contiguous()
        else:
            assert x_cond is None      # zeros in the reference; NULL for the kernel
        return x_cond, y_cond

    def _given(self, x, x_cond, y_cond, whole):
        """the given tokens of a teacher-forced pass, checked: x [N, D] of ids in [0, bins), a whole window of input_dims
        tokens when `whole`, else a causal prefix of 2 <= D <= input_dims; x_cond / y_cond as _check_conds takes them.
        Returns (x contiguous int64, x_cond, y_cond)."""
        x = self.preprocess(x)
        N, D = x.shape
        if whole:
            assert D == self.input_dims, f"whole sequences of {self.input_dims} tokens, got {D}"
        else:
            assert 1 < D <= self.input_dims, f"windows of 2 .. {self.input_dims} tokens, got {D}"
        assert (0 <= x).all() and (x < self.bins).all()
        x_cond, y_cond = self._check_conds(N, x_cond, y_cond)
        return x.contiguous(), x_cond, y_cond

    def _add_x_cond(self, acts, x_cond, t0, t1):
        """acts [N, t1 - t0, width] of positions [t0, t1) + x_cond where this model adds it behind the stack
        (add_cond_after_transformer, reference autoregressive.py:226-227); x_cond [N, input_dims or 1, width]: one row
        serves every position"""
        if not self.add_cond_after_transformer or x_cond is None:
            return acts
        return acts + (x_cond[:, t0:t1] if x_cond.shape[1] > 1 else x_cond)

    def _run(self, n_samples, prime, x_cond, y_cond, encoder_kv, fp16, temp, top_k, top_p, get_preds, sample_tokens,
             get_logprobs=False, select_every=None, select_keep=None, guide=None):
        """shared body of sample / primed_sample.  prime: LongTensor [N, P] of given tokens (P may be 0), or [1, P]
        with its conditioning of one row too: prefilled once and repeated to the N rows.  guide: a Guide, or None."""
        cls = SamplingWindow if fp16 else SamplingWindowF32
        win = cls(self, n_samples, prime, x_cond, y_cond, encoder_kv, fp16, temp, top_k, top_p, get_preds,
                  sample_tokens, get_logprobs=get_logprobs, select_every=select_every, select_keep=select_keep,
                  guide=guide)
        win.advance(win.sample_tokens)
        return win.finish()

    # ---- reference API -----------------------------------------------------------------------
    # get_logprobs=True (not in the reference) also returns logprobs, fp32 [N, sample_tokens]: at a drawn position the
    # log-likelihood of the drawn token under the model (log-softmax at temperature 1 of the unfiltered logits), at a
    # given position the teacher-forced log-likelihood of the given token within this window.  The result is then
    # (x, logprobs), or (x, preds, logprobs) with get_preds.  The tokens are those of the same call without it.
    # select_every=k, select_keep=m (not in the reference; keep-best selection): after every k drawn tokens the rows are
    # ranked by the log-likelihood of the tokens they drew in this window (keep_best_parents), the m likeliest keep
    # their rows and the others continue copies of them (SamplingWindow.select).  The result then ends with ancestry,
    # LongTensor [N]: the input item each returned row descends from.
    # guidance_scale (not in the reference; guided sampling): every drawn token comes from g = c + (guidance_scale - 1)
    # (c - u), c the logits under (x_cond, y_cond, encoder_kv) and u under the alternative (x_cond_alt, y_cond_alt,
    # encoder_kv_alt, of the same shapes; x_alt: the alternative given tokens, default the same), then temp / top-k /
    # top-p as unguided.  Scale 1 draws exactly the unguided tokens, > 1 is classifier-free guidance away from u, (0, 1)
    # blends the two.  The window runs 2N engine rows (rows N.. carry u), so N <= guided_items(); results are the N
    # conditional rows: logprobs / preds under c, keep-best selection moves each pair together.
    def sample(self, n_samples, x_cond=None, y_cond=None, encoder_kv=None, fp16=False, temp=1.0, top_k=0,
               top_p=0.0, get_preds=False, sample_tokens=None, get_logprobs=False, select_every=None, select_keep=None,
               guidance_scale=None, x_cond_alt=None, y_cond_alt=None, encoder_kv_alt=None):
        prime = t.zeros(n_samples, 0, dtype=t.long, device=self.x_emb.weight.device)
        guide = None if guidance_scale is None else Guide(guidance_scale, x_cond_alt, y_cond_alt, encoder_kv_alt)
        return self._run(n_samples, prime, x_cond, y_cond, encoder_kv, fp16, temp, top_k, top_p, get_preds,
                         sample_tokens, get_logprobs, select_every, select_keep, guide)

    def primed_sample(self, n_samples, x, x_cond=None, y_cond=None, encoder_kv=None, fp16=False, temp=1.0,
                      top_k=0, top_p=0.0, get_preds=False, chunk_size=None, sample_tokens=None, get_logprobs=False,
                      select_every=None, select_keep=None, guidance_scale=None, x_cond_alt=None, y_cond_alt=None,
                      encoder_kv_alt=None, x_alt=None):
        """`chunk_size` is accepted for compatibility: the prefill runs token by token through the
        same persistent kernel, which is what chunked prefill computes (reference check_chunks).
        x may be one row for n_samples > 1 (not in the reference): one prime, n_samples continuations.  x_cond, y_cond
        and encoder_kv then have one row as well; the prime is run once and its state repeated to every row, whose draws
        still differ (the sampler's random stream is keyed by row)."""
        with t.no_grad():
            x = self.preprocess(x)
        assert x.shape[0] == n_samples or (x.shape[0] == 1 and x.shape[1] > 0), \
            f"prime of {x.shape[0]} rows for {n_samples} samples: give n_samples rows, or one row of given tokens"
        guide = None if guidance_scale is None else Guide(guidance_scale, x_cond_alt, y_cond_alt, encoder_kv_alt, x_alt)
        return self._run(n_samples, x, x_cond, y_cond, encoder_kv, fp16, temp, top_k, top_p, get_preds,
                         sample_tokens, get_logprobs, select_every, select_keep, guide)

    def logprob(self, x, x_cond=None, y_cond=None, encoder_kv=None, fp16=True):
        """log-likelihood in nats of every token of whole sequences x [N, input_dims] given the ones before it, fp32
        [N, input_dims]: the activations of `forward` (fp16: the decode engine's prefill, or its steps beyond the prefill
        capacity, in pieces of items the engine takes; fp32: the fp32 path), + cond, then x_out and the log-softmax at the
        target in one fused kernel (jk_xout_logprob) - no logits tensor."""
        from ..score import xout_logprob
        assert not self.only_encode
        with t.no_grad():
            x, x_cond, y_cond = self._given(x, x_cond, y_cond, whole=True)
            N, D = x.shape
            acts = self._add_x_cond(self._stack_out(x, x_cond, y_cond, encoder_kv, fp16), x_cond, 0, D)
            return xout_logprob(acts.reshape(N * D, self.width), self.x_out.weight, x.view(-1)).view(N, D)

    def token_stats(self, x, x_cond=None, y_cond=None, encoder_kv=None, fp16=True, top_k=0):
        """Statistics of the model's prediction at every position of the tokens x [N, D] (2 <= D <= input_dims; the stack
        is causal, so a prefix is scored as in the full window): a score.TokenStats of logp [N, D] (the log-likelihood of
        x, as `logprob`), entropy [N, D] in nats, topk_ids [N, D, top_k] / topk_logp (the most likely tokens, ties to the
        lower id) and lse [N, D].  The activations are logprob's; x_out and the statistics run in one fused kernel
        (jk_xout_stats) - no logits tensor.  x_cond is [N, input_dims or 1, width]: a short window reads its first D rows."""
        from ..score import xout_stats, TokenStats
        assert not self.only_encode
        with t.no_grad():
            x, x_cond, y_cond = self._given(x, x_cond, y_cond, whole=False)
            N, D = x.shape
            acts = self._add_x_cond(self._stack_out(x, x_cond, y_cond, encoder_kv, fp16), x_cond, 0, D)
            st = xout_stats(acts.reshape(N * D, self.width), self.x_out.weight, x.view(-1), top_k=top_k)
            return TokenStats(*(None if v is None else v.view(N, D, *v.shape[1:]) for v in st))

    def forward(self, x, x_cond=None, y_cond=None, encoder_kv=None, fp16=False, loss_full=False, encode=False,
                get_preds=False, get_acts=False, get_sep_loss=False):
        """Whole-sequence forward (reference autoregressive.py:116-172): the shifted token embeddings go through the
        transformer in forward mode; returns the activations for an `only_encode` model (the lyric encoder of
        separated enc-dec priors, prior.py:285-301), else (loss in bits per token, preds | acts | None).

        fp16=True runs the causal stack through the fp16 decode engine (prefill kernels); fp16=False runs the fp32
        forward-mode path (csrc/f32_path.cu).  With attention recording on (Transformer.set_record_attn), fp16=True
        records in the same prefill when the window fits one prefill call (D <= prefill_capacity), else it takes the
        fp32 path.  No gradients: training is out of scope, the loss is an evaluation."""
        with t.no_grad():
            x, x_cond, y_cond = self._given(x, x_cond, y_cond, whole=True)
            N, D = x.shape
            if fp16 and self.transformer._record_layers:     # asked before an engine is built: else the fp32 path
                self._configure_engine()
                fp16 = 1 < D <= self.transformer.prefill_capacity(N)
            if fp16:
                acts = t.empty(N, D, self.width, dtype=t.float32, device=x.device)
                self._prefill(x, x_cond, y_cond, encoder_kv, h_out=acts, record=True)
            else:
                acts = self._f32_pass(x, x_cond, y_cond, encoder_kv)
            acts = self._add_x_cond(acts, x_cond, 0, D)
            if self.only_encode:
                return acts
            from ..transformer import f32
            preds = f32.linear_nk(acts.view(N * D, self.width), self.x_out.weight).view(N, D, self.bins)
            ln2 = float(np.log(2.))
            if get_sep_loss:
                assert self.prime_len is not None
                pl = self.prime_len
                loss = (F.cross_entropy(preds[:, :pl].reshape(-1, self.bins), x[:, :pl].reshape(-1)) / ln2,
                        F.cross_entropy(preds[:, pl:].reshape(-1, self.bins), x[:, pl:].reshape(-1)) / ln2)
            else:
                loss = F.cross_entropy(preds.view(-1, self.bins), x.view(-1)) / ln2
        if get_preds:
            return loss, preds
        if get_acts:
            return loss, acts
        return loss, None

    # ---- gradients (fine-tuning; not in the reference's evaluation API) ---------------------------------------------
    def grad_refusal(self, D=None):
        """why loss_grad cannot run on this model (a message), or None.  D: the window's length, when known."""
        params = [p for p in self.parameters() if p.requires_grad]
        if not params:
            return "no parameter of the prior requires grad: call requires_grad_(True) on what should be fine-tuned"
        if any(p.dtype != t.float32 for p in self.parameters()):
            return "fp16_params priors have no gradient path (fp32 parameters only)"
        if self.transformer.res_scale_unsupported():
            return "res_scale=True priors have no gradient path"
        bad = sorted({b.attn_func for b in self.transformer._attn_mods} - {0, 1, 2, 3, 6, 7})
        if bad:
            return f"attn_func {bad} has no backward in the fp32 path"
        if self.only_encode:
            return "an only_encode model has no loss"
        if D is not None and D != self.input_dims:
            return f"gradients are taken over whole windows of {self.input_dims} tokens, got {D}"
        if any(p.device.type != "cuda" for p in self.parameters()):
            return "loss_grad needs the module on a CUDA device (jukebox_b200 has no CPU path)"
        return None

    def _lowest_trainable(self):
        """the lowest layer the backward has to reach: 0 when an embedding table trains, else the lowest layer with a
        parameter that requires grad, None when only x_out does"""
        embs = [self.x_emb.weight, self.pos_emb.pos_emb] + ([] if self.y_cond else [self.start_token])
        if any(p.requires_grad for p in embs):
            return 0
        for i, blk in enumerate(self.transformer._attn_mods):
            if any(p.requires_grad for p in blk.parameters()):
                return i
        return None

    def loss_grad(self, x, x_cond=None, y_cond=None, encoder_kv=None, row_weights=None):
        """Gradients of sum_m w_m CE_m, CE_m the cross-entropy (nats) of token m of whole windows x [N, input_dims]
        given the tokens before it, with the window conditioned as `forward(fp16=False)` conditions it.  row_weights:
        w [N, input_dims] (default 1 / (N input_dims ln 2): the loss in bits per token).  Returns CE, fp32 [N, input_dims].

        The gradients are ADDED into p.grad (fp32, created when None) of every parameter of this model that requires
        grad; x_cond, y_cond and encoder_kv are constants.  The forward runs the fp32 path one layer at a time from the
        lowest layer that trains, keeping each layer's input; jk_f32_backward then recomputes and differentiates each
        layer on deterministic kernels (csrc/f32_grad.cu), so two identical calls add bit-identical gradients."""
        from ..transformer import f32
        why = self.grad_refusal(self.preprocess(x).shape[1])
        if why:
            raise ValueError(why)
        with t.no_grad():
            x, x_cond, y_cond = self._given(x, x_cond, y_cond, whole=True)
            N, D = x.shape
            if row_weights is None:
                row_weights = t.full((N, D), 1.0 / (N * D * float(np.log(2.))), dtype=t.float32, device=x.device)
            assert row_weights.shape == (N, D), f"row_weights {tuple(row_weights.shape)}, expected {(N, D)}"
            tr = self.transformer
            has6 = any(b.attn_func == 6 for b in tr._attn_mods)
            if has6:
                assert encoder_kv is not None and encoder_kv.shape == (N, tr.encoder_dims, self.width)
                encoder_kv = encoder_kv.float().contiguous()
            lowest = self._lowest_trainable()
            path = tr.f32_path()
            h0 = f32.embed(self, x, y_cond, x_cond, N, D, 0)
            out, saved = path.run_saving(h0, encoder_kv, first=self.depth - 1 if lowest is None else lowest)
            acts = self._add_x_cond(out, x_cond, 0, D).reshape(N * D, self.width).contiguous()
            w_out = self.x_out.weight
            dlogits = f32.linear_nk(acts, w_out)
            ce = f32.xent_backward(dlogits, x.view(-1), row_weights.reshape(-1))
            # a tied x_out / x_emb sums both of its gradients first and adds them to .grad once, so that a second
            # identical call doubles .grad exactly
            tied = w_out is self.x_emb.weight and w_out.requires_grad
            d_out = t.zeros_like(w_out, dtype=t.float32) if tied else \
                (f32.grad_buffer(w_out) if w_out.requires_grad else None)
            if d_out is not None:
                f32.linear_wgrad(dlogits, acts, dw=d_out)
            if lowest is not None:
                dh = path.backward(saved, f32.linear_kn(dlogits, w_out).view(N, D, self.width), encoder_kv, first=lowest)
                if lowest == 0:
                    f32.embed_backward(self, x, dh, d_x_emb=d_out if tied else None)
            if tied:
                f32.grad_buffer(w_out).add_(d_out)
            return ce.view(N, D)

    def regenerate(self, x, start, end, n_candidates, x_cond=None, y_cond=None, encoder_kv=None, fp16=True, temp=1.0,
                   top_k=0, top_p=0.0, pack=False):
        """Resample the span [start, end) of a window x [N, D] (1 < D <= input_dims) given the codes on both sides of it
        (not in the reference): sampling-importance-resampling.  Per item the prime x[i, :start] runs once on one row
        and is fanned out to n_candidates rows (primed_sample's one-row prime), the rows draw [start, end), the kept
        suffix x[i, end:] is teacher-forced on every row and each candidate is scored by the suffix's log-likelihood
        under it; the likeliest candidate is kept (ties to the lower index).  At temperature 1 (no top-k / top-p) that
        score is the importance weight of p(span | prefix, suffix).
        fp16: the drawn rows continue on the decode engine and the suffix is one continuation prefill (stepped when it
        exceeds the prefill capacity); fp32: the fp32 loop, stepping the suffix.  The scores are x_out + log-softmax at
        the suffix's codes over the stack's activations + cond, in one fused kernel (jk_xout_logprob).
        x_cond [N, input_dims or 1, width], y_cond [N, 1, width] and encoder_kv [N, ...] as sample takes them.
        Returns (x_new [N, D], scores fp32 [N, n_candidates]): x with the kept span, and every candidate's suffix
        log-likelihood in nats.  Codes outside [start, end) are returned unchanged.
        pack (not in the reference): the N items share ONE window of N * n_candidates engine rows (at most
        engine_rows()): the N primes run once on N rows, select fans item i out to rows [i K, (i + 1) K), the span is
        drawn on every row and the suffixes are teacher-forced in one continuation prefill.  One item draws exactly what
        the unpacked form draws; with more, the draws differ from it, since the sampler's stream is keyed by row."""
        from .._lib import JK_MAX_BATCH
        assert not self.only_encode
        with t.no_grad():
            x = self.preprocess(x)
            N, D = x.shape
            assert 1 < D <= self.input_dims, f"windows of 2 .. {self.input_dims} tokens, got {D}"
            start, end, K = int(start), int(end), int(n_candidates)
            if not 0 <= start < end <= D:
                raise ValueError(f"span [{start}, {end}) is empty or outside the window of {D} codes")
            if end == D:
                raise ValueError(f"span [{start}, {end}) leaves no codes after it to rank the candidates by")
            if not 1 <= K <= JK_MAX_BATCH:
                raise ValueError(f"n_candidates {K} outside [1, {JK_MAX_BATCH}]")
            if pack and N * K > self.engine_rows():
                raise ValueError(f"{N} packed items of {K} candidates need {N * K} engine rows: at most "
                                 f"{self.engine_rows()} fit one engine of this model")
            assert (0 <= x).all() and (x < self.bins).all()
            x_cond, y_cond = self._check_conds(N, x_cond, y_cond)
            y_cond = None if y_cond is None else y_cond.view(N, 1, self.width)
            x_new, scores = x.clone(), t.empty(N, K, dtype=t.float32, device=x.device)
            M = N if pack else 1
            part = lambda v, i: None if v is None else v[i:i + M]
            for i in range(0, N, M):
                x_new[i:i + M], scores[i:i + M] = self._regenerate_items(
                    x[i:i + M], start, end, K, part(x_cond, i), part(y_cond, i), part(encoder_kv, i), fp16, temp,
                    top_k, top_p)
            return x_new, scores

    def _regenerate_items(self, x, start, end, K, x_cond, y_cond, encoder_kv, fp16, temp, top_k, top_p):
        """regenerate's span of the M items x [M, D] in one window of M K rows: item i's candidates are rows
        [i K, (i + 1) K).  Returns (x_new [M, D], scores fp32 [M, K])."""
        from ..score import xout_logprob
        M, D = x.shape
        # the primes run on M rows; without one the M K rows start from the start token together
        prime = x[:, :start] if start else x.new_zeros(M * K, 0)
        rows = lambda v: None if v is None else (v if start else v.repeat_interleave(K, dim=0))
        cls = SamplingWindow if fp16 else SamplingWindowF32
        win = cls(self, M * K, prime, rows(x_cond), rows(y_cond), rows(encoder_kv), fp16, temp, top_k, top_p, False, D)
        win.advance(end)
        win.tokens[:, end:] = x[:, end:].repeat_interleave(K, dim=0)
        acts = self._suffix_acts(win, end, D)
        logp = xout_logprob(acts.reshape(-1, self.width), self.x_out.weight, win.tokens[:, end:].reshape(-1))
        scores = logp.view(M * K, D - end).double().sum(1).float().view(M, K)
        x_new = x.clone()
        for i in range(M):
            best = int(t.argmax(scores[i]))
            x_new[i, start:end] = win.tokens[i * K + best, start:end]
        self.transformer.del_cache()
        return x_new, scores

    def _suffix_acts(self, win, end, D):
        """the stack's output + cond at positions [end, D) of a window's rows, which stand at position end: one
        continuation prefill on the decode engine, or steps (beyond its prefill capacity, or on the fp32 loop)"""
        K = win.N
        h = t.empty(K, D - end, self.width, dtype=t.float32, device=win.tokens.device)
        if isinstance(win, SamplingWindow):
            eng = win.eng
            if D - end <= eng.prefill_capacity:
                eng.prefill(K, D - end, tokens=win.tokens, x_cond=win.x_cond, h_out=h)
            else:
                for j in range(D - end):
                    out = t.empty(K, self.width, dtype=t.float32, device=h.device)
                    eng.step(K, tokens=win.tokens, y_cond=win.y_cond, x_cond=win.x_cond, h_out=out)
                    h[:, j] = out
        else:
            from ..transformer import f32
            tr = self.transformer
            for j, pos in enumerate(range(end, D)):
                tr.check_cache(K, pos, False)
                e = f32.embed(self, win.tokens, win.y_cond, win.x_cond, K, 1, pos)
                h[:, j] = tr(e, encoder_kv=win.encoder_kv, sample=True, fp16=False).view(K, self.width)
        return self._add_x_cond(h, win.x_cond, end, D)

    def items_per_prefill(self, N):
        """items one fp16 prefill of this model takes: up to JK_MAX_BATCH, or half that when only the 16-row engine fits
        (5b_lyrics); 0 when the configuration has no prefill"""
        from .._lib import JK_MAX_BATCH
        self._configure_engine()
        for n in sorted({min(N, JK_MAX_BATCH), min(N, max(1, JK_MAX_BATCH // 2))}, reverse=True):
            if self.transformer.prefill_capacity(n) > 0:
                return n
        return 0

    def engine_rows(self):
        """the most rows one window of this model runs on one engine (items_per_prefill: 32 rows, 16 on 5b_lyrics)"""
        from .._lib import JK_MAX_BATCH
        return self.items_per_prefill(JK_MAX_BATCH) or JK_MAX_BATCH

    def guided_items(self):
        """the most items a guided window takes: its 2N rows must fit one engine of this model (engine_rows)"""
        return self.engine_rows() // 2

    def layer_acts(self, x, x_cond=None, y_cond=None, encoder_kv=None, layers=(), fp16=True, pool=True, add_cond=True,
                   t0=0):
        """Representations (not in the reference; JukeMIR, Castellon et al. 2021): the output of intermediate layers of
        the stack over the tokens x [N, D] (1 < D <= input_dims; the stack is causal, so a prefix's activations are the
        full window's).  Returns {layer: fp32 [N, width]} with pool (the mean over positions [t0, D)), else
        {layer: fp32 [N, D - t0, width]}.  It is what `forward` of an `only_encode` model truncated after that layer
        returns; with add_cond, x_cond is added as `forward` adds it (add_cond_after_transformer).  x_cond is
        [N, input_dims or 1, width]: a short window reads its first D rows.
        fp16: the decode engine's prefill, stopped after the deepest requested layer, with the layers' rows taken (and
        averaged) inside it (jk_act_capture); items in pieces of one engine; a window beyond the prefill capacity is an
        error.  fp32: the fp32 path up to the deepest layer, averaged by the same kernel (jk_pool_rows_f32)."""
        from .. import _lib
        from ..engine import Capture
        layers = sorted(set(int(l) for l in layers))
        assert layers and 0 <= layers[0] and layers[-1] < self.depth, f"layers {layers} outside [0, {self.depth})"
        with t.no_grad():
            x, x_cond, y_cond = self._given(x, x_cond, y_cond, whole=False)
            N, D = x.shape
            assert 0 <= t0 < D, f"t0 {t0} outside [0, {D})"
            addc = bool(add_cond) and self.add_cond_after_transformer and x_cond is not None
            dev, W = x.device, self.width
            if not fp16:
                outs = self._f32_pass(x, x_cond, y_cond, encoder_kv, layers=layers)
                res = {}
                for l, o in outs.items():
                    if pool:
                        res[l] = t.empty(N, W, dtype=t.float32, device=dev)
                        xc = x_cond if addc else None
                        _lib.check(_lib.lib().jk_pool_rows_f32(
                            _lib.ptr(o), N, D, W, int(t0), D, _lib.ptr(xc), 0 if xc is None else xc.shape[1],
                            _lib.ptr(res[l]), _lib.stream_ptr()))
                    else:
                        o = o[:, t0:]
                        res[l] = (self._add_x_cond(o, x_cond, t0, D) if add_cond else o).contiguous()
                return res
            step = self.items_per_prefill(N)
            cap = self.transformer.prefill_capacity(step) if step else 0
            if not 1 < D <= cap:
                raise RuntimeError(f"layer_acts(fp16=True): a window of {D} positions exceeds the prefill capacity "
                                   f"{cap} of this model; use fp16=False")
            res = {l: t.empty((N, W) if pool else (N, D - t0, W), dtype=t.float32, device=dev) for l in layers}
            self._prefill_items(x, x_cond, y_cond, encoder_kv, n_layers=layers[-1] + 1,
                                capture={l: Capture(b, t0, D, pool, addc) for l, b in res.items()})
            return res

    # ---- teacher-forced passes over given tokens ------------------------------------------------------------------
    def _stack_out(self, x, x_cond, y_cond, encoder_kv, fp16):
        """the stack's output fp32 [N, D, width] over the given tokens x [N, D] of any number of items (x_cond not yet
        added behind it): fp16 - the decode engine, in pieces (_prefill_items); fp32 - the fp32 path to the last layer"""
        if not fp16:
            return self._f32_pass(x, x_cond, y_cond, encoder_kv, layers=[self.depth - 1])[self.depth - 1]
        acts = t.empty(*x.shape, self.width, dtype=t.float32, device=x.device)
        self._prefill_items(x, x_cond, y_cond, encoder_kv, h_out=acts)
        return acts

    def _f32_pass(self, x, x_cond, y_cond, encoder_kv, layers=None):
        """the given tokens x [N, D] through f32.embed and the fp32 path (csrc/f32_path.cu).  With layers: {layer: its
        output [N, D, width]}, stopped after the deepest (F32Path.run_layers, any 2 <= D <= input_dims).  Without: forward
        mode's output of a whole window, which records the attention of the recorded layers (Transformer.forward)."""
        from ..transformer import f32
        N, D = x.shape
        h = f32.embed(self, x, y_cond, x_cond, N, D, 0)
        return self.transformer(h, encoder_kv=encoder_kv, fp16=False, layers=layers)

    def _prefill_items(self, x, x_cond, y_cond, encoder_kv, h_out=None, n_layers=0, capture=None):
        """_prefill over any number of items, in consecutive pieces of the one batching rule: as many items as one
        prefill takes (items_per_prefill: up to JK_MAX_BATCH, 16 for 5b_lyrics), or min(N, JK_MAX_BATCH) when no engine
        size of this model has a prefill (those pieces step their tokens).  Items are independent rows: each piece writes
        its own rows of h_out [N, ...] and of the capture buffers [N, ...]."""
        from .._lib import JK_MAX_BATCH
        N = x.shape[0]
        n = self.items_per_prefill(N) or min(N, JK_MAX_BATCH)
        rows = lambda v, i: None if v is None else v[i:i + n]
        for i in range(0, N, n):
            cap = None if capture is None else {l: c._replace(out=c.out[i:i + n]) for l, c in capture.items()}
            self._prefill(x[i:i + n], rows(x_cond, i), rows(y_cond, i), rows(encoder_kv, i), h_out=rows(h_out, i),
                          n_layers=n_layers, capture=cap)

    def _prefill(self, x, x_cond, y_cond, encoder_kv, h_out=None, record=False, n_layers=0, capture=None):
        """one teacher-forced pass of the given tokens x [N, D] on the fp16 decode engine: a fresh engine, one prefill
        that fills whichever of h_out (the stack's output, fp32 [N, D, width]), the recorded layers' attention weights
        (record: fp16, Transformer.store_ws), a stop after n_layers and the layer captures the caller asks for, then the
        caches emptied.  Position by position the prefill computes exactly the forward pass (reference check_sample,
        factored_attention.py:424-455).  A window beyond the prefill capacity steps its tokens, which gives h_out only."""
        N, D = x.shape
        tr = self.transformer
        eng = self._fresh_engine(N, encoder_kv)
        if 1 < D <= eng.prefill_capacity:
            ws = {i: t.empty(N, tr.n_head, D, tr.record_ld(i), dtype=t.float16, device=x.device)
                  for i in (tr._record_layers if record else ())}
            eng.prefill(N, D, tokens=x, y_cond=y_cond, x_cond=x_cond, h_out=h_out, record=ws, n_layers=n_layers,
                        capture=capture)
            if ws:
                tr.store_ws(ws)
        else:
            assert not (record and tr._record_layers) and not capture, "attention and captures come from the prefill"
            for i in range(D):
                out = t.empty(N, self.width, dtype=t.float32, device=x.device)
                eng.step(N, tokens=x, y_cond=y_cond, x_cond=x_cond, h_out=out)
                h_out[:, i] = out
        tr.del_cache()


def _pair_rows(a, b, name):
    """the conditional rows a and the alternative rows b of a guided window as one tensor of 2n rows"""
    if a is None and b is None:
        return None
    if a is None or b is None:
        raise ValueError(f"guidance: {name}_alt must be given exactly when {name} is")
    if tuple(a.shape) != tuple(b.shape):
        raise ValueError(f"guidance: {name}_alt {tuple(b.shape)} must have the shape of {name} {tuple(a.shape)}")
    return t.cat([a, b.to(a.device, a.dtype)], dim=0)


def keep_best_parents(scores, keep):
    """Keep-best selection of a window's rows: rows ranked by score (the log-likelihood of the tokens each drew so far,
    highest first, ties to the lower row; nan ranks last), the `keep` best keep their rows and every other row, in
    ascending order, becomes a copy of the kept rows taken round-robin in rank order.  Returns parents: row b continues
    row parents[b] (SamplingWindow.select)."""
    scores = [float(v) for v in scores]
    N = len(scores)
    assert 1 <= int(keep) <= N, f"select_keep {keep} outside [1, {N}]"
    order = sorted(range(N), key=lambda r: (-scores[r] if scores[r] == scores[r] else float("inf"), r))
    kept = order[:int(keep)]
    parents = list(range(N))
    for i, r in enumerate(sorted(set(range(N)) - set(kept))):
        parents[r] = kept[i % len(kept)]
    return parents


class _Rows:
    """The per-item state shared by both sampling windows: the rows' tokens / log-probabilities / logits and
    conditioning, which rows run (one row while a one-row prime is given, then every row), the rows' ancestry, and
    keep-best selection.  A subclass owns the K / V caches (_select_caches).
    A guided window (guide: a Guide) holds G = 2 rows per item: rows [0, items) are conditional, rows [items, 2 items)
    the alternative, each with its own conditioning and given tokens; self.N counts rows, and the results are the
    conditional rows."""

    def _init_rows(self, ca, n_samples, prime, x_cond, y_cond, encoder_kv, sample_tokens, get_preds, get_logprobs,
                   select_every, select_keep, guide=None):
        """returns encoder_kv, paired with the alternative's when guided"""
        self.ca = ca
        self.sample_tokens = ca.input_dims if sample_tokens is None else int(sample_tokens)
        self.items = n_samples
        self.G = G = 1 if guide is None else 2
        self.guide_s = None
        if guide is not None:
            limit = ca.guided_items()
            if n_samples > limit:
                raise ValueError(f"{n_samples} guided items need {2 * n_samples} engine rows: at most {limit} guided "
                                 "items fit one engine of this model")
            self.guide_s = float(guide.scale) - 1.0
            if not math.isfinite(self.guide_s):
                raise ValueError(f"guidance_scale {guide.scale} must be finite")
            x_alt = prime if guide.x is None else ca.preprocess(guide.x)
            if x_alt.shape != prime.shape:
                raise ValueError(f"guidance: x_alt {tuple(x_alt.shape)} must have the shape of x {tuple(prime.shape)}")
            prime = t.cat([prime, x_alt.to(prime.device)], dim=0)
            x_cond = _pair_rows(x_cond, guide.x_cond, "x_cond")
            y_cond = _pair_rows(y_cond, guide.y_cond, "y_cond")
            encoder_kv = _pair_rows(encoder_kv, guide.encoder_kv, "encoder_kv")
        self.N = N = G * n_samples
        self.P = P = prime.shape[1]
        assert P < self.sample_tokens <= ca.input_dims, \
            f"need given tokens {P} < sample_tokens {self.sample_tokens} <= input_dims {ca.input_dims}"
        # one given row for N samples: its positions run on one row (a pair of rows when guided), then its state is
        # repeated to all N (_fan_out); M given rows for N = M K rows (packed regeneration): row i's state goes to
        # rows [i K, (i + 1) K)
        self.n = prime.shape[0] if P else N
        assert self.n in (G, N) or (G == 1 and N % self.n == 0), f"prime of {self.n} rows for {N} samples"
        self.x_cond, self.y_cond = ca._check_conds(self.n, x_cond, y_cond)
        dev = ca.x_emb.weight.device
        self.tokens = t.zeros(N, self.sample_tokens, dtype=t.long, device=dev)
        if P:
            assert (0 <= prime).all() and (prime < ca.bins).all()
            # the given rows in rows [0, n), which the prefill and the steps of given positions read; _fan_out copies
            # them to the other rows
            self.tokens[:self.n, :P] = prime
        if (select_every is None) != (select_keep is None):
            raise ValueError("keep-best selection needs both select_every and select_keep")
        if select_every is not None:
            if not (int(select_every) >= 1 and 1 <= int(select_keep) <= self.items):
                raise ValueError(f"select_every {select_every} must be >= 1 and select_keep {select_keep} in "
                                 f"[1, {self.items}]")
            select_every, select_keep = int(select_every), int(select_keep)
        self.select_every, self.select_keep = select_every, select_keep
        self.ancestry = t.arange(self.items, device=dev).repeat(G)
        self.get_preds = get_preds
        self.preds = t.empty(N, self.sample_tokens, ca.bins, dtype=t.float32, device=dev) if get_preds else None
        # selection ranks rows by the log-likelihoods of their draws, which the sampling launch scores (get_logprobs)
        self.get_logprobs = get_logprobs
        self.scored = bool(get_logprobs or select_every)
        self.logprobs = t.zeros(N, self.sample_tokens, dtype=t.float32, device=dev) if self.scored else None
        # the key of this call's Philox stream comes from torch's default generator, so t.manual_seed /
        # seed_per_rank make sampling reproducible exactly as they do for the reference's Categorical
        self.seed = int(t.empty((), dtype=t.int64).random_().item())
        self.pos = 0
        self.fbuf = None
        self.logit_bias = None
        self._owned = {"tokens", "logprobs", "preds", "logit_bias"}     # tensors this window made itself
        if guide is not None:
            self._owned |= {"x_cond", "y_cond", "encoder_kv"}             # the paired copies
        return encoder_kv

    def select(self, parents):
        """row b of the window becomes a copy of row parents[b] (b < N, parents[b] < the rows now running): its K / V
        caches and every per-item tensor the window holds (tokens, logprobs, preds, x_cond, y_cond, logit_bias), and
        its ancestry.  The window goes on from the same position."""
        parents = [int(v) for v in (parents.tolist() if isinstance(parents, t.Tensor) else parents)]
        if len(parents) != self.N or not all(0 <= v < self.n for v in parents):
            raise ValueError(f"parents {parents}: need {self.N} rows, each in [0, {self.n})")
        self._select_caches(parents)
        idx = t.tensor(parents, dtype=t.long, device=self.tokens.device)
        moved = [b for b, v in enumerate(parents) if v != b]
        with t.no_grad():
            for name in ("tokens", "logprobs", "preds", "x_cond", "y_cond", "logit_bias", "encoder_kv"):
                v = getattr(self, name, None)
                if v is None:
                    continue
                if v.shape[0] == self.N and moved:      # in place, only the rows that change
                    if name not in self._owned:        # the caller's conditioning is copied, never written
                        v = v.clone()
                        setattr(self, name, v)
                        self._owned.add(name)
                    m = t.tensor(moved, dtype=t.long, device=v.device)
                    v[m] = v[idx[m].to(v.device)]
                elif v.shape[0] != self.N:              # a one-row tensor repeated to the N rows
                    setattr(self, name, v[idx.to(v.device)].contiguous())
                    self._owned.add(name)
            self.ancestry = self.ancestry[idx]
        self.n = self.N

    def _fan_out(self):
        """the given positions of a one-row prime are done: every row continues from it (guided: every conditional
        row from row 0, every alternative row from row 1; n given rows: each to N / n consecutive rows)"""
        self.select([b // (self.N // self.n) for b in range(self.N)])

    def _drawn(self, sample_t, x):
        """position sample_t of the running rows from their logits x [n, bins], then keep-best selection when the
        window has drawn a multiple of select_every tokens"""
        _draw(self, x, sample_t, sample_t >= self.P)
        if self.select_every and sample_t >= self.P and (sample_t + 1 - self.P) % self.select_every == 0:
            scores = self.logprobs[:self.items, self.P:sample_t + 1].double().sum(1).cpu()
            parents = keep_best_parents(scores.tolist(), self.select_keep)
            # a guided item's two rows move together: the alternative rows follow their conditional rows
            parents = [q + g * self.items for g in range(self.G) for q in parents]
            if parents != list(range(self.N)):
                self.select(parents)

    def _result(self, x):
        """x: the postprocessed tokens of the conditional rows"""
        k = self.items
        out = (x,) + ((self.preds[:k],) if self.get_preds else ()) + \
              ((self.logprobs[:k],) if self.get_logprobs else ()) + ((self.ancestry[:k],) if self.select_every else ())
        return out[0] if len(out) == 1 else out


class SamplingWindow(_Rows):
    """One sampling window in flight on the decode engine: the body of the reference's sample loop
    (prior/autoregressive.py:222-237, 300-345) split into begin / advance / finish, so that callers which
    need the window in pieces (bench.py times 1/8-window slices) drive the same code as `sample`.

    begin (constructor): caches emptied, encoder K/V loaded, the given tokens prefilled in one pass when the
    engine can (else they are stepped by `advance`).  advance(upto): one decode launch + one sampling launch
    per position, nothing synchronises with the host.  finish(): cache bookkeeping + postprocess.
    A prime of one row for N samples is prefilled (or stepped) on one row and then copied to the N rows on the engine
    (select); keep-best selection (select_every / select_keep) reorders the rows every select_every drawn tokens."""

    def __init__(self, ca, n_samples, prime, x_cond, y_cond, encoder_kv, fp16, temp, top_k, top_p, get_preds,
                 sample_tokens, get_logprobs=False, select_every=None, select_keep=None, guide=None):
        assert ca.training is False
        assert not ca.only_encode
        assert fp16, "SamplingWindowF32 is the fp32 loop"
        encoder_kv = self._init_rows(ca, n_samples, prime, x_cond, y_cond, encoder_kv, sample_tokens, get_preds,
                                     get_logprobs, select_every, select_keep, guide)
        N, n, P = self.N, self.n, self.P
        dev = ca.x_emb.weight.device
        self.eng = eng = ca._fresh_engine(N, encoder_kv)
        if encoder_kv is not None:
            assert encoder_kv.shape[0] == n, f"encoder_kv of {encoder_kv.shape[0]} rows for {n} given rows"
        self.tr = ca.transformer
        if get_preds:
            self.lbuf, self.tstride = self.preds, ca.bins
        else:
            self.lbuf, self.tstride = t.empty(N, ca.bins, dtype=t.float32, device=dev), 0
        self.temp, self.top_k, self.top_p, self.fp16 = temp, top_k, top_p, fp16
        # x_cond is added BEHIND the stack (autoregressive.py:226-227) and the logits are linear in the activation:
        # x_cond . x_out^T of every position is computed once per window, so that the engine's logits product can take
        # the fp16-valued h on the tensor cores and add this bias in its epilogue (jkb200.h: jk_step_args.logit_bias)
        if ca.add_cond_after_transformer and self.x_cond is not None and eng.has_logits_gemm:
            from ..transformer import f32
            with t.no_grad():
                Lc = self.x_cond.shape[1]
                self.logit_bias = f32.linear_nk(self.x_cond.reshape(n * Lc, ca.width), ca.x_out.weight).view(n, Lc, ca.bins)
        with t.no_grad():
            if 1 < P <= eng.prefill_capacity:
                # the given tokens go through all layers at once (the reference's chunked primed_sample,
                # autoregressive.py:300-338); chunk_size is moot - one chunk.  With get_preds their logits come from
                # the same pass: x_out over (activations + cond) in fp32 (autoregressive.py:318-325).  With get_logprobs
                # their log-likelihoods come from the same activations through the fused x_out + log-softmax kernel
                if get_preds or get_logprobs:
                    from ..transformer import f32
                    h = t.empty(n, P, ca.width, dtype=t.float32, device=dev)
                    eng.prefill(n, P, tokens=self.tokens, y_cond=self.y_cond, x_cond=self.x_cond, h_out=h)
                    h = ca._add_x_cond(h, self.x_cond, 0, P)
                    if get_preds:
                        self.preds[:n, :P] = f32.linear_nk(h.view(n * P, ca.width), ca.x_out.weight).view(n, P, ca.bins)
                    if get_logprobs:
                        from ..score import xout_logprob
                        self.logprobs[:n, :P] = xout_logprob(h.view(n * P, ca.width), ca.x_out.weight,
                                                             self.tokens[:n, :P].reshape(-1)).view(n, P)
                else:
                    eng.prefill(n, P, tokens=self.tokens, y_cond=self.y_cond, x_cond=self.x_cond)
                self.pos = P

    def _select_caches(self, parents):
        self.eng.select(parents)

    def advance(self, upto):
        """positions [self.pos, upto): given positions are teacher-forced, the others sampled"""
        upto = min(int(upto), self.sample_tokens)
        eng, P, tokens = self.eng, self.P, self.tokens
        with t.no_grad():
            for sample_t in get_range(range(self.pos, upto)):
                if sample_t >= P and self.n < self.N:
                    self._fan_out()
                n = self.n
                need = self.get_preds or self.scored or sample_t >= P
                eng.step(n, tokens=tokens, y_cond=self.y_cond, x_cond=self.x_cond,
                         logits=self.lbuf if need else None, logits_tstride=self.tstride, logit_bias=self.logit_bias)
                x = self.preds[:n, sample_t] if self.get_preds else self.lbuf[:n]
                self._drawn(sample_t, x)
        self.pos = max(self.pos, upto)

    def finish(self):
        assert self.pos == self.sample_tokens, f"window stopped at {self.pos} of {self.sample_tokens}"
        tr = self.tr
        with t.no_grad():
            for b in tr._attn_mods:
                b.attn._advance(self.N, self.sample_tokens, self.fp16)
            tr.check_cache(self.N, self.sample_tokens, self.fp16)
            tr.del_cache()
            x = self.ca.postprocess(self.tokens[:self.items], self.sample_tokens)
        return self._result(x)


def _draw(win, x, sample_t, drawn):
    """position sample_t of a window's running rows (the first win.n) from their logits x [n, bins]: the draw (x / temp
    -> top-k / nucleus filter, ops.py:113-142, one launch -> Categorical), and when the window scores its draws
    (get_logprobs, keep-best selection) the log-likelihood of the drawn or given token under x, from the same sampling
    launch"""
    if not drawn and not win.scored:
        return
    n = x.shape[0]
    if drawn and win.G == 2:     # guided: one launch draws each pair's token from its two rows (n = 2 items)
        k = win.items
        sample_guided(x[:k], x[k:], win.guide_s, win.temp, win.top_k, win.top_p, win.seed, sample_t, win.tokens[:k],
                      win.tokens[k:], win.logprobs[:k] if win.scored else None)
        return
    samp, temp = x, win.temp
    if drawn and (win.top_k or win.top_p):
        win.fbuf = filter_logits_scaled(x, win.temp, win.top_k, win.top_p, win.fbuf)
        samp, temp = win.fbuf, 1.0
    if win.scored:
        sample_categorical_scored(samp if drawn else None, x, temp, win.seed, sample_t, win.tokens[:n], win.logprobs[:n])
    else:
        sample_categorical(samp, temp, win.seed, sample_t, win.tokens[:n])


class SamplingWindowF32(_Rows):
    """sample(fp16=False) / primed_sample(fp16=False): the same loop on the fp32 path (csrc/f32_path.cu) - embedding
    row, all layers on fp32 K/V caches, + cond, x_out in fp32, then the shared filter / Categorical kernels.  Four C-ABI
    calls per token instead of one persistent kernel: exactness path, not the hot path (train.py:139 sample logging).
    Its caches are torch tensors (F32Path.caches), which select indexes."""

    def __init__(self, ca, n_samples, prime, x_cond, y_cond, encoder_kv, fp16, temp, top_k, top_p, get_preds,
                 sample_tokens, get_logprobs=False, select_every=None, select_keep=None, guide=None):
        assert ca.training is False and not ca.only_encode and not fp16
        encoder_kv = self._init_rows(ca, n_samples, prime, x_cond, y_cond, encoder_kv, sample_tokens, get_preds,
                                     get_logprobs, select_every, select_keep, guide)
        self.tr = ca.transformer
        self.tr.del_cache()
        if encoder_kv is not None:
            assert encoder_kv.shape[0] == self.n, f"encoder_kv of {encoder_kv.shape[0]} rows for {self.n} given rows"
        self.encoder_kv = encoder_kv
        self.temp, self.top_k, self.top_p = temp, top_k, top_p

    def _select_caches(self, parents):
        path = self.tr.f32_path()
        if path.caches is None:
            return
        idx = t.tensor(parents, dtype=t.long, device=path.dev)
        moved = t.tensor([b for b, v in enumerate(parents) if v != b], dtype=t.long, device=path.dev)
        for i, (k, v) in enumerate(path.caches):
            if k.shape[0] == self.N:
                if moved.numel():
                    k[moved], v[moved] = k[idx[moved]], v[idx[moved]]
            else:
                k, v = k[idx].contiguous(), v[idx].contiguous()
                path.caches[i] = (k, v)
                path.layers[i].k_cache, path.layers[i].v_cache = k.data_ptr(), v.data_ptr()
        path.cache_n = self.N
        for b in self.tr._attn_mods:
            if b.attn.cache:
                b.attn.cache["n_samples"] = self.N

    def advance(self, upto):
        from ..transformer import f32
        ca, P, tokens = self.ca, self.P, self.tokens
        upto = min(int(upto), self.sample_tokens)
        with t.no_grad():
            for sample_t in get_range(range(self.pos, upto)):
                if sample_t >= P and self.n < self.N:
                    self._fan_out()
                n = self.n
                self.tr.check_cache(n, sample_t, False)
                h = f32.embed(ca, tokens, self.y_cond, self.x_cond, n, 1, sample_t)
                h = self.tr(h, encoder_kv=self.encoder_kv, sample=True, fp16=False)
                h = ca._add_x_cond(h, self.x_cond, sample_t, sample_t + 1)
                if self.get_preds or self.scored or sample_t >= P:
                    x = f32.linear_nk(h.view(n, ca.width), ca.x_out.weight)
                    if self.get_preds:
                        self.preds[:n, sample_t] = x
                    self._drawn(sample_t, x)
        self.pos = max(self.pos, upto)

    def finish(self):
        assert self.pos == self.sample_tokens, f"window stopped at {self.pos} of {self.sample_tokens}"
        with t.no_grad():
            self.tr.check_cache(self.N, self.sample_tokens, False)
            self.tr.del_cache()
            x = self.ca.postprocess(self.tokens[:self.items], self.sample_tokens)
        return self._result(x)
