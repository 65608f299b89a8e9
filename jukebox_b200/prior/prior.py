"""SimplePrior: everything around the autoregressive model of one level - which upper-level codes and labels a
window is conditioned on, how lyric tokens enter (merged into the token sequence, or through a separate
encoder), and the hand-over to ConditionalAutoregressive2D (whose sampling loop runs on the decode engine).

The constructor signature, the sub-module names (they are state-dict keys: `prior`, `prime_prior`,
`prime_state_proj`, `prime_state_ln`, `prime_x_out`, `conditioner_blocks`, `y_emb`) and the attributes that
sample.py / train.py / the notebooks read (n_ctx, raw_to_tokens, n_tokens, labeller, level(s), z_shapes,
downsamples, cond_downsample, sample_length, prior_dims, ...) follow the reference (jukebox/prior/prior.py);
the methods are written around two small helpers:

  TokenSpaces  - the shared vocabulary of a `single_enc_dec` prior: lyric tokens and VQ codes live in one sequence,
                 VQ codes shifted past the lyric vocabulary (reference :168-203)
  LyricEncoder - the separate lyric encoder of an encoder-decoder prior: tokens -> activations -> projection ->
                 LayerNorm = the keys/values of the decoder's enc-dec attention layers (reference :285-301)

z_forward / forward evaluate the loss (bits per token), predictions and recorded attention weights of a full window
without gradients; loss_grad evaluates z_forward's loss and adds its gradient into the decoder's .grad (fine-tuning with
a torch optimiser; the optimiser step itself is torch's).
"""
import numpy as np
import torch as t
import torch.nn as nn
import torch.nn.functional as F

from ..utils import dist_adapter as dist
from ..utils.dist_adapter import print_once
from ..utils.torch_utils import assert_shape
from ..transformer.ops import LayerNorm, Conv1D
from ..transformer import f32
from ..data.labels import EmptyLabeller, Labeller
from ..vqvae.vqvae import calculate_strides
from .autoregressive import ConditionalAutoregressive2D
from .conditioners import Conditioner, LabelConditioner


class TokenSpaces:
    """Several token streams laid end to end in one sequence with disjoint id ranges."""

    def __init__(self, shapes, bins, width):
        self.shapes = [tuple(s) for s in shapes]
        self.bins = [int(b) for b in bins]
        self.dims = [int(np.prod(s)) for s in self.shapes]
        self.shift = [int(v) for v in np.cumsum([0, *self.bins])[:-1]]
        self.width = width

    def merge(self, streams, conds):
        """streams: LongTensors [N, ...], one per leading space; conds: per space [N, dims, width] or None (zeros).
        Returns (tokens [N, sum dims of the given streams], cond [N, sum dims, width])."""
        N = streams[0].shape[0]
        toks = []
        for i, x in enumerate(streams):
            assert x.dtype == t.long, x.dtype
            assert (0 <= x).all() and (x < self.bins[i]).all(), f"token stream {i} outside [0, {self.bins[i]})"
            toks.append(x.reshape(N, -1) + self.shift[i])
        parts = []
        for i, c in enumerate(conds):
            if c is None:
                c = t.zeros((N, self.dims[i], self.width), dtype=t.float, device=streams[0].device)
            else:
                assert_shape(c, (N, self.dims[i], self.width))
            parts.append(c)
        return t.cat(toks, dim=1), t.cat(parts, dim=1)

    def last(self, z):
        """the last space's tokens of a merged sequence (which may be shorter than full), ids un-shifted"""
        N = z.shape[0]
        lead = sum(self.dims[:-1])
        x = z[:, lead:] - self.shift[-1]
        x = t.clamp(x, min=0)           # a sampled id below the last space's range (a lyric id) maps to code 0
        assert (x < self.bins[-1]).all(), f"rank {dist.get_rank()}: id outside the {self.bins[-1]} codes"
        return x.reshape(N, -1, *self.shapes[-1][1:])


class SimplePrior(nn.Module):
    def __init__(self, z_shapes, l_bins, encoder, decoder, level, downs_t, strides_t, labels, prior_kwargs,
                 x_cond_kwargs, y_cond_kwargs, prime_kwargs, copy_input, labels_v3=False, merged_decoder=False,
                 single_enc_dec=False):
        super().__init__()
        self.use_tokens = prime_kwargs.pop('use_tokens')
        self.n_tokens = prime_kwargs.pop('n_tokens')
        self.prime_loss_fraction = prime_kwargs.pop('prime_loss_fraction')
        self.copy_input = copy_input
        if copy_input:
            prime_kwargs['bins'] = l_bins
        self.z_shapes, self.levels, self.level = z_shapes, len(z_shapes), level
        assert level < self.levels, f"Total levels {self.levels}, got level {level}"
        self.z_shape = z_shapes[level]
        self.l_bins = l_bins
        self.encoder, self.decoder = encoder, decoder       # bound methods of the VQ-VAE: not sub-modules
        self.cond_level = level + 1
        self.x_cond = level != self.levels - 1               # every level but the top sees the level above
        self.y_cond = labels
        self.single_enc_dec = single_enc_dec
        self._build_conditioning(z_shapes, l_bins, downs_t, strides_t, x_cond_kwargs, y_cond_kwargs)
        if single_enc_dec:
            self._build_joint(prime_kwargs, prior_kwargs)
        else:
            self._build_separate(prime_kwargs, prior_kwargs, merged_decoder)
        self.n_ctx = self.gen_loss_dims
        self.total_loss_dims = self.prime_loss_dims + self.gen_loss_dims
        self.downsamples = calculate_strides(strides_t, downs_t)
        self.cond_downsample = None if not self.x_cond else self.downsamples[level + 1]
        self.raw_to_tokens = int(np.prod(self.downsamples[:level + 1]))
        self.sample_length = self.n_ctx * self.raw_to_tokens
        self.labels_v3 = labels_v3 if labels else False
        self.labeller = Labeller(self.y_emb.max_bow_genre_size, self.n_tokens, self.sample_length,
                                 v3=labels_v3) if labels else EmptyLabeller()
        print(f"Level:{level}, Cond downsample:{self.cond_downsample}, Raw to tokens:{self.raw_to_tokens}, "
              f"Sample length:{self.sample_length}")

    # ---- construction ---------------------------------------------------------------------------------------
    def _build_conditioning(self, z_shapes, l_bins, downs_t, strides_t, x_cond_kwargs, y_cond_kwargs):
        if self.x_cond:
            print_once("Conditioning on 1 above level(s)")
            up = self.cond_level
            self.conditioner_blocks = nn.ModuleList([
                Conditioner(input_shape=z_shapes[up], bins=l_bins, down_t=downs_t[up], stride_t=strides_t[up],
                            **x_cond_kwargs)])
        if self.y_cond:
            self.n_time = self.z_shape[0]
            # an upsampler takes its timing from the codes above; the top level needs the time signal
            self.y_emb = LabelConditioner(n_time=self.n_time, include_time_signal=not self.x_cond, **y_cond_kwargs)

    def _build_joint(self, prime_kwargs, prior_kwargs):
        """lyrics and codes in ONE autoregressive sequence (1b_lyrics)"""
        spaces = TokenSpaces([(self.n_tokens,), prior_kwargs.pop('input_shape')],
                             [prime_kwargs['bins'], prior_kwargs.pop('bins')], prior_kwargs['width'])
        self.spaces = spaces
        self.prior_shapes, self.prior_bins, self.prior_dims = spaces.shapes, spaces.bins, spaces.dims
        self.prior_bins_shift, self.prior_width = np.asarray(spaces.shift), spaces.width
        print_once(f'Creating cond. autoregress with prior bins {spaces.bins}, dims {spaces.dims}, '
                   f'shift {self.prior_bins_shift}, input shape {sum(spaces.dims)}, input bins {sum(spaces.bins)}')
        self.prime_loss_dims, self.gen_loss_dims = spaces.dims
        self.prior = ConditionalAutoregressive2D(input_shape=(sum(spaces.dims),), bins=sum(spaces.bins),
                                                 x_cond=(self.x_cond or self.y_cond), y_cond=True,
                                                 prime_len=self.prime_loss_dims, **prior_kwargs)

    def _build_separate(self, prime_kwargs, prior_kwargs, merged_decoder):
        """codes only in the decoder; lyrics (if any) through their own encoder (5b_lyrics) or not at all"""
        self.prime_loss_dims = 0
        if self.n_tokens != 0 and self.use_tokens:
            self.prime_loss_dims = int(self.n_tokens)
            self.prime_acts_width, self.prime_state_width = prime_kwargs['width'], prior_kwargs['width']
            self.prime_prior = ConditionalAutoregressive2D(input_shape=(self.n_tokens,), x_cond=False, y_cond=False,
                                                           only_encode=True, **prime_kwargs)
            self.prime_state_proj = Conv1D(self.prime_acts_width, self.prime_state_width,
                                           init_scale=prime_kwargs['init_scale'])
            self.prime_state_ln = LayerNorm(self.prime_state_width)
            self.prime_bins = prime_kwargs['bins']
            self.prime_x_out = nn.Linear(self.prime_state_width, self.prime_bins, bias=False)
            nn.init.normal_(self.prime_x_out.weight, std=0.02 * prior_kwargs['init_scale'])
        self.gen_loss_dims = int(np.prod(self.z_shape))
        self.prior = ConditionalAutoregressive2D(x_cond=(self.x_cond or self.y_cond), y_cond=self.y_cond,
                                                 encoder_dims=self.prime_loss_dims, merged_decoder=merged_decoder,
                                                 **prior_kwargs)

    @property
    def has_lyric_encoder(self):
        return (not self.single_enc_dec) and self.n_tokens != 0 and bool(self.use_tokens)

    # ---- what a window is conditioned on ----------------------------------------------------------------------
    def get_y(self, labels, start, get_indices=False):
        """label rows for the window whose first token is `start`: total length, offset of the window in raw samples,
        window length, artist, genres, and the lyric tokens that fall under the window"""
        if isinstance(self.labeller, EmptyLabeller):
            return None
        y = labels['y'].clone()
        y[:, 1] += int(start * self.raw_to_tokens)
        y[:, 2] = int(self.sample_length)
        indices = self.labeller.set_y_lyric_tokens(y, labels)
        return (y, indices) if get_indices else y

    def get_z_conds(self, zs, start, end):
        """codes of the level above under tokens [start, end) of this level (None at the top level)"""
        if not self.x_cond:
            return None
        ds = self.cond_downsample
        assert start % ds == 0 and end % ds == 0, f"window [{start},{end}) not aligned to {ds}"
        above = zs[self.level + 1][:, start // ds:end // ds]
        assert above.shape[1] == self.n_ctx // ds
        return [above]

    def x_emb(self, z_conds):
        """upper-level codes -> [N, n_ctx, width] through the conditioner stack (one block: one level above)"""
        blocks = self.conditioner_blocks
        z_conds = z_conds[:self.cond_level - self.level]
        assert len(z_conds) == len(blocks) == self.cond_level - self.level
        out = None
        for block, codes in zip(reversed(list(blocks)), reversed(list(z_conds))):
            out = block(codes, out)
        return out

    def get_cond(self, z_conds, y, x_up=None):
        """-> (x_cond [N, n_ctx, W] or [N, 1, W] or None, y_cond [N, 1, W] or None, lyric tokens or None).  x_up: the
        upper-level codes through the conditioner (x_emb(z_conds)) when the caller has them already"""
        lyric = None
        if y is not None:
            n_labels = 4 + self.y_emb.max_bow_genre_size
            assert y.shape[1] == n_labels + self.n_tokens, \
                f"Expected {4} + {self.y_emb.max_bow_genre_size} + {self.n_tokens}, got {y.shape[1]}"
            y, lyric = y[:, :n_labels], y[:, n_labels:]
        y_cond = y_pos = None
        if self.y_cond:
            y_cond, y_pos = self.y_emb(y)
        if self.x_cond:
            x_cond = self.x_emb(z_conds) if x_up is None else x_up
        else:
            x_cond = y_pos
        return x_cond, y_cond, lyric

    def null_y(self, y):
        """the null label rows of y [N, label width]: the same total length, offset and window length, unknown artist,
        unknown genre and no lyrics (the labeller's row for artist "unknown", genre "unknown", lyrics "") - what
        classifier-free guidance steers away from.  A prior without labels has none: ValueError."""
        if isinstance(self.labeller, EmptyLabeller):
            raise ValueError("this prior has no labels, so there is no null conditioning to guide with")
        null = self.labeller.get_label(artist="unknown", genre="unknown", lyrics="", total_length=1, offset=0)["y"]
        out = y.clone()
        out[:, 3:] = t.as_tensor(null[3:], dtype=y.dtype, device=y.device)
        return out

    # single_enc_dec token-space helpers under the reference's names
    def prior_preprocess(self, xs, conds):
        return self.spaces.merge(xs, conds)

    def prior_postprocess(self, z):
        return self.spaces.last(z)

    # ---- VQ-VAE pass-through ----------------------------------------------------------------------------------
    def _level_span(self, start_level, end_level):
        return (self.level if start_level is None else start_level), (self.levels if end_level is None else end_level)

    def encode(self, x, start_level=None, end_level=None, bs_chunks=1):
        lo, hi = self._level_span(start_level, end_level)
        with t.no_grad():
            return self.encoder(x, start_level=lo, end_level=hi, bs_chunks=bs_chunks)

    def decode(self, zs, start_level=None, end_level=None, bs_chunks=1):
        lo, hi = self._level_span(start_level, end_level)
        assert len(zs) == hi - lo
        with t.no_grad():
            return self.decoder(zs, start_level=lo, end_level=hi, bs_chunks=bs_chunks)

    # ---- sampling -----------------------------------------------------------------------------------------------
    def sample(self, n_samples, z=None, z_conds=None, y=None, fp16=False, temp=1.0, top_k=0, top_p=0.0,
               chunk_size=None, sample_tokens=None, get_logprobs=False, select_every=None, select_keep=None,
               guidance_scale=None, guidance_y=None):
        """one window: z = codes of this level already in the window (None / empty: ancestral), z_conds = codes of the
        level above, y = label rows.  Returns the codes [N, sample_tokens or n_ctx].  With get_logprobs it returns
        (codes, logprobs): fp32 [N, sample_tokens or n_ctx], the log-likelihood in nats of each returned code under the
        model (ConditionalAutoregressive2D.sample), so that the samples of a window can be ranked.
        z of one row with n_samples > 1 (not in the reference): one prime, n_samples continuations; z_conds and y then
        have one row too, and the window runs the prime once (ConditionalAutoregressive2D.primed_sample).
        select_every / select_keep: keep-best selection inside the window (ConditionalAutoregressive2D.sample); the
        result then ends with ancestry, LongTensor [N], the input item each returned row descends from.
        guidance_scale: guided sampling (ConditionalAutoregressive2D.sample) away from, or towards, the alternative
        conditioning of the label rows guidance_y (the rows and layout of y; None: the null rows, null_y): its label
        embedding, its lyrics (merged ahead of the codes, or through the lyric encoder) and the same upper-level codes,
        whose conditioner runs once.  At most prior.guided_items() items per call."""
        fresh = z is None or z.shape[1] == 0
        rows = 1 if (not fresh and z.shape[0] == 1) else n_samples
        for name, v in (("z", z), ("y", y), *((f"z_conds[{i}]", c) for i, c in enumerate(z_conds or []))):
            assert v is None or v.shape[0] == rows, \
                f"{name}: expected batch {rows}{' (one given row)' if rows != n_samples else ''}, got {tuple(v.shape)}"
        if dist.get_rank() == 0:
            print(f"{'Ancestral' if fresh else 'Primed'} sampling {n_samples} samples with temp={temp}, "
                  f"top_k={top_k}, top_p={top_p}")
        how = dict(fp16=fp16, temp=temp, top_k=top_k, top_p=top_p)
        if get_logprobs:
            how["get_logprobs"] = True
        if select_every is not None or select_keep is not None:
            how.update(select_every=select_every, select_keep=select_keep)
        with t.no_grad():
            x_up = self.x_emb(z_conds) if self.x_cond else None
            x_cond, y_cond, lyric = self.get_cond(z_conds, y, x_up)
            alt = None
            if guidance_scale is not None:
                if isinstance(self.labeller, EmptyLabeller):
                    raise ValueError("guidance needs labels: this prior has none, so there is no other conditioning "
                                     "to guide with")
                y_alt = self.null_y(y) if guidance_y is None else guidance_y
                assert y_alt.shape == y.shape, f"guidance_y {tuple(y_alt.shape)}: expected the shape of y {tuple(y.shape)}"
                alt = self.get_cond(z_conds, y_alt.to(y.device), x_up)
                how["guidance_scale"] = guidance_scale
            if self.single_enc_dec:
                out = self._sample_joint(n_samples, None if fresh else z, lyric, x_cond, y_cond, chunk_size, sample_tokens, how, alt)
            else:
                out = self._sample_separate(n_samples, None if fresh else z, lyric, x_cond, y_cond, chunk_size, sample_tokens, how, alt)
        if sample_tokens is None:
            assert_shape(out[0] if isinstance(out, tuple) else out, (n_samples, *self.z_shape))
        return out

    def _sample_joint(self, N, z, lyric, x_cond, y_cond, chunk_size, sample_tokens, how, alt=None):
        # the lyric tokens are the head of the sequence: always a primed run of the joint model
        given = [lyric] if z is None else [lyric, z]
        seq, cond = self.spaces.merge(given, [None, x_cond])
        if alt is not None:     # the alternative's own lyric head ahead of the same codes
            x_alt, y_alt, lyric_alt = alt
            seq_alt, cond_alt = self.spaces.merge([lyric_alt] + given[1:], [None, x_alt])
            how = dict(how, x_alt=seq_alt, x_cond_alt=cond_alt, y_cond_alt=y_alt)
        total = None if sample_tokens is None else sample_tokens + self.n_tokens
        out = self.prior.primed_sample(N, seq, cond, y_cond, chunk_size=chunk_size, sample_tokens=total, **how)
        if not isinstance(out, tuple):
            return self.spaces.last(out)
        seq, *rest = out
        if how.get("get_logprobs"):
            rest[0] = rest[0][:, sum(self.spaces.dims[:-1]):]     # the lyric head stripped as from the codes
        return (self.spaces.last(seq), *rest)

    def _sample_separate(self, N, z, lyric, x_cond, y_cond, chunk_size, sample_tokens, how, alt=None):
        enc = self.get_encoder_kv(lyric, fp16=how["fp16"], sample=True)
        if alt is not None:
            x_alt, y_alt, lyric_alt = alt
            how = dict(how, x_cond_alt=x_alt, y_cond_alt=y_alt,
                       encoder_kv_alt=self.get_encoder_kv(lyric_alt, fp16=how["fp16"], sample=True))
        if z is None:
            return self.prior.sample(N, x_cond, y_cond, enc, sample_tokens=sample_tokens, **how)
        return self.prior.primed_sample(N, z, x_cond, y_cond, enc, chunk_size=chunk_size, sample_tokens=sample_tokens, **how)

    def get_encoder_kv(self, prime, fp16=False, sample=False):
        """lyric tokens -> encoder activations -> prime_state_proj (fp32 Conv1D) -> prime_state_ln: what the decoder's
        encoder-decoder attention layers read.  The reference parks the encoder on the CPU between windows to fit
        16 GB; with 180 GB it simply stays resident."""
        if not self.has_lyric_encoder:
            return None
        N = prime.shape[0]
        acts = self.prime_prior(prime, None, None, None, fp16=fp16)
        assert_shape(acts, (N, self.prime_loss_dims, self.prime_acts_width))
        assert acts.dtype == t.float
        states = f32.linear_kn(acts.reshape(-1, self.prime_acts_width), self.prime_state_proj.w,
                               self.prime_state_proj.b).view(N, self.prime_loss_dims, -1)
        kv = self.prime_state_ln(states)
        return kv.half() if (sample and fp16) else kv

    def get_prime_loss(self, encoder_kv, prime_t):
        """bits per lyric token of the encoder's next-token head (reference prior.py:303-310)"""
        if not self.use_tokens:
            return t.tensor(0.0, device=prime_t.device)
        N, L, W = encoder_kv.shape
        logits = f32.linear_nk(encoder_kv.float().reshape(N * L, W), self.prime_x_out.weight)
        return F.cross_entropy(logits, prime_t.reshape(-1)) / float(np.log(2.))

    def _condition(self, z, z_conds, y, fp16):
        """one window of codes z [N, D] and what it is conditioned on: the upper-level codes and labels (get_cond), the
        lyric tokens (with copy_input the window's own head), merged ahead of the codes for a single_enc_dec prior, else
        turned into the lyric encoder's keys.  Returns (the token sequence self.prior reads, x_cond, y_cond, encoder_kv or
        None, the lyric tokens, the length of the sequence's lyric head: prime_len for single_enc_dec, else 0)."""
        x_cond, y_cond, lyric = self.get_cond(z_conds, y)
        if self.copy_input:
            lyric = z[:, :self.n_tokens]
        if self.single_enc_dec:
            seq, x_cond = self.prior_preprocess([lyric, z], [None, x_cond])
            return seq, x_cond, y_cond, None, lyric, self.prior.prime_len
        return z, x_cond, y_cond, self.get_encoder_kv(lyric, fp16=fp16), lyric, 0

    def z_forward(self, z, z_conds=[], y=None, fp16=False, get_preds=False, get_attn_weights=False):
        """Evaluation forward over one full window of codes (reference prior.py:312-349): returns (loss, metrics), or -
        with get_attn_weights (True or a set of layer indices) - the recorded attention weights of those layers, which
        is what lyric alignment reads (reference jukebox/align.py get_alignment).
        No gradients are kept: the loss is the evaluation metric (bits per token); loss_grad is the same loss with the
        decoder's gradients."""
        assert isinstance(get_attn_weights, (bool, set))
        tr = self.prior.transformer
        if get_attn_weights:
            tr.set_record_attn(get_attn_weights)
        seq, x_cond, y_cond, enc, lyric, _ = self._condition(z, z_conds, y, fp16)
        if self.single_enc_dec:
            (prime_loss, gen_loss), preds = self.prior(seq, x_cond, y_cond, fp16=fp16, get_sep_loss=True,
                                                       get_preds=get_preds)
        else:
            prime_loss = self.get_prime_loss(enc, lyric) if enc is not None else t.tensor(0.0, device=z.device)
            gen_loss, preds = self.prior(seq, x_cond, y_cond, enc, fp16=fp16, get_preds=get_preds)
        if get_attn_weights:
            ws = tr.ws
            tr.set_record_attn(False)
            return ws
        total = self.total_loss_dims
        loss = self.prime_loss_fraction * prime_loss * self.prime_loss_dims / total + gen_loss * self.gen_loss_dims / total
        metrics = dict(bpd=gen_loss.clone(), prime_loss=prime_loss.clone(), gen_loss=gen_loss.clone())
        if get_preds:
            metrics["preds"] = preds.clone()
        return loss, metrics

    def loss_grad(self, z, z_conds=[], y=None):
        """Fine-tuning: z_forward(fp16=False)'s (loss, metrics) of one full window of codes, and the gradient of that loss
        ADDED into p.grad (fp32, created when None) of every parameter of self.prior (the ConditionalAutoregressive2D
        decoder) that requires grad.  The conditioner, the label embedding, the lyric encoder and the VQ-VAE are frozen:
        x_cond, y_cond and the encoder keys are constants, and a separate encoder's prime loss, which depends on them
        alone, adds no gradient.  Each token's cross-entropy enters with its weight in the loss: 1 / (N total_loss_dims
        ln 2) for a code, prime_loss_fraction times that for a lyric token of a single_enc_dec sequence.
            prior.prior.requires_grad_(True)        # or only the layers to train
            opt = torch.optim.Adam([p for p in prior.prior.parameters() if p.requires_grad], lr, betas=(0.9, beta2))
            loss, metrics = prior.loss_grad(z, z_conds, y); opt.step(); opt.zero_grad()
        Refused before any launch when nothing requires grad, for fp16_params or res_scale priors, attn_func 4 / 5,
        a partial window or a module off the GPU."""
        D = int(np.prod(z.shape[1:]))
        why = self.prior.grad_refusal()
        if why is None and D != self.gen_loss_dims:
            why = f"gradients are taken over whole windows of {self.gen_loss_dims} codes, got {D}"
        if why:
            raise ValueError(why)
        with t.no_grad():
            seq, x_cond, y_cond, enc, lyric, head = self._condition(z, z_conds, y, fp16=False)
            N = z.shape[0]
            ln2 = float(np.log(2.))
            unit = 1.0 / (N * self.total_loss_dims * ln2)
            w = t.full(tuple(seq.view(N, -1).shape), unit, dtype=t.float32, device=z.device)
            w[:, :head] = self.prime_loss_fraction * unit
        ce = self.prior.loss_grad(seq, x_cond, y_cond, enc, row_weights=w)
        with t.no_grad():
            ce = ce.double()
            gen_loss = (ce[:, head:].mean() / ln2).float()
            if self.single_enc_dec:
                prime_loss = (ce[:, :head].mean() / ln2).float()
            else:
                prime_loss = self.get_prime_loss(enc, lyric) if enc is not None else t.tensor(0.0, device=z.device)
            total = self.total_loss_dims
            loss = self.prime_loss_fraction * prime_loss * self.prime_loss_dims / total + gen_loss * self.gen_loss_dims / total
            metrics = dict(bpd=gen_loss.clone(), prime_loss=prime_loss.clone(), gen_loss=gen_loss.clone())
        return loss, metrics

    def score(self, z, z_conds=[], y=None, fp16=True):
        """Per-item bits per token of one full window of codes, conditioned exactly as z_forward conditions it: returns
        (gen [N], prime [N] or None).  gen is the mean over the window's codes, prime over its lyric tokens (priors with
        lyrics: the lyric head of a single_enc_dec sequence, split where get_sep_loss splits it, or the lyric encoder's
        next-token head prime_x_out).  Their item means are z_forward's gen_loss / prime_loss.  fp16 picks the
        activations as z_forward does (decode engine or fp32 path); x_out and the log-softmax at the target then run in
        one fused kernel, with no logits tensor, so that many candidates of a window can be ranked cheaply."""
        from ..score import xout_logprob
        ln2 = float(np.log(2.))
        with t.no_grad():
            seq, x_cond, y_cond, enc, lyric, pl = self._condition(z, z_conds, y, fp16)
            logp = self.prior.logprob(seq, x_cond, y_cond, enc, fp16=fp16)
            if self.single_enc_dec:
                bits = -logp / ln2
                return bits[:, pl:].mean(1), bits[:, :pl].mean(1)
            gen = -logp.mean(1) / ln2
            prime = None
            if enc is not None:
                N, L, W = enc.shape
                lp = xout_logprob(enc.float().reshape(N * L, W), self.prime_x_out.weight, lyric.reshape(-1))
                prime = -lp.view(N, L).mean(1) / ln2
            return gen, prime

    def token_stats(self, z, z_conds=[], y=None, fp16=True, top_k=0):
        """Per-code statistics of the model's prediction for codes z [N, D] (2 <= D <= n_ctx) of this level, conditioned
        exactly as score conditions a window: a score.TokenStats of logp / entropy / lse [N, D] and, with top_k,
        topk_ids / topk_logp [N, D, top_k] (ConditionalAutoregressive2D.token_stats).  A single_enc_dec prior takes its
        lyric head into the causal pass and returns the music positions only; its top-k ids are shifted into this
        level's code space as sampled tokens are, and an id of the lyric vocabulary comes back as -1 (its
        log-probability stays: the model put that mass there)."""
        from ..score import TokenStats
        with t.no_grad():
            seq, x_cond, y_cond, enc, _, pl = self._condition(z, z_conds, y, fp16)
            st = self.prior.token_stats(seq, x_cond, y_cond, enc, fp16=fp16, top_k=top_k)
            if not self.single_enc_dec:
                return st
            st = TokenStats(*(None if v is None else v[:, pl:] for v in st))
            if top_k:
                ids = st.topk_ids - self.spaces.shift[-1]
                st = st._replace(topk_ids=t.where(ids >= 0, ids, t.full_like(ids, -1)))
            return st

    def guided_items(self):
        """the most items one guided sample call takes (ConditionalAutoregressive2D.guided_items)"""
        return self.prior.guided_items()

    def engine_rows(self):
        """the most rows one window of this level runs on one engine (ConditionalAutoregressive2D.engine_rows)"""
        return self.prior.engine_rows()

    def regenerate(self, z, start, end, n_candidates, z_conds=[], y=None, fp16=True, temp=1.0, top_k=0, top_p=0.0,
                   pack=False):
        """Resample codes [start, end) of a window of codes z [N, D] of this level (not in the reference), conditioned as
        score conditions a window: n_candidates draws of the span per item, ranked by the log-likelihood of the codes
        after it (ConditionalAutoregressive2D.regenerate).  A single_enc_dec prior takes its lyric head into the
        sequence (the span moves behind it, and the codes are shifted into its token space as sampled codes are); a
        separate lyric encoder gives the encoder-decoder layers their keys, repeated to the candidate rows.  Returns
        (z_new [N, D], scores fp32 [N, n_candidates]): the kept span in z, and each candidate's suffix log-likelihood in
        nats.  pack: the N items (windows of one geometry) in one engine window of N * n_candidates <= engine_rows()
        rows, with their own conditioning (ConditionalAutoregressive2D.regenerate)."""
        with t.no_grad():
            seq, x_cond, y_cond, enc, _, pl = self._condition(z, z_conds, y, fp16)
            out, scores = self.prior.regenerate(seq, pl + int(start), pl + int(end), n_candidates, x_cond, y_cond, enc,
                                                fp16=fp16, temp=temp, top_k=top_k, top_p=top_p, pack=pack)
            return (self.spaces.last(out) if self.single_enc_dec else out), scores

    def layer_acts(self, z, z_conds=[], y=None, layers=(), fp16=True, pool=True):
        """Representations of codes z [N, D] (D <= n_ctx) of this level, conditioned exactly as z_forward / score
        condition them: {layer: fp32 [N, width]} (pool: the mean over the window's codes) or [N, D, width], the outputs
        of those layers of the stack + x_cond (ConditionalAutoregressive2D.layer_acts).  A single_enc_dec prior takes
        its lyric head into the causal pass but keeps only the music positions; a separate lyric encoder gives the
        encoder-decoder layers their keys as in score."""
        with t.no_grad():
            seq, x_cond, y_cond, enc, _, pl = self._condition(z, z_conds, y, fp16)
            return self.prior.layer_acts(seq, x_cond, y_cond, enc, layers=layers, fp16=fp16, pool=pool, t0=pl)

    def forward(self, x, y=None, fp16=False, decode=False, get_preds=False):
        """audio -> codes of every level -> z_forward at this level (reference prior.py:351-359)"""
        z, *z_conds = self.encode(x, bs_chunks=x.shape[0])
        loss, metrics = self.z_forward(z=z, z_conds=z_conds, y=y, fp16=fp16, get_preds=get_preds)
        x_out = self.decode([z, *z_conds]) if decode else None
        return x_out, loss, metrics
