"""Transformer stack whose sample-mode forward is ONE persistent CUDA kernel per token.

Surface kept from the reference (jukebox/transformer/transformer.py): MLP, ResAttnBlock,
Transformer(n_in, n_ctx, n_head, n_depth, ..., attn_order, blocks, encoder_dims, prime_len),
Transformer.forward(x, encoder_kv=None, sample=False, fp16=False, fp16_out=False),
check_cache, del_cache, set_record_attn, ws, _attn_mods and every parameter name.
"""
import torch as t
import torch.nn as nn

from .ops import Conv1D, LayerNorm
from .factored_attention import FactoredAttention

# per-layer attention pattern of each attn_order (reference transformer.py:110-124)
_ORDERS = {
    0: ([0], None), 1: ([1, 2], None), 2: ([1, 2, 3], None), 3: ([1, 4], None), 4: ([1, 5], None),
    5: ([1, 4, 1, 1], None), 6: ([1, 2, 3, 6], None), 7: ([1, 2, 3] * 5 + [6], None),
    8: ([1, 2, 3, 1, 2, 3, 1, 2, 3, 6], None), 9: ([1, 2, 3, 0], None),
    10: ([1, 2, 3] * 3 + [1, 2, 3, 1, 2, 3, 1, 2, 3, 6] * 7, None),
    11: ([1, 2, 3], [6, 6, 0]), 12: ([1, 2, 3], [7, 7, 0]),
}


def attn_func_of(attn_order, d):
    cyc, special = _ORDERS[attn_order]
    if special is not None:                 # orders 11/12: every 16th layer is a lyric / dense layer
        return special[d % 3] if d % 16 == 15 else cyc[d % 3]
    return cyc[d % len(cyc)]


class MLP(nn.Module):
    def __init__(self, n_in, n_state, resid_dropout=0.0, afn='quick_gelu', zero_out=False, init_scale=1.0):
        super().__init__()
        assert afn == 'quick_gelu', "only quick_gelu is used by the named models"
        self.c_fc = Conv1D(n_in, n_state, init_scale=init_scale)
        self.c_proj = Conv1D(n_state, n_in, zero_out, init_scale=init_scale)


class ResAttnBlock(nn.Module):
    def __init__(self, n_in, n_ctx, n_head, attn_dropout=0.0, resid_dropout=0.0, afn='quick_gelu', scale=True,
                 mask=False, zero_out=False, init_scale=1.0, res_scale=1.0, m_attn=0.25, m_mlp=1.,
                 checkpoint_attn=0, checkpoint_mlp=0, attn_func=0, blocks=None, spread=None,
                 encoder_dims=None, prime_len=None):
        super().__init__()
        self.attn = FactoredAttention(n_in=n_in, n_ctx=n_ctx, n_state=int(m_attn * n_in), n_head=n_head,
                                      attn_dropout=attn_dropout, resid_dropout=resid_dropout, scale=scale,
                                      mask=mask, zero_out=zero_out, init_scale=init_scale,
                                      checkpoint_attn=checkpoint_attn, attn_func=attn_func, blocks=blocks,
                                      spread=spread, encoder_dims=encoder_dims, prime_len=prime_len)
        self.ln_0 = LayerNorm(n_in)
        self.mlp = MLP(n_in=n_in, n_state=int(m_mlp * n_in), resid_dropout=resid_dropout, afn=afn,
                       zero_out=zero_out, init_scale=init_scale)
        self.ln_1 = LayerNorm(n_in)
        self.res_scale = res_scale
        self.n_in = n_in
        self.attn_func = attn_func


class Transformer(nn.Module):
    def __init__(self, n_in, n_ctx, n_head, n_depth, attn_dropout=0.0, resid_dropout=0.0, afn='quick_gelu',
                 scale=True, mask=False, zero_out=False, init_scale=1.0, res_scale=False, m_attn=0.25, m_mlp=1.,
                 checkpoint_attn=0, checkpoint_mlp=0, checkpoint_res=0, attn_order=0, blocks=None, spread=None,
                 encoder_dims=None, prime_len=None):
        super().__init__()
        self.n_in, self.n_ctx, self.n_head, self.n_depth = n_in, n_ctx, n_head, n_depth
        self.encoder_dims, self.blocks, self.prime_len = encoder_dims, blocks, prime_len
        self.m_attn, self.m_mlp = m_attn, m_mlp
        if blocks is not None:
            assert n_ctx % blocks == 0
            self.block_ctx = n_ctx // blocks
        rs = 1.0 / n_depth if res_scale else 1.0
        self._attn_mods = nn.ModuleList()
        for d in range(n_depth):
            f = attn_func_of(attn_order, d)
            self._attn_mods.append(ResAttnBlock(
                n_in=n_in, n_ctx=n_ctx, n_head=n_head, attn_dropout=attn_dropout, resid_dropout=resid_dropout,
                afn=afn, scale=scale, mask=mask, zero_out=zero_out if f != 6 else True, init_scale=init_scale,
                res_scale=rs, m_attn=m_attn, m_mlp=m_mlp, checkpoint_attn=checkpoint_attn,
                checkpoint_mlp=checkpoint_mlp, attn_func=f, blocks=blocks, spread=spread,
                encoder_dims=encoder_dims, prime_len=prime_len))
        self.checkpoint_res = checkpoint_res
        self.ws = []
        # decode engine state (not parameters)
        self._engine = None
        self._engine_version = None
        self._engine_cfg = dict(bins=0, add_cond_after=True)
        self._enc_loaded = False
        self._f32 = None
        self._record_layers = []
        self.register_load_state_dict_post_hook(lambda m, keys: m.drop_engine())

    # ---- engine management --------------------------------------------------------------
    def drop_engine(self):
        self._engine = None
        self._enc_loaded = False
        self._f32 = None

    def _apply(self, fn, *a, **k):          # .cuda() / .cpu() / .half(): packed weights are stale
        self.drop_engine()
        return super()._apply(fn, *a, **k)

    def configure_engine(self, bins=0, add_cond_after=True):
        """Called by ConditionalAutoregressive2D so the same kernel also produces the logits."""
        cfg = dict(bins=int(bins), add_cond_after=bool(add_cond_after))
        if cfg != self._engine_cfg:
            self._engine_cfg = cfg
            self.drop_engine()

    def engine(self, n_samples):
        from ..engine import DecodeEngine
        dev = self._attn_mods[0].ln_0.weight.device
        if dev.type != "cuda":
            raise RuntimeError("Transformer.forward(sample=True) needs the module on a CUDA device: "
                               "jukebox_b200 has no CPU path (use the oracle in tests)")
        if self._engine is not None and self._engine_version != self._weights_version():
            self.drop_engine()          # weights changed in place (an optimiser step): the packed copy is stale
        if not self._engine_fits(n_samples, dev):
            if self.res_scale_unsupported():
                raise NotImplementedError("res_scale=True priors are not supported by the decode engine yet")
            eng = DecodeEngine(device=dev, **self._engine_kwargs(n_samples))
            for i, blk in enumerate(self._attn_mods):
                eng.load_layer(i, blk)
            self._engine = eng
            self._engine_version = self._weights_version()
            self._enc_loaded = False
            for l in self._attn_mods:
                l.attn.del_cache()
        return self._engine

    def _weights_version(self):
        """the version counters of the stack's parameters: an in-place update (optimiser step) changes them, as
        load_state_dict / .cuda() change what drop_engine reacts to"""
        return tuple(p._version for p in self._attn_mods.parameters())

    def _engine_fits(self, n_samples, dev):
        return self._engine is not None and self._engine.max_batch >= n_samples and self._engine.device == dev

    def _engine_kwargs(self, n_samples):
        l0 = self._attn_mods[0]
        return dict(width=self.n_in, depth=self.n_depth, heads=self.n_head, n_state=l0.attn.n_state,
                    mlp_width=l0.mlp.c_fc.n_out, n_ctx=self.n_ctx, blocks=self.blocks,
                    attn_funcs=[l.attn_func for l in self._attn_mods], prime_len=self.prime_len,
                    encoder_dims=self.encoder_dims, max_batch=max(1, n_samples), **self._engine_cfg)

    def prefill_capacity(self, n_samples):
        """positions one fp16 prefill of n_samples can take, without building an engine when none is built yet: 0 when
        this stack has no prefill, or no engine for this configuration / batch (more than JK_MAX_BATCH samples)"""
        from ..engine import config_prefill_capacity
        dev = self._attn_mods[0].ln_0.weight.device
        if self._engine_fits(n_samples, dev):
            return self._engine.prefill_capacity
        if dev.type != "cuda" or self.res_scale_unsupported():
            return 0
        return config_prefill_capacity(dev, **self._engine_kwargs(n_samples))

    def res_scale_unsupported(self):
        return any(l.res_scale != 1.0 for l in self._attn_mods)

    # ---- reference surface --------------------------------------------------------------
    def set_record_attn(self, record_attn):
        """record_attn: False / True / a collection of layer indices (reference transformer.py:146-163).  Recorded
        weights appear in `self.ws` after the next whole-sequence forward, one [n, heads, queries, keys] tensor per
        recorded layer, keys indexed by absolute position (encoder row for an enc-dec layer; a prime layer keeps its
        music queries x lyric keys, [:, :, prime_len:, :prime_len]) - the reference's own layout.  Zeros outside a
        layer's pattern.  Which pass records them:
          ConditionalAutoregressive2D.forward(fp16=True) with a window that fits one prefill (prefill_capacity): the fp16
              prefill, fp16 weights fp16(softmax_fp32(fp16(fp16(q.k) * dh^-1/2))) - the reference's fp16 mode;
          any other whole-sequence forward (fp16=False, Transformer.forward(sample=False), longer windows): the fp32
              forward-mode path, fp32 weights."""
        def _on(layer_idx):
            if isinstance(record_attn, bool):
                return record_attn
            return layer_idx in record_attn
        self._record_layers = [i for i in range(self.n_depth) if _on(i)]
        for i, l in enumerate(self._attn_mods):
            l.attn.record_attn = _on(i)
        if not self._record_layers:
            self.ws = []
            for l in self._attn_mods:
                l.attn.w = None

    def f32_path(self):
        from .f32 import F32Path
        if self._f32 is None:
            self._f32 = F32Path(self)
        return self._f32

    def _forward_f32(self, x, encoder_kv, sample):
        path = self.f32_path()
        n, l = x.shape[0], x.shape[1]
        if sample:
            p0 = path.pos
            out, _ = path.run(x, encoder_kv, p0)
            path.pos = p0 + l
            for b in self._attn_mods:
                b.attn._advance(n, l, False)
            return out
        assert l == self.n_ctx, f"forward mode runs whole sequences of n_ctx = {self.n_ctx} positions, got {l}"
        path.reset()
        out, ws = path.run(x, encoder_kv, 0, record=self._record_layers)
        path.reset()
        if self._record_layers:
            self.store_ws(ws)
        return out

    def record_ld(self, layer):
        """keys per recorded row of `layer`: encoder rows (enc-dec), the lyric prefix (prime), else the context"""
        f = self._attn_mods[layer].attn_func
        return self.encoder_dims if f == 6 else self.prime_len if f == 7 else self.n_ctx

    def store_ws(self, ws):
        """ws: {layer: [n, heads, n_ctx, keys]} weights of the recorded layers -> self.ws / attn.w"""
        for i in self._record_layers:          # prime layers keep music queries x lyric keys (factored_attention.py:103-105)
            if self._attn_mods[i].attn_func == 7:
                ws[i] = ws[i][:, :, self.prime_len:, :self.prime_len]
        self.ws = [ws[i] for i in self._record_layers]
        for i in self._record_layers:
            self._attn_mods[i].attn.w = ws[i]

    def forward(self, x, encoder_kv=None, sample=False, fp16=False, fp16_out=False, layers=None):
        """layers (not in the reference): a collection of layer indices - forward mode stops after the deepest of them
        and returns {layer: that layer's output [n, P, width]}, computed on the fp32 path (any fp16 flag, as forward mode
        here always is).  P may be shorter than n_ctx: the stack is causal, so a prefix's outputs are the full window's."""
        assert x.dim() == 3 and x.shape[2] == self.n_in
        if layers is not None:
            assert not sample, "layer outputs come from forward mode"
            outs = self.f32_path().run_layers(x, encoder_kv, layers)
            return {l: (o.half() if fp16_out else o) for l, o in outs.items()}
        if not sample or not fp16:
            # forward mode over activations (any fp16 flag: computed in fp32, a superset of the reference's fp16
            # precision; the fp16 prefill starts from tokens, ConditionalAutoregressive2D._prefill) and fp32 sampling:
            # csrc/f32_path.cu
            out = self._forward_f32(x, encoder_kv, sample)
            return out.half() if fp16_out else out
        n, l = x.shape[0], x.shape[1]
        eng = self.engine(n)
        has6 = any(b.attn_func == 6 for b in self._attn_mods)
        if has6:
            assert encoder_kv is not None
            if eng.position == 0 and not self._enc_loaded:
                eng.set_encoder_kv(encoder_kv)
                self._enc_loaded = True
        x = x.float().contiguous()
        out = t.empty(n, l, self.n_in, dtype=t.float32, device=x.device)
        for i in range(l):                   # chunked prefill == token-by-token decode (reference check_chunks)
            xi = x[:, i].contiguous()
            oi = t.empty(n, self.n_in, dtype=t.float32, device=x.device)
            eng.step(n, x_in=xi, h_out=oi)
            out[:, i] = oi
        for b in self._attn_mods:
            b.attn._advance(n, l, fp16)
        return out.half() if fp16_out else out

    def check_cache(self, n_samples, sample_t, fp16):
        for l in self._attn_mods:
            l.attn.check_cache(n_samples, sample_t, fp16)
        if self._engine is not None:
            assert not fp16 or self._engine.position == sample_t, f"engine at {self._engine.position}, expected {sample_t}"
        if not fp16 and self._f32 is not None:
            assert self._f32.pos == sample_t, f"fp32 caches at {self._f32.pos}, expected {sample_t}"

    def del_cache(self):
        for l in self._attn_mods:
            l.attn.del_cache()
        self._enc_loaded = False
        if self._engine is not None:
            self._engine.reset(0)
        if self._f32 is not None:
            self._f32.reset()
