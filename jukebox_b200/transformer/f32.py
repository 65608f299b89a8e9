"""fp32 transformer path (csrc/f32_path.cu): Transformer.forward(fp16=False) in both modes.

  forward mode  - Transformer.forward(x, encoder_kv, sample=False): a whole sequence at once, the reference's training-shaped
                  call (transformer/transformer.py:169-192, masks of factored_attention.py:135-228), used by
                  ConditionalAutoregressive2D.forward (losses, get_preds, the only_encode lyric encoder) and by alignment
                  with record_attn (prior/prior.py:327-344);
  sampling mode - Transformer.forward(x, sample=True, fp16=False): positions appended one call at a time on fp32 K/V caches
                  (ConditionalAutoregressive2D.sample(fp16=False), which train.py:139 uses for its sample logging).

Not the hot path - the reference samples in fp16 (sample.py:239-241) and that is what the persistent decode kernel runs.
This path exists for exactness against the reference's fp32 outputs (tests at 2e-5) and as the fp32 side of the
reference's fp16-vs-fp32 criterion.  All arithmetic happens in libjkb200.so; there is no torch fallback.
"""
import ctypes as C

import torch as t

from .. import _lib


def layer_params(blk):
    """(field of jk_f32_layer / jk_f32_grad_layer, parameter) of one ResAttnBlock; c_enc_kv only in an enc-dec layer"""
    a, mlp = blk.attn, blk.mlp
    out = [("ln0_g", blk.ln_0.weight), ("ln0_b", blk.ln_0.bias), ("ln1_g", blk.ln_1.weight), ("ln1_b", blk.ln_1.bias),
           ("c_attn_w", a.c_attn.w), ("c_attn_b", a.c_attn.b), ("c_proj_w", a.c_proj.w), ("c_proj_b", a.c_proj.b),
           ("fc_w", mlp.c_fc.w), ("fc_b", mlp.c_fc.b), ("proj2_w", mlp.c_proj.w), ("proj2_b", mlp.c_proj.b)]
    if blk.attn_func == 6:
        out += [("c_enc_kv_w", a.c_enc_kv.w), ("c_enc_kv_b", a.c_enc_kv.b)]
    return out


def grad_buffer(p):
    """p.grad, created as fp32 zeros when None: the buffer a gradient kernel adds into"""
    if p.grad is None:
        p.grad = t.zeros_like(p, dtype=t.float32, memory_format=t.contiguous_format)
    g = p.grad
    if g.dtype != t.float32 or not g.is_contiguous() or g.device != p.device:
        raise RuntimeError(f"{tuple(p.shape)} parameter's .grad must be a contiguous fp32 tensor on {p.device}")
    return g


class F32Path:
    """Per-Transformer state of the fp32 path: fp32 parameter views, K/V caches of the current window, workspace."""

    def __init__(self, tr):
        self.tr = tr
        l0 = tr._attn_mods[0]
        self.dev = l0.ln_0.weight.device
        if self.dev.type != "cuda":
            raise RuntimeError("the fp32 transformer path needs the module on a CUDA device (jukebox_b200 has no CPU path)")
        self.W, self.S, self.M = tr.n_in, l0.attn.n_state, l0.mlp.c_fc.n_out
        self.depth = tr.n_depth
        self.keep = []          # fp32 copies of parameters stored in another dtype
        self.layers = (_lib.F32Layer * self.depth)()
        for i, blk in enumerate(tr._attn_mods):
            if blk.res_scale != 1.0:
                raise NotImplementedError("res_scale=True priors are not built (no named model uses them)")
            L = self.layers[i]
            a = blk.attn
            for name, p in layer_params(blk):
                setattr(L, name, self._f32(p))
            L.attn_func = blk.attn_func
        self.caches = None      # [(k, v)] per layer
        self.cache_n = 0
        self.pos = 0
        self.work = None

    def _f32(self, p):
        d = p.detach()
        if d.dtype != t.float32 or not d.is_contiguous():
            d = d.float().contiguous()
            self.keep.append(d)
        return d.data_ptr()

    def _alloc_caches(self, n, upto=None):
        """caches of layers [0, upto) (all when None); later layers get none and must not run"""
        tr = self.tr
        self.caches = []
        for i, blk in enumerate(tr._attn_mods):
            if upto is not None and i >= upto:
                self.layers[i].k_cache = self.layers[i].v_cache = 0
                continue
            rows = tr.encoder_dims if blk.attn_func == 6 else tr.n_ctx
            k = t.zeros(n, rows, self.S, dtype=t.float32, device=self.dev)
            v = t.zeros(n, rows, self.S, dtype=t.float32, device=self.dev)
            self.caches.append((k, v))
            self.layers[i].k_cache, self.layers[i].v_cache = k.data_ptr(), v.data_ptr()
        self.cache_n = n

    def reset(self):
        self.pos = 0
        self.caches = None
        self.cache_n = 0

    def run(self, x, encoder_kv, p0, record=None, first=0, count=None):
        """x: [n, P, width] fp32 CUDA (a new tensor is returned); positions [p0, p0 + P).  `record`: None or a list of
        layer indices whose attention weights are returned as {layer: [n, heads, P, keys]}.  first / count: the layers
        run, [first, first + count) (default: all); jk_f32_forward reads no absolute layer index, so a stretch of the
        stack is a pointer into the layer table and a smaller depth."""
        count = self.depth - first if count is None else count
        assert 0 <= first and 1 <= count and first + count <= self.depth
        tr = self.tr
        n, P, W = x.shape
        assert W == self.W
        if self.caches is None or self.cache_n != n:
            assert p0 == 0, "K/V caches of another batch size: call del_cache() first"
            self._alloc_caches(n)
        has6 = any(b.attn_func == 6 for b in tr._attn_mods)
        if has6 and p0 == 0:
            assert encoder_kv is not None and encoder_kv.shape == (n, tr.encoder_dims, W), \
                f"encoder_kv {None if encoder_kv is None else tuple(encoder_kv.shape)}, expected {(n, tr.encoder_dims, W)}"
            encoder_kv = encoder_kv.float().contiguous()
        else:
            encoder_kv = None
        out = x.float().contiguous().clone()
        ws = {}
        for i in range(self.depth):
            self.layers[i].attn_w = 0
        for i in (record or []):
            rows = tr.encoder_dims if tr._attn_mods[i].attn_func == 6 else tr.n_ctx
            ws[i] = t.empty(n, tr.n_head, P, rows, dtype=t.float32, device=self.dev)
            self.layers[i].attn_w = ws[i].data_ptr()
        a = _lib.F32Args(n=n, P=P, p0=p0, width=W, n_state=self.S, mlp_width=self.M, heads=tr.n_head, n_ctx=tr.n_ctx,
                         blocks=tr.blocks or 0, prime_len=tr.prime_len or 0, encoder_dims=tr.encoder_dims or 0,
                         depth=count, x=out.data_ptr(), encoder_kv=_lib.ptr(encoder_kv).value or 0, work=0)
        if not has6:
            a.encoder_dims = 0
        need = C.c_size_t(0)
        _lib.check(_lib.lib().jk_f32_workspace_floats(C.byref(a), C.byref(need)))
        if self.work is None or self.work.numel() < need.value:
            self.work = t.empty(need.value, dtype=t.float32, device=self.dev)
        a.work = self.work.data_ptr()
        table = C.cast(C.addressof(self.layers) + first * C.sizeof(_lib.F32Layer), C.POINTER(_lib.F32Layer))
        _lib.check(_lib.lib().jk_f32_forward(C.byref(a), table, _lib.stream_ptr()))
        return out, ws

    def run_saving(self, x, encoder_kv, first=0):
        """forward mode over a whole window x [n, n_ctx, width], one layer at a time from layer `first` on, keeping each
        of those layers' input (n * n_ctx * width floats per layer; the layers below `first` run in one call).
        Returns (output of the last layer, [input of layer first, ..., input of layer depth-1]) for backward."""
        n, P, _ = x.shape
        assert P == self.tr.n_ctx, f"whole windows of {self.tr.n_ctx} positions, got {P}"
        assert 0 <= first < self.depth
        self.reset()
        self._alloc_caches(n)
        saved = []
        try:
            h = x.float().contiguous()
            if first > 0:
                h, _ = self.run(h, encoder_kv, 0, first=0, count=first)
            for l in range(first, self.depth):
                saved.append(h)
                h, _ = self.run(h, encoder_kv, 0, first=l, count=1)
        finally:
            self.reset()
        return h, saved

    def backward(self, saved, dy, encoder_kv, first=0):
        """jk_f32_backward over layers depth-1 .. first: dy = dL/d(stack output) [n, n_ctx, width]; saved = run_saving's
        inputs of those layers.  Adds into p.grad (fp32, created when None) of every parameter of those layers with
        requires_grad; the others are frozen (NULL).  Returns dL/d(input of layer first)."""
        tr = self.tr
        n, P, W = dy.shape
        count = self.depth - first
        assert len(saved) == count and P == tr.n_ctx and W == self.W
        grads = (_lib.F32GradLayer * count)()
        for i in range(count):
            for name, p in layer_params(tr._attn_mods[first + i]):
                if p.requires_grad:
                    setattr(grads[i], name, grad_buffer(p).data_ptr())
        has6 = any(b.attn_func == 6 for b in tr._attn_mods[first:])
        if has6:
            assert encoder_kv is not None and encoder_kv.shape == (n, tr.encoder_dims, W)
            encoder_kv = encoder_kv.float().contiguous()
        else:
            encoder_kv = None
        a = _lib.F32Args(n=n, P=P, p0=0, width=W, n_state=self.S, mlp_width=self.M, heads=tr.n_head, n_ctx=tr.n_ctx,
                         blocks=tr.blocks or 0, prime_len=tr.prime_len or 0,
                         encoder_dims=(tr.encoder_dims or 0) if has6 else 0, depth=count, x=0,
                         encoder_kv=_lib.ptr(encoder_kv).value or 0, work=0)
        need = C.c_size_t(0)
        _lib.check(_lib.lib().jk_f32_backward_workspace_floats(C.byref(a), C.byref(need)))
        work = t.empty(need.value, dtype=t.float32, device=self.dev)
        a.work = work.data_ptr()
        ins = (C.c_void_p * count)(*[_lib.ptr(s).value for s in saved])
        dx = dy.float().contiguous().clone()
        table = C.cast(C.addressof(self.layers) + first * C.sizeof(_lib.F32Layer), C.POINTER(_lib.F32Layer))
        _lib.check(_lib.lib().jk_f32_backward(C.byref(a), table, grads, ins, _lib.ptr(dx), None, _lib.stream_ptr()))
        return dx

    def run_layers(self, x, encoder_kv, layers):
        """forward mode over positions [0, P) of x [n, P, width], stopped after the deepest of `layers`: returns
        {layer: [n, P, width] fp32 output of that layer}.  Each stretch between two of them is one jk_f32_forward call;
        caches are made for the layers that run only, and dropped afterwards."""
        layers = sorted(set(int(l) for l in layers))
        assert layers and 0 <= layers[0] and layers[-1] < self.depth, f"layers {layers} outside [0, {self.depth})"
        self.reset()
        self._alloc_caches(x.shape[0], upto=layers[-1] + 1)
        outs, h, first = {}, x, 0
        try:
            for l in layers:
                h, _ = self.run(h, encoder_kv, 0, first=first, count=l + 1 - first)
                outs[l] = h
                first = l + 1
        finally:
            self.reset()
        return outs


def embed(ca, tokens, y_cond, x_cond, n, P, p0):
    """[n, P, width] fp32 input rows of positions [p0, p0 + P) (csrc/f32_path.cu jk_f32_embed)."""
    dev = ca.x_emb.weight.device
    x = t.empty(n, P, ca.width, dtype=t.float32, device=dev)
    start = None if ca.y_cond else ca.start_token.detach().float().contiguous().view(-1)
    x_emb = ca.x_emb.weight.detach().float().contiguous()
    pos = ca.pos_emb.pos_emb.detach().float().contiguous()
    _lib.check(_lib.lib().jk_f32_embed(
        _lib.ptr(x), _lib.ptr(tokens), tokens.shape[1] if tokens is not None else 0, _lib.ptr(y_cond), _lib.ptr(x_cond),
        0 if x_cond is None else x_cond.shape[1], _lib.ptr(x_emb), _lib.ptr(pos), _lib.ptr(start), n, P, p0, ca.width,
        _lib.stream_ptr()))
    return x


def linear_nk(x, w):
    """x [M, K] . w[N, K]^T in fp32 (x_out, prior/autoregressive.py:86)"""
    M, K = x.shape
    N = w.shape[0]
    w = w.detach().float().contiguous()
    y = t.empty(M, N, dtype=t.float32, device=x.device)
    _lib.check(_lib.lib().jk_f32_linear(_lib.ptr(x.contiguous()), _lib.ptr(w), None, _lib.ptr(y), M, N, K, 1, _lib.stream_ptr()))
    return y


def linear_wgrad(x, dy, dw=None, db=None):
    """dw[K, N] += x[M, K]^T . dy[M, N], db[N] += sum_m dy[m] (jk_f32_linear_wgrad); dw / db are fp32 .grad buffers"""
    M, K = x.shape
    N = dy.shape[1]
    _lib.check(_lib.lib().jk_f32_linear_wgrad(_lib.ptr(x.contiguous()), _lib.ptr(dy.contiguous()), _lib.ptr(dw), _lib.ptr(db),
                                              M, K, N, 1, _lib.stream_ptr()))


def xent_backward(logits, targets, row_weight):
    """per-row cross-entropy (nats) of logits [M, bins] at targets [M]; logits become d(sum_m w_m loss_m)/dlogits"""
    M, bins = logits.shape
    loss = t.empty(M, dtype=t.float32, device=logits.device)
    _lib.check(_lib.lib().jk_f32_xent_backward(_lib.ptr(logits), _lib.ptr(targets.contiguous()),
                                               _lib.ptr(row_weight.float().contiguous()), _lib.ptr(loss), M, bins,
                                               _lib.stream_ptr()))
    return loss


def embed_backward(ca, tokens, dh, d_x_emb=None):
    """gradients of embed's tables (whole windows, p0 = 0) from dh = dL/dx [n, P, width], added into the .grad of those
    of x_emb, pos_emb and start_token that require grad (x_emb's into d_x_emb instead when given)"""
    n, P, W = dh.shape
    pick = lambda p: grad_buffer(p) if p is not None and p.requires_grad else None
    g_emb = d_x_emb if d_x_emb is not None else pick(ca.x_emb.weight)
    g_pos = pick(ca.pos_emb.pos_emb)
    g_start = None if ca.y_cond else pick(ca.start_token)
    if g_emb is None and g_pos is None and g_start is None:
        return
    work = t.empty(2 * n * max(P - 1, 1), dtype=t.int32, device=dh.device) if g_emb is not None else None
    _lib.check(_lib.lib().jk_f32_embed_backward(
        _lib.ptr(dh.contiguous()), _lib.ptr(tokens), tokens.shape[1], n, P, W, ca.x_emb.weight.shape[0], _lib.ptr(g_emb),
        _lib.ptr(g_pos), _lib.ptr(g_start), _lib.ptr(work), 1, _lib.stream_ptr()))


def linear_kn(x, w, b=None):
    """x [M, K] . w[K, N] + b in fp32 (Conv1D, transformer/ops.py:83-101)"""
    M, K = x.shape
    N = w.shape[1]
    w = w.detach().float().contiguous()
    b = None if b is None else b.detach().float().contiguous()
    y = t.empty(M, N, dtype=t.float32, device=x.device)
    _lib.check(_lib.lib().jk_f32_linear(_lib.ptr(x.float().contiguous()), _lib.ptr(w), _lib.ptr(b), _lib.ptr(y), M, N, K, 0,
                                        _lib.stream_ptr()))
    return y
