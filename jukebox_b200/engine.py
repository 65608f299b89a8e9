"""DecodeEngine - Python handle on the persistent decode kernel (C ABI: jk_prior_*).

Owns the arena (one torch uint8 CUDA tensor: packed weight streams, KV caches, activations)
and keeps every tensor whose address was handed to the library alive.
"""
import ctypes as C
from collections import namedtuple

import torch

from . import _lib
from ._lib import lib, check, ptr, stream_ptr


# one entry of DecodeEngine.prefill(capture=...): out receives the layer's fp32 rows of positions [t0, t1) (pool False:
# [n, t1 - t0, width]) or their mean (pool True: [n, width]), x_cond added first when add_x_cond (jk_act_capture)
Capture = namedtuple("Capture", "out t0 t1 pool add_x_cond")


def prior_config(*, width, depth, heads, n_state, mlp_width, n_ctx, blocks, attn_funcs, bins=0, prime_len=0,
                 encoder_dims=0, max_batch=16, add_cond_after=True):
    """the jk_prior_config of an engine (include/jkb200.h)"""
    cfg = _lib.PriorConfig()
    cfg.width, cfg.depth, cfg.heads, cfg.n_state, cfg.mlp_width = width, depth, heads, n_state, mlp_width
    cfg.n_ctx, cfg.blocks, cfg.bins = n_ctx, blocks or 0, bins
    cfg.prime_len, cfg.encoder_dims = prime_len or 0, encoder_dims or 0
    cfg.max_batch, cfg.add_cond_after = max_batch, int(bool(add_cond_after))
    assert len(attn_funcs) == depth <= _lib.JK_MAX_DEPTH
    for i, f in enumerate(attn_funcs):
        cfg.attn_func[i] = f
    return cfg


def config_prefill_capacity(device, **kw):
    """positions one prefill call of an engine built with DecodeEngine(**kw) could take, without building it; 0 when
    that configuration has no prefill or cannot make an engine at all (jk_prior_config_prefill_capacity)"""
    if kw.get("max_batch", 16) > _lib.JK_MAX_BATCH:
        return 0
    out = C.c_int(0)
    with torch.cuda.device(device):
        rc = lib().jk_prior_config_prefill_capacity(C.byref(prior_config(**kw)), C.byref(out))
    return out.value if rc == 0 else 0


def _parents(parents):
    """parents (a sequence or 1-D tensor of ints) as a C int32 array and its length"""
    if isinstance(parents, torch.Tensor):
        if parents.dim() != 1 or parents.dtype.is_floating_point or parents.dtype == torch.bool:
            raise RuntimeError(f"parents must be a 1-D integer tensor, got {parents.dtype} {tuple(parents.shape)}")
        parents = parents.tolist()
    vals = [int(v) for v in parents]
    if not 1 <= len(vals) <= _lib.JK_MAX_BATCH:
        raise RuntimeError(f"parents of {len(vals)} rows: 1 .. {_lib.JK_MAX_BATCH} rows can be selected")
    return (C.c_int32 * len(vals))(*vals), len(vals)


def select_plan(cfg, parents):
    """the jk_select_plan_info of a selection on an engine of configuration cfg (host arithmetic, no device):
    row b becomes a copy of row parents[b]"""
    arr, n = _parents(parents)
    info = _lib.SelectPlanInfo()
    check(lib().jk_prior_select_plan(C.byref(cfg), arr, n, C.byref(info)))
    return info


class DecodeEngine:
    def __init__(self, *, width, depth, heads, n_state, mlp_width, n_ctx, blocks, attn_funcs,
                 bins=0, prime_len=0, encoder_dims=0, max_batch=16, add_cond_after=True, device=None):
        device = torch.device(device if device is not None else "cuda")
        if device.type != "cuda":
            raise RuntimeError("DecodeEngine needs a CUDA device (jukebox_b200 has no CPU path)")
        if max_batch > _lib.JK_MAX_BATCH:
            raise RuntimeError(f"n_samples {max_batch} > {_lib.JK_MAX_BATCH} (the decode kernel's largest row count): "
                               "split the batch (sample.py does, via max_batch_size)")
        self.device = device
        cfg = prior_config(width=width, depth=depth, heads=heads, n_state=n_state, mlp_width=mlp_width, n_ctx=n_ctx,
                           blocks=blocks, attn_funcs=attn_funcs, bins=bins, prime_len=prime_len,
                           encoder_dims=encoder_dims, max_batch=max_batch, add_cond_after=add_cond_after)
        self.cfg = cfg
        self.max_batch = max_batch
        with torch.cuda.device(device):
            nbytes = C.c_size_t(0)
            check(lib().jk_prior_arena_bytes(C.byref(cfg), C.byref(nbytes)))
            self.arena = torch.empty(nbytes.value + 256, dtype=torch.uint8, device=device)
            base = (self.arena.data_ptr() + 255) // 256 * 256
            handle = C.c_void_p(0)
            check(lib().jk_prior_create(C.byref(cfg), C.c_void_p(base), C.c_size_t(nbytes.value),
                                        C.byref(handle), stream_ptr()))
        self.handle = handle
        self.arena_bytes = nbytes.value
        self._keep = {}
        self.position = 0

    def __del__(self):
        try:
            if getattr(self, "handle", None):
                lib().jk_prior_destroy(self.handle)
                self.handle = None
        except Exception:
            pass

    # ---- weights -------------------------------------------------------------------------
    def load_layer(self, layer, block):
        """block: a ResAttnBlock (parameter container with the reference's names)."""
        at, mlp = block.attn, block.mlp
        ws = [at.c_attn.w, at.c_proj.w, mlp.c_fc.w, mlp.c_proj.w]
        if at.attn_func == 6:
            ws.append(at.c_enc_kv.w)
        dts = {w.dtype for w in ws}
        if len(dts) != 1 or next(iter(dts)) not in (torch.float32, torch.float16):
            raise RuntimeError(f"Conv1D weights must be uniformly fp32 or fp16, got {dts}")
        bs = [at.c_attn.b, at.c_proj.b, mlp.c_fc.b, mlp.c_proj.b]
        bdt = {b.dtype for b in bs}
        if len(bdt) != 1:
            raise RuntimeError(f"mixed bias dtypes {bdt}")
        lw = _lib.LayerWeights()
        c = lambda t: ptr(t.detach().contiguous())
        tensors = dict(c_attn_w=at.c_attn.w, c_attn_b=at.c_attn.b, c_proj_w=at.c_proj.w, c_proj_b=at.c_proj.b,
                       fc_w=mlp.c_fc.w, fc_b=mlp.c_fc.b, proj2_w=mlp.c_proj.w, proj2_b=mlp.c_proj.b,
                       ln0_g=block.ln_0.weight.float(), ln0_b=block.ln_0.bias.float(),
                       ln1_g=block.ln_1.weight.float(), ln1_b=block.ln_1.bias.float())
        if at.attn_func == 6:
            tensors.update(c_enc_kv_w=at.c_enc_kv.w, c_enc_kv_b=at.c_enc_kv.b)
        keep = []
        for k, v in tensors.items():
            v = v.detach().contiguous()
            keep.append(v)
            setattr(lw, k, ptr(v))
        lw.w_dtype = 1 if next(iter(dts)) == torch.float16 else 0
        lw.b_dtype = 1 if next(iter(bdt)) == torch.float16 else 0
        with torch.cuda.device(self.device):
            check(lib().jk_prior_load_layer(self.handle, layer, C.byref(lw), stream_ptr()))
        # packing kernels read `keep` asynchronously on the current stream; torch's allocator is
        # stream-ordered, so dropping the references here is safe.
        del keep

    def set_embeddings(self, x_emb=None, pos_emb=None, x_out=None, start_token=None):
        ts = {}
        for name, t in (("x_emb", x_emb), ("pos_emb", pos_emb), ("x_out", x_out), ("start_token", start_token)):
            if t is not None:
                t = t.detach()
                if t.dtype != torch.float32:
                    raise RuntimeError(f"{name} must be fp32 (got {t.dtype})")
                t = t.contiguous()
            ts[name] = t
        self._keep["emb"] = ts
        check(lib().jk_prior_set_embeddings(self.handle, ptr(ts["x_emb"]), ptr(ts["pos_emb"]),
                                            ptr(ts["x_out"]), ptr(ts["start_token"])))

    # ---- per window ----------------------------------------------------------------------
    def reset(self, t0=0):
        with torch.cuda.device(self.device):
            check(lib().jk_prior_reset(self.handle, int(t0), stream_ptr()))
        self.position = int(t0)

    def set_encoder_kv(self, encoder_kv):
        enc = encoder_kv.detach().float().contiguous()
        self._keep["enc"] = enc
        with torch.cuda.device(self.device):
            check(lib().jk_prior_set_encoder_kv(self.handle, ptr(enc), enc.shape[0], stream_ptr()))

    # ---- chunked prefill ---------------------------------------------------------------
    @property
    def has_logits_gemm(self):
        """True if the logits run as a Conv1D on the tensor cores (then `step(logit_bias=...)` is worth computing)"""
        out = C.c_int(0)
        check(lib().jk_prior_has_logits_gemm(self.handle, C.byref(out)))
        return bool(out.value)

    @property
    def prefill_capacity(self):
        """positions one `prefill` call can take (0: this configuration steps its given tokens)"""
        out = C.c_int(0)
        check(lib().jk_prior_prefill_capacity(self.handle, C.byref(out)))
        return out.value

    def prefill(self, n, n_positions, *, tokens=None, y_cond=None, x_cond=None, h_out=None, record=None, n_layers=0,
                capture=None):
        """positions t0..t0+n_positions-1 of the first n rows through every layer at once (wgmma GEMMs), where t0 is the
        engine's position; afterwards the engine is at t0 + n_positions, as after that many steps.  At t0 = 0 this is
        the head of a window; at t0 > 0 a continuation on top of the rows' K / V caches (after steps, a prefill or a
        select): tokens is then the window's token tensor (position t reads tokens[:, t - 1]), x_cond and h_out are as
        at the head (x_cond indexed by absolute position, h_out row i is position t0 + i), y_cond is not read, and
        record, capture and a truncating n_layers are errors (jk_prefill_args in include/jkb200.h).

        record: {layer: w} - fp16 CUDA tensors [n, heads, n_positions, ld] that receive the layer's normalised attention
        weights (keys by absolute position, or encoder row for an encoder-decoder layer; keys >= ld are dropped; zeros
        outside the layer's pattern).  See jk_attn_record in include/jkb200.h.
        n_layers: 0 runs every layer; 1 <= n_layers < depth stops after layer n_layers - 1, and the engine (position -1)
        must be reset before it steps or prefills again.
        capture: {layer: Capture(out, t0, t1, pool, add_x_cond)} - the layer's activations (jk_act_capture)."""
        a = _lib.PrefillArgs()
        a.n_samples, a.n_positions = n, n_positions
        a.tokens = ptr(tokens)
        a.tok_stride = tokens.stride(0) if tokens is not None else 0
        a.y_cond = ptr(y_cond)
        a.x_cond = ptr(x_cond)
        a.x_cond_len = x_cond.shape[1] if x_cond is not None else 1
        a.h_out = ptr(h_out)
        if record:
            table = (_lib.AttnRecord * len(record))()
            for e, (layer, w) in zip(table, record.items()):
                if (w.dtype != torch.float16 or w.dim() != 4 or tuple(w.shape[:3]) != (n, self.cfg.heads, n_positions)
                        or w.device != self.device or not w.is_contiguous()):
                    raise RuntimeError(f"record[{layer}]: need a contiguous fp16 tensor [{n}, {self.cfg.heads}, "
                                       f"{n_positions}, ld] on {self.device}, got {w.dtype} {tuple(w.shape)} on {w.device}"
                                       f"{'' if w.is_contiguous() else ' (strided)'}")
                e.layer, e.ld, e.w = int(layer), w.shape[3], ptr(w)
            a.record, a.n_record = table, len(record)
        if capture:
            table = (_lib.ActCapture * len(capture))()
            for e, (layer, k) in zip(table, capture.items()):
                k = Capture(*k)
                want = (n, self.cfg.width) if k.pool else (n, k.t1 - k.t0, self.cfg.width)
                out = k.out
                if (out.dtype != torch.float32 or tuple(out.shape) != want or out.device != self.device
                        or not out.is_contiguous()):
                    raise RuntimeError(f"capture[{layer}]: need a contiguous fp32 tensor {list(want)} on {self.device}, "
                                       f"got {out.dtype} {tuple(out.shape)} on {out.device}"
                                       f"{'' if out.is_contiguous() else ' (strided)'}")
                e.layer, e.t0, e.t1 = int(layer), int(k.t0), int(k.t1)
                e.pool, e.add_x_cond, e.out = int(bool(k.pool)), int(bool(k.add_x_cond)), ptr(out)
            a.capture, a.n_capture = table, len(capture)
        a.n_layers = int(n_layers)
        with torch.cuda.device(self.device):
            check(lib().jk_prior_prefill(self.handle, C.byref(a), stream_ptr()))
        self.position = -1 if 0 < n_layers < self.cfg.depth else self.position + n_positions

    # ---- one token -----------------------------------------------------------------------
    def step(self, n, *, x_in=None, tokens=None, y_cond=None, x_cond=None, h_out=None, logits=None,
             logits_tstride=0, logit_bias=None):
        a = _lib.StepArgs()
        a.n_samples = n
        a.x_in = ptr(x_in)
        a.tokens = ptr(tokens)
        a.tok_stride = tokens.stride(0) if tokens is not None else 0
        a.y_cond = ptr(y_cond)
        a.x_cond = ptr(x_cond)
        a.x_cond_len = x_cond.shape[1] if x_cond is not None else 1
        a.h_out = ptr(h_out)
        a.logits = ptr(logits)
        if logits is not None:
            a.logits_bstride = logits.stride(0)
            a.logits_tstride = logits_tstride
        a.logit_bias = ptr(logit_bias)
        if logit_bias is not None:        # [n, 1 or n_ctx, bins] fp32: x_cond . x_out^T of every position (jkb200.h)
            a.logit_bias_bstride = logit_bias.stride(0)
            a.logit_bias_tstride = logit_bias.stride(1) if logit_bias.shape[1] > 1 else 0
        with torch.cuda.device(self.device):
            check(lib().jk_prior_step(self.handle, C.byref(a), stream_ptr()))
        self.position += 1

    # ---- sample selection ----------------------------------------------------------------
    def select_plan(self, parents):
        """what select(parents) would copy (jk_select_plan_info): rows it stashes, workspace and bytes moved"""
        return select_plan(self.cfg, parents)

    def select(self, parents):
        """row b of every layer's K / V cache becomes a copy of row parents[b], b < len(parents) (jk_prior_select):
        the histories of the rows are reordered, the position stays.  A workspace is allocated only when the selection
        overwrites a row that another row still reads (jk_select_plan_info.n_stash)."""
        arr, n = _parents(parents)
        info = select_plan(self.cfg, parents)
        ws = None
        if info.workspace_bytes:
            ws = torch.empty(info.workspace_bytes, dtype=torch.uint8, device=self.device)
        with torch.cuda.device(self.device):
            check(lib().jk_prior_select(self.handle, arr, n, ptr(ws), C.c_size_t(info.workspace_bytes), stream_ptr()))
        # the copies read `ws` on the current stream; torch's allocator is stream-ordered, so it may be released here
        return info

    def debug_buffer(self, which):
        p, n = C.c_void_p(0), C.c_size_t(0)
        check(lib().jk_prior_debug_buffer(self.handle, which, C.byref(p), C.byref(n)))
        off = p.value - self.arena.data_ptr()
        return self.arena[off: off + 2 * n.value].view(torch.float16)
