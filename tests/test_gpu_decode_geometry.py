"""The decode step (csrc/decode_engine.cu, jk_prior_step) at the priors' real geometry.

The tiny golden fixtures stop at width 192 and 96 positions; the full-size golden stacks compare a whole stack at a few
positions with a tolerance that a one-ulp error at one split or tile edge cannot move.  This file looks at one or two
layers of a DecodeEngine built at the 1b_lyrics, 5b_lyrics and upsampler shapes (oracle.synth weights, bins = 0, x_in
fed, h_out read).

a. LayerNorm probe layers, bit for bit.  The weights make everything but one LayerNorm exact: at position 0 the only
   key is the token itself, so softmax is exactly 1 and P.V = v; c_attn's V columns select n_state of the LN0 outputs
   and c_proj puts them back (the transposed selection); the MLP is zero.  So h_out = fp16(x + LN0(x)) on the selected
   columns and x elsewhere, where LN0(x) is the staging of oracle/decode_stats.py: the kernel's own fixed-point row
   statistics restated in integers and its fmaf chain restated exactly.  The selection rotates until every column was
   seen.  The same through the MLP checks LN1 (the proj epilogue's statistics), and a depth-2 engine whose layer 0 is
   zero checks layer 1's LN0 (the proj2 epilogue's statistics); with the input stage's, those are the three producers
   of statistics words.  quick_gelu may differ by one fp16 ulp where its float32 pre-rounding value lies within 2 ulps
   of an fp16 rounding boundary (the device's expf is not numpy's); nothing else may differ.  A row whose LayerNorm
   overflows fp16 (|x| past the clamp of the squares, where the variance can come out 0) is NaN in every column.

Every number is printed, one JSON line per case (pytest -s)."""
import json
from types import SimpleNamespace as NS

import numpy as np
import pytest
import torch

from jukebox_b200.engine import DecodeEngine
from oracle.decode_stats import quick_gelu16, staged
from oracle.synth import synth_tensor

pytestmark = pytest.mark.gpu

# width, heads, n_state, max batch the plan allows.  1104 / 272: a width that is not a multiple of 64 (69 sixteens:
# K split 1, partial column groups), with an n_state that is not one either (head_dim 272, 32-row attention tiles)
LN_GEOM = {1920: (1, 480, 32), 2048: (2, 512, 32), 4800: (8, 1200, 16), 1104: (1, 272, 32)}
BATCHES = (1, 16, 17, 32)


def record(row):
    print(json.dumps(row))


def probe_rows():
    """the rows the LayerNorm probes normalise, as (label, generator of a row of width W)"""
    rows = [(f"N(0, 2^{2 * e})", lambda W, g, e=e: (2.0 ** e) * torch.randn(W, generator=g)) for e in range(-8, 11)]
    rows += [("1000 + N(0, 1e-4)", lambda W, g: 1000 + 1e-2 * torch.randn(W, generator=g)),
             ("-250 + N(0, 1e-6)", lambda W, g: -250 + 1e-3 * torch.randn(W, generator=g)),
             ("3 + N(0, 2^-16)", lambda W, g: 3 + 2.0 ** -8 * torch.randn(W, generator=g)),
             ("const 0.1", lambda W, g: torch.full((W,), 0.1)),
             ("const 1000", lambda W, g: torch.full((W,), 1000.0)),
             ("const -7", lambda W, g: torch.full((W,), -7.0)),
             ("zero", lambda W, g: torch.zeros(W)),
             ("N(0, 3000^2)", lambda W, g: (3000 * torch.randn(W, generator=g)).clamp(-60000, 60000)),
             ("5000 + N(0, 100^2)", lambda W, g: 5000 + 100 * torch.randn(W, generator=g)),
             ("+-20000 alternating", lambda W, g: 20000.0 * (1 - 2 * (torch.arange(W) % 2)).float())]
    return rows


def row_batches(W, n, seed):
    """every probe row, in batches of n rows (the last batch topped up with N(0, 1) rows): [(labels, x [n, W] fp32)]"""
    g = torch.Generator().manual_seed(seed)
    rows = probe_rows()
    out = []
    for i in range(0, len(rows), n):
        chunk = rows[i:i + n]
        xs = [f(W, g) for _, f in chunk] + [torch.randn(W, generator=g) for _ in range(n - len(chunk))]
        out.append(([lab for lab, _ in chunk], torch.stack(xs).float()))
    return out


def zero_block(W, S, M, af=0):
    z = lambda *s: torch.zeros(*s)
    blk = NS(attn=NS(attn_func=af, c_attn=NS(w=z(W, 3 * S), b=z(3 * S)), c_proj=NS(w=z(S, W), b=z(W))),
             mlp=NS(c_fc=NS(w=z(W, M), b=z(M)), c_proj=NS(w=z(M, W), b=z(W))),
             ln_0=NS(weight=torch.ones(W), bias=z(W)), ln_1=NS(weight=torch.ones(W), bias=z(W)))
    return blk


def ln_params(W, seed):
    return (torch.from_numpy(synth_tensor("_attn_mods.0.ln_0.weight", (W,), seed)),
            torch.from_numpy(synth_tensor("_attn_mods.0.ln_0.bias", (W,), seed)))


def selection_block(W, S, M, which, cols, gamma, beta):
    """the probe layer of LayerNorm `which` (0 or 1): column j of the selection `cols` goes through the LayerNorm and
    back into the residual stream at column cols[j]"""
    blk = zero_block(W, S, M)
    j = torch.arange(len(cols))
    if which == 0:
        blk.ln_0 = NS(weight=gamma, bias=beta)
        blk.attn.c_attn.w[cols, 2 * S + j] = 1.0
        blk.attn.c_proj.w[j, cols] = 1.0
    else:
        blk.ln_1 = NS(weight=gamma, bias=beta)
        blk.mlp.c_fc.w[cols, j] = 1.0
        blk.mlp.c_proj.w[j, cols] = 1.0
    return blk


def to_cuda(blk):
    for mod in (blk.attn.c_attn, blk.attn.c_proj, blk.mlp.c_fc, blk.mlp.c_proj, blk.ln_0, blk.ln_1):
        for k, v in vars(mod).items():
            setattr(mod, k, v.cuda())
    return blk


def expected(x, which, cols, gamma, beta):
    """h_out of a probe layer (decode_stats restatement) and, for LN1, where quick_gelu may be one fp16 ulp off"""
    h = x.numpy().astype(np.float16)
    ln = staged(h, gamma.numpy(), beta.numpy())
    out = h.copy()
    near = np.zeros(h.shape, bool)
    alt = []
    if which == 0:
        y = ln[:, cols]
    else:
        y, nr = quick_gelu16(ln[:, cols])
        near[:, cols] = nr
        # the neighbours of quick_gelu's result where the device may round the other way
        for d in (-1, 1):
            yy = np.nextafter(y, np.float16(d * np.inf))
            o = out.copy()
            o[:, cols] = (h[:, cols].astype(np.float32) + yy.astype(np.float32)).astype(np.float16)
            alt.append(o)
    out[:, cols] = (h[:, cols].astype(np.float32) + y.astype(np.float32)).astype(np.float16)
    # a row whose LayerNorm overflows fp16 (past the 4096 clamp of the squares the variance can come out 0): inf times
    # the zero weights of the other Conv1D columns is NaN, and NaN reaches every column through c_proj / proj2
    blown = ~np.isfinite(ln).all(-1)
    out[blown] = np.nan
    for a in alt:
        a[blown] = np.nan
    return out.astype(np.float32), near, [a.astype(np.float32) for a in alt]


def run_probe(W, which, depth, batches):
    H, S, mb = LN_GEOM[W]
    M = W
    gamma, beta = ln_params(W, 7 + which)
    eng = DecodeEngine(width=W, depth=depth, heads=H, n_state=S, mlp_width=M, n_ctx=64, blocks=4,
                       attn_funcs=[0] * depth, bins=0, max_batch=mb)
    if depth == 2:
        eng.load_layer(0, to_cuda(zero_block(W, S, M)))
    width_sel = S if which == 0 else min(M, W)
    n_rot = -(-W // width_sel)
    stats = dict(rows=0, steps=0, mismatches=0, gelu_boundary_flips=0, gelu_boundary_elements=0)
    bad = []
    for r in range(n_rot):
        cols = (torch.arange(width_sel) + r * width_sel) % W
        eng.load_layer(depth - 1, to_cuda(selection_block(W, S, M, which, cols, gamma, beta)))
        cols_np = cols.numpy()
        for n in batches:
            if n > mb:
                continue
            for labels, x in row_batches(W, n, seed=1000 * W + 10 * n + r):
                eng.reset(0)
                h = torch.full((n, W), float("nan"), device="cuda")
                eng.step(n, x_in=x.cuda(), h_out=h)
                got = h.cpu().numpy()
                with np.errstate(over="ignore", invalid="ignore"):        # the overflowing row (expected())
                    want, near, alt = expected(x, which, cols_np, gamma, beta)
                same = lambda a, b: (a == b) | (np.isnan(a) & np.isnan(b))
                ok = same(got, want)
                if alt:
                    flip = ~ok & near & (same(got, alt[0]) | same(got, alt[1]))
                    stats["gelu_boundary_flips"] += int(flip.sum())
                    stats["gelu_boundary_elements"] += int(near.sum())
                    ok |= flip
                stats["rows"] += n
                stats["steps"] += 1
                if not ok.all():
                    stats["mismatches"] += int((~ok).sum())
                    i, j = np.argwhere(~ok)[0]
                    bad.append(dict(row=labels[i] if i < len(labels) else "N(0, 1) filler", col=int(j),
                                    got=float(got[i, j]), want=float(want[i, j]), x=float(x[i, j]), batch=n))
    return stats, bad


LN_CASES = [(W, 0, 1) for W in LN_GEOM] + [(W, 1, 1) for W in LN_GEOM] + [(W, 0, 2) for W in LN_GEOM]


@pytest.mark.parametrize("W, which, depth", LN_CASES)
def test_layernorm_probe_bit_exact(W, which, depth):
    producer = {(0, 1): "input stage", (1, 1): "proj epilogue", (0, 2): "proj2 epilogue"}[(which, depth)]
    stats, bad = run_probe(W, which, depth, BATCHES)
    H, S, mb = LN_GEOM[W]
    record(dict(case=f"LN{which} of layer {depth - 1}", width=W, n_state=S, statistics_from=producer,
                batches=[n for n in BATCHES if n <= mb], skipped_batches=[n for n in BATCHES if n > mb],
                **stats, first_mismatches=bad[:5]))
    assert stats["mismatches"] == 0, bad[:5]
