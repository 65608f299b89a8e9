"""Music representations from a prior's intermediate layers (JukeMIR: Castellon, Donahue & Liang, ISMIR 2021).

audio -> codes of the prior's level (VQ-VAE encoder) -> the prior's stack in forward mode, stopped after the requested
layers -> each layer's output + x_cond, averaged over time -> one vector per clip and layer.  The fp16 route runs the
decode engine's prefill truncated after the deepest layer, with the rows averaged inside it (csrc/prefill.cu,
jk_act_capture), so neither the later layers nor an activation tensor are computed.
"""
import torch as t


def jukemir_labels(prior, n):
    """JukeMIR's label rows: unknown artist and genre, no lyrics, offset 0 - [n, label width] int64, or None for a prior
    without labels"""
    if not prior.y_cond:
        return None
    meta = dict(artist="unknown", genre="unknown", lyrics="", total_length=prior.sample_length, offset=0)
    return prior.labeller.get_batch_labels([meta] * n, "cpu")["y"]


def windows(T, n_ctx):
    """consecutive non-overlapping [start, end) windows of n_ctx codes over T codes; a shorter final window is kept as a
    shorter causal window, except a final window of one code (no prefix to attend), which is dropped"""
    out = [(s, min(s + n_ctx, T)) for s in range(0, T, n_ctx)]
    if len(out) > 1 and out[-1][1] - out[-1][0] < 2:
        out.pop()
    return out


def audio_representations(prior, x, y=None, layers=(36,), fp16=True):
    """Per-clip features of audio x [N, T, 1] (fp32, the VQ-VAE's sample rate) from a top-level prior: {layer: fp32
    [N, width]}, the mean over all the clip's codes of that layer's output + x_cond.

    The codes of prior.level are cut into consecutive windows of n_ctx; each window is pooled on its own
    (SimplePrior.layer_acts) and the windows are combined into one mean over all positions, weighted by window length.
    y: label rows [N, label width] used for every window as given; None builds JukeMIR's row, which is

        y = prior.labeller.get_batch_labels(
                [dict(artist="unknown", genre="unknown", lyrics="", total_length=prior.sample_length, offset=0)] * N,
                "cuda")["y"]

    JukeMIR's recipe is prior_5b (no lyrics), layers=(36,), fp16=True."""
    assert not prior.x_cond, "representations are taken from a top-level prior (no codes of a level above)"
    N = x.shape[0]
    layers = tuple(int(l) for l in layers)
    with t.no_grad():
        z = prior.encode(x, start_level=prior.level, end_level=prior.level + 1, bs_chunks=N)[0]
        if y is None:
            y = jukemir_labels(prior, N)
        if y is not None:
            y = y.to(z.device)
        sums = {l: t.zeros(N, prior.prior.width, dtype=t.float64, device=z.device) for l in layers}
        total = 0
        for s, e in windows(z.shape[1], prior.n_ctx):
            acts = prior.layer_acts(z[:, s:e].contiguous(), [], y, layers=layers, fp16=fp16, pool=True)
            for l in layers:
                sums[l] += acts[l].double() * (e - s)
            total += e - s
        return {l: (sums[l] / total).float() for l in layers}
