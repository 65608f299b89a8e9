"""Per-layer outputs of the numpy transformer oracle (representations, JukeMIR's recipe).

Layer L's output is the output of the stack cut after layer L: TransformerOracle built with n_depth = L + 1 on the same
weights, which is what the reference computes for a prior built with prior_depth=L+1 and restored non-strictly.  The
attention pattern of a layer depends on its index only (transformer.py:110-124), so the cut stack is the full stack's
prefix.  (res_scale=True would scale by 1/depth and change with the cut; no named model uses it.)"""
import numpy as np

from oracle.transformer_np import TransformerOracle


def layer_outputs(sd, n_in, n_ctx, n_head, attn_order, blocks, encoder_dims, prime_len, layers, x, encoder_kv=None,
                  fp16=False, mode="full"):
    """{layer: fp32 output of that layer} for x [bs, n_ctx, n_in]: forward mode (mode "full", forward_full) or token by
    token (mode "step", [bs, n_ctx, n_in] from n_ctx steps)."""
    out = {}
    for L in sorted(set(int(l) for l in layers)):
        orc = TransformerOracle(sd, n_in, n_ctx, n_head, L + 1, attn_order, blocks, encoder_dims, prime_len)
        if mode == "full":
            out[L] = orc.forward_full(x, encoder_kv, fp16)
        else:
            out[L] = np.stack([orc.step(x[:, i], encoder_kv, fp16) for i in range(x.shape[1])], 1)
    return out
