"""Golden vectors of the reference's window loop (jukebox/sample.py:17-96, `sample_level`), driven on CPU with a
recording dummy prior.  TEST INFRASTRUCTURE: tests/test_sample_plan_cpu.py replays the same cases through
jukebox_b200.sample and compares with what this script stored.

    python oracle/make_golden_sample_plan.py          # needs the reference tree (oracle/ref_import.py)

writes tests/golden/sample_level.json: per case, either the stitched codes and the list of prior.sample calls, or
the type of the exception the reference raised.
"""
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OUT = os.path.join(ROOT, "tests", "golden", "sample_level.json")


class RecordingPrior:
    """prior.sample appends tokens that encode (call index, position), and records how it was called"""

    def __init__(self, n_ctx):
        self.n_ctx = n_ctx
        self.calls = []

    def get_z_conds(self, zs, start, end):
        return None

    def get_y(self, labels, start):
        return None

    def sample(self, n_samples, z=None, z_conds=None, y=None, sample_tokens=None, **kw):
        total = self.n_ctx if sample_tokens is None else sample_tokens
        self.calls.append([n_samples, z.shape[1], total, sorted(kw)])
        new = total - z.shape[1]
        assert new > 0
        fresh = 1000 * len(self.calls) + torch.arange(z.shape[1], total).view(1, -1).repeat(n_samples, 1)
        return torch.cat([z, fresh], dim=1)


class Hps(dict):
    __getattr__ = dict.__getitem__


CASES = [(total, n_ctx, hop, have, bs, mbs)
         for total, n_ctx, hop in [(40, 16, 8), (40, 16, 4), (16, 16, 8), (37, 16, 12), (10, 16, 8), (5, 16, 8), (33, 16, 16)]
         for have in (0, 3, 11, 16, 20) for bs, mbs in ((3, 2), (4, 4))]


def case_key(case):
    return ",".join(str(v) for v in case)


def run_case(sample_level, case):
    """sample_level of one module on one case -> {"codes": [[...]], "calls": [...]} or {"error": exception type}"""
    total, n_ctx, hop, have, bs, mbs = case
    prior = RecordingPrior(n_ctx)
    zs = [torch.arange(have).view(1, -1).repeat(bs, 1)]
    kw = dict(temp=0.9, fp16=True, max_batch_size=mbs)
    try:
        zs = sample_level(zs, None, kw, 0, prior, total, hop, Hps(n_samples=bs))
    except Exception as e:          # both sides must fail alike (e.g. negative slices)
        return dict(error=type(e).__name__)
    return dict(codes=zs[0].tolist(), calls=prior.calls)


def main():
    sys.path.insert(0, ROOT)
    from oracle.ref_import import load_reference
    load_reference()
    import jukebox.sample as ref
    out = {case_key(c): run_case(ref.sample_level, c) for c in CASES}
    with open(OUT, "w") as f:
        json.dump(out, f, separators=(",", ":"))
    print(f"wrote {OUT} ({os.path.getsize(OUT) / 1e3:.1f} kB, {len(out)} cases)")


if __name__ == "__main__":
    main()
