"""Helpers to read tests/golden/*.npz (written by oracle/make_golden.py)."""
import json
import os

import numpy as np

from oracle.synth import synth_state_dict

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


class Fixture:
    def __init__(self, name):
        self.z = np.load(os.path.join(GOLDEN, name + ".npz"), allow_pickle=False)
        self.cfg = json.loads(str(self.z["cfg"]))
        raw = json.loads(str(self.z["names"]))
        self.names = [(n, tuple(s)) for n, s, _ in raw]
        self.aliases = {n: a for n, _, a in raw if a}

    def __getitem__(self, k):
        return self.z[k]

    def __contains__(self, k):
        return k in self.z.files

    def weights(self, prefix=""):
        sd = synth_state_dict(self.names, self.cfg["seed"])
        for alias, target in self.aliases.items():      # tied parameters
            sd[alias] = sd[target]
        if prefix:
            sd = {k[len(prefix):]: v for k, v in sd.items() if k.startswith(prefix)}
        return sd


def logit_cols(fx, a):
    """the stored logit columns of a fixture that keeps a sample of the vocabulary (`pred_cols`), else all of them"""
    return a[..., fx["pred_cols"]] if "pred_cols" in fx else a


def rel_err(a, b):
    """max|a-b| / max|b|  (the metric SURVEY.md section 8d defines for logits)."""
    a = np.asarray(a, np.float64)
    b = np.asarray(b, np.float64)
    return float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-30))
