"""The C ABI is bound with ctypes: every struct of include/jkb200.h must have the size and field offsets of its ctypes
mirror in jukebox_b200/_lib.py.  The header is compiled as plain C with gcc (it is the contract a reference-side binding
would compile against) into a program that prints sizeof / offsetof of every field."""
import ctypes as C
import os
import re
import shutil
import subprocess
import tempfile

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PAIRS = {"jk_prior_config": "PriorConfig", "jk_layer_weights": "LayerWeights", "jk_prior_plan_info": "PlanInfo",
         "jk_step_args": "StepArgs", "jk_prefill_args": "PrefillArgs", "jk_conv_args": "ConvArgs",
         "jk_f32_layer": "F32Layer", "jk_f32_args": "F32Args", "jk_prefill_attn_args": "PrefillAttnArgs",
         "jk_prefill_attn_route": "PrefillAttnRoute"}


def _fields(header, name):
    body = re.search(r"typedef struct %s \{(.*?)\} %s;" % (name, name), header, re.S).group(1)
    body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
    out = []
    for decl in body.split(";"):
        decl = decl.strip()
        if not decl:
            continue
        for part in decl.split(","):
            m = re.search(r"(\w+)\s*(\[[^\]]*\])?\s*$", part.strip())
            out.append(m.group(1))
    return out


@pytest.mark.skipif(shutil.which("gcc") is None, reason="needs gcc")
def test_ctypes_mirrors_match_the_header():
    from jukebox_b200 import _lib
    header = open(os.path.join(ROOT, "include", "jkb200.h")).read()
    lines = ['#include <stdio.h>', '#include <stddef.h>', '#include "jkb200.h"', "int main(void) {"]
    for cname in PAIRS:
        lines.append('printf("%s size %%zu\\n", sizeof(%s));' % (cname, cname))
        for f in _fields(header, cname):
            lines.append('printf("%s %s %%zu\\n", offsetof(%s, %s));' % (cname, f, cname, f))
    lines += ["return 0;", "}"]
    with tempfile.TemporaryDirectory() as d:
        src, exe = os.path.join(d, "abi.c"), os.path.join(d, "abi")
        open(src, "w").write("\n".join(lines))
        subprocess.run(["gcc", "-std=c99", "-I", os.path.join(ROOT, "include"), src, "-o", exe], check=True)
        out = subprocess.run([exe], capture_output=True, text=True, check=True).stdout
    want = {}
    for line in out.splitlines():
        s, f, v = line.split()
        want.setdefault(s, {})[f] = int(v)
    for cname, pyname in PAIRS.items():
        cls = getattr(_lib, pyname)
        assert C.sizeof(cls) == want[cname]["size"], f"{cname}: ctypes {C.sizeof(cls)} bytes, C {want[cname]['size']}"
        cfields = [f for f in want[cname] if f != "size"]
        alias = {"inp": "in"}              # `in` is a Python keyword
        pyfields = [f[0] for f in cls._fields_]
        assert [alias.get(f, f) for f in pyfields] == cfields, f"{cname}: field order / names differ: {pyfields} vs {cfields}"
        for pf in pyfields:
            cf = alias.get(pf, pf)
            assert getattr(cls, pf).offset == want[cname][cf], f"{cname}.{cf}: ctypes offset {getattr(cls, pf).offset}, C {want[cname][cf]}"
