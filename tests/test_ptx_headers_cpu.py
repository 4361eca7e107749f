"""Inline PTX lives in two headers only: sm90_ptx.cuh (wgmma, mma.sync, cp.async, fences, single instructions) and
tma_bulk.cuh (TMA bulk copies and mbarriers).  A kernel that needs an instruction calls the wrapper there, so each
instruction form is written once, under one name."""
import os
import re

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "gps-gaussian_b200", "csrc")
PTX_HEADERS = {"sm90_ptx.cuh", "tma_bulk.cuh"}
ASM = re.compile(r"\b(?:asm|__asm|__asm__)\b")


def test_inline_ptx_only_in_the_ptx_headers():
    sources = sorted(f for f in os.listdir(CSRC) if f.endswith((".cu", ".cuh", ".h")))
    assert PTX_HEADERS <= set(sources)
    offenders = []
    for name in sources:
        if name in PTX_HEADERS:
            continue
        with open(os.path.join(CSRC, name)) as f:
            offenders += [f"{name}:{i}" for i, line in enumerate(f, 1) if ASM.search(line)]
    assert not offenders, "inline PTX outside sm90_ptx.cuh / tma_bulk.cuh: " + ", ".join(offenders)
