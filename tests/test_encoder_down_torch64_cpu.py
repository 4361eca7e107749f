"""CPU: the fp64 restatement of res2 / res3 (oracle/encoder_down_torch64.py) against the reference's own modules (the
golden file), the CPU emulation of the kernels' arithmetic within every stage bound in both precisions, and each
deliberate error of the emulation (MUTANTS) caught by a stage check."""
import os

import numpy as np
import pytest
import torch

from gps_gaussian_b200 import encoder
from oracle import encoder_down_torch64 as ed

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "encoder_down_golden.npz")


def _golden():
    z = np.load(GOLDEN)
    for name in sorted(k[:-2] for k in z.files if k.endswith("_x")):
        stage = name.split("_")[0]
        ps = [torch.from_numpy(z[f"{name}_p{i}"] if f"{name}_p{i}" in z.files else z[f"{stage}_p{i}"])
              for i in range(20)]
        yield name, torch.from_numpy(z[name + "_x"]), ps, torch.from_numpy(z[name + "_out"])


def test_forward64_is_the_reference():
    names = []
    for name, x, ps, want in _golden():
        got = ed.forward64(x, ps)["out"]
        assert got.shape == want.shape and torch.allclose(got, want, rtol=1e-10, atol=1e-10), name
        names.append(name)
    assert {"res2_9x5", "res2_1x1", "res2_zero_var_group", "res2_offset", "res3_5x3", "res3_1x1"} <= set(names)


def _case(cin, c, B, H, W, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.relu(torch.randn(B, cin, H, W, generator=g))
    ps = [(torch.rand(s, generator=g) * 2 - 1) * (0.1 if len(s) == 4 else 0.5) + (1.0 if i % 4 == 2 else 0.0)
          for i, s in enumerate(encoder.down_param_shapes(cin, c))]
    return x, ps


def _worst(x, ps, mode, mutant=None):
    em = ed.emulate(x, ps, mode, mutant=mutant)
    checks = ed.stage_checks(x, ps, [em[k] for k in ed.KEYS[:5]], mode)
    return max(float(ed.ratio(em[k], w, b)) for k, (w, b) in checks.items())


@pytest.mark.parametrize("mode", ["tf32", "fp16"])
@pytest.mark.parametrize("cin,c", encoder.DOWN_DIMS)
@pytest.mark.parametrize("B,H,W", [(1, 9, 7), (2, 1, 1), (1, 6, 17)])
def test_emulation_within_stage_bounds(cin, c, B, H, W, mode):
    x, ps = _case(cin, c, B, H, W, H * W + cin)
    assert _worst(x, ps, mode) <= 1.0


@pytest.mark.parametrize("mode", ["tf32", "fp16"])
@pytest.mark.parametrize("cin,c", encoder.DOWN_DIMS)
@pytest.mark.parametrize("mutant", ed.MUTANTS)
def test_each_mutant_breaks_a_check(mutant, cin, c, mode):
    x, ps = _case(cin, c, 1, 9, 7, 3)
    if mutant == "relu_drops_nan":                    # fmax(NaN, 0) = 0: visible only where a NaN reaches a ReLU
        x[0, 0, 4, 3] = float("nan")
        em = ed.emulate(x, ps, mode, mutant=mutant)
        assert not torch.isnan(em["out"]).all()
        assert torch.isnan(ed.emulate(x, ps, mode)["out"]).all()
        return
    assert _worst(x, ps, mode, mutant) > 1.0
