"""GPU: every kernel-launching entry point of include/xb200.h held to its documented memory contract with banded operands
(tests/abi_bounds.py, case table in tests/abi_bounds_cases.py).  Per case and shape:

  test_banded_contract   one launch with every operand inside a poisoned or sentinel-filled allocation: const inputs come
                         back bit-unchanged, no band or leading-dimension gap is written, every element of a fully-written
                         output is written, documented not-written elements keep their sentinel, and the grid reduction's
                         ticket is re-armed;
  test_banded_values     the banded launch's outputs against the family's float64 reference at the family's tolerance;
  test_tight_launch_is_not_influenced_by_the_bands
                         the valid outputs of the banded launch are bit-equal to those of a launch on tight torch.empty
                         buffers (every kernel here is bit-identical from launch to launch, so a difference is a read of a
                         band, a gap column or stale memory).

`-k banded` selects the two checks that run only on banded launches."""
import numpy as np
import pytest
import torch

import abi_bounds as ab
from abi_bounds_cases import CASES

pytestmark = pytest.mark.gpu
PARAMS = [pytest.param(c, s, id=i) for c in CASES for s, i in zip(c.shapes, c.ids())]


def _banded(case, shape):
    ops = ab.build_ops(case, shape)
    bufs, before = ab.launch_banded(case, shape, ops)
    return ops, bufs, before


@pytest.mark.parametrize("case,shape", PARAMS)
def test_banded_contract(case, shape):
    ops, bufs, before = _banded(case, shape)
    ab.check_contract(ops, bufs, before)
    print(f"{case.name} {ab.shape_id(shape)}: contract holds")


@pytest.mark.parametrize("case,shape", [p for p in PARAMS if p.values[0].values is not None])
def test_banded_values(case, shape):
    ops, bufs, before = _banded(case, shape)
    got = {k: (None if b is None else b.view.cpu()) for k, b in bufs.items()}
    errs = case.values(got, ab.inputs_of(ops), shape)
    print(f"{case.name} {ab.shape_id(shape)}: largest error vs float64 " +
          ", ".join(f"{k} {v:.3g}" for k, v in errs.items()))


@pytest.mark.parametrize("case,shape", PARAMS)
def test_tight_launch_is_not_influenced_by_the_bands(case, shape):
    ops, bufs, _ = _banded(case, shape)
    banded = ab.valid_outputs(ops, {k: (None if b is None else b.view) for k, b in bufs.items()})
    tight = ab.valid_outputs(ops, ab.launch_tight(case, shape, ops))
    for name, want in tight.items():
        assert torch.equal(ab.bits(banded[name]), ab.bits(want)), f"{name}: the banded launch differs from the tight one"
