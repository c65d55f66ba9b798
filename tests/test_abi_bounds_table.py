"""CPU: the banded-operand harness holds every kernel-launching entry point of include/xb200.h to its memory contract, so
every prototype there has a case in tests/abi_bounds_cases.py or an exclusion below with its reason, and every case names
a real prototype.  Then a new kernel cannot land without a contract case.  Also a self-test of banded() on CPU tensors:
the interior's offset and alignment, the band sizes, and the poison and sentinel patterns of each role."""
import numpy as np
import pytest
import torch

import abi_bounds as ab
from abi_bounds_cases import CASES
from test_abi_prototypes import _prototypes

_HOST = "host-only or informational: launches nothing"
_K12 = ("K12 tensor-core family: the exact-reduction replay pins it with sentinel outputs and test_gpu_k12_encoder checks "
        "its persistent padded buffers; banding it is a follow-up")
EXCLUDED = {
    "xb_version": _HOST, "xb_error_string": _HOST, "xb_device_info": _HOST, "xb_scratch_doubles": _HOST,
    "xb_ppo_gauss_ws_doubles": _HOST, "xb_npg_gauss_ws_doubles": _HOST, "xb_npg_segment_table": _HOST,
    "xb_qtran_encode_bwd_work": _HOST,
    "xb_debug_k12_timing": "test hook", "xb_debug_tma_box": "test hook",
    "xb_split_bf16": _K12, "xb_pack_conv_weight": _K12, "xb_pack_weights": _K12, "xb_gemm_gather_tc": _K12,
    "xb_gemm_box_tc": _K12, "xb_gemm_halo_tc": _K12, "xb_wgrad_box_tc": _K12, "xb_wgrad_gather_tc": _K12,
    "xb_wgrad_reduce": _K12,
}


def test_every_prototype_has_a_case_or_a_reasoned_exclusion():
    protos = set(_prototypes())
    cased = {c.name for c in CASES}
    assert not cased - protos, f"cases that name no prototype of include/xb200.h: {sorted(cased - protos)}"
    assert not set(EXCLUDED) - protos, f"exclusions that name no prototype: {sorted(set(EXCLUDED) - protos)}"
    assert not cased & set(EXCLUDED), f"both a case and an exclusion: {sorted(cased & set(EXCLUDED))}"
    missing = protos - cased - set(EXCLUDED)
    assert not missing, f"entry points with neither a banded case nor an exclusion: {sorted(missing)}"
    assert all(EXCLUDED[k] for k in EXCLUDED)


def test_every_case_has_shapes_and_unique_ids():
    ids = [i for c in CASES for i in c.ids()]
    assert len(ids) == len(set(ids))
    assert all(c.shapes for c in CASES)
    assert len({c.name for c in CASES}) == len(CASES), "one record per entry point"


def _bits_all(t, pattern):
    return bool((ab.bits(t) == pattern).all())


@pytest.mark.parametrize("align", [16, 4])
@pytest.mark.parametrize("dtype", [torch.float32, torch.int32, torch.uint8])
def test_banded_layout_and_alignment(dtype, align):
    b = ab.banded((3, 5), dtype, "out", align=align, device="cpu")
    size = b.whole.element_size()
    assert b.view.data_ptr() % 256 == align
    assert b.view.data_ptr() - b.whole.data_ptr() >= ab.BAND_BYTES
    tail = b.whole.data_ptr() + b.whole.numel() * size - (b.view.data_ptr() + b.view.numel() * size)
    assert tail >= ab.BAND_BYTES
    assert b.view.is_contiguous() and b.view.shape == (3, 5)
    assert int(b.inner.sum()) == 15


def test_banded_float64_and_int64_layout():
    for dtype in (torch.float64, torch.int64):
        b = ab.banded((7,), dtype, "out", device="cpu")
        assert b.view.data_ptr() % 256 == 16 and b.offset * 8 >= ab.BAND_BYTES
    with pytest.raises(AssertionError):
        ab.banded((7,), torch.float64, "out", align=4, device="cpu")


def test_band_and_interior_patterns_per_role():
    x = np.arange(6, dtype=np.float32).reshape(2, 3)
    band = lambda b: b.whole[~b.inner]
    b = ab.banded((2, 3), torch.float32, "in", data=x, device="cpu")
    assert _bits_all(band(b), ab.signed(ab.IN_NAN32, 4)) and np.array_equal(b.view.numpy(), x)
    b = ab.banded((2, 3), torch.float64, "in", data=x.astype(np.float64), device="cpu")
    assert _bits_all(band(b), ab.signed(ab.IN_NAN64, 8)) and torch.isnan(band(b)).all()
    b = ab.banded((4,), torch.uint8, "in", data=np.array([0, 1, 0, 1], np.uint8), device="cpu")
    assert (band(b) == 1).all()
    b = ab.banded((4,), torch.int64, "in", data=np.array([3, 1, 2, 0]), legal=2, device="cpu")
    assert (band(b) == 2).all()
    b = ab.banded((2, 3), torch.float32, "out", device="cpu")
    assert _bits_all(b.view, ab.payload_of(torch.float32)) and torch.isnan(b.view).all()
    assert (band(b).view(torch.uint8) == ab.SENTINEL_BYTE).all()
    assert not _bits_all(b.view, ab.signed(ab.IN_NAN32, 4))
    b = ab.banded((5,), torch.int32, "out", device="cpu")
    assert _bits_all(b.view, ab.payload_of(torch.int32))
    b = ab.banded((5,), torch.uint8, "out", device="cpu")
    assert (b.view == ab.OUT_U8).all()
    for role in ("out_scatter", "scratch"):
        b = ab.banded((2, 3), torch.float32, role, device="cpu")
        assert (b.view == 0).all() and (band(b).view(torch.uint8) == ab.SENTINEL_BYTE).all()
    b = ab.banded((2, 3), torch.float32, "out_partial", device="cpu")
    assert (b.whole.view(torch.uint8) == ab.SENTINEL_BYTE).all()
    assert _bits_all(b.view, ab.signed_sentinel(torch.float32))
    b = ab.banded((2, 3), torch.float32, "inout", data=x, device="cpu")
    assert np.array_equal(b.view.numpy(), x) and (band(b).view(torch.uint8) == ab.SENTINEL_BYTE).all()


def test_leading_dimension_gap_columns_are_band():
    av = np.array([[1, 0, 1], [0, 1, 1]], np.uint8)
    b = ab.banded((2, 3), torch.uint8, "in", ld=5, data=av, device="cpu")
    assert b.view.shape == (2, 3) and b.view.stride() == (5, 1)
    assert np.array_equal(b.view.numpy(), av)
    rows = b.whole[b.offset:b.offset + 10].view(2, 5)
    assert (rows[:, 3:] == 1).all() and not b.inner[b.offset:b.offset + 10].view(2, 5)[:, 3:].any()
    assert int(b.inner.sum()) == 6


def test_contract_check_sees_each_kind_of_violation():
    """check_contract on CPU buffers edited by hand: a write past the end, a stale interior element, a changed input,
    a written not-written element and a ticket left armed all fail; the untouched launch passes."""
    ops = {"x": ab.Op("in", (4,), torch.float32, data=np.ones(4, np.float32)), "y": ab.Op("out", (4,)),
           "z": ab.Op("out_partial", (4,), unwritten=np.array([False, True, False, False])),
           "s": ab.Op("scratch", (ab.XB_MAX_PARTIALS * 8 + 8,), torch.float64)}

    def fresh():
        bufs = {k: ab.banded(o.shape, o.dtype, o.role, data=o.data, device="cpu") for k, o in ops.items()}
        return bufs, {k: ab.bits(b.whole).clone() for k, b in bufs.items()}

    def written(bufs):
        bufs["y"].view.fill_(2.0)
        bufs["z"].view[[0, 2, 3]] = 3.0

    bufs, before = fresh()
    written(bufs)
    ab.check_contract(ops, bufs, before)
    edits = [lambda b: b["y"].whole.__setitem__(b["y"].end, 0.0), lambda b: b["y"].view.__setitem__(3, float("nan")),
             lambda b: b["x"].view.__setitem__(0, 2.0), lambda b: b["z"].view.__setitem__(1, 0.0),
             lambda b: b["s"].view.view(torch.int32).__setitem__(ab.TICKET_INT32, 1),
             lambda b: b["x"].whole.__setitem__(b["x"].offset - 1, 0.0)]
    for i, edit in enumerate(edits):
        bufs, before = fresh()
        written(bufs)
        if i == 1:
            bufs["y"].view[3] = torch.tensor(ab.payload_of(torch.float32), dtype=torch.int32).view(torch.float32)
        else:
            edit(bufs)
        with pytest.raises(AssertionError):
            ab.check_contract(ops, bufs, before)
