"""Banded operands: every buffer a kernel sees sits inside a larger allocation whose bands (and leading-dimension gap
columns) hold a role-specific poison or sentinel, so that a stray read or write past an operand's documented extent lands in
memory the test owns and shows up as a changed band, a NaN in a value, or a difference from a launch on tight buffers.

Roles, as include/xb200.h documents each operand:

  role          band                                    interior before the launch     checked after the launch
  in            float: quiet NaN (payload IN_NAN)       the test data                  whole buffer bit-unchanged
                uint8: 1;  int: a legal in-range value
  out           sentinel bytes 0xA5                     NaN with payload OUT_NAN       bands bit-unchanged; no interior
                                                                                       element still carries OUT_NAN
  out_scatter   sentinel                                zeros (pre-zeroed by contract) bands bit-unchanged
  out_partial   sentinel                                sentinel                       bands and the documented
                                                                                       not-written elements unchanged
  inout         sentinel                                the test data                  bands bit-unchanged
  scratch       sentinel                                zeros                          bands bit-unchanged; the grid
                                                                                       reduction's ticket is 0 again

Integer poison is always a value that is legal for the operand, so an over-read of an index can never become an address
outside an allocation.  Everything is compared as bit patterns (float32 viewed as int32, float64 as int64).

This module has no pytest fixtures and imports nothing CUDA-specific at import time, so its self-test runs on the CPU."""
from dataclasses import dataclass, field
from typing import Any, Callable, Optional

import numpy as np
import torch

BAND_BYTES = 4096            # > one 256-thread block of float32 on each side
ROLES = ("in", "out", "out_scatter", "out_partial", "inout", "scratch")
SENTINEL_BYTE = 0xA5
IN_NAN32, OUT_NAN32 = 0x7FC0BAD1, 0x7FC00DED                   # quiet NaNs with two different payloads
IN_NAN64, OUT_NAN64 = 0x7FF800000000BAD1, 0x7FF8000000000DED
OUT_U8 = 0x5A                                                  # no uint8 output of the ABI is a byte of this value
XB_MAX_PARTIALS = 2048                                         # xb_common.cuh; the ticket sits after 8 slot groups
TICKET_INT32 = 2 * 8 * XB_MAX_PARTIALS                         # scratch[8 * XB_MAX_PARTIALS] as an int32 index

_BITS = {torch.float32: torch.int32, torch.float64: torch.int64, torch.int32: torch.int32, torch.int64: torch.int64,
         torch.uint8: torch.uint8}


def bits(t):
    """The tensor's bit pattern as an integer tensor of the same element size (NaN payloads compare exactly)."""
    return t.view(_BITS[t.dtype])


def signed(pattern, size):
    """An unsigned bit pattern of `size` bytes as the signed integer bits() shows it."""
    u, s = {4: (np.uint32, np.int32), 8: (np.uint64, np.int64)}[size]
    return int(np.array([pattern], u).view(s)[0])


def _fill_bits(t, pattern):
    bits(t).fill_(signed(pattern, t.element_size()))


def _sentinel(t):
    t.view(torch.uint8).fill_(SENTINEL_BYTE)


def _band_fill(t, role, legal):
    """Write the band value of `role` into every element of `t` (a band or gap region)."""
    if role == "in":
        if t.dtype == torch.float32:
            _fill_bits(t, IN_NAN32)
        elif t.dtype == torch.float64:
            _fill_bits(t, IN_NAN64)
        elif t.dtype == torch.uint8:
            t.fill_(1)
        else:
            t.fill_(int(legal))
    else:
        _sentinel(t)


def _out_payload(t):
    if t.dtype == torch.uint8:
        t.fill_(OUT_U8)
    elif t.element_size() == 8:
        _fill_bits(t, OUT_NAN64)
    else:
        _fill_bits(t, OUT_NAN32)


def payload_of(dtype):
    """The bit pattern an `out` interior holds before the launch, as the integer bits() shows it."""
    size = torch.empty((), dtype=dtype).element_size()
    return OUT_U8 if size == 1 else signed(OUT_NAN64 if size == 8 else OUT_NAN32, size)


class Banded:
    """One banded operand: `view` is what the kernel gets (a view into `whole`), `inner` marks the view's elements in
    `whole` (gap columns of a leading-dimension operand are band)."""

    def __init__(self, view, whole, inner, offset, role):
        self.view, self.whole, self.inner, self.offset, self.role = view, whole, inner, offset, role

    def __iter__(self):
        return iter((self.view, self.whole))


def banded(shape, dtype, role, align=16, ld=None, legal=0, data=None, device="cuda"):
    """Allocate band + numel + band elements (leading-dimension operands: rows * ld, the columns past the width are
    band) and return a Banded whose `view` starts exactly at `align` bytes past a 256-byte boundary (16: aligned to 16
    and to no more; 4: the scalar-fallback misalignment).  `data` (array-like) fills the interior of in / inout operands.
    """
    assert role in ROLES, role
    shape = tuple(int(s) for s in shape)
    itemsize = torch.empty((), dtype=dtype).element_size()
    assert align % itemsize == 0 and align in (4, 16), (align, dtype)
    band = BAND_BYTES // itemsize
    width = shape[-1] if shape else 1
    rows = int(np.prod(shape[:-1])) if len(shape) > 1 else 1
    if ld is None:
        ld = width
    assert ld >= width
    span = rows * ld if shape else 1
    lead = band + align // itemsize
    total = lead + span + band
    raw = torch.empty(total + 256 // itemsize, dtype=dtype, device=device)
    shift = (-raw.data_ptr()) % 256 // itemsize                   # whole starts on a 256-byte boundary
    whole = raw[shift:shift + total]
    _band_fill(whole, role, legal)
    flat = whole[lead:lead + span]
    view = flat.view(rows, ld)[:, :width].view(shape) if ld != width else flat.view(shape)
    inner = torch.zeros(whole.numel(), dtype=torch.bool, device=device)
    inner[lead:lead + span].view(rows, ld)[:, :width] = True
    if role in ("in", "inout"):
        assert data is not None, "in / inout operands need data"
        view.copy_(torch.as_tensor(np.ascontiguousarray(data)).to(device=device, dtype=dtype).reshape(shape))
    elif role == "out":
        _out_payload(view)
    elif role in ("out_scatter", "scratch"):
        view.zero_()
    else:
        _sentinel(view)
    assert view.data_ptr() % 256 == align
    out = Banded(view, whole, inner, lead, role)
    out.end = lead + span
    return out


# ------------------------------------------------------------------------------------------------ case records
@dataclass
class Op:
    """One operand of a case: its role, dtype and shape, the data of in / inout operands, its leading dimension (gap
    columns are band), the legal band value of an integer input, whether it takes the 4-byte misalignment when the shape
    asks for it, and (out_partial) the boolean mask of the elements the contract leaves unwritten."""
    role: str
    shape: tuple
    dtype: Any = torch.float32
    data: Optional[np.ndarray] = None
    ld: Optional[int] = None
    legal: int = 0
    mis: bool = False
    unwritten: Optional[np.ndarray] = None


@dataclass
class Case:
    """One kernel-launching entry point.  build(shape, rng) -> {name: Op or None (NULL)}; launch(t, shape) calls the ABI
    with t[name] the device tensors (None for NULL); values(got, x, shape) checks the outputs got[name] (CPU tensors of
    the interior) against the family's float64 reference for inputs x[name] (the numpy data) and returns the largest
    error relative to float64 (raises AssertionError on a violation), or is None for a case whose values the family test
    pins on tight buffers and which this harness checks for contract and influence only."""
    name: str
    shapes: list
    build: Callable
    launch: Callable
    values: Optional[Callable] = None
    prototypes: tuple = field(default=())

    def ids(self):
        return [f"{self.name}[{shape_id(s)}]" for s in self.shapes]


def shape_id(shape):
    return ",".join(f"{k}={v}" for k, v in shape.items())


# ------------------------------------------------------------------------------------------------ running a case
def build_ops(case, shape, seed=0):
    return case.build(shape, np.random.default_rng(seed))


def launch_banded(case, shape, ops, device="cuda"):
    """Launch `case` with every operand banded.  Returns ({name: Banded or None}, {name: bits of whole before})."""
    align = shape.get("align", 16)
    bufs, before = {}, {}
    for name, op in ops.items():
        if op is None:
            bufs[name] = None
            continue
        bufs[name] = banded(op.shape, op.dtype, op.role, align=align if op.mis else 16, ld=op.ld, legal=op.legal,
                            data=op.data, device=device)
        before[name] = bits(bufs[name].whole).clone()
    case.launch({k: (None if b is None else b.view) for k, b in bufs.items()}, shape)
    torch.cuda.synchronize()
    return bufs, before


def launch_tight(case, shape, ops, device="cuda"):
    """The same launch on tight buffers: torch.empty outputs, zeroed scatter outputs and scratch, gap columns 0."""
    t = {}
    for name, op in ops.items():
        if op is None:
            t[name] = None
            continue
        width = op.shape[-1]
        full = (*op.shape[:-1], op.ld) if op.ld is not None else op.shape
        if op.role in ("in", "inout"):
            buf = torch.zeros(full, dtype=op.dtype, device=device)
            buf[..., :width] = torch.as_tensor(np.ascontiguousarray(op.data)).to(device=device, dtype=op.dtype).reshape(
                op.shape)
        elif op.role in ("out_scatter", "scratch"):
            buf = torch.zeros(full, dtype=op.dtype, device=device)
        else:
            buf = torch.empty(full, dtype=op.dtype, device=device)
        t[name] = buf[..., :width] if op.ld is not None else buf
    case.launch(t, shape)
    torch.cuda.synchronize()
    return t


def check_contract(ops, bufs, before):
    """The role checks of the module docstring; raises AssertionError naming the operand and what changed."""
    for name, op in ops.items():
        b = bufs.get(name)
        if b is None:
            continue
        now, was = bits(b.whole), before[name]
        if op.role == "in":
            changed = (now != was).nonzero()
            assert changed.numel() == 0, f"{name}: const input changed at {_where(b, changed)}"
            continue
        band = ~b.inner
        changed = ((now != was) & band).nonzero()
        assert changed.numel() == 0, f"{name}: {changed.numel()} band elements written, first at {_where(b, changed)}"
        if op.role == "out":
            left = (bits(b.view) == payload_of(op.dtype)).nonzero()
            assert left.numel() == 0, f"{name}: {left.shape[0]} interior elements never written, first at " \
                                      f"{tuple(left[0].tolist())}"
        if op.role == "out_partial" and op.unwritten is not None:
            mask = torch.as_tensor(op.unwritten, device=b.view.device)
            same = bits(b.view)[mask] == bits(b.view).new_full((), signed_sentinel(op.dtype))
            assert bool(same.all()), f"{name}: {int((~same).sum())} documented not-written elements were written"
        if op.role == "scratch" and op.dtype == torch.float64 and b.view.numel() * 2 > TICKET_INT32:
            ticket = int(b.view.view(torch.int32)[TICKET_INT32])
            assert ticket == 0, f"{name}: grid-reduction ticket left at {ticket}"


def signed_sentinel(dtype):
    size = torch.empty((), dtype=dtype).element_size()
    return SENTINEL_BYTE if size == 1 else signed(int.from_bytes(bytes([SENTINEL_BYTE]) * size, "little"), size)


def _where(b, changed):
    i = int(changed[0])
    rel = i - b.offset
    side = "before the operand" if rel < 0 else "past the operand" if i >= b.end else "in a leading-dimension gap"
    return f"element {rel} relative to the operand start ({side})"


def valid_outputs(ops, tensors):
    """{name: CPU copy} of what a launch writes: out / out_scatter / inout whole, out_partial with the documented
    not-written elements zeroed (they are compared elsewhere)."""
    out = {}
    for name, op in ops.items():
        t = tensors.get(name)
        if t is None or op.role in ("in", "scratch"):
            continue
        c = t.detach().cpu().clone()
        if op.role == "out_partial" and op.unwritten is not None:
            c[torch.as_tensor(op.unwritten)] = 0
        out[name] = c
    return out


def inputs_of(ops):
    return {k: op.data for k, op in ops.items() if op is not None and op.role in ("in", "inout")}
