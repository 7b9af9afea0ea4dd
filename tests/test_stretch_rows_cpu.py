"""CPU: the per-row time-stretch's host side -- the symbol is exported with its binding, and every refusal of
sopro_stretch_rows happens on the host before any launch (placeholder device pointers are never dereferenced)."""
import ctypes as C
import os

import pytest
import torch

from sopro_b200 import _lib
from sopro_b200 import stretch as ST

FAKE = 0x1000  # a non-null pointer no refused call may touch


def _call(B, x_stride, lens, S, y_stride, x=FAKE, y=FAKE, S_ptr=True):
    lib = _lib.load()
    lp = None if lens is None else (C.c_int64 * len(lens))(*lens)
    sp = (C.c_int32 * len(S))(*S) if S_ptr else None
    return lib.sopro_stretch_rows(x, B, x_stride, lp, sp, y, y_stride, None, None)


def test_symbol_is_exported_with_its_binding():
    lib = _lib.load()
    assert "sopro_stretch_rows" in _lib.SYMBOLS
    fn = lib.sopro_stretch_rows
    assert fn.restype is C.c_int and len(fn.argtypes) == 9
    with open(os.path.join(os.path.dirname(__file__), "..", "include", "sopro_b200.h")) as f:
        assert "int sopro_stretch_rows(" in f.read()


@pytest.mark.parametrize("args", [
    dict(B=2, x_stride=100, lens=[100, 50], S=[65536, 16383], y_stride=400),       # S below 0.25
    dict(B=2, x_stride=100, lens=[100, 50], S=[262145, 65536], y_stride=400),      # S above 4
    dict(B=3, x_stride=100, lens=[10, 20, 30], S=[65536, 65536, 0], y_stride=400),  # the last row's S
    dict(B=2, x_stride=100, lens=[100, 50], S=[65536, 65536], y_stride=400, S_ptr=False),  # no speeds
    dict(B=2, x_stride=100, lens=[100, 50], S=[65536, 65536], y_stride=400, x=None),
    dict(B=2, x_stride=100, lens=[100, 50], S=[65536, 65536], y_stride=400, y=None),
    dict(B=0, x_stride=100, lens=[], S=[], y_stride=400),
    dict(B=2, x_stride=-1, lens=None, S=[65536, 65536], y_stride=400),
    dict(B=2, x_stride=100, lens=[101, 50], S=[65536, 65536], y_stride=400),      # a row past x_stride
    dict(B=2, x_stride=100, lens=[-1, 50], S=[65536, 65536], y_stride=400),
    # y_stride under the longest row's outputs: 100 samples at 0.25 make 400, at 1 they make 100
    dict(B=2, x_stride=100, lens=[100, 100], S=[16384, 65536], y_stride=399),
    dict(B=2, x_stride=100, lens=[100, 60], S=[65536, 32768], y_stride=119),
    dict(B=2, x_stride=100, lens=None, S=[65536, 65536], y_stride=99),
])
def test_refusals_happen_before_any_launch(args):
    assert _call(**args) == -1  # SOPRO_ERR_INVALID, on a machine with or without a GPU
    assert _lib.load().sopro_last_error()


def test_nothing_to_write_is_not_an_error():
    # every row empty: no launch, no device needed
    assert _call(B=3, x_stride=100, lens=[0, 0, 0], S=[65536, 16384, 262144], y_stride=0) == 0


def test_python_refusals():
    """stretch_rows checks its speeds after the rows and before any allocation; a CPU tensor has no path."""
    with pytest.raises(_lib.SoproError):
        ST.stretch_rows(torch.zeros(2, 10), [1.0, 1.0])
    assert ST.quantise(1.0) == 65536  # every speed goes through the same quantisation as stretch
    for bad in (0.2, 4.5, float("nan"), True, "1"):
        with pytest.raises(ValueError):
            ST.quantise(bad)
