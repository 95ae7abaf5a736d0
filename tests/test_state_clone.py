"""CPU-only: the state clone entry points refuse with ENODEV without a device instead of computing anything."""
import ctypes as C

import pytest


def test_clone_entry_points_need_a_device():
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    from lighthouse_b200 import _ffi
    out, n, d = C.c_void_p(), C.c_uint64(0), C.c_int32(0)
    assert _ffi.lib.lhb200_state_clone(None, C.byref(out)) == _ffi.ENODEV
    assert _ffi.lib.lhb200_state_device_bytes(None, C.byref(n)) == _ffi.ENODEV
    assert _ffi.lib.lhb200_debug_state_disjoint(None, None, C.byref(d)) == _ffi.ENODEV
    assert _ffi.lib.lhb200_debug_state_live_bytes(None, C.byref(n)) == _ffi.ENODEV
    assert out.value is None
