"""The device dictionary's C ABI (bkgpu_dict_*, include/bkgpu.h) without a GPU: every malformed argument is refused with BKGPU_EINVAL
before any device is touched, and well-formed arguments without a device give BKGPU_ENODEV, not a fallback.  The pointers are never
dereferenced on these paths, so stand-in addresses serve as device buffers."""
import ctypes

import pytest

from baikaldb_b200 import _lib
from baikaldb_b200._lib import BkgpuBinaryColumn

FAKE = 0x1000   # a stand-in device address


def _cols(*specs):
    arr = (BkgpuBinaryColumn * max(len(specs), 1))()
    for i, (offsets, data, validity, voff, length) in enumerate(specs):
        arr[i].offsets, arr[i].data, arr[i].validity, arr[i].validity_offset, arr[i].length = offsets, data, validity, voff, length
    return arr


def _build(cols, ncols, device=0, out=True, hash_bits=0):
    h = ctypes.c_void_p()
    rc = _lib.lib().bkgpu_dict_build(ctypes.byref(h) if out else None, device, None, cols, ncols, hash_bits)
    assert not h.value   # nothing is handed out on a failure
    return rc


GOOD = (FAKE, FAKE, None, 0, 10)


@pytest.mark.parametrize("case, call", [
    ("out is NULL", lambda: _build(_cols(GOOD), 1, out=False)),
    ("cols is NULL", lambda: _build(None, 1)),
    ("no columns", lambda: _build(_cols(GOOD), 0)),
    ("negative column count", lambda: _build(_cols(GOOD), -1)),
    ("negative length", lambda: _build(_cols((FAKE, FAKE, None, 0, -1)), 1)),
    ("negative length in the second column", lambda: _build(_cols(GOOD, (FAKE, FAKE, None, 0, -5)), 2)),
    ("negative validity offset", lambda: _build(_cols((FAKE, FAKE, FAKE, -3, 10)), 1)),
    ("NULL offsets", lambda: _build(_cols((None, FAKE, None, 0, 10)), 1)),
    ("NULL data", lambda: _build(_cols((FAKE, None, None, 0, 10)), 1)),
    ("hash_bits out of range", lambda: _build(_cols(GOOD), 1, hash_bits=65)),
    ("negative hash_bits", lambda: _build(_cols(GOOD), 1, hash_bits=-1)),
])
def test_malformed_arguments_are_einval(case, call):
    assert call() == _lib.EINVAL, case
    assert _lib.lib().bkgpu_last_error(None).startswith(b"bkgpu_dict_build"), case


def test_calls_on_a_null_handle_are_einval():
    L = _lib.lib()
    n, b = ctypes.c_int64(), ctypes.c_int64()
    assert L.bkgpu_dict_size(None, ctypes.byref(n), ctypes.byref(b)) == _lib.EINVAL
    assert L.bkgpu_dict_copy(None, FAKE, FAKE, 1) == _lib.EINVAL
    assert L.bkgpu_dict_codes(None, 0, FAKE, FAKE, None) == _lib.EINVAL
    L.bkgpu_dict_free(None)   # a no-op


def test_no_device_is_enodev_not_a_fallback():
    L = _lib.lib()
    if L.bkgpu_device_count() > 0:
        assert _build(_cols(GOOD), 1, device=1 << 20) == _lib.EINVAL   # with a device, a bad index is still refused before any work
        pytest.skip("a GPU is visible here")
    assert _build(_cols(GOOD), 1) == _lib.ENODEV
    assert b"no CPU fallback" in L.bkgpu_last_error(None)
    assert _build(_cols(GOOD, (FAKE, FAKE, FAKE, 7, 0)), 2) == _lib.ENODEV   # an empty column with a validity offset is well-formed
