"""Host-side checks of the windowed scan's interface -- no GPU needed: the library exports it, and a window that is not a
multiple of 512 or is shorter than 4 KiB is refused, by the Python wrappers before the library is called at all, and by
the C entry points before any CUDA call."""
import ctypes as C
import os
import pytest
import agrep_b200 as ag
from agrep_b200 import _lib

BAD = [0, 511, 512, 2048, 4095, 4097, 4096 + 256, 1.5 * 4096, "4096", True]


def test_windowed_entry_points_are_exported():
    L = _lib.lib()
    for name in ("agb_scan_host_windowed", "agb_scan_fd_windowed"):
        assert name in _lib.EXPORTS and hasattr(L, name)


@pytest.mark.parametrize("window", BAD)
def test_python_wrappers_refuse_a_bad_window_before_calling_the_library(monkeypatch, window):
    p = ag.Pattern("because each", k=2)

    def no_library():
        raise AssertionError("the library was called")
    monkeypatch.setattr(_lib, "lib", no_library)
    with pytest.raises(ValueError, match="multiple of 512"):
        p.scan_host(b"because each\n" * 100, window=window)
    rd, wr = os.pipe()
    try:
        with pytest.raises(ValueError, match="multiple of 512"):
            p.scan_fd(rd, window=window)
    finally:
        os.close(rd)
        os.close(wr)


@pytest.mark.parametrize("window", [0, 511, 4095, 4097, 8192 + 64])
def test_c_entry_points_refuse_a_bad_window(window):
    L = _lib.lib()
    p = ag.Pattern("because each", k=2)
    data = b"because each\n" * 100
    res = _lib.Result()
    assert L.agb_scan_host_windowed(p._h, data, len(data), window, _lib.WANT_COUNT, None, 0, C.byref(res)) == -3
    assert b"multiple of 512" in L.agb_last_error()
    rd, wr = os.pipe()
    try:
        # refused before the pipe is read: it is still open for writing and nothing has been written
        assert L.agb_scan_fd_windowed(p._h, rd, window, _lib.WANT_COUNT, None, 0, C.byref(res)) == -3
    finally:
        os.close(rd)
        os.close(wr)
