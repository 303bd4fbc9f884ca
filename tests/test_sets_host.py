"""Host-side checks of the file-set scan's interface -- no GPU needed: the library exports agb_scan_set, and malformed
arguments are refused before any CUDA call."""
import ctypes as C
import agrep_b200 as ag
from agrep_b200 import _lib


def _call(p, texts, sizes, n, want=_lib.WANT_COUNT, records=None, capacity=0, per=True):
    L = _lib.lib()
    total = _lib.Result()
    per_file = (_lib.Result * max(n, 1))() if per else None
    rc = L.agb_scan_set(p._h, texts, sizes, n, want, records, capacity, per_file, C.byref(total))
    return rc, total


def test_set_entry_point_is_exported():
    assert "agb_scan_set" in _lib.EXPORTS and hasattr(_lib.lib(), "agb_scan_set")


def test_no_files_with_file_arrays_is_refused():
    p = ag.Pattern("because each", k=2)
    data = b"because each\n"
    texts = (C.c_void_p * 1)(C.cast(C.c_char_p(data), C.c_void_p))
    sizes = (C.c_uint64 * 1)(len(data))
    assert _call(p, texts, sizes, 0)[0] == -3
    assert b"no files" in _lib.lib().agb_last_error()
    rc, total = _call(p, None, None, 0, per=False)
    assert rc == 0 and total.n_matched == 0 and total.n_records == 0


def test_a_null_text_with_a_size_is_refused():
    p = ag.Pattern("because each", k=2)
    data = b"because each\n"
    texts = (C.c_void_p * 2)(C.cast(C.c_char_p(data), C.c_void_p), None)
    sizes = (C.c_uint64 * 2)(len(data), 5)
    assert _call(p, texts, sizes, 2)[0] == -3
    assert b"file 1 has no text" in _lib.lib().agb_last_error()


def test_a_capacity_without_a_list_is_refused():
    p = ag.Pattern("because each", k=2)
    data = b"because each\n"
    texts = (C.c_void_p * 1)(C.cast(C.c_char_p(data), C.c_void_p))
    sizes = (C.c_uint64 * 1)(len(data))
    assert _call(p, texts, sizes, 1, want=_lib.WANT_RECORDS, records=None, capacity=10)[0] == -3
    assert b"capacity without a record list" in _lib.lib().agb_last_error()


def test_missing_per_file_results_are_refused():
    p = ag.Pattern("because each", k=2)
    data = b"because each\n"
    texts = (C.c_void_p * 1)(C.cast(C.c_char_p(data), C.c_void_p))
    sizes = (C.c_uint64 * 1)(len(data))
    assert _call(p, texts, sizes, 1, per=False)[0] == -3
