"""ctypes binding of the checker's 320-bit rows (tests/_oracle_wide.c: orc_compile_wide, orc_scan_wide,
orc_scan_levels_wide) -- TEST INFRASTRUCTURE.  Same calling conventions as _oracle.compile/scan/scan_levels.
The library is compiled on first use into a temporary directory (nothing is written into the tree)."""
import ctypes as C
import hashlib
import os
import subprocess
import tempfile

import _oracle

HERE = os.path.dirname(os.path.abspath(__file__))
SOURCES = [os.path.join(HERE, "_oracle_wide.c"), os.path.join(_oracle.ROOT, "oracle", "agrep_oracle.c"),
           os.path.join(_oracle.ROOT, "oracle", "agrep_oracle.h")]

WIDE_WORDS = 5
WIDE_BITS = 64 * WIDE_WORDS


class Wide(C.Structure):
    _W = C.c_uint64 * WIDE_WORDS
    _fields_ = [("a", _oracle.Automaton), ("mask", _W * 256), ("init0", _W), ("init1", _W), ("noerr", _W), ("endpos", _W),
                ("dendpos", _W), ("dmask", _W), ("wildmask", _W)]


_lib = None


def _build():
    """compile the checker's 320-bit rows into <tmp>/agb_oracle_wide_<uid>_<hash of the sources>/ (once per source state)"""
    h = hashlib.sha256()
    for f in SOURCES:
        with open(f, "rb") as fh:
            h.update(fh.read())
    d = os.path.join(tempfile.gettempdir(), "agb_oracle_wide_%d_%s" % (os.getuid(), h.hexdigest()[:16]))
    so = os.path.join(d, "liboracle_wide.so")
    if not os.path.exists(so):
        os.makedirs(d, exist_ok=True)
        tmp = "%s.%d" % (so, os.getpid())
        subprocess.run([os.environ.get("CC") or "gcc", "-O2", "-Wall", "-Wextra", "-std=c11", "-fPIC", "-shared",
                        "-I", os.path.join(_oracle.ROOT, "oracle"), "-o", tmp, SOURCES[0]], check=True)
        os.replace(tmp, so)
    return so


def lib():
    global _lib
    if _lib is None:
        L = C.CDLL(_build())
        L.orc_compile_wide.argtypes = [C.c_char_p, C.POINTER(_oracle.Opts), C.POINTER(Wide), C.c_char_p, C.c_size_t]
        L.orc_scan_wide.restype = C.c_int64
        L.orc_scan_wide.argtypes = [C.POINTER(Wide), C.c_char_p, C.c_uint64, C.POINTER(_oracle.Record), C.c_uint64]
        L.orc_scan_levels_wide.restype = C.c_int64
        L.orc_scan_levels_wide.argtypes = [C.POINTER(Wide), C.c_int, C.c_char_p, C.c_uint64,
                                           C.POINTER(C.c_uint64), C.POINTER(_oracle.Record), C.c_uint64, C.c_int]
        _lib = L
    return _lib


def compile(pattern, **kw):
    """the automaton in 320-bit rows (kw as for _oracle.compile; width is set here)"""
    if isinstance(pattern, str):
        pattern = pattern.encode("latin-1")
    o = _oracle.Opts()
    for k, v in kw.items():
        if k == "delim" and isinstance(v, str):
            v = v.encode("latin-1")
        setattr(o, k, v)
    o.width = WIDE_BITS
    w = Wide()
    err = C.create_string_buffer(256)
    if lib().orc_compile_wide(pattern, C.byref(o), C.byref(w), err, 256) != 0:
        raise _oracle.OracleError(err.value.decode())
    return w


def scan(w, text, want_records=True, cap=None):
    """returns (count, [(begin, end, ordinal), ...])"""
    n = len(text)
    if not want_records:
        return lib().orc_scan_wide(C.byref(w), text, n, None, 0), []
    cap = cap or (n + 2)
    recs = (_oracle.Record * cap)()
    cnt = lib().orc_scan_wide(C.byref(w), text, n, recs, cap)
    return cnt, [(recs[i].begin, recs[i].end, recs[i].ordinal) for i in range(min(cnt, cap))]


def scan_levels(w, kmax, text, want_level=-1, cap=None):
    n = len(text)
    cap = cap or (n + 2)
    recs = (_oracle.Record * cap)()
    hist = (C.c_uint64 * 9)()
    cnt = lib().orc_scan_levels_wide(C.byref(w), kmax, text, n, hist, recs, cap, want_level)
    return cnt, list(hist), [(recs[i].begin, recs[i].end, recs[i].ordinal, recs[i].level) for i in range(min(cnt, cap))]
