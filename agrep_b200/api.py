"""Host-side mirror of the reference's scan interface for Python callers.

The reference exposes the scan path as `agrep [-# -i -w -x -v -n -p -I# -S# -D# -d delim -B -c] pattern file`
(agrep.c:2121-2739) and, as a library, `memagrep()/fileagrep()` (agrep.c:3282,3300).  `Pattern` takes the same
switches by name; `scan_*` return what exec() derives from the scan functions: num_of_matched and the
(lasti, print_end, j) triples handed to output() (agrep.c:3805).  All work happens in libagrepb200.so."""
import ctypes as C
import os
import stat
from . import _lib
from ._lib import (Options, Desc, Regex, Wide, Record, Result, CorpusSpec, WANT_COUNT, WANT_RECORDS, WANT_ORDINALS, WANT_LEVELS,
                   PLAN_ALL, PLAN_ANCHORS, ENGINE_NAMES, ENGINE_REGEX)


class AgrepError(Exception):
    pass


def _check_window(window):
    """a window is a multiple of 512 bytes (the cut rule puts window edges on 512-byte blocks) and at least 4 KiB"""
    if window is not None and (isinstance(window, bool) or not isinstance(window, int) or window < 4096 or window % 512):
        raise ValueError("window must be a multiple of 512 and at least 4096 bytes, got %r" % (window,))


class Pattern:
    """agb_compile(): checksg() + preprocess() + maskgen() of the reference, plus the device plan.
    regex: accept regular expressions (a pattern with an unescaped '|' or '*': re() of the reference, k <= 4, lines);
    without it such a pattern is refused.
    wide_approx: accept a simple literal of more than 63 positions (up to 255 characters) at k = 1..8, as the reference's
    sgrep() does, in 320-bit rows; without it such a pattern is refused as too long.
    sticky_delim: accept ins_free (-p) with a delimiter of two or more bytes, as the reference does: its positions are
    sticky too, so a record closes where the delimiter's bytes have occurred in order since the last close ("a ... b"
    for "ab"); without it such a pattern is refused.  The sharded scans refuse it either way."""

    def __init__(self, pattern, k=0, nocase=False, wordbound=False, wholeline=False, inverse=False,
                 linenum=False, ins_free=False, cost_i=0, cost_s=0, cost_d=0, bestmatch=False, delim=None, regex=False,
                 wide_approx=False, sticky_delim=False):
        if isinstance(pattern, str):
            pattern = pattern.encode("latin-1")
        if isinstance(delim, str):
            delim = delim.encode("latin-1")
        self.pattern = pattern
        self.opts = Options(k=k, nocase=int(nocase), wordbound=int(wordbound), wholeline=int(wholeline),
                            inverse=int(inverse), linenum=int(linenum), ins_free=int(ins_free),
                            cost_i=cost_i, cost_s=cost_s, cost_d=cost_d, bestmatch=int(bestmatch), regex=int(regex), delim=delim,
                            wide_approx=int(wide_approx), sticky_delim=int(sticky_delim))
        self._h = C.c_void_p()
        err = C.create_string_buffer(512)
        rc = _lib.lib().agb_compile(pattern, C.byref(self.opts), C.byref(self._h), err, 512)
        if rc != 0:
            raise AgrepError(err.value.decode("latin-1"))

    @property
    def desc(self):
        # a copy: the C object dies with this Pattern
        return Desc.from_buffer_copy(_lib.lib().agb_pattern_desc(self._h).contents)

    @property
    def regex(self):
        """the follow sets of a regular expression (a copy), None for every other engine"""
        r = _lib.lib().agb_pattern_regex(self._h)
        return Regex.from_buffer_copy(r.contents) if r else None

    @property
    def wide(self):
        """the 320-bit words of a simple literal of more than 63 positions (a copy; word 0 = bits 0..63 of each row; row 0
        of the post-delimiter and start rows in reset/start, rows 1..k in reset_up/start_up), None for every other pattern"""
        w = _lib.lib().agb_pattern_wide(self._h)
        return Wide.from_buffer_copy(w.contents) if w else None

    def __del__(self):
        try:
            if self._h:
                _lib.lib().agb_pattern_free(self._h)
        except Exception:
            pass

    # ---- scans -------------------------------------------------------------------------------
    def _finish(self, rc, res, recs, want):
        if rc != 0:
            raise AgrepError("agb_scan rc=%d: %s" % (rc, _lib.lib().agb_last_error().decode()))
        out = [(recs[i].begin, recs[i].end, recs[i].ordinal, recs[i].level) for i in range(res.n_records)] if recs is not None else []
        return res, out

    def scan_host(self, data, want_records=True, capacity=None, levels=False, ordinals=False, window=None):
        """data: bytes-like in host memory (the fill_buf path: H2D inside the call).
        ordinals: also fill Record.ordinal (the j that -n prints) and Result.n_closes on the device.
        window: None scans the whole text on the device (in windows only if it does not fit); a number of bytes (a
        multiple of 512, >= 4096) keeps at most that much text, plus halos, on the device at a time -- same result."""
        _check_window(window)
        n = len(data)
        want = (WANT_RECORDS if want_records else WANT_COUNT) | (WANT_LEVELS if levels else 0) | (WANT_ORDINALS if ordinals else 0)
        cap = (capacity if capacity is not None else n // 64 + 4096) if want_records else 0
        buf = (C.c_char * n).from_buffer_copy(data) if n else None
        while True:
            recs = (Record * cap)() if cap else None
            res = Result()
            if window is None:
                rc = _lib.lib().agb_scan_host(self._h, buf, n, want, recs, cap, C.byref(res))
            else:
                rc = _lib.lib().agb_scan_host_windowed(self._h, buf, n, window, want, recs, cap, C.byref(res))
            if rc != 0 or not res.truncated or capacity is not None:
                return self._finish(rc, res, recs, want)
            cap = res.n_matched          # the list did not fit (Result.truncated): once more with exactly n_matched entries

    def scan_fd(self, fd, want_records=True, capacity=None, levels=False, ordinals=False, window=None):
        """the text of file descriptor fd from its current offset to EOF (agb_scan_fd: regular files are pread(2) into
        the pinned ring, pipes read into a host buffer); the offset is left at EOF.  window: as in scan_host.
        Without a capacity the list is sized from the file's size and, when it did not fit, the file is scanned once
        more from the same offset -- a pipe cannot be read twice, so there the truncated result is returned."""
        _check_window(window)
        start = None
        try:
            start = os.lseek(fd, 0, os.SEEK_CUR)
            size = os.fstat(fd).st_size - start if stat.S_ISREG(os.fstat(fd).st_mode) else 0
        except OSError:                  # a pipe
            size = 0
        want = (WANT_RECORDS if want_records else WANT_COUNT) | (WANT_LEVELS if levels else 0) | (WANT_ORDINALS if ordinals else 0)
        cap = (capacity if capacity is not None else max(size, 0) // 64 + 4096) if want_records else 0
        while True:
            recs = (Record * cap)() if cap else None
            res = Result()
            if window is None:
                rc = _lib.lib().agb_scan_fd(self._h, fd, want, recs, cap, C.byref(res))
            else:
                rc = _lib.lib().agb_scan_fd_windowed(self._h, fd, window, want, recs, cap, C.byref(res))
            if rc != 0 or not res.truncated or capacity is not None or start is None:
                return self._finish(rc, res, recs, want)
            os.lseek(fd, start, os.SEEK_SET)
            cap = res.n_matched

    def scan_set(self, texts, want_records=True, capacity=None, levels=False, ordinals=False):
        """texts: a list of bytes-like host texts, scanned in one device pass (agb_scan_set), each as if alone.
        Returns (total Result, [Result per text], records) -- records as scan_host's tuples with the text's index last,
        file 0's first; offsets and ordinals relative to the record's own text.  capacity: as in scan_host, over the set."""
        nf = len(texts)
        want = (WANT_RECORDS if want_records else WANT_COUNT) | (WANT_LEVELS if levels else 0) | (WANT_ORDINALS if ordinals else 0)
        bufs = [(C.c_char * len(t)).from_buffer_copy(t) if len(t) else None for t in texts]
        ptrs = (C.c_void_p * nf)(*[C.cast(b, C.c_void_p) if b is not None else None for b in bufs]) if nf else None
        sizes = (C.c_uint64 * nf)(*[len(t) for t in texts]) if nf else None
        cap = (capacity if capacity is not None else sum(len(t) for t in texts) // 64 + 4096) if want_records else 0
        while True:
            recs = (Record * cap)() if cap else None
            total, per = Result(), ((Result * nf)() if nf else None)
            rc = _lib.lib().agb_scan_set(self._h, ptrs, sizes, nf, want, recs, cap, per, C.byref(total))
            if rc != 0:
                raise AgrepError("agb_scan_set rc=%d: %s" % (rc, _lib.lib().agb_last_error().decode()))
            if not total.truncated or capacity is not None:
                out = [(recs[i].begin, recs[i].end, recs[i].ordinal, recs[i].level, recs[i].pad) for i in range(total.n_records)]
                return total, (list(per) if nf else []), out
            cap = total.n_matched

    def scan_device(self, dev_ptr, n, stream=0, d_records=0, capacity=0, levels=False, ordinals=False):
        """dev_ptr: device address of n bytes (16-byte aligned, e.g. torch tensor .data_ptr())."""
        want = (WANT_RECORDS if capacity else WANT_COUNT) | (WANT_LEVELS if levels else 0) | (WANT_ORDINALS if ordinals else 0)
        res = Result()
        rc = _lib.lib().agb_scan_device(self._h, C.c_void_p(dev_ptr), n, want, C.c_void_p(d_records), capacity,
                                        C.c_void_p(stream), C.byref(res))
        if rc != 0:
            raise AgrepError("agb_scan_device rc=%d: %s" % (rc, _lib.lib().agb_last_error().decode()))
        return res


def bestmatch_device(pattern, dev_ptr, n, stream=0, d_records=0, capacity=0, **kw):
    """The -B sweep (agrep.c:3582-3728): returns (best_k or -1, Result); with d_records/capacity (device buffer of Record)
    also the ordered list of the records at the best level."""
    if isinstance(pattern, str):
        pattern = pattern.encode("latin-1")
    d = kw.pop("delim", None)
    if isinstance(d, str):
        d = d.encode("latin-1")
    o = Options(delim=d, **{k: int(v) for k, v in kw.items()})
    res, best, err = Result(), C.c_int(-1), C.create_string_buffer(512)
    rc = _lib.lib().agb_bestmatch_device(pattern, C.byref(o), C.c_void_p(dev_ptr), n, C.c_void_p(stream),
                                        C.c_void_p(d_records), capacity, C.byref(best), C.byref(res), err, 512)
    if rc != 0:
        raise AgrepError(err.value.decode() or _lib.lib().agb_last_error().decode())
    return best.value, res


def corpus_spec(n_bytes, seed=12345, first_page=0, paragraphs=False, needle=b"", needle_every=0, needle_maxedits=0):
    if isinstance(needle, str):
        needle = needle.encode()
    return CorpusSpec(seed=seed, n_bytes=n_bytes, first_page=first_page, paragraphs=int(paragraphs),
                      needle_every=needle_every, needle=needle, needle_maxedits=needle_maxedits)


def corpus_host(n_bytes, **kw):
    """bytes of the synthetic corpus, generated by the library's host generator (same code as the device's)."""
    spec = corpus_spec(n_bytes, **kw)
    buf = C.create_string_buffer(n_bytes)
    rc = _lib.lib().agb_corpus_fill_host(C.byref(spec), buf)
    if rc != 0:
        raise AgrepError(_lib.lib().agb_last_error().decode())
    return buf.raw


def corpus_device(dev_ptr, n_bytes, stream=0, **kw):
    spec = corpus_spec(n_bytes, **kw)
    rc = _lib.lib().agb_corpus_fill_device(C.byref(spec), C.c_void_p(dev_ptr), C.c_void_p(stream))
    if rc != 0:
        raise AgrepError(_lib.lib().agb_last_error().decode())
