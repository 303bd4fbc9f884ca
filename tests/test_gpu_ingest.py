"""Every way host bytes reach the device gives the answer of a scan of the same bytes already in device memory
(agb_scan_device): the whole-text host and file scans, the resident text, and the windowed scans -- from pageable and
page-locked memory, from a file read through the page cache or past it (AGB_ODIRECT=1), from a block-aligned offset and
from one that is not.  Counts, level histogram, delimiter total and the ordered record list with ordinals and levels,
byte for byte.  The sizes put a ragged tail behind three 64 MiB upload slices, end exactly on a slice boundary, or stay
inside one 16-byte chunk; the 96 MiB windows make upload ranges that start inside a slice.  A file that cannot be read (a
descriptor opened write-only) fails each file entry point with an error that names pread(2), and the device stays usable.
The O_DIRECT routes run on a file system that accepts O_DIRECT reads (tmpfs does not); where none does, they are skipped."""
import contextlib
import ctypes as C
import mmap
import os
import shutil
import tempfile
import pytest
import agrep_b200 as ag
from agrep_b200 import _lib

pytestmark = pytest.mark.gpu
MIB = 1 << 20
WANT = _lib.WANT_RECORDS | _lib.WANT_ORDINALS | _lib.WANT_LEVELS
CAP = 1 << 16
SIZES = {"three_slices_ragged": 3 * 64 * MIB + 12345, "two_slices_exact": 2 * 64 * MIB, "one_chunk": 15}


@pytest.fixture(scope="module")
def corpus():
    n = SIZES["three_slices_ragged"]
    return ag.corpus_host((n + 4095) // 4096 * 4096, needle="because each", needle_every=64, needle_maxedits=3)[:n]


def text_of(corpus, size):
    if size >= 4096:
        return corpus[:size]
    at = corpus.find(b"because each")           # a short text that still holds a match
    assert at >= 0
    return corpus[at:at + size]


def accepts_o_direct(d):
    """a 4 KiB O_DIRECT read of a file in directory d works (opened as the library opens it, through /proc/self/fd)"""
    probe = os.path.join(d, "probe")
    try:
        with open(probe, "wb") as f:
            f.write(b"x" * 8192)
        fd = os.open(probe, os.O_RDONLY)
        try:
            dfd = os.open("/proc/self/fd/%d" % fd, os.O_RDONLY | os.O_DIRECT)
            try:
                return os.preadv(dfd, [mmap.mmap(-1, 4096)], 0) == 4096      # (mmap: a page-aligned buffer)
            finally:
                os.close(dfd)
        finally:
            os.close(fd)
    except OSError:
        return False
    finally:
        if os.path.exists(probe):
            os.unlink(probe)


@pytest.fixture(scope="module")
def direct_dir(tmp_path_factory):
    """a scratch directory whose file system accepts O_DIRECT reads, or None"""
    found = None
    for base in (str(tmp_path_factory.mktemp("odirect")), "/var/tmp", os.path.expanduser("~")):
        try:
            d = tempfile.mkdtemp(prefix="agb_ingest_", dir=base)
        except OSError:
            continue
        if accepts_o_direct(d):
            found = d
            break
        shutil.rmtree(d, ignore_errors=True)
    yield found
    if found:
        shutil.rmtree(found, ignore_errors=True)


@contextlib.contextmanager
def odirect(on):
    old = os.environ.pop("AGB_ODIRECT", None)
    if on:
        os.environ["AGB_ODIRECT"] = "1"
    try:
        yield
    finally:
        os.environ.pop("AGB_ODIRECT", None)
        if old is not None:
            os.environ["AGB_ODIRECT"] = old


def device_answer(p, data):
    import torch
    dev = torch.frombuffer(bytearray(data + b"\0" * 64), dtype=torch.uint8).cuda()
    drec = torch.zeros((CAP, 4), dtype=torch.int64, device="cuda")
    r = p.scan_device(dev.data_ptr(), len(data), d_records=drec.data_ptr(), capacity=CAP, ordinals=True, levels=True)
    return (r.n_matched, list(r.level_hist), r.n_closes, r.n_records, drec[:r.n_records].cpu().numpy().tobytes())


def host_answer(fn):
    """fn(records, result) is one entry point's call; its answer in the form of device_answer"""
    L = _lib.lib()
    recs = (_lib.Record * CAP)()
    res = _lib.Result()
    rc = fn(recs, C.byref(res))
    assert rc == 0, L.agb_last_error()
    return (res.n_matched, list(res.level_hist), res.n_closes, res.n_records,
            C.string_at(C.addressof(recs), res.n_records * C.sizeof(_lib.Record)))


def text_answer(p, upload):
    """upload(&text) makes a resident text; agb_scan_text's answer over it"""
    L = _lib.lib()
    t = C.c_void_p()
    assert upload(C.byref(t)) == 0, L.agb_last_error()
    try:
        return host_answer(lambda recs, res: L.agb_scan_text(p._h, t, WANT, recs, CAP, res))
    finally:
        L.agb_text_free(t)


def fd_answer(direct, path, offset, scan):
    """scan(fd), one entry point's answer, on the file from `offset`, with or without AGB_ODIRECT=1; the descriptor is
    left at the file's end"""
    fd = os.open(str(path), os.O_RDONLY)
    try:
        os.lseek(fd, offset, os.SEEK_SET)
        with odirect(direct):
            got = scan(fd)
        assert os.lseek(fd, 0, os.SEEK_CUR) == os.fstat(fd).st_size
        return got
    finally:
        os.close(fd)


@pytest.mark.parametrize("direct", [False, True], ids=["page_cache", "o_direct"])
@pytest.mark.parametrize("size", list(SIZES.values()), ids=list(SIZES))
def test_every_route_gives_one_answer(tmp_path, direct_dir, corpus, size, direct):
    import torch
    if direct and direct_dir is None:
        pytest.skip("no scratch file system here accepts O_DIRECT reads")
    L = _lib.lib()
    data = text_of(corpus, size)
    n = len(data)
    p = ag.Pattern("because each", k=2)
    want = device_answer(p, data)
    assert want[0] > 0 and any(want[1])
    assert size < 4096 or any(want[1][1:])      # edited needles: records at levels 1 and 2 too

    skip = 1000                                 # not a multiple of the 4 KiB block: no direct reads from there
    where = tempfile.mkdtemp(dir=direct_dir) if direct else str(tmp_path)
    path, shifted = os.path.join(where, "text"), os.path.join(where, "shifted")
    with open(path, "wb") as f:
        f.write(data)
    with open(shifted, "wb") as f:
        f.write(b"z" * (skip - 1) + b"\n" + data)

    routes = {}
    if not direct:                              # (host memory routes do not depend on AGB_ODIRECT)
        pageable = C.create_string_buffer(data, n)
        pinned_t = torch.empty(n, dtype=torch.uint8, pin_memory=True)
        pinned_t.copy_(torch.frombuffer(bytearray(data), dtype=torch.uint8))
        for name, mem in (("pageable", pageable), ("pinned", C.c_void_p(pinned_t.data_ptr()))):
            routes["scan_host " + name] = lambda mem=mem: host_answer(
                lambda recs, res: L.agb_scan_host(p._h, mem, n, WANT, recs, CAP, res))
            routes["text_from_host " + name] = lambda mem=mem: text_answer(p, lambda t: L.agb_text_from_host(mem, n, t))
            for w in (4 * MIB, 96 * MIB):
                routes["scan_host_windowed %s %d MiB" % (name, w // MIB)] = lambda mem=mem, w=w: host_answer(
                    lambda recs, res: L.agb_scan_host_windowed(p._h, mem, n, w, WANT, recs, CAP, res))
    for file, off in ((path, 0), (shifted, skip)):
        routes["scan_fd at %d" % off] = lambda file=file, off=off: fd_answer(
            direct, file, off, lambda fd: host_answer(lambda recs, res: L.agb_scan_fd(p._h, fd, WANT, recs, CAP, res)))
        routes["text_from_fd at %d" % off] = lambda file=file, off=off: fd_answer(
            direct, file, off, lambda fd: text_answer(p, lambda t: L.agb_text_from_fd(fd, t)))
    for w in (4 * MIB, 96 * MIB):
        routes["scan_fd_windowed %d MiB" % (w // MIB)] = lambda w=w: fd_answer(
            direct, path, 0, lambda fd: host_answer(lambda recs, res: L.agb_scan_fd_windowed(p._h, fd, w, WANT, recs, CAP, res)))

    wrong = []
    try:
        for name, route in routes.items():
            got = route()
            if got != want:
                wrong.append((name, got[:4], want[:4]))
    finally:
        if direct:
            shutil.rmtree(where, ignore_errors=True)
    assert not wrong, wrong


def test_read_errors_leave_the_device_usable(tmp_path, corpus):
    """a regular file whose descriptor cannot be read: fstat says regular, pread(2) fails (EBADF)"""
    L = _lib.lib()
    data = corpus[:3 * MIB + 777]
    p = ag.Pattern("because each", k=2)
    path = tmp_path / "text"
    path.write_bytes(data)
    recs = (_lib.Record * CAP)()
    res = _lib.Result()
    fd = os.open(str(path), os.O_WRONLY)
    try:
        with odirect(False):
            for name, call in (("agb_scan_fd", lambda: L.agb_scan_fd(p._h, fd, WANT, recs, CAP, C.byref(res))),
                               ("agb_scan_fd_windowed", lambda: L.agb_scan_fd_windowed(p._h, fd, MIB, WANT, recs, CAP, C.byref(res)))):
                os.lseek(fd, 0, os.SEEK_SET)
                assert call() == -3, name                                   # AGB_ERR_ARG
                assert b"pread(2)" in L.agb_last_error(), (name, L.agb_last_error())
                assert os.lseek(fd, 0, os.SEEK_CUR) == len(data), name      # moved as a read to the end would have
            os.lseek(fd, 4096, os.SEEK_SET)
            t = C.c_void_p()
            assert L.agb_text_from_fd(fd, C.byref(t)) == -3
            assert b"pread(2)" in L.agb_last_error(), L.agb_last_error()
            assert os.lseek(fd, 0, os.SEEK_CUR) == 4096                     # the text was not taken: offset untouched
    finally:
        os.close(fd)
    buf = C.create_string_buffer(data, len(data))
    assert host_answer(lambda recs, res: L.agb_scan_host(p._h, buf, len(data), WANT, recs, CAP, res)) == device_answer(p, data)
