"""Windowed scans (agb_scan_host_windowed / agb_scan_fd_windowed, and agb_scan_host / agb_scan_fd falling back to windows
when a text does not fit): at most one window of text plus its halos on the device at a time, the same answer as the
whole-text scan -- counts, level histogram, delimiter total, truncation and the ordered record list with global offsets,
ordinals and levels.  Each window is scanned as a shard of the whole text (the cut rule of tests/test_gpu_shard.py);
halos too short for a long record or a long run of the delimiter are doubled until they suffice.  Small texts are also
checked against the checkers (tests/_oracle.py, tests/_regex_oracle.py)."""
import ctypes as C
import os, subprocess, threading
import pytest
import _oracle, _corpus
import _regex_oracle as R
import agrep_b200 as ag
from agrep_b200 import _lib

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KIB, MIB = 1 << 10, 1 << 20


@pytest.fixture(scope="module")
def plain():
    return ag.corpus_host(8 * MIB, needle="because each", needle_every=16, needle_maxedits=3)


@pytest.fixture(scope="module")
def para():
    return ag.corpus_host(8 * MIB, seed=7, paragraphs=True, needle="world", needle_every=8, needle_maxedits=1)


@pytest.fixture(scope="module")
def big():
    return ag.corpus_host(64 * MIB, seed=99, needle="because each", needle_every=64, needle_maxedits=3)


@pytest.fixture(scope="module")
def aba():
    return b"".join(_corpus.overlap_text("aba", s) for s in range(1, 41))


def rows(recs):
    return [tuple(r) for r in recs]


def same(p, data, window, **kw):
    """the windowed scan equals the whole-text scan, field by field; returns the whole-text answer"""
    r0, l0 = p.scan_host(data, **kw)
    r1, l1 = p.scan_host(data, window=window, **kw)
    key = (window, len(data), kw)
    assert (r1.n_matched, list(r1.level_hist), r1.n_closes, r1.truncated, r1.n_records) == \
           (r0.n_matched, list(r0.level_hist), r0.n_closes, r0.truncated, r0.n_records), key
    assert rows(l1) == rows(l0), key
    return r0, l0


# (corpus, pattern, Pattern keywords, scan keywords): every engine, the switches, the delimiter kinds, a regex with levels
CASES = [
    ("plain", "because each", dict(k=0, linenum=1), dict(ordinals=True)),                       # bitap
    ("plain", "government", dict(), dict()),                                                    # sgrep / bm
    ("plain", "the", dict(), dict(want_records=False)),                                         # exact count path
    ("plain", "because each", dict(k=2, linenum=1), dict(ordinals=True)),                       # asearch
    ("plain", "governmental", dict(k=6, linenum=1), dict(ordinals=True, levels=True)),          # asearch0
    ("plain", "between both", dict(k=2, cost_s=2, linenum=1), dict(ordinals=True)),             # asearch1
    ("plain", "the", dict(k=1, wordbound=1, linenum=1), dict(ordinals=True)),                   # -w
    ("plain", "the state", dict(k=4, wholeline=1, linenum=1), dict(ordinals=True)),             # -x
    ("plain", "Government", dict(k=1, nocase=1, linenum=1), dict(ordinals=True)),               # -i
    ("plain", "the", dict(k=1, inverse=1, linenum=1), dict(ordinals=True)),                     # -v list
    ("plain", "people", dict(inverse=1), dict(want_records=False)),                             # -c -v (complement shortcut)
    ("plain", "gov#ent", dict(k=1, linenum=1), dict(ordinals=True)),                            # '#'
    ("plain", "gvrnmnt", dict(ins_free=1, k=1, linenum=1), dict(ordinals=True)),                # -p
    ("para", "world", dict(k=1, wordbound=1, linenum=1, delim="$$"), dict(ordinals=True)),      # -d '$$'
    ("aba", "state", dict(k=1, linenum=1, delim="aba"), dict(ordinals=True)),                   # -d aba
    ("plain", "state", dict(k=1, nocase=1, linenum=1, delim="W"), dict(ordinals=True)),         # -i -d X
    ("plain", "gov(ern)*ment|(each|both) (st|wo)", dict(k=2, regex=True), dict(ordinals=True, levels=True)),
]


@pytest.mark.parametrize("window", [4 * KIB, 64 * KIB, 1 * MIB])
@pytest.mark.parametrize("corpus,pattern,kw,skw", CASES)
def test_engines_and_options(request, window, corpus, pattern, kw, skw):
    data = request.getfixturevalue(corpus)
    r0, _ = same(ag.Pattern(pattern, **kw), data, window, **skw)
    assert r0.n_matched > 0 or kw.get("wholeline")


@pytest.mark.parametrize("window", [64 * KIB, 1 * MIB])
def test_64mib_corpus(big, window):
    same(ag.Pattern("because each", k=2, linenum=1), big, window, ordinals=True)
    same(ag.Pattern("the", k=1, inverse=1), big, window, want_records=False, levels=True)


def oracle_rows(pattern, kw, data):
    a = _oracle.compile(pattern, **kw)
    cnt, recs = _oracle.scan(a, data)
    return cnt, list(recs)


def with_oracle(pattern, kw, data, window, keep=lambda t: t):
    """whole-text scan, windowed scan and the checker agree (begin, end, ordinal)"""
    p = ag.Pattern(pattern, **kw)
    r0, l0 = same(p, data, window, ordinals=True)
    cnt, recs = oracle_rows(pattern, kw, data)
    assert r0.n_matched == cnt
    assert [keep(r[:3]) for r in rows(l0)] == [keep(r) for r in recs]
    return cnt


def put(data, pos, s):
    return data[:pos] + s + data[pos + len(s):]


def test_small_texts_against_the_checkers():
    data = _corpus.make_text(3000, seed=21)
    for pattern, kw in (("because each", dict(k=2, linenum=1)), ("the", dict(k=0, linenum=1, inverse=1)),
                        ("governmental", dict(k=3, nocase=1, linenum=1))):
        assert with_oracle(pattern, kw, data, 4 * KIB) > 0
    for K in (0, 2):
        pat = "(each|both) (st|wo)"
        cnt, recs = R.scan(R.compile(pat, k=K), data)
        res, got = ag.Pattern(pat, k=K, regex=True).scan_host(data, window=4 * KIB, ordinals=True)
        assert res.n_matched == cnt > 0 and [r[:3] for r in rows(got)] == list(recs)


def test_edges_after_a_delimiter_and_inside_dollar_dollar():
    w = 4 * KIB
    data = _corpus.make_text(4000, seed=22, paragraphs=True)
    nl, dd = data, data
    for i, e in enumerate(range(w, len(data) - 8, w)):
        nl = put(nl, e - 1, b"\n")                  # the edge falls right after a newline
        dd = put(dd, e - 1 - (i % 3 == 0), b"\n\n")   # between the two bytes of "$$", or right after it
    assert with_oracle("the", dict(k=1, linenum=1), nl, w) > 0
    assert with_oracle("world", dict(k=1, linenum=1, delim="$$"), dd, w) > 0
    assert with_oracle("world", dict(k=0, linenum=1, delim="$$", inverse=1), dd, w) > 0


def test_an_edge_inside_a_run_of_2000_newlines_grows_the_left_halo():
    w = 4 * KIB
    head = _corpus.make_text(300, seed=23, paragraphs=True)
    tail = b"world of the people\n" + _corpus.make_text(300, seed=24, paragraphs=True)
    for shift in (0, 1, 700, 1999):                  # bytes of the run in front of the window edge (> 512: the left halo grows)
        pad = (-(len(head) + shift)) % w
        d = head + b"x" * pad + b"\n" * 2000 + tail
        assert (len(head) + pad + shift) % w == 0
        assert with_oracle("world", dict(k=1, linenum=1, delim="$$"), d, w) > 0
        assert with_oracle("people", dict(k=0, linenum=1, delim="$$", inverse=1), d, w) > 0


def test_a_3mib_record_grows_the_right_halo_over_many_windows():
    rec = b"because each " + b"z" * (3 * MIB) + b" government"
    data = _corpus.make_text(500, seed=25) + rec + b"\n" + _corpus.make_text(500, seed=26)
    for window in (4 * KIB, 64 * KIB):
        assert with_oracle("because each", dict(k=1, linenum=1), data, window) > 0
        assert with_oracle("government", dict(k=0, linenum=1), data, window) > 0


def test_a_300kib_regex_line_grows_the_right_halo():
    line = b"the government " + b"q" * (300 * KIB) + b" state of the world"
    data = _corpus.make_text(800, seed=27) + line + b"\n" + _corpus.make_text(800, seed=28)
    pat = "gov(ern)*ment|sta(t|x)e"
    for K in (0, 2):
        p = ag.Pattern(pat, k=K, regex=True)
        r0, l0 = same(p, data, 4 * KIB, ordinals=True, levels=True)
        cnt, recs = R.scan(R.compile(pat, k=K), data)
        assert r0.n_matched == cnt > 0 and [r[:3] for r in rows(l0)] == list(recs)


@pytest.mark.parametrize("name", ["unterminated", "starts_with_delimiter", "empty", "shorter_than_a_window", "exact_multiple"])
def test_text_and_window_sizes(name):
    w = 4 * KIB
    base = _corpus.make_text(900, seed=29)
    if name == "unterminated":
        data, pat, kw = base + b"because each of them", "because each", dict(k=1, linenum=1)
    elif name == "starts_with_delimiter":
        data, pat, kw = b"; " + base.replace(b"\n", b"; "), "world", dict(k=1, linenum=1, delim="; ")
    elif name == "empty":
        data, pat, kw = b"", "the", dict(linenum=1)
    elif name == "shorter_than_a_window":
        data, pat, kw = base[:3000], "the", dict(k=1, linenum=1)
    else:
        data, pat, kw = base[:(len(base) // w) * w], "because each", dict(k=2, linenum=1)
        assert len(data) % w == 0 and len(data) > 4 * w
    cnt = with_oracle(pat, kw, data, w)
    assert cnt > 0 or name == "empty"


def test_truncation(plain):
    p = ag.Pattern("the", k=1, linenum=1)
    r0, l0 = p.scan_host(plain, ordinals=True)
    cap = r0.n_matched // 3
    for window in (4 * KIB, 1 * MIB):
        r1, l1 = p.scan_host(plain, capacity=cap, window=window, ordinals=True)
        assert r1.truncated == 1 and r1.n_matched == r0.n_matched and r1.n_records == cap
        assert rows(l1) == rows(l0)[:cap]
        assert list(r1.level_hist) == list(r0.level_hist) and r1.n_closes == r0.n_closes


def test_scan_fd_windowed_on_a_file_at_an_offset_and_on_a_pipe(tmp_path, plain):
    path = str(tmp_path / "text")
    open(path, "wb").write(plain)
    p = ag.Pattern("because each", k=2, linenum=1)
    skip = 12345
    r0, l0 = p.scan_host(plain[skip:], ordinals=True)
    for window in (None, 64 * KIB):
        fd = os.open(path, os.O_RDONLY)
        try:
            os.lseek(fd, skip, os.SEEK_SET)
            r1, l1 = p.scan_fd(fd, ordinals=True, window=window)
            assert os.lseek(fd, 0, os.SEEK_CUR) == len(plain)           # where agb_scan_fd leaves it: EOF
        finally:
            os.close(fd)
        assert (r1.n_matched, r1.n_closes, r1.truncated) == (r0.n_matched, r0.n_closes, 0) and rows(l1) == rows(l0)
    rd, wr = os.pipe()

    def feed():
        view = memoryview(plain)[skip:]
        while len(view):
            view = view[os.write(wr, view[:MIB]):]
        os.close(wr)
    t = threading.Thread(target=feed)
    t.start()
    try:
        r2, l2 = p.scan_fd(rd, capacity=r0.n_matched + 10, ordinals=True, window=64 * KIB)
    finally:
        t.join()
        os.close(rd)
    assert (r2.n_matched, r2.n_closes) == (r0.n_matched, r0.n_closes) and rows(l2) == rows(l0)


def test_text_resident_refuses_above_the_cap(monkeypatch, tmp_path):
    monkeypatch.setenv("AGB_MAX_TEXT_BYTES", str(64 * KIB))
    L = _lib.lib()
    data = _corpus.make_text(3000, seed=30)
    t = C.c_void_p()
    buf = C.create_string_buffer(data, len(data))
    assert L.agb_text_from_host(buf, len(data), C.byref(t)) == -4 and b"AGB_MAX_TEXT_BYTES" in L.agb_last_error()
    path = str(tmp_path / "t")
    open(path, "wb").write(data)
    fd = os.open(path, os.O_RDONLY)
    try:
        assert L.agb_text_from_fd(fd, C.byref(t)) == -4
        assert os.lseek(fd, 0, os.SEEK_CUR) == 0                    # untouched: the caller reads the file another way
        # agb_scan_host / agb_scan_fd take such a text in windows
        p = ag.Pattern("because each", k=2, linenum=1)
        k0 = L.agb_kernel_launches()
        r1, l1 = p.scan_fd(fd, ordinals=True)
        windowed_launches = L.agb_kernel_launches() - k0
        r2, l2 = p.scan_host(data, ordinals=True)
    finally:
        os.close(fd)
    monkeypatch.delenv("AGB_MAX_TEXT_BYTES")
    k0 = L.agb_kernel_launches()
    r0, l0 = p.scan_host(data, ordinals=True)
    whole_launches = L.agb_kernel_launches() - k0
    assert r1.n_matched == r2.n_matched == r0.n_matched > 0 and rows(l1) == rows(l2) == rows(l0)
    assert windowed_launches > 10 * whole_launches          # 4 KiB windows (the smallest): dozens of them
    assert L.agb_text_from_host(buf, len(data), C.byref(t)) == 0
    L.agb_text_free(t)


CLI = os.path.join(ROOT, "agrep_b200", "agrep-b200")
DROP = os.path.join(ROOT, "oracle", "_ref", "agrep_dropin")


@pytest.fixture(scope="module")
def file_256mib(tmp_path_factory):
    path = str(tmp_path_factory.mktemp("agb_win_") / "big.txt")
    with open(path, "wb") as f:
        for i in range(4):
            f.write(ag.corpus_host(64 * MIB, first_page=i * (64 * MIB // 4096), needle="because each", needle_every=64, needle_maxedits=3))
    yield path
    os.unlink(path)


def run_both(binary, args, path):
    """stdout, stderr and exit status without the knob, and with AGB_MAX_TEXT_BYTES = 16 MiB (windows of 8 MiB)"""
    env = dict(os.environ)
    env.pop("AGB_MAX_TEXT_BYTES", None)
    out = []
    for cap in (None, str(16 * MIB)):
        if cap:
            env["AGB_MAX_TEXT_BYTES"] = cap
        p = subprocess.run([binary] + args + [path], capture_output=True, timeout=600, stdin=subprocess.DEVNULL, env=env)
        out.append((p.returncode, p.stdout, p.stderr))
    return out


@pytest.mark.parametrize("args", [["-c", "the"], ["-n", "because each"], ["-2", "-n", "because each"], ["-B", "-y", "goverment of the peple"]])
def test_knob_end_to_end_cli(file_256mib, args):
    if not os.path.exists(CLI):
        pytest.skip("agrep-b200 not built")
    whole, windowed = run_both(CLI, args, file_256mib)
    assert windowed == whole and len(whole[1]) > 2          # (the exit status is agrep's: the match count, modulo 256)


@pytest.mark.parametrize("args", [["-c", "the"], ["-n", "because each"]])
def test_knob_end_to_end_dropin(file_256mib, args):
    if not os.path.exists(DROP):
        pytest.skip("oracle/_ref binaries not built")
    whole, windowed = run_both(DROP, ["-V0"] + args, file_256mib)
    assert windowed == whole and len(whole[1]) > 2


def test_4gib_with_512mib_windows():
    """the headline query (`agrep -2 'because each'`, list and ordinals) over a 4 GiB host copy of the synthetic corpus"""
    n = 4 << 30
    L = _lib.lib()
    spec = ag.corpus_spec(n, needle="because each", needle_every=4096, needle_maxedits=3)
    buf = (C.c_char * n)()
    assert L.agb_corpus_fill_host(C.byref(spec), buf) == 0
    p = ag.Pattern("because each", k=2)
    cap = 1 << 21
    want = _lib.WANT_RECORDS | _lib.WANT_ORDINALS
    out = []
    for window in (None, 512 * MIB):
        recs, res = (_lib.Record * cap)(), _lib.Result()
        rc = (L.agb_scan_host(p._h, buf, n, want, recs, cap, C.byref(res)) if window is None else
              L.agb_scan_host_windowed(p._h, buf, n, window, want, recs, cap, C.byref(res)))
        assert rc == 0, L.agb_last_error()
        assert res.truncated == 0 and res.n_matched > 10000
        out.append((res.n_matched, res.n_closes, list(res.level_hist), C.string_at(C.addressof(recs), res.n_records * C.sizeof(_lib.Record))))
        del recs
    assert out[1] == out[0]
