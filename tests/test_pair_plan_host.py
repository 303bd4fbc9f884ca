"""The pair plan's chunk rule, modelled on the CPU (no device needed).

Stage 1 under the pair plan cuts the pattern into k + 2 disjoint, pairwise distinct literal pieces of one length and flags
a 16-byte chunk only where some piece starts in it and some *other* piece starts in it or in the next chunk (the last two
chunks of the text are always flagged).  k errors leave two pieces verbatim, and the later one starts at most
(o_last - o_first) + k bytes after the earlier one, so the rule cannot lose a match while that is at most 16.  Here:
  * on random texts and patterns with planted matches, every record the checker (tests/_oracle.py) reports holds a chunk
    the model flags;
  * the planner's choice of pieces (a model of scan.cu's pair_pieces) and its distance bound: a match whose two
    surviving pieces are as far apart as the bound allows is still caught, one byte further it would not be, and with
    k >= len (insertions and deletions may move two pieces past each other) the rule still holds."""
import random
import pytest
import _oracle, _corpus

CHUNK, REACH = 16, 16


def fold_bytes(b, fold):
    return bytes(c | 0x20 for c in b) if fold else bytes(b)


def pair_pieces(pattern, k, fold=False):
    """scan.cu pair_pieces for a pattern of literal bytes: k + 2 pieces of 4 bytes if they fit, else 3, taken from the
    left, pairwise distinct, (o_last - o_first) + k <= REACH.  Returns [(bytes, offset)] or None."""
    pat = fold_bytes(pattern, fold)
    np_ = k + 2
    if np_ > 4:
        return None
    for ln in (4, 3):
        for s0 in range(0, len(pat) - np_ * ln + 1):
            offs = [s0 + i * ln for i in range(np_)]
            vals = [pat[o:o + ln] for o in offs]
            if offs[-1] - offs[0] + k > REACH or len(set(vals)) < np_:
                continue
            return list(zip(vals, offs))
    return None


def chunk_flags(text, pieces, fold=False):
    t = fold_bytes(text, fold)
    nch = (len(t) + CHUNK - 1) // CHUNK
    pres = [0] * (nch + 1)
    for i, (v, _) in enumerate(pieces):
        p = t.find(v)
        while p >= 0:
            pres[p // CHUNK] |= 1 << i
            p = t.find(v, p + 1)
    flags = [bool(pres[c]) and bin(pres[c] | pres[c + 1]).count("1") >= 2 for c in range(nch)]
    for c in range(max(0, nch - 2), nch):
        flags[c] = True
    return flags


def covered(flags, begin, end):
    return any(flags[c] for c in range(max(0, begin // CHUNK), min(len(flags), (end + CHUNK - 1) // CHUNK)))


def random_case(rnd, k, alphabet="abcdefgh "):
    plen = rnd.randint(3 * (k + 2), 3 * (k + 2) + 4)
    pattern = "".join(rnd.choice("abcdefgh") for _ in range(plen))
    lines = []
    for _ in range(400):
        if rnd.random() < 0.3:
            line = _corpus.mutate(rnd, pattern, rnd.randint(0, k))
            line = "".join(rnd.choice(alphabet) for _ in range(rnd.randint(0, 20))) + line + \
                "".join(rnd.choice(alphabet) for _ in range(rnd.randint(0, 20)))
        else:
            line = "".join(rnd.choice(alphabet) for _ in range(rnd.randint(0, 60)))
        lines.append(line.replace("\n", ""))
    return pattern, ("\n".join(lines) + "\n").encode()


@pytest.mark.parametrize("k", [0, 1, 2])
@pytest.mark.parametrize("seed", range(6))
def test_every_match_has_a_flagged_chunk(k, seed):
    rnd = random.Random(1000 * k + seed)
    pattern, text = random_case(rnd, k)
    pieces = pair_pieces(pattern.encode(), k)
    if pieces is None:
        pytest.skip("no pair plan for %r" % pattern)
    flags = chunk_flags(text, pieces)
    cnt, recs = _oracle.scan(_oracle.compile(pattern, k=k, linenum=1), text)
    assert cnt > 0
    for b, e, _ in recs:
        assert covered(flags, b, e), (pattern, k, b, e, text[b:e])
    # the point of the rule: it flags no chunk in which no piece starts
    t = text
    for c, f in enumerate(flags[:-2]):
        if f:
            assert any(t.find(v, c * CHUNK, c * CHUNK + CHUNK + len(v) - 1) >= 0 for v, _ in pieces)


def test_nocase_model():
    rnd = random.Random(7)
    pattern, text = random_case(rnd, 2)
    text = bytes(c - 32 if 97 <= c <= 122 and rnd.random() < 0.3 else c for c in text)
    pieces = pair_pieces(pattern.encode(), 2, fold=True)
    flags = chunk_flags(text, pieces, fold=True)
    cnt, recs = _oracle.scan(_oracle.compile(pattern, k=2, nocase=1, linenum=1), text)
    assert cnt > 0
    for b, e, _ in recs:
        assert covered(flags, b, e)


def test_headline_pieces():
    assert pair_pieces(b"because each", 2) == [(b"bec", 0), (b"aus", 3), (b"e e", 6), (b"ach", 9)]
    # long enough for four-byte pieces
    assert pair_pieces(b"governmental policy", 2) == [(b"gove", 0), (b"rnme", 4), (b"ntal", 8), (b" pol", 12)]
    # k > 2 has no pair plan (stage 1 would pay more than one IMAD per window for each extra piece)
    assert pair_pieces(b"because each of them", 3) is None
    # pieces that repeat cannot be told apart
    assert pair_pieces(b"abcabcabcabc", 2) is None


def planted(first_at, gap, p, q, fill=b"x"):
    """a line in which piece p starts at byte first_at and piece q `gap` bytes after it"""
    line = bytearray(fill * (first_at + gap + len(q) + 8))
    line[first_at:first_at + len(p)] = p
    line[first_at + gap:first_at + gap + len(q)] = q
    return bytes(line)


@pytest.mark.parametrize("span,k", [(14, 2), (13, 3), (12, 4)])
def test_distance_bound_is_tight(span, k):
    """Two pieces at the bound: (gap between their starts) = span + k = REACH is caught when the first one starts at the
    last byte of a chunk; at REACH + 1 it would not be, which is why the planner refuses such plans."""
    p, q = b"QRS", b"UVW"
    pieces = [(p, 0), (q, span)]
    for gap, ok in ((span + k, True), (span + k + 1, False)):
        text = b"\n" * 32 + planted(15, gap, p, q) + b"\n" + b"z" * 64 + b"\n"
        at = 32 + 15
        flags = chunk_flags(text, pieces)
        assert flags[at // CHUNK] == ok
    assert (span + k <= REACH) and (span + k + 1 > REACH)


def test_swapped_pieces_with_k_at_least_len():
    """With k >= len the two pieces that stay verbatim may appear in the text in the other order.  The planner never
    builds such a plan (k <= 2 < 3 <= len), but the rule does not depend on it: pieces are paired by identity, not by
    pattern order, so the earlier one in the text still flags its chunk wherever the pair sits."""
    pieces = pair_pieces(b"abcdefghijkl", 2)
    assert pieces == [(b"abc", 0), (b"def", 3), (b"ghi", 6), (b"jkl", 9)]
    for lead in range(0, 32):
        line = b"y" * lead + b"defabc" + b"y" * 20                     # "def" before "abc"
        flags = chunk_flags(b"\n" + line + b"\n" * 40, pieces)
        assert flags[(1 + lead) // CHUNK]
