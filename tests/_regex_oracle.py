"""The reference's regular-expression search -- re() (agrep.c:1267-1917) with the positions of maskgen.c and the follow
sets of follow.c -- restated in Python as an independent checker.  TEST INFRASTRUCTURE, never the product.

Restated, in 64-bit words (up to 63 positions), without the reference's defects (SURVEY 8c): every follow entry
counts (compute_next keeps ten), '?' is the optional operator.  Records are lines; an unterminated last line is closed
by the newline appended at EOF, the empty line behind a final newline is no line -- as the other engines.

compile(pattern, k, nocase, inverse) -> Regex; scan(Regex, text) -> (count, [(begin, end, ordinal), ...]) with
begin/end the offsets of the newlines around the line (-1: the virtual one in front of the text; n: the appended one)
and ordinal the j of re() (-n prints j - 1)."""


class RegexError(Exception):
    pass


ANY = frozenset(range(256))


class Regex:
    pass


def is_regex(p):
    i = 0
    while i < len(p):
        if p[i] == 0x5C:
            i += 2
            continue
        if p[i] in b"|*":
            return True
        i += 1
    return False


class _Parser:
    def __init__(self, s, nocase):
        self.s, self.i, self.nocase = s, 0, nocase
        self.cls, self.prot = [None], [False]          # position 0: the start state
        self.fol = [set()]
        self.no_error, self.even = False, 0

    def pos(self, cls, prot=False):
        self.cls.append(frozenset(cls))
        self.prot.append(prot or self.no_error)
        self.fol.append(set())
        if len(self.cls) - 1 > 63:
            raise RegexError("regular expression too long")
        return len(self.cls) - 1

    def link(self, frm, to):
        for p in frm:
            self.fol[p] |= to

    def lit(self, c):
        if c == 10:
            return self.pos({10}, True)
        if self.nocase and 65 <= c <= 90:
            c += 32
        return self.pos({c, c - 32} if self.nocase and 97 <= c <= 122 else {c})

    def klass(self):
        s = self.s
        self.i += 1
        comp = False
        if self.i < len(s) and s[self.i] == ord("^"):
            comp, self.i = True, self.i + 1
        pairs = []

        def sym():
            c = s[self.i]
            if c == 0x5C:
                self.i += 1
                return s[self.i], True
            if c in b"$^":
                return 10, False
            return c, False

        while True:
            if self.i >= len(s):
                raise RegexError("unmatched '[', ']' (use \\[, \\] to search for [, ])")
            c, esc = sym()
            if not esc and c == ord("]"):
                break
            if not esc and c == ord("-"):
                if not pairs:
                    raise RegexError("illegal regular expression")
                self.i += 1
                hi, _ = sym()
                if self.nocase and 65 <= hi <= 90:
                    hi += 32
                if hi < pairs[-1][0]:
                    raise RegexError("illegal regular expression")
                pairs[-1] = (pairs[-1][0], hi)
            elif not esc and c == ord("."):
                pairs.append(("any", "any"))
            else:
                if not esc and c in b"#()<>|*,;":
                    raise NotImplementedError("metasymbol inside a class")
                if self.nocase and 65 <= c <= 90:
                    c += 32
                pairs.append((c, c))
            self.i += 1
        if not pairs:
            raise RegexError("illegal regular expression")
        cls = set()
        for lo, hi in pairs:
            cls |= ANY if lo == "any" else set(range(lo, hi + 1))
        if comp:
            cls = set(ANY) - cls
        if self.nocase:
            for u in range(65, 91):
                cls.discard(u)
                if u + 32 in cls:
                    cls.add(u)
        self.i += 1
        return self.pos(cls)

    def atom(self):
        s, c = self.s, self.s[self.i]
        if c == ord("("):
            self.i += 1
            f = self.alt()
            if self.i >= len(s) or s[self.i] != ord(")"):
                raise RegexError("illegal regular expression")
            self.i += 1
            return f
        if c == ord("["):
            p = self.klass()
        elif c == 0x5C:
            if self.i + 1 >= len(s):
                raise RegexError("illegal regular expression")
            p = self.lit(s[self.i + 1])
            self.i += 2
        elif c in b".#":
            p = self.pos(ANY)
            self.i += 1
            if c == ord("#"):
                self.link({p}, {p})
                return [{p}, {p}, True]
        elif c in b"^$":
            p = self.pos({10}, True)
            self.i += 1
        elif c in b"*?|)],;":
            raise RegexError("illegal regular expression")
        else:
            p = self.lit(c)
            self.i += 1
        return [{p}, {p}, False]

    def cat(self):
        s, out = self.s, None
        while self.i < len(s) and s[self.i] not in b"|)":
            if s[self.i] == ord("<"):
                self.no_error, self.even, self.i = True, self.even + 1, self.i + 1
                continue
            if s[self.i] == ord(">"):
                self.no_error, self.even, self.i = False, self.even - 1, self.i + 1
                if self.even < 0:
                    raise RegexError("unmatched '<', '>' (use \\<, \\> to search for <, >)")
                continue
            f = self.atom()
            while self.i < len(s) and s[self.i] in b"*?":
                if s[self.i] == ord("*"):
                    self.link(f[1], f[0])
                f = [f[0], f[1], True]
                self.i += 1
            if out is None:
                out = f
            else:
                self.link(out[1], f[0])
                out = [out[0] | (f[0] if out[2] else set()), f[1] | (out[1] if f[2] else set()), out[2] and f[2]]
        if out is None:
            raise RegexError("illegal regular expression")
        return out

    def alt(self):
        out = self.cat()
        while self.i < len(self.s) and self.s[self.i] == ord("|"):
            self.i += 1
            f = self.cat()
            out = [out[0] | f[0], out[1] | f[1], out[2] or f[2]]
        return out


def compile(pattern, k=0, nocase=False, inverse=False):
    if isinstance(pattern, str):
        pattern = pattern.encode("latin-1")
    if k > 4:
        raise RegexError("the maximum number of erorrs allowed for full regular expressions is 4")
    P = _Parser(pattern, nocase)
    lead = P.pos(ANY)
    first, last, nullable = P.alt()
    if P.i < len(pattern):
        raise RegexError("illegal regular expression")
    if P.even:
        raise RegexError("unmatched '<', '>' (use \\<, \\> to search for <, >)")
    trail = P.pos(ANY)
    M = trail
    P.fol[0] = {lead}
    P.fol[lead] |= first | ({trail} if nullable else set())
    P.link(last, {trail})
    bit = lambda p: 1 << (M - p)
    a = Regex()
    a.M, a.k, a.inverse = M, k, bool(inverse)
    a.follow = [sum(bit(q) for q in P.fol[p]) for p in range(M + 1)]
    a.mask = [0] * 256
    for p in range(1, M + 1):
        for c in P.cls[p]:
            a.mask[c] |= bit(p)
    a.noerr = ~sum(bit(p) for p in range(1, M + 1) if P.prot[p]) & ((1 << 64) - 1)
    a.init0 = (1 << M) | bit(1)
    a.init1 = a.init0 | 1
    # byte-sliced Next, as compute_next's table (any slicing gives the same union)
    fb = [a.follow[M - b] if b <= M else 0 for b in range(64)]
    a.tab = [[0] * 256 for _ in range(8)]
    for s in range(8):
        for v in range(1, 256):
            low = v & -v
            a.tab[s][v] = a.tab[s][v ^ low] | fb[8 * s + low.bit_length() - 1]
    init = [a.init0]
    for _ in range(k):
        init.append(init[-1] | _next(a, init[-1]))
    a.reset = _step(a, tuple(init), a.mask[10])
    a.cache = {}
    return a


def _next(a, S):
    t, r, s = a.tab, 0, 0
    while S:
        r |= t[s][S & 0xFF]
        S >>= 8
        s += 1
    return r


def _step(a, B, cm):
    A = [(_next(a, B[0]) & cm) | (a.init1 & B[0])]
    for j in range(1, len(B)):
        A.append((_next(a, B[j]) & cm) | (a.init1 & B[j]) | ((B[j - 1] | _next(a, A[j - 1] | B[j - 1])) & a.noerr))
    return tuple(A)


def _matches(a, S):
    t = (_next(a, S[-1]) & a.mask[10]) | (a.init1 & S[-1])
    t |= _next(a, t)                                                     # TAIL
    return bool(t & 1) != a.inverse


def scan(a, text, want_records=True):
    n = len(text)
    cache = a.cache
    count, recs = 0, []
    begin, j = -1, 1                                                     # the virtual '\n' is close number 1
    while begin + 1 < n:
        end = text.find(b"\n", begin + 1)
        if end < 0:
            end = n
        S = a.reset
        for c in text[begin + 1:end]:
            key = (S, c)
            nxt = cache.get(key)
            if nxt is None:
                nxt = cache[key] = _step(a, S, a.mask[c])
            S = nxt
        j += 1
        if _matches(a, S):
            count += 1
            if want_records:
                recs.append((begin, end, j))
        begin = end
    return count, recs
