"""Hand-built DEFLATE streams for the gunzip tests: blocks of any code shape, with zlib as the judge.

zlib's encoder writes only some of the shapes a DEFLATE decoder must take: its code sets are complete, its code-length
repeats never cross from the lit/len lengths into the distance lengths, and it never sends a literal-only block with a
single distance code, as Go's compress/flate and klauspost pgzip do.  `Writer` lays out stored, fixed and dynamic blocks
bit by bit from explicit code lengths, header fields and code-length sequences (valid or not), and records the bit
offset of every block header.  Each case of `cases()` declares whether it is valid; `self_check()` holds zlib's raw
inflate to that declaration and, on valid cases, to the bytes the writer meant.

`short_segments()` builds zlib streams with a sync flush every S bytes, so that the engine's gunzip cuts them into
segments shorter than the 32 KiB window whose back-references reach across many earlier segments."""
import random
import zlib
from collections import namedtuple

from tests import gzip_corpus as gc

LBASE = [3, 4, 5, 6, 7, 8, 9, 10, 11, 13, 15, 17, 19, 23, 27, 31, 35, 43, 51, 59, 67, 83, 99, 115, 131, 163, 195, 227, 258]
LEXT = [0] * 8 + [1] * 4 + [2] * 4 + [3] * 4 + [4] * 4 + [5] * 4 + [0]
DBASE = [1, 2, 3, 4, 5, 7, 9, 13, 17, 25, 33, 49, 65, 97, 129, 193, 257, 385, 513, 769, 1025, 1537, 2049, 3073, 4097,
         6145, 8193, 12289, 16385, 24577]
DEXT = [0, 0, 0, 0, 1, 1, 2, 2, 3, 3, 4, 4, 5, 5, 6, 6, 7, 7, 8, 8, 9, 9, 10, 10, 11, 11, 12, 12, 13, 13]
CL_ORDER = [16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15]
CL_EXTRA = {16: 2, 17: 3, 18: 7}
GZIP_HEADER_BITS = 80  # gc.gzip_member with no flags: the body starts at byte 10
EMPTY_STORED = b"\x00\x00\x00\xff\xff"  # a non-final empty stored block on a byte boundary: what a flush ends with


def length_sym(n):
    """(lit/len symbol, extra bits) of a match length; 258 is symbol 285, as every encoder writes it."""
    s = 28 if n == 258 else max(k for k in range(28) if LBASE[k] <= n)
    return 257 + s, n - LBASE[s]


def dist_sym(d):
    s = max(k for k in range(30) if DBASE[k] <= d)
    return s, d - DBASE[s]


def canonical(lens):
    """{symbol: (code, length)} of the canonical Huffman code with these lengths (RFC 1951 3.2.2).  An over-subscribed
    set gets codes that overflow their length; only invalid cases write those (masked to the length)."""
    count = [0] * 16
    for n in lens:
        count[n] += 1
    count[0] = 0
    code, nxt = 0, [0] * 16
    for n in range(1, 16):
        code = (code + count[n - 1]) << 1
        nxt[n] = code
    out = {}
    for s, n in enumerate(lens):
        if n:
            out[s] = (nxt[n] & ((1 << n) - 1), n)
            nxt[n] += 1
    return out


def complete(syms, n):
    """Lengths (a list of n) of a complete code over `syms` (at least two symbols), as even as possible: with 2^(k-1) <
    len(syms) <= 2^k, 2^k - len(syms) of them get k - 1 bits and the rest k."""
    syms = sorted(syms)
    assert len(syms) >= 2
    k = (len(syms) - 1).bit_length()
    short = (1 << k) - len(syms)
    lens = [0] * n
    for i, s in enumerate(syms):
        lens[s] = k - 1 if i < short else k
    return lens


def lens_of(n, assign):
    """A list of n lengths from {symbol: length}."""
    lens = [0] * n
    for s, v in assign.items():
        lens[s] = v
    return lens


def rle(lens):
    """The code-length sequence [(symbol 0-18, extra bits or None)] of `lens`, with repeats wherever they fit."""
    out, i = [], 0
    while i < len(lens):
        v, r = lens[i], 1
        while i + r < len(lens) and lens[i + r] == v:
            r += 1
        if v == 0 and r >= 3:
            k = min(r, 138)
            out.append((18, k - 11) if k >= 11 else (17, k - 3))
            i += k
        elif v and r >= 4:
            k = min(r - 1, 6)
            out += [(v, None), (16, k - 3)]
            i += 1 + k
        else:
            out.append((v, None))
            i += 1
    return out


class Writer(gc.BitWriter):
    """DEFLATE blocks bit by bit.  `headers` holds the bit offset of every block header, `out` what the blocks are
    meant to decode to.  Block operations:
        ('lit', byte)             a literal
        ('match', length, dist)   a match, with the usual symbols (length 258: symbol 285)
        ('match284', dist)        length 258 written as symbol 284 with extra bits 31
        ('sym', s)                the lit/len code of s alone (no extra bits, no output)
        ('dsym', d)               the distance code of d alone
        ('bits', v, k)            k raw bits
        ('mark',)                 append the current bit offset to `marks`"""

    def __init__(self):
        super().__init__()
        self.buf, self.acc, self.nacc = bytearray(), 0, 0
        self.headers, self.marks, self.out = [], [], bytearray()

    def put(self, v, k):  # gc.BitWriter.put, with the finished bytes moved out of the growing integer
        self.acc |= v << self.nacc
        self.nacc += k
        self.n += k
        if self.nacc >= 4096:
            nb = self.nacc // 8
            self.buf += (self.acc & ((1 << 8 * nb) - 1)).to_bytes(nb, "little")
            self.acc >>= 8 * nb
            self.nacc -= 8 * nb

    def bytes(self):
        return bytes(self.buf) + self.acc.to_bytes((self.nacc + 7) // 8, "little")

    def _header(self, final, btype):
        self.headers.append(self.n)
        self.put(1 if final else 0, 1)
        self.put(btype, 2)

    def _align(self):
        self.put(0, -self.n % 8)

    def stored(self, data=b"", final=False, length=None, nlen=None):
        """A stored block; `length` / `nlen` override the LEN and NLEN fields."""
        self._header(final, 0)
        self._align()
        ln = len(data) if length is None else length
        self.put(ln, 16)
        self.put(ln ^ 0xFFFF if nlen is None else nlen, 16)
        if data:
            self.put(int.from_bytes(data, "little"), 8 * len(data))
        self.out += data

    def fixed(self, ops, final=False):
        self._header(final, 1)
        self._ops(ops, self.lit, lambda d: self.code(d, 5))
        self.lit(256)

    def dynamic(self, lit_lens, dist_lens, ops, final=False, cl_seq=None, cl_lens=None, hclen=None, eob=True):
        """A dynamic block.  HLIT and HDIST come from len(lit_lens) and len(dist_lens) (257-288 and 1-32, so 287, 288,
        31 and 32 write the invalid field values); cl_seq is the code-length sequence (default: rle of both sets),
        cl_lens the 19 lengths of the code-length code (default: a complete code over the symbols cl_seq uses), hclen
        the number of them sent (default: as few as hold every nonzero one)."""
        nlen, ndist = len(lit_lens), len(dist_lens)
        assert 257 <= nlen <= 288 and 1 <= ndist <= 32
        if cl_seq is None:
            cl_seq = rle(list(lit_lens) + list(dist_lens))
        if cl_lens is None:
            used = {s for s, _ in cl_seq}
            cl_lens = complete(used if len(used) > 1 else used | {0 if 0 not in used else 1}, 19)
        if hclen is None:
            hclen = max(4, max(i + 1 for i, s in enumerate(CL_ORDER) if cl_lens[s]))
        self._header(final, 2)
        self.put(nlen - 257, 5)
        self.put(ndist - 1, 5)
        self.put(hclen - 4, 4)
        for s in CL_ORDER[:hclen]:
            self.put(cl_lens[s], 3)
        cl = canonical(cl_lens)
        for s, extra in cl_seq:
            self.code(*cl[s])
            if s in CL_EXTRA:
                self.put(extra, CL_EXTRA[s])
        lc, dc = canonical(lit_lens), canonical(dist_lens)
        self._ops(ops, lambda s: self.code(*lc[s]), lambda d: self.code(*dc[d]))
        if eob:
            self.code(*lc[256])

    def _ops(self, ops, lit, dist):
        for op in ops:
            kind = op[0]
            if kind == "lit":
                lit(op[1])
                self.out.append(op[1])
            elif kind in ("match", "match284"):
                n, d = (op[1], op[2]) if kind == "match" else (258, op[1])
                s, e = length_sym(n) if kind == "match" else (284, 31)
                lit(s)
                self.put(e, LEXT[s - 257])
                ds, de = dist_sym(d)
                dist(ds)
                self.put(de, DEXT[ds])
                assert d <= len(self.out), "match before the start of the stream"
                for _ in range(n):
                    self.out.append(self.out[-d])
            elif kind == "sym":
                lit(op[1])
            elif kind == "dsym":
                dist(op[1])
            elif kind == "bits":
                self.put(op[1], op[2])
            else:
                assert kind == "mark"
                self.marks.append(self.n)


def used_syms(ops):
    """(lit/len symbols, distance symbols) the ops write, EOB included."""
    lit, dist = {256}, set()
    for op in ops:
        if op[0] == "lit":
            lit.add(op[1])
        elif op[0] in ("match", "match284"):
            lit.add(length_sym(op[1])[0] if op[0] == "match" else 284)
            dist.add(dist_sym(op[2] if op[0] == "match" else op[1])[0])
    return lit, dist


def auto_lens(ops, nlen=286, ndist=30):
    """Complete lit/len and distance sets over the symbols the ops use (distance symbols 0 or 1 added to make two)."""
    lit, dist = used_syms(ops)
    while len(dist) < 2:
        dist.add(min({0, 1} - dist))
    return complete(lit, nlen), complete(dist, ndist)


# ---- cases ---------------------------------------------------------------------------------------------------------
Case = namedtuple("Case", "name valid body data headers trailer")


def _case(name, valid, w, trailer=True):
    return Case(name, valid, w.bytes(), bytes(w.out), list(w.headers), trailer)


def member(case):
    """The gzip member of a case: the body and, unless the case is a truncated stream, the trailer of what the writer
    meant (so an invalid case fails on its DEFLATE data alone)."""
    blob = gc.gzip_member(case.body, case.data)
    return blob if case.trailer else blob[:-8]


def points(case):
    """Bit offsets of the block headers of a case's member."""
    return [GZIP_HEADER_BITS + h for h in case.headers]


def _lits(rng, n, alphabet):
    return [("lit", rng.choice(alphabet)) for _ in range(n)]


def _matches(rng, n, dists, hist, lengths=(3, 4, 10, 31, 100, 258)):
    out = []
    for _ in range(n):
        d = rng.choice(dists)
        out.append(("match", rng.choice(lengths), min(d, hist)))
    return out


def cases():
    """Every case, valid and invalid, each named for what it covers."""
    rng = random.Random(1951)
    out = []
    hist = [("lit", rng.randrange(256)) for _ in range(32768)]

    # -- valid --------------------------------------------------------------------------------------------------------
    # lit/len codes of every length 1-15: 'a'..'n' get 1..14 bits, 'o' and EOB 15; 'o' is most of the data
    ll = lens_of(286, {**{97 + i: i + 1 for i in range(14)}, 111: 15, 256: 15})
    ops = [("lit", 111 if rng.random() < 0.6 else rng.randrange(97, 111)) for _ in range(4000)]
    w = Writer()
    w.dynamic(ll, [1, 1], ops, final=True, hclen=19)
    out.append(_case("litlen_lengths_1_to_15_hclen19", True, w))

    # distance codes of every length 1-15 (symbols 0-13: 1-14 bits, 14 and 15: 15 bits), the 15-bit ones most used
    dl = lens_of(30, {**{i: i + 1 for i in range(14)}, 14: 15, 15: 15})
    pre = [("lit", rng.randrange(256)) for _ in range(300)]
    ops = pre + [("match", rng.choice((3, 7, 20, 258)),
                  rng.choice((129, 150, 192, 193, 256)) if rng.random() < 0.6 else DBASE[rng.randrange(14)])
                 for _ in range(1500)]
    w = Writer()
    w.dynamic(auto_lens(ops)[0], dl, ops, final=True)
    out.append(_case("dist_lengths_1_to_15", True, w))

    # distance 32768 (symbol 29, 13 extra bits all ones) on a 15-bit code
    dl = lens_of(30, {**{i: i + 1 for i in range(14)}, 28: 15, 29: 15})
    ops = hist + [("match", 258, 32768)] * 50 + [("match", 5, 32767), ("match", 258, 24577), ("match", 3, 1)]
    w = Writer()
    w.dynamic(auto_lens(ops)[0], dl, ops, final=True)
    out.append(_case("dist_32768_on_15bit_code", True, w))

    # length 258 both ways: symbol 285, and symbol 284 with extra bits 31; 284 with its other extra values
    ops = hist[:2000] + [("match", 258, 1000), ("match284", 1000), ("match", 258, 3), ("match284", 2000)]
    ops += [("match", 227 + e, 500) for e in range(31)]
    w = Writer()
    w.dynamic(*auto_lens(ops), ops, final=True)
    out.append(_case("len258_sym284_extra31_and_sym285", True, w))

    # Go's literal-only / Huffman-only block: one distance code of length 1 (an incomplete set), never used
    ops = _lits(rng, 3000, b"etaoin shrdlu\n")
    w = Writer()
    w.dynamic(auto_lens(ops)[0], [1], ops, final=True)
    out.append(_case("go_literal_only_one_dist_code_unused", True, w))

    # the single distance code used: symbol 0 (distance 1), and symbol 10 (distances 33-48)
    ops = _lits(rng, 50, b"abc") + [("match", rng.choice((3, 50, 258)), 1) for _ in range(40)]
    w = Writer()
    w.dynamic(auto_lens(ops)[0], [1], ops, final=True)
    out.append(_case("one_dist_code_used_sym0", True, w))
    ops = _lits(rng, 60, b"xyz") + [("match", rng.choice((3, 50, 258)), rng.randrange(33, 49)) for _ in range(40)]
    w = Writer()
    w.dynamic(auto_lens(ops)[0], lens_of(11, {10: 1}), ops, final=True)
    out.append(_case("one_dist_code_used_sym10", True, w))

    # no distance codes at all (one zero length, and thirty), literals only
    ops = _lits(rng, 500, b"0123456789")
    w = Writer()
    w.dynamic(auto_lens(ops)[0], [0], ops)
    w.dynamic(auto_lens(ops, nlen=257)[0], [0] * 30, ops, final=True)
    out.append(_case("no_dist_codes", True, w))

    # a lit/len set of EOB alone: empty dynamic blocks around data
    w = Writer()
    w.dynamic(lens_of(257, {256: 1}), [0], [])
    w.fixed(_lits(rng, 10, b"mid"))
    w.dynamic(lens_of(257, {256: 1}), [1], [], final=True)
    out.append(_case("eob_only_blocks", True, w))

    # HLIT = 286 and HDIST = 30, both complete over every symbol
    ops = hist[:5000] + _matches(rng, 400, [DBASE[k] for k in range(30)], 5000)
    w = Writer()
    w.dynamic(complete(range(286), 286), complete(range(30), 30), ops, final=True)
    out.append(_case("hlit286_hdist30_complete", True, w))

    # HCLEN = 4 (8 code-length codes sent: 16, 17, 18, 0, 8, 7, 9, 6): lit/len lengths 8 and 9 only.  (Four codes,
    # HCLEN = 0, leave only zero lengths: no EOB, refused below.)
    ops = [("lit", rng.randrange(256)) for _ in range(800)]
    w = Writer()
    w.dynamic(complete(range(257), 257), [0], ops, final=True, hclen=8)
    out.append(_case("hclen4_8_codes", True, w))

    # HCLEN = 15 (all 19 sent) where the last ones are zero
    ops = _lits(rng, 200, b"hclen")
    w = Writer()
    w.dynamic(auto_lens(ops)[0], [0], ops, final=True, hclen=19)
    out.append(_case("hclen19_trailing_zeros", True, w))

    # a repeat 16 at position nlen copies the last lit/len length (5) into the distance lengths
    ll = lens_of(265, {**{i: 9 for i in range(256)}, 256: 2, **{257 + i: 5 for i in range(8)}})
    dl = [5] * 28 + [4] * 2
    seq = rle(ll) + [(16, 3)] * 4 + [(16, 1)] + [(4, None), (4, None)]  # 24 + 4 fives, then the two fours
    ops = hist[:3000] + [("match", rng.randrange(3, 11), min(3000, DBASE[rng.randrange(30)])) for _ in range(300)]
    w = Writer()
    w.dynamic(ll, dl, ops, final=True, cl_seq=seq)
    out.append(_case("repeat16_copies_last_litlen_into_dist", True, w))

    # repeats 17 and 18 of zero lengths that run from the lit/len lengths into the distance lengths
    lit = {**{97 + i: 4 for i in range(14)}, 256: 4, 257: 4}
    ll, dl = lens_of(261, lit), lens_of(4, {2: 1, 3: 1})  # zeros: lit/len 258-260 and distance 0-1
    seq = rle(ll[:258]) + [(17, 2)] + [(1, None), (1, None)]
    ops = _lits(rng, 30, b"abcdefghijklmn") + [("match", 3, rng.choice((3, 4))) for _ in range(50)]
    w = Writer()
    w.dynamic(ll, dl, ops, cl_seq=seq)
    ll, dl = lens_of(286, lit), lens_of(12, {10: 1, 11: 1})  # zeros: lit/len 258-285 and distance 0-9
    seq = rle(ll[:258]) + [(18, 38 - 11)] + [(1, None), (1, None)]
    ops = _lits(rng, 70, b"abcdefghijklmn") + [("match", 3, rng.randrange(33, 65)) for _ in range(50)]
    w.dynamic(ll, dl, ops, final=True, cl_seq=seq)
    out.append(_case("repeat17_and_18_cross_into_dist", True, w))

    # Go's ending: a dynamic block, then an empty final stored block (01 00 00 ff ff)
    ops = _lits(rng, 400, b"go flate")
    w = Writer()
    w.dynamic(*auto_lens(ops), ops)
    w.stored(b"", final=True)
    out.append(_case("go_dynamic_then_empty_final_stored", True, w))

    # runs of empty stored blocks (Flush() with nothing pending) between data blocks
    w = Writer()
    ops = _lits(rng, 300, b"flush")
    w.dynamic(*auto_lens(ops), ops)
    for _ in range(3):
        w.stored()
    w.fixed(_lits(rng, 50, b"fixed") + [("match", 20, 7)])
    for _ in range(5):
        w.stored()
    w.stored(bytes(rng.randrange(256) for _ in range(77)))
    w.stored()
    w.stored()
    w.fixed([("match", 258, 100)], final=True)
    out.append(_case("runs_of_empty_stored_blocks", True, w))

    # stored LEN 65535, then a match that reaches back into it
    w = Writer()
    w.stored(rng.randbytes(65535))
    w.fixed([("match", 258, 32768), ("lit", 1)], final=True)
    out.append(_case("stored_len_65535", True, w))

    # a stored block after a fixed block that ends at each bit offset 0-7 (9-bit literals move the end by one bit),
    # then a dynamic block after a fixed block that ends at the same offset
    for k in range(8):
        w = Writer()

        def fixed_ending_at_k():  # from a byte boundary: 3 + 8 a + 9 b + 7 bits end at bit 2 + b (mod 8)
            w.fixed([("lit", 150 + i) for i in range((k - 2) % 8)] + [("lit", 65)] * 5)
            assert w.n % 8 == k

        fixed_ending_at_k()
        w.stored(rng.randbytes(40))
        w.stored()  # an empty stored block: the next block starts on a byte boundary again
        fixed_ending_at_k()
        ops = _lits(rng, 30, b"dyn") + [("match", 30, 45)]
        w.dynamic(*auto_lens(ops), ops)
        w.stored()
        w.fixed([("match", 30, 45)], final=True)
        out.append(_case("stored_and_dynamic_after_block_ending_at_bit%d" % k, True, w))

    # -- invalid ------------------------------------------------------------------------------------------------------
    def bad(name, build, trailer=True):
        w = Writer()
        build(w)
        out.append(_case(name, False, w, trailer))

    ab = _lits(rng, 40, b"ab")
    bad("oversubscribed_litlen", lambda w: w.dynamic(lens_of(257, {97: 1, 98: 1, 256: 1}), [0], ab, final=True))
    ops = _lits(rng, 20, b"ab") + [("match", 3, 1), ("match", 3, 2), ("match", 3, 3)]
    bad("oversubscribed_dist", lambda w: w.dynamic(auto_lens(ops)[0], [1, 1, 1], ops, final=True))
    bad("oversubscribed_codelength", lambda w: w.dynamic(
        lens_of(257, {97: 1, 256: 1}), [0], ab[:1], final=True, cl_lens=lens_of(19, {0: 1, 1: 1, 18: 1})))
    bad("incomplete_litlen_maxlen2", lambda w: w.dynamic(lens_of(257, {97: 2, 98: 2, 256: 2}), [0], ab, final=True))
    ll = lens_of(286, {**{97 + i: i + 1 for i in range(14)}, 256: 15})  # 1..14 and one 15: one 15-bit code short
    bad("incomplete_litlen_maxlen15", lambda w: w.dynamic(ll, [0], _lits(rng, 100, b"abcdefghijklmn"), final=True))
    ops = _lits(rng, 20, b"ab") + [("match", 3, 1), ("match", 3, 2), ("match", 3, 3)]
    bad("incomplete_dist_maxlen2", lambda w: w.dynamic(auto_lens(ops)[0], [2, 2, 2], ops, final=True))
    bad("incomplete_codelength_maxlen2", lambda w: w.dynamic(
        lens_of(257, {97: 1, 256: 1}), [0], ab[:1], final=True, cl_lens=lens_of(19, {0: 2, 1: 2, 18: 2})))
    bad("incomplete_codelength_single_len1", lambda w: w.dynamic(
        [1] * 257, [1], [], final=True, eob=False, cl_seq=[(1, None)] * 258, cl_lens=lens_of(19, {1: 1})))
    bad("hclen0_4_codes_no_eob", lambda w: w.dynamic(
        [0] * 257, [0], [], final=True, eob=False, cl_lens=lens_of(19, {0: 1, 18: 1}), hclen=4))
    bad("missing_eob", lambda w: w.dynamic(lens_of(257, {97: 1, 98: 1}), [0], ab, final=True, eob=False))
    for nlen in (287, 288):
        bad("hlit%d" % (nlen - 257), lambda w: w.dynamic(complete(range(nlen), nlen), [0], ab, final=True))
    ops = hist[:100] + [("match", 3, d) for d in (1, 5, 17, 65, 99)]
    for ndist in (31, 32):
        bad("hdist%d" % (ndist - 1), lambda w: w.dynamic(auto_lens(ops)[0], complete(range(ndist), ndist), ops,
                                                        final=True))
    ll = lens_of(257, {97: 1, 256: 1})
    bad("repeat16_in_first_position", lambda w: w.dynamic(
        ll, [0], ab[:1], final=True, cl_seq=[(16, 0)] + rle(ll[3:] + [0])))
    bad("repeat16_past_nlen_ndist", lambda w: w.dynamic(
        ll, [1, 1], ab[:1], final=True, cl_seq=rle(ll) + [(1, None), (16, 0)]))
    bad("repeat18_past_nlen_ndist", lambda w: w.dynamic(
        lens_of(257, {97: 1, 256: 1}), [0] * 5, ab[:1], final=True, cl_seq=rle(ll) + [(18, 0)]))
    ll = lens_of(258, {97: 1, 256: 2, 257: 2})
    bad("match_with_empty_dist_set", lambda w: w.dynamic(
        ll, [0], [("lit", 97)] * 5 + [("sym", 257), ("bits", 0, 15)], final=True))
    bad("dist_symbol_absent_from_one_code_set", lambda w: w.dynamic(
        ll, [1], [("lit", 97)] * 5 + [("sym", 257), ("bits", 1, 1)], final=True))
    for d in (30, 31):
        bad("fixed_dist_symbol_%d" % d, lambda w: w.fixed([("lit", 97)] * 40 + [("sym", 257), ("dsym", d),
                                                                                 ("bits", 0, 13)], final=True))
    bad("stored_len_nlen_mismatch", lambda w: w.stored(b"abcd", final=True, nlen=0xFFFF ^ 5))

    # a stream that ends inside a 15-bit code
    ll = lens_of(286, {**{97 + i: i + 1 for i in range(14)}, 111: 15, 256: 15})
    w = Writer()
    w.dynamic(ll, [1, 1], [("lit", 111)] * 30 + [("mark",), ("lit", 111)] + [("lit", 97)] * 30, final=True)
    p = w.marks[0]
    body = w.bytes()[:p // 8 + 1]
    assert p < 8 * len(body) < p + 15
    out.append(Case("truncated_in_15bit_code", False, body, bytes(w.out), list(w.headers), False))

    names = [c.name for c in out]
    assert len(names) == len(set(names)), "duplicate case names"
    return out


def zlib_inflate(body: bytes):
    """zlib's raw inflate of a whole DEFLATE stream: the bytes, or None where zlib reports an error or the stream does
    not end with its final block."""
    d = zlib.decompressobj(-15)
    try:
        data = d.decompress(body) + d.flush()
    except zlib.error:
        return None
    return data if d.eof and not d.unused_data else None


def self_check():
    """zlib agrees with the validity every case declares, decodes every valid case to the bytes the writer meant, and
    Go's gzip reader (gc.go_gunzip) agrees on the members; the block headers cover every bit offset class."""
    cs = cases()
    for c in cs:
        got = zlib_inflate(c.body)
        assert (got is not None) == c.valid, (c.name, "zlib says", got is not None)
        if c.valid:
            assert got == c.data, c.name
        assert gc.go_gunzip(member(c)) == (c.data if c.valid else None), c.name
    assert {h % 8 for c in cs for h in points(c)} == set(range(8))
    return cs


# ---- short segments that reference across segments and windows -------------------------------------------------------
PERIODS = (32506, 32505, 32400, 32000, 31000)  # zlib's deflate finds matches up to 32768 - 262 = 32506 bytes back


def periodic(n: int, seed: int, noise=4096) -> bytes:
    """n bytes that repeat with periods just under 32 KiB, the period changing every 256 KiB, with about one random
    byte per `noise` bytes so that matches end and restart."""
    import numpy as np
    rng = np.random.default_rng(seed)
    base = rng.integers(0, 256, 32768, dtype=np.uint8)
    piece = 256 << 10
    parts = []
    for i in range(0, n, piece):
        p = PERIODS[(i // piece) % len(PERIODS)]
        parts.append(np.resize(base[:p], min(piece, n - i)))
    d = np.concatenate(parts) if parts else np.zeros(0, np.uint8)
    k = max(1, n // noise)
    d[rng.integers(0, max(1, n), k)] = rng.integers(0, 256, k, dtype=np.uint8)
    return d.tobytes()


def short_segments(data: bytes, S: int, empty_every=0, level=6):
    """(gzip member, segments): one zlib stream with a Z_SYNC_FLUSH after every S bytes, and after every
    `empty_every`-th flush an extra empty stored block (a flush with nothing pending, as Go's Flush() writes it), which
    the gunzip decodes as a segment of no bytes.  `segments` is how many segments the flush points cut the stream into:
    one per flush and empty block, and the final block."""
    c = zlib.compressobj(level, zlib.DEFLATED, -15, 9)
    body, segs = [], 1
    for k, i in enumerate(range(0, len(data), S)):
        body.append(c.compress(data[i:i + S]) + c.flush(zlib.Z_SYNC_FLUSH))
        segs += 1
        if empty_every and k % empty_every == empty_every - 1:
            body.append(EMPTY_STORED)
            segs += 1
    body.append(c.flush())
    return gc.gzip_member(b"".join(body), data), segs


def far_short_segments(n: int, S: int, seed: int):
    """(gzip member, data, segments), hand-built: fixed blocks of S output bytes, each ended by a flush (an empty stored
    block); after the first 32 KiB of literals every block copies from exactly 32768 bytes back, the distance zlib's
    encoder never writes, so each marker reaches over 32768 / S segments."""
    rng = random.Random(seed)
    w = Writer()
    segs = 1
    while len(w.out) < n:
        ops, k = [], 0
        while k < S:
            if len(w.out) + k < 32768 or S - k < 3:
                ops.append(("lit", rng.randrange(256)))
                k += 1
            else:
                ops.append(("match", min(258, S - k), 32768))
                k += ops[-1][1]
        w.fixed(ops)
        w.stored()
        segs += 1
    w.fixed([], final=True)
    return gc.gzip_member(w.bytes(), bytes(w.out)), bytes(w.out), segs


SHORT_S = (1, 100, 4096, 32767, 32768, 32769)


def short_cases():
    """(name, blob, data, segments): zlib streams with a sync flush every S bytes for every S of SHORT_S, about 2 MiB
    (600 KB at S = 1: zlib writes no matches into 1-byte flushes anyway), and a hand-built stream of 1000-byte
    segments with distance-32768 copies.  Each fits one output window on the device and spans several in the CPU
    mock."""
    out = []
    for S in SHORT_S:
        data = periodic(600_000 if S == 1 else 2 << 20, seed=S)
        blob, segs = short_segments(data, S, empty_every=5)
        out.append(("sync_flush_every_%d" % S, blob, data, segs))
    blob, data, segs = far_short_segments(600_000, 1000, seed=2)
    out.append(("dist32768_every_1000", blob, data, segs))
    return out
