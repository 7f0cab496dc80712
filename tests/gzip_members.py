"""Multi-member gzip blobs for the gunzip tests (bgzip / BGZF, eStargz, concatenated members), built with zlib, and the
helpers that drive an engine over them.  Expectations always come from `gzip_corpus.go_gunzip`."""
import ctypes as C
import io
import random
import struct
import tarfile
import zlib

from tests import gzip_corpus as gc

CAND_FLUSH, CAND_MEMBER = 1, 2  # candidate kinds of mksnap_inflate_core.h
BGZF_BLOCK = 0xFF00             # input bytes per BGZF member (what bgzip writes)
BGZF_EOF = bytes.fromhex("1f8b08040000000000ff0600424302001b0003000000000000000000")


def bgzf_member(data: bytes, level=6) -> bytes:
    """One BGZF block: FEXTRA with the `BC` subfield holding the block size minus one."""
    body = gc.deflate(data, level)
    bsize = 10 + 2 + 6 + len(body) + 8
    extra = b"BC" + struct.pack("<HH", 2, bsize - 1)
    return gc.gzip_member(body, data, flags=4, extra=extra)


def bgzf(data: bytes, block=BGZF_BLOCK, level=6, eof=True) -> bytes:
    out = [bgzf_member(data[i:i + block], level) for i in range(0, len(data), block)]
    return b"".join(out) + (BGZF_EOF if eof else b"")


def estargz(tar: bytes, chunk=4 << 20, level=6, toc_name="stargz.index.json") -> bytes:
    """eStargz-shaped: one member per tar entry (header and the first chunk of its data), one more per further `chunk`
    bytes of a large file, then a TOC entry, the end-of-archive blocks and an empty footer member with an FEXTRA."""
    tf = tarfile.open(fileobj=io.BytesIO(tar))
    cuts = set()
    for m in tf.getmembers():
        cuts.add(m.offset)
        for o in range(m.offset_data + chunk, m.offset_data + m.size, chunk):
            cuts.add(o)
    end = max(m.offset_data + -(-m.size // 512) * 512 for m in tf.getmembers()) if tf.getmembers() else 0
    toc = b'{"version":1,"entries":[%s]}' % b",".join(b'{"name":"%s"}' % m.name.encode() for m in tf.getmembers())
    buf = io.BytesIO()
    with tarfile.open(fileobj=buf, mode="w", format=tarfile.PAX_FORMAT) as t2:
        ti = tarfile.TarInfo(toc_name)
        ti.size, ti.mtime = len(toc), 1_500_000_000
        t2.addfile(ti, io.BytesIO(toc))
    stream = tar[:end] + buf.getvalue()  # the TOC entry, then the end-of-archive blocks
    cuts = sorted(c for c in cuts if 0 < c < end) + [end, end + len(buf.getvalue()) - 1024]
    out, prev = [], 0
    for c in cuts + [len(stream)]:
        if c > prev:
            piece = stream[prev:c]
            out.append(gc.gzip_member(gc.deflate(piece, level), piece))
            prev = c
    footer_extra = b"SG" + struct.pack("<H", 22) + (b"%016xSTARGZ" % (len(b"".join(out)) - 1))
    out.append(gc.gzip_member(gc.deflate(b""), b"", flags=4, extra=footer_extra))
    return b"".join(out)


def concat_flags(rng: random.Random, data: bytes, n=40) -> bytes:
    """Members of every header-flag combination (FTEXT, FHCRC, FEXTRA, FNAME, FCOMMENT, reserved bits), some empty."""
    flag_sets = list(range(32)) + [0x20, 0x40, 0x80, 0xFF & ~0xC0]
    out, pos = [], 0
    for i in range(n):
        f = flag_sets[i % len(flag_sets)]
        k = 0 if i % 7 == 3 else rng.randint(1, 9000)
        d = data[pos:pos + k]
        pos = (pos + k) % max(1, len(data) - 10_000)
        out.append(gc.gzip_member(gc.deflate(d, rng.choice([0, 1, 6, 9])), d, flags=f,
                                  extra=bytes(rng.randrange(256) for _ in range(rng.randint(0, 40))),
                                  name=b"f%d.tar" % i, comment=b"c" * rng.randint(0, 100), mtime=rng.randrange(1 << 32)))
    return b"".join(out)


def false_candidates(rng: random.Random, data: bytes) -> bytes:
    """Members whose compressed data holds `1f 8b 08` headers: stored blocks of whole gzip members (their bodies
    decode cleanly from the false start), headers with every flag, and a dynamic-Huffman member around them."""
    inner = b"".join(gc.gzip_member(gc.deflate(data[i:i + 3000]), data[i:i + 3000], flags=f, extra=b"ab",
                                    name=b"n", comment=b"c") for i, f in zip(range(0, 30_000, 3000), (0, 4, 8, 16, 2, 31)))
    wall = b"".join(b"\x1f\x8b\x08" + bytes([f]) + bytes(6) + (b"\x02\x00xy" if f & 4 else b"") for f in range(32)) * 20
    pieces = [inner, wall, data[:20_000] + inner + data[20_000:40_000]]
    out = []
    for i, p in enumerate(pieces):
        out.append(gc.gzip_member(gc.deflate(p, 0), p))
        out.append(gc.gzip_member(gc.deflate(p, 6), p, flags=8, name=b"x%d" % i))
    return b"".join(out)


def with_flushes(data: bytes) -> bytes:
    """Members that also carry sync / full flushes: both kinds of candidate in one member."""
    return (gc.pgzip(data[:200_000], block=30_000) + gc.flushed([data[i:i + 25_000] for i in range(0, 100_000, 25_000)])
            + gc.pgzip(data[200_000:260_000], block=16_000, level=1)
            + gc.flushed([data[:9000], data[9000:20_000]], flush=zlib.Z_SYNC_FLUSH))


def stored_member(n: int, seed=0) -> bytes:
    """A member of exactly 23 + n bytes (one stored block), for placing the next header at a chosen offset."""
    d = random.Random(seed).randbytes(n)
    return gc.gzip_member(b"\x01" + struct.pack("<HH", n, n ^ 0xFFFF) + d, d)


def straddling(data: bytes, chunk=4096):
    """(name, blob): a member header that starts a few bytes before a multiple of `chunk` (the scan's chunk), with and
    without FEXTRA / FNAME, so that its magic, its fields or its body start fall on either side of the edge."""
    out = []
    for back in (1, 2, 3, 5, 9, 10, 11, 12, 17, 40):
        for flags, extra, name in ((0, b"", b""), (4, b"BC\x02\x00\x00\x00", b""), (12, b"x" * 30, b"name.tar")):
            second = gc.gzip_member(gc.deflate(data[:5000]), data[:5000], flags=flags, extra=extra, name=name)
            third = gc.gzip_member(gc.deflate(data[5000:9000]), data[5000:9000])
            for edge in (chunk, 2 * chunk):
                first = stored_member(edge - back - 23, seed=back)
                out.append(("straddle_%d_f%d_at%d" % (back, flags, edge), first + second + third))
    return out


def malformed(data: bytes):
    """(name, blob) pairs that Go's reader refuses, and one it accepts, on multi-member blobs."""
    ms = [bgzf_member(data[i:i + 7000]) for i in range(0, 70_000, 7000)]
    good = b"".join(ms)
    out = [("trailing_garbage", good + b"garbage!"), ("zero_padding", good + bytes(512)),
           ("trailing_magic", good + b"\x1f\x8b"), ("truncated_last_header", good + ms[0][:14]),
           ("truncated_last_body", good + ms[0][:40]), ("eof_then_garbage", good + BGZF_EOF + b"\x00")]
    for k in (0, 4, 9):
        bad = bytearray(ms[k])
        bad[-6] ^= 0x10  # CRC-32 of member k of 10
        out.append(("bad_crc_member_%d" % k, b"".join(ms[:k]) + bytes(bad) + b"".join(ms[k + 1:])))
        bad = bytearray(ms[k])
        bad[-2] ^= 1     # ISIZE
        out.append(("bad_isize_member_%d" % k, b"".join(ms[:k]) + bytes(bad) + b"".join(ms[k + 1:])))
    bad_hcrc = bytearray(gc.gzip_member(gc.deflate(data[:500]), data[:500], flags=2))
    bad_hcrc[4] ^= 1
    out.append(("bad_hcrc_member_2", ms[0] + ms[1] + bytes(bad_hcrc) + ms[2]))
    return out


def header_wall(n: int) -> bytes:
    """A level-0 member whose stored data is a wall of valid member headers (10 to 14 bytes each, all flag layouts
    whose fields fit), so that nearly every header's body start is a candidate."""
    hs = [b"\x1f\x8b\x08\x00" + bytes(6), b"\x1f\x8b\x08\x04" + bytes(6) + b"\x02\x00BC",
          b"\x1f\x8b\x08\x08" + bytes(6) + b"a\x00", b"\x1f\x8b\x08\x18" + bytes(6) + b"\x00\x00"]
    h2 = bytearray(b"\x1f\x8b\x08\x02" + bytes(6))
    h2 += struct.pack("<H", zlib.crc32(bytes(h2)) & 0xFFFF)
    hs.append(bytes(h2))
    pat = bytearray()
    i = 0
    while len(pat) < n:
        pat += hs[i % len(hs)]
        i += 1
    pat = bytes(pat[:n])
    return gc.gzip_member(gc.deflate(pat, 0), pat), pat


def fuzz_cases(n: int, seed=5):
    """Truncated, bit-flipped, spliced and member-swapped variants of small multi-member blobs."""
    rng = random.Random(seed)
    d = gc.mixed(rng, 40_000)
    seeds = [bgzf(d, block=4000), bgzf(d[:9000], block=3000, level=0, eof=False), concat_flags(rng, d, 8),
             gc.pgzip(d[:10_000], block=3000) + bgzf(d[10_000:20_000], block=2500), false_candidates(rng, d[:8000])]
    spans = {s: member_spans(s) for s in seeds}
    out = []
    for _ in range(n):
        s = rng.choice(seeds)
        b = bytearray(s)
        k = rng.random()
        if k < 0.45:  # members dropped, repeated and reordered, sometimes then damaged once
            ms = [s[a:z] for a, z in spans[s]]
            ms = [rng.choice(ms) for _ in range(rng.randint(1, len(ms) + 2))]
            b = bytearray(b"".join(ms))
            if k < 0.15:
                b[rng.randrange(len(b))] ^= 1 << rng.randrange(8)
        elif k < 0.6:
            b = b[:rng.randrange(len(b))]
        elif k < 0.7:  # splice: a piece of one seed into another
            o = rng.choice(seeds)
            a = rng.randrange(len(o))
            p = rng.randrange(len(b))
            b[p:p] = o[a:a + rng.randint(1, 200)]
        else:
            for _ in range(rng.randint(1, 4)):
                p = rng.randrange(len(b))
                b[p] ^= 1 << rng.randrange(8)
            if k > 0.9:
                b = b[:rng.randrange(len(b))]
        out.append(bytes(b))
    return out


def member_spans(blob: bytes):
    """(header start, trailer end) of every member of a blob Go's reader accepts."""
    out, off = [], 0
    while off < len(blob):
        p = gc._header_end(blob, off)
        d = zlib.decompressobj(-15)
        d.decompress(blob[p:])
        end = len(blob) - len(d.unused_data) + 8
        out.append((off, end))
        off = end
    return out


def member_bodies(blob: bytes):
    """Body start of every member of a blob Go's reader accepts."""
    return [gc._header_end(blob, a) for a, _ in member_spans(blob)]


def cases():
    """(name, blob) pairs of the CPU and GPU tests."""
    rng = random.Random(1996)
    data = gc.mixed(rng, 600_000)
    out = [("bgzf", bgzf(data)), ("bgzf_no_eof", bgzf(data[:300_000], eof=False)),
           ("bgzf_level0", bgzf(data[:200_000], level=0)), ("bgzf_level1_small_blocks", bgzf(data, block=5000, level=1)),
           ("bgzf_eof_only", BGZF_EOF), ("bgzf_two_eofs", bgzf(data[:100_000]) + BGZF_EOF)]
    buf = io.BytesIO()
    with tarfile.open(fileobj=buf, mode="w", format=tarfile.PAX_FORMAT) as tf:
        for i, d in enumerate([data[:300_000], b"", rng.randbytes(70_000), data[300_000:301_000]]):
            ti = tarfile.TarInfo("usr/lib/f%d" % i)
            ti.size, ti.mtime = len(d), 1_500_000_000
            tf.addfile(ti, io.BytesIO(d))
    out += [("estargz", estargz(buf.getvalue(), chunk=65536)), ("estargz_big_chunks", estargz(buf.getvalue()))]
    out += [("concat_flags", concat_flags(rng, data)), ("empty_members", gc.gzip_member(gc.deflate(b""), b"") * 30),
            ("cat_gz", gc.gzip_member(gc.deflate(data[:100_000], 9), data[:100_000])
             + gc.gzip_member(gc.deflate(data[100_000:], 1), data[100_000:]))]
    out += [("false_candidates", false_candidates(rng, data)), ("with_flushes", with_flushes(data))]
    out += straddling(data)
    out += malformed(data)
    return out


# ---- driving an engine ----------------------------------------------------------------------------------------------
class GunzipTimes(C.Structure):
    _fields_ = [("ms_scan", C.c_float), ("ms_count", C.c_float), ("ms_write", C.c_float), ("ms_resolve", C.c_float),
                ("ms_crc", C.c_float), ("extra_decodes", C.c_uint32)]


def engine_gunzip_times(lib, h, blob: bytes, chunk=1 << 20):
    """(rc, bytes, info, extra_decodes) as gc.engine_gunzip, with the extra decodes of the open."""
    info = gc.GunzipInfo()
    rc = lib.mksnap_gunzip_open(h, blob, len(blob), C.byref(info))
    if rc:
        return rc, b"", info, None
    t = GunzipTimes()
    lib.mksnap_gunzip_get_times.argtypes = [C.c_void_p, C.POINTER(GunzipTimes)]
    assert lib.mksnap_gunzip_get_times(h, C.byref(t)) == 0
    parts, buf, got = [], C.create_string_buffer(chunk), C.c_uint64()
    try:
        while True:
            rc = lib.mksnap_gunzip_read(h, buf, chunk, C.byref(got))
            parts.append(buf.raw[:got.value])
            if rc or got.value < chunk:
                break
    finally:
        assert lib.mksnap_gunzip_close(h) == 0
    return rc, b"".join(parts), info, t.extra_decodes


def check(lib, h, name, blob, chunk=1 << 20):
    """The engine against Go's reader; on an accepted blob of several members, every member is at least one segment and
    (beyond blobs whose members hold more than K candidates) no start needs a decode of its own."""
    want = gc.go_gunzip(blob)
    rc, got, info, extra = engine_gunzip_times(lib, h, blob, chunk)
    if want is None:
        assert rc == gc.MKSNAP_E_DATA, (name, rc)
        return None, None
    assert rc == 0 and got == want, (name, rc, len(got), len(want))
    assert (info.gz_bytes, info.out_bytes) == (len(blob), len(want)), name
    n_members = len(member_bodies(blob))
    assert info.n_members == n_members and info.n_segments >= n_members, (name, info.n_members, info.n_segments)
    if not name.startswith(("false_candidates", "with_flushes")):
        assert extra == 0, (name, extra)
    return info, extra
