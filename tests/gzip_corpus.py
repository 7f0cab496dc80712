"""gzip blobs for the gunzip tests, generated with zlib, and the reference reader they are checked against.

`go_gunzip` is Go's compress/gzip Reader in multistream mode restated over zlib's raw inflate: zlib decides what DEFLATE
data is valid and what it decodes to; the gzip framing follows Go (FNAME / FCOMMENT at most 511 bytes, FHCRC checked,
reserved flag bits ignored, anything after a member that is not a member header -- garbage or zero padding -- is an
error, where Python's gzip module accepts zero padding)."""
import ctypes as C
import random
import struct
import zlib

MKSNAP_E_DATA = -7


def _header_end(b: bytes, off: int):
    if len(b) - off < 10 or b[off] != 0x1F or b[off + 1] != 0x8B or b[off + 2] != 8:
        return None
    flg, p = b[off + 3], off + 10
    if flg & 4:
        if p + 2 > len(b):
            return None
        p += 2 + int.from_bytes(b[p:p + 2], "little")
        if p > len(b):
            return None
    for f in (8, 16):
        if flg & f:
            z = b.find(b"\0", p, p + 512)
            if z < 0:
                return None
            p = z + 1
    if flg & 2:
        if p + 2 > len(b) or int.from_bytes(b[p:p + 2], "little") != zlib.crc32(b[off:p]) & 0xFFFF:
            return None
        p += 2
    return p


def go_gunzip(b: bytes):
    """The decompressed stream, or None where Go's reader reports an error."""
    out, off = [], 0
    while True:
        p = _header_end(b, off)
        if p is None:
            return None
        d = zlib.decompressobj(-15)
        try:
            data = d.decompress(b[p:]) + d.flush()
        except zlib.error:
            return None
        if not d.eof:
            return None
        rest = d.unused_data
        if len(rest) < 8:
            return None
        crc, size = struct.unpack("<II", rest[:8])
        if crc != zlib.crc32(data) or size != len(data) & 0xFFFFFFFF:
            return None
        out.append(data)
        off = len(b) - len(rest) + 8
        if off == len(b):
            return b"".join(out)


def gzip_member(body: bytes, data: bytes, flags=0, extra=b"", name=b"", comment=b"", mtime=0):
    """A member around an already deflated body."""
    h = bytearray(b"\x1f\x8b\x08" + bytes([flags]) + struct.pack("<I", mtime) + b"\x00\xff")
    if flags & 4:
        h += struct.pack("<H", len(extra)) + extra
    if flags & 8:
        h += name + b"\0"
    if flags & 16:
        h += comment + b"\0"
    if flags & 2:
        h += struct.pack("<H", zlib.crc32(bytes(h)) & 0xFFFF)
    return bytes(h) + body + struct.pack("<II", zlib.crc32(data), len(data) & 0xFFFFFFFF)


def deflate(data: bytes, level=6, wbits=-15, strategy=zlib.Z_DEFAULT_STRATEGY):
    c = zlib.compressobj(level, zlib.DEFLATED, wbits, 9, strategy)
    return c.compress(data) + c.flush()


def pgzip(data: bytes, block=1 << 20, level=6, flush=zlib.Z_SYNC_FLUSH):
    """The layout pgzip writes: blocks compressed independently, each with the previous block's last 32 KiB as a
    preset dictionary and ended by a flush (00 00 FF FF on a byte boundary), then an empty final block."""
    body = bytearray()
    for i in range(0, len(data), block):
        zd = data[max(0, i - 32768):i]
        c = zlib.compressobj(level, zlib.DEFLATED, -15, 9, zlib.Z_DEFAULT_STRATEGY, zd) if zd else \
            zlib.compressobj(level, zlib.DEFLATED, -15)
        body += c.compress(data[i:i + block]) + c.flush(flush)
    body += zlib.compressobj(level, zlib.DEFLATED, -15).flush(zlib.Z_FINISH)
    return gzip_member(bytes(body), data)


def flushed(pieces, level=6, flush=zlib.Z_FULL_FLUSH):
    """One DEFLATE stream with a flush between pieces (Z_FULL_FLUSH also resets the window)."""
    c = zlib.compressobj(level, zlib.DEFLATED, -15)
    body = b"".join(c.compress(p) + c.flush(flush) for p in pieces) + c.flush()
    return gzip_member(body, b"".join(pieces))


class BitWriter:
    """DEFLATE bit packing for hand-built blocks (fixed Huffman codes)."""

    def __init__(self):
        self.bits, self.n = 0, 0

    def put(self, v, k):
        self.bits |= v << self.n
        self.n += k

    def code(self, c, k):  # Huffman codes go MSB first
        self.put(int(format(c, "0%db" % k)[::-1], 2), k)

    def lit(self, s):
        if s < 144:
            self.code(0x30 + s, 8)
        elif s < 256:
            self.code(0x190 + s - 144, 9)
        elif s < 280:
            self.code(s - 256, 7)
        else:
            self.code(0xC0 + s - 280, 8)

    def match(self, length, dist):
        lb = [3, 4, 5, 6, 7, 8, 9, 10, 11, 13, 15, 17, 19, 23, 27, 31, 35, 43, 51, 59, 67, 83, 99, 115, 131, 163, 195,
              227, 258]
        le = [0] * 8 + [1] * 4 + [2] * 4 + [3] * 4 + [4] * 4 + [5] * 4 + [0]
        db = [1, 2, 3, 4, 5, 7, 9, 13, 17, 25, 33, 49, 65, 97, 129, 193, 257, 385, 513, 769, 1025, 1537, 2049, 3073,
              4097, 6145, 8193, 12289, 16385, 24577]
        de = [0, 0, 0, 0, 1, 1, 2, 2, 3, 3, 4, 4, 5, 5, 6, 6, 7, 7, 8, 8, 9, 9, 10, 10, 11, 11, 12, 12, 13, 13]
        i = 28 if length == 258 else max(k for k in range(28) if lb[k] <= length)
        self.lit(257 + i)
        self.put(length - lb[i], le[i])
        j = max(k for k in range(30) if db[k] <= dist)
        self.code(j, 5)
        self.put(dist - db[j], de[j])

    def bytes(self):
        return self.bits.to_bytes((self.n + 7) // 8, "little")


def fixed_block(ops, final=True):
    """A fixed-Huffman block from ('lit', byte) / ('match', length, dist) / ('raw', symbol) operations."""
    w = BitWriter()
    w.put(1 if final else 0, 1)
    w.put(1, 2)
    for op in ops:
        if op[0] == "lit":
            w.lit(op[1])
        elif op[0] == "match":
            w.match(op[1], op[2])
        else:
            w.lit(op[1])
    w.lit(256)
    return w.bytes()


def _expand(ops):
    out = bytearray()
    for op in ops:
        if op[0] == "lit":
            out.append(op[1])
        else:
            for _ in range(op[1]):
                out.append(out[-op[2]])
    return bytes(out)


def mixed(rng: random.Random, n: int) -> bytes:
    """Text-like, repetitive and random runs."""
    words = [bytes(rng.choice(b"abcdefghijklmnopqrstuvwxyz") for _ in range(rng.randint(2, 9))) for _ in range(200)]
    out = bytearray()
    while len(out) < n:
        k = rng.random()
        if k < 0.5:
            out += b" ".join(rng.choice(words) for _ in range(rng.randint(5, 200))) + b"\n"
        elif k < 0.8:
            out += rng.randbytes(rng.randint(1, 5000))
        else:
            out += bytes([rng.randrange(256)]) * rng.randint(1, 3000)
    return bytes(out[:n])


def corpus():
    """(name, blob) pairs: valid and invalid under Go's reader (go_gunzip decides which)."""
    rng = random.Random(1952)
    data = mixed(rng, 300_000)
    out = []
    for lvl in range(10):
        out.append(("level%d" % lvl, gzip_member(deflate(data, lvl), data)))
    out.append(("empty_member", gzip_member(deflate(b""), b"")))
    out.append(("fixed_only", gzip_member(deflate(data[:2000], 6, strategy=zlib.Z_FIXED), data[:2000])))
    out.append(("huffman_only", gzip_member(deflate(data, 6, strategy=zlib.Z_HUFFMAN_ONLY), data)))
    out.append(("rle", gzip_member(deflate(data, 6, strategy=zlib.Z_RLE), data)))
    base = [("lit", rng.randrange(256)) for _ in range(32768)]
    far = base + [("match", 258, 32768)] * 3 + [("lit", 7), ("match", 258, 1), ("match", 10, 3), ("match", 100, 2)]
    out.append(("len258_dist32768_overlap", gzip_member(fixed_block(far), _expand(far))))
    out.append(("dist_before_member_start", gzip_member(fixed_block([("lit", 1), ("match", 5, 2)]), b"\x01" * 6)))
    out.append(("invalid_length_symbol_286", gzip_member(fixed_block([("lit", 1), ("raw", 286)]), b"\x01")))
    st = bytes(rng.randrange(256) for _ in range(1000))
    stored = b"\x00" + struct.pack("<HH", 1000, 1000 ^ 0xFFFF) + st + b"\x01" + struct.pack("<HH", 0, 0xFFFF)
    out.append(("stored_then_empty_final", gzip_member(stored, st)))
    out.append(("stored_bad_nlen", gzip_member(b"\x01" + struct.pack("<HH", 3, 3) + b"abc", b"abc")))
    out.append(("block_type_3", gzip_member(b"\x07\x00", b"")))
    # pgzip-shaped: 64 KiB blocks so that a few hundred KB give many segments; data repeats across block boundaries
    rep = (data[:50_000] * 12)[:600_000]
    out.append(("pgzip_cross_refs", pgzip(rep, block=65536)))
    out.append(("pgzip_mixed", pgzip(data, block=65536, level=1)))
    out.append(("pgzip_level0", pgzip(data[:200_000], block=65536, level=0)))
    out.append(("full_flush", flushed([data[i:i + 40_000] for i in range(0, len(data), 40_000)])))
    out.append(("sync_flush_one_stream", flushed([data[i:i + 33_000] for i in range(0, len(data), 33_000)],
                                                 flush=zlib.Z_SYNC_FLUSH)))
    m1, m2, m3 = data[:1000], data[1000:90_000], b""
    multi = gzip_member(deflate(m1), m1) + pgzip(m2, block=30_000) + gzip_member(deflate(m3), m3)
    out.append(("multi_member", multi))
    for f in (1, 2, 4, 8, 16, 31, 0x20, 0xFF & ~0xC0):
        out.append(("flags_%02x" % f, gzip_member(deflate(m1), m1, flags=f, extra=b"XY\x02\x00ab", name=b"layer.tar",
                                                  comment=b"c" * 40)))
    out.append(("fname_511", gzip_member(deflate(m1), m1, flags=8, name=b"n" * 511)))
    out.append(("fname_512_go_rejects", gzip_member(deflate(m1), m1, flags=8, name=b"n" * 512)))
    bad_hcrc = bytearray(gzip_member(deflate(m1), m1, flags=2))
    bad_hcrc[10] ^= 1
    out.append(("bad_header_crc", bytes(bad_hcrc)))
    good = gzip_member(deflate(m1), m1)
    out.append(("trailing_garbage", good + b"garbage!!!!!"))
    out.append(("trailing_short_garbage", good + b"\x1f\x8b"))
    out.append(("zero_padding", good + bytes(512)))
    bad_crc = bytearray(good)
    bad_crc[-8] ^= 0x40
    out.append(("bad_crc", bytes(bad_crc)))
    bad_isize = bytearray(good)
    bad_isize[-4] ^= 1
    out.append(("bad_isize", bytes(bad_isize)))
    out.append(("bad_crc_second_member", good + bytes(bad_crc)))
    out.append(("truncated", good[:len(good) // 2]))
    out.append(("not_gzip", b"hello world, not gzip"))
    out.append(("empty_blob", b""))
    pat = b"\x00\x00\xff\xff" * 60_000
    out.append(("level0_flush_pattern", gzip_member(deflate(pat, 0), pat)))
    return out


def fuzz_cases(n: int, seed=7):
    """Truncated and bit-flipped variants of small valid blobs of every kind."""
    rng = random.Random(seed)
    d = mixed(rng, 20_000)
    seeds = [gzip_member(deflate(d, lvl), d) for lvl in (0, 1, 6, 9)]
    seeds += [pgzip(d, block=4096), flushed([d[:7000], d[7000:]]), gzip_member(deflate(d[:300], 6, strategy=zlib.Z_FIXED), d[:300]),
              gzip_member(deflate(d[:100]), d[:100], flags=31, extra=b"ab", name=b"x", comment=b"y") + pgzip(d[:9000], block=2048)]
    out = []
    for i in range(n):
        b = bytearray(rng.choice(seeds))
        k = rng.random()
        if k < 0.3:
            b = b[:rng.randrange(len(b))]
        else:
            for _ in range(rng.randint(1, 4)):
                p = rng.randrange(len(b))
                b[p] ^= 1 << rng.randrange(8)
            if k > 0.9:
                b = b[:rng.randrange(len(b))]
        out.append(bytes(b))
    return out


# ---- driving an engine (the real libmksnap or the CPU mock) through its C entry points ------------------------------
class GunzipInfo(C.Structure):
    _fields_ = [("gz_bytes", C.c_uint64), ("out_bytes", C.c_uint64), ("n_members", C.c_uint64),
                ("n_segments", C.c_uint64)]


def bind(lib):
    lib.mksnap_gunzip_open.argtypes = [C.c_void_p, C.c_char_p, C.c_uint64, C.POINTER(GunzipInfo)]
    lib.mksnap_gunzip_read.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64, C.POINTER(C.c_uint64)]
    lib.mksnap_gunzip_close.argtypes = [C.c_void_p]
    return lib


def engine_gunzip(lib, h, blob: bytes, chunk=1 << 20):
    """(rc, bytes, info): rc = 0 and the whole stream, or the first error code with the bytes read before it."""
    info = GunzipInfo()
    rc = lib.mksnap_gunzip_open(h, blob, len(blob), C.byref(info))
    if rc:
        return rc, b"", info
    parts, buf, got = [], C.create_string_buffer(chunk), C.c_uint64()
    try:
        while True:
            rc = lib.mksnap_gunzip_read(h, buf, chunk, C.byref(got))
            parts.append(buf.raw[:got.value])
            if rc or got.value < chunk:
                break
    finally:
        assert lib.mksnap_gunzip_close(h) == 0
    return rc, b"".join(parts), info


# ---- update_from_tar(MKHOST_GUNZIP) against the uncompressed ingest ---------------------------------------------------
def layer_blobs(seed=11):
    """(name, gzip blob) layers: the registry-style alpine fixture and generated layers in both layouts."""
    import io
    import os
    import tarfile

    import numpy as np

    from tests.mock_engine import scenarios

    here = os.path.dirname(os.path.abspath(__file__))
    out = [("alpine", open(os.path.join(here, "golden", "alpine_test_layer.tar.gz"), "rb").read())]
    rng = np.random.default_rng(seed)
    base = scenarios._base_tar(rng)
    out += [("base_pgzip", pgzip(base, block=65536)), ("base_gzip", gzip_member(deflate(base, 9), base))]
    buf = io.BytesIO()  # a member larger than a 1 MiB arena, text and random files, and two members
    with tarfile.open(fileobj=buf, mode="w", format=tarfile.PAX_FORMAT) as tf:
        r = random.Random(seed)
        for i, data in enumerate([mixed(r, 1_500_000), r.randbytes(200_000), mixed(r, 70_000), b""]):
            ti = tarfile.TarInfo("opt/f%d.bin" % i)
            ti.size, ti.mtime, ti.mode = len(data), scenarios.T, 0o644
            tf.addfile(ti, io.BytesIO(data))
    big = buf.getvalue()
    out.append(("big_member_multi", pgzip(big[:700_000], block=100_000) + gzip_member(deflate(big[700_000:], 1),
                                                                                      big[700_000:])))
    return out


def check_ingest(make_engine, tmp, name, blob, flags, arena_bytes=1 << 20):
    """update_from_tar(blob, MKHOST_GUNZIP | flags) equals update_from_tar(go_gunzip(blob), flags): result, file
    digests and (MKHOST_UNTAR) the tree written under the root."""
    import hashlib
    import os

    from makisu_b200 import host
    from tests.mock_engine import scenarios

    tar = go_gunzip(blob)
    assert tar is not None
    results, trees, digests = [], [], []
    for mode in ("plain", "gunzip"):
        d = os.path.join(tmp, "%s_%d_%s" % (name, flags, mode))
        root = os.path.join(d, "root")
        os.makedirs(root)
        src = os.path.join(d, "layer")
        open(src, "wb").write(tar if mode == "plain" else blob)
        fs = host.MemFS(root)
        with open(src, "rb") as f:
            results.append(fs.update_from_tar(make_engine(arena_bytes), scenarios.NOW, f.fileno(),
                                              flags=flags | (host.MKHOST_GUNZIP if mode == "gunzip" else 0)))
        trees.append(scenarios._tree(root, mtimes=True))
        import tarfile
        import io
        names = [m.name for m in tarfile.open(fileobj=io.BytesIO(tar)).getmembers() if m.isfile()]
        digests.append({n: fs.file_digest("/" + n.lstrip("./")) for n in names})
    assert results[0] == results[1], (name, flags)
    if not flags & host.MKHOST_NO_TAR_DIGEST:
        assert results[1]["tar_digest"] == "sha256:" + hashlib.sha256(tar).hexdigest()
    assert trees[0] == trees[1] and digests[0] == digests[1], (name, flags)
    if flags & host.MKHOST_FILE_DIGESTS:
        assert any(v is not None for v in digests[1].values())
    return results[1]
