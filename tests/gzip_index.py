"""Block indexes of gzip blobs for the indexed gunzip tests (mksnap_gunzip_open_indexed / _get_index).

`block_starts` is the reference: libz through ctypes, driven with inflate(Z_BLOCK) as zlib's examples/zran.c does, lists
every DEFLATE block header of every member as (bit offset in the blob, output offset in the decompressed stream).  The
case generators are seeded; nothing here uses the oracle."""
import ctypes as C
import ctypes.util
import random
import struct
import zlib

from tests import gzip_corpus as gc
from tests import gzip_members as gm

Z_BLOCK, Z_STREAM_END, Z_BUF_ERROR = 5, 1, -5
MKSNAP_E_INVAL = -1
SPLIT_OUT = 1 << 20


class _ZStream(C.Structure):
    _fields_ = [("next_in", C.c_void_p), ("avail_in", C.c_uint), ("total_in", C.c_ulong),
                ("next_out", C.c_void_p), ("avail_out", C.c_uint), ("total_out", C.c_ulong),
                ("msg", C.c_char_p), ("state", C.c_void_p), ("zalloc", C.c_void_p), ("zfree", C.c_void_p),
                ("opaque", C.c_void_p), ("data_type", C.c_int), ("adler", C.c_ulong), ("reserved", C.c_ulong)]


_libz = None


def _z():
    global _libz
    if _libz is None:
        _libz = C.CDLL(ctypes.util.find_library("z") or "libz.so.1")
        _libz.zlibVersion.restype = C.c_char_p
        _libz.inflateInit2_.argtypes = [C.POINTER(_ZStream), C.c_int, C.c_char_p, C.c_int]
        _libz.inflate.argtypes = [C.POINTER(_ZStream), C.c_int]
        _libz.inflateEnd.argtypes = [C.POINTER(_ZStream)]
    return _libz


def _member_blocks(blob: bytes, body: int):
    """Block headers of the raw DEFLATE stream at byte `body`: [(bit offset in blob, output offset in the member)],
    and the byte offset of the member trailer."""
    z = _z()
    s = _ZStream()
    assert z.inflateInit2_(C.byref(s), -15, z.zlibVersion(), C.sizeof(_ZStream)) == 0
    inp = C.create_string_buffer(blob[body:], len(blob) - body)
    out = C.create_string_buffer(1 << 20)
    s.next_in, s.avail_in = C.addressof(inp), len(blob) - body
    blocks = [(8 * body, 0)]
    try:
        while True:
            if s.avail_out == 0:
                s.next_out, s.avail_out = C.addressof(out), len(out)
            rc = z.inflate(C.byref(s), Z_BLOCK)
            if rc == Z_STREAM_END:
                return blocks, body + s.total_in
            assert rc == 0 or (rc == Z_BUF_ERROR and s.avail_out == 0), rc
            if s.data_type & 128 and not s.data_type & 64:
                bit = 8 * (body + s.total_in) - (s.data_type & 7)
                if bit != blocks[-1][0]:
                    blocks.append((bit, s.total_out))
    finally:
        z.inflateEnd(C.byref(s))


def block_starts(blob: bytes):
    """Every block header of a blob Go's reader accepts: [(bit offset, output offset in the whole stream)]."""
    out, off, base = [], 0, 0
    while off < len(blob):
        body = gc._header_end(blob, off)
        blocks, trailer = _member_blocks(blob, body)
        out += [(b, base + o) for b, o in blocks]
        base += struct.unpack("<I", blob[trailer + 4:trailer + 8])[0]  # ISIZE (members here are < 4 GiB)
        off = trailer + 8
    return out


# ---- cases ---------------------------------------------------------------------------------------------------------
def layer_data(n: int, seed=0) -> bytes:
    """n bytes of layer-like content: text-like runs from a 2 MiB pool, random runs, and repeats of recent output."""
    rng = random.Random(seed)
    pool = gc.mixed(rng, 2 << 20)
    out = bytearray()
    while len(out) < n:
        k = rng.random()
        if k < 0.5:
            a = rng.randrange(len(pool) - 200_000)
            out += pool[a:a + rng.randint(1000, 200_000)]
        elif k < 0.8:
            out += rng.randbytes(rng.randint(100, 100_000))
        else:
            a = max(0, len(out) - 32768)
            out += bytes(out[a:a + rng.randint(3, 20_000)])
    return bytes(out[:n])


def single(data: bytes, level=6, strategy=zlib.Z_DEFAULT_STRATEGY) -> bytes:
    return gc.gzip_member(gc.deflate(data, level, strategy=strategy), data)


def far_refs(n_blocks=40, seed=3) -> bytes:
    """Fixed-Huffman blocks of 32 KiB literals each followed by length-258 / distance-32768 copies, so that every block
    start is crossed by references that reach the whole window back."""
    rng = random.Random(seed)
    data = bytearray()
    w = gc.BitWriter()
    for i in range(n_blocks):
        ops = [("lit", rng.randrange(256)) for _ in range(rng.randint(200, 40_000))] if i % 3 == 0 else []
        ops += [("match", 258, 32768)] * rng.randint(1, 150) + [("match", 258, rng.randint(1, 32768))]
        final = i == n_blocks - 1
        w.put(1 if final else 0, 1)
        w.put(1, 2)
        for op in ops:
            if op[0] == "lit":
                w.lit(op[1])
                data.append(op[1])
            else:
                if len(data) < op[2]:  # the first block: reach only as far as there is output
                    continue
                w.match(op[1], op[2])
                for _ in range(op[1]):
                    data.append(data[-op[2]])
        w.lit(256)
    body = w.bytes()
    return gc.gzip_member(body, bytes(data))


def corpus():
    """(name, blob): the blobs the indexed open is checked on (all valid)."""
    d = layer_data(64 << 20, seed=1)
    out = [("level%d_4m" % lvl, single(d[:4 << 20], lvl)) for lvl in range(10)]
    out += [("single_16m", single(d[:16 << 20])), ("single_64m", single(d)),
            ("fixed_4m", single(d[:4 << 20], 6, zlib.Z_FIXED)), ("huffman_4m", single(d[:4 << 20], 6, zlib.Z_HUFFMAN_ONLY)),
            ("stored_4m", single(d[:4 << 20], 0)), ("far_refs", far_refs()),
            ("multi_member", single(d[:3 << 20], 1) + single(d[3 << 20:9 << 20], 9) + single(b"")),
            ("pgzip", gc.pgzip(d[:6 << 20])), ("bgzf", gm.bgzf(d[:3 << 20])),
            ("estargz", gm.estargz(_tar(d[:12 << 20]), chunk=4 << 20))]
    return out


def _tar(data: bytes) -> bytes:
    """A layer tar of files cut from `data` (sizes up to 6 MiB)."""
    import io
    import tarfile
    buf, rng, i, o = io.BytesIO(), random.Random(5), 0, 0
    with tarfile.open(fileobj=buf, mode="w", format=tarfile.PAX_FORMAT) as tf:
        while o < len(data):
            n = min(len(data) - o, rng.choice([0, 300, 70_000, 1 << 20, 6 << 20]))
            ti = tarfile.TarInfo("usr/lib/f%03d" % i)
            ti.size, ti.mtime = n, 1_500_000_000
            tf.addfile(ti, io.BytesIO(data[o:o + n]))
            o, i = o + n, i + 1
    return buf.getvalue()


def fuzz_cases(n: int, seed=11):
    """(blob, points): small valid and damaged blobs with random indexes (true, shifted and random points)."""
    rng = random.Random(seed)
    d = layer_data(300_000, seed=seed)
    seeds = [single(d, 6), single(d[:100_000], 1), single(d[:50_000], 9), gc.pgzip(d[:120_000], block=20_000),
             gm.bgzf(d[:60_000], block=9000), single(d[:30_000], 0), far_refs(6, seed)]
    starts = {s: [b for b, _ in block_starts(s)] for s in seeds}
    out = []
    for _ in range(n):
        s = rng.choice(seeds)
        b = bytearray(s)
        if rng.random() < 0.4:
            for _ in range(rng.randint(1, 3)):
                p = rng.randrange(len(b))
                b[p] ^= 1 << rng.randrange(8)
            if rng.random() < 0.3:
                b = b[:rng.randrange(1, len(b))]
        pts = set()
        for bit in starts[s]:
            k = rng.random()
            if k < 0.4:
                pts.add(bit)
            elif k < 0.6:
                pts.add(bit + rng.randint(-9, 9))
        pts |= {rng.randrange(8 * len(b)) for _ in range(rng.randint(0, 30))}
        out.append((bytes(b), sorted(p for p in pts if 0 <= p < 8 * len(b))))
    return out


# ---- driving an engine (the real libmksnap or the CPU mock) through its C entry points ------------------------------
from makisu_b200.abi import GunzipIndexInfo as IndexInfo  # noqa: E402  (the engine's own binding of the struct)


def bind(lib):
    gc.bind(lib)
    lib.mksnap_gunzip_open_indexed.argtypes = [C.c_void_p, C.c_char_p, C.c_uint64, C.POINTER(C.c_uint64), C.c_uint64,
                                               C.POINTER(gc.GunzipInfo)]
    lib.mksnap_gunzip_get_index.argtypes = [C.c_void_p, C.POINTER(C.c_uint64), C.c_uint64, C.POINTER(IndexInfo)]
    return lib


def engine_gunzip_indexed(lib, h, blob: bytes, points, chunk=1 << 20):
    """(rc, bytes, info, index info, index points) of an indexed open of `blob` with `points` (None: no index) and
    reads until the end or the first error."""
    info, ix = gc.GunzipInfo(), IndexInfo()
    arr = (C.c_uint64 * max(1, len(points or ())))(*(points or ()))
    rc = lib.mksnap_gunzip_open_indexed(h, blob, len(blob), arr if points is not None else None,
                                        len(points or ()), C.byref(info))
    if rc:
        return rc, b"", info, ix, []
    try:
        assert lib.mksnap_gunzip_get_index(h, None, 0, C.byref(ix)) == 0
        got_pts = (C.c_uint64 * max(1, ix.n_points))()
        assert lib.mksnap_gunzip_get_index(h, got_pts, ix.n_points, C.byref(ix)) == 0
        parts, buf, got = [], C.create_string_buffer(chunk), C.c_uint64()
        while True:
            rc = lib.mksnap_gunzip_read(h, buf, chunk, C.byref(got))
            parts.append(buf.raw[:got.value])
            if rc or got.value < chunk:
                break
    finally:
        assert lib.mksnap_gunzip_close(h) == 0
    return rc, b"".join(parts), info, ix, list(got_pts[:ix.n_points])


def check_indexed(lib, h, name, blob, want=None, chunk=4 << 20):
    """Record, then reopen with the recorded points: output equal to zlib both times, every recorded point a libz block
    start, a single member of at least 4 MiB cut into several segments, every returned point linked on the reopen.
    Returns the recorded points."""
    want = gc.go_gunzip(blob) if want is None else want
    starts = {b for b, _ in block_starts(blob)}
    rc, got, info, ix, pts = engine_gunzip_indexed(lib, h, blob, None, chunk)
    assert rc == 0 and got == want, (name, rc, len(got), len(want))
    assert ix.points_given == 0 and ix.n_points == len(pts) and pts == sorted(pts), name
    assert set(pts) <= starts, (name, sorted(set(pts) - starts)[:5])
    if info.n_members == 1 and len(want) >= 4 << 20:
        assert info.n_segments > 1, (name, info.n_segments)
    rc, got, info2, ix2, pts2 = engine_gunzip_indexed(lib, h, blob, pts, chunk)
    assert rc == 0 and got == want, (name, rc)
    assert ix2.points_given == len(pts) and ix2.points_linked == ix2.points_given, (name, ix2.points_linked, len(pts))
    assert info2.n_segments >= info.n_segments and set(pts) <= set(pts2), name
    return pts


# ---- update_from_tar(s)_indexed against the uncompressed ingest -------------------------------------------------------
def layer_tar(n: int, seed: int) -> bytes:
    """A layer tar of about n bytes: files of layer-like content, directories, a symlink."""
    import io
    import tarfile
    rng = random.Random(seed)
    data = layer_data(n, seed)
    buf, o, i = io.BytesIO(), 0, 0
    with tarfile.open(fileobj=buf, mode="w", format=tarfile.PAX_FORMAT) as tf:
        for d in ("usr", "usr/lib", "usr/lib/l%d" % seed):
            ti = tarfile.TarInfo(d)
            ti.type, ti.mode, ti.mtime = tarfile.DIRTYPE, 0o755, 1_500_000_000
            tf.addfile(ti)
        while o < len(data):
            k = min(len(data) - o, rng.choice([0, 100, 5000, 300_000, 2 << 20]))
            ti = tarfile.TarInfo("usr/lib/l%d/f%03d.so" % (seed, i))
            ti.size, ti.mtime, ti.mode = k, 1_500_000_000, 0o644
            tf.addfile(ti, io.BytesIO(data[o:o + k]))
            o, i = o + k, i + 1
        ti = tarfile.TarInfo("usr/lib/l%d/link" % seed)
        ti.type, ti.linkname, ti.mtime = tarfile.SYMTYPE, "f000.so", 1_500_000_000
        tf.addfile(ti)
    return buf.getvalue()


def _ingest(make_engine, tmp, tag, flags, blobs, call):
    """Apply `blobs` (tar or gzip bytes) to a fresh MemFS through call(fs, engine, fds); -> (result, tree, digests)."""
    import io
    import os
    import tarfile
    from makisu_b200 import host
    from tests.mock_engine import scenarios
    d = os.path.join(tmp, tag)
    root = os.path.join(d, "root")
    os.makedirs(root)
    fds = []
    for i, b in enumerate(blobs):
        p = os.path.join(d, "layer%d" % i)
        open(p, "wb").write(b)
        fds.append(os.open(p, os.O_RDONLY))
    try:
        fs = host.MemFS(root)
        res = call(fs, make_engine(4 << 20), fds)  # MKHOST_UNTAR wants each member in one arena
    finally:
        for f in fds:
            os.close(f)
    names = set()
    for b in blobs:
        tar = gc.go_gunzip(b) if b[:2] == b"\x1f\x8b" else b
        names |= {m.name for m in tarfile.open(fileobj=io.BytesIO(tar)).getmembers() if m.isfile()}
    digests = {n: fs.file_digest("/" + n) for n in sorted(names)}
    return res, scenarios._tree(root, mtimes=True), digests


def check_ingest_indexed(make_engine, tmp):
    """update_from_tar(s)_indexed through a cache, cold and then warm, against the uncompressed ingest (DiffID, entries,
    chunk root, tree, file digests; MKHOST_UNTAR when running as root); a save / load round trip; a key whose entry is
    another blob's; cache == None."""
    import os
    from makisu_b200 import host
    from tests.mock_engine import scenarios
    NOW, G = scenarios.NOW, host.MKHOST_GUNZIP
    tars = [layer_tar(5 << 20, 1), layer_tar(3 << 20, 2), layer_tar(200_000, 3)]
    blobs = [single(t) for t in tars]
    keys = ["sha%d" % i for i in range(len(blobs))]
    flag_sets = [0, host.MKHOST_FILE_DIGESTS] + ([host.MKHOST_UNTAR] if os.geteuid() == 0 else [])
    n = 0
    for flags in flag_sets:
        def tag(s):
            return "%s_%d" % (s, flags)
        want = _ingest(make_engine, tmp, tag("plain"), flags, tars[:1],
                       lambda fs, e, fds: fs.update_from_tar(e, NOW, fds[0], flags))
        cache = host.GzIndexCache()
        for phase in ("cold", "warm"):
            got = _ingest(make_engine, tmp, tag(phase), flags, blobs[:1],
                          lambda fs, e, fds: fs.update_from_tar_indexed(e, cache, keys[0], NOW, fds[0], flags | G))
            (res, st), tree, dg = got
            assert (res, tree, dg) == want, (phase, flags)
            assert st["blobs"] == 1 and len(cache) == 1, st
            if phase == "cold":
                assert st["blobs_with_index"] == 0 and st["points_recorded"] > 0, st
            else:
                assert st["blobs_with_index"] == 1 and st["points_given"] == st["points_linked"] > 0, st
        # a run of layers, cold then warm, against update_from_tars of the tars
        want = _ingest(make_engine, tmp, tag("plain_run"), flags, tars,
                       lambda fs, e, fds: fs.update_from_tars(e, NOW, fds, flags))
        run_cache = host.GzIndexCache()
        for phase in ("run_cold", "run_warm"):
            (res, st), tree, dg = _ingest(
                make_engine, tmp, tag(phase), flags, blobs,
                lambda fs, e, fds: fs.update_from_tars_indexed(e, run_cache, keys, NOW, [(f, G) for f in fds], flags))
            assert (res, tree, dg) == want, (phase, flags)
            assert st["blobs"] == 3 and st["blobs_with_index"] == (3 if phase == "run_warm" else 0), st
        n += 1
    # save / load round trip
    path = os.path.join(tmp, "gz_index.cache")
    cache.save(path)
    loaded = host.GzIndexCache(path)
    assert len(loaded) == 1
    (res, st), _, _ = _ingest(make_engine, tmp, "loaded", 0, blobs[:1],
                              lambda fs, e, fds: fs.update_from_tar_indexed(e, loaded, keys[0], NOW, fds[0], G))
    assert st["blobs_with_index"] == 1 and st["points_given"] == st["points_linked"] > 0, st
    # a key whose entry is another blob's: ignored when the length differs, harmless when it matches
    want = _ingest(make_engine, tmp, "plain_b", 0, tars[1:2], lambda fs, e, fds: fs.update_from_tar(e, NOW, fds[0], 0))
    (res, st), tree, dg = _ingest(make_engine, tmp, "wrong_key", 0, blobs[1:2],
                                  lambda fs, e, fds: fs.update_from_tar_indexed(e, loaded, keys[0], NOW, fds[0], G))
    assert (res, tree, dg) == want and st["blobs_with_index"] == 0, st
    pts_a = [p for p in gc_points(path) if p < 8 * len(blobs[1])]
    assert pts_a
    forged = os.path.join(tmp, "forged.cache")
    with open(forged, "wb") as f:  # blob A's points under blob B's length
        f.write(b"mkhost-gz-index-cache 1\n%d %d %s\n" % (len(blobs[1]), len(pts_a), keys[1].encode()))
        f.write(struct.pack("<%dQ" % len(pts_a), *pts_a))
    forged_cache = host.GzIndexCache(forged)
    (res, st), tree, dg = _ingest(make_engine, tmp, "forged", 0, blobs[1:2],
                                  lambda fs, e, fds: fs.update_from_tar_indexed(e, forged_cache, keys[1], NOW, fds[0], G))
    assert (res, tree, dg) == want and st["blobs_with_index"] == 1 and st["points_given"] == len(pts_a), st
    # a file that does not parse is refused
    with open(forged, "ab") as f:
        f.write(b"garbage")
    try:
        host.GzIndexCache(forged)
        raise AssertionError("a damaged cache file loaded")
    except host.HostError:
        pass
    # cache == None: the plain gunzip ingest, no stats
    want = _ingest(make_engine, tmp, "gunzip_plain", 0, blobs[:1], lambda fs, e, fds: fs.update_from_tar(e, NOW, fds[0], G))
    (res, st), tree, dg = _ingest(make_engine, tmp, "none", 0, blobs[:1],
                                  lambda fs, e, fds: fs.update_from_tar_indexed(e, None, keys[0], NOW, fds[0], G))
    assert (res, tree, dg) == want and not any(st.values()), st
    return n


def gc_points(path):
    """The points of the first entry of a saved mkhost-gz-index-cache file."""
    b = open(path, "rb").read()
    first = b.index(b"\n") + 1
    eol = b.index(b"\n", first)
    n = int(b[first:eol].split(b" ")[1])
    return list(struct.unpack("<%dQ" % n, b[eol + 1:eol + 1 + 8 * n]))
