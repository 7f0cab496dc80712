"""Scenarios of the batched incremental layer commit (MemFS.commit_layers_cached), shared by the CPU mock test and the
H100 test.  Every scenario compares a batch with sequential commit_copy_ops_cached calls, one per layer, on a fresh
MemFS with a copy of the same cache: per layer the tar bytes, TarDigest, n_entries and tar_bytes; the remembered file
digest of every regular destination; a probe layer described against both trees; and the bytes the two caches save.
The batch's root, n_chunks and n_unique are those of the uncached batch.

`make(arena_bytes, cdc=None, max_extents=4096)` returns an engine (the CPU mock or libmksnap) with
`work()`, a value that changes whenever the engine takes a submit, `mark()` and `uploaded()`, the bytes that went to
the device since mark() (on the mock: the arena bytes of the last session's submits)."""
from __future__ import annotations

import hashlib
import os
import tarfile

import numpy as np

NOW = 1_600_000_000
T = 1_500_000_000
ARENA = 1 << 20


def _mk(path, data):
    os.makedirs(os.path.dirname(path), exist_ok=True)
    with open(path, "wb") as f:
        f.write(data)
    os.utime(path, (T, T))


def make_ctx(tmp, seed=7):
    """A build context: six directories of small, empty and duplicate files, an empty directory, and `alt/` with other
    content for destinations that an earlier layer wrote."""
    c = os.path.join(tmp, "ctx")
    rng = np.random.default_rng(seed)
    for d in range(6):
        for i in range(6):
            n = 0 if i == 5 else int(rng.integers(1, 120_000))
            _mk(os.path.join(c, "d%d" % d, "f%03d.bin" % i), rng.bytes(n))
    same = rng.bytes(90_000)
    _mk(os.path.join(c, "d1", "dup.bin"), same)
    _mk(os.path.join(c, "d3", "dup.bin"), same)
    _mk(os.path.join(c, "alt", "f000.bin"), rng.bytes(77_777))
    _mk(os.path.join(c, "alt", "empty"), b"")
    os.makedirs(os.path.join(c, "e"))
    for d, _, _ in os.walk(c):
        os.utime(d, (T, T))
    return c


# one layer per entry: [(source relative to the context, destination)] -- the same source in two layers (0, 4), the same
# destination in two and three layers (0, 5, 7; 1, 6: the later one an empty file), a layer with no files (3)
LAYERS = [[("d0", "/app/d0/")], [("d1", "/app/d1/")], [("d2", "/app/d2/"), ("d3", "/app/d3/")], [("e", "/app/e/")],
          [("d0", "/again/d0/")], [("alt/f000.bin", "/app/d0/f000.bin")], [("alt/empty", "/app/d1/f001.bin")],
          [("d0", "/app/d0/")], [("d4", "/app/d4/")], [("d5", "/app/d5/")]]


def ops_of(ctx, layers):
    from makisu_b200 import host
    return [[host.CopyOperation(["/" + s], ctx, "/", d, 3, 4) for s, d in layer] for layer in layers]


def destinations(ctx, layers):
    """Every regular-file destination the layers write."""
    out = set()
    for layer in layers:
        for s, d in layer:
            src = os.path.join(ctx, s)
            if os.path.isfile(src):
                out.add(d)
                continue
            for r, _, files in os.walk(src):
                for n in files:
                    out.add(os.path.join(d, os.path.relpath(os.path.join(r, n), src)))
    return sorted(out)


def sources(ctx, layers):
    """Every regular source file the layers copy, once."""
    out = set()
    for layer in layers:
        for s, _ in layer:
            src = os.path.join(ctx, s)
            if os.path.isfile(src):
                out.add(src)
            for r, _, files in os.walk(src):
                out.update(os.path.join(r, n) for n in files)
    return sorted(out)


def copy_cache(cache, path):
    from makisu_b200 import host
    cache.save(path)
    return host.ChunkCache(path)


class Runner:
    def __init__(self, make, tmp, ctx):
        self.make, self.tmp, self.ctx, self.n = make, tmp, ctx, 0

    def _dir(self, name):
        self.n += 1
        d = os.path.join(self.tmp, "%s%03d" % (name, self.n))
        os.makedirs(d)
        return d

    def batch(self, eng, cache, layers, flags, with_tar=True, cached=True):
        """-> (MemFS, outs, stats or None, tar bytes per layer or None)."""
        from makisu_b200 import host
        fs = host.MemFS(self._dir("root"))
        tdir = self._dir("tars")
        files = [open(os.path.join(tdir, "l%02d.tar" % i), "wb") for i in range(len(layers))] if with_tar else []
        try:
            fds = [f.fileno() for f in files] if with_tar else None
            if cached:
                outs, st = fs.commit_layers_cached(eng, cache, NOW, ops_of(self.ctx, layers), 3, fds, flags)
            else:
                outs, st = fs.commit_layers(eng, NOW, ops_of(self.ctx, layers), 3, fds, flags), None
        finally:
            for f in files:
                f.close()
        tars = [open(f.name, "rb").read() for f in files] if with_tar else None
        return fs, outs, st, tars

    def sequential(self, eng, cache, layers, flags, with_tar=True):
        from makisu_b200 import host
        fs = host.MemFS(self._dir("root"))
        tdir = self._dir("tars")
        outs, stats, tars = [], [], []
        for i, ops in enumerate(ops_of(self.ctx, layers)):
            path = os.path.join(tdir, "l%02d.tar" % i)
            with open(path, "wb") as f:
                lay, st = fs.commit_copy_ops_cached(eng, cache, NOW, ops, 3, f.fileno() if with_tar else -1, flags)
            outs.append(lay)
            stats.append(st)
            tars.append(open(path, "rb").read() if with_tar else None)
        return fs, outs, stats, tars if with_tar else None

    def check(self, cache, flags, layers=LAYERS, with_tar=True, arena=ARENA, **kw):
        """The batch with `cache` equals one cached commit per layer with a copy of it -> (outs, stats, per-layer stats)."""
        ref_cache = copy_cache(cache, os.path.join(self._dir("cache"), "c")) if cache is not None else None
        eng = self.make(arena, **kw)
        eng.mark()
        fs_b, outs, st, tars = self.batch(eng, cache, layers, flags, with_tar)
        st["uploaded"] = eng.uploaded()
        fs_s, seq, seq_st, seq_tars = self.sequential(self.make(arena, **kw), ref_cache, layers, flags, with_tar)
        for i, (a, b) in enumerate(zip(outs, seq)):
            for k in ("tar_digest", "n_entries", "tar_bytes"):
                assert a[k] == b[k], (i, k, a[k], b[k])
        assert tars == seq_tars
        _, plain, _, _ = self.batch(self.make(arena, **kw), None, layers, flags, with_tar=False, cached=False)
        for o in outs:
            assert (o["root"], o["n_chunks"], o["n_unique"]) == (plain[0]["root"], plain[0]["n_chunks"], plain[0]["n_unique"])
        self.same_trees(fs_b, fs_s, layers)
        if cache is not None:
            d = self._dir("saved")
            cache.save(os.path.join(d, "batch"))
            ref_cache.save(os.path.join(d, "seq"))
            assert open(os.path.join(d, "batch"), "rb").read() == open(os.path.join(d, "seq"), "rb").read()
        for k in ("files_total", "bytes_total"):
            assert st[k] == sum(s[k] for s in seq_st), (k, st, seq_st)
        return outs, st, seq_st

    def same_trees(self, fs_a, fs_b, layers):
        from makisu_b200 import host
        for dst in destinations(self.ctx, layers):
            assert fs_a.file_digest(dst) == fs_b.file_digest(dst), dst
        probe = [host.CopyOperation(["/"], self.ctx, "/", "/app/", 3, 4)]
        assert fs_a.describe_copy_ops(NOW, probe) == fs_b.describe_copy_ops(NOW, probe)


def rewrite(path, seed):
    """New content, same size (and a new mtime/ctime, as an editor leaves it)."""
    n = os.path.getsize(path)
    with open(path, "wb") as f:
        f.write(np.random.default_rng(seed).bytes(n))


# ---- scenarios --------------------------------------------------------------------------------------------------
def cold_warm_edited(make, tmp):
    """Cold, warm and one-file-edited caches, with TarDigest on the device and under MKHOST_NO_TAR_DIGEST, with and
    without MKHOST_FILE_DIGESTS."""
    from makisu_b200 import host
    ctx = make_ctx(tmp)
    run = Runner(make, tmp, ctx)
    NTD, FD = host.MKHOST_NO_TAR_DIGEST, host.MKHOST_FILE_DIGESTS
    for flags in (0, NTD, FD, NTD | FD):
        cache = host.ChunkCache()
        _, st, seq = run.check(cache, flags)
        assert st["files_reused"] == 0 and st["bytes_chunked"] == st["bytes_total"], st
        assert len(cache) == len(sources(ctx, LAYERS)) and sum(s["files_reused"] for s in seq) > 0
        _, st, _ = run.check(cache, flags)
        assert st["files_reused"] == st["files_total"] and st["bytes_chunked"] == 0, st
        assert st["bytes_uploaded"] == (0 if flags == NTD else st["bytes_total"]), st
        edited = os.path.join(ctx, "d0", "f002.bin")
        rewrite(edited, 100 + flags)
        _, st, _ = run.check(cache, flags)
        size = os.path.getsize(edited)
        assert st["files_reused"] == st["files_total"] - 2 and st["bytes_chunked"] == 2 * size, st  # layers 0 and 4
    print("cold_warm_edited ok")


def no_tar_digest_no_fd(make, tmp):
    """MKHOST_NO_TAR_DIGEST without a tar_fd and a warm cache: no file is read or uploaded.  The arena keeps the mock's
    poison where the bodies would be and the results still hold; the engine takes no file bytes."""
    from makisu_b200 import host
    ctx = make_ctx(tmp)
    run = Runner(make, tmp, ctx)
    NTD = host.MKHOST_NO_TAR_DIGEST
    cache = host.ChunkCache()
    run.check(cache, NTD, with_tar=False)
    _, st, _ = run.check(cache, NTD, with_tar=False)
    assert st["files_reused"] == st["files_total"] and st["bytes_uploaded"] == 0, st
    assert st["uploaded"] < st["bytes_total"] // 20, st
    _, st, _ = run.check(cache, NTD, with_tar=True)  # the tars need every body: read, still not uploaded
    assert st["bytes_uploaded"] == 0 and st["uploaded"] < st["bytes_total"] // 20, st
    print("no_tar_digest_no_fd ok")


def file_digests_without_cache(make, tmp):
    """MKHOST_FILE_DIGESTS with no cache: the plain batch remembers every file's digest (the later layer's for a
    destination written twice, none for one an empty file replaced)."""
    from makisu_b200 import host
    ctx = make_ctx(tmp)
    run = Runner(make, tmp, ctx)
    for flags in (host.MKHOST_FILE_DIGESTS, host.MKHOST_FILE_DIGESTS | host.MKHOST_NO_TAR_DIGEST):
        run.check(None, flags)
        fs, _, _, _ = run.batch(make(ARENA), None, LAYERS, flags, with_tar=False, cached=False)
        assert fs.file_digest("/app/d0/f000.bin") == hashlib.sha256(open(os.path.join(ctx, "d0", "f000.bin"), "rb").read()).digest()
        assert fs.file_digest("/app/d1/f001.bin") is None
        assert fs.file_digest("/again/d0/f001.bin") == hashlib.sha256(open(os.path.join(ctx, "d0", "f001.bin"), "rb").read()).digest()
    print("file_digests_without_cache ok")


def one_entry_shares(make, tmp):
    """Arenas so small that every layer's share of one holds one entry."""
    from makisu_b200 import host
    ctx = make_ctx(tmp)
    run = Runner(make, tmp, ctx)
    for flags in (0, host.MKHOST_NO_TAR_DIGEST | host.MKHOST_FILE_DIGESTS):
        cache = host.ChunkCache()
        run.check(cache, flags, arena=256 << 10)
        rewrite(os.path.join(ctx, "d4", "f001.bin"), 7 + flags)
        _, st, _ = run.check(cache, flags, arena=256 << 10)
        assert st["files_reused"] == st["files_total"] - 1, st
    print("one_entry_shares ok")


def other_cdc(make, tmp):
    """A cache cut under other CDC parameters starts over."""
    from makisu_b200 import abi, host
    ctx = make_ctx(tmp)
    run = Runner(make, tmp, ctx)
    cache = host.ChunkCache()
    run.check(cache, host.MKHOST_NO_TAR_DIGEST)
    other = abi.CdcParams(2048, 8192, 65536, 15, 11)
    _, st, _ = run.check(cache, host.MKHOST_NO_TAR_DIGEST, cdc=other)
    assert st["files_reused"] == 0 and st["bytes_chunked"] == st["bytes_total"], st
    _, st, _ = run.check(cache, host.MKHOST_NO_TAR_DIGEST, cdc=other)
    assert st["files_reused"] == st["files_total"], st
    print("other_cdc ok")


def too_few_slots(make, tmp):
    """Layers plus files with content beyond max_streams: refused before anything is submitted; one slot more is enough."""
    from makisu_b200 import host
    ctx = make_ctx(tmp)
    run = Runner(make, tmp, ctx)
    layers = LAYERS[:2]
    n = sum(1 for p in sources(ctx, layers) if os.path.getsize(p))
    eng = make(ARENA, max_extents=len(layers) + n - 1)
    w = eng.work()
    try:
        run.batch(eng, host.ChunkCache(), layers, host.MKHOST_FILE_DIGESTS)
        raise AssertionError("expected a refusal")
    except host.HostError as e:
        assert "per-file digests need one stream slot per regular file" in str(e), str(e)
        assert "max_extents (%d)" % (len(layers) + n - 1) in str(e), str(e)
    assert eng.work() == w
    run.check(host.ChunkCache(), host.MKHOST_FILE_DIGESTS, layers=layers, max_extents=len(layers) + n)
    for flags in (host.MKHOST_MATERIALIZE, host.MKHOST_SCAN_CONTENT, host.MKHOST_UNTAR):
        try:
            run.batch(make(ARENA), None, layers, flags)
            raise AssertionError("expected a refusal")
        except host.HostError as e:
            assert "only MKHOST_NO_TAR_DIGEST and MKHOST_FILE_DIGESTS are supported for a batch" in str(e), str(e)
    print("too_few_slots ok")


def scan_catches_same_second_edit(make, tmp):
    """A file committed by a MKHOST_FILE_DIGESTS batch and then rewritten in the same second with the same size is
    caught by a later commit_scan(MKHOST_SCAN_CONTENT); after a batch without file digests it is not."""
    from makisu_b200 import host
    for flags, caught in ((host.MKHOST_FILE_DIGESTS, True), (0, False)):
        root = os.path.join(tmp, "root_scan%d" % flags)
        rng = np.random.default_rng(3)
        for d in ("a", "b"):
            for i in range(3):
                _mk(os.path.join(root, d, "f%d.bin" % i), rng.bytes(int(rng.integers(1, 50_000))))
        fs = host.MemFS(root)
        ops = [[host.CopyOperation(["/" + d], root, "/", "/%s/" % d, os.getuid(), os.getgid())] for d in ("a", "b")]
        fs.commit_layers_cached(make(ARENA), host.ChunkCache(), NOW, ops, flags=flags)
        victim = os.path.join(root, "b", "f1.bin")
        st = os.stat(victim)
        rewrite(victim, 9)
        os.utime(victim, ns=(st.st_atime_ns, st.st_mtime_ns))
        path = os.path.join(tmp, "scan%d.tar" % flags)
        with open(path, "wb") as f:
            fs.commit_scan(make(ARENA), NOW, tar_fd=f.fileno(), flags=host.MKHOST_SCAN_CONTENT)
        names = tarfile.open(path).getnames()
        assert ("b/f1.bin" in names) == caught, (flags, names)
        assert "a/f1.bin" not in names and "b/f0.bin" not in names, names
    print("scan_catches_same_second_edit ok")


ALL = ["cold_warm_edited", "no_tar_digest_no_fd", "file_digests_without_cache", "one_entry_shares", "other_cdc",
       "too_few_slots", "scan_catches_same_second_edit"]
