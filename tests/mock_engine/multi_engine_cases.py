"""Scenarios of the multi-engine calls (mkhost_context_crc32_multi, mkhost_memfs_commit_layers_multi), shared by the CPU
mock test and the H100 test.  Every scenario compares the multi-engine call over 1, 2, 3 and 5 engines with the
single-engine call on a fresh engine: for the cacheID the value, the stream length, the stats and the bytes the cache
saves afterwards (and the oracle's cacheID); for a batch every per-layer result (TarDigest, n_entries, tar_bytes, and
the batch's root / n_chunks / n_unique), the bytes written to every tar_fd, the stats, the remembered file digest of
every destination, a probe layer described against both trees, and the bytes the chunk caches save.

`make(arena_bytes, max_extents=4096, max_chunks=0, cdc=None)` returns an engine (the CPU mock or libmksnap) with `h`
and `work()`, a value that changes whenever the engine takes a submit."""
from __future__ import annotations

import hashlib
import os

import numpy as np

from tests import commit_layers_cases as cases

NOW = cases.NOW
ARENA = cases.ARENA
ENGINES = (1, 2, 3, 5)


def _saved(cache, path) -> bytes:
    cache.save(path)
    with open(path, "rb") as f:
        return f.read()


# ---- cacheID ----------------------------------------------------------------------------------------------------
def _crc_ctx(tmp, seed=11, big=0):
    """A context of files of many sizes, empty files, a symlink and nested directories; `big` adds one file larger than
    all the others together."""
    c = os.path.join(tmp, "crcctx")
    rng = np.random.default_rng(seed)
    for d in range(4):
        for i in range(5):
            cases._mk(os.path.join(c, "d%d" % d, "s%d" % i, "f%02d.bin" % i),
                      rng.bytes(0 if i == 4 else int(rng.integers(1, 200_000))))
    cases._mk(os.path.join(c, "Dockerfile"), b"FROM scratch\nCOPY . /app/\n")
    if big:
        cases._mk(os.path.join(c, "huge.bin"), rng.bytes(big))
    os.symlink("Dockerfile", os.path.join(c, "link"))
    for d, _, _ in os.walk(c):
        os.utime(d, (cases.T, cases.T))
    return c


def _cache_id_against(make, ctx, paths, arena, n_engines, cache_pair=None, prefix=b"seedCOPY. /app/"):
    """The multi-engine cacheID over n_engines engines equals the single-engine one; cache_pair = (multi, single) caches,
    which must save the same bytes afterwards -> (crc, stream length, stats)."""
    from makisu_b200 import host
    engines = [make(arena) for _ in range(n_engines)]
    got = host.context_crc32_multi(engines, prefix, ctx, paths, 3, cache_pair[0] if cache_pair else None)
    one = make(arena)
    if cache_pair:
        want = cache_pair[1].context_crc32(one, prefix, ctx, paths, 3)
        d = os.path.dirname(ctx)
        assert _saved(cache_pair[0], os.path.join(d, "m.cache")) == _saved(cache_pair[1], os.path.join(d, "s.cache"))
    else:
        crc, slen = host.context_crc32(one, prefix, ctx, paths, 3)
        want = (crc, slen, got[2])
        assert got[2]["files_reused"] == 0 and got[2]["bytes_sent"] == got[2]["bytes_total"], got[2]
    assert got == want, (n_engines, got, want)
    return got


def cache_id_cold_warm_edited(make, tmp):
    """No cache, then a cold, a warm and a one-file-edited cache; every value also equals the oracle's cacheID."""
    from makisu_b200 import host
    from oracle import ctx_crc
    ctx = _crc_ctx(tmp)
    seed = ctx_crc.from_step_cache_id(ctx_crc.plan_seed(True, False), "scratch")
    prefix = (seed + "COPY" + ". /app/").encode()
    for n in ENGINES:
        _cache_id_against(make, ctx, ["."], 256 << 10, n, prefix=prefix)
        caches = (host.CrcCache(), host.CrcCache())
        for step in ("cold", "warm", "edited"):
            if step == "edited":
                cases.rewrite(os.path.join(ctx, "d2", "s1", "f01.bin"), 40 + n)
            crc, _, st = _cache_id_against(make, ctx, ["."], 256 << 10, n, caches, prefix)
            assert "%x" % crc == ctx_crc.copy_step_cache_id(seed, "COPY", ". /app/", ctx, ["."]), (n, step)
            if step == "warm":
                assert st["files_reused"] == st["files_total"] and st["bytes_sent"] == 0, st
            if step == "edited":
                assert st["files_reused"] == st["files_total"] - 1, st
    print("cache_id_cold_warm_edited ok")


def cache_id_edges(make, tmp):
    """One file larger than all the others together (LPT gives it an engine of its own), more engines than files, an
    empty context, sources naming single files and a glob, and engines of other CDC parameters (irrelevant here)."""
    from makisu_b200 import abi
    ctx = _crc_ctx(tmp, big=3_000_000)
    for n in ENGINES:
        _cache_id_against(make, ctx, ["."], 512 << 10, n)
        _cache_id_against(make, ctx, ["huge.bin", "d1/s2", "d3/*/f0*.bin"], 512 << 10, n)
    few = os.path.join(tmp, "few")
    cases._mk(os.path.join(few, "a"), b"abc")
    cases._mk(os.path.join(few, "b"), b"")
    empty = os.path.join(tmp, "empty")
    os.makedirs(empty)
    for n in ENGINES:
        _cache_id_against(make, few, ["."], 64 << 10, n)
        _cache_id_against(make, empty, ["."], 64 << 10, n)
        _cache_id_against(make, empty, ["."], 64 << 10, n, prefix=b"")
    from makisu_b200 import host
    engines = [make(64 << 10), make(64 << 10, cdc=abi.CdcParams(2048, 8192, 65536, 15, 11))]
    assert host.context_crc32_multi(engines, b"p", few, ["."])[:2] == host.context_crc32(make(64 << 10), b"p", few, ["."])
    print("cache_id_edges ok")


# ---- batch commit -----------------------------------------------------------------------------------------------
def _commit(run, eng, cache, layers, flags):
    """One batch into a fresh MemFS: eng a list -> commit_layers_multi, else commit_layers_cached.
    -> (MemFS, outs, stats, tar bytes per layer)."""
    from makisu_b200 import host
    fs = host.MemFS(run._dir("root"))
    tdir = run._dir("tars")
    files = [open(os.path.join(tdir, "l%02d.tar" % i), "wb") for i in range(len(layers))]
    try:
        ops, fds = cases.ops_of(run.ctx, layers), [f.fileno() for f in files]
        if isinstance(eng, list):
            outs, st = fs.commit_layers_multi(eng, cache, NOW, ops, 3, fds, flags)
        else:
            outs, st = fs.commit_layers_cached(eng, cache, NOW, ops, 3, fds, flags)
    finally:
        for f in files:
            f.close()
    tars = []
    for f in files:
        with open(f.name, "rb") as g:
            tars.append(g.read())
    return fs, outs, st, tars


def _check_batch(run, make, n, cache, flags, layers=cases.LAYERS, arena=ARENA, **kw):
    """commit_layers_multi over n engines equals commit_layers_cached on one engine with a copy of the cache -> stats."""
    ref = cases.copy_cache(cache, os.path.join(run._dir("cache"), "c")) if cache is not None else None
    engines = [make(arena, **kw) for _ in range(n)]
    before = [e.work() for e in engines]
    fs_m, outs_m, st_m, tars_m = _commit(run, engines, cache, layers, flags)
    assert sum(e.work() != w for e, w in zip(engines, before)) == min(n, len(layers)), n  # every engine given a layer ran
    fs_s, outs_s, st_s, tars_s = _commit(run, make(arena, **kw), ref, layers, flags)
    for i, (a, b) in enumerate(zip(outs_m, outs_s)):
        assert a == b, (n, flags, i, a, b)
    assert len(outs_m) == len(outs_s) == len(layers)
    assert st_m == st_s, (n, flags, st_m, st_s)
    assert tars_m == tars_s, (n, flags)
    run.same_trees(fs_m, fs_s, layers)
    if cache is not None:
        d = run._dir("saved")
        assert _saved(cache, os.path.join(d, "multi")) == _saved(ref, os.path.join(d, "single")), (n, flags)
    return st_m


def batch_cold_warm_edited(make, tmp):
    """The ten layers of tests/commit_layers_cases.py (not a multiple of three engines; a source copied by two layers;
    destinations written by two and three layers) with TarDigest and under MKHOST_NO_TAR_DIGEST, with and
    without MKHOST_FILE_DIGESTS: no cache, then a cold, a warm and a one-file-edited cache.  The warm batch appends both
    remembered rows and the other engines' unique rows to engine 0's session."""
    from makisu_b200 import host
    ctx = cases.make_ctx(tmp)
    run = cases.Runner(make, tmp, ctx)
    NTD, FD = host.MKHOST_NO_TAR_DIGEST, host.MKHOST_FILE_DIGESTS
    for n in ENGINES:
        for flags in (0, NTD, FD, NTD | FD):
            _check_batch(run, make, n, None, flags)
            cache = host.ChunkCache()
            st = _check_batch(run, make, n, cache, flags)
            assert st["files_reused"] == 0, st
            st = _check_batch(run, make, n, cache, flags)
            assert st["files_reused"] == st["files_total"], st
            cases.rewrite(os.path.join(ctx, "d4", "f002.bin"), 10 * n + flags)
            st = _check_batch(run, make, n, cache, flags)
            assert st["files_reused"] == st["files_total"] - 1, st
    print("batch_cold_warm_edited ok")


def batch_small_shapes(make, tmp):
    """One layer only, two layers, and arenas so small that every layer's share of one holds one entry."""
    from makisu_b200 import host
    ctx = cases.make_ctx(tmp)
    run = cases.Runner(make, tmp, ctx)
    for n in ENGINES:
        for layers in (cases.LAYERS[:1], cases.LAYERS[3:4], cases.LAYERS[:2]):
            _check_batch(run, make, n, host.ChunkCache(), host.MKHOST_FILE_DIGESTS, layers=layers)
        cache = host.ChunkCache()
        for _ in range(2):
            _check_batch(run, make, n, cache, 0, arena=256 << 10)
    print("batch_small_shapes ok")


def destination_across_engines(make, tmp):
    """A destination written by two layers that LPT puts on different engines: the two largest layers go to engines 0
    and 1.  Whichever engine hashed the later layer, the tree keeps the later layer's digest."""
    from makisu_b200 import host
    ctx = os.path.join(tmp, "ctx")
    rng = np.random.default_rng(4)
    first, later = rng.bytes(600_000), rng.bytes(500_000)
    for earlier_larger in (True, False):
        a, b = (first, later) if earlier_larger else (later, first)
        cases._mk(os.path.join(ctx, "one", "x.bin"), a)
        cases._mk(os.path.join(ctx, "two", "x.bin"), b)
        cases._mk(os.path.join(ctx, "small", "s.bin"), rng.bytes(1000))
        layers = [[("one/x.bin", "/app/x.bin")], [("small", "/small/")], [("two/x.bin", "/app/x.bin")]]
        run = cases.Runner(make, os.path.join(tmp, str(earlier_larger)), ctx)
        os.makedirs(run.tmp)
        for n in (2, 3):
            for flags in (host.MKHOST_FILE_DIGESTS, host.MKHOST_FILE_DIGESTS | host.MKHOST_NO_TAR_DIGEST):
                _check_batch(run, make, n, host.ChunkCache(), flags, layers=layers)
                fs, _, _, _ = _commit(run, [make(ARENA) for _ in range(n)], None, layers, flags)
                assert fs.file_digest("/app/x.bin") == hashlib.sha256(b).digest()
    print("destination_across_engines ok")


def refusals(make, tmp):
    """A share that overflows its engine's stream slots is refused before any engine takes a submit, and no file digest
    is remembered; engines cut under other CDC parameters are refused; a union of tables larger than engine 0's
    max_chunks fails its finish and the cache records nothing."""
    from makisu_b200 import abi, host
    ctx = cases.make_ctx(tmp)
    run = cases.Runner(make, tmp, ctx)
    FD = host.MKHOST_FILE_DIGESTS
    layers = cases.LAYERS[:4]
    per_layer = [sum(1 for p in cases.sources(ctx, [l]) if os.path.getsize(p)) for l in layers]
    # the share holding the layer with the most files needs one slot more than that layer has files
    slots = max(per_layer)
    engines = [make(ARENA, max_extents=slots) for _ in range(2)]
    before = [e.work() for e in engines]
    try:
        _commit(run, engines, host.ChunkCache(), layers, FD)
        raise AssertionError("expected a refusal")
    except host.HostError as e:
        assert "per-file digests need one stream slot per regular file" in str(e), str(e)
    assert [e.work() for e in engines] == before
    fs = host.MemFS(run._dir("root"))
    try:
        fs.commit_layers_multi([make(ARENA, max_extents=slots) for _ in range(2)], None, NOW, cases.ops_of(ctx, layers),
                               flags=FD)
        raise AssertionError("expected a refusal")
    except host.HostError:
        pass
    assert all(fs.file_digest(d) is None for d in cases.destinations(ctx, layers))
    # enough slots for the whole batch
    _check_batch(run, make, 5, host.ChunkCache(), FD, layers=layers, max_extents=sum(per_layer) + len(layers))
    # other CDC parameters
    other = abi.CdcParams(2048, 8192, 65536, 15, 11)
    try:
        _commit(run, [make(ARENA), make(ARENA, cdc=other)], None, layers, 0)
        raise AssertionError("expected a refusal")
    except host.HostError as e:
        assert "other CDC parameters" in str(e), str(e)
    # the union does not fit engine 0's table: each engine's own rows do
    _, plain, _, _ = _commit(run, make(ARENA), None, cases.LAYERS, 0)
    cap = plain[0]["n_unique"] - 1
    cache = host.ChunkCache()
    try:
        _commit(run, [make(ARENA, max_chunks=cap), make(ARENA)], cache, cases.LAYERS, FD)
        raise AssertionError("expected a refusal")
    except host.HostError as e:
        assert "chunk table overflow" in str(e), str(e)
    assert len(cache) == 0
    # engine 0 holds its own rows and the other engines' unique ones: never more than one engine's rows of the batch
    _check_batch(run, make, 2, host.ChunkCache(), FD, max_chunks=plain[0]["n_chunks"])
    print("refusals ok")


ALL = ["cache_id_cold_warm_edited", "cache_id_edges", "batch_cold_warm_edited", "batch_small_shapes",
       "destination_across_engines", "refusals"]
