"""Scenarios of the sharded layer ingest (mkhost_memfs_update_from_tars_multi), shared by the CPU mock test and the H100
test.  Every scenario compares the call over 1, 2, 3 and 5 engines with update_from_tars_cached on one fresh engine, with
copies of the same caches: the per-layer results, both stats dicts (or the error message), the trees
(layer_cache_cases.Runner.same_trees: remembered file digests and a probe layer described against both), and the bytes
the layer cache and the gz index cache save afterwards.

`make(arena_bytes, max_extents=4096, max_chunks=0, cdc=None)` returns an engine (the CPU mock or libmksnap) with `h`
and `work()`, a value that changes whenever the engine takes a submit."""
from __future__ import annotations

import hashlib
import os
import threading

import numpy as np

from tests import apply_layers as al
from tests import gzip_corpus as gc
from tests import gzip_index as gi
from tests import layer_cache_cases as lcc

NOW = lcc.NOW
ARENA = lcc.ARENA
ENGINES = (1, 2, 3, 5)


def _saved(cache, path) -> bytes:
    if cache is None:
        return b""
    cache.save(path)
    with open(path, "rb") as f:
        return f.read()


def _copy(cache, path):
    """A copy of `cache` through its file (None stays None)."""
    if cache is None:
        return None
    cache.save(path)
    return type(cache)(path)


def _feed(w, blob):
    try:
        view = memoryview(blob)
        while view:
            view = view[os.write(w, view):]
    except BrokenPipeError:  # the call gave up on the layer
        pass
    finally:
        os.close(w)


def _call(run, make, n, paths, layers, keys, flags, lc, gz, arena=ARENA, pipe_at=None, **kw):
    """n engines: update_from_tars_multi; n == 0: update_from_tars_cached on one.  Layer pipe_at is read from a pipe.
    -> (MemFS, result or the HostError raised, engines)."""
    from makisu_b200 import host
    fs = host.MemFS(run._root())
    fds = [os.open(p, os.O_RDONLY) for p in paths]
    writer = None
    if pipe_at is not None:
        os.close(fds[pipe_at])
        fds[pipe_at], w = os.pipe()
        writer = threading.Thread(target=_feed, args=(w, layers[pipe_at][1]))
        writer.start()
    specs = [(f, host.MKHOST_GUNZIP if z else 0) for f, (_, _, z) in zip(fds, layers)]
    engines = [make(arena, **kw) for _ in range(max(1, n))]
    try:
        if n:
            res = fs.update_from_tars_multi(engines, lc, gz, keys, NOW, specs, flags)
        else:
            res = fs.update_from_tars_cached(engines[0], lc, gz, keys, NOW, specs, flags)
    except host.HostError as e:
        res = e
    finally:
        for f in fds:
            os.close(f)
        if writer is not None:
            writer.join()
    return fs, res, engines


def check(run, make, n, paths, layers, keys, flags, lc=None, gz=None, merged=None, **kw):
    """The call over n engines equals update_from_tars_cached on one, with copies of lc and gz -> its result.  The trees
    are compared over the names of `merged` (default: every layer)."""
    from makisu_b200 import host
    d = run._root()
    ref_lc, ref_gz = _copy(lc, os.path.join(d, "lc")), _copy(gz, os.path.join(d, "gz"))
    fs_m, got, _ = _call(run, make, n, paths, layers, keys, flags, lc, gz, **kw)
    fs_s, want, _ = _call(run, make, 0, paths, layers, keys, flags, ref_lc, ref_gz, **kw)
    if isinstance(want, Exception):
        assert isinstance(got, host.HostError), (n, flags, got)
        assert str(got) == str(want), (n, flags, str(got), str(want))
    else:
        assert not isinstance(got, Exception), (n, flags, got)
        assert len(got[0]) == len(layers)
        for i, (a, b) in enumerate(zip(got[0], want[0])):
            assert a == b, (n, flags, i, a, b)
        assert got[1:] == want[1:], (n, flags, got[1:], want[1:])
    if layers:
        run.same_trees(fs_m, fs_s, lcc.plain(layers if merged is None else merged))
    for name, a, b in (("lc", lc, ref_lc), ("gz", gz, ref_gz)):
        assert _saved(a, os.path.join(d, name + ".m")) == _saved(b, os.path.join(d, name + ".s")), (n, flags, name)
    return got


def _setup(tmp, layers):
    paths = lcc.write_blobs(os.path.join(tmp, "blobs"), layers)
    return paths, lcc._keys(layers), lcc.Runner(None, tmp)


# ---- scenarios --------------------------------------------------------------------------------------------------
def cold_warm_touched(make, tmp):
    """layer_cache_cases.layer_set() (plain, pgzip, single- and multi-member gzip, whiteouts, overwrites, hard links, an
    empty layer, a member larger than the arena, PAX and GNU long names) under flags 0, MKHOST_FILE_DIGESTS,
    MKHOST_NO_TAR_DIGEST and both: no cache, then a cold, a warm and a one-blob-touched layer cache with a gz index
    cache.  The warm run replays every layer on engine 0; the touched one mixes replays with an ingest."""
    from makisu_b200 import host
    layers = lcc.layer_set()
    paths, keys, run = _setup(tmp, layers)
    run.make = make
    NTD, FD = host.MKHOST_NO_TAR_DIGEST, host.MKHOST_FILE_DIGESTS
    for n in ENGINES:
        for flags in (0, FD, NTD, NTD | FD):
            check(run, make, n, paths, layers, keys, flags)
            lc, gz = host.LayerCache(), host.GzIndexCache()
            _, st, gst = check(run, make, n, paths, layers, keys, flags, lc, gz)
            assert st["layers_recorded"] == len(layers) and gst["blobs"] == sum(z for _, _, z in layers), (st, gst)
            _, st, _ = check(run, make, n, paths, layers, keys, flags, lc, gz)
            assert st["layers_replayed"] == len(layers) and st["blob_bytes_read"] == 0, st
            s = os.stat(paths[1])
            os.utime(paths[1], ns=(s.st_atime_ns, s.st_mtime_ns + 1000 * (n + 1) + flags))
            _, st, _ = check(run, make, n, paths, layers, keys, flags, lc, gz)
            assert st["layers_replayed"] == len(layers) - 1 and st["layers_recorded"] == 1, st
    print("cold_warm_touched ok")


def across_engines(make, tmp):
    """A layer whose whiteouts and overwrites act on an earlier layer that LPT puts on another engine, with the earlier
    layer the larger and the smaller one: the merge keeps the run's order and the later digest wins."""
    from makisu_b200 import host
    rng = np.random.default_rng(8)
    later_conf = b"x = 2\n" + rng.bytes(1000)
    for earlier_larger in (True, False):
        pad = [("pad.bin", "f", rng.bytes(400_000))]
        l0 = al.tar_of([("app", "d", None), ("app/a.txt", "f", rng.bytes(3000)), ("app/sub", "d", None),
                        ("app/sub/c", "f", rng.bytes(70_000)), ("etc", "d", None), ("etc/conf", "f", b"x = 1\n")]
                       + (pad if earlier_larger else []))
        l1 = al.tar_of([("app/a.txt", "w", None), ("app/sub", "w", None), ("etc/conf", "f", later_conf)]
                       + ([] if earlier_larger else pad))
        layers = [("first", l0, False), ("second", gc.pgzip(l1, block=65536), True)]
        d = os.path.join(tmp, str(earlier_larger))
        paths, keys, run = _setup(d, layers)
        run.make = make
        for n in (2, 3):
            for flags in (0, host.MKHOST_FILE_DIGESTS):
                check(run, make, n, paths, layers, keys, flags, host.LayerCache())
            fs, res, _ = _call(run, make, n, paths, layers, keys, host.MKHOST_FILE_DIGESTS, None, None)
            assert not isinstance(res, Exception), res
            assert fs.file_digest("/etc/conf") == hashlib.sha256(later_conf).digest()
            assert fs.file_digest("/app/a.txt") is None and fs.file_digest("/app/sub/c") is None
    print("across_engines ok")


def same_blob_twice(make, tmp):
    """The same single-member gzip blob twice in one run under one key (each with an fd of its own), around another
    layer: the two go to one engine, so the second open finds the index the first recorded, and gz_stats and the saved
    index are the single call's -- without a layer cache, and cold then warm with one."""
    from makisu_b200 import host
    lib = gi.layer_tar(600_000, 3)
    blob = gi.single(lib)
    other = al.layer_run(big=False)[0]
    layers = [("lib", blob, True), other, ("lib", blob, True)]
    paths, keys, run = _setup(tmp, layers)
    run.make = make
    paths[2], keys[2] = paths[0], keys[0]
    for n in ENGINES:
        gz = host.GzIndexCache()
        _, _, gst = check(run, make, n, paths, layers, keys, 0, None, gz)
        assert gst["blobs"] == 2 and gst["blobs_with_index"] == 1, gst
        _, _, gst = check(run, make, n, paths, layers, keys, 0, None, gz)
        assert gst["blobs_with_index"] == 2, gst
        lc, gz = host.LayerCache(), host.GzIndexCache()
        _, st, gst = check(run, make, n, paths, layers, keys, host.MKHOST_FILE_DIGESTS, lc, gz)
        assert st["layers_recorded"] == 3 and gst["blobs_with_index"] == 1, (st, gst)
        _, st, _ = check(run, make, n, paths, layers, keys, host.MKHOST_FILE_DIGESTS, lc, gz)
        assert st["layers_replayed"] == 3, st
    print("same_blob_twice ok")


def two_damaged(make, tmp):
    """Two damaged single-member gzip layers (CRC-32 flipped) on different engines, a good layer between them: the call
    fails with the lower-indexed layer's message, the single call's; the layers before it stay merged, the layer cache
    records nothing, and the gz index cache gets exactly the single call's entries (the later damaged layer's open also
    succeeded, on its own engine, but its entry is not applied)."""
    from makisu_b200 import host
    run_l = al.layer_run(big=False)

    def damaged(size, seed):
        b = bytearray(gi.single(gi.layer_tar(size, seed)))
        b[-6] ^= 1
        return bytes(b)
    for lower_larger in (True, False):
        a, b = damaged(700_000 if lower_larger else 500_000, 1), damaged(500_000 if lower_larger else 700_000, 2)
        layers = [run_l[0], ("bad_a", a, True), run_l[3], ("bad_b", b, True)]
        d = os.path.join(tmp, str(lower_larger))
        paths, keys, run = _setup(d, layers)
        run.make = make
        for n in ENGINES:
            lc, gz = host.LayerCache(), host.GzIndexCache()
            err = check(run, make, n, paths, layers, keys, 0, lc, gz, merged=[run_l[0], run_l[3]])
            assert isinstance(err, host.HostError) and "CRC-32 or length mismatch" in str(err), err
            assert str(err).startswith("update memfs from tars: "), str(err)
            assert len(lc) == 0 and len(gz) == 1, (len(lc), len(gz))
            fs, err, _ = _call(run, make, n, paths, layers, keys, host.MKHOST_FILE_DIGESTS, None, None)
            assert isinstance(err, host.HostError), err
            assert fs.file_digest("/app/keep") == hashlib.sha256(b"keep\n").digest()  # layer 0 stays merged
            assert fs.file_digest("/app/sub/d") is None                                # layer 2 is not
    print("two_damaged ok")


def refusals(make, tmp):
    """Refused before any engine takes a submit: MKHOST_UNTAR over several engines, engines cut under other CDC
    parameters, a share its engine's stream slots cannot hold (the layer cache left untouched).  A union beyond engine 0's max_chunks fails at finish and
    the layer cache records nothing.  As root, MKHOST_UNTAR over one engine is the single call (files on disk
    included)."""
    from makisu_b200 import abi, host
    layers = al.layer_run(big=False)
    paths, keys, run = _setup(tmp, layers)
    run.make = make
    FD = host.MKHOST_FILE_DIGESTS

    def refused(engines_kw, flags, text):
        for n, kw in engines_kw:
            engines = [make(ARENA, **kw(k)) for k in range(n)]
            before = [e.work() for e in engines]
            fs = host.MemFS(run._root())
            fds = [os.open(p, os.O_RDONLY) for p in paths]
            try:
                fs.update_from_tars_multi(engines, host.LayerCache(), host.GzIndexCache(), keys, NOW,
                                          [(f, host.MKHOST_GUNZIP if z else 0) for f, (_, _, z) in zip(fds, layers)], flags)
                raise AssertionError("expected a refusal")
            except host.HostError as e:
                assert text in str(e), str(e)
            finally:
                for f in fds:
                    os.close(f)
            assert [e.work() for e in engines] == before, text
            assert fs.file_digest("/app/keep") is None

    refused([(n, lambda k: {}) for n in (2, 3, 5)], host.MKHOST_UNTAR, "MKHOST_UNTAR")
    other = abi.CdcParams(2048, 8192, 65536, 15, 11)
    refused([(n, lambda k, last=n - 1: {"cdc": other} if k == last else {}) for n in (2, 3)], 0, "other CDC parameters")
    # four layers over two engines: a share of two or more, with per-file digests, needs three slots or more
    refused([(2, lambda k: {"max_extents": 2})], FD, "is too small")
    # a refusal leaves the layer cache as it was, even one that engines of other CDC parameters would start over
    lc = host.LayerCache()
    check(run, make, 2, paths, layers, keys, 0, lc)
    saved = _saved(lc, os.path.join(tmp, "lc_before"))
    fds = [os.open(p, os.O_RDONLY) for p in paths]
    try:
        host.MemFS(run._root()).update_from_tars_multi(
            [make(ARENA, max_extents=2, cdc=other) for _ in range(2)], lc, None, keys, NOW,
            [(f, host.MKHOST_GUNZIP if z else 0) for f, (_, _, z) in zip(fds, layers)], FD)
        raise AssertionError("expected a refusal")
    except host.HostError as e:
        assert "is too small" in str(e), str(e)
    finally:
        for f in fds:
            os.close(f)
    assert len(lc) == len(layers) and _saved(lc, os.path.join(tmp, "lc_after")) == saved
    check(run, make, 2, paths, layers, keys, FD, host.LayerCache(), max_extents=16)  # enough for the single call
    # the union does not fit engine 0's table: each engine's own rows do
    _, plain, _ = _call(run, make, 0, paths, layers, keys, 0, None, None)
    cap = plain[0][0]["n_unique"] - 1
    lc = host.LayerCache()
    fs = host.MemFS(run._root())
    fds = [os.open(p, os.O_RDONLY) for p in paths]
    try:
        fs.update_from_tars_multi([make(ARENA, max_chunks=cap), make(ARENA)], lc, None, keys, NOW,
                                  [(f, host.MKHOST_GUNZIP if z else 0) for f, (_, _, z) in zip(fds, layers)], 0)
        raise AssertionError("expected a refusal")
    except host.HostError as e:
        assert "chunk table overflow" in str(e), str(e)
    finally:
        for f in fds:
            os.close(f)
    assert len(lc) == 0
    if os.geteuid() == 0:  # MKHOST_UNTAR applies owners (chown)
        from tests.mock_engine import scenarios
        for flags in (host.MKHOST_UNTAR, host.MKHOST_UNTAR | FD):
            fs_m, got, _ = _call(run, make, 1, paths, layers, keys, flags, host.LayerCache(), None, arena=4 << 20)
            root_m = os.path.join(run.tmp, "root%03d" % run.n)
            fs_s, want, _ = _call(run, make, 0, paths, layers, keys, flags, host.LayerCache(), None, arena=4 << 20)
            root_s = os.path.join(run.tmp, "root%03d" % run.n)
            assert not isinstance(got, Exception) and got == want, (got, want)
            run.same_trees(fs_m, fs_s, lcc.plain(layers))
            assert scenarios._tree(root_m, mtimes=True) == scenarios._tree(root_s, mtimes=True)
    print("refusals ok")


def edges(make, tmp):
    """A pipe layer in the run (weight 0, never cached), more engines than layers, one layer, zero layers."""
    from makisu_b200 import host
    layers = al.layer_run()
    paths, keys, run = _setup(tmp, layers)
    run.make = make
    for n in ENGINES:
        for pipe_at in (0, 3):
            lc = host.LayerCache()
            for _ in range(2):
                _, st, _ = check(run, make, n, paths, layers, keys, 0, lc, host.GzIndexCache(), pipe_at=pipe_at)
                assert st["layers_recorded"] + st["layers_replayed"] == len(layers) - 1, st
        check(run, make, n, paths[:2], layers[:2], keys[:2], host.MKHOST_FILE_DIGESTS, host.LayerCache())
        for i in (0, 1, 4):
            check(run, make, n, paths[i:i + 1], layers[i:i + 1], keys[i:i + 1], 0, host.LayerCache(), host.GzIndexCache())
        got = check(run, make, n, [], [], [], 0, host.LayerCache(), host.GzIndexCache())
        assert got[0] == [] and not any(got[1].values()) and not any(got[2].values()), got
    # five engines, two layers: the engines given nothing take no submit
    engines = [make(ARENA) for _ in range(5)]
    before = [e.work() for e in engines]
    fs = host.MemFS(run._root())
    fds = [os.open(p, os.O_RDONLY) for p in paths[:2]]
    try:
        fs.update_from_tars_multi(engines, None, None, keys[:2], NOW, [(fds[0], 0), (fds[1], host.MKHOST_GUNZIP)], 0)
    finally:
        for f in fds:
            os.close(f)
    assert [e.work() != w for e, w in zip(engines, before)] == [True, True, False, False, False]
    print("edges ok")


ALL = ["cold_warm_touched", "across_engines", "same_blob_twice", "two_damaged", "refusals", "edges"]
