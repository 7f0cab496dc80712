"""Scenarios of the incremental layer ingest (MemFS.update_from_tars_cached with a LayerCache), shared by the CPU mock
test and the H100 test.  Every scenario compares the cached call with update_from_tars_indexed on a fresh MemFS: the
per-layer results and the run's chunk table, the remembered file digests, a probe layer described against both trees
(tests/apply_layers.py) and, under MKHOST_UNTAR, the files on disk.

`make(arena_bytes, cdc=None, max_chunks=0)` returns an engine (the CPU mock or libmksnap)."""
from __future__ import annotations

import io
import os
import tarfile
import threading

import numpy as np

from tests import apply_layers as al
from tests import gzip_corpus as gc
from tests import gzip_index as gi

NOW = al.NOW
ARENA = 1 << 20


def _gnu_tar(entries) -> bytes:
    """GNU-format tar: names and link targets longer than 100 bytes travel in ././@LongLink members."""
    buf = io.BytesIO()
    with tarfile.open(fileobj=buf, mode="w", format=tarfile.GNU_FORMAT) as tf:
        for name, kind, payload in entries:
            ti = tarfile.TarInfo(name)
            ti.mtime = al.T
            if kind == "f":
                ti.size, ti.mode = len(payload), 0o644
                tf.addfile(ti, io.BytesIO(payload))
            else:
                ti.type, ti.linkname, ti.mode = tarfile.SYMTYPE, payload, 0o777
                tf.addfile(ti)
    return buf.getvalue()


def layer_set(seed: int = 5, big: bool = True):
    """(name, blob, gzip) per layer: the run of tests/apply_layers.py (plain and pgzip blobs, whiteouts, overwrites,
    hard links, an empty layer, a member larger than the arena) plus a single-member and a multi-member gzip blob and
    PAX and GNU long names."""
    rng = np.random.default_rng(seed + 100)
    layers = al.layer_run(seed, big=big)
    long_dir = "srv/" + "d" * 120
    pax = al.tar_of([("srv", "d", None), (long_dir, "d", None), (long_dir + "/pax_" + "p" * 90, "f", rng.bytes(30_000)),
                     ("srv/lnk", "l", long_dir + "/pax_" + "p" * 90)])
    gnu = _gnu_tar([(long_dir + "/gnu_" + "g" * 110, "f", rng.bytes(20_000)),
                    ("srv/glnk", "l", long_dir + "/gnu_" + "g" * 110)])
    lib = gi.layer_tar(600_000, seed)
    half = len(lib) // 2
    layers += [("pax_long_names", pax, False), ("gnu_long_names", gnu, False),
               ("single_member", gi.single(lib), True),
               ("multi_member", gi.single(lib[:half], 1) + gi.single(lib[half:], 9), True)]
    return layers


def write_blobs(tmp, layers):
    os.makedirs(tmp, exist_ok=True)
    paths = []
    for i, (name, blob, _) in enumerate(layers):
        paths.append(os.path.join(tmp, "blob%02d_%s" % (i, name)))
        with open(paths[-1], "wb") as f:
            f.write(blob)
    return paths


def plain(layers):
    return [gc.go_gunzip(b) if z else b for _, b, z in layers]


class Runner:
    """Applies runs of blobs to fresh trees, cached and uncached, and compares them."""

    def __init__(self, make, tmp):
        self.make, self.tmp, self.n = make, tmp, 0

    def _root(self):
        self.n += 1
        r = os.path.join(self.tmp, "root%03d" % self.n)
        os.makedirs(r)
        return r

    def apply(self, paths, gz_flags, call, arena=ARENA, **kw):
        """-> (MemFS, root, call result or the HostError raised)."""
        from makisu_b200 import host
        root = self._root()
        fs = host.MemFS(root)
        fds = [os.open(p, os.O_RDONLY) for p in paths]
        try:
            res = call(fs, self.make(arena, **kw), [(f, g) for f, g in zip(fds, gz_flags)])
        except host.HostError as e:
            res = e
        finally:
            for f in fds:
                os.close(f)
        return fs, root, res

    def check(self, paths, layers, keys, flags, lc, gz=None, arena=ARENA, **kw):
        """The cached call equals update_from_tars_indexed on a fresh tree -> (outs, stats, gz stats)."""
        from makisu_b200 import host
        from tests.mock_engine import scenarios
        g = [host.MKHOST_GUNZIP if z else 0 for _, _, z in layers]
        fs_r, root_r, ref = self.apply(paths, g, lambda fs, e, s: fs.update_from_tars_indexed(e, None, keys, NOW, s, flags),
                                       arena, **kw)
        fs_c, root_c, got = self.apply(paths, g, lambda fs, e, s: fs.update_from_tars_cached(e, lc, gz, keys, NOW, s, flags),
                                       arena, **kw)
        assert not isinstance(ref, Exception), ref
        assert not isinstance(got, Exception), got
        assert got[0] == ref[0], (got[0], ref[0])
        self.same_trees(fs_r, fs_c, plain(layers))
        if flags & host.MKHOST_UNTAR:
            assert scenarios._tree(root_r, mtimes=True) == scenarios._tree(root_c, mtimes=True)
        return got

    def same_trees(self, fs_a, fs_b, tars):
        names = {m.name for t in tars for m in tarfile.open(fileobj=io.BytesIO(t)).getmembers()}
        for n in names:
            assert fs_a.file_digest("/" + n) == fs_b.file_digest("/" + n), n
        pr = os.path.join(self.tmp, "probe%03d.tar" % self.n)
        with open(pr, "wb") as f:
            f.write(al.probe(tars))
        texts = []
        for fs in (fs_a, fs_b):
            with open(pr, "rb") as f:
                texts.append(fs.describe_update_from_tar(NOW, f.fileno()))
        assert texts[0] == texts[1] and texts[0]


def _keys(layers):
    return ["sha%02d_%s" % (i, n) for i, (n, _, _) in enumerate(layers)]


# ---- scenarios --------------------------------------------------------------------------------------------------
def cold_warm(make, tmp):
    """Cold: equal to the uncached run, every layer recorded.  Warm: equal, every layer replayed, nothing read; the gz
    entries of replayed gzip layers stay as they were."""
    from makisu_b200 import host
    layers = layer_set()
    paths = write_blobs(os.path.join(tmp, "blobs"), layers)
    keys, n = _keys(layers), len(layers)
    run = Runner(make, tmp)
    for flags in (0, host.MKHOST_FILE_DIGESTS, host.MKHOST_NO_TAR_DIGEST):
        lc, gz = host.LayerCache(), host.GzIndexCache()
        outs, st, gst = run.check(paths, layers, keys, flags, lc, gz)
        assert st == {"layers": n, "layers_replayed": 0, "layers_recorded": n, "chunks_appended": 0,
                      "blob_bytes_read": sum(len(b) for _, b, _ in layers)}, st
        assert len(lc) == n and gst["blobs"] == sum(z for _, _, z in layers)
        gz_before = os.path.join(tmp, "gz_before_%d" % flags)
        gz.save(gz_before)
        outs2, st, gst = run.check(paths, layers, keys, flags, lc, gz)
        assert outs2 == outs
        assert st == {"layers": n, "layers_replayed": n, "layers_recorded": 0, "blob_bytes_read": 0,
                      "chunks_appended": outs[0]["n_chunks"]}, st
        assert not any(gst.values()), gst
        gz_after = os.path.join(tmp, "gz_after_%d" % flags)
        gz.save(gz_after)
        assert open(gz_before, "rb").read() == open(gz_after, "rb").read()
    print("cold_warm ok")


def mixed(make, tmp):
    """cached, new, cached: the new layer whites out and overwrites what the first added, the last hard-links to it."""
    from makisu_b200 import host
    layers = al.layer_run(big=False)  # adds, whiteouts_overwrites, empty, hard_links
    paths = write_blobs(os.path.join(tmp, "blobs"), layers)
    keys = _keys(layers)
    run = Runner(make, tmp)
    for flags in (0, host.MKHOST_FILE_DIGESTS):
        lc = host.LayerCache()
        sel = [0, 3]
        run.check([paths[i] for i in sel], [layers[i] for i in sel], [keys[i] for i in sel], flags, lc)
        assert len(lc) == 2
        sel = [0, 1, 3]
        outs, st, _ = run.check([paths[i] for i in sel], [layers[i] for i in sel], [keys[i] for i in sel], flags, lc)
        assert st["layers_replayed"] == 2 and st["layers_recorded"] == 1, st
        assert st["blob_bytes_read"] == len(layers[1][1]) and len(lc) == 3
    print("mixed ok")


def misses(make, tmp):
    """touch, a same-size rewrite and a key whose entry is another file's are misses, recorded afresh."""
    from makisu_b200 import host
    layers = al.layer_run(big=False)
    paths = write_blobs(os.path.join(tmp, "blobs"), layers)
    keys, n = _keys(layers), len(layers)
    run = Runner(make, tmp)
    lc = host.LayerCache()
    run.check(paths, layers, keys, 0, lc)
    st = os.stat(paths[0])
    os.utime(paths[0], ns=(st.st_atime_ns, st.st_mtime_ns + 1000))          # touch
    _, s, _ = run.check(paths, layers, keys, 0, lc)
    assert s["layers_replayed"] == n - 1 and s["layers_recorded"] == 1, s
    with open(paths[1], "r+b") as f:                                          # same size, same bytes
        f.write(layers[1][1])
    _, s, _ = run.check(paths, layers, keys, 0, lc)
    assert s["layers_replayed"] == n - 1 and s["layers_recorded"] == 1, s
    _, s, _ = run.check(paths, layers, keys, 0, lc)
    assert s["layers_replayed"] == n, s
    swapped = [keys[3], keys[1], keys[2], keys[0]]                            # each key names another file's entry
    _, s, _ = run.check(paths, layers, swapped, 0, lc)
    assert s["layers_replayed"] == 2 and s["layers_recorded"] == 2, s       # layers 1 and 2 kept their keys
    _, s, _ = run.check(paths, layers, [None] * n, 0, lc)                    # no keys: no cache
    assert s["layers_replayed"] == s["layers_recorded"] == 0 and s["blob_bytes_read"] > 0, s
    print("misses ok")


def what_an_entry_holds(make, tmp):
    """An entry recorded under MKHOST_NO_TAR_DIGEST cannot serve a DiffID; one recorded without MKHOST_FILE_DIGESTS
    cannot serve file digests; an entry with both serves a call that wants neither."""
    from makisu_b200 import host
    layers = al.layer_run(big=False)
    paths = write_blobs(os.path.join(tmp, "blobs"), layers)
    keys, n = _keys(layers), len(layers)
    run = Runner(make, tmp)
    NTD, FD = host.MKHOST_NO_TAR_DIGEST, host.MKHOST_FILE_DIGESTS
    lc = host.LayerCache()
    run.check(paths, layers, keys, NTD, lc)
    _, s, _ = run.check(paths, layers, keys, NTD, lc)
    assert s["layers_replayed"] == n, s
    _, s, _ = run.check(paths, layers, keys, 0, lc)          # needs DiffIDs: recorded again, now with them
    assert s["layers_replayed"] == 0 and s["layers_recorded"] == n, s
    _, s, _ = run.check(paths, layers, keys, FD, lc)         # needs file digests
    assert s["layers_replayed"] == 0 and s["layers_recorded"] == n, s
    for flags in (FD, 0, NTD, NTD | FD):                    # the entry now holds both
        _, s, _ = run.check(paths, layers, keys, flags, lc)
        assert s["layers_replayed"] == n, (flags, s)
    print("what_an_entry_holds ok")


def other_cdc(make, tmp):
    """An engine cut under other CDC parameters: the cache starts over."""
    from makisu_b200 import abi, host
    layers = al.layer_run(big=False)
    paths = write_blobs(os.path.join(tmp, "blobs"), layers)
    keys, n = _keys(layers), len(layers)
    run = Runner(make, tmp)
    lc = host.LayerCache()
    run.check(paths, layers, keys, 0, lc)
    other = abi.CdcParams(2048, 8192, 65536, 15, 11)
    _, s, _ = run.check(paths[:2], layers[:2], keys[:2], 0, lc, cdc=other)
    assert s["layers_replayed"] == 0 and s["layers_recorded"] == 2 and len(lc) == 2, (s, len(lc))
    _, s, _ = run.check(paths[:2], layers[:2], keys[:2], 0, lc, cdc=other)
    assert s["layers_replayed"] == 2, s
    _, s, _ = run.check(paths, layers, keys, 0, lc)         # and back
    assert s["layers_replayed"] == 0 and len(lc) == n, s
    print("other_cdc ok")


def untar(make, tmp):
    """MKHOST_UNTAR records but never replays; a later call without it replays what it recorded."""
    from makisu_b200 import host
    layers = al.layer_run(big=False)
    paths = write_blobs(os.path.join(tmp, "blobs"), layers)
    keys, n = _keys(layers), len(layers)
    run = Runner(make, tmp)
    lc = host.LayerCache()
    for flags in (host.MKHOST_UNTAR, host.MKHOST_UNTAR | host.MKHOST_FILE_DIGESTS):
        for _ in range(2):
            _, s, _ = run.check(paths, layers, keys, flags, lc, arena=4 << 20)
            assert s["layers_replayed"] == 0 and s["layers_recorded"] == n, s
    _, s, _ = run.check(paths, layers, keys, host.MKHOST_FILE_DIGESTS, lc)
    assert s["layers_replayed"] == n, s
    print("untar ok")


def pipe(make, tmp):
    """A layer read from a pipe is neither recorded nor replayed."""
    from makisu_b200 import host
    layers = al.layer_run(big=False)[:2]
    paths = write_blobs(os.path.join(tmp, "blobs"), layers)
    keys = _keys(layers)
    run = Runner(make, tmp)
    lc = host.LayerCache()
    run.check(paths, layers, keys, 0, lc)
    assert len(lc) == 2

    def through_pipe(fs, e, specs):
        r, w = os.pipe()
        t = threading.Thread(target=lambda: (os.write(w, layers[0][1]), os.close(w)))
        t.start()
        try:
            return fs.update_from_tars_cached(e, lc, None, keys, NOW, [(r, specs[0][1]), specs[1]], 0)
        finally:
            t.join()
            os.close(r)
    g = [host.MKHOST_GUNZIP if z else 0 for _, _, z in layers]
    for _ in range(2):
        fs_r, _, ref = run.apply(paths, g, lambda fs, e, s: fs.update_from_tars_indexed(e, None, keys, NOW, s, 0))
        fs_c, _, got = run.apply(paths, g, through_pipe)
        assert not isinstance(got, Exception), got
        assert got[0] == ref[0] and got[1]["layers_replayed"] == 1 and got[1]["layers_recorded"] == 0, got[1]
        assert got[1]["blob_bytes_read"] == len(layers[0][1]) and len(lc) == 2
        run.same_trees(fs_r, fs_c, plain(layers))
    print("pipe ok")


def save_load(make, tmp):
    """Save and load round-trip (the loaded cache replays every layer); a damaged file fails the load and leaves the
    cache as it was."""
    from makisu_b200 import host
    layers = layer_set(big=False)
    paths = write_blobs(os.path.join(tmp, "blobs"), layers)
    keys, n = _keys(layers), len(layers)
    run = Runner(make, tmp)
    for flags in (0, host.MKHOST_FILE_DIGESTS):
        lc = host.LayerCache()
        run.check(paths, layers, keys, flags, lc)
        path = os.path.join(tmp, "layers%d.cache" % flags)
        lc.save(path)
        loaded = host.LayerCache(path)
        assert len(loaded) == n
        again = os.path.join(tmp, "again%d.cache" % flags)
        loaded.save(again)
        good = open(path, "rb").read()
        assert open(again, "rb").read() == good
        _, s, _ = run.check(paths, layers, keys, flags, loaded)
        assert s["layers_replayed"] == n and s["blob_bytes_read"] == 0, s
    rng = np.random.default_rng(3)
    damaged = [good[:k] for k in (0, 5, len(good) // 3, len(good) - 1)] + [good + b"\0", b"x" + good[1:]]
    for _ in range(40):
        b = bytearray(good)
        for _ in range(4):
            b[int(rng.integers(21, 200))] ^= 0xFF  # counts and lengths of the header and the first entry
        damaged.append(bytes(b))
    bad = os.path.join(tmp, "bad.cache")
    refused = 0
    for d in damaged:
        with open(bad, "wb") as f:
            f.write(d)
        probe = host.LayerCache(path)
        try:
            probe.load(bad)
        except host.HostError as e:
            assert "not a mkhost-layer-cache file" in str(e), str(e)
            refused += 1
            assert len(probe) == n
            _, s, _ = run.check(paths[:2], layers[:2], keys[:2], flags, probe)
            assert s["layers_replayed"] == 2, s
    assert refused >= 6, refused
    print("save_load ok", refused)


def no_cache(make, tmp):
    """lc == None: the _indexed call (gz entries and gz stats included)."""
    from makisu_b200 import host
    layers = layer_set()
    paths = write_blobs(os.path.join(tmp, "blobs"), layers)
    keys = _keys(layers)
    run = Runner(make, tmp)
    g = [host.MKHOST_GUNZIP if z else 0 for _, _, z in layers]
    for flags in (0, host.MKHOST_FILE_DIGESTS):
        gz_a, gz_b = host.GzIndexCache(), host.GzIndexCache()
        fs_a, _, a = run.apply(paths, g, lambda fs, e, s: fs.update_from_tars_indexed(e, gz_a, keys, NOW, s, flags))
        fs_b, _, b = run.apply(paths, g, lambda fs, e, s: fs.update_from_tars_cached(e, None, gz_b, keys, NOW, s, flags))
        assert b[0] == a[0] and b[2] == a[1], (a, b)
        assert b[1]["layers_replayed"] == b[1]["layers_recorded"] == 0 and b[1]["layers"] == len(layers)
        pa, pb = os.path.join(tmp, "gz_a"), os.path.join(tmp, "gz_b")
        gz_a.save(pa)
        gz_b.save(pb)
        assert open(pa, "rb").read() == open(pb, "rb").read()
        run.same_trees(fs_a, fs_b, plain(layers))
    print("no_cache ok")


def corrupt_middle(make, tmp):
    """A damaged layer in the middle: the call fails like the uncached one, the layers before it stay merged, and the
    cache records nothing -- with the first layer cold and with it replayed."""
    from makisu_b200 import host
    layers = al.layer_run(big=False)
    bad = bytearray(layers[1][1])
    bad[-6] ^= 1  # gzip CRC-32
    run3 = [layers[0], ("damaged", bytes(bad), True), layers[3]]
    paths = write_blobs(os.path.join(tmp, "blobs"), run3)
    keys = _keys(run3)
    run = Runner(make, tmp)
    g = [host.MKHOST_GUNZIP if z else 0 for _, _, z in run3]
    for warm_first in (False, True):
        lc = host.LayerCache()
        if warm_first:
            run.check(paths[:1], run3[:1], keys[:1], 0, lc)
        fs_r, _, ref = run.apply(paths, g, lambda fs, e, s: fs.update_from_tars_indexed(e, None, keys, NOW, s, 0))
        fs_c, _, got = run.apply(paths, g, lambda fs, e, s: fs.update_from_tars_cached(e, lc, None, keys, NOW, s, 0))
        assert isinstance(ref, host.HostError) and isinstance(got, host.HostError)
        assert str(got) == str(ref) and "CRC-32 or length mismatch" in str(got), str(got)
        assert len(lc) == (1 if warm_first else 0)
        run.same_trees(fs_r, fs_c, plain([layers[0], layers[1], layers[3]]))
    print("corrupt_middle ok")


ALL = ["cold_warm", "mixed", "misses", "what_an_entry_holds", "other_cdc", "pipe", "save_load", "no_cache",
       "corrupt_middle"]
