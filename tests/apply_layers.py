"""Runs of layer tars for update_from_tars (test infrastructure only): generated layers that act on each other --
whiteouts and overwrites of what an earlier layer added, a hard link to an earlier layer's file, an empty layer, gzip
and plain blobs, a member larger than a 1 MiB arena, a damaged layer -- and the check that one run equals the same
layers applied by one update_from_tar call each."""
from __future__ import annotations

import io
import os
import tarfile
from typing import List, Sequence, Tuple

import numpy as np

from tests import gzip_corpus as gc

T = 1_500_000_000
NOW = 1_600_000_000


def tar_of(entries) -> bytes:
    """entries: (name, kind, payload) with kind 'f' (payload = bytes), 'd', 'l' (symlink target), 'h' (hard link
    target), 'w' (whiteout of `name`: an empty file .wh.<base>)."""
    buf = io.BytesIO()
    with tarfile.open(fileobj=buf, mode="w", format=tarfile.PAX_FORMAT) as tf:
        for name, kind, payload in entries:
            if kind == "w":
                d, b = os.path.split(name)
                name, kind, payload = os.path.join(d, ".wh." + b), "f", b""
            ti = tarfile.TarInfo(name)
            ti.mtime, ti.uid, ti.gid = T, 0, 0
            if kind == "f":
                ti.size, ti.mode = len(payload), 0o644
                tf.addfile(ti, io.BytesIO(payload))
                continue
            ti.type = {"d": tarfile.DIRTYPE, "l": tarfile.SYMTYPE, "h": tarfile.LNKTYPE}[kind]
            ti.mode = 0o755 if kind == "d" else 0o777
            if kind in "lh":
                ti.linkname = payload
            tf.addfile(ti)
    return buf.getvalue()


def layer_run(seed: int = 5, big: bool = True) -> List[Tuple[str, bytes, bool]]:
    """(name, blob, gzip) per layer, in apply order."""
    rng = np.random.default_rng(seed)

    def rnd(n):
        return rng.integers(0, 256, n, dtype=np.uint8).tobytes()

    l0 = tar_of([("app", "d", None), ("app/a.txt", "f", rnd(3000)), ("app/b.bin", "f", rnd(200_000)),
                 ("app/sub", "d", None), ("app/sub/c", "f", rnd(70_000)), ("app/keep", "f", b"keep\n"),
                 ("etc", "d", None), ("etc/conf", "f", b"x = 1\n"), ("app/ln", "l", "a.txt")])
    l1 = tar_of([("app/a.txt", "w", None), ("app/b.bin", "f", rnd(150_000)), ("app/sub", "w", None),
                 ("app/new", "f", rnd(5000)), ("etc/conf", "f", b"x = 2\n")])
    l2 = tar_of([])                                                   # an empty layer
    l3 = tar_of([("app/hard", "h", "app/keep"), ("etc/conf2", "h", "etc/conf"), ("app/sub", "d", None),
                 ("app/sub/d", "f", rnd(40_000))])
    layers = [("adds", l0, False), ("whiteouts_overwrites", l1, True), ("empty", l2, False),
              ("hard_links", l3, True)]
    if big:
        layers.append(("big_member", tar_of([("opt/big.bin", "f", rnd(1_500_000)), ("opt/small", "f", rnd(900))]), False))
    return [(n, gc.pgzip(b, block=65536) if z else b, z) for n, b, z in layers]


def plain(layers) -> List[bytes]:
    return [gc.go_gunzip(b) if z else b for _, b, z in layers]


def regular_bodies(tars: Sequence[bytes]):
    """(concatenation, offsets, lengths) of every regular member with content, over all tars: the bytes one session
    over the whole run chunks."""
    offs, lens, base = [], [], 0
    for t in tars:
        for m in tarfile.open(fileobj=io.BytesIO(t)).getmembers():
            if m.isreg() and m.size and m.type != tarfile.LNKTYPE:
                offs.append(base + m.offset_data)
                lens.append(m.size)
        base += len(t)
    return np.frombuffer(b"".join(tars), dtype=np.uint8), offs, lens


def probe(tars: Sequence[bytes]) -> bytes:
    """A layer naming every path of the run, each as a fresh regular file: describing it against a tree lists which
    of those paths the tree holds differently, so two trees that describe it alike hold the same headers."""
    names = set()
    for t in tars:
        for m in tarfile.open(fileobj=io.BytesIO(t)).getmembers():
            names.add(m.name)
            d = os.path.dirname(m.name)
            while d:
                names.add(d)
                d = os.path.dirname(d)
    return tar_of([(n, "f", b"probe") for n in sorted(names)])


def _open_all(paths):
    return [open(p, "rb") for p in paths]


def apply_both(make_engine, tmp, layers, flags, untar_tree=None, arena_bytes=1 << 20):
    """Apply `layers` once with one update_from_tar per layer and once with update_from_tars; -> (singles, run,
    (memfs_singles, memfs_run), (root_singles, root_run))."""
    from makisu_b200 import host
    paths = []
    for i, (name, blob, z) in enumerate(layers):
        p = os.path.join(tmp, "layer%d_%s%s" % (i, name, ".gz" if z else ".tar"))
        open(p, "wb").write(blob)
        paths.append(p)
    roots = [os.path.join(tmp, "root_single"), os.path.join(tmp, "root_run")]
    for r in roots:
        os.makedirs(r)
    fs_s, fs_r = host.MemFS(roots[0]), host.MemFS(roots[1])
    singles = []
    for p, (_, _, z) in zip(paths, layers):
        with open(p, "rb") as f:
            singles.append(fs_s.update_from_tar(make_engine(arena_bytes), NOW, f.fileno(),
                                                flags=flags | (host.MKHOST_GUNZIP if z else 0)))
    fh = _open_all(paths)
    try:
        run = fs_r.update_from_tars(make_engine(arena_bytes), NOW,
                                    [(f.fileno(), host.MKHOST_GUNZIP if z else 0) for f, (_, _, z) in zip(fh, layers)],
                                    flags=flags)
    finally:
        for f in fh:
            f.close()
    return singles, run, (fs_s, fs_r), roots


def check_run(make_engine, tmp, layers, flags, arena_bytes=1 << 20):
    """update_from_tars equals one update_from_tar per layer: per-layer DiffID, entries and tar bytes; the run's chunk
    table is that of one session over every layer's files; the trees describe a probe layer alike; remembered file
    digests and (MKHOST_UNTAR) the files on disk are the same.  -> run results."""
    import hashlib

    from makisu_b200 import host
    from oracle import lib as olib
    from tests.mock_engine import scenarios
    singles, run, (fs_s, fs_r), roots = apply_both(make_engine, tmp, layers, flags, arena_bytes=arena_bytes)
    tars = plain(layers)
    for i, (s, r) in enumerate(zip(singles, run)):
        for k in ("tar_digest", "n_entries", "tar_bytes"):
            assert s[k] == r[k], (i, k, s[k], r[k])
        if not flags & host.MKHOST_NO_TAR_DIGEST:
            assert r["tar_digest"] == "sha256:" + hashlib.sha256(tars[i]).hexdigest(), i
    arena, offs, lens = regular_bodies(tars)
    want = olib.chunk_table(arena, offs, lens)
    assert all(r["root"] == want["root"] and r["n_chunks"] == want["n_chunks"] and r["n_unique"] == want["n_unique"]
               for r in run)
    names = {m.name for t in tars for m in tarfile.open(fileobj=io.BytesIO(t)).getmembers()}
    for n in names:
        assert fs_s.file_digest("/" + n) == fs_r.file_digest("/" + n), n
    if flags & host.MKHOST_FILE_DIGESTS:
        assert any(fs_r.file_digest("/" + n) is not None for n in names)
    pr = os.path.join(tmp, "probe.tar")
    open(pr, "wb").write(probe(tars))
    texts = []
    for fs in (fs_s, fs_r):  # the probe merges into both trees: it comes after everything else that reads them
        with open(pr, "rb") as f:
            texts.append(fs.describe_update_from_tar(NOW, f.fileno()))
    assert texts[0] == texts[1] and len(texts[0]) > 0
    if flags & host.MKHOST_UNTAR:
        assert scenarios._tree(roots[0], mtimes=True) == scenarios._tree(roots[1], mtimes=True)
    return run
