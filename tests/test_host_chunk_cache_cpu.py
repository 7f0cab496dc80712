"""CPU: incremental layer commit (mkhost_memfs_commit_copy_ops_cached) under the CPU mock of the engine
(tests/mock_engine/mock_mksnap_chunks.cpp: mock_mksnap.cpp plus mksnap_chunks_add / mksnap_arena_submit_spans /
mksnap_get_cdc / mksnap_get_chunks).  The mock zeroes every arena byte outside the spans of a sparse submit, as the
device does, so a cached commit that leaves out a byte the engine reads gets a different root than the uncached one.
Each scenario runs in a fresh process that loads the mock with RTLD_GLOBAL before libmkhost:
    python -m tests.test_host_chunk_cache_cpu <mock.so> <scenario> <tmpdir>"""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
NOW = 1_600_000_000
T = 1_500_000_000


def make_ctx(tmp, seed=5, big=1_500_000):
    """A build context: small and empty files, duplicate content, a symlink, and one file larger than a 1 MiB arena."""
    c = os.path.join(tmp, "ctx")
    rng = np.random.default_rng(seed)

    def mk(rel, data):
        p = os.path.join(c, rel)
        os.makedirs(os.path.dirname(p), exist_ok=True)
        with open(p, "wb") as f:
            f.write(data)
        os.utime(p, (T, T))

    mk("Dockerfile", b"FROM scratch\nCOPY . /app/\n")
    for d in range(3):
        for i in range(5):
            mk(f"d{d}/f{i}.bin", rng.integers(0, 256, int(rng.integers(1, 200_000)), dtype=np.uint8).tobytes())
    same = rng.integers(0, 256, 150_000, dtype=np.uint8).tobytes()
    mk("dup/a.bin", same)
    mk("dup/b.bin", same)
    mk("empty", b"")
    mk("big.bin", rng.integers(0, 256, big, dtype=np.uint8).tobytes())
    os.symlink("big.bin", os.path.join(c, "link"))
    return c


def rewrite(path, seed):
    """New content, same size (and a new mtime/ctime, as an editor leaves it)."""
    n = os.path.getsize(path)
    with open(path, "wb") as f:
        f.write(np.random.default_rng(seed).integers(0, 256, n, dtype=np.uint8).tobytes())


def regular_files(ctx):
    out = []
    for d, _, files in os.walk(ctx):
        for n in files:
            p = os.path.join(d, n)
            if not os.path.islink(p):
                out.append(p)
    return out


def commit(eng, tmp, ctx, cache=None, flags=0, with_tar=True, tag="x"):
    """One layer `COPY . /app/` into a fresh MemFS -> (layer dict, stats dict or None, tar bytes or None).
    cache=False: the plain entry point; None: the cached entry point without a cache."""
    from makisu_b200 import host
    root = os.path.join(tmp, "root")
    os.makedirs(root, exist_ok=True)
    fs = host.MemFS(root)
    ops = [host.CopyOperation(["/"], ctx, "/", "/app/", 3, 4)]
    tar = None
    fd = -1
    if with_tar:
        path = os.path.join(tmp, "layer-%s.tar" % tag)
        f = open(path, "wb")
        fd = f.fileno()
    try:
        if cache is False:
            lay, st = fs.commit_copy_ops(eng, NOW, ops, n_threads=3, tar_fd=fd, flags=flags), None
        else:
            lay, st = fs.commit_copy_ops_cached(eng, cache, NOW, ops, n_threads=3, tar_fd=fd, flags=flags)
    finally:
        if with_tar:
            f.close()
            tar = open(path, "rb").read()
    return lay, st, tar


# ---------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def mock_so(tmp_path_factory):
    out = tmp_path_factory.mktemp("mock")
    obj, so = str(out / "mkoracle.o"), str(out / "libmock_mksnap_chunks.so")
    subprocess.check_call(["gcc", "-O2", "-fPIC", "-c", os.path.join(ROOT, "oracle", "mkoracle.c"), "-o", obj])
    subprocess.check_call(["g++", "-O1", "-g", "-std=c++17", "-fPIC", "-shared", "-Wall",
                           os.path.join(HERE, "mock_engine", "mock_mksnap_chunks.cpp"), obj, "-o", so])
    return so


@pytest.mark.parametrize("scenario", ["cold_warm_and_edited_no_tar_digest", "cold_warm_and_edited_tar_digest",
                                      "save_load_and_cdc_mismatch", "table_overflow_and_no_cache"])
def test_cached_commit_against_the_mock_engine(mock_so, tmp_path, scenario):
    r = subprocess.run([sys.executable, "-m", "tests.test_host_chunk_cache_cpu", mock_so, scenario, str(tmp_path)],
                       cwd=ROOT, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0 and "SCENARIO-OK" in r.stdout, r.stdout[-3000:] + r.stderr[-6000:]


class _Engine:
    def __init__(self, mock, arena=1 << 20, max_extents=1 << 10, max_chunks=0, cdc=None):
        from makisu_b200 import abi
        self.mock = mock
        cfg = abi.Config()
        cfg.n_host_arenas, cfg.host_arena_bytes, cfg.device_arena_bytes = 2, arena, arena
        cfg.max_extents, cfg.max_chunks = max_extents, max_chunks
        if cdc is not None:
            cfg.cdc = cdc
        self.h = C.c_void_p()
        mock.mksnap_create.argtypes = [C.POINTER(abi.Config), C.POINTER(C.c_void_p)]
        assert mock.mksnap_create(C.byref(cfg), C.byref(self.h)) == 0
        mock.mock_chunk_log.restype = C.c_size_t
        mock.mock_chunk_log.argtypes = [C.c_void_p, C.c_char_p, C.c_size_t]

    def log(self):
        n = self.mock.mock_chunk_log(self.h, None, 0)
        buf = C.create_string_buffer(n)
        self.mock.mock_chunk_log(self.h, buf, n)
        return [l for l in buf.value.decode().split("\n") if l]


def _submits(log):
    """(used, CDC extents, rows) of every submit, and the bytes of its spans (None: not a sparse submit)."""
    out = []
    for l in log:
        if l.startswith("submit"):
            head, _, sp = l.partition(" spans")
            kv = dict(x.split("=") for x in head.split()[1:])
            spans = [tuple(int(v) for v in s.split("+")) for s in sp.split()] if " spans" in l else None
            out.append((int(kv["used"]), int(kv["cdc"]), int(kv["rows"]), spans))
    return out


def _added(log):
    return sum(int(l.split()[1]) for l in log if l.startswith("add "))


def _same_layer(a, b):
    for k in ("tar_digest", "root", "n_entries", "tar_bytes", "n_chunks", "n_unique"):
        assert a[k] == b[k], (k, a[k], b[k])


def _cold_warm_edited(mock, tmp, flags):
    from makisu_b200 import host
    tar_digest = not (flags & host.MKHOST_NO_TAR_DIGEST)
    ctx = make_ctx(tmp)
    files = regular_files(ctx)
    total = sum(os.path.getsize(p) for p in files)
    eng = _Engine(mock)
    ref, _, ref_tar = commit(eng, tmp, ctx, cache=False, flags=flags, tag="ref")
    ref_log = _submits(eng.log())
    assert all(s[3] is None for s in ref_log)

    # cold: the uncached commit, the same CDC extents in the same submits, every file remembered
    cache = host.ChunkCache()
    cold, st, tar = commit(eng, tmp, ctx, cache=cache, flags=flags, tag="cold")
    _same_layer(cold, ref)
    assert tar == ref_tar
    log = _submits(eng.log())
    assert [s[:3] for s in log] == [s[:3] for s in ref_log] and _added(eng.log()) == 0
    assert st == {"files_total": len(files), "files_reused": 0, "bytes_total": total, "bytes_chunked": total,
                  "bytes_uploaded": total}
    assert len(cache) == len(files)
    for used, n_cdc, _, spans in log:  # the tar headers between file bodies are joined into one span
        assert all(o % 16 == 0 and n % 16 == 0 and o + n <= used for o, n in spans)
        assert len(spans) == (1 if n_cdc or tar_digest else 0)

    # warm: nothing chunked, every digest appended, the same layer
    warm, st, tar = commit(eng, tmp, ctx, cache=cache, flags=flags, tag="warm")
    _same_layer(warm, ref)
    assert tar == ref_tar
    log = _submits(eng.log())
    assert all(n_cdc == 0 and rows == 0 for _, n_cdc, rows, _ in log) and _added(eng.log()) == ref["n_chunks"]
    assert st["files_reused"] == st["files_total"] == len(files) and st["bytes_chunked"] == 0
    if tar_digest:  # the TarDigest chain reads every byte: the stream travels whole
        assert st["bytes_uploaded"] == total
        assert all(len(sp) == 1 for *_, sp in log)
    else:           # nothing on the device reads a byte: nothing travels
        assert st["bytes_uploaded"] == 0 and all(sp == [] for *_, sp in log)
        # without a tar to write nothing is read from disk either: the arena keeps the mock's poison where the bodies
        # would be, and the result holds
        quiet, st2, _ = commit(eng, tmp, ctx, cache=cache, flags=flags, with_tar=False)
        _same_layer(quiet, ref)
        assert st2["files_reused"] == len(files)

    # one small file and the file larger than the arena rewritten with the same sizes: only they are chunked
    for rel, seed in (("d1/f2.bin", 11), ("big.bin", 12)):
        rewrite(os.path.join(ctx, rel), seed)
    want, _, want_tar = commit(eng, tmp, ctx, cache=False, flags=flags, tag="ref2")
    edited, st, tar = commit(eng, tmp, ctx, cache=cache, flags=flags, tag="edited")
    _same_layer(edited, want)
    assert tar == want_tar and edited["root"] != ref["root"]
    changed = os.path.getsize(os.path.join(ctx, "d1/f2.bin")) + os.path.getsize(os.path.join(ctx, "big.bin"))
    assert st["files_reused"] == len(files) - 2 and st["bytes_chunked"] == changed
    assert st["bytes_uploaded"] == (total if tar_digest else changed)
    again, st, _ = commit(eng, tmp, ctx, cache=cache, flags=flags, tag="again")
    _same_layer(again, want)
    assert st["files_reused"] == len(files)

    # a duplicate of a cached file's content in a new file: n_unique dedups across remembered and fresh rows
    with open(os.path.join(ctx, "dup", "a.bin"), "rb") as f:
        same = f.read()
    with open(os.path.join(ctx, "dup", "c.bin"), "wb") as f:
        f.write(same)
    want, _, _ = commit(eng, tmp, ctx, cache=False, flags=flags, tag="ref3")
    got, st, _ = commit(eng, tmp, ctx, cache=cache, flags=flags, tag="dup")
    _same_layer(got, want)
    assert st["files_reused"] == len(files) and got["n_chunks"] > got["n_unique"]


def cold_warm_and_edited_no_tar_digest(mock, tmp):
    from makisu_b200 import host
    _cold_warm_edited(mock, tmp, host.MKHOST_NO_TAR_DIGEST)


def cold_warm_and_edited_tar_digest(mock, tmp):
    _cold_warm_edited(mock, tmp, 0)


def save_load_and_cdc_mismatch(mock, tmp):
    from makisu_b200 import abi, host
    ctx = make_ctx(tmp)
    n_files = len(regular_files(ctx))
    eng = _Engine(mock)
    cache = host.ChunkCache()
    ref, _, _ = commit(eng, tmp, ctx, cache=cache, flags=host.MKHOST_NO_TAR_DIGEST, with_tar=False)
    path = os.path.join(tmp, "chunks.cache")
    cache.save(path)
    loaded = host.ChunkCache(path)
    assert len(loaded) == len(cache) == n_files
    got, st, _ = commit(eng, tmp, ctx, cache=loaded, flags=host.MKHOST_NO_TAR_DIGEST, with_tar=False)
    _same_layer(got, ref)
    assert st["files_reused"] == n_files and st["bytes_uploaded"] == 0
    loaded.save(path + ".2")
    assert open(path, "rb").read() == open(path + ".2", "rb").read()
    # an engine cut under other parameters: the cache counts as empty, the layer is that engine's own
    cdc = abi.CdcParams(2048, 8192, 65536, 15, 11)
    other = _Engine(mock, cdc=cdc)
    want, _, _ = commit(other, tmp, ctx, cache=False, flags=host.MKHOST_NO_TAR_DIGEST, with_tar=False)
    got, st, _ = commit(other, tmp, ctx, cache=loaded, flags=host.MKHOST_NO_TAR_DIGEST, with_tar=False)
    _same_layer(got, want)
    assert got["root"] != ref["root"] and st["files_reused"] == 0 and st["bytes_chunked"] == st["bytes_total"]
    loaded.save(path + ".3")  # ... and now holds the other parameters' digests: the first engine starts over again
    back = host.ChunkCache(path + ".3")
    got, st, _ = commit(eng, tmp, ctx, cache=back, flags=host.MKHOST_NO_TAR_DIGEST, with_tar=False)
    _same_layer(got, ref)
    assert st["files_reused"] == 0
    # loading a file saved under other parameters on top replaces the entries instead of mixing them
    back.load(path)
    assert len(back) == n_files
    _, st, _ = commit(eng, tmp, ctx, cache=back, flags=host.MKHOST_NO_TAR_DIGEST, with_tar=False)
    assert st["files_reused"] == n_files
    with open(path + ".bad", "wb") as f:
        f.write(b"mkhost-crc-cache 1\n")
    with pytest.raises(host.HostError, match="not a mkhost-chunk-cache file"):
        host.ChunkCache(path + ".bad")
    with open(path + ".cut", "wb") as f:  # cut inside the digests of big.bin (the second entry; it has many)
        data = open(path, "rb").read()
        f.write(data[:data.index(b"big.bin\n") + 8 + 100])
    with pytest.raises(host.HostError):
        host.ChunkCache(path + ".cut")


def table_overflow_and_no_cache(mock, tmp):
    from makisu_b200 import host
    ctx = make_ctx(tmp)
    eng = _Engine(mock)
    cache = host.ChunkCache()
    ref, _, ref_tar = commit(eng, tmp, ctx, cache=cache, flags=host.MKHOST_NO_TAR_DIGEST)
    # the cached entry point without a cache is the plain commit: no spans, nothing appended
    got, st, tar = commit(eng, tmp, ctx, cache=None, flags=host.MKHOST_NO_TAR_DIGEST)
    _same_layer(got, ref)
    assert tar == ref_tar and all(s[3] is None for s in _submits(eng.log())) and _added(eng.log()) == 0
    assert st["files_reused"] == 0 and st["bytes_chunked"] == st["bytes_total"]
    # remembered rows past max_chunks: a capacity error at finish, like computed chunks
    small = _Engine(mock, max_chunks=ref["n_chunks"] - 1)
    with pytest.raises(host.HostError, match="chunk table overflow"):
        commit(small, tmp, ctx, cache=cache, flags=host.MKHOST_NO_TAR_DIGEST, with_tar=False)


def main():
    mock_path, scenario, tmp = sys.argv[1:4]
    mock = C.CDLL(mock_path, mode=C.RTLD_GLOBAL)  # BEFORE anything loads libmksnap / libmkhost
    from makisu_b200 import host
    host.load()
    assert C.cast(mock.mksnap_chunks_add, C.c_void_p).value == C.cast(C.CDLL(None).mksnap_chunks_add, C.c_void_p).value, \
        "libmkhost is not bound to the mock engine"
    globals()[scenario](mock, tmp)
    print("SCENARIO-OK", scenario)


if __name__ == "__main__":
    main()
