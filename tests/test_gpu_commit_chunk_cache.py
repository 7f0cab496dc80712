"""GPU: incremental layer commit -- remembered chunk digests for unchanged files (mkhost_memfs_commit_copy_ops_cached)
and the engine entry points under it (mksnap_chunks_add, mksnap_arena_submit_spans, mksnap_get_cdc).  Every cached
result is compared with the uncached commit of the same tree on the same engine."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

from tests.test_host_chunk_cache_cpu import commit, make_ctx, regular_files, rewrite

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)


def _engine(arena=1 << 20, **kw):
    from makisu_b200.abi import Engine
    return Engine(device=0, device_arena_bytes=arena, n_host_arenas=2, host_arena_bytes=arena, max_extents=1 << 10, **kw)


def _same_layer(a, b):
    for k in ("tar_digest", "root", "n_entries", "tar_bytes", "n_chunks", "n_unique"):
        assert a[k] == b[k], (k, a[k], b[k])


@pytest.mark.parametrize("no_tar_digest", [True, False])
def test_cold_warm_edited_and_duplicates(tmp_path, no_tar_digest):
    from makisu_b200 import host
    flags = host.MKHOST_NO_TAR_DIGEST if no_tar_digest else 0
    tmp = str(tmp_path)
    ctx = make_ctx(tmp)  # includes a file larger than the 1 MiB arena
    files = regular_files(ctx)
    total = sum(os.path.getsize(p) for p in files)
    with _engine() as eng:
        ref, _, ref_tar = commit(eng, tmp, ctx, cache=False, flags=flags, tag="ref")
        # 1. cold: the uncached result, and the cache holds every regular file
        cache = host.ChunkCache()
        cold, st, tar = commit(eng, tmp, ctx, cache=cache, flags=flags, tag="cold")
        _same_layer(cold, ref)
        assert tar == ref_tar and len(cache) == len(files)
        assert st == {"files_total": len(files), "files_reused": 0, "bytes_total": total, "bytes_chunked": total,
                      "bytes_uploaded": total}
        # 2. warm: identical, nothing chunked; without TarDigest the file bytes stay on the host
        h2d0 = eng.stats().h2d_bytes
        warm, st, tar = commit(eng, tmp, ctx, cache=cache, flags=flags, tag="warm")
        h2d = eng.stats().h2d_bytes - h2d0
        _same_layer(warm, ref)
        assert tar == ref_tar
        assert st["files_reused"] == st["files_total"] == len(files) and st["bytes_chunked"] == 0
        if no_tar_digest:
            assert st["bytes_uploaded"] == 0
            assert h2d < total // 8, (h2d, total)  # digests and tables only
            quiet, st, _ = commit(eng, tmp, ctx, cache=cache, flags=flags, with_tar=False)  # nothing read at all
            _same_layer(quiet, ref)
        else:
            assert st["bytes_uploaded"] == total and h2d >= total
        # 3. one small file and the file larger than the arena rewritten, same sizes: only they are chunked
        for rel, seed in (("d1/f2.bin", 11), ("big.bin", 12)):
            rewrite(os.path.join(ctx, rel), seed)
        want, _, want_tar = commit(eng, tmp, ctx, cache=False, flags=flags, tag="ref2")
        got, st, tar = commit(eng, tmp, ctx, cache=cache, flags=flags, tag="edited")
        _same_layer(got, want)
        assert tar == want_tar and got["root"] != ref["root"]
        changed = os.path.getsize(os.path.join(ctx, "d1/f2.bin")) + os.path.getsize(os.path.join(ctx, "big.bin"))
        assert st["files_reused"] == len(files) - 2 and st["bytes_chunked"] == changed
        # 4. the file larger than the arena, now cached
        got, st, _ = commit(eng, tmp, ctx, cache=cache, flags=flags, tag="again")
        _same_layer(got, want)
        assert st["files_reused"] == len(files)
        # 5. duplicate content across a cached and a fresh file: n_unique dedups across the union
        with open(os.path.join(ctx, "dup", "a.bin"), "rb") as f:
            same = f.read()
        with open(os.path.join(ctx, "dup", "c.bin"), "wb") as f:
            f.write(same)
        want, _, _ = commit(eng, tmp, ctx, cache=False, flags=flags, tag="ref3")
        got, st, _ = commit(eng, tmp, ctx, cache=cache, flags=flags, tag="dup")
        _same_layer(got, want)
        assert st["files_reused"] == len(files) and got["n_chunks"] > got["n_unique"]


_SAVE = """
import sys
sys.path.insert(0, {root!r})
from makisu_b200 import host
from tests.test_gpu_commit_chunk_cache import _engine
from tests.test_host_chunk_cache_cpu import commit
with _engine() as eng:
    cache = host.ChunkCache()
    commit(eng, {tmp!r}, {ctx!r}, cache=cache, flags=host.MKHOST_NO_TAR_DIGEST, with_tar=False)
    cache.save({path!r})
"""


def test_cache_saved_in_one_process_loaded_in_another(tmp_path):
    from makisu_b200 import host
    tmp = str(tmp_path)
    ctx = make_ctx(tmp, seed=8)
    path = os.path.join(tmp, "chunks.cache")
    subprocess.check_call([sys.executable, "-c", _SAVE.format(root=ROOT, tmp=tmp, ctx=ctx, path=path)], cwd=ROOT, timeout=600)
    cache = host.ChunkCache(path)
    assert len(cache) == len(regular_files(ctx))
    with _engine() as eng:
        ref, _, _ = commit(eng, tmp, ctx, cache=False, flags=host.MKHOST_NO_TAR_DIGEST, with_tar=False)
        got, st, _ = commit(eng, tmp, ctx, cache=cache, flags=host.MKHOST_NO_TAR_DIGEST, with_tar=False)
    _same_layer(got, ref)
    assert st["files_reused"] == st["files_total"] and st["bytes_uploaded"] == 0


def _fill(eng, data):
    ptr, cap, aid = eng.arena_acquire()
    assert cap >= data.size
    C.memmove(ptr, data.ctypes.data, data.size)
    return aid


def _ext(off, n):
    from makisu_b200.abi import Extent, MKSNAP_X_CDC
    e = Extent()
    e.arena_off, e.len, e.flags = off, n, MKSNAP_X_CDC
    return e


def test_engine_chunks_add_equals_chunking():
    """One session that chunks A and B equals one that chunks A and appends B's digests; appended rows end at
    UINT64_MAX; overflow past max_chunks fails finish; more than MKSNAP_CHUNKS_ADD_MAX rows per call is refused."""
    from makisu_b200.abi import MKSNAP_CHUNKS_ADD_MAX, MksnapError
    rng = np.random.default_rng(1)
    a = rng.integers(0, 256, 700_000, dtype=np.uint8)
    b = rng.integers(0, 256, 500_000, dtype=np.uint8)
    arena = np.zeros(2 << 20, dtype=np.uint8)
    arena[:a.size] = a
    off_b = (a.size + 511) // 512 * 512
    arena[off_b:off_b + b.size] = b
    used = (off_b + b.size + 511) // 512 * 512
    with _engine(arena=4 << 20) as eng:
        p = eng.get_cdc()
        assert (p.min_size, p.normal_size, p.max_size, p.strict_bits, p.loose_bits) == (4096, 16384, 131072, 16, 12)
        eng.begin()
        eng.arena_submit(_fill(eng, arena), used, [_ext(0, a.size), _ext(off_b, b.size)])
        both = eng.finish()
        eng.begin()  # B alone: its digests
        eng.arena_submit(_fill(eng, arena), used, [_ext(off_b, b.size)])
        rb = eng.finish()
        _, dig_b = eng.get_chunks(rb.n_chunks)
        eng.begin()  # A chunked, B appended
        eng.arena_submit(_fill(eng, arena), used, [_ext(0, a.size)])
        eng.chunks_add(dig_b)
        got = eng.finish()
        assert (bytes(got.root), got.n_chunks, got.n_unique) == (bytes(both.root), both.n_chunks, both.n_unique)
        ends, dig = eng.get_chunks(got.n_chunks)
        n_a = got.n_chunks - rb.n_chunks
        assert (ends[n_a:] == np.uint64(2 ** 64 - 1)).all() and (ends[:n_a] < 2 ** 63).all()
        assert (dig[n_a:] == dig_b).all()
        with pytest.raises(MksnapError, match="E_CAPACITY"):
            eng.begin()
            eng.chunks_add(np.zeros((MKSNAP_CHUNKS_ADD_MAX + 1, 32), dtype=np.uint8))
    with _engine(arena=4 << 20, max_chunks=100) as eng:
        eng.begin()
        eng.chunks_add(np.ones((60, 32), dtype=np.uint8))
        eng.chunks_add(np.ones((60, 32), dtype=np.uint8))  # 120 > 100 rows
        with pytest.raises(MksnapError, match="E_CAPACITY"):
            eng.finish()
        eng.begin()  # the handle is usable afterwards
        rows = rng.integers(0, 256, (50, 32), dtype=np.uint8)
        eng.chunks_add(rows)
        r = eng.finish()
        assert (r.n_chunks, r.n_unique) == (50, 50)
        assert (eng.get_table(50) == rows[np.lexsort(rows.T[::-1])]).all()  # sorted by digest bytes


def test_engine_spans_zero_the_rest_and_refuse_extents_outside():
    from makisu_b200.abi import MksnapError
    rng = np.random.default_rng(2)
    data = rng.integers(1, 256, 1 << 20, dtype=np.uint8)  # no zero byte: every zero read back was written by the engine
    spans = [(4096, 65536), (200_000, 100_000 // 16 * 16), (900_000, 16)]
    with _engine() as eng:
        eng.begin()
        with pytest.raises(MksnapError, match="E_INVAL"):  # an extent that reaches beyond its span
            eng.arena_submit_spans(_fill(eng, data), data.size, spans, [_ext(4096, 70_000)])
        eng.begin()  # reclaims the arena the refused submit held
        for bad in ([(8, 16)], [(4096, 100), (0, 16)], [(0, data.size + 16)]):  # unaligned, out of order, beyond used
            with pytest.raises(MksnapError, match="E_INVAL"):
                eng.arena_submit_spans(_fill(eng, data), data.size, bad, [])
            eng.begin()
        h2d0 = eng.stats().h2d_bytes
        eng.arena_submit_spans(_fill(eng, data), data.size, spans, [_ext(4096, 60_000), _ext(200_000, 50_000)])
        r = eng.finish()
        assert eng.stats().h2d_bytes - h2d0 < sum(n for _, n in spans) + 4096  # the spans and the tables
        got = eng.device_download(0, 0, data.size)
        want = np.zeros_like(data)
        for o, n in spans:
            want[o:o + n] = data[o:o + n]
        assert (got == want).all()
        # the chunks equal those of a full upload of the same extents
        eng.begin()
        eng.arena_submit(_fill(eng, data), data.size, [_ext(4096, 60_000), _ext(200_000, 50_000)])
        full = eng.finish()
        assert (bytes(r.root), r.n_chunks) == (bytes(full.root), full.n_chunks)
