"""-m gpu: the batched incremental layer commit (mkhost_memfs_commit_layers_cached) on libmksnap.  The scenarios of
tests/commit_layers_cases.py -- each compares a batch with one commit_copy_ops_cached call per layer on a fresh tree --
and the batch's chunk table against the oracle over the union of the layers' files."""
import os

import numpy as np
import pytest

from tests import commit_layers_cases as cases

pytestmark = pytest.mark.gpu


def make_engine(arena_bytes, cdc=None, max_extents=1 << 12):
    from makisu_b200.abi import Engine

    class _Engine(Engine):
        def work(self):
            s = self.stats()
            return s.kernel_launches, s.h2d_bytes

        def mark(self):
            self._h2d0 = self.stats().h2d_bytes

        def uploaded(self):
            return self.stats().h2d_bytes - self._h2d0

    return _Engine(device=0, device_arena_bytes=arena_bytes, n_host_arenas=2, host_arena_bytes=arena_bytes,
                   max_extents=max_extents, cdc=cdc)


@pytest.mark.parametrize("scenario", cases.ALL)
def test_commit_layers(scenario, tmp_path):
    getattr(cases, scenario)(make_engine, str(tmp_path))


def test_batch_chunk_table_against_the_oracle(tmp_path):
    """root and n_unique of a cold, a warm and an uncached batch equal the oracle's table over every file the layers
    copy (the table is sorted and unique: how often a file occurs does not change it)."""
    from makisu_b200 import host
    from oracle import lib as olib
    tmp = str(tmp_path)
    ctx = cases.make_ctx(tmp)
    bodies = [open(p, "rb").read() for p in cases.sources(ctx, cases.LAYERS)]
    offs, pos = [], 0
    for b in bodies:
        offs.append(pos)
        pos += (len(b) + 511) // 512 * 512
    arena = np.zeros(max(pos, 512), dtype=np.uint8)
    for o, b in zip(offs, bodies):
        arena[o:o + len(b)] = np.frombuffer(b, dtype=np.uint8)
    want = olib.chunk_table(arena, offs, [len(b) for b in bodies])
    run = cases.Runner(make_engine, tmp, ctx)
    cache = host.ChunkCache()
    for c in (None, cache, cache):
        _, outs, _, _ = run.batch(make_engine(cases.ARENA), c, cases.LAYERS, host.MKHOST_NO_TAR_DIGEST, with_tar=False)
        assert all((o["root"], o["n_unique"]) == (want["root"], want["n_unique"]) for o in outs)
    assert len(cache) == len(bodies)
