"""-m gpu: the multi-engine calls of libmkhost (mkhost_context_crc32_multi, mkhost_memfs_commit_layers_multi) on
libmksnap.  The scenarios of tests/mock_engine/multi_engine_cases.py -- each compares 1, 2, 3 and 5 engines with the
single-engine call -- with every engine on device 0 and arenas of 1 MiB or less, so each engine submits several
times; then the cacheID and a warm MKHOST_FILE_DIGESTS batch with one engine per device (skipped with fewer than two)."""
import os

import pytest

from tests.mock_engine import multi_engine_cases as cases

pytestmark = pytest.mark.gpu


def make_engine(arena_bytes, max_extents=1 << 12, max_chunks=0, cdc=None, device=0):
    from makisu_b200.abi import Engine

    class _Engine(Engine):
        def work(self):
            s = self.stats()
            return s.kernel_launches, s.h2d_bytes

    return _Engine(device=device, device_arena_bytes=arena_bytes, n_host_arenas=2, host_arena_bytes=arena_bytes,
                   max_extents=max_extents, max_chunks=max_chunks, cdc=cdc)


@pytest.mark.parametrize("scenario", cases.ALL)
def test_multi_engine_one_device(scenario, tmp_path):
    getattr(cases, scenario)(make_engine, str(tmp_path))


def test_one_engine_per_device(tmp_path):
    import torch
    n_dev = torch.cuda.device_count()
    if n_dev < 2:
        pytest.skip("needs two or more GPUs")
    from makisu_b200 import host
    tmp = str(tmp_path)
    k = [0]

    def make(arena, **kw):  # round robin over the devices
        k[0] += 1
        return make_engine(arena, device=(k[0] - 1) % n_dev, **kw)

    ctx = cases._crc_ctx(tmp)
    caches = (host.CrcCache(), host.CrcCache())
    for _ in range(2):
        k[0] = 0
        cases._cache_id_against(make, ctx, ["."], 256 << 10, n_dev, caches)
    bctx = cases.cases.make_ctx(os.path.join(tmp, "b"))
    run = cases.cases.Runner(make, os.path.join(tmp, "b"), bctx)
    cache = host.ChunkCache()
    for _ in range(2):  # cold, then warm: remembered and foreign rows on engine 0
        k[0] = 0
        cases._check_batch(run, make, n_dev, cache, host.MKHOST_FILE_DIGESTS)
