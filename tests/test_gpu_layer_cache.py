"""-m gpu: the incremental layer ingest (mkhost_memfs_update_from_tars_cached) on libmksnap.  The scenarios of
tests/layer_cache_cases.py -- each compares the cached run with update_from_tars_indexed on a fresh tree -- and two
larger ones: a 256 MiB pgzip layer and a 64 MiB single-member gzip layer cold then warm, and a warm run whose replayed
chunk rows take more than one mksnap_chunks_add batch (MKSNAP_CHUNKS_ADD_MAX)."""
import os

import numpy as np
import pytest

from tests import gzip_corpus as gc
from tests import gzip_index as gi
from tests import layer_cache_cases as cases

pytestmark = pytest.mark.gpu


def make_engine(arena_bytes, cdc=None, max_chunks=0, max_extents=1 << 12):
    from makisu_b200.abi import Engine
    return Engine(device=0, device_arena_bytes=arena_bytes, n_host_arenas=2, host_arena_bytes=arena_bytes,
                  max_extents=max_extents, max_chunks=max_chunks, cdc=cdc)


@pytest.mark.parametrize("scenario", cases.ALL)
def test_layer_cache(scenario, tmp_path):
    getattr(cases, scenario)(make_engine, str(tmp_path))


@pytest.mark.skipif(os.geteuid() != 0, reason="MKHOST_UNTAR applies owners (chown)")
def test_layer_cache_untar(tmp_path):
    cases.untar(make_engine, str(tmp_path))


def test_large_layers_cold_then_warm(tmp_path):
    from makisu_b200 import host
    layers = [("pgzip_256m", gc.pgzip(gi.layer_tar(256 << 20, 21), block=1 << 20, level=1), True),
              ("single_64m", gi.single(gi.layer_tar(64 << 20, 22)), True)]
    paths = cases.write_blobs(str(tmp_path / "blobs"), layers)
    keys = ["pgzip", "single"]
    run = cases.Runner(make_engine, str(tmp_path))
    lc = host.LayerCache()
    outs, st, _ = run.check(paths, layers, keys, host.MKHOST_FILE_DIGESTS, lc, arena=64 << 20, max_chunks=1 << 18)
    assert st["layers_recorded"] == 2 and st["blob_bytes_read"] == sum(len(b) for _, b, _ in layers), st
    warm, st, _ = run.check(paths, layers, keys, host.MKHOST_FILE_DIGESTS, lc, arena=64 << 20, max_chunks=1 << 18)
    assert warm == outs
    assert st["layers_replayed"] == 2 and st["blob_bytes_read"] == 0 and st["chunks_appended"] == outs[0]["n_chunks"], st


def test_warm_run_appends_more_than_one_batch(tmp_path):
    """Small chunks (about 1 KiB) over two 128 MiB layers: more replayed rows than one mksnap_chunks_add call takes."""
    from makisu_b200 import abi, host
    from tests import apply_layers as al
    rng = np.random.default_rng(31)
    layers = [("random_%d" % i, al.tar_of([("data%d" % i, "d", None)] + [("data%d/f%02d" % (i, k), "f",
                                                                          rng.integers(0, 256, 8 << 20, dtype=np.uint8).tobytes())
                                                                         for k in range(16)]), False) for i in range(2)]
    paths = cases.write_blobs(str(tmp_path / "blobs"), layers)
    cdc = abi.CdcParams(256, 1024, 8192, 11, 9)
    run = cases.Runner(make_engine, str(tmp_path))
    lc = host.LayerCache()
    kw = dict(arena=32 << 20, cdc=cdc, max_chunks=1 << 19)
    outs, _, _ = run.check(paths, layers, ["a", "b"], 0, lc, **kw)
    assert outs[0]["n_chunks"] > 2 * 65536, outs[0]["n_chunks"]
    warm, st, _ = run.check(paths, layers, ["a", "b"], 0, lc, **kw)
    assert warm == outs and st["layers_replayed"] == 2 and st["chunks_appended"] == outs[0]["n_chunks"], st
