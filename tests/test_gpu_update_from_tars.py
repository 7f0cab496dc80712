"""-m gpu: mkhost_memfs_update_from_tars on the device engine.  A run of layers (tests/apply_layers.py: whiteouts,
overwrites, a hard link to an earlier layer, an empty layer, gzip and plain blobs, a member larger than the arena)
equals one update_from_tar call per layer -- per-layer DiffID (also against hashlib), entries, tar bytes, tree, file
digests -- and the run's chunk table equals one session over every layer's files.  A run larger than the stream log
(1 GiB) is hashed in flushes on the device.  Deferred streams past 2^32 bits: tests/test_gpu_stream_defer.py."""
import hashlib
import os

import numpy as np
import pytest

from tests import apply_layers as al

pytestmark = pytest.mark.gpu


def make_engine(arena_bytes, max_extents=1 << 12, max_chunks=0):
    from makisu_b200.abi import Engine
    return Engine(device=0, device_arena_bytes=arena_bytes, n_host_arenas=2, host_arena_bytes=arena_bytes,
                  max_extents=max_extents, max_chunks=max_chunks)


@pytest.mark.parametrize("flags", ["tar-digest", "file-digests", "no-tar-digest"])
def test_run_equals_single_calls(flags, tmp_path):
    from makisu_b200 import host
    f = {"tar-digest": 0, "file-digests": host.MKHOST_FILE_DIGESTS, "no-tar-digest": host.MKHOST_NO_TAR_DIGEST}[flags]
    res = al.check_run(make_engine, str(tmp_path), al.layer_run(), f)
    if not f:
        digests = [r["tar_digest"] for r in res]
        assert len(set(digests)) == len(digests)


@pytest.mark.skipif(os.geteuid() != 0, reason="MKHOST_UNTAR applies owners (chown)")
def test_run_equals_single_calls_untar(tmp_path):
    from makisu_b200 import host
    al.check_run(make_engine, str(tmp_path), al.layer_run(big=False), host.MKHOST_UNTAR | host.MKHOST_FILE_DIGESTS)


def test_run_larger_than_the_stream_log(tmp_path):
    """Three layers of 400 MiB (1.2 GiB of DiffID bytes, more than the 1 GiB log), 64 MiB arenas: the log fills during
    the third layer and is hashed on the device before the rest of it is appended."""
    from makisu_b200 import host
    rng = np.random.default_rng(77)
    paths, want = [], []
    for i in range(3):
        blob = al.tar_of([("data/l%d.bin" % i, "f", rng.integers(0, 256, 400 << 20, dtype=np.uint8).tobytes()),
                          ("data/small%d" % i, "f", b"x" * (i + 1))])
        paths.append(str(tmp_path / ("l%d.tar" % i)))
        open(paths[-1], "wb").write(blob)
        want.append("sha256:" + hashlib.sha256(blob).hexdigest())
        del blob
    root = tmp_path / "root"
    root.mkdir()
    fh = [open(p, "rb") for p in paths]
    try:
        with make_engine(64 << 20, max_chunks=1 << 18) as e:   # the run's chunk table is one session's: ~80k chunks
            res = host.MemFS(str(root)).update_from_tars(e, al.NOW, [f.fileno() for f in fh])
            assert e.stats().ms_flush > 0
    finally:
        for f in fh:
            f.close()
    assert [r["tar_digest"] for r in res] == want
    (tmp_path / "described").mkdir()
    fs = host.MemFS(str(tmp_path / "described"))       # the same merges without a GPU
    for p, r in zip(paths, res):
        with open(p, "rb") as f:
            assert r["n_entries"] == len(fs.describe_update_from_tar(al.NOW, f.fileno()))
