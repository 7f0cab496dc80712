"""GPU: gunzip on the device (mksnap_gunzip_*) and update_from_tar(MKHOST_GUNZIP) on an H100.

Parity with Go's gzip reader (tests/gzip_corpus.py: zlib's inflate, Go's framing rules) on the generated corpus, a
multi-window pgzip-shaped blob of more than 1 GiB and a 64 MiB single-segment blob; a handful of malformed blobs from
the CPU fuzz, each followed by a valid blob on the same handle; and the GPU ingest of gzip layers against the
uncompressed ingest of zlib's output."""
import gzip
import random
import zlib

import numpy as np
import pytest

from tests import gzip_corpus as gc

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def eng():
    from makisu_b200.abi import Engine
    e = Engine(device=0, device_arena_bytes=64 << 20, n_host_arenas=2, host_arena_bytes=8 << 20, max_extents=1 << 14)
    yield e
    e.close()


def _lib():
    from makisu_b200 import abi
    return gc.bind(abi.load())


def _check(eng, blob, chunk=1 << 20):
    want = gc.go_gunzip(blob)
    rc, got, info = gc.engine_gunzip(_lib(), eng.h, blob, chunk)
    if want is None:
        assert rc == gc.MKSNAP_E_DATA
    else:
        assert rc == 0 and got == want
        assert info.out_bytes == len(want) and info.gz_bytes == len(blob)
    return info


@pytest.mark.parametrize("name", [n for n, _ in gc.corpus()])
def test_corpus_parity(eng, name):
    blob = dict(gc.corpus())[name]
    _check(eng, blob, chunk=100_000)


def test_alpine_fixture(eng):
    import hashlib
    import os
    blob = open(os.path.join(os.path.dirname(__file__), "golden", "alpine_test_layer.tar.gz"), "rb").read()
    assert hashlib.sha256(blob).hexdigest() == "393ccd5c4dd90344c9d725125e13f636ce0087c62f5ca89050faaacbb9e3ed5b"
    info = _check(eng, blob)
    assert (info.n_members, info.n_segments) == (1, 1)


def _big_data(n, seed):
    rng = random.Random(seed)
    base = np.frombuffer(gc.mixed(rng, 48 << 20), dtype=np.uint8)
    noise = np.random.default_rng(seed).integers(0, 256, n, dtype=np.uint8)
    reps = -(-n // base.size)
    d = np.tile(base, reps)[:n].copy()
    d[(np.arange(n) // 65536) % 5 == 4] = noise[(np.arange(n) // 65536) % 5 == 4]  # every 5th 64 KiB incompressible
    return d.tobytes()


def test_pgzip_multi_window_over_1gib(eng):
    data = _big_data((1 << 30) + 12345, 3)
    blob = gc.pgzip(data, level=1)
    rc, got, info = gc.engine_gunzip(_lib(), eng.h, blob, chunk=96 << 20)
    assert rc == 0 and info.out_bytes == len(data) and info.n_segments >= 1025 and info.n_members == 1
    assert got == data
    assert zlib.crc32(got) == zlib.crc32(data)


def test_single_segment_64mib(eng):
    data = _big_data(64 << 20, 4)
    blob = gzip.compress(data, 6)
    rc, got, info = gc.engine_gunzip(_lib(), eng.h, blob)
    assert rc == 0 and got == data and (info.n_segments, info.n_members) == (1, 1)


def test_malformed_then_valid_on_the_same_handle(eng):
    cases = [c for c in gc.fuzz_cases(400, seed=7) if gc.go_gunzip(c) is None][:12]
    good = dict(gc.corpus())["multi_member"]
    assert len(cases) == 12
    for c in cases:
        rc, _, _ = gc.engine_gunzip(_lib(), eng.h, c)
        assert rc == gc.MKSNAP_E_DATA
        _check(eng, good)


@pytest.mark.parametrize("flags", [0, 2, 32, 34, 1])
def test_update_from_tar_gunzip(tmp_path, flags):
    import os
    from makisu_b200.abi import Engine
    if flags & 32 and os.geteuid() != 0:
        pytest.skip("MKHOST_UNTAR: chown needs root")

    def make_engine(arena_bytes):
        return Engine(device=0, device_arena_bytes=arena_bytes, n_host_arenas=2, host_arena_bytes=arena_bytes,
                      max_extents=1 << 12)

    # 4 MiB arenas: every member fits one, so MKHOST_UNTAR takes every layer; members split over arenas are covered by
    # the CPU mock (1 MiB arenas) and by the uncompressed ingest tests
    for name, blob in gc.layer_blobs():
        gc.check_ingest(make_engine, str(tmp_path), name, blob, flags, arena_bytes=4 << 20)
