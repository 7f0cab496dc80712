"""GPU: the indexed gunzip (mksnap_gunzip_open_indexed / mksnap_gunzip_get_index) on an H100.

The scenarios of the CPU file (tests/test_host_gunzip_index_cpu.py) against the device engine, then what only the device
shows: a 1 GiB single member, recorded and reopened with its index, bit for bit against zlib, with the peak device memory
of both opens bounded by include/mksnap.h's statement rather than by the member size; the host ingest through the
gzip index cache against the uncompressed ingest."""
import time
import zlib

import pytest

from tests import gzip_index as gi
from tests import test_host_gunzip_index_cpu as cpu

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def eng():
    from makisu_b200.abi import Engine
    e = Engine(device=0, device_arena_bytes=64 << 20, n_host_arenas=2, host_arena_bytes=8 << 20, max_extents=1 << 14)
    yield e
    e.close()


def _lib():
    from makisu_b200 import abi
    return gi.bind(abi.load())


@pytest.mark.parametrize("scenario", ["corpus", "all_block_starts", "bad_indexes", "contract", "malformed"])
def test_index_scenarios(eng, scenario):
    getattr(cpu, scenario)(_lib(), eng.h)


def test_fuzz_random_indexes(eng):
    cpu.fuzz(_lib(), eng.h, n=600)


def test_update_from_tar_indexed_cold_warm(tmp_path):
    from makisu_b200.abi import Engine

    def make_engine(arena_bytes):
        return Engine(device=0, device_arena_bytes=arena_bytes, n_host_arenas=2, host_arena_bytes=arena_bytes,
                      max_extents=1 << 12)
    assert gi.check_ingest_indexed(make_engine, str(tmp_path)) >= 2


def _free():
    import torch
    return torch.cuda.mem_get_info(0)[0]


class _PeakSampler:
    """The least free device memory seen while the block runs (cudaMemGetInfo every millisecond from a thread)."""

    def __enter__(self):
        import threading
        self.low, self.stop = _free(), False

        def run():
            while not self.stop:
                self.low = min(self.low, _free())
                time.sleep(0.001)
        self.t = threading.Thread(target=run)
        self.t.start()
        return self

    def __exit__(self, *a):
        self.stop = True
        self.t.join()


def test_1gib_single_member_recorded_then_indexed(eng):
    from tests.test_gpu_gunzip import _big_data
    data = _big_data(1 << 30, 6)
    blob = gi.single(data, 6)  # the level of bench_gunzip_index.py
    lib = _lib()
    free0 = _free()
    # peak device memory of the recording open and its reads: the blob, 40 bytes per candidate, the record buffer,
    # 8 bytes per cut and one window of max(256 MiB, largest piece) at 3 bytes per output byte (include/mksnap.h) --
    # a plain open of this member would need a 3 GiB window alone
    with _PeakSampler() as peak:
        rc, got, info, ix, pts = gi.engine_gunzip_indexed(lib, eng.h, blob, None, 256 << 20)
    grew = free0 - peak.low
    assert rc == 0 and info.n_members == 1 and info.out_bytes == len(data)
    assert got == data
    got = None
    assert info.n_segments >= 512 and ix.points_recorded == len(pts), (info.n_segments, ix.n_points)
    n_cand_bound = 1024 + len(blob) // (1 << 20)  # false candidates in compressed data are rare
    bound = len(blob) + 48 * (n_cand_bound + len(pts)) + 24 * 65536 + 3 * (256 << 20) + (64 << 20)
    assert grew <= bound, (grew, bound)
    with _PeakSampler() as peak:
        rc, got, info2, ix2, pts2 = gi.engine_gunzip_indexed(lib, eng.h, blob, pts, 256 << 20)
    assert free0 - peak.low <= bound, (free0 - peak.low, bound)
    assert rc == 0 and ix2.points_linked == len(pts) and info2.n_segments == info.n_segments
    assert zlib.crc32(got) == zlib.crc32(data) and got == data
